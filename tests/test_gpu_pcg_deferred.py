"""The fused pipelined-CG iteration updates p and x every second iteration (DESIGN.md section 4a): an even
iteration leaves them and keeps r_k beside r_{k+1}, the odd one after it catches up on both, and a solve
whose last update was even finishes them after the loop.  Checked against the two-kernel loop (pcg_fused=0)
on one solver matrix, after every solve, for x and for the solver's own r and p vectors:

* fixed iteration counts 1-5 (issued one by one) and 16, 17 (graph replays), so the loop ends after an even
  and after an odd update, with warm-up 0 and 2, a nonzero x0 and several solves in a row on one solver;
* convergence met on even and on odd iterations;
* 27-point boxes with every row in a slice and with tile rows (the tail update), and a 7-point box, each with
  coded diagonals and with fp64 ones (symdiag_codes=0); and the fixed counts against the oracle.
"""
import numpy as np
import pytest

from test_gpu_pcg_fused import BOXES, OPTS

pytestmark = pytest.mark.gpu

OPTIONS = dict(OPTS, symdiag_codes=1)


@pytest.fixture
def options(ab):
    def set_(**kw):
        for k, v in dict(OPTIONS, **kw).items():
            ab.set_option(k, v)
    yield set_
    for k, v in OPTIONS.items():
        ab.set_option(k, v)


def _matrix(ab, box, seed):
    """Off-diagonal values from five levels in [-1, -0.75] and a diagonal half a unit above the neighbour count:
    strictly diagonally dominant, few enough distinct values for the codes, and Laplacian-like, so the fixed
    counts stay far from convergence (past it the two loops differ at the attainable accuracy)."""
    n, r, c, _ = BOXES[box]()
    rng = np.random.default_rng(seed)
    v = -1.0 + rng.integers(0, 5, len(r)) / 16.0
    v[r == c] = 6.5 if box == "7pt" else 26.5
    return ab.SymCsrMatrix.init_real_double(n, r, c, v).dsymv_init(0.5)


def _device(ptr, n):
    """n doubles at device address ptr (the solve has synchronised its stream)."""
    import torch

    class _View:
        __cuda_array_interface__ = {"shape": (n,), "typestr": "<f8", "data": (ptr, False), "version": 2}
    return torch.as_tensor(_View(), device="cuda").cpu().numpy().copy()


def _solve(cg, A, b, x0=None, **kw):
    x = A.vector()
    if x0 is not None:
        x.x[:] = x0
    code = cg.solve_pipelined(b, x, **kw)
    n = A.c.nownedrows
    return dict(code=code, nits=cg.c.niterations, rnrm2=cg.c.rnrm2, x=x.x.copy(),
                r=_device(cg.c.d_r, n), p=_device(cg.c.d_p, n))


def _same(got, want, scale):
    """Same return code and iterations; x to 1e-10 of its size.  r and p: rounding differences of the two loops'
    dot sums grow from |r_0| (scale), while a stale r buffer or a missing p update is off by the vector's size."""
    assert (got["code"], got["nits"]) == (want["code"], want["nits"])
    assert got["rnrm2"] == pytest.approx(want["rnrm2"], rel=1e-6)
    assert np.abs(got["x"] - want["x"]).max() <= 1e-10 * np.abs(want["x"]).max()
    for v in ("r", "p"):
        assert np.abs(got[v] - want[v]).max() <= 1e-3 * np.abs(want[v]).max() + 1e-12 * scale, v


def _run_both(ab, A, options, codes, cases):
    res = {}
    for on in (1, 0):
        options(pcg_fused=on, symdiag_codes=codes)
        cg = ab.SolverCuda(A)          # a fresh solver per setting: the cases run in the same order on each
        inf = cg.info()
        assert (inf["spmv_symdiag_codes"] > 0) == bool(codes)
        res[on] = [_solve(cg, A, b, **kw) for b, kw in cases]
        assert cg.info()["pcg_fused"] == on
        cg.free()
    return res


@pytest.mark.parametrize("codes", [1, 0])
@pytest.mark.parametrize("box", sorted(BOXES))
def test_fixed_counts(box, codes, ab, options, oracle):
    A = _matrix(ab, box, seed=101)
    n = A.c.nownedrows
    b = A.vector()
    b.x[:] = np.random.default_rng(102).standard_normal(len(b.x))
    x0 = np.random.default_rng(103).standard_normal(len(b.x))
    cases = [(b, dict(maxits=m)) for m in (1, 2, 3, 4, 5, 16, 17)]
    cases += [(b, dict(maxits=5, warmup=2)), (b, dict(maxits=16, warmup=2)), (b, dict(maxits=17, warmup=0)),
              (b, dict(maxits=4, x0=x0)), (b, dict(maxits=17, x0=x0)), (b, dict(maxits=3))]
    res = _run_both(ab, A, options, codes, cases)
    scale = np.abs(b.x).max() + np.abs(x0).max()
    for (_, kw), got, want in zip(cases, res[1], res[0]):
        assert got["nits"] == kw["maxits"], kw
        _same(got, want, scale)
    # a second solve of a case on the same solver (after others that ended on either parity)
    _same(res[1][-1], res[1][2], scale)
    csr = (A.frowptr.copy(), A.fcolidx.copy(), A.fa.copy())
    for i in (0, 3, 6):
        m = cases[i][1]["maxits"]
        want = oracle.cg_pipelined(csr, b.x, maxits=m)
        assert want["niterations"] == m
        assert np.abs(res[1][i]["x"][:n] - want["x"][:n]).max() <= 1e-9 * np.abs(want["x"]).max()
    A.free()


@pytest.mark.parametrize("codes", [1, 0])
@pytest.mark.parametrize("box", sorted(BOXES))
def test_converges_on_both_parities(box, codes, ab, options):
    """Tolerances just above the residual of iteration k - 1 stop the loop at k, for four consecutive k.  The
    margin (1e-6) is above the two loops' rounding differences in gamma, far below a step of the residual."""
    A = _matrix(ab, box, seed=111)
    b = A.vector()
    b.x[:] = np.random.default_rng(112).standard_normal(len(b.x))
    options(pcg_fused=0, symdiag_codes=codes)
    cg = ab.SolverCuda(A)
    nits = _solve(cg, A, b, maxits=2000, residualrtol=1e-10)["nits"]
    tols = []
    for k in range(nits - 6, nits - 2):
        _solve(cg, A, b, maxits=k)
        tols.append(cg.c.rnrm2 / cg.c.r0nrm2 * (1 + 1e-6))
    cg.free()
    res = _run_both(ab, A, options, codes, [(b, dict(maxits=2000, residualrtol=t)) for t in tols])
    for got, want in zip(res[1], res[0]):
        assert got["code"] == 0 and got["nits"] < 2000
        _same(got, want, np.abs(b.x).max())
    assert {r["nits"] % 2 for r in res[1]} == {0, 1}
    A.free()
