"""The fused pipelined-CG iteration updates p and x once per group of m iterations (option pcg_group, DESIGN.md
section 4a): the first m - 1 iterations of a group keep their r's in a ring, the last one catches up on p and
x for the whole group, and a solve that stops inside a group finishes it after the loop.  Checked for m = 2, 4,
8 and 16 against the two-kernel loop (pcg_fused=0), for x and for the solver's own r and p vectors:

* fixed counts m - 1, m, m + 1, 2m, 2m + 1 and 3m + m/2, so the loop ends at several places in a group, both
  before the first graph replay and after replays and single iterations, with warm-up 0 and 2 and a nonzero x0;
* convergence met at every place k % m of a group;
* m switched between solves on one solver, and the results of every m compared with those of m = 2;
* 27-point boxes with every row in a slice and with tile rows, and a 7-point box, with coded and fp64 diagonals.
"""
import numpy as np
import pytest

from test_gpu_pcg_deferred import OPTIONS, _matrix, _same, _solve
from test_gpu_pcg_fused import BOXES

pytestmark = pytest.mark.gpu

GROUPS = (2, 4, 8, 16)
DEFAULT_GROUP = 16          # the library's default (PCG_GROUP_DEFAULT in cgcuda.c)


@pytest.fixture
def options(ab):
    base = dict(OPTIONS, pcg_group=DEFAULT_GROUP)

    def set_(**kw):
        for k, v in dict(base, **kw).items():
            ab.set_option(k, v)
    yield set_
    for k, v in base.items():
        ab.set_option(k, v)


def _cases(m):
    return [dict(maxits=k) for k in (m - 1, m, m + 1, 2 * m, 2 * m + 1, 3 * m + m // 2)] + \
        [dict(maxits=2 * m + 1, warmup=2), dict(maxits=m - 1, warmup=2), dict(maxits=m + 1, x0=1),
         dict(maxits=3 * m + m // 2, x0=1, warmup=2)]


def _key(kw):
    return tuple(sorted(kw.items()))


def _close(got, want, bnrm2, scale):
    """_same, unless the reference is already near the attainable accuracy (the 7-point box's longest fixed
    counts), where the two loops' residuals part at the 1e-12 level: then the counts and x."""
    if want["rnrm2"] > 1e-9 * bnrm2:
        _same(got, want, scale)
    else:
        assert (got["code"], got["nits"]) == (want["code"], want["nits"])
        assert np.abs(got["x"] - want["x"]).max() <= 1e-10 * np.abs(want["x"]).max()


def _run(cg, A, b, x0, kw):
    kw = dict(kw)
    return _solve(cg, A, b, x0=x0 if kw.pop("x0", 0) else None, **kw)


@pytest.mark.parametrize("codes", [1, 0])
@pytest.mark.parametrize("box", sorted(BOXES))
def test_fixed_counts(box, codes, ab, options):
    A = _matrix(ab, box, seed=201)
    b = A.vector()
    b.x[:] = np.random.default_rng(202).standard_normal(len(b.x))
    x0 = np.random.default_rng(203).standard_normal(len(b.x))
    scale = np.abs(b.x).max() + np.abs(x0).max()
    options(pcg_fused=0, symdiag_codes=codes)
    cg = ab.SolverCuda(A)
    want = {}
    for m in GROUPS:
        for kw in _cases(m):
            if _key(kw) not in want:
                want[_key(kw)] = _run(cg, A, b, x0, kw)
    cg.free()
    # one fused solver for every group: the group changes between solves
    options(pcg_fused=1, symdiag_codes=codes)
    cg = ab.SolverCuda(A)
    assert (cg.info()["spmv_symdiag_codes"] > 0) == bool(codes)
    got = {}
    for m in GROUPS + (2,):
        ab.set_option("pcg_group", m)
        for kw in _cases(m):
            r = _run(cg, A, b, x0, kw)
            inf = cg.info()
            assert inf["pcg_fused"] == 1 and inf["pcg_group"] == m
            assert r["nits"] == kw["maxits"], (m, kw)
            _close(r, want[_key(kw)], np.linalg.norm(b.x), scale)
            # the same case under another group: the same FMAs, only the dot sums' order may differ
            if _key(kw) in got:
                _close(r, got[_key(kw)], np.linalg.norm(b.x), scale)
            got.setdefault(_key(kw), r)
    cg.free()
    A.free()


@pytest.mark.parametrize("codes", [1, 0])
@pytest.mark.parametrize("box", sorted(BOXES))
def test_converges_at_every_place_in_a_group(box, codes, ab, options):
    """Tolerances just above the residual of iteration k - 1 stop the loop at k, for 16 consecutive k: every
    k % m for each group.  The margin (1e-6) is above the two loops' rounding differences in gamma, far below a
    step of the residual."""
    A = _matrix(ab, box, seed=211)
    b = A.vector()
    b.x[:] = np.random.default_rng(212).standard_normal(len(b.x))
    options(pcg_fused=0, symdiag_codes=codes)
    cg = ab.SolverCuda(A)
    nits = _solve(cg, A, b, maxits=2000, residualrtol=1e-10)["nits"]
    assert nits >= 20
    tols = []
    for k in range(nits - 18, nits - 2):
        _solve(cg, A, b, maxits=k)
        tols.append(cg.c.rnrm2 / cg.c.r0nrm2 * (1 + 1e-6))
    want = [_solve(cg, A, b, maxits=2000, residualrtol=t) for t in tols]
    cg.free()
    options(pcg_fused=1, symdiag_codes=codes)
    cg = ab.SolverCuda(A)
    for m in GROUPS:
        ab.set_option("pcg_group", m)
        got = [_solve(cg, A, b, maxits=2000, residualrtol=t) for t in tols]
        assert cg.info()["pcg_group"] == m
        for g, w in zip(got, want):
            assert g["code"] == 0 and g["nits"] < 2000
            _same(g, w, np.abs(b.x).max())
        assert {g["nits"] % m for g in got} == set(range(m))
    cg.free()
    A.free()


def test_option_and_bytes(ab, options):
    """Only groups of 2, 4, 8 and 16 are accepted; the profiled iteration's bytes are the group's average."""
    for bad in (0, 1, 3, 6, 32):
        with pytest.raises(Exception):
            ab.set_option("pcg_group", bad)
    A = _matrix(ab, "27pt-full", seed=221)
    b = A.vector()
    b.x[:] = 1.0
    for m in GROUPS:
        options(pcg_fused=1, symdiag_codes=1, pcg_group=m)
        cg = ab.SolverCuda(A)
        _solve(cg, A, b, maxits=2 * m + 1)
        inf = cg.info()
        assert inf["pcg_fused"] == 1 and inf["pcg_group"] == m and inf["spmv_ntiles"] == 0
        rows, nd = inf["spmv_slice_rows"], inf["spmv_symdiag_diagonals"]
        assert inf["spmv_min_bytes"] == rows * nd + rows * (72 * m + 32) // m
        assert inf["pcg_fused_min_bytes"] == rows * (nd + 96)
        cg.free()
    A.free()
