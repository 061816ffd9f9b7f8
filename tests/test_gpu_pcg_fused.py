"""The fused pipelined-CG iteration (option "pcg_fused", DESIGN.md section 4a) on the H100.

* Against the two-kernel loop (pcg_fused=0) on the same solver matrix: a 27-point box whose rows are all in
  slices (one kernel per iteration), the ragged 27-point box of test_gpu_symdiag.py (tile rows: the tile
  kernel and their update run in front of the fused kernel) and a 7-point box.  Same return code, same
  iterations, x to 1e-10; and against the oracle's pipelined CG.
* Loop edges: odd and even maxits with the tolerances off and a second solve on the same solver (graph
  replay from parity 0 again), convergence on an odd iteration, maxits=0, warm-up 0 and 2, nonzero x0,
  pcg_fused switched between two solves on one solver.
* Which matrices take the path (info["pcg_fused"]) and the launches per replayed iteration.
"""
import numpy as np
import pytest

from acg_b200 import matgen as mg
from test_gpu_kernel_variants import DEFAULTS, big_stencil, rmat

pytestmark = pytest.mark.gpu

OPTS = dict(DEFAULTS, spmv_symdiag=1, pcg_fused=1)


@pytest.fixture
def options(ab):
    def set_(**kw):
        for k, v in dict(OPTS, **kw).items():
            ab.set_option(k, v)
    yield set_
    for k, v in OPTS.items():
        ab.set_option(k, v)


BOXES = {
    "27pt-full": lambda: mg.stencil3d_27pt(32, 20, 19),      # n % 32 == 0: every row in a slice
    "27pt-ragged": lambda: mg.stencil3d_27pt(21, 20, 19),    # tile rows after the slices
    "7pt": lambda: mg.laplace3d_7pt(31, 17, 23),
}


def _matrix(ab, box, seed=13):
    n, r, c, _ = BOXES[box]()
    rng = np.random.default_rng(seed)
    v = rng.standard_normal(len(r))
    v[r == c] += 30.0
    return ab.SymCsrMatrix.init_real_double(n, r, c, v).dsymv_init(0.5)


def _rhs(A, seed=14):
    b = A.vector()
    b.x[:] = np.random.default_rng(seed).standard_normal(len(b.x))
    return b


def _solve(cg, A, b, x0=None, **kw):
    x = A.vector()
    if x0 is not None:
        x.x[:] = x0
    code = cg.solve_pipelined(b, x, **kw)
    return code, cg.c.niterations, cg.c.rnrm2, x.x.copy()


def _same(got, want, tol=1e-10):
    (c1, it1, r1, x1), (c0, it0, r0, x0) = got, want
    assert c1 == c0 and it1 == it0, (got[:3], want[:3])
    assert np.abs(x1 - x0).max() <= tol * np.abs(x0).max()
    assert r1 == pytest.approx(r0, rel=1e-6)


@pytest.mark.parametrize("box", sorted(BOXES))
def test_fused_matches_two_kernel_loop_and_oracle(box, ab, options, oracle):
    A = _matrix(ab, box)
    b = _rhs(A)
    csr = (A.frowptr.copy(), A.fcolidx.copy(), A.fa.copy())
    res = {}
    cg = ab.SolverCuda(A)
    inf = cg.info()
    assert inf["spmv_symdiag_diagonals"] > 0
    assert (inf["spmv_ntiles"] == 0) == (box == "27pt-full")
    for on in (1, 0):
        options(pcg_fused=on)
        res[on] = _solve(cg, A, b, maxits=2000, residualrtol=1e-10)
        assert cg.info()["pcg_fused"] == on
    assert res[1][0] == 0 and res[1][1] > 0 and res[1][2] / cg.c.r0nrm2 < 1e-10
    _same(res[1], res[0])
    want = oracle.cg_pipelined(csr, b.x, maxits=2000, rtol=1e-10)
    assert want["status"] == 0 and want["niterations"] == res[1][1]
    assert np.abs(res[1][3] - want["x"]).max() <= 1e-9 * np.abs(want["x"]).max()
    cg.free()
    A.free()


@pytest.mark.parametrize("box", ["27pt-full", "27pt-ragged"])
def test_loop_edges(box, ab, options):
    A = _matrix(ab, box, seed=21)
    b = _rhs(A, seed=22)
    x0 = np.random.default_rng(23).standard_normal(len(b.x))
    # fixed counts stay short of convergence (about 26 iterations to 1e-10 here): past it, the two loops'
    # iterates differ at the attainable accuracy of pipelined CG rather than by the order of the sums
    cases = [dict(maxits=13), dict(maxits=14), dict(maxits=13), dict(maxits=3), dict(maxits=1),
             dict(maxits=12, warmup=2), dict(maxits=12, warmup=0), dict(maxits=15, x0=x0),
             dict(maxits=500, residualrtol=1e-10, x0=x0)]
    results = {}
    for on in (1, 0):
        options(pcg_fused=on)
        cg = ab.SolverCuda(A)          # a fresh solver per setting: the cases run in the same order on each
        results[on] = [_solve(cg, A, b, **kw) for kw in cases]
        assert cg.info()["pcg_fused"] == on
        cg.free()
    for kw, got, want in zip(cases, results[1], results[0]):
        _same(got, want)
    assert results[1][0][1] == 13 and results[1][1][1] == 14 and results[1][2][1] == 13
    # the same solve twice on one solver: the second replays the cached graph from parity 0 (the sums of the
    # dots are only equal up to the order of the per-CTA atomics)
    _same(results[1][2], results[1][0])
    A.free()


def test_converges_on_odd_and_even_iterations(ab, options):
    """Tolerances just above the residual of iteration k - 1 stop the loop near k, at odd and at even
    iterations; the control word is read from the slot of the parity the loop ended on."""
    A = _matrix(ab, "27pt-ragged", seed=31)
    b = _rhs(A, seed=32)
    cg = ab.SolverCuda(A)
    options(pcg_fused=0)
    _, nits, _, _ = _solve(cg, A, b, maxits=2000, residualrtol=1e-10)
    seen = set()
    for k in range(nits - 8, nits - 2):
        options(pcg_fused=0)
        _solve(cg, A, b, maxits=k)
        tol = cg.c.rnrm2 / cg.c.r0nrm2 * (1 + 1e-9)
        res = {}
        for on in (1, 0):
            options(pcg_fused=on)
            res[on] = _solve(cg, A, b, maxits=2000, residualrtol=tol)
        _same(res[1], res[0])
        assert res[1][0] == 0 and res[1][1] < 2000
        seen.add(res[1][1] % 2)
    assert seen == {0, 1}
    cg.free()
    A.free()


def test_maxits_zero_returns_x0(ab, options):
    A = _matrix(ab, "27pt-full", seed=41)
    b = _rhs(A, seed=42)
    x0 = np.random.default_rng(43).standard_normal(len(b.x))
    options()
    cg = ab.SolverCuda(A)
    code, nits, _, x = _solve(cg, A, b, x0=x0, maxits=0)
    assert nits == 0 and np.array_equal(x.view(np.int64), x0.view(np.int64))
    cg.free()
    A.free()


def test_switch_between_solves(ab, options):
    A = _matrix(ab, "27pt-ragged", seed=51)
    b = _rhs(A, seed=52)
    cg = ab.SolverCuda(A)
    seq = []
    for on in (1, 0, 1, 0):
        options(pcg_fused=on)
        seq.append(_solve(cg, A, b, maxits=16))
        assert cg.info()["pcg_fused"] == on
    _same(seq[0], seq[1])
    for k in (2, 3):
        _same(seq[k], seq[k - 2])
    cg.free()
    A.free()


def _path(ab, A, **opts):
    ab_opts = dict(OPTS, **opts)
    for k, v in ab_opts.items():
        ab.set_option(k, v)
    cg = ab.SolverCuda(A)
    b = _rhs(A, seed=61)
    _solve(cg, A, b, maxits=8)
    inf = cg.info()
    cg.free()
    return inf


def test_path_selection(ab, options):
    A = _matrix(ab, "27pt-ragged", seed=71)
    inf = _path(ab, A)
    assert inf["pcg_fused"] == 1 and inf["last_blas_ms"] == 0.0
    assert inf["pcg_fused_min_bytes"] == inf["spmv_slice_rows"] * (8 * inf["spmv_symdiag_diagonals"] + 96)
    assert _path(ab, A, spmv_symdiag=0)["pcg_fused"] == 0
    assert _path(ab, A, pcg_fused=0)["pcg_fused"] == 0
    # a solve of any other kind after a fused one: spmv_min_bytes is the product's again
    options()
    cg = ab.SolverCuda(A)
    b = _rhs(A)
    n = A.c.nownedrows
    B = np.ascontiguousarray(np.stack([b.x[:n], b.x[:n][::-1]], axis=1))
    others = {"solvempi": lambda: cg.solvempi(b, A.vector(), maxits=8),
              "solve_multi": lambda: cg.solve_multi(B, np.zeros((n, 2)), maxits=8),
              "solve_shifted": lambda: cg.solve_shifted(b.x[:n], [0.0, 0.5], maxits=8),
              "solve_minres": lambda: cg.solve_minres(b, A.vector(), maxits=8),
              "solve_mixed": lambda: cg.solve_mixed(b, A.vector(), maxits=8)}
    for name, solve in others.items():
        cg.solve_pipelined(b, A.vector(), maxits=8)
        inf = cg.info()
        assert inf["pcg_fused"] == 1, name
        fused_bytes = inf["spmv_min_bytes"]
        solve()
        inf = cg.info()
        assert inf["pcg_fused"] == 0 and inf["spmv_min_bytes"] < fused_bytes, name
    cg.free()
    A.free()
    # full storage that is not exactly symmetric: no mirrored diagonals
    n, r, c, _ = BOXES["27pt-ragged"]()
    v = np.random.default_rng(72).standard_normal(len(r))
    v[r == c] += 30.0
    U = ab.SymCsrMatrix.init_real_double(n, r, c, v).dsymv_init(0.0)
    i = n // 2
    U.fa[U.frowptr[i]] += 1.0
    inf = _path(ab, U)
    assert inf["spmv_symdiag_diagonals"] == 0 and inf["pcg_fused"] == 0
    U.free()
    # exception rows, merge tiles (R-MAT)
    for gen in (lambda: big_stencil(True), rmat):
        n, r, c = gen()
        v = np.random.default_rng(73).standard_normal(len(r))
        v[r == c] = np.abs(v).max() * 64.0
        M = ab.SymCsrMatrix.init_real_double(n, r, c, v).dsymv_init(0.0)
        inf = _path(ab, M)
        assert inf["pcg_fused"] == 0 and (inf["spmv_slice_exc"] > 0 or inf["spmv_merge_tiles"] > 0), inf
        M.free()
    # one part of a 2-way partition, solved on one GPU: ghost rows
    n, r, c, v = mg.stencil3d_27pt(24)
    G = ab.SymCsrMatrix.init_real_double(n, r, c, v)
    parts = G.partition(2, (np.arange(n) * 2 // n).astype(np.int32))
    P0 = parts[0].dsymv_init(0.0)
    assert P0.c.nghostrows > 0
    inf = _path(ab, P0)
    assert inf["pcg_fused"] == 0
    for m in parts:
        m.free()
    G.free()


@pytest.mark.parametrize("box,per_iter", [("27pt-full", 1), ("27pt-ragged", 3)])
def test_launches_per_iteration(box, per_iter, ab, options):
    A = _matrix(ab, box, seed=81)
    b = _rhs(A, seed=82)
    options()
    cg = ab.SolverCuda(A)
    counts = {}
    for its in (40, 60):
        _solve(cg, A, b, maxits=its)
        counts[its] = cg.info()["last_launches"]
    assert (counts[60] - counts[40]) == 20 * per_iter
    cg.free()
    A.free()
