"""MINRES on the H100: acgsolvercuda_solve_minres against the float64 restatement of tests/minresref.py on
the same assembled matrix: equal iteration counts and codes, x within 1e-10 relative, and the exact true
residual (tests/exactref.py) below 2 tol.  Matrices: a 27-point stencil (pattern slices, coded mirrored
diagonals), a 7-point stencil with an odd number of rows (the kernels' tail row), an R-MAT structure (merge
tiles), random_spd_60 from tests/golden, and both stencils shifted by dsymv_init(-sigma) to a known number
of negative eigenvalues (closed-form spectrum).  The same counts with the mirrored diagonals and their codes
switched off; the edge cases (maxits, maxits = 0, b = 0, both breakdowns, rejected calls) and the launches
of a replayed iteration.  The tolerances are about 1e-10 relative, tight enough that x is pinned by the
solution: at looser ones two roundings of an indefinite Lanczos process can part for a while and agree only
to about cond(A) tol."""
import functools
import os

import numpy as np
import pytest
import scipy.sparse as sp

from exactref import rows_exact
from minresref import indefinite_shift, minres, stencil_eigenvalues

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NOT_CONVERGED, INVALID_VALUE, NOT_SUPPORTED = 39, 29, 26
# stencil key -> (stencil kind, box): the matrix and its closed-form spectrum
BOXES = {"27pt": (27, (30, 31, 29)), "7pt-odd": (7, (25, 25, 25))}


@functools.lru_cache(maxsize=None)
def _coo(key):
    from acg_b200 import matgen as mg
    if key == "27pt":
        return mg.stencil3d_27pt(*BOXES[key][1])
    if key == "7pt-odd":
        return mg.laplace3d_7pt(*BOXES[key][1])                  # 15625 rows
    if key == "rmat":
        # diagonal 1, off-diagonal -1/(2 max(deg_i, deg_j)): eigenvalues in [0.5, 1.5] by Gershgorin
        from test_gpu_kernel_variants import rmat
        n, r, c = rmat()
        off = r != c
        r, c = r[off], c[off]
        deg = np.bincount(r, minlength=n) + np.bincount(c, minlength=n)
        v = -0.5 / np.maximum(deg[r], deg[c])
        d = np.arange(n, dtype=np.int32)
        r = np.concatenate([r, d]); c = np.concatenate([c, d]); v = np.concatenate([v, np.ones(n)])
        o = np.lexsort((c, r))
        return n, r[o], c[o], v[o]
    g = np.load(os.path.join(ROOT, "tests", "golden", "random_spd_60.npz"))
    return int(g["n"]), g["rows"], g["cols"], g["vals"]


def _sigma(key, nneg):
    """The shift that leaves exactly nneg negative eigenvalues (closed-form spectrum of the stencil)."""
    kind, box = BOXES[key]
    ev = stencil_eigenvalues(kind, *box)
    s = indefinite_shift(ev, nneg)
    assert int((ev < s).sum()) == nneg and ev.min() < s < ev.max()
    return s


def _matrix(ab, key, eps=0.0):
    n, r, c, v = _coo(key)
    return ab.SymCsrMatrix.init_real_double(n, r, c, v).dsymv_init(eps)


def _csr(A):
    n = A.c.nownedrows
    rp = A.frowptr[:n + 1].copy()
    ci = A.fcolidx[:rp[n]].copy()
    a = A.fa[:rp[n]].copy()
    return (rp, ci, a), sp.csr_matrix((a, ci - A.c.rowidxbase, rp), shape=(n, n))


def _solve(cg, A, b, x0, **kw):
    bv = A.vector(); bv.x[:] = b
    xv = A.vector(); xv.x[:] = x0
    code = cg.solve_minres(bv, xv, **kw)
    return code, xv.x[:A.c.nownedrows].copy()


def _compare(A, b, x0, code, x, its, maxits, atol, rtol):
    arrays, M = _csr(A)
    ref = minres(M, b, x0=x0, maxits=maxits, atol=atol, rtol=rtol)
    assert its == ref["niterations"], (its, ref["niterations"], ref["stop"])
    assert code == ref["status"], (code, ref["status"])
    scale = max(float(np.abs(ref["x"]).max()), 1e-300)
    assert float(np.abs(x - ref["x"]).max()) <= 1e-10 * scale
    tol = max(atol if atol > 0 else 0.0, rtol * ref["r0nrm2"])
    if code == 0 and tol > 0:
        rt, _, _ = rows_exact(*arrays, x, b)
        assert float(np.linalg.norm(rt)) < 2 * tol, (float(np.linalg.norm(rt)), tol)
    return ref


# Indefinite cases whose iteration counts do not depend on the order of the dot products' sums (checked
# on the CPU by reordering them in the restatement): the 27-point box's second to fourth eigenvalues form a
# tight cluster (0.534, 0.551, 0.569), and with a shift past it two roundings can take different counts.
CASES = [("27pt", 0), ("7pt-odd", 0), ("rmat", 0), ("random_spd_60", 0),
         ("27pt", 1), ("7pt-odd", 1), ("7pt-odd", 4)]


@pytest.mark.gpu
@pytest.mark.parametrize("key,nneg", CASES)
def test_against_restatement(key, nneg, ab):
    """rtol from x0 = 0 (warm-up 0) and atol from a nonzero x0 (warm-up 2); then the same solves with the
    mirrored diagonals and with their one-byte codes switched off give the same iteration counts."""
    eps = -_sigma(key, nneg) if nneg else 0.0
    A = _matrix(ab, key, eps)
    n = A.c.nownedrows
    rng = np.random.default_rng(11)
    b = rng.standard_normal(n)
    x0 = rng.standard_normal(n)
    r0 = float(np.linalg.norm(b - _csr(A)[1] @ x0))
    runs = [(np.zeros(n), 0.0, 1e-10, 0), (x0, 1e-10 * r0, 0.0, 2)]
    counts = []
    cg = ab.SolverCuda(A)
    try:
        for xi, atol, rtol, warmup in runs:
            code, x = _solve(cg, A, b, xi, maxits=4000, residualatol=atol, residualrtol=rtol, warmup=warmup)
            assert code == 0
            _compare(A, b, xi, code, x, cg.c.niterations, 4000, atol, rtol)
            assert cg.c.rnrm2 < max(atol, rtol * cg.c.r0nrm2)
            counts.append(int(cg.c.niterations))
        info = cg.info()
    finally:
        cg.free()
    if key == "27pt":
        assert info["spmv_symdiag_diagonals"] > 0 and info["spmv_symdiag_codes"] > 0
    for opts in ({"spmv_symdiag": 0}, {"symdiag_codes": 0}):
        for k, v in opts.items():
            ab.set_option(k, v)
        try:
            cg = ab.SolverCuda(A)
            for (xi, atol, rtol, warmup), its in zip(runs, counts):
                code, x = _solve(cg, A, b, xi, maxits=4000, residualatol=atol, residualrtol=rtol, warmup=warmup)
                assert code == 0 and cg.c.niterations == its, (opts, cg.c.niterations, its)
            cg.free()
        finally:
            for k in opts:
                ab.set_option(k, 1)
    A.free()


@pytest.mark.gpu
def test_edge_cases_and_rejected_calls(ab):
    """maxits reached (NOT_CONVERGED), maxits = 0 (x0 bitwise), b = 0 (no iteration, with or without a
    tolerance), tolerances off (exactly maxits), a negative maxits and a part of a partitioned matrix."""
    key = "7pt-odd"
    A = _matrix(ab, key, -_sigma(key, 1))
    n = A.c.nownedrows
    rng = np.random.default_rng(3)
    b = rng.standard_normal(n)
    x0 = rng.standard_normal(n)
    cg = ab.SolverCuda(A)
    try:
        code, x = _solve(cg, A, b, x0, maxits=15, residualrtol=1e-10)
        assert code == NOT_CONVERGED and cg.c.niterations == 15
        _compare(A, b, x0, code, x, 15, 15, 0.0, 1e-10)
        code, x = _solve(cg, A, b, x0, maxits=0, residualrtol=1e-8)
        assert code == NOT_CONVERGED and cg.c.niterations == 0 and np.array_equal(x, x0)
        for atol in (1e-8, 0.0):
            code, x = _solve(cg, A, np.zeros(n), np.zeros(n), maxits=50, residualatol=atol)
            assert code == 0 and cg.c.niterations == 0 and not x.any() and cg.c.rnrm2 == 0.0
        code, x = _solve(cg, A, b, x0, maxits=9, warmup=2)
        assert code == 0 and cg.c.niterations == 9
        _compare(A, b, x0, code, x, 9, 9, 0.0, 0.0)
        with pytest.raises(ab.AcgError) as e:
            _solve(cg, A, b, x0, maxits=-1)
        assert e.value.code == INVALID_VALUE
    finally:
        cg.free()
    parts = A.partition(2, (np.arange(n) >= n // 2).astype(np.int32))
    P = parts[0].dsymv_init(0.0)
    cgp = ab.SolverCuda(P)
    try:
        with pytest.raises(ab.AcgError) as e:
            cgp.solve_minres(P.vector(), P.vector(), maxits=3)
        assert e.value.code == NOT_SUPPORTED
    finally:
        cgp.free()


@pytest.mark.gpu
def test_breakdown(ab):
    """A diagonal matrix of mixed signs with b = 1.5 e_i: beta_2 = 0 ends the solve after one iteration with
    x = 1.5 / d_i e_i, with or without a tolerance; at a zero diagonal entry gamma_1 = 0 ends it before the
    update (0 iterations, x0 returned, NOT_CONVERGED under a tolerance)."""
    n = 4099
    d = np.random.default_rng(2).uniform(0.5, 4.0, n) * np.where(np.arange(n) % 3 == 0, -1.0, 1.0)
    d[77] = 0.0
    idx = np.arange(n, dtype=np.int32)
    A = ab.SymCsrMatrix.init_real_double(n, idx, idx.copy(), d).dsymv_init(0.0)
    cg = ab.SolverCuda(A)
    try:
        for i in (0, 1, 2, 1000, n - 1):
            for rtol in (0.0, 1e-10):
                b = np.zeros(n); b[i] = 1.5
                code, x = _solve(cg, A, b, np.zeros(n), maxits=20, residualrtol=rtol)
                want = np.zeros(n); want[i] = 1.5 / d[i]
                assert code == 0 and cg.c.niterations == 1 and cg.c.rnrm2 == 0.0, (i, rtol)
                assert np.abs(x - want).max() <= 1e-15 * abs(want[i])
        b = np.zeros(n); b[77] = 1.0
        x0 = np.zeros(n)
        code, x = _solve(cg, A, b, x0, maxits=20, residualrtol=1e-8)
        assert code == NOT_CONVERGED and cg.c.niterations == 0 and not x.any() and cg.c.rnrm2 == 1.0
        code, x = _solve(cg, A, b, x0, maxits=20)
        assert code == 0 and cg.c.niterations == 0 and not x.any()
    finally:
        cg.free()


@pytest.mark.gpu
def test_graph_replay_launches(ab):
    """With tolerances off the loop runs exactly maxits iterations as graph replays: per iteration the
    single-vector product, minres_lanczos_kernel and minres_update_kernel -- as many launches as a classic
    iteration, three when the product is one kernel.  Solves of other kinds in between do not change what
    a replay computes."""
    key = "27pt"
    A = _matrix(ab, key, -_sigma(key, 1))
    n = A.c.nownedrows
    b = np.random.default_rng(8).standard_normal(n)
    cg = ab.SolverCuda(A)
    try:
        inf = cg.info()
        launches = {}
        for m in (10, 30):
            code, x = _solve(cg, A, b, np.zeros(n), maxits=m)
            assert code == 0 and cg.c.niterations == m
            launches[("minres", m)] = cg.info()["last_launches"]
            bv = A.vector(); bv.x[:] = b
            assert cg.solvempi(bv, A.vector(), maxits=m) == 0
            launches[("classic", m)] = cg.info()["last_launches"]
        per = (launches[("minres", 30)] - launches[("minres", 10)]) / 20
        assert per == (launches[("classic", 30)] - launches[("classic", 10)]) / 20
        if inf["spmv_slices"] > 0 and inf["spmv_ntiles"] == 0 and inf["spmv_merge_tiles"] == 0 \
                and inf["spmv_nlong"] == 0 and inf["spmv_nmedium"] == 0:
            assert per == 3
        ref = _solve(cg, A, b, np.zeros(n), maxits=400, residualrtol=1e-10)
        cg.solve_shifted(b, [0.1, 1.0], maxits=40)
        bv = A.vector(); bv.x[:] = b
        cg.solve_pipelined(bv, A.vector(), maxits=40)
        again = _solve(cg, A, b, np.zeros(n), maxits=400, residualrtol=1e-10)
        assert ref[0] == again[0]
        assert float(np.abs(ref[1] - again[1]).max()) <= 1e-12 * float(np.abs(ref[1]).max())
    finally:
        cg.free()
