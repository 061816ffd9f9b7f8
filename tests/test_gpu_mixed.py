"""Mixed-precision CG with reliable updates on the H100.

The fp32 product (acgsolvercuda_spmv_f32) on every plan shape: rows through the mirrored diagonals are
bitwise fl32 of the fp64 product of the widened vector, every row is within half an fp32 ulp (plus the
fp64 chain's rounding) of the exact product, integer data gives the exact product bitwise, and the fused
dot is (x, y) in fp64.  acgsolvercuda_solve_mixed against the restatement of tests/mixedref.py on a
27-point stencil, a 7-point stencil with an odd number of rows, an R-MAT structure (merge tiles) and
random_spd_60, each also with the mirrored diagonals and with their codes switched off: the exact true
residual (tests/exactref.py) below tol, rnrm2 that residual, and counts within 2 iterations and 1 reliable
update of the restatement's (the dot products' order differs).  Then the edge cases, b scaled by 2^+-200,
(p, A p) = 0, rejected calls and the launches of a replayed iteration."""
import functools
import os

import numpy as np
import pytest
import scipy.sparse as sp

from exactref import rows_exact
from mixedref import mixed

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NOT_CONVERGED, INVALID_VALUE, NOT_SUPPORTED = 39, 29, 26


@functools.lru_cache(maxsize=None)
def _coo(key):
    from acg_b200 import matgen as mg
    if key == "27pt":
        return mg.stencil3d_27pt(30, 31, 29)
    if key == "7pt-odd":
        return mg.laplace3d_7pt(25, 25, 25)                  # 15625 rows
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


def _matrix(ab, key):
    n, r, c, v = _coo(key)
    return ab.SymCsrMatrix.init_real_double(n, r, c, v).dsymv_init(0.0)


def _csr(A):
    n = A.c.nownedrows
    rp = A.frowptr[:n + 1].copy()
    ci = A.fcolidx[:rp[n]].copy()
    a = A.fa[:rp[n]].copy()
    return (rp, ci, a), sp.csr_matrix((a, ci - A.c.rowidxbase, rp), shape=(n, n))


def _solve(cg, A, b, x0, **kw):
    bv = A.vector(); bv.x[:] = b
    xv = A.vector(); xv.x[:] = x0
    code = cg.solve_mixed(bv, xv, **kw)
    return code, xv.x[:A.c.nownedrows].copy()


def _check_solve(cg, A, b, x0, code, x, maxits, atol, rtol):
    """counts against the restatement, the exact residual of x below tol and equal to rnrm2"""
    arrays, M = _csr(A)
    ref = mixed(M, b, x0=x0, maxits=maxits, atol=atol, rtol=rtol)
    its, upd = int(cg.c.niterations), int(cg.info()["mixed_reliable_updates"])
    assert abs(its - ref["niterations"]) <= 2 and abs(upd - ref["nupdates"]) <= 1, (its, upd, ref["niterations"],
                                                                                   ref["nupdates"])
    assert code == ref["status"]
    rt, _, _ = rows_exact(*arrays, x, b)
    true = float(np.linalg.norm(rt))
    assert cg.c.rnrm2 == pytest.approx(true, rel=1e-8, abs=1e-13 * max(cg.c.bnrm2, cg.c.r0nrm2))
    if code == 0 and ref["tol"] > 0:
        assert true < ref["tol"], (true, ref["tol"])
    return ref


SHAPES = [("27pt", {}), ("27pt", {"symdiag_codes": 0}), ("27pt", {"spmv_symdiag": 0}), ("7pt-odd", {}),
          ("rmat", {}), ("random_spd_60", {})]


@pytest.mark.gpu
@pytest.mark.parametrize("key,opts", SHAPES)
def test_spmv_f32(key, opts, ab):
    for k, v in opts.items():
        ab.set_option(k, v)
    try:
        A = _matrix(ab, key)
        n = A.c.nownedrows
        arrays, _ = _csr(A)
        cg = ab.SolverCuda(A)
        try:
            info = cg.info()
            if key == "27pt":
                assert (info["spmv_symdiag_diagonals"] > 0) == (opts.get("spmv_symdiag", 1) != 0)
            x = np.random.default_rng(1).standard_normal(n).astype(np.float32)
            y, dot = cg.spmv_f32(x)
            assert y.dtype == np.float32 and np.isfinite(y).all()
            x64 = x.astype(np.float64)
            ex, scale, m = rows_exact(*arrays, x64)
            bound = np.abs(ex) * 2.0 ** -24 + (m + 2) * 2.0 ** -53 * scale + 1e-300
            assert (np.abs(y.astype(np.float64) - ex) <= bound).all()
            assert dot == pytest.approx(float(x64 @ y.astype(np.float64)), rel=1e-12, abs=1e-12 * n)
            y64, _ = cg.spmv_mode(0, np.pad(x64, (0, cg.c.r.num_nonzeros - n)))
            same = int(np.count_nonzero(y == y64.astype(np.float32)))
            if info["spmv_symdiag_diagonals"] > 0:
                assert same >= info["spmv_slice_rows"], (same, info["spmv_slice_rows"])
            # integer data and vector: every sum is exact in fp32, so the product is exact bitwise
            if key in ("27pt", "7pt-odd"):
                xi = np.random.default_rng(2).integers(-100, 101, n).astype(np.float32)
                yi, doti = cg.spmv_f32(xi)
                exi, _, _ = rows_exact(*arrays, xi.astype(np.float64))
                assert np.array_equal(yi.astype(np.float64), exi)
                assert doti == float(xi.astype(np.float64) @ exi)
        finally:
            cg.free()
        A.free()
    finally:
        for k in opts:
            ab.set_option(k, 1)


@pytest.mark.gpu
@pytest.mark.parametrize("key", ["27pt", "7pt-odd", "rmat", "random_spd_60"])
def test_against_restatement(key, ab):
    """rtol 1e-8 from x0 = 0 (warm-up 0) and an atol from a nonzero x0 (warm-up 2); then the same solves with
    the mirrored diagonals and with their codes switched off."""
    A = _matrix(ab, key)
    n = A.c.nownedrows
    rng = np.random.default_rng(11)
    b = rng.standard_normal(n)
    x0 = rng.standard_normal(n)
    r0 = float(np.linalg.norm(b - _csr(A)[1] @ x0))
    runs = [(np.zeros(n), 0.0, 1e-8, 0), (x0, 1e-10 * r0, 0.0, 2)]
    for opts in ({}, {"spmv_symdiag": 0}, {"symdiag_codes": 0}):
        for k, v in opts.items():
            ab.set_option(k, v)
        try:
            cg = ab.SolverCuda(A)
            try:
                for xi, atol, rtol, warmup in runs:
                    code, x = _solve(cg, A, b, xi, maxits=4000, residualatol=atol, residualrtol=rtol, warmup=warmup)
                    assert code == 0, opts
                    _check_solve(cg, A, b, xi, code, x, 4000, atol, rtol)
                    assert cg.info()["mixed_reliable_updates"] >= 1
            finally:
                cg.free()
        finally:
            for k in opts:
                ab.set_option(k, 1)
    A.free()


@pytest.mark.gpu
def test_edge_cases_scaling_and_rejected_calls(ab):
    """maxits reached (NOT_CONVERGED, rnrm2 the residual of the folded x), maxits = 0 (x0 bitwise), b = 0,
    tolerances off (exactly maxits), b scaled by 2^+-200 (counts within the dot-order allowance, x scaled),
    a negative maxits and a part of a partitioned matrix."""
    A = _matrix(ab, "7pt-odd")
    n = A.c.nownedrows
    rng = np.random.default_rng(3)
    b = rng.standard_normal(n)
    x0 = rng.standard_normal(n)
    cg = ab.SolverCuda(A)
    try:
        code, x = _solve(cg, A, b, x0, maxits=15, residualrtol=1e-10)
        assert code == NOT_CONVERGED and cg.c.niterations == 15
        _check_solve(cg, A, b, x0, code, x, 15, 0.0, 1e-10)
        code, x = _solve(cg, A, b, x0, maxits=0, residualrtol=1e-8)
        assert code == NOT_CONVERGED and cg.c.niterations == 0 and np.array_equal(x, x0)
        for atol in (1e-8, 0.0):
            code, x = _solve(cg, A, np.zeros(n), np.zeros(n), maxits=50, residualatol=atol)
            assert code == 0 and cg.c.niterations == 0 and not x.any() and cg.c.rnrm2 == 0.0
        code, x = _solve(cg, A, b, x0, maxits=9, warmup=2)
        assert code == 0 and cg.c.niterations == 9
        _check_solve(cg, A, b, x0, code, x, 9, 0.0, 0.0)
        code, xr = _solve(cg, A, b, np.zeros(n), maxits=1000, residualrtol=1e-10)
        its, upd = cg.c.niterations, cg.info()["mixed_reliable_updates"]
        for s in (200, -200):
            code, xs = _solve(cg, A, np.ldexp(b, s), np.zeros(n), maxits=1000, residualrtol=1e-10)
            assert code == 0 and abs(cg.c.niterations - its) <= 2
            assert abs(cg.info()["mixed_reliable_updates"] - upd) <= 1
            assert np.abs(np.ldexp(xs, -s) - xr).max() <= 1e-7 * np.abs(xr).max()
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
            cgp.solve_mixed(P.vector(), P.vector(), maxits=3)
        assert e.value.code == NOT_SUPPORTED
    finally:
        cgp.free()


@pytest.mark.gpu
def test_zero_curvature(ab):
    """A positive diagonal with one zero entry: b = 1.5 e_i on a power-of-two entry converges in one
    iteration; on the zero entry (p, A p) = 0 ends the solve before the update (0 iterations, x0 returned,
    rnrm2 = ||b||, NOT_CONVERGED under a tolerance)."""
    n = 4099
    d = np.ldexp(1.0, np.random.default_rng(2).integers(-3, 4, n))
    d[77] = 0.0
    idx = np.arange(n, dtype=np.int32)
    A = ab.SymCsrMatrix.init_real_double(n, idx, idx.copy(), d).dsymv_init(0.0)
    cg = ab.SolverCuda(A)
    try:
        for i in (0, 1000, n - 1):
            b = np.zeros(n); b[i] = 1.5
            code, x = _solve(cg, A, b, np.zeros(n), maxits=20, residualrtol=1e-10)
            want = np.zeros(n); want[i] = 1.5 / d[i]
            assert code == 0 and cg.c.niterations == 1 and np.array_equal(x, want), i
        b = np.zeros(n); b[77] = 1.0
        code, x = _solve(cg, A, b, np.zeros(n), maxits=20, residualrtol=1e-8)
        assert code == NOT_CONVERGED and cg.c.niterations == 0 and not x.any() and cg.c.rnrm2 == 1.0
        code, x = _solve(cg, A, b, np.zeros(n), maxits=20)
        assert code == 0 and cg.c.niterations == 0 and not x.any()
    finally:
        cg.free()


@pytest.mark.gpu
def test_graph_replay_launches(ab):
    """With tolerances off the loop runs exactly maxits iterations as graph replays: per iteration the fp32
    product, update_r, update_yp, the gated fp64 residual product and the replacement -- five launches when
    both products are one kernel.  Solves of other kinds in between do not change what a replay computes."""
    A = _matrix(ab, "27pt")
    n = A.c.nownedrows
    b = np.random.default_rng(8).standard_normal(n)
    cg = ab.SolverCuda(A)
    try:
        inf = cg.info()
        launches = {}
        for m in (10, 30):
            code, x = _solve(cg, A, b, np.zeros(n), maxits=m)
            assert code == 0 and cg.c.niterations == m
            launches[m] = cg.info()["last_launches"]
        per = (launches[30] - launches[10]) / 20
        if inf["spmv_slices"] > 0 and inf["spmv_slice_rows"] == n and inf["spmv_ntiles"] == 0:
            assert per == 5
        else:
            assert per >= 5
        ref = _solve(cg, A, b, np.zeros(n), maxits=400, residualrtol=1e-10)
        bv = A.vector(); bv.x[:] = b
        cg.solve_pipelined(bv, A.vector(), maxits=40)
        cg.solve_minres(bv, A.vector(), maxits=40)
        again = _solve(cg, A, b, np.zeros(n), maxits=400, residualrtol=1e-10)
        assert ref[0] == again[0] == 0
        assert float(np.abs(ref[1] - again[1]).max()) <= 1e-7 * float(np.abs(ref[1]).max())
    finally:
        cg.free()
