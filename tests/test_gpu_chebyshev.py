"""Chebyshev-preconditioned CG (acgsolvercuda_solve_chebyshev) on the H100.

Against the restatement of tests/chebref.py on a 27-point stencil through the fused inner step (coded and fp64
mirrored diagonals), a 7-point stencil with an odd number of rows (fused, with tile rows) and the same with the
mirrored diagonals off (the plan's product and the elementwise step), an R-MAT matrix on merge tiles with a
random b, and random_spd_60: degrees 0, 1, 2 and 4 with the estimated interval and degree 3 with a given one --
equal iteration counts and estimate steps, x within 1e-10 relative, the exact true residual (tests/exactref.py)
below 2 tol.  On a constant diagonal degree 0 is CG: solvempi's iteration count and x.  Then the launches of a
replayed iteration (3 + d on the fused path), the edge cases, the rejected calls and a breakdown."""
import functools
import os

import numpy as np
import pytest
import scipy.sparse as sp

from chebref import chebyshev
from exactref import rows_exact

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NOT_CONVERGED, INVALID_VALUE, NOT_SUPPORTED = 39, 29, 26


@functools.lru_cache(maxsize=None)
def _coo(key):
    from acg_b200 import matgen as mg
    if key == "27pt":
        return mg.stencil3d_27pt(30, 31, 29)
    if key == "27pt-32":
        return mg.stencil3d_27pt(32)
    if key == "7pt-odd":
        return mg.laplace3d_7pt(25, 25, 25)                  # 15625 rows
    if key == "rmat":
        # the R-MAT structure of the kernel-variant tests with the project's R-MAT values: -1 off the diagonal,
        # degree + 1 on it (the diagonal spans 1 to the largest degree)
        from test_gpu_kernel_variants import rmat
        n, r, c = rmat()
        off = r != c
        r, c = r[off], c[off]
        deg = np.bincount(r, minlength=n) + np.bincount(c, minlength=n)
        d = np.arange(n, dtype=np.int32)
        v = np.concatenate([-np.ones(r.size), deg + 1.0])
        r = np.concatenate([r, d]); c = np.concatenate([c, d])
        o = np.lexsort((c, r))
        return n, r[o], c[o], v[o]
    g = np.load(os.path.join(ROOT, "tests", "golden", "random_spd_60.npz"))
    return int(g["n"]), g["rows"], g["cols"], g["vals"]


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
    code = cg.solve_chebyshev(bv, xv, **kw)
    return code, xv.x[:A.c.nownedrows].copy()


def _check(cg, A, b, x0, code, x, **kw):
    """counts and x against the restatement, the exact residual of x below 2 tol"""
    arrays, M = _csr(A)
    ref = chebyshev(M, b, x0=x0, degree=kw["degree"], lmin=kw.get("lmin", 0.0), lmax=kw.get("lmax", 0.0),
                    maxits=kw["maxits"], atol=kw.get("residualatol", 0.0), rtol=kw.get("residualrtol", 0.0))
    inf = cg.info()
    got = (int(cg.c.niterations), int(inf["cheb_est_iterations"]), code)
    assert got == (ref["niterations"], ref["est_steps"], ref["status"]), (got, ref["niterations"], ref["est_steps"])
    assert inf["cheb_lmax"] == pytest.approx(ref["lmax"], rel=1e-8) and inf["cheb_lmin"] == pytest.approx(ref["lmin"], rel=1e-8)
    assert np.abs(x - ref["x"]).max() <= 1e-10 * np.abs(ref["x"]).max(), np.abs(x - ref["x"]).max()
    rt, _, _ = rows_exact(*arrays, x, b)
    if code == 0 and ref["tol"] > 0:
        assert float(np.linalg.norm(rt)) < 2 * ref["tol"]
    return ref


SHAPES = [("27pt", {}), ("27pt", {"symdiag_codes": 0}), ("7pt-odd", {}), ("7pt-odd", {"spmv_symdiag": 0}),
          ("rmat", {}), ("random_spd_60", {})]


@pytest.mark.gpu
@pytest.mark.parametrize("key,opts", SHAPES)
def test_against_restatement(key, opts, ab):
    for k, v in opts.items():
        ab.set_option(k, v)
    try:
        A = _matrix(ab, key)
        n = A.c.nownedrows
        rng = np.random.default_rng(11)
        b = rng.standard_normal(n)
        x0 = rng.standard_normal(n)
        cg = ab.SolverCuda(A)
        try:
            inf = cg.info()
            if key == "27pt":
                assert inf["spmv_symdiag_diagonals"] > 0 and (inf["spmv_symdiag_codes"] > 0) == ("symdiag_codes" not in opts)
            if key == "7pt-odd":
                assert (inf["spmv_symdiag_diagonals"] > 0) == ("spmv_symdiag" not in opts)
            if key == "rmat":
                assert inf["spmv_merge_tiles"] > 0
            for deg in (0, 1, 2, 4):
                kw = dict(degree=deg, maxits=2000, residualrtol=1e-8)
                code, x = _solve(cg, A, b, np.zeros(n), **kw)
                assert code == 0 and cg.info()["cheb_breakdown"] == 0
                _check(cg, A, b, np.zeros(n), code, x, **kw)
            ref = _csr(A)[1]
            lmax = 1.1 * float(np.abs(sp.diags(1 / ref.diagonal()) @ ref).sum(axis=1).max())   # Gershgorin
            kw = dict(degree=3, lmax=lmax, maxits=2000, residualatol=1e-9 * float(np.linalg.norm(b)), warmup=2)
            code, x = _solve(cg, A, b, x0, **kw)
            assert code == 0
            _check(cg, A, b, x0, code, x, **kw)
        finally:
            cg.free()
        A.free()
    finally:
        for k in opts:
            ab.set_option(k, 1)


@pytest.mark.gpu
def test_degree0_on_constant_diagonal_is_cg(ab):
    """The 27-point stencil's diagonal is constant: Jacobi PCG takes solvempi's iterations and gives its x."""
    A = _matrix(ab, "27pt")
    n = A.c.nownedrows
    b = np.random.default_rng(4).standard_normal(n)
    cg = ab.SolverCuda(A)
    try:
        code, x = _solve(cg, A, b, np.zeros(n), degree=0, maxits=1000, residualrtol=1e-8)
        its = cg.c.niterations
        bv = A.vector(); bv.x[:] = b
        xc = A.vector()
        assert cg.solvempi(bv, xc, maxits=1000, residualrtol=1e-8) == 0 and code == 0
        assert its == cg.c.niterations
        assert np.abs(x - xc.x[:n]).max() <= 1e-10 * np.abs(xc.x[:n]).max()
    finally:
        cg.free()


@pytest.mark.gpu
def test_graph_replay_launches(ab):
    """Tolerances off: exactly maxits iterations as graph replays, 3 + d launches each on the fused path when
    the mirrored diagonals cover every row (the product, the r/x kernel, d inner steps, the p kernel); a
    solve of another degree, interval or kind in between does not change what a replay computes (the graph
    of another interval is captured anew)."""
    A = _matrix(ab, "27pt-32")
    n = A.c.nownedrows
    b = np.random.default_rng(8).standard_normal(n)
    cg = ab.SolverCuda(A)
    try:
        inf = cg.info()
        covered = inf["spmv_slice_rows"] == n and inf["spmv_ntiles"] == 0 and inf["spmv_symdiag_diagonals"] > 0
        for deg in (0, 2, 5):
            launches = {}
            for m in (10, 30):
                code, x = _solve(cg, A, b, np.zeros(n), degree=deg, lmin=0.2, lmax=2.5, maxits=m)
                assert code == 0 and cg.c.niterations == m
                launches[m] = cg.info()["last_launches"]
            per = (launches[30] - launches[10]) / 20
            assert per == 3 + deg if covered else per >= 3 + deg, (deg, per, inf)
        ref = _solve(cg, A, b, np.zeros(n), degree=2, maxits=400, residualrtol=1e-10)
        its = cg.c.niterations
        _solve(cg, A, b, np.zeros(n), degree=2, lmin=0.1, lmax=3.0, maxits=40)
        bv = A.vector(); bv.x[:] = b
        cg.solve_pipelined(bv, A.vector(), maxits=40)
        cg.solve_mixed(bv, A.vector(), maxits=40)
        again = _solve(cg, A, b, np.zeros(n), degree=2, maxits=400, residualrtol=1e-10)
        # the dot products are sums of per-CTA atomics, so two runs agree to rounding, not bitwise
        assert ref[0] == again[0] == 0 and cg.c.niterations == its
        assert np.abs(ref[1] - again[1]).max() <= 1e-12 * np.abs(ref[1]).max()
    finally:
        cg.free()


@pytest.mark.gpu
def test_edge_cases_and_rejected_calls(ab):
    """maxits reached, maxits = 0 (x0 bitwise), b = 0, tolerances off (exactly maxits), every rejected
    argument, a non-positive diagonal (dsymv_init(-7) on the 7-point stencil), a part of a partitioned matrix."""
    A = _matrix(ab, "7pt-odd")
    n = A.c.nownedrows
    rng = np.random.default_rng(3)
    b = rng.standard_normal(n)
    x0 = rng.standard_normal(n)
    cg = ab.SolverCuda(A)
    try:
        kw = dict(degree=2, maxits=5, residualrtol=1e-10)
        code, x = _solve(cg, A, b, x0, **kw)
        assert code == NOT_CONVERGED and cg.c.niterations == 5
        _check(cg, A, b, x0, code, x, **kw)
        code, x = _solve(cg, A, b, x0, degree=2, maxits=0, residualrtol=1e-8)
        assert code == NOT_CONVERGED and cg.c.niterations == 0 and np.array_equal(x, x0)
        for atol in (1e-8, 0.0):
            code, x = _solve(cg, A, np.zeros(n), np.zeros(n), degree=1, maxits=50, residualatol=atol)
            assert code == 0 and cg.c.niterations == 0 and not x.any() and cg.c.rnrm2 == 0.0
        kw = dict(degree=1, maxits=9, warmup=2)
        code, x = _solve(cg, A, b, x0, **kw)
        assert code == 0 and cg.c.niterations == 9
        _check(cg, A, b, x0, code, x, **kw)
        for bad in (dict(degree=-1), dict(degree=17), dict(degree=2, lmin=1.0, lmax=1.0), dict(degree=2, lmin=2.0, lmax=1.0),
                    dict(degree=2, lmin=float("nan")), dict(degree=2, lmax=float("inf")), dict(degree=1, lmin=-0.1),
                    dict(degree=1, lmax=-1.0), dict(degree=2, lmin=50.0), dict(degree=0, maxits=-1)):
            args = dict(maxits=20, residualrtol=1e-8)
            args.update(bad)
            with pytest.raises(ab.AcgError) as e:
                _solve(cg, A, b, x0, **args)
            assert e.value.code == INVALID_VALUE, bad
        # breakdown: degree 1 over [0.3, 1.0] with lambda_max(D^-1 A) near 2 > a + b makes M^-1 indefinite
        kw = dict(degree=1, lmin=0.3, lmax=1.0, maxits=300, residualrtol=1e-10)
        code, x = _solve(cg, A, b, np.zeros(n), **kw)
        ref = _check(cg, A, b, np.zeros(n), code, x, **kw)
        assert ref["stop"] == "breakdown" and cg.info()["cheb_breakdown"] == 1 and code == NOT_CONVERGED
    finally:
        cg.free()
    neg = _matrix(ab, "7pt-odd", eps=-7.0)
    cgn = ab.SolverCuda(neg)
    try:
        with pytest.raises(ab.AcgError) as e:
            _solve(cgn, neg, b, x0, degree=0, maxits=20)
        assert e.value.code == INVALID_VALUE
    finally:
        cgn.free()
    parts = A.partition(2, (np.arange(n) >= n // 2).astype(np.int32))
    P = parts[0].dsymv_init(0.0)
    cgp = ab.SolverCuda(P)
    try:
        with pytest.raises(ab.AcgError) as e:
            cgp.solve_chebyshev(P.vector(), P.vector(), maxits=3)
        assert e.value.code == NOT_SUPPORTED
    finally:
        cgp.free()
