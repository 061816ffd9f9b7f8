"""Every solve entry point where its kernels take several trips of their grid-stride loops.

Below a few hundred thousand rows every BLAS-1 and update kernel runs one row pair per thread, and every
slice kernel one slice per warp: an accumulator reset per trip, an index that drifts with the trip or a
partial last trip of a warp-uniform loop would pass every other solver test.  Here:

* moderate matrices (27-point 69 x 70 x 71: n even, coded and fp64 mirrored diagonals; 7-point 73 x 71 x 67:
  n odd; R-MAT 400 k rows on merge tiles) with the grids capped to one CTA per SM (blas1_ctas, slice_max_ctas,
  spmv_max_ctas, merge_max_ctas), each with and without programmatic dependent launch: classic, two-kernel
  and fused pipelined CG against the oracle; solve_multi (1, 3, 8 columns) and solve_shifted (1, 5, 8
  shifts) against solvempi; MINRES, mixed precision and Chebyshev PCG (degrees 0, 2, 5) against the
  restatements of tests/minresref.py, mixedref.py and chebref.py -- with the tolerances of the solvers' own
  test files, and the true residual of every converged solve below 2 tol;
* the benchmark sizes (27-point 224^3, 7-point 256^3, R-MAT 2 M), uncapped: there the kernels without a cap
  option loop too (multi-vector product, fp32 rows);
* on the CPU: tests/exactref.rows_dd, the double-double residual these sizes need, against exact rational
  arithmetic, and a guard that every matrix here takes at least two trips on 114 and 132 SMs.

Every GPU test first asserts from info() that it is in the regime it claims.  The layout assertions are
skipped on the host-logic stand-in (ACGB200_TEST_LIB), which never takes the mirrored diagonals."""
import functools
import os
from fractions import Fraction

import numpy as np
import pytest
import scipy.sparse as sp

from chebref import chebyshev
from exactref import U, gamma, rows_dd, rows_exact
from minresref import indefinite_shift, minres, stencil_eigenvalues
from mixedref import mixed
from test_exactref import _fr_rows, _random_csr

NOT_CONVERGED = 39
STANDIN = bool(os.environ.get("ACGB200_TEST_LIB"))
BLAS1_THREADS = 512                 # kernels.cu: each thread of a BLAS-1 kernel takes a row pair per trip
SM_COUNTS = (114, 132)              # H100 PCIe, H100 SXM
MAX_THREADS_PER_SM = 2048
MERGE_ITEMS = 2048                  # cgcuda.c: merged items per merge-path tile by default
# every option a test here changes, and its default
CAPS = {"blas1_ctas": 1, "slice_max_ctas": 1, "spmv_max_ctas": 1, "merge_max_ctas": 1}
DEFAULTS = {"blas1_ctas": 0, "slice_max_ctas": 0, "spmv_max_ctas": 0, "merge_max_ctas": 0, "pdl": 0,
            "symdiag_codes": 1, "pcg_fused": 1}

# moderate matrices: key -> box (stencils) or R-MAT size
BOXES = {"27pt": (27, (69, 70, 71)), "7pt": (7, (73, 71, 67))}
RMAT = (400_000, 4_000_000, 5)
# (id, matrix key, plan options)
MATS = [("27pt-coded", "27pt", {}), ("27pt-fp64", "27pt", {"symdiag_codes": 0}), ("7pt-odd", "7pt", {}),
        ("rmat", "rmat", {})]
BENCH = {"27pt": (27, 224), "7pt": (7, 256)}


# ---------------------------------------------------------------------------------------------
# matrices


@functools.lru_cache(maxsize=None)
def _coo(key, values="cg"):
    """Upper-triangle COO.  R-MAT: values "cheb" are the generator's D + I - Adj (Jacobi-preconditioned
    solves converge on it); "cg": diagonal 1, off-diagonal -1/(2 max(deg_i, deg_j)), eigenvalues in
    [0.5, 1.5] by Gershgorin, so that the unpreconditioned solvers agree with their references to 1e-10
    instead of drifting apart at the condition number of a hub row."""
    from acg_b200 import matgen as mg
    if key in BOXES:
        kind, box = BOXES[key]
        return (mg.stencil3d_27pt if kind == 27 else mg.laplace3d_7pt)(*box)
    n, r, c, v = mg.rmat_spd(*RMAT[:2], seed=RMAT[2])
    if values == "cheb":
        return n, r, c, v
    off = r != c
    r, c = r[off], c[off]
    deg = np.bincount(r, minlength=n) + np.bincount(c, minlength=n)
    v = -0.5 / np.maximum(deg[r], deg[c])
    d = np.arange(n, dtype=np.int32)
    r = np.concatenate([r, d]); c = np.concatenate([c, d]); v = np.concatenate([v, np.ones(n)])
    o = np.lexsort((c, r))
    return n, r[o], c[o], v[o]


_MATRICES = {}


def _matrix(ab, key, values="cg", eps=0.0):
    k = (key, values, eps)
    if k not in _MATRICES:
        n, r, c, v = _coo(key, values)
        _MATRICES[k] = ab.SymCsrMatrix.init_real_double(n, r, c, v).dsymv_init(eps)
    return _MATRICES[k]


def _csr(A):
    n = A.c.nownedrows
    rp = A.frowptr[:n + 1].copy()
    ci = A.fcolidx[:rp[n]].copy()
    a = A.fa[:rp[n]].copy()
    return (rp, ci, a), sp.csr_matrix((a, ci - A.c.rowidxbase, rp), shape=(n, n))


def _residual(arrays, x, b):
    """||b - A x|| from the double-double rows (error far below any tolerance used here)"""
    r, _, _ = rows_dd(*arrays, x, b)
    return float(np.linalg.norm(r))


def teardown_module(module):
    for A in _MATRICES.values():
        A.free()
    _MATRICES.clear()
    _REF.clear()


# references shared by the pdl = 0 and pdl = 1 runs of a test (the restatements do not depend on it)
_REF = {}


def _ref(key, fn):
    if key not in _REF:
        _REF[key] = fn()
    return _REF[key]


# ---------------------------------------------------------------------------------------------
# the regime


@pytest.fixture
def capped(ab):
    """The moderate matrices' grids capped to one CTA per SM; the options back to their defaults after."""
    def set_(**kw):
        for k, v in {**CAPS, **kw}.items():
            ab.set_option(k, v)
    yield set_
    for k, v in DEFAULTS.items():
        ab.set_option(k, v)


def _in_regime(cg, n, key, opts, ncols=1, capped=True):
    """info(): the BLAS-1 kernels and the product's grid take at least two trips (every thread, every warp)."""
    inf = cg.info()
    sms = inf["num_sms"]
    per_sm = 1 if capped else MAX_THREADS_PER_SM // BLAS1_THREADS
    assert n * ncols // 2 >= 2 * sms * per_sm * BLAS1_THREADS, (n, ncols, sms)
    if STANDIN:
        return inf
    if key == "rmat":
        assert inf["spmv_merge_tiles"] > 0 and inf["spmv_slices"] == 0
        assert inf["spmv_merge_tiles"] >= 2 * inf["spmv_merge_grid"], inf
        if capped:
            assert inf["spmv_merge_grid"] <= sms
    else:
        assert inf["spmv_symdiag_diagonals"] > 0
        assert (inf["spmv_symdiag_codes"] > 0) == (opts.get("symdiag_codes", 1) != 0)
        assert inf["spmv_slices"] >= 2 * inf["spmv_slice_grid"] * inf["spmv_slice_threads"] // 32, inf
        if capped:
            assert inf["spmv_slice_grid"] <= sms
    return inf


def _vec(A, v):
    out = A.vector()
    out.x[:A.c.nownedrows] = v
    return out


# ---------------------------------------------------------------------------------------------
# the moderate matrices under caps


@pytest.mark.gpu
@pytest.mark.parametrize("pdl", [0, 1])
@pytest.mark.parametrize("mid,key,opts", MATS, ids=[m[0] for m in MATS])
def test_cg_against_oracle(mid, key, opts, pdl, ab, capped, oracle):
    """Classic, two-kernel pipelined and fused pipelined CG from a nonzero x0: the oracle's return code,
    iteration count and x (1e-9 relative, as test_gpu_parity), the true residual below 2 tol; then the
    same with tolerances off, an odd maxits and warm-up 2 (graph replays of a fixed count)."""
    capped(pdl=pdl, **opts)
    A = _matrix(ab, key)
    n = A.c.nownedrows
    arrays, _ = _csr(A)
    rng = np.random.default_rng(21)
    b, x0 = rng.standard_normal(n), rng.standard_normal(n)
    cg = ab.SolverCuda(A)
    try:
        _in_regime(cg, n, key, opts)
        for method, fused, orc in (("solvempi", 1, "cg"), ("solve_pipelined", 0, "cg_pipelined"),
                                   ("solve_pipelined", 1, "cg_pipelined")):
            ab.set_option("pcg_fused", fused)
            for maxits, rtol, warmup in ((2000, 1e-9, 1), (23, 0.0, 2)):
                want = _ref((key, orc, maxits), lambda: getattr(oracle, orc)(arrays, b, x0=x0, maxits=maxits, rtol=rtol))
                xv = _vec(A, x0)
                code = getattr(cg, method)(_vec(A, b), xv, maxits=maxits, residualrtol=rtol, warmup=warmup)
                x = xv.x[:n]
                tag = (method, fused, maxits)
                assert code == want["status"] == 0, tag
                assert cg.c.niterations == want["niterations"], (tag, cg.c.niterations, want["niterations"])
                assert np.abs(x - want["x"]).max() <= 1e-9 * np.abs(want["x"]).max(), tag
                if rtol > 0:
                    assert _residual(arrays, x, b) < 2 * rtol * want["r0nrm2"], tag
                if method == "solve_pipelined" and fused and not STANDIN and key != "rmat":
                    assert cg.info()["pcg_fused"] == 1
    finally:
        cg.free()


@pytest.mark.gpu
@pytest.mark.parametrize("pdl", [0, 1])
@pytest.mark.parametrize("mid,key,opts", MATS, ids=[m[0] for m in MATS])
def test_multi_against_solvempi(mid, key, opts, pdl, ab, capped):
    """solve_multi with 1, 3 and 8 columns (right-hand sides scaled by 4^j under one absolute tolerance, so
    the columns stop apart; random X0) column by column against solvempi: equal iteration counts, ||r||
    within 1e-10 ||r0||, x within 1e-10 relative, the true residual below 2 tol."""
    capped(pdl=pdl, **opts)
    A = _matrix(ab, key)
    n = A.c.nownedrows
    arrays, _ = _csr(A)
    rng = np.random.default_rng(31)
    B8 = rng.standard_normal((n, 8)) * 4.0 ** np.arange(8)
    X8 = rng.standard_normal((n, 8))
    atol = 1e-6 * float(np.linalg.norm(B8[:, 0]))
    cg = ab.SolverCuda(A)
    try:
        def single(j):
            xv = _vec(A, X8[:, j])
            code = cg.solvempi(_vec(A, B8[:, j]), xv, maxits=2000, residualatol=atol)
            return code, int(cg.c.niterations), float(cg.c.rnrm2), float(cg.c.r0nrm2), xv.x[:n].copy()

        for k, warmup in ((1, 0), (3, 2), (8, 1)):
            _in_regime(cg, n, key, opts, ncols=k)
            X = X8[:, :k].copy()                     # solve_multi overwrites it
            code, cols = cg.solve_multi(np.ascontiguousarray(B8[:, :k]), X, maxits=2000, residualatol=atol,
                                        warmup=warmup)
            assert code == 0 and cg.c.niterations == max(c["niterations"] for c in cols)
            if k > 1:
                assert len({c["niterations"] for c in cols}) > 1
            for j in range(k):
                cj, its, rn, r0, xj = _ref((key, "multi", j), lambda: single(j))
                assert cj == 0 and cols[j]["niterations"] == its, (k, j, cols[j], its)
                assert abs(cols[j]["rnrm2"] - rn) <= 1e-10 * r0, (k, j, cols[j], rn)
                assert float(np.abs(X[:, j] - xj).max()) <= 1e-10 * float(np.abs(xj).max()), (k, j)
                assert _residual(arrays, X[:, j], B8[:, j]) < 2 * atol, (k, j)
    finally:
        cg.free()


SHIFTS = [0.0, 1.0, 0.1, 0.01, 0.3, 0.03, 3.0, 1e-3]      # relative to the mean diagonal entry


@pytest.mark.gpu
@pytest.mark.parametrize("pdl", [0, 1])
@pytest.mark.parametrize("mid,key,opts", MATS, ids=[m[0] for m in MATS])
def test_shifted_against_solvempi(mid, key, opts, pdl, ab, capped):
    """solve_shifted with 1, 5 and 8 shifts (block widths 1, 8, 8) shift by shift against solvempi on a
    solver of dsymv_init(sigma_j): equal iteration counts and convergence flags, x within 1e-10 relative,
    the true residual of A + sigma_j I below 2 tol."""
    capped(pdl=pdl, **opts)
    A = _matrix(ab, key)
    n = A.c.nownedrows
    arrays, _ = _csr(A)
    rp, ci, a = arrays
    diag = np.flatnonzero(np.repeat(np.arange(n), np.diff(rp)) == ci)
    dmean = float(a[diag].mean())
    b = np.random.default_rng(41).standard_normal(n)
    rtol = 1e-10
    cg = ab.SolverCuda(A)
    try:
        _in_regime(cg, n, key, opts)

        def single(sigma):
            nn, r, c, v = _coo(key)
            Aj = ab.SymCsrMatrix.init_real_double(nn, r, c, v).dsymv_init(sigma)
            aj = a.copy()
            aj[diag] += sigma
            assert np.array_equal(Aj.fa[:len(a)], aj)        # the residual below uses these values
            cgj = ab.SolverCuda(Aj)
            try:
                _in_regime(cgj, n, key, opts)
                xv = Aj.vector()
                code = cgj.solvempi(_vec(Aj, b), xv, maxits=2000, residualrtol=rtol)
                return code, int(cgj.c.niterations), xv.x[:n].copy(), aj
            finally:
                cgj.free()
                Aj.free()

        for S in (1, 5, 8):
            shifts = [dmean * s for s in SHIFTS[:S]]
            code, X, cols = cg.solve_shifted(b, shifts, maxits=2000, residualrtol=rtol, warmup=2 if S == 5 else 0)
            assert code == 0 and X.shape == (n, S)
            assert cg.c.niterations == max(c["niterations"] for c in cols)
            for j, sigma in enumerate(shifts):
                cj, its, xj, aj = _ref((key, "shift", j), lambda: single(sigma))
                assert cj == 0 and cols[j]["niterations"] == its and cols[j]["converged"] == 1, (S, j, cols[j], its)
                assert float(np.abs(X[:, j] - xj).max()) <= 1e-10 * float(np.abs(xj).max()), (S, j)
                assert _residual((rp, ci, aj), X[:, j], b) < 2 * rtol * float(np.linalg.norm(b)), (S, j)
    finally:
        cg.free()


def _sigma(key, nneg):
    kind, box = BOXES[key]
    ev = stencil_eigenvalues(kind, *box)
    s = indefinite_shift(ev, nneg)
    assert int((ev < s).sum()) == nneg
    return s


@pytest.mark.gpu
@pytest.mark.parametrize("pdl", [0, 1])
@pytest.mark.parametrize("mid,key,opts", MATS, ids=[m[0] for m in MATS])
def test_minres_against_restatement(mid, key, opts, pdl, ab, capped):
    """MINRES against tests/minresref.py: positive definite from a nonzero x0 (absolute tolerance, warm-up
    2) and, on the stencils, shifted to one negative eigenvalue (closed-form spectrum) from x0 = 0 (rtol):
    equal iteration counts and codes, x within 1e-10 relative, the true residual below 2 tol.  The
    tolerances are about 1e-10 relative, where x is pinned by the solution (see test_gpu_minres.py)."""
    capped(pdl=pdl, **opts)
    cases = [(0, "x0")] + ([(1, "zero")] if key in BOXES else [])
    for nneg, start in cases:
        eps = -_sigma(key, nneg) if nneg else 0.0
        A = _matrix(ab, key, eps=eps)
        n = A.c.nownedrows
        arrays, M = _csr(A)
        rng = np.random.default_rng(51)
        b = rng.standard_normal(n)
        x0 = rng.standard_normal(n) if start == "x0" else np.zeros(n)
        r0 = float(np.linalg.norm(b - M @ x0))
        atol, rtol, warmup = (1e-10 * r0, 0.0, 2) if start == "x0" else (0.0, 1e-10, 0)
        cg = ab.SolverCuda(A)
        try:
            _in_regime(cg, n, key, opts)
            xv = _vec(A, x0)
            code = cg.solve_minres(_vec(A, b), xv, maxits=4000, residualatol=atol, residualrtol=rtol, warmup=warmup)
            x = xv.x[:n]
            ref = _ref((key, "minres", nneg), lambda: minres(M, b, x0=x0, maxits=4000, atol=atol, rtol=rtol))
            assert code == ref["status"] == 0 and cg.c.niterations == ref["niterations"], \
                (nneg, code, cg.c.niterations, ref["niterations"], ref["stop"])
            assert float(np.abs(x - ref["x"]).max()) <= 1e-10 * float(np.abs(ref["x"]).max()), nneg
            assert _residual(arrays, x, b) < 2 * max(atol, rtol * r0), nneg
        finally:
            cg.free()


@pytest.mark.gpu
@pytest.mark.parametrize("pdl", [0, 1])
@pytest.mark.parametrize("mid,key,opts", MATS, ids=[m[0] for m in MATS])
def test_mixed_against_restatement(mid, key, opts, pdl, ab, capped):
    """Mixed-precision CG against tests/mixedref.py, rtol 1e-8 from x0 = 0 and an absolute tolerance from a
    nonzero x0 with warm-up 2: counts within 2 CG steps and 1 reliable update (the dot products' order
    differs, as in test_gpu_mixed.py), rnrm2 the true residual of x, below tol."""
    capped(pdl=pdl, **opts)
    A = _matrix(ab, key)
    n = A.c.nownedrows
    arrays, M = _csr(A)
    rng = np.random.default_rng(61)
    b, x0 = rng.standard_normal(n), rng.standard_normal(n)
    r0 = float(np.linalg.norm(b - M @ x0))
    cg = ab.SolverCuda(A)
    try:
        _in_regime(cg, n, key, opts)
        for i, (xi, atol, rtol, warmup) in enumerate(((np.zeros(n), 0.0, 1e-8, 0), (x0, 1e-10 * r0, 0.0, 2))):
            xv = _vec(A, xi)
            code = cg.solve_mixed(_vec(A, b), xv, maxits=4000, residualatol=atol, residualrtol=rtol, warmup=warmup)
            x = xv.x[:n]
            ref = _ref((key, "mixed", i), lambda: mixed(M, b, x0=xi, maxits=4000, atol=atol, rtol=rtol))
            its, upd = int(cg.c.niterations), int(cg.info()["mixed_reliable_updates"])
            assert abs(its - ref["niterations"]) <= 2 and abs(upd - ref["nupdates"]) <= 1, \
                (i, its, upd, ref["niterations"], ref["nupdates"])
            assert code == ref["status"] == 0 and upd >= 1
            true = _residual(arrays, x, b)
            assert cg.c.rnrm2 == pytest.approx(true, rel=1e-8, abs=1e-13 * max(cg.c.bnrm2, cg.c.r0nrm2)), i
            assert true < ref["tol"], (i, true, ref["tol"])
    finally:
        cg.free()


@pytest.mark.gpu
@pytest.mark.parametrize("pdl", [0, 1])
@pytest.mark.parametrize("mid,key,opts", MATS, ids=[m[0] for m in MATS])
def test_chebyshev_against_restatement(mid, key, opts, pdl, ab, capped):
    """Chebyshev PCG against tests/chebref.py: degrees 0, 2 and 5 with the estimated interval (rtol 1e-8,
    x0 = 0), degree 2 with a given interval from a nonzero x0 (absolute tolerance, warm-up 2), and degree 2
    with tolerances off for an odd number of iterations: equal iteration counts and estimate steps, the
    interval to 1e-8, x within 1e-10 relative, the true residual below 2 tol.  R-MAT with the generator's
    values D + I - Adj, which the Jacobi scaling makes well conditioned."""
    capped(pdl=pdl, **opts)
    A = _matrix(ab, key, values="cheb")
    n = A.c.nownedrows
    arrays, M = _csr(A)
    rng = np.random.default_rng(71)
    b, x0 = rng.standard_normal(n), rng.standard_normal(n)
    lmax = 1.1 * float(np.abs(sp.diags(1 / M.diagonal()) @ M).sum(axis=1).max())     # Gershgorin
    runs = [dict(degree=0, maxits=2000, residualrtol=1e-8), dict(degree=2, maxits=2000, residualrtol=1e-8),
            dict(degree=5, maxits=2000, residualrtol=1e-8),
            dict(degree=2, lmax=lmax, maxits=2000, residualatol=1e-9 * float(np.linalg.norm(b)), warmup=2),
            dict(degree=2, lmin=0.05, lmax=lmax, maxits=17, warmup=2)]
    cg = ab.SolverCuda(A)
    try:
        _in_regime(cg, n, key, opts)
        for i, kw in enumerate(runs):
            xi = x0 if "residualatol" in kw or "residualrtol" not in kw else np.zeros(n)
            xv = _vec(A, xi)
            code = cg.solve_chebyshev(_vec(A, b), xv, **kw)
            x = xv.x[:n]
            ref = _ref((key, "cheb", i), lambda: chebyshev(
                M, b, x0=xi, degree=kw["degree"], lmin=kw.get("lmin", 0.0), lmax=kw.get("lmax", 0.0),
                maxits=kw["maxits"], atol=kw.get("residualatol", 0.0), rtol=kw.get("residualrtol", 0.0)))
            inf = cg.info()
            got = (int(cg.c.niterations), int(inf["cheb_est_iterations"]), code)
            assert got == (ref["niterations"], ref["est_steps"], ref["status"]) and code == 0, (kw, got, ref["stop"])
            assert inf["cheb_lmax"] == pytest.approx(ref["lmax"], rel=1e-8), kw
            assert inf["cheb_lmin"] == pytest.approx(ref["lmin"], rel=1e-8), kw
            assert float(np.abs(x - ref["x"]).max()) <= 1e-10 * float(np.abs(ref["x"]).max()), kw
            if ref["tol"] > 0:
                assert _residual(arrays, x, b) < 2 * ref["tol"], kw
    finally:
        cg.free()


# ---------------------------------------------------------------------------------------------
# the benchmark sizes, uncapped


def _bench_matrix(ab, key, eps=0.0):
    if key == "rmat":
        return ab.SymCsrMatrix.rmat_spd(2_000_000, 20_000_000, seed=42).dsymv_init(eps)
    kind, N = BENCH[key]
    return ab.SymCsrMatrix.stencil_part(kind, N, N, N, 1, 1, 1, 0).dsymv_init(eps)


def _arrays(A):
    n = A.c.nownedrows
    return A.frowptr[:n + 1], A.fcolidx, A.fa


@pytest.mark.gpu
def test_bench_27pt(ab):
    """27-point 224^3: solve_multi with 8 columns column by column against solvempi (rtol 1e-8), Chebyshev
    degree 0 against the first column (the diagonal is constant: Jacobi PCG is CG), fused pipelined CG;
    the return codes, and the true residuals (double-double) of the first column and of pipelined CG below
    2 tol."""
    A = _bench_matrix(ab, "27pt")
    n = A.c.nownedrows
    arrays = _arrays(A)
    rng = np.random.default_rng(81)
    cg = ab.SolverCuda(A)
    try:
        inf = _in_regime(cg, n, "27pt", {}, capped=False)
        rtol = 1e-8
        B = rng.standard_normal((n, 8))
        X = np.zeros((n, 8))
        code, cols = cg.solve_multi(B, X, maxits=3000, residualrtol=rtol)
        assert code == 0 and all(c["converged"] == 1 for c in cols)
        for j in range(8):
            xv = A.vector()
            assert cg.solvempi(_vec(A, B[:, j]), xv, maxits=3000, residualrtol=rtol) == 0
            assert cols[j]["niterations"] == cg.c.niterations, (j, cols[j], cg.c.niterations)
            assert float(np.abs(X[:, j] - xv.x[:n]).max()) <= 1e-10 * float(np.abs(xv.x[:n]).max()), j
        assert _residual(arrays, X[:, 0], B[:, 0]) < 2 * rtol * cols[0]["r0nrm2"]
        b = B[:, 0]
        xv = A.vector()
        code = cg.solve_chebyshev(_vec(A, b), xv, degree=0, maxits=3000, residualrtol=rtol)
        assert code == 0 and cg.c.niterations == cols[0]["niterations"]
        xc = xv.x[:n].copy()
        assert float(np.abs(xc - X[:, 0]).max()) <= 1e-10 * float(np.abs(X[:, 0]).max())
        xv = A.vector()
        assert cg.solve_pipelined(_vec(A, b), xv, maxits=3000, residualrtol=rtol) == 0
        if not STANDIN:
            assert cg.info()["pcg_fused"] == 1 and inf["spmv_symdiag_codes"] > 0
        assert _residual(arrays, xv.x[:n], b) < 2 * rtol * cg.c.r0nrm2
    finally:
        cg.free()
        A.free()


@pytest.mark.gpu
def test_bench_7pt(ab):
    """7-point 256^3: solve_shifted with 4 shifts against solvempi on dsymv_init(sigma) (one solver at a
    time on the device), MINRES, mixed precision and Chebyshev degree 2 for a few iterations against the
    restatements, then each to rtol 1e-8: return code 0, the true residual (double-double) below 2 tol, and
    for the mixed solve rnrm2 equal to it."""
    import torch
    A = _bench_matrix(ab, "7pt")
    n = A.c.nownedrows
    arrays = _arrays(A)
    b = np.random.default_rng(91).standard_normal(n)
    bn = float(np.linalg.norm(b))
    rtol = 1e-8
    cg = ab.SolverCuda(A)
    try:
        _in_regime(cg, n, "7pt", {}, capped=False)
        if not STANDIN:
            # the shifted solve holds 4 columns of x and p besides the single-vector state: a few GB
            free, _ = torch.cuda.mem_get_info()
            assert free > 8 * n * 8 * 12, free
        shifts = [0.0, 0.06, 0.6, 6e-3]                # diagonal 6: sigma / d = 0, 0.01, 0.1, 0.001
        code, X, cols = cg.solve_shifted(b, shifts, maxits=3000, residualrtol=rtol)
        assert code == 0 and all(c["converged"] == 1 for c in cols)
        assert len({c["niterations"] for c in cols}) > 1
        assert _residual(arrays, X[:, 0], b) < 2 * rtol * bn
        for j, sigma in enumerate(shifts):
            Aj = _bench_matrix(ab, "7pt", sigma) if sigma else A
            cgj = ab.SolverCuda(Aj) if sigma else cg
            try:
                xv = Aj.vector()
                assert cgj.solvempi(_vec(Aj, b), xv, maxits=3000, residualrtol=rtol) == 0
                assert cols[j]["niterations"] == cgj.c.niterations, (j, cols[j], cgj.c.niterations)
                assert float(np.abs(X[:, j] - xv.x[:n]).max()) <= 1e-10 * float(np.abs(xv.x[:n]).max()), j
                if j == 2:
                    assert _residual(_arrays(Aj), X[:, j], b) < 2 * rtol * bn
            finally:
                if sigma:
                    cgj.free()
                    Aj.free()
        M = sp.csr_matrix((arrays[2], arrays[1], arrays[0]), shape=(n, n))
        # a few iterations against the restatements (each scipy product of this matrix takes a while)
        xv = A.vector()
        assert cg.solve_minres(_vec(A, b), xv, maxits=7) == 0 and cg.c.niterations == 7
        ref = minres(M, b, maxits=7)
        assert ref["niterations"] == 7
        assert float(np.abs(xv.x[:n] - ref["x"]).max()) <= 1e-10 * float(np.abs(ref["x"]).max())
        xv = A.vector()
        assert cg.solve_mixed(_vec(A, b), xv, maxits=7) == 0 and cg.c.niterations == 7
        ref = mixed(M, b, maxits=7)
        assert ref["niterations"] == 7 and abs(cg.info()["mixed_reliable_updates"] - ref["nupdates"]) <= 1
        assert cg.c.rnrm2 == pytest.approx(ref["rnrm2"], rel=1e-6)
        xv = A.vector()
        assert cg.solve_chebyshev(_vec(A, b), xv, degree=2, lmin=0.1, lmax=2.0, maxits=5) == 0
        ref = chebyshev(M, b, degree=2, lmin=0.1, lmax=2.0, maxits=5)
        assert cg.c.niterations == ref["niterations"] == 5
        assert float(np.abs(xv.x[:n] - ref["x"]).max()) <= 1e-10 * float(np.abs(ref["x"]).max())
        del M
        for name, kw in (("solve_minres", {}), ("solve_mixed", {}), ("solve_chebyshev", {"degree": 2})):
            xv = A.vector()
            code = getattr(cg, name)(_vec(A, b), xv, maxits=3000, residualrtol=rtol, **kw)
            assert code == 0, name
            true = _residual(arrays, xv.x[:n], b)
            assert true < 2 * rtol * cg.c.r0nrm2, (name, true)
            if name == "solve_mixed":
                assert true < rtol * cg.c.r0nrm2
                assert cg.c.rnrm2 == pytest.approx(true, rel=1e-8, abs=1e-13 * cg.c.r0nrm2)
    finally:
        cg.free()
        A.free()


@pytest.mark.gpu
def test_bench_rmat(ab):
    """R-MAT 2 M / 20 M on merge tiles (the generator's values D + I - Adj): Chebyshev degree 2 for a few
    iterations against the restatement, and to rtol 1e-8 with the true residual (double-double) below 2 tol."""
    A = _bench_matrix(ab, "rmat")
    n = A.c.nownedrows
    arrays = _arrays(A)
    b = np.random.default_rng(101).standard_normal(n)
    rtol = 1e-8
    cg = ab.SolverCuda(A)
    try:
        _in_regime(cg, n, "rmat", {}, capped=False)
        M = sp.csr_matrix((arrays[2], arrays[1], arrays[0]), shape=(n, n))
        xv = A.vector()
        assert cg.solve_chebyshev(_vec(A, b), xv, degree=2, lmin=0.1, lmax=2.2, maxits=9) == 0
        ref = chebyshev(M, b, degree=2, lmin=0.1, lmax=2.2, maxits=9)
        assert cg.c.niterations == ref["niterations"] == 9
        assert float(np.abs(xv.x[:n] - ref["x"]).max()) <= 1e-10 * float(np.abs(ref["x"]).max())
        del M
        xv = A.vector()
        assert cg.solve_chebyshev(_vec(A, b), xv, degree=2, maxits=3000, residualrtol=rtol) == 0
        assert _residual(arrays, xv.x[:n], b) < 2 * rtol * cg.c.r0nrm2
    finally:
        cg.free()
        A.free()


# ---------------------------------------------------------------------------------------------
# CPU: the double-double residual and the regime guard


def _check_dd(rowptr, colidx, vals, x, b=None, chunk=7, long_row=64):
    """rows_dd within u |exact| + gamma(m+1)^2 scale of the exact value (Fraction), and of rows_exact."""
    got, scale, m = rows_dd(rowptr, colidx, vals, x, b, chunk=chunk, long_row=long_row)
    want = _fr_rows(rowptr, colidx, vals, x, b)
    ex, exscale, exm = rows_exact(rowptr, colidx, vals, x, b)
    assert np.array_equal(m, exm)
    assert np.allclose(scale, exscale, rtol=1e-12, atol=0)
    bound = gamma(m + 1) ** 2 * scale
    for i, w in enumerate(want):
        err = abs(Fraction(float(got[i])) - w)
        assert err <= Fraction(U) * abs(w) + Fraction(float(bound[i])) * (1 + Fraction(1, 10 ** 6)), (i, got[i], float(w))
        assert abs(got[i] - ex[i]) <= 2 * U * abs(ex[i]) + bound[i] * (1 + 1e-6), i
    return got, ex


@pytest.mark.parametrize("chunk,long_row", [(7, 64), (1 << 16, 64), (5, 12)])
def test_rows_dd_random(chunk, long_row):
    rng = np.random.default_rng(0)
    rowptr, colidx, vals = _random_csr(rng, 300, 40)
    x = rng.standard_normal(300)
    _check_dd(rowptr, colidx, vals, x, chunk=chunk, long_row=long_row)
    _check_dd(rowptr, colidx, vals, x, rng.standard_normal(300), chunk=chunk, long_row=long_row)


def test_rows_dd_catastrophic_cancellation():
    """Rows that cancel to about 1e-16 of their terms, and b - A x with b = fl(A x): the double-double
    value is within its bound of the exact one, where a plain float64 sum has no correct digit."""
    rng = np.random.default_rng(3)
    n, L = 50, 30
    rowptr = np.arange(0, n * L + 1, L, dtype=np.int64)
    colidx = np.tile(np.arange(L, dtype=np.int32), n)
    x = rng.standard_normal(L) * 2.0 ** rng.integers(-20, 20, L)
    vals = np.empty(n * L)
    for i in range(n):
        v = rng.standard_normal(L)
        v[-1] = -float(sum(Fraction(float(v[k])) * Fraction(float(x[k])) for k in range(L - 1)) / Fraction(float(x[-1])))
        vals[i * L:(i + 1) * L] = v
    got, ex = _check_dd(rowptr, colidx, vals, x)
    naive = np.array([vals[i * L:(i + 1) * L] @ x for i in range(n)])
    assert np.abs(naive - ex).max() > 1e3 * np.abs(got - ex).max()
    _check_dd(rowptr, colidx, vals, x, naive)
    _check_dd(rowptr, colidx, vals, x, naive, long_row=8)        # every row through math.fsum


@pytest.mark.parametrize("e", [50, -50])
def test_rows_dd_extreme_exponents(e):
    rng = np.random.default_rng(4)
    rowptr, colidx, vals = _random_csr(rng, 120, 25, lambda k: rng.standard_normal(k) * 2.0 ** e)
    x = rng.standard_normal(120) * 2.0 ** e
    _check_dd(rowptr, colidx, vals, x)
    _check_dd(rowptr, colidx, vals, x, rng.standard_normal(120) * 2.0 ** (2 * e))


def test_rows_dd_integer_data_exact():
    """Integer data: every product and partial sum is exact, so the value equals the exact sum bitwise."""
    rng = np.random.default_rng(5)
    rowptr, colidx, vals = _random_csr(rng, 200, 60, lambda k: rng.integers(-7, 8, k).astype(np.float64))
    x = rng.integers(-9, 10, 200).astype(np.float64)
    b = rng.integers(-50, 51, 200).astype(np.float64)
    for bb in (None, b):
        got, ex = _check_dd(rowptr, colidx, vals, x, bb, chunk=16, long_row=30)
        assert np.array_equal(got, ex)


def _stencil_csr(kind, nx, ny, nz):
    import acg_b200 as ab
    from acg_b200 import matgen as mg
    n, r, c, v = (mg.stencil3d_27pt if kind == 27 else mg.laplace3d_7pt)(nx, ny, nz)
    A = ab.SymCsrMatrix.init_real_double(n, r, c, v).dsymv_init(0.0)
    out = (A.frowptr[:n + 1].copy(), A.fcolidx[:A.frowptr[n]].copy())
    A.free()
    return n, out


def test_regime_guard():
    """Every matrix of this file takes at least two trips of every capped grid on 114 and 132 SMs (moderate
    sizes: one CTA per SM, slice CTAs of up to 256 threads) and of every grid at any occupancy up to 2048
    threads per SM (benchmark sizes), from the host plans and row counts."""
    import acg_b200 as ab
    for key, (kind, box) in BOXES.items():
        n, (rp, ci) = _stencil_csr(kind, *box)
        assert ab.symdiag_host(rp, ci)["reason"] == "eligible", key
        nsl = ab.slices_host(rp, ci)["nslices"]
        for sms in SM_COUNTS:
            assert n // 2 >= 2 * sms * BLAS1_THREADS, (key, sms)
            assert nsl >= 2 * sms * 256 // 32, (key, nsl, sms)
        assert n % 2 == (1 if key == "7pt" else 0) and n % 32
    n, r, c, v = _coo("rmat")
    A = ab.SymCsrMatrix.init_real_double(n, r, c, v).dsymv_init(0.0)
    rp = A.frowptr[:n + 1].copy()
    A.free()
    ntiles = len(ab.merge_plan_host(rp, items=MERGE_ITEMS)["tiles"])
    for sms in SM_COUNTS:
        assert n // 2 >= 2 * sms * BLAS1_THREADS and ntiles >= 2 * sms, (ntiles, sms)
    # benchmark sizes: the slices of one interior plane (the middle plane of a three-plane box: every plane
    # starts at a multiple of 32 rows, so its slices are those of every interior plane of the full box)
    for key, (kind, N) in BENCH.items():
        n = N ** 3
        _, (rp, ci) = _stencil_csr(kind, N, N, 3)
        sl = ab.slices_host(rp, ci)
        plane = sl["slices"][:, 0]
        per_plane = int(((plane >= N * N) & (plane + 32 <= 2 * N * N)).sum())
        assert ab.symdiag_host(rp, ci)["reason"] == "eligible"
        for sms in SM_COUNTS:
            assert n // 2 >= 2 * sms * MAX_THREADS_PER_SM, (key, sms)
            assert per_plane * (N - 2) >= 2 * sms * MAX_THREADS_PER_SM // 32, (key, per_plane, sms)
    n, nnz = 2_000_000, None
    A = ab.SymCsrMatrix.rmat_spd(n, 20_000_000, seed=42).dsymv_init(0.0)
    nnz = int(A.c.fnpnzs)
    A.free()
    for sms in SM_COUNTS:
        assert n // 2 >= 2 * sms * MAX_THREADS_PER_SM
        # merge-path tiles of MERGE_ITEMS rows + nonzeros; CTAs of 128 threads
        assert (n + nnz) // MERGE_ITEMS >= 2 * sms * MAX_THREADS_PER_SM // 128, (nnz, sms)
