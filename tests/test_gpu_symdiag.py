"""The mirrored-diagonal SpMV (spmv_symdiag_kernel, option "spmv_symdiag") on the H100.

* Every instantiated (UB, T) shape in all three epilogue modes on 27- and 7-point stencil boxes built
  with dsymv_init(sigma), sigma != 0: on integer data bitwise equal to the exact product and dots; on
  real data y bitwise equal to the same solver built with spmv_symdiag=0 (the slice kernel), which adds
  the same products in the same order.
* The fall-backs: full storage that is not exactly symmetric (one mirrored value changed) and a plan
  with exception rows keep the slice kernel, and stay exact.
* solvempi and solve_pipelined against spmv_symdiag=0: same iterations, same solution to 1e-10.
The host plan and the addressing are checked on the CPU in tests/test_symdiag.py."""
import numpy as np
import pytest

from acg_b200 import matgen as mg
from test_gpu_kernel_variants import DEFAULTS, SLICE_VARIANTS, _vid, big_stencil

OPTS = dict(DEFAULTS, spmv_symdiag=1)


@pytest.fixture
def options(ab):
    def set_(**kw):
        for k, v in dict(OPTS, **kw).items():
            ab.set_option(k, v)
    yield set_
    for k, v in OPTS.items():
        ab.set_option(k, v)


def _matrix(ab, n, r, c, kind, seed, sigma):
    rng = np.random.default_rng(seed)
    if kind == "int":
        v = rng.integers(-3, 4, len(r)).astype(np.float64)
        v[r == c] = rng.integers(1, 9, int((r == c).sum()))
    else:
        v = rng.standard_normal(len(r))
        v[r == c] += 30.0
    return ab.SymCsrMatrix.init_real_double(n, r, c, v).dsymv_init(sigma)


def _inputs(n, kind, seed):
    rng = np.random.default_rng(seed)
    if kind == "int":
        return rng.integers(-3, 4, n).astype(np.float64), rng.integers(-40, 41, n).astype(np.float64)
    return rng.standard_normal(n), rng.standard_normal(n)


def _exact(A, x, b):
    """y = A x, r = b - A x and the dots on integer data: every partial sum is an exact integer."""
    import scipy.sparse as sps
    n = len(x)
    M = sps.csr_matrix((A.fa.copy(), A.fcolidx.copy(), A.frowptr.copy()), shape=(n, n))
    y = M @ x
    r = b - y
    return {0: (y, 0.0), 1: (y, float(x @ y)), 2: (r, float(r @ r))}


def _check_exact(cg, A, x, b, tag):
    want = _exact(A, x, b)
    for mode in (0, 1, 2):
        y, dot = cg.spmv_mode(mode, x, b if mode == 2 else None)
        wy, wdot = want[mode]
        bad = np.flatnonzero(y != wy)
        assert bad.size == 0, (tag, mode, bad[:10], y[bad[:10]], wy[bad[:10]])
        assert dot == wdot, (tag, mode, dot, wdot)


BOXES = {"27pt": lambda: mg.stencil3d_27pt(21, 20, 19), "7pt": lambda: mg.laplace3d_7pt(31, 17, 23)}
NDIAG = {"27pt": 14, "7pt": 4}


@pytest.mark.gpu
@pytest.mark.parametrize("variant", SLICE_VARIANTS, ids=[_vid(v) for v in SLICE_VARIANTS])
@pytest.mark.parametrize("box", sorted(BOXES))
def test_symdiag_variant_all_modes(variant, box, ab, options):
    UB, T = variant
    n, r, c, _ = BOXES[box]()
    assert n % 32
    seed = 300 + SLICE_VARIANTS.index(variant)
    for kind, sigma in (("int", 2.0), ("real", 0.75)):
        A = _matrix(ab, n, r, c, kind, seed, sigma)
        x, b = _inputs(n, kind, seed + 1)
        got = {}
        for on in (1, 0):
            options(spmv_symdiag=on, slice_ub=UB, slice_threads=T, spmv_merge=0)
            cg = ab.SolverCuda(A)
            inf = cg.info()
            assert inf["spmv_slices"] > 0 and inf["spmv_slice_ub"] == UB and inf["spmv_slice_threads"] == T
            assert inf["spmv_symdiag_diagonals"] == (NDIAG[box] if on else 0), inf
            if on:
                assert inf["spmv_symdiag_bytes"] >= NDIAG[box] * n * 8
                assert inf["spmv_min_bytes"] < (inf["spmv_slice_value_bytes"] + 18 * inf["spmv_slice_rows"])
            if kind == "int":
                _check_exact(cg, A, x, b, (box, variant, on))
            got[on] = [cg.spmv_mode(m, x, b if m == 2 else None)[0] for m in (0, 1, 2)]
            cg.free()
        for m in (0, 1, 2):
            assert np.array_equal(got[1][m].view(np.int64), got[0][m].view(np.int64)), (box, variant, kind, m)
        A.free()


@pytest.mark.gpu
def test_symdiag_one_cta_per_sm(ab, options):
    """One CTA per SM on a larger box: every warp walks several slices, and their mirror reads reach back
    across other warps' slices."""
    n, r, c, _ = mg.stencil3d_27pt(47, 48, 33)
    A = _matrix(ab, n, r, c, "int", 7, 1.0)
    x, b = _inputs(n, "int", 8)
    options(slice_max_ctas=1)
    cg = ab.SolverCuda(A)
    inf = cg.info()
    assert inf["spmv_symdiag_diagonals"] == 14 and inf["spmv_slice_grid"] <= inf["num_sms"]
    assert inf["spmv_slices"] >= 2 * inf["spmv_slice_grid"] * (inf["spmv_slice_threads"] // 32)
    _check_exact(cg, A, x, b, "onecta")
    cg.free()
    A.free()


@pytest.mark.gpu
def test_not_symmetric_falls_back(ab, options):
    """Full storage whose lower entry differs from its mirror in one value: the device check rejects the
    layout, the slice kernel runs, the product is the exact one of the stored (unsymmetric) arrays."""
    n, r, c, _ = BOXES["27pt"]()
    A = _matrix(ab, n, r, c, "int", 9, 0.0)
    x, b = _inputs(n, "int", 10)
    options()
    cg = ab.SolverCuda(A)
    assert cg.info()["spmv_symdiag_diagonals"] == 14
    cg.free()
    i = n // 2
    rp, ci = A.frowptr, A.fcolidx
    k = rp[i]
    assert ci[k] < i
    A.fa[k] += 1.0                                # a[i, ci[k]] no longer equals a[ci[k], i]
    cg = ab.SolverCuda(A)
    inf = cg.info()
    assert inf["spmv_symdiag_diagonals"] == 0 and inf["spmv_symdiag_bytes"] == 0 and inf["spmv_slices"] > 0
    _check_exact(cg, A, x, b, "unsymmetric")
    cg.free()
    A.free()


@pytest.mark.gpu
def test_exception_rows_fall_back(ab, options):
    n, r, c = big_stencil(True)
    A = _matrix(ab, n, r, c, "int", 11, 1.0)
    x, b = _inputs(n, "int", 12)
    options()
    cg = ab.SolverCuda(A)
    inf = cg.info()
    assert inf["spmv_slice_exc"] > 0 and inf["spmv_symdiag_diagonals"] == 0
    _check_exact(cg, A, x, b, "exc")
    cg.free()
    A.free()


@pytest.mark.gpu
@pytest.mark.parametrize("solver", ["solvempi", "solve_pipelined"])
@pytest.mark.parametrize("box", sorted(BOXES))
def test_solvers_match_slice_kernel(solver, box, ab, options):
    n, r, c, _ = BOXES[box]()
    A = _matrix(ab, n, r, c, "real", 13, 0.5)
    b = A.vector()
    b.x[:] = np.random.default_rng(14).standard_normal(len(b.x))
    res = {}
    for on in (1, 0):
        options(spmv_symdiag=on)
        cg = ab.SolverCuda(A)
        assert cg.info()["spmv_symdiag_diagonals"] == (NDIAG[box] if on else 0)
        x = A.vector()
        code = getattr(cg, solver)(b, x, maxits=2000, residualrtol=1e-10)
        res[on] = (code, cg.c.niterations, cg.c.rnrm2 / cg.c.r0nrm2, x.x.copy())
        cg.free()
    (c1, it1, rr1, x1), (c0, it0, rr0, x0) = res[1], res[0]
    assert c1 == c0 == 0 and it1 == it0 > 0
    assert rr1 < 1e-10 and rr0 < 1e-10 and abs(rr1 - rr0) <= 1e-10
    assert np.abs(x1 - x0).max() <= 1e-10 * np.abs(x0).max()
    A.free()
