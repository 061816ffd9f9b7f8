"""The coded mirrored diagonals (option "symdiag_codes"): one-byte codes into a table of the diagonals'
distinct values, on the H100.

* Every instantiated (UB, T) shape in all three epilogue modes on the 27- and 7-point boxes of
  test_gpu_symdiag.py, with integer-valued and stencil-valued (-1, 26) matrices: the codes are taken, and
  y and the dots are bitwise those of the same solver built with symdiag_codes=0 and of the exact product.
* The table's boundaries: exactly 256 distinct bit patterns take codes and 257 keep the fp64 diagonals;
  +0.0 and -0.0 stay two values, and so do two values one ulp apart; a matrix that is not exactly
  symmetric keeps the slice kernel; random real values keep the fp64 diagonals.
* The solvers on coded matrices -- fused and two-kernel pipelined CG, classic CG, shifted systems --
  against symdiag_codes=0 and the oracle.
"""
import numpy as np
import pytest

from acg_b200 import matgen as mg
from test_gpu_kernel_variants import DEFAULTS, SLICE_VARIANTS, _vid

pytestmark = pytest.mark.gpu

OPTS = dict(DEFAULTS, spmv_symdiag=1, symdiag_codes=1, pcg_fused=1)


@pytest.fixture
def options(ab):
    def set_(**kw):
        for k, v in dict(OPTS, **kw).items():
            ab.set_option(k, v)
    yield set_
    for k, v in OPTS.items():
        ab.set_option(k, v)


BOXES = {"27pt": lambda: mg.stencil3d_27pt(21, 20, 19), "7pt": lambda: mg.laplace3d_7pt(31, 17, 23)}
NDIAG = {"27pt": 14, "7pt": 4}


def _values(r, c, kind, seed):
    if kind == "stencil":
        return np.where(r == c, 26.0, -1.0)
    rng = np.random.default_rng(seed)
    v = rng.integers(-3, 4, len(r)).astype(np.float64)
    v[r == c] = rng.integers(1, 9, int((r == c).sum()))
    return v


def _ncodes_expected(A):
    """Distinct bit patterns among the stored (upper) entries and the +0.0 of absent entries and margins."""
    rp, ci, fa = A.frowptr, A.fcolidx, A.fa
    rows = np.repeat(np.arange(len(rp) - 1), np.diff(rp))
    upper = fa[: rp[-1]][ci[: rp[-1]] >= rows]
    return len(set(upper.view(np.uint64).tolist()) | {0})


def _exact(A, x, b):
    import scipy.sparse as sps
    n = len(x)
    M = sps.csr_matrix((A.fa.copy(), A.fcolidx.copy(), A.frowptr.copy()), shape=(n, n))
    y = M @ x
    r = b - y
    return {0: (y, 0.0), 1: (y, float(x @ y)), 2: (r, float(r @ r))}


def _products(cg, x, b):
    return [cg.spmv_mode(m, x, b if m == 2 else None) for m in (0, 1, 2)]


def _same_bits(got, want, tag, exact_dots=True):
    for m, ((y1, d1), (y0, d0)) in enumerate(zip(got, want)):
        bad = np.flatnonzero(y1.view(np.int64) != y0.view(np.int64))
        assert bad.size == 0, (tag, m, bad[:10], y1[bad[:10]], y0[bad[:10]])
        if exact_dots:
            assert np.float64(d1).view(np.int64) == np.float64(d0).view(np.int64), (tag, m, d1, d0)
        else:
            assert d1 == pytest.approx(d0, rel=1e-13, abs=0.0), (tag, m, d1, d0)


@pytest.mark.parametrize("variant", SLICE_VARIANTS, ids=[_vid(v) for v in SLICE_VARIANTS])
@pytest.mark.parametrize("box", sorted(BOXES))
def test_codes_variant_all_modes(variant, box, ab, options):
    UB, T = variant
    n, r, c, _ = BOXES[box]()
    seed = 500 + SLICE_VARIANTS.index(variant)
    rng = np.random.default_rng(seed + 1)
    x, b = rng.integers(-3, 4, n).astype(np.float64), rng.integers(-40, 41, n).astype(np.float64)
    for kind in ("int", "stencil"):
        A = ab.SymCsrMatrix.init_real_double(n, r, c, _values(r, c, kind, seed)).dsymv_init(0.0)
        got = {}
        for codes in (1, 0):
            options(symdiag_codes=codes, slice_ub=UB, slice_threads=T, spmv_merge=0)
            cg = ab.SolverCuda(A)
            inf = cg.info()
            assert inf["spmv_slice_ub"] == UB and inf["spmv_slice_threads"] == T
            assert inf["spmv_symdiag_diagonals"] == NDIAG[box], inf
            if codes:
                assert inf["spmv_symdiag_codes"] == _ncodes_expected(A) > 0, inf
                assert inf["spmv_symdiag_code_bytes"] * 8 == inf["spmv_symdiag_bytes"]
            else:
                assert inf["spmv_symdiag_codes"] == 0 and inf["spmv_symdiag_code_bytes"] == 0
            got[codes] = _products(cg, x, b)
            cg.free()
        _same_bits(got[1], got[0], (box, variant, kind))
        want = _exact(A, x, b)
        for m in (0, 1, 2):
            y, dot = got[1][m]
            assert np.array_equal(y, want[m][0]) and dot == want[m][1], (box, variant, kind, m)
        A.free()


def _codes_of(ab, options, A, x, b, exact_dots=True, **kw):
    """symdiag_codes of a solver built on A, and its products bitwise against symdiag_codes=0."""
    got = {}
    ncodes = None
    for codes in (1, 0):
        options(symdiag_codes=codes, **kw)
        cg = ab.SolverCuda(A)
        inf = cg.info()
        if codes:
            ncodes = inf["spmv_symdiag_codes"]
        diags = inf["spmv_symdiag_diagonals"]
        got[codes] = _products(cg, x, b)
        cg.free()
    _same_bits(got[1], got[0], kw, exact_dots)
    return ncodes, diags, got[1]


@pytest.mark.parametrize("ndistinct,coded", [(255, True), (256, False)])
def test_table_size_boundary(ndistinct, coded, ab, options):
    """Upper entries cycling through `ndistinct` nonzero integers, plus the +0.0 of the margins: 256
    patterns fit the table, 257 do not."""
    n, r, c, _ = BOXES["27pt"]()
    v = 1.0 + (np.arange(len(r)) % ndistinct)
    A = ab.SymCsrMatrix.init_real_double(n, r, c, v).dsymv_init(0.0)
    assert _ncodes_expected(A) == ndistinct + 1
    rng = np.random.default_rng(61)
    x, b = rng.integers(-3, 4, n).astype(np.float64), rng.integers(-40, 41, n).astype(np.float64)
    ncodes, diags, got = _codes_of(ab, options, A, x, b)
    assert diags == 14
    assert ncodes == (ndistinct + 1 if coded else 0)
    want = _exact(A, x, b)
    for m in (0, 1, 2):
        assert np.array_equal(got[m][0], want[m][0]) and got[m][1] == want[m][1]
    A.free()


def test_signed_zeros_and_one_ulp_stay_distinct(ab, options):
    n, r, c, _ = BOXES["27pt"]()
    one_up = np.nextafter(1.0, 2.0)
    v = np.where(r == c, 26.0, -1.0)
    off = np.flatnonzero(r != c)
    v[off[3::11]] = 1.0
    v[off[5::11]] = one_up                 # one ulp above 1.0
    A = ab.SymCsrMatrix.init_real_double(n, r, c, v).dsymv_init(0.0)
    # -0.0 on the main diagonal of the full storage (the expansion turns a -0.0 input into +0.0; diagonal
    # entries have no mirror, so the matrix stays exactly symmetric), next to the margins' +0.0
    rp = A.frowptr
    rows = np.repeat(np.arange(n), np.diff(rp[: n + 1]))
    diag = np.flatnonzero(A.fcolidx[: rp[n]] == rows)
    A.fa[diag[::5]] = -0.0
    assert _ncodes_expected(A) == 6        # +0.0, -0.0, -1, 1, 1 + ulp, 26
    rng = np.random.default_rng(71)
    x, b = rng.integers(-3, 4, n).astype(np.float64), rng.integers(-40, 41, n).astype(np.float64)
    x[::5] = -0.0
    # y bitwise; the dots to rounding: the rows' sums are not integers here, and with codes the product
    # kernel may run more CTAs, which adds the per-CTA partial dots in another grouping
    ncodes, diags, _ = _codes_of(ab, options, A, x, b, exact_dots=False)
    assert diags == 14 and ncodes == 6
    A.free()


def test_unsymmetric_and_real_valued_keep_fp64(ab, options):
    n, r, c, _ = BOXES["27pt"]()
    rng = np.random.default_rng(81)
    x, b = rng.integers(-3, 4, n).astype(np.float64), rng.integers(-40, 41, n).astype(np.float64)
    # not exactly symmetric: no mirrored diagonals at all, the slice kernel
    A = ab.SymCsrMatrix.init_real_double(n, r, c, _values(r, c, "stencil", 0)).dsymv_init(0.0)
    i = n // 2
    k = A.frowptr[i]
    assert A.fcolidx[k] < i
    A.fa[k] += 1.0
    options()
    cg = ab.SolverCuda(A)
    inf = cg.info()
    assert inf["spmv_symdiag_diagonals"] == 0 and inf["spmv_symdiag_codes"] == 0 and inf["spmv_slices"] > 0
    got = _products(cg, x, b)
    want = _exact(A, x, b)
    for m in (0, 1, 2):
        assert np.array_equal(got[m][0], want[m][0]) and got[m][1] == want[m][1]
    cg.free()
    A.free()
    # random real values: far more than 256 patterns
    v = rng.standard_normal(len(r))
    v[r == c] += 30.0
    R = ab.SymCsrMatrix.init_real_double(n, r, c, v).dsymv_init(0.5)
    cg = ab.SolverCuda(R)
    inf = cg.info()
    assert inf["spmv_symdiag_diagonals"] == 14 and inf["spmv_symdiag_codes"] == 0
    assert inf["pcg_fused_min_bytes"] == inf["spmv_slice_rows"] * (8 * 14 + 96)
    cg.free()
    R.free()


SOLVE_BOXES = {
    "27pt-full": lambda: mg.stencil3d_27pt(32, 20, 19),      # every row in a slice
    "27pt-ragged": lambda: mg.stencil3d_27pt(21, 20, 19),    # tile rows after the slices
    "7pt": lambda: mg.laplace3d_7pt(31, 17, 23),
}


@pytest.mark.parametrize("box", sorted(SOLVE_BOXES))
def test_solvers_on_codes(box, ab, options, oracle):
    n, r, c, v = SOLVE_BOXES[box]()
    A = ab.SymCsrMatrix.init_real_double(n, r, c, v).dsymv_init(0.0)
    b = A.vector()
    b.x[:] = np.random.default_rng(91).standard_normal(len(b.x))
    csr = (A.frowptr.copy(), A.fcolidx.copy(), A.fa.copy())
    runs = [("solve_pipelined", 1), ("solve_pipelined", 0), ("solvempi", 1)]
    res = {}
    for codes in (1, 0):
        cg = None
        for solver, fused in runs:
            options(symdiag_codes=codes, pcg_fused=fused)
            if cg is None:
                cg = ab.SolverCuda(A)
                inf = cg.info()
                assert inf["spmv_symdiag_diagonals"] > 0
                assert (inf["spmv_symdiag_codes"] > 0) == bool(codes), inf
                if codes:
                    nd = inf["spmv_symdiag_diagonals"]
                    assert inf["pcg_fused_min_bytes"] == inf["spmv_slice_rows"] * (nd + 96)
            x = A.vector()
            code = getattr(cg, solver)(b, x, maxits=2000, residualrtol=1e-10)
            assert cg.info()["pcg_fused"] == (fused if solver == "solve_pipelined" else 0)
            res[codes, solver, fused] = (code, cg.c.niterations, cg.c.rnrm2 / cg.c.r0nrm2, x.x.copy())
        shifts = [0.0, 0.5, 2.0]
        scode, X, cols = cg.solve_shifted(b.x[:n].copy(), shifts, maxits=2000, residualrtol=1e-10)
        res[codes, "shifted", 0] = (scode, [cl["niterations"] for cl in cols], X.copy())
        cg.free()
    for solver, fused in runs:
        (c1, it1, rr1, x1), (c0, it0, rr0, x0) = res[1, solver, fused], res[0, solver, fused]
        assert c1 == c0 == 0 and it1 == it0 > 0, (solver, fused, it1, it0)
        assert rr1 < 1e-10 and abs(rr1 - rr0) <= 1e-10
        assert np.abs(x1 - x0).max() <= 1e-10 * np.abs(x0).max()
        ref = (oracle.cg if solver == "solvempi" else oracle.cg_pipelined)(csr, b.x, maxits=2000, rtol=1e-10)
        assert ref["status"] == 0 and ref["niterations"] == it1
        assert np.abs(x1 - ref["x"]).max() <= 1e-9 * np.abs(ref["x"]).max()
    (s1, its1, X1), (s0, its0, X0) = res[1, "shifted", 0], res[0, "shifted", 0]
    assert s1 == s0 == 0 and its1 == its0
    assert np.abs(X1 - X0).max() <= 1e-10 * np.abs(X0).max()
    A.free()
