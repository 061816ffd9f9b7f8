"""Several right-hand sides on the H100: the multi-vector product in every epilogue mode against an
exact reference, and acgsolvercuda_solve_multi against acgsolvercuda_solvempi column by column.

The multi-vector product is spmm_slices_kernel (rows in pattern slices, plain and with exception
rows) plus spmm_rows_kernel (every other row: tile, merge-tile, medium and long rows of the
single-vector plan, one or eight lanes per row).  Each plan shape is forced through the plan options
as in test_gpu_kernel_variants.py, and the product is run through acgsolvercuda_spmm_mode for
nrhs = 1, 2, 3, 4, 5, 8 (block widths K = 1, 2, 4, 8, with padding columns for 3 and 5):
* integer data: every column of Y and every fused dot BITWISE equal to the exact value;
* real data: every row within 2 gamma(m+1) sum |a x| (+ |b|) of the correctly rounded value.
Y is poisoned first, so a row no kernel writes would come back NaN.
"""
import functools
import zlib

import numpy as np
import pytest

from exactref import dot_exact, gamma, rows_exact
from test_gpu_kernel_variants import DEFAULTS, ragged, rmat, slice_matrix

NRHS = (1, 2, 3, 4, 5, 8)

# plan shapes: (name, matrix key, options)
PLANS = [
    ("slices", "slice", {}),
    ("slices-exc", "slice-exc", {}),
    ("tiles", "slice", {"spmv_slices": 0}),
    ("merge-tiles", "rmat", {}),
    ("medium+long", "rmat", {"spmv_merge": 0, "spmv_medium": 96, "spmv_slices": 0}),
    ("tiles+long", "ragged", {"spmv_merge": 0}),
]


def _structure(key):
    return {"slice": lambda: slice_matrix(False), "slice-exc": lambda: slice_matrix(True),
            "rmat": rmat, "ragged": lambda: ragged(8, 1)}[key]()


@pytest.fixture
def options(ab):
    def set_(**kw):
        for k, v in kw.items():
            ab.set_option(k, v)
    yield set_
    for k, v in DEFAULTS.items():
        ab.set_option(k, v)


@functools.lru_cache(maxsize=None)
def _data(key, kind):
    """Values, 8 columns of X and B, and the exact per-column answers of the three modes."""
    import acg_b200 as ab
    n, r, c = _structure(key)
    rng = np.random.default_rng(zlib.crc32(f"{key}/{kind}".encode()))
    diag = r == c
    if kind == "int":
        v = rng.integers(-3, 4, len(r)).astype(np.float64)
        v[diag] = rng.integers(1, 9, int(diag.sum()))
        X = rng.integers(-3, 4, (n, 8)).astype(np.float64)
        B = rng.integers(-40, 41, (n, 8)).astype(np.float64)
    else:
        v = rng.standard_normal(len(r))
        v[diag] += 4.0
        X = rng.standard_normal((n, 8))
        B = None
    A = ab.SymCsrMatrix.init_real_double(n, r, c, v).dsymv_init(0.0)
    csr = (A.frowptr.copy(), A.fcolidx.copy(), A.fa.copy())
    ex = {"y": [], "ys": [], "r": [], "rs": [], "m": None}
    Bs = []
    for j in range(8):
        y, s, m = rows_exact(*csr, X[:, j])
        b = B[:, j] if B is not None else y + 1e-8 * rng.standard_normal(n)
        rr, rs, _ = rows_exact(*csr, X[:, j], b)
        ex["y"].append(y); ex["ys"].append(s); ex["r"].append(rr); ex["rs"].append(rs); ex["m"] = m
        Bs.append(b)
    return A, np.ascontiguousarray(X), np.ascontiguousarray(np.stack(Bs, axis=1)), ex


def _check_mode(kind, mode, X, Y, dots, ex, k):
    assert not np.isnan(Y).any()
    for j in range(k):
        want = ex["r"][j] if mode == 2 else ex["y"][j]
        scale = ex["rs"][j] if mode == 2 else ex["ys"][j]
        if kind == "int":
            assert np.array_equal(Y[:, j], want), (mode, j, np.flatnonzero(Y[:, j] != want)[:5])
        else:
            bound = 2 * gamma(ex["m"] + 1) * scale
            assert np.all(np.abs(Y[:, j] - want) <= bound), (mode, j, float(np.max(np.abs(Y[:, j] - want) - bound)))
        if mode == 0:
            assert dots[j] == 0.0
            continue
        # the fused dot of the kernel's own y (in mode 2 y carries the rounding of a cancelling b - A x)
        u = X[:, j] if mode == 1 else Y[:, j]
        wd = dot_exact(u, Y[:, j])
        if kind == "int":
            assert dots[j] == wd, (mode, j, dots[j], wd)
        else:
            bound = 2 * gamma(len(u) + 1) * float(np.abs(u * Y[:, j]).sum())
            assert abs(dots[j] - wd) <= bound, (mode, j, dots[j], wd, bound)


@pytest.mark.gpu
@pytest.mark.parametrize("plan", PLANS, ids=[p[0] for p in PLANS])
@pytest.mark.parametrize("kind", ["int", "real"])
def test_spmm_all_modes(plan, kind, ab, options):
    name, key, opts = plan
    options(**opts)
    A, X8, B8, ex = _data(key, kind)
    cg = ab.SolverCuda(A)
    inf = cg.info()
    if name.startswith("slices"):
        assert inf["spmv_slices"] > 0 and (inf["spmv_slice_exc"] > 0) == (name == "slices-exc")
    elif name == "tiles":
        assert inf["spmv_slices"] == 0 and inf["spmv_ntiles"] > 0
    elif name == "merge-tiles":
        assert inf["spmv_merge_tiles"] > 0
    elif name == "medium+long":
        assert inf["spmv_nlong"] > 0 and inf["spmv_nmedium"] > 0 and inf["spmv_merge_tiles"] == 0
    else:
        assert inf["spmv_nlong"] > 0 and inf["spmv_ntiles"] > 0
    try:
        for k in NRHS:
            X = np.ascontiguousarray(X8[:, :k])
            B = np.ascontiguousarray(B8[:, :k])
            for mode in (0, 1, 2):
                Y, dots = cg.spmm_mode(mode, X, B if mode == 2 else None)
                _check_mode(kind, mode, X, Y, dots, ex, k)
    finally:
        cg.free()


# ---------------------------------------------------------------------------------------------
# solves


@functools.lru_cache(maxsize=None)
def _spd(key):
    """The 27-point stencil itself (long runs, slices: the same summation order as the single-vector
    kernel), or a structure with diagonal 1 and off-diagonal -1/(2 max(deg_i, deg_j)): eigenvalues in
    [0.5, 1.5] by Gershgorin.  Where the multi-vector kernels sum a row in another order than the
    single-vector plan (merge tiles, tiles, medium and long rows), the columns then agree with solvempi
    to rounding instead of drifting apart at the condition number of a hub row."""
    import acg_b200 as ab
    from acg_b200 import matgen as mg
    if key == "27pt":
        n, r, c, v = mg.stencil3d_27pt(30, 31, 29)
        return ab.SymCsrMatrix.init_real_double(n, r, c, v).dsymv_init(0.0)
    n, r, c = _structure(key)
    off = r != c
    r, c = r[off], c[off]
    deg = np.bincount(r, minlength=n) + np.bincount(c, minlength=n)
    v = -0.5 / np.maximum(deg[r], deg[c])
    d = np.arange(n, dtype=np.int32)
    r = np.concatenate([r, d]); c = np.concatenate([c, d]); v = np.concatenate([v, np.ones(n)])
    o = np.lexsort((c, r))
    return ab.SymCsrMatrix.init_real_double(n, r[o], c[o], v[o]).dsymv_init(0.0)


SOLVE_PLANS = [("slices", "27pt", {}), ("slices-exc", "slice-exc", {}), ("tiles", "slice", {"spmv_slices": 0}),
               ("merge-tiles", "rmat", {}), ("medium+long", "rmat", {"spmv_merge": 0, "spmv_medium": 96, "spmv_slices": 0}),
               ("tiles+long", "ragged", {"spmv_merge": 0})]


@pytest.mark.gpu
@pytest.mark.parametrize("plan", SOLVE_PLANS, ids=[p[0] for p in SOLVE_PLANS])
def test_solve_multi_against_solvempi(plan, ab, options, oracle):
    """Each column of solve_multi against solvempi on that column (same solver, same plan): identical
    iteration counts, ||r|| within 1e-10 ||r0||, x within 1e-10 relative.  Right-hand sides scaled by
    4^j and an absolute tolerance make the columns stop at different iterations; X0 is random; one
    column has b = x0 = 0 and is converged at r0.  Then the oracle on the same columns, and maxits = 0
    returning X bitwise."""
    name, key, opts = plan
    options(**opts)
    A = _spd(key)
    n = A.c.nownedrows
    csr = (A.frowptr.copy(), A.fcolidx.copy(), A.fa.copy())
    cg = ab.SolverCuda(A)
    rng = np.random.default_rng(11)
    try:
        for k, warmup in ((5, 0), (8, 2), (3, 1), (1, 0)):
            B = rng.standard_normal((n, k)) * 4.0 ** np.arange(k)
            X0 = rng.standard_normal((n, k))
            if k > 2:
                B[:, 2] = 0.0; X0[:, 2] = 0.0
            atol = 1e-6 * float(np.linalg.norm(B[:, 0]))
            X = X0.copy()
            code, cols = cg.solve_multi(B, X, maxits=400, residualatol=atol, warmup=warmup)
            assert code == 0
            assert cg.c.niterations == max(c["niterations"] for c in cols)
            if k > 2:
                assert cols[2]["niterations"] == 0 and cols[2]["converged"] == 1 and not X[:, 2].any()
            if k > 1:
                assert len({c["niterations"] for c in cols}) > 1
            for j in range(k):
                b = A.vector(); b.x[:] = B[:, j]
                x = A.vector(); x.x[:] = X0[:, j]
                cj = cg.solvempi(b, x, maxits=400, residualatol=atol)
                assert cj == 0 and cols[j]["niterations"] == cg.c.niterations, (j, cols[j], cg.c.niterations)
                assert abs(cols[j]["rnrm2"] - cg.c.rnrm2) <= 1e-10 * cg.c.r0nrm2 + 1e-300, (j, cols[j], cg.c.rnrm2)
                scale = max(float(np.abs(x.x).max()), 1e-300)
                assert float(np.abs(X[:, j] - x.x).max()) <= 1e-10 * scale, j
                ref = oracle.cg(csr, B[:, j], x0=X0[:, j], maxits=400, atol=atol)
                assert ref["niterations"] == cols[j]["niterations"]
                assert float(np.abs(X[:, j] - ref["x"]).max()) <= 1e-10 * max(float(np.abs(ref["x"]).max()), 1e-300), j
        X0 = rng.standard_normal((n, 5))
        X = X0.copy()
        code, cols = cg.solve_multi(rng.standard_normal((n, 5)), X, maxits=0, residualrtol=1e-8)
        assert code == 39 and cg.c.niterations == 0 and np.array_equal(X.view(np.uint64), X0.view(np.uint64))
    finally:
        cg.free()
