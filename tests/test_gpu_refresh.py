"""acgsolvercuda_update_values on the H100: a solver built on values V1, run through every entry point (so that
graphs, Chebyshev's D^-1 and the fp32 row chunks are cached), then given V2 = 2 V1 + a diagonal shift on the same
pattern, against a solver built fresh on V2.

* Plan shapes: a 27-pt box entirely in slices (coded mirrored diagonals), a ragged 27-pt box (tile rows), a 7-pt
  box with odd sides, R-MAT (merge tiles), random_spd_60 under forced medium- and long-row plans, an arrow matrix
  (a long row), a diagonal matrix, and one part of a 4-way partition (spmv_mode / spmv_ghost on paths 0 and 1).
  Products bitwise equal to the fresh solver's (and to tests/exactref.py on integer data), the plan in info()
  equal, every solve with the same iteration count and x within 1e-12.  R-MAT is the exception: its solves do
  not repeat bit for bit even on one solver (the reductions' order varies from run to run, and on this
  ill-conditioned matrix two runs of one solver end up to 2 iterations apart), so there the counts may differ
  by 3 and x by 1e-8.
* Transitions on one solver: codes -> fp64 -> codes, codes with another table, the 256/257-pattern boundary,
  full storage -> packed triangle -> full storage, 1-based indices, and full storage that is not symmetric
  (the slice kernel reading both triangles, exact on integer data, and no mirrored diagonals afterwards).
* Refusals leave the products and solves as they were; device memory is the same after ten refreshes.
* C3 (27-pt 224^3): 100 iterations of fused pipelined CG and of classic CG after a refresh, x within 1e-12.
  R-MAT 2M: the product bitwise equal to a fresh solver's and 100 iterations of classic CG.  Its solves are
  not compared: four runs of 100 classic iterations on one fresh solver ended with ||b - A x|| between 653
  and 1952 (H100 SXM, 700 W), so no tolerance on x would tell a stale value from that spread; the product
  does (a solver left on the old values gives a different product).
"""
import os

import numpy as np
import pytest

from acg_b200 import matgen as mg
from conftest import load_golden
from entrypoints import assert_same_products, assert_same_solves, product_inputs, run_products, run_solves
from exactref import rows_exact
from test_gpu_small_shapes import _arrow, _diagonal

pytestmark = pytest.mark.gpu

INVALID_VALUE = 29
DEFAULTS = {"spmv_slices": 1, "spmv_merge": -1, "merge_items": 0, "spmv_nnz_cap": 0, "spmv_medium": 0,
            "spmv_symdiag": 1, "symdiag_codes": 1, "pcg_fused": 1}
NOSLICE = {"spmv_slices": 0}
PLAN_KEYS = ("spmv_lanes_per_row", "spmv_rows_cap", "spmv_nnz_cap", "spmv_stages", "spmv_ntiles", "spmv_nlong",
             "spmv_grid", "spmv_smem_bytes", "spmv_min_bytes", "spmv_nmedium", "spmv_slices", "spmv_slice_rows",
             "spmv_slice_ub", "spmv_slice_grid", "spmv_merge_tiles", "spmv_merge_rows", "spmv_merge_split",
             "spmv_slice_exc", "spmv_threads", "spmv_unroll", "spmv_slice_threads", "spmv_merge_threads",
             "spmv_merge_grid", "spmv_merge_stages", "spmv_slice_value_bytes", "spmv_slice_nnz",
             "spmv_symdiag_diagonals", "spmv_symdiag_bytes", "pcg_fused_min_bytes", "spmv_symdiag_codes",
             "spmv_symdiag_code_bytes")


@pytest.fixture
def options(ab):
    def set_(**kw):
        for k, v in dict(DEFAULTS, **kw).items():
            ab.set_option(k, v)
    set_()
    yield set_
    set_()


def _rand60():
    g = load_golden(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "random_spd_60.npz"))
    return int(g["n"]), g["rows"].astype(np.int32), g["cols"].astype(np.int32), g["vals"].astype(np.float64)


SHAPES = {
    "27pt-all-slices": (lambda: mg.stencil3d_27pt(16, 16, 16), {}),
    "27pt-ragged": (lambda: mg.stencil3d_27pt(21, 20, 19), {}),
    "7pt-odd": (lambda: mg.laplace3d_7pt(31, 17, 23), {}),
    "rmat-merge": (lambda: mg.rmat_spd(3000, 40000, seed=1), {}),
    "rand60-medium": (_rand60, dict(NOSLICE, spmv_nnz_cap=8, spmv_medium=3)),
    "rand60-long": (_rand60, dict(NOSLICE, spmv_nnz_cap=8)),
    "arrow-long": (lambda: _arrow(100), dict(NOSLICE, spmv_nnz_cap=8)),
    "diagonal": (lambda: _diagonal(200), {}),
}


def _v2(r, c, v, shift=1.0):
    return 2.0 * v + np.where(r == c, shift, 0.0)


def _matrix(ab, n, r, c, v, full=True, base=0):
    A = ab.SymCsrMatrix.init_real_double(n, r + base, c + base, v, idxbase=base)
    return A.dsymv_init(0.0) if full else A


def _plan(cg):
    inf = cg.info()
    return {k: inf[k] for k in PLAN_KEYS}


def _is_int(v):
    return bool(np.all(v == np.round(v)))


def _check_exact(A, cg, prods):
    """y and the dots of spmv_mode against the correctly rounded products of the full storage (whole matrix)."""
    p = product_inputs(cg, A)
    x, b = p["x"], p["b"]
    n = A.c.nownedrows
    rp, ci, fa = A.frowptr[:n + 1].copy(), A.fcolidx.copy() - A.c.rowidxbase, A.fa.copy()
    y, _, _ = rows_exact(rp, ci, fa, x)
    r, _, _ = rows_exact(rp, ci, fa, x, b)
    for m, (want, dot) in enumerate(((y, 0.0), (y, float(x[:n] @ y)), (r, float(r @ r)))):
        got, gdot = prods[f"spmv_mode{m}_path0"]
        assert np.array_equal(got, want), (m, np.flatnonzero(got != want)[:10])      # +0.0 and -0.0 alike
        assert gdot == dot, (m, gdot, dot)


def _against_fresh(ab, cg, A, tag, solves=True, exact=None, paths=(0,), rel=1e-12, its_slack=0):
    """cg (refreshed to A) against a solver built on A: products bitwise, the plan, and every solve."""
    got_p = run_products(ab, cg, A, paths=paths)
    got_s = run_solves(ab, cg, A) if solves else {}
    fresh = ab.SolverCuda(A)
    try:
        want_p = run_products(ab, fresh, A, paths=paths)
        want_s = run_solves(ab, fresh, A) if solves else {}
        assert _plan(cg) == _plan(fresh), tag
    finally:
        fresh.free()
    integer = _is_int(A.fa) if exact is None else exact
    assert_same_products(got_p, want_p, tag, exact_dots=integer)
    if integer and A.c.nghostrows == 0:
        _check_exact(A, cg, got_p)
    assert_same_solves(got_s, want_s, tag, rel=rel, its_slack=its_slack)
    return got_s


@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_plan_shapes(shape, ab, options):
    gen, opts = SHAPES[shape]
    options(**opts)
    n, r, c, v = gen()
    A1 = _matrix(ab, n, r, c, v)
    cg = ab.SolverCuda(A1)
    try:
        before = run_solves(ab, cg, A1)
        run_products(ab, cg, A1)
        inf = cg.info()
        if shape == "27pt-all-slices":
            assert inf["spmv_slice_rows"] == n and inf["spmv_symdiag_codes"] > 0 and inf["spmv_ntiles"] == 0
        if shape == "27pt-ragged":
            assert inf["spmv_ntiles"] > 0 and inf["spmv_symdiag_diagonals"] > 0
        if shape == "rmat-merge":
            assert inf["spmv_merge_tiles"] > 0
        if shape == "rand60-medium":
            assert inf["spmv_nmedium"] > 0
        if shape in ("rand60-long", "arrow-long"):
            assert inf["spmv_nlong"] > 0
        A2 = _matrix(ab, n, r, c, _v2(r, c, v))
        cg.update_values(A2)
        assert cg.A is A2
        after = _against_fresh(ab, cg, A2, shape, **({"rel": 1e-8, "its_slack": 3} if shape == "rmat-merge" else {}))
        # the new values change the solves: a stale value would have shown
        assert any(not np.array_equal(after[k][2], before[k][2]) for k in after if before[k][2] is not None)
    finally:
        cg.free()


def test_partition_part(ab, options):
    """One part of a 4-way block partition of a 27-pt box (ghost and border rows): the local product through
    both paths and all three modes."""
    n, r, c, v = mg.stencil3d_27pt(16, 16, 16)
    import acg_b200.dist as abdist
    rowparts = abdist.block_partition(16, 16, 16, 2, 2, 1)

    def part(vals):
        A = ab.SymCsrMatrix.init_real_double(n, r, c, vals)
        P = A.partition(4, rowparts)[1]
        return P.dsymv_init(0.0)

    P1 = part(v)
    assert P1.c.nghostrows > 0 and P1.c.nborderrows > 0
    cg = ab.SolverCuda(P1)
    try:
        run_products(ab, cg, P1, paths=(0, 1))
        P2 = part(_v2(r, c, v))
        cg.update_values(P2)
        _against_fresh(ab, cg, P2, "part", solves=False, paths=(0, 1))
    finally:
        cg.free()


def _stencil(kind):
    n, r, c, _ = mg.stencil3d_27pt(21, 20, 19)
    rng = np.random.default_rng(3)
    if kind == "stencil":
        v = np.where(r == c, 26.0, -1.0)
    elif kind == "ints":
        v = rng.integers(-3, 4, len(r)).astype(np.float64)
        v[r == c] = rng.integers(100, 120, int((r == c).sum()))      # diagonally dominant: SPD
    elif kind == "reals":
        v = rng.standard_normal(len(r))
        v[r == c] += 60.0
    return n, r, c, v


def test_codes_transitions(ab, options):
    """codes -> fp64 -> codes, and codes with another table, on one solver; each state against a fresh solver."""
    n, r, c, v = _stencil("stencil")
    cg = ab.SolverCuda(_matrix(ab, n, r, c, v))
    try:
        run_solves(ab, cg, cg.A)
        stencil_codes = cg.info()["spmv_symdiag_codes"]
        assert stencil_codes > 0
        seen = []
        for kind in ("reals", "stencil", "ints", "reals"):
            A = _matrix(ab, *_stencil(kind))
            cg.update_values(A)
            _against_fresh(ab, cg, A, kind)
            seen.append(cg.info()["spmv_symdiag_codes"])
            assert cg.info()["spmv_symdiag_diagonals"] == 14
        assert seen[0] == 0 and seen[1] == stencil_codes and seen[2] not in (0, stencil_codes) and seen[3] == 0
    finally:
        cg.free()


def test_table_size_boundary(ab, options):
    """Upper entries cycling through 255 integers (with the diagonal's 3 values and the +0.0 of the margins:
    too many) and through fewer, alternately on one solver: the codes come and go with the values."""
    n, r, c, _ = _stencil("stencil")

    def mat(k):
        v = 1.0 + (np.arange(len(r)) % k)
        return _matrix(ab, n, r, c, v)

    def distinct(A):
        rp, ci, fa = A.frowptr, A.fcolidx, A.fa
        rows = np.repeat(np.arange(len(rp) - 1), np.diff(rp))
        return len(set(fa[: rp[-1]][ci[: rp[-1]] >= rows].view(np.uint64).tolist()) | {0})

    A255, A256 = mat(255), mat(256)
    assert distinct(A255) == 256 and distinct(A256) == 257
    cg = ab.SolverCuda(A255)
    try:
        run_solves(ab, cg, A255)
        assert cg.info()["spmv_symdiag_codes"] == 256
        for A, coded in ((A256, False), (A255, True)):
            cg.update_values(A)
            _against_fresh(ab, cg, A, f"coded={coded}", solves=False)
            assert (cg.info()["spmv_symdiag_codes"] > 0) == coded
    finally:
        cg.free()


def test_sources_and_index_base(ab, options):
    """Full storage -> packed triangle -> full storage on one solver built from full storage; a solver built
    from the packed triangle refreshed from full storage; 1-based indices."""
    n, r, c, v = mg.laplace3d_7pt(31, 17, 23)
    v2 = _v2(r, c, v)
    cg = ab.SolverCuda(_matrix(ab, n, r, c, v))
    try:
        run_solves(ab, cg, cg.A)
        for full, vals in ((False, v2), (True, v), (False, v)):
            A = _matrix(ab, n, r, c, vals, full=full)
            cg.update_values(A)
            _against_fresh(ab, cg, _matrix(ab, n, r, c, vals), f"full={full}")
    finally:
        cg.free()
    cg = ab.SolverCuda(_matrix(ab, n, r, c, v, full=False))
    try:
        run_solves(ab, cg, cg.A)
        cg.update_values(_matrix(ab, n, r, c, v2))
        _against_fresh(ab, cg, _matrix(ab, n, r, c, v2), "packed-init")
    finally:
        cg.free()
    cg = ab.SolverCuda(_matrix(ab, n, r, c, v, base=1))
    try:
        run_solves(ab, cg, cg.A)
        A = _matrix(ab, n, r, c, v2, base=1)
        cg.update_values(A)
        _against_fresh(ab, cg, A, "1-based")
    finally:
        cg.free()


def test_not_symmetric_falls_back(ab, options):
    """Full storage whose lower entry differs from its mirror: the refreshed solver drops the mirrored
    diagonals as a fresh one does, its products are exact on integer data, and a later refresh with symmetric
    values keeps the slice kernel (the documented difference from a fresh solver)."""
    n, r, c, v = _stencil("ints")
    cg = ab.SolverCuda(_matrix(ab, n, r, c, v))
    try:
        run_solves(ab, cg, cg.A)
        run_products(ab, cg, cg.A)
        assert cg.info()["spmv_symdiag_diagonals"] == 14
        A = _matrix(ab, n, r, c, _v2(r, c, v))
        rows = np.repeat(np.arange(n), np.diff(A.frowptr))
        k = int(np.flatnonzero((A.fcolidx < rows) & (rows > n // 2))[0])
        A.fa[k] += 1.0
        cg.update_values(A)
        assert cg.info()["spmv_symdiag_diagonals"] == 0
        _against_fresh(ab, cg, A, "nonsym", solves=False, exact=True)
        S = _matrix(ab, n, r, c, v)
        cg.update_values(S)
        assert cg.info()["spmv_symdiag_diagonals"] == 0
        _check_exact(S, cg, run_products(ab, cg, S))
    finally:
        cg.free()


def test_refusals_leave_the_solver_alone(ab, options):
    n, r, c, v = mg.stencil3d_27pt(16, 16, 16)
    A = _matrix(ab, n, r, c, v)
    cg = ab.SolverCuda(A)
    try:
        want_p, want_s = run_products(ab, cg, A), run_solves(ab, cg, A)
        # a moved column with the same counts
        k = int(np.flatnonzero((c > r + 1) & (c < n - 1))[0])
        row = r[k]
        free_col = next(j for j in range(row + 1, n) if not np.any((r == row) & (c == j)))
        c2 = c.copy(); c2[k] = free_col
        o = np.lexsort((c2, r))
        bad = [_matrix(ab, n, r[o], c2[o], v[o]), _matrix(ab, n, r[o], c2[o], v[o], full=False)]
        keep = np.ones(len(r), bool); keep[k] = False
        bad.append(_matrix(ab, n, r[keep], c[keep], v[keep]))
        part = ab.SymCsrMatrix.init_real_double(n, r, c, v).partition(2, (np.arange(n) >= n // 2).astype(np.int32))[0]
        bad.append(part.dsymv_init(0.0))
        for i, B in enumerate(bad):
            with pytest.raises(ab.AcgError) as e:
                cg.update_values(B)
            assert e.value.code == INVALID_VALUE, i
            assert cg.A is A
        assert_same_products(run_products(ab, cg, A), want_p, "refused")
        assert_same_solves(run_solves(ab, cg, A), want_s, "refused", rel=1e-12)
    finally:
        cg.free()
    with pytest.raises(ab.AcgError) as e:
        cg.update_values(A)
    assert e.value.code == INVALID_VALUE


def test_memory_after_ten_refreshes(ab, options):
    import torch
    n, r, c, v = _stencil("stencil")
    A1, A2 = _matrix(ab, n, r, c, v), _matrix(ab, n, r, c, _v2(r, c, v))
    cg = ab.SolverCuda(A1)
    try:
        run_solves(ab, cg, A1)
        cg.update_values(A2)
        run_solves(ab, cg, A2)
        torch.cuda.mem_get_info()                   # the first call initialises torch's use of the context
        free0 = torch.cuda.mem_get_info()[0]
        for i in range(10):
            cg.update_values(A1 if i % 2 == 0 else A2)
        run_solves(ab, cg, A2)
        assert torch.cuda.mem_get_info()[0] == free0
    finally:
        cg.free()


def _scale_packed(A):
    """V2 = 2 V1 + 1 on the diagonal, in place on the packed triangle."""
    rp, ci, a = A.rowptr, A.colidx, A.a
    rows = np.repeat(np.arange(A.c.nprows), np.diff(rp))
    a *= 2.0
    a[ci - A.c.rowidxbase == rows] += 1.0


@pytest.mark.parametrize("kind", ["27pt-224", "rmat-2M"])
def test_full_size(kind, ab, options):
    """100 iterations of fused pipelined CG (C3 only) and of classic CG on a refreshed solver against a fresh
    one; the product at full size."""
    if kind == "rmat-2M":
        A = ab.SymCsrMatrix.rmat_spd(2_000_000, 20_000_000, seed=42)
    else:
        A = ab.SymCsrMatrix.stencil_part(27, 224, 224, 224, 1, 1, 1, 0)
    n = A.c.nownedrows
    b = A.vector(); b.x[:] = np.random.default_rng(1).standard_normal(n)
    names = ("solve_pipelined", "solvempi") if kind == "27pt-224" else ("solvempi",)
    cg = ab.SolverCuda(A)
    try:
        for name in names:
            getattr(cg, name)(b, A.vector(), maxits=100)
        _scale_packed(A)
        cg.update_values(A)
        fresh = ab.SolverCuda(A)
        try:
            for name in names:
                x1, x0 = A.vector(), A.vector()
                getattr(cg, name)(b, x1, maxits=100)
                its1, fused1 = cg.c.niterations, cg.info()["pcg_fused"]
                getattr(fresh, name)(b, x0, maxits=100)
                assert its1 == fresh.c.niterations == 100 and fused1 == fresh.info()["pcg_fused"], name
                if kind == "27pt-224" and name == "solve_pipelined":
                    assert fused1 == 1
                if kind == "27pt-224":
                    d = float(np.abs(x1.x[:n] - x0.x[:n]).max()) / float(np.abs(x0.x[:n]).max())
                    assert d <= 1e-12, (name, d)
            x = np.random.default_rng(3).integers(-4, 5, n).astype(np.float64)
            assert cg.spmv(x)[0].tobytes() == fresh.spmv(x)[0].tobytes()
        finally:
            fresh.free()
    finally:
        cg.free()
