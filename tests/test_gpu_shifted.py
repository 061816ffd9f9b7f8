"""Shifted systems on the H100: acgsolvercuda_solve_shifted (multi-shift CG, (A + sigma_j I) x_j = b in
one Krylov space) against acgsolvercuda_solvempi on a solver built from dsymv_init(sigma_j), shift by
shift: equal iteration counts, equal codes, x within 1e-10 relative, and the exact true residual of
every converged shift below 2 tol.  Matrices: a 27-point stencil (pattern slices), a 7-point stencil
with an odd number of rows (the update kernel's tail row), an R-MAT structure (merge tiles) and
random_spd_60 from tests/golden.  Shift counts 1, 2, 3, 4, 5, 8 run every block width K = 1, 2, 4, 8,
with padding columns, and the shifts leave the active mask at different iterations."""
import functools
import os

import numpy as np
import pytest

from exactref import rows_exact

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NOT_CONVERGED, INVALID_VALUE, NOT_SUPPORTED = 39, 29, 26
SHIFTS = [0.0, 1.0, 0.1, 0.01, 0.3, 0.03, 3.0, 1e-3]      # relative to the mean diagonal entry
NONZERO = SHIFTS[1:] + [3e-3]
COUNTS = (1, 2, 3, 4, 5, 8)


@functools.lru_cache(maxsize=None)
def _coo(key):
    from acg_b200 import matgen as mg
    if key == "27pt":
        return mg.stencil3d_27pt(30, 31, 29)
    if key == "7pt-odd":
        return mg.laplace3d_7pt(25)                           # 15625 rows
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


def _matrix(key, sigma=0.0):
    import acg_b200 as ab
    n, r, c, v = _coo(key)
    return ab.SymCsrMatrix.init_real_double(n, r, c, v).dsymv_init(sigma)


def _diag_mean(A):
    rp, ci, a = A.frowptr, A.fcolidx, A.fa
    rows = np.repeat(np.arange(len(rp) - 1), np.diff(rp))
    return float(a[rows == ci].mean())


def _threshold(atol, rtol, r0):
    return max(atol if atol > 0 else 0.0, rtol * r0)


def _compare(ab, key, b, shifts, code, X, cols, maxits, atol, rtol):
    """Every shift against solvempi on a solver of dsymv_init(sigma_j), and its exact true residual."""
    tol = _threshold(atol, rtol, float(np.linalg.norm(b)))
    want_code = 0
    for j, sigma in enumerate(shifts):
        Aj = _matrix(key, sigma)
        cgj = ab.SolverCuda(Aj)
        try:
            bv = Aj.vector(); bv.x[:] = b
            x = Aj.vector()
            cj = cgj.solvempi(bv, x, maxits=maxits, residualatol=atol, residualrtol=rtol)
            if cj == NOT_CONVERGED:
                want_code = NOT_CONVERGED
            assert cols[j]["niterations"] == cgj.c.niterations, (key, sigma, cols[j], cgj.c.niterations)
            assert cols[j]["converged"] == (cj == 0) or atol == rtol == 0, (key, sigma, cols[j], cj)
            scale = max(float(np.abs(x.x).max()), 1e-300)
            assert float(np.abs(X[:, j] - x.x).max()) <= 1e-10 * scale, (key, sigma)
            if cols[j]["converged"] and tol > 0:
                rt, _, _ = rows_exact(Aj.frowptr.copy(), Aj.fcolidx.copy(), Aj.fa.copy(), X[:, j], b)
                assert float(np.linalg.norm(rt)) < 2 * tol, (key, sigma, float(np.linalg.norm(rt)), tol)
        finally:
            cgj.free()
            Aj.free()
    assert code == want_code, (key, code, want_code)


@pytest.mark.gpu
@pytest.mark.parametrize("key", ["27pt", "7pt-odd", "rmat", "random_spd_60"])
def test_every_shift_against_solvempi(key, ab):
    """Shift counts 1..8 (block widths 1, 2, 4, 8; 3 and 5 with padding columns), sigma = 0 present under
    a relative tolerance with warm-up 0, absent under an absolute tolerance with warm-up 2."""
    A = _matrix(key)
    n = A.c.nownedrows
    d = _diag_mean(A)
    rng = np.random.default_rng(17)
    cg = ab.SolverCuda(A)
    try:
        for S in COUNTS:
            b = rng.standard_normal(n)
            for shifts, atol, rtol, warmup in (([d * s for s in SHIFTS[:S]], 0.0, 1e-10, 0),
                                               ([d * s for s in NONZERO[:S]], 1e-7 * float(np.linalg.norm(b)), 0.0, 2)):
                code, X, cols = cg.solve_shifted(b, shifts, maxits=600, residualatol=atol, residualrtol=rtol,
                                                 warmup=warmup)
                assert X.shape == (n, S) and len(cols) == S
                assert cg.c.niterations == max(c["niterations"] for c in cols)
                if S > 1 and key != "rmat":
                    assert len({c["niterations"] for c in cols}) > 1, cols     # shifts leave the mask apart
                _compare(ab, key, b, shifts, code, X, cols, 600, atol, rtol)
    finally:
        cg.free()


@pytest.mark.gpu
def test_maxits_zero_rhs_and_rejected_calls(ab):
    """maxits reached (NOT_CONVERGED, against solvempi too), maxits = 0 (X = 0), b = 0 under an absolute
    tolerance (0 iterations), and the rejected calls: 0 or 9 shifts, a negative, NaN or infinite shift,
    and a part of a partitioned matrix."""
    key = "7pt-odd"
    A = _matrix(key)
    n = A.c.nownedrows
    b = np.random.default_rng(3).standard_normal(n)
    cg = ab.SolverCuda(A)
    try:
        shifts = [0.0, 0.05, 0.5, 5.0, 0.005]
        code, X, cols = cg.solve_shifted(b, shifts, maxits=15, residualrtol=1e-10)
        assert code == NOT_CONVERGED and cg.c.niterations == 15
        _compare(ab, key, b, shifts, code, X, cols, 15, 0.0, 1e-10)
        code, X, cols = cg.solve_shifted(b, [0.0, 1.0], maxits=0, residualrtol=1e-8)
        assert code == NOT_CONVERGED and cg.c.niterations == 0 and not X.any()
        code, X, cols = cg.solve_shifted(np.zeros(n), [0.0, 1.0, 0.1], maxits=50, residualatol=1e-8)
        assert code == 0 and cg.c.niterations == 0 and not X.any()
        assert all(c["niterations"] == 0 and c["converged"] == 1 for c in cols)
        for shifts in ([], [0.0] * 9, [0.0, -1e-3], [0.1, float("nan")], [float("inf")]):
            with pytest.raises(ab.AcgError) as e:
                cg.solve_shifted(b, shifts, maxits=3)
            assert e.value.code == INVALID_VALUE, shifts
    finally:
        cg.free()
    parts = A.partition(2, (np.arange(n) >= n // 2).astype(np.int32))
    P = parts[0].dsymv_init(0.0)
    cgp = ab.SolverCuda(P)
    try:
        with pytest.raises(ab.AcgError) as e:
            cgp.solve_shifted(np.ones(P.c.nownedrows), [0.0, 0.1], maxits=3)
        assert e.value.code == NOT_SUPPORTED
    finally:
        cgp.free()


@pytest.mark.gpu
def test_graph_replay_three_kernels_per_iteration(ab):
    """With tolerances off the loop runs exactly maxits iterations as graph replays: per iteration the
    single-vector product, cg_update_r_kernel and cg_shift_update_kernel -- the same count as a classic
    solve, three kernels when the product is one slice kernel.  Solves of other kinds and widths in
    between do not change what a replay issues or computes."""
    A = _matrix("27pt")
    n = A.c.nownedrows
    b = np.random.default_rng(8).standard_normal(n)
    cg = ab.SolverCuda(A)
    try:
        inf = cg.info()
        launches = {}
        for m in (10, 30):
            code, X, cols = cg.solve_shifted(b, [0.0, 0.1, 1.0], maxits=m)
            assert code == 0 and cg.c.niterations == m and all(c["niterations"] == m for c in cols)
            launches[("shifted", m)] = cg.info()["last_launches"]
            bv = A.vector(); bv.x[:] = b
            x = A.vector()
            assert cg.solvempi(bv, x, maxits=m) == 0
            launches[("single", m)] = cg.info()["last_launches"]
        per = (launches[("shifted", 30)] - launches[("shifted", 10)]) / 20
        assert per == (launches[("single", 30)] - launches[("single", 10)]) / 20
        if inf["spmv_slices"] > 0 and inf["spmv_ntiles"] == 0 and inf["spmv_merge_tiles"] == 0 \
                and inf["spmv_nlong"] == 0 and inf["spmv_nmedium"] == 0:
            assert per == 3
        ref = cg.solve_shifted(b, [0.0, 0.1, 1.0, 0.01], maxits=40, residualrtol=1e-9)
        cg.solve_multi(np.ascontiguousarray(np.stack([b] * 8, axis=1)), np.zeros((n, 8)), maxits=40, residualrtol=1e-9)
        cg.solve_shifted(b, [0.3], maxits=40, residualrtol=1e-9)
        again = cg.solve_shifted(b, [0.0, 0.1, 1.0, 0.01], maxits=40, residualrtol=1e-9)
        assert ref[0] == again[0] and [c["niterations"] for c in ref[2]] == [c["niterations"] for c in again[2]]
        assert float(np.abs(ref[1] - again[1]).max()) <= 1e-12 * float(np.abs(ref[1]).max())
    finally:
        cg.free()
