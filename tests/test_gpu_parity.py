"""Parity of the CUDA path with the oracle, through the C-ABI (H100, -m gpu)."""
import os

import numpy as np
import pytest

from acg_b200 import matgen as mg
from conftest import GOLDEN, load_golden

pytestmark = pytest.mark.gpu

# FP64 tolerances.  The device sums each row and each dot product in a different
# order than the CPU (and dot products through atomics, so not even run-to-run
# bitwise): entries of A*x agree to a few ulp of sum|a_ij x_j|; CG iterates agree
# with the oracle to 1e-10 relative in the residual norm (north-star) as long as
# the iteration count is O(100) and the matrix is well conditioned.
SPMV_RTOL = 1e-13
RES_RTOL = 1e-10


def _solver(ab, n, r, c, v):
    A = ab.SymCsrMatrix.init_real_double(n, r, c, v).dsymv_init(0.0)
    return A, ab.SolverCuda(A)


CASES = [
    ("27pt-12", lambda: mg.stencil3d_27pt(12)),
    ("27pt-aniso", lambda: mg.stencil3d_27pt(9, 40, 17)),
    ("7pt-31", lambda: mg.laplace3d_7pt(31, 17, 23)),
    ("1d5pt", lambda: mg.poisson1d_5pt(20000)),
    ("rand-dense-rows", lambda: mg.random_spd(400, 0.5, 2)),      # ~200 nnz/row: 16-lane groups
    ("rmat-longrows", lambda: mg.rmat_spd(30000, 600000, seed=8)),  # power-law: long-row path
    ("n1", lambda: mg.poisson1d_3pt(1)),
    ("n3", lambda: mg.poisson1d_3pt(3)),
]


@pytest.mark.parametrize("name,gen", CASES, ids=[c[0] for c in CASES])
def test_spmv_matches_oracle(name, gen, ab, oracle):
    n, r, c, v = gen()
    A, cg = _solver(ab, n, r, c, v)
    csr = (A.frowptr.copy(), A.fcolidx.copy(), A.fa.copy())
    x = np.random.default_rng(1).standard_normal(n)
    y, _ = cg.spmv(x)
    want = oracle.dsymv(csr, 1.0, x, 0.0, np.zeros(n))
    scale = oracle.dsymv((csr[0], csr[1], np.abs(csr[2])), 1.0, np.abs(x), 0.0, np.zeros(n))
    assert np.all(np.abs(y - want) <= SPMV_RTOL * scale + 1e-300)
    if name == "rmat-longrows":
        assert cg.info()["spmv_merge_tiles"] > 0           # power-law rows: merge-path tiles by default
    cg.free()


def test_spmv_ragged_rows(ab, oracle):
    """Rows with no entries at all, single-entry rows, rows longer than a tile
    (long-row path) and a dense last row next to each other: y = A x entry by entry."""
    n = 5000
    rng = np.random.default_rng(12)
    rows, cols = [], []
    for i in range(0, n, 3):                       # every third row has a diagonal entry; the others are empty so far
        rows.append(i); cols.append(i)
    hub = 7                                        # one row touching 60 % of the columns
    for j in rng.choice(np.arange(hub + 1, n), size=3000, replace=False):
        rows.append(hub); cols.append(int(j))
    for j in range(0, n - 1, 2):                   # dense-ish last column = last row of the full matrix
        rows.append(j); cols.append(n - 1)
    r = np.array(rows, np.int32); c = np.array(cols, np.int32)
    key = np.unique(r.astype(np.int64) * n + c)
    r, c = (key // n).astype(np.int32), (key % n).astype(np.int32)
    v = rng.standard_normal(len(r))
    A, cg = _solver(ab, n, r, c, v)
    lens = np.diff(A.frowptr)
    assert (lens == 0).sum() > 100 and lens.max() > 2000
    csr = (A.frowptr.copy(), A.fcolidx.copy(), A.fa.copy())
    x = rng.standard_normal(n)
    y, _ = cg.spmv(x)
    want = oracle.dsymv(csr, 1.0, x, 0.0, np.zeros(n))
    scale = oracle.dsymv((csr[0], csr[1], np.abs(csr[2])), 1.0, np.abs(x), 0.0, np.zeros(n))
    assert np.all(np.abs(y - want) <= SPMV_RTOL * scale + 1e-300)
    assert np.all(y[lens == 0] == 0.0)
    assert cg.info()["spmv_merge_tiles"] > 0 or cg.info()["spmv_nlong"] >= 1
    cg.free()


@pytest.mark.parametrize("method", ["solvempi", "solve_pipelined"])
@pytest.mark.parametrize("name,gen", CASES[:3] + [CASES[4]] + CASES[6:], ids=[c[0] for c in CASES[:3] + [CASES[4]] + CASES[6:]])
def test_cg_matches_oracle(name, gen, method, ab, oracle):
    n, r, c, v = gen()
    A, cg = _solver(ab, n, r, c, v)
    csr = (A.frowptr.copy(), A.fcolidx.copy(), A.fa.copy())
    b = A.vector()
    b.x[:] = np.random.default_rng(5).standard_normal(n)
    want = (oracle.cg if method == "solvempi" else oracle.cg_pipelined)(csr, b.x, maxits=300, rtol=1e-9, history=True)
    x = A.vector()
    code = getattr(cg, method)(b, x, maxits=300, residualrtol=1e-9, warmup=1)
    assert code == want["status"] == 0
    assert cg.c.niterations == want["niterations"]
    assert cg.c.bnrm2 == pytest.approx(want["bnrm2"], rel=1e-14)
    assert cg.c.r0nrm2 == pytest.approx(want["r0nrm2"], rel=1e-14)
    assert cg.c.rnrm2 / cg.c.r0nrm2 == pytest.approx(want["rnrm2"] / want["r0nrm2"], rel=1e-6, abs=RES_RTOL)
    assert np.abs(x.x - want["x"]).max() <= 1e-9 * np.abs(want["x"]).max()
    cg.free()


@pytest.mark.parametrize("method", ["solvempi", "solve_pipelined"])
@pytest.mark.parametrize("name,gen", [CASES[3], CASES[5]], ids=[CASES[3][0], CASES[5][0]])
def test_cg_ill_conditioned_fixed_iterations(name, gen, method, ab, oracle):
    """1-D 5-point (kappa ~ n^2, BASELINE config 1) and the power-law matrix do
    not converge in O(100) iterations: compare after a fixed number of
    iterations with tolerances off, as SURVEY.md 8(d) prescribes."""
    n, r, c, v = gen()
    A, cg = _solver(ab, n, r, c, v)
    csr = (A.frowptr.copy(), A.fcolidx.copy(), A.fa.copy())
    b = A.vector()
    b.x[:] = 1.0 if name == "1d5pt" else np.random.default_rng(5).standard_normal(n)
    # the power-law Laplacian (kappa ~ 2*maxdeg ~ 1e4) has near-breakdown spikes
    # in ||r_k|| from k~20 on, where any two summation orders part ways (numpy
    # vs the oracle differ by 1e-2 there); compare before that
    its = 40 if name == "1d5pt" else 10
    want = (oracle.cg if method == "solvempi" else oracle.cg_pipelined)(csr, b.x, maxits=its)
    x = A.vector()
    assert getattr(cg, method)(b, x, maxits=its) == want["status"] == 0
    assert cg.c.niterations == want["niterations"] == its
    assert cg.c.rnrm2 / cg.c.r0nrm2 == pytest.approx(want["rnrm2"] / want["r0nrm2"], rel=1e-8)
    assert np.abs(x.x - want["x"]).max() <= 1e-9 * np.abs(want["x"]).max()
    # and a run that cannot meet its tolerance reports ACG_ERR_NOT_CONVERGED like the oracle
    w2 = (oracle.cg if method == "solvempi" else oracle.cg_pipelined)(csr, b.x, maxits=10, rtol=1e-14)
    assert getattr(cg, method)(b, x, maxits=10, residualrtol=1e-14) == w2["status"] == 39
    cg.free()


@pytest.mark.parametrize("method", ["solvempi", "solve_pipelined"])
def test_residual_history_fixed_iterations(method, ab, oracle):
    """Same residual after k iterations for every k (tolerances off)."""
    n, r, c, v = mg.stencil3d_27pt(20)
    A, cg = _solver(ab, n, r, c, v)
    csr = (A.frowptr.copy(), A.fcolidx.copy(), A.fa.copy())
    b = A.vector(); b.x[:] = 1.0
    orc = oracle.cg if method == "solvempi" else oracle.cg_pipelined
    hist = orc(csr, b.x, maxits=40, history=True)["rnrm2hist"]
    for k in (1, 2, 3, 8, 25, 40):
        x = A.vector()
        assert getattr(cg, method)(b, x, maxits=k) == 0
        assert cg.c.niterations == k
        # classic: ||r_k||; pipelined reports the last tested iterate, ||r_{k-1}||
        want = hist[k] if method == "solvempi" else hist[k - 1]
        # 1e-9 relative while the residual is large; once the solve is down at rounding level (b = 1 on
        # this box converges to 1e-12 within 40 iterations) only the north-star bound relative to ||r0|| holds
        assert cg.c.rnrm2 == pytest.approx(want, rel=1e-9, abs=RES_RTOL * hist[0])
    cg.free()


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-4] for p in GOLDEN])
def test_golden_vectors(path, ab):
    """Fixtures produced by the reference's CPU solver alone (tools/make_golden.py)."""
    g = load_golden(path)
    n = int(g["n"])
    A, cg = _solver(ab, n, g["rows"], g["cols"], g["vals"])
    assert np.array_equal(A.frowptr, g["frowptr"]) and np.array_equal(A.fcolidx, g["fcolidx"]) and np.array_equal(A.fa, g["fa"])
    y, _ = cg.spmv(g["xs"])
    assert np.allclose(y, g["y"], rtol=1e-12, atol=1e-12 * np.abs(g["y"]).max())
    b = A.vector(); b.x[:] = g["b"]
    x = A.vector()
    code = cg.solvempi(b, x, maxits=int(g["maxits"]), residualrtol=float(g["rtol"]))
    assert code == int(g["status"])
    assert cg.c.niterations == int(g["niterations"])
    assert cg.c.bnrm2 == pytest.approx(float(g["bnrm2"]), rel=1e-14)
    assert cg.c.r0nrm2 == pytest.approx(float(g["r0nrm2"]), rel=1e-13)
    assert cg.c.rnrm2 == pytest.approx(float(g["rnrm2"]), rel=1e-6, abs=RES_RTOL * float(g["r0nrm2"]))
    assert np.abs(x.x - g["x"]).max() <= 1e-9 * np.abs(g["x"]).max()
    cg.free()


def test_interface_behaviour(ab):
    """Return codes of acg/cgcuda.c: :424 (diff tolerances), :1099-1107, and the
    NVSHMEM-only entry points (acg/cg-kernels-cuda.cu:1012)."""
    n, r, c, v = mg.stencil3d_27pt(8)
    A, cg = _solver(ab, n, r, c, v)
    b = A.vector(); b.x[:] = 1.0
    x = A.vector()
    assert cg.solvempi(b, x, maxits=0) == 0 and cg.c.niterations == 0 and np.all(x.x == 0)
    assert cg.solvempi(b, x, maxits=2, residualrtol=1e-30) == 39          # ACG_ERR_NOT_CONVERGED
    assert cg.c.niterations == 2
    with pytest.raises(ab.AcgError) as e:
        cg.solvempi(b, x, maxits=5, diffatol=1e-3)
    assert e.value.code == 26                                             # ACG_ERR_NOT_SUPPORTED
    cg.comm.c.type = 4                                                    # acgcomm_nvshmem
    try:
        for call in (cg.solve_device, cg.solve_device_pipelined):
            with pytest.raises(ab.AcgError) as e:
                call(b, x)
            assert e.value.code == 16                                         # ACG_ERR_NVSHMEM_NOT_SUPPORTED
    finally:
        cg.comm.c.type = 0
    # already-converged initial guess: zero iterations, success
    xs = A.vector(); xs.x[:] = np.random.default_rng(0).standard_normal(n)
    bb = A.vector(); bb.x[:], _ = cg.spmv(xs.x)
    assert cg.solvempi(bb, xs, maxits=10, residualatol=1e-6) == 0 and cg.c.niterations == 0
    assert cg.c.nsolves == 3 and cg.c.ntotaliterations == 2   # the rejected call returns before counting (acg/cgcuda.c:424)
    rep = cg.report()
    assert "total solver time:" in rep and "iterations: 0" in rep and "gemv:" in rep
    cg.free()


@pytest.mark.parametrize("entry,twin", [("solve_device", "solvempi"), ("solve_device_pipelined", "solve_pipelined"),
                                        ("solve", "solvempi")])
def test_device_and_plain_entry_points(entry, twin, ab, oracle):
    """acgsolvercuda_solve_device{,_pipelined} (acg/cg-kernels-cuda.cu:998,:1713) with a
    non-NVSHMEM communicator and acgsolvercuda_solve (acg/cgcuda.h:165) run the
    device-controlled loops: same iteration count, norms and solution as the oracle."""
    n, r, c, v = mg.stencil3d_27pt(16)
    A, cg = _solver(ab, n, r, c, v)
    csr = (A.frowptr.copy(), A.fcolidx.copy(), A.fa.copy())
    b = A.vector(); b.x[:] = np.random.default_rng(11).standard_normal(n)
    want = (oracle.cg_pipelined if "pipelined" in twin else oracle.cg)(csr, b.x, maxits=200, rtol=1e-9)
    x = A.vector()
    assert getattr(cg, entry)(b, x, maxits=200, residualrtol=1e-9) == 0
    assert cg.c.niterations == want["niterations"] and cg.c.nsolves == 1
    assert cg.c.rnrm2 / cg.c.r0nrm2 == pytest.approx(want["rnrm2"] / want["r0nrm2"], rel=1e-6, abs=RES_RTOL)
    assert np.abs(x.x - want["x"]).max() <= 1e-9 * np.abs(want["x"]).max()
    cg.free()


def test_eps_shift_and_reuse(ab, oracle):
    """--epsilon (acg/symcsrmatrix.c:796): diagonal shift; one solver, many solves."""
    n, r, c, v = mg.laplace3d_7pt(12)
    A = ab.SymCsrMatrix.init_real_double(n, r, c, v).dsymv_init(0.5)
    csr = oracle.full_csr(n, r, c, v, eps=0.5)
    cg = ab.SolverCuda(A)
    for seed in range(3):
        b = A.vector(); b.x[:] = np.random.default_rng(seed).standard_normal(n)
        x = A.vector()
        want = oracle.cg(csr, b.x, maxits=100, rtol=1e-10)
        assert cg.solvempi(b, x, maxits=100, residualrtol=1e-10) == 0
        assert cg.c.niterations == want["niterations"]
        assert np.abs(x.x - want["x"]).max() <= 1e-10 * np.abs(want["x"]).max()
    cg.free()


@pytest.mark.parametrize("kind", ["27pt-224", "7pt-256"])
def test_full_size_properties(kind, ab):
    """BASELINE.json's full sizes, through size-independent properties: the
    manufactured solution A*1 (row sums are known in closed form for the
    stencils), linearity and symmetry of the product, and a CG residual check
    recomputed from x."""
    # the threaded generator (one part = the whole box): the same arrays as the numpy generator +
    # init_real_double (tests/test_host_structs.py), in a tenth of the time
    N = 224 if kind == "27pt-224" else 256
    n = N ** 3
    A = ab.SymCsrMatrix.stencil_part(27 if kind == "27pt-224" else 7, N, N, N, 1, 1, 1, 0).dsymv_init(0.0)
    cg = ab.SolverCuda(A)
    nnz = A.c.fnpnzs
    assert nnz == ((3 * N - 2) ** 3 if kind == "27pt-224" else 7 * N ** 3 - 6 * N ** 2)
    ones = np.ones(n)
    y1, _ = cg.spmv(ones)
    # row sum = diag - (#neighbours): 26-(deg-1) resp. 6-(deg-1); deg from the row pointer
    deg = np.diff(A.frowptr)
    diag = 26.0 if kind == "27pt-224" else 6.0
    assert np.array_equal(y1, diag - (deg - 1))
    rng = np.random.default_rng(7)
    u, w = rng.standard_normal(n), rng.standard_normal(n)
    yu, _ = cg.spmv(u); yw, _ = cg.spmv(w); yuw, _ = cg.spmv(u + 2.0 * w)
    assert np.abs(yuw - (yu + 2.0 * yw)).max() <= 1e-12 * np.abs(yuw).max()
    assert abs(w @ yu - u @ yw) <= 1e-11 * abs(w @ yu)
    b = A.vector(); b.x[:] = y1            # exact solution: all ones
    for method in ("solvempi", "solve_pipelined"):
        x = A.vector()
        its = 50
        assert getattr(cg, method)(b, x, maxits=its) == 0 and cg.c.niterations == its
        ax, _ = cg.spmv(x.x)
        true_res = np.linalg.norm(b.x - ax)
        # the recurrence residual the solver reports is the true residual of the x
        # it returns (classic: r_k; pipelined reports r_{k-1}, one step behind)
        assert true_res < 0.2 * cg.c.r0nrm2
        if method == "solvempi":
            assert true_res == pytest.approx(cg.c.rnrm2, rel=1e-8)
        else:
            assert true_res <= cg.c.rnrm2 * 1.5
        # CG minimises the A-norm of the error monotonically: closer to the all-ones solution
        assert np.linalg.norm(x.x - 1.0) < np.linalg.norm(ones)
    cg.free()


@pytest.mark.parametrize("n,edges", [(2_000_000, 20_000_000)] +
                         ([(20_000_000, 200_000_000)] if os.environ.get("ACGB200_TEST_LARGE") == "1" else []),
                         ids=lambda v: str(v))
def test_power_law_properties(n, edges, ab):
    """BASELINE config 5 (R-MAT power-law SPD; the full 20 M / 200 M size with
    ACGB200_TEST_LARGE=1) through size-independent properties: every row of
    A = D + I - Adj sums to 1, so A*1 = 1 exactly in floating point (sums of small
    integers); symmetry of the product; the merge-path tiles are in use; and CG on
    b = A*x_true approaches x_true with a true residual equal to the reported one."""
    A = ab.SymCsrMatrix.rmat_spd(n, edges, seed=42).dsymv_init(0.0)
    cg = ab.SolverCuda(A)
    assert cg.info()["spmv_merge_tiles"] > 0 and cg.info()["spmv_merge_rows"] == n
    y1, _ = cg.spmv(np.ones(n))
    assert np.array_equal(y1, np.ones(n))
    rng = np.random.default_rng(3)
    u, w = rng.standard_normal(n), rng.standard_normal(n)
    yu, _ = cg.spmv(u); yw, _ = cg.spmv(w)
    assert abs(w @ yu - u @ yw) <= 1e-10 * abs(w @ yu)
    xt = 1.0 + 0.5 * np.sin(0.37 * np.arange(n))
    b = A.vector(); b.x[:], _ = cg.spmv(xt)
    x = A.vector()
    assert cg.solvempi(b, x, maxits=150) == 0 and cg.c.niterations == 150
    ax, _ = cg.spmv(x.x)
    assert np.linalg.norm(b.x - ax) == pytest.approx(cg.c.rnrm2, rel=1e-6, abs=1e-12 * cg.c.r0nrm2)
    # the hubs make the matrix ill conditioned (degrees up to ~1e5): convergence is slow but monotone
    # in the error (CPU oracle at the 2 M size: residual 3e-2, error 4e-2 after 150 iterations)
    assert cg.c.rnrm2 < 0.5 * cg.c.r0nrm2
    assert np.linalg.norm(x.x - xt) < 0.5 * np.linalg.norm(xt)
    cg.free()


SLICE_CASES = [CASES[0], CASES[1], CASES[2], CASES[3]]


@pytest.mark.parametrize("ub,threads", [(0, 0), (9, 128), (7, 256), (8, 128), (5, 128), (9, 256)])
@pytest.mark.parametrize("name,gen", SLICE_CASES, ids=[c[0] for c in SLICE_CASES])
def test_pattern_slices_match_oracle(name, gen, ub, threads, ab, oracle):
    """spmv_slices_kernel (slices.c): rows that repeat a pattern are multiplied from slice-major
    values without indices; every batch width / CTA size gives the oracle's product (full batches and
    the partial last one), the fused dots of both CG loops included, and agrees with the tile kernel
    (option off) to rounding."""
    n, r, c, v = gen()
    ab.set_option("slice_ub", ub); ab.set_option("slice_threads", threads)
    try:
        A, cg = _solver(ab, n, r, c, v)
        ab.set_option("spmv_slices", 0)
        cg_tiles = ab.SolverCuda(A)
    finally:
        ab.set_option("spmv_slices", 1); ab.set_option("slice_ub", 0); ab.set_option("slice_threads", 0)
    inf = cg.info()
    assert inf["spmv_slices"] > 0 and inf["spmv_slice_rows"] == 32 * inf["spmv_slices"]
    assert cg_tiles.info()["spmv_slices"] == 0
    csr = (A.frowptr.copy(), A.fcolidx.copy(), A.fa.copy())
    x = np.random.default_rng(1).standard_normal(n)
    y, _ = cg.spmv(x)
    y2, _ = cg_tiles.spmv(x)
    want = oracle.dsymv(csr, 1.0, x, 0.0, np.zeros(n))
    scale = oracle.dsymv((csr[0], csr[1], np.abs(csr[2])), 1.0, np.abs(x), 0.0, np.zeros(n))
    assert np.all(np.abs(y - want) <= SPMV_RTOL * scale + 1e-300)
    assert np.all(np.abs(y - y2) <= SPMV_RTOL * scale + 1e-300)
    if name != "1d5pt":
        b = A.vector(); b.x[:] = 1.0
        for method, oname in (("solvempi", "cg"), ("solve_pipelined", "cg_pipelined")):
            xs = A.vector()
            ref = getattr(oracle, oname)(csr, b.x, maxits=300, rtol=1e-9)
            assert getattr(cg, method)(b, xs, maxits=300, residualrtol=1e-9) == 0
            assert cg.c.niterations == ref["niterations"]
            assert np.abs(xs.x - ref["x"]).max() <= 1e-9 * np.abs(ref["x"]).max()
            assert abs(cg.c.rnrm2 - ref["rnrm2"]) <= RES_RTOL * ref["r0nrm2"]
    cg.free(); cg_tiles.free()


@pytest.mark.parametrize("method", ["solvempi", "solve_pipelined"])
def test_pdl_matches_oracle(method, ab, oracle):
    """Option pdl=1 (griddepcontrol along the iteration chain, also inside the captured
    graphs): same iterates as the default launches."""
    n, r, c, v = mg.stencil3d_27pt(24)
    A, cg = _solver(ab, n, r, c, v)
    csr = (A.frowptr.copy(), A.fcolidx.copy(), A.fa.copy())
    b = A.vector(); b.x[:] = np.random.default_rng(5).standard_normal(n)
    want = (oracle.cg if method == "solvempi" else oracle.cg_pipelined)(csr, b.x, maxits=300, rtol=1e-9)
    ab.set_option("pdl", 1)
    try:
        x = A.vector()
        assert getattr(cg, method)(b, x, maxits=300, residualrtol=1e-9) == 0
    finally:
        ab.set_option("pdl", 0)
    assert cg.c.niterations == want["niterations"]
    assert np.abs(x.x - want["x"]).max() <= 1e-9 * np.abs(want["x"]).max()
    cg.free()


MERGE_CASES = [CASES[5], CASES[4], CASES[3], ("7pt-31", CASES[2][1]), ("hub-100k", lambda: mg.rmat_spd(120000, 1500000, seed=11))]


@pytest.mark.parametrize("items,threads", [(1024, 128), (256, 128), (4096, 256), (64, 128)])
@pytest.mark.parametrize("name,gen", MERGE_CASES, ids=[c[0] for c in MERGE_CASES])
def test_merge_path_tiles_match_oracle(name, gen, items, threads, ab, oracle):
    """spmv_merge_kernel + spmv_merge_fix_kernel (mergeplan.c) forced on: power-law rows with hubs that span
    many tiles, dense rows, banded and stencil rows (every row complete inside a tile), tiny tiles in which
    most rows are cut -- the product equals the oracle's and the row-aligned tiles' to rounding, the fused
    dots drive both CG loops to the oracle's iterates."""
    n, r, c, v = gen()
    for k, val in (("spmv_merge", 1), ("spmv_slices", 0), ("merge_items", items), ("merge_threads", threads)):
        ab.set_option(k, val)
    try:
        A, cg = _solver(ab, n, r, c, v)
        ab.set_option("spmv_merge", 0)
        cg_rows = ab.SolverCuda(A)
    finally:
        for k, val in (("spmv_merge", -1), ("spmv_slices", 1), ("merge_items", 0), ("merge_threads", 0)):
            ab.set_option(k, val)
    inf = cg.info()
    if n < 1024:
        assert inf["spmv_merge_tiles"] == 0           # too small to bother
    else:
        assert inf["spmv_merge_tiles"] > 0 and inf["spmv_merge_rows"] == n and inf["spmv_ntiles"] == 0 and inf["spmv_nlong"] == 0
        if name in ("rmat-longrows", "hub-100k") or items <= 256:
            assert inf["spmv_merge_split"] > 0
    csr = (A.frowptr.copy(), A.fcolidx.copy(), A.fa.copy())
    x = np.random.default_rng(1).standard_normal(n)
    y, _ = cg.spmv(x)
    y2, _ = cg_rows.spmv(x)
    want = oracle.dsymv(csr, 1.0, x, 0.0, np.zeros(n))
    scale = oracle.dsymv((csr[0], csr[1], np.abs(csr[2])), 1.0, np.abs(x), 0.0, np.zeros(n))
    assert np.all(np.abs(y - want) <= SPMV_RTOL * scale + 1e-300)
    assert np.all(np.abs(y - y2) <= SPMV_RTOL * scale + 1e-300)
    b = A.vector(); b.x[:] = np.random.default_rng(2).standard_normal(n)
    # hubs of degree 1e4-1e5 make the power-law matrices ill conditioned: rounding differences between summation
    # orders are amplified from the first iterations on (the hub entry of x moves first)
    its, xtol = (10, 1e-9) if name not in ("rmat-longrows", "hub-100k") else (10, 1e-7)
    for method, orc in (("solvempi", oracle.cg), ("solve_pipelined", oracle.cg_pipelined)):
        ref = orc(csr, b.x, maxits=its, rtol=0.0)
        xs = A.vector()
        assert getattr(cg, method)(b, xs, maxits=its) == 0 and cg.c.niterations == its
        assert np.abs(xs.x - ref["x"]).max() <= xtol * np.abs(ref["x"]).max()
        assert abs(cg.c.rnrm2 - ref["rnrm2"]) <= xtol * ref["r0nrm2"]
    cg.free(); cg_rows.free()


def test_medium_row_kernel_matches_oracle(ab, oracle):
    """Option spmv_medium (spmv_medium_kernel): same product and same CG iterates on a power-law matrix."""
    n, r, c, v = mg.rmat_spd(30000, 600000, seed=8)
    ab.set_option("spmv_medium", 96); ab.set_option("spmv_merge", 0)      # row-aligned tiles + row lists
    try:
        A, cg = _solver(ab, n, r, c, v)
    finally:
        ab.set_option("spmv_medium", 0); ab.set_option("spmv_merge", -1)
    assert cg.info()["spmv_nmedium"] > 0 and cg.info()["spmv_nlong"] > 0 and cg.info()["spmv_merge_tiles"] == 0
    csr = (A.frowptr.copy(), A.fcolidx.copy(), A.fa.copy())
    x = np.random.default_rng(1).standard_normal(n)
    y, _ = cg.spmv(x)
    want = oracle.dsymv(csr, 1.0, x, 0.0, np.zeros(n))
    scale = oracle.dsymv((csr[0], csr[1], np.abs(csr[2])), 1.0, np.abs(x), 0.0, np.zeros(n))
    assert np.all(np.abs(y - want) <= SPMV_RTOL * scale + 1e-300)
    b = A.vector(); b.x[:] = np.random.default_rng(2).standard_normal(n)
    for method, orc in (("solvempi", oracle.cg), ("solve_pipelined", oracle.cg_pipelined)):
        ref = orc(csr, b.x, maxits=10, rtol=0.0)
        xs = A.vector()
        assert getattr(cg, method)(b, xs, maxits=10) == 0
        assert np.abs(xs.x - ref["x"]).max() <= 1e-9 * np.abs(ref["x"]).max()
    cg.free()


def test_public_blas1_building_blocks(ab):
    """acg/cg-kernels-cuda.h:45-97 on the device (torch only provides the device arrays)."""
    import ctypes as C
    import torch
    L = ab.lib()
    dev = lambda a: torch.tensor(np.atleast_1d(a), dtype=torch.float64, device="cuda")       # noqa: E731
    rng = np.random.default_rng(2)
    n = 100003
    rr, pap, rrp = dev(3.5), dev(1.25), dev(7.0)
    al, mal, be = dev(0.0), dev(0.0), dev(0.0)
    assert L.acgsolvercuda_alpha(al.data_ptr(), mal.data_ptr(), rr.data_ptr(), pap.data_ptr()) == 0
    assert L.acgsolvercuda_beta(be.data_ptr(), rr.data_ptr(), rrp.data_ptr()) == 0
    torch.cuda.synchronize()
    assert (al.item(), mal.item(), be.item()) == (2.8, -2.8, 0.5)
    x, y = rng.standard_normal(n), rng.standard_normal(n)
    dx = dev(x)
    for fn, want in ((L.acgsolvercuda_daxpy_alpha, y + 2.8 * x), (L.acgsolvercuda_daxpy_minus_alpha, y - 2.8 * x)):
        dy = dev(y)
        assert fn(n, rr.data_ptr(), pap.data_ptr(), dx.data_ptr(), dy.data_ptr()) == 0
        torch.cuda.synchronize()
        assert np.allclose(dy.cpu().numpy(), want, rtol=1e-15, atol=1e-15)
    dy = dev(y)
    assert L.acgsolvercuda_daypx_beta(n, rr.data_ptr(), rrp.data_ptr(), dy.data_ptr(), dx.data_ptr()) == 0
    torch.cuda.synchronize()
    assert np.allclose(dy.cpu().numpy(), 0.5 * y + x, rtol=1e-15, atol=1e-15)
    g, gp, d, ap = dev(2.0), dev(4.0), dev(3.0), dev(0.5)
    h = {k: rng.standard_normal(n) for k in "qprtxzw"}
    v = {k: dev(a) for k, a in h.items()}
    assert L.acgsolvercuda_pipelined_daxpy_fused(n, g.data_ptr(), gp.data_ptr(), d.data_ptr(), v["q"].data_ptr(), v["p"].data_ptr(),
                                                 v["r"].data_ptr(), v["t"].data_ptr(), v["x"].data_ptr(), v["z"].data_ptr(),
                                                 v["w"].data_ptr(), ap.data_ptr(), None) == 0
    torch.cuda.synchronize()
    beta = 0.5; alpha = 2.0 / (3.0 - beta * 2.0 / 0.5)
    z = h["q"] + beta * h["z"]; t = h["w"] + beta * h["t"]; p = h["r"] + beta * h["p"]
    for k, want in (("z", z), ("t", t), ("p", p), ("x", h["x"] + alpha * p), ("r", h["r"] - alpha * t), ("w", h["w"] - alpha * z)):
        assert np.allclose(v[k].cpu().numpy(), want, rtol=1e-14, atol=1e-14), k
    assert gp.item() == 2.0 and ap.item() == alpha
    m1, p1, z0 = C.c_void_p(), C.c_void_p(), C.c_void_p()
    assert L.acgsolvercuda_init_constants(C.byref(m1), C.byref(p1), C.byref(z0)) == 0
    got = torch.zeros(3, dtype=torch.float64, device="cuda")
    for i, q in enumerate((m1, p1, z0)):
        assert L.acgsolvercuda_daxpy_alpha(1, q.value, p1.value, p1.value, got[i:i + 1].data_ptr()) == 0    # got[i] += (q/1)*1
    torch.cuda.synchronize()
    assert got.cpu().tolist() == [-1.0, 1.0, 0.0]


# ---- nonzero initial guesses ------------------------------------------------------------------
# With x0 = 0 the set-up product r0 = b - A x0 is b - 0: a wrong sign or a wrong b[row] in an epilogue of mode
# r = b - A x, or a warm-up that clobbers x0, would go unnoticed.  These solves start elsewhere.

def _laplacian_values(n, r, c):
    """off-diagonal -1, diagonal 1 + degree: symmetric, strictly diagonally dominant"""
    off = r != c
    deg = np.bincount(r[off], minlength=n) + np.bincount(c[off], minlength=n)
    v = np.where(off, -1.0, 0.0)
    v[~off] = 1.0 + deg[r[~off]]
    return v


def _x0_plan(name):
    from test_gpu_kernel_variants import slice_matrix
    if name == "tiles":
        return mg.stencil3d_27pt(10, 9, 11), dict(spmv_slices=0, spmv_merge=0)
    if name == "slices":
        return mg.stencil3d_27pt(10, 9, 11), {}
    if name == "slices-exc":
        n, r, c = slice_matrix(True)
        return (n, r, c, _laplacian_values(n, r, c)), {}
    if name == "merge":
        return mg.rmat_spd(6000, 60000, seed=3), dict(spmv_merge=1, spmv_slices=0, merge_items=256)
    if name == "medium+long":
        return mg.rmat_spd(30000, 600000, seed=8), dict(spmv_medium=96, spmv_merge=0)
    raise ValueError(name)


X0_PLANS = ["tiles", "slices", "slices-exc", "merge", "medium+long"]
X0_ENTRIES = [("solvempi", "cg"), ("solve_pipelined", "cg_pipelined"), ("solve_device", "cg"),
              ("solve_device_pipelined", "cg_pipelined"), ("solve", "cg")]
_X0_DEFAULTS = {"spmv_slices": 1, "spmv_merge": -1, "merge_items": 0, "spmv_medium": 0}


@pytest.mark.parametrize("plan", X0_PLANS)
def test_nonzero_initial_guess(plan, ab, oracle):
    """All five entry points, warm-up 0 and 2, from a random x0 (against the oracle started from the same x0),
    from an x0 next to the solution (r0nrm2 against the exact ||b - A x0||) and with maxits = 0 (x comes back
    bitwise as x0)."""
    from exactref import gamma, rows_exact
    (n, r, c, v), opts = _x0_plan(plan)
    for k, val in opts.items():
        ab.set_option(k, val)
    try:
        A, cg = _solver(ab, n, r, c, v)
    finally:
        for k in opts:
            ab.set_option(k, _X0_DEFAULTS[k])
    inf = cg.info()
    assert {"tiles": inf["spmv_slices"] == 0 and inf["spmv_merge_tiles"] == 0 and inf["spmv_ntiles"] > 0,
            "slices": inf["spmv_slices"] > 0 and inf["spmv_slice_exc"] == 0,
            "slices-exc": inf["spmv_slice_exc"] > 0,
            "merge": inf["spmv_merge_tiles"] > 0 and inf["spmv_merge_split"] > 0,
            "medium+long": inf["spmv_nmedium"] > 0 and inf["spmv_nlong"] > 0}[plan], inf
    csr = (A.frowptr.copy(), A.fcolidx.copy(), A.fa.copy())
    rng = np.random.default_rng(21)
    b = A.vector(); b.x[:] = rng.standard_normal(n)
    x0 = rng.standard_normal(n)
    # the power-law matrices are ill conditioned: compare after a fixed number of iterations (as above)
    fixed = plan in ("merge", "medium+long")
    its, rtol, xtol = (10, 0.0, 1e-7) if fixed else (300, 1e-9, 1e-9)
    xs = rng.standard_normal(n)
    bs = A.vector(); bs.x[:] = rows_exact(*csr, xs)[0]
    xnear = xs + 1e-10 * rng.standard_normal(n)
    rexact, rscale, m = rows_exact(*csr, xnear, bs.x)
    for entry, oname in X0_ENTRIES:
        want = getattr(oracle, oname)(csr, b.x, x0=x0, maxits=its, rtol=rtol)
        for warmup in (0, 2):
            tag = (plan, entry, warmup)
            x = A.vector(); x.x[:] = x0
            code = getattr(cg, entry)(b, x, maxits=its, residualrtol=rtol, warmup=warmup)
            assert code == want["status"] == 0, tag
            assert cg.c.niterations == want["niterations"], tag
            assert cg.c.r0nrm2 == pytest.approx(want["r0nrm2"], rel=1e-13), tag
            assert cg.c.rnrm2 / cg.c.r0nrm2 == pytest.approx(want["rnrm2"] / want["r0nrm2"], rel=1e-6, abs=RES_RTOL), tag
            assert np.abs(x.x - want["x"]).max() <= xtol * np.abs(want["x"]).max(), tag
            # next to the solution: r0 = b - A x0 is 1e-9 of b, the exact norm is known
            x = A.vector(); x.x[:] = xnear
            getattr(cg, entry)(bs, x, maxits=1, warmup=warmup)
            bound = np.linalg.norm(2.0 * gamma(m + 1) * rscale)
            assert abs(cg.c.r0nrm2 - np.linalg.norm(rexact)) <= bound, (tag, cg.c.r0nrm2, np.linalg.norm(rexact), bound)
            # no iteration: x0 comes back untouched, whatever the warm-up did
            x = A.vector(); x.x[:] = x0
            assert getattr(cg, entry)(b, x, maxits=0, warmup=warmup) in (0, 39) and cg.c.niterations == 0, tag
            assert np.array_equal(x.x, x0), tag
    cg.free()
