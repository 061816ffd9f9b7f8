"""The NumPy restatement of mixed-precision CG with reliable updates (tests/mixedref.py) against fp64 CG and
spsolve: it reaches fp64 tolerances on the true residual, stops by the solver's rule, is invariant under
scaling b by powers of two, ends cleanly on (p, A p) = 0, and needs at most 25 % more iterations than fp64
CG on the stencil boxes of the issue's prototype."""
import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from acg_b200 import matgen as mg
from mixedref import NOT_CONVERGED, cg64, mixed


def full(gen):
    n, r, c, v = gen
    rp, ci, a = mg.upper_to_full_csr(n, np.asarray(r), np.asarray(c), np.asarray(v))
    return sp.csr_matrix((a, ci, rp), shape=(n, n))


@pytest.fixture(scope="module")
def boxes():
    return {"7pt": full(mg.laplace3d_7pt(14)), "27pt": full(mg.stencil3d_27pt(11, 9, 10))}


@pytest.mark.parametrize("name", ["7pt", "27pt"])
@pytest.mark.parametrize("rtol", [1e-8, 1e-10])
def test_reaches_fp64_tolerance(boxes, name, rtol):
    A = boxes[name]
    rng = np.random.default_rng(3)
    b = rng.standard_normal(A.shape[0])
    out = mixed(A, b, maxits=1000, rtol=rtol)
    assert out["status"] == 0 and out["stop"] == "tol"
    true = np.linalg.norm(b - A @ out["x"])
    assert true == pytest.approx(out["rnrm2"], rel=1e-12)
    assert true < rtol * np.linalg.norm(b)
    xs = spla.spsolve(A.tocsc(), b)
    assert np.linalg.norm(out["x"] - xs) < 100 * rtol * np.linalg.norm(xs)
    x64, _ = cg64(A, b, rtol=rtol)
    assert np.linalg.norm(out["x"] - x64) < 100 * rtol * np.linalg.norm(xs)
    assert 1 <= out["nupdates"] <= out["niterations"]


def test_stopping_rule(boxes):
    """maxits reached: NOT_CONVERGED, the increment folded in and rnrm2 the fp64 residual of that x;
    maxits = 0 returns x0 bitwise; an atol met at x0 runs no iteration; b = 0 runs none; tolerances off
    run exactly maxits and succeed; the iteration before the converged one was not converged."""
    A = boxes["7pt"]
    n = A.shape[0]
    rng = np.random.default_rng(4)
    b, x0 = rng.standard_normal(n), rng.standard_normal(n)
    short = mixed(A, b, x0=x0, maxits=7, rtol=1e-10)
    assert short["status"] == NOT_CONVERGED and short["niterations"] == 7 and short["stop"] == "maxits"
    assert short["rnrm2"] == np.linalg.norm(b - A @ short["x"])
    zero = mixed(A, b, x0=x0, maxits=0, rtol=1e-8)
    assert zero["niterations"] == 0 and np.array_equal(zero["x"], x0) and zero["status"] == NOT_CONVERGED
    met = mixed(A, b, x0=x0, maxits=50, atol=1e6)
    assert met["niterations"] == 0 and met["status"] == 0 and np.array_equal(met["x"], x0)
    bz = mixed(A, np.zeros(n), maxits=50)
    assert bz["niterations"] == 0 and bz["status"] == 0 and bz["rnrm2"] == 0.0
    off = mixed(A, b, maxits=9)
    assert off["niterations"] == 9 and off["status"] == 0
    conv = mixed(A, b, maxits=500, rtol=1e-9)
    before = mixed(A, b, maxits=conv["niterations"] - 1, rtol=1e-9)
    assert conv["status"] == 0 and before["status"] == NOT_CONVERGED
    assert before["rnrm2"] >= conv["tol"]


@pytest.mark.parametrize("shift", [200, -200])
def test_scale_invariance(boxes, shift):
    """sigma is a power of two chosen from the residual, so b 2^s gives the same iterations and x 2^s
    exactly (fp32 without the scaling would overflow or underflow here)."""
    A = boxes["27pt"]
    rng = np.random.default_rng(5)
    b = rng.standard_normal(A.shape[0])
    ref = mixed(A, b, maxits=500, rtol=1e-9)
    sc = mixed(A, np.ldexp(b, shift), maxits=500, rtol=1e-9)
    assert (sc["niterations"], sc["nupdates"], sc["status"]) == (ref["niterations"], ref["nupdates"], ref["status"])
    assert np.array_equal(sc["x"], np.ldexp(ref["x"], shift))


def test_zero_curvature_ends_before_the_update():
    """A diagonal matrix with a zero entry and b on it: (p, A p) = 0 in the first iteration ends the solve
    with no iteration counted and x0 returned."""
    d = np.array([3.0, 0.0, 2.0, 5.0])
    A = sp.diags(d).tocsr()
    b = np.array([0.0, 1.0, 0.0, 0.0])
    out = mixed(A, b, maxits=20, rtol=1e-8)
    assert out["stop"] == "breakdown" and out["niterations"] == 0 and out["status"] == NOT_CONVERGED
    assert np.array_equal(out["x"], np.zeros(4)) and out["rnrm2"] == 1.0


@pytest.mark.parametrize("gen,rhs", [(lambda: mg.laplace3d_7pt(48), "ones"), (lambda: mg.laplace3d_7pt(40), "normal"),
                                     (lambda: mg.stencil3d_27pt(40), "ones"), (lambda: mg.stencil3d_27pt(32), "normal")])
def test_iteration_overhead(gen, rhs):
    """At most 25 % more CG steps than fp64 CG to rtol 1e-8 from x0 = 0, with a true residual below tol."""
    A = full(gen())
    n = A.shape[0]
    b = np.ones(n) if rhs == "ones" else np.random.default_rng(6).standard_normal(n)
    _, k64 = cg64(A, b, rtol=1e-8)
    out = mixed(A, b, maxits=4 * k64, rtol=1e-8)
    assert out["status"] == 0
    assert out["niterations"] <= 1.25 * k64, (out["niterations"], k64)
    assert np.linalg.norm(b - A @ out["x"]) < 1e-8 * np.linalg.norm(b)
