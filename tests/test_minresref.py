"""The MINRES restatement of tests/minresref.py, pinned down on the CPU: its iterates equal those of
scipy.sparse.linalg.minres (rtol = 0, maxiter = m, x from the callback) within 1e-12 relative on small
positive definite and indefinite matrices and from a nonzero initial guess; at convergence its x equals
spsolve's; the breakdown cases end where the recurrence says (beta_{k+1} = 0 after one iteration for a
diagonal matrix and b = e_i, gamma_k = 0 before it for a zero row, b = 0 without an iteration); and the
stopping rule is solvempi's."""
import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from minresref import NOT_CONVERGED, indefinite_shift, minres, stencil_eigenvalues


def _laplace1d(n):
    return sp.diags([-np.ones(n - 1), 2.0 * np.ones(n), -np.ones(n - 1)], [-1, 0, 1], format="csr")


def _random_sym(n, seed, nneg):
    """A random sparse symmetric matrix with diagonal dominance; with nneg > 0 shifted to halfway between
    its nneg-th and (nneg+1)-th eigenvalue, so that nneg eigenvalues are negative and none is near 0."""
    rng = np.random.default_rng(seed)
    R = sp.random(n, n, density=0.1, random_state=rng, format="csr")
    S = (R + R.T) * 0.5
    A = (S + sp.diags(np.abs(S).sum(axis=1).A1 + 1.0)).tocsr()
    if nneg:
        ev = np.linalg.eigvalsh(A.toarray())
        A = (A - 0.5 * (ev[nneg - 1] + ev[nneg]) * sp.eye(n)).tocsr()
    return A


def _matrices():
    yield "laplace1d_spd", _laplace1d(60)
    yield "laplace1d_indefinite", (_laplace1d(60) - 1.3 * sp.eye(60)).tocsr()
    yield "random_spd", _random_sym(80, 1, 0)
    yield "random_indefinite", _random_sym(80, 2, 8)


def _eigs(A):
    return np.linalg.eigvalsh(A.toarray())


def test_matrices_are_what_they_claim():
    for name, A in _matrices():
        ev = _eigs(A)
        assert np.allclose(A.toarray(), A.toarray().T)
        if "indefinite" in name:
            assert ev.min() < 0 < ev.max(), name
        else:
            assert ev.min() > 0, name


@pytest.mark.parametrize("m", [1, 2, 5, 10, 15])
@pytest.mark.parametrize("nonzero_x0", [False, True])
def test_iterates_equal_scipy(m, nonzero_x0):
    for name, A in _matrices():
        n = A.shape[0]
        rng = np.random.default_rng(7)
        b = rng.standard_normal(n)
        x0 = rng.standard_normal(n) if nonzero_x0 else np.zeros(n)
        seen = []
        spla.minres(A, b, x0=x0.copy(), rtol=0.0, maxiter=m, callback=lambda xk: seen.append(xk.copy()))
        assert len(seen) == m, (name, len(seen))
        ref = minres(A, b, x0=x0, maxits=m)
        assert ref["niterations"] == m and ref["stop"] == "maxits" and ref["status"] == 0
        err = np.abs(ref["x"] - seen[-1]).max() / np.abs(seen[-1]).max()
        assert err < 1e-12, (name, m, err)
        # phi-bar is the residual norm of the iterate (exact arithmetic; here to rounding)
        true = np.linalg.norm(b - A @ ref["x"])
        assert ref["rnrm2"] == pytest.approx(true, rel=1e-8, abs=1e-12 * np.linalg.norm(b)), (name, m)


@pytest.mark.parametrize("name", ["laplace1d_spd", "laplace1d_indefinite", "random_spd", "random_indefinite"])
def test_converged_equals_spsolve(name):
    A = dict(_matrices())[name]
    n = A.shape[0]
    b = np.random.default_rng(3).standard_normal(n)
    ref = minres(A, b, maxits=10 * n, rtol=1e-12)
    assert ref["stop"] == "tol" and ref["status"] == 0
    assert ref["rnrm2"] < 1e-12 * np.linalg.norm(b)
    xs = spla.spsolve(A.tocsc(), b)
    cond = np.linalg.cond(A.toarray())
    assert np.abs(ref["x"] - xs).max() / np.abs(xs).max() < 1e-12 * cond * 10


def test_stopping_rule():
    A = dict(_matrices())["random_indefinite"]
    n = A.shape[0]
    b = np.random.default_rng(4).standard_normal(n)
    # rtol and atol: the strict test on phi-bar, the first iteration that meets it
    for atol, rtol in ((0.0, 1e-6), (1e-5, 0.0), (1e-5, 1e-6)):
        ref = minres(A, b, maxits=500, atol=atol, rtol=rtol)
        tol = max(atol, rtol * np.linalg.norm(b))
        assert ref["stop"] == "tol" and ref["rnrm2"] < tol and ref["status"] == 0
        before = minres(A, b, maxits=ref["niterations"] - 1, atol=atol, rtol=rtol)
        assert before["rnrm2"] >= tol and before["status"] == NOT_CONVERGED and before["stop"] == "maxits"
    # maxits = 0: x0 unchanged, not converged under a tolerance, success without one
    x0 = np.random.default_rng(5).standard_normal(n)
    ref = minres(A, b, x0=x0, maxits=0, rtol=1e-8)
    assert ref["niterations"] == 0 and np.array_equal(ref["x"], x0) and ref["status"] == NOT_CONVERGED
    assert minres(A, b, x0=x0, maxits=0)["status"] == 0
    # r0 meets the test: no iteration
    ref = minres(A, b, maxits=50, atol=2 * np.linalg.norm(b))
    assert ref["niterations"] == 0 and ref["status"] == 0 and ref["stop"] == "r0"


@pytest.mark.parametrize("kind,box", [(7, (5, 6, 7)), (27, (6, 5, 4)), (7, (11, 11, 11))])
def test_stencil_spectrum_in_closed_form(kind, box):
    """stencil_eigenvalues against eigvalsh of the assembled matrix, and indefinite_shift's count."""
    from acg_b200 import matgen as mg
    n, r, c, v = (mg.laplace3d_7pt if kind == 7 else mg.stencil3d_27pt)(*box)
    U = sp.csr_matrix((v, (r, c)), shape=(n, n))
    A = (U + sp.triu(U, 1).T).toarray()
    ev = np.linalg.eigvalsh(A)
    cf = stencil_eigenvalues(kind, *box)
    assert np.abs(ev - cf).max() < 1e-12 * np.abs(ev).max()
    for nneg in (1, 4, 7):
        try:
            sigma = indefinite_shift(cf, nneg)
        except ValueError:
            continue                          # a multiple eigenvalue straddles nneg
        assert int((ev - sigma < 0).sum()) == nneg


def test_breakdown_cases():
    d = np.array([3.0, -2.0, 0.5, -7.0, 4.0, 1.0])
    D = sp.diags(d, format="csr")
    for i in range(len(d)):
        b = np.zeros(len(d)); b[i] = 1.5
        for rtol in (0.0, 1e-10):
            ref = minres(D, b, maxits=20, rtol=rtol)
            assert ref["stop"] == "breakdown" and ref["niterations"] == 1, (i, ref)
            want = np.zeros(len(d)); want[i] = 1.5 / d[i]
            assert np.allclose(ref["x"], want, rtol=1e-15, atol=0) and ref["rnrm2"] == 0.0
            assert ref["status"] == 0
    # b = 0: no iteration, x0 = 0 returned
    ref = minres(D, np.zeros(len(d)), maxits=20, rtol=1e-8)
    assert ref["niterations"] == 0 and not ref["x"].any() and ref["stop"] == "r0" and ref["status"] == 0
    # a zero row and b = e_i there: gamma_1 = 0, stopped before the update, not converged under a tolerance
    Z = sp.diags(np.where(np.arange(len(d)) == 2, 0.0, d), format="csr")
    b = np.zeros(len(d)); b[2] = 1.0
    ref = minres(Z, b, maxits=20, rtol=1e-8)
    assert ref["stop"] == "gamma" and ref["niterations"] == 0 and not ref["x"].any()
    assert ref["rnrm2"] == 1.0 and ref["status"] == NOT_CONVERGED
