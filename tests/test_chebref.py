"""tests/chebref.py, the restatement of acgsolvercuda_solve_chebyshev, against scipy and dense linear algebra:
PCG with M^-1 = p_d(D^-1 A) D^-1 equals scipy.sparse.linalg.cg with that preconditioner after fixed iteration
counts; degree 0 is Jacobi PCG; M^-1 is positive definite exactly when the spectrum of D^-1 A lies in
(0, a + b); the estimate's Ritz values lie inside the spectrum of D^-1 A; and acgb200_cheb_interval_host (the
solver's Sturm bisection) gives the extreme eigenvalues of the Lanczos matrix."""
import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as sla

from acg_b200 import matgen as mg
from chebref import apply_prec, chebyshev, coefficients, estimate, lanczos_matrix, pcg_steps


def _full(n, r, c, v):
    U = sp.coo_matrix((v, (r, c)), shape=(n, n)).tocsr()
    return (U + U.T - sp.diags(U.diagonal())).tocsr()


MATS = {"7pt": lambda: _full(*mg.laplace3d_7pt(8, 7, 9)), "27pt": lambda: _full(*mg.stencil3d_27pt(7)),
        "rmat": lambda: _full(*mg.rmat_spd(1500, 20000, seed=3)), "spd": lambda: _full(*mg.random_spd(120, 0.08, seed=2))}


def _prec_matrix(A, degree, a, b):
    n = A.shape[0]
    dinv = 1 / A.diagonal()
    c0, steps = coefficients(degree, a, b)
    return np.column_stack([apply_prec(A, dinv, e, c0, steps) for e in np.eye(n)])


@pytest.mark.parametrize("key", sorted(MATS))
@pytest.mark.parametrize("degree", [0, 1, 2, 5])
def test_against_scipy_cg(key, degree):
    A = MATS[key]()
    n = A.shape[0]
    b = np.random.default_rng(1).standard_normal(n)
    dinv = 1 / A.diagonal()
    _, tmax, _ = estimate(A, dinv, b, 0.0)
    c0, steps = coefficients(degree, 0.11 * tmax, 1.1 * tmax)
    M = sla.LinearOperator((n, n), matvec=lambda r: apply_prec(A, dinv, np.ravel(r), c0, steps), dtype=np.float64)
    for its in (1, 3, 8):
        x, _, k, _, _, _, _ = pcg_steps(A, dinv, b, steps, 0.0, its, c0=c0, x=np.zeros(n))
        assert k == its
        xs, _ = sla.cg(A, b, x0=np.zeros(n), rtol=0.0, atol=0.0, maxiter=its, M=M)
        assert np.abs(x - xs).max() <= 1e-10 * np.abs(xs).max(), (its, np.abs(x - xs).max())


def test_degree0_is_jacobi_pcg():
    A = MATS["rmat"]()
    n = A.shape[0]
    b = np.random.default_rng(2).standard_normal(n)
    dinv = 1 / A.diagonal()
    ref = chebyshev(A, b, degree=0, maxits=500, rtol=1e-10)
    x, _, k, _, _, stop, _ = pcg_steps(A, dinv, b, [], 1e-10 * np.linalg.norm(b), 500, prec=lambda r: dinv * r,
                                       x=np.zeros(n))
    assert stop == "tol" and k == ref["niterations"] and np.array_equal(x, ref["x"])
    assert ref["est_steps"] == 0 and ref["lmax"] == 0.0


@pytest.mark.parametrize("key", ["7pt", "spd"])
@pytest.mark.parametrize("degree", [1, 2, 3, 4])
def test_spd_exactly_inside_the_interval(key, degree):
    """p_d(D^-1 A) D^-1 is SPD when every eigenvalue of D^-1 A lies in (0, a + b) and indefinite when one lies
    far enough beyond (odd degrees; even-degree polynomials stay positive on the real line here)."""
    A = MATS[key]()
    dinv = 1 / A.diagonal()
    lam = np.linalg.eigvalsh((sp.diags(np.sqrt(dinv)) @ A @ sp.diags(np.sqrt(dinv))).toarray())
    lmax = lam[-1]
    good = _prec_matrix(A, degree, 0.1 * lmax, 1.0 * lmax)
    assert np.abs(good - good.T).max() < 1e-12 * np.abs(good).max()
    assert np.linalg.eigvalsh((good + good.T) / 2)[0] > 0
    # a + b = 0.55 lambda_max: the residual polynomial 1 - lambda p(lambda) changes sign beyond a + b
    bad = _prec_matrix(A, degree, 0.05 * lmax, 0.5 * lmax)
    ev = np.linalg.eigvalsh((bad + bad.T) / 2)
    if degree % 2 == 1:
        assert ev[0] < 0 < ev[-1]
    lam_p = np.linalg.eigvals(sp.diags(dinv).toarray() @ A.toarray() @ bad).real
    assert (lam_p.min() <= 0) == (ev[0] <= 0)


@pytest.mark.parametrize("key", sorted(MATS))
def test_ritz_values_inside_the_spectrum(key):
    A = MATS[key]()
    dinv = 1 / A.diagonal()
    lam = np.linalg.eigvalsh((sp.diags(np.sqrt(dinv)) @ A @ sp.diags(np.sqrt(dinv))).toarray())
    b = np.random.default_rng(3).standard_normal(A.shape[0])
    tmin, tmax, k = estimate(A, dinv, b, 0.0)
    assert k == 10
    assert lam[0] * (1 - 1e-12) <= tmin <= tmax <= lam[-1] * (1 + 1e-12)
    assert tmax > 0.9 * lam[-1]


@pytest.mark.parametrize("key", sorted(MATS))
def test_interval_host_matches_eigvalsh(key):
    import acg_b200.api as api
    A = MATS[key]()
    dinv = 1 / A.diagonal()
    b = np.random.default_rng(4).standard_normal(A.shape[0])
    for kmax in (1, 2, 5, 10):
        _, _, k, al, be, _, _ = pcg_steps(A, dinv, b, [], 0.0, kmax, prec=lambda r: dinv * r)
        ev = np.linalg.eigvalsh(lanczos_matrix(al[:k], be[:k - 1]))
        tmin, tmax = api.cheb_interval_host(al[:k], be[:k - 1])
        assert tmax == pytest.approx(ev[-1], rel=1e-12)
        assert tmin == pytest.approx(ev[0], rel=1e-12, abs=1e-12 * ev[-1])
    with pytest.raises(api.AcgError):
        api.cheb_interval_host([1.0, -1.0], [0.5])
    with pytest.raises(api.AcgError):
        api.cheb_interval_host([1.0, 1.0], [float("nan")])
