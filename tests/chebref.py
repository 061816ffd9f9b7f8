"""NumPy restatement of the Chebyshev-preconditioned CG that acgsolvercuda_solve_chebyshev runs (DESIGN
section 15): PCG with M^-1 = p_d(D^-1 A) D^-1, z = M^-1 r formed by d steps of Jacobi-scaled Chebyshev
iteration on A z = r from z = 0 (Saad, Iterative Methods, Alg. 12.1), and, when no upper bound is given,
the bound b = 1.1 theta_max from the Lanczos matrix of 10 Jacobi-PCG steps.  Scalars and vectors are formed
in the kernels' order.  Products and dot products are plain sums here and per-row FMA chains and atomics of
per-CTA partial sums on the device, so the two agree to rounding, not bitwise.  Pinned against
scipy.sparse.linalg.cg by tests/test_chebref.py."""
import numpy as np

NOT_CONVERGED, INVALID_VALUE = 39, 29
MAXDEG, EST_STEPS = 16, 10


def threshold(atol, rtol, r0nrm2):
    """acg/cgcuda.c: ||r|| < atol or ||r|| < rtol ||r0||, each only when positive."""
    t = atol if atol > 0 else 0.0
    return max(t, rtol * r0nrm2)


def coefficients(degree, a, b):
    """c0 = 1/theta of the start d0 = c0 D^-1 r, and (c1_j, c2_j) = (rho_j rho_{j-1}, 2 rho_j / delta) of steps
    j = 1..degree."""
    theta, delta = (a + b) / 2, (b - a) / 2
    sigma = theta / delta
    rho = 1 / sigma
    steps = []
    for _ in range(degree):
        rn = 1 / (2 * sigma - rho)
        steps.append((rn * rho, 2 * rn / delta))
        rho = rn
    return 1 / theta, steps


def apply_prec(A, dinv, r, c0, steps):
    """z = p_d(D^-1 A) D^-1 r in the kernels' order; degree 0 (no steps): z = D^-1 r."""
    if not steps:
        return dinv * r
    res = r.copy()
    d = c0 * (dinv * r)
    z = d.copy()
    for c1, c2 in steps:
        res = res - A @ d
        d = c1 * d + c2 * (dinv * res)
        z = z + d
    return z


def lanczos_matrix(alpha, beta):
    """The k x k Lanczos tridiagonal of k CG steps: diagonal 1/alpha_j + beta_{j-1}/alpha_{j-1}, off-diagonal
    sqrt(beta_j)/alpha_j."""
    k = len(alpha)
    T = np.zeros((k, k))
    for j in range(k):
        T[j, j] = 1 / alpha[j] + (beta[j - 1] / alpha[j - 1] if j > 0 else 0.0)
        if j + 1 < k:
            T[j, j + 1] = T[j + 1, j] = np.sqrt(beta[j]) / alpha[j]
    return T


def pcg_steps(A, dinv, r0, steps, tol, maxits, c0=None, prec=None, x=None):
    """PCG from r0 in the kernels' order.  Returns (x or None, r, niterations, alphas, betas, stop, rr)."""
    prec = prec or (lambda r: apply_prec(A, dinv, r, c0, steps))
    r = r0.copy()
    z = prec(r)
    rz = float(r @ z)
    p = z.copy()
    alphas, betas = [], []
    k, stop, rr = 0, "maxits", float(r0 @ r0)
    while k < maxits:
        t = A @ p
        pap = float(p @ t)
        if not (rz > 0 and np.isfinite(rz)) or not (pap > 0 and np.isfinite(pap)):
            stop = "breakdown"
            break
        alpha = rz / pap
        alphas.append(alpha)
        if x is not None:
            x = x + alpha * p
        r = r - alpha * t
        rr = float(r @ r)
        z = prec(r)
        rzn = float(r @ z)
        beta = rzn / rz
        k += 1
        if tol > 0 and np.sqrt(rr) < tol:
            stop = "tol"
            break
        betas.append(beta)
        p = z + beta * p
        rz = rzn
    return x, r, k, alphas, betas, stop, rr


def estimate(A, dinv, r0, tol):
    """The interval estimate: EST_STEPS Jacobi-PCG steps from r0 (fewer on a breakdown or when ||r|| < tol),
    the extreme eigenvalues of their Lanczos matrix.  Returns (theta_min, theta_max, steps)."""
    _, _, k, alphas, betas, _, _ = pcg_steps(A, dinv, r0, [], tol, EST_STEPS)
    if k == 0:
        return 0.0, 0.0, 0
    ev = np.linalg.eigvalsh(lanczos_matrix(alphas[:k], betas[:k - 1]))
    return float(ev[0]), float(ev[-1]), k


def _status(tol, rnrm2, atol, rtol_scaled):
    """acgsolvercuda_solvempi's rule: not converged fails unless both tolerances are off."""
    return 0 if (tol > 0 and rnrm2 < tol) or (atol == 0 and rtol_scaled == 0) else NOT_CONVERGED


class Invalid(Exception):
    pass


def chebyshev(A, b, degree=2, x0=None, lmin=0.0, lmax=0.0, maxits=100, atol=0.0, rtol=0.0):
    """A: scipy sparse SPD (float64), b: float64.  Returns a dict with x, niterations, rnrm2 (the recursively
    updated residual norm), r0nrm2, bnrm2, status (0 or NOT_CONVERGED), stop ("tol", "breakdown", "maxits"
    or "none": no iteration ran), the interval [lmin, lmax] used, est_steps and products.  Raises Invalid
    where the solver returns ACG_ERR_INVALID_VALUE."""
    if not 0 <= degree <= MAXDEG:
        raise Invalid("degree")
    if degree > 0:
        if not (np.isfinite(lmin) and np.isfinite(lmax) and lmin >= 0 and lmax >= 0):
            raise Invalid("interval")
        if lmin > 0 and lmax > 0 and lmin >= lmax:
            raise Invalid("interval")
    diag = np.asarray(A.diagonal(), np.float64)
    if not np.all((diag > 0) & np.isfinite(diag)):
        raise Invalid("diagonal")
    dinv = 1 / diag
    b = np.asarray(b, np.float64)
    x = np.zeros_like(b) if x0 is None else np.array(x0, np.float64)
    r = b - A @ x
    rr0 = float(r @ r)
    r0 = float(np.sqrt(rr0))
    tol = threshold(atol, rtol, r0)
    out = {"r0nrm2": r0, "bnrm2": float(np.linalg.norm(b)), "niterations": 0, "tol": tol, "rnrm2": r0,
           "stop": "none", "lmin": 0.0, "lmax": 0.0, "est_steps": 0, "products": 1, "x": x}
    if maxits == 0 or (tol > 0 and r0 < tol) or rr0 == 0:
        out["status"] = _status(tol, r0, atol, rtol * r0)
        return out
    a_, b_ = 0.0, 0.0
    if degree > 0:
        b_ = lmax
        if lmax == 0:
            _, tmax, k = estimate(A, dinv, r, tol)
            out["est_steps"] = k
            out["products"] += k
            if k == 0:
                out.update(stop="breakdown", status=_status(tol, r0, atol, rtol * r0))
                return out
            b_ = 1.1 * tmax
        a_ = lmin if lmin > 0 else b_ / 10
        if not (np.isfinite(b_) and a_ < b_):
            raise Invalid("interval")
    out["lmin"], out["lmax"] = a_, b_
    c0, steps = coefficients(degree, a_, b_) if degree > 0 else (0.0, [])
    out["products"] += degree
    x, _, k, _, _, stop, rr = pcg_steps(A, dinv, r, steps, tol, maxits, c0=c0, x=x)
    out.update(x=x, niterations=k, stop=stop, products=out["products"] + k * (1 + degree))
    if k > 0:
        out["rnrm2"] = float(np.sqrt(rr))
    out["status"] = _status(tol, out["rnrm2"], atol, rtol * r0)
    return out
