"""Float64 NumPy restatement of the MINRES recurrence acgsolvercuda_solve_minres runs (DESIGN section 13):
unpreconditioned Paige-Saunders in the formulation of scipy.sparse.linalg.minres, with the solver's stopping
rule and breakdown handling, each vector and scalar formed in the order the kernels form it.  Dot products
are plain sums here and atomics of per-CTA partial sums on the device, so the two agree to rounding, not
bitwise.  Pinned against scipy and spsolve by tests/test_minresref.py."""
import numpy as np

NOT_CONVERGED = 39


def threshold(atol, rtol, r0nrm2):
    """acg/cgcuda.c: ||r|| < atol or ||r|| < rtol ||r0||, each only when positive."""
    t = atol if atol > 0 else 0.0
    return max(t, rtol * r0nrm2)


def stencil_eigenvalues(kind, nx, ny=None, nz=None):
    """The spectrum, sorted, of acg_b200.matgen's 7-point (diagonal 6) or 27-point (diagonal 26) stencil
    with off-diagonal -1 on an nx x ny x nz box, Dirichlet truncation, in closed form: with
    c_i = cos(i pi / (m + 1)) per axis, 6 - 2 (c_i + c_j + c_k) and 27 - (1 + 2 c_i)(1 + 2 c_j)(1 + 2 c_k)."""
    ny = nx if ny is None else ny
    nz = nx if nz is None else nz
    cx, cy, cz = (np.cos(np.pi * np.arange(1, m + 1) / (m + 1)) for m in (nx, ny, nz))
    if kind == 7:
        lam = 6.0 - 2.0 * (cx[:, None, None] + cy[None, :, None] + cz[None, None, :])
    elif kind == 27:
        lam = 27.0 - (1 + 2 * cx)[:, None, None] * (1 + 2 * cy)[None, :, None] * (1 + 2 * cz)[None, None, :]
    else:
        raise ValueError(kind)
    return np.sort(lam.ravel())


def indefinite_shift(eigs, nneg):
    """sigma halfway between the nneg-th and (nneg+1)-th smallest of the sorted eigenvalues: A - sigma I
    (dsymv_init(-sigma)) then has exactly nneg negative eigenvalues, none closer to 0 than half the gap."""
    lo, hi = float(eigs[nneg - 1]), float(eigs[nneg])
    if not hi - lo > 1e-6 * abs(hi):
        raise ValueError(f"no gap after eigenvalue {nneg}: {lo} {hi}")
    return 0.5 * (lo + hi)


def minres(A, b, x0=None, maxits=100, atol=0.0, rtol=0.0, callback=None):
    """Solve A x = b for symmetric A (anything with A @ v).  Returns a dict with x, niterations, rnrm2 (the
    final phi-bar), r0nrm2, bnrm2, status (0 or NOT_CONVERGED) and stop, one of 'r0' (converged or
    beta_1 = 0 at the start), 'maxits', 'tol', 'breakdown' (beta_{k+1} = 0, after the update) and 'gamma'
    (gamma_k = 0, before the update, which is not counted).  callback(x) runs after every counted iteration."""
    b = np.asarray(b, np.float64)
    n = len(b)
    x = np.zeros(n) if x0 is None else np.array(x0, np.float64)
    r = b - A @ x
    beta1 = float(np.sqrt(np.dot(r, r)))
    tol = threshold(atol, rtol, beta1)
    out = {"bnrm2": float(np.linalg.norm(b)), "r0nrm2": beta1, "rnrm2": beta1, "niterations": 0, "stop": "r0"}
    k = 0
    phibar = beta1
    if not (tol > 0 and beta1 < tol) and maxits > 0 and beta1 > 0:
        out["stop"] = "maxits"
        v = r * (1.0 / beta1)
        vprev = np.zeros(n)
        w2 = np.zeros(n)              # w_{k-2}
        w1 = np.zeros(n)              # w_{k-1}
        beta, cs, sn, dbar, eps = beta1, -1.0, 0.0, 0.0, 0.0
        while k < maxits:
            t = A @ v
            alpha = float(np.dot(v, t))
            u = (t - alpha * v) - beta * vprev
            bn = float(np.sqrt(np.dot(u, u)))
            delta = cs * dbar + sn * alpha
            gbar = sn * dbar - cs * alpha
            epsn = sn * bn
            dbarn = -cs * bn
            gamma = float(np.hypot(gbar, bn))
            if gamma == 0.0:
                out["stop"] = "gamma"
                break
            csn, snn = gbar / gamma, bn / gamma
            phi = csn * phibar
            phibar = snn * phibar
            w = ((v - eps * w2) - delta * w1) * (1.0 / gamma)
            x = x + phi * w
            vnext = u * (1.0 / bn) if bn > 0 else np.zeros(n)
            k += 1
            w2, w1 = w1, w
            vprev, v = v, vnext
            beta, cs, sn, dbar, eps = bn, csn, snn, dbarn, epsn
            if callback is not None:
                callback(x)
            if bn == 0.0:
                out["stop"] = "breakdown"
                break
            if tol > 0 and phibar < tol:
                out["stop"] = "tol"
                break
        out["rnrm2"] = phibar
    out["x"] = x
    out["niterations"] = k
    converged = tol > 0 and out["rnrm2"] < tol
    out["status"] = 0 if converged or (atol == 0 and rtol * beta1 == 0) else NOT_CONVERGED
    return out
