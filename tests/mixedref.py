"""NumPy restatement of the mixed-precision CG with reliable updates that acgsolvercuda_solve_mixed runs
(DESIGN section 14): r, p, t and y stored as float32 scaled by a power of two sigma, every operation in
float64 and each stored value rounded once, x and b in float64, and a reliable update -- y folded into x,
r replaced by b - A x from the fp64 product -- whenever the fp32 residual has fallen below 0.1 of its
largest value since the last one, or meets the tolerance.  Scalars and vectors are formed in the kernels'
order.  Products and dot products are plain sums here and per-row FMA chains and atomics of per-CTA
partial sums on the device, so the two agree to rounding, not bitwise.  Pinned against fp64 CG and
spsolve by tests/test_mixedref.py."""
import numpy as np

NOT_CONVERGED = 39
DELTA = 0.1
F32, F64 = np.float32, np.float64


def threshold(atol, rtol, r0nrm2):
    """acg/cgcuda.c: ||r|| < atol or ||r|| < rtol ||r0||, each only when positive."""
    t = atol if atol > 0 else 0.0
    return max(t, rtol * r0nrm2)


def scale_exp(rr):
    """e with sigma = 2^e = 2^round(log2 sqrt(rr))."""
    m, e = np.frexp(np.sqrt(rr))
    return int(e) - 1 if m < np.sqrt(0.5) else int(e)


def _dot(u, v):
    return float(np.dot(u.astype(F64), v.astype(F64)))


def mixed(A, b, x0=None, maxits=100, atol=0.0, rtol=0.0):
    """A: scipy sparse (float64), b: float64.  Returns a dict with x, niterations, nupdates, rnrm2 (the fp64
    residual norm of the x returned), r0nrm2, bnrm2, status (0 or NOT_CONVERGED) and stop ("tol",
    "breakdown", "maxits" or "none": no iteration ran)."""
    b = np.asarray(b, F64)
    x = np.zeros_like(b) if x0 is None else np.array(x0, F64)
    r64 = b - A @ x
    rr64 = float(r64 @ r64)
    r0 = float(np.sqrt(rr64))
    tol = threshold(atol, rtol, r0)
    out = {"r0nrm2": r0, "bnrm2": float(np.linalg.norm(b)), "niterations": 0, "nupdates": 0, "tol": tol}
    k, nupd, stop = 0, 0, "none"
    last_rr64 = rr64
    if maxits > 0 and not (tol > 0 and r0 < tol) and rr64 > 0:
        e = scale_exp(rr64)
        sigma, inv = np.ldexp(1.0, e), np.ldexp(1.0, -e)
        r = (r64 * inv).astype(F32)
        p = r.copy()
        y = np.zeros_like(r)
        rho = float(np.ldexp(rr64, -2 * e))
        M = np.sqrt(rho)
        stop = "maxits"
        while k < maxits:
            t = (A @ p.astype(F64)).astype(F32)
            pi = _dot(p, t)
            if not (pi != 0.0 and np.isfinite(pi)):
                stop = "breakdown"
                break
            alpha = rho / pi
            r = (r.astype(F64) - alpha * t.astype(F64)).astype(F32)
            rr = _dot(r, r)
            y = (y.astype(F64) + alpha * p.astype(F64)).astype(F32)
            nr = np.sqrt(rr)
            k += 1
            if not (nr < DELTA * M or sigma * nr < tol):
                beta = rr / rho
                p = (r.astype(F64) + beta * p.astype(F64)).astype(F32)
                rho, M = rr, max(M, nr)
                continue
            x = x + sigma * y.astype(F64)
            y[:] = 0.0
            r64 = b - A @ x
            rr64 = float(r64 @ r64)
            nupd += 1
            last_rr64 = rr64
            if np.sqrt(rr64) < tol or rr64 == 0.0:
                stop = "tol"
                break
            e = scale_exp(rr64)
            inv = np.ldexp(1.0, -e)
            bf = (rr64 / (sigma * sigma)) / rho * (sigma * inv)
            rv = r64 * inv
            p = (rv + bf * p.astype(F64)).astype(F32)
            r = rv.astype(F32)
            rho = float(np.ldexp(rr64, -2 * e))
            M = np.sqrt(rho)
            sigma = np.ldexp(1.0, e)
        if stop == "maxits":
            x = x + sigma * y.astype(F64)
            rf = b - A @ x
            last_rr64 = float(rf @ rf)
    rnrm2 = float(np.sqrt(last_rr64))
    converged = tol > 0 and rnrm2 < tol
    status = 0 if converged or (atol == 0 and rtol * r0 == 0) else NOT_CONVERGED
    out.update(x=x, niterations=k, nupdates=nupd, rnrm2=rnrm2, status=status, stop=stop)
    return out


def cg64(A, b, maxits=1000, rtol=1e-8):
    """Classic fp64 CG from x0 = 0 with the solver's test ||r|| < rtol ||r0|| on the recursive residual:
    (x, iterations)."""
    b = np.asarray(b, F64)
    x = np.zeros_like(b)
    r = b.copy()
    p = r.copy()
    rr = float(r @ r)
    tol = rtol * np.sqrt(rr)
    k = 0
    while k < maxits and not np.sqrt(rr) < tol:
        t = A @ p
        alpha = rr / float(p @ t)
        x += alpha * p
        r -= alpha * t
        rrn = float(r @ r)
        p = r + (rrn / rr) * p
        rr = rrn
        k += 1
    return x, k
