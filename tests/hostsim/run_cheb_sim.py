"""TEST INFRASTRUCTURE ONLY: drive acgsolvercuda_solve_chebyshev on the device stand-in
(tests/hostsim/libacgb200_hostsim_cheb.so: the host-logic stand-in plus the multi-vector, shifted-systems,
MINRES, mixed-precision and Chebyshev kernel stand-ins) and compare every solve with the restatement of
tests/chebref.py on the matrix assembled.  Runs in its own process so that the binding loads the stand-in;
prints one JSON object.  Used by tests/test_hostsim_cheb.py."""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np                                   # noqa: E402
import scipy.sparse as sp                            # noqa: E402

import acg_b200.api as api                           # noqa: E402
api._LIBPATH = os.path.join(HERE, "libacgb200_hostsim_cheb.so")    # before the first lib() call
import acg_b200 as ab                                # noqa: E402
from acg_b200 import matgen as mg                    # noqa: E402
from chebref import Invalid, chebyshev               # noqa: E402


def case(name):
    if name == "pairs":
        # 2 x 2 blocks [[2, 1], [1, 2]] times 1..20: D^-1 A has two eigenvalues, Jacobi PCG ends after 2 steps
        m = 20
        rows = np.concatenate([[2 * i, 2 * i, 2 * i + 1] for i in range(m)]).astype(np.int32)
        cols = np.concatenate([[2 * i, 2 * i + 1, 2 * i + 1] for i in range(m)]).astype(np.int32)
        vals = np.concatenate([[2.0 * (i + 1), 1.0 * (i + 1), 2.0 * (i + 1)] for i in range(m)])
        return 2 * m, rows, cols, vals
    return {"27pt": lambda: mg.stencil3d_27pt(9, 8, 10), "7pt": lambda: mg.laplace3d_7pt(11),
            "rmat": lambda: mg.rmat_spd(2000, 32000, seed=1)}[name]()


def matrix(A):
    n = A.c.nownedrows
    rp = A.frowptr[:n + 1].copy()
    return sp.csr_matrix((A.fa[:rp[n]].copy(), A.fcolidx[:rp[n]] - A.c.rowidxbase, rp), shape=(n, n))


def solve_run(cg, A, M, n, run, seed):
    rng = np.random.default_rng(seed)
    b = np.ones(n) if run.get("bones") else rng.standard_normal(n)
    if run.get("bzero"):
        b[:] = 0.0
    x0 = rng.standard_normal(n) if run.get("x0") else np.zeros(n)
    kw = dict(degree=run["degree"], lmin=run.get("lmin", 0.0), lmax=run.get("lmax", 0.0), maxits=run["maxits"])
    atol, rtol = run.get("atol", 0.0), run.get("rtol", 0.0)
    bv = A.vector(); bv.x[:] = b
    xv = A.vector(); xv.x[:] = x0
    ngemv0 = int(cg.c.ngemv)
    try:
        code = cg.solve_chebyshev(bv, xv, residualatol=atol, residualrtol=rtol, warmup=run.get("warmup", 0), **kw)
    except ab.AcgError as e:
        code = e.code
    try:
        ref = chebyshev(M, b, x0=x0, atol=atol, rtol=rtol, **kw)
    except Invalid:
        return {"run": run, "code": int(code), "ref_code": 29, "x_is_x0": bool(np.array_equal(xv.x[:n], x0))}
    x = xv.x[:n].copy()
    scale = max(float(np.abs(ref["x"]).max()), 1e-300)
    inf = cg.info()
    return {"run": run, "code": int(code), "ref_code": int(ref["status"]), "its": int(cg.c.niterations),
            "ref_its": int(ref["niterations"]), "ref_stop": ref["stop"], "xerr": float(np.abs(x - ref["x"]).max() / scale),
            "x_is_x0": bool(np.array_equal(x, x0)), "rnrm2": float(cg.c.rnrm2), "ref_rnrm2": float(ref["rnrm2"]),
            "r0nrm2": float(cg.c.r0nrm2), "ref_r0nrm2": float(ref["r0nrm2"]), "bnrm2": float(cg.c.bnrm2),
            "ref_bnrm2": float(ref["bnrm2"]), "est": int(inf["cheb_est_iterations"]), "ref_est": int(ref["est_steps"]),
            "lmin": inf["cheb_lmin"], "lmax": inf["cheb_lmax"], "ref_lmin": ref["lmin"], "ref_lmax": ref["lmax"],
            "breakdown": int(inf["cheb_breakdown"]), "deg": int(inf["cheb_degree"]), "ngemv": int(cg.c.ngemv) - ngemv0,
            "ref_products": int(ref["products"]), "launches": int(inf["last_launches"]),
            "true_rnrm2": float(np.linalg.norm(b - M @ x)), "tol": float(ref["tol"])}


def alternate(A, M, n):
    """solve_chebyshev, solvempi and solve_mixed in turn on one solver; then solvempi on it against one on a
    fresh solver, bitwise."""
    cg = ab.SolverCuda(A)
    bv = A.vector(); bv.x[:] = np.random.default_rng(5).standard_normal(n)
    out = {"steps": []}
    for kind in ("cheb2", "single", "cheb0", "mixed", "cheb2", "single", "cheb5", "mixed", "cheb0", "cheb2"):
        x = A.vector()
        if kind.startswith("cheb"):
            code = cg.solve_chebyshev(bv, x, degree=int(kind[4:]), maxits=80, residualrtol=1e-8)
        else:
            code = {"mixed": cg.solve_mixed, "single": cg.solvempi}[kind](bv, x, maxits=80, residualrtol=1e-8)
        out["steps"].append({"kind": kind, "code": int(code), "its": int(cg.c.niterations), "x": x.x[:n].tolist(),
                             "deg": int(cg.info()["cheb_degree"])})
    x1 = A.vector()
    cg.solvempi(bv, x1, maxits=80, residualrtol=1e-8)
    cg2 = ab.SolverCuda(A)
    x2 = A.vector()
    cg2.solvempi(bv, x2, maxits=80, residualrtol=1e-8)
    out["single_after"] = {"same_x": bool(np.array_equal(x1.x, x2.x)), "its": [int(cg.c.niterations), int(cg2.c.niterations)]}
    cg2.free()
    cg.free()
    return out


def main():
    spec = json.loads(sys.argv[1])
    n, r, c, v = case(spec["matrix"])
    A = ab.SymCsrMatrix.init_real_double(n, r, c, v).dsymv_init(spec.get("eps", 0.0))
    M = matrix(A)
    cg = ab.SolverCuda(A)
    out = {"runs": [], "n": n}
    for i, run in enumerate(spec.get("runs", [])):
        out["runs"].append(solve_run(cg, A, M, n, run, 100 + i))
    cg.free()
    if spec.get("alternate"):
        out["alternate"] = alternate(A, M, n)
    if spec.get("partitioned"):
        parts = A.partition(2, (np.arange(n) >= n // 2).astype(np.int32))
        P = parts[0].dsymv_init(0.0)
        cgp = ab.SolverCuda(P)
        try:
            cgp.solve_chebyshev(P.vector(), P.vector(), maxits=3)
            out["partitioned_code"] = 0
        except ab.AcgError as e:
            out["partitioned_code"] = e.code
        cgp.free()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
