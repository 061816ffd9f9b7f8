"""TEST INFRASTRUCTURE ONLY: drive acgsolvercuda_solve_shifted on the device stand-in
(tests/hostsim/libacgb200_hostsim_shifted.so: the host-logic stand-in plus kernels_multi_sim.c and
kernels_shifted_sim.c) and compare every shift with the oracle's classic CG on the matrix assembled with
dsymv_init at eps = sigma_j, from x0 = 0.  Runs in its own process so that the binding loads the
stand-in; prints one JSON object.  Used by tests/test_hostsim_shifted.py."""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np                                   # noqa: E402

import acg_b200.api as api                           # noqa: E402
api._LIBPATH = os.path.join(HERE, "libacgb200_hostsim_shifted.so")    # before the first lib() call
import acg_b200 as ab                                # noqa: E402
from acg_b200 import matgen as mg                    # noqa: E402
from exactref import rows_exact                      # noqa: E402
from oracle import Oracle                            # noqa: E402


def case(name):
    return {"27pt": lambda: mg.stencil3d_27pt(9, 8, 10), "7pt": lambda: mg.laplace3d_7pt(11)}[name]()


class Shifted:
    """The matrix of every shift, assembled by dsymv_init(sigma), as the oracle's CSR arrays."""

    def __init__(self, coo):
        self.coo = coo
        self.csr = {}

    def __call__(self, sigma):
        if sigma not in self.csr:
            n, r, c, v = self.coo
            A = ab.SymCsrMatrix.init_real_double(n, r, c, v).dsymv_init(sigma)
            self.csr[sigma] = (A.frowptr.copy(), A.fcolidx.copy(), A.fa.copy())
            A.free()
        return self.csr[sigma]


def threshold(atol, rtol, r0):
    t = atol if atol > 0 else 0.0
    return max(t, rtol * r0)


def solve_run(O, shifted, cg, n, run, seed):
    b = np.random.default_rng(seed).standard_normal(n) * run.get("bscale", 1.0)
    if run.get("bzero"):
        b[:] = 0.0
    shifts = run["shifts"]
    atol, rtol = run.get("atol", 0.0), run.get("rtol", 0.0)
    code, X, cols = cg.solve_shifted(b, shifts, maxits=run["maxits"], residualatol=atol, residualrtol=rtol,
                                     warmup=run.get("warmup", 0))
    out = {"run": run, "code": int(code), "its": int(cg.c.niterations), "cols": [], "x_zero": bool(not X.any()),
           "launches": int(cg.info()["last_launches"]), "nsolves": int(cg.c.nsolves)}
    tol = threshold(atol, rtol, float(np.linalg.norm(b)))
    ref_codes = []
    sr = 0.0
    for j, sigma in enumerate(shifts):
        csr = shifted(float(sigma))
        ref = O.cg(csr, b, maxits=run["maxits"], atol=atol, rtol=rtol)
        ref_codes.append(int(ref["status"]))
        scale = max(float(np.abs(ref["x"]).max()), 1e-300)
        c = cols[j]
        rtrue, _, _ = rows_exact(*csr, X[:, j], b)
        out["cols"].append({"sigma": sigma, "its": c["niterations"], "ref_its": int(ref["niterations"]),
                            "converged": c["converged"], "ref_status": int(ref["status"]),
                            "xerr": float(np.abs(X[:, j] - ref["x"]).max() / scale),
                            "rnrm2": c["rnrm2"], "ref_rnrm2": float(ref["rnrm2"]), "r0nrm2": c["r0nrm2"],
                            "bnrm2": c["bnrm2"], "ref_bnrm2": float(ref["bnrm2"]),
                            "true_rnrm2": float(np.linalg.norm(rtrue)), "tol": tol})
        sr += c["rnrm2"] ** 2
    out["ref_code"] = 39 if any(rc == 39 for rc in ref_codes) else 0
    out["ref_its"] = max(c["ref_its"] for c in out["cols"])
    bn = float(np.linalg.norm(b))
    out["frobenius_ok"] = bool(np.isclose(cg.c.bnrm2, np.sqrt(len(shifts)) * bn, rtol=1e-13, atol=1e-300)
                               and np.isclose(cg.c.r0nrm2, cg.c.bnrm2, rtol=0, atol=0)
                               and np.isclose(cg.c.rnrm2, np.sqrt(sr), rtol=1e-14, atol=1e-300))
    return out


def alternate(O, coo, A, n):
    """solve_multi, solve_shifted and solvempi in turn on one solver; then a single-vector solve on it
    against one on a fresh solver, bitwise."""
    cg = ab.SolverCuda(A)
    rng = np.random.default_rng(5)
    b = rng.standard_normal(n)
    out = {"steps": []}
    for kind, k in (("multi", 3), ("shifted", 5), ("single", 1), ("shifted", 2), ("multi", 8), ("shifted", 8),
                    ("single", 1), ("shifted", 3)):
        if kind == "multi":
            B = rng.standard_normal((n, k)); X = np.zeros((n, k))
            code, cols = cg.solve_multi(B, X, maxits=80, residualrtol=1e-8)
            its = [c["niterations"] for c in cols]
        elif kind == "shifted":
            code, X, cols = cg.solve_shifted(b, [0.0, 1.0, 0.1, 0.01, 0.3, 0.03, 3.0, 0.003][:k], maxits=80, residualrtol=1e-8)
            its = [c["niterations"] for c in cols]
        else:
            bv = A.vector(); bv.x[:] = b
            x = A.vector()
            code = cg.solvempi(bv, x, maxits=80, residualrtol=1e-8)
            its = [int(cg.c.niterations)]
        out["steps"].append({"kind": kind, "k": k, "code": int(code), "its": its})
    # the sigma = 0 shift against solvempi: the same recurrence
    code, X, cols = cg.solve_shifted(b, [0.5, 0.0], maxits=80, residualrtol=1e-8)
    bv = A.vector(); bv.x[:] = b
    x1 = A.vector()
    cg.solvempi(bv, x1, maxits=80, residualrtol=1e-8)
    its1, r1 = int(cg.c.niterations), float(cg.c.rnrm2)
    out["sigma0"] = {"its": [cols[1]["niterations"], its1],
                     "xerr": float(np.abs(X[:, 1] - x1.x).max() / np.abs(x1.x).max())}
    cg2 = ab.SolverCuda(A)
    x2 = A.vector()
    cg2.solvempi(bv, x2, maxits=80, residualrtol=1e-8)
    out["single_after"] = {"same_x": bool(np.array_equal(x1.x, x2.x)), "its": [its1, int(cg2.c.niterations)],
                           "rnrm2": [r1, float(cg2.c.rnrm2)]}
    cg2.free()
    cg.free()
    return out


def main():
    spec = json.loads(sys.argv[1])
    for k, v in spec.get("options", {}).items():
        ab.set_option(k, v)
    O = Oracle()
    coo = case(spec["matrix"])
    n, r, c, v = coo
    A = ab.SymCsrMatrix.init_real_double(n, r, c, v).dsymv_init(0.0)
    shifted = Shifted(coo)
    cg = ab.SolverCuda(A)
    out = {"runs": []}
    for i, run in enumerate(spec.get("runs", [])):
        out["runs"].append(solve_run(O, shifted, cg, n, run, 100 + i))
    errs = {}
    b = np.ones(n)
    for name, shifts in (("nshifts0", []), ("nshifts9", [0.0] * 9), ("negative", [0.0, -1e-3]),
                         ("nan", [0.1, float("nan")]), ("inf", [float("inf")])):
        try:
            cg.solve_shifted(b, shifts, maxits=3)
            errs[name] = 0
        except ab.AcgError as e:
            errs[name] = e.code
    out["errors"] = errs
    out["nsolves"] = int(cg.c.nsolves)
    cg.free()
    if spec.get("alternate"):
        out["alternate"] = alternate(O, coo, A, n)
    if spec.get("partitioned"):
        # a part of a partitioned matrix (ghost rows) is refused
        parts = A.partition(2, (np.arange(n) >= n // 2).astype(np.int32))
        P = parts[0].dsymv_init(0.0)
        cgp = ab.SolverCuda(P)
        try:
            cgp.solve_shifted(np.ones(P.c.nownedrows), [0.0, 0.1], maxits=3)
            out["partitioned_code"] = 0
        except ab.AcgError as e:
            out["partitioned_code"] = e.code
        cgp.free()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
