"""TEST INFRASTRUCTURE ONLY: drive acgsolvercuda_solve_mixed on the device stand-in
(tests/hostsim/libacgb200_hostsim_mixed.so: the host-logic stand-in plus the multi-vector, shifted-systems,
MINRES and mixed-precision kernel stand-ins) and compare every solve with the restatement of
tests/mixedref.py on the matrix assembled.  Runs in its own process so that the binding loads the
stand-in; prints one JSON object.  Used by tests/test_hostsim_mixed.py."""
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
api._LIBPATH = os.path.join(HERE, "libacgb200_hostsim_mixed.so")    # before the first lib() call
import acg_b200 as ab                                # noqa: E402
from acg_b200 import matgen as mg                    # noqa: E402
from exactref import rows_exact                      # noqa: E402
from mixedref import mixed, threshold              # noqa: E402

DIAG = [3.0, 2.0, 0.5, 7.0, 4.0, 1.0, 0.25, 9.0, 0.0, 2.5, 1.5]      # entry 8: a zero row ((p, A p) = 0)


def case(name):
    if name == "diag":
        n = len(DIAG)
        d = np.arange(n, dtype=np.int32)
        return n, d, d.copy(), np.array(DIAG)
    return {"27pt": lambda: mg.stencil3d_27pt(9, 8, 10), "7pt": lambda: mg.laplace3d_7pt(11)}[name]()


def csr_of(A):
    n = A.c.nownedrows
    rp = A.frowptr[:n + 1].copy()
    ci = A.fcolidx[:rp[n]].copy()
    a = A.fa[:rp[n]].copy()
    return (rp, ci, a), sp.csr_matrix((a, ci - A.c.rowidxbase, rp), shape=(n, n))


def solve_run(cg, A, arrays, M, n, run, seed):
    rng = np.random.default_rng(seed)
    if "unit" in run:
        b = np.zeros(n); b[run["unit"]] = 1.5
    else:
        b = rng.standard_normal(n) * run.get("bscale", 1.0)
    if run.get("bzero"):
        b[:] = 0.0
    x0 = rng.standard_normal(n) if run.get("x0") else np.zeros(n)
    atol, rtol = run.get("atol", 0.0), run.get("rtol", 0.0)
    bv = A.vector(); bv.x[:] = b
    xv = A.vector(); xv.x[:] = x0
    code = cg.solve_mixed(bv, xv, maxits=run["maxits"], residualatol=atol, residualrtol=rtol,
                          warmup=run.get("warmup", 0))
    x = xv.x[:n].copy()
    ref = mixed(M, b, x0=x0, maxits=run["maxits"], atol=atol, rtol=rtol)
    scale = max(float(np.abs(ref["x"]).max()), 1e-300)
    rtrue, _, _ = rows_exact(*arrays, x, b)
    return {"run": run, "code": int(code), "ref_code": int(ref["status"]), "its": int(cg.c.niterations),
            "ref_its": int(ref["niterations"]), "ref_stop": ref["stop"],
            "updates": int(cg.info()["mixed_reliable_updates"]), "ref_updates": int(ref["nupdates"]),
            "xerr": float(np.abs(x - ref["x"]).max() / scale), "x_is_x0": bool(np.array_equal(x, x0)),
            "rnrm2": float(cg.c.rnrm2), "ref_rnrm2": float(ref["rnrm2"]), "r0nrm2": float(cg.c.r0nrm2),
            "ref_r0nrm2": float(ref["r0nrm2"]), "bnrm2": float(cg.c.bnrm2), "ref_bnrm2": float(ref["bnrm2"]),
            "true_rnrm2": float(np.linalg.norm(rtrue)), "tol": threshold(atol, rtol, float(ref["r0nrm2"])),
            "launches": int(cg.info()["last_launches"]), "nsolves": int(cg.c.nsolves),
            "ntotaliterations": int(cg.c.ntotaliterations), "report_lines": len(cg.report().splitlines())}


def alternate(A, n):
    """solvempi, solve_multi (two columns), solve_shifted (shifts 0 and 0.5), solve_minres and solve_mixed in
    turn on one solver, with the reliable updates info() reports after each; then solvempi on it against one
    on a fresh solver, bitwise."""
    cg = ab.SolverCuda(A)
    rng = np.random.default_rng(5)
    b = rng.standard_normal(n)
    bv = A.vector(); bv.x[:] = b
    B = np.ascontiguousarray(np.stack([b, rng.standard_normal(n)], axis=1))
    out = {"steps": []}
    for kind in ("mixed", "single", "multi", "minres", "mixed", "shifted", "minres", "single", "mixed", "multi",
                 "shifted", "mixed"):
        if kind == "multi":
            X = np.zeros((n, 2))
            code, st = cg.solve_multi(B, X, maxits=80, residualrtol=1e-8)
            its, xs = [s["niterations"] for s in st], X.ravel()
        elif kind == "shifted":
            code, X, st = cg.solve_shifted(b, [0.0, 0.5], maxits=80, residualrtol=1e-8)
            its, xs = [s["niterations"] for s in st], X.ravel()
        else:
            x = A.vector()
            fn = {"mixed": cg.solve_mixed, "minres": cg.solve_minres, "single": cg.solvempi}[kind]
            code = fn(bv, x, maxits=80, residualrtol=1e-8)
            its, xs = [int(cg.c.niterations)], x.x[:n].copy()
        out["steps"].append({"kind": kind, "code": int(code), "its": its, "x": xs.tolist(),
                             "updates": int(cg.info()["mixed_reliable_updates"])})
    x1 = A.vector()
    cg.solvempi(bv, x1, maxits=80, residualrtol=1e-8)
    its1, r1 = int(cg.c.niterations), float(cg.c.rnrm2)
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
    n, r, c, v = case(spec["matrix"])
    A = ab.SymCsrMatrix.init_real_double(n, r, c, v).dsymv_init(0.0)
    arrays, M = csr_of(A)
    cg = ab.SolverCuda(A)
    out = {"runs": [], "n": n}
    for i, run in enumerate(spec.get("runs", [])):
        out["runs"].append(solve_run(cg, A, arrays, M, n, run, 100 + i))
    if spec.get("errors"):
        bv = A.vector(); xv = A.vector()
        try:
            cg.solve_mixed(bv, xv, maxits=-1)
            out["negative_maxits"] = 0
        except ab.AcgError as e:
            out["negative_maxits"] = e.code
    cg.free()
    if spec.get("alternate"):
        out["alternate"] = alternate(A, n)
    if spec.get("partitioned"):
        parts = A.partition(2, (np.arange(n) >= n // 2).astype(np.int32))
        P = parts[0].dsymv_init(0.0)
        cgp = ab.SolverCuda(P)
        try:
            cgp.solve_mixed(P.vector(), P.vector(), maxits=3)
            out["partitioned_code"] = 0
        except ab.AcgError as e:
            out["partitioned_code"] = e.code
        cgp.free()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
