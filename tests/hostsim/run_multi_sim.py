"""TEST INFRASTRUCTURE ONLY: drive acgsolvercuda_solve_multi / acgsolvercuda_spmm_mode on the device
stand-in (tests/hostsim/libacgb200_hostsim_multi.so: the host-logic stand-in plus kernels_multi_sim.c) and compare every column with the oracle's classic CG
on that column alone.  Runs in its own process so that the binding loads the stand-in; prints one
JSON object.  Used by tests/test_hostsim_multi.py."""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

import numpy as np                                   # noqa: E402

import acg_b200.api as api                           # noqa: E402
api._LIBPATH = os.path.join(HERE, "libacgb200_hostsim_multi.so")      # before the first lib() call
import acg_b200 as ab                                # noqa: E402
from acg_b200 import matgen as mg                    # noqa: E402
from oracle import Oracle                            # noqa: E402


def case(name):
    return {"27pt": lambda: mg.stencil3d_27pt(9, 8, 10), "7pt": lambda: mg.laplace3d_7pt(11),
            "rmat": lambda: mg.rmat_spd(30000, 600000, seed=8)}[name]()


def inputs(n, run, seed):
    """B with column j scaled by scale**j (columns converge at different iterations under an absolute
    tolerance); X0 zero or random; optionally one column with b = x0 = 0 (r0 = 0: converged at r0 under
    an absolute tolerance)."""
    k = run["nrhs"]
    rng = np.random.default_rng(seed)
    B = rng.standard_normal((n, k))
    B *= run.get("scale", 1.0) ** np.arange(k)
    X = rng.standard_normal((n, k)) if run.get("x0") == "random" else np.zeros((n, k))
    if run.get("zero_col") is not None:
        B[:, run["zero_col"]] = 0.0
        X[:, run["zero_col"]] = 0.0
    return np.ascontiguousarray(B), np.ascontiguousarray(X)


def solve_run(O, csr, cg, n, run, seed):
    B, X0 = inputs(n, run, seed)
    X = X0.copy()
    code, cols = cg.solve_multi(B, X, maxits=run["maxits"], residualatol=run.get("atol", 0.0),
                                residualrtol=run.get("rtol", 0.0), warmup=run.get("warmup", 0))
    out = {"run": run, "code": int(code), "its": int(cg.c.niterations), "cols": [],
           "x_bitwise_x0": bool(np.array_equal(X.view(np.uint64), X0.view(np.uint64))),
           "launches": int(cg.info()["last_launches"]), "nsolves": int(cg.c.nsolves)}
    ref_codes = []
    sb = sr0 = sr = 0.0
    for j in range(run["nrhs"]):
        ref = O.cg(csr, B[:, j], x0=X0[:, j], maxits=run["maxits"], atol=run.get("atol", 0.0), rtol=run.get("rtol", 0.0))
        ref_codes.append(int(ref["status"]))
        scale = max(float(np.abs(ref["x"]).max()), 1e-300)
        c = cols[j]
        out["cols"].append({"its": c["niterations"], "ref_its": int(ref["niterations"]), "converged": c["converged"],
                            "ref_status": int(ref["status"]), "xerr": float(np.abs(X[:, j] - ref["x"]).max() / scale),
                            "rnrm2": c["rnrm2"], "ref_rnrm2": float(ref["rnrm2"]), "r0nrm2": c["r0nrm2"],
                            "ref_r0nrm2": float(ref["r0nrm2"]), "bnrm2": c["bnrm2"], "ref_bnrm2": float(ref["bnrm2"])})
        sb += c["bnrm2"] ** 2; sr0 += c["r0nrm2"] ** 2; sr += c["rnrm2"] ** 2
    out["ref_code"] = 39 if any(rc == 39 for rc in ref_codes) else 0
    out["ref_its"] = max(c["ref_its"] for c in out["cols"])
    out["frobenius_ok"] = bool(np.isclose(cg.c.bnrm2, np.sqrt(sb), rtol=1e-14) and np.isclose(cg.c.r0nrm2, np.sqrt(sr0), rtol=1e-14)
                               and np.isclose(cg.c.rnrm2, np.sqrt(sr), rtol=1e-14))
    return out


def main():
    spec = json.loads(sys.argv[1])
    for k, v in spec.get("options", {}).items():
        ab.set_option(k, v)
    O = Oracle()
    n, r, c, v = case(spec["matrix"])
    A = ab.SymCsrMatrix.init_real_double(n, r, c, v).dsymv_init(0.0)
    csr = (A.frowptr.copy(), A.fcolidx.copy(), A.fa.copy())
    cg = ab.SolverCuda(A)
    out = {"runs": []}
    for i, run in enumerate(spec.get("runs", [])):
        out["runs"].append(solve_run(O, csr, cg, n, run, 100 + i))
    if spec.get("spmm"):
        # every mode against the oracle's product, column by column (the stand-in poisons rows it misses)
        rng = np.random.default_rng(3)
        res = []
        for k in spec["spmm"]:
            X = rng.standard_normal((n, k)); B = rng.standard_normal((n, k))
            for mode in (0, 1, 2):
                Y, dots = cg.spmm_mode(mode, X, B if mode == 2 else None)
                want = np.stack([O.dsymv(csr, 1.0, X[:, j], 0.0, np.zeros(n)) for j in range(k)], axis=1)
                if mode == 2:
                    want = B - want
                wdots = np.zeros(k) if mode == 0 else np.array([float(X[:, j] @ want[:, j]) if mode == 1 else float(want[:, j] @ want[:, j])
                                                                 for j in range(k)])
                res.append({"k": k, "mode": mode, "nan": bool(np.isnan(Y).any()),
                            "yerr": float(np.abs(Y - want).max() / np.abs(want).max()),
                            "doterr": float(np.abs(dots - wdots).max() / max(np.abs(wdots).max(), 1e-300)) if mode else float(np.abs(dots).max())})
        out["spmm"] = res
    if spec.get("single_after"):
        # a single-vector classic solve on this solver (after the multi solves) against a fresh solver
        b = A.vector(); b.x[:] = np.random.default_rng(9).standard_normal(n)
        x1 = A.vector()
        cg.solvempi(b, x1, maxits=40, residualrtol=1e-8)
        its1, r1 = int(cg.c.niterations), float(cg.c.rnrm2)
        cg2 = ab.SolverCuda(A)
        x2 = A.vector()
        cg2.solvempi(b, x2, maxits=40, residualrtol=1e-8)
        out["single_after"] = {"same_x": bool(np.array_equal(x1.x, x2.x)), "its": [its1, int(cg2.c.niterations)],
                               "rnrm2": [r1, float(cg2.c.rnrm2)]}
        cg2.free()
    errs = {}
    for k in (0, 9):
        try:
            cg.solve_multi(np.zeros((n, k)), np.zeros((n, k)), maxits=3)
        except ab.AcgError as e:
            errs[f"nrhs{k}"] = e.code
    out["errors"] = errs
    out["nsolves"] = int(cg.c.nsolves)
    cg.free()
    if spec.get("partitioned"):
        # a part of a partitioned matrix (ghost rows) is refused
        parts = A.partition(2, (np.arange(n) >= n // 2).astype(np.int32))
        P = parts[0].dsymv_init(0.0)
        cgp = ab.SolverCuda(P)
        try:
            cgp.solve_multi(np.zeros((P.c.nownedrows, 2)), np.zeros((P.c.nownedrows, 2)), maxits=3)
        except ab.AcgError as e:
            out["partitioned_code"] = e.code
        cgp.free()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
