#!/usr/bin/env python
"""tools/bench_chebyshev.py -- Chebyshev-preconditioned CG on one GPU (acgsolvercuda_solve_chebyshev).

    python tools/bench_chebyshev.py --workloads 27pt-224,7pt-256,rmat-2M --degrees 0,1,2,4,8

Prints one JSON line with, per workload of bench.py (its matrix; a seeded random b on R-MAT, where b = 1 is
an eigenvector of A and CG stops after one iteration):

  to_tol      from x0 = 0 to rtol 1e-8, for acgsolvercuda_solvempi (classic CG) and each degree with the
              estimated interval: device-window ms (CUDA events inside the library), iterations, products
              (the set-up's and the estimate's included), the estimate's steps and interval, the true residual
              ||b - A x|| / ||b|| and x against solvempi's (max |x - x_cg| / max |x_cg|); every solve is run
              twice, alternated with the others, and both times are kept
  kernels     a separate run under torch.profiler (degree 4, tolerances off): ms per launch of each kernel
              of the loop, and GB/s of the inner step against its byte model (fused: per covered row the
              stored diagonals' bytes plus 8 for the gathered d_{j-1}, plus 56 for the step's vectors, 48 for
              the last step of an application; unfused: the plan's product and 64 / 56 per row for the
              elementwise step)

The card name and its power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench import WORKLOADS, build_local_matrix, peaks, rhs, rhs_name     # noqa: E402
from bench_mixed import card                                               # noqa: E402

RTOL = 1e-8


def kernel_class(name):
    for k in ("spmv_symdiag_cheb_kernel", "cheb_step_kernel", "cheb_rx_kernel", "cheb_p_kernel"):
        if k in name:
            return k
    if "spmv_" in name:
        return "product"
    return None


def kernel_ms(cg, bv, xv, degree, iters):
    from torch.profiler import ProfilerActivity, profile
    xv.x[:] = 0.0
    cg.solve_chebyshev(bv, xv, degree=degree, maxits=iters)           # warm: modules, graph, the same interval
    lo, hi = cg.info()["cheb_lmin"], cg.info()["cheb_lmax"]
    xv.x[:] = 0.0
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        cg.solve_chebyshev(bv, xv, degree=degree, lmin=lo, lmax=hi, maxits=iters)
    out = {}
    for e in prof.events():
        k = kernel_class(e.name)
        if k:
            out.setdefault(k, []).append(e.device_time * 1e-3)
    return {k: {"ms": float(np.mean(v)), "launches": len(v)} for k, v in out.items()}


def solve(cg, fn, bv, xv, n, b, **kw):
    g0 = int(cg.c.ngemv)
    xv.x[:] = 0.0
    code = fn(bv, xv, residualrtol=RTOL, **kw)
    inf = cg.info()
    x = xv.x[:n].copy()
    y, _ = cg.spmv(x)
    out = {"code": int(code), "iterations": int(cg.c.niterations), "products": int(cg.c.ngemv) - g0,
           "device_ms": [inf["last_solve_ms"]],
           "true_residual_relative": float(np.linalg.norm(b - y)) / float(np.linalg.norm(b))}
    if fn == cg.solve_chebyshev:
        out.update(est_steps=int(inf["cheb_est_iterations"]), interval=[inf["cheb_lmin"], inf["cheb_lmax"]],
                   breakdown=int(inf["cheb_breakdown"]))
    return out, x


def bench_workload(args, name, degrees):
    import acg_b200 as ab
    w = WORKLOADS[name]
    A = build_local_matrix(w, "block", 0, 1)
    n = int(A.c.nownedrows)
    if w["kind"] == "rmat":
        b, bname = np.random.default_rng(7).standard_normal(n), "standard normal, seed 7"
    else:
        b, bname = np.ascontiguousarray(rhs(w, np.arange(n))), rhs_name(w)
    cg = ab.SolverCuda(A)
    inf = cg.info()
    res = {"workload": name, "n": n, "nnz": int(A.c.fnpnzs + A.c.onpnzs), "b": bname,
           "plan": {k: inf[k] for k in ("spmv_symdiag_diagonals", "spmv_symdiag_codes", "spmv_slice_rows",
                                        "spmv_ntiles", "spmv_merge_tiles", "spmv_nlong")}}
    try:
        bv, xv = A.vector(), A.vector()
        bv.x[:] = b
        runs = [("solvempi", cg.solvempi, {})] + [(f"degree{d}", cg.solve_chebyshev, {"degree": d}) for d in degrees]
        for _, fn, kw in runs:                                      # warm: modules, graphs
            xv.x[:] = 0.0
            fn(bv, xv, maxits=20, **kw)
        to_tol, xs = {}, {}
        for rep in range(2):
            for key, fn, kw in runs:
                out, x = solve(cg, fn, bv, xv, n, b, maxits=args.maxits, **kw)
                if rep == 0:
                    to_tol[key], xs[key] = out, x
                else:
                    to_tol[key]["device_ms"] += out["device_ms"]
        xc = xs["solvempi"]
        for key in to_tol:
            to_tol[key]["x_vs_solvempi"] = float(np.abs(xs[key] - xc).max() / np.abs(xc).max())
            to_tol[key]["speedup_vs_solvempi"] = min(to_tol["solvempi"]["device_ms"]) / min(to_tol[key]["device_ms"])
        res["to_tol"] = to_tol
        ks = kernel_ms(cg, bv, xv, args.kdegree, args.iters)
        elem = 1 if inf["spmv_symdiag_codes"] > 0 else 8
        rows = inf["spmv_slice_rows"]
        mean_step = (56 * (args.kdegree - 1) + 48) / args.kdegree
        if "spmv_symdiag_cheb_kernel" in ks:
            v = ks["spmv_symdiag_cheb_kernel"]
            v["model_bytes"] = rows * (elem * inf["spmv_symdiag_diagonals"] + 8 + mean_step) + (n - rows) * (8 + mean_step)
            v["achieved_gbs"] = v["model_bytes"] / (v["ms"] * 1e-3) / 1e9
        if "cheb_step_kernel" in ks:
            v = ks["cheb_step_kernel"]
            v["model_bytes"] = n * (mean_step + 8)
            v["achieved_gbs"] = v["model_bytes"] / (v["ms"] * 1e-3) / 1e9
        for k, m in (("cheb_rx_kernel", 80), ("cheb_p_kernel", 24)):
            if k in ks:
                ks[k]["model_bytes"] = m * n
                ks[k]["achieved_gbs"] = m * n / (ks[k]["ms"] * 1e-3) / 1e9
        res["kernels"] = {"degree": args.kdegree, "iterations": args.iters, "per_kernel": ks}
        bv.free(); xv.free()
    finally:
        cg.free()
        A.free()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--workloads", default="27pt-224,7pt-256,rmat-2M")
    ap.add_argument("--degrees", default="0,1,2,4,8")
    ap.add_argument("--maxits", type=int, default=20000, help="iteration cap of the solves to rtol 1e-8")
    ap.add_argument("--iters", type=int, default=50, help="iterations of the profiled solve")
    ap.add_argument("--kdegree", type=int, default=4, help="degree of the profiled solve")
    args = ap.parse_args()
    names = [s for s in args.workloads.split(",") if s]
    if any(w not in WORKLOADS for w in names):
        ap.error(f"--workloads: workloads of bench.py ({sorted(WORKLOADS)})")
    degrees = [int(d) for d in args.degrees.split(",") if d]
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_chebyshev.py: no CUDA device (the solver has no CPU path)")
    peak, peak_src = peaks()
    line = {"metric": "Chebyshev-preconditioned CG on one GPU (acgsolvercuda_solve_chebyshev)", "card": card(),
            "hbm_peak_gbs": peak, "peak_source": peak_src, "rtol": RTOL, "degrees": degrees,
            "workloads": [bench_workload(args, name, degrees) for name in names]}
    print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
