#!/usr/bin/env python
"""tools/bench_mixed.py -- mixed-precision CG with reliable updates on one GPU (acgsolvercuda_solve_mixed).

    python tools/bench_mixed.py --workloads 27pt-224,7pt-256 --steps 3 --warmup 1

Prints one JSON line with, per workload of bench.py (its matrix and b):

  loop        (a) tolerances off, ITERS iterations per step: mixed iterations/s against
              acgsolvercuda_solvempi (classic CG) and acgsolvercuda_solve_pipelined on the same solver,
              alternated, from the summed device-side solve windows (CUDA events inside the library)
  kernels     (b) ms per launch of each kernel of the mixed loop from torch.profiler over one tolerance-free
              solve, against the byte model (fp32 product: the fp64 product's model bytes less 8 per row;
              update_r 12 B/row; update_yp 20; the replacement 20 when active).  Launches of the gated fp64
              residual product and of the replacement are split into active and idle ones (below a tenth
              of an update_r launch): the idle ones are the cost of a gated launch with no reliable update
              due; the residual product's active launches include the set-up's and the final one
  to_tol      (c) from x0 = 0 to rtol 1e-8: iterations, reliable updates, device ms and the true residual
              ||b - A x|| / ||b|| (fp64 product) for the mixed solve, classic CG and pipelined CG

The card name and its power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench import WORKLOADS, build_local_matrix, peaks, rhs, rhs_name     # noqa: E402

RTOL = 1e-8


def card():
    """Name and power limit of GPU 0, read now."""
    import torch
    out = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,power.max_limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        lim, mx = (float(v) for v in q.stdout.strip().splitlines()[0].split(","))
        out["power_limit_w"], out["power_max_limit_w"] = lim, mx
    except Exception as e:                                   # noqa: BLE001
        out["power_limit_error"] = str(e)
    return out


def kernel_class(name):
    for k in ("mixed_update_r_kernel", "mixed_update_yp_kernel", "mixed_replace_kernel", "spmv_rows_f32_kernel"):
        if k in name:
            return k
    if "spmv_symdiag_kernel" in name and "float>" in name:
        return "spmv_symdiag_kernel<float>"
    if "spmv_" in name:
        return "fp64_residual_product"
    return None


def kernel_ms(cg, bv, xv, iters):
    """Per kernel of the mixed loop over one tolerance-free solve, from torch.profiler: mean ms per launch,
    split into active and idle launches for the gated ones."""
    from torch.profiler import ProfilerActivity, profile
    xv.x[:] = 0.0
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        cg.solve_mixed(bv, xv, maxits=iters)
    out = {}
    for e in prof.events():
        k = kernel_class(e.name)
        if k:
            out.setdefault(k, []).append(e.device_time * 1e-3)
    res = {}
    cut = 0.1 * float(np.mean(out["mixed_update_r_kernel"]))    # a tenth of a pass over two float vectors
    for k, v in out.items():
        v = np.array(v)
        act, idle = v[v >= cut], v[v < cut]
        res[k] = {"ms": float(v.mean()), "launches": len(v), "active_ms": float(act.mean()) if len(act) else None,
                  "active": len(act),
                  "idle_ms": float(idle.mean()) if len(idle) else None, "idle": len(idle)}
    return res


def timed(fn, bv, xv, iters, steps, warmup, info):
    for _ in range(warmup):
        xv.x[:] = 0.0
        fn(bv, xv, maxits=iters)
    ms = 0.0
    for _ in range(steps):
        xv.x[:] = 0.0
        assert fn(bv, xv, maxits=iters) == 0
        ms += info()["last_solve_ms"]
    return iters * steps / (ms * 1e-3)


def to_tol(cg, fn, bv, xv, b, n, maxits):
    xv.x[:] = 0.0
    fn(bv, xv, maxits=20)                                    # warm: modules, graph
    xv.x[:] = 0.0
    code = fn(bv, xv, maxits=maxits, residualrtol=RTOL)
    inf = cg.info()
    out = {"code": int(code), "iterations": int(cg.c.niterations), "device_ms": inf["last_solve_ms"],
           "rnrm2_relative": float(cg.c.rnrm2) / float(np.linalg.norm(b))}
    if fn == cg.solve_mixed:
        out["reliable_updates"] = int(inf["mixed_reliable_updates"])
    y, _ = cg.spmv(xv.x[:n].copy())
    out["true_residual_relative"] = float(np.linalg.norm(b - y)) / float(np.linalg.norm(b))
    return out


def bench_workload(args, name):
    import acg_b200 as ab
    w = WORKLOADS[name]
    A = build_local_matrix(w, "block", 0, 1)
    n = int(A.c.nownedrows)
    b = np.ascontiguousarray(rhs(w, np.arange(n)))
    cg = ab.SolverCuda(A)
    res = {"workload": name, "n": n, "nnz": int(A.c.fnpnzs + A.c.onpnzs), "b": rhs_name(w)}
    try:
        bv, xv = A.vector(), A.vector()
        bv.x[:] = b
        its = {}
        # alternate the three solvers so that all see the same clocks
        for rep in range(2):
            for kind, fn in (("classic", cg.solvempi), ("pipelined", cg.solve_pipelined), ("mixed", cg.solve_mixed)):
                v = timed(fn, bv, xv, args.iters, args.steps, args.warmup if rep == 0 else 0, cg.info)
                its.setdefault(kind, []).append(v)
        inf = cg.info()
        prod = int(inf["spmv_min_bytes"])
        res["loop"] = {f"{k}_iterations_per_s": v for k, v in its.items()}
        mx = float(np.mean(its["mixed"]))
        res["loop"]["mixed_over_classic"] = mx / float(np.mean(its["classic"]))
        res["loop"]["mixed_over_pipelined"] = mx / float(np.mean(its["pipelined"]))
        res["loop"]["model_bytes_mixed_iteration"] = prod - 8 * n + 32 * n
        res["loop"]["model_bytes_classic_iteration"] = prod + 64 * n
        ks = kernel_ms(cg, bv, xv, args.iters)
        model = {"spmv_symdiag_kernel<float>": prod - 8 * n, "mixed_update_r_kernel": 12 * n,
                 "mixed_update_yp_kernel": 20 * n, "mixed_replace_kernel": 20 * n, "fp64_residual_product": prod}
        for k, v in ks.items():
            if k in model and v["active_ms"]:
                v["model_bytes"] = model[k]
                v["achieved_gbs_active"] = model[k] / (v["active_ms"] * 1e-3) / 1e9
        res["kernels"] = ks
        res["to_tol"] = {kind: to_tol(cg, fn, bv, xv, b, n, args.maxits)
                         for kind, fn in (("mixed", cg.solve_mixed), ("classic", cg.solvempi),
                                          ("pipelined", cg.solve_pipelined))}
        fastest = min(("classic", "pipelined"), key=lambda k: res["to_tol"][k]["device_ms"])
        res["to_tol"]["faster_fp64"] = fastest
        res["to_tol"]["speedup_vs_faster_fp64"] = res["to_tol"][fastest]["device_ms"] / res["to_tol"]["mixed"]["device_ms"]
        bv.free(); xv.free()
    finally:
        cg.free()
        A.free()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--workloads", default="27pt-224,7pt-256")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--iters", type=int, default=100, help="iterations per step with tolerances off")
    ap.add_argument("--maxits", type=int, default=20000, help="iteration cap of the solves to rtol 1e-8")
    args = ap.parse_args()
    names = [s for s in args.workloads.split(",") if s]
    if any(w not in WORKLOADS or WORKLOADS[w]["kind"] == "rmat" for w in names):
        ap.error(f"--workloads: stencil workloads of bench.py only ({sorted(k for k, v in WORKLOADS.items() if v['kind'] != 'rmat')})")
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_mixed.py: no CUDA device (the solver has no CPU path)")
    peak, peak_src = peaks()
    line = {"metric": "mixed-precision CG with reliable updates on one GPU (acgsolvercuda_solve_mixed)",
            "card": card(), "hbm_peak_gbs": peak, "peak_source": peak_src, "iters_per_step": args.iters,
            "steps": args.steps, "warmup": args.warmup, "rtol": RTOL,
            "workloads": [bench_workload(args, name) for name in names]}
    print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
