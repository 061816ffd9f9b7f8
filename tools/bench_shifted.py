#!/usr/bin/env python
"""tools/bench_shifted.py -- shifted systems on one GPU (acgsolvercuda_solve_shifted, multi-shift CG).

    python tools/bench_shifted.py --workloads 27pt-224,7pt-256 --shifts 1,2,4,8 --steps 3 --warmup 1

(A + sigma_j I) x_j = b for S shifts of a workload matrix of bench.py (its b), x0 = 0, with the first S of
SIGMAS: 0, then a geometric spread with ratio sqrt(10) from 10^-2.5 to 10^0.5 (nested, so every S adds shifts
to the smaller sets).  Prints one JSON line with, per workload and S:

  loop       (a) tolerances off, ITERS iterations per step: loop iterations/s and per-system iterations/s
             (S x loop), from the summed device-side solve windows (CUDA events inside the library);
             the single-vector classic solver on the same matrix alongside
  to_rtol    (b) the device time to bring all S systems to rtol 1e-8 in one call, against the sum of S
             separate acgsolvercuda_solvempi solves on solvers built with dsymv_init(sigma_j) (made and
             freed one at a time, so at most one extra copy of the matrix exists)
  kernel     (c) cg_shift_update_kernel's ms per iteration (kernel durations from torch.profiler over one
             tolerance-free solve) against the byte model 24 B/row (seed r, p read, p written) + 32 B/row
             per shift (x_j, p_j read and written)
  parity     per shift: iterations against the standalone solve and the largest relative x difference

The card name and its power limit are read in the same run.  The matrix and b come from bench.py
(imported, unchanged).
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

from bench import WORKLOADS, build_local_matrix, peaks, rhs, rhs_name     # noqa: E402

SIGMAS = [0.0, 1.0, 0.1, 0.01, 10 ** -0.5, 10 ** -1.5, 10 ** 0.5, 10 ** -2.5]
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


def kernel_ms(cg, b, shifts, iters):
    """Mean duration of cg_shift_update_kernel over one tolerance-free solve, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        cg.solve_shifted(b, shifts, maxits=iters)
    durs = [e.device_time for e in prof.events() if "cg_shift_update_kernel" in e.name]
    return (float(np.mean(durs)) * 1e-3 if durs else None), len(durs)


def bench_workload(args, name, standalone_cache):
    import acg_b200 as ab
    from acg_b200 import dist as abdist
    w = WORKLOADS[name]
    A = build_local_matrix(w, "block", 0, 1)
    n = int(A.c.nownedrows)
    b = np.ascontiguousarray(rhs(w, np.arange(n)))
    cg = ab.SolverCuda(A)
    res = {"workload": name, "n": n, "nnz": int(A.c.fnpnzs + A.c.onpnzs), "b": rhs_name(w), "by_S": []}
    try:
        # the single-vector classic solver, tolerances off (the reference point of (a))
        bv, xv = A.vector(), A.vector()
        bv.x[:] = b
        for _ in range(args.warmup):
            cg.solvempi(bv, xv, maxits=args.iters)
        ms = 0.0
        for _ in range(args.steps):
            xv.x[:] = 0.0
            cg.solvempi(bv, xv, maxits=args.iters)
            ms += cg.info()["last_solve_ms"]
        res["classic_iterations_per_s"] = args.iters * args.steps / (ms * 1e-3)
        bv.free(); xv.free()
        for S in args.shifts:
            shifts = SIGMAS[:S]
            for _ in range(args.warmup):
                cg.solve_shifted(b, shifts, maxits=args.iters)
            ms = 0.0
            for _ in range(args.steps):
                code, X, cols = cg.solve_shifted(b, shifts, maxits=args.iters)
                assert code == 0 and cg.c.niterations == args.iters
                ms += cg.info()["last_solve_ms"]
            loop = args.iters * args.steps / (ms * 1e-3)
            kms, kcount = kernel_ms(cg, b, shifts, args.iters)
            model = n * (24 + 32 * S)
            # (b): all shifts to rtol in one call
            cg.solve_shifted(b, shifts, maxits=args.maxits, residualrtol=RTOL)      # warm
            code, X, cols = cg.solve_shifted(b, shifts, maxits=args.maxits, residualrtol=RTOL)
            t_all = cg.info()["last_solve_ms"]
            sep_ms, parity = 0.0, []
            for j, sigma in enumerate(shifts):
                key = (name, sigma)
                if key not in standalone_cache:
                    Aj = abdist.local_stencil_part(27 if w["kind"] == "27pt" else 7, w["N"], w["N"], w["N"], 0, 1, eps=sigma)
                    cgj = ab.SolverCuda(Aj)
                    bj, xj = Aj.vector(), Aj.vector()
                    bj.x[:] = b
                    cgj.solvempi(bj, xj, maxits=args.maxits, residualrtol=RTOL)        # warm
                    xj.x[:] = 0.0
                    cj = cgj.solvempi(bj, xj, maxits=args.maxits, residualrtol=RTOL)
                    standalone_cache[key] = (int(cj), int(cgj.c.niterations), cgj.info()["last_solve_ms"], xj.x[:n].copy())
                    bj.free(); xj.free(); cgj.free(); Aj.free()
                cj, its, tms, xs = standalone_cache[key]
                sep_ms += tms
                parity.append({"sigma": sigma, "iterations": cols[j]["niterations"], "standalone_iterations": its,
                               "iterations_equal": cols[j]["niterations"] == its, "code": int(code), "standalone_code": cj,
                               "max_rel_x_diff": float(np.abs(X[:, j] - xs).max() / np.abs(xs).max())})
            res["by_S"].append({
                "S": S, "shifts": shifts,
                "loop": {"loop_iterations_per_s": loop, "system_iterations_per_s": S * loop,
                         "ms_per_iteration": 1e3 / loop,
                         "vs_classic_system_iterations": S * loop / res["classic_iterations_per_s"]},
                "to_rtol": {"rtol": RTOL, "ms_all_shifts_one_call": t_all, "loop_iterations": int(cg.c.niterations),
                            "ms_sum_separate_solvempi": sep_ms, "speedup": sep_ms / t_all},
                "kernel": {"name": "cg_shift_update_kernel", "ms_per_iteration": kms, "launches_profiled": kcount,
                           "model_bytes": model, "achieved_gbs": (model / (kms * 1e-3) / 1e9) if kms else None},
                "parity": parity})
    finally:
        cg.free()
        A.free()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--workloads", default="27pt-224,7pt-256")
    ap.add_argument("--shifts", default="1,2,4,8", help="shift counts S to run, each 1-8")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--iters", type=int, default=100, help="CG iterations per step with tolerances off")
    ap.add_argument("--maxits", type=int, default=5000, help="iteration cap of the solves to rtol 1e-8")
    args = ap.parse_args()
    args.shifts = [int(s) for s in args.shifts.split(",")]
    if any(not 1 <= s <= 8 for s in args.shifts):
        ap.error("--shifts: every count must be between 1 and 8")
    names = args.workloads.split(",")
    if any(w not in WORKLOADS or WORKLOADS[w]["kind"] == "rmat" for w in names):
        ap.error(f"--workloads: stencil workloads of bench.py only ({sorted(k for k, v in WORKLOADS.items() if v['kind'] != 'rmat')})")
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_shifted.py: no CUDA device (the product has no CPU path)")
    peak, peak_src = peaks()
    line = {"metric": "multi-shift CG on one GPU (acgsolvercuda_solve_shifted)", "card": card(),
            "hbm_peak_gbs": peak, "peak_source": peak_src, "iters_per_step": args.iters, "steps": args.steps,
            "warmup": args.warmup, "dtype": "f64", "workloads": []}
    cache = {}
    for name in names:
        line["workloads"].append(bench_workload(args, name, cache))
        cache.clear()
    print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
