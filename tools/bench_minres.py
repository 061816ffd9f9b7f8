#!/usr/bin/env python
"""tools/bench_minres.py -- MINRES on one GPU (acgsolvercuda_solve_minres).

    python tools/bench_minres.py --workloads 27pt-224,7pt-256 --steps 3 --warmup 1

Prints one JSON line with:

  loop        (a) per workload of bench.py (its matrix and b), tolerances off, ITERS iterations per step:
              MINRES iterations/s against acgsolvercuda_solvempi (classic CG) on the same solver, from the
              summed device-side solve windows (CUDA events inside the library), and their ratio next to
              the byte model's (product + 64 B/row for classic CG, product + 96 B/row for MINRES)
  kernels     (b) ms per launch of the product, minres_lanczos_kernel and minres_update_kernel from
              torch.profiler over one tolerance-free solve, against their model bytes (product:
              acgb200_spmv_min_bytes; Lanczos 32 B/row; update 64 B/row)
  indefinite  (c) the 7-point stencil on 256^3 shifted by dsymv_init(-sigma), sigma halfway between two
              eigenvalues of its closed-form spectrum so that NNEG of them are negative: iterations, device
              ms and the true residual ||b - A x|| / ||b|| at rtol 1e-8, or the residual reached by maxits

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
from minresref import indefinite_shift, stencil_eigenvalues              # noqa: E402

RTOL = 1e-8
KERNELS = ("minres_lanczos_kernel", "minres_update_kernel", "spmv_")


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


def kernel_ms(cg, bv, xv, iters):
    """Mean duration per launch of the loop's kernels over one tolerance-free solve, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    xv.x[:] = 0.0
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        cg.solve_minres(bv, xv, maxits=iters)
    out = {}
    for e in prof.events():
        for k in KERNELS:
            if k in e.name:
                out.setdefault(k, []).append(e.device_time)
    return {k: {"ms": float(np.mean(v)) * 1e-3, "launches": len(v)} for k, v in out.items()}


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
        # alternate the two solvers so that both see the same clocks
        for rep in range(2):
            for kind, fn in (("classic", cg.solvempi), ("minres", cg.solve_minres)):
                v = timed(fn, bv, xv, args.iters, args.steps, args.warmup if rep == 0 else 0, cg.info)
                its.setdefault(kind, []).append(v)
        inf = cg.info()
        prod = int(inf["spmv_min_bytes"])
        model_classic, model_minres = prod + 64 * n, prod + 96 * n
        cl, mr = float(np.mean(its["classic"])), float(np.mean(its["minres"]))
        res["loop"] = {"classic_iterations_per_s": its["classic"], "minres_iterations_per_s": its["minres"],
                       "ratio_measured": mr / cl, "ratio_model": model_classic / model_minres,
                       "model_bytes_classic": model_classic, "model_bytes_minres": model_minres,
                       "minres_model_gbs": model_minres * mr / 1e9}
        ks = kernel_ms(cg, bv, xv, args.iters)
        model = {"spmv_": prod, "minres_lanczos_kernel": 32 * n, "minres_update_kernel": 64 * n}
        res["kernels"] = {k: dict(v, model_bytes=model[k], achieved_gbs=model[k] / (v["ms"] * 1e-3) / 1e9)
                          for k, v in ks.items()}
        bv.free(); xv.free()
    finally:
        cg.free()
        A.free()
    return res


def bench_indefinite(args):
    import acg_b200 as ab
    from acg_b200 import dist as abdist
    N = 256
    ev = stencil_eigenvalues(7, N, N, N)
    sigma = indefinite_shift(ev, args.nneg)
    nneg = int((ev < sigma).sum())
    A = abdist.local_stencil_part(7, N, N, N, 0, 1, eps=-sigma)
    n = int(A.c.nownedrows)
    w = WORKLOADS["7pt-256"]
    b = np.ascontiguousarray(rhs(w, np.arange(n)))
    cg = ab.SolverCuda(A)
    try:
        bv, xv = A.vector(), A.vector()
        bv.x[:] = b
        cg.solve_minres(bv, xv, maxits=20)                  # warm: modules, graph
        xv.x[:] = 0.0
        code = cg.solve_minres(bv, xv, maxits=args.maxits, residualrtol=RTOL)
        its, ms, phibar = int(cg.c.niterations), cg.info()["last_solve_ms"], float(cg.c.rnrm2)
        y, _ = cg.spmv(xv.x[:n].copy())
        true = float(np.linalg.norm(b - y))
        out = {"matrix": f"7pt-{N}^3 - sigma I", "n": n, "sigma": sigma, "negative_eigenvalues": nneg,
               "smallest_abs_eigenvalue": float(np.abs(ev - sigma).min()), "largest_eigenvalue": float(ev[-1] - sigma),
               "rtol": RTOL, "maxits": args.maxits, "code": int(code), "iterations": its, "device_ms": ms,
               "phibar_relative": phibar / float(np.linalg.norm(b)), "true_residual_relative": true / float(np.linalg.norm(b))}
        bv.free(); xv.free()
    finally:
        cg.free()
        A.free()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--workloads", default="27pt-224,7pt-256")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--iters", type=int, default=100, help="iterations per step with tolerances off")
    ap.add_argument("--nneg", type=int, default=4, help="negative eigenvalues of the indefinite workload")
    ap.add_argument("--maxits", type=int, default=20000, help="iteration cap of the indefinite solve")
    args = ap.parse_args()
    names = [s for s in args.workloads.split(",") if s]
    if any(w not in WORKLOADS or WORKLOADS[w]["kind"] == "rmat" for w in names):
        ap.error(f"--workloads: stencil workloads of bench.py only ({sorted(k for k, v in WORKLOADS.items() if v['kind'] != 'rmat')})")
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_minres.py: no CUDA device (the solver has no CPU path)")
    peak, peak_src = peaks()
    line = {"metric": "MINRES on one GPU (acgsolvercuda_solve_minres)", "card": card(), "hbm_peak_gbs": peak,
            "peak_source": peak_src, "iters_per_step": args.iters, "steps": args.steps, "warmup": args.warmup,
            "dtype": "f64", "workloads": [bench_workload(args, name) for name in names]}
    if args.nneg > 0:
        line["indefinite"] = bench_indefinite(args)
    print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
