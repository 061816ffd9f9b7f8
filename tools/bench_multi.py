#!/usr/bin/env python
"""tools/bench_multi.py -- several right-hand sides on one GPU (acgsolvercuda_solve_multi).

    python tools/bench_multi.py --workload 27pt-224 --nrhs 4 --steps 3 --warmup 1

K right-hand sides of one workload matrix of bench.py (column 0 bench.py's b, the others seeded normal),
X0 = 0, classic CG per column, ITERS iterations per step with tolerances off.  Prints one JSON line:

  value     per-vector iterations/s: K x ITERS x steps over the summed device-side solve windows
            (CUDA events inside the library, as bench.py's value)
  roofline  the multi-vector product (spmm_slices_kernel + spmm_rows_kernel) per application, timed
            with CUDA events in the library's profile mode, and its bytes from the byte model below
  parity    every column against acgsolvercuda_solvempi on that column alone (same solver): iteration
            counts and the largest relative differences of ||r|| and x

The matrix and right-hand side come from bench.py (imported, unchanged).
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import WORKLOADS, build_local_matrix, peaks, rhs, rhs_name     # noqa: E402


def spmm_bytes(info, n, nnz, k, mode):
    """Bytes one multi-vector product must move: the slice-major values of the pattern slices, values +
    column indices (12 B per nonzero) and a row pointer (4 B per row) for every other row, x and y (8 B
    each per row and column), and b in mode 2 (r = b - A x)."""
    srows, snnz = info["spmv_slice_rows"], info["spmv_slice_nnz"]
    return info["spmv_slice_value_bytes"] + 12 * (nnz - snnz) + 4 * (n - srows) + k * 16 * n + (8 * k * n if mode == 2 else 0)


def bench_multi(args, w, A, cg, nnz):
    """Classic CG on K right-hand sides at once (acgsolvercuda_solve_multi), one GPU; prints the JSON line."""
    import acg_b200 as ab
    k, iters = args.nrhs, args.iters
    n = int(A.c.nownedrows)
    rng = np.random.default_rng(2024)
    B = np.ascontiguousarray(rng.standard_normal((n, k)))         # K seeded right-hand sides
    B[:, 0] = rhs(w, np.arange(n))
    X = np.zeros((n, k))

    def step():
        X[:] = 0.0
        code, cols = cg.solve_multi(B, X, maxits=iters)
        assert code == 0 and cg.c.niterations == iters and all(c["niterations"] == iters for c in cols)
        return cols

    for _ in range(max(args.warmup, 0)):
        step()
    dev_ms = 0.0
    for _ in range(args.steps):
        step()
        dev_ms += cg.info()["last_solve_ms"]
    ab.set_option("profile", 1)
    spmv_ms = 0.0
    spmv_n = 0
    blas_ms = 0.0
    for _ in range(args.steps):
        cols = step()
        inf = cg.info()
        spmv_ms += inf["last_spmv_ms"]; spmv_n += inf["last_spmv_count"]; blas_ms += inf["last_blas_ms"]
    ab.set_option("profile", 0)
    info = cg.info()
    X_multi = X.copy()
    # parity: every column against the single-vector classic solver on that column alone
    b, x = A.vector(), A.vector()
    its_equal, dr, dx = True, 0.0, 0.0
    for j in range(k):
        b.x[:] = B[:, j]
        x.x[:] = 0.0
        cg.solvempi(b, x, maxits=iters)
        its_equal &= cg.c.niterations == iters
        dr = max(dr, abs(cols[j]["rnrm2"] - cg.c.rnrm2) / cg.c.rnrm2)
        dx = max(dx, float(np.abs(X_multi[:, j] - x.x[:n]).max() / np.abs(x.x[:n]).max()))
    b.free(); x.free()
    peak, peak_src = peaks()
    b1, b2 = spmm_bytes(info, n, nnz, block_width(k), 1), spmm_bytes(info, n, nnz, block_width(k), 2)   # padding columns move too
    nloop = spmv_n - args.steps                                   # one r0 = b - A x0 product per solve, the rest in the loop
    t_app = spmv_ms / max(spmv_n, 1) * 1e-3
    bytes_mean = (nloop * b1 + args.steps * b2) / max(spmv_n, 1)
    what = f"{w['kind']} stencil {w['N']}^3" if w["kind"] != "rmat" else f"R-MAT power-law SPD, n={w['N']}"
    line = {
        "metric": "per-vector CG iterations/sec, several right-hand sides (classic CG per column)",
        "value": k * iters * args.steps / (dev_ms * 1e-3), "unit": "vector-iterations/s",
        "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "ms_per_step": dev_ms / args.steps,
        "loop_iterations_per_s": iters * args.steps / (dev_ms * 1e-3),
        "higher_is_better": True, "dtype": "f64", "data": "synthetic",
        "config": {"workload": f"{what}, FP64, {k} right-hand sides (column 0 {rhs_name(w)}, the others seeded normal), "
                               f"X0=0, classic CG per column, {iters} iterations/step, tolerances off",
                   "n": n, "solver": "classic", "nrhs": k, "block_width": block_width(k), "iters_per_step": iters,
                   "entry_point": "acgsolvercuda_solve_multi"},
        "roofline": {"bound": "hbm", "kernel": " + ".join((["spmm_slices_kernel"] if info["spmv_slices"] > 0 else [])
                                                          + ["spmm_rows_kernel"]),
                     "ms_per_application": t_app * 1e3, "applications_timed": spmv_n,
                     "bytes_per_application": bytes_mean, "bytes_loop_application": b1, "bytes_r0_application": b2,
                     "achieved": bytes_mean / t_app / 1e9, "peak": peak, "peak_source": peak_src, "unit": "GB/s",
                     "frac": bytes_mean / t_app / 1e9 / peak, "ms_per_vector_application": t_app * 1e3 / k,
                     "update_ms_per_iteration": blas_ms / max(args.steps * iters, 1),
                     "note": "byte model of bench.py (spmm_bytes): slice values + 12 B/nonzero and 4 B/row outside the "
                             "slices + 16 B per row and column (x, y) + 8 B per row and column for b in the r0 product; "
                             "mean over the loop products (mode 1) and the r0 product of every solve (mode 2)"},
        "parity": {"what": "each column against acgsolvercuda_solvempi on that column alone, same solver",
                   "iterations_equal": bool(its_equal), "max_rel_rnrm2_diff": dr, "max_rel_x_diff": dx},
    }
    print(json.dumps(line), flush=True)


def block_width(k):
    """K of the multi-vector kernels: nrhs padded to 1, 2, 4 or 8 columns."""
    return 1 if k <= 1 else 2 if k <= 2 else 4 if k <= 4 else 8


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--workload", default="27pt-224", choices=sorted(WORKLOADS))
    ap.add_argument("--nrhs", type=int, required=True, help="right-hand sides, 1-8")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--iters", type=int, default=100, help="CG iterations per step")
    args = ap.parse_args()
    if not 1 <= args.nrhs <= 8:
        ap.error("--nrhs must be between 1 and 8")
    if args.steps < 1:
        ap.error("--steps must be at least 1")
    import torch
    import acg_b200 as ab
    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_multi.py: no CUDA device (the product has no CPU path)")
    w = WORKLOADS[args.workload]
    A = build_local_matrix(w, "block", 0, 1)
    cg = ab.SolverCuda(A)
    try:
        bench_multi(args, w, A, cg, int(A.c.fnpnzs + A.c.onpnzs))
    finally:
        cg.free()
        A.free()
    return 0


if __name__ == "__main__":
    sys.exit(main())
