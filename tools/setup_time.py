"""Set-up time of a solver with and without host-side full storage (GPU box only, development tool).

    python tools/setup_time.py --workload 27pt-224 [--refresh]

(a) the reference's route: acgsymcsrmatrix_dsymv_init on the host (threaded here), then
    acgsolvercuda_init uploads the expanded arrays;
(b) acgsolvercuda_init on the packed matrix: the packed triangle is uploaded and mirrored on the
    device (expand.cu).
Both solvers must produce bit-identical products (the arrays are byte-identical).
--refresh adds acgsolvercuda_update_values on each of the two solvers with the same matrix, next to the init that
built it: (b) from the packed triangle, (a) from the full storage.  Init and refresh both return after a
synchronise of the solver's stream, which ran all their device work; the card's name and power limit are
reported with the times."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np          # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="27pt-224")
    ap.add_argument("--refresh", action="store_true", help="also time acgsolvercuda_update_values")
    args = ap.parse_args()
    import bench
    import acg_b200 as ab
    w = bench.WORKLOADS[args.workload]
    N = w["N"]
    t0 = time.time()
    if w["kind"] == "rmat":
        mk = lambda: ab.SymCsrMatrix.rmat_spd(N, w["edges"], seed=42)                     # noqa: E731
    else:
        mk = lambda: ab.SymCsrMatrix.stencil_part(27 if w["kind"] == "27pt" else 7, N, N, N, 1, 1, 1, 0)    # noqa: E731
    A = mk()
    t_gen = time.time() - t0
    n = A.c.nprows
    x = np.random.default_rng(0).standard_normal(n)
    # CUDA context, module load and the first cudaMalloc are paid by a small solver first (both routes below
    # would otherwise differ by which one runs first)
    W = ab.SymCsrMatrix.stencil_part(27, 16, 16, 16, 1, 1, 1, 0)
    warm = ab.SolverCuda(W); warm.spmv(np.ones(W.c.nprows)); warm.free()
    refresh = {}
    t0 = time.time(); cg_b = ab.SolverCuda(A); t_b = time.time() - t0
    yb, _ = cg_b.spmv(x)
    inf_b = cg_b.info()
    if args.refresh:
        t0 = time.time(); cg_b.update_values(A); refresh["refresh_from_packed_s"] = time.time() - t0
        refresh["refresh_from_packed_products_bit_identical"] = bool(cg_b.spmv(x)[0].tobytes() == yb.tobytes())
    cg_b.free()
    t0 = time.time(); A.dsymv_init(0.0); t_host = time.time() - t0
    t0 = time.time(); cg_a = ab.SolverCuda(A); t_a = time.time() - t0
    ya, _ = cg_a.spmv(x)
    if args.refresh:
        t0 = time.time(); cg_a.update_values(A); refresh["refresh_from_full_storage_s"] = time.time() - t0
        refresh["refresh_from_full_storage_products_bit_identical"] = bool(cg_a.spmv(x)[0].tobytes() == ya.tobytes())
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True)
        refresh["gpu"] = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else None
    cg_a.free()
    t0 = time.time(); B = mk(); B.dsymv_init_cuda(0.0); t_cuda_back = time.time() - t0 - t_gen
    same = all(getattr(A, k).tobytes() == getattr(B, k).tobytes() for k in ("frowptr", "fcolidx", "fa"))
    print(json.dumps(dict(workload=args.workload, n=int(n), packed_nnz=int(A.c.pnzs) if hasattr(A.c, "pnzs") else None,
                          full_nnz=int(A.c.fnpnzs), generate_s=t_gen,
                          host_dsymv_init_s=t_host, init_with_full_storage_s=t_a, route_a_total_s=t_host + t_a,
                          init_from_packed_device_expansion_s=t_b,
                          dsymv_init_cuda_with_copy_back_s=t_cuda_back,
                          products_bit_identical=bool(ya.tobytes() == yb.tobytes()), arrays_byte_identical=bool(same),
                          slices=inf_b["spmv_slices"], threads=os.cpu_count(), **refresh)))


if __name__ == "__main__":
    main()
