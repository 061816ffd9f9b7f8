"""A/B of solver variants in ONE process per GPU (development tool, GPU box only).

    python tools/ab.py --workload 27pt-224 --variants base,noslices,s7,pdl ...
    python -m torch.distributed.run --nproc-per-node N ... tools/ab.py --variants ...

bench.py pays matrix generation + full-storage expansion (tens of seconds at C3) for
every line; here the rank's matrix is built once and every variant only re-creates the
solver (option set -> acgsolvercuda_init -> steps -> free).  One JSON object per
variant goes to OUT/ab_<tag>_n<ranks>.jsonl and a one-line summary to stdout.  The x of
every variant is compared with the first variant's (same solver kind) -- a cheap
cross-variant parity check at full size.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np          # noqa: E402

DEFAULTS = dict(profile=0, spmv_lanes=0, spmv_nnz_cap=0, spmv_rows_cap=0, spmv_stages=0, spmv_threads=0,
                spmv_unroll=0, spmv_max_ctas=0, graph=1, redstream=1, p2p=1, p2p_fuse=1, blas1_ctas=0, pdl=0,
                spmv_medium=0, spmv_merge=-1, merge_items=0, merge_threads=0, merge_stages=0, merge_max_ctas=0, spmv_slices=1, slice_ub=0, slice_threads=0, slice_max_ctas=0,
                spmv_symdiag=1, symdiag_evict_first=0, symdiag_codes=1, pcg_fused=1, pcg_evict_first=1,
                pcg_group=16)

VARIANTS = {
    "base": {},
    "noslices": {"spmv_slices": 0},
    "oldgrid": {"blas1_ctas": 4},
    "pdl": {"pdl": 1},
    "nograph": {"graph": 0},
    "med128": {"spmv_medium": 128},
    "med256": {"spmv_medium": 256},
    "med64": {"spmv_medium": 64},
    "med32": {"spmv_medium": 32},
    "nccl": {"p2p": 0},
    "nccl_graph": {"p2p": 0, "graph": 2},
    "unfused": {"p2p_fuse": 0},
    # slice kernel shapes: s<ub>[_t<threads>][_c<max ctas>]  (the prefetching / register-capped shapes were
    # dropped after measurement)
    "s9": {"slice_ub": 9}, "s8": {"slice_ub": 8}, "s7": {"slice_ub": 7}, "s5": {"slice_ub": 5},
    "s9_t256": {"slice_ub": 9, "slice_threads": 256}, "s7_t256": {"slice_ub": 7, "slice_threads": 256},
    "s9_c8": {"slice_ub": 9, "slice_max_ctas": 8},
    # mirrored diagonals (option spmv_symdiag): off (the slice kernel), their values evict-first in L2, and
    # resident CTAs per SM, which sets how far the grid-stride front runs ahead of the mirror reads
    "nosymdiag": {"spmv_symdiag": 0},
    "sd_ef": {"symdiag_evict_first": 1},
    "sd_c4": {"slice_max_ctas": 4}, "sd_c8": {"slice_max_ctas": 8},
    # pipelined CG: the two-kernel iteration instead of the fused one, and the fused kernel's vector streams
    # evict-normal in L2
    "nofuse": {"pcg_fused": 0}, "fuse_en": {"pcg_evict_first": 0},
    # the mirrored diagonals as fp64 values even where one-byte codes into a value table would do
    "nocodes": {"symdiag_codes": 0},
    # the fused pipelined-CG iteration's group: p and x updated once per 2, 4, 8 or 16 iterations
    "g2": {"pcg_group": 2}, "g4": {"pcg_group": 4}, "g8": {"pcg_group": 8}, "g16": {"pcg_group": 16},
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="27pt-224")
    ap.add_argument("--variants", default="base")
    ap.add_argument("--solvers", default="pipelined")
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--partition", default="block")
    ap.add_argument("--tag", default=None)
    ap.add_argument("--out", default=".", help="directory of the JSON lines")
    ap.add_argument("--opt", action="append", default=[], help="extra variant NAME:key=val,key=val")
    args = ap.parse_args()

    import torch
    import bench
    import acg_b200 as ab
    from acg_b200 import dist as abdist
    w = bench.WORKLOADS[args.workload]
    rank, world, local = abdist.init_process(backend="gloo")
    import torch.distributed as dist
    comm = abdist.nccl_comm(rank, world)
    t0 = time.time()
    A = bench.build_local_matrix(w, args.partition, rank, world)
    nown = A.c.nownedrows
    nnz_local = int(A.c.fnpnzs + A.c.onpnzs)
    if rank == 0:
        print(f"# {args.workload} x{world}: local rows {nown} nnz {nnz_local} ghosts {A.c.nghostrows} "
              f"border {A.c.nborderrows} built in {time.time() - t0:.1f} s", flush=True)
    b = A.vector()
    gidx = A.nzrows[:nown] if len(A.nzrows) >= nown else np.arange(nown)
    b.x[:] = 0.0
    b.x[:nown] = bench.rhs(w, gidx)
    x = A.vector()
    b.pin(); x.pin()
    variants = dict(VARIANTS)
    for o in args.opt:
        name, kv = o.split(":")
        variants[name] = {k: int(v) for k, v in (t.split("=") for t in kv.split(","))}
    out = open(os.path.join(args.out, f"ab_{args.tag or args.workload}_n{world}.jsonl"), "a") if rank == 0 else None
    xref = {}
    for solver in args.solvers.split(","):
        for name in args.variants.split(","):
            opts = dict(DEFAULTS); opts.update(variants[name])
            for k, v in opts.items():
                try:
                    ab.set_option(k, v)
                except Exception:
                    if v:
                        raise
            t_init = time.time()
            try:
                cg = ab.SolverCuda(A, comm)
            except Exception as e:
                if rank == 0:
                    print(f"{solver}/{name}: init failed: {e}", flush=True)
                continue
            init_s = time.time() - t_init
            solve = cg.solve_pipelined if solver == "pipelined" else cg.solvempi

            def step():
                x.x[:] = 0.0
                if world > 1:
                    dist.barrier()
                torch.cuda.synchronize()
                t = time.perf_counter()
                code = solve(b, x, maxits=args.iters)
                t = time.perf_counter() - t
                assert code == 0 and cg.c.niterations == args.iters, (code, cg.c.niterations)
                return t
            try:
                for _ in range(args.warmup):
                    step()
                host = dev = 0.0
                launches = 0
                for _ in range(args.steps):
                    host += step()
                    inf = cg.info()
                    dev += inf["last_solve_ms"]; launches += inf["last_launches"]
                ab.set_option("profile", 1)
                spmv_ms = blas_ms = 0.0
                spmv_n = 0
                for _ in range(2):
                    step()
                    inf = cg.info()
                    spmv_ms += inf["last_spmv_ms"]; spmv_n += inf["last_spmv_count"]; blas_ms += inf["last_blas_ms"]
                ab.set_option("profile", 0)
            except Exception as e:
                if rank == 0:
                    print(f"{solver}/{name}: FAILED: {e!r}", flush=True)
                cg.free()
                continue
            tt = torch.tensor([dev, host], dtype=torch.float64)
            if world > 1:
                dist.all_reduce(tt, op=dist.ReduceOp.MAX)
            xs = x.x[:nown].copy()
            key = solver
            if key not in xref:
                xref[key] = xs
                xdiff = 0.0
            else:
                xdiff = float(np.abs(xs - xref[key]).max() / max(np.abs(xref[key]).max(), 1e-300))
            inf = cg.info()
            rec = dict(workload=args.workload, n_gpus=world, solver=solver, variant=name, options=variants[name],
                       its_per_s=args.steps * args.iters / (float(tt[0]) * 1e-3),
                       e2e_its_per_s=args.steps * args.iters / float(tt[1]),
                       ms_per_iter=float(tt[0]) / (args.steps * args.iters),
                       spmv_ms=spmv_ms / max(spmv_n, 1), update_ms_per_iter=blas_ms / (2 * args.iters),
                       launches_per_step=launches / args.steps, resid=cg.c.rnrm2 / cg.c.r0nrm2,
                       max_rel_x_diff_vs_first=xdiff, ntiles=inf["spmv_ntiles"], slices=inf["spmv_slices"],
                       slice_rows=inf["spmv_slice_rows"], slice_ub=inf["spmv_slice_ub"], slice_grid=inf["spmv_slice_grid"],
                       nlong=inf["spmv_nlong"], nmedium=inf["spmv_nmedium"], init_s=init_s,
                       spmv_min_bytes=inf["spmv_min_bytes"], nnz_local=nnz_local, nown=nown,
                       spmv_gbs_min=inf["spmv_min_bytes"] / max(spmv_ms / max(spmv_n, 1), 1e-9) / 1e6)
            if rank == 0:
                out.write(json.dumps(rec) + "\n"); out.flush()
                print(f"{solver}/{name}: {rec['its_per_s']:.1f} it/s (e2e {rec['e2e_its_per_s']:.1f}) ms/iter {rec['ms_per_iter']:.4f} "
                      f"spmv {rec['spmv_ms']:.4f} ms ({rec['spmv_gbs_min']:.0f} GB/s min-bytes) upd {rec['update_ms_per_iter']:.4f} "
                      f"launches/step {rec['launches_per_step']:.0f} resid {rec['resid']:.3e} xdiff {xdiff:.2e} "
                      f"slices {rec['slices']} (ub {rec['slice_ub']} grid {rec['slice_grid']}) tiles {rec['ntiles']} init {init_s:.1f} s",
                      flush=True)
            cg.free()
    for k, v in DEFAULTS.items():
        try:
            ab.set_option(k, v)
        except Exception:
            pass
    b.free(); x.free()
    comm.destroy()
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
