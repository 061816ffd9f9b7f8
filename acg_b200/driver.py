"""Multi-GPU command-line solver on top of libacgb200 -- the part of
``cuda/acg-cuda.c`` that needs MPI in the reference (read, partition, scatter,
solve, report) done with one process per GPU under ``torch.distributed``:

    python -m torch.distributed.run --nproc-per-node 8 --master-addr 127.0.0.1 \\
        -m acg_b200.driver A.mtx --binary --solver acg-pipelined --partition metis

Differences from the reference driver's flow (cuda/acg-cuda.c:1297-1304 read on
root, :1486-1700 partition on root, :1782 scatter): every rank streams the
binary file and keeps its own rows (acgb200_mtx_read_part), so nobody holds the
matrix -- except for ``--partition metis``, where rank 0 reads it once to run
METIS (acgsymcsrmatrix_partition_rows) and broadcasts the row->part map.  The
options carry the reference's names; the solver report is the reference's
(acgsolvercuda_fwrite).  With one process this is a plain single-GPU run.
"""
from __future__ import annotations

import argparse
import os
import sys
import time

import numpy as np

SOLVERS = {"acg": "solvempi", "acg-pipelined": "solve_pipelined",
           "acg-device": "solve_device", "acg-device-pipelined": "solve_device_pipelined",
           "minres": "solve_minres", "mixed": "solve_mixed", "chebyshev": "solve_chebyshev"}
ONE_PROCESS = ("minres", "mixed", "chebyshev")


def parse_args(argv=None):
    ap = argparse.ArgumentParser(prog="acg_b200.driver", description=__doc__.split("\n\n")[0])
    ap.add_argument("A", help="symmetric Matrix Market file (matrix coordinate real symmetric)")
    ap.add_argument("--binary", action="store_true", help="aCG binary encoding (mtx2bin); required for more than one process")
    ap.add_argument("--solver", default="acg", choices=sorted(SOLVERS),
                    help="minres: MINRES for symmetric indefinite or singular A, e.g. with a negative --epsilon "
                         "(acgsolvercuda_solve_minres; one process only); mixed: CG with float vectors and "
                         "reliable updates to an fp64 tolerance (acgsolvercuda_solve_mixed; one process only); chebyshev: CG "
                         "preconditioned with a Chebyshev polynomial in D^-1 A of --degree "
                         "(acgsolvercuda_solve_chebyshev; one process only)")
    ap.add_argument("--max-iterations", type=int, default=100)
    ap.add_argument("--residual-atol", type=float, default=0.0)
    ap.add_argument("--residual-rtol", type=float, default=1e-9)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--epsilon", type=float, default=0.0, help="shift added to the diagonal (acgsymcsrmatrix_dsymv_init)")
    ap.add_argument("--partition", default="rows",
                    help="rows (contiguous blocks of equal row count), nnz (contiguous blocks of equal nonzero count; "
                         "rank 0 reads the matrix once), metis, or a Matrix Market vector file with 1-based part numbers "
                         "(mtxpartition output, as the reference's --partition=FILE)")
    ap.add_argument("--manufactured-solution", action="store_true",
                    help="random unit x*, b = A x*, report ||x - x*|| (cuda/acg-cuda.c:1969-1979, :2376-2385)")
    ap.add_argument("--nrhs", type=int, default=None,
                    help="solve K (1-8) seeded right-hand sides at once: classic CG per column, one pass over the matrix per "
                         "iteration for all of them (acgsolvercuda_solve_multi; one process only)")
    ap.add_argument("--shifts", default=None, metavar="S0,S1,...",
                    help="solve (A + s_j I) x_j = b for 1-8 comma-separated shifts s_j >= 0 at once from x0 = 0: one CG "
                         "on A drives every shifted system (acgsolvercuda_solve_shifted; one process, classic solver)")
    ap.add_argument("--degree", type=int, default=2,
                    help="--solver chebyshev: the polynomial's degree, 0-16 (0: Jacobi)")
    ap.add_argument("--interval", default=None, metavar="A,B",
                    help="--solver chebyshev: the interval [A, B] of D^-1 A's spectrum (default: B estimated from 10 "
                         "Jacobi-PCG steps, A = B/10)")
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--output-comm-matrix", metavar="PATH", help="write the halo send-count matrix (cuda/acg-cuda.c:1713-1775)")
    ap.add_argument("--output-solution", metavar="PATH", help="write x as a Matrix Market vector (text)")
    ap.add_argument("--dry-run", action="store_true", help="read, partition and report the decomposition; no solver, no GPU")
    ap.add_argument("-v", "--verbose", action="count", default=0)
    return ap.parse_args(argv)


def row_partition(args, n, rank, world):
    """Row -> part map, identical on every rank."""
    import torch.distributed as dist
    from . import dist as abdist, mtxio
    from .api import SymCsrMatrix
    if args.partition == "rows":
        return abdist.contiguous_partition(n, world)
    if args.partition in ("metis", "nnz"):
        box = [None]
        if rank == 0:
            whole = SymCsrMatrix.read_mtx(args.A, binary=True)
            box[0] = (whole.partition_rows(world, kway=False, seed=args.seed)[0] if args.partition == "metis"
                      else abdist.balanced_rows_partition(whole, world))
            whole.free()
        dist.broadcast_object_list(box, src=0)
        return np.ascontiguousarray(box[0], np.int32)
    rowparts = mtxio.read_rowparts(args.partition)
    if len(rowparts) != n:
        raise SystemExit(f"{args.partition}: expected {n} rows, found {len(rowparts)}")
    if rowparts.min() < 0 or rowparts.max() >= world:
        raise SystemExit(f"{args.partition}: part numbers must be 1..{world}")
    return rowparts


def local_rhs(args, A, n):
    """Owned entries of b (and of x* for a manufactured solution)."""
    no = A.c.nownedrows
    gidx = A.nzrows if len(A.nzrows) >= A.c.nprows else np.arange(A.c.nprows)
    if not args.manufactured_solution:
        return np.ones(no), None
    # the same global x* on every rank: random in [-1,1], normalised (cuda/acg-cuda.c:1969-1979)
    xs = np.random.default_rng(args.seed).uniform(-1.0, 1.0, n)
    xs /= np.linalg.norm(xs)
    xloc = xs[gidx]                                   # owned + ghost entries in local order
    import scipy.sparse as sp
    rp = A.frowptr[:no + 1]
    F = sp.csr_matrix((A.fa[:rp[no]], A.fcolidx[:rp[no]] - A.c.rowidxbase, rp), shape=(no, A.c.nprows))
    b = F @ xloc
    if A.c.onpnzs > 0:
        nb, off = A.c.nborderrows, A.c.borderrowoffset
        orp = A.orowptr[:nb + 1]
        # columns of the border x ghost block are rebased by -borderrowoffset (acg/symcsrmatrix.c:838)
        O = sp.csr_matrix((A.oa[:orp[nb]], A.ocolidx[:orp[nb]] - A.c.rowidxbase + off, orp), shape=(nb, A.c.nprows))
        b[off:off + nb] += O @ xloc
    return b, xloc[:no]


def multi_rhs(args, A, n):
    """--nrhs K: K seeded right-hand sides, or with --manufactured-solution K seeded unit-norm solutions
    X* and B = A X* (column j from seed + j).  Returns (B, X*) as (n, K) arrays; X* is None otherwise."""
    k = args.nrhs
    if not args.manufactured_solution:
        B = np.stack([np.random.default_rng(args.seed + j).uniform(-1.0, 1.0, n) for j in range(k)], axis=1)
        return np.ascontiguousarray(B), None
    Xs = np.stack([np.random.default_rng(args.seed + j).uniform(-1.0, 1.0, n) for j in range(k)], axis=1)
    Xs /= np.linalg.norm(Xs, axis=0)
    import scipy.sparse as sp
    rp = A.frowptr[:n + 1]
    F = sp.csr_matrix((A.fa[:rp[n]], A.fcolidx[:rp[n]] - A.c.rowidxbase, rp), shape=(n, n))
    return np.ascontiguousarray(F @ Xs), np.ascontiguousarray(Xs)


def solve_multi(args, A, cg, n, log):
    """The --nrhs run: one solve_multi call, the solver report, then iterations and residual per column
    (and the initial and final error norms with --manufactured-solution)."""
    B, Xs = multi_rhs(args, A, n)
    X = np.zeros_like(B)
    code, cols = cg.solve_multi(B, X, maxits=args.max_iterations, residualatol=args.residual_atol,
                                residualrtol=args.residual_rtol, warmup=args.warmup)
    log(cg.report())
    log(f"right-hand sides: {args.nrhs}")
    for j, c in enumerate(cols):
        line = (f"  column {j}: iterations {c['niterations']} converged {c['converged']} "
                f"residual 2-norm {c['rnrm2']:.15g} relative {c['rnrm2'] / c['r0nrm2'] if c['r0nrm2'] else 0.0:.3e}")
        if Xs is not None:
            line += (f" initial error 2-norm {np.linalg.norm(Xs[:, j]):.15g}"
                     f" error 2-norm {np.linalg.norm(X[:, j] - Xs[:, j]):.15g}")
        log(line)
    if args.output_solution:
        from . import mtxio
        for j in range(args.nrhs):
            root, ext = os.path.splitext(args.output_solution)
            mtxio.write_vector(f"{root}.{j}{ext}", X[:, j], binary=False)
    if code != 0:
        log(f"acg_b200.driver: solver returned {code} (not converged)")
    return code


def solve_shifted(args, A, cg, log):
    """The --shifts run: one solve_shifted call, the solver report, then per shift its iterations, its
    recursively updated residual norm and the true residual ||b - (A + s_j I) x_j||."""
    b, _ = local_rhs(args, A, A.c.nprows)
    code, X, cols = cg.solve_shifted(b, args.shifts, maxits=args.max_iterations, residualatol=args.residual_atol,
                                     residualrtol=args.residual_rtol, warmup=args.warmup)
    log(cg.report())
    log(f"shifts: {len(args.shifts)}")
    import scipy.sparse as sp
    n = A.c.nownedrows
    rp = A.frowptr[:n + 1]
    F = sp.csr_matrix((A.fa[:rp[n]], A.fcolidx[:rp[n]] - A.c.rowidxbase, rp), shape=(n, n))
    for j, (sigma, c) in enumerate(zip(args.shifts, cols)):
        true = float(np.linalg.norm(b - F @ X[:, j] - sigma * X[:, j]))
        log(f"  shift {j} ({sigma:.6g}): iterations {c['niterations']} converged {c['converged']} "
            f"residual 2-norm {c['rnrm2']:.15g} true residual 2-norm {true:.15g} "
            f"relative {true / c['bnrm2'] if c['bnrm2'] else 0.0:.3e}")
    if args.output_solution:
        from . import mtxio
        for j in range(len(args.shifts)):
            root, ext = os.path.splitext(args.output_solution)
            mtxio.write_vector(f"{root}.{j}{ext}", X[:, j], binary=False)
    if code != 0:
        log(f"acg_b200.driver: solver returned {code} (not converged)")
    return code


def solve_minres(args, A, cg, log):
    """The --solver minres, mixed and chebyshev runs: one solve_minres, solve_mixed or solve_chebyshev call, the
    solver report,
    then the iterations (and reliable updates), the solver's residual norm -- MINRES's recursively updated
    one, the mixed solve's fp64 one -- and the true residual ||b - A x|| (and the error norms with
    --manufactured-solution)."""
    n = A.c.nownedrows
    bo, xstar = local_rhs(args, A, n)
    b = A.vector(); x = A.vector()
    b.x[:] = 0.0
    b.x[:n] = bo
    kw = dict(maxits=args.max_iterations, residualatol=args.residual_atol, residualrtol=args.residual_rtol,
              warmup=args.warmup)
    if args.solver == "chebyshev":
        lmin, lmax = args.interval or (0.0, 0.0)
        kw.update(degree=args.degree, lmin=lmin, lmax=lmax)
    code = getattr(cg, SOLVERS[args.solver])(b, x, **kw)
    log(cg.report())
    import scipy.sparse as sp
    rp = A.frowptr[:n + 1]
    F = sp.csr_matrix((A.fa[:rp[n]], A.fcolidx[:rp[n]] - A.c.rowidxbase, rp), shape=(n, n))
    true = float(np.linalg.norm(bo - F @ x.x[:n]))
    inf = cg.info()
    upd = f" reliable updates {inf['mixed_reliable_updates']}" if args.solver == "mixed" else ""
    if args.solver == "chebyshev":
        how = "given" if args.interval else f"estimated from {inf['cheb_est_iterations']} steps"
        upd = (f" degree {args.degree} interval [{inf['cheb_lmin']:.6g}, {inf['cheb_lmax']:.6g}] ({how})"
               f" iterations {cg.c.niterations} products {cg.c.ngemv}")
        log(f"chebyshev:{upd} residual 2-norm {cg.c.rnrm2:.15g} true residual 2-norm {true:.15g} "
            f"relative {true / cg.c.bnrm2 if cg.c.bnrm2 else 0.0:.3e}")
    else:
        log(f"{args.solver}: iterations {cg.c.niterations}{upd} residual 2-norm {cg.c.rnrm2:.15g} "
            f"true residual 2-norm {true:.15g} relative {true / cg.c.bnrm2 if cg.c.bnrm2 else 0.0:.3e}")
    if xstar is not None:
        log(f"initial error 2-norm: {np.linalg.norm(xstar):.15g}")
        log(f"error 2-norm: {np.linalg.norm(x.x[:n] - xstar):.15g}")
    if args.output_solution:
        from . import mtxio
        mtxio.write_vector(args.output_solution, x.x[:n].copy(), binary=False)
    if code != 0:
        log(f"acg_b200.driver: solver returned {code} (not converged)")
    return code


def main(argv=None):
    args = parse_args(argv)
    # torchrun exports OMP_NUM_THREADS=1 unless the caller set it; the ingest and the full-storage
    # expansion are OpenMP code -- give every rank its share of the cores (before libgomp loads)
    if int(os.environ.get("WORLD_SIZE", "1")) > 1 and os.environ.get("OMP_NUM_THREADS") == "1":
        ncpu = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
        os.environ["OMP_NUM_THREADS"] = str(max(1, ncpu // int(os.environ.get("LOCAL_WORLD_SIZE", os.environ["WORLD_SIZE"]))))
    import torch
    import torch.distributed as dist
    from . import dist as abdist, mtxio
    from .api import SolverCuda, SymCsrMatrix, mtx_info

    if args.solver == "chebyshev":
        if not 0 <= args.degree <= 16:
            raise SystemExit("--degree must be between 0 and 16")
        if args.interval is not None:
            try:
                args.interval = tuple(float(t) for t in args.interval.split(","))
            except ValueError:
                args.interval = ()
            if len(args.interval) != 2 or not 0 < args.interval[0] < args.interval[1]:
                raise SystemExit("--interval must be A,B with 0 < A < B")
    elif args.interval is not None:
        raise SystemExit("--interval and --degree belong to --solver chebyshev")
    if args.solver in ONE_PROCESS:
        if int(os.environ.get("WORLD_SIZE", "1")) > 1:
            raise SystemExit(f"--solver {args.solver} runs in one process (one GPU, the whole matrix)")
        if args.nrhs is not None or args.shifts is not None:
            raise SystemExit(f"--solver {args.solver} cannot be combined with --nrhs or --shifts "
                             "(one system, classic CG options)")
    if args.nrhs is not None:
        if not 1 <= args.nrhs <= 8:
            raise SystemExit("--nrhs must be between 1 and 8")
        if int(os.environ.get("WORLD_SIZE", "1")) > 1:
            raise SystemExit("--nrhs runs in one process (one GPU, the whole matrix)")
        if args.solver != "acg":
            raise SystemExit("--nrhs solves with classic CG (--solver acg)")
    if args.shifts is not None:
        try:
            args.shifts = [float(v) for v in args.shifts.split(",")]
        except ValueError:
            raise SystemExit(f"--shifts: not a comma-separated list of numbers: {args.shifts!r}")
        if not 1 <= len(args.shifts) <= 8:
            raise SystemExit("--shifts takes between 1 and 8 shifts")
        if not all(np.isfinite(v) and v >= 0 for v in args.shifts):
            raise SystemExit("--shifts must be finite and >= 0")
        if int(os.environ.get("WORLD_SIZE", "1")) > 1:
            raise SystemExit("--shifts runs in one process (one GPU, the whole matrix)")
        if args.solver != "acg":
            raise SystemExit("--shifts solves with classic CG (--solver acg)")
        if args.nrhs is not None:
            raise SystemExit("--shifts and --nrhs cannot be combined (one right-hand side for all shifts)")
        if args.manufactured_solution:
            raise SystemExit("--shifts and --manufactured-solution cannot be combined (b = 1 for every shift)")
    rank, world, _local = abdist.init_process(backend="gloo")
    log = (lambda *a: print(*a, file=sys.stderr, flush=True)) if rank == 0 else (lambda *a: None)
    if world > 1 and not args.binary:
        raise SystemExit("more than one process needs the binary encoding (--binary): parts are read with pread")
    info = mtx_info(args.A)
    n = info["nrows"]
    t0 = time.perf_counter()
    if world == 1:
        A = SymCsrMatrix.read_mtx(args.A, binary=args.binary)
    else:
        rowparts = row_partition(args, n, rank, world)
        A = SymCsrMatrix.read_mtx_part(args.A, world, rowparts, rank)
    A.dsymv_init(args.epsilon)
    if args.verbose:
        log(f"read and partitioned in {time.perf_counter() - t0:.3f} s: {n} rows, {info['nnzs']} stored nonzeros, {world} part(s)")

    M = abdist.comm_matrix(A, rank, world)
    if args.output_comm_matrix and rank == 0:
        mtxio.write_comm_matrix(args.output_comm_matrix, M)
    if args.verbose or args.dry_run:
        rows = [None] * world
        mine = (int(A.c.nownedrows), int(A.c.ninnerrows), int(A.c.nborderrows), int(A.c.nghostrows), int(A.c.fnpnzs + A.c.onpnzs))
        if world > 1:
            dist.all_gather_object(rows, mine)
        else:
            rows = [mine]
        log("part: owned interior border ghost nonzeros sends")
        for p, r in enumerate(rows):
            log(f"  {p}: {r[0]} {r[1]} {r[2]} {r[3]} {r[4]} {int(M[p].sum())}")
    if args.dry_run:
        if world > 1:
            dist.barrier()
            dist.destroy_process_group()
        return 0

    if not torch.cuda.is_available():
        raise SystemExit("acg_b200.driver: no CUDA device (the solver has no CPU path; --dry-run stops before it)")
    comm = abdist.nccl_comm(rank, world)
    cg = SolverCuda(A, comm)
    if args.shifts is not None:
        code = solve_shifted(args, A, cg, log)
        cg.free()
        comm.destroy()
        return 0 if code == 0 else 1
    if args.solver in ONE_PROCESS:
        code = solve_minres(args, A, cg, log)
        cg.free()
        comm.destroy()
        return 0 if code == 0 else 1
    if args.nrhs is not None:
        code = solve_multi(args, A, cg, n, log)
        cg.free()
        comm.destroy()
        return 0 if code == 0 else 1
    b = A.vector(); x = A.vector()
    bo, xstar = local_rhs(args, A, n)
    no = A.c.nownedrows
    b.x[:] = 0.0
    b.x[:no] = bo
    code = getattr(cg, SOLVERS[args.solver])(b, x, maxits=args.max_iterations, residualatol=args.residual_atol,
                                             residualrtol=args.residual_rtol, warmup=args.warmup)
    if world > 1:
        # the report of acgsolvercuda_fwritempi (acg/cgcuda.c:1948-2216): times as the maximum,
        # flop / byte / message counters as the sum over the ranks, printed by rank 0
        mine = {k: getattr(cg.c, k) for k in SolverCuda.TIMES + SolverCuda.COUNTERS}
        every = [None] * world
        dist.all_gather_object(every, mine)
        agg = {k: max(e[k] for e in every) for k in SolverCuda.TIMES}
        agg.update({k: sum(e[k] for e in every) for k in SolverCuda.COUNTERS})
        log(cg.report(aggregate=agg))
        log(f"processes: {world}")
    else:
        log(cg.report())
    if args.manufactured_solution:
        e2 = np.array([np.sum(xstar ** 2), np.sum((x.x[:no] - xstar) ** 2)])
        if world > 1:
            t = torch.from_numpy(e2)
            dist.all_reduce(t)
        log(f"initial error 2-norm: {np.sqrt(e2[0]):.15g}")
        log(f"error 2-norm: {np.sqrt(e2[1]):.15g}")
    if args.output_solution:
        gidx = (A.nzrows[:no] if len(A.nzrows) >= no else np.arange(no)).copy()
        pieces = [None] * world
        if world > 1:
            dist.all_gather_object(pieces, (gidx, x.x[:no].copy()))
        else:
            pieces = [(gidx, x.x[:no].copy())]
        if rank == 0:
            xg = np.zeros(n)
            for gi, xv in pieces:
                xg[gi] = xv
            mtxio.write_vector(args.output_solution, xg, binary=False)
    cg.free()
    comm.destroy()
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()
    if code != 0:
        log(f"acg_b200.driver: solver returned {code} (not converged)")
    return 0 if code == 0 else 1


if __name__ == "__main__":
    sys.exit(main())
