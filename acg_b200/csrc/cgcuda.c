/*
 * cgcuda.c -- host side of the H100 conjugate-gradient solver (C).
 *
 * Implements the drop-in boundary declared in include/acgb200/cgcuda.h:
 * acgsolvercuda_init / _solvempi / _solve_pipelined / _solve / _fwrite /
 * _free (reference: acg/cgcuda.c).  The host only sequences kernels and
 * NCCL calls; all arithmetic happens in kernels.cu.  There is no CPU
 * fallback: every entry point fails with ACG_ERR_CUDA if no device is usable.
 *
 * Per-iteration schedule, classic CG (replaces acg/cgcuda.c:845-1019):
 *
 *   comm stream : [pack border of p -> ncclSend/Recv into ghost tail of p]
 *   main stream : t = A_loc p (+ p.t over interior rows)
 *                 [wait halo; t += A_off p on border rows (+ p.t over border)]
 *                 [allreduce p.t]
 *                 r -= alpha t  (+ r.r)           alpha = r.r_old / p.t
 *                 [allreduce r.r]
 *                 x += alpha p ; p = r + beta p   beta = r.r / r.r_old
 *
 * Scalars never leave the device.  Convergence is decided on the device by
 * the last kernel of each iteration, which also advances an iteration
 * counter; once "done" is set every later kernel returns immediately, so the
 * host may run ahead and only polls the control word every few iterations
 * (the reference synchronises the host on every iteration, :1007).
 */
#include "acgb200/cgcuda.h"
#include "acgb200/error.h"
#include "acgb200/ext.h"
#include "internal.h"
#include "p2p.h"

#include <cuda_runtime_api.h>
#include <float.h>
#include <math.h>
#include <pthread.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

/* ------------------------------------------------------------------------ */
/* tunables                                                                  */
/* ------------------------------------------------------------------------ */

#define SPMV_MAX_STAGES_HOST 8      /* SPMV_MAX_STAGES of kernels.cu */
#define PCG_GROUP_DEFAULT 16        /* option pcg_group: see the measurements in DESIGN.md section 4a */

static struct {
    int profile;        /* record CUDA events around each kernel class */
    int check_every;    /* iterations between convergence polls */
    int spmv_lanes;     /* 0 = heuristic */
    int spmv_nnz_cap, spmv_rows_cap, spmv_stages, spmv_threads, spmv_unroll;
    int spmv_max_ctas;  /* cap on resident SpMV CTAs per SM (0 = occupancy limit) */
    int graph;          /* replay iteration pairs as CUDA graphs */
    int redstream;      /* pipelined CG: allreduce on its own stream + communicator */
    int p2p;            /* halo + reductions through peer memory (CUDA IPC) instead of NCCL */
    int p2p_fuse;       /* 1: border x ghost block inside the SpMV, pushes inside the update kernels */
    int blas1_ctas;     /* CTAs per SM of the fused BLAS-1 kernels (0 = one full wave, from the occupancy) */
    int pdl;            /* 1: programmatic dependent launch along the iteration chain (opt-in) */
    int spmv_medium;    /* > 0: rows longer than this (and shorter than a tile) get a warp each (opt-in) */
    int spmv_merge;     /* merge-path tiles for irregular rows (mergeplan.c): -1 decide from the row lengths, 0 off, 1 on */
    int merge_items, merge_threads, merge_max_ctas, merge_stages;   /* their shape (0 = default) */
    int spmv_slices;    /* 1: pattern slices (slices.c) -- index-free slice-major storage of the rows that repeat a pattern */
    int slice_ub, slice_threads, slice_max_ctas;   /* slice kernel shape overrides (0 = default) */
    int spmv_symdiag;   /* 1: mirrored diagonals for the slice-covered rows when the matrix allows (slices.c), 0: off */
    int symdiag_evict_first;   /* 1: L2 evict-first policy on the stored diagonals (A/B; the default reuses them in L2) */
    int symdiag_codes;  /* 1: store the diagonals as one-byte codes into a table when they hold at most 256 distinct
                         * values (automatic), 0: always the fp64 diagonals (A/B) */
    int pcg_fused;      /* 1: pipelined CG runs each iteration's product and update in one kernel where the plan allows
                         * (one GPU, mirrored diagonals; DESIGN.md section 4a), 0: off (A/B) */
    int pcg_evict_first;   /* 1: L2 evict-first policy on the fused kernel's vector streams (A/B) */
    int pcg_group;      /* the fused iteration's p and x updates are done once per this many iterations: 2, 4, 8 or 16
                         * (DESIGN.md section 4a) */
    int loaded;
} cfg = { .check_every = 8, .graph = 1, .redstream = 1, .p2p = 1, .p2p_fuse = 1, .spmv_slices = 1, .spmv_merge = -1,
          .spmv_symdiag = 1, .symdiag_codes = 1, .pcg_fused = 1, .pcg_evict_first = 1, .pcg_group = PCG_GROUP_DEFAULT };

static int pcg_group_valid(int m) { return m == 2 || m == 4 || m == 8 || m == ACGB200_PCG_GROUP_MAX; }

static void cfg_load(void)
{
    if (cfg.loaded) return;
    cfg.loaded = 1;
    const char *s;
    if ((s = getenv("ACGB200_PROFILE"))) cfg.profile = atoi(s);
    if ((s = getenv("ACGB200_CHECK_EVERY"))) cfg.check_every = atoi(s);
    if ((s = getenv("ACGB200_SPMV_LANES"))) cfg.spmv_lanes = atoi(s);
    if ((s = getenv("ACGB200_SPMV_NNZ_CAP"))) cfg.spmv_nnz_cap = atoi(s);
    if ((s = getenv("ACGB200_SPMV_ROWS_CAP"))) cfg.spmv_rows_cap = atoi(s);
    if ((s = getenv("ACGB200_SPMV_STAGES"))) cfg.spmv_stages = atoi(s);
    if ((s = getenv("ACGB200_SPMV_THREADS"))) cfg.spmv_threads = atoi(s);
    if ((s = getenv("ACGB200_SPMV_UNROLL"))) cfg.spmv_unroll = atoi(s);
    if ((s = getenv("ACGB200_SPMV_MAX_CTAS"))) cfg.spmv_max_ctas = atoi(s);
    if ((s = getenv("ACGB200_GRAPH"))) cfg.graph = atoi(s);
    if ((s = getenv("ACGB200_REDSTREAM"))) cfg.redstream = atoi(s);
    if ((s = getenv("ACGB200_P2P"))) cfg.p2p = atoi(s);
    if ((s = getenv("ACGB200_P2P_FUSE"))) cfg.p2p_fuse = atoi(s);
    if ((s = getenv("ACGB200_BLAS1_CTAS"))) cfg.blas1_ctas = atoi(s);
    if (cfg.check_every < 1) cfg.check_every = 1;
    if ((s = getenv("ACGB200_PDL"))) cfg.pdl = atoi(s);
    if ((s = getenv("ACGB200_SPMV_MEDIUM"))) cfg.spmv_medium = atoi(s);
    if ((s = getenv("ACGB200_SPMV_MERGE"))) cfg.spmv_merge = atoi(s);
    if ((s = getenv("ACGB200_MERGE_ITEMS"))) cfg.merge_items = atoi(s);
    if ((s = getenv("ACGB200_MERGE_THREADS"))) cfg.merge_threads = atoi(s);
    if ((s = getenv("ACGB200_MERGE_MAX_CTAS"))) cfg.merge_max_ctas = atoi(s);
    if ((s = getenv("ACGB200_MERGE_STAGES"))) cfg.merge_stages = atoi(s);
    if ((s = getenv("ACGB200_SPMV_SLICES"))) cfg.spmv_slices = atoi(s);
    if ((s = getenv("ACGB200_SLICE_UB"))) cfg.slice_ub = atoi(s);
    if ((s = getenv("ACGB200_SLICE_THREADS"))) cfg.slice_threads = atoi(s);
    if ((s = getenv("ACGB200_SLICE_MAX_CTAS"))) cfg.slice_max_ctas = atoi(s);
    if ((s = getenv("ACGB200_SPMV_SYMDIAG"))) cfg.spmv_symdiag = atoi(s);
    if ((s = getenv("ACGB200_SYMDIAG_EVICT_FIRST"))) cfg.symdiag_evict_first = atoi(s);
    if ((s = getenv("ACGB200_SYMDIAG_CODES"))) cfg.symdiag_codes = atoi(s);
    if ((s = getenv("ACGB200_PCG_FUSED"))) cfg.pcg_fused = atoi(s);
    if ((s = getenv("ACGB200_PCG_EVICT_FIRST"))) cfg.pcg_evict_first = atoi(s);
    if ((s = getenv("ACGB200_PCG_GROUP")) && pcg_group_valid(atoi(s))) cfg.pcg_group = atoi(s);
    acgb200_blas1_set_ctas_per_sm(cfg.blas1_ctas);
    acgb200_set_pdl(cfg.pdl);
}

int acgb200_set_option(const char *key, int value)
{
    cfg_load();
    if (!strcmp(key, "profile")) cfg.profile = value;
    else if (!strcmp(key, "check_every")) cfg.check_every = value < 1 ? 1 : value;
    else if (!strcmp(key, "spmv_lanes")) cfg.spmv_lanes = value;
    else if (!strcmp(key, "spmv_nnz_cap")) cfg.spmv_nnz_cap = value;
    else if (!strcmp(key, "spmv_rows_cap")) cfg.spmv_rows_cap = value;
    else if (!strcmp(key, "spmv_stages")) cfg.spmv_stages = value;
    else if (!strcmp(key, "spmv_threads")) cfg.spmv_threads = value;
    else if (!strcmp(key, "spmv_unroll")) cfg.spmv_unroll = value;
    else if (!strcmp(key, "spmv_max_ctas")) cfg.spmv_max_ctas = value;
    else if (!strcmp(key, "graph")) cfg.graph = value;
    else if (!strcmp(key, "redstream")) cfg.redstream = value;
    else if (!strcmp(key, "p2p")) cfg.p2p = value;
    else if (!strcmp(key, "p2p_fuse")) cfg.p2p_fuse = value;
    else if (!strcmp(key, "blas1_ctas")) { cfg.blas1_ctas = value; acgb200_blas1_set_ctas_per_sm(value); }
    else if (!strcmp(key, "pdl")) { cfg.pdl = value; acgb200_set_pdl(value); }
    else if (!strcmp(key, "spmv_medium")) cfg.spmv_medium = value < 0 ? 0 : value;
    else if (!strcmp(key, "spmv_merge")) cfg.spmv_merge = value;
    else if (!strcmp(key, "merge_items")) cfg.merge_items = value;
    else if (!strcmp(key, "merge_threads")) cfg.merge_threads = value;
    else if (!strcmp(key, "merge_max_ctas")) cfg.merge_max_ctas = value;
    else if (!strcmp(key, "merge_stages")) cfg.merge_stages = value;
    else if (!strcmp(key, "spmv_slices")) cfg.spmv_slices = value;
    else if (!strcmp(key, "slice_ub")) cfg.slice_ub = value;
    else if (!strcmp(key, "slice_threads")) cfg.slice_threads = value;
    else if (!strcmp(key, "slice_max_ctas")) cfg.slice_max_ctas = value;
    else if (!strcmp(key, "spmv_symdiag")) cfg.spmv_symdiag = value;
    else if (!strcmp(key, "symdiag_evict_first")) cfg.symdiag_evict_first = value;
    else if (!strcmp(key, "symdiag_codes")) cfg.symdiag_codes = value;
    else if (!strcmp(key, "pcg_fused")) cfg.pcg_fused = value;
    else if (!strcmp(key, "pcg_evict_first")) cfg.pcg_evict_first = value;
    else if (!strcmp(key, "pcg_group") && pcg_group_valid(value)) cfg.pcg_group = value;
    else return ACG_ERR_INVALID_VALUE;
    return ACG_SUCCESS;
}

/* ------------------------------------------------------------------------ */
/* private per-solver state                                                  */
/* ------------------------------------------------------------------------ */

struct evpool { cudaEvent_t *ev; int n, cap; };

/* the loops a solver runs; each has its own cached graph */
enum solve_kind { KIND_CLASSIC, KIND_PIPELINED, KIND_MULTI, KIND_SHIFTED, KIND_MINRES, KIND_MIXED, KIND_CHEB, NKINDS };

struct priv {
    const struct acgsolvercuda *key;
    const void *d_r_id;                 /* cg->d_r: identifies the solver if the caller moves the struct */
    struct priv *next;
    struct acgb200_spmvplan plan;
    struct acgb200_devstate *d_st;
    struct acgb200_ctrl *h_ctrl;        /* pinned, 2 poll slots */
    void *h_st;                         /* pinned staging of every struct of device scalars (scalars_push / _pull) */
    int nrows, nowned, ninner, nborder, nghost, borderoff, nvec;
    int64_t fnnz, onnz;
    int device_expanded;                /* the full storage was built on the device (the host matrix has none) */
    cudaStream_t stream, commstream, redstream;
    cudaEvent_t ev_ready, ev_halo, ev_red, ev_poll[2];
    struct acgb200_p2p p2p;             /* peer-memory exchange (multi-GPU) */
    struct acgcomm redcomm;             /* private duplicate of the caller's communicator for reductions */
    int have_redcomm;
    double *d_b, *d_x;                  /* right-hand side / solution on the device, kept between solves */
    cudaGraphExec_t graph[NKINDS];      /* per solve kind: two iterations (parity 0 then 1), or a fused group */
    int graph_sig[NKINDS];              /* loop configuration each cached graph was captured with (graph_signature) */
    int graph_launches[NKINDS];         /* kernel/NCCL launches inside one replay */
    double last_h2d_ms, last_d2h_ms;    /* host time spent before / after the solve window */
    cudaEvent_t ev_t0, ev_t1;           /* device-side bracket of the solve window */
    double last_solve_ms;
    struct evpool gemv, blas;           /* profiling */
    int last_launches;                  /* kernels launched in the last solve's timed loop */
    double last_spmv_ms;                /* profiled SpMV time of the last solve */
    double last_blas_ms;                /* profiled fused-update time of the last solve */
    int last_spmv_n;
    int last_fused;                     /* the last solve ran the fused pipelined-CG iteration */
    /* fused pipelined CG: the second buffer of w, and slots 1 ... r_slots of the r ring, r_stride doubles apart
     * (made at the first such solve, the ring grown with the group) */
    double *d_w2, *d_rring;
    size_t r_stride;
    int r_slots;
    int last_group;                     /* the group of the last fused solve */
    int commsize;                       /* ranks of the communicator given to acgsolvercuda_init */
    /* several right-hand sides (acgsolvercuda_solve_multi), made at the first multi-vector call */
    struct acgb200_mstate *d_ms;        /* per-column scalars */
    double *d_mx, *d_mb, *d_mr, *d_mp, *d_mt;   /* block vectors X, B, R, P, T: nowned x mk, interleaved */
    int mk;                             /* their width */
    int *d_ranges;                      /* [2 * nranges] row chunks outside the pattern slices */
    int nranges, ranges_lanes, have_ranges;
    /* shifted systems (acgsolvercuda_solve_shifted): per-shift scalars; the vectors are the blocks above */
    struct acgb200_sstate *d_ss;
    /* MINRES (acgsolvercuda_solve_minres), made at the first such solve: its scalars and the two w buffers
     * (v lives in d_r / d_p, t and u in d_t) */
    struct acgb200_nstate *d_ns;
    double *d_nw[2];
    /* mixed precision (acgsolvercuda_solve_mixed), made at the first such solve: its scalars, the float
     * vectors r, p, t, y (one allocation; the fp64 residual lives in d_r) and the row chunks of its product
     * outside the mirrored diagonals */
    struct acgb200_xstate *d_xs;
    float *d_f32;
    int *d_franges;
    int nfranges, have_franges;
    int last_mixed_updates;
    /* Chebyshev-preconditioned CG (acgsolvercuda_solve_chebyshev), made at the first such solve: its scalars
     * and five vectors D^-1, z, res, d_0, d_1 (one allocation); baddiag: the diagonal entries that are <= 0 or
     * non-finite (-1: not counted yet); cheb_graph_ab: the interval whose coefficients the cached graph holds */
    struct acgb200_cstate *d_cs;
    double *d_cvec;
    int cheb_baddiag;
    double cheb_graph_ab[2];
    int last_cheb_degree, last_cheb_est, last_cheb_breakdown;
    double last_cheb_lmin, last_cheb_lmax;
};

/* The public struct has no room for private state (its layout is the
 * reference's), so it lives in a registry keyed by the solver's address.  The
 * lock only guards the list: one solver is driven by one host thread, as in the
 * reference, but different solvers may live on different threads. */
static struct priv *registry = NULL;
static pthread_mutex_t registry_lock = PTHREAD_MUTEX_INITIALIZER;

static struct priv *priv_of(const struct acgsolvercuda *cg)
{
    struct priv *found = NULL;
    pthread_mutex_lock(&registry_lock);
    for (struct priv *p = registry; p; p = p->next) if (p->key == cg) { found = p; break; }
    if (!found && cg->d_r) {
        /* the caller copied or moved the struct (the reference allows that: it is plain data).  The device
         * vector d_r is allocated by acgsolvercuda_init and belongs to exactly one solver: find the state
         * through it and follow the struct to its new address. */
        for (struct priv *p = registry; p; p = p->next)
            if (p->d_r_id == (const void *) cg->d_r) { found = p; p->key = cg; break; }
    }
    pthread_mutex_unlock(&registry_lock);
    return found;
}

static void priv_add(struct priv *pv)
{
    pthread_mutex_lock(&registry_lock);
    pv->next = registry; registry = pv;
    pthread_mutex_unlock(&registry_lock);
}

static void priv_drop(struct priv *pv)
{
    struct priv *d = NULL;
    pthread_mutex_lock(&registry_lock);
    for (struct priv **pp = &registry; *pp; pp = &(*pp)->next) {
        if (*pp == pv) { d = *pp; *pp = d->next; break; }
    }
    pthread_mutex_unlock(&registry_lock);
    free(d);
}

static double wall(void)
{
    struct timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return (double) ts.tv_sec + 1e-9 * (double) ts.tv_nsec;
}

#define CU(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { if (errcode) *errcode = (int) e_; return ACG_ERR_CUDA; } } while (0)
#define KL(call) do { int e_ = (call); if (e_) { if (errcode) *errcode = e_; return ACG_ERR_CUDA; } } while (0)
#define OK(call) do { int e_ = (call); if (e_) return e_; } while (0)

/* the size of h_st: the largest struct of device scalars */
static size_t staging_bytes(void)
{
    const size_t sizes[] = { sizeof(struct acgb200_devstate), sizeof(struct acgb200_mstate), sizeof(struct acgb200_sstate),
                             sizeof(struct acgb200_nstate), sizeof(struct acgb200_xstate), sizeof(struct acgb200_cstate) };
    size_t m = 0;
    for (size_t i = 0; i < sizeof(sizes) / sizeof(sizes[0]); i++) if (sizes[i] > m) m = sizes[i];
    return m;
}

/* a solver's struct of device scalars, made (zeroed) at its first use */
static int dev_scalars_once(struct priv *pv, void **d, size_t bytes, int *errcode)
{
    if (*d) return ACG_SUCCESS;
    CU(cudaMalloc(d, bytes));
    CU(cudaMemsetAsync(*d, 0, bytes, pv->stream));
    return ACG_SUCCESS;
}

/* ------------------------------------------------------------------------ */
/* free / init                                                               */
/* ------------------------------------------------------------------------ */

static void free_vecptr(struct acgvector **v)
{
    if (*v) { acgvector_free(*v); free(*v); *v = NULL; }
}

void acgsolvercuda_free(struct acgsolvercuda *cg)
{
    struct priv *pv = priv_of(cg);
    acgvector_free(&cg->r); acgvector_free(&cg->p); acgvector_free(&cg->t);
    free_vecptr(&cg->w); free_vecptr(&cg->q); free_vecptr(&cg->z); free_vecptr(&cg->dx);
    if (cg->halo) { acghalo_free(cg->halo); free(cg->halo); cg->halo = NULL; }
    if (cg->haloexchange) { acghaloexchange_free(cg->haloexchange); free(cg->haloexchange); cg->haloexchange = NULL; }
    cudaFree(cg->d_r); cudaFree(cg->d_p); cudaFree(cg->d_t);
    cudaFree(cg->d_w); cudaFree(cg->d_q); cudaFree(cg->d_z);
    cudaFree(cg->d_rowptr); cudaFree(cg->d_colidx); cudaFree(cg->d_a);
    cudaFree(cg->d_orowptr); cudaFree(cg->d_ocolidx); cudaFree(cg->d_oa);
    cg->d_r = cg->d_p = cg->d_t = cg->d_w = cg->d_q = cg->d_z = NULL;
    cg->d_rowptr = cg->d_colidx = cg->d_orowptr = cg->d_ocolidx = NULL;
    cg->d_a = cg->d_oa = NULL;
    if (pv) {
        if (pv->stream) cudaStreamSynchronize(pv->stream);
        if (pv->p2p.window) {
            /* unmap the peers' windows, wait until every rank has done so, then
             * release this rank's (collective, like the init that created it) */
            acgb200_p2p_free(&pv->p2p);
            if (pv->have_redcomm) { acgcomm_barrier(pv->stream, &pv->redcomm, NULL); cudaStreamSynchronize(pv->stream); }
            cudaFree(pv->p2p.window);
            pv->p2p.window = NULL;
        }
        if (pv->have_redcomm && pv->redcomm.ncclcomm) ncclCommDestroy(pv->redcomm.ncclcomm);
        for (int i = 0; i < NKINDS; i++) if (pv->graph[i]) cudaGraphExecDestroy(pv->graph[i]);
        cudaFree(pv->plan.d_tiles); cudaFree(pv->plan.d_longrows); cudaFree(pv->plan.d_long_scratch); cudaFree(pv->plan.d_medrows);
        cudaFree(pv->plan.d_slices); cudaFree(pv->plan.d_sval); cudaFree(pv->plan.d_spatoff); cudaFree(pv->plan.d_spatid);
        cudaFree(pv->plan.d_hval); cudaFree(pv->plan.d_symdiag_bad); cudaFree(pv->plan.d_hcode); cudaFree(pv->plan.d_codes);
        cudaFree(pv->plan.d_mtiles); cudaFree(pv->plan.d_msplit); cudaFree(pv->plan.d_mpart);
        cudaFree(pv->d_st);
        cudaFreeHost(pv->h_ctrl); cudaFreeHost(pv->h_st);
        if (pv->stream) cudaStreamDestroy(pv->stream);
        if (pv->commstream) cudaStreamDestroy(pv->commstream);
        if (pv->redstream) cudaStreamDestroy(pv->redstream);
        if (pv->ev_red) cudaEventDestroy(pv->ev_red);
        cudaFree(pv->d_b); cudaFree(pv->d_x); cudaFree(pv->d_w2); cudaFree(pv->d_rring);
        cudaFree(pv->d_ms); cudaFree(pv->d_ranges); cudaFree(pv->d_ss);
        cudaFree(pv->d_ns); cudaFree(pv->d_nw[0]); cudaFree(pv->d_nw[1]);
        cudaFree(pv->d_xs); cudaFree(pv->d_f32); cudaFree(pv->d_franges);
        cudaFree(pv->d_cs); cudaFree(pv->d_cvec);
        cudaFree(pv->d_mx); cudaFree(pv->d_mb); cudaFree(pv->d_mr); cudaFree(pv->d_mp); cudaFree(pv->d_mt);
        if (pv->ev_ready) cudaEventDestroy(pv->ev_ready);
        if (pv->ev_halo) cudaEventDestroy(pv->ev_halo);
        for (int i = 0; i < 2; i++) if (pv->ev_poll[i]) cudaEventDestroy(pv->ev_poll[i]);
        if (pv->ev_t0) cudaEventDestroy(pv->ev_t0);
        if (pv->ev_t1) cudaEventDestroy(pv->ev_t1);
        for (int i = 0; i < pv->gemv.cap; i++) cudaEventDestroy(pv->gemv.ev[i]);
        for (int i = 0; i < pv->blas.cap; i++) cudaEventDestroy(pv->blas.ev[i]);
        free(pv->gemv.ev); free(pv->blas.ev);
        priv_drop(pv);
    }
}

/* Cut rows [0,nrows) into TMA tiles (see internal.h): greedy, row-aligned, at
 * most rows_cap rows and nnz_cap nonzeros per tile; rows longer than nnz_cap go
 * to the long-row list.  Host-only, no CUDA: testable without a device. */
static int cut_tiles(const struct acgb200_spmvplan *pl, const int64_t *rowptr, const unsigned char *covered, int row_lo,
                     struct acgb200_tile *tiles, int *ntiles, int *longrows, int *nlong, int *medrows, int *nmed)
{
    const int n = pl->nrows;
    /* rows above `out` leave the tiles: the long ones (> nnz_cap) always, the medium ones on request */
    const int64_t out = pl->med_thr > 0 && pl->med_thr < pl->nnz_cap ? pl->med_thr : pl->nnz_cap;
    int nt = 0, nl = 0, nm = 0, r = row_lo;        /* rows below row_lo are in merge-path tiles (mergeplan.c) */
    while (r < n) {
        /* rows of a covered 32-row slice belong to the slice kernel (slices.c) */
        if (covered && covered[r >> 5]) { r = (r | 31) + 1; continue; }
        int64_t len = rowptr[r + 1] - rowptr[r];
        if (len > pl->nnz_cap) { longrows[nl++] = r++; continue; }
        if (len > out) { medrows[nm++] = r++; continue; }
        const int start = r;
        int64_t cnt = 0;
        while (r < n && r - start < pl->rows_cap) {
            if (covered && covered[r >> 5]) break;
            len = rowptr[r + 1] - rowptr[r];
            if (len > out || cnt + len > pl->nnz_cap) break;
            cnt += len; r++;
        }
        const int64_t kb = rowptr[start], ke = rowptr[r];
        if (ke > INT32_MAX) return ACG_ERR_INDEX_OUT_OF_BOUNDS;
        const int64_t k_al = kb & ~(int64_t) 3;
        tiles[nt].row_begin = start;
        tiles[nt].nrows = r - start;
        tiles[nt].k_al = (int) k_al;
        tiles[nt].nnz_al = (int) (((ke - k_al) + 3) & ~(int64_t) 3);
        nt++;
    }
    *ntiles = nt; *nlong = nl; *nmed = nm;
    return ACG_SUCCESS;
}

static int build_tiles(struct acgb200_spmvplan *pl, const int64_t *rowptr,
                       const struct acgb200_sliceplan *sp, const unsigned short *patid,
                       const struct acgb200_mergeplan *mp, int *errcode)
{
    const int n = pl->nrows;
    struct acgb200_tile *tiles = malloc(((size_t) n + 1) * sizeof(*tiles));
    int *longrows = malloc(((size_t) n + 1) * sizeof(*longrows));
    int *medrows = malloc(((size_t) n + 1) * sizeof(*medrows));
    if (!tiles || !longrows || !medrows) { free(tiles); free(longrows); free(medrows); return ACG_ERR_ERRNO; }
    int nt = 0, nl = 0, nm = 0;
    int err = cut_tiles(pl, rowptr, sp && sp->nslices > 0 ? sp->covered : NULL, mp && mp->ntiles > 0 ? mp->rows : 0,
                        tiles, &nt, longrows, &nl, medrows, &nm);
    if (err) { free(tiles); free(longrows); free(medrows); return err; }
    pl->ntiles = nt; pl->nlong = nl; pl->nmed = nm;
    pl->d_tiles = NULL; pl->d_longrows = NULL; pl->d_long_scratch = NULL; pl->d_medrows = NULL;
    cudaError_t e = cudaSuccess;
    if (!e && nt > 0) {
        e = cudaMalloc((void **) &pl->d_tiles, (size_t) nt * sizeof(*tiles));
        if (!e) e = cudaMemcpy(pl->d_tiles, tiles, (size_t) nt * sizeof(*tiles), cudaMemcpyHostToDevice);
    }
    if (!e && nl > 0) {
        e = cudaMalloc((void **) &pl->d_longrows, (size_t) nl * sizeof(int));
        if (!e) e = cudaMemcpy(pl->d_longrows, longrows, (size_t) nl * sizeof(int), cudaMemcpyHostToDevice);
        if (!e) e = cudaMalloc((void **) &pl->d_long_scratch, (size_t) nl * (size_t) pl->long_chunks * sizeof(double));
    }
    if (!e && nm > 0) {
        e = cudaMalloc((void **) &pl->d_medrows, (size_t) nm * sizeof(int));
        if (!e) e = cudaMemcpy(pl->d_medrows, medrows, (size_t) nm * sizeof(int), cudaMemcpyHostToDevice);
    }
    pl->nslices = 0;
    if (!e && sp && sp->nslices > 0) {
        pl->nslices = sp->nslices; pl->sval_blocks = sp->blocks; pl->slice_rows = sp->rows; pl->slice_nnz = sp->nnz;
        pl->slice_lpad = sp->lpad; pl->slice_npat = sp->npat; pl->slice_exc = sp->nexc; pl->slice_excnnz = sp->excnnz;
        patid = sp->patid;          /* ids as the slice kernel sees them (exception rows marked) */
        const size_t tab = (size_t) sp->npat * (size_t) sp->lpad;
        e = cudaMalloc((void **) &pl->d_slices, (size_t) sp->nslices * sizeof(*sp->slices));
        if (!e) e = cudaMemcpy(pl->d_slices, sp->slices, (size_t) sp->nslices * sizeof(*sp->slices), cudaMemcpyHostToDevice);
        if (!e) e = cudaMalloc((void **) &pl->d_spatoff, (tab + 4) * sizeof(int));
        if (!e) e = cudaMemset(pl->d_spatoff, 0, (tab + 4) * sizeof(int));
        if (!e) e = cudaMemcpy(pl->d_spatoff, sp->spatoff, tab * sizeof(int), cudaMemcpyHostToDevice);
        if (!e) e = cudaMalloc((void **) &pl->d_spatid, ((size_t) n + 32) * sizeof(unsigned short));
        if (!e) e = cudaMemset(pl->d_spatid, 0, ((size_t) n + 32) * sizeof(unsigned short));
        if (!e) e = cudaMemcpy(pl->d_spatid, patid, (size_t) n * sizeof(unsigned short), cudaMemcpyHostToDevice);
        if (!e) e = cudaMalloc((void **) &pl->d_sval, (size_t) sp->blocks * 32 * sizeof(double));
    }
    pl->nmtiles = 0;
    if (!e && mp && mp->ntiles > 0) {
        pl->nmtiles = mp->ntiles; pl->nsplit = mp->nsplit; pl->merge_items = mp->items; pl->merge_rows = mp->rows; pl->merge_nnz = mp->nnz;
        e = cudaMalloc((void **) &pl->d_mtiles, (size_t) mp->ntiles * sizeof(*mp->tiles));
        if (!e) e = cudaMemcpy(pl->d_mtiles, mp->tiles, (size_t) mp->ntiles * sizeof(*mp->tiles), cudaMemcpyHostToDevice);
        if (!e) e = cudaMalloc((void **) &pl->d_msplit, (size_t) (mp->nsplit > 0 ? mp->nsplit : 1) * sizeof(*mp->split));
        if (!e && mp->nsplit > 0) e = cudaMemcpy(pl->d_msplit, mp->split, (size_t) mp->nsplit * sizeof(*mp->split), cudaMemcpyHostToDevice);
        if (!e) e = cudaMalloc((void **) &pl->d_mpart, 2 * (size_t) mp->ntiles * sizeof(double));
        if (!e) e = cudaMemset(pl->d_mpart, 0, 2 * (size_t) mp->ntiles * sizeof(double));
    }
    free(tiles); free(longrows); free(medrows);
    CU(e);
    return ACG_SUCCESS;
}

/* ext.h: row-pattern dictionary of a CSR matrix, host only (compress.c) */
int acgb200_patterns_host(int nrows, const int64_t *rowptr, const int *colidx, int max_entries,
                          int *npat, int *nentries, int *patptr, int *patoff, unsigned short *patid, int64_t *nmatched)
{
    struct acgb200_patterns pat;
    int err = acgb200_patterns_build(nrows, rowptr, colidx, max_entries, &pat);
    if (err) return err;
    *npat = pat.npat; *nentries = pat.nentries; *nmatched = pat.nrows_matched;
    memcpy(patptr, pat.patptr, ((size_t) pat.npat + 1) * sizeof(int));
    memcpy(patoff, pat.patoff, (size_t) pat.nentries * sizeof(int));
    memcpy(patid, pat.patid, (size_t) nrows * sizeof(unsigned short));
    acgb200_patterns_free(&pat);
    return ACG_SUCCESS;
}

/* ext.h: the merge-path tile plan, host only (mergeplan.c) */
int acgb200_merge_plan_host(int hi, const int64_t *rowptr, int items, int *tiles4, int maxtiles,
                            int *split3, int *ntiles, int *nsplit)
{
    struct acgb200_mergeplan mp;
    int err = acgb200_merge_plan(hi, rowptr, items, &mp);
    if (!err && mp.ntiles > maxtiles) err = ACG_ERR_NO_BUFFER_SPACE;
    if (!err) {
        for (int t = 0; t < mp.ntiles; t++) {
            tiles4[4 * t] = mp.tiles[t].r0; tiles4[4 * t + 1] = mp.tiles[t].nre;
            tiles4[4 * t + 2] = mp.tiles[t].k0; tiles4[4 * t + 3] = mp.tiles[t].nnz;
        }
        for (int i = 0; i < mp.nsplit; i++) {
            split3[3 * i] = mp.split[i].row; split3[3 * i + 1] = mp.split[i].ta; split3[3 * i + 2] = mp.split[i].tb;
        }
        *ntiles = mp.ntiles; *nsplit = mp.nsplit;
    }
    acgb200_mergeplan_free(&mp);
    return err;
}

/* ext.h: the pattern-slice plan of a CSR matrix, host only (slices.c) */
int acgb200_slices_host(int nrows, int cover_hi, const int64_t *rowptr, const int *colidx,
                        int *slices4, int maxslices, unsigned char *covered, int64_t *totals6, int *spatoff,
                        unsigned short *patid, int64_t *exc2)
{
    struct acgb200_patterns pat;
    struct acgb200_sliceplan sp;
    int err = acgb200_patterns_build(nrows, rowptr, colidx, 4096, &pat);
    if (err) return err;
    err = acgb200_slices_plan(nrows, cover_hi, rowptr, &pat, &sp);
    if (!err && sp.nslices > maxslices) err = ACG_ERR_NO_BUFFER_SPACE;
    if (!err) {
        for (int i = 0; i < sp.nslices; i++) {
            slices4[4 * i] = sp.slices[i].row0; slices4[4 * i + 1] = sp.slices[i].nrows;
            slices4[4 * i + 2] = sp.slices[i].len; slices4[4 * i + 3] = sp.slices[i].vblk;
        }
        memcpy(covered, sp.covered, (size_t) ((nrows + 31) / 32));
        totals6[0] = sp.nslices; totals6[1] = sp.blocks; totals6[2] = sp.nnz; totals6[3] = sp.rows;
        totals6[4] = sp.lpad; totals6[5] = sp.npat;
        if (sp.nslices > 0) memcpy(spatoff, sp.spatoff, (size_t) sp.npat * (size_t) sp.lpad * sizeof(int));
        if (patid && sp.nslices > 0) memcpy(patid, sp.patid, (size_t) nrows * sizeof(*patid));
        if (exc2) { exc2[0] = sp.nexc; exc2[1] = sp.excnnz; }
    }
    acgb200_sliceplan_free(&sp);
    acgb200_patterns_free(&pat);
    return err;
}

/* ext.h: the mirrored-diagonal plan of a CSR matrix's pattern slices, host only (slices.c) */
int acgb200_symdiag_host(int nrows, int cover_hi, const int64_t *rowptr, const int *colidx, int *info5, int *o, int *d,
                         int *tab2)
{
    struct acgb200_patterns pat;
    struct acgb200_sliceplan sp;
    struct acgb200_symdiag sd;
    int err = acgb200_patterns_build(nrows, rowptr, colidx, 4096, &pat);
    if (err) return err;
    err = acgb200_slices_plan(nrows, cover_hi, rowptr, &pat, &sp);
    if (!err) err = acgb200_symdiag_plan(nrows, &sp, &pat, &sd);
    if (!err) {
        int margin = 0, stride = 0;
        struct acgb200_symdiag_entry tab[ACGB200_SYMDIAG_MAX];
        if (sd.reason == SYMDIAG_OK) acgb200_symdiag_layout(nrows, &sd, &margin, &stride, tab);
        info5[0] = sd.reason; info5[1] = sd.no; info5[2] = sd.nd; info5[3] = margin; info5[4] = stride;
        memcpy(o, sd.o, (size_t) sd.no * sizeof(int));
        memcpy(d, sd.d, (size_t) sd.nd * sizeof(int));
        if (sd.reason == SYMDIAG_OK)
            for (int e = 0; e < sd.no; e++) { tab2[2 * e] = tab[e].voff; tab2[2 * e + 1] = tab[e].coff; }
    }
    acgb200_sliceplan_free(&sp);
    acgb200_patterns_free(&pat);
    return err;
}

/* ext.h: the tile plan the solver would build for a CSR row-pointer array,
 * computed on the host without touching a device.  With colidx != NULL (0-based)
 * the pattern slices are planned too, exactly as acgsolvercuda_init does under option
 * "spmv_slices": the tiles then skip the rows of covered slices (acgb200_slices_host
 * returns the slices themselves). */
int acgb200_spmv_plan_host(int nrows, const int64_t *rowptr, struct acgb200_info *info,
                           int *tiles4, int maxtiles, int *longrows, int maxlong)
{
    return acgb200_spmv_plan_host2(nrows, rowptr, NULL, info, tiles4, maxtiles, longrows, maxlong);
}

int acgb200_spmv_plan_host2(int nrows, const int64_t *rowptr, const int *colidx, struct acgb200_info *info,
                            int *tiles4, int maxtiles, int *longrows, int maxlong)
{
    struct acgb200_spmvplan pl;
    memset(&pl, 0, sizeof(pl));
    int64_t maxlen = 0;
    for (int i = 0; i < nrows; i++) if (rowptr[i + 1] - rowptr[i] > maxlen) maxlen = rowptr[i + 1] - rowptr[i];
    acgb200_spmv_choose(&pl, nrows, rowptr[nrows] - rowptr[0], maxlen);
    cfg_load();
    if (cfg.spmv_lanes > 0) pl.lanes_per_row = cfg.spmv_lanes;
    if (cfg.spmv_nnz_cap > 0) pl.nnz_cap = cfg.spmv_nnz_cap;
    if (cfg.spmv_rows_cap > 0) pl.rows_cap = cfg.spmv_rows_cap;
    pl.med_thr = cfg.spmv_medium;
    struct acgb200_tile *tiles = malloc(((size_t) nrows + 1) * sizeof(*tiles));
    int *lr = malloc(((size_t) nrows + 1) * sizeof(*lr));
    int *mr = malloc(((size_t) nrows + 1) * sizeof(*mr));
    if (!tiles || !lr || !mr) { free(tiles); free(lr); free(mr); return ACG_ERR_ERRNO; }
    int nt = 0, nl = 0, nm = 0, nsl = 0, slrows = 0;
    int err = ACG_SUCCESS;
    struct acgb200_patterns pat;
    struct acgb200_sliceplan sp;
    memset(&pat, 0, sizeof(pat)); memset(&sp, 0, sizeof(sp));
    if (colidx && cfg.spmv_slices) {
        err = acgb200_patterns_build(nrows, rowptr, colidx, 4096, &pat);
        if (!err && pat.npat > 0) err = acgb200_slices_plan(nrows, nrows, rowptr, &pat, &sp);
        nsl = sp.nslices; slrows = sp.rows;
    }
    if (!err) err = cut_tiles(&pl, rowptr, sp.nslices > 0 ? sp.covered : NULL, 0, tiles, &nt, lr, &nl, mr, &nm);
    acgb200_sliceplan_free(&sp);
    acgb200_patterns_free(&pat);
    if (!err && (nt > maxtiles || nl > maxlong)) err = ACG_ERR_NO_BUFFER_SPACE;
    if (!err) {
        for (int t = 0; t < nt; t++) {
            tiles4[4 * t] = tiles[t].row_begin; tiles4[4 * t + 1] = tiles[t].nrows;
            tiles4[4 * t + 2] = tiles[t].k_al; tiles4[4 * t + 3] = tiles[t].nnz_al;
        }
        memcpy(longrows, lr, (size_t) nl * sizeof(int));
        memset(info, 0, sizeof(*info));
        info->spmv_lanes_per_row = pl.lanes_per_row; info->spmv_rows_cap = pl.rows_cap;
        info->spmv_nnz_cap = pl.nnz_cap; info->spmv_stages = pl.nstages;
        info->spmv_ntiles = nt; info->spmv_nlong = nl; info->spmv_slices = nsl; info->spmv_slice_rows = slrows;
        info->spmv_nmedium = nm;
    }
    free(tiles); free(lr); free(mr);
    return err;
}

/* upload a host int64 row-pointer array narrowed to int32 (acg/cgcuda.c:262-272)
 * with `pad` trailing entries repeating the last value */
static int upload_rowptr(int **d_out, const int64_t *rp, int64_t n, int pad, int *errcode)
{
    int *tmp = malloc(((size_t) n + 1 + (size_t) pad) * sizeof(*tmp));
    if (!tmp) return ACG_ERR_ERRNO;
    for (int64_t i = 0; i <= n; i++) {
        if (rp[i] > INT32_MAX) { free(tmp); return ACG_ERR_INDEX_OUT_OF_BOUNDS; }
        tmp[i] = (int) rp[i];
    }
    for (int i = 1; i <= pad; i++) tmp[n + i] = tmp[n];
    cudaError_t e = cudaMalloc((void **) d_out, ((size_t) n + 1 + (size_t) pad) * sizeof(*tmp));
    if (!e) e = cudaMemcpy(*d_out, tmp, ((size_t) n + 1 + (size_t) pad) * sizeof(*tmp), cudaMemcpyHostToDevice);
    free(tmp);
    if (e) { if (errcode) *errcode = (int) e; return ACG_ERR_CUDA; }
    return ACG_SUCCESS;
}

static int upload_block(int **d_col, double **d_val, const acgidx_t *col, const double *val,
                        int64_t nnz, int base, int pad, int *errcode)
{
    const size_t cap = (size_t) nnz + (size_t) pad;
    CU(cudaMalloc((void **) d_col, cap * sizeof(int)));
    CU(cudaMalloc((void **) d_val, cap * sizeof(double)));
    CU(cudaMemset(*d_col + nnz, 0, (size_t) pad * sizeof(int)));
    CU(cudaMemset(*d_val + nnz, 0, (size_t) pad * sizeof(double)));
    if (nnz > 0) {
        if (base == 0) {
            CU(cudaMemcpy(*d_col, col, (size_t) nnz * sizeof(int), cudaMemcpyHostToDevice));
        } else {
            int *tmp = malloc((size_t) nnz * sizeof(int));
            if (!tmp) return ACG_ERR_ERRNO;
            for (int64_t k = 0; k < nnz; k++) tmp[k] = col[k] - base;
            cudaError_t e = cudaMemcpy(*d_col, tmp, (size_t) nnz * sizeof(int), cudaMemcpyHostToDevice);
            free(tmp);
            CU(e);
        }
        CU(cudaMemcpy(*d_val, val, (size_t) nnz * sizeof(double), cudaMemcpyHostToDevice));
    }
    return ACG_SUCCESS;
}

/* The device full storage of A as the solver takes it: A's own full storage when it has one, else the packed
 * triangle mirrored on the device (expand.cu) into the arrays acgsymcsrmatrix_dsymv_init(A, 0) would have made.
 * Columns 0-based either way; padded for the tile kernel's bulk copies.  Nothing is left allocated on failure. */
static int upload_matrix(const struct acgsymcsrmatrix *A, struct acgb200_expanded *ex, cudaStream_t stream, int *errcode)
{
    if (!A->frowptr) return acgb200_expand_upload(A, 0.0, 8, 16, ex, stream, errcode);
    memset(ex, 0, sizeof(*ex));
    int err = upload_rowptr(&ex->d_rowptr, A->frowptr, A->nprows, 8, errcode);
    if (!err) err = upload_block(&ex->d_colidx, &ex->d_a, A->fcolidx, A->fa, A->fnpnzs, A->rowidxbase, 16, errcode);
    if (!err) err = upload_rowptr(&ex->d_orowptr, A->orowptr, (int64_t) A->nborderrows + A->nghostrows, 8, errcode);
    if (!err) err = upload_block(&ex->d_ocolidx, &ex->d_oa, A->ocolidx, A->oa, A->onpnzs, A->rowidxbase, 16, errcode);
    if (err) { acgb200_expanded_free(ex); return err; }
    ex->fnnz = A->fnpnzs; ex->onnz = A->onpnzs;
    return ACG_SUCCESS;
}

/* A has full storage, or the packed triangle to build it from */
static int matrix_usable(const struct acgsymcsrmatrix *A)
{
    if (!A->frowptr && !A->rowptr) return 0;
    return !A->frowptr || (A->fcolidx && A->fa);
}

static int init_impl(struct acgsolvercuda *cg, const struct acgsymcsrmatrix *A, const struct acgcomm *comm);
static int fill_values(struct acgsolvercuda *cg, struct priv *pv, int *errcode);

int acgsolvercuda_init(
    struct acgsolvercuda *cg, const struct acgsymcsrmatrix *A,
    cublasHandle_t cublas, cusparseHandle_t cusparse, const struct acgcomm *comm)
{
    (void) cublas; (void) cusparse;
    memset(cg, 0, sizeof(*cg));
    cfg_load();
    /* without full storage (no acgsymcsrmatrix_dsymv_init call) the packed triangle is expanded on the device */
    if (!matrix_usable(A)) return ACG_ERR_INVALID_VALUE;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev < 1) return ACG_ERR_CUDA;   /* no CPU fallback */
    int err = init_impl(cg, A, comm);
    if (err) acgsolvercuda_free(cg);       /* releases whatever was set up before the failure */
    return err;
}

static int init_impl(struct acgsolvercuda *cg, const struct acgsymcsrmatrix *A, const struct acgcomm *comm)
{
    int errcode_ = 0, *errcode = &errcode_;
    int commsize = 1;
    struct priv *pv = calloc(1, sizeof(*pv));
    if (!pv) return ACG_ERR_ERRNO;
    pv->key = cg;
    pv->cheb_baddiag = -1;              /* D^-1 is made at the first Chebyshev solve */
    priv_add(pv);

    /* host-side work vectors, as the reference keeps them (acg/cgcuda.c:145-153) */
    OK(acgsymcsrmatrix_vector(A, &cg->r)); acgvector_setzero(&cg->r);
    OK(acgsymcsrmatrix_vector(A, &cg->p)); acgvector_setzero(&cg->p);
    OK(acgsymcsrmatrix_vector(A, &cg->t)); acgvector_setzero(&cg->t);

    cg->halo = calloc(1, sizeof(*cg->halo));            /* zeroed: acgsolvercuda_free may run before they are filled */
    cg->haloexchange = calloc(1, sizeof(*cg->haloexchange));
    if (!cg->halo || !cg->haloexchange) return ACG_ERR_ERRNO;
    OK(acgsymcsrmatrix_halo(A, cg->halo));
    {
        /* communication kernels are tiny and latency-critical: give their streams
         * the highest priority so they are scheduled ahead of SpMV CTAs */
        int plo = 0, phi = 0;
        CU(cudaDeviceGetStreamPriorityRange(&plo, &phi));
        CU(cudaStreamCreateWithPriority(&pv->stream, cudaStreamNonBlocking, plo));
        CU(cudaStreamCreateWithPriority(&pv->commstream, cudaStreamNonBlocking, phi));
        CU(cudaStreamCreateWithPriority(&pv->redstream, cudaStreamNonBlocking, phi));
    }
    CU(cudaEventCreateWithFlags(&pv->ev_ready, cudaEventDisableTiming));
    CU(cudaEventCreateWithFlags(&pv->ev_halo, cudaEventDisableTiming));
    CU(cudaEventCreateWithFlags(&pv->ev_red, cudaEventDisableTiming));
    for (int i = 0; i < 2; i++) CU(cudaEventCreateWithFlags(&pv->ev_poll[i], cudaEventDisableTiming));
    CU(cudaEventCreate(&pv->ev_t0));
    CU(cudaEventCreate(&pv->ev_t1));
    OK(acghaloexchange_init_cuda(cg->haloexchange, cg->halo, ACG_DOUBLE, ACG_DOUBLE, comm, pv->commstream));
    cg->use_nvshmem = 0;
    if (comm && comm->type == acgcomm_nvshmem) return ACG_ERR_NVSHMEM_NOT_SUPPORTED;
    {
        /* a second communicator lets the pipelined allreduce run concurrently
         * with the halo exchange (operations on one NCCL communicator are
         * serialised).  Collective: every rank calls acgsolvercuda_init. */
        OK(acgcomm_size(comm, &commsize));
        if (cfg.redstream && commsize > 1 && comm->type == acgcomm_nccl) {
            int rank = 0;
            OK(acgcomm_rank(comm, &rank));
            ncclComm_t dup = NULL;
            ncclResult_t r = ncclCommSplit(comm->ncclcomm, 0, rank, &dup, NULL);
            if (r != ncclSuccess) { *errcode = (int) r; return ACG_ERR_NCCL; }
            OK(acgcomm_init_nccl(&pv->redcomm, dup, errcode));
            pv->have_redcomm = 1;
        }
        /* peer-memory exchange; all ranks must agree on whether it is usable */
        if (cfg.p2p && commsize > 1 && comm->type == acgcomm_nccl && pv->have_redcomm) {
            int perr = 0;
            int ok = acgb200_p2p_init(&pv->p2p, cg->halo, A->borderrowoffset, A->nborderrows, comm, pv->stream, &perr) == ACG_SUCCESS;
            if (!ok) (void) cudaGetLastError();
            int *d_ok = NULL, allok = 0;
            CU(cudaMalloc((void **) &d_ok, sizeof(int)));
            { cudaError_t ce0 = cudaMemcpy(d_ok, &ok, sizeof(int), cudaMemcpyHostToDevice); if (ce0) { cudaFree(d_ok); CU(ce0); } }
            ncclResult_t r = ncclAllReduce(d_ok, d_ok, 1, ncclInt, ncclMin, comm->ncclcomm, pv->stream);
            if (r != ncclSuccess) { cudaFree(d_ok); *errcode = (int) r; return ACG_ERR_NCCL; }
            cudaError_t ce = cudaMemcpyAsync(&allok, d_ok, sizeof(int), cudaMemcpyDeviceToHost, pv->stream);
            if (!ce) ce = cudaStreamSynchronize(pv->stream);
            cudaFree(d_ok);
            CU(ce);
            if (ok) {
                pv->p2p.h_desc.fuse = cfg.p2p_fuse;
                CU(cudaMemcpy(&pv->p2p.d_desc->fuse, &pv->p2p.h_desc.fuse, sizeof(int), cudaMemcpyHostToDevice));
            }
            if (!allok) {
                if (getenv("ACGB200_VERBOSE")) fprintf(stderr, "acgb200: peer-memory exchange unavailable (cuda error %d), using NCCL\n", perr);
                pv->p2p.enabled = 0;
            }
        }
    }

    pv->commsize = commsize;
    pv->nrows = A->nrows; pv->nowned = A->nownedrows; pv->ninner = A->ninnerrows; pv->nborder = A->nborderrows;
    pv->nghost = A->nghostrows; pv->borderoff = A->borderrowoffset;
    pv->nvec = cg->r.num_nonzeros;

    /* device scalars and control block */
    CU(cudaMalloc((void **) &pv->d_st, sizeof(*pv->d_st)));
    CU(cudaMemset(pv->d_st, 0, sizeof(*pv->d_st)));
    CU(cudaMallocHost((void **) &pv->h_ctrl, 2 * sizeof(*pv->h_ctrl)));
    CU(cudaMallocHost(&pv->h_st, staging_bytes()));

    /* device vectors: owned + ghost entries, padded to an even count */
    const size_t vbytes = ((size_t) pv->nvec + 2) * sizeof(double);
    CU(cudaMalloc((void **) &cg->d_r, vbytes)); CU(cudaMemset(cg->d_r, 0, vbytes));
    pv->d_r_id = cg->d_r;
    CU(cudaMalloc((void **) &cg->d_p, vbytes)); CU(cudaMemset(cg->d_p, 0, vbytes));
    CU(cudaMalloc((void **) &cg->d_t, vbytes)); CU(cudaMemset(cg->d_t, 0, vbytes));

    /* local block (rows [0,nowned) of the full storage) and border x ghost block */
    struct acgb200_expanded ex;
    OK(upload_matrix(A, &ex, pv->stream, errcode));
    cg->d_rowptr = ex.d_rowptr; cg->d_colidx = ex.d_colidx; cg->d_a = ex.d_a;
    cg->d_orowptr = ex.d_orowptr; cg->d_ocolidx = ex.d_ocolidx; cg->d_oa = ex.d_oa;
    pv->fnnz = ex.fnnz; pv->onnz = ex.onnz;
    const int64_t *frp = A->frowptr;          /* host row pointers / columns of the local block, for the plans */
    const acgidx_t *fcol = A->fcolidx;
    int64_t *frp_tmp = NULL;
    acgidx_t *fcol_tmp = NULL;
    if (!A->frowptr) {
        /* the caller did not build full storage: the packed triangle (half the bytes) was mirrored on the device,
         * and the planners work on the host -- row pointers always, columns only for the pattern dictionary */
        pv->device_expanded = 1;
        int *t = malloc(((size_t) A->nprows + 1) * sizeof(*t));
        frp_tmp = malloc(((size_t) A->nprows + 1) * sizeof(*frp_tmp));
        if (!t || !frp_tmp) { free(t); free(frp_tmp); return ACG_ERR_ERRNO; }
        cudaError_t ce = cudaMemcpy(t, cg->d_rowptr, ((size_t) A->nprows + 1) * sizeof(int), cudaMemcpyDeviceToHost);
        for (int64_t i = 0; i <= A->nprows; i++) frp_tmp[i] = t[i];
        free(t);
        if (!ce && cfg.spmv_slices && ex.fnnz > 0) {
            fcol_tmp = malloc((size_t) ex.fnnz * sizeof(*fcol_tmp));
            if (!fcol_tmp) { free(frp_tmp); return ACG_ERR_ERRNO; }
            ce = cudaMemcpy(fcol_tmp, cg->d_colidx, (size_t) ex.fnnz * sizeof(int), cudaMemcpyDeviceToHost);
        }
        if (ce) { free(frp_tmp); free(fcol_tmp); *errcode = (int) ce; return ACG_ERR_CUDA; }
        frp = frp_tmp; fcol = fcol_tmp;
    }
    const int colbase = A->frowptr ? A->rowidxbase : 0;     /* device-expanded columns are 0-based */

    /* SpMV tile plan */
    int64_t maxlen = 0;
    for (acgidx_t i = 0; i < A->nownedrows; i++) {
        const int64_t len = frp[i + 1] - frp[i];
        if (len > maxlen) maxlen = len;
    }
    acgb200_spmv_choose(&pv->plan, A->nownedrows, frp[A->nownedrows], maxlen);
    if (cfg.spmv_lanes > 0) pv->plan.lanes_per_row = cfg.spmv_lanes;
    if (cfg.spmv_nnz_cap > 0) pv->plan.nnz_cap = cfg.spmv_nnz_cap;
    if (cfg.spmv_rows_cap > 0) pv->plan.rows_cap = cfg.spmv_rows_cap;
    if (cfg.spmv_stages > 0) pv->plan.nstages = cfg.spmv_stages > 8 ? 8 : cfg.spmv_stages;
    if (cfg.spmv_threads > 0) pv->plan.threads = cfg.spmv_threads;
    if (cfg.spmv_unroll > 0) pv->plan.unroll = cfg.spmv_unroll;
    pv->plan.med_thr = cfg.spmv_medium;
    {
        struct acgb200_patterns pat;
        struct acgb200_sliceplan sp;
        memset(&pat, 0, sizeof(pat));
        memset(&sp, 0, sizeof(sp));
        int err = ACG_SUCCESS;
        if (cfg.spmv_slices && colbase == 0 && fcol)
            err = acgb200_patterns_build(A->nownedrows, frp, fcol, 4096, &pat);
        if (!err && cfg.spmv_slices && pat.npat > 0) {
            /* between GPUs the border rows stay with the tile kernel, which adds the border x ghost block */
            const int cover_hi = (commsize > 1 || A->nghostrows > 0) ? A->borderrowoffset : A->nownedrows;
            err = acgb200_slices_plan(A->nownedrows, cover_hi, frp, &pat, &sp);
        }
        /* irregular row lengths (power-law matrices): merge-path tiles instead of row-aligned ones for the rows
         * the slices did not take.  "Irregular": the longest row is far above the mean. */
        struct acgb200_mergeplan mp;
        memset(&mp, 0, sizeof(mp));
        if (!err && sp.nslices == 0 && cfg.spmv_merge != 0) {
            const int hi = (commsize > 1 || A->nghostrows > 0) ? A->borderrowoffset : A->nownedrows;
            const double avg = hi > 0 ? (double) frp[hi] / hi : 0.0;
            int64_t mx = 0;
            for (int i = 0; i < hi; i++) if (frp[i + 1] - frp[i] > mx) mx = frp[i + 1] - frp[i];
            if (hi >= 1024 && (cfg.spmv_merge > 0 || (double) mx > 8.0 * avg + 64.0))
                /* 2048 merged items per tile: faster on R-MAT 20 M than 1024 or 4096 */
                err = acgb200_merge_plan(hi, frp, cfg.merge_items > 0 ? cfg.merge_items : 2048, &mp);
        }
        if (!err) err = build_tiles(&pv->plan, frp, &sp, pat.patid, &mp, errcode);
        if (!err && pv->plan.nmtiles > 0) {
            pv->plan.merge_threads = cfg.merge_threads > 0 ? cfg.merge_threads : 128;
            pv->plan.merge_stages = cfg.merge_stages >= 1 && cfg.merge_stages <= SPMV_MAX_STAGES_HOST ? cfg.merge_stages : 2;
            pv->plan.merge_max_ctas = cfg.merge_max_ctas;
        }
        acgb200_mergeplan_free(&mp);
        if (!err && pv->plan.nslices > 0) {
            pv->plan.slice_domlen = sp.domlen;
            pv->plan.slice_ub_opt = cfg.slice_ub;
            pv->plan.slice_threads = cfg.slice_threads > 0 ? cfg.slice_threads : 128;
            pv->plan.slice_max_ctas = cfg.slice_max_ctas;
        }
        if (!err && pv->plan.nslices > 0 && cfg.spmv_symdiag) {
            /* mirrored diagonals: planned here, stored and checked by fill_values */
            struct acgb200_symdiag sd;
            err = acgb200_symdiag_plan(A->nownedrows, &sp, &pat, &sd);
            if (!err && sd.reason == SYMDIAG_OK) {
                struct acgb200_spmvplan *pl = &pv->plan;
                acgb200_symdiag_layout(A->nownedrows, &sd, &pl->symdiag_margin, &pl->symdiag_stride, pl->symdiag_tab);
                memcpy(pl->symdiag_d, sd.d, (size_t) sd.nd * sizeof(int));
                pl->symdiag_nd = sd.nd; pl->symdiag_no = sd.no;
                pl->symdiag_evict_first = cfg.symdiag_evict_first;
                pl->symdiag_try_codes = cfg.symdiag_codes;
            }
        }
        acgb200_sliceplan_free(&sp);
        acgb200_patterns_free(&pat);
        free(frp_tmp); free(fcol_tmp);
        if (err) return err;
    }
    pv->plan.max_ctas_per_sm = cfg.spmv_max_ctas;
    return fill_values(cg, pv, errcode);
}

/* Everything of the plan that depends on the matrix values rather than the pattern, made on the device from the
 * CSR values cg->d_a: the slice-major copy of the covered rows' values; with mirrored diagonals also those, the
 * check that every lower entry equals its mirror bit for bit and their codes; then the slice kernel's batch and
 * the grids, which depend on whether the diagonals and their codes were kept.  Run by acgsolvercuda_init and
 * again by acgsolvercuda_update_values. */
static int fill_values(struct acgsolvercuda *cg, struct priv *pv, int *errcode)
{
    struct acgb200_spmvplan *pl = &pv->plan;
    if (pl->nslices > 0) {
        if (pl->symdiag_nd > 0) {
            /* room for both layouts -- the fill builds and checks the codes from the fp64 diagonals -- and the
             * check "failed" until it has run and passed; what the values do not allow is freed below */
            const size_t ne = (size_t) pl->symdiag_nd * (size_t) pl->symdiag_stride;
            const int one = 1;
            if (!pl->d_hval) CU(cudaMalloc((void **) &pl->d_hval, ne * sizeof(double)));
            CU(cudaMalloc((void **) &pl->d_symdiag_bad, sizeof(int)));
            CU(cudaMemcpy(pl->d_symdiag_bad, &one, sizeof(int), cudaMemcpyHostToDevice));
            if (pl->symdiag_try_codes && !pl->d_hcode) CU(cudaMalloc((void **) &pl->d_hcode, ne));
            if (pl->symdiag_try_codes && !pl->d_codes) CU(cudaMalloc((void **) &pl->d_codes, sizeof(struct acgb200_codestate)));
            pl->symdiag_colidx = cg->d_colidx;
            pl->symdiag_codes = 0;
        }
        KL(acgb200_slices_fill(pl, cg->d_rowptr, cg->d_a, pv->stream));
        CU(cudaStreamSynchronize(pv->stream));
        pl->symdiag_colidx = NULL;
        if (pl->d_symdiag_bad) {
            int bad = 1;
            CU(cudaMemcpy(&bad, pl->d_symdiag_bad, sizeof(int), cudaMemcpyDeviceToHost));
            CU(cudaFree(pl->d_symdiag_bad));
            pl->d_symdiag_bad = NULL;
            int ncodes = 0;
            if (!bad && pl->d_codes) {
                /* the codes reproduce every stored double bit for bit: they replace the fp64 diagonals */
                int st[2] = { 0, 1 };
                CU(cudaMemcpy(st, (const char *) pl->d_codes + offsetof(struct acgb200_codestate, ncodes), sizeof(st),
                              cudaMemcpyDeviceToHost));
                if (st[0] >= 1 && st[0] <= ACGB200_CODES_MAX && !st[1]) ncodes = st[0];
            }
            if (bad || !ncodes) {
                /* more than 256 values, or no codes asked for: the fp64 diagonals */
                CU(cudaFree(pl->d_hcode)); CU(cudaFree(pl->d_codes));
                pl->d_hcode = NULL; pl->d_codes = NULL;
            } else {
                CU(cudaFree(pl->d_hval));
                pl->d_hval = NULL; pl->symdiag_codes = ncodes;
            }
            if (bad) {
                /* not exactly symmetric (or the check did not run): the slice kernel reads both triangles */
                CU(cudaFree(pl->d_hval));
                pl->d_hval = NULL; pl->symdiag_nd = 0; pl->symdiag_no = 0;
            }
        }
        /* batches that divide the row: |O| for the mirrored diagonals, else the most frequent row length */
        const int d = pl->symdiag_nd > 0 ? pl->symdiag_no : pl->slice_domlen;
        pl->slice_ub = pl->slice_ub_opt > 0 ? pl->slice_ub_opt
                                            : (d % 9 == 0 ? 9 : d % 7 == 0 ? 7 : d % 8 == 0 ? 8 : d % 5 == 0 ? 5 : 8);
    }
    KL(acgb200_spmv_configure(pl));
    return ACG_SUCCESS;
}

/* ACG_SUCCESS if the uploaded matrix ex has the solver's structure (row pointers and columns of both blocks),
 * ACG_ERR_INVALID_VALUE if it differs.  Compared on the device: only the first differing index comes back. */
static int same_pattern(const struct acgsolvercuda *cg, const struct priv *pv, const struct acgb200_expanded *ex,
                        int *errcode)
{
    if (ex->fnnz != pv->fnnz || ex->onnz != pv->onnz) return ACG_ERR_INVALID_VALUE;
    const int64_t nrp = (int64_t) pv->nowned + pv->nghost + 1, norp = (int64_t) pv->nborder + pv->nghost + 1;
    unsigned long long *d_first = NULL, first = 0;
    CU(cudaMalloc((void **) &d_first, sizeof(*d_first)));
    int e = (int) cudaMemsetAsync(d_first, 0xFF, sizeof(*d_first), pv->stream);
    if (!e) e = acgb200_first_diff(nrp, cg->d_rowptr, ex->d_rowptr, d_first, pv->stream);
    if (!e) e = acgb200_first_diff(pv->fnnz, cg->d_colidx, ex->d_colidx, d_first, pv->stream);
    if (!e) e = acgb200_first_diff(norp, cg->d_orowptr, ex->d_orowptr, d_first, pv->stream);
    if (!e) e = acgb200_first_diff(pv->onnz, cg->d_ocolidx, ex->d_ocolidx, d_first, pv->stream);
    if (!e) e = (int) cudaMemcpyAsync(&first, d_first, sizeof(first), cudaMemcpyDeviceToHost, pv->stream);
    if (!e) e = (int) cudaStreamSynchronize(pv->stream);
    cudaFree(d_first);
    if (e) { *errcode = e; return ACG_ERR_CUDA; }
    return first == ~0ULL ? ACG_SUCCESS : ACG_ERR_INVALID_VALUE;
}

/* ext.h: new values on the solver's pattern */
int acgsolvercuda_update_values(struct acgsolvercuda *cg, const struct acgsymcsrmatrix *A, int *errcode)
{
    int errcode_ = 0;
    if (!errcode) errcode = &errcode_;
    struct priv *pv = cg ? priv_of(cg) : NULL;
    if (!pv || !A || !matrix_usable(A)) return ACG_ERR_INVALID_VALUE;
    if (!acgb200_first_diff) return ACG_ERR_NOT_SUPPORTED;     /* the comparison kernel is linked in */
    if (A->nrows != pv->nrows || A->nownedrows != pv->nowned || A->ninnerrows != pv->ninner
        || A->nborderrows != pv->nborder || A->nghostrows != pv->nghost || A->borderrowoffset != pv->borderoff
        || (A->frowptr && (A->fnpnzs != pv->fnnz || A->onpnzs != pv->onnz)))
        return ACG_ERR_INVALID_VALUE;

    /* the new arrays go to temporaries; the solver's own change only once their structure has been found equal */
    struct acgb200_expanded ex;
    OK(upload_matrix(A, &ex, pv->stream, errcode));
    int err = same_pattern(cg, pv, &ex, errcode);
    if (!err) {
        /* in place: every pointer a kernel argument or a captured graph holds stays valid */
        cudaError_t e = cudaMemcpyAsync(cg->d_a, ex.d_a, (size_t) pv->fnnz * sizeof(double), cudaMemcpyDeviceToDevice,
                                        pv->stream);
        if (!e) e = cudaMemcpyAsync(cg->d_oa, ex.d_oa, (size_t) pv->onnz * sizeof(double), cudaMemcpyDeviceToDevice,
                                    pv->stream);
        if (!e) e = cudaStreamSynchronize(pv->stream);
        if (e) { *errcode = (int) e; err = ACG_ERR_CUDA; }
    }
    acgb200_expanded_free(&ex);
    if (err) return err;

    /* what was derived from the old values: the captured loops (their Chebyshev coefficients and the fused
     * iteration's grid among them), Chebyshev's D^-1, and the fp32 product's row chunks, which leave out the
     * mirrored diagonals' rows only while the plan keeps them */
    for (int i = 0; i < NKINDS; i++) {
        if (pv->graph[i]) cudaGraphExecDestroy(pv->graph[i]);
        pv->graph[i] = NULL; pv->graph_sig[i] = 0;
    }
    pv->cheb_graph_ab[0] = pv->cheb_graph_ab[1] = 0.0;
    pv->cheb_baddiag = -1;
    const int had_symdiag = pv->plan.symdiag_nd > 0;
    OK(fill_values(cg, pv, errcode));
    if (had_symdiag && pv->plan.symdiag_nd == 0 && pv->have_franges) {
        cudaFree(pv->d_franges);
        pv->d_franges = NULL; pv->nfranges = 0; pv->have_franges = 0;
    }
    return ACG_SUCCESS;
}

/* ------------------------------------------------------------------------ */
/* building blocks of one solve                                              */
/* ------------------------------------------------------------------------ */

struct solvectx {
    struct acgsolvercuda *cg;
    struct priv *pv;
    const struct acgcomm *comm;
    int multi, tag;
    int *errcode;
    double *d_b, *d_x;
    struct acgvector *x;      /* where solve_finish brings x back: the caller's vector, or */
    double *X;                /* the nrhs columns of the X block (host, row-major) */
    int nrhs;
    int launches;
    int capturing;            /* inside cudaStreamBeginCapture: no profiling marks */
    int p2p;                  /* loop exchanges go through peer memory */
    int mk;                   /* multi-vector loop: block width K (0: single vector) */
    enum solve_kind kind;     /* the loop iterate() runs, and so its graph slot */
    int fused;                /* pipelined loop: one fused iteration (acgb200_pcg_fused_launch); its control word
                               * alternates between ctrl[0] and ctrl[1] by iteration parity */
    int group;                /* fused pipelined loop: its group of iterations, even (DESIGN.md section 4a) */
    int issued;               /* iterations iterate() issued, inactive ones included */
    double t0;                /* host clock at the start of the solve window */
    /* Chebyshev loop: the degree, the fused inner step (acgb200_cheb_fused_step), the start's and the steps'
     * coefficients, and the r and x the r/x kernel updates (x NULL: the estimate) */
    int cheb_degree, cheb_fused;
    double cheb_c0, cheb_c[ACGB200_CHEB_MAXDEG][2];
    double *cheb_r, *cheb_x;
};

static int evpool_reserve(struct evpool *p, int n)
{
    if (n <= p->cap) return 0;
    cudaEvent_t *e = realloc(p->ev, (size_t) n * sizeof(*e));
    if (!e) return ACG_ERR_ERRNO;
    p->ev = e;
    for (int i = p->cap; i < n; i++) if (cudaEventCreate(&p->ev[i])) return ACG_ERR_CUDA;
    p->cap = n;
    return 0;
}

static void prof_mark(struct solvectx *c, struct evpool *p)
{
    if (!cfg.profile || c->capturing || p->n >= p->cap) return;
    cudaEventRecord(p->ev[p->n++], c->pv->stream);
}

static double evpool_sum_ms(struct evpool *p)
{
    double tot = 0;
    for (int i = 0; i + 1 < p->n; i += 2) {
        float ms = 0;
        if (cudaEventElapsedTime(&ms, p->ev[i], p->ev[i + 1]) == cudaSuccess) tot += ms;
    }
    return tot;
}

/* Open the timed window of a solve: profile events for up to maxits + 3 products, the counters of the last
 * solve reset, every rank past the barrier and the stream idle before the clocks start. */
static int window_open(struct solvectx *c, int maxits, double atol, double rtol, double diffatol, double diffrtol)
{
    struct acgsolvercuda *cg = c->cg;
    struct priv *pv = c->pv;
    int *errcode = c->errcode;
    if (cfg.profile) {
        OK(evpool_reserve(&pv->gemv, 2 * (maxits + 3)));
        OK(evpool_reserve(&pv->blas, 2 * (maxits + 3)));
    }
    pv->gemv.n = pv->blas.n = 0;
    cg->nsolves++; cg->niterations = 0;
    cg->bnrm2 = cg->r0nrm2 = cg->rnrm2 = cg->x0nrm2 = cg->dxnrm2 = INFINITY;
    cg->maxits = maxits; cg->diffatol = diffatol; cg->diffrtol = diffrtol;
    cg->residualatol = atol; cg->residualrtol = rtol;
    /* what acgsolvercuda_info reports of the last solve, whichever entry point runs it */
    pv->last_fused = c->fused;
    if (c->fused) pv->last_group = c->group;
    pv->last_mixed_updates = 0;
    pv->last_cheb_degree = pv->last_cheb_est = pv->last_cheb_breakdown = 0;
    pv->last_cheb_lmin = pv->last_cheb_lmax = 0;
    pv->last_spmv_ms = pv->last_blas_ms = 0; pv->last_spmv_n = 0;
    OK(acgcomm_barrier(pv->stream, c->comm, errcode));
    CU(cudaStreamSynchronize(pv->stream));
    c->t0 = wall();
    CU(cudaEventRecord(pv->ev_t0, pv->stream));
    c->launches = 0;
    return ACG_SUCCESS;
}

/* Close it: solve time on the host and device clocks, launches, and the profiled product and update times */
static int window_close(struct solvectx *c)
{
    struct acgsolvercuda *cg = c->cg;
    struct priv *pv = c->pv;
    int *errcode = c->errcode;
    CU(cudaEventRecord(pv->ev_t1, pv->stream));
    CU(cudaEventSynchronize(pv->ev_t1));
    cg->tsolve += wall() - c->t0;
    { float ms = 0; if (cudaEventElapsedTime(&ms, pv->ev_t0, pv->ev_t1) == cudaSuccess) pv->last_solve_ms = ms; }
    pv->last_launches = c->launches;
    if (cfg.profile) {
        pv->last_spmv_ms = evpool_sum_ms(&pv->gemv); pv->last_spmv_n = pv->gemv.n / 2;
        pv->last_blas_ms = evpool_sum_ms(&pv->blas);
        cg->tgemv += 1e-3 * pv->last_spmv_ms;
        cg->taxpy += 1e-3 * pv->last_blas_ms;
    }
    return ACG_SUCCESS;
}

/* offdiag_kernel's share of the epilogue of `mode` (o->acc set): add the border x ghost block to
 * y = A x, or subtract it from r = b - A x; dot over the finished rows as the SpMV kernels form it */
static void offdiag_epilogue(struct acgb200_offdiagargs *o, int mode)
{
    o->minus = (mode == SPMV_R_B_AX);
    o->dotkind = !o->acc ? 0 : (mode == SPMV_R_B_AX ? 2 : (mode == SPMV_Y_AX_DOT ? 1 : 0));
}

/* y = A x (or r = b - A x) over owned rows, including the halo exchange of x
 * and the border x ghost block when the matrix is distributed.  `acc` gets the
 * fused dot.  `gated`: take part in the device-side iteration control; 2: only
 * run when ctrl[2] is active, passing nothing on (the mixed-precision loop's
 * reliable update; the tile kernel's copy of the word goes to ctrl[3]). */
static int apply_A(struct solvectx *c, const double *x_ro, double *x_halo, double *y, const double *b,
                   int mode, double *acc, int gated, int housekeeping, int warmup, int pub_ch)
{
    struct acgsolvercuda *cg = c->cg;
    struct priv *pv = c->pv;
    int *errcode = c->errcode;
    /* loop iterations exchange ghosts through peer memory (already pushed by the
     * producer of x); set-up products (x0, r0) use the NCCL exchange */
    const int peer = c->multi && c->p2p && gated;
    if (c->multi && !peer) {
        /* the vector was produced on the main stream */
        CU(cudaEventRecord(pv->ev_ready, pv->stream));
        CU(cudaStreamWaitEvent(pv->commstream, pv->ev_ready, 0));
        OK(acghalo_exchange_cuda_begin(cg->halo, cg->haloexchange, pv->nvec, x_halo, ACG_DOUBLE,
                                       pv->nvec, x_halo, ACG_DOUBLE, c->comm, c->tag, errcode, warmup, pv->commstream));
        c->launches += 2;
    }
    struct acgb200_spmvargs a;
    memset(&a, 0, sizeof(a));
    a.plan = &pv->plan;
    a.rowptr = cg->d_rowptr; a.colidx = cg->d_colidx; a.a = cg->d_a;
    a.x = x_ro; a.y = y; a.b = b; a.acc = acc;
    a.dotrows = (c->multi && !peer) ? pv->borderoff : pv->nowned;
    a.mode = mode;
    if (gated == 2) { a.ctrl_in = &pv->d_st->ctrl[2]; a.ctrl_out = &pv->d_st->ctrl[3]; }
    else if (gated) { a.ctrl_in = &pv->d_st->ctrl[0]; a.ctrl_out = &pv->d_st->ctrl[1]; }
    a.st = pv->d_st; a.housekeeping = housekeeping;
    a.pub_ch = -1;
    const int fused = peer && pv->p2p.h_desc.fuse;
    if (peer && !fused) a.dotrows = pv->borderoff;
    if (fused) {
        /* one kernel: local block, then (for border rows) the border x ghost
         * block with ghosts read from the window, fused dot over all rows and,
         * if asked, publication of the dot to all ranks by the last CTA */
        a.p2p = pv->p2p.d_desc;
        a.od_rowoffset = pv->borderoff; a.od_nrows = pv->nborder;
        a.orowptr = cg->d_orowptr; a.ocolidx = cg->d_ocolidx; a.oa = cg->d_oa;
        if (pub_ch >= 0 && a.plan->nlong == 0 && a.plan->nmed == 0) a.pub_ch = pub_ch;
    }
    prof_mark(c, &pv->gemv);
    KL(acgb200_spmv_launch(&a, pv->stream));
    {
        /* kernels acgb200_spmv_launch issues for this plan (kernels.cu): slices | merge tiles (+ fix-up), the tile
         * kernel unless the first one forwards the control word itself, medium rows, long rows (two kernels) */
        const struct acgb200_spmvplan *pl = a.plan;
        const int first = pl->nslices > 0 || pl->nmtiles > 0;
        const int tilek = pl->ntiles > 0 || (a.ctrl_in && !(first && pl->ntiles == 0 && !a.p2p));
        c->launches += (pl->nslices > 0) + (pl->nmtiles > 0) + (pl->nmtiles > 0 && pl->nsplit > 0) + tilek
                       + (pl->nlong > 0 ? 2 : 0) + (pl->nmed > 0 ? 1 : 0);
    }
    if (c->multi && !fused) {
        if (!peer) {
            OK(acghalo_exchange_cuda_end(cg->halo, cg->haloexchange, pv->nvec, x_halo, ACG_DOUBLE,
                                         pv->nvec, x_halo, ACG_DOUBLE, c->comm, c->tag, errcode, warmup, pv->commstream));
            CU(cudaEventRecord(pv->ev_halo, pv->commstream));
            CU(cudaStreamWaitEvent(pv->stream, pv->ev_halo, 0));
        }
        struct acgb200_offdiagargs o;
        memset(&o, 0, sizeof(o));
        o.nrows = pv->nborder; o.rowoffset = pv->borderoff;
        o.orowptr = cg->d_orowptr; o.ocolidx = cg->d_ocolidx; o.oa = cg->d_oa;
        o.x = x_ro; o.y = y; o.acc = acc;
        offdiag_epilogue(&o, mode);
        if (gated) o.ctrl_in = &pv->d_st->ctrl[1];
        o.st = pv->d_st;
        o.p2p = peer ? pv->p2p.d_desc : NULL; o.p2p_iter_override = -1;
        KL(acgb200_offdiag_launch(&o, pv->stream));
        c->launches += (pv->nborder > 0);
    }
    prof_mark(c, &pv->gemv);
    return ACG_SUCCESS;
}

/* push the border entries of `vec` (and/or reduction partials) into the peers'
 * windows; see struct acgb200_postargs */
static int post(struct solvectx *c, int ctrl_slot, int iter_override, const double *vec,
                int ch, const double *redbase, int stride, int count, int par_off, int seq_off)
{
    struct priv *pv = c->pv;
    int *errcode = c->errcode;
    struct acgb200_postargs a;
    memset(&a, 0, sizeof(a));
    a.p2p = pv->p2p.d_desc;
    a.cin = &pv->d_st->ctrl[ctrl_slot]; a.st = pv->d_st;
    a.iter_override = iter_override;
    a.vec = vec; a.sendbufidx = (const int *) c->cg->haloexchange->d_sendbufidx;
    a.ch = ch; a.redbase = redbase; a.redstride = stride; a.redcount = count; a.par_off = par_off; a.seq_off = seq_off;
    KL(acgb200_comm_post(&a, pv->stream));
    c->launches += 1;
    return ACG_SUCCESS;
}

static int allreduce(struct solvectx *c, const double *src, double *dst, int count)
{
    if (!c->multi) return ACG_SUCCESS;
    return acgcomm_allreduce(src, dst, count, ACG_DOUBLE, ACG_SUM, c->pv->stream, c->comm, c->errcode);
}

/* the communicator of the one-GPU entry points */
static struct acgcomm one_gpu_comm = { .type = acgcomm_null };

/* one GPU, whole matrix: what the multi-vector, shifted, MINRES, mixed-precision and Chebyshev paths support */
static int one_gpu(const struct priv *pv, const struct acgsymcsrmatrix *A)
{
    return pv->nghost == 0 && pv->commsize == 1 && !(A && A->nghostrows > 0);
}

/* The refusals of a one-GPU entry point, in this order: an unknown solver or a missing argument
 * (ACG_ERR_INVALID_VALUE), missing kernels or a partitioned matrix (ACG_ERR_NOT_SUPPORTED), then arguments out of
 * range (ACG_ERR_INVALID_VALUE).  A refused call changes nothing. */
static int one_gpu_entry(struct acgsolvercuda *cg, const struct acgsymcsrmatrix *A, int args_given, int have_kernels,
                         int args_valid, struct priv **pv)
{
    cfg_load();
    *pv = priv_of(cg);
    if (!*pv || !args_given) return ACG_ERR_INVALID_VALUE;
    if (!have_kernels || !one_gpu(*pv, A)) return ACG_ERR_NOT_SUPPORTED;
    return args_valid ? ACG_SUCCESS : ACG_ERR_INVALID_VALUE;
}

static void ctx_init(struct solvectx *c, struct acgsolvercuda *cg, struct priv *pv, int *errcode)
{
    memset(c, 0, sizeof(*c));
    c->cg = cg; c->pv = pv; c->errcode = errcode;
}

/* global sum of a device-side reduction result, brought to the host */
static int reduce_to_host(struct solvectx *c, double *loc, double *glob, int count, double *host)
{
    int *errcode = c->errcode;
    OK(allreduce(c, loc, glob, count));
    CU(cudaMemcpyAsync(host, c->multi ? glob : loc, (size_t) count * sizeof(double), cudaMemcpyDeviceToHost, c->pv->stream));
    CU(cudaStreamSynchronize(c->pv->stream));
    return ACG_SUCCESS;
}

/* n x nrhs row-major host array <-> n x k interleaved device block (padding columns zero); with nrhs = k = 1,
 * n entries of a vector */
static int upload_block_vec(struct priv *pv, double *dst, const double *src, size_t n, int nrhs, int k, int *errcode)
{
    if (nrhs == k) {
        CU(cudaMemcpyAsync(dst, src, n * (size_t) k * sizeof(double), cudaMemcpyHostToDevice, pv->stream));
        CU(cudaStreamSynchronize(pv->stream));
        return ACG_SUCCESS;
    }
    double *tmp = calloc(n * (size_t) k + 1, sizeof(double));
    if (!tmp) return ACG_ERR_ERRNO;
    for (size_t i = 0; i < n; i++) memcpy(tmp + i * (size_t) k, src + i * (size_t) nrhs, (size_t) nrhs * sizeof(double));
    cudaError_t e = cudaMemcpyAsync(dst, tmp, n * (size_t) k * sizeof(double), cudaMemcpyHostToDevice, pv->stream);
    if (!e) e = cudaStreamSynchronize(pv->stream);
    free(tmp);
    CU(e);
    return ACG_SUCCESS;
}

static int download_block_vec(struct priv *pv, double *dst, const double *src, size_t n, int nrhs, int k, int *errcode)
{
    if (nrhs == k) {
        CU(cudaMemcpyAsync(dst, src, n * (size_t) k * sizeof(double), cudaMemcpyDeviceToHost, pv->stream));
        CU(cudaStreamSynchronize(pv->stream));
        return ACG_SUCCESS;
    }
    double *tmp = malloc((n * (size_t) k + 1) * sizeof(double));
    if (!tmp) return ACG_ERR_ERRNO;
    cudaError_t e = cudaMemcpyAsync(tmp, src, n * (size_t) k * sizeof(double), cudaMemcpyDeviceToHost, pv->stream);
    if (!e) e = cudaStreamSynchronize(pv->stream);
    if (!e) for (size_t i = 0; i < n; i++) memcpy(dst + i * (size_t) nrhs, tmp + i * (size_t) k, (size_t) nrhs * sizeof(double));
    free(tmp);
    CU(e);
    return ACG_SUCCESS;
}

/* an upload before the solve window; its host time goes to last_h2d_ms */
static int upload(struct solvectx *c, double *dst, const double *src, size_t n, int nrhs, int k)
{
    const double tb = wall();
    OK(upload_block_vec(c->pv, dst, src, n, nrhs, k, c->errcode));
    c->pv->last_h2d_ms += 1e3 * (wall() - tb);
    return ACG_SUCCESS;
}

/* a caller may hand over a longer vector than this part's owned + ghost entries: only those are used */
static size_t vec_entries(const struct priv *pv, const struct acgvector *v)
{
    return (size_t) (v->num_nonzeros < pv->nvec ? v->num_nonzeros : pv->nvec);
}

/* x0 from the caller's vector to the device */
static int upload_x0(struct solvectx *c, const struct acgvector *x)
{
    return upload(c, c->d_x, x->x, vec_entries(c->pv, x), 1, 1);
}

/* The context of a solve of vectors b, x of `kind`: b and x0 on the device */
static int solve_begin(struct solvectx *c, struct acgsolvercuda *cg, const struct acgsymcsrmatrix *A,
                       const struct acgvector *b, struct acgvector *x, double diffatol, double diffrtol,
                       struct acgcomm *comm, int tag, enum solve_kind kind, int *errcode)
{
    if (b->size < A->nrows || x->size < A->nrows || cg->r.size < A->nrows ||
        cg->p.size < A->nrows || cg->t.size < A->nrows) return ACG_ERR_INDEX_OUT_OF_BOUNDS;
    if (diffatol > 0 || diffrtol > 0) return ACG_ERR_NOT_SUPPORTED;     /* acg/cgcuda.c:424 */
    struct priv *pv = priv_of(cg);
    if (!pv) return ACG_ERR_INVALID_VALUE;
    if (b->num_nonzeros < pv->nowned || x->num_nonzeros < pv->nvec) return ACG_ERR_VECTOR_INCOMPATIBLE_SIZE;
    int commsize = 1;
    OK(acgcomm_size(comm, &commsize));
    ctx_init(c, cg, pv, errcode);
    c->comm = comm; c->multi = commsize > 1; c->tag = tag; c->kind = kind; c->x = x;
    if (c->multi && comm->type != acgcomm_nccl)
        return comm->type == acgcomm_mpi ? ACG_ERR_MPI_NOT_SUPPORTED : ACG_ERR_NVSHMEM_NOT_SUPPORTED;
    /* b and x0 to the device (acg/cgcuda.c:484-493).  The reference allocates and
     * frees the two device vectors in every solve; here they are kept with the
     * solver (their addresses are baked into the replayed CUDA graphs). */
    const size_t vbytes = ((size_t) pv->nvec + 2) * sizeof(double);
    if (!pv->d_b) {
        CU(cudaMalloc((void **) &pv->d_b, vbytes));
        CU(cudaMalloc((void **) &pv->d_x, vbytes));
        CU(cudaMemsetAsync(pv->d_b, 0, vbytes, pv->stream));
        CU(cudaMemsetAsync(pv->d_x, 0, vbytes, pv->stream));
    }
    c->d_b = pv->d_b; c->d_x = pv->d_x;
    pv->last_h2d_ms = 0;
    OK(upload(c, c->d_b, b->x, vec_entries(pv, b), 1, 1));
    return upload_x0(c, x);
}

/* The context of a solve of `kind` on the K-wide blocks; the caller uploads into them, and X gets the nrhs columns
 * of the X block back */
static void block_begin(struct solvectx *c, struct acgsolvercuda *cg, struct priv *pv, enum solve_kind kind, int K,
                        double *X, int nrhs, int *errcode)
{
    ctx_init(c, cg, pv, errcode);
    c->kind = kind; c->mk = K; c->X = X; c->nrhs = nrhs;
    c->d_b = pv->d_mb; c->d_x = pv->d_mx;
    pv->last_h2d_ms = 0;
}

/* the return-code rule of acg/cgcuda.c:1099-1107: a solve that did not converge fails unless both
 * tolerances are off */
static int convergence_status(int converged, double atol, double rtol_scaled)
{
    return !converged && !(atol == 0 && rtol_scaled == 0) ? ACG_ERR_NOT_CONVERGED : ACG_SUCCESS;
}

/* The end of every solve, after its counters are charged: ntotaliterations, the window closed, x (or the columns
 * of X) back on the host, the time of that in last_d2h_ms, and `status` unless the device reports an error */
static int solve_finish(struct solvectx *c, int status)
{
    struct priv *pv = c->pv;
    int *errcode = c->errcode;
    c->cg->ntotaliterations += c->cg->niterations;
    OK(window_close(c));
    const double te = wall();
    if (c->X) OK(download_block_vec(pv, c->X, c->d_x, (size_t) pv->nowned, c->nrhs, c->mk, errcode));
    else OK(download_block_vec(pv, c->x->x, c->d_x, vec_entries(pv, c->x), 1, 1, errcode));
    pv->last_d2h_ms = 1e3 * (wall() - te);
    CU(cudaGetLastError());
    return status;
}

/* one struct of device scalars (d_st, d_ms, d_ss, d_ns, d_xs, d_cs) from the host through the pinned staging
 * buffer h_st; both transfers are synchronous, so one buffer serves every struct */
static int scalars_push(struct solvectx *c, void *dev, const void *src, size_t bytes)
{
    int *errcode = c->errcode;
    /* everything queued before must be done with the staging buffer and with
     * the device state it is about to replace */
    CU(cudaStreamSynchronize(c->pv->stream));
    memcpy(c->pv->h_st, src, bytes);
    CU(cudaMemcpyAsync(dev, c->pv->h_st, bytes, cudaMemcpyHostToDevice, c->pv->stream));
    CU(cudaStreamSynchronize(c->pv->stream));
    return ACG_SUCCESS;
}

static int scalars_pull(struct solvectx *c, const void *dev, void *dst, size_t bytes)
{
    int *errcode = c->errcode;
    CU(cudaMemcpyAsync(c->pv->h_st, dev, bytes, cudaMemcpyDeviceToHost, c->pv->stream));
    CU(cudaStreamSynchronize(c->pv->stream));
    memcpy(dst, c->pv->h_st, bytes);
    return ACG_SUCCESS;
}

static double threshold(double atol, double rtol, double r0nrm2)
{
    /* acg/cgcuda.c:833,:1011-1012: converged if ||r|| < atol or ||r|| < rtol*||r0||,
     * each only when positive -- i.e. ||r|| < max of the enabled thresholds */
    double t = 0;
    if (atol > 0) t = atol;
    if (rtol * r0nrm2 > t) t = rtol * r0nrm2;
    return t;
}

/* the stopping test at r0 (acg/cgcuda.c:836-842): its threshold, rtol ||r0|| for convergence_status, and whether
 * r0 meets it */
static int r0_test(double atol, double rtol, double r0nrm2, double *tol, double *rtol_scaled)
{
    *tol = threshold(atol, rtol, r0nrm2);
    *rtol_scaled = rtol * r0nrm2;
    return *tol > 0 && r0nrm2 < *tol;
}

/* (b, b) into *bb and cg->bnrm2 (acg/cgcuda.c:727-739), the scalars zeroed first; `setup` (if given) is issued
 * between the two */
static int rhs_norm(struct solvectx *c, int (*setup)(struct solvectx *), double *bb)
{
    struct priv *pv = c->pv;
    int *errcode = c->errcode;
    struct acgb200_devstate h;
    memset(&h, 0, sizeof(h));
    OK(scalars_push(c, pv->d_st, &h, sizeof(h)));
    if (setup) OK(setup(c));
    KL(acgb200_dot(pv->nowned, c->d_b, c->d_b, &pv->d_st->tmp_loc[0], pv->stream));
    OK(reduce_to_host(c, &pv->d_st->tmp_loc[0], &pv->d_st->tmp[0], 1, bb));
    c->cg->bnrm2 = sqrt(*bb);
    return ACG_SUCCESS;
}

/* r = b - A x into d_r with (r, r) folded in (ungated, the scalars zeroed first), (r, r) into *rr: the r0 of
 * MINRES, mixed-precision and Chebyshev CG, and the fp64 residual of a mixed-precision x */
static int residual(struct solvectx *c, double *rr)
{
    struct priv *pv = c->pv;
    struct acgb200_devstate h;
    memset(&h, 0, sizeof(h));
    OK(scalars_push(c, pv->d_st, &h, sizeof(h)));
    *rr = 0;
    OK(apply_A(c, c->d_x, c->d_x, c->cg->d_r, c->d_b, SPMV_R_B_AX, &pv->d_st->tmp_loc[0], 0, 0, 0, -1));
    return reduce_to_host(c, &pv->d_st->tmp_loc[0], &pv->d_st->tmp[0], 1, rr);
}

/* The results of a solve of several columns (right-hand sides or shifts) from their squared norms: each column's
 * stats (if asked), the norms of the solver as those of the whole block, and the status by the rule of
 * convergence_status per column */
static int column_results(struct acgsolvercuda *cg, int ncols, const int *nits, const int *conv, const double *bb,
                          const double *rr0, const double *rr, double atol, const double *rtol_scaled,
                          struct acgb200_colstats *stats)
{
    double sb = 0, sr0 = 0, sr = 0;
    int status = ACG_SUCCESS;
    for (int j = 0; j < ncols; j++) {
        sb += bb[j]; sr0 += rr0[j]; sr += rr[j];
        if (convergence_status(conv[j], atol, rtol_scaled[j])) status = ACG_ERR_NOT_CONVERGED;
        if (stats) {
            stats[j].niterations = nits[j]; stats[j].converged = conv[j];
            stats[j].bnrm2 = sqrt(bb[j]); stats[j].r0nrm2 = sqrt(rr0[j]); stats[j].rnrm2 = sqrt(rr[j]);
        }
    }
    cg->bnrm2 = sqrt(sb); cg->r0nrm2 = sqrt(sr0); cg->rnrm2 = sqrt(sr);
    return status;
}

/* Capture iterations g ... 2g - 1 of `issue` into a graph (g = graph_group).  All
 * pointers the kernels and NCCL calls use are fixed for the life of the solver
 * and the iteration index only enters through its parity, or on the fused
 * pipelined path through its place in the group, so one graph of a group of
 * iterations serves the whole solve (and later solves). */
/* everything besides the (fixed) pointers and the solve kind (its own slot) that decides which kernels and
 * NCCL calls an iteration issues: a cached graph is only replayed for the configuration it was captured with
 * (options can change between two solves on one solver) */
static int graph_signature(const struct solvectx *c)
{
    return 1 | (c->multi ? 2 : 0) | (c->p2p ? 4 : 0) | (c->pv->p2p.h_desc.fuse ? 8 : 0) | (cfg.pdl ? 16 : 0)
           | (cfg.redstream ? 32 : 0) | (c->pv->have_redcomm ? 64 : 0) | (c->mk << 8) | (c->fused ? 1 << 16 : 0)
           | (c->cheb_degree << 18) | (c->cheb_fused ? 1 << 23 : 0) | (c->fused ? c->group << 24 : 0);
}

/* iterations per graph replay: the fused pipelined loop's group, two for every other loop */
static int graph_group(const struct solvectx *c) { return c->fused ? c->group : 2; }

static int capture_group(struct solvectx *c, int (*issue)(struct solvectx *, int))
{
    struct priv *pv = c->pv;
    int *errcode = c->errcode;
    const enum solve_kind kind = c->kind;
    if (pv->graph[kind] && pv->graph_sig[kind] == graph_signature(c)) return ACG_SUCCESS;
    if (pv->graph[kind]) { cudaGraphExecDestroy(pv->graph[kind]); pv->graph[kind] = NULL; }
    const int before = c->launches;
    cudaGraph_t g = NULL;
    c->capturing = 1;
    CU(cudaStreamBeginCapture(pv->stream, cudaStreamCaptureModeThreadLocal));
    int err = 0;
    for (int k = graph_group(c); k < 2 * graph_group(c) && !err; k++) err = issue(c, k);
    cudaError_t e = cudaStreamEndCapture(pv->stream, &g);
    c->capturing = 0;
    pv->graph_launches[kind] = c->launches - before;
    c->launches = before;
    if (err) { if (g) cudaGraphDestroy(g); return err; }
    CU(e);
    e = cudaGraphInstantiate(&pv->graph[kind], g, 0);
    cudaGraphDestroy(g);
    CU(e);
    pv->graph_sig[kind] = graph_signature(c);
    return ACG_SUCCESS;
}

/* Run `issue(c,k)` for k < maxits, polling the device control word.  The
 * first group of iterations (two, or the fused pipelined loop's group) is
 * issued directly (it also serves as the un-captured first use of every NCCL
 * path), then whole groups as replays of the graph, and the rest directly.
 * A replay may run past check_every: a converged solve then issues up to a
 * group of iterations that return at once. */
static int iterate(struct solvectx *c, int maxits, int poll, int (*issue)(struct solvectx *, int))
{
    struct priv *pv = c->pv;
    int *errcode = c->errcode;
    const enum solve_kind kind = c->kind;
    const int group = graph_group(c);
    int issued = 0, slot = 0, have_prev = 0, since_poll = 0;
    /* Replays are used on one GPU and with the peer-memory exchange (kernel nodes
     * only).  With the NCCL exchange the iteration also contains collectives on
     * two communicators and three streams; that combination ran in the
     * benchmarks but its test matrix is not closed yet, so it is only captured
     * on request (option "graph" = 2). */
    const int use_graph = cfg.graph && !cfg.profile && maxits >= 6 && (!c->multi || c->p2p || cfg.graph >= 2);
    while (issued < maxits) {
        if (use_graph && issued >= group && issued % group == 0 && maxits - issued >= group) {
            if (!pv->graph[kind] || pv->graph_sig[kind] != graph_signature(c)) OK(capture_group(c, issue));
            CU(cudaGraphLaunch(pv->graph[kind], pv->stream));
            c->launches += pv->graph_launches[kind];
            issued += group; since_poll += group;
        } else {
            OK(issue(c, issued));
            issued += 1; since_poll += 1;
        }
        if (!poll || (since_poll < cfg.check_every && issued < maxits)) continue;
        since_poll = 0;
        CU(cudaMemcpyAsync(&pv->h_ctrl[slot], &pv->d_st->ctrl[c->fused ? issued & 1 : 0], sizeof(struct acgb200_ctrl),
                           cudaMemcpyDeviceToHost, pv->stream));
        CU(cudaEventRecord(pv->ev_poll[slot], pv->stream));
        if (have_prev) {
            CU(cudaEventSynchronize(pv->ev_poll[slot ^ 1]));
            if (pv->h_ctrl[slot ^ 1].done) break;
        }
        have_prev = 1; slot ^= 1;
    }
    c->issued = issued;
    CU(cudaStreamSynchronize(pv->stream));
    if (c->multi) { CU(cudaStreamSynchronize(pv->commstream)); CU(cudaStreamSynchronize(pv->redstream)); }
    if (c->multi && c->p2p) {
        /* a kernel that waited in vain for a peer gave up instead of hanging the GPU */
        int gaveup = 0;
        OK(acgb200_p2p_timed_out(&pv->p2p, pv->stream, &gaveup));
        if (gaveup) { *errcode = (int) cudaErrorLaunchTimeout; return ACG_ERR_CUDA; }
    }
    return ACG_SUCCESS;
}

/* ------------------------------------------------------------------------ */
/* classic CG                                                                */
/* ------------------------------------------------------------------------ */

static int classic_iteration(struct solvectx *c, int k)
{
    struct acgsolvercuda *cg = c->cg;
    struct priv *pv = c->pv;
    struct acgb200_devstate *st = pv->d_st;
    int *errcode = c->errcode;
    const int s = k & 1, n = pv->nowned;
    const int peer = c->multi && c->p2p;
    double *pvec = cg->d_p;
    struct acgb200_p2pdev *desc = !peer ? NULL : pv->p2p.d_desc;
    const struct acgb200_spmvplan *pl = &pv->plan;
    OK(apply_A(c, pvec, pvec, cg->d_t, NULL, SPMV_Y_AX_DOT, &st->pap_loc[s], 1, 1, 0, 0));
    if (peer) {
        /* (p,Ap) is published by the SpMV's last CTA; with long rows the dot is
         * only complete after the finishing kernel, so a separate post does it */
        if (pl->nlong > 0 || pl->nmed > 0 || !pv->p2p.h_desc.fuse) OK(post(c, 1, -1, NULL, 0, &st->pap_loc[0], 1, 1, 0, 1));
    } else OK(allreduce(c, &st->pap_loc[s], &st->pap[s], 1));
    prof_mark(c, &pv->blas);
    KL(acgb200_cg_update_r(n, st, 1, 1, c->multi, desc, cg->d_t, cg->d_r, pv->stream));
    if (!peer) OK(allreduce(c, &st->rr_loc[s ^ 1], &st->rr[s ^ 1], 1));
    else if (!pv->p2p.h_desc.fuse) OK(post(c, 1, -1, NULL, 1, &st->rr_loc[0], 1, 1, 1, 1));
    KL(acgb200_cg_update_xp(n, st, 1, 0, c->multi, desc, cg->d_r, pvec, c->d_x, pv->stream));
    prof_mark(c, &pv->blas);
    if (peer && !pv->p2p.h_desc.fuse) OK(post(c, 0, -1, pvec, -1, NULL, 0, 0, 0, 0));     /* p for the next SpMV */
    c->launches += 2 + (c->multi && !peer ? 2 : 0);
    return ACG_SUCCESS;
}

static void account_classic(struct acgsolvercuda *cg, const struct priv *pv, int nits, int multi)
{
    /* the reference's analytic counters (acg/cgcuda.c:885-1001), per iteration */
    const int64_t n = pv->nowned, nnz = pv->fnnz + pv->onnz;
    const int64_t bgemv = nnz * 12 + n * 16 + (int64_t) (pv->nborder + pv->nghost) * 8 + (int64_t) pv->nvec * 8;
    cg->ngemv += nits; cg->nflops += (int64_t) nits * 3 * nnz; cg->Bgemv += (int64_t) nits * bgemv;
    cg->ndot += nits; cg->nflops += (int64_t) nits * 2 * n; cg->Bdot += (int64_t) nits * 16 * n;
    cg->nnrm2 += nits; cg->nflops += (int64_t) nits * 2 * n; cg->Bnrm2 += (int64_t) nits * 8 * n;
    cg->naxpy += 3 * (int64_t) nits; cg->nflops += (int64_t) nits * 6 * n; cg->Baxpy += (int64_t) nits * 48 * n;
    if (multi) {
        cg->nallreduce += 2 * (int64_t) nits; cg->Ballreduce += (int64_t) nits * 16;
        cg->nhalo += nits; cg->Bhalo += (int64_t) nits * cg->halo->sendsize * 8;
        cg->nhalomsgs += (int64_t) nits * cg->halo->nrecipients;
    }
}

int acgsolvercuda_solvempi(
    struct acgsolvercuda *cg, const struct acgsymcsrmatrix *A,
    const struct acgvector *b, struct acgvector *x,
    int maxits, double diffatol, double diffrtol, double residualatol, double residualrtol,
    int warmup, struct acgcomm *comm, int tag, int *errcode,
    cublasHandle_t cublas, cusparseHandle_t cusparse, cusparseSpMVAlg_t alg)
{
    (void) cublas; (void) cusparse; (void) alg;
    int errcode_ = 0;
    if (!errcode) errcode = &errcode_;
    cfg_load();
    struct solvectx c;
    OK(solve_begin(&c, cg, A, b, x, diffatol, diffrtol, comm, tag, KIND_CLASSIC, errcode));
    struct priv *pv = c.pv;
    struct acgb200_devstate *st = pv->d_st;
    const int n = pv->nowned;
    struct acgb200_devstate h;

    c.p2p = c.multi && pv->p2p.enabled && cfg.p2p;
    /* a rank that is ahead must not store into a peer's window while that peer's kernels of the
     * previous solve are still reading it: order the first post of this solve behind every rank */
    if (c.p2p) OK(acgcomm_barrier(pv->stream, comm, errcode));
    double *const pvec = cg->d_p;
    /* warm-up: `warmup` full iterations (every kernel, every communication path)
     * on state that is overwritten below (acg/cgcuda.c:607-705); d_r stands in
     * for x so the initial guess is untouched */
    if (warmup > 0) {
        memset(&h, 0, sizeof(h));
        h.maxits = warmup; h.rr_loc[0] = h.rr[0] = 1.0;
        OK(scalars_push(&c, pv->d_st, &h, sizeof(h)));
        double *xsave = c.d_x; c.d_x = cg->d_r;
        if (c.p2p) {
            OK(acgb200_p2p_begin(&pv->p2p, warmup, pv->stream));
            OK(post(&c, 0, 0, pvec, -1, NULL, 0, 0, 0, 0));
        }
        for (int i = 0; i < warmup; i++) OK(classic_iteration(&c, i));
        c.d_x = xsave;
        KL(acgb200_dot(n, c.d_b, c.d_b, &st->tmp_loc[0], pv->stream));
        CU(cudaStreamSynchronize(pv->stream));
    }
    OK(window_open(&c, maxits, residualatol, residualrtol, diffatol, diffrtol));

    double bb = 0, rr0 = 0, tol = 0, rtol_scaled = 0;
    OK(rhs_norm(&c, NULL, &bb));
    cg->nnrm2++; cg->nflops += 2 * (int64_t) n; cg->Bnrm2 += 8 * (int64_t) n;

    /* r0 = b - A x0 with (r0,r0) folded in (acg/cgcuda.c:761-799,:819-832); p = r0 */
    OK(apply_A(&c, c.d_x, c.d_x, cg->d_r, c.d_b, SPMV_R_B_AX, &st->rr_loc[0], 0, 0, 0, -1));
    CU(cudaMemcpyAsync(pvec, cg->d_r, (size_t) n * sizeof(double), cudaMemcpyDeviceToDevice, pv->stream));
    OK(reduce_to_host(&c, &st->rr_loc[0], &st->rr[0], 1, &rr0));
    cg->rnrm2 = cg->r0nrm2 = sqrt(rr0);
    cg->ngemv++; cg->ncopy += 2; cg->nnrm2++;
    int converged = r0_test(residualatol, residualrtol, cg->r0nrm2, &tol, &rtol_scaled);

    if (!converged && maxits > 0) {
        memset(&h, 0, sizeof(h));
        h.maxits = maxits; h.tol = tol;
        h.rr_loc[0] = h.rr[0] = rr0;
        OK(scalars_push(&c, pv->d_st, &h, sizeof(h)));
        if (c.p2p) {
            /* p_0 = r_0 goes to the neighbours' windows as exchange number 0 */
            OK(acgb200_p2p_begin(&pv->p2p, maxits, pv->stream));
            OK(post(&c, 0, 0, pvec, -1, NULL, 0, 0, 0, 0));
        }
        OK(iterate(&c, maxits, tol > 0, classic_iteration));
        OK(scalars_pull(&c, pv->d_st, &h, sizeof(h)));
        cg->niterations = h.ctrl[0].iter;
        converged = h.ctrl[0].done;
        const double rr = converged ? h.final_rr
            : (c.multi ? h.rr[cg->niterations & 1] : h.rr_loc[cg->niterations & 1]);
        cg->rnrm2 = sqrt(rr);
    }
    account_classic(cg, pv, cg->niterations, c.multi);
    return solve_finish(&c, convergence_status(converged, residualatol, rtol_scaled));
}

int acgsolvercuda_solve(
    struct acgsolvercuda *cg, const struct acgsymcsrmatrix *A,
    const struct acgvector *b, struct acgvector *x,
    int maxits, double diffatol, double diffrtol, double residualatol, double residualrtol, int warmup)
{
    int errcode = 0;
    return acgsolvercuda_solvempi(cg, A, b, x, maxits, diffatol, diffrtol, residualatol, residualrtol,
                                  warmup, &one_gpu_comm, 0, &errcode, NULL, NULL, 0);
}

/* ------------------------------------------------------------------------ */
/* several right-hand sides: classic CG per column, one matrix pass for all  */
/* ------------------------------------------------------------------------ */

/* the multi-vector kernels are linked in (see ACGB200_MULTI_LAUNCHER, internal.h) */
static int have_multi_kernels(void)
{
    return acgb200_spmm_launch && acgb200_cg_multi_update_r && acgb200_cg_multi_update_xp && acgb200_dot_multi;
}

static int block_width(int nrhs) { return nrhs <= 1 ? 1 : nrhs <= 2 ? 2 : nrhs <= 4 ? 4 : 8; }

/* Rows the pattern slices do not cover, as chunks for spmm_rows_kernel: made once from the single-vector
 * plan (its slices; every other row -- tile, merge, medium, long -- goes to the chunks).  Lanes per row
 * from the mean length of those rows. */
#define SPMM_CHUNK_LANES 128
/* (all rows if !use_slices: the fp32 product of a plan without mirrored diagonals) */
static int row_chunks(struct priv *pv, const struct acgsolvercuda *cg, int use_slices, int **d_out, int *nr_out,
                      int *lanes_out, int *errcode)
{
    const int n = pv->nowned, nsl = use_slices ? pv->plan.nslices : 0;
    unsigned char *cov = calloc((size_t) n + 1, 1);
    int *rp = malloc(((size_t) n + 1) * sizeof(int));
    struct acgb200_slice *sl = nsl > 0 ? malloc((size_t) nsl * sizeof(*sl)) : NULL;
    int *rg = malloc(((size_t) n + 1) * 2 * sizeof(int));
    if (!cov || !rp || (nsl > 0 && !sl) || !rg) { free(cov); free(rp); free(sl); free(rg); return ACG_ERR_ERRNO; }
    cudaError_t e = cudaMemcpy(rp, cg->d_rowptr, ((size_t) n + 1) * sizeof(int), cudaMemcpyDeviceToHost);
    if (!e && nsl > 0) e = cudaMemcpy(sl, pv->plan.d_slices, (size_t) nsl * sizeof(*sl), cudaMemcpyDeviceToHost);
    if (e) { free(cov); free(rp); free(sl); free(rg); *errcode = (int) e; return ACG_ERR_CUDA; }
    for (int s = 0; s < nsl; s++)
        for (int r = sl[s].row0; r < sl[s].row0 + 32 && r < n; r++) cov[r] = 1;
    int64_t urows = 0, unnz = 0;
    for (int r = 0; r < n; r++) if (!cov[r]) { urows++; unnz += rp[r + 1] - rp[r]; }
    const int lanes = urows > 0 && unnz > 12 * urows ? 8 : 1;
    const int chunk = SPMM_CHUNK_LANES / lanes;      /* rows per chunk: four passes of a warp */
    int nr = 0;
    for (int r = 0; r < n;) {
        if (cov[r]) { r++; continue; }
        const int r0 = r;
        while (r < n && !cov[r] && r - r0 < chunk) r++;
        rg[2 * nr] = r0; rg[2 * nr + 1] = r; nr++;
    }
    if (nr > 0) {
        e = cudaMalloc((void **) d_out, (size_t) nr * 2 * sizeof(int));
        if (!e) e = cudaMemcpy(*d_out, rg, (size_t) nr * 2 * sizeof(int), cudaMemcpyHostToDevice);
    }
    free(cov); free(rp); free(sl); free(rg);
    CU(e);
    *nr_out = nr; *lanes_out = lanes;
    return ACG_SUCCESS;
}

static int build_ranges(struct priv *pv, const struct acgsolvercuda *cg, int *errcode)
{
    if (pv->have_ranges) return ACG_SUCCESS;
    OK(row_chunks(pv, cg, 1, &pv->d_ranges, &pv->nranges, &pv->ranges_lanes, errcode));
    pv->have_ranges = 1;
    return ACG_SUCCESS;
}

/* per-column state and block vectors of width >= k, kept with the solver; a wider request replaces the
 * blocks (and the captured multi-vector loop, whose pointers they were) */
static int ensure_blocks(struct priv *pv, const struct acgsolvercuda *cg, int k, int *errcode)
{
    OK(dev_scalars_once(pv, (void **) &pv->d_ms, sizeof(*pv->d_ms), errcode));
    OK(build_ranges(pv, cg, errcode));
    if (pv->mk >= k) return ACG_SUCCESS;
    double **blk[5] = { &pv->d_mx, &pv->d_mb, &pv->d_mr, &pv->d_mp, &pv->d_mt };
    for (int i = 0; i < 5; i++) { cudaFree(*blk[i]); *blk[i] = NULL; }
    const enum solve_kind blockloops[2] = { KIND_MULTI, KIND_SHIFTED };
    for (int i = 0; i < 2; i++)
        if (pv->graph[blockloops[i]]) { cudaGraphExecDestroy(pv->graph[blockloops[i]]); pv->graph[blockloops[i]] = NULL; }
    pv->mk = 0;
    /* one spare row: the BLAS-1 kernels read pairs of entries */
    const size_t bytes = ((size_t) pv->nowned + 1) * (size_t) k * sizeof(double);
    for (int i = 0; i < 5; i++) {
        CU(cudaMalloc((void **) blk[i], bytes));
        CU(cudaMemsetAsync(*blk[i], 0, bytes, pv->stream));
    }
    pv->mk = k;
    return ACG_SUCCESS;
}

/* the multi-vector product of block x into block y (see struct acgb200_spmmargs) */
static int apply_A_multi(struct solvectx *c, const double *x, double *y, const double *b, int mode, double *acc, int gated)
{
    struct acgsolvercuda *cg = c->cg;
    struct priv *pv = c->pv;
    int *errcode = c->errcode;
    struct acgb200_spmmargs a;
    memset(&a, 0, sizeof(a));
    a.plan = &pv->plan; a.k = c->mk;
    a.nranges = pv->nranges; a.ranges = pv->d_ranges; a.lanes = pv->ranges_lanes;
    a.rowptr = cg->d_rowptr; a.colidx = cg->d_colidx; a.a = cg->d_a;
    a.x = x; a.y = y; a.b = b; a.acc = acc; a.mode = mode;
    a.st = pv->d_st;
    if (gated) { a.ctrl_in = &pv->d_st->ctrl[0]; a.ctrl_out = &pv->d_st->ctrl[1]; a.ms = pv->d_ms; }
    prof_mark(c, &pv->gemv);
    KL(acgb200_spmm_launch(&a, pv->stream));
    prof_mark(c, &pv->gemv);
    c->launches += (pv->plan.nslices > 0) + (pv->nranges > 0 || (gated && pv->plan.nslices == 0));
    return ACG_SUCCESS;
}

/* one iteration of the K recurrences: T = A P (+ p_j.t_j), R -= alpha T (+ r_j.r_j), X += alpha P ; P = R + beta P */
static int multi_iteration(struct solvectx *c, int k)
{
    struct priv *pv = c->pv;
    struct acgb200_mstate *ms = pv->d_ms;
    int *errcode = c->errcode;
    const int s = k & 1, n = pv->nowned;
    OK(apply_A_multi(c, pv->d_mp, pv->d_mt, NULL, SPMV_Y_AX_DOT, &ms->pap[s][0], 1));
    prof_mark(c, &pv->blas);
    KL(acgb200_cg_multi_update_r(n, c->mk, pv->d_st, ms, 1, 1, pv->d_mt, pv->d_mr, pv->stream));
    KL(acgb200_cg_multi_update_xp(n, c->mk, pv->d_st, ms, 1, 0, pv->d_mr, pv->d_mp, c->d_x, pv->stream));
    prof_mark(c, &pv->blas);
    c->launches += 2;
    return ACG_SUCCESS;
}

static void account_multi(struct acgsolvercuda *cg, const struct priv *pv, int nits, int k)
{
    /* per iteration: one pass over the matrix for K vectors, K columns of BLAS-1 */
    const int64_t n = pv->nowned, nnz = pv->fnnz + pv->onnz, kk = k;
    cg->ngemv += nits; cg->nflops += (int64_t) nits * 3 * nnz * kk;
    cg->Bgemv += (int64_t) nits * (nnz * 12 + n * 4 + kk * n * 24);
    cg->ndot += nits * kk; cg->nflops += (int64_t) nits * 2 * n * kk; cg->Bdot += (int64_t) nits * 16 * n * kk;
    cg->nnrm2 += nits * kk; cg->nflops += (int64_t) nits * 2 * n * kk; cg->Bnrm2 += (int64_t) nits * 8 * n * kk;
    cg->naxpy += 3 * (int64_t) nits * kk; cg->nflops += (int64_t) nits * 6 * n * kk; cg->Baxpy += (int64_t) nits * 48 * n * kk;
}

int acgsolvercuda_solve_multi(struct acgsolvercuda *cg, const struct acgsymcsrmatrix *A,
                              int nrhs, const double *B, double *X, int maxits, double residualatol, double residualrtol,
                              int warmup, struct acgb200_colstats *stats)
{
    int errcode_ = 0, *errcode = &errcode_;
    struct priv *pv;
    OK(one_gpu_entry(cg, A, 1, have_multi_kernels(), nrhs >= 1 && nrhs <= ACGB200_MAXK && B && X && maxits >= 0, &pv));
    const int K = block_width(nrhs), n = pv->nowned;
    OK(ensure_blocks(pv, cg, K, errcode));
    struct solvectx c;
    block_begin(&c, cg, pv, KIND_MULTI, K, X, nrhs, errcode);
    OK(upload(&c, c.d_b, B, (size_t) n, nrhs, K));
    OK(upload(&c, c.d_x, X, (size_t) n, nrhs, K));
    struct acgb200_devstate h;
    struct acgb200_mstate m;

    /* warm-up: `warmup` iterations of every column on state that is overwritten below; R stands in for X
     * (as d_r does in acgsolvercuda_solvempi), so the initial guesses are untouched */
    if (warmup > 0) {
        memset(&m, 0, sizeof(m));
        for (int j = 0; j < ACGB200_MAXK; j++) m.rr[0][j] = 1.0;
        OK(scalars_push(&c, pv->d_ms, &m, sizeof(m)));
        memset(&h, 0, sizeof(h));
        h.maxits = warmup; h.ctrl[0].pad0 = (1 << K) - 1;
        OK(scalars_push(&c, pv->d_st, &h, sizeof(h)));
        c.d_x = pv->d_mr;
        for (int i = 0; i < warmup; i++) OK(multi_iteration(&c, i));
        c.d_x = pv->d_mx;
        KL(acgb200_dot_multi(n, K, pv->d_mb, &pv->d_ms->tmp[0], pv->stream));
        CU(cudaStreamSynchronize(pv->stream));
    }
    OK(window_open(&c, maxits, residualatol, residualrtol, 0, 0));

    /* ||b_j|| ; r0 = B - A X0 with (r0_j,r0_j) folded in ; P = R */
    memset(&h, 0, sizeof(h));
    OK(scalars_push(&c, pv->d_st, &h, sizeof(h)));
    memset(&m, 0, sizeof(m));
    OK(scalars_push(&c, pv->d_ms, &m, sizeof(m)));
    KL(acgb200_dot_multi(n, K, pv->d_mb, &pv->d_ms->tmp[0], pv->stream));
    OK(apply_A_multi(&c, pv->d_mx, pv->d_mr, pv->d_mb, SPMV_R_B_AX, &pv->d_ms->rr[0][0], 0));
    CU(cudaMemcpyAsync(pv->d_mp, pv->d_mr, (size_t) n * K * sizeof(double), cudaMemcpyDeviceToDevice, pv->stream));
    OK(scalars_pull(&c, pv->d_ms, &m, sizeof(m)));
    c.launches += 1;
    double bb[ACGB200_MAXK], rr0[ACGB200_MAXK], tol[ACGB200_MAXK], rtol_scaled[ACGB200_MAXK];
    unsigned mask = 0;
    int poll = 0;
    for (int j = 0; j < nrhs; j++) {
        bb[j] = m.tmp[j]; rr0[j] = m.rr[0][j];
        if (!r0_test(residualatol, residualrtol, sqrt(rr0[j]), &tol[j], &rtol_scaled[j])) mask |= 1u << j;
        if (tol[j] > 0) poll = 1;
    }
    int nits[ACGB200_MAXK], conv[ACGB200_MAXK];
    double rr[ACGB200_MAXK];
    for (int j = 0; j < nrhs; j++) { nits[j] = 0; conv[j] = !(mask >> j & 1u); rr[j] = rr0[j]; }
    if (maxits > 0 && mask) {
        memset(&m, 0, sizeof(m));
        for (int j = 0; j < nrhs; j++) { m.tol[j] = tol[j]; m.rr[0][j] = rr0[j]; m.final_rr[j] = rr0[j]; }
        OK(scalars_push(&c, pv->d_ms, &m, sizeof(m)));
        memset(&h, 0, sizeof(h));
        h.maxits = maxits; h.ctrl[0].pad0 = (int) mask;
        OK(scalars_push(&c, pv->d_st, &h, sizeof(h)));
        OK(iterate(&c, maxits, poll, multi_iteration));
        OK(scalars_pull(&c, pv->d_st, &h, sizeof(h)));
        OK(scalars_pull(&c, pv->d_ms, &m, sizeof(m)));
        cg->niterations = h.ctrl[0].iter;
        for (int j = 0; j < nrhs; j++)
            if (mask >> j & 1u) { nits[j] = m.nits[j]; conv[j] = m.conv[j]; rr[j] = m.final_rr[j]; }
    }
    account_multi(cg, pv, cg->niterations, K);
    cg->ngemv++; cg->ncopy += 1; cg->nnrm2 += 2 * nrhs;
    return solve_finish(&c, column_results(cg, nrhs, nits, conv, bb, rr0, rr, residualatol, rtol_scaled, stats));
}

/* ------------------------------------------------------------------------ */
/* shifted systems: one seed CG on A drives every (A + sigma_j I) x_j = b    */
/* ------------------------------------------------------------------------ */

/* the shift kernels are linked in (see ACGB200_MULTI_LAUNCHER, internal.h) */
static int have_shift_kernels(void)
{
    return have_multi_kernels() && acgb200_shift_setup && acgb200_cg_shift_update;
}

/* 1 ... ACGB200_MAXK shifts, each finite and >= 0 */
static int valid_shifts(int nshifts, const double *shifts)
{
    if (nshifts < 1 || nshifts > ACGB200_MAXK || !shifts) return 0;
    for (int j = 0; j < nshifts; j++) if (!(isfinite(shifts[j]) && shifts[j] >= 0)) return 0;
    return 1;
}

/* r = p = b, X = 0 (X: c->d_x) and P_j = b */
static int shifted_setup(struct solvectx *c)
{
    int *errcode = c->errcode;
    KL(acgb200_shift_setup(c->pv->nowned, c->mk, c->d_b, c->cg->d_r, c->cg->d_p, c->d_x, c->pv->d_mp, c->pv->stream));
    return ACG_SUCCESS;
}

/* the state of iteration 0: zeta_0 = zeta_{-1} = 1, alpha_{-1} = 1, beta_{-1} = 0 */
static void sstate_init(struct acgb200_sstate *ss, int nshifts, const double *shifts, double tol, double r0nrm2)
{
    memset(ss, 0, sizeof(*ss));
    for (int j = 0; j < ACGB200_MAXK; j++) { ss->zeta[0][j] = 1.0; ss->zeta_prev[0][j] = 1.0; }
    ss->ab_prev[0][0] = 1.0; ss->ab_prev[0][1] = 0.0;
    for (int j = 0; j < nshifts; j++) { ss->sigma[j] = shifts[j]; ss->tol[j] = tol; ss->final_rnrm2[j] = r0nrm2; }
}

/* one seed iteration and the shift updates: t = A p (+ p.t), r -= alpha t (+ r.r), then
 * p = r + beta p and X_j += alpha_j P_j ; P_j = zeta_j r + beta_j P_j */
static int shifted_iteration(struct solvectx *c, int k)
{
    struct acgsolvercuda *cg = c->cg;
    struct priv *pv = c->pv;
    struct acgb200_devstate *st = pv->d_st;
    int *errcode = c->errcode;
    const int s = k & 1, n = pv->nowned;
    OK(apply_A(c, cg->d_p, cg->d_p, cg->d_t, NULL, SPMV_Y_AX_DOT, &st->pap_loc[s], 1, 1, 0, 0));
    prof_mark(c, &pv->blas);
    KL(acgb200_cg_update_r(n, st, 1, 1, 0, NULL, cg->d_t, cg->d_r, pv->stream));
    KL(acgb200_cg_shift_update(n, c->mk, st, pv->d_ss, 1, 0, cg->d_r, cg->d_p, c->d_x, pv->d_mp, pv->stream));
    prof_mark(c, &pv->blas);
    c->launches += 2;
    return ACG_SUCCESS;
}

static void account_shifted(struct acgsolvercuda *cg, const struct priv *pv, int nits, int nshifts)
{
    /* per iteration: the classic product, r -= alpha t with (r,r), p = r + beta p, and per shift
     * x_j += alpha_j p_j ; p_j = zeta_j r + beta_j p_j (x_j, p_j read and written: 32 B per row) */
    const int64_t n = pv->nowned, nnz = pv->fnnz + pv->onnz, s = nshifts;
    const int64_t bgemv = nnz * 12 + n * 16 + (int64_t) pv->nvec * 8;
    cg->ngemv += nits; cg->nflops += (int64_t) nits * 3 * nnz; cg->Bgemv += (int64_t) nits * bgemv;
    cg->ndot += nits; cg->nflops += (int64_t) nits * 2 * n; cg->Bdot += (int64_t) nits * 16 * n;
    cg->nnrm2 += nits; cg->nflops += (int64_t) nits * 2 * n; cg->Bnrm2 += (int64_t) nits * 8 * n;
    cg->naxpy += (int64_t) nits * (2 + 2 * s); cg->nflops += (int64_t) nits * (4 + 5 * s) * n;
    cg->Baxpy += (int64_t) nits * (48 + 32 * s) * n;
}

int acgsolvercuda_solve_shifted(struct acgsolvercuda *cg, const struct acgsymcsrmatrix *A,
                                int nshifts, const double *shifts, const double *b, double *X,
                                int maxits, double residualatol, double residualrtol, int warmup,
                                struct acgb200_colstats *stats)
{
    int errcode_ = 0, *errcode = &errcode_;
    struct priv *pv;
    OK(one_gpu_entry(cg, A, 1, have_shift_kernels(), valid_shifts(nshifts, shifts) && b && X && maxits >= 0, &pv));
    const int K = block_width(nshifts), n = pv->nowned;
    OK(ensure_blocks(pv, cg, K, errcode));
    OK(dev_scalars_once(pv, (void **) &pv->d_ss, sizeof(*pv->d_ss), errcode));
    struct solvectx c;
    block_begin(&c, cg, pv, KIND_SHIFTED, K, X, nshifts, errcode);
    /* b lives in the first n entries of the B block, which this loop does not otherwise use */
    OK(upload(&c, c.d_b, b, (size_t) n, 1, 1));
    struct acgb200_devstate h;
    struct acgb200_sstate ss;
    const unsigned all = (1u << nshifts) - 1u;

    /* warm-up: `warmup` iterations from the real set-up on state that is overwritten below; the R block
     * stands in for X, so X is untouched */
    if (warmup > 0) {
        c.d_x = pv->d_mr;
        OK(shifted_setup(&c));
        sstate_init(&ss, nshifts, shifts, 0.0, 1.0);
        OK(scalars_push(&c, pv->d_ss, &ss, sizeof(ss)));
        memset(&h, 0, sizeof(h));
        h.maxits = warmup; h.rr_loc[0] = h.rr[0] = 1.0; h.ctrl[0].pad0 = (int) all;
        OK(scalars_push(&c, pv->d_st, &h, sizeof(h)));
        for (int i = 0; i < warmup; i++) OK(shifted_iteration(&c, i));
        c.d_x = pv->d_mx;
        CU(cudaStreamSynchronize(pv->stream));
    }
    OK(window_open(&c, maxits, residualatol, residualrtol, 0, 0));

    /* r0 = p0 = b (x0 = 0 for every shift), X = 0, P_j = b ; ||b|| */
    double bb = 0, tol = 0, rtol_scaled[ACGB200_MAXK];
    OK(rhs_norm(&c, shifted_setup, &bb));
    c.launches += 2;
    const double bnrm2 = sqrt(bb);
    /* every shifted system starts from r0 = b, so all meet the test at r0 or none does */
    const unsigned mask = r0_test(residualatol, residualrtol, bnrm2, &tol, &rtol_scaled[0]) ? 0u : all;
    int nits[ACGB200_MAXK], conv[ACGB200_MAXK];
    double bbs[ACGB200_MAXK], rr[ACGB200_MAXK];
    for (int j = 0; j < nshifts; j++) {
        nits[j] = 0; conv[j] = !(mask >> j & 1u); bbs[j] = bb; rr[j] = bnrm2 * bnrm2; rtol_scaled[j] = rtol_scaled[0];
    }
    if (maxits > 0 && mask) {
        sstate_init(&ss, nshifts, shifts, tol, bnrm2);
        OK(scalars_push(&c, pv->d_ss, &ss, sizeof(ss)));
        memset(&h, 0, sizeof(h));
        h.maxits = maxits; h.rr_loc[0] = h.rr[0] = bb; h.ctrl[0].pad0 = (int) mask;
        OK(scalars_push(&c, pv->d_st, &h, sizeof(h)));
        OK(iterate(&c, maxits, tol > 0, shifted_iteration));
        OK(scalars_pull(&c, pv->d_st, &h, sizeof(h)));
        OK(scalars_pull(&c, pv->d_ss, &ss, sizeof(ss)));
        cg->niterations = h.ctrl[0].iter;
        for (int j = 0; j < nshifts; j++) {
            nits[j] = ss.nits[j]; conv[j] = ss.conv[j]; rr[j] = ss.final_rnrm2[j] * ss.final_rnrm2[j];
        }
    }
    account_shifted(cg, pv, cg->niterations, nshifts);
    cg->ncopy += 2; cg->nnrm2++;
    const int status = column_results(cg, nshifts, nits, conv, bbs, bbs, rr, residualatol, rtol_scaled, stats);
    cg->bnrm2 = cg->r0nrm2 = sqrt((double) nshifts * bb);
    return solve_finish(&c, status);
}

/* ------------------------------------------------------------------------ */
/* MINRES: symmetric A that may be indefinite                                */
/* ------------------------------------------------------------------------ */

/* the MINRES kernels are linked in (see ACGB200_MULTI_LAUNCHER, internal.h) */
static int have_minres_kernels(void)
{
    return acgb200_minres_setup && acgb200_minres_lanczos && acgb200_minres_update;
}

/* v_1 = r0 / beta_1 in d_r, v_0 = w_{-1} = w_0 = 0, and the scalars of the first iteration:
 * beta_1, c_0 = -1, s_0 = 0, delta-bar_1 = epsilon_1 = 0, phi-bar_1 = beta_1 */
static int minres_start(struct solvectx *c, int maxits, double tol, double beta1)
{
    struct priv *pv = c->pv;
    int *errcode = c->errcode;
    KL(acgb200_minres_setup(pv->nowned, beta1 > 0 ? 1.0 / beta1 : 0.0, c->cg->d_r, c->cg->d_p, pv->d_nw[0], pv->d_nw[1],
                            pv->stream));
    c->launches += 1;
    struct acgb200_nstate ns;
    memset(&ns, 0, sizeof(ns));
    ns.beta[0] = beta1; ns.cs[0] = -1.0; ns.phibar[0] = beta1;
    OK(scalars_push(c, pv->d_ns, &ns, sizeof(ns)));
    struct acgb200_devstate h;
    memset(&h, 0, sizeof(h));
    h.maxits = maxits; h.tol = tol;
    return scalars_push(c, pv->d_st, &h, sizeof(h));
}

/* iteration k: t = A v_k (+ alpha_k), u = t - alpha_k v_k - beta_k v_{k-1} (+ (u,u)), then the rotation, w_k, x
 * and v_{k+1}.  v_k is in d_r for even k and in d_p for odd k, v_{k+1} goes over v_{k-1}, w_k over w_{k-2}. */
static int minres_iteration(struct solvectx *c, int k)
{
    struct acgsolvercuda *cg = c->cg;
    struct priv *pv = c->pv;
    int *errcode = c->errcode;
    const int s = k & 1, n = pv->nowned;
    double *v = s ? cg->d_p : cg->d_r, *vprev = s ? cg->d_r : cg->d_p;
    OK(apply_A(c, v, v, cg->d_t, NULL, SPMV_Y_AX_DOT, &pv->d_ns->alpha[s], 1, 0, 0, 0));
    prof_mark(c, &pv->blas);
    KL(acgb200_minres_lanczos(n, pv->d_st, pv->d_ns, 1, v, vprev, cg->d_t, pv->stream));
    KL(acgb200_minres_update(n, pv->d_st, pv->d_ns, 1, 0, v, cg->d_t, pv->d_nw[s], pv->d_nw[s ^ 1], c->d_x, vprev,
                             pv->stream));
    prof_mark(c, &pv->blas);
    c->launches += 2;
    return ACG_SUCCESS;
}

static void account_minres(struct acgsolvercuda *cg, const struct priv *pv, int nits)
{
    /* per iteration: the classic product with (v, Av) folded in; u = t - alpha v - beta v_prev with (u,u)
     * (two axpys: t, v, v_prev read, u written) and w, x, v_{k+1} (three: v, u, both w, x read, w, x, v_{k+1}
     * written) -- 96 bytes per row the two kernels move */
    const int64_t n = pv->nowned, nnz = pv->fnnz + pv->onnz;
    const int64_t bgemv = nnz * 12 + n * 16 + (int64_t) pv->nvec * 8;
    cg->ngemv += nits; cg->nflops += (int64_t) nits * 3 * nnz; cg->Bgemv += (int64_t) nits * bgemv;
    cg->ndot += nits; cg->nflops += (int64_t) nits * 2 * n; cg->Bdot += (int64_t) nits * 16 * n;
    cg->nnrm2 += nits; cg->nflops += (int64_t) nits * 2 * n; cg->Bnrm2 += (int64_t) nits * 8 * n;
    cg->naxpy += 5 * (int64_t) nits; cg->nflops += (int64_t) nits * 12 * n; cg->Baxpy += (int64_t) nits * 96 * n;
}

int acgsolvercuda_solve_minres(struct acgsolvercuda *cg, const struct acgsymcsrmatrix *A,
                               const struct acgvector *b, struct acgvector *x, int maxits,
                               double residualatol, double residualrtol, int warmup, int *errcode)
{
    int errcode_ = 0;
    if (!errcode) errcode = &errcode_;
    struct priv *pv;
    OK(one_gpu_entry(cg, A, A && b && x, have_minres_kernels(), maxits >= 0, &pv));
    struct solvectx c;
    OK(solve_begin(&c, cg, A, b, x, 0.0, 0.0, &one_gpu_comm, 0, KIND_MINRES, errcode));
    const int n = pv->nowned;
    OK(dev_scalars_once(pv, (void **) &pv->d_ns, sizeof(*pv->d_ns), errcode));
    for (int i = 0; i < 2; i++)
        if (!pv->d_nw[i]) CU(cudaMalloc((void **) &pv->d_nw[i], ((size_t) pv->nvec + 2) * sizeof(double)));
    struct acgb200_devstate h;
    struct acgb200_nstate ns;

    /* warm-up: the set-up and `warmup` iterations on x itself, then x0 again from the caller's vector */
    if (warmup > 0) {
        double rr = 0;
        OK(residual(&c, &rr));
        OK(minres_start(&c, warmup, 0.0, sqrt(rr)));
        for (int i = 0; i < warmup; i++) OK(minres_iteration(&c, i));
        OK(upload_x0(&c, x));
    }
    OK(window_open(&c, maxits, residualatol, residualrtol, 0, 0));

    /* ||b|| ; r0 = b - A x0 and beta_1 = ||r0|| */
    double bb = 0, rr0 = 0, tol = 0, rtol_scaled = 0;
    OK(rhs_norm(&c, NULL, &bb));
    c.launches += 1;
    OK(residual(&c, &rr0));
    const double beta1 = sqrt(rr0);
    cg->rnrm2 = cg->r0nrm2 = beta1;
    cg->nnrm2 += 2; cg->nflops += 4 * (int64_t) n; cg->Bnrm2 += 8 * (int64_t) n; cg->ngemv++;
    int converged = r0_test(residualatol, residualrtol, beta1, &tol, &rtol_scaled);

    /* beta_1 = 0: x0 solves the system, there is no Krylov space to build */
    if (!converged && maxits > 0 && beta1 > 0) {
        OK(minres_start(&c, maxits, tol, beta1));
        OK(iterate(&c, maxits, tol > 0, minres_iteration));
        OK(scalars_pull(&c, pv->d_st, &h, sizeof(h)));
        OK(scalars_pull(&c, pv->d_ns, &ns, sizeof(ns)));
        cg->niterations = h.ctrl[0].iter;
        cg->rnrm2 = ns.phibar[cg->niterations & 1];
        converged = tol > 0 && cg->rnrm2 < tol;
    }
    account_minres(cg, pv, cg->niterations);
    return solve_finish(&c, convergence_status(converged, residualatol, rtol_scaled));
}

/* ------------------------------------------------------------------------ */
/* mixed-precision CG with reliable updates                                  */
/* ------------------------------------------------------------------------ */

/* the mixed-precision kernels are linked in (see ACGB200_MULTI_LAUNCHER, internal.h) */
static int have_mixed_kernels(void)
{
    return acgb200_spmv_f32_launch && acgb200_mixed_setup && acgb200_mixed_update_r && acgb200_mixed_update_yp
           && acgb200_mixed_replace && acgb200_mixed_fold;
}

/* the float vectors (16 bytes per row), the scalars and the product's row chunks, made once per solver */
static int mixed_alloc(struct priv *pv, const struct acgsolvercuda *cg, int *errcode)
{
    OK(dev_scalars_once(pv, (void **) &pv->d_xs, sizeof(*pv->d_xs), errcode));
    if (!pv->d_f32) {
        /* four vectors of nowned + 2 floats, each starting on an 8-byte boundary (the kernels read pairs) */
        const size_t bytes = 4 * (((size_t) pv->nowned + 2) & ~(size_t) 1) * sizeof(float);
        CU(cudaMalloc((void **) &pv->d_f32, bytes));
        CU(cudaMemsetAsync(pv->d_f32, 0, bytes, pv->stream));
    }
    if (!pv->have_franges) {
        int lanes = 0;
        OK(row_chunks(pv, cg, pv->plan.symdiag_nd > 0, &pv->d_franges, &pv->nfranges, &lanes, errcode));
        pv->have_franges = 1;
    }
    return ACG_SUCCESS;
}

static float *mixed_vec(const struct priv *pv, int i)     /* 0 r, 1 p, 2 t, 3 y */
{
    return pv->d_f32 + (size_t) i * (((size_t) pv->nowned + 2) & ~(size_t) 1);
}

/* the fp32 product t = fl32(A p) with (p, t) into acc; gated: by ctrl[0] */
static int apply_A_f32(struct solvectx *c, const float *x, float *y, double *acc, int gated)
{
    struct acgsolvercuda *cg = c->cg;
    struct priv *pv = c->pv;
    int *errcode = c->errcode;
    struct acgb200_spmvf32args a;
    memset(&a, 0, sizeof(a));
    a.plan = &pv->plan;
    a.nranges = pv->nfranges; a.ranges = pv->d_franges;
    a.rowptr = cg->d_rowptr; a.colidx = cg->d_colidx; a.a = cg->d_a;
    a.x = x; a.y = y; a.acc = acc;
    a.ctrl_in = gated ? &pv->d_st->ctrl[0] : NULL; a.st = pv->d_st;
    prof_mark(c, &pv->gemv);
    KL(acgb200_spmv_f32_launch(&a, pv->stream));
    prof_mark(c, &pv->gemv);
    c->launches += (pv->plan.nslices > 0 && pv->plan.symdiag_nd > 0) + (pv->nfranges > 0);
    return ACG_SUCCESS;
}

/* sigma = 2^round(log2 sqrt(rr)) as its exponent (as mixed_scale_exp of kernels.cu) */
static int mixed_scale_exp(double rr)
{
    int e = 0;
    const double m = frexp(sqrt(rr), &e);
    return m < 0.70710678118654752440 ? e - 1 : e;
}

/* r = fl32(r64 / sigma), p = r, y = 0 and the scalars of the first iteration; rr64 = (r64, r64) > 0 */
static int mixed_start(struct solvectx *c, int maxits, double tol, double rr64)
{
    struct priv *pv = c->pv;
    int *errcode = c->errcode;
    const int e = mixed_scale_exp(rr64);
    KL(acgb200_mixed_setup(pv->nowned, ldexp(1.0, -e), c->cg->d_r, mixed_vec(pv, 0), mixed_vec(pv, 1), mixed_vec(pv, 3),
                           pv->stream));
    c->launches += 1;
    struct acgb200_xstate xs;
    memset(&xs, 0, sizeof(xs));
    xs.rho[0] = ldexp(rr64, -2 * e); xs.mx[0] = sqrt(xs.rho[0]); xs.sigma[0] = ldexp(1.0, e);
    xs.last_rr64 = rr64;
    OK(scalars_push(c, pv->d_xs, &xs, sizeof(xs)));
    struct acgb200_devstate h;
    memset(&h, 0, sizeof(h));
    h.maxits = maxits; h.tol = tol;
    return scalars_push(c, pv->d_st, &h, sizeof(h));
}

/* iteration k: t = fl32(A p) (+ pi), r -= alpha t (+ rho'), y and p (or the fold), the fp64 residual and
 * the replacement -- the last two idle unless a reliable update is due */
static int mixed_iteration(struct solvectx *c, int k)
{
    struct priv *pv = c->pv;
    int *errcode = c->errcode;
    const int s = k & 1, n = pv->nowned;
    float *r = mixed_vec(pv, 0), *p = mixed_vec(pv, 1), *t = mixed_vec(pv, 2), *y = mixed_vec(pv, 3);
    OK(apply_A_f32(c, p, t, &pv->d_xs->pi[s], 1));
    prof_mark(c, &pv->blas);
    KL(acgb200_mixed_update_r(n, pv->d_st, pv->d_xs, t, r, pv->stream));
    KL(acgb200_mixed_update_yp(n, pv->d_st, pv->d_xs, r, p, y, c->d_x, pv->stream));
    prof_mark(c, &pv->blas);
    OK(apply_A(c, c->d_x, c->d_x, c->cg->d_r, c->d_b, SPMV_R_B_AX, &pv->d_xs->rr64[s], 2, 0, 0, -1));
    KL(acgb200_mixed_replace(n, pv->d_st, pv->d_xs, c->cg->d_r, r, p, pv->stream));
    c->launches += 3;
    return ACG_SUCCESS;
}

static void account_mixed(struct acgsolvercuda *cg, const struct priv *pv, int nits, int nupdates)
{
    /* per iteration: the product on float vectors (4-byte gathers and store) with (p, t) folded in, then
     * update_r (12 bytes per row) and update_yp (20); each reliable update adds an fp64 residual product
     * and the replacement (20 bytes per row) */
    const int64_t n = pv->nowned, nnz = pv->fnnz + pv->onnz;
    cg->ngemv += nits + nupdates; cg->nflops += (int64_t) (nits + nupdates) * 3 * nnz;
    cg->Bgemv += (int64_t) nits * (nnz * 12 + n * 12) + (int64_t) nupdates * (nnz * 12 + n * 24);
    cg->ndot += nits; cg->nflops += (int64_t) nits * 2 * n; cg->Bdot += (int64_t) nits * 8 * n;
    cg->nnrm2 += nits; cg->nflops += (int64_t) nits * 2 * n; cg->Bnrm2 += (int64_t) nits * 4 * n;
    cg->naxpy += 3 * (int64_t) nits; cg->nflops += (int64_t) nits * 6 * n; cg->Baxpy += (int64_t) nits * 32 * n;
}

int acgsolvercuda_solve_mixed(struct acgsolvercuda *cg, const struct acgsymcsrmatrix *A,
                              const struct acgvector *b, struct acgvector *x, int maxits,
                              double residualatol, double residualrtol, int warmup, int *errcode)
{
    int errcode_ = 0;
    if (!errcode) errcode = &errcode_;
    struct priv *pv;
    OK(one_gpu_entry(cg, A, A && b && x, have_mixed_kernels(), maxits >= 0, &pv));
    struct solvectx c;
    OK(solve_begin(&c, cg, A, b, x, 0.0, 0.0, &one_gpu_comm, 0, KIND_MIXED, errcode));
    const int n = pv->nowned;
    OK(mixed_alloc(pv, cg, errcode));
    struct acgb200_devstate h;
    struct acgb200_xstate xs;

    /* warm-up: the set-up and `warmup` iterations on x itself, then x0 again from the caller's vector */
    if (warmup > 0) {
        double rr = 0;
        OK(residual(&c, &rr));
        if (rr > 0) {
            OK(mixed_start(&c, warmup, 0.0, rr));
            for (int i = 0; i < warmup; i++) OK(mixed_iteration(&c, i));
        }
        OK(upload_x0(&c, x));
    }
    OK(window_open(&c, maxits, residualatol, residualrtol, 0, 0));

    /* ||b|| ; r0 = b - A x0 in fp64 */
    double bb = 0, rr0 = 0, tol = 0, rtol_scaled = 0;
    OK(rhs_norm(&c, NULL, &bb));
    c.launches += 1;
    OK(residual(&c, &rr0));
    cg->rnrm2 = cg->r0nrm2 = sqrt(rr0);
    cg->nnrm2 += 2; cg->nflops += 4 * (int64_t) n; cg->Bnrm2 += 8 * (int64_t) n; cg->ngemv++;
    int converged = r0_test(residualatol, residualrtol, cg->r0nrm2, &tol, &rtol_scaled);
    int nupdates = 0;

    /* ||r0|| = 0: x0 solves the system */
    if (!converged && maxits > 0 && rr0 > 0) {
        OK(mixed_start(&c, maxits, tol, rr0));
        OK(iterate(&c, maxits, 1, mixed_iteration));
        OK(scalars_pull(&c, pv->d_st, &h, sizeof(h)));
        OK(scalars_pull(&c, pv->d_xs, &xs, sizeof(xs)));
        cg->niterations = h.ctrl[0].iter;
        nupdates = xs.nupdates;
        if (xs.conv || xs.breakdown) {
            /* y was folded into x (or is dropped: a breakdown returns the last fold), whose residual is known */
            cg->rnrm2 = sqrt(xs.last_rr64);
        } else {
            /* maxits: the last fold, then the residual of the x returned */
            KL(acgb200_mixed_fold(n, xs.sigma[cg->niterations & 1], mixed_vec(pv, 3), c.d_x, pv->stream));
            double rr = 0;
            OK(residual(&c, &rr));
            c.launches += 1;
            cg->rnrm2 = sqrt(rr);
            cg->ngemv++;
        }
        converged = tol > 0 && cg->rnrm2 < tol;
    }
    account_mixed(cg, pv, cg->niterations, nupdates);
    pv->last_mixed_updates = nupdates;
    return solve_finish(&c, convergence_status(converged, residualatol, rtol_scaled));
}

/* ------------------------------------------------------------------------ */
/* Chebyshev-preconditioned CG                                               */
/* ------------------------------------------------------------------------ */

/* the Chebyshev kernels are linked in (see ACGB200_MULTI_LAUNCHER, internal.h) */
static int have_cheb_kernels(void)
{
    return acgb200_cheb_dinv && acgb200_cheb_rx && acgb200_cheb_step && acgb200_cheb_fused_step && acgb200_cheb_p;
}

static double *cheb_vec(const struct priv *pv, int i)     /* 0 D^-1, 1 z, 2 res, 3 d_0, 4 d_1 */
{
    return pv->d_cvec + (size_t) i * ((size_t) pv->nowned + 2);
}

/* the scalars and vectors, made once per solver, and D^-1 with its count of invalid diagonal entries */
static int cheb_alloc(struct solvectx *c)
{
    struct acgsolvercuda *cg = c->cg;
    struct priv *pv = c->pv;
    int *errcode = c->errcode;
    OK(dev_scalars_once(pv, (void **) &pv->d_cs, sizeof(*pv->d_cs), errcode));
    if (!pv->d_cvec) {
        const size_t bytes = 5 * ((size_t) pv->nowned + 2) * sizeof(double);
        CU(cudaMalloc((void **) &pv->d_cvec, bytes));
        CU(cudaMemsetAsync(pv->d_cvec, 0, bytes, pv->stream));
    }
    if (pv->cheb_baddiag < 0) {
        struct acgb200_cstate cs;
        memset(&cs, 0, sizeof(cs));
        OK(scalars_push(c, pv->d_cs, &cs, sizeof(cs)));
        KL(acgb200_cheb_dinv(pv->nowned, cg->d_rowptr, cg->d_colidx, cg->d_a, cheb_vec(pv, 0), pv->d_cs, pv->stream));
        OK(scalars_pull(c, pv->d_cs, &cs, sizeof(cs)));
        pv->cheb_baddiag = cs.baddiag;
    }
    return ACG_SUCCESS;
}

/* the start c0 = 1/theta and the steps' (rho_j rho_{j-1}, 2 rho_j / delta) of the interval [a, b] (Saad,
 * Iterative Methods, Alg. 12.1; tests/chebref.py coefficients) */
static void cheb_coefficients(struct solvectx *c, double a, double b)
{
    const double theta = (a + b) / 2, delta = (b - a) / 2, sigma = theta / delta;
    double rho = 1 / sigma;
    c->cheb_c0 = 1 / theta;
    for (int j = 0; j < c->cheb_degree; j++) {
        const double rn = 1 / (2 * sigma - rho);
        c->cheb_c[j][0] = rn * rho; c->cheb_c[j][1] = 2 * rn / delta;
        rho = rn;
    }
}

/* the d inner steps of z = M^-1 r after the r/x kernel: d_{j-1} in buffer (j-1)&1, d_j into the other */
static int cheb_steps(struct solvectx *c)
{
    struct acgsolvercuda *cg = c->cg;
    struct priv *pv = c->pv;
    int *errcode = c->errcode;
    const int n = pv->nowned;
    for (int j = 1; j <= c->cheb_degree; j++) {
        const double *dprev = cheb_vec(pv, 3 + ((j - 1) & 1));
        double *dnext = cheb_vec(pv, 3 + (j & 1));
        const int last = j == c->cheb_degree;
        const double c1 = c->cheb_c[j - 1][0], c2 = c->cheb_c[j - 1][1];
        if (c->cheb_fused) {
            struct acgb200_chebargs a;
            memset(&a, 0, sizeof(a));
            a.plan = &pv->plan; a.rowptr = cg->d_rowptr; a.colidx = cg->d_colidx; a.a = cg->d_a;
            a.st = pv->d_st; a.cs = pv->d_cs; a.c1 = c1; a.c2 = c2; a.last = last;
            a.q = cg->d_t; a.dinv = cheb_vec(pv, 0); a.dprev = dprev; a.dnext = dnext;
            a.res = cheb_vec(pv, 2); a.z = cheb_vec(pv, 1); a.r = c->cheb_r;
            KL(acgb200_cheb_fused_step(&a, pv->stream));
            c->launches += 1 + (pv->plan.ntiles > 0);
        } else {
            /* the plan's product into t (consumed by the r/x kernel already), gated by ctrl[2] */
            OK(apply_A(c, dprev, (double *) dprev, cg->d_t, NULL, SPMV_Y_AX, NULL, 2, 0, 0, -1));
            KL(acgb200_cheb_step(n, pv->d_st, pv->d_cs, c1, c2, last, cg->d_t, cheb_vec(pv, 0), dprev, dnext,
                                 cheb_vec(pv, 2), cheb_vec(pv, 1), c->cheb_r, pv->stream));
            c->launches += 1;
        }
    }
    return ACG_SUCCESS;
}

/* The set-up of a loop of c->cheb_degree from c->cheb_r: zeroed scalars, z_0 = M^-1 r_0 with (r_0, z_0) into rz
 * slot 0 (the preconditioner of "iteration -1": the r/x kernel's start and the inner steps, under a word with
 * iteration -1), p_0 = z_0, then the control words of iteration 0 */
static int cheb_start(struct solvectx *c, int maxits, double tol, int log)
{
    struct acgsolvercuda *cg = c->cg;
    struct priv *pv = c->pv;
    int *errcode = c->errcode;
    const int n = pv->nowned;
    struct acgb200_cstate cs;
    memset(&cs, 0, sizeof(cs));
    cs.log = log;
    OK(scalars_push(c, pv->d_cs, &cs, sizeof(cs)));
    struct acgb200_devstate h;
    memset(&h, 0, sizeof(h));
    h.maxits = maxits; h.tol = tol;
    h.ctrl[1].iter = h.ctrl[2].iter = -1;
    OK(scalars_push(c, pv->d_st, &h, sizeof(h)));
    KL(acgb200_cheb_rx(n, pv->d_st, pv->d_cs, 1, c->cheb_degree > 0, c->cheb_c0, cheb_vec(pv, 0), NULL, NULL, NULL,
                       c->cheb_r, cheb_vec(pv, 1), cheb_vec(pv, 2), cheb_vec(pv, 3), pv->stream));
    c->launches += 1;
    OK(cheb_steps(c));
    CU(cudaMemcpyAsync(cg->d_p, cheb_vec(pv, 1), (size_t) n * sizeof(double), cudaMemcpyDeviceToDevice, pv->stream));
    h.ctrl[1].iter = h.ctrl[2].iter = 0;
    return scalars_push(c, pv->d_st, &h, sizeof(h));
}

/* iteration k: t = A p (+ (p, t)), the r/x kernel, the d inner steps, the p kernel */
static int cheb_iteration(struct solvectx *c, int k)
{
    struct acgsolvercuda *cg = c->cg;
    struct priv *pv = c->pv;
    int *errcode = c->errcode;
    const int n = pv->nowned;
    OK(apply_A(c, cg->d_p, cg->d_p, cg->d_t, NULL, SPMV_Y_AX_DOT, &pv->d_cs->pap[k & 1], 1, 0, 0, 0));
    prof_mark(c, &pv->blas);
    KL(acgb200_cheb_rx(n, pv->d_st, pv->d_cs, 0, c->cheb_degree > 0, c->cheb_c0, cheb_vec(pv, 0), cg->d_t, cg->d_p,
                       c->cheb_x, c->cheb_r, cheb_vec(pv, 1), cheb_vec(pv, 2), cheb_vec(pv, 3), pv->stream));
    OK(cheb_steps(c));
    KL(acgb200_cheb_p(n, pv->d_st, pv->d_cs, cheb_vec(pv, 1), cg->d_p, pv->stream));
    prof_mark(c, &pv->blas);
    c->launches += 2;
    return ACG_SUCCESS;
}

/* eigenvalues of the symmetric tridiagonal (diagonal a, off-diagonal e) below x: the negative pivots of
 * T - x I = L D L^T (Sturm count; a zero pivot counts as negative) */
static int sturm_count(int k, const double *a, const double *e, double x)
{
    int cnt = 0;
    double q = 1.0;
    for (int j = 0; j < k; j++) {
        q = a[j] - x - (j > 0 ? e[j - 1] * e[j - 1] / q : 0.0);
        if (q == 0.0) q = -DBL_MIN;
        if (q < 0.0) cnt++;
    }
    return cnt;
}

/* eigenvalue i (ascending) of the tridiagonal by bisection of the Gershgorin interval [lo, hi] */
static double sturm_eigenvalue(int k, const double *a, const double *e, int i, double lo, double hi)
{
    for (int it = 0; it < 2200; it++) {
        const double mid = 0.5 * (lo + hi);
        if (mid <= lo || mid >= hi) break;
        if (sturm_count(k, a, e, mid) > i) hi = mid;
        else lo = mid;
    }
    return 0.5 * (lo + hi);
}

int acgb200_cheb_interval_host(int k, const double *alpha, const double *beta, double *theta_min, double *theta_max)
{
    if (k < 1 || !alpha || (k > 1 && !beta) || !theta_min || !theta_max) return ACG_ERR_INVALID_VALUE;
    for (int j = 0; j < k; j++) {
        if (!(alpha[j] > 0 && isfinite(alpha[j]))) return ACG_ERR_INVALID_VALUE;
        if (j + 1 < k && !(beta[j] >= 0 && isfinite(beta[j]))) return ACG_ERR_INVALID_VALUE;
    }
    double *a = malloc(2 * (size_t) k * sizeof(double));
    if (!a) return ACG_ERR_ERRNO;
    double *e = a + k;
    /* the Lanczos matrix of k CG steps: 1/alpha_j + beta_{j-1}/alpha_{j-1} on the diagonal, sqrt(beta_j)/alpha_j
     * beside it */
    double lo = INFINITY, hi = -INFINITY;
    for (int j = 0; j < k; j++) {
        a[j] = 1 / alpha[j] + (j > 0 ? beta[j - 1] / alpha[j - 1] : 0.0);
        if (j + 1 < k) e[j] = sqrt(beta[j]) / alpha[j];
    }
    for (int j = 0; j < k; j++) {
        const double rad = (j > 0 ? e[j - 1] : 0.0) + (j + 1 < k ? e[j] : 0.0);
        if (a[j] - rad < lo) lo = a[j] - rad;
        if (a[j] + rad > hi) hi = a[j] + rad;
    }
    const double pad = 4 * DBL_EPSILON * fmax(fabs(lo), fabs(hi)) + DBL_MIN;
    lo -= pad; hi += pad;
    *theta_min = sturm_eigenvalue(k, a, e, 0, lo, hi);
    *theta_max = sturm_eigenvalue(k, a, e, k - 1, lo, hi);
    free(a);
    return ACG_SUCCESS;
}

/* The upper bound's estimate: ACGB200_CHEB_EST Jacobi-PCG steps from r0 (in d_r) on scratch vectors -- r in
 * res, p and t in d_p and d_t, z in z, x not updated -- with their alpha and beta logged, stopping early on
 * ||r|| < tol or a breakdown; *steps of them ran, and theta_max is the largest eigenvalue of their Lanczos
 * matrix (0 if none ran). */
static int cheb_estimate(struct solvectx *c, double tol, int *steps, double *theta_max)
{
    struct priv *pv = c->pv;
    int *errcode = c->errcode;
    const int degree = c->cheb_degree, fused = c->cheb_fused;
    double *const r = c->cheb_r, *const x = c->cheb_x;
    c->cheb_degree = 0; c->cheb_fused = 0;
    c->cheb_r = cheb_vec(pv, 2); c->cheb_x = NULL;
    CU(cudaMemcpyAsync(c->cheb_r, c->cg->d_r, (size_t) pv->nowned * sizeof(double), cudaMemcpyDeviceToDevice,
                       pv->stream));
    OK(cheb_start(c, ACGB200_CHEB_EST, tol, 1));
    for (int i = 0; i < ACGB200_CHEB_EST; i++) OK(cheb_iteration(c, i));
    struct acgb200_devstate h;
    struct acgb200_cstate cs;
    OK(scalars_pull(c, pv->d_st, &h, sizeof(h)));
    OK(scalars_pull(c, pv->d_cs, &cs, sizeof(cs)));
    c->cheb_degree = degree; c->cheb_fused = fused; c->cheb_r = r; c->cheb_x = x;
    *steps = h.ctrl[0].iter;
    *theta_max = 0;
    double tmin = 0;
    if (*steps > 0) OK(acgb200_cheb_interval_host(*steps, cs.alpha_log, cs.beta_log, &tmin, theta_max));
    return ACG_SUCCESS;
}

static void account_cheb(struct acgsolvercuda *cg, const struct priv *pv, int nits, int degree, int fused,
                         int nsetup)
{
    /* Products: 1 + d per iteration and the set-up's (nsetup: the estimate's steps and the d steps of z_0), in the
     * CSR model of account_classic.  Vector bytes per row: the r/x kernel 64 at degree 0 (p, t, x, r, D^-1
     * read; x, r, z written) and 80 above it (res and d_0 written too); each inner step 56 (res, d_{j-1},
     * D^-1, z read; res, d_j, z written), the last 48 (r read, z written only), and 8 more without fusion (the
     * product's result read back); the p kernel 24 (z, p read; p written). */
    const int64_t n = pv->nowned, nnz = pv->fnnz + pv->onnz;
    const int64_t bgemv = nnz * 12 + n * 16 + (int64_t) pv->nvec * 8;
    const int64_t nprod = (int64_t) nits * (1 + degree) + nsetup;
    cg->ngemv += nprod; cg->nflops += nprod * 3 * nnz; cg->Bgemv += nprod * bgemv;
    cg->ndot += 2 * (int64_t) nits; cg->nflops += (int64_t) nits * 4 * n; cg->Bdot += (int64_t) nits * 16 * n;
    cg->nnrm2 += nits; cg->nflops += (int64_t) nits * 2 * n; cg->Bnrm2 += (int64_t) nits * 8 * n;
    const int64_t bstep = degree > 0 ? 56 * (int64_t) (degree - 1) + 48 + (fused ? 0 : 8 * (int64_t) degree) : 0;
    const int64_t bvec = (degree > 0 ? 80 : 64) + bstep + 24;
    cg->naxpy += (3 + 2 * (int64_t) degree) * nits; cg->nflops += (int64_t) nits * (6 + 5 * (int64_t) degree) * n;
    cg->Baxpy += (int64_t) nits * bvec * n;
}

int acgsolvercuda_solve_chebyshev(struct acgsolvercuda *cg, const struct acgsymcsrmatrix *A,
                                  const struct acgvector *b, struct acgvector *x, int degree,
                                  double lmin, double lmax, int maxits, double residualatol,
                                  double residualrtol, int warmup, int *errcode)
{
    int errcode_ = 0;
    if (!errcode) errcode = &errcode_;
    /* the interval: non-negative and finite (0: estimated), a given lower bound below a given upper one */
    const int interval_ok = degree == 0 || (isfinite(lmin) && lmin >= 0 && isfinite(lmax) && lmax >= 0 &&
                                            !(lmin > 0 && lmax > 0 && lmin >= lmax));
    struct priv *pv;
    OK(one_gpu_entry(cg, A, A && b && x, have_cheb_kernels(),
                     maxits >= 0 && degree >= 0 && degree <= ACGB200_CHEB_MAXDEG && interval_ok, &pv));
    struct solvectx c;
    OK(solve_begin(&c, cg, A, b, x, 0.0, 0.0, &one_gpu_comm, 0, KIND_CHEB, errcode));
    const int n = pv->nowned;
    OK(cheb_alloc(&c));
    if (pv->cheb_baddiag != 0) return ACG_ERR_INVALID_VALUE;
    c.cheb_degree = degree;
    /* one kernel per inner step where the pipelined solve fuses its iteration: mirrored diagonals for the slice
     * rows, all other rows in tiles (DESIGN.md sections 4a and 15) */
    const struct acgb200_spmvplan *pl = &pv->plan;
    c.cheb_fused = degree > 0 && pl->nslices > 0 && pl->symdiag_nd > 0 && pl->nmtiles == 0 && pl->nmed == 0
                   && pl->nlong == 0;
    c.cheb_r = cg->d_r; c.cheb_x = c.d_x;
    struct acgb200_devstate h;

    /* warm-up: the set-up and `warmup` iterations (any interval) on x itself, then x0 again from the caller's
     * vector */
    if (warmup > 0) {
        double rr = 0;
        OK(residual(&c, &rr));
        if (rr > 0) {
            cheb_coefficients(&c, 0.2, 2.0);
            OK(cheb_start(&c, warmup, 0.0, 0));
            for (int i = 0; i < warmup; i++) OK(cheb_iteration(&c, i));
        }
        OK(upload_x0(&c, x));
    }
    OK(window_open(&c, maxits, residualatol, residualrtol, 0, 0));
    pv->last_cheb_degree = degree;

    /* ||b|| ; r0 = b - A x0 */
    double bb = 0, rr0 = 0, tol = 0, rtol_scaled = 0;
    OK(rhs_norm(&c, NULL, &bb));
    c.launches += 1;
    OK(residual(&c, &rr0));
    cg->rnrm2 = cg->r0nrm2 = sqrt(rr0);
    cg->nnrm2 += 2; cg->nflops += 4 * (int64_t) n; cg->Bnrm2 += 8 * (int64_t) n; cg->ngemv++;
    int converged = r0_test(residualatol, residualrtol, cg->r0nrm2, &tol, &rtol_scaled);
    int nsetup = 0;

    /* ||r0|| = 0: x0 solves the system */
    if (!converged && maxits > 0 && rr0 > 0) {
        double a = 0, bnd = degree > 0 ? lmax : 0;
        int est = 0, started = 1;
        if (degree > 0) {
            if (lmax == 0) {
                double tmax = 0;
                OK(cheb_estimate(&c, tol, &est, &tmax));
                bnd = 1.1 * tmax;
                nsetup += est;
                pv->last_cheb_est = est;
            }
            if (est > 0 || lmax > 0) {
                a = lmin > 0 ? lmin : bnd / 10;
                if (!(isfinite(bnd) && a < bnd)) return ACG_ERR_INVALID_VALUE;
                pv->last_cheb_lmin = a; pv->last_cheb_lmax = bnd;
                cheb_coefficients(&c, a, bnd);
            } else {
                /* no estimate step ran: (p, A p) or (r, z) of Jacobi PCG from r0 broke down */
                started = 0;
                pv->last_cheb_breakdown = 1;
            }
        }
        if (started) {
            /* the coefficients are arguments of the replayed kernels: a graph of another interval is not reused */
            if (pv->graph[KIND_CHEB] && (pv->cheb_graph_ab[0] != a || pv->cheb_graph_ab[1] != bnd)) {
                cudaGraphExecDestroy(pv->graph[KIND_CHEB]);
                pv->graph[KIND_CHEB] = NULL;
            }
            pv->cheb_graph_ab[0] = a; pv->cheb_graph_ab[1] = bnd;
            OK(cheb_start(&c, maxits, tol, 0));
            nsetup += degree;
            OK(iterate(&c, maxits, 1, cheb_iteration));
            struct acgb200_cstate cs;
            OK(scalars_pull(&c, pv->d_st, &h, sizeof(h)));
            OK(scalars_pull(&c, pv->d_cs, &cs, sizeof(cs)));
            cg->niterations = h.ctrl[0].iter;
            if (cg->niterations > 0) cg->rnrm2 = sqrt(h.final_rr);
            pv->last_cheb_breakdown = cs.breakdown;
        }
        converged = tol > 0 && cg->rnrm2 < tol;
    }
    account_cheb(cg, pv, cg->niterations, degree, c.cheb_fused, nsetup);
    return solve_finish(&c, convergence_status(converged, residualatol, rtol_scaled));
}

/* ------------------------------------------------------------------------ */
/* pipelined CG                                                              */
/* ------------------------------------------------------------------------ */

static int ensure_vec(struct acgvector **hv, double **dv, const struct acgsymcsrmatrix *A, int nvec, int *errcode)
{
    if (!*hv) {
        *hv = malloc(sizeof(**hv));
        if (!*hv) return ACG_ERR_ERRNO;
        OK(acgsymcsrmatrix_vector(A, *hv));
        acgvector_setzero(*hv);
    }
    if (!*dv) CU(cudaMalloc((void **) dv, ((size_t) nvec + 2) * sizeof(double)));
    return ACG_SUCCESS;
}

static int pipelined_iteration(struct solvectx *c, int k)
{
    struct acgsolvercuda *cg = c->cg;
    struct priv *pv = c->pv;
    struct acgb200_devstate *st = pv->d_st;
    int *errcode = c->errcode;
    const int s = k & 1, n = pv->nowned;
    const int peer = c->multi && c->p2p;
    if (c->fused) {
        /* one GPU: iteration k gathers w from buffer k&1 and writes w_{k+1} into the other; it reads r_k from
         * ring slot k % m and writes r_{k+1} into slot (k+1) % m, and the last of each group of m also
         * updates p and x for the whole group (DESIGN.md section 4a) */
        const int m = c->group, j = k % m, jn = (j + 1) % m;
        struct acgb200_pcgargs a;
        memset(&a, 0, sizeof(a));
        a.plan = &pv->plan; a.rowptr = cg->d_rowptr; a.colidx = cg->d_colidx; a.a = cg->d_a;
        a.w = s ? pv->d_w2 : cg->d_w; a.w_next = s ? cg->d_w : pv->d_w2;
        a.r = j ? pv->d_rring + (size_t) (j - 1) * pv->r_stride : cg->d_r;
        a.r_next = jn ? pv->d_rring + (size_t) (jn - 1) * pv->r_stride : cg->d_r;
        a.r_ring = pv->d_rring; a.r_stride = pv->r_stride; a.group = m; a.catchup = j == m - 1;
        a.q = cg->d_q; a.z = cg->d_z; a.t = cg->d_t; a.p = cg->d_p; a.x = c->d_x;
        a.st = st; a.cin = s; a.vec_evict_first = cfg.pcg_evict_first;
        /* the whole iteration is timed as the product: no separate update time on this path */
        prof_mark(c, &pv->gemv);
        KL(acgb200_pcg_fused_launch(&a, pv->stream));
        prof_mark(c, &pv->gemv);
        c->launches += 1 + (pv->plan.ntiles > 0 ? 2 : 0);
        return ACG_SUCCESS;
    }
    /* One allreduce for {gamma,delta} (acg/cgcuda.c:1697).  The reference
     * issues it on the compute stream ahead of q = A w, i.e. serialised.  Here:
     * peer-memory mode -- the partials were pushed to every rank right after
     * the previous update and are summed by the update kernel itself; NCCL mode
     * -- the allreduce runs on its own stream and communicator and is only
     * joined before the update.  Either way it overlaps the SpMV, which is the
     * point of pipelined CG.  {gamma_0,delta_0} were reduced during setup. */
    const int side = c->multi && !peer && pv->have_redcomm;
    if (k > 0 && c->multi && !peer) {
        if (side) {
            CU(cudaEventRecord(pv->ev_ready, pv->stream));
            CU(cudaStreamWaitEvent(pv->redstream, pv->ev_ready, 0));
            OK(acgcomm_allreduce(&st->gd_loc[s][0], &st->gd[s][0], 2, ACG_DOUBLE, ACG_SUM, pv->redstream, &pv->redcomm, errcode));
            CU(cudaEventRecord(pv->ev_red, pv->redstream));
        } else {
            OK(allreduce(c, &st->gd_loc[s][0], &st->gd[s][0], 2));
        }
    }
    OK(apply_A(c, cg->d_w, cg->d_w, cg->d_q, NULL, SPMV_Y_AX, NULL, 1, 2, 0, -1));
    if (k > 0 && side) CU(cudaStreamWaitEvent(pv->stream, pv->ev_red, 0));
    prof_mark(c, &pv->blas);
    KL(acgb200_pcg_update(n, st, 1, 0, c->multi, peer ? pv->p2p.d_desc : NULL,
                          cg->d_q, cg->d_z, cg->d_w, cg->d_t, cg->d_p, cg->d_r, c->d_x, pv->stream));
    prof_mark(c, &pv->blas);
    /* in peer-memory mode the update kernel itself pushed w's border entries
     * and {gamma,delta} of the next iteration to the other ranks, unless fusion
     * is switched off */
    if (peer && !pv->p2p.h_desc.fuse) OK(post(c, 0, -1, cg->d_w, 0, &st->gd_loc[0][0], 2, 2, 0, 0));
    c->launches += 1 + (c->multi && !peer ? 1 : 0);
    return ACG_SUCCESS;
}

int acgsolvercuda_solve_pipelined(
    struct acgsolvercuda *cg, const struct acgsymcsrmatrix *A,
    const struct acgvector *b, struct acgvector *x,
    int maxits, double diffatol, double diffrtol, double residualatol, double residualrtol,
    int warmup, struct acgcomm *comm, int tag, int *errcode,
    cublasHandle_t cublas, cusparseHandle_t cusparse)
{
    (void) cublas; (void) cusparse;
    int errcode_ = 0;
    if (!errcode) errcode = &errcode_;
    cfg_load();
    struct solvectx c;
    OK(solve_begin(&c, cg, A, b, x, diffatol, diffrtol, comm, tag, KIND_PIPELINED, errcode));
    struct priv *pv = c.pv;
    struct acgb200_devstate *st = pv->d_st;
    const int n = pv->nowned;
    const size_t obytes = (size_t) n * sizeof(double);
    struct acgb200_devstate h;
    /* extra vectors are created on first use (acg/cgcuda.c:1167-1184) */
    OK(ensure_vec(&cg->w, &cg->d_w, A, pv->nvec, errcode));
    OK(ensure_vec(&cg->q, &cg->d_q, A, pv->nvec, errcode));
    OK(ensure_vec(&cg->z, &cg->d_z, A, pv->nvec, errcode));

    c.p2p = c.multi && pv->p2p.enabled && cfg.p2p;
    /* one kernel per iteration: one GPU, mirrored diagonals for the slice rows, all other rows in tiles */
    const struct acgb200_spmvplan *pl = &pv->plan;
    c.fused = cfg.pcg_fused && !c.multi && pv->nghost == 0 && pv->nborder == 0 && pl->symdiag_nd > 0 && pl->pcg_grid > 0
              && pl->nmtiles == 0 && pl->nmed == 0 && pl->nlong == 0;
    if (c.fused && !pv->d_w2) {
        CU(cudaMalloc((void **) &pv->d_w2, ((size_t) pv->nvec + 2) * sizeof(double)));
        CU(cudaMemsetAsync(pv->d_w2, 0, ((size_t) pv->nvec + 2) * sizeof(double), pv->stream));
    }
    if (c.fused) c.group = cfg.pcg_group;
    if (c.fused && pv->r_slots < c.group - 1) {
        /* slots 1 ... m-1 of the r ring (slot 0 is d_r), each on a 256-byte boundary */
        const size_t stride = ((size_t) pv->nvec + 2 + 31) & ~(size_t) 31;
        CU(cudaStreamSynchronize(pv->stream));
        cudaFree(pv->d_rring);
        pv->d_rring = NULL; pv->r_slots = 0;
        CU(cudaMalloc((void **) &pv->d_rring, (size_t) (c.group - 1) * stride * sizeof(double)));
        CU(cudaMemsetAsync(pv->d_rring, 0, (size_t) (c.group - 1) * stride * sizeof(double), pv->stream));
        pv->r_stride = stride; pv->r_slots = c.group - 1;
    }
    if (c.p2p) OK(acgcomm_barrier(pv->stream, comm, errcode));     /* as in acgsolvercuda_solvempi */
    if (warmup > 0) {
        memset(&h, 0, sizeof(h));
        h.maxits = warmup;
        for (int s = 0; s < 2; s++) { h.gd_loc[s][0] = h.gd[s][0] = 1; h.gd_loc[s][1] = h.gd[s][1] = 1; h.prev[s][0] = h.prev[s][1] = INFINITY; }
        OK(scalars_push(&c, pv->d_st, &h, sizeof(h)));
        /* x on r: the fused loop also writes the r ring, and the set-up below rewrites every slot before the
         * solve reads it (d_r from b - A x0, slot j in iteration j - 1) */
        double *xsave = c.d_x; c.d_x = cg->d_r;
        if (c.p2p) {
            OK(acgb200_p2p_begin(&pv->p2p, warmup, pv->stream));
            OK(post(&c, 0, 0, cg->d_w, -1, NULL, 0, 0, 0, 0));
        }
        for (int i = 0; i < warmup; i++) OK(pipelined_iteration(&c, i));
        c.d_x = xsave;
        KL(acgb200_dot(n, c.d_b, c.d_b, &st->tmp_loc[0], pv->stream));
        KL(acgb200_dot2(n, cg->d_r, cg->d_w, &st->tmp_loc[0], pv->stream));
        CU(cudaStreamSynchronize(pv->stream));
    }
    /* z = t = p = 0 (acg/cgcuda.c:1516-1522) */
    CU(cudaMemsetAsync(cg->d_z, 0, obytes, pv->stream));
    CU(cudaMemsetAsync(cg->d_t, 0, obytes, pv->stream));
    CU(cudaMemsetAsync(cg->d_p, 0, obytes, pv->stream));
    CU(cudaMemsetAsync(cg->d_w, 0, ((size_t) pv->nvec + 2) * sizeof(double), pv->stream));
    OK(window_open(&c, maxits, residualatol, residualrtol, diffatol, diffrtol));

    double bb = 0, gd0[2] = { 0, 0 };
    OK(rhs_norm(&c, NULL, &bb));

    /* r0 = b - A x0 ; w0 = A r0 (acg/cgcuda.c:1577-1671) */
    OK(apply_A(&c, c.d_x, c.d_x, cg->d_r, c.d_b, SPMV_R_B_AX, NULL, 0, 0, 0, -1));
    OK(apply_A(&c, cg->d_r, cg->d_r, cg->d_w, NULL, SPMV_Y_AX, NULL, 0, 0, 0, -1));
    /* gamma0 = (r0,r0), delta0 = (w0,r0): in the reference these are the first
     * two dots of the loop (acg/cgcuda.c:1680-1697); later ones come fused out
     * of the update kernel */
    KL(acgb200_dot2(n, cg->d_r, cg->d_w, &st->gd_loc[0][0], pv->stream));
    OK(reduce_to_host(&c, &st->gd_loc[0][0], &st->gd[0][0], 2, gd0));
    /* the loop makes the stopping test, from iteration 0 on */
    int converged = 0;
    double rtol_scaled = residualrtol, tol = 0;
    if (maxits > 0) {
        cg->rnrm2 = cg->r0nrm2 = sqrt(gd0[0]);                     /* acg/cgcuda.c:1760-1761 */
        (void) r0_test(residualatol, residualrtol, cg->r0nrm2, &tol, &rtol_scaled);
        memset(&h, 0, sizeof(h));
        h.maxits = maxits; h.tol = tol;
        h.gd_loc[0][0] = h.gd[0][0] = gd0[0];
        h.gd_loc[0][1] = h.gd[0][1] = gd0[1];
        h.prev[0][0] = h.prev[0][1] = INFINITY;                    /* acg/cgcuda.c:1513-1514 */
        OK(scalars_push(&c, pv->d_st, &h, sizeof(h)));
        if (c.p2p) {
            /* w_0 goes to the neighbours' windows as exchange number 0 */
            OK(acgb200_p2p_begin(&pv->p2p, maxits, pv->stream));
            OK(post(&c, 0, 0, cg->d_w, -1, NULL, 0, 0, 0, 0));
        }
        OK(iterate(&c, maxits, tol > 0, pipelined_iteration));
        if (c.fused) {
            /* a partial last group left p, x behind and its last r in the ring; launched wherever the solve
             * stopped, so the launch count of a solve does not depend on it */
            KL(acgb200_pcg_fused_finish(n, st, c.issued & 1, c.group, cg->d_r, pv->d_rring, pv->r_stride, cg->d_p,
                                        c.d_x, pv->stream));
            c.launches += 1;
        }
        OK(scalars_pull(&c, pv->d_st, &h, sizeof(h)));
        const struct acgb200_ctrl cw = h.ctrl[c.fused ? c.issued & 1 : 0];
        cg->niterations = cw.iter;
        converged = cw.done;
        /* the reference reports sqrt(gamma) of the last *tested* iterate
         * (acg/cgcuda.c:1760): gamma_k at convergence, gamma_{maxits-1} otherwise */
        const int kk = converged ? cg->niterations : (cg->niterations > 0 ? cg->niterations - 1 : 0);
        const double g = converged ? h.final_rr
            : (kk == 0 ? gd0[0] : (c.multi ? h.gd[kk & 1][0] : h.gd_loc[c.fused ? kk % 3 : kk & 1][0]));
        cg->rnrm2 = sqrt(g);
    }
    {
        const int64_t nits = cg->niterations, nnz = pv->fnnz + pv->onnz;
        const int64_t bgemv = nnz * 12 + (int64_t) n * 16 + (int64_t) (pv->nborder + pv->nghost) * 8 + (int64_t) pv->nvec * 8;
        cg->ngemv += nits + 2; cg->nflops += (nits + 2) * 3 * nnz; cg->Bgemv += (nits + 2) * bgemv;
        cg->nnrm2 += nits + 1; cg->ndot += nits; cg->nflops += nits * 4 * n; cg->Bnrm2 += nits * 8 * n; cg->Bdot += nits * 16 * n;
        cg->naxpy += nits; cg->nflops += nits * 12 * n; cg->Baxpy += nits * 56 * n;   /* acg/cgcuda.c:1783-1784 */
        if (c.multi) {
            cg->nallreduce += nits; cg->Ballreduce += nits * 16;
            cg->nhalo += nits + 2; cg->Bhalo += (nits + 2) * cg->halo->sendsize * 8;
            cg->nhalomsgs += (nits + 2) * cg->halo->nrecipients;
        }
    }
    return solve_finish(&c, convergence_status(converged, residualatol, rtol_scaled));
}

/* ------------------------------------------------------------------------ */
/* device-resident variants                                                  */
/* ------------------------------------------------------------------------ */

/*
 * acg/cg-kernels-cuda.cu:998 / :1713.  In the reference these are the solvers
 * whose iteration never returns to the host: one cooperative kernel per solve,
 * scalars and the convergence test on the device, halo values and reductions
 * moved by device-initiated NVSHMEM operations; they require an NVSHMEM
 * communicator and a build with NVSHMEM (ACG_ERR_NVSHMEM_NOT_SUPPORTED
 * otherwise, :1012, :1727).
 *
 * In this library those three properties already hold for the loops behind
 * acgsolvercuda_solvempi / _solve_pipelined: scalars and the stopping test live
 * in the device control ring, the host only replays a captured graph of a few
 * iterations and looks at the control word every few iterations, and between GPUs
 * the kernels themselves store halo values and reduction partials into the
 * peers' memory.  So with a null or NCCL communicator the device entry points
 * run those loops (same results, same report); what is *not* built is the fusion
 * of an iteration's two or three kernels into one persistent kernel with grid
 * barriers (DESIGN.md section 9).  An NVSHMEM communicator is refused as in a
 * reference build without NVSHMEM.
 */
int acgsolvercuda_solve_device(
    struct acgsolvercuda *cg, const struct acgsymcsrmatrix *A,
    const struct acgvector *b, struct acgvector *x,
    int maxits, double diffatol, double diffrtol, double residualatol, double residualrtol,
    int warmup, struct acgcomm *comm, int *errcode)
{
    if (comm && comm->type == acgcomm_nvshmem) return ACG_ERR_NVSHMEM_NOT_SUPPORTED;
    return acgsolvercuda_solvempi(cg, A, b, x, maxits, diffatol, diffrtol, residualatol, residualrtol,
                                  warmup, comm, 0, errcode, NULL, NULL, 0);
}

int acgsolvercuda_solve_device_pipelined(
    struct acgsolvercuda *cg, const struct acgsymcsrmatrix *A,
    const struct acgvector *b, struct acgvector *x,
    int maxits, double diffatol, double diffrtol, double residualatol, double residualrtol,
    int warmup, struct acgcomm *comm, int *errcode)
{
    if (comm && comm->type == acgcomm_nvshmem) return ACG_ERR_NVSHMEM_NOT_SUPPORTED;
    return acgsolvercuda_solve_pipelined(cg, A, b, x, maxits, diffatol, diffrtol, residualatol, residualrtol,
                                         warmup, comm, 0, errcode, NULL, NULL);
}

/* ------------------------------------------------------------------------ */
/* acg/cg-kernels-cuda.h:45-97: public BLAS-1 building blocks                 */
/* ------------------------------------------------------------------------ */

static double *d_constants = NULL;      /* {-1, 1, 0}: lives as long as the process, like the reference's __constant__ symbols */

int acgsolvercuda_init_constants(double **d_minus_one, double **d_one, double **d_zero)
{
    if (!d_constants) {
        const double h[3] = { -1.0, 1.0, 0.0 };
        if (cudaMalloc((void **) &d_constants, sizeof(h)) != cudaSuccess) return ACG_ERR_CUDA;
        if (cudaMemcpy(d_constants, h, sizeof(h), cudaMemcpyHostToDevice) != cudaSuccess) return ACG_ERR_CUDA;
    }
    *d_minus_one = d_constants; *d_one = d_constants + 1; *d_zero = d_constants + 2;
    return ACG_SUCCESS;
}

int acgsolvercuda_alpha(double *d_alpha, double *d_minus_alpha, const double *d_rnrm2sqr, const double *d_pdott)
{
    return acgb200_helper_scalars(0, d_alpha, d_minus_alpha, d_rnrm2sqr, d_pdott, 0) ? ACG_ERR_CUDA : ACG_SUCCESS;
}

int acgsolvercuda_beta(double *d_beta, const double *d_rnrm2sqr, const double *d_rnrm2sqr_prev)
{
    return acgb200_helper_scalars(1, d_beta, NULL, d_rnrm2sqr, d_rnrm2sqr_prev, 0) ? ACG_ERR_CUDA : ACG_SUCCESS;
}

int acgsolvercuda_daxpy_alpha(int n, const double *d_rnrm2sqr, const double *d_pdott, const double *d_x, double *d_y)
{
    return acgb200_helper_axpy(0, n, d_rnrm2sqr, d_pdott, d_x, d_y, 0) ? ACG_ERR_CUDA : ACG_SUCCESS;
}

int acgsolvercuda_daxpy_minus_alpha(int n, const double *d_rnrm2sqr, const double *d_pdott, const double *d_x, double *d_y)
{
    return acgb200_helper_axpy(1, n, d_rnrm2sqr, d_pdott, d_x, d_y, 0) ? ACG_ERR_CUDA : ACG_SUCCESS;
}

int acgsolvercuda_daypx_beta(int n, const double *d_rnrm2sqr, const double *d_rnrm2sqr_prev, double *d_y, const double *d_x)
{
    return acgb200_helper_axpy(2, n, d_rnrm2sqr, d_rnrm2sqr_prev, d_x, d_y, 0) ? ACG_ERR_CUDA : ACG_SUCCESS;
}

int acgsolvercuda_pipelined_daxpy_fused(
    int n, const double *d_gamma, double *d_gamma_prev, const double *d_delta, const double *d_q,
    double *d_p, double *d_r, double *d_t, double *d_x, double *d_z, double *d_w, double *d_alpha_prev,
    cudaStream_t stream)
{
    return acgb200_helper_pipelined(n, d_gamma, d_gamma_prev, d_delta, d_q, d_p, d_r, d_t, d_x, d_z, d_w, d_alpha_prev, stream)
        ? ACG_ERR_CUDA : ACG_SUCCESS;
}

/* ------------------------------------------------------------------------ */
/* report                                                                    */
/* ------------------------------------------------------------------------ */

static void opline(FILE *f, int indent, const char *name, double t, int64_t n, int64_t B)
{
    fprintf(f, "%*s  %s: %.6f seconds %" PRId64 " times %" PRId64 " B %.3f GB/s\n",
            indent, "", name, t, n, B, t > 0 ? 1.0e-9 * (double) B / t : 0.0);
}

/* same keys, order and units as acg/cgcuda.c:1893-1946, so scripts that parse
 * the reference's report keep working */
int acgsolvercuda_fwrite(FILE *f, const struct acgsolvercuda *cg, int indent)
{
    const double tother = cg->tsolve - (cg->tgemv + cg->tdot + cg->tnrm2 + cg->taxpy + cg->tcopy + cg->tallreduce + cg->thalo);
    fprintf(f, "%*sunknowns: %" PRIdx "\n", indent, "", cg->p.size);
    fprintf(f, "%*ssolves: %d\n", indent, "", cg->nsolves);
    fprintf(f, "%*stotal iterations: %d\n", indent, "", cg->ntotaliterations);
    fprintf(f, "%*stotal flops: %.3f Gflop\n", indent, "", 1.0e-9 * (double) cg->nflops);
    fprintf(f, "%*stotal flop rate: %.3f Gflop/s\n", indent, "", cg->tsolve > 0 ? 1.0e-9 * (double) cg->nflops / cg->tsolve : 0.0);
    fprintf(f, "%*stotal solver time: %.6f seconds\n", indent, "", cg->tsolve);
    fprintf(f, "%*sperformance breakdown:\n", indent, "");
    opline(f, indent, "gemv", cg->tgemv, cg->ngemv, cg->Bgemv);
    opline(f, indent, "dot", cg->tdot, cg->ndot, cg->Bdot);
    opline(f, indent, "nrm2", cg->tnrm2, cg->nnrm2, cg->Bnrm2);
    opline(f, indent, "axpy", cg->taxpy, cg->naxpy, cg->Baxpy);
    opline(f, indent, "copy", cg->tcopy, cg->ncopy, cg->Bcopy);
    opline(f, indent, "MPI_Allreduce", cg->tallreduce, cg->nallreduce, cg->Ballreduce);
    opline(f, indent, "MPI_HaloExchange", cg->thalo, cg->nhalo, cg->Bhalo);
    fprintf(f, "%*s  other: %.6f seconds\n", indent, "", tother);
    fprintf(f, "%*slast solve:\n", indent, "");
    fprintf(f, "%*s  stopping criterion:\n", indent, "");
    fprintf(f, "%*s    maximum iterations: %d\n", indent, "", cg->maxits);
    fprintf(f, "%*s    tolerance for residual: %.*g\n", indent, "", DBL_DIG, cg->residualatol);
    fprintf(f, "%*s    tolerance for relative residual: %.*g\n", indent, "", DBL_DIG, cg->residualrtol);
    fprintf(f, "%*s    tolerance for difference in solution iterates: %.*g\n", indent, "", DBL_DIG, cg->diffatol);
    fprintf(f, "%*s    tolerance for relative difference in solution iterates: %.*g\n", indent, "", DBL_DIG, cg->diffrtol);
    fprintf(f, "%*s  iterations: %d\n", indent, "", cg->niterations);
    fprintf(f, "%*s  right-hand side 2-norm: %.*g\n", indent, "", DBL_DIG, cg->bnrm2);
    fprintf(f, "%*s  initial guess 2-norm: %.*g\n", indent, "", DBL_DIG, cg->x0nrm2);
    fprintf(f, "%*s  initial residual 2-norm: %.*g\n", indent, "", DBL_DIG, cg->r0nrm2);
    fprintf(f, "%*s  residual 2-norm: %.*g\n", indent, "", DBL_DIG, cg->rnrm2);
    fprintf(f, "%*s  difference in solution iterates 2-norm: %.*g\n", indent, "", DBL_DIG, cg->dxnrm2);
    return ACG_SUCCESS;
}

#ifdef ACG_HAVE_MPI
/* acg/cgcuda.h:293 (acg/cgcuda.c:1948-2216): the same report on `root`, with
 * times taken as the maximum and flop/byte/message counters as the sum over the
 * ranks of `comm` -- the aggregation the reference performs with
 * MPI_Reduce (:1990-2012).  `verbose` adds one halo line per rank. */
int acgsolvercuda_fwritempi(FILE *f, const struct acgsolvercuda *cg, int indent, int verbose, MPI_Comm comm, int root)
{
    int rank = 0, size = 1;
    MPI_Comm_rank(comm, &rank);
    MPI_Comm_size(comm, &size);
    struct acgsolvercuda agg = *cg;
    double tin[8] = { cg->tsolve, cg->tgemv, cg->tdot, cg->tnrm2, cg->taxpy, cg->tcopy, cg->tallreduce, cg->thalo }, tout[8];
    int64_t cin[16] = { cg->nflops, cg->Bgemv, cg->Bdot, cg->Bnrm2, cg->Baxpy, cg->Bcopy, cg->Ballreduce, cg->Bhalo,
                        cg->nhalomsgs, 0, 0, 0, 0, 0, 0, 0 }, cout[16];
    memcpy(tout, tin, sizeof(tin)); memcpy(cout, cin, sizeof(cin));
    if (MPI_Reduce(tin, tout, 8, MPI_DOUBLE, MPI_MAX, root, comm)) return ACG_ERR_MPI;
    if (MPI_Reduce(cin, cout, 16, MPI_INT64_T, MPI_SUM, root, comm)) return ACG_ERR_MPI;
    if (rank == root) {
        agg.tsolve = tout[0]; agg.tgemv = tout[1]; agg.tdot = tout[2]; agg.tnrm2 = tout[3];
        agg.taxpy = tout[4]; agg.tcopy = tout[5]; agg.tallreduce = tout[6]; agg.thalo = tout[7];
        agg.nflops = cout[0]; agg.Bgemv = cout[1]; agg.Bdot = cout[2]; agg.Bnrm2 = cout[3]; agg.Baxpy = cout[4];
        agg.Bcopy = cout[5]; agg.Ballreduce = cout[6]; agg.Bhalo = cout[7]; agg.nhalomsgs = cout[8];
        int err = acgsolvercuda_fwrite(f, &agg, indent);
        if (err) return err;
        fprintf(f, "%*sprocesses: %d\n", indent, "", size);
    }
    if (verbose > 0 && cg->halo) {
        /* per-rank halo volume (the reference prints these under -v, :2060-2100) */
        int64_t mine[4] = { cg->halo->nrecipients, cg->halo->sendsize, cg->halo->nsenders, cg->halo->recvsize };
        int64_t *all = rank == root ? malloc((size_t) size * sizeof(mine)) : NULL;
        if (MPI_Gather(mine, 4, MPI_INT64_T, all, 4, MPI_INT64_T, root, comm)) { free(all); return ACG_ERR_MPI; }
        if (rank == root) {
            fprintf(f, "%*shalo exchange pattern (rank: recipients sendsize senders recvsize):\n", indent, "");
            for (int r = 0; r < size; r++)
                fprintf(f, "%*s  %d: %" PRId64 " %" PRId64 " %" PRId64 " %" PRId64 "\n", indent, "", r,
                        all[4 * r], all[4 * r + 1], all[4 * r + 2], all[4 * r + 3]);
            free(all);
        }
    }
    return ACG_SUCCESS;
}
#endif

/* ------------------------------------------------------------------------ */
/* extensions (include/acgb200/ext.h)                                        */
/* ------------------------------------------------------------------------ */

int acgsolvercuda_spmv(struct acgsolvercuda *cg, const double *x, double *y, int nrep, double *ms_per_spmv)
{
    int errcode_ = 0, *errcode = &errcode_;
    struct priv *pv = priv_of(cg);
    if (!pv) return ACG_ERR_INVALID_VALUE;
    if (pv->nghost > 0) return ACG_ERR_NOT_SUPPORTED;     /* whole-matrix use only */
    const int n = pv->nowned;
    CU(cudaMemcpyAsync(cg->d_p, x, (size_t) n * sizeof(double), cudaMemcpyHostToDevice, pv->stream));
    struct acgb200_spmvargs a;
    memset(&a, 0, sizeof(a));
    a.plan = &pv->plan; a.rowptr = cg->d_rowptr; a.colidx = cg->d_colidx; a.a = cg->d_a;
    a.x = cg->d_p; a.y = cg->d_t; a.mode = SPMV_Y_AX; a.dotrows = n;
    cudaEvent_t e0, e1;
    CU(cudaEventCreate(&e0)); CU(cudaEventCreate(&e1));
    KL(acgb200_spmv_launch(&a, pv->stream));               /* untimed first pass */
    CU(cudaEventRecord(e0, pv->stream));
    for (int i = 0; i < nrep; i++) KL(acgb200_spmv_launch(&a, pv->stream));
    CU(cudaEventRecord(e1, pv->stream));
    CU(cudaMemcpyAsync(y, cg->d_t, (size_t) n * sizeof(double), cudaMemcpyDeviceToHost, pv->stream));
    CU(cudaStreamSynchronize(pv->stream));
    float ms = 0;
    if (nrep > 0) CU(cudaEventElapsedTime(&ms, e0, e1));
    if (ms_per_spmv) *ms_per_spmv = nrep > 0 ? (double) ms / nrep : 0.0;
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    return ACG_SUCCESS;
}

/*
 * One part's share of the product on ONE device in any of the three epilogue modes, ghost values
 * supplied by the caller: x has the part's nvec = owned + ghost entries, b (mode 2 only) and y its
 * owned rows.  mode 0: y = A x; mode 1: y = A x and *dot = sum_owned x_i y_i; mode 2: y = b - A x
 * and *dot = sum_owned y_i^2 -- the fused dots as the solver's epilogues compute them (mode 0
 * passes the accumulator too, which must stay 0).  path 0 is what the set-up products and the NCCL
 * loop back-end run (local block through the SpMV kernels, then offdiag_kernel adding -- or, in
 * mode 2, subtracting -- the border x ghost block from the ghost tail of x: acg/cgcuda.c:858 +
 * :878); path 1 is the kernel of the peer-memory loop: border x ghost block inside the tile kernel,
 * ghost values read from a window whose senders' flags are waited for (here a loop-back window in
 * this device's memory, filled from x's tail, the flags already published).  Whole matrices (no
 * ghosts) take either path.  y is poisoned before the launch, so a row no kernel writes reads NaN.
 * Needs no communicator -- it exists so that every kernel's epilogues and the border x ghost path
 * of a partitioned matrix can be checked against exact products on a single GPU.
 */
int acgsolvercuda_spmv_mode(struct acgsolvercuda *cg, int mode, const double *x, const double *b, double *y,
                            int path, double *dot)
{
    int errcode_ = 0, *errcode = &errcode_;
    struct priv *pv = priv_of(cg);
    if (!pv || (path != 0 && path != 1)) return ACG_ERR_INVALID_VALUE;
    if (mode != SPMV_Y_AX && mode != SPMV_Y_AX_DOT && mode != SPMV_R_B_AX) return ACG_ERR_INVALID_VALUE;
    if (mode == SPMV_R_B_AX && !b) return ACG_ERR_INVALID_VALUE;
    const int n = pv->nowned;
    struct acgb200_devstate *st = pv->d_st;
    CU(cudaMemcpyAsync(cg->d_p, x, (size_t) pv->nvec * sizeof(double), cudaMemcpyHostToDevice, pv->stream));
    if (mode == SPMV_R_B_AX) CU(cudaMemcpyAsync(cg->d_r, b, (size_t) n * sizeof(double), cudaMemcpyHostToDevice, pv->stream));
    CU(cudaMemsetAsync(cg->d_t, 0xff, (size_t) n * sizeof(double), pv->stream));
    CU(cudaMemsetAsync(&st->tmp_loc[0], 0, sizeof(double), pv->stream));
    struct acgb200_spmvargs a;
    memset(&a, 0, sizeof(a));
    a.plan = &pv->plan; a.rowptr = cg->d_rowptr; a.colidx = cg->d_colidx; a.a = cg->d_a;
    a.x = cg->d_p; a.y = cg->d_t; a.b = mode == SPMV_R_B_AX ? cg->d_r : NULL;
    a.mode = mode; a.acc = &st->tmp_loc[0]; a.dotrows = n; a.pub_ch = -1;
    void *d_win = NULL;
    if (path == 0) {
        a.dotrows = pv->borderoff;                  /* the border rows' share of the dot comes from offdiag_kernel */
        KL(acgb200_spmv_launch(&a, pv->stream));
        struct acgb200_offdiagargs o;
        memset(&o, 0, sizeof(o));
        o.nrows = pv->nborder; o.rowoffset = pv->borderoff;
        o.orowptr = cg->d_orowptr; o.ocolidx = cg->d_ocolidx; o.oa = cg->d_oa;
        o.x = cg->d_p; o.y = cg->d_t; o.acc = &st->tmp_loc[0]; o.st = st; o.p2p_iter_override = -1;
        offdiag_epilogue(&o, mode);
        KL(acgb200_offdiag_launch(&o, pv->stream));
    } else {
        /* loop-back window: [descriptor | flags (one per sender slot) | ghost values] */
        const size_t goff = sizeof(struct acgb200_p2pdev) + ACGB200_MAXR * sizeof(unsigned long long);
        const size_t bytes = goff + ((size_t) pv->nghost + 2) * sizeof(double);
        struct acgb200_p2pdev *h = calloc(1, sizeof(*h));
        if (!h) return ACG_ERR_ERRNO;
        cudaError_t e = cudaMalloc(&d_win, bytes);
        if (!e) e = cudaMemsetAsync(d_win, 0, bytes, pv->stream);
        if (e) { free(h); cudaFree(d_win); *errcode = (int) e; return ACG_ERR_CUDA; }
        unsigned long long *d_flags = (unsigned long long *) ((char *) d_win + sizeof(*h));
        double *d_ghost = (double *) ((char *) d_win + goff);
        h->nranks = 1; h->rank = 0;
        h->nsenders = 3; h->senders[0] = 0; h->senders[1] = 5; h->senders[2] = ACGB200_MAXR - 1;
        h->my_hflag = d_flags; h->my_ghost[0] = h->my_ghost[1] = d_ghost;
        h->hbase = 41; h->timeout_ns = 2000000000ull;
        h->borderoff = pv->borderoff; h->nborder = pv->nborder;
        unsigned long long flags[ACGB200_MAXR];
        for (int i = 0; i < ACGB200_MAXR; i++) flags[i] = 0;
        flags[0] = 41; flags[5] = 42; flags[ACGB200_MAXR - 1] = 41;      /* published: sequence >= hbase + iteration 0 */
        e = cudaMemcpyAsync(d_win, h, sizeof(*h), cudaMemcpyHostToDevice, pv->stream);
        if (!e) e = cudaMemcpyAsync(d_flags, flags, sizeof(flags), cudaMemcpyHostToDevice, pv->stream);
        if (!e && pv->nghost > 0)
            e = cudaMemcpyAsync(d_ghost, cg->d_p + n, (size_t) pv->nghost * sizeof(double), cudaMemcpyDeviceToDevice, pv->stream);
        /* the tail of x itself is poisoned: path 1 must take the ghosts from the window */
        if (!e && pv->nghost > 0) e = cudaMemsetAsync(cg->d_p + n, 0xff, (size_t) pv->nghost * sizeof(double), pv->stream);
        if (!e) e = cudaStreamSynchronize(pv->stream);
        free(h);
        if (e) { cudaFree(d_win); *errcode = (int) e; return ACG_ERR_CUDA; }
        a.p2p = (const struct acgb200_p2pdev *) d_win;
        a.od_rowoffset = pv->borderoff; a.od_nrows = pv->nborder;
        a.orowptr = cg->d_orowptr; a.ocolidx = cg->d_ocolidx; a.oa = cg->d_oa;
        int le = acgb200_spmv_launch(&a, pv->stream);
        if (le) { cudaFree(d_win); *errcode = le; return ACG_ERR_CUDA; }
    }
    double hdot = 0;
    cudaError_t e = cudaMemcpyAsync(y, cg->d_t, (size_t) n * sizeof(double), cudaMemcpyDeviceToHost, pv->stream);
    if (!e) e = cudaMemcpyAsync(&hdot, &st->tmp_loc[0], sizeof(double), cudaMemcpyDeviceToHost, pv->stream);
    if (!e) e = cudaStreamSynchronize(pv->stream);
    cudaFree(d_win);
    CU(e);
    if (dot) *dot = hdot;
    return ACG_SUCCESS;
}

/* The fp32 product of acgsolvercuda_solve_mixed on host float vectors: y = fl32(A x) over the owned rows
 * (x: nowned floats), *dot = (x, y) in fp64.  y is poisoned on the device first, so a row no kernel writes
 * reads NaN. */
int acgsolvercuda_spmv_f32(struct acgsolvercuda *cg, const float *x, float *y, double *dot)
{
    int errcode_ = 0, *errcode = &errcode_;
    struct priv *pv = priv_of(cg);
    if (!pv || !x || !y) return ACG_ERR_INVALID_VALUE;
    if (!have_mixed_kernels() || !one_gpu(pv, NULL)) return ACG_ERR_NOT_SUPPORTED;
    OK(mixed_alloc(pv, cg, errcode));
    const int n = pv->nowned;
    struct acgb200_devstate *st = pv->d_st;
    CU(cudaMemcpyAsync(mixed_vec(pv, 1), x, (size_t) n * sizeof(float), cudaMemcpyHostToDevice, pv->stream));
    CU(cudaMemsetAsync(mixed_vec(pv, 2), 0xff, (size_t) n * sizeof(float), pv->stream));
    CU(cudaMemsetAsync(&st->tmp_loc[0], 0, sizeof(double), pv->stream));
    struct solvectx c;
    ctx_init(&c, cg, pv, errcode);
    OK(apply_A_f32(&c, mixed_vec(pv, 1), mixed_vec(pv, 2), &st->tmp_loc[0], 0));
    double hdot = 0;
    CU(cudaMemcpyAsync(y, mixed_vec(pv, 2), (size_t) n * sizeof(float), cudaMemcpyDeviceToHost, pv->stream));
    CU(cudaMemcpyAsync(&hdot, &st->tmp_loc[0], sizeof(double), cudaMemcpyDeviceToHost, pv->stream));
    CU(cudaStreamSynchronize(pv->stream));
    if (dot) *dot = hdot;
    return ACG_SUCCESS;
}

/* The multi-vector product of acgsolvercuda_solve_multi in any of the three epilogue modes, for
 * nrhs columns (padded to the block width K as the solver pads them): X, B (mode 2) and Y are host
 * arrays of nowned x nrhs doubles, row-major; dots[j] gets column j's fused dot.  Y is poisoned on
 * the device first, so a row no kernel writes reads NaN. */
int acgsolvercuda_spmm_mode(struct acgsolvercuda *cg, int mode, int nrhs, const double *X, const double *B, double *Y,
                            double *dots)
{
    int errcode_ = 0, *errcode = &errcode_;
    struct priv *pv = priv_of(cg);
    if (!pv) return ACG_ERR_INVALID_VALUE;
    if (!have_multi_kernels() || !one_gpu(pv, NULL)) return ACG_ERR_NOT_SUPPORTED;
    if (nrhs < 1 || nrhs > ACGB200_MAXK || !X || !Y) return ACG_ERR_INVALID_VALUE;
    if (mode != SPMV_Y_AX && mode != SPMV_Y_AX_DOT && mode != SPMV_R_B_AX) return ACG_ERR_INVALID_VALUE;
    if (mode == SPMV_R_B_AX && !B) return ACG_ERR_INVALID_VALUE;
    const int K = block_width(nrhs), n = pv->nowned;
    OK(ensure_blocks(pv, cg, K, errcode));
    OK(upload_block_vec(pv, pv->d_mp, X, (size_t) n, nrhs, K, errcode));
    if (mode == SPMV_R_B_AX) OK(upload_block_vec(pv, pv->d_mb, B, (size_t) n, nrhs, K, errcode));
    CU(cudaMemsetAsync(pv->d_mt, 0xff, (size_t) n * K * sizeof(double), pv->stream));
    CU(cudaMemsetAsync(&pv->d_ms->tmp[0], 0, sizeof(pv->d_ms->tmp), pv->stream));
    struct solvectx c;
    ctx_init(&c, cg, pv, errcode);
    c.mk = K;
    OK(apply_A_multi(&c, pv->d_mp, pv->d_mt, mode == SPMV_R_B_AX ? pv->d_mb : NULL, mode, &pv->d_ms->tmp[0], 0));
    OK(download_block_vec(pv, Y, pv->d_mt, (size_t) n, nrhs, K, errcode));
    double h[ACGB200_MAXK];
    CU(cudaMemcpy(h, &pv->d_ms->tmp[0], sizeof(h), cudaMemcpyDeviceToHost));
    if (dots) for (int j = 0; j < nrhs; j++) dots[j] = h[j];
    return ACG_SUCCESS;
}

int acgsolvercuda_spmv_ghost(struct acgsolvercuda *cg, const double *x, double *y, int path, double *dot)
{
    return acgsolvercuda_spmv_mode(cg, SPMV_Y_AX_DOT, x, NULL, y, path, dot);
}

int acgsolvercuda_info(const struct acgsolvercuda *cg, struct acgb200_info *info)
{
    const struct priv *pv = priv_of(cg);
    if (!pv) return ACG_ERR_INVALID_VALUE;
    memset(info, 0, sizeof(*info));
    info->spmv_lanes_per_row = pv->plan.lanes_per_row;
    info->spmv_rows_cap = pv->plan.rows_cap; info->spmv_nnz_cap = pv->plan.nnz_cap;
    info->spmv_stages = pv->plan.nstages; info->spmv_ntiles = pv->plan.ntiles;
    info->spmv_nlong = pv->plan.nlong; info->spmv_grid = pv->plan.grid; info->spmv_smem_bytes = pv->plan.smem_bytes;
    info->last_launches = pv->last_launches;
    info->last_spmv_ms = pv->last_spmv_ms; info->last_spmv_count = pv->last_spmv_n;
    info->last_solve_ms = pv->last_solve_ms;
    info->last_h2d_ms = pv->last_h2d_ms; info->last_d2h_ms = pv->last_d2h_ms;
    info->last_blas_ms = pv->last_blas_ms;
    info->num_sms = acgb200_num_sms();
    info->spmv_merge_tiles = pv->plan.nmtiles; info->spmv_merge_rows = pv->plan.merge_rows; info->spmv_merge_split = pv->plan.nsplit;
    info->spmv_slices = pv->plan.nslices; info->spmv_slice_rows = pv->plan.slice_rows;
    info->spmv_slice_exc = (int) pv->plan.slice_exc;
    info->spmv_slice_ub = pv->plan.slice_ub; info->spmv_slice_grid = pv->plan.slice_grid;
    info->spmv_nmedium = pv->plan.nmed;
    info->spmv_threads = pv->plan.threads; info->spmv_unroll = pv->plan.unroll;
    info->spmv_slice_threads = pv->plan.slice_threads;
    info->spmv_merge_threads = pv->plan.merge_threads; info->spmv_merge_grid = pv->plan.merge_grid;
    info->spmv_merge_stages = pv->plan.merge_stages;
    /* the bytes of what profile mode times as one product: the whole iteration on the fused path */
    info->spmv_min_bytes = pv->last_fused ? acgb200_pcg_iteration_min_bytes(&pv->plan, pv->last_group)
                                          : acgb200_spmv_min_bytes(&pv->plan);
    info->spmv_slice_value_bytes = pv->plan.nslices > 0 ? pv->plan.sval_blocks * 32 * (int64_t) sizeof(double) : 0;
    info->spmv_slice_nnz = pv->plan.nslices > 0 ? pv->plan.slice_nnz : 0;
    info->spmv_symdiag_diagonals = pv->plan.symdiag_nd;
    info->spmv_symdiag_bytes = (int64_t) pv->plan.symdiag_nd * pv->plan.symdiag_stride * (int64_t) sizeof(double);
    info->pcg_fused = pv->last_fused;
    info->pcg_fused_min_bytes = pv->plan.symdiag_nd > 0 ? acgb200_pcg_fused_min_bytes(&pv->plan) : 0;
    info->spmv_symdiag_codes = pv->plan.symdiag_codes;
    info->spmv_symdiag_code_bytes = pv->plan.symdiag_codes > 0 ? (int64_t) pv->plan.symdiag_nd * pv->plan.symdiag_stride : 0;
    info->mixed_reliable_updates = pv->last_mixed_updates;
    info->cheb_degree = pv->last_cheb_degree; info->cheb_est_iterations = pv->last_cheb_est;
    info->cheb_breakdown = pv->last_cheb_breakdown;
    info->cheb_lmin = pv->last_cheb_lmin; info->cheb_lmax = pv->last_cheb_lmax;
    info->pcg_group = pv->last_fused ? pv->last_group : 0;
    return ACG_SUCCESS;
}
