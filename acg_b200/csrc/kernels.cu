/*
 * kernels.cu -- hand-written sm_90a kernels of the CG hot path.
 *
 * What each kernel replaces in the reference (paths relative to the aCG tree):
 *
 *   spmv_tiles_kernel     cusparseSpMV(matA)  acg/cgcuda.c:858,:1724 (+:775,:1639)
 *                         + cublasDdot(p,t)   acg/cgcuda.c:894  (fused epilogue)
 *   spmv_long_*           same, rows longer than one tile (power-law inputs);
 *                         the role csrgemv_merge plays in acg/cg-kernels-cuda.cu:340
 *   offdiag_kernel        cusparseSpMV(matO)  acg/cgcuda.c:878,:1744; csrgemv :443
 *   cg_update_r_kernel    daxpy_minus_alpha   acg/cg-kernels-cuda.cu:153 + cublasDdot(r,r) acg/cgcuda.c:933
 *   cg_update_xp_kernel   daxpy_alpha :119 + daypx_beta :271 (one pass instead of two)
 *   pcg_update_kernel     pipelined_daxpy_fused :187 + cublasDdot x2 acg/cgcuda.c:1680,:1688
 *   gather/scatter        acghalo_pack/unpack_cuda_double acg/halo.cu:41,:94
 *
 * Design (details in DESIGN.md): FP64 SIMT, HBM-bound, tensor cores unused.
 * The CSR streams (values, column indices, row pointers) are moved by the TMA
 * engine -- 1-D cp.async.bulk global->shared copies completing on an mbarrier
 * -- into a multi-stage shared-memory ring, so the SMs' load/store units only
 * issue the x gathers and the y stores.  Rows are processed from shared memory
 * by G-lane groups (G=1: one thread per row, the warp's gathers of 32
 * consecutive rows then coalesce for banded/stencil matrices).  Dot products
 * are folded into the kernels that produce their operands: warp shuffle ->
 * per-CTA shared reduce -> one atomicAdd(double) per CTA into a device scalar.
 */
#include "internal.h"

#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>
#include <type_traits>

#define SPMV_THREADS 128
/* Resident CTAs per SM the register allocator must leave room for.  Without
 * it ptxas squeezes the kernel into 32 registers (full-occupancy default) and
 * serialises the x gathers; shared memory limits residency to ~10 CTAs of 128
 * threads anyway, so 48 registers cost no occupancy. */
#define SPMV_MINB(T) ((T) >= 512 ? 2 : 1280 / (T))
#define SPMV_MAX_STAGES 8
#define BLAS1_THREADS 512

/* ------------------------------------------------------------------------ */
/* PTX wrappers: mbarrier + bulk async copy (TMA, 1-D)                       */
/* ------------------------------------------------------------------------ */

__device__ __forceinline__ uint32_t smem_addr(const void *p)
{
    return (uint32_t) __cvta_generic_to_shared(p);
}

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_addr(bar)), "r"(count) : "memory");
}

__device__ __forceinline__ void mbar_init_fence()
{
    /* make the initialised barriers visible to the async (TMA) proxy */
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;"
                 :: "r"(smem_addr(bar)), "r"(bytes) : "memory");
}

__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity)
{
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra WAIT_DONE;\n"
        "bra WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" :: "r"(smem_addr(bar)), "r"(parity) : "memory");
}

__device__ __forceinline__ uint64_t l2_policy_evict_first()
{
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}

__device__ __forceinline__ uint64_t l2_policy_evict_normal()
{
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}

/* global -> shared bulk copy; bytes and both addresses are multiples of 16.
 * The matrix streams are read exactly once per SpMV: evict-first keeps them
 * from displacing the x vector in L2. */
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar, uint64_t pol)
{
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
        :: "r"(smem_addr(dst)), "l"(src), "r"(bytes), "r"(smem_addr(bar)), "l"(pol) : "memory");
}

/* gather of a vector entry through the read-only path.  volatile: the batch of
 * gathers of one row stays a batch (the compiler may not sink individual loads
 * down to their uses, which would serialise their latencies). */
__device__ __forceinline__ double ld_x(const double *p)
{
    double v;
    asm volatile("ld.global.nc.f64 %0, [%1];" : "=d"(v) : "l"(p));
    return v;
}

/* the same for a float vector (the fp32 product of the mixed-precision solve) */
__device__ __forceinline__ float ld_x(const float *p)
{
    float v;
    asm volatile("ld.global.nc.f32 %0, [%1];" : "=f"(v) : "l"(p));
    return v;
}

/* coalesced read of matrix data that is used exactly once per SpMV: no L1 line, evict-first in L2,
 * so the stream does not displace the x vector (which every row re-reads) from either cache */
__device__ __forceinline__ double ld_stream(const double *p, uint64_t pol)
{
    double v;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.f64 %0, [%1], %2;" : "=d"(v) : "l"(p), "l"(pol));
    return v;
}

/* the same for one-byte value codes (the coded mirrored diagonals), zero-extended into a register */
__device__ __forceinline__ unsigned ld_stream(const uint8_t *p, uint64_t pol)
{
    unsigned v;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u8 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol));
    return v;
}

/* a vector entry read once and written back by the same thread in the same kernel (the fused pipelined-CG
 * update): the coherent path, no L1 line, the caller's L2 policy */
__device__ __forceinline__ double ld_vec(const double *p, uint64_t pol)
{
    double v;
    asm volatile("ld.global.L1::no_allocate.L2::cache_hint.f64 %0, [%1], %2;" : "=d"(v) : "l"(p), "l"(pol));
    return v;
}

__device__ __forceinline__ void st_vec(double *p, double v, uint64_t pol)
{
    asm volatile("st.global.L2::cache_hint.f64 [%0], %1, %2;" :: "l"(p), "d"(v), "l"(pol) : "memory");
}

/* Programmatic dependent launch (opt-in, ACGB200_PDL=1).  Every kernel of the
 * iteration chain starts with this: wait until the preceding kernel of the
 * stream has completed and flushed (nothing in global memory is touched before),
 * then let the next kernel's CTAs be scheduled as soon as SM resources free up,
 * so its launch latency and CTA ramp overlap this kernel's tail.  Both
 * instructions are no-ops for a kernel launched without the attribute. */
__device__ __forceinline__ void pdl_prologue()
{
    asm volatile("griddepcontrol.wait;" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}

/* ------------------------------------------------------------------------ */
/* reductions                                                                */
/* ------------------------------------------------------------------------ */

__device__ __forceinline__ double warp_sum(double v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

template <int G>
__device__ __forceinline__ double group_sum(double v)
{
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

/* sum over the CTA, result valid in thread 0; `red` holds blockDim/32 doubles */
__device__ __forceinline__ double block_sum(double v, double *red)
{
    v = warp_sum(v);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    if (l == 0) red[w] = v;
    __syncthreads();
    const int nw = (blockDim.x + 31) >> 5;
    v = (threadIdx.x < nw) ? red[threadIdx.x] : 0.0;
    if (w == 0) v = warp_sum(v);
    __syncthreads();
    return v;
}

/* ------------------------------------------------------------------------ */
/* iteration control                                                         */
/* ------------------------------------------------------------------------ */

struct Gate { int iter; bool active; };

/* Read the incoming control word.  The word a kernel reads is never written
 * by that same kernel, so every thread sees the same value. */
__device__ __forceinline__ Gate gate_read(const acgb200_ctrl *cin, const acgb200_devstate *st)
{
    Gate g; g.iter = 0; g.active = true;
    if (cin) {
        const int4 c = *reinterpret_cast<const int4 *>(cin);
        g.iter = c.x;
        g.active = (c.y == 0) && (c.x < st->maxits);
    }
    return g;
}

/* The scalars of pipelined-CG update k on the fused path (one GPU): {gamma_k, delta_k} from accumulator ring
 * slot k % 3, the expressions of pcg_update_kernel.  Every kernel of the iteration computes them alike. */
struct PcgStep { double gamma, alpha, beta; bool conv; };

__device__ __forceinline__ PcgStep pcg_step(const acgb200_devstate *st, int iter)
{
    PcgStep o;
    const int s = iter & 1, slot = iter % 3;
    const double gamma = st->gd_loc[slot][0], delta = st->gd_loc[slot][1];
    const double gamma_prev = st->prev[s][0], alpha_prev = st->prev[s][1];
    o.gamma = gamma;
    o.conv = st->tol > 0.0 && sqrt(gamma) < st->tol;
    o.beta = gamma / gamma_prev;
    o.alpha = gamma / (delta - o.beta * gamma / alpha_prev);
    return o;
}

/*
 * Row i of update k, the fma chain of pcg_update_kernel: z=q+beta z; t=w+beta t; r-=alpha t; w'=w-alpha z,
 * w' into the other buffer; gamma'=(r,r), delta'=(w',r) accumulate in g2, d2.  r_k is read from r and
 * r_{k+1} written to r_next.  p and x feed nothing but themselves, so they lag (DESIGN section 4a): their
 * updates p=r+beta p; x+=alpha p are left to pcg_catchup once per group of iterations.
 */
__device__ __forceinline__ void pcg_row(int i, double qi, double wi, double alpha, double beta,
                                        double *__restrict__ z, double *__restrict__ t,
                                        const double *__restrict__ r, double *__restrict__ r_next,
                                        double *__restrict__ w_next, uint64_t pol, double &g2, double &d2)
{
    const double zi = ld_vec(z + i, pol), ti = ld_vec(t + i, pol), ri = ld_vec(r + i, pol);
    const double zv = fma(beta, zi, qi);
    const double tv = fma(beta, ti, wi);
    const double rv = fma(-alpha, tv, ri);
    const double wv = fma(-alpha, zv, wi);
    st_vec(z + i, zv, pol); st_vec(t + i, tv, pol);
    st_vec(r_next + i, rv, pol);
    st_vec(w_next + i, wv, pol);
    g2 = fma(rv, rv, g2);
    d2 = fma(wv, rv, d2);
}

/*
 * Row i's p and x updates of a whole group j = k-m+1 ... k, run by the group's last iteration k before its
 * pcg_row: p_j = r_j + beta_j p_{j-1}; x += alpha_j p_j, the FMAs of pcg_update_kernel in the same order.
 * r_j lives in ring slot j % m: slot 0 (r_{k-m+1}) is the solver's r -- the slot pcg_row then overwrites
 * with r_{k+1}, so the caller runs this first for the same rows on the same threads -- slot m-1 (r_k) is
 * rk, and slot s in between is lag->ring + (s - 1) lag->stride.  ks: {alpha_j, beta_j} in order and lag,
 * both in shared memory; the r's are loaded in batches of four ahead of their FMAs.
 */
struct PcgLag { const double *ring; size_t stride; int m; };

__device__ __forceinline__ void pcg_catchup(int i, const double *ks, const PcgLag *lag, const double *r0,
                                            const double *rk, double *__restrict__ p, double *__restrict__ x,
                                            uint64_t pol)
{
    const int m = lag->m;
    const size_t stride = lag->stride;
    const double *ring = lag->ring + i;
    double pv = ld_vec(p + i, pol), xv = ld_vec(x + i, pol);
    for (int j0 = 0; j0 < m; j0 += 4) {
        double rl[4];
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const int j = j0 + u;
            if (j < m) rl[u] = ld_vec(j == 0 ? r0 + i : j == m - 1 ? rk + i : ring + (size_t) (j - 1) * stride, pol);
        }
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const int j = j0 + u;
            if (j < m) {
                pv = fma(ks[2 * j + 1], pv, rl[u]);
                xv = fma(ks[2 * j], pv, xv);
            }
        }
    }
    st_vec(p + i, pv, pol);
    st_vec(x + i, xv, pol);
}

/* ------------------------------------------------------------------------ */
/* peer-memory exchange: flags and reductions                                */
/* ------------------------------------------------------------------------ */

__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long *p)
{
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}

__device__ __forceinline__ void st_release_sys(unsigned long long *p, unsigned long long v)
{
    asm volatile("st.release.sys.global.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory");
}

#define RED_IDX(ch, parity, rank) ((((ch) * 2 + (parity)) * ACGB200_MAXR + (rank)) * 2)

__device__ __forceinline__ unsigned long long global_ns()
{
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}

/* Spin until *f >= seq.  A peer that never publishes (it failed, or a protocol
 * error) must not hang the GPU: after timeout_ns the waiter raises the sticky
 * timed_out flag of its descriptor and gives up, every later wait of the solve
 * returns at once, and the host turns the flag into an error (the iterates are
 * garbage from then on).  The clock is only read every 1024 polls. */
__device__ __forceinline__ void p2p_spin(const unsigned long long *f, unsigned long long seq, const acgb200_p2pdev *P)
{
    unsigned long long t0 = 0;
    unsigned int polls = 0;
    volatile unsigned long long *flag = const_cast<volatile unsigned long long *>(&P->timed_out);
    while (ld_acquire_sys(f) < seq) {
        if ((++polls & 1023u) != 0) continue;
        if (*flag) return;
        if (P->timeout_ns == 0) continue;
        const unsigned long long now = global_ns();
        if (t0 == 0) t0 = now;
        else if (now - t0 > P->timeout_ns) { *flag = 1ull; __threadfence_system(); return; }
    }
}

/* Block-wide: wait until every sender has published halo sequence `seq`. */
__device__ __forceinline__ void p2p_wait_halo(const acgb200_p2pdev *P, unsigned long long seq)
{
    if ((int) threadIdx.x < P->nsenders) p2p_spin(P->my_hflag + P->senders[threadIdx.x], seq, P);
    __syncthreads();
}

/* Block-wide: wait until every rank has published sequence `seq` on channel
 * `ch`, then sum the partials of that parity in rank order (the same order on
 * every rank, so all ranks get bit-identical sums).  out[0..1] in shared memory. */
__device__ __forceinline__ void p2p_reduce(const acgb200_p2pdev *P, int ch, int parity, unsigned long long seq, double *out)
{
    if ((int) threadIdx.x < P->nranks) p2p_spin(P->my_rflag + ch * ACGB200_MAXR + threadIdx.x, seq, P);
    __syncthreads();
    if (threadIdx.x == 0) {
        double a = 0.0, b = 0.0;
        for (int r = 0; r < P->nranks; r++) {
            const volatile double *s = P->my_red + RED_IDX(ch, parity, r);
            a += s[0]; b += s[1];
        }
        out[0] = a; out[1] = b;
    }
    __syncthreads();
}

/* sum of an already complete parity slot (no waiting) */
__device__ __forceinline__ double p2p_sum_slot(const acgb200_p2pdev *P, int ch, int parity)
{
    double a = 0.0;
    for (int r = 0; r < P->nranks; r++) a += ((const volatile double *) P->my_red)[RED_IDX(ch, parity, r)];
    return a;
}

/* True in exactly one CTA of the grid: the last one to get here.  Every CTA
 * must have fenced its own stores (system scope) before calling. */
__device__ __forceinline__ bool p2p_last_block(acgb200_p2pdev *P, int *flag_smem)
{
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned int t = atomicAdd(&P->ticket, 1u);
        *flag_smem = (t == gridDim.x - 1);
        if (*flag_smem) P->ticket = 0;
    }
    __syncthreads();
    const bool last = *flag_smem != 0;
    if (last) __threadfence_system();
    return last;
}

/* last CTA: write `count` reduction partials read from `src` (device scalars
 * completed by atomics of all CTAs) into every rank's slot, then the flags */
__device__ __forceinline__ void p2p_publish_red(acgb200_p2pdev *P, int ch, int parity, unsigned long long seq,
                                                double *src, int count)
{
    if ((int) threadIdx.x < P->nranks) {
        double *dst = P->peer_red[threadIdx.x] + RED_IDX(ch, parity, P->rank);
        dst[0] = atomicAdd(&src[0], 0.0);
        dst[1] = count > 1 ? atomicAdd(&src[1], 0.0) : 0.0;
        __threadfence_system();
        st_release_sys(P->peer_rflag[threadIdx.x] + ch * ACGB200_MAXR + P->rank, seq);
    }
}

__device__ __forceinline__ void p2p_publish_halo(acgb200_p2pdev *P, unsigned long long seq)
{
    if ((int) threadIdx.x < P->nrecip) st_release_sys(P->peer_hflag[threadIdx.x], seq);
}

/* a producer thread pushes the new value of border row `row` to the neighbours */
__device__ __forceinline__ void p2p_push_row(const acgb200_p2pdev *P, int row, int parity, double v)
{
    const int b = row - P->borderoff;
    for (int e = P->bptr[b]; e < P->bptr[b + 1]; e++) P->peer_ghost[P->bq[e]][parity][P->bdst[e]] = v;
}

/* Push halo values and/or reduction partials into the peers' windows, then
 * publish the sequence numbers (last block to finish does the publishing). */
__global__ void __launch_bounds__(512)
comm_post_kernel(const acgb200_postargs A)
{
    __shared__ int is_last;
    acgb200_p2pdev *P = A.p2p;
    int iter = A.iter_override;
    if (iter < 0) {
        const Gate g = gate_read(A.cin, A.st);
        if (!g.active) return;
        iter = g.iter;
    }
    if (A.vec) {
        const int parity = iter & 1;
        for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < P->sendsize; i += gridDim.x * blockDim.x) {
            int q = 0;
            while (i >= P->sdispls[q + 1]) q++;
            P->peer_ghost[q][parity][P->peer_rdispl[q] + (i - P->sdispls[q])] = A.vec[A.sendbufidx[i]];
        }
    }
    if (A.ch >= 0 && blockIdx.x == 0 && (int) threadIdx.x < P->nranks) {
        const int parity = (iter + A.par_off) & 1;
        const double *src = A.redbase + parity * A.redstride;
        double *dst = P->peer_red[threadIdx.x] + RED_IDX(A.ch, parity, P->rank);
        dst[0] = src[0];
        dst[1] = A.redcount > 1 ? src[1] : 0.0;
    }
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned int t = atomicAdd(&P->ticket, 1u);
        is_last = (t == gridDim.x - 1);
    }
    __syncthreads();
    if (!is_last) return;
    __threadfence_system();
    if (A.vec && (int) threadIdx.x < P->nrecip)
        st_release_sys(P->peer_hflag[threadIdx.x], P->hbase + (unsigned long long) iter);
    if (A.ch >= 0 && (int) threadIdx.x < P->nranks)
        st_release_sys(P->peer_rflag[threadIdx.x] + A.ch * ACGB200_MAXR + P->rank,
                       P->rbase + (unsigned long long) (iter + A.seq_off));
    if (threadIdx.x == 0) P->ticket = 0;
}

/* ------------------------------------------------------------------------ */
/* SpMV over TMA-staged row tiles                                            */
/* ------------------------------------------------------------------------ */

struct SpmvParams {
    const acgb200_tile *tiles;
    int ntiles;
    int sc;                 /* slots per stage for values/indices (multiple of 4) */
    int stage_bytes;
    int nstages;
    const int *rowptr;
    const int *colidx;
    const double *a;
    const double *x;
    double *y;
    const double *b;
    double *acc;
    int dotrows;
    int mode;
    const acgb200_ctrl *ctrl_in;
    acgb200_ctrl *ctrl_out;
    acgb200_devstate *st;
    int housekeeping;
    acgb200_p2pdev *p2p;
    int od_rowoffset, od_nrows;
    const int *orowptr;
    const int *ocolidx;
    const double *oa;
    int pub_ch;
};

__device__ __forceinline__ void spmv_issue(
    const SpmvParams &P, const acgb200_tile &tl, unsigned char *stage, uint64_t *bar, uint64_t pol)
{
    const int row_al = tl.row_begin & ~3;
    const int nrp = (tl.row_begin + tl.nrows + 1 - row_al + 3) & ~3;
    double *vals = reinterpret_cast<double *>(stage);
    int *cols = reinterpret_cast<int *>(stage + (size_t) P.sc * 8);
    int *rptr = reinterpret_cast<int *>(stage + (size_t) P.sc * 12);
    mbar_arrive_expect_tx(bar, (uint32_t) tl.nnz_al * 12u + (uint32_t) nrp * 4u);
    if (tl.nnz_al > 0) {
        bulk_g2s(vals, P.a + tl.k_al, (uint32_t) tl.nnz_al * 8u, bar, pol);
        bulk_g2s(cols, P.colidx + tl.k_al, (uint32_t) tl.nnz_al * 4u, bar, pol);
    }
    bulk_g2s(rptr, P.rowptr + row_al, (uint32_t) nrp * 4u, bar, pol);
}

/*
 * G lanes per row, T threads per CTA, U gathers in flight per lane.  A tile of
 * R rows is processed in ceil(R / (T/G)) passes; in a pass every G-lane group
 * owns one row and walks it in batches of U*G nonzeros: all U column indices
 * and values are read from shared memory first, then the U x-gathers are
 * issued back to back, then the FMAs -- the only long-latency operation (the
 * gather, an L1/L2 access) is thus U-deep per lane.  Slots past the end of the
 * row multiply a zero value with x[row's first column], which is always a
 * valid address.
 */
template <int G, int T, int U>
__global__ void __launch_bounds__(T, SPMV_MINB(T))
spmv_tiles_kernel(const SpmvParams P)
{
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ __align__(8) uint64_t full_bar[SPMV_MAX_STAGES];
    __shared__ double red[T / 32];
    __shared__ int last_flag;

    const int tid = threadIdx.x;
    pdl_prologue();
    const Gate gate = gate_read(P.ctrl_in, P.st);
    if (blockIdx.x == 0 && tid == 0 && P.ctrl_in) {
        *P.ctrl_out = *P.ctrl_in;
        if (gate.active) {
            /* zero the accumulator the *next* producer will add into; nothing
             * reads that slot while this kernel runs (DESIGN.md, control ring) */
            const int s = gate.iter & 1;
            if (P.housekeeping == 1) P.st->rr_loc[s ^ 1] = 0.0;
            if (P.housekeeping == 2) { P.st->gd_loc[s ^ 1][0] = 0.0; P.st->gd_loc[s ^ 1][1] = 0.0; }
        }
    }
    if (!gate.active) return;

    const int S = P.nstages;
    uint64_t pol = 0;
    if (tid == 0) {
        pol = l2_policy_evict_first();
        for (int s = 0; s < S; s++) mbar_init(&full_bar[s], 1);
        mbar_init_fence();
        for (int s = 0; s < S; s++) {
            const int t = blockIdx.x + s * gridDim.x;
            if (t < P.ntiles) spmv_issue(P, P.tiles[t], smem + (size_t) s * P.stage_bytes, &full_bar[s], pol);
        }
    }
    __syncthreads();

    constexpr int RPP = T / G;                 /* rows per pass */
    const int lane = tid % G;
    const int grp = tid / G;
    double dot = 0.0;
    const double *xg = NULL;            /* ghost values (peer-memory mode), set on the first border tile */

    int i = 0;
    for (int t = blockIdx.x; t < P.ntiles; t += gridDim.x, i++) {
        const int s = i % S;
        const acgb200_tile tl = P.tiles[t];
        if (P.p2p && !xg && tl.row_begin + tl.nrows > P.od_rowoffset) {
            /* first tile with border rows: from here on the neighbours' values
             * are needed.  Border rows come last, so by now they have long
             * arrived and the wait is a single flag read per sender. */
            p2p_wait_halo(P.p2p, P.p2p->hbase + (unsigned long long) gate.iter);
            xg = P.p2p->my_ghost[gate.iter & 1] - P.od_nrows;
        }
        unsigned char *stage = smem + (size_t) s * P.stage_bytes;
        const double *vals = reinterpret_cast<const double *>(stage);
        const int *cols = reinterpret_cast<const int *>(stage + (size_t) P.sc * 8);
        const int *rp = reinterpret_cast<const int *>(stage + (size_t) P.sc * 12) + (tl.row_begin & 3);

        mbar_wait(&full_bar[s], (uint32_t) ((i / S) & 1));

        for (int base = 0; base < tl.nrows; base += RPP) {
            const int lr = base + grp;
            double sum = 0.0;
            if (lr < tl.nrows) {
                const int kb = rp[lr] - tl.k_al;
                const int ke = rp[lr + 1] - tl.k_al;
                for (int k = kb + lane; k < ke; k += U * G) {
                    int c[U];
                    double v[U], xv[U];
                    /* slots past the row end re-read its last entry and are
                     * zeroed after the load: straight-line code, no predicated
                     * loads, so all U gathers are issued before the first FMA */
#pragma unroll
                    for (int u = 0; u < U; u++) {
                        const int kk = min(k + u * G, ke - 1);
                        c[u] = cols[kk];
                        v[u] = vals[kk];
                    }
#pragma unroll
                    for (int u = 0; u < U; u++) xv[u] = ld_x(P.x + c[u]);
#pragma unroll
                    for (int u = 0; u < U; u++) sum = fma((k + u * G < ke) ? v[u] : 0.0, xv[u], sum);
                }
                if (xg && tl.row_begin + lr >= P.od_rowoffset) {
                    /* border x ghost block (acg/cgcuda.c:878), ocolidx rebased by
                     * -borderrowoffset so ghosts start at od_nrows */
                    const int ob = tl.row_begin + lr - P.od_rowoffset;
                    for (int k = P.orowptr[ob] + lane; k < P.orowptr[ob + 1]; k += G)
                        sum = fma(P.oa[k], xg[P.ocolidx[k]], sum);
                }
            }
            if (G > 1) sum = group_sum<G>(sum);
            if (lr < tl.nrows && lane == 0) {
                const int row = tl.row_begin + lr;
                if (P.mode == SPMV_R_B_AX) {
                    const double v = P.b[row] - sum;
                    P.y[row] = v;
                    if (row < P.dotrows) dot = fma(v, v, dot);
                } else {
                    P.y[row] = sum;
                    if (P.mode == SPMV_Y_AX_DOT && row < P.dotrows) dot = fma(__ldg(P.x + row), sum, dot);
                }
            }
        }

        __syncthreads();        /* every thread is done reading stage s */
        if (tid == 0) {
            const int tn = t + S * gridDim.x;
            if (tn < P.ntiles) spmv_issue(P, P.tiles[tn], stage, &full_bar[s], pol);
        }
    }

    if (P.acc) {
        const double v = block_sum(dot, red);
        if (tid == 0 && v != 0.0) atomicAdd(P.acc, v);
    }
    if (P.p2p && P.pub_ch >= 0 && P.p2p->fuse) {
        /* the last CTA to finish sends this rank's share of the fused dot to all ranks */
        __threadfence();
        if (p2p_last_block(P.p2p, &last_flag))
            p2p_publish_red(P.p2p, P.pub_ch, gate.iter & 1, P.p2p->rbase + (unsigned long long) gate.iter + 1ull, P.acc, 1);
    }
}

/* ------------------------------------------------------------------------ */
/* SpMV over pattern slices (slices.c): index-free, slice-major values         */
/* ------------------------------------------------------------------------ */

struct SliceParams {
    const acgb200_slice *slices;
    int nslices;
    const double *sval;
    const unsigned short *patid;   /* pattern id per row; ACGB200_NOPATTERN: exception row (EXC kernels only) */
    const int *spatoff;            /* [npat * lpad], zero beyond a pattern's length */
    int npat, lpad;
    const int *rowptr;             /* CSR row pointers / column indices: the columns of exception rows */
    const int *colidx;
    const double *x;
    double *y;
    const double *b;
    double *acc;
    int dotrows;
    int mode;
    const acgb200_ctrl *ctrl_in;
    acgb200_ctrl *ctrl_out;        /* NULL: the tile kernel launched behind this one forwards the word */
    acgb200_devstate *st;
    int housekeeping;
};

/*
 * One warp per slice, one row per lane.  Entry slot e of the slice's 32 rows is
 * one coalesced 256-byte load (ld_stream); the column of lane's entry is
 * row + offset[pattern of the row][e] from a zero-padded table in shared memory,
 * so padded slots (value 0) gather x[row].  UB value loads and UB gathers are
 * issued back to back before the UB FMAs; a row's products are added in CSR
 * order into one accumulator.  No shared-memory staging of the matrix: residency
 * is limited by registers only, the loads in flight per SM (warps x UB x 256 B
 * of values) cover the HBM latency.
 */
/* xr = x + row.  (Forming the column in 32-bit arithmetic first -- one IADD + IMAD.WIDE instead of the
 * sign extension and 64-bit add below -- was tried and was slower.) */
template <int UB>
__device__ __forceinline__ void slice_load(double (&vv)[UB], double (&xv)[UB], const double *v, const double *xr,
                                           const int *offs, int e, uint64_t pol)
{
#pragma unroll
    for (int u = 0; u < UB; u++) vv[u] = ld_stream(v + (size_t) (e + u) * 32, pol);
#pragma unroll
    for (int u = 0; u < UB; u++) xv[u] = ld_x(xr + offs[e + u]);
}

template <int UB>
__device__ __forceinline__ double slice_fma(const double (&vv)[UB], const double (&xv)[UB], double sum)
{
#pragma unroll
    for (int u = 0; u < UB; u++) sum = fma(vv[u], xv[u], sum);
    return sum;
}

/* Shapes tried and dropped because they were slower at C3: prefetching the next batch into a second
 * register set (64-96 registers cost more warps than the prefetch buys), register caps of 40 / 32 per
 * thread (spills), 32-bit column arithmetic, batches of 14, 256- and 64-thread CTAs, 3-5 wide batches.
 *
 * EXC: the plan has slices with exception rows (rows outside the dictionary, slices.c).  A warp whose 32 rows are
 * all in the dictionary runs the same loop as the plain kernel; otherwise the exception lanes take each slot's
 * column from the CSR index array (one extra load per slot for those lanes only), everything else is unchanged.
 * The plain instantiation does not contain the exception path. */
template <int UB, int T, bool EXC>
__global__ void __launch_bounds__(T, EXC ? 1280 / T : 0)
spmv_slices_kernel(const SliceParams P)
{
    extern __shared__ __align__(16) int spat_s[];
    __shared__ double red[T / 32];
    const int tid = threadIdx.x;
    pdl_prologue();
    const Gate gate = gate_read(P.ctrl_in, P.st);
    if (P.ctrl_out && blockIdx.x == 0 && tid == 0 && P.ctrl_in) {
        *P.ctrl_out = *P.ctrl_in;
        if (gate.active) {
            const int s = gate.iter & 1;
            if (P.housekeeping == 1) P.st->rr_loc[s ^ 1] = 0.0;
            if (P.housekeeping == 2) { P.st->gd_loc[s ^ 1][0] = 0.0; P.st->gd_loc[s ^ 1][1] = 0.0; }
        }
    }
    if (!gate.active) return;
    for (int i = tid; i < P.npat * P.lpad; i += T) spat_s[i] = P.spatoff[i];
    __syncthreads();

    const uint64_t pol = l2_policy_evict_first();
    const int lane = tid & 31;
    const int warp = (blockIdx.x * T + tid) >> 5;
    const int nwarps = (gridDim.x * T) >> 5;
    double dot = 0.0;
    for (int s = warp; s < P.nslices; s += nwarps) {
        const int4 sl = __ldg(reinterpret_cast<const int4 *>(P.slices) + s);     /* row0, nrows, len, vblk */
        const int row = sl.x + lane;
        const int pid = P.patid[row];
        const bool exc = EXC && pid == (int) ACGB200_NOPATTERN;
        const int *offs = spat_s + (exc ? 0 : pid) * P.lpad;
        const double *v = P.sval + ((size_t) sl.w << 5) + lane;
        const double *xr = P.x + row;
        const int L = sl.z;
        double sum = 0.0;
        int e = 0;
        if (EXC && __any_sync(0xffffffffu, exc)) {
            /* a slice with exception rows: those lanes take their columns from the index array (slots past the
             * row's end hold the value 0 and gather x[row]).  Branch-free: every lane issues the index load --
             * the lanes that do not need it read colidx[0], one cached sector for the whole warp -- and selects. */
            int kb = 0, len = 1;
            if (exc) { kb = P.rowptr[row]; len = P.rowptr[row + 1] - kb; }
            const int *cbase = P.colidx + kb;
            const int last = exc ? max(len - 1, 0) : 0;
            for (; e + UB <= L; e += UB) {
                double vv[UB], xv[UB];
                int cc[UB];
#pragma unroll
                for (int u = 0; u < UB; u++) vv[u] = ld_stream(v + (size_t) (e + u) * 32, pol);
#pragma unroll
                for (int u = 0; u < UB; u++) cc[u] = __ldg(cbase + min(e + u, last));
#pragma unroll
                for (int u = 0; u < UB; u++) {
                    const int col = exc ? (e + u < len ? cc[u] : row) : row + offs[e + u];
                    xv[u] = ld_x(P.x + col);
                }
                sum = slice_fma<UB>(vv, xv, sum);
            }
            for (; e < L; e++) {                                   /* the last, partial batch slot by slot */
                const int c1 = __ldg(cbase + min(e, last));
                const int col = exc ? (e < len ? c1 : row) : row + offs[e];
                sum = fma(ld_stream(v + (size_t) e * 32, pol), ld_x(P.x + col), sum);
            }
        }
        for (; e + UB <= L; e += UB) {
            double vv[UB], xv[UB];
            slice_load<UB>(vv, xv, v, xr, offs, e, pol);
            sum = slice_fma<UB>(vv, xv, sum);
        }
        if (e < L) {
            /* last, partial batch: slots past L are neither loaded nor added */
            double vv[UB], xv[UB];
#pragma unroll
            for (int u = 0; u < UB; u++) vv[u] = e + u < L ? ld_stream(v + (size_t) (e + u) * 32, pol) : 0.0;
#pragma unroll
            for (int u = 0; u < UB; u++) xv[u] = e + u < L ? ld_x(xr + offs[e + u]) : 0.0;
#pragma unroll
            for (int u = 0; u < UB; u++) if (e + u < L) sum = fma(vv[u], xv[u], sum);
        }
        if (P.mode == SPMV_R_B_AX) {
            const double r = P.b[row] - sum;
            P.y[row] = r;
            if (row < P.dotrows) dot = fma(r, r, dot);
        } else {
            P.y[row] = sum;
            if (P.mode == SPMV_Y_AX_DOT && row < P.dotrows) dot = fma(__ldg(P.x + row), sum, dot);
        }
    }
    if (P.acc) {
        const double v = block_sum(dot, red);
        if (tid == 0 && v != 0.0) atomicAdd(P.acc, v);
    }
}

/* slice-major copy of the covered rows' values out of the device CSR arrays (once, at init) */
__global__ void __launch_bounds__(256)
slices_fill_kernel(int nslices, const acgb200_slice *slices, const int *__restrict__ rowptr,
                   const double *__restrict__ a, double *__restrict__ sval)
{
    const int lane = threadIdx.x & 31;
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int nwarps = (gridDim.x * blockDim.x) >> 5;
    for (int s = warp; s < nslices; s += nwarps) {
        const acgb200_slice sl = slices[s];
        const int row = sl.row0 + lane;
        const int kb = rowptr[row], len = rowptr[row + 1] - kb;
        double *v = sval + ((size_t) sl.vblk << 5) + lane;
        for (int e = 0; e < sl.len; e++) v[(size_t) e * 32] = e < len ? a[kb + e] : 0.0;
    }
}

/* ------------------------------------------------------------------------ */
/* SpMV over mirrored diagonals (slices.c): each symmetric value read once     */
/* ------------------------------------------------------------------------ */

struct SymdiagParams {
    const acgb200_slice *slices;
    int nslices;
    int no;                        /* entries per row, |O| */
    int nrows;                     /* columns are clamped to [0, nrows) */
    int evict_first;
    const double *hval;            /* the stored diagonals (fp64 layout) */
    const uint8_t *hcode;          /* ... or one code per element, in the same layout (coded layout) */
    const double *vtab;            /* the codes' values, ncodes <= 256 of them */
    int ncodes;
    acgb200_symdiag_entry tab[ACGB200_SYMDIAG_MAX];   /* (value offset, column offset) per entry, O ascending */
    const double *x;
    double *y;
    const double *b;
    double *acc;
    int dotrows;
    int mode;
    const acgb200_ctrl *ctrl_in;
    acgb200_ctrl *ctrl_out;
    acgb200_devstate *st;
    int housekeeping;
    /* pipelined-CG epilogue (PCG): x above is w_k; z, t, p, xs updated in place, w_{k+1} into w_next, r_k
     * read from r and r_{k+1} written to r_next; the catch-up form reads the group's lagged r's from r_next
     * and r_ring (pcg_catchup) */
    double *z, *t, *p, *r, *r_next, *xs, *w_next;
    const double *r_ring;
    size_t r_stride;
    int group;
    int vec_evict_first;
};

/*
 * The slice kernel without per-row patterns: one warp per covered slice, one row per lane, UB value loads
 * and UB gathers per batch.  Entry e of every row is value hval[voff_e + row] times x[row + coff_e]:
 * (voff_e, coff_e) is the same for the whole warp, one shared-memory broadcast.  An upper entry (coff >= 0)
 * is the row's own element of diagonal coff, a lower one the element of diagonal -coff at the mirror row
 * row + coff -- a copy of the same value, so half of the values are read a second time, from L2: the
 * grid-stride front spans far more rows than the largest mirror distance (DESIGN section 3a).
 *
 * The sum is the row's CSR-order FMA chain of spmv_slices_kernel: entries in ascending offset, one
 * accumulator; an offset the row does not have contributes fma(0, x[col], sum) == sum.  One difference
 * follows: such a slot gathers x at its (clamped) column where the slice kernel's padding gathers x[row],
 * so a non-finite x there makes the row NaN (0 * Inf) where the slice kernel may not.
 *
 * PCG: the whole pipelined-CG iteration k for the covered rows (DESIGN section 4a).  The row's sum is q_i
 * and goes straight into the update (pcg_row) instead of to memory; the kernel is the iteration's last, so
 * block 0 advances the control word and zeroes ring slot (k+2) % 3 while every CTA adds into (k+1) % 3.
 * A met convergence test returns before the product.  At most 40 registers: 12 CTAs of 128 threads.
 * CATCH: k is the last of its group of P.group iterations, so a pass over the same rows before the product
 * catches up on p and x for the group (pcg_catchup).
 *
 * V: double reads the fp64 diagonals (hval); uint8_t reads one code per element (hcode) and decodes it from
 * a copy of the value table in shared memory just before the FMAs -- the same double, bit for bit, so the
 * same sums.  The codes of a batch are loaded with the values' L2 policy, 32 bytes per warp and entry.
 *
 * X: the vector type.  float (the mixed-precision solve, modes SPMV_Y_AX and SPMV_Y_AX_DOT only) gathers
 * floats, widens them and runs the same fp64 FMA chain, then stores the sum rounded once to float; the
 * fused dot is over (x_i, fl32(y_i)), products of two floats and so exact in fp64.
 */
/* X = float: P.x and P.y hold the addresses of float vectors (the parameter block stays as it is) */
template <typename X> __device__ __forceinline__ const X *sd_vec(const double *p) { return reinterpret_cast<const X *>(p); }
template <typename X> __device__ __forceinline__ X *sd_vec(double *p) { return reinterpret_cast<X *>(p); }

__device__ __forceinline__ double sd_decode(double v, const double *) { return v; }
__device__ __forceinline__ double sd_decode(unsigned c, const double *vtab_s) { return vtab_s[c]; }

/* Row `row`'s sum of the mirrored-diagonal product: L entries in batches of UB value loads and UB gathers,
 * one FMA chain in ascending offset.  tab_s and vtab_s are the kernel's shared copies of P.tab and P.vtab. */
template <int UB, typename V, typename X>
__device__ __forceinline__ double symdiag_row_sum(const SymdiagParams &P, const int2 *tab_s, const double *vtab_s, int row,
                                                  uint64_t pol, int cmax, int L)
{
    constexpr bool CODED = std::is_same<V, uint8_t>::value;
    typedef decltype(ld_stream((const V *) nullptr, 0)) R;      /* a loaded value or code */
    const V *hv = (CODED ? (const V *) P.hcode : (const V *) P.hval) + row;
    double sum = 0.0;
    int e = 0;
    for (; e + UB <= L; e += UB) {
        R cv[UB];
        double vv[UB], xv[UB];
#pragma unroll
        for (int u = 0; u < UB; u++) cv[u] = ld_stream(hv + tab_s[e + u].x, pol);
#pragma unroll
        for (int u = 0; u < UB; u++) xv[u] = ld_x(sd_vec<X>(P.x) + min(max(row + tab_s[e + u].y, 0), cmax));
#pragma unroll
        for (int u = 0; u < UB; u++) vv[u] = sd_decode(cv[u], vtab_s);
        sum = slice_fma<UB>(vv, xv, sum);
    }
    if (e < L) {
        /* last, partial batch: slots past L are neither loaded nor added */
        R cv[UB];
        double vv[UB], xv[UB];
#pragma unroll
        for (int u = 0; u < UB; u++) cv[u] = e + u < L ? ld_stream(hv + tab_s[e + u].x, pol) : (R) 0;
#pragma unroll
        for (int u = 0; u < UB; u++) xv[u] = e + u < L ? ld_x(sd_vec<X>(P.x) + min(max(row + tab_s[e + u].y, 0), cmax)) : 0.0;
#pragma unroll
        for (int u = 0; u < UB; u++) vv[u] = sd_decode(cv[u], vtab_s);
#pragma unroll
        for (int u = 0; u < UB; u++) if (e + u < L) sum = fma(vv[u], xv[u], sum);
    }
    return sum;
}

template <int UB, int T, bool PCG, typename V, typename X = double, bool CATCH = false>
__global__ void __launch_bounds__(T, PCG ? 1536 / T : 0)
spmv_symdiag_kernel(const SymdiagParams P)
{
    constexpr bool CODED = std::is_same<V, uint8_t>::value;
    constexpr bool F32 = std::is_same<X, float>::value;
    static_assert(!(F32 && PCG), "the fused pipelined-CG epilogue is fp64 only");
    static_assert(PCG || !CATCH, "the catch-up form belongs to the fused epilogue");
    __shared__ int2 tab_s[ACGB200_SYMDIAG_MAX];
    __shared__ double vtab_s[CODED ? 256 : 1];
    __shared__ double red[T / 32];
    const int tid = threadIdx.x;
    pdl_prologue();
    const Gate gate = gate_read(P.ctrl_in, P.st);
    PcgStep k;
    if (PCG) {
        k = pcg_step(P.st, gate.iter);
        if (blockIdx.x == 0 && tid == 0) {
            acgb200_ctrl c = *P.ctrl_in;
            if (gate.active) {
                const int s = gate.iter & 1, z = (gate.iter + 2) % 3;
                P.st->gd_loc[z][0] = 0.0; P.st->gd_loc[z][1] = 0.0;
                if (k.conv) { c.done = 1; P.st->final_rr = k.gamma; }
                else {
                    c.iter = gate.iter + 1;
                    P.st->prev[s ^ 1][0] = k.gamma; P.st->prev[s ^ 1][1] = k.alpha;
                    double *ab = P.st->ab[gate.iter % ACGB200_PCG_GROUP_MAX];
                    ab[0] = k.alpha; ab[1] = k.beta;
                }
            }
            *P.ctrl_out = c;
        }
        if (!gate.active || k.conv) return;
    } else if (P.ctrl_out && blockIdx.x == 0 && tid == 0 && P.ctrl_in) {
        *P.ctrl_out = *P.ctrl_in;
        if (gate.active) {
            const int s = gate.iter & 1;
            if (P.housekeeping == 1) P.st->rr_loc[s ^ 1] = 0.0;
            if (P.housekeeping == 2) { P.st->gd_loc[s ^ 1][0] = 0.0; P.st->gd_loc[s ^ 1][1] = 0.0; }
        }
    }
    if (!gate.active) return;
    /* CATCH: {alpha_j, beta_j} for j = k-m+1 ... k and the ring for pcg_catchup, in shared memory; this kernel
     * writes only slot k of the device ring */
    __shared__ double ks_s[CATCH ? 2 * ACGB200_PCG_GROUP_MAX : 1];
    __shared__ PcgLag lag_s;
    if (CATCH) {
        const int m = P.group;
        if (tid < 2 * (m - 1)) ks_s[tid] = P.st->ab[(gate.iter - (m - 1) + (tid >> 1)) % ACGB200_PCG_GROUP_MAX][tid & 1];
        if (tid == 0) {
            ks_s[2 * m - 2] = k.alpha; ks_s[2 * m - 1] = k.beta;
            lag_s.ring = P.r_ring; lag_s.stride = P.r_stride; lag_s.m = m;
        }
    }
    if (tid < P.no) tab_s[tid] = make_int2(P.tab[tid].voff, P.tab[tid].coff);
    if (CODED) for (int i = tid; i < P.ncodes; i += T) vtab_s[i] = __ldg(P.vtab + i);
    __syncthreads();

    /* L2 policy of the values: see the measurements in DESIGN section 3a */
    const uint64_t pol = P.evict_first ? l2_policy_evict_first() : l2_policy_evict_normal();
    const int lane = tid & 31;
    const int warp = (blockIdx.x * T + tid) >> 5;
    const int nwarps = (gridDim.x * T) >> 5;
    const int cmax = P.nrows - 1;
    const int L = P.no;
    double dot = 0.0, dot2 = 0.0;
    /* the vector streams of the update pass through L2 once: see the measurements in DESIGN section 4a */
    const uint64_t vpol = PCG ? (P.vec_evict_first ? l2_policy_evict_first() : l2_policy_evict_normal()) : 0;
    if (CATCH) {
        /* the group's p and x, in a pass of their own so that the product loop keeps the plain form's
         * registers; the same rows on the same threads as that loop, which overwrites r_{k-m+1} */
        for (int s = warp; s < P.nslices; s += nwarps)
            pcg_catchup(__ldg(&P.slices[s].row0) + lane, ks_s, &lag_s, P.r_next, P.r, P.p, P.xs, vpol);
    }
    for (int s = warp; s < P.nslices; s += nwarps) {
        const int row = __ldg(&P.slices[s].row0) + lane;
        const double sum = symdiag_row_sum<UB, V, X>(P, tab_s, vtab_s, row, pol, cmax, L);
        if (PCG) {
            /* w_i was gathered by this row a moment ago: an L1 hit, not a third stream */
            pcg_row(row, sum, __ldg(P.x + row), k.alpha, k.beta, P.z, P.t, P.r, P.r_next, P.w_next, vpol, dot, dot2);
        } else if (F32) {
            const X ys = (X) sum;
            sd_vec<X>(P.y)[row] = ys;
            if (P.mode == SPMV_Y_AX_DOT && row < P.dotrows) dot = fma((double) __ldg(sd_vec<X>(P.x) + row), (double) ys, dot);
        } else if (P.mode == SPMV_R_B_AX) {
            const double r = P.b[row] - sum;
            P.y[row] = r;
            if (row < P.dotrows) dot = fma(r, r, dot);
        } else {
            P.y[row] = sum;
            if (P.mode == SPMV_Y_AX_DOT && row < P.dotrows) dot = fma(__ldg(P.x + row), sum, dot);
        }
    }
    if (PCG) {
        dot = block_sum(dot, red);
        dot2 = block_sum(dot2, red);
        if (tid == 0) {
            /* coded: the iteration index read again rather than kept live through the loop (the word this
             * kernel reads is not written during it) -- the UB = 9 loop would otherwise spill it */
            double *acc = P.st->gd_loc[((CODED ? P.ctrl_in->iter : gate.iter) + 1) % 3];
            atomicAdd(&acc[0], dot);
            atomicAdd(&acc[1], dot2);
        }
    } else if (P.acc) {
        const double v = block_sum(dot, red);
        if (tid == 0 && v != 0.0) atomicAdd(P.acc, v);
    }
}

struct SymdiagList { int d[ACGB200_SYMDIAG_MAX]; };

/* the stored diagonals out of the device CSR arrays (once, at init): element j of diagonal d[k] is
 * a[j, j + d[k]] for every owned row j; the array was zeroed, margins included */
__global__ void __launch_bounds__(256)
symdiag_fill_kernel(int nrows, const int *__restrict__ rowptr, const int *__restrict__ colidx,
                    const double *__restrict__ a, double *__restrict__ hval, int nd, const SymdiagList D,
                    int stride, int margin)
{
    __shared__ int d_s[ACGB200_SYMDIAG_MAX];
    if (threadIdx.x < nd) d_s[threadIdx.x] = D.d[threadIdx.x];
    __syncthreads();
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < nrows; j += gridDim.x * blockDim.x) {
        for (int k = rowptr[j]; k < rowptr[j + 1]; k++) {
            const int d = colidx[k] - j;
            if (d < 0) continue;
            for (int q = 0; q < nd; q++)
                if (d_s[q] == d) { hval[(size_t) q * stride + margin + j] = a[k]; break; }
        }
    }
}

/* Every covered row's lower entries must be the mirror values the kernel reads, bit for bit: for each
 * o < 0 in O, a[i, i+o] (or +0.0 where row i has no such entry) against the stored value at the mirror
 * row.  The rows are sorted (slices.c), so one pass over the row's entries.  Any difference sets *bad. */
__global__ void __launch_bounds__(256)
symdiag_check_kernel(SymdiagParams P, const int *__restrict__ rowptr, const int *__restrict__ colidx,
                     const double *__restrict__ a, int *bad)
{
    const long long nt = (long long) P.nslices * 32;
    for (long long t = blockIdx.x * (long long) blockDim.x + threadIdx.x; t < nt; t += (long long) gridDim.x * blockDim.x) {
        const int i = P.slices[t >> 5].row0 + (int) (t & 31);
        int k = rowptr[i];
        const int ke = rowptr[i + 1];
        for (int e = 0; e < P.no && P.tab[e].coff < 0; e++) {
            const int o = P.tab[e].coff;
            while (k < ke && colidx[k] - i < o) k++;
            const double want = (k < ke && colidx[k] - i == o) ? a[k] : 0.0;
            const double got = P.hval[(long long) P.tab[e].voff + i];
            if (__double_as_longlong(want) != __double_as_longlong(got)) *bad = 1;
        }
    }
}

/* ---- the coded layout (once, at init): distinct bit patterns -> sorted table -> codes -> check ---- */

#define CODES_EMPTY 0xFFFFFFFFFFFFFFFFull

__device__ __forceinline__ unsigned codes_hash(unsigned long long v)
{
    return (unsigned) ((v * 0x9E3779B97F4A7C15ull) >> 54) & (ACGB200_CODES_SET - 1);
}

/* insert v (not CODES_EMPTY) into an open-addressing set of ACGB200_CODES_SET slots; 1: newly inserted,
 * 0: already there, -1: the set is full */
__device__ __forceinline__ int codes_insert(unsigned long long *set, unsigned long long v)
{
    unsigned h = codes_hash(v);
    for (int probe = 0; probe < ACGB200_CODES_SET; probe++) {
        const unsigned long long old = atomicCAS(set + h, CODES_EMPTY, v);
        if (old == CODES_EMPTY) return 1;
        if (old == v) return 0;
        h = (h + 1) & (ACGB200_CODES_SET - 1);
    }
    return -1;
}

/* The distinct bit patterns of the n stored elements into cs->set.  Each CTA dedupes into a set in shared
 * memory first (and each thread skips a repeat of its previous element), so the ~10^8 elements of a
 * stencil matrix, nearly all one value, do not all contend for one global slot.  A CTA that sees more
 * than 256 patterns sets cs->overflow and stops. */
__global__ void __launch_bounds__(256)
codes_collect_kernel(const unsigned long long *__restrict__ h, long long n, acgb200_codestate *cs)
{
    __shared__ unsigned long long set_s[ACGB200_CODES_SET];
    __shared__ int n_s, ones_s;
    for (int i = threadIdx.x; i < ACGB200_CODES_SET; i += blockDim.x) set_s[i] = CODES_EMPTY;
    if (threadIdx.x == 0) { n_s = 0; ones_s = 0; }
    __syncthreads();
    unsigned long long last = CODES_EMPTY;
    bool have = false;
    for (long long i = blockIdx.x * (long long) blockDim.x + threadIdx.x; i < n; i += (long long) gridDim.x * blockDim.x) {
        const unsigned long long v = __ldg(h + i);
        if (have && v == last) continue;
        last = v; have = true;
        if (v == CODES_EMPTY) { ones_s = 1; continue; }
        if (*(volatile int *) &n_s > ACGB200_CODES_MAX) break;
        const int ins = codes_insert(set_s, v);
        if (ins > 0) atomicAdd(&n_s, 1);
        else if (ins < 0) { atomicAdd(&n_s, ACGB200_CODES_SET); break; }
    }
    __syncthreads();
    if (n_s > ACGB200_CODES_MAX) { if (threadIdx.x == 0) cs->overflow = 1; return; }
    if (threadIdx.x == 0 && ones_s) cs->has_ones = 1;
    for (int i = threadIdx.x; i < ACGB200_CODES_SET; i += blockDim.x)
        if (set_s[i] != CODES_EMPTY && codes_insert(cs->set, set_s[i]) < 0) cs->overflow = 1;
}

/* one CTA: the set's patterns sorted ascending by bit pattern into cs->vtab (the rank of each pattern is
 * the number of smaller ones), cs->ncodes = their number, or 0 on overflow */
__global__ void __launch_bounds__(1024)
codes_sort_kernel(acgb200_codestate *cs)
{
    __shared__ unsigned long long k_s[ACGB200_CODES_SET + 1];
    __shared__ int n_s;
    if (threadIdx.x == 0) n_s = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < ACGB200_CODES_SET; i += blockDim.x) {
        const unsigned long long v = cs->set[i];
        if (v != CODES_EMPTY) k_s[atomicAdd(&n_s, 1)] = v;
    }
    __syncthreads();
    if (threadIdx.x == 0 && cs->has_ones) k_s[n_s++] = CODES_EMPTY;
    __syncthreads();
    const int n = n_s;
    if (cs->overflow || n > ACGB200_CODES_MAX) { if (threadIdx.x == 0) cs->ncodes = 0; return; }
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const unsigned long long v = k_s[i];
        int rank = 0;
        for (int j = 0; j < n; j++) rank += k_s[j] < v;
        cs->vtab[rank] = __longlong_as_double((long long) v);
    }
    if (threadIdx.x == 0) cs->ncodes = n;
}

/* code[i] = the index of h[i] in the sorted table (binary search; a thread reuses its previous element's
 * code when the pattern repeats) */
__global__ void __launch_bounds__(256)
codes_encode_kernel(const unsigned long long *__restrict__ h, uint8_t *__restrict__ code, long long n,
                    const acgb200_codestate *cs)
{
    __shared__ unsigned long long t_s[ACGB200_CODES_MAX];
    const int nc = cs->ncodes;
    if (nc == 0) return;
    for (int i = threadIdx.x; i < nc; i += blockDim.x) t_s[i] = (unsigned long long) __double_as_longlong(cs->vtab[i]);
    __syncthreads();
    unsigned long long last = t_s[0];
    int c = 0;
    for (long long i = blockIdx.x * (long long) blockDim.x + threadIdx.x; i < n; i += (long long) gridDim.x * blockDim.x) {
        const unsigned long long v = __ldg(h + i);
        if (v != last) {
            int lo = 0, hi = nc - 1;
            while (lo < hi) { const int mid = (lo + hi) >> 1; if (t_s[mid] < v) lo = mid + 1; else hi = mid; }
            last = v; c = lo;
        }
        code[i] = (uint8_t) c;
    }
}

/* every code must decode to its element bit for bit; any difference sets cs->bad */
__global__ void __launch_bounds__(256)
codes_check_kernel(const unsigned long long *__restrict__ h, const uint8_t *__restrict__ code, long long n,
                   acgb200_codestate *cs)
{
    __shared__ unsigned long long t_s[ACGB200_CODES_MAX];
    const int nc = cs->ncodes;
    if (nc == 0) return;
    for (int i = threadIdx.x; i < nc; i += blockDim.x) t_s[i] = (unsigned long long) __double_as_longlong(cs->vtab[i]);
    __syncthreads();
    bool bad = false;
    for (long long i = blockIdx.x * (long long) blockDim.x + threadIdx.x; i < n; i += (long long) gridDim.x * blockDim.x) {
        const int c = code[i];
        bad |= c >= nc || t_s[c] != __ldg(h + i);
    }
    if (__syncthreads_or(bad) && threadIdx.x == 0) cs->bad = 1;
}

/* ------------------------------------------------------------------------ */
/* SpMV over merge-path tiles (mergeplan.c): power-law row lengths             */
/* ------------------------------------------------------------------------ */

struct MergeParams {
    const acgb200_mtile *tiles;
    int ntiles;
    int sc, rc;                    /* value/index slots and row-pointer slots per stage (multiples of 4) */
    int stage_bytes, nstages;
    const int *rowptr;
    const int *colidx;
    const double *a;
    double *part;                  /* [2 * ntiles] */
    const double *x;
    double *y;
    const double *b;
    double *acc;
    int dotrows;
    int mode;
    const acgb200_ctrl *ctrl_in;
    acgb200_ctrl *ctrl_out;        /* NULL: the tile kernel launched behind this one forwards the word */
    acgb200_devstate *st;
    int housekeeping;
};

#define MERGE_LONGSEG 32           /* pieces longer than this are summed by a whole warp */
#define MERGE_LISTCAP 128

__device__ __forceinline__ void merge_issue(const MergeParams &P, const acgb200_mtile &tl, unsigned char *stage,
                                            uint64_t *bar, uint64_t pol)
{
    const int k_al = tl.k0 & ~3;
    const int nnz_al = (tl.k0 + tl.nnz - k_al + 3) & ~3;
    const int row_al = tl.r0 & ~3;
    const int nrp = (tl.r0 + tl.nre + 1 - row_al + 3) & ~3;
    double *vals = reinterpret_cast<double *>(stage);
    int *cols = reinterpret_cast<int *>(stage + (size_t) P.sc * 8);
    int *rptr = reinterpret_cast<int *>(stage + (size_t) P.sc * 12);
    mbar_arrive_expect_tx(bar, (uint32_t) nnz_al * 12u + (uint32_t) nrp * 4u);
    if (nnz_al > 0) {
        bulk_g2s(vals, P.a + k_al, (uint32_t) nnz_al * 8u, bar, pol);
        bulk_g2s(cols, P.colidx + k_al, (uint32_t) nnz_al * 4u, bar, pol);
    }
    bulk_g2s(rptr, P.rowptr + row_al, (uint32_t) nrp * 4u, bar, pol);
}

/* what a finished row does with its sum (same epilogues as the tile kernel) */
__device__ __forceinline__ void spmv_row_epilogue(int row, double sum, int mode, const double *x, double *y, const double *b,
                                                  int dotrows, double &dot)
{
    if (mode == SPMV_R_B_AX) {
        const double v = b[row] - sum;
        y[row] = v;
        if (row < dotrows) dot = fma(v, v, dot);
    } else {
        y[row] = sum;
        if (mode == SPMV_Y_AX_DOT && row < dotrows) dot = fma(__ldg(x + row), sum, dot);
    }
}

/*
 * Per tile: (1) every thread multiplies a strided share of the tile's nonzeros -- U gathers in
 * flight, equal work for all threads whatever the rows look like -- and leaves the products in
 * shared memory; (2) the tile's units (one per row end, plus the piece behind the last row end) are
 * summed from shared memory: a thread per unit, units longer than MERGE_LONGSEG by a warp.  A unit
 * that is a whole row gets the epilogue; the piece of a split row goes to part[] for the fix-up
 * kernel (slot 0: the row ends here but began in an earlier tile; slot 1: the row continues).
 */
template <int T, int U>
__global__ void __launch_bounds__(T)
spmv_merge_kernel(const MergeParams P)
{
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ __align__(8) uint64_t full_bar[SPMV_MAX_STAGES];
    __shared__ double red[T / 32];
    __shared__ int lst[MERGE_LISTCAP];
    __shared__ int nlst;

    const int tid = threadIdx.x;
    pdl_prologue();
    const Gate gate = gate_read(P.ctrl_in, P.st);
    if (P.ctrl_out && blockIdx.x == 0 && tid == 0 && P.ctrl_in) {
        *P.ctrl_out = *P.ctrl_in;
        if (gate.active) {
            const int s = gate.iter & 1;
            if (P.housekeeping == 1) P.st->rr_loc[s ^ 1] = 0.0;
            if (P.housekeeping == 2) { P.st->gd_loc[s ^ 1][0] = 0.0; P.st->gd_loc[s ^ 1][1] = 0.0; }
        }
    }
    if (!gate.active) return;

    const int S = P.nstages;
    double *prod = reinterpret_cast<double *>(smem + (size_t) S * P.stage_bytes);     /* [sc] products of the current tile */
    uint64_t pol = 0;
    if (tid == 0) {
        nlst = 0;
        pol = l2_policy_evict_first();
        for (int s = 0; s < S; s++) mbar_init(&full_bar[s], 1);
        mbar_init_fence();
        for (int s = 0; s < S; s++) {
            const int t = blockIdx.x + s * gridDim.x;
            if (t < P.ntiles) merge_issue(P, P.tiles[t], smem + (size_t) s * P.stage_bytes, &full_bar[s], pol);
        }
    }
    __syncthreads();

    double dot = 0.0;
    int i = 0;
    for (int t = blockIdx.x; t < P.ntiles; t += gridDim.x, i++) {
        const int s = i % S;
        const acgb200_mtile tl = P.tiles[t];
        unsigned char *stage = smem + (size_t) s * P.stage_bytes;
        const int koff = tl.k0 & 3;                    /* first own nonzero inside the 16-byte aligned slice */
        const double *vals = reinterpret_cast<const double *>(stage) + koff;
        const int *cols = reinterpret_cast<const int *>(stage + (size_t) P.sc * 8) + koff;
        const int *rp = reinterpret_cast<const int *>(stage + (size_t) P.sc * 12) + (tl.r0 & 3);    /* rp[j] = rowptr[r0 + j] */

        mbar_wait(&full_bar[s], (uint32_t) ((i / S) & 1));

        /* (1) products */
        for (int base = 0; base < tl.nnz; base += T * U) {
            int c[U];
            double v[U], xv[U];
#pragma unroll
            for (int u = 0; u < U; u++) {
                const int kk = min(base + u * T + tid, tl.nnz - 1);
                c[u] = cols[kk];
                v[u] = vals[kk];
            }
#pragma unroll
            for (int u = 0; u < U; u++) xv[u] = ld_x(P.x + c[u]);
#pragma unroll
            for (int u = 0; u < U; u++) {
                const int kk = base + u * T + tid;
                if (kk < tl.nnz) prod[kk] = v[u] * xv[u];
            }
        }
        __syncthreads();

        /* (2a) a thread per unit: j < nre is row r0 + j, j == nre the piece behind the last row end */
        const int kend = tl.k0 + tl.nnz;
        for (int j = tid; j <= tl.nre; j += T) {
            const int a0 = max(rp[j], tl.k0) - tl.k0;
            const int b0 = (j < tl.nre ? rp[j + 1] : kend) - tl.k0;
            if (b0 - a0 > MERGE_LONGSEG) {
                const int slot = atomicAdd(&nlst, 1);
                if (slot < MERGE_LISTCAP) { lst[slot] = j; continue; }
                /* (cannot happen: a tile holds fewer than MERGE_LISTCAP pieces of that length; summed here if it did) */
            }
            double sum = 0.0;
            for (int k = a0; k < b0; k++) sum += prod[k];
            if (j == tl.nre) P.part[2 * (size_t) t + 1] = sum;
            else if (j == 0 && rp[0] < tl.k0) P.part[2 * (size_t) t] = sum;
            else spmv_row_epilogue(tl.r0 + j, sum, P.mode, P.x, P.y, P.b, P.dotrows, dot);
        }
        if (tid == 0 && !(tl.nre > 0 && rp[0] < tl.k0)) P.part[2 * (size_t) t] = 0.0;      /* no head piece in this tile */
        __syncthreads();

        /* (2b) long units: a warp each, lanes stride over the piece, fixed shuffle tree */
        const int nl = min(nlst, MERGE_LISTCAP);
        for (int q = tid >> 5; q < nl; q += T / 32) {
            const int j = lst[q];
            const int a0 = max(rp[j], tl.k0) - tl.k0;
            const int b0 = (j < tl.nre ? rp[j + 1] : kend) - tl.k0;
            double sum = 0.0;
            for (int k = a0 + (tid & 31); k < b0; k += 32) sum += prod[k];
            sum = warp_sum(sum);
            if ((tid & 31) == 0) {
                if (j == tl.nre) P.part[2 * (size_t) t + 1] = sum;
                else if (j == 0 && rp[0] < tl.k0) P.part[2 * (size_t) t] = sum;
                else spmv_row_epilogue(tl.r0 + j, sum, P.mode, P.x, P.y, P.b, P.dotrows, dot);
            }
        }
        __syncthreads();        /* stage s, prod[] and the list are free again */
        if (tid == 0) {
            nlst = 0;
            const int tn = t + S * gridDim.x;
            if (tn < P.ntiles) merge_issue(P, P.tiles[tn], stage, &full_bar[s], pol);
        }
    }

    if (P.acc) {
        const double v = block_sum(dot, red);
        if (tid == 0 && v != 0.0) atomicAdd(P.acc, v);
    }
}

/* split rows: add the pieces in tile order (a warp per row), then the row's epilogue */
__global__ void __launch_bounds__(256)
spmv_merge_fix_kernel(int nsplit, const acgb200_msplit *split, const double *part,
                      const double *x, double *y, const double *b, double *acc, int dotrows, int mode,
                      const acgb200_ctrl *cin, const acgb200_devstate *st)
{
    __shared__ double red[8];
    if (!gate_read(cin, st).active) return;
    const int lane = threadIdx.x & 31;
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int nwarps = (gridDim.x * blockDim.x) >> 5;
    double dot = 0.0;
    for (int i = warp; i < nsplit; i += nwarps) {
        const acgb200_msplit sp = split[i];
        double sum = 0.0;
        for (int t = sp.ta + lane; t < sp.tb; t += 32) sum += part[2 * (size_t) t + 1];
        sum = warp_sum(sum);
        if (lane == 0) {
            sum += part[2 * (size_t) sp.tb];
            spmv_row_epilogue(sp.row, sum, mode, x, y, b, dotrows, dot);
        }
    }
    if (acc) {
        dot = block_sum(dot, red);
        if (threadIdx.x == 0 && dot != 0.0) atomicAdd(acc, dot);
    }
}

/* ---- long rows: several CTAs per row, partials to scratch, then a finisher -- */

__global__ void __launch_bounds__(256)
spmv_long_partial_kernel(int nlong, const int *longrows, int chunks,
                         const int *rowptr, const int *colidx, const double *a, const double *x,
                         double *scratch, const acgb200_ctrl *cin, const acgb200_devstate *st)
{
    __shared__ double red[8];
    if (!gate_read(cin, st).active) return;
    const int lrow = blockIdx.x / chunks, chunk = blockIdx.x % chunks;
    const int row = longrows[lrow];
    const long long kb = rowptr[row], ke = rowptr[row + 1];
    const long long len = ke - kb;
    const long long c0 = kb + len * chunk / chunks, c1 = kb + len * (chunk + 1) / chunks;
    double sum = 0.0;
    for (long long k = c0 + threadIdx.x; k < c1; k += blockDim.x)
        sum = fma(a[k], __ldg(x + colidx[k]), sum);
    sum = block_sum(sum, red);
    if (threadIdx.x == 0) scratch[blockIdx.x] = sum;
}

__global__ void spmv_long_finish_kernel(int nlong, const int *longrows, int chunks, const double *scratch,
                                        const double *x, double *y, const double *b, double *acc,
                                        int dotrows, int mode, const acgb200_ctrl *cin, const acgb200_devstate *st,
                                        const acgb200_p2pdev *p2p, int od_rowoffset, int od_nrows,
                                        const int *orowptr, const int *ocolidx, const double *oa)
{
    const Gate g = gate_read(cin, st);
    if (!g.active) return;
    /* peer-memory mode: long rows that are border rows also get their
     * border x ghost entries here (the tile kernel only sees rows in tiles) */
    const double *xg = NULL;
    if (p2p) {
        p2p_wait_halo(p2p, p2p->hbase + (unsigned long long) g.iter);
        xg = p2p->my_ghost[g.iter & 1] - od_nrows;
    }
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    double dot = 0.0;
    if (i < nlong) {
        const int row = longrows[i];
        double sum = 0.0;
        for (int c = 0; c < chunks; c++) sum += scratch[(size_t) i * chunks + c];
        if (xg && row >= od_rowoffset) {
            const int ob = row - od_rowoffset;
            for (int k = orowptr[ob]; k < orowptr[ob + 1]; k++) sum = fma(oa[k], xg[ocolidx[k]], sum);
        }
        if (mode == SPMV_R_B_AX) {
            const double v = b[row] - sum; y[row] = v;
            if (row < dotrows) dot = v * v;
        } else {
            y[row] = sum;
            if (mode == SPMV_Y_AX_DOT && row < dotrows) dot = x[row] * sum;
        }
    }
    dot = warp_sum(dot);
    if (acc && (threadIdx.x & 31) == 0 && dot != 0.0) atomicAdd(acc, dot);
}

/* ---- medium rows: one warp per row, straight from global memory (opt-in) ----- */

/*
 * Rows that would monopolise one G-lane group of a tile (a few hundred to a
 * couple of thousand nonzeros, the body of a power-law degree distribution) are
 * taken out of the tiles by the planner when option "spmv_medium" is set and
 * processed here: a warp walks its row with coalesced 32-wide accesses, four
 * gathers in flight per lane, and applies the same epilogue as the tile kernel.
 * Persistent grid, warps stride over the list; one atomic per CTA for the dot.
 */
__global__ void __launch_bounds__(256)
spmv_medium_kernel(int nmed, const int *medrows,
                   const int *rowptr, const int *colidx, const double *a, const double *x,
                   double *y, const double *b, double *acc, int dotrows, int mode,
                   const acgb200_ctrl *cin, const acgb200_devstate *st,
                   const acgb200_p2pdev *p2p, int od_rowoffset, int od_nrows,
                   const int *orowptr, const int *ocolidx, const double *oa)
{
    __shared__ double red[8];
    const Gate g = gate_read(cin, st);
    if (!g.active) return;
    const double *xg = NULL;
    if (p2p) {
        p2p_wait_halo(p2p, p2p->hbase + (unsigned long long) g.iter);
        xg = p2p->my_ghost[g.iter & 1] - od_nrows;
    }
    const int lane = threadIdx.x & 31;
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int nwarps = (gridDim.x * blockDim.x) >> 5;
    double dot = 0.0;
    for (int i = warp; i < nmed; i += nwarps) {
        const int row = medrows[i];
        const int kb = rowptr[row], ke = rowptr[row + 1];
        double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
        int k = kb + lane;
        for (; k + 96 < ke; k += 128) {
            const double x0 = __ldg(x + colidx[k]), x1 = __ldg(x + colidx[k + 32]);
            const double x2 = __ldg(x + colidx[k + 64]), x3 = __ldg(x + colidx[k + 96]);
            s0 = fma(a[k], x0, s0); s1 = fma(a[k + 32], x1, s1);
            s2 = fma(a[k + 64], x2, s2); s3 = fma(a[k + 96], x3, s3);
        }
        for (; k < ke; k += 32) s0 = fma(a[k], __ldg(x + colidx[k]), s0);
        double sum = (s0 + s1) + (s2 + s3);
        if (xg && row >= od_rowoffset) {
            const int ob = row - od_rowoffset;
            for (int j = orowptr[ob] + lane; j < orowptr[ob + 1]; j += 32) sum = fma(oa[j], xg[ocolidx[j]], sum);
        }
        sum = warp_sum(sum);
        if (lane == 0) {
            if (mode == SPMV_R_B_AX) {
                const double v = b[row] - sum;
                y[row] = v;
                if (row < dotrows) dot = fma(v, v, dot);
            } else {
                y[row] = sum;
                if (mode == SPMV_Y_AX_DOT && row < dotrows) dot = fma(x[row], sum, dot);
            }
        }
    }
    if (acc) {
        dot = block_sum(dot, red);
        if (threadIdx.x == 0 && dot != 0.0) atomicAdd(acc, dot);
    }
}

/* ---- border x ghost block: thread per border row, direct from global -------- */

__global__ void __launch_bounds__(256)
offdiag_kernel(const acgb200_offdiagargs A)
{
    __shared__ double red[8];
    const Gate g = gate_read(A.ctrl_in, A.st);
    if (!g.active) return;
    /* ghost values: the tail of x (filled by ncclRecv) or, with the peer-memory
     * exchange, this iteration's parity buffer of the window, valid once every
     * sender has published the iteration's sequence number.  ocolidx is rebased
     * by -borderrowoffset (acg/symcsrmatrix.c:838), ghosts start at nrows. */
    const double *xg = A.x + A.rowoffset;
    if (A.p2p) {
        const int it = A.p2p_iter_override >= 0 ? A.p2p_iter_override : g.iter;
        p2p_wait_halo(A.p2p, A.p2p->hbase + (unsigned long long) it);
        xg = A.p2p->my_ghost[it & 1] - A.nrows;
    }
    double dot = 0.0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < A.nrows; i += gridDim.x * blockDim.x) {
        const int kb = A.orowptr[i], ke = A.orowptr[i + 1];
        const int row = A.rowoffset + i;
        double sum = 0.0;
        for (int k = kb; k < ke; k++) sum = fma(A.oa[k], xg[A.ocolidx[k]], sum);
        double v = A.y[row];
        if (kb != ke) { v = A.minus ? v - sum : v + sum; A.y[row] = v; }
        if (A.dotkind == 1) dot = fma(__ldg(A.x + row), v, dot);
        else if (A.dotkind == 2) dot = fma(v, v, dot);
    }
    if (A.acc) {
        dot = block_sum(dot, red);
        if (threadIdx.x == 0 && dot != 0.0) atomicAdd(A.acc, dot);
    }
}

/* ------------------------------------------------------------------------ */
/* fused BLAS-1                                                              */
/* ------------------------------------------------------------------------ */

/* r -= alpha t with alpha = (r,r)/(p,Ap), and the new (r,r) in the same pass */
__global__ void __launch_bounds__(BLAS1_THREADS)
cg_update_r_kernel(int n, acgb200_devstate *st, int cin, int cout, int multi, acgb200_p2pdev *P,
                   const double *__restrict__ t, double *__restrict__ r)
{
    __shared__ double red[BLAS1_THREADS / 32];
    __shared__ double glob[2];
    __shared__ int last_flag;
    pdl_prologue();
    const Gate g = gate_read(&st->ctrl[cin], st);
    if (cin != cout && blockIdx.x == 0 && threadIdx.x == 0) st->ctrl[cout] = st->ctrl[cin];
    if (!g.active) return;
    const int s = g.iter & 1;
    double rr, pap;
    if (P) {
        /* (p,Ap) of this iteration arrives on channel 0; (r,r) was completed on
         * channel 1 one iteration ago (setup value for the first iteration) */
        p2p_reduce(P, 0, s, P->rbase + (unsigned long long) g.iter + 1ull, glob);
        pap = glob[0];
        rr = g.iter > 0 ? p2p_sum_slot(P, 1, s) : st->rr[0];
    } else {
        rr = multi ? st->rr[s] : st->rr_loc[s];
        pap = multi ? st->pap[s] : st->pap_loc[s];
    }
    const double alpha = rr / pap;
    double acc = 0.0;
    const int n2 = n >> 1;
    const double2 *t2 = reinterpret_cast<const double2 *>(t);
    double2 *r2 = reinterpret_cast<double2 *>(r);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n2; i += gridDim.x * blockDim.x) {
        const double2 tv = t2[i];
        double2 rv = r2[i];
        rv.x = fma(-alpha, tv.x, rv.x);
        rv.y = fma(-alpha, tv.y, rv.y);
        r2[i] = rv;
        acc = fma(rv.x, rv.x, acc);
        acc = fma(rv.y, rv.y, acc);
    }
    if ((n & 1) && blockIdx.x == 0 && threadIdx.x == 0) {
        const double rv = fma(-alpha, t[n - 1], r[n - 1]);
        r[n - 1] = rv;
        acc = fma(rv, rv, acc);
    }
    acc = block_sum(acc, red);
    if (threadIdx.x == 0) atomicAdd(&st->rr_loc[s ^ 1], acc);
    if (P && P->fuse) {
        __threadfence();
        if (p2p_last_block(P, &last_flag))
            p2p_publish_red(P, 1, s ^ 1, P->rbase + (unsigned long long) g.iter + 1ull, &st->rr_loc[s ^ 1], 1);
    }
}

/* x += alpha p ; p = r + beta p ; decides convergence for the next iteration */
__global__ void __launch_bounds__(BLAS1_THREADS)
cg_update_xp_kernel(int n, acgb200_devstate *st, int cin, int cout, int multi, acgb200_p2pdev *P,
                    const double *__restrict__ r, double *__restrict__ p, double *__restrict__ x)
{
    __shared__ double glob[2];
    __shared__ int last_flag;
    pdl_prologue();
    const Gate g = gate_read(&st->ctrl[cin], st);
    const int s = g.iter & 1;
    double rr, rrn, pap;
    if (P && g.active) {
        p2p_reduce(P, 1, s ^ 1, P->rbase + (unsigned long long) g.iter + 1ull, glob);
        rrn = glob[0];
        rr = g.iter > 0 ? p2p_sum_slot(P, 1, s) : st->rr[0];
        pap = p2p_sum_slot(P, 0, s);
    } else {
        rr = multi ? st->rr[s] : st->rr_loc[s];
        rrn = multi ? st->rr[s ^ 1] : st->rr_loc[s ^ 1];
        pap = multi ? st->pap[s] : st->pap_loc[s];
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        acgb200_ctrl c = st->ctrl[cin];
        if (g.active) {
            c.iter = g.iter + 1;
            if (P) st->rr[s ^ 1] = rrn;    /* keep the global value where the host reads it */
            /* acg/cgcuda.c:1008-1012: test ||r|| < tol with the norm, strictly */
            if (st->tol > 0.0 && sqrt(rrn) < st->tol) { c.done = 1; st->final_rr = rrn; }
            st->pap_loc[s ^ 1] = 0.0;      /* accumulator of the next SpMV */
        }
        st->ctrl[cout] = c;
    }
    if (!g.active) return;
    const double alpha = rr / pap;
    const double beta = rrn / rr;
    const int n2 = n >> 1;
    const double2 *r2 = reinterpret_cast<const double2 *>(r);
    double2 *p2 = reinterpret_cast<double2 *>(p);
    double2 *x2 = reinterpret_cast<double2 *>(x);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n2; i += gridDim.x * blockDim.x) {
        const double2 rv = r2[i];
        double2 pv = p2[i];
        double2 xv = x2[i];
        xv.x = fma(alpha, pv.x, xv.x);
        xv.y = fma(alpha, pv.y, xv.y);
        pv.x = fma(beta, pv.x, rv.x);
        pv.y = fma(beta, pv.y, rv.y);
        x2[i] = xv;
        p2[i] = pv;
        if (P && P->fuse && 2 * i + 1 >= P->borderoff) {
            /* p is the input of the next SpMV: its border entries go straight
             * into the neighbours' ghost buffers of the next iteration's parity */
            if (2 * i >= P->borderoff) p2p_push_row(P, 2 * i, s ^ 1, pv.x);
            p2p_push_row(P, 2 * i + 1, s ^ 1, pv.y);
        }
    }
    if ((n & 1) && blockIdx.x == 0 && threadIdx.x == 0) {
        const double pv = p[n - 1];
        x[n - 1] = fma(alpha, pv, x[n - 1]);
        const double pn = fma(beta, pv, r[n - 1]);
        p[n - 1] = pn;
        if (P && P->fuse && n - 1 >= P->borderoff) p2p_push_row(P, n - 1, s ^ 1, pn);
    }
    if (P && P->fuse) {
        __threadfence_system();
        if (p2p_last_block(P, &last_flag)) p2p_publish_halo(P, P->hbase + (unsigned long long) g.iter + 1ull);
    }
}

/* Pipelined CG: z=q+beta z; t=w+beta t; p=r+beta p; x+=alpha p; r-=alpha t;
 * w-=alpha z (acg/cg-kernels-cuda.cu:201-214), plus gamma'=(r,r), delta'=(w,r)
 * of the updated vectors for the next iteration. */
/* (Tried and dropped: two rows per thread and trip -- faster at one rank's share of the 8-GPU problem,
 * slower at C3, no gain between two GPUs; the system fence moved behind the border rows -- no effect.) */
__global__ void __launch_bounds__(BLAS1_THREADS)
pcg_update_kernel(int n, acgb200_devstate *st, int cin, int cout, int multi, acgb200_p2pdev *P,
                  const double *__restrict__ q, double *__restrict__ z, double *__restrict__ w,
                  double *__restrict__ t, double *__restrict__ p, double *__restrict__ r,
                  double *__restrict__ x)
{
    __shared__ double red[BLAS1_THREADS / 32];
    __shared__ double glob[2];
    __shared__ int last_flag;
    pdl_prologue();
    const Gate g = gate_read(&st->ctrl[cin], st);
    const int s = g.iter & 1;
    double gamma, delta;
    if (P && g.active && g.iter > 0) {
        /* {gamma,delta} pushed by every rank after its previous update */
        p2p_reduce(P, 0, s, P->rbase + (unsigned long long) g.iter, glob);
        gamma = glob[0]; delta = glob[1];
    } else {
        gamma = multi ? st->gd[s][0] : st->gd_loc[s][0];
        delta = multi ? st->gd[s][1] : st->gd_loc[s][1];
    }
    const double gamma_prev = st->prev[s][0], alpha_prev = st->prev[s][1];
    /* acg/cgcuda.c:1764-1772: the test precedes the update */
    const bool conv = st->tol > 0.0 && sqrt(gamma) < st->tol;
    const double beta = gamma / gamma_prev;
    const double alpha = gamma / (delta - beta * gamma / alpha_prev);
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        acgb200_ctrl c = st->ctrl[cin];
        if (g.active) {
            if (P) { st->gd[s][0] = gamma; st->gd[s][1] = delta; }   /* for the host's final report */
            if (conv) { c.done = 1; st->final_rr = gamma; }
            else { c.iter = g.iter + 1; st->prev[s ^ 1][0] = gamma; st->prev[s ^ 1][1] = alpha; }
        }
        st->ctrl[cout] = c;
    }
    if (!g.active || conv) return;
    double g2 = 0.0, d2 = 0.0;
    /* Peer-memory mode: border rows first.  Their new w values are stored into
     * the neighbours' ghost buffers (w is the input of the next SpMV), and
     * issuing those NVLink stores at the start lets them drain under the
     * interior rows instead of in front of the closing system fence. */
    const bool push = P && P->fuse;
    const int first = push ? P->borderoff : 0;
    const int gtid = blockIdx.x * blockDim.x + threadIdx.x, gstride = gridDim.x * blockDim.x;
    for (int pass = 0; pass < 2; pass++) {
        const int lo = pass == 0 ? first : 0, hi = pass == 0 ? n : first;
        for (int i = lo + gtid; i < hi; i += gstride) {
            const double zv = fma(beta, z[i], q[i]);
            const double tv = fma(beta, t[i], w[i]);
            const double pv = fma(beta, p[i], r[i]);
            const double rv = fma(-alpha, tv, r[i]);
            const double wv = fma(-alpha, zv, w[i]);
            z[i] = zv; t[i] = tv; p[i] = pv;
            x[i] = fma(alpha, pv, x[i]);
            r[i] = rv;
            w[i] = wv;
            g2 = fma(rv, rv, g2);
            d2 = fma(wv, rv, d2);
            if (push && pass == 0) p2p_push_row(P, i, s ^ 1, wv);
        }
    }
    g2 = block_sum(g2, red);
    d2 = block_sum(d2, red);
    if (threadIdx.x == 0) {
        atomicAdd(&st->gd_loc[s ^ 1][0], g2);
        atomicAdd(&st->gd_loc[s ^ 1][1], d2);
    }
    if (P && P->fuse) {
        /* last CTA: this rank's {gamma,delta} of the next iteration to every
         * rank, and the halo sequence number to the neighbours */
        __threadfence_system();
        if (p2p_last_block(P, &last_flag)) {
            const unsigned long long it1 = (unsigned long long) g.iter + 1ull;
            p2p_publish_red(P, 0, s ^ 1, P->rbase + it1, &st->gd_loc[s ^ 1][0], 2);
            p2p_publish_halo(P, P->hbase + it1);
        }
    }
}

/* Fused pipelined CG, rows outside the slices: the update of the tile rows from the tile kernel's q, the
 * row ranges of the tile plan, one CTA per tile and trip.  Adds into the same ring slot as the fused kernel,
 * which runs after it and advances the control word; this one only forwards it. */
#define PCG_TAIL_THREADS 128
template <bool CATCH>
__global__ void __launch_bounds__(PCG_TAIL_THREADS)
pcg_tail_update_kernel(const acgb200_tile *__restrict__ tiles, int ntiles, acgb200_devstate *st,
                       const acgb200_ctrl *cin, acgb200_ctrl *cout, const double *__restrict__ q,
                       const double *__restrict__ w, double *__restrict__ w_next, double *__restrict__ z,
                       double *__restrict__ t, double *__restrict__ p, const double *__restrict__ r,
                       double *__restrict__ r_next, const double *__restrict__ r_ring, size_t r_stride, int m,
                       double *__restrict__ x)
{
    __shared__ double red[PCG_TAIL_THREADS / 32];
    __shared__ double ks_s[CATCH ? 2 * ACGB200_PCG_GROUP_MAX : 1];
    __shared__ PcgLag lag_s;
    pdl_prologue();
    const Gate g = gate_read(cin, st);
    if (blockIdx.x == 0 && threadIdx.x == 0) *cout = *cin;
    if (!g.active) return;
    const PcgStep k = pcg_step(st, g.iter);
    if (k.conv) return;
    /* CATCH: the group's {alpha_j, beta_j} and the ring, as in spmv_symdiag_kernel */
    if (CATCH && threadIdx.x < 2 * (m - 1))
        ks_s[threadIdx.x] = st->ab[(g.iter - (m - 1) + (int) (threadIdx.x >> 1)) % ACGB200_PCG_GROUP_MAX][threadIdx.x & 1];
    if (CATCH && threadIdx.x == 0) {
        ks_s[2 * m - 2] = k.alpha; ks_s[2 * m - 1] = k.beta;
        lag_s.ring = r_ring; lag_s.stride = r_stride; lag_s.m = m;
    }
    if (CATCH) __syncthreads();
    const uint64_t pol = l2_policy_evict_normal();
    double g2 = 0.0, d2 = 0.0;
    for (int b = blockIdx.x; b < ntiles; b += gridDim.x) {
        const acgb200_tile tl = tiles[b];
        for (int i = tl.row_begin + (int) threadIdx.x; i < tl.row_begin + tl.nrows; i += PCG_TAIL_THREADS) {
            if (CATCH) pcg_catchup(i, ks_s, &lag_s, r_next, r, p, x, pol);
            pcg_row(i, q[i], w[i], k.alpha, k.beta, z, t, r, r_next, w_next, pol, g2, d2);
        }
    }
    g2 = block_sum(g2, red);
    d2 = block_sum(d2, red);
    if (threadIdx.x == 0) {
        double *acc = st->gd_loc[(g.iter + 1) % 3];
        atomicAdd(&acc[0], g2);
        atomicAdd(&acc[1], d2);
    }
}

/* Fused pipelined CG, after the loop: the final control word counts the updates it.  If it is not a multiple
 * of the group m, updates g = m floor(it/m) ... it - 1 left their p and x updates to a catch-up iteration that
 * did not run, and r_it sits in ring slot it - g: form p_j = r_j + beta_j p and x += alpha_j p_j for those j
 * (pcg_row's FMAs; r_g is r itself, the others are in the ring), and move r_it into r. */
__global__ void __launch_bounds__(BLAS1_THREADS)
pcg_fused_finish_kernel(int n, const acgb200_devstate *st, int cfin, int m, double *__restrict__ r,
                        const double *__restrict__ ring, size_t stride, double *__restrict__ p, double *__restrict__ x)
{
    const int it = st->ctrl[cfin].iter, lag = it % m, g = it - lag;
    if (lag == 0) return;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        double pv = p[i], xv = x[i];
        for (int j = 0; j < lag; j++) {
            const double *ab = st->ab[(g + j) % ACGB200_PCG_GROUP_MAX];
            pv = fma(ab[1], pv, j ? ring[(size_t) (j - 1) * stride + i] : r[i]);
            xv = fma(ab[0], pv, xv);
        }
        p[i] = pv;
        x[i] = xv;
        r[i] = ring[(size_t) (lag - 1) * stride + i];
    }
}

__global__ void __launch_bounds__(BLAS1_THREADS)
dot_kernel(int n, const double *__restrict__ x, const double *__restrict__ y, double *acc)
{
    __shared__ double red[BLAS1_THREADS / 32];
    double v = 0.0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) v = fma(x[i], y[i], v);
    v = block_sum(v, red);
    if (threadIdx.x == 0) atomicAdd(acc, v);
}

__global__ void __launch_bounds__(BLAS1_THREADS)
dot2_kernel(int n, const double *__restrict__ r, const double *__restrict__ w, double *acc2)
{
    __shared__ double red[BLAS1_THREADS / 32];
    double g = 0.0, d = 0.0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const double rv = r[i];
        g = fma(rv, rv, g);
        d = fma(w[i], rv, d);
    }
    g = block_sum(g, red);
    d = block_sum(d, red);
    if (threadIdx.x == 0) { atomicAdd(&acc2[0], g); atomicAdd(&acc2[1], d); }
}

__global__ void gather_kernel(int n, double *__restrict__ dst, const double *__restrict__ src, const int *__restrict__ idx)
{
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) dst[i] = src[idx[i]];
}

__global__ void scatter_kernel(int n, const double *__restrict__ src, double *__restrict__ dst, const int *__restrict__ idx)
{
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) dst[idx[i]] = src[i];
}

/* ------------------------------------------------------------------------ */
/* several right-hand sides: block vectors of K interleaved columns          */
/* ------------------------------------------------------------------------ */

/* the K entries of one row of a block vector through the read-only path: vector loads of two
 * doubles (16-byte aligned, as row*K is even for K >= 2), issued back to back like ld_x */
template <int K>
__device__ __forceinline__ void ld_xk(double (&v)[K], const double *p)
{
    if constexpr (K == 1) {
        v[0] = ld_x(p);
    } else {
#pragma unroll
        for (int h = 0; h < K / 2; h++)
            asm volatile("ld.global.nc.v2.f64 {%0, %1}, [%2];" : "=d"(v[2 * h]), "=d"(v[2 * h + 1]) : "l"(p + 2 * h));
    }
}

/* one finished row of K columns: y = A x (mode 0, 1, with dot_j += x_j y_j in mode 1) or
 * y = b - A x with dot_j += y_j^2 (mode 2) */
template <int K>
__device__ __forceinline__ void spmm_row_epilogue(int row, const double (&sum)[K], int mode, const double *x, double *y,
                                                  const double *b, double (&dot)[K])
{
    const size_t o = (size_t) row * K;
    if (mode == SPMV_R_B_AX) {
#pragma unroll
        for (int j = 0; j < K; j++) {
            const double v = b[o + j] - sum[j];
            y[o + j] = v;
            dot[j] = fma(v, v, dot[j]);
        }
    } else {
#pragma unroll
        for (int j = 0; j < K; j++) y[o + j] = sum[j];
        if (mode == SPMV_Y_AX_DOT) {
#pragma unroll
            for (int j = 0; j < K; j++) dot[j] = fma(__ldg(x + o + j), sum[j], dot[j]);
        }
    }
}

/* per-column sums over the CTA, then one atomicAdd per non-zero column sum; `red` holds
 * blockDim/32 * K doubles */
template <int K>
__device__ __forceinline__ void block_sum_k_add(double (&v)[K], double *red, double *acc)
{
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = (blockDim.x + 31) >> 5;
#pragma unroll
    for (int j = 0; j < K; j++) v[j] = warp_sum(v[j]);
    if (l == 0) {
#pragma unroll
        for (int j = 0; j < K; j++) red[w * K + j] = v[j];
    }
    __syncthreads();
    if ((int) threadIdx.x < K) {
        double s = 0.0;
        for (int i = 0; i < nw; i++) s += red[i * K + threadIdx.x];
        if (s != 0.0) atomicAdd(acc + threadIdx.x, s);
    }
}

/* the first kernel of a gated multi-vector product forwards the control word and clears the (r,r)
 * accumulators the update behind it adds into (nothing reads them during the product) */
__device__ __forceinline__ void spmm_housekeeping(const acgb200_ctrl *cin, acgb200_ctrl *cout, const Gate &g,
                                                  acgb200_mstate *ms)
{
    if (blockIdx.x == 0 && threadIdx.x == 0 && cin && cout) {
        *cout = *cin;
        if (g.active && ms) {
#pragma unroll
            for (int j = 0; j < ACGB200_MAXK; j++) ms->rr[(g.iter & 1) ^ 1][j] = 0.0;
        }
    }
}

struct SpmmParams {
    const acgb200_slice *slices;
    int nslices;
    const double *sval;
    const unsigned short *patid;
    const int *spatoff;
    int npat, lpad;
    const int2 *ranges;
    int nranges;
    const int *rowptr;
    const int *colidx;
    const double *a;
    const double *x;
    double *y;
    const double *b;
    double *acc;
    int mode;
    const acgb200_ctrl *ctrl_in;
    acgb200_ctrl *ctrl_out;        /* NULL: another kernel of the product forwards the word */
    const acgb200_devstate *st;
    acgb200_mstate *ms;
};

/*
 * The slice kernel for K columns: one warp per slice, one row per lane, the same slice-major values,
 * evict-first streaming loads and offset table as spmv_slices_kernel.  Each value is loaded once and
 * fused into K accumulators; the x entries of a slot are one vector gather of K doubles.  UB slots are
 * in flight per batch (UB * K gathers).  Every column is summed in slot (CSR) order, as the
 * single-vector kernel sums its one column.  EXC: lanes of exception rows take their columns from the
 * CSR index array; slots past a row's end hold the value 0 and gather x[row].
 */
template <int UB, int T, bool EXC, int K>
__global__ void __launch_bounds__(T)
spmm_slices_kernel(const SpmmParams P)
{
    extern __shared__ __align__(16) int spat_s[];
    __shared__ double red[T / 32 * K];
    const int tid = threadIdx.x;
    pdl_prologue();
    const Gate gate = gate_read(P.ctrl_in, P.st);
    spmm_housekeeping(P.ctrl_in, P.ctrl_out, gate, P.ms);
    if (!gate.active) return;
    for (int i = tid; i < P.npat * P.lpad; i += T) spat_s[i] = P.spatoff[i];
    __syncthreads();

    const uint64_t pol = l2_policy_evict_first();
    const int lane = tid & 31;
    const int warp = (blockIdx.x * T + tid) >> 5;
    const int nwarps = (gridDim.x * T) >> 5;
    double dot[K];
#pragma unroll
    for (int j = 0; j < K; j++) dot[j] = 0.0;
    for (int s = warp; s < P.nslices; s += nwarps) {
        const int4 sl = __ldg(reinterpret_cast<const int4 *>(P.slices) + s);     /* row0, nrows, len, vblk */
        const int row = sl.x + lane;
        const int pid = P.patid[row];
        const bool exc = EXC && pid == (int) ACGB200_NOPATTERN;
        const int *offs = spat_s + (exc ? 0 : pid) * P.lpad;
        const double *v = P.sval + ((size_t) sl.w << 5) + lane;
        const int L = sl.z;
        int kb = 0, len = 0;
        if (EXC && exc) { kb = P.rowptr[row]; len = P.rowptr[row + 1] - kb; }
        double sum[K];
#pragma unroll
        for (int j = 0; j < K; j++) sum[j] = 0.0;
        int e = 0;
        /* full batches: straight-line code, all UB value loads and UB*K gathers issued before the first FMA */
        for (; e + UB <= L; e += UB) {
            double vv[UB], xv[UB][K];
#pragma unroll
            for (int u = 0; u < UB; u++) vv[u] = ld_stream(v + (size_t) (e + u) * 32, pol);
#pragma unroll
            for (int u = 0; u < UB; u++) {
                int col = row + offs[e + u];
                if (EXC && exc) col = e + u < len ? __ldg(P.colidx + kb + e + u) : row;
                ld_xk<K>(xv[u], P.x + (size_t) col * K);
            }
#pragma unroll
            for (int u = 0; u < UB; u++) {
#pragma unroll
                for (int j = 0; j < K; j++) sum[j] = fma(vv[u], xv[u][j], sum[j]);
            }
        }
        /* last, partial batch slot by slot */
        for (; e < L; e++) {
            double xv[K];
            int col = row + offs[e];
            if (EXC && exc) col = e < len ? __ldg(P.colidx + kb + e) : row;
            const double vv = ld_stream(v + (size_t) e * 32, pol);
            ld_xk<K>(xv, P.x + (size_t) col * K);
#pragma unroll
            for (int j = 0; j < K; j++) sum[j] = fma(vv, xv[j], sum[j]);
        }
        spmm_row_epilogue<K>(row, sum, P.mode, P.x, P.y, P.b, dot);
    }
    if (P.acc) block_sum_k_add<K>(dot, red, P.acc);
}

/*
 * Every row outside the pattern slices (tile, merge, medium and long rows of the single-vector plan),
 * plain CSR: a warp per chunk of rows (P.ranges), G lanes per row, each column index and value read
 * once per nonzero and fused into K accumulators.  With G > 1 a row's lanes are combined by a fixed
 * shuffle tree.  Long rows are correct here, not fast.
 */
template <int G, int K>
__global__ void __launch_bounds__(256)
spmm_rows_kernel(const SpmmParams P)
{
    __shared__ double red[256 / 32 * K];
    pdl_prologue();
    const Gate gate = gate_read(P.ctrl_in, P.st);
    spmm_housekeeping(P.ctrl_in, P.ctrl_out, gate, P.ms);
    if (!gate.active) return;
    const int lane = threadIdx.x & 31;
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int nwarps = (gridDim.x * blockDim.x) >> 5;
    double dot[K];
#pragma unroll
    for (int j = 0; j < K; j++) dot[j] = 0.0;
    for (int c = warp; c < P.nranges; c += nwarps) {
        const int2 rg = P.ranges[c];
        for (int base = rg.x; base < rg.y; base += 32 / G) {
            const int row = base + lane / G;
            double sum[K];
#pragma unroll
            for (int j = 0; j < K; j++) sum[j] = 0.0;
            if (row < rg.y) {
                const int ke = P.rowptr[row + 1];
#pragma unroll 1
                for (int k = P.rowptr[row] + lane % G; k < ke; k += G) {
                    double xv[K];
                    const double av = __ldg(P.a + k);
                    ld_xk<K>(xv, P.x + (size_t) __ldg(P.colidx + k) * K);
#pragma unroll
                    for (int j = 0; j < K; j++) sum[j] = fma(av, xv[j], sum[j]);
                }
            }
            if (G > 1) {
#pragma unroll
                for (int j = 0; j < K; j++) sum[j] = group_sum<G>(sum[j]);
            }
            if (row < rg.y && lane % G == 0) spmm_row_epilogue<K>(row, sum, P.mode, P.x, P.y, P.b, dot);
        }
    }
    if (P.acc) block_sum_k_add<K>(dot, red, P.acc);
}

/* A thread of the grid-stride BLAS-1 loops over a block vector reads pairs of entries (double2) and the
 * stride is a multiple of K, so its columns never change: c0 = 2g mod K and c0 + 1 (both 0 for K = 1).
 * Per-column sums: lanes 2l mod K hold the same pair, so an xor-shuffle over offsets >= K/2 leaves the
 * warp's sums of columns 2l, 2l+1 in lane l < K/2; then one atomicAdd per column and CTA (of the
 * columns in `mask`). */
template <int K>
__device__ __forceinline__ void colpair_sum_add(double a0, double a1, double *red, double *acc, unsigned mask)
{
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = (blockDim.x + 31) >> 5;
    if constexpr (K == 1) {
        const double v = block_sum(a0 + a1, red);
        if (threadIdx.x == 0 && (mask & 1u)) atomicAdd(acc, v);
    } else {
#pragma unroll
        for (int o = 16; o >= K / 2; o >>= 1) {
            a0 += __shfl_xor_sync(0xffffffffu, a0, o);
            a1 += __shfl_xor_sync(0xffffffffu, a1, o);
        }
        if (l < K / 2) { red[w * K + 2 * l] = a0; red[w * K + 2 * l + 1] = a1; }
        __syncthreads();
        if ((int) threadIdx.x < K && (mask >> threadIdx.x & 1u)) {
            double s = 0.0;
            for (int i = 0; i < nw; i++) s += red[i * K + threadIdx.x];
            atomicAdd(acc + threadIdx.x, s);
        }
    }
}

/* R_j -= alpha_j T_j with alpha_j = (r_j,r_j)/(p_j,Ap_j), and the new (r_j,r_j), for the active columns */
template <int K>
__global__ void __launch_bounds__(BLAS1_THREADS)
cg_multi_update_r_kernel(int n, acgb200_devstate *st, acgb200_mstate *ms, int cin, int cout,
                         const double *__restrict__ t, double *__restrict__ r)
{
    __shared__ double red[BLAS1_THREADS / 32 * (K > 1 ? K : 1)];
    pdl_prologue();
    const Gate g = gate_read(&st->ctrl[cin], st);
    if (cin != cout && blockIdx.x == 0 && threadIdx.x == 0) st->ctrl[cout] = st->ctrl[cin];
    if (!g.active) return;
    const unsigned mask = (unsigned) st->ctrl[cin].pad0;
    const int s = g.iter & 1;
    const int gtid = blockIdx.x * blockDim.x + threadIdx.x, gstride = gridDim.x * blockDim.x;
    const int c0 = (2 * gtid) & (K - 1), c1 = K == 1 ? 0 : c0 + 1;
    const bool act0 = mask >> c0 & 1u, act1 = mask >> c1 & 1u;
    const double al0 = act0 ? ms->rr[s][c0] / ms->pap[s][c0] : 0.0;
    const double al1 = act1 ? ms->rr[s][c1] / ms->pap[s][c1] : 0.0;
    double acc0 = 0.0, acc1 = 0.0;
    const long long nk = (long long) n * K, n2 = nk >> 1;
    const double2 *t2 = reinterpret_cast<const double2 *>(t);
    double2 *r2 = reinterpret_cast<double2 *>(r);
    for (long long i = gtid; i < n2; i += gstride) {
        const double2 tv = t2[i];
        double2 rv = r2[i];
        if (act0) rv.x = fma(-al0, tv.x, rv.x);
        if (act1) rv.y = fma(-al1, tv.y, rv.y);
        r2[i] = rv;
        acc0 = fma(rv.x, rv.x, acc0);
        acc1 = fma(rv.y, rv.y, acc1);
    }
    if ((nk & 1) && blockIdx.x == 0 && threadIdx.x == 0 && act0) {     /* K = 1, n odd */
        const double rv = fma(-al0, t[nk - 1], r[nk - 1]);
        r[nk - 1] = rv;
        acc0 = fma(rv, rv, acc0);
    }
    colpair_sum_add<K>(acc0, acc1, red, &ms->rr[s ^ 1][0], mask);
}

/* X_j += alpha_j P_j ; P_j = R_j + beta_j P_j for the active columns.  Block 0 decides each column's
 * convergence for the next iteration: a column that meets its tolerance leaves the mask (its x is the
 * iterate just formed), its iteration count and final (r,r) are recorded; with no column left the
 * control word is marked done. */
template <int K>
__global__ void __launch_bounds__(BLAS1_THREADS)
cg_multi_update_xp_kernel(int n, acgb200_devstate *st, acgb200_mstate *ms, int cin, int cout,
                          const double *__restrict__ r, double *__restrict__ p, double *__restrict__ x)
{
    pdl_prologue();
    const Gate g = gate_read(&st->ctrl[cin], st);
    const int s = g.iter & 1;
    const unsigned mask = (unsigned) st->ctrl[cin].pad0;
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        acgb200_ctrl c = st->ctrl[cin];
        if (g.active) {
            unsigned next = mask;
            c.iter = g.iter + 1;
            for (int j = 0; j < K; j++) {
                if (!(mask >> j & 1u)) continue;
                const double rrn = ms->rr[s ^ 1][j];
                ms->nits[j] = g.iter + 1;
                ms->final_rr[j] = rrn;
                /* acg/cgcuda.c:1008-1012 per column: ||r_j|| < tol_j, strictly */
                if (ms->tol[j] > 0.0 && sqrt(rrn) < ms->tol[j]) { next &= ~(1u << j); ms->conv[j] = 1; }
            }
            for (int j = 0; j < ACGB200_MAXK; j++) ms->pap[s ^ 1][j] = 0.0;     /* accumulators of the next product */
            c.pad0 = (int) next;
            if (next == 0) c.done = 1;
        }
        st->ctrl[cout] = c;
    }
    if (!g.active) return;
    const int gtid = blockIdx.x * blockDim.x + threadIdx.x, gstride = gridDim.x * blockDim.x;
    const int c0 = (2 * gtid) & (K - 1), c1 = K == 1 ? 0 : c0 + 1;
    const bool act0 = mask >> c0 & 1u, act1 = mask >> c1 & 1u;
    const double al0 = act0 ? ms->rr[s][c0] / ms->pap[s][c0] : 0.0, be0 = act0 ? ms->rr[s ^ 1][c0] / ms->rr[s][c0] : 0.0;
    const double al1 = act1 ? ms->rr[s][c1] / ms->pap[s][c1] : 0.0, be1 = act1 ? ms->rr[s ^ 1][c1] / ms->rr[s][c1] : 0.0;
    const long long nk = (long long) n * K, n2 = nk >> 1;
    const double2 *r2 = reinterpret_cast<const double2 *>(r);
    double2 *p2 = reinterpret_cast<double2 *>(p);
    double2 *x2 = reinterpret_cast<double2 *>(x);
    for (long long i = gtid; i < n2; i += gstride) {
        const double2 rv = r2[i];
        double2 pv = p2[i];
        double2 xv = x2[i];
        if (act0) { xv.x = fma(al0, pv.x, xv.x); pv.x = fma(be0, pv.x, rv.x); }
        if (act1) { xv.y = fma(al1, pv.y, xv.y); pv.y = fma(be1, pv.y, rv.y); }
        x2[i] = xv;
        p2[i] = pv;
    }
    if ((nk & 1) && blockIdx.x == 0 && threadIdx.x == 0 && act0) {
        const double pv = p[nk - 1];
        x[nk - 1] = fma(al0, pv, x[nk - 1]);
        p[nk - 1] = fma(be0, pv, r[nk - 1]);
    }
}

/* acc[j] += sum_i x[i*K + j]^2 (set-up: ||b_j||^2) */
template <int K>
__global__ void __launch_bounds__(BLAS1_THREADS)
dot_multi_kernel(int n, const double *__restrict__ x, double *acc)
{
    __shared__ double red[BLAS1_THREADS / 32 * (K > 1 ? K : 1)];
    const int gtid = blockIdx.x * blockDim.x + threadIdx.x, gstride = gridDim.x * blockDim.x;
    const long long nk = (long long) n * K, n2 = nk >> 1;
    const double2 *x2 = reinterpret_cast<const double2 *>(x);
    double a0 = 0.0, a1 = 0.0;
    for (long long i = gtid; i < n2; i += gstride) {
        const double2 v = x2[i];
        a0 = fma(v.x, v.x, a0);
        a1 = fma(v.y, v.y, a1);
    }
    if ((nk & 1) && blockIdx.x == 0 && threadIdx.x == 0) a0 = fma(x[nk - 1], x[nk - 1], a0);
    colpair_sum_add<K>(a0, a1, red, acc, (1u << K) - 1u);
}

/* ---- shifted systems (multi-shift CG) ----------------------------------------------------------- */

struct ShiftScalars { double zn, as, bs; };

/* zeta_{k+1}, alpha^sigma_k = alpha_k zeta_{k+1}/zeta_k and beta^sigma_k = beta_k (zeta_{k+1}/zeta_k)^2 of one
 * shift, from the seed's alpha_k, beta_k, alpha_{k-1}, beta_{k-1} and the shift's zeta_k, zeta_{k-1}.  Explicit
 * fma, so that sigma = 0 gives zeta = 1, alpha^sigma = alpha and beta^sigma = beta exactly. */
__device__ __forceinline__ ShiftScalars shift_scalars(double al, double be, double alp, double bep, double z, double zp,
                                                      double sg)
{
    ShiftScalars o;
    const double den = fma(al * bep, zp - z, zp * alp * fma(sg, al, 1.0));
    o.zn = z * zp * alp / den;
    const double q = o.zn / z;
    o.as = al * q;
    o.bs = be * q * q;
    return o;
}

/* set-up of solve_shifted: r = p = b ; X_j = 0 ; P_j = b (all K columns) */
template <int K>
__global__ void __launch_bounds__(BLAS1_THREADS)
shift_setup_kernel(int n, const double *__restrict__ b, double *__restrict__ r, double *__restrict__ p,
                   double *__restrict__ x, double *__restrict__ pk)
{
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const double v = b[i];
        r[i] = v; p[i] = v;
#pragma unroll
        for (int j = 0; j < K; j++) { x[(long long) i * K + j] = 0.0; pk[(long long) i * K + j] = v; }
    }
}

/* One iteration's update behind cg_update_r_kernel (which left r = r_{k+1} and (r_{k+1},r_{k+1}) in rr_loc[s^1]):
 *   seed:            p = r + beta_k p
 *   active shift j:  X_j += alpha^sigma_k P_j ;  P_j = zeta_{k+1} r + beta^sigma_k P_j
 * A warp works on 32 row pairs at a time.  Lane l loads the seed's r and p of one pair, once, and updates p;
 * the X and P entries of the 32 pairs (32 K contiguous double2) are then read by consecutive lanes, each lane
 * taking the slots l, l + 32, ..., l + 32 (K - 1).  Since K divides 32, a lane always sees the same double2
 * slot e = l mod K of a pair, i.e. the same two columns (K = 1: one column, two rows), so it derives the
 * scalars of those two shifts only; the r value of the slot's row comes from the owning lane by shuffle.
 * Block 0 keeps the books: the next iteration's slot of the per-shift state, each active shift's test
 * |zeta_{k+1}| ||r_{k+1}|| < tol_j (a shift that meets it leaves the mask, its x the iterate just formed),
 * the next product's (p,Ap) accumulator, and the control word (done when no shift is left). */
template <int K>
__global__ void __launch_bounds__(BLAS1_THREADS)
cg_shift_update_kernel(int n, acgb200_devstate *st, acgb200_sstate *ss, int cin, int cout,
                       const double *__restrict__ r, double *__restrict__ p, double *__restrict__ x,
                       double *__restrict__ pk)
{
    pdl_prologue();
    const Gate g = gate_read(&st->ctrl[cin], st);
    const int s = g.iter & 1;
    const unsigned mask = (unsigned) st->ctrl[cin].pad0;
    const double rr = st->rr_loc[s], rrn = st->rr_loc[s ^ 1], pap = st->pap_loc[s];
    const double al = rr / pap, be = rrn / rr;
    const double alp = ss->ab_prev[s][0], bep = ss->ab_prev[s][1];
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        acgb200_ctrl c = st->ctrl[cin];
        if (g.active) {
            unsigned next = mask;
            c.iter = g.iter + 1;
            const double rn = sqrt(rrn);
            for (int j = 0; j < K; j++) {
                if (!(mask >> j & 1u)) continue;
                const double z = ss->zeta[s][j];
                const ShiftScalars o = shift_scalars(al, be, alp, bep, z, ss->zeta_prev[s][j], ss->sigma[j]);
                ss->zeta[s ^ 1][j] = o.zn;
                ss->zeta_prev[s ^ 1][j] = z;
                const double nrm = fabs(o.zn) * rn;
                ss->nits[j] = g.iter + 1;
                ss->final_rnrm2[j] = nrm;
                /* acg/cgcuda.c:1008-1012 per shift: ||r_j|| < tol_j, strictly */
                if (ss->tol[j] > 0.0 && nrm < ss->tol[j]) { next &= ~(1u << j); ss->conv[j] = 1; }
            }
            ss->ab_prev[s ^ 1][0] = al;
            ss->ab_prev[s ^ 1][1] = be;
            st->pap_loc[s ^ 1] = 0.0;       /* accumulator of the next product */
            c.pad0 = (int) next;
            if (next == 0) c.done = 1;
        }
        st->ctrl[cout] = c;
    }
    if (!g.active) return;
    const int lane = threadIdx.x & 31;
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
    const int e = lane & (K - 1);                           /* this lane's double2 slot of a row pair */
    const int c0 = (2 * e) & (K - 1), c1 = K == 1 ? 0 : c0 + 1;
    const bool hi = K > 1 && 2 * e >= K;                    /* the slot holds the pair's second row */
    const bool act0 = mask >> c0 & 1u, act1 = mask >> c1 & 1u;
    ShiftScalars o0 = { 0.0, 0.0, 0.0 }, o1 = o0;
    if (act0) o0 = shift_scalars(al, be, alp, bep, ss->zeta[s][c0], ss->zeta_prev[s][c0], ss->sigma[c0]);
    if (act1) o1 = shift_scalars(al, be, alp, bep, ss->zeta[s][c1], ss->zeta_prev[s][c1], ss->sigma[c1]);
    const int npairs = n >> 1;
    const double2 *r2 = reinterpret_cast<const double2 *>(r);
    double2 *p2 = reinterpret_cast<double2 *>(p);
    double2 *x2 = reinterpret_cast<double2 *>(x);
    double2 *q2 = reinterpret_cast<double2 *>(pk);
    for (int wb = warp * 32; wb < npairs; wb += nwarps * 32) {          /* uniform across the warp */
        const int i = wb + lane;
        double2 rv = make_double2(0.0, 0.0);
        if (i < npairs) {
            rv = r2[i];
            double2 pv = p2[i];
            pv.x = fma(be, pv.x, rv.x);
            pv.y = fma(be, pv.y, rv.y);
            p2[i] = pv;
        }
#pragma unroll
        for (int t = 0; t < K; t++) {
            const int m = lane + 32 * t;                    /* double2 slot among the warp's 32 K */
            const int pr = m / K;                           /* its row pair, relative to wb */
            const double rx = __shfl_sync(0xffffffffu, rv.x, pr);
            const double ry = __shfl_sync(0xffffffffu, rv.y, pr);
            if (!(act0 || act1) || wb + pr >= npairs) continue;
            const double ra = hi ? ry : rx, rb = K == 1 ? ry : ra;
            const long long o = (long long) wb * K + m;
            double2 xv = x2[o], qv = q2[o];
            if (act0) { xv.x = fma(o0.as, qv.x, xv.x); qv.x = fma(o0.bs, qv.x, o0.zn * ra); }
            if (act1) { xv.y = fma(o1.as, qv.y, xv.y); qv.y = fma(o1.bs, qv.y, o1.zn * rb); }
            x2[o] = xv;
            q2[o] = qv;
        }
    }
    if ((n & 1) && blockIdx.x == 0 && threadIdx.x == 0) {
        const double rv = r[n - 1];
        p[n - 1] = fma(be, p[n - 1], rv);
        for (int j = 0; j < K; j++) {
            if (!(mask >> j & 1u)) continue;
            const ShiftScalars oj = shift_scalars(al, be, alp, bep, ss->zeta[s][j], ss->zeta_prev[s][j], ss->sigma[j]);
            const long long o = (long long) (n - 1) * K + j;
            const double qv = pk[o];
            x[o] = fma(oj.as, qv, x[o]);
            pk[o] = fma(oj.bs, qv, oj.zn * rv);
        }
    }
}

/* ---- MINRES -------------------------------------------------------------------------------------- */

/* set-up of solve_minres: v_1 = r_0 / beta_1 in place (scale = 1 / beta_1), v_0 = w_{-1} = w_0 = 0 */
__global__ void __launch_bounds__(BLAS1_THREADS)
minres_setup_kernel(int n, double scale, double *__restrict__ v, double *__restrict__ vprev, double *__restrict__ w0,
                    double *__restrict__ w1)
{
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        v[i] = scale * v[i];
        vprev[i] = 0.0; w0[i] = 0.0; w1[i] = 0.0;
    }
}

/* u = t - alpha_k v_k - beta_k v_{k-1} in place in t (t = A v_k from the product, alpha_k its fused dot),
 * and beta_{k+1}^2 = (u,u) in the same pass */
__global__ void __launch_bounds__(BLAS1_THREADS)
minres_lanczos_kernel(int n, const acgb200_devstate *st, acgb200_nstate *ns, int cin, const double *__restrict__ v,
                      const double *__restrict__ vprev, double *__restrict__ t)
{
    __shared__ double red[BLAS1_THREADS / 32];
    pdl_prologue();
    const Gate g = gate_read(&st->ctrl[cin], st);
    if (!g.active) return;
    const int s = g.iter & 1;
    const double al = ns->alpha[s], be = ns->beta[s];
    double acc = 0.0;
    const int n2 = n >> 1;
    const double2 *v2 = reinterpret_cast<const double2 *>(v);
    const double2 *q2 = reinterpret_cast<const double2 *>(vprev);
    double2 *t2 = reinterpret_cast<double2 *>(t);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n2; i += gridDim.x * blockDim.x) {
        const double2 vv = v2[i], qv = q2[i];
        double2 tv = t2[i];
        tv.x = fma(-be, qv.x, fma(-al, vv.x, tv.x));
        tv.y = fma(-be, qv.y, fma(-al, vv.y, tv.y));
        t2[i] = tv;
        acc = fma(tv.x, tv.x, acc);
        acc = fma(tv.y, tv.y, acc);
    }
    if ((n & 1) && blockIdx.x == 0 && threadIdx.x == 0) {
        const double u = fma(-be, vprev[n - 1], fma(-al, v[n - 1], t[n - 1]));
        t[n - 1] = u;
        acc = fma(u, u, acc);
    }
    acc = block_sum(acc, red);
    if (threadIdx.x == 0) atomicAdd(&ns->uu[s], acc);
}

/* The scalars of MINRES iteration k from slot s: the previous rotation applied to the new column of the
 * Lanczos matrix, and the next rotation (scipy's minres, unpreconditioned).  gamma = 0 (only for singular
 * A) leaves the rotation at zero: the update kernel stops before dividing by it. */
struct MinresStep { double beta, delta, eps, gamma, cs, sn, phi, phibar, dbar, epsn; };

__device__ __forceinline__ MinresStep minres_step(const acgb200_nstate *ns, int s)
{
    MinresStep o;
    const double al = ns->alpha[s], cs = ns->cs[s], sn = ns->sn[s], dbar = ns->dbar[s], phibar = ns->phibar[s];
    o.beta = sqrt(ns->uu[s]);
    o.eps = ns->eps[s];
    o.delta = cs * dbar + sn * al;
    const double gbar = sn * dbar - cs * al;
    o.epsn = sn * o.beta;
    o.dbar = -cs * o.beta;
    o.gamma = hypot(gbar, o.beta);
    o.cs = o.gamma > 0.0 ? gbar / o.gamma : 0.0;
    o.sn = o.gamma > 0.0 ? o.beta / o.gamma : 0.0;
    o.phi = o.cs * phibar;
    o.phibar = o.sn * phibar;
    return o;
}

/* w_k = (v_k - eps_k w_{k-2} - delta_k w_{k-1}) / gamma_k into w (which held w_{k-2}), x += phi_k w_k,
 * v_{k+1} = u / beta_{k+1} into vnext (which held v_{k-1}).  Every thread derives the scalars from slot s;
 * block 0 writes slot s^1, applies the test phi-bar_{k+1} < tol, ends the loop on beta_{k+1} = 0 (exact
 * breakdown: x is then the minimal-residual solution) or gamma_k = 0 (before the update, which is not
 * counted), zeroes the next product's and Lanczos kernel's accumulators and advances the control word. */
__global__ void __launch_bounds__(BLAS1_THREADS)
minres_update_kernel(int n, acgb200_devstate *st, acgb200_nstate *ns, int cin, int cout, const double *__restrict__ v,
                     const double *__restrict__ u, double *__restrict__ w, const double *__restrict__ wprev,
                     double *__restrict__ x, double *__restrict__ vnext)
{
    pdl_prologue();
    const Gate g = gate_read(&st->ctrl[cin], st);
    const int s = g.iter & 1;
    const MinresStep k = minres_step(ns, s);
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        acgb200_ctrl c = st->ctrl[cin];
        if (g.active) {
            if (k.gamma == 0.0) c.done = 1;
            else {
                c.iter = g.iter + 1;
                ns->beta[s ^ 1] = k.beta; ns->cs[s ^ 1] = k.cs; ns->sn[s ^ 1] = k.sn;
                ns->dbar[s ^ 1] = k.dbar; ns->eps[s ^ 1] = k.epsn; ns->phibar[s ^ 1] = k.phibar;
                /* acg/cgcuda.c:1008-1012: the strict test, here on the recursively updated norm */
                if (k.beta == 0.0 || (st->tol > 0.0 && k.phibar < st->tol)) c.done = 1;
            }
            ns->alpha[s ^ 1] = 0.0;        /* accumulators of the next product and Lanczos kernel */
            ns->uu[s ^ 1] = 0.0;
        }
        st->ctrl[cout] = c;
    }
    if (!g.active || k.gamma == 0.0) return;
    const double ig = 1.0 / k.gamma, ib = k.beta > 0.0 ? 1.0 / k.beta : 0.0;
    const int n2 = n >> 1;
    const double2 *v2 = reinterpret_cast<const double2 *>(v);
    const double2 *u2 = reinterpret_cast<const double2 *>(u);
    const double2 *p2 = reinterpret_cast<const double2 *>(wprev);
    double2 *w2 = reinterpret_cast<double2 *>(w);
    double2 *x2 = reinterpret_cast<double2 *>(x);
    double2 *n2v = reinterpret_cast<double2 *>(vnext);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n2; i += gridDim.x * blockDim.x) {
        const double2 vv = v2[i], uv = u2[i], pv = p2[i];
        double2 wv = w2[i], xv = x2[i];
        wv.x = fma(-k.delta, pv.x, fma(-k.eps, wv.x, vv.x)) * ig;
        wv.y = fma(-k.delta, pv.y, fma(-k.eps, wv.y, vv.y)) * ig;
        xv.x = fma(k.phi, wv.x, xv.x);
        xv.y = fma(k.phi, wv.y, xv.y);
        w2[i] = wv;
        x2[i] = xv;
        n2v[i] = make_double2(uv.x * ib, uv.y * ib);
    }
    if ((n & 1) && blockIdx.x == 0 && threadIdx.x == 0) {
        const double wv = fma(-k.delta, wprev[n - 1], fma(-k.eps, w[n - 1], v[n - 1])) * ig;
        w[n - 1] = wv;
        x[n - 1] = fma(k.phi, wv, x[n - 1]);
        vnext[n - 1] = u[n - 1] * ib;
    }
}

/* ---- mixed-precision CG with reliable updates ------------------------------------------------------- */

/* The fp32 product's rows outside the mirrored diagonals (all rows without them): plain CSR, a warp per
 * chunk of rows (the chunk list of spmm_rows_kernel), one thread per row summing (double) a_k * x[col_k]
 * in CSR order into one fp64 accumulator, stored rounded once.  Correct on power-law rows, not tuned. */
#define MIXED_ROWS_T 256
__global__ void __launch_bounds__(MIXED_ROWS_T)
spmv_rows_f32_kernel(int nranges, const int2 *__restrict__ ranges, const int *__restrict__ rowptr,
                     const int *__restrict__ colidx, const double *__restrict__ a, const float *__restrict__ x,
                     float *__restrict__ y, double *acc, const acgb200_ctrl *cin, const acgb200_devstate *st)
{
    __shared__ double red[MIXED_ROWS_T / 32];
    pdl_prologue();
    if (!gate_read(cin, st).active) return;
    const int lane = threadIdx.x & 31;
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int nwarps = (gridDim.x * blockDim.x) >> 5;
    double dot = 0.0;
    for (int c = warp; c < nranges; c += nwarps) {
        const int2 rg = ranges[c];
        for (int row = rg.x + lane; row < rg.y; row += 32) {
            double sum = 0.0;
            const int ke = rowptr[row + 1];
#pragma unroll 4
            for (int k = rowptr[row]; k < ke; k++) sum = fma(__ldg(a + k), (double) ld_x(x + __ldg(colidx + k)), sum);
            const float ys = (float) sum;
            y[row] = ys;
            dot = fma((double) __ldg(x + row), (double) ys, dot);
        }
    }
    if (acc) {
        const double v = block_sum(dot, red);
        if (threadIdx.x == 0 && v != 0.0) atomicAdd(acc, v);
    }
}

/* r = fl32(r64 * scale), p = r, y = 0 */
__global__ void __launch_bounds__(BLAS1_THREADS)
mixed_setup_kernel(int n, double scale, const double *__restrict__ r64, float *__restrict__ r, float *__restrict__ p,
                   float *__restrict__ y)
{
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const float v = (float) (r64[i] * scale);
        r[i] = v; p[i] = v; y[i] = 0.0f;
    }
}

/* The scalars of mixed iteration k from slot s; every thread of the update kernels derives them alike.
 * pi = 0 or non-finite is a breakdown: the iteration does nothing and is not counted. */
#define MIXED_DELTA 0.1
struct MixedStep { double alpha, rr, beta; bool bad, due; };

__device__ __forceinline__ MixedStep mixed_step(const acgb200_devstate *st, const acgb200_xstate *xs, int s)
{
    MixedStep o;
    const double pi = xs->pi[s], rho = xs->rho[s];
    o.bad = !(pi != 0.0 && isfinite(pi));
    o.alpha = o.bad ? 0.0 : rho / pi;
    o.rr = xs->rr[s];
    const double nr = sqrt(o.rr);
    o.due = nr < MIXED_DELTA * xs->mx[s] || xs->sigma[s] * nr < st->tol;
    o.beta = rho > 0.0 ? o.rr / rho : 0.0;
    return o;
}

/* r = fl32(r - alpha t), (r, r) into xs->rr[s]; the products of two floats are exact in fp64 */
__global__ void __launch_bounds__(BLAS1_THREADS)
mixed_update_r_kernel(int n, const acgb200_devstate *st, acgb200_xstate *xs, const float *__restrict__ t,
                      float *__restrict__ r)
{
    __shared__ double red[BLAS1_THREADS / 32];
    pdl_prologue();
    const Gate g = gate_read(&st->ctrl[0], st);
    if (!g.active) return;
    const int s = g.iter & 1;
    const double pi = xs->pi[s];
    if (!(pi != 0.0 && isfinite(pi))) return;
    const double alpha = xs->rho[s] / pi;
    double acc = 0.0;
    const int n2 = n >> 1;
    const float2 *t2 = reinterpret_cast<const float2 *>(t);
    float2 *r2 = reinterpret_cast<float2 *>(r);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n2; i += gridDim.x * blockDim.x) {
        const float2 tv = t2[i];
        float2 rv = r2[i];
        rv.x = (float) __dsub_rn(rv.x, __dmul_rn(alpha, tv.x));
        rv.y = (float) __dsub_rn(rv.y, __dmul_rn(alpha, tv.y));
        r2[i] = rv;
        acc = fma((double) rv.x, (double) rv.x, acc);
        acc = fma((double) rv.y, (double) rv.y, acc);
    }
    if ((n & 1) && blockIdx.x == 0 && threadIdx.x == 0) {
        const float rv = (float) __dsub_rn(r[n - 1], __dmul_rn(alpha, t[n - 1]));
        r[n - 1] = rv;
        acc = fma((double) rv, (double) rv, acc);
    }
    acc = block_sum(acc, red);
    if (threadIdx.x == 0) atomicAdd(&xs->rr[s], acc);
}

__device__ __forceinline__ void mixed_yp_row(const MixedStep &k, double sigma, float ri, float &pi, float &yi, double &xi)
{
    const float yn = (float) __dadd_rn(yi, __dmul_rn(k.alpha, pi));
    if (k.due) {
        xi = __dadd_rn(xi, sigma * (double) yn);          /* sigma is a power of two: the product is exact */
        yi = 0.0f;
    } else {
        yi = yn;
        pi = (float) __dadd_rn(ri, __dmul_rn(k.beta, pi));
    }
}

/* y = fl32(y + alpha p); not due: p = fl32(r + beta p); due: x += sigma y (fp64), y = 0 and p is left for
 * the replacement.  Block 0 writes ctrl[1] (iteration k+1, or done on a breakdown) and ctrl[2] (active,
 * iteration k, only when a reliable update is due), the next slot when none is due, and zeroes the next
 * accumulators (and rr64[s] for this iteration's fp64 residual). */
__global__ void __launch_bounds__(BLAS1_THREADS)
mixed_update_yp_kernel(int n, acgb200_devstate *st, acgb200_xstate *xs, const float *__restrict__ r,
                       float *__restrict__ p, float *__restrict__ y, double *__restrict__ x)
{
    pdl_prologue();
    const Gate g = gate_read(&st->ctrl[0], st);
    const int s = g.iter & 1;
    const MixedStep k = mixed_step(st, xs, s);
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        acgb200_ctrl c1 = st->ctrl[0], c2 = st->ctrl[0];
        c2.done = 1;
        if (g.active) {
            if (k.bad) { c1.done = 1; xs->breakdown = 1; }
            else {
                c1.iter = g.iter + 1;
                if (k.due) { c2.done = 0; xs->rr64[s] = 0.0; }
                else {
                    xs->rho[s ^ 1] = k.rr; xs->mx[s ^ 1] = fmax(xs->mx[s], sqrt(k.rr)); xs->sigma[s ^ 1] = xs->sigma[s];
                }
            }
            xs->pi[s ^ 1] = 0.0;
            xs->rr[s ^ 1] = 0.0;
        }
        st->ctrl[1] = c1;
        st->ctrl[2] = c2;
    }
    if (!g.active || k.bad) return;
    const double sigma = xs->sigma[s];
    const int n2 = n >> 1;
    const float2 *r2 = reinterpret_cast<const float2 *>(r);
    float2 *p2 = reinterpret_cast<float2 *>(p);
    float2 *y2 = reinterpret_cast<float2 *>(y);
    double2 *x2 = reinterpret_cast<double2 *>(x);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n2; i += gridDim.x * blockDim.x) {
        const float2 rv = k.due ? make_float2(0.0f, 0.0f) : r2[i];
        float2 pv = p2[i], yv = y2[i];
        double2 xv = k.due ? x2[i] : make_double2(0.0, 0.0);
        mixed_yp_row(k, sigma, rv.x, pv.x, yv.x, xv.x);
        mixed_yp_row(k, sigma, rv.y, pv.y, yv.y, xv.y);
        y2[i] = yv;
        if (k.due) x2[i] = xv;
        else p2[i] = pv;
    }
    if ((n & 1) && blockIdx.x == 0 && threadIdx.x == 0) {
        float pv = p[n - 1], yv = y[n - 1];
        double xv = x[n - 1];
        mixed_yp_row(k, sigma, r[n - 1], pv, yv, xv);
        y[n - 1] = yv;
        if (k.due) x[n - 1] = xv;
        else p[n - 1] = pv;
    }
}

/* sigma' = 2^round(log2 sqrt(rr64)) as its exponent */
__device__ __forceinline__ int mixed_scale_exp(double rr64)
{
    int e = 0;
    const double m = frexp(sqrt(rr64), &e);
    return m < 0.70710678118654752440 ? e - 1 : e;
}

/* The reliable update's second half (gated by ctrl[2]): r64 = b - A x has just been formed with
 * rr64 = (r64, r64).  sqrt(rr64) < tol, or rr64 = 0, ends the solve (the iteration counted); otherwise
 * sigma' = 2^round(log2 sqrt(rr64)), p = fl32(r64/sigma' + beta (sigma/sigma') p) with
 * beta = (rr64/sigma^2)/rho_k, r = fl32(r64/sigma'), and the next slot restarts M.  Block 0 writes ctrl[0]:
 * the word above, or ctrl[1] when no update was due. */
__global__ void __launch_bounds__(BLAS1_THREADS)
mixed_replace_kernel(int n, acgb200_devstate *st, acgb200_xstate *xs, const double *__restrict__ r64,
                     float *__restrict__ r, float *__restrict__ p)
{
    pdl_prologue();
    const Gate g = gate_read(&st->ctrl[2], st);
    const int s = g.iter & 1;
    const double rr64 = xs->rr64[s];
    const bool stop = sqrt(rr64) < st->tol || rr64 == 0.0;
    const int e = g.active && !stop ? mixed_scale_exp(rr64) : 0;
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        acgb200_ctrl c = st->ctrl[1];
        if (g.active) {
            xs->nupdates += 1;
            xs->last_rr64 = rr64;
            c.iter = g.iter + 1; c.done = 0;
            if (stop) { c.done = 1; xs->conv = 1; }
            else {
                const double rho = ldexp(rr64, -2 * e);
                xs->rho[s ^ 1] = rho; xs->mx[s ^ 1] = sqrt(rho); xs->sigma[s ^ 1] = ldexp(1.0, e);
            }
        }
        st->ctrl[0] = c;
    }
    if (!g.active || stop) return;
    const double sigma = xs->sigma[s];
    const double is = ldexp(1.0, -e);
    const double bf = (rr64 / (sigma * sigma)) / xs->rho[s] * (sigma * is);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const double rv = r64[i] * is;
        p[i] = (float) __dadd_rn(rv, __dmul_rn(bf, (double) p[i]));
        r[i] = (float) rv;
    }
}

/* x += sigma y */
__global__ void __launch_bounds__(BLAS1_THREADS)
mixed_fold_kernel(int n, double sigma, const float *__restrict__ y, double *__restrict__ x)
{
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        x[i] = __dadd_rn(x[i], sigma * (double) y[i]);
}

/* ---- Chebyshev-preconditioned CG (DESIGN section 15) ----------------------------------------------- */

/* dinv_i = 1 / a_ii, a_ii the sum of row i's diagonal entries in the full-storage block (0 if it has none);
 * entries that are <= 0 or non-finite are counted into cs->baddiag */
__global__ void __launch_bounds__(256)
cheb_dinv_kernel(int n, const int *__restrict__ rowptr, const int *__restrict__ colidx, const double *__restrict__ a,
                 double *__restrict__ dinv, acgb200_cstate *cs)
{
    int bad = 0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        double v = 0.0;
        for (int k = rowptr[i]; k < rowptr[i + 1]; k++) if (colidx[k] == i) v += a[k];
        if (!(v > 0.0 && isfinite(v))) bad++;
        dinv[i] = 1.0 / v;
    }
    if (bad) atomicAdd(&cs->baddiag, bad);
}

/* The r/x kernel of iteration k (reads ctrl[1], writes ctrl[2]): (p, A p) or (r_k, z_k) <= 0 or non-finite
 * ends the solve before the update; otherwise alpha = (r_k, z_k) / (p, A p), x += alpha p (unless x is NULL),
 * r -= alpha t with (r, r) into rr[s], and the preconditioner's start from the new r: with cheb, res = r,
 * d0 = c0 (D^-1 r) and z = d0; without, z = D^-1 r with (r, z) into rz[(k+1)%3].  start: the set-up's
 * preconditioner start from r as it is (the word's iteration is -1, so it adds into rz slot 0). */
__global__ void __launch_bounds__(BLAS1_THREADS)
cheb_rx_kernel(int n, acgb200_devstate *st, acgb200_cstate *cs, int start, int cheb, double c0,
               const double *__restrict__ dinv, const double *__restrict__ t, const double *__restrict__ p,
               double *__restrict__ x, double *__restrict__ r, double *__restrict__ z, double *__restrict__ res,
               double *__restrict__ d0)
{
    __shared__ double red[BLAS1_THREADS / 32];
    pdl_prologue();
    const Gate g = gate_read(&st->ctrl[1], st);
    const int s = g.iter & 1;
    const double rz = start ? 1.0 : cs->rz[g.iter % 3], pap = start ? 1.0 : cs->pap[s];
    const bool bad = !(rz > 0.0 && isfinite(rz)) || !(pap > 0.0 && isfinite(pap));
    const double alpha = rz / pap;
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        acgb200_ctrl c = st->ctrl[1];
        if (g.active && bad) { c.done = 1; cs->breakdown = 1; }
        else if (g.active && !start && cs->log && g.iter < ACGB200_CHEB_EST) cs->alpha_log[g.iter] = alpha;
        st->ctrl[2] = c;
    }
    if (!g.active || bad) return;
    double rr = 0.0, rzn = 0.0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        double ri = r[i];
        if (!start) {
            if (x) x[i] = fma(alpha, p[i], x[i]);
            ri = fma(-alpha, t[i], ri);
            r[i] = ri;
            rr = fma(ri, ri, rr);
        }
        const double zi = dinv[i] * ri;
        if (cheb) {
            const double dv = c0 * zi;
            res[i] = ri; d0[i] = dv; z[i] = dv;
        } else {
            z[i] = zi;
            rzn = fma(ri, zi, rzn);
        }
    }
    if (!start) {
        rr = block_sum(rr, red);
        if (threadIdx.x == 0) atomicAdd(&cs->rr[s], rr);
    }
    if (!cheb) {
        rzn = block_sum(rzn, red);
        if (threadIdx.x == 0) atomicAdd(&cs->rz[(g.iter + 1) % 3], rzn);
    }
}

/* one row of a Chebyshev step, q_i = (A dprev)_i: res -= q, dnext = c1 dprev + c2 D^-1 res, z += dnext; the
 * last step stores z only and adds r_i z_i into rz */
__device__ __forceinline__ void cheb_row(int i, double qi, double c1, double c2, bool last, const double *__restrict__ dinv,
                                         const double *__restrict__ dprev, double *__restrict__ dnext,
                                         double *__restrict__ res, double *__restrict__ z, const double *__restrict__ r,
                                         double &rz)
{
    const double rv = res[i] - qi;
    const double dn = fma(c1, dprev[i], c2 * (dinv[i] * rv));
    const double zv = z[i] + dn;
    z[i] = zv;
    if (last) rz = fma(r[i], zv, rz);
    else { res[i] = rv; dnext[i] = dn; }
}

/* a Chebyshev step after the plan's ordinary product q = A dprev (reads ctrl[2]) */
__global__ void __launch_bounds__(BLAS1_THREADS)
cheb_step_kernel(int n, const acgb200_devstate *st, acgb200_cstate *cs, double c1, double c2, int last,
                 const double *__restrict__ q, const double *__restrict__ dinv, const double *__restrict__ dprev,
                 double *__restrict__ dnext, double *__restrict__ res, double *__restrict__ z,
                 const double *__restrict__ r)
{
    __shared__ double red[BLAS1_THREADS / 32];
    pdl_prologue();
    const Gate g = gate_read(&st->ctrl[2], st);
    if (!g.active) return;
    double rz = 0.0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        cheb_row(i, q[i], c1, c2, last, dinv, dprev, dnext, res, z, r, rz);
    if (last) {
        rz = block_sum(rz, red);
        if (threadIdx.x == 0) atomicAdd(&cs->rz[(g.iter + 1) % 3], rz);
    }
}

/* the Chebyshev step's part of the fused kernel's parameters; P.x of SymdiagParams is dprev */
struct ChebStep {
    const acgb200_tile *tiles;
    int ntiles;
    int last;
    acgb200_cstate *cs;
    double c1, c2;
    const double *q, *dinv, *r;
    double *dnext, *res, *z;
};

/*
 * One Chebyshev step in one kernel: the mirrored-diagonal product of dprev (symdiag_row_sum, the row sums of
 * spmv_symdiag_kernel bit for bit) goes straight into the row's step (cheb_row) instead of to memory.  Rows
 * outside the slices -- the tiles -- take their product from q, written by the tile kernel just before; each
 * CTA then finishes whole tiles.  dnext is another buffer than dprev: other rows still gather dprev.  The
 * coefficients are arguments.  Reads ctrl[2] and writes no control word.  At most 40 registers: 12 CTAs of
 * 128 threads, as the fused pipelined-CG kernel.
 */
template <int UB, int T, typename V>
__global__ void __launch_bounds__(T, 1536 / T)
spmv_symdiag_cheb_kernel(const SymdiagParams P, const ChebStep C)
{
    constexpr bool CODED = std::is_same<V, uint8_t>::value;
    __shared__ int2 tab_s[ACGB200_SYMDIAG_MAX];
    __shared__ double vtab_s[CODED ? 256 : 1];
    __shared__ double red[T / 32];
    const int tid = threadIdx.x;
    pdl_prologue();
    if (!gate_read(P.ctrl_in, P.st).active) return;
    if (tid < P.no) tab_s[tid] = make_int2(P.tab[tid].voff, P.tab[tid].coff);
    if (CODED) for (int i = tid; i < P.ncodes; i += T) vtab_s[i] = __ldg(P.vtab + i);
    __syncthreads();
    const uint64_t pol = P.evict_first ? l2_policy_evict_first() : l2_policy_evict_normal();
    const int lane = tid & 31;
    const int warp = (blockIdx.x * T + tid) >> 5;
    const int nwarps = (gridDim.x * T) >> 5;
    const int cmax = P.nrows - 1;
    double rz = 0.0;
    for (int s = warp; s < P.nslices; s += nwarps) {
        const int row = __ldg(&P.slices[s].row0) + lane;
        const double sum = symdiag_row_sum<UB, V, double>(P, tab_s, vtab_s, row, pol, cmax, P.no);
        cheb_row(row, sum, C.c1, C.c2, C.last, C.dinv, P.x, C.dnext, C.res, C.z, C.r, rz);
    }
    for (int b = blockIdx.x; b < C.ntiles; b += gridDim.x) {
        const acgb200_tile tl = C.tiles[b];
        for (int i = tl.row_begin + tid; i < tl.row_begin + tl.nrows; i += T)
            cheb_row(i, C.q[i], C.c1, C.c2, C.last, C.dinv, P.x, C.dnext, C.res, C.z, C.r, rz);
    }
    if (C.last) {
        rz = block_sum(rz, red);
        /* the iteration index read again rather than kept live through the loop (the word is not written
         * during this kernel) */
        if (tid == 0) atomicAdd(&C.cs->rz[(P.ctrl_in->iter + 1) % 3], rz);
    }
}

/* The p kernel of iteration k (reads ctrl[2], writes ctrl[0]): the iteration is counted; ||r_{k+1}|| < tol
 * (strict) ends the solve, otherwise beta = (r_{k+1}, z_{k+1}) / (r_k, z_k) and p = z + beta p.  Block 0 zeroes
 * the next iteration's accumulators pap[s^1], rr[s^1] and rz[(k+2)%3]. */
__global__ void __launch_bounds__(BLAS1_THREADS)
cheb_p_kernel(int n, acgb200_devstate *st, acgb200_cstate *cs, const double *__restrict__ z, double *__restrict__ p)
{
    pdl_prologue();
    const Gate g = gate_read(&st->ctrl[2], st);
    const int s = g.iter & 1;
    const double rr = cs->rr[s];
    const bool conv = st->tol > 0.0 && sqrt(rr) < st->tol;
    const double beta = cs->rz[(g.iter + 1) % 3] / cs->rz[g.iter % 3];
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        acgb200_ctrl c = st->ctrl[2];
        if (g.active) {
            c.iter = g.iter + 1;
            st->final_rr = rr;
            if (conv) c.done = 1;
            if (cs->log && g.iter < ACGB200_CHEB_EST) cs->beta_log[g.iter] = beta;
            cs->pap[s ^ 1] = 0.0;
            cs->rr[s ^ 1] = 0.0;
            cs->rz[(g.iter + 2) % 3] = 0.0;
        }
        st->ctrl[0] = c;
    }
    if (!g.active || conv) return;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) p[i] = fma(beta, p[i], z[i]);
}

/* ------------------------------------------------------------------------ */
/* host-side launchers (C linkage)                                           */
/* ------------------------------------------------------------------------ */

static int g_num_sms = 0;

extern "C" int acgb200_num_sms(void)
{
    if (g_num_sms == 0) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess) return 132;
        if (cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || g_num_sms <= 0)
            g_num_sms = 132;
    }
    return g_num_sms;
}

/* CTAs per SM for the BLAS-1 kernels: 0 = as many as are resident at once */
static int g_blas1_ctas_per_sm = 0;

extern "C" void acgb200_blas1_set_ctas_per_sm(int v) { g_blas1_ctas_per_sm = v < 0 ? 0 : v; }


/* One wave of grid-stride CTAs: SMs x resident CTAs of that kernel (a grid that
 * is not a multiple of it ends in a partial wave at a fraction of the memory
 * parallelism), fewer when the vector is short.  `slot` caches the occupancy. */
static int blas1_grid(int n, const void *fn, int *slot)
{
    if (*slot == 0) {
        int per_sm = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, BLAS1_THREADS, 0) != cudaSuccess || per_sm < 1)
            per_sm = 2;
        *slot = per_sm;
    }
    const int per = BLAS1_THREADS * 2;
    long long want = ((long long) n + per - 1) / per;
    const long long cap = (long long) acgb200_num_sms() * (g_blas1_ctas_per_sm > 0 ? g_blas1_ctas_per_sm : *slot);
    if (want > cap) want = cap;
    if (want < 1) want = 1;
    return (int) want;
}

/* kernel launch, with the programmatic-dependency attribute when PDL is on */
static int g_pdl = 0;

extern "C" void acgb200_set_pdl(int v) { g_pdl = v != 0; }

template <typename... Params, typename... Args>
static cudaError_t launch_chain(void (*kernel)(Params...), int grid, int block, size_t smem, cudaStream_t stream, Args... args)
{
    cudaLaunchConfig_t lc = {};
    lc.gridDim = dim3((unsigned) grid); lc.blockDim = dim3((unsigned) block);
    lc.dynamicSmemBytes = smem; lc.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    lc.attrs = attr; lc.numAttrs = g_pdl ? 1 : 0;
    return cudaLaunchKernelEx(&lc, kernel, args...);
}

typedef void (*spmv_fn)(const SpmvParams);

/* instantiated (lanes per row, threads per CTA) pairs; gathers in flight U=8 */
#define SPMV_VARIANTS(X) \
    X(1, 64) X(2, 64) X(4, 64) X(8, 128) X(16, 128) X(32, 128) X(1, 128) X(1, 256) X(2, 128) X(2, 256) X(2, 512) X(4, 128) X(4, 256) X(4, 512) \
    X(8, 256) X(8, 512) X(16, 256) X(16, 512) X(32, 256) X(32, 512)

static spmv_fn spmv_variant(int G, int T, int U)
{
    if (U == 4 && G == 1 && T == 128) return spmv_tiles_kernel<1, 128, 4>;
    if (U == 16 && G == 1 && T == 128) return spmv_tiles_kernel<1, 128, 16>;
    if (U == 16 && G == 1 && T == 256) return spmv_tiles_kernel<1, 256, 16>;
    if (U == 4 && G == 2 && T == 256) return spmv_tiles_kernel<2, 256, 4>;
    if (U == 16 && G == 2 && T == 256) return spmv_tiles_kernel<2, 256, 16>;
    if (U == 4 && G == 4 && T == 512) return spmv_tiles_kernel<4, 512, 4>;
    if (U == 4 && G == 4 && T == 128) return spmv_tiles_kernel<4, 128, 4>;
    if (U == 4 && G == 4 && T == 256) return spmv_tiles_kernel<4, 256, 4>;
#define X(g, t) if (G == g && T == t) return spmv_tiles_kernel<g, t, 8>;
    SPMV_VARIANTS(X)
#undef X
    return NULL;
}

static inline int stage_slots(const acgb200_spmvplan *pl) { return (pl->nnz_cap + 8 + 3) & ~3; }
static inline int stage_rslots(const acgb200_spmvplan *pl) { return (pl->rows_cap + 1 + 8 + 3) & ~3; }
static inline int stage_bytes(const acgb200_spmvplan *pl)
{
    const int sc = stage_slots(pl);
    const int rc = stage_rslots(pl);
    return (sc * 12 + rc * 4 + 127) & ~127;
}

typedef void (*slice_fn)(const SliceParams);

/* (values + gathers in flight per lane, threads per CTA) of the slice kernel */
static slice_fn slice_variant(int UB, int T, int EXC)
{
#define X(u, t) if (UB == u && T == t) return EXC ? spmv_slices_kernel<u, t, true> : spmv_slices_kernel<u, t, false>;
    X(5, 128) X(7, 128) X(8, 128) X(9, 128) X(7, 256) X(8, 256) X(9, 256)
#undef X
    return NULL;
}

typedef void (*symdiag_fn)(const SymdiagParams);

/* the mirrored-diagonal kernel for exactly the (UB, T) pairs of slice_variant; pcg: with the fused
 * pipelined-CG epilogue, catchup: its form for the last iteration of a group; coded: reading one-byte codes
 * (the plan's symdiag_codes > 0) */
static symdiag_fn symdiag_variant(int UB, int T, bool pcg, bool catchup, bool coded)
{
#define V(u, t, c) (pcg ? (catchup ? spmv_symdiag_kernel<u, t, true, c, double, true> : spmv_symdiag_kernel<u, t, true, c>) \
                        : spmv_symdiag_kernel<u, t, false, c>)
#define X(u, t) if (UB == u && T == t) return coded ? V(u, t, uint8_t) : V(u, t, double);
    X(5, 128) X(7, 128) X(8, 128) X(9, 128) X(7, 256) X(8, 256) X(9, 256)
#undef X
#undef V
    return NULL;
}

static symdiag_fn symdiag_variant(const acgb200_spmvplan *pl, bool pcg, bool catchup = false)
{
    return symdiag_variant(pl->slice_ub, pl->slice_threads, pcg, catchup, pl->symdiag_codes > 0);
}

/* the float-vector product of the mixed-precision solve, for the same (UB, T) pairs */
static symdiag_fn symdiag_f32_variant(const acgb200_spmvplan *pl)
{
    const int UB = pl->slice_ub, T = pl->slice_threads;
    const bool coded = pl->symdiag_codes > 0;
#define X(u, t) if (UB == u && T == t) \
        return coded ? spmv_symdiag_kernel<u, t, false, uint8_t, float> : spmv_symdiag_kernel<u, t, false, double, float>;
    X(5, 128) X(7, 128) X(8, 128) X(9, 128) X(7, 256) X(8, 256) X(9, 256)
#undef X
    return NULL;
}

typedef void (*symdiag_cheb_fn)(const SymdiagParams, const ChebStep);

/* the fused Chebyshev step, for the same (UB, T) pairs */
static symdiag_cheb_fn symdiag_cheb_variant(const acgb200_spmvplan *pl)
{
    const int UB = pl->slice_ub, T = pl->slice_threads;
    const bool coded = pl->symdiag_codes > 0;
#define X(u, t) if (UB == u && T == t) \
        return coded ? spmv_symdiag_cheb_kernel<u, t, uint8_t> : spmv_symdiag_cheb_kernel<u, t, double>;
    X(5, 128) X(7, 128) X(8, 128) X(9, 128) X(7, 256) X(8, 256) X(9, 256)
#undef X
    return NULL;
}

/* the kernel's view of the plan's stored diagonals, fp64 or coded */
static void symdiag_params(const acgb200_spmvplan *pl, SymdiagParams &S)
{
    S.slices = pl->d_slices; S.nslices = pl->nslices; S.no = pl->symdiag_no; S.nrows = pl->nrows;
    S.evict_first = pl->symdiag_evict_first; S.hval = pl->d_hval;
    S.hcode = pl->symdiag_codes > 0 ? pl->d_hcode : NULL;
    S.vtab = pl->symdiag_codes > 0 ? pl->d_codes->vtab : NULL;
    S.ncodes = pl->symdiag_codes;
    memcpy(S.tab, pl->symdiag_tab, sizeof(S.tab));
}

typedef void (*merge_fn)(const MergeParams);

static merge_fn merge_variant(int T)
{
    if (T == 128) return spmv_merge_kernel<128, 8>;
    if (T == 256) return spmv_merge_kernel<256, 4>;
    return NULL;
}

static inline int merge_slots(const acgb200_spmvplan *pl) { return (pl->merge_items + 8 + 3) & ~3; }
static inline int merge_rslots(const acgb200_spmvplan *pl) { return (pl->merge_items + 1 + 8 + 3) & ~3; }
static inline int merge_stage_bytes(const acgb200_spmvplan *pl) { return (merge_slots(pl) * 12 + merge_rslots(pl) * 4 + 127) & ~127; }

/* acgb200_spmv_choose (tile-plan heuristic) and acgb200_spmv_min_bytes are host-only: plan.c */

extern "C" int acgb200_spmv_configure(acgb200_spmvplan *pl)
{
    const void *fn = (const void *) spmv_variant(pl->lanes_per_row, pl->threads, pl->unroll);
    if (!fn) return (int) cudaErrorInvalidConfiguration;
    pl->smem_bytes = stage_bytes(pl) * pl->nstages;
    cudaError_t err = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, pl->smem_bytes);
    if (err) return (int) err;
    int per_sm = 0;
    err = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, pl->threads, pl->smem_bytes);
    if (err) return (int) err;
    if (per_sm < 1) per_sm = 1;
    if (pl->max_ctas_per_sm > 0 && per_sm > pl->max_ctas_per_sm) per_sm = pl->max_ctas_per_sm;
    long long grid = (long long) acgb200_num_sms() * per_sm;
    if (grid > pl->ntiles) grid = pl->ntiles;
    if (grid < 1) grid = 1;
    pl->grid = (int) grid;
    if (pl->nmtiles > 0) {
        merge_fn mfn = merge_variant(pl->merge_threads);
        if (!mfn) return (int) cudaErrorInvalidConfiguration;
        pl->merge_smem = merge_stage_bytes(pl) * pl->merge_stages + merge_slots(pl) * (int) sizeof(double);
        err = cudaFuncSetAttribute((const void *) mfn, cudaFuncAttributeMaxDynamicSharedMemorySize, pl->merge_smem);
        if (err) return (int) err;
        int mper = 0;
        err = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&mper, (const void *) mfn, pl->merge_threads, pl->merge_smem);
        if (err) return (int) err;
        if (mper < 1) mper = 1;
        if (pl->merge_max_ctas > 0 && mper > pl->merge_max_ctas) mper = pl->merge_max_ctas;
        long long mgrid = (long long) acgb200_num_sms() * mper;
        if (mgrid > pl->nmtiles) mgrid = pl->nmtiles;
        pl->merge_grid = (int) (mgrid < 1 ? 1 : mgrid);
    }
    if (pl->nslices > 0) {
        /* the mirrored-diagonal kernel, when the plan has them, takes the slice kernel's place and grid rule */
        const void *sfn = pl->symdiag_nd > 0 ? (const void *) symdiag_variant(pl, false)
                                             : (const void *) slice_variant(pl->slice_ub, pl->slice_threads, pl->slice_exc > 0);
        if (!sfn) return (int) cudaErrorInvalidConfiguration;
        pl->slice_smem = pl->symdiag_nd > 0 ? 0 : ((pl->slice_npat * pl->slice_lpad + 3) & ~3) * (int) sizeof(int);
        err = cudaFuncSetAttribute(sfn, cudaFuncAttributeMaxDynamicSharedMemorySize, pl->slice_smem);
        if (err) return (int) err;
        int sper = 0;
        err = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&sper, sfn, pl->slice_threads, pl->slice_smem);
        if (err) return (int) err;
        if (sper < 1) sper = 1;
        if (pl->slice_max_ctas > 0 && sper > pl->slice_max_ctas) sper = pl->slice_max_ctas;
        if (pl->symdiag_nd > 0 && pl->slice_max_ctas <= 0) {
            /* The lower entries are read from L2 only if a value is still there when its mirror row reads it.
             * The grid-stride front -- one slice per resident warp -- spans far more rows than the largest
             * mirror distance, and its rows' bytes (8 |D| + 16 per row) are what passes through L2 between the
             * two reads: keep them within half of the L2.  C3 (14 diagonals): 12 of the 16 CTAs of 128
             * threads the registers allow, 1026-1029 it/s against 937-939 with 16 (H100 SXM, 400 W, DESIGN
             * section 3a); C2 (4 diagonals) stays at 16.  The fused pipelined-CG kernel moves 80 more bytes per
             * row, all evict-first; with it C3 ran at 1154 (8), 1217 (10), 1204 (12), 1204 (16) it/s, so the
             * rule stands (DESIGN section 4a). */
            int dev = 0, l2 = 0;
            if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetAttribute(&l2, cudaDevAttrL2CacheSize, dev) == cudaSuccess && l2 > 0) {
                /* one byte per diagonal in the coded layout: at C3 the cap (49) then no longer binds */
                const long long row_bytes = (pl->symdiag_codes > 0 ? 1LL : 8LL) * pl->symdiag_nd + 16;
                long long cap = (long long) l2 / 2 / ((long long) acgb200_num_sms() * pl->slice_threads * row_bytes);
                if (cap < 1) cap = 1;
                if (sper > cap) sper = (int) cap;
            }
        }
        long long sgrid = (long long) acgb200_num_sms() * sper;
        const long long need = ((long long) pl->nslices * 32 + pl->slice_threads - 1) / pl->slice_threads;
        if (sgrid > need) sgrid = need;
        pl->slice_grid = (int) (sgrid < 1 ? 1 : sgrid);
        pl->pcg_grid = 0;
        if (pl->symdiag_nd > 0) {
            /* the fused pipelined-CG kernel: the same grid, unless the registers of its plain or its catch-up
             * form allow fewer CTAs */
            int fper = 0, oper = 0;
            err = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&fper, (const void *) symdiag_variant(pl, true, false),
                                                                pl->slice_threads, 0);
            if (!err) err = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&oper, (const void *) symdiag_variant(pl, true, true),
                                                                          pl->slice_threads, 0);
            if (err) return (int) err;
            if (oper < fper) fper = oper;
            const long long fgrid = (long long) acgb200_num_sms() * (fper < 1 ? 1 : fper);
            pl->pcg_grid = (int) (fgrid < pl->slice_grid ? fgrid : pl->slice_grid);
        }
    }
    return 0;
}

extern "C" int acgb200_slices_fill(const acgb200_spmvplan *pl, const int *d_rowptr, const double *d_a, cudaStream_t stream)
{
    if (pl->nslices <= 0) return 0;
    long long grid = ((long long) pl->nslices * 32 + 255) / 256;
    const long long cap = (long long) acgb200_num_sms() * 8;
    if (grid > cap) grid = cap;
    slices_fill_kernel<<<(int) grid, 256, 0, stream>>>(pl->nslices, pl->d_slices, d_rowptr, d_a, pl->d_sval);
    cudaError_t err = cudaGetLastError();
    if (err || pl->symdiag_nd <= 0 || !pl->d_hval || !pl->symdiag_colidx || !pl->d_symdiag_bad) return (int) err;
    /* mirrored diagonals: zero (margins and absent entries), fill from every owned row, then check */
    err = cudaMemsetAsync(pl->d_hval, 0, (size_t) pl->symdiag_nd * (size_t) pl->symdiag_stride * sizeof(double), stream);
    if (!err) err = cudaMemsetAsync(pl->d_symdiag_bad, 0, sizeof(int), stream);
    if (err) return (int) err;
    SymdiagParams S;
    memset(&S, 0, sizeof(S));
    S.slices = pl->d_slices; S.nslices = pl->nslices; S.no = pl->symdiag_no; S.nrows = pl->nrows; S.hval = pl->d_hval;
    memcpy(S.tab, pl->symdiag_tab, sizeof(S.tab));
    SymdiagList D;
    memcpy(D.d, pl->symdiag_d, sizeof(D.d));
    long long fgrid = ((long long) pl->nrows + 255) / 256;
    if (fgrid > cap) fgrid = cap;
    symdiag_fill_kernel<<<(int) (fgrid < 1 ? 1 : fgrid), 256, 0, stream>>>(pl->nrows, d_rowptr, pl->symdiag_colidx, d_a, pl->d_hval,
                                                                          pl->symdiag_nd, D, pl->symdiag_stride, pl->symdiag_margin);
    symdiag_check_kernel<<<(int) grid, 256, 0, stream>>>(S, d_rowptr, pl->symdiag_colidx, d_a, pl->d_symdiag_bad);
    err = cudaGetLastError();
    if (err || !pl->d_hcode || !pl->d_codes) return (int) err;
    /* the coded layout: distinct patterns, their sorted table, the codes and their check (each kernel after
     * the sort finds ncodes == 0 on overflow and does nothing) */
    acgb200_codestate *cs = pl->d_codes;
    err = cudaMemsetAsync(cs, 0, sizeof(*cs), stream);
    if (!err) err = cudaMemsetAsync(cs->set, 0xFF, sizeof(cs->set), stream);
    if (err) return (int) err;
    const long long n = (long long) pl->symdiag_nd * pl->symdiag_stride;
    long long cgrid = (n + 255) / 256;
    if (cgrid > cap) cgrid = cap;
    const unsigned long long *h = (const unsigned long long *) pl->d_hval;
    codes_collect_kernel<<<(int) cgrid, 256, 0, stream>>>(h, n, cs);
    codes_sort_kernel<<<1, 1024, 0, stream>>>(cs);
    codes_encode_kernel<<<(int) cgrid, 256, 0, stream>>>(h, pl->d_hcode, n, cs);
    codes_check_kernel<<<(int) cgrid, 256, 0, stream>>>(h, pl->d_hcode, n, cs);
    return (int) cudaGetLastError();
}

/* the tile kernel over the plan's tiles */
static int launch_tiles(const acgb200_spmvargs *a, cudaStream_t stream)
{
    const acgb200_spmvplan *pl = a->plan;
    SpmvParams P;
    P.tiles = pl->d_tiles; P.ntiles = pl->ntiles;
    P.sc = stage_slots(pl); P.stage_bytes = stage_bytes(pl); P.nstages = pl->nstages;
    P.rowptr = a->rowptr; P.colidx = a->colidx; P.a = a->a; P.x = a->x; P.y = a->y; P.b = a->b;
    P.acc = a->acc; P.dotrows = a->dotrows; P.mode = a->mode;
    P.ctrl_in = a->ctrl_in; P.ctrl_out = a->ctrl_out; P.st = a->st; P.housekeeping = a->housekeeping;
    P.p2p = (acgb200_p2pdev *) a->p2p; P.od_rowoffset = a->od_rowoffset; P.od_nrows = a->od_nrows;
    P.orowptr = a->orowptr; P.ocolidx = a->ocolidx; P.oa = a->oa; P.pub_ch = a->p2p ? a->pub_ch : -1;
    const cudaError_t le = launch_chain(spmv_variant(pl->lanes_per_row, pl->threads, pl->unroll),
                                        pl->grid, pl->threads, (size_t) pl->smem_bytes, stream, P);
    if (le) return (int) le;
    return (int) cudaGetLastError();
}

extern "C" int acgb200_spmv_launch(const acgb200_spmvargs *a, cudaStream_t stream)
{
    const acgb200_spmvplan *pl = a->plan;
    /* with neither tiles nor a peer-memory duty for the tile kernel, the slice kernel forwards the
     * control word itself and the tile kernel is not launched */
    const bool slices_forward = (pl->nslices > 0 || pl->nmtiles > 0) && pl->ntiles == 0 && !a->p2p;
    if (pl->nmtiles > 0) {
        /* rows [0, merge_rows) of an irregular matrix: merge-path tiles, then the rows cut by tile boundaries */
        MergeParams M;
        M.tiles = pl->d_mtiles; M.ntiles = pl->nmtiles; M.sc = merge_slots(pl); M.rc = merge_rslots(pl);
        M.stage_bytes = merge_stage_bytes(pl); M.nstages = pl->merge_stages;
        M.rowptr = a->rowptr; M.colidx = a->colidx; M.a = a->a; M.part = pl->d_mpart;
        M.x = a->x; M.y = a->y; M.b = a->b; M.acc = a->acc; M.dotrows = a->dotrows; M.mode = a->mode;
        M.ctrl_in = a->ctrl_in; M.ctrl_out = slices_forward ? a->ctrl_out : NULL; M.st = a->st; M.housekeeping = a->housekeeping;
        const cudaError_t le = launch_chain(merge_variant(pl->merge_threads), pl->merge_grid, pl->merge_threads,
                                            (size_t) pl->merge_smem, stream, M);
        if (le) return (int) le;
        if (pl->nsplit > 0) {
            long long grid = ((long long) pl->nsplit * 32 + 255) / 256;
            const long long cap = (long long) acgb200_num_sms() * 8;
            if (grid > cap) grid = cap;
            /* reads the control word the merge kernel read (ctrl_in is only rewritten by the iteration's last kernel) */
            spmv_merge_fix_kernel<<<(int) grid, 256, 0, stream>>>(pl->nsplit, pl->d_msplit, pl->d_mpart, a->x, a->y, a->b, a->acc,
                                                                 a->dotrows, a->mode, a->ctrl_in, a->st);
            const cudaError_t fe = cudaGetLastError();
            if (fe) return (int) fe;
        }
    }
    if (pl->nslices > 0 && pl->symdiag_nd > 0) {
        SymdiagParams S;
        symdiag_params(pl, S);
        S.x = a->x; S.y = a->y; S.b = a->b; S.acc = a->acc; S.dotrows = a->dotrows; S.mode = a->mode;
        S.ctrl_in = a->ctrl_in; S.ctrl_out = slices_forward ? a->ctrl_out : NULL; S.st = a->st; S.housekeeping = a->housekeeping;
        const cudaError_t le = launch_chain(symdiag_variant(pl, false), pl->slice_grid, pl->slice_threads,
                                            (size_t) 0, stream, S);
        if (le) return (int) le;
    } else if (pl->nslices > 0) {
        /* first: the tile kernel's last CTA publishes the fused dot, which these rows add into */
        SliceParams S;
        S.slices = pl->d_slices; S.nslices = pl->nslices; S.sval = pl->d_sval;
        S.patid = pl->d_spatid; S.spatoff = pl->d_spatoff; S.npat = pl->slice_npat; S.lpad = pl->slice_lpad;
        S.rowptr = a->rowptr; S.colidx = a->colidx;
        S.x = a->x; S.y = a->y; S.b = a->b; S.acc = a->acc; S.dotrows = a->dotrows; S.mode = a->mode;
        S.ctrl_in = a->ctrl_in; S.ctrl_out = slices_forward ? a->ctrl_out : NULL; S.st = a->st; S.housekeeping = a->housekeeping;
        const cudaError_t le = launch_chain(slice_variant(pl->slice_ub, pl->slice_threads, pl->slice_exc > 0), pl->slice_grid, pl->slice_threads,
                                            (size_t) pl->slice_smem, stream, S);
        if (le) return (int) le;
    }
    if (pl->ntiles > 0 || (a->ctrl_in && !slices_forward)) {   /* with no tiles the kernel still forwards the control word */
        const int err = launch_tiles(a, stream);
        if (err) return err;
    }
    if (pl->nmed > 0) {
        long long grid = ((long long) pl->nmed + 7) / 8;
        const long long cap = (long long) acgb200_num_sms() * 8;
        if (grid > cap) grid = cap;
        spmv_medium_kernel<<<(int) grid, 256, 0, stream>>>(
            pl->nmed, pl->d_medrows, a->rowptr, a->colidx, a->a, a->x, a->y, a->b, a->acc,
            a->dotrows, a->mode, a->ctrl_in, a->st,
            a->p2p, a->od_rowoffset, a->od_nrows, a->orowptr, a->ocolidx, a->oa);
        cudaError_t err = cudaGetLastError();
        if (err) return (int) err;
    }
    if (pl->nlong > 0) {
        if (!pl->d_long_scratch) return (int) cudaErrorInvalidValue;
        spmv_long_partial_kernel<<<pl->nlong * pl->long_chunks, 256, 0, stream>>>(
            pl->nlong, pl->d_longrows, pl->long_chunks, a->rowptr, a->colidx, a->a, a->x, pl->d_long_scratch,
            a->ctrl_in, a->st);
        spmv_long_finish_kernel<<<(pl->nlong + 127) / 128, 128, 0, stream>>>(
            pl->nlong, pl->d_longrows, pl->long_chunks, pl->d_long_scratch, a->x, a->y, a->b, a->acc,
            a->dotrows, a->mode, a->ctrl_in, a->st,
            a->p2p, a->od_rowoffset, a->od_nrows, a->orowptr, a->ocolidx, a->oa);
        cudaError_t err = cudaGetLastError();
        if (err) return (int) err;
    }
    return 0;
}

extern "C" int acgb200_offdiag_launch(const acgb200_offdiagargs *a, cudaStream_t stream)
{
    if (a->nrows <= 0) return 0;
    int grid = (a->nrows + 255) / 256;
    const int cap = acgb200_num_sms() * 8;
    if (grid > cap) grid = cap;
    offdiag_kernel<<<grid, 256, 0, stream>>>(*a);
    return (int) cudaGetLastError();
}

extern "C" int acgb200_cg_update_r(int n, acgb200_devstate *st, int cin, int cout, int multi,
                                   acgb200_p2pdev *p2p,
                                   const double *t, double *r, cudaStream_t stream)
{
    static int occ = 0;
    return (int) launch_chain(cg_update_r_kernel, blas1_grid(n, (const void *) cg_update_r_kernel, &occ), BLAS1_THREADS, 0, stream,
                              n, st, cin, cout, multi, p2p, t, r);
}

extern "C" int acgb200_cg_update_xp(int n, acgb200_devstate *st, int cin, int cout, int multi,
                                    acgb200_p2pdev *p2p,
                                    const double *r, double *p, double *x, cudaStream_t stream)
{
    static int occ = 0;
    return (int) launch_chain(cg_update_xp_kernel, blas1_grid(n, (const void *) cg_update_xp_kernel, &occ), BLAS1_THREADS, 0, stream,
                              n, st, cin, cout, multi, p2p, r, p, x);
}

extern "C" int acgb200_pcg_update(int n, acgb200_devstate *st, int cin, int cout, int multi,
                                  acgb200_p2pdev *p2p,
                                  const double *q, double *z, double *w, double *t, double *p,
                                  double *r, double *x, cudaStream_t stream)
{
    static int occ = 0;
    return (int) launch_chain(pcg_update_kernel, blas1_grid(n, (const void *) pcg_update_kernel, &occ), BLAS1_THREADS, 0, stream,
                              n, st, cin, cout, multi, p2p, q, z, w, t, p, r, x);
}

extern "C" int acgb200_pcg_fused_launch(const acgb200_pcgargs *a, cudaStream_t stream)
{
    const acgb200_spmvplan *pl = a->plan;
    if (pl->symdiag_nd <= 0 || pl->pcg_grid <= 0 || pl->nmtiles > 0 || pl->nmed > 0 || pl->nlong > 0)
        return (int) cudaErrorInvalidConfiguration;
    acgb200_ctrl *ctrl = a->st->ctrl;
    const int cout = a->cin ^ 1;
    int fin = a->cin;                   /* the control word the fused kernel reads */
    if (pl->ntiles > 0) {
        /* rows outside the slices: q = A w over the tiles, then their update (control words cin -> 2 -> 3) */
        acgb200_spmvargs s;
        memset(&s, 0, sizeof(s));
        s.plan = pl; s.rowptr = a->rowptr; s.colidx = a->colidx; s.a = a->a; s.x = a->w; s.y = a->q;
        s.mode = SPMV_Y_AX; s.ctrl_in = &ctrl[a->cin]; s.ctrl_out = &ctrl[2]; s.st = a->st;
        int err = launch_tiles(&s, stream);
        if (err) return err;
        long long grid = pl->ntiles;
        const long long cap = (long long) acgb200_num_sms() * 8;
        if (grid > cap) grid = cap;
        const cudaError_t le = launch_chain(a->catchup ? pcg_tail_update_kernel<true> : pcg_tail_update_kernel<false>,
                                            (int) grid, PCG_TAIL_THREADS, 0, stream,
                                            (const acgb200_tile *) pl->d_tiles, pl->ntiles, a->st,
                                            (const acgb200_ctrl *) &ctrl[2], &ctrl[3], (const double *) a->q, a->w,
                                            a->w_next, a->z, a->t, a->p, (const double *) a->r, a->r_next,
                                            (const double *) a->r_ring, a->r_stride, a->group, a->x);
        if (le) return (int) le;
        fin = 3;
    }
    SymdiagParams S;
    memset(&S, 0, sizeof(S));
    symdiag_params(pl, S);
    S.x = a->w; S.mode = SPMV_Y_AX;
    S.ctrl_in = &ctrl[fin]; S.ctrl_out = &ctrl[cout]; S.st = a->st;
    S.z = a->z; S.t = a->t; S.p = a->p; S.r = a->r; S.r_next = a->r_next; S.xs = a->x; S.w_next = a->w_next;
    S.r_ring = a->r_ring; S.r_stride = a->r_stride; S.group = a->group;
    S.vec_evict_first = a->vec_evict_first;
    const cudaError_t le = launch_chain(symdiag_variant(pl, true, a->catchup != 0), pl->pcg_grid, pl->slice_threads,
                                        (size_t) 0, stream, S);
    if (le) return (int) le;
    return (int) cudaGetLastError();
}

extern "C" int acgb200_pcg_fused_finish(int n, const acgb200_devstate *st, int cfin, int group, double *r,
                                        const double *r_ring, size_t r_stride, double *p, double *x, cudaStream_t stream)
{
    static int occ = 0;
    pcg_fused_finish_kernel<<<blas1_grid(n, (const void *) pcg_fused_finish_kernel, &occ), BLAS1_THREADS, 0, stream>>>(
        n, st, cfin, group, r, r_ring, r_stride, p, x);
    return (int) cudaGetLastError();
}

extern "C" int acgb200_comm_post(const acgb200_postargs *a, cudaStream_t stream)
{
    /* a handful of CTAs moves a halo of 10^4-10^5 doubles in a few microseconds;
     * a reduction-only post needs one */
    const int grid = a->vec ? 8 : 1;
    comm_post_kernel<<<grid, 512, 0, stream>>>(*a);
    return (int) cudaGetLastError();
}

extern "C" int acgb200_dot(int n, const double *x, const double *y, double *acc, cudaStream_t stream)
{
    static int occ = 0;
    dot_kernel<<<blas1_grid(n, (const void *) dot_kernel, &occ), BLAS1_THREADS, 0, stream>>>(n, x, y, acc);
    return (int) cudaGetLastError();
}

extern "C" int acgb200_dot2(int n, const double *r, const double *w, double *acc2, cudaStream_t stream)
{
    static int occ = 0;
    dot2_kernel<<<blas1_grid(n, (const void *) dot2_kernel, &occ), BLAS1_THREADS, 0, stream>>>(n, r, w, acc2);
    return (int) cudaGetLastError();
}

/* ---- several right-hand sides -------------------------------------------------------------- */

typedef void (*spmm_fn)(const SpmmParams);

/* slots per batch of the multi-vector slice kernel: UB * K gathers in flight per lane (16 for K >= 2) */
#define SPMM_SLICE_UB(K) ((K) == 1 ? 8 : 16 / (K) < 2 ? 2 : 16 / (K))
#define SPMM_SLICE_T 128
#define SPMM_ROWS_T 256

static spmm_fn spmm_slice_variant(int K, int EXC)
{
#define XS(k) if (K == k) return EXC ? spmm_slices_kernel<SPMM_SLICE_UB(k), SPMM_SLICE_T, true, k> \
                                     : spmm_slices_kernel<SPMM_SLICE_UB(k), SPMM_SLICE_T, false, k>;
    XS(1) XS(2) XS(4) XS(8)
#undef XS
    return NULL;
}

static spmm_fn spmm_rows_variant(int G, int K)
{
#define XR(k) if (K == k) return G == 8 ? spmm_rows_kernel<8, k> : G == 1 ? spmm_rows_kernel<1, k> : NULL;
    XR(1) XR(2) XR(4) XR(8)
#undef XR
    return NULL;
}

/* resident CTAs per SM of a kernel (cached per function) */
static int spmm_per_sm(const void *fn, int threads, size_t smem)
{
    static const void *fns[64];
    static int val[64], nfn = 0;
    for (int i = 0; i < nfn; i++) if (fns[i] == fn) return val[i];
    int per = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, fn, threads, smem) != cudaSuccess || per < 1) per = 1;
    if (nfn < 64) { fns[nfn] = fn; val[nfn] = per; nfn++; }
    return per;
}

extern "C" int acgb200_spmm_launch(const acgb200_spmmargs *a, cudaStream_t stream)
{
    const acgb200_spmvplan *pl = a->plan;
    SpmmParams P;
    memset(&P, 0, sizeof(P));
    P.slices = pl->d_slices; P.nslices = pl->nslices; P.sval = pl->d_sval;
    P.patid = pl->d_spatid; P.spatoff = pl->d_spatoff; P.npat = pl->slice_npat; P.lpad = pl->slice_lpad;
    P.ranges = reinterpret_cast<const int2 *>(a->ranges); P.nranges = a->nranges;
    P.rowptr = a->rowptr; P.colidx = a->colidx; P.a = a->a;
    P.x = a->x; P.y = a->y; P.b = a->b; P.acc = a->acc; P.mode = a->mode;
    P.ctrl_in = a->ctrl_in; P.st = a->st; P.ms = a->ms;
    /* the first kernel forwards the control word; the second reads the same incoming word (only the
     * iteration's last kernel rewrites it) */
    bool forwarded = false;
    if (pl->nslices > 0) {
        const spmm_fn fn = spmm_slice_variant(a->k, pl->slice_exc > 0);
        if (!fn) return (int) cudaErrorInvalidConfiguration;
        const size_t smem = (size_t) ((pl->slice_npat * pl->slice_lpad + 3) & ~3) * sizeof(int);
        if (smem > 48 * 1024) {
            const cudaError_t e = cudaFuncSetAttribute((const void *) fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem);
            if (e) return (int) e;
        }
        long long grid = (long long) acgb200_num_sms() * spmm_per_sm((const void *) fn, SPMM_SLICE_T, smem);
        const long long need = ((long long) pl->nslices * 32 + SPMM_SLICE_T - 1) / SPMM_SLICE_T;
        if (grid > need) grid = need;
        P.ctrl_out = a->ctrl_out;
        forwarded = true;
        const cudaError_t le = launch_chain(fn, (int) (grid < 1 ? 1 : grid), SPMM_SLICE_T, smem, stream, P);
        if (le) return (int) le;
    }
    if (a->nranges > 0 || (a->ctrl_in && !forwarded)) {
        const spmm_fn fn = spmm_rows_variant(a->lanes, a->k);
        if (!fn) return (int) cudaErrorInvalidConfiguration;
        long long grid = (long long) acgb200_num_sms() * spmm_per_sm((const void *) fn, SPMM_ROWS_T, 0);
        const long long need = ((long long) a->nranges + SPMM_ROWS_T / 32 - 1) / (SPMM_ROWS_T / 32);
        if (grid > need) grid = need;
        P.ctrl_out = forwarded ? NULL : a->ctrl_out;
        P.ms = forwarded ? NULL : a->ms;
        const cudaError_t le = launch_chain(fn, (int) (grid < 1 ? 1 : grid), SPMM_ROWS_T, 0, stream, P);
        if (le) return (int) le;
    }
    return (int) cudaGetLastError();
}

/* the BLAS-1 grid of a block vector: as blas1_grid over its n*K entries */
#define MULTI_K_DISPATCH(k, call) \
    ((k) == 1 ? (call(1)) : (k) == 2 ? (call(2)) : (k) == 4 ? (call(4)) : (k) == 8 ? (call(8)) : cudaErrorInvalidValue)

extern "C" int acgb200_cg_multi_update_r(int n, int k, acgb200_devstate *st, acgb200_mstate *ms, int cin, int cout,
                                         const double *t, double *r, cudaStream_t stream)
{
    static int occ[9];
#define CALL(K) launch_chain(cg_multi_update_r_kernel<K>, blas1_grid(n * K, (const void *) cg_multi_update_r_kernel<K>, &occ[K]), \
                             BLAS1_THREADS, 0, stream, n, st, ms, cin, cout, t, r)
    return (int) MULTI_K_DISPATCH(k, CALL);
#undef CALL
}

extern "C" int acgb200_cg_multi_update_xp(int n, int k, acgb200_devstate *st, acgb200_mstate *ms, int cin, int cout,
                                          const double *r, double *p, double *x, cudaStream_t stream)
{
    static int occ[9];
#define CALL(K) launch_chain(cg_multi_update_xp_kernel<K>, blas1_grid(n * K, (const void *) cg_multi_update_xp_kernel<K>, &occ[K]), \
                             BLAS1_THREADS, 0, stream, n, st, ms, cin, cout, r, p, x)
    return (int) MULTI_K_DISPATCH(k, CALL);
#undef CALL
}

extern "C" int acgb200_dot_multi(int n, int k, const double *x, double *acc, cudaStream_t stream)
{
    static int occ[9];
#define CALL(K) (dot_multi_kernel<K><<<blas1_grid(n * K, (const void *) dot_multi_kernel<K>, &occ[K]), BLAS1_THREADS, 0, stream>>>(n, x, acc), \
                 cudaGetLastError())
    return (int) MULTI_K_DISPATCH(k, CALL);
#undef CALL
}

extern "C" int acgb200_shift_setup(int n, int k, const double *b, double *r, double *p, double *x, double *pk,
                                   cudaStream_t stream)
{
    static int occ[9];
#define CALL(K) (shift_setup_kernel<K><<<blas1_grid(n, (const void *) shift_setup_kernel<K>, &occ[K]), BLAS1_THREADS, 0, stream>>>( \
                     n, b, r, p, x, pk), cudaGetLastError())
    return (int) MULTI_K_DISPATCH(k, CALL);
#undef CALL
}

/* grid: as blas1_grid over the n rows (one row pair per thread, 32 pairs per warp) */
extern "C" int acgb200_cg_shift_update(int n, int k, acgb200_devstate *st, acgb200_sstate *ss, int cin, int cout,
                                       const double *r, double *p, double *x, double *pk, cudaStream_t stream)
{
    static int occ[9];
#define CALL(K) launch_chain(cg_shift_update_kernel<K>, blas1_grid(n, (const void *) cg_shift_update_kernel<K>, &occ[K]), \
                             BLAS1_THREADS, 0, stream, n, st, ss, cin, cout, r, p, x, pk)
    return (int) MULTI_K_DISPATCH(k, CALL);
#undef CALL
}

extern "C" int acgb200_minres_setup(int n, double scale, double *v, double *vprev, double *w0, double *w1,
                                    cudaStream_t stream)
{
    static int occ = 0;
    minres_setup_kernel<<<blas1_grid(n, (const void *) minres_setup_kernel, &occ), BLAS1_THREADS, 0, stream>>>(
        n, scale, v, vprev, w0, w1);
    return (int) cudaGetLastError();
}

extern "C" int acgb200_minres_lanczos(int n, const acgb200_devstate *st, acgb200_nstate *ns, int cin, const double *v,
                                      const double *vprev, double *t, cudaStream_t stream)
{
    static int occ = 0;
    return (int) launch_chain(minres_lanczos_kernel, blas1_grid(n, (const void *) minres_lanczos_kernel, &occ),
                              BLAS1_THREADS, 0, stream, n, st, ns, cin, v, vprev, t);
}

extern "C" int acgb200_minres_update(int n, acgb200_devstate *st, acgb200_nstate *ns, int cin, int cout, const double *v,
                                     const double *u, double *w, const double *wprev, double *x, double *vnext,
                                     cudaStream_t stream)
{
    static int occ = 0;
    return (int) launch_chain(minres_update_kernel, blas1_grid(n, (const void *) minres_update_kernel, &occ),
                              BLAS1_THREADS, 0, stream, n, st, ns, cin, cout, v, u, w, wprev, x, vnext);
}

extern "C" int acgb200_spmv_f32_launch(const acgb200_spmvf32args *a, cudaStream_t stream)
{
    const acgb200_spmvplan *pl = a->plan;
    if (pl->nslices > 0 && pl->symdiag_nd > 0) {
        const symdiag_fn fn = symdiag_f32_variant(pl);
        if (!fn) return (int) cudaErrorInvalidConfiguration;
        int per_sm = 0;
        const cudaError_t oe = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, (const void *) fn, pl->slice_threads, 0);
        if (oe) return (int) oe;
        SymdiagParams S;
        memset(&S, 0, sizeof(S));
        symdiag_params(pl, S);
        S.x = reinterpret_cast<const double *>(a->x); S.y = reinterpret_cast<double *>(a->y);
        S.acc = a->acc; S.dotrows = pl->nrows;
        S.mode = a->acc ? SPMV_Y_AX_DOT : SPMV_Y_AX;
        S.ctrl_in = a->ctrl_in; S.st = (acgb200_devstate *) a->st;
        /* the fp64 product's grid (its L2 cap included), unless the float instantiation fits fewer CTAs */
        const long long fgrid = (long long) acgb200_num_sms() * (per_sm < 1 ? 1 : per_sm);
        const int grid = (int) (fgrid < pl->slice_grid ? fgrid : pl->slice_grid);
        const cudaError_t le = launch_chain(fn, grid, pl->slice_threads, (size_t) 0, stream, S);
        if (le) return (int) le;
    }
    if (a->nranges > 0) {
        static int occ = 0;
        if (occ == 0 && (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, (const void *) spmv_rows_f32_kernel, MIXED_ROWS_T, 0) || occ < 1))
            occ = 1;
        long long grid = (long long) acgb200_num_sms() * occ;
        const long long need = ((long long) a->nranges + MIXED_ROWS_T / 32 - 1) / (MIXED_ROWS_T / 32);
        if (grid > need) grid = need;
        const cudaError_t le = launch_chain(spmv_rows_f32_kernel, (int) (grid < 1 ? 1 : grid), MIXED_ROWS_T, (size_t) 0,
                                            stream, a->nranges, reinterpret_cast<const int2 *>(a->ranges), a->rowptr,
                                            a->colidx, a->a, a->x, a->y, a->acc, a->ctrl_in, a->st);
        if (le) return (int) le;
    }
    return (int) cudaGetLastError();
}

extern "C" int acgb200_mixed_setup(int n, double scale, const double *r64, float *r, float *p, float *y, cudaStream_t stream)
{
    static int occ = 0;
    mixed_setup_kernel<<<blas1_grid(n, (const void *) mixed_setup_kernel, &occ), BLAS1_THREADS, 0, stream>>>(
        n, scale, r64, r, p, y);
    return (int) cudaGetLastError();
}

extern "C" int acgb200_mixed_update_r(int n, const acgb200_devstate *st, acgb200_xstate *xs, const float *t, float *r,
                                      cudaStream_t stream)
{
    static int occ = 0;
    return (int) launch_chain(mixed_update_r_kernel, blas1_grid(n, (const void *) mixed_update_r_kernel, &occ),
                              BLAS1_THREADS, 0, stream, n, st, xs, t, r);
}

extern "C" int acgb200_mixed_update_yp(int n, acgb200_devstate *st, acgb200_xstate *xs, const float *r, float *p,
                                       float *y, double *x, cudaStream_t stream)
{
    static int occ = 0;
    return (int) launch_chain(mixed_update_yp_kernel, blas1_grid(n, (const void *) mixed_update_yp_kernel, &occ),
                              BLAS1_THREADS, 0, stream, n, st, xs, r, p, y, x);
}

extern "C" int acgb200_mixed_replace(int n, acgb200_devstate *st, acgb200_xstate *xs, const double *r64, float *r,
                                     float *p, cudaStream_t stream)
{
    static int occ = 0;
    return (int) launch_chain(mixed_replace_kernel, blas1_grid(n, (const void *) mixed_replace_kernel, &occ),
                              BLAS1_THREADS, 0, stream, n, st, xs, r64, r, p);
}

extern "C" int acgb200_mixed_fold(int n, double sigma, const float *y, double *x, cudaStream_t stream)
{
    static int occ = 0;
    mixed_fold_kernel<<<blas1_grid(n, (const void *) mixed_fold_kernel, &occ), BLAS1_THREADS, 0, stream>>>(n, sigma, y, x);
    return (int) cudaGetLastError();
}

extern "C" int acgb200_cheb_dinv(int n, const int *rowptr, const int *colidx, const double *a, double *dinv,
                                 acgb200_cstate *cs, cudaStream_t stream)
{
    if (n <= 0) return 0;
    long long grid = ((long long) n + 255) / 256;
    const long long cap = (long long) acgb200_num_sms() * 8;
    if (grid > cap) grid = cap;
    cheb_dinv_kernel<<<(int) grid, 256, 0, stream>>>(n, rowptr, colidx, a, dinv, cs);
    return (int) cudaGetLastError();
}

extern "C" int acgb200_cheb_rx(int n, acgb200_devstate *st, acgb200_cstate *cs, int start, int cheb, double c0,
                               const double *dinv, const double *t, const double *p, double *x, double *r, double *z,
                               double *res, double *d0, cudaStream_t stream)
{
    static int occ = 0;
    return (int) launch_chain(cheb_rx_kernel, blas1_grid(n, (const void *) cheb_rx_kernel, &occ), BLAS1_THREADS, 0,
                              stream, n, st, cs, start, cheb, c0, dinv, t, p, x, r, z, res, d0);
}

extern "C" int acgb200_cheb_step(int n, const acgb200_devstate *st, acgb200_cstate *cs, double c1, double c2, int last,
                                 const double *q, const double *dinv, const double *dprev, double *dnext, double *res,
                                 double *z, const double *r, cudaStream_t stream)
{
    static int occ = 0;
    return (int) launch_chain(cheb_step_kernel, blas1_grid(n, (const void *) cheb_step_kernel, &occ), BLAS1_THREADS, 0,
                              stream, n, st, cs, c1, c2, last, q, dinv, dprev, dnext, res, z, r);
}

extern "C" int acgb200_cheb_fused_step(const acgb200_chebargs *a, cudaStream_t stream)
{
    const acgb200_spmvplan *pl = a->plan;
    const symdiag_cheb_fn fn = symdiag_cheb_variant(pl);
    if (!fn || pl->nslices <= 0 || pl->symdiag_nd <= 0 || pl->nmtiles > 0 || pl->nmed > 0 || pl->nlong > 0)
        return (int) cudaErrorInvalidConfiguration;
    acgb200_devstate *st = const_cast<acgb200_devstate *>(a->st);
    if (pl->ntiles > 0) {
        /* rows outside the slices: q = A dprev over the tiles (its copy of the word goes to ctrl[3], read by nobody) */
        acgb200_spmvargs s;
        memset(&s, 0, sizeof(s));
        s.plan = pl; s.rowptr = a->rowptr; s.colidx = a->colidx; s.a = a->a; s.x = a->dprev; s.y = a->q;
        s.mode = SPMV_Y_AX; s.ctrl_in = &st->ctrl[2]; s.ctrl_out = &st->ctrl[3]; s.st = st;
        const int err = launch_tiles(&s, stream);
        if (err) return err;
    }
    int per_sm = 0;
    const cudaError_t oe = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, (const void *) fn, pl->slice_threads, 0);
    if (oe) return (int) oe;
    SymdiagParams S;
    memset(&S, 0, sizeof(S));
    symdiag_params(pl, S);
    S.x = a->dprev; S.mode = SPMV_Y_AX; S.ctrl_in = &st->ctrl[2]; S.st = st;
    ChebStep C;
    C.tiles = pl->d_tiles; C.ntiles = pl->ntiles; C.last = a->last; C.cs = a->cs; C.c1 = a->c1; C.c2 = a->c2;
    C.q = a->q; C.dinv = a->dinv; C.r = a->r; C.dnext = a->dnext; C.res = a->res; C.z = a->z;
    /* the product's grid (its L2 cap included), unless the registers allow fewer CTAs */
    const long long fgrid = (long long) acgb200_num_sms() * (per_sm < 1 ? 1 : per_sm);
    const int grid = (int) (fgrid < pl->slice_grid ? fgrid : pl->slice_grid);
    const cudaError_t le = launch_chain(fn, grid, pl->slice_threads, (size_t) 0, stream, S, C);
    if (le) return (int) le;
    return (int) cudaGetLastError();
}

extern "C" int acgb200_cheb_p(int n, acgb200_devstate *st, acgb200_cstate *cs, const double *z, double *p,
                              cudaStream_t stream)
{
    static int occ = 0;
    return (int) launch_chain(cheb_p_kernel, blas1_grid(n, (const void *) cheb_p_kernel, &occ), BLAS1_THREADS, 0,
                              stream, n, st, cs, z, p);
}

extern "C" int acgb200_gather(int n, double *dst, const double *src, const int *idx, cudaStream_t stream)
{
    if (n <= 0) return 0;
    gather_kernel<<<(n + 255) / 256, 256, 0, stream>>>(n, dst, src, idx);
    return (int) cudaGetLastError();
}

extern "C" int acgb200_scatter(int n, const double *src, double *dst, const int *idx, cudaStream_t stream)
{
    if (n <= 0) return 0;
    scatter_kernel<<<(n + 255) / 256, 256, 0, stream>>>(n, src, dst, idx);
    return (int) cudaGetLastError();
}

/* *first = min(*first, the smallest k < n with a[k] != b[k]); a thread stops at its first difference, as every
 * later index of its stride is larger */
__global__ void first_diff_kernel(long long n, const int *__restrict__ a, const int *__restrict__ b,
                                  unsigned long long *__restrict__ first)
{
    const long long stride = (long long) gridDim.x * blockDim.x;
    for (long long k = (long long) blockIdx.x * blockDim.x + threadIdx.x; k < n; k += stride)
        if (a[k] != b[k]) { atomicMin(first, (unsigned long long) k); return; }
}

extern "C" int acgb200_first_diff(int64_t n, const int *a, const int *b, unsigned long long *first, cudaStream_t stream)
{
    if (n <= 0) return 0;
    long long grid = (n + 255) / 256;
    const long long cap = (long long) acgb200_num_sms() * 8;
    if (grid > cap) grid = cap;
    first_diff_kernel<<<(int) grid, 256, 0, stream>>>(n, a, b, first);
    return (int) cudaGetLastError();
}

/* ------------------------------------------------------------------------ */
/* BLAS-1 building blocks of acg/cg-kernels-cuda.h:45-97 (public, unused by   */
/* this library's own loops)                                                  */
/* ------------------------------------------------------------------------ */

enum { HELP_AXPY_QUOT = 0, HELP_AXMY_QUOT = 1, HELP_AYPX_QUOT = 2 };

/* y = (num/den) x + y | y = -(num/den) x + y | y = (num/den) y + x, the quotient read on the device */
template <int OP>
__global__ void __launch_bounds__(BLAS1_THREADS)
helper_axpy_kernel(int n, const double *num, const double *den, const double *__restrict__ x, double *__restrict__ y)
{
    const double a = OP == HELP_AXMY_QUOT ? -(*num) / (*den) : (*num) / (*den);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        y[i] = OP == HELP_AYPX_QUOT ? fma(a, y[i], x[i]) : fma(a, x[i], y[i]);
}

__global__ void helper_scalars_kernel(double *out0, double *out1, const double *num, const double *den, int op)
{
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    const double q = (*num) / (*den);
    if (op == 0) { *out0 = q; *out1 = -q; }        /* alpha, -alpha */
    else *out0 = q;                                /* beta */
}

/* the recurrences of acg/cg-kernels-cuda.cu:201-214; the scalars gamma_prev, alpha_prev are updated by
 * the single-thread kernel launched behind it (stream order replaces the reference's grid sync) */
__global__ void __launch_bounds__(BLAS1_THREADS)
helper_pipelined_kernel(int n, const double *gamma, const double *gamma_prev, const double *delta, const double *alpha_prev,
                        const double *__restrict__ q, double *__restrict__ p, double *__restrict__ r, double *__restrict__ t,
                        double *__restrict__ x, double *__restrict__ z, double *__restrict__ w)
{
    const double beta = (*gamma) / (*gamma_prev);
    const double alpha = (*gamma) / ((*delta) - beta * (*gamma) / (*alpha_prev));
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const double zv = fma(beta, z[i], q[i]);
        const double tv = fma(beta, t[i], w[i]);
        const double pv = fma(beta, p[i], r[i]);
        z[i] = zv; t[i] = tv; p[i] = pv;
        x[i] = fma(alpha, pv, x[i]);
        r[i] = fma(-alpha, tv, r[i]);
        w[i] = fma(-alpha, zv, w[i]);
    }
}

__global__ void helper_pipelined_scalars_kernel(const double *gamma, double *gamma_prev, const double *delta, double *alpha_prev)
{
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    const double beta = (*gamma) / (*gamma_prev);
    const double alpha = (*gamma) / ((*delta) - beta * (*gamma) / (*alpha_prev));
    *gamma_prev = *gamma;
    *alpha_prev = alpha;
}

extern "C" int acgb200_helper_axpy(int op, int n, const double *num, const double *den, const double *x, double *y, cudaStream_t stream)
{
    static int occ = 0;
    const int grid = blas1_grid(n, (const void *) helper_axpy_kernel<HELP_AXPY_QUOT>, &occ);
    if (op == HELP_AXPY_QUOT) helper_axpy_kernel<HELP_AXPY_QUOT><<<grid, BLAS1_THREADS, 0, stream>>>(n, num, den, x, y);
    else if (op == HELP_AXMY_QUOT) helper_axpy_kernel<HELP_AXMY_QUOT><<<grid, BLAS1_THREADS, 0, stream>>>(n, num, den, x, y);
    else helper_axpy_kernel<HELP_AYPX_QUOT><<<grid, BLAS1_THREADS, 0, stream>>>(n, num, den, x, y);
    return (int) cudaGetLastError();
}

extern "C" int acgb200_helper_scalars(int op, double *out0, double *out1, const double *num, const double *den, cudaStream_t stream)
{
    helper_scalars_kernel<<<1, 32, 0, stream>>>(out0, out1, num, den, op);
    return (int) cudaGetLastError();
}

extern "C" int acgb200_helper_pipelined(int n, const double *gamma, double *gamma_prev, const double *delta, const double *q,
                                        double *p, double *r, double *t, double *x, double *z, double *w, double *alpha_prev,
                                        cudaStream_t stream)
{
    static int occ = 0;
    const int grid = blas1_grid(n, (const void *) helper_pipelined_kernel, &occ);
    helper_pipelined_kernel<<<grid, BLAS1_THREADS, 0, stream>>>(n, gamma, gamma_prev, delta, alpha_prev, q, p, r, t, x, z, w);
    helper_pipelined_scalars_kernel<<<1, 32, 0, stream>>>(gamma, gamma_prev, delta, alpha_prev);
    return (int) cudaGetLastError();
}
