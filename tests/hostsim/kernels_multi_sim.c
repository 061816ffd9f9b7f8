/*
 * kernels_multi_sim.c -- TEST INFRASTRUCTURE ONLY.  Plain-C stand-ins for the multi-vector launch
 * interface of acg_b200/csrc/kernels.cu (internal.h: acgb200_spmm_launch, acgb200_cg_multi_update_r,
 * acgb200_cg_multi_update_xp, acgb200_dot_multi), with the kernels' index arithmetic, lane split and
 * per-column summation order.  Linked with the objects of the host-logic stand-in (Makefile) into
 * libacgb200_hostsim_multi.so by Makefile.multi, so that the CPU test-suite can drive the host code of
 * acgsolvercuda_solve_multi (padding, active masks, per-column convergence, graph signature, buffer
 * lifetime) and compare it with the oracle.  It says nothing about the CUDA kernels -- those are tested
 * on the H100 (tests/test_gpu_multi_rhs.py).
 */
#include "internal.h"
#include "hostsim.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

struct gate { int iter, active; };

/* as gate_read of kernels.cu (and of kernels_sim.c) */
static struct gate gate_read(const struct acgb200_ctrl *cin, const struct acgb200_devstate *st)
{
    struct gate g = { 0, 1 };
    if (cin) { g.iter = cin->iter; g.active = cin->done == 0 && cin->iter < st->maxits; }
    return g;
}

/* ---- several right-hand sides (block vectors of K interleaved columns) ---------------- */

static void spmm_row_epilogue(const struct acgb200_spmmargs *a, int row, const double *sum, double *dot)
{
    const int K = a->k;
    const size_t o = (size_t) row * (size_t) K;
    for (int j = 0; j < K; j++) {
        if (a->mode == SPMV_R_B_AX) {
            const double v = a->b[o + j] - sum[j];
            a->y[o + j] = v;
            dot[j] = fma(v, v, dot[j]);
        } else {
            a->y[o + j] = sum[j];
            if (a->mode == SPMV_Y_AX_DOT) dot[j] = fma(a->x[o + j], sum[j], dot[j]);
        }
    }
}

/* spmm_slices_kernel + spmm_rows_kernel: the slices through the slice-major values and the offset table, the
 * chunks through the CSR arrays with the kernel's lane split and shuffle tree; a row that no kernel or two
 * kernels compute reads NaN */
static void spmm_exec(void *vp)
{
    const struct acgb200_spmmargs *a = vp;
    const struct acgb200_spmvplan *pl = a->plan;
    const int K = a->k, n = pl->nrows;
    const struct gate g = gate_read(a->ctrl_in, a->st);
    if (a->ctrl_in && a->ctrl_out) {
        *a->ctrl_out = *a->ctrl_in;
        if (g.active && a->ms) for (int j = 0; j < ACGB200_MAXK; j++) a->ms->rr[(g.iter & 1) ^ 1][j] = 0.0;
    }
    if (!g.active) return;
    unsigned char *seen = calloc((size_t) n + 1, 1);
    double dot[ACGB200_MAXK] = { 0 }, sum[ACGB200_MAXK];
    for (int s = 0; s < pl->nslices; s++) {
        const struct acgb200_slice sl = pl->d_slices[s];
        for (int lane = 0; lane < 32; lane++) {
            const int row = sl.row0 + lane, id = pl->d_spatid[row];
            const int exc = id == (int) ACGB200_NOPATTERN;
            const int kb = a->rowptr[row], len = a->rowptr[row + 1] - kb;
            if ((!exc && id >= pl->slice_npat) || (exc && pl->slice_exc <= 0)) { seen[row] = 2; continue; }
            for (int j = 0; j < K; j++) sum[j] = 0.0;
            for (int e = 0; e < sl.len; e++) {
                const double v = pl->d_sval[((size_t) sl.vblk << 5) + (size_t) e * 32 + lane];
                const int col = exc ? (e < len ? a->colidx[kb + e] : row) : row + pl->d_spatoff[(size_t) id * pl->slice_lpad + e];
                for (int j = 0; j < K; j++) sum[j] = fma(v, a->x[(size_t) col * K + j], sum[j]);
            }
            spmm_row_epilogue(a, row, sum, dot);
            seen[row]++;
        }
    }
    const int G = a->lanes;
    for (int c = 0; c < a->nranges; c++) {
        for (int row = a->ranges[2 * c]; row < a->ranges[2 * c + 1]; row++) {
            double part[32][ACGB200_MAXK];
            for (int l = 0; l < G; l++) for (int j = 0; j < K; j++) part[l][j] = 0.0;
            for (int k = a->rowptr[row]; k < a->rowptr[row + 1]; k++) {
                const int l = (k - a->rowptr[row]) % G;
                for (int j = 0; j < K; j++) part[l][j] = fma(a->a[k], a->x[(size_t) a->colidx[k] * K + j], part[l][j]);
            }
            for (int o = G / 2; o > 0; o >>= 1) {               /* group_sum: xor tree over the row's lanes */
                double w[32][ACGB200_MAXK];
                for (int l = 0; l < G; l++) for (int j = 0; j < K; j++) w[l][j] = part[l][j] + part[l ^ o][j];
                memcpy(part, w, sizeof(w));
            }
            spmm_row_epilogue(a, row, part[0], dot);
            seen[row]++;
        }
    }
    for (int r = 0; r < n; r++)
        if (seen[r] != 1) for (int j = 0; j < K; j++) a->y[(size_t) r * K + j] = NAN;
    free(seen);
    if (a->acc) for (int j = 0; j < K; j++) a->acc[j] += dot[j];
}

int acgb200_spmm_launch(const struct acgb200_spmmargs *a, cudaStream_t stream)
{
    (void) stream;
    if (a->k != 1 && a->k != 2 && a->k != 4 && a->k != 8) return 1;
    if (a->nranges > 0 && a->lanes != 1 && a->lanes != 8) return 1;
    return hostsim_run_or_record(spmm_exec, a, sizeof(*a));
}

struct mupd_args {
    int n, k; struct acgb200_devstate *st; struct acgb200_mstate *ms; int cin, cout;
    const double *t; double *r; double *p; double *x;
};

static void multi_update_r_exec(void *vp)
{
    const struct mupd_args *a = vp;
    struct acgb200_devstate *st = a->st;
    struct acgb200_mstate *ms = a->ms;
    const struct gate g = gate_read(&st->ctrl[a->cin], st);
    if (a->cin != a->cout) st->ctrl[a->cout] = st->ctrl[a->cin];
    if (!g.active) return;
    const unsigned mask = (unsigned) st->ctrl[a->cin].pad0;
    const int s = g.iter & 1, K = a->k;
    double alpha[ACGB200_MAXK], acc[ACGB200_MAXK];
    for (int j = 0; j < K; j++) { alpha[j] = (mask >> j & 1u) ? ms->rr[s][j] / ms->pap[s][j] : 0.0; acc[j] = 0.0; }
    for (size_t i = 0; i < (size_t) a->n * K; i++) {
        const int j = (int) (i % (size_t) K);
        if (!(mask >> j & 1u)) continue;
        const double rv = fma(-alpha[j], a->t[i], a->r[i]);
        a->r[i] = rv;
        acc[j] = fma(rv, rv, acc[j]);
    }
    for (int j = 0; j < K; j++) if (mask >> j & 1u) ms->rr[s ^ 1][j] += acc[j];
}

static void multi_update_xp_exec(void *vp)
{
    const struct mupd_args *a = vp;
    struct acgb200_devstate *st = a->st;
    struct acgb200_mstate *ms = a->ms;
    const struct gate g = gate_read(&st->ctrl[a->cin], st);
    const int s = g.iter & 1, K = a->k;
    const unsigned mask = (unsigned) st->ctrl[a->cin].pad0;
    double alpha[ACGB200_MAXK], beta[ACGB200_MAXK];
    for (int j = 0; j < K; j++) {
        const int act = mask >> j & 1u;
        alpha[j] = act ? ms->rr[s][j] / ms->pap[s][j] : 0.0;
        beta[j] = act ? ms->rr[s ^ 1][j] / ms->rr[s][j] : 0.0;
    }
    struct acgb200_ctrl c = st->ctrl[a->cin];
    if (g.active) {
        unsigned next = mask;
        c.iter = g.iter + 1;
        for (int j = 0; j < K; j++) {
            if (!(mask >> j & 1u)) continue;
            const double rrn = ms->rr[s ^ 1][j];
            ms->nits[j] = g.iter + 1;
            ms->final_rr[j] = rrn;
            if (ms->tol[j] > 0.0 && sqrt(rrn) < ms->tol[j]) { next &= ~(1u << j); ms->conv[j] = 1; }
        }
        for (int j = 0; j < ACGB200_MAXK; j++) ms->pap[s ^ 1][j] = 0.0;
        c.pad0 = (int) next;
        if (next == 0) c.done = 1;
    }
    st->ctrl[a->cout] = c;
    if (!g.active) return;
    for (size_t i = 0; i < (size_t) a->n * K; i++) {
        const int j = (int) (i % (size_t) K);
        if (!(mask >> j & 1u)) continue;
        const double pv = a->p[i];
        a->x[i] = fma(alpha[j], pv, a->x[i]);
        a->p[i] = fma(beta[j], pv, a->r[i]);
    }
}

int acgb200_cg_multi_update_r(int n, int k, struct acgb200_devstate *st, struct acgb200_mstate *ms, int cin, int cout,
                              const double *t, double *r, cudaStream_t stream)
{
    (void) stream;
    struct mupd_args a;
    memset(&a, 0, sizeof(a));
    a.n = n; a.k = k; a.st = st; a.ms = ms; a.cin = cin; a.cout = cout; a.t = t; a.r = r;
    return hostsim_run_or_record(multi_update_r_exec, &a, sizeof(a));
}

int acgb200_cg_multi_update_xp(int n, int k, struct acgb200_devstate *st, struct acgb200_mstate *ms, int cin, int cout,
                               const double *r, double *p, double *x, cudaStream_t stream)
{
    (void) stream;
    struct mupd_args a;
    memset(&a, 0, sizeof(a));
    a.n = n; a.k = k; a.st = st; a.ms = ms; a.cin = cin; a.cout = cout; a.r = (double *) r; a.p = p; a.x = x;
    return hostsim_run_or_record(multi_update_xp_exec, &a, sizeof(a));
}

struct dotm_args { int n, k; const double *x; double *acc; };

static void dot_multi_exec(void *vp)
{
    const struct dotm_args *a = vp;
    double acc[ACGB200_MAXK] = { 0 };
    for (size_t i = 0; i < (size_t) a->n * a->k; i++) acc[i % (size_t) a->k] = fma(a->x[i], a->x[i], acc[i % (size_t) a->k]);
    for (int j = 0; j < a->k; j++) a->acc[j] += acc[j];
}

int acgb200_dot_multi(int n, int k, const double *x, double *acc, cudaStream_t stream)
{
    (void) stream;
    struct dotm_args a = { n, k, x, acc };
    return hostsim_run_or_record(dot_multi_exec, &a, sizeof(a));
}
