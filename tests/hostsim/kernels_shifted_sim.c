/*
 * kernels_shifted_sim.c -- TEST INFRASTRUCTURE ONLY.  Plain-C stand-ins for the shifted-systems launch
 * interface of acg_b200/csrc/kernels.cu (internal.h: acgb200_shift_setup, acgb200_cg_shift_update), with
 * the kernels' scalar recurrence (the same fma grouping), the warp's row-pair / double2-slot arithmetic and
 * the update order.  Linked with the host-logic stand-in and kernels_multi_sim.c into
 * libacgb200_hostsim_shifted.so by Makefile.shifted, so that the CPU test-suite can drive the host code of
 * acgsolvercuda_solve_shifted (padding, active masks, per-shift convergence, graph slot and signature,
 * warm-up) and compare it with the oracle.  It says nothing about the CUDA kernels -- those are tested on
 * the H100 (tests/test_gpu_shifted.py).
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

struct shift_scalars { double zn, as, bs; };

/* shift_scalars of kernels.cu */
static struct shift_scalars shift_scalars(double al, double be, double alp, double bep, double z, double zp, double sg)
{
    struct shift_scalars o;
    const double den = fma(al * bep, zp - z, zp * alp * fma(sg, al, 1.0));
    o.zn = z * zp * alp / den;
    const double q = o.zn / z;
    o.as = al * q;
    o.bs = be * q * q;
    return o;
}

struct setup_args { int n, k; const double *b; double *r, *p, *x, *pk; };

static void setup_exec(void *vp)
{
    const struct setup_args *a = vp;
    for (int i = 0; i < a->n; i++) {
        const double v = a->b[i];
        a->r[i] = v; a->p[i] = v;
        for (int j = 0; j < a->k; j++) { a->x[(size_t) i * a->k + j] = 0.0; a->pk[(size_t) i * a->k + j] = v; }
    }
}

int acgb200_shift_setup(int n, int k, const double *b, double *r, double *p, double *x, double *pk, cudaStream_t stream)
{
    (void) stream;
    if (k != 1 && k != 2 && k != 4 && k != 8) return 1;
    struct setup_args a = { n, k, b, r, p, x, pk };
    return hostsim_run_or_record(setup_exec, &a, sizeof(a));
}

struct supd_args {
    int n, k; struct acgb200_devstate *st; struct acgb200_sstate *ss; int cin, cout;
    const double *r; double *p, *x, *pk;
};

static void shift_update_exec(void *vp)
{
    const struct supd_args *a = vp;
    struct acgb200_devstate *st = a->st;
    struct acgb200_sstate *ss = a->ss;
    const int K = a->k, n = a->n;
    const struct gate g = gate_read(&st->ctrl[a->cin], st);
    const int s = g.iter & 1;
    const unsigned mask = (unsigned) st->ctrl[a->cin].pad0;
    const double rr = st->rr_loc[s], rrn = st->rr_loc[s ^ 1], pap = st->pap_loc[s];
    const double al = rr / pap, be = rrn / rr;
    const double alp = ss->ab_prev[s][0], bep = ss->ab_prev[s][1];
    /* every thread's scalars, from slot s (before block 0 writes slot s^1) */
    struct shift_scalars o[ACGB200_MAXK];
    for (int j = 0; j < K; j++)
        if (mask >> j & 1u) o[j] = shift_scalars(al, be, alp, bep, ss->zeta[s][j], ss->zeta_prev[s][j], ss->sigma[j]);
    struct acgb200_ctrl c = st->ctrl[a->cin];
    if (g.active) {
        unsigned next = mask;
        c.iter = g.iter + 1;
        const double rn = sqrt(rrn);
        for (int j = 0; j < K; j++) {
            if (!(mask >> j & 1u)) continue;
            ss->zeta_prev[s ^ 1][j] = ss->zeta[s][j];
            ss->zeta[s ^ 1][j] = o[j].zn;
            const double nrm = fabs(o[j].zn) * rn;
            ss->nits[j] = g.iter + 1;
            ss->final_rnrm2[j] = nrm;
            if (ss->tol[j] > 0.0 && nrm < ss->tol[j]) { next &= ~(1u << j); ss->conv[j] = 1; }
        }
        ss->ab_prev[s ^ 1][0] = al;
        ss->ab_prev[s ^ 1][1] = be;
        st->pap_loc[s ^ 1] = 0.0;
        c.pad0 = (int) next;
        if (next == 0) c.done = 1;
    }
    st->ctrl[a->cout] = c;
    if (!g.active) return;
    /* warps of 32 row pairs; the pair's 2K entries of X and P are K double2 slots, slot e holding
     * columns (2e) mod K and (2e + 1) mod K of row 2 pr + (2e >= K) (K = 1: rows 2 pr and 2 pr + 1) */
    const int npairs = n >> 1;
    for (int wb = 0; wb < npairs; wb += 32) {
        for (int l = 0; l < 32 && wb + l < npairs; l++) {
            const int i = wb + l;
            a->p[2 * i] = fma(be, a->p[2 * i], a->r[2 * i]);
            a->p[2 * i + 1] = fma(be, a->p[2 * i + 1], a->r[2 * i + 1]);
        }
        for (int l = 0; l < 32; l++) {
            const int e = l & (K - 1);
            const int c0 = (2 * e) & (K - 1), c1 = K == 1 ? 0 : c0 + 1;
            const int hi = K > 1 && 2 * e >= K;
            const int act0 = mask >> c0 & 1u, act1 = mask >> c1 & 1u;
            for (int t = 0; t < K; t++) {
                const int m = l + 32 * t, pr = m / K;
                if (!(act0 || act1) || wb + pr >= npairs) continue;
                const double rx = a->r[2 * (wb + pr)], ry = a->r[2 * (wb + pr) + 1];
                const double ra = hi ? ry : rx, rb = K == 1 ? ry : ra;
                const size_t o2 = 2 * ((size_t) wb * K + m);
                if (act0) {
                    const double q = a->pk[o2];
                    a->x[o2] = fma(o[c0].as, q, a->x[o2]);
                    a->pk[o2] = fma(o[c0].bs, q, o[c0].zn * ra);
                }
                if (act1) {
                    const double q = a->pk[o2 + 1];
                    a->x[o2 + 1] = fma(o[c1].as, q, a->x[o2 + 1]);
                    a->pk[o2 + 1] = fma(o[c1].bs, q, o[c1].zn * rb);
                }
            }
        }
    }
    if (n & 1) {
        const double rv = a->r[n - 1];
        a->p[n - 1] = fma(be, a->p[n - 1], rv);
        for (int j = 0; j < K; j++) {
            if (!(mask >> j & 1u)) continue;
            const size_t o1 = (size_t) (n - 1) * K + j;
            const double q = a->pk[o1];
            a->x[o1] = fma(o[j].as, q, a->x[o1]);
            a->pk[o1] = fma(o[j].bs, q, o[j].zn * rv);
        }
    }
}

int acgb200_cg_shift_update(int n, int k, struct acgb200_devstate *st, struct acgb200_sstate *ss, int cin, int cout,
                            const double *r, double *p, double *x, double *pk, cudaStream_t stream)
{
    (void) stream;
    if (k != 1 && k != 2 && k != 4 && k != 8) return 1;
    struct supd_args a;
    memset(&a, 0, sizeof(a));
    a.n = n; a.k = k; a.st = st; a.ss = ss; a.cin = cin; a.cout = cout; a.r = r; a.p = p; a.x = x; a.pk = pk;
    return hostsim_run_or_record(shift_update_exec, &a, sizeof(a));
}
