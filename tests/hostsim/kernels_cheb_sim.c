/*
 * kernels_cheb_sim.c -- TEST INFRASTRUCTURE ONLY.  Plain-C stand-ins for the Chebyshev-preconditioned CG launch
 * interface of acg_b200/csrc/kernels.cu (internal.h: acgb200_cheb_dinv, acgb200_cheb_rx, acgb200_cheb_step,
 * acgb200_cheb_fused_step, acgb200_cheb_p), with the kernels' order of operations, scalar rules, slot
 * discipline and control-word writes.  Linked with the host-logic stand-in into libacgb200_hostsim_cheb.so by
 * Makefile.cheb, so that the CPU test-suite can drive the host code of acgsolvercuda_solve_chebyshev (set-up,
 * the interval estimate, stopping, breakdowns, graph slot and signature, warm-up) and compare it with
 * tests/chebref.py.  It says nothing about the CUDA kernels -- those are tested on the H100
 * (tests/test_gpu_chebyshev.py).
 */
#include "internal.h"
#include "hostsim.h"

#include <math.h>
#include <string.h>

struct gate { int iter, active; };

/* as gate_read of kernels.cu */
static struct gate gate_read(const struct acgb200_ctrl *cin, const struct acgb200_devstate *st)
{
    struct gate g = { 0, 1 };
    if (cin) { g.iter = cin->iter; g.active = cin->done == 0 && cin->iter < st->maxits; }
    return g;
}

struct dinv_args { int n; const int *rowptr, *colidx; const double *a; double *dinv; struct acgb200_cstate *cs; };

static void dinv_exec(void *vp)
{
    const struct dinv_args *a = vp;
    for (int i = 0; i < a->n; i++) {
        double v = 0.0;
        for (int k = a->rowptr[i]; k < a->rowptr[i + 1]; k++) if (a->colidx[k] == i) v += a->a[k];
        if (!(v > 0.0 && isfinite(v))) a->cs->baddiag++;
        a->dinv[i] = 1.0 / v;
    }
}

int acgb200_cheb_dinv(int n, const int *rowptr, const int *colidx, const double *a, double *dinv,
                      struct acgb200_cstate *cs, cudaStream_t stream)
{
    (void) stream;
    struct dinv_args x = { n, rowptr, colidx, a, dinv, cs };
    return hostsim_run_or_record(dinv_exec, &x, sizeof(x));
}

struct rx_args {
    int n; struct acgb200_devstate *st; struct acgb200_cstate *cs; int start, cheb; double c0;
    const double *dinv, *t, *p; double *x, *r, *z, *res, *d0;
};

static void rx_exec(void *vp)
{
    const struct rx_args *a = vp;
    struct acgb200_devstate *st = a->st;
    struct acgb200_cstate *cs = a->cs;
    const struct gate g = gate_read(&st->ctrl[1], st);
    const int s = g.iter & 1;
    const double rz = a->start ? 1.0 : cs->rz[g.iter % 3], pap = a->start ? 1.0 : cs->pap[s];
    const int bad = !(rz > 0.0 && isfinite(rz)) || !(pap > 0.0 && isfinite(pap));
    const double alpha = rz / pap;
    struct acgb200_ctrl c = st->ctrl[1];
    if (g.active && bad) { c.done = 1; cs->breakdown = 1; }
    else if (g.active && !a->start && cs->log && g.iter < ACGB200_CHEB_EST) cs->alpha_log[g.iter] = alpha;
    st->ctrl[2] = c;
    if (!g.active || bad) return;
    double rr = 0.0, rzn = 0.0;
    for (int i = 0; i < a->n; i++) {
        double ri = a->r[i];
        if (!a->start) {
            if (a->x) a->x[i] = fma(alpha, a->p[i], a->x[i]);
            ri = fma(-alpha, a->t[i], ri);
            a->r[i] = ri;
            rr = fma(ri, ri, rr);
        }
        const double zi = a->dinv[i] * ri;
        if (a->cheb) {
            const double dv = a->c0 * zi;
            a->res[i] = ri; a->d0[i] = dv; a->z[i] = dv;
        } else {
            a->z[i] = zi;
            rzn = fma(ri, zi, rzn);
        }
    }
    if (!a->start) cs->rr[s] += rr;
    if (!a->cheb) cs->rz[(g.iter + 1) % 3] += rzn;
}

int acgb200_cheb_rx(int n, struct acgb200_devstate *st, struct acgb200_cstate *cs, int start, int cheb, double c0,
                    const double *dinv, const double *t, const double *p, double *x, double *r, double *z,
                    double *res, double *d0, cudaStream_t stream)
{
    (void) stream;
    struct rx_args a = { n, st, cs, start, cheb, c0, dinv, t, p, x, r, z, res, d0 };
    return hostsim_run_or_record(rx_exec, &a, sizeof(a));
}

struct step_args {
    int n; const struct acgb200_devstate *st; struct acgb200_cstate *cs; double c1, c2; int last;
    const double *q, *dinv, *dprev; double *dnext, *res, *z; const double *r;
};

static void step_exec(void *vp)
{
    const struct step_args *a = vp;
    const struct gate g = gate_read(&a->st->ctrl[2], a->st);
    if (!g.active) return;
    double rz = 0.0;
    for (int i = 0; i < a->n; i++) {
        const double rv = a->res[i] - a->q[i];
        const double dn = fma(a->c1, a->dprev[i], a->c2 * (a->dinv[i] * rv));
        const double zv = a->z[i] + dn;
        a->z[i] = zv;
        if (a->last) rz = fma(a->r[i], zv, rz);
        else { a->res[i] = rv; a->dnext[i] = dn; }
    }
    if (a->last) a->cs->rz[(g.iter + 1) % 3] += rz;
}

int acgb200_cheb_step(int n, const struct acgb200_devstate *st, struct acgb200_cstate *cs, double c1, double c2,
                      int last, const double *q, const double *dinv, const double *dprev, double *dnext, double *res,
                      double *z, const double *r, cudaStream_t stream)
{
    (void) stream;
    struct step_args a = { n, st, cs, c1, c2, last, q, dinv, dprev, dnext, res, z, r };
    return hostsim_run_or_record(step_exec, &a, sizeof(a));
}

/* the stand-in's plans have no mirrored diagonals (kernels_sim.c), so the host never selects the fused step */
int acgb200_cheb_fused_step(const struct acgb200_chebargs *a, cudaStream_t stream)
{
    (void) a; (void) stream;
    return 1;
}

struct p_args { int n; struct acgb200_devstate *st; struct acgb200_cstate *cs; const double *z; double *p; };

static void p_exec(void *vp)
{
    const struct p_args *a = vp;
    struct acgb200_devstate *st = a->st;
    struct acgb200_cstate *cs = a->cs;
    const struct gate g = gate_read(&st->ctrl[2], st);
    const int s = g.iter & 1;
    const double rr = cs->rr[s];
    const int conv = st->tol > 0.0 && sqrt(rr) < st->tol;
    const double beta = cs->rz[(g.iter + 1) % 3] / cs->rz[g.iter % 3];
    struct acgb200_ctrl c = st->ctrl[2];
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
    if (!g.active || conv) return;
    for (int i = 0; i < a->n; i++) a->p[i] = fma(beta, a->p[i], a->z[i]);
}

int acgb200_cheb_p(int n, struct acgb200_devstate *st, struct acgb200_cstate *cs, const double *z, double *p,
                   cudaStream_t stream)
{
    (void) stream;
    struct p_args a = { n, st, cs, z, p };
    return hostsim_run_or_record(p_exec, &a, sizeof(a));
}
