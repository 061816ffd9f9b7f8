/*
 * kernels_mixed_sim.c -- TEST INFRASTRUCTURE ONLY.  Plain-C stand-ins for the mixed-precision launch
 * interface of acg_b200/csrc/kernels.cu (internal.h: acgb200_spmv_f32_launch, acgb200_mixed_setup,
 * acgb200_mixed_update_r, acgb200_mixed_update_yp, acgb200_mixed_replace, acgb200_mixed_fold), with the
 * kernels' roundings, scalar rules, slot discipline and control-word writes.  Linked with the host-logic
 * stand-in into libacgb200_hostsim_mixed.so by Makefile.mixed, so that the CPU test-suite can drive the host
 * code of acgsolvercuda_solve_mixed (set-up, gating of the reliable update, stopping, the fold at maxits,
 * graph slot and signature, warm-up) and compare it with tests/mixedref.py.  It says nothing about the CUDA
 * kernels -- those are tested on the H100 (tests/test_gpu_mixed.py).
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

static void spmv_f32_exec(void *vp)
{
    const struct acgb200_spmvf32args *a = vp;
    if (!gate_read(a->ctrl_in, a->st).active) return;
    /* the stand-in's plans have no mirrored diagonals: every row is in the chunks */
    double dot = 0.0;
    for (int c = 0; c < a->nranges; c++)
        for (int row = a->ranges[2 * c]; row < a->ranges[2 * c + 1]; row++) {
            double sum = 0.0;
            for (int k = a->rowptr[row]; k < a->rowptr[row + 1]; k++) sum = fma(a->a[k], (double) a->x[a->colidx[k]], sum);
            const float ys = (float) sum;
            a->y[row] = ys;
            dot = fma((double) a->x[row], (double) ys, dot);
        }
    if (a->acc) *a->acc += dot;
}

int acgb200_spmv_f32_launch(const struct acgb200_spmvf32args *a, cudaStream_t stream)
{
    (void) stream;
    if (a->plan->nslices > 0 && a->plan->symdiag_nd > 0) return 1;
    return hostsim_run_or_record(spmv_f32_exec, a, sizeof(*a));
}

struct setup_args { int n; double scale; const double *r64; float *r, *p, *y; };

static void setup_exec(void *vp)
{
    const struct setup_args *a = vp;
    for (int i = 0; i < a->n; i++) {
        const float v = (float) (a->r64[i] * a->scale);
        a->r[i] = v; a->p[i] = v; a->y[i] = 0.0f;
    }
}

int acgb200_mixed_setup(int n, double scale, const double *r64, float *r, float *p, float *y, cudaStream_t stream)
{
    (void) stream;
    struct setup_args a = { n, scale, r64, r, p, y };
    return hostsim_run_or_record(setup_exec, &a, sizeof(a));
}

struct step { double alpha, rr, beta; int bad, due; };

/* mixed_step of kernels.cu */
static struct step mixed_step(const struct acgb200_devstate *st, const struct acgb200_xstate *xs, int s)
{
    struct step o;
    const double pi = xs->pi[s], rho = xs->rho[s];
    o.bad = !(pi != 0.0 && isfinite(pi));
    o.alpha = o.bad ? 0.0 : rho / pi;
    o.rr = xs->rr[s];
    const double nr = sqrt(o.rr);
    o.due = nr < 0.1 * xs->mx[s] || xs->sigma[s] * nr < st->tol;
    o.beta = rho > 0.0 ? o.rr / rho : 0.0;
    return o;
}

struct update_r_args { int n; const struct acgb200_devstate *st; struct acgb200_xstate *xs; const float *t; float *r; };

static void update_r_exec(void *vp)
{
    const struct update_r_args *a = vp;
    const struct gate g = gate_read(&a->st->ctrl[0], a->st);
    if (!g.active) return;
    const int s = g.iter & 1;
    const double pi = a->xs->pi[s];
    if (!(pi != 0.0 && isfinite(pi))) return;
    const double alpha = a->xs->rho[s] / pi;
    double acc = 0.0;
    for (int i = 0; i < a->n; i++) {
        const float rv = (float) ((double) a->r[i] - alpha * (double) a->t[i]);
        a->r[i] = rv;
        acc = fma((double) rv, (double) rv, acc);
    }
    a->xs->rr[s] += acc;
}

int acgb200_mixed_update_r(int n, const struct acgb200_devstate *st, struct acgb200_xstate *xs, const float *t, float *r,
                           cudaStream_t stream)
{
    (void) stream;
    struct update_r_args a = { n, st, xs, t, r };
    return hostsim_run_or_record(update_r_exec, &a, sizeof(a));
}

struct update_yp_args { int n; struct acgb200_devstate *st; struct acgb200_xstate *xs; const float *r; float *p, *y; double *x; };

static void update_yp_exec(void *vp)
{
    const struct update_yp_args *a = vp;
    struct acgb200_devstate *st = a->st;
    struct acgb200_xstate *xs = a->xs;
    const struct gate g = gate_read(&st->ctrl[0], st);
    const int s = g.iter & 1;
    const struct step k = mixed_step(st, xs, s);
    struct acgb200_ctrl c1 = st->ctrl[0], c2 = st->ctrl[0];
    c2.done = 1;
    if (g.active) {
        if (k.bad) { c1.done = 1; xs->breakdown = 1; }
        else {
            c1.iter = g.iter + 1;
            if (k.due) { c2.done = 0; xs->rr64[s] = 0.0; }
            else { xs->rho[s ^ 1] = k.rr; xs->mx[s ^ 1] = fmax(xs->mx[s], sqrt(k.rr)); xs->sigma[s ^ 1] = xs->sigma[s]; }
        }
        xs->pi[s ^ 1] = 0.0;
        xs->rr[s ^ 1] = 0.0;
    }
    st->ctrl[1] = c1;
    st->ctrl[2] = c2;
    if (!g.active || k.bad) return;
    const double sigma = xs->sigma[s];
    for (int i = 0; i < a->n; i++) {
        const float yn = (float) ((double) a->y[i] + k.alpha * (double) a->p[i]);
        if (k.due) { a->x[i] = a->x[i] + sigma * (double) yn; a->y[i] = 0.0f; }
        else { a->y[i] = yn; a->p[i] = (float) ((double) a->r[i] + k.beta * (double) a->p[i]); }
    }
}

int acgb200_mixed_update_yp(int n, struct acgb200_devstate *st, struct acgb200_xstate *xs, const float *r, float *p,
                            float *y, double *x, cudaStream_t stream)
{
    (void) stream;
    struct update_yp_args a = { n, st, xs, r, p, y, x };
    return hostsim_run_or_record(update_yp_exec, &a, sizeof(a));
}

static int scale_exp(double rr64)
{
    int e = 0;
    const double m = frexp(sqrt(rr64), &e);
    return m < 0.70710678118654752440 ? e - 1 : e;
}

struct replace_args { int n; struct acgb200_devstate *st; struct acgb200_xstate *xs; const double *r64; float *r, *p; };

static void replace_exec(void *vp)
{
    const struct replace_args *a = vp;
    struct acgb200_devstate *st = a->st;
    struct acgb200_xstate *xs = a->xs;
    const struct gate g = gate_read(&st->ctrl[2], st);
    const int s = g.iter & 1;
    const double rr64 = xs->rr64[s];
    const int stop = sqrt(rr64) < st->tol || rr64 == 0.0;
    const int e = g.active && !stop ? scale_exp(rr64) : 0;
    const double sigma = xs->sigma[s], rho = xs->rho[s];
    struct acgb200_ctrl c = st->ctrl[1];
    if (g.active) {
        xs->nupdates += 1;
        xs->last_rr64 = rr64;
        c.iter = g.iter + 1; c.done = 0;
        if (stop) { c.done = 1; xs->conv = 1; }
        else {
            const double rn = ldexp(rr64, -2 * e);
            xs->rho[s ^ 1] = rn; xs->mx[s ^ 1] = sqrt(rn); xs->sigma[s ^ 1] = ldexp(1.0, e);
        }
    }
    st->ctrl[0] = c;
    if (!g.active || stop) return;
    const double is = ldexp(1.0, -e);
    const double bf = (rr64 / (sigma * sigma)) / rho * (sigma * is);
    for (int i = 0; i < a->n; i++) {
        const double rv = a->r64[i] * is;
        a->p[i] = (float) (rv + bf * (double) a->p[i]);
        a->r[i] = (float) rv;
    }
}

int acgb200_mixed_replace(int n, struct acgb200_devstate *st, struct acgb200_xstate *xs, const double *r64, float *r,
                          float *p, cudaStream_t stream)
{
    (void) stream;
    struct replace_args a = { n, st, xs, r64, r, p };
    return hostsim_run_or_record(replace_exec, &a, sizeof(a));
}

struct fold_args { int n; double sigma; const float *y; double *x; };

static void fold_exec(void *vp)
{
    const struct fold_args *a = vp;
    for (int i = 0; i < a->n; i++) a->x[i] = a->x[i] + a->sigma * (double) a->y[i];
}

int acgb200_mixed_fold(int n, double sigma, const float *y, double *x, cudaStream_t stream)
{
    (void) stream;
    struct fold_args a = { n, sigma, y, x };
    return hostsim_run_or_record(fold_exec, &a, sizeof(a));
}
