/*
 * kernels_minres_sim.c -- TEST INFRASTRUCTURE ONLY.  Plain-C stand-ins for the MINRES launch interface of
 * acg_b200/csrc/kernels.cu (internal.h: acgb200_minres_setup, acgb200_minres_lanczos, acgb200_minres_update),
 * with the kernels' scalar recurrence (minres_step), fma grouping, slot discipline and control-word writes.
 * Linked with the host-logic stand-in into libacgb200_hostsim_minres.so by Makefile.minres, so that the CPU
 * test-suite can drive the host code of acgsolvercuda_solve_minres (set-up, buffer parity, stopping,
 * breakdown, graph slot and signature, warm-up) and compare it with tests/minresref.py.  It says nothing
 * about the CUDA kernels -- those are tested on the H100 (tests/test_gpu_minres.py).
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

struct setup_args { int n; double scale; double *v, *vprev, *w0, *w1; };

static void setup_exec(void *vp)
{
    const struct setup_args *a = vp;
    for (int i = 0; i < a->n; i++) {
        a->v[i] = a->scale * a->v[i];
        a->vprev[i] = 0.0; a->w0[i] = 0.0; a->w1[i] = 0.0;
    }
}

int acgb200_minres_setup(int n, double scale, double *v, double *vprev, double *w0, double *w1, cudaStream_t stream)
{
    (void) stream;
    struct setup_args a = { n, scale, v, vprev, w0, w1 };
    return hostsim_run_or_record(setup_exec, &a, sizeof(a));
}

struct lanczos_args { int n; const struct acgb200_devstate *st; struct acgb200_nstate *ns; int cin; const double *v, *vprev; double *t; };

static void lanczos_exec(void *vp)
{
    const struct lanczos_args *a = vp;
    const struct gate g = gate_read(&a->st->ctrl[a->cin], a->st);
    if (!g.active) return;
    const int s = g.iter & 1;
    const double al = a->ns->alpha[s], be = a->ns->beta[s];
    double acc = 0.0;
    for (int i = 0; i < a->n; i++) {
        const double u = fma(-be, a->vprev[i], fma(-al, a->v[i], a->t[i]));
        a->t[i] = u;
        acc = fma(u, u, acc);
    }
    a->ns->uu[s] += acc;
}

int acgb200_minres_lanczos(int n, const struct acgb200_devstate *st, struct acgb200_nstate *ns, int cin,
                           const double *v, const double *vprev, double *t, cudaStream_t stream)
{
    (void) stream;
    struct lanczos_args a = { n, st, ns, cin, v, vprev, t };
    return hostsim_run_or_record(lanczos_exec, &a, sizeof(a));
}

struct step { double beta, delta, eps, gamma, cs, sn, phi, phibar, dbar, epsn; };

/* minres_step of kernels.cu */
static struct step minres_step(const struct acgb200_nstate *ns, int s)
{
    struct step o;
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

struct update_args {
    int n; struct acgb200_devstate *st; struct acgb200_nstate *ns; int cin, cout;
    const double *v, *u; double *w; const double *wprev; double *x, *vnext;
};

static void update_exec(void *vp)
{
    const struct update_args *a = vp;
    struct acgb200_devstate *st = a->st;
    struct acgb200_nstate *ns = a->ns;
    const struct gate g = gate_read(&st->ctrl[a->cin], st);
    const int s = g.iter & 1;
    const struct step k = minres_step(ns, s);      /* every thread's scalars, from slot s */
    struct acgb200_ctrl c = st->ctrl[a->cin];
    if (g.active) {
        if (k.gamma == 0.0) c.done = 1;
        else {
            c.iter = g.iter + 1;
            ns->beta[s ^ 1] = k.beta; ns->cs[s ^ 1] = k.cs; ns->sn[s ^ 1] = k.sn;
            ns->dbar[s ^ 1] = k.dbar; ns->eps[s ^ 1] = k.epsn; ns->phibar[s ^ 1] = k.phibar;
            if (k.beta == 0.0 || (st->tol > 0.0 && k.phibar < st->tol)) c.done = 1;
        }
        ns->alpha[s ^ 1] = 0.0;
        ns->uu[s ^ 1] = 0.0;
    }
    st->ctrl[a->cout] = c;
    if (!g.active || k.gamma == 0.0) return;
    const double ig = 1.0 / k.gamma, ib = k.beta > 0.0 ? 1.0 / k.beta : 0.0;
    for (int i = 0; i < a->n; i++) {
        const double wv = fma(-k.delta, a->wprev[i], fma(-k.eps, a->w[i], a->v[i])) * ig;
        a->w[i] = wv;
        a->x[i] = fma(k.phi, wv, a->x[i]);
        a->vnext[i] = a->u[i] * ib;
    }
}

int acgb200_minres_update(int n, struct acgb200_devstate *st, struct acgb200_nstate *ns, int cin, int cout,
                          const double *v, const double *u, double *w, const double *wprev, double *x, double *vnext,
                          cudaStream_t stream)
{
    (void) stream;
    struct update_args a;
    memset(&a, 0, sizeof(a));
    a.n = n; a.st = st; a.ns = ns; a.cin = cin; a.cout = cout; a.v = v; a.u = u; a.w = w; a.wprev = wprev;
    a.x = x; a.vnext = vnext;
    return hostsim_run_or_record(update_exec, &a, sizeof(a));
}
