"""TEST INFRASTRUCTURE ONLY: what every solve entry point reports around its loop, on the device stand-in of
tests/hostsim (libacgb200_hostsim_refresh.so: the host-logic stand-in with every kernel stand-in).  For a 7-point
Laplacian and an R-MAT matrix, each entry point runs converged, maxits-bound and maxits = 0 solves, each with
warm-up 0 and 2 and a nonzero initial guess, on one solver per matrix (so the counters accumulate), and then every
refused call.  Each run records the return code, the iterations, the norms, every counter of struct acgsolvercuda,
the launch and product counts of acgsolvercuda_info, its solver-specific fields and the 2-norm of x.  Prints one
JSON object of one record per line, the content of tests/golden/entry_frame.json:

    OMP_NUM_THREADS=2 python tests/hostsim/run_frame_sim.py > tests/golden/entry_frame.json

Used by tests/test_hostsim_frame.py.  argv[1] (optional): the library to load instead."""
import ctypes as C
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import numpy as np                                   # noqa: E402

import acg_b200.api as api                           # noqa: E402
api._LIBPATH = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "libacgb200_hostsim_refresh.so")
import acg_b200 as ab                                # noqa: E402
from acg_b200 import matgen as mg                    # noqa: E402

COUNTERS = ("maxits", "nsolves", "ntotaliterations", "niterations", "nflops", "ngemv", "ndot", "nnrm2", "naxpy",
            "ncopy", "nallreduce", "nhalo", "Bgemv", "Bdot", "Bnrm2", "Baxpy", "Bcopy", "Ballreduce", "Bhalo",
            "nhalomsgs", "bnrm2", "r0nrm2", "rnrm2", "residualatol", "residualrtol", "diffatol", "diffrtol")
INFO = ("last_launches", "last_spmv_count", "pcg_fused", "pcg_group", "mixed_reliable_updates", "cheb_degree",
        "cheb_est_iterations", "cheb_breakdown", "cheb_lmin", "cheb_lmax")
FIELDS = COUNTERS + INFO
SCENARIOS = {"converged": dict(maxits=400, residualrtol=1e-10), "maxits": dict(maxits=5, residualrtol=1e-14),
             "maxits0": dict(maxits=0, residualrtol=1e-10)}


def matrices():
    return {"7pt": mg.laplace3d_7pt(11, 9, 7), "rmat": mg.rmat_spd(1500, 20000, seed=3)}


def state(cg):
    """The values of FIELDS, in that order."""
    info = cg.info()
    return {"state": [getattr(cg.c, k) for k in COUNTERS] + [info[k] for k in INFO]}


def vec_entry(name, **extra):
    def run(cg, A, b, x0, kw, warmup):
        bv = A.vector(); bv.x[:len(b)] = b
        xv = A.vector(); xv.x[:len(x0)] = x0
        if name == "solve_pipelined_2k":
            ab.set_option("pcg_fused", 0)
            try:
                code = cg.solve_pipelined(bv, xv, warmup=warmup, **kw)
            finally:
                ab.set_option("pcg_fused", 1)
        else:
            code = getattr(cg, name)(bv, xv, warmup=warmup, **kw, **extra)
        return code, {"x_nrm2": float(np.linalg.norm(xv.x[:len(x0)]))}
    return run


def multi(cg, A, b, x0, kw, warmup):
    B = np.stack([b, np.roll(b, 1), -b], axis=1)
    X = np.ascontiguousarray(np.stack([x0, 0 * x0, np.roll(x0, 3)], axis=1))
    code, st = cg.solve_multi(B, X, warmup=warmup, **kw)
    return code, {"x_nrm2": float(np.linalg.norm(X)), "cols": st}


def shifted(cg, A, b, x0, kw, warmup):
    code, X, st = cg.solve_shifted(b, [0.0, 0.25, 3.0], warmup=warmup, **kw)
    return code, {"x_nrm2": float(np.linalg.norm(X)), "cols": st}


ENTRIES = {"solvempi": vec_entry("solvempi"), "solve": vec_entry("solve"), "solve_device": vec_entry("solve_device"),
           "solve_pipelined": vec_entry("solve_pipelined"), "solve_pipelined_2k": vec_entry("solve_pipelined_2k"),
           "solve_device_pipelined": vec_entry("solve_device_pipelined"), "solve_multi": multi,
           "solve_shifted": shifted, "solve_minres": vec_entry("solve_minres"),
           "solve_mixed": vec_entry("solve_mixed"), "solve_cheb0": vec_entry("solve_chebyshev", degree=0),
           "solve_cheb2": vec_entry("solve_chebyshev", degree=2),
           "solve_cheb3_interval": vec_entry("solve_chebyshev", degree=3, lmin=0.05, lmax=20.0)}


def solves(cg, A, n):
    rng = np.random.default_rng(5)
    b = rng.standard_normal(n)
    x0 = 0.1 * rng.standard_normal(n)
    out = {}
    for name, fn in ENTRIES.items():
        for sc, kw in SCENARIOS.items():
            for warmup in (0, 2):
                code, extra = fn(cg, A, b, x0, kw, warmup)
                out[f"{name}/{sc}/w{warmup}"] = dict(code=code, **extra, **state(cg))
    return out


def raw(L, fn, *args):
    """A call through a function pointer without argument conversion, so that NULL can be passed anywhere."""
    f = getattr(L, fn)
    f.restype = C.c_int
    return f(*args)


def refusals(cg, A, P, n):
    """Each refused call with its code and the solver's counters after it.  P is one part of a 2-way partition
    of A (ghost rows): a one-GPU entry point refuses it."""
    L = C.CDLL(api._LIBPATH)
    pc, pA, pP = C.byref(cg.c), C.byref(A.c), C.byref(P.c)
    b = A.vector(); b.x[:] = 1.0
    x = A.vector()
    pb, px = C.byref(b.c), C.byref(x.c)
    B = np.ones((n, 2)); X = np.zeros((n, 2)); bh = np.ones(n)
    Bp, Xp, bhp = (M.ctypes.data_as(C.c_void_p) for M in (B, X, bh))
    sh = np.array([0.0, 0.5]); shp = sh.ctypes.data_as(C.c_void_p)
    bad_sh = {"neg": np.array([0.0, -1.0]), "nan": np.array([np.nan, 0.0]), "inf": np.array([0.0, np.inf])}
    d, i = C.c_double, C.c_int
    err = C.c_int(0); pe = C.byref(err)
    null = ab.Comm()
    cases = {
        "solvempi/diffatol": lambda: raw(L, "acgsolvercuda_solvempi", pc, pA, pb, px, i(10), d(1e-3), d(0), d(0), d(0),
                                         i(0), C.byref(null.c), i(0), pe, None, None, i(0)),
        "solve_pipelined/diffrtol": lambda: raw(L, "acgsolvercuda_solve_pipelined", pc, pA, pb, px, i(10), d(0), d(1e-3),
                                                d(0), d(0), i(0), C.byref(null.c), i(0), pe, None, None),
        "solve/diffatol": lambda: raw(L, "acgsolvercuda_solve", pc, pA, pb, px, i(10), d(1e-3), d(0), d(0), d(0), i(0)),
    }

    def multi_call(nrhs, Bq, Xq, maxits, M=pA):
        return lambda: raw(L, "acgsolvercuda_solve_multi", pc, M, i(nrhs), Bq, Xq, i(maxits), d(0), d(1e-8), i(0), None)
    cases.update({"multi/nrhs0": multi_call(0, Bp, Xp, 10), "multi/nrhs9": multi_call(9, Bp, Xp, 10),
                  "multi/B": multi_call(2, None, Xp, 10), "multi/X": multi_call(2, Bp, None, 10),
                  "multi/maxits": multi_call(2, Bp, Xp, -1), "multi/partitioned": multi_call(2, Bp, Xp, 10, pP),
                  "multi/partitioned_B": multi_call(2, None, Xp, 10, pP)})

    def shift_call(ns, s, bq, Xq, maxits, M=pA):
        return lambda: raw(L, "acgsolvercuda_solve_shifted", pc, M, i(ns), s, bq, Xq, i(maxits), d(0), d(1e-8), i(0),
                           None)
    cases.update({"shifted/n0": shift_call(0, shp, bhp, Xp, 10), "shifted/n9": shift_call(9, shp, bhp, Xp, 10),
                  "shifted/shifts": shift_call(2, None, bhp, Xp, 10), "shifted/b": shift_call(2, shp, None, Xp, 10),
                  "shifted/X": shift_call(2, shp, bhp, None, 10), "shifted/maxits": shift_call(2, shp, bhp, Xp, -1),
                  "shifted/partitioned": shift_call(2, shp, bhp, Xp, 10, pP),
                  "shifted/partitioned_b": shift_call(2, shp, None, Xp, 10, pP)})
    for k, s in bad_sh.items():
        cases[f"shifted/{k}"] = shift_call(2, s.ctypes.data_as(C.c_void_p), bhp, Xp, 10)

    for fn in ("minres", "mixed"):
        def vcall(M, bq, xq, maxits, fn=fn):
            return lambda: raw(L, f"acgsolvercuda_solve_{fn}", pc, M, bq, xq, i(maxits), d(0), d(1e-8), i(0), pe)
        cases.update({f"{fn}/A": vcall(None, pb, px, 10), f"{fn}/b": vcall(pA, None, px, 10),
                      f"{fn}/x": vcall(pA, pb, None, 10), f"{fn}/maxits": vcall(pA, pb, px, -1),
                      f"{fn}/partitioned": vcall(pP, pb, px, 10), f"{fn}/partitioned_b": vcall(pP, None, px, 10),
                      f"{fn}/partitioned_maxits": vcall(pP, pb, px, -1)})

    def ccall(M, bq, xq, degree, lmin, lmax, maxits):
        return lambda: raw(L, "acgsolvercuda_solve_chebyshev", pc, M, bq, xq, i(degree), d(lmin), d(lmax), i(maxits),
                           d(0), d(1e-8), i(0), pe)
    cases.update({"cheb/A": ccall(None, pb, px, 2, 0, 0, 10), "cheb/b": ccall(pA, None, px, 2, 0, 0, 10),
                  "cheb/x": ccall(pA, pb, None, 2, 0, 0, 10), "cheb/maxits": ccall(pA, pb, px, 2, 0, 0, -1),
                  "cheb/degree-1": ccall(pA, pb, px, -1, 0, 0, 10), "cheb/degree17": ccall(pA, pb, px, 17, 0, 0, 10),
                  "cheb/lmin_nan": ccall(pA, pb, px, 2, float("nan"), 0, 10),
                  "cheb/lmax_neg": ccall(pA, pb, px, 2, 0, -1.0, 10),
                  "cheb/lmax_inf": ccall(pA, pb, px, 2, 0, float("inf"), 10),
                  "cheb/lmin_ge_lmax": ccall(pA, pb, px, 2, 2.0, 1.0, 10),
                  "cheb/deg0_any_interval": ccall(pA, pb, px, 0, float("nan"), -1.0, 10),
                  "cheb/lmin_above_estimate": ccall(pA, pb, px, 2, 1e6, 0, 10),
                  "cheb/partitioned": ccall(pP, pb, px, 2, 0, 0, 10),
                  "cheb/partitioned_degree": ccall(pP, pb, px, -1, 0, 0, 10)})

    xf = np.ones(n, np.float32); yf = np.zeros(n, np.float32)
    xfp, yfp = xf.ctypes.data_as(C.c_void_p), yf.ctypes.data_as(C.c_void_p)
    Yp = np.zeros((n, 2)).ctypes.data_as(C.c_void_p)
    cases.update({
        "spmv_f32/x": lambda: raw(L, "acgsolvercuda_spmv_f32", pc, None, yfp, None),
        "spmv_f32/y": lambda: raw(L, "acgsolvercuda_spmv_f32", pc, xfp, None, None),
        "spmm_mode/nrhs0": lambda: raw(L, "acgsolvercuda_spmm_mode", pc, i(0), i(0), Xp, None, Yp, None),
        "spmm_mode/X": lambda: raw(L, "acgsolvercuda_spmm_mode", pc, i(0), i(2), None, None, Yp, None),
        "spmm_mode/mode": lambda: raw(L, "acgsolvercuda_spmm_mode", pc, i(3), i(2), Xp, None, Yp, None),
        "spmm_mode/B": lambda: raw(L, "acgsolvercuda_spmm_mode", pc, i(2), i(2), Xp, None, Yp, None)})
    out = {}
    for name, call in cases.items():
        code = call()
        out[name] = dict(code=code, **state(cg))
    return out


def products(cg, A, n):
    """The two products whose solve context is built by hand: their dots and the 2-norms of their results."""
    rng = np.random.default_rng(9)
    x32 = rng.integers(-4, 5, n).astype(np.float32)
    y, dot = cg.spmv_f32(x32)
    out = {"spmv_f32": {"y_nrm2": float(np.linalg.norm(y.astype(np.float64))), "dot": dot}}
    X, B = rng.integers(-4, 5, (n, 3)).astype(np.float64), rng.integers(-4, 5, (n, 3)).astype(np.float64)
    for m in (0, 1, 2):
        Y, dots = cg.spmm_mode(m, X, B if m == 2 else None)
        out[f"spmm_mode{m}"] = {"y_nrm2": float(np.linalg.norm(Y)), "dots": dots.tolist()}
    return out


def negated_diagonal(n, r, c, v):
    """Chebyshev refuses a matrix with a nonpositive diagonal entry, after its set-up."""
    w = np.where((r == c) & (r == n // 2), -v, v)
    A = ab.SymCsrMatrix.init_real_double(n, r, c, w).dsymv_init(0.0)
    cg = ab.SolverCuda(A)
    bv = A.vector(); bv.x[:] = 1.0
    xv = A.vector()
    try:
        code = cg.solve_chebyshev(bv, xv, degree=2, maxits=10)
    except ab.AcgError as e:
        code = e.code
    out = dict(code=code, **state(cg))
    cg.free()
    return out


def main():
    res = {"fields": FIELDS}
    for mname, (n, r, c, v) in matrices().items():
        A = ab.SymCsrMatrix.init_real_double(n, r, c, v).dsymv_init(0.0)
        P = ab.SymCsrMatrix.init_real_double(n, r, c, v).partition(2, (np.arange(n) >= n // 2).astype(np.int32))[0]
        P = P.dsymv_init(0.0)
        cg = ab.SolverCuda(A)
        for part, fn in (("solves", solves), ("refusals", lambda cg, A, n: refusals(cg, A, P, n)),
                         ("products", products)):
            res.update({f"{mname}/{part}/{k}": v for k, v in fn(cg, A, n).items()})
        cg.free()
        res[f"{mname}/cheb_baddiag"] = negated_diagonal(n, r, c, v)
    # one record per line
    print("{\n" + ",\n".join(f"{json.dumps(k)}: {json.dumps(v, sort_keys=True)}" for k, v in res.items()) + "\n}")


if __name__ == "__main__":
    main()
