"""TEST INFRASTRUCTURE ONLY: drive acgsolvercuda_update_values on the device stand-in
(tests/hostsim/libacgb200_hostsim_refresh.so: the host-logic stand-in with every kernel stand-in, the comparison included) and compare the
refreshed solver with one built fresh on the same values.  Runs in its own process so that the binding loads the
stand-in; one mode per call (argv[1], JSON), asserts, and prints one JSON object.  Used by
tests/test_hostsim_refresh.py."""
import ctypes as C
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np                                   # noqa: E402

import acg_b200.api as api                           # noqa: E402
api._LIBPATH = os.path.join(HERE, "libacgb200_hostsim_refresh.so")    # before the first lib() call
import acg_b200 as ab                                # noqa: E402
from acg_b200 import matgen as mg                    # noqa: E402
from entrypoints import assert_same_products, assert_same_solves, run_products, run_solves   # noqa: E402

INVALID_VALUE = 29


def case(name):
    return {"27pt": lambda: mg.stencil3d_27pt(9, 8, 10), "7pt": lambda: mg.laplace3d_7pt(11, 9, 7),
            "rmat": lambda: mg.rmat_spd(2000, 32000, seed=1)}[name]()


def v2(r, c, v):
    return 2.0 * v + np.where(r == c, 1.0, 0.0)


def matrix(n, r, c, v, full=True):
    A = ab.SymCsrMatrix.init_real_double(n, r, c, v)
    return A.dsymv_init(0.0) if full else A


def run_all(cg, A):
    return run_products(ab, cg, A), run_solves(ab, cg, A)


def against_fresh(cg, A, tag):
    got_p, got_s = run_all(cg, A)
    fresh = ab.SolverCuda(A)
    want_p, want_s = run_all(fresh, A)
    fresh.free()
    assert_same_products(got_p, want_p, tag)
    assert_same_solves(got_s, want_s, tag)
    return got_s


def device_bytes(cg):
    """The solver's device arrays (host memory on the stand-in) and the public struct, as bytes."""
    out = [bytes(C.string_at(C.addressof(cg.c), C.sizeof(cg.c)))]
    nrp = cg.A.c.nownedrows + cg.A.c.nghostrows + 1
    norp = cg.A.c.nborderrows + cg.A.c.nghostrows + 1
    for name, count in (("d_rowptr", 4 * nrp), ("d_orowptr", 4 * norp)):
        out.append(C.string_at(getattr(cg.c, name), count))
    fnnz, onnz = int(np.frombuffer(out[1], np.int32)[-1]), int(np.frombuffer(out[2], np.int32)[-1])
    for name, count in (("d_colidx", 4 * fnnz), ("d_a", 8 * fnnz), ("d_ocolidx", 4 * onnz), ("d_oa", 8 * onnz)):
        if count:
            out.append(C.string_at(getattr(cg.c, name), count))
    return out


def mode_entrypoints(spec):
    """Every entry point before and after a refresh (full storage or packed source) against a fresh solver."""
    n, r, c, v = case(spec["matrix"])
    cg = ab.SolverCuda(matrix(n, r, c, v, full=spec.get("init_full", True)))
    before = run_all(cg, cg.A)[1]
    A2 = matrix(n, r, c, v2(r, c, v), full=spec.get("full", True))
    cg.update_values(A2)
    assert cg.A is A2
    after = against_fresh(cg, A2, "refresh")
    changed = [k for k in after if after[k][2] is not None and not np.array_equal(after[k][2], before[k][2])]
    cg.free()
    return {"changed": changed, "solves": sorted(after)}


def mode_alternate(spec):
    """Three refreshes alternating two value sets, each against a fresh solver."""
    n, r, c, v = case(spec["matrix"])
    A1, A2 = matrix(n, r, c, v), matrix(n, r, c, v2(r, c, v))
    cg = ab.SolverCuda(A1)
    run_all(cg, A1)
    its = []
    for A in (A2, A1, A2):
        cg.update_values(A)
        its.append(against_fresh(cg, A, "alternate")["solvempi"][1])
    cg.free()
    return {"its": its}


def mode_cheb_rmat(spec):
    """Jacobi PCG (Chebyshev degree 0) on R-MAT, then on the same pattern with the diagonal doubled: D^-1 is
    recomputed, so the count is the fresh solver's."""
    n, r, c, v = case("rmat")
    w = np.where(r == c, 2.0 * v, v)
    A1, A2 = matrix(n, r, c, v), matrix(n, r, c, w)
    b = np.random.default_rng(4).standard_normal(n)

    def solve(cg, A):
        bv = A.vector(); bv.x[:] = b
        xv = A.vector()
        cg.solve_chebyshev(bv, xv, degree=0, maxits=500, residualrtol=1e-10)
        return int(cg.c.niterations), xv.x[:n].copy()

    cg = ab.SolverCuda(A1)
    its1, _ = solve(cg, A1)
    cg.update_values(A2)
    its2, x2 = solve(cg, A2)
    fresh = ab.SolverCuda(A2)
    its0, x0 = solve(fresh, A2)
    fresh.free(); cg.free()
    assert x2.tobytes() == x0.tobytes()
    return {"its_v1": its1, "its_refreshed": its2, "its_fresh": its0}


def mode_refusals(spec):
    """Refused calls leave the solver bitwise as it was: its struct, its device arrays and its results."""
    n, r, c, v = case("27pt")
    A = matrix(n, r, c, v)
    cg = ab.SolverCuda(A)
    want = run_all(cg, A)
    snap = device_bytes(cg)
    k = int(np.flatnonzero((c > r + 1) & (c < n - 1))[0])
    row = int(r[k])
    free_col = next(j for j in range(row + 1, n) if not np.any((r == row) & (c == j)))
    c2 = c.copy(); c2[k] = free_col
    o = np.lexsort((c2, r))
    keep = np.ones(len(r), bool); keep[k] = False
    part = ab.SymCsrMatrix.init_real_double(n, r, c, v).partition(2, (np.arange(n) >= n // 2).astype(np.int32))[0]
    bad = {"moved-column": matrix(n, r[o], c2[o], v[o]), "moved-column-packed": matrix(n, r[o], c2[o], v[o], full=False),
           "entry-count": matrix(n, r[keep], c[keep], v[keep]),
           "entry-count-packed": matrix(n, r[keep], c[keep], v[keep], full=False),
           "partition": part.dsymv_init(0.0)}
    codes = {}
    for name, B in bad.items():
        try:
            cg.update_values(B)
            codes[name] = 0
        except ab.AcgError as e:
            codes[name] = e.code
        assert cg.A is A
        assert device_bytes(cg) == snap, name
    got = run_all(cg, A)
    assert_same_products(got[0], want[0], "refused")
    assert_same_solves(got[1], want[1], "refused")
    cg.free()
    try:
        cg.update_values(A)
        codes["freed"] = 0
    except ab.AcgError as e:
        codes["freed"] = e.code
    return {"codes": codes}


def mode_rank(spec):
    """One rank of a 2-rank partitioned solver: classic CG on V1, a refresh to V2 and classic CG again, then a
    fresh solver on V2; x of both solves on V2."""
    rank = spec["rank"]
    n, r, c, v = case("27pt")
    rowparts = (np.arange(n) >= n // 2).astype(np.int32)
    comm = ab.Comm.init_nccl(2, rank, bytes.fromhex(spec["uid"]))

    def part(vals):
        return ab.SymCsrMatrix.init_real_double(n, r, c, vals).partition(2, rowparts)[rank].dsymv_init(0.0)

    P1, P2 = part(v), part(v2(r, c, v))
    b = np.random.default_rng(6).standard_normal(n)
    no = P1.c.nownedrows
    gidx = P1.nzrows[:no].copy()

    def solve(cg, P):
        bv = P.vector(); bv.x[:no] = b[gidx]
        xv = P.vector()
        cg.solvempi(bv, xv, maxits=300, residualrtol=1e-10)
        return int(cg.c.niterations), xv.x[:no].tolist()

    cg = ab.SolverCuda(P1, comm)
    its1, _ = solve(cg, P1)
    cg.update_values(P2)
    its2, x2 = solve(cg, P2)
    fresh = ab.SolverCuda(P2, comm)
    its0, x0 = solve(fresh, P2)
    fresh.free(); cg.free()
    comm.destroy()
    return {"its_v1": its1, "its_refreshed": its2, "its_fresh": its0, "same_x": x2 == x0}


def mode_ranks(spec):
    uid = ab.Comm.unique_id().hex()
    procs = [subprocess.Popen([sys.executable, __file__, json.dumps({"mode": "rank", "rank": q, "uid": uid})],
                              stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True) for q in range(2)]
    outs = []
    for p in procs:
        so, se = p.communicate(timeout=600)
        assert p.returncode == 0, se[-3000:]
        outs.append(json.loads(so.strip().splitlines()[-1]))
    return {"ranks": outs}


def main():
    spec = json.loads(sys.argv[1])
    print(json.dumps(globals()["mode_" + spec["mode"]](spec)))


if __name__ == "__main__":
    main()
