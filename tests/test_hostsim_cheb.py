"""Host logic of acgsolvercuda_solve_chebyshev (CG preconditioned with a Chebyshev polynomial in D^-1 A) on the
device stand-in of tests/hostsim, against the restatement of tests/chebref.py: equal codes, iteration counts,
estimate steps, intervals and product counts, x within 1e-12 relative, and the recursively updated residual
norm.  Covers degrees 0, 1, 2, 5 and 16, a given and an estimated interval, an estimate cut short, maxits
reached, maxits = 0, r0 = 0, warm-up 0 and 2, every rejected call, a breakdown from an interval with a + b
below lambda_max(D^-1 A), and solve_chebyshev, solvempi and solve_mixed alternating on one solver.  The
stand-in keeps the kernels' order of operations, scalar rules and slot discipline; the kernels themselves
are checked on the H100 by test_gpu_chebyshev.py."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIM = os.path.join(ROOT, "tests", "hostsim")
NOT_CONVERGED, INVALID_VALUE, NOT_SUPPORTED = 39, 29, 26


@pytest.fixture(scope="module")
def simlib():
    p = subprocess.run(["make", "-C", SIM, "-f", "Makefile.cheb"], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
    assert "warning" not in p.stderr
    return os.path.join(SIM, "libacgb200_hostsim_cheb.so")


def _run(spec):
    p = subprocess.run([sys.executable, os.path.join(SIM, "run_cheb_sim.py"), json.dumps(spec)], capture_output=True,
                       text=True, timeout=900, env=dict(os.environ, OMP_NUM_THREADS="2"))
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-3000:]
    return json.loads(p.stdout.strip().splitlines()[-1])


def _check(out):
    for r in out["runs"]:
        assert r["code"] == r["ref_code"], r
        if r["ref_code"] == INVALID_VALUE:
            assert r["x_is_x0"], r
            continue
        assert r["its"] == r["ref_its"], r
        assert r["est"] == r["ref_est"], r
        assert r["ngemv"] == r["ref_products"], r
        assert r["deg"] == r["run"]["degree"]
        assert r["breakdown"] == (r["ref_stop"] == "breakdown"), r
        assert r["lmin"] == pytest.approx(r["ref_lmin"], rel=1e-12) and r["lmax"] == pytest.approx(r["ref_lmax"], rel=1e-12)
        assert r["xerr"] < r["run"].get("xtol", 1e-12), r
        assert r["bnrm2"] == pytest.approx(r["ref_bnrm2"], rel=1e-13, abs=1e-300)
        assert r["r0nrm2"] == pytest.approx(r["ref_r0nrm2"], rel=1e-13, abs=1e-300)
        # the recursively updated norm near the tolerance carries the rounding of the sums in its last digits
        assert r["rnrm2"] == pytest.approx(r["ref_rnrm2"], rel=1e-6, abs=max(1e-13 * r["bnrm2"], 0.1 * r["tol"])), r
        if r["code"] == 0 and r["tol"] > 0:
            assert r["true_rnrm2"] < 2 * r["tol"], r


@pytest.mark.parametrize("matrix", ["7pt", "27pt", "rmat"])
def test_against_restatement(matrix, simlib):
    """Degrees 0, 1, 2, 5 and 16 with the estimated interval, and degree 2 with a given one (both bounds, and
    the upper bound alone), from x0 = 0 and a nonzero x0, with warm-up 0 and 2."""
    runs = [{"degree": d, "maxits": 400, "rtol": 1e-10} for d in (0, 1, 2, 5, 16)]
    runs += [{"degree": 2, "lmin": 0.1, "lmax": 2.2, "maxits": 400, "rtol": 1e-10, "x0": 1, "warmup": 2},
             {"degree": 3, "lmax": 2.2, "maxits": 400, "atol": 1e-9, "warmup": 2}]
    out = _run({"matrix": matrix, "runs": runs})
    _check(out)
    assert all(r["ref_stop"] == "tol" and r["code"] == 0 for r in out["runs"])
    assert all(r["est"] == 10 for r in out["runs"][1:5])
    assert out["runs"][5]["est"] == 0 and out["runs"][5]["lmin"] == 0.1 and out["runs"][5]["lmax"] == 2.2
    assert out["runs"][6]["lmin"] == pytest.approx(0.22)


def test_estimate_cut_short(simlib):
    """2 x 2 blocks: D^-1 A has two eigenvalues, so Jacobi PCG meets the tolerance after 2 steps and the
    estimate uses those 2; the interval is then [0.165, 1.65].  R-MAT with b = 1: 1 is an eigenvector of A but
    not of D^-1 A, so the estimate there runs its 10 steps."""
    out = _run({"matrix": "pairs", "runs": [{"degree": d, "maxits": 50, "rtol": 1e-8} for d in (1, 2)]})
    _check(out)
    for r in out["runs"]:
        assert r["est"] == 2 and r["lmax"] == pytest.approx(1.65) and r["code"] == 0, r
    out = _run({"matrix": "rmat", "runs": [{"degree": 2, "maxits": 100, "rtol": 1e-8, "bones": 1}]})
    _check(out)
    assert out["runs"][0]["est"] == 10


def test_edges(simlib):
    """maxits reached gives NOT_CONVERGED; maxits = 0 returns x0 bitwise; r0 = 0 runs no iteration (under a
    tolerance or not); tolerances off run exactly maxits."""
    out = _run({"matrix": "7pt", "runs": [
        {"degree": 2, "maxits": 5, "rtol": 1e-10, "x0": 1},
        {"degree": 2, "maxits": 0, "rtol": 1e-8, "x0": 1},
        {"degree": 2, "maxits": 50, "atol": 1e-8, "bzero": True},
        {"degree": 0, "maxits": 50, "bzero": True},
        {"degree": 1, "maxits": 9, "warmup": 2, "x0": 1}]})
    _check(out)
    short, zero, bzero, bzero_off, off = out["runs"]
    assert short["code"] == NOT_CONVERGED and short["its"] == 5 and short["ref_stop"] == "maxits"
    assert zero["code"] == NOT_CONVERGED and zero["its"] == 0 and zero["x_is_x0"] and zero["est"] == 0
    assert bzero["code"] == 0 and bzero["its"] == 0 and bzero["x_is_x0"]
    assert bzero_off["code"] == 0 and bzero_off["its"] == 0 and bzero_off["rnrm2"] == 0
    assert off["code"] == 0 and off["its"] == 9


def test_rejected_calls(simlib):
    """degree -1 or 17, lmin >= lmax (given or estimated), NaN, infinite or negative bounds: INVALID_VALUE
    with x0 left alone; degree 0 ignores the interval."""
    bad = [{"degree": -1}, {"degree": 17}, {"degree": 2, "lmin": 1.0, "lmax": 1.0}, {"degree": 2, "lmin": 2.0, "lmax": 1.0},
           {"degree": 2, "lmin": float("nan")}, {"degree": 2, "lmax": float("inf")}, {"degree": 1, "lmin": -0.1},
           {"degree": 1, "lmax": -1.0}, {"degree": 2, "lmin": 50.0}]
    runs = [dict(b, maxits=20, rtol=1e-8, x0=1) for b in bad] + [{"degree": 0, "lmin": -1.0, "maxits": 100, "rtol": 1e-8}]
    out = _run({"matrix": "7pt", "runs": runs})
    _check(out)
    assert all(r["code"] == INVALID_VALUE for r in out["runs"][:-1])
    assert out["runs"][-1]["code"] == 0


def test_nonpositive_diagonal(simlib):
    """dsymv_init with eps = -7 leaves the 7-pt stencil's diagonal at -1: INVALID_VALUE at set-up."""
    out = _run({"matrix": "7pt", "eps": -7.0, "runs": [{"degree": d, "maxits": 20, "rtol": 1e-8, "x0": 1} for d in (0, 2)]})
    _check(out)
    assert all(r["code"] == INVALID_VALUE and r["x_is_x0"] for r in out["runs"])


def test_breakdown(simlib):
    """degree 1 over [0.3, 1.0] on the 7-pt stencil (lambda_max(D^-1 A) = 1.97 > a + b): M^-1 is indefinite
    and (r, z) <= 0 ends the solve after one iteration; degree 2 over the same interval still converges (in 52
    iterations, as many as Jacobi PCG: its polynomial is positive on the spectrum but poorly fitted, and x
    agrees to 1e-10 only)."""
    out = _run({"matrix": "7pt", "runs": [{"degree": 1, "lmin": 0.3, "lmax": 1.0, "maxits": 300, "rtol": 1e-10},
                                          {"degree": 1, "lmin": 0.3, "lmax": 1.0, "maxits": 300},
                                          {"degree": 2, "lmin": 0.3, "lmax": 1.0, "maxits": 300, "rtol": 1e-10,
                                           "xtol": 1e-10}]})
    _check(out)
    a, b, c = out["runs"]
    assert a["ref_stop"] == "breakdown" and a["its"] == 1 and a["breakdown"] == 1 and a["code"] == NOT_CONVERGED
    assert b["ref_stop"] == "breakdown" and b["code"] == 0
    assert c["ref_stop"] == "tol" and c["breakdown"] == 0 and c["code"] == 0


def test_alternating_with_other_solves(simlib):
    """solve_chebyshev (degrees 0, 2, 5), solvempi and solve_mixed in turn on one solver: every call gives what it
    gives alone; a solvempi afterwards matches one on a fresh solver bitwise."""
    out = _run({"matrix": "27pt", "alternate": 1})
    alt = out["alternate"]
    first = {}
    for s in alt["steps"]:
        assert s["code"] == 0, s["kind"]
        assert s["deg"] == (int(s["kind"][4:]) if s["kind"].startswith("cheb") else 0)
        first.setdefault(s["kind"], s)
        assert first[s["kind"]]["its"] == s["its"] and first[s["kind"]]["x"] == s["x"], s["kind"]
    xc, xs = np.array(first["cheb2"]["x"]), np.array(first["single"]["x"])
    assert np.abs(xc - xs).max() < 1e-6 * np.abs(xs).max()
    s = alt["single_after"]
    assert s["same_x"] and s["its"][0] == s["its"][1]


def test_partitioned_matrix_is_refused(simlib):
    out = _run({"matrix": "7pt", "partitioned": 1})
    assert out["partitioned_code"] == NOT_SUPPORTED


def test_plain_hostsim_build_refuses():
    """Without the Chebyshev launchers (the plain host-logic stand-in) the call is refused."""
    p = subprocess.run(["make", "-C", SIM], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
    code = ("import sys; sys.path.insert(0, %r)\n"
            "import acg_b200.api as api; api._LIBPATH = %r\n"
            "import acg_b200 as ab; from acg_b200 import matgen as mg\n"
            "n, r, c, v = mg.laplace3d_7pt(5); A = ab.SymCsrMatrix.init_real_double(n, r, c, v).dsymv_init(0.0)\n"
            "cg = ab.SolverCuda(A); b = A.vector(); b.x[:] = 1.0; x = A.vector()\n"
            "try:\n    cg.solve_chebyshev(b, x); print('ran')\n"
            "except ab.AcgError as e:\n    print('code', e.code)\n"
            "cg.free()\n") % (ROOT, os.path.join(SIM, "libacgb200_hostsim.so"))
    p = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stderr[-2000:]
    assert p.stdout.strip().splitlines()[-1] == f"code {NOT_SUPPORTED}"
