"""Host logic of acgsolvercuda_solve_mixed (CG with float vectors and reliable updates) on the device
stand-in of tests/hostsim, against the restatement of tests/mixedref.py: equal iteration and
reliable-update counts and codes, x within 1e-12 relative, and rnrm2 the fp64 residual of the x returned
(against the exact residual of tests/exactref.py).
Covers nonzero x0, rtol and atol stopping, maxits reached, maxits = 0 returning x0 bitwise, b = 0, warm-up
0 and 2, (p, A p) = 0, rejected calls, and solvempi, solve_multi, solve_shifted, solve_minres and
solve_mixed alternating on one solver.  The stand-in keeps the kernels' roundings, scalar rules and slot
discipline; the kernels themselves are checked on the H100 by test_gpu_mixed.py."""
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
    p = subprocess.run(["make", "-C", SIM, "-f", "Makefile.mixed"], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
    assert "warning" not in p.stderr
    return os.path.join(SIM, "libacgb200_hostsim_mixed.so")


def _run(spec):
    p = subprocess.run([sys.executable, os.path.join(SIM, "run_mixed_sim.py"), json.dumps(spec)], capture_output=True,
                       text=True, timeout=900, env=dict(os.environ, OMP_NUM_THREADS="2"))
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-3000:]
    return json.loads(p.stdout.strip().splitlines()[-1])


def _check(out):
    for i, r in enumerate(out["runs"]):
        assert r["nsolves"] == i + 1
        assert r["code"] == r["ref_code"], r
        assert r["its"] == r["ref_its"], r
        assert r["updates"] == r["ref_updates"], r
        assert r["xerr"] < 1e-12, r
        assert r["bnrm2"] == pytest.approx(r["ref_bnrm2"], rel=1e-13, abs=1e-300)
        assert r["r0nrm2"] == pytest.approx(r["ref_r0nrm2"], rel=1e-13, abs=1e-300)
        # the fp64 residual of the x returned, to the rounding of b - A x against the exact one
        assert r["rnrm2"] == pytest.approx(r["true_rnrm2"], rel=1e-8, abs=1e-13 * max(r["bnrm2"], r["r0nrm2"])), r
        assert r["report_lines"] > 0
        if r["code"] == 0 and r["tol"] > 0:
            assert r["true_rnrm2"] < r["tol"], r


@pytest.mark.parametrize("matrix", ["7pt", "27pt"])
def test_against_restatement(matrix, simlib):
    """rtol from x0 = 0 with warm-up 0; atol from a nonzero x0 with warm-up 2; rtol and atol together."""
    out = _run({"matrix": matrix, "runs": [
        {"maxits": 600, "rtol": 1e-10},
        {"maxits": 600, "atol": 1e-8, "x0": 1, "bscale": 10.0, "warmup": 2},
        {"maxits": 600, "atol": 1e-9, "rtol": 1e-11, "x0": 1}]})
    _check(out)
    assert all(r["ref_stop"] == "tol" and r["code"] == 0 and r["updates"] >= 1 for r in out["runs"])


def test_maxits_zero_rhs_and_tolerances_off(simlib):
    """maxits reached gives NOT_CONVERGED with rnrm2 the residual of the folded x; maxits = 0 returns x0
    bitwise; b = 0 runs no iteration, under a tolerance or not; tolerances off run exactly maxits."""
    out = _run({"matrix": "7pt", "runs": [
        {"maxits": 12, "rtol": 1e-10, "x0": 1},
        {"maxits": 0, "rtol": 1e-8, "x0": 1},
        {"maxits": 50, "atol": 1e-8, "bzero": True},
        {"maxits": 50, "bzero": True},
        {"maxits": 9, "warmup": 2, "x0": 1}], "errors": 1})
    _check(out)
    short, zero, bzero, bzero_off, off = out["runs"]
    assert short["code"] == NOT_CONVERGED and short["its"] == 12 and short["ref_stop"] == "maxits"
    assert zero["code"] == NOT_CONVERGED and zero["its"] == 0 and zero["x_is_x0"]
    assert bzero["code"] == 0 and bzero["its"] == 0 and bzero["x_is_x0"]
    assert bzero_off["code"] == 0 and bzero_off["its"] == 0 and bzero_off["x_is_x0"] and bzero_off["rnrm2"] == 0
    assert off["code"] == 0 and off["its"] == 9
    assert out["negative_maxits"] == INVALID_VALUE


def test_zero_curvature(simlib):
    """A diagonal matrix: b = 1.5 e_i with a power-of-two entry d_i converges exactly in one iteration; at the
    zero entry (p, A p) = 0 ends the solve before the update (0 iterations, x0 returned, NOT_CONVERGED under
    a tolerance)."""
    runs = [{"maxits": 20, "unit": i, "rtol": 1e-10} for i in (2, 5, 6)]
    runs += [{"maxits": 20, "unit": 8, "rtol": 1e-8}, {"maxits": 20, "unit": 8}]
    out = _run({"matrix": "diag", "runs": runs})
    _check(out)
    for r in out["runs"][:-2]:
        assert r["its"] == 1 and r["code"] == 0, r
    for r in out["runs"][-2:]:
        assert r["its"] == 0 and r["ref_stop"] == "breakdown" and r["x_is_x0"], r
    assert out["runs"][-2]["code"] == NOT_CONVERGED and out["runs"][-1]["code"] == 0


def test_alternating_with_other_solves(simlib):
    """solve_mixed, solvempi, solve_multi, solve_shifted and solve_minres in turn on one solver: every call
    gives what it gives alone (the captured loops are replayed only for their own kind) and info() counts
    the reliable updates of the last solve only; a solvempi afterwards matches one on a fresh solver
    bitwise."""
    out = _run({"matrix": "27pt", "alternate": 1})
    alt = out["alternate"]
    first = {}
    for s in alt["steps"]:
        assert s["code"] == 0, s["kind"]
        if s["kind"] == "mixed":
            assert s["updates"] >= 1, s["kind"]
        else:
            assert s["updates"] == 0, s["kind"]
        first.setdefault(s["kind"], s)
        assert first[s["kind"]]["its"] == s["its"], s["kind"]
        assert first[s["kind"]]["x"] == s["x"], s["kind"]
    xm, xc = np.array(first["mixed"]["x"]), np.array(first["single"]["x"])
    assert np.abs(xm - xc).max() < 1e-6 * np.abs(xc).max()
    s = alt["single_after"]
    assert s["same_x"] and s["its"][0] == s["its"][1] and s["rnrm2"][0] == s["rnrm2"][1]


def test_partitioned_matrix_is_refused(simlib):
    out = _run({"matrix": "7pt", "partitioned": 1})
    assert out["partitioned_code"] == NOT_SUPPORTED


def test_plain_hostsim_build_refuses():
    """Without the mixed-precision launchers (the plain host-logic stand-in) the call is refused."""
    p = subprocess.run(["make", "-C", SIM], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
    code = ("import sys; sys.path.insert(0, %r)\n"
            "import acg_b200.api as api; api._LIBPATH = %r\n"
            "import acg_b200 as ab; from acg_b200 import matgen as mg\n"
            "n, r, c, v = mg.laplace3d_7pt(5); A = ab.SymCsrMatrix.init_real_double(n, r, c, v).dsymv_init(0.0)\n"
            "cg = ab.SolverCuda(A); b = A.vector(); b.x[:] = 1.0; x = A.vector()\n"
            "try:\n    cg.solve_mixed(b, x); print('ran')\n"
            "except ab.AcgError as e:\n    print('code', e.code)\n"
            "cg.free()\n") % (ROOT, os.path.join(SIM, "libacgb200_hostsim.so"))
    p = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stderr[-2000:]
    assert p.stdout.strip().splitlines()[-1] == f"code {NOT_SUPPORTED}"
