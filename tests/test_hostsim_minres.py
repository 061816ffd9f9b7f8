"""Host logic of acgsolvercuda_solve_minres (MINRES for symmetric, possibly indefinite A) on the device
stand-in of tests/hostsim, against the restatement of tests/minresref.py: equal iteration counts and codes,
x within 1e-10 relative, phi-bar equal to the restatement's, and the exact true residual (tests/exactref.py)
of every converged solve below 2 tol.  Covers positive definite and indefinite stencils (the number of
negative eigenvalues from the closed-form spectrum), nonzero x0, rtol and atol stopping, maxits reached,
maxits = 0 returning x0 bitwise, b = 0, both breakdowns, warm-up 0 and 2, rejected calls, and solvempi,
solve_shifted and solve_minres alternating on one solver.  The stand-in keeps the kernels' scalar
recurrence and slot discipline; the kernels themselves are checked on the H100 by test_gpu_minres.py."""
import json
import os
import subprocess
import sys

import pytest

from minresref import indefinite_shift, stencil_eigenvalues

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIM = os.path.join(ROOT, "tests", "hostsim")
NOT_CONVERGED, INVALID_VALUE, NOT_SUPPORTED = 39, 29, 26
BOX = {"7pt": (7, (11, 11, 11)), "27pt": (27, (9, 8, 10))}      # the matrices of run_minres_sim.py


@pytest.fixture(scope="module")
def simlib():
    p = subprocess.run(["make", "-C", SIM, "-f", "Makefile.minres"], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
    assert "warning" not in p.stderr
    return os.path.join(SIM, "libacgb200_hostsim_minres.so")


def _run(spec):
    p = subprocess.run([sys.executable, os.path.join(SIM, "run_minres_sim.py"), json.dumps(spec)], capture_output=True,
                       text=True, timeout=900, env=dict(os.environ, OMP_NUM_THREADS="2"))
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-3000:]
    return json.loads(p.stdout.strip().splitlines()[-1])


def _check(out):
    for i, r in enumerate(out["runs"]):
        assert r["nsolves"] == i + 1
        assert r["code"] == r["ref_code"], r
        assert r["its"] == r["ref_its"], r
        assert r["xerr"] < 1e-10, r
        assert r["bnrm2"] == pytest.approx(r["ref_bnrm2"], rel=1e-13, abs=1e-300)
        assert r["r0nrm2"] == pytest.approx(r["ref_r0nrm2"], rel=1e-13, abs=1e-300)
        assert r["rnrm2"] == pytest.approx(r["ref_rnrm2"], rel=1e-8, abs=1e-11 * r["ref_bnrm2"]), r
        assert r["report_lines"] > 0
        if r["code"] == 0 and r["tol"] > 0:
            assert r["true_rnrm2"] < 2 * r["tol"], r


def _eps(matrix, nneg):
    """dsymv_init's eps for nneg negative eigenvalues (0: the matrix itself, positive definite)."""
    if nneg == 0:
        return 0.0
    kind, box = BOX[matrix]
    ev = stencil_eigenvalues(kind, *box)
    sigma = indefinite_shift(ev, nneg)
    assert int((ev < sigma).sum()) == nneg
    return -sigma


@pytest.mark.parametrize("matrix,nneg", [("7pt", 0), ("7pt", 1), ("7pt", 4), ("27pt", 0), ("27pt", 1), ("27pt", 3)])
def test_against_restatement(matrix, nneg, simlib):
    """rtol from x0 = 0 with warm-up 0; atol from a nonzero x0 with warm-up 2; rtol and atol together.  The
    tolerances are tight enough (about 1e-10 relative) that x is pinned by the solution itself: at looser
    ones two roundings of an indefinite Lanczos process can part for a while (loss of orthogonality), and x
    then agrees only to about cond(A) tol."""
    out = _run({"matrix": matrix, "eps": _eps(matrix, nneg), "runs": [
        {"maxits": 600, "rtol": 1e-10},
        {"maxits": 600, "atol": 1e-8, "x0": 1, "bscale": 10.0, "warmup": 2},
        {"maxits": 600, "atol": 1e-9, "rtol": 1e-11, "x0": 1}]})
    _check(out)
    assert all(r["ref_stop"] == "tol" and r["code"] == 0 for r in out["runs"])


def test_maxits_zero_rhs_and_tolerances_off(simlib):
    """maxits reached gives NOT_CONVERGED; maxits = 0 returns x0 bitwise (NOT_CONVERGED under a tolerance);
    b = 0 under an absolute tolerance is converged at r0 (0 iterations); b = 0 without a tolerance still
    runs no iteration (beta_1 = 0); tolerances off run exactly maxits and return success."""
    out = _run({"matrix": "7pt", "eps": _eps("7pt", 1), "runs": [
        {"maxits": 12, "rtol": 1e-10},
        {"maxits": 0, "rtol": 1e-8, "x0": 1},
        {"maxits": 50, "atol": 1e-8, "bzero": True},
        {"maxits": 50, "bzero": True},
        {"maxits": 9, "warmup": 2, "x0": 1}], "errors": 1})
    _check(out)
    short, zero, bzero, bzero_off, off = out["runs"]
    assert short["code"] == NOT_CONVERGED and short["its"] == 12
    assert zero["code"] == NOT_CONVERGED and zero["its"] == 0 and zero["x_is_x0"]
    assert bzero["code"] == 0 and bzero["its"] == 0 and bzero["x_is_x0"]
    assert bzero_off["code"] == 0 and bzero_off["its"] == 0 and bzero_off["x_is_x0"] and bzero_off["rnrm2"] == 0
    assert off["code"] == 0 and off["its"] == 9
    assert out["negative_maxits"] == INVALID_VALUE


def test_breakdown(simlib):
    """A diagonal matrix with b = 1.5 e_i: beta_2 = 0 ends the solve after one iteration with x = b_i / d_i
    e_i, tolerance or not; at the zero diagonal entry gamma_1 = 0 ends it before the update (0 iterations,
    x0 returned, NOT_CONVERGED under a tolerance)."""
    runs = [{"maxits": 20, "unit": i, "rtol": rt} for i in (0, 1, 3, 6, 10) for rt in (0.0, 1e-10)]
    runs += [{"maxits": 20, "unit": 8, "rtol": 1e-8}, {"maxits": 20, "unit": 8}]
    out = _run({"matrix": "diag", "runs": runs})
    _check(out)
    for r in out["runs"][:-2]:
        assert r["its"] == 1 and r["ref_stop"] == "breakdown" and r["code"] == 0 and r["rnrm2"] == 0.0, r
        assert r["xerr"] < 1e-15
    g_tol, g_off = out["runs"][-2:]
    for r in (g_tol, g_off):
        assert r["its"] == 0 and r["ref_stop"] == "gamma" and r["x_is_x0"], r
    assert g_tol["code"] == NOT_CONVERGED and g_off["code"] == 0


def test_alternating_with_other_solves(simlib):
    """solve_minres, solvempi and solve_shifted in turn on one solver: every call gives what it gives alone
    (the captured loops are replayed only for their own kind); on this positive definite matrix MINRES
    and CG reach the same solution; a solvempi afterwards matches one on a fresh solver bitwise."""
    import numpy as np
    out = _run({"matrix": "27pt", "alternate": 1})
    alt = out["alternate"]
    first = {}
    for s in alt["steps"]:
        assert s["code"] == 0, s["kind"]
        first.setdefault(s["kind"], s)
        assert first[s["kind"]]["its"] == s["its"], s["kind"]
        assert first[s["kind"]]["x"] == s["x"], s["kind"]          # bitwise: the same loop on the same data
    xm, xc = np.array(first["minres"]["x"]), np.array(first["single"]["x"])
    assert np.abs(xm - xc).max() < 1e-7 * np.abs(xc).max()
    s = alt["single_after"]
    assert s["same_x"] and s["its"][0] == s["its"][1] and s["rnrm2"][0] == s["rnrm2"][1]


def test_partitioned_matrix_is_refused(simlib):
    out = _run({"matrix": "7pt", "partitioned": 1})
    assert out["partitioned_code"] == NOT_SUPPORTED


def test_plain_hostsim_build_refuses(tmp_path):
    """Without the MINRES launchers (the plain host-logic stand-in) the call is refused, nothing else runs."""
    p = subprocess.run(["make", "-C", SIM], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
    code = ("import sys; sys.path.insert(0, %r)\n"
            "import acg_b200.api as api; api._LIBPATH = %r\n"
            "import acg_b200 as ab; from acg_b200 import matgen as mg\n"
            "n, r, c, v = mg.laplace3d_7pt(5); A = ab.SymCsrMatrix.init_real_double(n, r, c, v).dsymv_init(0.0)\n"
            "cg = ab.SolverCuda(A); b = A.vector(); b.x[:] = 1.0; x = A.vector()\n"
            "try:\n    cg.solve_minres(b, x); print('ran')\n"
            "except ab.AcgError as e:\n    print('code', e.code)\n"
            "cg.free()\n") % (ROOT, os.path.join(SIM, "libacgb200_hostsim.so"))
    p = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stderr[-2000:]
    assert p.stdout.strip().splitlines()[-1] == f"code {NOT_SUPPORTED}"
