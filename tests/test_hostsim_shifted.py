"""Host logic of acgsolvercuda_solve_shifted (multi-shift CG: (A + sigma_j I) x_j = b for several shifts
in one Krylov space) on the device stand-in of tests/hostsim, shift by shift against the oracle's
classic CG on the matrix assembled by dsymv_init at eps = sigma_j from x0 = 0: equal iteration counts,
x within 1e-10 relative, equal codes, and the true residual of every converged shift (exact, by
tests/exactref.py) below 2 tol.  Covers padding of the shift count to the block width, sigma = 0
present and absent, shifts that stop at different iterations under rtol and atol, maxits reached,
maxits = 0, b = 0, warm-up, rejected calls, and solve_multi / solve_shifted / solvempi alternating on
one solver.  The stand-in keeps the kernels' scalar recurrence and index arithmetic; the kernels
themselves are checked on the H100 by test_gpu_shifted.py."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIM = os.path.join(ROOT, "tests", "hostsim")
NOT_CONVERGED, INVALID_VALUE, NOT_SUPPORTED = 39, 29, 26

WITH_ZERO = [0.0, 1.0, 0.1, 0.01, 1e-3, 0.3, 0.03, 3e-3]
WITHOUT_ZERO = [1e-3, 1.0, 0.1, 0.01, 0.3, 0.03, 3e-3, 3.0]


@pytest.fixture(scope="module")
def simlib():
    p = subprocess.run(["make", "-C", SIM, "-f", "Makefile.shifted"], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
    assert "warning" not in p.stderr
    return os.path.join(SIM, "libacgb200_hostsim_shifted.so")


def _run(spec):
    p = subprocess.run([sys.executable, os.path.join(SIM, "run_shifted_sim.py"), json.dumps(spec)], capture_output=True,
                       text=True, timeout=900, env=dict(os.environ, OMP_NUM_THREADS="2"))
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-3000:]
    return json.loads(p.stdout.strip().splitlines()[-1])


def _check(out):
    for i, r in enumerate(out["runs"]):
        assert r["nsolves"] == i + 1
        assert r["code"] == r["ref_code"], r
        assert r["its"] == r["ref_its"], r             # the loop runs as long as the slowest shift
        assert r["frobenius_ok"], r
        for c in r["cols"]:
            assert c["its"] == c["ref_its"], (r["run"], c)
            assert c["converged"] == (c["ref_status"] == 0) or r["run"].get("atol", 0) == r["run"].get("rtol", 0) == 0, c
            assert c["xerr"] < 1e-10, (r["run"], c)
            assert c["r0nrm2"] == c["bnrm2"] == pytest.approx(c["ref_bnrm2"], rel=1e-13, abs=1e-300)
            assert c["rnrm2"] == pytest.approx(c["ref_rnrm2"], rel=1e-8, abs=1e-12 * c["ref_bnrm2"]), c
            if c["converged"] and c["tol"] > 0:
                assert c["true_rnrm2"] < 2 * c["tol"], c


@pytest.mark.parametrize("matrix", ["7pt", "27pt"])
@pytest.mark.parametrize("nshifts", [1, 2, 3, 4, 5, 6, 7, 8])
def test_every_shift_is_its_own_classic_cg(matrix, nshifts, simlib):
    """nshifts = 1..8 (3, 5, 6, 7 padded to K = 4 or 8 with inactive columns), sigma = 0 present under a
    relative tolerance and absent under an absolute one (with warm-up 2); the 7-point matrix has an
    odd number of rows (the kernel's tail row)."""
    out = _run({"matrix": matrix, "runs": [
        {"shifts": WITH_ZERO[:nshifts], "maxits": 300, "rtol": 1e-10},
        {"shifts": WITHOUT_ZERO[:nshifts], "maxits": 300, "atol": 1e-6, "bscale": 10.0, "warmup": 2}]})
    _check(out)
    assert out["errors"] == {"nshifts0": INVALID_VALUE, "nshifts9": INVALID_VALUE, "negative": INVALID_VALUE,
                             "nan": INVALID_VALUE, "inf": INVALID_VALUE}
    if nshifts > 1:
        for run in out["runs"]:
            assert len({c["its"] for c in run["cols"]}) > 1      # the shifts did stop at different iterations


def test_maxits_zero_rhs_and_tolerances_off(simlib):
    """maxits reached gives NOT_CONVERGED; maxits = 0 returns X = 0 (NOT_CONVERGED under a tolerance);
    b = 0 under an absolute tolerance is converged at r0 (0 iterations, success); tolerances off run
    exactly maxits and return success."""
    out = _run({"matrix": "7pt", "runs": [
        {"shifts": [0.0, 0.1, 1.0], "maxits": 12, "rtol": 1e-10},
        {"shifts": [0.0, 0.5], "maxits": 0, "rtol": 1e-8},
        {"shifts": [0.2, 0.0, 2.0, 0.02, 0.5], "maxits": 50, "atol": 1e-8, "bzero": True},
        {"shifts": [0.0, 0.1, 1.0, 0.01], "maxits": 9, "warmup": 2}]})
    _check(out)
    short, zero, bzero, off = out["runs"]
    assert short["code"] == NOT_CONVERGED and short["its"] == 12
    assert zero["code"] == NOT_CONVERGED and zero["its"] == 0 and zero["x_zero"]
    assert bzero["code"] == 0 and bzero["its"] == 0 and bzero["x_zero"]
    assert all(c["its"] == 0 and c["converged"] == 1 for c in bzero["cols"])
    assert off["code"] == 0 and off["its"] == 9 and all(c["its"] == 9 for c in off["cols"])


def test_alternating_with_other_solves(simlib):
    """solve_multi, solve_shifted (block widths 1 to 8) and solvempi in turn on one solver: every call
    gives what it gives alone (the captured loops are replayed only for their own kind and width); the
    sigma = 0 shift runs the single-vector classic recurrence; a single-vector solve afterwards matches
    one on a fresh solver bitwise."""
    out = _run({"matrix": "27pt", "alternate": 1})
    alt = out["alternate"]
    first = {}
    for s in alt["steps"]:
        assert s["code"] == 0, s
        key = (s["kind"], s["k"])
        if s["kind"] == "shifted":
            # the same b and shift list prefix each time: each shift's iteration count never changes
            for j, it in enumerate(s["its"]):
                first.setdefault(("shift", j), it)
                assert first[("shift", j)] == it, (s, j)
        first.setdefault(key, s["its"])
        assert first[key] == s["its"], s
    single = [s["its"][0] for s in alt["steps"] if s["kind"] == "single"]
    assert first[("shift", 0)] == single[0]           # sigma = 0 first in the list: the seed's own count
    assert alt["sigma0"]["its"][0] == alt["sigma0"]["its"][1] and alt["sigma0"]["xerr"] < 1e-12
    s = alt["single_after"]
    assert s["same_x"] and s["its"][0] == s["its"][1] and s["rnrm2"][0] == s["rnrm2"][1]


def test_partitioned_matrix_is_refused(simlib):
    out = _run({"matrix": "7pt", "partitioned": 1})
    assert out["partitioned_code"] == NOT_SUPPORTED
    assert out["errors"]["nshifts0"] == INVALID_VALUE


def test_plain_hostsim_build_refuses(tmp_path):
    """Without the shift launchers (the plain host-logic stand-in) the call is refused, nothing else runs."""
    p = subprocess.run(["make", "-C", SIM], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
    code = ("import sys, numpy as np; sys.path.insert(0, %r)\n"
            "import acg_b200.api as api; api._LIBPATH = %r\n"
            "import acg_b200 as ab; from acg_b200 import matgen as mg\n"
            "n, r, c, v = mg.laplace3d_7pt(5); A = ab.SymCsrMatrix.init_real_double(n, r, c, v).dsymv_init(0.0)\n"
            "cg = ab.SolverCuda(A)\n"
            "try:\n    cg.solve_shifted(np.ones(n), [0.0, 0.1]); print('ran')\n"
            "except ab.AcgError as e:\n    print('code', e.code)\n"
            "cg.free()\n") % (ROOT, os.path.join(SIM, "libacgb200_hostsim.so"))
    p = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stderr[-2000:]
    assert p.stdout.strip().splitlines()[-1] == f"code {NOT_SUPPORTED}"
