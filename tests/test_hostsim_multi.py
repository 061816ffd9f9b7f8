"""Host logic of acgsolvercuda_solve_multi (several right-hand sides, one matrix pass per iteration for
all of them) on the device stand-in of tests/hostsim, column by column against the oracle's classic
CG on that column alone: padding of nrhs to the block width K, per-column tolerances and active
masks, columns converging at different iterations or at r0, non-zero initial guesses, warm-up,
maxits = 0 and maxits reached, rejected calls, graph re-capture when K changes on one solver, and the
single-vector solver on the same solver afterwards.  The stand-in computes the products with the
kernels' index arithmetic and per-column summation order; the kernels themselves are checked on the
H100 by test_gpu_multi_rhs.py."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIM = os.path.join(ROOT, "tests", "hostsim")
NOT_CONVERGED, INVALID_VALUE, NOT_SUPPORTED = 39, 29, 26


@pytest.fixture(scope="module")
def simlib():
    p = subprocess.run(["make", "-C", SIM, "-f", "Makefile.multi"], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
    assert "warning" not in p.stderr
    return os.path.join(SIM, "libacgb200_hostsim_multi.so")


def _run(spec):
    p = subprocess.run([sys.executable, os.path.join(SIM, "run_multi_sim.py"), json.dumps(spec)], capture_output=True,
                       text=True, timeout=900, env=dict(os.environ, OMP_NUM_THREADS="2"))
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-3000:]
    return json.loads(p.stdout.strip().splitlines()[-1])


def _check(out, xtol=1e-12):
    for i, r in enumerate(out["runs"]):
        assert r["nsolves"] == i + 1
        assert r["code"] == r["ref_code"], r
        assert r["its"] == r["ref_its"], r             # the loop runs as long as the slowest column
        assert r["frobenius_ok"], r
        for c in r["cols"]:
            assert c["its"] == c["ref_its"], (r["run"], c)
            assert c["converged"] == (c["ref_status"] == 0) or r["run"].get("atol", 0) == r["run"].get("rtol", 0) == 0, c
            assert c["xerr"] < xtol, (r["run"], c)
            assert c["r0nrm2"] == pytest.approx(c["ref_r0nrm2"], rel=1e-13, abs=1e-300)
            assert c["bnrm2"] == pytest.approx(c["ref_bnrm2"], rel=1e-13, abs=1e-300)
            assert c["rnrm2"] == pytest.approx(c["ref_rnrm2"], rel=1e-9, abs=1e-12 * c["ref_r0nrm2"]), c


@pytest.mark.parametrize("matrix", ["7pt", "27pt"])
@pytest.mark.parametrize("nrhs", [1, 2, 3, 4, 5, 6, 7, 8])
def test_every_column_is_its_own_classic_cg(matrix, nrhs, simlib):
    """nrhs = 1..8 (3, 5, 6, 7 padded to K = 4 or 8 with inactive columns): relative tolerance, then an
    absolute one with right-hand sides scaled by 10^j so that the columns stop at different
    iterations, from non-zero initial guesses, with warm-up 0 and 2."""
    out = _run({"matrix": matrix, "runs": [
        {"nrhs": nrhs, "maxits": 200, "rtol": 1e-9},
        {"nrhs": nrhs, "maxits": 200, "atol": 1e-5, "scale": 10.0, "x0": "random", "warmup": 2}]})
    _check(out)
    assert out["errors"] == {"nrhs0": INVALID_VALUE, "nrhs9": INVALID_VALUE}
    if nrhs > 1:
        its = [c["its"] for c in out["runs"][1]["cols"]]
        assert len(set(its)) > 1                       # the scaled columns did stop at different iterations


def test_converged_at_r0_maxits_and_not_converged(simlib):
    """A zero column under an absolute tolerance is converged at r0 (0 iterations, x untouched) while
    the others iterate; maxits = 0 returns X bitwise; maxits reached gives NOT_CONVERGED; tolerances
    off run exactly maxits and return success."""
    out = _run({"matrix": "7pt", "runs": [
        {"nrhs": 4, "maxits": 200, "atol": 1e-6, "zero_col": 2, "x0": "random", "warmup": 2},
        {"nrhs": 3, "maxits": 0, "x0": "random", "rtol": 1e-9},
        {"nrhs": 6, "maxits": 0, "x0": "random"},
        {"nrhs": 5, "maxits": 7, "rtol": 1e-9, "x0": "random"},
        {"nrhs": 2, "maxits": 9}]})
    _check(out)
    r0, z1, z2, short, off = out["runs"]
    assert r0["code"] == 0 and r0["cols"][2]["its"] == 0 and r0["cols"][2]["converged"] == 1
    assert z1["x_bitwise_x0"] and z2["x_bitwise_x0"] and z1["its"] == z2["its"] == 0
    assert z1["code"] == NOT_CONVERGED and z2["code"] == 0
    assert short["code"] == NOT_CONVERGED and short["its"] == 7
    assert off["code"] == 0 and off["its"] == 9 and all(c["its"] == 9 for c in off["cols"])


def test_block_width_changes_and_single_solve_afterwards(simlib):
    """K alternating on one solver (1, 8, 2, 8, 4: the captured loop is replayed only for the width it
    was captured with, and a wider request replaces the blocks); then a single-vector classic solve on
    the same solver matches one on a fresh solver bitwise."""
    runs = [{"nrhs": k, "maxits": 60, "rtol": 1e-8} for k in (1, 8, 2, 7, 4, 3)]
    out = _run({"matrix": "27pt", "runs": runs, "single_after": 1})
    _check(out)
    s = out["single_after"]
    assert s["same_x"] and s["its"][0] == s["its"][1] and s["rnrm2"][0] == s["rnrm2"][1]


def test_products_and_power_law_rows(simlib):
    """spmm_mode in all three modes (every row written exactly once: the stand-in poisons rows the plan
    misses or covers twice), on a stencil (slices + chunks) and on power-law rows (chunks only, eight
    lanes per row), and a short solve on the latter."""
    for matrix in ("27pt", "rmat"):
        spec = {"matrix": matrix, "spmm": [1, 2, 3, 8]}
        if matrix == "rmat":
            spec["runs"] = [{"nrhs": 3, "maxits": 8, "x0": "random"}]
        out = _run(spec)
        _check(out, xtol=1e-12 if matrix == "27pt" else 1e-8)     # power-law rows: 8-lane sums, another order
        for s in out["spmm"]:
            assert not s["nan"] and s["yerr"] < 1e-13 and s["doterr"] < 1e-12, s


def test_partitioned_matrix_is_refused(simlib):
    out = _run({"matrix": "7pt", "partitioned": 1})
    assert out["partitioned_code"] == NOT_SUPPORTED
    assert out["errors"] == {"nrhs0": INVALID_VALUE, "nrhs9": INVALID_VALUE}
