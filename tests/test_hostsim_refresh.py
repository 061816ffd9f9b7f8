"""Host logic of acgsolvercuda_update_values on the device stand-in of tests/hostsim (which has no mirrored
diagonals; those are checked on the H100 by test_gpu_refresh.py): refused calls leave the solver bitwise as it
was; after a refresh every product and solve entry point -- run once before it, so that graphs, Chebyshev's D^-1
and the row chunks are cached -- gives bitwise what a solver built fresh on the new values gives, from full
storage or from the packed triangle; three refreshes alternating two value sets; Jacobi PCG on R-MAT with the
diagonal doubled; and a 2-rank partitioned classic solve after both ranks refreshed."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIM = os.path.join(ROOT, "tests", "hostsim")
INVALID_VALUE, NOT_SUPPORTED = 29, 26


@pytest.fixture(scope="module")
def simlib():
    p = subprocess.run(["make", "-C", SIM, "-f", "Makefile.refresh"], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
    assert "warning" not in p.stderr
    return os.path.join(SIM, "libacgb200_hostsim_refresh.so")


def _run(spec):
    p = subprocess.run([sys.executable, os.path.join(SIM, "run_refresh_sim.py"), json.dumps(spec)], capture_output=True,
                       text=True, timeout=900, env=dict(os.environ, OMP_NUM_THREADS="2"))
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-3000:]
    return json.loads(p.stdout.strip().splitlines()[-1])


def test_refusals_leave_the_solver_unchanged(simlib):
    """A moved column with equal counts, a different entry count (from full storage and from the packed
    triangle), a different partition and a freed solver: ACG_ERR_INVALID_VALUE, and the solver's struct, device
    arrays and results are bitwise those from before."""
    out = _run({"mode": "refusals"})
    assert out["codes"] == {k: INVALID_VALUE for k in ("moved-column", "moved-column-packed", "entry-count",
                                                        "entry-count-packed", "partition", "freed")}


@pytest.mark.parametrize("matrix,init_full,full", [("27pt", True, True), ("27pt", True, False), ("7pt", False, True),
                                                   ("rmat", True, True)])
def test_every_entry_point_matches_a_fresh_solver(matrix, init_full, full, simlib):
    out = _run({"mode": "entrypoints", "matrix": matrix, "init_full": init_full, "full": full})
    assert len(out["solves"]) == 12
    assert "solvempi" in out["changed"] and "solve_cheb2" in out["changed"]


def test_three_refreshes_alternating(simlib):
    its = _run({"mode": "alternate", "matrix": "7pt"})["its"]
    assert its[0] == its[2]


def test_jacobi_after_doubling_the_diagonal(simlib):
    out = _run({"mode": "cheb_rmat"})
    assert out["its_refreshed"] == out["its_fresh"] != out["its_v1"]


def test_two_rank_partitioned_solve(simlib):
    ranks = _run({"mode": "ranks"})["ranks"]
    for r in ranks:
        assert r["same_x"] and r["its_refreshed"] == r["its_fresh"] != r["its_v1"], r
    assert ranks[0]["its_fresh"] == ranks[1]["its_fresh"]


def test_plain_hostsim_build_refuses():
    """Without the comparison launcher (the plain host-logic stand-in) the call is refused and the solver still
    solves as before."""
    p = subprocess.run(["make", "-C", SIM], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
    code = ("import sys; sys.path.insert(0, %r)\n"
            "import acg_b200.api as api; api._LIBPATH = %r\n"
            "import acg_b200 as ab; from acg_b200 import matgen as mg\n"
            "n, r, c, v = mg.laplace3d_7pt(5); A = ab.SymCsrMatrix.init_real_double(n, r, c, v).dsymv_init(0.0)\n"
            "cg = ab.SolverCuda(A); b = A.vector(); b.x[:] = 1.0\n"
            "x = A.vector(); cg.solvempi(b, x, maxits=50); its = cg.c.niterations\n"
            "try:\n    cg.update_values(A); print('ran')\n"
            "except ab.AcgError as e:\n    print('code', e.code, cg.A is A)\n"
            "y = A.vector(); cg.solvempi(b, y, maxits=50); print(cg.c.niterations == its and (x.x == y.x).all())\n"
            "cg.free()\n") % (ROOT, os.path.join(SIM, "libacgb200_hostsim.so"))
    p = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stderr[-2000:]
    assert p.stdout.strip().splitlines()[-2:] == [f"code {NOT_SUPPORTED} True", "True"]
