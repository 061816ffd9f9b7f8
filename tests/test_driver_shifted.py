"""acg_b200.driver --shifts: several shifted systems (A + s_j I) x_j = b in one call.  CPU: the
combinations it refuses; GPU: a run whose per-shift report matches solvempi on dsymv_init(s_j)."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from acg_b200 import matgen as mg
from acg_b200 import mtxio

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _driver(argv, env=None, timeout=240):
    return subprocess.run([sys.executable, "-m", "acg_b200.driver"] + argv, capture_output=True, text=True,
                          env=dict(os.environ, PYTHONPATH=ROOT, OMP_NUM_THREADS="2", **(env or {})), cwd=ROOT,
                          timeout=timeout)


@pytest.mark.parametrize("extra,message", [
    (["--solver", "acg-pipelined"], "classic CG"),
    (["--nrhs", "2"], "cannot be combined"),
    (["--manufactured-solution"], "cannot be combined"),
    (["--shifts", "0,-1"], "finite and >= 0"),
    (["--shifts", "0,nan"], "finite and >= 0"),
    (["--shifts", "0,1,2,3,4,5,6,7,8"], "between 1 and 8"),
    (["--shifts", "0,x"], "comma-separated"),
])
def test_refused_combinations(extra, message, tmp_path):
    n, r, c, v = mg.laplace3d_7pt(5)
    path = str(tmp_path / "A.mtx")
    mtxio.write_symmetric(path, n, r, c, v, binary=False)
    argv = [path] + (extra if "--shifts" in extra else ["--shifts", "0,0.1"] + extra)
    p = _driver(argv)
    assert p.returncode != 0 and message in p.stderr, p.stderr[-2000:]


def test_refused_with_more_than_one_process(tmp_path):
    n, r, c, v = mg.laplace3d_7pt(5)
    path = str(tmp_path / "A.mtx")
    mtxio.write_symmetric(path, n, r, c, v, binary=False)
    p = _driver([path, "--shifts", "0,0.1"], env={"WORLD_SIZE": "2"})
    assert p.returncode != 0 and "one process" in p.stderr, p.stderr[-2000:]


@pytest.mark.gpu
def test_driver_shifts(ab, tmp_path):
    """Every shift of one driver run: iterations equal to solvempi on dsymv_init(s_j), true residual
    below 2 rtol ||b||, and the written solutions equal to that solve's x within 1e-10."""
    n, r, c, v = mg.stencil3d_27pt(16)
    path = str(tmp_path / "A.mtx")
    mtxio.write_symmetric(path, n, r, c, v, binary=True)
    sol = str(tmp_path / "x.mtx")
    shifts = [0.0, 0.001, 0.1, 2.0]
    p = _driver([path, "--binary", "--shifts", ",".join(map(str, shifts)), "--max-iterations", "400",
                 "--residual-rtol", "1e-9", "--warmup", "2", "--output-solution", sol])
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-3000:]
    rows = re.findall(r"^\s+shift (\d+) \((\S+)\): iterations (\d+) converged (\d) residual 2-norm (\S+) "
                      r"true residual 2-norm (\S+)", p.stderr, re.M)
    assert len(rows) == len(shifts), p.stderr[-3000:]
    b = np.ones(n)
    for j, sigma in enumerate(shifts):
        A = ab.SymCsrMatrix.init_real_double(n, r, c, v).dsymv_init(sigma)
        cg = ab.SolverCuda(A)
        bv = A.vector(); bv.x[:] = b
        x = A.vector()
        assert cg.solvempi(bv, x, maxits=400, residualrtol=1e-9) == 0
        assert int(rows[j][2]) == cg.c.niterations and rows[j][3] == "1"
        assert float(rows[j][5]) < 2e-9 * np.sqrt(n)
        xj = np.array([float(t) for t in open(f"{sol[:-4]}.{j}.mtx").read().split("\n")[2:] if t])
        assert np.abs(xj - x.x).max() <= 1e-10 * np.abs(x.x).max()
        cg.free()
