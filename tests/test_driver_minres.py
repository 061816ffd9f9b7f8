"""acg_b200.driver --solver minres: MINRES for symmetric indefinite systems.  CPU: the combinations it
refuses; GPU: a run on a 7-point stencil shifted to have negative eigenvalues (--epsilon < 0) whose report
matches solve_minres through the API and whose true residual meets the tolerance."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from acg_b200 import matgen as mg
from acg_b200 import mtxio
from minresref import indefinite_shift, stencil_eigenvalues

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _driver(argv, env=None, timeout=240):
    return subprocess.run([sys.executable, "-m", "acg_b200.driver"] + argv, capture_output=True, text=True,
                          env=dict(os.environ, PYTHONPATH=ROOT, OMP_NUM_THREADS="2", **(env or {})), cwd=ROOT,
                          timeout=timeout)


@pytest.mark.parametrize("extra", [["--nrhs", "2"], ["--shifts", "0,0.1"]])
def test_refused_combinations(extra, tmp_path):
    n, r, c, v = mg.laplace3d_7pt(5)
    path = str(tmp_path / "A.mtx")
    mtxio.write_symmetric(path, n, r, c, v, binary=False)
    p = _driver([path, "--solver", "minres"] + extra)
    assert p.returncode != 0 and "cannot be combined" in p.stderr, p.stderr[-2000:]


def test_refused_with_more_than_one_process(tmp_path):
    n, r, c, v = mg.laplace3d_7pt(5)
    path = str(tmp_path / "A.mtx")
    mtxio.write_symmetric(path, n, r, c, v, binary=False)
    p = _driver([path, "--solver", "minres"], env={"WORLD_SIZE": "2"})
    assert p.returncode != 0 and "one process" in p.stderr, p.stderr[-2000:]


@pytest.mark.gpu
def test_driver_minres_indefinite(ab, tmp_path):
    """A 7-point stencil on 15^3 shifted by -sigma with 4 negative eigenvalues: iterations equal to
    solve_minres through the API, phi-bar below the tolerance, the true residual below 2 rtol ||b|| and
    the written solution equal to the API's x within 1e-10."""
    N = 15
    ev = stencil_eigenvalues(7, N, N, N)
    sigma = indefinite_shift(ev, 4)
    assert int((ev < sigma).sum()) == 4
    n, r, c, v = mg.laplace3d_7pt(N)
    path = str(tmp_path / "A.mtx")
    mtxio.write_symmetric(path, n, r, c, v, binary=True)
    sol = str(tmp_path / "x.mtx")
    p = _driver([path, "--binary", "--solver", "minres", "--epsilon", repr(-sigma), "--max-iterations", "3000",
                 "--residual-rtol", "1e-10", "--warmup", "2", "--output-solution", sol])
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-3000:]
    m = re.search(r"^minres: iterations (\d+) residual 2-norm (\S+) true residual 2-norm (\S+)", p.stderr, re.M)
    assert m, p.stderr[-3000:]
    its, phibar, true = int(m.group(1)), float(m.group(2)), float(m.group(3))
    bn = np.sqrt(n)
    assert phibar < 1e-10 * bn and true < 2e-10 * bn
    A = ab.SymCsrMatrix.init_real_double(n, r, c, v).dsymv_init(-sigma)
    cg = ab.SolverCuda(A)
    bv = A.vector(); bv.x[:] = 1.0
    x = A.vector()
    assert cg.solve_minres(bv, x, maxits=3000, residualrtol=1e-10) == 0
    assert cg.c.niterations == its
    xs = np.array([float(t) for t in open(sol).read().split("\n")[2:] if t])
    assert np.abs(xs - x.x).max() <= 1e-10 * np.abs(x.x).max()
    cg.free()
