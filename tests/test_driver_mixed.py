"""acg_b200.driver --solver mixed: CG with float vectors and reliable updates.  CPU: the combinations it
refuses; GPU: a run on a 7-point stencil whose iterations match solve_mixed through the API and whose
residual and true residual meet the tolerance."""
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


@pytest.mark.parametrize("extra", [["--nrhs", "2"], ["--shifts", "0,0.1"]])
def test_refused_combinations(extra, tmp_path):
    n, r, c, v = mg.laplace3d_7pt(5)
    path = str(tmp_path / "A.mtx")
    mtxio.write_symmetric(path, n, r, c, v, binary=False)
    p = _driver([path, "--solver", "mixed"] + extra)
    assert p.returncode != 0 and "cannot be combined" in p.stderr, p.stderr[-2000:]


def test_refused_with_more_than_one_process(tmp_path):
    n, r, c, v = mg.laplace3d_7pt(5)
    path = str(tmp_path / "A.mtx")
    mtxio.write_symmetric(path, n, r, c, v, binary=False)
    p = _driver([path, "--solver", "mixed"], env={"WORLD_SIZE": "2"})
    assert p.returncode != 0 and "one process" in p.stderr, p.stderr[-2000:]


@pytest.mark.gpu
def test_driver_mixed(ab, tmp_path):
    """A 7-point stencil on 20^3 to rtol 1e-10: iterations within the dot-order allowance of solve_mixed
    through the API, the fp64 residual and the true residual below rtol ||b||, at least one reliable update,
    and the written solution equal to the API's x within 1e-7."""
    N = 20
    n, r, c, v = mg.laplace3d_7pt(N)
    path = str(tmp_path / "A.mtx")
    mtxio.write_symmetric(path, n, r, c, v, binary=True)
    sol = str(tmp_path / "x.mtx")
    p = _driver([path, "--binary", "--solver", "mixed", "--max-iterations", "2000", "--residual-rtol", "1e-10",
                 "--warmup", "2", "--output-solution", sol])
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-3000:]
    m = re.search(r"^mixed: iterations (\d+) reliable updates (\d+) residual 2-norm (\S+) true residual 2-norm (\S+)",
                  p.stderr, re.M)
    assert m, p.stderr[-3000:]
    its, upd, rn, true = int(m.group(1)), int(m.group(2)), float(m.group(3)), float(m.group(4))
    bn = np.sqrt(n)
    assert upd >= 1 and rn < 1e-10 * bn and true < 1e-10 * bn
    A = ab.SymCsrMatrix.init_real_double(n, r, c, v).dsymv_init(0.0)
    cg = ab.SolverCuda(A)
    bv = A.vector(); bv.x[:] = 1.0
    x = A.vector()
    assert cg.solve_mixed(bv, x, maxits=2000, residualrtol=1e-10) == 0
    assert abs(cg.c.niterations - its) <= 2
    xs = np.array([float(t) for t in open(sol).read().split("\n")[2:] if t])
    assert np.abs(xs - x.x).max() <= 1e-7 * np.abs(x.x).max()
    cg.free()
