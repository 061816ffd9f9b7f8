"""acg_b200.driver --solver chebyshev: CG preconditioned with a Chebyshev polynomial in D^-1 A.  CPU: the
arguments and combinations it refuses; GPU: runs on a 7-point stencil with the estimated and a given interval
whose iterations and products match solve_chebyshev through the API and whose residual and true residual meet
the tolerance."""
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


@pytest.fixture()
def small(tmp_path):
    n, r, c, v = mg.laplace3d_7pt(5)
    path = str(tmp_path / "A.mtx")
    mtxio.write_symmetric(path, n, r, c, v, binary=False)
    return path


@pytest.mark.parametrize("extra,msg", [(["--nrhs", "2"], "cannot be combined"), (["--shifts", "0,0.1"], "cannot be combined"),
                                       (["--degree", "17"], "--degree"), (["--degree", "-1"], "--degree"),
                                       (["--interval", "1,0.5"], "--interval"), (["--interval", "0.1"], "--interval"),
                                       (["--interval", "a,b"], "--interval")])
def test_refused_arguments(extra, msg, small):
    p = _driver([small, "--solver", "chebyshev"] + extra)
    assert p.returncode != 0 and msg in p.stderr, p.stderr[-2000:]


def test_refused_elsewhere(small):
    p = _driver([small, "--solver", "chebyshev"], env={"WORLD_SIZE": "2"})
    assert p.returncode != 0 and "one process" in p.stderr, p.stderr[-2000:]
    p = _driver([small, "--interval", "0.1,2"])
    assert p.returncode != 0 and "--solver chebyshev" in p.stderr, p.stderr[-2000:]


LINE = (r"^chebyshev: degree (\d+) interval \[(\S+), (\S+)\] \((estimated from (\d+) steps|given)\) iterations (\d+) "
        r"products (\d+) residual 2-norm (\S+) true residual 2-norm (\S+)")


@pytest.mark.gpu
@pytest.mark.parametrize("degree,interval", [(2, None), (0, None), (4, "0.1,2.2")])
def test_driver_chebyshev(degree, interval, ab, tmp_path):
    """A 7-point stencil on 20^3 to rtol 1e-10: the line's iterations, products and interval equal
    solve_chebyshev's through the API, the residual and true residual are below rtol ||b||, and the written
    solution equals the API's x within 1e-10."""
    N = 20
    n, r, c, v = mg.laplace3d_7pt(N)
    path = str(tmp_path / "A.mtx")
    mtxio.write_symmetric(path, n, r, c, v, binary=True)
    sol = str(tmp_path / "x.mtx")
    argv = [path, "--binary", "--solver", "chebyshev", "--degree", str(degree), "--max-iterations", "2000",
            "--residual-rtol", "1e-10", "--warmup", "2", "--output-solution", sol]
    p = _driver(argv + (["--interval", interval] if interval else []))
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-3000:]
    m = re.search(LINE, p.stderr, re.M)
    assert m, p.stderr[-3000:]
    assert int(m.group(1)) == degree and (m.group(4) == "given") == (interval is not None)
    its, prods, rn, true = int(m.group(6)), int(m.group(7)), float(m.group(8)), float(m.group(9))
    bn = np.sqrt(n)
    assert rn < 1e-10 * bn and true < 2e-10 * bn
    A = ab.SymCsrMatrix.init_real_double(n, r, c, v).dsymv_init(0.0)
    cg = ab.SolverCuda(A)
    bv = A.vector(); bv.x[:] = 1.0
    x = A.vector()
    lo, hi = (float(t) for t in interval.split(",")) if interval else (0.0, 0.0)
    assert cg.solve_chebyshev(bv, x, degree=degree, lmin=lo, lmax=hi, maxits=2000, residualrtol=1e-10) == 0
    assert cg.c.niterations == its and cg.c.ngemv == prods
    inf = cg.info()
    assert float(m.group(2)) == pytest.approx(inf["cheb_lmin"], rel=1e-5) and float(m.group(3)) == pytest.approx(inf["cheb_lmax"], rel=1e-5)
    xs = np.array([float(t) for t in open(sol).read().split("\n")[2:] if t])
    assert np.abs(xs - x.x).max() <= 1e-10 * np.abs(x.x).max()
    cg.free()
