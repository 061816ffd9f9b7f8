"""Every product and solve entry point of a SolverCuda, run once on fixed inputs, and the comparison of two such
runs: what the tests of acgsolvercuda_update_values compare between a refreshed and a freshly built solver
(test_hostsim_refresh.py on the device stand-in, test_gpu_refresh.py on the H100).  Product inputs are small
integers, so that every product and dot of an integer-valued matrix is exact."""
import numpy as np


def _call(ab, fn):
    try:
        return 0, fn()
    except ab.AcgError as e:
        return e.code, None


def product_inputs(cg, A, seed=7):
    n = A.c.nownedrows
    rng = np.random.default_rng(seed)
    return {"x": rng.integers(-4, 5, cg.c.r.num_nonzeros).astype(np.float64),
            "b": rng.integers(-4, 5, n).astype(np.float64),
            "X": rng.integers(-4, 5, (n, 3)).astype(np.float64),
            "B": rng.integers(-4, 5, (n, 3)).astype(np.float64),
            "x32": rng.integers(-4, 5, n).astype(np.float32)}


def run_products(ab, cg, A, seed=7, paths=(0,)):
    """name -> (y, dot or dots) of every product; a partitioned matrix (ghost rows) only takes spmv_mode and
    spmv_ghost."""
    p = product_inputs(cg, A, seed)
    out = {}
    for path in paths:
        for m in (0, 1, 2):
            out[f"spmv_mode{m}_path{path}"] = cg.spmv_mode(m, p["x"], p["b"] if m == 2 else None, path=path)
        out[f"spmv_ghost_path{path}"] = cg.spmv_ghost(p["x"], path)
    if A.c.nghostrows > 0:
        return out
    out["spmv"] = (cg.spmv(p["x"])[0], 0.0)
    for m in (0, 1, 2):
        out[f"spmm_mode{m}"] = cg.spmm_mode(m, p["X"], p["B"] if m == 2 else None)
    out["spmv_f32"] = cg.spmv_f32(p["x32"])
    return out


def run_solves(ab, cg, A, seed=11, maxits=400, rtol=1e-10):
    """name -> (code, iterations, x) of every solve entry point from x0 = 0 (one GPU, whole matrix)."""
    n = A.c.nownedrows
    rng = np.random.default_rng(seed)
    b = rng.standard_normal(n)
    B = rng.standard_normal((n, 3))
    out = {}

    def vec_solve(name, fn):
        bv = A.vector(); bv.x[:n] = b
        xv = A.vector()
        code, _ = _call(ab, lambda: fn(bv, xv))
        out[name] = (code, int(cg.c.niterations), xv.x[:n].copy())

    kw = dict(maxits=maxits, residualrtol=rtol)
    for name in ("solvempi", "solve_pipelined", "solve_device", "solve_device_pipelined", "solve"):
        vec_solve(name, lambda bv, xv, name=name: getattr(cg, name)(bv, xv, **kw))
    ab.set_option("pcg_fused", 0)
    try:
        vec_solve("solve_pipelined_2k", lambda bv, xv: cg.solve_pipelined(bv, xv, **kw))
    finally:
        ab.set_option("pcg_fused", 1)
    X = np.zeros((n, 3))
    code, res = _call(ab, lambda: cg.solve_multi(B.copy(), X, **kw))
    out["solve_multi"] = (code, [s["niterations"] for s in res[1]] if res else None, X.copy())
    code, res = _call(ab, lambda: cg.solve_shifted(b, [0.0, 0.5], **kw))
    out["solve_shifted"] = (code, [s["niterations"] for s in res[2]] if res else None, res[1] if res else None)
    vec_solve("solve_minres", lambda bv, xv: cg.solve_minres(bv, xv, **kw))
    vec_solve("solve_mixed", lambda bv, xv: cg.solve_mixed(bv, xv, **kw))
    vec_solve("solve_cheb0", lambda bv, xv: cg.solve_chebyshev(bv, xv, degree=0, **kw))
    vec_solve("solve_cheb2", lambda bv, xv: cg.solve_chebyshev(bv, xv, degree=2, **kw))
    return out


def assert_same_products(got, want, tag, exact_dots=True):
    assert sorted(got) == sorted(want), tag
    for k in want:
        (y1, d1), (y0, d0) = got[k], want[k]
        y1, y0 = np.asarray(y1), np.asarray(y0)
        assert y1.dtype == y0.dtype and y1.shape == y0.shape, (tag, k)
        assert y1.tobytes() == y0.tobytes(), (tag, k, np.flatnonzero(y1 != y0)[:10])
        d1, d0 = np.asarray(d1, np.float64), np.asarray(d0, np.float64)
        if exact_dots:
            assert d1.tobytes() == d0.tobytes(), (tag, k, d1, d0)
        else:
            assert np.allclose(d1, d0, rtol=1e-13, atol=0.0), (tag, k, d1, d0)


def assert_same_solves(got, want, tag, rel=0.0, its_slack=0):
    """Equal codes; iteration counts equal or within its_slack; x equal (rel = 0) or within rel of the largest
    entry."""
    assert sorted(got) == sorted(want), tag
    for k in want:
        (c1, i1, x1), (c0, i0, x0) = got[k], want[k]
        assert c1 == c0, (tag, k, c1, c0)
        assert (i1 is None) == (i0 is None), (tag, k, i1, i0)
        if i0 is not None:
            assert np.all(np.abs(np.asarray(i1) - np.asarray(i0)) <= its_slack), (tag, k, i1, i0)
        if x0 is None:
            assert x1 is None, (tag, k)
            continue
        x1, x0 = np.asarray(x1), np.asarray(x0)
        if rel == 0.0:
            assert x1.tobytes() == x0.tobytes(), (tag, k)
        else:
            scale = max(float(np.abs(x0).max()), 1e-300)
            assert float(np.abs(x1 - x0).max()) <= rel * scale, (tag, k, float(np.abs(x1 - x0).max()) / scale)
