"""Every solve entry point and product on the smallest matrices and at the 32-row slice boundaries.

Every other exact comparison of the newer solve paths runs matrices of 60 rows or more.  Below that the
index and grid arithmetic meets its edges: fewer rows than one pattern slice (one BLAS-1 CTA whose threads
mostly have no row, one partly filled tile), n = 1 (the row-pair loops do nothing and only the odd-last-row
branches run), exactly one covered slice with or without tile rows after it (which kernel forwards the
control word; a mirrored-diagonal margin as wide as the matrix), and matrices whose Krylov space is
exhausted before the solver stops.  Here:

* a ladder of small matrices -- the 1-D 3-point chain at n = 1 .. 97 around the multiples of 32, diagonal
  matrices (slices without mirrored diagonals: "no gain"), 27- and 7-point boxes with degenerate dimensions,
  a random SPD matrix under forced medium-row and long-row plans, and an arrow matrix (a hub row) under
  long-row and merge-path plans (a single 1024-row tile; 64-item tiles that split the hub over 32) -- each
  pinned to its plan regime from the host planners (CPU) and from info() (GPU);
* the products (spmv_mode, spmm_mode for 1, 2, 3, 5, 8 columns, spmv_f32) in every epilogue mode against the
  exact reference of tests/exactref.py: bitwise on integer data, signed zeros included (the contract is
  stated at _check_product), within 2 gamma(m+1) sum|a x| on real data;
* classic, device and pipelined CG (fused and two-kernel) against the oracle, solve_multi and solve_shifted
  against solvempi, MINRES (positive definite, indefinite, singular and consistent), mixed precision and
  Chebyshev PCG against the restatements: converged solves at two tolerances, fixed iteration counts around
  the polling interval (graph replays), maxits = 0 at n = 1, and subsets with programmatic dependent launch
  and with the host polling after every iteration.  Every converged solve's true residual is below 2 tol
  and its x within ||r|| / lambda_min of the dense solution.

The layout assertions are skipped on the host-logic stand-in (ACGB200_TEST_LIB), which never takes the
mirrored diagonals."""
import functools
import os

import numpy as np
import pytest
import scipy.sparse as sp

from chebref import chebyshev
from exactref import U, dot_exact, gamma, rows_exact
from minresref import minres
from mixedref import mixed

STANDIN = bool(os.environ.get("ACGB200_TEST_LIB"))
MAXITS = 2000
# Two comparisons on the arrow matrix that are not understood yet.  Every other assertion of their tests still
# runs; these are reported as expected failures with the numbers, not hidden behind a looser bound.
OPEN_PIPELINED = ("open: two-kernel pipelined CG on the 100-row arrow stops one iteration after the oracle at "
                  "rtol 1e-9 (13 against 12); the oracle's count does not move when b changes in its last bit: ")
OPEN_SHIFTED = ("open: after 7 steps on the 1024-row arrow, solve_shifted's x for sigma = 0.1 mean(diag) parts "
                "from solvempi's by 2.7e-5 relative, where the oracle's residual is 3.8e-5 ||b|| and the guard "
                "that skips rounding-level iterates should have applied; and at rtol 1e-10 the iteration count "
                "of one shift has differed by one from solvempi's in one run of several (12 against 13): ")
# every option a test here changes, and its default
DEFAULTS = {"spmv_slices": 1, "spmv_merge": -1, "merge_items": 0, "spmv_nnz_cap": 0, "spmv_medium": 0,
            "symdiag_codes": 1, "pcg_fused": 1, "pdl": 0, "check_every": 8}
OPTSETS = {"default": {}, "pdl": {"pdl": 1}, "poll1": {"check_every": 1}}


# ---------------------------------------------------------------------------------------------
# the ladder


def _arrow(n):
    """Row 0 coupled to every row (a hub of n entries), the other rows diagonal plus that coupling:
    diagonally dominant, with distinct leaf diagonals 2 + i/n, so that the spectrum is spread (n distinct
    eigenvalues) and the Krylov solvers do not meet repeated eigenvalues."""
    r = np.concatenate([np.arange(n), np.zeros(n - 1, np.int64)])
    c = np.concatenate([np.arange(n), np.arange(1, n)])
    v = np.concatenate([[n + 1.0], 2.0 + np.arange(1, n) / n, -np.ones(n - 1)])
    o = np.lexsort((c, r))
    return n, r[o].astype(np.int32), c[o].astype(np.int32), v[o]


def _diagonal(n):
    d = np.arange(n, dtype=np.int32)
    return n, d, d.copy(), 1.0 + 0.5 * np.arange(n)


def _neumann(n):
    """The 1-D chain with diagonal 1 at both ends: singular, null space the constant vector."""
    from acg_b200 import matgen as mg
    n, r, c, v = mg.poisson1d_3pt(n)
    v = v.copy()
    v[(r == c) & ((r == 0) | (r == n - 1))] = 1.0
    return n, r, c, v


@functools.lru_cache(maxsize=None)
def _gen(key):
    from acg_b200 import matgen as mg
    kind, arg = key
    if kind == "1d":
        return mg.poisson1d_3pt(arg)
    if kind == "diag":
        return _diagonal(arg)
    if kind == "27pt":
        return mg.stencil3d_27pt(*arg)
    if kind == "7pt":
        return mg.laplace3d_7pt(*arg)
    if kind == "rand":
        return mg.random_spd(arg)
    if kind == "arrow":
        return _arrow(arg)
    if kind == "neumann":
        return _neumann(arg)
    raise ValueError(key)


class E:
    """A ladder entry: matrix key, forced plan options and the regime they give.  slices: covered 32-row
    slices; tile_rows: rows left to the tile kernel (or to medium / long rows); reason: the host
    mirrored-diagonal plan's verdict; D: the stored diagonals when eligible; wide: margin >= n."""

    def __init__(self, eid, key, slices=0, tile_rows=None, reason="no slices", D=None, opts=None, wide=False,
                 merge=None, nlong=0, nmed=0):
        self.eid, self.key, self.slices, self.reason, self.D = eid, key, slices, reason, D
        self.opts = dict(opts or {})
        self.wide, self.merge, self.nlong, self.nmed = wide, merge, nlong, nmed
        n = _gen(key)[0]
        self.tile_rows = n - 32 * slices if tile_rows is None else tile_rows

    @property
    def symdiag(self):
        return self.reason == "eligible"

    @property
    def fused(self):
        """the fused pipelined iteration applies: mirrored diagonals, every other row in tiles"""
        return self.symdiag and self.nmed == 0 and self.nlong == 0 and not self.merge


NOSLICE = {"spmv_slices": 0, "spmv_merge": 0}
LADDER = [E(f"1d-{n}", ("1d", n)) for n in (1, 2, 3, 5, 8, 31)] + [
    E("1d-32", ("1d", 32), 1, reason="eligible", D=[0, 1], wide=True),
    E("1d-33", ("1d", 33), 1, reason="eligible", D=[0, 1]),
    E("1d-33-medium", ("1d", 33), 1, reason="eligible", D=[0, 1], opts={"spmv_medium": 1}, nmed=1),
    E("1d-63", ("1d", 63), 1, reason="eligible", D=[0, 1]),
    E("1d-64", ("1d", 64), 2, reason="eligible", D=[0, 1]),
    E("1d-65", ("1d", 65), 2, reason="eligible", D=[0, 1]),
    E("1d-97", ("1d", 97), 3, reason="eligible", D=[0, 1]),
    E("diag-1", ("diag", 1)),
    E("diag-32", ("diag", 32), 1, reason="no gain"),
    E("diag-33", ("diag", 33), 1, reason="no gain"),
    E("27pt-2x2x8", ("27pt", (2, 2, 8)), 1, reason="eligible", D=list(range(8)), wide=True),
    E("27pt-3x3x4", ("27pt", (3, 3, 4))),
    E("27pt-4x4x4", ("27pt", (4, 4, 4))),
    E("27pt-5x1x7", ("27pt", (5, 1, 7)), 1, reason="eligible", D=[0, 1, 4, 5, 6]),
    E("27pt-1x1x40", ("27pt", (1, 1, 40)), 1, reason="eligible", D=[0, 1]),
    E("7pt-2x3x5", ("7pt", (2, 3, 5))),
    E("7pt-3x3x4", ("7pt", (3, 3, 4)), 1, reason="eligible", D=[0, 1, 3, 9]),
    E("7pt-1x33x1", ("7pt", (1, 33, 1)), 1, reason="eligible", D=[0, 1]),
    E("rand-40", ("rand", 40)),
    E("rand-40-long", ("rand", 40), opts=dict(NOSLICE, spmv_nnz_cap=8), nlong=1),
    E("rand-40-medium", ("rand", 40), opts=dict(NOSLICE, spmv_nnz_cap=8, spmv_medium=3), nlong=1, nmed=27),
    E("arrow-100", ("arrow", 100), 2, reason="too many offsets"),
    E("arrow-100-long", ("arrow", 100), opts=dict(NOSLICE, spmv_nnz_cap=8), nlong=1),
    E("arrow-1024-merge1", ("arrow", 1024), tile_rows=0, opts={"spmv_slices": 0, "spmv_merge": 1, "merge_items": 4096},
      merge=(1, 0)),
    E("arrow-1024-merge64", ("arrow", 1024), tile_rows=0, opts={"spmv_slices": 0, "spmv_merge": 1, "merge_items": 64},
      merge=(64, 32)),
]
BY_ID = {e.eid: e for e in LADDER}
IDS = [e.eid for e in LADDER]
# the subsets run again with PDL on and with the host polling after every iteration
SUBSET = ["1d-1", "1d-3", "1d-31", "1d-32", "1d-33", "1d-33-medium", "1d-97", "diag-33", "27pt-2x2x8",
          "7pt-3x3x4", "rand-40-medium", "arrow-100-long", "arrow-1024-merge1", "arrow-1024-merge64"]
RUNS = [(e, "default") for e in IDS] + [(e, o) for o in ("pdl", "poll1") for e in SUBSET]
RUN_IDS = [f"{e}-{o}" for e, o in RUNS]


# ---------------------------------------------------------------------------------------------
# matrices, options, regime


_MATRICES = {}


def _matrix(ab, key, eps=0.0):
    k = (key, eps)
    if k not in _MATRICES:
        n, r, c, v = _gen(key)
        _MATRICES[k] = ab.SymCsrMatrix.init_real_double(n, r, c, v).dsymv_init(eps)
    return _MATRICES[k]


def teardown_module(module):
    for A in _MATRICES.values():
        A.free()
    _MATRICES.clear()


def _csr(A):
    n = A.c.nownedrows
    rp = A.frowptr[:n + 1].copy()
    return (rp, A.fcolidx[:rp[n]].copy(), A.fa[:rp[n]].copy())


def _scipy(csr):
    rp, ci, a = csr
    n = len(rp) - 1
    return sp.csr_matrix((a, ci, rp), shape=(n, n))


@functools.lru_cache(maxsize=None)
def _spectrum(key, eps=0.0, jacobi=False):
    """eigenvalues (ascending) of the dense matrix A + eps I -- with jacobi, of D^-1/2 A D^-1/2, which has the
    eigenvalues of D^-1 A that Jacobi and Chebyshev PCG see -- and the number of distinct ones"""
    from acg_b200 import matgen as mg
    n, r, c, v = _gen(key)
    M = mg.upper_to_dense(n, r, c, v) + eps * np.eye(n)
    if jacobi:
        s = 1 / np.sqrt(np.diag(M))
        M = s[:, None] * M * s[None, :]
    ev = np.linalg.eigvalsh(M)
    ndist = 1 + int((np.diff(ev) > 1e-9 * np.abs(ev).max()).sum())
    return ev, ndist


@pytest.fixture
def options(ab):
    """set_option for the next SolverCuda; every option this file touches back to its default after."""
    def set_(**kw):
        for k, v in dict(DEFAULTS, **kw).items():
            ab.set_option(k, v)
    yield set_
    for k, v in DEFAULTS.items():
        ab.set_option(k, v)


def _ncodes(A, codes_on=True):
    """The code table the solver builds: the distinct bit patterns of the stored (upper) entries and the +0.0
    of absent entries and margins, when there are at most 256 of them and codes are on (else 0)."""
    rp, ci, fa = _csr(A)
    rows = np.repeat(np.arange(len(rp) - 1), np.diff(rp))
    k = len(set(fa[ci >= rows].view(np.uint64).tolist()) | {0})
    return k if codes_on and k <= 256 else 0


def _in_regime(cg, e, ncodes=None):
    """info(): the plan is the one the ladder entry names (ncodes: the code table's size; None: any)."""
    inf = cg.info()
    if STANDIN:
        return inf
    tag = (e.eid, inf)
    assert inf["spmv_slices"] == e.slices and inf["spmv_slice_rows"] == 32 * e.slices, tag
    assert inf["spmv_nlong"] == e.nlong and inf["spmv_nmedium"] == e.nmed, tag
    assert (inf["spmv_ntiles"] > 0) == (e.tile_rows - e.nlong - e.nmed > 0), tag
    if e.merge:
        assert (inf["spmv_merge_tiles"], inf["spmv_merge_split"]) == e.merge and inf["spmv_merge_rows"] == cg.A.c.nownedrows, tag
    else:
        assert inf["spmv_merge_tiles"] == 0, tag
    assert inf["spmv_symdiag_diagonals"] == (len(e.D) if e.symdiag else 0), tag
    if e.symdiag:
        if ncodes is None:
            assert inf["spmv_symdiag_codes"] > 0, tag
        else:
            assert inf["spmv_symdiag_codes"] == ncodes, tag
    return inf


def _vec(A, v):
    out = A.vector()
    out.x[:A.c.nownedrows] = v
    return out


def _true_residual(csr, x, b):
    r, _, _ = rows_exact(*csr, x, b)
    return float(np.linalg.norm(r))


def _check_solution(key, csr, x, b, tol, eps=0.0, ref_x=None):
    """A converged solve: the true residual (exact rows) below 2 tol, and x within ||r|| / lambda_min (plus
    the dense solve's own rounding, kappa u ||x||) of numpy.linalg.solve of the fp64 matrix.  With ref_x
    (the reference's solution) tol is at least that solution's true residual: below it the recursively
    updated residual has parted from the true one in the reference too (attainable accuracy)."""
    if ref_x is not None:
        tol = max(tol, _true_residual(csr, ref_x, b))
    res = _true_residual(csr, x, b)
    assert res < 2 * tol, (res, tol)
    ev, _ = _spectrum(key, eps)
    lmin = float(np.abs(ev).min())
    xs = np.linalg.solve(_scipy(csr).toarray(), b)
    kappa = float(np.abs(ev).max()) / lmin
    err = float(np.linalg.norm(x - xs))
    assert err <= 2 * tol / lmin + 100 * kappa * U * float(np.linalg.norm(xs)), (err, tol, lmin)


def _rounding_level(ref):
    """a fixed-count reference whose residual is down to 1e-4 of ||r0||: the Krylov space is nearly exhausted
    and the iterates amplify rounding, so only the counts are compared"""
    return ref["rnrm2"] < 1e-4 * ref["r0nrm2"]


def _xtol(e, pipelined=False):
    """x against the reference: 1e-10 relative; 1e-9 (test_gpu_parity.py's bound) for pipelined CG, whose x
    parts from the oracle's by about kappa u per step on the kappa ~ 4000 chains; 1e-8 on the arrow matrices,
    whose iterates amplify rounding: b changed in its last bit moves the oracle's own x after 7 CG steps on
    the 100-row arrow by 8e-9 relative"""
    if e.key[0] == "arrow":
        return 1e-8
    return 1e-9 if pipelined else 1e-10


def _counts(check_every):
    return sorted({m for m in (1, 2, 3, check_every - 1, check_every, check_every + 1) if m >= 1})


def _fixed_counts(key, check_every, eps=0.0, jacobi=False):
    """fixed iteration counts around the polling interval below the number of distinct eigenvalues of the
    operator the solver's Krylov space is built from (jacobi: D^-1 A): at or past it the Krylov space is
    exhausted and r is 0 up to rounding"""
    _, ndist = _spectrum(key, eps, jacobi)
    return [m for m in _counts(check_every) if m < ndist - 1]


# ---------------------------------------------------------------------------------------------
# CPU: the regime guard


def test_regime_guard(ab):
    """Every ladder entry is in its regime by the host planners: covered slices and the rows outside them,
    the mirrored-diagonal verdict and diagonals, a margin at least n where that is the point, and the tile,
    long-row, medium-row and merge-path plans under the entry's options."""
    try:
        for e in LADDER:
            for k, v in dict(DEFAULTS, **e.opts).items():
                ab.set_option(k, v)
            n, r, c, v = _gen(e.key)
            A = ab.SymCsrMatrix.init_real_double(n, r, c, v).dsymv_init(0.0)
            rp, ci, _ = _csr(A)
            A.free()
            use_slices = e.opts.get("spmv_slices", 1) != 0
            sl = ab.slices_host(rp, ci)
            sd = ab.symdiag_host(rp, ci)
            if use_slices:
                assert sl["nslices"] == e.slices and int(sl["covered"].sum()) == e.slices, (e.eid, sl["nslices"])
                assert sd["reason"] == e.reason, (e.eid, sd["reason"])
                if e.symdiag:
                    assert list(sd["D"]) == e.D, (e.eid, sd["D"])
                    assert (sd["margin"] >= n) == e.wide, (e.eid, sd["margin"])
            pl = ab.spmv_plan_host(rp, ci)
            if e.merge:
                mp = ab.merge_plan_host(rp, items=e.opts["merge_items"])
                assert (len(mp["tiles"]), len(mp["split"])) == e.merge and n >= 1024, e.eid
                assert (rp[n] + n) <= e.opts["merge_items"] or len(mp["split"]) > 0
                continue
            assert pl["slices"] == (e.slices if use_slices else 0), e.eid
            assert len(pl["longrows"]) == e.nlong and pl["nmedium"] == e.nmed, (e.eid, pl["longrows"], pl["nmedium"])
            rows_in_tiles = int(pl["tiles"][:, 1].sum()) if len(pl["tiles"]) else 0
            assert rows_in_tiles + e.nlong + e.nmed == e.tile_rows, (e.eid, rows_in_tiles)
            if n < 32:
                assert len(pl["tiles"]) == 1 and pl["tiles"][0, 1] == n, e.eid
    finally:
        for k, v in DEFAULTS.items():
            ab.set_option(k, v)
    # what the entries are there for
    assert {BY_ID[f"1d-{n}"].tile_rows for n in (32, 64)} == {0} and BY_ID["1d-33"].tile_rows == 1
    assert _gen(("1d", 97))[0] == 3 * 32 + 1 and _gen(("7pt", (2, 3, 5)))[0] == 30 < 32
    for n in (1, 2, 3, 5, 8):
        assert _spectrum(("1d", n))[1] == n                 # Krylov space exhausted within n steps


# ---------------------------------------------------------------------------------------------
# products against the exact reference


def _product_data(key, kind, seed):
    """values and inputs: "int" small integers, "stencil" the generator's values with integer x and b (exact
    where the values are integers), "real" random reals.  At n <= 3 some entries of x and b are -0.0."""
    n, r, c, v = _gen(key)
    rng = np.random.default_rng(seed)
    diag = r == c
    if kind == "int":
        v = rng.integers(-3, 4, len(r)).astype(np.float64)
        v[diag] = rng.integers(1, 9, int(diag.sum()))
    elif kind == "real":
        v = rng.standard_normal(len(r))
        v[diag] += 4.0
    if kind == "real":
        x = rng.standard_normal(n)
        b = rng.standard_normal(n)
    else:
        x = rng.integers(-3, 4, n).astype(np.float64)
        b = rng.integers(-40, 41, n).astype(np.float64)
        if n <= 3:
            x[::2] = -0.0
            b[: 2] = -0.0
            x[x == 0] = -0.0
    # integer values and inputs: every partial sum is exact, whatever the order
    exact = kind != "real" and bool(np.all(v == np.round(v)))
    return n, r, c, v, x, b, exact


def _same_bits(got, want):
    return np.flatnonzero(np.asarray(got, np.float64).view(np.int64) != np.asarray(want, np.float64).view(np.int64))


def _check_product(csr, x, b, mode, y, dot, exact, tag):
    """y (and the fused dot) of one epilogue mode against the exact value: bitwise with signed zeros on
    integer data, within 2 gamma(m+1) sum|a x| (+|b|) on real data.

    Signed zeros are a contract of the products, beyond what IEEE fixes for a sum in no particular order:
    every fp64 kernel (tiles, slices, mirrored diagonals, merge path, medium and long rows, multi-vector)
    accumulates a row from +0.0, y_i = +0.0 + sum_j a_ij x_j, and forms r_i = b_i - y_i.  So a row whose
    exact value is 0 gives y_i = +0.0 -- a single product -0.0 (n = 1, x = -0.0) included -- and r_i keeps
    the sign of b_i: -0.0 exactly where b_i is -0.0.  That makes the bits of every result independent of
    the plan that computed them."""
    assert not np.isnan(y).any(), (tag, np.flatnonzero(np.isnan(y))[:10])
    want, scale, m = rows_exact(*csr, x, b if mode == 2 else None)
    if exact:
        # y_i = +0.0 + sum_j a_ij x_j; r_i = b_i - y_i
        want = want + 0.0 if mode != 2 else b - (rows_exact(*csr, x)[0] + 0.0)
        bad = _same_bits(y, want)
        assert bad.size == 0, (tag, bad[:10], y[bad[:10]], want[bad[:10]])
    else:
        err = np.abs(y - want)
        bad = np.flatnonzero(err > 2.0 * gamma(m + 1) * scale)
        assert bad.size == 0, (tag, bad[:10], err[bad[:10]])
    if mode == 0:
        assert dot == 0.0, tag
        return
    u = x if mode == 1 else y
    wdot = dot_exact(u, y)
    if exact:
        assert dot == wdot, (tag, dot, wdot)
    else:
        assert abs(dot - wdot) <= 2.0 * gamma(len(y)) * float(np.abs(u * y).sum()), (tag, dot, wdot)


def _product_runs(e):
    """data kinds and options: on these sizes even random reals fit the code table, so the fp64 diagonals
    are forced with symdiag_codes=0"""
    kinds = [("int", {}), ("stencil", {}), ("real", {})]
    if e.symdiag:
        kinds += [("int", {"symdiag_codes": 0}), ("real", {"symdiag_codes": 0})]
    return kinds


@pytest.mark.gpu
@pytest.mark.parametrize("eid", IDS)
def test_products_against_exact(eid, ab, options):
    """spmv_mode in the three epilogue modes, spmm_mode for 1, 2, 3, 5 and 8 columns in the three modes, and
    spmv_f32, on integer, stencil-valued and real data (and integer data with symdiag_codes=0 where the
    mirrored diagonals apply).  The outputs are poisoned with NaN on the device before each product."""
    e = BY_ID[eid]
    for i, (kind, extra) in enumerate(_product_runs(e)):
        n, r, c, v, x, b, exact = _product_data(e.key, kind, 300 + i)
        A = ab.SymCsrMatrix.init_real_double(n, r, c, v).dsymv_init(0.0)
        try:
            options(**e.opts, **extra)
            cg = ab.SolverCuda(A)
            try:
                _in_regime(cg, e, ncodes=_ncodes(A, extra.get("symdiag_codes", 1) != 0))
                csr = _csr(A)
                xg = np.pad(x, (0, cg.c.r.num_nonzeros - n))
                for mode in (0, 1, 2):
                    y, dot = cg.spmv_mode(mode, xg, b if mode == 2 else None)
                    _check_product(csr, x, b, mode, y, dot, exact, (eid, kind, extra, "spmv", mode))
                rng = np.random.default_rng(400 + i)
                for k in (1, 2, 3, 5, 8):
                    if exact:
                        X = rng.integers(-3, 4, (n, k)).astype(np.float64)
                        B = rng.integers(-40, 41, (n, k)).astype(np.float64)
                        X[:, 0], B[:, 0] = x, b                     # the signed zeros of the single vector
                    else:
                        X, B = rng.standard_normal((n, k)), rng.standard_normal((n, k))
                    for mode in (0, 1, 2):
                        Y, dots = cg.spmm_mode(mode, X, B if mode == 2 else None)
                        for j in range(k):
                            _check_product(csr, X[:, j], B[:, j], mode, Y[:, j], dots[j], exact,
                                           (eid, kind, extra, "spmm", k, mode, j))
                # the fp32 product of solve_mixed, by the rule of test_gpu_mixed.py::test_spmv_f32
                xf = rng.standard_normal(n).astype(np.float32)
                yf, dotf = cg.spmv_f32(xf)
                assert yf.dtype == np.float32 and np.isfinite(yf).all(), (eid, kind)
                ex, scale, m = rows_exact(*csr, xf.astype(np.float64))
                bound = np.abs(ex) * 2.0 ** -24 + (m + 2) * 2.0 ** -53 * scale + 1e-300
                assert (np.abs(yf.astype(np.float64) - ex) <= bound).all(), (eid, kind)
                assert dotf == pytest.approx(float(xf.astype(np.float64) @ yf.astype(np.float64)), rel=1e-12,
                                             abs=1e-12 * n)
                if exact:
                    xi = rng.integers(-100, 101, n).astype(np.float32)
                    yi, doti = cg.spmv_f32(xi)
                    exi, _, _ = rows_exact(*csr, xi.astype(np.float64))
                    assert np.array_equal(yi.astype(np.float64), exi), (eid, kind)
                    assert doti == float(xi.astype(np.float64) @ exi), (eid, kind)
            finally:
                cg.free()
        finally:
            A.free()


# ---------------------------------------------------------------------------------------------
# classic and pipelined CG against the oracle


CG_METHODS = [("solvempi", 1, "cg"), ("solve", 1, "cg"), ("solve_device", 1, "cg"),
              ("solve_pipelined", 0, "cg_pipelined"), ("solve_pipelined", 1, "cg_pipelined")]


@pytest.mark.gpu
@pytest.mark.parametrize("eid,optset", RUNS, ids=RUN_IDS)
def test_cg_against_oracle(eid, optset, ab, options, oracle):
    """solvempi, solve, solve_device and pipelined CG (two-kernel, and fused where the plan allows it) from a
    nonzero x0 at rtol 1e-12 (pipelined: 1e-9; on the arrow: 1e-10) and 1e-6: the oracle's return code and
    iteration count, x within _xtol, the converged solution checked against the dense solve; then fixed iteration counts with
    tolerances off (graph replays) against the oracle at every count."""
    e = BY_ID[eid]
    opts = OPTSETS[optset]
    options(**e.opts, **opts)
    A = _matrix(ab, e.key)
    n = A.c.nownedrows
    csr = _csr(A)
    rng = np.random.default_rng(11)
    b, x0 = rng.standard_normal(n), rng.standard_normal(n)
    check_every = opts.get("check_every", DEFAULTS["check_every"])
    open_findings = []
    cg = ab.SolverCuda(A)
    try:
        _in_regime(cg, e)
        for method, fused, orc in CG_METHODS:
            ab.set_option("pcg_fused", fused)
            # pipelined CG's attainable accuracy on the kappa ~ 4000 chains lies near 1e-12: 1e-9 there; on the
            # arrow (||A|| ~ 100 from the hub) classic CG's residual reaches 1.8e-12 ||r0|| one step before the
            # oracle stops at 1e-12, within rounding of the threshold: 1e-10 there
            rtols = (1e-9, 1e-6) if orc == "cg_pipelined" else (1e-10, 1e-6) if e.key[0] == "arrow" else (1e-12, 1e-6)
            runs = [(MAXITS, rtol) for rtol in rtols] + [(m, 0.0) for m in _fixed_counts(e.key, check_every)]
            for maxits, rtol in runs:
                want = getattr(oracle, orc)(csr, b, x0=x0, maxits=maxits, rtol=rtol)
                xv = _vec(A, x0)
                code = getattr(cg, method)(_vec(A, b), xv, maxits=maxits, residualrtol=rtol, warmup=1)
                x = xv.x[:n]
                tag = (method, fused, maxits, rtol)
                assert code == want["status"] == 0, (tag, code, want["status"])
                if (orc == "cg_pipelined" and e.key == ("arrow", 100) and maxits == MAXITS
                        and cg.c.niterations != want["niterations"]):
                    open_findings.append((tag, cg.c.niterations, want["niterations"]))
                    continue
                assert cg.c.niterations == want["niterations"], (tag, cg.c.niterations, want["niterations"])
                if rtol == 0:
                    assert cg.c.niterations == maxits, tag
                    if _rounding_level(want):
                        continue
                assert np.abs(x - want["x"]).max() <= _xtol(e, orc == "cg_pipelined") * np.abs(want["x"]).max(), tag
                if rtol > 0:
                    _check_solution(e.key, csr, x, b, rtol * want["r0nrm2"], ref_x=want["x"])
                if method == "solve_pipelined" and not STANDIN:
                    assert cg.info()["pcg_fused"] == (1 if fused and e.fused else 0), tag
    finally:
        cg.free()
    if open_findings:
        pytest.xfail(OPEN_PIPELINED + repr(open_findings))


@pytest.mark.gpu
@pytest.mark.parametrize("eid", ["1d-1", "diag-1"])
def test_maxits_zero_returns_x0(eid, ab, options):
    """maxits = 0 at n = 1 on every entry point: x0 back bitwise (solve_shifted: x = 0), no iteration."""
    e = BY_ID[eid]
    options(**e.opts)
    A = _matrix(ab, e.key)
    x0, b = np.array([-0.3125]), np.array([1.75])
    cg = ab.SolverCuda(A)
    try:
        _in_regime(cg, e)
        for name, kw in (("solvempi", {}), ("solve", {}), ("solve_device", {}), ("solve_pipelined", {}),
                         ("solve_minres", {}), ("solve_mixed", {}), ("solve_chebyshev", {"degree": 0}),
                         ("solve_chebyshev", {"degree": 2})):
            xv = _vec(A, x0)
            getattr(cg, name)(_vec(A, b), xv, maxits=0, residualrtol=1e-8, **kw)
            assert cg.c.niterations == 0 and _same_bits(xv.x[:1], x0).size == 0, (name, kw, xv.x[:1])
        X = x0.reshape(1, 1).copy()
        _, cols = cg.solve_multi(b.reshape(1, 1).copy(), X, maxits=0, residualrtol=1e-8)
        assert cols[0]["niterations"] == 0 and _same_bits(X[:, 0], x0).size == 0
        _, X, cols = cg.solve_shifted(b, [0.0, 0.5], maxits=0, residualrtol=1e-8)
        assert all(c["niterations"] == 0 for c in cols) and _same_bits(X.ravel(), [0.0, 0.0]).size == 0
    finally:
        cg.free()


# ---------------------------------------------------------------------------------------------
# several right-hand sides and shifted systems against solvempi


@pytest.mark.gpu
@pytest.mark.parametrize("eid,optset", RUNS, ids=RUN_IDS)
def test_multi_against_solvempi(eid, optset, ab, options):
    """solve_multi with 1, 3 and 8 columns (column j of B scaled by 2^j under one absolute tolerance, random
    X0, column 2 with b = x0 = 0) column by column against solvempi: equal iteration counts, ||r|| within
    1e-10 ||r0||, x within 1e-10 relative, the converged solution against the dense solve; then 3 columns
    for fixed iteration counts with tolerances off."""
    e = BY_ID[eid]
    options(**e.opts, **OPTSETS[optset])
    A = _matrix(ab, e.key)
    n = A.c.nownedrows
    csr = _csr(A)
    rng = np.random.default_rng(21)
    B8 = rng.standard_normal((n, 8)) * 2.0 ** np.arange(8)
    X8 = rng.standard_normal((n, 8))
    B8[:, 2] = X8[:, 2] = 0.0
    atol = 1e-8 * float(np.linalg.norm(B8[:, 0]))
    cg = ab.SolverCuda(A)
    single = {}
    try:
        _in_regime(cg, e)

        def solvempi(j, maxits, tol):
            if (j, maxits) not in single:
                xv = _vec(A, X8[:, j])
                code = cg.solvempi(_vec(A, B8[:, j]), xv, maxits=maxits, residualatol=tol)
                single[j, maxits] = (code, int(cg.c.niterations), float(cg.c.rnrm2), float(cg.c.r0nrm2), xv.x[:n].copy())
            return single[j, maxits]

        # fixed counts: three columns without the zero one (with tolerances off, b = 0 leaves 0/0 to the loop)
        runs = [(list(range(k)), MAXITS, atol) for k in (1, 3, 8)] + [([0, 1, 3], m, 0.0) for m in _fixed_counts(e.key, 8)]
        for idx, maxits, tol in runs:
            X = np.ascontiguousarray(X8[:, idx])
            code, cols = cg.solve_multi(np.ascontiguousarray(B8[:, idx]), X, maxits=maxits, residualatol=tol, warmup=1)
            assert code == 0 and cg.c.niterations == max(c["niterations"] for c in cols), (idx, maxits, cols)
            for i, j in enumerate(idx):
                cj, its, rn, r0, xj = solvempi(j, maxits, tol)
                tag = (idx, maxits, j, cols[i], its)
                assert cj == 0 and cols[i]["niterations"] == its, tag
                if tol == 0 and _rounding_level({"rnrm2": _true_residual(csr, xj, B8[:, j]),
                                                 "r0nrm2": _true_residual(csr, X8[:, j], B8[:, j])}):
                    continue
                assert abs(cols[i]["rnrm2"] - rn) <= 1e-10 * r0, tag
                assert float(np.abs(X[:, i] - xj).max()) <= _xtol(e) * float(np.abs(xj).max()), tag
                if j == 2:
                    assert not X[:, i].any() and its == 0, tag
                elif tol > 0:
                    _check_solution(e.key, csr, X[:, i], B8[:, j], atol, ref_x=xj)
    finally:
        cg.free()


SHIFTS = [0.0, 1.0, 0.1, 0.01, 0.3, 0.03, 3.0, 1e-3]      # relative to the mean diagonal entry


@pytest.mark.gpu
@pytest.mark.parametrize("eid,optset", RUNS, ids=RUN_IDS)
def test_shifted_against_solvempi(eid, optset, ab, options):
    """solve_shifted with 1, 3 and 8 shifts, shift by shift against solvempi on a solver of dsymv_init(sigma):
    equal iteration counts and convergence flags, x within 1e-10 relative, the converged solution of
    A + sigma I against the dense solve; then 3 shifts for fixed iteration counts with tolerances off."""
    e = BY_ID[eid]
    options(**e.opts, **OPTSETS[optset])
    A = _matrix(ab, e.key)
    n = A.c.nownedrows
    rp, ci, a = _csr(A)
    dmean = float(a[np.repeat(np.arange(n), np.diff(rp)) == ci].mean())
    b = np.random.default_rng(41).standard_normal(n)
    rtol = 1e-10
    open_findings = []
    cg = ab.SolverCuda(A)
    single = {}
    try:
        _in_regime(cg, e)

        def solvempi(sigma, maxits, tol):
            if (sigma, maxits) not in single:
                Aj = _matrix(ab, e.key, sigma)
                cgj = ab.SolverCuda(Aj)
                try:
                    _in_regime(cgj, e)
                    xv = Aj.vector()
                    code = cgj.solvempi(_vec(Aj, b), xv, maxits=maxits, residualrtol=tol)
                    xj, csrj = xv.x[:n].copy(), _csr(Aj)
                    # the residual of x itself: with tolerances off the solver's rnrm2 is not kept up
                    norms = {"rnrm2": _true_residual(csrj, xj, b), "r0nrm2": float(np.linalg.norm(b))}
                    single[sigma, maxits] = (code, int(cgj.c.niterations), xj, csrj, norms)
                finally:
                    cgj.free()
            return single[sigma, maxits]

        runs = [(S, MAXITS, rtol) for S in (1, 3, 8)] + [(3, m, 0.0) for m in _fixed_counts(e.key, 8)]
        for S, maxits, tol in runs:
            shifts = [dmean * s for s in SHIFTS[:S]]
            code, X, cols = cg.solve_shifted(b, shifts, maxits=maxits, residualrtol=tol, warmup=1)
            assert code == 0 and X.shape == (n, S)
            assert cg.c.niterations == max(c["niterations"] for c in cols)
            for j, sigma in enumerate(shifts):
                cj, its, xj, csrj, norms = solvempi(sigma, maxits, tol)
                tag = (S, maxits, j, cols[j], its)
                assert cj == 0, tag
                if e.key == ("arrow", 1024) and cols[j]["niterations"] != its:
                    open_findings.append((tag, "iterations"))
                    continue
                assert cols[j]["niterations"] == its, tag
                if tol > 0:
                    assert cols[j]["converged"] == 1, tag
                elif _rounding_level(norms):
                    continue
                err = float(np.abs(X[:, j] - xj).max())
                if tol == 0 and e.key == ("arrow", 1024) and err > _xtol(e) * float(np.abs(xj).max()):
                    open_findings.append((tag, err, norms))
                    continue
                assert err <= _xtol(e) * float(np.abs(xj).max()), tag
                if tol > 0:
                    _check_solution(e.key, csrj, X[:, j], b, rtol * float(np.linalg.norm(b)), eps=sigma, ref_x=xj)
    finally:
        cg.free()
    if open_findings:
        pytest.xfail(OPEN_SHIFTED + repr(open_findings))


# ---------------------------------------------------------------------------------------------
# MINRES, mixed precision and Chebyshev PCG against their restatements


def _indefinite_shift(key):
    """sigma in the middle of the widest gap between consecutive eigenvalues (None for n = 1): A - sigma I
    has eigenvalues of both signs, none closer to 0 than half that gap -- the best-conditioned indefinite
    shift (on the arrow the two smallest eigenvalues are 1e-3 apart, its widest gap is about 1000)"""
    ev, ndist = _spectrum(key)
    if ndist < 2:
        return None
    k = int(np.argmax(np.diff(ev))) + 1
    return 0.5 * (float(ev[k - 1]) + float(ev[k]))


def _minres_runs(e, check_every):
    """(matrix shift, start, atol relative to ||r0||, rtol, maxits, warmup) of the MINRES comparisons of one
    entry"""
    runs = []
    sigma = _indefinite_shift(e.key)
    for eps in [0.0] + ([-sigma] if sigma is not None else []):
        runs.append((eps, "x0", 1e-10, 0.0, MAXITS, 2))
        runs.append((eps, "zero", 0.0, 1e-10, MAXITS, 0))
        runs += [(eps, "x0", 0.0, 0.0, m, 1) for m in _fixed_counts(e.key, check_every, eps)]
    return runs


@pytest.mark.gpu
@pytest.mark.parametrize("eid,optset", RUNS, ids=RUN_IDS)
def test_minres_against_restatement(eid, optset, ab, options):
    """MINRES against tests/minresref.py on the matrix (positive definite) and, from n = 2 on, on A - sigma I
    with sigma in the widest gap of the spectrum (eigenvalues of both signs): from a nonzero x0
    under an absolute tolerance (warm-up 2), from x0 = 0 under rtol 1e-10, and for fixed iteration counts;
    equal iteration counts and codes, x within 1e-10 relative, the converged solution against the dense
    solve."""
    e = BY_ID[eid]
    opts = OPTSETS[optset]
    options(**e.opts, **opts)
    n = _gen(e.key)[0]
    rng = np.random.default_rng(51)
    b, x0 = rng.standard_normal(n), rng.standard_normal(n)
    for eps, start, atol_rel, rtol, maxits, warmup in _minres_runs(e, opts.get("check_every", 8)):
        A = _matrix(ab, e.key, eps)
        csr = _csr(A)
        M = _scipy(csr)
        xi = x0 if start == "x0" else np.zeros(n)
        r0 = float(np.linalg.norm(b - M @ xi))
        atol = atol_rel * r0
        cg = ab.SolverCuda(A)
        try:
            _in_regime(cg, e)
            xv = _vec(A, xi)
            code = cg.solve_minres(_vec(A, b), xv, maxits=maxits, residualatol=atol, residualrtol=rtol, warmup=warmup)
            x = xv.x[:n]
        finally:
            cg.free()
        ref = minres(M, b, x0=xi, maxits=maxits, atol=atol, rtol=rtol)
        tag = (eps, start, maxits, code, cg.c.niterations, ref["niterations"], ref["stop"])
        assert code == ref["status"] == 0, tag
        if ref["niterations"] >= _spectrum(e.key, eps)[1] - 1:
            # a run into the last dimension of the Krylov space or past it: the residual there falls to rounding
            # level in one step or is driven by rounding, and the two may stop a step or two apart
            assert abs(cg.c.niterations - ref["niterations"]) <= 2, tag
        else:
            assert cg.c.niterations == ref["niterations"], tag
            if maxits == MAXITS or not _rounding_level(ref):
                assert float(np.abs(x - ref["x"]).max()) <= _xtol(e) * float(np.abs(ref["x"]).max()), tag
        if atol > 0 or rtol > 0:
            _check_solution(e.key, csr, x, b, max(atol, rtol * r0), eps=eps, ref_x=ref["x"])


@pytest.mark.gpu
@pytest.mark.parametrize("n", [2, 5, 8, 32, 33])
def test_minres_singular_consistent(n, ab, options):
    """MINRES on the singular 1-D chain with Neumann ends (null space: the constant vector) and b = A y for an
    integer y, so that b is exactly in the range, from x0 = 0 and from a random x0: against the restatement
    (counts, x within 1e-10), the true residual below 2 tol."""
    options()
    key = ("neumann", n)
    A = _matrix(ab, key)
    csr = _csr(A)
    M = _scipy(csr)
    rng = np.random.default_rng(57)
    y = rng.integers(-5, 6, n).astype(np.float64)
    b = M @ y
    assert abs(float(b.sum())) == 0.0
    x0 = rng.standard_normal(n)
    cg = ab.SolverCuda(A)
    try:
        for xi, rtol in ((np.zeros(n), 1e-10), (x0, 1e-10)):
            xv = _vec(A, xi)
            code = cg.solve_minres(_vec(A, b), xv, maxits=MAXITS, residualrtol=rtol)
            x = xv.x[:n]
            ref = minres(M, b, x0=xi, maxits=MAXITS, rtol=rtol)
            tag = (n, code, cg.c.niterations, ref["niterations"], ref["stop"])
            assert code == ref["status"] and cg.c.niterations == ref["niterations"], tag
            assert float(np.abs(x - ref["x"]).max()) <= 1e-10 * float(np.abs(ref["x"]).max()), tag
            r, _, _ = rows_exact(*csr, x, b)
            assert float(np.linalg.norm(r)) < 2 * rtol * ref["r0nrm2"], tag
    finally:
        cg.free()


@pytest.mark.gpu
@pytest.mark.parametrize("eid,optset", RUNS, ids=RUN_IDS)
def test_mixed_against_restatement(eid, optset, ab, options):
    """Mixed-precision CG against tests/mixedref.py, rtol 1e-8 from x0 = 0 and an absolute tolerance from a
    nonzero x0 with warm-up 2: counts within 2 CG steps and 1 reliable update (the dot products' order
    differs, as in test_gpu_mixed.py), rnrm2 the exact residual of x and below tol, x against the dense
    solve; fixed iteration counts: exactly that many steps, rnrm2 within 1e-6 of the restatement's."""
    e = BY_ID[eid]
    opts = OPTSETS[optset]
    options(**e.opts, **opts)
    A = _matrix(ab, e.key)
    n = A.c.nownedrows
    csr = _csr(A)
    M = _scipy(csr)
    rng = np.random.default_rng(61)
    b, x0 = rng.standard_normal(n), rng.standard_normal(n)
    r0 = float(np.linalg.norm(b - M @ x0))
    runs = [(np.zeros(n), 0.0, 1e-8, MAXITS, 0), (x0, 1e-10 * r0, 0.0, MAXITS, 2)]
    runs += [(x0, 0.0, 0.0, m, 1) for m in _fixed_counts(e.key, opts.get("check_every", 8))]
    cg = ab.SolverCuda(A)
    try:
        _in_regime(cg, e)
        for xi, atol, rtol, maxits, warmup in runs:
            xv = _vec(A, xi)
            code = cg.solve_mixed(_vec(A, b), xv, maxits=maxits, residualatol=atol, residualrtol=rtol, warmup=warmup)
            x = xv.x[:n]
            ref = mixed(M, b, x0=xi, maxits=maxits, atol=atol, rtol=rtol)
            its, upd = int(cg.c.niterations), int(cg.info()["mixed_reliable_updates"])
            tag = (atol, rtol, maxits, its, upd, ref["niterations"], ref["nupdates"], ref["stop"])
            assert code == ref["status"] == 0, tag
            r, _, _ = rows_exact(*csr, x, b)
            true = float(np.linalg.norm(r))
            assert cg.c.rnrm2 == pytest.approx(true, rel=1e-8, abs=1e-13 * max(cg.c.bnrm2, cg.c.r0nrm2)), tag
            if maxits < MAXITS:
                # fp32 vectors: the two part by the fp32 rounding of the steps, about 1e-7 of ||r0|| each
                assert its == ref["niterations"] == maxits and abs(upd - ref["nupdates"]) <= 1, tag
                assert abs(cg.c.rnrm2 - ref["rnrm2"]) <= 1e-6 * ref["rnrm2"] + 1e-5 * r0, tag
                continue
            assert abs(its - ref["niterations"]) <= 2 and abs(upd - ref["nupdates"]) <= 1 and upd >= 1, tag
            assert true < ref["tol"], tag
            _check_solution(e.key, csr, x, b, ref["tol"], ref_x=ref["x"])
    finally:
        cg.free()


@pytest.mark.gpu
@pytest.mark.parametrize("eid,optset", RUNS, ids=RUN_IDS)
def test_chebyshev_against_restatement(eid, optset, ab, options):
    """Chebyshev PCG against tests/chebref.py: degrees 0, 2 and 5 with the estimated interval (rtol 1e-8,
    x0 = 0), degrees 2 and 5 with a given interval (Gershgorin bound of D^-1 A) from a nonzero x0 under an
    absolute tolerance with warm-up 2, and degree 2 with the given interval for fixed iteration counts:
    equal iteration counts, estimate steps (at most n below 9 rows: the estimate stops when its space is
    exhausted), return codes and breakdown flags, the interval to 1e-8, x within 1e-10 relative, the
    converged solution against the dense solve.  On a diagonal matrix degree 0 (Jacobi) takes one step."""
    e = BY_ID[eid]
    opts = OPTSETS[optset]
    options(**e.opts, **opts)
    A = _matrix(ab, e.key)
    n = A.c.nownedrows
    csr = _csr(A)
    M = _scipy(csr)
    rng = np.random.default_rng(71)
    b, x0 = rng.standard_normal(n), rng.standard_normal(n)
    lmax = 1.1 * float(np.abs(sp.diags(1 / M.diagonal()) @ M).sum(axis=1).max())
    lmin = lmax / 40
    atol = 1e-9 * float(np.linalg.norm(b))
    runs = [dict(degree=d, maxits=MAXITS, residualrtol=1e-8) for d in (0, 2, 5)]
    runs += [dict(degree=d, lmin=lmin, lmax=lmax, maxits=MAXITS, residualatol=atol, warmup=2) for d in (2, 5)]
    runs += [dict(degree=2, lmin=lmin, lmax=lmax, maxits=m, warmup=1)
             for m in _fixed_counts(e.key, opts.get("check_every", 8), jacobi=True)]
    cg = ab.SolverCuda(A)
    try:
        _in_regime(cg, e)
        for kw in runs:
            xi = np.zeros(n) if "residualrtol" in kw else x0
            xv = _vec(A, xi)
            code = cg.solve_chebyshev(_vec(A, b), xv, **kw)
            x = xv.x[:n]
            ref = chebyshev(M, b, x0=xi, degree=kw["degree"], lmin=kw.get("lmin", 0.0), lmax=kw.get("lmax", 0.0),
                            maxits=kw["maxits"], atol=kw.get("residualatol", 0.0), rtol=kw.get("residualrtol", 0.0))
            inf = cg.info()
            got = (int(cg.c.niterations), int(inf["cheb_est_iterations"]) if kw["degree"] and "lmax" not in kw else 0, code)
            tag = (kw, got, ref["niterations"], ref["est_steps"], ref["stop"])
            assert got == (ref["niterations"], ref["est_steps"], ref["status"]) and code == 0, tag
            assert inf["cheb_breakdown"] == (ref["stop"] == "breakdown"), tag
            if n <= 8:
                assert ref["est_steps"] <= n, tag
            if kw["degree"] > 0:
                assert inf["cheb_lmax"] == pytest.approx(ref["lmax"], rel=1e-8), tag
                assert inf["cheb_lmin"] == pytest.approx(ref["lmin"], rel=1e-8), tag
            if kw["degree"] == 0 and e.key[0] == "diag":
                assert cg.c.niterations == 1, tag
            if ref["tol"] == 0 and _rounding_level(ref):
                continue
            assert float(np.abs(x - ref["x"]).max()) <= _xtol(e) * float(np.abs(ref["x"]).max()), tag
            if ref["tol"] > 0:
                _check_solution(e.key, csr, x, b, ref["tol"], ref_x=ref["x"])
    finally:
        cg.free()
