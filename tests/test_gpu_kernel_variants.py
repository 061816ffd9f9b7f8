"""Every instantiated SpMV kernel shape in every epilogue mode against an exact reference.

The SpMV has three epilogue modes and every kernel carries its own copy of them:
* mode 0, y = A x (the pipelined loop's product);
* mode 1, y = A x with the fused x.y (classic CG's p.Ap);
* mode 2, r = b - A x with the fused r.r (the set-up residual r0 = b - A x0).
Each kernel is forced in turn through the plan options and checked in all three modes through
acgsolvercuda_spmv_mode.  The kernels are the tile kernel (every (G, T, U) of spmv_variant), the
slice kernel (every (UB, T) of slice_variant, plain and EXC), the merge-path kernel plus its fix-up
(every merge_variant), the medium-row kernel and the long-row kernels.  Two data sets are used:

* integer-exact: small integers in A, x and b, so that every partial sum is exact in FP64 whatever
  the order or the atomics -- y, r and both fused dots must equal the exact value BITWISE, and a
  dropped, duplicated or mis-signed term cannot hide in a tolerance;
* random real, compared with the correctly rounded value from tests/exactref.py under the rigorous
  bound 2 gamma(m_i + 1) sum_j |a_ij x_j| (+ |b_i|) per row; in mode 2 b = A x + 1e-8 noise, so the
  subtraction cancels heavily.

Each shape also runs with one CTA per SM and 1, 2, 3 and 8 pipeline stages on a plan with at least
twice grid x stages tiles, so every CTA walks its TMA ring at least twice (stage reuse, the mbarrier
parity flip, the re-issue after __syncthreads), and with more rows per tile than a CTA covers in
one pass.
"""
import functools
import os
import re

import numpy as np
import pytest

from acg_b200 import matgen as mg
from exactref import dot_exact, gamma, rows_exact

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# The shapes kernels.cu instantiates (spmv_variant, slice_variant, merge_variant).
# test_variant_lists_match_kernels_cu keeps these lists in step with the source.
TILE_VARIANTS = [(1, 128, 4), (1, 128, 16), (1, 256, 16), (2, 256, 4), (2, 256, 16), (4, 512, 4), (4, 128, 4),
                 (4, 256, 4),
                 (1, 64, 8), (2, 64, 8), (4, 64, 8), (8, 128, 8), (16, 128, 8), (32, 128, 8), (1, 128, 8),
                 (1, 256, 8), (2, 128, 8), (2, 256, 8), (2, 512, 8), (4, 128, 8), (4, 256, 8), (4, 512, 8),
                 (8, 256, 8), (8, 512, 8), (16, 256, 8), (16, 512, 8), (32, 256, 8), (32, 512, 8)]
SLICE_VARIANTS = [(5, 128), (7, 128), (8, 128), (9, 128), (7, 256), (8, 256), (9, 256)]
MERGE_VARIANTS = [(128, 8), (256, 4)]          # (threads, products in flight per thread)

STAGES = (1, 2, 3, 8)
HUB = 6200                                     # longer than the largest default tile (6144 nonzeros): long-row path
DEFAULTS = {"spmv_lanes": 0, "spmv_threads": 0, "spmv_unroll": 0, "spmv_rows_cap": 0, "spmv_nnz_cap": 0,
            "spmv_stages": 0, "spmv_max_ctas": 0, "spmv_slices": 1, "slice_ub": 0, "slice_threads": 0,
            "slice_max_ctas": 0, "spmv_merge": -1, "merge_items": 0, "merge_threads": 0, "merge_max_ctas": 0,
            "merge_stages": 0, "spmv_medium": 0}


def _vid(v):
    return "-".join(str(e) for e in v)


# ---------------------------------------------------------------------------------------------
# the variant lists against the source (CPU)


def test_variant_lists_match_kernels_cu():
    src = open(os.path.join(ROOT, "acg_b200", "csrc", "kernels.cu")).read()
    tiles = set()
    body = src[src.index("static spmv_fn spmv_variant("):]
    body = body[:body.index("\n}\n")]
    tiles |= {tuple(map(int, m)) for m in re.findall(r"spmv_tiles_kernel<(\d+), (\d+), (\d+)>", body)}
    macro = src[src.index("#define SPMV_VARIANTS(X)"):]
    macro = macro[:macro.index("\n\n")]
    pairs = re.findall(r"X\((\d+), (\d+)\)", macro)
    assert pairs and "spmv_tiles_kernel<g, t, 8>" in body
    tiles |= {(int(g), int(t), 8) for g, t in pairs}
    assert tiles == set(TILE_VARIANTS) and len(TILE_VARIANTS) == len(set(TILE_VARIANTS)) == 28
    body = src[src.index("static slice_fn slice_variant("):]
    body = body[:body.index("\n}\n")]
    assert "spmv_slices_kernel<u, t, true> : spmv_slices_kernel<u, t, false>" in body
    assert {tuple(map(int, m)) for m in re.findall(r"X\((\d+), (\d+)\)", body)} == set(SLICE_VARIANTS)
    body = src[src.index("static merge_fn merge_variant("):]
    body = body[:body.index("\n}\n")]
    got = {(int(t), int(t2), int(u)) for t, t2, u in re.findall(r"T == (\d+)\) return spmv_merge_kernel<(\d+), (\d+)>", body)}
    assert all(t == t2 for t, t2, _ in got)
    assert {(t, u) for t, _, u in got} == set(MERGE_VARIANTS)


# ---------------------------------------------------------------------------------------------
# matrices (upper triangle, row-sorted COO; values filled in per data set)


def _coo(n, rows, cols):
    rows = np.asarray(rows, np.int64); cols = np.asarray(cols, np.int64)
    lo, hi = np.minimum(rows, cols), np.maximum(rows, cols)
    key = np.unique(lo * n + hi)
    return n, (key // n).astype(np.int32), (key % n).astype(np.int32)


def _cliques(r0, sizes):
    """Dense diagonal blocks of the given sizes from row r0 on (size 0: an empty row)."""
    rows, cols = [], []
    r = r0
    for s in sizes:
        if s > 0:
            iu, ju = np.triu_indices(s)
            rows.append(r + iu); cols.append(r + ju)
        r += max(s, 1)
    return r, rows, cols


@functools.lru_cache(maxsize=None)
def ragged(ug, tail):
    """Row lengths 0, 1, UG-1, UG, UG+1, 2UG next to each other, then short rows (1-4 entries, empty
    rows) up to ~9000 rows, and one hub row of HUB entries (a long row; its partners get one more).
    n = 1, 2 or 3 (mod 4) by `tail`, never a multiple of 32."""
    rng = np.random.default_rng(ug * 7 + tail)
    sizes = [0, 1, ug - 1, 0, ug, 1, ug + 1, 0, 2 * ug, 1, 1]
    sizes += list(rng.choice([0, 1, 1, 2, 3, 4], 4000))
    r, rows, cols = _cliques(0, sizes)
    n = max(r, HUB + 1000)
    n += (tail - n) % 4
    assert n % 4 == tail and n % 32
    hub = n - 500
    partners = rng.choice(np.setdiff1d(np.arange(n), [hub]), HUB - 1, replace=False)
    rows.append(np.full(HUB - 1, hub)); cols.append(partners)
    rows.append(np.arange(r, n)); cols.append(np.arange(r, n))          # diagonal for the rows after the cliques
    return _coo(n, np.concatenate(rows), np.concatenate(cols))


@functools.lru_cache(maxsize=None)
def slice_matrix(exc):
    """Regions of 32 s rows made of cliques of size s, s = 1..18: 32-row slices with every longest
    row length L = 1..18, so L takes every residue modulo every batch width UB; then a 27-point
    stencil on a 7 x 6 x 5 box whose last rows do not fill a slice (ragged end).  With `exc`, one row
    in every 16 also gets a coupling at an offset no other row has (both ends of it): hundreds of
    patterns that each occur once, so the pattern table overflows and those rows stay in their
    slices as exception rows."""
    rows, cols = [], []
    r = 0
    for s in range(1, 19):
        r, rr, cc = _cliques(r, [s] * 32)
        rows += rr; cols += cc
    m, sr, sc, _ = mg.stencil3d_27pt(7, 6, 5)
    rows.append(sr.astype(np.int64) + r); cols.append(sc.astype(np.int64) + r)
    n = r + m
    if exc:
        a = np.arange(3, n // 2, 16)
        d = n // 2 + np.arange(len(a))                  # distinct offsets
        keep = a + d < n
        rows.append(a[keep]); cols.append(a[keep] + d[keep])
    return _coo(n, np.concatenate(rows), np.concatenate(cols))


@functools.lru_cache(maxsize=None)
def big_stencil(exc):
    """27-point stencil on 47 x 48 x 33 (2326 full slices and a ragged end), with `exc` one row in 64
    coupled at an offset of its own: enough slices for every warp of a one-CTA-per-SM grid to take
    several."""
    n, r, c, _ = mg.stencil3d_27pt(47, 48, 33)
    rows, cols = [r.astype(np.int64)], [c.astype(np.int64)]
    if exc:
        a = np.arange(5, n // 2, 64)
        d = n // 2 + np.arange(len(a))
        keep = a + d < n
        rows.append(a[keep]); cols.append(a[keep] + d[keep])
    return _coo(n, np.concatenate(rows), np.concatenate(cols))


@functools.lru_cache(maxsize=None)
def rmat():
    n, r, c, _ = mg.rmat_spd(30000, 600000, seed=8)
    return n, r, c


# ---------------------------------------------------------------------------------------------
# data sets and exact references


class Case:
    """One matrix structure with its two data sets: values, inputs, and the exact answers of the
    three modes (computed once, shared by every plan the matrix is run with)."""

    def __init__(self, ab, n, r, c, seed):
        self.n = n
        rng = np.random.default_rng(seed)
        diag = r == c
        self.data = {}
        for kind in ("int", "real"):
            if kind == "int":
                v = rng.integers(-3, 4, len(r)).astype(np.float64)
                v[diag] = rng.integers(1, 9, int(diag.sum()))
                x = rng.integers(-3, 4, n).astype(np.float64)
                b = rng.integers(-40, 41, n).astype(np.float64)
            else:
                v = rng.standard_normal(len(r))
                v[diag] += 4.0
                x = rng.standard_normal(n)
                b = None
            A = ab.SymCsrMatrix.init_real_double(n, r, c, v).dsymv_init(0.0)
            csr = (A.frowptr.copy(), A.fcolidx.copy(), A.fa.copy())
            y, scale, m = rows_exact(*csr, x)
            if b is None:                              # b = A x + tiny noise: b - A x cancels to ~1e-8
                b = y + 1e-8 * rng.standard_normal(n)
            rr, rscale, _ = rows_exact(*csr, x, b)
            self.data[kind] = dict(A=A, csr=csr, x=x, b=b, m=m, exact={0: (y, scale), 1: (y, scale), 2: (rr, rscale)})

    def free(self):
        for d in self.data.values():
            d["A"].free()


def check(cg, case, kind, modes=(0, 1, 2), paths=(0,), what=""):
    d = case.data[kind]
    x, b, m = d["x"], d["b"], d["m"]
    for mode in modes:
        want, scale = d["exact"][mode]
        for path in paths:
            tag = (what, kind, mode, path)
            y, dot = cg.spmv_mode(mode, x, b if mode == 2 else None, path)
            assert not np.isnan(y).any(), tag
            if kind == "int":
                bad = np.flatnonzero(y != want)
                assert bad.size == 0, (tag, bad[:10], y[bad[:10]], want[bad[:10]])
            else:
                err = np.abs(y - want)
                bound = 2.0 * gamma(m + 1) * scale
                bad = np.flatnonzero(err > bound)
                assert bad.size == 0, (tag, bad[:10], err[bad[:10]], bound[bad[:10]])
            # the fused dot against the exact dot of the vectors the device returned
            if mode == 0:
                assert dot == 0.0, tag
                continue
            u = x if mode == 1 else y
            wdot = dot_exact(u, y)
            if kind == "int":
                assert dot == wdot, (tag, dot, wdot)
            else:
                assert abs(dot - wdot) <= 2.0 * gamma(case.n) * float(np.abs(u * y).sum()), (tag, dot, wdot)


@pytest.fixture
def options(ab):
    """set_option for the plan of the next SolverCuda; every option back to its default afterwards."""
    touched = set()

    def set_(**kw):
        for k, v in kw.items():
            touched.add(k)
            ab.set_option(k, v)
    yield set_
    for k in touched:
        ab.set_option(k, DEFAULTS[k])


def _solver(ab, case, kind, set_, opts):
    set_(**{k: DEFAULTS[k] for k in DEFAULTS})
    set_(**opts)
    return ab.SolverCuda(case.data[kind]["A"])


_CASES = {}


def _case(ab, key, gen, seed):
    if key not in _CASES:
        n, r, c = gen()
        _CASES[key] = Case(ab, n, r, c, seed)
    return _CASES[key]


def teardown_module(module):
    for c in _CASES.values():
        c.free()
    _CASES.clear()


# ---------------------------------------------------------------------------------------------
# tile kernel: spmv_tiles_kernel<G, T, U>


def _stage_bytes(nnz_cap, rows_cap):
    return ((((nnz_cap + 8 + 3) & ~3) * 12 + ((rows_cap + 1 + 8 + 3) & ~3) * 4 + 127) & ~127)


@pytest.mark.gpu
@pytest.mark.parametrize("variant", TILE_VARIANTS, ids=[_vid(v) for v in TILE_VARIANTS])
def test_tile_variant_all_modes(variant, ab, options):
    G, T, U = variant
    ug = U * G
    k = TILE_VARIANTS.index(variant)
    case = _case(ab, ("ragged", ug, k % 3 + 1), lambda: ragged(ug, k % 3 + 1), seed=k)
    lens = np.diff(case.data["int"]["csr"][0])
    for want in (0, 1, ug - 1, ug, ug + 1, 2 * ug):
        assert (lens == want).any(), want
    base = dict(spmv_slices=0, spmv_merge=0, spmv_lanes=G, spmv_threads=T, spmv_unroll=U)
    rpp = T // G

    # the planner's tile sizes with this shape (one pass per tile), both data sets, both device paths
    for kind in ("int", "real"):
        cg = _solver(ab, case, kind, options, dict(base, spmv_rows_cap=rpp))
        inf = cg.info()
        assert (inf["spmv_lanes_per_row"], inf["spmv_threads"], inf["spmv_unroll"]) == variant
        assert inf["spmv_slices"] == 0 and inf["spmv_merge_tiles"] == 0 and inf["spmv_nlong"] >= 1
        check(cg, case, kind, paths=(0, 1), what="plan")
        cg.free()

    # one CTA per SM, two rows per tile: every CTA walks its ring of S stages at least twice
    rp = case.data["int"]["csr"][0]
    maxlen = int(np.sort(lens)[-2])                  # longest row that is not the hub
    nnz_cap = (2 * maxlen + 3) & ~3
    for S in STAGES:
        opts = dict(base, spmv_rows_cap=2, spmv_nnz_cap=nnz_cap, spmv_stages=S, spmv_max_ctas=1)
        for kind in ("int", "real") if S == 3 else ("int",):
            cg = _solver(ab, case, kind, options, opts)
            inf = cg.info()
            assert (inf["spmv_lanes_per_row"], inf["spmv_threads"], inf["spmv_unroll"], inf["spmv_stages"]) == variant + (S,)
            assert inf["spmv_grid"] <= inf["num_sms"] and inf["spmv_ntiles"] >= 2 * inf["spmv_grid"] * S, inf
            if S == 1:
                # tiles start at every offset inside a 16-byte line (the TMA copies start at k & ~3)
                tiles = ab.spmv_plan_host(rp)["tiles"]
                assert len(tiles) == inf["spmv_ntiles"] and set((rp[tiles[:, 0]] & 3).tolist()) == {0, 1, 2, 3}
            check(cg, case, kind, what=f"ring{S}")
            cg.free()

    # more rows per tile than the CTA's groups: a tile takes several passes
    rows_cap = 2 * rpp + 1
    nnz_cap = (rows_cap * (2 * ug + 2) + 3) & ~3
    while _stage_bytes(nnz_cap, rows_cap) > 200 * 1024:
        nnz_cap = (nnz_cap // 2 + 3) & ~3
    cg = _solver(ab, case, "int", options, dict(base, spmv_rows_cap=rows_cap, spmv_nnz_cap=nnz_cap, spmv_stages=1,
                                                spmv_max_ctas=1))
    inf = cg.info()
    assert inf["spmv_rows_cap"] == rows_cap > rpp
    tiles = ab.spmv_plan_host(rp)["tiles"]
    assert len(tiles) == inf["spmv_ntiles"] and tiles[:, 1].max() > rpp      # some tile takes 2-3 passes
    check(cg, case, "int", paths=(0, 1), what="passes")
    cg.free()


# ---------------------------------------------------------------------------------------------
# slice kernel: spmv_slices_kernel<UB, T, EXC>


SLICE_IDS = [f"{_vid(v)}-{'exc' if e else 'plain'}" for e in (False, True) for v in SLICE_VARIANTS]


@pytest.mark.gpu
@pytest.mark.parametrize("variant,exc", [(v, e) for e in (False, True) for v in SLICE_VARIANTS], ids=SLICE_IDS)
def test_slice_variant_all_modes(variant, exc, ab, options):
    UB, T = variant
    case = _case(ab, ("slices", exc), lambda: slice_matrix(exc), seed=100 + exc)
    n = case.n
    assert n % 4 and n % 32
    rp, ci, _ = case.data["int"]["csr"]
    Ls = ab.slices_host(rp, ci)["slices"][:, 2]
    base = dict(spmv_merge=0, slice_ub=UB, slice_threads=T)
    for kind in ("int", "real"):
        cg = _solver(ab, case, kind, options, base)
        inf = cg.info()
        assert inf["spmv_slices"] > 0 and inf["spmv_slice_ub"] == UB and inf["spmv_slice_threads"] == T
        assert (inf["spmv_slice_exc"] > 0) == exc, inf["spmv_slice_exc"]
        assert inf["spmv_ntiles"] > 0                              # the ragged end is in tiles
        check(cg, case, kind, paths=(0, 1), what="plan")
        cg.free()
    assert set(int(L) % UB for L in Ls) == set(range(UB))
    # one CTA per SM on a larger matrix: each warp walks at least two slices
    big = _case(ab, ("big", exc), lambda: big_stencil(exc), seed=110 + exc)
    cg = _solver(ab, big, "int", options, dict(base, slice_max_ctas=1))
    inf = cg.info()
    assert inf["spmv_slice_ub"] == UB and inf["spmv_slice_threads"] == T and (inf["spmv_slice_exc"] > 0) == exc
    assert inf["spmv_slice_grid"] <= inf["num_sms"] and inf["spmv_slices"] >= 2 * inf["spmv_slice_grid"] * (T // 32), inf
    check(cg, big, "int", what="onecta")
    cg.free()


# ---------------------------------------------------------------------------------------------
# merge-path kernel + fix-up: spmv_merge_kernel<T, U>, spmv_merge_fix_kernel


@pytest.mark.gpu
@pytest.mark.parametrize("variant", MERGE_VARIANTS, ids=[_vid(v) for v in MERGE_VARIANTS])
@pytest.mark.parametrize("matrix", ["rmat", "ragged"])
def test_merge_variant_all_modes(variant, matrix, ab, options):
    T, _ = variant
    if matrix == "rmat":
        case, items = _case(ab, ("rmat",), rmat, seed=200), 128
    else:
        case, items = _case(ab, ("ragged", 256, 2), lambda: ragged(256, 2), seed=201), 64
    base = dict(spmv_merge=1, spmv_slices=0, merge_threads=T)
    for kind in ("int", "real"):
        cg = _solver(ab, case, kind, options, dict(base, merge_items=1024))
        inf = cg.info()
        assert inf["spmv_merge_threads"] == T and inf["spmv_merge_tiles"] > 0 and inf["spmv_merge_rows"] == case.n
        assert inf["spmv_merge_split"] > 0                       # hubs span several tiles
        check(cg, case, kind, paths=(0, 1), what="plan")
        cg.free()
    # one CTA per SM, small tiles (most rows cut): every CTA walks its ring of S stages at least twice
    for S in STAGES:
        for kind in ("int", "real") if S == 2 else ("int",):
            cg = _solver(ab, case, kind, options, dict(base, merge_items=items, merge_stages=S, merge_max_ctas=1))
            inf = cg.info()
            assert inf["spmv_merge_stages"] == S and inf["spmv_merge_grid"] <= inf["num_sms"]
            assert inf["spmv_merge_tiles"] >= 2 * inf["spmv_merge_grid"] * S, inf
            check(cg, case, kind, what=f"ring{S}")
            cg.free()


# ---------------------------------------------------------------------------------------------
# medium rows (a warp each) and long rows (partial + finish kernels)


@pytest.mark.gpu
def test_medium_and_long_rows_all_modes(ab, options):
    case = _case(ab, ("rmat",), rmat, seed=200)
    for kind in ("int", "real"):
        cg = _solver(ab, case, kind, options, dict(spmv_medium=96, spmv_merge=0, spmv_slices=0))
        inf = cg.info()
        assert inf["spmv_nmedium"] > 0 and inf["spmv_nlong"] > 0 and inf["spmv_merge_tiles"] == 0
        check(cg, case, kind, paths=(0, 1), what="medium+long")
        cg.free()
