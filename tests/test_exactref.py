"""tests/exactref.py against exact rational arithmetic (CPU).  The GPU tests of the SpMV kernels
trust this helper for their reference values, so it is checked on its own first."""
from fractions import Fraction

import numpy as np
import pytest

from exactref import U, dot_exact, gamma, rows_exact, two_prod


def _fr_rows(rowptr, colidx, vals, x, b=None):
    out = []
    for i in range(len(rowptr) - 1):
        s = sum((Fraction(float(vals[k])) * Fraction(float(x[colidx[k]])) for k in range(rowptr[i], rowptr[i + 1])),
                Fraction(0))
        out.append(Fraction(float(b[i])) - s if b is not None else s)
    return out


def _random_csr(rng, n, maxlen, scale_fn=None):
    lens = rng.integers(0, maxlen + 1, n)
    lens[0] = 0                                   # an empty row
    rowptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    colidx = rng.integers(0, n, rowptr[-1]).astype(np.int32)
    vals = rng.standard_normal(rowptr[-1]) if scale_fn is None else scale_fn(rowptr[-1])
    return rowptr, colidx, vals


def _check_rows(rowptr, colidx, vals, x, b=None):
    got, scale, m = rows_exact(rowptr, colidx, vals, x, b)
    want = _fr_rows(rowptr, colidx, vals, x, b)
    for i, w in enumerate(want):
        assert got[i] == float(w), (i, got[i], float(w))            # float(Fraction) rounds to nearest
        s = sum(abs(float(vals[k]) * float(x[colidx[k]])) for k in range(rowptr[i], rowptr[i + 1]))
        s += abs(float(b[i])) if b is not None else 0.0
        assert scale[i] == pytest.approx(s, rel=1e-12)
    assert np.array_equal(m, np.diff(rowptr))


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_two_prod_is_exact(seed):
    rng = np.random.default_rng(seed)
    a = rng.standard_normal(2000) * 2.0 ** rng.integers(-40, 40, 2000)
    b = rng.standard_normal(2000) * 2.0 ** rng.integers(-40, 40, 2000)
    p, e = two_prod(a, b)
    for ai, bi, pi, ei in zip(a, b, p, e):
        assert Fraction(float(pi)) + Fraction(float(ei)) == Fraction(float(ai)) * Fraction(float(bi))
        assert pi == ai * bi


@pytest.mark.parametrize("seed", [0, 1])
def test_rows_random(seed):
    rng = np.random.default_rng(seed)
    rowptr, colidx, vals = _random_csr(rng, 300, 40)
    x = rng.standard_normal(300)
    _check_rows(rowptr, colidx, vals, x)
    _check_rows(rowptr, colidx, vals, x, rng.standard_normal(300))


def test_rows_catastrophic_cancellation():
    """Terms that cancel to far below their size: naive float64 sums are wrong in every digit."""
    rng = np.random.default_rng(3)
    n, L = 50, 30
    rowptr = np.arange(0, n * L + 1, L, dtype=np.int64)
    colidx = np.tile(np.arange(L, dtype=np.int32), n)
    x = rng.standard_normal(L) * 2.0 ** rng.integers(-20, 20, L)
    vals = np.empty(n * L)
    for i in range(n):
        v = rng.standard_normal(L)
        v[-1] = -float(sum(Fraction(float(v[k])) * Fraction(float(x[k])) for k in range(L - 1)) / Fraction(float(x[-1])))
        vals[i * L:(i + 1) * L] = v
    got, scale, _ = rows_exact(rowptr, colidx, vals, x)
    assert np.all(np.abs(got) < 1e-10 * scale)             # really cancelled
    _check_rows(rowptr, colidx, vals, x)
    # b - A x with b equal to A x up to rounding: cancellation in the subtraction too
    naive = np.array([vals[i * L:(i + 1) * L] @ x for i in range(n)])
    _check_rows(rowptr, colidx, vals, x, naive)


@pytest.mark.parametrize("e", [50, -50])
def test_rows_extreme_exponents(e):
    rng = np.random.default_rng(4)
    rowptr, colidx, vals = _random_csr(rng, 120, 25, lambda k: rng.standard_normal(k) * 2.0 ** e)
    x = rng.standard_normal(120) * 2.0 ** e
    _check_rows(rowptr, colidx, vals, x)
    _check_rows(rowptr, colidx, vals, x, rng.standard_normal(120) * 2.0 ** (2 * e))


def test_rows_integer_data_are_exact_sums():
    rng = np.random.default_rng(5)
    rowptr, colidx, vals = _random_csr(rng, 200, 60, lambda k: rng.integers(-7, 8, k).astype(np.float64))
    x = rng.integers(-9, 10, 200).astype(np.float64)
    b = rng.integers(-50, 51, 200).astype(np.float64)
    got, _, _ = rows_exact(rowptr, colidx, vals, x, b)
    want = np.array([b[i] - int(vals[rowptr[i]:rowptr[i + 1]].astype(np.int64) @ x[colidx[rowptr[i]:rowptr[i + 1]]].astype(np.int64))
                     for i in range(200)], np.float64)
    assert np.array_equal(got, want)
    _check_rows(rowptr, colidx, vals, x, b)


@pytest.mark.parametrize("kind", ["random", "cancel", "tiny", "huge"])
def test_dot_exact(kind):
    rng = np.random.default_rng(6)
    x = rng.standard_normal(3000)
    y = rng.standard_normal(3000)
    if kind == "cancel":
        y = np.concatenate([y[:1500], -y[:1500]]); x = np.concatenate([x[:1500], x[:1500] * (1 + 2.0 ** -40)])
    elif kind == "tiny":
        x *= 2.0 ** -50; y *= 2.0 ** -50
    elif kind == "huge":
        x *= 2.0 ** 50; y *= 2.0 ** 50
    want = sum((Fraction(float(a)) * Fraction(float(b)) for a, b in zip(x, y)), Fraction(0))
    assert dot_exact(x, y) == float(want)


def test_gamma():
    assert U == 2.0 ** -53
    assert gamma(1) == pytest.approx(U, rel=1e-15)
    assert gamma(28) == pytest.approx(28 * U / (1 - 28 * U), rel=1e-15)
    assert np.all(np.diff(gamma(np.arange(1, 100))) > 0)
