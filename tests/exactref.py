"""Exact reference for sparse products and dot products in FP64 (numpy + math.fsum).

Every product a*x of two doubles is split without error into p + e (Dekker's two_prod on
Veltkamp's split), and math.fsum adds any list of doubles with a single rounding at the end.
So `rows_exact` returns the correctly rounded value of sum_j a_ij x_j (or of b_i - sum_j a_ij x_j)
for every row: the value a kernel would produce with infinitely precise arithmetic followed by
one rounding.  A kernel result is then checked against it with a rigorous error bound instead of
an empirical tolerance: a sum of m products in any order is within gamma(m) * sum|a_ij x_j| of
the exact value (Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., eq. 3.5).

Valid as long as no product over- or underflows (|a x| well inside [2^-969, 2^1023]); the GPU
tests use data far from both ends.
"""
import math

import numpy as np

U = 2.0 ** -53                 # unit roundoff of IEEE binary64
_SPLITTER = 134217729.0        # 2^27 + 1


def _split(a):
    c = _SPLITTER * a
    hi = c - (c - a)
    return hi, a - hi


def two_prod(a, b):
    """p, e with p = fl(a*b) and a*b = p + e exactly (elementwise, numpy arrays or scalars)."""
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    p = a * b
    ah, al = _split(a)
    bh, bl = _split(b)
    e = ((ah * bh - p) + ah * bl + al * bh) + al * bl
    return p, e


def gamma(m):
    """gamma(m) = m u / (1 - m u): bound of the relative error of m floating-point operations."""
    mu = np.asarray(m, np.float64) * U
    return mu / (1.0 - mu)


def rows_exact(rowptr, colidx, vals, x, b=None):
    """Per row i of the CSR matrix: the correctly rounded value of sum_j a_ij x_j (b is None) or of
    b_i - sum_j a_ij x_j, the scale sum_j |a_ij x_j| (+ |b_i|), and the row length m_i.
    Returns (value, scale, m) as float64, float64, int64 arrays."""
    rowptr = np.asarray(rowptr, np.int64)
    n = len(rowptr) - 1
    m = np.diff(rowptr)
    xv = np.asarray(x, np.float64)[np.asarray(colidx[:rowptr[-1]], np.int64)]
    p, e = two_prod(np.asarray(vals[:rowptr[-1]], np.float64), xv)
    rows = np.repeat(np.arange(n), m)
    scale = np.bincount(rows, weights=np.abs(p), minlength=n).astype(np.float64)
    pl, el = p.tolist(), e.tolist()
    rp = rowptr.tolist()
    out = np.empty(n, np.float64)
    if b is None:
        for i in range(n):
            k0, k1 = rp[i], rp[i + 1]
            out[i] = math.fsum(pl[k0:k1] + el[k0:k1])
    else:
        bl = np.asarray(b, np.float64).tolist()
        for i in range(n):
            k0, k1 = rp[i], rp[i + 1]
            out[i] = -math.fsum([-bl[i]] + pl[k0:k1] + el[k0:k1])
        scale += np.abs(np.asarray(b, np.float64))
    return out, scale, m


def _two_sum(a, b):
    """s, t with s = fl(a + b) and a + b = s + t exactly (Knuth's TwoSum, elementwise)."""
    s = a + b
    z = s - a
    return s, (a - (s - z)) + (b - z)


def rows_dd(rowptr, colidx, vals, x, b=None, chunk=1 << 16, long_row=64):
    """rows_exact for large matrices: per row the value of sum_j a_ij x_j (or b_i - sum_j a_ij x_j)
    accumulated in double-double and rounded once, the scale sum_j |a_ij x_j| (+ |b_i|), and m_i.

    Rows are taken in chunks; in a chunk, entry e of every row at once (ELL-like from rowptr): the
    product split by two_prod, the high part added by TwoSum and both low parts into a second word
    (Ogita, Rump and Oishi, Accurate sum and dot product, SIAM J. Sci. Comput. 26 (2005), Dot2).
    So, with b_i counted as one more term, |value - exact| <= u |exact| + gamma(m_i + 1)^2 * scale
    (ibid., Proposition 5.5): exact for integer data whose partial sums stay below 2^53, within a few
    units of u^2 * scale otherwise.  Rows longer than `long_row` (hubs) go through math.fsum instead,
    correctly rounded."""
    rowptr = np.asarray(rowptr, np.int64)
    n = len(rowptr) - 1
    m = np.diff(rowptr)
    xv = np.asarray(x, np.float64)
    out = np.empty(n, np.float64)
    scale = np.zeros(n, np.float64)
    bb = None if b is None else np.asarray(b, np.float64)
    for i0 in range(0, n, chunk):
        i1 = min(n, i0 + chunk)
        start, mc = rowptr[i0:i1], m[i0:i1]
        hi = np.zeros(i1 - i0) if bb is None else bb[i0:i1].copy()
        lo = np.zeros(i1 - i0)
        sc = np.zeros(i1 - i0) if bb is None else np.abs(bb[i0:i1])
        short = mc <= long_row
        for e in range(int(mc[short].max()) if short.any() else 0):
            idx = np.flatnonzero(short & (mc > e))
            k = start[idx] + e
            p, err = two_prod(np.asarray(vals[k], np.float64), xv[np.asarray(colidx[k], np.int64)])
            if bb is not None:
                p, err = -p, -err
            hi[idx], t = _two_sum(hi[idx], p)
            lo[idx] += t + err
            sc[idx] += np.abs(p)
        out[i0:i1] = hi + lo
        scale[i0:i1] = sc
        for j in np.flatnonzero(~short):
            i = i0 + int(j)
            v, s, _ = rows_exact(rowptr[i:i + 2] - rowptr[i], colidx[rowptr[i]:rowptr[i + 1]],
                                 vals[rowptr[i]:rowptr[i + 1]], xv, None if bb is None else bb[i:i + 1])
            out[i], scale[i] = v[0], s[0]
    return out, scale, m


def dot_exact(x, y):
    """The correctly rounded value of sum_i x_i y_i."""
    p, e = two_prod(np.asarray(x, np.float64).ravel(), np.asarray(y, np.float64).ravel())
    return math.fsum(p.tolist() + e.tolist())
