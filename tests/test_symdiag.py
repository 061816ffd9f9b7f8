"""Host plan of the mirrored diagonals (acg_b200/csrc/slices.c, acgb200_symdiag_host), CPU only.

The slice-covered rows of a symmetric matrix can read every stored value once: the upper diagonals D of
the covered rows' offsets O are stored for every owned row, and a lower entry a[i, i+o] (o < 0) is read
from its mirror row as a[i+o, i].  These tests check the accept/reject decision and O and D, and emulate
spmv_symdiag_kernel's addressing in numpy from the hook's output: every covered row's (value, column)
pairs, with the slots of offsets the row does not have dropped, must be the row's CSR sequence bit for
bit, and the dropped slots must hold +0.0 -- so the kernel's FMA chain is the slice kernel's.  The kernel
itself runs on the H100 in tests/test_gpu_symdiag.py."""
import numpy as np
import pytest

from acg_b200 import matgen as mg


def _full(ab, n, r, c, v=None, seed=0):
    if v is None:
        v = np.random.default_rng(seed).standard_normal(len(r))
        v[r == c] += 30.0
    A = ab.SymCsrMatrix.init_real_double(n, r, c, v).dsymv_init(0.0)
    out = n, A.frowptr.copy(), A.fcolidx.copy(), A.fa.copy()
    A.free()
    return out


def _stencil_offsets(kind, nx, ny):
    rng = (-1, 0, 1)
    if kind == 27:
        offs = {dz * nx * ny + dy * nx + dx for dx in rng for dy in rng for dz in rng}
    else:
        offs = {0, 1, -1, nx, -nx, nx * ny, -nx * ny}
    return np.array(sorted(offs))


def emulate(n, rp, col, a, sd, covered_rows):
    """The stored diagonals as acgb200_slices_fill makes them, and every covered row's products as
    spmv_symdiag_kernel forms them; asserts they are the row's CSR (value, column) sequence."""
    D, margin, stride = sd["D"], sd["margin"], sd["stride"]
    assert margin % 32 == 0 and stride % 32 == 0 and margin >= D.max() and stride >= margin + n
    hval = np.zeros(len(D) * stride)
    rows = np.repeat(np.arange(n), np.diff(rp))
    d = col - rows
    keep = np.isin(d, D)
    hval[np.searchsorted(D, d[keep]) * stride + margin + rows[keep]] = a[keep]
    i = np.asarray(covered_rows)
    V = hval[sd["voff"][None, :] + i[:, None]]                       # [rows, |O|]
    C = np.clip(i[:, None] + sd["coff"][None, :], 0, n - 1)
    # the row's own entries: slot of each nonzero in O; ascending slots = the row's CSR order
    lens = np.diff(rp)[i]
    k = np.concatenate([np.arange(rp[r], rp[r + 1]) for r in i])
    owner = np.repeat(np.arange(len(i)), lens)
    slot = np.searchsorted(sd["O"], col[k] - i[owner])
    assert np.array_equal(sd["O"][slot], col[k] - i[owner])         # every offset of a covered row is in O
    assert (np.diff(slot)[np.diff(owner) == 0] > 0).all()
    M = np.zeros(V.shape, bool)
    M[owner, slot] = True
    assert np.array_equal(V[owner, slot].view(np.int64), a[k].view(np.int64))
    assert np.array_equal(C[owner, slot], col[k])
    assert not V[~M].view(np.int64).any()                            # +0.0 in every slot the row does not have
    return int(M.sum())


def _covered_rows(ab, rp, col, cover_hi=None):
    sp = ab.slices_host(rp, col, cover_hi=cover_hi)
    return np.concatenate([np.arange(r0, r0 + 32) for r0 in sp["slices"][:, 0]]), sp


@pytest.mark.parametrize("kind,box", [(27, (5, 6, 7)), (27, (9, 4, 11)), (7, (9, 7, 5)), (7, (31, 17, 23))],
                         ids=["27pt-5x6x7", "27pt-9x4x11", "7pt-9x7x5", "7pt-31x17x23"])
def test_stencil_boxes(kind, box, ab):
    gen = mg.stencil3d_27pt if kind == 27 else mg.laplace3d_7pt
    n, r, c, _ = gen(*box)
    assert n % 32
    n, rp, col, a = _full(ab, n, r, c, seed=kind)
    sd = ab.symdiag_host(rp, col)
    O = _stencil_offsets(kind, box[0], box[1])
    assert sd["reason"] == "eligible"
    assert np.array_equal(sd["O"], O) and np.array_equal(sd["D"], O[O >= 0])
    assert len(sd["O"]) == kind and len(sd["D"]) == (14 if kind == 27 else 4)
    assert np.array_equal(sd["coff"], O)
    rows, sp = _covered_rows(ab, rp, col)
    assert rows.min() + O.min() < 0                                   # mirror offsets reach below row 0
    nnz = emulate(n, rp, col, a, sd, rows)
    assert nnz == sp["nnz"]


def test_big_stencil(ab):
    """27-point stencil on 47 x 48 x 33 (tests/test_gpu_kernel_variants.py's big_stencil without extra couplings)."""
    n, r, c, _ = mg.stencil3d_27pt(47, 48, 33)
    n, rp, col, a = _full(ab, n, r, c, seed=3)
    sd = ab.symdiag_host(rp, col)
    assert sd["reason"] == "eligible" and len(sd["O"]) == 27 and len(sd["D"]) == 14
    rows, _ = _covered_rows(ab, rp, col)
    emulate(n, rp, col, a, sd, rows)


def test_big_stencil_with_couplings_of_their_own(ab):
    """One row in 64 coupled at an offset of its own: hundreds of patterns that each occur once, which
    overflow the pattern table and stay in their slices as exception rows -- the layout is not used."""
    from test_gpu_kernel_variants import big_stencil
    n, r, c = big_stencil(True)
    n, rp, col, a = _full(ab, n, r, c, seed=4)
    sp = ab.slices_host(rp, col)
    assert sp["nexc"] > 0
    sd = ab.symdiag_host(rp, col)
    assert sd["reason"] == "exception rows" and len(sd["O"]) == 0


def test_slice_matrix_no_gain(ab):
    """Cliques of 1..18 rows and a small stencil: 50-odd offsets, and as many stored diagonals per row cost
    more than the slice-major values of rows this short -- the layout is not used."""
    from test_gpu_kernel_variants import slice_matrix
    n, r, c = slice_matrix(False)
    n, rp, col, a = _full(ab, n, r, c, seed=5)
    sp = ab.slices_host(rp, col)
    sd = ab.symdiag_host(rp, col)
    assert sd["reason"] == "no gain"
    O = sd["O"]
    assert (np.diff(O) > 0).all() and np.array_equal(sd["D"], np.unique(np.abs(O)))
    assert len(sd["D"]) * sp["rows"] >= 32 * sp["blocks"]
    rows, _ = _covered_rows(ab, rp, col)
    offs = np.unique(np.concatenate([col[rp[i]:rp[i + 1]] - i for i in rows]))
    assert np.array_equal(O, offs)


def test_unsorted_rows(ab):
    """Rows whose columns are not ascending break the CSR-order argument: the layout is not used."""
    n, r, c, _ = mg.stencil3d_27pt(8, 8, 8)
    n, rp, col, a = _full(ab, n, r, c, seed=6)
    assert ab.symdiag_host(rp, col)["reason"] == "eligible"
    col = col.copy()
    for i in range(200, 232):                                         # one slice of 32 rows, swapped the same way
        k = rp[i]
        col[k], col[k + 1] = col[k + 1], col[k]
    sp = ab.slices_host(rp, col)
    assert sp["covered"][200 // 32] or sp["covered"][231 // 32]
    assert ab.symdiag_host(rp, col)["reason"] == "unsorted row"


def test_no_slices(ab):
    n, r, c, _ = mg.random_spd(600, 0.05, 3)
    n, rp, col, a = _full(ab, n, r, c)
    assert ab.symdiag_host(rp, col)["reason"] == "no slices"


@pytest.mark.parametrize("nparts", [2, 8])
def test_partition_blocks(nparts, ab):
    """The parts of a geometric block partition of a 27-point stencil on 48^3 (rows below borderrowoffset are
    eligible for slices).  Two parts: every slice-covered row repeats a dictionary pattern and the layout is
    used.  Eight parts: exception rows, not used."""
    from acg_b200 import dist as abdist
    for part in range(nparts):
        A = abdist.local_stencil_part(27, 48, 48, 48, part, nparts)
        no, bo = A.c.nownedrows, A.c.borderrowoffset
        rp = A.frowptr[:no + 1].copy()
        col = A.fcolidx[:rp[no]].copy()
        a = A.fa[:rp[no]].copy()
        sd = ab.symdiag_host(rp, col, cover_hi=bo)
        if nparts == 8:
            assert sd["reason"] == "exception rows", (part, sd["reason"])
            continue
        assert sd["reason"] == "eligible", (part, sd["reason"])
        assert len(sd["O"]) <= 64 and np.array_equal(sd["D"], np.unique(np.abs(sd["O"])))
        rows, _ = _covered_rows(ab, rp, col, cover_hi=bo)
        assert rows.max() < bo
        emulate(no, rp, col, a, sd, rows)
