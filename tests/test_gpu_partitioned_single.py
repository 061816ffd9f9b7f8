"""Rows a4 / a9 / a10 of SURVEY.md section 8 on ONE GPU (H100, -m gpu).

The multi-GPU tests (test_multirank.py::test_multi_gpu) need >= 2 devices and are skipped on a
one-GPU box.  Everything a rank does *locally* in the distributed SpMV can be checked without
a second device:

* border x ghost block (acg/cgcuda.c:878, csrgemv acg/cg-kernels-cuda.cu:443): every part of a
  partitioned matrix, ghost values taken from the global vector, both device paths --
  local block + offdiag_kernel (set-up products / NCCL loop) and the fused tile kernel of the
  peer-memory loop reading a window behind sequence flags -- against the oracle's product with
  the GLOBAL matrix, entry by entry, plus the fused dot;
* acghalo_pack_cuda / acghalo_unpack_cuda (acg/halo.cu:41,:94) on device buffers with every
  part's own index lists: what is packed for neighbour q is exactly what q expects in its
  ghost tail (send list of p and receive list of q name the same global rows, in order);
* acgcomm_allreduce / acgcomm_barrier / acghalo_exchange_cuda over a real (one-rank) NCCL
  communicator on device memory (acg/comm.c:350-398, :314; acg/halo.c:1272).
"""
import ctypes as C

import numpy as np
import pytest

from acg_b200 import matgen as mg

pytestmark = pytest.mark.gpu
SPMV_RTOL = 1e-13


def _rowparts(kind, n, nparts, dims=None):
    if kind == "block":
        from acg_b200 import dist as abdist
        nx, ny, nz = dims
        px, py, pz = abdist.grid_factors(nparts)
        return abdist.block_partition(nx, ny, nz, px, py, pz)
    if kind == "contiguous":
        return (np.arange(n, dtype=np.int64) * nparts // n).astype(np.int32)
    if kind == "random":
        return np.random.default_rng(5).integers(0, nparts, n).astype(np.int32)
    raise ValueError(kind)


CASES = [
    ("27pt-24-block8", lambda: mg.stencil3d_27pt(24), "block", 8, (24, 24, 24)),
    ("27pt-24-block4", lambda: mg.stencil3d_27pt(24), "block", 4, (24, 24, 24)),
    ("27pt-aniso-block6", lambda: mg.stencil3d_27pt(12, 30, 18), "block", 6, (12, 30, 18)),
    ("7pt-20-contig5", lambda: mg.laplace3d_7pt(20), "contiguous", 5, None),
    ("rmat-random4", lambda: mg.rmat_spd(20000, 300000, seed=3), "random", 4, None),     # most nonzeros couple to ghosts
    ("rmat-contig3", lambda: mg.rmat_spd(30000, 600000, seed=8), "contiguous", 3, None),  # long rows that are border rows
]


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    assert torch.cuda.is_available()
    return torch


@pytest.mark.parametrize("name,gen,pkind,nparts,dims", CASES, ids=[c[0] for c in CASES])
def test_border_ghost_spmv_of_every_part(name, gen, pkind, nparts, dims, ab, oracle):
    n, r, c, v = gen()
    A = ab.SymCsrMatrix.init_real_double(n, r, c, v)
    csr = oracle.full_csr(n, r, c, v)
    xg = np.random.default_rng(2).standard_normal(n)
    want = oracle.dsymv(csr, 1.0, xg, 0.0, np.zeros(n))
    scale = oracle.dsymv((csr[0], csr[1], np.abs(csr[2])), 1.0, np.abs(xg), 0.0, np.zeros(n))
    parts = A.partition(nparts, _rowparts(pkind, n, nparts, dims))
    covered = np.zeros(n, bool)
    ghost_nnz = 0
    exc_rows = 0
    for p, m in enumerate(parts):
        m.dsymv_init(0.0)
        no, nv = m.c.nownedrows, m.c.nprows
        gl = m.nzrows[:nv].astype(np.int64)            # local -> global row numbers, owned then ghost
        assert m.c.nghostrows > 0 and m.c.onpnzs > 0, "a part without ghosts tests nothing"
        ghost_nnz += int(m.c.onpnzs)
        cg = ab.SolverCuda(m)
        exc_rows += cg.info()["spmv_slice_exc"]
        xl = xg[gl]
        for path in (0, 1):
            y, dot = cg.spmv_ghost(xl, path)
            err = np.abs(y - want[gl[:no]])
            assert np.all(err <= SPMV_RTOL * scale[gl[:no]] + 1e-300), (name, p, path, float(err.max()))
            wdot = float(xl[:no] @ want[gl[:no]])
            assert abs(dot - wdot) <= 1e-12 * float(np.abs(xl[:no]) @ scale[gl[:no]]), (name, p, path, dot, wdot)
        covered[gl[:no]] = True
        cg.free()
    assert covered.all() and ghost_nnz > 0
    if name == "27pt-24-block8":
        # the interior rows next to a block's border shell are not in the pattern dictionary: they stay in their
        # slices as exception rows (spmv_slices_kernel<.., EXC>), which this test therefore exercises
        assert exc_rows > 0
    for m in parts:
        m.free()
    A.free()


def _dev(torch, arr, dtype):
    return torch.from_numpy(np.ascontiguousarray(arr)).to(device="cuda", dtype=dtype)


@pytest.mark.parametrize("name,gen,pkind,nparts,dims", CASES[:4] + CASES[4:5], ids=[c[0] for c in CASES[:5]])
def test_pack_unpack_on_device_with_every_parts_lists(name, gen, pkind, nparts, dims, ab, torch_cuda):
    torch = torch_cuda
    L = ab.lib()
    vp, ip = C.c_void_p, C.c_int
    L.acghalo_pack_cuda.argtypes = [ip, vp, ip, ip, vp, vp, vp, C.POINTER(C.c_int64), C.POINTER(ip)]
    L.acghalo_unpack_cuda.argtypes = [ip, vp, ip, ip, vp, vp, vp, C.POINTER(C.c_int64), C.POINTER(ip)]
    ACG_DOUBLE = 0
    n, r, c, v = gen()
    A = ab.SymCsrMatrix.init_real_double(n, r, c, v)
    parts = A.partition(nparts, _rowparts(pkind, n, nparts, dims))
    xg = np.random.default_rng(4).standard_normal(n)
    halos = [m.halo() for m in parts]
    packed = {}
    for p, (m, h) in enumerate(zip(parts, halos)):
        nv = m.c.nprows
        gl = m.nzrows[:nv].astype(np.int64)
        xl = xg[gl].copy()
        xl[m.c.nownedrows:] = np.nan                         # ghosts unknown before the exchange
        d_x = _dev(torch, xl, torch.float64)
        ss = len(h["sendbufidx"])
        d_idx = _dev(torch, h["sendbufidx"], torch.int32)
        d_send = torch.full((max(ss, 1),), float("nan"), dtype=torch.float64, device="cuda")
        nbytes, err = C.c_int64(0), C.c_int(0)
        code = L.acghalo_pack_cuda(ss, d_send.data_ptr(), ACG_DOUBLE, nv, d_x.data_ptr(), d_idx.data_ptr(), None,
                                   C.byref(nbytes), C.byref(err))
        torch.cuda.synchronize()
        assert code == 0 and nbytes.value == 8 * ss
        send = d_send.cpu().numpy()[:ss]
        assert np.array_equal(send, xl[h["sendbufidx"]])          # gather is exact
        for i, q in enumerate(h["recipients"]):
            packed[(p, int(q))] = send[h["sdispls"][i]:h["sdispls"][i] + h["sendcounts"][i]]
    for q, (m, h) in enumerate(zip(parts, halos)):
        nv, no = m.c.nprows, m.c.nownedrows
        gl = m.nzrows[:nv].astype(np.int64)
        rs = len(h["recvbufidx"])
        recv = np.full(max(rs, 1), np.nan)
        for j, p in enumerate(h["senders"]):
            seg = packed[(int(p), q)]
            assert len(seg) == h["recvcounts"][j]
            recv[h["rdispls"][j]:h["rdispls"][j] + h["recvcounts"][j]] = seg
        xl = xg[gl].copy()
        xl[no:] = np.nan
        d_x = _dev(torch, xl, torch.float64)
        d_recv = _dev(torch, recv, torch.float64)
        d_idx = _dev(torch, h["recvbufidx"], torch.int32)
        nbytes, err = C.c_int64(0), C.c_int(0)
        code = L.acghalo_unpack_cuda(rs, d_recv.data_ptr(), ACG_DOUBLE, nv, d_x.data_ptr(), d_idx.data_ptr(), None,
                                     C.byref(nbytes), C.byref(err))
        torch.cuda.synchronize()
        assert code == 0 and nbytes.value == 8 * rs
        # after pack on the senders + unpack here, the local vector equals the global one at all its rows
        assert np.array_equal(d_x.cpu().numpy(), xg[gl]), (name, q)
    for m in parts:
        m.free()
    A.free()


def test_collectives_over_one_rank_nccl(ab, oracle, torch_cuda):
    """acgcomm_allreduce, acgcomm_barrier and the halo exchange entry points go through NCCL
    itself (a one-rank communicator is legal), on device memory; the solver accepts the
    communicator and reproduces the oracle."""
    torch = torch_cuda
    L = ab.lib()
    comm = ab.Comm.init_nccl(1, 0, ab.Comm.unique_id())
    assert comm.size() == 1 and comm.rank() == 0
    vp, ip = C.c_void_p, C.c_int
    L.acgcomm_allreduce.argtypes = [vp, vp, ip, ip, ip, vp, vp, C.POINTER(ip)]
    L.acgcomm_barrier.argtypes = [vp, vp, C.POINTER(ip)]
    ACG_DOUBLE, ACG_SUM, ACG_IN_PLACE = 0, 0, C.c_void_p(1)       # include/acgb200/comm.h:28,:47-48
    src = torch.tensor([1.5, -2.25, 3.0], dtype=torch.float64, device="cuda")
    dst = torch.zeros(3, dtype=torch.float64, device="cuda")
    err = C.c_int(0)
    assert L.acgcomm_allreduce(src.data_ptr(), dst.data_ptr(), 3, ACG_DOUBLE, ACG_SUM, None, C.byref(comm.c), C.byref(err)) == 0
    assert L.acgcomm_barrier(None, C.byref(comm.c), C.byref(err)) == 0
    torch.cuda.synchronize()
    assert torch.equal(src, dst)
    assert L.acgcomm_allreduce(ACG_IN_PLACE, dst.data_ptr(), 3, ACG_DOUBLE, ACG_SUM, None, C.byref(comm.c), C.byref(err)) == 0
    torch.cuda.synchronize()
    assert torch.equal(src, dst)
    n, r, c, v = mg.stencil3d_27pt(12)
    A = ab.SymCsrMatrix.init_real_double(n, r, c, v).dsymv_init(0.0)
    csr = (A.frowptr.copy(), A.fcolidx.copy(), A.fa.copy())
    cg = ab.SolverCuda(A, comm)
    b = A.vector(); b.x[:] = 1.0
    for method, orc in (("solvempi", oracle.cg), ("solve_pipelined", oracle.cg_pipelined)):
        x = A.vector()
        code = getattr(cg, method)(b, x, maxits=60, residualrtol=1e-9, warmup=1)
        want = orc(csr, b.x, maxits=60, rtol=1e-9)
        assert code == 0 and cg.c.niterations == want["niterations"]
        assert np.abs(x.x - want["x"]).max() <= 1e-10 * np.abs(want["x"]).max()
    cg.free()
    comm.destroy()


@pytest.mark.parametrize("name,gen,pkind,nparts,dims", CASES, ids=[c[0] for c in CASES])
def test_border_ghost_residual_mode_of_every_part(name, gen, pkind, nparts, dims, ab, oracle):
    """r = b - A x with the fused r.r (the set-up product of a solve from x0 != 0) and y = A x without a dot,
    on both device paths of every part: offdiag_kernel then SUBTRACTS the border x ghost block and folds r_i^2
    into the dot (path 0), the fused kernels do both for the border rows (path 1).  Against the correctly
    rounded global product (tests/exactref.py), b = A x + 1e-8 noise so that the subtraction cancels."""
    from exactref import dot_exact, gamma, rows_exact
    n, r, c, v = gen()
    A = ab.SymCsrMatrix.init_real_double(n, r, c, v)
    csr = oracle.full_csr(n, r, c, v)
    rng = np.random.default_rng(9)
    xg = rng.standard_normal(n)
    yx, yscale, m = rows_exact(*csr, xg)
    bg = yx + 1e-8 * rng.standard_normal(n)
    rx, rscale, _ = rows_exact(*csr, xg, bg)
    parts = A.partition(nparts, _rowparts(pkind, n, nparts, dims))
    for p, pm in enumerate(parts):
        pm.dsymv_init(0.0)
        no, nv = pm.c.nownedrows, pm.c.nprows
        gl = pm.nzrows[:nv].astype(np.int64)
        assert pm.c.nborderrows > 0
        cg = ab.SolverCuda(pm)
        xl = xg[gl]
        own = gl[:no]
        for path in (0, 1):
            for mode, want, scale in ((0, yx, yscale), (2, rx, rscale)):
                tag = (name, p, path, mode)
                y, dot = cg.spmv_mode(mode, xl, bg[own] if mode == 2 else None, path)
                err = np.abs(y - want[own])
                bound = 2.0 * gamma(m[own] + 1) * scale[own]
                assert np.all(err <= bound), (tag, float((err - bound).max()))
                if mode == 0:
                    assert dot == 0.0, tag
                else:
                    assert abs(dot - dot_exact(y, y)) <= 2.0 * gamma(no) * float(y @ y), (tag, dot, dot_exact(y, y))
        cg.free()
    for pm in parts:
        pm.free()
    A.free()
