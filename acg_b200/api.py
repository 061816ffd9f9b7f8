"""ctypes mirror of the aCG C interface served by libacgb200.so.

The classes keep the reference's names and argument meaning
(acg/symcsrmatrix.h, acg/vector.h, acg/comm.h, acg/cgcuda.h) so that tests read
like calls into the reference: ``SymCsrMatrix`` ~ ``struct acgsymcsrmatrix`` +
``acgsymcsrmatrix_*``, ``Vector`` ~ ``acgvector``, ``Comm`` ~ ``acgcomm``,
``SolverCuda`` ~ ``acgsolvercuda``.

There is no fallback: if the shared library is missing or no CUDA device is
usable, loading / ``SolverCuda`` raises.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIBPATH = os.path.join(_HERE, "libacgb200.so")
_lib = None

ACG_SUCCESS = 0
ACG_ERR_CUDA = 4
ACG_ERR_NVSHMEM_NOT_SUPPORTED = 16
ACG_ERR_NOT_SUPPORTED = 26
ACG_ERR_INDEX_OUT_OF_BOUNDS = 31
ACG_ERR_NOT_CONVERGED = 39


class AcgError(RuntimeError):
    def __init__(self, code, where, detail=0):
        self.code = code
        self.errcode = detail          # third-party code behind ACG_ERR_CUDA / ACG_ERR_NCCL (cudaError_t, ncclResult_t)
        msg = lib().acgerrcodestr(code, detail).decode()
        super().__init__(f"{where}: {msg} (acgerrcode {code})")


def build(verbose: bool = False) -> str:
    """Compile libacgb200.so in-tree (nvcc sm_90a + gcc)."""
    subprocess.run(["make", "-C", os.path.join(_HERE, "csrc")], check=True,
                   stdout=None if verbose else subprocess.DEVNULL)
    return _LIBPATH


class acgvector(C.Structure):
    _fields_ = [("nparts", C.c_int), ("parttag", C.c_int), ("nprocs", C.c_int), ("npparts", C.c_int),
                ("ownerrank", C.c_int), ("ownerpart", C.c_int),
                ("size", C.c_int), ("x", C.POINTER(C.c_double)),
                ("num_nonzeros", C.c_int), ("idxbase", C.c_int), ("idx", C.POINTER(C.c_int)),
                ("num_ghost_nonzeros", C.c_int)]


class acgsymcsrmatrix(C.Structure):
    _fields_ = [("graph", C.c_void_p), ("nrows", C.c_int), ("nprows", C.c_int),
                ("nzrows", C.POINTER(C.c_int)), ("nnzs", C.c_int64), ("npnzs", C.c_int64),
                ("rowidxbase", C.c_int), ("rownnzs", C.POINTER(C.c_int64)), ("rowptr", C.POINTER(C.c_int64)),
                ("rowidx", C.POINTER(C.c_int)), ("colidx", C.POINTER(C.c_int)),
                ("nownedrows", C.c_int), ("ninnerrows", C.c_int), ("nborderrows", C.c_int),
                ("borderrowoffset", C.c_int), ("nghostrows", C.c_int), ("ghostrowoffset", C.c_int),
                ("ninnernzs", C.c_int64), ("ninterfacenzs", C.c_int64),
                ("nborderrowinnernzs", C.POINTER(C.c_int64)), ("nborderrowinterfacenzs", C.POINTER(C.c_int64)),
                ("a", C.POINTER(C.c_double)),
                ("fnpnzs", C.c_int64), ("onpnzs", C.c_int64),
                ("frowptr", C.POINTER(C.c_int64)), ("orowptr", C.POINTER(C.c_int64)),
                ("fcolidx", C.POINTER(C.c_int)), ("ocolidx", C.POINTER(C.c_int)),
                ("fa", C.POINTER(C.c_double)), ("oa", C.POINTER(C.c_double))]


class acghalo(C.Structure):
    _fields_ = [("nrecipients", C.c_int), ("recipients", C.POINTER(C.c_int)), ("sendcounts", C.POINTER(C.c_int)),
                ("sdispls", C.POINTER(C.c_int)), ("sendsize", C.c_int), ("sendbufidx", C.POINTER(C.c_int)),
                ("nsenders", C.c_int), ("senders", C.POINTER(C.c_int)), ("recvcounts", C.POINTER(C.c_int)),
                ("rdispls", C.POINTER(C.c_int)), ("recvsize", C.c_int), ("recvbufidx", C.POINTER(C.c_int)),
                ("nexchanges", C.c_int), ("texchange", C.c_double),
                ("tpack", C.c_double), ("tunpack", C.c_double), ("tsendrecv", C.c_double),
                ("tmpiirecv", C.c_double), ("tmpisend", C.c_double), ("tmpiwaitall", C.c_double),
                ("npack", C.c_int64), ("nunpack", C.c_int64), ("nmpiirecv", C.c_int64), ("nmpisend", C.c_int64),
                ("Bpack", C.c_int64), ("Bunpack", C.c_int64), ("Bmpiirecv", C.c_int64), ("Bmpisend", C.c_int64),
                ("maxexchangestats", C.c_int), ("thaloexchangestats", C.c_void_p)]


class acgsolvercuda(C.Structure):
    _fields_ = ([("r", acgvector), ("p", acgvector), ("t", acgvector)] +
                [(n, C.c_void_p) for n in ("w", "q", "z", "dx", "halo", "haloexchange")] +
                [("maxits", C.c_int)] +
                [(n, C.c_double) for n in ("diffatol", "diffrtol", "residualatol", "residualrtol",
                                           "bnrm2", "r0nrm2", "rnrm2", "x0nrm2", "dxnrm2")] +
                [(n, C.c_void_p) for n in ("d_minus_one", "d_one", "d_zero", "d_inf", "d_bnrm2sqr", "d_r0nrm2sqr",
                                           "d_rnrm2sqr", "d_rnrm2sqr_prev", "d_pdott", "d_alpha", "d_minus_alpha",
                                           "d_beta", "d_niterations", "d_converged", "d_r", "d_p", "d_t", "d_w",
                                           "d_q", "d_z", "d_rowptr", "d_orowptr", "d_colidx", "d_ocolidx",
                                           "d_a", "d_oa")] +
                [("use_nvshmem", C.c_int), ("nsolves", C.c_int), ("ntotaliterations", C.c_int),
                 ("niterations", C.c_int), ("nflops", C.c_int64), ("tsolve", C.c_double)] +
                [(n, C.c_double) for n in ("tgemv", "tdot", "tnrm2", "taxpy", "tcopy", "tallreduce", "thalo")] +
                [(n, C.c_int64) for n in ("ngemv", "ndot", "nnrm2", "naxpy", "ncopy", "nallreduce", "nhalo",
                                          "Bgemv", "Bdot", "Bnrm2", "Baxpy", "Bcopy", "Ballreduce", "Bhalo",
                                          "nhalomsgs")])


class acgcomm(C.Structure):
    _fields_ = [("type", C.c_int), ("ncclcomm", C.c_void_p)]


class acgb200_info(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("spmv_lanes_per_row", "spmv_rows_cap", "spmv_nnz_cap", "spmv_stages",
                                       "spmv_ntiles", "spmv_nlong", "spmv_grid", "spmv_smem_bytes", "num_sms",
                                       "last_launches", "last_spmv_count")] + [("last_spmv_ms", C.c_double),
                                                                                  ("last_solve_ms", C.c_double),
                                                                                  ("last_h2d_ms", C.c_double),
                                                                                  ("last_d2h_ms", C.c_double),
                                                                                  ("last_blas_ms", C.c_double),
                                                                                  ("reserved0", C.c_int),
                                                                                  ("spmv_min_bytes", C.c_int64),
                                                                                  ("spmv_nmedium", C.c_int),
                                                                                  ("reserved1", C.c_int),
                                                                                  ("spmv_slices", C.c_int),
                                                                                  ("spmv_slice_rows", C.c_int),
                                                                                  ("spmv_slice_ub", C.c_int),
                                                                                  ("spmv_slice_grid", C.c_int),
                                                                                  ("spmv_merge_tiles", C.c_int),
                                                                                  ("spmv_merge_rows", C.c_int),
                                                                                  ("spmv_merge_split", C.c_int),
                                                                                  ("spmv_slice_exc", C.c_int)] + \
        [(n, C.c_int) for n in ("spmv_threads", "spmv_unroll", "spmv_slice_threads", "spmv_merge_threads",
                                "spmv_merge_grid", "spmv_merge_stages")] + \
        [("spmv_slice_value_bytes", C.c_int64), ("spmv_slice_nnz", C.c_int64)] + \
        [("spmv_symdiag_diagonals", C.c_int), ("spmv_symdiag_bytes", C.c_int64)] + \
        [("pcg_fused", C.c_int), ("pcg_fused_min_bytes", C.c_int64)] + \
        [("spmv_symdiag_codes", C.c_int), ("spmv_symdiag_code_bytes", C.c_int64)] + \
        [("mixed_reliable_updates", C.c_int)] + \
        [("cheb_degree", C.c_int), ("cheb_est_iterations", C.c_int), ("cheb_breakdown", C.c_int),
         ("cheb_lmin", C.c_double), ("cheb_lmax", C.c_double)] + \
        [("pcg_group", C.c_int)]


class acgb200_colstats(C.Structure):
    _fields_ = [("niterations", C.c_int), ("converged", C.c_int), ("bnrm2", C.c_double), ("r0nrm2", C.c_double),
                ("rnrm2", C.c_double)]


class acgb200_mtxinfo(C.Structure):
    _fields_ = [("nrows", C.c_int64), ("ncols", C.c_int64), ("nnzs", C.c_int64), ("data_offset", C.c_int64),
                ("field", C.c_int), ("symmetric", C.c_int)]


# every symbol include/acgb200/*.h declares (checked by tests/test_abi.py)
EXPORTS = [
    "acgerrcodestr",
    "acgvector_init_empty", "acgvector_free", "acgvector_init_copy", "acgvector_alloc",
    "acgvector_init_real_double", "acgvector_alloc_packed", "acgvector_setzero",
    "acgvector_set_constant_real_double", "acgvector_copy", "acgvector_daxpy", "acgvector_dnrm2",
    "acgvector_usga", "acgvector_ussc",
    "acgsymcsrmatrix_init_real_double", "acgsymcsrmatrix_init_rowwise_real_double", "acgsymcsrmatrix_free",
    "acgsymcsrmatrix_vector", "acgsymcsrmatrix_partition", "acgsymcsrmatrix_partition_rows", "acgsymcsrmatrix_halo", "acgsymcsrmatrix_dsymv_init", "acgsymcsrmatrix_dsymv_init_cuda",
    "acgcommtypestr", "acgcomm_init_nccl", "acgcomm_free", "acgcomm_size", "acgcomm_rank", "acgcomm_barrier",
    "acgcomm_allreduce",
    "acghalo_free", "acghaloexchange_init_cuda", "acghaloexchange_free", "acghaloexchange_profile",
    "acghalo_pack_cuda", "acghalo_unpack_cuda", "acghalo_exchange_cuda_begin", "acghalo_exchange_cuda_end",
    "acghalo_exchange_cuda",
    "acgsolvercuda_free", "acgsolvercuda_init", "acgsolvercuda_solvempi", "acgsolvercuda_solve_pipelined",
    "acgsolvercuda_solve", "acgsolvercuda_solve_device", "acgsolvercuda_solve_device_pipelined",
    "acgsolvercuda_init_constants", "acgsolvercuda_alpha", "acgsolvercuda_beta", "acgsolvercuda_daxpy_alpha",
    "acgsolvercuda_daxpy_minus_alpha", "acgsolvercuda_daypx_beta", "acgsolvercuda_pipelined_daxpy_fused",
    "acgsolvercuda_fwrite",
    "acgb200_set_option", "acgsolvercuda_spmv", "acgsolvercuda_spmv_ghost", "acgsolvercuda_spmv_mode", "acgsolvercuda_solve_multi", "acgsolvercuda_spmm_mode", "acgsolvercuda_solve_shifted", "acgsolvercuda_solve_minres", "acgsolvercuda_solve_mixed", "acgsolvercuda_spmv_f32", "acgsolvercuda_solve_chebyshev", "acgsolvercuda_update_values", "acgb200_cheb_interval_host", "acgsolvercuda_info", "acgb200_sizeof", "acgb200_have_mpi",
    "acgb200_nccl_unique_id", "acgb200_comm_init_rank", "acgb200_comm_destroy",
    "acgb200_host_register", "acgb200_host_unregister", "acgb200_spmv_plan_host", "acgb200_spmv_plan_host2", "acgb200_slices_host", "acgb200_symdiag_host", "acgb200_merge_plan_host", "acgb200_p2p_inverse_map", "acgb200_patterns_host", "acgb200_stencil_part",
    "acgb200_mtx_info", "acgb200_mtx_read", "acgb200_mtx_read_part", "acgb200_comm_matrix_row", "acgb200_partition_rows_grid", "acgb200_grid_factors", "acgb200_rmat_spd",
]


def lib() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIBPATH):
        raise RuntimeError(f"{_LIBPATH} not built: run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(there is no fallback implementation)")
    L = C.CDLL(_LIBPATH, mode=C.RTLD_LOCAL)
    L.acgerrcodestr.restype = C.c_char_p
    L.acgerrcodestr.argtypes = [C.c_int, C.c_int]
    L.acgb200_sizeof.restype = C.c_size_t
    L.acgb200_sizeof.argtypes = [C.c_char_p]
    for name, st in (("acgvector", acgvector), ("acgsymcsrmatrix", acgsymcsrmatrix), ("acghalo", acghalo),
                     ("acgsolvercuda", acgsolvercuda), ("acgcomm", acgcomm)):
        got = L.acgb200_sizeof(name.encode())
        if got != C.sizeof(st):
            raise RuntimeError(f"ABI mismatch for struct {name}: library {got} B, binding {C.sizeof(st)} B")
    P = C.POINTER
    i32p = np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")
    i64p = np.ctypeslib.ndpointer(np.int64, flags="C_CONTIGUOUS")
    f64p = np.ctypeslib.ndpointer(np.float64, flags="C_CONTIGUOUS")
    L.acgsymcsrmatrix_init_real_double.argtypes = [P(acgsymcsrmatrix), C.c_int, C.c_int64, C.c_int, i32p, i32p, f64p]
    L.acgsymcsrmatrix_init_rowwise_real_double.argtypes = [P(acgsymcsrmatrix), C.c_int, C.c_int, i64p, i32p, f64p]
    L.acgsymcsrmatrix_free.restype = None
    L.acgsymcsrmatrix_free.argtypes = [P(acgsymcsrmatrix)]
    L.acgsymcsrmatrix_vector.argtypes = [P(acgsymcsrmatrix), P(acgvector)]
    L.acgsymcsrmatrix_partition.argtypes = [P(acgsymcsrmatrix), C.c_int, i32p, P(acgsymcsrmatrix), C.c_int]
    L.acgsymcsrmatrix_partition_rows.argtypes = [P(acgsymcsrmatrix), C.c_int, C.c_int, i32p, P(C.c_int), C.c_int, C.c_int]
    L.acgsymcsrmatrix_halo.argtypes = [P(acgsymcsrmatrix), P(acghalo)]
    L.acgb200_stencil_part.argtypes = [C.c_int] * 8 + [P(acgsymcsrmatrix)]
    L.acgb200_mtx_info.argtypes = [C.c_char_p, P(acgb200_mtxinfo)]
    L.acgb200_partition_rows_grid.argtypes = [C.c_int] * 6 + [np.ctypeslib.ndpointer(np.int32, flags="C")]
    L.acgb200_grid_factors.argtypes = [C.c_int, P(C.c_int), P(C.c_int), P(C.c_int)]
    L.acgb200_grid_factors.restype = None
    L.acgb200_rmat_spd.argtypes = [C.c_int64, C.c_int64, C.c_uint64, P(C.c_double), P(acgsymcsrmatrix)]
    L.acgb200_comm_matrix_row.argtypes = [P(acgsymcsrmatrix), C.c_int, np.ctypeslib.ndpointer(np.int64, flags="C")]
    L.acgb200_mtx_read.argtypes = [C.c_char_p, C.c_int, P(acgsymcsrmatrix)]
    L.acgb200_mtx_read_part.argtypes = [C.c_char_p, C.c_int, np.ctypeslib.ndpointer(np.int32, flags="C"), C.c_int,
                                        P(acgsymcsrmatrix)]
    L.acgsymcsrmatrix_dsymv_init.argtypes = [P(acgsymcsrmatrix), C.c_double]
    L.acgsymcsrmatrix_dsymv_init_cuda.argtypes = [P(acgsymcsrmatrix), C.c_double, P(C.c_int)]
    L.acghalo_free.restype = None
    L.acghalo_free.argtypes = [P(acghalo)]
    L.acgvector_free.restype = None
    L.acgvector_free.argtypes = [P(acgvector)]
    L.acgvector_alloc.argtypes = [P(acgvector), C.c_int]
    L.acgvector_setzero.argtypes = [P(acgvector)]
    L.acgvector_usga.argtypes = [P(acgvector), P(acgvector)]
    L.acgvector_ussc.argtypes = [P(acgvector), P(acgvector)]
    L.acgsolvercuda_free.restype = None
    L.acgsolvercuda_free.argtypes = [P(acgsolvercuda)]
    L.acgsolvercuda_init.argtypes = [P(acgsolvercuda), P(acgsymcsrmatrix), C.c_void_p, C.c_void_p, P(acgcomm)]
    common = [P(acgsolvercuda), P(acgsymcsrmatrix), P(acgvector), P(acgvector), C.c_int,
              C.c_double, C.c_double, C.c_double, C.c_double, C.c_int]
    L.acgsolvercuda_solvempi.argtypes = common + [P(acgcomm), C.c_int, P(C.c_int), C.c_void_p, C.c_void_p, C.c_int]
    L.acgsolvercuda_solve_pipelined.argtypes = common + [P(acgcomm), C.c_int, P(C.c_int), C.c_void_p, C.c_void_p]
    L.acgsolvercuda_solve.argtypes = common
    L.acgsolvercuda_solve_device.argtypes = common + [P(acgcomm), P(C.c_int)]
    # acg/cg-kernels-cuda.h:45-97: device pointers as plain addresses
    vp = C.c_void_p
    L.acgsolvercuda_init_constants.argtypes = [P(vp), P(vp), P(vp)]
    L.acgsolvercuda_alpha.argtypes = [vp, vp, vp, vp]
    L.acgsolvercuda_beta.argtypes = [vp, vp, vp]
    L.acgsolvercuda_daxpy_alpha.argtypes = [C.c_int, vp, vp, vp, vp]
    L.acgsolvercuda_daxpy_minus_alpha.argtypes = [C.c_int, vp, vp, vp, vp]
    L.acgsolvercuda_daypx_beta.argtypes = [C.c_int, vp, vp, vp, vp]
    L.acgsolvercuda_pipelined_daxpy_fused.argtypes = [C.c_int] + [vp] * 11 + [vp]
    L.acgsolvercuda_solve_device_pipelined.argtypes = common + [P(acgcomm), P(C.c_int)]
    L.acgsolvercuda_fwrite.argtypes = [C.c_void_p, P(acgsolvercuda), C.c_int]
    L.acgsolvercuda_spmv.argtypes = [P(acgsolvercuda), f64p, f64p, C.c_int, P(C.c_double)]
    L.acgsolvercuda_spmv_ghost.argtypes = [P(acgsolvercuda), f64p, f64p, C.c_int, P(C.c_double)]
    L.acgsolvercuda_spmv_mode.argtypes = [P(acgsolvercuda), C.c_int, f64p, C.c_void_p, f64p, C.c_int, P(C.c_double)]
    L.acgsolvercuda_solve_multi.argtypes = [P(acgsolvercuda), P(acgsymcsrmatrix), C.c_int, f64p, f64p, C.c_int,
                                            C.c_double, C.c_double, C.c_int, P(acgb200_colstats)]
    L.acgsolvercuda_spmm_mode.argtypes = [P(acgsolvercuda), C.c_int, C.c_int, f64p, C.c_void_p, f64p, P(C.c_double)]
    L.acgsolvercuda_solve_shifted.argtypes = [P(acgsolvercuda), P(acgsymcsrmatrix), C.c_int, f64p, f64p, f64p, C.c_int,
                                              C.c_double, C.c_double, C.c_int, P(acgb200_colstats)]
    L.acgsolvercuda_solve_minres.argtypes = [P(acgsolvercuda), P(acgsymcsrmatrix), P(acgvector), P(acgvector), C.c_int,
                                             C.c_double, C.c_double, C.c_int, P(C.c_int)]
    L.acgsolvercuda_solve_chebyshev.argtypes = [P(acgsolvercuda), P(acgsymcsrmatrix), P(acgvector), P(acgvector), C.c_int,
                                                C.c_double, C.c_double, C.c_int, C.c_double, C.c_double, C.c_int,
                                                P(C.c_int)]
    L.acgb200_cheb_interval_host.argtypes = [C.c_int, f64p, f64p, P(C.c_double), P(C.c_double)]
    L.acgsolvercuda_solve_mixed.argtypes = [P(acgsolvercuda), P(acgsymcsrmatrix), P(acgvector), P(acgvector), C.c_int,
                                            C.c_double, C.c_double, C.c_int, P(C.c_int)]
    f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
    L.acgsolvercuda_spmv_f32.argtypes = [P(acgsolvercuda), f32p, f32p, P(C.c_double)]
    L.acgsolvercuda_update_values.argtypes = [P(acgsolvercuda), P(acgsymcsrmatrix), P(C.c_int)]
    L.acgsolvercuda_info.argtypes = [P(acgsolvercuda), P(acgb200_info)]
    L.acgb200_set_option.argtypes = [C.c_char_p, C.c_int]
    L.acgb200_nccl_unique_id.argtypes = [C.c_void_p]
    L.acgb200_host_register.argtypes = [C.c_void_p, C.c_size_t]
    L.acgb200_host_unregister.argtypes = [C.c_void_p]
    u16p = np.ctypeslib.ndpointer(np.uint16, flags="C_CONTIGUOUS")
    L.acgb200_patterns_host.argtypes = [C.c_int, i64p, i32p, C.c_int, P(C.c_int), P(C.c_int), i32p, i32p, u16p, P(C.c_int64)]
    L.acgb200_p2p_inverse_map.argtypes = [P(acghalo), C.c_int, C.c_int, i32p, i32p, i32p, i32p]
    L.acgb200_spmv_plan_host2.argtypes = [C.c_int, i64p, C.c_void_p, P(acgb200_info), i32p, C.c_int, i32p, C.c_int]
    L.acgb200_merge_plan_host.argtypes = [C.c_int, i64p, C.c_int, i32p, C.c_int, i32p, P(C.c_int), P(C.c_int)]
    L.acgb200_slices_host.argtypes = [C.c_int, C.c_int, i64p, C.c_void_p, i32p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_void_p]
    L.acgb200_symdiag_host.argtypes = [C.c_int, C.c_int, i64p, i32p, i32p, i32p, i32p, i32p]
    L.acgb200_spmv_plan_host.argtypes = [C.c_int, i64p, P(acgb200_info), i32p, C.c_int, i32p, C.c_int]
    L.acgb200_comm_init_rank.argtypes = [P(acgcomm), C.c_int, C.c_void_p, C.c_int, P(C.c_int)]
    L.acgb200_comm_destroy.argtypes = [P(acgcomm)]
    L.acgcomm_size.argtypes = [P(acgcomm), P(C.c_int)]
    L.acgcomm_rank.argtypes = [P(acgcomm), P(C.c_int)]
    _lib = L
    return L


def _check(code, where, detail=0):
    if code != ACG_SUCCESS:
        raise AcgError(code, where, detail)


def mtx_info(path: str) -> dict:
    """acgb200_mtx_info: sizes and data offset of a Matrix Market coordinate file."""
    inf = acgb200_mtxinfo()
    _check(lib().acgb200_mtx_info(os.fsencode(path), C.byref(inf)), "acgb200_mtx_info")
    return {k: getattr(inf, k) for k, _ in acgb200_mtxinfo._fields_}


def set_option(key: str, value: int) -> None:
    _check(lib().acgb200_set_option(key.encode(), int(value)), f"acgb200_set_option({key})")


def patterns_host(rowptr, colidx, max_entries: int = 4096) -> dict:
    """Row-pattern dictionary of a 0-based CSR matrix (host only, compress.c)."""
    rowptr = np.ascontiguousarray(rowptr, np.int64)
    colidx = np.ascontiguousarray(colidx, np.int32)
    n = len(rowptr) - 1
    npat, nent, nm = C.c_int(0), C.c_int(0), C.c_int64(0)
    patptr = np.zeros(max_entries + 2, np.int32)
    patoff = np.zeros(max_entries + 1, np.int32)
    patid = np.zeros(max(n, 1), np.uint16)
    _check(lib().acgb200_patterns_host(n, rowptr, colidx, max_entries, C.byref(npat), C.byref(nent), patptr, patoff,
                                       patid, C.byref(nm)), "acgb200_patterns_host")
    return dict(npat=npat.value, patptr=patptr[:npat.value + 1].copy(), patoff=patoff[:nent.value].copy(),
                patid=patid[:n].copy(), nmatched=nm.value)


def merge_plan_host(rowptr, items: int = 1024, hi=None) -> dict:
    """The merge-path tile plan of rows [0,hi) (mergeplan.c), computed on the host: tiles as rows of
    (r0, nre, k0, nnz), split rows as rows of (row, ta, tb)."""
    rowptr = np.ascontiguousarray(rowptr, dtype=np.int64)
    n = len(rowptr) - 1 if hi is None else hi
    cap = int((n + rowptr[n]) // items + 2)
    tiles = np.zeros(4 * cap, np.int32)
    split = np.zeros(3 * cap, np.int32)
    nt, ns = C.c_int(0), C.c_int(0)
    _check(lib().acgb200_merge_plan_host(n, rowptr, items, tiles, cap, split, C.byref(nt), C.byref(ns)), "acgb200_merge_plan_host")
    return dict(tiles=tiles[:4 * nt.value].reshape(nt.value, 4).copy(), split=split[:3 * ns.value].reshape(ns.value, 3).copy())


def slices_host(rowptr, colidx, cover_hi=None) -> dict:
    """The pattern-slice plan acgsolvercuda_init would build (slices.c), computed on the host: the
    covered 32-row slices as rows of (row0, nrows, len, vblk), the per-slice cover flags, and totals."""
    rowptr = np.ascontiguousarray(rowptr, dtype=np.int64)
    colidx = np.ascontiguousarray(colidx, dtype=np.int32)
    n = len(rowptr) - 1
    nsl = (n + 31) // 32
    slices4 = np.zeros(4 * max(nsl, 1), dtype=np.int32)
    covered = np.zeros(max(nsl, 1), dtype=np.uint8)
    totals = np.zeros(6, dtype=np.int64)
    spatoff = np.zeros(8192, dtype=np.int32)
    patid = np.full(max(n, 1), 0xFFFF, dtype=np.uint16)
    exc2 = np.zeros(2, dtype=np.int64)
    _check(lib().acgb200_slices_host(n, n if cover_hi is None else cover_hi, rowptr, colidx.ctypes.data_as(C.c_void_p),
                                     slices4, nsl, covered.ctypes.data_as(C.c_void_p), totals.ctypes.data_as(C.c_void_p),
                                     spatoff.ctypes.data_as(C.c_void_p), patid.ctypes.data_as(C.c_void_p),
                                     exc2.ctypes.data_as(C.c_void_p)), "acgb200_slices_host")
    ns = int(totals[0])
    return dict(nslices=ns, slices=slices4[:4 * ns].reshape(ns, 4).copy(), covered=covered[:nsl].astype(bool),
                blocks=int(totals[1]), nnz=int(totals[2]), rows=int(totals[3]), lpad=int(totals[4]), npat=int(totals[5]),
                spatoff=spatoff, patid=patid[:n], nexc=int(exc2[0]), excnnz=int(exc2[1]))


SYMDIAG_REASONS = ("eligible", "no slices", "exception rows", "unsorted row", "too many offsets", "no gain", "too large")


def symdiag_host(rowptr, colidx, cover_hi=None) -> dict:
    """The mirrored-diagonal plan acgsolvercuda_init would use for the pattern slices (slices.c), computed on
    the host: ``reason`` (one of SYMDIAG_REASONS; "eligible" means the layout is used if the values pass the
    device's symmetry check), the offsets ``O`` of the covered rows, the stored diagonals ``D``, and for an
    eligible plan the ``margin``, ``stride`` and per-entry ``voff`` / ``coff`` of the kernel's addressing."""
    rowptr = np.ascontiguousarray(rowptr, dtype=np.int64)
    colidx = np.ascontiguousarray(colidx, dtype=np.int32)
    n = len(rowptr) - 1
    info = np.zeros(5, np.int32)
    o = np.zeros(64, np.int32)
    d = np.zeros(64, np.int32)
    tab = np.zeros(128, np.int32)
    _check(lib().acgb200_symdiag_host(n, n if cover_hi is None else cover_hi, rowptr, colidx, info, o, d, tab),
           "acgb200_symdiag_host")
    no, nd = int(info[1]), int(info[2])
    t = tab[:2 * no].reshape(no, 2)
    return dict(reason=SYMDIAG_REASONS[int(info[0])], O=o[:no].copy(), D=d[:nd].copy(), margin=int(info[3]),
                stride=int(info[4]), voff=t[:, 0].copy(), coff=t[:, 1].copy())


def cheb_interval_host(alpha, beta) -> tuple:
    """acgb200_cheb_interval_host: the extreme eigenvalues (theta_min, theta_max) of the Lanczos tridiagonal
    that acgsolvercuda_solve_chebyshev builds from k CG steps' alpha (k) and beta (k - 1)."""
    alpha = np.ascontiguousarray(alpha, np.float64)
    beta = np.ascontiguousarray(beta if len(beta) else [0.0], np.float64)
    tmin, tmax = C.c_double(0), C.c_double(0)
    _check(lib().acgb200_cheb_interval_host(len(alpha), alpha, beta, C.byref(tmin), C.byref(tmax)),
           "acgb200_cheb_interval_host")
    return tmin.value, tmax.value


def spmv_plan_host(rowptr, colidx=None) -> dict:
    """Tile plan of the SpMV for a CSR row-pointer array (host only, no device).
    With ``colidx`` the pattern slices are planned too and the tiles skip the rows they cover
    (``slices``, ``slice_rows``; acg_b200.slices_host lists the slices themselves)."""
    rowptr = np.ascontiguousarray(rowptr, np.int64)
    n = len(rowptr) - 1
    tiles = np.zeros(4 * (n + 1), np.int32)
    longrows = np.zeros(n + 1, np.int32)
    inf = acgb200_info()
    cptr = None
    if colidx is not None:
        colidx = np.ascontiguousarray(colidx, np.int32)
        cptr = colidx.ctypes.data_as(C.c_void_p)
    _check(lib().acgb200_spmv_plan_host2(n, rowptr, cptr, C.byref(inf), tiles, n + 1, longrows, n + 1), "acgb200_spmv_plan_host")
    nt, nl = inf.spmv_ntiles, inf.spmv_nlong
    t4 = tiles[:4 * nt].reshape(nt, 4).copy()
    return dict(lanes=inf.spmv_lanes_per_row, rows_cap=inf.spmv_rows_cap, nnz_cap=inf.spmv_nnz_cap,
                stages=inf.spmv_stages, tiles=t4, longrows=longrows[:nl].copy(), nmedium=inf.spmv_nmedium,
                slices=inf.spmv_slices, slice_rows=inf.spmv_slice_rows)


def _view(ptr, n, dtype):
    if n <= 0 or not ptr:
        return np.zeros(0, dtype)
    return np.ctypeslib.as_array(ptr, shape=(int(n),))


class Vector:
    """``struct acgvector`` (acg/vector.h:58): owned entries first, ghosts last."""

    def __init__(self, size=None):
        self.c = acgvector()
        self._owns = False
        if size is not None:
            _check(lib().acgvector_alloc(C.byref(self.c), int(size)), "acgvector_alloc")
            lib().acgvector_setzero(C.byref(self.c))
            self._owns = True

    @property
    def x(self) -> np.ndarray:
        return _view(self.c.x, self.c.num_nonzeros, np.float64)

    @property
    def idx(self) -> np.ndarray:
        return _view(self.c.idx, self.c.num_nonzeros, np.int32)

    @property
    def nowned(self) -> int:
        return self.c.num_nonzeros - self.c.num_ghost_nonzeros

    def pin(self):
        """Page-lock the storage (caller-side optimisation of the H2D/D2H copies)."""
        _check(lib().acgb200_host_register(self.c.x, self.c.num_nonzeros * 8), "cudaHostRegister")
        self._pinned = True
        return self

    def free(self):
        if getattr(self, "_pinned", False):
            lib().acgb200_host_unregister(self.c.x)
            self._pinned = False
        if self._owns:
            lib().acgvector_free(C.byref(self.c))
            self._owns = False

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class SymCsrMatrix:
    """``struct acgsymcsrmatrix`` (acg/symcsrmatrix.h:62)."""

    def __init__(self):
        self.c = acgsymcsrmatrix()
        self._owns = False

    @classmethod
    def init_real_double(cls, n, rowidx, colidx, a, idxbase=0):
        """acgsymcsrmatrix_init_real_double: upper-triangle COO -> packed CSR."""
        self = cls()
        rowidx = np.ascontiguousarray(rowidx, np.int32)
        colidx = np.ascontiguousarray(colidx, np.int32)
        a = np.ascontiguousarray(a, np.float64)
        _check(lib().acgsymcsrmatrix_init_real_double(C.byref(self.c), n, len(a), idxbase, rowidx, colidx, a),
               "acgsymcsrmatrix_init_real_double")
        self._owns = True
        return self

    @classmethod
    def rmat_spd(cls, n: int, nedges: int, seed: int = 42):
        """acgb200_rmat_spd: threaded R-MAT power-law SPD matrix (BASELINE config 5)."""
        self = cls()
        _check(lib().acgb200_rmat_spd(n, nedges, seed, None, C.byref(self.c)), "acgb200_rmat_spd")
        self._owns = True
        return self

    @classmethod
    def read_mtx(cls, path: str, binary: bool = True):
        """acgb200_mtx_read: a "matrix coordinate real symmetric" Matrix Market file, text
        or aCG binary (acg/mtxfile.c:1107-1127), as a 0-based packed matrix."""
        self = cls()
        _check(lib().acgb200_mtx_read(os.fsencode(path), 1 if binary else 0, C.byref(self.c)), "acgb200_mtx_read")
        self._owns = True
        return self

    @classmethod
    def read_mtx_part(cls, path: str, nparts: int, rowparts, part: int):
        """acgb200_mtx_read_part: this part of a row partition straight from a binary
        file; no process holds the whole matrix."""
        self = cls()
        rowparts = np.ascontiguousarray(rowparts, np.int32)
        _check(lib().acgb200_mtx_read_part(os.fsencode(path), nparts, rowparts, part, C.byref(self.c)),
               "acgb200_mtx_read_part")
        self._owns = True
        return self

    @classmethod
    def stencil_part(cls, kind: int, nx: int, ny: int, nz: int, px: int, py: int, pz: int, part: int):
        """One part of a block-partitioned 7/27-point stencil matrix, built without the global matrix."""
        self = cls()
        _check(lib().acgb200_stencil_part(kind, nx, ny, nz, px, py, pz, part, C.byref(self.c)), "acgb200_stencil_part")
        self._owns = True
        return self

    def dsymv_init(self, eps: float = 0.0):
        _check(lib().acgsymcsrmatrix_dsymv_init(C.byref(self.c), eps), "acgsymcsrmatrix_dsymv_init")
        return self

    def dsymv_init_cuda(self, eps: float = 0.0):
        """acgsymcsrmatrix_dsymv_init computed on the current CUDA device (expand.cu), copied back into the matrix."""
        err = C.c_int(0)
        code = lib().acgsymcsrmatrix_dsymv_init_cuda(C.byref(self.c), eps, C.byref(err))
        if code != ACG_SUCCESS:
            raise AcgError(code, "acgsymcsrmatrix_dsymv_init_cuda", err.value)
        return self

    def partition_rows(self, nparts: int, kway: bool = False, seed: int = 0):
        """acgsymcsrmatrix_partition_rows: METIS row->part map; returns (rowparts, edge cut)."""
        rowparts = np.zeros(max(self.c.nprows, 1), np.int32)
        cut = C.c_int(0)
        _check(lib().acgsymcsrmatrix_partition_rows(C.byref(self.c), nparts, 1 if kway else 0, rowparts, C.byref(cut), seed, 0),
               "acgsymcsrmatrix_partition_rows")
        return rowparts[:self.c.nprows], cut.value

    def partition(self, nparts: int, rowparts) -> list["SymCsrMatrix"]:
        rowparts = np.ascontiguousarray(rowparts, np.int32)
        arr = (acgsymcsrmatrix * nparts)()
        _check(lib().acgsymcsrmatrix_partition(C.byref(self.c), nparts, rowparts, arr, 0), "acgsymcsrmatrix_partition")
        out = []
        for p in range(nparts):
            m = SymCsrMatrix()
            C.memmove(C.byref(m.c), C.byref(arr[p]), C.sizeof(acgsymcsrmatrix))
            m._owns = True
            out.append(m)
        return out

    def comm_matrix_row(self, nparts: int) -> np.ndarray:
        """Border values this part sends to every other part per halo exchange
        (one row of the driver's --output-comm-matrix, cuda/acg-cuda.c:1713-1775)."""
        row = np.zeros(nparts, np.int64)
        _check(lib().acgb200_comm_matrix_row(C.byref(self.c), nparts, row), "acgb200_comm_matrix_row")
        return row

    def vector(self) -> Vector:
        v = Vector()
        _check(lib().acgsymcsrmatrix_vector(C.byref(self.c), C.byref(v.c)), "acgsymcsrmatrix_vector")
        lib().acgvector_setzero(C.byref(v.c))
        v._owns = True
        return v

    def p2p_inverse_map(self, rdispl_at_recipient) -> dict:
        """Inverse send map of the peer-memory exchange for this part (host only)."""
        h = acghalo()
        _check(lib().acgsymcsrmatrix_halo(C.byref(self.c), C.byref(h)), "acgsymcsrmatrix_halo")
        nb = self.c.nborderrows
        bptr = np.zeros(nb + 1, np.int32)
        bq = np.zeros(max(h.sendsize, 1), np.int32)
        bdst = np.zeros(max(h.sendsize, 1), np.int32)
        rd = np.ascontiguousarray(rdispl_at_recipient, np.int32)
        code = lib().acgb200_p2p_inverse_map(C.byref(h), self.c.borderrowoffset, nb, rd if len(rd) else np.zeros(1, np.int32),
                                             bptr, bq, bdst)
        n = h.sendsize
        lib().acghalo_free(C.byref(h))
        _check(code, "acgb200_p2p_inverse_map")
        return dict(bptr=bptr, bq=bq[:n], bdst=bdst[:n])

    def halo(self) -> dict:
        h = acghalo()
        _check(lib().acgsymcsrmatrix_halo(C.byref(self.c), C.byref(h)), "acgsymcsrmatrix_halo")
        out = dict(
            recipients=_view(h.recipients, h.nrecipients, np.int32).copy(),
            sendcounts=_view(h.sendcounts, h.nrecipients, np.int32).copy(),
            sdispls=_view(h.sdispls, h.nrecipients, np.int32).copy(),
            sendbufidx=_view(h.sendbufidx, h.sendsize, np.int32).copy(),
            senders=_view(h.senders, h.nsenders, np.int32).copy(),
            recvcounts=_view(h.recvcounts, h.nsenders, np.int32).copy(),
            rdispls=_view(h.rdispls, h.nsenders, np.int32).copy(),
            recvbufidx=_view(h.recvbufidx, h.recvsize, np.int32).copy())
        lib().acghalo_free(C.byref(h))
        return out

    # read-only numpy views of the arrays the device path consumes
    @property
    def rowptr(self): return _view(self.c.rowptr, self.c.nprows + 1, np.int64)
    @property
    def colidx(self): return _view(self.c.colidx, self.c.npnzs, np.int32)
    @property
    def a(self): return _view(self.c.a, self.c.npnzs, np.float64)
    @property
    def nzrows(self): return _view(self.c.nzrows, self.c.nprows, np.int32)
    @property
    def frowptr(self): return _view(self.c.frowptr, self.c.nprows + 1, np.int64)
    @property
    def fcolidx(self): return _view(self.c.fcolidx, self.c.fnpnzs, np.int32)
    @property
    def fa(self): return _view(self.c.fa, self.c.fnpnzs, np.float64)
    @property
    def orowptr(self): return _view(self.c.orowptr, self.c.nborderrows + self.c.nghostrows + 1, np.int64)
    @property
    def ocolidx(self): return _view(self.c.ocolidx, self.c.onpnzs, np.int32)
    @property
    def oa(self): return _view(self.c.oa, self.c.onpnzs, np.float64)

    def free(self):
        if self._owns:
            lib().acgsymcsrmatrix_free(C.byref(self.c))
            self._owns = False

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class Comm:
    """``struct acgcomm`` (acg/comm.h:103): null (single process) or NCCL."""

    def __init__(self):
        self.c = acgcomm()
        self.c.type = 0
        self._nccl = False

    @staticmethod
    def unique_id() -> bytes:
        buf = C.create_string_buffer(128)
        _check(lib().acgb200_nccl_unique_id(buf), "ncclGetUniqueId")
        return buf.raw

    @classmethod
    def init_nccl(cls, nranks: int, rank: int, unique_id: bytes):
        self = cls()
        err = C.c_int(0)
        buf = C.create_string_buffer(unique_id, 128)
        _check(lib().acgb200_comm_init_rank(C.byref(self.c), nranks, buf, rank, C.byref(err)), "ncclCommInitRank", err.value)
        self._nccl = True
        return self

    def size(self) -> int:
        n = C.c_int(0)
        _check(lib().acgcomm_size(C.byref(self.c), C.byref(n)), "acgcomm_size")
        return n.value

    def rank(self) -> int:
        n = C.c_int(0)
        _check(lib().acgcomm_rank(C.byref(self.c), C.byref(n)), "acgcomm_rank")
        return n.value

    def destroy(self):
        if self._nccl:
            lib().acgb200_comm_destroy(C.byref(self.c))
            self._nccl = False


class SolverCuda:
    """``struct acgsolvercuda`` + acgsolvercuda_* (acg/cgcuda.h:68-300)."""

    def __init__(self, A: SymCsrMatrix, comm: Comm | None = None):
        self.c = acgsolvercuda()
        self.A = A
        self.comm = comm if comm is not None else Comm()
        self._live = False
        _check(lib().acgsolvercuda_init(C.byref(self.c), C.byref(A.c), None, None, C.byref(self.comm.c)),
               "acgsolvercuda_init")
        self._live = True

    def _solve(self, fn_name, b: Vector, x: Vector, maxits, diffatol, diffrtol, residualatol, residualrtol, warmup,
               raise_on_not_converged):
        L = lib()
        err = C.c_int(0)
        args = [C.byref(self.c), C.byref(self.A.c), C.byref(b.c), C.byref(x.c), int(maxits),
                float(diffatol), float(diffrtol), float(residualatol), float(residualrtol), int(warmup),
                C.byref(self.comm.c)]
        if fn_name == "solvempi":
            code = L.acgsolvercuda_solvempi(*args, 0, C.byref(err), None, None, 0)
        elif fn_name == "solve_pipelined":
            code = L.acgsolvercuda_solve_pipelined(*args, 0, C.byref(err), None, None)
        elif fn_name == "solve_device":
            code = L.acgsolvercuda_solve_device(*args, C.byref(err))
        elif fn_name == "solve_device_pipelined":
            code = L.acgsolvercuda_solve_device_pipelined(*args, C.byref(err))
        else:
            raise ValueError(fn_name)
        if code != ACG_SUCCESS and (raise_on_not_converged or code != ACG_ERR_NOT_CONVERGED):
            raise AcgError(code, f"acgsolvercuda_{fn_name}", err.value)
        return code

    def solvempi(self, b, x, maxits=100, diffatol=0.0, diffrtol=0.0, residualatol=0.0, residualrtol=0.0,
                 warmup=0, raise_on_not_converged=False):
        return self._solve("solvempi", b, x, maxits, diffatol, diffrtol, residualatol, residualrtol, warmup,
                           raise_on_not_converged)

    def solve_pipelined(self, b, x, maxits=100, diffatol=0.0, diffrtol=0.0, residualatol=0.0, residualrtol=0.0,
                        warmup=0, raise_on_not_converged=False):
        return self._solve("solve_pipelined", b, x, maxits, diffatol, diffrtol, residualatol, residualrtol, warmup,
                           raise_on_not_converged)

    def solve_device(self, b, x, maxits=100, diffatol=0.0, diffrtol=0.0, residualatol=0.0, residualrtol=0.0,
                     warmup=0, raise_on_not_converged=False):
        """acgsolvercuda_solve_device: the classic loop (control and communication are
        device-resident in every loop of this library); NVSHMEM communicators are refused."""
        return self._solve("solve_device", b, x, maxits, diffatol, diffrtol, residualatol, residualrtol, warmup,
                           raise_on_not_converged)

    def solve_device_pipelined(self, b, x, maxits=100, diffatol=0.0, diffrtol=0.0, residualatol=0.0,
                               residualrtol=0.0, warmup=0, raise_on_not_converged=False):
        return self._solve("solve_device_pipelined", b, x, maxits, diffatol, diffrtol, residualatol, residualrtol,
                           warmup, raise_on_not_converged)

    def solve(self, b, x, maxits=100, diffatol=0.0, diffrtol=0.0, residualatol=0.0, residualrtol=0.0, warmup=0,
              raise_on_not_converged=False):
        """acgsolvercuda_solve (acg/cgcuda.h:165, declared but not defined in the reference):
        classic CG on one GPU without a communicator."""
        code = lib().acgsolvercuda_solve(C.byref(self.c), C.byref(self.A.c), C.byref(b.c), C.byref(x.c), int(maxits),
                                         float(diffatol), float(diffrtol), float(residualatol), float(residualrtol),
                                         int(warmup))
        if code != ACG_SUCCESS and (raise_on_not_converged or code != ACG_ERR_NOT_CONVERGED):
            raise AcgError(code, "acgsolvercuda_solve", 0)
        return code

    def spmv(self, x: np.ndarray, nrep: int = 0):
        """y = A x on the device (host arrays in/out); returns (y, ms_per_spmv)."""
        x = np.ascontiguousarray(x, np.float64)
        y = np.zeros(self.A.c.nownedrows, np.float64)
        ms = C.c_double(0)
        _check(lib().acgsolvercuda_spmv(C.byref(self.c), x, y, nrep, C.byref(ms)), "acgsolvercuda_spmv")
        return y, ms.value

    def spmv_ghost(self, x: np.ndarray, path: int):
        """One part's share of y = A x with the ghost entries of x given (acgsolvercuda_spmv_ghost);
        returns (y over the owned rows, fused dot x.y)."""
        x = np.ascontiguousarray(x, np.float64)
        assert len(x) == self.c.r.num_nonzeros
        y = np.zeros(self.A.c.nownedrows, np.float64)
        dot = C.c_double(0)
        _check(lib().acgsolvercuda_spmv_ghost(C.byref(self.c), x, y, path, C.byref(dot)), "acgsolvercuda_spmv_ghost")
        return y, dot.value

    SPMV_Y_AX, SPMV_Y_AX_DOT, SPMV_R_B_AX = 0, 1, 2

    def spmv_mode(self, mode: int, x: np.ndarray, b: np.ndarray | None = None, path: int = 0):
        """The product in one of the SpMV epilogue modes (acgsolvercuda_spmv_mode): mode 0 y = A x,
        1 y = A x with dot = x.y, 2 y = b - A x with dot = y.y.  x has the owned + ghost entries,
        b the owned rows (mode 2).  Returns (y over the owned rows, fused dot)."""
        x = np.ascontiguousarray(x, np.float64)
        assert len(x) == self.c.r.num_nonzeros
        no = self.A.c.nownedrows
        bp = None
        if b is not None:
            b = np.ascontiguousarray(b, np.float64)
            assert len(b) == no
            bp = b.ctypes.data_as(C.c_void_p)
        y = np.zeros(no, np.float64)
        dot = C.c_double(0)
        _check(lib().acgsolvercuda_spmv_mode(C.byref(self.c), int(mode), x, bp, y, int(path), C.byref(dot)),
               "acgsolvercuda_spmv_mode")
        return y, dot.value

    def _block(self, M, name):
        if not (isinstance(M, np.ndarray) and M.dtype == np.float64 and M.ndim == 2 and M.flags.c_contiguous):
            raise ValueError(f"{name} must be a C-contiguous float64 array of shape (n, k)")
        if M.shape[0] != self.A.c.nownedrows:
            raise ValueError(f"{name} has shape {M.shape}: want ({self.A.c.nownedrows}, k)")
        return M

    def solve_multi(self, B, X, maxits=100, residualatol=0.0, residualrtol=0.0, warmup=0,
                    raise_on_not_converged=False):
        """acgsolvercuda_solve_multi: classic CG on the k columns of B at once, one pass over the matrix
        per iteration for all of them; each column runs exactly the recurrence ``solvempi`` runs for it
        alone.  B and X are C-contiguous float64 arrays of shape (n, k), 1 <= k <= 8; X holds the initial
        guesses and is updated in place.  Returns (code, [per-column dict of niterations, converged,
        bnrm2, r0nrm2, rnrm2])."""
        B = self._block(B, "B")
        X = self._block(X, "X")
        if B.shape != X.shape:
            raise ValueError(f"B {B.shape} and X {X.shape} differ")
        k = B.shape[1]
        st = (acgb200_colstats * k)()
        code = lib().acgsolvercuda_solve_multi(C.byref(self.c), C.byref(self.A.c), k, B, X, int(maxits),
                                               float(residualatol), float(residualrtol), int(warmup), st)
        if code != ACG_SUCCESS and (raise_on_not_converged or code != ACG_ERR_NOT_CONVERGED):
            raise AcgError(code, "acgsolvercuda_solve_multi", 0)
        return code, [{n: getattr(s, n) for n, _ in acgb200_colstats._fields_} for s in st]

    def solve_shifted(self, b, shifts, maxits=100, residualatol=0.0, residualrtol=0.0, warmup=0,
                      raise_on_not_converged=False):
        """acgsolvercuda_solve_shifted: (A + shifts[j] I) x_j = b for 1 <= S <= 8 finite shifts >= 0 in one
        Krylov space (multi-shift CG): one product per iteration for all shifts.  Every system starts from
        x0 = 0; shift j stops by the rule ``solvempi`` applies to that system alone.  b: float64 array of
        the owned rows.  Returns (code, X of shape (n, S), [per-shift dict of niterations, converged,
        bnrm2, r0nrm2, rnrm2])."""
        b = np.ascontiguousarray(b, np.float64)
        if b.shape != (self.A.c.nownedrows,):
            raise ValueError(f"b has shape {b.shape}: want ({self.A.c.nownedrows},)")
        shifts = np.ascontiguousarray(np.atleast_1d(np.asarray(shifts, np.float64)))
        if shifts.ndim != 1:
            raise ValueError(f"shifts must be one-dimensional, not of shape {shifts.shape}")
        S = len(shifts)
        X = self._block(np.zeros((self.A.c.nownedrows, max(S, 1)), np.float64), "X")
        st = (acgb200_colstats * max(S, 1))()
        code = lib().acgsolvercuda_solve_shifted(C.byref(self.c), C.byref(self.A.c), S,
                                                 shifts if S else np.zeros(1), b, X, int(maxits),
                                                 float(residualatol), float(residualrtol), int(warmup), st)
        if code != ACG_SUCCESS and (raise_on_not_converged or code != ACG_ERR_NOT_CONVERGED):
            raise AcgError(code, "acgsolvercuda_solve_shifted", 0)
        return code, X, [{n: getattr(s, n) for n, _ in acgb200_colstats._fields_} for s in st[:S]]

    def solve_minres(self, b, x, maxits=100, residualatol=0.0, residualrtol=0.0, warmup=0,
                     raise_on_not_converged=False):
        """acgsolvercuda_solve_minres: MINRES on the solver's operator, which may be indefinite or singular
        (one GPU, whole matrix).  b, x: Vectors as for ``solvempi``, x the initial guess, updated in place.
        Stops by ``solvempi``'s rule on MINRES's recursively updated residual norm (``c.rnrm2``), or on an
        exact Krylov breakdown.  Returns the code like ``solve()``."""
        err = C.c_int(0)
        code = lib().acgsolvercuda_solve_minres(C.byref(self.c), C.byref(self.A.c), C.byref(b.c), C.byref(x.c),
                                                int(maxits), float(residualatol), float(residualrtol), int(warmup),
                                                C.byref(err))
        if code != ACG_SUCCESS and (raise_on_not_converged or code != ACG_ERR_NOT_CONVERGED):
            raise AcgError(code, "acgsolvercuda_solve_minres", err.value)
        return code

    def solve_chebyshev(self, b, x, degree=2, lmin=0.0, lmax=0.0, maxits=100, residualatol=0.0, residualrtol=0.0,
                        warmup=0, raise_on_not_converged=False):
        """acgsolvercuda_solve_chebyshev: CG preconditioned with a degree-``degree`` Chebyshev polynomial in
        D^-1 A over [lmin, lmax] (degree 0: Jacobi) on the solver's (positive definite) operator (one GPU, whole
        matrix).  lmax = 0 estimates the upper bound from 10 Jacobi-PCG steps, lmin = 0 takes lmax / 10.  b, x:
        Vectors as for ``solvempi``, x the initial guess, updated in place.  ``info()`` reports cheb_degree,
        cheb_est_iterations, cheb_breakdown and the interval used (cheb_lmin, cheb_lmax).  Returns the code
        like ``solve()``."""
        err = C.c_int(0)
        code = lib().acgsolvercuda_solve_chebyshev(C.byref(self.c), C.byref(self.A.c), C.byref(b.c), C.byref(x.c),
                                                   int(degree), float(lmin), float(lmax), int(maxits),
                                                   float(residualatol), float(residualrtol), int(warmup),
                                                   C.byref(err))
        if code != ACG_SUCCESS and (raise_on_not_converged or code != ACG_ERR_NOT_CONVERGED):
            raise AcgError(code, "acgsolvercuda_solve_chebyshev", err.value)
        return code

    def solve_mixed(self, b, x, maxits=100, residualatol=0.0, residualrtol=0.0, warmup=0,
                    raise_on_not_converged=False):
        """acgsolvercuda_solve_mixed: CG with float vectors and reliable updates to an fp64 tolerance on
        the solver's (positive definite) operator (one GPU, whole matrix).  b, x: Vectors as for
        ``solvempi``, x the initial guess, updated in place.  ``c.rnrm2`` is the fp64 residual of the x
        returned; ``info()["mixed_reliable_updates"]`` counts the reliable updates.  Returns the code like
        ``solve()``."""
        err = C.c_int(0)
        code = lib().acgsolvercuda_solve_mixed(C.byref(self.c), C.byref(self.A.c), C.byref(b.c), C.byref(x.c),
                                               int(maxits), float(residualatol), float(residualrtol), int(warmup),
                                               C.byref(err))
        if code != ACG_SUCCESS and (raise_on_not_converged or code != ACG_ERR_NOT_CONVERGED):
            raise AcgError(code, "acgsolvercuda_solve_mixed", err.value)
        return code

    def spmv_f32(self, x: np.ndarray):
        """The fp32 product of solve_mixed (acgsolvercuda_spmv_f32): y = fl32(A x) for float32 x over the
        owned rows, each row summed in fp64.  Returns (y as float32, the fp64 dot x.y)."""
        no = self.A.c.nownedrows
        x = np.ascontiguousarray(x, np.float32)
        assert len(x) == no
        y = np.zeros(no, np.float32)
        dot = C.c_double(0)
        _check(lib().acgsolvercuda_spmv_f32(C.byref(self.c), x, y, C.byref(dot)), "acgsolvercuda_spmv_f32")
        return y, dot.value

    def spmm_mode(self, mode: int, X: np.ndarray, B: np.ndarray | None = None):
        """The multi-vector product of solve_multi in one of the epilogue modes (acgsolvercuda_spmm_mode):
        mode 0 Y = A X, 1 Y = A X with dots[j] = x_j.y_j, 2 Y = B - A X with dots[j] = y_j.y_j.
        X, B: float64 (n, k).  Returns (Y, dots)."""
        X = self._block(np.ascontiguousarray(X, np.float64), "X")
        k = X.shape[1]
        bp = None
        if B is not None:
            B = self._block(np.ascontiguousarray(B, np.float64), "B")
            bp = B.ctypes.data_as(C.c_void_p)
        Y = np.zeros_like(X)
        dots = (C.c_double * k)()
        _check(lib().acgsolvercuda_spmm_mode(C.byref(self.c), int(mode), k, X, bp, Y, dots), "acgsolvercuda_spmm_mode")
        return Y, np.array(dots[:], np.float64)

    def update_values(self, A: SymCsrMatrix):
        """acgsolvercuda_update_values: take A's values (full storage if A has it, else its packed triangle)
        into the solver, keeping every plan built from the pattern.  A must have the partition and pattern of
        the matrix the solver was built on; anything else raises with the solver unchanged.  Solves then take
        A as their matrix."""
        err = C.c_int(0)
        _check(lib().acgsolvercuda_update_values(C.byref(self.c), C.byref(A.c), C.byref(err)),
               "acgsolvercuda_update_values", err.value)
        self.A = A

    def info(self) -> dict:
        inf = acgb200_info()
        _check(lib().acgsolvercuda_info(C.byref(self.c), C.byref(inf)), "acgsolvercuda_info")
        return {n: getattr(inf, n) for n, _ in acgb200_info._fields_}

    def stats(self) -> dict:
        keys = ["maxits", "bnrm2", "r0nrm2", "rnrm2", "nsolves", "ntotaliterations", "niterations", "nflops",
                "tsolve", "tgemv", "taxpy", "ngemv", "Bgemv", "naxpy", "Baxpy", "nallreduce", "nhalo", "Bhalo"]
        return {k: getattr(self.c, k) for k in keys}

    TIMES = ("tsolve", "tgemv", "tdot", "tnrm2", "taxpy", "tcopy", "tallreduce", "thalo")
    COUNTERS = ("nflops", "Bgemv", "Bdot", "Bnrm2", "Baxpy", "Bcopy", "Ballreduce", "Bhalo", "nhalomsgs")

    def report(self, aggregate=None) -> str:
        """acgsolvercuda_fwrite into a string.  ``aggregate``: dict of field values to print instead of
        this rank's (times as the maximum, flop/byte/message counters as the sum over the ranks: what
        acgsolvercuda_fwritempi reduces with MPI, acg/cgcuda.c:1990-2012)."""
        src = self.c
        if aggregate:
            src = acgsolvercuda()
            C.memmove(C.byref(src), C.byref(self.c), C.sizeof(acgsolvercuda))
            for k, v in aggregate.items():
                setattr(src, k, v)
        return self._fwrite(src)

    def _fwrite(self, struct) -> str:
        libc = C.CDLL(None)
        libc.fopen.restype = C.c_void_p
        libc.fopen.argtypes = [C.c_char_p, C.c_char_p]
        libc.fclose.argtypes = [C.c_void_p]
        with tempfile.NamedTemporaryFile("r", suffix=".txt") as tf:
            f = libc.fopen(tf.name.encode(), b"w")
            _check(lib().acgsolvercuda_fwrite(f, C.byref(struct), 0), "acgsolvercuda_fwrite")
            libc.fclose(f)
            return tf.read()

    def free(self):
        if self._live:
            lib().acgsolvercuda_free(C.byref(self.c))
            self._live = False

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass
