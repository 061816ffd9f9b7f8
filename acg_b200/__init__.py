"""acg_b200 -- H100-native conjugate-gradient hot path behind aCG's C interface.

The product is ``libacgb200.so`` (C host code + hand-written sm_90a CUDA
kernels, sources under ``acg_b200/csrc``, public C-ABI under ``include/``).
This package is only the ctypes mirror of that interface plus host-side
synthetic matrix generators.
"""
from . import matgen  # noqa: F401
from .api import (AcgError, Comm, SolverCuda, SymCsrMatrix, Vector, build, lib, mtx_info, set_option, spmv_plan_host, patterns_host, slices_host, symdiag_host, merge_plan_host)  # noqa: F401
