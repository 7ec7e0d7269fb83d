"""splatt_b200 -- an H100-native MTTKRP engine behind SPLATT's C API.

The product is splatt_b200/libsplatt_b200.so (hand-written sm_90a CUDA, C ABI in
include/splatt_b200.h).  This package is the thin Python host layer over it.
"""
from . import _abi  # noqa: F401
from .api import (Csf, MttkrpWorkspace, MultiGpu, SplattError, Tensor, build_count,  # noqa: F401
                  cache_clear, cpd_als, csf_alloc, default_opts, launch_count, mttkrp)

__all__ = ["Csf", "MttkrpWorkspace", "MultiGpu", "SplattError", "Tensor", "build_count",
           "cache_clear", "cpd_als", "csf_alloc", "default_opts", "launch_count", "mttkrp"]
