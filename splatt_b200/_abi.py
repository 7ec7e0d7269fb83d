"""ctypes view of include/splatt_b200.h: struct layouts, constants and the loader.

The library is the product; there is no Python/CPU fallback.  `load()` raises if
libsplatt_b200.so has not been built (run `python -m splatt_b200.build`).
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

MAX_NMODES = 8

SPLATT_SUCCESS = 1
SPLATT_ERROR_BADINPUT = 2
SPLATT_ERROR_NOMEMORY = 3

# option slots (include/splatt_b200.h, reference include/splatt/types_config.h:103-123)
(OPTION_NTHREADS, OPTION_TOLERANCE, OPTION_REGULARIZE, OPTION_NITER, OPTION_VERBOSITY,
 OPTION_RANDSEED, OPTION_CSF_ALLOC, OPTION_TILE, OPTION_TILELEVEL, OPTION_PRIVTHRESH,
 OPTION_DECOMP, OPTION_COMM, OPTION_NOPTIONS) = range(13)

CSF_ONEMODE, CSF_TWOMODE, CSF_ALLMODE = 0, 1, 2
NOTILE, DENSETILE = 0, 1
VERBOSITY_NONE, VERBOSITY_LOW, VERBOSITY_HIGH, VERBOSITY_MAX = 0, 1, 2, 3
LAYOUT_ALLROOT, LAYOUT_ASGIVEN = 0, 1
KIND_NAMES = {0: "root", 1: "internal", 2: "leaf"}

idx_t = C.c_uint64
val_t = C.c_double
idx_p = C.POINTER(idx_t)
val_p = C.POINTER(val_t)
f32_p = C.POINTER(C.c_float)


class CsfSparsity(C.Structure):
    _fields_ = [("nfibs", idx_t * MAX_NMODES),
                ("fptr", idx_p * MAX_NMODES),
                ("fids", idx_p * MAX_NMODES),
                ("vals", val_p)]


class SplattCsf(C.Structure):
    _fields_ = [("nnz", idx_t),
                ("nmodes", idx_t),
                ("dims", idx_t * MAX_NMODES),
                ("dim_perm", idx_t * MAX_NMODES),
                ("dim_iperm", idx_t * MAX_NMODES),
                ("which_tile", C.c_int),
                ("ntiles", idx_t),
                ("ntiled_modes", idx_t),
                ("tile_dims", idx_t * MAX_NMODES),
                ("pt", C.POINTER(CsfSparsity))]


class SplattKruskal(C.Structure):
    _fields_ = [("rank", idx_t),
                ("factors", val_p * MAX_NMODES),
                ("lambda_", val_p),
                ("nmodes", idx_t),
                ("dims", idx_t * MAX_NMODES),
                ("fit", C.c_double)]


class MttkrpWs(C.Structure):
    _fields_ = [("num_csf", idx_t),
                ("mode_csf_map", idx_t * MAX_NMODES),
                ("num_threads", idx_t),
                ("tile_partition", idx_p * MAX_NMODES),
                ("tree_partition", idx_p * MAX_NMODES),
                ("is_privatized", C.c_bool * MAX_NMODES),
                ("privatize_buffer", C.POINTER(val_p)),
                ("reduction_time", C.c_double)]


class Matrix(C.Structure):
    _fields_ = [("I", idx_t), ("J", idx_t), ("vals", val_p), ("rowmajor", C.c_int)]


class BuildOpts(C.Structure):
    _fields_ = [("layout", C.c_int32), ("device", C.c_int32), ("shard_rank", C.c_int32),
                ("shard_count", C.c_int32), ("verbosity", C.c_int32),
                ("ncolumns_hint", C.c_int32), ("ktile", C.c_int32),
                ("reserved", C.c_int32 * 9)]


class GroupSync(C.Structure):
    _fields_ = [("mc_flag", C.c_void_p), ("local_flag", C.c_void_p), ("target", C.c_uint32),
                ("rank", C.c_uint32), ("world", C.c_uint32), ("reserved", C.c_uint32)]


LIB_PATH = Path(__file__).resolve().parent / "libsplatt_b200.so"

# every symbol include/splatt_b200.h declares
EXPORTS = [
    "splatt_mttkrp", "splatt_mttkrp_alloc_ws", "splatt_mttkrp_free_ws", "splatt_mttkrp_csf",
    "splatt_cpd_als", "splatt_free_kruskal", "splatt_default_opts", "splatt_free_opts",
    "splatt_b200_tensor_from_csf", "splatt_b200_tensor_from_coo", "splatt_b200_tensor_free",
    "splatt_b200_tensor_info", "splatt_b200_mode_info", "splatt_b200_csf_alloc",
    "splatt_b200_csf_free", "splatt_b200_mttkrp", "splatt_b200_mttkrp_f32", "splatt_b200_launch_count",
    "splatt_b200_version", "splatt_b200_level_orders", "splatt_b200_cta_tiling", "splatt_b200_shard_range", "splatt_b200_mttkrp_multicast", "splatt_b200_gather_probe", "splatt_b200_gather_probe_ex", "splatt_b200_mttkrp_columns",
    "splatt_b200_als_tail_create", "splatt_b200_als_tail_free", "splatt_b200_als_tail_gram",
    "splatt_b200_als_tail_update", "splatt_b200_als_tail_fit", "splatt_b200_csf_to_coo",
    "splatt_b200_als_tail_gram_f32", "splatt_b200_als_tail_update_f32",
    "splatt_b200_als_tail_fit_f32", "splatt_b200_cpd_als_device", "splatt_b200_cpd_als_device_f32",
    "splatt_b200_tensor_shard", "splatt_b200_mttkrp_multicast_sync",
    "splatt_b200_mttkrp_multicast_sync_columns", "splatt_b200_tensor_sse", "splatt_b200_tc_als_device",
    "splatt_b200_multi_env_devices", "splatt_b200_multi_create", "splatt_b200_multi_free",
    "splatt_b200_multi_info", "splatt_b200_multi_mttkrp_host", "splatt_b200_multi_cpd_als",
    "splatt_b200_multi_last_ms", "splatt_b200_build_count", "splatt_b200_cache_clear",
]

_lib = None


def load() -> C.CDLL:
    """Load libsplatt_b200.so and declare prototypes.  Fails loudly if absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise RuntimeError(
            f"{LIB_PATH} is missing: the CUDA extension is the product and there is no "
            "fallback.  Build it with `python -m splatt_b200.build`.")
    lib = C.CDLL(str(LIB_PATH))
    vpp = C.POINTER(val_p)
    csf_p = C.POINTER(SplattCsf)
    u32pp = C.POINTER(C.POINTER(C.c_uint32))

    lib.splatt_mttkrp.restype = C.c_int
    lib.splatt_mttkrp.argtypes = [idx_t, idx_t, csf_p, vpp, val_p, C.POINTER(C.c_double)]
    lib.splatt_mttkrp_alloc_ws.restype = C.POINTER(MttkrpWs)
    lib.splatt_mttkrp_alloc_ws.argtypes = [csf_p, idx_t, C.POINTER(C.c_double)]
    lib.splatt_mttkrp_free_ws.restype = None
    lib.splatt_mttkrp_free_ws.argtypes = [C.POINTER(MttkrpWs)]
    lib.splatt_mttkrp_csf.restype = None
    lib.splatt_mttkrp_csf.argtypes = [csf_p, C.POINTER(C.POINTER(Matrix)), idx_t, C.c_void_p,
                                      C.POINTER(MttkrpWs), C.POINTER(C.c_double)]
    lib.splatt_cpd_als.restype = C.c_int
    lib.splatt_cpd_als.argtypes = [csf_p, idx_t, C.POINTER(C.c_double), C.POINTER(SplattKruskal)]
    lib.splatt_free_kruskal.restype = None
    lib.splatt_free_kruskal.argtypes = [C.POINTER(SplattKruskal)]
    lib.splatt_default_opts.restype = C.POINTER(C.c_double)
    lib.splatt_default_opts.argtypes = []
    lib.splatt_free_opts.restype = None
    lib.splatt_free_opts.argtypes = [C.POINTER(C.c_double)]

    lib.splatt_b200_tensor_from_csf.restype = C.c_int
    lib.splatt_b200_tensor_from_csf.argtypes = [csf_p, C.c_int, C.POINTER(BuildOpts),
                                                C.POINTER(C.c_void_p)]
    lib.splatt_b200_tensor_from_coo.restype = C.c_int
    lib.splatt_b200_tensor_from_coo.argtypes = [C.c_int, idx_p, C.c_uint64, u32pp, val_p, C.c_int,
                                                C.c_int, C.POINTER(BuildOpts),
                                                C.POINTER(C.c_void_p)]
    lib.splatt_b200_tensor_free.restype = None
    lib.splatt_b200_tensor_free.argtypes = [C.c_void_p]
    lib.splatt_b200_tensor_info.restype = C.c_int
    lib.splatt_b200_tensor_info.argtypes = [C.c_void_p, C.POINTER(C.c_int), idx_p, idx_p, idx_p,
                                            idx_p]
    lib.splatt_b200_mode_info.restype = C.c_int
    lib.splatt_b200_mode_info.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_int),
                                          C.POINTER(C.c_int), idx_p, idx_p]
    lib.splatt_b200_csf_alloc.restype = C.c_int
    lib.splatt_b200_csf_alloc.argtypes = [C.c_int, idx_p, C.c_uint64, u32pp, val_p, C.c_int,
                                          C.c_int, C.POINTER(csf_p)]
    lib.splatt_b200_csf_free.restype = None
    lib.splatt_b200_csf_free.argtypes = [csf_p, C.c_int]
    lib.splatt_b200_mttkrp.restype = C.c_int
    lib.splatt_b200_mttkrp.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, vpp, val_p,
                                       C.c_void_p]
    lib.splatt_b200_mttkrp_f32.restype = C.c_int
    lib.splatt_b200_mttkrp_f32.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int,
                                           C.POINTER(f32_p), f32_p, C.c_void_p]
    lib.splatt_b200_mttkrp_multicast.restype = C.c_int
    lib.splatt_b200_mttkrp_multicast.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, vpp, val_p,
                                                 C.c_void_p]
    lib.splatt_b200_mttkrp_columns.restype = C.c_int
    lib.splatt_b200_mttkrp_columns.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, vpp, val_p,
                                               C.c_int, C.c_int, C.c_void_p]
    lib.splatt_b200_als_tail_create.restype = C.c_int
    lib.splatt_b200_als_tail_create.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p,
                                                C.POINTER(C.c_void_p)]
    lib.splatt_b200_als_tail_free.restype = None
    lib.splatt_b200_als_tail_free.argtypes = [C.c_void_p]
    lib.splatt_b200_als_tail_gram.restype = C.c_int
    lib.splatt_b200_als_tail_gram.argtypes = [C.c_void_p, C.c_int, val_p, C.c_uint64]
    lib.splatt_b200_als_tail_update.restype = C.c_int
    lib.splatt_b200_als_tail_update.argtypes = [C.c_void_p, C.c_int, val_p, val_p, C.c_uint64,
                                                C.c_int]
    lib.splatt_b200_als_tail_fit.restype = C.c_int
    lib.splatt_b200_als_tail_fit.argtypes = [C.c_void_p, val_p, val_p, C.c_uint64, C.c_double,
                                             C.POINTER(C.c_double), val_p]
    lib.splatt_b200_als_tail_gram_f32.restype = C.c_int
    lib.splatt_b200_als_tail_gram_f32.argtypes = [C.c_void_p, C.c_int, f32_p, C.c_uint64]
    lib.splatt_b200_als_tail_update_f32.restype = C.c_int
    lib.splatt_b200_als_tail_update_f32.argtypes = [C.c_void_p, C.c_int, f32_p, f32_p, C.c_uint64,
                                                    C.c_int]
    lib.splatt_b200_als_tail_fit_f32.restype = C.c_int
    lib.splatt_b200_als_tail_fit_f32.argtypes = [C.c_void_p, f32_p, f32_p, C.c_uint64, C.c_double,
                                                 C.POINTER(C.c_double), val_p]
    lib.splatt_b200_cpd_als_device.restype = C.c_int
    lib.splatt_b200_cpd_als_device.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_double),
                                               vpp, val_p, C.POINTER(C.c_double),
                                               C.POINTER(C.c_int), C.c_void_p]
    lib.splatt_b200_cpd_als_device_f32.restype = C.c_int
    lib.splatt_b200_cpd_als_device_f32.argtypes = [C.c_void_p, C.c_int, C.c_int,
                                                   C.POINTER(C.c_double), C.POINTER(f32_p), val_p,
                                                   C.POINTER(C.c_double), C.POINTER(C.c_int),
                                                   C.c_void_p]
    lib.splatt_b200_tensor_sse.restype = C.c_int
    lib.splatt_b200_tensor_sse.argtypes = [C.c_void_p, C.c_int, C.c_int, vpp, val_p,
                                           C.POINTER(C.c_double), C.c_void_p]
    lib.splatt_b200_tc_als_device.restype = C.c_int
    lib.splatt_b200_tc_als_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                              C.POINTER(C.c_double), vpp, val_p,
                                              C.POINTER(C.c_int), C.c_void_p]
    lib.splatt_b200_csf_to_coo.restype = C.c_int
    lib.splatt_b200_csf_to_coo.argtypes = [csf_p, u32pp, val_p]
    lib.splatt_b200_gather_probe.restype = C.c_int
    lib.splatt_b200_gather_probe.argtypes = [val_p, C.c_int, C.c_int, C.POINTER(C.c_uint32),
                                             C.c_uint64, val_p, C.c_void_p]
    lib.splatt_b200_gather_probe_ex.restype = C.c_int
    lib.splatt_b200_gather_probe_ex.argtypes = [val_p, C.c_int, C.c_int, C.POINTER(C.c_uint32),
                                                C.c_uint64, val_p, C.c_int, C.c_int, C.c_int,
                                                C.c_int, C.c_void_p]
    lib.splatt_b200_tensor_shard.restype = C.c_int
    lib.splatt_b200_tensor_shard.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int,
                                             C.POINTER(C.c_void_p)]
    lib.splatt_b200_mttkrp_multicast_sync.restype = C.c_int
    lib.splatt_b200_mttkrp_multicast_sync.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, vpp,
                                                      val_p, C.POINTER(GroupSync), C.c_void_p]
    lib.splatt_b200_mttkrp_multicast_sync_columns.restype = C.c_int
    lib.splatt_b200_mttkrp_multicast_sync_columns.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int,
                                                              vpp, val_p, C.c_int, C.c_int,
                                                              C.POINTER(GroupSync), C.c_void_p]
    lib.splatt_b200_multi_env_devices.restype = C.c_int
    lib.splatt_b200_multi_env_devices.argtypes = [C.POINTER(C.c_int), C.c_int]
    lib.splatt_b200_multi_create.restype = C.c_int
    lib.splatt_b200_multi_create.argtypes = [csf_p, C.c_int, C.c_int, C.POINTER(C.c_int), C.c_int,
                                             C.c_int, C.POINTER(C.c_void_p)]
    lib.splatt_b200_multi_free.restype = None
    lib.splatt_b200_multi_free.argtypes = [C.c_void_p]
    lib.splatt_b200_multi_info.restype = C.c_int
    lib.splatt_b200_multi_info.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int),
                                           idx_p, idx_p]
    lib.splatt_b200_multi_mttkrp_host.restype = C.c_int
    lib.splatt_b200_multi_mttkrp_host.argtypes = [C.c_void_p, C.c_int, vpp, val_p]
    lib.splatt_b200_multi_cpd_als.restype = C.c_int
    lib.splatt_b200_multi_cpd_als.argtypes = [C.c_void_p, csf_p, C.POINTER(C.c_double),
                                              C.POINTER(SplattKruskal)]
    lib.splatt_b200_multi_last_ms.restype = C.c_double
    lib.splatt_b200_multi_last_ms.argtypes = [C.c_void_p]
    lib.splatt_b200_build_count.restype = C.c_uint64
    lib.splatt_b200_build_count.argtypes = []
    lib.splatt_b200_cache_clear.restype = None
    lib.splatt_b200_cache_clear.argtypes = []
    lib.splatt_b200_launch_count.restype = C.c_uint64
    lib.splatt_b200_launch_count.argtypes = []
    lib.splatt_b200_version.restype = C.c_char_p
    lib.splatt_b200_version.argtypes = []
    lib.splatt_b200_level_orders.restype = C.c_int
    lib.splatt_b200_level_orders.argtypes = [idx_p, C.c_int, C.c_int, C.POINTER(C.c_int),
                                             C.POINTER(C.c_int)]
    lib.splatt_b200_cta_tiling.restype = C.c_int
    lib.splatt_b200_cta_tiling.argtypes = [C.c_int, idx_p, C.POINTER(C.c_int), C.c_uint64, C.c_int,
                                           C.c_int, C.c_int, C.c_int, C.POINTER(C.c_uint32),
                                           C.POINTER(C.c_uint32)]
    lib.splatt_b200_shard_range.restype = None
    lib.splatt_b200_shard_range.argtypes = [C.c_uint64, C.c_int, C.c_int, idx_p, idx_p]
    _lib = lib
    return lib
