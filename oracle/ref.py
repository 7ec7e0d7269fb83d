"""ctypes wrapper over oracle/_ref/libsplatt_ref.so (the unmodified reference +
ref_driver.c).  TEST INFRASTRUCTURE ONLY -- see oracle/__init__.py."""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path
from typing import Optional, Sequence

import numpy as np

from splatt_b200 import _abi as A   # struct layouts only (the ABI is shared)

HERE = Path(__file__).resolve().parent
LIB_PATH = HERE / "_ref" / "libsplatt_ref.so"
CLI_PATH = HERE / "_ref" / "splatt"

_lib = None


def available() -> bool:
    return LIB_PATH.exists()


def load() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise RuntimeError(f"{LIB_PATH} missing; run oracle/build_ref.sh where the reference sources exist")
    lib = C.CDLL(str(LIB_PATH), mode=os.RTLD_LOCAL)
    u64p = C.POINTER(C.c_uint64)
    u64pp = C.POINTER(u64p)
    dp = C.POINTER(C.c_double)
    dpp = C.POINTER(dp)
    csf_p = C.POINTER(A.SplattCsf)
    lib.refdrv_tt_from_coo.restype = C.c_void_p
    lib.refdrv_tt_from_coo.argtypes = [C.c_uint64, u64p, C.c_uint64, u64pp, dp]
    lib.refdrv_tt_read.restype = C.c_void_p
    lib.refdrv_tt_read.argtypes = [C.c_char_p]
    lib.refdrv_tt_free.restype = None
    lib.refdrv_tt_free.argtypes = [C.c_void_p]
    lib.refdrv_tt_nmodes.restype = C.c_uint64
    lib.refdrv_tt_nmodes.argtypes = [C.c_void_p]
    lib.refdrv_tt_nnz.restype = C.c_uint64
    lib.refdrv_tt_nnz.argtypes = [C.c_void_p]
    lib.refdrv_tt_dims.restype = None
    lib.refdrv_tt_dims.argtypes = [C.c_void_p, u64p]
    lib.refdrv_tt_copy_out.restype = None
    lib.refdrv_tt_copy_out.argtypes = [C.c_void_p, u64pp, dp]
    lib.refdrv_tt_remove_empty.restype = C.c_uint64
    lib.refdrv_tt_remove_empty.argtypes = [C.c_void_p]
    lib.refdrv_default_opts.restype = dp
    lib.refdrv_default_opts.argtypes = []
    lib.refdrv_free_opts.restype = None
    lib.refdrv_free_opts.argtypes = [dp]
    lib.refdrv_csf_alloc.restype = csf_p
    lib.refdrv_csf_alloc.argtypes = [C.c_void_p, dp]
    lib.refdrv_csf_free.restype = None
    lib.refdrv_csf_free.argtypes = [csf_p, dp]
    lib.refdrv_mode_order.restype = None
    lib.refdrv_mode_order.argtypes = [u64p, C.c_uint64, C.c_int, C.c_uint64, u64p]
    lib.refdrv_partition_weighted.restype = u64p
    lib.refdrv_partition_weighted.argtypes = [u64p, C.c_uint64, C.c_uint64, u64p]
    lib.refdrv_free.restype = None
    lib.refdrv_free.argtypes = [C.c_void_p]
    lib.refdrv_mttkrp_stream.restype = None
    lib.refdrv_mttkrp_stream.argtypes = [C.c_void_p, C.c_uint64, dpp, C.c_uint64, dp, C.c_int]
    lib.refdrv_mttkrp_csf.restype = None
    lib.refdrv_mttkrp_csf.argtypes = [csf_p, dp, C.c_uint64, dpp, C.c_uint64, dp, C.c_int, C.c_int, dp]
    lib.refdrv_splatt_mttkrp.restype = C.c_int
    lib.refdrv_splatt_mttkrp.argtypes = [C.c_uint64, C.c_uint64, csf_p, dpp, dp, dp]
    lib.refdrv_cpd_als.restype = C.c_double
    lib.refdrv_cpd_als.argtypes = [csf_p, C.c_uint64, dp, C.c_uint, dpp, dp]
    lib.refdrv_abi.restype = C.c_uint64
    lib.refdrv_abi.argtypes = [u64p]
    _lib = lib
    return lib


# csf_mode_type (reference: src/csf.h:18-26)
CSF_SORTED_SMALLFIRST, CSF_SORTED_BIGFIRST, CSF_INORDER_MINUSONE, CSF_SORTED_MINUSONE, \
    CSF_MODE_CUSTOM = range(5)


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def default_opts() -> np.ndarray:
    lib = load()
    p = lib.refdrv_default_opts()
    o = np.ctypeslib.as_array(p, shape=(A.OPTION_NOPTIONS,)).copy()
    lib.refdrv_free_opts(p)
    return o


class RefTensor:
    """A reference sptensor_t (COO)."""

    def __init__(self, handle):
        self.lib = load()
        self.h = handle
        self.nmodes = int(self.lib.refdrv_tt_nmodes(handle))
        self.nnz = int(self.lib.refdrv_tt_nnz(handle))
        d = (C.c_uint64 * 8)()
        self.lib.refdrv_tt_dims(handle, d)
        self.dims = [int(d[m]) for m in range(self.nmodes)]

    @classmethod
    def from_coo(cls, dims, ind, vals) -> "RefTensor":
        lib = load()
        dims_a = np.ascontiguousarray(dims, dtype=np.uint64)
        inds = [np.ascontiguousarray(i, dtype=np.uint64) for i in ind]
        vals_a = np.ascontiguousarray(vals, dtype=np.float64)
        ip = (C.POINTER(C.c_uint64) * len(inds))(
            *[i.ctypes.data_as(C.POINTER(C.c_uint64)) for i in inds])
        h = lib.refdrv_tt_from_coo(len(dims_a), dims_a.ctypes.data_as(C.POINTER(C.c_uint64)),
                                   len(vals_a), ip, _dp(vals_a))
        return cls(h)

    @classmethod
    def read(cls, path: str) -> "RefTensor":
        h = load().refdrv_tt_read(str(path).encode())
        if not h:
            raise RuntimeError(f"reference tt_read failed for {path}")
        return cls(h)

    def coo(self):
        """(ind list of uint64 arrays, vals) in the tensor's CURRENT order."""
        inds = [np.empty(self.nnz, dtype=np.uint64) for _ in range(self.nmodes)]
        vals = np.empty(self.nnz, dtype=np.float64)
        ip = (C.POINTER(C.c_uint64) * self.nmodes)(
            *[i.ctypes.data_as(C.POINTER(C.c_uint64)) for i in inds])
        self.lib.refdrv_tt_copy_out(self.h, ip, _dp(vals))
        return inds, vals

    def mttkrp_stream(self, mats: Sequence[np.ndarray], mode: int, nthreads: int = 1) -> np.ndarray:
        R = mats[(mode + 1) % self.nmodes].shape[1]
        keep = [np.ascontiguousarray(m, dtype=np.float64) if m is not None
                else np.zeros((self.dims[i], R)) for i, m in enumerate(mats)]
        mp = (C.POINTER(C.c_double) * self.nmodes)(*[_dp(k) for k in keep])
        out = np.empty((self.dims[mode], R), dtype=np.float64)
        self.lib.refdrv_mttkrp_stream(self.h, R, mp, mode, _dp(out), nthreads)
        return out

    def free(self):
        if self.h:
            self.lib.refdrv_tt_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class RefCsf:
    """CSF(s) built by the reference's csf_alloc.  NOTE: sorts `tt` in place."""

    def __init__(self, tt: RefTensor, opts: np.ndarray):
        self.lib = load()
        self.opts = np.ascontiguousarray(opts, dtype=np.float64)
        self.ptr = self.lib.refdrv_csf_alloc(tt.h, _dp(self.opts))
        self.csf_alloc = int(self.opts[A.OPTION_CSF_ALLOC])
        self.nmodes = tt.nmodes
        self.dims = list(tt.dims)

    @property
    def count(self) -> int:
        return {A.CSF_ONEMODE: 1, A.CSF_TWOMODE: 2}.get(self.csf_alloc, self.nmodes)

    def arrays(self, c: int = 0, tile: int = 0) -> dict:
        from splatt_b200.api import Csf
        return Csf.arrays(self, c, tile)   # same struct layout

    def _mats(self, mats, R):
        keep = [np.ascontiguousarray(m, dtype=np.float64) if m is not None
                else np.zeros((self.dims[i], R)) for i, m in enumerate(mats)]
        mp = (C.POINTER(C.c_double) * self.nmodes)(*[_dp(k) for k in keep])
        return keep, mp

    def mttkrp_csf(self, mats, mode: int, *, warm: int = 0, iters: int = 1,
                   opts: Optional[np.ndarray] = None):
        """Reference mttkrp_csf with ws/thds allocated once.  Returns (out, times[s])."""
        o = self.opts if opts is None else np.ascontiguousarray(opts, dtype=np.float64)
        R = [m for i, m in enumerate(mats) if i != mode and m is not None][0].shape[1]
        keep, mp = self._mats(mats, R)
        out = np.empty((self.dims[mode], R), dtype=np.float64)
        times = np.zeros(max(iters, 1), dtype=np.float64)
        self.lib.refdrv_mttkrp_csf(self.ptr, _dp(o), R, mp, mode, _dp(out), warm, iters, _dp(times))
        return out, times[:iters]

    def splatt_mttkrp(self, mats, mode: int) -> np.ndarray:
        R = [m for i, m in enumerate(mats) if i != mode and m is not None][0].shape[1]
        keep, mp = self._mats(mats, R)
        out = np.empty((self.dims[mode], R), dtype=np.float64)
        rc = self.lib.refdrv_splatt_mttkrp(mode, R, self.ptr, mp, _dp(out), _dp(self.opts))
        assert rc == A.SPLATT_SUCCESS
        return out

    def cpd_als(self, R: int, seed: int, opts: Optional[np.ndarray] = None):
        o = self.opts if opts is None else np.ascontiguousarray(opts, dtype=np.float64)
        facs = [np.empty((d, R), dtype=np.float64) for d in self.dims]
        fp = (C.POINTER(C.c_double) * self.nmodes)(*[_dp(f) for f in facs])
        lam = np.empty(R, dtype=np.float64)
        fit = self.lib.refdrv_cpd_als(self.ptr, R, _dp(o), seed, fp, _dp(lam))
        return float(fit), lam, facs

    def free(self):
        if self.ptr:
            self.lib.refdrv_csf_free(self.ptr, _dp(self.opts))
            self.ptr = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def mode_order(dims, which: int, mode: int = 0):
    lib = load()
    d = np.ascontiguousarray(dims, dtype=np.uint64)
    perm = np.zeros(8, dtype=np.uint64)
    lib.refdrv_mode_order(d.ctypes.data_as(C.POINTER(C.c_uint64)), len(d), which, mode,
                          perm.ctypes.data_as(C.POINTER(C.c_uint64)))
    return [int(x) for x in perm[:len(d)]]


def partition_weighted(weights, nparts: int):
    lib = load()
    w = np.ascontiguousarray(weights, dtype=np.uint64)
    bn = C.c_uint64()
    p = lib.refdrv_partition_weighted(w.ctypes.data_as(C.POINTER(C.c_uint64)), len(w), nparts,
                                      C.byref(bn))
    parts = np.ctypeslib.as_array(p, shape=(nparts + 1,)).copy()
    lib.refdrv_free(p)
    return parts, int(bn.value)


def abi_facts():
    lib = load()
    buf = (C.c_uint64 * 128)()
    n = lib.refdrv_abi(buf)
    return [int(buf[i]) for i in range(n)]
