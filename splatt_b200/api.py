"""Host-side mirror of the reference's MTTKRP / CPD interface over libsplatt_b200.so.

Names and argument meaning follow the reference's public API
(include/splatt/api_kernels.h, api_factorization.h, api_options.h):
`default_opts`, `csf_alloc`, `mttkrp`, `mttkrp_alloc_ws` / `mttkrp_csf` /
`mttkrp_free_ws`, `cpd_als`.  `Tensor` is the device-resident engine handle.
Everything computes in the CUDA library; numpy / torch only carry buffers.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

import numpy as np

from . import _abi as A


class SplattError(RuntimeError):
    def __init__(self, code: int, what: str):
        names = {A.SPLATT_ERROR_BADINPUT: "SPLATT_ERROR_BADINPUT",
                 A.SPLATT_ERROR_NOMEMORY: "SPLATT_ERROR_NOMEMORY"}
        super().__init__(f"{what}: {names.get(code, code)}")
        self.code = code


def _check(code: int, what: str) -> None:
    if code != A.SPLATT_SUCCESS:
        raise SplattError(code, what)


def default_opts() -> np.ndarray:
    """splatt_default_opts(): a fresh options array (numpy float64[NOPTIONS])."""
    lib = A.load()
    p = lib.splatt_default_opts()
    o = np.ctypeslib.as_array(p, shape=(A.OPTION_NOPTIONS,)).copy()
    lib.splatt_free_opts(p)
    return o


def _dptr(a: np.ndarray):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def _coo_args(dims, ind, vals):
    dims_a = np.ascontiguousarray(dims, dtype=np.uint64)
    nm = len(dims_a)
    inds = [np.ascontiguousarray(i, dtype=np.uint32) for i in ind]
    vals_a = np.ascontiguousarray(vals, dtype=np.float64)
    nnz = len(vals_a)
    for i in inds:
        if len(i) != nnz:
            raise ValueError("index arrays and values must have the same length")
    ip = (C.POINTER(C.c_uint32) * nm)(*[i.ctypes.data_as(C.POINTER(C.c_uint32)) for i in inds])
    return dims_a, nm, nnz, inds, vals_a, ip


class Csf:
    """Owner of a host `splatt_csf` array built by this library (splatt_b200_csf_alloc).

    Field-for-field what the reference's csf_alloc returns; `.ptr` can be handed to
    any function taking `splatt_csf const *` (ours or the reference's)."""

    def __init__(self, ptr, csf_alloc: int):
        self.ptr = ptr
        self.csf_alloc = csf_alloc

    @property
    def count(self) -> int:
        if self.csf_alloc == A.CSF_ONEMODE:
            return 1
        if self.csf_alloc == A.CSF_TWOMODE:
            return 2
        return int(self.ptr[0].nmodes)

    def arrays(self, c: int = 0, tile: int = 0) -> dict:
        """numpy copies of CSF c's arrays (for tests / inspection)."""
        t = self.ptr[c]
        n = int(t.nmodes)
        pt = t.pt[tile]
        out = {"nnz": int(t.nnz), "nmodes": n, "dims": [int(t.dims[m]) for m in range(n)],
               "dim_perm": [int(t.dim_perm[m]) for m in range(n)],
               "dim_iperm": [int(t.dim_iperm[m]) for m in range(n)],
               "ntiles": int(t.ntiles), "nfibs": [int(pt.nfibs[m]) for m in range(n)],
               "fptr": [], "fids": []}
        for l in range(n):
            nf = int(pt.nfibs[l])
            out["fids"].append(None if not pt.fids[l] else
                               np.ctypeslib.as_array(pt.fids[l], shape=(nf,)).copy())
            if l < n - 1:
                out["fptr"].append(np.ctypeslib.as_array(pt.fptr[l], shape=(nf + 1,)).copy())
        out["vals"] = np.ctypeslib.as_array(pt.vals, shape=(int(t.nnz),)).copy()
        return out

    def free(self) -> None:
        if self.ptr is not None:
            A.load().splatt_b200_csf_free(self.ptr, self.csf_alloc)
            self.ptr = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def csf_alloc(dims, ind, vals, opts: Optional[np.ndarray] = None) -> Csf:
    """Build the CSF(s) the reference's csf_alloc(tt, opts) would build (untiled)."""
    lib = A.load()
    o = default_opts() if opts is None else opts
    alloc = int(o[A.OPTION_CSF_ALLOC])
    dims_a, nm, nnz, inds, vals_a, ip = _coo_args(dims, ind, vals)
    out = C.POINTER(A.SplattCsf)()
    rc = lib.splatt_b200_csf_alloc(nm, dims_a.ctypes.data_as(A.idx_p), nnz, ip, _dptr(vals_a), 0,
                                   alloc, C.byref(out))
    _check(rc, "splatt_b200_csf_alloc")
    return Csf(out, alloc)


def _mat_ptrs(mats: Sequence[Optional[np.ndarray]]):
    keep = [None if m is None else np.ascontiguousarray(m, dtype=np.float64) for m in mats]
    arr = (A.val_p * len(keep))(*[A.val_p() if k is None else _dptr(k) for k in keep])
    return keep, arr


def mttkrp(mode: int, ncolumns: int, csf_ptr, matrices: Sequence[Optional[np.ndarray]],
           opts: np.ndarray) -> np.ndarray:
    """splatt_mttkrp(): host factor matrices in, host result out."""
    lib = A.load()
    csf0 = csf_ptr[0]
    out = np.empty((int(csf0.dims[mode]), ncolumns), dtype=np.float64)
    keep, arr = _mat_ptrs(matrices)
    o = np.ascontiguousarray(opts, dtype=np.float64)
    rc = lib.splatt_mttkrp(mode, ncolumns, csf_ptr, arr, _dptr(out), _dptr(o))
    _check(rc, "splatt_mttkrp")
    return out


class MttkrpWorkspace:
    """splatt_mttkrp_alloc_ws / splatt_mttkrp_csf / splatt_mttkrp_free_ws."""

    def __init__(self, csf_ptr, ncolumns: int, opts: np.ndarray):
        self.lib = A.load()
        self.csf_ptr = csf_ptr
        self.ncolumns = ncolumns
        self.opts = np.ascontiguousarray(opts, dtype=np.float64)
        self.ws = self.lib.splatt_mttkrp_alloc_ws(csf_ptr, ncolumns, _dptr(self.opts))
        if not self.ws:
            raise SplattError(A.SPLATT_ERROR_NOMEMORY, "splatt_mttkrp_alloc_ws")
        self.nmodes = int(csf_ptr[0].nmodes)
        self.dims = [int(csf_ptr[0].dims[m]) for m in range(self.nmodes)]

    def mttkrp_csf(self, mats: Sequence[np.ndarray], mode: int, out: np.ndarray) -> np.ndarray:
        """mats[m]: C-contiguous float64 dims[m] x R (mats[mode] unused); out dims[mode] x R."""
        store = (A.Matrix * (A.MAX_NMODES + 1))()
        ptrs = (C.POINTER(A.Matrix) * (A.MAX_NMODES + 1))()
        for m in range(self.nmodes):
            a = mats[m]
            store[m].I = self.dims[m]
            store[m].J = self.ncolumns
            store[m].rowmajor = 1
            store[m].vals = _dptr(a) if a is not None else A.val_p()
            ptrs[m] = C.pointer(store[m])
        store[A.MAX_NMODES].I = out.shape[0]
        store[A.MAX_NMODES].J = self.ncolumns
        store[A.MAX_NMODES].rowmajor = 1
        store[A.MAX_NMODES].vals = _dptr(out)
        ptrs[A.MAX_NMODES] = C.pointer(store[A.MAX_NMODES])
        self.lib.splatt_mttkrp_csf(self.csf_ptr, ptrs, mode, None, self.ws, _dptr(self.opts))
        return out

    def free(self):
        if self.ws:
            self.lib.splatt_mttkrp_free_ws(self.ws)
            self.ws = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def cpd_als(csf_ptr, nfactors: int, opts: np.ndarray, seed: Optional[int] = None):
    """splatt_cpd_als(): returns (fit, lambda, [factor matrices])."""
    lib = A.load()
    if seed is not None:
        C.CDLL(None).srand(C.c_uint(seed))   # the CLI seeds libc rand() (cmd_cpd.c:167)
    k = A.SplattKruskal()
    o = np.ascontiguousarray(opts, dtype=np.float64)
    rc = lib.splatt_cpd_als(csf_ptr, nfactors, _dptr(o), C.byref(k))
    _check(rc, "splatt_cpd_als")
    n = int(k.nmodes)
    lam = np.ctypeslib.as_array(k.lambda_, shape=(nfactors,)).copy()
    facs = [np.ctypeslib.as_array(k.factors[m], shape=(int(k.dims[m]), nfactors)).copy()
            for m in range(n)]
    fit = float(k.fit)
    lib.splatt_free_kruskal(C.byref(k))
    return fit, lam, facs


class Tensor:
    """Device-resident sparse tensor (splatt_b200_tensor): per-mode fiber streams in HBM."""

    def __init__(self, handle, lib):
        self.h = handle
        self.lib = lib
        nm = C.c_int()
        dims = (A.idx_t * A.MAX_NMODES)()
        tot = A.idx_t()
        loc = A.idx_t()
        byt = A.idx_t()
        _check(lib.splatt_b200_tensor_info(self.h, C.byref(nm), dims, C.byref(tot), C.byref(loc),
                                           C.byref(byt)), "splatt_b200_tensor_info")
        self.nmodes = nm.value
        self.dims = [int(dims[m]) for m in range(self.nmodes)]
        self.nnz = int(tot.value)
        self.nnz_local = int(loc.value)
        self.device_bytes = int(byt.value)

    @staticmethod
    def _bopts(layout, device, shard_rank, shard_count, verbosity, ncolumns_hint=0, ktile=0):
        bo = A.BuildOpts()
        bo.ncolumns_hint = ncolumns_hint
        bo.ktile = ktile
        bo.layout = layout
        bo.device = device
        bo.shard_rank = shard_rank
        bo.shard_count = shard_count
        bo.verbosity = verbosity
        return bo

    @classmethod
    def from_coo(cls, dims, ind, vals, *, csf_alloc: int = A.CSF_TWOMODE,
                 layout: int = A.LAYOUT_ALLROOT, device: int = -1, shard_rank: int = 0,
                 shard_count: int = 1, verbosity: int = 0, ncolumns_hint: int = 0,
                 ktile: int = 0) -> "Tensor":
        """ind/vals: numpy (host) arrays, or torch CUDA tensors (int32/uint32 + float64 or
        float32; float32 values are widened exactly to float64).
        ncolumns_hint: the rank the tensor will be multiplied at (enables leaf tiling)."""
        lib = A.load()
        on_device = 0
        try:
            import torch
            if isinstance(vals, torch.Tensor) and vals.is_cuda:
                on_device = 1
        except ImportError:
            pass
        bo = cls._bopts(layout, device, shard_rank, shard_count, verbosity, ncolumns_hint, ktile)
        out = C.c_void_p()
        if on_device:
            dims_a = np.ascontiguousarray(dims, dtype=np.uint64)
            nm = len(dims_a)
            nnz = int(vals.numel())
            keep = [i.contiguous() for i in ind]
            if vals.dtype == torch.float32:
                vals = vals.to(torch.float64)            # exact
            elif vals.dtype != torch.float64:
                raise ValueError(f"device values must be float64 or float32, not {vals.dtype}")
            v = vals.contiguous()
            ip = (C.POINTER(C.c_uint32) * nm)(
                *[C.cast(C.c_void_p(i.data_ptr()), C.POINTER(C.c_uint32)) for i in keep])
            vp = C.cast(C.c_void_p(v.data_ptr()), A.val_p)
            rc = lib.splatt_b200_tensor_from_coo(nm, dims_a.ctypes.data_as(A.idx_p), nnz, ip, vp, 1,
                                                 csf_alloc, C.byref(bo), C.byref(out))
        else:
            dims_a, nm, nnz, inds, vals_a, ip = _coo_args(dims, ind, vals)
            rc = lib.splatt_b200_tensor_from_coo(nm, dims_a.ctypes.data_as(A.idx_p), nnz, ip,
                                                 _dptr(vals_a), 0, csf_alloc, C.byref(bo),
                                                 C.byref(out))
        _check(rc, "splatt_b200_tensor_from_coo")
        return cls(out, lib)

    @classmethod
    def from_csf(cls, csf_ptr, csf_alloc: int, *, layout: int = A.LAYOUT_ALLROOT, device: int = -1,
                 shard_rank: int = 0, shard_count: int = 1, verbosity: int = 0,
                 ncolumns_hint: int = 0, ktile: int = 0) -> "Tensor":
        lib = A.load()
        bo = cls._bopts(layout, device, shard_rank, shard_count, verbosity, ncolumns_hint, ktile)
        out = C.c_void_p()
        rc = lib.splatt_b200_tensor_from_csf(csf_ptr, csf_alloc, C.byref(bo), C.byref(out))
        _check(rc, "splatt_b200_tensor_from_csf")
        return cls(out, lib)

    def mode_info(self, mode: int, ncolumns: int) -> dict:
        kind = C.c_int()
        perm = (C.c_int * A.MAX_NMODES)()
        nf = (A.idx_t * A.MAX_NMODES)()
        ab = A.idx_t()
        _check(self.lib.splatt_b200_mode_info(self.h, mode, ncolumns, C.byref(kind), perm, nf,
                                              C.byref(ab)), "splatt_b200_mode_info")
        return {"kind": A.KIND_NAMES[kind.value],
                "level_perm": [perm[l] for l in range(self.nmodes)],
                "nfibs": [int(nf[l]) for l in range(self.nmodes)],
                "alg_bytes": int(ab.value)}

    def mttkrp(self, mode: int, mats, out, ncolumns: Optional[int] = None, stream=None):
        """Enqueue one MTTKRP.  mats[m], out: torch CUDA tensors of one dtype, row-major, same
        leading dimension (>= ncolumns).  float64: the leading dimension is even.  float32
        (splatt_b200_mttkrp_f32: fp32 arithmetic): it is a multiple of 4.  No host sync."""
        import torch
        if out.dtype == torch.float64:
            ptr_t, sym, align = A.val_p, "splatt_b200_mttkrp", "even"
        elif out.dtype == torch.float32:
            ptr_t, sym, align = A.f32_p, "splatt_b200_mttkrp_f32", "a multiple of 4"
        else:
            raise ValueError(f"MTTKRP output must be float64 or float32, not {out.dtype}")
        ldm = out.stride(0)
        if out.dtype == torch.float32 and ldm % 4:
            raise ValueError(f"float32 MTTKRP needs a leading dimension (stride(0)) that is a "
                             f"multiple of 4, got {ldm}")
        R = out.shape[1] if ncolumns is None else ncolumns
        ptrs = (ptr_t * self.nmodes)()
        for m in range(self.nmodes):
            if m == mode or mats[m] is None:
                ptrs[m] = ptr_t()
                continue
            t = mats[m]
            if t.dtype != out.dtype:
                raise ValueError(f"factor matrix {m} is {t.dtype} but the output is {out.dtype}")
            if not (t.is_cuda and t.stride(1) == 1 and t.stride(0) == ldm):
                raise ValueError(f"factor matrices must be CUDA {out.dtype} row-major with the "
                                 f"output's leading dimension ({align})")
            ptrs[m] = C.cast(C.c_void_p(t.data_ptr()), ptr_t)
        s = torch.cuda.current_stream().cuda_stream if stream is None else stream
        rc = getattr(self.lib, sym)(self.h, mode, R, ldm, ptrs,
                                    C.cast(C.c_void_p(out.data_ptr()), ptr_t), C.c_void_p(s))
        _check(rc, sym)
        return out

    def cpd_als(self, rank: int, factors=None, *, dtype=None, niters: int = 50, tol: float = 1e-5,
                seed: int = 0, verbosity: int = 0, stream=None):
        """CPD-ALS of this (whole) tensor on its device (splatt_b200_cpd_als_device, or _f32 for
        float32: fp32 factors and MTTKRP, fp64 Grams, solves, lambda and fit).  The tensor must
        live on the current CUDA device, as for Tensor.mttkrp: the start buffers and the default
        stream are taken from it.

        factors: list of CUDA tensors (dims[m] x rank) of one dtype, the start; copied into
        padded buffers, never written.  None: uniform on [-3, 3) (the reference's rand_val range)
        from a torch.Generator seeded with `seed`, in `dtype` (default float64).  Stops after
        `niters` iterations or when the fit moves by less than `tol`.  In float32 the fit is
        formed from the fp32 MTTKRP result and, close to 1, resolved only to about 1e-4 (see
        splatt_b200_cpd_als_device_f32 in include/splatt_b200.h): a `tol` below that may not stop
        the run before `niters` there.
        Returns (fit, lambda (numpy float64[rank]), factors (2-normalised, CUDA views
        dims[m] x rank), iterations)."""
        import torch
        if factors is not None:
            dt = factors[0].dtype
            if dtype is not None and dtype != dt:
                raise ValueError(f"factor matrix 0 is {dt} but dtype is {dtype}")
            for m, f in enumerate(factors):
                if f.dtype != dt:
                    raise ValueError(f"factor matrix {m} is {f.dtype} but factor matrix 0 is {dt}")
            if len(factors) != self.nmodes:
                raise ValueError(f"{len(factors)} factor matrices for a {self.nmodes}-mode tensor")
        dev = torch.device("cuda", torch.cuda.current_device())
        if factors is not None:
            for m, f in enumerate(factors):
                if f.device != dev or tuple(f.shape) != (self.dims[m], rank):
                    raise ValueError(f"factor matrix {m} must be a tensor of shape "
                                     f"({self.dims[m]}, {rank}) on the current device {dev}")
        else:
            dt = torch.float64 if dtype is None else dtype
        if dt == torch.float64:
            ptr_t, sym, ldm = A.val_p, "splatt_b200_cpd_als_device", rank + (rank & 1)
        elif dt == torch.float32:
            ptr_t, sym, ldm = A.f32_p, "splatt_b200_cpd_als_device_f32", (rank + 3) & ~3
        else:
            raise ValueError(f"CPD factors must be float64 or float32, not {dt}")
        bufs = [torch.zeros((d, ldm), dtype=dt, device=dev) for d in self.dims]
        if factors is None:
            g = torch.Generator(device=dev).manual_seed(seed)
            for b in bufs:
                b[:, :rank].uniform_(-3.0, 3.0, generator=g)
        else:
            for b, f in zip(bufs, factors):
                b[:, :rank].copy_(f)
        o = default_opts()
        o[A.OPTION_NITER] = niters
        o[A.OPTION_TOLERANCE] = tol
        o[A.OPTION_VERBOSITY] = verbosity
        if stream is None:
            s = torch.cuda.current_stream(dev).cuda_stream
        else:
            torch.cuda.current_stream(dev).synchronize()    # the buffers were filled there
            s = stream
        ptrs = (ptr_t * self.nmodes)(*[C.cast(C.c_void_p(b.data_ptr()), ptr_t) for b in bufs])
        lam = np.zeros(rank)
        fit = C.c_double()
        its = C.c_int()
        rc = getattr(self.lib, sym)(self.h, rank, ldm, _dptr(o), ptrs, _dptr(lam), C.byref(fit),
                                    C.byref(its), C.c_void_p(s))
        _check(rc, sym)
        return fit.value, lam, [b[:, :rank] for b in bufs], its.value

    def sse(self, factors, lam=None, stream=None) -> float:
        """Sum over this tensor's nonzeros of (v - sum_r lam_r prod_m factors[m][i_m, r])^2
        (splatt_b200_tensor_sse; lam None = all ones).  factors: float64 CUDA tensors
        (dims[m] x rank) on the current device; rank <= 64.  Synchronises the stream once."""
        import torch
        dev = torch.device("cuda", torch.cuda.current_device())
        if len(factors) != self.nmodes:
            raise ValueError(f"{len(factors)} factor matrices for a {self.nmodes}-mode tensor")
        rank = factors[0].shape[1] if factors[0].dim() == 2 else -1
        for m, f in enumerate(factors):
            if f.dtype != torch.float64:
                raise ValueError(f"factor matrix {m} is {f.dtype}; Tensor.sse is float64 only")
            if f.device != dev or tuple(f.shape) != (self.dims[m], rank):
                raise ValueError(f"factor matrix {m} must be a tensor of shape "
                                 f"({self.dims[m]}, {rank}) on the current device {dev}")
        ldm = rank + (rank & 1)
        bufs = [torch.zeros((d, ldm), dtype=torch.float64, device=dev) for d in self.dims]
        for b, f in zip(bufs, factors):
            b[:, :rank].copy_(f)
        lam_a = None if lam is None else np.ascontiguousarray(lam, dtype=np.float64)
        if lam_a is not None and lam_a.shape != (rank,):
            raise ValueError(f"lam must have {rank} entries")
        if stream is None:
            s = torch.cuda.current_stream(dev).cuda_stream
        else:
            torch.cuda.current_stream(dev).synchronize()    # the buffers were filled there
            s = stream
        ptrs = (A.val_p * self.nmodes)(*[C.cast(C.c_void_p(b.data_ptr()), A.val_p) for b in bufs])
        out = C.c_double()
        rc = self.lib.splatt_b200_tensor_sse(self.h, rank, ldm, ptrs,
                                             A.val_p() if lam_a is None else _dptr(lam_a),
                                             C.byref(out), C.c_void_p(s))
        _check(rc, "splatt_b200_tensor_sse")
        return out.value

    def complete(self, rank: int, factors=None, *, validate: Optional["Tensor"] = None, reg: float,
                 niters: int = 50, tol: float = 1e-4, seed: int = 0, verbosity: int = 0,
                 stream=None):
        """Tensor completion by row-wise ALS (splatt_b200_tc_als_device): fits
        sum_r prod_m U_m[i_m, r] to this tensor's stored entries only, with the penalty
        reg * sum_m ||U_m||_F^2 (reg > 0).  Needs a whole tensor built with the ALLROOT layout
        on the current CUDA device, and 1 <= rank <= 64.  float64 only.

        factors: list of float64 CUDA tensors (dims[m] x rank), the start; copied into padded
        buffers, never written.  None: uniform on [0, 1) from a torch.Generator on the current
        device seeded with `seed`, drawn mode by mode.  validate: a Tensor with the same shape,
        scored after every iteration.  Stops after `niters` iterations or, from the second on,
        when the objective moved by less than `tol` relative.
        Returns (history: numpy float64 [iterations x 3] of (objective, training RMSE,
        validation RMSE or NaN), factors (CUDA views dims[m] x rank), iterations)."""
        import torch
        dev = torch.device("cuda", torch.cuda.current_device())
        if factors is not None:
            if len(factors) != self.nmodes:
                raise ValueError(f"{len(factors)} factor matrices for a {self.nmodes}-mode tensor")
            for m, f in enumerate(factors):
                if f.dtype != torch.float64:
                    raise ValueError(f"factor matrix {m} is {f.dtype}; completion is float64 only")
                if f.device != dev or tuple(f.shape) != (self.dims[m], rank):
                    raise ValueError(f"factor matrix {m} must be a tensor of shape "
                                     f"({self.dims[m]}, {rank}) on the current device {dev}")
        if validate is not None and not isinstance(validate, Tensor):
            raise ValueError("validate must be a Tensor")
        ldm = rank + (rank & 1)
        bufs = [torch.zeros((d, ldm), dtype=torch.float64, device=dev) for d in self.dims]
        if factors is None:
            g = torch.Generator(device=dev).manual_seed(seed)
            for b in bufs:
                b[:, :rank].uniform_(0.0, 1.0, generator=g)
        else:
            for b, f in zip(bufs, factors):
                b[:, :rank].copy_(f)
        o = default_opts()
        o[A.OPTION_NITER] = niters
        o[A.OPTION_TOLERANCE] = tol
        o[A.OPTION_VERBOSITY] = verbosity
        o[A.OPTION_REGULARIZE] = reg
        if stream is None:
            s = torch.cuda.current_stream(dev).cuda_stream
        else:
            torch.cuda.current_stream(dev).synchronize()    # the buffers were filled there
            s = stream
        ptrs = (A.val_p * self.nmodes)(*[C.cast(C.c_void_p(b.data_ptr()), A.val_p) for b in bufs])
        hist = np.full((max(int(niters), 0), 3), np.nan)
        its = C.c_int()
        rc = self.lib.splatt_b200_tc_als_device(self.h, None if validate is None else validate.h,
                                                rank, ldm, _dptr(o), ptrs, _dptr(hist),
                                                C.byref(its), C.c_void_p(s))
        _check(rc, "splatt_b200_tc_als_device")
        return hist[:its.value].copy(), [b[:, :rank] for b in bufs], its.value

    def shard(self, rank: int, count: int, device: int = -1) -> "Tensor":
        """Cut shard `rank` of `count` out of this (whole) tensor onto `device`
        (splatt_b200_tensor_shard): the equal-nnz chunk range of every stream, copied
        device to device instead of being rebuilt."""
        out = C.c_void_p()
        _check(self.lib.splatt_b200_tensor_shard(self.h, rank, count, device, C.byref(out)),
               "splatt_b200_tensor_shard")
        return Tensor(out, self.lib)

    def free(self):
        if self.h:
            self.lib.splatt_b200_tensor_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def launch_count() -> int:
    return int(A.load().splatt_b200_launch_count())


def build_count() -> int:
    """Fiber streams built (sort + scans) in this process so far."""
    return int(A.load().splatt_b200_build_count())


def cache_clear() -> None:
    """Drop the device mirrors kept by the bare splatt_mttkrp entry point."""
    A.load().splatt_b200_cache_clear()


class MultiGpu:
    """Single-process multi-GPU engine (splatt_b200_multi): one host process, several
    devices, the exchange fused into the MTTKRP kernel over NVLink multicast (or the
    peer-memory reduce where there is no multicast)."""

    def __init__(self, csf_ptr, csf_alloc: int, ncolumns: int, devices: Sequence[int],
                 verbosity: int = 0):
        self.lib = A.load()
        self.csf_ptr = csf_ptr
        self.ncolumns = ncolumns
        devs = (C.c_int * len(devices))(*devices)
        self.h = C.c_void_p()
        _check(self.lib.splatt_b200_multi_create(csf_ptr, csf_alloc, ncolumns, devs, len(devices),
                                                 verbosity, C.byref(self.h)),
               "splatt_b200_multi_create")
        self.nmodes = int(csf_ptr[0].nmodes)
        self.dims = [int(csf_ptr[0].dims[m]) for m in range(self.nmodes)]
        nd, mc = C.c_int(), C.c_int()
        nl = (A.idx_t * 16)()
        db = (A.idx_t * 16)()
        _check(self.lib.splatt_b200_multi_info(self.h, C.byref(nd), C.byref(mc), nl, db),
               "splatt_b200_multi_info")
        self.ndevices = nd.value
        self.multicast = bool(mc.value)
        self.nnz_local = [int(nl[i]) for i in range(self.ndevices)]
        self.device_bytes = [int(db[i]) for i in range(self.ndevices)]

    def mttkrp_host(self, mode: int, mats: Sequence[Optional[np.ndarray]],
                    out: Optional[np.ndarray] = None) -> np.ndarray:
        if out is None:
            out = np.empty((self.dims[mode], self.ncolumns), dtype=np.float64)
        keep, arr = _mat_ptrs([None if m == mode else mats[m] for m in range(self.nmodes)])
        _check(self.lib.splatt_b200_multi_mttkrp_host(self.h, mode, arr, _dptr(out)),
               "splatt_b200_multi_mttkrp_host")
        return out

    def cpd_als(self, opts: np.ndarray, seed: Optional[int] = None):
        if seed is not None:
            C.CDLL(None).srand(C.c_uint(seed))
        k = A.SplattKruskal()
        o = np.ascontiguousarray(opts, dtype=np.float64)
        _check(self.lib.splatt_b200_multi_cpd_als(self.h, self.csf_ptr, _dptr(o), C.byref(k)),
               "splatt_b200_multi_cpd_als")
        n = int(k.nmodes)
        R = self.ncolumns
        lam = np.ctypeslib.as_array(k.lambda_, shape=(R,)).copy()
        facs = [np.ctypeslib.as_array(k.factors[m], shape=(int(k.dims[m]), R)).copy()
                for m in range(n)]
        fit = float(k.fit)
        self.lib.splatt_free_kruskal(C.byref(k))
        return fit, lam, facs

    def free(self):
        if self.h:
            self.lib.splatt_b200_multi_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass
