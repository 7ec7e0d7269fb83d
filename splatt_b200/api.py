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


def _launch_args(bufs, stream, ptr_t=A.val_p):
    """(stream handle, ctypes pointer array) for an entry point that reads the device buffers
    `bufs`, filled on the current stream: an explicit `stream` first waits for them."""
    import torch
    cur = torch.cuda.current_stream(bufs[0].device)
    if stream is None:
        s = cur.cuda_stream
    else:
        cur.synchronize()    # the buffers were filled there
        s = stream
    return s, (ptr_t * len(bufs))(*[C.cast(C.c_void_p(b.data_ptr()), ptr_t) for b in bufs])


def _u32_ptrs(bufs):
    """ctypes array of uint32 pointers to int32/uint32 CUDA tensors (indices below 2^31)."""
    for b in bufs:
        if b.element_size() != 4 or not b.is_contiguous():
            raise ValueError("index buffers must be contiguous 32-bit integer tensors")
    return (C.POINTER(C.c_uint32) * len(bufs))(*[C.cast(C.c_void_p(b.data_ptr()), C.POINTER(C.c_uint32))
                                                  for b in bufs])


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
        fit, lam, facs, its, _ = self._cpd_device(False, rank, factors, dtype, niters, tol, seed,
                                                  verbosity, stream)
        return fit, lam, facs, its

    def cpd_nonneg(self, rank: int, factors=None, *, dtype=None, niters: int = 50,
                   tol: float = 1e-5, seed: int = 0, verbosity: int = 0, stream=None):
        """Nonnegative CPD by HALS (splatt_b200_cpd_nonneg_device, or _f32 for float32: fp32
        factors and MTTKRP, fp64 Hadamard Grams, sweep, lambda and fit) of this (whole) tensor on
        its device: nonnegative factors with unit 2-norm columns and lambda >= 0 that minimise
        1/2 ||X - K||^2, unstored entries read as zeros.  Tensor values may have any sign.  One
        Gauss-Seidel sweep over the columns per mode and iteration, with every entry floored at
        1e-16 (see include/splatt_b200.h).  The tensor must live on the current CUDA device.

        factors: list of CUDA tensors (dims[m] x rank) of one dtype, the start (finite, >= 0, no
        zero column); copied into padded buffers, never written.  None: uniform on [0, 1) from a
        torch.Generator seeded with `seed`, in `dtype` (default float64).  Stops as cpd_als does.
        Returns (fit, lambda (numpy float64[rank]), factors (CUDA views dims[m] x rank),
        iterations, history (numpy float64[iterations]: the fit of every iteration))."""
        return self._cpd_device(True, rank, factors, dtype, niters, tol, seed, verbosity, stream)

    def _check_factors(self, factors, cols, dtype, what):
        """Raise ValueError unless factors (None: no start given) holds one tensor of shape
        (dims[m], cols[m]) per mode on the current device, each of `dtype` (`what`: the entry
        point named in the error; None: the caller checked the dtypes)."""
        import torch
        if factors is None:
            return
        dev = torch.device("cuda", torch.cuda.current_device())
        if len(factors) != self.nmodes:
            raise ValueError(f"{len(factors)} factor matrices for a {self.nmodes}-mode tensor")
        for m, f in enumerate(factors):
            if what is not None and f.dtype != dtype:
                raise ValueError(f"factor matrix {m} is {f.dtype}; {what} is float64 only")
            if f.device != dev or tuple(f.shape) != (self.dims[m], cols[m]):
                raise ValueError(f"factor matrix {m} must be a tensor of shape "
                                 f"({self.dims[m]}, {cols[m]}) on the current device {dev}")

    def _start_factors(self, factors, cols, ldm, dtype, seed=0, draw=None):
        """One zero-padded (dims[m], ldm) `dtype` buffer per mode on the current device, its
        first cols[m] columns copied from factors[m] (checked by _check_factors) or, when factors
        is None, drawn by draw(view, generator) mode by mode from a torch.Generator seeded with
        `seed`."""
        import torch
        dev = torch.device("cuda", torch.cuda.current_device())
        bufs = [torch.zeros((d, ldm), dtype=dtype, device=dev) for d in self.dims]
        if factors is None:
            g = torch.Generator(device=dev).manual_seed(seed)
            for b, r in zip(bufs, cols):
                draw(b[:, :r], g)
        else:
            for b, f, r in zip(bufs, factors, cols):
                b[:, :r].copy_(f)
        return bufs

    def _cpd_device(self, nonneg, rank, factors, dtype, niters, tol, seed, verbosity, stream):
        """cpd_als (nonneg False) or cpd_nonneg: (fit, lambda, factors, iterations, history)."""
        import torch
        if factors is not None:
            dt = factors[0].dtype
            if dtype is not None and dtype != dt:
                raise ValueError(f"factor matrix 0 is {dt} but dtype is {dtype}")
            for m, f in enumerate(factors):
                if f.dtype != dt:
                    raise ValueError(f"factor matrix {m} is {f.dtype} but factor matrix 0 is {dt}")
        else:
            dt = torch.float64 if dtype is None else dtype
        self._check_factors(factors, [rank] * self.nmodes, dt, None)
        if dt == torch.float64:
            ptr_t, sym, ldm = A.val_p, "splatt_b200_cpd_als_device", rank + (rank & 1)
        elif dt == torch.float32:
            ptr_t, sym, ldm = A.f32_p, "splatt_b200_cpd_als_device_f32", (rank + 3) & ~3
        else:
            raise ValueError(f"CPD factors must be float64 or float32, not {dt}")
        lo, hi = (0.0, 1.0) if nonneg else (-3.0, 3.0)
        bufs = self._start_factors(factors, [rank] * self.nmodes, ldm, dt, seed,
                                   lambda v, g: v.uniform_(lo, hi, generator=g))
        o = default_opts()
        o[A.OPTION_NITER] = niters
        o[A.OPTION_TOLERANCE] = tol
        o[A.OPTION_VERBOSITY] = verbosity
        s, ptrs = _launch_args(bufs, stream, ptr_t)
        lam = np.zeros(rank)
        fit = C.c_double()
        its = C.c_int()
        if nonneg:
            sym = sym.replace("_als_", "_nonneg_")
            hist = np.full(max(int(niters), 0), np.nan)
            rc = getattr(self.lib, sym)(self.h, rank, ldm, _dptr(o), ptrs, _dptr(lam), C.byref(fit),
                                        C.byref(its), _dptr(hist), C.c_void_p(s))
        else:
            hist = None
            rc = getattr(self.lib, sym)(self.h, rank, ldm, _dptr(o), ptrs, _dptr(lam), C.byref(fit),
                                        C.byref(its), C.c_void_p(s))
        _check(rc, sym)
        return (fit.value, lam, [b[:, :rank] for b in bufs], its.value,
                None if hist is None else hist[:its.value].copy())

    def sse(self, factors, lam=None, stream=None) -> float:
        """Sum over this tensor's nonzeros of (v - sum_r lam_r prod_m factors[m][i_m, r])^2
        (splatt_b200_tensor_sse; lam None = all ones).  factors: float64 CUDA tensors
        (dims[m] x rank) on the current device; rank <= 64.  Synchronises the stream once."""
        import torch
        rank = factors[0].shape[1] if len(factors) == self.nmodes and factors[0].dim() == 2 else -1
        self._check_factors(factors, [rank] * self.nmodes, torch.float64, "Tensor.sse")
        ldm = rank + (rank & 1)
        bufs = self._start_factors(factors, [rank] * self.nmodes, ldm, torch.float64)
        lam_a = None if lam is None else np.ascontiguousarray(lam, dtype=np.float64)
        if lam_a is not None and lam_a.shape != (rank,):
            raise ValueError(f"lam must have {rank} entries")
        s, ptrs = _launch_args(bufs, stream)
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
        self._check_factors(factors, [rank] * self.nmodes, torch.float64, "completion")
        if validate is not None and not isinstance(validate, Tensor):
            raise ValueError("validate must be a Tensor")
        ldm = rank + (rank & 1)
        bufs = self._start_factors(factors, [rank] * self.nmodes, ldm, torch.float64, seed,
                                   lambda v, g: v.uniform_(0.0, 1.0, generator=g))
        o = default_opts()
        o[A.OPTION_NITER] = niters
        o[A.OPTION_TOLERANCE] = tol
        o[A.OPTION_VERBOSITY] = verbosity
        o[A.OPTION_REGULARIZE] = reg
        s, ptrs = _launch_args(bufs, stream)
        hist = np.full((max(int(niters), 0), 3), np.nan)
        its = C.c_int()
        rc = self.lib.splatt_b200_tc_als_device(self.h, None if validate is None else validate.h,
                                                rank, ldm, _dptr(o), ptrs, _dptr(hist),
                                                C.byref(its), C.c_void_p(s))
        _check(rc, "splatt_b200_tc_als_device")
        return hist[:its.value].copy(), [b[:, :rank] for b in bufs], its.value

    def complete_lbfgs(self, rank: int, factors=None, *, validate: Optional["Tensor"] = None,
                       reg: float, memory: int = 5, niters: int = 100, tol: float = 1e-6,
                       seed: int = 0, verbosity: int = 0, stream=None):
        """Tensor completion by whole-model L-BFGS with an exact line search
        (splatt_b200_tc_lbfgs_device): the model and objective of `complete`, minimised over all
        factors at once along L-BFGS directions from the last `memory` steps (0: steepest
        descent), each step the exact minimiser of the objective along its direction.  reg >= 0.
        Needs what `complete` needs; factors, seed and validate as in `complete`.  Stops after
        `niters` iterations, when the gradient is zero or no decrease is found, or, from the
        second iteration on, when the objective decreased by less than `tol` relative.
        Returns (history: numpy float64 [iterations x 5] of (objective, training RMSE,
        validation RMSE or NaN, step length, gradient norm), factors (CUDA views
        dims[m] x rank), iterations)."""
        import torch
        self._check_factors(factors, [rank] * self.nmodes, torch.float64, "completion")
        if validate is not None and not isinstance(validate, Tensor):
            raise ValueError("validate must be a Tensor")
        ldm = rank + (rank & 1)
        bufs = self._start_factors(factors, [rank] * self.nmodes, ldm, torch.float64, seed,
                                   lambda v, g: v.uniform_(0.0, 1.0, generator=g))
        o = default_opts()
        o[A.OPTION_NITER] = niters
        o[A.OPTION_TOLERANCE] = tol
        o[A.OPTION_VERBOSITY] = verbosity
        o[A.OPTION_REGULARIZE] = reg
        lo = A.TcLbfgsOpts(memory)
        s, ptrs = _launch_args(bufs, stream)
        hist = np.full((max(int(niters), 0), 5), np.nan)
        its = C.c_int()
        rc = self.lib.splatt_b200_tc_lbfgs_device(self.h, None if validate is None else validate.h,
                                                  rank, ldm, _dptr(o), C.byref(lo), ptrs,
                                                  _dptr(hist), C.byref(its), C.c_void_p(s))
        _check(rc, "splatt_b200_tc_lbfgs_device")
        return hist[:its.value].copy(), [b[:, :rank] for b in bufs], its.value

    def cp_apr(self, rank: int, factors=None, *, niters: int = 100, tol: float = 1e-4,
               max_inner: int = 10, kappa: float = 0.01, kappa_tol: float = 1e-10,
               eps: float = 1e-10, seed: int = 0, verbosity: int = 0, stream=None):
        """Poisson CP decomposition by CP-APR (splatt_b200_cp_apr_device) of this count tensor:
        a nonnegative model lam_r a_r^(1) o ... o a_r^(N) with column-stochastic factors that
        maximises the Poisson log-likelihood, unstored coordinates being zero counts.  Needs a
        whole tensor built with the ALLROOT layout on the current CUDA device, values finite and
        >= 0, and 1 <= rank <= 64.  float64 only.

        factors: list of float64 CUDA tensors (dims[m] x rank), the start (nonnegative, every
        column with a positive sum); copied into padded buffers, never written.  None: uniform on
        [0, 1) from a torch.Generator on the current device seeded with `seed`, drawn mode by
        mode.  Each mode runs at most `max_inner` multiplicative updates and stops early when its
        KKT violation is below `tol`; the run stops after `niters` outer iterations or after one
        in which every mode stopped at its first update.  kappa / kappa_tol: the shift that frees
        entries pinned at zero; eps: the floor of the model value in a division or a log.
        Returns (lam (numpy float64[rank]), factors (CUDA views dims[m] x rank), history (numpy
        float64 [iterations x 3] of (log-likelihood, largest final KKT violation, inner
        iterations summed over the modes)), iterations)."""
        import torch
        self._check_factors(factors, [rank] * self.nmodes, torch.float64, "CP-APR")
        ldm = rank + (rank & 1)
        bufs = self._start_factors(factors, [rank] * self.nmodes, ldm, torch.float64, seed,
                                   lambda v, g: v.uniform_(0.0, 1.0, generator=g))
        o = default_opts()
        o[A.OPTION_NITER] = niters
        o[A.OPTION_TOLERANCE] = tol
        o[A.OPTION_VERBOSITY] = verbosity
        ao = A.AprOpts(max_inner, kappa, kappa_tol, eps)
        s, ptrs = _launch_args(bufs, stream)
        lam = np.zeros(rank)
        hist = np.full((max(int(niters), 0), 3), np.nan)
        its = C.c_int()
        rc = self.lib.splatt_b200_cp_apr_device(self.h, rank, ldm, _dptr(o), C.byref(ao), ptrs,
                                                _dptr(lam), _dptr(hist), C.byref(its), C.c_void_p(s))
        _check(rc, "splatt_b200_cp_apr_device")
        return lam, [b[:, :rank] for b in bufs], hist[:its.value].copy(), its.value

    def cp_apr_pdnr(self, rank: int, factors=None, *, niters: int = 50, tol: float = 1e-4,
                    max_inner: int = 10, max_backtrack: int = 8, mu0: float = 1e-5,
                    eps_active: float = 1e-8, eps: float = 1e-10, seed: int = 0,
                    verbosity: int = 0, stream=None):
        """Poisson CP decomposition by CP-APR with row-wise projected damped Newton steps
        (PDNR, splatt_b200_cp_apr_pdnr_device): the model and objective of `cp_apr`, each mode's
        rows solved as separate convex problems by up to `max_inner` Newton steps with a
        `max_backtrack`-point projected line search, damping `mu0` and epsilon-active set
        `eps_active`.  Needs what `cp_apr` needs; factors and seed as in `cp_apr`.  A row stops
        when its KKT violation is below `tol`; the run stops after `niters` outer iterations or
        after one in which every row stopped at its first evaluation.
        Returns (lam (numpy float64[rank]), factors (CUDA views dims[m] x rank), history (numpy
        float64 [iterations x 4] of (log-likelihood, largest last KKT violation, lockstep
        iterations summed over the modes, Newton steps attempted summed over rows and modes)),
        iterations)."""
        import torch
        self._check_factors(factors, [rank] * self.nmodes, torch.float64, "CP-APR")
        ldm = rank + (rank & 1)
        bufs = self._start_factors(factors, [rank] * self.nmodes, ldm, torch.float64, seed,
                                   lambda v, g: v.uniform_(0.0, 1.0, generator=g))
        o = default_opts()
        o[A.OPTION_NITER] = niters
        o[A.OPTION_TOLERANCE] = tol
        o[A.OPTION_VERBOSITY] = verbosity
        po = A.PdnrOpts(max_inner, max_backtrack, mu0, eps_active, eps)
        s, ptrs = _launch_args(bufs, stream)
        lam = np.zeros(rank)
        hist = np.full((max(int(niters), 0), 4), np.nan)
        its = C.c_int()
        rc = self.lib.splatt_b200_cp_apr_pdnr_device(self.h, rank, ldm, _dptr(o), C.byref(po),
                                                     ptrs, _dptr(lam), _dptr(hist), C.byref(its),
                                                     C.c_void_p(s))
        _check(rc, "splatt_b200_cp_apr_pdnr_device")
        return lam, [b[:, :rank] for b in bufs], hist[:its.value].copy(), its.value

    def cp_apr_pqnr(self, rank: int, factors=None, *, niters: int = 50, tol: float = 1e-4,
                    max_inner: int = 10, max_backtrack: int = 8, lbfgs_mem: int = 3,
                    eps_active: float = 1e-8, eps: float = 1e-10, seed: int = 0,
                    verbosity: int = 0, stream=None):
        """Poisson CP decomposition by CP-APR with row-wise projected quasi-Newton steps
        (PQNR, splatt_b200_cp_apr_pqnr_device): `cp_apr_pdnr` with the Newton direction replaced
        by an L-BFGS direction from the last `lbfgs_mem` steps of each row, so no Hessian is
        formed.  A row whose line search moves nothing continues the halving for up to two more
        rounds, then stops.  Arguments, stop rule and return value as in `cp_apr_pdnr`; history
        column 4 counts the line searches run."""
        import torch
        self._check_factors(factors, [rank] * self.nmodes, torch.float64, "CP-APR")
        ldm = rank + (rank & 1)
        bufs = self._start_factors(factors, [rank] * self.nmodes, ldm, torch.float64, seed,
                                   lambda v, g: v.uniform_(0.0, 1.0, generator=g))
        o = default_opts()
        o[A.OPTION_NITER] = niters
        o[A.OPTION_TOLERANCE] = tol
        o[A.OPTION_VERBOSITY] = verbosity
        po = A.PqnrOpts(max_inner, max_backtrack, lbfgs_mem, eps_active, eps)
        s, ptrs = _launch_args(bufs, stream)
        lam = np.zeros(rank)
        hist = np.full((max(int(niters), 0), 4), np.nan)
        its = C.c_int()
        rc = self.lib.splatt_b200_cp_apr_pqnr_device(self.h, rank, ldm, _dptr(o), C.byref(po),
                                                     ptrs, _dptr(lam), _dptr(hist), C.byref(its),
                                                     C.c_void_p(s))
        _check(rc, "splatt_b200_cp_apr_pqnr_device")
        return lam, [b[:, :rank] for b in bufs], hist[:its.value].copy(), its.value

    def ttmc(self, mode: int, mats, out, ranks):
        """TTMc (splatt_b200_ttmc): out = X_(mode) times the Kronecker product of mats[m][:, :ranks[m]],
        m != mode, columns in mode order with the highest mode fastest.  mats: float64 CUDA tensors
        (dims[m] x >= ranks[m]; mats[mode] may be None); out: a contiguous float64 CUDA tensor of
        shape (dims[mode], prod_{m != mode} ranks[m]).  Needs a whole ALLROOT tensor on the current
        device, 1 <= ranks[m] <= min(32, dims[m]) and at most 1024 columns.  Enqueued on the current
        stream; returns out."""
        import torch
        dev = torch.device("cuda", torch.cuda.current_device())
        ranks = [int(r) for r in ranks]
        if len(mats) != self.nmodes or len(ranks) != self.nmodes:
            raise ValueError(f"need {self.nmodes} matrices and ranks")
        C_ = int(np.prod([r for m, r in enumerate(ranks) if m != mode]))
        if (out.dtype != torch.float64 or out.device != dev or not out.is_contiguous() or
                tuple(out.shape) != (self.dims[mode], C_)):
            raise ValueError(f"out must be a contiguous float64 tensor of shape ({self.dims[mode]}, {C_}) "
                             f"on {dev}")
        ldm = max(ranks) + (max(ranks) & 1)
        bufs = []
        for m, f in enumerate(mats):
            if m == mode:
                bufs.append(None)
                continue
            if f.dtype != torch.float64 or f.device != dev or f.dim() != 2 or f.shape[0] != self.dims[m] \
                    or f.shape[1] < ranks[m]:
                raise ValueError(f"matrix {m} must be a float64 tensor of shape ({self.dims[m]}, >= "
                                 f"{ranks[m]}) on {dev}")
            b = torch.zeros((self.dims[m], ldm), dtype=torch.float64, device=dev)
            b[:, :ranks[m]].copy_(f[:, :ranks[m]])
            bufs.append(b)
        ptrs = (A.val_p * self.nmodes)(*[A.val_p() if b is None else C.cast(C.c_void_p(b.data_ptr()), A.val_p)
                                         for b in bufs])
        rk = (C.c_int * self.nmodes)(*ranks)
        s = torch.cuda.current_stream(dev).cuda_stream
        rc = self.lib.splatt_b200_ttmc(self.h, mode, rk, ldm, ptrs,
                                       C.cast(C.c_void_p(out.data_ptr()), A.val_p), C.c_void_p(s))
        _check(rc, "splatt_b200_ttmc")
        torch.cuda.current_stream(dev).synchronize()     # the padded copies must outlive the kernel
        return out

    def tucker(self, ranks, factors=None, *, niters: int = 50, tol: float = 1e-5, max_power: int = 50,
               svd_tol: float = 1e-10, seed: int = 0, verbosity: int = 0, stream=None):
        """Sparse Tucker decomposition by HOOI (splatt_b200_tucker_hooi_device):
        X ~ core x_0 U_0 ... x_{N-1} U_{N-1} with orthonormal factors U_m (dims[m] x ranks[m]).
        Needs a whole ALLROOT tensor on the current CUDA device, 1 <= ranks[m] <= min(32, dims[m])
        and ranks[n] <= prod_{m != n} ranks[m] <= 1024.  float64 only.

        factors: list of float64 CUDA tensors (dims[m] x ranks[m]), the start (orthonormalised by
        the call; its columns must be independent); copied into padded buffers, never written.
        None: standard normal from a torch.Generator on the current device seeded with `seed`,
        drawn mode by mode.  Each mode runs at most `max_power` orthogonal-iteration steps and
        stops them when the subspace moved by <= svd_tol; the run stops after `niters`
        iterations or when the fit moved by less than `tol`.
        Returns (core (numpy float64 of shape ranks), factors (CUDA views dims[m] x ranks[m]),
        history (numpy float64 [iterations x 4] of (fit, ||core||_F, orthogonal-iteration steps
        summed over the modes, largest final subspace residual)), iterations)."""
        import torch
        ranks = [int(r) for r in ranks]
        if len(ranks) != self.nmodes:
            raise ValueError(f"{len(ranks)} ranks for a {self.nmodes}-mode tensor")
        self._check_factors(factors, ranks, torch.float64, "Tucker")
        ldm = max(ranks) + (max(ranks) & 1)
        bufs = self._start_factors(factors, ranks, ldm, torch.float64, seed,
                                   lambda v, g: v.normal_(0.0, 1.0, generator=g))
        o = default_opts()
        o[A.OPTION_NITER] = niters
        o[A.OPTION_TOLERANCE] = tol
        o[A.OPTION_VERBOSITY] = verbosity
        to = A.TuckerOpts(max_power, svd_tol)
        s, ptrs = _launch_args(bufs, stream)
        rk = (C.c_int * self.nmodes)(*ranks)
        core = np.zeros(int(np.prod(ranks)))
        hist = np.full((max(int(niters), 0), 4), np.nan)
        its = C.c_int()
        rc = self.lib.splatt_b200_tucker_hooi_device(self.h, rk, ldm, _dptr(o), C.byref(to), ptrs,
                                                     _dptr(core), _dptr(hist), C.byref(its),
                                                     C.c_void_p(s))
        _check(rc, "splatt_b200_tucker_hooi_device")
        return (core.reshape(ranks), [b[:, :r] for b, r in zip(bufs, ranks)], hist[:its.value].copy(),
                its.value)

    def to_coo(self, stream=None):
        """This tensor's (local) nonzeros as coordinates in the record order of its first stream
        (splatt_b200_tensor_to_coo).  Returns (inds: one int32 CUDA tensor per mode, vals: a
        float64 CUDA tensor), on the current device."""
        import torch
        dev = torch.device("cuda", torch.cuda.current_device())
        inds = [torch.empty(self.nnz_local, dtype=torch.int32, device=dev) for _ in range(self.nmodes)]
        vals = torch.empty(self.nnz_local, dtype=torch.float64, device=dev)
        s = torch.cuda.current_stream(dev).cuda_stream if stream is None else stream
        rc = self.lib.splatt_b200_tensor_to_coo(self.h, _u32_ptrs(inds), C.cast(C.c_void_p(vals.data_ptr()), A.val_p),
                                                C.c_void_p(s))
        _check(rc, "splatt_b200_tensor_to_coo")
        return inds, vals

    def gcp_sample(self, seed: int, step: int, p: int, q: int, estimate: bool = False, stream=None):
        """One GCP sample set as the driver draws it (splatt_b200_gcp_sample): p stored entries
        drawn with replacement, then q uniform coordinates with value 0, from the Philox stream of
        `seed` at step `step` (estimate: the estimate sample's purposes).  Returns (inds: one int32
        CUDA tensor of p + q per mode, vals: float64 CUDA tensor of p + q)."""
        import torch
        dev = torch.device("cuda", torch.cuda.current_device())
        n = max(int(p) + int(q), 0)
        inds = [torch.empty(n, dtype=torch.int32, device=dev) for _ in range(self.nmodes)]
        vals = torch.empty(n, dtype=torch.float64, device=dev)
        s = torch.cuda.current_stream(dev).cuda_stream if stream is None else stream
        rc = self.lib.splatt_b200_gcp_sample(self.h, int(seed), int(step), int(bool(estimate)), int(p), int(q),
                                             _u32_ptrs(inds), C.cast(C.c_void_p(vals.data_ptr()), A.val_p),
                                             C.c_void_p(s))
        _check(rc, "splatt_b200_gcp_sample")
        return inds, vals

    def gcp_sampled(self, loss, inds, vals, p: int, q: int, w_nz: float, w_z: float, factors, *,
                    rank: Optional[int] = None, grads=True, stream=None):
        """The GCP kernel primitive (splatt_b200_gcp_sampled) on an explicit sample: inds (one
        int32 CUDA tensor of >= p + q per mode) and vals (float64, the first p are read) with
        samples 0..p-1 stored entries of weight w_nz and p..p+q-1 coordinates of weight w_z.
        factors: float64 CUDA tensors (dims[m] x >= rank), used in place when they share one
        even, 16-byte-aligned row stride, else copied into padded buffers.  grads: True (new
        buffers), False (value only), or a list of float64 CUDA tensors laid out like the
        factors, whose first `rank` columns are overwritten.  Returns (value, grads or None)."""
        import torch
        loss = A.GCP_LOSSES[loss] if isinstance(loss, str) else int(loss)
        R = factors[0].shape[1] if rank is None else int(rank)
        dev = torch.device("cuda", torch.cuda.current_device())
        ldm = factors[0].stride(0)
        direct = (len(factors) == self.nmodes and ldm % 2 == 0 and ldm >= R and
                  all(f.dtype == torch.float64 and f.device == dev and f.stride(1) == 1 and f.stride(0) == ldm
                      and f.data_ptr() % 16 == 0 and tuple(f.shape[:1]) == (self.dims[m],) and f.shape[1] >= R
                      for m, f in enumerate(factors)))
        if not direct:
            self._check_factors([f[:, :R] for f in factors], [R] * self.nmodes, torch.float64, "GCP")
            ldm = R + (R & 1)
            factors = self._start_factors([f[:, :R] for f in factors], [R] * self.nmodes, ldm, torch.float64)
        if grads is True:
            gbufs = [torch.zeros((d, ldm), dtype=torch.float64, device=dev) for d in self.dims]
        elif grads:
            gbufs = list(grads)
            if any(g.stride(0) != ldm or g.stride(1) != 1 or g.dtype != torch.float64 for g in gbufs):
                raise ValueError("grads must be float64 CUDA tensors with the factors' row stride")
        else:
            gbufs = None
        if stream is not None:
            torch.cuda.current_stream(dev).synchronize()      # the buffers were filled there
        s = torch.cuda.current_stream(dev).cuda_stream if stream is None else stream
        fp = (A.val_p * self.nmodes)(*[C.cast(C.c_void_p(f.data_ptr()), A.val_p) for f in factors])
        gp = None if gbufs is None else (A.val_p * self.nmodes)(*[C.cast(C.c_void_p(g.data_ptr()), A.val_p)
                                                                  for g in gbufs])
        out = C.c_double()
        rc = self.lib.splatt_b200_gcp_sampled(self.h, loss, int(p), int(q), float(w_nz), float(w_z),
                                              _u32_ptrs(inds), C.cast(C.c_void_p(vals.data_ptr()), A.val_p),
                                              R, ldm, fp, gp, C.byref(out), C.c_void_p(s))
        _check(rc, "splatt_b200_gcp_sampled")
        return out.value, None if gbufs is None else [g[:, :R] for g in gbufs]

    def gcp(self, rank: int, loss="bernoulli-logit", factors=None, *, niters: int = 50,
            tol: float = 1e-4, grad_samples=(1 << 16, 1 << 16), est_samples=(1 << 20, 1 << 20),
            epoch_iters: int = 1000, lr: float = 1e-3, beta1: float = 0.9, beta2: float = 0.999,
            epsilon: float = 1e-8, decay: float = 0.1, max_fails: int = 1, seed: int = 0,
            verbosity: int = 0, stream=None):
        """Generalized CP decomposition by sampled gradients and Adam (GCP-Adam,
        splatt_b200_gcp_device): fits sum_r prod_m U_m[i_m, r] to every coordinate of this
        tensor (unstored ones being 0) under `loss` ("gaussian", "bernoulli-logit" or
        "poisson-log").  Each step draws grad_samples = (p stored entries, q coordinates) and
        applies one Adam update; an epoch of `epoch_iters` steps is scored on one fixed sample of
        est_samples and accepted if the estimate did not rise, else undone with lr *= decay.
        Stops after `niters` epochs, more than `max_fails` failed epochs, or an accepted epoch
        that decreased the estimate by less than `tol` relative.  Needs a whole tensor on the
        current CUDA device, values allowed by the loss, and 1 <= rank <= 64.  float64 only.

        factors: list of float64 CUDA tensors (dims[m] x rank), the start; copied into padded
        buffers, never written.  None: N(0, 1) R^(-1/(2N)) entries from a torch.Generator on the
        current device seeded with `seed` (so the model starts with unit variance); `seed` also
        keys every sample.
        Returns (factors (CUDA views dims[m] x rank), history (numpy float64 [epochs x 3] of
        (estimate, lr used, accepted 1/0)), epochs, f_start (the estimate at the start))."""
        import torch
        self._check_factors(factors, [rank] * self.nmodes, torch.float64, "GCP")
        if loss not in A.GCP_LOSSES:
            raise ValueError(f"loss must be one of {sorted(A.GCP_LOSSES)}, not {loss!r}")
        ldm = rank + (rank & 1)
        scale = float(rank) ** (-1.0 / (2 * self.nmodes)) if rank > 0 else 1.0
        bufs = self._start_factors(factors, [rank] * self.nmodes, ldm, torch.float64, seed,
                                   lambda v, g: v.normal_(0.0, 1.0, generator=g).mul_(scale))
        o = default_opts()
        o[A.OPTION_NITER] = niters
        o[A.OPTION_TOLERANCE] = tol
        o[A.OPTION_VERBOSITY] = verbosity
        go = A.GcpOpts(A.GCP_LOSSES[loss], int(grad_samples[0]), int(grad_samples[1]), int(est_samples[0]),
                       int(est_samples[1]), int(epoch_iters), lr, beta1, beta2, epsilon, decay,
                       int(max_fails), int(seed) & 0xFFFFFFFFFFFFFFFF)
        s, ptrs = _launch_args(bufs, stream)
        hist = np.full((max(int(niters), 0), 3), np.nan)
        f0 = C.c_double(np.nan)
        its = C.c_int()
        rc = self.lib.splatt_b200_gcp_device(self.h, rank, ldm, _dptr(o), C.byref(go), ptrs, _dptr(hist),
                                             C.byref(f0), C.byref(its), C.c_void_p(s))
        _check(rc, "splatt_b200_gcp_device")
        return [b[:, :rank] for b in bufs], hist[:its.value].copy(), its.value, f0.value

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
