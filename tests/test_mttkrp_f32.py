"""Single-precision MTTKRP (splatt_b200_mttkrp_f32 / Tensor.mttkrp on float32 buffers).

The fp32 kernels are the fp64 stream kernels instantiated for float: a lane carries four
columns (float4), so one launch covers 128 columns and the lane-group width L follows from
the columns of each 128-column pass (<= 16: L = 4, <= 32: 8, <= 64: 16, else 32).  The
records keep their fp64 values; the kernel rounds each one to fp32 once and computes in fp32.

The oracle is torch fp64 on the device, from the fp32 factors upcast exactly and the fp64
values.  For output row i with n_i nonzeros every entry of [:, :R] must satisfy

    |out - ref| <= 2 * gamma(n_i + N + 1) * absref + n_i * 2^-126,  u = 2^-24,

(the +1 is the rounding of the value; the absolute term covers red.add.f32 flushing subnormal
sums to zero).  Rows without nonzeros are exactly +0.0, and [rpad4, ldm) is zero.
"""
from __future__ import annotations

import ctypes as C
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

from splatt_b200 import _abi as A
from tests import test_kernel_matrix as KM
from tests.test_kernel_matrix import ALLROOT, CANARY, LANES, MATRIX, NAN, ONEMODE, TILED

ROOT = Path(__file__).resolve().parent.parent
U32 = 2.0 ** -24
TINY = 2.0 ** -126
CANARY32 = -1.2345e30                 # fp32 outputs start out holding this


# ---------------------------------------------------------------------------------------
# The case table (fp32 lane rule)
# ---------------------------------------------------------------------------------------
# Per (N, layout): an L = 8 row, an L = 16 row and a two-pass row (L = 32, then L = 4).
# TILED: the CTA-tiled 3-mode stream, which fp32 multiplies with the generic kernel.
CASES = []
for _N in range(2, 9):
    _Rs = (20, 40, 130) if _N % 2 == 0 else (17, 64, 131)
    for _layout in (ALLROOT, ONEMODE):
        for _j, _R in enumerate(_Rs):
            CASES.append((_N, _layout, _R, 4 * ((_j + _N + (_layout == ONEMODE)) % 3)))
CASES.append((3, TILED, 130, 4))


def _case_id(c):
    return f"n{c[0]}-{c[1]}-R{c[2]}-ldm+{c[3]}"


def rpad4(R):
    return (R + 3) & ~3


def passes(R):
    """Active columns of the 128-column launches of a whole-matrix fp32 call."""
    end = rpad4(R)
    return [min(128, end - c) for c in range(0, end, 128)]


def lanes(ncols):
    return 4 if ncols <= 16 else 8 if ncols <= 32 else 16 if ncols <= 64 else 32


def _covers(lib, case):
    N, layout, R, _ = case
    kinds = set(KM._kinds(lib, KM._gapped_dims(MATRIX[N][0]), layout))
    widths = passes(R)
    out = {(N, layout, k, lanes(w)) for k in kinds for w in widths}
    if len(widths) >= 2:
        out |= {(N, layout, k, "multi") for k in kinds}
    return out


def _required(lib):
    req = {(3, TILED, "root", "multi")}
    for N in range(2, 9):
        for layout in (ALLROOT, ONEMODE):
            for k in set(KM._kinds(lib, KM._gapped_dims(MATRIX[N][0]), layout)):
                req |= {(N, layout, k, L) for L in LANES}
                req.add((N, layout, k, "multi"))
    return req


def test_f32_case_table_reaches_every_kernel(lib):
    """CPU: under the fp32 lane rule the table reaches every (N, layout, kind, L), a
    multi-pass call per (N, layout, kind) and the forced CTA-tiled stream; no row is
    redundant."""
    req = _required(lib)
    got = [_covers(lib, c) & req for c in CASES]
    assert req - set().union(*got) == set()
    for i, c in enumerate(CASES):
        others = set().union(*(g for j, g in enumerate(got) if j != i))
        assert got[i] - others, f"row {c} reaches nothing the other rows do not"


def test_f32_declared():
    """CPU: the header declares the entry and the loader gives it a prototype."""
    hdr = (ROOT / "include" / "splatt_b200.h").read_text()
    assert "int splatt_b200_mttkrp_f32(" in hdr
    assert "splatt_b200_mttkrp_f32" in A.EXPORTS
    lib = A.load()
    f = lib.splatt_b200_mttkrp_f32
    assert f.restype is C.c_int
    assert f.argtypes == [C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(A.f32_p), A.f32_p,
                          C.c_void_p]


_KERNEL = re.compile(r"mttkrp_stream_kernelI([fd])((?:L[ib]\d+E)+)E")


def _stream_kernel_resources():
    """{(value type, N, L, kind, batch, KT, MC, MINB, STAGES): (registers, stack, local)} of
    every stream kernel in the built library (cuobjdump -res-usage)."""
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not Path(tool).exists():
        pytest.skip("cuobjdump not found")
    txt = subprocess.run([tool, "-res-usage", str(A.LIB_PATH)], capture_output=True, text=True,
                         check=True).stdout
    out, cur = {}, None
    for line in txt.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            k = _KERNEL.search(m.group(1))
            cur = ((k.group(1),) + tuple(int(v) for v in re.findall(r"L[ib](\d+)E", k.group(2))[:8])
                   if k else None)
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+) .*LOCAL:(\d+)", line)
        if m and cur is not None:
            out[cur] = tuple(int(x) for x in m.groups())
            cur = None
    return out


def test_f32_kernels_within_f64_registers():
    """CPU: every fp32 stream kernel in the built library holds no more registers than its
    fp64 counterpart (same N, L, kind, batch, variant), so it runs at least as many CTAs per
    SM, and uses no stack or local memory (no spills)."""
    A.load()
    res = _stream_kernel_resources()
    f32 = {k: v for k, v in res.items() if k[0] == "f"}
    assert len(f32) == 92, len(f32)                       # 7 N x 4 L x (intl, leaf, root[, KT])
    for k, (reg, stack, local) in f32.items():
        ref = res[("d",) + k[1:]]
        assert reg <= ref[0], f"fp32 kernel {k[1:]}: {reg} registers, fp64 {ref[0]}"
        assert stack == 0 and local == 0, f"fp32 kernel {k[1:]} spills"


# ---------------------------------------------------------------------------------------
# Oracle and checks
# ---------------------------------------------------------------------------------------
def poisoned_f32(dims, ind, R, ldm, seed):
    """fp32 factors uniform in [-3, 3) on referenced rows; NaN elsewhere and in [R, ldm)."""
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    mats = []
    for d, i in zip(dims, ind):
        x = torch.full((d, ldm), NAN, dtype=torch.float32, device="cuda")
        rows = torch.unique(i)
        x[rows, :R] = torch.rand((len(rows), R), dtype=torch.float32, device="cuda", generator=g) * 6 - 3
        mats.append(x)
    return mats


def oracle32(dims, ind_d, vals_d, mats32, mode, R):
    return KM.oracle(dims, ind_d, vals_d, [m.double() for m in mats32], mode, R)


def check_f32(out, R, ora, N, what):
    """A whole-matrix fp32 call: [:, :R] within the bound, empty rows +0.0, [rpad4, ldm) 0."""
    import torch
    ref, absref, n = ora
    got = out[:, :R].double()
    nf = n.to(torch.float64)[:, None]
    k = nf + N + 1
    bound = 2.0 * (k * U32 / (1.0 - k * U32)) * absref + nf * TINY
    err = (got - ref).abs()
    bad = ~(err <= bound)
    if bool(bad.any()):
        r, c = [int(x) for x in bad.nonzero()[0]]
        raise AssertionError(f"{what}: {int(bad.sum())} entries out of bound, first at row {r} "
                             f"col {c}: got {float(got[r, c])!r}, want {float(ref[r, c])!r}, "
                             f"bound {float(bound[r, c])!r}, n_i {int(n[r])}")
    empty = out[n == 0]
    assert bool((empty[:, :R] == 0).all()) and not bool(empty[:, :R].signbit().any()), \
        f"{what}: an empty row is not +0.0"
    tail = out[:, rpad4(R):]
    assert bool((tail == 0).all()) and not bool(tail.signbit().any()), f"{what}: [rpad4, ldm) not 0"


def run_modes32(S, T, dims, ind_d, vals_d, R, ldm, what, seed=0):
    import torch
    N = len(dims)
    mats = poisoned_f32(dims, ind_d, R, ldm, seed)
    for m in range(N):
        out = torch.full((dims[m], ldm), CANARY32, dtype=torch.float32, device="cuda")
        before = S.launch_count()
        T.mttkrp(m, mats, out, ncolumns=R)
        assert S.launch_count() - before == (len(passes(R)) if T.nnz_local else 0), (what, m)
        torch.cuda.synchronize()
        check_f32(out, R, oracle32(dims, ind_d, vals_d, mats, m, R), N, f"{what} mode {m}")


@pytest.fixture(scope="module")
def S():
    import splatt_b200
    return splatt_b200


# ---------------------------------------------------------------------------------------
# GPU tests
# ---------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_f32_kernel_matrix(S, lib, case):
    N, layout, R, extra = case
    dims, inds, vals = KM.matrix_tensor(N)
    ind_d, vals_d = KM.to_dev(inds, vals)
    T = KM.build(S, dims, inds, vals, layout)
    kinds = KM._kinds(lib, dims, layout)
    for m in range(N):
        assert T.mode_info(m, R)["kind"] == kinds[m], (case, m)
    run_modes32(S, T, dims, ind_d, vals_d, R, rpad4(R) + extra, _case_id(case), seed=N)
    T.free()


@pytest.mark.gpu
@pytest.mark.parametrize("N", range(2, 9))
def test_f32_traversal_edges(S, N):
    """The traversal-edge tensors at R = 3 (L = 4) and R = 129 (L = 32, then a second
    pass), ALLROOT and ONEMODE; an empty tensor zeroes the output and launches nothing."""
    import torch
    for name, dims, inds, vals in KM._edge_tensors(N):
        ind_d, vals_d = KM.to_dev(inds, vals)
        for layout in (ALLROOT, ONEMODE):
            T = KM.build(S, dims, inds, vals, layout)
            for R, extra in ((3, 4), (129, 0)):
                run_modes32(S, T, dims, ind_d, vals_d, R, rpad4(R) + extra,
                            f"n{N} {name} {layout} R{R}", seed=N + R)
            T.free()
    e = np.zeros(0, np.uint64)
    dims = [4 + m for m in range(N)]
    for layout in (ALLROOT, ONEMODE):
        T = KM.build(S, dims, [e] * N, np.zeros(0), layout)
        mats = [torch.ones((d, 8), dtype=torch.float32, device="cuda") for d in dims]
        for m in range(N):
            out = torch.full((dims[m], 8), CANARY32, dtype=torch.float32, device="cuda")
            before = S.launch_count()
            T.mttkrp(m, mats, out, ncolumns=5)
            assert S.launch_count() == before
            torch.cuda.synchronize()
            assert bool((out == 0).all()) and not bool(out.signbit().any()), (N, layout, m)
        T.free()


@pytest.mark.gpu
@pytest.mark.parametrize("layout", [ALLROOT, ONEMODE])
@pytest.mark.parametrize("N", [3, 5])
def test_f32_shards(S, N, layout):
    """2 and 3 shards built with shard_count: the sum of the fp32 partials meets the bound."""
    import torch
    dims, inds, vals = KM.matrix_tensor(N)
    ind_d, vals_d = KM.to_dev(inds, vals)
    R = 37
    ldm = rpad4(R)
    mats = poisoned_f32(dims, ind_d, R, ldm, seed=11)
    for count in (2, 3):
        Ts = [KM.build(S, dims, inds, vals, layout, shard_rank=r, shard_count=count)
              for r in range(count)]
        assert sum(T.nnz_local for T in Ts) == len(vals)
        for m in range(N):
            total = torch.zeros((dims[m], ldm), dtype=torch.float64, device="cuda")
            for T in Ts:
                out = torch.full((dims[m], ldm), CANARY32, dtype=torch.float32, device="cuda")
                T.mttkrp(m, mats, out, ncolumns=R)
                total += out.double()
            torch.cuda.synchronize()
            ora = oracle32(dims, ind_d, vals_d, mats, m, R)
            check_f32(total, R, ora, N, f"n{N} {layout} {count} shards mode {m}")
        for T in Ts:
            T.free()


@pytest.mark.gpu
@pytest.mark.parametrize("layout", [ALLROOT, ONEMODE, TILED])
def test_f32_mixed_with_f64(S, layout):
    """fp64 and fp32 calls interleaved on one tensor each meet their own bound."""
    import torch
    N = 3 if layout == TILED else 4
    dims, inds, vals = KM.matrix_tensor(N)
    ind_d, vals_d = KM.to_dev(inds, vals)
    T = KM.build(S, dims, inds, vals, layout)
    R = 33
    m32 = poisoned_f32(dims, ind_d, R, rpad4(R), seed=3)
    m64 = KM.poisoned_factors(dims, ind_d, R, KM._rpad(R), seed=4)
    for rnd in range(2):
        for m in range(N):
            o64 = torch.full((dims[m], KM._rpad(R)), CANARY, dtype=torch.float64, device="cuda")
            o32 = torch.full((dims[m], rpad4(R)), CANARY32, dtype=torch.float32, device="cuda")
            T.mttkrp(m, m64, o64, ncolumns=R)
            T.mttkrp(m, m32, o32, ncolumns=R)
            torch.cuda.synchronize()
            KM.check_whole(o64, R, KM.oracle(dims, ind_d, vals_d, m64, m, R), N,
                           f"{layout} fp64 round {rnd} mode {m}")
            check_f32(o32, R, oracle32(dims, ind_d, vals_d, m32, m, R), N,
                      f"{layout} fp32 round {rnd} mode {m}")
    T.free()


def _call_f32(T, mode, R, ldm, mats, out_ptr):
    import torch
    ptrs = (A.f32_p * len(mats))(*[A.f32_p() if k == mode else C.cast(C.c_void_p(p), A.f32_p)
                                   for k, p in enumerate(mats)])
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    return T.lib.splatt_b200_mttkrp_f32(T.h, mode, R, ldm, ptrs, C.cast(C.c_void_p(out_ptr), A.f32_p), s)


@pytest.mark.gpu
@pytest.mark.parametrize("layout", [ALLROOT, TILED])
def test_f32_bad_input(S, layout):
    """ldm % 4 != 0, ldm < rpad4, a factor 4 bytes off 16-byte alignment and a null output
    return SPLATT_ERROR_BADINPUT and leave the canary-filled output untouched."""
    import torch
    N = 3
    dims, inds, vals = KM.matrix_tensor(N)
    ind_d, vals_d = KM.to_dev(inds, vals)
    T = KM.build(S, dims, inds, vals, layout)
    R = 5
    for m in range(N):
        for ldm, shift in ((10, 0), (4, 0), (8, 1)):
            bufs = [torch.zeros(d * ldm + 4, dtype=torch.float32, device="cuda") for d in dims]
            mats = [b.data_ptr() + 4 * shift for b in bufs]
            out = torch.full((dims[m] * 12,), CANARY32, dtype=torch.float32, device="cuda")
            rc = _call_f32(T, m, R, ldm, mats, out.data_ptr())
            assert rc == A.SPLATT_ERROR_BADINPUT, (layout, m, ldm, shift)
            torch.cuda.synchronize()
            assert bool((out == CANARY32).all()), (layout, m, ldm, shift)
        good = [torch.zeros((d, 8), dtype=torch.float32, device="cuda") for d in dims]
        assert _call_f32(T, m, R, 8, [g.data_ptr() for g in good], 0) == A.SPLATT_ERROR_BADINPUT
        # the same call with an output runs
        out = torch.full((dims[m], 8), CANARY32, dtype=torch.float32, device="cuda")
        assert _call_f32(T, m, R, 8, [g.data_ptr() for g in good], out.data_ptr()) == A.SPLATT_SUCCESS
        torch.cuda.synchronize()
        assert bool((out == 0).all())
    T.free()


@pytest.mark.gpu
def test_f32_python_dtype_rules(S):
    """Mixed dtypes and other dtypes raise ValueError; float32 needs stride(0) % 4 == 0."""
    import torch
    dims, inds, vals = KM.matrix_tensor(3)
    T = KM.build(S, dims, inds, vals, ALLROOT)
    m32 = [torch.zeros((d, 8), dtype=torch.float32, device="cuda") for d in dims]
    m64 = [torch.zeros((d, 8), dtype=torch.float64, device="cuda") for d in dims]
    with pytest.raises(ValueError, match="float32"):
        T.mttkrp(0, m32, torch.zeros((dims[0], 8), dtype=torch.float64, device="cuda"), ncolumns=5)
    with pytest.raises(ValueError, match="float64"):
        T.mttkrp(0, m64, torch.zeros((dims[0], 8), dtype=torch.float32, device="cuda"), ncolumns=5)
    mixed = [m64[0], m32[1], m64[2]]
    with pytest.raises(ValueError):
        T.mttkrp(0, mixed, torch.zeros((dims[0], 8), dtype=torch.float64, device="cuda"), ncolumns=5)
    with pytest.raises(ValueError):
        T.mttkrp(0, [m.half() for m in m32], torch.zeros((dims[0], 8), dtype=torch.float16,
                                                         device="cuda"), ncolumns=5)
    m6 = [torch.zeros((d, 6), dtype=torch.float32, device="cuda") for d in dims]
    with pytest.raises(ValueError, match="multiple of 4"):
        T.mttkrp(0, m6, torch.zeros((dims[0], 6), dtype=torch.float32, device="cuda"), ncolumns=5)
    T.free()


@pytest.mark.gpu
def test_from_coo_float32_values(S):
    """Device float32 values are widened exactly: the tensor equals the one built from the
    widened float64 values (same structure, same fp64 products); other dtypes raise."""
    import torch
    N = 3
    dims, inds, vals = KM.matrix_tensor(N)
    ind_d = [torch.from_numpy(i.astype(np.int32)).cuda() for i in inds]
    v32 = torch.from_numpy(vals.astype(np.float32)).cuda()
    v64 = v32.to(torch.float64)
    Ta = S.Tensor.from_coo(dims, ind_d, v32)
    Tb = S.Tensor.from_coo(dims, ind_d, v64)
    R = 9
    mats = KM.poisoned_factors(dims, [i.long() for i in ind_d], R, KM._rpad(R), seed=8)
    for m in range(N):
        assert Ta.mode_info(m, R) == Tb.mode_info(m, R)
        ora = KM.oracle(dims, [i.long() for i in ind_d], v64, mats, m, R)
        for T in (Ta, Tb):
            out = torch.full((dims[m], KM._rpad(R)), CANARY, dtype=torch.float64, device="cuda")
            T.mttkrp(m, mats, out, ncolumns=R)
            torch.cuda.synchronize()
            KM.check_whole(out, R, ora, N, f"from_coo float32 mode {m}")
    Ta.free()
    Tb.free()
    with pytest.raises(ValueError):
        S.Tensor.from_coo(dims, ind_d, v32.half())


@pytest.mark.gpu
def test_f32_config2_full_size(S):
    """bench.py's headline tensor (10K^3, 10 M nonzeros, R = 32): every mode in fp32 meets
    the bound against fp64 (default build: the CTA-tiled stream where it applies)."""
    import torch
    import bench
    dev = torch.device("cuda", torch.cuda.current_device())
    dims = [bench.DIM] * bench.NMODES
    ind, vals = bench.make_coo_gpu(bench.NNZ_PER_GPU, dev)
    T = S.Tensor.from_coo(dims, ind, vals)
    ind_d = [i.long() for i in ind]
    del ind
    R = bench.RANK
    mats = [torch.from_numpy(m).to(dev).float() for m in bench.make_factors_host(bench.SEED, dims, R)]
    for m in range(len(dims)):
        out = torch.empty((dims[m], R), dtype=torch.float32, device=dev)
        before = S.launch_count()
        T.mttkrp(m, mats, out)
        assert S.launch_count() - before == 1
        torch.cuda.synchronize()
        check_f32(out, R, oracle32(dims, ind_d, vals, mats, m, R), len(dims), f"config 2 mode {m}")
    T.free()
