"""Nonnegative CPD by HALS (splatt_b200_cpd_nonneg_device / _f32, Tensor.cpd_nonneg) against the
numpy restatement in oracle/cpd_nonneg.py.

CPU: the oracle's sweep is exact coordinate descent (repeated sweeps reach scipy's nnls on every
row), its fit never decreases, it recovers a planted model; the case table; the new symbols; no
new kernel spills.
GPU: parity with the oracle at every mode count, precision and sweep kernel; the layouts; every
run's result is well formed; a planted model; pad columns; input rules.

Parity bars.  fp64: |dfit| <= 1e-9, lambda rtol 1e-6, factor entries within 1e-6.  The device
sums the MTTKRP, the Grams and the column norms in other orders than numpy (atomics among them),
so every step differs from the oracle's by rounding, and three iterations carry that forward; the
factors have unit columns, so 1e-6 absolute is a relative bound on each column.  fp32: the bars
of CPD-ALS's fp32 entry against its fp64 reference (tests/test_cpd_matrix.check_reference):
|dfit| <= 1e-6, lambda rtol 1e-4, relative Frobenius 1e-4 per factor.
Some trajectories are ill-conditioned: a column swept almost entirely to the floor keeps a few
entries formed by cancellation, and its direction after the normalisation is set by rounding.
On the 2-mode problems (where G is a single Gram, with large off-diagonal entries) and at N = 4,
R = 40 the oracle itself moves by up to 1e-3 in fit after three iterations when its values and
start are perturbed by 1e-13 relative.  So each bar is the larger of the one above and 10 times
the oracle's own spread under a perturbation at the precision's rounding level (1e-13 in fp64,
1e-7 in fp32); on the well-conditioned cases, which include every sweep kernel at N = 3, the
fixed bars decide.
"""
from __future__ import annotations

import ctypes as C
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

from oracle import cpd_nonneg as O
from splatt_b200 import _abi as A
from tests import test_cpd_matrix as CM
from tests import test_kernel_matrix as KM
from tests.util import random_coo, rel_fro

HERE = Path(__file__).resolve().parent
ITS = 3
DTYPES = ("float64", "float32")

# (N, R, SPLATT_B200_TAIL_GENERIC): at every mode count one rank per sweep kernel (register tile
# 16 / 32 / 64 and the generic kernel), and at N = 3 the ranks around every tile edge up to 128.
# Problems: tests/test_cpd_matrix.problem (empty first, last and interior slices in every mode,
# 40 duplicate coordinates, values of either sign).
CASES = sorted({(N, R, g) for N in range(2, 9) for R, g in ((5, "0"), (20, "0"), (40, "0"), (7, "1"))}
               | {(3, R, "0") for R in (1, 5, 16, 17, 32, 33, 64, 65, 128)})


def tier(R, generic):
    """The sweep kernel DevTail::hals (cpd.cu) launches: k_hals_rows_reg<rt> for
    rt = R <= 16 ? 16 : R <= 32 ? 32 : R <= 64 ? 64 : 0, k_hals_rows when rt == 0 or under
    SPLATT_B200_TAIL_GENERIC=1."""
    if generic == "1" or R > 64:
        return "generic"
    return 16 if R <= 16 else 32 if R <= 32 else 64


def nonneg_start(dims, R, seed):
    rng = np.random.default_rng(seed)
    return [rng.uniform(0.0, 1.0, size=(d, R)) for d in dims]


def planted(seed=0):
    """30 x 40 x 50, exact rank 4, factors 40 % nonzero: every nonzero entry stored."""
    rng = np.random.default_rng(seed)
    dims, R = (30, 40, 50), 4
    F = [rng.uniform(0.0, 1.0, size=(d, R)) * (rng.uniform(size=(d, R)) < 0.4) for d in dims]
    X = np.einsum("ir,jr,kr->ijk", *F)
    idx = np.nonzero(X)
    return list(dims), [i.astype(np.uint64) for i in idx], X[idx], F


def congruence(F, A):
    """Smallest per-component congruence (product over the modes of the column cosines) after the
    best matching of the columns."""
    from scipy.optimize import linear_sum_assignment
    C_ = np.ones((F[0].shape[1], A[0].shape[1]))
    for f, a in zip(F, A):
        C_ *= (f / np.linalg.norm(f, axis=0)).T @ (a / np.linalg.norm(a, axis=0))
    r, c = linear_sum_assignment(-C_)
    return float(C_[r, c].min())


# ---------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------
def test_oracle_sweep_is_coordinate_descent():
    """With M and G fixed, repeated sweeps reach the solution of every row's problem
    min_b 1/2 b^T G b - m^T b, b >= 0, i.e. nnls(L^T, L^-1 m) with G = L L^T."""
    from scipy.optimize import nnls
    rng = np.random.default_rng(3)
    R, I = 6, 40
    mats = [rng.uniform(size=(30, R)) for _ in range(2)]
    mats = [a / np.linalg.norm(a, axis=0) for a in mats]
    G = (mats[0].T @ mats[0]) * (mats[1].T @ mats[1])
    M = rng.standard_normal((I, R))
    B = rng.uniform(size=(I, R))
    for _ in range(3000):
        B = O.sweep(B, M, G)
    L = np.linalg.cholesky(G)
    for i in range(I):
        want, _ = nnls(L.T, np.linalg.solve(L, M[i]))
        assert np.max(np.abs(B[i] - want)) <= 1e-8, (i, B[i], want)
    assert np.any(B <= O.EPS)            # the bound is active somewhere


def test_oracle_fit_never_decreases():
    dims, inds, vals = random_coo((25, 30, 20), 1500, seed=5)
    fit, lam, A_, h = O.cpd_nonneg(dims, inds, vals, nonneg_start(dims, 6, 1), 30, 0.0)
    assert len(h) == 30 and h[-1] < 0.9
    assert np.all(np.diff(h) >= -1e-12), np.diff(h).min()
    assert all(np.all(a >= 0) for a in A_) and np.all(lam >= 0)


def test_oracle_recovers_planted_model():
    dims, inds, vals, F = planted()
    assert 10000 < len(vals) < 13000
    fit, lam, A_, h = O.cpd_nonneg(dims, inds, vals, nonneg_start(dims, 4, 0), 50, 1e-10)
    assert 1 - fit < 1e-6, h
    assert congruence(F, A_) >= 0.999


def test_case_table_reaches_every_mode_count_and_kernel():
    """Every case runs in both precisions; together they reach every (N, dtype, kernel)."""
    got = {(N, dt, tier(R, g)) for N, R, g in CASES for dt in DTYPES}
    want = {(N, dt, t) for N in range(2, 9) for dt in DTYPES for t in (16, 32, 64, "generic")}
    assert got == want
    assert {R for N, R, g in CASES if N == 3} >= {1, 5, 16, 17, 32, 33, 64, 65, 128}


def test_nonneg_symbols_declared():
    hdr = (HERE.parent / "include" / "splatt_b200.h").read_text()
    for sym in ("splatt_b200_cpd_nonneg_device", "splatt_b200_cpd_nonneg_device_f32"):
        assert f"int {sym}(" in hdr and sym in A.EXPORTS


def hals_resources():
    """{kernel symbol: (registers, stack, local bytes)} of the HALS kernels in the library."""
    A.load()
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not Path(tool).exists():
        pytest.skip("cuobjdump not found")
    txt = subprocess.run([tool, "-res-usage", str(A.LIB_PATH)], capture_output=True, text=True,
                         check=True).stdout
    found, cur = {}, None
    for line in txt.splitlines():
        m = re.search(r"Function (\S*(k_hals|k_nonneg_check)\S*):", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+) .*LOCAL:(\d+)", line)
        if m and cur:
            found[cur] = tuple(int(x) for x in m.groups())
            cur = None
    return found


def test_hals_kernels_do_not_spill():
    found = hals_resources()
    assert sum("k_hals_rows_regI" in k for k in found) == 3 * 2
    assert sum("k_hals_rowsI" in k for k in found) == 2
    assert sum("k_hals_formE" in k for k in found) == 1
    assert sum("k_nonneg_checkI" in k for k in found) == 2
    for k, (reg, stack, local) in found.items():
        assert stack == 0 and local == 0, f"{k} spills"


# ---------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def S():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import splatt_b200 as S
    return S


def run(T, R, start, dtype, niters, tol=0.0):
    """Tensor.cpd_nonneg: (fit, lambda, factors (numpy fp64), iterations, history)."""
    import torch
    init = [torch.from_numpy(np.asarray(a)).to("cuda", getattr(torch, dtype)) for a in start]
    fit, lam, fac, its, hist = T.cpd_nonneg(R, init, niters=niters, tol=tol)
    torch.cuda.synchronize()
    return fit, lam, [f.double().cpu().numpy() for f in fac], its, hist


def check_well_formed(inds, vals, got, what, fp32, inexact=True):
    """The reported fit is the fit of the returned model (CPD-ALS's check, with its fp32 bound);
    unit columns; every entry >= 0; history[its - 1] == fit; and, on a problem that does not fit
    exactly, a history that does not decrease (fp32: beyond its fit resolution of 1e-6).
    On an exact problem the fit 1 - sqrt(||X||^2 + ||K||^2 - 2<X,K>) / ||X|| resolves only about
    sqrt(u) (the residual is a difference of terms of size ||X||^2, each off by a few u), so there
    the reported fit is held to sqrt(64 u) of the recomputed one."""
    fit, lam, facs, its, hist = got
    if inexact:
        CM.check_model(inds, vals, fit, lam, facs, what, fp32=fp32)
    else:
        u = CM.U32 if fp32 else 2.0 ** -53
        want = CM.model_fit(inds, vals, lam, facs)[0]
        assert abs(fit - want) <= np.sqrt(64 * u), (what, fit, want)
        for a in facs:
            assert np.allclose(np.linalg.norm(a, axis=0), 1.0, rtol=2 * CM.U32 if fp32 else 1e-12, atol=0)
    assert all(np.all(a >= 0) for a in facs) and np.all(lam >= 0), what
    assert len(hist) == its and hist[-1] == fit, (what, hist, fit)
    if inexact:
        assert np.all(np.diff(hist) >= -(1e-6 if fp32 else 1e-12)), (what, hist)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", CASES, ids=lambda c: f"n{c[0]}-R{c[1]}-generic{c[2]}")
def test_parity_with_oracle(S, case, dtype, monkeypatch):
    N, R, generic = case
    monkeypatch.setenv("SPLATT_B200_TAIL_GENERIC", generic)
    dims, inds, vals = CM.problem(N)
    start = nonneg_start(dims, R, seed=N * 1000 + R)
    T = S.Tensor.from_coo(dims, inds, vals)
    got = run(T, R, start, dtype, ITS)
    T.free()
    fp32 = dtype == "float32"
    what = f"{case} {dtype}"
    assert got[3] == ITS
    check_well_formed(inds, vals, got, what, fp32)
    ref = O.cpd_nonneg(dims, inds, vals, start, ITS, 0.0)
    sf, sl, sa = oracle_spread(dims, inds, vals, start, ref, 1e-7 if fp32 else 1e-13)
    assert abs(got[0] - ref[0]) <= max(1e-6 if fp32 else 1e-9, 10 * sf), (what, got[0], ref[0], sf)
    assert np.allclose(got[1], ref[1], rtol=max(1e-4 if fp32 else 1e-6, 10 * sl), atol=0), what
    for m, (a, b) in enumerate(zip(got[2], ref[2])):
        err = rel_fro(a, b) if fp32 else np.max(np.abs(a - b))
        assert err <= max(1e-4 if fp32 else 1e-6, 10 * sa[m]), (what, m, err, sa[m])


def oracle_spread(dims, inds, vals, start, ref, rel):
    """How far the oracle's result moves when the values and the start are perturbed by `rel`
    (relative, seeded): |dfit|, the largest relative change of lambda, and per factor the change
    in the measure the parity test uses (relative Frobenius for rel >= 1e-7, else max entry)."""
    rng = np.random.default_rng(9)
    v = vals * (1 + rel * rng.standard_normal(len(vals)))
    st = [x * (1 + rel * rng.standard_normal(x.shape)) for x in start]
    f, lam, A_, _ = O.cpd_nonneg(dims, inds, v, st, len(ref[3]), 0.0)
    da = [rel_fro(a, b) if rel >= 1e-7 else float(np.max(np.abs(a - b))) for a, b in zip(A_, ref[2])]
    return abs(f - ref[0]), float(np.max(np.abs(lam - ref[1]) / ref[1])), da


@pytest.mark.gpu
@pytest.mark.parametrize("layout", [KM.ONEMODE, KM.TILED, "ktile"])
def test_layouts_match_untiled(S, layout):
    """ONEMODE (every MTTKRP kind of the one CSF), a CTA-tiled stream and leaf-tiled (ktile > 0)
    streams give the untiled ALLROOT result to 1e-12 (fp64)."""
    N, R = 3, 17
    dims, inds, vals = CM.problem(N)
    start = nonneg_start(dims, R, seed=11)
    T = S.Tensor.from_coo(dims, inds, vals, ktile=-1)
    base = run(T, R, start, "float64", ITS)
    T.free()
    if layout == "ktile":
        T = S.Tensor.from_coo(dims, inds, vals, ktile=64)
    else:
        T = KM.build(S, dims, inds, vals, layout)
    got = run(T, R, start, "float64", ITS)
    T.free()
    check_well_formed(inds, vals, got, layout, False)
    assert abs(got[0] - base[0]) <= 1e-12
    assert np.allclose(got[1], base[1], rtol=1e-12, atol=0)
    for a, b in zip(got[2], base[2]):
        assert np.max(np.abs(a - b)) <= 1e-12


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
def test_planted_model_recovered(S, dtype):
    """fp64 reaches 1 - fit < 1e-6; fp32 is held to its fit resolution near 1 (1e-4, see
    splatt_b200_cpd_als_device_f32); both recover the components to a congruence of 0.999."""
    dims, inds, vals, F = planted()
    T = S.Tensor.from_coo(dims, inds, vals)
    got = run(T, 4, nonneg_start(dims, 4, 0), dtype, 60, tol=0.0 if dtype == "float32" else 1e-10)
    T.free()
    check_well_formed(inds, vals, got, f"planted {dtype}", dtype == "float32", inexact=False)
    assert 1 - got[0] < (1e-4 if dtype == "float32" else 1e-6), got[4]
    assert congruence(F, got[2]) >= 0.999


def _raw(T, R, ldm, bufs, dtype, its=ITS):
    """splatt_b200_cpd_nonneg_device / _f32 on the given buffers: (rc, fit, lambda, history)."""
    import torch
    lib = A.load()
    ptr_t = A.val_p if dtype == torch.float64 else A.f32_p
    sym = "splatt_b200_cpd_nonneg_device" + ("" if dtype == torch.float64 else "_f32")
    ptrs = (ptr_t * len(bufs))(*[C.cast(C.c_void_p(b.data_ptr()), ptr_t) for b in bufs])
    o = S_opts(its)
    lam = np.zeros(max(R, 1))
    hist = np.full(its, np.nan)
    fit, n = C.c_double(), C.c_int()
    torch.cuda.synchronize()
    rc = getattr(lib, sym)(T.h, R, ldm, o.ctypes.data_as(C.POINTER(C.c_double)), ptrs,
                           lam.ctypes.data_as(A.val_p), C.byref(fit), C.byref(n),
                           hist.ctypes.data_as(A.val_p), C.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return rc, fit.value, lam[:R], hist[:n.value]


def S_opts(its):
    import splatt_b200 as S
    o = S.default_opts()
    o[A.OPTION_NITER], o[A.OPTION_TOLERANCE], o[A.OPTION_VERBOSITY] = its, 0.0, 0
    return o


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("R", [5, 7, 17, 35, 67])
def test_pad_columns_untouched_and_unread(S, R, dtype):
    """NaN in columns [R, ldm) of every factor: the pads stay bit-identical and the result is
    that of a run with ldm = rpad and zero pads (within the atomics' rounding: 1e-12 in fp64,
    the fp32 bars in fp32).  Odd ranks put a pad column inside the last pair / float4 of the
    register-tiled sweep, and R = 67 runs the generic one."""
    import torch
    dt = getattr(torch, dtype)
    dims, inds, vals = CM.problem(3)
    init = nonneg_start(dims, R, seed=R)
    rpad = R + (R & 1) if dt == torch.float64 else (R + 3) & ~3
    T = S.Tensor.from_coo(dims, inds, vals)
    out = []
    for ldm, fill in ((rpad, 0.0), (rpad + 4, float("nan"))):
        bufs = [torch.full((d, ldm), fill, dtype=dt, device="cuda") for d in dims]
        for b, a in zip(bufs, init):
            b[:, :R] = torch.from_numpy(a).to("cuda", dt)
        rc, fit, lam, hist = _raw(T, R, ldm, bufs, dt)
        assert rc == A.SPLATT_SUCCESS and len(hist) == ITS
        out.append((fit, lam, bufs))
    T.free()
    ity = torch.int64 if dt == torch.float64 else torch.int32
    nan_bits = torch.full((1,), float("nan"), dtype=dt).view(ity).item()
    for b in out[1][2]:
        assert bool((b[:, R:].contiguous().view(ity) == nan_bits).all())
    bar = 1e-12 if dt == torch.float64 else 1e-4
    assert abs(out[0][0] - out[1][0]) <= (1e-12 if dt == torch.float64 else 1e-6)
    assert np.allclose(out[0][1], out[1][1], rtol=bar, atol=0)
    for a, b in zip(out[0][2], out[1][2]):
        assert rel_fro(b[:, :R].double().cpu().numpy(), a[:, :R].double().cpu().numpy()) <= bar


@pytest.mark.gpu
def test_bad_input_rejected_untouched(S):
    """A negative, NaN or Inf start entry, a zero start column, R = 0 or 129, a bad ldm, a
    misaligned factor and a shard: BADINPUT, and the factors are left bit-identical."""
    import torch
    dims, inds, vals = CM.problem(3)
    T = S.Tensor.from_coo(dims, inds, vals)
    R = 6

    def call(tensor, R, ldm, dtype, poison=None, shift=0):
        bufs = [torch.rand(d * ldm + 8, dtype=dtype, device="cuda") for d in dims]
        if poison is not None:
            poison(bufs)
        views = [b[shift:shift + d * ldm].view(d, ldm) for b, d in zip(bufs, dims)]
        saved = [b.clone() for b in bufs]
        rc, *_ = _raw(tensor, R, ldm, views, dtype)
        assert rc == A.SPLATT_ERROR_BADINPUT, (R, ldm, dtype, shift)
        for b, s in zip(bufs, saved):
            assert torch.equal(b.view(torch.uint8), s.view(torch.uint8))

    def entry(m, i, c, x, ldm):
        def f(bufs):
            bufs[m][i * ldm + c] = x
        return f

    def zero_column(m, c, ldm):
        def f(bufs):
            bufs[m][:dims[m] * ldm].view(dims[m], ldm)[:, c] = 0.0
        return f

    for dtype, ldm in ((torch.float64, 6), (torch.float32, 8)):
        tiny = -1e-300 if dtype == torch.float64 else -1e-30      # negative, not -0 in fp32
        for x in (tiny, float("nan"), float("inf"), -float("inf")):
            call(T, R, ldm, dtype, entry(1, dims[1] - 1, R - 1, x, ldm))
            call(T, R, ldm, dtype, entry(0, 0, 0, x, ldm))
        call(T, R, ldm, dtype, zero_column(2, 3, ldm))
        call(T, 0, ldm, dtype)
    call(T, 129, 130, torch.float64)
    call(T, 129, 132, torch.float32)
    call(T, 5, 5, torch.float64)                  # odd ldm
    call(T, 6, 6, torch.float32)                  # fp32 ldm not a multiple of 4
    call(T, 6, 4, torch.float32)                  # fp32 ldm < rpad4
    call(T, 6, 6, torch.float64, shift=1)         # not 16-byte aligned
    call(T, 6, 8, torch.float32, shift=2)
    T.free()
    shard = S.Tensor.from_coo(dims, inds, vals, shard_rank=0, shard_count=2)
    call(shard, 6, 6, torch.float64)
    call(shard, 6, 8, torch.float32)
    shard.free()


@pytest.mark.gpu
def test_python_rules(S):
    """ValueError for mixed or unsupported dtypes, a wrong shape, a host tensor and a wrong number
    of factors; the caller's factors are never written; the default start is seeded."""
    import torch
    dims, inds, vals = CM.problem(3)
    T = S.Tensor.from_coo(dims, inds, vals)
    good = [torch.rand((d, 4), dtype=torch.float32, device="cuda") for d in dims]
    saved = [g.clone() for g in good]
    for bad in ([good[0], good[1].double(), good[2]], [good[0], good[1][:, :3], good[2]],
                [good[0], good[1].cpu(), good[2]], good[:2]):
        with pytest.raises(ValueError):
            T.cpd_nonneg(4, bad, niters=1)
    with pytest.raises(ValueError):
        T.cpd_nonneg(4, good, dtype=torch.float64, niters=1)
    with pytest.raises(ValueError):
        T.cpd_nonneg(4, dtype=torch.float16, niters=1)
    fit, lam, fac, its, hist = T.cpd_nonneg(4, good, niters=2)
    assert its == 2 and fac[0].dtype == torch.float32 and hist.shape == (2,)
    for g, s in zip(good, saved):
        assert torch.equal(g, s)
    a = T.cpd_nonneg(4, niters=2, seed=5)
    b = T.cpd_nonneg(4, niters=2, seed=5)
    assert a[0] == b[0] or abs(a[0] - b[0]) < 1e-12
    assert np.all(np.asarray([bool((f >= 0).all()) for f in a[2]]))
    T.free()
