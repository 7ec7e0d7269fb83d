"""CPD-ALS at every mode count, MTTKRP kind and dense-tail tier, against the reference's iteration.

The entries: `splatt_cpd_als` with the dense tail on the device and on the host
(SPLATT_B200_HOST_SOLVE), the device-tensor entries `splatt_b200_cpd_als_device` / `_f32`, the
multi-GPU engine on a device list naming this GPU several times (no multicast mapping there, so
the whole tail runs on device 0 with the same kernels, after the peer-memory reduce) and
`parallel.cpd_als_sharded` (world 1).  CASES below names the runs; a CPU test derives what each
row reaches (entry per mode count, MTTKRP kind inside the fp64 loop, tail tier) and fails if
anything is unreached.

Oracle: `oracle.restate.cpd_als`, the restatement of the reference's cpd_als_iterate
(pinned to the compiled reference by tests/test_oracle.py), 8 iterations from its own start
(`_libc_rand_factors`).  Bars: fp64 |dfit| < 1e-8, lambda rtol 1e-6 / atol 1e-9, factors rtol
1e-5 / atol 1e-8; fp32 |dfit| <= 1e-6, lambda rtol 1e-4, relative Frobenius 1e-4 per factor.

Every problem has an empty first, last and interior slice in every mode and 40 exact
duplicate coordinates; every mode has at least 2R rows at the ranks it runs.  The reference
keeps duplicates as separate nonzeros, so ||X||^2 is the sum of v^2 over records.

Every run also checks that the returned fit describes the returned model (see model_fit), that
the returned factors have unit 2-norm columns, and that no run printed the pseudo-inverse
fallback's message: the restatement has no fallback, so such a case would compare two
different algorithms.
"""
from __future__ import annotations

import ctypes as C
import functools

import numpy as np
import pytest

from splatt_b200 import _abi as A
from tests import test_kernel_matrix as KM
from tests.util import random_coo, rel_fro

ITS, SEED = 8, 7
U32 = 2.0 ** -24
ALLROOT, ONEMODE, TILED = KM.ALLROOT, KM.ONEMODE, KM.TILED
NOT_SPD = "Gram matrix is not SPD"

# Per problem: base dims and nonzeros (each mode gets 3 more rows, left empty: KM._gapped).
# N = 3 also carries the tail tiers up to R = 128; "syrk" has a mode of 40003 rows (>= 32768,
# 40003 = 625 * 64 + 3: the SYRK's last 64-row tile is short).
PROBLEMS = {
    2: ((150, 120), 2500),
    3: ((400, 360, 330), 50000),
    4: ((40, 36, 42, 38), 6000),
    5: ((38, 40, 36, 35, 37), 6000),
    6: ((36, 38, 35, 37, 36, 35), 6000),
    7: ((36, 35, 37, 36, 35, 38, 36), 6000),
    8: ((35, 36, 37, 35, 36, 38, 35, 36), 6000),
    "syrk": ((40000, 147, 137), 150000),
}

# Entries.  Those marked F64_LOOP run the fp64 device loop (run_device_als<double> or the
# multi engine's tail) on the MTTKRP kinds of their tensor.
SPLATT, SPLATT_HOST, DEV64, DEV32 = "splatt_cpd_als", "splatt_cpd_als_host", "device_f64", "device_f32"
MULTI3, MULTI2, SHARDED = "multi_0_0_0", "multi_0_0", "sharded"
F64_LOOP = {SPLATT, DEV64, MULTI3, MULTI2, SHARDED}
SWEEP = (SPLATT, SPLATT_HOST, DEV64, DEV32, MULTI3)
SHARDED_N = (2, 5, 8)
TAIL_R = (1, 16, 17, 32, 33, 64, 65, 100, 128)

# (problem, layout, R, SPLATT_B200_TAIL_GENERIC, entries)
CASES = (
    # 1. mode-count sweep
    [(N, ALLROOT, R, "0", SWEEP + ((SHARDED,) if N in SHARDED_N else ()))
     for N in range(2, 9) for R in (5, 17)]
    # 2. MTTKRP kinds inside the loop: every depth of the one CSF, and a forced CTA-tiled stream
    + [(N, ONEMODE, 17, "0", (DEV64, DEV32)) for N in range(2, 9)]
    + [(3, TILED, 17, "0", (DEV64, DEV32))]
    # 3. tail tiers: register-tiled 16 / 32 / 64 and generic (R = 17 on the register-tiled tail
    #    is a sweep row), then the SYRK Gram
    + [(3, ALLROOT, R, g, (DEV64, SPLATT)) for R in TAIL_R for g in ("0", "1") if (R, g) != (17, "0")]
    + [("syrk", ALLROOT, R, "0", (DEV64, SPLATT, MULTI2)) for R in (16, 32, 64)]
)


def _case_id(c):
    return f"{'n' + str(c[0]) if isinstance(c[0], int) else c[0]}-{c[1]}-R{c[2]}-generic{c[3]}"


@functools.lru_cache(maxsize=None)
def problem(key):
    """(dims, inds, vals) in numpy: seeded, 40 exact duplicate coordinates, and the first,
    last and one interior slice of every mode empty."""
    base, nnz = PROBLEMS[key]
    seed = 200 + (key if isinstance(key, int) else 99)
    _, inds, vals = random_coo(base, nnz, seed=seed, unique=False)
    inds = [np.concatenate([i, i[:40]]) for i in inds]
    vals = np.concatenate([vals, vals[:40][::-1] - 0.5])
    dims, inds = KM._gapped(base, inds)
    return list(dims), inds, vals


def _tier(R, generic):
    """The dense tail's kernels at rank R.  DevTail::alloc (cpd.cu) sets
    rt = R <= 16 ? 16 : R <= 32 ? 32 : R <= 64 ? 64 : 0, and 0 under SPLATT_B200_TAIL_GENERIC=1;
    rt != 0 runs k_solve_rows_reg<rt>, rt == 0 the generic k_solve_rows / k_gram."""
    if generic == "1":
        return "generic"
    return 16 if R <= 16 else 32 if R <= 32 else 64 if R <= 64 else "generic"


def _syrk(rt, rows):
    """DevTail::gram_into (cpd.cu): k_gram_syrk<rt> for a factor of >= 32768 rows when rt != 0."""
    return rt != "generic" and rows >= 32768


def _reaches(lib, case):
    key, layout, R, generic, entries = case
    dims = KM._gapped_dims(PROBLEMS[key][0])
    N = len(dims)
    out = {("entry", N, e) for e in entries}
    if F64_LOOP & set(entries):
        out |= {("kind", N, k) for k in KM._kinds(lib, dims, layout)}
        if layout == TILED:
            out.add(("kind", N, "cta_tiled"))
        rt = _tier(R, generic)
        out |= {("tail", rt, _syrk(rt, I)) for I in dims}
    return out


def _required(lib):
    req = {("entry", N, e) for N in range(2, 9) for e in SWEEP}
    req |= {("entry", N, SHARDED) for N in SHARDED_N}
    for N in range(2, 9):
        dims = KM._gapped_dims(PROBLEMS[N][0])
        req |= {("kind", N, k) for k in set(KM._kinds(lib, dims, ONEMODE)) | {"root"}}
    req.add(("kind", 3, "cta_tiled"))
    req |= {("tail", rt, s) for rt in (16, 32, 64) for s in (False, True)}
    req.add(("tail", "generic", False))
    return req


def test_case_table_reaches_every_entry_kind_and_tier(lib):
    """CPU: the table reaches every (N, entry) for N = 2..8 (sharded at N = 2, 5, 8), every
    MTTKRP kind of every N inside the fp64 loop (root / internal / leaf of the one CSF, and the
    CTA-tiled 3-mode stream), and every tail tier (rt 16 / 32 / 64 with and without the SYRK
    Gram, and the generic kernels); every mode has at least 2R rows; no two rows are the same run."""
    assert len({_case_id(c) for c in CASES}) == len(CASES)
    req = _required(lib)
    assert {k for (t, N, k) in req if t == "kind"} >= {"root", "internal", "leaf", "cta_tiled"}
    got = set().union(*(_reaches(lib, c) for c in CASES))
    assert req - got == set(), sorted(map(str, req - got))
    for key, layout, R, generic, entries in CASES:
        assert min(KM._gapped_dims(PROBLEMS[key][0])) >= 2 * R, (key, R)


# ---------------------------------------------------------------------------------------
# Checks
# ---------------------------------------------------------------------------------------
def model_fit(inds, vals, lam, facs):
    """The fit of the model (lam, facs) to the COO tensor, in numpy fp64:
    1 - sqrt(||X||^2 + ||K||^2 - 2 <X, K>) / ||X||, where ||X||^2 = sum of v^2 over records (the
    reference's semantics: duplicates are separate nonzeros, csf_frobsq), <X, K> sums
    v * sum_r lam_r prod_m A_m[i_m, r] over records, and ||K||^2 = lam^T (*_m A_m^T A_m) lam.
    Also returns ||X||^2, sum over records of |v| sum_r |lam_r| prod_m |A_m[i_m, r]| and
    |lam|^T (*_m |A_m|^T |A_m|) |lam| (the scales of the rounding bounds)."""
    lam = np.asarray(lam, dtype=np.float64)
    prod = np.broadcast_to(lam, (len(vals), len(lam))).copy()
    aprod = np.abs(prod)
    G = np.ones((len(lam), len(lam)))
    Gabs = np.ones_like(G)
    for i, a in zip(inds, facs):
        rows = a[np.asarray(i, dtype=np.int64)]
        prod *= rows
        aprod *= np.abs(rows)
        G *= a.T @ a
        Gabs *= np.abs(a).T @ np.abs(a)
    xx = float(np.sum(vals * vals))
    inner = float(vals @ prod.sum(axis=1))
    kk = float(lam @ G @ lam)
    resid = xx + kk - 2 * inner
    resid = np.sqrt(resid) if resid > 0 else resid
    return 1 - resid / np.sqrt(xx), xx, float(np.abs(vals) @ aprod.sum(axis=1)), \
        float(np.abs(lam) @ Gabs @ np.abs(lam))


def check_model(inds, vals, fit, lam, facs, what, fp32=False, unit=True):
    """The reported fit is the fit of the returned (lambda, factors): post-processing only
    moves the column norms of the last iteration's factors into lambda.
    fp64: within 1e-10.  fp32: the reported fit was formed in fp64 from the loop's fp32 factors
    and the last mode's fp32 MTTKRP M1; the returned factors are those divided by their column
    norms in fp64 and rounded to fp32 once (relative error <= u = 2^-24 per entry), lambda
    absorbs the norms in fp64.  With rho^2 = ||X||^2 + ||K||^2 - 2<X,K>, to first order:
      <X,K>: every rank-one term of the returned model moves by <= N u (N rounded entries),
             and the loop's inner product used M1 = the fp32 MTTKRP, off by <= 2 gamma(n + N)
             of the same sum on absolute values (n: most nonzeros in a slice of the last mode,
             gamma(k) = k u / (1 - k u), the bound of tests/test_kernel_matrix.py in fp32);
             both scale with S1 = sum |v| sum_r |lam_r| prod_m |A_m[i_m, r]|;
      ||K||^2: every Gram entry moves by <= 2u of |A|^T|A|, so ||K||^2 by <= 2 N u S2 with
             S2 = |lam|^T (*_m |A_m|^T |A_m|) |lam|;
    so |rho_rep^2 - rho^2| <= E = 2 (N u + 2 gamma(n + N)) S1 + 2 N u S2, and since
    rho_rep = ||X|| (1 - fit_rep), |fit_rep - fit| <= E / ((rho_rep + rho) ||X||)."""
    got, xx, s1, s2 = model_fit(inds, vals, lam, facs)
    if not fp32:
        assert abs(fit - got) <= 1e-10, (what, fit, got)
    else:
        N = len(inds)
        n = int(np.bincount(np.asarray(inds[-1], dtype=np.int64)).max())
        k = n + N
        gamma = k * U32 / (1 - k * U32)
        E = 2 * (N * U32 + 2 * gamma) * s1 + 2 * N * U32 * s2
        nx = np.sqrt(xx)
        rho_rep, rho = nx * (1 - fit), nx * (1 - got)
        assert rho_rep > 0 and rho > 0, (what, fit, got)
        bound = E / ((rho_rep + rho) * nx)
        assert abs(fit - got) <= bound, (what, fit, got, bound)
    if unit:
        tol = 2 * U32 if fp32 else 1e-12
        for m, a in enumerate(facs):
            assert np.allclose(np.linalg.norm(a, axis=0), 1.0, rtol=tol, atol=0), (what, m)


def check_reference(got, ref, what, fp32=False):
    fit, lam, facs = got
    fit_ref, lam_ref, fac_ref = ref
    if fp32:
        assert abs(fit - fit_ref) <= 1e-6, (what, fit, fit_ref)
        assert np.allclose(lam, lam_ref, rtol=1e-4, atol=0), (what, lam, lam_ref)
        for m, (a, b) in enumerate(zip(facs, fac_ref)):
            assert rel_fro(a, b) <= 1e-4, (what, m, rel_fro(a, b))
    else:
        assert abs(fit - fit_ref) < 1e-8, (what, fit, fit_ref)
        assert np.allclose(lam, lam_ref, rtol=1e-6, atol=1e-9), (what, lam, lam_ref)
        for m, (a, b) in enumerate(zip(facs, fac_ref)):
            assert np.allclose(a, b, rtol=1e-5, atol=1e-8), (what, m, float(np.abs(a - b).max()))


def check_no_fallback(capfd, what):
    err = capfd.readouterr().err
    assert NOT_SPD not in err, f"{what}: a normal matrix fell back to the pseudo-inverse\n{err[-2000:]}"


@functools.lru_cache(maxsize=None)
def reference(key, R):
    from oracle import restate
    dims, inds, vals = problem(key)
    return restate.cpd_als(dims, inds, vals, R, ITS, 0.0, SEED)


@functools.lru_cache(maxsize=None)
def start(key, R):
    from tests.test_gpu_parity import _libc_rand_factors
    return _libc_rand_factors(problem(key)[0], R, SEED)


# ---------------------------------------------------------------------------------------
# The entries
# ---------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def S():
    import splatt_b200
    return splatt_b200


@pytest.fixture
def env(monkeypatch):
    for k in ("SPLATT_B200_HOST_SOLVE", "SPLATT_B200_TAIL_GENERIC", "SPLATT_B200_LAYOUT",
              "SPLATT_B200_DEVICES", "SPLATT_B200_NGPUS"):
        monkeypatch.delenv(k, raising=False)
    return monkeypatch


def _opts(S, its):
    o = S.default_opts()
    o[A.OPTION_NTHREADS], o[A.OPTION_NITER], o[A.OPTION_TOLERANCE], o[A.OPTION_VERBOSITY] = 1, its, 0.0, 0
    return o


def _splatt(S, key, R, host, env, its=ITS):
    """splatt_cpd_als (host CSF, factors drawn after srand(SEED)); returns (fit, lambda, factors)
    and the kernel launches it made."""
    dims, inds, vals = problem(key)
    env.setenv("SPLATT_B200_HOST_SOLVE", "1" if host else "0")
    o = _opts(S, its)
    csf = S.csf_alloc(dims, inds, vals, o)
    before = S.launch_count()
    out = S.cpd_als(csf.ptr, R, o, seed=SEED)
    launches = S.launch_count() - before
    csf.free()
    return out, launches


def _multi(S, key, R, devs):
    dims, inds, vals = problem(key)
    o = _opts(S, ITS)
    csf = S.csf_alloc(dims, inds, vals, o)
    mg = S.MultiGpu(csf.ptr, int(o[A.OPTION_CSF_ALLOC]), R, devs)
    assert mg.ndevices == len(devs) and not mg.multicast
    out = mg.cpd_als(o, seed=SEED)
    mg.free()
    csf.free()
    return out


def _device(T, key, R, dtype, its=ITS):
    """Tensor.cpd_als from the reference's start: (fit, lambda, factors (numpy fp64)) and the
    kernel launches it made."""
    from tests.test_cpd_device import _run
    fit, lam, fac, n, launches = _run(T, R, start(key, R), dtype, its)
    assert n == its
    return (fit, lam, fac), launches


def _sharded(S, T, key, R):
    """parallel.cpd_als_sharded, world 1: lambda and factors as the last iteration left them
    (not post-processed)."""
    import torch
    from splatt_b200 import parallel
    _, _, vals = problem(key)
    init = [torch.from_numpy(a).cuda() for a in start(key, R)]
    fit, lam, fac, times = parallel.cpd_als_sharded(T, R, init, float(np.sum(vals * vals)),
                                                   niters=ITS, tol=0.0)
    assert len(times) == ITS
    return fit, lam, [f.cpu().numpy() for f in fac]


def _post_process(lam, facs):
    """The reference's post-processing (src/cpd.c:391-411): 2-normalise into lambda."""
    lam = lam.copy()
    out = []
    for a in facs:
        nrm = np.linalg.norm(a, axis=0)
        lam *= nrm
        out.append(a / nrm)
    return lam, out


def _tensor(S, key, layout):
    dims, inds, vals = problem(key)
    if layout == ALLROOT:
        return S.Tensor.from_coo(dims, inds, vals)
    return KM.build(S, dims, inds, vals, layout)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_cpd_matrix(S, lib, case, env, capfd):
    """Every entry of the row against the restatement, and its returned model against its
    returned fit."""
    key, layout, R, generic, entries = case
    env.setenv("SPLATT_B200_TAIL_GENERIC", generic)
    dims, inds, vals = problem(key)
    ref = reference(key, R)
    T = None
    if {DEV64, DEV32, SHARDED} & set(entries):
        T = _tensor(S, key, layout)
        kinds = KM._kinds(lib, dims, layout)
        assert [T.mode_info(m, R)["kind"] for m in range(len(dims))] == kinds, case
        if layout == TILED:          # leaf-tile segments split nodes: the stream is the tiled one
            assert any(T.mode_info(m, 1)["nfibs"][:-1] !=
                       KM.prefix_counts(inds, T.mode_info(m, 1)["level_perm"])[:-1]
                       for m in range(len(dims))), case
    for e in entries:
        what = f"{_case_id(case)} {e}"
        fp32, unit = e == DEV32, True
        if e in (SPLATT, SPLATT_HOST):
            got, _ = _splatt(S, key, R, e == SPLATT_HOST, env)
        elif e in (DEV64, DEV32):
            got, _ = _device(T, key, R, "float32" if fp32 else "float64")
        elif e in (MULTI3, MULTI2):
            got = _multi(S, key, R, [0] * (3 if e == MULTI3 else 2))
        else:
            got = _sharded(S, T, key, R)
            unit = False
        check_model(inds, vals, *got, what, fp32=fp32, unit=unit)
        if e == SHARDED:
            got = (got[0],) + _post_process(got[1], got[2])
        check_reference(got, ref, what, fp32=fp32)
        check_no_fallback(capfd, what)
    if T is not None:
        T.free()


@pytest.mark.gpu
@pytest.mark.parametrize("N", range(2, 9))
def test_launches_per_iteration(S, N, env):
    """At every mode count the fp64 device entry launches as many kernels per iteration as
    splatt_cpd_als with the device tail (difference of 2 and 1 iterations)."""
    R = 5
    T = _tensor(S, N, ALLROOT)
    dev = [_device(T, N, R, "float64", its=k)[1] for k in (1, 2)]
    spl = [_splatt(S, N, R, False, env, its=k)[1] for k in (1, 2)]
    assert dev[1] - dev[0] == spl[1] - spl[0], (N, dev, spl)
    T.free()


# ---------------------------------------------------------------------------------------
# Columns [R, ldm) of the caller's factors
# ---------------------------------------------------------------------------------------
def _pad_run(S, T, R, ldm, dtype, init, fill, its):
    """splatt_b200_cpd_als_device / _f32 on factors of leading dimension ldm whose columns
    [R, ldm) hold `fill`: (fit, lambda, factor buffers)."""
    import torch
    lib = A.load()
    bufs = []
    for a in init:
        b = torch.full((a.shape[0], ldm), fill, dtype=dtype, device="cuda")
        b[:, :R] = torch.from_numpy(a).to("cuda", dtype)
        bufs.append(b)
    ptr_t, sym = (A.val_p, "splatt_b200_cpd_als_device") if dtype == torch.float64 else \
        (A.f32_p, "splatt_b200_cpd_als_device_f32")
    ptrs = (ptr_t * len(bufs))(*[C.cast(C.c_void_p(b.data_ptr()), ptr_t) for b in bufs])
    o = _opts(S, its)
    lam = np.zeros(R)
    fit, n = C.c_double(), C.c_int()
    rc = getattr(lib, sym)(T.h, R, ldm, o.ctypes.data_as(C.POINTER(C.c_double)), ptrs,
                           lam.ctypes.data_as(A.val_p), C.byref(fit), C.byref(n),
                           C.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    assert rc == A.SPLATT_SUCCESS and n.value == its
    return fit.value, lam, bufs


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["float64", "float32"])
@pytest.mark.parametrize("R", [5, 6, 7, 17, 35, 67])
def test_pad_columns_untouched_and_unread(S, R, dtype, env, capfd):
    """The device entries on factors with ldm = rpad + 4 (fp64) / rpad4 + 4 (fp32) and NaN in
    columns [R, ldm) of every factor give what a run with ldm = rpad / rpad4 and zero pads
    gives from the same start, and leave every pad column bit-identical NaN.  Within rounding:
    the fp64 atomics sum in a varying order (1e-12); fp32 within the fp32 bars.  R = 5, 17
    (1 mod 4), 6 (2 mod 4), 7, 35, 67 (3 mod 4): odd ranks put a pad column inside the last
    column pair (fp64) and inside the last float4 (fp32) of the register-tiled solve (R <= 64)
    and of the generic one (R = 67)."""
    import torch
    dt = getattr(torch, dtype)
    key, its = 3, 3
    rpad = R + (R & 1) if dt == torch.float64 else (R + 3) & ~3
    T = _tensor(S, key, ALLROOT)
    init = start(key, R)
    base = _pad_run(S, T, R, rpad, dt, init, 0.0, its)
    got = _pad_run(S, T, R, rpad + 4, dt, init, float("nan"), its)
    T.free()
    ity = torch.int64 if dt == torch.float64 else torch.int32
    nan_bits = torch.full((1,), float("nan"), dtype=dt).view(ity).item()
    for m, b in enumerate(got[2]):
        assert bool((b[:, R:].contiguous().view(ity) == nan_bits).all()), (R, dtype, m)
    fac0 = [b[:, :R].double().cpu().numpy() for b in base[2]]
    fac1 = [b[:, :R].double().cpu().numpy() for b in got[2]]
    bar = 1e-12 if dt == torch.float64 else 1e-4
    assert abs(got[0] - base[0]) <= (1e-12 if dt == torch.float64 else 1e-6), (got[0], base[0])
    assert np.allclose(got[1], base[1], rtol=bar, atol=0), (got[1], base[1])
    for m, (a, b) in enumerate(zip(fac1, fac0)):
        assert rel_fro(a, b) <= bar, (R, dtype, m, rel_fro(a, b))
    check_no_fallback(capfd, f"pad R{R} {dtype}")
