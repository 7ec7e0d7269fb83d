"""CPD-ALS on a device-resident tensor (splatt_b200_cpd_als_device / _f32, Tensor.cpd_als) and
the fp32 dense ALS tail (splatt_b200_als_tail_*_f32).

Precision contract of the fp32 path: factors and M1 are stored in fp32 and the MTTKRP is
splatt_b200_mttkrp_f32; Grams, the normal matrix, its Cholesky factor / pseudo-inverse, lambda,
the fit's inner product and the fit are fp64; a row is solved in fp64 from its fp32 values and
rounded once; column scaling is done in fp64 and rounded once.
"""
import ctypes as C
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

from splatt_b200 import _abi as A

U32 = 2.0 ** -24
U64 = 2.0 ** -53
ROOT = Path(__file__).resolve().parent.parent
NEW_SYMBOLS = ["splatt_b200_als_tail_gram_f32", "splatt_b200_als_tail_update_f32",
               "splatt_b200_als_tail_fit_f32", "splatt_b200_cpd_als_device",
               "splatt_b200_cpd_als_device_f32"]
# the problems of test_gpu_parity.test_cpd_als_tracks_reference
SPECS = [((60, 50, 40), 6000, 6), ((30, 25, 20, 15), 5000, 5), ((200, 150, 100), 30000, 16)]


# ---------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------
def test_new_symbols_declared_and_exported():
    hdr = (ROOT / "include" / "splatt_b200.h").read_text()
    lib = A.load()
    for name in NEW_SYMBOLS:
        assert re.search(rf"\b{name}\s*\(", hdr), name
        assert name in A.EXPORTS, name
        assert getattr(lib, name).restype is C.c_int, name


_TAIL = re.compile(r"\d(k_(?:gram_syrk|gram|solve_rows_reg|solve_rows|colnorm|scale_cols|inner))"
                   r"I(?:Li(\d+)E)?([fd])EE")


def _tail_kernel_resources():
    """{(kernel, RT, 'f' | 'd'): (registers, stack)} of the templated ALS tail kernels."""
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not Path(tool).exists():
        pytest.skip("cuobjdump not found")
    txt = subprocess.run([tool, "-res-usage", str(A.LIB_PATH)], capture_output=True, text=True,
                         check=True).stdout
    out, cur = {}, None
    for line in txt.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            k = _TAIL.search(m.group(1))
            cur = (k.group(1), int(k.group(2) or 0), k.group(3)) if k else None
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+)", line)
        if m and cur is not None:
            out[cur] = (int(m.group(1)), int(m.group(2)))
            cur = None
    return out


def test_f32_tail_kernels_within_f64_registers():
    """CPU: every fp32 instance of the tail kernels holds no more registers than its fp64
    counterpart and no more stack.  The stack of k_gram is its per-thread arrays (no spill, in
    both); k_solve_rows_reg<64> holds a 64-entry fp64 row in registers and spills in both
    precisions (ptxas -v, CUDA 12.9: fp64 88 B, fp32 72 B).  Every other instance has no stack."""
    A.load()
    res = _tail_kernel_resources()
    f32 = {k: v for k, v in res.items() if k[2] == "f"}
    assert len(f32) == 11, sorted(f32)          # 5 kernels + 3 k_solve_rows_reg + 3 k_gram_syrk
    for k, (reg, stack) in f32.items():
        ref_reg, ref_stack = res[k[:2] + ("d",)]
        assert reg <= ref_reg, f"fp32 {k}: {reg} registers, fp64 {ref_reg}"
        assert stack <= ref_stack, f"fp32 {k}: {stack} B stack, fp64 {ref_stack}"
        if k[0] not in ("k_gram", "k_solve_rows_reg") or k[1] in (16, 32):
            assert stack == 0, f"fp32 {k}: {stack} B stack"


# ---------------------------------------------------------------------------------------
# GPU helpers
# ---------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def S():
    import splatt_b200
    return splatt_b200


def _problem(spec):
    from tests.util import cover_all_slices, random_coo
    dims, inds, vals = random_coo(spec[0], spec[1], seed=3)
    return cover_all_slices(dims, inds, vals)


def _libc_start(dims, R, seed):
    from tests.test_gpu_parity import _libc_rand_factors
    return _libc_rand_factors(dims, R, seed)


def _run(T, R, start, dtype, niters, tol=0.0):
    """(fit, lambda, factors (numpy fp64), iterations, launches)"""
    import torch
    import splatt_b200 as S
    init = [torch.from_numpy(np.asarray(a)).to("cuda", getattr(torch, dtype)) for a in start]
    before = S.launch_count()
    fit, lam, fac, its = T.cpd_als(R, init, niters=niters, tol=tol)
    torch.cuda.synchronize()
    return fit, lam, [f.double().cpu().numpy() for f in fac], its, S.launch_count() - before


def _rel_fro(a, b):
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


# ---------------------------------------------------------------------------------------
# The device entries
# ---------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("spec", SPECS)
def test_fp64_entry_matches_reference_and_splatt_cpd_als(S, spec, monkeypatch):
    """fp64 device entry from the reference's start: the reference's fit, lambda and factors
    (the tolerances of test_cpd_als_tracks_reference), and per iteration the same number of
    launches as splatt_cpd_als."""
    from oracle import restate
    monkeypatch.delenv("SPLATT_B200_HOST_SOLVE", raising=False)
    dims, inds, vals = _problem(spec)
    R, seed, its = spec[2], 7, 8
    fit_ref, lam_ref, fac_ref = restate.cpd_als(dims, inds, vals, R, its, 0.0, seed)
    T = S.Tensor.from_coo(dims, inds, vals)
    fit, lam, fac, n, _ = _run(T, R, _libc_start(dims, R, seed), "float64", its)
    assert n == its
    assert abs(fit - fit_ref) < 1e-8
    assert np.allclose(lam, lam_ref, rtol=1e-6, atol=1e-9)
    for a, b in zip(fac, fac_ref):
        assert np.allclose(a, b, rtol=1e-5, atol=1e-8)
    # launches per iteration: (2 iterations) - (1 iteration), for both entries
    o = S.default_opts()
    o[0], o[1], o[4] = 1, 0.0, 0
    csf = S.csf_alloc(dims, inds, vals, o)
    per_it = []
    for k in (1, 2):
        o[3] = k
        b = S.launch_count()
        S.cpd_als(csf.ptr, R, o, seed=seed)
        per_it.append(S.launch_count() - b)
    start = _libc_start(dims, R, seed)
    dev = [_run(T, R, start, "float64", k)[4] for k in (1, 2)]
    assert dev[1] - dev[0] == per_it[1] - per_it[0]


@pytest.mark.gpu
@pytest.mark.parametrize("spec", SPECS)
def test_fp32_trajectory_tracks_fp64(S, spec):
    """fp32 entry from the same start, rounded: after 1, 2, 4 and 8 iterations the fit is within
    1e-6 of the fp64 entry's (a CPU emulation of the contract gives at most 3.6e-9 on these
    problems, so the bound has a margin of ~300x), the normalised factors within relative
    Frobenius 1e-4, and the fp32 run launches as many kernels as the fp64 one."""
    dims, inds, vals = _problem(spec)
    R = spec[2]
    start = _libc_start(dims, R, 7)
    T = S.Tensor.from_coo(dims, inds, vals)
    for its in (1, 2, 4, 8):
        f64 = _run(T, R, start, "float64", its)
        f32 = _run(T, R, start, "float32", its)
        assert f32[3] == f64[3] == its
        assert abs(f32[0] - f64[0]) <= 1e-6, (its, f32[0], f64[0])
        assert f32[4] == f64[4], (its, f32[4], f64[4])
        if its == 8:
            assert np.allclose(f32[1], f64[1], rtol=1e-4)
            for a, b in zip(f32[2], f64[2]):
                assert _rel_fro(a, b) <= 1e-4


@pytest.mark.gpu
def test_fp32_pseudo_inverse_fallback(S):
    """The singular normal matrix of test_cpd_als_rank_deficient_falls_back (rank 5 > dims[0] = 3):
    the fp32 entry takes the pseudo-inverse path, gives a finite fit and lambda, and tracks the
    fp64 entry to 1e-6."""
    from tests.util import cover_all_slices, random_coo
    dims, inds, vals = random_coo((3, 40, 30), 600, seed=9)
    dims, inds, vals = cover_all_slices(dims, inds, vals)
    T = S.Tensor.from_coo(dims, inds, vals)
    start = _libc_start(dims, 5, 2)
    f64 = _run(T, 5, start, "float64", 3)
    f32 = _run(T, 5, start, "float32", 3)
    assert np.isfinite(f32[0]) and np.all(np.isfinite(f32[1]))
    assert abs(f32[0] - f64[0]) <= 1e-6


@pytest.mark.gpu
def test_fp32_planted_rank3(S):
    """Dense 30^3 tensor of exact rank 3, 30 iterations: the fp32 factors match the fp64 ones to
    relative Frobenius 1e-4, and the fp32 fit is within 1e-3 of the fp64 fit.  Near an exact fit
    the fit 1 - sqrt(||X||^2 + ||K||^2 - 2<X,K>) / ||X|| resolves no better than about
    sqrt(2 eps) for a relative error eps in <X,K>, and <X,K> is formed from the fp32 M1 (rounding
    of sums of 900 products per entry: eps ~ 30 u32, sqrt(2 eps) ~ 2e-3).  Measured on an H100:
    fp64 reaches fit 1.0 exactly, fp32 0.99989 (|dfit| 1.1e-4; the issue's emulation with numpy
    float32 accumulation gave 6.8e-6)."""
    rng = np.random.default_rng(5)
    U = [rng.standard_normal((30, 3)) for _ in range(3)]
    X = np.einsum("ir,jr,kr->ijk", *U)
    idx = np.nonzero(np.ones_like(X))
    inds = [i.astype(np.uint64) for i in idx]
    T = S.Tensor.from_coo([30] * 3, inds, X[idx])
    start = [rng.uniform(-3, 3, (30, 3)) for _ in range(3)]
    f64 = _run(T, 3, start, "float64", 30)
    f32 = _run(T, 3, start, "float32", 30)
    for a, b in zip(f32[2], f64[2]):
        assert _rel_fro(a, b) <= 1e-4
    assert abs(f32[0] - f64[0]) <= 1e-3, (f32[0], f64[0])


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["asgiven", "cta_tiled"])
def test_fp32_layouts(S, layout, monkeypatch):
    """The fp32 loop through other MTTKRP kernels: ASGIVEN (internal and leaf kernels) and a
    CTA-tiled 3-mode stream (fp32 runs the leaf-tiled generic kernel there).  Fits agree with
    fp64 to 1e-6."""
    from tests.util import cover_all_slices, random_coo
    R = 16
    if layout == "asgiven":
        dims, inds, vals = _problem(SPECS[1])
        T = S.Tensor.from_coo(dims, inds, vals, layout=A.LAYOUT_ASGIVEN)
        kinds = {T.mode_info(m, R)["kind"] for m in range(len(dims))}
        assert kinds != {"root"}, kinds
    else:
        dims, inds, vals = random_coo((400, 300, 2000), 60000, seed=4)
        dims, inds, vals = cover_all_slices(dims, inds, vals)
        monkeypatch.setenv("SPLATT_B200_TILED", "2")
        monkeypatch.setenv("SPLATT_B200_TILE_ROWS", "256")
        T = S.Tensor.from_coo(dims, inds, vals, ncolumns_hint=R)
        monkeypatch.delenv("SPLATT_B200_TILED")
        monkeypatch.delenv("SPLATT_B200_TILE_ROWS")
    start = [np.random.default_rng(m).uniform(-3, 3, (d, R)) for m, d in enumerate(dims)]
    f64 = _run(T, R, start, "float64", 6)
    f32 = _run(T, R, start, "float32", 6)
    assert abs(f32[0] - f64[0]) <= 1e-6, (f32[0], f64[0])


@pytest.mark.gpu
def test_bad_input_rejected_untouched(S):
    """Odd / misaligned / too small ldm, R in {0, 129}, a shard, a NULL factor: BADINPUT, nothing
    enqueued, factors byte-identical.  Mixed or unsupported dtypes from Python: ValueError."""
    import torch
    dims, inds, vals = _problem(SPECS[0])
    T = S.Tensor.from_coo(dims, inds, vals)
    lib = A.load()
    o = S.default_opts()
    o[A.OPTION_NITER] = 2

    def call(tensor, R, ldm, dtype, shift=0, null=False):
        bufs = [torch.randn(d * ldm + 8, dtype=dtype, device="cuda") for d in dims]
        views = [b[shift:shift + d * ldm] for b, d in zip(bufs, dims)]
        saved = [b.clone() for b in bufs]
        ptr_t = A.val_p if dtype == torch.float64 else A.f32_p
        ptrs = (ptr_t * 3)(*[ptr_t() if null and m == 1 else C.cast(C.c_void_p(v.data_ptr()), ptr_t)
                             for m, v in enumerate(views)])
        sym = "splatt_b200_cpd_als_device" if dtype == torch.float64 else "splatt_b200_cpd_als_device_f32"
        lam = np.zeros(max(R, 1))
        fit, its = C.c_double(), C.c_int()
        rc = getattr(lib, sym)(tensor.h, R, ldm, o.ctypes.data_as(C.POINTER(C.c_double)), ptrs,
                               lam.ctypes.data_as(A.val_p), C.byref(fit), C.byref(its), None)
        torch.cuda.synchronize()
        assert rc == A.SPLATT_ERROR_BADINPUT, (R, ldm, dtype, shift)
        for b, s in zip(bufs, saved):
            assert torch.equal(b.view(torch.uint8), s.view(torch.uint8))

    call(T, 5, 5, torch.float64)                 # odd ldm
    call(T, 6, 6, torch.float64, shift=1)        # rows not 16-byte aligned
    call(T, 6, 6, torch.float32)                 # fp32 ldm not a multiple of 4
    call(T, 6, 4, torch.float32)                 # fp32 ldm < rpad4
    call(T, 6, 8, torch.float32, shift=2)        # fp32 base not 16-byte aligned
    call(T, 0, 8, torch.float64)
    call(T, 129, 130, torch.float64)
    call(T, 129, 132, torch.float32)
    call(T, 6, 8, torch.float32, null=True)
    shard = S.Tensor.from_coo(dims, inds, vals, shard_rank=0, shard_count=2)
    call(shard, 6, 6, torch.float64)
    call(shard, 6, 8, torch.float32)
    # the library rejects a good call's arguments only where they are bad: sanity
    good = [torch.randn(d, 6, dtype=torch.float32, device="cuda") for d in dims]
    saved = [g.clone() for g in good]
    with pytest.raises(ValueError):
        T.cpd_als(6, [good[0], good[1].double(), good[2]], niters=1)
    with pytest.raises(ValueError):
        T.cpd_als(6, good, dtype=torch.float64, niters=1)
    with pytest.raises(ValueError):
        T.cpd_als(6, dtype=torch.float16, niters=1)
    for g, s in zip(good, saved):
        assert torch.equal(g, s)
    fit, lam, fac, its = T.cpd_als(6, good, niters=1)
    assert its == 1 and np.isfinite(fit) and fac[0].dtype == torch.float32
    for g, s in zip(good, saved):
        assert torch.equal(g, s)                 # the caller's factors are copied, not written


@pytest.mark.gpu
def test_default_start_and_tolerance(S):
    """factors=None draws a seeded start: the same seed gives the same result, another seed a
    different one.  (Same result up to rounding: ||X||^2, the Grams and lambda are sums of fp64
    atomics whose order differs between runs.)  tol stops early; the returned factors are
    2-normalised."""
    dims, inds, vals = _problem(SPECS[0])
    T = S.Tensor.from_coo(dims, inds, vals)
    a = T.cpd_als(6, seed=3, niters=4, tol=0.0)
    b = T.cpd_als(6, seed=3, niters=4, tol=0.0)
    d = T.cpd_als(6, seed=4, niters=4, tol=0.0)
    assert a[3] == b[3] == d[3] == 4
    assert abs(a[0] - b[0]) <= 1e-12
    for fa, fb, fd in zip(a[2], b[2], d[2]):
        fa, fb, fd = (f.double().cpu().numpy() for f in (fa, fb, fd))
        assert _rel_fro(fb, fa) <= 1e-10
        assert _rel_fro(fd, fa) > 1e-2
    for f in a[2]:
        assert np.allclose(f.double().norm(dim=0).cpu().numpy(), 1.0, rtol=1e-12)
    c = T.cpd_als(6, seed=3, niters=50, tol=1e-1)
    assert 2 <= c[3] < 50


# ---------------------------------------------------------------------------------------
# One fp32 tail step against a torch fp64 oracle that rounds where the contract rounds
# ---------------------------------------------------------------------------------------
class _Tail:
    def __init__(self, N, R, ldm):
        import torch
        self.lib = A.load()
        self.h = C.c_void_p()
        s = torch.cuda.current_stream().cuda_stream
        assert self.lib.splatt_b200_als_tail_create(N, R, ldm, C.c_void_p(s), C.byref(self.h)) \
            == A.SPLATT_SUCCESS

    def __del__(self):
        self.lib.splatt_b200_als_tail_free(self.h)


def _fp(t):
    return C.cast(C.c_void_p(t.data_ptr()), A.f32_p)


@pytest.mark.gpu
@pytest.mark.parametrize("rows", [1000, 40000])
@pytest.mark.parametrize("first", [1, 0])
@pytest.mark.parametrize("generic", ["0", "1"])
@pytest.mark.parametrize("R", [1, 5, 16, 17, 32, 63, 64, 65, 100, 128])
def test_f32_tail_step_bounds(S, R, generic, first, rows, monkeypatch):
    """Grams (tail_gram_f32), one update (tail_update_f32) and the fit (tail_fit_f32) on given
    fp32 factors and an fp32 M1 whose pad columns hold NaN.
    Update: every entry satisfies |got - ref| <= 4 u32 |ref| + 8 R kappa(V) u64 ||row||: the solve
    result and the scaled value are each rounded to fp32 once (an ulp apart in the worst case
    when the fp64 results differ in their last bits), plus the fp64 solve's own error.  The
    factor's pad columns keep their NaN.  Grams and fit: within 1e-10 of the fp64 oracle (an fp32
    accumulation of the Grams or the inner product would miss it by orders of magnitude).
    Rows below and above 32768, the switch to the register-tiled SYRK."""
    import torch
    monkeypatch.setenv("SPLATT_B200_TAIL_GENERIC", generic)
    N, ldm = 3, (R + 3) & ~3
    ldm += 4 if R % 3 == 0 else 0                  # some cases with columns past rpad4
    dims = [rows, 700, 900]
    g = torch.Generator(device="cuda").manual_seed(R * 7 + first)
    nan = float("nan")

    def mat(d):
        x = torch.full((d, ldm), nan, dtype=torch.float32, device="cuda")
        x[:, :R] = torch.randn((d, R), generator=g, device="cuda", dtype=torch.float32)
        return x
    F = [mat(d) for d in dims]
    M1 = mat(rows)
    t = _Tail(N, R, ldm)
    lib = t.lib
    for m in range(N):
        assert lib.splatt_b200_als_tail_gram_f32(t.h, m, _fp(F[m]), dims[m]) == A.SPLATT_SUCCESS
    # update mode 0
    X = F[0].clone()
    assert lib.splatt_b200_als_tail_update_f32(t.h, 0, _fp(M1), _fp(X), rows, first) == A.SPLATT_SUCCESS
    torch.cuda.synchronize()
    Fd = [f[:, :R].double() for f in F]
    G = [f.T @ f for f in Fd]
    V = G[1] * G[2]
    Y = torch.linalg.solve(V, M1[:, :R].double().T).T      # rows of M1 V^-1, fp64
    Y32 = Y.float().double()                                # stored in fp32 once
    if first:
        lam = torch.sqrt((Y32 * Y32).sum(0))
    else:
        lam = torch.clamp(Y32.max(0).values, min=0.0).clamp(min=1.0)
    ref = Y32 / lam
    got = X[:, :R].double()
    kappa = float(torch.linalg.cond(V))
    rown = ref.norm(dim=1, keepdim=True)
    bound = 4 * U32 * ref.abs() + 8 * R * kappa * U64 * rown
    err = (got - ref).abs()
    assert bool((err <= bound).all()), (float((err / bound).max()), kappa)
    assert bool(torch.isnan(X[:, R:]).all()), "pad columns of the factor were written"
    # fit after the update: Grams of F1, F2 and of the new X, lambda of this update
    Xd = got
    G[0] = Xd.T @ Xd
    lam_c = np.zeros(R)
    fit = C.c_double()
    AV = G[0] * G[1] * G[2]
    inner0 = float(((Xd * M1[:, :R].double()).sum(0) * lam).sum())
    knorm0 = float(abs((AV * torch.outer(lam, lam)).sum()))
    ttnormsq = knorm0 + 2.0 * abs(inner0) + 1.0            # residual well away from 0
    assert lib.splatt_b200_als_tail_fit_f32(t.h, _fp(X), _fp(M1), rows, ttnormsq, C.byref(fit),
                                            lam_c.ctypes.data_as(A.val_p)) == A.SPLATT_SUCCESS
    lam_d = torch.from_numpy(lam_c).cuda()                  # the device's lambda of this update
    inner = float(((Xd * M1[:, :R].double()).sum(0) * lam_d).sum())
    knorm = float(abs((AV * torch.outer(lam_d, lam_d)).sum()))
    resid = ttnormsq + knorm - 2 * inner
    fit_ref = 1 - (np.sqrt(resid) if resid > 0 else resid) / np.sqrt(ttnormsq)
    assert abs(fit.value - fit_ref) <= 1e-10, (fit.value, fit_ref)


@pytest.mark.gpu
def test_f32_tail_rejects_unaligned_handle(S):
    """A handle whose ldm is not a multiple of 4 rejects the fp32 entries (fp32 rows would not
    be 16-byte aligned)."""
    import torch
    t = _Tail(3, 6, 6)
    x = torch.zeros((10, 8), dtype=torch.float32, device="cuda")
    lib = t.lib
    assert lib.splatt_b200_als_tail_gram_f32(t.h, 0, _fp(x), 10) == A.SPLATT_ERROR_BADINPUT
    assert lib.splatt_b200_als_tail_update_f32(t.h, 0, _fp(x), _fp(x), 10, 1) == A.SPLATT_ERROR_BADINPUT
    f = C.c_double()
    assert lib.splatt_b200_als_tail_fit_f32(t.h, _fp(x), _fp(x), 10, 1.0, C.byref(f), None) \
        == A.SPLATT_ERROR_BADINPUT


@pytest.mark.gpu
def test_config2_fp32_tracks_fp64(S):
    """Config 2 at full size (10K^3, 10 M nonzeros, rank 32, bench.py's generator): after 5
    iterations |fit32 - fit64| <= 1e-6."""
    import torch
    import bench
    dims = [10_000] * 3
    ind, vals = bench.make_coo_gpu(10_000_000, torch.device("cuda"), dims=dims, seed=1)
    T = S.Tensor.from_coo(dims, ind, vals)
    del ind, vals
    g = torch.Generator(device="cuda").manual_seed(11)
    start = [torch.empty((d, 32), dtype=torch.float64, device="cuda").uniform_(-3, 3, generator=g)
             for d in dims]
    fit64, _, _, n64 = T.cpd_als(32, start, niters=5, tol=0.0)
    fit32, _, _, n32 = T.cpd_als(32, [s.float() for s in start], niters=5, tol=0.0)
    assert n64 == n32 == 5
    assert abs(fit32 - fit64) <= 1e-6, (fit32, fit64)
