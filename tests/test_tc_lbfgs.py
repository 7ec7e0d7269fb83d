"""Tensor completion by whole-model L-BFGS (splatt_b200_tc_lbfgs_device / Tensor.complete_lbfgs)
and its line-search root finder (splatt_b200_poly_argmin) against the numpy restatement in
oracle/tc_lbfgs.py.

CPU: the oracle's gradient against torch.autograd, its line coefficients against direct
evaluations, its two-loop direction against a dense BFGS inverse, the library's root finder
against the oracle's and a dense grid, planted recovery by the oracle, the declarations and the
new kernels' register use.
GPU: one iteration per (N, rank), five iterations with a wrapping ring, leaf-tiled streams,
bitwise reproducibility, ring-wrapping tensors at scale, the history, the stop rules, planted
recovery against ALS, input rules and pad columns.
"""
import ctypes as C
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

from oracle import tc as T0
from oracle import tc_lbfgs as O
from splatt_b200 import _abi as A
from tests.util import random_coo, rel_fro

RANKS = (1, 3, 16, 17, 32, 33, 64)
DIMS = {2: (70, 90), 3: (40, 30, 50), 4: (14, 12, 16, 10), 5: (9, 8, 10, 7, 6),
        6: (6, 7, 5, 8, 6, 5), 7: (5, 6, 4, 5, 6, 4, 5), 8: (5, 6, 5, 5, 6, 5, 5, 5)}


def problem(dims, nnz, seed):
    """Coordinates with empty first, last and middle rows in every mode and 30 duplicated
    coordinates (as tests/test_tc_als.py builds them)."""
    rng = np.random.default_rng(seed)
    inds = []
    for d in dims:
        allowed = np.setdiff1d(np.arange(d), [0, d - 1, d // 2])
        inds.append(rng.choice(allowed, size=nnz).astype(np.uint64))
    dup = rng.integers(0, nnz, size=30)
    inds = [np.concatenate([i, i[dup]]) for i in inds]
    vals = rng.uniform(0.0, 1.0, size=nnz + 30)
    return list(dims), inds, vals


def start(dims, R, seed=7, scale=1.0):
    rng = np.random.default_rng(seed)
    return [scale * rng.uniform(0.0, 1.0, size=(d, R)) for d in dims]


def _argmin_c(c):
    lib = A.load()
    c = np.ascontiguousarray(c, dtype=np.float64)
    a, d = C.c_double(), C.c_double()
    rc = lib.splatt_b200_poly_argmin(len(c) - 1, c.ctypes.data_as(A.val_p), C.byref(a), C.byref(d))
    assert rc == A.SPLATT_SUCCESS
    return a.value, d.value


# ---------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("reg", [0.0, 0.3])
def test_oracle_gradient_matches_autograd(reg):
    """The vectorised gradient equals torch.autograd's of the objective (fp64, CPU) to 1e-12,
    with empty rows, duplicate coordinates and reg = 0."""
    torch = pytest.importorskip("torch")
    for dims in ((9, 7, 8), (5, 6, 4, 5)):
        dims, inds, vals = problem(dims, 150, seed=len(dims))
        f = start(dims, 4, scale=0.8)
        got = O.gradient(dims, inds, vals, f, reg)
        U = [torch.tensor(x, requires_grad=True) for x in f]
        idx = [torch.from_numpy(i.astype(np.int64)) for i in inds]
        prod = torch.ones((len(vals), 4), dtype=torch.float64)
        for m, W in enumerate(U):
            prod = prod * W[idx[m]]
        L = ((torch.from_numpy(vals) - prod.sum(1)) ** 2).sum() + reg * sum((W * W).sum() for W in U)
        L.backward()
        for m in range(len(dims)):
            want = U[m].grad.numpy()
            assert np.abs(got[m] - want).max() <= 1e-12 * max(1.0, np.abs(want).max()), m
            for i in (0, dims[m] - 1, dims[m] // 2):       # empty rows: 2 reg U
                np.testing.assert_allclose(got[m][i], 2 * reg * f[m][i], rtol=0, atol=1e-15)


def test_oracle_line_coefficients_match_direct_evaluation():
    """phi(a) from the coefficients equals L(U + a D) evaluated directly at random a."""
    rng = np.random.default_rng(1)
    for N in (2, 3, 5):
        dims, inds, vals = problem(DIMS[N][:N] if N > 2 else (12, 9), 300, seed=N)
        f = start(dims, 3)
        D = [rng.standard_normal(U.shape) for U in f]
        reg = 0.2
        c, cd = O.line_coefs(inds, vals, f, D, reg)
        assert len(c) == 2 * N + 1
        for a in rng.uniform(-1.5, 1.5, size=12):
            want = T0.objective(inds, vals, [U + a * W for U, W in zip(f, D)], reg)
            got = np.polyval(c[::-1], a)
            assert abs(got - want) <= 1e-12 * abs(want), (N, a, got, want)


def test_oracle_two_loop_matches_dense_bfgs():
    """The two-loop direction equals -H g with H built explicitly by the BFGS inverse update from
    H0 = gamma I over the same pairs."""
    rng = np.random.default_rng(2)
    n = 12
    A_ = rng.standard_normal((n, n))
    Hs = A_ @ A_.T + n * np.eye(n)                        # a convex quadratic: s.y > 0
    pairs = []
    for _ in range(4):
        s = rng.standard_normal(n)
        pairs.append((s, Hs @ s))
    g = rng.standard_normal(n)
    s, y = pairs[-1]
    H = (s @ y) / (y @ y) * np.eye(n)
    for s, y in pairs:
        rho = 1.0 / (s @ y)
        V = np.eye(n) - rho * np.outer(y, s)
        H = V.T @ H @ V + rho * np.outer(s, s)
    np.testing.assert_allclose(O.two_loop(g, pairs), -H @ g, rtol=1e-12, atol=1e-12)
    np.testing.assert_array_equal(O.two_loop(g, []), -g)


def test_poly_argmin_matches_oracle_and_grid():
    """On 3000 random line polynomials of degree 2N <= 16 that are bounded below on [0, inf)
    (sums of squares plus a nonnegative quadratic, as the objective's are), the library's
    decrease is at least the oracle's and a 4001-point grid's on [0, B], and equals the decrease
    evaluated at its alpha; plus hand cases: a double root of phi', a minimiser at 0, phi' = 0,
    and a non-convex phi whose global minimum is not its first stationary point."""
    rng = np.random.default_rng(3)
    for t in range(3000):
        N = int(rng.integers(1, 9))
        c = np.zeros(2 * N + 1)
        for _ in range(int(rng.integers(1, 4))):
            e = rng.standard_normal(N + 1) * 10.0 ** rng.uniform(-3, 1)
            c += np.convolve(e, e)
        if rng.random() < 0.5:
            u, d = rng.standard_normal(5), rng.standard_normal(5)
            reg = rng.uniform(0, 1)
            c[0] += reg * u @ u
            c[1] += 2 * reg * u @ d
            c[2] += reg * d @ d
        a, dec = _argmin_c(c)
        ao, deco = O.poly_argmin(c)
        # the rounding of a decrease evaluated at x is about eps * sum_j |c_j| x^j
        mag = lambda x: sum(abs(v) * x ** j for j, v in enumerate(c))   # noqa: E731
        assert a >= 0.0 and dec >= 0.0
        assert abs(dec - O.decrease(c, a)) <= 1e-13 * mag(a), t
        assert dec >= deco - 1e-12 * max(mag(a), mag(ao)), (t, a, dec, ao, deco)
        dp = np.array([j * c[j] for j in range(1, len(c))])
        B = 1.0 + np.max(np.abs(dp[:-1] / dp[-1])) if len(dp) > 1 else 1.0
        grid = np.linspace(0.0, min(B, 1e6), 4001)
        gx = max(grid, key=lambda x: O.decrease(c, x))
        assert dec >= O.decrease(c, gx) - 1e-12 * max(mag(a), mag(gx)), (t, a, dec, gx)
    # phi' = 4 (a - 1)^2 (a - 2): the double root at 1 is not a minimiser, 2 is
    c = np.array([0.0, -8.0, 10.0, -16.0 / 3.0, 1.0])
    a, dec = _argmin_c(c)
    assert abs(a - 2.0) <= 1e-12 and abs(dec - O.decrease(c, 2.0)) <= 1e-14
    # phi increasing on [0, inf): alpha = 0, decrease 0
    assert _argmin_c([1.0, 1.0, 1.0]) == (0.0, 0.0)
    assert _argmin_c([3.0, 0.0, 0.0, 0.0]) == (0.0, 0.0)
    # phi' = (a - 1)(a - 2)(a - 4): local minima at 1 and 4, phi(4) < phi(1)
    dp = np.polynomial.polynomial.polyfromroots([1.0, 2.0, 4.0])
    c = np.concatenate([[5.0], dp / np.arange(1, 4 + 1)])
    assert O.decrease(c, 4.0) > O.decrease(c, 1.0)
    a, dec = _argmin_c(c)
    assert abs(a - 4.0) <= 1e-12, a
    # a quadratic: the closed form
    a, dec = _argmin_c([2.0, -3.0, 0.75])
    assert abs(a - 2.0) <= 1e-15 and abs(dec - 3.0) <= 1e-15
    lib = A.load()
    x = C.c_double(7.0)
    bad = np.array([1.0, np.nan, 1.0])
    assert lib.splatt_b200_poly_argmin(2, bad.ctypes.data_as(A.val_p), C.byref(x), C.byref(x)) == \
        A.SPLATT_ERROR_BADINPUT and x.value == 7.0
    assert lib.splatt_b200_poly_argmin(17, np.ones(18).ctypes.data_as(A.val_p), C.byref(x),
                                       C.byref(x)) == A.SPLATT_ERROR_BADINPUT


def planted(dims, R, frac, noise, seed):
    """A rank-R model observed at `frac` of the cells with Gaussian noise, 10 % of the
    observations held out: (train (inds, vals), validate (inds, vals))."""
    rng = np.random.default_rng(seed)
    F = [rng.standard_normal(size=(d, R)) / R ** 0.25 for d in dims]
    cells = rng.permutation(int(np.prod(dims)))[: int(frac * np.prod(dims))]
    idx = [i.astype(np.uint64) for i in np.unravel_index(cells, dims)]
    vals = T0.model_values(idx, F) + noise * rng.standard_normal(len(cells))
    cut = len(cells) * 9 // 10
    return ([i[:cut] for i in idx], vals[:cut]), ([i[cut:] for i in idx], vals[cut:])


def test_oracle_planted_completion():
    """Planted rank-3 model with noise 0.01, 10 % held out: the oracle reaches a validation RMSE
    within 10 % of the noise level."""
    dims, noise = [30, 25, 20], 0.01
    tr, va = planted(dims, 3, 0.3, noise, seed=5)
    f0 = [np.random.default_rng(6).uniform(0, 1, (d, 3)) for d in dims]
    hist, _, _ = O.tc_lbfgs(dims, tr[0], tr[1], f0, 1e-4, 5, 400, 0.0, validate=va)
    assert hist[-1, 2] < 1.1 * noise, hist[-1]


def test_symbols_and_option_declared():
    hdr = (Path(__file__).resolve().parent.parent / "include" / "splatt_b200.h").read_text()
    for name in ("splatt_b200_tc_lbfgs_device", "splatt_b200_poly_argmin"):
        assert f"int {name}(" in hdr and name in A.EXPORTS
    assert re.search(r"int memory;.*\n\} splatt_b200_tc_lbfgs_opts;", hdr)
    assert [f for f, _ in A.TcLbfgsOpts._fields_] == ["memory"]


def test_kernels_do_not_spill():
    """Every k_tcg_ kernel of the built library uses no stack or local memory, for N = 2..8."""
    A.load()
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not Path(tool).exists():
        pytest.skip("cuobjdump not found")
    txt = subprocess.run([tool, "-res-usage", str(A.LIB_PATH)], capture_output=True, text=True,
                         check=True).stdout
    found, cur = {}, None
    for line in txt.splitlines():
        m = re.search(r"Function (\S*k_tcg_\w+?)(I\S*)?:", line)
        if m:
            cur = m.group(0)
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+) .*LOCAL:(\d+)", line)
        if m and cur:
            found[cur] = tuple(int(x) for x in m.groups())
            cur = None
    assert sum("k_tcg_grad" in k for k in found) == 7 * 2
    assert sum("k_tcg_line" in k for k in found) == 7
    assert {"k_tcg_dot", "k_tcg_axpy", "k_tcg_combine", "k_tcg_copy"} <= \
        {re.search(r"k_tcg_[a-z]+", k).group(0) for k in found}
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


def _cuda(mats):
    import torch
    return [torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in mats]


def _np(mats):
    return [x.cpu().numpy() for x in mats]


ONE = [(f"n{n}_r{r}", n, r) for n in range(2, 9) for r in RANKS] + [("skew_r17", 3, 17)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,n,R", ONE, ids=[c[0] for c in ONE])
def test_one_iteration_matches_oracle(S, name, n, R):
    """One iteration from the same start: the factors (U - alpha g, so the gradient and alpha
    together) to 1e-10 relative per mode, alpha and the history row to 1e-10.  "skew": the
    hottest row spans many ranges and is assembled from boundary slots."""
    if name.startswith("skew"):
        dims, inds, vals = random_coo((300, 200, 150), 40000, seed=3, unique=False, skew=[1.4, 0, 0])
        assert np.bincount(inds[0].astype(np.int64)).max() > 64 * 40
    else:
        dims, inds, vals = problem(DIMS[n], 2500, seed=n * 100 + R)
    T = S.Tensor.from_coo(dims, inds, vals)
    reg = 0.05
    f0 = start(dims, R, scale=0.5)
    want, wf, _ = O.tc_lbfgs(dims, inds, vals, f0, reg, 5, 1, 0.0)
    hist, got, its = T.complete_lbfgs(R, _cuda(f0), reg=reg, niters=1)
    assert its == 1 and hist.shape == (1, 5)
    assert want[0, 3] > 0
    assert abs(hist[0, 3] - want[0, 3]) <= 1e-10 * want[0, 3], (hist[0], want[0])
    for m in range(n):
        err = rel_fro(got[m].cpu().numpy(), wf[m])
        assert err < 1e-10, (name, m, err)
    np.testing.assert_allclose(hist[0, [0, 1, 4]], want[0, [0, 1, 4]], rtol=1e-10)
    T.free()


def _spread(dims, inds, vals, f0, reg, mem, its, validate=None, k=2):
    """The oracle's own relative spread in the factors under 1e-14 relative changes of the start."""
    base = O.tc_lbfgs(dims, inds, vals, f0, reg, mem, its, 0.0, validate)
    rng = np.random.default_rng(99)
    sp = 0.0
    for _ in range(k):
        fp = [U * (1 + 1e-14 * rng.standard_normal(U.shape)) for U in f0]
        _, ff, _ = O.tc_lbfgs(dims, inds, vals, fp, reg, mem, its, 0.0, validate)
        sp = max(sp, max(rel_fro(a, b) for a, b in zip(ff, base[1])))
    return base, sp


@pytest.mark.gpu
@pytest.mark.parametrize("mem", [1, 3])
@pytest.mark.parametrize("reg", [0.0, 0.1])
def test_five_iterations_match_oracle(S, mem, reg):
    """Five iterations with memory 1 and 3 (3 wraps its ring), reg 0 and 0.1: the factors and the
    history within 1e-8 or ten times the oracle's own spread under 1e-14 relative changes of the
    start.  A larger difference must come with a rounding-level s.y or decrease in the oracle."""
    dims, inds, vals = problem((40, 30, 50), 6000, seed=11)
    R = 8
    f0 = start(dims, R, scale=0.7)
    (want, wf, info), sp = _spread(dims, inds, vals, f0, reg, mem, 5)
    T = S.Tensor.from_coo(dims, inds, vals)
    hist, got, its = T.complete_lbfgs(R, _cuda(f0), reg=reg, memory=mem, niters=5, tol=0.0)
    assert its == len(want) == 5
    bar = max(1e-8, 10 * sp)
    err = max(rel_fro(a.cpu().numpy(), b) for a, b in zip(got, wf))
    herr = float(np.max(np.abs(hist[:, [0, 1, 3, 4]] - want[:, [0, 1, 3, 4]]) /
                        np.abs(want[:, [0, 1, 3, 4]])))
    if max(err, herr) > bar:
        fragile = any((x["sy"] is not None and abs(x["sy"]) < 1e-12) or
                      x["decrease"] <= 1e-13 * x["phi0"] for x in info)
        assert fragile, (err, herr, bar, info)
    assert np.all(np.diff(hist[:, 0]) < 0)
    T.free()


def _tiled(S, monkeypatch, dims, inds, vals, path, R):
    if path == "cta":
        monkeypatch.setenv("SPLATT_B200_TILED", "2")
        monkeypatch.setenv("SPLATT_B200_TILE_ROWS", "128")
        T = S.Tensor.from_coo(dims, inds, vals, ncolumns_hint=R)
        monkeypatch.delenv("SPLATT_B200_TILED")
        monkeypatch.delenv("SPLATT_B200_TILE_ROWS")
        return T
    return S.Tensor.from_coo(dims, inds, vals, ktile=64)


@pytest.mark.gpu
@pytest.mark.parametrize("R", [16, 33])
def test_tiled_streams_match_untiled(S, monkeypatch, R):
    """CTA-tiled and ktile leaf-tiled streams (gradient rows added with red.add) give the
    factors and history of the untiled build over 3 iterations, to 1e-10."""
    dims, inds, vals = random_coo((300, 200, 2000), 60000, seed=5, unique=False)
    f0 = start(dims, R, scale=0.5)
    U = S.Tensor.from_coo(dims, inds, vals, ktile=-1)
    hb, base, _ = U.complete_lbfgs(R, _cuda(f0), reg=0.1, niters=3, tol=0.0)
    for path in ("cta", "ktile"):
        T = _tiled(S, monkeypatch, dims, inds, vals, path, R)
        h, got, its = T.complete_lbfgs(R, _cuda(f0), reg=0.1, niters=3, tol=0.0)
        assert its == 3
        for m in range(3):
            assert rel_fro(got[m].cpu().numpy(), base[m].cpu().numpy()) < 1e-10, (path, m)
        np.testing.assert_allclose(h, hb, rtol=1e-10)
        T.free()
    U.free()


@pytest.mark.gpu
def test_bitwise_reproducible(S):
    """Two runs on an untiled stream give bitwise the same factors, alpha and objective."""
    import torch
    dims, inds, vals = random_coo((300, 200, 150), 40000, seed=3, unique=False, skew=[1.4, 0, 0])
    T = S.Tensor.from_coo(dims, inds, vals, ktile=-1)
    f0 = _cuda(start(dims, 24, scale=0.5))
    h1, a, _ = T.complete_lbfgs(24, f0, reg=0.01, memory=3, niters=6, tol=0.0)
    h2, b, _ = T.complete_lbfgs(24, f0, reg=0.01, memory=3, niters=6, tol=0.0)
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.int64), y.view(torch.int64))
    assert np.array_equal(h1[:, [0, 1, 3, 4]], h2[:, [0, 1, 3, 4]])
    T.free()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["n3", "n4"])
def test_one_iteration_at_scale(S, name):
    """On 6 M-record tensors that wrap every warp's record ring (n3: a Zipf row spanning hundreds
    of ranges): one iteration is bitwise the same twice; U_1 = U_0 - alpha g with g computed in
    torch from all records, and alpha matches the minimiser of a torch computation of the line
    coefficients over all records."""
    import torch
    import zlib
    from tests.test_walk_at_scale import SCALE, assert_ring_wraps, check_shape, device_coo
    dims, nnz, skew = SCALE[name]
    dims, i32, idx, vals = device_coo(dims, nnz, skew, zlib.crc32(name.encode()))
    check_shape(name, idx)
    T = S.Tensor.from_coo(dims, i32, vals, ktile=-1)
    assert_ring_wraps(T)
    R, reg = 16, 0.1
    g_ = torch.Generator(device="cuda").manual_seed(R)
    f0 = [0.5 * torch.rand((d, R), dtype=torch.float64, device="cuda", generator=g_) for d in dims]
    h1, got, its = T.complete_lbfgs(R, f0, reg=reg, niters=1)
    h2, again, _ = T.complete_lbfgs(R, f0, reg=reg, niters=1)
    assert its == 1 and np.array_equal(h1[:, [0, 1, 3, 4]], h2[:, [0, 1, 3, 4]])
    for a, b in zip(got, again):
        assert torch.equal(a.view(torch.int64), b.view(torch.int64))
    del again
    N = len(dims)
    # the gradient in torch
    xh = torch.ones((nnz, R), dtype=torch.float64, device="cuda")
    for m in range(N):
        xh *= f0[m][idx[m]]
    r = vals - xh.sum(1)
    del xh
    G = []
    for m in range(N):
        h = torch.ones((nnz, R), dtype=torch.float64, device="cuda")
        for n in range(N):
            if n != m:
                h *= f0[n][idx[n]]
        G.append(2 * reg * f0[m] - 2 * torch.zeros_like(f0[m]).index_add_(0, idx[m], r[:, None] * h))
        del h
    gn = float(torch.sqrt(sum((x * x).sum() for x in G)))
    assert abs(h1[0, 4] - gn) <= 1e-10 * gn
    # the line coefficients in torch, d = -g
    P = torch.zeros((nnz, R, N + 1), dtype=torch.float64, device="cuda")
    P[:, :, 0] = 1.0
    for m in range(N):
        u, d = f0[m][idx[m]], -G[m][idx[m]]
        Q = P * u[:, :, None]
        Q[:, :, 1:] += P[:, :, :-1] * d[:, :, None]
        P = Q
    e = -P.sum(1)
    del P, Q
    e[:, 0] += vals
    Mx = (e.T @ e).cpu().numpy()
    c = np.zeros(2 * N + 1)
    for i in range(N + 1):
        for j in range(N + 1):
            c[i + j] += Mx[i, j]
    c[0] += reg * float(sum((x * x).sum() for x in f0))
    c[1] += 2 * reg * float(sum((x * -y).sum() for x, y in zip(f0, G)))
    c[2] += reg * float(sum((y * y).sum() for y in G))
    alpha, _ = O.poly_argmin(c)
    assert abs(h1[0, 3] - alpha) <= 1e-9 * alpha, (h1[0, 3], alpha)
    for m in range(N):
        want = f0[m] - h1[0, 3] * G[m]
        err = float(torch.linalg.norm(got[m] - want) / torch.linalg.norm(want))
        assert err < 1e-10, (name, m, err)
    T.free()


@pytest.mark.gpu
def test_history_matches_sse(S):
    """Column 0 of the last row equals oracle.tc.objective of the returned factors, the training
    RMSE equals Tensor.sse's and the validation RMSE validate.sse's, every row; without
    validate the column is NaN."""
    dims, inds, vals = problem((40, 30, 50), 6000, seed=12)
    cut = len(vals) * 9 // 10
    tr = [i[:cut] for i in inds], vals[:cut]
    va = [i[cut:] for i in inds], vals[cut:]
    R, reg = 8, 0.2
    T = S.Tensor.from_coo(dims, *tr)
    V = S.Tensor.from_coo(dims, *va)
    f0 = start(dims, R, scale=0.5)
    for k in (1, 2, 4):
        hist, got, its = T.complete_lbfgs(R, _cuda(f0), validate=V, reg=reg, niters=k, tol=0.0)
        assert its == k
        f = _np(got)
        L = T0.objective(tr[0], tr[1], f, reg)
        assert abs(hist[-1, 0] - L) <= 1e-10 * L, (hist[-1, 0], L)
        assert abs(hist[-1, 1] - np.sqrt(T.sse(got) / cut)) <= 1e-9 * hist[-1, 1]
        assert abs(hist[-1, 2] - np.sqrt(V.sse(got) / (len(vals) - cut))) <= 1e-12 * hist[-1, 2]
    want, _, _ = O.tc_lbfgs(dims, tr[0], tr[1], f0, reg, 5, 4, 0.0, validate=va)
    np.testing.assert_allclose(hist[:, 2], want[:, 2], rtol=1e-8)
    h2, _, _ = T.complete_lbfgs(R, _cuda(f0), reg=reg, niters=2, tol=0.0)
    assert np.isnan(h2[:, 2]).all()


@pytest.mark.gpu
@pytest.mark.parametrize("n", range(2, 9))
def test_zero_start_stops_with_zero_gradient(S, n):
    """All-zero start factors: every h is 0, so g = 0 exactly (reg > 0 too); the run stops after
    one iteration with alpha = 0, |g| = 0 and the factors unchanged."""
    import torch
    dims, inds, vals = problem(DIMS[n], 800, seed=n)
    T = S.Tensor.from_coo(dims, inds, vals)
    f0 = [np.zeros((d, 5)) for d in dims]
    hist, got, its = T.complete_lbfgs(5, _cuda(f0), reg=0.1, niters=10)
    assert its == 1 and hist[0, 3] == 0.0 and hist[0, 4] == 0.0
    assert hist[0, 0] == pytest.approx(float(vals @ vals), rel=1e-12)
    assert all(not torch.any(x) for x in got)
    T.free()


@pytest.mark.gpu
def test_tol_and_niters_stop(S):
    """niters caps the run; a loose tol stops it early, where the oracle stops."""
    dims, inds, vals = problem((40, 30, 50), 6000, seed=13)
    T = S.Tensor.from_coo(dims, inds, vals)
    f0 = start(dims, 6, scale=0.5)
    hist, _, its = T.complete_lbfgs(6, _cuda(f0), reg=0.1, niters=7, tol=0.0)
    assert its == 7 and hist.shape == (7, 5)
    hist, _, its = T.complete_lbfgs(6, _cuda(f0), reg=0.1, niters=200, tol=1e-3)
    want, _, _ = O.tc_lbfgs(dims, inds, vals, f0, 0.1, 5, 200, 1e-3)
    assert 2 <= its < 200 and its == len(want), (its, len(want))
    dec = (hist[-2, 0] - hist[-1, 0]) / (hist[-1, 0] + (hist[-2, 0] - hist[-1, 0]))
    assert dec < 1e-3
    T.free()


@pytest.mark.gpu
def test_planted_model_against_als(S):
    """A planted rank-4 model with noise, 10 % of the observations held out: from the same start
    L-BFGS reaches a validation RMSE within 10 % of ALS's."""
    dims, noise = [80, 70, 60], 0.01
    tr, va = planted(dims, 4, 0.1, noise, seed=8)
    T = S.Tensor.from_coo(dims, *tr)
    V = S.Tensor.from_coo(dims, *va)
    f0 = _cuda([np.random.default_rng(9).uniform(0, 1, (d, 4)) for d in dims])
    ha, _, _ = T.complete(4, f0, validate=V, reg=1e-3, niters=200, tol=1e-9)
    hl, _, _ = T.complete_lbfgs(4, f0, validate=V, reg=1e-3, niters=1000, tol=1e-12)
    assert hl[-1, 2] <= 1.1 * ha[-1, 2], (hl[-1], ha[-1], len(hl), len(ha))
    assert hl[-1, 2] < 1.5 * noise


def _raw(S, T, R, ldm, opts, bufs, validate=None, memory=5, lopts=True):
    import torch
    torch.cuda.synchronize()
    ptrs = (A.val_p * len(bufs))(*[C.cast(C.c_void_p(b.data_ptr()), A.val_p) for b in bufs])
    hist = np.zeros(5 * 4)
    its = C.c_int()
    lo = A.TcLbfgsOpts(memory)
    rc = T.lib.splatt_b200_tc_lbfgs_device(T.h, None if validate is None else validate.h, R, ldm,
                                           opts.ctypes.data_as(C.POINTER(C.c_double)),
                                           C.byref(lo) if lopts else None, ptrs,
                                           hist.ctypes.data_as(C.POINTER(C.c_double)), C.byref(its),
                                           None)
    torch.cuda.synchronize()
    return rc, hist


@pytest.mark.gpu
def test_bad_input_rejected_and_pad_columns(S):
    """Every input rule returns BADINPUT with the factors bit-identical; NaN pad columns stay
    bit-identical and do not change the result; reg = 0 and lopts = NULL are accepted."""
    import torch
    dims, inds, vals = problem((20, 15, 18), 1500, seed=4)
    R = 5
    T = S.Tensor.from_coo(dims, inds, vals)
    o = S.default_opts()
    o[A.OPTION_NITER] = 2
    o[A.OPTION_TOLERANCE] = 0.0
    o[A.OPTION_REGULARIZE] = 0.1
    f0 = start(dims, R, scale=0.5)

    def bufs(ldm, fill=float("nan")):
        b = [torch.full((d, ldm), fill, dtype=torch.float64, device="cuda") for d in dims]
        for x, y in zip(b, f0):
            x[:, :R].copy_(torch.from_numpy(y))
        return b

    def check_bad(rc, b, ldm):
        assert rc == A.SPLATT_ERROR_BADINPUT
        ref = bufs(ldm)
        for x, y in zip(b, ref):
            assert torch.equal(x.view(torch.int64), y.view(torch.int64))

    for ldm in (5, 4):
        b = bufs(6)
        check_bad(_raw(S, T, R, ldm, o, b)[0], b, 6)
    for r in (0, 65):
        b = bufs(66)
        check_bad(_raw(S, T, r, 66, o, b)[0], b, 66)
    for reg in (-1.0, float("nan"), float("inf")):
        oo = o.copy()
        oo[A.OPTION_REGULARIZE] = reg
        b = bufs(6)
        check_bad(_raw(S, T, R, 6, oo, b)[0], b, 6)
    for mem in (-1, 33):
        b = bufs(6)
        check_bad(_raw(S, T, R, 6, o, b, memory=mem)[0], b, 6)
    big = torch.zeros(dims[0] * 6 + 1, dtype=torch.float64, device="cuda")
    b = bufs(6)
    b0 = big[1:].view(dims[0], 6)
    b0.copy_(b[0])
    assert _raw(S, T, R, 6, o, [b0] + b[1:])[0] == A.SPLATT_ERROR_BADINPUT
    V = S.Tensor.from_coo([d + 1 for d in dims], inds, vals)
    b = bufs(6)
    check_bad(_raw(S, T, R, 6, o, b, validate=V)[0], b, 6)
    for bad in (S.Tensor.from_coo(dims, inds, vals, layout=A.LAYOUT_ASGIVEN), T.shard(0, 2)):
        b = bufs(6)
        check_bad(_raw(S, bad, R, 6, o, b)[0], b, 6)
        bad.free()
    # reg = 0, memory 0 and 32, and the NULL options are accepted
    oo = o.copy()
    oo[A.OPTION_REGULARIZE] = 0.0
    for mem in (0, 32):
        assert _raw(S, T, R, 6, oo, bufs(6), memory=mem)[0] == A.SPLATT_SUCCESS
    assert _raw(S, T, R, 6, o, bufs(6), lopts=False)[0] == A.SPLATT_SUCCESS
    # pad columns: NaN in [R, ldm) changes nothing and stays bit-identical
    b_nan, b_zero = bufs(8), bufs(8, 0.0)
    pad_before = [x[:, R:].clone() for x in b_nan]
    rc1, h1 = _raw(S, T, R, 8, o, b_nan)
    rc2, h2 = _raw(S, T, R, 8, o, b_zero)
    assert rc1 == rc2 == A.SPLATT_SUCCESS
    np.testing.assert_array_equal(h1[:10], h2[:10])
    for x, y, p in zip(b_nan, b_zero, pad_before):
        assert torch.equal(x[:, :R], y[:, :R])
        assert torch.equal(x[:, R:].view(torch.int64), p.view(torch.int64))
    T.free()


@pytest.mark.gpu
def test_python_rules(S):
    import torch
    dims, inds, vals = problem((20, 15, 18), 1500, seed=4)
    T = S.Tensor.from_coo(dims, inds, vals)
    f32 = [torch.rand((d, 4), dtype=torch.float32, device="cuda") for d in dims]
    with pytest.raises(ValueError):
        T.complete_lbfgs(4, f32, reg=0.1)
    with pytest.raises(ValueError):
        T.complete_lbfgs(4, [torch.rand((d, 5), dtype=torch.float64, device="cuda") for d in dims], reg=0.1)
    with pytest.raises(ValueError):
        T.complete_lbfgs(4, [torch.rand((d, 4), dtype=torch.float64) for d in dims], reg=0.1)
    with pytest.raises(ValueError):
        T.complete_lbfgs(4, reg=0.1, validate="x")
    with pytest.raises(S.SplattError):
        T.complete_lbfgs(4, reg=-1.0)
    with pytest.raises(S.SplattError):
        T.complete_lbfgs(4, reg=0.1, memory=40)
    # the default start is seeded and the same draw as `complete`'s
    h1, f1, _ = T.complete_lbfgs(4, reg=0.1, niters=3, seed=9)
    h2, f2, _ = T.complete_lbfgs(4, reg=0.1, niters=3, seed=9)
    assert all(torch.equal(a, b) for a, b in zip(f1, f2))
    _, fa, _ = T.complete(4, reg=0.1, niters=0, seed=9)
    _, fb, _ = T.complete_lbfgs(4, reg=0.1, niters=0, seed=9)
    assert all(torch.equal(a, b) for a, b in zip(fa, fb))
    T.free()
