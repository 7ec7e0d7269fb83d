"""Tensor completion by row-wise ALS (splatt_b200_tc_als_device / Tensor.complete) and the model
SSE (splatt_b200_tensor_sse / Tensor.sse) against the numpy restatement in oracle/tc.py.

CPU: the oracle against an independent least-squares formulation and a hand-checked case; the
case table reaches every mode count, rank tier and kernel path; the new kernels do not spill.
GPU: one sweep per (N, rank tier), the boundary-slot and leaf-tiled paths, the iteration history,
a planted low-rank model, the SSE, input rules and pad columns.
"""
import ctypes as C
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

from oracle import tc as O
from splatt_b200 import _abi as A
from tests.util import random_coo, rel_fro

TIERS = {1: 16, 3: 16, 16: 16, 17: 32, 32: 32, 64: 64}     # rank -> padded-rank tier of the kernel

# (name, nmodes, rank, path): path "slots" = whole slices solved in the row-update kernel and cut
# slices through the boundary slots; "skew" = one row spanning many ranges; "cta" / "ktile" =
# leaf-tiled streams (per-row packs)
CASES = ([(f"sweep_n{n}_r{r}", n, r, "slots") for n in range(2, 9) for r in TIERS] +
         [("skew_r17", 3, 17, "skew"), ("skew_r5", 4, 5, "skew"),
          ("cta_r16", 3, 16, "cta"), ("cta_r33", 3, 33, "cta"), ("ktile_r8", 3, 8, "ktile")])

DIMS = {2: (70, 90), 3: (40, 30, 50), 4: (14, 12, 16, 10), 5: (9, 8, 10, 7, 6),
        6: (6, 7, 5, 8, 6, 5), 7: (5, 6, 4, 5, 6, 4, 5), 8: (5, 6, 5, 5, 6, 5, 5, 5)}


def problem(dims, nnz, seed):
    """Coordinates with empty first, last and middle rows in every mode, 30 duplicated
    coordinates, and many rows with fewer observations than the rank."""
    rng = np.random.default_rng(seed)
    inds = []
    for d in dims:
        allowed = np.setdiff1d(np.arange(d), [0, d - 1, d // 2])
        inds.append(rng.choice(allowed, size=nnz).astype(np.uint64))
    dup = rng.integers(0, nnz, size=30)
    inds = [np.concatenate([i, i[dup]]) for i in inds]
    vals = rng.uniform(0.0, 1.0, size=nnz + 30)
    return list(dims), inds, vals


def start(dims, R, seed=7):
    rng = np.random.default_rng(seed)
    return [rng.uniform(0.0, 1.0, size=(d, R)) for d in dims]


# ---------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------
def test_oracle_matches_lstsq():
    """Per row, the regularised normal equations solved by np.linalg.solve equal the
    least-squares solution of the stacked system [H; sqrt(reg) I] u = [v; 0]."""
    dims, inds, vals = problem((9, 7, 8), 200, seed=3)
    R, reg = 4, 0.3
    f = start(dims, R)
    for m in range(3):
        got = O.update_mode(dims, inds, vals, f, m, reg)
        for i, (H, v) in enumerate(O.row_systems(dims, inds, vals, f, m)):
            Hs = np.vstack([H, np.sqrt(reg) * np.eye(R)])
            vs = np.concatenate([v, np.zeros(R)])
            want = np.linalg.lstsq(Hs, vs, rcond=None)[0] if len(v) else np.zeros(R)
            np.testing.assert_allclose(got[i], want, rtol=0, atol=1e-12)


def test_oracle_hand_checked_two_modes():
    """2 x 2 matrix, rank 1, entries (0,0)=2, (0,1)=4, (1,1)=3, U_1 = [1, 2], reg = 1:
    row 0 of U_0 = (1*2 + 2*4) / (1 + 4 + 1) = 10/6; row 1 = 2*3 / (4 + 1) = 6/5.
    Then U_1 from the new U_0: row 0 = (10/6 * 2) / ((10/6)^2 + 1), row 1 =
    (10/6 * 4 + 6/5 * 3) / ((10/6)^2 + (6/5)^2 + 1)."""
    dims = [2, 2]
    inds = [np.array([0, 0, 1], np.uint64), np.array([0, 1, 1], np.uint64)]
    vals = np.array([2.0, 4.0, 3.0])
    f = [np.zeros((2, 1)), np.array([[1.0], [2.0]])]
    u0, u1 = O.sweep(dims, inds, vals, f, 1.0)
    a, b = 10 / 6, 6 / 5
    np.testing.assert_allclose(u0[:, 0], [a, b], rtol=1e-15)
    np.testing.assert_allclose(u1[:, 0], [2 * a / (a * a + 1), (4 * a + 3 * b) / (a * a + b * b + 1)],
                               rtol=1e-15)
    L = O.objective(inds, vals, [u0, u1], 1.0)
    x = np.array([u0[0, 0] * u1[0, 0], u0[0, 0] * u1[1, 0], u0[1, 0] * u1[1, 0]])
    assert abs(L - (((vals - x) ** 2).sum() + (u0 ** 2).sum() + (u1 ** 2).sum())) < 1e-14


def test_case_table_reaches_every_path():
    """Every N in 2..8 meets every rank tier (and the tier boundaries 16/17), and the table has
    the skewed boundary-slot case, both leaf-tiled stream kinds and the SSE tests below."""
    seen = {(n, TIERS[r]) for _, n, r, p in CASES if p == "slots"}
    assert seen == {(n, t) for n in range(2, 9) for t in (16, 32, 64)}
    assert {r for _, _, r, p in CASES if p == "slots"} >= {1, 3, 16, 17, 32, 64}
    assert {p for *_, p in CASES} == {"slots", "skew", "cta", "ktile"}
    assert {"test_sse_matches_numpy", "test_sse_scores_cpd_result"} <= set(globals())


def test_tc_symbols_declared():
    hdr = (Path(__file__).resolve().parent.parent / "include" / "splatt_b200.h").read_text()
    for name in ("splatt_b200_tensor_sse", "splatt_b200_tc_als_device"):
        assert f"int {name}(" in hdr and name in A.EXPORTS


def test_tc_kernels_do_not_spill():
    """Every row-update, solve, SSE and norm kernel of the built library uses no stack or local
    memory, and the row-update kernels fit the CTAs per SM they are compiled for."""
    A.load()
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not Path(tool).exists():
        pytest.skip("cuobjdump not found")
    txt = subprocess.run([tool, "-res-usage", str(A.LIB_PATH)], capture_output=True, text=True,
                         check=True).stdout
    found, cur = {}, None
    for line in txt.splitlines():
        m = re.search(r"Function (\S*k_tc_\w+?)(I\S*)?:", line)
        if m:
            cur = m.group(0)
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+) .*LOCAL:(\d+)", line)
        if m and cur:
            found[cur] = tuple(int(x) for x in m.groups())
            cur = None
    upd = {k: v for k, v in found.items() if "k_tc_update" in k}
    assert len(upd) == 7 * 3 * 2, len(upd)
    assert sum("k_tc_sse" in k for k in found) == 7 and sum("k_tc_solve" in k for k in found) == 3
    for k, (reg, stack, local) in found.items():
        assert stack == 0 and local == 0, f"{k} spills"
    for k, (reg, _, _) in upd.items():
        tier = int(re.search(r"ILi\d+ELi(\d+)E", k).group(1))
        assert reg <= (128 if tier <= 32 else 255), (k, reg)


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


def _build(S, path, n, seed):
    """(dims, inds, vals, Tensor) of one case."""
    if path in ("slots",):
        dims, inds, vals = problem(DIMS[n], {2: 2500, 3: 3000}.get(n, 2500), seed)
        return dims, inds, vals, S.Tensor.from_coo(dims, inds, vals)
    if path == "skew":
        dims = (300, 200, 150) if n == 3 else (60, 50, 40, 30)
        dims, inds, vals = random_coo(dims, 40000, seed=seed, unique=False, skew=[1.4] + [0] * (n - 1))
        return dims, inds, vals, S.Tensor.from_coo(dims, inds, vals)
    raise AssertionError(path)


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
@pytest.mark.parametrize("name,n,R,path", [c for c in CASES if c[3] in ("slots", "skew")],
                         ids=[c[0] for c in CASES if c[3] in ("slots", "skew")])
def test_one_sweep_matches_oracle(S, name, n, R, path):
    """One iteration from the same start equals oracle.tc.sweep to 1e-10 relative Frobenius per
    mode (empty rows, duplicates, rows with fewer observations than R; "skew": the hottest row
    spans many ranges and is assembled from boundary slots)."""
    dims, inds, vals, T = _build(S, path, n, seed=n * 100 + R)
    if path == "skew":
        hot = np.bincount(inds[0].astype(np.int64)).max()
        assert hot > 64 * 40, hot                          # spans many 64-record chunks
    reg = 0.05
    f0 = start(dims, R)
    want = O.sweep(dims, inds, vals, f0, reg)
    hist, got, its = T.complete(R, _cuda(f0), reg=reg, niters=1)
    assert its == 1
    for m in range(n):
        err = rel_fro(got[m].cpu().numpy(), want[m])
        assert err < 1e-10, (name, m, err)
    for i in range(n):
        assert not np.any(got[i].cpu().numpy()[[0, dims[i] - 1]]) or path == "skew"
    T.free()


@pytest.mark.gpu
@pytest.mark.parametrize("R", [16, 33])
def test_cta_tiled_and_ktile_streams_match_untiled(S, monkeypatch, R):
    """A CTA-tiled 3-mode stream (per-row packs) and an L1 leaf-tiled one (ktile > 0) give the
    factors of the untiled build (ktile = -1), and both match the oracle."""
    dims, inds, vals = random_coo((300, 200, 2000), 60000, seed=5, unique=False)
    f0 = start(dims, R)
    reg = 0.1
    U = S.Tensor.from_coo(dims, inds, vals, ktile=-1)
    _, base, _ = U.complete(R, _cuda(f0), reg=reg, niters=1)
    want = O.sweep(dims, inds, vals, f0, reg)
    for path in ("cta", "ktile"):
        T = _tiled(S, monkeypatch, dims, inds, vals, path, R)
        _, got, _ = T.complete(R, _cuda(f0), reg=reg, niters=1)
        for m in range(3):
            assert rel_fro(got[m].cpu().numpy(), base[m].cpu().numpy()) < 1e-12, (path, m)
            assert rel_fro(got[m].cpu().numpy(), want[m]) < 1e-10, (path, m)
        T.free()


@pytest.mark.gpu
def test_history_matches_oracle(S):
    """Five iterations: (objective, train RMSE, validation RMSE) per iteration to 1e-9."""
    dims, inds, vals = problem((40, 30, 50), 6000, seed=11)
    cut = len(vals) * 9 // 10
    tr = [i[:cut] for i in inds], vals[:cut]
    va = [i[cut:] for i in inds], vals[cut:]
    R, reg = 8, 0.2
    T = S.Tensor.from_coo(dims, *tr)
    V = S.Tensor.from_coo(dims, *va)
    f0 = start(dims, R)
    hist, got, its = T.complete(R, _cuda(f0), validate=V, reg=reg, niters=5, tol=0.0)
    want, wf = O.tc_als(dims, tr[0], tr[1], f0, reg, 5, 0.0, validate=va)
    assert its == 5 and hist.shape == (5, 3)
    np.testing.assert_allclose(hist, want, rtol=1e-9)
    hist2, _, _ = T.complete(R, _cuda(f0), reg=reg, niters=2, tol=0.0)
    assert np.isnan(hist2[:, 2]).all()
    np.testing.assert_allclose(hist2[:, :2], want[:2, :2], rtol=1e-9)


@pytest.mark.gpu
def test_planted_model_recovered(S):
    """An exact rank-4 3-mode tensor, 20 % of its entries observed and 5 % held out: after at
    most 30 iterations the validation RMSE is below 1e-3 of the held-out values' RMS."""
    rng = np.random.default_rng(0)
    dims, R = (60, 50, 40), 4
    F = [rng.standard_normal(size=(d, R)) for d in dims]
    cells = rng.permutation(np.prod(dims))
    ntr, nva = int(0.20 * len(cells)), int(0.05 * len(cells))
    def coo(c):
        idx = np.unravel_index(c, dims)
        inds = [i.astype(np.uint64) for i in idx]
        return inds, O.model_values(inds, F)
    tr, va = coo(cells[:ntr]), coo(cells[ntr:ntr + nva])
    T = S.Tensor.from_coo(list(dims), *tr)
    V = S.Tensor.from_coo(list(dims), *va)
    f0 = [np.random.default_rng(4).standard_normal((d, R)) for d in dims]
    hist, _, its = T.complete(R, _cuda(f0), validate=V, reg=1e-9, niters=30, tol=0.0)
    rms = np.sqrt(np.mean(va[1] ** 2))
    assert hist[-1, 2] < 1e-3 * rms, (hist[-1], rms, its)


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["allroot", "asgiven"])
def test_sse_matches_numpy(S, layout):
    """SSE with and without lambda, N = 3 and 5, odd rank with NaN in the pad column."""
    import torch
    for dims, R in (((30, 20, 40), 7), ((9, 8, 10, 7, 6), 12)):
        dims, inds, vals = problem(dims, 3000, seed=R)
        lay = A.LAYOUT_ALLROOT if layout == "allroot" else A.LAYOUT_ASGIVEN
        T = S.Tensor.from_coo(dims, inds, vals, layout=lay)
        f = [np.random.default_rng(m).uniform(-1, 1, (d, R)) for m, d in enumerate(dims)]
        lam = np.linspace(0.5, 2.0, R)
        for lm in (None, lam):
            got = T.sse(_cuda(f), lm)
            want = O.sse(inds, vals, f, lm)
            assert abs(got - want) <= 1e-11 * want, (layout, dims, got, want)
        # the raw entry with NaN pad columns
        ldm = R + 3 if (R + 3) % 2 == 0 else R + 4
        bufs = [torch.full((d, ldm), float("nan"), dtype=torch.float64, device="cuda") for d in dims]
        for b, x in zip(bufs, f):
            b[:, :R].copy_(torch.from_numpy(x))
        ptrs = (A.val_p * len(dims))(*[C.cast(C.c_void_p(b.data_ptr()), A.val_p) for b in bufs])
        out = C.c_double()
        assert T.lib.splatt_b200_tensor_sse(T.h, R, ldm, ptrs, None, C.byref(out), None) == A.SPLATT_SUCCESS
        assert abs(out.value - O.sse(inds, vals, f)) <= 1e-11 * out.value
        T.free()


@pytest.mark.gpu
def test_sse_scores_cpd_result(S):
    """Tensor.sse of a Tensor.cpd_als result is ||X - K||^2 at the nonzeros."""
    dims, inds, vals = random_coo((30, 40, 20), 4000, seed=2)
    T = S.Tensor.from_coo(dims, inds, vals)
    fit, lam, facs, _ = T.cpd_als(6, niters=5, seed=3)
    f = [x.cpu().numpy() for x in facs]
    got = T.sse(facs, lam)
    want = O.sse(inds, vals, f, lam)
    assert abs(got - want) <= 1e-10 * want


def _raw(S, T, R, ldm, opts, bufs, validate=None):
    import torch
    torch.cuda.synchronize()
    ptrs = (A.val_p * len(bufs))(*[C.cast(C.c_void_p(b.data_ptr()), A.val_p) for b in bufs])
    hist = np.zeros(3 * 4)
    its = C.c_int()
    rc = T.lib.splatt_b200_tc_als_device(T.h, None if validate is None else validate.h, R, ldm,
                                         opts.ctypes.data_as(C.POINTER(C.c_double)), ptrs,
                                         hist.ctypes.data_as(C.POINTER(C.c_double)), C.byref(its),
                                         None)
    torch.cuda.synchronize()
    return rc, hist


@pytest.mark.gpu
def test_bad_input_rejected_and_pad_columns(S):
    """Every input rule returns BADINPUT with the factors bit-identical; NaN pad columns stay
    bit-identical and do not change the result."""
    import torch
    dims, inds, vals = problem((20, 15, 18), 1500, seed=4)
    R = 5
    T = S.Tensor.from_coo(dims, inds, vals)
    o = S.default_opts()
    o[A.OPTION_NITER] = 2
    o[A.OPTION_TOLERANCE] = 0.0
    o[A.OPTION_REGULARIZE] = 0.1
    f0 = start(dims, R)

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

    for ldm in (5, 4):                                           # odd, < R
        b = bufs(6)
        rc, _ = _raw(S, T, R, ldm, o, b)
        check_bad(rc, b, 6)
    for r in (0, 65):
        b = bufs(66)
        rc, _ = _raw(S, T, r, 66, o, b)
        check_bad(rc, b, 66)
    for reg in (0.0, -1.0, float("nan"), float("inf")):
        oo = o.copy()
        oo[A.OPTION_REGULARIZE] = reg
        b = bufs(6)
        rc, _ = _raw(S, T, R, 6, oo, b)
        check_bad(rc, b, 6)
    # misaligned factor
    big = torch.zeros(dims[0] * 6 + 1, dtype=torch.float64, device="cuda")
    b = bufs(6)
    b0 = big[1:].view(dims[0], 6)
    b0.copy_(b[0])
    rc, _ = _raw(S, T, R, 6, o, [b0] + b[1:])
    assert rc == A.SPLATT_ERROR_BADINPUT
    # validation tensor of another shape, ASGIVEN, a shard
    V = S.Tensor.from_coo([d + 1 for d in dims], inds, vals)
    b = bufs(6)
    rc, _ = _raw(S, T, R, 6, o, b, validate=V)
    check_bad(rc, b, 6)
    for bad in (S.Tensor.from_coo(dims, inds, vals, layout=A.LAYOUT_ASGIVEN), T.shard(0, 2)):
        b = bufs(6)
        rc, _ = _raw(S, bad, R, 6, o, b)
        check_bad(rc, b, 6)
        bad.free()
    # pad columns: NaN in [R, ldm) changes nothing and stays bit-identical
    b_nan, b_zero = bufs(8), bufs(8, 0.0)
    pad_before = [x[:, R:].clone() for x in b_nan]
    rc1, h1 = _raw(S, T, R, 8, o, b_nan)
    rc2, h2 = _raw(S, T, R, 8, o, b_zero)
    assert rc1 == rc2 == A.SPLATT_SUCCESS
    np.testing.assert_allclose(h1, h2, rtol=1e-13)          # sums reduced with atomics
    for x, y, p in zip(b_nan, b_zero, pad_before):
        assert torch.equal(x[:, :R], y[:, :R])
        assert torch.equal(x[:, R:].view(torch.int64), p.view(torch.int64))


@pytest.mark.gpu
def test_python_rules(S):
    import torch
    dims, inds, vals = problem((20, 15, 18), 1500, seed=4)
    T = S.Tensor.from_coo(dims, inds, vals)
    f32 = [torch.rand((d, 4), dtype=torch.float32, device="cuda") for d in dims]
    with pytest.raises(ValueError):
        T.complete(4, f32, reg=0.1)
    with pytest.raises(ValueError):
        T.complete(4, [torch.rand((d, 5), dtype=torch.float64, device="cuda") for d in dims], reg=0.1)
    with pytest.raises(ValueError):
        T.complete(4, [torch.rand((d, 4), dtype=torch.float64) for d in dims], reg=0.1)
    with pytest.raises(ValueError):
        T.sse(f32)
    with pytest.raises(ValueError):
        T.sse([torch.rand((d, 4), dtype=torch.float64) for d in dims])
    with pytest.raises(S.SplattError):
        T.complete(4, reg=0.0)
    # the default start is seeded: two runs give bitwise the same factors (the row solves are
    # deterministic; the history's sums are reduced with atomics and may differ in the last bits)
    h1, f1, _ = T.complete(4, reg=0.1, niters=2, seed=9)
    h2, f2, _ = T.complete(4, reg=0.1, niters=2, seed=9)
    assert all(torch.equal(a, b) for a, b in zip(f1, f2))
    np.testing.assert_allclose(h1, h2, rtol=1e-13)
