"""Sparse Tucker by HOOI (splatt_b200_ttmc / splatt_b200_tucker_hooi_device, Tensor.ttmc /
Tensor.tucker) against the numpy restatement in oracle/tucker.py.

CPU: the oracle's TTMc against a dense einsum; hooi_exact on an exact Tucker tensor, its core
norm ascent, hooi_power against hooi_exact; the case table; the new symbols; no spills; the SASS
of the completion, CP-APR and CPD kernels is the parent build's.
GPU: the TTMc for N = 2..8 on every stream path, reproducibility, step-exact parity with
hooi_power, planted problems, orthonormality, the reported fit, a rank-deficient mode, input
rules and pad columns.
"""
import ctypes as C
import hashlib
import json
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

from oracle import tucker as O
from splatt_b200 import _abi as A
from tests.util import random_coo

HERE = Path(__file__).resolve().parent

# (name, ranks, path): "slots" = whole slices stored and cut slices through the boundary slots;
# "skew" = one row spanning many ranges; "cta" / "ktile" = leaf-tiled streams (red.add)
CASES = [("n2_r3x5", (3, 5), "slots"), ("n2_r1x32", (1, 32), "slots"),
         ("n3_r32_c1024", (32, 32, 32), "slots"), ("n3_r1x7x4", (1, 7, 4), "slots"),
         ("n4_r2345", (2, 3, 4, 5), "slots"), ("n4_c1024", (8, 8, 16, 2), "slots"),
         ("n5_mixed", (1, 2, 3, 2, 2), "slots"), ("n6_mixed", (2, 2, 1, 3, 2, 2), "slots"),
         ("n7_mixed", (2, 1, 2, 2, 1, 2, 3), "slots"), ("n8_r2", (2,) * 8, "slots"),
         ("skew_n3", (5, 7, 3), "skew"), ("skew_n4", (3, 2, 4, 3), "skew"),
         ("cta_n3", (16, 16, 16), "cta"), ("ktile_n3", (5, 7, 9), "ktile")]

DIMS = {2: (70, 90), 3: (40, 36, 50), 4: (20, 18, 24, 12), 5: (9, 8, 10, 7, 6),
        6: (6, 7, 5, 8, 6, 5), 7: (5, 6, 4, 5, 6, 4, 5), 8: (5, 6, 5, 5, 6, 5, 5, 5)}


def problem(dims, nnz, seed):
    """Random values at random coordinates with 30 duplicated coordinates."""
    rng = np.random.default_rng(seed)
    inds = [rng.integers(0, d, size=nnz).astype(np.uint64) for d in dims]
    dup = rng.integers(0, nnz, size=30)
    inds = [np.concatenate([i, i[dup]]) for i in inds]
    vals = rng.standard_normal(nnz + 30)
    return list(dims), inds, vals


def dense(dims, inds, vals):
    X = np.zeros(dims)
    np.add.at(X, tuple(np.asarray(i, dtype=np.int64) for i in inds), vals)
    return X


def mats_for(dims, ranks, seed=3):
    rng = np.random.default_rng(seed)
    return [rng.standard_normal((d, r)) for d, r in zip(dims, ranks)]


def exact_tucker(dims, ranks, seed=0, noise=0.0):
    """A dense tensor G x U (orthonormal U, a core with a clear spectrum) plus optional noise,
    every entry stored."""
    rng = np.random.default_rng(seed)
    U = [np.linalg.qr(rng.standard_normal((d, r)))[0] for d, r in zip(dims, ranks)]
    G = rng.standard_normal(ranks) + 3.0
    X = G
    for m, u in enumerate(U):
        X = np.moveaxis(np.tensordot(u, np.moveaxis(X, m, 0), axes=(1, 0)), 0, m)
    X = X + noise * rng.standard_normal(dims)
    idx = np.indices(dims).reshape(len(dims), -1)
    return list(dims), [i.astype(np.uint64) for i in idx], X.reshape(-1), U


def projector_err(U, V):
    return np.linalg.norm(U @ U.T - V @ V.T)


# ---------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [2, 3, 4, 5])
def test_oracle_ttmc_matches_dense(N):
    dims = DIMS[N] if N < 5 else (6, 5, 7, 4, 5)
    dims, inds, vals = problem(dims, 300, seed=N)
    ranks = [2, 3, 1, 4, 2][:N]
    mats = mats_for(dims, ranks)
    X = dense(dims, inds, vals)
    letters = "abcdefgh"
    for n in range(N):
        others = [m for m in range(N) if m != n]
        spec = letters[:N] + "," + ",".join(letters[m] + letters[m].upper() for m in others) + "->" + \
            letters[n] + "".join(letters[m].upper() for m in others)
        want = np.einsum(spec, X, *[mats[m] for m in others]).reshape(dims[n], -1)
        got = O.ttmc(dims, inds, vals, mats, n, ranks)
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12)


def test_oracle_exact_tucker_recovered():
    dims, inds, vals, U = exact_tucker((12, 10, 9), (3, 2, 4))
    G, F, hist = O.hooi_exact(dims, inds, vals, (3, 2, 4), mats_for(dims, (3, 2, 4)), 10, 0.0)
    assert hist[-1, 0] >= 1 - 1e-12
    for f, u in zip(F, U):
        assert projector_err(f, u) < 1e-10


def test_oracle_core_norm_never_decreases():
    dims, inds, vals = problem((15, 12, 14), 600, seed=2)
    _, _, hist = O.hooi_exact(dims, inds, vals, (4, 3, 5), mats_for(dims, (4, 3, 5)), 10, 0.0)
    assert np.all(np.diff(hist[:, 1]) >= -1e-12 * hist[:-1, 1])


def test_oracle_power_matches_exact():
    dims, inds, vals, U = exact_tucker((14, 12, 10), (3, 4, 2), seed=5, noise=1e-2)
    f0 = mats_for(dims, (3, 4, 2))
    Ge, Fe, he = O.hooi_exact(dims, inds, vals, (3, 4, 2), f0, 6, 0.0)
    Gp, Fp, hp = O.hooi_power(dims, inds, vals, (3, 4, 2), f0, 6, 0.0, max_power=300, svd_tol=1e-13)
    for a, b in zip(Fe, Fp):
        assert projector_err(a, b) < 1e-9
    assert abs(he[-1, 0] - hp[-1, 0]) < 1e-11


def test_case_table_reaches_every_path():
    assert {len(r) for _, r, _ in CASES} == set(range(2, 9))
    assert {p for *_, p in CASES} == {"slots", "skew", "cta", "ktile"}
    cols = {int(np.prod(r)) // r[n] for _, r, _ in CASES for n in range(len(r))}
    assert 1024 in cols and 1 in cols
    assert any(len(set(r)) > 1 and any(x % 2 for x in r) for _, r, _ in CASES)


def test_tucker_symbols_declared():
    hdr = (HERE.parent / "include" / "splatt_b200.h").read_text()
    for sym in ("splatt_b200_ttmc", "splatt_b200_tucker_hooi_device"):
        assert f"int {sym}(" in hdr and sym in A.EXPORTS
    assert "} splatt_b200_tucker_opts;" in hdr
    assert [f for f, _ in A.TuckerOpts._fields_] == ["max_power", "svd_tol"]


def _res_usage():
    A.load()
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not Path(tool).exists():
        pytest.skip("cuobjdump not found")
    return tool


def test_tucker_kernels_do_not_spill():
    tool = _res_usage()
    txt = subprocess.run([tool, "-res-usage", str(A.LIB_PATH)], capture_output=True, text=True,
                         check=True).stdout
    found, cur = {}, None
    for line in txt.splitlines():
        m = re.search(r"Function (\S*tucker_cu\S*):", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+) .*LOCAL:(\d+)", line)
        if m and cur:
            found[cur] = tuple(int(x) for x in m.groups())
            cur = None
    assert sum("k_ttmcI" in k for k in found) == 7 * 3 * 2
    for name in ("k_ttmc_combine", "k_atb_part", "k_atb_fin", "k_ab", "k_chol_inv", "k_sumsq_part",
                 "k_sumsq_fin", "k_xnorm_part", "k_absmax_part", "k_absmax_fin", "k_flip_cols"):
        assert sum(f"{len(name)}{name}E" in k for k in found) == 1, name
    for k, (reg, stack, local) in found.items():
        assert stack == 0 and local == 0, f"{k} spills"


ANON = re.compile(r"_GLOBAL__N__[0-9a-f]+_\d+_\w+?_cu_[0-9a-f]+")


def test_existing_kernels_keep_their_sass():
    """The completion, CP-APR and CPD kernels that share walk.cuh / jacobi.cuh with Tucker compile
    to the SASS of the build before Tucker was added (digests in tests/golden, symbol names
    aside)."""
    tool = _res_usage()
    want = json.loads((HERE / "golden" / "sass_walk_cpd.json").read_text())
    txt = subprocess.run([tool, "-sass", str(A.LIB_PATH)], capture_output=True, text=True, check=True).stdout
    got, cur, body = {}, None, []
    for line in txt.splitlines() + ["Function : end"]:
        m = re.search(r"Function : (\S+)", line)
        if m:
            if cur is not None:
                got[ANON.sub("ANON", cur)] = hashlib.sha256("\n".join(body).encode()).hexdigest()
            cur, body = m.group(1), []
            continue
        if "/* 0x" in line:                       # an instruction or its control word
            body.append(ANON.sub("ANON", re.sub(r"/\*[0-9a-f]{4,}\*/", "", line).strip()))
    changed = [k for k, h in want.items() if got.get(k) != h]
    assert not changed, changed


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


def _np(facs):
    return [x.cpu().numpy() for x in facs]


def _build(S, monkeypatch, ranks, path, seed):
    N = len(ranks)
    if path == "slots":
        dims, inds, vals = problem(DIMS[N], 2500, seed)
        return dims, inds, vals, S.Tensor.from_coo(dims, inds, vals, ktile=-1)
    if path == "skew":
        dims = (300, 200, 150) if N == 3 else (60, 50, 40, 30)
        dims, inds, vals = random_coo(dims, 40000, seed=seed, unique=False, skew=[1.4] + [0] * (N - 1))
        return dims, inds, vals, S.Tensor.from_coo(dims, inds, vals, ktile=-1)
    dims, inds, vals = random_coo((300, 200, 2000), 60000, seed=seed, unique=False)
    if path == "cta":
        monkeypatch.setenv("SPLATT_B200_TILED", "2")
        monkeypatch.setenv("SPLATT_B200_TILE_ROWS", "128")
        T = S.Tensor.from_coo(dims, inds, vals, ncolumns_hint=16)
        monkeypatch.delenv("SPLATT_B200_TILED")
        monkeypatch.delenv("SPLATT_B200_TILE_ROWS")
    else:
        T = S.Tensor.from_coo(dims, inds, vals, ktile=64)
    return dims, inds, vals, T


def _ttmc_kernels(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return {m.group(1) for e in prof.events() for m in [re.search(r"k_ttmc<\d+, \d+, (\w+)>", e.name)] if m}


@pytest.mark.gpu
@pytest.mark.parametrize("name,ranks,path", CASES, ids=[c[0] for c in CASES])
def test_ttmc_matches_oracle(S, monkeypatch, name, ranks, path):
    """Every mode's TTMc within 2^-40 of the oracle's |X| (x) |U| bound, elementwise; on untiled
    streams bitwise reproducible; the leaf-tiled paths really ran the red.add kernel."""
    import torch
    dims, inds, vals, T = _build(S, monkeypatch, ranks, path, seed=len(ranks) * 10 + sum(ranks))
    mats = mats_for(dims, ranks)
    for n in range(len(dims)):
        want = O.ttmc(dims, inds, vals, mats, n, ranks)
        bound = O.ttmc(dims, inds, np.abs(vals), [np.abs(x) for x in mats], n, ranks)
        out = torch.empty(want.shape, dtype=torch.float64, device="cuda")
        kinds = _ttmc_kernels(lambda: T.ttmc(n, _cuda(mats), out, ranks))
        # (a profiler session after others in the same process may record no kernel names)
        assert not kinds - ({"true"} if path in ("cta", "ktile") else {"false"}), (path, kinds)
        got = out.cpu().numpy()
        assert np.all(np.abs(got - want) <= 2.0 ** -40 * bound + 1e-300), (name, n)
        if path in ("slots", "skew"):
            again = torch.empty_like(out)
            T.ttmc(n, _cuda(mats), again, ranks)
            assert torch.equal(out.view(torch.int64), again.view(torch.int64))
    T.free()


def _check_orthonormal(F):
    for f in F:
        assert np.all(np.isfinite(f))
        assert np.linalg.norm(f.T @ f - np.eye(f.shape[1])) <= 1e-12


@pytest.mark.gpu
@pytest.mark.parametrize("ranks", [(3, 4, 5), (2, 3, 2, 3), (1, 2, 2)])
def test_step_exact_parity_with_power_oracle(S, ranks):
    dims = DIMS[len(ranks)]
    dims, inds, vals = problem(dims, 3000, seed=4)
    f0 = mats_for(dims, ranks, seed=8)
    T = S.Tensor.from_coo(dims, inds, vals)
    G, F, h, its = T.tucker(ranks, _cuda(f0), niters=3, tol=0.0, max_power=4, svd_tol=0.0)
    Gw, Fw, hw = O.hooi_power(dims, inds, vals, ranks, f0, 3, 0.0, max_power=4, svd_tol=0.0)
    assert its == 3 and np.array_equal(h[:, 2], hw[:, 2])
    for a, b in zip(_np(F), Fw):
        assert np.max(np.abs(a - b)) < 1e-10
    assert np.max(np.abs(G - Gw)) < 1e-10 * max(1.0, np.abs(Gw).max())
    np.testing.assert_allclose(h[:, 0], hw[:, 0], atol=1e-10)
    _check_orthonormal(_np(F))
    # bitwise reproducible on an untiled stream
    G2, F2, h2, _ = T.tucker(ranks, _cuda(f0), niters=3, tol=0.0, max_power=4, svd_tol=0.0)
    assert np.array_equal(G, G2) and np.array_equal(h, h2)
    for a, b in zip(F, F2):
        assert np.array_equal(a.cpu().numpy().view(np.int64), b.cpu().numpy().view(np.int64))
    T.free()


@pytest.mark.gpu
def test_planted_problems(S):
    ranks = (3, 4, 2)
    dims, inds, vals, U = exact_tucker((30, 25, 20), ranks, seed=1, noise=1e-2)
    f0 = mats_for(dims, ranks, seed=2)
    T = S.Tensor.from_coo(dims, inds, vals)
    G, F, h, its = T.tucker(ranks, _cuda(f0), niters=20, tol=1e-12)
    Ge, Fe, he = O.hooi_exact(dims, inds, vals, ranks, f0, 20, 1e-12)
    for a, b in zip(_np(F), Fe):
        assert projector_err(a, b) < 1e-8
    assert abs(h[-1, 0] - he[-1, 0]) < 1e-10
    _check_orthonormal(_np(F))
    T.free()
    dims, inds, vals, U = exact_tucker((20, 18, 16, 6), (2, 3, 2, 2), seed=3)
    T = S.Tensor.from_coo(dims, inds, vals)
    G, F, h, its = T.tucker((2, 3, 2, 2), niters=10, tol=0.0)
    assert h[-1, 0] >= 1 - 1e-10
    _check_orthonormal(_np(F))
    T.free()


@pytest.mark.gpu
def test_reported_fit_matches_dense(S):
    """The history's fit equals the fit of the returned core and factors on the dense tensor
    (duplicates summed)."""
    dims, inds, vals = problem((12, 10, 9), 500, seed=6)
    ranks = (3, 2, 4)
    T = S.Tensor.from_coo(dims, inds, vals)
    G, F, h, its = T.tucker(ranks, niters=4, tol=0.0, seed=3)
    X = dense(dims, inds, vals)
    M = np.einsum("abc,ia,jb,kc->ijk", G, *_np(F))
    fit = 1 - np.linalg.norm(X - M) / np.linalg.norm(X)
    assert abs(h[-1, 0] - fit) < 1e-10
    assert abs(h[-1, 1] - np.linalg.norm(G)) < 1e-12 * np.linalg.norm(G)
    T.free()


@pytest.mark.gpu
def test_rank_deficient_mode(S):
    """Mode 0 has 2 nonempty rows but rank 4: its factor is still orthonormal, no NaN anywhere."""
    rng = np.random.default_rng(1)
    dims = [10, 12, 9]
    nnz = 400
    inds = [rng.choice([3, 7], size=nnz).astype(np.uint64),
            rng.integers(0, 12, size=nnz).astype(np.uint64), rng.integers(0, 9, size=nnz).astype(np.uint64)]
    vals = rng.standard_normal(nnz)
    T = S.Tensor.from_coo(dims, inds, vals)
    G, F, h, its = T.tucker((4, 3, 3), niters=5, tol=0.0)
    _check_orthonormal(_np(F))
    assert np.all(np.isfinite(G)) and np.all(np.isfinite(h))
    T.free()


def _raw(T, ranks, ldm, opts, bufs, topts=None):
    import torch
    torch.cuda.synchronize()
    ptrs = (A.val_p * len(bufs))(*[C.cast(C.c_void_p(b.data_ptr()), A.val_p) for b in bufs])
    core = np.zeros(max(int(np.prod(ranks)), 1))
    hist = np.zeros(4 * 4)
    its = C.c_int()
    rk = (C.c_int * len(ranks))(*ranks)
    rc = T.lib.splatt_b200_tucker_hooi_device(T.h, rk, ldm, opts.ctypes.data_as(C.POINTER(C.c_double)),
                                              None if topts is None else C.byref(topts), ptrs,
                                              core.ctypes.data_as(C.POINTER(C.c_double)),
                                              hist.ctypes.data_as(C.POINTER(C.c_double)), C.byref(its), None)
    torch.cuda.synchronize()
    return rc, core, hist


@pytest.mark.gpu
def test_bad_input_rejected_and_pad_columns(S):
    import torch
    dims, inds, vals = problem((20, 15, 18), 1500, seed=4)
    ranks = [3, 4, 5]
    T = S.Tensor.from_coo(dims, inds, vals)
    o = S.default_opts()
    o[A.OPTION_NITER] = 2
    o[A.OPTION_TOLERANCE] = 0.0
    f0 = mats_for(dims, [5, 5, 5])

    def bufs(ldm, fill=float("nan"), f=f0):
        b = [torch.full((d, ldm), fill, dtype=torch.float64, device="cuda") for d in dims]
        for x, y in zip(b, f):
            x[:, :5].copy_(torch.from_numpy(y))
        return b

    def check_bad(rc, b, ldm, f=f0):
        assert rc == A.SPLATT_ERROR_BADINPUT
        for x, y in zip(b, bufs(ldm, f=f)):
            assert torch.equal(x.view(torch.int64), y.view(torch.int64))

    for ldm in (5, 4):                                         # odd, < max rank
        b = bufs(6)
        check_bad(_raw(T, ranks, ldm, o, b)[0], b, 6)
    for rk in ([0, 4, 5], [3, 4, 33], [3, 16, 5], [1, 1, 5]):    # R < 1, R > 32, R > dims, R_n > C_n
        b = bufs(34)
        check_bad(_raw(T, rk, 34, o, b)[0], b, 34)
    for key, x in ((A.OPTION_NITER, -1.0), (A.OPTION_NITER, float("nan")), (A.OPTION_TOLERANCE, -1.0),
                   (A.OPTION_TOLERANCE, float("inf"))):
        oo = o.copy()
        oo[key] = x
        b = bufs(6)
        check_bad(_raw(T, ranks, 6, oo, b)[0], b, 6)
    for to in (A.TuckerOpts(0, 1e-10), A.TuckerOpts(5, -1.0), A.TuckerOpts(5, float("nan"))):
        b = bufs(6)
        check_bad(_raw(T, ranks, 6, o, b, to)[0], b, 6)
    f = [y.copy() for y in f0]
    f[1][:, 2] = f[1][:, 0]                                    # dependent start columns
    b = bufs(6, f=f)
    check_bad(_raw(T, ranks, 6, o, b)[0], b, 6, f=f)
    big = torch.zeros(dims[0] * 6 + 1, dtype=torch.float64, device="cuda")
    b = bufs(6)
    b0 = big[1:].view(dims[0], 6)
    b0.copy_(b[0])
    assert _raw(T, ranks, 6, o, [b0] + b[1:])[0] == A.SPLATT_ERROR_BADINPUT
    for bad in (S.Tensor.from_coo(dims, inds, vals, layout=A.LAYOUT_ASGIVEN), T.shard(0, 2)):
        b = bufs(6)
        check_bad(_raw(bad, ranks, 6, o, b)[0], b, 6)
        bad.free()
    # pad columns: NaN in [R_m, ldm) changes nothing and stays bit-identical
    b_nan, b_zero = bufs(8), bufs(8, 0.0)
    pad_before = [x[:, r:].clone() for x, r in zip(b_nan, ranks)]
    rc1, c1, h1 = _raw(T, ranks, 8, o, b_nan)
    rc2, c2, h2 = _raw(T, ranks, 8, o, b_zero)
    assert rc1 == rc2 == A.SPLATT_SUCCESS
    assert np.array_equal(c1, c2) and np.array_equal(h1, h2)
    for x, y, p, r in zip(b_nan, b_zero, pad_before, ranks):
        assert torch.equal(x[:, :r], y[:, :r])
        assert torch.equal(x[:, r:].view(torch.int64), p.view(torch.int64))
    T.free()


@pytest.mark.gpu
def test_python_rules(S):
    import torch
    dims, inds, vals = problem((20, 15, 18), 1500, seed=4)
    T = S.Tensor.from_coo(dims, inds, vals)
    with pytest.raises(ValueError):
        T.tucker((2, 2, 2), [torch.rand((d, 2), dtype=torch.float32, device="cuda") for d in dims])
    with pytest.raises(ValueError):
        T.tucker((2, 2, 2), [torch.rand((d, 3), dtype=torch.float64, device="cuda") for d in dims])
    with pytest.raises(S.SplattError):
        T.tucker((2, 2, 33))
    G1, F1, h1, i1 = T.tucker((2, 3, 2), niters=3, seed=9)
    G2, F2, h2, i2 = T.tucker((2, 3, 2), niters=3, seed=9)
    assert i1 == i2 and np.array_equal(G1, G2) and G1.shape == (2, 3, 2) and h1.shape == (i1, 4)
    T.free()
