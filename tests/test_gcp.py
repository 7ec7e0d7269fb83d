"""Generalized CP decomposition by sampled gradients and Adam (splatt_b200_gcp_device /
Tensor.gcp), its sampler and kernel primitive (splatt_b200_gcp_sample / _sampled) and the decode of
a device tensor to coordinates (splatt_b200_tensor_to_coo), against oracle/gcp.py.

CPU: Philox4x32-10 against the Random123 known-answer vectors, the oracle's objective and gradient
against torch.autograd, the estimator's exact unbiasedness, the epoch rule on scripted estimates,
the draws' ranges, the declarations and the new kernels' register use.
GPU: to_coo on every stream kind, the sampler bitwise against the oracle, the primitive within an
elementwise fp64 bound, the driver against the oracle driver, failed epochs and the stop rules,
planted recovery for every loss, and the input rules.
"""
import ctypes as C
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

from oracle import gcp as O
from splatt_b200 import _abi as A
from tests.util import random_coo, rel_fro

DIMS = {2: (70, 90), 3: (40, 30, 50), 4: (14, 12, 16, 10), 5: (9, 8, 10, 7, 6),
        6: (6, 7, 5, 8, 6, 5), 7: (5, 6, 4, 5, 6, 4, 5), 8: (5, 6, 5, 5, 6, 5, 5, 5)}
LOSSES = ("gaussian", "bernoulli-logit", "poisson-log")


def values_for(loss, n, rng):
    if loss == "gaussian":
        return rng.standard_normal(n)
    if loss == "bernoulli-logit":
        return np.ones(n)
    return rng.integers(1, 6, size=n).astype(np.float64)


def problem(dims, nnz, loss, seed, dup=20):
    """Coordinates with `dup` duplicated entries and values allowed by the loss."""
    rng = np.random.default_rng(seed)
    inds = [rng.integers(0, d, size=nnz).astype(np.uint64) for d in dims]
    pick = rng.integers(0, nnz, size=dup)
    inds = [np.concatenate([i, i[pick]]) for i in inds]
    return list(dims), inds, values_for(loss, nnz + dup, rng)


# ---------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------
def test_philox_known_answers():
    """Random123's known-answer vectors of Philox4x32-10."""
    cases = [((0, 0), (0, 0, 0, 0), "6627e8d5 e169c58d bc57ac4c 9b00dbd8"),
             ((0xffffffff,) * 2, (0xffffffff,) * 4, "408f276d 41c83b0e a20bc7c6 6d5451fd"),
             ((0xa4093822, 0x299f31d0), (0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344),
              "d16cfe09 94fdcceb 5001e420 24126ea1")]
    for key, ctr, want in cases:
        assert " ".join(f"{int(w):08x}" for w in O.philox(key, ctr)) == want


@pytest.mark.parametrize("loss", LOSSES)
def test_oracle_matches_autograd(loss):
    """The oracle's dense objective and gradient equal torch.autograd's of
    sum_all f(0, m) + sum_stored (f(x, m) - f(0, m)) over a small dense tensor, duplicates
    included."""
    torch = pytest.importorskip("torch")
    L = O.LOSS_NAMES[loss]
    dims, inds, vals = problem((4, 3, 5), 25, loss, seed=1, dup=6)
    f = [np.random.default_rng(2).normal(0, 0.6, (d, 3)) for d in dims]
    U = [torch.tensor(x, requires_grad=True) for x in f]
    M = torch.einsum("az,bz,cz->abc", *U)
    idx = [torch.from_numpy(i.astype(np.int64)) for i in inds]
    m = M[idx[0], idx[1], idx[2]]
    x = torch.from_numpy(vals)

    def ft(x, m):
        if L == O.GAUSSIAN:
            return (x - m) ** 2
        if L == O.BERNOULLI_LOGIT:
            return torch.nn.functional.softplus(m) - x * m
        return torch.exp(m) - x * m
    F = ft(0.0, M).sum() + (ft(x, m) - ft(0.0, m)).sum()
    F.backward()
    got = O.objective(L, dims, inds, vals, f)
    assert abs(got - F.item()) <= 1e-12 * abs(F.item())
    for n, G in enumerate(O.gradient(L, dims, inds, vals, f)):
        want = U[n].grad.numpy()
        assert np.abs(G - want).max() <= 1e-12 * np.abs(want).max(), n


@pytest.mark.parametrize("loss", LOSSES)
def test_estimator_is_unbiased_exactly(loss):
    """Averaging the estimator over every record position (weight nnz / 1 per draw, 1 / nnz
    probability) and every coordinate is the same as one sample holding each position and each
    coordinate once with weights 1: it gives F and grad F to 1e-12."""
    L = O.LOSS_NAMES[loss]
    dims, inds, vals = problem((3, 2, 4), 5, loss, seed=3, dup=2)
    nnz = len(vals)
    f = [np.random.default_rng(4).normal(0, 0.7, (d, 2)) for d in dims]
    coords = np.indices(dims).reshape(3, -1)
    P = coords.shape[1]
    si = [np.concatenate([np.asarray(i, dtype=np.int64), c]) for i, c in zip(inds, coords)]
    sv = np.concatenate([vals, np.zeros(P)])
    # E over one uniform draw of each kind, times the draw counts p = q = 1
    val, G = O.sampled(L, nnz, P, 1.0, 1.0, si, sv, f)
    F = O.objective(L, dims, inds, vals, f)
    assert abs(val - F) <= 1e-12 * abs(F)
    for a, b in zip(G, O.gradient(L, dims, inds, vals, f)):
        assert np.abs(a - b).max() <= 1e-12 * np.abs(b).max()


def test_epoch_rule_on_scripted_estimates():
    """Accept when finite and not above the last accepted estimate; otherwise revert and decay;
    stop after more than max_fails failures, on a small relative decrease, or after NITER."""
    def make(script):
        it = iter(script)
        log = []

        def epoch(lr):
            log.append(("run", lr))
            return next(it)
        epoch.revert = lambda: log.append(("revert",))
        return epoch, log

    ep, log = make([9.0, 11.0, float("nan"), 8.0])
    hist, n = O.run_epochs(10.0, ep, 4, 0.0, 5, 0.5, 1.0)
    assert n == 4
    np.testing.assert_array_equal(hist[:, 2], [1, 0, 0, 1])
    np.testing.assert_array_equal(hist[:, 1], [1.0, 1.0, 0.5, 0.25])
    assert [e[0] for e in log].count("revert") == 2
    # more than max_fails = 1 failures
    ep, log = make([12.0, 13.0, 1.0])
    hist, n = O.run_epochs(10.0, ep, 10, 0.0, 1, 0.1, 1.0)
    assert n == 2 and list(hist[:, 2]) == [0, 0]
    # tolerance: 9.99 is a 1e-3 relative decrease
    ep, _ = make([9.0, 8.99, 5.0])
    hist, n = O.run_epochs(10.0, ep, 10, 2e-3, 1, 0.1, 1.0)
    assert n == 2
    # NITER
    ep, _ = make([9.0, 8.0, 7.0, 6.0])
    _, n = O.run_epochs(10.0, ep, 3, 0.0, 1, 0.1, 1.0)
    assert n == 3
    # an equal estimate is accepted and counts as no decrease
    ep, _ = make([10.0])
    hist, n = O.run_epochs(10.0, ep, 5, 1e-12, 1, 0.1, 1.0)
    assert n == 1 and hist[0, 2] == 1


def test_draws_in_range():
    """mulhi64 maps every 64-bit value into [0, n), including a mode of 2^29 rows, and draws of
    different steps or purposes differ."""
    v = np.array([0, 1, 2**63, 2**64 - 1], dtype=np.uint64)
    for n in (1, 7, 2**29, 2**32 - 1):
        r = O.mulhi64(v, n)
        assert r.max() < n and r[0] == 0 and int(r[-1]) == n - 1
    c = O.draw_coords(5, 3, 1, 4000, (2**29, 3, 1))
    assert c[0].max() < 2**29 and c[0].max() > 2**28 and set(c[1]) == {0, 1, 2} and set(c[2]) == {0}
    a = O.draw_positions(5, 3, 0, 100, 1000)
    assert not np.array_equal(a, O.draw_positions(5, 4, 0, 100, 1000))
    assert not np.array_equal(a, O.draw_positions(5, 3, 2, 100, 1000))


def test_symbols_and_options_declared():
    hdr = (Path(__file__).resolve().parent.parent / "include" / "splatt_b200.h").read_text()
    for name in ("splatt_b200_tensor_to_coo", "splatt_b200_gcp_sample", "splatt_b200_gcp_sampled",
                 "splatt_b200_gcp_device"):
        assert f"int {name}(" in hdr and name in A.EXPORTS
    assert re.search(r"uint64_t seed;.*\n\} splatt_b200_gcp_opts;", hdr)
    assert [f for f, _ in A.GcpOpts._fields_] == [
        "loss", "grad_nnz", "grad_zeros", "est_nnz", "est_zeros", "epoch_iters", "lr", "beta1",
        "beta2", "epsilon", "decay", "max_fails", "seed"]
    for name, v in (("GAUSSIAN", 0), ("BERNOULLI_LOGIT", 1), ("POISSON_LOG", 2)):
        assert f"SPLATT_B200_GCP_{name} = {v}" in hdr


def test_kernels_do_not_spill():
    """Every k_gcp_ kernel of the built library uses no stack or local memory."""
    A.load()
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not Path(tool).exists():
        pytest.skip("cuobjdump not found")
    txt = subprocess.run([tool, "-res-usage", str(A.LIB_PATH)], capture_output=True, text=True,
                         check=True).stdout
    found, cur = {}, None
    for line in txt.splitlines():
        m = re.search(r"Function (\S*k_gcp_\w+?)(I\S*)?:", line)
        if m:
            cur = m.group(0)
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+) .*LOCAL:(\d+)", line)
        if m and cur:
            found[cur] = tuple(int(x) for x in m.groups())
            cur = None
    assert sum("k_gcp_sampled" in k for k in found) == 7 * 3
    assert sum("k_gcp_decode" in k for k in found) == 7
    assert {"k_gcp_sample", "k_gcp_adam", "k_gcp_check"} <= \
        {re.search(r"k_gcp_[a-z]+", k).group(0) for k in found}
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


def _np_coo(T):
    inds, vals = T.to_coo()
    return [i.cpu().numpy().astype(np.int64) for i in inds], vals.cpu().numpy()


def _multiset(inds, vals):
    key = np.stack([np.asarray(i, dtype=np.int64) for i in inds] + [np.asarray(vals).view(np.int64)], 1)
    return key[np.lexsort(key.T[::-1])]


@pytest.mark.gpu
@pytest.mark.parametrize("n", range(2, 9))
def test_to_coo_returns_the_input(S, n):
    """Untiled, ktile > 0 and ASGIVEN builds return the input multiset; on an untiled stream the
    records are in the lexicographic order of one of the tensor's level orders."""
    dims, inds, vals = random_coo(DIMS[n] if n > 2 else (700, 900), 4000, seed=n)
    want = _multiset(inds, vals)
    for kw in ({"ktile": -1}, {"ktile": 16}, {"layout": A.LAYOUT_ASGIVEN, "ktile": -1}):
        T = S.Tensor.from_coo(dims, inds, vals, **kw)
        gi, gv = _np_coo(T)
        np.testing.assert_array_equal(_multiset(gi, gv), want, err_msg=str(kw))
        if kw.get("ktile") == -1 and "layout" not in kw:
            perms = [T.mode_info(m, 16)["level_perm"] for m in range(n)]
            ident = np.arange(len(gv))
            assert any(np.array_equal(np.lexsort([gi[p] for p in perm[::-1]]), ident) for perm in perms), \
                "untiled records are not in lexicographic order"
        T.free()


@pytest.mark.gpu
@pytest.mark.parametrize("rows", [1, 5, 37])
def test_to_coo_on_cta_tiled_streams(S, rows, monkeypatch):
    """A CTA-tiled 3-mode stream (forced tiny tiles) decodes to the input multiset."""
    monkeypatch.setenv("SPLATT_B200_TILED", "2")
    monkeypatch.setenv("SPLATT_B200_TILE_ROWS", str(rows))
    dims, inds, vals = random_coo((300, 200, 400), 20000, seed=rows)
    T = S.Tensor.from_coo(dims, inds, vals, ncolumns_hint=16)
    gi, gv = _np_coo(T)
    np.testing.assert_array_equal(_multiset(gi, gv), _multiset(inds, vals))
    T.free()


@pytest.mark.gpu
@pytest.mark.parametrize("n", range(2, 9))
def test_gcp_sample_bitwise_matches_oracle(S, n):
    """The library's draws equal the oracle's bit for bit for several seeds and steps (one above
    2^32), both purposes pairs, given the tensor's own record order."""
    dims, inds, vals = random_coo(DIMS[n], 3000, seed=10 + n)
    T = S.Tensor.from_coo(dims, inds, vals)
    ci, cv = _np_coo(T)
    for seed, step, est in ((0, 0, False), (7, 1, False), (2**40 + 3, 2**33 + 5, True), (123, 999, True)):
        gi, gv = T.gcp_sample(seed, step, 1500, 1700, estimate=est)
        wi, wv = O.sample(dims, ci, cv, seed, step, est, 1500, 1700)
        for m in range(n):
            np.testing.assert_array_equal(gi[m].cpu().numpy().astype(np.int64), wi[m])
        np.testing.assert_array_equal(gv.cpu().numpy(), wv)
    T.free()


@pytest.mark.gpu
def test_gcp_sample_on_a_mode_of_2_29_rows(S):
    dims = [2**29, 3, 6]
    rng = np.random.default_rng(1)
    inds = [rng.integers(0, d, size=500).astype(np.uint64) for d in dims]
    vals = rng.uniform(size=500)
    T = S.Tensor.from_coo(dims, inds, vals)
    ci, cv = _np_coo(T)
    gi, gv = T.gcp_sample(99, 12, 300, 5000)
    wi, wv = O.sample(dims, ci, cv, 99, 12, False, 300, 5000)
    for m in range(3):
        np.testing.assert_array_equal(gi[m].cpu().numpy().astype(np.int64), wi[m])
    np.testing.assert_array_equal(gv.cpu().numpy(), wv)
    assert wi[0][300:].max() > 2**28
    T.free()


def _bounds(L, p, q, w_nz, w_z, inds, vals, factors):
    """Elementwise fp64 bounds of the sampled value and gradient.  m carries at most
    16 eps sum_r prod |U| of rounding (products of <= 8 factors, sums over <= 64 columns); it
    moves f by |f'| times that and y by |w f''| times that.  A sum of k terms in any order
    (the atomics' order, the oracle's) is within k eps of the sum of their absolute values, so a
    row hit by k samples gets (2 k + 64) eps of its absolute terms."""
    idx = [np.asarray(i, dtype=np.int64)[:p + q] for i in inds]
    m = O.model_values(idx, factors)
    eps = np.finfo(np.float64).eps
    dm = 16 * eps * O.model_values(idx, [np.abs(U) for U in factors])
    x = np.asarray(vals, dtype=np.float64)[:p]
    w = np.concatenate([np.full(p, abs(w_nz)), np.full(q, abs(w_z))])
    vt = np.concatenate([w_nz * O.f_corr(L, x, m[:p]), w_z * O.f(L, 0.0, m[p:])])
    slope = w * np.abs(np.concatenate([O.df_corr(L, x, m[:p]), O.df(L, 0.0, m[p:])]))
    vb = (2 * (p + q) + 64) * eps * np.abs(vt).sum() + (slope * dm).sum()
    fpp = {O.GAUSSIAN: 2.0, O.BERNOULLI_LOGIT: 0.25}.get(L, None)
    fpp = np.exp(m) if fpp is None else np.full(p + q, fpp)
    fpp[:p] = 0.0                                          # the stored-entry y does not depend on m
    gs = []
    for n, U in enumerate(factors):
        h = np.ones((p + q, U.shape[1]))
        for k, W in enumerate(factors):
            if k != n:
                h *= np.abs(W[idx[k]])
        cnt = np.bincount(idx[n], minlength=U.shape[0]).astype(np.float64)
        A_ = np.zeros_like(U)
        D_ = np.zeros_like(U)
        np.add.at(A_, idx[n], slope[:, None] * h)
        np.add.at(D_, idx[n], (w * fpp * dm)[:, None] * h)
        gs.append((2 * cnt[:, None] + 64) * eps * A_ + D_ + 1e-300)
    return vb, gs


@pytest.mark.gpu
@pytest.mark.parametrize("loss", LOSSES)
@pytest.mark.parametrize("n", range(2, 9))
def test_gcp_sampled_matches_oracle(S, loss, n):
    """Value and every mode's gradient within an elementwise fp64 bound, for R in
    {1, 2, 31, 32, 33, 64}; 40% of the samples hit row 0 of every mode.  NaN pad columns of the
    factors and the gradient buffers are never read into a result and never written."""
    import torch
    L = O.LOSS_NAMES[loss]
    dims = list(DIMS[n])
    rng = np.random.default_rng(n * 7 + L)
    T = S.Tensor.from_coo(dims, [rng.integers(0, d, size=50).astype(np.uint64) for d in dims],
                          values_for(loss, 50, rng))
    p, q = 2000, 3000
    inds = [rng.integers(0, d, size=p + q) for d in dims]
    hot = rng.random(p + q) < 0.4
    for i in inds:
        i[hot] = 0
    vals = np.concatenate([values_for(loss, p, rng), np.zeros(q)])
    for R in (1, 2, 31, 32, 33, 64):
        scale = (0.8 / R) ** (1.0 / n)
        f = [rng.normal(0, scale, (d, R)) for d in dims]
        ldm = R + (R & 1) + 2
        bufs, gbufs = [], []
        for d, U in zip(dims, f):
            b = torch.full((d, ldm), float("nan"), dtype=torch.float64, device="cuda")
            b[:, :R] = torch.from_numpy(U).cuda()
            bufs.append(b)
            gbufs.append(torch.full((d, ldm), float("nan"), dtype=torch.float64, device="cuda"))
        di = [torch.from_numpy(i.astype(np.int32)).cuda() for i in inds]
        dv = torch.from_numpy(vals).cuda()
        w_nz, w_z = 3.5, 17.25
        val, G = T.gcp_sampled(loss, di, dv, p, q, w_nz, w_z, [b[:, :R] for b in bufs], rank=R,
                               grads=[g[:, :R] for g in gbufs])
        wval, wG = O.sampled(L, p, q, w_nz, w_z, inds, vals, f)
        vb, gb = _bounds(L, p, q, w_nz, w_z, inds, vals, f)
        assert abs(val - wval) <= vb, (R, val, wval, vb)
        for m in range(n):
            g = G[m].cpu().numpy()
            assert np.all(np.abs(g - wG[m]) <= gb[m]), (loss, n, R, m, np.abs(g - wG[m]).max())
            assert torch.isnan(gbufs[m][:, R:]).all(), "pad columns written"
        assert np.isfinite(val)
    T.free()


@pytest.mark.gpu
def test_gcp_sampled_stays_finite_at_large_m(S):
    """Bernoulli at |m| ~ 700 and Poisson at m ~ 700 give finite values and gradients."""
    import torch
    dims = [4, 5]
    T = S.Tensor.from_coo(dims, [np.array([0, 1], dtype=np.uint64), np.array([2, 3], dtype=np.uint64)],
                          np.array([1.0, 1.0]))
    f = [np.full((4, 1), 700.0), np.array([[1.0], [-1.0], [1.0], [-1.0], [0.999]])]
    inds = [np.array([0, 1, 2, 3, 0, 1, 2, 3]), np.array([0, 1, 2, 3, 4, 4, 1, 0])]
    di = [torch.from_numpy(i.astype(np.int32)).cuda() for i in inds]
    vals = torch.tensor([1.0, 1.0, 0, 0, 0, 0, 0, 0], dtype=torch.float64, device="cuda")
    for loss in ("bernoulli-logit", "poisson-log"):
        L = O.LOSS_NAMES[loss]
        ff = f if loss == "bernoulli-logit" else [f[0], np.abs(f[1])]
        val, G = T.gcp_sampled(loss, di, vals, 2, 6, 1.0, 1.0, _cuda(ff))
        wval, wG = O.sampled(L, 2, 6, 1.0, 1.0, inds, vals.cpu().numpy(), ff)
        assert np.isfinite(val) and all(torch.isfinite(g).all() for g in G)
        assert abs(val - wval) <= 1e-13 * abs(wval)
        for g, w in zip(G, wG):
            np.testing.assert_allclose(g.cpu().numpy(), w, rtol=1e-13, atol=0)
    T.free()


def _driver_case(S, loss, seed=5):
    dims, inds, vals = problem((30, 25, 20), 1500, loss, seed=seed)
    T = S.Tensor.from_coo(dims, inds, vals)
    ci, cv = _np_coo(T)
    R = 4
    f0 = [np.random.default_rng(seed).normal(0, 0.5, (d, R)) for d in dims]
    return T, dims, ci, cv, R, f0


@pytest.mark.gpu
@pytest.mark.parametrize("loss", LOSSES)
def test_driver_matches_oracle(S, loss):
    """Two epochs of five steps from the same start and the same draws: the start estimate to
    1e-13, the history to 1e-9 and the factors to 1e-9 relative.  The gradients are summed with
    atomics in a different order (relative changes ~1e-16 per step) and Adam maps them almost
    one-to-one to the update, so ten steps stay far inside that bar."""
    T, dims, ci, cv, R, f0 = _driver_case(S, loss)
    kw = dict(grad_nnz=400, grad_zeros=600, est_nnz=2000, est_zeros=3000, epoch_iters=5,
              lr=0.01, seed=17, loss=O.LOSS_NAMES[loss])
    wf, wh, wn, wf0 = O.gcp(dims, ci, cv, f0, 2, -1.0, **kw)
    got, hist, n, fs = T.gcp(R, loss, _cuda(f0), niters=2, tol=-1.0, grad_samples=(400, 600),
                             est_samples=(2000, 3000), epoch_iters=5, lr=0.01, seed=17)
    assert n == wn == 2
    assert abs(fs - wf0) <= 1e-13 * abs(wf0)
    np.testing.assert_allclose(hist, wh, rtol=1e-9)
    for a, b in zip(got, wf):
        assert rel_fro(a.cpu().numpy(), b) < 1e-9
    T.free()


@pytest.mark.gpu
def test_failed_epochs_restore_and_decay(S):
    """With a huge lr every epoch fails: U comes back bitwise, lr halves with decay 0.5, and the
    run stops after max_fails + 1 failures."""
    T, dims, ci, cv, R, f0 = _driver_case(S, "bernoulli-logit")
    got, hist, n, fs = T.gcp(R, "bernoulli-logit", _cuda(f0), niters=10, tol=0.0, grad_samples=(400, 600),
                             est_samples=(2000, 3000), epoch_iters=5, lr=1e3, decay=0.5, max_fails=2)
    assert n == 3
    np.testing.assert_array_equal(hist[:, 2], [0, 0, 0])
    np.testing.assert_array_equal(hist[:, 1], [1e3, 5e2, 2.5e2])
    assert all(h > fs or not np.isfinite(h) for h in hist[:, 0])
    for a, b in zip(got, f0):
        np.testing.assert_array_equal(a.cpu().numpy(), b)
    T.free()


@pytest.mark.gpu
def test_niter_and_tolerance_stops(S):
    T, dims, ci, cv, R, f0 = _driver_case(S, "gaussian")
    common = dict(grad_samples=(400, 600), est_samples=(2000, 3000), epoch_iters=5, lr=1e-3)
    _, hist, n, _ = T.gcp(R, "gaussian", _cuda(f0), niters=3, tol=-1.0, max_fails=10, **common)
    assert n == 3 and hist.shape == (3, 3)
    _, hist, n, _ = T.gcp(R, "gaussian", _cuda(f0), niters=10, tol=1e9, max_fails=10, **common)
    first = int(np.argmax(hist[:, 2] == 1))
    assert hist[-1, 2] == 1 and n == first + 1
    _, hist, n, _ = T.gcp(R, "gaussian", _cuda(f0), niters=0, tol=0.0, **common)
    assert n == 0 and hist.shape == (0, 3)
    T.free()


def _dense_F(L, dims, inds, vals, factors):
    return O.objective(L, dims, inds, vals, [f.cpu().numpy() if hasattr(f, "cpu") else f for f in factors])


@pytest.mark.gpu
def test_planted_bernoulli_logit(S, capsys):
    """A binary tensor drawn from a rank-3 logit model on 100 x 120 x 140: the fitted model's
    exact F (computed densely) comes within the margin recorded in DESIGN.md of the planted
    model's, starting from far above it."""
    import torch
    rng = np.random.default_rng(21)
    dims, R = (100, 120, 140), 3
    U = [rng.normal(0, 1.6, (d, R)) for d in dims]
    M = np.einsum("az,bz,cz->abc", *U)
    P = 1.0 / (1.0 + np.exp(-M))
    X = rng.random(dims) < P
    inds = [i.astype(np.uint64) for i in np.nonzero(X)]
    vals = np.ones(len(inds[0]))
    T = S.Tensor.from_coo(list(dims), inds, vals)
    got, hist, n, fs = T.gcp(R, "bernoulli-logit", niters=40, tol=1e-5, grad_samples=(1 << 14, 1 << 14),
                             est_samples=(1 << 18, 1 << 18), epoch_iters=200, lr=1e-2, seed=3)
    Ft = _dense_F(O.BERNOULLI_LOGIT, dims, inds, vals, U)
    Fg = _dense_F(O.BERNOULLI_LOGIT, dims, inds, vals, got)
    with capsys.disabled():
        print(f"\nplanted bernoulli: F(planted) {Ft:.6e}  F(gcp) {Fg:.6e}  ratio {Fg / Ft:.5f}  "
              f"epochs {n}  f_start {fs:.4e}")
    assert fs > 1.3 * Ft
    assert Fg <= 1.02 * Ft
    T.free()


@pytest.mark.gpu
def test_planted_poisson_log(S, capsys):
    """A count tensor drawn from a rank-3 log-rate model on 40 x 50 x 60."""
    rng = np.random.default_rng(22)
    dims, R = (40, 50, 60), 3
    U = [rng.normal(0, 0.9, (d, R)) for d in dims]
    M = np.einsum("az,bz,cz->abc", *U)
    X = rng.poisson(np.exp(M))
    nz = np.nonzero(X)
    inds = [i.astype(np.uint64) for i in nz]
    vals = X[nz].astype(np.float64)
    T = S.Tensor.from_coo(list(dims), inds, vals)
    got, hist, n, fs = T.gcp(R, "poisson-log", niters=40, tol=1e-5, grad_samples=(1 << 14, 1 << 14),
                             est_samples=(1 << 18, 1 << 18), epoch_iters=200, lr=1e-2, seed=4)
    Ft = _dense_F(O.POISSON_LOG, dims, inds, vals, U)
    Fg = _dense_F(O.POISSON_LOG, dims, inds, vals, got)
    with capsys.disabled():
        print(f"\nplanted poisson: F(planted) {Ft:.6e}  F(gcp) {Fg:.6e}  diff/|F| {(Fg - Ft) / abs(Ft):.5f}  "
              f"epochs {n}")
    assert Fg - Ft <= 0.06 * abs(Ft)
    T.free()


@pytest.mark.gpu
def test_gaussian_against_cpd_als(S, capsys):
    """With the Gaussian loss GCP minimises ||X - M||^2 over every coordinate, as CPD-ALS does;
    at the same rank its final residual comes within the recorded margin of ALS's."""
    rng = np.random.default_rng(23)
    dims, R = (60, 70, 80), 4
    U = [rng.uniform(0, 1, (d, R)) for d in dims]
    M = np.einsum("az,bz,cz->abc", *U)
    keep = rng.random(dims) < 0.2
    X = np.where(keep, M + 0.05 * rng.standard_normal(dims), 0.0)
    nz = np.nonzero(keep)
    inds = [i.astype(np.uint64) for i in nz]
    vals = X[nz]
    T = S.Tensor.from_coo(list(dims), inds, vals)
    fit, lam, facs, _ = T.cpd_als(R, niters=200, tol=1e-9)
    xn2 = float((vals ** 2).sum())
    als = ((1.0 - fit) ** 2) * xn2
    got, hist, n, fs = T.gcp(R, "gaussian", niters=40, tol=1e-5, grad_samples=(1 << 14, 1 << 14),
                             est_samples=(1 << 18, 1 << 18), epoch_iters=200, lr=1e-2, seed=5)
    Mg = np.einsum("az,bz,cz->abc", *[g.cpu().numpy() for g in got])
    res = float(((X - Mg) ** 2).sum())
    with capsys.disabled():
        print(f"\ngaussian: ||X-M||^2 gcp {res:.6e}  als {als:.6e}  ratio {res / als:.5f}  epochs {n}")
    assert res <= 1.01 * als
    T.free()


@pytest.mark.gpu
def test_input_rules(S):
    """Every rule returns BADINPUT with the factors bitwise untouched."""
    import torch
    lib = A.load()
    dims, inds, vals = problem((20, 15, 10), 300, "bernoulli-logit", seed=9)
    T = S.Tensor.from_coo(dims, inds, vals)
    R, ldm = 4, 4
    f = [torch.randn((d, ldm), dtype=torch.float64, device="cuda") for d in dims]
    keep = [x.clone() for x in f]
    ptrs = (A.val_p * 3)(*[C.cast(C.c_void_p(x.data_ptr()), A.val_p) for x in f])
    o = S.default_opts()
    o[A.OPTION_NITER] = 2

    def good():
        return A.GcpOpts(1, 100, 100, 1000, 1000, 3, 1e-3, 0.9, 0.999, 1e-8, 0.1, 1, 0)

    def run(t=T, R=R, ldm=ldm, go=None, opts=o):
        return lib.splatt_b200_gcp_device(t.h, R, ldm, opts.ctypes.data_as(A.val_p), C.byref(go or good()),
                                          ptrs, None, None, None, None)
    cases = []
    for field, bad in (("loss", 3), ("loss", -1), ("grad_nnz", -1), ("est_zeros", -5), ("epoch_iters", 0),
                       ("lr", 0.0), ("lr", float("nan")), ("beta1", 1.0), ("beta2", -0.1), ("epsilon", 0.0),
                       ("decay", 0.0), ("decay", 1.5), ("max_fails", -1)):
        g = good()
        setattr(g, field, bad)
        cases.append((field, dict(go=g)))
    g = good(); g.grad_nnz = g.grad_zeros = 0
    cases.append(("empty gradient sample", dict(go=g)))
    g = good(); g.est_nnz = g.est_zeros = 0
    cases.append(("empty estimate sample", dict(go=g)))
    cases += [("R 0", dict(R=0)), ("R 65", dict(R=65, ldm=66)), ("ldm odd", dict(ldm=5)),
              ("ldm < R", dict(R=4, ldm=2))]
    bo = o.copy(); bo[A.OPTION_NITER] = -1
    cases.append(("NITER", dict(opts=bo)))
    bo = o.copy(); bo[A.OPTION_TOLERANCE] = float("inf")
    cases.append(("TOLERANCE", dict(opts=bo)))
    Sh = T.shard(0, 2)
    cases.append(("sharded", dict(t=Sh)))
    for name, kw in cases:
        assert run(**kw) == A.SPLATT_ERROR_BADINPUT, name
    # values against each loss's rule
    for loss, bad in ((1, 0.5), (2, -1.0), (0, float("inf"))):
        vb = vals.copy()
        vb[7] = bad
        Tb = S.Tensor.from_coo(dims, inds, vb)
        g = good(); g.loss = loss
        assert run(t=Tb, go=g) == A.SPLATT_ERROR_BADINPUT, (loss, bad)
        Tb.free()
    torch.cuda.synchronize()
    for a, b in zip(f, keep):
        assert torch.equal(a, b)
    # the good call runs
    assert run() == A.SPLATT_SUCCESS
    with pytest.raises(ValueError):
        T.gcp(R, "logistic")
    Sh.free()
    T.free()
