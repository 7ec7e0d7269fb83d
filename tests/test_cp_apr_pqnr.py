"""Poisson CP decomposition by row-wise projected quasi-Newton (splatt_b200_cp_apr_pqnr_device /
Tensor.cp_apr_pqnr) against the numpy restatement in oracle/apr_pqnr.py.

CPU: the oracle's rank-1 closed form, its row problems against scipy's L-BFGS-B, the monotone
row objectives and log-likelihood, fewer outer iterations than MU on a planted model (with rows
that continue their line search); the symbols are declared; k_pqnr_step does not spill.
GPU: one outer iteration per (N, rank) against the oracle, lbfgs_mem 1 and 8, leaf-tiled streams
against untiled, reproducibility, the history, the planted model against MU, a row that gives
up, a mode whose rows all stop at once (no line search launched), input rules, pad columns, the
Python rules, and one outer iteration on tensors that wrap every warp's record ring.
"""
import ctypes as C
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

from oracle import apr as OM
from oracle import apr_pqnr as Q
from splatt_b200 import _abi as A
from tests.test_cp_apr import DIMS, congruence, marginals, planted, problem, start
from tests.test_cp_apr_pdnr import (_data, _differing_rows, _perturbed, _row_problem, _sample_rows,
                                    _tiled)
from tests.test_walk_at_scale import assert_ring_wraps, bits, scale  # noqa: F401 (scale: fixture)
from tests.util import random_coo, rel_fro

RANKS = (1, 2, 16, 17, 32, 33, 64)
CASES = ([(f"sweep_n{n}_r{r}", n, r, "slots") for n in range(2, 9) for r in RANKS] +
         [("whole_r40", 2, 40, "whole"), ("skew_r17", 3, 17, "skew"), ("skew_r40", 4, 40, "skew")])


# ---------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------
def test_oracle_rank1_closed_form():
    """At rank 1 every row's minimiser is b_i = sum_{x in X_i} v_x, so one outer iteration with
    enough steps gives lam = sum v and A_n = marginals / sum v.  A row without records has
    g = 1 at every b, so it stores no pair and walks to 0 along d = -1 one unit per step: the
    rows with records converge within 20 evaluations, the empty ones take longer."""
    dims, inds, vals = problem((11, 9, 13), 300, seed=5)
    tot, want = marginals(dims, inds, vals)
    lam, Af, hist, info = Q.cp_apr_pqnr(dims, inds, vals, start(dims, 1), 1, 1e-13, max_inner=400)
    assert abs(lam[0] - tot) <= 1e-12 * tot
    for a, w in zip(Af, want):
        np.testing.assert_allclose(a, w, rtol=1e-12, atol=1e-15)
    assert any(r["nnz"] == 0 for r in info["rows"])
    assert all(r["kkt"] < 1e-12 * max(1.0, r["nnz"]) for r in info["rows"])
    assert max(r["evals"] for r in info["rows"] if r["nnz"]) <= 20
    assert max(r["evals"] for r in info["rows"] if not r["nnz"]) > 20


@pytest.mark.parametrize("R", list(range(1, 17)))
def test_oracle_rows_match_lbfgsb(R):
    """Seeded row problems, including rows with fewer records than R and rows with none: the
    oracle's objective matches scipy's L-BFGS-B (bounds b >= 0) to 1e-8 relative, and its last
    kkt is below tol."""
    from scipy.optimize import minimize
    rng = np.random.default_rng(100 + R)
    tol = 1e-9
    for nnz in (0, max(R // 2, 1), R, 4 * R + 10):
        b0, Pi, v = _row_problem(rng, R, nnz)
        b, info = Q.row_subproblem(b0, Pi, v, tol, max_inner=300)
        assert info["kkt"] < tol, (R, nnz, info["kkt"])

        def f(x):
            m = np.maximum(Pi @ x, 1e-10)
            return x.sum() - v @ np.log(m), np.ones(R) - Pi.T @ (v / m)
        ref = minimize(f, b0, jac=True, method="L-BFGS-B", bounds=[(0, None)] * R,
                       options={"ftol": 1e-15, "gtol": 1e-12, "maxiter": 10000})
        fo = Q._row_f(b, Pi, v, 1e-10)
        assert abs(fo - ref.fun) <= 1e-8 * max(1.0, abs(ref.fun)), (R, nnz, fo, ref.fun)


def test_oracle_is_monotone():
    """Every row's f is non-increasing through its steps, and the log-likelihood does not
    decrease from mode to mode or from outer iteration to outer iteration."""
    dims, inds, vals = problem((20, 15, 18), 1200, seed=8)
    lam, Af, hist, info = Q.cp_apr_pqnr(dims, inds, vals, start(dims, 5), 4, 0.0, max_inner=8)
    for r in info["rows"]:
        f = np.array(r["f"])
        assert np.all(np.diff(f) <= 1e-12 * np.abs(f[:-1]) + 1e-300), f
    ll = np.array(info["ll_modes"])
    assert np.all(np.diff(ll) >= -1e-12 * np.abs(ll[:-1])), ll
    assert np.all(np.diff(hist[:, 0]) >= -1e-12 * np.abs(hist[:-1, 0]))


PQNR_PLANTED_ITERS = 40
PQNR_PLANTED_OUTER = 25          # the oracle's counts on the planted model when the test was written
PQNR_PLANTED_LOCKSTEP = 569


def _planted_start(dims):
    return [np.random.default_rng(4).uniform(0.1, 1.0, (d, 3)) for d in dims]


def test_oracle_pqnr_needs_fewer_outer_iterations_than_mu():
    """On the planted model, from the same start, PQNR reaches max kkt < 1e-4 in fewer outer
    iterations than MU, recovers the model, and some rows continue their line search after one
    that moved nothing (an entry at the floor makes |g| huge and the first trial points fail)."""
    dims, inds, vals, F = planted()
    f0 = _planted_start(dims)
    _, Ap, hp, info = Q.cp_apr_pqnr(dims, inds, vals, f0, PQNR_PLANTED_ITERS, 1e-4)
    assert hp[-1, 1] < 1e-4 and hp[-1, 3] == 0, hp
    assert len(hp) == PQNR_PLANTED_OUTER and hp[:, 2].sum() == PQNR_PLANTED_LOCKSTEP, hp
    _, Am, hm, _ = OM.cp_apr(dims, inds, vals, f0, len(hp), 1e-4)
    assert hm[-1, 1] >= 1e-4, hm[-1]                     # MU has not converged after as many
    assert congruence(F, Ap) >= 0.99
    assert any(r["levels"] for r in info["rows"])


def _give_up_problem():
    """A zero start row with eps = 1e-200: m = 0 at every record, g is about -1e200, and every
    trial point along d = -g, halved 8 times per round, fails; the row gives up at its fourth
    evaluation."""
    dims, inds, vals = problem((20, 15, 18), 1500, seed=4)
    f0 = start(dims, 4)
    f0[0][5] = 0.0
    return dims, inds, vals, f0, {"eps": 1e-200, "max_inner": 6}


def test_oracle_gives_up_after_three_rounds():
    dims, inds, vals, f0, kw = _give_up_problem()
    _, _, _, info = Q.cp_apr_pqnr(dims, inds, vals, f0, 1, 0.0, **kw)
    r = next(r for r in info["rows"] if r["mode"] == 0 and r["row"] == 5)
    assert r["gave_up"] and r["levels"] == [1, 2, 3] and r["ks"] == [-1, -1, -1] and r["evals"] == 4, r


def test_pqnr_symbols_declared():
    hdr = (Path(__file__).resolve().parent.parent / "include" / "splatt_b200.h").read_text()
    assert "int splatt_b200_cp_apr_pqnr_device(" in hdr
    assert "splatt_b200_cp_apr_pqnr_device" in A.EXPORTS
    assert "} splatt_b200_pqnr_opts;" in hdr
    assert [f for f, _ in A.PqnrOpts._fields_] == ["max_inner", "max_backtrack", "lbfgs_mem",
                                                   "eps_active", "eps_div_zero"]


def test_pqnr_kernels_do_not_spill():
    """k_pqnr_step and k_pqnr_init of the built library use no stack or local memory."""
    A.load()
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not Path(tool).exists():
        pytest.skip("cuobjdump not found")
    txt = subprocess.run([tool, "-res-usage", str(A.LIB_PATH)], capture_output=True, text=True,
                         check=True).stdout
    found, cur = {}, None
    for line in txt.splitlines():
        m = re.search(r"Function (\S*k_pqnr_\w*?)(E\S*)?:", line)
        if m:
            cur = m.group(0)
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+) .*LOCAL:(\d+)", line)
        if m and cur:
            found[cur] = tuple(int(x) for x in m.groups())
            cur = None
    assert sum("k_pqnr_step" in k for k in found) == 1, found
    assert sum("k_pqnr_init" in k for k in found) == 1, found
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


def _np(facs):
    return [x.cpu().numpy() for x in facs]


def _row_tied(r):
    """The oracle row r made a decision at rounding level: a line-search margin within 1e-12 of
    zero relative to f_i with a trial step that moves b by more than rounding, or a candidate
    pair whose s.y lies within 1e-12 of zero relative to |s| |y|."""
    scale = max(abs(r["f"][0]), 1.0)
    return (any(abs(d[1]) <= 1e-12 * scale and d[2] > 1e-13 for d in r["decisions"]) or
            any(abs(p[0]) <= 1e-12 * p[2] for p in r["pairs"]))


def _check_against_oracle(name, dims, got, lam, wf, wl, info, perturbed):
    """Every mode of the device's factors, and lambda, equal the oracle's to 1e-10 relative, or
    to ten times the oracle's own spread there when its start moves by 1e-14 relative
    (perturbed(seed): the oracle's (lam, factors) from such a start; two seeds), whichever is
    larger: the unscaled first step d = -g and the continued line searches magnify rounding in
    some rows, and the device's sums are ordered differently.  Else the first mode
    that differs is explained by the oracle: every row that differs (after matching column sums)
    made a decision at rounding level, at most 5 % of the mode's rows (or 3) differ, and the mode
    differs by less than 0.1 (1e-8 when no row differs beyond the column sums).  Returns True
    when the 1e-10 bar held, so that the caller also holds the counts and the kkt to the oracle's."""
    n = len(dims)
    g = _np(got)
    errs = [rel_fro(g[m], wf[m]) for m in range(n)]
    worst = max(errs + [rel_fro(lam, wl)])
    if worst < 1e-10:
        return True
    runs = [perturbed(seed) for seed in (1, 2)]
    spread = [max(rel_fro(pf[m], wf[m]) for _, pf in runs) for m in range(n)]
    spread_lam = max(rel_fro(pl, wl) for pl, _ in runs)
    if (all(e < max(1e-10, 10 * sp) for e, sp in zip(errs, spread)) and
            rel_fro(lam, wl) < max(1e-10, 10 * spread_lam)):
        return False
    m = next((m for m, e in enumerate(errs) if e >= bar), n - 1)
    rows = _differing_rows(g[m], wf[m])
    tied = {r["row"] for r in info["rows"] if r["mode"] == m and _row_tied(r)}
    assert set(rows.tolist()) <= tied, (name, m, errs, rows[:10], sorted(tied)[:10])
    assert len(rows) <= max(3, dims[m] // 20), (name, m, len(rows))
    assert errs[m] < (0.1 if len(rows) else 1e-8), (name, m, errs)
    return False


@pytest.mark.gpu
@pytest.mark.parametrize("name,n,R,path", CASES, ids=[c[0] for c in CASES])
def test_one_outer_iteration_matches_oracle(S, name, n, R, path):
    """One outer iteration with tol = 0 and max_inner = 6 equals the oracle to its bar
    (_check_against_oracle: 1e-10 relative per mode and for lambda, or the oracle's own spread),
    with the oracle's lockstep and line-search counts; a larger difference must be explained by
    the oracle's rounding-level decisions."""
    dims, inds, vals = _data(path, n, R, seed=n * 100 + R)
    T = S.Tensor.from_coo(dims, inds, vals)
    if path == "skew":
        hot = np.bincount(inds[0].astype(np.int64)).max()
        assert hot > 64 * 40, hot                          # spans many 64-record chunks
    f0 = start(dims, R)
    wl, wf, wh, info = Q.cp_apr_pqnr(dims, inds, vals, f0, 1, 0.0, max_inner=6)
    lam, got, hist, its = T.cp_apr_pqnr(R, _cuda(f0), niters=1, tol=0.0, max_inner=6)
    assert its == 1
    perturbed = lambda seed: Q.cp_apr_pqnr(dims, inds, vals, _perturbed(f0, seed), 1, 0.0,  # noqa: E731
                                           max_inner=6)[:2]
    if _check_against_oracle(name, dims, got, lam, wf, wl, info, perturbed):
        assert np.array_equal(hist[0, 2:], wh[0, 2:]), (hist, wh)
        np.testing.assert_allclose(hist[0, 1], wh[0, 1], rtol=1e-8)
    T.free()


@pytest.mark.gpu
@pytest.mark.parametrize("mem", [1, 8])
def test_lbfgs_memory(S, mem):
    """lbfgs_mem 1 and 8 over two outer iterations of 12 lockstep iterations (rows store more
    pairs than 8, so the ring wraps) against the oracle."""
    dims, inds, vals = problem(DIMS[3], 6000, seed=31)
    R = 12
    f0 = start(dims, R)
    T = S.Tensor.from_coo(dims, inds, vals)
    wl, wf, wh, info = Q.cp_apr_pqnr(dims, inds, vals, f0, 2, 0.0, max_inner=12, lbfgs_mem=mem)
    assert max(sum(p[1] for p in r["pairs"]) for r in info["rows"]) > mem
    lam, got, hist, its = T.cp_apr_pqnr(R, _cuda(f0), niters=2, tol=0.0, max_inner=12, lbfgs_mem=mem)
    assert its == 2
    perturbed = lambda seed: Q.cp_apr_pqnr(dims, inds, vals, _perturbed(f0, seed), 2, 0.0,  # noqa: E731
                                           max_inner=12, lbfgs_mem=mem)[:2]
    if _check_against_oracle(f"mem{mem}", dims, got, lam, wf, wl, info, perturbed):
        assert np.array_equal(hist[:, 2:], wh[:, 2:]), (hist, wh)
    T.free()


def _phi_kernels(fn):
    """The ROWS template arguments of the k_apr_phi kernels fn launched."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return {m.group(1) for e in prof.events() for m in [re.search(r"k_apr_phi<\d+, (\w+)>", e.name)] if m}


@pytest.mark.gpu
@pytest.mark.parametrize("R", [8, 16, 33])
def test_cta_tiled_and_ktile_streams_match_untiled(S, monkeypatch, R):
    """A CTA-tiled 3-mode stream and an L1 leaf-tiled one (ktile > 0) give the result of the
    untiled build, over two outer iterations, to 1e-12 or to ten times the untiled run's own
    spread under a 1e-14 relative change of the start, whichever is larger."""
    dims, inds, vals = random_coo((300, 200, 400), 120000, seed=5, unique=False)
    vals = np.floor(vals * 4.0) + 1.0
    f0 = start(dims, R)
    U = S.Tensor.from_coo(dims, inds, vals, ktile=-1)
    bl, bf, bh, _ = U.cp_apr_pqnr(R, _cuda(f0), niters=2, tol=0.0, max_inner=4)
    pl, pf, _, _ = U.cp_apr_pqnr(R, _cuda(_perturbed(f0)), niters=2, tol=0.0, max_inner=4)
    bar = max(1e-12, 10 * max([rel_fro(pl, bl)] + [rel_fro(a, b) for a, b in zip(_np(pf), _np(bf))]))
    assert bar < 1e-8, bar                               # the problem is well conditioned
    assert not _phi_kernels(lambda: U.cp_apr_pqnr(R, _cuda(f0), niters=1, max_inner=1)) & {"true"}
    for path in ("cta", "ktile"):
        T = _tiled(S, monkeypatch, dims, inds, vals, path, R)
        assert _phi_kernels(lambda: T.cp_apr_pqnr(R, _cuda(f0), niters=1, max_inner=1)) == {"true"}, path
        lam, got, hist, _ = T.cp_apr_pqnr(R, _cuda(f0), niters=2, tol=0.0, max_inner=4)
        assert rel_fro(lam, bl) < bar, path
        for m in range(3):
            assert rel_fro(_np(got)[m], _np(bf)[m]) < bar, (path, m)
        np.testing.assert_allclose(hist[:, 0], bh[:, 0], rtol=1e-12)
        assert np.array_equal(hist[:, 2:], bh[:, 2:])
        T.free()


@pytest.mark.gpu
def test_untiled_runs_are_bitwise_reproducible(S):
    dims, inds, vals = random_coo((300, 200, 150), 40000, seed=9, unique=False, skew=[1.4, 0, 0])
    vals = np.floor(vals * 5.0)
    T = S.Tensor.from_coo(dims, inds, vals, ktile=-1)
    f0 = start(dims, 17)
    l1, f1, h1, i1 = T.cp_apr_pqnr(17, _cuda(f0), niters=3, tol=1e-3)
    l2, f2, h2, i2 = T.cp_apr_pqnr(17, _cuda(f0), niters=3, tol=1e-3)
    assert i1 == i2 and np.array_equal(l1, l2) and np.array_equal(h1[:, 1:], h2[:, 1:])
    for a, b in zip(f1, f2):
        assert np.array_equal(a.cpu().numpy().view(np.int64), b.cpu().numpy().view(np.int64))


@pytest.mark.gpu
def test_history_matches_oracle_and_ll_ascends(S):
    """Several outer iterations with tol > 0: the log-likelihood never decreases (1e-12
    relative), matches the oracle's to 1e-9, and the lockstep and line-search counts are the
    oracle's."""
    dims, inds, vals = problem((40, 30, 50), 6000, seed=11)
    R, tol = 6, 1e-3
    f0 = start(dims, R)
    T = S.Tensor.from_coo(dims, inds, vals)
    wl, wf, wh, info = Q.cp_apr_pqnr(dims, inds, vals, f0, 6, tol, max_inner=6)
    lam, got, hist, its = T.cp_apr_pqnr(R, _cuda(f0), niters=6, tol=tol, max_inner=6)
    assert np.all(np.diff(hist[:, 0]) >= -1e-12 * np.abs(hist[:-1, 0])), hist[:, 0]
    assert its == len(wh)
    np.testing.assert_allclose(hist[:, 0], wh[:, 0], rtol=1e-9)
    assert np.array_equal(hist[:, 2:], wh[:, 2:]), (hist, wh)
    assert len(set(wh[:, 3])) > 1                      # the counts vary, so the test means something


@pytest.mark.gpu
def test_planted_model_recovered_faster_than_mu(S):
    dims, inds, vals, F = planted()
    f0 = _planted_start(dims)
    T = S.Tensor.from_coo(dims, inds, vals)
    lam, got, hist, its = T.cp_apr_pqnr(3, _cuda(f0), niters=PQNR_PLANTED_ITERS, tol=1e-4)
    assert hist[-1, 1] < 1e-4 and its < PQNR_PLANTED_ITERS, hist
    assert congruence(F, _np(got)) >= 0.99
    for g in _np(got):
        np.testing.assert_allclose(g.sum(axis=0), 1.0, rtol=1e-12)
        assert (g >= 0).all()
    _, _, hm, itm = T.cp_apr(3, _cuda(f0), niters=its, tol=1e-4)
    assert hm[-1, 1] >= 1e-4                           # MU has not converged in as many


@pytest.mark.gpu
def test_row_gives_up_like_oracle(S):
    """The row of _give_up_problem fails three rounds of line searches and stops; the run
    matches the oracle, counts included."""
    dims, inds, vals, f0, kw = _give_up_problem()
    wl, wf, wh, info = Q.cp_apr_pqnr(dims, inds, vals, f0, 1, 0.0, **kw)
    assert any(r["gave_up"] for r in info["rows"])
    T = S.Tensor.from_coo(dims, inds, vals)
    lam, got, hist, its = T.cp_apr_pqnr(4, _cuda(f0), niters=1, tol=0.0, max_inner=kw["max_inner"],
                                        eps=kw["eps"])
    assert rel_fro(lam, wl) < 1e-10
    for m in range(3):
        assert rel_fro(_np(got)[m], wf[m]) < 1e-10, m
    assert np.array_equal(hist[0, 2:], wh[0, 2:]), (hist, wh)


@pytest.mark.gpu
def test_rows_stopping_at_once_skip_the_line_search(S):
    """With every row below tol at its first evaluation, one outer iteration launches per mode
    only B = A diag(lambda), the init, the Phi walk and its combine, k_pqnr_step, the kkt max,
    the column sums (2) and the normalisation -- no ladder and no accept -- besides the start's
    checks (1 + 3 per mode), its normalisation (1 per mode) and the log-likelihood (1)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    dims, inds, vals = problem(DIMS[3], 3000, seed=12)
    T = S.Tensor.from_coo(dims, inds, vals, ktile=-1)
    N = len(dims)
    f0 = _cuda(start(dims, 8))
    torch.cuda.synchronize()
    before = S.launch_count()
    lam, got, hist, its = T.cp_apr_pqnr(8, f0, niters=5, tol=1e30)
    assert its == 1 and hist[0, 2] == N and hist[0, 3] == 0, hist
    assert S.launch_count() - before == 2 + 5 * N + 8 * N
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        T.cp_apr_pqnr(8, _cuda(start(dims, 8)), niters=1, tol=1e30)
        torch.cuda.synchronize()
    names = {e.name for e in prof.events()}
    assert any("k_pqnr_step" in x for x in names), names
    assert not any("k_pdnr_ladder" in x or "k_pdnr_accept" in x for x in names), names


def _raw(T, R, ldm, opts, bufs, po=None):
    import torch
    torch.cuda.synchronize()
    ptrs = (A.val_p * len(bufs))(*[C.cast(C.c_void_p(b.data_ptr()), A.val_p) for b in bufs])
    lam = np.zeros(max(R, 1))
    hist = np.zeros(4 * 4)
    its = C.c_int()
    rc = T.lib.splatt_b200_cp_apr_pqnr_device(T.h, R, ldm, opts.ctypes.data_as(C.POINTER(C.c_double)),
                                              None if po is None else C.byref(po), ptrs,
                                              lam.ctypes.data_as(C.POINTER(C.c_double)),
                                              hist.ctypes.data_as(C.POINTER(C.c_double)), C.byref(its),
                                              None)
    torch.cuda.synchronize()
    return rc, lam, hist


@pytest.mark.gpu
def test_bad_input_rejected_and_pad_columns(S):
    """Every input rule returns BADINPUT with the factors bit-identical; NaN pad columns change
    nothing and stay bit-identical."""
    import torch
    dims, inds, vals = problem((20, 15, 18), 1500, seed=4)
    R = 5
    T = S.Tensor.from_coo(dims, inds, vals)
    o = S.default_opts()
    o[A.OPTION_NITER] = 2
    o[A.OPTION_TOLERANCE] = 0.0
    f0 = start(dims, R)

    def bufs(ldm, fill=float("nan"), f=f0):
        b = [torch.full((d, ldm), fill, dtype=torch.float64, device="cuda") for d in dims]
        for x, y in zip(b, f):
            x[:, :R].copy_(torch.from_numpy(y))
        return b

    def check_bad(rc, b, ldm, f=f0):
        assert rc == A.SPLATT_ERROR_BADINPUT
        for x, y in zip(b, bufs(ldm, f=f)):
            assert torch.equal(x.view(torch.int64), y.view(torch.int64))

    for ldm in (5, 4):
        b = bufs(6)
        check_bad(_raw(T, R, ldm, o, b)[0], b, 6)
    for r in (0, 65):
        b = bufs(66)
        check_bad(_raw(T, r, 66, o, b)[0], b, 66)
    for key, x in ((A.OPTION_NITER, -1.0), (A.OPTION_NITER, float("nan")), (A.OPTION_TOLERANCE, -1.0),
                   (A.OPTION_TOLERANCE, float("nan"))):
        oo = o.copy()
        oo[key] = x
        b = bufs(6)
        check_bad(_raw(T, R, 6, oo, b)[0], b, 6)
    nan, inf = float("nan"), float("inf")
    for po in (A.PqnrOpts(0, 8, 3, 1e-8, 1e-10), A.PqnrOpts(10, 0, 3, 1e-8, 1e-10),
               A.PqnrOpts(10, 9, 3, 1e-8, 1e-10), A.PqnrOpts(10, 8, 0, 1e-8, 1e-10),
               A.PqnrOpts(10, 8, 9, 1e-8, 1e-10), A.PqnrOpts(10, 8, -1, 1e-8, 1e-10),
               A.PqnrOpts(10, 8, 3, -1e-8, 1e-10), A.PqnrOpts(10, 8, 3, nan, 1e-10),
               A.PqnrOpts(10, 8, 3, inf, 1e-10), A.PqnrOpts(10, 8, 3, 1e-8, 0.0),
               A.PqnrOpts(10, 8, 3, 1e-8, nan), A.PqnrOpts(10, 8, 3, 1e-8, -1e-10)):
        b = bufs(6)
        check_bad(_raw(T, R, 6, o, b, po)[0], b, 6)
    for m, (i, c, x) in enumerate([(3, 1, -0.5), (4, 2, nan), (0, 0, inf)]):
        f = [y.copy() for y in f0]
        f[m][i, c] = x
        b = bufs(6, f=f)
        check_bad(_raw(T, R, 6, o, b)[0], b, 6, f=f)
    f = [y.copy() for y in f0]
    f[2][:, 4] = 0.0
    b = bufs(6, f=f)
    check_bad(_raw(T, R, 6, o, b)[0], b, 6, f=f)
    neg = vals.copy()
    neg[7] = -1.0
    for bad in (S.Tensor.from_coo(dims, inds, vals, layout=A.LAYOUT_ASGIVEN), T.shard(0, 2),
                S.Tensor.from_coo(dims, inds, neg)):
        b = bufs(6)
        check_bad(_raw(bad, R, 6, o, b)[0], b, 6)
        bad.free()
    b_nan, b_zero = bufs(8), bufs(8, 0.0)
    pad_before = [x[:, R:].clone() for x in b_nan]
    rc1, l1, h1 = _raw(T, R, 8, o, b_nan)
    rc2, l2, h2 = _raw(T, R, 8, o, b_zero)
    assert rc1 == rc2 == A.SPLATT_SUCCESS
    assert np.array_equal(l1, l2)
    np.testing.assert_allclose(h1, h2, rtol=1e-13)
    for x, y, p in zip(b_nan, b_zero, pad_before):
        assert torch.equal(x[:, :R], y[:, :R])
        assert torch.equal(x[:, R:].view(torch.int64), p.view(torch.int64))


@pytest.mark.gpu
def test_python_rules(S):
    import torch
    dims, inds, vals = problem((20, 15, 18), 1500, seed=4)
    T = S.Tensor.from_coo(dims, inds, vals)
    with pytest.raises(ValueError):
        T.cp_apr_pqnr(4, [torch.rand((d, 4), dtype=torch.float32, device="cuda") for d in dims])
    with pytest.raises(ValueError):
        T.cp_apr_pqnr(4, [torch.rand((d, 5), dtype=torch.float64, device="cuda") for d in dims])
    with pytest.raises(ValueError):
        T.cp_apr_pqnr(4, [torch.rand((d, 4), dtype=torch.float64) for d in dims])
    with pytest.raises(S.SplattError):
        T.cp_apr_pqnr(65)
    with pytest.raises(S.SplattError):
        T.cp_apr_pqnr(4, lbfgs_mem=9)
    with pytest.raises(S.SplattError):
        T.cp_apr_pqnr(4, max_backtrack=0)
    l1, f1, h1, i1 = T.cp_apr_pqnr(4, niters=3, seed=9)
    l2, f2, h2, i2 = T.cp_apr_pqnr(4, niters=3, seed=9)
    assert i1 == i2 and np.array_equal(l1, l2)
    assert all(torch.equal(a, b) for a, b in zip(f1, f2))
    assert h1.shape == (i1, 4)


# At scale: the tensors of tests/test_walk_at_scale.py (6 M records: every warp's record ring
# wraps; n3's mode 0 is Zipf-skewed, its hottest row spanning hundreds of ranges).
AT_SCALE = [("n3", 16), ("n4", 33)]
AT_SCALE_INNER = 5


@pytest.mark.gpu
@pytest.mark.parametrize("name,R", AT_SCALE, ids=[f"{n}-R{r}" for n, r in AT_SCALE])
def test_cp_apr_pqnr_at_scale(S, scale, name, R):
    """One Tensor.cp_apr_pqnr outer iteration with tol = 0 on a tensor that wraps every warp's
    record ring, bitwise the same on a second run, checked mode by mode on sampled rows (the
    hottest, the empty ones, the median one and random ones) against oracle.apr_pqnr's
    row_subproblem run on the rows the device saw, up to one scale per column (as in
    test_cp_apr_pdnr_at_scale), to 1e-8 relative per row or ten times the oracle's own spread
    for that row, whichever is larger.  The spread is the largest change of the oracle's row
    under 1e-14 relative changes of its start and under reorderings of its records (the device
    sums them in another order): rows that continue their line search after one that moved
    nothing take their last steps at rounding level.  The column
    scales are fitted on the rows whose spread is below 1e-12, and some sampled row must be such a
    row."""
    import torch
    dims, idx, vals, T = scale(name)
    assert_ring_wraps(T)
    N = len(dims)
    g = torch.Generator(device="cuda").manual_seed(R)
    f0 = [torch.rand((d, R), dtype=torch.float64, device="cuda", generator=g) for d in dims]
    lam, got, hist, its = T.cp_apr_pqnr(R, f0, niters=1, tol=0.0, max_inner=AT_SCALE_INNER)
    assert its == 1 and hist[0, 2] == AT_SCALE_INNER * N
    lam2, got2, hist2, _ = T.cp_apr_pqnr(R, f0, niters=1, tol=0.0, max_inner=AT_SCALE_INNER)
    assert np.array_equal(lam.view(np.int64), lam2.view(np.int64))
    assert np.array_equal(hist[:, 1:], hist2[:, 1:])
    for a, b in zip(got, got2):
        assert torch.equal(bits(a), bits(b))
    del got2
    cnts = [torch.bincount(i, minlength=d).cpu().numpy() for i, d in zip(idx, dims)]
    s0 = [f.sum(dim=0) for f in f0]
    cur = [f / s for f, s in zip(f0, s0)]                 # the factors as mode n sees them
    scale_in = torch.stack(s0).prod(dim=0)                # lambda entering mode 0
    rng = np.random.default_rng(R)
    for n in range(N):
        b_start = (cur[n] * scale_in).cpu().numpy()
        rows = _sample_rows(cnts[n], R, rng)
        want, dev, spread = [], [], []
        for i in rows:
            sel = (idx[n] == i).nonzero().squeeze(1)
            Pi = torch.ones((len(sel), R), dtype=torch.float64, device="cuda")
            for m in range(N):
                if m != n:
                    Pi *= cur[m][idx[m][sel]]
            pn, vn = Pi.cpu().numpy(), vals[sel].cpu().numpy()
            b, _ = Q.row_subproblem(b_start[i], pn, vn, 0.0, max_inner=AT_SCALE_INNER)
            sp = 0.0
            for seed in (1, 2):                           # the start moved, the records reordered
                u = np.random.default_rng(seed).uniform(-1.0, 1.0, R)
                o = np.random.default_rng(seed).permutation(len(vn))
                for b2, _ in (Q.row_subproblem(b_start[i] * (1.0 + 1e-14 * u), pn, vn, 0.0,
                                               max_inner=AT_SCALE_INNER),
                              Q.row_subproblem(b_start[i], pn[o], vn[o], 0.0, max_inner=AT_SCALE_INNER)):
                    sp = max(sp, np.abs(b2 - b).max() / max(np.abs(b).max(), 1e-300))
            want.append(b)
            spread.append(sp)
            dev.append(got[n][i].cpu().numpy())
        want, dev, spread = np.array(want), np.array(dev), np.array(spread)
        if n == N - 1:
            c = lam.copy()
        else:                                             # fitted on the rows rounding cannot move
            calm = spread < 1e-12 if (spread < 1e-12).any() else np.ones(len(rows), bool)
            den = dev[calm].sum(axis=0)
            c = np.where(den > 0, want[calm].sum(axis=0) / np.where(den > 0, den, 1.0), 1.0)
        err = np.abs(dev * c[None, :] - want).max(axis=1) / np.maximum(np.abs(want).max(axis=1), 1e-300)
        err[np.abs(want).max(axis=1) == 0] = np.abs(dev[np.abs(want).max(axis=1) == 0]).max(axis=1)
        bar = np.maximum(1e-8, 10 * spread)
        assert (err < bar).all(), (name, n, [(r, e, b) for r, e, b in zip(rows, err, bar) if e >= b][:5])
        assert (spread < 1e-12).any(), (name, n, spread)   # some rows are held to 1e-8
        cur[n] = got[n]
        scale_in = torch.from_numpy(c).cuda()
