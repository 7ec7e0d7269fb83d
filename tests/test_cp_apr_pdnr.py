"""Poisson CP decomposition by row-wise projected damped Newton (splatt_b200_cp_apr_pdnr_device /
Tensor.cp_apr_pdnr) against the numpy restatement in oracle/apr_pdnr.py.

CPU: the oracle's rank-1 closed form, its row problems against scipy's L-BFGS-B, the monotone
row objectives and log-likelihood, fewer outer iterations than MU on a planted model; the case
table reaches every kernel path; the symbols are declared; the new kernels do not spill.
GPU: one outer iteration per (N, rank) against the oracle, leaf-tiled streams against untiled,
reproducibility, the history, the rank-1 closed form, the planted model against MU, the Cholesky
fallback and a failed line search, input rules, pad columns and the Python rules.
"""
import ctypes as C
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

from oracle import apr as OM
from oracle import apr_pdnr as O
from splatt_b200 import _abi as A
from tests.test_cp_apr import DIMS, congruence, marginals, planted, problem, start
from tests.test_walk_at_scale import assert_ring_wraps, bits, scale  # noqa: F401 (scale: fixture)
from tests.util import random_coo, rel_fro

RANKS = (1, 2, 16, 17, 32, 33, 64)

# (name, nmodes, rank, path): "slots" = rows finished in the gradient walk (whole slices) and
# through the boundary slots and k_pdnr_solve (cut slices), every problem() mode with empty rows;
# "whole" = a 2-mode tensor long enough that the rank-64 tier has whole slices too; "skew" = one
# row spanning many ranges; "cta" / "ktile" = leaf-tiled streams (pieces added with red.add);
# "fallback" = a zero start row with eps = 1e-200 (H overflows: the Cholesky falls back to
# d = -g and every trial point fails the line search).  test_case_table_reaches_every_path
# counts the whole and the cut rows of every tier from the stream layout.
CASES = ([(f"sweep_n{n}_r{r}", n, r, "slots") for n in range(2, 9) for r in RANKS] +
         [("whole_r40", 2, 40, "whole"), ("skew_r17", 3, 17, "skew"), ("skew_r40", 4, 40, "skew"),
          ("cta_r16", 3, 16, "cta"), ("cta_r33", 3, 33, "cta"), ("ktile_r8", 3, 8, "ktile"),
          ("fallback_r4", 3, 4, "fallback")])


def _row_problem(rng, R, nnz):
    Pi = rng.uniform(0.0, 1.0, size=(nnz, R)) * rng.uniform(0.0, 0.2, size=(1, R))
    v = rng.poisson(3.0, size=nnz).astype(np.float64)
    b0 = rng.uniform(0.0, 2.0, size=R)
    return b0, Pi, v


# ---------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------
def test_oracle_rank1_closed_form():
    """At rank 1 every row's minimiser is b_i = sum_{x in X_i} v_x, so one outer iteration with
    enough Newton steps gives lam = sum v and A_n = marginals / sum v."""
    dims, inds, vals = problem((11, 9, 13), 300, seed=5)
    tot, want = marginals(dims, inds, vals)
    lam, Af, hist, info = O.cp_apr_pdnr(dims, inds, vals, start(dims, 1), 1, 0.0, max_inner=20)
    assert abs(lam[0] - tot) <= 1e-12 * tot
    for a, w in zip(Af, want):
        np.testing.assert_allclose(a, w, rtol=1e-12, atol=1e-15)
    assert any(r["nnz"] == 0 for r in info["rows"])
    assert all(r["kkt"] < 1e-12 * max(1.0, r["nnz"]) for r in info["rows"])


@pytest.mark.parametrize("R", [1, 2, 3, 5, 8, 12, 16])
def test_oracle_rows_match_lbfgsb(R):
    """Seeded row problems, including rows with fewer records than R (singular H) and rows with
    none: the oracle's objective matches scipy's L-BFGS-B (bounds b >= 0) to 1e-8 relative, and
    its last kkt is below tol."""
    from scipy.optimize import minimize
    rng = np.random.default_rng(100 + R)
    tol = 1e-9
    for nnz in (0, max(R // 2, 1), R, 4 * R + 10):
        b0, Pi, v = _row_problem(rng, R, nnz)
        b, info = O.row_subproblem(b0, Pi, v, tol, max_inner=100)
        assert info["kkt"] < tol, (R, nnz, info["kkt"])

        def f(x):
            m = np.maximum(Pi @ x, 1e-10)
            return x.sum() - v @ np.log(m), np.ones(R) - Pi.T @ (v / m)
        ref = minimize(f, b0, jac=True, method="L-BFGS-B", bounds=[(0, None)] * R,
                       options={"ftol": 1e-15, "gtol": 1e-12, "maxiter": 10000})
        fo = O._row_f(b, Pi, v, 1e-10)
        assert fo <= ref.fun + 1e-8 * max(1.0, abs(ref.fun)), (R, nnz, fo, ref.fun)
        assert abs(fo - ref.fun) <= 1e-8 * max(1.0, abs(ref.fun)), (R, nnz, fo, ref.fun)


def test_oracle_is_monotone():
    """Every row's f is non-increasing through its steps, and the log-likelihood does not
    decrease from mode to mode or from outer iteration to outer iteration."""
    dims, inds, vals = problem((20, 15, 18), 1200, seed=8)
    lam, Af, hist, info = O.cp_apr_pdnr(dims, inds, vals, start(dims, 5), 4, 0.0, max_inner=6)
    for r in info["rows"]:
        f = np.array(r["f"])
        assert np.all(np.diff(f) <= 1e-12 * np.abs(f[:-1]) + 1e-300), f
    ll = np.array(info["ll_modes"])
    assert np.all(np.diff(ll) >= -1e-12 * np.abs(ll[:-1])), ll
    assert np.all(np.diff(hist[:, 0]) >= -1e-12 * np.abs(hist[:-1, 0]))


PDNR_PLANTED_ITERS = 40


def test_oracle_pdnr_needs_fewer_outer_iterations_than_mu():
    """On the planted model, from the same start, PDNR reaches max kkt < 1e-4 in fewer outer
    iterations than MU (the counts when the test was written: PDNR 26, MU 93)."""
    dims, inds, vals, F = planted()
    f0 = [np.random.default_rng(4).uniform(0.1, 1.0, (d, 3)) for d in dims]
    _, Ap, hp, _ = O.cp_apr_pdnr(dims, inds, vals, f0, PDNR_PLANTED_ITERS, 1e-4)
    assert hp[-1, 1] < 1e-4 and hp[-1, 3] == 0, hp
    _, Am, hm, _ = OM.cp_apr(dims, inds, vals, f0, len(hp), 1e-4)
    assert hm[-1, 1] >= 1e-4, hm[-1]                     # MU has not converged after as many
    assert congruence(F, Ap) >= 0.99


def tier(R):
    return 16 if R <= 16 else 32 if R <= 32 else 64


def grad_warps(R, sms=132):
    """Warps of the gradient walk's grid: every resident CTA (2 per SM at tiers 16 and 32, 1 at
    tier 64, by the kernel's launch bounds and shared memory) times 8 warps."""
    return sms * 8 * (2 if R <= 32 else 1)


def slice_kinds(cnt, warps):
    """(whole, cut) rows of an untiled root stream whose rows hold cnt[i] records, in row order:
    the walk splits ceil(nrec / 64) chunks of 64 records evenly over the warps, and a row is
    finished in the walk (whole) when its records lie strictly inside one warp's range, neither
    its first nor its last slice; every other row with records goes through the boundary slots."""
    cnt = np.asarray(cnt, dtype=np.int64)
    cnt = cnt[cnt > 0]
    e = np.cumsum(cnt)
    s = e - cnt
    nrec = int(e[-1])
    nch = -(-nrec // 64)
    bnd = np.minimum(np.arange(warps + 1, dtype=np.int64) * nch // warps * 64, nrec)
    k = np.searchsorted(bnd, s, side="right") - 1          # the range of the row's first record
    whole = (bnd[k] < s) & (e < bnd[k + 1])
    return int(whole.sum()), int((~whole).sum())


def _data(path, n, R, seed):
    """The (dims, inds, vals) of a parity case, on the host."""
    if path == "slots":
        return problem(DIMS[n], max(2500, 200 * R), seed)
    if path == "whole":
        return problem((1500, 50), 300000, seed)
    dims = (300, 200, 150) if n == 3 else (60, 50, 40, 30)
    dims, inds, vals = random_coo(dims, 40000, seed=seed, unique=False, skew=[1.4] + [0] * (n - 1))
    return dims, inds, np.floor(vals * 5.0)                # counts 0..4, stored zeros included


PARITY = ("slots", "whole", "skew")


def test_case_table_reaches_every_path():
    """Every N in 2..8 meets every rank of RANKS, which covers the three rank tiers (16: the
    Hessian in registers; 32 and 64: in shared memory) and odd ranks.  Counted from the stream
    layout of the parity cases, every tier has rows finished in the gradient walk and rows
    assembled from boundary slots, and some row spans several ranges.  The table has both
    leaf-tiled stream kinds and the fallback / failed-line-search case.  problem() leaves empty
    rows in every mode; the sweep runs from a random start, so rows have active-set entries after
    their first projected step (test_oracle_case_paths)."""
    seen = {(n, r) for _, n, r, p in CASES if p == "slots"}
    assert seen == {(n, r) for n in range(2, 9) for r in RANKS}
    assert {p for *_, p in CASES} == {"slots", "whole", "skew", "cta", "ktile", "fallback"}
    kinds = {16: [0, 0], 32: [0, 0], 64: [0, 0]}
    longest = 0
    for _, n, R, path in CASES:
        if path not in PARITY:
            continue
        dims, inds, vals = _data(path, n, R, seed=n * 100 + R)
        for i, d in zip(inds, dims):
            cnt = np.bincount(np.asarray(i, dtype=np.int64), minlength=d)
            w, c = slice_kinds(cnt, grad_warps(R))
            kinds[tier(R)][0] += w
            kinds[tier(R)][1] += c
            longest = max(longest, int(cnt.max()) * grad_warps(R) // len(vals))
    assert all(w > 0 and c > 0 for w, c in kinds.values()), kinds
    assert longest >= 3, longest                           # a row longer than 3 warps' ranges


def test_oracle_case_paths():
    """The oracle side of the case table: a sweep case has active-set entries and rows with
    several accepted step lengths; the fallback case falls back and fails its line search."""
    dims, inds, vals = problem(DIMS[3], 3000, seed=3 * 100 + 17)
    _, _, _, info = O.cp_apr_pdnr(dims, inds, vals, start(dims, 17), 1, 0.0)
    assert any(a > 0 for r in info["rows"] for a in r["active"])
    assert any(r["nnz"] == 0 for r in info["rows"])
    dims, inds, vals, f0, kw = _fallback_problem()
    _, _, _, info = O.cp_apr_pdnr(dims, inds, vals, f0, 1, 0.0, **kw)
    assert any(r["fallbacks"] > 0 and -1 in r["ks"] for r in info["rows"])


def _fallback_problem():
    dims, inds, vals = problem((20, 15, 18), 1500, seed=4)
    f0 = start(dims, 4)
    f0[0][5] = 0.0                                       # m = 0 at every record of row 5
    return dims, inds, vals, f0, {"eps": 1e-200, "max_inner": 3}


def test_pdnr_symbols_declared():
    hdr = (Path(__file__).resolve().parent.parent / "include" / "splatt_b200.h").read_text()
    assert "int splatt_b200_cp_apr_pdnr_device(" in hdr
    assert "splatt_b200_cp_apr_pdnr_device" in A.EXPORTS
    assert "} splatt_b200_pdnr_opts;" in hdr
    assert [f for f, _ in A.PdnrOpts._fields_] == ["max_inner", "max_backtrack", "mu0",
                                                   "eps_active", "eps_div_zero"]


def test_pdnr_kernels_do_not_spill():
    """Every PDNR kernel of the built library uses no stack or local memory."""
    A.load()
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not Path(tool).exists():
        pytest.skip("cuobjdump not found")
    txt = subprocess.run([tool, "-res-usage", str(A.LIB_PATH)], capture_output=True, text=True,
                         check=True).stdout
    found, cur = {}, None
    for line in txt.splitlines():
        m = re.search(r"Function (\S*(k_pdnr_|pdnr_step)\w*?)(I\S*)?:", line)
        if m:
            cur = m.group(0)
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+) .*LOCAL:(\d+)", line)
        if m and cur:
            found[cur] = tuple(int(x) for x in m.groups())
            cur = None
    assert sum("k_pdnr_grad" in k for k in found) == 7 * 3 * 2
    assert sum("k_pdnr_ladder" in k for k in found) == 7 * 2
    assert sum("k_pdnr_solve" in k for k in found) == 3
    for name in ("k_pdnr_accept", "k_pdnr_init", "k_pdnr_kktmax"):
        assert sum(name in k for k in found) == 1, name
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


def _build(S, path, n, R, seed):
    dims, inds, vals = _data(path, n, R, seed)
    return dims, inds, vals, S.Tensor.from_coo(dims, inds, vals)


def _perturbed(f0, seed=1, rel=1e-14):
    """The start with every entry moved by up to rel relative (seeded)."""
    rng = np.random.default_rng(seed)
    return [f * (1.0 + rel * rng.uniform(-1.0, 1.0, f.shape)) for f in f0]


def _row_tied(r):
    """The oracle row r made a decision at rounding level: a Cholesky pivot within 1e-10 of zero
    relative to its diagonal (or a fallback), or a line-search margin within 1e-12 of zero
    relative to f_i with a trial step that moves b by more than rounding."""
    return (min(r["pivots"], default=1.0) < 1e-10 or
            any(abs(d[1]) <= 1e-12 * max(abs(r["f"][0]), 1.0) and d[2] > 1e-13 for d in r["decisions"]))


def _differing_rows(got, want, tol=1e-9):
    """Rows of a normalised factor that differ once each column is rescaled by the median ratio
    of the two (a changed row moves the column sum and so every row of its column a little)."""
    ratio = np.ones(got.shape[1])
    for r in range(got.shape[1]):
        ok = (got[:, r] > 0) & (want[:, r] > 0)
        if ok.any():
            ratio[r] = np.median(want[ok, r] / got[ok, r])
    scaled = got * ratio[None, :]
    d = np.abs(scaled - want).max(axis=1) / np.maximum(np.abs(want).max(axis=1), 1e-300)
    return np.nonzero(d > tol)[0]


@pytest.mark.gpu
@pytest.mark.parametrize("name,n,R,path", [c for c in CASES if c[3] in PARITY],
                         ids=[c[0] for c in CASES if c[3] in PARITY])
def test_one_outer_iteration_matches_oracle(S, name, n, R, path):
    """One outer iteration with tol = 0 (every row runs all max_inner steps) equals the oracle
    to 1e-10 relative per mode and for lambda; the lockstep and step counts are equal.  Rows get
    about 200 records per column of the rank so their Hessians are well conditioned.  Where a
    result still differs by more, it must be explained by the oracle: in the first mode that
    differs, every row that differs (after the column sums are matched) must have made a
    decision at rounding level (_row_tied), at most 5 % of its rows (or 3) may differ, and the
    mode differs by less than 0.1 in all (1e-8 when no row differs beyond matching the column
    sums).  A row whose Cholesky pivot sits at rounding level can take the fallback direction
    in one run and the Newton direction in the other, and then its path and its value differ."""
    dims, inds, vals, T = _build(S, path, n, R, seed=n * 100 + R)
    if path == "skew":
        hot = np.bincount(inds[0].astype(np.int64)).max()
        assert hot > 64 * 40, hot                          # spans many 64-record chunks
    f0 = start(dims, R)
    wl, wf, wh, info = O.cp_apr_pdnr(dims, inds, vals, f0, 1, 0.0, max_inner=5)
    lam, got, hist, its = T.cp_apr_pdnr(R, _cuda(f0), niters=1, tol=0.0, max_inner=5)
    assert its == 1
    assert hist[0, 2] == wh[0, 2] == 5 * n and hist[0, 3] == wh[0, 3] == 5 * sum(dims)
    g = _np(got)
    errs = [rel_fro(g[m], wf[m]) for m in range(n)]
    if max(errs + [rel_fro(lam, wl)]) >= 1e-10:
        m = next((m for m, e in enumerate(errs) if e >= 1e-10), n - 1)
        rows = _differing_rows(g[m], wf[m])
        tied = {r["row"] for r in info["rows"] if r["mode"] == m and _row_tied(r)}
        assert set(rows.tolist()) <= tied, (name, m, errs, rows[:10], sorted(tied)[:10])
        assert len(rows) <= max(3, dims[m] // 20), (name, m, len(rows))
        assert errs[m] < (0.1 if len(rows) else 1e-8), (name, m, errs)
    else:
        np.testing.assert_allclose(hist[0, 1], wh[0, 1], rtol=1e-8)
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


def _grad_kernels(fn):
    """The ROWS template arguments of the k_pdnr_grad kernels fn launched."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return {m.group(1) for e in prof.events() for m in [re.search(r"k_pdnr_grad<\d+, \d+, (\w+)>", e.name)] if m}


@pytest.mark.gpu
@pytest.mark.parametrize("R", [8, 16, 33])
def test_cta_tiled_and_ktile_streams_match_untiled(S, monkeypatch, R):
    """A CTA-tiled 3-mode stream and an L1 leaf-tiled one (ktile > 0) give the result of the
    untiled build, over two outer iterations, to 1e-12 or to ten times the untiled run's own
    spread under a 1e-14 relative change of the start, whichever is larger (the atomics reorder
    the sums, and a Newton step magnifies rounding by the row Hessian's condition)."""
    dims, inds, vals = random_coo((300, 200, 400), 120000, seed=5, unique=False)
    vals = np.floor(vals * 4.0) + 1.0
    f0 = start(dims, R)
    U = S.Tensor.from_coo(dims, inds, vals, ktile=-1)
    bl, bf, bh, _ = U.cp_apr_pdnr(R, _cuda(f0), niters=2, tol=0.0, max_inner=4)
    pl, pf, _, _ = U.cp_apr_pdnr(R, _cuda(_perturbed(f0)), niters=2, tol=0.0, max_inner=4)
    bar = max(1e-12, 10 * max([rel_fro(pl, bl)] + [rel_fro(a, b) for a, b in zip(_np(pf), _np(bf))]))
    assert bar < 1e-9, bar                               # the problem is well conditioned
    assert not _grad_kernels(lambda: U.cp_apr_pdnr(R, _cuda(f0), niters=1, max_inner=1)) & {"true"}
    for path in ("cta", "ktile"):
        T = _tiled(S, monkeypatch, dims, inds, vals, path, R)
        assert _grad_kernels(lambda: T.cp_apr_pdnr(R, _cuda(f0), niters=1, max_inner=1)) == {"true"}, path
        lam, got, hist, _ = T.cp_apr_pdnr(R, _cuda(f0), niters=2, tol=0.0, max_inner=4)
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
    l1, f1, h1, i1 = T.cp_apr_pdnr(17, _cuda(f0), niters=3, tol=1e-3)
    l2, f2, h2, i2 = T.cp_apr_pdnr(17, _cuda(f0), niters=3, tol=1e-3)
    assert i1 == i2 and np.array_equal(l1, l2) and np.array_equal(h1[:, 1:], h2[:, 1:])
    for a, b in zip(f1, f2):
        assert np.array_equal(a.cpu().numpy().view(np.int64), b.cpu().numpy().view(np.int64))


@pytest.mark.gpu
def test_history_matches_oracle_and_ll_ascends(S):
    """Several outer iterations with tol > 0: the log-likelihood never decreases (1e-12
    relative), matches the oracle's to 1e-9, and the lockstep and step counts are the oracle's."""
    dims, inds, vals = problem((40, 30, 50), 6000, seed=11)
    R, tol = 6, 1e-3
    f0 = start(dims, R)
    T = S.Tensor.from_coo(dims, inds, vals)
    wl, wf, wh, info = O.cp_apr_pdnr(dims, inds, vals, f0, 6, tol, max_inner=4)
    lam, got, hist, its = T.cp_apr_pdnr(R, _cuda(f0), niters=6, tol=tol, max_inner=4)
    assert np.all(np.diff(hist[:, 0]) >= -1e-12 * np.abs(hist[:-1, 0])), hist[:, 0]
    assert its == len(wh)
    np.testing.assert_allclose(hist[:, 0], wh[:, 0], rtol=1e-9)
    assert np.array_equal(hist[:, 2:], wh[:, 2:]), (hist, wh)
    assert len(set(wh[:, 3])) > 1                      # the counts vary, so the test means something


@pytest.mark.gpu
@pytest.mark.parametrize("n", [2, 3, 5, 8])
def test_rank1_closed_form(S, n):
    dims, inds, vals = problem(DIMS[n], 2500, seed=n)
    T = S.Tensor.from_coo(dims, inds, vals)
    tot, want = marginals(dims, inds, vals)
    lam, got, hist, its = T.cp_apr_pdnr(1, _cuda(start(dims, 1)), niters=1, tol=0.0, max_inner=20)
    assert abs(lam[0] - tot) <= 1e-12 * tot
    for g, w in zip(_np(got), want):
        assert rel_fro(g, w) < 1e-12
    T.free()


@pytest.mark.gpu
def test_planted_model_recovered_faster_than_mu(S):
    dims, inds, vals, F = planted()
    f0 = [np.random.default_rng(4).uniform(0.1, 1.0, (d, 3)) for d in dims]
    T = S.Tensor.from_coo(dims, inds, vals)
    lam, got, hist, its = T.cp_apr_pdnr(3, _cuda(f0), niters=PDNR_PLANTED_ITERS, tol=1e-4)
    assert hist[-1, 1] < 1e-4 and its < PDNR_PLANTED_ITERS, hist
    assert congruence(F, _np(got)) >= 0.99
    for g in _np(got):
        np.testing.assert_allclose(g.sum(axis=0), 1.0, rtol=1e-12)
        assert (g >= 0).all()
    _, _, hm, itm = T.cp_apr(3, _cuda(f0), niters=its, tol=1e-4)
    assert hm[-1, 1] >= 1e-4                           # MU has not converged in as many


@pytest.mark.gpu
def test_fallback_and_failed_line_search_match_oracle(S):
    """A zero start row with eps = 1e-200: its Hessian overflows, the Cholesky falls back to
    d = -g, and no trial point passes; the run still matches the oracle."""
    dims, inds, vals, f0, kw = _fallback_problem()
    wl, wf, wh, info = O.cp_apr_pdnr(dims, inds, vals, f0, 1, 0.0, **kw)
    assert any(r["fallbacks"] > 0 and -1 in r["ks"] for r in info["rows"])
    T = S.Tensor.from_coo(dims, inds, vals)
    lam, got, hist, its = T.cp_apr_pdnr(4, _cuda(f0), niters=1, tol=0.0, max_inner=kw["max_inner"],
                                        eps=kw["eps"])
    assert rel_fro(lam, wl) < 1e-10
    for m in range(3):
        assert rel_fro(_np(got)[m], wf[m]) < 1e-10, m


def _raw(T, R, ldm, opts, bufs, po=None):
    import torch
    torch.cuda.synchronize()
    ptrs = (A.val_p * len(bufs))(*[C.cast(C.c_void_p(b.data_ptr()), A.val_p) for b in bufs])
    lam = np.zeros(max(R, 1))
    hist = np.zeros(4 * 4)
    its = C.c_int()
    rc = T.lib.splatt_b200_cp_apr_pdnr_device(T.h, R, ldm, opts.ctypes.data_as(C.POINTER(C.c_double)),
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
    for po in (A.PdnrOpts(0, 8, 1e-5, 1e-8, 1e-10), A.PdnrOpts(10, 0, 1e-5, 1e-8, 1e-10),
               A.PdnrOpts(10, 9, 1e-5, 1e-8, 1e-10), A.PdnrOpts(10, 8, 0.0, 1e-8, 1e-10),
               A.PdnrOpts(10, 8, -1e-5, 1e-8, 1e-10), A.PdnrOpts(10, 8, nan, 1e-8, 1e-10),
               A.PdnrOpts(10, 8, inf, 1e-8, 1e-10), A.PdnrOpts(10, 8, 1e-5, -1e-8, 1e-10),
               A.PdnrOpts(10, 8, 1e-5, nan, 1e-10), A.PdnrOpts(10, 8, 1e-5, 1e-8, 0.0),
               A.PdnrOpts(10, 8, 1e-5, 1e-8, nan)):
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
        T.cp_apr_pdnr(4, [torch.rand((d, 4), dtype=torch.float32, device="cuda") for d in dims])
    with pytest.raises(ValueError):
        T.cp_apr_pdnr(4, [torch.rand((d, 5), dtype=torch.float64, device="cuda") for d in dims])
    with pytest.raises(ValueError):
        T.cp_apr_pdnr(4, [torch.rand((d, 4), dtype=torch.float64) for d in dims])
    with pytest.raises(S.SplattError):
        T.cp_apr_pdnr(65)
    with pytest.raises(S.SplattError):
        T.cp_apr_pdnr(4, max_backtrack=9)
    l1, f1, h1, i1 = T.cp_apr_pdnr(4, niters=3, seed=9)
    l2, f2, h2, i2 = T.cp_apr_pdnr(4, niters=3, seed=9)
    assert i1 == i2 and np.array_equal(l1, l2)
    assert all(torch.equal(a, b) for a, b in zip(f1, f2))
    assert h1.shape == (i1, 4)


# At scale: the tensors of tests/test_walk_at_scale.py (6 M records: every warp's record ring
# wraps; n3's mode 0 is Zipf-skewed, its hottest row spanning hundreds of ranges).  (name, R,
# whether the layout has rows finished in the gradient walk)
AT_SCALE = [("n3", 16, True), ("n2", 32, True), ("n4", 33, False)]
AT_SCALE_INNER = 5


def _sample_rows(cnt, R, rng, k=12):
    """The hottest row, the empty rows, the row of median count and k random rows with at least
    4 R records (well-conditioned Hessians)."""
    cnt = np.asarray(cnt)
    rows = {int(cnt.argmax())} | set(np.nonzero(cnt == 0)[0][:3].tolist())
    nz = np.nonzero(cnt > 0)[0]
    rows.add(int(nz[np.argsort(cnt[nz], kind="stable")[len(nz) // 2]]))
    good = np.nonzero(cnt >= 4 * R)[0]
    if len(good):
        rows |= set(rng.choice(good, size=min(k, len(good)), replace=False).tolist())
    return sorted(rows)


@pytest.mark.gpu
@pytest.mark.parametrize("name,R,whole", AT_SCALE, ids=[f"{n}-R{r}" for n, r, _ in AT_SCALE])
def test_cp_apr_pdnr_at_scale(S, scale, name, R, whole):
    """One Tensor.cp_apr_pdnr outer iteration with tol = 0 on a tensor that wraps every warp's
    record ring, bitwise the same on a second run, checked mode by mode on sampled rows (the
    hottest, the empty ones, the median one and random ones) against oracle.apr_pdnr's
    row_subproblem run on the rows the device saw.  Mode n's rows start from the normalised start
    times the column sums of mode n - 1's B and use the returned factors of modes < n; the
    device returns B_n normalised, so each sampled row must equal the oracle's up to one scale
    per column, fitted on the sample (the last mode's scale is the returned lambda itself), to
    1e-8 relative per row."""
    import torch
    dims, idx, vals, T = scale(name)
    assert_ring_wraps(T)
    N = len(dims)
    g = torch.Generator(device="cuda").manual_seed(R)
    f0 = [torch.rand((d, R), dtype=torch.float64, device="cuda", generator=g) for d in dims]
    lam, got, hist, its = T.cp_apr_pdnr(R, f0, niters=1, tol=0.0, max_inner=AT_SCALE_INNER)
    assert its == 1 and hist[0, 2] == AT_SCALE_INNER * N and hist[0, 3] == AT_SCALE_INNER * sum(dims)
    lam2, got2, hist2, _ = T.cp_apr_pdnr(R, f0, niters=1, tol=0.0, max_inner=AT_SCALE_INNER)
    assert np.array_equal(lam.view(np.int64), lam2.view(np.int64))
    assert np.array_equal(hist[:, 1:], hist2[:, 1:])
    for a, b in zip(got, got2):
        assert torch.equal(bits(a), bits(b))
    del got2
    cnts = [torch.bincount(i, minlength=d).cpu().numpy() for i, d in zip(idx, dims)]
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    kinds = [slice_kinds(c, grad_warps(R, sms)) for c in cnts]
    assert sum(c for _, c in kinds) > 0 and (sum(w for w, _ in kinds) > 0) == whole, kinds
    s0 = [f.sum(dim=0) for f in f0]
    cur = [f / s for f, s in zip(f0, s0)]                 # the factors as mode n sees them
    scale_in = torch.stack(s0).prod(dim=0)                # lambda entering mode 0
    rng = np.random.default_rng(R)
    for n in range(N):
        b_start = (cur[n] * scale_in).cpu().numpy()
        rows = _sample_rows(cnts[n], R, rng)
        want, dev = [], []
        for i in rows:
            sel = (idx[n] == i).nonzero().squeeze(1)
            Pi = torch.ones((len(sel), R), dtype=torch.float64, device="cuda")
            for m in range(N):
                if m != n:
                    Pi *= cur[m][idx[m][sel]]
            b, _ = O.row_subproblem(b_start[i], Pi.cpu().numpy(), vals[sel].cpu().numpy(), 0.0,
                                    max_inner=AT_SCALE_INNER)
            want.append(b)
            dev.append(got[n][i].cpu().numpy())
        want, dev = np.array(want), np.array(dev)
        if n == N - 1:
            c = lam.copy()
        else:
            den = dev.sum(axis=0)
            c = np.where(den > 0, want.sum(axis=0) / np.where(den > 0, den, 1.0), 1.0)
        err = np.abs(dev * c[None, :] - want).max(axis=1) / np.maximum(np.abs(want).max(axis=1), 1e-300)
        err[np.abs(want).max(axis=1) == 0] = np.abs(dev[np.abs(want).max(axis=1) == 0]).max(axis=1)
        assert err.max() < 1e-8, (name, n, [(r, e) for r, e in zip(rows, err) if e >= 1e-8][:5])
        cur[n] = got[n]
        scale_in = torch.from_numpy(c).cuda()
