"""Completion, CP-APR, Tucker's TTMc and the model sums on tensors large enough that every warp's
record range wraps its TMA ring (walk.cuh) many times.

The kernels that walk a root stream with walk_range / walk_levels give each warp an nnz-balanced
range of 64-record chunks and stream it through a private ring of kStages = 3 stages of
kStageRecs = 128 records.  They launch at least 132 SMs x 8 warps, so a tensor of a few ten
thousand records gives every warp one chunk and never fills a second stage.  The tensors here
have about 6 M records (10 M for the default-tiling case): with TG_max = 64 x SMs resident warps
every stream has nchunks >= 8 TG_max, so each warp's range holds at least 512 records (4 stages)
whatever occupancy the library picks.  Every GPU test asserts that at run time.

The references are torch fp64 restatements of each operation (device-agnostic, records processed
in chunks of at most ~2 GB of temporaries) that also return the "absolute" version of what they
compute: the same formula on |v| and |U|.  The CPU tests pin them to the numpy oracle (oracle/tc.py,
oracle/apr.py, oracle/tucker.py) on small tensors with duplicates and empty rows, so the GPU checks
inherit the oracle's pinning.  Every GPU check is elementwise or per row and holds for any
summation order, with gamma(k) = k u / (1 - k u), u = 2^-53; each test also recomputes its
reference with one record of the hottest row removed and requires the same comparison to fail by
at least 100x, so the bound is tight enough to see one dropped or doubled record.
"""
from __future__ import annotations

import ctypes as C
import math
import time
import zlib

import numpy as np
import pytest

from oracle import apr as OA
from oracle import tc as OT
from oracle import tucker as OK
from splatt_b200 import _abi as A

torch = pytest.importorskip("torch")

U_RND = 2.0 ** -53
BUDGET = 2 ** 31               # bytes of one per-record temporary of a reference
H100_SMS = 132
RING_CHUNK = 64                # records per chunk of the stream format
MAX_INNER = 10                 # CP-APR inner updates per mode (the library's default)
EPS = 1e-10                    # CP-APR floor of the model value
MARGIN = 100.0                 # a dropped record must exceed the bound by this factor
_SEEN = {"bound": [], "dropped": []}   # err / bound of this test's checks and of its mutation


def gamma(k):
    return k * U_RND / (1.0 - k * U_RND)


# ---------------------------------------------------------------------------------------
# The case table
# ---------------------------------------------------------------------------------------
# name: (dims before three empty rows are added to every mode, records, Zipf exponent per mode
# (0: uniform)).  n3: mode 0 is Zipf-skewed (its hottest row holds ~1/5 of the records and
# spans ~20 % of the warps' ranges), mode 1 has a median slice of ~300 records (whole slices
# inside one range that still cross stage boundaries).
SCALE = {
    "n2": ((40_000, 30_000), 6_000_000, (0, 0)),
    "n3": ((50_000, 20_000, 3_000), 6_000_000, (1.2, 0, 0)),
    "n4": ((200, 150, 120, 100), 6_000_000, (0, 0, 0, 0)),
    "n8": ((10,) * 8, 6_000_000, (0,) * 8),
}
MEDIAN_MODE = ("n3", 1)
# Tucker TTMc rank sets: on N = 3 the register tiles TT = 2, 8, 32 (C = 64, 256, 1024); N = 4 takes
# the emap / A path
TTMC = {"n2": [(5, 32)], "n3": [(8, 8, 8), (16, 16, 16), (32, 32, 32)], "n4": [(6, 5, 4, 3)],
        "n8": [(2, 3, 2, 1, 2, 2, 3, 2)]}
COMPLETE = [("n3", 16), ("n3", 32), ("n3", 64), ("n2", 16), ("n4", 16), ("n8", 16)]
APR = [("n3", 16), ("n4", 5)]
TUCKER = ("n3", (8, 8, 8))
SSE_RANK = 7
TILING = ((10_000,) * 3, 10_000_000)     # configuration-2 density, tiled by the default rules


def ttmc_tile(C_):
    return 2 if C_ <= 64 else 8 if C_ <= 256 else 32


def rank_tier(R):
    return 16 if R <= 16 else 32 if R <= 32 else 64


# ---------------------------------------------------------------------------------------
# torch fp64 restatements (any device)
# ---------------------------------------------------------------------------------------
def _steps(n, width):
    """[lo, hi) record chunks with at most BUDGET bytes of `width` doubles per record."""
    step = max(1, BUDGET // (8 * max(1, width)))
    return [(lo, min(n, lo + step)) for lo in range(0, n, step)]


def _by_row(nrows, idx, vals, m, width, shapes, make):
    """Sums per row of mode m the per-record tensors make(idx_chunk, vals_chunk) returns (a list,
    entry k of shape (records,) + shapes[k]).  Records are sorted by row and each chunk is reduced
    by segments, so no output row takes more than one addition per chunk.  Returns (sums, the
    records per row)."""
    order = torch.argsort(idx[m], stable=True)
    sidx = [i[order] for i in idx]
    svals = vals[order]
    acc = [torch.zeros((nrows,) + tuple(s), dtype=torch.float64, device=vals.device) for s in shapes]
    for lo, hi in _steps(len(svals), width):
        parts = make([i[lo:hi] for i in sidx], svals[lo:hi])
        rows, cnt = torch.unique_consecutive(sidx[m][lo:hi], return_counts=True)
        for a, p in zip(acc, parts):
            a.index_add_(0, rows, torch.segment_reduce(p, "sum", lengths=cnt, axis=0))
    return acc, torch.bincount(idx[m], minlength=nrows)


def ref_sse(idx, vals, mats, lam=None):
    """(sum_x (v - x)^2, sum_x |v - x| x^), x = sum_r lam_r prod_m U_m[i_m, r] and x^ the same on
    |lam| and |U|: (v - x)^2 moves by 2 |v - x| dx at first order, |dx| <= gamma(R + N) x^."""
    R = mats[0].shape[1]
    lt = torch.ones(R, dtype=torch.float64, device=vals.device) if lam is None else \
        torch.as_tensor(np.asarray(lam, dtype=np.float64), device=vals.device)
    s = torch.zeros((), dtype=torch.float64, device=vals.device)
    a = torch.zeros_like(s)
    for lo, hi in _steps(len(vals), 4 * R):
        P = lt[None, :].repeat(hi - lo, 1)
        Pa = P.abs()
        for m, M in enumerate(mats):
            rows = M[idx[m][lo:hi]]
            P *= rows
            Pa *= rows.abs()
        r = vals[lo:hi] - P.sum(1)
        s += (r * r).sum()
        a += (r.abs() * Pa.sum(1)).sum()
    return float(s), float(a)


def ref_ttmc(nrows, idx, vals, mats, n, ranks):
    """(Y_n, the same on |v| and |U|, records per row): Y_n = X_(n) (kron_{m != n} U_m[:, :ranks[m]]),
    the other modes in increasing order with the highest fastest (oracle.tucker.ttmc)."""
    N = len(idx)
    C_ = int(np.prod([r for m, r in enumerate(ranks) if m != n]))

    def make(ix, v):
        K, Ka = v[:, None], v.abs()[:, None]
        for m in range(N):
            if m == n:
                continue
            Um = mats[m][:, :ranks[m]][ix[m]]
            K = (K[:, :, None] * Um[:, None, :]).reshape(len(v), -1)
            Ka = (Ka[:, :, None] * Um.abs()[:, None, :]).reshape(len(v), -1)
        return [K, Ka]
    (Y, Ya), cnt = _by_row(nrows, idx, vals, n, 4 * C_, [(C_,), (C_,)], make)
    return Y, Ya, cnt


def tc_systems(nrows, idx, vals, mats, m, reg):
    """One row update of completion: per row i of mode m the Gram G_i = H_i^T H_i + reg I and
    right-hand side b_i = H_i^T v_i (H_i: the Hadamard products h_x of the other modes' rows at
    the row's records), and |H_i|^T |H_i| + reg I, |H_i|^T |v_i|.  Returns (G, b, Ga, ba, records
    per row).  mats[m] is not read."""
    R = next(M.shape[1] for k, M in enumerate(mats) if k != m)

    def make(ix, v):
        h = torch.ones((len(v), R), dtype=torch.float64, device=v.device)
        for k, M in enumerate(mats):
            if k != m:
                h *= M[ix[k]]
        ha = h.abs()
        return [h[:, :, None] * h[:, None, :], v[:, None] * h,
                ha[:, :, None] * ha[:, None, :], v.abs()[:, None] * ha]
    (G, b, Ga, ba), cnt = _by_row(nrows, idx, vals, m, 2 * R * R + 4 * R, [(R, R), (R,), (R, R), (R,)],
                                  make)
    eye = reg * torch.eye(R, dtype=torch.float64, device=vals.device)
    return G + eye, b, Ga + eye, ba, cnt


def tc_sweep(dims, idx, vals, factors, reg):
    """One completion iteration (modes in order, every row by a dense solve of its system)."""
    f = [x.clone() for x in factors]
    for m in range(len(dims)):
        G, b, _, _, cnt = tc_systems(dims[m], idx, vals, f, m, reg)
        u = torch.zeros_like(f[m])
        rows = (cnt > 0).nonzero().squeeze(1)
        u[rows] = torch.linalg.solve(G[rows], b[rows][:, :, None]).squeeze(2)
        f[m] = u
    return f


def _normalize(M):
    s = M.sum(0)
    return torch.where(s[None, :] > 0, M / torch.where(s > 0, s, 1.0)[None, :], 0.0), s


def apr_phi(nrows, idx, vals, A_, B, n, eps=EPS):
    """Phi_n[i] = sum over the records x of row i of (v_x / max(B[i] . Pi_x, eps)) Pi_x."""
    R = B.shape[1]

    def make(ix, v):
        Pi = torch.ones((len(v), R), dtype=torch.float64, device=v.device)
        for k, M in enumerate(A_):
            if k != n:
                Pi *= M[ix[k]]
        w = v / torch.clamp_min((B[ix[n]] * Pi).sum(1), eps)
        return [w[:, None] * Pi]
    (phi,), _ = _by_row(nrows, idx, vals, n, 3 * R, [(R,)], make)
    return phi


def apr_loglik(idx, vals, A_, lam, eps=EPS):
    """(sum_x v log max(m_x, eps) - sum_r lam_r, sum_x |v log max(m_x, eps)|, sum_x |v|, sum_r |lam_r|)."""
    R = A_[0].shape[1]
    lt = torch.as_tensor(np.asarray(lam, dtype=np.float64), device=vals.device)
    s = torch.zeros((), dtype=torch.float64, device=vals.device)
    sa, sv = torch.zeros_like(s), torch.zeros_like(s)
    for lo, hi in _steps(len(vals), 3 * R):
        P = lt[None, :].repeat(hi - lo, 1)
        for m, M in enumerate(A_):
            P *= M[idx[m][lo:hi]]
        t = vals[lo:hi] * torch.log(torch.clamp_min(P.sum(1), eps))
        s += t.sum()
        sa += t.abs().sum()
        sv += vals[lo:hi].abs().sum()
    return float(s) - float(lt.sum()), float(sa), float(sv), float(lt.abs().sum())


def apr_outer(dims, idx, vals, factors, max_inner=MAX_INNER, eps=EPS):
    """One CP-APR outer iteration from `factors` (the first: no shift) with every inner update
    run: columns normalised (lam = the product of the column sums), then per mode max_inner
    times B <- B * Phi and the normalisation.  Returns (lam, factors, log-likelihood and its
    absolute version sum |v log m| + sum |lam|).  Every term is nonnegative, so lam and the
    factors are their own absolute versions."""
    A_, lam = [], torch.ones(factors[0].shape[1], dtype=torch.float64, device=vals.device)
    for Uf in factors:
        a, s = _normalize(Uf)
        A_.append(a)
        lam = lam * s
    for n in range(len(dims)):
        B = A_[n] * lam[None, :]
        for _ in range(max_inner):
            B = B * apr_phi(dims[n], idx, vals, A_, B, n, eps)
        A_[n], lam = _normalize(B)
    ll, lla, _, laml = apr_loglik(idx, vals, A_, lam.cpu().numpy(), eps)
    return lam, A_, ll, lla + laml


def tucker_core(dims, idx, vals, factors):
    """(G, Gn): the core G = X x_0 U_0^T ... x_{N-1} U_{N-1}^T (shape: the ranks) and, per entry of
    the first N-1 modes' index, Gn = sum_i |X|-TTMc[i, c] ||U_{N-1}[i, :]||_2 -- the absolute
    version with the last factor's rows measured by their 2-norm, since the device forms the core
    through a rotation of that factor's columns."""
    N = len(dims)
    ranks = [f.shape[1] for f in factors]
    Y, Ya, _ = ref_ttmc(dims[N - 1], idx, vals, factors, N - 1, ranks)
    Ul = factors[N - 1]
    return (Y.T @ Ul).reshape(ranks), Ya.T @ torch.linalg.vector_norm(Ul, dim=1)


# ---------------------------------------------------------------------------------------
# CPU: the restatements against the numpy oracle, and the case table
# ---------------------------------------------------------------------------------------
def small_problem(dims, nnz, seed):
    """Counts 1..5 at random coordinates, rows 0, d // 2 and d - 1 of every mode empty, 25
    duplicated coordinates."""
    rng = np.random.default_rng(seed)
    inds = []
    for d in dims:
        allowed = np.setdiff1d(np.arange(d), [0, d // 2, d - 1])
        inds.append(rng.choice(allowed, size=nnz))
    dup = rng.integers(0, nnz, size=25)
    inds = [np.concatenate([i, i[dup]]).astype(np.uint64) for i in inds]
    vals = rng.integers(1, 6, size=nnz + 25).astype(np.float64)
    return list(dims), inds, vals


def _t(inds, vals):
    return [torch.from_numpy(i.astype(np.int64)) for i in inds], torch.from_numpy(vals)


def _close(got, want):
    got = got.numpy() if isinstance(got, torch.Tensor) else np.asarray(got)
    want = np.asarray(want)
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12 * max(np.abs(want).max(), 1e-300))


SMALL = {2: (14, 11), 3: (9, 7, 8), 4: (6, 7, 5, 6)}


@pytest.mark.parametrize("N", sorted(SMALL))
def test_restatements_match_oracle(N):
    """SSE, TTMc, one completion sweep, one CP-APR outer iteration and the Tucker core, and each
    one's absolute version, equal the numpy oracle to 1e-12 (duplicates, empty rows)."""
    dims, inds, vals = small_problem(SMALL[N], 300, seed=N)
    idx, v = _t(inds, vals)
    rng = np.random.default_rng(10 + N)
    R = 3
    f = [rng.uniform(-1, 1, (d, R)) for d in dims]
    ft = [torch.from_numpy(x) for x in f]
    absf = [np.abs(x) for x in f]
    lam = np.array([0.5, 2.0, 1.25])
    # SSE
    for lm in (None, lam):
        s, sa = ref_sse(idx, v, ft, lm)
        _close(s, OT.sse(inds, vals, f, lm))
        x = OT.model_values(inds, f, lm)
        xa = OT.model_values(inds, absf, None if lm is None else np.abs(lm))
        _close(sa, np.sum(np.abs(vals - x) * xa))
    # TTMc
    ranks = [2, 3, 1, 2][:N]
    for n in range(N):
        Y, Ya, cnt = ref_ttmc(dims[n], idx, v, ft, n, ranks)
        _close(Y, OK.ttmc(dims, inds, vals, f, n, ranks))
        _close(Ya, OK.ttmc(dims, inds, np.abs(vals), absf, n, ranks))
        assert np.array_equal(cnt.numpy(), np.bincount(inds[n].astype(np.int64), minlength=dims[n]))
    # completion: the systems and their absolute versions, and one sweep
    reg = 0.3
    f0 = [rng.uniform(0, 1, (d, R)) for d in dims]
    for m in range(N):
        G, b, Ga, ba, _ = tc_systems(dims[m], idx, v, [torch.from_numpy(x) for x in f0], m, reg)
        for i, (H, y) in enumerate(OT.row_systems(dims, inds, vals, f0, m)):
            _close(G[i], H.T @ H + reg * np.eye(R))
            _close(b[i], H.T @ y)
            _close(Ga[i], np.abs(H).T @ np.abs(H) + reg * np.eye(R))
            _close(ba[i], np.abs(H).T @ np.abs(y))
    got = tc_sweep(dims, idx, v, [torch.from_numpy(x) for x in f0], reg)
    for g, w in zip(got, OT.sweep(dims, inds, vals, f0, reg)):
        _close(g, w)
    # CP-APR
    wl, wf, wh, _ = OA.cp_apr(dims, inds, vals, f0, 1, 0.0)
    lam_t, A_t, ll, lla = apr_outer(dims, idx, v, [torch.from_numpy(x) for x in f0])
    _close(lam_t, wl)
    for g, w in zip(A_t, wf):
        _close(g, w)
    _close(ll, wh[0, 0])
    mv = OA.model_values(inds, wf, wl)
    _close(lla, np.sum(np.abs(vals * np.log(np.maximum(mv, EPS)))) + np.sum(np.abs(wl)))
    # Tucker core
    tr = [2, 3, 2, 2][:N]
    F = [np.linalg.qr(rng.standard_normal((d, r)))[0] for d, r in zip(dims, tr)]
    G, Gn = tucker_core(dims, idx, v, [torch.from_numpy(x) for x in F])
    _close(G, (OK.ttmc(dims, inds, vals, F, N - 1, tr).T @ F[N - 1]).reshape(tr))
    _close(Gn, OK.ttmc(dims, inds, np.abs(vals), [np.abs(x) for x in F], N - 1, tr).T @
           np.linalg.norm(F[N - 1], axis=1))


def test_case_table():
    """Every scale tensor wraps the ring at 132 SMs (nchunks >= 8 x 64 x SMs), and the table
    reaches N = 2, 3, 4, 8, a Zipf mode of exponent ~1.2 on N = 3, a mode whose slices hold
    200-400 records, the TTMc tiles 2 / 8 / 32 on N = 3 plus N = 4 and N = 8 rank sets, every
    completion rank tier on N = 3 and R = 16 on N = 2, 4, 8."""
    for name, (dims, nnz, skew) in SCALE.items():
        assert -(-nnz // RING_CHUNK) >= 8 * 64 * H100_SMS, name
        assert len(dims) == len(skew) == int(name[1:])
    assert -(-TILING[1] // RING_CHUNK) >= 8 * 64 * H100_SMS
    assert {len(d) for d, _, _ in SCALE.values()} == {2, 3, 4, 8}
    assert 1.1 <= max(SCALE["n3"][2]) <= 1.3
    name, m = MEDIAN_MODE
    dims, nnz, skew = SCALE[name]
    assert not skew[m] and 200 <= nnz / dims[m] <= 400
    for name, sets in TTMC.items():
        dims = [d + 3 for d in SCALE[name][0]]
        for ranks in sets:
            assert len(ranks) == len(dims) and all(1 <= r <= min(32, d) for r, d in zip(ranks, dims))
            assert all(int(np.prod(ranks)) // r <= 1024 for r in ranks)
    tiles = {ttmc_tile(int(np.prod(r)) // r[n]) for r in TTMC["n3"] for n in range(3)}
    assert tiles == {2, 8, 32}
    assert TTMC["n4"] and TTMC["n8"]
    assert {rank_tier(R) for name, R in COMPLETE if name == "n3"} == {16, 32, 64}
    assert {name for name, R in COMPLETE if R == 16} == {"n2", "n3", "n4", "n8"}
    assert "n3" in {n for n, _ in APR} and TUCKER[0] == "n3"      # both see the Zipf row


# ---------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def S():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import splatt_b200 as S
    return S


@pytest.fixture(autouse=True)
def _cost(request):
    """Prints each test's wall time and peak torch allocation (run with -s to see them)."""
    gpu = torch.cuda.is_available()
    if gpu:
        torch.cuda.reset_peak_memory_stats()
    for v in _SEEN.values():
        v.clear()
    t0 = time.perf_counter()
    yield
    if gpu:
        torch.cuda.synchronize()
        worst = max(_SEEN["bound"], default=float("nan"))
        weakest = min(_SEEN["dropped"], default=float("nan"))
        print(f"\n[cost] {request.node.name}: {time.perf_counter() - t0:.1f} s, "
              f"max_memory_allocated {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB, "
              f"largest err/bound {worst:.3g}, dropped record at {weakest:.3g} x bound")


def device_coo(dims, nnz, skew, seed):
    """Seeded COO on the device: Zipf(s) or uniform indices, the last 1000 records duplicating
    the coordinates of the first 1000, counts 1..5, and rows 0, d // 2 + 1 and d + 2 of every
    mode left empty (dims grow by 3).  Returns (dims, int32 indices, int64 indices, values)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    ind = []
    for d, s in zip(dims, skew):
        if s:
            p = torch.arange(1, d + 1, dtype=torch.float64, device="cuda") ** -s
            i = torch.multinomial(p, nnz, replacement=True, generator=g)
        else:
            i = torch.randint(0, d, (nnz,), device="cuda", generator=g)
        i[-1000:] = i[:1000]
        ind.append(torch.where(i < d // 2, i + 1, i + 2))
    vals = torch.randint(1, 6, (nnz,), device="cuda", generator=g).to(torch.float64)
    return [d + 3 for d in dims], [i.to(torch.int32) for i in ind], ind, vals


@pytest.fixture(scope="module")
def scale(S):
    """name -> (dims, int64 indices, values, untiled Tensor), built once per module."""
    cache = {}

    def get(name):
        if name not in cache:
            dims, nnz, skew = SCALE[name]
            dims, i32, idx, vals = device_coo(dims, nnz, skew, zlib.crc32(name.encode()))
            check_shape(name, idx)
            cache[name] = (dims, idx, vals, S.Tensor.from_coo(dims, i32, vals, ktile=-1))
        return cache[name]
    yield get
    for *_, T in cache.values():
        T.free()
    cache.clear()
    torch.cuda.empty_cache()


def check_shape(name, idx):
    """The table's slice shapes on the generated tensor: the median slice of MEDIAN_MODE holds
    200-400 records, and a Zipf mode's hottest row spans at least 16 warps' ranges even at the
    longest ranges (one CTA of 8 warps per SM)."""
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    cnt = [torch.bincount(i) for i in idx]
    if name == MEDIAN_MODE[0]:
        c = cnt[MEDIAN_MODE[1]]
        med = float(c[c > 0].median())
        assert 200 <= med <= 400, med
    per_warp = -(-len(idx[0]) // (RING_CHUNK * 8 * sms)) * RING_CHUNK
    for m, s in enumerate(SCALE[name][2]):
        if s:
            assert int(cnt[m].max()) >= 16 * per_warp, (name, m, int(cnt[m].max()), per_warp)


def assert_ring_wraps(T):
    """Every stream has nchunks >= 8 x 64 x SMs: each warp's range spans >= 4 ring stages at
    any occupancy."""
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    for m in range(T.nmodes):
        nrec = T.mode_info(m, 1)["nfibs"][-1]
        nchunks = -(-nrec // RING_CHUNK)
        assert nchunks >= 8 * 64 * sms, (m, nrec, nchunks, sms)


def ratio(err, bound):
    """max err / bound (0 / 0 = 0; NaN counts as infinitely out of bound)."""
    r = torch.where(err == 0, torch.zeros_like(err), err / bound)
    return float(torch.nan_to_num(r, nan=math.inf).max()) if r.numel() else 0.0


def within(r, what):
    _SEEN["bound"].append(r)
    assert r <= 1.0, (what, "err / bound", r)


def sees_drop(r, what):
    _SEEN["dropped"].append(r)
    assert r >= MARGIN, (what, "a dropped record is only", r, "times the bound")


def drop(idx, vals, j):
    keep = torch.ones(len(vals), dtype=torch.bool, device=vals.device)
    keep[j] = False
    return [i[keep] for i in idx], vals[keep]


def hot_records(idx, m):
    """(hottest row of mode m, its records)."""
    cnt = torch.bincount(idx[m])
    hot = int(cnt.argmax())
    return hot, (idx[m] == hot).nonzero().squeeze(1)


def bits(t):
    return t.contiguous().view(torch.int64)


def ttmc_bound(Ya, cnt, N):
    """2 gamma(n_i + N + 1) |X|-TTMc: each entry is a sum of n_i products of N numbers, rounded
    by the kernel and by the reference in any order."""
    return 2.0 * gamma(cnt.to(torch.float64) + N + 1)[:, None] * Ya


def check_ttmc(out, Y, Ya, cnt, N, what):
    within(ratio((out - Y).abs(), ttmc_bound(Ya, cnt, N)), what)
    empty = out[cnt == 0]
    assert bool((empty == 0).all()) and not bool(empty.signbit().any()), what


def ttmc_mutation(out, dims, idx, vals, mats, n, ranks, what):
    """Drops the record of mode n's hottest row with the largest |v| prod max|U| and requires the
    TTMc comparison to fail by MARGIN."""
    hot, recs = hot_records(idx, n)
    score = vals[recs].abs()
    for m, M in enumerate(mats):
        if m != n:
            score = score * M[:, :ranks[m]].abs().amax(1)[idx[m][recs]]
    di, dv = drop(idx, vals, recs[score.argmax()])
    Y, Ya, cnt = ref_ttmc(dims[n], di, dv, mats, n, ranks)
    sees_drop(ratio((out - Y).abs(), ttmc_bound(Ya, cnt, len(dims))), what)


def run_ttmc(T, dims, n, mats, ranks):
    C_ = int(np.prod([r for m, r in enumerate(ranks) if m != n]))
    out = torch.empty((dims[n], C_), dtype=torch.float64, device="cuda")
    T.ttmc(n, [None if m == n else x for m, x in enumerate(mats)], out, ranks)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(TTMC))
def test_ttmc_at_scale(S, scale, name):
    """Tensor.ttmc of every mode at every rank set of the table, elementwise within
    2 gamma(n_i + N + 1) of the |X|-TTMc (any summation order, reference and kernel), rows without
    records exactly +0, and bitwise the same on a second run (untiled stream, boundary slots added
    in range order)."""
    dims, idx, vals, T = scale(name)
    assert_ring_wraps(T)
    N = len(dims)
    g = torch.Generator(device="cuda").manual_seed(17)
    for k, ranks in enumerate(TTMC[name]):
        mats = [torch.randn((d, r), dtype=torch.float64, device="cuda", generator=g) for d, r in zip(dims, ranks)]
        for n in range(N):
            out = run_ttmc(T, dims, n, mats, ranks)
            assert torch.equal(bits(out), bits(run_ttmc(T, dims, n, mats, ranks))), (name, ranks, n)
            Y, Ya, cnt = ref_ttmc(dims[n], idx, vals, mats, n, ranks)
            check_ttmc(out, Y, Ya, cnt, N, (name, ranks, n))
            del Y, Ya
            if k == 0 and n == 0:
                ttmc_mutation(out, dims, idx, vals, mats, n, ranks, (name, ranks, n))
            del out


def sse_raw(T, f, R, ldm, lam):
    """splatt_b200_tensor_sse on buffers whose pad columns [R, ldm) hold NaN."""
    bufs = [torch.full((x.shape[0], ldm), float("nan"), dtype=torch.float64, device="cuda") for x in f]
    for b, x in zip(bufs, f):
        b[:, :R].copy_(x)
    torch.cuda.synchronize()
    ptrs = (A.val_p * len(bufs))(*[C.cast(C.c_void_p(b.data_ptr()), A.val_p) for b in bufs])
    lam_a = None if lam is None else np.ascontiguousarray(lam, dtype=np.float64)
    out = C.c_double()
    rc = T.lib.splatt_b200_tensor_sse(T.h, R, ldm, ptrs,
                                      None if lam_a is None else lam_a.ctypes.data_as(A.val_p),
                                      C.byref(out), None)
    assert rc == A.SPLATT_SUCCESS
    return out.value


def sse_bound(s, sa, nnz, R, N):
    """2 [gamma(nnz + 2) sum (v - x)^2 + 2 gamma(R + N + 1) sum |v - x| x^]: the sum of nnz
    nonnegative terms in any order, and each term's model value x (R products of N + 1 numbers)
    moving (v - x)^2 by 2 |v - x| dx; kernel and reference."""
    return 2.0 * (gamma(nnz + 2) * s + 2.0 * gamma(R + N + 1) * sa)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(SCALE))
def test_sse_at_scale(S, scale, name):
    """Tensor.sse and the raw entry with NaN pad columns, odd rank, with and without lambda,
    against the torch fp64 sum."""
    dims, idx, vals, T = scale(name)
    assert_ring_wraps(T)
    N, R = len(dims), SSE_RANK
    g = torch.Generator(device="cuda").manual_seed(5)
    f = [torch.rand((d, R), dtype=torch.float64, device="cuda", generator=g) for d in dims]
    lam = np.linspace(0.5, 2.0, R)
    for lm in (None, lam):
        s, sa = ref_sse(idx, vals, f, lm)
        bound = sse_bound(s, sa, len(vals), R, N)
        for got in (T.sse(f, lm), sse_raw(T, f, R, R + 1, lm)):
            within(abs(got - s) / bound, (name, lm is None, got, s))
    # one record of mode 0's hottest row, the one with the largest term, dropped
    got = T.sse(f, None)
    _, recs = hot_records(idx, 0)
    x = torch.ones((len(recs), R), dtype=torch.float64, device="cuda")
    for m, M in enumerate(f):
        x *= M[idx[m][recs]]
    di, dv = drop(idx, vals, recs[((vals[recs] - x.sum(1)) ** 2).argmax()])
    s, sa = ref_sse(di, dv, f)
    sees_drop(abs(got - s) / sse_bound(s, sa, len(dv), R, N), name)


def tc_bound(cnt, N, R):
    """Per row with n_i records, multiplying ||G^_i||_inf ||u_i||_inf + ||b^_i||_inf:
    4 gamma(n_i + N + 1): G_i and b_i are sums of n_i products of <= N + 1 numbers, formed by the
    kernel and again by the reference (hats: the absolute versions); 2 R gamma(3R + 1): Cholesky
    and the two triangular solves are backward stable with |dG| <= gamma(3R + 1) |L||L^T|, whose
    entries are at most max_k G_kk; gamma(R + 1): the residual's own matrix-vector product."""
    return 4.0 * gamma(cnt.to(torch.float64) + N + 1) + 2.0 * R * gamma(3 * R + 1) + gamma(R + 1)


def tc_ratio(G, b, Ga, ba, u, cnt, N, R):
    """max over rows with records of ||G_i u_i - b_i||_inf / bound."""
    rows = cnt > 0
    res = (G[rows] @ u[rows][:, :, None]).squeeze(2) - b[rows]
    scale = Ga[rows].abs().sum(2).amax(1) * u[rows].abs().amax(1) + ba[rows].abs().amax(1)
    return ratio(res.abs().amax(1), tc_bound(cnt[rows], N, R) * scale)


def check_completion(dims, idx, vals, f0, got, reg, what, mutate=False):
    """Mode m was updated from the returned factors of modes < m and the start of modes > m: every
    row's residual in its own system is within tc_bound, rows without records are exactly 0."""
    N, R = len(dims), f0[0].shape[1]
    for m in range(N):
        mats = list(got[:m]) + [None] + list(f0[m + 1:])
        G, b, Ga, ba, cnt = tc_systems(dims[m], idx, vals, mats, m, reg)
        u = got[m]
        within(tc_ratio(G, b, Ga, ba, u, cnt, N, R), (what, m))
        assert bool((u[cnt == 0] == 0).all()), (what, m)
        del G, Ga
        if mutate and m == 0:
            # drop the hottest row's record with the largest |h|_inf |h . u - v|
            hot, recs = hot_records(idx, 0)
            h = torch.ones((len(recs), R), dtype=torch.float64, device="cuda")
            for k in range(1, N):
                h *= mats[k][idx[k][recs]]
            score = h.abs().amax(1) * ((h * u[hot]).sum(1) - vals[recs]).abs()
            di, dv = drop(idx, vals, recs[score.argmax()])
            G, b, Ga, ba, cnt = tc_systems(dims[0], di, dv, mats, 0, reg)
            sees_drop(tc_ratio(G, b, Ga, ba, u, cnt, N, R), what)
            del G, Ga


@pytest.mark.gpu
@pytest.mark.parametrize("name,R", COMPLETE, ids=[f"{n}-R{r}" for n, r in COMPLETE])
def test_completion_sweep_at_scale(S, scale, name, R):
    """One Tensor.complete iteration: every row's solve checked by its residual in the system
    rebuilt from the factors it was formed from (no dependence on conditioning), and bitwise the
    same factors on a second run."""
    dims, idx, vals, T = scale(name)
    assert_ring_wraps(T)
    g = torch.Generator(device="cuda").manual_seed(R)
    f0 = [torch.rand((d, R), dtype=torch.float64, device="cuda", generator=g) for d in dims]
    reg = 0.1
    _, got, its = T.complete(R, f0, reg=reg, niters=1)
    assert its == 1
    _, again, _ = T.complete(R, f0, reg=reg, niters=1)
    for m, (a, b) in enumerate(zip(got, again)):
        assert torch.equal(bits(a), bits(b)), (name, R, m)
    del again
    check_completion(dims, idx, vals, f0, got, reg, (name, R), mutate=True)


def apr_bound(N, R, nmax, maxdim):
    """Relative Frobenius bound of lambda and the factors after one outer iteration: every Phi
    entry is a sum of n_i nonnegative terms, each v over a dot product of R nonnegative products
    of N numbers, so it carries a relative error of at most gamma(n_max + N + R + 1); Phi is
    homogeneous of degree 0 in B and in every other factor, so the errors of the max_inner
    updates of each of the N modes add at first order; the normalisation adds gamma(dims + N)."""
    return MAX_INNER * N * gamma(nmax + N + R + 1) + 2.0 * gamma(maxdim + N)


def rel(a, b):
    return float(torch.linalg.vector_norm(a - b) / torch.linalg.vector_norm(b))


def apr_ratio(lam, facs, wl, wf, bound):
    return max([rel(lam, wl)] + [rel(a, b) for a, b in zip(facs, wf)]) / bound


@pytest.mark.gpu
@pytest.mark.parametrize("name,R", APR, ids=[f"{n}-R{r}" for n, r in APR])
def test_cp_apr_at_scale(S, scale, name, R):
    """One Tensor.cp_apr outer iteration with tol = 0 (all 10 inner updates of every mode):
    lambda and every factor against the torch restatement by relative Frobenius norm (apr_bound),
    the log-likelihood against a torch fp64 sum of the returned model, and bitwise the same lambda
    and factors on a second run."""
    dims, idx, vals, T = scale(name)
    assert_ring_wraps(T)
    N = len(dims)
    g = torch.Generator(device="cuda").manual_seed(R)
    f0 = [torch.rand((d, R), dtype=torch.float64, device="cuda", generator=g) for d in dims]
    lam, got, hist, its = T.cp_apr(R, f0, niters=1, tol=0.0, max_inner=MAX_INNER, eps=EPS)
    assert its == 1 and hist[0, 2] == MAX_INNER * N
    lam2, got2, _, _ = T.cp_apr(R, f0, niters=1, tol=0.0, max_inner=MAX_INNER, eps=EPS)
    assert np.array_equal(lam.view(np.int64), lam2.view(np.int64))
    for a, b in zip(got, got2):
        assert torch.equal(bits(a), bits(b))
    del got2
    nmax = max(int(torch.bincount(i).max()) for i in idx)
    bound = apr_bound(N, R, nmax, max(dims))
    lam_t = torch.from_numpy(lam).cuda()
    wl, wf, _, _ = apr_outer(dims, idx, vals, f0)
    within(apr_ratio(lam_t, got, wl, wf, bound), name)
    # the log-likelihood: 2 [gamma(nnz + 2) sum |v log m| + (gamma(R + N + 1) + 2u) sum |v|] +
    # gamma(R + 1) sum lam -- the sum, each term's log of a model value with relative error
    # gamma(R + N) plus the log's own rounding, kernel and reference; and sum_r lam_r
    ll, lla, sv, sl = apr_loglik(idx, vals, got, lam)
    llb = 2.0 * (gamma(len(vals) + 2) * lla + (gamma(R + N + 1) + 2 * U_RND) * sv) + gamma(R + 1) * sl
    within(abs(hist[0, 0] - ll) / llb, (name, "log-likelihood", hist[0, 0], ll))
    # one record of the hottest row (of the mode with the most records in a row) dropped
    m = max(range(N), key=lambda k: int(torch.bincount(idx[k]).max()))
    _, recs = hot_records(idx, m)
    di, dv = drop(idx, vals, recs[vals[recs].argmax()])
    wl, wf, _, _ = apr_outer(dims, di, dv, f0)
    sees_drop(apr_ratio(lam_t, got, wl, wf, bound), name)


def core_bound(Gn, nmax, N, I, R):
    """Per core entry (c, j): 4 gamma(n_max + N + I + 2R + 2) Gn[c].  The device forms
    G = (Y^T Q) V with U = Q V: Y's entries carry gamma(n_i + N + 1) |X|-TTMc, Y^T Q a sum over
    I rows, and the rotation by V R terms; sum_k |Q_ik| |V_kj| <= ||U_i||_2, so every error is
    at most gamma(.) sum_i |X|-TTMc[i, c] ||U_i||_2; the reference Y^T U adds as much again."""
    return 4.0 * gamma(nmax + N + I + 2 * R + 2) * Gn


def xnorm_sq(dims, idx, vals):
    """(||X||^2, the same of |X|) with duplicate coordinates summed."""
    key = torch.zeros_like(idx[0])
    for d, i in zip(dims, idx):
        key = key * d + i
    _, inv = torch.unique(key, return_inverse=True)
    s = torch.zeros(int(inv.max()) + 1, dtype=torch.float64, device=vals.device)
    sa = torch.zeros_like(s)
    s.index_add_(0, inv, vals)
    sa.index_add_(0, inv, vals.abs())
    return float((s * s).sum()), float((sa * sa).sum())


@pytest.mark.gpu
def test_tucker_at_scale(S, scale):
    """Two Tensor.tucker iterations: the returned core against the torch core of the returned
    factors elementwise (core_bound), the last fit against the fit recomputed from ||X||^2 and
    that core, orthonormal factors, and bitwise the same core and factors on a second run."""
    name, ranks = TUCKER
    dims, idx, vals, T = scale(name)
    assert_ring_wraps(T)
    N = len(dims)
    core, F, hist, its = T.tucker(ranks, niters=2, tol=0.0, seed=3)
    assert its == 2
    core2, F2, _, _ = T.tucker(ranks, niters=2, tol=0.0, seed=3)
    assert np.array_equal(core.view(np.int64), core2.view(np.int64))
    for a, b in zip(F, F2):
        assert torch.equal(bits(a), bits(b))
    del F2
    for f in F:
        eye = torch.eye(f.shape[1], dtype=torch.float64, device="cuda")
        assert float(torch.linalg.matrix_norm(f.T @ f - eye)) <= 1e-12
    got = torch.from_numpy(core).cuda()
    nmax = int(torch.bincount(idx[N - 1]).max())
    C_ = int(np.prod(ranks[:-1]))

    def cmp(G, Gn, nmax):
        b = core_bound(Gn, nmax, N, dims[N - 1], max(ranks))[:, None]
        return ratio((got.reshape(C_, -1) - G.reshape(C_, -1)).abs(), b)
    G, Gn = tucker_core(dims, idx, vals, F)
    within(cmp(G, Gn, nmax), "core")
    # the fit 1 - sqrt(xsq - gsq) / sqrt(xsq): the device's ||X||^2 within gamma(nnz + 2) of the
    # |X| version and its ||core||^2 within gamma(C R + 2); first order through the square roots,
    # kernel and reference, plus a few roundings of the formula
    xsq, xsa = xnorm_sq(dims, idx, vals)
    gsq = float((got * got).sum())
    D = max(xsq - gsq, 0.0)
    dx, dg = gamma(len(vals) + 2) * xsa, gamma(C_ * ranks[-1] + 2) * gsq
    fit = 1.0 - math.sqrt(D) / math.sqrt(xsq)
    fb = 2.0 * ((dx + dg) / (2.0 * math.sqrt(D * xsq)) + math.sqrt(D) * dx / (2.0 * xsq ** 1.5)) + 8 * U_RND
    within(abs(hist[-1, 0] - fit) / fb, ("fit", hist[-1, 0], fit))
    # one record of mode N-1's hottest row, the one with the largest |v| prod max|U|, dropped
    _, recs = hot_records(idx, N - 1)
    score = vals[recs].abs()
    for m, f in enumerate(F):
        score = score * f.abs().amax(1)[idx[m][recs]]
    di, dv = drop(idx, vals, recs[score.argmax()])
    G, Gn = tucker_core(dims, di, dv, F)
    sees_drop(cmp(G, Gn, int(torch.bincount(di[N - 1]).max())), "core")


def cta_policy(lib, dims, perm, nnz, sms):
    d = np.ascontiguousarray(dims, dtype=np.uint64)
    p = (C.c_int * len(dims))(*perm)
    rows, acc = C.c_uint32(), C.c_uint32()
    return lib.splatt_b200_cta_tiling(len(dims), d.ctypes.data_as(A.idx_p), p, nnz, 1, 1, sms, 0,
                                      C.byref(rows), C.byref(acc))


@pytest.mark.gpu
def test_default_tiling_at_scale(S):
    """A 3-mode tensor of configuration-2 density built with the default rules and a rank hint is
    CTA-tiled (the policy says so for every stream, and the built streams hold more fibers than the
    untiled build: leaf tiles split them).  Completion, CP-APR and TTMc on it, and on the untiled
    build of the same tensor, pass the reference checks; the two TTMc outputs agree within twice
    the bound."""
    R = 16
    dims, nnz = TILING
    dims, i32, idx, vals = device_coo(dims, nnz, (0, 0, 0), seed=2)
    Tt = S.Tensor.from_coo(dims, i32, vals, ncolumns_hint=R)
    Tu = S.Tensor.from_coo(dims, i32, vals, ktile=-1)
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    for T in (Tt, Tu):
        assert_ring_wraps(T)
    for m in range(3):
        it, iu = Tt.mode_info(m, R), Tu.mode_info(m, R)
        assert it["kind"] == "root" and cta_policy(A.load(), dims, it["level_perm"], nnz, sms) == 1, m
        assert it["nfibs"][1] > iu["nfibs"][1], (m, it["nfibs"], iu["nfibs"])
    N = 3
    g = torch.Generator(device="cuda").manual_seed(1)
    f0 = [torch.rand((d, R), dtype=torch.float64, device="cuda", generator=g) for d in dims]
    wl, wf, _, _ = apr_outer(dims, idx, vals, f0)
    bound = apr_bound(N, R, max(int(torch.bincount(i).max()) for i in idx), max(dims))
    for what, T in (("tiled", Tt), ("untiled", Tu)):
        _, got, _ = T.complete(R, f0, reg=0.1, niters=1)
        check_completion(dims, idx, vals, f0, got, 0.1, what)
        del got
        lam, got, _, _ = T.cp_apr(R, f0, niters=1, tol=0.0, max_inner=MAX_INNER, eps=EPS)
        within(apr_ratio(torch.from_numpy(lam).cuda(), got, wl, wf, bound), what)
        del got
    del wf
    ranks = (16, 16, 16)
    mats = [torch.randn((d, r), dtype=torch.float64, device="cuda", generator=g) for d, r in zip(dims, ranks)]
    for n in range(N):
        out_t = run_ttmc(Tt, dims, n, mats, ranks)
        out_u = run_ttmc(Tu, dims, n, mats, ranks)
        Y, Ya, cnt = ref_ttmc(dims[n], idx, vals, mats, n, ranks)
        check_ttmc(out_t, Y, Ya, cnt, N, ("tiled", n))
        check_ttmc(out_u, Y, Ya, cnt, N, ("untiled", n))
        within(ratio((out_t - out_u).abs(), 2.0 * ttmc_bound(Ya, cnt, N)), ("tiled - untiled", n))
        del Y, Ya, out_u
        if n == 0:
            ttmc_mutation(out_t, dims, idx, vals, mats, n, ranks, ("tiled", n))
    Tt.free()
    Tu.free()


BIG = 1 << 29                    # the largest row count the stream format holds
BIG_NEEDS = 32 * 2 ** 30


@pytest.mark.gpu
def test_largest_row_index(S):
    """dims (2^29, 2^29, 3), indices 0 and 2^29 - 1 in both large modes, 400 records, R = 1
    (ldm 2): the TTMc at ranks (1, 1, 1), the SSE and one completion sweep decode those rows and
    form their offsets right; rows no record references stay exactly 0.  (400 records cannot wrap
    the ring; this test is about the row index, not the walk.)"""
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < BIG_NEEDS:
        pytest.skip(f"needs {BIG_NEEDS / 2 ** 30:.0f} GiB of free device memory for 2^29-row fp64 "
                    f"factors and their padded copies (has {free / 2 ** 30:.1f} GiB)")
    rng = np.random.default_rng(29)
    dims = [BIG, BIG, 3]
    nnz = 400
    i0 = rng.integers(0, BIG, nnz)
    i1 = rng.integers(0, BIG, nnz)
    i0[:4] = [0, BIG - 1, BIG - 1, 0]
    i1[:4] = [BIG - 1, 0, BIG - 1, 0]
    i0[10:40] = BIG - 1                      # a row with many records at the last index
    i1[40:70] = 0
    i2 = rng.integers(0, 3, nnz)
    idx = [torch.from_numpy(i).cuda() for i in (i0, i1, i2)]
    vals = torch.from_numpy(rng.integers(1, 6, nnz).astype(np.float64)).cuda()
    T = S.Tensor.from_coo(dims, [i.to(torch.int32) for i in idx], vals)
    g = torch.Generator(device="cuda").manual_seed(3)

    def factors():
        out = []
        for d, i in zip(dims, idx):
            x = torch.zeros((d, 1), dtype=torch.float64, device="cuda")
            rows = torch.unique(i)
            x[rows, 0] = torch.rand(len(rows), dtype=torch.float64, device="cuda", generator=g) + 0.5
            out.append(x)
        return out

    def compact(m):
        """idx with mode m's rows renumbered 0 .. distinct - 1, and those rows."""
        rows, inv = torch.unique(idx[m], return_inverse=True)
        return rows, [inv if k == m else i for k, i in enumerate(idx)]

    # TTMc, ranks (1, 1, 1)
    mats = factors()
    for n in range(3):
        out = run_ttmc(T, dims, n, mats, (1, 1, 1))
        rows, cidx = compact(n)
        Y, Ya, cnt = ref_ttmc(len(rows), cidx, vals, mats, n, (1, 1, 1))
        check_ttmc(out[rows], Y, Ya, cnt, 3, ("ttmc", n))
        if n == 0:
            ttmc_mutation(out[rows], [len(rows)] + dims[1:], cidx, vals, mats, n, (1, 1, 1), "ttmc")
        out[rows] = 0.0
        assert int(torch.count_nonzero(out)) == 0, n
        del out
    # SSE
    s, sa = ref_sse(idx, vals, mats)
    within(abs(T.sse(mats) - s) / sse_bound(s, sa, nnz, 1, 3), "sse")
    torch.cuda.empty_cache()
    # one completion sweep
    reg = 0.1
    _, got, _ = T.complete(1, mats, reg=reg, niters=1)
    for m in range(3):
        rows, cidx = compact(m)
        ms = list(got[:m]) + [None] + list(mats[m + 1:])
        G, b, Ga, ba, cnt = tc_systems(len(rows), cidx, vals, ms, m, reg)
        within(tc_ratio(G, b, Ga, ba, got[m][rows], cnt, 3, 1), ("completion", m))
        if dims[m] == BIG:
            z = got[m].clone()
            z[rows] = 0.0
            assert int(torch.count_nonzero(z)) == 0, m
            del z
    del got, mats
    T.free()
    torch.cuda.empty_cache()
