"""Generalized CP decomposition (GCP) by sampled gradients and Adam, restated in numpy.

The semantics of splatt_b200_gcp_device, splatt_b200_gcp_sample and splatt_b200_gcp_sampled
(include/splatt_b200.h), written out plainly: Philox4x32-10 and the mapping of its words to
record positions and coordinates; the three losses; the weighted sampled value and gradient;
GCP-Adam with its epoch rule (accept, or revert and decay).  Stored entries are given in the
record order of the tensor's first stream, as Tensor.to_coo returns them, so record positions
drawn here name the same entries the library draws.
"""
from __future__ import annotations

import numpy as np

GAUSSIAN, BERNOULLI_LOGIT, POISSON_LOG = 0, 1, 2
LOSS_NAMES = {"gaussian": GAUSSIAN, "bernoulli-logit": BERNOULLI_LOGIT, "poisson-log": POISSON_LOG}

_M32 = np.uint64(0xFFFFFFFF)
_PM0, _PM1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_PW0, _PW1 = 0x9E3779B9, 0xBB67AE85


# ---- Philox4x32-10 ------------------------------------------------------------------------------
def philox(key, ctr):
    """Philox4x32-10 of counters ctr = (c0, c1, c2, c3) (ints or uint arrays of one shape) under
    key = (k0, k1): the four 32-bit output words, as uint64 arrays."""
    c = [np.asarray(x, dtype=np.uint64) & _M32 for x in ctr]
    c = np.broadcast_arrays(*c)
    c = [x.copy() for x in c]
    k0, k1 = int(key[0]) & 0xFFFFFFFF, int(key[1]) & 0xFFFFFFFF
    for r in range(10):
        if r:
            k0, k1 = (k0 + _PW0) & 0xFFFFFFFF, (k1 + _PW1) & 0xFFFFFFFF
        p0 = _PM0 * c[0]
        p1 = _PM1 * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ np.uint64(k0), p1 & _M32,
             (p0 >> np.uint64(32)) ^ c[3] ^ np.uint64(k1), p0 & _M32]
    return c


def mulhi64(v, n):
    """floor(v * n / 2^64) for uint64 v and 0 <= n < 2^32: a value in [0, n)."""
    v = np.asarray(v, dtype=np.uint64)
    n = np.uint64(n)
    hi, lo = v >> np.uint64(32), v & _M32
    return (hi * n + ((lo * n) >> np.uint64(32))) >> np.uint64(32)


def _word64(w, a):
    return (w[a] << np.uint64(32)) | w[a + 1]


def _key(seed):
    seed = int(seed)
    return seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF


def draw_positions(seed, t, purpose, p, nnz):
    """Record positions of p stored-entry draws of step t under `purpose` (0 or 2)."""
    j = np.arange(p, dtype=np.uint64)
    w = philox(_key(seed), (j, int(t) & 0xFFFFFFFF, int(t) >> 32, 4 * purpose))
    return mulhi64(_word64(w, 0), nnz).astype(np.int64)


def draw_coords(seed, t, purpose, q, dims):
    """[N][q] coordinates of q uniform draws of step t under `purpose` (1 or 3)."""
    j = np.arange(q, dtype=np.uint64)
    out = []
    blocks = {}
    for n, d in enumerate(dims):
        b = n // 2
        if b not in blocks:
            blocks[b] = philox(_key(seed), (j, int(t) & 0xFFFFFFFF, int(t) >> 32, 4 * purpose + b))
        out.append(mulhi64(_word64(blocks[b], 2 * (n % 2)), d).astype(np.int64))
    return out


def sample(dims, coo_inds, coo_vals, seed, t, estimate, p, q):
    """One sample set as splatt_b200_gcp_sample draws it: p stored entries (coordinates and
    values gathered from the COO), then q coordinates with value 0.  Returns ([N][p+q] int64,
    float64[p+q])."""
    nnz = len(coo_vals)
    pos = draw_positions(seed, t, 2 if estimate else 0, p, nnz)
    co = draw_coords(seed, t, 3 if estimate else 1, q, dims)
    inds = [np.concatenate([np.asarray(ci, dtype=np.int64)[pos], c]) for ci, c in zip(coo_inds, co)]
    vals = np.concatenate([np.asarray(coo_vals, dtype=np.float64)[pos], np.zeros(q)])
    return inds, vals


# ---- losses -------------------------------------------------------------------------------------
def softplus(m):
    return np.maximum(m, 0.0) + np.log1p(np.exp(-np.abs(m)))


def sigmoid(m):
    e = np.exp(-np.abs(m))
    return np.where(m >= 0, 1.0 / (1.0 + e), e / (1.0 + e))


def f(loss, x, m):
    if loss == GAUSSIAN:
        return (x - m) ** 2
    if loss == BERNOULLI_LOGIT:
        return softplus(m) - x * m
    return np.exp(m) - x * m


def df(loss, x, m):
    if loss == GAUSSIAN:
        return 2.0 * (m - x)
    if loss == BERNOULLI_LOGIT:
        return sigmoid(m) - x
    return np.exp(m) - x


def f_corr(loss, x, m):
    """f(x, m) - f(0, m), evaluated without cancellation: x^2 - 2 x m, or -x m."""
    return x * x - 2.0 * x * m if loss == GAUSSIAN else -x * m


def df_corr(loss, x, m):
    """df(x, m) - df(0, m): -2 x, or -x."""
    return -2.0 * x if loss == GAUSSIAN else -x


def value_ok(loss, vals):
    v = np.asarray(vals, dtype=np.float64)
    if loss == GAUSSIAN:
        return bool(np.all(np.isfinite(v)))
    if loss == BERNOULLI_LOGIT:
        return bool(np.all((v == 0.0) | (v == 1.0)))
    return bool(np.all(np.isfinite(v) & (v >= 0.0)))


# ---- model, sampled estimator, exact objective ---------------------------------------------------
def model_values(inds, factors):
    R = factors[0].shape[1]
    prod = np.ones((len(inds[0]), R))
    for i, U in zip(inds, factors):
        prod *= U[np.asarray(i, dtype=np.int64)]
    return prod.sum(1)


def sampled(loss, p, q, w_nz, w_z, inds, vals, factors, grads=True):
    """(value, [G_n]) of splatt_b200_gcp_sampled: samples 0..p-1 are stored entries (weight w_nz,
    the correction f(x,m) - f(0,m)), samples p..p+q-1 coordinates (weight w_z, f(0,m))."""
    idx = [np.asarray(i, dtype=np.int64)[:p + q] for i in inds]
    m = model_values(idx, factors)
    x = np.asarray(vals, dtype=np.float64)[:p]
    val = w_nz * f_corr(loss, x, m[:p]).sum() + w_z * f(loss, 0.0, m[p:]).sum()
    if not grads:
        return val, None
    y = np.concatenate([w_nz * df_corr(loss, x, m[:p]), w_z * df(loss, 0.0, m[p:])])
    out = []
    for n, U in enumerate(factors):
        h = np.ones((p + q, U.shape[1]))
        for k, W in enumerate(factors):
            if k != n:
                h *= W[idx[k]]
        G = np.zeros_like(U, dtype=np.float64)
        np.add.at(G, idx[n], y[:, None] * h)
        out.append(G)
    return val, out


def dense_model(factors):
    """The full model tensor sum_r prod_n U_n[:, r] (small tensors only)."""
    N = len(factors)
    spec = ",".join(f"{'abcdefgh'[n]}z" for n in range(N)) + "->" + "abcdefgh"[:N]
    return np.einsum(spec, *factors)


def objective(loss, dims, inds, vals, factors):
    """F(U) = sum over every coordinate of f(0, m) + sum over stored x of f(x_v, m) - f(0, m)."""
    M = dense_model(factors)
    m = model_values(inds, factors)
    x = np.asarray(vals, dtype=np.float64)
    return float(f(loss, 0.0, M).sum() + (f(loss, x, m) - f(loss, 0.0, m)).sum())


def gradient(loss, dims, inds, vals, factors):
    """Exact gradient of F: every coordinate's df(0, m) term plus the stored corrections."""
    N = len(factors)
    M = dense_model(factors)
    D = df(loss, 0.0, M)
    coords = np.indices(dims).reshape(N, -1)
    x = np.asarray(vals, dtype=np.float64)
    m = model_values(inds, factors)
    all_idx = [np.concatenate([coords[n], np.asarray(inds[n], dtype=np.int64)]) for n in range(N)]
    y = np.concatenate([D.ravel(), df(loss, x, m) - df(loss, 0.0, m)])
    out = []
    for n, U in enumerate(factors):
        h = np.ones((len(y), U.shape[1]))
        for k, W in enumerate(factors):
            if k != n:
                h *= W[all_idx[k]]
        G = np.zeros_like(U, dtype=np.float64)
        np.add.at(G, all_idx[n], y[:, None] * h)
        out.append(G)
    return out


# ---- GCP-Adam -----------------------------------------------------------------------------------
DEFAULTS = dict(loss=BERNOULLI_LOGIT, grad_nnz=1 << 16, grad_zeros=1 << 16, est_nnz=1 << 20,
                est_zeros=1 << 20, epoch_iters=1000, lr=1e-3, beta1=0.9, beta2=0.999,
                epsilon=1e-8, decay=0.1, max_fails=1, seed=0)


def adam(U, Mo, V, G, k, lr, b1, b2, eps):
    """One Adam update of step count k (1-based) in place, columns of U only."""
    c1, c2 = 1.0 / (1.0 - b1 ** k), 1.0 / (1.0 - b2 ** k)
    Mo *= b1
    Mo += (1.0 - b1) * G
    V *= b2
    V += (1.0 - b2) * G * G
    U -= lr * (Mo * c1) / (np.sqrt(V * c2) + eps)


def run_epochs(f_start, epoch, niters, tol, max_fails, decay, lr):
    """The epoch rule.  epoch(lr) runs one epoch from the current state and returns its
    estimate; revert() is epoch's attribute and restores the epoch-start state.  Returns
    (history [epochs x 3] of (estimate, lr used, accepted), epochs run)."""
    hist = []
    prev, fails = f_start, 0
    for _ in range(int(niters)):
        est = epoch(lr)
        ok = bool(np.isfinite(est) and est <= prev)
        hist.append((est, lr, 1.0 if ok else 0.0))
        if ok:
            rel = (prev - est) / abs(prev) if prev != 0 else 0.0
            prev = est
            if rel < tol:
                break
        else:
            epoch.revert()
            lr *= decay
            fails += 1
            if fails > max_fails:
                break
    return np.array(hist).reshape(-1, 3), len(hist)


def gcp(dims, coo_inds, coo_vals, factors, niters, tol, **opts):
    """The oracle driver: (factors, history, epochs, f_start) of splatt_b200_gcp_device from the
    start `factors`, given the COO in stream record order."""
    o = dict(DEFAULTS)
    o.update(opts)
    loss = o["loss"]
    nnz = len(coo_vals)
    total = float(np.prod(np.asarray(dims, dtype=np.float64)))
    U = [np.array(x, dtype=np.float64) for x in factors]
    Mo = [np.zeros_like(x) for x in U]
    V = [np.zeros_like(x) for x in U]
    gp, gq, ep, eq = o["grad_nnz"], o["grad_zeros"], o["est_nnz"], o["est_zeros"]
    gw = (nnz / gp if gp else 0.0, total / gq if gq else 0.0)
    ew = (nnz / ep if ep else 0.0, total / eq if eq else 0.0)
    ei, evs = sample(dims, coo_inds, coo_vals, o["seed"], 0, True, ep, eq)

    def estimate():
        return sampled(loss, ep, eq, ew[0], ew[1], ei, evs, U, grads=False)[0]

    state = {"t": 0}

    def epoch(lr):
        epoch.saved = ([x.copy() for x in U], [x.copy() for x in Mo], [x.copy() for x in V], state["t"])
        for _ in range(o["epoch_iters"]):
            t = state["t"]
            si, sv = sample(dims, coo_inds, coo_vals, o["seed"], t, False, gp, gq)
            _, G = sampled(loss, gp, gq, gw[0], gw[1], si, sv, U)
            for n in range(len(U)):
                adam(U[n], Mo[n], V[n], G[n], t + 1, lr, o["beta1"], o["beta2"], o["epsilon"])
            state["t"] = t + 1
        return estimate()

    def revert():
        su, sm, sv, st = epoch.saved
        for n in range(len(U)):
            U[n][...] = su[n]
            Mo[n][...] = sm[n]
            V[n][...] = sv[n]
        state["t"] = st

    epoch.revert = revert
    f0 = estimate()
    hist, its = run_epochs(f0, epoch, niters, tol, o["max_fails"], o["decay"], o["lr"])
    return U, hist, its, f0
