"""Tensor completion by row-wise ALS, restated in numpy (the reference has no completion).

The semantics of splatt_b200_tc_als_device (include/splatt_b200.h), written out plainly:
model x^ = sum_r prod_m U_m[i_m, r] (no lambda); objective
L = sum over stored entries (v - x^)^2 + reg * sum_m ||U_m||_F^2; one iteration updates the modes
in order, every row by an explicit np.linalg.solve of its regularised normal equations.
"""
from __future__ import annotations

import numpy as np


def model_values(inds, factors, lam=None):
    """x^ at every coordinate (inds[m]: index arrays)."""
    R = factors[0].shape[1]
    prod = np.ones((len(inds[0]), R))
    for m, U in enumerate(factors):
        prod *= U[np.asarray(inds[m], dtype=np.int64)]
    if lam is not None:
        prod *= np.asarray(lam)[None, :]
    return prod.sum(axis=1)


def sse(inds, vals, factors, lam=None):
    r = np.asarray(vals, dtype=np.float64) - model_values(inds, factors, lam)
    return float(r @ r)


def row_systems(dims, inds, vals, factors, m):
    """Per row i of mode m: (H_i, v_i), the stacked h_x and values of its observations."""
    idx = [np.asarray(i, dtype=np.int64) for i in inds]
    R = factors[0].shape[1]
    h = np.ones((len(vals), R))
    for n, U in enumerate(factors):
        if n != m:
            h *= U[idx[n]]
    order = np.argsort(idx[m], kind="stable")
    rows = idx[m][order]
    bounds = np.searchsorted(rows, np.arange(dims[m] + 1))
    v = np.asarray(vals, dtype=np.float64)[order]
    h = h[order]
    return [(h[bounds[i]:bounds[i + 1]], v[bounds[i]:bounds[i + 1]]) for i in range(dims[m])]


def update_mode(dims, inds, vals, factors, m, reg):
    """New U_m: every row solves (H^T H + reg I) u = H^T v; a row without observations is 0."""
    R = factors[0].shape[1]
    out = np.zeros((dims[m], R))
    for i, (H, v) in enumerate(row_systems(dims, inds, vals, factors, m)):
        if len(v):
            out[i] = np.linalg.solve(H.T @ H + reg * np.eye(R), H.T @ v)
    return out


def sweep(dims, inds, vals, factors, reg):
    """One iteration: modes 0..N-1 in order (Gauss-Seidel).  Returns new factors."""
    f = [np.array(U, dtype=np.float64, copy=True) for U in factors]
    for m in range(len(dims)):
        f[m] = update_mode(dims, inds, vals, f, m, reg)
    return f


def objective(inds, vals, factors, reg):
    return sse(inds, vals, factors) + reg * sum(float((U * U).sum()) for U in factors)


def tc_als(dims, inds, vals, factors, reg, niters, tol, validate=None):
    """Returns (history [iters x 3]: L, train RMSE, validation RMSE or NaN; factors).
    validate: optional (inds, vals) of held-out entries."""
    f = [np.array(U, dtype=np.float64, copy=True) for U in factors]
    hist = []
    prev = None
    for it in range(niters):
        f = sweep(dims, inds, vals, f, reg)
        s = sse(inds, vals, f)
        L = s + reg * sum(float((U * U).sum()) for U in f)
        vr = float("nan")
        if validate is not None:
            vr = np.sqrt(sse(validate[0], validate[1], f) / len(validate[1]))
        hist.append((L, np.sqrt(s / len(vals)), vr))
        if it > 0 and abs(prev - L) / prev < tol:
            break
        prev = L
    return np.array(hist), f
