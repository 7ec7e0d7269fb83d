"""Poisson CP decomposition by CP-APR with row-wise projected damped Newton steps (PDNR),
restated in numpy: the semantics of splatt_b200_cp_apr_pdnr_device (include/splatt_b200.h).
Model, start, normalisation and log-likelihood are those of oracle/apr.py (MU)."""
from __future__ import annotations

import numpy as np

from oracle.apr import _idx, loglik, normalize_columns

# The semantics of splatt_b200_cp_apr_pdnr_device (include/splatt_b200.h), after Hansen,
# Plantenga & Kolda (Optim. Methods Softw. 2015).  Mode n's subproblem splits into one convex
# problem per row i of B = A_n diag(lam):
#     f_i(b) = sum_r b_r - sum_{x in X_i} v_x log(max(m_x(b), eps)),   m_x(b) = b . Pi_x,
#     g = 1 - sum_x (v_x / max(m_x, eps)) Pi_x,   H = sum_x (v_x / max(m_x, eps)^2) Pi_x Pi_x^T.
# Every row runs up to max_inner projected damped Newton steps from b = B[i] with mu = mu0:
#   kkt = max_r |min(b_r, g_r)|; stop when kkt < tol;
#   eps_i = min(eps_active, ||b - max(b - g, 0)||_2); active set A = {r: b_r <= eps_i, g_r > 0};
#   d_A = -g_A, (H_FF + mu I) d_F = -g_F by Cholesky (d = -g when a pivot is <= 0 or not finite);
#   trial points b_k = max(b + 2^-k d, 0), k = 0 .. max_backtrack - 1; accept the smallest k with
#   f(b_k) <= f(b) + 1e-4 g.(b_k - b) and f(b_k) <= f(b), the change f(b_k) - f(b) evaluated
#   as in f_change;
#   mu <- max(mu / 3.5, mu0) when k = 0 was accepted, else mu <- 3.5 mu (b unchanged when no k
#   passed).
# Then lam = the column sums of B and A_n = B diag(1 / lam).  The accept rule never raises an
# f_i, and sum_i f_i(B[i]) = -LL, so the log-likelihood never decreases from mode to mode.

ARMIJO = 1e-4
DAMPING = 3.5


def _row_f(b, Pi, v, eps):
    return float(b.sum() - np.dot(v, np.log(np.maximum(Pi @ b, eps))))


def f_change(b, bk, Pi, v, m, eps):
    """f_i(bk) - f_i(b) = sum_r (bk - b)_r - sum_x v_x log(max(m_x + delta_x, eps) / max(m_x, eps))
    with m_x = b . Pi_x and delta_x = (bk - b) . Pi_x, the log of the ratio by log1p(delta / m)
    where neither value is floored.  Accurate to the rounding of the change rather than of f, so
    the line search can still tell a decrease near the row's minimum."""
    s = bk - b
    delta = Pi @ s
    mk = m + delta
    plain = (m >= eps) & (mk >= eps)
    with np.errstate(divide="ignore", invalid="ignore"):
        lr = np.where(plain, np.log1p(np.where(plain, delta / np.where(plain, m, 1.0), 0.0)),
                      np.log(np.maximum(mk, eps)) - np.log(np.maximum(m, eps)))
    return float(s.sum() - np.dot(v, lr))


def chol_solve(M, rhs, pivots=None):
    """x with M x = rhs by the right-looking Cholesky M = U^T U and two triangular solves, the
    order the device uses; None when a pivot is <= 0 or not finite.  pivots: a list that gets
    the smallest pivot relative to its diagonal entry of M (0 when the factorisation failed)."""
    U = np.array(M, dtype=np.float64, copy=True)
    x = np.array(rhs, dtype=np.float64, copy=True)
    n = len(x)
    rel = float("inf")
    for k in range(n):
        p = U[k, k]
        if not (p > 0.0 and np.isfinite(p)):
            if pivots is not None:
                pivots.append(0.0)
            return None
        rel = min(rel, p / M[k, k])
        d = np.sqrt(p)
        U[k, k + 1:] *= 1.0 / d
        U[k, k] = d
        U[k + 1:, k + 1:] -= np.outer(U[k, k + 1:], U[k, k + 1:])
    for k in range(n):
        x[k] /= U[k, k]
        x[k + 1:] -= U[k, k + 1:] * x[k]
    for k in range(n - 1, -1, -1):
        x[k] /= U[k, k]
        x[:k] -= U[:k, k] * x[k]
    if pivots is not None:
        pivots.append(rel)
    return x


def row_subproblem(b, Pi, v, tol, max_inner=10, max_backtrack=8, mu0=1e-5, eps_active=1e-8,
                   eps=1e-10):
    """Minimises f_i from b by the projected damped Newton steps above.  Pi: the row's records'
    Pi_x (nnz_i x R), v their values.  Returns (b, info): info["evals"] kkt evaluations,
    ["steps"] Newton steps, ["kkt"] the last kkt, ["mu"] the final damping, ["f"] f_i after every
    step (f[0] at the start), ["ks"] the accepted k of every step (-1: none passed),
    ["active"] active-set sizes, ["fallbacks"] steps with d = -g, ["pivots"] every step's
    smallest relative Cholesky pivot (0 for a fallback), and ["decisions"]: for every
    trial point tried, (k, margin, step) with margin = max(df - 1e-4 g.(b_k - b), df),
    df = f_change(b, b_k) (the trial passes when margin <= 0) and step = ||b_k - b|| / max(||b||, tiny)."""
    b = np.array(b, dtype=np.float64, copy=True)
    Pi = np.asarray(Pi, dtype=np.float64)
    v = np.asarray(v, dtype=np.float64)
    mu = mu0
    info = {"evals": 0, "steps": 0, "kkt": float("nan"), "mu": mu, "f": [_row_f(b, Pi, v, eps)],
            "ks": [], "active": [], "fallbacks": 0, "pivots": [], "decisions": []}
    for _ in range(max_inner):
        mm = np.maximum(Pi @ b, eps)
        g = 1.0 - Pi.T @ (v / mm)
        h = Pi * (np.sqrt(v) / mm)[:, None]          # H = h^T h: no v / m^2 to underflow
        H = h.T @ h
        kkt = float(np.abs(np.minimum(b, g)).max())
        info["evals"] += 1
        info["kkt"] = kkt
        if kkt < tol:
            break
        info["steps"] += 1
        e = min(eps_active, float(np.linalg.norm(b - np.maximum(b - g, 0.0))))
        act = (b <= e) & (g > 0.0)
        free = ~act
        info["active"].append(int(act.sum()))
        d = -g
        x = chol_solve(H[np.ix_(free, free)] + mu * np.eye(int(free.sum())), -g[free], info["pivots"])
        if x is None:
            info["fallbacks"] += 1
        else:
            d = d.copy()
            d[free] = x
        m = Pi @ b
        acc, bn = -1, b
        nb = max(float(np.linalg.norm(b)), 1e-300)
        for k in range(max_backtrack):
            bk = np.maximum(b + 2.0 ** -k * d, 0.0)
            df = f_change(b, bk, Pi, v, m, eps)
            margin = max(df - ARMIJO * float(np.dot(g, bk - b)), df)
            info["decisions"].append((k, margin, float(np.linalg.norm(bk - b)) / nb))
            if margin <= 0.0:
                acc, bn = k, bk
                break
        info["ks"].append(acc)
        b = bn
        mu = max(mu / DAMPING, mu0) if acc == 0 else mu * DAMPING
        info["f"].append(_row_f(b, Pi, v, eps))
    info["mu"] = mu
    return b, info


def others(inds, factors, n):
    """Pi_x of every record for mode n: the Hadamard product of the other factors' rows."""
    idx = _idx(inds)
    Pi = np.ones((len(idx[0]), factors[0].shape[1]))
    for m, A in enumerate(factors):
        if m != n:
            Pi *= A[idx[m]]
    return Pi


def cp_apr_pdnr(dims, inds, vals, factors, niters, tol, max_inner=10, max_backtrack=8, mu0=1e-5,
                eps_active=1e-8, eps=1e-10):
    """Returns (lam, factors, history [iters x 4]: LL, largest last kkt, lockstep iterations
    summed over the modes, Newton steps attempted (line searches run) summed over rows and
    modes; info: {"rows": one dict per (outer iteration, mode, row) with the row_subproblem info
    plus "it", "mode", "row", "nnz"; "ll_modes": LL after every mode})."""
    N = len(dims)
    vals = np.asarray(vals, dtype=np.float64)
    A, lam = [], np.ones(factors[0].shape[1])
    for U in factors:
        a, s = normalize_columns(np.array(U, dtype=np.float64, copy=True))
        A.append(a)
        lam = lam * s
    idx = _idx(inds)
    hist, info = [], {"rows": [], "ll_modes": []}
    for it in range(niters):
        converged, kmax, lockstep, steps = True, 0.0, 0, 0
        for n in range(N):
            B = A[n] * lam[None, :]
            Pi = others(inds, A, n)
            order = np.argsort(idx[n], kind="stable")
            bounds = np.searchsorted(idx[n][order], np.arange(dims[n] + 1))
            evals = 0
            for i in range(dims[n]):
                sel = order[bounds[i]:bounds[i + 1]]
                B[i], ri = row_subproblem(B[i], Pi[sel], vals[sel], tol, max_inner, max_backtrack,
                                          mu0, eps_active, eps)
                ri.update(it=it, mode=n, row=i, nnz=len(sel))
                info["rows"].append(ri)
                evals = max(evals, ri["evals"])
                steps += ri["steps"]
                kmax = max(kmax, ri["kkt"])
                converged = converged and ri["steps"] == 0
            lockstep += evals
            A[n], lam = normalize_columns(B)
            info["ll_modes"].append(loglik(inds, vals, A, lam, eps))
        hist.append((loglik(inds, vals, A, lam, eps), kmax, lockstep, steps))
        if converged:
            break
    return lam, A, np.array(hist), info
