"""Poisson CP decomposition by CP-APR with row-wise projected quasi-Newton steps (PQNR),
restated in numpy: the semantics of splatt_b200_cp_apr_pqnr_device (include/splatt_b200.h).
Model, start, outer loop, line search and history are those of oracle/apr_pdnr.py (PDNR); only
the direction differs."""
from __future__ import annotations

import numpy as np

from oracle.apr import _idx, loglik, normalize_columns
from oracle.apr_pdnr import ARMIJO, _row_f, f_change, others

# Every row i of B = A_n diag(lam) starts from b = B[i] with no stored pair and level j = 0 and
# runs up to max_inner lockstep evaluations:
#   1. g = 1 - sum_x (v_x / max(m_x, eps)) Pi_x, kkt = max_r |min(b_r, g_r)|; stop when kkt < tol.
#   2. After a step, if b is bitwise b_prev (the last line search moved nothing): j <- j + 1; at
#      j = 3 the row gives up; else d <- 2^-max_backtrack d (the trial points continue the
#      halving) and go to 5.
#   3. Otherwise j = 0, and after a step the pair s = b - b_prev, y = g - g_prev is stored (the
#      oldest of lbfgs_mem dropped) when s.y > 0 and 1 / s.y is finite.
#   4. eps_i and the active set A as in PDNR; q = -g with q_A = 0; the L-BFGS two-loop recursion,
#      newest to oldest, scale by gamma = s.y / y.y of the newest pair (1 without a pair), oldest
#      to newest; d = q, d_A = -g_A; d = -g when d is not finite.
#   5. b_prev = b, g_prev = g; PDNR's line search along d (b unchanged when no trial point passes).
# Every scaling of d is a power of two, so the device's trial points are bitwise these.

CONTINUE_ROUNDS = 3


def _same(a, b):
    return bool(np.array_equal(np.ascontiguousarray(a).view(np.int64), np.ascontiguousarray(b).view(np.int64)))


def row_subproblem(b, Pi, v, tol, max_inner=10, max_backtrack=8, lbfgs_mem=3, eps_active=1e-8,
                   eps=1e-10):
    """Minimises f_i from b by the projected quasi-Newton steps above.  Pi: the row's records'
    Pi_x (nnz_i x R), v their values.  Returns (b, info): info["evals"] kkt evaluations,
    ["steps"] line searches run, ["kkt"] the last kkt, ["f"] f_i after every step (f[0] at the
    start), ["ks"] the accepted k of every step (-1: none passed), ["decisions"] (k, margin,
    step) for every trial point tried as in oracle.apr_pdnr, ["pairs"] (s.y, kept, |s| |y|) of
    every candidate pair, ["levels"] the continuation level of every continuation (3: gave up),
    ["gave_up"] whether the row stopped after CONTINUE_ROUNDS continuations."""
    b = np.array(b, dtype=np.float64, copy=True)
    Pi = np.asarray(Pi, dtype=np.float64)
    v = np.asarray(v, dtype=np.float64)
    S, Y, rho = [], [], []                                  # the stored pairs, oldest first
    j, bp, gp, d = 0, None, None, None
    info = {"evals": 0, "steps": 0, "kkt": float("nan"), "f": [_row_f(b, Pi, v, eps)], "ks": [],
            "decisions": [], "pairs": [], "levels": [], "gave_up": False}
    for _ in range(max_inner):
        mm = np.maximum(Pi @ b, eps)
        g = 1.0 - Pi.T @ (v / mm)
        kkt = float(np.abs(np.minimum(b, g)).max())
        info["evals"] += 1
        info["kkt"] = kkt
        if kkt < tol:
            break
        if bp is not None and _same(b, bp):
            j += 1
            info["levels"].append(j)
            if j == CONTINUE_ROUNDS:
                info["gave_up"] = True
                break
            d = d * 2.0 ** -max_backtrack
        else:
            j = 0
            if bp is not None:
                s, y = b - bp, g - gp
                sty = float(np.dot(s, y))
                with np.errstate(divide="ignore"):
                    keep = sty > 0.0 and bool(np.isfinite(1.0 / sty))
                info["pairs"].append((sty, keep, float(np.linalg.norm(s) * np.linalg.norm(y))))
                if keep:
                    S.append(s)
                    Y.append(y)
                    rho.append(1.0 / sty)
                    if len(S) > lbfgs_mem:
                        S.pop(0), Y.pop(0), rho.pop(0)
            e = min(eps_active, float(np.linalg.norm(b - np.maximum(b - g, 0.0))))
            act = (b <= e) & (g > 0.0)
            q = np.where(act, 0.0, -g)
            alpha = [0.0] * len(S)
            for k in range(len(S) - 1, -1, -1):
                alpha[k] = rho[k] * float(np.dot(S[k], q))
                q = q - alpha[k] * Y[k]
            if S:
                q = (float(np.dot(S[-1], Y[-1])) / float(np.dot(Y[-1], Y[-1]))) * q
            for k in range(len(S)):
                beta = rho[k] * float(np.dot(Y[k], q))
                q = q + (alpha[k] - beta) * S[k]
            d = np.where(act, -g, q)
            if not np.isfinite(d).all():
                d = -g
        info["steps"] += 1
        bp, gp = b, g
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
        info["f"].append(_row_f(b, Pi, v, eps))
    return b, info


def cp_apr_pqnr(dims, inds, vals, factors, niters, tol, max_inner=10, max_backtrack=8, lbfgs_mem=3,
                eps_active=1e-8, eps=1e-10):
    """Returns (lam, factors, history [iters x 4]: LL, largest last kkt, lockstep iterations
    summed over the modes, line searches run summed over rows and modes; info: {"rows": one dict
    per (outer iteration, mode, row) with the row_subproblem info plus "it", "mode", "row",
    "nnz"; "ll_modes": LL after every mode})."""
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
                                          lbfgs_mem, eps_active, eps)
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
