"""Sparse Tucker decomposition by HOOI, written out plainly in numpy: the semantics of
splatt_b200_ttmc and splatt_b200_tucker_hooi_device (include/splatt_b200.h).

X ~ G x_0 U_0 ... x_{N-1} U_{N-1}; unstored coordinates are zeros and duplicate coordinates add.
Y_n = X_(n) (kron_{m != n} U_m), the other modes in increasing order with the highest fastest.

hooi_exact takes each U_n from np.linalg.svd of Y_n.  hooi_power restates the device's procedure:
warm-started orthogonal iteration Q <- orth(Y Y^T Q + mu Q) with orth = CholeskyQR2 and
mu = 2^-20 ||Y||_F^2, stopped after max_power steps or when ||Q_new - Q_old (Q_old^T Q_new)||_F
<= svd_tol, then one Rayleigh-Ritz step and the sign convention (in each column the entry of
largest magnitude positive, the lowest row on a tie).
"""
from __future__ import annotations

import numpy as np

MU_REL = 2.0 ** -20


def ttmc(dims, inds, vals, mats, n, ranks, block=4096):
    """Y_n (dims[n] x prod_{m != n} ranks[m]) from COO, duplicates adding."""
    N = len(dims)
    inds = [np.asarray(i, dtype=np.int64) for i in inds]
    vals = np.asarray(vals, dtype=np.float64)
    C = int(np.prod([ranks[m] for m in range(N) if m != n]))
    Y = np.zeros((dims[n], C))
    for lo in range(0, len(vals), block):
        hi = min(lo + block, len(vals))
        K = vals[lo:hi, None]
        for m in range(N):
            if m == n:
                continue
            U = np.asarray(mats[m])[inds[m][lo:hi], :ranks[m]]
            K = (K[:, :, None] * U[:, None, :]).reshape(hi - lo, -1)
        np.add.at(Y, inds[n][lo:hi], K)
    return Y


def xnorm_sq(dims, inds, vals):
    """||X||^2 with duplicate coordinates summed."""
    key = np.ravel_multi_index([np.asarray(i, dtype=np.int64) for i in inds], dims)
    _, inv = np.unique(key, return_inverse=True)
    s = np.zeros(inv.max() + 1 if len(inv) else 0)
    np.add.at(s, inv, np.asarray(vals, dtype=np.float64))
    return float(np.sum(s * s))


def cholqr2(Z):
    """CholeskyQR2; raises np.linalg.LinAlgError when a Gram is not positive definite."""
    Q = Z
    for _ in range(2):
        L = np.linalg.cholesky(Q.T @ Q)
        Q = Q @ np.linalg.inv(L).T
    return Q


def fix_signs(U):
    """+-1 per column: the entry of largest magnitude positive (np.argmax: the lowest row on a tie)."""
    idx = np.argmax(np.abs(U), axis=0)
    return np.where(U[idx, np.arange(U.shape[1])] < 0, -1.0, 1.0)


def _fit(xsq, G):
    gsq = float(np.sum(G * G))
    return 1.0 - np.sqrt(max(xsq - gsq, 0.0)) / np.sqrt(xsq) if xsq > 0 else 1.0, gsq


def _stop(it, fit, old, tol):
    return fit == 1.0 or (it > 0 and abs(fit - old) < tol)


def hooi_power(dims, inds, vals, ranks, factors, niters, tol, max_power=50, svd_tol=1e-10):
    """The device's procedure.  Returns (core (shape ranks), factors, history [its x 4])."""
    N = len(dims)
    xsq = xnorm_sq(dims, inds, vals)
    F = [cholqr2(np.asarray(f, dtype=np.float64)[:, :r]) for f, r in zip(factors, ranks)]
    hist, old, G = [], 0.0, None
    for it in range(int(niters)):
        steps, rmax = 0, 0.0
        for n in range(N):
            Y = ttmc(dims, inds, vals, F, n, ranks)
            ysq = float(np.sum(Y * Y))
            mu = MU_REL * ysq if ysq > 0 else 1.0
            Q = F[n]
            res = 0.0
            for _ in range(max_power):
                Z = Y @ (Y.T @ Q) + mu * Q
                Qn = cholqr2(Z)
                res = float(np.linalg.norm(Q @ (Q.T @ Qn) - Qn))
                Q = Qn
                steps += 1
                if res <= svd_tol:
                    break
            rmax = max(rmax, res)
            W = Y.T @ Q
            lam, V = np.linalg.eigh(W.T @ W)
            V = V[:, np.argsort(-lam, kind="stable")]
            U = Q @ V
            sg = fix_signs(U)
            F[n] = U * sg
            if n == N - 1:
                G = (W @ V) * sg
        fit, gsq = _fit(xsq, G)
        hist.append((fit, np.sqrt(gsq), steps, rmax))
        if _stop(it, fit, old, tol):
            break
        old = fit
    return G.reshape(ranks), F, np.array(hist)


def hooi_exact(dims, inds, vals, ranks, factors, niters, tol):
    """HOOI with the leading left singular vectors of each Y_n from np.linalg.svd."""
    N = len(dims)
    xsq = xnorm_sq(dims, inds, vals)
    F = [np.linalg.qr(np.asarray(f, dtype=np.float64)[:, :r])[0] for f, r in zip(factors, ranks)]
    hist, old, G = [], 0.0, None
    for it in range(int(niters)):
        for n in range(N):
            Y = ttmc(dims, inds, vals, F, n, ranks)
            U = np.linalg.svd(Y, full_matrices=False)[0][:, :ranks[n]]
            F[n] = U * fix_signs(U)
        G = Y.T @ F[N - 1]
        fit, gsq = _fit(xsq, G)
        hist.append((fit, np.sqrt(gsq)))
        if _stop(it, fit, old, tol):
            break
        old = fit
    return G.reshape(ranks), F, np.array(hist)
