"""Nonnegative CPD by HALS, restated in numpy (the reference has no nonnegative CPD).

The semantics of splatt_b200_cpd_nonneg_device (include/splatt_b200.h), written out plainly:
model K = sum_r lam_r a_r^(0) o ... o a_r^(N-1) with nonnegative, 2-normalised factors;
unstored coordinates are zeros; duplicate coordinates are separate nonzeros (||X||^2 sums v^2
over them).  Per mode: M = the MTTKRP, G = the Hadamard product of the other Grams,
B = A_n diag(lam), one Gauss-Seidel sweep over the columns of B floored at EPS, lam = the column
2-norms of B and A_n = B diag(1 / lam).  The fit and the stopping rule are CPD-ALS's.
"""
from __future__ import annotations

import numpy as np

EPS = 1e-16


def _idx(inds):
    return [np.asarray(i, dtype=np.int64) for i in inds]


def mttkrp(dims, inds, vals, factors, n):
    """M[i, :] = sum over the coordinates x with i_n(x) = i of v_x prod_{m != n} A_m[i_m(x), :]."""
    idx = _idx(inds)
    P = np.asarray(vals, dtype=np.float64)[:, None] * np.ones((1, factors[0].shape[1]))
    for m, A in enumerate(factors):
        if m != n:
            P = P * A[idx[m]]
    out = np.zeros((dims[n], factors[0].shape[1]))
    np.add.at(out, idx[n], P)
    return out


def hadamard_grams(grams, n):
    G = np.ones_like(grams[0])
    for m, g in enumerate(grams):
        if m != n:
            G = G * g
    return G


def sweep(B, M, G, eps=EPS):
    """One HALS sweep over the columns r = 0 .. R-1 (columns j < r already updated):
    B[:, r] <- max(eps, (M[:, r] - sum_{j != r} B[:, j] G[j, r]) / G[r, r])."""
    B = np.array(B, dtype=np.float64, copy=True)
    R = B.shape[1]
    for r in range(R):
        others = [j for j in range(R) if j != r]
        s = M[:, r] - B[:, others] @ G[others, r]
        B[:, r] = np.maximum(eps, s / G[r, r])
    return B


def fit(xx, grams, lam, inner):
    """CPD-ALS's fit 1 - sqrt(||X||^2 + ||K||^2 - 2<X,K>) / ||X|| (residual left unrooted when it
    is not positive)."""
    G = np.ones_like(grams[0])
    for g in grams:
        G = G * g
    kk = abs(float(lam @ G @ lam))
    resid = xx + kk - 2 * inner
    resid = np.sqrt(resid) if resid > 0 else resid
    return 1 - resid / np.sqrt(xx)


def cpd_nonneg(dims, inds, vals, factors, niters, tol, eps=EPS):
    """Returns (fit, lam, factors, history: the fit of every iteration run)."""
    N = len(dims)
    A, lam = [], np.ones(factors[0].shape[1])
    for U in factors:
        U = np.array(U, dtype=np.float64, copy=True)
        assert np.all(np.isfinite(U)) and np.all(U >= 0), "start entries must be finite and >= 0"
        nrm = np.linalg.norm(U, axis=0)
        assert np.all(nrm > 0), "a start column is zero"
        A.append(U / nrm)
        lam = lam * nrm
    grams = [a.T @ a for a in A]
    xx = float(np.sum(np.asarray(vals, dtype=np.float64) ** 2))
    hist, f, oldfit = [], 0.0, 0.0
    for it in range(niters):
        for n in range(N):
            M = mttkrp(dims, inds, vals, A, n)
            B = sweep(A[n] * lam[None, :], M, hadamard_grams(grams, n), eps)
            lam = np.linalg.norm(B, axis=0)
            A[n] = B / lam
            grams[n] = A[n].T @ A[n]
        inner = float(np.sum(A[N - 1] * M * lam[None, :]))
        f = fit(xx, grams, lam, inner)
        hist.append(f)
        if f == 1.0 or (it > 0 and abs(f - oldfit) < tol):
            break
        oldfit = f
    return f, lam, A, np.array(hist)
