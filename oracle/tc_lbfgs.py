"""Tensor completion by whole-model L-BFGS with an exact line search, restated in numpy.

The semantics of splatt_b200_tc_lbfgs_device (include/splatt_b200.h), written out plainly: the
model and objective of oracle/tc.py; the gradient of all modes at the same factors (vectorised);
the line coefficients from explicit polynomial products per nonzero; the minimiser of the line
polynomial by np.roots on its derivative with Newton polishing; the direction by the L-BFGS
two-loop recursion; the stop rules of the contract.  Vectors over all factors are the
concatenation of the modes' blocks, row-major.
"""
from __future__ import annotations

import numpy as np

from oracle.tc import model_values, sse


def _idx(inds):
    return [np.asarray(i, dtype=np.int64) for i in inds]


def gradient(dims, inds, vals, factors, reg):
    """[G_m]: G_m[i] = -2 sum_{x: i_m(x) = i} r_x h_x + 2 reg U_m[i], r_x = v_x - x^_x."""
    idx = _idx(inds)
    r = np.asarray(vals, dtype=np.float64) - model_values(inds, factors)
    out = []
    for m, U in enumerate(factors):
        h = np.ones((len(r), U.shape[1]))
        for n, W in enumerate(factors):
            if n != m:
                h *= W[idx[n]]
        G = 2.0 * reg * np.asarray(U, dtype=np.float64)
        acc = np.zeros_like(G)
        np.add.at(acc, idx[m], r[:, None] * h)
        out.append(G - 2.0 * acc)
    return out


def flat(blocks):
    return np.concatenate([np.asarray(b, dtype=np.float64).ravel() for b in blocks])


def unflat(v, like):
    out, o = [], 0
    for b in like:
        out.append(v[o:o + b.size].reshape(b.shape))
        o += b.size
    return out


def line_coefs(inds, vals, factors, D, reg):
    """(c, c_data): phi(a) = L(U + a D) = sum_j c[j] a^j (2N + 1 coefficients) and its data part.
    Per nonzero and column the N + 1 coefficients of prod_m (u_m + a d_m) are formed by explicit
    polynomial products; e(a) = v - their column sum, and phi_data = sum_x e(a)^2."""
    idx = _idx(inds)
    N = len(factors)
    nnz, R = len(idx[0]), factors[0].shape[1]
    P = np.zeros((nnz, R, N + 1))
    P[:, :, 0] = 1.0
    for m in range(N):
        u = factors[m][idx[m]]
        d = D[m][idx[m]]
        Q = np.zeros_like(P)
        Q[:, :, :] = P * u[:, :, None]
        Q[:, :, 1:] += P[:, :, :-1] * d[:, :, None]
        P = Q
    e = -P.sum(axis=1)
    e[:, 0] += np.asarray(vals, dtype=np.float64)
    Mx = e.T @ e
    cd = np.zeros(2 * N + 1)
    for i in range(N + 1):
        for j in range(N + 1):
            cd[i + j] += Mx[i, j]
    c = cd.copy()
    uu = sum(float((U * U).sum()) for U in factors)
    ud = sum(float((U * W).sum()) for U, W in zip(factors, D))
    dd = sum(float((W * W).sum()) for W in D)
    c[0] += reg * uu
    c[1] += 2.0 * reg * ud
    c[2] += reg * dd
    return c, cd


def decrease(c, a):
    """-sum_{j>=1} c[j] a^j, evaluated from the coefficients."""
    t = 0.0
    for j in range(len(c) - 1, 0, -1):
        t = t * a + c[j]
    return -(t * a)


def poly_argmin(c):
    """(alpha, decrease): the minimiser of sum_j c[j] a^j over [0, B], B the Cauchy bound of the
    derivative's roots; candidates 0 and the real roots of the derivative in (0, B] (np.roots,
    then Newton polishing), the smallest candidate with the least value."""
    c = np.asarray(c, dtype=np.float64)
    dp = np.array([j * c[j] for j in range(1, len(c))])
    while len(dp) and dp[-1] == 0.0:
        dp = dp[:-1]
    best, bestd = 0.0, 0.0
    if len(dp) == 0:
        return best, bestd
    B = 1.0 + (np.max(np.abs(dp[:-1] / dp[-1])) if len(dp) > 1 else 0.0)
    cand = []
    if len(dp) > 1:
        ddp = np.array([j * dp[j] for j in range(1, len(dp))])
        for z in np.roots(dp[::-1]):
            if abs(z.imag) > 1e-6 * max(1.0, abs(z.real)):
                continue
            x = float(z.real)
            for _ in range(8):
                f1 = np.polyval(dp[::-1], x)
                f2 = np.polyval(ddp[::-1], x)
                if f2 == 0.0 or not np.isfinite(f1 / f2):
                    break
                nx = x - f1 / f2
                if abs(np.polyval(dp[::-1], nx)) >= abs(f1):
                    break
                x = nx
            if 0.0 < x <= B:
                cand.append(x)
    for x in sorted(cand):
        dec = decrease(c, x)
        if dec > bestd:
            best, bestd = x, dec
    return best, bestd


def two_loop(g, pairs):
    """-H g by the L-BFGS two-loop recursion over pairs [(s, y)] (oldest first), H0 = gamma I,
    gamma = s.y / y.y of the newest pair; -g without pairs."""
    q = -g.copy()
    if not pairs:
        return q
    al = []
    for s, y in reversed(pairs):
        a = (s @ q) / (s @ y)
        al.append(a)
        q = q - a * y
    s, y = pairs[-1]
    q = q * ((s @ y) / (y @ y))
    for (s, y), a in zip(pairs, reversed(al)):
        b = (y @ q) / (s @ y)
        q = q + (a - b) * s
    return q


def tc_lbfgs(dims, inds, vals, factors, reg, memory, niters, tol, validate=None):
    """Returns (history [iters x 5]: L, train RMSE, validation RMSE or NaN, alpha, ||g||;
    factors; info: per iteration a dict of the decrease, phi(0), the newest pair's s.y (None
    when no pair was formed), whether the pairs were cleared and whether a retry ran)."""
    f = [np.array(U, dtype=np.float64, copy=True) for U in factors]
    n = len(vals)
    pairs = []
    hist, info = [], []
    g_prev = d_prev = None
    alpha_prev = 0.0
    for it in range(niters):
        g = flat(gradient(dims, inds, vals, f, reg))
        sy = None
        if it > 0 and memory > 0 and alpha_prev > 0.0:
            s = alpha_prev * d_prev
            y = g - g_prev
            sy = float(s @ y)
            if sy > 0.0:
                pairs.append((s, y))
                pairs = pairs[-memory:]
        gg = float(g @ g)
        cleared = retry = False
        if pairs:
            d = two_loop(g, pairs)
            lb = True
            if not (g @ d < 0.0):
                pairs, d, lb, cleared = [], -g, False, True
        else:
            d, lb = -g, False
        c, cd = line_coefs(inds, vals, f, unflat(d, f), reg)
        stop = False
        if gg == 0.0:
            alpha, dec, stop = 0.0, 0.0, True
        else:
            alpha, dec = poly_argmin(c)
            if not dec > 0.0 and lb:
                pairs, d, retry = [], -g, True
                c, cd = line_coefs(inds, vals, f, unflat(d, f), reg)
                alpha, dec = poly_argmin(c)
            if not dec > 0.0:
                alpha, dec, stop = 0.0, 0.0, True
        trs = float(np.polyval(cd[::-1], alpha))
        if not stop:
            f = [U + alpha * W for U, W in zip(f, unflat(d, f))]
        vr = float("nan")
        if validate is not None:
            vr = np.sqrt(sse(validate[0], validate[1], f) / len(validate[1]))
        hist.append((c[0] - dec, np.sqrt(max(trs, 0.0) / n), vr, alpha, np.sqrt(gg)))
        info.append(dict(decrease=dec, phi0=c[0], sy=sy, cleared=cleared, retry=retry))
        g_prev, d_prev, alpha_prev = g, d, alpha
        if stop or (it > 0 and dec / c[0] < tol):
            break
    return np.array(hist), f, info
