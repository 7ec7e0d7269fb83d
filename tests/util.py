"""Shared helpers for the test-suite: seeded synthetic tensors and error norms."""
from __future__ import annotations

import numpy as np


def random_coo(dims, nnz, seed=0, unique=True, skew=None):
    """Seeded random COO.  unique=True removes duplicate coordinates (the order of
    duplicates inside a CSF leaf is sort-implementation specific).  skew: optional
    list of per-mode Zipf exponents (None = uniform)."""
    rng = np.random.default_rng(seed)
    dims = list(dims)
    inds = []
    for m, d in enumerate(dims):
        if skew is not None and skew[m]:
            p = 1.0 / np.arange(1, d + 1) ** skew[m]
            p /= p.sum()
            perm = rng.permutation(d)
            inds.append(perm[rng.choice(d, size=nnz, p=p)].astype(np.uint64))
        else:
            inds.append(rng.integers(0, d, size=nnz, dtype=np.uint64))
    vals = rng.uniform(0.0, 1.0, size=nnz)
    if unique:
        key = np.zeros(nnz, dtype=np.uint64)
        for m, d in enumerate(dims):
            key = key * np.uint64(d) + inds[m]
        _, first = np.unique(key, return_index=True)
        first.sort()
        inds = [i[first] for i in inds]
        vals = vals[first]
    return dims, inds, vals


def cover_all_slices(dims, inds, vals, seed=1):
    """Append one nonzero per (mode, index) so that no slice is empty."""
    rng = np.random.default_rng(seed)
    extra = [[] for _ in dims]
    for m, d in enumerate(dims):
        missing = np.setdiff1d(np.arange(d, dtype=np.uint64), inds[m])
        for mm, dd in enumerate(dims):
            if mm == m:
                extra[mm].append(missing)
            else:
                extra[mm].append(rng.integers(0, dd, size=len(missing), dtype=np.uint64))
    inds2 = [np.concatenate([inds[m]] + extra[m]) for m in range(len(dims))]
    n_extra = len(inds2[0]) - len(vals)
    vals2 = np.concatenate([vals, rng.uniform(0.0, 1.0, size=n_extra)])
    return dims, inds2, vals2


def factor_mats(dims, R, seed=0):
    """Seeded factors, uniform [-3, 3] like the reference's mat_rand (src/util.c:15-23)."""
    rng = np.random.default_rng(1000 + seed)
    return [np.ascontiguousarray(rng.uniform(-3.0, 3.0, size=(d, R))) for d in dims]


def rel_fro(a, b):
    den = np.linalg.norm(b)
    return float(np.linalg.norm(a - b) / (den if den > 0 else 1.0))


# Seeded tensors of the GPU parity tests (dims, nnz); "t3_skew" has Zipf(1) modes 0 and 1.
PARITY_TENSORS = {
    "t2_matrix": ((300, 500), 9000),
    "t3_small": ((13, 7, 11), 150),
    "t3_tiny": ((5, 4, 3), 20),
    "t3_mid": ((300, 200, 400), 20000),
    "t3_long_fibers": ((50, 40, 3000), 30000),
    "t3_skew": ((2000, 1500, 60), 40000),
    "t4": ((40, 30, 50, 20), 15000),
    "t5": ((12, 15, 10, 20, 9), 8000),
    "t6": ((6, 7, 5, 8, 9, 4), 4000),
    "t7": ((5, 6, 4, 5, 7, 4, 6), 3500),
    "t8": ((4, 3, 5, 4, 3, 6, 2, 5), 3000),
}


def parity_tensor(name):
    import zlib
    dims, nnz = PARITY_TENSORS[name]
    skew = [1.0, 1.0, 0] if name == "t3_skew" else None
    return random_coo(dims, nnz, seed=zlib.crc32(name.encode()) % 1000, skew=skew)   # stable seed


def mttkrp_gold(dims, inds, vals, mats):
    """Every mode's MTTKRP from oracle/restate.c, the restatement of the reference's gold
    mttkrp_stream that tests/test_oracle.py pins to output recorded from the reference."""
    from oracle import restate
    return [restate.mttkrp_coo(dims, inds, vals, mats, m) for m in range(len(dims))]
