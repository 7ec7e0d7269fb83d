"""Every MTTKRP kernel the dispatcher can launch, against an elementwise fp64 bound.

The dispatcher picks a kernel by mode count N (2..8), lane-group width L (4/8/16/32 lanes,
set by the columns of each 64-column pass), kind (root / internal / leaf output) and, for
the root kernel, a batch variant.  CASES below names the (N, layout, R, ldm) runs that reach
every (N, kind, L) and a multi-pass call for every (N, kind); a CPU test derives what each
row reaches from the library's own level orders and fails if any row is dropped.

The oracle is plain torch fp64 on the device (gather the factor rows, multiply,
index_add_).  For output row i with n_i nonzeros, every entry of [:, :R] must satisfy

    |out - ref| <= 2 * gamma(n_i + N) * absref,   gamma(k) = k u / (1 - k u),  u = 2^-53,

where absref is the same product on |vals| and |factors|.  That holds for any summation
order (RED partials, FMAs, the oracle's own atomics) and catches one dropped or doubled
nonzero in a row of fewer than ~1e7 comparable terms.  Rows without nonzeros must be
exactly +0.0.  Factor rows no nonzero references, and every pad column [R, ldm), hold NaN,
so a kernel that reads a wrong row or column fails.  Whole-matrix calls must leave
[rpad, ldm) zero; column-block calls must leave everything outside the block bit-identical.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

from splatt_b200 import _abi as A
from tests.util import random_coo

ROOT = Path(__file__).resolve().parent.parent
U = 2.0 ** -53
NAN = float("nan")
CANARY = -1.2345e300
ALLROOT, ONEMODE, TILED = "allroot", "onemode", "tiled"
LANES = (4, 8, 16, 32)
BIG = 1 << 29                      # the largest row count the stream format holds


# ---------------------------------------------------------------------------------------
# The case table
# ---------------------------------------------------------------------------------------
# Per mode count: base dims and nonzeros of the matrix tensor (each mode gets 3 more rows,
# left empty: the first, the last and one interior slice; see _gapped).
MATRIX = {2: ((300, 500), 9000), 3: ((60, 50, 70), 20000), 4: ((20, 25, 30, 15), 15000),
          5: ((10, 12, 9, 11, 8), 12000), 6: ((6, 7, 5, 8, 6, 5), 8000),
          7: ((5, 4, 6, 5, 4, 6, 5), 8000), 8: ((4, 3, 5, 4, 3, 4, 2, 5), 6000)}

# (N, layout, R, extra leading-dimension columns).  Per (N, layout): an L = 8 row (R = 9 or
# 16), an L = 16 row (R = 17) and a multi-pass row (R = 65: L = 32 then 4; R = 130: 32, 32,
# then 4).  TILED is the CTA-tiled 3-mode stream (SPLATT_B200_TILED=2), one launch with
# 32-column slabs inside.
CASES = [
    (2, ALLROOT, 9, 0), (2, ALLROOT, 17, 6), (2, ALLROOT, 65, 0),
    (2, ONEMODE, 16, 6), (2, ONEMODE, 17, 0), (2, ONEMODE, 130, 6),
    (3, ALLROOT, 16, 0), (3, ALLROOT, 17, 6), (3, ALLROOT, 130, 0),
    (3, ONEMODE, 9, 6), (3, ONEMODE, 17, 0), (3, ONEMODE, 65, 6),
    (3, TILED, 65, 6),
    (4, ALLROOT, 9, 0), (4, ALLROOT, 17, 6), (4, ALLROOT, 65, 0),
    (4, ONEMODE, 16, 6), (4, ONEMODE, 17, 0), (4, ONEMODE, 130, 6),
    (5, ALLROOT, 16, 0), (5, ALLROOT, 17, 6), (5, ALLROOT, 130, 0),
    (5, ONEMODE, 9, 6), (5, ONEMODE, 17, 0), (5, ONEMODE, 65, 6),
    (6, ALLROOT, 9, 0), (6, ALLROOT, 17, 6), (6, ALLROOT, 65, 0),
    (6, ONEMODE, 16, 6), (6, ONEMODE, 17, 0), (6, ONEMODE, 130, 6),
    (7, ALLROOT, 16, 0), (7, ALLROOT, 17, 6), (7, ALLROOT, 130, 0),
    (7, ONEMODE, 9, 6), (7, ONEMODE, 17, 0), (7, ONEMODE, 65, 6),
    (8, ALLROOT, 9, 0), (8, ALLROOT, 17, 6), (8, ALLROOT, 65, 0),
    (8, ONEMODE, 16, 6), (8, ONEMODE, 17, 0), (8, ONEMODE, 130, 6),
]


def _case_id(c):
    return f"n{c[0]}-{c[1]}-R{c[2]}-ldm+{c[3]}"


def _rpad(R):
    return R + (R & 1)


def _passes(c0, c1):
    """Active (even) column counts of the 64-column launches of the block [c0, c1)."""
    end = c1 + (c1 & 1)
    return [min(64, end - c) for c in range(c0, end, 64)]


def _lanes(ncols):
    return 4 if ncols <= 8 else 8 if ncols <= 16 else 16 if ncols <= 32 else 32


def _kind_of_depth(depth, N):
    return "root" if depth == 0 else ("leaf" if depth == N - 1 else "internal")


def _level_orders(lib, dims, alloc):
    d = np.ascontiguousarray(dims, dtype=np.uint64)
    perms = (C.c_int * 64)()
    mp = (C.c_int * 8)()
    n = lib.splatt_b200_level_orders(d.ctypes.data_as(A.idx_p), len(dims), alloc, perms, mp)
    return [[perms[c * 8 + l] for l in range(len(dims))] for c in range(n)]


def _gapped_dims(base):
    return tuple(d + 3 for d in base)


def _kinds(lib, dims, layout):
    """Kernel kind of every mode (ONEMODE: the depth of the mode in the one CSF)."""
    if layout != ONEMODE:
        return ["root"] * len(dims)
    perm = _level_orders(lib, dims, A.CSF_ONEMODE)[0]
    return [_kind_of_depth(perm.index(m), len(dims)) for m in range(len(dims))]


def _covers(lib, case):
    N, layout, R, _ = case
    kinds = set(_kinds(lib, _gapped_dims(MATRIX[N][0]), layout))
    widths = _passes(0, R)
    out = {(N, layout, k, _lanes(w)) for k in kinds for w in widths}
    if len(widths) >= 2:
        out |= {(N, layout, k, "multi") for k in kinds}
    return out


def _required(lib):
    req = {(3, TILED, "root", "multi")}
    for N in range(2, 9):
        for layout in (ALLROOT, ONEMODE):
            for k in set(_kinds(lib, _gapped_dims(MATRIX[N][0]), layout)):
                req |= {(N, layout, k, L) for L in LANES}
                req.add((N, layout, k, "multi"))
    return req


def test_case_table_reaches_every_kernel(lib):
    """CPU: the table reaches every (N, layout, kind, L) and a multi-pass call per (N, layout,
    kind), and every row is the only one to reach something (so no row can be dropped)."""
    req = _required(lib)
    assert {k for N in range(3, 9) for k in _kinds(lib, _gapped_dims(MATRIX[N][0]), ONEMODE)} == \
        {"root", "internal", "leaf"}
    got = [_covers(lib, c) & req for c in CASES]
    assert req - set().union(*got) == set()
    for i, c in enumerate(CASES):
        others = set().union(*(g for j, g in enumerate(got) if j != i))
        assert got[i] - others, f"row {c} reaches nothing the other rows do not"


# ---------------------------------------------------------------------------------------
# Oracle and checks (torch fp64 on the device)
# ---------------------------------------------------------------------------------------
def oracle(dims, ind, vals, mats, mode, R):
    """ref, absref and the nonzeros per output row.  ind: int64 CUDA tensors."""
    import torch
    prod = vals[:, None].expand(-1, R).clone()
    aprod = prod.abs()
    for m in range(len(dims)):
        if m != mode:
            rows = mats[m].index_select(0, ind[m])[:, :R]
            prod *= rows
            aprod *= rows.abs()
    ref = torch.zeros((dims[mode], R), dtype=torch.float64, device=vals.device)
    ref.index_add_(0, ind[mode], prod)
    absref = torch.zeros_like(ref)
    absref.index_add_(0, ind[mode], aprod)
    n = torch.bincount(ind[mode], minlength=dims[mode])
    return ref, absref, n


def check_cols(got, ref, absref, n, N, what):
    """got/ref/absref: the same columns of the output and of the oracle."""
    import torch
    k = (n + N).to(torch.float64)[:, None]
    bound = 2.0 * (k * U / (1.0 - k * U)) * absref
    err = (got - ref).abs()
    bad = ~(err <= bound)                           # NaN fails too
    if bool(bad.any()):
        r, c = [int(x) for x in bad.nonzero()[0]]
        raise AssertionError(f"{what}: {int(bad.sum())} entries out of bound, first at row {r} "
                             f"col {c}: got {float(got[r, c])!r}, want {float(ref[r, c])!r}, "
                             f"bound {float(bound[r, c])!r}, n_i {int(n[r])}")
    empty = got[n == 0]
    assert not bool(torch.signbit(empty).any()), f"{what}: an empty row holds -0.0"


def check_whole(out, R, ora, N, what):
    """A whole-matrix call: [:, :R] within the bound, [rpad, ldm) zeroed."""
    ref, absref, n = ora
    check_cols(out[:, :R], ref, absref, n, N, what)
    tail = out[:, _rpad(R):]
    assert bool((tail == 0).all()) and not bool(tail.signbit().any()), f"{what}: [rpad, ldm) not 0"


def bits(t):
    import torch
    return t.contiguous().view(torch.int64)


def poisoned_factors(dims, ind, R, ldm, seed):
    """Factors uniform in [-3, 3) on the rows some nonzero references; NaN on every other row
    and in the pad columns [R, ldm)."""
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    mats = []
    for d, i in zip(dims, ind):
        x = torch.full((d, ldm), NAN, dtype=torch.float64, device="cuda")
        rows = torch.unique(i)
        x[rows, :R] = torch.rand((len(rows), R), dtype=torch.float64, device="cuda", generator=g) * 6 - 3
        mats.append(x)
    return mats


def _gapped(dims, inds):
    """Spread every mode over d + 3 rows: rows 0, d//2 + 1 and d + 2 stay empty."""
    out = []
    for d, i in zip(dims, inds):
        mid = d // 2
        out.append(np.where(i < mid, i + 1, i + 2).astype(np.uint64))
    return _gapped_dims(dims), out


def matrix_tensor(N):
    """Seeded N-mode tensor with duplicate coordinates and empty first / last / interior
    slices in every mode (numpy)."""
    base, nnz = MATRIX[N]
    _, inds, vals = random_coo(base, nnz, seed=100 + N, unique=False)
    inds = [np.concatenate([i, i[:40]]) for i in inds]            # 40 exact duplicates
    vals = np.concatenate([vals, vals[:40][::-1] - 0.5])
    dims, inds = _gapped(base, inds)
    return list(dims), inds, vals


def to_dev(inds, vals):
    import torch
    ind_d = [torch.from_numpy(np.asarray(i, dtype=np.int64)).cuda() for i in inds]
    return ind_d, torch.from_numpy(np.asarray(vals, dtype=np.float64)).cuda()


def build(S, dims, inds, vals, layout, **kw):
    """inds/vals: numpy, or torch CUDA (int32 / float64)."""
    if layout == TILED:
        # forced CTA tiling with leaf tiles of 16 rows (both read per build)
        os.environ.update(SPLATT_B200_TILED="2", SPLATT_B200_TILE_ROWS="16")
        try:
            return S.Tensor.from_coo(dims, inds, vals, **kw)
        finally:
            del os.environ["SPLATT_B200_TILED"], os.environ["SPLATT_B200_TILE_ROWS"]
    if layout == ONEMODE:
        return S.Tensor.from_coo(dims, inds, vals, layout=A.LAYOUT_ASGIVEN,
                                 csf_alloc=A.CSF_ONEMODE, ktile=-1, **kw)
    return S.Tensor.from_coo(dims, inds, vals, ktile=-1, **kw)


def prefix_counts(inds, perm):
    """Distinct level prefixes (= CSF nodes per level) of the coordinates in level order."""
    nnz = len(inds[0])
    if nnz == 0:
        return [0] * len(perm)
    keys = [np.asarray(inds[p], dtype=np.int64) for p in perm]
    order = np.lexsort(keys[::-1])
    new = np.zeros(nnz, dtype=bool)
    new[0] = True
    out = []
    for k in keys:
        s = k[order]
        new[1:] |= s[1:] != s[:-1]
        out.append(int(new.sum()))
    return out


def check_structure(T, inds, what):
    """Every mode's stream holds one node per distinct level prefix (leaf level: one record
    per nonzero)."""
    nnz = len(inds[0])
    for m in range(T.nmodes):
        info = T.mode_info(m, 1)
        want = prefix_counts(inds, info["level_perm"])
        assert info["nfibs"][:-1] == want[:-1], (what, m, info["level_perm"], info["nfibs"], want)
        assert info["nfibs"][-1] == nnz, (what, m)


def run_modes(S, T, dims, ind_d, vals_d, R, ldm, what, launches=None, seed=0):
    """Whole-matrix MTTKRP of every mode into a canary-filled output, checked."""
    import torch
    N = len(dims)
    mats = poisoned_factors(dims, ind_d, R, ldm, seed)
    for m in range(N):
        out = torch.full((dims[m], ldm), CANARY, dtype=torch.float64, device="cuda")
        before = S.launch_count()
        T.mttkrp(m, mats, out, ncolumns=R)
        if launches is not None:
            assert S.launch_count() - before == launches, (what, m, S.launch_count() - before)
        torch.cuda.synchronize()
        check_whole(out, R, oracle(dims, ind_d, vals_d, mats, m, R), N, f"{what} mode {m}")


@pytest.fixture(scope="module")
def S():
    import splatt_b200
    return splatt_b200


# ---------------------------------------------------------------------------------------
# GPU tests
# ---------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_kernel_matrix(S, lib, case):
    N, layout, R, extra = case
    dims, inds, vals = matrix_tensor(N)
    ind_d, vals_d = to_dev(inds, vals)
    T = build(S, dims, inds, vals, layout)
    kinds = _kinds(lib, dims, layout)
    for m in range(N):
        assert T.mode_info(m, R)["kind"] == kinds[m], (case, m)
    if layout != TILED:                # leaf-tile segments break nodes on purpose
        check_structure(T, inds, case)
    launches = 1 if layout == TILED else len(_passes(0, R))
    run_modes(S, T, dims, ind_d, vals_d, R, _rpad(R) + extra, _case_id(case), launches, seed=N)
    T.free()


def _edge_tensors(N):
    """Traversal edges for N modes: (name, dims, inds, vals) in numpy."""
    rng = np.random.default_rng(7 * N)
    out = []
    dims = [2] + [40 + 3 * m for m in range(1, N)]       # mode 0 is the ONEMODE root
    # one root slice holding every nonzero, split over every lane group
    nnz = 150_000
    inds = [np.full(nnz, 1, np.uint64)] + [rng.integers(0, d, nnz).astype(np.uint64) for d in dims[1:]]
    out.append(("one_slice", dims, inds, rng.uniform(-1, 1, nnz)))
    # a path: one node per non-leaf level (one fiber), and a single nonzero
    for n in (1, 200):
        inds = [np.full(n, d // 2, np.uint64) for d in dims[:-1]] + \
            [rng.permutation(dims[-1])[:n].astype(np.uint64) if n <= dims[-1]
             else rng.integers(0, dims[-1], n).astype(np.uint64)]
        out.append((f"path{n}", dims, inds, rng.uniform(-1, 1, n)))
    # lines of 63, 64 and 65 nonzeros along every mode: a node with that many children at
    # whatever level the mode sits in any stream
    fdims = [70 + m for m in range(N)]
    cols = [[] for _ in range(N)]
    for m in range(N):
        for length in (63, 64, 65):
            base = rng.integers(0, 60, N)
            for k in range(N):
                cols[k].append(np.arange(length) if k == m else np.full(length, base[k]))
    inds = [np.concatenate(c).astype(np.uint64) for c in cols]
    out.append(("fanout_63_64_65", fdims, inds, rng.uniform(-1, 1, len(inds[0]))))
    # nonzero counts around the 64-record chunk (duplicates allowed)
    for n in (1, 63, 64, 65, 127, 128, 129):
        d, i, v = random_coo([5 + m for m in range(N)], n, seed=n + N, unique=False)
        out.append((f"nnz{n}", list(d), i, v))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("N", range(2, 9))
def test_traversal_edges(S, N):
    """Single slice, path, fan-outs of 63/64/65, small nonzero counts, an empty tensor:
    every mode, ALLROOT and ONEMODE, at L = 4 and L = 32."""
    import torch
    for name, dims, inds, vals in _edge_tensors(N):
        ind_d, vals_d = to_dev(inds, vals)
        for layout in (ALLROOT, ONEMODE):
            T = build(S, dims, inds, vals, layout)
            check_structure(T, inds, (N, name, layout))
            for R, extra in ((3, 2), (33, 0)):
                run_modes(S, T, dims, ind_d, vals_d, R, _rpad(R) + extra,
                          f"n{N} {name} {layout} R{R}", len(_passes(0, R)), seed=N + R)
            T.free()
    # an empty tensor launches nothing and zeroes the whole output
    e = np.zeros(0, np.uint64)
    dims = [4 + m for m in range(N)]
    for layout in (ALLROOT, ONEMODE):
        T = build(S, dims, [e] * N, np.zeros(0), layout)
        mats = [torch.ones((d, 8), dtype=torch.float64, device="cuda") for d in dims]
        for m in range(N):
            out = torch.full((dims[m], 8), CANARY, dtype=torch.float64, device="cuda")
            before = S.launch_count()
            T.mttkrp(m, mats, out, ncolumns=5)
            assert S.launch_count() == before
            torch.cuda.synchronize()
            assert bool((out == 0).all()) and not bool(out.signbit().any()), (N, layout, m)
        T.free()


RING = {3: (3000, 2000, 1000), 5: (200, 150, 100, 120, 80), 8: (30,) * 8}
RING_NNZ = 5_000_000


def _dev_coo(dims, nnz, seed):
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    ind = [torch.randint(0, d, (nnz,), device="cuda", dtype=torch.int32, generator=g) for d in dims]
    vals = torch.rand(nnz, device="cuda", dtype=torch.float64, generator=g) - 0.5
    return ind, vals


@pytest.mark.gpu
@pytest.mark.parametrize("layout", [ALLROOT, ONEMODE])
@pytest.mark.parametrize("N", sorted(RING))
def test_ring_reuse(S, N, layout):
    """5 M nonzeros, no CTA tiling: every lane group's range spans several times the
    3-stage ring, at every L."""
    dims = list(RING[N])
    ind, vals = _dev_coo(dims, RING_NNZ, seed=N)
    ind_d = [i.long() for i in ind]
    T = build(S, dims, ind, vals, layout)
    for R in (2, 34):
        run_modes(S, T, dims, ind_d, vals, R, _rpad(R), f"ring n{N} {layout} R{R}",
                  len(_passes(0, R)), seed=R)
    T.free()


@pytest.mark.gpu
@pytest.mark.parametrize("layout", [ALLROOT, ONEMODE])
def test_ring_reuse_single_slice(S, layout):
    """5 M nonzeros in one root slice: every lane group's partial lands in one output row
    (n_i = 5 M keeps the bound meaningful)."""
    import torch
    dims = [4, 2000, 3000]
    ind, vals = _dev_coo(dims, RING_NNZ, seed=33)
    ind[0] = torch.full_like(ind[0], 2)
    ind_d = [i.long() for i in ind]
    T = build(S, dims, ind, vals, layout)
    for R in (2, 34):
        run_modes(S, T, dims, ind_d, vals, R, _rpad(R), f"one slice {layout} R{R}",
                  len(_passes(0, R)), seed=R)
    T.free()


def _ptrs(mats, mode):
    return (A.val_p * len(mats))(*[A.val_p() if k == mode else C.cast(C.c_void_p(x.data_ptr()), A.val_p)
                                   for k, x in enumerate(mats)])


def _columns(T, mode, R, ldm, mats, out, c0, count):
    import torch
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    return T.lib.splatt_b200_mttkrp_columns(T.h, mode, R, ldm, _ptrs(mats, mode),
                                            C.cast(C.c_void_p(out.data_ptr()), A.val_p), c0, count, s)


BLOCKS_R = 71                                         # blocks [0,2) [2,60) [60,70) [70,71)
BLOCKS = [(0, 2), (2, 60), (60, 70), (70, 71)]


@pytest.mark.gpu
@pytest.mark.parametrize("layout", [ALLROOT, ONEMODE])
@pytest.mark.parametrize("N", [2, 3, 4, 8])
def test_column_blocks(S, N, layout):
    """Column blocks launched one by one into a canary-filled output: each writes exactly its
    columns (an odd block also its pad column), and together they make the whole product."""
    import torch
    dims, inds, vals = matrix_tensor(N)
    ind_d, vals_d = to_dev(inds, vals)
    T = build(S, dims, inds, vals, layout)
    R = BLOCKS_R
    ldm = _rpad(R) + 6
    mats = poisoned_factors(dims, ind_d, R, ldm, seed=5)
    for m in range(N):
        ref, absref, n = oracle(dims, ind_d, vals_d, mats, m, R)
        out = torch.full((dims[m], ldm), CANARY, dtype=torch.float64, device="cuda")
        for c0, c1 in BLOCKS:
            prev = out.clone()
            before = S.launch_count()
            assert _columns(T, m, R, ldm, mats, out, c0, c1 - c0) == A.SPLATT_SUCCESS
            assert S.launch_count() - before == len(_passes(c0, c1))
            torch.cuda.synchronize()
            w1 = c1 + (c1 & 1)
            what = f"n{N} {layout} mode {m} block [{c0}, {c1})"
            assert torch.equal(bits(out[:, :c0]), bits(prev[:, :c0])), what
            assert torch.equal(bits(out[:, w1:]), bits(prev[:, w1:])), what
            check_cols(out[:, c0:c1], ref[:, c0:c1], absref[:, c0:c1], n, N, what)
        check_cols(out[:, :R], ref, absref, n, N, f"n{N} {layout} mode {m} union")
        assert bool((out[:, _rpad(R):] == CANARY).all())
    T.free()


@pytest.mark.gpu
@pytest.mark.parametrize("layout", [ALLROOT, ONEMODE, TILED])
def test_invalid_column_blocks_rejected(S, layout):
    """An odd col_begin, a col_begin at or past the padded rank and a block that ends past it
    return SPLATT_ERROR_BADINPUT and touch nothing: every matrix is a view between guard
    rows of its allocation, so a call that did write past the block changes memory the test
    owns."""
    import torch
    N = 3
    dims, inds, vals = matrix_tensor(N)
    ind_d, vals_d = to_dev(inds, vals)
    T = build(S, dims, inds, vals, layout)
    for R, ldm, bad in ((6, 6, [(1, 2), (6, 2), (8, 2), (4, 3), (2, 5)]),
                        (5, 6, [(4, 3), (3, 2), (6, 1)])):
        mats = []
        for x in poisoned_factors(dims, ind_d, R, ldm, seed=R):
            g = torch.full((x.shape[0] + 2, ldm), CANARY, dtype=torch.float64, device="cuda")
            g[1:-1] = x
            mats.append(g[1:-1])
        for m in range(N):
            buf = torch.full((dims[m] + 2, ldm), CANARY, dtype=torch.float64, device="cuda")
            out = buf[1:-1]
            for c0, cnt in bad:
                assert _columns(T, m, R, ldm, mats, out, c0, cnt) == A.SPLATT_ERROR_BADINPUT, \
                    (layout, R, m, c0, cnt)
                torch.cuda.synchronize()
                assert bool((buf == CANARY).all()), (layout, R, m, c0, cnt)
            # the widest legal blocks still run: [4, 6) and, for R = 5, the odd [4, 5)
            ref, absref, n = oracle(dims, ind_d, vals_d, mats, m, R)
            for c0, cnt in ((4, 2), (4, 1)):
                if c0 + cnt > R:
                    continue
                buf.fill_(CANARY)
                assert _columns(T, m, R, ldm, mats, out, c0, cnt) == A.SPLATT_SUCCESS
                torch.cuda.synchronize()
                assert bool((buf[0] == CANARY).all()) and bool((buf[-1] == CANARY).all())
                assert bool((out[:, :c0] == CANARY).all())
                check_cols(out[:, c0:c0 + cnt], ref[:, c0:c0 + cnt], absref[:, c0:c0 + cnt], n, N,
                           (layout, R, m, c0, cnt))
    T.free()


@pytest.mark.gpu
@pytest.mark.parametrize("layout", [ALLROOT, ONEMODE])
def test_max_row_index(S, layout):
    """dims (2^29, 2^29, 3): indices 0 and 2^29 - 1 in both large modes, R = 1 (ldm 2)."""
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < 32 * 2 ** 30:
        pytest.skip(f"needs 32 GiB of free device memory for two 2^29 x 2 fp64 matrices "
                    f"(has {free / 2 ** 30:.1f} GiB)")
    rng = np.random.default_rng(29)
    dims = [BIG, BIG, 3]
    nnz = 400
    i0 = rng.integers(0, BIG, nnz)
    i1 = rng.integers(0, BIG, nnz)
    i0[:4] = [0, BIG - 1, BIG - 1, 0]
    i1[:4] = [BIG - 1, 0, BIG - 1, 0]
    i0[10:40] = BIG - 1                      # a row with many nonzeros at the last index
    i1[40:70] = 0
    inds = [i0.astype(np.uint64), i1.astype(np.uint64), rng.integers(0, 3, nnz).astype(np.uint64)]
    vals = rng.uniform(-1, 1, nnz)
    T = build(S, dims, inds, vals, layout)
    check_structure(T, inds, layout)
    ind_d, vals_d = to_dev(inds, vals)
    R, ldm = 1, 2
    g = torch.Generator(device="cuda").manual_seed(3)
    for m in range(3):
        mats = []
        for k, (d, i) in enumerate(zip(dims, ind_d)):
            if k == m:
                mats.append(None)
                continue
            x = torch.empty((d, ldm), dtype=torch.float64, device="cuda")   # only used rows written
            rows = torch.unique(i)
            x[rows, 0] = torch.rand(len(rows), dtype=torch.float64, device="cuda", generator=g) * 6 - 3
            x[rows, 1] = NAN
            mats.append(x)
        out = torch.empty((dims[m], ldm), dtype=torch.float64, device="cuda")
        before = S.launch_count()
        T.mttkrp(m, mats, out, ncolumns=R)
        assert S.launch_count() - before == 1
        torch.cuda.synchronize()
        # the oracle on the compacted output rows
        rows, inv = torch.unique(ind_d[m], return_inverse=True)
        cdims = list(dims)
        cdims[m] = len(rows)
        cind = list(ind_d)
        cind[m] = inv
        ref, absref, n = oracle(cdims, cind, vals_d, mats, m, R)
        check_cols(out[rows, :R], ref, absref, n, 3, f"{layout} mode {m}")
        out[rows] = 0.0
        assert int(torch.count_nonzero(out)) == 0, (layout, m)
        del mats, out
        torch.cuda.empty_cache()
    T.free()


@pytest.mark.gpu
def test_too_many_rows_rejected(S):
    e = np.zeros(1, np.uint64)
    for layout in (ALLROOT, ONEMODE):
        for m in range(3):
            dims = [4, 5, 6]
            dims[m] = BIG + 1
            with pytest.raises(S.SplattError) as ei:
                build(S, dims, [e, e, e], np.ones(1), layout)
            assert ei.value.code == A.SPLATT_ERROR_BADINPUT


# Sort-key widths: one 64-bit LSD pass, two (65, 69, 80, 81 bits) and three (136 bits).
SORT_DIMS = [
    (65536,) * 4,
    (65537, 65536, 65536, 65536),
    (40000, 55000, 70000, 48000, 62000),
    (600, 590, 610, 600, 605, 595, 600, 600),
    (2 ** 22 + 3,) * 3,
    (70000,) * 8,
]


def _clustered_coo(dims, nnz, seed):
    """Indices drawn from ~40 values per mode (0 and d - 1 included), so that nodes share
    prefixes at every level; unique coordinates."""
    rng = np.random.default_rng(seed)
    inds = []
    for d in dims:
        pool = np.unique(np.concatenate([[0, d - 1], rng.integers(0, d, 38)]))
        inds.append(pool[rng.integers(0, len(pool), nnz)].astype(np.uint64))
    key = np.stack(inds, axis=1)
    _, first = np.unique(key, axis=0, return_index=True)
    first.sort()
    return [i[first] for i in inds], rng.uniform(-1, 1, len(first))


def numpy_csf(dims, inds, vals, perm):
    """The CSF of the coordinates in level order perm (lexsort)."""
    keys = [np.asarray(inds[p], dtype=np.int64) for p in perm]
    order = np.lexsort(keys[::-1])
    nnz = len(order)
    new = np.zeros(nnz, dtype=bool)
    new[0] = True
    starts = []
    for k in keys:
        s = k[order]
        new[1:] |= s[1:] != s[:-1]
        starts.append(np.flatnonzero(new))
    fids = [keys[l][order][starts[l]] for l in range(len(perm))]
    nfibs = [len(s) for s in starts]
    fptr = [np.append(np.searchsorted(starts[l + 1], starts[l]), nfibs[l + 1])
            for l in range(len(perm) - 1)]
    if nfibs[0] == dims[perm[0]]:
        fids[0] = None
    return {"nfibs": nfibs, "fptr": fptr, "fids": fids, "vals": np.asarray(vals)[order]}


@pytest.mark.gpu
@pytest.mark.parametrize("dims", SORT_DIMS, ids=lambda d: f"{len(d)}x{d[0]}")
def test_structure_at_sort_key_widths(S, lib, dims):
    """splatt_b200_csf_alloc's arrays equal a numpy lexsort CSF builder's, and every
    stream's node counts equal numpy's distinct level prefixes, at sort keys that take one,
    two and three radix passes.  (No MTTKRP runs here: a mis-sorted stream only splits nodes,
    which leaves MTTKRP sums unchanged.)"""
    inds, vals = _clustered_coo(dims, 60_000, seed=len(dims) + dims[0] % 97)
    dims = list(dims)
    o = S.default_opts()
    o[A.OPTION_CSF_ALLOC] = A.CSF_ALLMODE
    csf = S.csf_alloc(dims, inds, vals, o)
    perms = _level_orders(lib, dims, A.CSF_ALLMODE)
    assert csf.count == len(perms)
    for c, perm in enumerate(perms):
        got = csf.arrays(c)
        assert got["dim_perm"] == perm, c
        want = numpy_csf(dims, inds, vals, perm)
        assert got["nfibs"] == want["nfibs"], (c, got["nfibs"], want["nfibs"])
        for l in range(len(dims) - 1):
            assert np.array_equal(got["fptr"][l], want["fptr"][l]), (c, l)
        for l in range(len(dims)):
            if want["fids"][l] is None:
                assert got["fids"][l] is None, (c, l)
            else:
                assert np.array_equal(got["fids"][l], want["fids"][l]), (c, l)
        assert np.array_equal(got["vals"], want["vals"]), c
    csf.free()
    for layout in (ALLROOT, ONEMODE):
        T = build(S, dims, inds, vals, layout)
        check_structure(T, inds, (dims, layout))
        T.free()


# ---------------------------------------------------------------------------------------
# Knobs the library reads once per process: each setting runs in a child process
# ---------------------------------------------------------------------------------------
KNOBS = {
    "batch2_minb4": ({"SPLATT_B200_BATCH": "2", "SPLATT_B200_MINB": "4"}, "engine"),  # 4 modes: 2-stage ring
    "batch3_minb3": ({"SPLATT_B200_BATCH": "3", "SPLATT_B200_MINB": "3"}, "engine"),
    "batch3_minb4": ({"SPLATT_B200_BATCH": "3", "SPLATT_B200_MINB": "4"}, "engine"),
    "batch4_minb4": ({"SPLATT_B200_BATCH": "4", "SPLATT_B200_MINB": "4"}, "engine"),
    "batch3": ({"SPLATT_B200_BATCH": "3"}, "engine"),
    "batch4_minb3": ({"SPLATT_B200_BATCH": "4", "SPLATT_B200_MINB": "3"}, "engine"),
    "batch4": ({"SPLATT_B200_BATCH": "4"}, "engine"),                                 # 5+ modes
    "batch8": ({"SPLATT_B200_BATCH": "8"}, "engine"),
    "stagger1": ({"SPLATT_B200_STAGGER": "1"}, "engine"),
    "stagger2": ({"SPLATT_B200_STAGGER": "2"}, "engine"),
    "tiled_kernel0": ({"SPLATT_B200_TILED_KERNEL": "0"}, "tiled"),
    "stage0": ({"SPLATT_B200_STAGE": "0"}, "dropin"),
    "pipeline0": ({"SPLATT_B200_PIPELINE": "0"}, "dropin"),
}
CHILD_N = (2, 3, 4, 5, 8)
CHILD_R = (3, 33, 70)


def child_main(what):
    """Run in a child process with one knob set: the reduced matrix, checked by the oracle.
    Any mismatch raises (non-zero exit status)."""
    import torch
    import splatt_b200 as S
    if what == "engine":
        for N in CHILD_N:
            dims, inds, vals = matrix_tensor(N)
            ind_d, vals_d = to_dev(inds, vals)
            for layout in (ALLROOT, ONEMODE):
                T = build(S, dims, inds, vals, layout)
                for R in CHILD_R:
                    run_modes(S, T, dims, ind_d, vals_d, R, _rpad(R), f"n{N} {layout} R{R}",
                              len(_passes(0, R)), seed=R)
                T.free()
    elif what == "tiled":
        # a CTA-tiled stream multiplied by the generic kernel (its leaf-tiled variant)
        dims, inds, vals = matrix_tensor(3)
        ind_d, vals_d = to_dev(inds, vals)
        T = build(S, dims, inds, vals, TILED)
        # leaf-tile segments split nodes: the stream really is the tiled one
        assert any(T.mode_info(m, 1)["nfibs"][:-1] != prefix_counts(inds, T.mode_info(m, 1)["level_perm"])[:-1]
                   for m in range(3))
        for R in CHILD_R:
            run_modes(S, T, dims, ind_d, vals_d, R, _rpad(R) + 2, f"tiled R{R}",
                      len(_passes(0, R)), seed=R)
        T.free()
    else:
        # the drop-in entry with pageable host buffers
        for N in (3, 4):
            dims, inds, vals = matrix_tensor(N)
            ind_d, vals_d = to_dev(inds, vals)
            o = S.default_opts()
            csf = S.csf_alloc(dims, inds, vals, o)
            for R in CHILD_R:
                mats = poisoned_factors(dims, ind_d, R, R, seed=R)
                host = [x.cpu().numpy() for x in mats]
                ws = S.MttkrpWorkspace(csf.ptr, R, o)
                for m in range(N):
                    out = np.full((dims[m], R), np.nan)
                    ws.mttkrp_csf(host, m, out)
                    got = torch.from_numpy(out).cuda()
                    ref, absref, n = oracle(dims, ind_d, vals_d, mats, m, R)
                    check_cols(got, ref, absref, n, N, f"dropin n{N} R{R} mode {m}")
                ws.free()
            csf.free()
    torch.cuda.synchronize()
    print(f"child {what} ok")
    return 0


@pytest.mark.gpu
@pytest.mark.parametrize("knob", list(KNOBS))
def test_process_cached_knobs(knob):
    """Each setting of a knob read once per process, in a fresh child process."""
    env_set, what = KNOBS[knob]
    env = {k: v for k, v in os.environ.items() if not k.startswith("SPLATT_B200_")}
    env.update(env_set)
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [
        "-c", "import sys; from tests.test_kernel_matrix import child_main; "
              "sys.exit(child_main(sys.argv[1]))", what]
    r = subprocess.run(cmd, cwd=str(ROOT), env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, f"{knob}: exit {r.returncode}\n{r.stdout[-2000:]}\n{r.stderr[-4000:]}"
    assert f"child {what} ok" in r.stdout
