"""When a stream is built for the shared-memory leaf-tile root kernel (splatt_b200_cta_tiling),
and what that kernel computes on tensors the policy tiles without any rank hint."""
import ctypes as C

import numpy as np
import pytest

from splatt_b200 import _abi as A
from tests.util import factor_mats, rel_fro

H100_SMS = 132


def policy(lib, dims, nnz, perm=None, shard_count=1, root_only=1, force=0):
    d = np.ascontiguousarray(dims, dtype=np.uint64)
    p = (C.c_int * len(dims))(*(perm or range(len(dims))))
    rows, acc = C.c_uint32(), C.c_uint32()
    on = lib.splatt_b200_cta_tiling(len(dims), d.ctypes.data_as(A.idx_p), p, nnz, shard_count,
                                    root_only, H100_SMS, force, C.byref(rows), C.byref(acc))
    return on, rows.value, acc.value


def test_headline_tensor_is_tiled(lib):
    """bench.py's headline: 10K^3, 10M nonzeros -- tiled for every root order."""
    for perm in ([0, 1, 2], [1, 0, 2], [2, 1, 0]):
        on, rows, acc = policy(lib, [10_000] * 3, 10_000_000, perm)
        assert on == 1 and rows >= 200 and acc >= 10_000 // H100_SMS + 1, (perm, rows, acc)


@pytest.mark.parametrize("dims,nnz,why", [
    ([100_000] * 3, 100_000_000, "config 4: ~3 nonzeros per (slice, tile) piece"),
    ([1_000_000, 1_000_000, 1_000], 200_000_000, "config 5: root rows per range overflow smem"),
    ([1_000, 1_000_000, 1_000_000], 200_000_000, "config 5: leaf rows re-used < 3x per SM"),
    ([10_000] * 3, 100_000, "small tensor"),
    ([300, 200, 400], 20_000, "small tensor"),
])
def test_generic_where_tiling_does_not_pay(lib, dims, nnz, why):
    assert policy(lib, dims, nnz)[0] == 0, why


def test_generic_for_four_modes_sharded_builds_and_non_root_streams(lib):
    assert policy(lib, [2_000] * 4, 50_000_000)[0] == 0
    assert policy(lib, [10_000] * 3, 5_000_000, shard_count=2)[0] == 0
    assert policy(lib, [10_000] * 3, 10_000_000, root_only=0)[0] == 0


def test_forced_tiling_ignores_the_performance_rules(lib):
    on, rows, acc = policy(lib, [50, 60, 70], 3_000, shard_count=2, root_only=0, force=1)
    assert on == 1 and rows >= 1 and acc >= 50


# ------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def S():
    import splatt_b200
    return splatt_b200


@pytest.fixture(scope="module")
def headline():
    """A tensor the policy tiles on an H100, at a size the suite can afford: 4K^3, 4M nonzeros
    (same per-slice density as bench.py's 10K^3 / 10M)."""
    import torch
    g = torch.Generator(device="cuda").manual_seed(5)
    dims = [4_000] * 3
    nnz = 4_000_000
    ind = [torch.randint(0, d, (nnz,), device="cuda", dtype=torch.int32, generator=g) for d in dims]
    vals = torch.rand(nnz, device="cuda", dtype=torch.float64, generator=g)
    return dims, ind, vals


@pytest.mark.gpu
@pytest.mark.parametrize("R", [2, 31, 32, 33, 64, 128])
def test_default_built_tiled_tensor_matches_untiled(S, headline, R):
    """Default build (no rank hint) runs the tiled kernel, one launch per mode at every rank
    (column slabs inside the launch), and agrees with the generic kernel and with a torch
    fp64 MTTKRP."""
    import torch
    dims, ind, vals = headline
    lib = A.load()
    assert policy(lib, dims, vals.numel())[0] == 1
    T = S.Tensor.from_coo(dims, ind, vals)
    G = S.Tensor.from_coo(dims, ind, vals, ktile=-1)
    ldm = R + (R & 1)                     # rows of every matrix padded to an even length
    mats = [torch.zeros((d, ldm), dtype=torch.float64, device="cuda") for d in dims]
    for x, h in zip(mats, factor_mats(dims, R)):
        x[:, :R] = torch.from_numpy(h)
    idx = [i.long() for i in ind]
    for m in range(3):
        a, b = [x for x in range(3) if x != m]
        gold = torch.zeros((dims[m], R), dtype=torch.float64, device="cuda")
        gold.index_add_(0, idx[m], vals[:, None] * (mats[a][idx[a]] * mats[b][idx[b]])[:, :R])
        out_t = torch.empty((dims[m], ldm), dtype=torch.float64, device="cuda")
        out_g = torch.empty_like(out_t)
        before = S.launch_count()
        T.mttkrp(m, mats, out_t, ncolumns=R)
        assert S.launch_count() - before == 1
        G.mttkrp(m, mats, out_g, ncolumns=R)
        torch.cuda.synchronize()
        got = out_t[:, :R].cpu().numpy()
        assert rel_fro(got, gold.cpu().numpy()) < 1e-12, (R, m)
        assert rel_fro(got, out_g[:, :R].cpu().numpy()) < 1e-13, (R, m)
    T.free()
    G.free()


@pytest.mark.gpu
def test_tiled_column_blocks(S, headline):
    """Column blocks of a tiled stream (what the drop-in's copy/compute pipeline launches)
    run the tiled kernel and fill exactly their columns."""
    import torch
    dims, ind, vals = headline
    R = 40
    T = S.Tensor.from_coo(dims, ind, vals)
    mats = [torch.from_numpy(m).cuda() for m in factor_mats(dims, R)]
    full = torch.empty((dims[0], R), dtype=torch.float64, device="cuda")
    T.mttkrp(0, mats, full)
    part = torch.full_like(full, 7.0)
    ptrs = (A.val_p * 3)(A.val_p(), *[C.cast(C.c_void_p(m.data_ptr()), A.val_p) for m in mats[1:]])
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    before = S.launch_count()
    for c0, c1 in ((0, 18), (18, 40)):
        rc = T.lib.splatt_b200_mttkrp_columns(T.h, 0, R, R, ptrs,
                                              C.cast(C.c_void_p(part.data_ptr()), A.val_p),
                                              c0, c1 - c0, s)
        assert rc == A.SPLATT_SUCCESS
    assert S.launch_count() - before == 2
    torch.cuda.synchronize()
    assert rel_fro(part.cpu().numpy(), full.cpu().numpy()) < 1e-13
    T.free()
