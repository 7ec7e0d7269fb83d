"""The leaf-tiled 3-mode root MTTKRP on forced small leaf tiles: tiles where a lane group has
no records or fewer than a gather batch, record counts that are not a multiple of the batch,
warps whose part of a tile takes several staging rounds, many tile loads by whichever warp
finishes a tile last, and column slabs."""
import ctypes as C

import pytest

from splatt_b200 import _abi as A
from tests.util import factor_mats, rel_fro

# (dims, nonzeros, leaf-tile rows): ~0-3 records per lane group and tile; several staging
# rounds per warp and tile
SHAPES = [((300, 250, 400), 60_000, 7), ((200, 150, 40), 1_200_000, 16)]


@pytest.fixture(scope="module")
def S():
    import splatt_b200
    return splatt_b200


def _coo(dims, nnz, seed):
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    ind = [torch.randint(0, d, (nnz,), device="cuda", dtype=torch.int32, generator=g) for d in dims]
    vals = torch.rand(nnz, device="cuda", dtype=torch.float64, generator=g) - 0.5
    return ind, vals


def _tiled(S, monkeypatch, dims, ind, vals, rows):
    monkeypatch.setenv("SPLATT_B200_TILED", "2")
    monkeypatch.setenv("SPLATT_B200_TILE_ROWS", str(rows))
    T = S.Tensor.from_coo(dims, ind, vals)
    monkeypatch.delenv("SPLATT_B200_TILED")
    monkeypatch.delenv("SPLATT_B200_TILE_ROWS")
    return T


@pytest.mark.gpu
@pytest.mark.parametrize("shape", range(len(SHAPES)))
@pytest.mark.parametrize("R", [2, 16, 31, 32, 33, 64, 128])
def test_forced_small_tiles_match_torch_and_untiled(S, monkeypatch, shape, R):
    import torch
    dims, nnz, rows = SHAPES[shape]
    ind, vals = _coo(dims, nnz, seed=11 + shape)
    T = _tiled(S, monkeypatch, dims, ind, vals, rows)
    G = S.Tensor.from_coo(dims, ind, vals, ktile=-1)
    ldm = R + (R & 1)
    mats = [torch.zeros((d, ldm), dtype=torch.float64, device="cuda") for d in dims]
    for x, h in zip(mats, factor_mats(dims, R, seed=3)):
        x[:, :R] = torch.from_numpy(h)
    idx = [i.long() for i in ind]
    for m in range(3):
        a, b = [x for x in range(3) if x != m]
        gold = torch.zeros((dims[m], R), dtype=torch.float64, device="cuda")
        gold.index_add_(0, idx[m], vals[:, None] * (mats[a][idx[a]] * mats[b][idx[b]])[:, :R])
        out_t = torch.full((dims[m], ldm), 9.0, dtype=torch.float64, device="cuda")
        out_g = torch.empty_like(out_t)
        before = S.launch_count()
        T.mttkrp(m, mats, out_t, ncolumns=R)
        assert S.launch_count() - before == 1          # one tiled launch, slabs inside
        G.mttkrp(m, mats, out_g, ncolumns=R)
        torch.cuda.synchronize()
        got = out_t[:, :R].cpu().numpy()
        assert rel_fro(got, gold.cpu().numpy()) < 1e-12, (shape, R, m)
        assert rel_fro(got, out_g[:, :R].cpu().numpy()) < 1e-13, (shape, R, m)
    T.free()
    G.free()


@pytest.mark.gpu
@pytest.mark.parametrize("shape", range(len(SHAPES)))
def test_forced_small_tiles_column_blocks(S, monkeypatch, shape):
    """Column blocks that split a 32-wide slab, launched separately, fill exactly their
    columns and add up to the whole product."""
    import torch
    dims, nnz, rows = SHAPES[shape]
    ind, vals = _coo(dims, nnz, seed=21 + shape)
    T = _tiled(S, monkeypatch, dims, ind, vals, rows)
    R = 72
    mats = [torch.from_numpy(x).cuda() for x in factor_mats(dims, R, seed=4)]
    for m in range(3):
        full = torch.empty((dims[m], R), dtype=torch.float64, device="cuda")
        T.mttkrp(m, mats, full)
        part = torch.full_like(full, 7.0)
        ptrs = (A.val_p * 3)(*[A.val_p() if k == m else C.cast(C.c_void_p(x.data_ptr()), A.val_p)
                               for k, x in enumerate(mats)])
        s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        for c0, c1 in ((0, 10), (10, 46), (46, 72)):
            rc = T.lib.splatt_b200_mttkrp_columns(T.h, m, R, R, ptrs,
                                                  C.cast(C.c_void_p(part.data_ptr()), A.val_p),
                                                  c0, c1 - c0, s)
            assert rc == A.SPLATT_SUCCESS
        torch.cuda.synchronize()
        assert rel_fro(part.cpu().numpy(), full.cpu().numpy()) < 1e-13, (shape, m)
    T.free()
