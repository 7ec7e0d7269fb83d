"""GPU parity: the CUDA path, called through the C ABI, against the reference.

Gold is the reference's own gold (tests/mttkrp_test.c:66), mttkrp_stream on COO, as
oracle/restate.c restates it; tests/test_oracle.py pins that restatement (and its CPD-ALS)
to output recorded from the compiled reference.  CSFs in the reference's layout come from
splatt_b200_csf_alloc, whose arrays test_csf_alloc_matches_reference pins to the ones the
reference's csf_alloc builds.  The north-star bar is 1e-6 relative Frobenius; fp64 with a
different summation order lands ~1e-15, so the tests assert 1e-11 (and the reference's own
abs 1e-10 scaled by magnitude).
"""
import os

import numpy as np
import pytest

from oracle import restate
from tests import recorded
from tests.util import (PARITY_TENSORS, cover_all_slices, factor_mats, mttkrp_gold, parity_tensor,
                        random_coo, rel_fro)

pytestmark = pytest.mark.gpu

TOL = 1e-11

TENSORS = [n for n in PARITY_TENSORS if n != "t3_tiny"]
_tensor = parity_tensor


@pytest.fixture(scope="module")
def S():
    import splatt_b200
    return splatt_b200


@pytest.mark.parametrize("name", list(TENSORS))
@pytest.mark.parametrize("R", [3, 16, 32])
@pytest.mark.parametrize("layout", ["allroot", "asgiven"])
def test_dropin_mttkrp_on_reference_csf(S, name, R, layout, monkeypatch):
    """splatt_mttkrp (ours) on CSFs laid out as the reference's csf_alloc lays them out,
    every mode, every allocation policy -- the drop-in scenario."""
    monkeypatch.setenv("SPLATT_B200_LAYOUT", layout)
    dims, inds, vals = _tensor(name)
    mats = factor_mats(dims, R)
    gold = mttkrp_gold(dims, inds, vals, mats)
    for alloc in (0, 1, 2):
        o = S.default_opts()
        o[0] = 1
        o[6] = alloc
        csf = S.csf_alloc(dims, inds, vals, o)
        for m in range(len(dims)):
            out = S.mttkrp(m, R, csf.ptr, mats, o)
            assert rel_fro(out, gold[m]) < TOL, (name, R, layout, alloc, m)
        csf.free()


@pytest.mark.parametrize("R", [1, 2, 5, 10, 48, 64, 70, 130])
def test_ranks(S, R):
    dims, inds, vals = _tensor("t3_mid")
    mats = factor_mats(dims, R)
    gold = mttkrp_gold(dims, inds, vals, mats)
    o = S.default_opts()
    o[0] = 1
    csf = S.csf_alloc(dims, inds, vals, o)
    for m in range(3):
        out = S.mttkrp(m, R, csf.ptr, mats, o)
        assert rel_fro(out, gold[m]) < TOL, (R, m)


@pytest.mark.parametrize("name", ["t3_mid", "t4", "t5"])
@pytest.mark.parametrize("tilelevel", [0, 1, 2])
def test_dropin_on_densetiled_reference_csf(S, refmod, name, tilelevel):
    """Reference CSFs built with SPLATT_DENSETILE (tests/mttkrp_test.c:201-259); only the
    reference's csf_alloc builds them, so this runs where oracle/_ref is built."""
    dims, inds, vals = _tensor(name)
    R = 8
    mats = factor_mats(dims, R)
    tt = refmod.RefTensor.from_coo(dims, inds, vals)
    gold = mttkrp_gold(dims, inds, vals, mats)
    for alloc in (0, 1, 2):
        o = refmod.default_opts()
        o[0] = 3
        o[6] = alloc
        o[7] = 1          # SPLATT_DENSETILE
        o[8] = tilelevel
        csf = refmod.RefCsf(tt, o)
        for m in range(len(dims)):
            out = S.mttkrp(m, R, csf.ptr, mats, o)
            assert rel_fro(out, gold[m]) < TOL, (name, tilelevel, alloc, m)
        csf.free()


@pytest.mark.parametrize("name", ["t2_matrix", "t3_small", "t3_mid", "t4", "t5", "t8"])
@pytest.mark.parametrize("alloc", [0, 1, 2])
def test_csf_alloc_matches_reference(S, name, alloc):
    """splatt_b200_csf_alloc builds bit-identical CSF arrays to the reference's csf_alloc
    (structure tests of tests/csf_test.c:31-61): sizes, orders and a digest of every array
    against the ones recorded from the reference."""
    dims, inds, vals = _tensor(name)
    o = S.default_opts()
    o[0] = 1
    o[6] = alloc
    want = recorded.csf_digests(name, alloc)
    mine = S.csf_alloc(dims, inds, vals, o)
    assert mine.count == len(want)
    for c in range(mine.count):
        assert recorded.csf_digest(mine.arrays(c)) == want[c], c


def test_csf_alloc_gaps_keep_root_ids(S):
    """Empty root slices => fids[0] is materialised (src/csf.c:303-309)."""
    dims, inds, vals = random_coo((500, 40, 30), 300, seed=5)
    o = S.default_opts()
    o[6] = 0
    mine = S.csf_alloc(dims, inds, vals, o)
    a = mine.arrays(0)
    assert recorded.csf_digest(a) == recorded.csf_digests("gaps", 0)[0]
    R = 4
    mats = factor_mats(dims, R)
    gold = mttkrp_gold(dims, inds, vals, mats)
    for m in range(3):
        assert rel_fro(S.mttkrp(m, R, mine.ptr, mats, o), gold[m]) < TOL


@pytest.mark.parametrize("layout", [0, 1])
@pytest.mark.parametrize("name", ["t2_matrix", "t3_mid", "t3_skew", "t4", "t5"])
def test_engine_device_path(S, name, layout):
    """Device-resident API: COO -> fiber streams -> MTTKRP on torch CUDA tensors."""
    import torch
    dims, inds, vals = _tensor(name)
    R = 16
    mats = factor_mats(dims, R)
    gold = mttkrp_gold(dims, inds, vals, mats)
    T = S.Tensor.from_coo(dims, inds, vals, layout=layout, csf_alloc=1)
    dmats = [torch.from_numpy(m).cuda() for m in mats]
    for m in range(len(dims)):
        info = T.mode_info(m, R)
        if layout == 0:
            assert info["kind"] == "root"
        out = torch.empty((dims[m], R), dtype=torch.float64, device="cuda")
        T.mttkrp(m, dmats, out)
        torch.cuda.synchronize()
        assert rel_fro(out.cpu().numpy(), gold[m]) < TOL, (name, layout, m, info)
    T.free()


@pytest.mark.parametrize("name", ["t3_mid", "t3_long_fibers", "t3_skew", "t4", "t5"])
@pytest.mark.parametrize("ktile", [1, 7, 64])
def test_leaf_tiled_streams(S, name, ktile):
    """Leaf-tile re-ordered streams (the L1-reuse layout) give the same MTTKRP, for the
    root kernels and for the internal/leaf kernels, sharded or not."""
    import torch
    dims, inds, vals = _tensor(name)
    R = 16
    mats = factor_mats(dims, R)
    gold = mttkrp_gold(dims, inds, vals, mats)
    dmats = [torch.from_numpy(m).cuda() for m in mats]
    for layout in (0, 1):
        for world in (1, 3):
            shards = [S.Tensor.from_coo(dims, inds, vals, layout=layout, csf_alloc=0, shard_rank=r,
                                        shard_count=world, ncolumns_hint=R, ktile=ktile)
                      for r in range(world)]
            for m in range(len(dims)):
                acc = torch.zeros((dims[m], R), dtype=torch.float64, device="cuda")
                for s in shards:
                    out = torch.empty_like(acc)
                    s.mttkrp(m, dmats, out)
                    acc += out
                assert rel_fro(acc.cpu().numpy(), gold[m]) < TOL, (name, ktile, layout, world, m)
            for s in shards:
                s.free()


@pytest.mark.parametrize("name", ["t3_small", "t3_mid", "t3_long_fibers", "t3_skew"])
@pytest.mark.parametrize("rows", [1, 5, 37])
@pytest.mark.parametrize("R", [2, 16, 32, 64])
def test_cta_tiled_kernel(S, name, rows, R, monkeypatch):
    """The shared-memory leaf-tile kernel (mttkrp_tiled.cu), forced on small tensors with
    tiny tiles, sharded or not, against the reference's gold."""
    import torch
    monkeypatch.setenv("SPLATT_B200_TILED", "2")
    monkeypatch.setenv("SPLATT_B200_TILE_ROWS", str(rows))
    dims, inds, vals = _tensor(name)
    mats = factor_mats(dims, R)
    gold = mttkrp_gold(dims, inds, vals, mats)
    dmats = [torch.from_numpy(m).cuda() for m in mats]
    for world in (1, 2):
        shards = [S.Tensor.from_coo(dims, inds, vals, shard_rank=r, shard_count=world,
                                    ncolumns_hint=R) for r in range(world)]
        before = S.launch_count()
        for m in range(3):
            acc = torch.zeros((dims[m], R), dtype=torch.float64, device="cuda")
            for s in shards:
                out = torch.empty_like(acc)
                s.mttkrp(m, dmats, out)
                acc += out
            assert rel_fro(acc.cpu().numpy(), gold[m]) < TOL, (name, rows, R, world, m)
        assert S.launch_count() - before == 3 * world
        for s in shards:
            s.free()


def test_sharded_partials_sum_to_whole(S):
    """shard_count > 1: per-shard partial outputs add up to the full MTTKRP
    (what the NCCL all-reduce does across ranks)."""
    import torch
    dims, inds, vals = _tensor("t3_skew")
    R = 32
    mats = factor_mats(dims, R)
    gold = mttkrp_gold(dims, inds, vals, mats)
    dmats = [torch.from_numpy(m).cuda() for m in mats]
    for world in (2, 3, 8):
        for layout in (0, 1):
            shards = [S.Tensor.from_coo(dims, inds, vals, layout=layout, shard_rank=r,
                                        shard_count=world) for r in range(world)]
            assert sum(s.nnz_local for s in shards) == len(vals)
            for m in range(3):
                acc = torch.zeros((dims[m], R), dtype=torch.float64, device="cuda")
                for s in shards:
                    out = torch.empty_like(acc)
                    s.mttkrp(m, dmats, out)
                    acc += out
                assert rel_fro(acc.cpu().numpy(), gold[m]) < TOL, (world, layout, m)


@pytest.mark.parametrize("host_solve", ["0", "1"])
@pytest.mark.parametrize("spec", [((60, 50, 40), 6000, 6), ((30, 25, 20, 15), 5000, 5),
                                  ((200, 150, 100), 30000, 16)])
def test_cpd_als_tracks_reference(S, host_solve, spec, monkeypatch):
    """CPD-ALS: same seed, same iteration count => same fit, lambda and factors, with the
    dense ALS tail on the device (default) and on the host (north-star wording).
    (The reference has no CPD result test; parity here is against the compiled
    reference itself.)"""
    monkeypatch.setenv("SPLATT_B200_HOST_SOLVE", host_solve)
    dims, inds, vals = random_coo(spec[0], spec[1], seed=3)
    dims, inds, vals = cover_all_slices(dims, inds, vals)
    R = spec[2]
    o = S.default_opts()
    o[0] = 1
    o[3] = 8          # iterations
    o[1] = 0.0        # tolerance: run them all
    o[4] = 0          # quiet
    csf = S.csf_alloc(dims, inds, vals, o)
    fit_ref, lam_ref, fac_ref = restate.cpd_als(dims, inds, vals, R, int(o[3]), float(o[1]), 7)
    fit, lam, fac = S.cpd_als(csf.ptr, R, o, seed=7)
    assert abs(fit - fit_ref) < 1e-8
    assert np.allclose(lam, lam_ref, rtol=1e-6, atol=1e-9)
    for a, b in zip(fac, fac_ref):
        assert np.allclose(a, b, rtol=1e-5, atol=1e-8)


def test_cpd_als_rank_deficient_falls_back(S, monkeypatch):
    """Duplicate factor columns cannot arise from random init, so force a singular normal
    matrix with rank > number of distinct rows: both the reference (GELSS) and we
    (pseudo-inverse) must return a finite fit and agree, with the dense ALS tail on the
    device and on the host (SPLATT_B200_HOST_SOLVE=0/1)."""
    dims, inds, vals = random_coo((3, 40, 30), 600, seed=9)
    dims, inds, vals = cover_all_slices(dims, inds, vals)
    o = S.default_opts()
    o[0], o[3], o[1], o[4] = 1, 3, 0.0, 0
    csf = S.csf_alloc(dims, inds, vals, o)
    fit_ref, _, _ = restate.cpd_als(dims, inds, vals, 5, int(o[3]), float(o[1]), 2)      # rank 5 > dims[0] = 3: Gram of mode 0 singular
    for host_solve in ("0", "1"):
        monkeypatch.setenv("SPLATT_B200_HOST_SOLVE", host_solve)
        fit, lam, fac = S.cpd_als(csf.ptr, 5, o, seed=2)
        assert np.isfinite(fit) and np.all(np.isfinite(lam)), host_solve
        assert abs(fit - fit_ref) < 1e-6, (host_solve, fit, fit_ref)


@pytest.mark.parametrize("R", [8, 17, 32, 70])
def test_pinned_dropin_path(S, monkeypatch, R):
    """SPLATT_B200_PIN=1: caller buffers are page-locked on first sight; with page-locked
    buffers and >= 16 columns the call runs as a two-block column pipeline (PCIe copies of one
    block overlap the kernel of the other).  Same results; buffers released with the workspace."""
    monkeypatch.setenv("SPLATT_B200_PIN", "1")
    dims, inds, vals = _tensor("t3_mid")
    mats = factor_mats(dims, R)
    gold = mttkrp_gold(dims, inds, vals, mats)
    o = S.default_opts()
    csf = S.csf_alloc(dims, inds, vals, o)
    for rep in range(2):                      # a second workspace re-registers the same buffers
        ws = S.MttkrpWorkspace(csf.ptr, R, o)
        outs = [np.empty((d, R)) for d in dims]
        for _ in range(2):
            for m in range(3):
                ws.mttkrp_csf(mats, m, outs[m])
                assert rel_fro(outs[m], gold[m]) < TOL
        ws.free()


def test_pinned_shared_maxdim_output(S, monkeypatch):
    """SPLATT_B200_PIN=1 with ONE output buffer of maxdim x R reused for every mode, smallest
    mode first -- what the reference's CPD driver does (src/cpd.c:322-327): the registration
    must grow with the extent actually used."""
    monkeypatch.setenv("SPLATT_B200_PIN", "1")
    dims, inds, vals = random_coo((40, 900, 300), 30000, seed=5)
    R = 16
    mats = factor_mats(dims, R)
    gold = mttkrp_gold(dims, inds, vals, mats)
    o = S.default_opts()
    csf = S.csf_alloc(dims, inds, vals, o)
    ws = S.MttkrpWorkspace(csf.ptr, R, o)
    shared = np.empty((max(dims), R))
    for _ in range(2):
        for m in range(3):
            out = shared[:dims[m]]
            ws.mttkrp_csf(mats, m, out)
            assert rel_fro(out, gold[m]) < TOL, m
    ws.free()


@pytest.mark.parametrize("R", [1, 5, 17, 32])
def test_pageable_paths(S, R):
    """Pageable caller buffers, staged through the workspace's page-locked bounce buffers.
    (SPLATT_B200_STAGE is read once per process: tests/test_kernel_matrix.py runs the
    direct-cudaMemcpy path in a child process.)"""
    dims, inds, vals = _tensor("t3_skew")
    mats = factor_mats(dims, R)
    gold = mttkrp_gold(dims, inds, vals, mats)
    o = S.default_opts()
    csf = S.csf_alloc(dims, inds, vals, o)
    ws = S.MttkrpWorkspace(csf.ptr, R, o)
    for _ in range(2):
        for m in range(3):
            out = np.full((dims[m], R), np.nan)
            ws.mttkrp_csf(mats, m, out)
            assert rel_fro(out, gold[m]) < TOL, (R, m)
    ws.free()


def test_bare_mttkrp_reuses_device_mirror(S, monkeypatch):
    """splatt_mttkrp (no workspace handle; matlab/splatt_mttkrp.c:68) builds the device
    mirror once per tensor: later calls find it in the cache (no stream build), a different
    tensor gets its own, and a tensor whose content changed in place is rebuilt."""
    monkeypatch.setenv("SPLATT_B200_CACHE", "2")
    S.cache_clear()
    dims, inds, vals = _tensor("t3_mid")
    R = 8
    mats = factor_mats(dims, R)
    gold = mttkrp_gold(dims, inds, vals, mats)
    o = S.default_opts()
    csf = S.csf_alloc(dims, inds, vals, o)
    b0 = S.build_count()
    for rep in range(3):
        for m in range(3):
            assert rel_fro(S.mttkrp(m, R, csf.ptr, mats, o), gold[m]) < TOL
        if rep == 0:
            b1 = S.build_count()
            assert b1 - b0 == 3            # one stream per mode (ALLROOT), built on the first call
    assert S.build_count() == b1           # 8 more calls, no rebuild
    # another tensor: its own mirror; the first one is still cached
    d2, i2, v2 = _tensor("t4")
    m2 = factor_mats(d2, R)
    gold2 = mttkrp_gold(d2, i2, v2, m2)
    csf2 = S.csf_alloc(d2, i2, v2, o)
    assert rel_fro(S.mttkrp(0, R, csf2.ptr, m2, o), gold2[0]) < TOL
    b2 = S.build_count()
    assert b2 - b1 == 4
    assert rel_fro(S.mttkrp(1, R, csf.ptr, mats, o), gold[1]) < TOL
    assert S.build_count() == b2
    # values changed in place (same addresses): the fingerprint must not match
    arr = csf.ptr[0].pt[0].vals
    n = int(csf.ptr[0].nnz)
    for c in range(csf.count):
        v = csf.ptr[c].pt[0].vals
        for i in range(n):
            v[i] = 2.0 * v[i]
    assert rel_fro(S.mttkrp(2, R, csf.ptr, mats, o), 2.0 * gold[2]) < TOL
    assert S.build_count() > b2
    del arr
    S.cache_clear()
    # cache off: rebuilt on every call, same answers
    monkeypatch.setenv("SPLATT_B200_CACHE", "0")
    b3 = S.build_count()
    assert rel_fro(S.mttkrp(0, R, csf2.ptr, m2, o), gold2[0]) < TOL
    assert rel_fro(S.mttkrp(0, R, csf2.ptr, m2, o), gold2[0]) < TOL
    assert S.build_count() - b3 == 8


@pytest.mark.parametrize("R", [20, 32, 48, 64])
@pytest.mark.parametrize("generic", ["0", "1"])
def test_cpd_als_tail_kernels(S, monkeypatch, R, generic):
    """The register-tiled solve / SYRK kernels of the device tail (rank padded to 32 / 64) and
    the generic ones (SPLATT_B200_TAIL_GENERIC=1) against the compiled reference."""
    monkeypatch.setenv("SPLATT_B200_TAIL_GENERIC", generic)
    dims, inds, vals = random_coo((260, 150, 100), 40000, seed=17)
    dims, inds, vals = cover_all_slices(dims, inds, vals)
    o = S.default_opts()
    o[0], o[3], o[1], o[4] = 4, 5, 0.0, 0
    csf = S.csf_alloc(dims, inds, vals, o)
    fit_ref, lam_ref, fac_ref = restate.cpd_als(dims, inds, vals, R, int(o[3]), float(o[1]), 9)
    fit, lam, fac = S.cpd_als(csf.ptr, R, o, seed=9)
    assert abs(fit - fit_ref) < 1e-8, (R, generic, fit, fit_ref)
    assert np.allclose(lam, lam_ref, rtol=1e-6, atol=1e-9)
    for a, b in zip(fac, fac_ref):
        assert np.allclose(a, b, rtol=1e-5, atol=1e-8)


def test_cpd_als_rank_128_device_tail(S):
    """Rank 128: the device tail's shared-memory needs (R*R + R*rows doubles for the row
    solve, R*R for the Cholesky) must be sized to the device, not assumed (round-1 advice):
    results still track the compiled reference."""
    dims, inds, vals = random_coo((300, 250, 200), 60000, seed=13)
    dims, inds, vals = cover_all_slices(dims, inds, vals)
    R = 128
    o = S.default_opts()
    o[0], o[3], o[1], o[4] = 4, 3, 0.0, 0
    csf = S.csf_alloc(dims, inds, vals, o)
    fit_ref, lam_ref, fac_ref = restate.cpd_als(dims, inds, vals, R, int(o[3]), float(o[1]), 5)
    fit, lam, fac = S.cpd_als(csf.ptr, R, o, seed=5)
    assert np.isfinite(fit)
    assert abs(fit - fit_ref) < 1e-7, (fit, fit_ref)
    assert np.allclose(lam, lam_ref, rtol=1e-5, atol=1e-8)


def test_alias_output_with_own_factor(S):
    """matrices[mode] may alias matout (matlab/splatt_mttkrp.c:47-68)."""
    dims, inds, vals = _tensor("t3_mid")
    R = 8
    mats = factor_mats(dims, R)
    gold = mttkrp_gold(dims, inds, vals, mats)
    o = S.default_opts()
    csf = S.csf_alloc(dims, inds, vals, o)
    ws = S.MttkrpWorkspace(csf.ptr, R, o)
    for m in range(3):
        mm = [x.copy() for x in mats]
        ws.mttkrp_csf(mm, m, mm[m])       # output written over the mode's own factor
        assert rel_fro(mm[m], gold[m]) < TOL
    ws.free()


# ---------------------------------------------------------------------------------------
# BASELINE.json sizes.  Gold: (1) the reference's gold (oracle/restate.c) on the same tensor
# for the configurations it finishes in seconds on one host thread (configs 2 and 3 at full
# size -- tests/mttkrp_test.c:49-125 is the shape of that check); (2) an independent fp64 formulation in plain
# torch ops (gather rows, multiply, index_add); (3) size-independent properties (linearity in
# the values, agreement of the root kernel with the internal/leaf kernels).
# ---------------------------------------------------------------------------------------
def _torch_mttkrp(dims, ind, vals, mats, mode):
    import torch
    acc = vals.clone().unsqueeze(1).expand(-1, mats[0].shape[1]).clone()
    for m in range(len(dims)):
        if m != mode:
            acc *= mats[m].index_select(0, ind[m].long())
    out = torch.zeros((dims[mode], mats[0].shape[1]), dtype=torch.float64, device=vals.device)
    out.index_add_(0, ind[mode].long(), acc)
    return out


def _gen(dims, nnz, seed, zipf=False):
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    ind = []
    for m, d in enumerate(dims):
        if zipf and m < 2:
            w = 1.0 / torch.arange(1, d + 1, device="cuda", dtype=torch.float64)
            cdf = torch.cumsum(w / w.sum(), 0)
            u = torch.rand(nnz, device="cuda", dtype=torch.float64, generator=g)
            r = torch.searchsorted(cdf, u).clamp_(max=d - 1)
            ind.append(torch.randperm(d, device="cuda", generator=g)[r].to(torch.int32))
        else:
            ind.append(torch.randint(0, d, (nnz,), device="cuda", dtype=torch.int32, generator=g))
    vals = torch.rand(nnz, device="cuda", dtype=torch.float64, generator=g)
    return ind, vals


FULL = {
    "config2_10K3_10M_R32": ((10000, 10000, 10000), 10_000_000, 32, False),
    "config3_5K4_50M_R16": ((5000, 5000, 5000, 5000), 50_000_000, 16, False),
    "config4_shard_100K3_12.5M_R32": ((100000, 100000, 100000), 12_500_000, 32, False),
    "config5_family_zipf_1Mx1Mx1K_25M_R64": ((1000000, 1000000, 1000), 25_000_000, 64, True),
}


@pytest.mark.parametrize("name", ["config2_10K3_10M_R32", "config3_5K4_50M_R16"])
def test_full_size_against_reference(S, name):
    """Full-size BASELINE configs 2 and 3: the CUDA path (device-resident engine AND the
    drop-in C entry on a CSF in the reference's layout) against the reference's gold."""
    import os
    import torch
    dims, nnz, R, zipf = FULL[name]
    ind, vals = _gen(dims, nnz, seed=11, zipf=zipf)
    g = torch.Generator(device="cuda").manual_seed(5)
    mats = [torch.rand(d, R, device="cuda", dtype=torch.float64, generator=g) * 6 - 3 for d in dims]
    mats_h = [m.cpu().numpy() for m in mats]
    ind_h = [i.cpu().numpy().astype(np.uint64) for i in ind]
    vals_h = vals.cpu().numpy()
    o = S.default_opts()
    o[0] = min(len(os.sched_getaffinity(0)), 32)
    csf = S.csf_alloc(list(dims), ind_h, vals_h, o)            # TWOMODE, the reference's layout
    T = S.Tensor.from_coo(dims, ind, vals)
    for m in range(len(dims)):
        gold = restate.mttkrp_coo(list(dims), ind_h, vals_h, mats_h, m)
        out = torch.empty((dims[m], R), dtype=torch.float64, device="cuda")
        T.mttkrp(m, mats, out)
        assert rel_fro(out.cpu().numpy(), gold) < TOL, (name, m)
        if m == 0:                                              # drop-in entry on the host CSF
            assert rel_fro(S.mttkrp(m, R, csf.ptr, mats_h, o), gold) < TOL, (name, "dropin")
    S.cache_clear()
    T.free()
    csf.free()


@pytest.mark.parametrize("name", list(FULL))
def test_full_size_against_torch_fp64(S, name):
    import torch
    dims, nnz, R, zipf = FULL[name]
    ind, vals = _gen(dims, nnz, seed=11, zipf=zipf)
    g = torch.Generator(device="cuda").manual_seed(5)
    mats = [torch.rand(d, R, device="cuda", dtype=torch.float64, generator=g) * 6 - 3 for d in dims]
    T = S.Tensor.from_coo(dims, ind, vals)                      # ALLROOT: root kernels
    T2 = S.Tensor.from_coo(dims, ind, vals, layout=1, csf_alloc=0)   # ONEMODE: root+internal+leaf
    for m in range(len(dims)):
        want = _torch_mttkrp(dims, ind, vals, mats, m)
        out = torch.empty_like(want)
        T.mttkrp(m, mats, out)
        err = (torch.linalg.norm(out - want) / torch.linalg.norm(want)).item()
        assert err < 1e-12, (name, m, err)                       # north-star bar: 1e-6
        out2 = torch.empty_like(want)
        T2.mttkrp(m, mats, out2)
        err2 = (torch.linalg.norm(out2 - want) / torch.linalg.norm(want)).item()
        assert err2 < 1e-12, (name, m, T2.mode_info(m, R)["kind"], err2)
    # linearity in the tensor values: MTTKRP(2.5 * X) = 2.5 * MTTKRP(X)
    T3 = S.Tensor.from_coo(dims, ind, vals * 2.5)
    a = torch.empty((dims[0], R), dtype=torch.float64, device="cuda")
    b = torch.empty_like(a)
    T.mttkrp(0, mats, a)
    T3.mttkrp(0, mats, b)
    assert (torch.linalg.norm(b - 2.5 * a) / torch.linalg.norm(a)).item() < 1e-13
    for t in (T, T2, T3):
        t.free()


def test_degenerate_inputs(S):
    """Edge cases the reference's tests touch: a single nonzero, one long fiber, one
    dense slice, duplicate coordinates, nnz below one chunk and exactly on chunk edges."""
    import torch
    cases = []
    cases.append(([5, 4, 3], [np.array([2], dtype=np.uint64), np.array([1], dtype=np.uint64),
                              np.array([0], dtype=np.uint64)], np.array([1.5])))
    n = 300                       # one fiber holding everything
    cases.append(([3, 3, 500], [np.full(n, 1, np.uint64), np.full(n, 2, np.uint64),
                                np.arange(n, dtype=np.uint64)], np.linspace(0.1, 1, n)))
    n = 256                       # one slice, exactly 4 chunks; duplicates included
    rng = np.random.default_rng(0)
    cases.append(([2, 16, 16], [np.zeros(n, np.uint64), rng.integers(0, 16, n).astype(np.uint64),
                                rng.integers(0, 16, n).astype(np.uint64)], rng.uniform(0, 1, n)))
    for nn in (63, 64, 65, 127, 128, 129):
        d, i, v = random_coo((9, 8, 7), nn, seed=nn, unique=False)
        cases.append((d, i, v))
    for dims, inds, vals in cases:
        R = 6
        mats = factor_mats(dims, R)
        gold = mttkrp_gold(dims, inds, vals, mats)
        dm = [torch.from_numpy(x).cuda() for x in mats]
        for layout in (0, 1):
            T = S.Tensor.from_coo(dims, inds, vals, layout=layout, csf_alloc=0)
            for m in range(len(dims)):
                out = torch.empty((dims[m], R), dtype=torch.float64, device="cuda")
                T.mttkrp(m, dm, out)
                assert rel_fro(out.cpu().numpy(), gold[m]) < TOL, (dims, len(vals), layout, m)
            T.free()


def test_empty_tensor_and_bad_input(S):
    import torch
    from splatt_b200 import _abi as A
    dims = [4, 5, 6]
    e = np.zeros(0, dtype=np.uint64)
    T = S.Tensor.from_coo(dims, [e, e, e], np.zeros(0))
    mats = [torch.ones(d, 4, dtype=torch.float64, device="cuda") for d in dims]
    out = torch.full((4, 4), 7.0, dtype=torch.float64, device="cuda")
    T.mttkrp(0, mats, out)
    torch.cuda.synchronize()
    assert float(out.abs().sum()) == 0.0          # output is zeroed (src/mttkrp.c:1305)
    with pytest.raises(S.SplattError) as ei:      # 1-mode "tensors" are rejected
        S.Tensor.from_coo([4], [e], np.zeros(0))
    assert ei.value.code == A.SPLATT_ERROR_BADINPUT
    with pytest.raises(S.SplattError):            # more than SPLATT_MAX_NMODES modes
        S.Tensor.from_coo([2] * 9, [e] * 9, np.zeros(0))
    # odd leading dimension (rows would not be 16-byte aligned) is rejected by the library
    odd = [torch.ones(d, 5, dtype=torch.float64, device="cuda")[:, :3] for d in dims]
    with pytest.raises(S.SplattError) as ei:
        T.mttkrp(0, odd, torch.ones(4, 5, dtype=torch.float64, device="cuda")[:, :3])
    assert ei.value.code == A.SPLATT_ERROR_BADINPUT


def _libc_rand_factors(dims, R, seed):
    """The reference's factor initialisation: srand(seed), then mat_rand per mode in order
    (src/cpd.c:36-40, src/util.c:15-23: two rand() draws per value)."""
    import ctypes
    libc = ctypes.CDLL(None)
    libc.srand(ctypes.c_uint(seed))
    RAND_MAX = 2147483647
    out = []
    for d in dims:
        a = np.empty((d, R))
        flat = a.reshape(-1)
        for x in range(flat.size):
            v = 3.0 * (libc.rand() / RAND_MAX)
            if libc.rand() % 2 == 0:
                v *= -1
            flat[x] = v
        out.append(a)
    return out


@pytest.mark.parametrize("spec", [((60, 50, 40), 6000, 6), ((30, 25, 20, 15), 5000, 5)])
def test_sharded_cpd_driver_matches_splatt_cpd_als(S, spec):
    """splatt_b200.parallel.cpd_als_sharded (MTTKRP -> exchange -> device tail through the
    splatt_b200_als_tail_* entry points; here world = 1) walks the same trajectory as
    splatt_cpd_als and as the compiled reference."""
    import torch
    from splatt_b200 import parallel
    dims, inds, vals = random_coo(spec[0], spec[1], seed=3)
    dims, inds, vals = cover_all_slices(dims, inds, vals)
    R, seed, its = spec[2], 7, 8
    o = S.default_opts()
    o[0], o[3], o[1], o[4] = 1, its, 0.0, 0
    csf = S.csf_alloc(dims, inds, vals, o)
    fit_ref, lam_ref, fac_ref = restate.cpd_als(dims, inds, vals, R, int(o[3]), float(o[1]), seed)
    init = [torch.from_numpy(a).cuda() for a in _libc_rand_factors(dims, R, seed)]
    T = S.Tensor.from_coo(dims, inds, vals)
    fit, lam, fac, times = parallel.cpd_als_sharded(T, R, init, float(np.sum(vals * vals)),
                                                   niters=its, tol=0.0)
    assert len(times) == its
    assert abs(fit - fit_ref) < 1e-8
    # the reference post-processes (2-normalises factors into lambda, src/cpd.c:391-411)
    lam_pp = lam.copy()
    for m, a in enumerate(fac):
        a = a.cpu().numpy()
        nrm = np.sqrt((a * a).sum(axis=0))
        lam_pp *= nrm
        assert np.allclose(a / nrm, fac_ref[m], rtol=1e-5, atol=1e-8)
    assert np.allclose(lam_pp, lam_ref, rtol=1e-6, atol=1e-9)
