"""The single-process multi-GPU engine behind the C ABI (splatt_b200/csrc/multi.cu) and the
stream slicing it is built on.

On a 1-GPU box the engine is exercised with a device list that names the same GPU twice
(`SPLATT_B200_DEVICES=0,0`): shards, per-device streams, the event-ordered peer-memory
reduce, the replicated ALS tail and the drop-in plumbing all run; only the NVLink multicast
mapping and the in-kernel group barrier need two real GPUs -- those tests run when
`torch.cuda.device_count() >= 2` and are skipped otherwise.

Gold: the reference's gold mttkrp_stream for MTTKRP and its cpd_als for CPD (reference shape
of the distributed loop: src/mpi/mpi_cpd.c:627-804), both as oracle/restate.c restates them
(pinned to output recorded from the compiled reference by tests/test_oracle.py).  CSFs in the
reference's layout come from splatt_b200_csf_alloc.  "t3_tiny" has fewer chunks than devices:
empty shards.
"""
import numpy as np
import pytest

from oracle import restate
from tests.util import cover_all_slices, factor_mats, mttkrp_gold, parity_tensor, random_coo, rel_fro

pytestmark = pytest.mark.gpu

TOL = 1e-11

_tensor = parity_tensor


@pytest.fixture(scope="module")
def S():
    import splatt_b200
    return splatt_b200


def _ngpus():
    import torch
    return torch.cuda.device_count()


@pytest.mark.parametrize("name", ["t3_mid", "t3_skew", "t4", "t5", "t2_matrix", "t3_tiny"])
@pytest.mark.parametrize("world", [2, 3, 8])
def test_sliced_shards_equal_rank_built_shards(S, name, world):
    """splatt_b200_tensor_shard (slice a whole tensor, re-base node numbers) gives what a
    rank-local build with shard_rank/shard_count gives: same nnz, same node counts, same
    partial MTTKRP -- and the partials sum to the whole."""
    import torch
    dims, inds, vals = _tensor(name)
    R = 16
    mats = factor_mats(dims, R)
    gold = mttkrp_gold(dims, inds, vals, mats)
    dmats = [torch.from_numpy(m).cuda() for m in mats]
    whole = S.Tensor.from_coo(dims, inds, vals)
    acc = [torch.zeros((dims[m], R), dtype=torch.float64, device="cuda") for m in range(len(dims))]
    for r in range(world):
        cut = whole.shard(r, world)
        built = S.Tensor.from_coo(dims, inds, vals, shard_rank=r, shard_count=world)
        assert cut.nnz_local == built.nnz_local
        for m in range(len(dims)):
            ic, ib = cut.mode_info(m, R), built.mode_info(m, R)
            assert ic["nfibs"] == ib["nfibs"], (name, world, r, m)
            assert ic["alg_bytes"] == ib["alg_bytes"]
            oc = torch.empty_like(acc[m])
            ob = torch.empty_like(acc[m])
            cut.mttkrp(m, dmats, oc)
            built.mttkrp(m, dmats, ob)
            torch.cuda.synchronize()
            assert rel_fro(oc.cpu().numpy(), ob.cpu().numpy()) < 1e-13 or float(ob.abs().sum()) == 0
            acc[m] += oc
        cut.free()
        built.free()
    for m in range(len(dims)):
        assert rel_fro(acc[m].cpu().numpy(), gold[m]) < TOL, (name, world, m)
    whole.free()


def _devlists():
    n = _ngpus()
    lists = [[0, 0], [0, 0, 0]]                 # one GPU named several times: peer-reduce path
    if n >= 2:
        lists.append(list(range(min(n, 2))))
    if n >= 4:
        lists.append(list(range(4)))
    if n >= 8:
        lists.append(list(range(8)))
    return lists


@pytest.mark.parametrize("name", ["t3_mid", "t3_skew", "t4", "t2_matrix", "t3_tiny"])
@pytest.mark.parametrize("R", [3, 16, 32, 70])
def test_multi_mttkrp_host_matches_reference(S, name, R):
    """splatt_b200_multi_mttkrp_host on every available device list (duplicated single GPU;
    2/4/8 real GPUs with the fused multicast exchange) vs the reference's gold; repeated
    calls and a changing mode order exercise buffer re-use."""
    dims, inds, vals = _tensor(name)
    mats = factor_mats(dims, R)
    gold = mttkrp_gold(dims, inds, vals, mats)
    o = S.default_opts()
    o[0] = 1
    csf = S.csf_alloc(dims, inds, vals, o)
    for devs in _devlists():
        mg = S.MultiGpu(csf.ptr, int(o[6]), R, devs)
        assert mg.ndevices == len(devs)
        assert sum(mg.nnz_local) == len(vals)
        order = list(range(len(dims))) * 2 + list(reversed(range(len(dims)))) + [0, 0]
        for m in order:
            out = mg.mttkrp_host(m, mats)
            assert rel_fro(out, gold[m]) < TOL, (name, R, devs, m, mg.multicast)
        mg.free()
    csf.free()


@pytest.mark.parametrize("devs", ["0,0", "0,0,0,0"])
def test_dropin_symbols_honour_device_list(S, devs, monkeypatch):
    """SPLATT_B200_DEVICES routes splatt_mttkrp_alloc_ws / splatt_mttkrp_csf / splatt_mttkrp
    through the multi engine (row e' of the scope table: multi-GPU behind the C API)."""
    monkeypatch.setenv("SPLATT_B200_DEVICES", devs)
    dims, inds, vals = _tensor("t3_mid")
    R = 16
    mats = factor_mats(dims, R)
    gold = mttkrp_gold(dims, inds, vals, mats)
    o = S.default_opts()
    csf = S.csf_alloc(dims, inds, vals, o)
    ws = S.MttkrpWorkspace(csf.ptr, R, o)
    outs = [np.empty((d, R)) for d in dims]
    for _ in range(2):
        for m in range(3):
            ws.mttkrp_csf(mats, m, outs[m])
            assert rel_fro(outs[m], gold[m]) < TOL
    ws.free()
    for m in range(3):
        assert rel_fro(S.mttkrp(m, R, csf.ptr, mats, o), gold[m]) < TOL
    csf.free()


def test_dropin_ngpus_env_on_real_gpus(S, monkeypatch):
    if _ngpus() < 2:
        pytest.skip("needs >= 2 GPUs")
    monkeypatch.setenv("SPLATT_B200_NGPUS", str(min(_ngpus(), 8)))
    dims, inds, vals = _tensor("t3_skew")
    R = 32
    mats = factor_mats(dims, R)
    gold = mttkrp_gold(dims, inds, vals, mats)
    o = S.default_opts()
    csf = S.csf_alloc(dims, inds, vals, o)
    ws = S.MttkrpWorkspace(csf.ptr, R, o)
    outs = [np.empty((d, R)) for d in dims]
    for _ in range(3):
        for m in range(3):
            ws.mttkrp_csf(mats, m, outs[m])
            assert rel_fro(outs[m], gold[m]) < TOL
    ws.free()
    csf.free()


@pytest.mark.parametrize("spec", [((60, 50, 40), 6000, 6), ((30, 25, 20, 15), 5000, 5),
                                  ((200, 150, 100), 30000, 16)])
def test_multi_cpd_als_tracks_reference(S, spec):
    """CPD-ALS over several devices: same seed and iteration count as the compiled reference
    => same fit / lambda / factors (the tolerances of the single-GPU CPD test)."""
    dims, inds, vals = random_coo(spec[0], spec[1], seed=3)
    dims, inds, vals = cover_all_slices(dims, inds, vals)
    R = spec[2]
    o = S.default_opts()
    o[0], o[3], o[1], o[4] = 1, 8, 0.0, 0
    csf = S.csf_alloc(dims, inds, vals, o)
    fit_ref, lam_ref, fac_ref = restate.cpd_als(dims, inds, vals, R, int(o[3]), float(o[1]), 7)
    for devs in _devlists():
        mg = S.MultiGpu(csf.ptr, int(o[6]), R, devs)
        fit, lam, fac = mg.cpd_als(o, seed=7)
        assert abs(fit - fit_ref) < 1e-8, (devs, fit, fit_ref)
        assert np.allclose(lam, lam_ref, rtol=1e-6, atol=1e-9)
        for a, b in zip(fac, fac_ref):
            assert np.allclose(a, b, rtol=1e-5, atol=1e-8)
        mg.free()
    csf.free()


def test_splatt_cpd_als_honours_device_list(S, monkeypatch):
    dims, inds, vals = random_coo((60, 50, 40), 6000, seed=3)
    dims, inds, vals = cover_all_slices(dims, inds, vals)
    o = S.default_opts()
    o[0], o[3], o[1], o[4] = 1, 6, 0.0, 0
    csf = S.csf_alloc(dims, inds, vals, o)
    fit_ref, _, _ = restate.cpd_als(dims, inds, vals, 6, int(o[3]), float(o[1]), 11)
    n = _ngpus()
    monkeypatch.setenv("SPLATT_B200_DEVICES", "0,1" if n >= 2 else "0,0")
    fit, lam, fac = S.cpd_als(csf.ptr, 6, o, seed=11)
    assert abs(fit - fit_ref) < 1e-8
    csf.free()


def test_multi_cpd_factors_stay_single_valued(S):
    """An ill-conditioned problem (rank 32 on a 300^3 random tensor): with a tail replicated
    on every device the factor replicas drift apart within ~10 iterations and the fit blows up
    (seen on 2 GPUs).  The engine runs the tail once and hands the factor to the other
    devices, so many iterations later it still tracks the single-GPU run."""
    dims, inds, vals = random_coo((300, 300, 300), 200000, seed=21)
    dims, inds, vals = cover_all_slices(dims, inds, vals)
    R = 32
    o = S.default_opts()
    o[0], o[3], o[1], o[4] = 1, 16, 0.0, 0
    csf = S.csf_alloc(dims, inds, vals, o)
    fit1, _, _ = S.cpd_als(csf.ptr, R, o, seed=3)
    assert 0.0 < fit1 < 1.0
    for devs in _devlists():
        mg = S.MultiGpu(csf.ptr, int(o[6]), R, devs)
        fit, lam, fac = mg.cpd_als(o, seed=3)
        assert np.isfinite(fit) and abs(fit - fit1) < 1e-5, (devs, fit, fit1)
        mg.free()
    csf.free()


def test_real_gpus_use_the_multicast_exchange(S):
    """On an NVSwitch box the engine must come up with the fused multicast exchange (the
    peer-reduce path is only the fallback); SPLATT_B200_MULTICAST=0 forces the fallback."""
    import os
    if _ngpus() < 2:
        pytest.skip("needs >= 2 GPUs")
    dims, inds, vals = _tensor("t3_mid")
    o = S.default_opts()
    csf = S.csf_alloc(dims, inds, vals, o)
    mg = S.MultiGpu(csf.ptr, int(o[6]), 8, [0, 1])
    assert mg.multicast or os.environ.get("SPLATT_B200_MULTICAST") == "0"
    mg.free()
    os.environ["SPLATT_B200_MULTICAST"] = "0"
    try:
        mg = S.MultiGpu(csf.ptr, int(o[6]), 8, [0, 1])
        assert not mg.multicast
        mats = factor_mats(dims, 8)
        gold = restate.mttkrp_coo(dims, inds, vals, mats, 1)
        assert rel_fro(mg.mttkrp_host(1, mats), gold) < TOL
        mg.free()
    finally:
        os.environ.pop("SPLATT_B200_MULTICAST")
    csf.free()
