"""Generic vs leaf-tiled root MTTKRP on the bench.py headline tensor (config 2: 10K^3, 10M
nonzeros, rank 32, fp64), built twice in one process and timed alternately.

  generic: Tensor.from_coo(..., ktile=-1)           every nonzero gathers its leaf row from L2
  tiled:   Tensor.from_coo(...)  (default policy)   leaf rows served from shared memory
           --opt-in: SPLATT_B200_TILED=1 and ncolumns_hint=R, for builds whose default is generic

Every launch is timed with CUDA events after a 256 MB write that flushes L2; the two tensors
alternate launch by launch.  Bytes moved L2 -> SM are counted from the streams' shapes:
  generic: leaf rows (one per nonzero) + parent rows (one per fiber) + records
  tiled:   parent rows (one per fiber; tile cuts split some fibers) + one pass of the leaf
           factor per CTA (grid = SMs) + records + root ids
Prints one JSON line with per-mode medians, achieved rates, the gather probe and the card.
usage: python scripts/leaf_tile_compare.py [--launches 60] [--opt-in]"""
import argparse
import json
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402
import splatt_b200 as S  # noqa: E402
from splatt_b200 import _abi as A  # noqa: E402


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True,
                           timeout=30)
        return dict(zip(q.split(","), [x.strip() for x in r.stdout.strip().split(",")]))
    except Exception as e:  # pragma: no cover
        return {"error": str(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=60)
    ap.add_argument("--opt-in", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    R, dims, nnz = bench.RANK, [bench.DIM] * bench.NMODES, bench.NNZ_PER_GPU
    ind, vals = bench.make_coo_gpu(nnz, dev)
    T = {"generic": S.Tensor.from_coo(dims, ind, vals, layout=A.LAYOUT_ALLROOT, ktile=-1)}
    if args.opt_in:
        os.environ["SPLATT_B200_TILED"] = "1"
        T["tiled"] = S.Tensor.from_coo(dims, ind, vals, layout=A.LAYOUT_ALLROOT, ncolumns_hint=R)
        del os.environ["SPLATT_B200_TILED"]
    else:
        T["tiled"] = S.Tensor.from_coo(dims, ind, vals, layout=A.LAYOUT_ALLROOT)
    mats = [torch.from_numpy(m).to(dev) for m in bench.make_factors_host(bench.SEED, dims, R)]
    outs = {k: [torch.empty((d, R), dtype=torch.float64, device=dev) for d in dims] for k in T}
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    pitch = R * 8

    sampler = bench.ClockSampler(0).start()
    times = {k: [[] for _ in dims] for k in T}
    for m in range(len(dims)):
        for k in T:                                     # warm-up
            for _ in range(3):
                T[k].mttkrp(m, mats, outs[k][m])
        for _ in range(args.launches):
            for k in T:
                flush.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                T[k].mttkrp(m, mats, outs[k][m])
                e1.record()
                times[k][m].append((e0, e1))
        torch.cuda.synchronize()
    clocks = sampler.stop()
    probe_gbs, probe_ms = bench.gather_probe_gbs(dev)

    res = {"workload": bench.workload_config(1)["workload"], "launches_per_mode": args.launches,
           "l2": "flushed before every launch (256 MB write)", "card": card(), "clocks": clocks,
           "gather_probe_GBps": probe_gbs, "sms": sms, "modes": []}
    for m in range(len(dims)):
        row = {"mode": m}
        for k in T:
            ms = [a.elapsed_time(b) for a, b in times[k][m]]
            info = T[k].mode_info(m, R)
            nf = info["nfibs"]
            leaf = dims[info["level_perm"][-1]]
            if k == "generic":
                byts = nf[-1] * pitch + nf[-2] * pitch + nf[-1] * 16
            else:
                byts = nf[-2] * pitch + sms * leaf * pitch + nf[-1] * (16 + 4)
            med = float(np.median(ms))
            row[k] = {"ms_median": med, "ms_min": float(min(ms)), "ms_max": float(max(ms)),
                      "nfibs": nf, "l2_to_sm_bytes": int(byts),
                      "l2_to_sm_GBps": byts / (med * 1e-3) / 1e9}
        row["tiled_over_generic"] = row["tiled"]["ms_median"] / row["generic"]["ms_median"]
        row["rel_fro_tiled_vs_generic"] = bench.rel_fro(outs["tiled"][m].cpu().numpy(),
                                                        outs["generic"][m].cpu().numpy())
        res["modes"].append(row)
    for m in res["modes"]:
        print(f"mode {m['mode']}: generic {m['generic']['ms_median']:.3f} ms "
              f"({m['generic']['l2_to_sm_GBps']:.0f} GB/s)  tiled {m['tiled']['ms_median']:.3f} ms "
              f"({m['tiled']['l2_to_sm_GBps']:.0f} GB/s)  ratio {m['tiled_over_generic']:.3f}  "
              f"rel_fro {m['rel_fro_tiled_vs_generic']:.1e}", file=sys.stderr)
    print(json.dumps(res))
    for t in T.values():
        t.free()


if __name__ == "__main__":
    main()
