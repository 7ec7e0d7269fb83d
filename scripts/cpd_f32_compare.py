"""fp64 vs fp32 CPD-ALS on a device tensor (Tensor.cpd_als: splatt_b200_cpd_als_device and
_f32) on configs 2 and 4 (BASELINE.json configs[1] and [3], one GPU), each tensor built once.

Both precisions start from the same factors (the fp32 start is the fp64 one rounded) and run
alternately, --reps times each.  Time per iteration is the difference of two runs of k1 and k2
iterations at tol = 0, divided by k2 - k1 (bench.py's method for cpd_als_iteration): set-up,
||X||^2, Grams and post-processing cancel.  Each run is timed on the host around the call, which
ends in a stream synchronisation.  Reports both fits after k1 and k2 iterations and the largest
|fit32 - fit64|, with the card, power limit and SM clock read in the same run.
Prints one JSON document (and writes it to --json PATH if given).
usage: python scripts/cpd_f32_compare.py [--reps 5] [--configs 2,4] [--json PATH]"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402
import splatt_b200 as S  # noqa: E402

# config: (dims, nnz, rank, seed, k1, k2) -- generator and seeds of scripts/f32_compare.py
# (k2 - k1 iterations take >= 100 ms, well above the run-to-run spread of one call's set-up)
CONFIGS = {"2": ([10_000] * 3, 10_000_000, 32, 1, 2, 52),
           "4": ([100_000] * 3, 100_000_000, 32, 3, 2, 12)}


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else f"nvidia-smi failed: {r.stderr}"


def timed(T, R, start, niters):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fit, _, _, its = T.cpd_als(R, start, niters=niters, tol=0.0)
    dt = time.perf_counter() - t0
    assert its == niters
    return fit, dt


def run_config(name, reps):
    dims, nnz, R, seed, k1, k2 = CONFIGS[name]
    ind, vals = bench.make_coo_gpu(nnz, torch.device("cuda"), dims=dims, seed=seed)
    T = S.Tensor.from_coo(dims, ind, vals)
    del ind, vals
    g = torch.Generator(device="cuda").manual_seed(100 + seed)
    s64 = [torch.empty((d, R), dtype=torch.float64, device="cuda").uniform_(-3, 3, generator=g)
           for d in dims]
    starts = {"f64": s64, "f32": [s.float() for s in s64]}
    for p in ("f64", "f32"):                       # warm-up: module loads, allocator
        timed(T, R, starts[p], 1)
    per_it = {"f64": [], "f32": []}
    fits = {"f64": {}, "f32": {}}
    for _ in range(reps):
        for p in ("f64", "f32"):
            f1, t1 = timed(T, R, starts[p], k1)
            f2, t2 = timed(T, R, starts[p], k2)
            per_it[p].append((t2 - t1) / (k2 - k1) * 1e3)
            fits[p] = {k1: f1, k2: f2}
    dfit = max(abs(fits["f32"][k] - fits["f64"][k]) for k in (k1, k2))
    out = {"config": name, "dims": dims, "nnz": nnz, "rank": R, "k1": k1, "k2": k2, "reps": reps,
           "ms_per_iteration": {p: {"median": float(np.median(v)), "min": float(min(v)),
                                    "max": float(max(v))} for p, v in per_it.items()},
           "fits": {p: {str(k): v for k, v in f.items()} for p, f in fits.items()},
           "max_abs_dfit": dfit}
    out["speedup_f64_over_f32"] = (out["ms_per_iteration"]["f64"]["median"] /
                                   out["ms_per_iteration"]["f32"]["median"])
    T.free()
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--configs", default="2,4")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    res = {"gpu": gpu_info(), "results": [run_config(c, a.reps) for c in a.configs.split(",")]}
    res["gpu_after"] = gpu_info()
    txt = json.dumps(res, indent=1)
    print(txt)
    if a.json:
        Path(a.json).write_text(txt)


if __name__ == "__main__":
    main()
