"""Nonnegative CPD (Tensor.cpd_nonneg, HALS) against CPD-ALS (Tensor.cpd_als) on a device tensor,
configs 2 and 4 (BASELINE.json configs[1] and [3], one GPU), each tensor built once.

Per (rank, precision) both methods start from the same nonnegative factors (uniform [0, 1), the
fp32 start is the fp64 one rounded) and run alternately, --reps times each.  Time per iteration is
the difference of two runs of k1 and k2 iterations at tol = 0, divided by k2 - k1 (the method of
scripts/cpd_f32_compare.py): set-up, ||X||^2, the start check and post-processing cancel.  Each run
is timed on the host around the call, which ends in a stream synchronisation.

Then, in a separate run under torch.profiler (CUDA activities), one k2 - k1 iteration pair of each
method: the device time per iteration of every kernel, grouped by name (the MTTKRP kernels
together), so that the sweep (k_hals_rows*, k_hals_form) can be set against the solve
(k_solve_rows*, k_form_chol).
Reports the card, power limit and SM clock read in the same run.  Prints one JSON document (and
writes it to --json PATH if given).
usage: python scripts/cpd_nonneg_bench.py [--reps 3] [--configs 2,4] [--ranks 16,32,64]
                                          [--dtypes float64,float32] [--json PATH]"""
import argparse
import json
import re
import subprocess
import sys
import time
from collections import defaultdict
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402
import splatt_b200 as S  # noqa: E402

# config: (dims, nnz, seed, k1, k2) -- generator and seeds of scripts/cpd_f32_compare.py
CONFIGS = {"2": ([10_000] * 3, 10_000_000, 1, 2, 22),
           "4": ([100_000] * 3, 100_000_000, 3, 2, 12)}


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else f"nvidia-smi failed: {r.stderr}"


def call(T, method, R, start, niters):
    if method == "nonneg":
        fit, _, _, its, _ = T.cpd_nonneg(R, start, niters=niters, tol=0.0)
    else:
        fit, _, _, its = T.cpd_als(R, start, niters=niters, tol=0.0)
    assert its == niters
    return fit


def timed(T, method, R, start, niters):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fit = call(T, method, R, start, niters)
    return fit, time.perf_counter() - t0


def kernel_group(name):
    m = re.search(r"(k_\w+?)(<|\(|$)", name)
    base = m.group(1) if m else name
    return "mttkrp" if "mttkrp" in base.lower() or "root" in base.lower() else base


def kernel_ms_per_iteration(T, method, R, start, k1, k2):
    """{kernel group: device ms per iteration}: profiled k2 minus profiled k1 iterations."""
    from torch.profiler import ProfilerActivity, profile
    per = []
    for k in (k1, k2):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call(T, method, R, start, k)
            torch.cuda.synchronize()
        acc = defaultdict(float)
        for e in prof.key_averages():
            if e.device_time_total > 0:
                acc[kernel_group(e.key)] += e.device_time_total / 1e3      # us -> ms
        per.append(acc)
    keys = set(per[0]) | set(per[1])
    out = {k: (per[1].get(k, 0.0) - per[0].get(k, 0.0)) / (k2 - k1) for k in keys}
    return {k: round(v, 4) for k, v in sorted(out.items(), key=lambda kv: -kv[1]) if abs(v) > 1e-4}


def run_config(name, ranks, dtypes, reps):
    dims, nnz, seed, k1, k2 = CONFIGS[name]
    ind, vals = bench.make_coo_gpu(nnz, torch.device("cuda"), dims=dims, seed=seed)
    T = S.Tensor.from_coo(dims, ind, vals)
    del ind, vals
    rows = []
    for R in ranks:
        g = torch.Generator(device="cuda").manual_seed(100 + seed)
        s64 = [torch.empty((d, R), dtype=torch.float64, device="cuda").uniform_(0, 1, generator=g)
               for d in dims]
        for dt in dtypes:
            start = s64 if dt == "float64" else [s.float() for s in s64]
            for m in ("als", "nonneg"):                  # warm-up: module loads, allocator
                call(T, m, R, start, 1)
            per_it = {"als": [], "nonneg": []}
            fits = {}
            for _ in range(reps):
                for m in ("als", "nonneg"):
                    f1, t1 = timed(T, m, R, start, k1)
                    f2, t2 = timed(T, m, R, start, k2)
                    per_it[m].append((t2 - t1) / (k2 - k1) * 1e3)
                    fits[m] = {k1: f1, k2: f2}
            res = {"config": name, "rank": R, "dtype": dt, "k1": k1, "k2": k2, "reps": reps,
                   "ms_per_iteration": {m: {"median": float(np.median(v)), "min": float(min(v)),
                                            "max": float(max(v))} for m, v in per_it.items()},
                   "fits": {m: {str(k): v for k, v in f.items()} for m, f in fits.items()}}
            res["nonneg_over_als"] = (res["ms_per_iteration"]["nonneg"]["median"] /
                                      res["ms_per_iteration"]["als"]["median"])
            rows.append(res)
            print(json.dumps(res), file=sys.stderr, flush=True)
    # kernel times, in a run of their own
    for res in rows:
        R, dt = res["rank"], res["dtype"]
        g = torch.Generator(device="cuda").manual_seed(100 + seed)
        start = [torch.empty((d, R), dtype=torch.float64, device="cuda").uniform_(0, 1, generator=g)
                 for d in dims]
        if dt == "float32":
            start = [s.float() for s in start]
        res["kernel_ms_per_iteration"] = {m: kernel_ms_per_iteration(T, m, R, start, k1, k1 + 4)
                                          for m in ("als", "nonneg")}
    T.free()
    torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--configs", default="2,4")
    ap.add_argument("--ranks", default="16,32,64")
    ap.add_argument("--dtypes", default="float64,float32")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    ranks = [int(r) for r in a.ranks.split(",")]
    dtypes = a.dtypes.split(",")
    res = {"gpu": gpu_info(), "results": []}
    for c in a.configs.split(","):
        res["results"] += run_config(c, ranks, dtypes, a.reps)
    res["gpu_after"] = gpu_info()
    txt = json.dumps(res, indent=1)
    print(txt)
    if a.json:
        Path(a.json).write_text(txt)


if __name__ == "__main__":
    main()
