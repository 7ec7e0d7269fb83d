"""Completion by L-BFGS (Tensor.complete_lbfgs) against row-wise ALS (Tensor.complete) on planted
config-2-shaped tensors: 10K x 10K x 10K, 10 M records, split 90/10 into training and validation.

    python scripts/tc_lbfgs_bench.py [--ranks 16,32,64] [--als-iters 25] [--lbfgs-iters 150]

The values are a planted rank-R model (uniform factors scaled so the mean value is about 1) plus
Gaussian noise of 0.05.  Both solvers start from the same factors.  Reported per rank:
  * ms per iteration (CUDA events, median of 3 alternating repetitions), as the difference of a
    long and a short run divided by the extra iterations, so set-up is not counted;
  * kernel times of one L-BFGS iteration from torch.profiler in a call of its own: the gradient
    walk per mode, the line walk, the vector kernels (dot, axpy, combine) and the validation SSE;
  * the validation RMSE against wall time for both solvers (the per-iteration time times the
    iteration count), and the best validation RMSE each reaches within ALS's wall time.
Writes nothing; prints one JSON line per rank and the card it ran on.
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import splatt_b200 as S  # noqa: E402

DIM, NNZ, NOISE, REG = 10_000, 10_000_000, 0.05, 1e-3


def card():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                           "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                          capture_output=True, text=True).stdout.strip()


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), out


def kernel_times(fn, names):
    """{name: [device us of every launch, in order]} of one call of fn under torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {n: [] for n in names}
    evs = sorted((e for e in prof.events() if e.device_type.name == "CUDA"),
                 key=lambda e: e.time_range.start)
    for e in evs:
        for n in names:
            if n in e.name:
                out[n].append(e.time_range.elapsed_us())
    return out


def run(R, als_iters, lbfgs_iters):
    dims = [DIM] * 3
    g = torch.Generator(device="cuda").manual_seed(R)
    scale = 2.0 / R ** (1.0 / 3.0)
    F = [scale * torch.rand((d, R), dtype=torch.float64, device="cuda", generator=g) for d in dims]
    inds = [torch.randint(0, DIM, (NNZ,), device="cuda", generator=g) for _ in dims]
    x = torch.ones((NNZ, R), dtype=torch.float64, device="cuda")
    for f, i in zip(F, inds):
        x *= f[i]
    vals = x.sum(1) + NOISE * torch.randn(NNZ, dtype=torch.float64, device="cuda", generator=g)
    del x
    cut = NNZ * 9 // 10
    i32 = [i.to(torch.int32) for i in inds]
    T = S.Tensor.from_coo(dims, [i[:cut] for i in i32], vals[:cut])
    V = S.Tensor.from_coo(dims, [i[cut:] for i in i32], vals[cut:])
    f0 = [torch.rand((d, R), dtype=torch.float64, device="cuda", generator=g) for d in dims]

    def als(k):
        return T.complete(R, f0, validate=V, reg=REG, niters=k, tol=0.0)

    def lbfgs(k):
        return T.complete_lbfgs(R, f0, validate=V, reg=REG, niters=k, tol=0.0)

    als(1)
    lbfgs(2)
    per = {"als": [], "lbfgs": []}
    for _ in range(3):                               # alternate the two solvers
        for name, fn, k0, k1 in (("als", als, 2, 6), ("lbfgs", lbfgs, 5, 25)):
            t0, (_, _, i0) = timed(lambda: fn(k0))
            t1, (_, _, i1) = timed(lambda: fn(k1))
            assert (i0, i1) == (k0, k1), (name, i0, i1)
            per[name].append((t1 - t0) / (k1 - k0))
    ms = {k: float(np.median(v)) for k, v in per.items()}

    names = ["k_tcg_grad", "k_tcg_line", "k_tcg_dot", "k_tcg_axpy", "k_tcg_combine", "k_tcg_copy",
             "k_tc_sse"]
    kit = 6
    kt = kernel_times(lambda: lbfgs(kit), names)
    grad = kt["k_tcg_grad"]
    kern = {
        "grad_ms_per_mode": [round(float(np.median(grad[m::3])) / 1e3, 3) for m in range(3)],
        "line_ms": round(float(np.median(kt["k_tcg_line"])) / 1e3, 3),
        "vector_ms_per_iter": round(sum(sum(kt[n]) for n in ("k_tcg_dot", "k_tcg_axpy", "k_tcg_combine",
                                                              "k_tcg_copy")) / kit / 1e3, 3),
        "val_sse_ms": round(float(np.median(kt["k_tc_sse"])) / 1e3, 3),
        "launches_per_iter": round(sum(len(kt[n]) for n in names) / kit, 1),
    }

    ha, _, _ = als(als_iters)
    hl, _, itl = lbfgs(lbfgs_iters)
    budget = len(ha) * ms["als"]
    within = hl[: max(1, min(len(hl), int(budget / ms["lbfgs"])))]
    curve = lambda h, t: [(round((k + 1) * t, 1), float(h[k, 2])) for k in range(len(h))]   # noqa: E731
    return {
        "R": R, "nnz_train": cut, "noise": NOISE, "reg": REG,
        "ms_per_iter": {k: round(v, 3) for k, v in ms.items()},
        "kernels_lbfgs": kern,
        "als": {"iters": len(ha), "wall_ms": round(budget, 1), "val_rmse": float(ha[-1, 2]),
                "best_val_rmse": float(np.min(ha[:, 2]))},
        "lbfgs": {"iters": int(itl), "wall_ms": round(len(hl) * ms["lbfgs"], 1),
                  "val_rmse": float(hl[-1, 2]), "best_val_rmse": float(np.nanmin(hl[:, 2])),
                  "iters_within_als_wall": len(within),
                  "best_val_rmse_within_als_wall": float(np.nanmin(within[:, 2])),
                  "last_alpha": float(hl[-1, 3])},
        "curve_als": curve(ha, ms["als"])[::max(1, len(ha) // 12)],
        "curve_lbfgs": curve(hl, ms["lbfgs"])[::max(1, len(hl) // 12)],
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ranks", default="16,32,64")
    ap.add_argument("--als-iters", type=int, default=25)
    ap.add_argument("--lbfgs-iters", type=int, default=150)
    a = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    for R in [int(r) for r in a.ranks.split(",")]:
        print(json.dumps(run(R, a.als_iters, a.lbfgs_iters)), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
