"""GCP-Adam (Tensor.gcp) on a planted binary tensor of config-2 shape: 10K x 10K x 10K with about
10 M ones.

    python scripts/gcp_bench.py [--ranks 16,32,64] [--steps 400] [--epochs 8]

The ones come from a planted block model: each is drawn from one of 8 components, each component
a block of 600 rows per mode; duplicate coordinates are dropped.  Default sample sizes (65536
stored entries + 65536 coordinates per step, 2^20 + 2^20 for the estimate).  Reported per rank:
  * ms per step and per epoch (CUDA events), each as the difference of a long and a short run,
    so set-up (the decode, the value check, the estimate sample) is not counted;
  * samples per second, and the factor-row bytes the gradient kernel gathers per second
    (N rows of R doubles per sample), to set beside the 7.9 TB/s the root MTTKRP reaches;
  * device time per step of the three kernels, from torch.profiler in a call of its own;
  * with the Gaussian loss: the estimate of ||X - M||^2 after `epochs` epochs and the wall time,
    against CPD-ALS's ||X - M||^2 = ((1 - fit) ||X||)^2 and wall time at the same rank.
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

DIM, NNZ, COMPONENTS, WIDTH = 10_000, 10_000_000, 8, 600


def card():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                           "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                          capture_output=True, text=True).stdout.strip()


def planted(seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    n = int(NNZ * 1.02)
    comp = torch.randint(0, COMPONENTS, (n,), generator=g, device="cuda")
    inds = []
    for _ in range(3):
        start = torch.randint(0, DIM, (COMPONENTS,), generator=g, device="cuda")
        inds.append((start[comp] + torch.randint(0, WIDTH, (n,), generator=g, device="cuda")) % DIM)
    key = torch.unique((inds[0] * DIM + inds[1]) * DIM + inds[2])[:NNZ]
    inds = [(key // (DIM * DIM)), (key // DIM) % DIM, key % DIM]
    return [i.to(torch.int32).contiguous() for i in inds], torch.ones(key.numel(), dtype=torch.float64, device="cuda")


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), out


def kernel_times(fn, names):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {n: [] for n in names}
    for e in prof.events():
        if e.device_type.name == "CUDA":
            for n in names:
                if n in e.name:
                    out[n].append(e.time_range.elapsed_us())
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ranks", default="16,32,64")
    ap.add_argument("--steps", type=int, default=400)
    ap.add_argument("--epochs", type=int, default=8)
    args = ap.parse_args()
    print(json.dumps({"card": card()}))
    inds, vals = planted()
    T = S.Tensor.from_coo([DIM] * 3, inds, vals)
    P = 65536 * 2
    for R in [int(r) for r in args.ranks.split(",")]:
        run = lambda loss, niters, iters, **kw: T.gcp(R, loss, niters=niters, tol=-1.0, epoch_iters=iters,
                                                    max_fails=1000, seed=1, **kw)
        run("bernoulli-logit", 1, 10)                                       # warm-up
        t1, _ = timed(lambda: run("bernoulli-logit", 1, args.steps))
        t2, _ = timed(lambda: run("bernoulli-logit", 1, 2 * args.steps))
        step_ms = (t2 - t1) / args.steps
        t3, _ = timed(lambda: run("bernoulli-logit", 2, args.steps))
        epoch_ms = t3 - t1
        kt = kernel_times(lambda: run("bernoulli-logit", 1, 50), ["k_gcp_sample(", "k_gcp_sampled<", "k_gcp_adam("])
        per = {k: float(np.median(v)) for k, v in kt.items() if v}
        # Gaussian: the estimate of ||X - M||^2 against CPD-ALS at the same rank
        tg, (_, hist, ep, f0) = timed(lambda: run("gaussian", args.epochs, 1000))
        ta, (fit, _, _, its) = timed(lambda: T.cpd_als(R, niters=25, tol=0.0, seed=1))
        als_res = ((1.0 - fit) ** 2) * float(vals.numel())
        print(json.dumps({
            "rank": R, "step_ms": round(step_ms, 4), "epoch_ms_at_steps": [args.steps, round(epoch_ms, 3)],
            "samples_per_s": round(P / step_ms * 1e3, 1),
            "gather_TB_per_s": round(P * 3 * R * 8 / step_ms * 1e3 / 1e12, 3),
            "kernel_us_per_step": {k: round(v, 2) for k, v in per.items()},
            "gaussian_gcp": {"epochs": ep, "s": round(tg / 1e3, 3), "start_estimate": f0,
                             "final_estimate": float(hist[-1, 0]) if ep else None,
                             "best_estimate": float(np.nanmin(hist[:, 0])) if ep else None},
            "cpd_als": {"iterations": its, "s": round(ta / 1e3, 3), "residual_sq": als_res, "fit": fit},
        }))


if __name__ == "__main__":
    main()
