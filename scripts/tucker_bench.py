"""Sparse Tucker by HOOI (Tensor.tucker) on the config 2 and config 4 shapes: time per iteration,
the TTMc kernel per mode next to the fp64 MTTKRP at R = R_m on the same tensor, the dense steps'
share of an iteration, the orthogonal-iteration steps per iteration, and a parity check of the
TTMc against an explicit Kronecker sum on 256 sampled rows.

    python scripts/tucker_bench.py [--runs 2:8,2:16,2:32,4:16] [--iters 5]

Uniform seeded nonzeros, cubic ranks R x R x R.  Writes nothing; prints one JSON line per run
and the card it ran on.
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

CONFIGS = {2: (10_000, 10_000_000), 4: (100_000, 100_000_000)}
FP64_PEAK = 34e12        # H100 SXM data sheet, fp64 without tensor cores


def card():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                           "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                          capture_output=True, text=True).stdout.strip()


def kernel_us(fn, names):
    """{name: [device us of every launch, in order]} of one call of fn under torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {n: [] for n in names}
    out["all"] = []
    for e in sorted((e for e in prof.events() if e.device_type.name == "CUDA"),
                    key=lambda e: e.time_range.start):
        out["all"].append(e.time_range.elapsed_us())
        for n in names:
            if n in e.name:
                out[n].append(e.time_range.elapsed_us())
    return out


def timed(fn, reps):
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms))


def parity(T, inds, vals, U, R, nrows=256):
    """Mode 0's TTMc on sampled rows against sum_x v_x U_1[j] (x) U_2[k] formed with torch."""
    dim = U[0].shape[0]
    Y = torch.empty((dim, R * R), dtype=torch.float64, device="cuda")
    T.ttmc(0, U, Y, [R, R, R])
    rows = torch.randperm(dim, generator=torch.Generator(device="cuda").manual_seed(5), device="cuda")[:nrows]
    pick = torch.isin(inds[0], rows)
    K = (U[1][inds[1][pick].long()][:, :, None] * U[2][inds[2][pick].long()][:, None, :]).reshape(-1, R * R)
    want = torch.zeros((dim, R * R), dtype=torch.float64, device="cuda")
    want.index_add_(0, inds[0][pick].long(), vals[pick, None] * K)
    return float((Y[rows] - want[rows]).norm() / want[rows].norm())


def run(cfg, R, iters):
    dim, nnz = CONFIGS[cfg]
    dims = [dim] * 3
    g = torch.Generator(device="cuda").manual_seed(cfg)
    inds = [torch.randint(0, dim, (nnz,), device="cuda", dtype=torch.int32, generator=g) for _ in dims]
    vals = torch.rand(nnz, device="cuda", dtype=torch.float64, generator=g)
    T = S.Tensor.from_coo(dims, inds, vals)
    ranks = [R] * 3
    # a converged start, so that the timed iterations run the steady state's power steps
    _, U, _, _ = T.tucker(ranks, niters=3, tol=0.0)
    U = [u.contiguous() for u in U]
    one = lambda: T.tucker(ranks, U, niters=1, tol=0.0)          # noqa: E731
    one()
    it_ms = timed(one, iters)
    kt = kernel_us(one, ["k_ttmc<", "k_ttmc_combine"])
    comb = kt["k_ttmc_combine"][-3:] or [0.0] * 3      # leaf-tiled streams have no combine step
    ttmc_ms = [(a + b) / 1e3 for a, b in zip(kt["k_ttmc<"][-3:], comb)]
    gpu_ms = sum(kt["all"]) / 1e3
    _, _, hist, _ = T.tucker(ranks, U, niters=1, tol=0.0)
    ldm = R + (R & 1)
    mats = [torch.zeros((d, ldm), dtype=torch.float64, device="cuda") for d in dims]
    for x, u in zip(mats, U):
        x[:, :R].copy_(u)
    out = torch.empty((dim, ldm), dtype=torch.float64, device="cuda")
    mt = []
    for m in range(3):
        T.mttkrp(m, mats, out, ncolumns=R)
        mt.append(timed(lambda: T.mttkrp(m, mats, out, ncolumns=R), 10))
    flop = 2.0 * R * R * nnz           # upper bound: one C-entry FMA pass per nonzero (per fiber close)
    res = {
        "config": cfg, "dims": dims, "nnz": nnz, "ranks": ranks,
        "ms_per_iteration_median": it_ms,
        "ttmc_ms_per_mode": ttmc_ms,
        "mttkrp_fp64_ms_per_mode_at_R": mt,
        "ttmc_over_mttkrp": [a / b for a, b in zip(ttmc_ms, mt)],
        "gpu_kernel_ms_per_iteration": gpu_ms,
        "dense_share_of_iteration": (it_ms - sum(ttmc_ms)) / it_ms,
        "power_steps_per_iteration": float(hist[0, 2]),
        "ttmc_fp64_share_of_peak_upper_bound": [flop / (t * 1e-3) / FP64_PEAK for t in ttmc_ms],
        "parity_rel_err_256_rows": parity(T, inds, vals, U, R),
    }
    T.free()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", default="2:8,2:16,2:32,4:16")
    ap.add_argument("--iters", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("tucker_bench.py needs a GPU")
    print(json.dumps({"card": card()}), flush=True)
    for run_ in a.runs.split(","):
        cfg, R = (int(x) for x in run_.split(":"))
        print(json.dumps(run(cfg, R, a.iters)), flush=True)


if __name__ == "__main__":
    main()
