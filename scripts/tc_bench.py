"""Tensor completion (Tensor.complete) on the config 2 and config 4 shapes: time per iteration,
row-update kernel time per mode next to the fp64 MTTKRP of the same mode, SSE kernel time,
achieved fp64 FLOP/s, and a parity check of one sweep against the numpy semantics on 256 rows.

    python scripts/tc_bench.py [--configs 2,4] [--ranks 16,32,64] [--iters 10]

Uniform seeded nonzeros, split 90/10 into training and validation tensors.  Writes nothing;
prints one JSON line per (config, rank) and the card it ran on.
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
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                        "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                       capture_output=True, text=True).stdout.strip()
    return q


def flops_per_mode(nnz, N, R):
    """Per nonzero: R(R+1) for the triangle of h h^T, 2R for v h, (N-2) R for the Hadamard."""
    return nnz * (R * (R + 1) + 2 * R + (N - 2) * R)


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


def parity(T, dims, inds, vals, f0, R, reg, nrows=256):
    """One sweep's mode-0 rows (they depend on the start only) against explicit per-row solves
    of (H^T H + reg I) u = H^T v on 256 sampled rows."""
    _, got, _ = T.complete(R, f0, reg=reg, niters=1)
    g = torch.Generator(device="cuda").manual_seed(5)
    rows = torch.randperm(dims[0], generator=g, device="cuda")[:nrows]
    pick = torch.isin(inds[0], rows)
    i0 = inds[0][pick].long()
    h = torch.ones((int(pick.sum()), R), dtype=torch.float64, device="cuda")
    for m in range(1, len(dims)):
        h *= f0[m][inds[m][pick].long()]
    v = vals[pick]
    worst = 0.0
    for r in rows.tolist():
        sel = i0 == r
        H = h[sel]
        want = torch.linalg.solve(H.T @ H + reg * torch.eye(R, dtype=torch.float64, device="cuda"),
                                  H.T @ v[sel])
        err = float((got[0][r] - want).norm() / max(float(want.norm()), 1e-300))
        worst = max(worst, err)
    return worst


def run(cfg, R, iters, reg=0.1):
    dim, nnz = CONFIGS[cfg]
    dims = [dim] * 3
    g = torch.Generator(device="cuda").manual_seed(cfg)
    inds = [torch.randint(0, dim, (nnz,), device="cuda", dtype=torch.int32, generator=g) for _ in dims]
    vals = torch.rand(nnz, device="cuda", dtype=torch.float64, generator=g)
    cut = nnz * 9 // 10
    T = S.Tensor.from_coo(dims, [i[:cut] for i in inds], vals[:cut])
    V = S.Tensor.from_coo(dims, [i[cut:] for i in inds], vals[cut:])
    f0 = [torch.rand((d, R), dtype=torch.float64, device="cuda", generator=g) for d in dims]

    # end to end: ms per iteration, CUDA events around one-iteration calls, median
    T.complete(R, f0, validate=V, reg=reg, niters=1)
    ms = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        T.complete(R, f0, validate=V, reg=reg, niters=1)
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))

    # kernels of one iteration (profiled in a call of its own)
    kt = kernel_times(lambda: T.complete(R, f0, validate=V, reg=reg, niters=1),
                      ["k_tc_update", "k_tc_solve", "k_tc_sse", "k_tc_sumsq"])
    upd = kt["k_tc_update"]
    # the fp64 MTTKRP of the same modes on the same tensor (CUDA events, median of 10)
    ldm = R + (R & 1)
    mats = [torch.zeros((d, ldm), dtype=torch.float64, device="cuda") for d in dims]
    for x, f in zip(mats, f0):
        x[:, :R].copy_(f)
    out = torch.empty((dim, ldm), dtype=torch.float64, device="cuda")
    mt = []
    for m in range(3):
        T.mttkrp(m, mats, out, ncolumns=R)
        t = []
        for _ in range(10):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            T.mttkrp(m, mats, out, ncolumns=R)
            b.record()
            torch.cuda.synchronize()
            t.append(a.elapsed_time(b))
        mt.append(float(np.median(t)))
    fl = flops_per_mode(cut, 3, R)
    upd_ms = [u / 1e3 for u in upd[:3]]
    res = {
        "config": cfg, "dims": dims, "nnz_train": cut, "nnz_validate": nnz - cut, "rank": R,
        "ms_per_iteration_median": float(np.median(ms)),
        "row_update_ms_per_mode": upd_ms,
        "boundary_solve_ms_per_mode": [u / 1e3 for u in kt["k_tc_solve"][:3]],
        "mttkrp_fp64_ms_per_mode": mt,
        "sse_ms_train_validate": [u / 1e3 for u in kt["k_tc_sse"][:2]],
        "gflop_per_mode": fl / 1e9,
        "row_update_tflops": [fl / (u * 1e-3) / 1e12 for u in upd_ms],
        "share_of_fp64_peak": [fl / (u * 1e-3) / FP64_PEAK for u in upd_ms],
        "parity_max_rel_err_256_rows": parity(T, dims, inds=[i[:cut] for i in inds], vals=vals[:cut],
                                              f0=f0, R=R, reg=reg),
    }
    T.free()
    V.free()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="2,4")
    ap.add_argument("--ranks", default="16,32,64")
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("tc_bench.py needs a GPU")
    print(json.dumps({"card": card()}), flush=True)
    for cfg in (int(c) for c in a.configs.split(",")):
        for R in (int(r) for r in a.ranks.split(",")):
            print(json.dumps(run(cfg, R, a.iters)), flush=True)


if __name__ == "__main__":
    main()
