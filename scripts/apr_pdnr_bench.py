"""CP-APR by PDNR (Tensor.cp_apr_pdnr) and by PQNR (Tensor.cp_apr_pqnr) against MU (Tensor.cp_apr)
on planted Poisson count tensors of the config 2 and config 4 shapes.

    python scripts/apr_pdnr_bench.py [--runs 2:16,2:32,2:64,4:32] [--cap 60] [--tol 1e-4]

The tensor is drawn on the device from a seeded rank-R model: each record's component r with
probability proportional to lambda, then each index from column r of A_m (a few hot rows per
column), duplicates merged into counts.  The three solvers start from the same seeded uniform
start and are alternated.  Per (config, rank) it prints one JSON line with: outer iterations,
lockstep iterations (PDNR, PQNR) and wall time to max kkt < tol (at most --cap outer
iterations), the LL each reached, MU's LL after about PDNR's and after about PQNR's wall time,
the kernel times of one PDNR and one PQNR outer iteration by kind from torch.profiler (separate
runs) with their lockstep counts, the time between kernels there (launches and read-backs), and
the card's name and power limit read in the same run.  Writes nothing.
"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import splatt_b200 as S  # noqa: E402

CONFIGS = {2: (10_000, 10_000_000), 4: (100_000, 100_000_000)}
KINDS = ["k_pdnr_grad", "k_pdnr_ladder", "k_pdnr_solve", "k_pdnr_accept", "k_apr_phi", "k_pqnr_step",
         "k_apr_combine", "k_apr_ll"]


def card():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                           str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()


def planted(dim, nnz, R, seed):
    """(inds [3 x nnz'] int32 CUDA, counts float64 CUDA) drawn from a planted rank-R model."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    lam = torch.rand(R, generator=g, device="cuda", dtype=torch.float64) + 0.5
    comp = torch.multinomial(lam / lam.sum(), nnz, replacement=True, generator=g)
    per = torch.bincount(comp, minlength=R)
    order = torch.argsort(comp)
    inds = torch.empty((3, nnz), dtype=torch.int64, device="cuda")
    for m in range(3):
        A = torch.rand((dim, R), generator=g, device="cuda", dtype=torch.float64) ** 8
        col = torch.cat([torch.multinomial(A[:, r], int(per[r]), replacement=True, generator=g)
                         for r in range(R)])
        inds[m, order] = col
    key = (inds[0] * dim + inds[1]) * dim + inds[2]
    key, counts = torch.unique(key, return_counts=True)
    out = torch.stack([key // (dim * dim), (key // dim) % dim, key % dim]).to(torch.int32)
    return out, counts.to(torch.float64)


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, r


def profile(fn):
    from torch.profiler import ProfilerActivity, profile as prof
    with prof(activities=[ProfilerActivity.CUDA]) as p:
        fn()
        torch.cuda.synchronize()
    evs = sorted((e for e in p.events() if e.device_type.name == "CUDA"), key=lambda e: e.time_range.start)
    kern = {k: sum(e.time_range.elapsed_us() for e in evs if k in e.name) / 1e3 for k in KINDS}
    kern["other"] = sum(e.time_range.elapsed_us() for e in evs
                        if not any(k in e.name for k in KINDS)) / 1e3
    gaps = sum(max(0, b.time_range.start - a.time_range.end) for a, b in zip(evs, evs[1:])) / 1e3
    return kern, gaps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", default="2:16,2:32,2:64,4:32")
    ap.add_argument("--cap", type=int, default=60)
    ap.add_argument("--tol", type=float, default=1e-4)
    args = ap.parse_args()
    print(card(), flush=True)
    for spec in args.runs.split(","):
        cfg, R = (int(x) for x in spec.split(":"))
        dim, nnz = CONFIGS[cfg]
        inds, vals = planted(dim, nnz, R, seed=cfg * 1000 + R)
        T = S.Tensor.from_coo([dim] * 3, [inds[m] for m in range(3)], vals)
        g = torch.Generator(device="cuda").manual_seed(7)
        f0 = [torch.rand((dim, R), generator=g, device="cuda", dtype=torch.float64) + 0.1 for _ in range(3)]
        row = {"config": cfg, "R": R, "nnz": int(vals.numel()), "card": card()}
        T.cp_apr_pdnr(R, f0, niters=1, max_inner=1)             # warm-up of every launch shape
        T.cp_apr_pqnr(R, f0, niters=1, max_inner=1)
        T.cp_apr(R, f0, niters=1, max_inner=1)
        solvers = (("pdnr", lambda: T.cp_apr_pdnr(R, f0, niters=args.cap, tol=args.tol)),
                   ("pqnr", lambda: T.cp_apr_pqnr(R, f0, niters=args.cap, tol=args.tol)),
                   ("mu", lambda: T.cp_apr(R, f0, niters=args.cap, tol=args.tol)))
        res = {}
        for rep in range(2):                                     # alternated
            for name, fn in solvers:
                sec, (lam, _, hist, its) = timed(fn)
                res.setdefault(name, []).append(sec)
                row[name] = {"iters": its, "final_kkt": float(hist[-1, 1]), "ll": float(hist[-1, 0]),
                             "converged": bool(hist[-1, 1] < args.tol and its < args.cap)}
                if name != "mu":
                    row[name]["lockstep"] = int(hist[:, 2].sum())
        for name, _ in solvers:
            row[name]["sec"] = min(res[name])
        # MU's LL after about PDNR's and PQNR's wall time
        per_mu = row["mu"]["sec"] / row["mu"]["iters"]
        for name in ("pdnr", "pqnr"):
            k = max(1, round(row[name]["sec"] / per_mu))
            _, (_, _, hist, _) = timed(lambda: T.cp_apr(R, f0, niters=k, tol=0.0))
            row[f"mu_at_{name}_time"] = {"iters": k, "ll": float(hist[-1, 0])}
        for name, fn in (("pdnr", T.cp_apr_pdnr), ("pqnr", T.cp_apr_pqnr)):
            out = {}
            kern, gaps = profile(lambda: out.setdefault("r", fn(R, f0, niters=1, tol=0.0)))
            row[f"{name}_outer_iteration_ms"] = {k: round(v, 3) for k, v in kern.items()}
            row[f"{name}_outer_iteration_lockstep"] = int(out["r"][2][0, 2])
            row[f"{name}_gaps_ms"] = round(gaps, 3)
        print(json.dumps(row), flush=True)
        T.free()
        del inds, vals, f0
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
