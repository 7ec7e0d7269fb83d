"""fp32 vs fp64 MTTKRP on configs 2, 3 and 4 (one GPU), every mode, three variants timed
alternately launch by launch in one process:

  f64_default: Tensor.from_coo(...)            fp64, default policy (CTA-tiled kernel where it applies)
  f64_generic: Tensor.from_coo(..., ktile=-1)  fp64, generic stream kernel
  f32:         the default-built tensor, float32 factors and output (splatt_b200_mttkrp_f32)

Every launch is timed with CUDA events after a 256 MB write that flushes L2; warm-up, then
--launches timed launches per variant; min / median reported.  Row bytes moved L2 -> SM are
counted from the streams' shapes (rows of pitch rpad * element size):
  generic kernels: one row per node of levels 1..N-1 (leaf rows per nonzero, parent rows per
                   fiber, ...) + records (16 B, +4 B ancestor id for N >= 4)
  CTA-tiled fp64:  parent rows per fiber + one pass of the leaf factor per SM + records + root ids
The gather probe (random whole-row gathers, 3 CTAs x 8 warps per SM, 8 rows in flight) is run
at the fp64 row (ncolumns = R) and at the byte-equivalent of the fp32 row (fp64 ncolumns = R/2).
Error: fp32 output against a torch fp64 oracle on the upcast fp32 factors, as the largest ratio
to the DESIGN.md section 5 bound (fp32 form) and as relative Frobenius; also relative Frobenius
against the fp64 default path on the unrounded factors.
Prints one JSON document.  usage: python scripts/f32_compare.py [--launches 20] [--configs 2,3,4]"""
import argparse
import ctypes as C
import json
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

# config: (dims, nnz, rank, seed) -- the generator and seeds of bench.py / config_bench.py
CONFIGS = {"2": ([10_000] * 3, 10_000_000, 32, 1),
           "3": ([5_000] * 4, 50_000_000, 16, 2),
           "4": ([100_000] * 3, 100_000_000, 32, 3)}
U32 = 2.0 ** -24
TINY = 2.0 ** -126


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True,
                           timeout=30)
        return dict(zip(q.split(","), [x.strip() for x in r.stdout.strip().split(",")]))
    except Exception as e:  # pragma: no cover
        return {"error": str(e)}


def probe_gbs(dev, dim, ncolumns, n):
    """Gather-probe rate (GB/s) for fp64 rows of `ncolumns` columns from a dim-row matrix."""
    lib = A.load()
    g = torch.Generator(device=dev).manual_seed(7)
    idx = torch.randint(0, dim, (n,), device=dev, dtype=torch.int32, generator=g)
    mat = torch.rand(dim, ncolumns, device=dev, dtype=torch.float64, generator=g)
    sink = torch.zeros(8, device=dev, dtype=torch.float64)
    s = torch.cuda.current_stream().cuda_stream
    ip = C.cast(C.c_void_p(idx.data_ptr()), C.POINTER(C.c_uint32))
    mp = C.cast(C.c_void_p(mat.data_ptr()), A.val_p)
    sp = C.cast(C.c_void_p(sink.data_ptr()), A.val_p)

    def run():
        if ncolumns in (16, 32, 64):
            rc = lib.splatt_b200_gather_probe_ex(mp, ncolumns, ncolumns, ip, n, sp, 3, 8, 0, 0,
                                                 C.c_void_p(s))
        else:   # L = 4 rows: the plain probe (3 CTAs per SM, 8 rows in flight too)
            rc = lib.splatt_b200_gather_probe(mp, ncolumns, ncolumns, ip, n, sp, C.c_void_p(s))
        assert rc == A.SPLATT_SUCCESS
    for _ in range(3):
        run()
    ts = []
    for _ in range(10):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        run()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ms = float(np.median(ts))
    return n * ncolumns * 8 / (ms * 1e-3) / 1e9


def oracle(dims, ind, vals, mats64, mode, R, chunk=10_000_000):
    """ref, absref (fp64) and nonzeros per row, in chunks of nonzeros."""
    ref = torch.zeros((dims[mode], R), dtype=torch.float64, device=vals.device)
    absref = torch.zeros_like(ref)
    for c0 in range(0, len(vals), chunk):
        sl = slice(c0, c0 + chunk)
        prod = vals[sl, None].expand(-1, R).clone()
        aprod = prod.abs()
        for m in range(len(dims)):
            if m != mode:
                rows = mats64[m].index_select(0, ind[m][sl].long())[:, :R]
                prod *= rows
                aprod *= rows.abs()
        im = ind[mode][sl].long()
        ref.index_add_(0, im, prod)
        absref.index_add_(0, im, aprod)
        del prod, aprod
    n = torch.bincount(ind[mode].long(), minlength=dims[mode])
    return ref, absref, n


def rel_fro(a, b):
    den = float(torch.linalg.norm(b))
    return float(torch.linalg.norm(a - b)) / (den if den > 0 else 1.0)


def row_bytes(T, kind, m, R, nnz, sms, dims, cta_tiled):
    """cta_tiled: T was built CTA-tiled (its fp64 calls run the shared-memory tile kernel)."""
    info = T.mode_info(m, R)
    nf = info["nfibs"]
    pitch = ((R + 3) & ~3) * 4 if kind == "f32" else (R + (R & 1)) * 8
    N = len(nf)
    if kind == "f64_default" and cta_tiled:
        rows = nf[-2] * pitch + sms * dims[info["level_perm"][-1]] * pitch
        rec = nnz * (16 + 4)
    else:
        rows = sum(nf[1:]) * pitch
        rec = nnz * (16 + (4 if N >= 4 else 0))
    return int(rows), int(rec), nf


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--configs", default="2,3,4")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    res = {"card": card(), "sms": sms, "launches_per_variant": args.launches,
           "l2": "flushed before every launch (256 MB write)", "configs": []}
    sampler = bench.ClockSampler(0).start()
    for cfg in args.configs.split(","):
        dims, nnz, R, seed = CONFIGS[cfg]
        N = len(dims)
        ind, vals = bench.make_coo_gpu(nnz, dev, dims=dims, seed=seed)
        Td = S.Tensor.from_coo(dims, ind, vals)
        Tg = S.Tensor.from_coo(dims, ind, vals, ktile=-1)
        # the default build is CTA-tiled iff its stream differs from the generic one
        tiled = any(Td.mode_info(m, R)["nfibs"] != Tg.mode_info(m, R)["nfibs"] for m in range(N))
        m64 = [torch.from_numpy(x).to(dev) for x in bench.make_factors_host(seed, dims, R)]
        m32 = [x.float() for x in m64]
        var = {"f64_default": (Td, m64, torch.float64), "f64_generic": (Tg, m64, torch.float64),
               "f32": (Td, m32, torch.float32)}
        outs = {k: [torch.empty((d, R), dtype=v[2], device=dev) for d in dims] for k, v in var.items()}
        times = {k: [[] for _ in dims] for k in var}
        for m in range(N):
            for k, (T, mats, _) in var.items():
                for _ in range(3):
                    T.mttkrp(m, mats, outs[k][m])
            for _ in range(args.launches):
                for k, (T, mats, _) in var.items():
                    flush.zero_()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    T.mttkrp(m, mats, outs[k][m])
                    e1.record()
                    times[k][m].append((e0, e1))
            torch.cuda.synchronize()
        row = {"config": cfg, "dims": dims, "nnz": nnz, "rank": R, "seed": seed,
               "default_build_cta_tiled": bool(tiled),
               "probe_GBps_f64_row": probe_gbs(dev, dims[0], R, 2 * nnz) if R in (16, 32, 64) else None,
               "probe_GBps_f32_row_equiv": probe_gbs(dev, dims[0], R // 2, 2 * nnz),
               "modes": []}
        for m in range(N):
            mr = {"mode": m}
            for k, (T, _, _) in var.items():
                ms = [a.elapsed_time(b) for a, b in times[k][m]]
                med = float(np.median(ms))
                rows, rec, nf = row_bytes(T, k, m, R, nnz, sms, dims, tiled)
                mr[k] = {"ms_min": float(min(ms)), "ms_median": med, "nfibs": nf,
                         "row_bytes": rows, "record_bytes": rec,
                         "l2_to_sm_GBps": (rows + rec) / (med * 1e-3) / 1e9}
            mr["f32_over_f64_default"] = mr["f32"]["ms_median"] / mr["f64_default"]["ms_median"]
            mr["f32_over_f64_generic"] = mr["f32"]["ms_median"] / mr["f64_generic"]["ms_median"]
            ref, absref, n = oracle(dims, ind, vals, [x.double() for x in m32], m, R)
            got = outs["f32"][m].double()
            nf_ = n.to(torch.float64)[:, None]
            k_ = nf_ + N + 1
            bound = 2.0 * (k_ * U32 / (1.0 - k_ * U32)) * absref + nf_ * TINY
            err = (got - ref).abs()
            ratio = torch.where(bound > 0, err / bound, torch.where(err > 0, torch.inf, 0.0))
            mr["f32_max_ratio_to_bound"] = float(ratio.max())
            mr["f32_rel_fro_vs_f64_oracle_same_factors"] = rel_fro(got, ref)
            mr["f32_rel_fro_vs_f64_default"] = rel_fro(got, outs["f64_default"][m])
            del ref, absref, got, err, bound, ratio
            row["modes"].append(mr)
            print(f"config {cfg} mode {m}: f64 default {mr['f64_default']['ms_median']:.3f} ms, "
                  f"f64 generic {mr['f64_generic']['ms_median']:.3f} ms, f32 {mr['f32']['ms_median']:.3f} ms "
                  f"({mr['f32']['l2_to_sm_GBps']:.0f} GB/s), bound ratio {mr['f32_max_ratio_to_bound']:.3f}",
                  file=sys.stderr)
        res["configs"].append(row)
        Td.free()
        Tg.free()
        del ind, vals, outs, m64, m32
        torch.cuda.empty_cache()
    res["clocks"] = sampler.stop()
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
