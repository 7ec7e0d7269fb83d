"""Sweep the gather probe (splatt_b200_gather_probe_ex): random whole-row fp64 gathers from an
L2-resident factor matrix at {1..8} CTAs/SM x {2,4,8,16} rows in flight x {default,
L1::no_allocate}, an L1 squeeze at the generic root kernel's shape, and the leaf-tiled root
kernel's shapes (32, 24 and 16 warps/SM, no-allocate, rows in flight x shared memory reserved).
The best point is the measured ceiling of the MTTKRP's access pattern.
  python scripts/probe_sweep.py [rows] [rank] [ngathers]
Prints one JSON line."""
import ctypes as C
import json
import sys

import numpy as np
import torch

sys.path.insert(0, ".")
from splatt_b200 import _abi as A  # noqa: E402

rows = int(sys.argv[1]) if len(sys.argv) > 1 else 10_000
R = int(sys.argv[2]) if len(sys.argv) > 2 else 32
n = int(sys.argv[3]) if len(sys.argv) > 3 else 20_000_000
lib = A.load()
dev = torch.device("cuda", 0)
g = torch.Generator(device=dev).manual_seed(7)
idx = torch.randint(0, rows, (n,), device=dev, dtype=torch.int32, generator=g)
mat = torch.rand(rows, R, device=dev, dtype=torch.float64, generator=g)
sink = torch.zeros(8, device=dev, dtype=torch.float64)
s = torch.cuda.current_stream().cuda_stream
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
out = []


def timed(ctas, rif, na, smem):
    def run():
        rc = lib.splatt_b200_gather_probe_ex(
            C.cast(C.c_void_p(mat.data_ptr()), A.val_p), R, R,
            C.cast(C.c_void_p(idx.data_ptr()), C.POINTER(C.c_uint32)), n,
            C.cast(C.c_void_p(sink.data_ptr()), A.val_p), ctas, rif, na, smem, C.c_void_p(s))
        assert rc == A.SPLATT_SUCCESS, rc
    for _ in range(2):
        run()
    ts = []
    for _ in range(7):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); run(); e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ms = float(np.median(ts))
    return {"no_allocate": na, "ctas_per_sm": ctas, "rows_in_flight": rif, "smem_per_cta": smem,
            "warps_per_sm": ctas * 8, "ms": ms, "TBps": n * R * 8 / (ms * 1e-3) / 1e12}


# 1. occupancy x rows in flight x L1 policy, full L1 (no shared-memory reservation)
for na in (0, 1):
    for ctas in (1, 2, 3, 4, 6, 8):
        for rif in (2, 4, 8, 16):
            out.append(timed(ctas, rif, na, 0))
# 2. the MTTKRP kernel's shape (3 CTAs x 8 rows) with less and less L1 left
l1 = [timed(3, 8, 0, sm) for sm in (0, 8192, 16384, 32768, 49152, 65536, 73728)]
# 3. the leaf-tiled root kernel's shape: 32 warps/SM (4 x 8; the kernel runs one CTA of 32
#    warps), parent rows not allocated in L1, gathers in flight per lane group x shared memory
#    reserved per CTA (what is left of the 256 KB L1 holds the in-flight lines); the earlier
#    24 warps/SM (3 x 8); and 16 warps/SM (2 x 8), fewer warps with more registers each
KB = 1024
tiled32 = [timed(4, rif, 1, sm * KB) for rif in (2, 4, 8) for sm in (0, 32, 48, 55)]
tiled = [timed(3, rif, 1, sm * KB) for rif in (4, 8, 16) for sm in (0, 16, 32, 48, 64, 72)]
tiled16 = [timed(2, rif, 1, sm * KB) for rif in (4, 8, 16) for sm in (0, 64, 96, 108)]
best = max(out, key=lambda r: r["TBps"])
print(json.dumps({"matrix_rows": rows, "rank": R, "gathers": n, "row_bytes": R * 8,
                  "best": best, "l1_squeeze_3ctas_8rows": l1, "tiled_shape_32warps": tiled32,
                  "tiled_shape_24warps": tiled,
                  "tiled_shape_16warps": tiled16, "sweep": out}))
