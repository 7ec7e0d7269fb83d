"""One process per GPU (torchrun + NCCL, splatt_b200/parallel.py): the fused multicast exchange
with the group barrier in the kernel's tail against kernel + NCCL all-reduce, and the sharded
CPD-ALS with either exchange -- scripts/test_fused.py under torchrun, which asserts
  * fused == NCCL result to 1e-12 over 20 sweeps x 3 modes (the in-kernel barrier must order
    the remote reductions every time),
  * identical CPD fits with both exchanges.
Needs >= 2 GPUs; skipped on a machine with one."""
import re
import subprocess
import sys
from pathlib import Path

import pytest

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent


def test_fused_exchange_and_sharded_cpd_under_torchrun():
    import torch
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1",
                        "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port",
                        "29531", str(ROOT / "scripts" / "test_fused.py")],
                       capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    m = re.search(r"worst rel err ([0-9.e+-]+)", r.stdout)
    assert m and float(m.group(1)) < 1e-12, r.stdout[-1000:]
    f = re.search(r"fit fused ([0-9.]+) nccl ([0-9.]+)", r.stdout)
    assert f and abs(float(f.group(1)) - float(f.group(2))) < 1e-9
