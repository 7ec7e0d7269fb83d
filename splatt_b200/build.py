"""In-tree build of libsplatt_b200.so (nvcc, sm_90a only).

`python -m splatt_b200.build` or `splatt_b200.build.build()`.  Objects are
compiled in parallel (one nvcc per translation unit; the kernel templates are
instantiated once per mode count) and linked into splatt_b200/libsplatt_b200.so,
next to the package sources.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

HERE = Path(__file__).resolve().parent
CSRC = HERE / "csrc"
OUT = HERE / "libsplatt_b200.so"
OBJ = HERE / "_obj"

NVCC = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC,-fopenmp,-O3",
          "-Xcudafe", "--diag_suppress=177"]


def _units():
    units = []
    for n in range(2, 9):
        units.append((f"mttkrp_inst_n{n}", CSRC / "mttkrp_inst.cu", [f"-DSPB200_INST_N={n}"]))
        units.append((f"mttkrp_inst_f32_n{n}", CSRC / "mttkrp_inst.cu",
                      [f"-DSPB200_INST_N={n}", "-DSPB200_INST_F32"]))
    for name in ("mttkrp_launch", "mttkrp_tiled", "stream_build", "engine", "dropin", "cpd", "multi", "tc"):
        units.append((name, CSRC / f"{name}.cu", []))
    return units


def _deps_hash(extra: list[str]) -> str:
    h = hashlib.sha256()
    for p in sorted(CSRC.glob("*")) + [HERE.parent / "include" / "splatt_b200.h"]:
        h.update(p.name.encode())
        h.update(p.read_bytes())
    h.update(" ".join(ARCH + COMMON + extra).encode())
    return h.hexdigest()


def _compile(unit):
    name, src, extra = unit
    obj = OBJ / f"{name}.o"
    stamp = OBJ / f"{name}.hash"
    want = _deps_hash(extra)
    if obj.exists() and stamp.exists() and stamp.read_text() == want:
        return obj, ""
    cmd = [NVCC, *ARCH, *COMMON, *extra, "-c", str(src), "-o", str(obj)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src.name}:\n{' '.join(cmd)}\n{r.stdout}\n{r.stderr}")
    stamp.write_text(want)
    return obj, r.stderr


def build(verbose: bool = False) -> Path:
    OBJ.mkdir(exist_ok=True)
    units = _units()
    with ThreadPoolExecutor(max_workers=min(len(units), os.cpu_count() or 4)) as ex:
        results = list(ex.map(_compile, units))
    objs = [str(o) for o, _ in results]
    if verbose:
        for _, log in results:
            if log.strip():
                print(log, file=sys.stderr)
    newest = max(Path(o).stat().st_mtime for o in objs)
    if OUT.exists() and OUT.stat().st_mtime >= newest:
        return OUT
    tmp = OUT.with_suffix(".so.tmp")      # link beside, then rename: never a half-written library
    cmd = [NVCC, *ARCH, "-shared", "-o", str(tmp), *objs,
           "-Xcompiler", "-fopenmp", "-Xlinker", "-Bsymbolic", "-lgomp"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{' '.join(cmd)}\n{r.stdout}\n{r.stderr}")
    os.replace(tmp, OUT)
    return OUT


if __name__ == "__main__":
    print(build(verbose="-v" in sys.argv))
