"""CPU: the C-ABI library loads, exports every symbol include/splatt_b200.h declares,
and its boundary structs are layout-identical to the reference's."""
import ctypes as C
import re
from pathlib import Path

import numpy as np
import pytest

from splatt_b200 import _abi as A
from tests import recorded

ROOT = Path(__file__).resolve().parent.parent


def test_library_loads_and_exports_every_declared_symbol(lib):
    header = (ROOT / "include" / "splatt_b200.h").read_text()
    # every function declared in the header: "name(" at the start of a declaration line
    declared = set(re.findall(r"^\s*(?:[A-Za-z_][\w\s\*]*?)\b(splatt_\w+)\s*\(", header, re.M))
    declared = {d for d in declared if not d.endswith("_t")}
    assert {"splatt_mttkrp", "splatt_mttkrp_alloc_ws", "splatt_mttkrp_free_ws",
            "splatt_mttkrp_csf", "splatt_cpd_als", "splatt_b200_mttkrp"} <= declared
    for name in declared | set(A.EXPORTS):
        assert hasattr(lib, name), f"{name} declared in include/splatt_b200.h but not exported"


def test_version_and_default_opts(lib):
    assert b"splatt_b200" in lib.splatt_b200_version()
    import splatt_b200 as S
    o = S.default_opts()
    # reference defaults: src/opts.c:10-47
    assert o[A.OPTION_TOLERANCE] == 1e-5 and o[A.OPTION_NITER] == 50
    assert o[A.OPTION_CSF_ALLOC] == A.CSF_TWOMODE and o[A.OPTION_TILE] == A.NOTILE
    assert o[A.OPTION_PRIVTHRESH] == 0.02 and o[A.OPTION_TILELEVEL] == 1
    assert o[A.OPTION_VERBOSITY] == A.VERBOSITY_LOW and o[A.OPTION_NTHREADS] >= 1


def test_struct_layouts_match_reference_headers():
    """Offsets computed by the C compiler from the reference's own headers
    (oracle/ref_driver.c:refdrv_abi, recorded in tests/golden/reference.npz) vs the ctypes
    mirror of include/splatt_b200.h."""
    f = iter(recorded.load()["abi_facts"].tolist())

    def nxt():
        return next(f)

    assert nxt() == C.sizeof(A.idx_t) and nxt() == C.sizeof(A.val_t) and nxt() == A.MAX_NMODES
    assert nxt() == C.sizeof(A.CsfSparsity)
    for fld in ("nfibs", "fptr", "fids", "vals"):
        assert nxt() == getattr(A.CsfSparsity, fld).offset, fld
    assert nxt() == C.sizeof(A.SplattCsf)
    for fld in ("nnz", "nmodes", "dims", "dim_perm", "dim_iperm", "which_tile", "ntiles",
                "ntiled_modes", "tile_dims", "pt"):
        assert nxt() == getattr(A.SplattCsf, fld).offset, fld
    assert nxt() == C.sizeof(A.SplattKruskal)
    for fld in ("rank", "factors", "lambda_", "nmodes", "dims", "fit"):
        assert nxt() == getattr(A.SplattKruskal, fld).offset, fld
    assert nxt() == C.sizeof(A.MttkrpWs)
    for fld in ("num_csf", "mode_csf_map", "num_threads", "tile_partition", "tree_partition",
                "is_privatized", "privatize_buffer", "reduction_time"):
        assert nxt() == getattr(A.MttkrpWs, fld).offset, fld
    assert nxt() == C.sizeof(A.Matrix)
    for fld in ("I", "J", "vals", "rowmajor"):
        assert nxt() == getattr(A.Matrix, fld).offset, fld
    assert [nxt(), nxt(), nxt()] == [A.SPLATT_SUCCESS, A.SPLATT_ERROR_BADINPUT,
                                     A.SPLATT_ERROR_NOMEMORY]
    assert [nxt() for _ in range(13)] == list(range(13))     # option enum order


def test_header_struct_layout_compiles_to_the_same_offsets(tmp_path):
    """Compile include/splatt_b200.h with gcc and compare sizeof/offsetof to the reference."""
    import subprocess
    src = tmp_path / "abi.c"
    src.write_text('''
#include <stdio.h>
#include <stddef.h>
#include "splatt_b200.h"
int main(void){
 printf("%zu %zu %zu %zu %zu\\n", sizeof(csf_sparsity), sizeof(splatt_csf), sizeof(splatt_kruskal),
        sizeof(splatt_mttkrp_ws), sizeof(splatt_b200_matrix_t));
 printf("%zu %zu %zu %zu\\n", offsetof(splatt_csf, which_tile), offsetof(splatt_csf, ntiles),
        offsetof(splatt_csf, pt), offsetof(splatt_mttkrp_ws, privatize_buffer));
 return 0; }''')
    exe = tmp_path / "abi"
    subprocess.run(["gcc", "-std=c99", f"-I{ROOT / 'include'}", str(src), "-o", str(exe)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True,
                                          check=True).stdout.split()]
    facts = recorded.load()["abi_facts"].tolist()
    assert got[:5] == [facts[3], facts[8], facts[19], facts[26], facts[35]]
    assert got[5:] == [A.SplattCsf.which_tile.offset, A.SplattCsf.ntiles.offset,
                       A.SplattCsf.pt.offset, A.MttkrpWs.privatize_buffer.offset]
