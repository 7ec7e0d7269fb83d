"""Generate the committed golden vectors from the reference's own fixtures and code.

Run where the reference sources exist and oracle/_ref has been built from them
(oracle/build_ref.sh; SPLATT_REFERENCE names the source tree):
    SPLATT_REFERENCE=<reference tree> python tests/golden/make_golden.py

(1) For every tensor the reference's MTTKRP tests use (tests/splatt_test.h:11-27:
small, med, small4, med4, med5 + small4_zeroidx) one .npz with:
  dims, ind (uint32, nmodes x nnz, as read by the reference's tt_read, i.e.
  0-based), vals, and for R in RANKS and every mode the output of the
  reference's gold mttkrp_stream (tests/mttkrp_test.c:66) on seeded factors
  (numpy default_rng(1000+R), uniform [-3,3] -- tests/util.py:factor_mats), plus
  the node counts of the reference's default TWOMODE CSFs.
The med* fixtures are cut to a seeded sample of SUBSAMPLE nonzeros (dims kept)
so that every stored file stays small.  The parity tests recompute the factors
from the seed, so only tensors and expected outputs are stored.  An output of
more than SAMPLE rows is stored as: SAMPLE seeded rows (+ their row numbers),
the column sums and the Frobenius norm.

(2) reference.npz: what the other tests compare against, recorded from the
compiled reference so that the suite needs neither the reference sources nor a
build of them (see tests/recorded.py for the keys).
"""
import json
import os
import subprocess
import sys
import tempfile
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
from oracle import ref  # noqa: E402
from tests import recorded  # noqa: E402
from tests.util import factor_mats, random_coo  # noqa: E402

REF_TENSORS = Path(os.environ["SPLATT_REFERENCE"]) / "tests" / "tensors"
NAMES = ["small", "med", "small4", "med4", "med5", "small4_zeroidx"]
RANKS = [3, 16]
SAMPLE = 256
SUBSAMPLE = 3000
HERE = Path(__file__).parent


def fixtures():
    for name in NAMES:
        tt = ref.RefTensor.read(REF_TENSORS / f"{name}.tns")
        dims = list(tt.dims)
        inds, vals = tt.coo()
        if name.startswith("med"):
            keep = np.sort(np.random.default_rng(11).choice(len(vals), SUBSAMPLE, replace=False))
            inds, vals = [i[keep] for i in inds], vals[keep]
        tt = ref.RefTensor.from_coo(dims, inds, vals)
        out = {"dims": np.array(dims, dtype=np.uint64),
               "ind": np.stack(inds).astype(np.uint32), "vals": vals}
        for R in RANKS:
            mats = factor_mats(dims, R, seed=R)
            for m in range(len(dims)):
                g = tt.mttkrp_stream(mats, m, nthreads=1)
                if g.shape[0] <= SAMPLE:
                    rows = np.arange(g.shape[0])
                else:
                    rows = np.sort(np.random.default_rng(7 + m).choice(g.shape[0], SAMPLE, replace=False))
                out[f"gold_R{R}_m{m}_rows"] = rows.astype(np.uint32)
                out[f"gold_R{R}_m{m}_vals"] = g[rows]
                out[f"gold_R{R}_m{m}_colsum"] = g.sum(axis=0)
                out[f"gold_R{R}_m{m}_fro"] = np.array([np.linalg.norm(g)])
        o = ref.default_opts()
        o[0] = 1
        csf = ref.RefCsf(tt, o)     # sorts tt (after the COO copy above)
        for c in range(csf.count):
            a = csf.arrays(c)
            out[f"csf{c}_perm"] = np.array(a["dim_perm"], dtype=np.uint64)
            out[f"csf{c}_nfibs"] = np.array(a["nfibs"], dtype=np.uint64)
        if name == "med":
            out["cli_fit_r16_i5"] = np.array([cli_fit(out["ind"], vals)])
        path = HERE / f"{name}.npz"
        np.savez_compressed(path, **out)
        print(name, dims, len(vals), path.stat().st_size // 1024, "KiB")


def cli_fit(ind, vals):
    """Final fit of the reference CLI: `splatt cpd -r 16 -t 1 --seed 1 -i 5`."""
    from tests.test_config1_cli import _write_tns, cli_fits
    with tempfile.TemporaryDirectory() as d:
        tns = Path(d) / "med.tns"
        _write_tns(tns, ind, vals)
        r = subprocess.run([str(ref.CLI_PATH), "cpd", str(tns), "-r", "16", "-t", "1", "--seed", "1",
                            "--nowrite", "-i", "5"], capture_output=True, text=True, check=True)
    return cli_fits(r.stdout)[-1]


def records():
    out, csfs = {}, {}
    out["abi_facts"] = np.array(ref.abi_facts(), dtype=np.int64)
    for k, dims in enumerate(recorded.ORDER_DIMS):
        n = len(dims)
        out[f"order{k}_small"] = np.array(ref.mode_order(dims, ref.CSF_SORTED_SMALLFIRST))
        out[f"order{k}_minusone"] = np.array([ref.mode_order(dims, ref.CSF_SORTED_MINUSONE, m)
                                              for m in range(n)])
        out[f"order{k}_last"] = np.array([ref.mode_order(dims, w, n - 1) for w in range(4)])
    for key, (dims, inds, vals) in recorded.csf_cases():
        for alloc in (0, 1, 2):
            o = ref.default_opts()
            o[0], o[6] = 1, alloc
            tt = ref.RefTensor.from_coo(dims, inds, vals)
            rc = ref.RefCsf(tt, o)
            csfs[f"{key}/{alloc}"] = [recorded.csf_digest(rc.arrays(c)) for c in range(rc.count)]
            rc.free()
    for k, (shape, nnz) in enumerate(recorded.ORACLE_SPECS):
        dims, inds, vals = random_coo(shape, nnz, seed=11)
        mats = factor_mats(dims, 5)
        tt = ref.RefTensor.from_coo(dims, inds, vals)
        for m in range(len(dims)):
            out[f"spec{k}_m{m}"] = tt.mttkrp_stream(mats, m)
    for key, (_, _, R, _, its, seed) in recorded.CPD_CASES.items():
        dims, inds, vals = recorded.cpd_tensor(key)
        o = ref.default_opts()
        o[0], o[3], o[1], o[4] = 1, its, 0.0, 0
        rc = ref.RefCsf(ref.RefTensor.from_coo(dims, inds, vals), o)
        fit, lam, fac = rc.cpd_als(R, seed)
        out[f"cpd_{key}_fit"] = np.array([fit])
        out[f"cpd_{key}_lambda"] = lam
        for m, a in enumerate(fac):
            out[f"cpd_{key}_colsum{m}"] = a.sum(axis=0)
            if a.size <= 1000:
                out[f"cpd_{key}_factor{m}"] = a
    out["csf_digests"] = np.array(json.dumps(csfs, sort_keys=True).encode())
    path = HERE / "reference.npz"
    np.savez_compressed(path, **out)
    print("reference", path.stat().st_size // 1024, "KiB")


if __name__ == "__main__":
    fixtures()
    records()
