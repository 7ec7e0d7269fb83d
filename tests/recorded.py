"""What the suite compares against, recorded from the compiled reference.

tests/golden/reference.npz is written by tests/golden/make_golden.py where the reference
is built; the tests read it, so they need neither the reference sources nor a build of
them.  Keys:
  abi_facts                    sizes / offsets / enum values from the reference headers
                               (oracle/ref_driver.c:refdrv_abi)
  order<k>_small|minusone|last csf_find_mode_order for ORDER_DIMS[k]
  csf_digests                  JSON: "<case>/<alloc>" -> per-CSF structure digest of the
                               reference's csf_alloc (csf_digest below)
  spec<k>_m<m>                 mttkrp_stream of ORACLE_SPECS[k] (factor_mats(dims, 5))
  cpd_<key>_fit|lambda|colsum<m>|factor<m>
                               the reference's cpd_als on CPD_CASES[key] (factors only when
                               small; their column sums always)
"""
from __future__ import annotations

import hashlib
import json
from functools import lru_cache
from pathlib import Path

import numpy as np

from tests.util import cover_all_slices, parity_tensor, random_coo

PATH = Path(__file__).parent / "golden" / "reference.npz"

ORDER_DIMS = [[30, 10, 20], [10, 10, 10], [30, 10, 20, 10], [5, 4, 3, 2, 1], [7, 7, 3, 7, 3, 9],
              [2425, 10816, 29567], [60114, 83826, 23034, 1132, 100], [4, 3, 5, 4, 3, 6, 2, 5]]

ORACLE_SPECS = [((30, 50), 700), ((13, 7, 11), 150), ((40, 30, 50, 20), 5000),
                ((12, 15, 10, 20, 9), 3000), ((5, 6, 4, 7, 3, 5), 1500)]

CSF_TENSORS = ["t2_matrix", "t3_small", "t3_mid", "t4", "t5", "t8"]

# key -> (dims, nnz, rank, tensor seed, iterations, cpd seed); tensors are
# cover_all_slices(random_coo(dims, nnz, seed=tensor seed))
CPD_CASES = {
    "s3": ((60, 50, 40), 6000, 6, 3, 8, 7),
    "s4": ((30, 25, 20, 15), 5000, 5, 3, 8, 7),
    "m3": ((200, 150, 100), 30000, 16, 3, 8, 7),
    "deficient": ((3, 40, 30), 600, 5, 9, 3, 2),
    "tail20": ((260, 150, 100), 40000, 20, 17, 5, 9),
    "tail32": ((260, 150, 100), 40000, 32, 17, 5, 9),
    "tail48": ((260, 150, 100), 40000, 48, 17, 5, 9),
    "tail64": ((260, 150, 100), 40000, 64, 17, 5, 9),
    "r128": ((300, 250, 200), 60000, 128, 13, 3, 5),
    "s3_six": ((60, 50, 40), 6000, 6, 3, 6, 11),
}


def cpd_tensor(key):
    dims, nnz, _, tseed, _, _ = CPD_CASES[key]
    return cover_all_slices(*random_coo(dims, nnz, seed=tseed))


def csf_cases():
    """(case key, (dims, inds, vals)) of every tensor whose reference CSFs are recorded."""
    for name in CSF_TENSORS:
        yield name, parity_tensor(name)
    yield "gaps", random_coo((500, 40, 30), 300, seed=5)
    for k, (shape, nnz) in enumerate(ORACLE_SPECS):
        yield f"spec{k}", random_coo(shape, nnz, seed=11)


def _sha(a, dtype):
    return hashlib.sha256(np.ascontiguousarray(a, dtype).tobytes()).hexdigest()[:16]


def csf_digest(arrays):
    """Structure of one CSF (a Csf.arrays() dict): sizes, orders and a (64-bit prefix of a)
    sha256 per array."""
    h = {k: [int(x) for x in arrays[k]] for k in ("dim_perm", "dim_iperm", "nfibs", "dims")
         if k in arrays}
    if "nnz" in arrays:
        h["nnz"] = int(arrays["nnz"])
    h["fids"] = [None if f is None else _sha(f, np.uint64) for f in arrays["fids"]]
    h["fptr"] = [_sha(f, np.uint64) for f in arrays["fptr"]]
    h["vals"] = _sha(arrays["vals"], np.float64)
    return h


@lru_cache(maxsize=1)
def load():
    z = np.load(PATH)
    return {k: z[k] for k in z.files}


def csf_digests(case, alloc):
    return json.loads(load()["csf_digests"].item().decode())[f"{case}/{alloc}"]


def check_cpd(key, fit, lam, fac):
    """A CPD-ALS result (post-processed like the reference's cpd_als) against the record."""
    z = load()
    assert abs(fit - z[f"cpd_{key}_fit"][0]) < 1e-12, (key, fit, z[f"cpd_{key}_fit"][0])
    assert np.allclose(lam, z[f"cpd_{key}_lambda"], rtol=1e-10, atol=1e-12), key
    for m, a in enumerate(fac):
        assert np.allclose(a.sum(axis=0), z[f"cpd_{key}_colsum{m}"], rtol=1e-9, atol=1e-10), (key, m)
        if f"cpd_{key}_factor{m}" in z:
            assert np.allclose(a, z[f"cpd_{key}_factor{m}"], rtol=1e-9, atol=1e-12), (key, m)
