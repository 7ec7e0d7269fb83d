"""CPU: pin the oracle.

(1) oracle/restate.c against the committed golden vectors, which were produced by
    the reference's own gold (mttkrp_stream) on the reference's own fixtures
    (tests/golden/make_golden.py).  Tolerance = the reference's own test
    tolerance, abs 1e-10 (tests/mttkrp_test.c:25-30), plus 1e-12 relative.
(2) oracle/restate.c against output recorded from the compiled reference
    (tests/recorded.py) on seeded random tensors: CSF arrays bit-exact, MTTKRP (COO and
    CSF walk) 1e-12, CPD-ALS on every problem the GPU tests solve.
"""
from pathlib import Path

import numpy as np
import pytest

from oracle import restate
from tests import recorded
from tests.util import factor_mats, random_coo, rel_fro

GOLD = Path(__file__).parent / "golden"
NAMES = ["small", "med", "small4", "med4", "med5", "small4_zeroidx"]


def load_golden(name):
    z = np.load(GOLD / f"{name}.npz")
    dims = [int(d) for d in z["dims"]]
    inds = [z["ind"][m].astype(np.uint64) for m in range(len(dims))]
    return z, dims, inds, z["vals"]


def check_against_golden(z, R, m, out):
    rows = z[f"gold_R{R}_m{m}_rows"]
    assert np.allclose(out[rows], z[f"gold_R{R}_m{m}_vals"], rtol=1e-12, atol=1e-10)
    assert np.allclose(out.sum(axis=0), z[f"gold_R{R}_m{m}_colsum"], rtol=1e-11, atol=1e-9)
    assert abs(np.linalg.norm(out) - z[f"gold_R{R}_m{m}_fro"][0]) <= 1e-11 * z[f"gold_R{R}_m{m}_fro"][0]


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("R", [3, 16])
def test_restatement_coo_vs_golden(name, R):
    z, dims, inds, vals = load_golden(name)
    mats = factor_mats(dims, R, seed=R)
    for m in range(len(dims)):
        check_against_golden(z, R, m, restate.mttkrp_coo(dims, inds, vals, mats, m))


@pytest.mark.parametrize("name", NAMES)
def test_restatement_csf_vs_golden(name):
    """CSF build + tree-walk MTTKRP (root / internal / leaf) on the default TWOMODE CSFs."""
    z, dims, inds, vals = load_golden(name)
    R = 3
    mats = factor_mats(dims, R, seed=R)
    perms, mode_map = restate.csf_policy(dims, 1)
    csfs = [restate.OracleCsf(dims, inds, vals, p) for p in perms]
    for c, csf in enumerate(csfs):
        a = csf.arrays()
        assert a["dim_perm"] == [int(x) for x in z[f"csf{c}_perm"]]
        assert a["nfibs"] == [int(x) for x in z[f"csf{c}_nfibs"]]
        assert a["nfibs"][-1] == len(vals)
    for m in range(len(dims)):
        # every mode on every CSF: exercises all output depths
        for csf in csfs:
            check_against_golden(z, R, m, csf.mttkrp(mats, m))


def test_zero_index_fixture_equals_one_index_fixture():
    """tests/io_test.c:35-53: 0- and 1-indexed files describe the same tensor."""
    _, d0, i0, v0 = load_golden("small4")
    _, d1, i1, v1 = load_golden("small4_zeroidx")
    assert d0 == d1 and np.array_equal(v0, v1)
    for a, b in zip(i0, i1):
        assert np.array_equal(a, b)


SPECS = recorded.ORACLE_SPECS


@pytest.mark.parametrize("spec", SPECS)
@pytest.mark.parametrize("alloc", [0, 1, 2])
def test_restatement_vs_compiled_reference(spec, alloc):
    k = SPECS.index(spec)
    dims, inds, vals = random_coo(spec[0], spec[1], seed=11)
    mats = factor_mats(dims, 5)
    z = recorded.load()
    gold = [z[f"spec{k}_m{m}"] for m in range(len(dims))]
    perms, mode_map = restate.csf_policy(dims, alloc)
    want = recorded.csf_digests(f"spec{k}", alloc)
    assert len(want) == len(perms)
    for c, perm in enumerate(perms):
        oc = restate.OracleCsf(dims, inds, vals, perm)
        got = recorded.csf_digest(oc.arrays())
        assert got == {key: want[c][key] for key in got}, c
        for m in range(len(dims)):
            assert rel_fro(oc.mttkrp(mats, m), gold[m]) < 1e-12
    for m in range(len(dims)):
        assert rel_fro(restate.mttkrp_coo(dims, inds, vals, mats, m), gold[m]) < 1e-13


def test_restatement_cpd_vs_compiled_reference():
    dims, inds, vals = recorded.cpd_tensor("s3")
    recorded.check_cpd("s3", *restate.cpd_als(dims, inds, vals, 6, 8, 0.0, 7))


@pytest.mark.parametrize("key", list(recorded.CPD_CASES))
def test_restatement_cpd_matches_recorded_reference(key):
    """Every CPD-ALS problem the GPU tests check against the restatement: the restatement
    reproduces the reference's fit, lambda and factors on it."""
    _, _, R, _, its, seed = recorded.CPD_CASES[key]
    dims, inds, vals = recorded.cpd_tensor(key)
    recorded.check_cpd(key, *restate.cpd_als(dims, inds, vals, R, its, 0.0, seed))


def test_compiled_reference_matches_golden(refmod):
    """The compiled reference reproduces the committed vectors (guards the build flags of
    oracle/build_ref.sh; runs where oracle/_ref is built)."""
    z, dims, inds, vals = load_golden("med")
    tt = refmod.RefTensor.from_coo(dims, inds, vals)
    mats = factor_mats(dims, 3, seed=3)
    for m in range(3):
        check_against_golden(z, 3, m, tt.mttkrp_stream(mats, m))
