"""CPU: the aggregate_verify batch cases (tests/aggregate_verify_cases.py) fail or pass in the C oracle for the reason each
was built for, the closed-form scale batches verify, the C and Python oracles agree on a subset, and the plan of the device's
segmented product (modelled in Python) ends with every segment in at most two pieces after about log32 of its length
levels."""
from __future__ import annotations

import math

import pytest

from oracle import bls_oracle as bo
from tests import aggregate_verify_cases as av
from tests import torsion_cases as tc


@pytest.fixture(scope="module")
def O(oracle_bls_c):
    return av.bind(oracle_bls_c)


@pytest.fixture(scope="module")
def cases(O):
    return av.crafted(O, tc.g1_cases(), tc.g2_cases())


def test_crafted_cases_get_the_code_they_were_built_for(O, cases):
    codes = av.oracle_codes(O, cases)
    for c, k in zip(cases, codes):
        assert k == c["want"], (c["name"], c["why"], k)
    by_name = {c["name"]: k for c, k in zip(cases, codes)}
    # the crossed, changed and short tuples fail only because of the change: their control passes
    assert by_name["three signers"] == av.SUCCESS
    for name in ("two messages swapped", "two keys swapped", "wrong message", "one signer left out"):
        assert by_name[name] == av.VERIFY_FAIL
    sizes = {len(c["pks"]) for c in cases if c["name"].startswith("valid n ")}
    assert sizes == set(av.VALID_SIZES)
    assert {len(m) for c in cases for m in c["msgs"]} >= set(av.MSG_LENGTHS)
    assert set(codes) == {av.SUCCESS, av.BAD_ENCODING, av.NOT_ON_CURVE, av.NOT_IN_GROUP, av.VERIFY_FAIL, av.PK_IS_INFINITY}


def test_scale_batches_verify(O):
    for T, n, bad in ((7, 33, 3), (5, 1, 2), (2, 64, 0)):
        tuples = av.scale(O, T, n, seed=T, bad_every=bad)
        assert av.oracle_codes(O, tuples) == [t["want"] for t in tuples], (T, n)
        assert (av.VERIFY_FAIL in [t["want"] for t in tuples]) == bool(bad)


def test_c_and_python_oracles_agree(O, cases):
    small = [c for c in cases if len(c["pks"]) <= 3 and len(c["msgs"]) <= 3][::3][:8]
    assert len(small) >= 6
    for c, k in zip(small, av.oracle_codes(O, small)):
        assert bo.aggregate_verify(c["pks"], c["msgs"], c["sig"]) == k, c["name"]


def test_flatten_round_trip(cases):
    keys, koff, msgs, grp, sigs = av.flatten(cases)
    assert len(keys) == 48 * koff[-1] and len(sigs) == 96 * len(cases) and len(msgs) == grp[-1]
    for t, c in enumerate(cases):
        assert keys[48 * koff[t]:48 * koff[t + 1]] == b"".join(c["pks"]) and msgs[grp[t]:grp[t + 1]] == c["msgs"]


@pytest.mark.parametrize("name", list(av.segment_layouts()))
def test_fold_plan_depth(name):
    lengths = av.segment_layouts()[name]
    levels = av.fold_levels(lengths)
    assert max(levels[-1][1], default=0) <= 2
    longest = max(lengths)
    assert len(levels) <= max(1, math.ceil(math.log(max(longest, 2), 32)) + 1), (name, len(levels))
    for (n_in, pieces), (n_next, _) in zip(levels, levels[1:]):
        assert n_next == sum(pieces) and n_next < n_in
