"""CPU: the groups of tests/aggregate_batch_cases.py are what they claim to be.  Their expected verdicts and sums (closed
forms of the progressions, codes by construction) agree with oracle/bls_oracle.py's aggregate and
eth_aggregate_public_keys; tests/test_aggregate_batch_gpu.py runs the same groups through the CUDA kernels."""
from __future__ import annotations

import pytest

from oracle import bls_oracle as bo
from tests import aggregate_batch_cases as ac
from tests import torsion_cases as tc


@pytest.fixture(scope="module")
def torsion():
    return tc.g1_cases(), tc.g2_cases()


def test_progressions_match_their_closed_form():
    h = bo.hash_to_g2(b"progression")
    for E, base in ((ac.G1, bo.G1_GEN), (ac.G2, h)):
        pts = ac.progression(E, base, 12345, 7, 9)
        acc = None
        for k, p in enumerate(pts):
            assert p == E.mul(base, 12345 + 7 * k)
            acc = E.add(acc, p)
        assert acc == ac.progression_sum(E, base, 12345, 7, 9)
        assert E.add(pts[2], pts[2]) == E.mul(pts[2], 2) and E.add(pts[2], E.neg(pts[2])) is None


def test_signature_groups_against_the_oracle(torsion):
    gs = ac.sig_groups(torsion[1])
    assert {g["want"][0] for g in gs if g["want"]} == {0, 1, 2, 3, 16}
    for g in gs:
        got = bo.aggregate(g["items"])
        if g["want"] is not None:
            assert got == g["want"], g["name"]
        else:
            assert got[0] == 0, g["name"]


def test_key_groups_against_the_oracle(torsion):
    gs = ac.key_groups(torsion[0])
    assert {g["want"][0] for g in gs if g["want"]} == {0, 1, 2, 3, 6, 16}
    for g in gs:
        got = bo.eth_aggregate_public_keys(g["items"])
        if g["want"] is not None:
            assert got == g["want"], g["name"]
        else:
            assert got[0] == 0, g["name"]


def test_registry_layout_holds_every_invalid_kind(torsion):
    keys, groups = ac.registry_layout(torsion[0], n_valid=60)
    codes = [bo.key_validate(k)[0] for k in keys]
    assert set(codes) == {0, 1, 2, 3, 6}
    assert all(0 <= i < len(keys) for g in groups for i in g)
    assert any(len(g) != len(set(g)) for g in groups) and [] in groups


def test_small_slot_matches_the_oracle():
    s = ac.slot(committees=2, size=5)
    for c in range(2):
        sigs, keys = s["sigs"][5 * c:5 * c + 5], s["keys"][5 * c:5 * c + 5]
        assert bo.aggregate(sigs) == (0, s["agg_sig"][c])
        assert bo.eth_aggregate_public_keys(keys) == (0, s["agg_pk"][c])
        assert bo.fast_aggregate_verify(keys, s["msgs"][c], s["agg_sig"][c]) == 0
    assert s["offsets"] == [0, 5, 10]
