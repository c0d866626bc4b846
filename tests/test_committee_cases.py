"""The beacon-committee cases (tests/committee_cases.py) on the CPU: the oracle's two formulations of
get_beacon_committee agree, the committee-count regimes are the ones each case is built for, the assignment inverse
matches the committees (and the closed form the device uses for it), and every attestation gets its intended code."""
from __future__ import annotations

import numpy as np
import pytest

from oracle import duties_oracle as do
from tests import committee_cases as cc
from tests import committee_oracle as co

CASES = cc.cases()


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_regime(case):
    for e, want in case.cps.items():
        assert co.committee_count_per_slot(case.st, e) == want, e
    committees = co.beacon_committees(case.st, max(case.cps))
    n = len(do.active_indices(case.st, max(case.cps)))
    assert sum(len(c) for c in committees) == n
    assert sorted(v for c in committees for v in c) == do.active_indices(case.st, max(case.cps)).tolist()
    if n < len(committees):
        assert any(len(c) == 0 for c in committees)


@pytest.mark.parametrize("case", [c for c in CASES if c.small], ids=lambda c: c.name)
def test_two_formulations(case):
    for e in case.cps:
        assert co.beacon_committees(case.st, e, "index") == co.beacon_committees(case.st, e, "list"), e
    slot = do.slot(case.st)
    assert co.beacon_committee(case.st, slot, 0, "index") == co.beacon_committee(case.st, slot, 0, "list")


@pytest.mark.parametrize("case", [c for c in CASES if len(c.st.validators) < 20000], ids=lambda c: c.name)
def test_assignment_inverse(case):
    st = case.st
    spe = co.spe(st)
    for e in case.cps:
        committees = co.beacon_committees(st, e)
        cps = len(committees) // spe
        count = len(committees)
        a = co.committee_assignment(st, e, committees=committees)
        active = set(do.active_indices(st, e).tolist())
        assert set(a) == active
        n = len(active)
        offsets = [n * k // count for k in range(count + 1)]
        for k, members in enumerate(committees):
            for j, v in enumerate(members):
                assert a[v] == (e * spe + k // cps, k % cps, len(members), cps, j)
                p = offsets[k] + j
                kk = ((p + 1) * count - 1) // n   # the closed form of the device's duty kernel
                assert kk == k and p - offsets[kk] == j
        rows = co.duty_rows(st, e, range(len(st.validators)))
        for v in range(len(st.validators)):
            assert (rows[v] == co.NOT_ACTIVE).all() == (v not in active)


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_codes(case):
    cache = {}
    seen = set()
    for data, bits, want in case.attestations:
        code, idx = co.attesting_indices(case.st, data, bits, committees=cache)
        assert code == want, (co.CODES[code], co.CODES[want])
        assert (code == co.OK) == bool(idx)
        assert idx == sorted(set(idx))
        seen.add(code)
    assert {co.OK, co.INDICES_EMPTY, co.BITFIELD, co.INVALID_TARGET_EPOCH, co.NO_DELAY, co.INVALID_INDEX,
            co.MALFORMED_BITS} <= seen or case.name == "minimal_genesis"


def test_every_code_and_length_covered():
    codes, lengths = set(), set()
    for c in CASES:
        for data, bits, want in c.attestations:
            codes.add(want)
            n = co.bitlist_len(bits)
            if n is not None and want in (co.OK, co.INDICES_EMPTY):
                lengths.add(n)
    assert codes == set(co.CODES)
    for L in (0, 7, 8, 9, 15, 16, 17):
        assert L in lengths, L


def test_bitlist_decoding():
    assert co.bitlist_len(b"") is None and co.bitlist_len(b"\x00") is None and co.bitlist_len(b"\xff\x00") is None
    assert co.bitlist_len(b"\x01") == 0 and co.bitlist_len(b"\xff\x01") == 8 and co.bitlist_len(b"\x80") == 7
    assert co.bitlist_len(co.bitlist([True] * 2048)) == 2048 and co.bitlist_len(co.bitlist([True] * 2049)) is None
    for n in (0, 1, 7, 8, 9, 511, 512):
        bits = list(np.random.default_rng(n).random(n) < 0.5)
        b = co.bitlist(bits)
        assert co.bitlist_len(b) == n and len(b) == n // 8 + 1
