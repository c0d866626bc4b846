"""The committee grid cases (tests/committee_grid_cases.py) on the CPU: each sits on the kernel or host edge it claims,
checked with the oracle (tests/committee_oracle.py): committee lengths and n mod C, each Bitlist's set-bit count, padded
sort size and the gather chunk and lane of its last set bit, every code where it is meant to be, the duty states'
residues and launch tails, the 2^20-attestation batch's vectorised expectation, and the cache model's walk."""
from __future__ import annotations

import numpy as np
import pytest

from oracle import duties_oracle as do
from tests import committee_cases as cc
from tests import committee_grid_cases as gc
from tests import committee_oracle as co

GATHER = gc.gather_cases()
OVER = gc.over_limit_cases()
DUTY = gc.duty_cases()


def set_bits(att) -> list:
    n = co.bitlist_len(att.bits)
    return [i for i in range(n) if att.bits[i // 8] >> (i % 8) & 1]


@pytest.mark.parametrize("case", GATHER, ids=[c.name for c in GATHER])
def test_gather_shapes(case):
    st = case.st
    n = len(do.active_indices(st, gc.E))
    assert n == len(do.active_indices(st, gc.E + 1)) and len(st.validators) == n + 4
    assert co.committee_count_per_slot(st, gc.E) == 4
    L = case.lengths[0]
    assert n == (32 * L + 16 if len(case.lengths) == 2 else 32 * 2048) and n % 32 in (0, 16)
    for e in (gc.E, gc.E + 1):
        assert sorted({len(c) for c in co.beacon_committees(st, e)}) == list(case.lengths)
    # the inactive validators sit at both ends of the index range
    v = st.validators
    assert (v["exit_epoch"][[0, 1, -2, -1]] == gc.DEAD_EXIT).all()
    by = {}
    for a in case.attestations:
        if a.code == co.OK:
            by.setdefault(a.length, {})[a.tag] = a
    assert sorted(by) == list(case.lengths)
    for length, atts in by.items():
        assert {a.epoch for a in atts.values()} == {gc.E, gc.E + 1}
        last = set_bits(atts["last"])
        assert last == [length - 1]
        chunk, warp, lane = gc.chunk_lane(length - 1)
        assert chunk == (length - 1) // 256 and lane == (length - 1) % 32
        assert set_bits(atts["all"]) == list(range(length)) and gc.sort_size(length) == 1 << (length - 1).bit_length()
        assert set_bits(atts["bit0"]) == [0]
        assert len(set_bits(atts["all_but_one"])) == length - 1
        if length > 256:
            assert set_bits(atts["cut255_256"]) == [255, 256]
            assert [gc.chunk_lane(i)[0] for i in (255, 256)] == [0, 1]
            assert length % 256 == 0 or chunk >= 1       # a ragged last chunk beyond the first
        if length > 32:
            assert {gc.chunk_lane(i)[2] for i in set_bits(atts["warp_31_32"])} == {0, 31}
        k = 0
        while (1 << k) + 1 <= length:
            for c in (1 << k, (1 << k) + 1):
                assert len(set_bits(atts[f"count{c}"])) == c
            # 2^k + 1 entries pad to 2^(k + 1): 2^k - 1 pads
            assert gc.sort_size((1 << k) + 1) - ((1 << k) + 1) == (1 << k) - 1
            k += 1
        for d in (0.5, 0.99):
            assert 0 < len(set_bits(atts[f"density{d}"])) <= length
    sizes = {gc.sort_size(len(set_bits(a))) for a in case.attestations if a.code == co.OK}
    assert max(sizes) == gc.sort_size(max(case.lengths))
    if max(case.lengths) > 1024:
        assert 2048 in sizes
    # every failure code once; first and last fail; two failures next to each other in the middle
    codes = [a.code for a in case.attestations]
    assert sorted(c for c in codes if c) == sorted(gc.FAILS)
    assert codes[0] == co.MALFORMED_BITS and codes[-1] == co.INDICES_EMPTY
    assert any(codes[j] and codes[j + 1] for j in range(1, len(codes) - 2))
    cache = {}
    for a in case.attestations:
        code, idx = co.attesting_indices(st, a.data, a.bits, committees=cache)
        assert code == a.code, (a.tag, co.CODES[code])
        if code == co.OK:
            assert len(idx) == len(set_bits(a))


def test_gather_lengths_covered():
    lengths = set()
    sizes = set()
    for c in GATHER:
        for a in c.attestations:
            if a.code == co.OK:
                lengths.add(a.length)
                sizes.add(gc.sort_size(len(set_bits(a))))
    assert lengths == {31, 32, 255, 256, 511, 512, 1023, 1024, 2047, 2048}
    assert sizes == {1 << k for k in range(12)}


@pytest.mark.parametrize("case", OVER, ids=[c.name for c in OVER])
def test_over_limit_shapes(case):
    st = case.st
    for e in (gc.E, gc.E + 1):
        committees = co.beacon_committees(st, e)
        lengths = [len(c) for c in committees]
        assert max(lengths) == 2049 and sorted(set(lengths)) == list(case.lengths)
        if case.name == "over_one":
            assert lengths.count(2049) == 1 and lengths[31] == 2049
    cache = {}
    for a in case.attestations:
        assert a.length == 2049
        assert co.attesting_indices(st, a.data, a.bits, committees=cache)[0] == a.code
        assert co.bitlist_len(a.bits) == (2048 if a.code == co.BITFIELD else None)
    ok = gc.over_one_ok(OVER[0])
    assert co.attesting_indices(OVER[0].st, ok.data, ok.bits)[0] == co.OK and ok.length == 2048


@pytest.mark.parametrize("case", DUTY, ids=[c.name for c in DUTY])
def test_duty_shapes(case):
    st = case.st
    N = len(st.validators)
    n = len(do.active_indices(st, gc.E))
    C = case.C
    assert C == co.spe(st) * co.committee_count_per_slot(st, gc.E)
    assert n < C or n % C in (0, 1, C - 1)
    assert N % gc.ROW_THREADS in (0, 1, 255)
    rows = co.duty_rows(st, gc.E, range(N))
    assert rows[0, 0] == co.NOT_ACTIVE and rows[N - 1, 0] == co.NOT_ACTIVE
    for n_rows, v in case.lists.items():
        assert v.size == n_rows and int(v[0]) == N - 1
        if n_rows > 1:
            assert len(set(v.tolist())) < n_rows and 0 in v.tolist()
            assert (rows[v.astype(np.int64), 0] == co.NOT_ACTIVE).any() and (rows[v.astype(np.int64), 0] != co.NOT_ACTIVE).any()
    # the closed form of k_attester_duties at every position, and positions where (p + 1) C is a multiple of n
    p = np.arange(n, dtype=object)
    k = ((p + 1) * C - 1) // n
    start = n * k // C
    assert all(start <= p) and all(p < n * (k + 1) // C)
    assert n < C or any(((p + 1) * C) % n == 0)


def test_duty_cases_cover_presets_and_residues():
    seen = {(c.st.preset, (len(do.active_indices(c.st, gc.E)) % c.C if len(do.active_indices(c.st, gc.E)) >= c.C else "below")) for c in DUTY}
    for preset, C in (("minimal", 32), ("mainnet", 64)):
        assert {(preset, 0), (preset, 1), (preset, C - 1), (preset, "below")} <= seen
    assert {len(c.st.validators) % 256 for c in DUTY} == {0, 1, 255}


def test_appended_records():
    case = gc.duty_cases()[1]
    st = case.st
    N = len(st.validators)
    recs, bal = gc.appended(st, N + 101, seed=1300)
    st.add_validators(recs, bal)
    assert len(st.validators) > 2 * N
    act = {e: set(do.active_indices(st, e).tolist()) for e in (gc.E, gc.E + 1)}
    new = range(N, len(st.validators))
    assert all(i in act[gc.E] for i in new[0::3]) and all(i in act[gc.E + 1] for i in new[0::3])
    assert not any(i in act[gc.E] or i in act[gc.E + 1] for i in new[1::3])
    assert all(i in act[gc.E] and i not in act[gc.E + 1] for i in new[2::3])


def test_bound_batch():
    b = gc.bound_batch()
    A = b.codes.size
    assert A == gc.MAX_ATTESTATIONS and b.bits.shape == (A, 5)
    assert b.members.shape == (60, gc.BOUND_L)
    st = b.st
    for e in (gc.E, gc.E + 1):
        assert {len(c) for c in co.beacon_committees(st, e)} == {gc.BOUND_L}
    codes, counts = np.unique(b.codes, return_counts=True)
    got = dict(zip(codes.tolist(), counts.tolist()))
    assert set(got) == {co.OK, co.INDICES_EMPTY, co.BITFIELD, co.NO_DELAY, co.INVALID_INDEX, co.MALFORMED_BITS}
    assert got[co.OK] > A - 300 and b.codes[-1] != co.OK
    off, idx = gc.bound_expected(b)
    assert off.size == A + 1 and idx.size == int(off[-1])
    # the vectorised expectation against the oracle on a sample and on every failure
    rng = np.random.default_rng(0)
    sample = sorted(set(rng.choice(A, 3000, replace=False).tolist()) | set(np.nonzero(b.codes != co.OK)[0].tolist()))
    cache = {}
    for a in sample:
        code, want = co.attesting_indices(st, b.data[a].tobytes(), b.bits[a].tobytes(), committees=cache)
        assert code == b.codes[a], a
        assert idx[off[a]:off[a + 1]].tolist() == want, a


def test_lru_model():
    m = gc.LRU()
    launches = [m.use(e) for e in gc.LRU_WALK]
    E = gc.E
    assert launches[:4] == [gc.MISS] * 4 and launches[4] == 0           # E - 1 again: a hit
    assert launches[5] == gc.MISS and launches[6] == gc.MISS            # E + 3 evicts E, which then misses
    assert 0 in launches[7:] and launches.count(gc.MISS) > 6
    assert len(m.entries) == 4 and list(m.entries)[-1] == gc.LRU_WALK[-1]
    d = gc.LRU()
    assert [d.duties(E), d.duties(E), d.use(E + 1), d.duties(E + 1)] == [gc.MISS + 2, 1, gc.MISS, 2]
