"""Beacon committees on the device at their kernels' launch edges (tests/committee_grid_cases.py) against the oracle
(tests/committee_oracle.py), value for value and with launch counts: `k_attesting_indices` over committees of 31 to
2 048 members with Bitlists at every gather-chunk, warp and sort-size edge, mixed with failures of every code;
committees of 2 049 members refused before the gather; `k_attester_duties` at committee cuts, launch tails and after
the registry more than doubles; a 2^22 + 3-validator mainnet state; exactly 2^20 attestations in one call; and the
four-entry committee cache: eviction order, rebuilt inverse maps, two handles, shared shuffle scratch, writes that
change no record, and a slot that crosses into the next epoch."""
from __future__ import annotations

import time

import numpy as np
import pytest

from ethereum_consensus_b200 import _lib, duties, epoch, shuffling, ssz
from ethereum_consensus_b200 import state as S
from oracle import duties_oracle as do
from tests import committee_grid_cases as gc
from tests import committee_oracle as co

pytestmark = pytest.mark.gpu
E = gc.E
MISS = gc.MISS
GATHER = gc.gather_cases()
OVER = gc.over_limit_cases()
DUTY = gc.duty_cases()


@pytest.fixture(scope="module", autouse=True)
def _wall():
    t = time.time()
    yield
    print(f"\ntest_committee_grid_gpu.py wall {time.time() - t:.1f} s")


def counted(fn):
    L = _lib.lib()
    c0 = L.b200_launch_count()
    r = fn()
    return r, L.b200_launch_count() - c0


def upload(st):
    return ssz.DeviceBeaconState(S.serialize(st), st.preset)


def rows_of(dev, e, validators=None) -> np.ndarray:
    return duties.attester_duties(dev, e, validators).view(np.uint64).reshape(-1, 5)


def raw_attesting(dev, data: np.ndarray, bits: np.ndarray, bits_offsets: np.ndarray):
    """b200_state_attesting_indices on numpy buffers -> (indices, out_offsets, codes).  The index buffer holds every set
    bit of every Bitlist, delimiters included, so no total the host could compute overruns it."""
    n = bits_offsets.size - 1
    cap = max(1, int(np.unpackbits(bits).sum()))
    out = np.zeros(cap, np.uint64)
    off = np.zeros(n + 1, np.uint32)
    codes = np.zeros(n, np.int32)
    _lib.check(_lib.lib().b200_state_attesting_indices(dev._h, n, _lib.ptr(data), _lib.ptr(bits), _lib.ptr(bits_offsets),
                                                       _lib.ptr(out), _lib.ptr(off), _lib.ptr(codes)), "state_attesting_indices")
    return out, off, codes


def check_batch(dev, st, atts):
    """One attesting_indices call on `atts`, compared with the oracle: codes, out_offsets and indices.  -> launches."""
    data = np.frombuffer(b"".join(a.data for a in atts), np.uint8).copy()
    bits = np.frombuffer(b"".join(a.bits for a in atts) or bytes(1), np.uint8).copy()
    boff = np.concatenate([[0], np.cumsum([len(a.bits) for a in atts])]).astype(np.uint32)
    (out, off, codes), k = counted(lambda: raw_attesting(dev, data, bits, boff))
    cache = {}
    want = [co.attesting_indices(st, a.data, a.bits, committees=cache) for a in atts]
    assert [w[0] for w in want] == [a.code for a in atts]
    bad = [(j, a.tag) for j, (a, w, c) in enumerate(zip(atts, want, codes)) if int(c) != w[0]]
    assert bad == [], bad
    want_off = np.concatenate([[0], np.cumsum([len(w[1]) for w in want])]).astype(np.uint32)
    assert off.tolist() == want_off.tolist()
    bad = [(j, a.tag, a.length) for j, (a, w) in enumerate(zip(atts, want)) if out[off[j]:off[j + 1]].tolist() != w[1]]
    assert bad == [], bad
    return k


# ---- 1. gather chunks and sort sizes ----
@pytest.mark.parametrize("case", GATHER, ids=[c.name for c in GATHER])
def test_gather(engine, case):
    dev = upload(case.st)
    # both epochs built on first use, then one gather over every passing attestation
    assert check_batch(dev, case.st, case.attestations) == 2 * MISS + 1
    assert check_batch(dev, case.st, case.attestations) == 1
    # failures alone: nothing passes, no gather
    assert check_batch(dev, case.st, [a for a in case.attestations if a.code != co.OK]) == 0
    dev.close()


# ---- 2. past MAX_VALIDATORS_PER_COMMITTEE ----
@pytest.mark.parametrize("case", OVER, ids=[c.name for c in OVER])
def test_over_limit(engine, case):
    st = case.st
    dev = upload(st)
    epochs = sorted({a.epoch for a in case.attestations})
    # BITFIELD reaches the committee (its epoch is built), MALFORMED_BITS does not; neither launches the gather
    assert check_batch(dev, st, case.attestations) == MISS * len(epochs)
    assert check_batch(dev, st, case.attestations) == 0
    N = len(st.validators)
    for e in (E, E + 1):
        want = co.beacon_committees(st, e)
        idx, off, cps = duties.beacon_committees(dev, e)
        lengths = np.diff(off.astype(np.int64))
        assert cps == 4 and sorted(set(lengths.tolist())) == list(case.lengths)
        assert [idx[off[k]:off[k + 1]].tolist() for k in range(len(off) - 1)] == want
        rows = rows_of(dev, e)
        assert np.array_equal(rows, co.duty_rows(st, e, range(N))), e
        active = rows[:, 0] != co.NOT_ACTIVE
        assert (rows[active, 2] == 2049).sum() == sum(len(c) for c in want if len(c) == 2049)
    if case.name == "over_one":
        assert check_batch(dev, st, case.attestations + [gc.over_one_ok(case)]) == 1
    dev.close()


# ---- 3. duty rows at committee cuts ----
@pytest.mark.parametrize("case", DUTY, ids=[c.name for c in DUTY])
def test_duty_rows(engine, case):
    st = case.st
    dev = upload(st)
    N = len(st.validators)
    for e in (E, E + 1):
        want = co.duty_rows(st, e, range(N))
        rows, k = counted(lambda: rows_of(dev, e))
        assert k == MISS + 1 + 1, e            # the epoch, its inverse map, the rows
        assert np.array_equal(rows, want), (e, np.nonzero((rows != want).any(1))[0][:8])
        for n_rows, v in case.lists.items():
            got, k = counted(lambda: rows_of(dev, e, v))
            assert k == 1 and np.array_equal(got, want[v.astype(np.int64)]), (e, n_rows)
    dev.close()


def test_duty_rows_after_append(engine):
    case = gc.duty_cases()[1]                   # minimal, n_active = 1 (mod 32), N = 1 (mod 256)
    st = case.st
    dev = upload(st)
    N = len(st.validators)
    assert np.array_equal(rows_of(dev, E), co.duty_rows(st, E, range(N)))
    recs, bal = gc.appended(st, N + 101, seed=1300)
    dev.add_validators(recs.tobytes(), bal)
    st.add_validators(recs, bal)
    N2 = len(st.validators)
    assert N2 > 2 * N and dev.n_validators == N2
    for e in (E, E + 1):
        want = co.duty_rows(st, e, range(N2))
        rows, k = counted(lambda: rows_of(dev, e))
        # the records changed: the epoch is rebuilt and its inverse map built again at N2 entries
        assert k == MISS + 1 + 1, e
        assert np.array_equal(rows, want), (e, np.nonzero((rows != want).any(1))[0][:8])
        new = np.array([N, N + 1, N + 2, N2 - 1, N2 - 2, N2 - 3, N - 1, 0], np.uint64)
        assert np.array_equal(rows_of(dev, e, new), want[new.astype(np.int64)])
        assert (want[N::3, 0] != co.NOT_ACTIVE).all() and (want[N + 1::3, 0] == co.NOT_ACTIVE).all()
        assert (want[N + 2::3, 0] != co.NOT_ACTIVE).all() == (e == E)
    dev.close()


# ---- 4. one large mainnet state past the limit ----
@pytest.fixture(scope="module")
def big():
    # 2^22 + 3 active: 2 048 committees of 2 048 and three of 2 049; the slot is the first of E + 1, so E is "previous"
    return gc.grid_state((1 << 22) + 3, "mainnet", seed=1100, dead=4, slot_in_epoch=32)


def test_big_state_past_limit(engine, big):
    t0 = time.time()
    st = big
    dev = upload(st)
    N = len(st.validators)
    for e in (E, E + 1):
        seed = duties.get_seed(dev, e, duties.DOMAIN_BEACON_ATTESTER)
        shuffled = shuffling.state_shuffled_active_indices(dev, e, seed)
        n = shuffled.size
        assert n == (1 << 22) + 3
        idx, off, cps = duties.beacon_committees(dev, e)
        assert cps == 64 and off.size == 2049 and np.array_equal(idx, shuffled)
        assert off.tolist() == [n * k // 2048 for k in range(2049)]
        lengths = np.diff(off.astype(np.int64))
        assert (lengths == 2049).sum() == 3 and (lengths == 2048).sum() == 2045
        want = np.full((N, 5), co.NOT_ACTIVE, np.uint64)
        for k in range(2048):
            m = shuffled[off[k]:off[k + 1]]
            want[m.astype(np.int64)] = np.stack([np.full(m.size, e * 32 + k // 64), np.full(m.size, k % 64), np.full(m.size, m.size),
                                                 np.full(m.size, 64), np.arange(m.size)], 1).astype(np.uint64)
        rows = rows_of(dev, e)
        assert np.array_equal(rows, want), (e, np.nonzero((rows != want).any(1))[0][:8])
        del rows, want
        if e != E:
            continue
        # every 2 048-member committee of E fully attested, and one 2 048-bit list on a 2 049-member committee
        full = co.bitlist([True] * 2048)
        atts, expect = [], []
        for k in range(2048):
            d = co.attestation_data(e * 32 + k // 64, k % 64, e)
            if lengths[k] == 2048:
                atts.append((d, full))
                expect.append((co.OK, np.sort(idx[off[k]:off[k + 1]])))
        k_over = int(np.nonzero(lengths == 2049)[0][1])
        atts.insert(1000, (co.attestation_data(e * 32 + k_over // 64, k_over % 64, e), full))
        expect.insert(1000, (co.BITFIELD, np.zeros(0, np.uint64)))
        (got, codes), k = counted(lambda: duties.attesting_indices(dev, atts))
        assert k == 1
        assert codes.tolist() == [c for c, _ in expect]
        assert all(np.array_equal(g, w) for g, (_, w) in zip(got, expect))
    dev.close()
    print(f"\n2^22 + 3-validator state: {time.time() - t0:.1f} s")


# ---- 5. the batch bound ----
def test_attestation_bound(engine):
    b = gc.bound_batch()
    dev = upload(b.st)
    want_off, want_idx = gc.bound_expected(b)
    for e in (E, E + 1):                        # both epochs cached: the call launches the gather alone
        duties.committee_count_per_slot(dev, e)
    boff = (np.arange(b.bits.shape[0] + 1) * b.bits.shape[1]).astype(np.uint32)
    (out, off, codes), k = counted(lambda: raw_attesting(dev, b.data.reshape(-1), b.bits.reshape(-1), boff))
    assert codes.size == gc.MAX_ATTESTATIONS and k == 1
    assert np.array_equal(codes, b.codes)
    assert (codes == co.OK).sum() > gc.MAX_ATTESTATIONS - 300      # about 2^20 gather CTAs in one launch
    assert np.array_equal(off, want_off)
    assert np.array_equal(out[:int(off[-1])], want_idx)
    dev.close()


# ---- 6. the cache ----
def answers_equal(dev, st, e):
    want = co.beacon_committees(st, e)
    idx, off, cps = duties.beacon_committees(dev, e)
    assert cps == len(want) // co.spe(st)
    assert [idx[off[k]:off[k + 1]].tolist() for k in range(len(off) - 1)] == want


def test_cache_lru_order(engine):
    st = gc.grid_state(300, "minimal", seed=1400)
    dev = upload(st)
    model = gc.LRU()
    for e in gc.LRU_WALK:
        c, k = counted(lambda: duties.committee_count_per_slot(dev, e))
        assert (c, k) == (co.committee_count_per_slot(st, e), model.use(e)), e
        (_, k2) = counted(lambda: answers_equal(dev, st, e))
        assert k2 == model.use(e) == 0
    dev.close()


def test_cache_rebuilds_inverse_map(engine):
    st = gc.grid_state(1000, "minimal", seed=1401)
    dev = upload(st)
    N = len(st.validators)
    model = gc.LRU()
    want = {e: co.duty_rows(st, e, range(N)) for e in range(E - 3, E + 3)}

    def duty(e):
        rows, k = counted(lambda: rows_of(dev, e))
        assert k == model.duties(e) and np.array_equal(rows, want[e]), e
        return k
    assert [duty(e) for e in (E - 1, E, E + 1, E + 2)] == [MISS + 2] * 4
    assert duty(E) == 1
    # E - 3 and E - 2 take the entries of E - 1 and E + 1, whose maps were built
    for e in (E - 3, E - 2):
        (_, k) = counted(lambda: duties.committee_count_per_slot(dev, e))
        assert k == model.use(e) == MISS
    assert duty(E - 2) == 1 + 1 and duty(E - 3) == 1 + 1 and duty(E - 3) == 1
    assert duty(E - 1) == MISS + 2 and duty(E + 1) == MISS + 2 and duty(E - 1) == 1
    dev.close()


def test_cache_both_epochs_evicted(engine):
    st = gc.grid_state(700, "minimal", seed=1402)
    dev = upload(st)
    atts = gc.some_attestations(st, 1402)
    assert check_batch(dev, st, atts) == 2 * MISS + 1
    for e in (E - 4, E - 3, E - 2, E + 2):      # four other epochs: E (previous) and E + 1 (current) evicted
        duties.committee_count_per_slot(dev, e)
    assert check_batch(dev, st, atts) == 2 * MISS + 1
    assert check_batch(dev, st, atts) == 1
    dev.close()


def test_cache_two_handles(engine):
    a = gc.grid_state(400, "minimal", seed=1403)
    b = gc.grid_state(650, "minimal", seed=1404)
    b.randao_mixes = a.randao_mixes.copy()      # equal seeds at every epoch
    da, db = upload(a), upload(b)
    assert duties.get_seed(da, E, duties.DOMAIN_BEACON_ATTESTER) == duties.get_seed(db, E, duties.DOMAIN_BEACON_ATTESTER)
    atts = {id(a): gc.some_attestations(a, 1), id(b): gc.some_attestations(b, 2)}
    for rnd in range(2):
        for e in (E, E + 1):
            for st, dev in ((a, da), (b, db)):
                answers_equal(dev, st, e)
                assert np.array_equal(rows_of(dev, e), co.duty_rows(st, e, range(len(st.validators))))
        for st, dev in ((b, db), (a, da)):
            assert check_batch(dev, st, atts[id(st)]) == 1
    da.close()
    db.close()


def test_cache_survives_shared_scratch(engine):
    st = gc.grid_state(500, "minimal", seed=1405)
    dev = upload(st)
    other = upload(gc.grid_state(20000, "minimal", seed=1406))
    atts = gc.some_attestations(st, 3)
    before = [duties.beacon_committees(dev, e) for e in (E, E + 1)]
    rows = [rows_of(dev, e) for e in (E, E + 1)]
    check_batch(dev, st, atts)

    def unchanged():
        for e, (idx, off, cps), r in zip((E, E + 1), before, rows):
            (got, k) = counted(lambda: duties.beacon_committees(dev, e))
            assert k == 0 and np.array_equal(got[0], idx) and np.array_equal(got[1], off) and got[2] == cps
            (got, k) = counted(lambda: rows_of(dev, e))
            assert k == 1 and np.array_equal(got, r)
        assert check_batch(dev, st, atts) == 1
    shuffling.state_shuffled_active_indices(other, E, bytes(range(32)))
    unchanged()
    duties.proposer_indices(dev, E + 1)
    duties.proposer_indices(other, E)
    unchanged()
    duties.next_sync_committee(dev)
    duties.committee_count_per_slot(other, E)
    unchanged()
    shuffling.state_shuffled_active_indices(dev, E, bytes(32))
    unchanged()
    answers_equal(dev, st, E)
    dev.close()
    other.close()


def test_cache_kept_without_record_change(engine):
    st = gc.grid_state(600, "minimal", seed=1407)
    dev = upload(st)
    vo, vlen = S.layout(st)["validators"]
    recs = dev.read_bytes(vo, vlen)
    for e in (E, E + 1):
        answers_equal(dev, st, e)
        rows_of(dev, e)
    for steps in (["participation_flag_updates"], ["registry_updates"], ["participation_flag_updates", "registry_updates"]):
        epoch.process_epoch(dev, steps)
        assert dev.read_bytes(vo, vlen) == recs, steps   # nothing to eject or activate
        for e in (E, E + 1):
            (_, k) = counted(lambda: answers_equal(dev, st, e))
            assert k == 0, steps
            (r, k) = counted(lambda: rows_of(dev, e))
            assert k == 1 and np.array_equal(r, co.duty_rows(st, e, range(len(st.validators))))
    dev.close()


def test_cache_slot_advance(engine):
    st = gc.grid_state(800, "minimal", seed=1408)   # slot: the last of E + 1
    dev = upload(st)
    assert check_batch(dev, st, gc.some_attestations(st, 4)) == 2 * MISS + 1
    slot = (E + 2) * 8 + 5
    dev.update_bytes(S.layout(st)["slot"][0], slot.to_bytes(8, "little"))
    st.fixed["slot"] = slot.to_bytes(8, "little")
    atts = gc.some_attestations(st, 5)              # previous E + 1 (cached as the old current), current E + 2
    assert {a.epoch for a in atts} == {E + 1, E + 2}
    assert check_batch(dev, st, atts) == MISS + 1
    old = gc.some_attestations(gc.grid_state(800, "minimal", seed=1408), 4)
    got, codes = duties.attesting_indices(dev, [(a.data, a.bits) for a in old])
    assert [int(c) for c in codes] == [co.INVALID_TARGET_EPOCH if a.epoch == E else co.OK for a in old]
    dev.close()
