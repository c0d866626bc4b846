"""CPU checks of the duty cases (tests/duties_cases.py) against the oracle (oracle/duties_oracle.py): the two
formulations of both sampling loops agree on every case, hand-checkable cases hold, and each case hits its regime."""
from __future__ import annotations

import hashlib

import numpy as np
import pytest

from oracle import duties_oracle as do
from oracle import shuffle_oracle as sh
from tests import duties_cases as dc

CASES = dc.cases()
IDS = [c.name for c in CASES]


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_formulations_agree(case):
    for e in case.epochs:
        assert do.proposer_indices(case.st, e, "index") == do.proposer_indices(case.st, e, "list"), e
    if case.committee:
        assert do.next_sync_committee_indices(case.st, "index") == do.next_sync_committee_indices(case.st, "list")


def _slot_seed(st, epoch, j):
    spe = do.PRESET[st.preset]["SLOTS_PER_EPOCH"]
    base = do.get_seed(st, epoch, do.DOMAIN_BEACON_PROPOSER)
    return hashlib.sha256(base + (epoch * spe + j).to_bytes(8, "little")).digest()


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_regime(case):
    st, P = case.st, do.PRESET[case.st.preset]
    size, spe, rounds = P["SYNC_COMMITTEE_SIZE"], P["SLOTS_PER_EPOCH"], P["SHUFFLE_ROUND_COUNT"]
    epoch = do.slot(st) // spe + 1
    active = do.active_indices(st, epoch)
    r = case.regime
    if r == "one_active":
        assert len(active) == 1
        for e in case.epochs:
            assert do.proposer_indices(st, e) == [int(active[0])] * spe
        assert do.next_sync_committee_indices(st) == [int(active[0])] * size
    elif r == "all_32eth":
        # candidate 0 is always accepted: the proposer is active[compute_shuffled_index(0)] of the slot's seed
        assert (st.validators["effective_balance"] == 32 * dc.ETH).all()
        for e in case.epochs:
            act = do.active_indices(st, e)
            want = [int(act[sh.compute_shuffled_index(0, len(act), _slot_seed(st, e, j), rounds)]) for j in range(spe)]
            assert do.proposer_indices(st, e) == want
        seed = do.get_seed(st, epoch, do.DOMAIN_SYNC_COMMITTEE)
        want = [int(active[sh.compute_shuffled_index(i % len(active), len(active), seed, rounds)]) for i in range(size)]
        assert do.next_sync_committee_indices(st) == want
        assert do.candidates_drawn(st) == size
    elif r == "mixed":
        assert set(np.unique(st.validators["effective_balance"]) // dc.ETH) == {0, 1, 16, 31, 32}
        assert do.candidates_drawn(st) > size
    elif r == "several_windows":
        assert do.candidates_drawn(st) > 4 * size   # windows of size, 2 size, 4 size, ... candidates: at least three
    elif r == "all_0eth":
        assert (st.validators["effective_balance"] == 0).all()
        assert do.candidates_drawn(st) > 64 * size   # accepted only on a random byte of 0
    elif r.startswith("active_"):
        k = int(r.split("_")[1])
        assert len(active) == k and len(do.active_indices(st, case.epochs[0])) == k
        assert do.candidates_drawn(st) > k          # i mod n wraps
    elif r == "inactive_majority":
        assert len(active) < len(st.validators) // 10
    elif r == "minimal":
        assert st.preset == "minimal" and len(do.proposer_indices(st, case.epochs[0])) == 8
        assert len(do.next_sync_committee_indices(st)) == 32
    elif r == "randao_wrap":
        ephv = P["EPOCHS_PER_HISTORICAL_VECTOR"]
        mixes = {(e + ephv - 2) % (1 << 64) % ephv for e in case.epochs + case.seed_epochs}
        assert {ephv - 2, ephv - 1, 0} <= mixes
        assert any(e + ephv - 2 >= 1 << 64 for e in case.seed_epochs)
        assert case.epochs[-1] == (2**64 - 1) // spe
        with pytest.raises(OverflowError):
            do.proposer_indices(st, case.epochs[-1] + 1)
    elif r == "overflow":
        assert int(st.validators["effective_balance"][6]) * 255 % (1 << 64) == 254
        assert any(do.proposer_indices(st, e) != do.proposer_indices(st, e, wrap=False) for e in case.epochs)
        assert do.next_sync_committee_indices(st) != do.next_sync_committee_indices(st, wrap=False)
    elif r == "repeated_keys":
        got = do.sync_committee_indices(st, "current")
        pk = st.validators["public_key"]
        assert all(int(i) >= 300 - 7 for i in got)   # the last holder of each of the 7 tiled keys
        assert got != [j for j in range(512)] and all(pk[i].tobytes() == st.current_sync_committee[48 * j:48 * j + 48]
                                                      for j, i in enumerate(got))
    elif r == "missing_key":
        assert do.sync_committee_indices(st, "current")[5] == do.MISSING
        assert do.sync_committee_indices(st, "next")[511] == do.MISSING
        assert sum(x == do.MISSING for x in do.sync_committee_indices(st, "current")) == 1
    else:
        raise AssertionError(r)


def test_no_active_validator_and_cap():
    st = dc.only_active(dc.base(20, seed=15), [])
    with pytest.raises(do.NoActiveValidator):
        do.proposer_indices(st, 1000)
    with pytest.raises(do.NoActiveValidator):
        do.next_sync_committee_indices(st)


def test_seed_spec():
    st = dc.base(10, seed=16)
    mix = st.randao_mixes[65534].tobytes()
    assert do.get_seed(st, 0, b"\x07\0\0\0") == hashlib.sha256(b"\x07\0\0\0" + bytes(8) + mix).digest()
    mix = st.randao_mixes[(2**64 - 1 + 65534) % 2**64 % 65536].tobytes()
    assert do.get_seed(st, 2**64 - 1, b"\0\0\0\0") == hashlib.sha256(bytes(4) + b"\xff" * 8 + mix).digest()


def test_rotation_oracle():
    st = dc.rotation_state(boundary=True)
    rotated, code, new = do.process_sync_committee_updates(st, aggregate=lambda keys: (0, bytes(48)))
    assert rotated and code == 0 and new.current_sync_committee == st.next_sync_committee
    idx = do.next_sync_committee_indices(st)
    assert new.next_sync_committee[:48 * 512] == b"".join(st.validators["public_key"][i].tobytes() for i in idx)
    st = dc.rotation_state(boundary=False)
    assert do.process_sync_committee_updates(st, aggregate=lambda keys: (0, bytes(48)))[:2] == (False, 0)
