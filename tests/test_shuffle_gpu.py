"""GPU parity for committee shuffling (SURVEY.md §8f-3) against the oracle's two formulations of
ethereum-consensus/src/phase0/helpers.rs:249-360 and `get_active_validator_indices` (:646-676)."""
import hashlib

import numpy as np
import pytest

from ethereum_consensus_b200 import shuffling, ssz, state as S
from oracle import shuffle_oracle as sh

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("rounds", [10, 90])
def test_shuffled_indices_small_sizes(engine, rounds):
    for n in list(range(0, 20)) + [255, 256, 257, 300, 1000, 4097]:
        seed = hashlib.sha256(b"gpu seed %d" % n).digest()
        got = shuffling.compute_shuffled_indices(n, seed, rounds)
        assert got.tolist() == sh.compute_shuffled_indices(list(range(n)), seed, rounds), n
    seed = hashlib.sha256(b"vals").digest()
    vals = np.arange(777, dtype=np.uint64) * 13 + 5
    assert shuffling.compute_shuffled_indices(vals, seed, rounds).tolist() == sh.compute_shuffled_indices(vals.tolist(), seed, rounds)
    assert shuffling.compute_shuffled_index(5, 300, seed, rounds) == sh.compute_shuffled_index(5, 300, seed, rounds)
    with pytest.raises(ValueError):
        shuffling.compute_shuffled_index(300, 300, seed, rounds)


def test_shuffled_indices_full_registry(engine):
    """n = 2**20 (BASELINE's registry size), 90 rounds, against the vectorised oracle; a permutation by construction."""
    seed = hashlib.sha256(b"epoch seed").digest()
    n = 1 << 20
    got = shuffling.compute_shuffled_indices(n, seed, 90)
    assert np.array_equal(got, sh.shuffled_indices_numpy(n, seed, 90))
    assert np.array_equal(np.sort(got), np.arange(n, dtype=np.uint64))


def test_active_indices_and_state_resident_shuffle(engine):
    st = S.synth_state(70_001, "mainnet", n_historical_summaries=3, n_historical_roots=2)
    ser = S.serialize(st)
    vo, vl = S.layout(st)["validators"]
    recs = ser[vo: vo + vl]
    dev = ssz.DeviceBeaconState(ser, "mainnet")
    assert dev.n_validators == 70_001
    seed = hashlib.sha256(b"attester seed").digest()
    for epoch in (0, 1 << 17, 1 << 18, 2**64 - 1):
        want_act = sh.get_active_validator_indices(bytes(recs), epoch)
        got_act = shuffling.get_active_validator_indices(recs, epoch)
        assert got_act.tolist() == want_act
        got = shuffling.state_shuffled_active_indices(dev, epoch, seed, 90)
        assert np.array_equal(got, sh.shuffled_indices_numpy(np.array(want_act, dtype=np.uint64), seed, 90))
        if len(want_act) >= 64:   # get_beacon_committee = a slice of the shuffled list (compute_committee)
            c = shuffling.compute_committee(got, 3, 64)
            n = len(want_act)
            assert c.tolist() == got[n * 3 // 64: n * 4 // 64].tolist()
    dev.close()
    assert shuffling.get_active_validator_indices(np.zeros(0, dtype=np.uint8), 5).tolist() == []
