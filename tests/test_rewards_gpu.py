"""The reward and penalty deltas on the device-resident state (ethereum_consensus_b200.epoch.deltas) against the oracle
(tests/rewards_oracle.py): every seeded case list for list, a 2^20-validator state, refusals, the call leaving the state
and its caches as they were, the deltas applied on the host against process_epoch's rewards_and_penalties, interleaving
with process_epoch, the duties and the registry on one handle, and the pinned launch count."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from ethereum_consensus_b200 import _lib, crypto, duties, epoch, ssz
from ethereum_consensus_b200 import state as S
from oracle import bls_oracle as bo
from oracle import duties_oracle as do
from oracle import epoch_oracle as eo
from tests import epoch_cases as ec
from tests import rewards_cases as rc
from tests import rewards_oracle as ro

pytestmark = pytest.mark.gpu
CASES = rc.cases()
CODE = {"bad_arg": _lib.ERR_BAD_ARG, "limit": _lib.ERR_LIMIT}


def upload(st):
    return ssz.DeviceBeaconState(S.serialize(st), st.preset)


def balances(dev, st) -> np.ndarray:
    o, ln = S.layout(st)["balances"]
    return np.frombuffer(dev.read_bytes(o, ln), "<u8").astype(np.uint64)


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_case_matches_oracle(engine, case):
    dev = upload(case.st)
    before, root = dev.read_bytes(0, dev.serialized_len()), dev.hash_tree_root()
    if case.refusal:
        with pytest.raises(_lib.EngineError) as ei:
            epoch.deltas(dev)
        assert ei.value.code == CODE[case.refusal]
    else:
        got = epoch.deltas(dev)
        want = ro.deltas(case.st)
        assert got.shape == want.shape and got.dtype == np.uint64
        for k, name in enumerate(epoch.DELTAS):
            for j, what in enumerate(("rewards", "penalties")):
                assert np.array_equal(got[k, j], want[k, j]), (name, what)
    assert dev.read_bytes(0, len(before)) == before
    assert dev.hash_tree_root_incremental() == root == dev.hash_tree_root()
    dev.close()


def big_state(n=1 << 20):
    rng = np.random.default_rng(2021)
    st = ec.base(n, 1000, seed=2021)
    v = st.validators
    v["slashed"][rng.random(n) < 0.002] = 1
    exited = rng.random(n) < 0.01
    v["exit_epoch"][exited] = rng.integers(900, 1010, exited.sum(), dtype=np.uint64)
    v["withdrawable_epoch"][exited] = v["exit_epoch"][exited] + rng.integers(0, 300, exited.sum(), dtype=np.uint64)
    v["effective_balance"][rng.random(n) < 0.01] = 16 * ec.ETH
    v["activation_epoch"][rng.random(n) < 0.002] = 1000
    st.inactivity_scores[rng.random(n) < 0.05] = 5000
    return st


def test_two_pow_20(engine):
    st = big_state()
    dev = upload(st)
    assert np.array_equal(epoch.deltas(dev), ro.deltas(st))
    # and in a leak, where the flag rewards vanish
    st.fixed["finalized_checkpoint"] = ec._cp(900, b"f")
    dev2 = upload(st)
    got = epoch.deltas(dev2)
    assert not got[:, 0].any()
    assert np.array_equal(got, ro.deltas(st))


def test_refusals(engine):
    L = _lib.lib()
    st = ec.base(100, 1000, seed=160)
    dev = upload(st)
    before, root = dev.read_bytes(0, dev.serialized_len()), dev.hash_tree_root()
    out = np.zeros(8 * 101, np.uint64)
    assert L.b200_state_epoch_deltas(None, out.ctypes.data, 100) == _lib.ERR_BAD_ARG
    assert L.b200_state_epoch_deltas(dev._h, None, 100) == _lib.ERR_BAD_ARG
    for n in (0, 99, 101):
        assert L.b200_state_epoch_deltas(dev._h, out.ctypes.data, n) == _lib.ERR_BAD_ARG, n
    odd = ec.base(100, 1000, seed=161)
    odd.current_epoch_participation = odd.current_epoch_participation[:99].copy()
    dev_odd = upload(odd)
    r_odd = dev_odd.hash_tree_root()
    with pytest.raises(_lib.EngineError) as ei:
        epoch.deltas(dev_odd)
    assert ei.value.code == _lib.ERR_BAD_ARG
    assert dev_odd.hash_tree_root_incremental() == r_odd
    from ethereum_consensus_b200 import parallel
    parallel.comm_init(0, 1)
    shd = ssz.DeviceBeaconState(S.serialize(st), "mainnet", sharded=True)
    assert L.b200_state_epoch_deltas(shd._h, out.ctypes.data, 100) == _lib.ERR_BAD_ARG
    assert shd.hash_tree_root() == root
    assert dev.read_bytes(0, len(before)) == before
    assert dev.hash_tree_root_incremental() == root == dev.hash_tree_root()
    assert np.array_equal(epoch.deltas(dev), ro.deltas(st))


def test_read_only(engine):
    """Bytes, both roots, the incremental root's work and a cached committee epoch are as they were after the call."""
    L = _lib.lib()
    st = ec.base(3000, 1000, seed=162)
    dev = upload(st)
    before = dev.read_bytes(0, dev.serialized_len())
    root = dev.hash_tree_root()
    dev.hash_tree_root_incremental()
    c0 = L.b200_launch_count()
    assert dev.hash_tree_root_incremental() == root
    idle = L.b200_launch_count() - c0
    cached = duties.beacon_committees(dev, 1000)
    for _ in range(2):
        d = epoch.deltas(dev)
        c0 = L.b200_launch_count()
        assert dev.hash_tree_root_incremental() == root
        assert L.b200_launch_count() - c0 == idle
        c0 = L.b200_launch_count()
        again = duties.beacon_committees(dev, 1000)
        assert L.b200_launch_count() - c0 == 0
        assert all(np.array_equal(a, b) for a, b in zip(again, cached))
    assert dev.read_bytes(0, len(before)) == before
    assert dev.hash_tree_root() == root
    assert np.array_equal(d, ro.deltas(st))


@pytest.mark.parametrize("case", [c for c in CASES if not c.refusal and eo.current_epoch(c.st) > 0 and len(c.st.validators)],
                         ids=lambda c: c.name)
def test_applied_deltas_are_process_epochs(engine, case):
    """Applying the deltas on the host, pair by pair with saturation, gives the balances process_epoch's
    rewards_and_penalties leaves on the device."""
    dev = upload(case.st)
    d = epoch.deltas(dev)
    epoch.process_epoch(dev, "rewards_and_penalties")
    assert np.array_equal(ro.apply(case.st.balances, d), balances(dev, case.st))
    dev.close()


def test_interleaving(engine):
    st = ec.base(256, 7, "minimal", seed=163, keys=True)
    st.validators["effective_balance"][::11] = 16 * ec.ETH
    st.fixed["finalized_checkpoint"] = ec._cp(1, b"f")
    dev = upload(st)
    reg = crypto.Registry.from_state(dev)
    assert np.array_equal(epoch.deltas(dev), ro.deltas(st))
    post, code = eo.process_epoch(st)
    assert code == 0
    epoch.process_epoch(dev)
    assert np.array_equal(epoch.deltas(dev), ro.deltas(post))     # scores, flags and checkpoints of the new epoch
    for e in (8, 9):
        assert duties.proposer_indices(dev, e).tolist() == do.proposer_indices(post, e), e
    duties.attester_duties(dev, 8)
    keys = ec.valid_pubkeys(260)[256:]
    recs = np.zeros(4, dtype=S.VALIDATOR_DTYPE)
    recs["public_key"] = keys.view("V48").reshape(4)
    recs["effective_balance"] = 32 * ec.ETH
    recs["activation_eligibility_epoch"] = recs["activation_epoch"] = 0
    recs["exit_epoch"] = recs["withdrawable_epoch"] = ec.FAR
    dev.add_validators(recs, np.full(4, 32 * ec.ETH, np.uint64))
    post.add_validators(recs, np.full(4, 32 * ec.ETH, np.uint64))
    reg.sync(dev)
    group = np.array([0, 257], np.uint32)
    agg, codes = reg.aggregate_public_keys(group, np.array([0, 2], np.uint32))
    want_code, want = bo.eth_aggregate_public_keys([post.validators["public_key"][i].tobytes() for i in group])
    assert codes.tolist() == [want_code] and agg[0].tobytes() == want
    got = epoch.deltas(dev)
    assert got.shape == (4, 2, 260)
    assert np.array_equal(got, ro.deltas(post))                   # the appended validators are eligible
    assert dev.read_bytes(0, dev.serialized_len()) == S.serialize(post).tobytes()
    post2, code = eo.process_epoch(post)
    epoch.process_epoch(dev)
    assert dev.read_bytes(0, dev.serialized_len()) == S.serialize(post2).tobytes()
    assert np.array_equal(epoch.deltas(dev), ro.deltas(post2))


def test_launch_count(engine):
    L = _lib.lib()
    dev = upload(ec.base(3000, 1000, seed=164))
    c0 = L.b200_launch_count()
    epoch.deltas(dev)
    assert L.b200_launch_count() - c0 == 3   # k_epoch_totals, k_epoch_reduce, k_epoch_deltas
    assert L.b200_last_kernel_ms() > 0
    empty = upload(ec.base(0, 1000, seed=165))
    c0 = L.b200_launch_count()
    got = epoch.deltas(empty)
    assert got.shape == (4, 2, 0)
    assert L.b200_launch_count() - c0 == 0
    assert L.b200_last_kernel_ms() == 0
    assert L.b200_state_epoch_deltas(empty._h, None, 0) == _lib.SUCCESS
