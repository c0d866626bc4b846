"""process_epoch on the device-resident state (ethereum_consensus_b200.epoch) against the oracle (oracle/epoch_oracle.py):
every seeded case with all sub-steps and with each one alone, byte for byte and root for root; a walk of consecutive epochs
across every period boundary; a 2^20-validator state; refusals; interleaving with the duty, shuffling and registry calls;
read-back after every kind of update; the pinned launch count."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from ethereum_consensus_b200 import _lib, crypto, duties, epoch, shuffling, ssz
from ethereum_consensus_b200 import state as S
from oracle import bls_oracle as bo
from oracle import duties_oracle as do
from oracle import epoch_oracle as eo
from oracle import shuffle_oracle as sh
from tests import epoch_cases as ec

pytestmark = pytest.mark.gpu
CASES = ec.cases()
MASKS = [("all", eo.ALL)] + list(eo.STEP.items())


def upload(st):
    return ssz.DeviceBeaconState(S.serialize(st), st.preset)


def c_root(orc, st) -> bytes:
    b = S.serialize(st)
    out = C.create_string_buffer(32)
    assert orc.orc_htr_beacon_state_deneb(b.ctypes.data, b.size, _lib.PRESET[st.preset], 8, out) == 0
    return out.raw


def check_device(dev, want_st, orc):
    want = S.serialize(want_st).tobytes()
    assert dev.serialized_len() == len(want)
    got = dev.read_bytes(0, len(want))
    if got != want:
        lay = S.layout(want_st)
        bad = [k for k, (o, n) in lay.items() if got[o:o + n] != want[o:o + n]]
        raise AssertionError(f"fields differ: {bad}")
    root = c_root(orc, want_st)
    assert dev.hash_tree_root_incremental() == root
    assert dev.hash_tree_root() == root


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_case_matches_oracle(engine, oracle_ssz_c, case):
    for name, m in MASKS:
        dev = upload(case.st)
        before = dev.read_bytes(0, dev.serialized_len())
        root0 = dev.hash_tree_root()
        try:
            want, code = eo.process_epoch(case.st, m)
        except eo.Refused as r:
            with pytest.raises(_lib.EngineError) as ei:
                epoch.process_epoch(dev, m)
            assert ei.value.code == {"bad_arg": _lib.ERR_BAD_ARG, "limit": _lib.ERR_LIMIT}[r.kind], name
            assert dev.read_bytes(0, len(before)) == before
            assert dev.hash_tree_root_incremental() == root0 == dev.hash_tree_root()
            dev.close()
            continue
        if code:
            with pytest.raises(crypto.BLSTError) as ei:
                epoch.process_epoch(dev, m)
            assert ei.value.code == code
        else:
            epoch.process_epoch(dev, m)
        check_device(dev, want, oracle_ssz_c)
        dev.close()


def test_walk_minimal(engine, oracle_ssz_c):
    """26 consecutive epochs (40 .. 65) of a minimal-preset state with valid keys: eth1 voting, historical root, sync
    committee periods and the randao wrap all crossed; flags written and the slot advanced between epochs."""
    rng = np.random.default_rng(77)
    st = ec.base(64, 40, "minimal", seed=77, keys=True)
    st.validators["effective_balance"][::9] = 17 * ec.ETH
    st.balances[::9] = 16_900_000_000
    dev = upload(st)
    lay = S.layout(st)
    n = len(st.validators)
    for cur in range(40, 66):
        if cur > 40:
            flags = rng.integers(0, 8, n, dtype=np.uint8)
            flags[rng.random(n) < 0.1] = 0
            idx = np.arange(n, dtype=np.uint64)
            dev.update_elements("current_epoch_participation", idx, flags)
            st.current_epoch_participation = flags.copy()
            slot = (cur * 8 + 7).to_bytes(8, "little")
            dev.update_bytes(lay["slot"][0], slot)
            st.fixed["slot"] = slot
        st, code = eo.process_epoch(st, eo.ALL)
        assert code == 0
        epoch.process_epoch(dev, eo.ALL)
        assert dev.hash_tree_root_incremental() == c_root(oracle_ssz_c, st), cur
        assert dev.read_bytes(0, dev.serialized_len()) == S.serialize(st).tobytes(), cur
    assert dev.hash_tree_root() == c_root(oracle_ssz_c, st)


def big_state(n=1 << 20):
    rng = np.random.default_rng(2020)
    st = ec.base(n, 1000, seed=2020)
    v = st.validators
    v["slashed"][rng.random(n) < 0.002] = 1
    hit = rng.random(n) < 0.001
    v["withdrawable_epoch"][hit] = 1000 + 4096
    v["slashed"][hit] = 1
    v["effective_balance"][rng.random(n) < 0.01] = 16 * ec.ETH
    exited = rng.random(n) < 0.01
    v["exit_epoch"][exited] = rng.integers(900, 1010, exited.sum(), dtype=np.uint64)
    pend = rng.random(n) < 0.002
    v["activation_epoch"][pend] = ec.FAR
    v["activation_eligibility_epoch"][pend] = rng.integers(980, 999, pend.sum(), dtype=np.uint64)
    st.balances[rng.random(n) < 0.05] = 33_400_000_000
    st.inactivity_scores[rng.random(n) < 0.05] = 5000
    st.slashings[5] = 400 * ec.ETH
    st.fixed["finalized_checkpoint"] = ec._cp(997, b"f")
    return st


def test_two_pow_20(engine, oracle_ssz_c):
    st = big_state()
    dev = upload(st)
    want, code = eo.process_epoch(st, eo.ALL)
    assert code == 0
    epoch.process_epoch(dev, eo.ALL)
    lay = S.layout(want)
    for f in ("validators", "balances", "inactivity_scores", "previous_epoch_participation", "current_epoch_participation"):
        o, ln = lay[f]
        assert dev.read_bytes(o, ln) == getattr(want, f).tobytes(), f
    root = c_root(oracle_ssz_c, want)
    assert dev.hash_tree_root_incremental() == root
    assert dev.hash_tree_root() == root
    assert dev.read_bytes(0, dev.serialized_len()) == S.serialize(want).tobytes()


def test_refusals_leave_state(engine):
    L = _lib.lib()
    code = C.c_int32(0)
    st = ec.base(100, 1000, seed=90)
    dev = upload(st)
    before, root = dev.read_bytes(0, dev.serialized_len()), dev.hash_tree_root()
    assert L.b200_state_process_epoch(None, eo.ALL, C.byref(code)) == _lib.ERR_BAD_ARG
    for m in (1 << 12, 1 << 31, 0xffffffff):
        assert L.b200_state_process_epoch(dev._h, m, C.byref(code)) == _lib.ERR_BAD_ARG
    assert L.b200_state_process_epoch(dev._h, eo.ALL, None) == _lib.ERR_BAD_ARG
    out = np.zeros(16, np.uint8)
    n = dev.serialized_len()
    assert L.b200_state_read_bytes(dev._h, n - 8, _lib.ptr(out), 16) == _lib.ERR_BAD_ARG
    assert L.b200_state_read_bytes(dev._h, n + 1, _lib.ptr(out), 0) == _lib.ERR_BAD_ARG
    assert L.b200_state_read_bytes(None, 0, _lib.ptr(out), 16) == _lib.ERR_BAD_ARG
    assert dev.read_bytes(n, 0) == b""
    assert dev.read_bytes(0, n) == before
    assert dev.hash_tree_root_incremental() == root == dev.hash_tree_root()
    # lists of different lengths
    odd = ec.base(100, 1000, seed=91)
    odd.inactivity_scores = odd.inactivity_scores[:99].copy()
    dev_odd = upload(odd)
    r_odd = dev_odd.hash_tree_root()
    assert L.b200_state_process_epoch(dev_odd._h, eo.ALL, C.byref(code)) == _lib.ERR_BAD_ARG
    assert dev_odd.hash_tree_root_incremental() == r_odd
    # a sharded handle (world 1)
    from ethereum_consensus_b200 import parallel
    parallel.comm_init(0, 1)
    shd = ssz.DeviceBeaconState(S.serialize(st), "mainnet", sharded=True)
    assert L.b200_state_process_epoch(shd._h, eo.ALL, C.byref(code)) == _lib.ERR_BAD_ARG
    assert L.b200_state_read_bytes(shd._h, 0, _lib.ptr(out), 16) == _lib.ERR_BAD_ARG
    assert shd.hash_tree_root() == root
    # and the handle still processes its epoch
    epoch.process_epoch(dev, eo.ALL)
    assert dev.read_bytes(0, n) == S.serialize(eo.process_epoch(st)[0]).tobytes()


def test_interleaving(engine):
    st = ec.base(256, 7, "minimal", seed=95, keys=True)
    st.validators["effective_balance"][::11] = 16 * ec.ETH
    dev = upload(st)
    reg = crypto.Registry.from_state(dev)
    post, code = eo.process_epoch(st)
    assert code == 0
    epoch.process_epoch(dev)
    for e in (8, 9):
        assert duties.proposer_indices(dev, e).tolist() == do.proposer_indices(post, e), e
        seed = duties.get_seed(dev, e, duties.DOMAIN_BEACON_ATTESTER)
        active = do.active_indices(post, e)
        assert shuffling.state_shuffled_active_indices(dev, e, seed, 10).tolist() == \
            sh.shuffled_indices_numpy(active, seed, 10).tolist()
    # new deposits after the epoch: the registry follows the resident state
    keys = ec.valid_pubkeys(260)[256:]
    recs = np.zeros(4, dtype=S.VALIDATOR_DTYPE)
    recs["public_key"] = keys.view("V48").reshape(4)
    recs["activation_eligibility_epoch"] = recs["activation_epoch"] = recs["exit_epoch"] = recs["withdrawable_epoch"] = ec.FAR
    dev.add_validators(recs, np.full(4, 32 * ec.ETH, np.uint64))
    post.add_validators(recs, np.full(4, 32 * ec.ETH, np.uint64))
    reg.sync(dev)
    assert reg.n == 260
    group = np.array([0, 5, 257, 259], np.uint32)
    agg, codes = reg.aggregate_public_keys(group, np.array([0, 4], np.uint32))
    want_code, want = bo.eth_aggregate_public_keys([post.validators["public_key"][i].tobytes() for i in group])
    assert codes.tolist() == [want_code] and agg[0].tobytes() == want
    # and the next epoch runs on the grown state
    post2, code = eo.process_epoch(post)
    epoch.process_epoch(dev)
    assert dev.read_bytes(0, dev.serialized_len()) == S.serialize(post2).tobytes()


def test_read_bytes_round_trips(engine):
    st = ec.base(300, 1000, seed=96)
    dev = upload(st)
    assert dev.read_bytes(0, dev.serialized_len()) == S.serialize(st).tobytes()
    rng = np.random.default_rng(96)
    idx = np.array([0, 7, 299], np.uint64)
    bal = np.array([1, 2, 3], "<u8")
    dev.update_elements("balances", idx, bal)
    st.balances[idx] = bal
    recs = st.validators[[1, 2]].copy()
    recs["effective_balance"] = 31 * ec.ETH
    dev.update_elements("validators", np.array([1, 2], np.uint64), recs.tobytes())
    st.validators[[1, 2]] = recs
    lay = S.layout(st)
    mix = rng.integers(0, 256, 32, dtype=np.uint8)
    dev.update_bytes(lay["randao_mixes"][0] + 32 * 5, mix.tobytes())
    st.randao_mixes[5] = mix
    assert dev.read_bytes(0, dev.serialized_len()) == S.serialize(st).tobytes()
    new = st.validators[:3].copy()
    dev.add_validators(new, np.full(3, 5, np.uint64))
    st.add_validators(new, np.full(3, 5, np.uint64))
    dev.set_field("eth1_data_votes", b"")
    st.set_field("eth1_data_votes", b"")
    hdr = bytearray(st.payload_header())[:584] + b"xyz"
    dev.set_field("latest_execution_payload_header", bytes(hdr))
    st.set_field("latest_execution_payload_header", bytes(hdr))
    dev.append_elements("historical_summaries", bytes(range(64)))
    st.append_elements("historical_summaries", bytes(range(64)))
    assert dev.serialize().tobytes() == S.serialize(st).tobytes()
    lay = S.layout(st)
    o, ln = lay["balances"]
    assert dev.read_bytes(o - 3, 20) == S.serialize(st).tobytes()[o - 3:o + 17]   # across a field boundary


def test_launch_count(engine):
    L = _lib.lib()
    dev = upload(ec.base(3000, 1000, seed=97))
    c0 = L.b200_launch_count()
    epoch.process_epoch(dev, eo.ALL)
    # k_epoch_totals, k_epoch_reduce, k_epoch_apply, k_activation_select; the rotation is a copy and a memset
    assert L.b200_launch_count() - c0 == 4
    assert L.b200_last_kernel_ms() > 0
    c0 = L.b200_launch_count()
    epoch.process_epoch(dev, "randao_mixes_reset")
    assert L.b200_launch_count() - c0 == 2
