"""Proposer and sync-committee duties on the device (ethereum_consensus_b200.duties) against the oracle
(oracle/duties_oracle.py): every seeded case index for index, a 2^20-validator state with valid tiled keys, the
committee rotation with both roots, registry-mode sync aggregates, refusals, interleaving and pinned launch counts."""
from __future__ import annotations

import ctypes as C
import hashlib

import numpy as np
import pytest

from ethereum_consensus_b200 import _lib, crypto, duties, shuffling, ssz
from ethereum_consensus_b200 import state as S
from oracle import bls_oracle as bo
from oracle import duties_oracle as do
from tests import duties_cases as dc

pytestmark = pytest.mark.gpu
R_ORDER = 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001
SK0, DELTA = 0x1234567 % R_ORDER, 0x89abcdef12345 % R_ORDER   # key i = (SK0 + DELTA * i) G1


def upload(st):
    return ssz.DeviceBeaconState(S.serialize(st), st.preset)


def valid_keys(orc, n):
    out = np.empty((n, 48), dtype=np.uint8)
    orc.orc_pk_sequence(SK0.to_bytes(32, "big"), DELTA.to_bytes(32, "big"), n, out.ctypes.data)
    return out


def c_aggregate(orc):
    def agg(keys):
        if not keys:
            return bo.EMPTY_AGGREGATE, None
        out = C.create_string_buffer(48)
        code = orc.orc_eth_aggregate_public_keys(b"".join(keys), len(keys), out)
        return code, (out.raw if code == 0 else None)
    return agg


@pytest.mark.parametrize("case", dc.cases(), ids=lambda c: c.name)
def test_case_matches_oracle(engine, case):
    st = case.st
    dev = upload(st)
    for e in case.epochs + case.seed_epochs:
        for dom in (duties.DOMAIN_BEACON_PROPOSER, duties.DOMAIN_BEACON_ATTESTER, duties.DOMAIN_SYNC_COMMITTEE):
            assert duties.get_seed(dev, e, dom) == do.get_seed(st, e, dom), (e, dom)
    for e in case.epochs:
        assert duties.proposer_indices(dev, e).tolist() == do.proposer_indices(st, e), e
    if case.committee:
        idx, committee, code = duties.next_sync_committee(dev)
        w_idx, w_committee, w_code = do.next_sync_committee(st)
        assert idx.tolist() == w_idx and code == w_code and committee == w_committee
    for which in ("current", "next"):
        got = duties.sync_committee_indices(dev, which, missing_ok=True).tolist()
        assert got == do.sync_committee_indices(st, which), which
    if case.regime == "missing_key":
        with pytest.raises(KeyError):
            duties.sync_committee_indices(dev, "current")


@pytest.fixture(scope="module")
def big(oracle_bls_c):
    """2^20 validators, 2^15 distinct valid keys tiled (validator i holds key i mod 2^15)."""
    n, nd = 1 << 20, 1 << 15
    keys = valid_keys(oracle_bls_c, nd)
    st = dc.base(n, seed=21, slot_epoch=5000)
    st.validators["public_key"] = keys[np.arange(n) % nd].view("V48").reshape(n)
    rng = np.random.default_rng(21)
    st.validators["exit_epoch"][rng.integers(0, 100, n) == 0] = 10   # ~1 % exited
    return st, keys


def test_big_state(engine, oracle_bls_c, big):
    st, keys = big
    nd = len(keys)
    dev = upload(st)
    for e in (5000, 5001, 77777):
        assert duties.proposer_indices(dev, e).tolist() == do.proposer_indices(st, e), e
    idx, committee, code = duties.next_sync_committee(dev)
    w_idx, w_committee, w_code = do.next_sync_committee(st, c_aggregate(oracle_bls_c))
    assert idx.tolist() == w_idx and code == w_code == 0 and committee == w_committee
    members = keys[np.asarray(w_idx) % nd]
    agg, codes = crypto.eth_aggregate_public_keys_batch(members.reshape(-1), np.array([0, 512], np.uint32))
    assert codes.tolist() == [0] and agg[0].tobytes() == committee[-48:]
    # mixed balances
    mixed = dc.base(1 << 20, seed=22, slot_epoch=5000)
    mixed.validators["public_key"] = st.validators["public_key"]
    mixed.validators["effective_balance"] = np.random.default_rng(22).choice(np.array([0, 1, 16, 31, 32], np.uint64) * dc.ETH, 1 << 20)
    dev2 = upload(mixed)
    for e in (5000, 5001):
        assert duties.proposer_indices(dev2, e).tolist() == do.proposer_indices(mixed, e), e
    assert duties.next_sync_committee(dev2)[0].tolist() == do.next_sync_committee_indices(mixed)
    # key lookup on the repeated keys: the largest holder of key k is k + nd * (2^20 / nd - 1)
    blob = members.tobytes() + bytes(48)
    dev.update_bytes(S.layout(st)["current_sync_committee"][0], blob)
    got = duties.sync_committee_indices(dev, "current")
    assert got.tolist() == [int(i) % nd + nd * ((1 << 20) // nd - 1) for i in w_idx]


def test_rotation_roots(engine, oracle_bls_c, oracle_ssz_c):
    def htr(s):
        b = S.serialize(s)
        out = C.create_string_buffer(32)
        assert oracle_ssz_c.orc_htr_beacon_state_deneb(b.ctypes.data, b.size, _lib.PRESET[s.preset], 8, out) == 0
        return out.raw
    for preset in ("mainnet", "minimal"):
        st = dc.rotation_state(300, preset)
        st.validators["public_key"] = valid_keys(oracle_bls_c, 300).view("V48").reshape(300)
        dev = upload(st)
        root0 = dev.hash_tree_root()
        assert root0 == htr(st)
        rotated, code, want = do.process_sync_committee_updates(st, c_aggregate(oracle_bls_c))
        assert rotated and code == 0
        assert duties.process_sync_committee_updates(dev) is True
        assert dev.hash_tree_root_incremental() == htr(want)
        assert dev.hash_tree_root() == htr(want)
        # off a boundary: nothing changes
        off = dc.rotation_state(300, preset, boundary=False)
        dev_off = upload(off)
        r0 = dev_off.hash_tree_root()
        assert duties.process_sync_committee_updates(dev_off) is False
        assert dev_off.hash_tree_root_incremental() == r0 == htr(off)
    # random (invalid) keys: the aggregation's code comes back and the state stays as it was
    bad = dc.rotation_state(300)
    dev_bad = upload(bad)
    r0 = dev_bad.hash_tree_root()
    want_code = do.next_sync_committee(bad)[2]
    assert want_code != 0
    with pytest.raises(crypto.BLSTError) as ei:
        duties.process_sync_committee_updates(dev_bad)
    assert ei.value.code == want_code
    assert dev_bad.hash_tree_root_incremental() == r0 and dev_bad.hash_tree_root() == r0


def test_registry_sync_aggregate(engine, oracle_bls_c):
    from ethereum_consensus_b200 import block, signing
    n = 4096
    st = dc.base(n, seed=24)
    keys = valid_keys(oracle_bls_c, n)
    st.validators["public_key"] = keys.view("V48").reshape(n)
    rng = np.random.default_rng(24)
    members = rng.integers(0, n, 512)
    st = dc.set_committees(st, members, members[::-1])
    dev = upload(st)
    idx = duties.sync_committee_indices(dev, "current")
    assert idx.tolist() == members.tolist()
    reg = crypto.Registry.from_state(dev)
    fork = signing.Fork(b"\x03\0\0\0", b"\x04\0\0\0", 0)
    gvr, root = hashlib.sha256(b"gvr").digest(), hashlib.sha256(b"block").digest()
    slot = do.slot(st)
    committee_keys = [keys[i].tobytes() for i in members]
    for bits_seed, corrupt in ((1, False), (2, True), (3, False)):
        bits = np.random.default_rng(bits_seed).random(512) < 0.9
        sel = [int(members[j]) for j in range(512) if bits[j]]
        sk = sum(SK0 + DELTA * i for i in sel) % R_ORDER
        ss = block.SignatureSet()
        prev = slot - 1
        domain = signing.get_domain(fork, gvr, signing.DomainType.SyncCommittee, signing.compute_epoch_at_slot(prev, 32))
        msg = signing.compute_signing_root(root, domain)
        sig = C.create_string_buffer(96)
        oracle_bls_c.orc_sign((sk if not corrupt else sk + 1).to_bytes(32, "big"), msg, 32, sig)
        ss.add_sync_aggregate(committee_keys, bits.tolist(), sig.raw, slot, root, fork, gvr, committee_indices=idx)
        assert ss.verify(registry=reg).tolist() == ss.verify().tolist() == [5 if corrupt else 0]


def test_refusals_leave_handle(engine):
    L = _lib.lib()
    st = dc.base(500, seed=25)
    dev = upload(st)
    root = dev.hash_tree_root()
    out = np.zeros(512, np.uint64)
    committee = np.zeros(513 * 48, np.uint8)
    code, rot = C.c_int32(0), C.c_int32(0)
    seed = (C.c_uint8 * 32)()
    for h in (None,):
        assert L.b200_state_get_seed(h, 0, bytes(4), seed) == _lib.ERR_BAD_ARG
        assert L.b200_state_proposer_indices(h, 0, _lib.ptr(out)) == _lib.ERR_BAD_ARG
        assert L.b200_state_next_sync_committee(h, _lib.ptr(out), _lib.ptr(committee), C.byref(code)) == _lib.ERR_BAD_ARG
        assert L.b200_state_sync_committee_updates(h, C.byref(rot), C.byref(code)) == _lib.ERR_BAD_ARG
        assert L.b200_state_sync_committee_indices(h, 0, _lib.ptr(out)) == _lib.ERR_BAD_ARG
    # epoch * SLOTS_PER_EPOCH overflows; bad `which`
    assert L.b200_state_proposer_indices(dev._h, (2**64 - 1) // 32 + 1, _lib.ptr(out)) == _lib.ERR_BAD_ARG
    assert L.b200_state_sync_committee_indices(dev._h, 2, _lib.ptr(out)) == _lib.ERR_BAD_ARG
    # no active validator at the epoch
    none = upload(dc.only_active(dc.base(50, seed=26), []))
    r_none = none.hash_tree_root()
    assert L.b200_state_proposer_indices(none._h, 1000, _lib.ptr(out)) == _lib.ERR_BAD_ARG
    assert L.b200_state_next_sync_committee(none._h, _lib.ptr(out), _lib.ptr(committee), C.byref(code)) == _lib.ERR_BAD_ARG
    assert none.hash_tree_root_incremental() == r_none
    assert dev.hash_tree_root_incremental() == root and dev.hash_tree_root() == root
    # after the refusals the handle answers as before
    assert duties.proposer_indices(dev, 1000).tolist() == do.proposer_indices(st, 1000)
    # a sharded handle (world 1)
    from ethereum_consensus_b200 import parallel
    parallel.comm_init(0, 1)
    sh = ssz.DeviceBeaconState(S.serialize(st), "mainnet", sharded=True)
    assert L.b200_state_get_seed(sh._h, 0, bytes(4), seed) == _lib.ERR_BAD_ARG
    assert L.b200_state_proposer_indices(sh._h, 1000, _lib.ptr(out)) == _lib.ERR_BAD_ARG
    assert L.b200_state_next_sync_committee(sh._h, _lib.ptr(out), _lib.ptr(committee), C.byref(code)) == _lib.ERR_BAD_ARG
    assert L.b200_state_sync_committee_updates(sh._h, C.byref(rot), C.byref(code)) == _lib.ERR_BAD_ARG
    assert L.b200_state_sync_committee_indices(sh._h, 0, _lib.ptr(out)) == _lib.ERR_BAD_ARG
    assert sh.hash_tree_root() == root


def test_interleaving_and_launch_counts(engine, oracle_bls_c):
    L = _lib.lib()
    n = 3000
    st = dc.base(n, seed=27)
    st.validators["public_key"] = valid_keys(oracle_bls_c, n).view("V48").reshape(n)
    dev = upload(st)
    want_p = do.proposer_indices(st, 1000)
    want_c = do.next_sync_committee(st, c_aggregate(oracle_bls_c))
    want_i = do.sync_committee_indices(st, "current")
    seed = duties.get_seed(dev, 1000, duties.DOMAIN_BEACON_ATTESTER)
    want_shuf = shuffling.state_shuffled_active_indices(dev, 1000, seed).tolist()

    def counted(fn):
        c0 = L.b200_launch_count()
        r = fn()
        return r, L.b200_launch_count() - c0
    # all 32 ETH: 3 active-index launches + the proposer sampler; + one window and its selection + gather, K1,
    # aggregate, compress; one matcher launch
    p, k = counted(lambda: duties.proposer_indices(dev, 1000))
    assert p.tolist() == want_p and k == 4
    c, k = counted(lambda: duties.next_sync_committee(dev))
    assert (c[0].tolist(), c[1], c[2]) == want_c and k == 9
    i, k = counted(lambda: duties.sync_committee_indices(dev, "current", missing_ok=True))
    assert i.tolist() == want_i and k == 1
    reg = crypto.Registry.from_state(dev)
    fav = lambda: crypto.fast_aggregate_verify_batch(  # noqa: E731
        np.frombuffer(want_c[1][:96], np.uint8), np.array([0, 2], np.uint32), np.zeros(32, np.uint8), np.zeros(96, np.uint8)).tolist()
    want_fav = fav()
    for _ in range(2):
        assert shuffling.state_shuffled_active_indices(dev, 1000, seed).tolist() == want_shuf
        assert duties.proposer_indices(dev, 1000).tolist() == want_p
        agg, codes = reg.aggregate_public_keys(np.asarray(want_c[0], np.uint32), np.array([0, 512], np.uint32))
        assert codes.tolist() == [0] and agg[0].tobytes() == want_c[1][-48:]
        c = duties.next_sync_committee(dev)
        assert (c[0].tolist(), c[1], c[2]) == want_c
        assert fav() == want_fav
        assert duties.sync_committee_indices(dev, "current", missing_ok=True).tolist() == want_i
    # several windows: all 1 ETH draws windows of 512, 1024, 2048, ... candidates, two launches each
    one = upload(dc.base(3000, seed=5, eff=1 * dc.ETH))
    drawn = do.candidates_drawn(dc.base(3000, seed=5, eff=1 * dc.ETH))
    windows, total = 0, 0
    while total < drawn:
        total += 512 << windows
        windows += 1
    _, k = counted(lambda: duties.next_sync_committee(one))
    assert k == 3 + 2 * windows + 4
