"""Beacon committees on the device (ethereum_consensus_b200.duties: committee_count_per_slot, beacon_committees,
attester_duties, attesting_indices) against the oracle (tests/committee_oracle.py): every seeded case value for value, a
2^20-validator state against numpy slices of the shuffled active list, the per-handle committee cache across every write
that changes what it holds, a block of 128 attestations x 512 signers through registry-mode verification, and refusals."""
from __future__ import annotations

import ctypes as C
import hashlib

import numpy as np
import pytest

from ethereum_consensus_b200 import _lib, block, crypto, duties, epoch, shuffling, ssz
from ethereum_consensus_b200 import state as S
from oracle import duties_oracle as do
from tests import committee_cases as cc
from tests import committee_oracle as co

pytestmark = pytest.mark.gpu
R_ORDER = 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001
SK0, DELTA = 0x1234567 % R_ORDER, 0x89abcdef12345 % R_ORDER   # key i = (SK0 + DELTA * i) G1
E = cc.EPOCH


def upload(st):
    return ssz.DeviceBeaconState(S.serialize(st), st.preset)


def fresh(dev):
    """A new handle of the same bytes as `dev` holds now."""
    return ssz.DeviceBeaconState(dev.serialize(), dev.preset)


def committees_equal(dev, st, e, want=None):
    idx, off, cps = duties.beacon_committees(dev, e)
    want = want if want is not None else co.beacon_committees(st, e)
    assert cps == len(want) // co.spe(st)
    assert [idx[off[k]:off[k + 1]].tolist() for k in range(len(off) - 1)] == want


def answers(dev, epochs):
    """Everything the committee calls say about `epochs` (all validators' duties included)."""
    out = []
    for e in epochs:
        idx, off, cps = duties.beacon_committees(dev, e)
        out.append((duties.committee_count_per_slot(dev, e), idx.tolist(), off.tolist(), cps,
                    duties.attester_duties(dev, e).tobytes()))
    return out


@pytest.mark.parametrize("case", cc.cases(), ids=lambda c: c.name)
def test_case_matches_oracle(engine, case):
    st = case.st
    dev = upload(st)
    for e in case.cps:
        assert duties.committee_count_per_slot(dev, e) == co.committee_count_per_slot(st, e) == case.cps[e]
        want = co.beacon_committees(st, e)
        committees_equal(dev, st, e, want)
        rows = duties.attester_duties(dev, e)
        wrows = co.duty_rows(st, e, range(len(st.validators)))
        assert rows.view(np.uint64).reshape(-1, 5).tolist() == wrows.tolist(), e
        some = np.array([len(st.validators) - 1, 0, 0, len(st.validators) // 2], np.uint64)
        assert duties.attester_duties(dev, e, some).view(np.uint64).reshape(-1, 5).tolist() == wrows[some.astype(np.int64)].tolist()
    got, codes = duties.attesting_indices(dev, [(d, b) for d, b, _ in case.attestations])
    cache = {}
    for (d, b, want_code), g, c in zip(case.attestations, got, codes):
        w_code, w_idx = co.attesting_indices(st, d, b, committees=cache)
        assert (int(c), g.tolist()) == (w_code, w_idx) and w_code == want_code


@pytest.fixture(scope="module")
def big():
    n = 1 << 20
    st = cc.state(n, "mainnet", seed=31, edges=False)
    st.validators["exit_epoch"][np.random.default_rng(31).integers(0, 100, n) == 0] = 10   # ~1 % exited
    return st


def test_big_state(engine, big):
    st = big
    dev = upload(st)
    n_all = len(st.validators)
    for e in (E, E + 1):
        seed = duties.get_seed(dev, e, duties.DOMAIN_BEACON_ATTESTER)
        shuffled = shuffling.state_shuffled_active_indices(dev, e, seed)
        n = shuffled.size
        idx, off, cps = duties.beacon_committees(dev, e)
        assert cps == 64 and off.size == 2049 and np.array_equal(idx, shuffled)
        assert off.tolist() == [n * k // 2048 for k in range(2049)]
        # the numpy inverse: committee by committee, no closed form
        want = np.full((n_all, 5), co.NOT_ACTIVE, np.uint64)
        for k in range(2048):
            m = shuffled[off[k]:off[k + 1]]
            want[m.astype(np.int64)] = np.stack([np.full(m.size, e * 32 + k // 64), np.full(m.size, k % 64), np.full(m.size, m.size),
                                                 np.full(m.size, 64), np.arange(m.size)], 1).astype(np.uint64)
        assert np.array_equal(duties.attester_duties(dev, e).view(np.uint64).reshape(-1, 5), want), e
        # one committee through the oracle's per-member formulation
        assert duties.beacon_committee(dev, e * 32 + 31, 63).tolist() == co.beacon_committee(st, e * 32 + 31, 63, "index")


def test_cache_follows_the_state(engine):
    L = _lib.lib()
    st = cc.state(5000, "mainnet", seed=41, edges=False)
    v = st.validators
    v["effective_balance"][7] = 16 * cc.ETH      # ejected by the registry updates below
    dev = upload(st)
    epochs = (E - 1, E, E + 1)
    first = answers(dev, epochs)
    assert first == answers(fresh(dev), epochs)

    def counted(fn):
        c0 = L.b200_launch_count()
        r = fn()
        return r, L.b200_launch_count() - c0
    # a cached epoch: no shuffle, no active-set scan; duties with the inverse map built: the row kernel alone
    (_, k1) = counted(lambda: duties.beacon_committees(dev, E))
    (_, k2) = counted(lambda: duties.committee_count_per_slot(dev, E))
    (_, k3) = counted(lambda: duties.attester_duties(dev, E))
    assert (k1, k2, k3) == (0, 0, 1)
    assert answers(dev, epochs) == first

    lay = S.layout(st)
    vo = lay["validators"][0]
    # (1) a validator's exit epoch, by update_elements: validator 11 leaves at E
    r = bytearray(dev.read_bytes(vo + 121 * 11, 121))
    exit_at = 48 + 32 + 8 + 1 + 8 + 8   # pubkey, withdrawal_credentials, effective_balance, slashed, eligibility, activation
    r[exit_at:exit_at + 8] = E.to_bytes(8, "little")
    dev.update_elements("validators", [11], bytes(r))
    after = answers(dev, epochs)
    assert after == answers(fresh(dev), epochs) and after != first
    assert all(11 not in a[1] for a in after[1:])
    # (2) new validators (a deposit batch), active from epoch 0
    recs = bytearray(dev.read_bytes(vo, 121 * 40))
    for j in range(40):
        recs[121 * j:121 * j + 48] = hashlib.sha256(b"new%d" % j).digest() + bytes(16)
    dev.add_validators(bytes(recs), np.full(40, 32 * cc.ETH, np.uint64))
    after2 = answers(dev, epochs)
    assert after2 == answers(fresh(dev), epochs) and after2 != after
    # (3) a process_epoch that ejects validator 7 (its record changes; the active sets of these epochs do not)
    before_epoch = dev.read_bytes(vo + 121 * 7, 121)
    epoch.process_epoch(dev, ["registry_updates"])
    assert dev.read_bytes(vo + 121 * 7, 121) != before_epoch
    _, k = counted(lambda: duties.beacon_committees(dev, E))
    assert k > 0   # rebuilt, not served from the cache
    after3 = answers(dev, epochs)
    assert after3 == answers(fresh(dev), epochs)
    # (4) a randao mix: the seed of E + 1 reads mix (E + 1 + EPHV - 2) mod EPHV
    mixes = lay["randao_mixes"][0]
    m = (E + 1 + 65536 - 2) % 65536
    dev.update_bytes(mixes + 32 * m, hashlib.sha256(b"mix").digest())
    after4 = answers(dev, epochs)
    assert after4 == answers(fresh(dev), epochs)
    assert after4[:2] == after3[:2] and after4[2][1] != after3[2][1]


class _Keys:
    """validator_pubkeys of a state whose validator i holds tiled key i mod nd."""

    def __init__(self, keys, n):
        self.keys, self.n = keys, n

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        return self.keys[int(i) % len(self.keys)].tobytes()


def test_block_of_attestations(engine, oracle_bls_c):
    """128 attestations x 512 signers: attesting_indices, then registry-mode verification, against the strict path and
    the C oracle; one attestation signed without one of its signers, one signed over another message."""
    n, nd = 1 << 20, 1 << 15
    st = cc.state(n, "mainnet", seed=51, edges=False)   # 2^20 active: 2048 committees of exactly 512
    keys = np.empty((nd, 48), dtype=np.uint8)
    oracle_bls_c.orc_pk_sequence(SK0.to_bytes(32, "big"), DELTA.to_bytes(32, "big"), nd, keys.ctypes.data)
    st.validators["public_key"] = keys[np.arange(n) % nd].view("V48").reshape(n)
    dev = upload(st)
    slot = do.slot(st)
    rng = np.random.default_rng(51)
    atts, msgs, sigs, signers = [], [], [], []
    ks = rng.choice([k for k in range(2048) if (E - 1) * 32 + k // 64 + 1 <= slot], 128, replace=False)
    for a, k in enumerate(ks):
        s = (E - 1) * 32 + k // 64
        data = co.attestation_data(s, k % 64, E - 1, root=hashlib.sha256(b"root%d" % a).digest())
        committee = duties.beacon_committee(dev, s, k % 64)
        assert committee.size == 512
        bits = [True] * 512 if a % 2 == 0 else list(rng.random(512) < 0.9)
        sel = sorted(int(committee[i]) for i in range(512) if bits[i])
        msg = hashlib.sha256(data).digest()
        signed = sel[1:] if a == 5 else sel
        sk = sum(SK0 + DELTA * (i % nd) for i in signed) % R_ORDER
        sig = C.create_string_buffer(96)
        oracle_bls_c.orc_sign(sk.to_bytes(32, "big"), hashlib.sha256(b"other").digest() if a == 9 else msg, 32, sig)
        atts.append((data, co.bitlist(bits)))
        msgs.append(msg)
        sigs.append(sig.raw)
        signers.append(sel)
    got, codes = duties.attesting_indices(dev, atts)
    assert codes.tolist() == [0] * 128
    assert [g.tolist() for g in got] == signers
    pk = _Keys(keys, n)
    ss = block.SignatureSet()
    for g, m, s in zip(got, msgs, sigs):
        ss.add_indexed_attestation("attestation", pk, g.tolist(), m, s)
    reg = crypto.Registry.from_state(dev)
    want = [5 if a in (5, 9) else 0 for a in range(128)]
    assert ss.verify(registry=reg).tolist() == ss.verify().tolist() == want
    # the C oracle on the same tuples
    flat = np.concatenate([keys[np.asarray(g, np.int64) % nd].reshape(-1) for g in got])
    off = np.cumsum([0] + [len(g) for g in got]).astype(np.uint32)
    ms = np.frombuffer(b"".join(msgs), np.uint8).copy()
    sg = np.frombuffer(b"".join(sigs), np.uint8).copy()
    out = np.empty(128, np.int32)
    oracle_bls_c.orc_fast_aggregate_verify_batch(flat.ctypes.data, off.ctypes.data, ms.ctypes.data, sg.ctypes.data, 128,
                                                 out.ctypes.data, 8)
    assert out.tolist() == want
    # the indices straight into the registry batch
    idx = np.concatenate([g for g in got]).astype(np.uint32)
    assert reg.verify_batch(idx, off, ms, sg).tolist() == want


def test_refusals_leave_handle(engine):
    L = _lib.lib()
    st = cc.state(3000, "mainnet", seed=61, edges=False)
    dev = upload(st)
    epochs = (E - 1, E, E + 1)
    before = answers(dev, epochs)
    blob = dev.serialize().tobytes()
    cps, n_out = C.c_uint64(0), C.c_size_t(0)
    idx = np.zeros(4000, np.uint64)
    off = np.zeros(2049, np.uint32)
    rows = np.zeros(5 * 4000, np.uint64)
    codes = np.zeros(4, np.int32)
    data = np.zeros(4 * 128, np.uint8)
    bits = np.ones(16, np.uint8)
    boff = np.array([0, 4, 8, 12, 16], np.uint32)
    oidx, ooff = np.zeros(64, np.uint64), np.zeros(5, np.uint32)
    BAD = _lib.ERR_BAD_ARG
    P = _lib.ptr

    def all_calls(h):
        return [L.b200_state_committee_count_per_slot(h, E, C.byref(cps)),
                L.b200_state_beacon_committees(h, E, P(idx), P(off), C.byref(cps), C.byref(n_out)),
                L.b200_state_attester_duties(h, E, None, 3000, P(rows)),
                L.b200_state_attesting_indices(h, 4, P(data), P(bits), P(boff), P(oidx), P(ooff), P(codes))]
    assert all_calls(None) == [BAD] * 4
    # NULL outputs; NULL validators with n != N; an index past the registry; an epoch after the next; epoch * 32 overflow
    assert L.b200_state_committee_count_per_slot(dev._h, E, None) == BAD
    assert L.b200_state_beacon_committees(dev._h, E, None, P(off), C.byref(cps), C.byref(n_out)) == BAD
    assert L.b200_state_attester_duties(dev._h, E, None, 2999, P(rows)) == BAD
    three = np.array([0, 3000, 1], np.uint64)
    assert L.b200_state_attester_duties(dev._h, E, P(three), 3, P(rows)) == BAD
    assert L.b200_state_attester_duties(dev._h, E + 2, None, 3000, P(rows)) == BAD
    assert L.b200_state_attester_duties(dev._h, E, None, 3000, None) == BAD
    # attesting_indices: offsets not starting at 0 / decreasing, NULL buffers, more than 2^20 attestations
    assert L.b200_state_attesting_indices(dev._h, 4, P(data), P(bits), P(np.array([1, 4, 8, 12, 16], np.uint32)), P(oidx), P(ooff), P(codes)) == BAD
    assert L.b200_state_attesting_indices(dev._h, 4, P(data), P(bits), P(np.array([0, 8, 4, 12, 16], np.uint32)), P(oidx), P(ooff), P(codes)) == BAD
    assert L.b200_state_attesting_indices(dev._h, 4, None, P(bits), P(boff), P(oidx), P(ooff), P(codes)) == BAD
    assert L.b200_state_attesting_indices(dev._h, 4, P(data), None, P(boff), P(oidx), P(ooff), P(codes)) == BAD
    assert L.b200_state_attesting_indices(dev._h, 4, P(data), P(bits), P(boff), None, P(ooff), P(codes)) == BAD
    assert L.b200_state_attesting_indices(dev._h, 4, P(data), P(bits), P(boff), P(oidx), P(ooff), None) == BAD
    assert L.b200_state_attesting_indices(dev._h, (1 << 20) + 1, P(data), P(bits), P(boff), P(oidx), P(ooff), P(codes)) == BAD
    # no active validator: committees refused; count 1, every duty row NOT_ACTIVE, a zero-length Bitlist empty
    st0 = cc.state(50, "mainnet", seed=62, edges=False)
    st0.validators["exit_epoch"] = 0
    none = upload(st0)
    assert L.b200_state_beacon_committees(none._h, E, P(idx), P(off), C.byref(cps), C.byref(n_out)) == BAD
    assert duties.committee_count_per_slot(none, E) == 1
    assert (duties.attester_duties(none, E).view(np.uint64) == co.NOT_ACTIVE).all()
    got, c = duties.attesting_indices(none, [(co.attestation_data(E * 32, 0, E), co.bitlist([]))])
    assert c.tolist() == [co.INDICES_EMPTY] and got[0].size == 0
    # the handle: byte for byte as it was, and the same answers
    assert dev.serialize().tobytes() == blob
    assert answers(dev, epochs) == before
    got, c = duties.attesting_indices(dev, [])
    assert got == [] and c.size == 0
    # a sharded handle (world 1)
    from ethereum_consensus_b200 import parallel
    parallel.comm_init(0, 1)
    sh = ssz.DeviceBeaconState(S.serialize(st), "mainnet", sharded=True)
    assert all_calls(sh._h) == [BAD] * 4
