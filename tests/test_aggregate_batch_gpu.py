"""GPU: aggregate / eth_aggregate_public_keys over T groups per call (tests/aggregate_batch_cases.py).  For every group the
batch call, the single call and the C oracle agree byte for byte (the oracle on every group at small scale, on a seeded
subsample at full scale); the registry path equals the strict path on the same key bytes however the registry was built;
the aggregates of a slot verify against their committees; one engine interleaves batch aggregation with the verify
batches without either seeing the other's buffers; malformed calls are refused and leave the registry as it was."""
from __future__ import annotations

import ctypes as C
import random

import numpy as np
import pytest

from tests import aggregate_batch_cases as ac
from tests import torsion_cases as tc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torsion():
    return tc.g1_cases(), tc.g2_cases()


@pytest.fixture(scope="module")
def slot():
    return ac.slot()


def _arr(items, width):
    return np.frombuffer(b"".join(items), dtype=np.uint8).copy() if items else np.zeros(0, dtype=np.uint8)


def _single(fn, items, width):
    from ethereum_consensus_b200 import _lib
    out = (C.c_uint8 * width)()
    flat = b"".join(items)
    code = getattr(_lib.lib(), fn)(flat if flat else None, len(items), out)
    return int(code), bytes(out) if code == 0 else None


def _oracle(O, fn, items, width):
    out = C.create_string_buffer(width)
    code = getattr(O, fn)(b"".join(items), len(items), out)
    return int(code), out.raw if code == 0 else None


def _rows(out, codes):
    return [(int(c), bytes(o) if c == 0 else None) for o, c in zip(out, codes)]


def _check_rows(out, codes, width):
    for o, c in zip(out, codes):
        if c != 0:
            assert bytes(o) == bytes(width)   # a failed group's bytes are zero


def test_signature_groups_three_ways(engine, oracle_bls_c, torsion):
    from ethereum_consensus_b200 import crypto
    gs = ac.sig_groups(torsion[1])
    flat, off = ac.flatten(gs)
    out, codes = crypto.aggregate_batch(np.frombuffer(flat, dtype=np.uint8), off)
    assert crypto.last_kernel_ms() > 0
    _check_rows(out, codes, 96)
    got = _rows(out, codes)
    for g, row in zip(gs, got):
        assert row == _single("b200_aggregate", g["items"], 96), g["name"]
        assert row == _oracle(oracle_bls_c, "orc_aggregate", g["items"], 96), g["name"]
        if g["want"] is not None:
            assert row == g["want"], g["name"]


def test_key_groups_three_ways(engine, oracle_bls_c, torsion):
    from ethereum_consensus_b200 import crypto
    gs = ac.key_groups(torsion[0])
    flat, off = ac.flatten(gs)
    out, codes = crypto.eth_aggregate_public_keys_batch(np.frombuffer(flat, dtype=np.uint8), off)
    _check_rows(out, codes, 48)
    for g, row in zip(gs, _rows(out, codes)):
        assert row == _single("b200_eth_aggregate_public_keys", g["items"], 48), g["name"]
        assert row == _oracle(oracle_bls_c, "orc_eth_aggregate_public_keys", g["items"], 48), g["name"]
        if g["want"] is not None:
            assert row == g["want"], g["name"]


def test_slot_and_a_group_of_32768(engine, oracle_bls_c, slot):
    """64 x 512 and one group of 2^15 in one call (chunks of more than 32 signatures), checked against the closed forms, a
    seeded subsample of single calls and the C oracle."""
    from ethereum_consensus_b200 import crypto
    big, big_sum = ac.big_group()
    sigs = slot["sigs"] + big
    off = slot["offsets"] + [slot["offsets"][-1] + len(big)]
    out, codes = crypto.aggregate_batch(_arr(sigs, 96), off)
    assert codes.tolist() == [0] * 65
    assert [bytes(o) for o in out] == slot["agg_sig"] + [big_sum]
    rnd = random.Random(7)
    for c in rnd.sample(range(64), 3):
        items = slot["sigs"][off[c]:off[c + 1]]
        assert _single("b200_aggregate", items, 96) == (0, slot["agg_sig"][c])
        assert _oracle(oracle_bls_c, "orc_aggregate", items, 96) == (0, slot["agg_sig"][c])
    assert _single("b200_aggregate", big, 96) == (0, big_sum)
    # the same slot's keys, strict
    kout, kcodes = crypto.eth_aggregate_public_keys_batch(_arr(slot["keys"], 48), slot["offsets"])
    assert kcodes.tolist() == [0] * 64 and [bytes(o) for o in kout] == slot["agg_pk"]
    for c in rnd.sample(range(64), 3):
        items = slot["keys"][off[c]:off[c + 1]]
        assert _oracle(oracle_bls_c, "orc_eth_aggregate_public_keys", items, 48) == (0, slot["agg_pk"][c])


def test_slot_round_trip(engine, slot):
    """The committee aggregates verify against their committees' keys; one flipped member fails that tuple only."""
    from ethereum_consensus_b200 import crypto
    out, codes = crypto.aggregate_batch(_arr(slot["sigs"], 96), slot["offsets"])
    assert codes.tolist() == [0] * 64
    msgs = _arr(slot["msgs"], 32)
    pks = _arr(slot["keys"], 48)
    off = np.array(slot["offsets"], dtype=np.uint32)
    assert crypto.fast_aggregate_verify_batch(pks, off, msgs, out.reshape(-1)).tolist() == [0] * 64
    sigs = list(slot["sigs"])
    sigs[512 * 9 + 100] = sigs[512 * 9 + 101]        # committee 9: a duplicate in place of one member
    out2, codes2 = crypto.aggregate_batch(_arr(sigs, 96), slot["offsets"])
    assert codes2.tolist() == [0] * 64
    assert [bytes(o) for o in out2] != [bytes(o) for o in out]
    want = [0] * 64
    want[9] = 5
    assert crypto.fast_aggregate_verify_batch(pks, off, msgs, out2.reshape(-1)).tolist() == want


def _registry_equals_strict(reg, keys, groups):
    from ethereum_consensus_b200 import crypto
    idx = np.array([i for g in groups for i in g], dtype=np.uint32)
    off = np.cumsum([0] + [len(g) for g in groups]).astype(np.uint32)
    rout, rcodes = reg.aggregate_public_keys(idx, off)
    sout, scodes = crypto.eth_aggregate_public_keys_batch(_arr([keys[i] for i in idx], 48), off)
    assert rcodes.tolist() == scodes.tolist()
    assert np.array_equal(rout, sout)
    return rcodes


def test_registry_paths_equal_the_strict_batch(engine, oracle_bls_c, torsion):
    from ethereum_consensus_b200 import crypto, ssz, state as S
    keys, groups = ac.registry_layout(torsion[0])
    flat = _arr(keys, 48)
    reg = crypto.Registry(flat)
    codes = _registry_equals_strict(reg, keys, groups)
    assert set(codes.tolist()) == {0, 1, 2, 3, 6, 16}
    for g, c in zip(groups[:12], codes[:12]):
        assert (int(c) != 0) == (_oracle(oracle_bls_c, "orc_eth_aggregate_public_keys", [keys[i] for i in g], 48)[0] != 0)
    key_codes = reg.key_codes().tolist()
    # built by appends
    reg = crypto.Registry(flat[:48 * 200])
    reg.append(flat[48 * 200:48 * 450])
    reg.append(flat[48 * 450:])
    assert _registry_equals_strict(reg, keys, groups).tolist() == codes.tolist()
    assert reg.key_codes().tolist() == key_codes
    # built from a resident state, then synced after the state grew: a sync committee of 512 with repeats
    n0 = 400
    st = S.synth_state(len(keys), "minimal", pubkeys=flat.reshape(-1, 48))
    st0 = S.synth_state(n0, "minimal", pubkeys=flat.reshape(-1, 48)[:n0])
    h = ssz.DeviceBeaconState(S.serialize(st0), "minimal")
    reg = crypto.Registry.from_state(h)
    assert _registry_equals_strict(reg, keys[:n0], [g for g in groups if all(i < n0 for i in g)]) is not None
    h.close()
    h = ssz.DeviceBeaconState(S.serialize(st), "minimal")
    reg.sync(h)
    assert reg.n == len(keys)
    assert _registry_equals_strict(reg, keys, groups).tolist() == codes.tolist()
    rnd = random.Random(512)
    valid = [i for i, c in enumerate(key_codes) if c == 0]
    committee = [rnd.choice(valid) for _ in range(512)]
    _registry_equals_strict(reg, keys, [committee])
    out, c = reg.aggregate_public_keys(np.array(committee, dtype=np.uint32), [0, 512])
    assert c.tolist() == [0]
    assert _oracle(oracle_bls_c, "orc_eth_aggregate_public_keys", [keys[i] for i in committee], 48) == (0, bytes(out[0]))
    h.close()


def test_one_engine_interleaves_aggregation_and_verification(engine, slot, torsion):
    """Groups growing then shrinking, strict and registry verify batches in between: each result equals the result of the
    same call on a fresh sequence, and the registry's key codes do not move."""
    from ethereum_consensus_b200 import crypto
    reg = crypto.Registry(_arr(slot["keys"], 48))
    key_codes = reg.key_codes().tolist()
    msgs = _arr(slot["msgs"], 32)
    off = np.array(slot["offsets"], dtype=np.uint32)
    agg, _ = crypto.aggregate_batch(_arr(slot["sigs"], 96), slot["offsets"])
    sig_gs = ac.sig_groups(torsion[1], seed=2)
    flat_small, off_small = ac.flatten(sig_gs)
    want_small = crypto.aggregate_batch(np.frombuffer(flat_small, dtype=np.uint8), off_small)
    for size in (1, 8, 64, 512, 64, 8, 1):
        sub = [slot["sigs"][512 * c + i] for c in range(64) for i in range(size)]
        o, c = crypto.aggregate_batch(_arr(sub, 96), [size * c for c in range(65)])
        assert c.tolist() == [0] * 64
        ko, kc = reg.aggregate_public_keys(np.array([512 * c + i for c in range(64) for i in range(size)], dtype=np.uint32),
                                           [size * c for c in range(65)])
        so, sc = crypto.eth_aggregate_public_keys_batch(_arr([slot["keys"][512 * c + i] for c in range(64) for i in range(size)], 48),
                                                        [size * c for c in range(65)])
        assert kc.tolist() == sc.tolist() == [0] * 64 and np.array_equal(ko, so)
        assert crypto.fast_aggregate_verify_batch(_arr([bytes(k) for k in ko], 48), np.arange(65, dtype=np.uint32), msgs,
                                                  o.reshape(-1)).tolist() == [0] * 64
        assert reg.verify_batch(np.arange(64 * 512, dtype=np.uint32), off, msgs, agg.reshape(-1)).tolist() == [0] * 64
        assert crypto.fast_aggregate_verify_batch(_arr(slot["keys"], 48), off, msgs, agg.reshape(-1)).tolist() == [0] * 64
        got = crypto.aggregate_batch(np.frombuffer(flat_small, dtype=np.uint8), off_small)
        assert np.array_equal(got[0], want_small[0]) and np.array_equal(got[1], want_small[1])
    assert reg.key_codes().tolist() == key_codes


def test_refusals_leave_the_registry_as_it_was(engine):
    from ethereum_consensus_b200 import _lib, crypto
    keys, _, _, _ = ac.key_pool(9, 40)
    reg = crypto.Registry(_arr(keys, 48))
    codes = reg.key_codes().tolist()
    L = _lib.lib()
    out, oc = (C.c_uint8 * (48 * 4))(), (C.c_int32 * 4)()
    out96 = (C.c_uint8 * (96 * 4))()
    sigs = np.zeros(96 * 8, dtype=np.uint8)
    pks = _arr(keys, 48)
    idx = np.arange(40, dtype=np.uint32)
    dec = np.array([0, 5, 3], dtype=np.uint32)                 # decreasing offsets
    good = np.array([0, 3, 5], dtype=np.uint32)
    past, one = np.array([0, 40, 1], dtype=np.uint32), np.array([0, 3], dtype=np.uint32)   # index 40 is past the registry
    for rc in (L.b200_aggregate_batch(_lib.ptr(sigs), _lib.ptr(dec), 2, out96, oc),
               L.b200_eth_aggregate_public_keys_batch(_lib.ptr(pks), _lib.ptr(dec), 2, out, oc),
               L.b200_registry_aggregate_public_keys(_lib.ptr(idx), _lib.ptr(dec), 2, out, oc),
               L.b200_aggregate_batch(None, _lib.ptr(good), 2, out96, oc),
               L.b200_eth_aggregate_public_keys_batch(None, _lib.ptr(good), 2, out, oc),
               L.b200_registry_aggregate_public_keys(None, _lib.ptr(good), 2, out, oc),
               L.b200_aggregate_batch(_lib.ptr(sigs), None, 2, out96, oc),
               L.b200_eth_aggregate_public_keys_batch(_lib.ptr(pks), _lib.ptr(good), 2, None, oc),
               L.b200_registry_aggregate_public_keys(_lib.ptr(idx), _lib.ptr(good), 2, out, None),
               L.b200_registry_aggregate_public_keys(_lib.ptr(past), _lib.ptr(one), 1, out, oc)):
        assert rc == _lib.ERR_BAD_ARG
    # n_groups == 0 succeeds, changes nothing, and needs no buffers
    oc[0] = 77
    assert L.b200_aggregate_batch(None, None, 0, None, None) == 0
    assert L.b200_registry_aggregate_public_keys(None, None, 0, None, oc) == 0 and oc[0] == 77
    with pytest.raises(ValueError):
        reg.aggregate_public_keys(idx, [1, 3])
    with pytest.raises(ValueError):
        crypto.aggregate_batch(sigs, [0, 9])
    with pytest.raises(_lib.EngineError):
        reg.aggregate_public_keys(np.array([41], dtype=np.uint32), [0, 1])
    assert reg.n == 40 and reg.key_codes().tolist() == codes
    o, c = reg.aggregate_public_keys(idx, [0, 40])
    assert c.tolist() == [0]
    assert bytes(o[0]) == bytes(crypto.eth_aggregate_public_keys(keys))
