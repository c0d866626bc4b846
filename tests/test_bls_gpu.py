"""GPU parity: the CUDA BLS path (through the C ABI / the crypto mirror) vs the oracle's golden verdicts, bit-exact."""
import json
from pathlib import Path

import numpy as np
import pytest

from ethereum_consensus_b200 import crypto
from tests.test_oracle_bls import B1_PK, B2_MSG, B2_SIG, B2_SK, GOOD_PK, GOOD_SIG

pytestmark = pytest.mark.gpu
GOLDEN = json.loads((Path(__file__).parent / "golden" / "bls_cases.json").read_text())
FAV = GOLDEN["fast_aggregate_verify"]


def _call(fn, *a):
    """Ok(()) -> 0, Err(InvalidSignature) -> 5, Err(BLST(code)) -> code, EmptyAggregate -> 16."""
    try:
        fn(*a)
        return 0
    except crypto.InvalidSignature:
        return 5
    except crypto.BLSTError as e:
        return e.code
    except crypto.EmptyAggregate:
        return 16


def test_fp_selftest_on_device(engine):
    assert crypto.fp_selftest(1 << 16, 1) == 0
    assert crypto.fp_selftest(1 << 12, 2) == 0


def test_kat_b2_through_the_device(engine):
    from oracle import bls_oracle as bo
    pk = bo.sk_to_pk(B2_SK)
    crypto.verify_signature(pk, B2_MSG, B2_SIG)
    with pytest.raises(crypto.InvalidSignature):
        crypto.verify_signature(pk, B2_MSG + b"!", B2_SIG)
    with pytest.raises(crypto.InvalidSignature):
        crypto.verify_signature(B1_PK, B2_MSG, B2_SIG)
    # decode-only KATs (crypto/bls.rs:381-390, 453-461): well-formed points, wrong signature for this key/message
    assert _call(crypto.verify_signature, GOOD_PK, B2_MSG, GOOD_SIG) == 5


def test_byte_length_rules(engine):
    # crypto/bls.rs:372-377, 393-406, 463-487
    for n in (0, 95, 97):
        with pytest.raises(crypto.SimpleSerializeError):
            crypto.Signature(bytes(n))
    for n in (0, 47, 49):
        with pytest.raises(crypto.SimpleSerializeError):
            crypto.PublicKey(bytes(n))
    crypto.PublicKey(bytes(48)); crypto.PublicKey(bytes([0xC0]) + bytes(47)); crypto.Signature()
    assert crypto.Signature(bytes([0xC0]) + bytes(95)).is_infinity()


@pytest.mark.parametrize("case", FAV, ids=lambda c: c["name"])
def test_fast_aggregate_verify_single(engine, case):
    pks = [bytes.fromhex(p) for p in case["pks"]]
    m, s = bytes.fromhex(case["msg"]), bytes.fromhex(case["sig"])
    assert _call(crypto.fast_aggregate_verify, pks, m, s) == case["code"]
    want_eth = 0 if (not pks and s == bytes([0xC0]) + bytes(95)) else case["code"]
    assert _call(crypto.eth_fast_aggregate_verify, pks, m, s) == want_eth
    if len(pks) == 1:
        assert _call(crypto.verify_signature, pks[0], m, s) == case["code"]


def _batch_inputs(cases, reps=1):
    cases = [c for c in cases if len(c["msg"]) == 64] * reps
    pks = b"".join(bytes.fromhex(p) for c in cases for p in c["pks"])
    off = np.cumsum([0] + [len(c["pks"]) for c in cases]).astype(np.uint32)
    msgs = b"".join(bytes.fromhex(c["msg"]) for c in cases)
    sigs = b"".join(bytes.fromhex(c["sig"]) for c in cases)
    want = np.array([c["code"] for c in cases], dtype=np.int32)
    return np.frombuffer(pks, dtype=np.uint8), off, np.frombuffer(msgs, dtype=np.uint8), np.frombuffer(sigs, dtype=np.uint8), want


def test_fast_aggregate_verify_batch_all_golden(engine):
    pks, off, msgs, sigs, want = _batch_inputs(FAV)
    got = crypto.fast_aggregate_verify_batch(pks, off, msgs, sigs)
    assert got.tolist() == want.tolist()
    # same batch repeated and permuted: per-tuple verdicts are independent of batch composition
    pks, off, msgs, sigs, want = _batch_inputs(list(reversed(FAV)), reps=3)
    got = crypto.fast_aggregate_verify_batch(pks, off, msgs, sigs)
    assert got.tolist() == want.tolist()


def test_vm_launch_shapes_same_codes_on_ragged_golden_batch(engine):
    """The strict batch with the VM kernels at every CTA size, with and without 16-lane teams: launch shapes only — the
    golden codes (ragged K, empty tuples, every failure kind) must not move."""
    pks, off, msgs, sigs, want = _batch_inputs(list(reversed(FAV)), reps=3)
    try:
        for vm_cta in (32, 64, 128):
            crypto.tune("vm_cta", vm_cta)
            for team16_max in (0, 1 << 20):
                crypto.tune("vm_team16_max", team16_max)
                got = crypto.fast_aggregate_verify_batch(pks, off, msgs, sigs)
                assert got.tolist() == want.tolist(), (vm_cta, team16_max)
        with pytest.raises(Exception):
            crypto.tune("no_such_knob", 1)
    finally:
        for k, v in (("vm_cta", 32), ("bls_small_cta", 0), ("vm_team16_max", 2048)):
            crypto.tune(k, v)


def test_registry_mode_matches_strict(engine):
    cases = [c for c in FAV if len(c["msg"]) == 64]
    uniq = sorted({p for c in cases for p in c["pks"]})
    pos = {p: i for i, p in enumerate(uniq)}
    reg = crypto.Registry(np.frombuffer(b"".join(bytes.fromhex(p) for p in uniq), dtype=np.uint8))
    from oracle import bls_oracle as bo
    codes = reg.key_codes()
    for p, c in zip(uniq[:8] + uniq[-8:], list(codes[:8]) + list(codes[-8:])):
        assert bo.key_validate(bytes.fromhex(p))[0] == c
    idx = np.array([pos[p] for c in cases for p in c["pks"]], dtype=np.uint32)
    off = np.cumsum([0] + [len(c["pks"]) for c in cases]).astype(np.uint32)
    msgs = np.frombuffer(b"".join(bytes.fromhex(c["msg"]) for c in cases), dtype=np.uint8)
    sigs = np.frombuffer(b"".join(bytes.fromhex(c["sig"]) for c in cases), dtype=np.uint8)
    got = reg.verify_batch(idx, off, msgs, sigs)
    assert got.tolist() == [c["code"] for c in cases]


def test_mixed_mode_extra_keys_validated_in_call(engine):
    """`..._batch_mixed`: every other distinct key lives in the registry, the rest arrive as extra keys (incl. the golden
    cases' undecodable / infinite / off-curve / out-of-subgroup keys) — same codes as the strict path, twice in a row
    (the registry's spare tail is reused), and an index past registry + extras is refused."""
    cases = [c for c in FAV if len(c["msg"]) == 64]
    uniq = sorted({p for c in cases for p in c["pks"]})
    in_reg = uniq[::2]
    extra = uniq[1::2]
    reg = crypto.Registry(np.frombuffer(b"".join(bytes.fromhex(p) for p in in_reg), dtype=np.uint8))
    pos = {p: i for i, p in enumerate(in_reg)}
    pos.update({p: len(in_reg) + j for j, p in enumerate(extra)})
    idx = np.array([pos[p] for c in cases for p in c["pks"]], dtype=np.uint32)
    off = np.cumsum([0] + [len(c["pks"]) for c in cases]).astype(np.uint32)
    msgs = np.frombuffer(b"".join(bytes.fromhex(c["msg"]) for c in cases), dtype=np.uint8)
    sigs = np.frombuffer(b"".join(bytes.fromhex(c["sig"]) for c in cases), dtype=np.uint8)
    xk = np.frombuffer(b"".join(bytes.fromhex(p) for p in extra), dtype=np.uint8)
    want = [c["code"] for c in cases]
    for _ in range(2):
        assert reg.verify_batch(idx, off, msgs, sigs, extra_keys=xk).tolist() == want
    bad = idx.copy()
    bad[0] = len(uniq)
    with pytest.raises(Exception):
        reg.verify_batch(bad, off, msgs, sigs, extra_keys=xk)
    with pytest.raises(Exception):      # extra-key indices without the extra keys
        reg.verify_batch(idx, off, msgs, sigs)
    # the registry itself is untouched by the calls
    assert crypto.Registry.key_codes(reg).tolist() == [c for c in reg.key_codes()]


@pytest.mark.parametrize("case", GOLDEN["aggregate_verify"], ids=lambda c: c["name"])
def test_aggregate_verify(engine, case):
    pks = [bytes.fromhex(p) for p in case["pks"]]
    msgs = [bytes.fromhex(m) for m in case["msgs"]]
    assert _call(crypto.aggregate_verify, pks, msgs, bytes.fromhex(case["sig"])) == case["code"]


@pytest.mark.parametrize("case", GOLDEN["aggregate"], ids=lambda c: c["name"])
def test_aggregate(engine, case):
    sigs = [bytes.fromhex(s) for s in case["sigs"]]
    try:
        out = crypto.aggregate(sigs)
        assert case["code"] == 0 and bytes(out).hex() == case["out"]
    except crypto.BLSTError as e:
        assert e.code == case["code"]
    with pytest.raises(crypto.EmptyAggregate):
        crypto.aggregate([])


@pytest.mark.parametrize("case", GOLDEN["eth_aggregate_public_keys"], ids=lambda c: c["name"])
def test_eth_aggregate_public_keys(engine, case):
    pks = [bytes.fromhex(s) for s in case["pks"]]
    try:
        out = crypto.eth_aggregate_public_keys(pks)
        assert case["code"] == 0 and bytes(out).hex() == case["out"]
    except crypto.BLSTError as e:
        assert e.code == case["code"]
    with pytest.raises(crypto.EmptyAggregate):
        crypto.eth_aggregate_public_keys([])


def test_aggregate_then_verify_roundtrip(engine):
    """crypto/bls.rs:489-523: aggregate n signatures, then (fast_)aggregate_verify — here with golden material."""
    c = GOLDEN["aggregate_verify"][0]
    pks = [bytes.fromhex(p) for p in c["pks"]]
    msgs = [bytes.fromhex(m) for m in c["msgs"]]
    agg = crypto.aggregate([bytes.fromhex(s) for s in GOLDEN["aggregate"][0]["sigs"]])
    assert bytes(agg).hex() == c["sig"]
    crypto.aggregate_verify(pks, msgs, agg)
