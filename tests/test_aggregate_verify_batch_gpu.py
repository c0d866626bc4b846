"""GPU: aggregate_verify over T tuples per call (tests/aggregate_verify_cases.py).  For every tuple the batch call, the
single call b200_aggregate_verify and the C oracle agree code for code: the golden cases as one batch, every crafted tuple,
shuffled, and closed-form batches of 256 x 64 (8-lane programs), 1 x 2048 (one fold over three levels) and 4096 x 1.  Also:
both team sizes and every vm_cta; the registry path equals the strict path, keys appended after the load and keys that
failed validation included; the one-thread pairing kernels (B200_PAIRING_VM=0, in a child process); the segmented Gt
product value by value (b200_pairing_eval); one engine interleaving this call with the other families; every refusal,
each followed by a good call; and the launches per call shape."""
from __future__ import annotations

import ctypes as C
import json
import os
import random
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

from oracle import bls_oracle as bo
from tests import aggregate_verify_cases as av
from tests import pairing_cases as pc
from tests import torsion_cases as tc

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent
GOLDEN = json.loads((ROOT / "tests" / "golden" / "bls_cases.json").read_text())["aggregate_verify"]

# Launches per call (b200_launch_count).  K1 per-key validation, K3 signature decode, K4 hash_to_G2 (two kernels), K2 per-tuple
# key-code scan, the pair operands, the Miller loops, one launch per level of the segmented product, final exponentiations.
STRICT_1x4 = 1 + 1 + 2 + 1 + 1 + 1 + 1 + 1           # 5 Miller values: one level
STRICT_1x2048 = 1 + 1 + 2 + 1 + 1 + 1 + 3 + 1        # 2049 values -> 65 -> 3 -> two per tuple: three levels
STRICT_4096x1 = 1 + 1 + 2 + 1 + 1 + 1 + 0 + 1        # two Miller values per tuple already: no level
STRICT_256x64 = 1 + 1 + 2 + 1 + 1 + 1 + 2 + 1        # 65 values per tuple: in up to three pieces, then one level more
STRICT_SHAPE_ONLY = 1 + 1 + 2 + 1 + 1 + 0 + 0 + 1    # no tuple has a pairing: no Miller loop, no level
REGISTRY_1x4 = STRICT_1x4 - 1                         # no K1
VM0_STRICT_1x4 = 1 + 1 + 2 + 1 + 1 + 1                # one thread per pair: the keys themselves, Miller, final
VM0_REGISTRY_1x4 = 1 + 2 + 1 + 1 + 1 + 1              # K3, K4, K2, the registry points gathered, Miller, final


@pytest.fixture(scope="module")
def O(oracle_bls_c):
    return av.bind(oracle_bls_c)


@pytest.fixture(scope="module")
def cases(O):
    return av.crafted(O, tc.g1_cases(), tc.g2_cases())


@pytest.fixture(scope="module")
def big(O):
    return av.scale(O, 256, 64, seed=3, bad_every=37)


def _arr(b: bytes):
    return np.frombuffer(b, dtype=np.uint8).copy() if b else np.zeros(0, dtype=np.uint8)


def _batch(tuples):
    from ethereum_consensus_b200 import crypto
    keys, koff, msgs, grp, sigs = av.flatten(tuples)
    return crypto.aggregate_verify_batch(_arr(keys), koff, msgs, grp, _arr(sigs)).tolist()


def _registry_batch(reg, where, tuples):
    idx = [where[k] for t in tuples for k in t["pks"]]
    _, koff, msgs, grp, sigs = av.flatten(tuples)
    return reg.aggregate_verify_batch(np.array(idx, dtype=np.uint32), koff, msgs, grp, _arr(sigs)).tolist()


def _single(t) -> int:
    from ethereum_consensus_b200 import _lib
    msgs = [bytes(m) for m in t["msgs"]]
    bufs = [C.create_string_buffer(m, max(len(m), 1)) for m in msgs]
    ptrs = (C.c_void_p * max(len(msgs), 1))(*[C.addressof(b) for b in bufs])
    lens = (C.c_size_t * max(len(msgs), 1))(*[len(m) for m in msgs])
    keys = b"".join(t["pks"])
    return int(_lib.lib().b200_aggregate_verify(keys if keys else None, len(t["pks"]), C.cast(ptrs, C.c_void_p),
                                                C.cast(lens, C.c_void_p), len(msgs), t["sig"]))


def _launches():
    from ethereum_consensus_b200 import _lib
    return int(_lib.lib().b200_launch_count())


def _counted(fn, *a):
    n0 = _launches()
    r = fn(*a)
    return r, _launches() - n0


def _vm_cta_in_effect():
    v = int(os.environ.get("B200_VM_CTA", "32"))
    return v if v in (32, 64, 128) else 32


def test_golden_cases_as_one_batch(engine):
    tuples = av.golden(GOLDEN)
    got = _batch(tuples)
    assert got == [t["want"] for t in tuples]
    assert got == [_single(t) for t in tuples]


def test_crafted_tuples_three_ways(engine, O, cases):
    from ethereum_consensus_b200 import crypto
    want = [t["want"] for t in cases]
    got = _batch(cases)
    assert crypto.last_kernel_ms() > 0
    assert got == want
    assert [_single(t) for t in cases] == want
    assert av.oracle_codes(O, cases) == want
    rnd = random.Random(5)
    for _ in range(3):
        order = list(range(len(cases)))
        rnd.shuffle(order)
        assert _batch([cases[i] for i in order]) == [want[i] for i in order]


def test_scale(engine, O, big):
    from ethereum_consensus_b200 import crypto
    rnd = random.Random(11)
    # 256 x 64: 16 640 Miller loops, beyond vm_team16_max -> the 8-lane programs
    got = _batch(big)
    assert got == [t["want"] for t in big] and got.count(av.VERIFY_FAIL) == 6
    sample = rnd.sample(range(256), 6) + [36, 37]
    assert av.oracle_codes(O, [big[i] for i in sample]) == [got[i] for i in sample]
    assert [_single(big[i]) for i in sample[:3]] == [got[i] for i in sample[:3]]
    # one tuple of 2048 pairs, alone and next to one with the other's signature
    long2 = av.scale(O, 2, 2048, seed=4, bad_every=1)
    assert _batch(long2[1:]) == [av.SUCCESS]
    assert _batch(long2) == [av.VERIFY_FAIL, av.SUCCESS]
    assert av.oracle_codes(O, long2[1:]) == [av.SUCCESS]
    # 4096 x 1: the same tuples through fast_aggregate_verify_batch with K = 1 (32-byte messages) give the same codes
    wide = av.scale(O, 4096, 1, seed=5, bad_every=101)
    got = _batch(wide)
    assert got == [t["want"] for t in wide] and got.count(av.VERIFY_FAIL) == 40
    keys = _arr(b"".join(t["pks"][0] for t in wide))
    fast = crypto.fast_aggregate_verify_batch(keys, np.arange(4097, dtype=np.uint32), _arr(b"".join(t["msgs"][0] for t in wide)),
                                              _arr(b"".join(t["sig"] for t in wide)))
    assert fast.tolist() == got
    assert av.oracle_codes(O, [wide[i] for i in (0, 100, 101, 4095)]) == [got[i] for i in (0, 100, 101, 4095)]


def test_team_sizes_and_cta(engine, O, cases):
    from ethereum_consensus_b200 import crypto
    mid = av.scale(O, 40, 33, seed=6, bad_every=7)
    want_c, want_m = [t["want"] for t in cases], [t["want"] for t in mid]
    try:
        for team16_max in (0, 1 << 30):       # always the 8-lane programs / always the 16-lane programs
            crypto.tune("vm_team16_max", team16_max)
            for cta in (32, 64, 128):
                crypto.tune("vm_cta", cta)
                assert _batch(cases) == want_c, (team16_max, cta)
                assert _batch(mid) == want_m, (team16_max, cta)
    finally:
        crypto.tune("vm_team16_max", 2048)
        crypto.tune("vm_cta", _vm_cta_in_effect())


def _registry_keys(tuples):
    keys = []
    for t in tuples:
        keys += [k for k in t["pks"] if k not in keys]
    return keys


def test_registry_equals_strict(engine, cases, big):
    from ethereum_consensus_b200 import crypto
    keys = _registry_keys(cases)
    where = {k: i for i, k in enumerate(keys)}
    cut = len(keys) * 3 // 5
    reg = crypto.Registry(_arr(b"".join(keys[:cut])))
    reg.append(_arr(b"".join(keys[cut:])))             # keys appended after the load
    codes = reg.key_codes().tolist()
    assert len(codes) == len(keys) and any(codes[:cut]) and any(codes[cut:])   # failed validation on both sides of the cut
    strict = _batch(cases)
    assert _registry_batch(reg, where, cases) == strict
    rnd = random.Random(8)
    order = list(range(len(cases)))
    rnd.shuffle(order)
    assert _registry_batch(reg, where, [cases[i] for i in order]) == [strict[i] for i in order]
    # the big batch from a registry of its own keys
    keys = [k for t in big for k in t["pks"]]
    reg = crypto.Registry(_arr(b"".join(keys)))
    assert _registry_batch(reg, {k: i for i, k in enumerate(keys)}, big) == [t["want"] for t in big]
    assert reg.key_codes().tolist() == [0] * len(keys)


def _dump(tuples, path):
    path.write_text(json.dumps([{**t, "pks": [k.hex() for k in t["pks"]], "msgs": [m.hex() for m in t["msgs"]], "sig": t["sig"].hex()}
                                for t in tuples]))


def _load(path):
    return [{**t, "pks": [bytes.fromhex(k) for k in t["pks"]], "msgs": [bytes.fromhex(m) for m in t["msgs"]], "sig": bytes.fromhex(t["sig"])}
            for t in json.loads(Path(path).read_text())]


def _child(path):
    """B200_PAIRING_VM=0 (set by the parent): refusal without a registry, then the codes and launches of each path."""
    from ethereum_consensus_b200 import _lib, crypto
    _lib.init(0)
    tuples = _load(path)
    L = _lib.lib()
    keys, koff, msgs, grp, sigs = av.flatten(tuples[:2])
    moff = np.cumsum([0] + [len(m) for m in msgs]).astype(np.uint32)
    flat, g, out = _arr(b"".join(msgs)), np.array(grp, dtype=np.uint32), np.zeros(2, dtype=np.int32)
    idx = np.zeros(koff[-1], dtype=np.uint32)
    res = {"no_registry": L.b200_aggregate_verify_batch_indexed(_lib.ptr(idx), _lib.ptr(np.array(koff, dtype=np.uint32)), _lib.ptr(flat),
                                                                _lib.ptr(moff), _lib.ptr(g), _lib.ptr(_arr(sigs)), 2, _lib.ptr(out))}
    res["codes"] = _batch(tuples)
    four = [t for t in tuples if len(t["pks"]) == 4 and len(t["msgs"]) == 4][:1]
    res["strict_1x4"] = list(_counted(_batch, four))
    keys = _registry_keys(tuples)
    reg = crypto.Registry(_arr(b"".join(keys[:20])))
    reg.append(_arr(b"".join(keys[20:])))
    where = {k: i for i, k in enumerate(keys)}
    res["registry"] = _registry_batch(reg, where, tuples)
    res["registry_1x4"] = list(_counted(_registry_batch, reg, where, four))
    print("RESULT " + json.dumps(res))


def test_without_pairing_vm(engine, cases, tmp_path):
    """The one-thread-per-pair kernels (k_miller + k_final) take the batch's multi-pair tuples through pair_off."""
    from ethereum_consensus_b200 import _lib
    path = tmp_path / "cases.json"
    _dump(cases, path)
    p = subprocess.run([sys.executable, "-m", "tests.test_aggregate_verify_batch_gpu", str(path)], cwd=str(ROOT), capture_output=True,
                       text=True, env=dict(os.environ, B200_PAIRING_VM="0"), timeout=1200)
    assert p.returncode == 0, p.stdout + p.stderr
    res = json.loads(next(ln for ln in p.stdout.splitlines() if ln.startswith("RESULT "))[7:])
    want = [t["want"] for t in cases]
    assert res["no_registry"] == _lib.ERR_BAD_ARG
    assert res["codes"] == want and res["registry"] == want
    assert res["strict_1x4"] == [[av.SUCCESS], VM0_STRICT_1x4]
    assert res["registry_1x4"] == [[av.SUCCESS], VM0_REGISTRY_1x4]


def test_fold_segments_value_by_value(engine):
    from ethereum_consensus_b200 import _lib, crypto
    rnd = random.Random(17)
    pool = [x for x in pc.tower_elements(18, n_random=200) if any(x)]
    one = pc.to_real(pc.to_raw([1] + [0] * 11))
    for name, lengths in av.segment_layouts().items():
        T, total = len(lengths), sum(lengths)
        n = max(total + 3, 2 * T)                       # values past the last offset are ignored
        rows = [pool[rnd.randrange(len(pool))] for _ in range(n)]
        a = pc.pack(rows)
        b = np.zeros_like(a)
        off = np.cumsum([0] + lengths).astype(np.uint32)
        b.reshape(-1)[0] = T
        b.reshape(-1)[1:T + 2] = off
        out = crypto.pairing_eval("fold_segments", a, b)
        raw = pc.unpack(out)
        assert all(max(r) < bo.P for r in raw[:2 * T]), name
        got = [pc.to_real(r) for r in raw]
        for t in range(T):
            lo, hi = int(off[t]), int(off[t + 1])
            if lo == hi:
                assert raw[2 * t] == [0] * 12 and raw[2 * t + 1] == [0] * 12, (name, t)
                continue
            acc = bo.f12_one()
            for i in range(lo, hi):
                acc = bo.f12_mul(acc, pc.to_oracle(pc.to_real(rows[i])))
            assert bo.f12_mul(pc.to_oracle(got[2 * t]), pc.to_oracle(got[2 * t + 1])) == acc, (name, t)
            if (hi - 1) // 32 == lo // 32:
                assert got[2 * t + 1] == one, (name, t)   # one piece: padded with Fp12 one
    # malformed layouts are refused
    a = pc.pack(pool[:8])
    for words in ([0, 0], [5, 0, 1, 2, 3, 4, 5], [2, 1, 2, 3], [2, 0, 3, 2], [2, 0, 4, 9]):
        b = np.zeros_like(a)
        b.reshape(-1)[:len(words)] = words
        with pytest.raises(_lib.EngineError):
            crypto.pairing_eval("fold_segments", a, b)


def test_one_engine_interleaves_the_families(engine, O, cases, big):
    from ethereum_consensus_b200 import crypto, ssz, state as S
    small = av.scale(O, 3, 2, seed=9, bad_every=2)
    mid = av.scale(O, 64, 33, seed=10, bad_every=9)
    st = S.synth_state(300, "minimal")
    root = ssz.hash_tree_root_beacon_state(S.serialize(st), "minimal")
    fk = _arr(b"".join(t["pks"][0] for t in mid))
    fm = _arr(b"".join(hashlib_msgs(64)))
    fs = _arr(b"".join(t["sig"] for t in mid))
    fast_want = crypto.fast_aggregate_verify_batch(fk, np.arange(65, dtype=np.uint32), fm, fs).tolist()
    agg_sigs = [t["sig"] for t in mid]
    agg_want = crypto.aggregate_batch(_arr(b"".join(agg_sigs)), [0, 10, 10, 64])
    for batch in (small, mid, big, cases, mid, small, big[:5], small):
        assert _batch(batch) == [t["want"] for t in batch]
        assert crypto.fast_aggregate_verify_batch(fk, np.arange(65, dtype=np.uint32), fm, fs).tolist() == fast_want
        o, c = crypto.aggregate_batch(_arr(b"".join(agg_sigs)), [0, 10, 10, 64])
        assert np.array_equal(o, agg_want[0]) and np.array_equal(c, agg_want[1])
        assert ssz.hash_tree_root_beacon_state(S.serialize(st), "minimal") == root


def hashlib_msgs(n):
    import hashlib
    return [hashlib.sha256(b"interleave %d" % i).digest() for i in range(n)]


def test_refusals_then_good_calls(engine, cases):
    from ethereum_consensus_b200 import _lib, crypto
    L = _lib.lib()
    good = [t for t in cases if t["name"] in ("three signers", "two messages swapped", "valid n 2")]
    want = [t["want"] for t in good]
    keys, koff, msgs, grp, sigs = av.flatten(good)
    K, KO = _arr(keys), np.array(koff, dtype=np.uint32)
    M = _arr(b"".join(msgs))
    MO = np.cumsum([0] + [len(m) for m in msgs]).astype(np.uint32)
    G, S = np.array(grp, dtype=np.uint32), _arr(sigs)
    reg_keys = _registry_keys(good)
    reg = crypto.Registry(_arr(b"".join(reg_keys)))
    reg_codes = reg.key_codes().tolist()
    IDX = np.array([reg_keys.index(k) for t in good for k in t["pks"]], dtype=np.uint32)
    out = np.zeros(3, dtype=np.int32)
    p = _lib.ptr

    def strict(k=K, ko=KO, m=M, mo=MO, g=G, s=S, o=out, t=3):
        return L.b200_aggregate_verify_batch(p(k) if k is not None else None, p(ko) if ko is not None else None, p(m) if m is not None else None,
                                             p(mo) if mo is not None else None, p(g) if g is not None else None, p(s) if s is not None else None,
                                             t, p(o) if o is not None else None)

    def indexed(i=IDX, ko=KO, t=3):
        return L.b200_aggregate_verify_batch_indexed(p(i) if i is not None else None, p(ko), p(M), p(MO), p(G), p(S), t, p(out))

    def u32(v):
        return np.array(v, dtype=np.uint32)
    refusals = [
        lambda: strict(k=None), lambda: strict(ko=None), lambda: strict(m=None), lambda: strict(mo=None), lambda: strict(g=None),
        lambda: strict(s=None), lambda: strict(o=None),
        lambda: strict(ko=u32([1, 3, 5, 7])), lambda: strict(ko=u32([0, 5, 3, 7])),
        lambda: strict(g=u32([1, 3, 5, 7])), lambda: strict(g=u32([0, 5, 3, 7])),
        lambda: strict(mo=MO + 1), lambda: strict(mo=np.concatenate([MO[:2], MO[:1], MO[3:]])),
        lambda: strict(ko=u32([0, 0x40000000, 0x40000000, 0x40000000])),
        lambda: strict(g=u32([0, 0x40000000, 0x40000000, 0x40000000])),
        lambda: strict(t=(1 << 26) + 1),
        lambda: indexed(i=None), lambda: indexed(i=IDX + 100), lambda: indexed(ko=u32([0, 3, 2, 7])),
    ]
    for r in refusals:
        assert r() == _lib.ERR_BAD_ARG
        out[:] = -1
        assert strict() == 0 and out.tolist() == want
        out[:] = -1
        assert indexed() == 0 and out.tolist() == want
    assert reg.key_codes().tolist() == reg_codes and reg.n == len(reg_keys)
    # n_tuples == 0 succeeds and needs no buffers
    assert L.b200_aggregate_verify_batch(None, None, None, None, None, None, 0, None) == 0
    assert L.b200_aggregate_verify_batch_indexed(None, None, None, None, None, None, 0, None) == 0
    with pytest.raises(ValueError):
        crypto.aggregate_verify_batch(K, koff, msgs, grp[:-1], S)
    with pytest.raises(ValueError):
        crypto.aggregate_verify_batch(K, koff, msgs[:-1], grp, S)
    with pytest.raises(ValueError):
        reg.aggregate_verify_batch(IDX[:-1], koff, msgs, grp, S)
    assert crypto.aggregate_verify_batch(K, koff, msgs, grp, S).tolist() == want


def test_launches_per_call(engine, O, cases, big):
    from ethereum_consensus_b200 import crypto
    four = [t for t in cases if len(t["pks"]) == 4 and len(t["msgs"]) == 4][:1]
    assert len(four) == 1
    assert _counted(_batch, four) == ([av.SUCCESS], STRICT_1x4)
    long1 = av.scale(O, 1, 2048, seed=12)
    assert _counted(_batch, long1) == ([av.SUCCESS], STRICT_1x2048)
    wide = av.scale(O, 4096, 1, seed=13)
    assert _counted(_batch, wide) == ([av.SUCCESS] * 4096, STRICT_4096x1)
    assert _counted(_batch, big) == ([t["want"] for t in big], STRICT_256x64)
    shape = [t for t in cases if t["name"] in ("3 keys, 2 messages", "no keys, no messages, a signature")]
    assert _counted(_batch, shape) == ([av.VERIFY_FAIL] * 2, STRICT_SHAPE_ONLY)
    keys = _registry_keys(four)
    reg = crypto.Registry(_arr(b"".join(keys)))
    assert _counted(_registry_batch, reg, {k: i for i, k in enumerate(keys)}, four) == ([av.SUCCESS], REGISTRY_1x4)


if __name__ == "__main__":
    _child(sys.argv[1])
