"""Tuples for aggregate_verify over T tuples per call, shared by the CPU check (tests/test_aggregate_verify_cases.py) and
the device run (tests/test_aggregate_verify_batch_gpu.py).  No device code here.

A tuple is a dict: name, pks (48-byte encodings), msgs (bytes of any length), sig (96 bytes), want (the code it was built
to get) and why (what decides it).  Crafted tuples are signed with the plain-C oracle (orc_sign, then orc_aggregate over
the signers' signatures); the scale batches use closed forms instead: with sk_{t,j} = a + t + j d and messages m_j shared by
all tuples, the aggregate signature of tuple t is (a + t) A + d B for A = sum_j H(m_j), B = sum_j j H(m_j), so a batch of
T tuples costs T additions on top of n hashes.  The C oracle's codes of many tuples come from T independent
orc_aggregate_verify calls on a thread pool (ctypes releases the GIL)."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import random
from concurrent.futures import ThreadPoolExecutor

from oracle import bls_oracle as bo
from tests import aggregate_batch_cases as ac

P, R = bo.P, bo.R
SUCCESS, BAD_ENCODING, NOT_ON_CURVE, NOT_IN_GROUP, VERIFY_FAIL, PK_IS_INFINITY = 0, 1, 2, 3, 5, 6
INF_SIG, INF_PK = ac.INF_SIG, ac.INF_PK
VALID_SIZES = (1, 2, 3, 31, 32, 33, 63, 64, 65, 127, 128, 129, 2048)
MSG_LENGTHS = (0, 1, 32, 255, 256, 300)
THREADS = max(1, min(32, os.cpu_count() or 1))


def bind(O):
    """The argument types this module calls the C oracle with (the library object is shared with conftest's fixture)."""
    cp, sz, vp = C.c_char_p, C.c_size_t, C.c_void_p
    O.orc_aggregate_verify.argtypes = [cp, sz, vp, vp, sz, cp]
    O.orc_aggregate.argtypes = [cp, sz, cp]
    O.orc_sk_to_pk.argtypes = [cp, cp]
    O.orc_sign.argtypes = [cp, cp, sz, cp]
    O.orc_hash_to_g2.argtypes = [cp, sz, cp]
    O.orc_pk_sequence.argtypes = [cp, cp, sz, vp]
    return O


def _sk(tag: bytes) -> int:
    return 1 + int.from_bytes(hashlib.sha256(tag).digest(), "big") % (R - 1)


def _b32(k: int) -> bytes:
    return (k % R).to_bytes(32, "big")


def _pool_map(fn, items):
    with ThreadPoolExecutor(THREADS) as ex:
        return list(ex.map(fn, items))


def oracle_code(O, tup) -> int:
    """orc_aggregate_verify of one tuple."""
    msgs = [bytes(m) for m in tup["msgs"]]
    bufs = [C.create_string_buffer(m, max(len(m), 1)) for m in msgs]
    ptrs = (C.c_void_p * max(len(msgs), 1))(*[C.addressof(b) for b in bufs])
    lens = (C.c_size_t * max(len(msgs), 1))(*[len(m) for m in msgs])
    return int(O.orc_aggregate_verify(b"".join(tup["pks"]), len(tup["pks"]), ptrs, lens, len(msgs), tup["sig"]))


def oracle_codes(O, tuples):
    """The C oracle's code of every tuple: T independent orc_aggregate_verify calls on THREADS threads."""
    return _pool_map(lambda t: oracle_code(O, t), tuples)


# -------------------------------------------------------------------------------------------------- signing
def _pk(O, sk: int) -> bytes:
    out = C.create_string_buffer(48)
    O.orc_sk_to_pk(_b32(sk), out)
    return out.raw


def _sign(O, sk: int, msg: bytes) -> bytes:
    out = C.create_string_buffer(96)
    O.orc_sign(_b32(sk), msg, len(msg), out)
    return out.raw


def _aggregate(O, sigs) -> bytes:
    out = C.create_string_buffer(96)
    assert O.orc_aggregate(b"".join(sigs), len(sigs), out) == 0
    return out.raw


def signed(O, sks, msgs):
    """(keys, aggregate signature) of the signers sks over msgs (pairwise)."""
    pks = _pool_map(lambda k: _pk(O, k), sks)
    sigs = _pool_map(lambda km: _sign(O, *km), list(zip(sks, msgs)))
    return pks, _aggregate(O, sigs), sigs


def _tuple(name, pks, msgs, sig, want, why):
    return {"name": name, "pks": list(pks), "msgs": [bytes(m) for m in msgs], "sig": bytes(sig), "want": want, "why": why}


def _msgs(tag: str, n: int):
    return [hashlib.sha256(b"%s %d" % (tag.encode(), j)).digest() for j in range(n)]


# -------------------------------------------------------------------------------------------------- crafted tuples
def crafted(O, torsion_g1, torsion_g2, seed=1):
    """Every kind of tuple once, in an order that mixes sizes and codes."""
    rnd = random.Random(0xA7 + seed)
    out = []
    for n in VALID_SIZES:   # valid tuples of every size around the 32-value chunks of the fold
        sks = [_sk(b"av %d sk %d %d" % (seed, n, j)) for j in range(n)]
        msgs = _msgs(f"av {seed} msg {n}", n)
        pks, sig, _ = signed(O, sks, msgs)
        out.append(_tuple(f"valid n {n}", pks, msgs, sig, SUCCESS, "every pair signed"))
    sks3 = [_sk(b"av %d three %d" % (seed, j)) for j in range(3)]
    m3 = _msgs(f"av {seed} three", 3)
    pks3, sig3, sigs3 = signed(O, sks3, m3)
    good_sig = sig3
    out.append(_tuple("three signers", pks3, m3, sig3, SUCCESS, "the control of the crossed and changed tuples below"))
    out.append(_tuple("no keys, no messages, infinity signature", [], [], INF_SIG, VERIFY_FAIL, "no keys"))
    out.append(_tuple("no keys, no messages, a signature", [], [], good_sig, VERIFY_FAIL, "no keys"))
    out.append(_tuple("no keys, one message", [], m3[:1], good_sig, VERIFY_FAIL, "no keys"))
    out.append(_tuple("3 keys, 2 messages", pks3, m3[:2], sig3, VERIFY_FAIL, "more keys than messages"))
    out.append(_tuple("2 keys, 3 messages", pks3[:2], m3, sig3, VERIFY_FAIL, "more messages than keys"))
    out.append(_tuple("two messages swapped", pks3, [m3[1], m3[0], m3[2]], sig3, VERIFY_FAIL,
                      "each signature is valid for its own pair, the pairs are crossed"))
    out.append(_tuple("two keys swapped", [pks3[1], pks3[0], pks3[2]], m3, sig3, VERIFY_FAIL, "the pairs are crossed"))
    out.append(_tuple("wrong message", pks3, [m3[0], b"not what was signed", m3[2]], sig3, VERIFY_FAIL, "a message changed"))
    out.append(_tuple("one signer left out", pks3, m3, _aggregate(O, sigs3[:2]), VERIFY_FAIL, "aggregate misses a signer"))
    out.append(_tuple("one signer twice", pks3, m3, _aggregate(O, sigs3 + sigs3[:1]), VERIFY_FAIL, "aggregate has a signer twice"))
    # duplicates are allowed (no distinct-message check in crypto/bls.rs:95-112)
    dm = [m3[0], m3[0], m3[1]]
    pks, sig, _ = signed(O, sks3, dm)
    out.append(_tuple("duplicate messages", pks, dm, sig, SUCCESS, "duplicates allowed"))
    dk = [sks3[0], sks3[0], sks3[1]]
    pks, sig, _ = signed(O, dk, m3)
    out.append(_tuple("duplicate keys", pks, m3, sig, SUCCESS, "duplicates allowed"))
    pks, sig, _ = signed(O, [sks3[2]] * 4, [m3[2]] * 4)
    out.append(_tuple("one pair four times", pks, [m3[2]] * 4, sig, SUCCESS, "duplicates allowed"))
    lm = [bytes(rnd.randrange(256) for _ in range(k)) for k in MSG_LENGTHS]
    sks = [_sk(b"av %d len %d" % (seed, k)) for k in MSG_LENGTHS]
    pks, sig, _ = signed(O, sks, lm)
    out.append(_tuple("messages of 0, 1, 32, 255, 256, 300 bytes", pks, lm, sig, SUCCESS, "any length"))
    pks, sig, _ = signed(O, sks[:1], [b""])
    out.append(_tuple("empty message only", pks, [b""], sig, SUCCESS, "empty message"))
    # keys
    bad_keys = ac.invalid_keys(torsion_g1, rnd)   # infinity, off the curve, small / mixed order, bad encodings
    for enc, code in bad_keys:
        for at in (0, 2):
            pks = list(pks3)
            pks[at] = enc
            out.append(_tuple(f"invalid key ({code}) at {at}", pks, m3, sig3, code, "first invalid key"))
    (e1, c1), (e2, c2) = bad_keys[1], bad_keys[5]
    out.append(_tuple("two invalid keys", [pks3[0], e1, e2], m3, sig3, c1, "the first invalid key in order"))
    out.append(_tuple("invalid keys, other order", [pks3[0], e2, e1], m3, sig3, c2, "the first invalid key in order"))
    # signatures
    bad_sigs = [(e, BAD_ENCODING) for e in ac.bad_encodings(96, rnd)] + [(ac.not_on_curve_g2(rnd), NOT_ON_CURVE)]
    for enc, code in bad_sigs:
        out.append(_tuple(f"signature decode error {code}", pks3, m3, enc, code, "signature decoding"))
    for enc in ac.small_order(torsion_g2, 3, rnd):
        out.append(_tuple("signature outside G2", pks3, m3, enc, VERIFY_FAIL, "signature group check"))
    out.append(_tuple("infinity signature", pks3, m3, INF_SIG, VERIFY_FAIL, "pairing product"))
    # precedence: key code > signature decode code > shape > signature group check > pairing
    out.append(_tuple("bad key and bad signature", [pks3[0], bad_keys[0][0], pks3[2]], m3, bad_sigs[0][0], bad_keys[0][1],
                      "keys are checked first"))
    out.append(_tuple("bad key and a length mismatch", [pks3[0], bad_keys[3][0]], m3, sig3, bad_keys[3][1], "keys before shape"))
    out.append(_tuple("bad signature and a length mismatch", pks3[:2], m3, bad_sigs[3][0], NOT_ON_CURVE, "signature before shape"))
    out.append(_tuple("bad signature, no keys", [], [], bad_sigs[1][0], BAD_ENCODING, "signature before shape"))
    out.append(_tuple("small-order key, signature outside G2", [pks3[0], ac.small_order(torsion_g1, 1, rnd)[0], pks3[2]], m3,
                      ac.small_order(torsion_g2, 1, rnd)[0], NOT_IN_GROUP, "keys before the signature group check"))
    out.append(_tuple("signature outside G2, length mismatch", pks3[:2], m3, ac.small_order(torsion_g2, 1, rnd)[0], VERIFY_FAIL,
                      "shape and group check both fail"))
    rnd.shuffle(out)
    return out


def golden(cases):
    """tests/golden/bls_cases.json's aggregate_verify cases as tuples."""
    return [_tuple(c["name"], [bytes.fromhex(p) for p in c["pks"]], [bytes.fromhex(m) for m in c["msgs"]], bytes.fromhex(c["sig"]),
                   c["code"], "golden") for c in cases]


# -------------------------------------------------------------------------------------------------- scale batches
def _h2g2(O, msg: bytes):
    out = C.create_string_buffer(192)
    O.orc_hash_to_g2(msg, len(msg), out)
    v = [int.from_bytes(out.raw[48 * i:48 * i + 48], "big") for i in range(4)]
    return ((v[0], v[1]), (v[2], v[3]))


def scale(O, T: int, n: int, seed=1, bad_every=0):
    """T valid tuples of n pairs in closed form (module docstring); with bad_every > 0 every bad_every-th tuple gets its
    successor's signature (VERIFY_FAIL)."""
    msgs = _msgs(f"scale {seed} {n}", n)
    hs = _pool_map(lambda m: _h2g2(O, m), msgs)
    A, B, suffix = None, None, None
    for j in range(n - 1, -1, -1):   # B = sum_j j H(m_j) = sum over j >= 1 of the suffix sums
        suffix = ac.G2.add(suffix, hs[j])
        if j >= 1:
            B = ac.G2.add(B, suffix)
    A = suffix
    a, d = _sk(b"scale a %d" % seed) % (R // 2), 1 + _sk(b"scale d %d" % seed) % 1000
    cur = ac.G2.add(ac.G2.mul(A, a), ac.G2.mul(B, d) if B is not None else None)

    def keys(t):
        out = C.create_string_buffer(48 * n)
        O.orc_pk_sequence(_b32(a + t), _b32(d), n, out)
        return [out.raw[48 * j:48 * j + 48] for j in range(n)]
    pks = _pool_map(keys, range(T))
    sigs = []
    for t in range(T):
        sigs.append(bo.g2_compress(cur))
        cur = ac.G2.add(cur, A)
    out = [_tuple(f"scale {T}x{n} #{t}", pks[t], msgs, sigs[t], SUCCESS, "closed form") for t in range(T)]
    if bad_every:
        for t in range(bad_every - 1, T - 1, bad_every):
            out[t]["sig"], out[t]["want"], out[t]["why"] = sigs[t + 1], VERIFY_FAIL, "the next tuple's signature"
    return out


# -------------------------------------------------------------------------------------------------- batch layout
def flatten(tuples):
    """-> (flat keys, key offsets, messages, message groups, flat signatures) of one batch call."""
    koff, grp = [0], [0]
    for t in tuples:
        koff.append(koff[-1] + len(t["pks"]))
        grp.append(grp[-1] + len(t["msgs"]))
    return (b"".join(b"".join(t["pks"]) for t in tuples), koff, [m for t in tuples for m in t["msgs"]], grp,
            b"".join(t["sig"] for t in tuples))


# -------------------------------------------------------------------------------------------------- fold layouts
def fold_levels(lengths):
    """Python model of the device's segmented product plan (capi_bls.cu plan_fold, no skip): [(n_in, pieces per segment)]
    per level; the last level leaves every segment in at most two pieces."""
    off = [0]
    for L in lengths:
        off.append(off[-1] + L)
    levels = []
    while True:
        pieces = [((off[t + 1] - 1) // 32 - off[t] // 32 + 1) if off[t + 1] > off[t] else 0 for t in range(len(lengths))]
        levels.append((off[-1], pieces))
        if max(pieces, default=0) <= 2:
            return levels
        off = [0]
        for p in pieces:
            off.append(off[-1] + p)


def segment_layouts(seed=1):
    """Segment length lists for the device fold: many short segments per warp, segments across warp (32) and CTA (64)
    boundaries, empty and single-value segments, and one segment of thousands of values."""
    rnd = random.Random(0xF0 + seed)
    return {
        "short, packed": [rnd.randrange(0, 6) for _ in range(300)],
        "one value each": [1] * 97,
        "two values each": [2] * 70,
        "across warps and CTAs": [31, 33, 1, 63, 65, 0, 64, 32, 2, 127, 129, 3],
        "offset by one": [1, 32, 1, 64, 1, 96, 1, 31],
        "mixed": [rnd.choice((0, 1, 2, 3, 5, 17, 31, 32, 33, 40, 70, 200)) for _ in range(60)],
        "one long": [3001],
        "long after short": [1, 2, 3, 2049, 4, 0, 65],
    }
