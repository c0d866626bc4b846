"""GPU: the adversarial BLS parity soak through the CUDA kernels, case by case against the C oracle.

tests/soak_parity.py runs the same generators (tests/bls_soak_cases.py) through the g++ build of the .cuh headers; the
device build differs (inline-PTX products at ptxas -O1, carry-chain asm, Kaliski inverse, the shared-memory pow table,
register caps), and the per-tuple G1 sum, the G2 sum and the two-launch hash_to_G2 have no host build at all.  Here every
case goes through the kernels and its code (and, where there is one, its output bytes) is compared with the oracle's.

Sections: a. key validation, b. signature decode + subgroup check, c. hash_to_G2 by verdict, d. equal / opposite points
meeting in the aggregation lanes and trees, e. whole tuples (plain, chunked, RLC).  B200_G1_VARIANT, B200_PAIRING_VM and
B200_G1_SMALL_N are read once per process, so sections a, d and e run again in one child process per setting; with
B200_G1_SMALL_N=0 every key of those sections goes through the role-split per-key kernel, not only the tiled loads.

    B200_SOAK_SCALE=1 (default) python -m pytest tests/test_bls_device_soak_gpu.py -m gpu -s
"""
from __future__ import annotations

import hashlib
import os
import pickle
import subprocess
import sys
import time
from collections import Counter
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from tests import bls_soak_cases as sc  # noqa: E402

pytestmark = pytest.mark.gpu
SCALE = float(os.environ.get("B200_SOAK_SCALE", "1"))
SMALL_N = 3 * 148 * 384          # bls_g1.cu g_g1_small_n: up to here the per-key kernel goes out as 128-thread CTAs
RLC_SEED = hashlib.sha256(b"device soak rlc").digest()
# the last: every per-key launch through the role-split kernel (k_g1_validate_split), whatever its size
ENV_VARIANTS = [{"B200_G1_VARIANT": "0", "B200_PAIRING_VM": "1"}, {"B200_G1_VARIANT": "6", "B200_PAIRING_VM": "1"},
                {"B200_G1_VARIANT": "7", "B200_PAIRING_VM": "0"},
                {"B200_G1_VARIANT": "7", "B200_PAIRING_VM": "1", "B200_G1_SMALL_N": "0"}]


def _env_id(e):
    small = "-small_n_%s" % e["B200_G1_SMALL_N"] if "B200_G1_SMALL_N" in e else ""
    return "g1_variant_%s-vm_%s%s" % (e["B200_G1_VARIANT"], e["B200_PAIRING_VM"], small)


def _n(x):
    return max(1, int(x * SCALE))


def _min(x):
    """Minimum case count a section must reach at this scale (the issue's counts at scale 1)."""
    return max(50, int(x * min(SCALE, 1.0)))


# ---------------------------------------------------------------------------------------------------------- helpers
def report(name, want, got):
    """Compares case by case, prints one summary line like the CPU soak, returns (cases, mismatches)."""
    want, got = list(want), list(got)
    assert len(want) == len(got), (name, len(want), len(got))
    bad = [i for i, (w, g) in enumerate(zip(want, got)) if w != g]
    hist = Counter((w[0] if isinstance(w, tuple) else w) for w in want)
    h = ", ".join(f"{c}: {k}" for c, k in sorted(hist.items(), key=lambda kv: str(kv[0])))
    print(f"{name:44s} cases {len(want):6d}  mismatches {len(bad)}   verdict histogram {{{h}}}")
    sys.stdout.flush()
    if bad:
        i = bad[0]
        print(f"  first mismatch: case {i}: oracle {want[i]!r}, device {got[i]!r}")
    return len(want), len(bad)


def _neg(enc: bytes) -> bytes:
    b = bytearray(enc)
    b[0] ^= 0x20
    return bytes(b)


def _pack(tuples):
    """[(pks bytes, msg32, sig96)] -> the batch entry points' flat arrays."""
    pks = np.frombuffer(b"".join(t[0] for t in tuples), dtype=np.uint8)
    off = np.cumsum([0] + [len(t[0]) // 48 for t in tuples]).astype(np.uint32)
    msgs = np.frombuffer(b"".join(t[1] for t in tuples), dtype=np.uint8)
    sigs = np.frombuffer(b"".join(t[2] for t in tuples), dtype=np.uint8)
    return pks, off, msgs, sigs


def _oracle_batch(O, tuples):
    pks, off, msgs, sigs = (np.ascontiguousarray(a) for a in _pack(tuples))
    out = np.empty(max(len(tuples), 1), dtype=np.int32)
    O.orc_fast_aggregate_verify_batch(pks.ctypes.data if pks.size else 0, off.ctypes.data, msgs.ctypes.data, sigs.ctypes.data,
                                      len(tuples), out.ctypes.data, 8)
    return out[:len(tuples)].tolist()


def _sign_batch(O, sks, msgs):
    s = np.frombuffer(b"".join(sks), dtype=np.uint8).copy()
    m = np.frombuffer(b"".join(msgs), dtype=np.uint8).copy()
    out = np.empty((len(sks), 96), dtype=np.uint8)
    O.orc_sign_batch(s.ctypes.data, m.ctypes.data, len(sks), out.ctypes.data, 8)
    return [bytes(r) for r in out]


def _code(fn, *a):
    from ethereum_consensus_b200 import crypto
    try:
        r = fn(*a)
        return (0, bytes(r)) if r is not None else 0
    except crypto.InvalidSignature:
        return 5
    except crypto.BLSTError as e:
        return e.code


def _oracle_bytes(fn, data, n, width):
    import ctypes as C
    buf = C.create_string_buffer(width)
    rc = fn(data, n, buf)
    return (0, buf.raw) if rc == 0 else rc


def _sk(x):
    return (x % sc.R if x % sc.R else 1).to_bytes(32, "big")


# ---------------------------------------------------------------------------------------------------------- inputs
_CACHE = {}


def keys_data(O):
    """a. >= 20 000 G1 encodings with the oracle's key_validate codes, K = 1 tuples on valid keys and their negations,
    and single-key aggregations with the oracle's bytes."""
    if "keys" in _CACHE:
        return _CACHE["keys"]
    rng = np.random.default_rng(0xA1)
    n = _n(6000)
    keys, sk0, d = sc.valid_keys(O, n, seed=11)
    cases = [keys[i].tobytes() for i in range(n)]
    cases += [r.tobytes() for r in sc.random_g1_encodings(rng, _n(8000))]
    cases += [sc.mutate(keys[i % n].tobytes(), 48, i % sc.N_MUTATIONS, rng) for i in range(_n(6000))]
    cases += sc.g1_edge_encodings([keys[i] for i in range(8)])
    want = [O.orc_key_validate(c) for c in cases]
    m = min(n, _n(1000))
    tup = []
    sks, msgs = [], []
    for i in range(m):
        s = (sk0 + i * d) % sc.R
        for sign, pk in ((1, keys[i].tobytes()), (-1, _neg(keys[i].tobytes()))):
            msg = hashlib.sha256(b"dev/k%d/%d" % (i, sign)).digest()
            tup.append([pk, msg, None])
            sks.append(_sk(sign * s)); msgs.append(msg)
    for t, sg in zip(tup, _sign_batch(O, sks, msgs)):
        t[2] = sg
    tup = [tuple(t) for t in tup]
    one = [c for i, c in enumerate(cases) if i % max(1, len(cases) // 200) == 0] + [_neg(keys[i].tobytes()) for i in range(100)]
    one_want = [_oracle_bytes(O.orc_eth_aggregate_public_keys, c, 1, 48) for c in one]
    _CACHE["keys"] = {"cases": cases, "want": want, "tuples": tup, "tuples_want": _oracle_batch(O, tup), "one": one, "one_want": one_want}
    return _CACHE["keys"]


def sigs_data(O):
    """b. >= 8 000 G2 encodings with the oracle's aggregate([sig]) result, and K = 1 tuples that carry them."""
    rng = np.random.default_rng(0xB2)
    n = _n(1500)
    sigs = sc.valid_sigs(O, n)
    cases = [sigs[i].tobytes() for i in range(n)]
    cases += [r.tobytes() for r in sc.random_g2_encodings(rng, _n(4000))]
    cases += [sc.mutate(sigs[i % n].tobytes(), 96, i % sc.N_MUTATIONS, rng) for i in range(_n(2500))]
    cases += sc.g2_edge_encodings([sigs[i] for i in range(4)])
    want = [_oracle_bytes(O.orc_aggregate, c, 1, 96) for c in cases]
    import ctypes as C
    pk = C.create_string_buffer(48)
    pks = []
    for i in range(n):
        O.orc_sk_to_pk(sc.sig_secret(i).to_bytes(32, "big"), pk)
        pks.append(pk.raw)
    tup = [(pks[j % n], sc.sig_message(j % n), c) for j, c in enumerate(cases)]
    return {"cases": cases, "want": want, "tuples": tup, "tuples_want": _oracle_batch(O, tup)}


def h2c_data(O):
    """c. messages of every length 0..300 (all SHA-256 padding edges) and random longer ones, signed by one key."""
    import ctypes as C
    rng = np.random.default_rng(0xC3)
    sk = sc.sig_secret(10_000).to_bytes(32, "big")
    pk = C.create_string_buffer(48)
    O.orc_sk_to_pk(sk, pk)
    lens = list(range(0, 301)) + [int(x) for x in rng.integers(301, 2048, _n(40))]
    msgs = [rng.integers(0, 256, ln, dtype=np.uint8).tobytes() for ln in lens]
    sig = C.create_string_buffer(96)
    sigs = []
    for m in msgs:
        O.orc_sign(sk, m, len(m), sig)
        sigs.append(sig.raw)
    # one batch of 32-byte roots (every fifth one signed over a different root)
    nb = max(4096, _n(4096))
    keys, sk0, d = sc.valid_keys(O, 64, seed=12)
    roots = [hashlib.sha256(b"dev/h%d" % t).digest() for t in range(nb)]
    sign_roots = [r if t % 5 else hashlib.sha256(r).digest() for t, r in enumerate(roots)]
    bsig = _sign_batch(O, [_sk(sk0 + (t % 64) * d) for t in range(nb)], sign_roots)
    btup = [(keys[t % 64].tobytes(), roots[t], bsig[t]) for t in range(nb)]
    # aggregate_verify over many messages of mixed lengths
    na = 64
    am = [rng.integers(0, 256, (i * 47) % 301, dtype=np.uint8).tobytes() for i in range(na)]
    apk = []
    asig = b""
    for i in range(na):
        s = sc.sig_secret(20_000 + i).to_bytes(32, "big")
        O.orc_sk_to_pk(s, pk)
        apk.append(pk.raw)
        O.orc_sign(s, am[i], len(am[i]), sig)
        asig += sig.raw
    agg = _oracle_bytes(O.orc_aggregate, asig, na, 96)[1]
    flipped = list(am); flipped[17] = bytes([flipped[17][0] ^ 1]) + flipped[17][1:]
    swapped = list(apk); swapped[3], swapped[40] = swapped[40], swapped[3]
    av = [(apk, am, agg), (apk, flipped, agg), (swapped, am, agg), (apk[:-1], am[:-1], agg)]
    av_want = []
    for pks_, ms_, sg_ in av:
        arr = (C.c_char_p * len(ms_))(*ms_)
        ln = (C.c_size_t * len(ms_))(*[len(m) for m in ms_])
        av_want.append(O.orc_aggregate_verify(b"".join(pks_), len(pks_), C.cast(arr, C.c_void_p), C.cast(ln, C.c_void_p), len(ms_), sg_))
    O.orc_sk_to_pk(sk, pk)
    return {"key": pk.raw, "msgs": msgs, "sigs": sigs, "batch": btup, "batch_want": _oracle_batch(O, btup), "av": av, "av_want": av_want}


def _shapes():
    """Multisets of key indices (index, sign) that make equal or opposite points meet in k_g1_aggregate's lanes (lane j sums
    positions j, j + 32, ...) and in its 5-level tree (level s adds lane j + s into lane j), and in k_g2_sum_compress."""
    out = []
    for K in (2, 32, 33, 64, 512, 2048):
        out.append((f"[P] * {K}", [(7, 1)] * K))
    for i in (0, 5, 31):                                     # mixed-add doubling inside one lane
        s = [(100 + j, 1) for j in range(64)]; s[i + 32] = s[i]
        out.append((f"P at {i} and {i + 32}", s))
    for K, i in ((32, 0), (32, 3), (32, 15), (16, 2), (8, 1), (4, 0), (2, 0), (48, 7)):   # equal partial sums at each tree level
        h = K // 2 if K <= 32 else 16
        s = [(200 + j, 1) for j in range(K)]; s[i + h] = s[i]
        out.append((f"P at {i} and {i + h} (K {K})", s))
    for k in (0, 9, 31):                                     # a whole lane sums to infinity
        s = [(300 + j, 1) for j in range(64)]; s[k + 32] = (s[k][0], -1)
        out.append((f"P at {k}, -P at {k + 32}", s))
    for K, i in ((32, 0), (32, 11), (16, 3), (8, 0), (4, 1), (2, 0)):   # the tree cancels
        h = K // 2
        s = [(400 + j, 1) for j in range(K)]; s[i + h] = (s[i][0], -1)
        out.append((f"P at {i}, -P at {i + h} (K {K})", s))
    s = [(500 + j, 1) for j in range(32)]; s[8] = (s[0][0], -1); s[24] = (s[16][0], -1)   # lanes 0 and 8 cancel at level 8
    out.append(("lanes 0+16 and 8+24 cancel", s))
    s = [(600 + j, 1) for j in range(64)]
    for j in range(32):
        s[j + 32] = (s[j][0], -1)
    out.append(("every lane cancels", s))
    for K, pos in ((64, 20), (33, 32), (2048, 1000), (32, 0)):   # all keys equal except one
        s = [(7, 1)] * K; s[pos] = (700 + pos, 1)
        out.append((f"all equal but one (K {K}, at {pos})", s))
    return out


def shapes_data(O):
    """d. the shapes as key multisets (tuples signed with the sum of the secrets) and as signature multisets."""
    if "shapes" in _CACHE:
        return _CACHE["shapes"]
    keys, sk0, d = sc.valid_keys(O, 1800, seed=13)
    shapes = _shapes()
    enc = lambda i, g: keys[i].tobytes() if g > 0 else _neg(keys[i].tobytes())   # noqa: E731
    tup, sks, msgs = [], [], []
    for t, (name, s) in enumerate(shapes):
        secret = sum(g * (sk0 + i * d) for i, g in s)
        msg = hashlib.sha256(b"dev/shape%d" % t).digest()
        tup.append([b"".join(enc(i, g) for i, g in s), msg, None])
        sks.append(_sk(secret)); msgs.append(msg)
    for t, sg in zip(tup, _sign_batch(O, sks, msgs)):
        t[2] = sg
    tup = [tuple(t) for t in tup]
    agg_want = [_oracle_bytes(O.orc_eth_aggregate_public_keys, t[0], len(t[0]) // 48, 48) for t in tup]
    # signatures: S_i = sig_secret(i) * H(m0); the same index patterns
    ids = sorted({i for _, s in shapes for i, _ in s})
    m0 = hashlib.sha256(b"dev/shape sigs").digest()
    S = dict(zip(ids, _sign_batch(O, [sc.sig_secret(i).to_bytes(32, "big") for i in ids], [m0] * len(ids))))
    sig_sets = [b"".join(S[i] if g > 0 else _neg(S[i]) for i, g in s) for _, s in shapes]
    sig_want = [_oracle_bytes(O.orc_aggregate, f, len(f) // 96, 96) for f in sig_sets]
    uniq = sorted({p for t in tup for p in (t[0][48 * j: 48 * j + 48] for j in range(len(t[0]) // 48))})
    _CACHE["shapes"] = {"names": [n for n, _ in shapes], "tuples": tup, "want": _oracle_batch(O, tup), "agg_want": agg_want,
                        "sig_sets": sig_sets, "sig_want": sig_want, "uniq": uniq}
    return _CACHE["shapes"]


def tuples_data(O):
    """e. the soak's eight small-K kinds, plus K in {31, 32, 33, 64, 65, 512}, in one batch."""
    if "tuples" in _CACHE:
        return _CACHE["tuples"]
    rng = np.random.default_rng(0xE5)
    keys, sk0, d = sc.valid_keys(O, 1024, seed=14)
    cases = [sc.tuple_case(keys, sk0, d, t, rng) for t in range(_n(3000))]
    t0 = len(cases)
    for K in (31, 32, 33, 64, 65, 512):
        for j in range(sc.N_TUPLE_KINDS):
            cases.append(sc.tuple_case(keys, sk0, d, t0, rng, K=K))
            t0 += 1
    sigs = _sign_batch(O, [c["sk"] for c in cases], [c["sign_msg"] for c in cases])
    tup = [(c["pks"], c["msg"], sc.finish_tuple(c, s)) for c, s in zip(cases, sigs)]
    _CACHE["tuples"] = {"tuples": tup, "kind": [c["kind"] for c in cases], "K": [c["K"] for c in cases], "want": _oracle_batch(O, tup)}
    return _CACHE["tuples"]


# ---------------------------------------------------------------------------------------------------------- device checks
def check_keys(D, tag=""):
    """Returns [(section, cases, mismatches)]."""
    from ethereum_consensus_b200 import crypto
    res = []
    flat = np.frombuffer(b"".join(D["cases"]), dtype=np.uint8)
    res.append(("a. key_validate, 128-thread CTAs" + tag, *report("a. key_validate (registry, n <= %d)%s" % (SMALL_N, tag), D["want"],
                                                                  crypto.Registry(flat).key_codes().tolist())))
    reps = SMALL_N // len(D["cases"]) + 2
    big = np.tile(flat, reps)
    got = crypto.Registry(big).key_codes().tolist()
    res.append(("a. key_validate, tiled" + tag, *report(f"a. key_validate (registry, n = {len(got)}){tag}", D["want"] * reps, got)))
    got = crypto.fast_aggregate_verify_batch(*_pack(D["tuples"])).tolist()
    res.append(("a. decoded keys, K = 1" + tag, *report("a. P and -P, K = 1 strict batch" + tag, D["tuples_want"], got)))
    got = [_code(crypto.eth_aggregate_public_keys, [c]) for c in D["one"]]
    res.append(("a. recompression" + tag, *report("a. eth_aggregate_public_keys([pk])" + tag, D["one_want"], got)))
    return res


def check_shapes(D, rlc, tag=""):
    from ethereum_consensus_b200 import crypto
    res = []
    tup, want = D["tuples"], D["want"]
    res.append(("d. strict batch" + tag, *report("d. shapes: strict batch" + tag, want, crypto.fast_aggregate_verify_batch(*_pack(tup)).tolist())))
    uniq = D["uniq"]
    pos = {p: i for i, p in enumerate(uniq)}
    idx = np.array([pos[t[0][48 * j: 48 * j + 48]] for t in tup for j in range(len(t[0]) // 48)], dtype=np.uint32)
    _, off, msgs, sigs = _pack(tup)
    reg = crypto.Registry(np.frombuffer(b"".join(uniq), dtype=np.uint8))
    res.append(("d. registry" + tag, *report("d. shapes: registry verify_batch" + tag, want, reg.verify_batch(idx, off, msgs, sigs).tolist())))
    half = len(uniq) // 2                                     # the second half arrive as extra keys
    order = uniq[half:] + uniq[:half]
    pos2 = {p: i for i, p in enumerate(order)}
    idx2 = np.array([pos2[t[0][48 * j: 48 * j + 48]] for t in tup for j in range(len(t[0]) // 48)], dtype=np.uint32)
    reg = crypto.Registry(np.frombuffer(b"".join(order[:len(uniq) - half]), dtype=np.uint8))
    extra = np.frombuffer(b"".join(order[len(uniq) - half:]), dtype=np.uint8)
    res.append(("d. mixed" + tag, *report("d. shapes: _batch_mixed" + tag, want, reg.verify_batch(idx2, off, msgs, sigs, extra_keys=extra).tolist())))
    got = [_code(crypto.eth_aggregate_public_keys, [t[0][48 * j: 48 * j + 48] for j in range(len(t[0]) // 48)]) for t in tup]
    res.append(("d. eth_aggregate_public_keys" + tag, *report("d. shapes: eth_aggregate_public_keys" + tag, D["agg_want"], got)))
    got = [_code(crypto.aggregate, [f[96 * j: 96 * j + 96] for j in range(len(f) // 96)]) for f in D["sig_sets"]]
    res.append(("d. aggregate (signatures)" + tag, *report("d. shapes: aggregate(signatures)" + tag, D["sig_want"], got)))
    if rlc:
        ok = [t for t, w in zip(tup, want) if w == 0]
        got = [crypto.fast_aggregate_verify_batch_all(*_pack(tup), seed=RLC_SEED), crypto.fast_aggregate_verify_batch_all(*_pack(ok), seed=RLC_SEED)]
        res.append(("d. RLC" + tag, *report("d. shapes: fast_aggregate_verify_batch_all" + tag, [all(w == 0 for w in want), True], got)))
    return res


def check_tuples(D, rlc, tag=""):
    from ethereum_consensus_b200 import crypto
    res = []
    tup, want = D["tuples"], D["want"]
    args = _pack(tup)
    res.append(("e. strict batch" + tag, *report("e. tuples: strict batch" + tag, want, crypto.fast_aggregate_verify_batch(*args).tolist())))
    try:
        crypto.tune("bls_chunks", 5); crypto.tune("bls_chunk_min_tuples", 2)
        got = crypto.fast_aggregate_verify_batch(*args).tolist()
    finally:
        crypto.tune("bls_chunks", 1); crypto.tune("bls_chunk_min_tuples", 2048)
    res.append(("e. chunked" + tag, *report("e. tuples: 5 chunks" + tag, want, got)))
    if rlc:
        ok = [t for t, w in zip(tup, want) if w == 0]
        wants, gots = [True], [crypto.fast_aggregate_verify_batch_all(*_pack(ok), seed=RLC_SEED)]
        for kind in range(1, sc.N_TUPLE_KINDS):
            bad = next((t for t, w, k in zip(tup, want, D["kind"]) if k == kind and w != 0), None)
            if bad is not None:
                wants.append(False)
                gots.append(crypto.fast_aggregate_verify_batch_all(*_pack(ok[:40] + [bad] + ok[40:80]), seed=RLC_SEED))
        res.append(("e. RLC" + tag, *report("e. tuples: batch_all, valid and each class" + tag, wants, gots)))
    return res


def _assert_clean(res, minimum=None):
    for name, n, bad in res:
        assert bad == 0, f"{name}: {bad} of {n} cases differ from the oracle"
        if minimum:
            assert n >= minimum.get(name, 1), (name, n)


# ---------------------------------------------------------------------------------------------------------- tests
def test_a_key_validation(engine, oracle_bls_c):
    t = time.time()
    D = keys_data(oracle_bls_c)
    res = check_keys(D)
    print(f"a. wall {time.time() - t:.1f} s")
    _assert_clean(res, {"a. key_validate, 128-thread CTAs": _min(20_000), "a. key_validate, tiled": SMALL_N,
                        "a. decoded keys, K = 1": _min(2000), "a. recompression": _min(300)})


def test_b_signature_decode_and_subgroup(engine, oracle_bls_c):
    from ethereum_consensus_b200 import crypto
    t = time.time()
    D = sigs_data(oracle_bls_c)
    res = [("b. aggregate([sig])", *report("b. aggregate([sig]): code + 96 bytes", D["want"], [_code(crypto.aggregate, [c]) for c in D["cases"]]))]
    args = _pack(D["tuples"])
    try:
        for cta in (32, 128):
            crypto.tune("bls_small_cta", cta)
            res.append((f"b. batch, small CTA {cta}", *report(f"b. K = 1 batch, bls_small_cta {cta}", D["tuples_want"],
                                                              crypto.fast_aggregate_verify_batch(*args).tolist())))
    finally:
        crypto.tune("bls_small_cta", 0)
    print(f"b. wall {time.time() - t:.1f} s")
    _assert_clean(res, {"b. aggregate([sig])": _min(8000)})
    hist = Counter(w[0] if isinstance(w, tuple) else w for w in D["want"])
    assert hist[0] and hist[3] and hist[1] and hist[2], hist      # every decode outcome, and "not in subgroup", is present


def test_c_hash_to_g2(engine, oracle_bls_c):
    from ethereum_consensus_b200 import crypto
    t = time.time()
    D = h2c_data(oracle_bls_c)
    pk = D["key"]
    ok = [_code(crypto.verify_signature, pk, m, s) for m, s in zip(D["msgs"], D["sigs"])]
    res = [("c. verify_signature, lengths 0..300+", *report("c. verify_signature, message lengths 0..300 + random", [0] * len(ok), ok))]
    flips, fw = [], []
    rng = np.random.default_rng(0xC4)
    for m, s in zip(D["msgs"], D["sigs"]):
        if not m:
            continue
        b = bytearray(m)
        b[int(rng.integers(0, len(b)))] ^= 1 << int(rng.integers(0, 8))
        flips.append(_code(crypto.verify_signature, pk, bytes(b), s))
        fw.append(oracle_bls_c.orc_verify_signature(pk, bytes(b), len(b), s))
    res.append(("c. one bit flipped", *report("c. verify_signature, one message bit flipped", fw, flips)))
    assert set(fw) == {5}
    res.append(("c. batch of 32-byte roots", *report("c. strict batch of 32-byte roots", D["batch_want"],
                                                     crypto.fast_aggregate_verify_batch(*_pack(D["batch"])).tolist())))
    got = [_code(crypto.aggregate_verify, p, m, s) for p, m, s in D["av"]]
    res.append(("c. aggregate_verify", *report("c. aggregate_verify, 64 messages of mixed lengths", D["av_want"], got)))
    assert D["av_want"][0] == 0 and D["av_want"][1] == 5
    print(f"c. wall {time.time() - t:.1f} s")
    _assert_clean(res, {"c. verify_signature, lengths 0..300+": 301, "c. batch of 32-byte roots": 4096})


def test_d_aggregation_edge_cases(engine, oracle_bls_c):
    t = time.time()
    D = shapes_data(oracle_bls_c)
    res = check_shapes(D, rlc=True)
    print(f"d. wall {time.time() - t:.1f} s")
    _assert_clean(res, {"d. strict batch": 30})
    assert 0 in D["want"] and any(w != 0 for w in D["want"])   # both verdicts occur among the shapes


def test_e_whole_tuples(engine, oracle_bls_c):
    t = time.time()
    D = tuples_data(oracle_bls_c)
    res = check_tuples(D, rlc=True)
    print(f"e. wall {time.time() - t:.1f} s")
    _assert_clean(res, {"e. strict batch": _min(3000)})
    assert len(set(D["want"])) >= 4


@pytest.mark.parametrize("env", ENV_VARIANTS, ids=_env_id)
def test_env_variants_in_child_processes(oracle_bls_c, tmp_path, env):
    """Sections a, d and e under a per-key kernel variant / the one-thread-per-pair pairing kernels, which only the
    environment selects (read once per process): one child process per setting, inputs and oracle verdicts from here."""
    t = time.time()
    data = {"keys": keys_data(oracle_bls_c), "shapes": shapes_data(oracle_bls_c), "tuples": tuples_data(oracle_bls_c)}
    path = tmp_path / "soak.pkl"
    path.write_bytes(pickle.dumps(data))
    child_env = dict(os.environ, **env)
    p = subprocess.Popen([sys.executable, "-m", "tests.test_bls_device_soak_gpu", str(path)], cwd=str(ROOT), env=child_env,
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    try:
        out = p.communicate(timeout=1200)[0]
    except subprocess.TimeoutExpired:
        p.kill()
        out = p.communicate()[0]
    print(out)
    print(f"child {env} wall {time.time() - t:.1f} s")
    assert p.returncode == 0, out
    assert "CHILD_OK" in out, out


def _child(path):
    from ethereum_consensus_b200 import _lib
    _lib.init(0)
    data = pickle.loads(Path(path).read_bytes())
    rlc = os.environ.get("B200_PAIRING_VM", "1") != "0"     # the RLC entry points refuse the one-thread-per-pair kernels
    tag = " [G1 %s, VM %s, small n %s]" % (os.environ.get("B200_G1_VARIANT", "7"), os.environ.get("B200_PAIRING_VM", "1"),
                                          os.environ.get("B200_G1_SMALL_N", "default"))
    res = check_keys(data["keys"], tag) + check_shapes(data["shapes"], rlc, tag) + check_tuples(data["tuples"], rlc, tag)
    _assert_clean(res)
    print("CHILD_OK")


if __name__ == "__main__":
    _child(sys.argv[1])
