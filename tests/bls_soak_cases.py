"""Case generators of the BLS parity soaks, shared by the CPU soak (tests/soak_parity.py: the host build of the .cuh
headers against the C oracle) and the device soak (tests/test_bls_device_soak_gpu.py: the CUDA kernels against the
same oracle).  Every generator draws from the caller's numpy Generator in a fixed order, so one seed gives one case list.
`O` is the C oracle (oracle/c/bls_oracle.c) loaded through ctypes."""
from __future__ import annotations

import hashlib

import numpy as np

P = 0x1a0111ea397fe69a4b1ba7b6434bacd764774b84f38512bf6730d2a0f6b0f6241eabfffeb153ffffb9feffffffffaaab
R = 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001
N_MUTATIONS = 9
N_TUPLE_KINDS = 8


def valid_keys(O, n, seed=1):
    """n valid public keys pk_i = (sk0 + i d) g1; returns (keys uint8[n, 48], sk0, d)."""
    keys = np.empty((n, 48), dtype=np.uint8)
    sk0 = int.from_bytes(hashlib.sha256(b"soak/sk0%d" % seed).digest(), "big") % R
    d = int.from_bytes(hashlib.sha256(b"soak/d%d" % seed).digest(), "big") % R
    O.orc_pk_sequence(sk0.to_bytes(32, "big"), d.to_bytes(32, "big"), n, keys.ctypes.data)
    return keys, sk0, d


def sig_secret(i):
    """Secret key of valid_sigs' signature i (its message is sig_message(i))."""
    return (int.from_bytes(hashlib.sha256(b"soak/ssk%d" % i).digest(), "big") % (R - 1)) + 1


def sig_message(i):
    return hashlib.sha256(b"soak/m%d" % i).digest()


def valid_sigs(O, n):
    """n valid signatures: signature i is sig_secret(i) * H(sig_message(i))."""
    sks = np.frombuffer(b"".join(sig_secret(i).to_bytes(32, "big") for i in range(n)), dtype=np.uint8).copy()
    msgs = np.frombuffer(b"".join(sig_message(i) for i in range(n)), dtype=np.uint8).copy()
    out = np.empty((n, 96), dtype=np.uint8)
    O.orc_sign_batch(sks.ctypes.data, msgs.ctypes.data, n, out.ctypes.data, 8)
    return out


def mutate(enc: bytes, width: int, k: int, rng) -> bytes:
    """One of N_MUTATIONS corruptions of a compressed point (width 48: G1, 96: G2); kind 8 draws from `rng`."""
    b = bytearray(enc)
    if k == 0: b[0] ^= 0x20                                    # other y
    elif k == 1: b[0] ^= 0x40                                  # infinity flag on a finite point
    elif k == 2: b[0] &= 0x7f                                  # compression bit cleared
    elif k == 3:                                               # non-canonical x (first coordinate) = x + p if it fits
        hi = int.from_bytes(b[:48], "big") & ((1 << 381) - 1)
        if hi + P < (1 << 381):
            b[:48] = ((hi + P) | (b[0] >> 5 << 381)).to_bytes(48, "big")
    elif k == 4: b[-1] ^= 1                                    # neighbouring x
    elif k == 5: b = bytearray([0xc0] + [0] * (width - 2) + [1])  # infinity with junk
    elif k == 6: b = bytearray([0xc0] + [0] * (width - 1))     # the point at infinity
    elif k == 7: b = bytearray([0xe0] + [0] * (width - 1))     # infinity with the sign bit
    elif k == 8: b[rng.integers(0, width)] ^= 1 << int(rng.integers(0, 8))
    return bytes(b)


def random_g1_encodings(rng, n):
    """n compressed, finite G1 encodings with random x < 2^381: about half are on the curve, few in the subgroup."""
    rnd = rng.integers(0, 256, (n, 48), dtype=np.uint8)
    rnd[:, 0] = ((rnd[:, 0] & 0x3f) | 0x80) & 0xbf
    return rnd


def random_g2_encodings(rng, n):
    """n compressed, finite G2 encodings with random x.c1 < 2^381 and x.c0 < 2^381 (about 80 % of those are < p)."""
    rnd = rng.integers(0, 256, (n, 96), dtype=np.uint8)
    rnd[:, 0] = ((rnd[:, 0] & 0x3f) | 0x80) & 0xbf
    rnd[:, 48] &= 0x1f
    return rnd


def edge_x_values():
    """x values where decoders go wrong: 0, 1, p - 1, p, p + 1, 2^381 - 1, 2^380, and x + p for small x (still < 2^381)."""
    return [0, 1, 2, P - 1, P, P + 1, P + 2, (1 << 381) - 1, (1 << 380), (1 << 381) - 1 - P]


def g1_edge_encodings(valid):
    """Every flag-bit combination on the edge x values and on x + p of a few valid keys."""
    out = []
    xs = edge_x_values() + [(int.from_bytes(bytes(v), "big") & ((1 << 381) - 1)) + P for v in valid]
    for x in xs:
        if x >= 1 << 381:
            continue
        for flags in range(8):
            out.append(((flags << 381) | x).to_bytes(48, "big"))
    return out


def g2_edge_encodings(valid):
    """The same for G2: the edge x values in each coordinate (the other one 0 or taken from a valid signature)."""
    out = []
    for v in valid:
        c1 = int.from_bytes(bytes(v[:48]), "big") & ((1 << 381) - 1)
        c0 = int.from_bytes(bytes(v[48:]), "big")
        for x in edge_x_values() + [c1 + P]:
            if x >= 1 << 381:
                continue
            for flags in range(8):
                out.append(((flags << 381) | x).to_bytes(48, "big") + c0.to_bytes(48, "big"))
                out.append(((flags << 381) | c1).to_bytes(48, "big") + x.to_bytes(48, "big"))
        if c0 + P < 1 << 384:
            out.append(bytes(v[:48]) + (c0 + P).to_bytes(48, "big"))
    for x in edge_x_values():
        if x < 1 << 381:
            for flags in range(8):
                out.append(((flags << 381) | x).to_bytes(48, "big") + bytes(48))
    return out


def tuple_case(keys, sk0, d, t, rng, K=None):
    """Small fast_aggregate_verify tuple t of the soak, kind t % N_TUPLE_KINDS: 0 valid, 1 wrong signer set, 2 wrong
    message, 3 infinity key, 4 P and -P, 5 infinity signature, 6 mutated signature, 7 mutated key.  keys[i] must be
    (sk0 + i d) g1.  Returns the tuple before signing: sign `sign_msg` with `sk`, then pass the signature to finish_tuple."""
    if K is None:
        K = int(rng.integers(1, 9))
    idx = rng.integers(0, len(keys), K)
    msg = hashlib.sha256(b"soak/t%d" % t).digest()
    s = sum((sk0 + int(i) * d) % R for i in idx) % R
    kind = t % N_TUPLE_KINDS
    if kind == 1: s = (s + 1) % R                              # wrong signer set
    pks = bytearray(keys[idx].tobytes())
    sig_mut = None
    if kind == 3: pks[0:48] = mutate(bytes(pks[0:48]), 48, 6, rng)  # infinity key
    if kind == 4 and K >= 2:                                   # P and -P
        pks[48:96] = mutate(bytes(pks[0:48]), 48, 0, rng)
    if kind == 5: sig_mut = (6, None)                          # infinity signature
    if kind == 6:
        k = int(rng.integers(0, N_MUTATIONS))
        sig_mut = (k, rng.integers(0, 96) if k == 8 else None, int(rng.integers(0, 8)) if k == 8 else None)
    if kind == 7: pks[0:48] = mutate(bytes(pks[0:48]), 48, int(rng.integers(0, N_MUTATIONS)), rng)
    return {"kind": kind, "K": K, "pks": bytes(pks), "msg": msg, "sk": (s if s else 1).to_bytes(32, "big"),
            "sign_msg": msg if kind != 2 else hashlib.sha256(msg).digest(), "sig_mut": sig_mut}


def finish_tuple(case, sig: bytes) -> bytes:
    """The tuple's signature from the one made over case["sign_msg"] with case["sk"]."""
    m = case["sig_mut"]
    if m is None:
        return sig
    if m[0] == 8:
        b = bytearray(sig)
        b[m[1]] ^= 1 << m[2]
        return bytes(b)
    return mutate(sig, 96, m[0], None)
