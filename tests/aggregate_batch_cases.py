"""Seeded groups for aggregate / eth_aggregate_public_keys over T groups per call, shared by the CPU check
(tests/test_aggregate_batch_cases.py) and the device run (tests/test_aggregate_batch_gpu.py).  No device code here.

Valid material is cheap when it comes in arithmetic progressions: with sk_i = a + i d,
    sig_i = sig_{i-1} + d H(m)   and   pk_i = pk_{i-1} + d g1,
one affine addition per member, and the aggregate of n members is (n a + d n (n - 1) / 2) H(m) (or g1) in closed form.
Every group carries its expected (code, bytes) where it is known by construction; the others are left to the oracles.
Group shapes: empty and single-member groups, members summing to infinity, infinity signatures, duplicates, decode and
group-check failures in either order at chunk boundaries (the device splits a group into chunks of a multiple of 32
signatures) and inside chunks, small- and mixed-order points from tests/torsion_cases.py, invalid keys of every kind."""
from __future__ import annotations

import hashlib
import random

from oracle import bls_oracle as bo

P, R = bo.P, bo.R
SUCCESS, BAD_ENCODING, NOT_ON_CURVE, NOT_IN_GROUP, PK_IS_INFINITY, EMPTY = 0, 1, 2, 3, 6, 16
INF_SIG = bytes([0xC0]) + bytes(95)
INF_PK = bytes([0xC0]) + bytes(47)


# ------------------------------------------------------------------------------------------------ affine arithmetic
def _f2_inv(a):
    t = pow((a[0] * a[0] + a[1] * a[1]) % P, -1, P)
    return (a[0] * t % P, (-a[1]) * t % P)


class _Aff:
    """Affine addition on E(Fp) or E'(Fp2) with one inversion (None = infinity)."""

    def __init__(self, F, inv):
        self.F, self.inv = F, inv

    def add(self, a, b):
        F = self.F
        if a is None:
            return b
        if b is None:
            return a
        if a[0] == b[0]:
            if F.add(a[1], b[1]) == F.zero:
                return None
            lam = F.mul(F.mul(F.sqr(a[0]), (3 if F is bo.F1 else (3, 0))), self.inv(F.add(a[1], a[1])))
        else:
            lam = F.mul(F.sub(b[1], a[1]), self.inv(F.sub(b[0], a[0])))
        x = F.sub(F.sub(F.sqr(lam), a[0]), b[0])
        return (x, F.sub(F.mul(lam, F.sub(a[0], x)), a[1]))

    def mul(self, a, k):
        return bo.pt_to_affine(self.F, bo.pt_mul(self.F, bo.pt_from_affine(self.F, a), k % R))

    def neg(self, a):
        return None if a is None else (a[0], self.F.neg(a[1]))


G1 = _Aff(bo.F1, lambda a: pow(a, -1, P))
G2 = _Aff(bo.F2, _f2_inv)


def progression(E, base, a, d, n):
    """[a + i d] base for i < n, by one addition each."""
    out, cur, step = [], E.mul(base, a), E.mul(base, d)
    for _ in range(n):
        out.append(cur)
        cur = E.add(cur, step)
    return out


def progression_sum(E, base, a, d, n):
    return E.mul(base, n * a + d * n * (n - 1) // 2)


def _scalar(tag: bytes) -> int:
    return int.from_bytes(hashlib.sha256(tag).digest(), "big") % R


# ------------------------------------------------------------------------------------------------ invalid encodings
def not_on_curve_g2(rnd):
    while True:
        b = bytearray(rnd.randbytes(96))
        b[0] = (b[0] & 0x1F) | 0x80
        if bo.g2_uncompress(bytes(b))[0] == NOT_ON_CURVE:
            return bytes(b)


def not_on_curve_g1(rnd):
    while True:
        b = bytearray(rnd.randbytes(48))
        b[0] = (b[0] & 0x1F) | 0x80
        if bo.g1_uncompress(bytes(b))[0] == NOT_ON_CURVE:
            return bytes(b)


def bad_encodings(width, rnd):
    """Each -> BAD_ENCODING: compression bit clear, infinity flag with a payload, x >= p (non-canonical)."""
    clear = bytes([rnd.randrange(0x80)]) + rnd.randbytes(width - 1)
    inf_payload = bytes([0xC0]) + bytes(width - 2) + b"\x01"
    big = bytearray((P + rnd.randrange(1, 1000)).to_bytes(48, "big") + rnd.randbytes(width - 48))
    big[0] |= 0x80
    return [clear, inf_payload, bytes(big)]


def small_order(torsion, n, rnd, valid=False):
    """n encodings from torsion_cases' list: code 3 (small or mixed order), or code 0 (the valid controls)."""
    pool = [c for c in torsion["cases"] if (c["code"] == SUCCESS) == valid and c["pt"] is not None]
    return [rnd.choice(pool)["enc"] for _ in range(n)]


# ------------------------------------------------------------------------------------------------ groups
def _group(name, items, want=None):
    return {"name": name, "items": list(items), "want": want}


def sig_groups(torsion_g2, seed=1):
    """Signature groups of one call: dicts name, items (96-byte encodings), want ((code, 96 bytes or None) or None)."""
    rnd = random.Random(0xA66 + seed)
    h = bo.hash_to_g2(b"aggregate batch %d" % seed)
    a, d = _scalar(b"agg sig a%d" % seed), 1 + _scalar(b"agg sig d%d" % seed) % 1000
    chain = progression(G2, h, a, d, 100)
    enc = [bo.g2_compress(p) for p in chain]
    ok = lambda pt: (SUCCESS, bo.g2_compress(pt))  # noqa: E731
    gs = [
        _group("empty", [], (EMPTY, None)),
        _group("single", enc[:1], ok(chain[0])),
        _group("chain of 5", enc[:5], ok(progression_sum(G2, h, a, d, 5))),
        _group("chain of 100", enc, ok(progression_sum(G2, h, a, d, 100))),
        _group("P, -P", [enc[7], bo.g2_compress(G2.neg(chain[7]))], (SUCCESS, INF_SIG)),
        _group("infinity alone", [INF_SIG], (SUCCESS, INF_SIG)),
        _group("infinity between", [enc[0], INF_SIG, enc[1], INF_SIG], ok(progression_sum(G2, h, a, d, 2))),
        _group("duplicates", [enc[3]] * 3, ok(G2.mul(chain[3], 3))),
        _group("duplicate pairs", [enc[3], enc[4], enc[3], enc[4]], ok(G2.mul(G2.add(chain[3], chain[4]), 2))),
        _group("empty again", [], (EMPTY, None)),
    ]
    # failures at chunk boundaries (31 | 32, 63 | 64) and inside chunks, in either order: decode errors always win, and the
    # first decode error in signature order decides between two of them
    bads = bad_encodings(96, rnd)
    for i, j in ((31, 32), (32, 31), (63, 64), (64, 63), (5, 17), (17, 5), (0, 99), (99, 0)):
        items = list(enc)
        items[i] = small_order(torsion_g2, 1, rnd)[0]
        items[j] = bads[(i + j) % 3]
        gs.append(_group(f"group-check at {i}, decode at {j}", items, (BAD_ENCODING, None)))
    for i, j in ((31, 32), (64, 40), (10, 90)):
        items = list(enc)
        items[i] = not_on_curve_g2(rnd)
        items[j] = bads[0]
        gs.append(_group(f"not on curve at {i}, bad encoding at {j}", items, (NOT_ON_CURVE if i < j else BAD_ENCODING, None)))
    for i in (0, 31, 32, 99):
        items = list(enc)
        items[i] = small_order(torsion_g2, 1, rnd)[0]
        gs.append(_group(f"small or mixed order at {i}", items, (NOT_IN_GROUP, None)))
    gs.append(_group("small or mixed order only", small_order(torsion_g2, 6, rnd), (NOT_IN_GROUP, None)))
    gs.append(_group("torsion controls", small_order(torsion_g2, 6, rnd, valid=True)))
    gs.append(_group("single bad encoding", bads[1:2], (BAD_ENCODING, None)))
    return gs


def key_pool(seed, n):
    """n valid keys pk_i = (a + i d) g1 (48-byte encodings) and their aggregate scalar parameters."""
    a, d = _scalar(b"agg pk a%d" % seed), 1 + _scalar(b"agg pk d%d" % seed) % 1000
    pts = progression(G1, bo.G1_GEN, a, d, n)
    return [bo.g1_compress(p) for p in pts], pts, a, d


def invalid_keys(torsion_g1, rnd):
    """(encoding, code): infinity, off the curve, outside G1 (small and mixed order), non-canonical / bad encodings."""
    out = [(INF_PK, PK_IS_INFINITY), (not_on_curve_g1(rnd), NOT_ON_CURVE)]
    out += [(e, NOT_IN_GROUP) for e in small_order(torsion_g1, 3, rnd)]
    out += [(e, BAD_ENCODING) for e in bad_encodings(48, rnd)]
    return out


def key_groups(torsion_g1, seed=1):
    """Key groups of one call, as sig_groups; the first failing key in order decides a group's code."""
    rnd = random.Random(0xB66 + seed)
    enc, pts, a, d = key_pool(seed, 100)
    ok = lambda pt: (SUCCESS, bo.g1_compress(pt))  # noqa: E731
    bad = invalid_keys(torsion_g1, rnd)
    gs = [
        _group("empty", [], (EMPTY, None)),
        _group("single", enc[:1], ok(pts[0])),
        _group("chain of 100", enc, ok(progression_sum(G1, bo.G1_GEN, a, d, 100))),
        _group("P, -P", [enc[9], bo.g1_compress(G1.neg(pts[9]))], (SUCCESS, INF_PK)),
        _group("duplicates", [enc[2]] * 4, ok(G1.mul(pts[2], 4))),
        _group("empty again", [], (EMPTY, None)),
    ]
    for e, code in bad:
        for i in (0, 31, 32, 99):
            items = list(enc)
            items[i] = e
            gs.append(_group(f"invalid ({code}) at {i}", items, (code, None)))
    for (e1, c1), (e2, c2) in zip(bad, bad[1:] + bad[:1]):
        items = list(enc)
        items[40], items[33] = e1, e2
        gs.append(_group(f"invalid {c2} at 33 before {c1} at 40", items, (c2, None)))
    gs.append(_group("torsion controls", small_order(torsion_g1, 5, rnd, valid=True)))
    return gs


def registry_layout(torsion_g1, seed=1, n_valid=600):
    """A registry of n_valid progression keys with invalid keys spliced in, and index groups over it (repeats, invalid
    keys first and last, empty groups).  -> (keys: list of 48-byte encodings, groups: list of index lists)."""
    rnd = random.Random(0xC66 + seed)
    keys, _, _, _ = key_pool(seed + 100, n_valid)
    bad = invalid_keys(torsion_g1, rnd)
    for k, (e, _) in enumerate(bad):
        keys.insert(rnd.randrange(len(keys)), e)
    n = len(keys)
    bad_idx = [i for i, k in enumerate(keys) if k in {e for e, _ in bad}]
    groups = [[], [0], [n - 1], list(range(n)), [5, 5, 5], []]
    groups += [rnd.choices(range(n), k=rnd.randrange(1, 80)) for _ in range(40)]
    groups += [[b] + rnd.choices(range(n), k=10) for b in bad_idx] + [rnd.choices(range(n), k=10) + [b] for b in bad_idx]
    return keys, groups


def slot(seed=1, committees=64, size=512):
    """One slot of single-signer attestations: committee c has keys (a_c + i d) g1 and signatures (a_c + i d) H(m_c) of its
    own message m_c.  -> dict msgs (32 bytes each), sigs / keys (flat bytes, committee-major), offsets, agg_sig / agg_pk
    (the closed-form aggregates)."""
    d = 1 + _scalar(b"slot d%d" % seed) % 1000
    out = {"msgs": [], "sigs": [], "keys": [], "agg_sig": [], "agg_pk": [], "offsets": [0]}
    for c in range(committees):
        m = hashlib.sha256(b"slot %d committee %d" % (seed, c)).digest()
        h, a = bo.hash_to_g2(m), _scalar(b"slot %d a%d" % (seed, c))
        out["msgs"].append(m)
        out["sigs"] += [bo.g2_compress(p) for p in progression(G2, h, a, d, size)]
        out["keys"] += [bo.g1_compress(p) for p in progression(G1, bo.G1_GEN, a, d, size)]
        out["agg_sig"].append(bo.g2_compress(progression_sum(G2, h, a, d, size)))
        out["agg_pk"].append(bo.g1_compress(progression_sum(G1, bo.G1_GEN, a, d, size)))
        out["offsets"].append(out["offsets"][-1] + size)
    return out


def big_group(seed=1, n=1 << 15):
    """One group of n signatures of one message -> (flat 96-byte encodings, the closed-form aggregate)."""
    h = bo.hash_to_g2(b"big group %d" % seed)
    a, d = _scalar(b"big a%d" % seed), 1 + _scalar(b"big d%d" % seed) % 1000
    return [bo.g2_compress(p) for p in progression(G2, h, a, d, n)], bo.g2_compress(progression_sum(G2, h, a, d, n))


def flatten(groups):
    """-> (flat bytes, offsets list)."""
    off = [0]
    for g in groups:
        off.append(off[-1] + len(g["items"]))
    return b"".join(b"".join(g["items"]) for g in groups), off
