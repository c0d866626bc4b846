"""CPU-only parity soak (no GPU needed): the product's own __host__ __device__ math (tests/host_math, compiled from
ethereum_consensus_b200/csrc/*.cuh — the same source the kernels compile) against the independent plain-C oracle on
tens of thousands of random and adversarial inputs.  SURVEY.md §8c asks for >= 10^4 such cases because the reference's
own offline KATs only pin the accept side.

    python tests/soak_parity.py [scale] > soak_parity.txt        (scale 1.0 ~ a few minutes on 8 cores)
"""
import ctypes as C, hashlib, subprocess, sys, time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent  # tests/ -> repo root
sys.path.insert(0, str(ROOT))
P = 0x1a0111ea397fe69a4b1ba7b6434bacd764774b84f38512bf6730d2a0f6b0f6241eabfffeb153ffffb9feffffffffaaab
R = 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001
scale = float(sys.argv[1]) if len(sys.argv) > 1 else 1.0

subprocess.run(["make", "-s", "-C", str(ROOT / "oracle")], check=True)
src = ROOT / "tests" / "host_math" / "host_math.cpp"
lib = ROOT / "tests" / "host_math" / "libhost_math.so"
deps = [src] + list((ROOT / "ethereum_consensus_b200" / "csrc").glob("*.cuh"))
if not lib.exists() or any(d.stat().st_mtime > lib.stat().st_mtime for d in deps):
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-fvisibility=hidden", "-o", str(lib), str(src)], check=True)
H = C.CDLL(str(lib))
O = C.CDLL(str(ROOT / "oracle" / "liboracle_bls.so"))
cp, sz, vp = C.c_char_p, C.c_size_t, C.c_void_p
O.orc_key_validate.argtypes = [cp]
O.orc_aggregate.argtypes = [cp, sz, cp]
O.orc_hash_to_g2.argtypes = [cp, sz, cp]
O.orc_fast_aggregate_verify.argtypes = [cp, sz, cp, sz, cp]
O.orc_pk_sequence.argtypes = [cp, cp, sz, vp]
O.orc_sign_batch.argtypes = [vp, vp, sz, vp, C.c_int]
H.hm_g1_key_validate.argtypes = [cp, cp, cp]
H.hm_g2_uncompress.argtypes = [cp, cp, vp, vp, cp]
H.hm_hash_to_g2.argtypes = [cp, sz, vp, vp]
H.hm_fast_aggregate_verify.argtypes = [cp, sz, cp, sz, cp]

rng = np.random.default_rng(0xB200)
t_start = time.time()


def valid_keys(n, seed=1):
    keys = np.empty((n, 48), dtype=np.uint8)
    sk0 = int.from_bytes(hashlib.sha256(b"soak/sk0%d" % seed).digest(), "big") % R
    d = int.from_bytes(hashlib.sha256(b"soak/d%d" % seed).digest(), "big") % R
    O.orc_pk_sequence(sk0.to_bytes(32, "big"), d.to_bytes(32, "big"), n, keys.ctypes.data)
    return keys, sk0, d


def valid_sigs(n):
    sks = np.frombuffer(b"".join(((int.from_bytes(hashlib.sha256(b"soak/ssk%d" % i).digest(), "big") % (R - 1)) + 1).to_bytes(32, "big")
                                 for i in range(n)), dtype=np.uint8).copy()
    msgs = np.frombuffer(b"".join(hashlib.sha256(b"soak/m%d" % i).digest() for i in range(n)), dtype=np.uint8).copy()
    out = np.empty((n, 96), dtype=np.uint8)
    O.orc_sign_batch(sks.ctypes.data, msgs.ctypes.data, n, out.ctypes.data, 8)
    return out


def mutate(enc: bytes, width: int, k: int) -> bytes:
    b = bytearray(enc)
    x = int.from_bytes(b, "big") & ((1 << (8 * width - 3)) - 1)
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


def report(name, n, bad, codes):
    hist = ", ".join(f"{c}: {k}" for c, k in sorted(codes.items()))
    print(f"{name:34s} cases {n:6d}  mismatches {bad}   verdict histogram {{{hist}}}")
    sys.stdout.flush()


total_bad = 0
# ---- 1. public-key validation (blst key_validate semantics)
n = int(6000 * scale)
keys, _, _ = valid_keys(n)
cases = [keys[i].tobytes() for i in range(n)]
rnd = rng.integers(0, 256, (int(8000 * scale), 48), dtype=np.uint8)
rnd[:, 0] = (rnd[:, 0] & 0x3f) | 0x80 | (rnd[:, 0] & 0x20)    # compressed, finite: x < 2^381.. about half are on the curve
rnd[:, 0] &= 0xbf
cases += [r.tobytes() for r in rnd]
cases += [mutate(keys[i % n].tobytes(), 48, i % 9) for i in range(int(6000 * scale))]
bad, hist = 0, {}
xy, rec = C.create_string_buffer(96), C.create_string_buffer(48)
for c in cases:
    a = H.hm_g1_key_validate(c, xy, rec)
    b = O.orc_key_validate(c)
    hist[b] = hist.get(b, 0) + 1
    if a != b or (a == 0 and rec.raw != c):
        bad += 1
report("G1 key_validate", len(cases), bad, hist); total_bad += bad

# ---- 2. signature decode + subgroup check (Signature::from_bytes + sig_groupcheck)
n = int(1500 * scale)
sigs = valid_sigs(n)
cases = [sigs[i].tobytes() for i in range(n)]
rnd = rng.integers(0, 256, (int(4000 * scale), 96), dtype=np.uint8)
rnd[:, 0] = ((rnd[:, 0] & 0x3f) | 0x80) & 0xbf
rnd[:, 48] &= 0x1f                                            # x.c0 < 2^381 (about 80 % of those are < p)
cases += [r.tobytes() for r in rnd]
cases += [mutate(sigs[i % n].tobytes(), 96, i % 9) for i in range(int(2500 * scale))]
bad, hist = 0, {}
o192, inf, ing, rec96, agg = C.create_string_buffer(192), C.c_int(), C.c_int(), C.create_string_buffer(96), C.create_string_buffer(96)
for c in cases:
    a = H.hm_g2_uncompress(c, o192, C.byref(inf), C.byref(ing), rec96)
    b = O.orc_aggregate(c, 1, agg)                            # decode error | NOT_IN_GROUP (3) | 0 with the point re-compressed
    hist[b] = hist.get(b, 0) + 1
    mine = a if a else (0 if (inf.value or ing.value) else 3)
    if mine != b or (b == 0 and (rec96.raw != c or agg.raw != c)):
        bad += 1
report("G2 decode + subgroup", len(cases), bad, hist); total_bad += bad

# ---- 3. hash_to_G2 (RFC 9380, the ciphersuite DST)
n = int(6000 * scale)
bad = 0
o2 = C.create_string_buffer(192)
for i in range(n):
    ln = int(rng.integers(0, 200)) if i % 3 else 32
    m = rng.integers(0, 256, ln, dtype=np.uint8).tobytes()
    H.hm_hash_to_g2(m, len(m), o192, C.byref(inf))
    O.orc_hash_to_g2(m, len(m), o2)
    if inf.value or o192.raw != o2.raw:
        bad += 1
report("hash_to_G2", n, bad, {}); total_bad += bad

# ---- 4. whole fast_aggregate_verify on small tuples, valid and adversarial
n = int(400 * scale)
bad, hist = 0, {}
keys, sk0, d = valid_keys(64, seed=2)
for t in range(n):
    K = int(rng.integers(1, 9))
    idx = rng.integers(0, 64, K)
    msg = hashlib.sha256(b"soak/t%d" % t).digest()
    s = sum((sk0 + int(i) * d) % R for i in idx) % R
    kind = t % 8
    if kind == 1: s = (s + 1) % R                              # wrong signer set
    sk = np.frombuffer((s if s else 1).to_bytes(32, "big"), dtype=np.uint8).copy()
    mm = np.frombuffer(msg if kind != 2 else hashlib.sha256(msg).digest(), dtype=np.uint8).copy()   # wrong message
    sig = np.empty(96, dtype=np.uint8)
    O.orc_sign_batch(sk.ctypes.data, mm.ctypes.data, 1, sig.ctypes.data, 1)
    pks = bytearray(keys[idx].tobytes())
    sigb = sig.tobytes()
    if kind == 3: pks[0:48] = mutate(bytes(pks[0:48]), 48, 6)  # infinity key
    if kind == 4 and K >= 2:                                   # P and -P
        pks[48:96] = mutate(bytes(pks[0:48]), 48, 0)
    if kind == 5: sigb = mutate(sigb, 96, 6)                   # infinity signature
    if kind == 6: sigb = mutate(sigb, 96, int(rng.integers(0, 9)))
    if kind == 7: pks[0:48] = mutate(bytes(pks[0:48]), 48, int(rng.integers(0, 9)))
    a = H.hm_fast_aggregate_verify(bytes(pks), K, msg, 32, sigb)
    b = O.orc_fast_aggregate_verify(bytes(pks), K, msg, 32, sigb)
    hist[b] = hist.get(b, 0) + 1
    bad += a != b
report("fast_aggregate_verify (K<=8)", n, bad, hist); total_bad += bad
# ---- 5. triangulation: the spec-level Python big-int oracle (in_subgroup = [r]P by definition, generic square roots)
#         against the C oracle on a sample of the same case generators
from oracle import bls_oracle as bo  # noqa: E402
n = int(500 * scale)
keys, _, _ = valid_keys(n, seed=3)
sample = [keys[i].tobytes() for i in range(n // 4)]
rnd = rng.integers(0, 256, (n // 2, 48), dtype=np.uint8)
rnd[:, 0] = ((rnd[:, 0] & 0x3f) | 0x80) & 0xbf
sample += [r.tobytes() for r in rnd] + [mutate(keys[i].tobytes(), 48, i % 9) for i in range(n // 4)]
bad = sum(bo.key_validate(c)[0] != O.orc_key_validate(c) for c in sample)
report("py vs C: key_validate", len(sample), bad, {}); total_bad += bad
sg = valid_sigs(n // 8)
sample = [sg[i].tobytes() for i in range(n // 8)]
rnd = rng.integers(0, 256, (n // 4, 96), dtype=np.uint8)
rnd[:, 0] = ((rnd[:, 0] & 0x3f) | 0x80) & 0xbf
rnd[:, 48] &= 0x1f
sample += [r.tobytes() for r in rnd] + [mutate(sg[i % (n // 8)].tobytes(), 96, i % 9) for i in range(n // 8)]
bad = 0
for c in sample:
    code, out = bo.aggregate([c])
    b = O.orc_aggregate(c, 1, agg)
    bad += code != b or (code == 0 and out != agg.raw)
report("py vs C: sig decode + subgroup", len(sample), bad, {}); total_bad += bad
bad = 0
for i in range(n // 5):
    m = rng.integers(0, 256, int(rng.integers(0, 120)), dtype=np.uint8).tobytes()
    O.orc_hash_to_g2(m, len(m), o2)
    (x, y) = bo.hash_to_g2(m)
    bad += o2.raw != b"".join(v.to_bytes(48, "big") for v in (x[0], x[1], y[0], y[1]))
report("py vs C: hash_to_G2", n // 5, bad, {}); total_bad += bad
print(f"total mismatches {total_bad}   wall {time.time() - t_start:.0f} s   (blst codes: 0 ok, 1 bad encoding, 2 not on curve, 3 not in group, "
      f"5 verify fail, 6 pk is infinity)")
sys.exit(1 if total_bad else 0)
