"""CPU-only parity soak (no GPU needed): the product's own __host__ __device__ math (tests/host_math, compiled from
ethereum_consensus_b200/csrc/*.cuh — the same source the kernels compile) against the independent plain-C oracle on
tens of thousands of random and adversarial inputs.  SURVEY.md §8c asks for >= 10^4 such cases because the reference's
own offline KATs only pin the accept side.

    python tests/soak_parity.py [scale] > soak_parity.txt        (scale 1.0 ~ a few minutes on 8 cores)
"""
import ctypes as C, subprocess, sys, time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent  # tests/ -> repo root
sys.path.insert(0, str(ROOT))
from tests import bls_soak_cases as sc  # noqa: E402  (the case generators, shared with the device soak)
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


def report(name, n, bad, codes):
    hist = ", ".join(f"{c}: {k}" for c, k in sorted(codes.items()))
    print(f"{name:34s} cases {n:6d}  mismatches {bad}   verdict histogram {{{hist}}}")
    sys.stdout.flush()


total_bad = 0
# ---- 1. public-key validation (blst key_validate semantics)
n = int(6000 * scale)
keys, _, _ = sc.valid_keys(O, n)
cases = [keys[i].tobytes() for i in range(n)]
cases += [r.tobytes() for r in sc.random_g1_encodings(rng, int(8000 * scale))]   # about half are on the curve
cases += [sc.mutate(keys[i % n].tobytes(), 48, i % 9, rng) for i in range(int(6000 * scale))]
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
sigs = sc.valid_sigs(O, n)
cases = [sigs[i].tobytes() for i in range(n)]
cases += [r.tobytes() for r in sc.random_g2_encodings(rng, int(4000 * scale))]
cases += [sc.mutate(sigs[i % n].tobytes(), 96, i % 9, rng) for i in range(int(2500 * scale))]
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
keys, sk0, d = sc.valid_keys(O, 64, seed=2)
for t in range(n):
    c = sc.tuple_case(keys, sk0, d, t, rng)
    sk = np.frombuffer(c["sk"], dtype=np.uint8).copy()
    mm = np.frombuffer(c["sign_msg"], dtype=np.uint8).copy()
    sig = np.empty(96, dtype=np.uint8)
    O.orc_sign_batch(sk.ctypes.data, mm.ctypes.data, 1, sig.ctypes.data, 1)
    pks, K, msg, sigb = c["pks"], c["K"], c["msg"], sc.finish_tuple(c, sig.tobytes())
    a = H.hm_fast_aggregate_verify(pks, K, msg, 32, sigb)
    b = O.orc_fast_aggregate_verify(pks, K, msg, 32, sigb)
    hist[b] = hist.get(b, 0) + 1
    bad += a != b
report("fast_aggregate_verify (K<=8)", n, bad, hist); total_bad += bad
# ---- 5. triangulation: the spec-level Python big-int oracle (in_subgroup = [r]P by definition, generic square roots)
#         against the C oracle on a sample of the same case generators
from oracle import bls_oracle as bo  # noqa: E402
n = int(500 * scale)
keys, _, _ = sc.valid_keys(O, n, seed=3)
sample = [keys[i].tobytes() for i in range(n // 4)]
sample += [r.tobytes() for r in sc.random_g1_encodings(rng, n // 2)] + [sc.mutate(keys[i].tobytes(), 48, i % 9, rng) for i in range(n // 4)]
bad = sum(bo.key_validate(c)[0] != O.orc_key_validate(c) for c in sample)
report("py vs C: key_validate", len(sample), bad, {}); total_bad += bad
sg = sc.valid_sigs(O, n // 8)
sample = [sg[i].tobytes() for i in range(n // 8)]
sample += [r.tobytes() for r in sc.random_g2_encodings(rng, n // 4)] + [sc.mutate(sg[i % (n // 8)].tobytes(), 96, i % 9, rng) for i in range(n // 8)]
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
