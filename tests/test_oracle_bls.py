"""CPU: pins the BLS oracle to the reference's own KATs, then checks the product's host-compiled math against it."""
import ctypes as C
import json
import random
from pathlib import Path

import pytest

from oracle import bls_oracle as bo

ROOT = Path(__file__).resolve().parent.parent

GOLDEN = json.loads((Path(__file__).parent / "golden" / "bls_cases.json").read_text())
F1, F2 = bo.F1, bo.F2

# KAT B-2: ethereum-consensus/src/crypto/bls.rs:530-544 (`test_can_sign`)
B2_SK = int("40094c5c6c378857eac09b8ec64c87182f58700c056a8b371ad0eb0a5b983d50", 16)
B2_MSG = b"blst is such a blast"
B2_SIG = bytes.fromhex("a01e49276730e4752eef31b0570c8707de501398dac70dd144438cd1bd05fb9b9bb3e1a9ceef0a68cc08904362cafa3f"
                       "1005e5b699a41847fff6f5552260468846de5bdbf94a9aedeb29bc6cdb2c1d34922d9e9af4c0593a69ae978a90b5aba6")
# KAT B-1: ethereum-consensus/src/bin/ec/validator/keystores.rs:239-249 (EIP-2335)
B1_SK = int("000000000019d6689c085ae165831e934ff763ae46a2a6c172b3f1b60a8ce26f", 16)
B1_PK = bytes.fromhex("9612d7a727c9d0a22e185a1c768478dfe919cada9266988cb32359c11f2b7b27f4ae4040902382ae2910c15e2b420d07")
# KAT B-2b: decode-only points, crypto/bls.rs:381-390 and :453-461
GOOD_SIG = bytes.fromhex("abb0124c7574f281a293f4185cad3cb22681d520917ce46665243eacb051000d8bacf75e1451870ca6b3b9e6c9d41a7b"
                         "02ead2685a84188a4fafd3825daf6a989625d719ccd2d83a40101f4a453fca62878c890eca622363f9ddb8f367a91e84")
GOOD_PK = bytes.fromhex("a99a76ed7796f7be22d5b7e85deeb7c5677e88e511e0b337618f8c4eb61349b4bf2d153f649f7b53359fe8b94a38e44c")


def test_kat_b1_sk_to_pk():
    assert bo.sk_to_pk(B1_SK) == B1_PK


def test_kat_b2_sign_and_verify():
    assert bo.sign(B2_SK, B2_MSG) == B2_SIG
    pk = bo.sk_to_pk(B2_SK)
    assert bo.verify_signature(pk, B2_MSG, B2_SIG) == bo.SUCCESS
    assert bo.verify_signature(pk, B2_MSG + b"!", B2_SIG) == bo.VERIFY_FAIL
    assert bo.verify_signature(B1_PK, B2_MSG, B2_SIG) == bo.VERIFY_FAIL


def test_kat_b2b_decode_only_points():
    code, pt = bo.g2_uncompress(GOOD_SIG)
    assert code == 0 and bo.on_curve(F2, pt) and bo.g2_compress(pt) == GOOD_SIG
    assert bo.key_validate(GOOD_PK)[0] == 0


def test_curve_constants():
    assert bo.on_curve(F1, bo.G1_GEN) and bo.on_curve(F2, bo.G2_GEN)
    assert bo.in_subgroup(F1, bo.G1_GEN) and bo.in_subgroup(F2, bo.G2_GEN)
    z = -bo.Z_ABS
    assert bo.R == z ** 4 - z ** 2 + 1 and bo.P == (z - 1) ** 2 * bo.R // 3 + z


def test_pairing_bilinear_nondegenerate():
    a, b = 0xdeadbeef, 0xfeedface
    aP = bo.pt_to_affine(F1, bo.pt_mul(F1, bo.pt_from_affine(F1, bo.G1_GEN), a))
    bQ = bo.pt_to_affine(F2, bo.pt_mul(F2, bo.pt_from_affine(F2, bo.G2_GEN), b))
    mabP = bo.pt_to_affine(F1, bo.pt_mul(F1, bo.pt_from_affine(F1, bo.G1_GEN), bo.R - a * b % bo.R))
    assert bo.pairing_check([(aP, bQ), (mabP, bo.G2_GEN)])
    assert not bo.pairing_check([(bo.G1_GEN, bo.G2_GEN)])


def test_golden_file_matches_oracle_spotcheck():
    for c in GOLDEN["fast_aggregate_verify"]:
        if len(c["pks"]) <= 4:
            got = bo.fast_aggregate_verify([bytes.fromhex(p) for p in c["pks"]], bytes.fromhex(c["msg"]), bytes.fromhex(c["sig"]))
            assert got == c["code"], c["name"]


def _b48(x): return x.to_bytes(48, "big")


def test_host_math_fields_match_oracle(host_math):
    rnd = random.Random(7)
    out = C.create_string_buffer(48)
    for i in range(300):
        a, b = rnd.randrange(bo.P), rnd.randrange(bo.P)
        if i == 0: a, b = 0, 0
        if i == 1: a, b = bo.P - 1, bo.P - 1
        for op, want in ((0, (a + b) % bo.P), (1, (a - b) % bo.P), (2, a * b % bo.P), (5, -a % bo.P)):
            host_math.hm_fp_op(op, _b48(a), _b48(b), out)
            assert int.from_bytes(out.raw, "big") == want
    out = C.create_string_buffer(96)
    for i in range(20):
        a = (rnd.randrange(bo.P), rnd.randrange(bo.P)); b = (rnd.randrange(bo.P), rnd.randrange(bo.P))
        enc = lambda v: _b48(v[0]) + _b48(v[1])  # noqa: E731
        dec = lambda o: (int.from_bytes(o.raw[:48], "big"), int.from_bytes(o.raw[48:], "big"))  # noqa: E731
        host_math.hm_fp2_op(0, enc(a), enc(b), out); assert dec(out) == bo.f2_mul(a, b)
        host_math.hm_fp2_op(2, enc(a), enc(b), out); assert dec(out) == bo.f2_inv(a)
        ok = host_math.hm_fp2_op(3, enc(a), enc(b), out); assert bool(ok) == (bo.f2_sqrt(a) is not None)
        assert host_math.hm_fp2_op(4, enc(a), enc(b), out) == bo.f2_sgn0(a)
    # complex-method square root (two exponentiations, shared between the residue / non-residue sub-cases): every
    # sub-case of fp2_sqrt_with_norm_root and the real-input path, checked by squaring
    qr = next(x for x in range(2, 50) if pow(x, (bo.P - 1) // 2, bo.P) == 1)
    nqr = next(x for x in range(2, 50) if pow(x, (bo.P - 1) // 2, bo.P) == bo.P - 1)
    cases = [(0, 0), (qr, 0), (nqr, 0), (0, qr), (0, nqr), (bo.P - 1, 0), (1, 0)]
    cases += [bo.f2_sqr((rnd.randrange(bo.P), rnd.randrange(bo.P))) for _ in range(40)]
    cases += [(rnd.randrange(bo.P), rnd.randrange(bo.P)) for _ in range(40)]
    n_sq = 0
    for a in cases:
        ok = host_math.hm_fp2_op(3, enc(a), enc(a), out)
        assert bool(ok) == (bo.f2_sqrt(a) is not None), a
        if ok:
            n_sq += 1
            assert bo.f2_sqr(dec(out)) == (a[0] % bo.P, a[1] % bo.P)
    assert 45 < n_sq < len(cases)
    assert host_math.hm_fp12_selftest() == 63


def test_host_math_hash_to_g2_matches_oracle(host_math):
    o = C.create_string_buffer(192); inf = C.c_int()
    import hashlib
    for m in [b"", b"abc", B2_MSG, bytes(32), bytes(range(100)), bytes(255)] + [hashlib.sha256(b"h2c%d" % i).digest() for i in range(24)]:
        host_math.hm_hash_to_g2(m, len(m), o, C.byref(inf))
        pt = ((int.from_bytes(o.raw[0:48], "big"), int.from_bytes(o.raw[48:96], "big")),
              (int.from_bytes(o.raw[96:144], "big"), int.from_bytes(o.raw[144:], "big")))
        assert inf.value == 0 and pt == bo.hash_to_g2(m)


def test_host_math_kat_b2(host_math):
    pk = bo.sk_to_pk(B2_SK)
    assert host_math.hm_fast_aggregate_verify(pk, 1, B2_MSG, len(B2_MSG), B2_SIG) == 0
    assert host_math.hm_fast_aggregate_verify(pk, 1, B2_MSG + b"!", len(B2_MSG) + 1, B2_SIG) == 5


@pytest.mark.parametrize("case", GOLDEN["fast_aggregate_verify"], ids=lambda c: c["name"])
def test_host_math_fast_aggregate_verify_golden(host_math, case):
    """Every golden tuple through the product's own (host-compiled) decode / subgroup / hash / pairing code."""
    pks = b"".join(bytes.fromhex(p) for p in case["pks"])
    m, s = bytes.fromhex(case["msg"]), bytes.fromhex(case["sig"])
    assert host_math.hm_fast_aggregate_verify(pks, len(case["pks"]), m, len(m), s) == case["code"]


# ---------------------------------------------------------------------------------------------- the plain-C oracle
def test_c_oracle_kats(oracle_bls_c):
    o48, o96 = C.create_string_buffer(48), C.create_string_buffer(96)
    oracle_bls_c.orc_sk_to_pk(B1_SK.to_bytes(32, "big"), o48)
    assert o48.raw == B1_PK
    oracle_bls_c.orc_sign(B2_SK.to_bytes(32, "big"), B2_MSG, len(B2_MSG), o96)
    assert o96.raw == B2_SIG
    oracle_bls_c.orc_sk_to_pk(B2_SK.to_bytes(32, "big"), o48)
    assert oracle_bls_c.orc_verify_signature(o48.raw, B2_MSG, len(B2_MSG), B2_SIG) == 0
    assert oracle_bls_c.orc_verify_signature(o48.raw, B2_MSG + b"!", len(B2_MSG) + 1, B2_SIG) == 5
    assert oracle_bls_c.orc_key_validate(GOOD_PK) == 0


def test_host_math_sswu_fraction_variant_matches_oracles(host_math_sswu_fraction, oracle_bls_c):
    """The default-off `B200_SSWU_FRACTION` build of hash_to_G2 (no inversion in the SSWU map) is bit-identical to the
    Python oracle on the fixed messages and to the C oracle on 600 random ones (both branches of the map, both signs)."""
    import hashlib
    hm = host_math_sswu_fraction
    o = C.create_string_buffer(192); o2 = C.create_string_buffer(192); inf = C.c_int()
    for m in (b"", b"abc", B2_MSG, bytes(32), bytes(range(100)), bytes(255)):
        hm.hm_hash_to_g2(m, len(m), o, C.byref(inf))
        pt = ((int.from_bytes(o.raw[0:48], "big"), int.from_bytes(o.raw[48:96], "big")),
              (int.from_bytes(o.raw[96:144], "big"), int.from_bytes(o.raw[144:], "big")))
        assert inf.value == 0 and pt == bo.hash_to_g2(m)
    for i in range(600):
        m = hashlib.sha256(b"frac%d" % i).digest()[: 1 + i % 32]
        hm.hm_hash_to_g2(m, len(m), o, C.byref(inf))
        oracle_bls_c.orc_hash_to_g2(m, len(m), o2)
        assert inf.value == 0 and o.raw == o2.raw, i


def test_c_oracle_hash_to_g2_matches_python(oracle_bls_c):
    o = C.create_string_buffer(192)
    for m in (b"", b"abc", bytes(32), bytes(range(200))):
        oracle_bls_c.orc_hash_to_g2(m, len(m), o)
        pt = ((int.from_bytes(o.raw[0:48], "big"), int.from_bytes(o.raw[48:96], "big")),
              (int.from_bytes(o.raw[96:144], "big"), int.from_bytes(o.raw[144:], "big")))
        assert pt == bo.hash_to_g2(m)


def test_c_oracle_group_check_shortcuts_agree_with_definition(oracle_bls_c):
    """phi / psi membership tests vs [r]P == inf on curve points inside and outside the prime-order subgroups."""
    for x in range(1, 60):
        for flag in (0x80, 0xA0):
            assert oracle_bls_c.orc_g1_group_checks_agree(bytes([flag]) + x.to_bytes(48, "big")[1:]) == 1
            assert oracle_bls_c.orc_g2_group_checks_agree(bytes([flag]) + bytes(47) + x.to_bytes(48, "big")) == 1
    for c in GOLDEN["fast_aggregate_verify"][:6]:
        for p in c["pks"]:
            assert oracle_bls_c.orc_g1_group_checks_agree(bytes.fromhex(p)) == 1
        assert oracle_bls_c.orc_g2_group_checks_agree(bytes.fromhex(c["sig"])) == 1


@pytest.mark.parametrize("case", GOLDEN["fast_aggregate_verify"], ids=lambda c: c["name"])
def test_c_oracle_fast_aggregate_verify_golden(oracle_bls_c, case):
    pks = b"".join(bytes.fromhex(p) for p in case["pks"])
    m, s = bytes.fromhex(case["msg"]), bytes.fromhex(case["sig"])
    assert oracle_bls_c.orc_fast_aggregate_verify(pks, len(case["pks"]), m, len(m), s) == case["code"]


def test_c_oracle_other_entry_points_golden(oracle_bls_c):
    for c in GOLDEN["aggregate_verify"]:
        msgs = [bytes.fromhex(m) for m in c["msgs"]]
        arr = (C.c_char_p * max(len(msgs), 1))(*msgs) if msgs else (C.c_char_p * 1)()
        lens = (C.c_size_t * max(len(msgs), 1))(*[len(m) for m in msgs])
        pks = b"".join(bytes.fromhex(p) for p in c["pks"])
        got = oracle_bls_c.orc_aggregate_verify(pks, len(c["pks"]), C.cast(arr, C.c_void_p), C.cast(lens, C.c_void_p), len(msgs),
                                                bytes.fromhex(c["sig"]))
        assert got == c["code"], c["name"]
    o96, o48 = C.create_string_buffer(96), C.create_string_buffer(48)
    for c in GOLDEN["aggregate"]:
        got = oracle_bls_c.orc_aggregate(b"".join(bytes.fromhex(s) for s in c["sigs"]), len(c["sigs"]), o96)
        assert got == c["code"] and (got != 0 or o96.raw.hex() == c["out"]), c["name"]
    for c in GOLDEN["eth_aggregate_public_keys"]:
        got = oracle_bls_c.orc_eth_aggregate_public_keys(b"".join(bytes.fromhex(s) for s in c["pks"]), len(c["pks"]), o48)
        assert got == c["code"] and (got != 0 or o48.raw.hex() == c["out"]), c["name"]
    assert oracle_bls_c.orc_aggregate(b"", 0, o96) == 16 and oracle_bls_c.orc_eth_aggregate_public_keys(b"", 0, o48) == 16


def test_fp_mul_ptx_emulation(host_math):
    """The generated inline-PTX Montgomery product, emulated instruction by instruction in C, equals the portable
    product and the big-int result (tools/gen_fp_mul_ptx.py emits both from one instruction list)."""
    rnd = random.Random(11)
    A12 = C.c_uint32 * 12
    lim = lambda x: A12(*[(x >> (32 * i)) & 0xFFFFFFFF for i in range(12)])  # noqa: E731
    edge = [0, 1, 2, bo.P - 1, bo.P - 2, (1 << 380), (bo.P - 1) // 2, 0xFFFFFFFF]
    cases = [(a, b) for a in edge for b in edge] + [(rnd.randrange(bo.P), rnd.randrange(bo.P)) for _ in range(20000)]
    for a, b in cases:
        assert host_math.hm_fp_mul_emul_matches(lim(a), lim(b)) == 1


def test_lazily_reduced_field_on_operands_up_to_2p(host_math):
    """fpl.cuh (the per-key kernel's arithmetic): the emulated PTX product / square WITHOUT the final subtraction map
    [0, 2p) x [0, 2p) into [0, 2p) and are correct modulo p; add / sub / neg stay in [0, 2p)."""
    host_math.hm_fp_emul_raw.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    host_math.hm_fpl_op.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    rnd = random.Random(12)
    A12 = C.c_uint32 * 12
    lim = lambda x: A12(*[(x >> (32 * i)) & 0xFFFFFFFF for i in range(12)])  # noqa: E731
    val = lambda arr: sum(int(arr[i]) << (32 * i) for i in range(12))        # noqa: E731
    P, R = bo.P, 1 << 384
    rinv = pow(R, -1, P)
    edge = [0, 1, P - 1, P, P + 1, 2 * P - 1, 2 * P - 2, (1 << 381), 2 * P - (1 << 200)]
    cases = [(a, b) for a in edge for b in edge] + [(rnd.randrange(2 * P), rnd.randrange(2 * P)) for _ in range(20000)]
    out = A12()
    worst = 0
    for a, b in cases:
        host_math.hm_fp_emul_raw(0, lim(a), lim(b), out)
        r = val(out)
        assert r < 2 * P and r % P == a * b * rinv % P, (hex(a), hex(b))
        worst = max(worst, r)
        host_math.hm_fp_emul_raw(1, lim(a), lim(a), out)
        r = val(out)
        assert r < 2 * P and r % P == a * a * rinv % P, hex(a)
        worst = max(worst, r)
        host_math.hm_fpl_op(0, lim(a), lim(b), out); r = val(out); assert r < 2 * P and r % P == (a + b) % P
        host_math.hm_fpl_op(1, lim(a), lim(b), out); r = val(out); assert r < 2 * P and r % P == (a - b) % P
        host_math.hm_fpl_op(2, lim(a), lim(b), out); r = val(out); assert r < 2 * P and r % P == (-a) % P
    assert worst < 1.41 * P + 1     # the bound DESIGN.md section 4 derives: a b / R + p < (4p / R) p + p


def test_adx_build_of_the_c_oracle_agrees_with_the_portable_build(oracle_bls_c):
    """bench.py times oracle/liboracle_bls_adx.so (same source, -mbmi2 -madx) when the host CPU has both features: it must return
    what the portable build returns — every golden fast_aggregate_verify case and a run of key validations."""
    try:
        flags = set(next(ln for ln in open("/proc/cpuinfo") if ln.startswith("flags")).split())
    except (OSError, StopIteration):
        flags = set()
    if not {"adx", "bmi2"} <= flags:
        pytest.skip("host CPU without adx / bmi2")
    adx = C.CDLL(str(ROOT / "oracle" / "liboracle_bls_adx.so"))
    for lib in (adx, oracle_bls_c):
        lib.orc_fast_aggregate_verify.argtypes = [C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t, C.c_char_p]
        lib.orc_key_validate.argtypes = [C.c_char_p]
    golden = json.loads((ROOT / "tests" / "golden" / "bls_cases.json").read_text())
    for c in golden["fast_aggregate_verify"]:
        pks = b"".join(bytes.fromhex(p) for p in c["pks"])
        m, sg = bytes.fromhex(c["msg"]), bytes.fromhex(c["sig"])
        a = adx.orc_fast_aggregate_verify(pks, len(c["pks"]), m, len(m), sg)
        assert a == oracle_bls_c.orc_fast_aggregate_verify(pks, len(c["pks"]), m, len(m), sg) == c["code"], c["name"]
        for p in c["pks"][:4]:
            assert adx.orc_key_validate(bytes.fromhex(p)) == oracle_bls_c.orc_key_validate(bytes.fromhex(p))


def test_kaliski_inverse_equals_fermat_inverse(host_math):
    """fp.cuh's device inverse (Kaliski almost-inverse + two products) on the host: the same Montgomery-form value as a^(p-2)
    for 0, 1, p - 1, powers of two, R mod p, values whose loop runs the minimum / maximum number of rounds, and 3 000 random
    elements — and that value really is the inverse."""
    host_math.hm_fp_inv_both.argtypes = [C.c_void_p, C.c_void_p]
    rnd = random.Random(2024)
    A12, A24 = C.c_uint32 * 12, C.c_uint32 * 24
    lim = lambda x: A12(*[(x >> (32 * i)) & 0xFFFFFFFF for i in range(12)])  # noqa: E731
    P, R = bo.P, 1 << 384
    edge = [0, 1, 2, 3, P - 1, P - 2, (P - 1) // 2, (P + 1) // 2, R % P, R * R % P, pow(R, -1, P), (1 << 380), (1 << 380) + 1,
            (1 << 255) - 19, 0xffffffff, 1 << 32, (1 << 352) - 1] + [1 << j for j in range(0, 381, 7)]
    out = A24()
    for x in edge + [rnd.randrange(P) for _ in range(3000)]:
        host_math.hm_fp_inv_both(lim(x), out)
        k = sum(int(out[i]) << (32 * i) for i in range(12))
        f = sum(int(out[12 + i]) << (32 * i) for i in range(12))
        assert k == f, hex(x)
        if x:   # x = a R, k = a^-1 R  =>  x * k = R^2
            assert x * k % P == R * R % P, hex(x)


def test_pairing_vm_programs_match_direct_evaluation(host_math):
    """The statically scheduled lane-parallel Miller / final-exponentiation programs (tools/gen_pairing_vm.py), run by
    the product's interpreter on the host, reproduce miller_loop bit for bit and final_exp_is_one's verdict."""
    enc1 = lambda a: _b48(a[0]) + _b48(a[1])  # noqa: E731
    enc2 = lambda a: _b48(a[0][0]) + _b48(a[0][1]) + _b48(a[1][0]) + _b48(a[1][1])  # noqa: E731
    g1 = lambda k: bo.pt_to_affine(F1, bo.pt_mul(F1, bo.pt_from_affine(F1, bo.G1_GEN), k))  # noqa: E731
    g2 = lambda k: bo.pt_to_affine(F2, bo.pt_mul(F2, bo.pt_from_affine(F2, bo.G2_GEN), k))  # noqa: E731
    a, b = 0xabcdef123, 0x987654321
    assert host_math.hm_vm_matches_direct(enc1(g1(a)), enc2(g2(b)), enc1(g1(bo.R - a * b % bo.R)), enc2(bo.G2_GEN)) == 3
    assert host_math.hm_vm_matches_direct(enc1(g1(a)), enc2(g2(b)), enc1(g1(bo.R - a * b % bo.R + 5)), enc2(bo.G2_GEN)) == 1
