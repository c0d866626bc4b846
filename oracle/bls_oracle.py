"""BLS12-381 signature oracle in pure Python big-ints (TEST INFRASTRUCTURE — never imported by the product path).

The reference's BLS arithmetic lives in the un-vendored crate `blst = "0.3.11"` (Cargo.toml:21);
what the reference checkout holds is the byte-typed wrapper ethereum-consensus/src/crypto/bls.rs.  This
file restates, slowly and obviously:

* the wrapper semantics — which checks run, in which order, what maps to Ok/Err:
    verify_signature            crypto/bls.rs:64-77
    aggregate                   crypto/bls.rs:79-93
    aggregate_verify            crypto/bls.rs:95-112
    fast_aggregate_verify       crypto/bls.rs:114-132
    eth_aggregate_public_keys   crypto/bls.rs:135-148
    eth_fast_aggregate_verify   crypto/bls.rs:150-160
    key_validate / from_bytes   crypto/bls.rs:279-285, 330-336
    SecretKey::{public_key,sign} crypto/bls.rs:212-220 (for the KATs)
* the published algorithms blst implements: IETF BLS signatures (ciphersuite named by the DST at crypto/bls.rs:22),
  RFC 9380 hash_to_curve (expand_message_xmd/SHA-256, SSWU, 3-isogeny, cofactor clearing), ZCash point
  serialization, the optimal-ate pairing.

Return codes are blst's BLST_ERROR numbers (order pinned by crypto/bls.rs:48-62): 0 SUCCESS, 1 BAD_ENCODING,
2 POINT_NOT_ON_CURVE, 3 POINT_NOT_IN_GROUP, 4 AGGR_TYPE_MISMATCH, 5 VERIFY_FAIL, 6 PK_IS_INFINITY, 7 BAD_SCALAR;
16 = the wrapper's Error::EmptyAggregate.

Pinned (tests/test_oracle_bls.py) by the reference's own KATs: B-1 sk->pk (bin/ec/validator/keystores.rs:239-249),
B-2 `test_can_sign` (crypto/bls.rs:530-544), B-2b decode-only points (crypto/bls.rs:381-390, 453-461).  Everything
else blst-specific (error precedence, infinity rules) is asserted from the specification, not executed against blst:
"parity weakly pinned" (SURVEY.md §8c).

Pairing note: `pairing_check` tests prod e(P_i, Q_i) == 1 with f_{|z|,Q}(P) (no final conjugation for the negative
BLS parameter): that is the inverse of the optimal-ate pairing, which is itself bilinear and non-degenerate, so the
accept set of the product check is identical.
"""
from __future__ import annotations

import hashlib
from typing import List, Optional, Sequence, Tuple

SUCCESS, BAD_ENCODING, POINT_NOT_ON_CURVE, POINT_NOT_IN_GROUP = 0, 1, 2, 3
AGGR_TYPE_MISMATCH, VERIFY_FAIL, PK_IS_INFINITY, BAD_SCALAR = 4, 5, 6, 7
EMPTY_AGGREGATE = 16

P = 0x1a0111ea397fe69a4b1ba7b6434bacd764774b84f38512bf6730d2a0f6b0f6241eabfffeb153ffffb9feffffffffaaab
R = 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001
Z_ABS = 0xd201000000010000  # the BLS parameter is -Z_ABS
DST = b"BLS_SIG_BLS12381G2_XMD:SHA-256_SSWU_RO_POP_"  # crypto/bls.rs:22

G1_GEN = (0x17f1d3a73197d7942695638c4fa9ac0fc3688c4f9774b905a14e3a3f171bac586c55e83ff97a1aeffb3af00adb22c6bb,
          0x08b3f481e3aaa0f1a09e30ed741d8ae4fcf5e095d5d00af600db18cb2c04b3edd03cc744a2888ae40caa232946c5e7e1)
G2_GEN = ((0x024aa2b2f08f0a91260805272dc51051c6e47ad4fa403b02b4510b647ae3d1770bac0326a805bbefd48056c8c121bdb8,
           0x13e02b6052719f607dacd3a088274f65596bd0d09920b61ab5da61bbdc7f5049334cf11213945d57e5ac7d055d042b7e),
          (0x0ce5d527727d6e118cc9cdc6da2e351aadfd9baa8cbdd3a76d429a695160d12c923ac9cc3baca289e193548608b82801,
           0x0606c4a02ea734cc32acd2b02bc28b99cb3e287e85a763af267492ab572e99ab3f370d275cec1da1aaa9075ff05f79be))

Fp2 = Tuple[int, int]

# ------------------------------------------------------------------------------------------------ Fp2
F2_ZERO: Fp2 = (0, 0)
F2_ONE: Fp2 = (1, 0)


def f2_add(a, b): return ((a[0] + b[0]) % P, (a[1] + b[1]) % P)
def f2_sub(a, b): return ((a[0] - b[0]) % P, (a[1] - b[1]) % P)
def f2_neg(a): return ((-a[0]) % P, (-a[1]) % P)
def f2_mul(a, b): return ((a[0] * b[0] - a[1] * b[1]) % P, (a[0] * b[1] + a[1] * b[0]) % P)
def f2_sqr(a): return ((a[0] * a[0] - a[1] * a[1]) % P, (2 * a[0] * a[1]) % P)
def f2_muli(a, k): return ((a[0] * k) % P, (a[1] * k) % P)
def f2_is_zero(a): return a[0] % P == 0 and a[1] % P == 0


def f2_inv(a):
    d = pow((a[0] * a[0] + a[1] * a[1]) % P, P - 2, P)
    return ((a[0] * d) % P, (-a[1] * d) % P)


def f2_pow(a, e):
    r = F2_ONE
    while e:
        if e & 1:
            r = f2_mul(r, a)
        a = f2_sqr(a)
        e >>= 1
    return r


def f2_sqrt(a) -> Optional[Fp2]:
    """Square root in Fp2 for p = 3 (mod 4) (SURVEY.md Appendix A); None if `a` is not a square."""
    if f2_is_zero(a):
        return F2_ZERO
    a1 = f2_pow(a, (P - 3) // 4)
    alpha = f2_mul(f2_sqr(a1), a)
    x0 = f2_mul(a1, a)
    if alpha == (P - 1, 0):
        x = ((-x0[1]) % P, x0[0])  # u * x0
    else:
        b = f2_pow(f2_add(F2_ONE, alpha), (P - 1) // 2)
        x = f2_mul(b, x0)
    return x if f2_sqr(x) == (a[0] % P, a[1] % P) else None


def f2_sgn0(a) -> int:
    """RFC 9380 sgn0 for m = 2."""
    s0, z0, s1 = a[0] & 1, a[0] == 0, a[1] & 1
    return s0 | (int(z0) & s1)


# ------------------------------------------------------------------------------------------------ curves
# Jacobian coordinates (X, Y, Z); infinity <=> Z == 0.  `F` bundles the field ops so G1 (Fp) and G2 (Fp2) share code.
class _Field:
    def __init__(self, add, sub, mul, sqr, neg, inv, is_zero, zero, one, b):
        self.add, self.sub, self.mul, self.sqr, self.neg, self.inv = add, sub, mul, sqr, neg, inv
        self.is_zero, self.zero, self.one, self.b = is_zero, zero, one, b


F1 = _Field(lambda a, b: (a + b) % P, lambda a, b: (a - b) % P, lambda a, b: (a * b) % P, lambda a: (a * a) % P,
            lambda a: (-a) % P, lambda a: pow(a, P - 2, P), lambda a: a % P == 0, 0, 1, 4)
F2 = _Field(f2_add, f2_sub, f2_mul, f2_sqr, f2_neg, f2_inv, f2_is_zero, F2_ZERO, F2_ONE, (4, 4))


def pt_inf(F): return (F.one, F.one, F.zero)
def pt_is_inf(F, p): return F.is_zero(p[2])
def pt_from_affine(F, a): return pt_inf(F) if a is None else (a[0], a[1], F.one)


def pt_to_affine(F, p):
    if pt_is_inf(F, p):
        return None
    zi = F.inv(p[2])
    zi2 = F.sqr(zi)
    return (F.mul(p[0], zi2), F.mul(p[1], F.mul(zi2, zi)))


def pt_double(F, p):
    if pt_is_inf(F, p):
        return p
    X, Y, Zc = p
    A = F.sqr(X); B = F.sqr(Y); C = F.sqr(B)
    D = F.sub(F.sqr(F.add(X, B)), F.add(A, C)); D = F.add(D, D)
    E = F.add(F.add(A, A), A); Fq = F.sqr(E)
    X3 = F.sub(Fq, F.add(D, D))
    C8 = F.add(C, C); C8 = F.add(C8, C8); C8 = F.add(C8, C8)
    Y3 = F.sub(F.mul(E, F.sub(D, X3)), C8)
    Z3 = F.mul(F.add(Y, Y), Zc)
    return (X3, Y3, Z3)


def pt_add(F, p, q):
    if pt_is_inf(F, p):
        return q
    if pt_is_inf(F, q):
        return p
    X1, Y1, Z1 = p
    X2, Y2, Z2 = q
    Z1Z1 = F.sqr(Z1); Z2Z2 = F.sqr(Z2)
    U1 = F.mul(X1, Z2Z2); U2 = F.mul(X2, Z1Z1)
    S1 = F.mul(Y1, F.mul(Z2, Z2Z2)); S2 = F.mul(Y2, F.mul(Z1, Z1Z1))
    if F.is_zero(F.sub(U1, U2)):
        if F.is_zero(F.sub(S1, S2)):
            return pt_double(F, p)
        return pt_inf(F)
    H = F.sub(U2, U1); Rr = F.sub(S2, S1)
    HH = F.sqr(H); HHH = F.mul(H, HH); V = F.mul(U1, HH)
    X3 = F.sub(F.sub(F.sqr(Rr), HHH), F.add(V, V))
    Y3 = F.sub(F.mul(Rr, F.sub(V, X3)), F.mul(S1, HHH))
    Z3 = F.mul(F.mul(Z1, Z2), H)
    return (X3, Y3, Z3)


def pt_neg(F, p): return (p[0], F.neg(p[1]), p[2])


def pt_mul(F, p, k: int):
    r = pt_inf(F)
    for bit in bin(k)[2:] if k else "":
        r = pt_double(F, r)
        if bit == "1":
            r = pt_add(F, r, p)
    return r


def pt_eq(F, p, q):
    a, b = pt_to_affine(F, p), pt_to_affine(F, q)
    return a == b


def on_curve(F, a) -> bool:
    if a is None:
        return True
    return F.sub(F.sqr(a[1]), F.add(F.mul(F.sqr(a[0]), a[0]), F.b)) == F.zero


def in_subgroup(F, a) -> bool:
    """Definition: [r]P == infinity (blst uses endomorphism shortcuts with the same accept set)."""
    return pt_is_inf(F, pt_mul(F, pt_from_affine(F, a), R))


# ------------------------------------------------------------------------------------------------ serialization
def g1_compress(a) -> bytes:
    if a is None:
        return bytes([0xC0]) + bytes(47)
    x, y = a
    b = bytearray(x.to_bytes(48, "big"))
    b[0] |= 0x80
    if y > (P - 1) // 2:
        b[0] |= 0x20
    return bytes(b)


def g2_compress(a) -> bytes:
    if a is None:
        return bytes([0xC0]) + bytes(95)
    (x0, x1), (y0, y1) = a
    b = bytearray(x1.to_bytes(48, "big") + x0.to_bytes(48, "big"))
    b[0] |= 0x80
    big = (y1 > (P - 1) // 2) if y1 != 0 else (y0 > (P - 1) // 2)
    if big:
        b[0] |= 0x20
    return bytes(b)


def g1_uncompress(b: bytes):
    """-> (code, affine|None).  blst `PublicKey::from_bytes` / p1 uncompress rules (SURVEY.md §8a notes)."""
    if len(b) != 48 or not (b[0] & 0x80):
        return BAD_ENCODING, None
    if b[0] & 0x40:
        if (b[0] & 0x3F) == 0 and not any(b[1:]):
            return SUCCESS, None
        return BAD_ENCODING, None
    x = int.from_bytes(bytes([b[0] & 0x1F]) + b[1:], "big")
    if x >= P:
        return BAD_ENCODING, None
    y2 = (x * x * x + 4) % P
    y = pow(y2, (P + 1) // 4, P)
    if (y * y) % P != y2:
        return POINT_NOT_ON_CURVE, None
    if (y > (P - 1) // 2) != bool(b[0] & 0x20):
        y = P - y
    return SUCCESS, (x, y)


def g2_uncompress(b: bytes):
    if len(b) != 96 or not (b[0] & 0x80):
        return BAD_ENCODING, None
    if b[0] & 0x40:
        if (b[0] & 0x3F) == 0 and not any(b[1:]):
            return SUCCESS, None
        return BAD_ENCODING, None
    x1 = int.from_bytes(bytes([b[0] & 0x1F]) + b[1:48], "big")
    x0 = int.from_bytes(b[48:], "big")
    if x1 >= P or x0 >= P:
        return BAD_ENCODING, None
    x = (x0, x1)
    y2 = f2_add(f2_mul(f2_sqr(x), x), (4, 4))
    y = f2_sqrt(y2)
    if y is None:
        return POINT_NOT_ON_CURVE, None
    big = (y[1] > (P - 1) // 2) if y[1] != 0 else (y[0] > (P - 1) // 2)
    if big != bool(b[0] & 0x20):
        y = f2_neg(y)
    return SUCCESS, (x, y)


def key_validate(b: bytes):
    """blst `PublicKey::key_validate` (crypto/bls.rs:283): uncompress, reject infinity, subgroup check."""
    code, a = g1_uncompress(b)
    if code:
        return code, None
    if a is None:
        return PK_IS_INFINITY, None
    if not in_subgroup(F1, a):
        return POINT_NOT_IN_GROUP, None
    return SUCCESS, a


# ------------------------------------------------------------------------------------------------ hash to G2
def expand_message_xmd(msg: bytes, dst: bytes, n: int) -> bytes:
    ell = (n + 31) // 32
    dst_prime = dst + bytes([len(dst)])
    b0 = hashlib.sha256(bytes(64) + msg + n.to_bytes(2, "big") + b"\x00" + dst_prime).digest()
    bi = hashlib.sha256(b0 + b"\x01" + dst_prime).digest()
    out = bi
    for i in range(2, ell + 1):
        bi = hashlib.sha256(bytes(x ^ y for x, y in zip(b0, bi)) + bytes([i]) + dst_prime).digest()
        out += bi
    return out[:n]


def hash_to_field_fp2(msg: bytes, dst: bytes = DST) -> Tuple[Fp2, Fp2]:
    u = expand_message_xmd(msg, dst, 256)
    e = [int.from_bytes(u[64 * j:64 * j + 64], "big") % P for j in range(4)]
    return (e[0], e[1]), (e[2], e[3])


SSWU_A: Fp2 = (0, 240)
SSWU_B: Fp2 = (1012, 1012)
SSWU_Z: Fp2 = (P - 2, P - 1)  # -(2 + u)


def sswu(t: Fp2):
    """Simplified SWU map to E'': y^2 = x^3 + A'x + B' (RFC 9380 6.6.2, straight-line definition)."""
    A, B, Zc = SSWU_A, SSWU_B, SSWU_Z
    t2 = f2_sqr(t)
    tv1 = f2_add(f2_mul(f2_sqr(Zc), f2_sqr(t2)), f2_mul(Zc, t2))
    if f2_is_zero(tv1):
        x1 = f2_mul(B, f2_inv(f2_mul(Zc, A)))
    else:
        x1 = f2_mul(f2_mul(f2_neg(B), f2_inv(A)), f2_add(F2_ONE, f2_inv(tv1)))
    gx1 = f2_add(f2_add(f2_mul(f2_sqr(x1), x1), f2_mul(A, x1)), B)
    y1 = f2_sqrt(gx1)
    if y1 is not None:
        x, y = x1, y1
    else:
        x = f2_mul(f2_mul(Zc, t2), x1)
        gx2 = f2_add(f2_add(f2_mul(f2_sqr(x), x), f2_mul(A, x)), B)
        y = f2_sqrt(gx2)
        assert y is not None
    if f2_sgn0(t) != f2_sgn0(y):
        y = f2_neg(y)
    return x, y


def _h(s: str) -> int: return int(s, 16)


# 3-isogeny E'' -> E' coefficients (RFC 9380 Appendix E.3; SURVEY.md Appendix A), as (c0, c1)
_K1 = [(_h("5c759507e8e333ebb5b7a9a47d7ed8532c52d39fd3a042a88b58423c50ae15d5c2638e343d9c71c6238aaaaaaaa97d6"),) * 2,
       (0, _h("11560bf17baa99bc32126fced787c88f984f87adf7ae0c7f9a208c6b4f20a4181472aaa9cb8d555526a9ffffffffc71a")),
       (_h("11560bf17baa99bc32126fced787c88f984f87adf7ae0c7f9a208c6b4f20a4181472aaa9cb8d555526a9ffffffffc71e"),
        _h("8ab05f8bdd54cde190937e76bc3e447cc27c3d6fbd7063fcd104635a790520c0a395554e5c6aaaa9354ffffffffe38d")),
       (_h("171d6541fa38ccfaed6dea691f5fb614cb14b4e7f4e810aa22d6108f142b85757098e38d0f671c7188e2aaaaaaaa5ed1"), 0)]
_K2 = [(0, P - 72), (12, P - 12), (1, 0)]
_K3 = [(_h("1530477c7ab4113b59a4c18b076d11930f7da5d4a07f649bf54439d87d27e500fc8c25ebf8c92f6812cfc71c71c6d706"),) * 2,
       (0, _h("5c759507e8e333ebb5b7a9a47d7ed8532c52d39fd3a042a88b58423c50ae15d5c2638e343d9c71c6238aaaaaaaa97be")),
       (_h("11560bf17baa99bc32126fced787c88f984f87adf7ae0c7f9a208c6b4f20a4181472aaa9cb8d555526a9ffffffffc71c"),
        _h("8ab05f8bdd54cde190937e76bc3e447cc27c3d6fbd7063fcd104635a790520c0a395554e5c6aaaa9354ffffffffe38f")),
       (_h("124c9ad43b6cf79bfbf7043de3811ad0761b0f37a1e26286b0e977c69aa274524e79097a56dc4bd9e1b371c71c718b10"), 0)]
_K4 = [(P - 432, P - 432), (0, P - 216), (18, P - 18), (1, 0)]


def _horner(coeffs, x):
    r = F2_ZERO
    for c in reversed(coeffs):
        r = f2_add(f2_mul(r, x), c)
    return r


def iso3(pt):
    x, y = pt
    xn, xd, yn, yd = _horner(_K1, x), _horner(_K2, x), _horner(_K3, x), _horner(_K4, x)
    if f2_is_zero(xd) or f2_is_zero(yd):
        return None
    return f2_mul(xn, f2_inv(xd)), f2_mul(y, f2_mul(yn, f2_inv(yd)))


H_EFF = _h("bc69f08f2ee75b3584c6a0ea91b352888e2a8e9145ad7689986ff031508ffe1329c2f178731db956d82bf015d1212b02"
           "ec0ec69d7477c1ae954cbc06689f6a359894c0adebbf6b4e8020005aaa95551")


def hash_to_g2(msg: bytes, dst: bytes = DST):
    """-> affine point of G2 (or None for infinity)."""
    u0, u1 = hash_to_field_fp2(msg, dst)
    q0, q1 = iso3(sswu(u0)), iso3(sswu(u1))
    s = pt_add(F2, pt_from_affine(F2, q0), pt_from_affine(F2, q1))
    return pt_to_affine(F2, pt_mul(F2, s, H_EFF))


# ------------------------------------------------------------------------------------------------ Fp12 and pairing
# Fp12 = Fp[w]/(w^12 - 2 w^6 + 2); u = w^6 - 1 (then u^2 = -1 and w^6 = 1 + u = xi).  An element is 12 ints.
def f12_one(): return [1] + [0] * 11


def f12_mul(a, b):
    t = [0] * 23
    for i, ai in enumerate(a):
        if ai:
            for j, bj in enumerate(b):
                if bj:
                    t[i + j] += ai * bj
    for k in range(22, 11, -1):  # w^12 = 2 w^6 - 2
        c = t[k]
        if c:
            t[k - 6] += 2 * c
            t[k - 12] -= 2 * c
    return [x % P for x in t[:12]]


def f12_from_fp2(a: Fp2, shift: int = 0):
    """a * w^shift for an Fp2 element a = a0 + a1*u = (a0 - a1) + a1*w^6; shift in 0..5."""
    r = [0] * 12
    r[shift] = (a[0] - a[1]) % P
    r[shift + 6] = a[1] % P
    return r


def f12_pow(a, e):
    r = f12_one()
    for bit in bin(e)[2:]:
        r = f12_mul(r, r)
        if bit == "1":
            r = f12_mul(r, a)
    return r


def _line(T, Q2, Pa):
    """Line through T and Q2 (affine points of E'(Fp2); tangent if equal) evaluated at P in G1, scaled by w^3:
       l = (lambda*xT - yT) - lambda*xP * w^2 + yP * w^3   (SURVEY-style sparse form).  Returns (l, T+Q2)."""
    xP, yP = Pa
    (x1, y1), (x2, y2) = T, Q2
    if x1 == x2 and y1 == y2:
        lam = f2_mul(f2_muli(f2_sqr(x1), 3), f2_inv(f2_add(y1, y1)))
    else:
        lam = f2_mul(f2_sub(y2, y1), f2_inv(f2_sub(x2, x1)))
    x3 = f2_sub(f2_sub(f2_sqr(lam), x1), x2)
    y3 = f2_sub(f2_mul(lam, f2_sub(x1, x3)), y1)
    c0 = f12_from_fp2(f2_sub(f2_mul(lam, x1), y1), 0)
    c2 = f12_from_fp2(f2_muli(f2_neg(lam), xP), 2)
    l = [(c0[i] + c2[i]) % P for i in range(12)]
    l[3] = (l[3] + yP) % P
    return l, (x3, y3)


def miller_loop(Qa, Pa):
    """f_{|z|,Q}(P) for affine Q in E'(Fp2), P in E(Fp); 1 if either is infinity."""
    if Qa is None or Pa is None:
        return f12_one()
    f = f12_one()
    T = Qa
    for bit in bin(Z_ABS)[3:]:
        l, T = _line(T, T, Pa)
        f = f12_mul(f12_mul(f, f), l)
        if bit == "1":
            l, T = _line(T, Qa, Pa)
            f = f12_mul(f, l)
    return f


FINAL_EXP = (P ** 12 - 1) // R


def pairing_check(pairs: Sequence[Tuple[object, object]]) -> bool:
    """prod e(P_i, Q_i) == 1 for affine (G1, G2) pairs."""
    f = f12_one()
    for Pa, Qa in pairs:
        f = f12_mul(f, miller_loop(Qa, Pa))
    return f12_pow(f, FINAL_EXP) == f12_one()


# ------------------------------------------------------------------------------------------------ wrapper semantics
G1_GEN_NEG = (G1_GEN[0], P - G1_GEN[1])


def sk_to_pk(sk: int) -> bytes:
    return g1_compress(pt_to_affine(F1, pt_mul(F1, pt_from_affine(F1, G1_GEN), sk)))


def sign(sk: int, msg: bytes) -> bytes:
    return g2_compress(pt_to_affine(F2, pt_mul(F2, pt_from_affine(F2, hash_to_g2(msg)), sk)))


def _core_aggregate_verify(pks_aff: List[object], msgs: List[bytes], sig_aff) -> int:
    """blst `Signature::aggregate_verify(sig_groupcheck=true, ...)` on already-decoded inputs."""
    if len(pks_aff) == 0 or len(pks_aff) != len(msgs):
        return VERIFY_FAIL
    for a in pks_aff:
        if a is None:
            return VERIFY_FAIL  # PAIRING_Aggregate rejects an infinite public key
    if sig_aff is not None and not in_subgroup(F2, sig_aff):
        return VERIFY_FAIL
    pairs = [(a, hash_to_g2(m)) for a, m in zip(pks_aff, msgs)]
    pairs.append((G1_GEN_NEG, sig_aff))
    return SUCCESS if pairing_check(pairs) else VERIFY_FAIL


def fast_aggregate_verify(pks: Sequence[bytes], msg: bytes, sig: bytes) -> int:
    """crypto/bls.rs:114-132.  Codes 1,2,3,6 correspond to Err(Error::BLST(..)); 5 to Err(InvalidSignature)."""
    affs = []
    for b in pks:
        code, a = key_validate(b)
        if code:
            return code
        affs.append(a)
    code, s = g2_uncompress(sig)
    if code:
        return code
    if not affs:
        return VERIFY_FAIL  # AggregatePublicKey::aggregate(&[]) errors -> wrapper maps to InvalidSignature
    agg = pt_inf(F1)
    for a in affs:
        agg = pt_add(F1, agg, pt_from_affine(F1, a))
    return _core_aggregate_verify([pt_to_affine(F1, agg)], [msg], s)


def verify_signature(pk: bytes, msg: bytes, sig: bytes) -> int:
    """crypto/bls.rs:64-77."""
    code, a = key_validate(pk)
    if code:
        return code
    code, s = g2_uncompress(sig)
    if code:
        return code
    return _core_aggregate_verify([a], [msg], s)


def aggregate_verify(pks: Sequence[bytes], msgs: Sequence[bytes], sig: bytes) -> int:
    """crypto/bls.rs:95-112 (no message-distinctness requirement)."""
    affs = []
    for b in pks:
        code, a = key_validate(b)
        if code:
            return code
        affs.append(a)
    code, s = g2_uncompress(sig)
    if code:
        return code
    return _core_aggregate_verify(affs, list(msgs), s)


def eth_fast_aggregate_verify(pks: Sequence[bytes], msg: bytes, sig: bytes) -> int:
    """crypto/bls.rs:150-160."""
    if len(pks) == 0 and sig == bytes([0xC0]) + bytes(95):
        return SUCCESS
    return fast_aggregate_verify(pks, msg, sig)


def aggregate(sigs: Sequence[bytes]):
    """crypto/bls.rs:79-93 -> (code, 96 bytes | None)."""
    if len(sigs) == 0:
        return EMPTY_AGGREGATE, None
    affs = []
    for b in sigs:
        code, a = g2_uncompress(b)
        if code:
            return code, None
        affs.append(a)
    acc = pt_inf(F2)
    for a in affs:
        if a is not None and not in_subgroup(F2, a):
            return POINT_NOT_IN_GROUP, None
        acc = pt_add(F2, acc, pt_from_affine(F2, a))
    return SUCCESS, g2_compress(pt_to_affine(F2, acc))


def eth_aggregate_public_keys(pks: Sequence[bytes]):
    """crypto/bls.rs:135-148 -> (code, 48 bytes | None)."""
    if len(pks) == 0:
        return EMPTY_AGGREGATE, None
    acc = pt_inf(F1)
    for b in pks:
        code, a = key_validate(b)
        if code:
            return code, None
        acc = pt_add(F1, acc, pt_from_affine(F1, a))
    return SUCCESS, g1_compress(pt_to_affine(F1, acc))
