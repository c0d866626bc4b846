"""Curve points whose order is not r: generators shared by the CPU check (tests/test_torsion_cases.py) and the device
run (tests/test_torsion_gpu.py).  No device code here.

E(Fp) has h1 r points and E'(Fp2) has h2 r points.  A point of small order l (l | h) and a valid point plus such a
component (Q + T) are the only inputs that drive the double-and-add ladders of the subgroup checks and of the cofactor
clearing (jac_mul_u64 / jac_mul_u64_jac, curve.cuh) into their exceptional branches: the accumulator meets the base point
(doubling), its negation (inverse) or infinity.  Every case carries its expected code from the definition-level Python
oracle ([r]P == infinity, oracle/bls_oracle.py) and the exceptional branches it reaches, found by replaying the ladder on
the accumulator's multiple modulo the base point's order (no curve arithmetic).

Everything is seeded; B200_SOAK_SCALE scales the case counts like the other soaks."""
from __future__ import annotations

import hashlib
import math
import os
import random

from oracle import bls_oracle as bo

P, R, Z_ABS = bo.P, bo.R, bo.Z_ABS
Z = -Z_ABS
F1, F2 = bo.F1, bo.F2
SCALE = float(os.environ.get("B200_SOAK_SCALE", "1"))

H1 = (Z - 1) ** 2 // 3
H1_PRIMES = {3: 1, 11: 2, 10177: 2, 859267: 2, 52437899: 2}           # l: exponent in h1
H2 = (Z ** 8 - 4 * Z ** 7 + 5 * Z ** 6 - 4 * Z ** 4 + 6 * Z ** 3 - 4 * Z ** 2 - 4 * Z + 13) // 9
H2_SMALL = {13: 2, 23: 2, 2713: 1, 11953: 1, 262069: 1}
H2_Q = H2 // math.prod(l ** e for l, e in H2_SMALL.items())            # the 135-digit prime
N1, N2 = H1 * R, H2 * R                                                 # #E(Fp), #E'(Fp2)
BRANCHES_MIXED = ("madd_dbl", "madd_inv", "madd_inf")                   # jac_add_mixed: p == q, p == -q, p at infinity
BRANCHES_GENERAL = ("add_dbl", "add_inv", "add_inf")                    # jac_add: p == q, p == -q, an operand at infinity


def _n(x):
    return max(1, int(x * SCALE))


# ------------------------------------------------------------------------------------------------ affine helpers
def mul(F, a, k):
    """[k]a for affine a (None = infinity), any integer k."""
    if k < 0:
        return neg(F, mul(F, a, -k))
    return bo.pt_to_affine(F, bo.pt_mul(F, bo.pt_from_affine(F, a), k))


def add(F, a, b):
    return bo.pt_to_affine(F, bo.pt_add(F, bo.pt_from_affine(F, a), bo.pt_from_affine(F, b)))


def neg(F, a):
    return None if a is None else (a[0], F.neg(a[1]))


def g1_random(rnd):
    while True:
        x = rnd.randrange(P)
        y2 = (x * x * x + 4) % P
        y = pow(y2, (P + 1) // 4, P)
        if y * y % P == y2:
            return (x, y if rnd.getrandbits(1) else P - y)


def g2_random(rnd):
    while True:
        x = (rnd.randrange(P), rnd.randrange(P))
        y = bo.f2_sqrt(bo.f2_add(bo.f2_mul(bo.f2_sqr(x), x), (4, 4)))
        if y is not None:
            return (x, y if rnd.getrandbits(1) else bo.f2_neg(y))


def torsion_point(F, n_total, ell, exp, rnd, rand_pt):
    """A point of order exactly `ell` (ell^exp || n_total / r, and the l-part has exponent l: ell_part_exponent):
    [n_total / ell^exp] of random points until one is finite."""
    while True:
        t = mul(F, rand_pt(rnd), n_total // ell ** exp)
        if t is not None:
            return t


def ell_part_exponent(F, n_total, ell, exp, rnd, rand_pt, tries=3):
    """The exponent of the l-primary part: 1 if [n / l^exp]P is killed by l for every random P (so for exp = 2 it is
    Z/l x Z/l), else l^2 (a cyclic factor of order l^2 exists)."""
    for _ in range(tries):
        u = mul(F, rand_pt(rnd), n_total // ell ** exp)
        if u is not None and mul(F, u, ell) is not None:
            return ell ** 2
    return ell


# ------------------------------------------------------------------------------------------------ endomorphisms
def _g1_beta():
    """The cube root of unity beta with phi(G) = (beta x, y) = -[z^2] G on G1 (the product's B200_FP_BETA)."""
    b = pow(2, (P - 1) // 3, P)
    want = neg(F1, mul(F1, bo.G1_GEN, Z_ABS * Z_ABS))
    return b if (b * bo.G1_GEN[0] % P, bo.G1_GEN[1]) == want else b * b % P


BETA = _g1_beta()
_XI = (1, 1)
PSI_X = bo.f2_inv(bo.f2_pow(_XI, (P - 1) // 3))
PSI_Y = bo.f2_inv(bo.f2_pow(_XI, (P - 1) // 2))


def phi(a):
    return None if a is None else (BETA * a[0] % P, a[1])


def psi(a):
    """untwist-Frobenius-twist on E'(Fp2): (conj(x) cx, conj(y) cy); psi(Q) = [z]Q on G2."""
    if a is None:
        return None
    conj = lambda v: (v[0], (-v[1]) % P)   # noqa: E731
    return (bo.f2_mul(conj(a[0]), PSI_X), bo.f2_mul(conj(a[1]), PSI_Y))


def dlog(F, target, base, order):
    """k in [0, order) with [k]base == target, or None (baby-step giant-step over affine points)."""
    m = math.isqrt(order) + 1
    baby, cur = {}, None
    for j in range(m):
        baby.setdefault(cur, j)
        cur = add(F, cur, base)
    step = neg(F, mul(F, base, m))
    g = target
    for i in range(m + 1):
        if g in baby:
            return (i * m + baby[g]) % order
        g = add(F, g, step)
    return None


def cube_roots_of_unity(ell):
    """The non-trivial cube roots of 1 mod ell (the possible eigenvalues of phi on the l-torsion)."""
    if ell % 3 != 1:
        return []
    return [x for x in range(2, ell) if (x * x + x + 1) % ell == 0]


def psi_eigen(ell, rnd):
    """Eigenvalues of psi on E'[l], found by observation: for cyclic l-torsion psi(T) = [lam]T for one lam; on
    Z/l x Z/l the projections V = psi(T) - [mu]T that are finite and satisfy psi(V) = [lam]V.  -> {lam: V}."""
    t = torsion_point(F2, N2, ell, H2_SMALL[ell], rnd, g2_random)
    if H2_SMALL[ell] == 1:
        lam = dlog(F2, psi(t), t, ell)
        assert lam is not None, ell
        return {lam: t}
    out = {}
    pt = psi(t)
    for mu in range(ell):
        v = add(F2, pt, neg(F2, mul(F2, t, mu)))
        if v is None:
            continue
        lam = dlog(F2, psi(v), v, ell)
        if lam is not None:
            out.setdefault(lam, v)
    return out


# ------------------------------------------------------------------------------------------------ ladder replay
def ladder_branches(order, mixed, k=Z_ABS):
    """Exceptional branches taken by [k] base (left-to-right double-and-add from infinity, curve.cuh) for a base point
    of the given order: the accumulator is [a] base, so at an add it is infinity iff a = 0, the base iff a = 1 and its
    negation iff a = -1 (mod order).  The first add onto the initial infinity is not exceptional.  order 1: the base
    itself is infinity (general add only)."""
    out, a, started = set(), 0, False
    for bit in range(63, -1, -1):
        if started:
            a = 2 * a % order
        if (k >> bit) & 1:
            pre = "madd" if mixed else "add"
            if order == 1:
                out.add("add_inf")
            elif a == 0:
                if started:
                    out.add(pre + "_inf")
            elif a == 1:
                out.add(pre + "_dbl")
            elif a == order - 1:
                out.add(pre + "_inv")
            a = (a + 1) % order
            started = True
    return out


def g1_check_branches(order):
    """g1_in_subgroup(_lazy): t = [|z|]P (mixed adds), then [|z|]t (general adds)."""
    return ladder_branches(order, True) | ladder_branches(order // math.gcd(order, Z_ABS), False)


def g2_check_branches(order):
    """g2_in_subgroup: [|z|]Q with mixed adds."""
    return ladder_branches(order, True)


def order_of(F, a, bound):
    """Exact order of a, given a multiple `bound` of it (a small product of primes)."""
    if a is None:
        return 1
    o = bound
    for ell in _factor_small(bound):
        while o % ell == 0 and mul(F, a, o // ell) is None:
            o //= ell
    return o


def _factor_small(n):
    return [l for l in list(H1_PRIMES) + list(H2_SMALL) if n % l == 0]


def clear_cofactor_branches(a, order):
    """g2_clear_cofactor's two ladders: [|z|]P and [|z|]([z]P + psi(P)), both with general adds."""
    t2 = add(F2, mul(F2, a, Z), psi(a))
    return ladder_branches(order, False) | ladder_branches(order_of(F2, t2, order), False)


# ------------------------------------------------------------------------------------------------ the cases
def _negated(kw):
    """The fields of -P: its secret (if it has one) is R - s."""
    return {**kw, "sk": R - kw["sk"]} if "sk" in kw else kw


def _case(F, a, family, order, **kw):
    comp = bo.g1_compress if F is F1 else bo.g2_compress
    return dict(pt=a, enc=comp(a), family=family, order=order, **kw)


def g1_cases(seed=1):
    """-> dict: cases (both sign encodings of every point; fields pt, enc, family, order (of the small-order part; r
    for valid keys, r m for Q + T), code (bo.key_validate), branches, sk (valid keys and Q + T: the secret of Q)),
    structure {l: exponent}, eigen {l: [(lam, T)]}."""
    rnd = random.Random(0x7051 + seed)
    structure = {l: ell_part_exponent(F1, N1, l, e, rnd, g1_random) for l, e in H1_PRIMES.items()}
    base = {l: [torsion_point(F1, N1, l, H1_PRIMES[l], rnd, g1_random) for _ in range(1 if l == 3 else 3)] for l in H1_PRIMES}
    pts = []
    # pure torsion of every prime order: multiples of a few base points, both sheets of Z/l x Z/l
    for l, ts in base.items():
        n = 1 if l == 3 else _n(12)
        for t in ts:
            for _ in range(n):
                pts.append((mul(F1, t, rnd.randrange(1, l)), "torsion", l, {}))
        if len(ts) > 1:
            pts.append((add(F1, ts[0], ts[1]), "torsion", l, {}))
    # composite orders
    for combo in ((3, 11), (3, 10177), (11, 859267), (10177, 52437899), (3, 52437899), (11, 10177, 859267),
                  tuple(H1_PRIMES)):
        for _ in range(_n(6)):
            t = None
            for l in combo:
                t = add(F1, t, mul(F1, base[l][rnd.randrange(len(base[l]))], rnd.randrange(1, l)))
            pts.append((t, "torsion", math.prod(combo), {}))
    # phi eigenspaces: T_lam = phi(T) - [mu]T
    eigen = {}
    for l in H1_PRIMES:
        roots = cube_roots_of_unity(l)
        eigen[l] = []
        for lam in roots:
            mu = next(r for r in roots if r != lam)
            v = add(F1, phi(base[l][0]), neg(F1, mul(F1, base[l][0], mu)))
            eigen[l].append((lam, v))
            for _ in range(_n(10)):
                pts.append((mul(F1, v, rnd.randrange(1, l)), "eigen", l, {"lam": lam}))
    # Q + T and -Q + T, and the valid keys Q as controls
    torsion_pool = [(a, o) for a, f, o, _ in pts]
    sk0 = int.from_bytes(hashlib.sha256(b"torsion/g1 sk%d" % seed).digest(), "big") % R
    n_keys = _n(190)
    step = mul(F1, bo.G1_GEN, 1 + sk0 % 1000)
    q = mul(F1, bo.G1_GEN, sk0)
    for i in range(n_keys):
        s = (sk0 + i * (1 + sk0 % 1000)) % R
        pts.append((q, "valid", R, {"sk": s}))
        for sign in (1, -1):
            t, o = torsion_pool[rnd.randrange(len(torsion_pool))]
            pts.append((add(F1, q if sign > 0 else neg(F1, q), t), "Q+T" if sign > 0 else "-Q+T", R * o,
                        {"sk": s if sign > 0 else R - s, "t_order": o}))
        q = add(F1, q, step)
    cases = []
    for a, fam, o, kw in pts:
        for b, k in ((a, kw), (neg(F1, a), _negated(kw))):
            c = _case(F1, b, fam, o, **k)
            c["code"] = bo.key_validate(c["enc"])[0]
            c["branches"] = g1_check_branches(o)
            cases.append(c)
    return {"cases": cases, "structure": structure, "eigen": eigen, "base": base}


def g2_cases(seed=1):
    """The same families on E'(Fp2) as 96-byte encodings (code: aggregate([sig]) by the definition, i.e. 0 or 3), plus
    sigma + T for valid signatures sigma = s H(m) (fields sk, msg), and cc_branches: the exceptional branches of
    g2_clear_cofactor's ladders on the pure-torsion points."""
    rnd = random.Random(0x7052 + seed)
    structure = {l: ell_part_exponent(F2, N2, l, e, rnd, g2_random) for l, e in H2_SMALL.items()}
    base = {l: [torsion_point(F2, N2, l, H2_SMALL[l], rnd, g2_random) for _ in range(2 if H2_SMALL[l] == 2 else 1)] for l in H2_SMALL}
    eigen = {l: psi_eigen(l, rnd) for l in H2_SMALL}
    pts = []
    for l, ts in base.items():
        for t in ts:
            for _ in range(_n(8)):
                pts.append((mul(F2, t, rnd.randrange(1, l)), "torsion", l, {}))
        if len(ts) > 1:
            pts.append((add(F2, ts[0], ts[1]), "torsion", l, {}))
    for combo in ((13, 23), (13, 2713), (23, 262069), (2713, 11953, 262069), (13, 11953), tuple(H2_SMALL)):
        for _ in range(_n(5)):
            t = None
            for l in combo:
                t = add(F2, t, mul(F2, base[l][rnd.randrange(len(base[l]))], rnd.randrange(1, l)))
            pts.append((t, "torsion", math.prod(combo), {}))
    for l, ev in eigen.items():
        if H2_SMALL[l] == 2:
            for lam, v in ev.items():
                for _ in range(_n(8)):
                    pts.append((mul(F2, v, rnd.randrange(1, l)), "eigen", l, {"lam": lam}))
    torsion_pool = [(a, o) for a, f, o, _ in pts]
    msgs = [hashlib.sha256(b"torsion/g2 m%d" % j).digest() for j in range(4)]
    hs = [bo.hash_to_g2(m) for m in msgs]
    sk0 = int.from_bytes(hashlib.sha256(b"torsion/g2 sk%d" % seed).digest(), "big") % R
    d = 1 + sk0 % 1000
    for j, (m, h) in enumerate(zip(msgs, hs)):
        sig, step = mul(F2, h, sk0), mul(F2, h, d)
        for i in range(_n(26)):
            s = (sk0 + i * d) % R
            pts.append((sig, "valid", R, {"sk": s, "msg": m}))
            t, o = torsion_pool[rnd.randrange(len(torsion_pool))]
            pts.append((add(F2, sig, t), "sigma+T", R * o, {"sk": s, "msg": m, "t_order": o}))
            sig = add(F2, sig, step)
    cases = []
    for a, fam, o, kw in pts:
        for b, k in ((a, kw), (neg(F2, a), _negated(kw))):
            c = _case(F2, b, fam, o, **k)
            c["code"] = bo.SUCCESS if bo.in_subgroup(F2, b) else bo.POINT_NOT_IN_GROUP
            c["branches"] = g2_check_branches(o)
            if o < R:
                c["cc_branches"] = clear_cofactor_branches(b, o)
            cases.append(c)
    return {"cases": cases, "structure": structure, "eigen": eigen, "base": base}


def sswu_inputs(n_random, seed=1):
    """u for the map stage: 0 (the tv1 == 0 branch), +-1, the sgn0 edges (c0 = 0 or c1 = 0, with either parity), p - 1,
    and random u."""
    rnd = random.Random(0x7053 + seed)
    us = [(0, 0), (1, 0), (P - 1, 0), (0, 1), (0, P - 1), (1, 1), (P - 1, P - 1), (2, 0), (0, 2)]
    for _ in range(8):
        a = rnd.randrange(1, P)
        us += [(a, 0), (0, a), (a | 1, 0), (0, a | 1), (a & ~1, 0), (0, a & ~1)]
    us += [(rnd.randrange(P), rnd.randrange(P)) for _ in range(n_random)]
    return us
