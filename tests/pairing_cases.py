"""Cases and plain-integer references for the device pairing (b200_pairing_eval); no device code.

Representation.  The device stores an Fp12 as twelve Fp slots in memory order c0.c0.c0, c0.c0.c1, c0.c1.c0, ..., c1.c2.c1
(Fp6 = Fp2[v]/(v^3 - xi), Fp12 = Fp6[w]/(w^2 - v), xi = 1 + u): the Fp2 coefficient c_h.c_j sits at w^(2j + h) and
w^6 = xi.  The oracle (bo.f12_*) works in Fp[w]/(w^12 - 2 w^6 + 2) with u = w^6 - 1, so a0 + a1 u at w^k is (a0 - a1) at
w^k plus a1 at w^(k + 6) (bo.f12_from_fp2), and back: a1 = r[k + 6], a0 = r[k] + r[k + 6].  The device holds x R mod p
(R = 2^384); every value here is a plain residue ("real") unless it is called raw.

The Miller loop is restated from pairing.cuh / curve.cuh: Jacobian T on the M-twist, doubling with Z3 = 2 Y Z, addition
with Z3 = Z H, the sparse line A + B v + C v w, the closing conjugation (z < 0).  Those choices fix the representative,
so the restated value is the device's bit for bit.  With P given as G1Pre (X Z, Y, Z^3) the lane-parallel programs scale
every line by lambda = Z^3 in Fp (their A picks up the factor explicitly, B and C through X Z and Y); a product of E lines
picks up lambda^E, with E counted by the same loop (miller_lambda_exponent)."""
from __future__ import annotations

import random
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from oracle import bls_oracle as bo  # noqa: E402

P, R, Z_ABS = bo.P, bo.R, bo.Z_ABS
RM = 1 << 384
RINV = pow(RM, -1, P)
FINAL_EXP3 = 3 * bo.FINAL_EXP          # the device's exponent: 3 (p^12 - 1) / r
XI = (1, 1)
W = 145                                # words of a b200_pairing_eval record
FOLD_SIZES = (1, 2, 31, 32, 33, 63, 64, 65, 1023, 1024, 1025, 4097)


# ------------------------------------------------------------------------------------------------------ representation
def mont(x: int) -> int: return x * RM % P
def real(x: int) -> int: return x * RINV % P


def slot_power(m: int) -> int:
    """w-power of the m-th Fp2 coefficient in memory order (c0.c0, c0.c1, c0.c2, c1.c0, c1.c1, c1.c2)."""
    return 2 * (m % 3) + m // 3


def to_oracle(s):
    """12 real slots (memory order) -> the oracle's 12 coefficients."""
    r = [0] * 12
    for m in range(6):
        a0, a1 = s[2 * m], s[2 * m + 1]
        k = slot_power(m)
        r[k] = (r[k] + a0 - a1) % P
        r[k + 6] = (r[k + 6] + a1) % P
    return r


def from_oracle(r):
    s = [0] * 12
    for m in range(6):
        k = slot_power(m)
        s[2 * m], s[2 * m + 1] = (r[k] + r[k + 6]) % P, r[k + 6] % P
    return s


def fp2s(s):
    """12 slots -> six Fp2 pairs in memory order."""
    return [(s[2 * m], s[2 * m + 1]) for m in range(6)]


def slots(f2list):
    return [x for a in f2list for x in a]


ONE = [1] + [0] * 11                   # the same in both bases


def conj(s):
    """f -> conj(f) (w -> -w, = f^(p^6)): negate c1."""
    return s[:6] + [(-x) % P for x in s[6:]]


# --------------------------------------------------------------------------------------- tower inverse (for inputs only)
def _mxi(a): return ((a[0] - a[1]) % P, (a[0] + a[1]) % P)


def _f6_mul(a, b):
    m, ad = bo.f2_mul, bo.f2_add
    c0 =ad(m(a[0], b[0]), _mxi(ad(m(a[1], b[2]), m(a[2], b[1]))))
    c1 = ad(ad(m(a[0], b[1]), m(a[1], b[0])), _mxi(m(a[2], b[2])))
    c2 = ad(ad(m(a[0], b[2]), m(a[1], b[1])), m(a[2], b[0]))
    return (c0, c1, c2)


def _f6_inv(a):
    m, sb, ad = bo.f2_mul, bo.f2_sub, bo.f2_add
    c0 = sb(bo.f2_sqr(a[0]), _mxi(m(a[1], a[2])))
    c1 = sb(_mxi(bo.f2_sqr(a[2])), m(a[0], a[1]))
    c2 = sb(bo.f2_sqr(a[1]), m(a[0], a[2]))
    d = ad(m(a[0], c0), _mxi(ad(m(a[2], c1), m(a[1], c2))))
    di = bo.f2_inv(d) if not bo.f2_is_zero(d) else (0, 0)
    return (m(c0, di), m(c1, di), m(c2, di))


def inverse(s):
    """f^-1 through the tower (0 -> 0); the CPU test ties it to f * f^-1 == 1 in the oracle's field."""
    e = fp2s(s)
    a0, a1 = tuple(e[:3]), tuple(e[3:])
    t1 = _f6_mul(a1, a1)
    t = tuple(bo.f2_sub(x, y) for x, y in zip(_f6_mul(a0, a0), (_mxi(t1[2]), t1[0], t1[1])))
    ti = _f6_inv(t)
    return slots(list(_f6_mul(a0, ti)) + [bo.f2_neg(x) for x in _f6_mul(a1, ti)])


# ---------------------------------------------------------------------------------------------- Frobenius as a linear map
_FROB = {}


def _frob_images(k):
    """(w^i)^(p^k) for i = 0..11 in the oracle basis."""
    if k not in _FROB:
        wp = bo.f12_pow([0, 1] + [0] * 10, P ** k)
        imgs = [ONE]
        for _ in range(11):
            imgs.append(bo.f12_mul(imgs[-1], wp))
        _FROB[k] = imgs
    return _FROB[k]


def frobenius(r, k):
    """r^(p^k) in the oracle basis: the coefficients are in Fp, so only w moves."""
    out = [0] * 12
    for c, img in zip(r, _frob_images(k)):
        if c:
            for j in range(12):
                out[j] += c * img[j]
    return [x % P for x in out]


def easy_part(r):
    """r^((p^6 - 1)(p^2 + 1)) in the oracle basis (zero stays zero): the cyclotomic-subgroup inputs."""
    s = from_oracle(r)
    t = bo.f12_mul(to_oracle(conj(s)), to_oracle(inverse(s)))
    return bo.f12_mul(frobenius(t, 2), t)


def final_exp(r):
    """The definition: r^(3 (p^12 - 1) / r), oracle basis."""
    return bo.f12_pow(r, FINAL_EXP3)


# ------------------------------------------------------------------------------------------------ restated Miller loop
f2_add, f2_sub, f2_mul, f2_sqr, f2_neg = bo.f2_add, bo.f2_sub, bo.f2_mul, bo.f2_sqr, bo.f2_neg


def f2_mul_fp(a, k): return (a[0] * k % P, a[1] * k % P)
def f2_dbl(a): return f2_add(a, a)


def jac_double(t):
    """curve.cuh jac_double (dbl-2009-l)."""
    X, Y, Z = t
    A, B = f2_sqr(X), f2_sqr(Y)
    C = f2_sqr(B)
    D = f2_dbl(f2_sub(f2_sub(f2_sqr(f2_add(X, B)), A), C))
    E = f2_add(f2_dbl(A), A)
    x3 = f2_sub(f2_sqr(E), f2_dbl(D))
    y3 = f2_sub(f2_mul(E, f2_sub(D, x3)), f2_dbl(f2_dbl(f2_dbl(C))))
    return (x3, y3, f2_dbl(f2_mul(Y, Z)))


def miller_double_step(t, xp, yp, z3p=1):
    """pairing.cuh miller_double_step; z3p != 1: the lane-parallel program's A * Z^3 (xp, yp are then X Z and Y)."""
    X, Y, Z = t
    xx, yy, zz = f2_sqr(X), f2_sqr(Y), f2_sqr(Z)
    e = f2_add(f2_dbl(xx), xx)
    A = f2_mul_fp(f2_sub(f2_mul(e, X), f2_dbl(yy)), z3p)
    B = f2_neg(f2_mul_fp(f2_mul(e, zz), xp))
    t2 = jac_double(t)
    C = f2_mul_fp(f2_mul(t2[2], zz), yp)
    return t2, A, B, C


def miller_add_step(t, q, xp, yp, z3p=1):
    X, Y, Z = t
    zz = f2_sqr(Z)
    zzz = f2_mul(zz, Z)
    h = f2_sub(f2_mul(q[0], zz), X)
    rr = f2_sub(f2_mul(q[1], zzz), Y)
    z3 = f2_mul(Z, h)
    A = f2_mul_fp(f2_sub(f2_mul(rr, q[0]), f2_mul(q[1], z3)), z3p)
    B = f2_neg(f2_mul_fp(rr, xp))
    C = f2_mul_fp(z3, yp)
    hh = f2_sqr(h)
    hhh = f2_mul(hh, h)
    v = f2_mul(X, hh)
    x3 = f2_sub(f2_sub(f2_sqr(rr), hhh), f2_dbl(v))
    y3 = f2_sub(f2_mul(rr, f2_sub(v, x3)), f2_mul(Y, hhh))
    return (x3, y3, z3), A, B, C


def line_slots(A, B, C):
    """A + B v + C v w as 12 slots: c0.c0 = A, c0.c1 = B, c1.c1 = C."""
    return slots([A, B, (0, 0), (0, 0), C, (0, 0)])


def miller_loop(p, q, z3p=1):
    """The device's f for P = (xp, yp) (or G1Pre (X Z, Y) with z3p = Z^3) and affine Q = ((x0, x1), (y0, y1)); None is
    infinity.  Returns 12 real slots."""
    if p is None or q is None:
        return list(ONE)
    xp, yp = p
    t = (q[0], q[1], (1, 0))
    f = bo.f12_one()
    first = True
    for bit in range(62, -1, -1):
        if not first:
            f = bo.f12_mul(f, f)
        first = False
        t, A, B, C = miller_double_step(t, xp, yp, z3p)
        f = bo.f12_mul(f, to_oracle(line_slots(A, B, C)))
        if (Z_ABS >> bit) & 1:
            t, A, B, C = miller_add_step(t, q, xp, yp, z3p)
            f = bo.f12_mul(f, to_oracle(line_slots(A, B, C)))
    return conj(from_oracle(f))


def miller_lambda_exponent():
    """E with VM(P, Q, Z) = direct(P, Q) * (Z^3)^E: every line carries one factor, every squaring doubles the count."""
    e, first = 0, True
    for bit in range(62, -1, -1):
        if not first:
            e *= 2
        first = False
        e += 1 + ((Z_ABS >> bit) & 1)
    return e


def scale(s, k):
    return [x * k % P for x in s]


def pow_z(r):
    return bo.f12_pow(r, Z_ABS)


# ------------------------------------------------------------------------------------------------------------- records
def pack(rows, flags=None):
    """Lists of up to 12 raw slot values (+ flags) -> uint32[n, 145]."""
    import numpy as np
    n = len(rows)
    buf = bytearray(n * W * 4)
    for i, row in enumerate(rows):
        base = i * W * 4
        for s, v in enumerate(row):
            buf[base + 48 * s: base + 48 * s + 48] = int(v).to_bytes(48, "little")
        if flags is not None:
            buf[base + 576: base + 580] = int(flags[i]).to_bytes(4, "little")
    return np.frombuffer(bytes(buf), dtype=np.uint32).reshape(n, W).copy()


def unpack(arr, n_slots=12):
    """uint32[n, 145] -> lists of raw slot ints."""
    b = arr.astype("<u4").tobytes()
    out = []
    for i in range(arr.shape[0]):
        base = i * W * 4
        out.append([int.from_bytes(b[base + 48 * s: base + 48 * s + 48], "little") for s in range(n_slots)])
    return out


def to_raw(s): return [mont(x) for x in s]
def to_real(s): return [real(x) for x in s]


# ---------------------------------------------------------------------------------------------------------- generators
def edge_fp():
    """The raw edge values of tests/test_fp_device_gpu.py: 0, 1, p - 1, (p +- 1)/2, R mod p, all-ones limbs, p minus one
    limb unit, [2^380, p), ..."""
    from tests.test_fp_device_gpu import _edge_fp
    return _edge_fp()


def tower_elements(seed, n_random=2000):
    """Raw Fp12 elements: every edge value in every slot, one edge value in all slots, sparse elements, one, -1, random."""
    rnd = random.Random(seed)
    edge = edge_fp()
    els = []
    for k in range(len(edge)):                                 # edge values cycle through all twelve slots
        els.append([edge[(k + 7 * j) % len(edge)] for j in range(12)])
    els += [[e] * 12 for e in edge[:: max(1, len(edge) // 24)]]
    for j in range(12):                                        # sparse: one non-zero coefficient
        els.append([0] * j + [rnd.randrange(P)] + [0] * (11 - j))
        els.append([0] * j + [edge[rnd.randrange(len(edge))]] + [0] * (11 - j))
    els.append(to_raw(ONE))
    els.append(to_raw([P - 1] + [0] * 11))
    els += [[rnd.randrange(P) for _ in range(12)] for _ in range(n_random)]
    els += [[rnd.randrange(1 << 380, P) for _ in range(12)] for _ in range(n_random // 10)]
    return els


def tower_pairs(seed, n_random=2000):
    """Operand pairs for the products: edge x random, random x random, (a, a^-1), (a, conj(a)), (a, one), (a, -1)."""
    rnd = random.Random(seed)
    els = tower_elements(seed, n_random)
    pairs = [(a, els[rnd.randrange(len(els))]) for a in els]
    one, m1 = to_raw(ONE), to_raw([P - 1] + [0] * 11)
    for a in els[:: max(1, len(els) // 64)]:
        ar = to_real(a)
        if any(ar):
            pairs.append((a, to_raw(inverse(ar))))
        pairs.append((a, to_raw(conj(ar))))
        pairs += [(a, one), (a, m1)]
    return pairs


def cyclotomic_elements(seed, n):
    """Raw elements of the cyclotomic subgroup: random elements and Miller-like sparse ones through the easy part."""
    rnd = random.Random(seed)
    out = []
    for i in range(n):
        r = [rnd.randrange(P) for _ in range(12)] if i % 4 else to_oracle([rnd.randrange(P)] * 4 + [0] * 8)
        out.append(to_raw(from_oracle(easy_part(r))))
    out.append(to_raw(ONE))                                    # (-1 is not in it: p^4 - p^2 + 1 is odd)
    return out


def g1_mul(k): return bo.pt_to_affine(bo.F1, bo.pt_mul(bo.F1, bo.pt_from_affine(bo.F1, bo.G1_GEN), k))
def g2_mul(k): return bo.pt_to_affine(bo.F2, bo.pt_mul(bo.F2, bo.pt_from_affine(bo.F2, bo.G2_GEN), k))


def g1_points(seed, n_random):
    """Real affine G1 inputs: the generator, -g1, random multiples and their negatives, and edge coordinates (the formulas
    are polynomial identities, so P need not be on the curve)."""
    rnd = random.Random(seed)
    pts = [bo.G1_GEN, bo.G1_GEN_NEG]
    for _ in range(n_random):
        a = g1_mul(rnd.randrange(1, R))
        pts += [a, (a[0], (-a[1]) % P)]
    edge = edge_fp()
    pts += [(real(edge[rnd.randrange(len(edge))]), real(edge[rnd.randrange(len(edge))])) for _ in range(n_random)]
    pts += [(real(0), real(1)), (real(P - 1), real(P - 1)), (real(RM % P), 0)]
    return pts


def g2_points(seed, n_random):
    rnd = random.Random(seed)
    return [bo.G2_GEN] + [g2_mul(rnd.randrange(1, R)) for _ in range(n_random)]


def lambda_values(seed, n_random):
    """Real lambda = z3 of a G1Pre, the Fp scale of every VM line: each non-zero raw edge value (so the z3 slot holds the
    edge limbs themselves) and random ones; 0 excluded (K2 and k_rlc_scale flag that point as infinity)."""
    rnd = random.Random(seed)
    return [real(e) for e in edge_fp() if e] + [rnd.randrange(1, P) for _ in range(n_random)]


def jacobian_steps(seed, n):
    """(T, Q, (xp, yp)) for the single Miller steps: edge and random coordinates, Z = 1 and not."""
    rnd = random.Random(seed)
    edge = [real(e) for e in edge_fp()]
    pick = lambda: edge[rnd.randrange(len(edge))] if rnd.random() < 0.3 else rnd.randrange(P)  # noqa: E731
    out = []
    for i in range(n):
        t = tuple((pick(), pick()) for _ in range(3))
        if i % 5 == 0:
            t = (t[0], t[1], (1, 0))
        out.append((t, ((pick(), pick()), (pick(), pick())), (pick(), pick())))
    return out


def g2_fold_points(seed, n):
    """n Jacobian G2 points (real).  k_rlc_reduce's first shuffle step adds lane l + 16 onto lane l (l < 16), the only step
    that sees the inputs themselves, so the exceptional operands sit at that distance: in lanes 16..31 of a warp, the point
    of lane l - 16 again (same coordinates, or rescaled to another Z: the doubling branch) or its negation (the inverse
    branch); infinities anywhere."""
    rnd = random.Random(seed)
    base = [g2_mul(k) for k in (1, 2, 3, 5, 7)] + [g2_mul(rnd.randrange(1, R)) for _ in range(3)]
    pts = []
    for i in range(n):
        kind = i % 6
        partner = pts[i - 16] if i % 32 >= 16 else None
        if partner is not None and kind == 1:
            pts.append(partner)                                       # duplicate, same coordinates
        elif partner is not None and kind == 2:
            x, y, z = partner
            l = (rnd.randrange(1, P), rnd.randrange(P))
            l2 = f2_sqr(l)
            pts.append((f2_mul(x, l2), f2_mul(y, f2_mul(l2, l)), f2_mul(z, l)))   # duplicate, another Z
        elif partner is not None and kind == 3:
            x, y, z = partner
            pts.append((x, f2_neg(y), z))                             # -P
        elif kind == 4:
            pts.append(((1, 0), (1, 0), (0, 0)))                      # infinity
        else:
            pts.append(jac(base[rnd.randrange(len(base))], (rnd.randrange(1, P), rnd.randrange(P))))
    return pts


def jac(a, z):
    z2 = f2_sqr(z)
    return (f2_mul(a[0], z2), f2_mul(a[1], f2_mul(z2, z)), z)


def jac_sum_affine(pts):
    """Sum of real Jacobian G2 points, affine (None = infinity)."""
    acc = bo.pt_inf(bo.F2)
    for p in pts:
        acc = bo.pt_add(bo.F2, acc, p)
    return bo.pt_to_affine(bo.F2, acc)
