"""GPU: the device's base-field and Fp2 arithmetic, one operation at a time (b200_fp_eval), against Python integers.

The host tests (test_oracle_bls.py) check the g++ build of the same headers; on the device the products are inline PTX,
add / sub are carry-chain asm, the inverse is Kaliski and fp_pow's table lives in shared memory, so the device build is
checked here on its own: the exact representative (canonical < p for Fp, < 2p and the 1.41 p bound for the lazily
reduced FpL), not only the residue."""
import random

import numpy as np
import pytest

from ethereum_consensus_b200 import crypto
from oracle import bls_oracle as bo

pytestmark = pytest.mark.gpu

P = bo.P
RM = 1 << 384                  # Montgomery radix
RINV = pow(RM, -1, P)
N_RANDOM = 50_000
MASK32 = (1 << 32) - 1


def _limbs(values, width=24):
    """Python ints (or pairs of ints for Fp2) -> uint32[n, 24]."""
    out = np.zeros((len(values), width), dtype=np.uint32)
    for i, v in enumerate(values):
        parts = v if isinstance(v, tuple) else (v,)
        for j, x in enumerate(parts):
            out[i, 12 * j: 12 * j + 12] = [(x >> (32 * k)) & MASK32 for k in range(12)]
    return out


def _ints(arr, col=0):
    a = arr[:, 12 * col: 12 * col + 12].astype(object)
    return [sum(int(row[k]) << (32 * k) for k in range(12)) for row in a]


def _edge_fp():
    """Canonical edge values, shared with the host tests, plus [2^380, p) and limb patterns below p."""
    edge = {0, 1, 2, 3, P - 1, P - 2, (P - 1) // 2, (P + 1) // 2, 1 << 380, (1 << 380) + 1, 0xFFFFFFFF, 1 << 32,
            (1 << 352) - 1, (1 << 255) - 19, RM % P, RM * RM % P, pow(RM, -1, P), P - (1 << 380), P - 0xFFFFFFFF}
    edge |= {1 << j for j in range(0, 381, 7)}
    edge |= {(1 << (32 * k)) - 1 for k in range(1, 12)}                       # all-ones low limbs
    edge |= {((1 << 32) - 1) << (32 * k) for k in range(11)}                  # one all-ones limb
    edge |= {P - (1 << (32 * k)) for k in range(12)}                          # p minus one limb unit
    edge |= {(1 << 381) - 1 - P + k for k in range(3)}
    rnd = random.Random(91)
    edge |= {rnd.randrange(1 << 380, P) for _ in range(64)}                   # [2^380, p): the top bit of the 381
    return sorted(e for e in edge if 0 <= e < P)


def _edge_fpl():
    """Representatives in [0, 2p) for the lazily reduced field: the canonical edges, the same plus p, and [p, 2p) edges."""
    e = _edge_fp()
    extra = {P, P + 1, 2 * P - 1, 2 * P - 2, 1 << 381, (1 << 381) + 1, 2 * P - (1 << 200), (1 << 382) - 1 - 2 * P}
    extra |= {(1 << (32 * 11 + k)) - 1 for k in range(30) if (1 << (32 * 11 + k)) - 1 < 2 * P}   # all-ones below 2p
    rnd = random.Random(92)
    extra |= {rnd.randrange(P, 2 * P) for _ in range(64)}
    return sorted({x for x in e} | {x + P for x in e} | {x for x in extra if x < 2 * P})


def _pairs(edge, lo, hi, seed):
    rnd = random.Random(seed)
    pairs = [(a, b) for a in edge for b in edge[:: max(1, len(edge) // 40)]]
    pairs += [(rnd.randrange(lo, hi), rnd.randrange(lo, hi)) for _ in range(N_RANDOM)]
    pairs += [(rnd.randrange(1 << 380, min(hi, P)), rnd.randrange(1 << 380, min(hi, P))) for _ in range(N_RANDOM // 10)]
    if hi > P:
        pairs += [(rnd.randrange(P, hi), rnd.randrange(P, hi)) for _ in range(N_RANDOM // 10)]
    return pairs


def _run(op, a, b=None):
    return crypto.fp_eval(op, _limbs(a), _limbs(b) if b is not None else None)


def _check(name, got, want):
    bad = [i for i, (g, w) in enumerate(zip(got, want)) if g != w]
    print(f"{name:22s} cases {len(want):6d}  mismatches {len(bad)}")
    assert not bad, f"{name}: {len(bad)} mismatches, first at case {bad[0]}: got {got[bad[0]]!r}, want {want[bad[0]]!r}"


@pytest.fixture(scope="module")
def fp_pairs():
    return _pairs(_edge_fp(), 0, P, 1)


@pytest.fixture(scope="module")
def fpl_pairs():
    return _pairs(_edge_fpl(), 0, 2 * P, 2)


def test_reduced_products_sums_and_raw_carries(engine, fp_pairs):
    """fp_mul / fp_sqr (PTX products + final subtraction), fp_add / fp_sub / fp_neg and the raw carry-chain add / subtract
    with their carry and borrow: exact canonical values for operands below p."""
    a = [x for x, _ in fp_pairs]
    b = [y for _, y in fp_pairs]
    assert len(a) >= N_RANDOM
    want = {
        "fp_mul": [x * y * RINV % P for x, y in fp_pairs],
        "fp_sqr": [x * x * RINV % P for x in a],
        "fp_add": [(x + y) % P for x, y in fp_pairs],
        "fp_sub": [(x - y) % P for x, y in fp_pairs],
        "fp_neg": [(-x) % P for x in a],
    }
    for op, w in want.items():
        out = _run(op, a, b)
        _check(op, _ints(out), w)
    out = _run("fp_add_raw", a, b)
    _check("fp_add_raw", list(zip(_ints(out), out[:, 24].tolist())), [((x + y) % RM, (x + y) >> 384) for x, y in fp_pairs])
    out = _run("fp_sub_raw", a, b)
    _check("fp_sub_raw", list(zip(_ints(out), out[:, 24].tolist())), [((x - y) % RM, int(x < y)) for x, y in fp_pairs])
    # the raw operations on full 384-bit patterns (carry out of the top limb)
    rnd = random.Random(3)
    big = [(rnd.getrandbits(384), rnd.getrandbits(384)) for _ in range(4096)] + [(RM - 1, 1), (RM - 1, RM - 1), (0, RM - 1), (RM - 1, 0)]
    out = _run("fp_add_raw", [x for x, _ in big], [y for _, y in big])
    _check("fp_add_raw (2^384)", list(zip(_ints(out), out[:, 24].tolist())), [((x + y) % RM, (x + y) >> 384) for x, y in big])
    out = _run("fp_sub_raw", [x for x, _ in big], [y for _, y in big])
    _check("fp_sub_raw (2^384)", list(zip(_ints(out), out[:, 24].tolist())), [((x - y) % RM, int(x < y)) for x, y in big])


def test_lazily_reduced_field_on_operands_up_to_2p(engine, fpl_pairs):
    """FpL (the per-key kernel's field): products WITHOUT the final subtraction map [0, 2p) x [0, 2p) into [0, 1.41 p) and
    are right modulo p; add / sub / neg stay in [0, 2p)."""
    a = [x for x, _ in fpl_pairs]
    b = [y for _, y in fpl_pairs]
    worst = 0
    for op, w in (("fpl_mul", [x * y * RINV % P for x, y in fpl_pairs]), ("fpl_sqr", [x * x * RINV % P for x in a]),
                  ("fpl_add", [(x + y) % P for x, y in fpl_pairs]), ("fpl_sub", [(x - y) % P for x, y in fpl_pairs]),
                  ("fpl_neg", [(-x) % P for x in a])):
        got = _ints(_run(op, a, b))
        over = [i for i, g in enumerate(got) if g >= 2 * P]
        assert not over, f"{op}: representative >= 2p for case {over[0]}"
        _check(op, [g % P for g in got], w)
        if op in ("fpl_mul", "fpl_sqr"):
            worst = max(worst, max(got))
    assert worst < 1.41 * P + 1        # DESIGN.md section 4: a b / R + p < (4p / R) p + p


def test_inverses_agree_with_each_other_and_with_pow(engine):
    """Kaliski (the device's fp_inv) == Fermat (a^(p-2) with the shared-memory table) == pow(x, -1, p) in Montgomery form."""
    rnd = random.Random(4)
    xs = _edge_fp() + [rnd.randrange(P) for _ in range(N_RANDOM // 5)]
    want = [0 if x == 0 else RM * RM * pow(x, -1, P) % P for x in xs]
    _check("fp_inv_kaliski", _ints(_run("fp_inv_kaliski", xs)), want)
    _check("fp_inv_fermat", _ints(_run("fp_inv_fermat", xs)), want)


def test_square_roots_pow_and_sign(engine):
    """fp_sqrt (value and flag), fpl_pow with the square-root exponent on [0, 2p) inputs, fp_is_lex_largest."""
    rnd = random.Random(5)
    xs = _edge_fp() + [rnd.randrange(P) for _ in range(N_RANDOM // 5)]
    e = (P + 1) // 4
    real = [x * RINV % P for x in xs]
    roots = [pow(v, e, P) for v in real]
    out = _run("fp_sqrt", xs)
    _check("fp_sqrt", list(zip(_ints(out), out[:, 24].tolist())),
           [(r * RM % P, int(r * r % P == v)) for r, v in zip(roots, real)])
    xl = _edge_fpl() + [rnd.randrange(2 * P) for _ in range(N_RANDOM // 10)]
    got = _ints(_run("fpl_pow_sqrt", xl))
    assert max(got) < 2 * P
    _check("fpl_pow_sqrt", [g % P for g in got], [pow(x * RINV % P, e, P) * RM % P for x in xl])
    out = _run("fp_is_lex_largest", xs)
    _check("fp_is_lex_largest", out[:, 24].tolist(), [int(v > (P - 1) // 2) for v in real])


def test_fp2_in_the_signature_unit(engine):
    """Fp2 mul / sqr / inv / sqrt / sgn0 as bls_g2.cu compiles them (inlined products, 255 registers) vs the Python tower."""
    rnd = random.Random(6)
    ed = [0, 1, P - 1, (P - 1) // 2, 1 << 380, RM % P]
    vals = [(x, y) for x in ed for y in ed] + [(rnd.randrange(P), rnd.randrange(P)) for _ in range(4000)]
    vals += [(rnd.randrange(1 << 380, P), rnd.randrange(1 << 380, P)) for _ in range(500)]
    other = [(rnd.randrange(P), rnd.randrange(P)) for _ in vals]
    mont = lambda v: (v[0] * RM % P, v[1] * RM % P)       # noqa: E731
    real = lambda v: (v[0] * RINV % P, v[1] * RINV % P)   # noqa: E731
    a_r, b_r = [real(v) for v in vals], [real(v) for v in other]
    out = _run("fp2_mul", vals, other)
    _check("fp2_mul", list(zip(_ints(out, 0), _ints(out, 1))), [mont(bo.f2_mul(x, y)) for x, y in zip(a_r, b_r)])
    out = _run("fp2_sqr", vals)
    _check("fp2_sqr", list(zip(_ints(out, 0), _ints(out, 1))), [mont(bo.f2_mul(x, x)) for x in a_r])
    nz = [v for v in vals if v != (0, 0)]
    out = _run("fp2_inv", nz)
    _check("fp2_inv", list(zip(_ints(out, 0), _ints(out, 1))), [mont(bo.f2_inv(real(v))) for v in nz])
    out = _run("fp2_sgn0", vals)
    _check("fp2_sgn0", out[:, 24].tolist(), [bo.f2_sgn0(x) for x in a_r])
    # square roots: squares and random elements (about half are squares); either root is fine, its square must match
    sq = [mont(bo.f2_sqr(real(v))) for v in vals[:1500]] + vals[:1500]
    out = _run("fp2_sqrt", sq)
    flags = out[:, 24].tolist()
    want = [int(bo.f2_sqrt(real(v)) is not None) for v in sq]
    _check("fp2_sqrt flag", flags, want)
    roots = [real(r) for r in zip(_ints(out, 0), _ints(out, 1))]
    got_sq = [bo.f2_sqr(r) if f else None for r, f in zip(roots, flags)]
    _check("fp2_sqrt value", got_sq, [real(v) if f else None for v, f in zip(sq, want)])
    assert 1500 < sum(flags) < len(sq)


def test_fp_eval_rejects_unknown_ops(engine):
    a = np.zeros((1, 24), dtype=np.uint32)
    for op in (17, 31, 37, -1):
        assert crypto._lib.lib().b200_fp_eval(op, 1, crypto._lib.ptr(a), crypto._lib.ptr(a), crypto._lib.ptr(np.zeros((1, 25), np.uint32))) == crypto._lib.ERR_BAD_ARG
