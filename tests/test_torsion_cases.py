"""CPU: the small-order and mixed-order curve points of tests/torsion_cases.py are what they claim to be, every exceptional
branch the subgroup-check and cofactor-clearing ladders can take is reached, and the C oracle and the host build of the
product headers agree with the definition ([r]P == infinity) on every case.  tests/test_torsion_gpu.py runs the same
cases through the CUDA kernels."""
from __future__ import annotations

import ctypes as C
import math
import random
from itertools import combinations

import pytest

from oracle import bls_oracle as bo
from tests import torsion_cases as tc

F1, F2, P, R = bo.F1, bo.F2, bo.P, bo.R


@pytest.fixture(scope="module")
def g1():
    return tc.g1_cases()


@pytest.fixture(scope="module")
def g2():
    return tc.g2_cases()


def _is_prime(n, rounds=24):
    if n < 1 << 32:
        return n > 1 and all(n % k for k in range(2, math.isqrt(n) + 1))
    d, s = n - 1, 0
    while d % 2 == 0:
        d, s = d // 2, s + 1
    rnd = random.Random(5)
    for _ in range(rounds):
        x = pow(rnd.randrange(2, n - 1), d, n)
        if x in (1, n - 1):
            continue
        for _ in range(s - 1):
            x = x * x % n
            if x == n - 1:
                break
        else:
            return False
    return True


def _primes(d):
    return [l for l in list(tc.H1_PRIMES) + list(tc.H2_SMALL) if d % l == 0]


def _divisors(primes):
    return [math.prod(c) for k in range(1, len(primes) + 1) for c in combinations(primes, k)]


def test_cofactors_group_orders_and_endomorphisms():
    z = tc.Z
    assert tc.H1 == 3 * 11 ** 2 * 10177 ** 2 * 859267 ** 2 * 52437899 ** 2
    assert tc.N1 == P + 1 - (z + 1)                                   # #E(Fp) = p + 1 - t, t = z + 1
    assert tc.H2 == 13 ** 2 * 23 ** 2 * 2713 * 11953 * 262069 * tc.H2_Q
    assert len(str(tc.H2_Q)) == 135 and _is_prime(tc.H2_Q)
    assert all(_is_prime(l) for l in list(tc.H1_PRIMES) + list(tc.H2_SMALL))
    rnd = random.Random(3)
    for _ in range(2):
        assert tc.mul(F1, tc.g1_random(rnd), tc.N1) is None
        assert tc.mul(F2, tc.g2_random(rnd), tc.N2) is None
    # the endomorphisms as the product uses them: phi(P) = -[z^2]P on G1, psi(Q) = [z]Q on G2
    assert tc.phi(bo.G1_GEN) == tc.neg(F1, tc.mul(F1, bo.G1_GEN, tc.Z_ABS ** 2))
    assert tc.psi(bo.G2_GEN) == tc.mul(F2, bo.G2_GEN, z)
    # -z^2 = -1 mod every G1 torsion prime: no eigenvalue of phi there equals the test scalar
    assert all((-z * z) % l == l - 1 for l in tc.H1_PRIMES)


def test_torsion_structure(g1, g2):
    """The l-primary part has exponent l for every small l (so Z/l x Z/l where l^2 divides the cofactor)."""
    assert g1["structure"] == {l: l for l in tc.H1_PRIMES}
    assert g2["structure"] == {l: l for l in tc.H2_SMALL}


def test_claimed_orders_are_exact(g1, g2):
    rnd = random.Random(4)
    for F, D in ((F1, g1), (F2, g2)):
        for c in D["cases"]:
            d = c["order"]
            if d < R:                                                    # pure torsion: [d]T = inf, [d / l]T != inf
                assert tc.mul(F, c["pt"], d) is None, c["family"]
                for l in _primes(d):
                    assert tc.mul(F, c["pt"], d // l) is not None, (c["family"], d, l)
        mixed = [c for c in D["cases"] if c["order"] > R]
        for c in rnd.sample(mixed, 40):                                 # Q + T: order r * ord(T)
            o = c["t_order"]
            assert c["order"] == R * o and tc.mul(F, c["pt"], R * o) is None
            assert tc.mul(F, c["pt"], R) is not None
            for l in _primes(o):
                assert tc.mul(F, c["pt"], R * o // l) is not None


def test_every_small_prime_appears(g1, g2):
    orders1 = {c["order"] for c in g1["cases"] if c["order"] < R}
    orders2 = {c["order"] for c in g2["cases"] if c["order"] < R}
    assert {l for d in orders1 for l in _primes(d)} == set(tc.H1_PRIMES)
    assert {l for d in orders2 for l in _primes(d)} == set(tc.H2_SMALL)
    assert any(len(_primes(d)) > 1 for d in orders1) and any(len(_primes(d)) > 1 for d in orders2)
    for D, n, fams in ((g1, 1500, {"torsion", "eigen", "valid", "Q+T", "-Q+T"}), (g2, 600, {"torsion", "eigen", "valid", "sigma+T"})):
        if tc.SCALE >= 1:
            assert len(D["cases"]) >= n
        assert {c["family"] for c in D["cases"]} == fams
        assert {c["code"] for c in D["cases"]} == {bo.SUCCESS, bo.POINT_NOT_IN_GROUP}


def test_eigenspace_points(g1, g2):
    """phi has eigenvalues only mod 10177 and 859267 (the non-trivial cube roots of 1); psi has them mod 13 (two), 2713,
    11953 and 262069 (one each: cyclic), none mod 23.  Every eigen case satisfies phi(T) = [lam]T or psi(T) = [lam]T."""
    assert {l for l, v in g1["eigen"].items() if v} == {10177, 859267}
    for l, v in g1["eigen"].items():
        assert sorted(lam for lam, _ in v) == tc.cube_roots_of_unity(l)
    assert {l: len(v) for l, v in g2["eigen"].items()} == {13: 2, 23: 0, 2713: 1, 11953: 1, 262069: 1}
    # the observed eigenvalues are roots of psi^2 - t psi + p mod l; where the l-torsion over Fp2 is cyclic psi acts by
    # one of the two roots only (the other one's eigenvectors are not defined over Fp2)
    for l, v in g2["eigen"].items():
        roots = {x for x in range(l) if (x * x - (tc.Z + 1) * x + P) % l == 0}
        assert set(v) <= roots and (set(v) == roots if tc.H2_SMALL[l] == 2 else len(roots) == 2)
    for F, f, D in ((F1, tc.phi, g1), (F2, tc.psi, g2)):
        eig = [c for c in D["cases"] if c["family"] == "eigen"]
        assert eig
        for c in eig:
            assert f(c["pt"]) == tc.mul(F, c["pt"], c["lam"])
    for l in (10177, 859267):                                           # a generic torsion point is not an eigenvector
        t = g1["base"][l][0]
        assert all(tc.phi(t) != tc.mul(F1, t, lam) for lam in tc.cube_roots_of_unity(l))


def _ladder_on_points(F, base, k=tc.Z_ABS, mixed=True):
    """jac_mul_u64 / jac_mul_u64_jac run on affine points, recording which exceptional branch each add takes."""
    out, acc, started = set(), None, False
    pre = "madd" if mixed else "add"
    for bit in range(63, -1, -1):
        if started:
            acc = tc.add(F, acc, acc)
        if (k >> bit) & 1:
            if base is None:
                out.add("add_inf")
            elif acc is None:
                if started:
                    out.add(pre + "_inf")
            elif acc == base:
                out.add(pre + "_dbl")
            elif acc == tc.neg(F, base):
                out.add(pre + "_inv")
            acc = tc.add(F, acc, base)
            started = True
    return out, acc


def test_ladder_replay_matches_the_points(g1, g2):
    """The branches replayed on integers mod the order are the ones the ladder takes on the actual points."""
    for c in [c for c in g1["cases"] if c["order"] < R][::3]:
        b1, t = _ladder_on_points(F1, c["pt"])
        b2, _ = _ladder_on_points(F1, t, mixed=False)
        assert b1 | b2 == c["branches"], c["order"]
    for c in [c for c in g2["cases"] if c["order"] < R][::3]:
        assert _ladder_on_points(F2, c["pt"])[0] == c["branches"], c["order"]
        b1, t1 = _ladder_on_points(F2, c["pt"], mixed=False)
        t2 = tc.add(F2, tc.neg(F2, t1), tc.psi(c["pt"]))
        b2, _ = _ladder_on_points(F2, t2, mixed=False)
        assert b1 | b2 == c["cc_branches"], c["order"]


def test_every_reachable_branch_is_reached(g1, g2):
    """Every exceptional branch that some small order can drive each ladder into is reached by a case.  On G1 the
    subgroup check reaches all six (order 3: inverse and infinity; order 11: doubling, at bit 60 where 12T = T).  On G2
    no order dividing h2 / q gives the doubling branch: order 13 reaches the inverse at bit 60 (12T = -T), then adds
    onto infinity, in g2_in_subgroup and in g2_clear_cofactor's first ladder."""
    reach1 = set().union(*(tc.g1_check_branches(d) for d in _divisors(list(tc.H1_PRIMES))))
    reach2 = set().union(*(tc.g2_check_branches(d) for d in _divisors(list(tc.H2_SMALL))))
    reach_cc = set().union(*(tc.ladder_branches(d, False) for d in [1] + _divisors(list(tc.H2_SMALL))))
    assert reach1 == set(tc.BRANCHES_MIXED) | set(tc.BRANCHES_GENERAL)
    assert reach2 == {"madd_inv", "madd_inf"}
    got1 = set().union(*(c["branches"] for c in g1["cases"]))
    got2 = set().union(*(c["branches"] for c in g2["cases"]))
    got_cc = set().union(*(c.get("cc_branches", set()) for c in g2["cases"]))
    assert got1 == reach1 and got2 == reach2
    assert got_cc == reach_cc & {"add_inv", "add_inf"} and got_cc == {"add_inv", "add_inf"}
    assert tc.g1_check_branches(3) >= {"madd_inv"} and "madd_dbl" in tc.g1_check_branches(11)
    assert tc.g2_check_branches(13) == {"madd_inv", "madd_inf"}
    for c in g1["cases"] + g2["cases"]:                                  # only pure torsion reaches any of them
        assert bool(c["branches"]) <= (c["order"] < R)


def test_c_oracle_and_host_build_agree_with_the_definition(g1, g2, oracle_bls_c, host_math):
    O, H = oracle_bls_c, host_math
    xy, rec, inf, grp = C.create_string_buffer(192), C.create_string_buffer(96), C.c_int(), C.c_int()
    bad = []
    for c in g1["cases"]:
        e = c["enc"]
        got = (O.orc_key_validate(e), O.orc_g1_group_checks_agree(e), H.hm_g1_key_validate(e, xy, rec))
        if got != (c["code"], 1, c["code"]):
            bad.append(("g1", c["family"], c["order"], got, c["code"]))
    for c in g2["cases"]:
        e = c["enc"]
        rc = H.hm_g2_uncompress(e, xy, C.byref(inf), C.byref(grp), rec)
        got = (O.orc_aggregate(e, 1, rec), O.orc_g2_group_checks_agree(e), rc, grp.value)
        if got != (c["code"], 1, 0, int(c["code"] == 0)):
            bad.append(("g2", c["family"], c["order"], got, c["code"]))
    assert not bad, bad[:5]


def _f2_bytes(v):
    return v[0].to_bytes(48, "big") + v[1].to_bytes(48, "big")


def test_host_sswu_iso_matches_the_oracle(host_math):
    """hm_sswu_iso (sswu_map then iso3_map, h2c.cuh) = iso3(sswu(u)) at u = 0 (tv1 == 0), +-1, the sgn0 edges and random
    u.  -1/Z is not a square in Fp2, so u = 0 is the only input with tv1 == 0."""
    zc = bo.SSWU_Z
    assert bo.f2_sqrt(bo.f2_neg(bo.f2_inv(zc))) is None
    us = tc.sswu_inputs(200)
    out, inf = C.create_string_buffer(192), C.c_int()
    tv1_zero = 0
    for u in us:
        t2 = bo.f2_sqr(u)
        tv1_zero += bo.f2_is_zero(bo.f2_add(bo.f2_mul(bo.f2_sqr(zc), bo.f2_sqr(t2)), bo.f2_mul(zc, t2)))
        want = bo.iso3(bo.sswu(u))
        host_math.hm_sswu_iso(_f2_bytes(u), out, C.byref(inf))
        r = out.raw
        got = None if inf.value else ((int.from_bytes(r[:48], "big"), int.from_bytes(r[48:96], "big")),
                                      (int.from_bytes(r[96:144], "big"), int.from_bytes(r[144:], "big")))
        assert got == want, u
    assert tv1_zero == 1 and us[0] == (0, 0)
