"""CPU: the references of tests/test_pairing_device_gpu.py are tied to the definition, and the host build of the pairing
headers (hm_pairing_eval) equals them bit for bit.

- The restated Miller loop (tests/pairing_cases.py) is the pairing: its value times the oracle's f_{|z|,Q}(P) vanishes
  under (p^12 - 1)/r (after the final exponentiation the device's closing conjugation is an inversion).
- The lane-parallel programs' value for a G1Pre (X Z, Y, Z^3) is the direct value times (Z^3)^E.
- The Frobenius linear map is x -> x^p, x -> x^(p^2); the tower inverse and the easy part do what the inputs need.
- Every named boundary, fold size and edge value is in the generated lists.
- hm_pairing_eval: the one-thread operations and the VM programs (vm_run_host, Z != 1) on the host."""
from __future__ import annotations

import ctypes as C
import random
from concurrent.futures import ProcessPoolExecutor

import numpy as np
import pytest

from oracle import bls_oracle as bo
from tests import pairing_cases as pc

P = bo.P


def _vanishes(args):
    dev, p, q = args
    x = bo.f12_mul(pc.to_oracle(dev), bo.miller_loop(q, p))
    return bo.f12_pow(x, bo.FINAL_EXP) == bo.f12_one()


def test_restated_miller_loop_is_the_pairing():
    rnd = random.Random(11)
    pairs = [(bo.G1_GEN, bo.G2_GEN), (bo.G1_GEN_NEG, bo.G2_GEN)]
    pairs += [(pc.g1_mul(rnd.randrange(1, bo.R)), pc.g2_mul(rnd.randrange(1, bo.R))) for _ in range(14)]
    jobs = [(pc.miller_loop(p, q), p, q) for p, q in pairs]
    with ProcessPoolExecutor() as ex:
        ok = list(ex.map(_vanishes, jobs))
    assert all(ok), [i for i, v in enumerate(ok) if not v]
    # and the check has teeth: a one-limb change of the restated value does not vanish
    bad = list(jobs[0][0])
    bad[5] = (bad[5] + 1) % P
    assert not _vanishes((bad, pairs[0][0], pairs[0][1]))


def test_g1pre_input_scales_the_loop_by_lambda_to_the_e():
    e = pc.miller_lambda_exponent()
    assert e > 1 << 63
    rnd = random.Random(12)
    q = pc.g2_mul(5)
    for z in [2, P - 1, pc.real(pc.RM % P)] + [rnd.randrange(1, P) for _ in range(3)]:
        p = pc.g1_mul(rnd.randrange(1, bo.R))
        z3 = pow(z, 3, P)
        pre = (p[0] * z3 % P, p[1] * z3 % P)
        assert pc.miller_loop(pre, q, z3) == pc.scale(pc.miller_loop(p, q), pow(z3, e, P))


def test_frobenius_map_inverse_and_easy_part():
    rnd = random.Random(13)
    for _ in range(3):
        a = [rnd.randrange(P) for _ in range(12)]
        assert pc.frobenius(a, 1) == bo.f12_pow(a, P)
        assert pc.frobenius(a, 2) == bo.f12_pow(a, P * P)
        s = pc.from_oracle(a)
        assert pc.to_oracle(pc.from_oracle(a)) == a
        assert bo.f12_mul(a, pc.to_oracle(pc.inverse(s))) == bo.f12_one()
        assert pc.to_oracle(pc.conj(s)) == bo.f12_pow(a, P ** 6)
        g = pc.easy_part(a)
        assert bo.f12_mul(g, pc.to_oracle(pc.conj(pc.from_oracle(g)))) == bo.f12_one()       # g^(p^6 + 1) = 1
    assert pc.inverse([0] * 12) == [0] * 12
    # the slot order: c0.c1 is v = w^2, c1.c0 is w, c1.c1 is v w = w^3
    assert [pc.slot_power(m) for m in range(6)] == [0, 2, 4, 1, 3, 5]
    assert pc.to_oracle(pc.slots([(0, 0), (0, 0), (0, 0), (1, 0), (0, 0), (0, 0)])) == [0, 1] + [0] * 10


def test_generated_lists_hold_every_named_edge():
    edge = pc.edge_fp()
    rm = pc.RM % P
    for v in (0, 1, P - 1, (P - 1) // 2, (P + 1) // 2, rm, (1 << 352) - 1, P - (1 << 32)):
        assert v in edge
    assert any(v >= 1 << 380 for v in edge) and max(edge) < P
    els = pc.tower_elements(1, n_random=10)
    seen = {v for e in els for v in e}
    assert set(edge) <= seen
    for j in range(12):                                   # every edge value reaches every slot
        assert {e[j] for e in els} >= set(edge)
    assert pc.to_raw(pc.ONE) in els and pc.to_raw([P - 1] + [0] * 11) in els
    assert any(sum(1 for v in e if v) == 1 for e in els)
    assert set(pc.FOLD_SIZES) == {1, 2, 31, 32, 33, 63, 64, 65, 1023, 1024, 1025, 4097}
    pts = pc.g2_fold_points(3, 100)
    inf = ((1, 0), (1, 0), (0, 0))
    assert inf in pts
    # the exceptional operands meet in the fold's first shuffle step: lane l + 16 onto lane l
    partners = [(pts[i - 16], pts[i]) for i in range(16, 100) if i % 32 >= 16 and pts[i - 16] != inf]
    same = lambda p, q: bo.pt_eq(bo.F2, p, q)  # noqa: E731
    assert any(p == q for p, q in partners)                                           # duplicate, same coordinates
    assert any(p != q and same(p, q) for p, q in partners)                            # duplicate, another Z
    assert any(same(p, (q[0], pc.f2_neg(q[1]), q[2])) for p, q in partners)          # P, -P
    lams = pc.lambda_values(4, 3)
    assert {pc.mont(v) for v in lams} >= {e for e in edge if e} and 0 not in lams


# --------------------------------------------------------------------------------------------------- host build
@pytest.fixture(scope="module")
def hm(host_math):
    host_math.hm_pairing_eval.argtypes = [C.c_int, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
    host_math.hm_pairing_eval.restype = None
    return host_math


def _hm(hm, op, a_rows, b_rows=None, a_flags=None, b_flags=None):
    a = pc.pack(a_rows, a_flags)
    b = pc.pack(b_rows if b_rows is not None else [[0] * 12] * len(a_rows), b_flags)
    out = np.zeros_like(a)
    hm.hm_pairing_eval(op, len(a_rows), a.ctypes.data, b.ctypes.data, out.ctypes.data)
    return [pc.to_real(r) for r in pc.unpack(out)], out[:, 144].tolist()


def test_host_build_tower_ops(hm):
    """Every one-thread tower op of hm_pairing_eval against the same references as the device test."""
    pairs = pc.tower_pairs(21, n_random=40)[::3]
    a = [x for x, _ in pairs]
    b = [y for _, y in pairs]
    ar, br = [pc.to_real(x) for x in a], [pc.to_real(y) for y in b]
    ao, bo_ = [pc.to_oracle(x) for x in ar], [pc.to_oracle(y) for y in br]
    c0 = lambda s: s[:6] + [0] * 6  # noqa: E731
    want = {
        2: [pc.from_oracle(bo.f12_mul(x, y)) for x, y in zip(ao, bo_)],
        3: [pc.from_oracle(bo.f12_mul(x, x)) for x in ao],
        0: [pc.from_oracle(bo.f12_mul(pc.to_oracle(c0(x)), pc.to_oracle(c0(y))))[:6] + x[6:] for x, y in zip(ar, br)],
        4: [pc.inverse(x) for x in ar],
        1: [pc.inverse(c0(x))[:6] + x[6:] for x in ar],                 # the Fp6 inverse is the Fp12 one of an Fp6 element
        5: [pc.from_oracle(bo.f12_mul(x, pc.to_oracle(pc.line_slots(tuple(y[0:2]), tuple(y[2:4]), tuple(y[4:6])))))
            for x, y in zip(ao, br)],
        6: [pc.from_oracle(pc.frobenius(x, 1)) for x in ao],
        7: [pc.from_oracle(pc.frobenius(x, 2)) for x in ao],
    }
    for op, w in want.items():
        assert _hm(hm, op, a, b)[0] == w, op
    cyc = pc.cyclotomic_elements(26, 6)
    cr = [pc.to_oracle(pc.to_real(x)) for x in cyc]
    assert _hm(hm, 8, cyc)[0] == [pc.from_oracle(bo.f12_mul(x, x)) for x in cr]
    assert _hm(hm, 9, cyc)[0] == [pc.from_oracle(pc.pow_z(x)) for x in cr]


def test_host_build_miller_steps(hm):
    steps = pc.jacobian_steps(27, 200)
    a = [pc.to_raw([c for f2 in t for c in f2] + [0] * 6) for t, _, _ in steps]
    b = [pc.to_raw([q[0][0], q[0][1], q[1][0], q[1][1], xp, yp] + [0] * 6) for _, q, (xp, yp) in steps]

    def flat(t, A, B, C):
        return [c for f2 in (*t, A, B, C) for c in f2]
    assert _hm(hm, 10, a, b)[0] == [flat(*pc.miller_double_step(t, xp, yp)) for t, _, (xp, yp) in steps]
    assert _hm(hm, 11, a, b)[0] == [flat(*pc.miller_add_step(t, q, xp, yp)) for t, q, (xp, yp) in steps]


def test_host_build_miller_and_vm_programs(hm):
    rnd = random.Random(22)
    ps = pc.g1_points(23, 2)
    qs = pc.g2_points(24, 2)
    pq = [(ps[i % len(ps)], qs[i % len(qs)]) for i in range(8)]
    a = [pc.to_raw([p[0], p[1]] + [0] * 10) for p, _ in pq]
    b = [pc.to_raw([q[0][0], q[0][1], q[1][0], q[1][1]] + [0] * 8) for _, q in pq]
    want = [pc.miller_loop(p, q) for p, q in pq]
    got, _ = _hm(hm, 12, a, b)
    assert got == want
    got, _ = _hm(hm, 12, a[:2], b[:2], a_flags=[1, 0], b_flags=[0, 1])
    assert got == [pc.ONE, pc.ONE]
    # the programs with G1Pre inputs of any lambda = z3 (K2 / k_rlc_scale hand over Jacobian sums), edge limbs in the z3
    # slot and, every third case, in the xz and y slots too: restatement on (xz / z3, y / z3) times lambda^E
    e = pc.miller_lambda_exponent()
    edge = [pc.real(v) for v in pc.edge_fp()]
    lams = pc.lambda_values(25, 2)[::4]
    pre, b_pre, want_vm = [], [], []
    for i, lam in enumerate(lams):
        p, q = pq[i % len(pq)]
        xz, y = (edge[(7 * i) % len(edge)], edge[(11 * i) % len(edge)]) if i % 3 == 2 else (p[0] * lam % P, p[1] * lam % P)
        li = pow(lam, -1, P)
        pre.append(pc.to_raw([xz, y, lam] + [0] * 9))
        b_pre.append(b[i % len(pq)])
        want_vm.append(pc.scale(pc.miller_loop((xz * li % P, y * li % P), q), pow(lam, e, P)))
    for op in (32, 33):
        got, _ = _hm(hm, op, pre, b_pre)
        assert got == want_vm, op
        z1 = [pc.to_raw([p[0], p[1], 1] + [0] * 9) for p, _ in pq]
        assert _hm(hm, op, z1, b)[0] == want
    # the final program: its six outputs are final_exp(f0 f1); the pair (P, Q), (-P, Q) multiplies to exactly one
    g = bo.G1_GEN
    f0 = pc.to_raw(pc.miller_loop(g, qs[1]))
    f1 = pc.to_raw(pc.miller_loop(bo.G1_GEN_NEG, qs[1]))
    rnd_f = [rnd.randrange(P) for _ in range(12)]
    prod, _ = _hm(hm, 2, [f0, f0], [f1, rnd_f])
    fe, fe_flag = _hm(hm, 13, [pc.to_raw(x) for x in prod])
    assert fe_flag == [1, 0] and fe[0] == pc.ONE
    assert fe[1] == pc.from_oracle(pc.final_exp(pc.to_oracle(prod[1])))
    for op in (34, 35):
        got, flag = _hm(hm, op, [f0, f0], [f1, rnd_f])
        assert got == fe and flag == [1, 0], op
