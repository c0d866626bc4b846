"""GPU: the device pairing value by value (b200_pairing_eval) against plain integers (tests/pairing_cases.py).

Every op runs in the unit whose production kernel runs it, so the values below are those of that unit's products, inlining
and ptxas level.  Exact representatives are compared, and every coefficient must be below p (fp12_is_one and the VM
final's fp2_eq / fp2_is_zero compare representatives).  Sections:
a. tower operations (Fp6 / Fp12 products, squares, inverses, the sparse line product, Frobenius, cyclotomic squaring,
   pow_z) against the oracle's field, b. Miller steps and loop against the restatement, c. the final exponentiation against
   f^(3 (p^12 - 1) / r) and bilinearity, d. the lane-parallel Miller and final programs at teams of 8 and 16 under every
   vm_cta and every alternative schedule, e. the RLC folds of Fp12 values and G2 points at the batch sizes that end a
   warp or a launch partly filled.

    python -m pytest tests/test_pairing_device_gpu.py -m gpu -s
"""
from __future__ import annotations

import multiprocessing
import os
import random
import subprocess
import sys
import time
from concurrent.futures import ProcessPoolExecutor
from pathlib import Path

import numpy as np
import pytest

from ethereum_consensus_b200 import crypto
from oracle import bls_oracle as bo
from tests import pairing_cases as pc

pytestmark = pytest.mark.gpu
P = bo.P
ROOT = Path(__file__).resolve().parent.parent
_DEVICE_S = [0.0, 0]


def _run(op, a_rows, b_rows=None, a_flags=None, b_flags=None):
    """Raw rows in, (real slot lists, flags) out; every output coefficient must be canonical."""
    a = pc.pack(a_rows, a_flags)
    b = pc.pack(b_rows, b_flags) if b_rows is not None else None
    t = time.perf_counter()
    out = crypto.pairing_eval(op, a, b)
    _DEVICE_S[0] += time.perf_counter() - t
    _DEVICE_S[1] += 1
    raw = pc.unpack(out)
    over = [i for i, r in enumerate(raw) if max(r) >= P]
    assert not over, f"{op}: a coefficient >= p in case {over[0]}"
    return [pc.to_real(r) for r in raw], out[:, 144].tolist()


def _check(name, got, want):
    bad = [i for i, (g, w) in enumerate(zip(got, want)) if g != w]
    print(f"{name:34s} cases {len(want):6d}  mismatches {len(bad)}")
    assert len(got) == len(want)
    assert not bad, f"{name}: {len(bad)} mismatches, first at case {bad[0]}: got {got[bad[0]]!r}, want {want[bad[0]]!r}"


def _o(s):
    return pc.to_oracle(s)


def _g1_row(p, z3=None):
    if z3 is None:
        return pc.to_raw([p[0], p[1]] + [0] * 10)
    return pc.to_raw([p[0] * z3 % P, p[1] * z3 % P, z3] + [0] * 9)


def _g2_row(q):
    return pc.to_raw([q[0][0], q[0][1], q[1][0], q[1][1]] + [0] * 8)


def _pool_map(fn, *items):
    """The references in worker processes; spawned, since this process has initialised CUDA."""
    with ProcessPoolExecutor(mp_context=multiprocessing.get_context("spawn")) as ex:
        return list(ex.map(fn, *items, chunksize=max(1, len(items[0]) // 64)))


def _vm_cta_in_effect():
    """The vm_cta this process started with: B200_VM_CTA when it names a valid shape, else the default."""
    v = os.environ.get("B200_VM_CTA", "")
    return int(v) if v.strip() in ("32", "64", "128") else 32


def _miller_all(pq):
    return _pool_map(pc.miller_loop, [p for p, _ in pq], [q for _, q in pq])


@pytest.fixture(scope="module", autouse=True)
def _device_time():
    yield
    print(f"\ndevice calls {_DEVICE_S[1]}, wall time in b200_pairing_eval {_DEVICE_S[0]:.2f} s (launches, copies, allocation)")


# ---------------------------------------------------------------------------------------------------------- a. tower
def test_a_tower_operations(engine):
    pairs = pc.tower_pairs(31)
    a = [x for x, _ in pairs]
    b = [y for _, y in pairs]
    ar, br = [pc.to_real(x) for x in a], [pc.to_real(y) for y in b]
    ao, bo_ = [_o(x) for x in ar], [_o(y) for y in br]
    assert len(pairs) >= 2000
    got, _ = _run("fp12_mul", a, b)
    _check("a. fp12_mul", got, [pc.from_oracle(bo.f12_mul(x, y)) for x, y in zip(ao, bo_)])
    got, _ = _run("fp12_sqr", a)
    _check("a. fp12_sqr", got, [pc.from_oracle(bo.f12_mul(x, x)) for x in ao])
    # Fp6: the c0 halves; c1 of operand a passes through
    c0 = lambda s: s[:6] + [0] * 6  # noqa: E731
    got, _ = _run("fp6_mul", a, b)
    _check("a. fp6_mul", got, [pc.from_oracle(bo.f12_mul(_o(c0(x)), _o(c0(y))))[:6] + x[6:] for x, y in zip(ar, br)])
    got, _ = _run("fp6_inv", a)
    _check("a. fp6_inv (a d == 1, 0 -> 0)", [pc.from_oracle(bo.f12_mul(_o(c0(x)), _o(c0(d)))) if any(x[:6]) else d[:6]
                                           for x, d in zip(ar, got)],
           [pc.ONE if any(x[:6]) else [0] * 6 for x in ar])
    assert [d[6:] for d in got] == [x[6:] for x in ar]
    # the inverse is unique: a d == 1 exactly, and 0 -> 0
    got, _ = _run("fp12_inv", a)
    _check("a. fp12_inv (a d == 1, 0 -> 0)", [pc.from_oracle(bo.f12_mul(x, _o(d))) if any(x) else d for x, d in zip(ao, got)],
           [pc.ONE if any(x) else [0] * 12 for x in ao])
    # the sparse line product: b's slots 0..5 are A, B, C
    lines = [pc.line_slots(tuple(y[0:2]), tuple(y[2:4]), tuple(y[4:6])) for y in br]
    got, _ = _run("fp12_mul_by_line", a, b)
    _check("a. fp12_mul_by_line", got, [pc.from_oracle(bo.f12_mul(x, _o(l))) for x, l in zip(ao, lines)])
    for k in (1, 2):
        got, _ = _run(f"fp12_frobenius{k}", a)
        _check(f"a. fp12_frobenius<{k}>", got, [pc.from_oracle(pc.frobenius(x, k)) for x in ao])
    # cyclotomic squaring and pow_z: only defined on the cyclotomic subgroup
    cyc = pc.cyclotomic_elements(32, 254)
    cr = [_o(pc.to_real(x)) for x in cyc]
    got, _ = _run("fp12_cyclotomic_sqr", cyc)
    _check("a. fp12_cyclotomic_sqr", got, [pc.from_oracle(bo.f12_mul(x, x)) for x in cr])
    got, _ = _run("fp12_pow_z", cyc)
    _check("a. fp12_pow_z", got, [pc.from_oracle(w) for w in _pool_map(pc.pow_z, cr)])


# ----------------------------------------------------------------------------------------------------- b. Miller
def _miller_cases():
    ps = pc.g1_points(41, 6)
    qs = pc.g2_points(42, 5)
    rnd = random.Random(43)
    pq = [(p, qs[i % len(qs)]) for i, p in enumerate(ps)] + [(ps[rnd.randrange(len(ps))], q) for q in qs]
    return pq


def test_b_miller_steps_and_loop(engine):
    steps = pc.jacobian_steps(44, 2000)
    a = [pc.to_raw([c for f2 in t for c in f2] + [0] * 6) for t, _, _ in steps]
    b = [pc.to_raw([q[0][0], q[0][1], q[1][0], q[1][1], xp, yp] + [0] * 6) for _, q, (xp, yp) in steps]

    def flat(t, A, B, C):
        return [c for f2 in (*t, A, B, C) for c in f2]
    got, _ = _run("miller_double_step", a, b)
    _check("b. miller_double_step", got, [flat(*pc.miller_double_step(t, xp, yp)) for t, _, (xp, yp) in steps])
    got, _ = _run("miller_add_step", a, b)
    _check("b. miller_add_step", got, [flat(*pc.miller_add_step(t, q, xp, yp)) for t, q, (xp, yp) in steps])
    pq = _miller_cases()
    want = _miller_all(pq)
    got, _ = _run("miller_loop", [_g1_row(p) for p, _ in pq], [_g2_row(q) for _, q in pq])
    _check("b. miller_loop", got, want)
    # a point at infinity on either side: exactly one
    n = 4
    got, _ = _run("miller_loop", [_g1_row(p) for p, _ in pq[:n]], [_g2_row(q) for _, q in pq[:n]],
                  a_flags=[1, 0, 1, 0], b_flags=[0, 1, 1, 0])
    _check("b. miller_loop (infinity)", got, [pc.ONE, pc.ONE, pc.ONE, want[3]])


# -------------------------------------------------------------------------------------------- c. final exponentiation
def test_c_final_exponentiation(engine):
    rnd = random.Random(51)
    g, q = bo.G1_GEN, pc.g2_points(52, 1)[1]
    k1, k2 = rnd.randrange(1, bo.R), rnd.randrange(1, bo.R)
    pa, qb = pc.g1_mul(k1), pc.g2_mul(k2)
    pairs = [(g, bo.G2_GEN), (pa, qb), (bo.G1_GEN_NEG, bo.G2_GEN), (g, q), (pc.g1_mul(k1 * k2 % bo.R), bo.G2_GEN),
             (bo.G1_GEN_NEG, q)]
    ml, _ = _run("miller_loop", [_g1_row(p) for p, _ in pairs], [_g2_row(q_) for _, q_ in pairs])
    mlo = [_o(f) for f in ml]
    valid = [bo.f12_mul(mlo[0], mlo[2]), bo.f12_mul(mlo[3], mlo[5])]           # e(P, Q) e(-P, Q): exactly one
    invalid = [bo.f12_mul(mlo[0], mlo[5]), mlo[1], mlo[3], bo.f12_mul(mlo[1], mlo[2]), bo.f12_mul(mlo[1], bo.f12_mul(mlo[4], mlo[4]))]
    randoms = [[rnd.randrange(P) for _ in range(12)] for _ in range(40)]
    general = invalid + randoms + [[0] * 12]
    sub = []                                                  # Fp, Fp2 and Fp6 elements: the easy part sends them to 1
    for _ in range(8):
        sub.append(pc.to_oracle([rnd.randrange(1, P)] + [0] * 11))
        sub.append(pc.to_oracle([rnd.randrange(P), rnd.randrange(1, P)] + [0] * 10))
        sub.append(pc.to_oracle([rnd.randrange(1, P) for _ in range(6)] + [0] * 6))
    t = time.time()
    want_general = _pool_map(pc.final_exp, general)
    print(f"reference final exponentiations: {len(general)} in {time.time() - t:.1f} s")
    inputs = general + valid[:2] + sub
    want = [pc.from_oracle(w) for w in want_general] + [pc.ONE] * (2 + len(sub))
    got, flag = _run("final_exp", [pc.to_raw(pc.from_oracle(x)) for x in inputs])
    assert len(inputs) >= 48
    _check("c. final_exp", got, want)
    _check("c. final_exp verdict == (value == 1)", flag, [int(w == pc.ONE) for w in want])
    assert want[len(general) - 1] == [0] * 12                 # 0 -> 0 on the inverse path
    # bilinearity on device values: e([a] g1, [b] Q) = e(g1, Q)^(ab), e(g1, g2)^r = 1, e(g1, g2) != 1
    e_val, _ = _run("final_exp", [pc.to_raw(ml[0]), pc.to_raw(ml[1]), pc.to_raw(ml[4])])
    e_gg, e_ab, e_abg = (_o(x) for x in e_val)
    assert e_gg != bo.f12_one()
    assert bo.f12_pow(e_gg, bo.R) == bo.f12_one()
    assert e_abg == bo.f12_pow(e_gg, k1 * k2 % bo.R)
    # e([k1] g1, [k2] g2) against e([k1 k2] g1, g2)
    assert e_ab == e_abg
    print("c. bilinearity                      e(aP, bQ) == e(P, Q)^(ab) == e(abP, Q), e^r == 1, e != 1")


# ------------------------------------------------------------------------------------------------- d. VM programs
def _blob(tmp_path, *args):
    out = tmp_path / ("prog_" + "_".join(args) + ".bin")
    subprocess.run([sys.executable, str(ROOT / "tools" / "gen_pairing_vm.py"), *args, "--blob", str(out)], check=True,
                   capture_output=True, cwd=ROOT)
    return np.fromfile(out, dtype=np.uint32)


def _vm_cases():
    """(G1Pre row, G2 row, flags, want): Z = 1, then every edge value of the list in the z3 slot (and in the xz and y
    slots), random z3, and infinities.  The relation VM = direct * lambda^E holds for any lambda = z3 in Fp*, with the
    direct loop run on P = (xz / z3, y / z3)."""
    e = pc.miller_lambda_exponent()
    ps = pc.g1_points(61, 3)
    qs = pc.g2_points(62, 3)
    rnd = random.Random(64)
    base = [(ps[i % len(ps)], qs[i % len(qs)]) for i in range(12)]
    pre = []                                                                  # real (xz, y, z3, Q)
    edge = [pc.real(v) for v in pc.edge_fp()]
    for k, lam in enumerate(pc.lambda_values(63, 6)):
        p, q = base[k % len(base)]
        if k % 3 == 2:                                                         # edge limbs in all three slots
            xz, y = edge[rnd.randrange(len(edge))], edge[rnd.randrange(len(edge))]
        else:
            xz, y = p[0] * lam % P, p[1] * lam % P
        pre.append((xz, y, lam, q))
    direct = _miller_all(base + [((xz * pow(lam, -1, P) % P, y * pow(lam, -1, P) % P), q) for xz, y, lam, q in pre])
    cases = []
    for i, (p, q) in enumerate(base):
        cases.append((_g1_row(p, 1), _g2_row(q), (0, 0), direct[i]))                # Z = 1: the one-thread value
    for (xz, y, lam, q), d in zip(pre, direct[len(base):]):
        cases.append((pc.to_raw([xz, y, lam] + [0] * 9), _g2_row(q), (0, 0), pc.scale(d, pow(lam, e, P))))
    cases.append((_g1_row(base[0][0], 1), _g2_row(base[0][1]), (1, 0), pc.ONE))
    cases.append((_g1_row(base[1][0], 1), _g2_row(base[1][1]), (0, 1), pc.ONE))
    return cases, base


def test_d_vm_programs_every_team_cta_and_schedule(engine, tmp_path):
    cases, base = _vm_cases()
    n_all = len(cases)
    a = [c[0] for c in cases]
    b = [c[1] for c in cases]
    af = [c[2][0] for c in cases]
    bf = [c[2][1] for c in cases]
    want = [c[3] for c in cases]
    # Z = 1 equals op b's device value bit for bit
    one_thread, _ = _run("miller_loop", [r[:2] + [0] * 10 for r in a[:len(base)]], b[:len(base)])
    _check("d. miller_loop (Z = 1 cases)", one_thread, want[:len(base)])
    # final program inputs: (f0, f1) pairs whose product is one, and ones that are not; want = op c on f0 f1
    rnd = random.Random(65)
    fr = [pc.to_raw(w) for w in want]
    f0 = [fr[i] for i in range(len(fr))]
    f1 = [fr[(i + 1) % len(fr)] for i in range(len(fr))]
    negs, _ = _run("miller_loop", [pc.to_raw([bo.G1_GEN_NEG[0], bo.G1_GEN_NEG[1]] + [0] * 10)] * 2 +
                   [pc.to_raw([bo.G1_GEN[0], bo.G1_GEN[1]] + [0] * 10)] * 2,
                   [_g2_row(base[0][1]), _g2_row(base[3][1])] * 2)
    f0 += [pc.to_raw(negs[2]), pc.to_raw(negs[3]), [rnd.randrange(P) for _ in range(12)]]
    f1 += [pc.to_raw(negs[0]), pc.to_raw(negs[1]), [0] * 12]
    prods = [pc.to_raw(pc.from_oracle(bo.f12_mul(_o(pc.to_real(x)), _o(pc.to_real(y))))) for x, y in zip(f0, f1)]
    fin_want, fin_flag = _run("final_exp", prods)
    assert fin_flag[-3:] == [1, 1, 0] and fin_want[-1] == [0] * 12
    defaults = {t: _blob(tmp_path, str(t)) for t in (8, 16)}
    schedules = [("default", None), ("8 mix-light", ("8", "--mix-light", "--heavy-min", "8")),
                 ("16 mix-light", ("16", "--mix-light", "--heavy-min", "4")), ("8 window 64", ("8", "64", "64"))]
    try:
        for sname, args in schedules:
            if args:
                crypto.vm_load_programs(_blob(tmp_path, *args))
            for cta in (32, 64, 128):
                crypto.tune("vm_cta", cta)
                for team in (8, 16):
                    for n in sorted({1, 3, 5, 17, n_all}):
                        got, _ = _run(f"vm_miller{team}", a[:n], b[:n], af[:n], bf[:n])
                        _check(f"d. vm_miller{team} cta {cta} n {n} {sname}", got, want[:n])
                    for n in sorted({1, 3, 5, 17, len(f0)}):
                        sel = list(range(len(f0) - n, len(f0)))          # the tail holds the ones, the zero and the random f
                        got, flag = _run(f"vm_final{team}", [f0[i] for i in sel], [f1[i] for i in sel])
                        _check(f"d. vm_final{team} cta {cta} n {n} {sname}", list(zip(got, flag)),
                               [(fin_want[i], fin_flag[i]) for i in sel])
        # the kernel's own "== 1" test on every coefficient: an empty final program (every word a NOP) leaves f0's six
        # coefficients in its output slots, so the verdict must be 1 for one and 0 for one with any single slot changed
        one = pc.to_raw(pc.ONE)
        probes = [one] + [one[:j] + [pc.mont(2 if j == 0 else 1)] + one[j + 1:] for j in range(12)]
        for team in (8, 16):
            empty = np.array([0xB200564D, team, 1, 12, 0, 1, 2, 3, 4, 5, 1, 12, 0, 1, 2, 3, 4, 5] + [0] * (2 * team),
                             dtype=np.uint32)
            crypto.vm_load_programs(empty)
            for cta in (32, 128):
                crypto.tune("vm_cta", cta)
                got, flag = _run(f"vm_final{team}", probes, [[0] * 12] * len(probes))
                _check(f"d. vm_final{team} cta {cta} verdict per slot", list(zip(got, flag)),
                       [(pc.to_real(x), int(i == 0)) for i, x in enumerate(probes)])
    finally:
        for t in (8, 16):
            crypto.vm_load_programs(defaults[t])
        crypto.tune("vm_cta", _vm_cta_in_effect())


# ----------------------------------------------------------------------------------------------------------- e. folds
def test_e_rlc_folds(engine):
    rnd = random.Random(71)
    pool = [x for x in pc.tower_elements(72, n_random=300) if any(x)]     # non-zero factors: the product is never zero
    pool_real = [pc.to_real(x) for x in pool]
    for n in pc.FOLD_SIZES:
        idx = [rnd.randrange(len(pool)) for _ in range(n)]
        acc = bo.f12_one()
        for i in idx:
            acc = bo.f12_mul(acc, _o(pool_real[i]))
        assert any(acc)
        got, _ = _run("fold_fp12", [pool[i] for i in idx])
        _check(f"e. fold_fp12 n {n}", got[:1], [pc.from_oracle(acc)])
    # one zero factor, in the last launch's partly filled warp: the product is zero
    rows = [pool[rnd.randrange(len(pool))] for _ in range(1025)]
    rows[1024] = [0] * 12
    got, _ = _run("fold_fp12", rows)
    _check("e. fold_fp12 n 1025 (one zero factor)", got[:1], [[0] * 12])
    for n in pc.FOLD_SIZES:
        pts = pc.g2_fold_points(73 + n, n)
        want = pc.jac_sum_affine(pts)
        rows = [pc.to_raw([c for f2 in p for c in f2] + [0] * 6) for p in pts]
        got, flag = _run("fold_g2", rows)
        g = None if flag[0] else ((got[0][0], got[0][1]), (got[0][2], got[0][3]))
        _check(f"e. fold_g2 n {n}", [g], [want])
    # the doubling branch with a checked value: P in lanes 0 and 16 (the first shuffle step's partners), once with the same
    # coordinates and once with another Z, everything else infinity -> [2]P
    inf = ((1, 0), (1, 0), (0, 0))
    a = pc.jac(pc.g2_mul(9), (3, 4))
    for name, b in (("same Z", a), ("other Z", pc.jac(pc.g2_mul(9), (5, 7)))):
        pts = [a] + [inf] * 15 + [b] + [inf] * 15
        got, flag = _run("fold_g2", [pc.to_raw([c for f2 in p for c in f2] + [0] * 6) for p in pts])
        _check(f"e. fold_g2 [2]P ({name})", [None if flag[0] else ((got[0][0], got[0][1]), (got[0][2], got[0][3]))],
               [pc.g2_mul(18)])
    # sums that cancel: P, -P pairs only (and infinities) -> infinity
    pts = [a, (a[0], pc.f2_neg(a[1]), a[2])] * 16 + [inf]
    got, flag = _run("fold_g2", [pc.to_raw([c for f2 in p for c in f2] + [0] * 6) for p in pts])
    _check("e. fold_g2 (cancelling)", flag[:1], [1])


def test_pairing_eval_rejects_unknown_ops(engine):
    a = np.zeros((1, 145), dtype=np.uint32)
    lib = crypto._lib.lib()
    for op in (14, 31, 36, 47, 50, -1):
        assert lib.b200_pairing_eval(op, 1, crypto._lib.ptr(a), crypto._lib.ptr(a), crypto._lib.ptr(a.copy())) == crypto._lib.ERR_BAD_ARG
    assert lib.b200_pairing_eval(2, (1 << 24) + 1, crypto._lib.ptr(a), crypto._lib.ptr(a), crypto._lib.ptr(a.copy())) == crypto._lib.ERR_BAD_ARG
