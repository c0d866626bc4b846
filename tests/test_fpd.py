"""The per-key kernel's split validation: the FP64 field (fpd.cuh) and the subgroup check on the isomorphic curve.

CPU, exact: FpD products, squares and sums against Python big integers (random operands of either sign up to 2p, the
edge values, and limbs at the balanced maximum so that every column collects its largest sum); the conversions from and
to Fp limbs; the FP64 square-root chain against fpl_sqrt_chain, squares and non-squares; g1_in_subgroup_iso against
g1_in_subgroup_lazy on the small- and mixed-order points of tests/torsion_cases.py; and the split validation's codes
and points against g1_key_validate on those points' encodings, valid keys and random bytes.
GPU: the same keys through both K1 kernels (the 128-thread CTAs run g1_key_validate, the 384-thread CTAs the split)."""
import ctypes
import random
import subprocess
from pathlib import Path

import numpy as np
import pytest

from oracle import bls_oracle as bo

ROOT = Path(__file__).resolve().parent.parent
P = bo.P
RM = 1 << 384
RINV = pow(RM, -1, P)
MASK32 = (1 << 32) - 1
B47 = 1 << 47


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    src = ROOT / "tests" / "host_math" / "fpd_host.cpp"
    lib = tmp_path_factory.mktemp("fpd") / "libfpd_host.so"
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-fvisibility=hidden", "-ffp-contract=off",
                    "-o", str(lib), str(src)], check=True)
    L = ctypes.CDLL(str(lib))
    L.hm_fpd_op.argtypes = [ctypes.c_int, ctypes.c_uint32] + [ctypes.c_void_p] * 3
    L.hm_fpd_roundtrip.argtypes = [ctypes.c_uint32] + [ctypes.c_void_p] * 3
    L.hm_fpd_sqrt_chain.argtypes = [ctypes.c_uint32] + [ctypes.c_void_p] * 3
    L.hm_key_validate_split.argtypes = [ctypes.c_uint32] + [ctypes.c_void_p] * 5
    L.hm_subgroup_iso.argtypes = [ctypes.c_void_p] * 4
    return L


def _limbs(values):
    out = np.zeros((len(values), 12), dtype=np.uint32)
    for i, v in enumerate(values):
        out[i] = [(v >> (32 * k)) & MASK32 for k in range(12)]
    return out


def _ints(arr):
    return [sum(int(row[k]) << (32 * k) for k in range(12)) for row in arr.astype(object)]


def _balanced(v):
    """v (any sign, |v| < 2^382) -> 8 balanced 48-bit digits d with v = sum d_k 2^(48k)"""
    d = []
    for k in range(7):
        r = v % (1 << 48)
        if r >= B47:
            r -= 1 << 48
        d.append(r)
        v = (v - r) >> 48
    return d + [v]


def _to_fpd(digits):
    return np.array([float(dk) * 2.0 ** (48 * k) for k, dk in enumerate(digits)], dtype=np.float64)


def _from_fpd(row):
    """exact integer value of FpD limbs; every limb is an integer multiple of its weight"""
    total = 0
    for k, x in enumerate(row.tolist()):
        m = int(x / 2.0 ** (48 * k))
        assert float(m) * 2.0 ** (48 * k) == x
        total += m << (48 * k)
    return total


def _is_balanced(row):
    return all(abs(x) <= 2.0 ** (48 * k + 47) for k, x in enumerate(row.tolist()[:7]))


def _operands():
    rnd = random.Random(11)
    edge = [0, 1, P - 1, P, P + 1, 2 * P - 1]
    vals = edge + [-v for v in edge] + [rnd.randrange(-2 * P + 1, 2 * P) for _ in range(4000)]
    vals += [rnd.randrange(P, 2 * P) for _ in range(500)] + [-rnd.randrange(P, 2 * P) for _ in range(500)]
    digits = [_balanced(v) for v in vals]
    # every limb at the balanced maximum, of either sign, with the top limb as large as |a| < 2p allows
    top = (2 * P) >> 336
    for s in (1, -1):
        for alt in (False, True):
            d = [s * (B47 if not (alt and k % 2) else -B47) for k in range(7)]
            low = sum(x << (48 * k) for k, x in enumerate(d))
            t = s * (top - 1)
            d.append(t)
            assert abs(low + (t << 336)) < 2 * P
            digits.append(d)
    return digits


def _run(host, op, da, db):
    a = np.stack([_to_fpd(d) for d in da])
    b = np.stack([_to_fpd(d) for d in db])
    out = np.zeros_like(a)
    host.hm_fpd_op(op, len(da), a.ctypes.data, b.ctypes.data, out.ctypes.data)
    return out


def test_fpd_mul_sqr_add_exact(host):
    da = _operands()
    db = da[1:] + da[:1]
    va = [sum(x << (48 * k) for k, x in enumerate(d)) for d in da]
    vb = [sum(x << (48 * k) for k, x in enumerate(d)) for d in db]
    for op, want in ((0, lambda a, b: a * b * RINV), (1, lambda a, b: a * a * RINV), (2, lambda a, b: a + b)):
        out = _run(host, op, da, db)
        for i, (a, b) in enumerate(zip(va, vb)):
            got = _from_fpd(out[i])
            assert _is_balanced(out[i]), (op, i)
            assert (got - want(a, b)) % P == 0, (op, i, hex(a), hex(b))
            if op < 2:
                assert abs(got) < P, (op, i)   # |a|, |b| < 2p -> |ab/R| + p/2 < 0.91 p


def test_fpd_conversions_round_trip(host):
    rnd = random.Random(12)
    xs = [0, 1, P - 1, P, 2 * P - 1] + [rnd.randrange(2 * P) for _ in range(2000)]
    d = np.zeros((len(xs), 8), dtype=np.float64)
    back = np.zeros((len(xs), 12), dtype=np.uint32)
    a = _limbs(xs)
    host.hm_fpd_roundtrip(len(xs), a.ctypes.data, d.ctypes.data, back.ctypes.data)
    for i, x in enumerate(xs):
        assert _from_fpd(d[i]) == x and _is_balanced(d[i])
    assert _ints(back) == xs


def test_fpd_sqrt_chain_matches_fpl_chain(host):
    rnd = random.Random(13)
    xs = [0, 1, 2, P - 1, P, 2 * P - 1, RM % P] + [rnd.randrange(2 * P) for _ in range(300)]
    a = _limbs(xs)
    got_d, got_l = np.zeros_like(a), np.zeros_like(a)
    host.hm_fpd_sqrt_chain(len(xs), a.ctypes.data, got_d.ctypes.data, got_l.ctypes.data)
    d, l = _ints(got_d), _ints(got_l)
    assert max(d) < 2 * P
    assert [v % P for v in d] == [v % P for v in l]
    squares = sum(pow(x * RINV % P, (P - 1) // 2, P) == 1 for x in xs)
    assert 50 < squares < len(xs) - 50     # both squares and non-squares


def _torsion_cases():
    from tests import torsion_cases as tc
    return [c for c in tc.g1_cases()["cases"] if c["pt"] is not None]


def test_subgroup_iso_matches_lazy_on_torsion_points(host):
    cases = _torsion_cases()
    rnd = random.Random(14)
    pts = [tuple(c["pt"]) for c in cases]
    for _ in range(16):   # random points of E(Fp), mostly outside G1
        while True:
            x = rnd.randrange(P)
            y2 = (x ** 3 + 4) % P
            y = pow(y2, (P + 1) // 4, P)
            if y * y % P != y2:
                continue
            pts.append((x, y))
            break
    pts.append(bo.G1_GEN)
    outcomes = set()
    for x, y in pts:
        lazy, iso = ctypes.c_int32(), ctypes.c_int32()
        xl, yl = _limbs([x * RM % P]), _limbs([y * RM % P])
        host.hm_subgroup_iso(xl.ctypes.data, yl.ctypes.data, ctypes.byref(lazy), ctypes.byref(iso))
        assert lazy.value == iso.value, hex(x)
        outcomes.add(iso.value)
    assert outcomes == {0, 1}


def _keys():
    rnd = random.Random(15)
    keys = [bytes(c["enc"]) for c in _torsion_cases()]
    keys += [bo.sk_to_pk(rnd.randrange(1, 1 << 255)) for _ in range(24)]
    keys += [bytes([0xc0]) + bytes(47), bytes([0xc0]) + bytes(46) + b"\x01", bytes(48), bytes([0x80]) + bytes(47)]
    keys += [bytes([0x9a]) + bytes.fromhex("ff" * 47)]       # x >= p
    keys += [bytes([0x80 | rnd.randrange(0x20) | (0x20 * rnd.randrange(2))]) + rnd.randbytes(47) for _ in range(200)]
    return keys


def test_split_validation_matches_key_validate(host):
    keys = _keys()
    n = len(keys)
    buf = np.frombuffer(b"".join(keys), dtype=np.uint8).copy()
    cr, cs = np.zeros(n, np.int32), np.zeros(n, np.int32)
    pr, ps = np.zeros((n, 24), np.uint32), np.zeros((n, 24), np.uint32)
    host.hm_key_validate_split(n, buf.ctypes.data, cr.ctypes.data, pr.ctypes.data, cs.ctypes.data, ps.ctypes.data)
    assert cr.tolist() == cs.tolist()
    assert pr.tolist() == ps.tolist()
    assert set(cr.tolist()) >= {0, 1, 2, 3, 6}
    assert cr.tolist() == [bo.key_validate(k)[0] for k in keys]


@pytest.mark.gpu
def test_device_split_kernel_matches_host(engine, host):
    """One-key groups through eth_aggregate_public_keys_batch: a call of fewer keys than three waves of 384-thread CTAs
    runs g1_key_validate in 128-thread CTAs; a larger one runs the role-split kernel.  Both give the same codes and
    keys, key for key, and accept exactly the keys the host accepts."""
    from ethereum_consensus_b200 import crypto
    keys = _keys()
    n = len(keys)
    buf = np.frombuffer(b"".join(keys), dtype=np.uint8).copy()
    cr, cs = np.zeros(n, np.int32), np.zeros(n, np.int32)
    pr, ps = np.zeros((n, 24), np.uint32), np.zeros((n, 24), np.uint32)
    host.hm_key_validate_split(n, buf.ctypes.data, cr.ctypes.data, pr.ctypes.data, cs.ctypes.data, ps.ctypes.data)
    reps = (3 * 148 * 384) // n + 2
    big = np.tile(buf, reps)
    out_s, codes_s = crypto.eth_aggregate_public_keys_batch(buf, np.arange(n + 1, dtype=np.uint32))
    out_b, codes_b = crypto.eth_aggregate_public_keys_batch(big, np.arange(reps * n + 1, dtype=np.uint32))
    assert ((codes_s == 0) == (cr == 0)).all()
    assert codes_b.tolist() == np.tile(codes_s, reps).tolist()
    assert np.array_equal(out_b, np.tile(out_s, (reps, 1)))
    ok = cr == 0
    assert np.array_equal(out_s[ok], buf.reshape(n, 48)[ok])
