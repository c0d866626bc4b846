"""GPU: the role-split per-key kernel's arithmetic and its shared-memory hand-off, against Python integers, the host
build of the same headers and the C oracle.

FpD (fpd.cuh) value by value through b200_fp_eval, built in bls_g1.cu at the per-key kernel's ptxas level and with nvcc's
default FMA contraction: products, squares and sums exact against big integers and limb for limb equal to the g++ build
(tests/host_math/fpd_host.cpp); the conversions; the FP64 square-root chain against fpl_sqrt_chain and the exponentiation;
g1_y_from_x_fpd against Python for both sign flags.  g1_in_subgroup_iso (x alone) through b200_curve_eval against
g1_in_subgroup_lazy on the full point and the oracle's membership.

k_g1_validate_split's slots and tails: a pool of keys of every class placed at the in-CTA positions where the FP64 warps'
two keys per thread and the integer warps' edges meet (j = 0, 1, 127, 128, 129, 255), loaded into the registry at sizes
whose last CTA holds 1, 128, 129, 255 and 256 keys; codes against the oracle, and the points through one-key and two-key
aggregations against the oracle's eth_aggregate_public_keys (a two-key sum depends on all of y, not just its sign).
Calls below three waves run the 128-thread kernel unless B200_G1_SMALL_N=0, read once per process: the small sizes run in
a child process with that setting.
"""
from __future__ import annotations

import os
import pickle
import random
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from oracle import bls_oracle as bo  # noqa: E402
from tests import torsion_cases as tc  # noqa: E402
from tests.test_bls_device_soak_gpu import _oracle_bytes  # noqa: E402
from tests.test_fpd import B47, P, RINV, RM, _balanced, _ints, _limbs, _operands, build_host  # noqa: E402

pytestmark = pytest.mark.gpu
F1 = bo.F1
W = 2.0 ** (48 * np.arange(8))               # limb weights
BOUND = 2.0 ** (48 * np.arange(7) + 47)      # balanced limbs 0..6: |l_k| <= 2^(48k+47)
TOP = (2 * P) >> 336                         # |a| < 2p: |top limb| < TOP 2^336 once the low limbs are balanced
SMALL_N = 3 * 148 * 384                      # bls_g1.cu g_g1_small_n
SPECIAL = (0, 1, 127, 128, 129, 255)         # FP64 thread t: keys t and t + 128; integer warps' edges
TAILS = (1, 128, 129, 255, 256)              # keys in the last 256-key CTA of SMALL_N + r keys (SMALL_N = 666 * 256)
CHILD_NS = (1, 2, 127, 128, 129, 255, 256, 257, 383, 384, 385, 511, 512, 513)
_CACHE = {}


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    return build_host(tmp_path_factory.mktemp("fpd_dev"))


def _g1_cases():
    """tests/torsion_cases.py's G1 points (valid keys, small-order and mixed-order points), generated once."""
    if "g1" not in _CACHE:
        _CACHE["g1"] = tc.g1_cases()["cases"]
    return _CACHE["g1"]


# ---------------------------------------------------------------------------------------------------------- FpD records
def _fpd(digits):
    """[[d_0 .. d_7]] balanced digits -> float64[n, 8] limbs d_k 2^(48k) (exact: |d_k| < 2^53, power-of-two scaling)."""
    return np.array(digits, dtype=np.float64) * W


def _values(D):
    """float64[n, 8] -> exact integer values; asserts every limb is an integer multiple of its weight."""
    q = D / W
    assert np.all(q == np.round(q)) and np.all(np.abs(q) < 2.0 ** 53)
    return [sum(int(x) << (48 * k) for k, x in enumerate(row)) for row in q.astype(np.int64).tolist()]


def _balanced_rows(D):
    return np.all(np.abs(D[:, :7]) <= BOUND, axis=1)


def _rec(D):
    """FpD limbs -> b200_fp_eval operand slots (words 0..15)."""
    a = np.zeros((len(D), 24), dtype=np.uint32)
    a.view(np.float64)[:, :8] = D
    return a


def _dev(op, A, B=None):
    from ethereum_consensus_b200 import crypto
    out = crypto.fp_eval(op, _rec(A), _rec(B if B is not None else np.zeros_like(A)))
    return np.ascontiguousarray(out[:, :24]).view(np.float64)[:, :8].copy()


def _host(host, op, A, B):
    A, B = np.ascontiguousarray(A), np.ascontiguousarray(B)
    out = np.zeros_like(A)
    host.hm_fpd_op(op, len(A), A.ctypes.data, B.ctypes.data, out.ctypes.data)
    return out


def _rand_digits(rnd):
    """A random value inside the contract with balanced low limbs and a top limb of |.| <= TOP - 2."""
    return [rnd.randrange(-B47, B47 + 1) for _ in range(7)] + [rnd.randrange(-(TOP - 2), TOP - 1)]


def _edge_operands():
    """The contract's corners as FpD limbs: single limbs at the balanced maximum, every limb at it (same and alternating
    signs), +-(2p - 1), +-p, and zero with limbs of +0.0 and of -0.0."""
    digits = []
    for k in range(8):
        for s in (1, -1):
            d = [0] * 8
            d[k] = s * (B47 if k < 7 else TOP - 1)
            digits.append(d)
    for s in (1, -1):
        for alt in (False, True):
            d = [s * (B47 if not (alt and k % 2) else -B47) for k in range(7)]
            low = sum(x << (48 * k) for k, x in enumerate(d))
            d.append(s * (TOP - 1))
            assert abs(low + (d[7] << 336)) < 2 * P
            digits.append(d)
    for v in (2 * P - 1, P, -P, -(2 * P - 1)):
        digits.append(_balanced(v))
    D = _fpd(digits)
    return np.concatenate([D, np.zeros((1, 8)), np.full((1, 8), -0.0)])


def _tie_pairs(rnd):
    """Operand pairs whose limb sum k lands exactly on +-2^(48k+47) before fpd_normalize, where the carry rounds to even;
    directly, and after a carry of +-2^(48k) out of limb k - 1."""
    A, B = [], []
    for k in range(7):
        for s in (1, -1):
            for carry_in in (0, 1, -1):
                for _ in range(3):
                    a, b = _rand_digits(rnd), _rand_digits(rnd)
                    a[k] = s * rnd.randrange(0, B47 + 1)
                    b[k] = s * B47 - a[k] - carry_in
                    if abs(b[k]) > B47 or (carry_in and k == 0):
                        continue
                    if carry_in:      # limb k - 1 sums to +-2^(48(k-1)+48): carries exactly carry_in into limb k
                        a[k - 1] = carry_in * B47
                        b[k - 1] = carry_in * B47
                    A.append(a)
                    B.append(b)
    return _fpd(A), _fpd(B)


def test_fpd_mul_sqr_add_exact_and_equal_to_host(engine, host):
    """Products, squares and sums on the device: exact against Python integers, balanced, and limb for limb equal to the
    -ffp-contract=off host build, compared with float ==, then bit for bit.  The sign of a zero limb is the only thing
    float == would let differ; on an H100 (sm_90a, nvcc's default --fmad=true, ptxas -O2) no limb differed even there, so
    the bitwise comparison is asserted too."""
    rnd = random.Random(51)
    base = _fpd(_operands())
    edge = _edge_operands()
    rand = _fpd([_balanced(rnd.randrange(-2 * P + 1, 2 * P)) for _ in range(50_000)])
    ops = np.concatenate([base, edge, rand])
    # every operand against a shifted partner, and every corner against every corner (each column at its largest sum)
    A = np.concatenate([ops, np.repeat(edge, len(edge), axis=0)])
    B = np.concatenate([np.roll(ops, 1, axis=0), np.tile(edge, (len(edge), 1))])
    ta, tb = _tie_pairs(rnd)
    va, vb = _values(A), _values(B)
    assert all(abs(v) < 2 * P for v in va + vb)
    assert _balanced_rows(A).all() and _balanced_rows(B).all()
    bit_diffs = {}
    for op, name in ((0, "fpd_mul"), (1, "fpd_sqr"), (2, "fpd_add")):
        a, b = (np.concatenate([A, ta]), np.concatenate([B, tb])) if op == 2 else (A, B)
        xa, xb = (va + _values(ta), vb + _values(tb)) if op == 2 else (va, vb)
        got = _dev(name, a, b)
        assert _balanced_rows(got).all(), name
        vals = _values(got)
        if op == 0:
            bad = [i for i, (g, x, y) in enumerate(zip(vals, xa, xb)) if (g - x * y * RINV) % P or abs(g) >= P]
        elif op == 1:
            bad = [i for i, (g, x) in enumerate(zip(vals, xa)) if (g - x * x * RINV) % P or abs(g) >= P]
        else:
            bad = [i for i, (g, x, y) in enumerate(zip(vals, xa, xb)) if g != x + y]
        assert not bad, f"{name}: {len(bad)} of {len(vals)} wrong, first a = {hex(xa[bad[0]])}, b = {hex(xb[bad[0]])}"
        want = _host(host, op, a, b)
        neq = np.nonzero(~np.all(got == want, axis=1))[0]
        assert not len(neq), f"{name}: {len(neq)} results differ from the host build, first at {neq[0]}"
        bit_diffs[name] = int(np.count_nonzero(got.view(np.uint64) != want.view(np.uint64)))
    print("FpD limbs equal to the host build but not bit for bit (zero signs):", bit_diffs)
    assert not any(bit_diffs.values()), bit_diffs


def test_fpd_conversions(engine, host):
    """fpd_from_fp over [0, 2p) (equal to the host's limbs) and back through fpd_to_fpl; fpd_to_fpl on balanced values down
    to -(2p - 1), which it returns as v + 2p."""
    rnd = random.Random(52)
    xs = [0, 1, P - 1, P, P + 1, 2 * P - 2, 2 * P - 1, RM % P] + [rnd.randrange(2 * P) for _ in range(4000)]
    a = np.zeros((len(xs), 24), dtype=np.uint32)
    a[:, :12] = _limbs(xs)
    from ethereum_consensus_b200 import crypto
    d = np.ascontiguousarray(crypto.fp_eval("fpd_from_fp", a)[:, :24]).view(np.float64)[:, :8].copy()
    assert _values(d) == xs
    assert _balanced_rows(d).all()
    hd, hb = np.zeros((len(xs), 8)), np.zeros((len(xs), 12), dtype=np.uint32)
    hl = _limbs(xs)
    host.hm_fpd_roundtrip(len(xs), hl.ctypes.data, hd.ctypes.data, hb.ctypes.data)
    assert np.array_equal(d.view(np.uint64), hd.view(np.uint64))
    assert _ints(crypto.fp_eval("fpd_to_fpl", _rec(d))[:, :12]) == xs
    vs = [-(2 * P - 1), -2 * P + 2, -P - 1, -P, -P + 1, -1, 0] + [-rnd.randrange(1, 2 * P) for _ in range(2000)]
    vs += [rnd.randrange(-2 * P + 1, 2 * P) for _ in range(2000)]
    D = np.concatenate([_fpd([_balanced(v) for v in vs]), np.full((1, 8), -0.0)])
    got = _ints(crypto.fp_eval("fpd_to_fpl", _rec(D))[:, :12])
    assert got == [v % (2 * P) for v in vs] + [0]


def test_fpd_sqrt_chain(engine, host):
    """fpd_sqrt_chain (from Fp, back to [0, 2p)) against fpl_sqrt_chain (op 18), x^((p+1)/4) and the host build."""
    from ethereum_consensus_b200 import crypto
    rnd = random.Random(53)
    xs = [0, 1, 2, P - 1, P, P + 1, 2 * P - 1, RM % P] + [rnd.randrange(2 * P) for _ in range(2400)]
    a = np.zeros((len(xs), 24), dtype=np.uint32)
    a[:, :12] = _limbs(xs)
    d = _ints(crypto.fp_eval("fpd_sqrt_chain", a)[:, :12])
    lz = _ints(crypto.fp_eval("fpl_sqrt_chain", a)[:, :12])
    assert max(d) < 2 * P
    bad = [i for i, (g, l) in enumerate(zip(d, lz)) if (g - l) % P]
    assert not bad, f"fpd_sqrt_chain != fpl_sqrt_chain for {len(bad)} inputs, first x = {hex(xs[bad[0]])}"
    bad = [i for i, (g, x) in enumerate(zip(d, xs)) if g * RINV % P != pow(x * RINV % P, (P + 1) // 4, P)]
    assert not bad, f"fpd_sqrt_chain != x^((p+1)/4) for {len(bad)} inputs, first x = {hex(xs[bad[0]])}"
    hd, hl = np.zeros((len(xs), 12), dtype=np.uint32), np.zeros((len(xs), 12), dtype=np.uint32)
    hx = _limbs(xs)
    host.hm_fpd_sqrt_chain(len(xs), hx.ctypes.data, hd.ctypes.data, hl.ctypes.data)
    assert _ints(hd) == d
    squares = sum(pow(x * RINV % P, (P - 1) // 2, P) == 1 for x in xs)
    assert 500 < squares < len(xs) - 500     # both squares and non-squares


def _y_want(x, largest):
    y2 = (x * x * x + 4) % P
    y = pow(y2, (P + 1) // 4, P)
    if y * y % P != y2:
        return None
    return (P - y) % P if (y > (P - 1) // 2) != largest else y


def test_fpd_y_from_x(engine):
    """g1_y_from_x_fpd for both sign flags: x of valid keys, x = 0 (y = +-2), x = p - 1 and random x, half of which lie
    off the curve; y canonical Montgomery with the requested sign, the flag word the on-curve verdict."""
    from ethereum_consensus_b200 import crypto
    rnd = random.Random(54)
    valid = [c["pt"][0] for c in _g1_cases() if c["family"] == "valid"][::4]
    xs = valid + [0, 1, P - 1, P - 2] + [rnd.randrange(P) for _ in range(600)]
    rows = [(x, f) for x in xs for f in (0, 1)]
    a = np.zeros((len(rows), 24), dtype=np.uint32)
    b = np.zeros_like(a)
    a[:, :12] = _limbs([x * RM % P for x, _ in rows])
    b[:, 0] = [f for _, f in rows]
    out = crypto.fp_eval("fpd_y_from_x", a, b)
    flags, ys = out[:, 24].tolist(), _ints(out[:, :12])
    want = [_y_want(x, bool(f)) for x, f in rows]
    bad = [i for i, (w, fl) in enumerate(zip(want, flags)) if fl != (w is not None)]
    assert not bad, f"on-curve verdict wrong for {len(bad)}, first x = {hex(rows[bad[0]][0])}"
    bad = [i for i, (w, y) in enumerate(zip(want, ys)) if w is not None and y != w * RM % P]
    assert not bad, f"y wrong for {len(bad)}, first x = {hex(rows[bad[0]][0])}, flag {rows[bad[0]][1]}"
    assert _y_want(0, False) == 2 and _y_want(0, True) == P - 2
    on = sum(w is not None for w in want[2 * len(valid) + 8:])
    assert 400 < on < 800          # about half of the random x are off the curve


def test_subgroup_iso_matches_lazy_and_oracle(engine):
    """g1_in_subgroup_iso from x alone against g1_in_subgroup_lazy on the full point (op 2) and [r]P == infinity."""
    from ethereum_consensus_b200 import crypto
    from tests.test_torsion_gpu import _aff_rec, _records
    rnd = random.Random(55)
    cases = _g1_cases()
    pts = [c["pt"] for c in cases]
    want = [int(c["code"] == 0) for c in cases]
    extra = [tc.g1_random(rnd) for _ in range(48)] + [bo.G1_GEN, tc.neg(F1, bo.G1_GEN)]
    extra += [tc.mul(F1, bo.G1_GEN, rnd.randrange(1, bo.R)) for _ in range(16)]
    pts += extra
    want += [int(bo.in_subgroup(F1, q)) for q in extra]
    recs = _records([_aff_rec(F1, q) for q in pts])
    iso = crypto.curve_eval("g1_in_subgroup_iso", recs)[:, 72].tolist()
    lazy = crypto.curve_eval("g1l_in_subgroup", recs)[:, 72].tolist()
    bad = [i for i, (a, b, w) in enumerate(zip(iso, lazy, want)) if not a == b == w]
    assert not bad, f"{len(bad)} of {len(pts)} differ, first {pts[bad[0]]}: iso {iso[bad[0]]} lazy {lazy[bad[0]]} oracle {want[bad[0]]}"
    assert set(want) == {0, 1}
    assert sum(want[len(cases):len(cases) + 48]) < 48    # random points of E(Fp): mostly outside G1


def test_new_ops_are_bounded(engine):
    from ethereum_consensus_b200 import crypto
    lib, ptr = crypto._lib.lib(), crypto._lib.ptr
    a = np.zeros((1, 24), dtype=np.uint32)
    for op in (39, 47):
        assert lib.b200_fp_eval(op, 1, ptr(a), ptr(a), ptr(np.zeros((1, 25), np.uint32))) == crypto._lib.ERR_BAD_ARG
    c = np.zeros((1, 73), dtype=np.uint32)
    for op in (3, 5, 7):
        assert lib.b200_curve_eval(op, 1, ptr(c), ptr(c), ptr(c.copy())) == crypto._lib.ERR_BAD_ARG


# ---------------------------------------------------------------------------------------------------------- split slots
def pool_data(O):
    """About 300 keys in classes, with the oracle's code and one-key aggregation for each."""
    if "pool" in _CACHE:
        return _CACHE["pool"]
    rnd = random.Random(56)
    cases = _g1_cases()
    valid = [c["enc"] for c in cases if c["family"] == "valid"][:96]        # P, -P: both sign flags
    inf = bytes([0xC0]) + bytes(47)
    enc_x = lambda x, flags: bytes([flags | (x >> 376)]) + (x % (1 << 376)).to_bytes(47, "big")   # noqa: E731
    off = []
    while len(off) < 16:
        x = rnd.randrange(P)
        if _y_want(x, False) is None:
            off.append(enc_x(x, 0x80 | 0x20 * (len(off) & 1)))
    classes = {
        "valid": valid,
        "infinity": [inf, bytes([0xE0]) + bytes(47), bytes([0xC1]) + bytes(47), inf[:47] + b"\x01", inf[:20] + b"\x10" + inf[21:]],
        "no compression flag": [bytes([v[0] & 0x7F]) + v[1:] for v in valid[:8]] + [bytes(48), bytes([0x40]) + bytes(47)],
        "x >= p": [enc_x(x, f) for x in (P, P + 1, (1 << 381) - 1) for f in (0x80, 0xA0)],
        "x = p - 1": [enc_x(P - 1, f) for f in (0x80, 0xA0)],
        "off curve": off,
        "small order": [c["enc"] for c in cases if c["family"] in ("torsion", "eigen")][::8],
        "mixed order": [c["enc"] for c in cases if c["family"] in ("Q+T", "-Q+T")][::16],
        "random bytes": [rnd.randbytes(48) for _ in range(8)] + [bytes([0x80 | rnd.randrange(0x40)]) + rnd.randbytes(47) for _ in range(16)],
    }
    keys, cls = [], []
    for k, (name, ks) in enumerate(classes.items()):
        keys += ks
        cls += [k] * len(ks)
    codes = np.array([O.orc_key_validate(k) for k in keys], dtype=np.int32)
    one = [_oracle_bytes(O.orc_eth_aggregate_public_keys, k, 1, 48) for k in keys]
    one_code = np.array([o[0] if isinstance(o, tuple) else o for o in one], dtype=np.int32)
    assert np.array_equal(one_code, codes)
    one_bytes = np.zeros((len(keys), 48), dtype=np.uint8)
    for i, o in enumerate(one):
        if isinstance(o, tuple):
            one_bytes[i] = np.frombuffer(o[1], dtype=np.uint8)
    cls = np.array(cls)
    members = [np.nonzero(cls == k)[0] for k in range(len(classes))]
    assert (codes[members[0]] == 0).all() and all(codes[m].min() > 0 for m in members[1:4])
    _CACHE["pool"] = {"names": list(classes), "arr": np.frombuffer(b"".join(keys), dtype=np.uint8).reshape(-1, 48),
                      "codes": codes, "one_bytes": one_bytes, "members": members, "valid": codes == 0, "pairs": {}}
    return _CACHE["pool"]


def _stream(n):
    """Fixed pseudo-random words: key i of every size gets the same one."""
    if "stream" not in _CACHE or len(_CACHE["stream"]) < n:
        _CACHE["stream"] = np.random.default_rng(57).integers(0, 1 << 32, max(n, SMALL_N + 512), dtype=np.int64)
    return _CACHE["stream"][:n]


def layout(n, D):
    """Pool index of each of n keys.  Position j of CTA c (256 keys) holds class (c + s) mod classes at the s-th special
    position, so that over the CTAs every class meets every special position; elsewhere mostly valid keys; the last key is
    valid (the last CTA's last FP64 key)."""
    members = D["members"]
    i = np.arange(n, dtype=np.int64)
    h = _stream(n)
    valid, other = members[0], np.concatenate(members[1:])
    lay = np.where(h % 10 < 7, valid[(h >> 4) % len(valid)], other[(h >> 12) % len(other)])
    c, j = i // 256, i % 256
    for s, pos in enumerate(SPECIAL):
        for k, m in enumerate(members):
            sel = (j == pos) & ((c + s) % len(members) == k)
            lay[sel] = m[(c[sel] * 7 + s) % len(m)]
    lay[n - 1] = valid[n % len(valid)]
    return lay


def groups(n, lay, D):
    """Pairs of valid keys in different slots: (j, j + 128) in every CTA (all j in the first and the last, a few
    elsewhere), the two sides of each CTA boundary, neighbours in the last CTA, and the last key with the first valid one."""
    ok = D["valid"][lay]
    out = []
    n_cta = (n + 255) // 256
    for c in range(n_cta):
        b = 256 * c
        edge = c in (0, n_cta - 1)
        js = range(128) if edge else sorted({0, 1, 127} | {int(w) % 128 for w in _stream(b + 8)[b:b + 8] >> 20})
        out += [(b + j, b + j + 128) for j in js if b + j + 128 < n and ok[b + j] and ok[b + j + 128]]
        if b + 256 < n and ok[b + 255] and ok[b + 256]:
            out.append((b + 255, b + 256))
    b = 256 * (n_cta - 1)
    out += [(k, k + 1) for k in range(b, n - 1) if ok[k] and ok[k + 1]]
    first = int(np.argmax(ok))
    if first != n - 1:
        out.append((first, n - 1))
    return out


def want_pairs(O, D, ns):
    """The oracle's eth_aggregate_public_keys of every pool pair the groups of these sizes need."""
    cache = D["pairs"]
    for n in ns:
        lay = layout(n, D)
        for a, b in groups(n, lay, D):
            key = (int(lay[a]), int(lay[b]))
            if key not in cache:
                k = D["arr"][key[0]].tobytes() + D["arr"][key[1]].tobytes()
                cache[key] = _oracle_bytes(O.orc_eth_aggregate_public_keys, k, 2, 48)
    return cache


def _where(i):
    return f"key {i} (CTA {i // 256}, j = {i % 256})"


def check_split(n, D, tag=""):
    """Registry load of n keys of the layout; returns [(name, cases, mismatches)] for codes, one-key and two-key sums."""
    from ethereum_consensus_b200 import crypto
    lay = layout(n, D)
    reg = crypto.Registry(np.ascontiguousarray(D["arr"][lay]).reshape(-1))
    res = []

    def record(name, total, bad, first):
        print(f"{name + tag:52s} cases {total:7d}  mismatches {len(bad)}")
        if len(bad):
            print(f"  first mismatch: {first(bad[0])}")
        res.append((name + tag, total, len(bad)))

    codes = reg.key_codes()
    bad = np.nonzero(codes != D["codes"][lay])[0]
    record(f"n = {n}: key codes", n, bad, lambda i: f"{_where(i)}: {codes[i]}, oracle {D['codes'][lay[i]]}")
    out, gc = reg.aggregate_public_keys(np.arange(n, dtype=np.uint32), np.arange(n + 1, dtype=np.uint32))
    bad = np.nonzero((gc != D["codes"][lay]) | ~np.all(out == D["one_bytes"][lay], axis=1))[0]
    record(f"n = {n}: one-key aggregation", n, bad, lambda i: f"{_where(i)}: code {gc[i]} {out[i].tobytes().hex()}")
    pairs = groups(n, lay, D)
    if pairs:
        idx = np.array(pairs, dtype=np.uint32).reshape(-1)
        out, gc = reg.aggregate_public_keys(idx, np.arange(0, 2 * len(pairs) + 1, 2, dtype=np.uint32))
        got = [(0, out[t].tobytes()) if gc[t] == 0 else int(gc[t]) for t in range(len(pairs))]
        want = [D["pairs"][(int(lay[a]), int(lay[b]))] for a, b in pairs]
        bad = [t for t in range(len(pairs)) if got[t] != want[t]]
        record(f"n = {n}: two-key aggregation", len(pairs), bad,
               lambda t: f"{_where(pairs[t][0])} + {_where(pairs[t][1])}: {got[t]!r}, oracle {want[t]!r}")
    return res


def _assert_clean(res):
    for name, n, bad in res:
        assert bad == 0, f"{name}: {bad} of {n} cases differ from the oracle"


def test_pool_and_layout_cover_every_class_and_slot(oracle_bls_c):
    D = pool_data(oracle_bls_c)
    n = SMALL_N + 256
    lay = layout(n, D)
    cls = np.zeros(len(D["arr"]), dtype=np.int64)
    for k, m in enumerate(D["members"]):
        cls[m] = k
    j = np.arange(n) % 256
    for pos in SPECIAL:
        assert set(cls[lay[j == pos]].tolist()) == set(range(len(D["members"]))), pos
    assert 250 <= len(D["arr"]) <= 400
    assert set(D["codes"].tolist()) >= {0, 1, 2, 3, 6}


@pytest.mark.parametrize("r", (0,) + TAILS)
def test_split_slots_and_tails_in_registry_loads(engine, oracle_bls_c, r):
    """n = SMALL_N + r keys: 666 full CTAs of the role-split kernel and a last one of r keys (r = 0: the 128-thread kernel
    on the same keys, the control)."""
    t = time.time()
    D = pool_data(oracle_bls_c)
    want_pairs(oracle_bls_c, D, [SMALL_N + r])
    res = check_split(SMALL_N + r, D)
    print(f"wall {time.time() - t:.1f} s")
    _assert_clean(res)


def test_split_slots_small_calls_in_child_process(oracle_bls_c, tmp_path):
    """Every size around the 128-key halves and the 256-key CTAs, through k_g1_validate_split alone (B200_G1_SMALL_N=0,
    read once per process)."""
    t = time.time()
    D = pool_data(oracle_bls_c)
    want_pairs(oracle_bls_c, D, CHILD_NS)
    path = tmp_path / "pool.pkl"
    path.write_bytes(pickle.dumps(D))
    env = dict(os.environ, B200_G1_SMALL_N="0")
    p = subprocess.Popen([sys.executable, "-m", "tests.test_fpd_device_gpu", str(path)], cwd=str(ROOT), env=env,
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    try:
        out = p.communicate(timeout=600)[0]
    except subprocess.TimeoutExpired:
        p.kill()
        out = p.communicate()[0]
    print(out)
    print(f"child B200_G1_SMALL_N=0 wall {time.time() - t:.1f} s")
    assert p.returncode == 0, out
    assert "CHILD_OK" in out, out


def _child(path):
    from ethereum_consensus_b200 import _lib
    _lib.init(0)
    D = pickle.loads(Path(path).read_bytes())
    res = []
    for n in CHILD_NS:
        res += check_split(n, D, " [B200_G1_SMALL_N=0]")
    _assert_clean(res)
    print("CHILD_OK")


if __name__ == "__main__":
    _child(sys.argv[1])
