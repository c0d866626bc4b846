"""GPU: the per-key kernel's fused reductions and its FpL doubling, built as the kernel builds them (bls_g1.cu, by-value
calls), against Python integers: f_mul_sub_mul / f_mul_sub_8sqr through b200_fp_eval (exact representative), and
jac_double on FpL through b200_curve_eval with every coordinate given as v or v + p."""
from __future__ import annotations

import random

import numpy as np
import pytest

from oracle import bls_oracle as bo
from tests import torsion_cases as tc
from tests.test_fpl_fused import EDGE, P, RINV, _affine, _ints, _jac_rec, _limbs, redc

pytestmark = pytest.mark.gpu
F1 = bo.F1


def _fixup(r):
    if r >= 4 * P:
        r -= 4 * P
    if r >= 2 * P:
        r -= 2 * P
    return r


def test_device_fused_reductions_match_big_integers(engine):
    from ethereum_consensus_b200 import crypto
    rnd = random.Random(41)
    t = [(a, b, c, d) for a in EDGE for b in EDGE for c in EDGE for d in EDGE[::2]]
    t += [tuple(rnd.randrange(2 * P) for _ in range(4)) for _ in range(20000)]
    a = np.concatenate([_limbs([x[0] for x in t]), _limbs([x[1] for x in t])], axis=1)
    b = np.concatenate([_limbs([x[2] for x in t]), _limbs([x[3] for x in t])], axis=1)
    got = _ints(crypto.fp_eval("fpl_mul_sub_mul", a, b)[:, :12])
    want = [redc(x * y + c * (2 * P - d)) for x, y, c, d in t]
    bad = [i for i, (g, w) in enumerate(zip(got, want)) if g != w]
    assert not bad, f"fpl_mul_sub_mul: {len(bad)} of {len(t)} differ, first {tuple(map(hex, t[bad[0]]))}"
    assert all(g % P == (x * y - c * d) * RINV % P for g, (x, y, c, d) in zip(got[:2000], t))
    got = _ints(crypto.fp_eval("fpl_mul_sub_8sqr", a, b)[:, :12])
    want = [_fixup(redc(x * y + 32 * P * P - 8 * c * c)) for x, y, c, _ in t]
    bad = [i for i, (g, w) in enumerate(zip(got, want)) if g != w]
    assert not bad, f"fpl_mul_sub_8sqr: {len(bad)} of {len(t)} differ, first {tuple(map(hex, t[bad[0]]))}"
    assert max(got) < 2 * P


def test_device_fpl_double_on_both_representatives(engine):
    from ethereum_consensus_b200 import crypto
    rnd = random.Random(42)
    D = tc.g1_cases()["cases"]
    pts = [c["pt"] for c in D if c["pt"] is not None][:40] + [tc.g1_random(rnd) for _ in range(24)] + [None]
    rows, want = [], []
    for q in pts:
        for s in range(8):
            rec = np.zeros(73, dtype=np.uint32)
            for k, v in enumerate(_jac_rec(q, rnd.randrange(1, P), s)):
                rec[24 * k: 24 * k + 12] = _limbs([v])[0]
            rows.append(rec)
            want.append(tc.add(F1, q, q))
    out = crypto.curve_eval("g1l_double", np.stack(rows))
    recs = [_ints(out[:, 24 * k: 24 * k + 12]) for k in range(3)]
    assert max(max(r) for r in recs) < 2 * P
    got = [_affine(r) for r in zip(*recs)]
    bad = [i for i, (g, w) in enumerate(zip(got, want)) if g != w]
    assert not bad, f"g1l_double: {len(bad)} of {len(want)} differ"


def test_new_eval_ops_are_bounded(engine):
    from ethereum_consensus_b200 import crypto
    a = np.zeros((1, 24), dtype=np.uint32)
    for op in (21, 22):
        assert crypto._lib.lib().b200_fp_eval(op, 1, crypto._lib.ptr(a), crypto._lib.ptr(a), crypto._lib.ptr(np.zeros((1, 25), np.uint32))) == crypto._lib.ERR_BAD_ARG
    c = np.zeros((1, 73), dtype=np.uint32)
    for op in (3, 5):
        assert crypto._lib.lib().b200_curve_eval(op, 1, crypto._lib.ptr(c), crypto._lib.ptr(c), crypto._lib.ptr(c.copy())) == crypto._lib.ERR_BAD_ARG
