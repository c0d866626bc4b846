"""GPU: small-order and mixed-order curve points (tests/torsion_cases.py) through the CUDA kernels, case by case against
the definition-level oracle ([r]P == infinity).

These are the only inputs that take the subgroup checks' ladders into their doubling / inverse / infinity branches, and
in the per-key kernel those branches run on lazily reduced FpL, where "zero" may be the representative p.  Sections:
a. keys through every key entry point, b. signatures through aggregate and K = 1 tuples, c. one torsion-laden key or
signature in an otherwise valid RLC batch, d. single curve stages through b200_curve_eval (subgroup checks without a
decode in front, psi, cofactor clearing, the map, hash_to_G2's second half, and the FpL / Fp2 additions on their
exceptional operands).  B200_G1_SMALL_N is read once per process, so section a runs again in a child process with
every per-key launch through the role-split kernel.

    B200_SOAK_SCALE=1 (default) python -m pytest tests/test_torsion_gpu.py -m gpu -s
"""
from __future__ import annotations

import hashlib
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
from tests.test_bls_device_soak_gpu import SMALL_N, _code, _oracle_batch, _pack, _sign_batch, report  # noqa: E402

pytestmark = pytest.mark.gpu
F1, F2, P, R = bo.F1, bo.F2, bo.P, bo.R
RM = 1 << 384
RINV = pow(RM, -1, P)
RLC_SEED = hashlib.sha256(b"torsion rlc").digest()
W = 73                                     # words of a b200_curve_eval record


# ---------------------------------------------------------------------------------------------------------- records
def _put(rec, slot, v):
    """Fp (int) or Fp2 (pair) value v, already a raw representative, into 24-word slot `slot`."""
    parts = v if isinstance(v, tuple) else (v,)
    for j, x in enumerate(parts):
        rec[24 * slot + 12 * j: 24 * slot + 12 * j + 12] = [(x >> (32 * k)) & 0xFFFFFFFF for k in range(12)]


def _get(rec, slot, fp2):
    vals = [sum(int(rec[24 * slot + 12 * j + k]) << (32 * k) for k in range(12)) for j in range(2 if fp2 else 1)]
    return tuple(vals) if fp2 else vals[0]


def _mont(v):
    return tuple(x * RM % P for x in v) if isinstance(v, tuple) else v * RM % P


def _real(v):
    return tuple(x * RINV % P for x in v) if isinstance(v, tuple) else v * RINV % P


def _jac(F, a, z=None):
    """Affine a -> Jacobian (X, Y, Z) in the real domain with Z = z (1 by default); infinity -> (1, 1, 0)."""
    if a is None:
        return (F.one, F.one, F.zero)
    z = F.one if z is None else z
    z2 = F.sqr(z)
    return (F.mul(a[0], z2), F.mul(a[1], F.mul(z2, z)), z)


def _records(pts):
    """[(X, Y, Z, flag)] real-domain coordinates -> uint32[n, 73] in Montgomery form."""
    out = np.zeros((max(len(pts), 1), W), dtype=np.uint32)
    for i, (x, y, z, flag) in enumerate(pts):
        _put(out[i], 0, _mont(x)); _put(out[i], 1, _mont(y)); _put(out[i], 2, _mont(z))
        out[i, 72] = flag
    return out[:len(pts)]


def _affine_out(F, out):
    fp2 = F is F2
    return [bo.pt_to_affine(F, tuple(_real(_get(r, s, fp2)) for s in range(3))) for r in out]


def _aff_rec(F, a):
    x, y, z = _jac(F, a)
    return (x, y, z, 1 if a is None else 0)


# ---------------------------------------------------------------------------------------------------------- inputs
_CACHE = {}


def data(O):
    """Generated once per process: both case lists, signatures over them (C oracle) and the tuples built on them."""
    if "d" in _CACHE:
        return _CACHE["d"]
    t = time.time()
    g1, g2 = tc.g1_cases(), tc.g2_cases()
    keys = g1["cases"]
    msgs1 = [hashlib.sha256(b"torsion/key%d" % i).digest() for i in range(len(keys))]
    sks1 = [(c.get("sk", 1) % R or 1).to_bytes(32, "big") for c in keys]
    key_tuples = [(c["enc"], m, s) for c, m, s in zip(keys, msgs1, _sign_batch(O, sks1, msgs1))]
    sigs = g2["cases"]
    import ctypes as C
    pkbuf = C.create_string_buffer(48)
    sig_tuples = []
    for i, c in enumerate(sigs):
        O.orc_sk_to_pk((c.get("sk", 1 + i) % R or 1).to_bytes(32, "big"), pkbuf)
        sig_tuples.append((pkbuf.raw, c.get("msg", hashlib.sha256(b"torsion/sig%d" % i).digest()), c["enc"]))
    d = {"g1": g1, "g2": g2, "key_tuples": key_tuples, "key_tuples_want": _oracle_batch(O, key_tuples),
         "sig_tuples": sig_tuples, "sig_tuples_want": _oracle_batch(O, sig_tuples)}
    print(f"inputs: {len(keys)} G1 and {len(sigs)} G2 encodings, {time.time() - t:.1f} s")
    _CACHE["d"] = d
    return d


def _keys_section(D):
    """The part of `data` that section a needs, picklable for the child processes."""
    keys = D["g1"]["cases"]
    valid = [c["enc"] for c in keys if c["family"] == "valid"][:64]
    return {"enc": [c["enc"] for c in keys], "code": [c["code"] for c in keys], "valid": valid,
            "tuples": D["key_tuples"], "tuples_oracle": D["key_tuples_want"]}


def _report_points(name, want, got, is_inf=lambda w: w is None):
    """report() for point-valued results: the summary line counts infinite and finite expected points."""
    want, got = list(want), list(got)
    assert len(want) == len(got), (name, len(want), len(got))
    bad = [i for i, (w, g) in enumerate(zip(want, got)) if w != g]
    n_inf = sum(1 for w in want if is_inf(w))
    print(f"{name:44s} cases {len(want):6d}  mismatches {len(bad)}   infinity {n_inf}, finite {len(want) - n_inf}")
    sys.stdout.flush()
    if bad:
        print(f"  first mismatch: case {bad[0]}: oracle {want[bad[0]]!r}, device {got[bad[0]]!r}")
    return len(want), len(bad)


def _assert_clean(res):
    for name, n, bad in res:
        assert bad == 0, f"{name}: {bad} of {n} cases differ from the oracle"


# ---------------------------------------------------------------------------------------------------------- section a
def check_keys(K, tag=""):
    from ethereum_consensus_b200 import crypto
    res = []
    enc, code = K["enc"], K["code"]
    flat = np.frombuffer(b"".join(enc), dtype=np.uint8)
    res.append(("a. registry" + tag, *report("a. key_validate (registry, 128-thread CTAs)" + tag, code,
                                             crypto.Registry(flat).key_codes().tolist())))
    reps = SMALL_N // len(enc) + 2
    got = crypto.Registry(np.tile(flat, reps)).key_codes().tolist()
    res.append(("a. registry tiled" + tag, *report(f"a. key_validate (registry, n = {len(got)})" + tag, code * reps, got)))
    tup = K["tuples"]
    want = [c if c else 0 for c in code]                        # a valid key carries a valid signature
    assert K["tuples_oracle"] == want
    res.append(("a. strict K = 1" + tag, *report("a. K = 1 strict batch, signature valid for Q" + tag, want,
                                                 crypto.fast_aggregate_verify_batch(*_pack(tup)).tolist())))
    # the keys as `..._batch_mixed` extras behind a registry of valid keys
    reg = crypto.Registry(np.frombuffer(b"".join(K["valid"]), dtype=np.uint8))
    idx = np.arange(len(K["valid"]), len(K["valid"]) + len(tup), dtype=np.uint32)
    _, off, msgs, sigs = _pack(tup)
    got = reg.verify_batch(idx, off, msgs, sigs, extra_keys=flat).tolist()
    res.append(("a. mixed extras" + tag, *report("a. K = 1 as _batch_mixed extra keys" + tag, want, got)))
    got = [_code(crypto.eth_aggregate_public_keys, [e]) for e in enc]
    res.append(("a. eth_aggregate_public_keys" + tag, *report("a. eth_aggregate_public_keys([pk])" + tag,
                                                             [(0, e) if c == 0 else c for e, c in zip(enc, code)], got)))
    return res


def test_a_keys(engine, oracle_bls_c):
    t = time.time()
    D = data(oracle_bls_c)
    res = check_keys(_keys_section(D))
    print(f"a. wall {time.time() - t:.1f} s")
    _assert_clean(res)


# ---------------------------------------------------------------------------------------------------------- section b
def _g2_bad_decodes():
    """One encoding that fails to decode with each code (1: compression bit clear, 2: x not on E')."""
    x = 0
    while bo.g2_uncompress((0x80 << 760 | x).to_bytes(96, "big"))[0] != bo.POINT_NOT_ON_CURVE:
        x += 1
    return [bytes(96), (0x80 << 760 | x).to_bytes(96, "big")]


def test_b_signatures(engine, oracle_bls_c):
    from ethereum_consensus_b200 import crypto
    t = time.time()
    D = data(oracle_bls_c)
    cases = D["g2"]["cases"]
    res = []
    want = [(0, c["enc"]) if c["code"] == 0 else c["code"] for c in cases]
    res.append(("b. aggregate([sig])", *report("b. aggregate([sig])", want, [_code(crypto.aggregate, [c["enc"]]) for c in cases])))
    # among valid signatures, and with a decode error after it (decode errors win over the group check)
    valid = [c for c in cases if c["family"] == "valid"]
    bad_dec = _g2_bad_decodes()
    rnd = random.Random(7)
    want3, got3, want_d, got_d, sample = [], [], [], [], []
    for i, c in enumerate(cases):
        v1, v2 = valid[rnd.randrange(len(valid))], valid[rnd.randrange(len(valid))]
        if c["code"]:
            want3.append(c["code"])
        else:
            want3.append((0, bo.g2_compress(tc.add(F2, tc.add(F2, v1["pt"], c["pt"]), v2["pt"]))))
        got3.append(_code(crypto.aggregate, [v1["enc"], c["enc"], v2["enc"]]))
        bd = bad_dec[i % 2]
        want_d.append(bo.g2_uncompress(bd)[0])
        got_d.append(_code(crypto.aggregate, [v1["enc"], c["enc"], bd]))
        if i % 40 == 0:
            sample.append(([v1["enc"], c["enc"], v2["enc"]], want3[-1]))
            sample.append(([v1["enc"], c["enc"], bd], want_d[-1]))
    for sig_list, w in sample:                                 # the definition's aggregate agrees with the rule used here
        code, out = bo.aggregate(sig_list)
        assert ((0, out) if code == 0 else code) == w
    res.append(("b. aggregate among valid", *report("b. aggregate([v, sig, v])", want3, got3)))
    res.append(("b. decode error wins", *report("b. aggregate([v, sig, bad decode])", want_d, got_d)))
    tup = D["sig_tuples"]
    want_t = [0 if c["code"] == 0 else bo.VERIFY_FAIL for c in cases]
    assert D["sig_tuples_want"] == want_t
    args = _pack(tup)
    try:
        for cta in (32, 128):
            crypto.tune("bls_small_cta", cta)
            res.append((f"b. K = 1, small CTA {cta}", *report(f"b. K = 1 with sigma + T, bls_small_cta {cta}", want_t,
                                                             crypto.fast_aggregate_verify_batch(*args).tolist())))
    finally:
        crypto.tune("bls_small_cta", 0)
    print(f"b. wall {time.time() - t:.1f} s")
    _assert_clean(res)


# ---------------------------------------------------------------------------------------------------------- section c
def test_c_rlc_one_torsion_point_per_batch(engine, oracle_bls_c):
    """Sound only if every point reaching it is in G2 / G1: one torsion-laden key or signature among 16 valid tuples,
    first, middle or last, must give False through both whole-batch entry points; the all-valid batch gives True."""
    from ethereum_consensus_b200 import crypto
    t = time.time()
    D = data(oracle_bls_c)
    keys, sigs = D["g1"]["cases"], D["g2"]["cases"]
    ok_k = [tp for tp, c in zip(D["key_tuples"], keys) if c["family"] == "valid"][:16]
    bad_k = [tp for tp, c in zip(D["key_tuples"], keys) if c["code"]]
    bad_s = [tp for tp, c in zip(D["sig_tuples"], sigs) if c["code"]]
    stride_k, stride_s = max(1, len(bad_k) // 60), max(1, len(bad_s) // 60)
    bad = bad_k[::stride_k] + bad_s[::stride_s]
    pool = ok_k + [tp for tp in bad]
    uniq = sorted({tp[0] for tp in pool})
    pos = {p: i for i, p in enumerate(uniq)}
    reg = crypto.Registry(np.frombuffer(b"".join(uniq), dtype=np.uint8))
    want, got_f, got_r = [], [], []
    batches = [ok_k]
    for b in bad:
        for where in (0, len(ok_k) // 2, len(ok_k)):
            batches.append(ok_k[:where] + [b] + ok_k[where:])
    for bt in batches:
        want.append(bt is ok_k)
        args = _pack(bt)
        got_f.append(crypto.fast_aggregate_verify_batch_all(*args, seed=RLC_SEED))
        idx = np.array([pos[tp[0]] for tp in bt], dtype=np.uint32)
        got_r.append(reg.verify_batch_all(idx, args[1], args[2], args[3], seed=RLC_SEED))
    res = [("c. fast_aggregate_verify_batch_all", *report("c. RLC, one torsion-laden point", want, got_f)),
           ("c. Registry.verify_batch_all", *report("c. RLC over the registry, one torsion-laden point", want, got_r))]
    print(f"c. wall {time.time() - t:.1f} s")
    _assert_clean(res)
    assert len(batches) > 300


# ---------------------------------------------------------------------------------------------------------- section d
def test_d_subgroup_checks_without_decode(engine, oracle_bls_c):
    from ethereum_consensus_b200 import crypto
    D = data(oracle_bls_c)
    res = []
    for F, op, cases in ((F1, "g1l_in_subgroup", D["g1"]["cases"]), (F2, "g2_in_subgroup", D["g2"]["cases"])):
        pts = [c["pt"] for c in cases] + [None]
        want = [int(c["code"] == 0) for c in cases] + [1]
        got = crypto.curve_eval(op, _records([_aff_rec(F, a) for a in pts]))[:, 72].tolist()
        res.append((f"d. {op}", *report(f"d. {op} on the decoded points", want, got)))
    _assert_clean(res)


def test_d_psi_and_clear_cofactor(engine, oracle_bls_c):
    from ethereum_consensus_b200 import crypto
    D = data(oracle_bls_c)
    cases = D["g2"]["cases"]
    rnd = random.Random(8)
    tors = [c["pt"] for c in cases if c["order"] < R]
    mixed = [c["pt"] for c in cases if c["family"] == "sigma+T"][::4]
    valid = [c["pt"] for c in cases if c["family"] == "valid"][::8]     # psi(P) = [z]P: [z]P + psi(P) is a doubling
    randoms = [tc.g2_random(rnd) for _ in range(24)]
    pts = tors + mixed + valid + randoms + [None]
    recs = _records([_jac(F2, a, (rnd.randrange(1, P), rnd.randrange(P))) + (0,) for a in pts])
    res = [("d. g2_psi", *_report_points("d. g2_psi (Jacobian, random Z)", [tc.psi(a) for a in pts],
                                 _affine_out(F2, crypto.curve_eval("g2_psi", recs))))]
    want = [tc.mul(F2, a, bo.H_EFF) for a in pts]
    assert all(w is None for w in want[:len(tors)])
    res.append(("d. g2_clear_cofactor", *_report_points("d. g2_clear_cofactor = [h_eff]P", want,
                                                _affine_out(F2, crypto.curve_eval("g2_clear_cofactor", recs)))))
    _assert_clean(res)


def test_d_map_and_finish(engine, oracle_bls_c):
    from ethereum_consensus_b200 import crypto
    rnd = random.Random(9)
    us = tc.sswu_inputs(2000)
    recs = _records([(u, bo.F2_ONE, bo.F2_ONE, 0) for u in us])
    got = _affine_out(F2, crypto.curve_eval("g2_sswu_iso", recs))
    res = [("d. map", *_report_points("d. B200_SSWU_ISO(u) = iso3(sswu(u))", [bo.iso3(bo.sswu(u)) for u in us], got))]
    # finish(q0, q1) = [h_eff](q0 + q1) on Jacobian inputs: q1 = q0, q1 = -q0, an infinity operand, torsion-laden q0
    D = data(oracle_bls_c)
    tors = [c["pt"] for c in D["g2"]["cases"] if c["order"] < R][::6]
    q0s = [g for g in got[:40] if g is not None] + tors
    pairs = []
    for q in q0s:
        other = got[100 + len(pairs) % 50]
        pairs += [(q, q), (q, tc.neg(F2, q)), (q, None), (None, q), (q, other)]
    z = lambda: (rnd.randrange(1, P), rnd.randrange(P))   # noqa: E731
    a = _records([_jac(F2, p0, z()) + (0,) for p0, _ in pairs])
    b = _records([_jac(F2, p1, z()) + (0,) for _, p1 in pairs])
    out = crypto.curve_eval("g2_h2c_finish", a, b)
    want = [tc.mul(F2, tc.add(F2, p0, p1), bo.H_EFF) for p0, p1 in pairs]
    res.append(("d. finish", *_report_points("d. hash_to_g2_finish(q0, q1)", [(w is None, w) for w in want],
                                            [(bool(o[72]), g) for o, g in zip(out, _affine_out(F2, out))], lambda w: w[0])))
    _assert_clean(res)
    assert bo.f2_is_zero(us[0]) and sum(w is None for w in want) >= 2 * len(q0s)


def _shifted(v, shift):
    """Raw Montgomery representative of real value v, plus p when shift (both in [0, 2p))."""
    return _mont(v) + (P if shift else 0)


def test_d_lazy_and_fp2_additions_on_exceptional_operands(engine, oracle_bls_c):
    """jac_add_mixed / jac_add on FpL (the per-key kernel's field) with every coordinate given as v or v + p, so that the
    h == 0 / rr == 0 tests see the representative p; and the Fp2 formulas of the signature unit on equal, opposite and
    infinite operands."""
    from ethereum_consensus_b200 import crypto
    D = data(oracle_bls_c)
    rnd = random.Random(10)
    g1 = D["g1"]["cases"]
    base = [c["pt"] for c in g1 if c["family"] == "valid"][:4] + [c["pt"] for c in g1 if c["order"] in (3, 11)][:4]
    a_rows, b_rows, want = [], [], []

    def row(x, y, z, sx, sy, sz):
        r = np.zeros(W, dtype=np.uint32)
        _put(r, 0, _shifted(x, sx)); _put(r, 1, _shifted(y, sy)); _put(r, 2, _shifted(z, sz))
        return r

    for q in base:
        other = base[(base.index(q) + 1) % len(base)]
        for rel, pa in (("dbl", q), ("inv", tc.neg(F1, q)), ("gen", other), ("inf", None)):
            for zc in (1, rnd.randrange(2, P)):
                X, Y, Zc = _jac(F1, pa, zc) if pa is not None else (1, 1, 0)
                QX, QY, QZ = _jac(F1, q, rnd.randrange(2, P))
                expect = tc.add(F1, pa, q)
                for s in range(32):                              # mixed: (X, Y, Z) x (qx, qy) shifts
                    a_rows.append(row(X, Y, Zc, s & 1, s >> 1 & 1, s >> 2 & 1))
                    b_rows.append(row(q[0], q[1], 1, s >> 3 & 1, s >> 4 & 1, 0))
                    want.append(("mixed", expect))
                for s in rnd.sample(range(64), 16):              # general: both Jacobian
                    a_rows.append(row(X, Y, Zc, s & 1, s >> 1 & 1, s >> 2 & 1))
                    b_rows.append(row(QX, QY, QZ, s >> 3 & 1, s >> 4 & 1, s >> 5 & 1))
                    want.append(("general", expect))
                    a_rows.append(row(QX, QY, QZ, s >> 3 & 1, s >> 4 & 1, s >> 5 & 1))    # q + p, operands swapped
                    b_rows.append(row(X, Y, Zc, s & 1, s >> 1 & 1, s >> 2 & 1))
                    want.append(("general", expect))
    a, b = np.stack(a_rows), np.stack(b_rows)
    res = []
    for kind, op in (("mixed", "g1l_add_mixed"), ("general", "g1l_add")):
        sel = [i for i, w in enumerate(want) if w[0] == kind]
        out = crypto.curve_eval(op, a[sel], b[sel])
        assert all(_get(o, s, False) < 2 * P for o in out for s in range(3))
        res.append((f"d. {op}", *_report_points(f"d. {op} on [0, 2p) representatives", [want[i][1] for i in sel], _affine_out(F1, out))))
    # G2: the signature unit's formulas on torsion points and their multiples: equal, opposite, infinite operands
    g2 = [c["pt"] for c in D["g2"]["cases"] if c["order"] < R][::5] + [c["pt"] for c in D["g2"]["cases"] if c["family"] == "valid"][:6]
    z = lambda: (rnd.randrange(1, P), rnd.randrange(P))   # noqa: E731
    pairs = [(q, p) for q in g2 for p in (q, tc.neg(F2, q), None, g2[rnd.randrange(len(g2))])]
    pairs += [(None, q) for q in g2[:8]]
    a = _records([_jac(F2, p, z()) + (0,) for p, _ in pairs])
    b = _records([_jac(F2, q, z()) + (0,) for _, q in pairs])
    bm = _records([_aff_rec(F2, q) for _, q in pairs])
    want = [tc.add(F2, p, q) for p, q in pairs]
    res.append(("d. g2_add", *_report_points("d. g2 jac_add", want, _affine_out(F2, crypto.curve_eval("g2_add", a, b)))))
    sel = [i for i, (_, q) in enumerate(pairs) if q is not None]
    res.append(("d. g2_add_mixed", *_report_points("d. g2 jac_add_mixed", [want[i] for i in sel],
                                           _affine_out(F2, crypto.curve_eval("g2_add_mixed", a[sel], bm[sel])))))
    res.append(("d. g2_double", *_report_points("d. g2 jac_double", [tc.add(F2, p, p) for p, _ in pairs],
                                        _affine_out(F2, crypto.curve_eval("g2_double", a)))))
    _assert_clean(res)


def test_curve_eval_rejects_unknown_ops(engine):
    from ethereum_consensus_b200 import crypto
    a = np.zeros((1, W), dtype=np.uint32)
    for op in (3, 31, 40, -1):
        assert crypto._lib.lib().b200_curve_eval(op, 1, crypto._lib.ptr(a), crypto._lib.ptr(a), crypto._lib.ptr(a.copy())) == crypto._lib.ERR_BAD_ARG


# ---------------------------------------------------------------------------------------------------------- variants
CHILD_ENVS = {"small_n_0": {"B200_G1_SMALL_N": "0"}}


@pytest.mark.parametrize("variant", list(CHILD_ENVS))
def test_a_keys_per_g1_variant_in_child_processes(oracle_bls_c, tmp_path, variant):
    """Section a with every per-key launch through the role-split kernel (B200_G1_SMALL_N=0), which only the
    environment selects (read once per process)."""
    t = time.time()
    path = tmp_path / "keys.pkl"
    path.write_bytes(pickle.dumps(_keys_section(data(oracle_bls_c))))
    env = dict(os.environ, **CHILD_ENVS[variant])
    p = subprocess.Popen([sys.executable, "-m", "tests.test_torsion_gpu", str(path)], cwd=str(ROOT), env=env,
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    try:
        out = p.communicate(timeout=600)[0]
    except subprocess.TimeoutExpired:
        p.kill()
        out = p.communicate()[0]
    print(out)
    print(f"child {CHILD_ENVS[variant]} wall {time.time() - t:.1f} s")
    assert p.returncode == 0, out
    assert "CHILD_OK" in out, out


def _child(path):
    from ethereum_consensus_b200 import _lib
    _lib.init(0)
    K = pickle.loads(Path(path).read_bytes())
    _assert_clean(check_keys(K, " [small n %s]" % os.environ.get("B200_G1_SMALL_N", "default")))
    print("CHILD_OK")


if __name__ == "__main__":
    _child(sys.argv[1])
