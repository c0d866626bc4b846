"""CPU: the RLC soak's generators (tests/rlc_soak_cases.py) sit on the boundaries they name, the C oracle's per-tuple
codes match what the cases were built to be, and the exponent model agrees with the oracle's own pairing on every small
batch, crafted ones included, for every seed tried."""
from __future__ import annotations

import hashlib

import pytest

from tests import rlc_soak_cases as rc


@pytest.fixture(scope="module")
def soak(oracle_bls_c):
    return rc.all_cases(oracle_bls_c)


def test_rlc_scalar_is_the_documented_derivation():
    seed = bytes(range(32))
    h = hashlib.sha256(seed + (5).to_bytes(8, "little")).digest()
    assert rc.rlc_scalar(seed, 5) == int.from_bytes(h[:8], "little")
    assert rc.rlc_scalar(seed, 5) != rc.rlc_scalar(seed, 1 << 32 | 5)       # all 64 bits of t are hashed
    assert rc.rlc_scalar(seed, 5) != rc.rlc_scalar(rc.SEED, 5)
    assert max(rc.rlc_scalar(rc.SEED, t) for t in range(64)) >= 1 << 60       # 64-bit scalars, not 32


def test_every_boundary_and_family_is_present(soak):
    _, _, fam = soak
    tags = set().union(*(c.tags for cs in fam.values() for c in cs))
    for K in (1, 2, 33, 512):
        assert f"A:K{K}" in tags
    for t in ("A:(0,T-1)", "A:(t,t+32)", "A:across warps", "A:across the second fold level", "A:zero seed", "A:infinity signature",
              "A:control trunc32", "A:control swap", "A:control defect+1"):
        assert t in tags, t
    for s in (16, 8, 4, 2, 1):
        assert f"B:level1 s{s}" in tags
    for t in ("B:level2", "B:level3", "B:S=inf", "B:equal", "B:opposite", "B:defect"):
        assert t in tags, t
    for T in rc.SMALL_T + rc.LARGE_T:
        assert f"C:T{T}" in tags
    # the fold's launch boundaries (T + 1 crossing 32 and 1 024) and the team-16 -> team-8 switch (T + 1 = 2 048)
    sizes = {len(c.batch) for c in fam["C"]}
    assert {30, 31, 32, 1022, 1023, 1024, 2046, 2047, 2048}.issubset({T - 1 for T in sizes} | {T for T in sizes})
    assert {31, 32, 33, 1023, 1024, 1025, 2047, 2048, 2049}.issubset(sizes)
    c = fam["C"]
    for T in rc.SMALL_T:
        for what in ("defect", "dead"):
            assert sorted(int(x.name.rsplit(" ", 1)[1]) for x in c if x.name.startswith(f"C T {T} {what} at")) == list(range(T))
    for T in rc.LARGE_T:
        got = {int(x.name.rsplit(" ", 1)[1]) for x in c if x.name.startswith(f"C T {T} defect at")}
        want = {0, T - 1} | {p for w in range((T + 31) // 32) for p in (32 * w, min(32 * w + 31, T - 1))}
        assert got == want, T
    dead = {t.dead for x in c for t in x.batch if t.dead}
    assert dead == set(rc.DEAD_KINDS)


def test_family_a_cancels_only_under_its_seed(soak):
    _, _, fam = soak
    crafted = [c for c in fam["A"] if "A:crafted" in c.tags]
    assert len(crafted) >= 14
    for c in crafted:
        assert all(t.defect for t in c.batch), c.name                     # every tuple invalid on its own
        assert c.runs[0][1] is True, c.name
        assert [w for _, w in c.runs[1:]] == [False] * (len(c.runs) - 1), c.name
        assert c.runs[-1] == (None, False)
        assert {rc.ZERO_SEED, rc.SEED} & {s for s, _ in c.runs[1:]}
    for c in fam["A"]:
        if c.tags & {"A:control trunc32", "A:control swap", "A:control defect+1"}:
            assert c.runs == [(c.runs[0][0], False)], c.name
    # K in {1, 2, 33, 512}: the aggregate of each crafted tuple goes through K keys
    assert {len(t.keys) for c in crafted for t in c.batch} >= {1, 2, 33, 512}


def test_family_b_meets_equal_and_opposite_operands(soak):
    _, _, fam = soak
    for c in fam["B"]:
        want = "B:defect" not in c.tags
        assert c.runs == [(rc.SEED, want)], c.name
        if "B:S=inf" in c.tags:
            assert sum(rc.rlc_scalar(rc.SEED, t) * x.sigma for t, x in enumerate(c.batch)) % rc.R == 0
    # each solved level-1 target really makes its jac_add operands equal / opposite
    for name, T, level, w, s, lane, sign, _tags in rc.b_targets():
        case = next(c for c in fam["B"] if c.name == f"B {name}")
        op = next(o for o in rc.fold_ops(T) if o[:4] == (level, w, s, lane))
        sc = lambda ix: sum(rc.rlc_scalar(rc.SEED, t) * case.batch[t].sigma for t in ix) % rc.R   # noqa: E731
        assert sc(op[5]) == (sign * sc(op[4])) % rc.R, name


def test_fold_ops_mirror_the_launches():
    assert [o[:4] for o in rc.fold_ops(2)][-1] == (1, 0, 1, 0)
    ops = rc.fold_ops(1025)
    assert max(o[0] for o in ops) == 3 and max(o[0] for o in rc.fold_ops(1024)) == 2
    last = ops[-1]
    assert set(last[4]) == set(range(1024)) and set(last[5]) == {1024}


def test_oracle_codes_match_the_construction(soak, oracle_bls_c):
    keys, M, fam = soak
    tuples = list(dict.fromkeys(t for f in ("A", "B") for c in fam[f] for t in c.batch))
    tuples += list(dict.fromkeys(t for c in fam["C"] if len(c.batch) <= 65 for t in c.batch))
    tuples = list(dict.fromkeys(tuples))
    codes = M.codes(tuples)
    for t, code in zip(tuples, codes):
        want = rc.expected_code(t)
        if want is None:
            assert code not in (0,), (t.dead, code)
        else:
            assert code == want, (t, code)
    crafted = {t for c in fam["A"] if "A:crafted" in c.tags for t in c.batch}
    assert {M.code[t] for t in crafted} == {5}
    # infinity key: PK_IS_INFINITY; cleared compression bit: BAD_ENCODING; x one off: off the curve, or on it but outside
    # the subgroup (which fast_aggregate_verify reports as VERIFY_FAIL); no keys: VERIFY_FAIL
    allowed = {"inf_key": {6}, "sig_encoding": {1}, "sig_x": {2, 5}, "empty": {5}}
    for t in tuples:
        if t.dead:
            assert M.code[t] in allowed[t.dead], (t.dead, M.code[t])


def test_model_against_the_oracle_pairing(soak, oracle_bls_c):
    """The model's verdict equals aggregate_verify over the r_t-scaled keys and signatures, evaluated by the oracle's
    Miller loop and final exponentiation, for every batch of at most 48 tuples and several seeds."""
    _, M, fam = soak
    seeds = [rc.SEED, rc.ZERO_SEED, hashlib.sha256(b"rlc soak cpu").digest()]
    n = 0
    seen_true = seen_false = 0
    for f in ("A", "B", "C"):
        for c in fam[f]:
            if len(c.batch) > 48:
                continue
            if f == "C" and not (c.name.endswith(" all valid") or c.name.endswith(f" at {len(c.batch) - 1}") or c.name.endswith(" at 0")):
                continue                                   # the sweep's first and last positions stand for the rest
            for sd in dict.fromkeys([s for s, _ in c.runs if s is not None] + seeds):
                want = rc.model(c.batch, sd)
                assert rc.oracle_rlc(oracle_bls_c, M, c.batch, sd) == want, (c.name, sd.hex())
                n += 1
                seen_true += want
                seen_false += not want
    assert n >= 300 and seen_true >= 30 and seen_false >= 100, (n, seen_true, seen_false)
