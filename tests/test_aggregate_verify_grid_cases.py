"""CPU: the aggregate_verify batches of tests/aggregate_verify_grid_cases.py land on the chunk, lane, level count, pieces,
warp and team size they were built for, at vm_cta 32, 64 and 128 and vm_team16_max 0, 2 048 and 2^30; every named edge
occurs; the expected codes hold in the C oracle (closed forms on a sample, every crafted small tuple) and the Python
oracle agrees with it on the infinity-signature tuples.  tests/test_aggregate_verify_grid_gpu.py runs them on the device."""
from __future__ import annotations

import random

import pytest

from oracle import bls_oracle as bo
from tests import aggregate_verify_cases as av
from tests import aggregate_verify_grid_cases as g

CONFIGS = [(cta, tm) for cta in g.VM_CTAS for tm in g.TEAM16_MAXES]


@pytest.fixture(scope="module")
def O(oracle_bls_c):
    return g.bind(oracle_bls_c)


def _cases(section):
    return [c for c in g.all_cases() if c.section == section]


def _check_claims(case, L: g.Layout):
    """The shape `case` was built for, under the layout's knobs; returns the list of claims that hold."""
    cl, held = case.claim, []
    if "start" in cl:
        for t, lane in cl["start"].items():
            assert L.start_lane(t) == lane and L.pairs[t] == cl["c"], (case.name, t)
        held.append("start")
        sb = cl["shape_before"]
        shapes = [t for t in range(sb) if case.specs[t].pairs == 0]
        assert shapes and all(case.specs[t].msgs or case.specs[t].n for t in shapes[:1])
        # without the shape failures the target starts at the same pair
        rest = [x for x in case.specs if x.pairs or x is case.specs[sb]]
        assert g.Layout(rest).poff[rest.index(case.specs[sb])] == L.poff[sb], case.name
    if "levels" in cl:
        assert len(L.levels) == cl["levels"], (case.name, len(L.levels))
        held.append("levels")
    if "target" in cl:
        t = cl["target"]
        assert L.start_lane(t) == cl["lane"] and L.pairs[t] == cl["c"], case.name
        if cl.get("bound") == "smallest" and cl["c"] > 2:    # one value less: one level less
            fewer = list(case.specs)
            fewer[t] = g.Spec("valid", cl["c"] - 2)
            assert len(g.Layout(fewer).levels) == cl["levels"] - 1, case.name
        if cl.get("bound") == "largest":
            more = list(case.specs)
            more[t] = g.Spec("valid", cl["c"])
            assert len(g.Layout(more).levels) == cl["levels"] + 1, case.name
        for s in range(t + 1, L.T):    # the short tuples behind it: at most two pieces at level 0, yet every level
            if L.pairs[s]:
                assert L.pieces(s)[1] <= 2 if len(L.levels) else True
    if "n_pairs" in cl:
        assert L.n_pairs == cl["n_pairs"], case.name
    if "miller_team" in cl and L.team16_max == g.TEAM16_MAX:
        assert L.miller_team == cl["miller_team"], case.name
    if "final_team" in cl and "final_lone" not in cl and L.team16_max == g.TEAM16_MAX:
        assert L.final_team == cl["final_team"], case.name
    if "T" in cl:
        assert L.T == cl["T"], case.name
    if "team" in cl and L.miller_team == cl["team"]:
        warps = L.miller_warps()
        w = L.miller_per_warp
        for i, pos in cl["lone"].items():
            runs, live = warps[i // w]
            assert i % w == pos and runs == {pos}, (case.name, i, runs)
        for i in cl["trivial_alone"]:
            runs, live = warps[i // w]
            assert i % w == 0 and runs == set() and live == {0} and L.specs[L.pair_tuple[i]].trivial_last, (case.name, i)
            assert i == L.poff[L.pair_tuple[i] + 1] - 1
        dead = [k for k, (_, live) in enumerate(warps) if not live]
        lives = [k for k, (_, live) in enumerate(warps) if live]
        assert dead[0] == 0 and dead[-1] == len(warps) - 1 and any(lives[0] < k < lives[-1] for k in dead), case.name
        n_last, live_last, cap = L.last_miller_cta()
        assert 0 < n_last < cap and live_last == 0, (case.name, L.vm_cta, n_last, cap)
        held.append("warps")
    if "final_lone" in cl and L.final_team == cl["final_team"]:
        w = L.final_per_warp
        fw = L.final_warps()
        for t, pos in cl["final_lone"].items():
            assert t % w == pos and fw[t // w] == {pos}, (case.name, t)
        assert len({t % w for t in cl["final_lone"]}) == w
        assert not fw[0] and not fw[-1] and not fw[-2] and L.T % w == 1
        assert any(not fw[k] and fw[k - 1] and fw[k + 1] for k in range(1, len(fw) - 1))
        held.append("final_warps")
    if "first_bad" in cl:
        for t, p in cl["first_bad"].items():
            sp = case.specs[t]
            assert min(sp.bad)[0] == p and p >= 32 or len({q % 32 for q, _ in sp.bad}) == 1, (case.name, t)
        held.append("keys")
    return held


@pytest.mark.parametrize("cta,team16_max", CONFIGS)
def test_every_case_lands_where_it_was_built(cta, team16_max):
    seen = set()
    for case in g.all_cases():
        L = g.layout(case, cta, team16_max)
        seen.update(_check_claims(case, L))
        assert L.launches == g.layout(case, cta, team16_max).launches
        P = g.layout(g.poison(case), cta, team16_max)
        assert P.T >= L.T and P.n_pairs >= L.n_pairs and len(P.levels) % 2 == len(L.levels) % 2, case.name
        assert all(x.want == g.SUCCESS for x in g.poison(case).specs)
    assert {"start", "levels", "keys"} <= seen
    if team16_max == 0:
        assert {"warps", "final_warps"} <= seen
    if team16_max == 1 << 30:
        assert "warps" in seen and "final_warps" in seen


def test_alignment_edges():
    got = {}
    for case in _cases("align"):
        L = g.layout(case)
        for t in case.claim["start"]:
            p = L.pieces(t)
            got.setdefault("pieces", set()).add(p[1] if len(p) > 1 else None)
            lo, hi = L.poff[t], L.poff[t + 1]
            if hi % 32 == 0 and lo // 32 == (hi - 1) // 32:
                got.setdefault("last lane 31, first lane 0", set()).add(case.claim["c"])
            if L.crosses_cta(t):
                got.setdefault("64-value edge", set()).add(case.claim["c"])
        kinds = {x.kind for x in case.specs[:case.claim["start"].__iter__().__next__() + 40]}
        got.setdefault("pad kinds", set()).update(k for k in kinds if k in ("badkey", "badsig", "nig", "valid"))
    assert {1, 2, 3} <= got["pieces"]
    assert {32} <= got["last lane 31, first lane 0"]
    assert {2, 3, 31, 32, 33} <= got["64-value edge"]
    assert got["pad kinds"] == {"badkey", "badsig", "nig", "valid"}
    # every pair count at every start lane, valid and failing
    cover = {(c.claim["c"], s, c.specs[t].kind) for c in _cases("align") for t, s in c.claim["start"].items()}
    assert cover == {(c, s, k) for c in g.ALIGN_C for s in g.ALIGN_LANES for k in ("valid", "fail")}


def test_depth_edges():
    cs = _cases("depth")
    got = {(c.claim["levels"], c.claim["lane"], c.claim.get("bound")): c.claim["c"] for c in cs}
    assert got[(1, 0, "smallest")] == 3 and got[(1, 0, "largest")] == 64
    assert got[(2, 0, "smallest")] == 65 and got[(2, 0, "largest")] == 2048
    assert got[(3, 0, "smallest")] == 2049 and got[(3, 0, "largest")] == 65536
    assert got[(4, 0, "smallest")] == 65537 and (4, 0, "largest") not in got
    assert got[(1, 31, "smallest")] == 2 and all((L, 31, "smallest") in got for L in (1, 2, 3, 4))
    assert any(c.claim["c"] == 32769 for c in cs)
    for c in cs:    # the short tuples behind the long one go through levels they do not need
        L = g.layout(c)
        assert all(L.pieces(s)[1] <= 2 for s in range(c.claim["target"] + 1, L.T) if L.pairs[s])


def test_skip_rule_and_launches():
    a, b, shapes = _cases("skip")
    La, Lb, Ls = g.layout(a), g.layout(b), g.layout(shapes)
    assert set(La.pairs) == {0, 2} and len(La.levels) == 0
    assert len(Lb.levels) == 1 and Lb.pairs[-1] == 3
    assert Ls.n_pairs == 0 and Ls.levels == []
    # K1, K3, K4 x 2, K2, pair operands, Miller, levels, final
    assert La.launches == 1 + 1 + 2 + 1 + 1 + 1 + 0 + 1 and Lb.launches == La.launches + 1
    assert Ls.launches == 1 + 1 + 2 + 1 + 1 + 0 + 0 + 1
    assert g.layout(a, registry=True).launches == La.launches - 1
    # with the rule `len == 2` only, the first batch would plan a level: only its launch count shows it
    assert any(p == 0 for p in La.pairs)


def test_team_switches():
    cs = {c.name: c for c in _cases("switch")}
    for name, c in cs.items():
        L = g.layout(c)
        if "n_pairs" in c.claim:
            assert L.n_pairs == c.claim["n_pairs"] and L.miller_team == c.claim["miller_team"], name
        if "final_team" in c.claim:
            assert L.T == c.claim["T"] and L.final_team == c.claim["final_team"], name
    odd = g.layout(cs["T = 2 049, mostly shape failures"])
    assert odd.n_pairs < 2048 and odd.miller_team == 16 and odd.final_team == 8
    # forcing either team size moves both
    for tm, team in ((0, 8), (1 << 30, 16)):
        for c in cs.values():
            L = g.layout(c, team16_max=tm)
            assert L.miller_team == team and (L.final_team == team)


def test_vm_cta_halving_never_binds_with_the_compiled_programs():
    for team in (8, 16):
        for cta in g.VM_CTAS:
            assert g.cta_threads(team, cta, False) == cta and g.cta_threads(team, cta, True) == cta
    assert g.vm_slots()[8][0] > 12 and g.vm_slots()[16][1] > 12


def test_shifted_padding_moves_a_case_off_its_edge():
    case = next(c for c in _cases("align") if c.claim["c"] == 33)
    specs = list(case.specs)
    specs[0] = g.Spec(specs[0].kind, specs[0].n + 1, bad=specs[0].bad, k=specs[0].k) if specs[0].pairs else specs[0]
    moved = g.Case(case.name, case.section, specs, case.claim)
    with pytest.raises(AssertionError):
        _check_claims(moved, g.layout(moved))


# ------------------------------------------------------------------------------------------------ oracles
def _small_specs():
    """Every distinct tuple of at most 64 pairs (or a shape failure) among the cases, and each one's first use."""
    out = {}
    for case in g.all_cases():
        for sp in case.specs:
            if sp.pairs <= 64 and sp not in out:
                out[sp] = case.name
    return out


def test_crafted_small_tuples_get_the_c_oracle_code(O):
    small = [sp for sp in _small_specs() if sp.kind not in ("valid", "fail") or not sp.shape_ok]
    mats = g.materials(small)
    got = av.oracle_codes(O, mats)
    bad = [(sp, w, c) for sp, m, c in zip(small, mats, got) for w in [sp.want] if c != w]
    assert not bad, bad[:5]
    assert {sp.kind for sp in small} >= {"badkey", "badsig", "noc", "nig", "triv2", "triv3", "inf1", "trivfail", "valid"}


def test_closed_form_tuples_pass_the_c_oracle(O):
    rnd = random.Random(3)
    sizes = [1, 2, 3, 30, 32, 63, 64, g.PERIOD - 1, g.PERIOD, g.PERIOD + 3]
    specs = [g.Spec("valid", n, k=rnd.randrange(40)) for n in sizes] + [g.Spec("fail", n, k=2) for n in (1, 33)]
    specs.append(g.Spec("valid", 1, k=2048))
    mats = g.materials(specs)
    assert av.oracle_codes(O, mats) == [sp.want for sp in specs]
    # consecutive k differ by A_n: tuple k + 1's signature is tuple k's plus the message sum
    n = 5
    A = g._A_sig0(n)[0]
    assert g.valid_sig(n, 3) == g.ac.G2.add(g.valid_sig(n, 2), A)


def test_python_and_c_oracles_agree_on_infinity_signature_tuples(O):
    specs = [g.Spec("triv2", 2, k=k) for k in (1, 21)] + [g.Spec("triv3", 3, k=23), g.Spec("inf1", 1, k=24),
                                                          g.Spec("trivfail", 2, k=25)]
    mats = g.materials(specs)
    c_codes = av.oracle_codes(O, mats)
    py_codes = [bo.aggregate_verify(m["pks"], m["msgs"], m["sig"]) for m in mats]
    assert c_codes == py_codes == [g.SUCCESS, g.SUCCESS, g.SUCCESS, g.VERIFY_FAIL, g.VERIFY_FAIL]
    # the keys really cancel and the signature is the infinity encoding
    for m in mats[:3]:
        acc = None
        for k in m["pks"]:
            acc = g.ac.G1.add(acc, bo.g1_uncompress(k)[1])
        assert acc is None and m["sig"] == g.INF_SIG
