"""CPU checks of the process_epoch oracle (oracle/epoch_oracle.py): its literal and vectorised formulations give identical
post-states for every seeded case (tests/epoch_cases.py), with all sub-steps and with each one alone, and every case hits
the regime it was built for."""
from __future__ import annotations

import numpy as np
import pytest

from ethereum_consensus_b200 import state as S
from oracle import epoch_oracle as eo
from tests import epoch_cases as ec

CASES = ec.cases()
MASKS = [("all", eo.ALL)] + [(name, bit) for name, bit in eo.STEP.items()]


def run(st, steps, formulation):
    try:
        post, code = eo.process_epoch(st, steps, formulation)
        return S.serialize(post).tobytes(), code
    except eo.Refused as r:
        return "refused", r.kind


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_formulations_agree(case):
    before = S.serialize(case.st).tobytes()
    for name, m in MASKS:
        assert run(case.st, m, "literal") == run(case.st, m, "vector"), name
    assert S.serialize(case.st).tobytes() == before   # the input is never changed


def _after_jf(st):
    post, _ = eo.process_epoch(st, "justification_and_finalization")
    return post


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_case_hits_regime(case):
    st, r = case.st, case.regime
    cur = eo.current_epoch(st)
    v = eo._Vector(eo.clone(st))
    if r.startswith("grid:"):
        GRID_SHAPES[r[5:]](ec.grid(st), st)
        if not case.refusal:
            return
    if case.refusal:
        with pytest.raises(eo.Refused) as ei:
            eo.process_epoch(st, eo.ALL)
        assert ei.value.kind == case.refusal
        return
    post, code = eo.process_epoch(st, eo.ALL)
    if r in ("epoch0", "epoch1"):
        assert cur == int(r[-1])
    elif r.startswith("finality"):
        rule = int(r[-1])
        old = st.fixed["previous_justified_checkpoint" if rule <= 2 else "current_justified_checkpoint"]
        assert _after_jf(st).fixed["finalized_checkpoint"] == old != st.fixed["finalized_checkpoint"]
    elif r == "leak":
        assert eo.is_in_inactivity_leak(_after_jf(st))
    elif r == "recovery":
        assert not eo.is_in_inactivity_leak(_after_jf(st))
        after, _ = eo.process_epoch(st, "inactivity_updates")
        assert (after.inactivity_scores.astype(np.int64) < st.inactivity_scores.astype(np.int64) - 1).any()
    elif r == "all_participating":
        assert (st.previous_epoch_participation == 7).all()
    elif r == "none_participating":
        assert (st.previous_epoch_participation == 0).all() and (st.current_epoch_participation == 0).all()
    elif r.startswith("slashings"):
        total = v.total_active()
        s = int(st.slashings.astype(object).sum()) * eo.PROPORTIONAL_SLASHING_MULTIPLIER_BELLATRIX
        assert (s >= total) == (r == "slashings_capped")
        after, _ = eo.process_epoch(st, "slashings")
        assert (after.balances < st.balances).sum() == 12
    elif r.startswith("eject"):
        e0, c0, L = v.exit_queue()
        act_exit = eo.compute_activation_exit_epoch(cur)
        real = st.validators["exit_epoch"][st.validators["exit_epoch"] != ec.FAR]
        n_eject = int((v.active(cur) & (st.validators["effective_balance"] <= eo.EJECTION_BALANCE)
                       & (st.validators["exit_epoch"] == ec.FAR)).sum())
        assert n_eject > L
        want = {"eject_below": int(real.max()) < act_exit, "eject_at": int(real.max()) == act_exit and 0 < c0 < L,
                "eject_above": int(real.max()) > act_exit and c0 < L, "eject_c0_ge_L": c0 >= L}[r]
        assert want, (e0, c0, L)
    elif r == "activation_queue":
        fin = int.from_bytes(st.fixed["finalized_checkpoint"][:8], "little")
        vv = st.validators
        q = (vv["activation_eligibility_epoch"] <= fin) & (vv["activation_epoch"] == ec.FAR)
        limit = min(eo.PRESET[st.preset]["MAX_PER_EPOCH_ACTIVATION_CHURN_LIMIT"], v.exit_queue()[2])
        assert q.sum() > limit
        assert ((vv["activation_eligibility_epoch"] > fin) & (vv["activation_epoch"] == ec.FAR)).any() or st.preset == "minimal"
        el = np.sort(vv["activation_eligibility_epoch"][q])[:limit + 1]
        assert len(set(el.tolist())) < len(el)   # ties at the cut
        activated = (post.validators["activation_epoch"] != vv["activation_epoch"]).sum()
        assert activated == limit
    elif r == "hysteresis":
        after, _ = eo.process_epoch(st, "effective_balance_updates")
        changed = after.validators["effective_balance"] != st.validators["effective_balance"]
        d = st.balances.astype(np.int64) - st.validators["effective_balance"].astype(np.int64)
        assert (changed == ((d < -250_000_000) | (d > 1_250_000_000))).all()
        assert (d == -250_000_000).any() and (d == 1_250_000_000).any()
    elif r == "saturate":
        assert (post.balances == 0).any() and not (st.balances == 0).all()
    elif r == "above_max":
        assert (post.validators["effective_balance"] == eo.MAX_EFFECTIVE_BALANCE).all()
        assert (st.balances > eo.MAX_EFFECTIVE_BALANCE + 2 * eo.INC).all()
    elif r == "wrapping":
        eb = st.validators["effective_balance"].astype(object)
        assert any(int(a) * int(b) > eo.U64 for a, b in zip(eb, st.inactivity_scores))
        after, _ = eo.process_epoch(st, "rewards_and_penalties")
        assert (after.balances[:20] < 10**12).any()   # an increase wrapped past 2^64
    elif r == "one_validator":
        assert len(st.validators) == 1
    elif r == "none_active_previous":
        assert not v.active(cur - 1).any() and v.active(cur).all()
    elif r == "minimal":
        assert st.preset == "minimal"
    elif r == "boundaries":
        assert code == 0
        assert len(post.eth1_data_votes) == 0 < len(st.eth1_data_votes)
        assert len(post.historical_summaries) == len(st.historical_summaries) + 1
        assert post.current_sync_committee == st.next_sync_committee != post.next_sync_committee
    elif r == "randao_wrap":
        assert code == 0 and (cur + 1) % eo.PRESET[st.preset]["EPOCHS_PER_HISTORICAL_VECTOR"] == 0
        assert (post.randao_mixes[0] == st.randao_mixes[-1]).all()
    elif r == "eth1_boundary":
        assert len(post.eth1_data_votes) == 0 and len(post.historical_summaries) == len(st.historical_summaries)
    elif r == "aggregation_fails":
        assert code != 0
        assert post.current_sync_committee == st.current_sync_committee
        assert len(post.eth1_data_votes) == 0 and len(post.historical_summaries) == len(st.historical_summaries) + 1
        assert (post.balances != st.balances).any()
    else:
        raise AssertionError(r)


def _step_at_cta_edges(g):
    """The ranks where the closed form's exit epoch steps up whose two ejections lie in different CTAs."""
    return [k for k in g.ranks_cross() if g.cta(g.eject[k - 1]) != g.cta(g.eject[k])]


def _head(g, c0, from_largest_exit):
    assert g.c0 == c0 == len(g.head) and 0 < c0 < g.L
    assert (g.e0 > g.act_exit) == from_largest_exit and g.e0 >= g.act_exit
    assert _step_at_cta_edges(g)


def _overflow_only_across_ctas(g, k):
    whole, cta, _ = g.overflow(k)
    assert whole and not cta


def _refused_under(st, bits):
    for name, m in MASKS:
        try:
            eo.process_epoch(st, m)
            refused = False
        except eo.Refused as r:
            assert r.kind == "limit"
            refused = True
        assert refused == bool(m & bits), name


def _shape_changed(g, want):
    assert g.pushes == want
    assert len(g.winners) == 1   # the activated record also changes its effective balance: two pushes


def _head_c0_3_warps(g, st):
    _head(g, 3, True)
    assert len(set(g.cta(g.head))) == 1 < len(set(g.warp(g.head)))
    assert g.eject[_step_at_cta_edges(g)[0]] % ec.THREADS == 0


def _head_c0_2_first_last_cta(g, st):
    _head(g, 2, False)
    assert set(g.cta(g.head)) == {0, g.nb - 1}


def _head_c0_1_ragged(g, st):
    _head(g, 1, True)
    assert g.n % ec.THREADS and g.head.tolist() == [g.n - 1]


def _head_c0_17_minimal(g, st):
    _head(g, g.L - 1, True)
    assert st.preset == "minimal" and set(g.cta(g.head)) == set(range(g.nb))
    assert len(_step_at_cta_edges(g)) >= 2


def _eject_lanes_threads(g, st):
    assert {0, 31} <= set(g.lane(g.eject)) and {0, ec.THREADS - 1} <= set(g.eject % ec.THREADS)
    assert len(g.eject) > g.L and g.c0 == 0 and len(set(g.cta(g.eject))) >= 3


def _eject_ragged_last_cta(g, st):
    assert g.n % ec.THREADS and set(g.cta(g.eject)) == {g.nb - 1} and g.c0 == 1
    assert g.eject[0] % ec.THREADS == 0 and g.eject[-1] == g.n - 1
    assert len(g.ranks_cross()) and not _step_at_cta_edges(g)


def _eject_one_per_cta(g, st):
    _head(g, g.L - 2, True)
    assert np.bincount(g.cta(g.eject), minlength=g.nb).tolist() == [1] * g.nb


def _sum_2p64_across_ctas(g, st):
    _overflow_only_across_ctas(g, 0)
    assert sum(g.sums[0]) == 1 << 64


def _sum_2p64_minus_1_across_ctas(g, st):
    assert sum(g.sums[0]) == ec.U64 and not g.overflow(0)[0] and g.pushes > 0
    eb = st.validators["effective_balance"]
    assert any(int(e) * int(s) > ec.U64 for e, s in zip(eb, st.inactivity_scores))   # the inactivity penalty wraps


def _overflow_previous_only(g, st):
    assert [g.overflow(k)[0] for k in range(5)] == [False, True, True, True, False]
    for k in (1, 2, 3):
        _overflow_only_across_ctas(g, k)
    _refused_under(st, eo.STEP["justification_and_finalization"] | eo.STEP["rewards_and_penalties"])


def _activation_many_in_one_cta(g, st):
    assert g.offered.max() > g.limit == len(g.winners)
    assert set(g.cta(g.winners)) == {int(g.offered.argmax())}


def _activation_last_cta_only(g, st):
    assert g.n % ec.THREADS and set(g.cta(g.winners)) == {g.nb - 1} and len(g.winners) == g.limit
    assert g.offered[:-1].sum() > 0 and st.validators["activation_epoch"][g.n - 1] == ec.FAR


def _activation_short_queue(g, st):
    assert 0 < len(g.winners) == g.offered.sum() < g.limit and len(set(g.cta(g.winners))) > 1


def _ties_across_ctas(g, st):
    vv = st.validators
    fin = int.from_bytes(st.fixed["finalized_checkpoint"][:8], "little")
    q = np.nonzero((vv["activation_eligibility_epoch"] <= fin) & (vv["activation_epoch"] == ec.FAR))[0]
    last = vv["activation_eligibility_epoch"][g.winners].max()
    tied = q[vv["activation_eligibility_epoch"][q] == last]
    losers = np.setdiff1d(tied, g.winners)
    assert len(g.winners) == g.limit and len(losers) and len(set(g.cta(tied))) >= 3
    assert losers.min() > g.winners.max() and len(set(g.cta(g.winners))) > 1


GRID_SHAPES = {
    "head_c0_3_warps": _head_c0_3_warps,
    "head_c0_2_first_last_cta": _head_c0_2_first_last_cta,
    "head_c0_1_ragged": _head_c0_1_ragged,
    "head_c0_17_minimal": _head_c0_17_minimal,
    "eject_lanes_threads": _eject_lanes_threads,
    "eject_ragged_last_cta": _eject_ragged_last_cta,
    "eject_one_per_cta": _eject_one_per_cta,
    "sum_2p64_across_ctas": _sum_2p64_across_ctas,
    "sum_2p64_minus_1_across_ctas": _sum_2p64_minus_1_across_ctas,
    "overflow_previous_only": _overflow_previous_only,
    "activation_many_in_one_cta": _activation_many_in_one_cta,
    "activation_ties_across_ctas": _ties_across_ctas,
    "activation_last_cta_only": _activation_last_cta_only,
    "activation_short_queue": _activation_short_queue,
    "changed_4096": lambda g, st: _shape_changed(g, g.threshold),
    "changed_4097": lambda g, st: _shape_changed(g, g.threshold + 1),
}


def test_refusal_kinds_cover_every_rule():
    kinds = {c.name: c.refusal for c in CASES if c.refusal}
    assert set(kinds) == {"refuse_block_root", "refuse_total_overflow", "refuse_withdrawable_overflow", "refuse_no_active_next",
                          "sum_2p64_across_ctas", "overflow_previous_only"}
    with pytest.raises(eo.Refused):
        eo.process_epoch(CASES[0].st, 1 << 12)
