"""CPU: the reward and penalty deltas oracle (tests/rewards_oracle.py) on every case of tests/rewards_cases.py — its two
formulations agree, each case is in its regime, and applying the deltas pair by pair gives the balances of
epoch_oracle's process_rewards_and_penalties, in both formulations."""
from __future__ import annotations

import numpy as np
import pytest

from oracle import epoch_oracle as eo
from tests import rewards_cases as rc
from tests import rewards_oracle as ro

CASES = rc.cases()


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_case_hits_its_regime(case):
    assert rc.regime_holds(case), case.regime


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_formulations_agree(case):
    before = case.st.validators.tobytes(), case.st.balances.tobytes(), case.st.inactivity_scores.tobytes()
    if case.refusal:
        for form in ("vector", "literal"):
            with pytest.raises(eo.Refused) as ei:
                ro.deltas(case.st, form)
            assert ei.value.kind == case.refusal, form
        return
    v, lit = ro.deltas(case.st, "vector"), ro.deltas(case.st, "literal")
    assert v.shape == lit.shape == (4, 2, len(case.st.validators))
    assert v.dtype == lit.dtype == np.uint64
    assert np.array_equal(v, lit)
    assert not v[3, 0].any()                                           # inactivity rewards are always zero
    assert not v[2, 1].any()                                           # no head penalty
    assert (case.st.validators.tobytes(), case.st.balances.tobytes(), case.st.inactivity_scores.tobytes()) == before


@pytest.mark.parametrize("case", [c for c in CASES if not c.refusal and eo.current_epoch(c.st) > 0], ids=lambda c: c.name)
@pytest.mark.parametrize("form", ["vector", "literal"])
def test_applied_deltas_are_process_rewards_and_penalties(case, form):
    post, code = eo.process_epoch(case.st, "rewards_and_penalties", form)
    assert code == 0
    assert np.array_equal(ro.apply(case.st.balances, ro.deltas(case.st, form)), post.balances.astype(np.uint64))


def test_genesis_reads_current_participation():
    """At epoch 0 the deltas follow current_epoch_participation; previous_epoch_participation does not enter."""
    st = next(c.st for c in CASES if c.name == "genesis")
    d = ro.deltas(st)
    other = eo.clone(st)
    other.previous_epoch_participation[:] = 7
    assert np.array_equal(ro.deltas(other), d)
    other.current_epoch_participation[:] = 0
    assert not np.array_equal(ro.deltas(other), d)


def test_leak_pays_no_flag_rewards():
    for name in ("leak", "leak_delay_wraps", "minimal_leak"):
        d = ro.deltas(next(c.st for c in CASES if c.name == name))
        assert not d[:, 0].any() and d[:3, 1].any(), name


def test_bad_lengths_refused():
    st = rc.base(10, 1000, seed=150)
    st.inactivity_scores = st.inactivity_scores[:9].copy()
    for form in ("vector", "literal"):
        with pytest.raises(eo.Refused) as ei:
            ro.deltas(st, form)
        assert ei.value.kind == "bad_arg"
