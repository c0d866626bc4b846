"""CPU oracle for the reward and penalty deltas — test infrastructure for ethereum_consensus_b200.epoch.deltas, over a
`state.SynthState` (builds on oracle/epoch_oracle.py's two formulations of process_epoch).

`deltas(st, formulation)` is what the spec-test `rewards` handler compares: get_flag_index_deltas (altair/helpers.rs:265)
for flags 0, 1, 2 and get_inactivity_penalty_deltas (bellatrix/helpers.rs:13) on the state as it is, as a uint64 array
of shape (4, 2, n) ([k, 0] rewards, [k, 1] penalties):
  * "literal": the oracle's loop-for-loop delta functions (membership sets, Python ints wrapped to u64);
  * "vector":  numpy over whole columns, the same formulas as the oracle's vectorised process_rewards_and_penalties.
`apply(balances, d)` folds them into balances as process_rewards_and_penalties does: each pair in turn, the reward
wrapping and the penalty saturating at zero.  Both functions leave their inputs untouched; an overflowing
get_total_balance raises epoch_oracle.Refused("limit").
"""
from __future__ import annotations

import numpy as np

from oracle import epoch_oracle as eo


def _check_lengths(st) -> None:
    n = len(st.validators)
    if any(len(x) != n for x in (st.balances, st.previous_epoch_participation, st.current_epoch_participation,
                                 st.inactivity_scores)):
        raise eo.Refused("bad_arg", "the five big lists differ in length")


def _literal(st) -> np.ndarray:
    lit = eo._Literal(st)
    pairs = [lit.flag_index_deltas(f) for f in range(3)] + [lit.inactivity_penalty_deltas()]
    return np.array(pairs, dtype=np.uint64).reshape(4, 2, len(st.validators))


def _vector(st) -> np.ndarray:
    v = eo._Vector(st)
    n = len(st.validators)
    out = np.zeros((4, 2, n), np.uint64)
    eb = v._cols()[0]
    el = v.eligible()
    prev = v.prev()
    total = v.total_active()
    active_inc = total // eo.INC
    bpi = np.uint64(eo.INC * eo.BASE_REWARD_FACTOR // eo.integer_sqrt(total))
    leak = eo.is_in_inactivity_leak(st)
    with np.errstate(over="ignore"):
        base = eb // np.uint64(eo.INC) * bpi
        for f in range(3):
            part = v.participating(f, prev)
            inc = np.uint64(v.total(eb, part) // eo.INC)
            w = np.uint64(eo.PARTICIPATION_FLAG_WEIGHTS[f])
            if not leak:
                out[f, 0] = np.where(el & part, base * w * inc // np.uint64(active_inc * eo.WEIGHT_DENOMINATOR), np.uint64(0))
            if f != eo.TIMELY_HEAD_FLAG_INDEX:
                out[f, 1] = np.where(el & ~part, base * w // np.uint64(eo.WEIGHT_DENOMINATOR), np.uint64(0))
        tgt = v.participating(eo.TIMELY_TARGET_FLAG_INDEX, prev)
        s = st.inactivity_scores.astype(np.uint64)
        den = np.uint64(eo.INACTIVITY_SCORE_BIAS * eo.INACTIVITY_PENALTY_QUOTIENT_BELLATRIX)
        out[3, 1] = np.where(el & ~tgt, eb * s // den, np.uint64(0))
    return out


def deltas(st, formulation: str = "vector") -> np.ndarray:
    _check_lengths(st)
    return {"literal": _literal, "vector": _vector}[formulation](st)


def apply(balances, d: np.ndarray) -> np.ndarray:
    bal = np.asarray(balances).astype(np.uint64)
    with np.errstate(over="ignore"):
        for k in range(4):
            bal = bal + d[k, 0]
            bal = np.where(d[k, 1] > bal, np.uint64(0), bal - np.minimum(d[k, 1], bal))
    return bal
