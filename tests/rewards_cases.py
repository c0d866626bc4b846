"""Seeded deneb states for the reward and penalty deltas on the device-resident state (ethereum_consensus_b200.epoch.deltas),
each built for one regime of get_flag_index_deltas / get_inactivity_penalty_deltas.  Built on epoch_cases.py's `base`;
shared by test_rewards_cases.py (CPU: the oracle's two formulations agree, each case hits its regime) and
test_rewards_gpu.py (the device against the oracle)."""
from __future__ import annotations

import numpy as np

from oracle import epoch_oracle as eo
from tests import epoch_cases as ec
from tests.epoch_cases import ETH, U64, Case, base

# k_epoch_reduce folds the per-CTA partials in REDUCE_THREADS ranges of `per` CTAs (epoch_cases.grid)
RANGE_EDGE_SIZES = (ec.THREADS * ec.REDUCE_THREADS,             # 512 CTAs: one per range
                    ec.THREADS * (ec.REDUCE_THREADS + 1),       # 513 CTAs: per = 2, the last range holds one CTA
                    ec.THREADS * 2 * ec.REDUCE_THREADS - 1)     # 1024 CTAs, per = 2, the last one ragged


def _only_flag(st, f: int) -> None:
    """Every validator has flag f and no other at the previous epoch (and the current one, for the genesis epoch)."""
    st.previous_epoch_participation[:] = 1 << f
    st.current_epoch_participation[:] = 1 << f


def _overflow(st, flag: int | None) -> None:
    """get_total_balance overflows in exactly one sum: the total active balance (flag None) or flag `flag`'s unslashed
    participating balance.  Four validators of 2^62 (and 5 more gwei) carry it: for a flag they exit at the current epoch
    (active at the previous epoch only) and hold that flag alone; for the active sum they activate at the current epoch."""
    cur = eo.current_epoch(st)
    big = [10, 11, 200, 201]
    st.validators["effective_balance"][big] = [1 << 62, 1 << 62, 1 << 62, (1 << 62) + 5]
    if flag is None:
        st.validators["activation_epoch"][big] = cur
    else:
        ec.exits(st, big, cur)
        st.previous_epoch_participation[big] = 1 << flag


def cases() -> list:
    out = []
    add = lambda name, st, regime, refusal=None: out.append(Case(name, st, regime, refusal))  # noqa: E731

    add("no_leak", base(300, 1000, seed=101), "no_leak")             # finalized 997: delay 2
    st = base(300, 1000, seed=102)
    st.fixed["finalized_checkpoint"] = ec._cp(990, b"f")             # delay 9 > MIN_EPOCHS_TO_INACTIVITY_PENALTY
    st.inactivity_scores[:] = np.arange(300, dtype=np.uint64) * 7
    add("leak", st, "leak")
    st = base(300, 1000, seed=103)
    st.fixed["finalized_checkpoint"] = ec._cp(1005, b"f")            # finalized after previous: the delay wraps
    add("leak_delay_wraps", st, "leak_wrap")
    st = base(200, 0, seed=104)                                      # previous == current: the current flags count
    st.previous_epoch_participation[:] = 0
    add("genesis", st, "genesis")
    st = base(200, 0, seed=105)
    st.previous_epoch_participation[:] = 7
    st.current_epoch_participation[::3] = 0
    add("genesis_prev_all", st, "genesis")
    add("epoch1", base(200, 1, seed=106), "epoch1")
    st = base(240, 1000, seed=107)                                   # slashed, exited: eligible while prev + 1 < withdrawable
    v = st.validators
    v["slashed"][::4] = 1
    ec.exits(st, np.arange(0, 240, 8), 900)                          # inactive at the previous epoch
    v["withdrawable_epoch"][0:240:16] = 1000                         # prev + 1 == withdrawable: not eligible
    v["withdrawable_epoch"][8:240:16] = 1001                         # prev + 1 < withdrawable: eligible
    st.previous_epoch_participation[::2] = 7
    add("slashed_eligible", st, "slashed_eligible")
    st = base(200, 1000, seed=108)
    st.validators["activation_epoch"][50:120] = 1000                 # active now, not at the previous epoch
    add("active_now_only", st, "active_now_only")
    st = base(256, 1000, seed=109)
    rng = np.random.default_rng(109)
    eb = rng.integers(0, 40 * ETH, 256, dtype=np.uint64)
    eb[::17] = 0
    eb[5::17] = ETH - 1
    st.validators["effective_balance"] = eb
    add("odd_effective_balances", st, "odd_eb")
    st = base(200, 1000, seed=110)
    st.inactivity_scores[:] = (1 << 40) + np.arange(200, dtype=np.uint64) * 12345   # eb * score wraps
    st.previous_epoch_participation[::2] &= np.uint8(5)             # no target flag: the penalty applies
    st.validators["effective_balance"][7] = 1 << 60                 # base reward products wrap
    add("score_wraps", st, "score_wrap")
    st = base(150, 1000, seed=111)
    st.previous_epoch_participation[:] = 7
    add("all_flags", st, "all_flags")
    st = base(150, 1000, seed=112)
    st.previous_epoch_participation[:] = 0
    add("no_flags", st, "no_flags")
    for f in range(3):
        st = base(150, 1000, seed=113 + f)
        _only_flag(st, f)
        add(f"only_flag{f}", st, f"only_flag{f}")
    add("minimal", base(64, 1000, "minimal", seed=116), "minimal")
    st = base(64, 1000, "minimal", seed=117)
    st.fixed["finalized_checkpoint"] = ec._cp(980, b"f")
    add("minimal_leak", st, "leak")
    for n in (0, 1, 255, 256, 257):
        add(f"n{n}", base(n, 1000, seed=120 + n % 7), "size")
    for k, n in enumerate(RANGE_EDGE_SIZES):
        st = base(n, 1000, seed=130 + k)
        v = st.validators
        nb = -(-n // ec.THREADS)
        per = -(-nb // ec.REDUCE_THREADS)
        edges = np.array([b * ec.THREADS for b in range(0, nb, per)] + [min(n, (b + per) * ec.THREADS) - 1 for b in range(0, nb, per)])
        v["effective_balance"][edges] = 31 * ETH + edges.astype(np.uint64) % ETH   # distinct balances at each range's ends
        st.previous_epoch_participation[edges] = (edges % 8).astype(np.uint8)
        add(f"reduce_edges_{n}", st, "size")
    st = base(600, 1000, seed=140)                                   # the active sum at exactly 2^64 - 1: not refused
    eb = st.validators["effective_balance"]
    rest = int(eb.astype(object).sum()) - 2 * int(eb[0])
    eb[[3, 400]] = [1 << 63, U64 - rest - (1 << 63)]
    add("sum_2p64_minus_1", st, "no_overflow")
    add("overflow_active", _with(base(300, 1000, seed=141), None), "refusal", "limit")
    for f, name in enumerate(("source", "target", "head")):
        add(f"overflow_{name}", _with(base(300, 1000, seed=142 + f), f), "refusal", "limit")
    return out


def _with(st, flag):
    _overflow(st, flag)
    return st


def sums(st) -> list:
    """The four sums get_total_balance takes (total active, then flags 0..2), before the max with one increment."""
    v = eo._Vector(st)
    eb = v._cols()[0].astype(object)
    masks = [v.active(v.cur())] + [v.participating(f, v.prev()) for f in range(3)]
    return [int(eb[m].sum()) for m in masks]


def regime_holds(c: Case) -> bool:
    """Whether the case's state is in the regime its name promises."""
    st = c.st
    cur = eo.current_epoch(st)
    prev = cur - 1 if cur else 0
    n = len(st.validators)
    vv = eo._Vector(st)
    v = st.validators
    leak = eo.is_in_inactivity_leak(st)
    fin = int.from_bytes(st.fixed["finalized_checkpoint"][:8], "little")
    s = sums(st)
    part = [vv.participating(f, prev) for f in range(3)]
    el = vv.eligible()
    if c.regime == "refusal":
        return sum(x > U64 for x in s) == 1
    if any(x > U64 for x in s):
        return False
    r = c.regime
    if r == "no_leak":
        return not leak and cur > 1
    if r == "leak":
        return leak and fin < prev
    if r == "leak_wrap":
        return leak and fin > prev
    if r == "genesis":
        return cur == 0 and not np.array_equal(st.previous_epoch_participation, st.current_epoch_participation)
    if r == "epoch1":
        return cur == 1 and prev == 0
    if r == "slashed_eligible":
        slashed = v["slashed"] != 0
        ex = slashed & ~vv.active(prev)
        return bool((ex & el).any() and (ex & ~el).any())
    if r == "active_now_only":
        now = vv.active(cur) & ~vv.active(prev)
        return bool(now.any() and not el[now].any())
    if r == "odd_eb":
        eb = v["effective_balance"]
        return bool((eb == 0).any() and (eb % ETH != 0).any())
    if r == "score_wrap":
        eb = v["effective_balance"].astype(object)
        sc = st.inactivity_scores.astype(object)
        return any(eb[i] * sc[i] > U64 and el[i] and not part[1][i] for i in range(n))
    if r == "all_flags":
        return all(p[el].all() for p in part)
    if r == "no_flags":
        return not any(p.any() for p in part)
    if r.startswith("only_flag"):
        f = int(r[-1])
        return bool(part[f][el].all()) and not any(part[g].any() for g in range(3) if g != f)
    if r == "minimal":
        return st.preset == "minimal" and not leak
    if r == "size":
        return n in (0, 1, 255, 256, 257) + RANGE_EDGE_SIZES
    if r == "no_overflow":
        return s[0] == U64
    raise KeyError(r)
