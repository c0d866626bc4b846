"""Mainnet states too large for the literal oracle, built so that process_epoch's values cross k_epoch_reduce's ranges
(511 / 512 / 513 and 1 025 CTAs), the whole-list re-hash threshold, and the activation churn limit of 7 and 8 with
candidates past CTA 1 023 (csrc/epoch.cu).  Shared by test_epoch_grid_cases.py (CPU: each state hits its shape; a
minimal-preset replica runs through both oracle formulations) and test_epoch_grid_gpu.py (the device against the
vectorised oracle and the C state root)."""
from __future__ import annotations

import numpy as np

from tests import epoch_cases as ec

T = ec.THREADS


def reduce_edges(n: int, seed: int):
    """n = 131 071 / 131 072 / 131 073 / 262 145: the exit-queue head (c0 = 2 or 3 < L = 4) on both sides of a
    k_epoch_reduce warp or range edge and in the last CTA, ejections at range ends and at the last valid thread,
    candidates at both ends of the list."""
    st = ec.base(n, 1000, seed=seed)
    nb = -(-n // T)
    per = -(-nb // ec.REDUCE_THREADS)
    last = n - 1
    if per == 1:
        head = [32 * T - 1, 32 * T]                         # CTAs 31 and 32: reduce lanes 31 and 32, two warps
        ej = [0, 32 * T - 2, 32 * T + 1, last]              # (2 + k) / 4 steps at k = 2: CTA 31 -> 32
    else:
        head = [per * T - 1, per * T, (nb - 2) * T + 5]     # the last CTA of range 0, the first of range 1
        ej = [per * T + 5, (2 * per) * T - 1, 2 * per * T, last]
    ec.exits(st, head, 1008)
    ec.exits(st, [11, 12], 990)
    ec.ejects(st, ej)
    ec.pending(st, [3, last - 1], 990)
    ec.pending(st, [(nb // 2) * T + 31], 991)
    st.fixed["finalized_checkpoint"] = ec._cp(995, b"f")
    return st


def range_overflow():
    """n = 131 073 (per = 2): the effective balances of CTAs 0 and 1, k_epoch_reduce thread 0's range, sum to exactly
    2^64 while each CTA stays below it: only the range fold carries."""
    st = ec.base(131073, 1000, seed=80)
    eb = st.validators["effective_balance"]
    others = 2 * T * int(eb[0]) - 2 * int(eb[0])
    eb[[3, T + 44]] = [1 << 63, (1 << 63) - others]
    return st


def rehash(count: int):
    """n = 2^17: `count` changed records (n / 16 = 8 192 is the threshold) — eligibility set on records with FAR
    eligibility and MAX effective balance, plus one activated record whose effective balance changes too."""
    n = 1 << 17
    st = ec.base(n, 1000, seed=81)
    st.balances[:] = 32 * ec.ETH
    st.validators["activation_eligibility_epoch"][1:count - 1] = ec.FAR
    ec.pending(st, [n - 1], 990)
    st.balances[n - 1] = 40 * ec.ETH
    st.validators["effective_balance"][n - 1] = 30 * ec.ETH
    return st


# the pending validators of the churn-limit states: CTA 1100 offers 30 (five at 984), CTA 2 offers three at 985 with
# lower indices, CTA 1500 two at 986
WIDE = 1100 * T + np.arange(0, 240, 8)
PENDING = np.concatenate([WIDE, [600, 601, 700], 1500 * T + np.array([0, 255])])


def activation_limit(n_active: int):
    """Mainnet with 524 287 or 524 288 active validators: activation churn limit 7 or 8."""
    n = n_active + len(PENDING)
    st = ec.base(n, 1000, seed=82)
    ec.pending(st, PENDING, 985)
    ec.pending(st, WIDE[:5], 984)
    ec.pending(st, PENDING[-2:], 986)
    ec.ejects(st, [10, 1100 * T + 1, n - 1])
    return st


def states():
    """(name, state, process_epoch(ALL) refused)"""
    out = [(f"edges_{n}", reduce_edges(n, 70 + k), False) for k, n in enumerate((131071, 131072, 131073, 262145))]
    out.append(("range_overflow", range_overflow(), True))
    out += [(f"rehash_{c}", rehash(c), False) for c in (8192, 8193)]
    out += [(f"limit_{n - 524280}", activation_limit(n), False) for n in (524287, 524288)]
    return out


def replica(st):
    """A minimal-preset state of 128 validators (L = 4, one CTA) with the same E0, c0 and L as `st`, its exit-queue
    holders and ejections at the same lanes, spread over the four warps: small enough for the literal oracle."""
    g = ec.grid(st)
    r = ec.base(128, 1000, "minimal", seed=90)
    lanes = lambda idx: [32 * (j % 4) + int(i) % 32 for j, i in enumerate(idx)]  # noqa: E731
    head = lanes(g.head)
    ec.exits(r, head, g.e0)
    ec.ejects(r, [i for i in lanes(g.eject) if i not in head])
    return r
