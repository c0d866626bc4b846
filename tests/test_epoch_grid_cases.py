"""CPU checks of the large process_epoch states (tests/epoch_grid_cases.py): each hits the launch-shape edge it was built
for, from the vectorised oracle's intermediates; a minimal-preset replica of each exit-queue shape gives identical
post-states under both oracle formulations."""
from __future__ import annotations

import numpy as np
import pytest

from ethereum_consensus_b200 import state as S
from oracle import epoch_oracle as eo
from tests import epoch_cases as ec
from tests import epoch_grid_cases as gc

STATES = gc.states()
T = ec.THREADS


def _edges(g):
    assert 0 < g.c0 < g.L == 4 and g.e0 > g.act_exit
    assert g.eject[-1] == g.n - 1 and g.cta(g.eject[-1]) == g.nb - 1           # the last valid thread ejects
    assert 0 < len(g.winners) == g.offered.sum() < g.limit                     # a short queue, at both ends of the list
    assert g.cta(g.winners).min() == 0 and g.winners.max() == g.n - 2
    heads = g.rthread(g.head)
    if g.per == 1:   # holders on both sides of a k_epoch_reduce warp edge (lanes 31 and 32 of the reduce CTA)
        assert set(heads.tolist()) == {31, 32}
    else:            # and on both sides of a range edge, plus the last range
        assert {0, 1} <= set(heads.tolist()) and g.cta(g.head[0]) % g.per == g.per - 1 and g.cta(g.head[1]) % g.per == 0
        starts = [int(g.cta(i)) % g.per == 0 for i in g.eject]
        ends = [int(g.cta(i)) % g.per == g.per - 1 for i in g.eject]
        assert any(starts) and any(ends)
        assert g.nb % g.per and g.nb == ec.REDUCE_THREADS * (g.per - 1) + 1   # ragged ranges: threads past nb / per idle
    steps = g.ranks_cross()
    assert len(steps) and all(g.cta(g.eject[k - 1]) != g.cta(g.eject[k]) for k in steps)


def _range_overflow(g):
    s = g.sums[0]
    assert s[0] + s[1] == 1 << 64 and max(s) <= ec.U64 and g.per == 2 and g.overflow(0) == (True, False, True)
    st = dict((x[0], x[1]) for x in STATES)["range_overflow"]
    with pytest.raises(eo.Refused):   # slashings alone reads the total active balance and nothing else
        eo.process_epoch(st, "slashings")


def _rehash(g, want):
    assert g.threshold == g.n // 16 > ec.REHASH_MIN and g.pushes == want and len(g.winners) == 1


def _limit(g, want):
    assert g.L == g.limit == want
    assert 9 <= g.offered.max() <= 40 and g.cta(gc.WIDE[0]) >= 1024
    assert len(g.winners) == want and (g.cta(g.winners) >= 1024).sum() == 5 and (g.cta(g.winners) < 1024).any()
    assert g.offered[g.cta(gc.WIDE[0])] == len(gc.WIDE) > g.limit


SHAPES = {"range_overflow": _range_overflow, "rehash_8192": lambda g: _rehash(g, g.threshold),
          "rehash_8193": lambda g: _rehash(g, g.threshold + 1), "limit_7": lambda g: _limit(g, 7),
          "limit_8": lambda g: _limit(g, 8)}


@pytest.mark.parametrize("name,st,refused", STATES, ids=[s[0] for s in STATES])
def test_grid_state_shape(name, st, refused):
    g = ec.grid(st)
    SHAPES.get(name, _edges)(g)
    assert (g.pushes < 0) == refused
    if not refused:
        assert g.per == -(-g.nb // ec.REDUCE_THREADS) and g.nb == -(-len(st.validators) // T)


def test_grid_sizes():
    n = {name: len(st.validators) for name, st, _ in STATES}
    assert [n[f"edges_{k}"] for k in (131071, 131072, 131073, 262145)] == [511 * T + 255, 512 * T, 512 * T + 1, 1024 * T + 1]
    assert n["rehash_8192"] == n["rehash_8193"] == 1 << 17


@pytest.mark.parametrize("name", [s[0] for s in STATES if s[0].startswith("edges")])
def test_replica_formulations_agree(name):
    st = dict((s[0], s[1]) for s in STATES)[name]
    g, r = ec.grid(st), gc.replica(st)
    gr = ec.grid(r)
    assert (gr.e0 - gr.act_exit, gr.c0, gr.L) == (g.e0 - g.act_exit, g.c0, g.L)
    assert sorted(gr.lane(gr.head).tolist()) == sorted(g.lane(g.head).tolist())
    assert len(set(gr.warp(gr.head).tolist())) == len(g.head)
    assert len(gr.eject) >= 3 and len(gr.ranks_cross())
    for m in (eo.ALL, eo.STEP["registry_updates"]):
        lit, _ = eo.process_epoch(r, m, "literal")
        vec, _ = eo.process_epoch(r, m, "vector")
        assert S.serialize(lit).tobytes() == S.serialize(vec).tobytes()
