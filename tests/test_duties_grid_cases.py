"""CPU checks of the launch-shape duty cases (tests/duties_grid_cases.py): each committee cut lands at the window, chunk,
scan warp, ballot and lane it was built for; each proposer's first accept at its window and lane; each matcher holder on
its grid-stride pass and each prefix collision as built; the searched constants still qualify; the oracle's two
formulations agree on the small states and on the first candidates of the large ones."""
from __future__ import annotations

import numpy as np
import pytest

from oracle import duties_oracle as do
from tests import duties_grid_cases as gc

COMMITTEE = gc.committee_cases()
PROPOSER = gc.proposer_cases()


def test_window_map():
    wm = gc.window_map("mainnet")
    assert wm.words[:9] == [16 << k for k in range(9)] and sum(wm.words) == gc.CAP_WORDS
    assert [wm.chunks(k) for k in (5, 6, 7, 8)] == [1, 1, 2, 4]
    assert wm.candidate(8) == 130560 and wm.candidate(8, 3, 31, 31, 31) == 32 * (4080 + 4096) - 1
    assert wm.where(wm.candidate(7, 1, 2, 3, 4)) == (7, 1, 2, 3, 4)
    assert wm.where(wm.candidate(6) - 1) == (5, 0, 15, 31, 31)
    mm = gc.window_map("minimal")
    assert mm.words[:6] == [1, 2, 4, 8, 16, 32] and sum(mm.words) == gc.CAP_WORDS
    assert mm.where(31) == (0, 0, 0, 0, 31) and mm.where(32) == (1, 0, 0, 0, 0)
    # the last window is cut short so that all windows hold exactly 2^26 candidates
    assert wm.words[-1] < 2 * wm.words[-2] and wm.start[-1] + wm.words[-1] == gc.CAP_WORDS
    assert gc.match_stride(gc.matcher_n(132), 132) == 528 * 256 and gc.match_stride(1000, 132) == 4 * 256


def _stream(case):
    wm = gc.window_map(case.preset)
    count = wm.candidate(8, 1) if case.zero_eth else max((case.cut,) + case.after) + 64
    return gc.Stream(case.st, count)


@pytest.mark.parametrize("case", COMMITTEE, ids=[c.name for c in COMMITTEE])
def test_committee_cut_lands(case):
    st, wm = case.st, gc.window_map(case.preset)
    s = _stream(case)
    acc = s.accepts(st)
    assert s.cut(st, wm.size) == case.cut and acc[:case.cut].sum() == wm.size - 1
    w = wm.where(case.cut)
    for k, v in case.shape.items():
        assert getattr(w, k) == v, (k, w)
    eff = st.validators["effective_balance"]
    assert set(np.unique(eff).tolist()) <= {0, 32 * gc.ETH}
    assert acc[list(case.after)].all()
    ballot = lambda i: i // 32  # noqa: E731
    before = acc[ballot(case.cut) * 32:case.cut].sum()   # accepts earlier in the cut's ballot
    later = acc[case.cut + 1:(ballot(case.cut) + 1) * 32].sum()
    if not case.zero_eth and w.window:   # have carried: something accepted in every earlier window and chunk
        for k in range(w.window):
            assert acc[wm.candidate(k):wm.candidate(k + 1)].any(), k
        for c in range(w.chunk):
            assert acc[wm.candidate(w.window, c):wm.candidate(w.window, c + 1)].any(), c
    n = case.name
    if n == "lane0":
        assert w.lane == 0 and later >= 3                          # the in-ballot rank < size stop
    elif n == "lane31":
        assert w.lane == 31 and before >= 4 and acc[case.cut + 1:case.cut + 33].any()
    elif n == "warp_last_ballot":
        assert w.ballot == 31 and later and acc[case.cut + 1 - w.lane + 31:case.cut + 64].any()  # next warp accepts
    elif n == "warp_first_ballot":
        assert w.ballot == 0 and w.warp and acc[case.cut - w.lane - 32:case.cut - w.lane].any()   # previous warp's
    elif n in ("window3_first", "window8_first"):
        assert case.cut == wm.candidate(w.window) and w == (int(n[6]), 0, 0, 0, 0)              # have = SIZE - 1
        assert acc[:wm.candidate(w.window)].sum() == wm.size - 1 and later
    elif n == "w6_chunk0_last":
        assert wm.chunks(6) == 1 and (w.warp, w.ballot) == (31, 31) and later
    elif n == "w7_first_ballot":
        assert before and later and acc[wm.candidate(6):wm.candidate(7)].any()
    elif n == "w7_chunk0_last":
        assert wm.chunks(7) == 2 and (w.chunk, w.warp, w.ballot) == (0, 31, 31)
        assert acc[wm.candidate(7, 1):wm.candidate(7, 1) + 32].any()   # accepts in chunk 1 that must not be read
    elif n == "w7_chunk1_first":
        assert (w.chunk, w.warp, w.ballot) == (1, 0, 0) and before and later
        assert acc[wm.candidate(7):wm.candidate(7, 1)].sum() >= 10      # chunk 0's total moves chunk 1's base
    elif n == "zero_eth_w7_chunk1":
        assert (eff == 0).all() and w[:2] == (7, 1)
        assert acc[wm.candidate(7, 1):case.cut].sum() >= 50              # many accepts read from chunk 1
    elif n == "zero_eth_w8_wrapped":
        assert (eff == 0).all() and w[:2] == (8, 0) and case.cut > s.n + 32 * 64   # candidates past n wrap i mod n
        assert (s.cand[s.n:case.cut] == s.shuffled[:case.cut - s.n]).all()
        # chunks 1 to 3 of window 8 are drawn but never read: a cut there needs 512 zero bytes to come later than
        # candidate 163 328, where about 638 are expected (5 standard deviations)
        assert acc[:wm.candidate(8, 1)].sum() >= wm.size
    elif n == "minimal_w0_lane31":
        assert wm.words[0] == 1 and w == (0, 0, 0, 0, 31) and acc[:32].all()   # one warp of the CTA is busy
    elif n in ("minimal_w5", "minimal_w6"):
        assert w.window == int(n[-1]) >= 5
    else:
        raise AssertionError(n)


def test_committee_oracle_and_formulations():
    """The stream's accepted candidates are the oracle's committee (list formulation) on every case; the per-index
    formulation agrees on the minimal cases and on the first 2 048 candidates (and 64 wrapped ones) of the large ones."""
    for case in COMMITTEE:
        s = _stream(case)
        size = gc.window_map(case.preset).size
        want = [int(c) for c in s.cand[np.flatnonzero(s.accepts(case.st))[:size]]]
        assert do.next_sync_committee_indices(case.st, "list") == want, case.name
        if case.preset == "minimal":
            assert do.next_sync_committee_indices(case.st, "index") == want, case.name
    for case in (COMMITTEE[0], gc.zero_eth_case("w8_wrapped")):
        s = _stream(case)
        act = do.active_indices(case.st, gc.committee_epoch(case.st))
        idx = do._Sampler(case.st, act, s.seed, "index")
        lst = do._Sampler(case.st, act, s.seed, "list")
        for i in list(range(2048)) + list(range(s.n - 32, s.n + 32)):
            assert idx.candidate(i) == lst.candidate(i) == int(s.shuffled[i % s.n]), i


def test_searched_constants():
    assert gc.search_committee_mix(gc.COMMITTEE_MIX) == gc.COMMITTEE_MIX
    for name, k in gc.ZERO_ETH_MIX.items():
        assert gc.search_zero_eth_mix(name, k) == k
    assert gc.search_proposer_epoch(gc.PROPOSER_EPOCH) == gc.PROPOSER_EPOCH


def _first_accepts(st, epoch, counts):
    act = do.active_indices(st, epoch)
    out = []
    for seed, t in zip(gc.slot_seeds(st, epoch), counts):
        c = gc.slot_candidates(st, act, seed, t + 1)
        acc = gc.accepted(st.validators["effective_balance"][c], gc.random_bytes(seed, t + 1))
        out.append((int(np.argmax(acc)), int(c[np.argmax(acc)])) if acc.any() else None)
    return out


def test_proposer_placed_slots():
    case = PROPOSER[0]
    st, e = case.st, case.epochs[0]
    firsts = _first_accepts(st, e, case.targets)
    assert [f[0] for f in firsts] == case.targets
    where = [(t // 32, t % 32) for t in case.targets]
    assert {(0, 0), (0, 31), (1, 0)} <= set(where) and max(w for w, _ in where) >= 40
    ctas = [[where[4 * b + j][0] for j in range(gc.SAMPLE_WARPS)] for b in range(8)]
    assert max(ctas[1]) >= 40 and min(ctas[1]) == 0 and max(ctas[2]) >= 8 and min(ctas[2]) == 0
    assert do.proposer_indices(st, e) == [f[1] for f in firsts]
    assert (st.validators["effective_balance"] > 0).sum() <= 32


@pytest.mark.parametrize("case", PROPOSER[1:], ids=[c.name for c in PROPOSER[1:]])
def test_small_active_sets(case):
    st = case.st
    k = int(case.name.split("_")[1])
    for e in case.epochs:
        assert len(do.active_indices(st, e)) == k
        assert do.proposer_indices(st, e, "index") == do.proposer_indices(st, e, "list"), e
    assert do.next_sync_committee_indices(st, "index") == do.next_sync_committee_indices(st, "list")
    assert do.candidates_drawn(st) > 2 * k      # i mod n wraps inside the first ballots
    assert set((np.unique(st.validators["effective_balance"][9:9 + k]) // gc.ETH).tolist()) == {0, 1, 16, 31, 32}


@pytest.mark.parametrize("sms", (132, 114, 78))
def test_matcher_shape(sms):
    case, = gc.matcher_cases(sms)
    st, stride = case.st, case.stride
    n = len(st.validators)
    assert stride == 4 * sms * gc.MATCH_THREADS and -(-n // stride) == 3
    assert [e // stride for e in case.edges] == [0, 1, 2, 2] and case.edges == [stride - 1, stride, 2 * stride + 1, n - 1]
    K = st.validators["public_key"].copy().view(np.uint8).reshape(n, 48)
    prefix = lambda k: bytes(k[:8])  # noqa: E731
    for which in ("current", "next"):
        blob = getattr(st, f"{which}_sync_committee")
        keys = [np.frombuffer(blob[48 * j:48 * j + 48], np.uint8) for j in range(512)]
        got = do.sync_committee_indices(st, which)
        assert got == [case.holders[which].get(j, do.MISSING) for j in range(512)], which
        pre = {prefix(k) for k in keys}
        for d in case.decoys[which]:   # a committee prefix, another tail; one byte from a committee key: past its holder
            assert prefix(K[d]) in pre and K[d].tobytes() not in {k.tobytes() for k in keys}
            near = [j for j in range(512) if len(np.flatnonzero(keys[j] != K[d])) == 1]
            assert any(got[j] == do.MISSING or got[j] < d for j in near) or which == "current"
            assert which == "current" or near
        if which == "current":
            assert len(pre) == 1 and len({k.tobytes() for k in keys}) == 512
            assert got[:4] == case.edges and got[4] // stride == 2
            assert sum((K[:, :] == keys[4]).all(1)) >= 19 and sum(x == do.MISSING for x in got) == 3
        else:
            diff = lambda a, b: np.flatnonzero(keys[a] != keys[b]).tolist()  # noqa: E731
            assert diff(0, 1) == diff(2, 3) == [8] and diff(4, 5) == diff(6, 7) == [47]
            assert keys[0][8] < keys[1][8] and keys[2][8] > keys[3][8] and keys[4][47] < keys[5][47] and keys[6][47] > keys[7][47]
            assert {0, (1 << 64) - 1} <= {int.from_bytes(prefix(k), "big") for k in keys}
            assert got[10] == do.MISSING and sum(x == do.MISSING for x in got) == 1
            assert len({k.tobytes() for k in keys}) == 510   # two repeated committee positions
            assert {g // stride for g in got if g != do.MISSING} == {0, 1, 2}
