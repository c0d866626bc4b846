"""CPU: the groups of tests/aggregate_grid_cases.py land where they were built to land, at 132 and 114 SMs (H100 SXM and
PCIe), and their expected codes and sums are right: the first-failure rule and the closed forms against the Python and C
oracles.  tests/test_aggregate_grid_gpu.py runs them through the CUDA kernels."""
from __future__ import annotations

import ctypes as C
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from oracle import bls_oracle as bo
from oracle import duties_oracle as do
from tests import aggregate_grid_cases as gc

CHUNKS = (32, 64, 96, 128)


def _chunk_scalars(g, m: gc.G2Map):
    """The discrete log of each chunk's partial sum (None for a chunk holding an invalid encoding)."""
    out = []
    for k in range(m.chunks_of(len(g.items))):
        part = g.items[k * m.chunk:(k + 1) * m.chunk]
        out.append(None if any(isinstance(it, bytes) and it != gc.INF_SIG for it in part)
                   else sum(gc.item_scalar(it) for it in part) % bo.R)
    return out


def _bad_positions(g):
    return [i for i, it in enumerate(g.items) if isinstance(it, bytes) and it != gc.INF_SIG]


def _check_group(call, gi, g, m):
    claim, C = g.claim, m.chunk
    where = lambda i: m.where(gi, i)  # noqa: E731
    if "same_lane" in claim:
        p1, p2 = claim["same_lane"]
        (c1, _, l1, s1), (c2, _, l2, s2) = where(p1), where(p2)
        assert l1 == l2 and (c1 == c2) == claim["same_chunk"], (call.name, g.name)
        assert (s2 > s1) if claim["same_chunk"] else (c2 == c1 + 1 and s1 == s2 == 0), (call.name, g.name)
        assert _bad_positions(g) == [p1, p2]
    if "cut" in claim:
        a, b = claim["cut"]
        assert where(a)[1:] == (0, 31, C // 32 - 1) and where(b)[1:] == (1, 0, 0), (call.name, g.name)
    if "ragged" in claim:
        nck = m.chunks_of(len(g.items))
        assert len(g.items) % C != 0 and where(claim["ragged"][-1])[1] == nck - 1 == 2, (call.name, g.name)
    if "finisher" in claim:
        k1, k2 = claim["finisher"]
        (l1, s1), (l2, s2) = m.finisher(k1), m.finisher(k2)
        assert l1 == l2 == k1 % 32 and s2 == s1 + 1, (call.name, g.name)
        bad = _bad_positions(g)
        if bad:
            assert [where(i)[1] for i in bad] == [k1, k2], (call.name, g.name)
    if "n_chunks" in claim:
        assert m.chunks_of(len(g.items)) == claim["n_chunks"], (call.name, g.name)
    for pos, k in claim.get("chunk_of", {}).items():
        assert where(pos)[1] == k and pos in _bad_positions(g), (call.name, g.name)
    if "chunk_of" in claim and "65 chunks" in g.name:
        assert m.chunks_of(len(g.items)) == 65
    sc = None
    if {"equal_chunks", "opposite_chunks", "zero_chunk"} & claim.keys():
        sc = _chunk_scalars(g, m)
    if "equal_chunks" in claim:
        ks = claim["equal_chunks"]
        assert len({sc[k] for k in ks}) == 1 and sc[ks[0]] != 0, (call.name, g.name)
        if len(ks) == 64:      # a block of exactly `chunk` tiled: every finisher lane adds two equal sums, so does the butterfly
            assert len(sc) == 64 and len(set(sc)) == 1
    if "opposite_chunks" in claim:
        k1, k2 = claim["opposite_chunks"]
        assert sc[k1] != 0 and (sc[k1] + sc[k2]) % bo.R == 0, (call.name, g.name)
        if k2 - k1 != 32:     # butterfly partners: one chunk per lane
            assert len(sc) <= 32 and (k1 ^ k2) in (1, 2, 4, 8, 16)
            if k1 ^ k2 == 1:  # every other chunk sums to infinity, so the two meet as they are in the last round
                assert all(s == 0 for k, s in enumerate(sc) if k not in (k1, k2))
    if "zero_chunk" in claim:
        k = claim["zero_chunk"]
        assert sc[k] == 0 and all(s != 0 for j, s in enumerate(sc) if j != k), (call.name, g.name)
    if claim.get("filler"):
        assert g.items == [i % gc.BLOCK for i in range(len(g.items))]


@pytest.mark.parametrize("sms", gc.SMS)
def test_filled_calls_land_where_built(sms):
    calls = gc.sig_calls(sms)
    want_n = {n for n, _ in gc.call_sizes(sms)}
    assert {len(c.groups) and c.map.n for c in calls} == want_n
    seen = {C: set() for C in CHUNKS}
    for call in calls:
        m = call.map
        assert m.n in want_n and m.chunk == call.chunk == gc.g2_chunk(m.n, sms), call.name
        assert m.n % (256 * sms) in (0, 1) and m.chunk == 32 * (m.n // (256 * sms) + m.n % (256 * sms))
        assert m.cta == 128 and m.launches == 2
        fillers = [g for g in call.groups if g.claim.get("filler")]
        assert len(fillers) == 1 and 0 < call.groups.index(fillers[0]) < len(call.groups) - 1
        assert m.chunks_of(len(fillers[0].items)) > 32      # the filler's finisher loop has more than one pass
        assert any(len(g.items) == 0 for g in call.groups[1:-1])
        # chunk_off / chunk_group as the host builds them
        assert m.chunk_group == [g for g in range(len(call.groups)) for _ in range(m.chunk_off[g + 1] - m.chunk_off[g])]
        for gi, g in enumerate(call.groups):
            _check_group(call, gi, g, m)
            seen[m.chunk].add(g.name)
    for C in CHUNKS:
        assert {g.name for g in gc.sig_cases(C)} <= seen[C], C
    # every same-lane order reaches a lane's second pass inside one chunk at chunk >= 64, and p + chunk - 32 at >= 96
    for C in (64, 96, 128):
        same = [g.claim["same_lane"] for g in gc.sig_cases(C) if g.claim.get("same_chunk")]
        assert {(p, p + 32) for p in (0, 5, 31)} <= set(same)
        if C > 64:
            assert {(p, p + C - 32) for p in (0, 5, 31)} <= set(same)


@pytest.mark.parametrize("sms", gc.SMS)
def test_edge_calls_switch_the_cta(sms):
    lo, hi = gc.edge_calls(sms)
    for call, n_chunks, cta in ((lo, 4 * sms - 1, 32), (hi, 4 * sms, 128)):
        m = call.map
        assert (m.chunk, m.n_chunks, m.cta) == (32, n_chunks, cta), call.name
        for gi, g in enumerate(call.groups):
            _check_group(call, gi, g, m)
    assert gc.g2_map([], sms).launches == 1 and gc.g2_map([0, 0, 0], sms).n_chunks == 3


def test_first_failure_rule_against_the_python_oracle():
    """The decode-error groups of every chunk size (cheap for the oracle: it stops at the first decode error) and the small
    groups whose verdict needs the subgroup checks or the sum."""
    for C in (32, 96):
        for g in gc.sig_cases(C):
            if g.want[0] in (gc.BAD_ENCODING, gc.NOT_ON_CURVE) and len(g.items) <= 2 * C + 17:
                assert bo.aggregate([gc.item_bytes(it) for it in g.items]) == g.want, (C, g.name)
    small = [g for g in gc.sig_cases(32) if g.name.startswith(("same lane nig@0", "cut nig", "two equal", "3 chunks, chunk 1 of"))]
    small.append(gc.Group("P, -P and infinity", [3, ~3, gc.INF_SIG, 4]))
    assert len(small) >= 5
    for g in small:
        assert bo.aggregate([gc.item_bytes(it) for it in g.items]) == g.want, g.name
    codes = {nm: c for nm, (e, c) in gc.sig_invalid().items()}
    for nm, (e, c) in gc.sig_invalid().items():
        got, pt = bo.g2_uncompress(e)
        if c == gc.NOT_IN_GROUP:
            assert got == 0 and pt is not None and not bo.in_subgroup(bo.F2, pt)
        else:
            assert got == c
    assert codes == {"bad": 1, "noc": 2, "nig": 3}


def _c_aggregate(O, items):
    out = C.create_string_buffer(96)
    code = O.orc_aggregate(b"".join(gc.item_bytes(it) for it in items), len(items), out)
    return int(code), (out.raw if code == 0 else None)


def test_expectations_against_the_c_oracle(oracle_bls_c):
    """Every group of up to 2 200 signatures at every chunk size, code for code and byte for byte."""
    gs = {}
    for Cc in CHUNKS:
        for g in gc.sig_cases(Cc):
            if 0 < len(g.items) <= 2200:
                gs.setdefault((g.name, len(g.items)), g)
    with ThreadPoolExecutor(8) as ex:
        got = list(ex.map(lambda g: _c_aggregate(oracle_bls_c, g.items), gs.values()))
    for g, row in zip(gs.values(), got):
        assert row == g.want, g.name
    assert {g.want[0] for g in gs.values()} == {0, 1, 2, 3}


def test_closed_forms_and_the_tiled_filler(oracle_bls_c):
    h, a, d, pts, enc, neg = gc.sig_pool()
    for i in (0, 1, 517, gc.POOL - 1):
        assert pts[i] == gc.ac.G2.mul(h, a + i * d)
        assert bo.g2_uncompress(neg[i])[1] == gc.ac.G2.neg(pts[i])
    for L in (gc.BLOCK - 1, 2 * gc.BLOCK + 37, 33_792 - 5_000):
        f = gc.filler(L)
        s = gc.filler_closed_form(L)
        assert s == sum(gc.item_scalar(it) for it in f.items) % bo.R
        assert f.want == (0, bo.g2_compress(gc.ac.G2.mul(h, s)))
    f = gc.filler(2 * gc.BLOCK + 37)
    assert _c_aggregate(oracle_bls_c, f.items) == f.want


# ------------------------------------------------------------------------------------------------ keys
def test_key_tuples_land_on_one_lane():
    cases = gc.key_cases()
    pairs = [g for g in cases if "same_lane" in g.claim]
    assert len(pairs) == 3 * 2 * 12
    assert {(g.want[0], gc.key_bytes(g.slots[g.claim["same_lane"][1]])) for g in pairs}
    for T in gc.KEY_T:
        gs = gc.key_call(T)
        assert T % 4 in (0, 1, 3) and gc.compress_cta(T) == (32 if T <= 32 else 128)
        for t, g in enumerate(gs):
            if "same_lane" in g.claim:
                p, q = g.claim["same_lane"]
                (b1, w1, l1, s1), (b2, w2, l2, s2) = gc.k2_map(t, p), gc.k2_map(t, q)
                assert (b1, w1, l1) == (b2, w2, l2) and s2 - s1 == (q - p) // 32
        last_cta = [g for t, g in enumerate(gs) if t // 4 == (T - 1) // 4]
        assert any(g.want[0] != 0 for g in last_cta), T
    assert {T % 4 for T in gc.KEY_T} == {0, 1, 3} and {32, 33, 127, 128, 129} <= set(gc.KEY_T)
    # every ordered pair of distinct codes at both gaps
    got = {(g.claim["same_lane"][1] - g.claim["same_lane"][0], g.slots[g.claim["same_lane"][0]][0],
            g.slots[g.claim["same_lane"][1]][0]) for g in pairs}
    assert got == {(gap, c1, c2) for gap in (32, 64) for c1 in gc.KEY_CODES for c2 in gc.KEY_CODES if c1 != c2}


def test_key_expectations_against_the_oracles(oracle_bls_c):
    cases = gc.key_cases()
    _, _, _, _, inv = gc.key_material()
    for c, encs in inv.items():
        assert [bo.key_validate(e)[0] for e in encs] == [c, c] and (c == gc.PK_IS_INFINITY or encs[0] != encs[1])
    for g in cases:
        assert bo.eth_aggregate_public_keys([gc.key_bytes(s) for s in g.slots]) == g.want, g.name
    # the C oracle's strict batch: the first failing key decides the tuple
    keys = [gc.key_bytes(s) for g in cases for s in g.slots]
    off = np.cumsum([0] + [len(g.slots) for g in cases]).astype(np.uint32)
    pks = np.frombuffer(b"".join(keys), dtype=np.uint8)
    msgs = np.frombuffer(b"".join(gc.verify_msg(t) for t in range(len(cases))), dtype=np.uint8)
    sigs = np.frombuffer(gc.verify_sig() * len(cases), dtype=np.uint8)
    out = np.zeros(len(cases), dtype=np.int32)
    oracle_bls_c.orc_fast_aggregate_verify_batch(pks.ctypes.data, off.ctypes.data, msgs.ctypes.data, sigs.ctypes.data,
                                                 len(cases), out.ctypes.data, 8)
    assert out.tolist() == [gc.verify_want(g) for g in cases]
    keys, where = gc.registry_keys()
    assert [keys[where[s]] for s in where] == [gc.key_bytes(s) for s in where]


def test_sync_committee_positions():
    st = gc.sync_state()
    idx = do.next_sync_committee_indices(st, "list")
    assert len(idx) == 512
    cases = gc.sync_cases(idx)
    assert len(cases) == 24 and {q - p for p, q, _, _ in cases} == set(gc.SYNC_GAPS)
    for p, q, c1, c2 in cases:
        assert p % 32 == q % 32 and q // 32 > p // 32 and idx[p] != idx[q]
        assert idx.index(idx[p]) == p and idx.index(idx[q]) == q and c1 != c2


def c_aggregate(O):
    def agg(keys):
        out = C.create_string_buffer(48)
        code = O.orc_eth_aggregate_public_keys(b"".join(keys), len(keys), out)
        return int(code), (out.raw if code == 0 else None)
    return agg


def test_sync_committee_code_is_the_earlier_position(oracle_bls_c):
    st = gc.sync_state()
    idx = do.next_sync_committee_indices(st, "list")
    pk = st.validators["public_key"]
    for p, q, c1, c2 in gc.sync_cases(idx)[::5]:
        keep = pk[idx[p]].copy(), pk[idx[q]].copy()
        pk[idx[p]] = np.frombuffer(gc.key_material()[4][c1][0], dtype="V48")[0]
        pk[idx[q]] = np.frombuffer(gc.key_material()[4][c2][1], dtype="V48")[0]
        assert do.next_sync_committee_indices(st, "list") == idx
        assert do.next_sync_committee(st, c_aggregate(oracle_bls_c), "list")[2] == c1, (p, q, c1, c2)
        pk[idx[p]], pk[idx[q]] = keep
