"""CPU: the shape-changing step scripts (tests/state_reshape_cases.py) on the host mirror, before they reach the device.

After every step of every script the mirror's serialization must be a valid deneb BeaconState on which the C oracle
and the hashlib oracle agree (hashlib where the state is small), the layout must follow the reshape (update_bytes
offsets move with it), every named boundary must be among the scripts, and every refused step must be refused by the
mirror with the code the library returns — leaving the mirror as it was.
"""
import ctypes
import os

import numpy as np
import pytest

from oracle import ssz_oracle as so
from ethereum_consensus_b200 import state as S
from tests import ssz_soak_cases as sc
from tests import state_reshape_cases as rc

NT = os.cpu_count() or 1


def c_root(O, b, preset):
    b = np.ascontiguousarray(b, dtype=np.uint8)
    out = ctypes.create_string_buffer(32)
    r = O.orc_htr_beacon_state_deneb(b.ctypes.data, b.size, 0 if preset == "mainnet" else 1, NT, out)
    return out.raw if r == 0 else r


def hashlib_root(b, preset):
    return so.beacon_state_type(preset).htr(S.to_oracle_value(sc.deserialize(b, preset)))


def run(O, st, steps, hashlib_every=1):
    """Apply the steps to the mirror; returns (accepted, refused kinds) and checks the oracles after every step."""
    accepted, refused = 0, []
    for i, step in enumerate(steps):
        before = S.serialize(st).copy()
        try:
            rc.apply(st, step)
        except S.ReshapeRefused as e:
            refused.append(e.kind)
            assert np.array_equal(S.serialize(st), before), (i, step[:2])
            continue
        accepted += 1
        b = S.serialize(st)
        assert np.array_equal(S.serialize(sc.deserialize(b, st.preset)), b), (i, step[:2])
        assert sc.layout_of(b, st.preset) == S.layout(st), (i, step[:2])
        r = c_root(O, b, st.preset)
        assert isinstance(r, bytes), (i, step[:2], r)
        if hashlib_every and i % hashlib_every == 0 and len(st.validators) <= 2100:
            assert hashlib_root(b, st.preset) == r, (i, step[:2])
    return accepted, refused


def test_every_boundary_is_a_script():
    names = {s["name"] for s in rc.boundary_scripts()}
    for what, scripts in rc.boundaries().items():
        for s in scripts:
            assert s in names, (what, s)


def test_boundary_scripts_on_the_host(oracle_ssz_c):
    want_refused = {
        "eth1_data_votes 0 / 1 / bound / bound + 1": ["limit", "limit"],
        "headers and malformed encodings": ["malformed", "malformed", "malformed", "malformed", "malformed", "bad_arg", "bad_arg"],
        "update_bytes over a moved offset": ["bad_arg", "bad_arg"],
    }
    for spec in rc.boundary_scripts():
        if spec["big"]:
            continue   # the 2^17 and relocation scripts are checked on the GPU against the C oracle only
        st, steps = rc.boundary_run(spec)
        n0 = len(st.validators)
        acc, ref = run(oracle_ssz_c, st, steps, hashlib_every=1 if n0 < 300 else 0)
        assert ref == want_refused.get(spec["name"], []), (spec["name"], ref)
        assert acc > 0, spec["name"]


def test_boundary_sizes_are_crossed():
    """The hand-off, fold and capacity scripts start below their boundary and end above it."""
    cross = {"validators 64 / 65 hand-off": ("validators", 1, rc.HANDOFF),
             "balances 256 / 257 hand-off": ("balances", 4, rc.HANDOFF),
             "participation 2048 / 2049 hand-off": ("current_epoch_participation", 32, rc.HANDOFF),
             "validators 2^17 +- 1 (fold)": ("validators", 1, rc.COOP_MAX),
             "validators from 0": ("validators", 1, 0)}
    for spec in rc.boundary_scripts():
        if spec["name"] not in cross:
            continue
        field, per, edge = cross[spec["name"]]
        st, steps = rc.boundary_run(spec)
        sizes = [len(getattr(st, field))]
        for step in steps:
            rc.apply(st, step)
            sizes.append(len(getattr(st, field)))
        assert min(sizes) < per * edge or min(sizes) == 0, spec["name"]
        assert {per * edge, per * edge + 1} <= set(sizes), (spec["name"], sizes)


def test_chain_walk_on_the_host(oracle_ssz_c):
    """The minimal-preset walk: >= 5 eth1 voting-period resets, >= 2 historical_summaries appends, every extra_data
    length 0..32, deposits of 0..16, and both oracles equal after every step (hashlib after every fifth step)."""
    spec = rc.walk_spec()
    st, steps = rc.walk(spec)
    kinds, resets, summaries, extra, deps = [], 0, 0, set(), set()
    recorded = []
    for step in steps:
        recorded.append(step)
        if step[:2] == ("set", "eth1_data_votes") and not step[2]:
            resets += 1
        if step[:2] == ("push", "historical_summaries"):
            summaries += 1
        if step[:2] == ("set", "latest_execution_payload_header"):
            extra.add(len(step[2]) - 584)
        if step[0] == "deposits":
            deps.add(len(step[1]) // 121)
        rc.apply(st, step)
        kinds.append(step[0])
    assert resets >= 5 and summaries >= 2, (resets, summaries)
    assert extra == set(range(33))
    assert max(deps) == rc.MAX_DEPOSITS and min(deps) >= 1
    st2, _ = rc.walk(spec)
    acc, ref = run(oracle_ssz_c, st2, recorded, hashlib_every=5)
    assert ref == [] and acc == len(recorded)
    assert np.array_equal(S.serialize(st2), S.serialize(st))


def test_refused_steps_leave_the_mirror_unchanged():
    st = rc.initial_state("minimal", 3, 1, votes=32)
    before = S.serialize(st).copy()
    for step, kind in ((("push", "eth1_data_votes", bytes(72)), "limit"),
                       (("set", "eth1_data_votes", bytes(71)), "malformed"),
                       (("set", "latest_execution_payload_header", bytes(584)), "malformed"),
                       (("push", "validators", bytes(120)), "malformed"),
                       (("push", "historical_roots", bytes(32)), "bad_arg"),
                       (("elements", "balances", [3], bytes(8)), "bad_arg")):
        with pytest.raises(S.ReshapeRefused) as e:
            rc.apply(st, step)
        assert e.value.kind == kind, step[:2]
        assert np.array_equal(S.serialize(st), before), step[:2]
