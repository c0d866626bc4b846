"""CPU: the multi-epoch scripts of tests/state_chain_cases.py reach every event they are built for, the oracle's two
process_epoch formulations agree along the minimal leg, and a script is a pure function of its seed."""
from __future__ import annotations

import numpy as np
import pytest

from ethereum_consensus_b200 import state as S
from oracle import epoch_oracle as eo
from tests import state_chain_cases as cc


@pytest.fixture(scope="module")
def legs():
    return {name: cc.walk(cc.leg_spec(name)) for name in ("minimal", "mainnet")}


def test_every_event_is_reached(legs):
    seen = {}
    for _, ev, _ in legs.values():
        for k, where in ev.seen.items():
            seen.setdefault(k, where)
    for name in cc.EVENTS:
        print(f"{name:40s} {seen.get(name, 'MISSING')}")
    assert [e for e in cc.EVENTS if e not in seen] == []
    mini, main = legs["minimal"][1].seen, legs["mainnet"][1].seen
    assert mini["capacity crossed by one"][1] == mini["relocation minimal"][1] == cc.leg_spec("minimal")["cross"]
    assert main["relocation mainnet"][1] == cc.leg_spec("mainnet")["cross"]
    for e in ("cache: relocation", "cache: process_epoch records", "cache: randao seed"):
        assert e in mini and e in main, e


def test_leg_shapes(legs):
    st, _, _ = legs["minimal"]
    assert len(st.validators) > 200 + (1 << 16)
    st, _, _ = legs["mainnet"]
    assert len(st.validators) > (1 << 18) + (1 << 16)
    # the mainnet leg relocates lists long enough for the multi-CTA ranges of k_epoch_reduce (256-thread CTAs, more than
    # one 512-thread reduce block of them)
    assert len(st.validators) // 256 > 512


def test_literal_and_vector_agree_on_the_small_leg():
    spec = cc.leg_spec("small")
    n = {"epochs": 0}
    st, steps = cc.run(spec)
    for step in steps:
        if step[0] == "process_epoch" and step[1] != cc.BAD_MASK:
            lit, c1 = eo.process_epoch(st, step[1], formulation="literal")
            vec, c2 = eo.process_epoch(st, step[1], formulation="vector")
            assert c1 == c2 == 0
            assert S.serialize(lit).tobytes() == S.serialize(vec).tobytes(), step
            n["epochs"] += 1
        try:
            cc.apply(st, step)
        except eo.Refused:
            assert step == ("process_epoch", cc.BAD_MASK)
    assert n["epochs"] == spec["epochs"]
    assert len(st.validators) > 80


def test_script_is_a_pure_function_of_its_seed(legs):
    spec = cc.leg_spec("minimal")
    assert cc.walk(spec)[2] == legs["minimal"][2]
    other = dict(spec, seed=spec["seed"] + 1)
    st, _, digest = cc.walk(other)
    assert digest != legs["minimal"][2]
    assert np.array_equal(st.validators["public_key"][:200], legs["minimal"][0].validators["public_key"][:200])
