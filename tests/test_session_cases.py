"""CPU: the engine session (tests/session_cases.py) contains every transition it exists for, and its expected answers
agree with each other and with independent oracles."""
from __future__ import annotations

import ctypes
import hashlib

import numpy as np
import pytest

from tests import session_cases as sn

_CACHE = {}


@pytest.fixture(scope="module")
def session():
    if "s" not in _CACHE:
        _CACHE["s"] = sn.build_session()
    return _CACHE["s"]


def _n_keys(s):
    """Entries of the shared key staging buffer (BlsState::keys) a step fills, or None if it does not use it."""
    a = s.args
    if s.family in ("strict", "rlc") and "pks" in a:
        return a["pks"].size // 48
    if s.op == "verify_batch":
        return a["extra"].size // 48
    if s.op == "eth_aggregate_public_keys":
        return len(a["pks"])
    return None


def _n_tuples(s):
    """Tuples of a batch step (BlsState::out / stage / sig_code / g2pts), or None."""
    if s.family in ("strict", "rlc") or s.op == "verify_batch":
        return len(s.args["off"]) - 1
    if s.op == "aggregate":
        return len(s.args["sigs"])
    return None


def _n_ssz(s):
    """Bytes of a one-shot SSZ call (Engine::staging / arena / fields), or None."""
    a = s.args
    if s.op == "hash":
        return len(a["data"])
    if s.op == "merkleize":
        return a["chunks"].size
    if s.op in ("htr_validators", "htr_beacon_state"):
        return a["ssz"].size
    return None


def _n_shuffle(s, n_state):
    """Positions of a shuffle (the static shuffle scratch), or None."""
    if s.op == "compute_shuffled_indices":
        return s.args["n"]
    if s.op == "get_active_validator_indices":
        return s.args["recs"].size // 121
    if s.op == "state_shuffled_active_indices":
        return n_state
    return None


def _grow_then_shrink(sizes):
    """(step of a growth past every earlier size, the next user's step) pairs where the next user is smaller."""
    out, top = [], -1
    for k, (i, n) in enumerate(sizes):
        if n > top:
            top = n
            if k + 1 < len(sizes) and sizes[k + 1][1] < n:
                out.append((i, sizes[k + 1][0]))
    return out


def test_census_shared_buffers_shrink_right_after_growth(session):
    steps = session.steps
    n_state = session.meta["n0"]
    series = {"keys": [], "tuples": [], "ssz": [], "shuffle": []}
    for s in steps:
        if s.op == "add_validators":
            n_state += len(s.args["balances"])
        for name, n in (("keys", _n_keys(s)), ("tuples", _n_tuples(s)), ("ssz", _n_ssz(s)), ("shuffle", _n_shuffle(s, n_state))):
            if n is not None:
                series[name].append((s.i, n))
    for name, sizes in series.items():
        pairs = _grow_then_shrink(sizes)
        print(f"{name:8s} users {len(sizes):3d}  growths followed by a shrink {len(pairs)}")
        assert pairs, name


def test_census_launch_shape_thresholds(session):
    strict = [s for s in session.steps if s.family == "strict" and not isinstance(s.want, tuple) or
              (s.family == "strict" and s.want and s.want[0] != "refused")]
    shapes = [(len(s.args["off"]) - 1, int(s.args["off"][-1])) for s in strict]
    assert (1, 1) in shapes
    assert any(T == 1024 for T, _ in shapes) and any(T == 1025 for T, _ in shapes)   # 2 048 / 2 050 Miller pairs
    assert 2 * 1024 <= sn.VM_TEAM16_MAX < 2 * 1025
    assert any(k >= sn.SMALL_CTA_KEYS and T > 1024 for T, k in shapes)
    assert any(k > sn.K1_WIDE_KEYS for _, k in shapes)
    assert any(k >= sn.SPLIT_KEYS for _, k in shapes)
    ragged = [np.diff(s.args["off"].astype(np.int64)) for s in strict if len(s.args["off"]) == 66]
    assert ragged and set(ragged[0].tolist()) == set(range(65))
    # the 2 048 / 2 050 pair batches run right after each other, and under vm_team16_max 0 and the alternative schedule
    idx = [s.i for s in strict if len(s.args["off"]) - 1 in (1024, 1025)]
    assert any(b - a == 1 for a, b in zip(idx, idx[1:]))


def test_census_relocations_and_mixed_calls_around_them(session):
    steps = session.steps
    n0 = session.meta["n0"]
    big = [s for s in steps if s.op == "add_validators" and ("relocate", "state") in s.tags]
    assert len(big) == 1
    before = sum(len(s.args["balances"]) for s in steps if s.op == "add_validators" and s.i < big[0].i)
    n_big = len(big[0].args["balances"])
    assert n_big > sn.rc.headroom(n0 + before)                          # the state's lists move
    cap = n0 + max(sn.HEADROOM_MIN, n0 // 16) + sn.REG_EXTRA + 1         # registry arrays as from_state sized them
    assert n0 + before + n_big + sn.REG_EXTRA + 1 > cap                  # the registry's arrays move
    mixed = [s.i for s in steps if s.op == "verify_batch" and not s.want[:1] == ("refused",)]
    assert any(i < big[0].i for i in mixed) and any(i > big[0].i for i in mixed)
    sync = [s for s in steps if s.op == "sync"]
    assert any(s.i > big[0].i and ("relocate", "registry") in s.tags for s in sync)


def test_census_every_refusal_is_followed_by_its_family(session):
    steps = session.steps
    seen = set()
    for s in steps:
        kinds = [t[1] for t in s.tags if t[0] == "refusal"]
        if not kinds:
            continue
        assert s.want[0] == "refused", s.describe()
        nxt = steps[s.i + 1]
        assert nxt.family == s.family and nxt.want[:1] != ("refused",), (s.describe(), nxt.describe())
        assert ("after", kinds[0]) in nxt.tags
        seen.add(kinds[0])
    assert seen == set(sn.REFUSALS)
    # after the last refusal the resident objects read as before the first one
    roots = [s.want for s in steps if s.op in ("state_root", "incremental_root")]
    assert roots[-1] == roots[-2] == roots[-3] == session.meta["final_root"]
    codes = [s.want for s in steps if s.op == "key_codes"]
    assert len(set(codes[-3:])) == 1 and codes[-1][0] == session.meta["final_n"]


def test_census_settings_rlc_singles_ssz_shuffles_evals(session):
    steps = session.steps
    tunes = [(s.args["knob"], s.args["value"]) for s in steps if s.op == "tune"]
    for kv in (("vm_cta", 64), ("vm_cta", 128), ("vm_team16_max", 0), ("bls_small_cta", 128)):
        assert kv in tunes, kv
    last = {}
    for k, v in tunes:
        last[k] = v
    assert last == {"vm_cta": 32, "vm_team16_max": sn.VM_TEAM16_MAX, "bls_small_cta": 0}
    loads = [s for s in steps if s.op == "vm_load_programs"]
    assert len(loads) == 3 and [("restore",) in s.tags for s in loads] == [False, True, True]
    assert any(s.family in ("strict", "rlc") for s in steps[loads[0].i:loads[1].i])
    # RLC: both entry points, True and False, T above and below the previous call's
    rlc = [s for s in steps if s.family == "rlc"]
    for op in ("fast_aggregate_verify_batch_all", "registry_verify_batch_all"):
        assert {s.want for s in rlc if s.op == op} == {True, False}, op
    ts = [len(s.args["off"]) - 1 for s in rlc]
    assert any(b > a for a, b in zip(ts, ts[1:])) and any(b < a for a, b in zip(ts, ts[1:]))
    assert any(s.args["seed"] is None for s in rlc)
    # per-tuple batches between the RLC checks
    fams = [s.family for s in steps if s.family in ("rlc", "strict")]
    assert any(a == "rlc" and b == "strict" for a, b in zip(fams, fams[1:]))
    ops = {s.op for s in steps if s.family == "single"}
    assert ops == {"verify_signature", "fast_aggregate_verify", "eth_fast_aggregate_verify", "aggregate_verify", "aggregate",
                   "eth_aggregate_public_keys"}
    inf = [s for s in steps if s.op == "eth_fast_aggregate_verify"]
    assert inf and all(s.args["sig"] == bytes([0xC0]) + bytes(95) and s.want == 0 for s in inf)
    hashes = [len(s.args["data"]) for s in steps if s.op == "hash"]
    assert hashes[:3] == [1 << 20, 0, 55]
    mk = [s.args["chunks"].size // 32 for s in steps if s.op == "merkleize"]
    assert mk[:2] == [1 << 20, 1]
    assert {s.args["depth"] for s in steps if s.op == "is_valid_merkle_branch"} == {0, 1, 40, 64}
    presets = {s.args["preset"] for s in steps if s.op == "htr_beacon_state"}
    assert presets == {"mainnet"} and session.init_state is not None            # the resident state is minimal
    sh = [s for s in steps if s.family == "shuffle" or s.op == "state_shuffled_active_indices"]
    j = next(k for k, s in enumerate(sh) if s.op == "compute_shuffled_indices" and s.args["n"] == 1 << 20)
    a, b2 = sh[j], sh[j + 1]
    assert b2.args["n"] == 5 and b2.args["seed"] == a.args["seed"] and b2.args["rounds"] == a.args["rounds"]
    assert any(x.args["n"] == 5 and x.args["seed"] != a.args["seed"] for x in sh[j + 2:] if x.op == "compute_shuffled_indices")
    k = next(k for k, s in enumerate(sh) if s.op == "state_shuffled_active_indices" and k > j)
    assert sh[k - 1].op == "get_active_validator_indices" and steps[sh[k].i - 1].i == sh[k - 1].i
    assert any(x.op == "get_active_validator_indices" for x in steps[sh[k].i + 1:sh[k].i + 3])
    assert {s.op for s in steps if s.family == "eval"} == {"fp_eval", "curve_eval", "pairing_eval"}


# ---------------------------------------------------------------------------------------------------------- consistency
def test_blocks_registry_model_is_key_validate_of_the_state_keys(session):
    """After every block the registry's expected codes are key_validate of the mirror state's public keys (each distinct
    key validated by the C oracle once)."""
    B, _ = sn.oracles()
    st = session.meta["mirror"]
    pk = np.frombuffer(st.validators.tobytes(), np.uint8).reshape(-1, 121)[:, :48]
    uniq, inv = np.unique(pk, axis=0, return_inverse=True)
    codes = np.array([B.orc_key_validate(u.tobytes()) for u in uniq], dtype=np.int32)[inv.reshape(-1)]
    want = [s.want for s in session.steps if s.op == "key_codes"]
    assert want[-1] == sn.digest(codes)
    n = session.meta["n0"]
    for s in session.steps:
        if s.op == "add_validators":
            n += len(s.args["balances"])
        if s.op == "sync":
            assert s.want == n
        if s.op == "key_codes" and s.want[0] == n:
            assert s.want == sn.digest(codes[:n])


def test_blocks_incremental_root_model_is_the_full_root(session):
    """Each block's expected incremental root == the Python SSZ oracle's root of the mirror then (the small states), and the
    C oracle's full root of the final mirror."""
    from ethereum_consensus_b200 import state as S
    from oracle import ssz_oracle as so
    steps = session.steps
    small = [(i, st) for i, st in session.meta["snapshots"] if st is not None]
    assert len(small) >= 3
    T = so.beacon_state_type("minimal")
    for i, st in small[:3]:
        assert steps[i].want == T.htr(S.to_oracle_value(st)), i
    _, Z = sn.oracles()
    assert sn.state_root(Z, session.meta["mirror"]) == session.meta["final_root"]
    assert [st is None for _, st in session.meta["snapshots"]].count(True) >= 1


def test_tiled_batches_repeat_their_base_codes(session):
    """The big strict batches repeat a small batch's tuples: a sample of their tuples re-verified by the C oracle."""
    B, _ = sn.oracles()
    rng = np.random.default_rng(5)
    for name in ("big_side", "big_k1", "big_split"):
        b = session.meta["batches"][name]
        ts = rng.choice(b.T, 24, replace=False)
        keys = b.flat.reshape(-1, 48)
        flat = np.concatenate([keys[b.off[t]:b.off[t + 1]] for t in ts])
        off = np.concatenate([[0], np.cumsum([b.off[t + 1] - b.off[t] for t in ts])]).astype(np.uint32)
        msgs = b.msgs.reshape(-1, 32)[ts]
        sigs = b.sigs.reshape(-1, 96)[ts]
        assert sn.oracle_codes(B, flat, off, msgs, sigs) == tuple(b.codes[t] for t in ts), name
    assert len(set(session.meta["batches"]["ragged"].codes)) >= 4


def test_merkle_branches_and_refusals_match_the_python_oracles(session):
    from oracle import ssz_oracle as so
    for s in session.steps:
        if s.op == "is_valid_merkle_branch":
            a = s.args
            assert so.is_valid_merkle_branch(a["leaf"], a["branch"], a["depth"], a["index"], a["root"]) == s.want
        if s.op == "hash":
            assert hashlib.sha256(s.args["data"]).digest() == s.want


def test_shuffled_order_keeps_dependent_steps_in_order(session):
    steps = session.steps
    order = sn.shuffled_order(steps, 0x0D0E)
    pos = {j: p for p, j in enumerate(order)}
    assert sorted(order) == list(range(len(steps))) and order != list(range(len(steps)))
    for j in range(len(steps)):
        for i in range(j):
            if sn.depends(steps[i], steps[j]):
                assert pos[i] < pos[j], (i, j)
    moved = sum(1 for p, j in enumerate(order) if p != j)
    assert moved > len(steps) // 2
    need = sn.closure(steps, len(steps) - 1)        # the last key_codes needs the registry's and the state's history
    assert 0 in need and any(steps[k].op == "sync" for k in need)
