"""Seeded case generators for the SSZ / incremental re-hash / shuffling soak (no device code, no torch).

tests/test_ssz_device_soak_gpu.py runs these cases through the CUDA library; tests/test_ssz_soak_cases.py checks on the
CPU that they hit every planner boundary, that the C and hashlib oracles agree on them, and that the C oracle rejects
every malformed encoding.  Everything is a pure function of its seed, so a child process regenerates the same inputs.

Planner boundaries (csrc/ssz_plan.cu, csrc/shuffle.cu) the sizes are chosen around:
  * a list of <= 64 nodes goes straight to the single-CTA finisher (kHandoff): 64 / 65 validators, 256 / 257 balances
    (4 per chunk), 2 048 / 2 049 participation flags (32 per chunk);
  * a REDUCE job with <= 2^17 inputs is folded into k_merkle_coop (kCoopMaxInputs): 2^17 +- 1 validators, 2^19 +- 4
    balances;
  * the one-shot Validator upload goes out in min(16, max(1, n / 32 768)) slices of whole 256-record CTAs, the last one
    possibly short;
  * a ragged last CTA (n mod 256 != 0);
  * k_active_scan sums more than one block count per thread above 1 024 CTAs (262 144 validators).
"""
from __future__ import annotations

import hashlib
import os
import struct
import sys
from pathlib import Path
from typing import Dict, List

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from ethereum_consensus_b200 import state as S  # noqa: E402

SCALE = float(os.environ.get("B200_SOAK_SCALE", "1"))
HANDOFF = 64                 # SszPlan::kHandoff
COOP_MAX = 1 << 17           # kCoopMaxInputs in SszPlan::run
CTA = 256                    # kStageThreads; also shuffle.cu's kThreads
SLICE_MIN = 32768            # records per pipelined Validator slice (at least)
SCAN_CTAS = 1024             # k_active_scan's block size
FAR = S.FAR_FUTURE_EPOCH
FIELDS_28 = ["genesis_time", "genesis_validators_root", "slot", "fork", "latest_block_header", "block_roots", "state_roots",
             "historical_roots", "eth1_data", "eth1_data_votes", "eth1_deposit_index", "validators", "balances",
             "randao_mixes", "slashings", "previous_epoch_participation", "current_epoch_participation",
             "justification_bits", "previous_justified_checkpoint", "current_justified_checkpoint", "finalized_checkpoint",
             "inactivity_scores", "current_sync_committee", "next_sync_committee", "latest_execution_payload_header",
             "next_withdrawal_index", "next_withdrawal_validator_index", "historical_summaries"]
BIG_LISTS = {"validators": 121, "balances": 8, "previous_epoch_participation": 1, "current_epoch_participation": 1,
             "inactivity_scores": 8}
CHAINS = list(BIG_LISTS) + ["block_roots", "state_roots", "randao_mixes", "slashings"]
ELEM = {**BIG_LISTS, "block_roots": 32, "state_roots": 32, "historical_roots": 32, "eth1_data_votes": 72,
        "randao_mixes": 32, "slashings": 8, "historical_summaries": 64}


def n_scaled(x: int) -> int:
    return max(1, int(x * SCALE))


def slices(n: int) -> List[int]:
    """Record counts of the pipelined Validator upload's slices (ssz_plan.cu, SszPlan::run)."""
    k = min(16, max(1, n // SLICE_MIN))
    per = ((n + k - 1) // k + CTA - 1) // CTA * CTA
    return [min(per, n - lo) for lo in range(0, n, per)]


# ---------------------------------------------------------------------------------------------------------- states
def state_specs() -> List[dict]:
    """Whole-state cases: both presets, validator counts across every planner boundary, and the variable-size small
    fields at 0 / the 64-node handoff / beyond it, eth1_data_votes at 0 and at its bound, extra_data of 0, 1, 31, 32 bytes."""
    m, M = "minimal", "mainnet"
    mb, Mb = S.PRESETS[m]["ETH1_DATA_VOTES_BOUND"], S.PRESETS[M]["ETH1_DATA_VOTES_BOUND"]
    rows = [  # preset, validators, historical_roots, historical_summaries, eth1 votes, extra_data length
        (m, 0, 0, 0, 0, 0), (m, 1, 64, 65, mb, 32), (m, 5, 65, 64, 0, 1), (m, 64, 300, 0, mb, 31), (m, 65, 0, 300, 7, 0),
        (m, 256, 65, 65, mb, 32), (m, 257, 64, 64, 1, 1), (m, 2048, 3, 2, mb, 0), (m, 2049, 300, 300, 0, 31),
        (M, 0, 0, 0, Mb, 0), (M, 3, 65, 64, 0, 32), (M, 257, 64, 65, Mb, 1), (M, 1000, 300, 3, 100, 31),
        (M, 2049, 0, 0, Mb, 32), (M, 4097, 2, 3, 1024, 4),
        (M, 65535, 65, 300, Mb, 0), (M, 65536, 3, 2, 0, 32), (M, 65537, 300, 65, 1024, 31),
        (M, COOP_MAX - 1, 64, 64, Mb, 1), (M, COOP_MAX, 0, 0, 1024, 32), (M, COOP_MAX + 1, 65, 65, 0, 0),
        (M, 4 * COOP_MAX - 4, 2, 3, 1024, 4), (M, 4 * COOP_MAX, 2, 3, 1024, 4), (M, 4 * COOP_MAX + 4, 65, 300, Mb, 32),
    ]
    out = []
    for i, (preset, n, hr, hs, votes, ex) in enumerate(rows):
        out.append(dict(name=f"{preset}:{n}:hr{hr}:hs{hs}:v{votes}:x{ex}", preset=preset, n=n, hr=hr, hs=hs, votes=votes,
                        extra=bytes((7 * j + ex) & 0xff for j in range(ex)), seed=0x55A0 + i))
    return out


def boundaries() -> Dict[str, list]:
    """Each named planner boundary -> the (preset, validators) pairs that must be among the state cases."""
    M = "mainnet"
    return {
        "validators: finisher hand-off 64 / 65": [("minimal", HANDOFF), ("minimal", HANDOFF + 1)],
        "balances: finisher hand-off 256 / 257": [("minimal", 4 * HANDOFF), ("minimal", 4 * HANDOFF + 1)],
        "participation: finisher hand-off 2 048 / 2 049": [("minimal", 32 * HANDOFF), ("minimal", 32 * HANDOFF + 1)],
        "validators: coop limit 2^17 - 1, 2^17, 2^17 + 1": [(M, COOP_MAX - 1), (M, COOP_MAX), (M, COOP_MAX + 1)],
        "balances: coop limit 2^19 - 4, 2^19, 2^19 + 4": [(M, 4 * COOP_MAX - 4), (M, 4 * COOP_MAX), (M, 4 * COOP_MAX + 4)],
        "upload: one slice": [(M, 65535)],
        "upload: two whole slices": [(M, 65536)],
        "upload: two slices, short last slice": [(M, 65537)],
        "upload: 16 slices, short last slice": [(M, 4 * COOP_MAX + 4)],
        "ragged last CTA": [(M, 65537), (M, COOP_MAX + 1), ("minimal", 257)],
        "no validators": [("minimal", 0), (M, 0)],
    }


def state_for(spec: dict) -> S.SynthState:
    st = S.synth_state(spec["n"], spec["preset"], seed=spec["seed"], n_eth1_votes=spec["votes"],
                       n_historical_summaries=spec["hs"], n_historical_roots=spec["hr"], extra_data=spec["extra"])
    return st


def serialized(spec: dict) -> np.ndarray:
    return S.serialize(state_for(spec))


def fixed_len(preset: str) -> int:
    P = S.PRESETS[preset]
    return (8 + 32 + 8 + 16 + 112 + 2 * 32 * P["SLOTS_PER_HISTORICAL_ROOT"] + 4 + 72 + 4 + 8 + 4 + 4
            + 32 * P["EPOCHS_PER_HISTORICAL_VECTOR"] + 8 * P["EPOCHS_PER_SLASHINGS_VECTOR"] + 4 + 4 + 1 + 3 * 40 + 4
            + 2 * (48 * P["SYNC_COMMITTEE_SIZE"] + 48) + 4 + 8 + 8 + 4)


def offset_positions(preset: str) -> List[int]:
    """Byte positions of the nine 4-byte offsets in the fixed part, in field order."""
    P = S.PRESETS[preset]
    sc = 48 * P["SYNC_COMMITTEE_SIZE"] + 48
    o_hr = 8 + 32 + 8 + 16 + 112 + 2 * 32 * P["SLOTS_PER_HISTORICAL_ROOT"]
    o_votes = o_hr + 4 + 72
    o_val = o_votes + 4 + 8
    o_bal = o_val + 4
    o_prev = o_bal + 4 + 32 * P["EPOCHS_PER_HISTORICAL_VECTOR"] + 8 * P["EPOCHS_PER_SLASHINGS_VECTOR"]
    o_cur = o_prev + 4
    o_inact = o_cur + 4 + 1 + 120
    o_hdr = o_inact + 4 + 2 * sc
    o_hs = o_hdr + 4 + 16
    return [o_hr, o_votes, o_val, o_bal, o_prev, o_cur, o_inact, o_hdr, o_hs]


def layout_of(b, preset: str) -> Dict[str, tuple]:
    """{field: (offset, length)} read from a serialization (the same names as state.layout)."""
    b = memoryview(np.ascontiguousarray(b)).cast("B")
    P = S.PRESETS[preset]
    offs = [struct.unpack_from("<I", b, p)[0] for p in offset_positions(preset)] + [len(b)]
    names_var = ["historical_roots", "eth1_data_votes", "validators", "balances", "previous_epoch_participation",
                 "current_epoch_participation", "inactivity_scores", "latest_execution_payload_header", "historical_summaries"]
    sc = 48 * P["SYNC_COMMITTEE_SIZE"] + 48
    fixed = [("genesis_time", 8), ("genesis_validators_root", 32), ("slot", 8), ("fork", 16), ("latest_block_header", 112),
             ("block_roots", 32 * P["SLOTS_PER_HISTORICAL_ROOT"]), ("state_roots", 32 * P["SLOTS_PER_HISTORICAL_ROOT"]), 0,
             ("eth1_data", 72), 1, ("eth1_deposit_index", 8), 2, 3, ("randao_mixes", 32 * P["EPOCHS_PER_HISTORICAL_VECTOR"]),
             ("slashings", 8 * P["EPOCHS_PER_SLASHINGS_VECTOR"]), 4, 5, ("justification_bits", 1),
             ("previous_justified_checkpoint", 40), ("current_justified_checkpoint", 40), ("finalized_checkpoint", 40), 6,
             ("current_sync_committee", sc), ("next_sync_committee", sc), 7, ("next_withdrawal_index", 8),
             ("next_withdrawal_validator_index", 8), 8]
    out, pos = {}, 0
    for p in fixed:
        if isinstance(p, int):
            out["offset:" + names_var[p]] = (pos, 4); pos += 4
        else:
            out[p[0]] = (pos, p[1]); pos += p[1]
    for k, name in enumerate(names_var):
        out[name] = (offs[k], offs[k + 1] - offs[k])
    return out


def deserialize(b, preset: str) -> S.SynthState:
    """The SynthState a (valid) serialization encodes: the inverse of state.serialize, for the hashlib oracle."""
    b = np.ascontiguousarray(b, dtype=np.uint8)
    lay = layout_of(b, preset)
    get = lambda f: bytes(b[lay[f][0]: lay[f][0] + lay[f][1]])  # noqa: E731
    arr = lambda f, w: b[lay[f][0]: lay[f][0] + lay[f][1]].reshape(-1, w).copy()  # noqa: E731
    st = S.SynthState(preset=preset)
    st.fixed = {k: get(k) for k in ["genesis_time", "genesis_validators_root", "slot", "fork", "latest_block_header",
                                    "eth1_data", "eth1_deposit_index", "justification_bits", "previous_justified_checkpoint",
                                    "current_justified_checkpoint", "finalized_checkpoint", "next_withdrawal_index",
                                    "next_withdrawal_validator_index"]}
    st.block_roots, st.state_roots, st.randao_mixes = arr("block_roots", 32), arr("state_roots", 32), arr("randao_mixes", 32)
    st.historical_roots, st.eth1_data_votes = arr("historical_roots", 32), arr("eth1_data_votes", 72)
    st.historical_summaries = arr("historical_summaries", 64)
    st.validators = np.frombuffer(get("validators"), dtype=S.VALIDATOR_DTYPE).copy()
    st.balances = np.frombuffer(get("balances"), dtype="<u8").copy()
    st.slashings = np.frombuffer(get("slashings"), dtype="<u8").copy()
    st.inactivity_scores = np.frombuffer(get("inactivity_scores"), dtype="<u8").copy()
    st.previous_epoch_participation = np.frombuffer(get("previous_epoch_participation"), dtype=np.uint8).copy()
    st.current_epoch_participation = np.frombuffer(get("current_epoch_participation"), dtype=np.uint8).copy()
    st.current_sync_committee, st.next_sync_committee = get("current_sync_committee"), get("next_sync_committee")
    hdr = get("latest_execution_payload_header")
    st.payload_header_fixed, st.extra_data = hdr[:584], hdr[584:]
    return st


# ---------------------------------------------------------------------------------------------------------- update scripts
def _pinned(lay: Dict[str, tuple], lo: int, hi: int):
    """Positions in [lo, hi) whose value a patch must keep or constrain: the nine offsets and the header's extra_data
    offset (only their own value is an in-place update), `slashed` bytes (booleans) and justification_bits (4 bits)."""
    keep, bool_pos, bits4 = [], [], []
    for k, (o, ln) in lay.items():
        if k.startswith("offset:") and o < hi and lo < o + ln:
            keep += range(max(o, lo), min(o + ln, hi))
    ho = lay["latest_execution_payload_header"][0] + 436
    keep += [p for p in range(ho, ho + 4) if lo <= p < hi]
    vo, vl = lay["validators"]
    if vl and vo < hi and lo < vo + vl:
        first = max(0, (lo - vo - 88 + 120) // 121)
        for i in range(first, vl // 121):
            p = vo + 121 * i + 88
            if p >= hi:
                break
            if p >= lo:
                bool_pos.append(p)
    jb = lay["justification_bits"][0]
    if lo <= jb < hi:
        bits4.append(jb)
    return keep, bool_pos, bits4


def make_patch(host: np.ndarray, lay, lo: int, hi: int, rng) -> bytes:
    """Random new bytes for [lo, hi) that keep the serialization's layout and stay in every field's value range."""
    data = rng.integers(0, 256, hi - lo, dtype=np.uint8)
    keep, bool_pos, bits4 = _pinned(lay, lo, hi)
    for p in keep:
        data[p - lo] = host[p]
    for p in bool_pos:
        data[p - lo] &= 1
    for p in bits4:
        data[p - lo] &= 0x0f
    return data.tobytes()


def _elements(field: str, idx, rng, host, lay) -> bytes:
    """New SSZ encodings for elements `idx` of a big list."""
    w = ELEM[field]
    vals = rng.integers(0, 256, (len(idx), w), dtype=np.uint8)
    if field == "validators":
        vals[:, 88] &= 1
    return vals.tobytes()


def script(spec: dict, seed: int) -> List[tuple]:
    """An update script for the state `spec`: a list of
        ("elements", field, indices u64 array, values bytes) -> DeviceBeaconState.update_elements
        ("bytes", offset, data)                              -> DeviceBeaconState.update_bytes
        ("root", label)                                      -> check the incremental, full and oracle roots
    It is generated against a host copy so that patches keep offsets and value ranges; apply() replays it on bytes."""
    host = serialized(spec).copy()
    lay = layout_of(host, spec["preset"])
    rng = np.random.default_rng(seed)
    steps: List[tuple] = []

    def put_bytes(o, data, note):
        steps.append(("bytes", int(o), bytes(data), note))
        host[o:o + len(data)] = np.frombuffer(data, dtype=np.uint8)

    def put_elems(field, idx, note, vals=None):
        idx = np.asarray(idx, dtype=np.uint64)
        if vals is None:
            vals = _elements(field, idx, rng, host, lay)
        steps.append(("elements", field, idx, vals, note))
        apply(host, steps[-1], spec["preset"], lay)

    def root(label):
        if not steps or steps[-1][0] != "root":
            steps.append(("root", label))

    def count(f):
        return lay[f][1] // ELEM[f]

    fields_small = [f for f in FIELDS_28 if f not in BIG_LISTS]
    root("upload")
    # 1. every field of the 28: first element, last element, one whole 32-byte chunk
    for f in FIELDS_28:
        o, ln = lay[f]
        if ln == 0:
            continue
        if f in BIG_LISTS:
            n = count(f)
            put_elems(f, [0], f"{f}: first element")
            put_elems(f, [n - 1], f"{f}: last element")
            per = 32 // ELEM[f] if ELEM[f] < 32 else 1
            c = int(rng.integers(0, max(1, n // per)))
            idx = [i for i in range(c * per, min(n, c * per + per))]
            put_elems(f, idx, f"{f}: every element of chunk {c}")
        else:
            w = ELEM.get(f, ln)
            put_bytes(o, make_patch(host, lay, o, o + min(w, ln), rng), f"{f}: first element")
            put_bytes(o + ln - min(w, ln), make_patch(host, lay, o + ln - min(w, ln), o + ln, rng), f"{f}: last element")
            c = int(rng.integers(0, max(1, ln // 32)))
            a, z = o + 32 * c, min(o + ln, o + 32 * c + 32)
            if a < z:
                put_bytes(a, make_patch(host, lay, a, z, rng), f"{f}: bytes of chunk {c}")
        if f in ("validators", "historical_summaries", "latest_execution_payload_header", "slashings", "block_roots"):
            root(f"after {f}")
    root("every field")
    # 2. an unchanged value written back, and one element written twice before one root
    for f in CHAINS + fields_small[:4]:
        o, ln = lay[f]
        if ln == 0:
            continue
        if f in BIG_LISTS:
            i = int(rng.integers(0, count(f)))
            w = ELEM[f]
            put_elems(f, [i], f"{f}: unchanged element {i}", bytes(host[o + w * i: o + w * i + w]))
            put_elems(f, [i], f"{f}: element {i}, first write")
            put_elems(f, [i], f"{f}: element {i}, second write")
        else:
            put_bytes(o, bytes(host[o:o + min(ln, 40)]), f"{f}: unchanged bytes")
            put_bytes(o, make_patch(host, lay, o, o + min(ln, 8), rng), f"{f}: first write")
            put_bytes(o, make_patch(host, lay, o, o + min(ln, 8), rng), f"{f}: second write")
    root("unchanged values and double writes")
    # 3. a patch straddling every pair of adjacent parts of the serialization (offsets keep their own value)
    parts = sorted(lay.items(), key=lambda kv: kv[1][0])
    for (fa, (oa, la)), (fb, (ob, lb)) in zip(parts, parts[1:]):
        if oa + la != ob:
            continue
        lo = max(0, ob - int(rng.integers(1, 40)))
        hi = min(len(host), ob + int(rng.integers(1, 40)))
        put_bytes(lo, make_patch(host, lay, lo, hi, rng), f"straddle {fa} | {fb}")
    root("straddling patches")
    # 4. many dirty inputs: > 256 at every level a list has, in all lists at once
    for f in BIG_LISTS:
        n = count(f)
        if n:
            k = min(n, n_scaled(4096))
            put_elems(f, np.sort(rng.choice(n, k, replace=False)), f"{f}: {k} scattered elements")
    for f in ("block_roots", "randao_mixes"):
        o, ln = lay[f]
        for c in np.sort(rng.choice(ln // 32, min(ln // 32, 300), replace=False)):
            put_bytes(o + 32 * int(c), rng.integers(0, 256, 32, dtype=np.uint8).tobytes(), f"{f}: chunk {c}")
    root("many dirty inputs")
    # 5. whole-list rewrites: each list once (big lists through update_elements, the rest through bytes)
    for f in CHAINS + ["historical_roots", "eth1_data_votes", "historical_summaries"]:
        o, ln = lay[f]
        if ln == 0:
            continue
        if f in BIG_LISTS:
            put_elems(f, np.arange(count(f)), f"{f}: whole list")
        else:
            put_bytes(o, make_patch(host, lay, o, o + ln, rng), f"{f}: whole field")
    root("whole-list rewrites")
    # 6. the whole serialization rewritten in place with the same lengths
    other = dict(spec, seed=spec["seed"] ^ seed ^ 0x5A5A)
    other["extra"] = bytes((x + 1) & 0xff for x in spec["extra"])
    new = serialized(other)
    assert len(new) == len(host)
    put_bytes(0, new.tobytes(), "whole serialization, same layout")
    root("whole serialization")
    return steps


def apply(host: np.ndarray, step: tuple, preset: str, lay=None) -> None:
    """Applies one script step to the host bytes."""
    if step[0] == "bytes":
        o, data = step[1], step[2]
        host[o:o + len(data)] = np.frombuffer(data, dtype=np.uint8)
    elif step[0] == "elements":
        f, idx, vals = step[1], step[2], step[3]
        lay = lay or layout_of(host, preset)
        o, w = lay[f][0], ELEM[f]
        v = np.frombuffer(vals, dtype=np.uint8).reshape(-1, w)
        pos = o + w * idx.astype(np.int64)
        for k in range(w):
            host[pos + k] = v[:, k]


def script_specs() -> List[dict]:
    """States the update scripts run on (a subset of state_specs: both presets, every hand-off and the coop limit)."""
    want = {("minimal", 5), ("minimal", 65), ("minimal", 257), ("minimal", 2049), ("mainnet", 0), ("mainnet", 257),
            ("mainnet", 65537), ("mainnet", COOP_MAX + 1)}
    return [s for s in state_specs() if (s["preset"], s["n"]) in want]


def script_fields_covered(steps, lay) -> set:
    """Names of the 28 fields some write of the script touches."""
    hit = set()
    spans = [(f, lay[f]) for f in FIELDS_28]
    for st in steps:
        if st[0] == "elements":
            hit.add(st[1])
        elif st[0] == "bytes":
            lo, hi = st[1], st[1] + len(st[2])
            for f, (o, ln) in spans:
                if ln and o < hi and lo < o + ln:
                    hit.add(f)
    return hit


# ---------------------------------------------------------------------------------------------------------- malformed
def malformed_cases() -> List[tuple]:
    """(name, preset, bytes, should_accept).  Built from valid states; `should_accept` marks the controls (re-partitions
    and edge values the SSZ rules allow) that sit next to each rejected encoding."""
    out = []
    for preset, n in (("minimal", 5), ("mainnet", 3)):
        bound = S.PRESETS[preset]["ETH1_DATA_VOTES_BOUND"]
        spec = dict(preset=preset, n=n, hr=2, hs=3, votes=3, extra=b"xyz!", seed=0xBAD0 + n)
        good = serialized(spec)
        fl = fixed_len(preset)
        offs = offset_positions(preset)

        def with_off(k, v, base=None):
            b = (good if base is None else base).copy()
            b[offs[k]: offs[k] + 4] = np.frombuffer(struct.pack("<I", v & 0xffffffff), dtype=np.uint8)
            return b

        def off(k, base=None):
            b = good if base is None else base
            return struct.unpack_from("<I", bytes(b[offs[k]: offs[k] + 4]))[0]

        P = preset
        out.append((f"{P}: valid", P, good, True))
        out.append((f"{P}: first offset fixed + 32", P, with_off(0, fl + 32), False))
        out.append((f"{P}: first offset fixed - 1", P, with_off(0, fl - 1), False))
        out.append((f"{P}: first offset 0", P, with_off(0, 0), False))
        for k in range(1, 9):
            out.append((f"{P}: offset {k} below offset {k - 1}", P, with_off(k, off(k - 1) - 1), False))
            out.append((f"{P}: offset {k} beyond len", P, with_off(k, len(good) + 1), False))
        out.append((f"{P}: last offset = len + 64", P, with_off(8, len(good) + 64), False))
        out.append((f"{P}: offsets 2 and 3 swapped", P, with_off(3, off(2), with_off(2, off(3))), False))
        # list byte lengths that are not a multiple of the element size
        out.append((f"{P}: historical_roots 33 bytes", P, with_off(1, off(1) + 1), False))
        out.append((f"{P}: eth1_data_votes not x 72", P, with_off(2, off(2) + 1), False))
        out.append((f"{P}: validators not x 121", P, with_off(3, off(3) - 8), False))
        out.append((f"{P}: balances not x 8", P, with_off(4, off(4) + 1), False))
        out.append((f"{P}: inactivity_scores not x 8", P, with_off(7, off(7) - 4), False))
        out.append((f"{P}: historical_summaries not x 64", P, good[:-1].copy(), False))
        out.append((f"{P}: historical_summaries + 1 byte", P, np.append(good, np.uint8(0)), False))
        out.append((f"{P}: historical_summaries + 64 bytes", P, np.append(good, np.zeros(64, np.uint8)), True))
        out.append((f"{P}: participation re-split by one byte", P, with_off(5, off(5) + 1), True))
        out.append((f"{P}: validators x 121 moved into balances", P, with_off(3, off(3) - 121 + 0), False))
        # eth1_data_votes at and above the bound
        for votes, ok in ((bound, True), (bound + 1, False)):
            out.append((f"{P}: {votes} eth1_data_votes", P, serialized(dict(spec, votes=votes)), ok))
        # ExecutionPayloadHeader: short fixed part, too much extra_data, wrong internal offset
        st = state_for(spec)
        for hdr_len, ok in ((583, False), (580, False), (0, False)):
            s2 = state_for(spec)
            s2.payload_header_fixed, s2.extra_data = st.payload_header_fixed[:hdr_len], b""
            out.append((f"{P}: payload header {hdr_len} bytes", P, S.serialize(s2), ok))
        for ex, ok in ((0, True), (32, True), (33, False), (64, False)):
            s2 = state_for(spec)
            s2.extra_data = bytes(range(ex))
            out.append((f"{P}: extra_data {ex} bytes", P, S.serialize(s2), ok))
        for v, ok in ((585, False), (583, False), (0, False), (584 + (1 << 16), False)):
            s2 = state_for(spec)
            s2.payload_header_fixed = st.payload_header_fixed[:436] + struct.pack("<I", v) + st.payload_header_fixed[440:]
            out.append((f"{P}: payload header extra_data offset {v}", P, S.serialize(s2), ok))
        # a truncated fixed part
        for cut in (1, 100, fl // 2, fl - 1):
            out.append((f"{P}: truncated to {cut} bytes", P, good[:cut].copy(), False))
        out.append((f"{P}: fixed part only, every list empty", P, _empty_lists(good, preset), False))
    return out


def _empty_lists(good: np.ndarray, preset: str) -> np.ndarray:
    """The fixed part with every offset = fixed length: every list empty, but the header's 584 bytes missing."""
    fl = fixed_len(preset)
    b = good[:fl].copy()
    for p in offset_positions(preset):
        b[p:p + 4] = np.frombuffer(struct.pack("<I", fl), dtype=np.uint8)
    return b


# ---------------------------------------------------------------------------------------------------------- shuffling
SEEDS = {"zero": bytes(32), "ff": b"\xff" * 32, "random": hashlib.sha256(b"ssz soak shuffle seed").digest()}
ROUNDS = [0, 1, 2, 10, 90, 255]


def shuffle_sizes() -> List[int]:
    sizes = list(range(0, 21))
    for k in range(8, 22):
        sizes += [(1 << k) - 1, 1 << k, (1 << k) + 1]
    return sizes


def shuffle_cases() -> List[dict]:
    """(n, rounds, seed name, identity or full 64-bit index list).  Every (rounds, seed) pair on the sizes up to 4 097;
    above that one pair per size, chosen so that every round count still meets sizes near 2^k, and the heavy round counts
    stay on sizes up to 2^17."""
    out = []
    pairs = [(r, s) for r in ROUNDS for s in SEEDS]
    for i, n in enumerate(shuffle_sizes()):
        if n <= 4097:
            for j, (r, s) in enumerate(pairs):
                out.append(dict(n=n, rounds=r, seed=s, values=(j % 3 == 0), vseed=1000 * n + j))
        else:
            light = [p for p in pairs if p[0] <= (90 if n <= (1 << 17) + 1 else 10)]
            r, s = light[i % len(light)]
            out.append(dict(n=n, rounds=r, seed=s, values=(i % 2 == 0), vseed=1000 * n))
    return out


def shuffle_values(case: dict):
    """The index list of a case: None for the identity, else full 64-bit values."""
    if not case["values"]:
        return None
    rng = np.random.default_rng(case["vseed"])
    v = rng.integers(0, 1 << 64, case["n"], dtype=np.uint64, endpoint=False)
    if case["n"]:
        v[0] = np.uint64((1 << 64) - 1)
    return v


def registry_cases() -> List[dict]:
    """Validator registries for get_active_validator_indices: (name, n, pattern, epoch list).  Epochs fall exactly on
    activation_epoch and exit_epoch; the patterns change at warp (32) and CTA (256) edges; 262 145 and 2^20 records reach
    k_active_scan's multi-block branch (more than 1 024 CTAs)."""
    E = 1000
    out = []
    for n in (1, 31, 32, 33, 255, 256, 257, 1000):
        for pat in ("all", "none", "edges", "runs", "random"):
            out.append(dict(name=f"{pat}:{n}", n=n, pattern=pat, epochs=[0, E - 1, E, E + 1, FAR - 1, FAR]))
    for n in (70_001, SCAN_CTAS * CTA - 1, SCAN_CTAS * CTA, SCAN_CTAS * CTA + 1, 1 << 20):
        out.append(dict(name=f"runs:{n}", n=n, pattern="runs", epochs=[E - 1, E, E + 1]))
        out.append(dict(name=f"random:{n}", n=n, pattern="random", epochs=[E]))
    out.append(dict(name=f"all:{SCAN_CTAS * CTA + 1}", n=SCAN_CTAS * CTA + 1, pattern="all", epochs=[E]))
    out.append(dict(name=f"none:{1 << 20}", n=1 << 20, pattern="none", epochs=[E]))
    return out


def registry_epochs(n: int, pattern: str, seed: int = 7, E: int = 1000):
    """(activation_epoch, exit_epoch) arrays.  'edges': every record sits on a boundary of epoch E (activation = E, exit =
    E, exit = E + 1, activation = E + 1, ...); 'runs': active / inactive runs of 31, 32, 33, 255, 256, 257 records."""
    rng = np.random.default_rng(seed + n)
    act = np.zeros(n, dtype=np.uint64)
    ext = np.full(n, FAR, dtype=np.uint64)
    if pattern == "none":
        act[:] = FAR
    elif pattern == "edges":
        kinds = np.arange(n) % 6
        act[kinds == 0] = E                        # active from E
        ext[kinds == 1] = E                        # exited at E
        ext[kinds == 2] = E + 1                    # last active epoch E
        act[kinds == 3] = E + 1                    # not yet active at E
        act[kinds == 4] = E - 1; ext[kinds == 4] = E
        act[kinds == 5] = FAR - 1                  # active only at FAR - 1
    elif pattern == "runs":
        runs = [31, 32, 33, 255, 256, 257]
        pos, k, on = 0, 0, True
        while pos < n:
            ln = runs[k % len(runs)]
            if not on:
                (act if k % 4 < 2 else ext)[pos:pos + ln] = E + 1 if k % 4 < 2 else E
            pos += ln; k += 1; on = not on
    elif pattern == "random":
        act = rng.integers(E - 3, E + 3, n, dtype=np.uint64)
        ext = np.where(rng.integers(0, 4, n) == 0, rng.integers(E - 2, E + 4, n, dtype=np.uint64), np.uint64(FAR))
    return act, ext


def registry(n: int, pattern: str) -> np.ndarray:
    """n SSZ Validator records (n x 121 uint8) with the pattern's epochs."""
    v = np.zeros(n, dtype=S.VALIDATOR_DTYPE)
    if n:
        rng = np.random.default_rng(n)
        v["public_key"] = rng.integers(0, 256, (n, 48), dtype=np.uint8).view("V48").reshape(n)
        v["effective_balance"] = 32 * 10**9
        act, ext = registry_epochs(n, pattern)
        v["activation_epoch"], v["exit_epoch"] = act, ext
    return v.view(np.uint8).reshape(-1)


def active_numpy(recs: np.ndarray, epoch: int) -> np.ndarray:
    """get_active_validator_indices over N x 121 bytes, vectorised (pinned to shuffle_oracle's loop by the CPU test)."""
    v = np.ascontiguousarray(recs).view(S.VALIDATOR_DTYPE)
    e = np.uint64(epoch)
    return np.nonzero((v["activation_epoch"] <= e) & (e < v["exit_epoch"]))[0].astype(np.uint64)
