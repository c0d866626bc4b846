"""Synthetic deneb `BeaconState` instances (numpy) and their SSZ serialization.

Field order and sizes follow ethereum-consensus/src/deneb/beacon_state.rs:26-63 and the presets
(ethereum-consensus/src/phase0/presets/mainnet.rs:5-36,82-83, altair/presets/mainnet.rs:19).
Used by bench.py (config 3 of BASELINE.json: 2**20 validators) and by the parity tests.  Data is synthetic:
pubkeys are pseudo-random 48-byte strings unless `pubkeys=` is given (hashing does not interpret them).
"""
from __future__ import annotations

import hashlib
from dataclasses import dataclass, field
from typing import Dict

import numpy as np

PRESETS: Dict[str, Dict[str, int]] = {
    "mainnet": dict(SLOTS_PER_HISTORICAL_ROOT=8192, HISTORICAL_ROOTS_LIMIT=1 << 24, ETH1_DATA_VOTES_BOUND=2048,
                    VALIDATOR_REGISTRY_LIMIT=1 << 40, EPOCHS_PER_HISTORICAL_VECTOR=65536,
                    EPOCHS_PER_SLASHINGS_VECTOR=8192, SYNC_COMMITTEE_SIZE=512),
    "minimal": dict(SLOTS_PER_HISTORICAL_ROOT=64, HISTORICAL_ROOTS_LIMIT=1 << 24, ETH1_DATA_VOTES_BOUND=32,
                    VALIDATOR_REGISTRY_LIMIT=1 << 40, EPOCHS_PER_HISTORICAL_VECTOR=64,
                    EPOCHS_PER_SLASHINGS_VECTOR=64, SYNC_COMMITTEE_SIZE=32),
}

# SSZ `Validator` (121 bytes) — ethereum-consensus/src/phase0/validator.rs:10-26
VALIDATOR_DTYPE = np.dtype([
    ("public_key", "V48"), ("withdrawal_credentials", "V32"), ("effective_balance", "<u8"), ("slashed", "u1"),
    ("activation_eligibility_epoch", "<u8"), ("activation_epoch", "<u8"), ("exit_epoch", "<u8"),
    ("withdrawable_epoch", "<u8")])
assert VALIDATOR_DTYPE.itemsize == 121

FAR_FUTURE_EPOCH = (1 << 64) - 1


@dataclass
class SynthState:
    preset: str
    fixed: Dict[str, bytes] = field(default_factory=dict)     # small fixed-size fields, already serialized
    block_roots: np.ndarray = None
    state_roots: np.ndarray = None
    historical_roots: np.ndarray = None        # (n,32) u8
    eth1_data_votes: np.ndarray = None         # (n,72) u8
    validators: np.ndarray = None              # VALIDATOR_DTYPE
    balances: np.ndarray = None                # <u8
    randao_mixes: np.ndarray = None            # (n,32) u8
    slashings: np.ndarray = None               # <u8
    previous_epoch_participation: np.ndarray = None  # u1
    current_epoch_participation: np.ndarray = None
    inactivity_scores: np.ndarray = None       # <u8
    current_sync_committee: bytes = b""        # 48*(size+1)
    next_sync_committee: bytes = b""
    payload_header_fixed: bytes = b""          # 584 bytes incl. the extra_data offset
    extra_data: bytes = b""
    historical_summaries: np.ndarray = None    # (n,64) u8


def _rand_bytes(rng: np.random.Generator, n: int, width: int) -> np.ndarray:
    return rng.integers(0, 256, size=(n, width), dtype=np.uint8)


def synth_state(n_validators: int, preset: str = "mainnet", seed: int = 0xB200, n_eth1_votes: int | None = None,
                n_historical_summaries: int = 300, n_historical_roots: int = 0, pubkeys: np.ndarray | None = None,
                extra_data: bytes = b"b200") -> SynthState:
    """Config 3 of BASELINE.json (SURVEY.md §8d): deterministic pseudo-random deneb state with `n_validators`."""
    P = PRESETS[preset]
    rng = np.random.default_rng(seed)
    n = n_validators
    if n_eth1_votes is None:
        n_eth1_votes = P["ETH1_DATA_VOTES_BOUND"] // 2
    st = SynthState(preset=preset)
    v = np.zeros(n, dtype=VALIDATOR_DTYPE)
    pk = _rand_bytes(rng, n, 48) if pubkeys is None else np.ascontiguousarray(pubkeys, dtype=np.uint8).reshape(n, 48)
    v["public_key"] = pk.view("V48").reshape(n)
    wc = _rand_bytes(rng, n, 32)
    wc[:, 0] = 1
    wc[:, 1:12] = 0
    v["withdrawal_credentials"] = wc.view("V32").reshape(n)
    v["effective_balance"] = 32 * 10**9
    v["slashed"] = (rng.integers(0, 1024, size=n) == 0).astype(np.uint8)
    v["activation_eligibility_epoch"] = rng.integers(0, 1 << 18, size=n, dtype=np.uint64)
    v["activation_epoch"] = rng.integers(0, 1 << 18, size=n, dtype=np.uint64)
    exited = rng.integers(0, 100, size=n) == 0
    v["exit_epoch"] = np.where(exited, rng.integers(0, 1 << 18, size=n, dtype=np.uint64), np.uint64(FAR_FUTURE_EPOCH))
    v["withdrawable_epoch"] = np.where(exited, rng.integers(0, 1 << 18, size=n, dtype=np.uint64), np.uint64(FAR_FUTURE_EPOCH))
    st.validators = v
    st.balances = (32 * 10**9 + rng.integers(0, 10**9, size=n, dtype=np.uint64)).astype("<u8")
    st.previous_epoch_participation = rng.integers(0, 8, size=n, dtype=np.uint8)
    st.current_epoch_participation = rng.integers(0, 8, size=n, dtype=np.uint8)
    st.inactivity_scores = np.where(rng.integers(0, 20, size=n) == 0, rng.integers(0, 100, size=n), 0).astype("<u8")
    st.block_roots = _rand_bytes(rng, P["SLOTS_PER_HISTORICAL_ROOT"], 32)
    st.state_roots = _rand_bytes(rng, P["SLOTS_PER_HISTORICAL_ROOT"], 32)
    st.randao_mixes = _rand_bytes(rng, P["EPOCHS_PER_HISTORICAL_VECTOR"], 32)
    st.slashings = np.zeros(P["EPOCHS_PER_SLASHINGS_VECTOR"], dtype="<u8")
    st.slashings[::97] = 10**9
    st.historical_roots = _rand_bytes(rng, n_historical_roots, 32)
    votes = _rand_bytes(rng, n_eth1_votes, 72)
    votes[:, 32:40] = np.frombuffer(np.arange(n_eth1_votes, dtype="<u8").tobytes(), dtype=np.uint8).reshape(-1, 8)
    st.eth1_data_votes = votes
    st.historical_summaries = _rand_bytes(rng, n_historical_summaries, 64)
    sc = P["SYNC_COMMITTEE_SIZE"]
    idx = np.arange(sc) % max(n, 1)
    keys = pk[idx] if n else np.zeros((sc, 48), np.uint8)
    st.current_sync_committee = keys.tobytes() + hashlib.sha256(b"agg0").digest() + bytes(16)
    st.next_sync_committee = keys[::-1].tobytes() + hashlib.sha256(b"agg1").digest() + bytes(16)
    h = lambda tag: hashlib.sha256(tag).digest()  # noqa: E731
    u64 = lambda x: int(x).to_bytes(8, "little")  # noqa: E731
    st.fixed = {
        "genesis_time": u64(1606824023),
        "genesis_validators_root": h(b"gvr"),
        "slot": u64(8_626_176),
        "fork": bytes.fromhex("03000000") + bytes.fromhex("04000000") + u64(269568),
        "latest_block_header": u64(8_626_175) + u64(12345 % max(n, 1)) + h(b"parent") + bytes(32) + h(b"body"),
        "eth1_data": h(b"deposit_root") + u64(n) + h(b"eth1_block"),
        "eth1_deposit_index": u64(n),
        "justification_bits": bytes([0b0111]),
        "previous_justified_checkpoint": u64(269566) + h(b"pj"),
        "current_justified_checkpoint": u64(269567) + h(b"cj"),
        "finalized_checkpoint": u64(269566) + h(b"fin"),
        "next_withdrawal_index": u64(31_000_000),
        "next_withdrawal_validator_index": u64(777 % max(n, 1)),
    }
    st.extra_data = extra_data
    st.payload_header_fixed = (
        h(b"parent_hash") + h(b"fee")[:20] + h(b"state_root") + h(b"receipts") + rng.integers(0, 256, 256, dtype=np.uint8).tobytes()
        + h(b"randao") + u64(19_000_000) + u64(30_000_000) + u64(12_345_678) + u64(1_710_000_000) + (584).to_bytes(4, "little")
        + (7 * 10**9).to_bytes(32, "little") + h(b"block_hash") + h(b"txroot") + h(b"wroot") + u64(131072) + u64(0))
    assert len(st.payload_header_fixed) == 584
    return st


def serialize(st: SynthState) -> np.ndarray:
    """SSZ bytes of the state as a contiguous uint8 array (fixed part with 4-byte offsets, then the 9 variable fields)."""
    f = st.fixed
    var = [st.historical_roots.tobytes(), st.eth1_data_votes.tobytes(), st.validators.tobytes(), st.balances.tobytes(),
           st.previous_epoch_participation.tobytes(), st.current_epoch_participation.tobytes(),
           st.inactivity_scores.tobytes(), st.payload_header_fixed + st.extra_data, st.historical_summaries.tobytes()]
    OFF = object()
    parts = [f["genesis_time"], f["genesis_validators_root"], f["slot"], f["fork"], f["latest_block_header"],
             st.block_roots.tobytes(), st.state_roots.tobytes(), OFF, f["eth1_data"], OFF, f["eth1_deposit_index"], OFF, OFF,
             st.randao_mixes.tobytes(), st.slashings.tobytes(), OFF, OFF, f["justification_bits"],
             f["previous_justified_checkpoint"], f["current_justified_checkpoint"], f["finalized_checkpoint"], OFF,
             st.current_sync_committee, st.next_sync_committee, OFF, f["next_withdrawal_index"],
             f["next_withdrawal_validator_index"], OFF]
    fixed_len = sum(4 if p is OFF else len(p) for p in parts)
    total = fixed_len + sum(len(x) for x in var)
    out = np.empty(total, dtype=np.uint8)
    pos, voff, vi = 0, fixed_len, 0
    for p in parts:
        if p is OFF:
            out[pos:pos + 4] = np.frombuffer(int(voff).to_bytes(4, "little"), dtype=np.uint8)
            voff += len(var[vi]); vi += 1; pos += 4
        else:
            out[pos:pos + len(p)] = np.frombuffer(p, dtype=np.uint8); pos += len(p)
    for x in var:
        out[pos:pos + len(x)] = np.frombuffer(x, dtype=np.uint8); pos += len(x)
    assert pos == total
    return out


def layout(st: SynthState) -> Dict[str, tuple]:
    """{field: (byte offset, byte length)} of every part of `serialize(st)` — the coordinates `b200_state_update_bytes`
    takes (variable-size fields by name, fixed-size ones by the names used in `SynthState.fixed`)."""
    names_var = ["historical_roots", "eth1_data_votes", "validators", "balances", "previous_epoch_participation",
                 "current_epoch_participation", "inactivity_scores", "latest_execution_payload_header", "historical_summaries"]
    var_len = [st.historical_roots.nbytes, st.eth1_data_votes.nbytes, st.validators.nbytes, st.balances.nbytes,
               st.previous_epoch_participation.nbytes, st.current_epoch_participation.nbytes, st.inactivity_scores.nbytes,
               len(st.payload_header_fixed) + len(st.extra_data), st.historical_summaries.nbytes]
    f = st.fixed
    OFF = None
    parts = [("genesis_time", len(f["genesis_time"])), ("genesis_validators_root", 32), ("slot", 8), ("fork", len(f["fork"])),
             ("latest_block_header", len(f["latest_block_header"])), ("block_roots", st.block_roots.nbytes),
             ("state_roots", st.state_roots.nbytes), OFF, ("eth1_data", len(f["eth1_data"])), OFF, ("eth1_deposit_index", 8), OFF, OFF,
             ("randao_mixes", st.randao_mixes.nbytes), ("slashings", st.slashings.nbytes), OFF, OFF, ("justification_bits", 1),
             ("previous_justified_checkpoint", 40), ("current_justified_checkpoint", 40), ("finalized_checkpoint", 40), OFF,
             ("current_sync_committee", len(st.current_sync_committee)), ("next_sync_committee", len(st.next_sync_committee)), OFF,
             ("next_withdrawal_index", 8), ("next_withdrawal_validator_index", 8), OFF]
    out, pos, k = {}, 0, 0
    for p in parts:
        if p is OFF:
            out["offset:" + names_var[k]] = (pos, 4); k += 1; pos += 4
        else:
            out[p[0]] = (pos, p[1]); pos += p[1]
    for name, ln in zip(names_var, var_len):
        out[name] = (pos, ln); pos += ln
    return out


def to_oracle_value(st: SynthState) -> dict:
    """The same state as the dict-of-python-values the oracle's SSZ type system consumes (small N only)."""
    f = st.fixed
    def cp(b): return {"epoch": int.from_bytes(b[:8], "little"), "root": b[8:]}
    def sync(b, size): return {"public_keys": [b[48 * i:48 * i + 48] for i in range(size)], "aggregate_public_key": b[48 * size:]}
    size = PRESETS[st.preset]["SYNC_COMMITTEE_SIZE"]
    ph = st.payload_header_fixed
    names = VALIDATOR_DTYPE.names
    vals = []
    for rec in st.validators:
        d = {}
        for nme in names:
            x = rec[nme]
            d[nme] = x.tobytes() if nme in ("public_key", "withdrawal_credentials") else (bool(x) if nme == "slashed" else int(x))
        vals.append(d)
    hb = f["latest_block_header"]
    return {
        "genesis_time": int.from_bytes(f["genesis_time"], "little"),
        "genesis_validators_root": f["genesis_validators_root"],
        "slot": int.from_bytes(f["slot"], "little"),
        "fork": {"previous_version": f["fork"][:4], "current_version": f["fork"][4:8], "epoch": int.from_bytes(f["fork"][8:], "little")},
        "latest_block_header": {"slot": int.from_bytes(hb[:8], "little"), "proposer_index": int.from_bytes(hb[8:16], "little"),
                                "parent_root": hb[16:48], "state_root": hb[48:80], "body_root": hb[80:112]},
        "block_roots": [r.tobytes() for r in st.block_roots],
        "state_roots": [r.tobytes() for r in st.state_roots],
        "historical_roots": [r.tobytes() for r in st.historical_roots],
        "eth1_data": {"deposit_root": f["eth1_data"][:32], "deposit_count": int.from_bytes(f["eth1_data"][32:40], "little"), "block_hash": f["eth1_data"][40:]},
        "eth1_data_votes": [{"deposit_root": r[:32].tobytes(), "deposit_count": int.from_bytes(r[32:40].tobytes(), "little"),
                             "block_hash": r[40:].tobytes()} for r in st.eth1_data_votes],
        "eth1_deposit_index": int.from_bytes(f["eth1_deposit_index"], "little"),
        "validators": vals,
        "balances": [int(x) for x in st.balances],
        "randao_mixes": [r.tobytes() for r in st.randao_mixes],
        "slashings": [int(x) for x in st.slashings],
        "previous_epoch_participation": [int(x) for x in st.previous_epoch_participation],
        "current_epoch_participation": [int(x) for x in st.current_epoch_participation],
        "justification_bits": [bool((f["justification_bits"][0] >> i) & 1) for i in range(4)],
        "previous_justified_checkpoint": cp(f["previous_justified_checkpoint"]),
        "current_justified_checkpoint": cp(f["current_justified_checkpoint"]),
        "finalized_checkpoint": cp(f["finalized_checkpoint"]),
        "inactivity_scores": [int(x) for x in st.inactivity_scores],
        "current_sync_committee": sync(st.current_sync_committee, size),
        "next_sync_committee": sync(st.next_sync_committee, size),
        "latest_execution_payload_header": {
            "parent_hash": ph[0:32], "fee_recipient": ph[32:52], "state_root": ph[52:84], "receipts_root": ph[84:116],
            "logs_bloom": ph[116:372], "prev_randao": ph[372:404], "block_number": int.from_bytes(ph[404:412], "little"),
            "gas_limit": int.from_bytes(ph[412:420], "little"), "gas_used": int.from_bytes(ph[420:428], "little"),
            "timestamp": int.from_bytes(ph[428:436], "little"), "extra_data": st.extra_data,
            "base_fee_per_gas": int.from_bytes(ph[440:472], "little"), "block_hash": ph[472:504],
            "transactions_root": ph[504:536], "withdrawals_root": ph[536:568],
            "blob_gas_used": int.from_bytes(ph[568:576], "little"), "excess_blob_gas": int.from_bytes(ph[576:584], "little")},
        "next_withdrawal_index": int.from_bytes(f["next_withdrawal_index"], "little"),
        "next_withdrawal_validator_index": int.from_bytes(f["next_withdrawal_validator_index"], "little"),
        "historical_summaries": [{"block_summary_root": r[:32].tobytes(), "state_summary_root": r[32:].tobytes()}
                                 for r in st.historical_summaries],
    }
