"""Seeded step scripts that change the shape of a deneb BeaconState the way blocks do (no device code, no torch).

A step is one call of the device-resident state's API (ethereum_consensus_b200.ssz.DeviceBeaconState), applied to a host
mirror (state.SynthState) by `apply` in the same way:
  ("push", field, bytes)             append_elements (the spec's `.push`)
  ("set", field, bytes)              set_field (eth1_data_votes, latest_execution_payload_header)
  ("deposits", records, balances)    add_validators: one deposit batch across the five big lists
  ("elements", field, idx, bytes)    update_elements
  ("bytes", offset, bytes)           update_bytes at an offset of the serialization as it is at that step
A refused step raises state.ReshapeRefused from `apply`; the library must refuse it with the matching code and leave the
handle as it was.

Scripts are generators over the mirror they shape: after each yielded step the caller applies it (to the mirror and,
on the GPU, to the device), and the next step is computed from the mirror as it now is — so update_bytes offsets follow
every reshape, and indexed writes can hit validators appended in the same block.

tests/test_state_reshape_cases.py checks the scripts on the CPU (both oracles agree after every step, every boundary is
among them, refusals are recognised); tests/test_state_reshape_gpu.py runs them through the CUDA library.
"""
from __future__ import annotations

import sys
from pathlib import Path
from typing import Dict, Iterator, List

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from ethereum_consensus_b200 import state as S  # noqa: E402
from tests import ssz_soak_cases as sc  # noqa: E402

HANDOFF = sc.HANDOFF
COOP_MAX = sc.COOP_MAX
HEADROOM_MIN = 1 << 16        # capi_ssz.cu headroom(): a big list's reserved elements beyond its upload length
MAX_DEPOSITS = 16             # MAX_DEPOSITS per block


def headroom(n: int) -> int:
    return max(HEADROOM_MIN, n // 16)


# ---------------------------------------------------------------------------------------------------------- the mirror
def apply(st: S.SynthState, step: tuple) -> None:
    """Apply one step to the host mirror; raises state.ReshapeRefused where the library refuses."""
    kind = step[0]
    if kind == "push":
        st.append_elements(step[1], step[2])
    elif kind == "set":
        st.set_field(step[1], step[2])
    elif kind == "deposits":
        st.add_validators(step[1], step[2])
    elif kind == "elements":
        field, idx, vals = step[1], np.asarray(step[2], dtype=np.uint64), step[3]
        arr = getattr(st, field)
        if len(idx) and int(idx.max()) >= len(arr):
            raise S.ReshapeRefused("bad_arg", f"{field}: index beyond the list")
        new = np.frombuffer(bytes(vals), dtype=arr.dtype)
        arr[idx.astype(np.int64)] = new
    elif kind == "bytes":
        off, data = step[1], bytes(step[2])
        b = S.serialize(st)
        if off + len(data) > b.size:
            raise S.ReshapeRefused("bad_arg", "update_bytes beyond the serialization")
        pos = sc.offset_positions(st.preset)
        before = [bytes(b[p:p + 4]) for p in pos]
        hdr = sc.layout_of(b, st.preset)["latest_execution_payload_header"][0] + 436
        hdr_before = bytes(b[hdr:hdr + 4])
        b[off:off + len(data)] = np.frombuffer(data, dtype=np.uint8)
        if [bytes(b[p:p + 4]) for p in pos] != before or bytes(b[hdr:hdr + 4]) != hdr_before:
            raise S.ReshapeRefused("bad_arg", "update_bytes changes a variable-size field's offset")
        st.__dict__.update(sc.deserialize(b, st.preset).__dict__)
    else:
        raise ValueError(kind)


# ---------------------------------------------------------------------------------------------------------- step values
def validator_records(rng, n: int, epoch: int) -> np.ndarray:
    """`n` fresh Validator records (as add_validator_to_registry makes them: not yet active), a share of them with an
    activation epoch <= `epoch` so that the shuffling sees some of them as active."""
    v = np.zeros(n, dtype=S.VALIDATOR_DTYPE)
    v["public_key"] = rng.integers(0, 256, (n, 48), dtype=np.uint8).view("V48").reshape(n)
    wc = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    wc[:, 0] = 1
    v["withdrawal_credentials"] = wc.view("V32").reshape(n)
    v["effective_balance"] = 32 * 10**9
    active = rng.integers(0, 2, n).astype(bool)
    far = np.uint64(S.FAR_FUTURE_EPOCH)
    v["activation_eligibility_epoch"] = np.where(active, np.uint64(max(0, epoch - 2)), far)
    v["activation_epoch"] = np.where(active, np.uint64(max(0, epoch - 1)), far)
    v["exit_epoch"] = S.FAR_FUTURE_EPOCH
    v["withdrawable_epoch"] = S.FAR_FUTURE_EPOCH
    return v


def vote(rng, k: int) -> bytes:
    return rng.integers(0, 256, 32, dtype=np.uint8).tobytes() + int(k).to_bytes(8, "little") + \
        rng.integers(0, 256, 32, dtype=np.uint8).tobytes()


def header(rng, extra_len: int, block: int) -> bytes:
    h = bytearray(rng.integers(0, 256, 584, dtype=np.uint8).tobytes())
    h[404:412] = int(block).to_bytes(8, "little")
    h[436:440] = (584).to_bytes(4, "little")
    return bytes(h) + bytes((block * 13 + j) & 0xff for j in range(extra_len))


def deposits(rng, n: int, epoch: int) -> tuple:
    recs = validator_records(rng, n, epoch)
    bal = (32 * 10**9 + rng.integers(0, 10**6, n, dtype=np.uint64)).astype("<u8")
    return ("deposits", recs.tobytes(), bal)


def _u64s(rng, n, hi=1 << 40) -> bytes:
    return rng.integers(0, hi, n, dtype=np.uint64).astype("<u8").tobytes()


# ---------------------------------------------------------------------------------------------------------- scripts
def initial_state(preset: str, n: int, seed: int, votes: int = 0, summaries: int = 3) -> S.SynthState:
    return S.synth_state(n, preset, seed=seed, n_eth1_votes=votes, n_historical_summaries=summaries, extra_data=b"")


def chain_walk(st: S.SynthState, n_blocks: int, seed: int, start_slot: int = 0) -> Iterator[tuple]:
    """Deneb-shaped blocks on `st`: per block one eth1 vote (the list is reset every EPOCHS_PER_ETH1_VOTING_PERIOD x
    SLOTS_PER_EPOCH slots, i.e. at its bound), a new payload header whose extra_data length cycles through 0..32,
    0..16 deposits, balances and participation writes (some at validators appended in the same block), slot /
    block_roots / state_roots / randao_mixes through update_bytes at the current offsets, and a historical summary every
    SLOTS_PER_HISTORICAL_ROOT slots."""
    rng = np.random.default_rng(seed)
    P = S.PRESETS[st.preset]
    bound, sphr = P["ETH1_DATA_VOTES_BOUND"], P["SLOTS_PER_HISTORICAL_ROOT"]
    for b in range(n_blocks):
        slot = start_slot + b + 1
        epoch = slot // 8
        if len(st.eth1_data_votes) >= bound:           # voting period end (process_eth1_data_reset)
            yield ("set", "eth1_data_votes", b"")
        yield ("push", "eth1_data_votes", vote(rng, slot))
        yield ("set", "latest_execution_payload_header", header(rng, b % 33, slot))
        k = int(rng.integers(0, MAX_DEPOSITS + 1))
        if k:
            yield deposits(rng, k, epoch)
        n = len(st.validators)
        if n:
            m = int(min(n, rng.integers(1, 9)))
            idx = np.unique(np.concatenate([rng.integers(0, n, m), np.arange(max(0, n - k), n)])).astype(np.uint64)
            yield ("elements", "balances", idx, _u64s(rng, len(idx)))
            yield ("elements", "current_epoch_participation", idx, rng.integers(0, 8, len(idx), dtype=np.uint8).tobytes())
            yield ("elements", "previous_epoch_participation", idx[::2], rng.integers(0, 8, len(idx[::2]), dtype=np.uint8).tobytes())
            if b % 5 == 0:
                yield ("elements", "inactivity_scores", idx[:3], _u64s(rng, len(idx[:3]), 100))
        lay = S.layout(st)
        yield ("bytes", lay["slot"][0], int(slot).to_bytes(8, "little"))
        yield ("bytes", lay["block_roots"][0] + 32 * (slot % sphr), rng.integers(0, 256, 32, dtype=np.uint8).tobytes())
        yield ("bytes", lay["state_roots"][0] + 32 * (slot % sphr), rng.integers(0, 256, 32, dtype=np.uint8).tobytes())
        ehv = P["EPOCHS_PER_HISTORICAL_VECTOR"]
        yield ("bytes", lay["randao_mixes"][0] + 32 * (epoch % ehv), rng.integers(0, 256, 32, dtype=np.uint8).tobytes())
        if slot % sphr == 0:
            yield ("push", "historical_summaries", rng.integers(0, 256, 64, dtype=np.uint8).tobytes())


def walk_spec(preset: str = "minimal", n0: int = 40, n_blocks: int = 200, seed: int = 0x5EED) -> dict:
    return dict(name=f"walk:{preset}:{n0}:{n_blocks}", preset=preset, n=n0, blocks=n_blocks, seed=seed)


def walk(spec: dict):
    """(initial mirror, step generator) of a chain walk."""
    st = initial_state(spec["preset"], spec["n"], spec["seed"], votes=5, summaries=2)
    return st, chain_walk(st, spec["blocks"], spec["seed"] + 1)


def _singles(rng, count: int, epoch: int = 100) -> Iterator[tuple]:
    for _ in range(count):
        yield deposits(rng, 1, epoch)


def boundary_scripts() -> List[dict]:
    """Named boundary scripts: initial state, and the steps (a generator over the mirror)."""
    out = []

    def add(name, preset, n, make, votes=3, big=False):
        out.append(dict(name=name, preset=preset, n=n, votes=votes, make=make, big=big))

    # big lists at the finisher hand-off, from empty, across the fold and across the reserved capacity
    add("validators from 0", "minimal", 0, lambda st, r: _singles(r, 3))
    add("validators 64 / 65 hand-off", "minimal", HANDOFF - 2, lambda st, r: _singles(r, 4))
    add("balances 256 / 257 hand-off", "minimal", 4 * HANDOFF - 2, lambda st, r: _singles(r, 4))
    add("participation 2048 / 2049 hand-off", "minimal", 32 * HANDOFF - 2, lambda st, r: _singles(r, 4))
    add("validators 2^17 +- 1 (fold)", "mainnet", COOP_MAX - 2, lambda st, r: _singles(r, 4), big=True)

    def relocate(st, r):
        room = headroom(len(st.validators))
        yield deposits(r, room - 1, 100)            # all five lists one below their reserved capacity
        yield ("push", "validators", validator_records(r, 1, 100).tobytes())   # validators exactly at capacity
        yield deposits(r, 3, 100)                   # all five past capacity: relocated together in one block
        yield deposits(r, 5, 100)                   # appends into the fresh headroom
        yield ("elements", "balances", np.arange(len(st.balances) - 4, len(st.balances), dtype=np.uint64), _u64s(r, 4))
    add("capacity: relocation", "minimal", 10, relocate, big=True)

    # eth1_data_votes at 0 -> 1, bound - 1 -> bound, bound -> bound + 1 (refused), reset
    def votes(st, r):
        bound = S.PRESETS[st.preset]["ETH1_DATA_VOTES_BOUND"]
        yield ("push", "eth1_data_votes", vote(r, 1))
        yield ("push", "eth1_data_votes", b"".join(vote(r, k) for k in range(bound - 2)))
        yield ("push", "eth1_data_votes", vote(r, bound))
        yield ("push", "eth1_data_votes", vote(r, bound + 1))           # refused: LIMIT
        yield ("set", "eth1_data_votes", b"".join(vote(r, k) for k in range(bound + 1)))   # refused: LIMIT
        yield ("set", "eth1_data_votes", b"")
        yield ("push", "eth1_data_votes", vote(r, 7))
    add("eth1_data_votes 0 / 1 / bound / bound + 1", "minimal", 70, votes, votes=0)

    # headers: extra_data 0, 1, 31, 32 bytes; 33 refused; malformed encodings refused
    def headers(st, r):
        for x in (0, 1, 31, 32, 5):
            yield ("set", "latest_execution_payload_header", header(r, x, x))
        yield ("set", "latest_execution_payload_header", header(r, 33, 33))           # refused: extra_data > 32
        yield ("set", "latest_execution_payload_header", header(r, 0, 1)[:583])        # refused: short
        bad = bytearray(header(r, 2, 2)); bad[436:440] = (585).to_bytes(4, "little")
        yield ("set", "latest_execution_payload_header", bytes(bad))                   # refused: wrong internal offset
        yield ("set", "eth1_data_votes", vote(r, 1) + b"\0")                           # refused: not a multiple of 72
        yield ("set", "eth1_data_votes", vote(r, 1)[:71])                              # refused
        yield ("push", "no_such_list", b"\0" * 8)                                      # refused: unknown field
        yield ("set", "validators", b"")                                               # refused: not a settable field
        yield ("push", "historical_summaries", r.integers(0, 256, 128, dtype=np.uint8).tobytes())
    add("headers and malformed encodings", "minimal", 70, headers)

    # update_bytes with pre-append bytes over an offset word: refused after the append moved that offset
    def stale(st, r):
        b = S.serialize(st)
        pos = sc.offset_positions(st.preset)[2]            # the validators offset, behind eth1_deposit_index
        old = bytes(b[pos - 8:pos + 4])
        yield ("push", "eth1_data_votes", vote(r, 9))
        yield ("bytes", pos - 8, old)                      # refused: would restore the old offset
        yield ("bytes", pos - 8, bytes(S.serialize(st)[pos - 8:pos]))   # the same bytes minus the offset word: accepted
        hs = sc.offset_positions(st.preset)[8]
        old_hs = bytes(S.serialize(st)[hs:hs + 4])
        yield deposits(r, 2, 100)
        yield ("bytes", hs, old_hs)                        # refused: historical_summaries moved with the deposits
    add("update_bytes over a moved offset", "minimal", 70, stale)
    return out


def boundary_run(spec: dict, seed: int = 11):
    st = initial_state(spec["preset"], spec["n"], seed, votes=spec["votes"])
    return st, spec["make"](st, np.random.default_rng(seed))


def boundaries() -> Dict[str, List[str]]:
    """Each boundary the issue of shape changes names -> the scripts that must cover it."""
    return {
        "appends from 0 validators": ["validators from 0"],
        "hand-off 64 / 65 validators": ["validators 64 / 65 hand-off"],
        "hand-off 256 / 257 balances": ["balances 256 / 257 hand-off"],
        "hand-off 2048 / 2049 participation flags": ["participation 2048 / 2049 hand-off"],
        "fold 2^17 +- 1 validators": ["validators 2^17 +- 1 (fold)"],
        "reserved capacity": ["capacity: relocation"],
        "votes 0 -> 1, bound - 1 -> bound, bound + 1 refused": ["eth1_data_votes 0 / 1 / bound / bound + 1"],
        "extra_data 0 / 1 / 31 / 32, 33 refused, malformed headers and votes": ["headers and malformed encodings"],
        "update_bytes over a moved offset word": ["update_bytes over a moved offset"],
    }


def mainnet_blocks(st: S.SynthState, n_blocks: int, seed: int) -> Iterator[tuple]:
    """Mainnet-sized blocks: 16 deposits, one vote, a new header, 513 balances and N/32 participation flags each."""
    rng = np.random.default_rng(seed)
    for b in range(n_blocks):
        yield ("push", "eth1_data_votes", vote(rng, b))
        yield ("set", "latest_execution_payload_header", header(rng, (7 * b) % 33, b))
        yield deposits(rng, MAX_DEPOSITS, 1000)
        n = len(st.validators)
        idx = np.unique(np.concatenate([rng.integers(0, n, 513 - MAX_DEPOSITS), np.arange(n - MAX_DEPOSITS, n)])).astype(np.uint64)
        yield ("elements", "balances", idx, _u64s(rng, len(idx)))
        fl = np.unique(rng.integers(0, n, n // 32)).astype(np.uint64)
        yield ("elements", "current_epoch_participation", fl, rng.integers(0, 8, len(fl), dtype=np.uint8).tobytes())
        yield ("root", b)
