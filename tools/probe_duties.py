"""What the duty selections cost on the GPU at 2^20 validators: one JSON line (DESIGN.md §8).

  proposers_32eth     one epoch's proposer lookahead (32 slots), every effective balance 32 ETH
  proposers_mixed     the same, effective balances drawn from {0, 1, 16, 31, 32} ETH
  next_sync_committee get_next_sync_committee: 512 members sampled, their keys gathered, validated and aggregated
  rotation            process_sync_committee_updates at a period boundary, then the incremental root
  committee_indices   the committee-key -> validator-index lookup of process_sync_aggregate
  oracle_proposer     the Python oracle's host time for ONE get_beacon_proposer_index (active set with numpy, seed, the
                      per-index sampling loop); "oracle_proposer_list" with the shuffled-list formulation (the whole
                      active list shuffled, numpy).  These are the Python oracle, not the Rust reference.
Outputs are checked against the oracle before anything is timed.  Each row: median and min-max over --runs timed calls
after --warmup untimed ones, as wall time around the call (every call ends in a device synchronise) and as the device
time of the call (b200_last_kernel_ms).  The card's name and power limit are read with nvidia-smi in the same run.

    python tools/probe_duties.py [--runs 7] [--warmup 2] [--n 1048576]
"""
from __future__ import annotations

import argparse
import ctypes as C
import hashlib
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from ethereum_consensus_b200 import _lib, duties, ssz  # noqa: E402
from ethereum_consensus_b200 import state as S  # noqa: E402
from oracle import duties_oracle as do  # noqa: E402
from tests import duties_cases as dc  # noqa: E402

SK0, DELTA = 0x1234567, 0x89abcdef12345


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, check=True).stdout.strip().splitlines()[0]
    name, power = (x.strip() for x in out.split(","))
    return {"gpu": name, "power_limit": power}


def row(v):
    return {"median": round(statistics.median(v), 3), "min": round(min(v), 3), "max": round(max(v), 3)}


def timed(fn, runs: int, warmup: int, device=True) -> dict:
    lib = _lib.lib()
    wall, dev = [], []
    for i in range(warmup + runs):
        t = time.perf_counter()
        ms = fn()
        w = (time.perf_counter() - t) * 1e3
        if i >= warmup:
            wall.append(w)
            dev.append(ms if ms is not None else lib.b200_last_kernel_ms())
    return {"wall_ms": row(wall), "kernel_ms": row(dev)} if device else {"wall_ms": row(wall)}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1 << 20)
    ap.add_argument("--runs", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    lib = _lib.init()
    info = card()
    subprocess.run(["make", "-s", "-C", str(ROOT / "oracle")], check=True, capture_output=True)
    orc = C.CDLL(str(ROOT / "oracle" / "liboracle_bls.so"))
    orc.orc_pk_sequence.argtypes = [C.c_char_p, C.c_char_p, C.c_size_t, C.c_void_p]
    nd = min(a.n, 1 << 15)
    keys = np.empty((nd, 48), dtype=np.uint8)
    orc.orc_pk_sequence(SK0.to_bytes(32, "big"), DELTA.to_bytes(32, "big"), nd, keys.ctypes.data)
    pk = keys[np.arange(a.n) % nd].view("V48").reshape(a.n)
    res = {"n_validators": a.n, "runs": a.runs, "warmup": a.warmup}

    st = dc.rotation_state(a.n, seed=31)   # one epoch before a sync-committee period boundary
    st.validators["public_key"] = pk
    members = np.random.default_rng(31).integers(0, a.n, 512)
    dc.set_committees(st, members, members[::-1])   # committees of held keys (repeats: the lookup's largest holder)
    epoch = do.slot(st) // 32
    mixed = dc.rotation_state(a.n, seed=32)
    mixed.validators["public_key"] = pk
    mixed.validators["effective_balance"] = np.random.default_rng(32).choice(np.array([0, 1, 16, 31, 32], np.uint64) * dc.ETH, a.n)
    dev, dev_mixed = ssz.DeviceBeaconState(S.serialize(st)), ssz.DeviceBeaconState(S.serialize(mixed))

    assert duties.proposer_indices(dev, epoch).tolist() == do.proposer_indices(st, epoch)
    assert duties.proposer_indices(dev_mixed, epoch).tolist() == do.proposer_indices(mixed, epoch)
    idx, committee, code = duties.next_sync_committee(dev)
    assert code == 0 and idx.tolist() == do.next_sync_committee_indices(st)
    res["proposers_32eth"] = timed(lambda: [duties.proposer_indices(dev, epoch), None][1], a.runs, a.warmup)
    res["proposers_mixed"] = timed(lambda: [duties.proposer_indices(dev_mixed, epoch), None][1], a.runs, a.warmup)
    res["next_sync_committee"] = timed(lambda: [duties.next_sync_committee(dev), None][1], a.runs, a.warmup)

    def rotate():   # device time: the rotation call's plus the incremental root's
        assert duties.process_sync_committee_updates(dev) is True
        ms = lib.b200_last_kernel_ms()
        dev.hash_tree_root_incremental()
        return ms + lib.b200_last_kernel_ms()
    res["rotation"] = timed(rotate, a.runs, a.warmup)
    want = do.sync_committee_indices(st, "current")   # the state's own committee bytes (every key is held)
    dev_fresh = ssz.DeviceBeaconState(S.serialize(st))
    assert duties.sync_committee_indices(dev_fresh, "current").tolist() == want
    res["committee_indices"] = timed(lambda: [duties.sync_committee_indices(dev_fresh, "current"), None][1], a.runs, a.warmup)

    def oracle_one(formulation):
        def run():
            active = do.active_indices(st, epoch)
            seed = hashlib.sha256(do.get_seed(st, epoch, do.DOMAIN_BEACON_PROPOSER) + (epoch * 32).to_bytes(8, "little")).digest()
            do.compute_proposer_index(st, active, seed, formulation)
            return 0.0
        return run
    res["oracle_proposer"] = timed(oracle_one("index"), 3, 1, device=False)
    res["oracle_proposer_list"] = timed(oracle_one("list"), 1, 0, device=False)
    res["oracle_note"] = "Python oracle (numpy + hashlib) on one host core, not the Rust reference"
    print(json.dumps({**info, **res}))


if __name__ == "__main__":
    main()
