"""What batch aggregation costs on the GPU: one JSON line (DESIGN.md §8).

  slot_batch        one slot of single-signer attestations at 2^20 validators: 64 committees x 512 signatures into 64
                    aggregates by ONE aggregate_batch call
  slot_single       the same slot as 64 b200_aggregate calls
  keys_strict       eth_aggregate_public_keys_batch on the slot's 64 x 512 keys (every key decompressed and validated)
  keys_registry     Registry.aggregate_public_keys on the same validator indices of a 2^20-key registry
  sync_committee    Registry.aggregate_public_keys of one 512-key sync committee
  cpu_slot          the C oracle's aggregate on the same slot, 64 calls on one host core (the plain-C restatement
                    built with gcc -O3, not blst)
Outputs are checked against the single-call path (and the slot's closed-form aggregates) before anything is timed.
Each row: median and min-max over --runs timed calls after --warmup untimed ones, as wall time around the call (every call
ends in a device synchronise) and as device time of its kernels (b200_last_kernel_ms).  The card's name and power limit
are read with nvidia-smi in the same run.

    python tools/probe_aggregate.py [--runs 7] [--warmup 2] [--n 1048576] [--cpu-runs 1]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from ethereum_consensus_b200 import _lib, crypto  # noqa: E402
from tests import aggregate_batch_cases as ac  # noqa: E402

SK0, DELTA = 0x5eed0123456789abcdef, 0xfedcba98765


def oracle():
    subprocess.run(["make", "-s", "-C", str(ROOT / "oracle")], check=True, capture_output=True)
    orc = C.CDLL(str(ROOT / "oracle" / "liboracle_bls.so"))
    orc.orc_pk_sequence.argtypes = [C.c_char_p, C.c_char_p, C.c_size_t, C.c_void_p]
    orc.orc_aggregate.argtypes = [C.c_char_p, C.c_size_t, C.c_char_p]
    return orc


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, check=True).stdout.strip().splitlines()[0]
    name, power = (x.strip() for x in out.split(","))
    return {"gpu": name, "power_limit": power}


def row(v):
    return {"median": round(statistics.median(v), 3), "min": round(min(v), 3), "max": round(max(v), 3)}


def timed(fn, runs: int, warmup: int, device=True) -> dict:
    wall, dev = [], []
    for i in range(warmup + runs):
        t = time.perf_counter()
        ms = fn()
        w = (time.perf_counter() - t) * 1e3
        if i >= warmup:
            wall.append(w)
            dev.append(ms if ms is not None else crypto.last_kernel_ms())
    return {"wall_ms": row(wall), "kernel_ms": row(dev)} if device else {"wall_ms": row(wall)}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1 << 20)
    ap.add_argument("--runs", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--cpu-runs", type=int, default=1)
    a = ap.parse_args()
    lib = _lib.init()
    info = card()
    orc = oracle()
    slot = ac.slot()
    sigs = np.frombuffer(b"".join(slot["sigs"]), dtype=np.uint8)
    off = np.array(slot["offsets"], dtype=np.uint32)
    res = {"committees": 64, "committee_size": 512, "n_validators": a.n, "runs": a.runs, "warmup": a.warmup}

    # outputs first: the batch against the 64 single calls and the closed forms
    out, codes = crypto.aggregate_batch(sigs, off)
    assert codes.tolist() == [0] * 64 and [bytes(o) for o in out] == slot["agg_sig"]
    single = [crypto.aggregate(slot["sigs"][off[c]:off[c + 1]]) for c in range(64)]
    assert single == slot["agg_sig"]

    def singles():
        ms = 0.0
        buf = (C.c_uint8 * 96)()
        for c in range(64):
            assert lib.b200_aggregate(sigs[96 * off[c]:].ctypes.data, 512, buf) == 0
            ms += crypto.last_kernel_ms()
        return ms

    res["slot_batch"] = timed(lambda: crypto.aggregate_batch(sigs, off) and None, a.runs, a.warmup)
    res["slot_single"] = timed(singles, a.runs, a.warmup)

    keys = np.empty((a.n, 48), dtype=np.uint8)
    orc.orc_pk_sequence(SK0.to_bytes(32, "big"), DELTA.to_bytes(32, "big"), a.n, keys.ctypes.data)
    reg = crypto.Registry(keys.reshape(-1))
    rng = np.random.default_rng(3)
    idx = rng.permutation(a.n)[:64 * 512].astype(np.uint32)
    strict = np.ascontiguousarray(keys[idx]).reshape(-1)
    kout, kcodes = crypto.eth_aggregate_public_keys_batch(strict, off)
    rout, rcodes = reg.aggregate_public_keys(idx, off)
    assert kcodes.tolist() == rcodes.tolist() == [0] * 64 and np.array_equal(kout, rout)
    for c in (0, 31, 63):
        assert bytes(kout[c]) == crypto.eth_aggregate_public_keys([bytes(k) for k in keys[idx[off[c]:off[c + 1]]]])
    res["keys_strict"] = timed(lambda: crypto.eth_aggregate_public_keys_batch(strict, off) and None, a.runs, a.warmup)
    res["keys_registry"] = timed(lambda: reg.aggregate_public_keys(idx, off) and None, a.runs, a.warmup)
    committee = rng.integers(0, a.n, 512).astype(np.uint32)
    sc_off = np.array([0, 512], dtype=np.uint32)
    sout, scodes = reg.aggregate_public_keys(committee, sc_off)
    assert scodes.tolist() == [0] and bytes(sout[0]) == crypto.eth_aggregate_public_keys([bytes(k) for k in keys[committee]])
    res["sync_committee"] = timed(lambda: reg.aggregate_public_keys(committee, sc_off) and None, a.runs, a.warmup)

    cbuf = C.create_string_buffer(96)

    def cpu():
        for c in range(64):
            assert orc.orc_aggregate(bytes(sigs[96 * off[c]:96 * off[c + 1]]), 512, cbuf) == 0
        return 0.0
    cpu()
    assert cbuf.raw == slot["agg_sig"][63]
    res["cpu_slot"] = timed(cpu, a.cpu_runs, 0, device=False)
    res["cpu_slot"]["cpu_baseline"] = {"cores": 1, "kind": "port",
                                       "note": "plain-C restatement built with gcc -O3, not blst; one host core"}
    print(json.dumps({**info, **res}))


if __name__ == "__main__":
    main()
