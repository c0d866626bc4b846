"""Per-block cost of following the chain with the device-resident state, against re-uploading it.

On BASELINE config 3 (2^20 validators, mainnet preset), per block with the L2 flushed first (a 256 MiB memset, as
bench.py does):
  (i)  the block's shape changes and writes on the resident state — one eth1 vote appended, a new payload header,
       16 deposits, 513 balances, N/32 participation flags, slot / block_roots / state_roots / randao_mixes through
       update_bytes — then b200_state_root_incremental: host wall time end to end, and the root's device time;
  (ii) what a host without reshaping has to do: hash_tree_root of the whole serialization, uploaded from pinned memory
       (b200_htr_beacon_state_deneb): wall time and device time.
Both roots are checked against each other every block.  Prints one JSON line (medians, min / max) with the card's name
and power limit read in the same run.

    python tools/probe_state_chain.py [--blocks 24] [--warmup 3] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))


def card() -> dict:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (x.strip() for x in r.stdout.splitlines()[0].split(","))
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def stats(xs):
    a = np.asarray(xs)
    return {"median": round(float(np.median(a)), 4), "min": round(float(a.min()), 4), "max": round(float(a.max()), 4),
            "n": int(a.size)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=24)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--validators", type=int, default=1 << 20)
    ap.add_argument("--out", default="")
    args = ap.parse_args()

    import torch
    from ethereum_consensus_b200 import _lib, ssz, state as S
    from tests import state_reshape_cases as rc

    lib = _lib.init(0)
    flush_buf = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")

    def flush_l2():
        flush_buf.zero_()
        torch.cuda.synchronize()

    st = S.synth_state(args.validators, "mainnet")
    dev = ssz.DeviceBeaconState(S.serialize(st), "mainnet")
    rng = np.random.default_rng(0xC4A1)
    P = S.PRESETS["mainnet"]
    i_wall, i_dev, ii_wall, ii_dev = [], [], [], []
    for b in range(args.warmup + args.blocks):
        slot = 8_626_177 + b
        n = len(st.validators)
        steps = [("push", "eth1_data_votes", rc.vote(rng, slot)),
                 ("set", "latest_execution_payload_header", rc.header(rng, b % 33, slot)),
                 rc.deposits(rng, rc.MAX_DEPOSITS, 1000)]
        n2 = n + rc.MAX_DEPOSITS
        bi = np.unique(np.concatenate([rng.integers(0, n, 513 - rc.MAX_DEPOSITS), np.arange(n, n2)])).astype(np.uint64)
        fl = np.unique(rng.integers(0, n2, n2 // 32)).astype(np.uint64)
        steps += [("elements", "balances", bi, rng.integers(1, 1 << 40, len(bi), dtype=np.uint64).astype("<u8").tobytes()),
                  ("elements", "current_epoch_participation", fl, rng.integers(0, 8, len(fl), dtype=np.uint8).tobytes())]
        for s in steps:   # the host mirror first, so that the update_bytes offsets below are the reshaped ones
            rc.apply(st, s)
        lay = S.layout(st)
        small = [(lay["slot"][0], slot.to_bytes(8, "little")),
                 (lay["block_roots"][0] + 32 * (slot % P["SLOTS_PER_HISTORICAL_ROOT"]), rng.bytes(32)),
                 (lay["state_roots"][0] + 32 * (slot % P["SLOTS_PER_HISTORICAL_ROOT"]), rng.bytes(32)),
                 (lay["randao_mixes"][0] + 32 * ((slot // 32) % P["EPOCHS_PER_HISTORICAL_VECTOR"]), rng.bytes(32))]
        for o, d in small:
            rc.apply(st, ("bytes", o, d))
        recs, bal = steps[2][1], steps[2][2]
        flush_l2()
        t0 = time.perf_counter()
        dev.append_elements("eth1_data_votes", steps[0][2])
        dev.set_field("latest_execution_payload_header", steps[1][2])
        dev.add_validators(recs, bal)
        dev.update_elements("balances", steps[3][2], steps[3][3])
        dev.update_elements("current_epoch_participation", steps[4][2], steps[4][3])
        for o, d in small:
            dev.update_bytes(o, d)
        root_i = dev.hash_tree_root_incremental()
        t1 = time.perf_counter()
        k_i = float(lib.b200_last_kernel_ms())
        ser = torch.from_numpy(S.serialize(st)).pin_memory()
        flush_l2()
        t2 = time.perf_counter()
        root_ii = ssz.hash_tree_root_beacon_state(ser, "mainnet")
        t3 = time.perf_counter()
        k_ii = float(lib.b200_last_kernel_ms())
        assert root_i == root_ii, f"block {b}: incremental {root_i.hex()} != re-upload {root_ii.hex()}"
        if b >= args.warmup:
            i_wall.append(1e3 * (t1 - t0)); i_dev.append(k_i); ii_wall.append(1e3 * (t3 - t2)); ii_dev.append(k_ii)
    dev.close()
    res = {"probe": "state_chain", "validators_at_start": args.validators, "blocks": args.blocks,
           "block": "1 vote, new header, 16 deposits, 513 balances, N/32 flags, 4 update_bytes", "l2": "256 MiB memset before each",
           "i_reshape_write_incremental_root_ms": {"wall": stats(i_wall), "root_device": stats(i_dev)},
           "ii_reupload_full_root_ms": {"wall": stats(ii_wall), "device": stats(ii_dev)}, **card()}
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
