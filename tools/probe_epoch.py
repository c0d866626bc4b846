"""Measure process_epoch on a device-resident state at 2^20 validators (mainnet preset): device and wall time of a
non-boundary epoch, the incremental root after it, achieved bytes/s against HBM3's 3.35 TB/s from the byte model below,
and the vectorised Python oracle on one host core (the oracle, not the reference).  Prints one JSON line, and writes it to
the file `--out` names; the card's name and power limit are read in the same run.

    python tools/probe_epoch.py [--n 1048576] [--iters 20] [--warmup 3] [--out result.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from ethereum_consensus_b200 import _lib, epoch, ssz  # noqa: E402
from ethereum_consensus_b200 import state as S  # noqa: E402
from oracle import epoch_oracle as eo  # noqa: E402
from tests import epoch_cases as ec  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def byte_model(n: int) -> int:
    """Bytes a non-boundary epoch must move: k_epoch_totals reads the records and both flag lists; k_epoch_apply reads
    the records, balances, scores and previous flags and writes balances and scores back; the rotation reads one flag
    list and writes two.  Record writes (a few percent of records) are left out."""
    totals = n * (121 + 2)
    apply = n * (121 + 8 + 8 + 1) + n * (8 + 8)
    rotation = n * 3
    return totals + apply + rotation


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1 << 20)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    _lib.init(0)
    st = ec.base(args.n, 1000, seed=2020)
    rng = np.random.default_rng(2020)
    st.validators["effective_balance"][rng.random(args.n) < 0.01] = 16 * ec.ETH
    st.balances[rng.random(args.n) < 0.05] = 33_400_000_000
    dev = ssz.DeviceBeaconState(S.serialize(st), "mainnet")
    dev.hash_tree_root()
    L = _lib.lib()
    dev_ms, wall_ms, root_ms = [], [], []
    for it in range(args.warmup + args.iters):
        t0 = time.perf_counter()
        epoch.process_epoch(dev, epoch.ALL)
        t1 = time.perf_counter()
        k = L.b200_last_kernel_ms()
        t2 = time.perf_counter()
        dev.hash_tree_root_incremental()
        t3 = time.perf_counter()
        if it >= args.warmup:
            dev_ms.append(k)
            wall_ms.append((t1 - t0) * 1e3)
            root_ms.append((t3 - t2) * 1e3)
    t0 = time.perf_counter()
    eo.process_epoch(st, eo.ALL, "vector")
    oracle_s = time.perf_counter() - t0
    med = float(np.median(dev_ms))
    nbytes = byte_model(args.n)

    def stats(x):
        return {"median": round(float(np.median(x)), 4), "min": round(float(np.min(x)), 4), "max": round(float(np.max(x)), 4)}
    out = {"probe": "process_epoch", "n": args.n, "preset": "mainnet", **card(), "iters": args.iters,
           "epoch_device_ms": stats(dev_ms), "epoch_wall_ms": stats(wall_ms), "root_incremental_wall_ms": stats(root_ms),
           "model_bytes": nbytes, "achieved_bytes_per_s": nbytes / (med * 1e-3),
           "share_of_hbm_peak": nbytes / (med * 1e-3) / HBM_BYTES_PER_S, "python_oracle_vector_one_core_s": round(oracle_s, 3)}
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
