"""Measure the reward and penalty deltas (epoch.deltas) on a device-resident state at 2^20 validators (mainnet preset):
device time of the call's three kernels and wall time of the whole call (the 64 MiB copy of the lists to the host
included), achieved bytes/s against HBM3's 3.35 TB/s from the byte model below, and the vectorised Python oracle on one
host core (the oracle, not the reference).  Prints one JSON line, and writes it to the file `--out` names; the card's name
and power limit are read in the same run.

    python tools/probe_rewards.py [--n 1048576] [--iters 20] [--warmup 3] [--out result.json]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from ethereum_consensus_b200 import _lib, epoch, ssz  # noqa: E402
from ethereum_consensus_b200 import state as S  # noqa: E402
from tests import epoch_cases as ec  # noqa: E402
from tests import rewards_oracle as ro  # noqa: E402
from tools.probe_epoch import card  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def byte_model(n: int) -> int:
    """Bytes the call must move on the device: k_epoch_totals reads the records and two flag lists (123 B per validator);
    k_epoch_deltas reads the records, one flag list and the scores and writes eight u64 lists."""
    totals = n * (121 + 2)
    deltas = n * (121 + 1 + 8) + n * 64
    return totals + deltas


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
    st.validators["slashed"][rng.random(args.n) < 0.002] = 1
    st.inactivity_scores[rng.random(args.n) < 0.05] = 5000
    dev = ssz.DeviceBeaconState(S.serialize(st), "mainnet")
    L = _lib.lib()
    dev_ms, wall_ms = [], []
    for it in range(args.warmup + args.iters):
        t0 = time.perf_counter()
        got = epoch.deltas(dev)
        t1 = time.perf_counter()
        if it >= args.warmup:
            dev_ms.append(L.b200_last_kernel_ms())
            wall_ms.append((t1 - t0) * 1e3)
    t0 = time.perf_counter()
    want = ro.deltas(st, "vector")
    oracle_s = time.perf_counter() - t0
    assert np.array_equal(got, want), "device deltas differ from the oracle"
    med = float(np.median(dev_ms))
    nbytes = byte_model(args.n)

    def stats(x):
        return {"median": round(float(np.median(x)), 4), "min": round(float(np.min(x)), 4), "max": round(float(np.max(x)), 4)}
    out = {"probe": "epoch_deltas", "n": args.n, "preset": "mainnet", **card(), "iters": args.iters,
           "deltas_device_ms": stats(dev_ms), "deltas_wall_ms": stats(wall_ms),
           "model_bytes": nbytes, "achieved_bytes_per_s": nbytes / (med * 1e-3),
           "share_of_hbm_peak": nbytes / (med * 1e-3) / HBM_BYTES_PER_S, "python_oracle_vector_one_core_s": round(oracle_s, 3)}
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
