"""What growing the validated-key registry costs on the GPU, against reloading it: one JSON line (DESIGN.md §7).

On a 2^20-validator deneb state (`state.synth_state`, valid public keys) resident in HBM:
  load          Registry(pks): 2^20 keys from pinned host memory, every key validated (K1)
  from_state    Registry.from_state(state): the same keys gathered from the state's Validator records in HBM
  sync          after state.add_validators(16 records): Registry.sync(state), which validates only the 16 new keys
  reload        the alternative to sync: Registry(pks) of every key the state then holds (2^20 + 16 per batch so far)
  append        Registry.append of 16 keys from the host
Each row: median and min-max over --runs timed calls after --warmup untimed ones, as wall time around the call (every call
ends in a device synchronise) and as device time of its kernels (b200_last_kernel_ms).  The card's name and power limit
are read with nvidia-smi in the same run.

    python tools/probe_registry_grow.py [--runs 7] [--warmup 2] [--n 1048576]
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

from ethereum_consensus_b200 import _lib, crypto, ssz, state as S  # noqa: E402

R = 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001
SK0, DELTA = 0x5eed0123456789abcdef, 0xfedcba98765


def valid_keys(n: int, distinct: int = 1 << 14) -> np.ndarray:
    """n valid keys: `distinct` of them from the C oracle, tiled (K1's cost does not depend on repeats)."""
    subprocess.run(["make", "-s", "-C", str(ROOT / "oracle")], check=True, capture_output=True)
    orc = C.CDLL(str(ROOT / "oracle" / "liboracle_bls.so"))
    orc.orc_pk_sequence.argtypes = [C.c_char_p, C.c_char_p, C.c_size_t, C.c_void_p]
    d = min(n, distinct)
    keys = np.empty((d, 48), dtype=np.uint8)
    orc.orc_pk_sequence(SK0.to_bytes(32, "big"), DELTA.to_bytes(32, "big"), d, keys.ctypes.data)
    return np.ascontiguousarray(np.resize(keys, (n, 48)))


def pinned(a: np.ndarray):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).reshape(-1)).pin_memory()


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, check=True).stdout.strip().splitlines()[0]
    name, power = (x.strip() for x in out.split(","))
    return {"gpu": name, "power_limit": power}


def timed(fn, runs: int, warmup: int, prepare=None) -> dict:
    wall, dev = [], []
    for i in range(warmup + runs):
        if prepare:
            prepare()
        t = time.perf_counter()
        fn()
        w = (time.perf_counter() - t) * 1e3
        if i >= warmup:
            wall.append(w)
            dev.append(crypto.last_kernel_ms())
    row = lambda v: {"median": round(statistics.median(v), 3), "min": round(min(v), 3), "max": round(max(v), 3)}  # noqa: E731
    return {"wall_ms": row(wall), "kernel_ms": row(dev)}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1 << 20)
    ap.add_argument("--runs", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    _lib.init()
    info = card()
    n, k = a.n, 16
    keys = valid_keys(n + k * (a.warmup + a.runs + 1))
    st = S.synth_state(n, "mainnet", pubkeys=keys[:n])
    h = ssz.DeviceBeaconState(S.serialize(st), "mainnet")
    rng = np.random.default_rng(1)
    res = {"n_validators": n, "new_keys": k, "runs": a.runs, "warmup": a.warmup}

    pks = pinned(keys[:n])
    res["load"] = timed(lambda: crypto.Registry(pks), a.runs, a.warmup)
    res["from_state"] = timed(lambda: crypto.Registry.from_state(h), a.runs, a.warmup)
    assert crypto.Registry.from_state(h).key_codes().tolist() == [0] * n

    # sync after a deposit batch of k validators, each run on a registry that matched the state before the batch
    box = {}

    def deposit():
        box["reg"] = crypto.Registry.from_state(h)
        m = h.n_validators
        recs = np.zeros(k, dtype=S.VALIDATOR_DTYPE)
        recs["public_key"] = keys[m:m + k].view("V48").reshape(k)
        recs["withdrawal_credentials"] = rng.integers(0, 256, (k, 32), dtype=np.uint8).view("V32").reshape(k)
        recs["effective_balance"] = 32 * 10**9
        for f in ("activation_eligibility_epoch", "activation_epoch", "exit_epoch", "withdrawable_epoch"):
            recs[f] = S.FAR_FUTURE_EPOCH
        h.add_validators(recs.tobytes(), np.full(k, 32 * 10**9, "<u8"))
    res["sync"] = timed(lambda: box["reg"].sync(h), a.runs, a.warmup, prepare=deposit)
    assert box["reg"].n == h.n_validators and box["reg"].key_codes().tolist() == [0] * h.n_validators
    all_pks = pinned(keys[:h.n_validators])
    res["reload"] = timed(lambda: crypto.Registry(all_pks), a.runs, a.warmup)
    res["reload"]["n_keys"] = h.n_validators

    new = pinned(keys[n:n + k])
    box["reg"] = crypto.Registry(pks)
    res["append"] = timed(lambda: box["reg"].append(new), a.runs, a.warmup)
    assert box["reg"].key_codes().tolist() == [0] * box["reg"].n
    h.close()
    print(json.dumps({**info, **res}))


if __name__ == "__main__":
    main()
