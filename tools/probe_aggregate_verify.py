"""What aggregate_verify in batches costs on the GPU: one JSON line (DESIGN.md §8).

  single_vs_batch   T = 1, n in {1, 16, 128, 512}: b200_aggregate_verify against
                    aggregate_verify_batch (lane-parallel Miller loops, segmented product, lane-parallel final exponentiation)
  t64_n128          T = 64, n = 128: one batch call against 64 single calls
  t4096_n1          T = 4096, n = 1: aggregate_verify_batch against fast_aggregate_verify_batch with K = 1 on the same tuples
                    (two pairs per tuple either way: the difference is the new path's overhead)
  registry          the T = 64, n = 128 and T = 4096, n = 1 batches with their keys named by registry index
Every batch's codes are checked against the single calls or the closed forms before anything is timed.  Each figure: the
median over --runs calls after --warmup untimed ones, as device time of the call's kernels (b200_last_kernel_ms) and as
wall time around the call (every call ends in a device synchronise).  The card's name and power limit are read with
nvidia-smi in the same run.

    python tools/probe_aggregate_verify.py [--runs 5] [--warmup 2]
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
from tests import aggregate_verify_cases as av  # noqa: E402


def oracle():
    subprocess.run(["make", "-s", "-C", str(ROOT / "oracle")], check=True, capture_output=True)
    return av.bind(C.CDLL(str(ROOT / "oracle" / "liboracle_bls.so")))


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, check=True).stdout.strip().splitlines()[0]
    name, power = (x.strip() for x in out.split(","))
    return {"gpu": name, "power_limit": power}


def timed(fn, runs: int, warmup: int) -> dict:
    for _ in range(warmup):
        fn()
    wall, dev = [], []
    for _ in range(runs):
        t = time.perf_counter()
        ms = fn()
        wall.append((time.perf_counter() - t) * 1e3)
        dev.append(ms if isinstance(ms, float) else crypto.last_kernel_ms())   # the single-call loops return their summed time
    return {"kernel_ms": round(statistics.median(dev), 3), "wall_ms": round(statistics.median(wall), 3)}


def _arr(b: bytes):
    return np.frombuffer(b, dtype=np.uint8).copy() if b else np.zeros(0, dtype=np.uint8)


class Batch:
    """One batch's call arguments, built once."""

    def __init__(self, tuples):
        self.tuples = tuples
        keys, koff, msgs, grp, sigs = av.flatten(tuples)
        self.keys, self.koff, self.msgs, self.grp, self.sigs = _arr(keys), koff, msgs, grp, _arr(sigs)
        self.want = [t["want"] for t in tuples]

    def batch(self):
        return crypto.aggregate_verify_batch(self.keys, self.koff, self.msgs, self.grp, self.sigs).tolist()

    def singles(self):
        """T single calls; returns the codes and the summed kernel time."""
        L, codes, ms = _lib.lib(), [], 0.0
        for t in self.tuples:
            bufs = [C.create_string_buffer(m, max(len(m), 1)) for m in t["msgs"]]
            ptrs = (C.c_void_p * len(bufs))(*[C.addressof(b) for b in bufs])
            lens = (C.c_size_t * len(bufs))(*[len(m) for m in t["msgs"]])
            codes.append(int(L.b200_aggregate_verify(b"".join(t["pks"]), len(t["pks"]), C.cast(ptrs, C.c_void_p),
                                                     C.cast(lens, C.c_void_p), len(bufs), t["sig"])))
            ms += crypto.last_kernel_ms()
        return codes, ms

    def registry(self):
        keys = [k for t in self.tuples for k in t["pks"]]
        reg = crypto.Registry(_arr(b"".join(keys)))
        idx = np.arange(len(keys), dtype=np.uint32)
        return lambda: reg.aggregate_verify_batch(idx, self.koff, self.msgs, self.grp, self.sigs).tolist()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    O = oracle()
    _lib.init(0)
    res = {**card(), "runs": a.runs, "warmup": a.warmup, "single_vs_batch": {}}
    for n in (1, 16, 128, 512):
        b = Batch(av.scale(O, 1, n, seed=100 + n))
        assert b.batch() == b.want == b.singles()[0], n
        res["single_vs_batch"][f"n{n}"] = {"single": timed(lambda: b.singles()[1], a.runs, a.warmup),
                                           "batch": timed(b.batch, a.runs, a.warmup)}
    b = Batch(av.scale(O, 64, 128, seed=7, bad_every=9))
    assert b.batch() == b.want == b.singles()[0]
    res["t64_n128"] = {"batch": timed(b.batch, a.runs, a.warmup), "singles": timed(lambda: b.singles()[1], a.runs, a.warmup)}
    reg = b.registry()
    assert reg() == b.want
    res["registry"] = {"t64_n128": timed(reg, a.runs, a.warmup)}
    w = Batch(av.scale(O, 4096, 1, seed=8, bad_every=101))
    fk = _arr(b"".join(t["pks"][0] for t in w.tuples))
    fm = _arr(b"".join(t["msgs"][0] for t in w.tuples))
    foff = np.arange(4097, dtype=np.uint32)
    fast = lambda: crypto.fast_aggregate_verify_batch(fk, foff, fm, w.sigs).tolist()  # noqa: E731
    assert w.batch() == w.want == fast()
    res["t4096_n1"] = {"aggregate_verify_batch": timed(w.batch, a.runs, a.warmup),
                       "fast_aggregate_verify_batch_k1": timed(fast, a.runs, a.warmup)}
    reg = w.registry()
    assert reg() == w.want
    res["registry"]["t4096_n1"] = timed(reg, a.runs, a.warmup)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
