"""A/B timing of the per-key validation kernel (K1, k_g1_validate) between builds of the library, on bench.py's headline
workload (fast_aggregate_verify, T = 4096 tuples x K = 512 keys, strict mode).

Every library runs in a process of its own (B200_LIB selects it); the libraries take turns, round after round, so that
clock and neighbour drift fall on all of them alike.  Each run warms up, then reads crypto.last_dominant_kernel_ms()
(CUDA events around K1) and crypto.last_kernel_ms() (the whole device pipeline) after each of --launches calls, and
checks the verdict codes against the workload's expectation.  The card's name, power limit and SM clocks are printed
with the numbers.

  python tools/k1_ab.py ethereum_consensus_b200/libb200_consensus.so other_build.so --rounds 5 --launches 12
"""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def child(work: str, warmup: int, launches: int) -> None:
    import numpy as np
    from ethereum_consensus_b200 import _lib, crypto
    w = np.load(work)
    _lib.init(0)
    args = (w["pks"], w["off"], w["msgs"], w["sigs"])
    for _ in range(warmup):
        codes = crypto.fast_aggregate_verify_batch(*args)
    k1, dev = [], []
    for _ in range(launches):
        codes = crypto.fast_aggregate_verify_batch(*args)
        k1.append(crypto.last_dominant_kernel_ms())
        dev.append(crypto.last_kernel_ms())
    ok = codes.tolist() == w["expect"].tolist()
    print(json.dumps({"k1_ms": k1, "device_ms": dev, "codes_ok": ok,
                      "codes_sha256": hashlib.sha256(np.ascontiguousarray(codes).tobytes()).hexdigest()}))


def card() -> str:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    except FileNotFoundError:
        return "nvidia-smi unavailable"
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "nvidia-smi unavailable"


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("libs", nargs="+", help="library builds to compare (paths to libb200_consensus*.so)")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--launches", type=int, default=12)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--tuples", type=int, default=4096)
    ap.add_argument("--keys", type=int, default=512)
    ap.add_argument("--child", metavar="WORKLOAD", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        child(args.child, args.warmup, args.launches)
        return 0

    import ctypes
    import numpy as np
    from tests.workloads import make_bls_workload
    subprocess.run(["make", "-s", "-C", str(ROOT / "oracle")], check=True)
    orc = ctypes.CDLL(str(ROOT / "oracle" / "liboracle_bls.so"))
    orc.orc_pk_sequence.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_size_t, ctypes.c_void_p]
    orc.orc_sign_batch.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_int]
    w = make_bls_workload(orc, args.tuples, args.keys, 0, threads=os.cpu_count() or 8)
    libs = [str(Path(p).resolve()) for p in args.libs]
    print(f"card: {card()}", flush=True)
    res = {p: {"k1": [], "dev": [], "sha": set()} for p in libs}
    with tempfile.TemporaryDirectory() as tmp:
        work = os.path.join(tmp, "work.npz")
        np.savez(work, pks=w["pks"], off=w["off"], msgs=w["msgs"], sigs=w["sigs"], expect=w["expect"])
        for rnd in range(args.rounds):
            for p in libs:
                env = {**os.environ, "B200_LIB": p}
                r = subprocess.run([sys.executable, __file__, "--child", work, "--warmup", str(args.warmup),
                                    "--launches", str(args.launches), p], capture_output=True, text=True, env=env, cwd=ROOT)
                if r.returncode != 0:
                    print(r.stdout, r.stderr, file=sys.stderr)
                    return 1
                d = json.loads(r.stdout.strip().splitlines()[-1])
                if not d["codes_ok"]:
                    print(f"{p}: verdicts differ from the workload's expectation", file=sys.stderr)
                    return 1
                k1 = statistics.median(d["k1_ms"])
                res[p]["k1"].append(k1)
                res[p]["dev"].append(statistics.median(d["device_ms"]))
                res[p]["sha"].add(d["codes_sha256"])
                print(f"round {rnd}  {Path(p).name:40s} K1 {k1:8.3f} ms  device {res[p]['dev'][-1]:8.3f} ms", flush=True)
    print(f"card: {card()}")
    base = statistics.median(res[libs[0]]["k1"])
    for p in libs:
        k = res[p]["k1"]
        print(f"{Path(p).name:40s} K1 median {statistics.median(k):8.3f} ms  range {min(k):8.3f}-{max(k):8.3f}  "
              f"device median {statistics.median(res[p]['dev']):8.3f} ms  K1 vs first {statistics.median(k) / base - 1:+.2%}")
    if len({s for p in libs for s in res[p]["sha"]}) != 1:
        print("verdict codes differ between libraries", file=sys.stderr)
        return 1
    return 0


if __name__ == "__main__":
    sys.exit(main())
