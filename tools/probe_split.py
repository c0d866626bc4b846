"""A/B of the split key copy (b200_tune "bls_key_split") on the bench workload: device ms and END-TO-END wall ms from pinned
host buffers, strict T x K.   python tools/probe_split.py [T] [K]"""
import os
import sys
import time
sys.path.insert(0, ".")
import bench
from ethereum_consensus_b200 import crypto, _lib
from tests import workloads

T = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
K = int(sys.argv[2]) if len(sys.argv) > 2 else 512
orc_bls, _ = bench.load_oracles()
w = workloads.make_bls_workload(orc_bls, T, K, 0, threads=len(os.sched_getaffinity(0)))
_lib.init(0)
import torch
pks, off, msgs, sigs = (bench.pin(w[k]) for k in ("pks", "off", "msgs", "sigs"))
want = w["expect"].tolist()
CONFIGS = [(1, 384, 0), (1, 128, 0), (1, 128, 64), (1, 128, 32), (1, 384, 64), (1, 384, 32), (1, 384, 0), (1, 128, 64)] if os.environ.get("B200_PROBE_CTA") else [(1, 384, 0), (0, 384, 0), (1, 384, 0), (0, 384, 0)]
for split, first_cta, small_cta in CONFIGS:
    crypto.tune("bls_key_split", split); crypto.tune("bls_k1_first_cta", first_cta); crypto.tune("bls_small_cta", small_cta)
    dev, wall = [], []
    for i in range(7):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        got = crypto.fast_aggregate_verify_batch(pks, off, msgs, sigs)
        dt = (time.perf_counter() - t0) * 1e3
        assert got.tolist() == want
        if i >= 2:
            dev.append(crypto.last_kernel_ms()); wall.append(dt)
    print(f"T={T} K={K} key_split={split} k1_first_cta={first_cta} small_cta={small_cta or 'auto'}: device {min(dev):.2f} ms | end-to-end wall {min(wall):.2f} ms "
          f"(median {sorted(wall)[len(wall)//2]:.2f}) | per-key kernels {crypto.last_dominant_kernel_ms():.2f} ms", flush=True)
