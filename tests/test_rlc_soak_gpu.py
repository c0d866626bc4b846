"""GPU: the RLC whole-batch check (bls_rlc.cu and the rlc_tail phase of capi_bls.cu) against its exact
exponent model (tests/rlc_soak_cases.py), case by case, through every entry point.

a. family A: every tuple invalid, defects cancelling under one seed: True under that seed, False under every other seed,
   under a library-drawn seed and for each control batch; b. family B: valid batches whose scaled signatures meet as
   equal or opposite points at every level of the G2 fold, and whose sum is infinity, each also with one defect;
c. family C: one invalid tuple (a defect, or dead) at every position that matters for T up to 4 096.
Each device verdict is compared with model() through fast_aggregate_verify_batch_all, Registry.verify_batch_all and
the sharded call at world 1; the strict per-tuple batch is compared with the C oracle's codes.  Sections b and c run
again under each pairing-VM launch shape (vm_cta 32 / 64 / 128, vm_team16_max 0).

    B200_SOAK_SCALE=1 (default) python -m pytest tests/test_rlc_soak_gpu.py -m gpu -s
"""
from __future__ import annotations

import os
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from tests import rlc_soak_cases as rc  # noqa: E402
from tests.test_bls_device_soak_gpu import report  # noqa: E402

pytestmark = pytest.mark.gpu
SCALE = float(os.environ.get("B200_SOAK_SCALE", "1"))
TUNES = [("vm_cta", 32), ("vm_cta", 64), ("vm_cta", 128), ("vm_team16_max", 0)]
TUNE_DEFAULTS = [("vm_cta", 32), ("vm_team16_max", 2048)]


def _min(x):
    return max(10, int(x * min(SCALE, 1.0)))


# ---------------------------------------------------------------------------------------------------------- inputs
_CACHE = {}


def soak(O):
    """Keys, encoded tuples and the cases of the three families (host-built once per process)."""
    if "soak" not in _CACHE:
        t = time.time()
        keys, M, fam = rc.all_cases(O, SCALE)
        M.prepare([x for cs in fam.values() for c in cs for x in c.batch])
        print(f"host-side keys and signatures: {time.time() - t:.1f} s")
        _CACHE["soak"] = (keys, M, fam)
    return _CACHE["soak"]


class Registry:
    """One device registry holding every key of a family's cases; indices by encoding."""

    def __init__(self, M, cases):
        from ethereum_consensus_b200 import crypto
        encs = list(dict.fromkeys(k for c in cases for t in c.batch for k in self._keys(M, t)))
        self.pos = {e: i for i, e in enumerate(encs)}
        self.reg = crypto.Registry(np.frombuffer(b"".join(encs), dtype=np.uint8))

    @staticmethod
    def _keys(M, t):
        pks = M.encode(t)[0]
        return [pks[48 * j: 48 * j + 48] for j in range(len(pks) // 48)]

    def verify_all(self, M, batch, seed):
        idx = np.array([self.pos[k] for t in batch for k in self._keys(M, t)], dtype=np.uint32)
        _, off, msgs, sigs = M.pack(batch)
        return self.reg.verify_batch_all(idx, off, msgs, sigs, seed=seed)


# ---------------------------------------------------------------------------------------------------------- device checks
def check_family(name, M, cases, entry_points=("plain", "registry", "sharded"), strict=None, tag="", few=None):
    """Every (case, seed) through each entry point against model(); `few`: the cases the registry and sharded calls
    take (default all); strict: cases whose per-tuple batch is compared with the oracle's codes.
    Returns [(section, cases, mismatches)]."""
    from ethereum_consensus_b200 import crypto, parallel
    res = []
    runs = [(c, s, w) for c in cases for s, w in c.runs]
    want = [(w, c.name) for c, _, w in runs]
    if "plain" in entry_points:
        got = [(crypto.fast_aggregate_verify_batch_all(*M.pack(c.batch), seed=s), c.name) for c, s, _ in runs]
        res.append((f"{name} batch_all{tag}", *report(f"{name}: fast_aggregate_verify_batch_all{tag}", want, got)))
    if few is not None:
        cases = few
        runs = [(c, s, w) for c in cases for s, w in c.runs]
        want = [(w, c.name) for c, _, w in runs]
    if "registry" in entry_points:
        reg = Registry(M, cases)
        got = [(reg.verify_all(M, c.batch, s), c.name) for c, s, _ in runs]
        res.append((f"{name} registry{tag}", *report(f"{name}: Registry.verify_batch_all{tag}", want, got)))
    if "sharded" in entry_points:
        parallel.comm_init(0, 1)
        sub = [(c, s, w) for c, s, w in runs if s is not None]     # the ranks must share a caller seed
        got = [(crypto.fast_aggregate_verify_batch_all(*M.pack(c.batch), seed=s, sharded=True), c.name) for c, s, _ in sub]
        res.append((f"{name} sharded{tag}", *report(f"{name}: batch_all sharded, world 1{tag}", [(w, c.name) for c, _, w in sub], got)))
    if strict:
        want = [tuple(M.codes(c.batch)) for c in strict]
        got = [tuple(crypto.fast_aggregate_verify_batch(*M.pack(c.batch)).tolist()) for c in strict]
        res.append((f"{name} strict{tag}", *report(f"{name}: strict batch vs oracle codes{tag}", want, got)))
    return res


def _ends(cases):
    """The C cases with the invalid tuple first or last, and the all-valid ones."""
    return [c for c in cases if c.name.endswith(" all valid") or c.name.endswith(" at 0") or c.name.endswith(f" at {len(c.batch) - 1}")]


def _few(cases):
    """The C cases the other entry points and launch shapes take: every small batch, and the large ones at their ends."""
    ends = set(map(id, _ends(cases)))
    return [c for c in cases if len(c.batch) <= 65 or id(c) in ends]


def _assert_clean(res, minimum=None):
    for name, n, bad in res:
        assert bad == 0, f"{name}: {bad} of {n} verdicts differ from the model"
        if minimum:
            assert n >= minimum.get(name, 1), (name, n)


# ---------------------------------------------------------------------------------------------------------- tests
def test_a_cancelling_defects(engine, oracle_bls_c):
    t = time.time()
    _, M, fam = soak(oracle_bls_c)
    A = fam["A"]
    res = check_family("a. cancelling defects", M, A, strict=A)
    print(f"a. wall {time.time() - t:.1f} s")
    _assert_clean(res, {"a. cancelling defects batch_all": _min(120)})
    crafted = [c for c in A if "A:crafted" in c.tags]
    assert all(set(M.codes(c.batch)) == {5} and c.runs[0][1] for c in crafted)    # all invalid, accepted under the seed


def test_b_fold_edges(engine, oracle_bls_c):
    t = time.time()
    _, M, fam = soak(oracle_bls_c)
    res = check_family("b. fold edges", M, fam["B"], strict=fam["B"])
    print(f"b. wall {time.time() - t:.1f} s")
    _assert_clean(res, {"b. fold edges batch_all": 70})


def test_c_position_sweep(engine, oracle_bls_c):
    t = time.time()
    _, M, fam = soak(oracle_bls_c)
    res = check_family("c. position sweep", M, fam["C"], strict=_ends(fam["C"]), few=_few(fam["C"]))
    print(f"c. wall {time.time() - t:.1f} s")
    _assert_clean(res, {"c. position sweep batch_all": _min(2000)})


@pytest.mark.parametrize("knob,value", TUNES, ids=[f"{k}_{v}" for k, v in TUNES])
def test_bc_under_vm_launch_shapes(engine, oracle_bls_c, knob, value):
    """Sections b and c again with the pairing VM's CTA size, or with team-8 Miller loops at every batch size."""
    from ethereum_consensus_b200 import crypto
    t = time.time()
    _, M, fam = soak(oracle_bls_c)
    try:
        crypto.tune(knob, value)
        tag = f" [{knob} {value}]"
        res = check_family("b. fold edges", M, fam["B"], entry_points=("plain",), tag=tag)
        res += check_family("c. position sweep", M, _few(fam["C"]), entry_points=("plain",), tag=tag)
    finally:
        for k, v in TUNE_DEFAULTS:
            crypto.tune(k, v)
    print(f"{knob} {value} wall {time.time() - t:.1f} s")
    _assert_clean(res)


def _gpu_count():
    try:
        out = subprocess.run(["nvidia-smi", "-L"], capture_output=True, text=True, timeout=60).stdout
        return sum(1 for ln in out.splitlines() if ln.startswith("GPU "))
    except Exception:
        return 0


@pytest.mark.skipif(_gpu_count() < 2, reason="needs >= 2 GPUs")
def test_crafted_batch_on_two_ranks(oracle_bls_c, oracle_ssz_c, tmp_path):
    """The RLC section of the world-2 case list (tests/sharded_cases.py) over NCCL, one GPU per rank: defects that cancel
    only across the rank boundary under the crafting seed, so each rank must hash its global t0 + t; both ranks accept
    them under that seed and reject them under the four others."""
    from tests import sharded_cases as sh
    from tests.test_sharded_loopback_gpu import check, run_ranks
    data = sh.write_cases(tmp_path / "box", 2, oracle_bls_c, oracle_ssz_c)
    ranks = run_ranks(tmp_path / "box", 2, transport="nccl", devices=[0, 1], sections=["rlc"])
    n, bad = check(ranks, data, sections={"rlc"})
    assert not bad, "\n".join(bad[:40])
