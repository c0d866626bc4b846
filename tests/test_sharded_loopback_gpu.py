"""GPU: the sharded entry points at world 2, 3, 4, 5 and 8 on one GPU, one process per rank, exchanging through the
loopback communicator (b200_comm_init_loopback).  The cases (tests/sharded_cases.py) sit on the rank boundaries of every
split: strict verify against the C oracle's codes, the RLC check against the exponent model with the global tuple index,
the sharded state roots against the C oracle, the host all-gathers, and the refusals.  Every rank must return the expected
values, identical across ranks, with exactly one collective per sharded call and none per refusal.  World 2 runs again
with team-8 Miller loops at every batch size (B200_VM_TEAM16_MAX=0).

The parent process builds the cases and never touches the GPU; each group of workers runs under a timeout and is killed
and reaped on any failure."""
from __future__ import annotations

import os
import pickle
import subprocess
import sys
import time
from pathlib import Path

import pytest

from tests import sharded_cases as sh

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent
WORKER = ROOT / "tests" / "mp_loopback_worker.py"
CONFIGS = [(w, {}) for w in sh.WORLDS] + [(2, {"B200_VM_TEAM16_MAX": "0"})]


def _compute_mode():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=compute_mode", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=60).stdout.strip()
        return out or "unknown"
    except Exception:   # noqa: BLE001
        return "unknown"


def run_ranks(box: Path, world: int, transport: str = "loopback", env=None, devices=None, sections=None, timeout=900):
    """Starts `world` workers on box/cases.pkl and returns their records; kills and reaps every worker on any failure."""
    procs, logs = [], []
    try:
        for r in range(world):
            e = dict(os.environ, B200_TEST_RANK=str(r), B200_TEST_WORLD=str(world), B200_TEST_DIR=str(box), B200_TEST_TRANSPORT=transport,
                     **(env or {}))
            if devices is not None:
                e["CUDA_VISIBLE_DEVICES"] = str(devices[r])
            if sections:
                e["B200_TEST_SECTIONS"] = ",".join(sections)
            log = open(box / f"rank{r}.log", "w")
            logs.append(log)
            procs.append(subprocess.Popen([sys.executable, str(WORKER)], cwd=str(ROOT), env=e, stdout=log, stderr=subprocess.STDOUT))
        t_end = time.time() + timeout
        for p in procs:
            p.wait(timeout=max(1.0, t_end - time.time()))
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
            p.wait()
        for log in logs:
            log.close()
    out = []
    for r, p in enumerate(procs):
        text = (box / f"rank{r}.log").read_text()
        assert p.returncode == 0 and "WORKER_OK" in text, f"rank {r} exited {p.returncode}:\n{text[-4000:]}"
        out.append(pickle.loads((box / f"rank{r}.pkl").read_bytes()))
    return out


def expected(data):
    """{name: (value, return code, collectives)} of every record the worker writes."""
    want = {}
    single = data["strict"][0]["want"]
    for st in data["states"]:
        want[st["name"]] = (st["want"], 0, 1)
        if st["resident"]:
            want[st["name"] + ": resident upload"] = (None, 0, 1)
            want[st["name"] + ": resident root"] = (st["want"], 0, 1)
            want[st["name"] + ": single-GPU verify between"] = (single, 0, 0)
            want[st["name"] + ": resident root again"] = (st["want"], 0, 1)
    for c in data["strict"]:
        want[c["name"]] = (c["want"], 0, 1)
    for c in data["rlc"]:
        for i, (_seed, w) in enumerate(c["runs"]):
            want[f"{c['name']} [seed {i}]"] = (w, 0, 1)
    w = data["world"]
    want["comm_all_gather_codes"] = ([int(x) for r in range(w) for x in sh.gather_codes(r)], 0, 1)
    for n in data["gather"]:
        want[f"all_gather_bytes {n}"] = (b"".join(sh.gather_payload(r, n) for r in range(w)), 0, 1 if n else 0)
    for name, code in data["refusals"]:
        want[name] = (None, code, 0)
    if any(name == "update_bytes on a sharded handle" for name, _ in data["refusals"]):
        want["upload sharded: the handle the next refusals take"] = (None, 0, 1)
    return want


def check(ranks, data, sections=None):
    """Mismatches of every rank against the expected values, and between ranks; returns (records per rank, mismatches)."""
    want = expected(data)
    bad = []
    for r, recs in enumerate(ranks):
        for sec, name, value, rc, ncoll in recs:
            if sec == "slot":
                continue
            assert name in want, name
            if (value, rc, ncoll) != want[name]:
                bad.append(f"rank {r} {sec} {name}: got {value!r:.200} rc 0x{rc:x} collectives {ncoll}, want {want[name]!r:.200}")
        names = {n for s, n, *_ in recs if s != "slot"}
        missing = [n for n in want if n not in names and (sections is None or _section_of(n, data) in sections)]
        bad += [f"rank {r}: no record of {n}" for n in missing]
    for r in range(1, len(ranks)):
        if [x for x in ranks[r] if x[0] != "slot"] != [x for x in ranks[0] if x[0] != "slot"]:
            bad.append(f"rank {r}'s records differ from rank 0's")
    return sum(len(x) for x in ranks), bad


def _section_of(name, data):
    if any(name.startswith(st["name"]) for st in data["states"]):
        return "states"
    if any(name == c["name"] for c in data["strict"]):
        return "strict"
    if any(name.startswith(c["name"]) for c in data["rlc"]):
        return "rlc"
    if name.startswith("comm_all_gather") or name.startswith("all_gather"):
        return "gather"
    return "refusals"


@pytest.fixture(scope="module")
def cases(tmp_path_factory, oracle_bls_c, oracle_ssz_c):
    """box per world with cases.pkl; states shared across the worlds."""
    root = tmp_path_factory.mktemp("sharded")
    shared, out = {}, {}
    t = time.time()
    for w in sh.WORLDS:
        out[w] = (root / f"w{w}", sh.write_cases(root / f"w{w}", w, oracle_bls_c, oracle_ssz_c, shared))
    print(f"cases and expected values: {time.time() - t:.1f} s")
    return out


@pytest.mark.parametrize("world,env", CONFIGS, ids=[f"world{w}" + "".join(f"-{k}={v}" for k, v in e.items()) for w, e in CONFIGS])
def test_sharded_entry_points_over_loopback(cases, world, env, tmp_path):
    mode = _compute_mode()
    if mode not in ("Default", "unknown"):
        pytest.skip(f"the GPU's compute mode is {mode}: it refuses a second context, and the test never changes it")
    src, data = cases[world]
    box = tmp_path / "box"
    box.mkdir()
    (box / "cases.pkl").write_bytes((src / "cases.pkl").read_bytes())
    t = time.time()
    ranks = run_ranks(box, world, env=env)
    n, bad = check(ranks, data)
    print(f"world {world} {env}: {n} records, {len(bad)} mismatches, wall {time.time() - t:.1f} s")
    assert not bad, "\n".join(bad[:40])
    for r, recs in enumerate(ranks):   # two identical RLC calls put the same bytes in the rank's slot: Gt, flag 0, zeros
        slots = next(v for s, n_, v, *_ in recs if s == "slot" and n_ == "rlc slot twice")
        assert len(slots) == 2 and slots[0] == slots[1], r
        assert slots[0][576:] == bytes(16) and any(slots[0][:576]), r
