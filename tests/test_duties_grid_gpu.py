"""Proposer and sync-committee duties on the device at the sampling and matching kernels' launch-shape edges
(tests/duties_grid_cases.py) against the oracle (oracle/duties_oracle.py), index for index: committee cuts at lane,
scan-warp, window and chunk edges with the launch count each implies, all-0-ETH committees drawn into windows 7 and 8,
proposer warps of very different depths in one CTA, 31 to 65 active validators, committee keys with equal prefixes and
holders on every grid-stride pass; and a child process whose first duty call grows the sampling scratch between windows."""
from __future__ import annotations

import os
import subprocess
import sys
import time
from functools import lru_cache
from pathlib import Path

import pytest

from ethereum_consensus_b200 import _lib, duties, shuffling
from oracle import duties_oracle as do
from oracle import shuffle_oracle as sh
from tests import duties_cases as dc
from tests import duties_grid_cases as gc
from tests.test_duties_gpu import c_aggregate, upload

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent
COMMITTEE = gc.committee_cases()
PROPOSER = gc.proposer_cases()


@pytest.fixture(scope="module", autouse=True)
def _wall():
    t = time.time()
    yield
    print(f"\ntest_duties_grid_gpu.py wall {time.time() - t:.1f} s")


def counted(fn):
    L = _lib.lib()
    c0 = L.b200_launch_count()
    r = fn()
    return r, L.b200_launch_count() - c0


@lru_cache(maxsize=None)
def want_committee(name: str):
    case = next(c for c in COMMITTEE if c.name == name)
    return do.next_sync_committee_indices(case.st, "list")


def check_committee(dev, case):
    """-> ((indices, committee bytes, code), launches) of the device's next_sync_committee, the indices checked against
    the oracle's"""
    (idx, committee, code), k = counted(lambda: duties.next_sync_committee(dev))
    want = want_committee(case.name)
    assert idx.tolist() == want, (case.name, next(j for j in range(len(want)) if idx[j] != want[j]))
    if code:
        assert committee == bytes(len(committee))
    return (idx.tolist(), committee, code), k


@pytest.mark.parametrize("case", COMMITTEE, ids=[c.name for c in COMMITTEE])
def test_committee_case(engine, oracle_bls_c, case):
    dev = upload(case.st)
    got, _ = check_committee(dev, case)
    assert got == do.next_sync_committee(case.st, c_aggregate(oracle_bls_c), "list")
    # counted on a second call: the first BLS call of a process adds its one-time set-up launches
    again, k = check_committee(dev, case)
    assert again == got and k == gc.window_map(case.preset).launches(case.cut), case.name
    for which in ("current", "next"):
        assert duties.sync_committee_indices(dev, which, missing_ok=True).tolist() == do.sync_committee_indices(case.st, which)
    dev.close()


@pytest.mark.parametrize("case", PROPOSER, ids=[c.name for c in PROPOSER])
def test_proposer_case(engine, case):
    dev = upload(case.st)
    for e in case.epochs:
        (got, k) = counted(lambda: duties.proposer_indices(dev, e))
        assert got.tolist() == do.proposer_indices(case.st, e), e
        assert k == 4
    if case.name.startswith("active_"):
        assert duties.next_sync_committee(dev)[0].tolist() == do.next_sync_committee_indices(case.st, "list")
    dev.close()


def sm_count() -> int:
    import torch
    return torch.cuda.get_device_properties(int(os.environ.get("LOCAL_RANK", "0"))).multi_processor_count


def test_matcher_case(engine):
    case, = gc.matcher_cases(sm_count())
    dev = upload(case.st)
    for which in ("current", "next"):
        got, k = counted(lambda: duties.sync_committee_indices(dev, which, missing_ok=True))
        want = do.sync_committee_indices(case.st, which)
        assert want == [case.holders[which].get(j, do.MISSING) for j in range(512)]
        bad = [j for j in range(512) if got[j] != want[j]]
        assert not bad, (which, bad[:8], [(int(got[j]), want[j]) for j in bad[:8]])
        assert k == 1
    dev.close()


def test_cold_scratch_child_process():
    """A fresh process whose first duty call is the window-8 all-0-ETH committee: the sampling scratch is reallocated
    between windows while candidates are already accepted.  Then the same call warm, after a proposer lookahead and a
    key match (both reuse that scratch) and after a shuffle (which reuses the committee's output list)."""
    t = time.time()
    p = subprocess.Popen([sys.executable, "-m", "tests.test_duties_grid_gpu"], cwd=str(ROOT), stdout=subprocess.PIPE,
                         stderr=subprocess.STDOUT, text=True)
    try:
        out = p.communicate(timeout=600)[0]
    except subprocess.TimeoutExpired:
        p.kill()
        out = p.communicate()[0]
    print(out)
    print(f"child wall {time.time() - t:.1f} s")
    assert p.returncode == 0, out
    assert "CHILD_OK" in out, out


def _child():
    _lib.init(int(os.environ.get("LOCAL_RANK", "0")))
    case = gc.zero_eth_case("w8_wrapped")
    st = case.st
    wm = gc.window_map("mainnet")
    members = want_committee(case.name)
    st = dc.set_committees(st, members[::-1], members[7:] + members[:7])
    dev = upload(st)
    first, k0 = check_committee(dev, case)   # the first duty call of the process
    again, k = check_committee(dev, case)
    assert again == first and k0 >= k == wm.launches(case.cut)
    print("cold committee: windows", wm.where(case.cut).window + 1, "launches", k0, "then", k)
    pcase = PROPOSER[0]
    pdev = upload(pcase.st)
    e = pcase.epochs[0]
    assert duties.proposer_indices(pdev, e).tolist() == do.proposer_indices(pcase.st, e)
    assert check_committee(dev, case)[0] == first
    for which in ("current", "next"):
        assert duties.sync_committee_indices(dev, which, missing_ok=True).tolist() == do.sync_committee_indices(st, which)
    assert check_committee(dev, case)[0] == first
    epoch = gc.committee_epoch(st)
    seed = duties.get_seed(dev, epoch, duties.DOMAIN_BEACON_ATTESTER)
    act = do.active_indices(st, epoch)
    assert shuffling.state_shuffled_active_indices(dev, epoch, seed).tolist() == sh.shuffled_indices_numpy(act, seed).tolist()
    assert check_committee(dev, case)[0] == first
    print("CHILD_OK")


if __name__ == "__main__":
    _child()
