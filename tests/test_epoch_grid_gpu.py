"""process_epoch on device-resident states too large for the literal oracle (tests/epoch_grid_cases.py) against the
vectorised oracle and the C state root: k_epoch_reduce at 511 / 512 / 513 and 1 025 CTAs, a carry inside one reduce
range, changed-record counts on both sides of the whole-list re-hash, activation churn limits 7 and 8 with candidates past
CTA 1 023; and a 16-epoch walk on 2^18 + 37 validators whose exit-queue head is the one the device wrote."""
from __future__ import annotations

import numpy as np
import pytest

from ethereum_consensus_b200 import _lib, epoch
from ethereum_consensus_b200 import state as S
from oracle import epoch_oracle as eo
from tests import epoch_cases as ec
from tests import epoch_grid_cases as gc
from tests.test_epoch_gpu import c_root, upload

pytestmark = pytest.mark.gpu
STATES = gc.states()
MASKS = [("all", eo.ALL), ("registry", eo.STEP["registry_updates"]),
         ("effective", eo.STEP["effective_balance_updates"])]
BIG = ("validators", "balances", "inactivity_scores", "previous_epoch_participation", "current_epoch_participation")


def check_big(dev, want, orc):
    lay = S.layout(want)
    for f in BIG:
        o, ln = lay[f]
        assert dev.read_bytes(o, ln) == getattr(want, f).tobytes(), f
    assert dev.read_bytes(0, dev.serialized_len()) == S.serialize(want).tobytes()
    root = c_root(orc, want)
    assert dev.hash_tree_root_incremental() == root
    assert dev.hash_tree_root() == root


@pytest.mark.parametrize("name,st,refused", STATES, ids=[s[0] for s in STATES])
def test_grid_state(engine, oracle_ssz_c, name, st, refused):
    # a refused state also runs slashings alone, the one sub-step that reads only the total active balance
    for mname, m in MASKS + ([("slashings", eo.STEP["slashings"])] if refused else []):
        dev = upload(st)
        try:
            want, code = eo.process_epoch(st, m)
        except eo.Refused as r:
            assert refused and m in (eo.ALL, eo.STEP["slashings"]), mname
            root0 = dev.hash_tree_root()
            with pytest.raises(_lib.EngineError) as ei:
                epoch.process_epoch(dev, m)
            assert ei.value.code == {"bad_arg": _lib.ERR_BAD_ARG, "limit": _lib.ERR_LIMIT}[r.kind]
            assert dev.read_bytes(0, dev.serialized_len()) == S.serialize(st).tobytes()
            assert dev.hash_tree_root_incremental() == root0
            dev.close()
            continue
        assert code == 0
        epoch.process_epoch(dev, m)
        check_big(dev, want, oracle_ssz_c)
        dev.close()


def test_walk_multi_cta(engine, oracle_ssz_c):
    """16 consecutive epochs (1080 .. 1095, the eth1 voting period ends after 1087; no sync-committee boundary) of a
    mainnet state with 2^18 + 37 validators (1 025 CTAs, three per k_epoch_reduce thread).  Before each epoch: ten
    effective balances at the ejection balance at CTA edges and lanes 0 / 31 (more than L = 4, so the exit queue runs
    ahead and its head and count are the ones the device wrote), three pending validators with tied eligibility in
    different CTAs, new flags, the next slot.  Roots after most epochs, and after two epochs in a row for others."""
    rng = np.random.default_rng(4242)
    n = (1 << 18) + 37
    st = ec.base(n, 1080, seed=4242)
    dev = upload(st)
    lay = S.layout(st)
    nb = -(-n // ec.THREADS)
    heads = []
    for step, cur in enumerate(range(1080, 1096)):
        if step:
            ctas = rng.choice(nb - 1, 10, replace=False)
            idx = np.unique(ctas * ec.THREADS + rng.choice([0, 31, 32, 255], 10)).astype(np.uint64)
            idx = idx[st.validators["exit_epoch"][idx] == ec.FAR]
            pend = np.unique(rng.choice(n, 3, replace=False)).astype(np.uint64)
            pend = pend[(st.validators["exit_epoch"][pend] == ec.FAR) & ~np.isin(pend, idx)]
            ec.ejects(st, idx)
            ec.pending(st, pend, 1070)
            touched = np.concatenate([idx, pend])
            dev.update_elements("validators", touched, st.validators[touched].tobytes())
            flags = rng.integers(0, 8, n, dtype=np.uint8)
            dev.update_elements("current_epoch_participation", np.arange(n, dtype=np.uint64), flags)
            st.current_epoch_participation = flags.copy()
            slot = (cur * 32 + 31).to_bytes(8, "little")
            dev.update_bytes(lay["slot"][0], slot)
            st.fixed["slot"] = slot
        g = eo._Vector(eo.clone(st)).exit_queue()
        heads.append(g)
        st, code = eo.process_epoch(st, eo.ALL)
        assert code == 0
        epoch.process_epoch(dev, eo.ALL)
        if step % 3 != 1:
            assert dev.hash_tree_root_incremental() == c_root(oracle_ssz_c, st), cur
    assert dev.read_bytes(0, dev.serialized_len()) == S.serialize(st).tobytes()
    assert dev.hash_tree_root() == c_root(oracle_ssz_c, st)
    # the walk read device-written queue heads with 0 < c0 < L, and with c0 = L
    assert any(e0 > eo.compute_activation_exit_epoch(1080 + k) and 0 < c0 < L for k, (e0, c0, L) in enumerate(heads))
    assert any(c0 >= L for _, c0, L in heads)
