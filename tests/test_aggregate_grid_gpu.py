"""GPU: batch aggregation where the device splits a group (tests/aggregate_grid_cases.py, shapes checked on the CPU by
tests/test_aggregate_grid_cases.py).  Every group of every filled call, at the chunk size this device's SM count gives,
against its expected code and bytes; the single `aggregate` call and the C oracle on the test groups; the launches of
each call.  Key tuples with two invalid keys on one lane through every K2 entry point, at tuple counts around the CTA
edges, and the sync-committee aggregate of a resident mainnet state with two invalid member keys on one lane."""
from __future__ import annotations

import ctypes as C
import os
import time

import numpy as np
import pytest

from ethereum_consensus_b200 import _lib, crypto, duties
from oracle import duties_oracle as do
from tests import aggregate_grid_cases as gc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _wall():
    t = time.time()
    yield
    print(f"\ntest_aggregate_grid_gpu.py wall {time.time() - t:.1f} s")


def sm_count() -> int:
    import torch
    return torch.cuda.get_device_properties(int(os.environ.get("LOCAL_RANK", "0"))).multi_processor_count


def counted(fn):
    L = _lib.lib()
    c0 = L.b200_launch_count()
    r = fn()
    return r, L.b200_launch_count() - c0


def _single(items):
    flat = b"".join(gc.item_bytes(it) for it in items)
    out = (C.c_uint8 * 96)()
    code = _lib.lib().b200_aggregate(flat, len(items), out)
    return int(code), bytes(out) if code == 0 else None


def _oracle(O, items):
    out = C.create_string_buffer(96)
    code = O.orc_aggregate(b"".join(gc.item_bytes(it) for it in items), len(items), out)
    return int(code), out.raw if code == 0 else None


def _where(call, m, gi, g):
    bad = [i for i, it in enumerate(g.items) if isinstance(it, bytes) and it != gc.INF_SIG][:4]
    return (f"call {call.name}, group {gi} '{g.name}', chunk {m.chunk}, {call.sms} SMs, invalid at "
            + (", ".join(f"{i} (chunk {m.where(gi, i)[1]} lane {m.where(gi, i)[2]} pass {m.where(gi, i)[3]})" for i in bad) or "none"))


def _run_calls(calls, O, oracle_max):
    bad = []
    checked = set()
    for call in calls:
        m = call.map
        flat, off = gc.flat_sigs(call.groups)
        (out, codes), k = counted(lambda: crypto.aggregate_batch(flat, off))
        if k != m.launches:
            bad.append(f"call {call.name}: {k} launches, want {m.launches}")
        for gi, (g, o, c) in enumerate(zip(call.groups, out, codes)):
            row = (int(c), bytes(o) if c == 0 else None)
            if c != 0 and bytes(o) != bytes(96):
                bad.append(_where(call, m, gi, g) + ": failed row not zero")
            if row != g.want:
                bad.append(_where(call, m, gi, g) + (f": got code {row[0]}, want {g.want[0]}" if row[0] != g.want[0] else ": bytes differ"))
            if not g.items or g.claim.get("filler") or id(g) in checked:
                continue
            checked.add(id(g))
            if _single(g.items) != g.want:
                bad.append(_where(call, m, gi, g) + ": single aggregate differs")
            if len(g.items) <= oracle_max and _oracle(O, g.items) != g.want:
                bad.append(_where(call, m, gi, g) + ": C oracle differs")
    return bad


def test_filled_calls(engine, oracle_bls_c):
    sms = sm_count()
    crypto.aggregate_batch(np.frombuffer(gc.INF_SIG, dtype=np.uint8), [0, 1])   # the process's one-time set-up launches
    calls = gc.sig_calls(sms)
    assert {c.map.chunk for c in calls} == {32, 64, 96, 128}
    bad = _run_calls(calls, oracle_bls_c, 150)
    assert not bad, "\n".join(bad[:20])


def test_cta_edge_calls_and_no_signatures(engine, oracle_bls_c):
    sms = sm_count()
    calls = gc.edge_calls(sms)
    assert [c.map.cta for c in calls] == [32, 128]
    bad = _run_calls(calls, oracle_bls_c, 0)
    assert not bad, "\n".join(bad[:20])
    (out, codes), k = counted(lambda: crypto.aggregate_batch(np.zeros(0, np.uint8), [0, 0, 0, 0]))
    assert codes.tolist() == [gc.EMPTY] * 3 and not out.any() and k == gc.g2_map([0, 0, 0], sms).launches == 1


# ------------------------------------------------------------------------------------------------ keys (K2)
def _key_rows(out, codes):
    return [(int(c), bytes(o) if c == 0 else None) for o, c in zip(out, codes)]


def _mismatch(path, T, gs, got):
    return [f"{path} T={T} tuple {t} (CTA {t // 4} warp {t % 4}) '{g.name}': got {r[0]}, want {g.want[0]}"
            for t, (g, r) in enumerate(zip(gs, got)) if r != g.want]


def test_key_groups_every_path(engine):
    keys, where = gc.registry_keys()
    reg = crypto.Registry(np.frombuffer(b"".join(keys), dtype=np.uint8))
    codes = reg.key_codes().tolist()
    assert [codes[where[s]] for s in where] == [s[0] for s in where]
    # extra keys of the mixed call: the second invalid key of each code, so that p reads the registry and p + gap the call
    extra = [gc.key_bytes((c, 1)) for c in gc.KEY_CODES]
    xidx = {(c, 1): reg.n + j for j, c in enumerate(gc.KEY_CODES)}
    bad = []
    for T in gc.KEY_T:
        gs = gc.key_call(T)
        flat = np.frombuffer(b"".join(gc.key_bytes(s) for g in gs for s in g.slots), dtype=np.uint8)
        off = np.cumsum([0] + [len(g.slots) for g in gs]).astype(np.uint32)
        (out, cs), k = counted(lambda: crypto.eth_aggregate_public_keys_batch(flat, off))
        bad += _mismatch("strict aggregate", T, gs, _key_rows(out, cs)) + ([f"strict T={T}: {k} launches"] if k != 3 else [])
        idx = np.array([s if isinstance(s, int) else where[s] for g in gs for s in g.slots], dtype=np.uint32)
        (rout, rcs), k = counted(lambda: reg.aggregate_public_keys(idx, off))
        bad += _mismatch("registry aggregate", T, gs, _key_rows(rout, rcs)) + ([f"registry T={T}: {k} launches"] if k != 2 else [])
        msgs = np.frombuffer(b"".join(gc.verify_msg(t) for t in range(T)), dtype=np.uint8)
        sigs = np.frombuffer(gc.verify_sig() * T, dtype=np.uint8)
        want = [gc.verify_want(g) for g in gs]
        for path, got in (("strict verify", crypto.fast_aggregate_verify_batch(flat, off, msgs, sigs)),
                          ("registry verify", reg.verify_batch(idx, off, msgs, sigs))):
            bad += [f"{path} T={T} tuple {t} '{g.name}': got {int(c)}, want {w}" for t, (g, c, w) in enumerate(zip(gs, got, want)) if c != w]
        midx = np.array([s if isinstance(s, int) else xidx.get(s, where[s]) for g in gs for s in g.slots], dtype=np.uint32)
        got = reg.verify_batch(midx, off, msgs, sigs, extra_keys=np.frombuffer(b"".join(extra), dtype=np.uint8))
        bad += [f"mixed verify T={T} tuple {t} '{g.name}': got {int(c)}, want {w}" for t, (g, c, w) in enumerate(zip(gs, got, want)) if c != w]
    assert not bad, "\n".join(bad[:20])
    assert reg.key_codes().tolist() == codes


def test_sync_committee_two_invalid_keys_on_one_lane(engine):
    from tests.test_duties_gpu import upload
    st = gc.sync_state()
    want_idx = do.next_sync_committee_indices(st, "list")
    dev = upload(st)
    idx, committee, code = duties.next_sync_committee(dev)
    assert idx.tolist() == want_idx and code == 0
    recs = st.validators
    inv = gc.key_material()[4]
    bad = []
    for p, q, c1, c2 in gc.sync_cases(want_idx):
        vp, vq = want_idx[p], want_idx[q]
        rp, rq = recs[vp].copy(), recs[vq].copy()
        rp["public_key"] = np.frombuffer(inv[c1][0], dtype="V48")[0]
        rq["public_key"] = np.frombuffer(inv[c2][1], dtype="V48")[0]
        dev.update_elements("validators", [vp, vq], rp.tobytes() + rq.tobytes())
        got_idx, got_committee, got = duties.next_sync_committee(dev)
        if got_idx.tolist() != want_idx or got != c1 or got_committee != bytes(len(got_committee)):
            bad.append(f"positions {p} (lane {p % 32} pass {p // 32}) and {q} (pass {q // 32}), codes {c1}, {c2}: got {got}")
        dev.update_elements("validators", [vp, vq], recs[vp].tobytes() + recs[vq].tobytes())
    again = duties.next_sync_committee(dev)
    dev.close()
    assert not bad, "\n".join(bad)
    assert again[2] == 0 and again[1] == committee
