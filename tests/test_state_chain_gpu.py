"""GPU: one device-resident BeaconState per leg, driven epoch after epoch by the scripts of tests/state_chain_cases.py,
every answer against its oracle on the host mirror.

Each leg runs block writes, a query phase, attestations whose attesting indices decide the participation flags, and
process_epoch, across a relocation of the five big lists (minimal: 200 validators filled to exactly their reserved
capacity, then one past it, then 11 more epochs; mainnet: 2^18 validators past 2^18 + 2^16).  The query phase compares
committee_count_per_slot, beacon_committees and attester_duties of the previous, current and next epoch (all validators,
and lists holding inactive, repeated and out-of-range indices), proposer_indices, get_seed, next_sync_committee,
sync_committee_indices and state_shuffled_active_indices.  After each process_epoch and each relocation the whole
serialization is read back byte for byte and the incremental, full and one-shot roots equal the C oracle's.  The
validated-key registry is loaded from the handle before the relocation and synced after every deposit block: key codes
and the current sync committee's aggregate against the strict batch on the mirror's keys.  Committee-cache probes count
launches around each invalidating write.  A mismatch names the leg, epoch, step and call, to replay from the seed.
"""
from __future__ import annotations

import ctypes as C
import os
import time
from collections import Counter

import numpy as np
import pytest

from ethereum_consensus_b200 import _lib, crypto, duties, epoch, shuffling, ssz
from ethereum_consensus_b200 import state as S
from oracle import duties_oracle as do
from oracle import epoch_oracle as eo
from oracle import shuffle_oracle as sh
from tests import committee_oracle as co
from tests import state_chain_cases as cc

pytestmark = pytest.mark.gpu
NT = os.cpu_count() or 1
BIG = ("validators", "balances", "previous_epoch_participation", "current_epoch_participation", "inactivity_scores")
DOMAINS = (duties.DOMAIN_BEACON_PROPOSER, duties.DOMAIN_BEACON_ATTESTER, duties.DOMAIN_SYNC_COMMITTEE)


def c_root(O, st) -> bytes:
    b = S.serialize(st)
    out = C.create_string_buffer(32)
    assert O.orc_htr_beacon_state_deneb(b.ctypes.data, b.size, _lib.PRESET[st.preset], NT, out) == 0
    return out.raw


def duty_rows(st, e, committees) -> np.ndarray:
    """uint64[n, 5]: get_committee_assignment of every validator from the oracle's committees (NOT_ACTIVE if on none)."""
    rows = np.full((len(st.validators), 5), co.NOT_ACTIVE, np.uint64)
    cps = len(committees) // co.spe(st)
    for k, m in enumerate(committees):
        m = np.asarray(m, np.int64)
        rows[m] = np.stack([np.full(m.size, e * co.spe(st) + k // cps), np.full(m.size, k % cps), np.full(m.size, m.size),
                            np.full(m.size, cps), np.arange(m.size)], 1).astype(np.uint64)
    return rows


class Leg:
    def __init__(self, name, O, B):
        self.spec = cc.leg_spec(name)
        self.O = O
        self.aggregate = lambda keys: self._c_aggregate(B, keys)
        self.st, self.steps = cc.run(self.spec)
        self.dev = ssz.DeviceBeaconState(S.serialize(self.st), self.st.preset)
        self.L = _lib.lib()
        self.cap = len(self.st.validators) + cc.rc.headroom(len(self.st.validators))
        self.counts, self.relocations, self.reg, self.codes = Counter(), [], None, None
        self.epoch, self.pos, self.attested = None, 0, None

    @staticmethod
    def _c_aggregate(B, keys):
        out = C.create_string_buffer(48)
        code = B.orc_eth_aggregate_public_keys(b"".join(keys), len(keys), out)
        return int(code), out.raw if code == 0 else None

    def at(self, call) -> str:
        return f"leg {self.spec['name']} seed {self.spec['seed']:#x} epoch {self.epoch} step {self.pos}: {call}"

    def eq(self, got, want, call, family):
        assert got == want, self.at(call)
        self.counts[family] += 1

    def launches(self, fn):
        c0 = self.L.b200_launch_count()
        r = fn()
        return r, self.L.b200_launch_count() - c0

    # ------------------------------------------------------------------------------------------------------ steps
    def run(self):
        for self.pos, step in enumerate(self.steps):
            getattr(self, "do_" + step[0], self.do_write)(step)
            self.counts["steps"] += 1
        self.dev.close()

    def do_epoch(self, step):
        self.epoch = step[1]
        self.counts["epochs"] += 1

    def do_write(self, step):
        kind, h, n0 = step[0], self.dev, len(self.st.validators)
        cc.apply(self.st, step)
        if self.attested is not None:
            assert kind == "elements" and step[1] == "current_epoch_participation", self.at("flags after attest")
            assert set(np.asarray(step[2]).tolist()) == self.attested, self.at("flags from the device attesting indices")
            self.attested = None
        if kind == "push":
            h.append_elements(step[1], step[2])
        elif kind == "set":
            h.set_field(step[1], step[2])
        elif kind == "deposits":
            h.add_validators(step[1], step[2])
            n = len(self.st.validators)
            if n > self.cap:
                self.relocations.append((self.epoch, n0, n, self.cap))
                self.cap = n + cc.rc.headroom(n)
        elif kind == "elements":
            h.update_elements(step[1], step[2], step[3])
        elif kind == "bytes":
            h.update_bytes(step[1], step[2])
        else:
            raise ValueError(kind)
        assert h.n_validators == len(self.st.validators), self.at(kind)

    def do_process_epoch(self, step):
        m = step[1]
        try:
            post, code = eo.process_epoch(self.st, m, aggregate=self.aggregate)
        except eo.Refused as r:
            rc = self.L.b200_state_process_epoch(self.dev._h, m, C.byref(C.c_int32(0)))
            self.eq(rc, {"bad_arg": _lib.ERR_BAD_ARG, "limit": _lib.ERR_LIMIT}[r.kind], f"process_epoch({m:#x}) refused",
                    "process_epoch")
            self.eq(self.dev.read_bytes(0, self.dev.serialized_len()), S.serialize(self.st).tobytes(),
                    "state after a refused process_epoch", "read_bytes")
            return
        self.st.__dict__.update(post.__dict__)
        if code:
            with pytest.raises(crypto.BLSTError) as ei:
                epoch.process_epoch(self.dev, m)
            self.eq(ei.value.code, code, f"process_epoch({m:#x}) code", "process_epoch")
        else:
            epoch.process_epoch(self.dev, m)
            self.counts["process_epoch"] += 1

    def do_check(self, step):
        st, dev = self.st, self.dev
        want = S.serialize(st)
        lay = S.layout(st)
        for f in BIG:
            o, ln = lay[f]
            self.eq(dev.read_bytes(o, ln), getattr(st, f).tobytes(), f"read_bytes({f})", "read_bytes")
        got = dev.read_bytes(0, dev.serialized_len())
        if got != want.tobytes():
            bad = [k for k, (o, n) in lay.items() if got[o:o + n] != want[o:o + n].tobytes()]
            raise AssertionError(self.at(f"read_bytes of the serialization: fields differ {bad}"))
        self.counts["read_bytes"] += 1
        root = c_root(self.O, st)
        self.eq(dev.hash_tree_root_incremental(), root, "hash_tree_root_incremental", "roots")
        self.eq(dev.hash_tree_root(), root, "hash_tree_root", "roots")
        self.eq(ssz.hash_tree_root_beacon_state(want, st.preset), root, "hash_tree_root_beacon_state", "roots")

    def do_probe(self, step):
        _, e, expect, why = step
        (idx, off, cps), k = self.launches(lambda: duties.beacon_committees(self.dev, e))
        want = co.beacon_committees(self.st, e)
        self.eq([idx[off[j]:off[j + 1]].tolist() for j in range(len(off) - 1)], want, f"beacon_committees({e}) probe {why}",
                "committees")
        if expect == "hit":
            self.eq(k, 0, f"beacon_committees({e}) served from the cache ({why})", "cache")
        elif expect == "miss":
            assert k > 0, self.at(f"beacon_committees({e}) rebuilt after the {why} write")
            self.counts["cache"] += 1

    def do_registry(self, step):
        n = len(self.st.validators)
        keys = np.ascontiguousarray(self.st.validators["public_key"]).view(np.uint8).reshape(n, 48)
        if step[1] == "load":
            self.reg, lo, prev = crypto.Registry.from_state(self.dev), 0, np.zeros(0, np.int32)
        else:
            lo, prev = len(self.codes), self.codes
            self.reg.sync(self.dev)
        self.eq(self.reg.n, n, f"registry {step[1]} n", "registry")
        codes = self.reg.key_codes()
        _, strict = crypto.eth_aggregate_public_keys_batch(np.ascontiguousarray(keys[lo:]).reshape(-1),
                                                           np.arange(n - lo + 1, dtype=np.uint32))
        self.eq(codes[:lo].tolist(), prev.tolist(), "key_codes of the keys loaded before", "registry")
        self.eq(codes[lo:].tolist(), strict.tolist(), f"key_codes {lo}..{n} against the strict batch", "registry")
        self.codes = codes.copy()
        self.registry_sync_committee(keys)

    def registry_sync_committee(self, keys):
        idx = np.array([i for i in do.sync_committee_indices(self.st, "current") if i != do.MISSING], np.uint32)
        off = np.array([0, idx.size], np.uint32)
        rout, rcodes = self.reg.aggregate_public_keys(idx, off)
        sout, scodes = crypto.eth_aggregate_public_keys_batch(np.ascontiguousarray(keys[idx.astype(np.int64)]).reshape(-1), off)
        self.eq((rcodes.tolist(), rout.tobytes()), (scodes.tolist(), sout.tobytes()),
                "registry aggregate_public_keys of the current sync committee", "registry")

    def do_attest(self, step):
        atts = step[1]
        got, codes = duties.attesting_indices(self.dev, atts)
        cache, self.attested = {}, set()
        cur = do.slot(self.st) // co.spe(self.st)
        for a, ((d, b), g, c) in enumerate(zip(atts, got, codes)):
            w_code, w_idx = co.attesting_indices(self.st, d, b, committees=cache)
            self.eq((int(c), g.tolist()), (w_code, w_idx), f"attesting_indices[{a}]", "attesting_indices")
            if c == 0 and int.from_bytes(d[88:96], "little") == cur:
                self.attested.update(g.tolist())
        self.attested = self.attested or None
        assert any(c != 0 for c in codes) and any(c == 0 for c in codes), self.at("attesting_indices codes")

    def do_query(self, step):
        e, st, dev = step[1], self.st, self.dev
        n = len(st.validators)
        rounds = do.PRESET[st.preset]["SHUFFLE_ROUND_COUNT"]
        for ep in (e - 1, e, e + 1):
            self.eq(duties.committee_count_per_slot(dev, ep), co.committee_count_per_slot(st, ep),
                    f"committee_count_per_slot({ep})", "committees")
            want = co.beacon_committees(st, ep)
            idx, off, cps = duties.beacon_committees(dev, ep)
            self.eq((cps, [idx[off[j]:off[j + 1]].tolist() for j in range(len(off) - 1)]), (len(want) // co.spe(st), want),
                    f"beacon_committees({ep})", "committees")
            rows = duty_rows(st, ep, want)
            got = duties.attester_duties(dev, ep).view(np.uint64).reshape(-1, 5)
            self.eq(np.array_equal(got, rows), True, f"attester_duties({ep}, None)", "attester_duties")
            inactive = np.nonzero(rows[:, 0] == co.NOT_ACTIVE)[0][-3:]
            some = np.concatenate([[n - 1, 0, 0], inactive, [n // 2, 3, 5]]).astype(np.uint64)
            got = duties.attester_duties(dev, ep, some).view(np.uint64).reshape(-1, 5)
            self.eq(got.tolist(), rows[some.astype(np.int64)].tolist(), f"attester_duties({ep}, {some.tolist()})",
                    "attester_duties")
            with pytest.raises(_lib.EngineError) as ei:
                duties.attester_duties(dev, ep, np.array([0, n, 1], np.uint64))
            self.eq(ei.value.code, _lib.ERR_BAD_ARG, f"attester_duties({ep}) with index {n} refused", "attester_duties")
            for dom in DOMAINS:
                self.eq(duties.get_seed(dev, ep, dom), do.get_seed(st, ep, dom), f"get_seed({ep}, {dom.hex()})", "get_seed")
        for ep in (e, e + 1):
            self.eq(duties.proposer_indices(dev, ep).tolist(), do.proposer_indices(st, ep), f"proposer_indices({ep})",
                    "proposer_indices")
        idx, blob, code = duties.next_sync_committee(dev)
        w_idx, w_blob, w_code = do.next_sync_committee(st, self.aggregate, "list")
        self.eq((idx.tolist(), blob, code), (w_idx, w_blob, w_code), "next_sync_committee", "sync")
        for which in ("current", "next"):
            self.eq(duties.sync_committee_indices(dev, which, missing_ok=True).tolist(), do.sync_committee_indices(st, which),
                    f"sync_committee_indices({which})", "sync")
        seed = duties.get_seed(dev, e, duties.DOMAIN_BEACON_ATTESTER)
        self.eq(shuffling.state_shuffled_active_indices(dev, e, seed, rounds).tolist(),
                sh.shuffled_indices_numpy(do.active_indices(st, e), seed, rounds).tolist(),
                f"state_shuffled_active_indices({e})", "shuffling")


@pytest.mark.parametrize("name", ["minimal", "mainnet"])
def test_leg(engine, oracle_ssz_c, oracle_bls_c, name):
    t = time.time()
    leg = Leg(name, oracle_ssz_c, oracle_bls_c)
    leg.run()
    c = leg.counts
    print(f"\n{name}: {c['epochs']} epochs, {c['steps']} steps, relocations (epoch, n before, n after, capacity) "
          f"{leg.relocations}, wall {time.time() - t:.1f} s")
    print("  compared: " + ", ".join(f"{k} {v}" for k, v in sorted(c.items()) if k not in ("epochs", "steps")))
    spec = leg.spec
    assert c["epochs"] == spec["epochs"]
    assert [r[0] for r in leg.relocations] == [spec["cross"]]
    assert c["cache"] > 0 and c["registry"] > 0 and c["attesting_indices"] > 0 and c["process_epoch"] >= spec["epochs"]
