"""Seeded scripts that drive one device-resident deneb BeaconState across many epochs (no device code, no torch).

A leg is one handle's life: an upload, then epoch after epoch of
  1. block writes (tests/state_reshape_cases.py steps): eth1 votes, deposits through add_validators, slot / block_roots /
     state_roots / randao_mixes through update_bytes, slashings as Validator record writes, balance writes;
  2. a query phase: every committee, duty, seed, sync-committee and shuffling call is compared with its oracle;
  3. attestations: their attesting indices decide the current epoch's participation flags (update_elements);
  4. process_epoch, with all sub-steps or with one.
The first big deposit block fills the five big lists to exactly their reserved capacity, the next one crosses it, so that
everything after runs on relocated device buffers.  Committee-cache probes sit around the three kinds of write that must
invalidate a cached epoch: a relocation, a process_epoch that changed records, a randao mix that changes the seed.

Steps are tuples.  Besides the kinds of state_reshape_cases.apply:
  ("bytes", offset, data)         update_bytes inside slot / block_roots / state_roots / randao_mixes / slashings
  ("epoch", e)                    marks the start of epoch e's steps
  ("process_epoch", mask)         the mirror runs oracle/epoch_oracle.py; a mask above bit 11 is refused
  ("query", epoch)                the query phase at the state as it is
  ("attest", [(data, bits)])      attesting_indices of a batch; the next step writes the flags they decide
  ("probe", epoch, expect, why)   beacon_committees(epoch): "hit" served from the cache, "miss" rebuilt, "any"
  ("registry", "load" | "sync")   Registry.from_state / Registry.sync
  ("check",)                      bytes and roots of the whole state
Scripts are generators over the mirror: after each yielded step the caller applies it with `apply` (and, on the GPU, to
the handle); the next step is computed from the mirror as it then is.

tests/test_state_chain_cases.py checks on the CPU that the scripts reach every event in `EVENTS`; tests/
test_state_chain_gpu.py runs them through the CUDA library.
"""
from __future__ import annotations

import hashlib
import sys
from functools import lru_cache
from pathlib import Path
from typing import Iterator

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from ethereum_consensus_b200 import state as S  # noqa: E402
from oracle import duties_oracle as do  # noqa: E402
from oracle import epoch_oracle as eo  # noqa: E402
from tests import committee_oracle as co  # noqa: E402
from tests import epoch_cases as ec  # noqa: E402
from tests import state_reshape_cases as rc  # noqa: E402

ETH = 10**9
FAR = S.FAR_FUTURE_EPOCH
POOL = 192                     # distinct valid keys; validator i of a tiled list carries pool key i % POOL
BAD_MASK = 1 << 12             # a process_epoch mask bit above the twelve sub-steps: refused
TARGET_FLAG = 1 << 1           # TIMELY_TARGET_FLAG_INDEX

EVENTS = ("relocation minimal", "relocation mainnet", "capacity exactly filled", "capacity crossed by one",
          "10 epochs after the relocation", "sync period 1", "sync period 2", "sync rotation right after a relocation",
          "eth1 votes reset", "historical summary appended", "activation queue", "appended validators activated",
          "ejection", "exit", "cache: relocation", "cache: process_epoch records", "cache: randao seed",
          "process_epoch single steps", "process_epoch refused")


@lru_cache(maxsize=None)
def pool_keys() -> np.ndarray:
    return ec.valid_pubkeys(POOL)


def bad_keys(n: int, seed: int) -> np.ndarray:
    """Compressed-looking keys that do not decode to a curve point (or the infinity encoding)."""
    k = np.random.default_rng(seed).integers(0, 256, (n, 48), dtype=np.uint8)
    k[:, 0] = (k[:, 0] & 0x1F) | 0x80
    if n:
        k[0] = 0
        k[0, 0] = 0xC0
    return k


def leg_spec(name: str) -> dict:
    """`small` is the minimal leg at a few hundred validators (the oracle's literal formulation keeps up with it):
    the reserved capacity is modelled as 64 + 16 instead of 2^16 and no relocation happens on a device."""
    if name == "minimal":
        return dict(name=name, preset="minimal", n0=200, e0=44, epochs=14, fill=45, cross=46, randao=50,
                    singles={49: "registry_updates", 52: "effective_balance_updates"}, refuse=53,
                    eject=47, exit=(46, 50), slash={45: 2, 51: 2}, seed=0xC4A1, headroom=rc.headroom)
    if name == "small":
        return dict(leg_spec("minimal"), name=name, n0=64, headroom=lambda n: max(16, n // 16))
    if name == "mainnet":
        return dict(name=name, preset="mainnet", n0=1 << 18, e0=1000, epochs=4, fill=None, cross=1001, randao=1002,
                    singles={1003: "effective_balance_updates"}, refuse=None, eject=None, exit=None, slash={1000: 2},
                    seed=0xC4A2, headroom=rc.headroom)
    raise ValueError(name)


def initial_state(spec: dict) -> S.SynthState:
    n, e0, preset = spec["n0"], spec["e0"], spec["preset"]
    st = ec.base(n, e0, preset, seed=spec["seed"])
    keys = pool_keys()[np.arange(n) % POOL]
    st.validators["public_key"] = keys.view("V48").reshape(n)
    size = do.PRESET[preset]["SYNC_COMMITTEE_SIZE"]
    st.current_sync_committee = keys[np.arange(size) % n].tobytes() + bytes(48)
    st.next_sync_committee = keys[(np.arange(size) * 7 + 1) % n].tobytes() + bytes(48)
    st.fixed["slot"] = int(e0 * co.spe(st)).to_bytes(8, "little")
    return st


# ---------------------------------------------------------------------------------------------------------- the mirror
def _patch(st: S.SynthState, off: int, data: bytes) -> None:
    lay = S.layout(st)
    for name in ("slot", "block_roots", "state_roots", "randao_mixes", "slashings"):
        o, ln = lay[name]
        if o <= off and off + len(data) <= o + ln:
            if name == "slot":
                b = bytearray(st.fixed["slot"])
                b[off - o:off - o + len(data)] = data
                st.fixed["slot"] = bytes(b)
            else:
                getattr(st, name).view(np.uint8).reshape(-1)[off - o:off - o + len(data)] = np.frombuffer(data, np.uint8)
            return
    raise ValueError(f"update_bytes at {off}: not inside a field these scripts write")


def apply(st: S.SynthState, step: tuple, aggregate=None):
    """Apply one step to the mirror.  process_epoch returns its aggregation code and raises epoch_oracle.Refused where
    the library refuses; the query, probe, registry and check markers change nothing."""
    kind = step[0]
    if kind == "bytes":
        _patch(st, step[1], bytes(step[2]))
    elif kind == "process_epoch":
        post, code = eo.process_epoch(st, step[1], aggregate=aggregate)
        st.__dict__.update(post.__dict__)
        return code
    elif kind in ("epoch", "query", "attest", "probe", "registry", "check"):
        pass
    else:
        rc.apply(st, step)
    return None


# ---------------------------------------------------------------------------------------------------------- step values
def deposit_records(rng, n: int, lo: int, epoch: int, bad: int = 0) -> tuple:
    """`n` deposits for validators lo .. lo + n - 1 carrying tiled pool keys: about half of them already active (so that
    committees and duties see appended validators at once), the rest as add_validator_to_registry leaves them (waiting
    for eligibility, then for activation under the churn limit).  The last `bad` carry undecodable keys and 1 ETH, so
    that they are never eligible and never sit on a committee."""
    v = np.zeros(n, dtype=S.VALIDATOR_DTYPE)
    keys = pool_keys()[np.arange(lo, lo + n) % POOL].copy()
    if bad:
        keys[n - bad:] = bad_keys(bad, lo)
    v["public_key"] = keys.view("V48").reshape(n)
    wc = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    wc[:, 0] = 1
    v["withdrawal_credentials"] = wc.view("V32").reshape(n)
    v["effective_balance"] = 32 * ETH
    active = rng.random(n) < 0.5
    v["activation_eligibility_epoch"] = np.where(active, np.uint64(max(0, epoch - 3)), np.uint64(FAR))
    v["activation_epoch"] = np.where(active, np.uint64(max(0, epoch - 2)), np.uint64(FAR))
    v["exit_epoch"] = FAR
    v["withdrawable_epoch"] = FAR
    bal = (32 * ETH + rng.integers(0, ETH // 2, n, dtype=np.uint64)).astype("<u8")
    if bad:
        v["effective_balance"][n - bad:] = ETH
        v["activation_eligibility_epoch"][n - bad:] = FAR
        v["activation_epoch"][n - bad:] = FAR
        bal[n - bad:] = ETH
    return ("deposits", v.tobytes(), bal)


def record_write(st, idx, **fields) -> tuple:
    recs = st.validators[np.asarray(idx, np.int64)].copy()
    for k, val in fields.items():
        recs[k] = val
    return ("elements", "validators", np.asarray(idx, np.uint64), recs.tobytes())


def attestations(st, e: int, rng, sample: int | None):
    """Attestations of epoch `e` for every committee of slots e * SPE .. e * SPE + SPE - 2 (or `sample` of them), about
    nine in ten members set, then three that fail: a target two epochs back, a Bitlist one bit short, an index past the
    committee count.  -> (list of (data, bits), {validator: flags})."""
    spe = co.spe(st)
    comm = co.beacon_committees(st, e)
    cps = len(comm) // spe
    pairs = [(s, i) for s in range(spe - 1) for i in range(cps)]
    if sample is not None and sample < len(pairs):
        pairs = [pairs[int(k)] for k in np.sort(rng.choice(len(pairs), sample, replace=False))]
    atts, flags = [], {}
    for s, i in pairs:
        members = comm[s * cps + i]
        bits = rng.random(len(members)) < 0.9
        root = hashlib.sha256(b"%d:%d:%d" % (e, s, i)).digest()
        atts.append((co.attestation_data(e * spe + s, i, e, root=root), co.bitlist(bits.tolist())))
        f = TARGET_FLAG | int(rng.integers(0, 8))
        for v, b in zip(members, bits):
            if b:
                flags[v] = flags.get(v, 0) | f
    members = comm[0]
    atts.append((co.attestation_data((e - 2) * spe, 0, e - 2), co.bitlist([True] * 3)))
    atts.append((co.attestation_data(e * spe, 0, e), co.bitlist([True] * (len(members) - 1))))
    atts.append((co.attestation_data(e * spe + 1, cps, e), co.bitlist([True] * len(members))))
    return atts, flags


def _u64s(rng, n, lo, hi) -> bytes:
    return rng.integers(lo, hi, n, dtype=np.uint64).astype("<u8").tobytes()


# ---------------------------------------------------------------------------------------------------------- the script
def script(spec: dict, st: S.SynthState) -> Iterator[tuple]:
    rng = np.random.default_rng(spec["seed"])
    P = S.PRESETS[st.preset]
    spe = co.spe(st)
    sphr, ehv = P["SLOTS_PER_HISTORICAL_ROOT"], P["EPOCHS_PER_HISTORICAL_VECTOR"]
    mainnet = st.preset == "mainnet"
    cap = len(st.validators) + spec["headroom"](len(st.validators))
    yield ("registry", "load")
    for e in range(spec["e0"], spec["e0"] + spec["epochs"]):
        yield ("epoch", e)
        lay = S.layout(st)
        # ---- 1. blocks: two per epoch, the second at the epoch's last slot (where process_epoch runs)
        for j, slot in enumerate((e * spe + 1, e * spe + spe - 1)):
            n = len(st.validators)
            yield ("push", "eth1_data_votes", rc.vote(rng, slot))
            yield ("bytes", lay["slot"][0], int(slot).to_bytes(8, "little"))
            yield ("bytes", lay["block_roots"][0] + 32 * (slot % sphr), rng.integers(0, 256, 32, dtype=np.uint8).tobytes())
            yield ("bytes", lay["state_roots"][0] + 32 * (slot % sphr), rng.integers(0, 256, 32, dtype=np.uint8).tobytes())
            yield ("bytes", lay["randao_mixes"][0] + 32 * (e % ehv), rng.integers(0, 256, 32, dtype=np.uint8).tobytes())
            if e == spec["fill"] and j == 0:
                k, bad = cap - n, 3                      # exactly the reserved capacity
            elif e == spec["cross"] and j == 0:
                if spec["fill"] is None:
                    k, bad = cap - n + 1, 0              # past the capacity in one block
                else:
                    k, bad = 1, 0                        # one past it
                yield ("probe", e, "any", "relocation")
                yield ("probe", e, "hit", "relocation")
            elif spec["fill"] is not None and spec["fill"] <= e < spec["cross"]:
                k, bad = 0, 0                            # the lists stay exactly at capacity until the crossing block
            else:
                k, bad = int(rng.integers(0, rc.MAX_DEPOSITS + 1)), int(j == 1 and e % 3 == 0)
                k = max(k, bad)
            if k:
                yield deposit_records(rng, k, n, e, bad)
                if len(st.validators) > cap:
                    cap = len(st.validators) + spec["headroom"](len(st.validators))
                    yield ("check",)
                    yield ("probe", e, "miss", "relocation")
                yield ("registry", "sync")
            n = len(st.validators)
            idx = np.unique(np.concatenate([rng.integers(0, n, 6), np.arange(max(0, n - k), n)[:6]])).astype(np.uint64)
            if spec["eject"] is not None and e == spec["eject"] and j == 0:
                idx = np.union1d(idx, [3]).astype(np.uint64)
            bal = np.frombuffer(_u64s(rng, len(idx), 31 * ETH, 33 * ETH), "<u8").copy()
            if spec["eject"] is not None and e == spec["eject"] and j == 0:
                bal[np.searchsorted(idx, 3)] = 15 * ETH + ETH // 2     # effective 15 ETH at this epoch, ejected at the next
            yield ("elements", "balances", idx, bal.tobytes())
            if j == 1 and e in spec["slash"]:
                act = do.active_indices(st, e)
                act = act[(st.validators["slashed"][act.astype(np.int64)] == 0) & (act != 3)]
                who = np.sort(rng.choice(act, spec["slash"][e], replace=False))
                half = P["EPOCHS_PER_SLASHINGS_VECTOR"] // 2
                yield record_write(st, who, slashed=1, exit_epoch=e + 5, withdrawable_epoch=e + half)
                s_off = lay["slashings"][0] + 8 * (e % P["EPOCHS_PER_SLASHINGS_VECTOR"])
                yield ("bytes", s_off, int(st.slashings[e % P["EPOCHS_PER_SLASHINGS_VECTOR"]] + 64 * ETH).to_bytes(8, "little"))
            if spec["exit"] is not None and e == spec["exit"][0] and j == 1:
                yield record_write(st, [5], exit_epoch=spec["exit"][1])
        # ---- 2. queries
        yield ("query", e)
        if e == spec["randao"]:
            yield ("probe", e + 1, "any", "randao")
            yield ("probe", e + 1, "hit", "randao")
            m = (e + 1 + ehv - 2) % ehv                  # the mix get_seed(e + 1) reads
            yield ("bytes", lay["randao_mixes"][0] + 32 * m, hashlib.sha256(b"mix%d" % e).digest())
            yield ("probe", e + 1, "miss", "randao")
        # ---- 3. attestations decide the current epoch's flags
        atts, flags = attestations(st, e, rng, 48 if mainnet else None)
        yield ("attest", atts)
        if flags:
            who = np.array(sorted(flags), np.uint64)
            f = st.current_epoch_participation[who.astype(np.int64)] | np.array([flags[int(v)] for v in who], np.uint8)
            yield ("elements", "current_epoch_participation", who, f.astype(np.uint8).tobytes())
        # ---- 4. process_epoch
        if spec["refuse"] == e:
            yield ("process_epoch", BAD_MASK)
        yield ("probe", e + 1, "any", "process_epoch")
        yield ("probe", e + 1, "hit", "process_epoch")
        before = st.validators.copy()
        yield ("process_epoch", eo.mask([spec["singles"][e]]) if e in spec["singles"] else eo.ALL)
        yield ("check",)
        changed = not np.array_equal(before, st.validators)
        yield ("probe", e + 1, "miss" if changed else "hit", "process_epoch")


def run(spec: dict):
    """(initial mirror, step generator) of a leg."""
    st = initial_state(spec)
    return st, script(spec, st)


# ---------------------------------------------------------------------------------------------------------- events
class Events:
    """What a leg reached, derived from the mirror as the steps are applied (`observe` before and after each)."""

    def __init__(self, spec: dict, st: S.SynthState):
        self.spec, self.seen = spec, {}
        self.cap = len(st.validators) + spec["headroom"](len(st.validators))
        self.epoch, self.relocated_at, self.last_write = None, None, None

    def hit(self, name, where):
        self.seen.setdefault(name, where)

    def observe(self, st, step, pre: dict, epoch: int, pos: int):
        kind = step[0]
        where = (self.spec["name"], epoch, pos)
        if kind == "deposits":
            lens = {len(st.validators), len(st.balances), len(st.previous_epoch_participation),
                    len(st.current_epoch_participation), len(st.inactivity_scores)}
            assert len(lens) == 1
            n = lens.pop()
            if n == self.cap:
                self.hit("capacity exactly filled", where)
            if n > self.cap:
                if pre["n"] <= self.cap:
                    self.hit("relocation mainnet" if st.preset == "mainnet" else "relocation minimal", where)
                    if n == self.cap + 1 and pre["n"] == self.cap:
                        self.hit("capacity crossed by one", where)
                    self.relocated_at = epoch
                self.cap = n + self.spec["headroom"](n)
            self.last_write = "relocation" if pre["n"] <= pre["cap"] < n else "deposits"
        elif kind == "bytes":
            lay = S.layout(st)
            o, ln = lay["randao_mixes"]
            self.last_write = "randao" if o <= step[1] < o + ln else "bytes"
        elif kind == "process_epoch":
            if step[1] == BAD_MASK:
                self.hit("process_epoch refused", where)
                return
            if step[1] != eo.ALL:
                self.hit("process_epoch single steps", where)
            v0, v1 = pre["validators"], st.validators
            self.last_write = "process_epoch records" if not np.array_equal(v0, v1) else "process_epoch"
            if pre["sync"] != st.current_sync_committee:
                k = 2 if "sync period 1" in self.seen else 1
                self.hit(f"sync period {k}", where)
                if self.relocated_at is not None and epoch - self.relocated_at <= 2:
                    self.hit("sync rotation right after a relocation", where)
            if pre["votes"] and not len(st.eth1_data_votes):
                self.hit("eth1 votes reset", where)
            if len(st.historical_summaries) > pre["summaries"]:
                self.hit("historical summary appended", where)
            queue = (v1["activation_eligibility_epoch"] != FAR) & (v1["activation_epoch"] == FAR)
            if queue.any():
                self.hit("activation queue", where)
            new = np.nonzero((v0["activation_epoch"] == FAR) & (v1["activation_epoch"] != FAR))[0]
            if (new >= self.spec["n0"]).any():
                self.activated = getattr(self, "activated", set()) | {epoch}
                if len(self.activated) >= 2:
                    self.hit("appended validators activated", where)
            if ((v0["exit_epoch"] == FAR) & (v1["exit_epoch"] != FAR) & (v0["slashed"] == 0)).any():
                self.hit("ejection", where)
            if self.relocated_at is not None and epoch - self.relocated_at >= 10:
                self.hit("10 epochs after the relocation", where)
        elif kind == "query":
            e = step[1]
            if e > self.spec["e0"]:
                left = np.setdiff1d(do.active_indices(pre["st_prev_active"], e - 1), do.active_indices(st, e))
                if len(left):
                    self.hit("exit", where)
        elif kind == "probe" and step[2] == "miss":
            why = step[3]
            if why == "relocation" and self.last_write == "relocation":
                self.hit("cache: relocation", where)
            if why == "randao" and self.last_write == "randao":
                self.hit("cache: randao seed", where)
            if why == "process_epoch" and self.last_write == "process_epoch records":
                self.hit("cache: process_epoch records", where)


def snapshot(st, cap) -> dict:
    return dict(n=len(st.validators), cap=cap, validators=st.validators.copy(), sync=st.current_sync_committee,
                votes=len(st.eth1_data_votes), summaries=len(st.historical_summaries))


def walk(spec: dict, on_step=None, aggregate=None):
    """Apply a whole leg to its mirror (`on_step(st, step, epoch, pos)` after each).  -> (mirror, Events, digest of
    every step)."""
    st, steps = run(spec)
    ev = Events(spec, st)
    h = hashlib.sha256()
    epoch, prev_active = spec["e0"], None
    for pos, step in enumerate(steps):
        h.update(repr([x.tobytes() if isinstance(x, np.ndarray) else x for x in step]).encode())
        if step[0] == "epoch":
            epoch = step[1]
        pre = snapshot(st, ev.cap)
        pre["st_prev_active"] = prev_active
        try:
            apply(st, step, aggregate)
        except eo.Refused:
            assert step == ("process_epoch", BAD_MASK), step
        ev.observe(st, step, pre, epoch, pos)
        if step[0] == "query":
            prev_active = _Active(st.validators.copy())
        if on_step:
            on_step(st, step, epoch, pos)
    return st, ev, h.hexdigest()


class _Active:
    """Enough of a state for duties_oracle.active_indices."""

    def __init__(self, validators):
        self.validators = validators
