"""GPU: one long-lived engine across calls.  The session of tests/session_cases.py (every entry-point family interleaved,
shared buffers grown and shrunk, knobs and the VM schedule changed and restored, a refusal of every family followed by a
step of the same family) through the CUDA library, every answer against the oracles' answer in the step.

a. the session in script order (this process);
b. the same session in a seeded topological shuffle (dependent steps keep their order) in a child process; every answer
   equal to a's; a step that differs is replayed alone, with the steps it depends on, in a fresh child process;
d. four worker threads that never called b200_init, each with its own resident handle, running the session's state steps
   on it and a share of the one-shot, shuffle and batch steps, all at once; they read the registry and change nothing
   shared.  Every answer equal to a's.

    B200_SOAK_SCALE=1 (default) python -m pytest tests/test_engine_session_gpu.py -m gpu -s
"""
from __future__ import annotations

import pickle
import subprocess
import sys
import threading
import time
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from tests import session_cases as sn  # noqa: E402

pytestmark = pytest.mark.gpu
SHUFFLE_SEED = 0x0D0E
WORKERS = 4
CHILD_TIMEOUT = 1800


# ---------------------------------------------------------------------------------------------------------- the runner
class Context:
    """The resident objects a run of steps works on: one state handle and the process's registry."""

    def __init__(self, init_state):
        self.init_state = init_state
        self.state = None
        self.reg = None

    def close(self):
        if self.state is not None:
            self.state.close()
            self.state = None


def _refusal(e) -> tuple:
    from ethereum_consensus_b200 import _lib, ssz
    if isinstance(e, _lib.EngineError):
        return sn.refused(e.code)
    if isinstance(e, ssz.MerkleizationError):
        return sn.refused(_lib.ERR_LIMIT if "exceeds limit" in str(e) else _lib.ERR_SSZ_MALFORMED)
    raise e


def _fp_rows(values):
    out = np.zeros((len(values), 24), dtype=np.uint32)
    for i, x in enumerate(values):
        out[i, :12] = [(x >> (32 * k)) & 0xFFFFFFFF for k in range(12)]
    return out


def execute(step, ctx: Context):
    """Run one step through the library; its answer in the form the step's `want` has (a refusal as ("refused", code))."""
    from ethereum_consensus_b200 import _lib, crypto, shuffling, ssz
    a, op = step.args, step.op
    try:
        if step.family == "strict":
            return tuple(crypto.fast_aggregate_verify_batch(a["pks"], a["off"], a["msgs"], a["sigs"]).tolist())
        if step.family == "rlc":
            if op == "fast_aggregate_verify_batch_all":
                return crypto.fast_aggregate_verify_batch_all(a["pks"], a["off"], a["msgs"], a["sigs"], seed=a["seed"])
            return ctx.reg.verify_batch_all(a["idx"], a["off"], a["msgs"], a["sigs"], seed=a["seed"])
        if step.family == "single":
            return _single(op, a)
        if step.family == "registry":
            if op == "from_state":
                ctx.reg = crypto.Registry.from_state(ctx.state)
                return ctx.reg.n
            if op == "sync":
                ctx.reg.sync(ctx.state)
                return ctx.reg.n
            if op == "key_codes":
                return sn.digest(ctx.reg.key_codes().astype(np.int32))
            if op == "verify_batch":
                return tuple(ctx.reg.verify_batch(a["idx"], a["off"], a["msgs"], a["sigs"], extra_keys=a["extra"]).tolist())
            if op == "sync_smaller":
                small = ssz.DeviceBeaconState(a["ssz"], "minimal")
                try:
                    n = ctx.reg.n
                    ctx.reg.sync(small)
                    return ctx.reg.n
                except _lib.EngineError as e:
                    ctx.reg.n = n
                    return sn.refused(e.code)
                finally:
                    small.close()
        if step.family == "state":
            h = ctx.state
            if op == "upload":
                ctx.close()
                ctx.state = ssz.DeviceBeaconState(ctx.init_state, "minimal")
                return None
            if op == "state_root":
                return h.hash_tree_root()
            if op == "incremental_root":
                return h.hash_tree_root_incremental()
            if op == "add_validators":
                h.add_validators(a["records"], a["balances"])
                return None
            if op == "append_elements":
                h.append_elements(a["field"], a["values"])
                return None
            if op == "set_field":
                h.set_field(a["field"], a["data"])
                return None
            if op == "update_bytes":
                h.update_bytes(a["offset"], a["data"])
                return None
            if op == "state_shuffled_active_indices":
                return sn.digest(shuffling.state_shuffled_active_indices(h, a["epoch"], a["seed"], a["rounds"]).astype(np.uint64))
        if step.family == "ssz":
            if op == "hash":
                return ssz.hash(a["data"])
            if op == "merkleize":
                return ssz.merkleize(a["chunks"], a["limit"])
            if op == "htr_validators":
                return ssz.hash_tree_root_validators(a["ssz"])
            if op == "htr_beacon_state":
                return ssz.hash_tree_root_beacon_state(a["ssz"], a["preset"])
            if op == "is_valid_merkle_branch":
                return ssz.is_valid_merkle_branch(a["leaf"], a["branch"], a["depth"], a["index"], a["root"])
        if step.family == "shuffle":
            if op == "compute_shuffled_indices":
                return sn.digest(shuffling.compute_shuffled_indices(a["n"], a["seed"], a["rounds"]).astype(np.uint64))
            if op == "get_active_validator_indices":
                return sn.digest(shuffling.get_active_validator_indices(a["recs"], a["epoch"]).astype(np.uint64))
        if step.family == "eval":
            return _eval(op, a)
        if step.family == "settings":
            if op == "tune":
                crypto.tune(a["knob"], a["value"])
            else:
                crypto.vm_load_programs(a["blob"])
            return None
    except Exception as e:  # noqa: BLE001 - a refusal is an answer; anything else is re-raised by _refusal
        return _refusal(e)
    raise ValueError(f"unknown step {step.family}.{op}")


def _single(op, a):
    from ethereum_consensus_b200 import _lib, crypto
    fn = getattr(crypto, op)
    try:
        if op == "verify_signature":
            fn(a["pk"], a["msg"], a["sig"])
        elif op in ("fast_aggregate_verify", "eth_fast_aggregate_verify"):
            fn(a["pks"], a["msg"], a["sig"])
        elif op == "aggregate_verify":
            fn(a["pks"], a["msgs"], a["sig"])
        elif op == "aggregate":
            return (0, bytes(fn(a["sigs"])))
        elif op == "eth_aggregate_public_keys":
            return (0, bytes(fn(a["pks"])))
        return 0
    except crypto.InvalidSignature:
        code = _lib.VERIFY_FAIL
    except crypto.EmptyAggregate:
        code = _lib.EMPTY_AGGREGATE
    except crypto.BLSTError as e:
        code = e.code
    return (code, None) if op in ("aggregate", "eth_aggregate_public_keys") else code


def _eval(op, a):
    from ethereum_consensus_b200 import _lib, crypto
    from tests import pairing_cases as pc
    from tests.test_torsion_gpu import _aff_rec, _records
    from oracle import bls_oracle as bo
    if op == "fp_eval":
        out = crypto.fp_eval(a["op"], _fp_rows(a["a"]), _fp_rows(a["b"]))
        return tuple(sum(int(r[k]) << (32 * k) for k in range(12)) for r in out)
    if op == "curve_eval":
        recs = _records([_aff_rec(bo.F1, p) for p in a["pts"]])
        if isinstance(a["op"], int):     # an op id the library does not know
            out = np.zeros_like(recs)
            rc = _lib.lib().b200_curve_eval(a["op"], recs.shape[0], _lib.ptr(recs), _lib.ptr(np.zeros_like(recs)), _lib.ptr(out))
            return sn.refused(rc) if rc else tuple(out[:, 72].tolist())
        return tuple(crypto.curve_eval(a["op"], recs)[:, 72].tolist())
    if op == "pairing_eval":
        out = crypto.pairing_eval(a["op"], pc.pack(a["a"]), pc.pack(a["b"]))
        return tuple(tuple(pc.to_real(r)) for r in pc.unpack(out))
    raise ValueError(op)


def run_steps(steps, init_state, order=None, on_answer=None):
    """Answers of `steps` (run in `order`, default script order), indexed by step number."""
    ctx = Context(init_state)
    got = {}
    try:
        for j in (order if order is not None else range(len(steps))):
            got[steps[j].i] = execute(steps[j], ctx)
            if on_answer:
                on_answer(steps[j], got[steps[j].i])
    finally:
        ctx.close()
    return got


def mismatches(steps, got, want=None):
    """Indices whose answer differs from the step's `want` (or from the answers `want`)."""
    return [s.i for s in steps if s.i in got and got[s.i] != (s.want if want is None else want[s.i])]


# ---------------------------------------------------------------------------------------------------------- the session
_CACHE = {}


def session():
    if "s" not in _CACHE:
        t = time.time()
        s = sn.build_session()
        print(f"session: {len(s.steps)} steps, host-side oracles {time.time() - t:.1f} s")
        _CACHE["s"] = s
    return _CACHE["s"]


def _print_context(steps_by_i, order, i, got):
    """The step that differs and the three steps that ran just before it (the likely cause)."""
    pos = order.index(i)
    for j in order[max(0, pos - 3):pos + 1]:
        s = steps_by_i[j]
        mark = ">>" if j == i else "  "
        print(f"{mark} {s.describe()[:200]}")
        if j == i:
            print(f"   got  {got[j]!r}"[:300])
            print(f"   want {s.want!r}"[:300])


@pytest.fixture(scope="module")
def sequential(engine):
    s = session()
    t = time.time()
    got = run_steps(s.steps, s.init_state)
    wall = time.time() - t
    _CACHE["a"] = got
    return got, wall


def _child(mode, tmp_path, payload):
    path = tmp_path / f"{mode}.pkl"
    path.write_bytes(pickle.dumps(payload))
    out = tmp_path / f"{mode}.out.pkl"
    p = subprocess.run([sys.executable, "-m", "tests.test_engine_session_gpu", mode, str(path), str(out)], cwd=str(ROOT),
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                       timeout=CHILD_TIMEOUT)
    print(p.stdout[-4000:])
    assert p.returncode == 0, p.stdout[-4000:]
    return pickle.loads(out.read_bytes())


# ---------------------------------------------------------------------------------------------------------- a
def test_a_script_order(sequential):
    s = session()
    got, wall = sequential
    bad = mismatches(s.steps, got)
    order = list(range(len(s.steps)))
    for i in bad[:5]:
        _print_context(s.steps, order, i, got)
    fams = sorted({x.family for x in s.steps})
    for f in fams:
        n = [x for x in s.steps if x.family == f]
        print(f"a. {f:9s} steps {len(n):4d}  mismatches {sum(1 for x in n if x.i in bad)}")
    print(f"a. script order: {len(s.steps)} steps, mismatches {len(bad)}, wall {wall:.1f} s")
    assert not bad, f"{len(bad)} answers differ from the oracles, first at step {bad[0]}"


# ---------------------------------------------------------------------------------------------------------- b
def test_b_shuffled_order_in_a_child(sequential, tmp_path):
    s = session()
    got_a, _ = sequential
    order = sn.shuffled_order(s.steps, SHUFFLE_SEED)
    assert order != list(range(len(s.steps)))
    t = time.time()
    got_b = _child("run", tmp_path, dict(steps=s.steps, init=s.init_state, order=order))
    differ = [i for i in range(len(s.steps)) if got_b[i] != got_a[i]]
    for i in differ[:5]:
        _print_context(s.steps, order, i, got_b)
        need = sn.closure(s.steps, i)
        alone = _child("run", tmp_path, dict(steps=s.steps, init=s.init_state, order=need))[i]
        wrong = [name for name, g in (("script order", got_a[i]), ("shuffled order", got_b[i])) if g != alone]
        print(f"   step {i} replayed alone (with the {len(need) - 1} steps it depends on): {alone!r}"[:300])
        print(f"   oracle {'agrees' if alone == s.steps[i].want else 'disagrees'} with the replay; wrong run(s): {wrong}")
    moved = sum(1 for p, j in enumerate(order) if p != j)
    print(f"b. shuffled order (seed {SHUFFLE_SEED:#x}): {len(s.steps)} steps, {moved} moved, mismatches {len(differ)}, "
          f"wall {time.time() - t:.1f} s")
    assert not differ, f"{len(differ)} answers depend on the order, first at step {differ[0]}"
    assert not mismatches(s.steps, got_b)


# ---------------------------------------------------------------------------------------------------------- d
def worker_plan(steps):
    """Per worker: every state step (on its own handle) and a quarter of the one-shot, shuffle, batch and registry-read
    steps; never a step that changes the registry, the knobs or the VM schedule."""
    shared = [x for x in steps if x.family in ("strict", "rlc", "single", "ssz", "shuffle", "eval")
              and not x.writes and (x.reads <= {"registry"})]
    state = [x for x in steps if x.family == "state"]
    return [state + shared[w::WORKERS] for w in range(WORKERS)]


def test_d_worker_threads(sequential):
    from ethereum_consensus_b200 import _lib
    s = session()
    got_a, _ = sequential
    plans = worker_plan(s.steps)
    reg = crypto_registry()
    results, errors = [None] * WORKERS, [None] * WORKERS
    start = threading.Barrier(WORKERS)

    def work(w):
        ctx = Context(s.init_state)
        ctx.reg = reg
        got = {}
        try:
            start.wait()
            for step in plans[w]:
                got[step.i] = execute(step, ctx)
        except BaseException as e:  # noqa: BLE001 - reported below
            errors[w] = e
        finally:
            ctx.close()
            results[w] = got

    t = time.time()
    launches = _lib.lib().b200_launch_count()
    threads = [threading.Thread(target=work, args=(w,), name=f"session-worker-{w}") for w in range(WORKERS)]
    for th in threads:
        th.start()
    for th in threads:
        th.join(timeout=CHILD_TIMEOUT)
    assert not any(th.is_alive() for th in threads), "a worker thread did not finish"
    assert not any(errors), errors
    total = 0
    for w, got in enumerate(results):
        differ = [i for i in got if got[i] != got_a[i]]
        total += len(differ)
        order = [x.i for x in plans[w]]
        for i in differ[:3]:
            _print_context({x.i: x for x in s.steps}, order, i, got)
        print(f"d. worker {w}: {len(got)} steps, mismatches {len(differ)}")
    print(f"d. {WORKERS} worker threads: wall {time.time() - t:.1f} s, {_lib.lib().b200_launch_count() - launches} launches")
    assert total == 0


def crypto_registry():
    """The registry as section a left it (its last step: key_codes), for the workers to read."""
    from ethereum_consensus_b200 import crypto
    s = session()
    reg = crypto.Registry.__new__(crypto.Registry)
    reg.n = s.meta["final_n"]
    assert reg.key_codes().shape == (reg.n,)
    return reg


# ---------------------------------------------------------------------------------------------------------- child
def _main(mode, path, out):
    from ethereum_consensus_b200 import _lib
    _lib.init(0)
    data = pickle.loads(Path(path).read_bytes())
    assert mode == "run"
    t = time.time()
    got = run_steps(data["steps"], data["init"], order=data["order"])
    Path(out).write_bytes(pickle.dumps(got))
    print(f"child: {len(got)} steps in {time.time() - t:.1f} s")


if __name__ == "__main__":
    _main(*sys.argv[1:4])
