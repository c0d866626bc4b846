"""GPU: what the BLS host pipeline (csrc/capi_bls.cu) does for each call shape: the verdicts, and exactly how many kernels
it launches (b200_launch_count).  Which phases run, on how many key ranges and in which order is decided on the host,
so a launch count that moves means a path changed; the codes say it still computes the same thing.

Launch names: K1 per-key validation, K3 signature decode, K4 hash_to_G2 (two kernels: map, finish), K2 per-tuple
aggregate, K5 Miller loops and K6 final exponentiations on the pairing VM."""
import json

import numpy as np
import pytest

from ethereum_consensus_b200 import _lib, crypto, parallel
from tests.test_bls_gpu import FAV, GOLDEN, _batch_inputs, _call

pytestmark = pytest.mark.gpu

# batch of fast-aggregate tuples with keys: K1 + K3 + K4 (2) + K2 + K5 + K6
STRICT = 1 + 1 + 2 + 1 + 1 + 1
# registry batch: no K1 (the keys are resident and validated), K3 + K4 (2) + K2 + K5 + K6
REGISTRY = 1 + 2 + 1 + 1 + 1
# big strict batch (>= 4 x 227 328 keys): K1 on the first 227 328 keys, a second K1 on the rest behind their copy
SPLIT = STRICT + 1
# RLC tail: K_scale, the signature folds (ceil(n / 32) per level), K_finish, K5 on T + 1 pairs, the Gt folds, K_one, K6
def rlc(t):
    def folds(n):
        k = 0
        while True:
            n, k = (n + 31) // 32, k + 1
            if n <= 1:
                return k
    return 1 + folds(t) + 1 + 1 + folds(t + 1) + 1 + 1
# aggregate_verify, a batch of one tuple with 4 messages: K1 + K3 + K4 (2) + K2 + pair operands + K5 + one fold level
# (5 Miller values, one piece) + K6
AGG_VERIFY = 1 + 1 + 2 + 1 + 1 + 1 + 1 + 1
# aggregate_verify with len(pks) != len(msgs): no messages to hash, no pairs, no fold: K1 + K3 + K2 + pair operands + K6
AGG_VERIFY_MISMATCH = 1 + 1 + 1 + 1 + 1
# aggregate_verify with no keys and no messages: K3 + K2 + K6
AGG_VERIFY_EMPTY = 1 + 1 + 1
AGGREGATE = 2          # signature decode + sum / compress
AGG_PUBKEYS = 3        # K1 + aggregate + compress

CASES = [c for c in FAV if len(c["msg"]) == 64]
VALID = [c for c in CASES if c["code"] == 0]
BIG_T, BIG_K = 1776, 512
KNOB_DEFAULTS = {"bls_small_cta": 0, "vm_team16_max": 2048, "vm_cta": 32}
# knobs earlier versions took; b200_tune refuses them like any unknown name
RETIRED_KNOBS = ("bls_chunks", "bls_chunk_min_tuples", "bls_chunk_k1_cta", "bls_chunk_alt", "bls_key_split", "bls_k1_first_cta")


def _launches() -> int:
    return int(_lib.lib().b200_launch_count())


def _counted(fn, *a):
    n0 = _launches()
    r = fn(*a)
    return r, _launches() - n0


def _counted_code(fn, *a):
    n0 = _launches()
    code = _call(fn, *a)
    return code, _launches() - n0


def _big_batch():
    """T = 1 776 tuples x K = 512 keys from the golden keys, messages and signatures, tiled."""
    pks, _, msgs, sigs, _ = _batch_inputs(FAV)
    off = (np.arange(BIG_T + 1, dtype=np.uint64) * BIG_K).astype(np.uint32)
    return np.resize(pks, BIG_T * BIG_K * 48), off, np.resize(msgs, 32 * BIG_T), np.resize(sigs, 96 * BIG_T)


def _registry_inputs(cases, keys):
    pos = {p: i for i, p in enumerate(keys)}
    idx = np.array([pos[p] for c in cases for p in c["pks"]], dtype=np.uint32)
    off = np.cumsum([0] + [len(c["pks"]) for c in cases]).astype(np.uint32)
    msgs = np.frombuffer(b"".join(bytes.fromhex(c["msg"]) for c in cases), dtype=np.uint8)
    sigs = np.frombuffer(b"".join(bytes.fromhex(c["sig"]) for c in cases), dtype=np.uint8)
    return idx, off, msgs, sigs


def _flat(keys):
    return np.frombuffer(b"".join(bytes.fromhex(p) for p in keys), dtype=np.uint8)


def _case(section, name):
    return next(c for c in GOLDEN[section] if c["name"] == name)


def shared_shapes() -> dict:
    """One call of each shape: name -> (codes, launches)."""
    crypto.fast_aggregate_verify_batch(*_batch_inputs(FAV)[:4])   # first use builds the pipeline's state (2 launches)
    res = {}
    codes, n = _counted(crypto.fast_aggregate_verify_batch, *_batch_inputs(FAV)[:4])
    res["strict"] = (codes.tolist(), n)
    codes, n = _counted(crypto.fast_aggregate_verify_batch, *_big_batch())
    res["big"] = (codes.tolist(), n)
    uniq = sorted({p for c in CASES for p in c["pks"]})
    reg, n = _counted(crypto.Registry, _flat(uniq))
    res["registry_load"] = (reg.key_codes().tolist(), n)
    codes, n = _counted(reg.verify_batch, *_registry_inputs(CASES, uniq))
    res["registry"] = (codes.tolist(), n)
    in_reg, extra = uniq[::2], uniq[1::2]
    reg = crypto.Registry(_flat(in_reg))
    codes, n = _counted(lambda: reg.verify_batch(*_registry_inputs(CASES, in_reg + extra), extra_keys=_flat(extra)))
    res["mixed"] = (codes.tolist(), n)
    one = next(c for c in FAV if c["name"] == "valid K=1")
    k3 = next(c for c in FAV if c["name"] == "valid K=3")
    none = next(c for c in FAV if c["name"] == "no keys")
    h = bytes.fromhex
    res["verify_signature"] = _counted_code(crypto.verify_signature, h(one["pks"][0]), h(one["msg"]), h(one["sig"]))
    res["fast_aggregate_verify"] = _counted_code(crypto.fast_aggregate_verify, [h(p) for p in k3["pks"]], h(k3["msg"]), h(k3["sig"]))
    res["fast_aggregate_verify_no_keys"] = _counted_code(crypto.fast_aggregate_verify, [], h(none["msg"]), h(none["sig"]))
    c = _case("aggregate", "4 sigs")
    out, n = _counted(crypto.aggregate, [h(s) for s in c["sigs"]])
    res["aggregate"] = (bytes(out).hex(), n)
    c = _case("eth_aggregate_public_keys", "8 keys")
    out, n = _counted(crypto.eth_aggregate_public_keys, [h(p) for p in c["pks"]])
    res["eth_aggregate_public_keys"] = (bytes(out).hex(), n)
    return res


def check_shared(res: dict):
    want = [c["code"] for c in CASES]
    assert res["strict"] == [want, STRICT]
    assert res["big"][1] == SPLIT
    assert res["registry_load"][1] == 1
    assert res["registry"] == [want, REGISTRY]
    assert res["mixed"] == [want, STRICT]
    assert res["verify_signature"] == [0, STRICT]
    assert res["fast_aggregate_verify"] == [0, STRICT]
    assert res["fast_aggregate_verify_no_keys"] == [5, STRICT - 1]          # no keys: no K1
    assert res["aggregate"] == [_case("aggregate", "4 sigs")["out"], AGGREGATE]
    assert res["eth_aggregate_public_keys"] == [_case("eth_aggregate_public_keys", "8 keys")["out"], AGG_PUBKEYS]


@pytest.fixture
def knobs(engine):
    """Every knob at its default around the test."""
    for k, v in KNOB_DEFAULTS.items():
        crypto.tune(k, v)
    yield
    for k, v in KNOB_DEFAULTS.items():
        crypto.tune(k, v)


@pytest.fixture(scope="module")
def default_shapes(engine):
    for k, v in KNOB_DEFAULTS.items():
        crypto.tune(k, v)
    return json.loads(json.dumps(shared_shapes()))


def test_shared_shapes_default_process(default_shapes):
    check_shared(default_shapes)


def test_aggregate_verify_single_call_is_batch_of_one(knobs):
    """The single aggregate_verify call runs as an aggregate_verify batch of one tuple: its codes and launches per shape,
    and on a valid tuple the same code and launch count as aggregate_verify_batch."""
    crypto.fast_aggregate_verify_batch(*_batch_inputs(FAV)[:4])   # first use builds the pipeline's state (2 launches)
    h = bytes.fromhex
    for name, want in (("4 distinct messages", (0, AGG_VERIFY)), ("length mismatch", (5, AGG_VERIFY_MISMATCH)),
                       ("empty", (5, AGG_VERIFY_EMPTY))):
        c = _case("aggregate_verify", name)
        assert _counted_code(crypto.aggregate_verify, [h(p) for p in c["pks"]], [h(m) for m in c["msgs"]], h(c["sig"])) == want, name
    c = _case("aggregate_verify", "4 distinct messages")
    codes, n = _counted(crypto.aggregate_verify_batch, _flat(c["pks"]), [0, len(c["pks"])], [h(m) for m in c["msgs"]],
                        [0, len(c["msgs"])], np.frombuffer(h(c["sig"]), dtype=np.uint8))
    assert (codes.tolist(), n) == ([0], AGG_VERIFY)


def test_whole_batch_calls(knobs):
    seed = bytes(range(32))
    golden = _batch_inputs(FAV)[:4]
    valid = _batch_inputs(VALID)[:4]
    assert _counted(crypto.fast_aggregate_verify_batch_all, *golden, seed) == (False, STRICT - 2 + rlc(len(CASES)))
    assert _counted(crypto.fast_aggregate_verify_batch_all, *valid, seed) == (True, STRICT - 2 + rlc(len(VALID)))
    assert _counted(crypto.fast_aggregate_verify_batch_all, *valid) == (True, STRICT - 2 + rlc(len(VALID)))
    uniq = sorted({p for c in CASES for p in c["pks"]})
    reg = crypto.Registry(_flat(uniq))
    assert _counted(reg.verify_batch_all, *_registry_inputs(CASES, uniq), seed) == (False, REGISTRY - 2 + rlc(len(CASES)))
    assert _counted(reg.verify_batch_all, *_registry_inputs(VALID, uniq), seed) == (True, REGISTRY - 2 + rlc(len(VALID)))


def test_sharded_calls_world1(knobs):
    parallel.comm_init(0, 1)
    want = [c["code"] for c in CASES]
    golden = _batch_inputs(FAV)[:4]
    codes, n = _counted(parallel.sharded_verify_batch, *golden)
    assert (codes.tolist(), n) == (want, STRICT)                 # the world-1 exchange is a device copy, no launch
    seed = bytes(range(32))
    assert _counted(lambda: crypto.fast_aggregate_verify_batch_all(*golden, seed=seed, sharded=True)) == (False, STRICT - 2 + rlc(len(CASES)))
    valid = _batch_inputs(VALID)[:4]
    assert _counted(lambda: crypto.fast_aggregate_verify_batch_all(*valid, seed=seed, sharded=True)) == (True, STRICT - 2 + rlc(len(VALID)))


def test_tune_accepts_every_documented_knob(engine):
    for k, v in KNOB_DEFAULTS.items():
        crypto.tune(k, v)
    for k in ("no_such_knob", *RETIRED_KNOBS):
        with pytest.raises(_lib.EngineError) as e:
            crypto.tune(k, 1)
        assert e.value.code == _lib.ERR_BAD_ARG, k
