"""One rank of the sharded-call tests: tests/test_sharded_loopback_gpu.py (every rank a process on the same GPU, the
loopback communicator of b200_comm_init_loopback) and the two-GPU tests of test_config_scale_gpu.py and
test_rlc_soak_gpu.py (one GPU per rank, NCCL; rank 0 hands the 128-byte NCCL id over through a file).  No torch.

Reads B200_TEST_DIR/cases.pkl (tests/sharded_cases.write_cases), runs every section in the same order on every rank and
writes B200_TEST_DIR/rank<r>.pkl: one (section, name, value, return code, collectives issued) record per call.
B200_TEST_TRANSPORT: loopback (default) | nccl.  B200_TEST_SECTIONS: a comma list (default all)."""
import ctypes as C
import os
import pickle
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from ethereum_consensus_b200 import _lib, crypto, parallel, ssz  # noqa: E402
from tests import sharded_cases as sh  # noqa: E402

rank, world = int(os.environ["B200_TEST_RANK"]), int(os.environ["B200_TEST_WORLD"])
box = Path(os.environ["B200_TEST_DIR"])
transport = os.environ.get("B200_TEST_TRANSPORT", "loopback")
sections = os.environ.get("B200_TEST_SECTIONS", "states,strict,rlc,gather,refusals").split(",")
data = pickle.loads((box / "cases.pkl").read_bytes())
assert data["world"] == world
lib = _lib.init(int(os.environ.get("B200_TEST_DEVICE", "0")))
LOOP = box / "loopback.bin"


def connect():
    if transport == "loopback":
        _lib.check(lib.b200_comm_init_loopback(str(LOOP).encode(), rank, world, sh.SLOT_BYTES, sh.TIMEOUT_MS), "comm_init_loopback")
        return
    ident = (C.c_uint8 * 128)()
    id_file = box / "nccl_id.bin"
    if rank == 0:
        _lib.check(lib.b200_comm_unique_id(ident), "comm_unique_id")
        tmp = box / "nccl_id.tmp"
        tmp.write_bytes(bytes(ident))
        tmp.rename(id_file)
    else:
        t0 = time.time()
        while not id_file.exists():
            if time.time() - t0 > 120:
                raise SystemExit("timed out waiting for the NCCL id")
            time.sleep(0.05)
        C.memmove(ident, id_file.read_bytes(), 128)
    _lib.check(lib.b200_comm_init(ident, rank, world), "comm_init")


connect()
assert parallel.comm_info()[:2] == (rank, world)
BASE = lib.b200_collective_count()
records = []


def call(section, name, fn):
    c0 = lib.b200_collective_count()
    try:
        value, rc = fn(), 0
    except Exception as e:   # noqa: BLE001 - an engine error is a result; anything else is recorded as -1
        value, rc = None, getattr(e, "code", -1)
        if rc == -1:
            value = repr(e)
    records.append((section, name, value, rc, int(lib.b200_collective_count() - c0)))
    return value


def own_slot():
    """This rank's slot of the last loopback generation (csrc/comm_loopback.h layout)."""
    g = lib.b200_collective_count() - BASE - 1
    raw = LOOP.read_bytes()
    at = sh.HEADER_BYTES + ((g & 1) * world + rank) * sh.SLOT_BYTES
    return raw[at: at + sh.RLC_PART]


# ---- states: the one-call root, and the resident handle (root twice, another family's single-GPU call in between)
if "states" in sections:
    single = data["strict"][0]
    for st in data["states"]:
        ser = np.load(st["path"])
        call("states", st["name"], lambda: parallel.sharded_state_root(ser, st["preset"]))
        if st["resident"]:
            box_h = []
            call("states", st["name"] + ": resident upload", lambda: box_h.append(ssz.DeviceBeaconState(ser, st["preset"], sharded=True)))
            dev = box_h[0] if box_h else None
            call("states", st["name"] + ": resident root", lambda: dev.hash_tree_root())
            call("states", st["name"] + ": single-GPU verify between", lambda: crypto.fast_aggregate_verify_batch(*single["args"]).tolist())
            call("states", st["name"] + ": resident root again", lambda: dev.hash_tree_root())
            if dev is not None:
                dev.close()

# ---- strict verify
if "strict" in sections:
    for c in data["strict"]:
        call("strict", c["name"], lambda: parallel.sharded_verify_batch(*c["args"]).tolist())

# ---- RLC, under the crafting seed and four others; the exchanged slot of two identical calls
if "rlc" in sections:
    for c in data["rlc"]:
        for i, (seed, _want) in enumerate(c["runs"]):
            call("rlc", f"{c['name']} [seed {i}]", lambda: crypto.fast_aggregate_verify_batch_all(*c["args"], seed=seed, sharded=True))
    if transport == "loopback":
        c = next(c for c in data["rlc"] if "sum to infinity" in c["name"])
        slots = []
        for _ in range(2):
            if call("slot", c["name"], lambda: crypto.fast_aggregate_verify_batch_all(*c["args"], seed=c["runs"][0][0], sharded=True)) is not None:
                slots.append(own_slot())
        records.append(("slot", "rlc slot twice", slots, 0, 0))

# ---- host all-gathers
if "gather" in sections:
    call("gather", "comm_all_gather_codes", lambda: parallel.comm_all_gather_codes(sh.gather_codes(rank)).tolist())
    for n in data["gather"]:
        send = np.frombuffer(sh.gather_payload(rank, n), dtype=np.uint8)
        recv = np.zeros(max(1, n * world), dtype=np.uint8)

        def gather():
            _lib.check(lib.b200_comm_all_gather_bytes(_lib.ptr(send) if n else None, n, _lib.ptr(recv)), "comm_all_gather_bytes")
            return recv[: n * world].tobytes()
        call("gather", f"all_gather_bytes {n}", gather)

# ---- refusals: the same code on every rank, no exchange
if "refusals" in sections:
    pks, off, msgs, sigs = data["rlc"][0]["args"]
    T = len(off) - 1
    down = off.copy()
    down[1] = down[-1] + 1
    seed = np.frombuffer(bytes(32), dtype=np.uint8)
    codes = np.zeros(T + 1, dtype=np.int32)
    ok = C.c_int32(0)
    out = (C.c_uint8 * 32)()
    P = _lib.ptr
    strict = lib.b200_fast_aggregate_verify_batch_sharded
    rlc = lib.b200_fast_aggregate_verify_batch_all_sharded
    got = {
        "strict: decreasing offsets": lambda: strict(P(pks), P(down), P(msgs), P(sigs), T, P(codes)),
        "strict: n_tuples > 2^26": lambda: strict(P(pks), P(off), P(msgs), P(sigs), sh.MAX_TUPLES + 1, P(codes)),
        "rlc: decreasing offsets": lambda: rlc(P(pks), P(down), P(msgs), P(sigs), T, P(seed), C.byref(ok)),
        "rlc: n_tuples > 2^26": lambda: rlc(P(pks), P(off), P(msgs), P(sigs), sh.MAX_TUPLES + 1, P(seed), C.byref(ok)),
        "rlc: NULL seed": lambda: rlc(P(pks), P(off), P(msgs), P(sigs), T, None, C.byref(ok)),
        "rlc: T < world": lambda: rlc(P(pks), P(off), P(msgs), P(sigs), world - 1, P(seed), C.byref(ok)),
    }
    bad_preset, bad = data["malformed"]
    good_preset, good = data["small_state"]
    h = C.c_void_p()
    got["htr sharded: malformed state"] = lambda: lib.b200_htr_beacon_state_deneb_sharded(P(bad), len(bad), _lib.PRESET[bad_preset], out)
    got["upload sharded: malformed state"] = lambda: lib.b200_state_upload_deneb_sharded(P(bad), len(bad), _lib.PRESET[bad_preset], C.byref(h))
    got[f"htr sharded: world {world}"] = lambda: lib.b200_htr_beacon_state_deneb_sharded(P(good), len(good), _lib.PRESET[good_preset], out)
    got[f"upload sharded: world {world}"] = lambda: lib.b200_state_upload_deneb_sharded(P(good), len(good), _lib.PRESET[good_preset], C.byref(h))
    idx = np.zeros(1, dtype=np.uint64)
    val = np.zeros(8, dtype=np.uint8)
    got["update_bytes on a sharded handle"] = lambda: lib.b200_state_update_bytes(h, 0, P(val), 1)
    got["update_elements on a sharded handle"] = lambda: lib.b200_state_update_elements(h, 1, P(idx), P(val), 1)
    got["registry_load_state on a sharded handle"] = lambda: lib.b200_registry_load_state(h)

    def root_after_world1():
        lib.b200_comm_destroy()
        parallel.comm_init(0, 1)
        return lib.b200_state_root(h, out)
    got["state_root on a sharded handle after the communicator became world 1"] = root_after_world1
    for name, _want in data["refusals"]:
        if name == "update_bytes on a sharded handle":
            call("refusals", "upload sharded: the handle the next refusals take",
                 lambda: lib.b200_state_upload_deneb_sharded(P(good), len(good), _lib.PRESET[good_preset], C.byref(h)) or None)
        c0 = lib.b200_collective_count()
        rc = got[name]()
        records.append(("refusals", name, None, int(rc), int(lib.b200_collective_count() - c0)))
    if h:
        lib.b200_state_free(h)

parallel.comm_destroy()
(box / f"rank{rank}.pkl").write_bytes(pickle.dumps(records))
print("WORKER_OK rank", rank, "records", len(records), flush=True)
