"""One rank of tests/test_rlc_soak_gpu.py::test_crafted_batch_on_two_ranks (also runnable by hand on a machine with two
GPUs).  The batch is a family-A case of tests/rlc_soak_cases.py: every tuple invalid, defects cancelling only for the
scalars r_t of the global tuple index t under the crafting seed.  Each rank verifies its block and must hash t0 + t,
so both ranks accept it under that seed and reject it under another.  The NCCL id travels through a file, as in
tests/mp_sharded_worker.py."""
import ctypes as C
import os
import pickle
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from ethereum_consensus_b200 import _lib, crypto, parallel  # noqa: E402

rank, world = int(os.environ["B200_TEST_RANK"]), int(os.environ["B200_TEST_WORLD"])
box = Path(os.environ["B200_TEST_DIR"])
lib = _lib.init(int(os.environ.get("B200_TEST_DEVICE", "0")))
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
assert parallel.comm_info()[:2] == (rank, world)

case = pickle.loads((box / "case.pkl").read_bytes())
args = case["args"]
assert crypto.fast_aggregate_verify_batch_all(*args, seed=case["seed"], sharded=True) is True, rank
assert crypto.fast_aggregate_verify_batch_all(*args, seed=case["other"], sharded=True) is False, rank
assert crypto.fast_aggregate_verify_batch_all(*args, seed=case["seed"]) is True, rank      # the unsharded call agrees
parallel.comm_destroy()
print("RLC_SHARDED_OK", rank)
