"""What the beacon-committee calls cost on the GPU at 2^20 validators, mainnet: one JSON line (DESIGN.md §8).

  committees_cold       b200_state_beacon_committees on an epoch the handle has not cached (each run first rewrites
                        one Validator record with its own bytes, which makes the cache stale): active-set scan, whole-list
                        shuffle and the 8 MB list to the host
  committees_cached     the same epoch again, from the cache: the list to the host only
  attester_duties_all   AttestationDuty rows of all 2^20 validators of a cached epoch (inverse map built)
  attesting_128x512     attesting_indices of 128 attestations of 512-member committees (~90 % of bits set)
  attesting_2048x512    the same for all 2048 committees of the epoch
  block_128_verdicts    a block's 128 attestations from Bitlists to verdicts: attesting_indices, then one registry-mode
                        SignatureSet.verify (device time: the two calls' kernels; wall: includes the Python between them)
Outputs are checked before anything is timed.  Each row: median and min-max over --runs timed calls after --warmup
untimed ones, as wall time around the call and as b200_last_kernel_ms.  The card's name and power limit are read with
nvidia-smi in the same run.

    python tools/probe_committees.py [--runs 9] [--warmup 3]
"""
from __future__ import annotations

import argparse
import ctypes as C
import hashlib
import json
import subprocess
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from ethereum_consensus_b200 import _lib, block, crypto, duties, shuffling, ssz  # noqa: E402
from ethereum_consensus_b200 import state as S  # noqa: E402
from oracle import duties_oracle as do  # noqa: E402
from tests import committee_cases as cc  # noqa: E402
from tests import committee_oracle as co  # noqa: E402
from tools.probe_duties import card, timed  # noqa: E402

R_ORDER = 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001
SK0, DELTA = 0x1234567, 0x89abcdef12345


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=9)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    n, nd = 1 << 20, 1 << 15
    lib = _lib.init()
    info = card()
    subprocess.run(["make", "-s", "-C", str(ROOT / "oracle")], check=True, capture_output=True)
    orc = C.CDLL(str(ROOT / "oracle" / "liboracle_bls.so"))
    orc.orc_pk_sequence.argtypes = [C.c_char_p, C.c_char_p, C.c_size_t, C.c_void_p]
    orc.orc_sign.argtypes = [C.c_char_p, C.c_char_p, C.c_size_t, C.c_char_p]
    keys = np.empty((nd, 48), dtype=np.uint8)
    orc.orc_pk_sequence(SK0.to_bytes(32, "big"), DELTA.to_bytes(32, "big"), nd, keys.ctypes.data)
    st = cc.state(n, "mainnet", seed=71, edges=False)   # 2^20 active: 64 committees per slot of exactly 512
    st.validators["public_key"] = keys[np.arange(n) % nd].view("V48").reshape(n)
    dev = ssz.DeviceBeaconState(S.serialize(st))
    E = cc.EPOCH
    res = {"n_validators": n, "preset": "mainnet", "runs": a.runs, "warmup": a.warmup}

    # checks: the committees are slices of the shuffled active list, duties their inverse
    seed = duties.get_seed(dev, E - 1, duties.DOMAIN_BEACON_ATTESTER)
    shuffled = shuffling.state_shuffled_active_indices(dev, E - 1, seed)
    idx, off, cps = duties.beacon_committees(dev, E - 1)
    assert cps == 64 and np.array_equal(idx, shuffled) and off.tolist() == [512 * k for k in range(2049)]
    rows = duties.attester_duties(dev, E - 1).view(np.uint64).reshape(-1, 5)
    pos = np.empty(n, np.int64)
    pos[shuffled.astype(np.int64)] = np.arange(n)
    assert np.array_equal(rows[:, 4], pos % 512) and np.array_equal(rows[:, 0], (E - 1) * 32 + pos // 512 // 64)

    vo = S.layout(st)["validators"][0]
    rec0 = np.frombuffer(dev.read_bytes(vo, 121), np.uint8)

    def cold():
        dev.update_elements("validators", [0], rec0)   # same bytes: the records' generation moves on
        duties.beacon_committees(dev, E)
        return lib.b200_last_kernel_ms()
    res["committees_cold"] = timed(cold, a.runs, a.warmup)
    res["committees_cached"] = timed(lambda: [duties.beacon_committees(dev, E), None][1], a.runs, a.warmup)
    res["attester_duties_all"] = timed(lambda: [duties.attester_duties(dev, E), None][1], a.runs, a.warmup)

    # attestations of epoch E - 1 (every slot of it is timely at the state's slot)
    rng = np.random.default_rng(71)
    atts, members = [], []
    for k in range(2048):
        s = (E - 1) * 32 + k // 64
        bits = rng.random(512) < 0.9
        atts.append((co.attestation_data(s, k % 64, E - 1, root=hashlib.sha256(b"r%d" % k).digest()), co.bitlist(bits.tolist())))
        members.append(np.sort(idx[off[k]:off[k + 1]][bits]))
    pick = rng.choice(2048, 128, replace=False)
    block_atts = [atts[k] for k in pick]
    got, codes = duties.attesting_indices(dev, atts)
    assert (codes == 0).all() and all(np.array_equal(g, m) for g, m in zip(got, members))
    res["attesting_128x512"] = timed(lambda: [duties.attesting_indices(dev, block_atts), None][1], a.runs, a.warmup)
    res["attesting_2048x512"] = timed(lambda: [duties.attesting_indices(dev, atts), None][1], a.runs, a.warmup)

    # a block: 128 signed attestations, Bitlists to verdicts in registry mode
    msgs, sigs = [], []
    for k in pick:
        msg = hashlib.sha256(atts[k][0]).digest()
        sk = sum(SK0 + DELTA * (int(i) % nd) for i in members[k]) % R_ORDER
        sig = C.create_string_buffer(96)
        orc.orc_sign(sk.to_bytes(32, "big"), msg, 32, sig)
        msgs.append(msg)
        sigs.append(sig.raw)
    reg = crypto.Registry.from_state(dev)

    class Keys:
        def __len__(self):
            return n

        def __getitem__(self, i):
            return keys[int(i) % nd].tobytes()
    pk = Keys()

    def verdicts():
        got, codes = duties.attesting_indices(dev, block_atts)
        ms = lib.b200_last_kernel_ms()
        ss = block.SignatureSet()
        for g, m, s in zip(got, msgs, sigs):
            ss.add_indexed_attestation("attestation", pk, g.tolist(), m, s)
        v = ss.verify(registry=reg)
        assert v.tolist() == [0] * 128 and codes.tolist() == [0] * 128
        return ms + lib.b200_last_kernel_ms()
    res["block_128_verdicts"] = timed(verdicts, a.runs, a.warmup)
    print(json.dumps({**info, **res}))


if __name__ == "__main__":
    main()
