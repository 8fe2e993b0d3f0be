"""Generates tests/golden/pb_kat.json from the numpy PB model (tests/pb_oracle.py).

Frozen: the group split and the parity bytes of one tiny stripe per code, PB(4,2), PB(6,3), PB(10,4) and PB(16,4)
with Vandermonde and Cauchy parity rows (data = the first k*64 bytes of the splitmix64 stream with seed
0x6761726167650020, shard_len 64: halves of 32 bytes).

    python tests/golden/make_pb_kat.py
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import pb_oracle as PB  # noqa: E402
import rs_oracle_np as NP  # noqa: E402

SEED = 0x6761726167650020
SHARD_LEN = 64
CODES = [(4, 2), (6, 3), (10, 4), (16, 4)]


def case(k, m, kind):
    P = PB.build(k, m, kind)
    data = NP.fill_random(k * SHARD_LEN, SEED).reshape(k, SHARD_LEN)
    par = PB.encode(P, data)
    return {"k": k, "m": m, "kind": kind, "groups": PB.groups(k, m), "matrix_hex": [bytes(r).hex() for r in P],
            "kat_parity_hex": [bytes(r).hex() for r in par]}


if __name__ == "__main__":
    out = {"seed": SEED, "shard_len": SHARD_LEN,
           "cases": {"pb_%d_%d_%s" % (k, m, "cauchy" if kind else "vand"): case(k, m, kind)
                     for k, m in CODES for kind in (0, 1)}}
    with open(os.path.join(HERE, "pb_kat.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
