"""Generates tests/golden/lrc_kat.json from the numpy LRC model (tests/lrc_oracle.py).

Frozen: the parity rows of LRC(6,2,2), LRC(10,2,2) and LRC(12,2,2), the parity of one tiny stripe per code
(data = the first k*16 bytes of the splitmix64 stream with seed 0x6761726167650010, shard_len 16), and the number
of recoverable erasure patterns (rank test, want = every absent shard) per erasure count 0..m.

    python tests/golden/make_lrc_kat.py
"""
import itertools
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import lrc_oracle as LO  # noqa: E402
import rs_oracle_np as NP  # noqa: E402

SEED = 0x6761726167650010
CODES = [(6, 2, 2), (10, 2, 2), (12, 2, 2)]


def case(k, l, r):
    m = l + r
    P = LO.build_lrc(k, l, r)
    data = NP.fill_random(k * 16, SEED).reshape(k, 16)
    par = LO.encode(P, data)
    counts = {}
    for e in range(m + 1):
        ok = 0
        for er in itertools.combinations(range(k + m), e):
            pr = [0 if i in er else 1 for i in range(k + m)]
            ok += LO.recoverable(k, P, pr)
        counts[str(e)] = ok
    return {"k": k, "l": l, "r": r, "matrix_hex": [bytes(row).hex() for row in P],
            "kat_parity_hex": [bytes(row).hex() for row in par], "recoverable_by_erasures": counts}


if __name__ == "__main__":
    out = {"seed": SEED, "shard_len": 16, "cases": {"lrc_%d_%d_%d" % c: case(*c) for c in CODES}}
    with open(os.path.join(HERE, "lrc_kat.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
