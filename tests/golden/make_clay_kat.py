"""Regenerate tests/golden/clay_kat.json: Clay(k, m) encodings of one seeded stripe at L = 16 * alpha, frozen as the
base-code rows and the SHA-256 of the parity shards (the parity of Clay(10,4) alone is 16 KiB)."""
import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import clay_oracle as CO  # noqa: E402
import oracle_lib as O  # noqa: E402

SEED = 0x434C4159


def main():
    cases = {}
    for k, m in [(4, 2), (6, 3), (10, 4), (10, 3)]:
        for kind in (0, 1):
            alpha = CO.params(k, m)[4]
            L = 16 * alpha
            P = CO.build(k, m, kind)
            data = O.fill_random(k * L, SEED).reshape(k, L)
            par = CO.encode(k, m, P, data)
            cases["clay_%d_%d_%s" % (k, m, "cauchy" if kind else "vandermonde")] = {
                "k": k, "m": m, "kind": kind, "shard_len": L,
                "base_rows_hex": [bytes(r).hex() for r in P],
                "parity_sha256": hashlib.sha256(par.tobytes()).hexdigest(),
                "parity_head_hex": [bytes(r[:32]).hex() for r in par],
            }
    with open(os.path.join(HERE, "clay_kat.json"), "w") as f:
        json.dump({"seed": SEED, "cases": cases}, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
