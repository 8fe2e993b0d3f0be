"""Repair by segment through the block manager (DESIGN.md section 5.15): bytes and wall time of a resync that repairs
bit rot, for RS(10,4), LRC(10,2,2), PB(10,4) and, as the unchanged control, Clay(10,4).

Per code: --blocks 1 MiB blocks on a file store under /dev/shm.  One node (node 0, which holds one index of every
block) has one byte flipped in adler8 segment b mod 8 of block b's shard; a scrub of that node quarantines them and
resync_all (8 workers) repairs them.  Control rounds in the same run flip a byte in all eight segments of the same
shards, which forces the whole-shard rebuild.  The two kinds of round alternate, --rounds of each.  Per round: the bytes
resync fetched and read per block (resync_bytes_fetched / resync_bytes_read), garage_bm_segment_repair_metrics, and the
resync wall time.  The byte total of every one-segment round is checked against garage_ec_segment_read_ranges for each
block's lost unit, and split by the role of the repaired index.  The card's name and power limit are read in the same
run and written beside every row.  One JSON line per row (stdout, and --out)."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import garage_b200 as G  # noqa: E402
from garage_b200 import block_manager as BM  # noqa: E402

K, M = 10, 4
CODES = {
    "rs_10_4": ({}, lambda: G.GarageEc(0, K, M)),
    "lrc_10_2_2": ({"local_groups": 2}, lambda: G.GarageEc.lrc(0, K, 2, M - 2)),
    "pb_10_4": ({"piggyback": True}, lambda: G.GarageEc.piggyback(0, K, M)),
    "clay_10_4": ({"clay": True}, None),
}


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    name, plim = (x.strip() for x in out[0].split(","))
    return name, plim


def role(code, i):
    if i < K:
        return "data"
    if code == "lrc_10_2_2" and i < K + 2:
        return "local_parity"
    return "parity"


def planned(ec, code, idx, g, L):
    """garage_ec_segment_read_ranges' bytes for index idx missing the unit of segment g"""
    sp = np.full(K + M, 0xFF, np.uint8)
    sp[idx] &= ~np.uint8((1 << g) | ((1 << (g ^ 4)) if code == "pb_10_4" else 0))
    return sum(n for _, _, n in ec.segment_read_ranges(sp, L, want=np.eye(K + M, dtype=np.uint8)[idx]))


def run_code(code, nblocks, rounds, workers, name, plim, rows):
    kw, make_ec = CODES[code]
    d = tempfile.mkdtemp(prefix="segment_repair_bench_", dir="/dev/shm")
    try:
        with BM.BlockManager(K, M, data_dir=d, **kw) as bm:
            rng = np.random.default_rng(7)
            hs = []
            for _ in range(nblocks):
                blk = rng.integers(0, 256, 1 << 20, dtype=np.uint8)
                h = BM.blake2sum(blk)
                assert bm.rpc_put_block(h, blk) == BM.OK
                hs.append(h)
            node = 0
            L = bm.block_info(hs[0])[1]["block_len"]
            L = -(-L // K)
            if kw.get("piggyback"):
                L = -(-L // 128) * 128
            if kw.get("clay"):
                with G.GarageEc.clay(0, K, M) as ec:
                    L = ec.code_shard_len(1 << 20)
            S = (-(-L // 8) + 15) // 16 * 16
            idx = [bm.storage_nodes_of(h).index(node) for h in hs]
            expect, by_role = 0, {}
            if make_ec:
                with make_ec() as ec:
                    for b, i in enumerate(idx):
                        n = planned(ec, code, i, b % 8, L)
                        expect += n
                        by_role.setdefault(role(code, i), []).append(n)
            for r in range(2 * rounds):
                case = "one_segment" if r % 2 == 0 else "all_segments"
                for b, h in enumerate(hs):
                    for g in ([b % 8] if case == "one_segment" else range(8)):
                        assert bm.corrupt_shard(node, h, g * S + 3 + r) == BM.OK
                rc, _, corrupt = bm.scrub(node)
                assert rc == BM.OK and corrupt == nblocks
                m0, s0 = bm.metrics(), bm.segment_repair_metrics()
                t0 = time.perf_counter()
                failed, done = bm.resync_all(node, workers=workers)
                wall = time.perf_counter() - t0
                assert (failed, done) == (0, nblocks)
                m1, s1 = bm.metrics(), bm.segment_repair_metrics()
                seg = {k: s1[k] - s0[k] for k in s1}
                fetched = m1["resync_bytes_fetched"] - m0["resync_bytes_fetched"]
                if case == "one_segment" and make_ec:
                    assert seg["repairs"] == nblocks and seg["bytes_fetched"] == expect == fetched, (seg, expect)
                else:
                    assert seg["repairs"] == 0
                row = dict(tool="segment_repair_bench", code=code, case=case, round=r // 2, blocks=nblocks,
                           block_len=1 << 20, shard_len=L, store="/dev/shm", workers=workers,
                           resync_bytes_fetched_per_block=round(fetched / nblocks, 1),
                           resync_bytes_read_per_block=round((m1["resync_bytes_read"] - m0["resync_bytes_read"]) / nblocks, 1),
                           segment_repair={k: v for k, v in seg.items()},
                           resync_ms_per_block=round(1e3 * wall / nblocks, 4), gpu=name, power_limit=plim)
                if case == "one_segment" and make_ec:
                    row["planned_bytes_fetched_by_role"] = {k: round(float(np.mean(v)), 1) for k, v in sorted(by_role.items())}
                rows.append(row)
                print(json.dumps(row), flush=True)
            for h in hs[:: max(1, nblocks // 16)]:
                rc, info = bm.block_info(h, check_tags=True)
                assert rc == BM.OK and info["state"] == [BM.SHARD_VALID] * (K + M)
    finally:
        shutil.rmtree(d, ignore_errors=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--workers", type=int, default=8)
    ap.add_argument("--codes", default=",".join(CODES))
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, plim = card()
    rows = []
    for code in a.codes.split(","):
        run_code(code, a.blocks, a.rounds, a.workers, name, plim, rows)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            for row in rows:
                f.write(json.dumps(row) + "\n")


if __name__ == "__main__":
    main()
