#!/usr/bin/env python
"""Repair traffic of a node loss under the block manager: a 14-node file store on /dev/shm holding 256 x 1 MiB blocks
under RS(10,4), PB(10,4) and Clay(10,4) in turn; one node's directory is wiped, then repair_enqueue_missing +
resync_all rebuild it.  One JSON line per code: resync_bytes_fetched per block (what the rebuild is handed, which is
what would cross the network in Garage), resync_bytes_read per block (what the holders read from disk) and the wall
time of the resync.

    python tools/repair_bench.py [--blocks 256] [--node 5]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import oracle_lib as O  # noqa: E402

from garage_b200 import block_manager as BM  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--blocks", type=int, default=256)
ap.add_argument("--node", type=int, default=5)
args = ap.parse_args()


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True, timeout=30).stdout.strip()
    return out.splitlines()[0] if out else None


blocks = [O.fill_random(1 << 20, 0x5EB0 + i) for i in range(args.blocks)]
hashes = [BM.blake2sum(b) for b in blocks]
base = "/dev/shm" if os.path.isdir("/dev/shm") else None
for code, kw in (("RS(10,4)", {}), ("PB(10,4)", {"piggyback": True}), ("Clay(10,4)", {"clay": True})):
    d = tempfile.mkdtemp(prefix="repair_bench_", dir=base)
    try:
        with BM.BlockManager(k=10, m=4, n_nodes=14, data_dir=d, **kw) as bm:
            for h, b in zip(hashes, blocks):
                assert bm.rpc_put_block(h, b) == 0
            nd = os.path.join(d, "node%d" % args.node)
            held = sum(len(f) for _, _, f in os.walk(nd))
            shutil.rmtree(nd)
            os.makedirs(nd)
            m0 = bm.metrics()
            t0 = time.perf_counter()
            bm.repair_enqueue_missing(args.node)
            failed, done = bm.resync_all(args.node)
            wall = time.perf_counter() - t0
            m1 = bm.metrics()
            ok = failed == 0 and done == held
            for h, b in zip(hashes, blocks):
                rc, got = bm.rpc_get_block(h)
                ok = ok and rc == 0 and bytes(got) == bytes(b)
            fetched = m1["resync_bytes_fetched"] - m0["resync_bytes_fetched"]
            read = m1["resync_bytes_read"] - m0["resync_bytes_read"]
            print(json.dumps({"code": code, "blocks": args.blocks, "shards_rebuilt": done, "ok": bool(ok),
                              "fetched_bytes_per_block": round(fetched / max(done, 1)),
                              "read_bytes_per_block": round(read / max(done, 1)), "wall_s": round(wall, 3),
                              "gpu": gpu_info()}), flush=True)
    finally:
        shutil.rmtree(d, ignore_errors=True)
