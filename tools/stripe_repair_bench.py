#!/usr/bin/env python
"""Repair of a correlated failure under the block manager: a 14-node file store on /dev/shm holding 256 x 1 MiB blocks
under RS(10,4), LRC(10,2,2), PB(10,4) and Clay(10,4) in turn; e in {1, 2, 3} holders are down while the blocks are
written, then come back.  Two identical stores are repaired:
  - per node: each returning node runs repair_enqueue_missing + resync_all while the other returning nodes' shards are
    still missing (what each sees when they come back together and resync concurrently; the order is fixed so the
    byte counts are exact);
  - stripe: stripe_repair_all, every owner's sweep once.
One JSON line per (code, e): bytes fetched per block (handed to the rebuild: what would cross the network in Garage)
and read per block (what the holders read from disk) for each path, the shards rebuilt, the time inside
garage_ec_reconstruct_stripes and the wall time of the repair, with the GPU name and power limit of the run.

    python tools/stripe_repair_bench.py [--blocks 256]
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
args = ap.parse_args()

CODES = (("RS(10,4)", {}), ("LRC(10,2,2)", {"local_groups": 2}), ("PB(10,4)", {"piggyback": True}),
         ("Clay(10,4)", {"clay": True}))
DOWN = [1, 5, 9]


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True, timeout=30).stdout.strip()
    return out.splitlines()[0] if out else None


def store(base, kw, down):
    d = tempfile.mkdtemp(prefix="stripe_repair_bench_", dir=base)
    bm = BM.BlockManager(k=10, m=4, n_nodes=14, data_dir=d, **kw)
    for n in down:
        bm.set_node_up(n, False)
    for h, b in zip(hashes, blocks):
        assert bm.rpc_put_block(h, b) == 0
    return d, bm


def check(bm):
    ok = all(bm.node_shard_index(n, h) == i for h in hashes for i, n in enumerate(bm.storage_nodes_of(h)))
    for h, b in zip(hashes, blocks):
        rc, got = bm.rpc_get_block(h)
        ok = ok and rc == 0 and bytes(got) == bytes(b)
    return ok


def per_node(bm, down):
    m0 = bm.metrics()
    t0 = time.perf_counter()
    done = 0
    for d in down:
        bm.set_node_up(d, True)
        bm.repair_enqueue_missing(d)
        failed, n = bm.resync_all(d)
        assert failed == 0
        done += n
        bm.set_node_up(d, False)
    wall = time.perf_counter() - t0
    for d in down:
        bm.set_node_up(d, True)
    m1 = bm.metrics()
    return {"fetched_bytes_per_block": round((m1["resync_bytes_fetched"] - m0["resync_bytes_fetched"]) / len(blocks)),
            "read_bytes_per_block": round((m1["resync_bytes_read"] - m0["resync_bytes_read"]) / len(blocks)),
            "shards_rebuilt": done, "gpu_call_s": (m1["reconstruct_call_us"] - m0["reconstruct_call_us"]) / 1e6,
            "wall_s": round(wall, 3), "ok": check(bm)}


def stripe(bm, down):
    for d in down:
        bm.set_node_up(d, True)
    s0 = bm.stripe_repair_metrics()
    t0 = time.perf_counter()
    _, rebuilt = bm.stripe_repair_all()
    wall = time.perf_counter() - t0
    s1 = bm.stripe_repair_metrics()
    d = {k: s1[k] - s0[k] for k in s1}
    return {"fetched_bytes_per_block": round(d["stripe_repair_bytes_fetched"] / len(blocks)),
            "read_bytes_per_block": round(d["stripe_repair_bytes_read"] / len(blocks)), "shards_rebuilt": rebuilt,
            "gpu_call_s": d["stripe_repair_call_us"] / 1e6, "wall_s": round(wall, 3),
            "ok": d["stripe_repair_errors"] == 0 and check(bm)}


blocks = [O.fill_random(1 << 20, 0x5EC0 + i) for i in range(args.blocks)]
hashes = [BM.blake2sum(b) for b in blocks]
base = "/dev/shm" if os.path.isdir("/dev/shm") else None
gpu = gpu_info()
for code, kw in CODES:
    for e in (1, 2, 3):
        down = DOWN[:e]
        res = {}
        for name, fn in (("per_node", per_node), ("stripe", stripe)):
            d, bm = store(base, kw, down)
            try:
                res[name] = fn(bm, down)
            finally:
                bm.close()
                shutil.rmtree(d, ignore_errors=True)
        print(json.dumps({"code": code, "e": e, "blocks": args.blocks, "per_node": res["per_node"],
                          "stripe": res["stripe"],
                          "fetched_ratio": round(res["stripe"]["fetched_bytes_per_block"] /
                                                 max(res["per_node"]["fetched_bytes_per_block"], 1), 4),
                          "gpu": gpu}), flush=True)
