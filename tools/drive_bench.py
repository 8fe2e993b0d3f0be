#!/usr/bin/env python
"""Drives under the block manager (DESIGN.md section 5.7): a 14-node file store on /dev/shm whose nodes each spread
their shard files over 4 drives of equal capacity, holding 256 x 1 MiB blocks.

  - lost: one drive of node 0 is wiped (RS(10,4), then Clay(10,4)).  The node restarts without it
    (garage_bm_set_data_dirs), repair_enqueue_missing queues its shards and resync_all rebuilds them on the GPU from
    the other nodes.  Recorded: the shards rebuilt against the count the drive layout predicts, resync_bytes_fetched
    (what would cross the network in Garage) and the wall time of the resync.
  - added: a fifth drive joins every node, then one rebalance pass per node.  Recorded: the files and bytes moved
    against the counts the drive layout predicts, and the wall time.

One JSON line per experiment, with the GPU name and power limit read in the same run.  Host file I/O dominates
these times; they are not a speed claim.

    python tools/drive_bench.py [--blocks 256] [--out FILE]
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
from garage_b200 import placement as P  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--blocks", type=int, default=256)
ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
args = ap.parse_args()

N, DRIVES = 14, [("d0", 1), ("d1", 1), ("d2", 1), ("d3", 1)]
LOST_NODE, LOST_DRIVE = 0, 1
CODES = (("RS(10,4)", {}), ("Clay(10,4)", {"clay": True}))


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True, timeout=30).stdout.strip()
    return out.splitlines()[0] if out else None


def emit(rec):
    line = json.dumps(rec)
    print(line, flush=True)
    if args.out:
        with open(args.out, "a") as f:
            f.write(line + "\n")


def shard_path(d, node, drive, h):
    return os.path.join(d, "node%d" % node, drive, h[:1].hex(), h[1:2].hex(), h.hex() + ".shard")


def check(bm):
    return all(bm.rpc_get_block(h)[0] == 0 and bytes(bm.rpc_get_block(h)[1]) == bytes(b) for h, b in zip(hashes, blocks))


def store(base, kw):
    d = tempfile.mkdtemp(prefix="drive_bench_", dir=base)
    bm = BM.BlockManager(k=10, m=4, n_nodes=N, data_dir=d, data_dirs=DRIVES, **kw)
    for h, b in zip(hashes, blocks):
        assert bm.rpc_put_block(h, b) == 0
    return d, bm


def lost(base, code, kw):
    d, bm = store(base, kw)
    try:
        layout = P.DriveLayout.init([c for _, c in DRIVES])
        predicted = sum(1 for h in hashes if LOST_NODE in bm.storage_nodes_of(h)
                        and layout.primary(P.drive_partition_of(h)) == LOST_DRIVE)
        shutil.rmtree(os.path.join(d, "node%d" % LOST_NODE, DRIVES[LOST_DRIVE][0]))
        rc_same = bm.set_data_dirs(LOST_NODE, DRIVES)
        rc_without = bm.set_data_dirs(LOST_NODE, [x for i, x in enumerate(DRIVES) if i != LOST_DRIVE])
        m0 = bm.metrics()
        queued = bm.repair_enqueue_missing(LOST_NODE)
        t0 = time.perf_counter()
        failed, done = bm.resync_all(LOST_NODE)
        wall = time.perf_counter() - t0
        m1 = bm.metrics()
        fetched = m1["resync_bytes_fetched"] - m0["resync_bytes_fetched"]
        emit({"experiment": "lost_drive", "code": code, "blocks": len(blocks), "nodes": N, "drives_per_node": len(DRIVES),
              "set_same_list_rc": rc_same, "set_without_rc": rc_without, "predicted_shards": predicted,
              "queued": queued, "shards_rebuilt": done, "failed": failed, "resync_bytes_fetched": fetched,
              "fetched_per_shard": round(fetched / max(done, 1)),
              "reconstruct_call_s": (m1["reconstruct_call_us"] - m0["reconstruct_call_us"]) / 1e6,
              "resync_wall_s": round(wall, 3), "gets_ok": check(bm), "gpu": gpu})
    finally:
        bm.close()
        shutil.rmtree(d, ignore_errors=True)


def added(base):
    d, bm = store(base, {})
    try:
        new = DRIVES + [("d4", 1)]
        before = P.DriveLayout.init([c for _, c in DRIVES])
        after = before.update([0, 1, 2, 3, -1], [c for _, c in new])
        files, nbytes = 0, 0
        for h in hashes:
            p = P.drive_partition_of(h)
            if after.primary(p) != before.primary(p):
                for node in bm.storage_nodes_of(h):
                    files += 1
                    nbytes += os.path.getsize(shard_path(d, node, DRIVES[before.primary(p)][0], h))
        for node in range(N):
            assert bm.set_data_dirs(node, new) == 0
        t0 = time.perf_counter()
        moved = bm.rebalance_all()
        wall = time.perf_counter() - t0
        dm = bm.drive_metrics()
        emit({"experiment": "add_drive_rebalance", "code": "RS(10,4)", "blocks": len(blocks), "nodes": N,
              "drives_per_node": len(new), "predicted_files": files, "predicted_bytes": nbytes, "files_moved": moved,
              "rebalance_files_moved": dm["rebalance_files_moved"], "rebalance_bytes_moved": dm["rebalance_bytes_moved"],
              "rebalance_errors": dm["rebalance_errors"], "second_pass_moved": bm.rebalance_all(),
              "rebalance_wall_s": round(wall, 3), "gets_ok": check(bm), "gpu": gpu})
    finally:
        bm.close()
        shutil.rmtree(d, ignore_errors=True)


blocks = [O.fill_random(1 << 20, 0xD21E + i) for i in range(args.blocks)]
hashes = [BM.blake2sum(b) for b in blocks]
base = "/dev/shm" if os.path.isdir("/dev/shm") else None
gpu = gpu_info()
for code, kw in CODES:
    lost(base, code, kw)
added(base)
