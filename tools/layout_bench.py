"""Rate of changing the cluster layout: a file store of N blocks under RS(10,4), two sweeps of layout_sync_step over
every node.  With --clay each sweep also runs on a Clay(10,4) store (clay_layout = 1), next to RS(10,4) in the same run.

  copy:    14 storage nodes -> 16: the new nodes copy their shards from the old holders (one shard read per shard).
  rebuild: 15 storage nodes, one of them down, then removed: its shards are rebuilt on the GPU from k survivors each
           (Clay: from the garage_ec_read_ranges runs of the 13 others; bytes_fetched counts what the rebuilds and
           copies were handed, bytes_read what the holders read to check their tags).

Reports GiB/s of moved shard bytes over the sweep's wall time, the bytes moved against garage_layout_transition's shard
count x shard size, and the share of the sweep spent inside garage_ec_* calls.  The store lives under /dev/shm when it
exists (the sweep then measures the manager and the GPU, not a disk).  Prints one JSON line.

    python tools/layout_bench.py --blocks 256 --clay
"""
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
from garage_b200 import block_manager as BM  # noqa: E402
from garage_b200 import placement as PL  # noqa: E402

N_NODES, K, M = 16, 10, 4
CAP = 1 << 40


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def run(kind, nblocks, block_len, base, clay=False):
    rng = np.random.default_rng(11)
    blocks = [rng.integers(0, 256, block_len, dtype=np.uint8) for _ in range(nblocks)]
    hashes = [BM.blake2sum(b) for b in blocks]
    zone = [0] * N_NODES
    if kind == "copy":
        before = [CAP] * 14 + [0] * 2
        after = [CAP] * N_NODES
        dead = None
    else:
        before = [CAP] * 15 + [0]
        dead = 3
        after = [c if n != dead else 0 for n, c in enumerate(before)]
    d = tempfile.mkdtemp(prefix="layout_bench_", dir=base)
    try:
        with BM.BlockManager(K, M, n_nodes=N_NODES, data_dir=d, layout={"zone": zone, "capacity": before}, clay=clay,
                             clay_layout=clay) as bm:
            for h, b in zip(hashes, blocks):
                assert bm.rpc_put_block(h, b) == BM.OK
            if dead is not None:
                bm.set_node_up(dead, False)
            assert bm.apply_layout(zone, after)[0] == BM.OK
            base_mt = bm.metrics()
            t0 = time.perf_counter()
            moved = bm.layout_sync_all()
            el = time.perf_counter() - t0
            mt = bm.metrics()
            for i in range(0, nblocks, max(1, nblocks // 16)):  # spot-check the result
                rc, got = bm.rpc_get_block(hashes[i])
                assert rc == BM.OK and np.array_equal(got, blocks[i])
            versions = bm.layout_versions()
        l1 = PL.Layout.compute(zone, before, K + M)
        l2 = PL.Layout.compute(zone, after, K + M, previous=l1, version=2)
        shards = sum(len(l1.transition_to(l2, PL.partition_of(h))) for h in hashes)
        L = -(-block_len // K)
        if clay:  # rounded up to 16 * alpha = 4096
            L = -(-L // 4096) * 4096
        rebuild_read = (K + M - 1) if clay else K  # whole shards read per rebuilt shard
        gpu_us = sum(mt[x] - base_mt[x] for x in ("reconstruct_call_us", "encode_call_us", "convert_call_us"))
        assert moved == shards and mt["layout_sync_errors"] == 0 and versions == [2], (moved, shards, versions)
        return {
            "code": "Clay(10,4)" if clay else "RS(10,4)", "sweep": kind, "blocks": nblocks, "block_len": block_len,
            "sweep_s": round(el, 4),
            "shards_moved": moved, "transition_shards": shards,
            "gib_per_s": round(moved * L / el / (1 << 30), 3),
            "bytes_written": mt["layout_bytes_written"], "bytes_written_algorithmic": shards * L,
            "bytes_read": mt["layout_bytes_read"],
            "bytes_read_algorithmic": shards * L * (1 if kind == "copy" else rebuild_read),
            "bytes_fetched": mt["layout_bytes_fetched"],
            "bytes_fetched_per_shard": round(mt["layout_bytes_fetched"] / max(1, moved)),
            "copied": mt["layout_shards_copied"], "rebuilt": mt["layout_shards_rebuilt"],
            "gpu_call_share": round(gpu_us / 1e6 / el, 3),
        }
    finally:
        shutil.rmtree(d, ignore_errors=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=256)
    ap.add_argument("--block-len", type=int, default=1 << 20)
    ap.add_argument("--sweeps", default="copy,rebuild")
    ap.add_argument("--clay", action="store_true", help="each sweep on a Clay(10,4) store too")
    a = ap.parse_args()
    base = "/dev/shm" if os.path.isdir("/dev/shm") and os.access("/dev/shm", os.W_OK) else None
    codes = [False, True] if a.clay else [False]
    res = [run(s, a.blocks, a.block_len, base, clay) for s in a.sweeps.split(",") for clay in codes]
    print(json.dumps({"card": card(), "store": base or tempfile.gettempdir(), "runs": res}))


if __name__ == "__main__":
    main()
