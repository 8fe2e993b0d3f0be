#!/usr/bin/env python
"""Resync during an outage, with and without Garage's backoff: a 14-node file store on /dev/shm holding 256 x 1 MiB
blocks under RS(10,4) and LRC(10,2,2) in turn.  m+1 holders go down; one of them (node 0) comes back at once with an
empty disk, so its RepairWorker queues every block while the other m stay down and each of its resyncs reaches k-1
survivors, too few to rebuild from.  The test clock runs a six-hour outage minute by minute on two identical stores:
  - drain: garage_bm_resync_all every minute (every failed hash straight back in the queue);
  - step: garage_bm_resync_step every minute (ErrorCounter backoff, 1 minute up to 64 minutes).
Then the m holders return and the same call runs every minute until node 0 holds every shard and has no error entry.
One JSON line per (code, path): resync attempts and survivor bytes read during the outage, the minutes from the
holders' return to a clean queue, and the GPU name and power limit of the run.  These are counts, not timings.

    python tools/resync_backoff_bench.py [--blocks 256] [--hours 6] [--out profiles/resync_backoff_bench_h100.jsonl]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import oracle_lib as O  # noqa: E402

from garage_b200 import block_manager as BM  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--blocks", type=int, default=256)
ap.add_argument("--hours", type=float, default=6.0)
ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "resync_backoff_bench_h100.jsonl"))
args = ap.parse_args()

CODES = (("RS(10,4)", {}), ("LRC(10,2,2)", {"local_groups": 2}))
T0 = 1_700_000_000_000  # ms: the test clock at the start of the outage
MINUTE = 60000
NODE = 0  # the holder that returns with an empty disk


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True, timeout=30).stdout.strip()
    return out.splitlines()[0] if out else None


def run(kw, path, blocks, hashes, base):
    d = tempfile.mkdtemp(prefix="resync_backoff_bench_", dir=base)
    try:
        with BM.BlockManager(k=10, m=4, n_nodes=14, data_dir=d, **kw) as bm:
            assert bm.debug_set_clock_ms(T0) == BM.OK
            for h, b in zip(hashes, blocks):
                assert bm.rpc_put_block(h, b) == BM.OK
            down = list(range(1, 5))  # with NODE: m+1 holders of every block
            for h in hashes:
                assert bm.drop_shard(NODE, h) == BM.OK
            for n in down:
                bm.set_node_up(n, False)
            assert bm.repair_enqueue_missing(NODE) == len(hashes)

            def tick(minute):
                assert bm.debug_set_clock_ms(T0 + minute * MINUTE) == BM.OK
                if path == "drain":
                    bm.resync_all(NODE)
                else:
                    assert bm.resync_step(NODE)[0] == BM.OK

            m0 = bm.metrics()
            outage = int(round(args.hours * 60))
            for minute in range(outage):
                tick(minute)
            m1 = bm.metrics()
            at_return = len(bm.list_resync_errors(NODE)[1])
            for n in down:
                bm.set_node_up(n, True)
            minute = outage
            while True:
                tick(minute)
                minute += 1
                clean = all(bm.node_shard_index(NODE, h) >= 0 for h in hashes) and bm.list_resync_errors(NODE)[1] == []
                if clean or minute > outage + 24 * 60:
                    break
            ok = clean
            for h, b in zip(hashes, blocks):
                rc, got = bm.rpc_get_block(h)
                ok = ok and rc == BM.OK and got.tobytes() == b.tobytes()
            attempts = (m1["resync_counter"] + m1["resync_error_counter"]) - (m0["resync_counter"] + m0["resync_error_counter"])
            return {"outage_attempts": attempts, "outage_survivor_bytes_read": m1["resync_bytes_read"] - m0["resync_bytes_read"],
                    "minutes_to_clean_queue": minute - outage, "error_entries_at_return": at_return,
                    "resync_metrics": bm.resync_metrics(), "ok": ok}
    finally:
        shutil.rmtree(d, ignore_errors=True)


base = "/dev/shm" if os.path.isdir("/dev/shm") else None
blocks = [O.fill_random(1 << 20, 0x7265737963 + i) for i in range(args.blocks)]
hashes = [BM.blake2sum(b) for b in blocks]
gpu = gpu_info()
os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
with open(args.out, "w") as f:
    for name, kw in CODES:
        res = {p: run(kw, p, blocks, hashes, base) for p in ("drain", "step")}
        for p, r in res.items():
            line = {"code": name, "path": p, "blocks": args.blocks, "outage_hours": args.hours, **r, "gpu": gpu}
            if p == "step":
                line["survivor_bytes_ratio"] = round(r["outage_survivor_bytes_read"] / max(1, res["drain"]["outage_survivor_bytes_read"]), 5)
            print(json.dumps(line), flush=True)
            f.write(json.dumps(line) + "\n")
