#!/usr/bin/env python
"""Node-level rate of one block manager on several dispatcher groups (garage_bm_create_on_devices, DESIGN.md section
5.13), closed loop on the memory store with the native load generator (garage_bm_bench): T client threads PUT 1 MiB
blocks, GET them back healthy, then GET them with m holders down (every block rebuilt on the GPU).  The load threads
are bound round robin to the listed devices' NUMA nodes, so on a two-socket host with GPUs on both they run on both.

Configurations, one JSON line each:
  - "distinct": the first n visible GPUs, n in 1, 2, 4, 8 (a count larger than the visible GPUs is recorded as not
    measured);
  - "one_device": n groups on GPU 0, n in 1, 2, 4, 8: what the routing and the per-group pools cost or give on one card;
  - "compare": 2 GPUs on two NUMA nodes against 2 groups on one GPU, alternated --repeats times in this one call
    (recorded as not measured when the host has no two GPUs on different nodes).
Each line carries the card names and power limits read in the same run, and per group: batches, blocks, bytes and the
local / remote routing counts of the run.

    python tools/multi_gpu_bench.py [--threads 32] [--blocks 96] [--out profiles/multi_gpu_bench_h100.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import garage_b200 as G  # noqa: E402
from garage_b200 import block_manager as BM  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--threads", type=int, default=32)
ap.add_argument("--blocks", type=int, default=96, help="blocks per thread and run (32 x 96 x 1 MiB = 3 GiB)")
ap.add_argument("--k", type=int, default=10)
ap.add_argument("--m", type=int, default=4)
ap.add_argument("--counts", default="1,2,4,8")
ap.add_argument("--repeats", type=int, default=3, help="alternations of the two-device comparison")
ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
args = ap.parse_args()

B = 1 << 20
out_f = open(args.out, "a") if args.out else None


def emit(rec):
    line = json.dumps(rec)
    print(line, flush=True)
    if out_f:
        out_f.write(line + "\n")
        out_f.flush()


def gpus():
    """index -> {name, power_limit_w, numa_node} read now (nvidia-smi queries only)"""
    q = subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit,pci.bus_id", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True).stdout
    info = {}
    for row in q.strip().splitlines():
        i, name, pl, bus = [x.strip() for x in row.split(",")]
        node = -1
        try:
            node = int(open("/sys/bus/pci/devices/%s/numa_node" % bus.lower()[4:]).read())
        except (OSError, ValueError):
            pass
        info[int(i)] = {"name": name, "power_limit_w": float(pl), "numa_node": node}
    return info


def host():
    nodes = [x for x in os.listdir("/sys/devices/system/node") if x.startswith("node")] \
        if os.path.isdir("/sys/devices/system/node") else []
    return {"host_cpus": len(os.sched_getaffinity(0)), "host_numa_nodes": max(1, len(nodes))}


def measure(kind, devices, info):
    bm = BM.BlockManager(args.k, args.m, batch_max_blocks=64, block_ram_buffer_max=4 << 30, cuda_devices=devices)
    rec = {"kind": kind, "devices": devices, "measured": True, "threads": args.threads,
           "blocks_per_run": args.threads * args.blocks, "block_bytes": B, "k": args.k, "m": args.m,
           "gpus": {str(d): info.get(d) for d in sorted(set(devices))}, **host()}
    try:
        for mode, name, down in ((0, "put", False), (1, "get_healthy", False), (1, "get_m_down", True)):
            if down:
                for n in range(args.m):
                    bm.set_node_up(n, False)
            before = bm.device_metrics()
            rc, gibs, errs = bm.bench(args.threads, args.blocks, B, mode, seed=11)
            assert rc == 0 and errs == 0, (rc, errs)
            after = bm.device_metrics()
            rec[name + "_GiBs"] = round(gibs, 2)
            rec[name + "_groups"] = [{f: a[f] - b[f] for f in ("batches", "blocks", "bytes", "routed_local",
                                                               "routed_remote")} for a, b in zip(after, before)]
        rec["group_numa_nodes"] = [g["numa_node"] for g in bm.device_metrics()]
        rec["pool_numa_nodes"] = [g["pool_numa_node"] for g in bm.device_metrics()]
    finally:
        bm.close()
    return rec


def main():
    info = gpus()
    ndev = int(G.load_library().garage_ec_device_count())
    stamp = time.strftime("%Y-%m-%dT%H:%M:%SZ", time.gmtime())
    emit({"kind": "host", "time": stamp, "visible_gpus": ndev, "gpus": {str(i): v for i, v in info.items()}, **host()})
    counts = [int(c) for c in args.counts.split(",")]
    for n in counts:
        if n > ndev:
            emit({"kind": "distinct", "devices": list(range(n)), "measured": False,
                  "reason": "%d GPU(s) visible" % ndev})
        else:
            emit(measure("distinct", list(range(n)), info))
    for n in counts:
        if n > 1:  # one group on GPU 0 is the "distinct" n = 1 line
            emit(measure("one_device", [0] * n, info))
    by_node = {}
    for i in range(ndev):
        by_node.setdefault(info.get(i, {}).get("numa_node", -1), i)
    pair = [v for k, v in sorted(by_node.items()) if k >= 0][:2]
    if len(pair) < 2:
        emit({"kind": "compare", "measured": False,
              "reason": "no two GPUs on different NUMA nodes (%d visible)" % ndev})
        return
    for r in range(args.repeats):
        for kind, devs in (("compare_two_sockets", pair), ("compare_one_device", [pair[0], pair[0]])):
            rec = measure(kind, devs, info)
            rec["repeat"] = r
            emit(rec)


if __name__ == "__main__":
    main()
