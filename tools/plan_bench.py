#!/usr/bin/env python
"""Time the decode planner on its own: the plan kernel that garage_ec_reconstruct (DEVICE mode) launches before its
apply kernels, read from a torch.profiler trace, since a timer around the call cannot separate the two.  Cases: RS(10,4),
RS(32,8), LRC(10,2,2) and PB(10,4), each with m random erasures per stripe (some LRC stripes are unrecoverable) and
with one random lost data shard.  One JSON line per case; the planner does not read shard bytes, so the shards are
small.

    python tools/plan_bench.py [--so path/to/libgarage_ec.so] [--blocks 4096 --iters 50]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ap = argparse.ArgumentParser()
ap.add_argument("--so", default=None)
ap.add_argument("--blocks", type=int, default=4096)
ap.add_argument("--iters", type=int, default=50)
ap.add_argument("--tag", default="")
args = ap.parse_args()

from garage_b200 import _build  # noqa: E402

if args.so:
    _build.SO = os.path.abspath(args.so)
    _build.stale = lambda: False
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

import garage_b200 as G  # noqa: E402

CODES = [("RS(10,4)", lambda: G.GarageEc(0, 10, 4), 10, 4), ("RS(32,8)", lambda: G.GarageEc(0, 32, 8), 32, 8),
         ("LRC(10,2,2)", lambda: G.GarageEc.lrc(0, 10, 2, 2), 10, 4), ("PB(10,4)", lambda: G.GarageEc.piggyback(0, 10, 4), 10, 4)]


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:
        return None


def plan_times(ec, k, m, pattern):
    """device time in us of each plan-kernel launch over args.iters reconstruct calls"""
    n, tot, stride = args.blocks, k + m, 256
    g = torch.Generator().manual_seed(11)
    if pattern == "random_m":
        erased = torch.rand(n, tot, generator=g).argsort(dim=1)[:, :m]
    else:
        erased = torch.randint(0, k, (n, 1), generator=g)
    present = torch.ones(n, tot, dtype=torch.uint8)
    present.scatter_(1, erased, 0)
    pd = present.cuda()
    shards = torch.zeros(n * tot * stride, dtype=torch.uint8, device="cuda")
    status = torch.zeros(n, dtype=torch.int32, device="cuda")
    for _ in range(3):
        ec.reconstruct(shards, pd, stride, n, status=status)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.iters):
            ec.reconstruct(shards, pd, stride, n, status=status)
        torch.cuda.synchronize()
    ts = [e.time_range.elapsed_us() for e in prof.events() if "plan_kernel" in e.name and e.device_type.name == "CUDA"]
    assert len(ts) == args.iters, len(ts)
    return ts


def main():
    gpu, watts = torch.cuda.get_device_name(0), power_limit()
    for name, make, k, m in CODES:
        with make() as ec:
            for pattern in ("random_m", "one_data"):
                ts = sorted(plan_times(ec, k, m, pattern))
                print(json.dumps({"tag": args.tag or (args.so or "default"), "code": name, "pattern": pattern,
                                  "stripes": args.blocks, "launches": len(ts), "median_us": round(ts[len(ts) // 2], 2),
                                  "mean_us": round(sum(ts) / len(ts), 2), "min_us": round(ts[0], 2),
                                  "gpu": gpu, "power_limit_W": watts}), flush=True)


if __name__ == "__main__":
    main()
