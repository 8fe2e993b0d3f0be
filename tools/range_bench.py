#!/usr/bin/env python
"""Ranged reads (DESIGN.md section 2.5) for RS(10,4), LRC(10,2,2), PB(10,4) and Clay(10,4) on 1 MiB blocks.

(a) block manager, file store on /dev/shm: per ranged GET, range_bytes_read (tag-span bytes read from shard files) and
    range_bytes_fetched (the planned runs: what would cross the network) for ranges of 4 KiB, 64 KiB, 256 KiB and the
    whole block, healthy and with the holder of the touched data shard down, against a full rpc_get_block of the same
    blocks in the same run (bytes_read), and the wall time of each sweep.  Also the plan's bytes alone
    (garage_ec_range_plan, exact from shapes).
(b) time, DEVICE: garage_ec_decode_range of N degraded 64 KiB ranges (one absent data shard per stripe, the range
    inside it) against garage_ec_reconstruct of the same N stripes (want = that shard), CUDA events, warm-up,
    alternating rounds.

    python tools/range_bench.py [--blocks 4096 --rounds 5 --iters 10]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ap = argparse.ArgumentParser()
ap.add_argument("--blocks", type=int, default=4096)
ap.add_argument("--rounds", type=int, default=5)
ap.add_argument("--iters", type=int, default=10)
ap.add_argument("--bm-blocks", type=int, default=64)
args = ap.parse_args()

import shutil  # noqa: E402
import tempfile  # noqa: E402
import time  # noqa: E402

import torch  # noqa: E402

import garage_b200 as G  # noqa: E402
from garage_b200 import block_manager as BM  # noqa: E402

B = 1 << 20
CODES = [("RS(10,4)", lambda: G.GarageEc(0, 10, 4)), ("LRC(10,2,2)", lambda: G.GarageEc.lrc(0, 10, 2, 2)),
         ("PB(10,4)", lambda: G.GarageEc.piggyback(0, 10, 4)), ("Clay(10,4)", lambda: G.GarageEc.clay(0, 10, 4))]
LENS = [("4KiB", 4096), ("64KiB", 65536), ("256KiB", 262144), ("block", B)]
LOST = 3  # the data shard that is down in the degraded cases


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:
        return None


def plan_bytes(ec, present, off, ln):
    runs, _ = ec.range_plan(present, B, off, ln)
    return sum(r[2] for r in runs)


def byte_table(name, ec):
    tot = ec.k + ec.m
    L = ec.code_shard_len(B)
    rng = np.random.default_rng(1)
    for degraded in (False, True):
        present = np.ones(tot, dtype=np.uint8)
        if degraded:
            present[LOST] = 0
        want = np.array([1] * ec.k + [0] * ec.m, dtype=np.uint8)
        full = sum(r[2] for r in ec.read_ranges(present, L, want=want)) if degraded else ec.k * L
        for lname, ln in LENS:
            if ln == B:
                offs = [0]
            elif degraded:  # ranges inside the lost shard (or as much of it as they can)
                offs = [int(LOST * L + x) for x in rng.integers(0, max(1, L - ln), 64)]
                offs = [min(o, B - ln) for o in offs]
            else:
                offs = [int(x) for x in rng.integers(0, B - ln, 64)]
            got = [plan_bytes(ec, present, o, ln) for o in offs]
            print(json.dumps({"table": "bytes", "code": name, "degraded": degraded, "range": lname,
                              "fetched_mean": float(np.mean(got)), "fetched_max": int(max(got)),
                              "full_get": int(full), "ratio": round(float(np.mean(got)) / full, 4)}), flush=True)


BM_CODES = {"RS(10,4)": dict(k=10, m=4), "LRC(10,2,2)": dict(k=10, m=4, local_groups=2),
            "PB(10,4)": dict(k=10, m=4, piggyback=True), "Clay(10,4)": dict(k=10, m=4, clay=True)}


def bm_table(name, L):
    root = "/dev/shm" if os.path.isdir("/dev/shm") else None
    d = tempfile.mkdtemp(prefix="range_bench_", dir=root)
    try:
        with BM.BlockManager(n_nodes=14, data_dir=d, **BM_CODES[name]) as bm:
            rng = np.random.default_rng(7)
            blocks = [rng.integers(0, 256, B, dtype=np.uint8) for _ in range(args.bm_blocks)]
            hashes = [BM.blake2sum(b) for b in blocks]
            for h, b in zip(hashes, blocks):
                assert bm.rpc_put_block(h, b) == BM.OK
            m0, t0 = bm.metrics(), time.perf_counter()
            for h in hashes:
                assert bm.rpc_get_block(h)[0] == BM.OK
            full_s, m1 = time.perf_counter() - t0, bm.metrics()
            full_read = (m1["bytes_read"] - m0["bytes_read"]) / len(hashes)
            for degraded in (False, True):
                for lname, ln in LENS:
                    offs = [0] if ln == B else [int(LOST * L + x) for x in rng.integers(0, max(1, L - ln), len(hashes))]
                    offs = [min(o, B - ln) for o in offs]
                    m0, t0 = bm.metrics(), time.perf_counter()
                    for x, h in enumerate(hashes):
                        o = offs[x % len(offs)]
                        node = bm.storage_nodes_of(h)[LOST]
                        if degraded:
                            bm.set_node_up(node, False)
                        rc, got = bm.rpc_get_block_range(h, o, ln)
                        if degraded:
                            bm.set_node_up(node, True)
                        assert rc == BM.OK and np.array_equal(got, blocks[x][o:o + ln])
                    dt, m1 = time.perf_counter() - t0, bm.metrics()
                    n = len(hashes)
                    print(json.dumps({"table": "block_manager", "code": name, "degraded": degraded, "range": lname,
                                      "range_bytes_read": (m1["range_bytes_read"] - m0["range_bytes_read"]) / n,
                                      "range_bytes_fetched": (m1["range_bytes_fetched"] - m0["range_bytes_fetched"]) / n,
                                      "range_degraded": m1["range_degraded"] - m0["range_degraded"],
                                      "full_get_bytes_read": full_read, "sweep_s": round(dt, 4),
                                      "full_get_sweep_s": round(full_s, 4), "requests": n}), flush=True)
    finally:
        shutil.rmtree(d, ignore_errors=True)


def time_device(name, ec):
    n, tot = args.blocks, ec.k + ec.m
    L = ec.code_shard_len(B)
    stride = ec.stride_for(L)
    shards = torch.empty(n * tot * stride, dtype=torch.uint8, device="cuda")
    ec.fill_random(shards, shards.numel(), 0x72616E6765)
    present = torch.ones(n, tot, dtype=torch.uint8, device="cuda")
    present[:, LOST] = 0
    want = torch.zeros(n, tot, dtype=torch.uint8, device="cuda")
    want[:, LOST] = 1
    lens32 = torch.full((n,), L, dtype=torch.int32, device="cuda")
    g = torch.Generator().manual_seed(3)
    ln = 65536
    offs = (LOST * L + torch.randint(0, L - ln, (n,), generator=g)).to(torch.int32).cuda()
    blen = torch.full((n,), B, dtype=torch.int32, device="cuda")
    rlen = torch.full((n,), ln, dtype=torch.int32, device="cuda")
    out = torch.empty(n * ln, dtype=torch.uint8, device="cuda")
    status = torch.empty(n, dtype=torch.int32, device="cuda")

    def ranged():
        ec.decode_range(shards, present, blen, offs, rlen, stride, out, ln, status=status)

    def whole():
        ec.reconstruct(shards, present, stride, n, want=want, status=status, shard_len=lens32)

    t = {"range": [], "reconstruct": []}
    for f in (ranged, whole):  # warm-up of every shape
        f()
    torch.cuda.synchronize()
    for _ in range(args.rounds):
        for key, f in (("range", ranged), ("reconstruct", whole)):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.iters):
                f()
            b.record()
            b.synchronize()
            t[key].append(a.elapsed_time(b) / args.iters)
    assert int(status.abs().sum()) == 0
    r, w = float(np.median(t["range"])), float(np.median(t["reconstruct"]))
    print(json.dumps({"table": "device_time", "code": name, "requests": n, "range_bytes": ln,
                      "decode_range_ms": round(r, 4), "reconstruct_ms": round(w, 4), "speedup": round(w / r, 2),
                      "decode_range_ms_rounds": [round(x, 4) for x in t["range"]],
                      "reconstruct_ms_rounds": [round(x, 4) for x in t["reconstruct"]]}))
    del shards, out


def main():
    assert torch.cuda.is_available(), "range_bench needs a GPU"
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit(), "block_bytes": B}))
    for name, make in CODES:
        with make() as ec:
            byte_table(name, ec)
            L = ec.code_shard_len(B)
            time_device(name, ec)
        bm_table(name, L)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
