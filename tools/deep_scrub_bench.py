#!/usr/bin/env python
"""Deep scrub measurements.

(a) Kernels, DEVICE mode, --blocks x 1 MiB stripes (encoded, every shard's tail past L poisoned) for RS(10,4),
    LRC(10,2,2), PB(10,4) and Clay(10,4): garage_ec_verify alone and garage_ec_deep_check end to end (CUDA events,
    warm-up, --rounds rounds alternating the codes, --iters calls per timing), then blake2sum_blocks_kernel alone from a
    torch.profiler run of its own.  Next to it, garage_ec_blake2sum of the same number of 1 MiB blocks on every host
    thread: the host work the hash kernel replaces.
(b) Block manager: a deep scrub of all 14 nodes of an RS(10,4) file store on /dev/shm holding --bm-blocks x 1 MiB:
    wall time, bytes read per block ((k+m)*L expected) and the share of deep_check_call_us.
One JSON line per result, with the card name and power limit read in the same run.

    python tools/deep_scrub_bench.py [--blocks 4096] [--rounds 3] [--iters 5] [--bm-blocks 256]
"""
import argparse
import ctypes as C
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

import garage_b200 as G  # noqa: E402
import oracle_lib as O  # noqa: E402
from garage_b200 import block_manager as BM  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--blocks", type=int, default=4096)
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--iters", type=int, default=5)
ap.add_argument("--bm-blocks", type=int, default=256)
args = ap.parse_args()
BLOCK = 1 << 20


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True, timeout=30).stdout.strip()
    return out.splitlines()[0] if out else None


def emit(**kw):
    print(json.dumps({**kw, "gpu": GPU}), flush=True)


GPU = gpu_info()
assert torch.cuda.is_available(), "needs cuda:0"

# ---- (a) kernels
CODES = [("RS(10,4)", lambda: G.GarageEc(0, 10, 4)), ("LRC(10,2,2)", lambda: G.GarageEc.lrc(0, 10, 2, 2)),
         ("PB(10,4)", lambda: G.GarageEc.piggyback(0, 10, 4)), ("Clay(10,4)", lambda: G.GarageEc.clay(0, 10, 4))]
n = args.blocks
setups = []
for name, mk in CODES:
    ec = mk()
    k, m = ec.k, ec.m
    L = ec.code_shard_len(BLOCK)
    stride = (L + 127) // 128 * 128
    data = torch.zeros((n, k, stride), dtype=torch.uint8, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(0xD5B)
    for s0 in range(0, n, 256):  # in slices: a whole batch of random int64 would not fit next to the shards
        blk = torch.randint(0, 256, (min(256, n - s0), k * L), generator=g, device="cuda", dtype=torch.uint8)
        blk[:, BLOCK:] = 0
        data[s0:s0 + blk.shape[0], :, :L] = blk.view(-1, k, L)
    parity = torch.zeros((n, m, stride), dtype=torch.uint8, device="cuda")
    sl = torch.full((n,), L, dtype=torch.int32, device="cuda")
    ec.encode(data, parity, stride, n, shard_len=sl)
    sh = torch.cat([data, parity], dim=1).contiguous()
    del data, parity
    sh[:, :, L:] = 0xA5
    blen = torch.full((n,), BLOCK, dtype=torch.int32, device="cuda")
    hashes = torch.zeros((n, 32), dtype=torch.uint8, device="cuda")
    bad = torch.zeros(n, dtype=torch.uint8, device="cuda")
    mm = torch.zeros(n, dtype=torch.int32, device="cuda")
    setups.append(dict(name=name, ec=ec, sh=sh, sl=sl, blen=blen, hashes=hashes, bad=bad, mm=mm, stride=stride, L=L))
    torch.cuda.synchronize()


def run_verify(x):
    x["ec"].verify(x["sh"], x["mm"], x["stride"], n, shard_len=x["sl"])


def run_deep(x):
    x["ec"].deep_check(x["sh"], x["blen"], x["hashes"], x["bad"], x["mm"], x["stride"], n)


def timed(fn, x):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(args.iters):
        fn(x)
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / args.iters


for x in setups:  # warm-up
    run_verify(x)
    run_deep(x)
    torch.cuda.synchronize()
    assert int(x["bad"].sum()) == n  # the zero hashes are wrong for every block
    run_verify(x)
    torch.cuda.synchronize()
    assert int(x["mm"].abs().sum()) == 0, x["name"]
res = {x["name"]: {"verify_ms": [], "deep_check_ms": []} for x in setups}
for r in range(args.rounds):
    for x in setups:
        res[x["name"]]["verify_ms"].append(round(timed(run_verify, x), 3))
        res[x["name"]]["deep_check_ms"].append(round(timed(run_deep, x), 3))

# the hash kernel alone, from a profiler run of its own
from torch.profiler import ProfilerActivity, profile  # noqa: E402

hash_ms = {}
for x in setups:
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.iters):
            run_deep(x)
        torch.cuda.synchronize()
    durs = [e.device_time_total / max(e.count, 1) for e in prof.key_averages() if "blake2sum_blocks_kernel" in e.key]
    hash_ms[x["name"]] = round(durs[0] / 1000.0, 3) if durs else None
for x in setups:
    emit(bench="deep_check_kernels", code=x["name"], blocks=n, block_bytes=BLOCK, shard_len=x["L"],
         hash_kernel_ms=hash_ms[x["name"]], **res[x["name"]])
del setups
torch.cuda.empty_cache()

# host threads: garage_ec_blake2sum of the same number of 1 MiB blocks
lib = G.load_library()
host = torch.randint(0, 256, (n, BLOCK), dtype=torch.uint8, device="cuda").cpu().numpy()
out = bytearray(32 * n)
threads = os.cpu_count() or 1


def hash_one(s):
    lib.garage_ec_blake2sum(C.c_void_p(host[s].ctypes.data), BLOCK, (C.c_char * 32).from_buffer(out, 32 * s))


walls = []
with ThreadPoolExecutor(threads) as ex:
    list(ex.map(hash_one, range(min(n, threads))))  # warm-up
    for r in range(args.rounds):
        t0 = time.perf_counter()
        list(ex.map(hash_one, range(n)))
        walls.append(round((time.perf_counter() - t0) * 1000, 1))
emit(bench="host_blake2sum", blocks=n, block_bytes=BLOCK, threads=threads, wall_ms=walls)
del host

# ---- (b) block manager sweep
blocks = [O.fill_random(BLOCK, 0xD5C0 + i) for i in range(args.bm_blocks)]
bhash = [BM.blake2sum(b) for b in blocks]
base = "/dev/shm" if os.path.isdir("/dev/shm") else None
d = tempfile.mkdtemp(prefix="deep_scrub_bench_", dir=base)
try:
    with BM.BlockManager(k=10, m=4, n_nodes=14, data_dir=d) as bm:
        for h, b in zip(bhash, blocks):
            assert bm.rpc_put_block(h, b) == 0
        for node in range(14):  # warm-up: pinned batch buffer, contexts, kernels
            bm.deep_scrub_step(node, None, 1)
        m0 = bm.metrics()
        t0 = time.perf_counter()
        checked = repaired = 0
        for node in range(14):
            rc, _, fin, c, r = bm.deep_scrub_step(node)
            assert rc == 0 and fin
            checked += c
            repaired += r
        wall = time.perf_counter() - t0
        m1 = bm.metrics()
        L = G.GarageEc(0, 10, 4).code_shard_len(BLOCK)
        emit(bench="bm_deep_scrub", code="RS(10,4)", blocks=args.bm_blocks, checked=checked, repaired=repaired,
             wall_s=round(wall, 3), read_bytes_per_block=round((m1["bytes_read"] - m0["bytes_read"]) / max(checked, 1)),
             expected_bytes_per_block=14 * L,
             deep_check_share=round((m1["deep_check_call_us"] - m0["deep_check_call_us"]) / 1e6 / wall, 3))
finally:
    shutil.rmtree(d, ignore_errors=True)
