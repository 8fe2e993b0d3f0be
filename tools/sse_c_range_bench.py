#!/usr/bin/env python
"""Ranged SSE-C open measurements (DESIGN.md 4.10).

(a) DEVICE mode, --blocks sealed 1 MiB blocks under RS(10,4), one 4 KiB and one 64 KiB plaintext range per block at
    seeded offsets, healthy and with the data shard holding the range's first byte absent.  CUDA events, a warm-up call
    of every variant, then --rounds rounds that run the variants in alternating order; median and spread (min, max)
    of each: garage_ec_open_range, garage_ec_open of the same blocks (whole-block rebuild, hash, every tag, decrypt),
    and garage_ec_decode_range of the same prefix and span bytes (the unencrypted ranged read of those bytes).  Every
    range's output is compared with the plaintext.  A separate torch.profiler run gives each kernel's time.
(b) Block manager on /dev/shm, RS, LRC, PB and Clay: the bytes one 4 KiB garage_bm_rpc_get_block_range_opened fetches
    (planned runs) and reads (the holders' tag spans), chunk-aligned and not, healthy and with the holder of the touched
    data shard down, against the bytes garage_bm_rpc_get_block_opened of the same block reads.  Counts, no timing.
One JSON line per result, with the card's name and power limit read in the same run.

    python tools/sse_c_range_bench.py [--blocks 4096] [--rounds 7] [--out profiles/sse_c_range_bench_h100.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import garage_b200 as G  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--blocks", type=int, default=4096)
ap.add_argument("--rounds", type=int, default=7)
ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "sse_c_range_bench_h100.jsonl"))
args = ap.parse_args()
BLOCK = 1 << 20


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True, timeout=30).stdout.strip()
    return out.splitlines()[0] if out else None


assert torch.cuda.is_available(), "needs cuda:0"
GPU = gpu_info()
OUT = open(args.out, "w")


def emit(**kw):
    line = json.dumps({**kw, "gpu": GPU})
    print(line, flush=True)
    OUT.write(line + "\n")
    OUT.flush()


n = args.blocks
ec = G.GarageEc(0, 10, 4)
k, m, tot = 10, 4, 14
S = G.sealed_len(BLOCK)
L = ec.code_shard_len(S)
stride = ec.stride_for(L)
gen = torch.Generator(device="cuda").manual_seed(1)
plain = torch.randint(0, 256, (n * BLOCK,), dtype=torch.uint8, device="cuda", generator=gen)
keys = torch.randint(0, 256, (n * 32,), dtype=torch.uint8, device="cuda", generator=gen)
nonces = torch.randint(0, 256, (n * 8,), dtype=torch.uint8, device="cuda", generator=gen)
plen = torch.full((n,), BLOCK, dtype=torch.int32, device="cuda")
shards = torch.zeros(n * tot * stride, dtype=torch.uint8, device="cuda")
hashes = torch.zeros(n * 32, dtype=torch.uint8, device="cuda")
ec.seal(plain, BLOCK, plen, keys, nonces, shards, stride, hashes, n=n)
torch.cuda.synchronize()
sealed = torch.full((n,), S, dtype=torch.int32, device="cuda")

rng = np.random.default_rng(7)
RANGES = {}
for size in (4096, 65536):
    offs = rng.integers(0, BLOCK - size + 1, n).astype(np.uint32)
    spans = [ec.sealed_range(S, int(o), size) for o in offs]
    pres = np.ones((n, tot), dtype=np.uint8)
    # degraded: the data shard that holds the span's first byte is absent
    deg = pres.copy()
    for s, sp in enumerate(spans):
        deg[s, sp[0] // L] = 0
    RANGES[size] = dict(offs=offs, spans=spans, healthy=pres, degraded=deg)

out_open = torch.empty(n * BLOCK, dtype=torch.uint8, device="cuda")
plen_out = torch.zeros(n, dtype=torch.int32, device="cuda")
hash_bad = torch.zeros(n, dtype=torch.uint8, device="cuda")
status = torch.zeros(n, dtype=torch.int32, device="cuda")


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int32) if a.dtype == np.uint32 else a).cuda()


VARIANTS = {}
for size, R in RANGES.items():
    o_stride = size
    d_off, d_len = dev(R["offs"]), dev(np.full(n, size, dtype=np.uint32))
    out = torch.empty(n * o_stride, dtype=torch.uint8, device="cuda")
    # decode_range of the same bytes: request 2s = the prefix, 2s + 1 = the span
    sp = np.array(R["spans"], dtype=np.uint32)
    dr_off = np.stack([np.zeros(n, np.uint32), sp[:, 0]], 1).reshape(-1)
    dr_len = np.stack([np.full(n, 8, np.uint32), sp[:, 1]], 1).reshape(-1)
    dr_stride = (int(dr_len.max()) + 15) // 16 * 16
    dr_out = torch.empty(2 * n * dr_stride, dtype=torch.uint8, device="cuda")
    dr_blen = torch.full((2 * n,), S, dtype=torch.int32, device="cuda")
    for health in ("healthy", "degraded"):
        pr = dev(R[health].reshape(-1))
        pr2 = dev(np.repeat(R[health], 2, axis=0).reshape(-1))
        VARIANTS[("open_range", size, health)] = (
            lambda pr=pr, d_off=d_off, d_len=d_len, out=out, o_stride=o_stride:
            ec.open_range(shards, pr, sealed, keys, d_off, d_len, stride, out, o_stride, status), out, d_off, size)
        if size == 4096:
            VARIANTS[("open", BLOCK, health)] = (
                lambda pr=pr: ec.open(shards, pr, sealed, hashes, keys, out_open, BLOCK, plen_out, hash_bad, status,
                                      stride, n=n), None, None, BLOCK)
        VARIANTS[("decode_range_same_bytes", size, health)] = (
            (lambda pr2=pr2, d_o=dev(dr_off), d_l=dev(dr_len), dr_out=dr_out, dr_stride=dr_stride:
             ec.decode_range(shards2, pr2, dr_blen, d_o, d_l, stride, dr_out, dr_stride)), None, None, size)

# decode_range's request s reads stripe s: a copy of the stripes with each one twice (prefix request, span request)
shards2 = shards.view(n, tot * stride).repeat_interleave(2, dim=0).reshape(-1)

# correctness of every open_range variant before timing
for key, (fn, out, d_off, size) in VARIANTS.items():
    fn()
    torch.cuda.synchronize()
    if key[0] == "open_range":
        assert int(status.abs().sum()) == 0, key
        o = d_off.cpu().numpy().view(np.uint32).astype(np.int64)
        got = out.view(n, size)
        idx = torch.from_numpy(o).cuda()[:, None] + torch.arange(size, device="cuda")[None, :]
        want = plain.view(n, BLOCK).gather(1, idx)
        assert torch.equal(got, want), key
    elif key[0] == "open":
        assert int(status.abs().sum()) == 0 and int(hash_bad.sum()) == 0, key
        assert torch.equal(out_open, plain), key

names = list(VARIANTS)
times = {kk: [] for kk in names}
ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
for r in range(args.rounds):
    order = names if r % 2 == 0 else names[::-1]
    for kk in order:
        fn = VARIANTS[kk][0]
        torch.cuda.synchronize()
        ev[0].record()
        fn()
        ev[1].record()
        torch.cuda.synchronize()
        times[kk].append(ev[0].elapsed_time(ev[1]))
for kk in names:
    t = sorted(times[kk])
    emit(bench="device_" + kk[0], code="RS(10,4)", blocks=n, block=BLOCK, range_bytes=kk[1], holders=kk[2],
         rounds=args.rounds, ms_median=t[len(t) // 2], ms_min=t[0], ms_max=t[-1])

# per-kernel times: one call of each 4 KiB variant and one whole-block open, in a profiler run of its own
from torch.profiler import ProfilerActivity, profile  # noqa: E402

for kk in [("open_range", 4096, "healthy"), ("open_range", 4096, "degraded"), ("open", BLOCK, "healthy")]:
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        VARIANTS[kk][0]()
        torch.cuda.synchronize()
    kern = {}
    for e in prof.events():
        if e.device_type.name == "CUDA" and "Memcpy" not in e.name and "Memset" not in e.name:
            kern[e.name.split("(")[0]] = kern.get(e.name.split("(")[0], 0.0) + e.device_time_total / 1000.0
    emit(bench="kernels_" + kk[0], range_bytes=kk[1], holders=kk[2], blocks=n,
         kernel_ms={a: round(b, 4) for a, b in sorted(kern.items(), key=lambda x: -x[1])})

# (b) bytes per 4 KiB ranged opened GET through the block manager on /dev/shm, against the opened GET of the block:
# garage_bm_rpc_get_block_range_opened's counters (fetched: planned run bytes; read: the tag spans the holders read)
# and bytes_read of garage_bm_rpc_get_block_opened.  Counts, no timing.
import tempfile  # noqa: E402

from garage_b200 import block_manager as BM  # noqa: E402

BM_CODES = {"RS(10,4)": dict(k=10, m=4), "LRC(10,2,2)": dict(k=10, m=4, local_groups=2),
            "PB(10,4)": dict(k=10, m=4, piggyback=True), "Clay(10,4)": dict(k=10, m=4, clay=True)}
shm = "/dev/shm" if os.path.isdir("/dev/shm") else None
for name, kw in BM_CODES.items():
    with tempfile.TemporaryDirectory(dir=shm) as d, BM.BlockManager(n_nodes=14, data_dir=d, **kw) as bm:
        key = bytes(range(32))
        p = np.random.default_rng(3).integers(0, 256, BLOCK, dtype=np.uint8)
        rc, h = bm.rpc_put_block_sealed(key, p)
        assert rc == BM.OK
        for aligned in (True, False):
            o = 4096 * 100 + (0 if aligned else 7)
            for health in ("healthy", "holder_down"):
                row = bm.storage_nodes_of(h)
                down = None
                if health == "holder_down":
                    with (G.GarageEc.clay(0, 10, 4) if kw.get("clay") else G.GarageEc.piggyback(0, 10, 4)
                          if kw.get("piggyback") else G.GarageEc(0, 10, 4)) as c:
                        down = row[c.sealed_range(S, o, 4096)[0] // c.code_shard_len(S)]
                    bm.set_node_up(down, False)
                m0 = bm.get_sealed_range_metrics()
                rc, got = bm.rpc_get_block_range_opened(h, key, o, 4096)
                m1 = bm.get_sealed_range_metrics()
                assert rc == BM.OK and np.array_equal(got, p[o:o + 4096]), (name, aligned, health)
                b0 = bm.metrics()["bytes_read"]
                rc, whole = bm.rpc_get_block_opened(h, key)
                b1 = bm.metrics()["bytes_read"]
                assert rc == BM.OK and np.array_equal(whole, p)
                if down is not None:
                    bm.set_node_up(down, True)
                emit(bench="bm_bytes_4KiB_ranged_opened_get", code=name, aligned=aligned, holders=health,
                     fetched=m1["bytes_fetched"] - m0["bytes_fetched"], read=m1["bytes_read"] - m0["bytes_read"],
                     degraded=m1["degraded_gets"] - m0["degraded_gets"], opened_get_read=b1 - b0, store=shm or "tmp")
OUT.close()
