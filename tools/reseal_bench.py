#!/usr/bin/env python
"""SSE-C copies with re-encryption (DESIGN.md 4.11), against the two calls they replace.

(a) DEVICE mode, --blocks x 1 MiB sealed blocks under RS(10,4): garage_ec_reseal of a 1:1 key rotation on healthy
    stripes and with 4 erasures per source stripe, and of a re-chunk where every destination is the unaligned tail of
    one source and the head of the next; against garage_ec_open into device plaintext followed by garage_ec_seal of
    the same blocks.  CUDA events, one warm-up call of each, then --rounds alternating rounds; median and range.  A
    torch.profiler run of one reseal and one open + seal gives each kernel's time.
(b) HOST mode on pinned buffers, --host-blocks x 1 MiB: garage_ec_reseal_stripes against garage_ec_open_stripes
    followed by garage_ec_seal_blocks, wall clock, alternating rounds.
(c) The block manager on a file store under /dev/shm, RS(10,4), 14 nodes: --bm-blocks sealed 1 MiB blocks copied under a
    new key by garage_bm_rpc_put_block_resealed from 16 threads, healthy and with m = 4 holders of every source
    without their shard (the nodes stay up, so the new blocks reach their write quorum);
    bytes read per source and written per destination, fallbacks, batches and wall time.
One JSON line per result, with the card's name and power limit read in the same run.

    python tools/reseal_bench.py [--blocks 4096] [--rounds 5] [--host-blocks 256] [--bm-blocks 256] [--out profiles/reseal_bench_h100.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import garage_b200 as G  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--blocks", type=int, default=4096)
ap.add_argument("--rounds", type=int, default=5)
ap.add_argument("--host-blocks", type=int, default=256)
ap.add_argument("--bm-blocks", type=int, default=256)
ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "reseal_bench_h100.jsonl"))
ap.add_argument("--profile-dir", default=None, help="write the torch.profiler traces here")
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


def event_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def alternate(fns, rounds, clock):
    """one warm-up call of each, then `rounds` rounds calling them in turn; per fn: (median, min, max) ms"""
    for f in fns.values():
        clock(f)
    t = {name: [] for name in fns}
    for _ in range(rounds):
        for name, f in fns.items():
            t[name].append(clock(f))
    return {name: (float(np.median(v)), min(v), max(v)) for name, v in t.items()}


def wall_ms(fn):
    t0 = time.perf_counter()
    fn()
    return (time.perf_counter() - t0) * 1e3


k, m, tot = 10, 4, 14
ec = G.GarageEc(0, k, m)
sealed = G.sealed_len(BLOCK)
stride = ec.stride_for(ec.code_shard_len(sealed))


def dev32(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int32)).cuda()


# ---- (a) DEVICE
n = args.blocks
gen = torch.Generator(device="cuda").manual_seed(1)
plain = torch.randint(0, 256, (n * BLOCK,), dtype=torch.uint8, device="cuda", generator=gen)
keys = torch.randint(0, 256, (n * 32,), dtype=torch.uint8, device="cuda", generator=gen)
nonces = torch.randint(0, 256, (n * 8,), dtype=torch.uint8, device="cuda", generator=gen)
new_keys = torch.randint(0, 256, (n * 32,), dtype=torch.uint8, device="cuda", generator=gen)
plen = dev32(np.full(n, BLOCK, dtype=np.uint32))
src = torch.zeros(n * tot * stride, dtype=torch.uint8, device="cuda")
hashes = torch.zeros(n * 32, dtype=torch.uint8, device="cuda")
ec.seal(plain, BLOCK, plen, keys, nonces, src, stride, hashes, n=n)
torch.cuda.synchronize()
del plain
src_len = dev32(np.full(n, sealed, dtype=np.uint32))
healthy = torch.ones(n * tot, dtype=torch.uint8, device="cuda")
rng = np.random.default_rng(2)
er = np.ones((n, tot), dtype=np.uint8)
for s in range(n):
    er[s, rng.choice(tot, 4, replace=False)] = 0
erased = torch.from_numpy(er.reshape(-1)).cuda()

rot_pieces = np.stack([np.arange(n), np.zeros(n), np.full(n, BLOCK)], axis=1).astype(np.uint32)
off = (4097 + 16 * np.arange(n) + np.arange(n) % 13).astype(np.uint32)  # unaligned, every residue mod 16
chunk_pieces = np.stack([np.stack([np.arange(n), off, BLOCK - off], axis=1),
                         np.stack([(np.arange(n) + 1) % n, np.zeros(n), off], axis=1)], axis=1).reshape(-1, 3).astype(np.uint32)
layouts = {"rotation": (dev32(rot_pieces), dev32(np.arange(n + 1, dtype=np.uint32))),
           "rechunk": (dev32(chunk_pieces), dev32(2 * np.arange(n + 1, dtype=np.uint32)))}

dst = torch.zeros(n * tot * stride, dtype=torch.uint8, device="cuda")
dst_hashes = torch.zeros(n * 32, dtype=torch.uint8, device="cuda")
dst_len = torch.zeros(n, dtype=torch.int32, device="cuda")
bad = torch.zeros(n, dtype=torch.uint8, device="cuda")
src_status = torch.zeros(n, dtype=torch.int32, device="cuda")
status = torch.zeros(n, dtype=torch.int32, device="cuda")
pt = torch.zeros(n * BLOCK, dtype=torch.uint8, device="cuda")
plen_out = torch.zeros(n, dtype=torch.int32, device="cuda")
work = src.clone()


def reseal(present, layout):
    pieces, start = layouts[layout]
    return lambda: ec.reseal(work, present, src_len, hashes, keys, pieces, start, new_keys, nonces, dst, dst_hashes,
                             dst_len, bad, src_status, status, stride, n_src=n, n_dst=n)


def open_seal(present):
    def f():
        ec.open(work, present, src_len, hashes, keys, pt, BLOCK, plen_out, bad, status, stride, n=n)
        ec.seal(pt, BLOCK, plen_out, new_keys, nonces, dst, stride, dst_hashes, n=n)
    return f


for layout, present, label in (("rotation", healthy, "rotation_healthy"), ("rotation", erased, "rotation_4_erasures"),
                               ("rechunk", healthy, "rechunk_2_pieces")):
    fns = {"reseal": reseal(present, layout), "open+seal": open_seal(present)}
    res = alternate(fns, args.rounds, event_ms)
    st = status.cpu().numpy()
    assert (st == 0).all(), st
    for name, (med, lo, hi) in res.items():
        emit(part="a_device", workload=label, call=name, blocks=n, block_bytes=BLOCK, code="RS(10,4)",
             ms_median=round(med, 3), ms_min=round(lo, 3), ms_max=round(hi, 3), rounds=args.rounds,
             plaintext_gib_s=round(n * BLOCK / (med / 1e3) / 2**30, 2))

# kernel breakdown, a run of its own
from torch.profiler import ProfilerActivity, profile  # noqa: E402

for name, fn in (("reseal", reseal(healthy, "rotation")), ("open+seal", open_seal(healthy))):
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    if args.profile_dir:
        os.makedirs(args.profile_dir, exist_ok=True)
        prof.export_chrome_trace(os.path.join(args.profile_dir, "reseal_bench_%s.pt.trace.json" % name.replace("+", "_")))
    rows = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
        if t > 0:
            rows[e.key[:90]] = round(t / 1e3, 3)
    emit(part="a_kernels", workload="rotation_healthy", call=name, kernel_ms=dict(sorted(rows.items(), key=lambda x: -x[1])))

del work, src, dst, pt
torch.cuda.empty_cache()

# ---- (b) HOST, pinned
hn = args.host_blocks
held = []


def pinned(nbytes):
    a, p = ec.host_alloc(nbytes)
    held.append(p)
    return a


h_plain = pinned(hn * BLOCK)
h_plain[:] = np.random.default_rng(3).integers(0, 256, hn * BLOCK, dtype=np.uint8)
hk = np.random.default_rng(4).integers(0, 256, (hn, 32), dtype=np.uint8)
hk2 = np.random.default_rng(5).integers(0, 256, (hn, 32), dtype=np.uint8)
hnon = np.random.default_rng(6).integers(0, 256, (hn, 8), dtype=np.uint8)
h_src = pinned(hn * tot * stride)
h_hash = np.zeros((hn, 32), dtype=np.uint8)
ec.seal_blocks([h_plain[s * BLOCK:(s + 1) * BLOCK] for s in range(hn)], hk, hnon, h_src, stride, h_hash)
stripes = [h_src[s * tot * stride:(s + 1) * tot * stride] for s in range(hn)]
h_dst = pinned(hn * tot * stride)
h_out = pinned(hn * BLOCK)
outs = [h_out[s * BLOCK:(s + 1) * BLOCK] for s in range(hn)]
h_pres = np.ones((hn, tot), dtype=np.uint8)
h_len = np.full(hn, sealed, dtype=np.uint32)
h_pieces = np.stack([np.arange(hn), np.zeros(hn), np.full(hn, BLOCK)], axis=1).astype(np.uint32)
h_start = np.arange(hn + 1, dtype=np.uint32)
h_dh, h_dl = np.zeros((hn, 32), dtype=np.uint8), np.zeros(hn, dtype=np.uint32)
h_bad, h_sst, h_st = np.zeros(hn, dtype=np.uint8), np.zeros(hn, dtype=np.int32), np.zeros(hn, dtype=np.int32)


def h_reseal():
    assert ec.reseal_stripes(stripes, h_pres, h_len, h_hash, hk, h_pieces, h_start, hk2, hnon, h_dst, h_dh, h_dl,
                             h_bad, h_sst, h_st, stride) == 0


def h_open_seal():
    assert ec.open_stripes(stripes, h_pres, h_len, h_hash, hk, outs, h_dl, h_bad, h_st, stride) == 0
    ec.seal_blocks(outs, hk2, hnon, h_dst, stride, h_dh)


res = alternate({"reseal_stripes": h_reseal, "open_stripes+seal_blocks": h_open_seal}, args.rounds, wall_ms)
for name, (med, lo, hi) in res.items():
    emit(part="b_host_pinned", workload="rotation_healthy", call=name, blocks=hn, block_bytes=BLOCK, code="RS(10,4)",
         ms_median=round(med, 3), ms_min=round(lo, 3), ms_max=round(hi, 3), rounds=args.rounds,
         plaintext_gib_s=round(hn * BLOCK / (med / 1e3) / 2**30, 2))
for p in held:
    ec.host_free(p)
ec.close()

# ---- (c) block manager on /dev/shm
import shutil  # noqa: E402
import tempfile  # noqa: E402
from concurrent.futures import ThreadPoolExecutor  # noqa: E402

from garage_b200 import block_manager as BM  # noqa: E402

bn = args.bm_blocks
d = tempfile.mkdtemp(dir="/dev/shm" if os.path.isdir("/dev/shm") else None)
try:
    with BM.BlockManager(k=10, m=4, n_nodes=14, data_dir=d, batch_max_blocks=32) as bm:
        rng = np.random.default_rng(7)
        old_key, new_key = bytes(rng.integers(0, 256, 32, dtype=np.uint8)), bytes(rng.integers(0, 256, 32, dtype=np.uint8))
        srcs = []
        for i in range(bn):
            rc, h = bm.rpc_put_block_sealed(old_key, rng.integers(0, 256, BLOCK, dtype=np.uint8))
            assert rc == BM.OK
            srcs.append(h)

        def copy(h):
            rc, _, _ = bm.put_block_resealed([(h, 0, BLOCK)], old_key, new_key)
            assert rc == BM.OK, rc

        for label, lost in (("healthy", 0), ("m_holders_without_their_shard", 4)):
            for h in srcs:  # the nodes stay up: every new block needs its write quorum
                row = bm.storage_nodes_of(h)
                for i in range(lost):
                    assert bm.drop_shard(row[i], h) == BM.OK
            m0, w0 = bm.reseal_metrics(), bm.metrics()["bytes_written"]
            t0 = time.perf_counter()
            with ThreadPoolExecutor(16) as ex:
                list(ex.map(copy, srcs))
            wall = time.perf_counter() - t0
            m1, w1 = bm.reseal_metrics(), bm.metrics()["bytes_written"]
            emit(part="c_block_manager", workload=label, blocks=bn, block_bytes=BLOCK, code="RS(10,4)", threads=16,
                 wall_s=round(wall, 3), plaintext_gib_s=round(bn * BLOCK / wall / 2**30, 3),
                 bytes_read_per_source=(m1["bytes_read"] - m0["bytes_read"]) / bn,
                 bytes_written_per_destination=(w1 - w0) / bn, fallbacks=m1["fallbacks"] - m0["fallbacks"],
                 batches=m1["batches"] - m0["batches"], calls=m1["calls"] - m0["calls"],
                 reseal_call_s=round((m1["reseal_call_us"] - m0["reseal_call_us"]) / 1e6, 3))
finally:
    shutil.rmtree(d, ignore_errors=True)
