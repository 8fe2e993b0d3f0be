#!/usr/bin/env python
"""SSE-C seal and open measurements (DESIGN.md 4.9).

(a) DEVICE mode, --blocks x 1 MiB under RS(10,4), CUDA events over --iters calls after a warm-up: garage_ec_seal (GCM,
    encode, content hash), garage_ec_open on healthy stripes and with 4 erasures per stripe (rebuild, hash, tag check,
    decrypt); next to them, from the same run, a device copy of the plaintext, garage_ec_encode of the same stripes and
    a deep check (blake2sum_blocks_kernel + verify).  A torch.profiler run of one seal and one open gives each kernel's
    time.
(b) HOST mode on pinned buffers, --host-blocks x 1 MiB: garage_ec_seal_blocks and garage_ec_open_stripes.
(c) What Garage pays on the CPU instead: STREAM seal (`cryptography`'s AES-256-GCM) plus blake2b of the sealed block,
    on every host thread; "not measured" when `cryptography` is absent.
One JSON line per result, with the card's name and power limit read in the same run.

    python tools/sse_c_bench.py [--blocks 4096] [--iters 5] [--host-blocks 256] [--out profiles/sse_c_bench_h100.jsonl]
"""
import argparse
import hashlib
import json
import os
import struct
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import garage_b200 as G  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--blocks", type=int, default=4096)
ap.add_argument("--iters", type=int, default=5)
ap.add_argument("--host-blocks", type=int, default=256)
ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "sse_c_bench_h100.jsonl"))
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


def timed(fn, iters):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


n = args.blocks
ec = G.GarageEc(0, 10, 4)
k, m, tot = 10, 4, 14
sealed = G.sealed_len(BLOCK)
L = ec.code_shard_len(sealed)
stride = ec.stride_for(L)
gen = torch.Generator(device="cuda").manual_seed(1)
plain = torch.randint(0, 256, (n * BLOCK,), dtype=torch.uint8, device="cuda", generator=gen)
plen = torch.full((n,), BLOCK, dtype=torch.int32, device="cuda")
keys = torch.randint(0, 256, (n * 32,), dtype=torch.uint8, device="cuda", generator=gen)
nonces = torch.randint(0, 256, (n * 8,), dtype=torch.uint8, device="cuda", generator=gen)
shards = torch.zeros(n * tot * stride, dtype=torch.uint8, device="cuda")
hashes = torch.zeros(n * 32, dtype=torch.uint8, device="cuda")
GiB = n * BLOCK / 2**30


def seal():
    ec.seal(plain, BLOCK, plen, keys, nonces, shards, stride, hashes, n=n)


t_seal = timed(seal, args.iters)
emit(bench="seal_device", code="RS(10,4)", blocks=n, block=BLOCK, ms=t_seal, plain_GiB_per_s=GiB / (t_seal / 1e3))

stored = shards.clone()
present = torch.ones(n * tot, dtype=torch.uint8, device="cuda")
deg = torch.ones(n, tot, dtype=torch.uint8)
rng = np.random.default_rng(3)
for s in range(n):
    deg[s, torch.from_numpy(rng.choice(tot, 4, replace=False))] = 0
deg = deg.reshape(-1).cuda()
slen = torch.full((n,), sealed, dtype=torch.int32, device="cuda")
out = torch.zeros(n * BLOCK, dtype=torch.uint8, device="cuda")
olen = torch.zeros(n, dtype=torch.int32, device="cuda")
bad = torch.zeros(n, dtype=torch.uint8, device="cuda")
status = torch.zeros(n, dtype=torch.int32, device="cuda")
for name, pres in (("open_device_healthy", present), ("open_device_4_erasures", deg)):
    t = timed(lambda: ec.open(shards, pres, slen, hashes, keys, out, BLOCK, olen, bad, status, stride, n=n), args.iters)
    torch.cuda.synchronize()
    ok = int(status.abs().sum()) == 0 and int(bad.sum()) == 0 and torch.equal(out, plain)
    emit(bench=name, code="RS(10,4)", blocks=n, block=BLOCK, ms=t, plain_GiB_per_s=GiB / (t / 1e3), round_trip_ok=ok)
    shards.copy_(stored)

t_copy = timed(lambda: out.copy_(plain), args.iters)
emit(bench="device_copy", bytes=n * BLOCK, ms=t_copy, GiB_per_s=GiB / (t_copy / 1e3))
par = torch.zeros(n * m * stride, dtype=torch.uint8, device="cuda")
dl = torch.full((n,), L, dtype=torch.int32, device="cuda")
data = shards.view(n, tot, stride)[:, :k].contiguous().view(-1)
t_enc = timed(lambda: ec.encode(data, par, stride, n, shard_len=dl), args.iters)
emit(bench="rs_encode_device", code="RS(10,4)", blocks=n, shard_len=L, ms=t_enc)
del data, par
mm = torch.zeros(n, dtype=torch.int32, device="cuda")
t_deep = timed(lambda: ec.deep_check(shards, slen, hashes, bad, mm, stride, n), args.iters)
emit(bench="deep_check_device", code="RS(10,4)", blocks=n, block=sealed, ms=t_deep)

# per-kernel times of one seal and one degraded open
with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    seal()
    ec.open(shards, deg, slen, hashes, keys, out, BLOCK, olen, bad, status, stride, n=n)
    torch.cuda.synchronize()
kern = {}
for e in prof.key_averages():
    if e.device_type == torch.autograd.DeviceType.CUDA:
        kern[e.key] = kern.get(e.key, 0.0) + e.device_time_total / 1e3
emit(bench="kernels_seal_and_degraded_open", code="RS(10,4)", blocks=n,
     kernel_ms={kname[:80]: round(v, 3) for kname, v in sorted(kern.items(), key=lambda x: -x[1])[:12]})
del plain, shards, stored, out
torch.cuda.empty_cache()

# ---- (b) HOST mode on pinned buffers
hn = args.host_blocks
pin_plain, pp = ec.host_alloc(hn * BLOCK)
pin_plain[:] = np.random.default_rng(5).integers(0, 256, hn * BLOCK, dtype=np.uint8)
pin_sh, ps = ec.host_alloc(hn * tot * stride)
hk = np.random.default_rng(6).integers(0, 256, hn * 32, dtype=np.uint8)
hnon = np.random.default_rng(7).integers(0, 256, hn * 8, dtype=np.uint8)
hh = np.zeros(hn * 32, dtype=np.uint8)
blocks = [pin_plain[s * BLOCK:(s + 1) * BLOCK] for s in range(hn)]
ec.seal_blocks(blocks, hk, hnon, pin_sh, stride, hh)
t0 = time.perf_counter()
for _ in range(args.iters):
    ec.seal_blocks(blocks, hk, hnon, pin_sh, stride, hh)
dt = (time.perf_counter() - t0) / args.iters
emit(bench="seal_blocks_host_pinned", code="RS(10,4)", blocks=hn, ms=dt * 1e3, plain_GiB_per_s=hn * BLOCK / 2**30 / dt)
pin_out, po = ec.host_alloc(hn * BLOCK)
stripes = [pin_sh[s * tot * stride:(s + 1) * tot * stride] for s in range(hn)]
outs = [pin_out[s * BLOCK:(s + 1) * BLOCK] for s in range(hn)]
hpres = np.ones(hn * tot, dtype=np.uint8)
hsl = np.full(hn, sealed, dtype=np.uint32)
hol, hbad, hst = np.zeros(hn, dtype=np.uint32), np.zeros(hn, dtype=np.uint8), np.zeros(hn, dtype=np.int32)
ec.open_stripes(stripes, hpres, hsl, hh, hk, outs, hol, hbad, hst, stride)
t0 = time.perf_counter()
for _ in range(args.iters):
    ec.open_stripes(stripes, hpres, hsl, hh, hk, outs, hol, hbad, hst, stride)
dt = (time.perf_counter() - t0) / args.iters
emit(bench="open_stripes_host_pinned_healthy", code="RS(10,4)", blocks=hn, ms=dt * 1e3,
     plain_GiB_per_s=hn * BLOCK / 2**30 / dt, round_trip_ok=bool(np.array_equal(pin_out, pin_plain) and not hst.any()))
for p in (pp, ps, po):
    ec.host_free(p)

# ---- (c) the CPU stage Garage runs instead
try:
    from cryptography.hazmat.primitives.ciphers.aead import AESGCM
except ImportError:
    AESGCM = None
if AESGCM is None:
    emit(bench="cpu_stream_seal_plus_blake2b", result="not measured: cryptography is not installed")
else:
    threads = os.cpu_count()
    body = np.random.default_rng(8).integers(0, 256, BLOCK, dtype=np.uint8).tobytes()

    def one(i):
        g = AESGCM(bytes(32))
        nonce = struct.pack("<Q", i)
        b = bytearray(nonce)
        for c in range(256):
            b += g.encrypt(nonce + struct.pack("<I", c | ((c == 255) << 31)), body[4096 * c:4096 * (c + 1)], None)
        hashlib.blake2b(bytes(b)).digest()

    cnt = max(hn, threads * 4)
    with ThreadPoolExecutor(threads) as ex:
        list(ex.map(one, range(threads)))
        t0 = time.perf_counter()
        list(ex.map(one, range(cnt)))
        dt = time.perf_counter() - t0
    emit(bench="cpu_stream_seal_plus_blake2b", threads=threads, blocks=cnt, s=dt,
         plain_GiB_per_s=cnt * BLOCK / 2**30 / dt)
OUT.close()
