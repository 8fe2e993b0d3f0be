#!/usr/bin/env python
"""The cost of the S3 CRC32 / CRC32C checksums in the SSE-C seal and reseal (DESIGN.md 4.12).

(a) DEVICE mode, --blocks x 1 MiB blocks under RS(10,4): garage_ec_seal_crc and garage_ec_reseal_crc (a key rotation,
    and a re-chunk where every destination is the unaligned tail of one source and the head of the next) with every
    block's kind none / CRC32 / CRC32C.  CUDA events, one warm-up call of each, then --rounds rounds alternating the
    three kinds; whole-call median and range.  A torch.profiler run of each (call, kind) gives the chunk kernel's time.
(b) The block manager on a file store under /dev/shm, RS(10,4), 14 nodes: a --bm-mib MiB object sealed with
    garage_bm_rpc_put_block_sealed_crc, then its key rotated block by block with garage_bm_rpc_put_block_resealed_crc
    from 16 threads; the folded checksum is checked against zlib, and the wall time reported.
One JSON line per result, with the card's name and power limit read in the same run.

    python tools/crc_bench.py [--blocks 4096] [--rounds 3] [--bm-mib 64] [--out profiles/crc_bench_h100.jsonl]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time
import zlib
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

import garage_b200 as G  # noqa: E402
from garage_b200 import block_manager as BM  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--blocks", type=int, default=4096)
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--bm-mib", type=int, default=64)
ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "crc_bench_h100.jsonl"))
args = ap.parse_args()
BLOCK = 1 << 20
KINDS = {"none": None, "crc32": G.CRC32, "crc32c": G.CRC32C}


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


def dev32(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int32)).cuda()


k, m, tot = 10, 4, 14
ec = G.GarageEc(0, k, m)
sealed = G.sealed_len(BLOCK)
stride = ec.stride_for(ec.code_shard_len(sealed))

# ---- (a) DEVICE
n = args.blocks
gen = torch.Generator(device="cuda").manual_seed(3)
plain = torch.randint(0, 256, (n * BLOCK,), dtype=torch.uint8, device="cuda", generator=gen)
keys = torch.randint(0, 256, (n * 32,), dtype=torch.uint8, device="cuda", generator=gen)
nonces = torch.randint(0, 256, (n * 8,), dtype=torch.uint8, device="cuda", generator=gen)
new_keys = torch.randint(0, 256, (n * 32,), dtype=torch.uint8, device="cuda", generator=gen)
plen = dev32(np.full(n, BLOCK, dtype=np.uint32))
src = torch.zeros(n * tot * stride, dtype=torch.uint8, device="cuda")
hashes = torch.zeros(n * 32, dtype=torch.uint8, device="cuda")
dst = torch.zeros(n * tot * stride, dtype=torch.uint8, device="cuda")
dst_hashes = torch.zeros(n * 32, dtype=torch.uint8, device="cuda")
crcs = torch.zeros(n, dtype=torch.int32, device="cuda")
kind_arr = {name: None if v is None else torch.full((n,), v, dtype=torch.uint8, device="cuda") for name, v in KINDS.items()}
ec.seal(plain, BLOCK, plen, keys, nonces, src, stride, hashes, n=n)
torch.cuda.synchronize()

src_len = dev32(np.full(n, sealed, dtype=np.uint32))
healthy = torch.ones(n * tot, dtype=torch.uint8, device="cuda")
rot_pieces = np.stack([np.arange(n), np.zeros(n), np.full(n, BLOCK)], axis=1).astype(np.uint32)
off = (4097 + 16 * np.arange(n) + np.arange(n) % 13).astype(np.uint32)  # unaligned, every residue mod 16
chunk_pieces = np.stack([np.stack([np.arange(n), off, BLOCK - off], axis=1),
                         np.stack([(np.arange(n) + 1) % n, np.zeros(n), off], axis=1)], axis=1).reshape(-1, 3).astype(np.uint32)
layouts = {"rotation": (dev32(rot_pieces), dev32(np.arange(n + 1, dtype=np.uint32))),
           "rechunk_2_pieces": (dev32(chunk_pieces), dev32(2 * np.arange(n + 1, dtype=np.uint32)))}
dst_len = torch.zeros(n, dtype=torch.int32, device="cuda")
bad = torch.zeros(n, dtype=torch.uint8, device="cuda")
src_status = torch.zeros(n, dtype=torch.int32, device="cuda")
status = torch.zeros(n, dtype=torch.int32, device="cuda")


def seal(kind):
    kw = {} if kind_arr[kind] is None else {"crc_kind": kind_arr[kind], "crcs": crcs}
    return lambda: ec.seal(plain, BLOCK, plen, new_keys, nonces, dst, stride, dst_hashes, n=n, **kw)


def reseal(layout, kind):
    pieces, start = layouts[layout]
    kw = {} if kind_arr[kind] is None else {"crc_kind": kind_arr[kind], "crcs": crcs}
    return lambda: ec.reseal(src, healthy, src_len, hashes, keys, pieces, start, new_keys, nonces, dst, dst_hashes,
                             dst_len, bad, src_status, status, stride, n_src=n, n_dst=n, **kw)


def spot_check(kind, call, layout=None):
    """a few blocks' checksums against zlib / CRC32C of the plaintext (the measured calls compute the right thing)"""
    if KINDS[kind] is None:
        return
    got = crcs.cpu().numpy().view(np.uint32)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import crc_oracle as CO

    for d in (0, n // 2, n - 1):
        if call == "seal" or layout == "rotation":
            q = plain[d * BLOCK:(d + 1) * BLOCK].cpu().numpy()
        else:
            o = int(off[d])
            q = torch.cat([plain[d * BLOCK + o:(d + 1) * BLOCK], plain[((d + 1) % n) * BLOCK:((d + 1) % n) * BLOCK + o]]).cpu().numpy()
        want = zlib.crc32(q.tobytes()) if KINDS[kind] == G.CRC32 else CO.crc(CO.CRC32C, q)
        assert int(got[d]) == want, (call, layout, kind, d)


def chunk_kernel_ms(fn):
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    t = {}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
        if us > 0:
            t[e.key] = us / 1e3
    return round(sum(v for key, v in t.items() if "sse_chunk_kernel" in key), 3), \
        round(sum(v for key, v in t.items() if "sse_crc_pass_kernel" in key), 3)


workloads = [("seal", None, {kind: seal(kind) for kind in KINDS})]
workloads += [("reseal", layout, {kind: reseal(layout, kind) for kind in KINDS}) for layout in layouts]
for call, layout, fns in workloads:
    for f in fns.values():
        event_ms(f)
    t = {kind: [] for kind in fns}
    for _ in range(args.rounds):
        for kind, f in fns.items():
            t[kind].append(event_ms(f))
            spot_check(kind, call, layout)
    assert call == "seal" or (status.cpu().numpy() == 0).all()
    for kind, v in t.items():
        chunk, passes = chunk_kernel_ms(fns[kind])
        emit(part="a_device", call=call, workload=layout or "seal", kind=kind, blocks=n, block_bytes=BLOCK,
             code="RS(10,4)", ms_median=round(float(np.median(v)), 3), ms_min=round(min(v), 3), ms_max=round(max(v), 3),
             rounds=args.rounds, chunk_kernel_ms=chunk, crc_pass_kernels_ms=passes)

del plain, src, dst
torch.cuda.empty_cache()
ec.close()

# ---- (b) the block manager on /dev/shm: a checksummed object's key rotation
nb = args.bm_mib
d = tempfile.mkdtemp(dir="/dev/shm" if os.path.isdir("/dev/shm") else None)
try:
    with BM.BlockManager(k=10, m=4, n_nodes=14, data_dir=d, batch_max_blocks=32) as bm:
        rng = np.random.default_rng(9)
        old_key, new_key = bytes(rng.integers(0, 256, 32, dtype=np.uint8)), bytes(rng.integers(0, 256, 32, dtype=np.uint8))
        obj = rng.integers(0, 256, nb * BLOCK, dtype=np.uint8)
        want = zlib.crc32(obj.tobytes())
        srcs = []
        for i in range(nb):
            rc, h, c = bm.rpc_put_block_sealed_crc(old_key, obj[i * BLOCK:(i + 1) * BLOCK], BM.CRC32)
            assert rc == BM.OK
            srcs.append((h, c))
        put_fold = 0
        for _, c in srcs:
            put_fold = G.crc_combine(G.CRC32, put_fold, c, BLOCK)
        assert put_fold == want
        del obj  # the copy below is given hashes and keys only

        def copy(h):
            rc, _, _, c = bm.put_block_resealed_crc([(h, 0, BLOCK)], old_key, new_key, BM.CRC32)
            assert rc == BM.OK, rc
            return c

        m0 = bm.reseal_metrics()
        t0 = time.perf_counter()
        with ThreadPoolExecutor(16) as ex:
            out = list(ex.map(copy, [h for h, _ in srcs]))
        wall = time.perf_counter() - t0
        m1 = bm.reseal_metrics()
        fold = 0
        for c in out:
            fold = G.crc_combine(G.CRC32, fold, c, BLOCK)
        assert fold == want
        emit(part="b_block_manager", workload="key_rotation_crc32", object_mib=nb, block_bytes=BLOCK, code="RS(10,4)",
             threads=16, wall_s=round(wall, 3), plaintext_gib_s=round(nb * BLOCK / wall / 2**30, 3),
             folded_crc_matches_zlib=True, plaintext_bytes_in_host_memory=0,
             how_checked="the copies are given block hashes and keys only; the sources are gathered as stored "
                         "(sealed) shards, each checksum returns as 4 bytes from the GPU call, and fallbacks = %d"
                         % (m1["fallbacks"] - m0["fallbacks"]),
             batches=m1["batches"] - m0["batches"], reseal_call_s=round((m1["reseal_call_us"] - m0["reseal_call_us"]) / 1e6, 3))
finally:
    shutil.rmtree(d, ignore_errors=True)
