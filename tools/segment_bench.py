"""Device time of garage_ec_reconstruct_segments on 4096 x 1 MiB RS(10,4) stripes with 5 and with 8 damaged shards per
stripe (their damage in disjoint adler8 segments), alternated in one process with garage_ec_reconstruct of 4 erasures
per stripe.  CUDA events around each call, after a warm-up of every shape; the card's name and power limit are read in
the same run and written beside every time.  One JSON line per measurement (stdout, and --out).

Then, through the block manager on /dev/shm (a file store), --bm-blocks 1 MiB RS(10,4) blocks each with m+1 shards
damaged in different segments: the salvage wall time of one GET per block and the shard bytes salvage read per block
(garage_bm_salvage_metrics).

A rescue path: no speed-up is expected or claimed.  Algorithmic bytes (DESIGN.md 4.13) = survivor units read + rebuilt
units written."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import garage_b200 as G  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    name, plim = (x.strip() for x in out[0].split(","))
    return name, plim


def bm_salvage(nblocks, name, plim):
    import shutil
    import tempfile
    import time

    from garage_b200 import block_manager as BM

    k, m = 10, 4
    d = tempfile.mkdtemp(prefix="segment_bench_", dir="/dev/shm")
    try:
        with BM.BlockManager(k, m, data_dir=d) as bm:
            rng = np.random.default_rng(3)
            hs = []
            for b in range(nblocks):
                blk = rng.integers(0, 256, 1 << 20, dtype=np.uint8)
                h = BM.blake2sum(blk)
                assert bm.rpc_put_block(h, blk) == BM.OK
                hs.append(h)
            L = -(-(1 << 20) // k)
            S = (-(-L // 8) + 15) // 16 * 16
            for h in hs:
                who = bm.storage_nodes_of(h)
                for i in range(m + 1):
                    assert bm.corrupt_shard(who[i], h, i * S + 7) == BM.OK
            t0 = time.perf_counter()
            for h in hs:
                rc, _ = bm.rpc_get_block(h)
                assert rc == BM.OK
            wall = time.perf_counter() - t0
            mt = bm.salvage_metrics()
            assert mt["salvage_blocks"] == nblocks
            return dict(tool="segment_bench", case="bm_salvaged_get", store="/dev/shm", blocks=nblocks,
                        damaged_shards=m + 1, ms_per_get=round(1e3 * wall / nblocks, 3),
                        salvage_bytes_read_per_block=mt["salvage_bytes_read"] // nblocks,
                        salvage_call_ms_per_block=round(mt["salvage_call_us"] / 1e3 / nblocks, 3),
                        gpu=name, power_limit=plim)
    finally:
        shutil.rmtree(d, ignore_errors=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=4096)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    ap.add_argument("--bm-blocks", type=int, default=64)
    a = ap.parse_args()
    import torch

    k, m, n = 10, 4, a.n
    tot = k + m
    name, plim = card()
    rows = []
    with G.GarageEc(0, k, m) as ec:
        L = ec.shard_len(1 << 20)
        stride = ec.stride_for(L)
        seg = (-(-L // 8) + 15) // 16 * 16
        sh = torch.empty(n * tot * stride, dtype=torch.uint8, device="cuda")
        v = sh.view(n, tot, stride)
        gen = torch.Generator(device="cuda").manual_seed(1)
        v[:, :k] = torch.randint(0, 256, (n, k, stride), dtype=torch.uint8, device="cuda", generator=gen)
        v[:, :, L:] = 0
        par = torch.zeros(n * m * stride, dtype=torch.uint8, device="cuda")
        ec.encode(v[:, :k].contiguous().view(-1), par, stride, n)
        v[:, k:] = par.view(n, m, stride)
        orig = sh.clone()
        rng = np.random.default_rng(2)

        def seg_map(nbad):
            sp = np.full((n, tot), 0xFF, dtype=np.uint8)
            for s in range(n):
                units = rng.permutation(8)
                for j, i in enumerate(rng.choice(tot, nbad, replace=False)):
                    sp[s, i] &= ~np.uint8(1 << int(units[j % 8]))
            return torch.from_numpy(sp.reshape(-1)).cuda()

        present = np.ones((n, tot), dtype=np.uint8)
        for s in range(n):
            present[s, rng.choice(tot, m, replace=False)] = 0
        cases = {"segments_5": seg_map(5), "segments_8": seg_map(8), "reconstruct_4": torch.from_numpy(present).cuda()}
        status = torch.zeros(n, dtype=torch.int32, device="cuda")

        def call(case):
            if case == "reconstruct_4":
                ec.reconstruct(sh, cases[case], stride, n, status=status)
            else:
                ec.reconstruct_segments(sh, cases[case], stride, n, status=status)

        for case in cases:  # warm-up, and the bytes come back
            call(case)
            torch.cuda.synchronize()
            assert int(status.abs().sum()) == 0 and torch.equal(sh, orig), case
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for r in range(a.rounds):
            for case in cases:
                e0.record()
                for _ in range(a.reps):
                    call(case)
                e1.record()
                torch.cuda.synchronize()
                ms = e0.elapsed_time(e1) / a.reps
                nbad = int(case.split("_")[1])
                # reconstruct reads k survivors and writes m shards; segments read k survivor segments and write one
                # segment per damaged shard, in every unit with damage
                rd, wr = ((k * L, m * L) if case == "reconstruct_4" else (min(nbad, 8) * k * seg, nbad * seg))
                row = dict(tool="segment_bench", case=case, round=r, n=n, shard_len=L, ms=round(ms, 4),
                           algo_bytes_per_stripe=rd + wr, gbps=round(n * (rd + wr) / ms / 1e6, 1), gpu=name,
                           power_limit=plim)
                rows.append(row)
                print(json.dumps(row), flush=True)
    rows.append(bm_salvage(a.bm_blocks, name, plim))
    print(json.dumps(rows[-1]), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            for row in rows:
                f.write(json.dumps(row) + "\n")


if __name__ == "__main__":
    main()
