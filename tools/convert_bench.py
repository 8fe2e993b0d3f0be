"""Rate of changing a store's code: a file store of N blocks stored under RS(6,3), separately as rf = 3 plain
replicas, and separately under Clay(10,4) (--sources clay104), is restarted as RS(10,4) and converted by one
convert_step sweep over every node.

Reports GiB/s of block bytes over the sweep's wall time, the share of that time spent inside garage_ec_transcode, and
the bytes read and written per block against the algorithmic k_s*L_s read and (k_d+m_d)*L_d written.  The store lives
under /dev/shm when it exists (the sweep then measures the manager and the GPU, not a disk).  Prints one JSON line.

    python tools/convert_bench.py --blocks 256
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from garage_b200 import block_manager as BM  # noqa: E402

N_NODES = 14


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def write_replicas(d, h, b, rf):
    for i in range(rf):
        node = (h[0] % N_NODES + i) % N_NODES
        sub = os.path.join(d, "node%d" % node, h[:1].hex(), h[1:2].hex())
        os.makedirs(sub, exist_ok=True)
        with open(os.path.join(sub, h.hex()), "wb") as f:
            f.write(b.tobytes())


def run(source, nblocks, block_len, base):
    rng = np.random.default_rng(7)
    blocks = [rng.integers(0, 256, block_len, dtype=np.uint8) for _ in range(nblocks)]
    hashes = [BM.blake2sum(b) for b in blocks]
    d = tempfile.mkdtemp(prefix="convert_bench_", dir=base)
    try:
        if source == "rs63":
            with BM.BlockManager(6, 3, n_nodes=N_NODES, data_dir=d) as old:
                for h, b in zip(hashes, blocks):
                    assert old.rpc_put_block(h, b) == BM.OK
            kw, read_alg = {"previous_codes": [(6, 3, 0, 0)]}, 6 * -(-block_len // 6)
        elif source == "clay104":
            with BM.BlockManager(10, 4, n_nodes=N_NODES, data_dir=d, clay=True) as old:
                for h, b in zip(hashes, blocks):
                    assert old.rpc_put_block(h, b) == BM.OK
            L = -(-(-(-block_len // 10)) // 4096) * 4096  # rounded up to 16 * alpha
            kw, read_alg = {"previous_codes": [(10, 4, 0, 0, 1)]}, 10 * L
        else:
            for h, b in zip(hashes, blocks):
                write_replicas(d, h, b, 3)
            kw, read_alg = {"legacy_replicas": 3}, block_len
        with BM.BlockManager(10, 4, n_nodes=N_NODES, data_dir=d, **kw) as bm:
            t0 = time.perf_counter()
            converted = bm.convert_all()
            el = time.perf_counter() - t0
            mt = bm.metrics()
            for i in range(0, nblocks, max(1, nblocks // 16)):  # spot-check the result
                rc, got = bm.rpc_get_block(hashes[i])
                assert rc == BM.OK and np.array_equal(got, blocks[i])
        assert converted == nblocks and mt["convert_errors"] == 0, (converted, mt["convert_errors"])
        return {
            "source": source, "blocks": nblocks, "block_len": block_len, "sweep_s": round(el, 4),
            "gib_per_s": round(nblocks * block_len / el / (1 << 30), 3),
            "transcode_share": round(mt["convert_call_us"] / 1e6 / el, 3),
            "read_per_block": mt["convert_bytes_read"] / nblocks, "read_algorithmic": read_alg,
            "written_per_block": mt["convert_bytes_written"] / nblocks, "written_algorithmic": 14 * -(-block_len // 10),
        }
    finally:
        shutil.rmtree(d, ignore_errors=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=256)
    ap.add_argument("--block-len", type=int, default=1 << 20)
    ap.add_argument("--sources", default="rs63,rep3,clay104")
    a = ap.parse_args()
    base = "/dev/shm" if os.path.isdir("/dev/shm") and os.access("/dev/shm", os.W_OK) else None
    res = [run(s, a.blocks, a.block_len, base) for s in a.sources.split(",")]
    print(json.dumps({"card": card(), "store": base or tempfile.gettempdir(), "runs": res}))


if __name__ == "__main__":
    main()
