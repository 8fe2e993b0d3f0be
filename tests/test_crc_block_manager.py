"""S3 CRC32 / CRC32C checksums through the block manager's SSE-C writes (DESIGN.md 2.9, 5.12): a multipart object of
uneven blocks sealed under CRC32C folds, block by block with garage_ec_crc_combine, to the CRC of its whole plaintext;
its key rotation, re-chunked so that new blocks straddle old ones, folds to the same value; and so does the same copy
with a source shard lost and with a stale source shard, the path that falls back to rpc_get_block and retries on the
GPU.  Expected values come from zlib and the bitwise C oracle (tests/crc_oracle.py)."""
import os
import sys
import zlib

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import crc_oracle as CO  # noqa: E402
import oracle_lib as O  # noqa: E402

import garage_b200 as G  # noqa: E402
from garage_b200 import block_manager as BM  # noqa: E402

pytestmark = pytest.mark.gpu
# multipart parts cut into blocks: full blocks, then each part's short tail
PART_BLOCKS = [1 << 20, 1 << 20, 300001, 1 << 20, 4097, 77777, 1]


def manager(d):
    return BM.BlockManager(k=10, m=4, n_nodes=14, data_dir=str(d), batch_max_blocks=8)


def key_of(i):
    return bytes((13 * i + 5 * j + 3) & 0xFF for j in range(32))


def fold(kind, crcs, lens):
    acc = 0
    for c, n in zip(crcs, lens):
        acc = G.crc_combine(kind, acc, c, n)
    return acc


def seal_object(bm, key, plain, kind):
    """the object's blocks PUT with their checksums: [(hash, offset, len)], per-block CRCs"""
    blocks, crcs, off = [], [], 0
    for n in PART_BLOCKS:
        rc, h, c = bm.rpc_put_block_sealed_crc(key, plain[off:off + n], kind)
        assert rc == BM.OK
        assert c == CO.crc(kind, plain[off:off + n])
        blocks.append((h, off, n))
        crcs.append(c)
        off += n
    return blocks, crcs


def rechunk(blocks, size):
    """destinations of `size` plaintext bytes (the last one shorter), as piece lists over the source blocks"""
    total = sum(n for _, _, n in blocks)
    dests = []
    for d0 in range(0, total, size):
        d1, pieces = min(total, d0 + size), []
        for h, o, n in blocks:
            a, b = max(d0, o), min(d1, o + n)
            if a < b:
                pieces.append((h, a - o, b - a))
        dests.append((pieces, d1 - d0))
    return dests


def rotate(bm, dests, old, new, kind):
    crcs, lens = [], []
    for pieces, n in dests:
        rc, h, stored, c = bm.put_block_resealed_crc(pieces, old, new, kind)
        assert rc == BM.OK, rc
        assert stored == G.sealed_len(n)
        crcs.append(c)
        lens.append(n)
    return crcs, lens


def test_multipart_object_and_rechunked_key_rotation(tmp_path):
    with manager(tmp_path) as bm:
        old, new = key_of(0), key_of(1)
        plain = O.fill_random(sum(PART_BLOCKS), 0xC4C0)
        want = CO.crc(CO.CRC32C, plain)
        blocks, crcs = seal_object(bm, old, plain, CO.CRC32C)
        assert fold(CO.CRC32C, crcs, PART_BLOCKS) == want
        # every block's plaintext still opens under its key: the checksum changed nothing that is stored
        rc, got = bm.rpc_get_block_opened(blocks[2][0], old)
        assert rc == BM.OK and np.array_equal(got, plain[blocks[2][1]:blocks[2][1] + blocks[2][2]])
        # re-chunked so that destinations straddle source blocks
        dests = rechunk(blocks, 700000)
        assert any(len(p) > 1 for p, _ in dests)
        rcrcs, lens = rotate(bm, dests, old, new, CO.CRC32C)
        assert fold(CO.CRC32C, rcrcs, lens) == want
        # the same copy under CRC32 (a change of algorithm: Calculate) folds to zlib's value
        rcrcs, lens = rotate(bm, dests, old, new, CO.CRC32)
        assert fold(CO.CRC32, rcrcs, lens) == zlib.crc32(plain.tobytes())
        # no checksum asked: 0, and the copy is stored as before
        rc, h, stored, c = bm.put_block_resealed_crc(dests[0][0], old, new, BM.CRC_NONE)
        assert rc == BM.OK and c == 0
        m = bm.reseal_metrics()
        assert m["fallbacks"] == 0 and m["auth_failures"] == 0
        # unknown kinds are refused
        rc, _, _ = bm.rpc_put_block_sealed_crc(old, plain[:10], 3)
        assert rc == G.E_INVALID
        rc, _, _, _ = bm.put_block_resealed_crc(dests[0][0], old, new, 3)
        assert rc == G.E_INVALID


def test_rotation_with_a_lost_shard_and_a_stale_shard(tmp_path):
    with manager(tmp_path) as bm:
        old, new = key_of(2), key_of(3)
        plain = O.fill_random(sum(PART_BLOCKS), 0xC4C1)
        want = CO.crc(CO.CRC32C, plain)
        blocks, crcs = seal_object(bm, old, plain, CO.CRC32C)
        dests = rechunk(blocks, 900001)
        # a holder of the first source loses its shard: rebuilt on the GPU, no fallback
        row = bm.storage_nodes_of(blocks[0][0])
        assert bm.drop_shard(row[0], blocks[0][0]) == BM.OK
        rcrcs, lens = rotate(bm, dests, old, new, CO.CRC32C)
        assert fold(CO.CRC32C, rcrcs, lens) == want
        assert bm.reseal_metrics()["fallbacks"] == 0
        # a stale but self-consistent shard of the second source: read through rpc_get_block, then the GPU retry
        # seals the copy and computes its checksum
        row = bm.storage_nodes_of(blocks[1][0])
        assert bm.plant_stale_shard(row[3], blocks[1][0]) == BM.OK
        rcrcs, lens = rotate(bm, dests, old, new, CO.CRC32C)
        assert bm.reseal_metrics()["fallbacks"] >= 1
        assert fold(CO.CRC32C, rcrcs, lens) == want
