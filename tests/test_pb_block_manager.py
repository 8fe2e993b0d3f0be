"""The block manager on a PB(10,4) cluster: resync of one lost data shard fetches only the planned halves (14 halves,
734 720 bytes for a 1 MiB block, against 10 whole shards on RS(10,4)), re-plans when a planned half turns out bad,
reads back every block with any 4 of its nodes down (MDS), and records the code in the shard file header so that a
shard of another code is quarantined."""
import os
import random
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import oracle_lib as O  # noqa: E402
import pb_oracle as PB  # noqa: E402

from garage_b200 import block_manager as BM  # noqa: E402

pytestmark = pytest.mark.gpu


def _put_blocks(bm, lens, seed):
    blocks = [O.fill_random(n, seed + i) for i, n in enumerate(lens)]
    hashes = [BM.blake2sum(b) for b in blocks]
    for h, b in zip(hashes, blocks):
        assert bm.rpc_put_block(h, b) == 0
    return blocks, hashes


@pytest.mark.parametrize("piggyback", [True, False])
def test_resync_of_one_data_shard_reads_the_planned_halves(piggyback):
    lens = [1 << 20, (1 << 20) - 977, 300001]
    with BM.BlockManager(k=10, m=4, n_nodes=14, piggyback=piggyback) as bm:
        blocks, hashes = _put_blocks(bm, lens, 0x8E0)
        for h, b in zip(hashes, blocks):
            for idx, halves in ((3, 14), (7, 13)):
                node = bm.storage_nodes_of(h)[idx]
                assert bm.drop_shard(node, h) == 0
                m0 = bm.metrics()
                assert bm.resync_block(node, h) == 0
                m1 = bm.metrics()
                shards = m1["resync_shards_read"] - m0["resync_shards_read"]
                nbytes = m1["resync_bytes_read"] - m0["resync_bytes_read"]
                if piggyback:
                    L = PB.shard_len(b.size, 10)
                    assert (shards, nbytes) == (11, halves * L // 2), (idx, b.size)
                    if b.size == 1 << 20 and idx == 3:
                        assert nbytes == 734720
                else:
                    assert (shards, nbytes) == (10, 10 * -(-b.size // 10))
                assert bm.node_shard_index(node, h) == idx
                rc, got = bm.rpc_get_block(h)
                assert rc == 0 and np.array_equal(got, b)


def test_resync_replans_when_a_planned_half_is_bad(tmp_path):
    d = str(tmp_path / "store")
    with BM.BlockManager(k=10, m=4, n_nodes=14, piggyback=True, data_dir=d) as bm:
        blocks, hashes = _put_blocks(bm, [1 << 20], 0x9E0)
        h, b = hashes[0], blocks[0]
        nodes = bm.storage_nodes_of(h)
        L = PB.shard_len(b.size, 10)
        # flip a byte in the b-half of parity 1, which rule 1 reads for data shard 3
        path = os.path.join(d, "node%d" % nodes[11], h[:1].hex(), h[1:2].hex(), h.hex() + ".shard")
        raw = bytearray(open(path, "rb").read())
        assert raw[:4] == b"GEC1" and raw[52] == 0 and raw[53] == 1  # pad[0]: not LRC, pad[1]: PB
        raw[64 + L // 2 + 1000] ^= 0x40
        open(path, "wb").write(bytes(raw))
        assert bm.drop_shard(nodes[3], h) == 0
        c0 = bm.metrics()["corruption_counter"]
        assert bm.resync_block(nodes[3], h) == 0
        assert bm.metrics()["corruption_counter"] == c0 + 1  # parity 1 quarantined, the rest re-planned
        assert bm.node_shard_index(nodes[3], h) == 3
        rc, got = bm.rpc_get_block(h)
        assert rc == 0 and np.array_equal(got, b)


def test_get_with_any_four_nodes_down():
    """MDS: blocks PUT with every node up read back with any 4 of their 14 nodes down (a seeded sample of the 1001
    sets); PUT itself needs k+1 stored shards, so it is tested with 3 nodes down"""
    with BM.BlockManager(k=10, m=4, n_nodes=14, piggyback=True) as bm:
        blocks, hashes = _put_blocks(bm, [1 << 20, 123457], 0xAE0)
        import itertools

        sets = list(itertools.combinations(range(14), 4))
        random.Random(11).shuffle(sets)
        for down in sets[:80] + [(0, 1, 2, 3), (10, 11, 12, 13), (3, 7, 10, 11)]:
            for nd in down:
                bm.set_node_up(nd, False)
            for h, b in zip(hashes, blocks):
                rc, got = bm.rpc_get_block(h)
                assert rc == 0 and np.array_equal(got, b), down
            for nd in down:
                bm.set_node_up(nd, True)
        for nd in (2, 6, 12):
            bm.set_node_up(nd, False)
        b3, h3 = _put_blocks(bm, [777777], 0xBE0)
        rc, got = bm.rpc_get_block(h3[0])
        assert rc == 0 and np.array_equal(got, b3[0])


def test_file_store_records_the_code_and_quarantines_another(tmp_path):
    d = str(tmp_path / "store")
    with BM.BlockManager(k=10, m=4, n_nodes=14, piggyback=True, data_dir=d) as bm:
        blocks, hashes = _put_blocks(bm, [1 << 20], 0xCE0)
        h = hashes[0]
        rc, got = bm.rpc_get_block(h)
        assert rc == 0 and np.array_equal(got, blocks[0])
    # the same files read by an RS(10,4) manager: every shard says PB, so none is accepted
    with BM.BlockManager(k=10, m=4, n_nodes=14, data_dir=d) as rs:
        rc, _ = rs.rpc_get_block(h)
        assert rc == BM.E_MISSING_BLOCK
        assert rs.metrics()["corruption_counter"] >= 10
    # and the other way round: RS shards are not accepted by a PB manager
    d2 = str(tmp_path / "store_rs")
    with BM.BlockManager(k=10, m=4, n_nodes=14, data_dir=d2) as rs:
        blocks, hashes = _put_blocks(rs, [1 << 20], 0xDE0)
    with BM.BlockManager(k=10, m=4, n_nodes=14, piggyback=True, data_dir=d2) as bm:
        rc, _ = bm.rpc_get_block(hashes[0])
        assert rc == BM.E_MISSING_BLOCK
        assert bm.metrics()["corruption_counter"] >= 10
