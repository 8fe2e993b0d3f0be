"""The block manager on an LRC(10,2,2) cluster: resync of one lost shard reads only its local group (5 shards,
against 10 on RS(10,4)), PUT/GET identity with any 3 nodes down, the shard file header and the wire message
record the code, and a shard of another code is quarantined."""
import itertools
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import oracle_lib as O  # noqa: E402

from garage_b200 import block_manager as BM  # noqa: E402


def test_wire_carries_l_only_for_lrc():
    H, S = bytes(range(32)), bytes(range(32, 64))
    rs = BM.wire_encode(H, 0, 10, 4, 3, 1000, 100, 1, S)
    assert b"\xa1l" not in rs[8:] and BM.wire_decode(rs)["k"] == 10 and "l" not in BM.wire_decode(rs)
    lrc = BM.wire_encode(H, 0, 10, 4, 3, 1000, 100, 1, S, l=2)
    assert lrc[8] == 0x8A and lrc.endswith(b"\xa1l\x02")
    d = BM.wire_decode(lrc)
    assert d["l"] == 2 and d["m"] == 4 and d["index"] == 3
    assert BM.wire_encode(H, 0, 10, 4, 3, 1000, 100, 1, S, l=3) == b""  # k % l != 0
    assert BM.wire_encode(H, 0, 10, 4, 3, 1000, 100, 1, S, l=4) == b""  # no global parity left


def test_bad_local_groups_rejected():
    for l in (-1, 3, 4):
        with pytest.raises(BM.BlockManagerError):
            BM.BlockManager(k=10, m=4, local_groups=l)


def _put_blocks(bm, n, seed):
    blocks = [O.fill_random((1 << 20) - 977 * i, seed + i) for i in range(n)]
    hashes = [BM.blake2sum(b) for b in blocks]
    for h, b in zip(hashes, blocks):
        assert bm.rpc_put_block(h, b) == 0
    return blocks, hashes


@pytest.mark.gpu
@pytest.mark.parametrize("local_groups,reads", [(2, 5), (0, 10)])
def test_resync_of_one_shard_reads_its_group(local_groups, reads):
    with BM.BlockManager(k=10, m=4, n_nodes=14, local_groups=local_groups) as bm:
        blocks, hashes = _put_blocks(bm, 3, 0x8C0)
        for h, b in zip(hashes, blocks):
            node = bm.storage_nodes_of(h)[3]  # the node holding data shard 3
            assert bm.drop_shard(node, h) == 0
            before = bm.metrics()["resync_shards_read"]
            assert bm.resync_block(node, h) == 0
            assert bm.metrics()["resync_shards_read"] - before == reads
            assert bm.node_shard_index(node, h) == 3
            rc, got = bm.rpc_get_block(h)
            assert rc == 0 and np.array_equal(got, b)


@pytest.mark.gpu
def test_put_get_identity_with_any_three_nodes_down():
    with BM.BlockManager(k=10, m=4, n_nodes=14, local_groups=2) as bm:
        blocks, hashes = _put_blocks(bm, 2, 0x9C0)
        for down in itertools.combinations(range(14), 3):
            for nd in down:
                bm.set_node_up(nd, False)
            for h, b in zip(hashes, blocks):
                rc, got = bm.rpc_get_block(h)
                assert rc == 0 and np.array_equal(got, b), down
            for nd in down:
                bm.set_node_up(nd, True)


@pytest.mark.gpu
def test_file_store_records_the_code_and_quarantines_another(tmp_path):
    d = str(tmp_path / "store")
    with BM.BlockManager(k=10, m=4, n_nodes=14, local_groups=2, data_dir=d) as bm:
        blocks, hashes = _put_blocks(bm, 1, 0xAC0)
        h = hashes[0]
        node = bm.storage_nodes_of(h)[7]
        path = os.path.join(d, "node%d" % node, h[:1].hex(), h[1:2].hex(), h.hex() + ".shard")
        raw = bytearray(open(path, "rb").read())
        assert raw[:4] == b"GEC1" and raw[52] == 2  # ShardFileHeader.pad[0]
        rc, got = bm.rpc_get_block(h)
        assert rc == 0 and np.array_equal(got, blocks[0])
    # the same files read by an RS(10,4) manager: every shard says LRC, so none is accepted
    with BM.BlockManager(k=10, m=4, n_nodes=14, data_dir=d) as rs:
        rc, _ = rs.rpc_get_block(h)
        assert rc == BM.E_MISSING_BLOCK
        assert rs.metrics()["corruption_counter"] >= 10
