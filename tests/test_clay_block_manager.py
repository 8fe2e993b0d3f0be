"""The block manager on a Clay(10,4) cluster: PUT/GET identity (short blocks too), resync of a wiped node handing the
rebuild 1/4 of each of the 13 other shards (13 x 26 624 bytes for a 1 MiB block, whatever index was lost), GET with
any 4 nodes down, a corrupt helper quarantined with a correct fallback rebuild, the file store's header and restart,
an RS(10,4) -> Clay(10,4) conversion stopped at every file operation, and the refused configurations."""
import os
import random
import shutil
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import clay_oracle as CO  # noqa: E402
import oracle_lib as O  # noqa: E402

from garage_b200 import block_manager as BM  # noqa: E402

E_INVALID = -1
N = 14


def _put_blocks(bm, lens, seed):
    blocks = [O.fill_random(n, seed + i) for i, n in enumerate(lens)]
    hashes = [BM.blake2sum(b) for b in blocks]
    for h, b in zip(hashes, blocks):
        assert bm.rpc_put_block(h, b) == 0
    return blocks, hashes


def _shard_path(d, node, h):
    return os.path.join(d, "node%d" % node, h[:1].hex(), h[1:2].hex(), h.hex() + ".shard")


def _assert_clay_stripe(d, bm, h, b):
    """every shard file holds the oracle's Clay(10,4) encoding of the block, with pad[1] = 2"""
    L = CO.shard_len(b.size, 10, 4)
    flat = np.zeros(10 * L, dtype=np.uint8)
    flat[:b.size] = b
    data = flat.reshape(10, L)
    full = np.concatenate([data, CO.encode(10, 4, CO.build(10, 4), data)])
    for i, node in enumerate(bm.storage_nodes_of(h)):
        raw = open(_shard_path(d, node, h), "rb").read()
        assert raw[:4] == b"GEC1" and raw[6] == i and raw[53] == 2, (i, node)
        assert raw[64:] == full[i].tobytes(), i


@pytest.mark.gpu
def test_put_get_identity_with_short_blocks():
    with BM.BlockManager(k=10, m=4, n_nodes=N, clay=True) as bm:
        blocks, hashes = _put_blocks(bm, [1 << 20, 777777, 65536, 16384, 31, 1], 0xC100)
        for h, b in zip(hashes, blocks):
            rc, got = bm.rpc_get_block(h)
            assert rc == 0 and np.array_equal(got, b)


@pytest.mark.gpu
def test_wiped_node_is_rebuilt_from_a_quarter_of_each_helper(tmp_path):
    d = str(tmp_path / "store")
    with BM.BlockManager(k=10, m=4, n_nodes=N, clay=True, data_dir=d) as bm:
        blocks, hashes = _put_blocks(bm, [1 << 20] * 14 + [300001], 0xC200)
        seen = set()
        for h, b in zip(hashes, blocks):  # every index, one block each
            idx = len(seen) % 14
            seen.add(idx)
            node = bm.storage_nodes_of(h)[idx]
            assert bm.drop_shard(node, h) == 0
            m0 = bm.metrics()
            assert bm.resync_block(node, h) == 0
            m1 = bm.metrics()
            fetched = m1["resync_bytes_fetched"] - m0["resync_bytes_fetched"]
            L = CO.shard_len(b.size, 10, 4)
            assert fetched == 13 * L // 4, (idx, b.size)
            if b.size == 1 << 20:
                assert fetched == 13 * 26624
            assert m1["resync_bytes_read"] - m0["resync_bytes_read"] == 13 * L  # holders read whole shards for the tag
            assert bm.node_shard_index(node, h) == idx
            rc, got = bm.rpc_get_block(h)
            assert rc == 0 and np.array_equal(got, b)
        assert len(seen) == 14
        for h, b in zip(hashes, blocks):
            _assert_clay_stripe(d, bm, h, b)
        # a whole node wiped: resync_all rebuilds every shard it held
        shutil.rmtree(os.path.join(d, "node5"))
        os.makedirs(os.path.join(d, "node5"))
        m0 = bm.metrics()
        bm.repair_enqueue_missing(5)
        failed, done = bm.resync_all(5)
        assert failed == 0 and done == len(blocks)
        m1 = bm.metrics()
        assert m1["resync_bytes_fetched"] - m0["resync_bytes_fetched"] == sum(
            13 * CO.shard_len(b.size, 10, 4) // 4 for b in blocks)
        for h, b in zip(hashes, blocks):
            _assert_clay_stripe(d, bm, h, b)


@pytest.mark.gpu
def test_get_with_any_four_nodes_down():
    with BM.BlockManager(k=10, m=4, n_nodes=N, clay=True) as bm:
        blocks, hashes = _put_blocks(bm, [1 << 20, 123457], 0xC300)
        import itertools

        sets = list(itertools.combinations(range(N), 4))
        random.Random(12).shuffle(sets)
        for down in sets[:40] + [(0, 1, 2, 3), (10, 11, 12, 13), (3, 7, 10, 11)]:
            for nd in down:
                bm.set_node_up(nd, False)
            for h, b in zip(hashes, blocks):
                rc, got = bm.rpc_get_block(h)
                assert rc == 0 and np.array_equal(got, b), down
            for nd in down:
                bm.set_node_up(nd, True)


@pytest.mark.gpu
def test_corrupt_helper_is_quarantined_and_the_rebuild_falls_back(tmp_path):
    d = str(tmp_path / "store")
    with BM.BlockManager(k=10, m=4, n_nodes=N, clay=True, data_dir=d) as bm:
        blocks, hashes = _put_blocks(bm, [1 << 20], 0xC400)
        h, b = hashes[0], blocks[0]
        nodes = bm.storage_nodes_of(h)
        path = _shard_path(d, nodes[12], h)
        raw = bytearray(open(path, "rb").read())
        raw[64 + 5000] ^= 0x40
        open(path, "wb").write(bytes(raw))
        assert bm.drop_shard(nodes[3], h) == 0
        c0 = bm.metrics()["corruption_counter"]
        m0 = bm.metrics()
        assert bm.resync_block(nodes[3], h) == 0
        m1 = bm.metrics()
        assert m1["corruption_counter"] == c0 + 1
        L = CO.shard_len(b.size, 10, 4)
        assert m1["resync_bytes_fetched"] - m0["resync_bytes_fetched"] == 10 * L  # k whole shards
        assert bm.node_shard_index(nodes[3], h) == 3
        rc, got = bm.rpc_get_block(h)
        assert rc == 0 and np.array_equal(got, b)
        bm.repair_enqueue_missing(nodes[12])
        assert bm.resync_all(nodes[12])[0] == 0
        _assert_clay_stripe(d, bm, h, b)


@pytest.mark.gpu
def test_file_store_restart_and_quarantine_by_another_code(tmp_path):
    d = str(tmp_path / "store")
    with BM.BlockManager(k=10, m=4, n_nodes=N, clay=True, data_dir=d) as bm:
        blocks, hashes = _put_blocks(bm, [1 << 20, 4097], 0xC500)
        for h, b in zip(hashes, blocks):
            _assert_clay_stripe(d, bm, h, b)
    with BM.BlockManager(k=10, m=4, n_nodes=N, clay=True, data_dir=d) as bm:  # restart
        for h, b in zip(hashes, blocks):
            rc, got = bm.rpc_get_block(h)
            assert rc == 0 and np.array_equal(got, b)
    with BM.BlockManager(k=10, m=4, n_nodes=N, data_dir=d) as rs:  # an RS(10,4) manager accepts none of them
        rc, _ = rs.rpc_get_block(hashes[0])
        assert rc == BM.E_MISSING_BLOCK
        assert rs.metrics()["corruption_counter"] >= 10
    with BM.BlockManager(k=10, m=4, n_nodes=N, data_dir=str(tmp_path / "rs")) as rs:
        rblocks, rhashes = _put_blocks(rs, [1 << 20], 0xC600)
    with BM.BlockManager(k=10, m=4, n_nodes=N, clay=True, data_dir=str(tmp_path / "rs")) as bm:
        rc, _ = bm.rpc_get_block(rhashes[0])
        assert rc == BM.E_MISSING_BLOCK


@pytest.mark.gpu
def test_apply_layout_is_refused_on_a_clay_store(tmp_path):
    with BM.BlockManager(k=10, m=4, n_nodes=N, clay=True, data_dir=str(tmp_path / "s")) as bm:
        rc, _ = bm.apply_layout([0] * 14, [1] * 14)
        assert rc == E_INVALID


@pytest.mark.gpu
def test_rs_to_clay_conversion_stopped_at_every_step(tmp_path):
    blocks = [O.fill_random(n, 0xC700 + i) for i, n in enumerate([1 << 20, 5])]
    hashes = [BM.blake2sum(b) for b in blocks]
    pristine = str(tmp_path / "pristine")
    with BM.BlockManager(k=10, m=4, n_nodes=N, data_dir=pristine) as rs:
        for h, b in zip(hashes, blocks):
            assert rs.rpc_put_block(h, b) == 0
    prev = [(10, 4, 0, 0)]
    n, finished = 0, False
    while not finished:
        d = str(tmp_path / ("run%d" % n))
        shutil.copytree(pristine, d)
        with BM.BlockManager(k=10, m=4, n_nodes=N, clay=True, data_dir=d, previous_codes=prev) as bm:
            bm.debug_convert_stop_after(n)
            bm.convert_all()
            mt = bm.metrics()
            finished = mt["convert_blocks"] == 2 and mt["legacy_deleted"] == 28
        with BM.BlockManager(k=10, m=4, n_nodes=N, clay=True, data_dir=d, previous_codes=prev) as bm:
            for h, b in zip(hashes, blocks):
                rc, got = bm.rpc_get_block(h)
                assert rc == 0 and np.array_equal(got, b), n
            assert bm.metrics()["corruption_counter"] == 0
            bm.convert_all()
            assert bm.metrics()["convert_errors"] == 0
            for node in range(N):
                bm.repair_enqueue_missing(node)
                assert bm.resync_all(node)[0] == 0
            for h, b in zip(hashes, blocks):
                _assert_clay_stripe(d, bm, h, b)
        with BM.BlockManager(k=10, m=4, n_nodes=N, clay=True, data_dir=d) as bm:
            for h, b in zip(hashes, blocks):
                rc, got = bm.rpc_get_block(h)
                assert rc == 0 and np.array_equal(got, b), n
        shutil.rmtree(d)
        n += 1
    assert n > 2 * 14


@pytest.mark.parametrize("kw", [
    {"m": 5, "n_nodes": 15},                                  # m > 4
    {"k": 14, "m": 4, "n_nodes": 18},                         # alpha = 1024
    {"k": 10, "m": 4, "local_groups": 2},                     # with LRC
    {"k": 10, "m": 4, "piggyback": True},                     # with PB
    {"k": 10, "m": 4, "layout": {"zone": [0] * 14, "capacity": [1] * 14}},  # with a layout
])
def test_bad_clay_configs_are_rejected_before_any_cuda_call(kw):
    args = dict(k=10, m=4, n_nodes=N, clay=True)
    args.update(kw)
    with pytest.raises(BM.BlockManagerError) as e:
        BM.BlockManager(**args)
    assert e.value.code == E_INVALID
