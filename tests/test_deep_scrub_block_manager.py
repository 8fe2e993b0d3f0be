"""garage_bm_deep_scrub_step on RS(10,4), LRC(10,2,2), PB(10,4) and Clay(10,4) stores: a clean sweep checks every
block once; a stale parity shard (valid tag, wrong bytes), which the per-shard scrub and GET never see, is quarantined
and rebuilt before it can poison a degraded read (with the control that fails without the deep scrub); a stale data
shard goes through the hunt; a whole wrong stripe is a content error that touches no file; the owner moves off a down
node; a missing shard skips its block and queues its resync; the cursor; a restarted file store; the metrics."""
import os
import shutil
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import oracle_lib as O  # noqa: E402

from garage_b200 import block_manager as BM  # noqa: E402

N = 14
CODES = {"rs": {}, "lrc": {"local_groups": 2}, "pb": {"piggyback": True}, "clay": {"clay": True}}
# data holders taken down after the stale parity: 4 losses each code decodes with every parity good
DOWN = {"rs": (0, 1, 2, 3), "lrc": (0, 1, 5, 6), "pb": (0, 1, 2, 3), "clay": (0, 1, 2, 3)}
STALE_PARITY = {"rs": 10, "lrc": 12, "pb": 10, "clay": 11}


def manager(code, **kw):
    kw.setdefault("batch_max_blocks", 8)
    return BM.BlockManager(k=10, m=4, n_nodes=kw.pop("n_nodes", N), **CODES[code], **kw)


def put_blocks(bm, lens, seed):
    blocks = [O.fill_random(n, seed + i) for i, n in enumerate(lens)]
    hashes = [BM.blake2sum(b) for b in blocks]
    for h, b in zip(hashes, blocks):
        assert bm.rpc_put_block(h, b) == BM.OK
    return blocks, hashes


def sweep(bm):
    """one full deep scrub over the up nodes -> (checked, repaired)"""
    checked = repaired = 0
    for node in range(bm.n_nodes):
        if node in bm._down:
            assert bm.deep_scrub_step(node)[0] == BM.E_MESSAGE
            continue
        rc, _, finished, c, r = bm.deep_scrub_step(node)
        assert rc == BM.OK and finished
        checked += c
        repaired += r
    return checked, repaired


def delta(m0, m1, key):
    return m1[key] - m0[key]


@pytest.mark.gpu
@pytest.mark.parametrize("code", list(CODES))
def test_clean_store_every_block_once(code):
    with manager(code) as bm:
        blocks, hashes = put_blocks(bm, [1 << 20, 777777, 65536, 4097, 129, 31, 1] * 2, 0xD500)
        m0 = bm.metrics()
        assert sweep(bm) == (len(blocks), 0)
        m1 = bm.metrics()
        assert delta(m0, m1, "deep_scrub_blocks") == len(blocks)
        for key in ("deep_scrub_skipped", "deep_scrub_parity_bad", "deep_scrub_content_errors", "corruption_counter"):
            assert delta(m0, m1, key) == 0, key
        assert m1["deep_check_call_us"] > m0["deep_check_call_us"]


def _stale_parity_setup(bm, code):
    blocks, hashes = put_blocks(bm, [1 << 20, 300001], 0xD600)
    h, b = hashes[0], blocks[0]
    row = bm.storage_nodes_of(h)
    p = STALE_PARITY[code]
    assert bm.plant_stale_shard(row[p], h) == BM.OK
    for node in range(N):  # the per-shard scrub accepts the stale parity's tag
        rc, _, corrupt = bm.scrub(node)
        assert rc == BM.OK and corrupt == 0
    rc, got = bm.rpc_get_block(h)
    assert rc == BM.OK and np.array_equal(got, b)
    return h, b, row, p


def _take_down(bm, row, code):
    for i in DOWN[code]:
        bm.set_node_up(row[i], False)


@pytest.mark.gpu
@pytest.mark.parametrize("code", list(CODES))
def test_stale_parity_is_quarantined_and_rebuilt(code):
    with manager(code) as bm:
        h, b, row, p = _stale_parity_setup(bm, code)
        m0 = bm.metrics()
        assert sweep(bm) == (2, 1)
        m1 = bm.metrics()
        assert delta(m0, m1, "deep_scrub_parity_bad") == 1 and delta(m0, m1, "deep_scrub_content_errors") == 0
        assert delta(m0, m1, "corruption_counter") == 1
        assert bm.node_shard_index(row[p], h) < 0  # quarantined
        failed, done = bm.resync_all(row[p])
        assert failed == 0 and done >= 1
        assert bm.node_shard_index(row[p], h) == p
        assert sweep(bm) == (2, 0)
        _take_down(bm, row, code)
        rc, got = bm.rpc_get_block(h)
        assert rc == BM.OK and np.array_equal(got, b)


@pytest.mark.gpu
@pytest.mark.parametrize("code", list(CODES))
def test_without_deep_scrub_the_stale_parity_loses_the_block(code):
    with manager(code) as bm:
        h, b, row, p = _stale_parity_setup(bm, code)
        _take_down(bm, row, code)
        rc, _ = bm.rpc_get_block(h)
        assert rc == BM.E_CORRUPT_DATA


@pytest.mark.gpu
@pytest.mark.parametrize("code", list(CODES))
def test_stale_data_shard_goes_through_the_hunt(code):
    with manager(code) as bm:
        blocks, hashes = put_blocks(bm, [1 << 20, 54321], 0xD700)
        h, b = hashes[1], blocks[1]
        row = bm.storage_nodes_of(h)
        assert bm.plant_stale_shard(row[3], h) == BM.OK
        m0 = bm.metrics()
        assert sweep(bm) == (2, 1)
        m1 = bm.metrics()
        assert delta(m0, m1, "deep_scrub_content_errors") == 0 and delta(m0, m1, "deep_scrub_parity_bad") == 0
        assert bm.node_shard_index(row[3], h) < 0
        assert bm.resync_all(row[3])[0] == 0
        rc, got = bm.rpc_get_block(h)
        assert rc == BM.OK and np.array_equal(got, b)
        assert sweep(bm) == (2, 0)


def _shard_path(d, node, h):
    return os.path.join(d, "node%d" % node, h[:1].hex(), h[1:2].hex(), h.hex() + ".shard")


@pytest.mark.gpu
def test_whole_wrong_stripe_is_a_content_error_and_touches_nothing(tmp_path):
    d = str(tmp_path / "store")
    with manager("rs", data_dir=d) as bm:
        blocks, hashes = put_blocks(bm, [400000, 400000], 0xD800)
        a, b = hashes
        ra, rb = bm.storage_nodes_of(a), bm.storage_nodes_of(b)
        for i in range(14):
            shutil.copyfile(_shard_path(d, rb[i], b), _shard_path(d, ra[i], a))
        before = {i: open(_shard_path(d, ra[i], a), "rb").read() for i in range(14)}
        m0 = bm.metrics()
        assert sweep(bm) == (2, 0)
        m1 = bm.metrics()
        assert delta(m0, m1, "deep_scrub_content_errors") == 1 and delta(m0, m1, "corruption_counter") == 0
        for i in range(14):
            assert open(_shard_path(d, ra[i], a), "rb").read() == before[i]
            assert os.path.exists(_shard_path(d, rb[i], b))
        rc, got = bm.rpc_get_block(b)
        assert rc == BM.OK and np.array_equal(got, blocks[1])


@pytest.mark.gpu
def test_owner_moves_off_a_down_node():
    with manager("rs", n_nodes=16) as bm:
        blocks, hashes = put_blocks(bm, [20000 + 7 * i for i in range(40)], 0xD900)
        rows = [bm.storage_nodes_of(h) for h in hashes]
        down = rows[0][0]
        bm.set_node_up(down, False)
        m0 = bm.metrics()
        checked, repaired = sweep(bm)
        m1 = bm.metrics()
        whole = sum(down not in r for r in rows)
        assert 0 < whole < len(hashes)
        assert (checked, repaired) == (whole, 0)
        assert delta(m0, m1, "deep_scrub_skipped") == len(hashes) - whole  # every block visited once
        # the blocks whose first holder is down were visited by the next holder of their row
        moved = [r for r in rows if r[0] == down]
        assert moved
        for r in moved:
            rc, _, _, c, _ = bm.deep_scrub_step(r[0])
            assert rc == BM.E_MESSAGE


@pytest.mark.gpu
def test_missing_shard_skips_and_queues_its_resync():
    with manager("pb") as bm:
        blocks, hashes = put_blocks(bm, [1 << 20, 9999], 0xDA00)
        h = hashes[0]
        node = bm.storage_nodes_of(h)[5]
        assert bm.drop_shard(node, h) == BM.OK
        m0 = bm.metrics()
        assert sweep(bm) == (1, 0)
        m1 = bm.metrics()
        assert delta(m0, m1, "deep_scrub_skipped") == 1
        assert m1["resync_queue_length"] >= 1
        failed, done = bm.resync_all(node)
        assert failed == 0 and done >= 1
        assert sweep(bm) == (2, 0)


@pytest.mark.gpu
def test_cursor_steps_visit_every_block_once_in_hash_order():
    with manager("clay") as bm:
        blocks, hashes = put_blocks(bm, [3000 + i for i in range(30)], 0xDB00)
        owned = {}
        for h in hashes:
            owned.setdefault(bm.storage_nodes_of(h)[0], []).append(h)
        total = 0
        for node in range(N):
            mine = sorted(owned.get(node, []))
            cursor, seen = None, 0
            while True:
                rc, cur, finished, c, r = bm.deep_scrub_step(node, cursor, 3)
                assert rc == BM.OK and r == 0
                assert c == min(3, len(mine) - seen)
                seen += c
                if c:
                    assert cur == mine[seen - 1]
                cursor = cur
                if finished:
                    break
            assert seen == len(mine)
            total += seen
        assert total == len(hashes)


@pytest.mark.gpu
@pytest.mark.parametrize("code", ["rs", "lrc", "pb"])
def test_file_store_after_restart(tmp_path, code):
    d = str(tmp_path / "store")
    with manager(code, data_dir=d) as bm:
        blocks, hashes = put_blocks(bm, [1 << 20, 250000, 77], 0xDC00)
    with manager(code, data_dir=d) as bm:
        assert sweep(bm) == (3, 0)
        h = hashes[1]
        row = bm.storage_nodes_of(h)
        assert bm.plant_stale_shard(row[13], h) == BM.OK
        assert sweep(bm) == (3, 1)
        assert bm.resync_all(row[13])[0] == 0
        assert sweep(bm) == (3, 0)
        for h, b in zip(hashes, blocks):
            rc, got = bm.rpc_get_block(h)
            assert rc == BM.OK and np.array_equal(got, b)
