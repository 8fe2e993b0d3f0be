"""GPU tests of a block manager whose nodes spread their shard files over several drives (DESIGN.md section 5.7):
placement by the drive layout, adding a drive and rebalancing, losing a drive and rebuilding its shards on the GPU
from the other nodes, read-only drives, scrub across drives, a rebalance stopped midway, code conversion of replicas
placed by the drive layout, and a single-directory store restarted with drives.  Where files should be comes from
the model of tests/test_drive_layout_cpu.py, written from the rules alone."""
import os
import shutil
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle_lib as O  # noqa: E402
from test_drive_layout_cpu import model_init, model_update, parse_image  # noqa: E402

from garage_b200 import block_manager as BM  # noqa: E402
from garage_b200 import placement as P  # noqa: E402

pytestmark = pytest.mark.gpu
N = 14
CODES = {
    "rs": {"k": 10, "m": 4},
    "clay": {"k": 10, "m": 4, "clay": True},
    "lrc": {"k": 10, "m": 4, "local_groups": 2},
}
CLAY_REPAIR_BYTES_1MIB = 346112  # Clay(10,4): the 1/m runs of the 13 helpers of one lost shard of a 1 MiB block


# ---------------------------------------------------------------- helpers
def manager(d, dirs, code="rs", **kw):
    kw.setdefault("batch_max_blocks", 8)
    return BM.BlockManager(n_nodes=N, data_dir=str(d), data_dirs=dirs, **CODES[code], **kw)


def make_blocks(n, seed, size=None):
    rng = np.random.default_rng(seed)
    sizes = [size or int(rng.integers(1, 1 << 20)) for _ in range(n)]
    blocks = [O.fill_random(s, seed * 1000 + i) for i, s in enumerate(sizes)]
    return blocks, [BM.blake2sum(b) for b in blocks]


def put_all(bm, blocks, hashes):
    for h, b in zip(hashes, blocks):
        assert bm.rpc_put_block(h, b) == BM.OK


def assert_gets(bm, blocks, hashes):
    for h, b in zip(hashes, blocks):
        rc, got = bm.rpc_get_block(h)
        assert rc == BM.OK and np.array_equal(got, b)


def root_of(d, node, drive):
    nd = os.path.join(str(d), "node%d" % node)
    return nd if drive == "." else os.path.join(nd, drive)


def file_path(d, node, drive, h, ext=".shard"):
    return os.path.join(root_of(d, node, drive), h[:1].hex(), h[1:2].hex(), h.hex() + ext)


def where(d, node, names, h, ext=".shard"):
    """the drives holding file `ext` of h on node"""
    return [n for n in names if os.path.exists(file_path(d, node, n, h, ext))]


def part(h):
    return P.drive_partition_of(h)


def persisted(d, node):
    """(capacities, primaries, secondaries) of the layout in node's data_layout file"""
    with open(os.path.join(str(d), "node%d" % node, "data_layout")) as f:
        words = f.read().split()
    return parse_image(bytes.fromhex(words[words.index("layout") + 1]))


def holders(bm, h):
    return bm.storage_nodes_of(h)


# ---------------------------------------------------------------- placement
def test_every_shard_lies_in_its_primary_drive(tmp_path):
    dirs = [("d0", 1), ("d1", 2), ("d2", 1)]
    names = [x[0] for x in dirs]
    model = model_init([1, 2, 1], [0, 0, 0])
    blocks, hashes = make_blocks(40, 1)
    with manager(tmp_path, dirs) as bm:
        put_all(bm, blocks, hashes)
        for h in hashes:
            for node in holders(bm, h):
                assert where(tmp_path, node, names, h) == [names[model[1][part(h)]]]
                assert not os.path.exists(file_path(tmp_path, node, ".", h))  # nothing in the old single directory
        assert_gets(bm, blocks, hashes)
        for node in range(N):
            assert persisted(tmp_path, node) == model
            for n in names:
                assert os.path.exists(os.path.join(root_of(tmp_path, node, n), "garage-marker"))


# ---------------------------------------------------------------- adding a drive, rebalance, restart
def test_add_drive_then_rebalance_moves_exactly_the_predicted_files(tmp_path):
    dirs = [("d0", 1), ("d1", 1), ("d2", 1)]
    new_dirs = dirs + [("d3", 1)]
    names = [x[0] for x in new_dirs]
    blocks, hashes = make_blocks(48, 2)
    before = model_init([1, 1, 1], [0, 0, 0])
    after = model_update(before, [0, 1, 2, -1], [1, 1, 1, 1], [0, 0, 0, 0])
    with manager(tmp_path, dirs) as bm:
        put_all(bm, blocks, hashes)
        for node in range(N):
            assert bm.set_data_dirs(node, new_dirs) == BM.OK
            assert persisted(tmp_path, node) == after
        assert_gets(bm, blocks, hashes)  # readable from the secondaries before any move
        predicted = sum(1 for h in hashes for node in holders(bm, h) if after[1][part(h)] != before[1][part(h)])
        file_bytes = {}
        for h in hashes:
            for node in holders(bm, h):
                if after[1][part(h)] != before[1][part(h)]:
                    file_bytes[(node, h)] = os.path.getsize(file_path(tmp_path, node, names[before[1][part(h)]], h))
        assert predicted > 0
        assert bm.rebalance_all() == predicted
        dm = bm.drive_metrics()
        assert dm["rebalance_files_moved"] == predicted and dm["rebalance_errors"] == 0
        assert dm["rebalance_bytes_moved"] == sum(file_bytes.values())
        for node in range(N):
            cap, prim, sec = persisted(tmp_path, node)
            assert prim == after[1] and not any(sec)
        for h in hashes:
            for node in holders(bm, h):
                assert where(tmp_path, node, names, h) == [names[after[1][part(h)]]]
        assert bm.rebalance_all() == 0
        assert_gets(bm, blocks, hashes)
    with manager(tmp_path, dirs) as bm:  # restart: the data_layout files win over the configured list
        for node in range(N):
            cap, prim, sec = persisted(tmp_path, node)
            assert cap == [1, 1, 1, 1] and prim == after[1] and not any(sec)
        assert_gets(bm, blocks, hashes)
        assert bm.drive_metrics()["drive_marker_errors"] == 0


# ---------------------------------------------------------------- a lost drive
@pytest.mark.parametrize("code", ["rs", "clay", "lrc"])
def test_lost_drive_is_rebuilt_from_the_other_nodes(tmp_path, code):
    dirs = [("d0", 1), ("d1", 1), ("d2", 1)]
    names = [x[0] for x in dirs]
    node = 3
    blocks, hashes = make_blocks(24, 3, size=1 << 20)
    before = model_init([1, 1, 1], [0, 0, 0])
    after = model_update(before, [0, 2], [1, 1], [0, 0])
    with manager(tmp_path, dirs, code) as bm:
        put_all(bm, blocks, hashes)
        lost = [h for h in hashes if node in holders(bm, h) and before[1][part(h)] == 1]
        assert lost
        shutil.rmtree(root_of(tmp_path, node, "d1"))  # the drive dies, its files with it
        assert bm.set_data_dirs(node, dirs) == BM.E_MESSAGE  # the marker is gone: Garage would not start
        assert bm.drive_metrics()["drive_marker_errors"] == 1
        assert bm.rebalance_step(node)[0] == BM.E_MESSAGE  # the node is down
        assert_gets(bm, blocks, hashes)  # degraded reads meanwhile
        assert bm.set_data_dirs(node, [dirs[0], dirs[2]]) == BM.OK
        assert persisted(tmp_path, node) == after
        assert_gets(bm, blocks, hashes)
        fetched0 = bm.metrics()["resync_bytes_fetched"]
        assert bm.repair_enqueue_missing(node) == len(lost)
        failed, done = bm.resync_all(node)
        assert failed == 0 and done == len(lost)
        if code == "clay":
            assert bm.metrics()["resync_bytes_fetched"] - fetched0 == len(lost) * CLAY_REPAIR_BYTES_1MIB
        for h in hashes:
            if node in holders(bm, h):
                assert where(tmp_path, node, ["d0", "d2"], h) == [names[[0, 2][after[1][part(h)]]]]
        assert bm.repair_enqueue_missing(node) == 0
        if code != "lrc":  # MDS codes: with m other holders down every GET needs node's shards
            for other in (10, 11, 12, 13):
                bm.set_node_up(other, False)
            assert_gets(bm, blocks, hashes)


def test_lost_drive_rebuilt_by_stripe_repair(tmp_path):
    dirs = [("d0", 1), ("d1", 1)]
    node = 5
    blocks, hashes = make_blocks(16, 4)
    before = model_init([1, 1], [0, 0])
    with manager(tmp_path, dirs) as bm:
        put_all(bm, blocks, hashes)
        lost = [h for h in hashes if node in holders(bm, h) and before[1][part(h)] == 0]
        shutil.rmtree(root_of(tmp_path, node, "d0"))
        assert bm.set_data_dirs(node, dirs) == BM.E_MESSAGE
        assert bm.set_data_dirs(node, [dirs[1]]) == BM.OK
        assert bm.stripe_repair_all() == (len(lost), len(lost))
        for h in hashes:
            if node in holders(bm, h):
                assert where(tmp_path, node, ["d1"], h) == ["d1"]
        assert_gets(bm, blocks, hashes)


# ---------------------------------------------------------------- read-only drive
def test_read_only_drive_is_served_never_written_and_rebalanced_off(tmp_path):
    dirs = [("d0", 1), ("d1", 1)]
    ro = [("d0", 1), ("d1", 0, True)]
    node = 0
    blocks, hashes = make_blocks(24, 5)
    with manager(tmp_path, dirs) as bm:
        put_all(bm, blocks[:16], hashes[:16])
        on_d1 = [h for h in hashes[:16] if where(tmp_path, node, ["d1"], h)]
        assert on_d1
        assert bm.set_data_dirs(node, ro) == BM.OK
        cap, prim, sec = persisted(tmp_path, node)
        assert set(prim) == {0} and all(s == [1] for s in sec[512:])
        # node's shards are needed: m other holders down
        for other in (1, 2, 3, 4):
            bm.set_node_up(other, False)
        assert_gets(bm, blocks[:16], hashes[:16])
        for other in (1, 2, 3, 4):
            bm.set_node_up(other, True)
        put_all(bm, blocks[16:], hashes[16:])
        assert all(not where(tmp_path, node, ["d1"], h) for h in hashes[16:])  # never written
        assert bm.rebalance_all(nodes=[node]) == len(on_d1)
        assert all(not where(tmp_path, node, ["d1"], h) for h in hashes)
        assert all(where(tmp_path, node, ["d0"], h) == ["d0"] for h in hashes)
        assert_gets(bm, blocks, hashes)


# ---------------------------------------------------------------- scrub across drives
def test_scrub_quarantines_next_to_the_file_and_resync_writes_the_primary(tmp_path):
    dirs = [("d0", 1), ("d1", 1)]
    new_dirs = dirs + [("d2", 2)]
    names = [x[0] for x in new_dirs]
    node = 2
    blocks, hashes = make_blocks(32, 6)
    after = model_update(model_init([1, 1], [0, 0]), [0, 1, -1], [1, 1, 2], [0, 0, 0])
    with manager(tmp_path, dirs) as bm:
        put_all(bm, blocks, hashes)
        assert bm.set_data_dirs(node, new_dirs) == BM.OK
        # a shard still on drive 2 (d1, now a secondary) whose primary is d2
        h = next(h for h in hashes if where(tmp_path, node, names, h) == ["d1"] and after[1][part(h)] == 2)
        assert bm.corrupt_shard(node, h, 1000) == BM.OK
        rc, checked, corrupt = bm.scrub(node)
        assert rc == BM.OK and corrupt == 1
        assert os.path.exists(file_path(tmp_path, node, "d1", h, ".corrupted"))
        assert where(tmp_path, node, names, h) == []
        failed, done = bm.resync_all(node)
        assert failed == 0 and done == 1
        assert where(tmp_path, node, names, h) == ["d2"]
        assert_gets(bm, blocks, hashes)


# ---------------------------------------------------------------- rebalance stopped midway
def test_rebalance_stopped_midway_stays_readable_and_completes(tmp_path):
    dirs = [("d0", 1), ("d1", 1)]
    new_dirs = dirs + [("d2", 1)]
    names = [x[0] for x in new_dirs]
    node = 1
    blocks, hashes = make_blocks(40, 7)
    before = model_init([1, 1], [0, 0])
    after = model_update(before, [0, 1, -1], [1, 1, 1], [0, 0, 0])
    with manager(tmp_path, dirs) as bm:
        put_all(bm, blocks, hashes)
        assert bm.set_data_dirs(node, new_dirs) == BM.OK
        predicted = sum(1 for h in hashes if node in holders(bm, h) and after[1][part(h)] != before[1][part(h)])
        assert predicted >= 4
        bm.debug_convert_stop_after(3)  # one move and a half: a write, a removal, a write
        rc, _, finished, moved = bm.rebalance_step(node)
        assert rc == BM.OK and finished and moved == 1
        bm.debug_convert_stop_after(-1)
        assert any(persisted(tmp_path, node)[2])  # not a clean pass: the secondaries stay
        assert_gets(bm, blocks, hashes)
        for h in hashes:  # every shard readable from node, wherever it is now
            if node in holders(bm, h):
                assert bm.node_shard_index(node, h) >= 0
        rc, cur, finished, a = bm.rebalance_step(node, max_files=2)
        assert rc == BM.OK and not finished
        rc, _, finished, b = bm.rebalance_step(node, cursor=cur)
        assert rc == BM.OK and finished
        assert not any(persisted(tmp_path, node)[2])  # a clean pass from cursor NULL to the end drops the secondaries
        assert bm.rebalance_step(node)[3] == 0
        # the file whose removal was stopped had been written already: the second pass only removed its old copy
        assert 1 + a + b == predicted - 1 == bm.drive_metrics()["rebalance_files_moved"]
        assert bm.drive_metrics()["rebalance_errors"] >= 1
        for h in hashes:
            if node in holders(bm, h):
                assert where(tmp_path, node, names, h) == [names[after[1][part(h)]]]
        assert_gets(bm, blocks, hashes)


# ---------------------------------------------------------------- code conversion of replicas placed by the drives
def test_replicas_placed_by_the_drive_layout_convert(tmp_path):
    rf = 3
    dirs = [("d0", 1), ("d1", 1)]
    names = [x[0] for x in dirs]
    model = model_init([1, 1], [0, 0])
    blocks, hashes = make_blocks(12, 8)
    for h, b in zip(hashes, blocks):  # a replicated Garage cluster whose nodes had two drives
        for i in range(rf):
            p = file_path(tmp_path, (h[0] % N + i) % N, names[model[1][part(h)]], h, "")
            os.makedirs(os.path.dirname(p), exist_ok=True)
            with open(p, "wb") as f:
                f.write(b.tobytes())
    with manager(tmp_path, dirs, legacy_replicas=rf) as bm:
        assert_gets(bm, blocks, hashes)  # served from the replicas
        assert bm.convert_all() == len(hashes)
        for h in hashes:
            for node in range(N):
                assert where(tmp_path, node, names, h, "") == []
        assert_gets(bm, blocks, hashes)


# ---------------------------------------------------------------- a single-directory store restarted with drives
def test_single_directory_store_restarted_with_drives(tmp_path):
    blocks, hashes = make_blocks(32, 9)
    with BM.BlockManager(n_nodes=N, data_dir=str(tmp_path), batch_max_blocks=8) as bm:
        put_all(bm, blocks, hashes)
        rows = {bytes(h): holders(bm, h) for h in hashes}
    dirs = [(".", 1), ("d1", 1)]
    names = [x[0] for x in dirs]
    model = model_init([1, 1], [1, 0])  # "." holds files: a secondary wherever it is not primary
    with manager(tmp_path, dirs) as bm:
        for node in range(N):
            assert persisted(tmp_path, node) == model
        assert_gets(bm, blocks, hashes)
        predicted = sum(1 for h in hashes for node in rows[bytes(h)] if model[1][part(h)] == 1)
        assert bm.rebalance_all() == predicted
        for h in hashes:
            for node in rows[bytes(h)]:
                assert where(tmp_path, node, names, h) == [names[model[1][part(h)]]]
        assert_gets(bm, blocks, hashes)
        assert not any(persisted(tmp_path, 0)[2])


def test_drives_unset_keeps_todays_paths(tmp_path):
    blocks, hashes = make_blocks(8, 10)
    with BM.BlockManager(n_nodes=N, data_dir=str(tmp_path), batch_max_blocks=8) as bm:
        put_all(bm, blocks, hashes)
        for h in hashes:
            for node in holders(bm, h):
                assert os.path.exists(file_path(tmp_path, node, ".", h))
        assert bm.rebalance_step(0)[0] == -1  # no drives: nothing to rebalance
    assert not any(os.path.exists(os.path.join(str(tmp_path), "node%d" % n, x))
                   for n in range(N) for x in ("data_layout", "garage-marker"))


def test_memory_store_refuses_drives():
    with pytest.raises(BM.BlockManagerError) as e:
        BM.BlockManager(n_nodes=N, data_dirs=[("d0", 1)])
    assert e.value.code == -1
