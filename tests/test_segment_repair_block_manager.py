"""Repair by segment in the block manager (DESIGN.md section 5.15): a resync of a shard its node quarantined because
its adler8 tag failed keeps the copy's units that pass their segment tags and rebuilds only the others, from the same
columns of the survivors -- the garage_ec_segment_read_ranges runs.  The shard comes back byte for byte with its
original tag; anything the partial path cannot prove falls back to the whole-shard rebuild.  Memory and file stores,
RS(10,4), LRC(10,2,2) and PB(10,4)."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import garage_b200 as G  # noqa: E402
from garage_b200 import block_manager as BM  # noqa: E402
from test_segment_block_manager import CODES, K, M, STORES, block, manager, put, seg_bytes  # noqa: E402

pytestmark = pytest.mark.gpu

IDX = 2  # a data shard: LRC repairs it from its local group
ZERO = {"repairs": 0, "units_rebuilt": 0, "bytes_read": 0, "bytes_fetched": 0, "fallbacks": 0, "call_us": 0}


def ec_of(code):
    if code == "lrc":
        return G.GarageEc.lrc(0, K, 2, M - 2)
    if code == "pb":
        return G.GarageEc.piggyback(0, K, M)
    return G.GarageEc(0, K, M)


def shard_len(code, n=1 << 20):
    with ec_of(code) as ec:
        return ec.code_shard_len(n)


def planned_bytes(code, L, idx, bad):
    """what garage_ec_segment_read_ranges names for index idx missing segments `bad`"""
    sp = np.full(K + M, 0xFF, np.uint8)
    for g in bad:
        sp[idx] &= ~np.uint8(1 << g)
        if code == "pb":
            sp[idx] &= ~np.uint8(1 << (g ^ 4))
    with ec_of(code) as ec:
        return sum(n for _, _, n in ec.segment_read_ranges(sp, L, want=np.eye(K + M, dtype=np.uint8)[idx]))


def shard_file(tmp_path, node, h, ext=".shard"):
    return os.path.join(str(tmp_path / "store"), "node%d" % node, h[:1].hex(), h[1:2].hex(), h.hex() + ext)


def read(path):
    with open(path, "rb") as f:
        return f.read()


def rot(bm, code, h, idx, segs):
    """flip a byte of index idx's shard in each segment of segs, then scrub its node: the tag fails there"""
    node = bm.storage_nodes_of(h)[idx]
    S = seg_bytes(bm, code, h)
    for g in segs:
        assert bm.corrupt_shard(node, h, g * S + 5) == BM.OK
    rc, _, corrupt = bm.scrub(node)
    assert rc == BM.OK and corrupt == 1
    return node


def all_valid(bm, h, b):
    rc, info = bm.block_info(h, check_tags=True)
    assert rc == BM.OK and info["state"] == [BM.SHARD_VALID] * (K + M), info["state"]
    rc, got = bm.rpc_get_block(h)
    assert rc == BM.OK and np.array_equal(got, b)


@pytest.mark.parametrize("store", STORES)
@pytest.mark.parametrize("code", sorted(CODES))
@pytest.mark.parametrize("segs", [[1], [1, 6]], ids=["one", "two"])
def test_rotten_segments_are_rebuilt_alone(tmp_path, store, code, segs):
    with manager(tmp_path, store, code) as bm:
        b, h = put(bm)
        node = bm.storage_nodes_of(h)[IDX]
        orig = read(shard_file(tmp_path, node, h)) if store == "file" else None
        rot(bm, code, h, IDX, segs)
        m0, s0 = bm.metrics(), bm.segment_repair_metrics()
        assert s0 == ZERO
        assert bm.resync_all(node) == (0, 1)
        m1, s1 = bm.metrics(), bm.segment_repair_metrics()
        L = shard_len(code)
        fetched = planned_bytes(code, L, IDX, segs)
        if code == "rs":
            assert fetched == 131200 * len(segs)
        if code == "lrc":
            assert fetched == 65600 * len(segs)
        assert s1["repairs"] == 1 and s1["fallbacks"] == 0 and s1["units_rebuilt"] == len(segs)
        assert s1["bytes_fetched"] == fetched and s1["bytes_read"] == L + fetched
        assert m1["resync_bytes_fetched"] - m0["resync_bytes_fetched"] == fetched
        assert m1["resync_bytes_read"] - m0["resync_bytes_read"] == L + fetched
        assert m1["resync_counter"] - m0["resync_counter"] == 1
        if store == "file":
            assert read(shard_file(tmp_path, node, h)) == orig  # same bytes, same header and tag
            assert os.path.exists(shard_file(tmp_path, node, h, ".corrupted"))
        all_valid(bm, h, b)
        assert bm.segment_repair_metrics()["repairs"] == 1


def fallback_case(bm, code, h, case, tmp_path):
    """damage index IDX so that the partial path must not (or cannot) finish; -> its node"""
    who = bm.storage_nodes_of(h)
    node = who[IDX]
    S = seg_bytes(bm, code, h)
    if case == "all_segments":
        rot(bm, code, h, IDX, range(8))
    elif case == "bad_header":
        assert bm.corrupt_shard(node, h, S + 5) == BM.OK
        assert bm.corrupt_shard_header(node, h, 1) == BM.OK
        assert bm.scrub(node)[2] == 1
    elif case == "hunted_stale":
        assert bm.plant_stale_shard(node, h) == BM.OK
        rc, _ = bm.rpc_get_block(h)  # the content-hash hunt quarantines it
        assert rc == BM.OK and bm.metrics()["corruption_counter"] == 1
    elif case == "stale_then_rot":
        assert bm.plant_stale_shard(node, h) == BM.OK
        rot(bm, code, h, IDX, [1])  # its other seven segments pass the stale tag; the post-check fails
    elif case == "bad_survivor":
        rot(bm, code, h, IDX, [1])
        # survivor 0, not scrubbed, in a piece the rebuild of unit 1 reads (PB: its b-half, segment 5)
        assert bm.corrupt_shard(who[0], h, (5 if code == "pb" else 1) * S + 9) == BM.OK
    return node


CASES = ["all_segments", "bad_header", "hunted_stale", "stale_then_rot", "bad_survivor"]


@pytest.mark.parametrize("store", STORES)
@pytest.mark.parametrize("code", sorted(CODES))
@pytest.mark.parametrize("case", CASES)
def test_whole_shard_fallbacks(tmp_path, store, code, case):
    with manager(tmp_path, store, code) as bm:
        b, h = put(bm)
        node = bm.storage_nodes_of(h)[IDX]
        orig = read(shard_file(tmp_path, node, h)) if store == "file" else None
        fallback_case(bm, code, h, case, tmp_path)
        m0 = bm.metrics()
        assert bm.resync_block(node, h) == BM.OK
        s1, m1 = bm.segment_repair_metrics(), bm.metrics()
        assert s1["repairs"] == 0 and s1["fallbacks"] == 1, s1
        if case == "all_segments" and code == "rs":  # the whole-shard rebuild's k whole shards, as before
            assert m1["resync_bytes_fetched"] - m0["resync_bytes_fetched"] == 1048580
        if store == "file":
            assert read(shard_file(tmp_path, node, h)) == orig
            assert os.path.exists(shard_file(tmp_path, node, h, ".corrupted"))
        if case == "bad_survivor":  # survivor 0 was quarantined by its span read; its own resync is partial
            w0 = bm.storage_nodes_of(h)[0]
            assert bm.resync_block(w0, h) == BM.OK
            assert bm.segment_repair_metrics()["repairs"] == 1
        all_valid(bm, h, b)


@pytest.mark.parametrize("code", sorted(CODES))
def test_file_store_restart_forgets_the_hint(tmp_path, code):
    with manager(tmp_path, "file", code) as bm:
        b, h = put(bm)
        node = rot(bm, code, h, IDX, [3])
        orig_copy = read(shard_file(tmp_path, node, h, ".corrupted"))
    with manager(tmp_path, "file", code) as bm:
        assert bm.resync_block(node, h) == BM.OK
        s = bm.segment_repair_metrics()
        assert s["repairs"] == 0 and s["fallbacks"] == 1 and s["bytes_fetched"] == 0
        assert read(shard_file(tmp_path, node, h, ".corrupted")) == orig_copy
        all_valid(bm, h, b)


@pytest.mark.parametrize("kw", [{"shard_sum_kind": BM.SUM_BLAKE2}, {"clay": True}], ids=["blake2", "clay"])
@pytest.mark.parametrize("store", STORES)
def test_blake2_and_clay_stores_are_unchanged(tmp_path, kw, store):
    with BM.BlockManager(K, M, data_dir=str(tmp_path / "store") if store == "file" else None, **kw) as bm:
        b, h = block(5)
        assert bm.rpc_put_block(h, b) == BM.OK
        node = bm.storage_nodes_of(h)[IDX]
        assert bm.corrupt_shard(node, h, 40000) == BM.OK
        assert bm.scrub(node)[2] == 1
        m0 = bm.metrics()
        assert bm.resync_all(node) == (0, 1)
        if "clay" in kw:  # the 1/m runs of the 13 helpers, as before
            assert bm.metrics()["resync_bytes_fetched"] - m0["resync_bytes_fetched"] == 346112
        assert bm.segment_repair_metrics() == ZERO
        all_valid(bm, h, b)


def test_multi_version_store_is_unchanged(tmp_path):
    n, cap = 16, 1 << 40
    layout = dict(zone=[0] * n, capacity=[cap] * 14 + [0, 0])
    with BM.BlockManager(k=K, m=M, n_nodes=n, data_dir=str(tmp_path / "store"), layout=layout, batch_max_blocks=8) as bm:
        blocks = [block(20 + i) for i in range(4)]
        for b, h in blocks:
            assert bm.rpc_put_block(h, b) == BM.OK
        rows1 = [bm.storage_nodes_of(h) for _, h in blocks]
        assert bm.apply_layout([0] * n, [cap] * n)[0] == BM.OK
        assert len(bm.layout_versions()) == 2
        b, h = blocks[0]
        i = next(i for i in range(K + M) if rows1[0][i] == bm.storage_nodes_of(h)[i])  # the same holder in both
        node = rows1[0][i]
        assert bm.corrupt_shard(node, h, 5) == BM.OK
        assert bm.scrub(node)[2] == 1
        bm.resync_block(node, h)
        assert bm.segment_repair_metrics() == ZERO


def test_multi_drive_repair_lands_on_the_primary(tmp_path):
    from test_drive_block_manager import make_blocks, model_init, model_update, part, put_all, where  # noqa: E402
    from test_drive_block_manager import manager as drive_manager

    dirs = [("d0", 1), ("d1", 1)]
    new_dirs = dirs + [("d2", 2)]
    names = [x[0] for x in new_dirs]
    node = 2
    blocks, hashes = make_blocks(32, 6)
    after = model_update(model_init([1, 1], [0, 0]), [0, 1, -1], [1, 1, 2], [0, 0, 0])
    with drive_manager(tmp_path, dirs) as bm:
        put_all(bm, blocks, hashes)
        assert bm.set_data_dirs(node, new_dirs) == BM.OK
        # a shard still on drive d1 (now a secondary) whose primary is d2
        j = next(j for j, h in enumerate(hashes) if where(tmp_path, node, names, h) == ["d1"] and after[1][part(h)] == 2)
        h = hashes[j]
        assert bm.corrupt_shard(node, h, 1000) == BM.OK
        assert bm.scrub(node)[2] == 1
        assert where(tmp_path, node, names, h, ".corrupted") == ["d1"]
        assert bm.resync_all(node) == (0, 1)
        assert where(tmp_path, node, names, h) == ["d2"]
        s = bm.segment_repair_metrics()
        assert s["repairs"] == 1 and s["fallbacks"] == 0 and s["units_rebuilt"] == 1
        rc, info = bm.block_info(h, check_tags=True)
        assert rc == BM.OK and info["state"] == [BM.SHARD_VALID] * (K + M)
        rc, got = bm.rpc_get_block(h)
        assert rc == BM.OK and np.array_equal(got, blocks[j])


@pytest.mark.parametrize("code", sorted(CODES))
def test_eight_workers_agree_with_one(tmp_path, code):
    """many blocks, one rotten segment each on the same node: eight resync workers repair them all, with the same
    bytes and counters as one worker"""
    out = []
    for workers in (1, 8):
        with manager(tmp_path / ("w%d" % workers), "memory", code) as bm:
            node = 0
            blocks = [block(100 + s, (1 << 20) - 4099 * s) for s in range(24)]
            for s, (b, h) in enumerate(blocks):
                assert bm.rpc_put_block(h, b) == BM.OK
                S = seg_bytes(bm, code, h)
                assert bm.corrupt_shard(node, h, (s % 8) * S + 11) == BM.OK
            rc, _, corrupt = bm.scrub(node)
            assert rc == BM.OK and corrupt == len(blocks)
            assert bm.resync_all(node, workers=workers) == (0, len(blocks))
            s = bm.segment_repair_metrics()
            assert s["repairs"] == len(blocks) and s["fallbacks"] == 0
            for b, h in blocks:
                all_valid(bm, h, b)
            out.append({k: v for k, v in s.items() if k != "call_us"})
    assert out[0] == out[1]
