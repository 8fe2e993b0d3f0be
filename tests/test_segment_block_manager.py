"""Salvage in the block manager (DESIGN.md section 5.14): a block whose configured stripe has more than m damaged
shards, their damage in different adler8 segments, is rebuilt segment by segment from the live shards and their
quarantined copies, proven by its content hash, returned by GET and healed by resync and stripe repair.  Memory and
file stores, RS(10,4), LRC(10,2,2) and PB(10,4)."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from garage_b200 import block_manager as BM  # noqa: E402

pytestmark = pytest.mark.gpu

K, M = 10, 4
CODES = {"rs": {}, "lrc": {"local_groups": 2}, "pb": {"piggyback": True}}


def manager(tmp_path, store, code, **kw):
    return BM.BlockManager(K, M, data_dir=str(tmp_path / "store") if store == "file" else None, **CODES[code], **kw)


def block(seed, n=1 << 20):
    b = np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8)
    return b, BM.blake2sum(b)


def seg_bytes(bm, code, h):
    """the adler8 segment length of h's shards"""
    L = -(-bm.block_info(h)[1]["block_len"] // K)
    if code == "pb":
        L = -(-L // 128) * 128
    return (-(-L // 8) + 15) // 16 * 16


def put(bm, seed=1):
    b, h = block(seed)
    assert bm.rpc_put_block(h, b) == BM.OK
    return b, h


def damage(bm, code, h, idx_seg):
    """flip a byte of index i's shard in segment g, for each (i, g)"""
    who = bm.storage_nodes_of(h)
    S = seg_bytes(bm, code, h)
    for i, g in idx_seg:
        assert bm.corrupt_shard(who[i], h, g * S + 5) == BM.OK


def spread(n):
    """n damaged indices, index i in segment i mod 8: at most one per segment up to 8, two (g and g + 4 are one PB
    unit) per PB unit, never more than m per unit"""
    return [(i, i % 8) for i in range(n)]


STORES = ["memory", "file"]


@pytest.mark.parametrize("store", STORES)
@pytest.mark.parametrize("code", sorted(CODES))
@pytest.mark.parametrize("nbad", [M + 1, 2 * M])
def test_salvaged_get_then_heal(tmp_path, store, code, nbad):
    with manager(tmp_path, store, code) as bm:
        b, h = put(bm)
        damage(bm, code, h, spread(nbad))
        rc, got = bm.rpc_get_block(h)
        assert rc == BM.OK and np.array_equal(got, b)
        mt = bm.salvage_metrics()
        assert mt["salvage_blocks"] == 1 and mt["salvage_failures"] == 0 and mt["salvage_units_rebuilt"] >= nbad
        assert mt["salvage_quarantined_segments"] >= nbad * 7 // 8 and mt["salvage_bytes_read"] > 0
        # heal: resync (memory store) or stripe repair (file store) rewrites every damaged index
        if store == "memory":
            for node in range(bm.n_nodes):
                bm.resync_all(node)
        else:
            bm.stripe_repair_all()
        rc, info = bm.block_info(h, check_tags=True)
        assert rc == BM.OK and info["state"] == [BM.SHARD_VALID] * (K + M), info["state"]
        before = bm.salvage_metrics()["salvage_attempts"]
        rc, got = bm.rpc_get_block(h)
        assert rc == BM.OK and np.array_equal(got, b)
        assert bm.salvage_metrics()["salvage_attempts"] == before


@pytest.mark.parametrize("code", sorted(CODES))
def test_mixed_loss(tmp_path, code):
    """m - 1 holders down and two rotten shards in different segments (m + 1 indices out) salvage; m holders down and
    one rotten shard leave a segment with only k - 1 valid shards: no code can rebuild it, and nothing is written"""
    with manager(tmp_path, "memory", code) as bm:
        b, h = put(bm)
        who = bm.storage_nodes_of(h)
        for i in range(M - 1):
            bm.set_node_up(who[K + M - 1 - i], False)
        damage(bm, code, h, [(0, 1), (1, 2)])
        rc, got = bm.rpc_get_block(h)
        assert rc == BM.OK and np.array_equal(got, b)
        for node in range(bm.n_nodes):
            bm.set_node_up(node, True)
        b2, h2 = put(bm, seed=2)
        who2 = bm.storage_nodes_of(h2)
        for i in range(M):
            bm.set_node_up(who2[K + i], False)
        damage(bm, code, h2, [(0, 3)])
        rc, _ = bm.rpc_get_block(h2)
        assert rc == BM.E_MISSING_BLOCK
        assert bm.salvage_metrics()["salvage_failures"] == 1


@pytest.mark.parametrize("store", STORES)
@pytest.mark.parametrize("code", sorted(CODES))
def test_same_segment_in_m_plus_one_shards_is_not_salvaged(tmp_path, store, code):
    with manager(tmp_path, store, code) as bm:
        b, h = put(bm)
        damage(bm, code, h, [(i, 0) for i in range(M + 1)])
        rc, _ = bm.rpc_get_block(h)
        assert rc == BM.E_MISSING_BLOCK
        mt = bm.salvage_metrics()
        assert mt["salvage_attempts"] == 1 and mt["salvage_failures"] == 1 and mt["salvage_blocks"] == 0
        for node in range(bm.n_nodes):  # resync fails as before and writes nothing
            bm.resync_all(node)
        rc, info = bm.block_info(h)
        assert [info["state"][i] for i in range(M + 1)] == [BM.SHARD_QUARANTINED] * (M + 1)


@pytest.mark.parametrize("kw", [{"shard_sum_kind": BM.SUM_BLAKE2}, {"clay": True}], ids=["blake2", "clay"])
def test_blake2_and_clay_stores_are_not_salvaged(tmp_path, kw):
    with BM.BlockManager(K, M, **kw) as bm:
        b, h = block(3)
        assert bm.rpc_put_block(h, b) == BM.OK
        L = bm.block_info(h)[1]["block_len"]
        who = bm.storage_nodes_of(h)
        for i in range(M + 1):
            bm.corrupt_shard(who[i], h, (i + 1) * 1024)
        rc, _ = bm.rpc_get_block(h)
        assert rc == BM.E_MISSING_BLOCK and L == len(b)
        for node in range(bm.n_nodes):
            bm.resync_all(node)
        assert bm.salvage_metrics()["salvage_attempts"] == 0
        rc, info = bm.block_info(h)
        assert info["state"][: M + 1] == [BM.SHARD_QUARANTINED] * (M + 1)


@pytest.mark.parametrize("store", STORES)
def test_stale_quarantined_copy_yields_no_wrong_bytes(tmp_path, store):
    with manager(tmp_path, store, "rs") as bm:
        b, h = put(bm)
        who = bm.storage_nodes_of(h)
        assert bm.plant_stale_shard(who[0], h) == BM.OK
        rc, got = bm.rpc_get_block(h)  # the hunt quarantines the stale index 0: its .corrupted copy is tag-consistent
        assert rc == BM.OK and np.array_equal(got, b)
        damage(bm, "rs", h, [(i, i) for i in range(1, M + 1)])
        rc, got = bm.rpc_get_block(h)
        assert rc == BM.E_MISSING_BLOCK and got is None
        mt = bm.salvage_metrics()
        assert mt["salvage_attempts"] == 1 and mt["salvage_failures"] == 1 and mt["salvage_blocks"] == 0


@pytest.mark.parametrize("code", sorted(CODES))
def test_ranged_and_opened_gets_of_a_salvageable_block(tmp_path, code):
    with manager(tmp_path, "memory", code) as bm:
        b, h = put(bm)
        damage(bm, code, h, spread(M + 2))
        for off, n in ((0, 4096), (123457, 70000), ((1 << 20) - 100, 100)):
            rc, got = bm.rpc_get_block_range(h, off, n)
            assert rc == BM.OK and np.array_equal(got, b[off:off + n])
        key = bytes(range(32))
        p = np.random.default_rng(9).integers(0, 256, 300000, dtype=np.uint8)
        rc, hs = bm.rpc_put_block_sealed(key, p)
        assert rc == BM.OK
        damage(bm, code, hs, spread(M + 1))
        rc, got = bm.rpc_get_block_opened(hs, key)
        assert rc == BM.OK and np.array_equal(got, p)
        assert bm.salvage_metrics()["salvage_blocks"] >= 2


@pytest.mark.parametrize("code", sorted(CODES))
def test_file_store_restart_salvages_from_corrupted_files(tmp_path, code):
    with manager(tmp_path, "file", code) as bm:
        b, h = put(bm)
        damage(bm, code, h, spread(M + 2))
        rc, got = bm.rpc_get_block(h)  # quarantines the damaged shards into .corrupted files
        assert rc == BM.OK and np.array_equal(got, b)
    n_corrupted = sum(f.endswith(".corrupted") for _, _, fs in os.walk(tmp_path) for f in fs)
    assert n_corrupted == M + 2
    with manager(tmp_path, "file", code) as bm:
        rc, got = bm.rpc_get_block(h)
        assert rc == BM.OK and np.array_equal(got, b)
        assert bm.salvage_metrics()["salvage_blocks"] == 1
