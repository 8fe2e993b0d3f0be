"""Copies with re-encryption through the block manager (DESIGN.md 5.11), on file stores: a key rotation under every
code stores the oracle's seal of the plaintext under the nonce in its first 8 bytes, opens under the new key, fails
under the old one and leaves the sources alone; plaintext sources; a multipart re-chunk and an UploadPartCopy range;
m holders of a source without their shards; a planted stale source shard found through one fallback and quarantined; a source held only under a
previous code; a wrong source key and a missing source store nothing; argument refusals; concurrent copies batch
together; the new block resyncs, deep-scrubs clean and survives a restart; and the metrics."""
import os
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import oracle_lib as O  # noqa: E402
import sse_c_oracle as S  # noqa: E402

import garage_b200 as G  # noqa: E402
from garage_b200 import block_manager as BM  # noqa: E402

pytestmark = pytest.mark.gpu
CODES = {"rs": {}, "lrc": {"local_groups": 2}, "pb": {"piggyback": True}, "clay": {"clay": True}}
LENS = [1 << 20, 1, 4096, 4097, 54321]
SEALED_MAX = G.sealed_len(1 << 20)


def manager(code, d, **kw):
    kw.setdefault("batch_max_blocks", 8)
    return BM.BlockManager(k=10, m=4, n_nodes=14, data_dir=str(d), **CODES[code], **kw)


def key_of(i):
    return bytes((11 * i + 3 * j + 1) & 0xFF for j in range(32))


def put_sources(bm, seed, key=key_of(0), lens=LENS):
    out = []
    for i, n in enumerate(lens):
        p = O.fill_random(n, seed + i)
        rc, h = bm.rpc_put_block_sealed(key, p)
        assert rc == BM.OK
        out.append((h, p))
    return out


def check_stored(bm, h, n, q, new_key, old_key):
    """the stored block is the oracle's seal of q under its own nonce; it opens under new_key only"""
    rc, b = bm.rpc_get_block(h, cap=SEALED_MAX)
    assert rc == BM.OK and len(b) == n == G.sealed_len(len(q)) and BM.blake2sum(b) == h
    assert b.tobytes() == S.seal(new_key, b[:8].tobytes(), q.tobytes())
    rc, got = bm.rpc_get_block_opened(h, new_key)
    assert rc == BM.OK and np.array_equal(got, q)
    if old_key is not None:
        rc, got = bm.rpc_get_block_opened(h, old_key)
        assert rc == G.E_AUTH


@pytest.mark.parametrize("code", list(CODES))
def test_key_rotation_stores_the_oracle_seal(code, tmp_path):
    with manager(code, tmp_path) as bm:
        old, new = key_of(0), key_of(1)
        srcs = put_sources(bm, 0x6E5E)
        before = [bm.rpc_get_block(h, cap=SEALED_MAX)[1] for h, _ in srcs]
        w0 = bm.metrics()["bytes_written"]
        for (h, p), b in zip(srcs, before):
            rc, h2, n = bm.put_block_resealed([(h, 0, p.size)], old, new)
            assert rc == BM.OK and h2 != h
            check_stored(bm, h2, n, p, new, old)
        assert bm.metrics()["bytes_written"] > w0
        for (h, p), b in zip(srcs, before):  # the sources are untouched and still open under the old key
            rc, again = bm.rpc_get_block(h, cap=SEALED_MAX)
            assert rc == BM.OK and np.array_equal(again, b)
            rc, got = bm.rpc_get_block_opened(h, old)
            assert rc == BM.OK and np.array_equal(got, p)
        m = bm.reseal_metrics()
        assert m["calls"] == len(LENS) and m["sources_gathered"] == len(LENS) and m["batches"] >= 1
        assert m["fallbacks"] == 0 and m["auth_failures"] == 0
        assert m["bytes_read"] >= sum(G.sealed_len(p.size) for _, p in srcs)
        assert m["reseal_call_us"] > 0 and m["call_us"] >= m["reseal_call_us"] / 8


def test_plaintext_sources_rechunk_and_part_copy(tmp_path):
    with manager("rs", tmp_path) as bm:
        new = key_of(2)
        a, b = put_sources(bm, 0x6E60, key=None, lens=[1 << 20, 300000])
        # plaintext to SSE-C, a whole block
        rc, h, n = bm.put_block_resealed([(a[0], 0, a[1].size)], None, new)
        assert rc == BM.OK
        check_stored(bm, h, n, a[1], new, None)
        # sealed sources: save_stream's re-chunk (the tail of A, then the head of B) and an UploadPartCopy range
        old = key_of(3)
        (ha, pa), (hb, pb) = put_sources(bm, 0x6E61, key=old, lens=[1 << 20, 1 << 20])
        cut = 777777
        rc, h, n = bm.put_block_resealed([(ha, cut, pa.size - cut), (hb, 0, cut)], old, new)
        assert rc == BM.OK
        check_stored(bm, h, n, np.concatenate([pa[cut:], pb[:cut]]), new, old)
        rc, h, n = bm.put_block_resealed([(hb, 4093, 123457)], old, new)
        assert rc == BM.OK
        check_stored(bm, h, n, pb[4093:4093 + 123457], new, old)
        # the same source twice, and many small pieces
        pieces = [(ha, (37 * i) % 500000, 1 + i % 17) for i in range(64)]
        rc, h, n = bm.put_block_resealed(pieces, old, new)
        assert rc == BM.OK
        check_stored(bm, h, n, np.concatenate([pa[o:o + ln] for _, o, ln in pieces]), new, old)
        assert bm.reseal_metrics()["fallbacks"] == 0


def test_m_holders_down_and_stale_source_shard(tmp_path):
    with manager("rs", tmp_path) as bm:
        old, new = key_of(4), key_of(5)
        (h, p), (h2, p2) = put_sources(bm, 0x6E62, key=old, lens=[1 << 20, 54321])
        # m holders of the source lose their shards (the nodes stay up: the new block needs its write quorum)
        row = bm.storage_nodes_of(h)
        for i in range(4):
            assert bm.drop_shard(row[i], h) == BM.OK
        rc, hn, n = bm.put_block_resealed([(h, 0, p.size)], old, new)
        assert rc == BM.OK and bm.reseal_metrics()["fallbacks"] == 0
        check_stored(bm, hn, n, p, new, old)
        # a stale but self-consistent shard of the source: one fallback through rpc_get_block, which quarantines it
        row2 = bm.storage_nodes_of(h2)
        assert bm.plant_stale_shard(row2[3], h2) == BM.OK
        rc, hn, n = bm.put_block_resealed([(h2, 0, p2.size)], old, new)
        assert rc == BM.OK
        check_stored(bm, hn, n, p2, new, old)
        assert bm.reseal_metrics()["fallbacks"] == 1
        assert bm.block_info(h2)[1]["state"][3] in (BM.SHARD_QUARANTINED, BM.SHARD_ABSENT)
        rc, hn, n = bm.put_block_resealed([(h2, 5, 100)], old, new)  # the culprit is gone: no second fallback
        assert rc == BM.OK and bm.reseal_metrics()["fallbacks"] == 1


def test_source_held_only_under_a_previous_code(tmp_path):
    old, new = key_of(6), key_of(7)
    with BM.BlockManager(k=10, m=4, n_nodes=14, data_dir=str(tmp_path), batch_max_blocks=8) as bm:
        (h, p), = put_sources(bm, 0x6E63, key=old, lens=[200000])
    with BM.BlockManager(k=6, m=3, n_nodes=14, data_dir=str(tmp_path), batch_max_blocks=8,
                         previous_codes=[(10, 4, 0, 0)]) as bm:
        rc, hn, n = bm.put_block_resealed([(h, 0, p.size)], old, new)
        assert rc == BM.OK and bm.reseal_metrics()["fallbacks"] == 1
        check_stored(bm, hn, n, p, new, old)


def test_wrong_key_missing_source_and_refusals(tmp_path):
    with manager("rs", tmp_path) as bm:
        old, new = key_of(8), key_of(9)
        (h, p), = put_sources(bm, 0x6E64, key=old, lens=[100000])
        w0 = bm.metrics()["bytes_written"]
        rc, _, _ = bm.put_block_resealed([(h, 0, p.size)], key_of(10), new)
        assert rc == G.E_AUTH
        assert bm.reseal_metrics()["auth_failures"] == 1
        rc, _, _ = bm.put_block_resealed([(bytes(range(32)), 0, 10)], old, new)
        assert rc == BM.E_MISSING_BLOCK
        assert bm.metrics()["bytes_written"] == w0  # nothing was stored
        for pieces, dk in (([], new), ([(h, 0, 1)] * (BM.MAX_PIECES + 1), new), ([(h, 0, 1)], None),
                           ([(h, 0, 0)], new), ([(h, p.size - 5, 6)], new), ([(h, 0, p.size)] * 11, new)):
            rc, _, _ = bm.put_block_resealed(pieces, old, dk)
            assert rc == G.E_INVALID, (len(pieces), dk is None)
        assert bm.metrics()["bytes_written"] == w0


def test_concurrent_copies_batch_resync_deep_scrub_and_restart(tmp_path):
    old, new = key_of(11), key_of(12)
    with manager("rs", tmp_path, batch_max_blocks=32, batch_linger_us=2000) as bm:
        srcs = put_sources(bm, 0x6E65, key=old, lens=[20000 + 977 * i for i in range(32)])

        def copy(job):
            h, p = job
            return bm.put_block_resealed([(h, 0, p.size)], old, new)

        with ThreadPoolExecutor(32) as ex:
            res = list(ex.map(copy, srcs))
        for (h, p), (rc, hn, n) in zip(srcs, res):
            assert rc == BM.OK
            check_stored(bm, hn, n, p, new, None)
        m = bm.reseal_metrics()
        assert m["calls"] == 32 and m["batches"] < 32, m
        hn, n = res[0][1], res[0][2]
        rc, before = bm.rpc_get_block(hn, cap=SEALED_MAX)
        row = bm.storage_nodes_of(hn)
        assert bm.drop_shard(row[2], hn) == BM.OK
        assert bm.repair_enqueue_missing(row[2]) == 1
        assert bm.resync_all(row[2]) == (0, 1)
        assert bm.node_shard_index(row[2], hn) == 2
        for node in range(14):
            rc, _, finished, checked, repaired = bm.deep_scrub_step(node)
            assert rc == BM.OK and finished and repaired == 0
        assert bm.metrics()["deep_scrub_content_errors"] == 0
    with manager("rs", tmp_path) as bm:
        rc, after = bm.rpc_get_block(hn, cap=SEALED_MAX)
        assert rc == BM.OK and np.array_equal(after, before)
        check_stored(bm, hn, n, srcs[0][1], new, old)
