"""SSE-C through the block manager (DESIGN.md 5.9) on file stores of RS(10,4) and Clay(10,4): a sealed PUT stores the
oracle's seal of the plaintext under the nonce in its first 8 bytes and returns its content address; the opened GET
returns the plaintext with m holders down and no fallback; a planted stale shard is found through one fallback; a
wrong key is GARAGE_EC_E_AUTH; a dropped shard resyncs byte-identical and the deep scrub is clean; sealed blocks
survive a restart; concurrent sealed and plain PUTs batch together."""
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
CODES = {"rs": {}, "clay": {"clay": True}}
LENS = [1 << 20, 1, 4096, 4097, 54321]


def manager(code, d, **kw):
    kw.setdefault("batch_max_blocks", 8)
    return BM.BlockManager(k=10, m=4, n_nodes=14, data_dir=str(d), **CODES[code], **kw)


def key_of(i):
    return bytes((7 * i + j) & 0xFF for j in range(32))


def sealed_puts(bm, seed):
    out = []
    for i, n in enumerate(LENS):
        p = O.fill_random(n, seed + i)
        rc, h = bm.rpc_put_block_sealed(key_of(i), p)
        assert rc == BM.OK
        out.append((h, p, key_of(i)))
    return out


@pytest.mark.parametrize("code", list(CODES))
def test_sealed_put_stores_the_oracle_seal_and_opens_degraded(code, tmp_path):
    with manager(code, tmp_path) as bm:
        puts = sealed_puts(bm, 0x5EA1)
        for h, p, key in puts:
            rc, b = bm.rpc_get_block(h, cap=G.sealed_len(1 << 20))
            assert rc == BM.OK and len(b) == G.sealed_len(p.size)
            assert BM.blake2sum(b) == h
            assert b.tobytes() == S.seal(key, b[:8].tobytes(), p)
        m0 = bm.sealed_metrics()
        assert m0["sealed_puts"] == len(LENS) and m0["sealed_batches"] >= 1
        for h, p, key in puts:
            row = bm.storage_nodes_of(h)
            for i in range(4):
                bm.set_node_up(row[i], False)
            rc, got = bm.rpc_get_block_opened(h, key)
            assert rc == BM.OK and np.array_equal(got, p)
            for i in range(4):
                bm.set_node_up(row[i], True)
        m1 = bm.sealed_metrics()
        assert m1["opened_gets"] - m0["opened_gets"] == len(LENS)
        assert m1["opened_fallbacks"] == m0["opened_fallbacks"] == 0
        # a wrong key fails authentication
        h, p, key = puts[0]
        rc, got = bm.rpc_get_block_opened(h, bytes(32))
        assert rc == G.E_AUTH and got is None
        assert bm.sealed_metrics()["opened_auth_failures"] == 1
        # a plaintext PUT through the same call
        p = O.fill_random(3000, 99)
        rc, h = bm.rpc_put_block_sealed(None, p)
        assert rc == BM.OK and h == BM.blake2sum(p)
        rc, got = bm.rpc_get_block(h)
        assert rc == BM.OK and np.array_equal(got, p)


@pytest.mark.parametrize("code", list(CODES))
def test_stale_shard_found_through_one_fallback(code, tmp_path):
    with manager(code, tmp_path) as bm:
        h, p, key = sealed_puts(bm, 0x5EA2)[4]
        row = bm.storage_nodes_of(h)
        assert bm.plant_stale_shard(row[3], h) == BM.OK
        m0 = bm.sealed_metrics()
        rc, got = bm.rpc_get_block_opened(h, key)
        assert rc == BM.OK and np.array_equal(got, p)
        assert bm.sealed_metrics()["opened_fallbacks"] - m0["opened_fallbacks"] == 1


@pytest.mark.parametrize("code", list(CODES))
def test_sealed_shard_resyncs_and_deep_scrub_is_clean_and_restart(code, tmp_path):
    with manager(code, tmp_path) as bm:
        puts = sealed_puts(bm, 0x5EA3)
        h, p, key = puts[0]
        row = bm.storage_nodes_of(h)
        rc, before = bm.rpc_get_block(h, cap=G.sealed_len(1 << 20))
        assert rc == BM.OK
        assert bm.drop_shard(row[2], h) == BM.OK
        assert bm.repair_enqueue_missing(row[2]) == 1
        failed, done = bm.resync_all(row[2])
        assert (failed, done) == (0, 1)
        assert bm.node_shard_index(row[2], h) == 2
        for node in range(14):
            rc, _, finished, checked, repaired = bm.deep_scrub_step(node)
            assert rc == BM.OK and finished and repaired == 0
        assert bm.metrics()["deep_scrub_content_errors"] == 0
    with manager(code, tmp_path) as bm:
        for h, p, key in puts:
            rc, got = bm.rpc_get_block_opened(h, key)
            assert rc == BM.OK and np.array_equal(got, p)
        rc, after = bm.rpc_get_block(puts[0][0], cap=G.sealed_len(1 << 20))
        assert rc == BM.OK and np.array_equal(after, before)


def test_concurrent_sealed_and_plain_puts_batch_together(tmp_path):
    with manager("rs", tmp_path, batch_max_blocks=16) as bm:
        jobs = []
        for i in range(48):
            p = O.fill_random(20000 + 977 * i, 0x5EA4 + i)
            jobs.append((i % 3, p))

        def put(job):
            kind, p = job
            if kind == 0:
                h = BM.blake2sum(p)
                return bm.rpc_put_block(h, p), h, None
            key = key_of(kind * 100) if kind == 1 else None
            rc, h = bm.rpc_put_block_sealed(key, p)
            return rc, h, key

        with ThreadPoolExecutor(16) as ex:
            res = list(ex.map(put, jobs))
        for (kind, p), (rc, h, key) in zip(jobs, res):
            assert rc == BM.OK
            if key is None:
                rc, got = bm.rpc_get_block(h)
            else:
                rc, got = bm.rpc_get_block_opened(h, key)
            assert rc == BM.OK and np.array_equal(got, p), kind
        assert bm.sealed_metrics()["sealed_puts"] == 32
