"""Every kind of reconstruct item in one dispatcher batch (DESIGN.md 5.5, 5.9, 5.10): a degraded whole GET, a degraded
ranged GET, opened GETs with the right and a wrong key and a ranged opened GET with a wrong key, submitted concurrently
under a long batch linger, share a batch and each gets its kind's result and bytes; a GET of a block with too few
shards is GARAGE_BM_E_MISSING_BLOCK.  The range, sealed-range and opened counters move by exactly what each request
implies."""
import os
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import oracle_lib as O  # noqa: E402

import garage_b200 as G  # noqa: E402
from garage_b200 import block_manager as BM  # noqa: E402

pytestmark = pytest.mark.gpu
K, M, B = 10, 4, 1 << 20
LOST = 3  # the data shard dropped from the degraded block


def tag_span_bytes(runs, L):
    """the adler8 tag-span bytes a gather reads for these runs: one span per shard, covering all of its runs"""
    lo, hi = {}, {}
    for sh, o, n in runs:
        lo[sh] = min(lo.get(sh, o), o)
        hi[sh] = max(hi.get(sh, 0), o + n)
    return sum(G.tag_span(BM.SUM_ADLER8, L, lo[sh], hi[sh] - lo[sh])[1] for sh in lo)


def test_every_item_kind_shares_one_batch(tmp_path):
    # a linger far longer than the gathers: the concurrent requests' items meet in one batch
    with BM.BlockManager(k=K, m=M, n_nodes=K + M, data_dir=str(tmp_path / "s"), batch_max_blocks=16,
                         batch_linger_us=500_000) as bm:
        a = O.fill_random(B, 0xD150)
        ha = BM.blake2sum(a)
        c = O.fill_random(B // 2, 0xD151)
        hc = BM.blake2sum(c)
        assert bm.rpc_put_block(ha, a) == BM.OK and bm.rpc_put_block(hc, c) == BM.OK
        key, wrong = bytes(range(32)), bytes(32)
        p = O.fill_random(300001, 0xD152)
        rc, hs = bm.rpc_put_block_sealed(key, p)
        assert rc == BM.OK
        assert bm.drop_shard(bm.storage_nodes_of(ha)[LOST], ha) == BM.OK  # a missing data shard: both GETs of a rebuild
        for i in range(M + 1):  # one shard more than the code can lose
            assert bm.drop_shard(bm.storage_nodes_of(hc)[i], hc) == BM.OK

        S = G.sealed_len(p.size)
        with G.GarageEc(0, K, M) as ec:
            L, Ls = ec.code_shard_len(B), ec.code_shard_len(S)
            off, ln = LOST * L + 1000, 4096  # inside the dropped shard
            present = np.ones(K + M, dtype=np.uint8)
            present[LOST] = 0
            runs, gpu = ec.range_plan(present, B, off, ln)
            assert gpu == 1
            soff, sln = 4096 * 20 + 5, 4096
            sruns, sgpu = ec.open_range_plan(np.ones(K + M, dtype=np.uint8), S, soff, sln)
            assert sgpu == 0

        requests = {
            "whole": lambda: bm.rpc_get_block(ha),
            "range": lambda: bm.rpc_get_block_range(ha, off, ln),
            "open": lambda: bm.rpc_get_block_opened(hs, key),
            "open_wrong_key": lambda: bm.rpc_get_block_opened(hs, wrong),
            "open_range_wrong_key": lambda: bm.rpc_get_block_range_opened(hs, wrong, soff, sln),
            "too_few_shards": lambda: bm.rpc_get_block(hc),
        }
        m0, s0, o0 = bm.metrics(), bm.get_sealed_range_metrics(), bm.sealed_metrics()
        with ThreadPoolExecutor(len(requests)) as pool:
            futs = {name: pool.submit(f) for name, f in requests.items()}
            got = {name: f.result() for name, f in futs.items()}
        m1, s1, o1 = bm.metrics(), bm.get_sealed_range_metrics(), bm.sealed_metrics()

        # rebuild and range: status 0 -> OK; open: OK with the plaintext, a wrong key GARAGE_EC_E_AUTH; open-range:
        # GARAGE_EC_E_AUTH, confirmed by one whole-block opened GET
        assert got["whole"][0] == BM.OK and np.array_equal(got["whole"][1], a)
        assert got["range"][0] == BM.OK and np.array_equal(got["range"][1], a[off:off + ln])
        assert got["open"][0] == BM.OK and np.array_equal(got["open"][1], p)
        assert got["open_wrong_key"] == (G.E_AUTH, None)
        assert got["open_range_wrong_key"] == (G.E_AUTH, None)
        assert got["too_few_shards"] == (BM.E_MISSING_BLOCK, None)

        # five items reach the dispatchers together and the ranged opened GET's whole-block re-check follows them: two
        # batches when the five share one, and fewer than the five alone would take apart
        batches = m1["reconstruct_batches"] - m0["reconstruct_batches"]
        assert 2 <= batches < 5, batches
        assert m1["reconstruct_calls"] - m0["reconstruct_calls"] == 1  # the degraded whole GET's rebuild
        assert m1["corruption_counter"] == m0["corruption_counter"]  # nothing stale, nothing quarantined

        assert {n: m1[n] - m0[n] for n, _ in BM.RangeMetrics._fields_} == {
            "range_gets": 1, "range_degraded": 1, "range_bytes_read": tag_span_bytes(runs, L),
            "range_bytes_fetched": sum(r[2] for r in runs)}
        ds = {n: s1[n] - s0[n] for n in s0 if not n.endswith("call_us")}
        assert ds == {"gets": 1, "degraded_gets": 0, "bytes_read": tag_span_bytes(sruns, Ls),
                      "bytes_fetched": sum(r[2] for r in sruns), "auth_failures": 1, "fallbacks": 1}
        assert s1["open_range_call_us"] > s0["open_range_call_us"] and o1["open_call_us"] > o0["open_call_us"]
        do = {n: o1[n] - o0[n] for n in o0 if not n.endswith("call_us")}
        assert do == {"sealed_puts": 0, "sealed_batches": 0, "opened_gets": 1, "opened_auth_failures": 2,
                      "opened_fallbacks": 0}
