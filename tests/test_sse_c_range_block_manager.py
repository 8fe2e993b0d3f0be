"""Ranged SSE-C GETs in the block manager (garage_bm_rpc_get_block_range_opened, DESIGN.md 5.10) on file stores: for
every code a ranged opened GET equals the slice of rpc_get_block_opened -- healthy, with holders down, across two
active layout versions, under a previous code and after a restart -- a healthy 4 KiB range reads exactly the adler8 tag
spans of its planned runs, a stale shard in the span is served through one whole-block fallback and quarantined, and a
wrong key is GARAGE_EC_E_AUTH."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import oracle_lib as O  # noqa: E402

import garage_b200 as G  # noqa: E402
from garage_b200 import block_manager as BM  # noqa: E402

pytestmark = pytest.mark.gpu

CODES = {
    "rs10_4": dict(k=10, m=4),
    "lrc10_2_2": dict(k=10, m=4, local_groups=2),
    "pb10_4": dict(k=10, m=4, piggyback=True),
    "clay10_4": dict(k=10, m=4, clay=True),
    "rs4_2": dict(k=4, m=2),
}
SIZES = [1 << 20, (1 << 20) - 977, 300001]
FR = 4112


def key_of(i):
    return bytes((11 * i + 3 * j) & 0xFF for j in range(32))


def sealed_puts(bm, sizes, seed):
    out = []
    for i, n in enumerate(sizes):
        p = O.fill_random(n, seed + i)
        rc, h = bm.rpc_put_block_sealed(key_of(seed + i), p)
        assert rc == BM.OK
        out.append((h, p, key_of(seed + i)))
    return out


def ranges(P):
    rng = np.random.default_rng(P)
    out = [(0, 1), (4096 * 7, 4096), (4096 * 7 + 9, 4096), (P - 100, 100), (P // 3, 65536), (0, P), (P // 2, 0)]
    o = int(rng.integers(0, P))
    out.append((o, int(rng.integers(1, min(P - o, 200000) + 1))))
    return [(o, n) for o, n in out if o >= 0 and o + n <= P]


def assert_ranges(bm, puts):
    for h, p, key in puts:
        rc, whole = bm.rpc_get_block_opened(h, key)
        assert rc == BM.OK and np.array_equal(whole, p)
        for off, n in ranges(p.size):
            rc, got = bm.rpc_get_block_range_opened(h, key, off, n)
            assert rc == BM.OK and np.array_equal(got, whole[off:off + n]), (off, n)


def shard_of(off, L):
    """the data shard holding the first byte of plaintext offset off's chunk"""
    return (8 + FR * (off // 4096) + off % 4096) // L


@pytest.mark.parametrize("code", list(CODES))
def test_ranged_opened_get_equals_the_slice(tmp_path, code):
    kw = CODES[code]
    tot = kw["k"] + kw["m"]
    with BM.BlockManager(n_nodes=tot, data_dir=str(tmp_path / "s"), batch_max_blocks=8, **kw) as bm:
        puts = sealed_puts(bm, SIZES, 0x6A00)
        assert_ranges(bm, puts)
        m0 = bm.get_sealed_range_metrics()
        assert m0["degraded_gets"] == 0 and m0["fallbacks"] == 0 and m0["auth_failures"] == 0
        assert m0["gets"] == sum(len(ranges(p.size)) for _, p, _ in puts)
        # holders down: one data shard, a data shard and a parity (shard 0: the prefix is rebuilt), then m holders
        worst = [0, 5, 12, 13] if kw.get("local_groups") else list(range(kw["m"]))
        for idx in ([3], [0, kw["k"]], worst):
            for h, p, key in puts:
                row = bm.storage_nodes_of(h)
                for i in idx:
                    bm.set_node_up(row[i], False)
                for off, n in ranges(p.size):
                    rc, got = bm.rpc_get_block_range_opened(h, key, off, n)
                    assert rc == BM.OK and np.array_equal(got, p[off:off + n]), (code, idx, off, n)
                for i in idx:
                    bm.set_node_up(row[i], True)
        mt = bm.get_sealed_range_metrics()
        assert mt["degraded_gets"] > 0 and mt["fallbacks"] == 0 and mt["auth_failures"] == 0
        assert mt["bytes_fetched"] <= mt["bytes_read"] and mt["open_range_call_us"] > 0
        assert bm.metrics()["corruption_counter"] == 0
        rc, _ = bm.rpc_get_block_range_opened(puts[0][0], puts[0][2], SIZES[0] - 1, 2)
        assert rc == G.E_INVALID  # past the plaintext


def test_healthy_4k_range_reads_the_tag_spans_of_its_plan(tmp_path):
    with BM.BlockManager(k=10, m=4, n_nodes=14, data_dir=str(tmp_path / "s")) as bm:
        (h, p, key), = sealed_puts(bm, [1 << 20], 0x6B00)
        S = G.sealed_len(p.size)
        with G.GarageEc(0, 10, 4) as ec:
            L = ec.code_shard_len(S)
            for off in (4096 * 40, 4096 * 40 + 7, 4096 * 127 + 3000):
                runs, gpu = ec.open_range_plan(np.ones(14, dtype=np.uint8), S, off, 4096)
                assert gpu == 0
                lo, hi = {}, {}
                for sh, o, n in runs:
                    lo[sh] = min(lo.get(sh, o), o)
                    hi[sh] = max(hi.get(sh, 0), o + n)
                want_read = sum(G.tag_span(BM.SUM_ADLER8, L, lo[sh], hi[sh] - lo[sh])[1] for sh in lo)
                m0 = bm.get_sealed_range_metrics()
                rc, got = bm.rpc_get_block_range_opened(h, key, off, 4096)
                m1 = bm.get_sealed_range_metrics()
                assert rc == BM.OK and np.array_equal(got, p[off:off + 4096])
                assert m1["bytes_read"] - m0["bytes_read"] == want_read, off
                # the prefix and one sealed chunk when aligned, two when not
                assert m1["bytes_fetched"] - m0["bytes_fetched"] == sum(r[2] for r in runs) == (
                    8 + FR * (1 if off % 4096 == 0 else 2))
                assert m1["degraded_gets"] == m0["degraded_gets"]


def test_stale_shard_in_the_span_is_served_through_one_fallback(tmp_path):
    with BM.BlockManager(k=10, m=4, n_nodes=14, data_dir=str(tmp_path / "s")) as bm:
        (h, p, key), = sealed_puts(bm, [1 << 20], 0x6C00)
        L = -(-G.sealed_len(p.size) // 10)
        off = 4096 * 80 + 100
        i = shard_of(off, L)
        row = bm.storage_nodes_of(h)
        assert bm.plant_stale_shard(row[i], h) == BM.OK
        m0, c0 = bm.get_sealed_range_metrics(), bm.metrics()["corruption_counter"]
        rc, got = bm.rpc_get_block_range_opened(h, key, off, 4096)
        m1 = bm.get_sealed_range_metrics()
        assert rc == BM.OK and np.array_equal(got, p[off:off + 4096])
        assert m1["fallbacks"] - m0["fallbacks"] == 1 and m1["auth_failures"] == m0["auth_failures"]
        assert bm.metrics()["corruption_counter"] > c0  # the hunt quarantined the stale shard
        # quarantined: the next ranged GET rebuilds that shard's window and needs no fallback
        rc, got = bm.rpc_get_block_range_opened(h, key, off, 4096)
        m2 = bm.get_sealed_range_metrics()
        assert rc == BM.OK and np.array_equal(got, p[off:off + 4096])
        assert m2["fallbacks"] == m1["fallbacks"] and m2["degraded_gets"] == m1["degraded_gets"] + 1


def test_wrong_key_is_auth(tmp_path):
    with BM.BlockManager(k=10, m=4, n_nodes=14, data_dir=str(tmp_path / "s")) as bm:
        (h, p, key), = sealed_puts(bm, [300001], 0x6D00)
        m0 = bm.get_sealed_range_metrics()
        rc, got = bm.rpc_get_block_range_opened(h, bytes(32), 5000, 100)
        m1 = bm.get_sealed_range_metrics()
        assert rc == G.E_AUTH and got is None
        assert m1["auth_failures"] == m0["auth_failures"] + 1
        assert bm.metrics()["corruption_counter"] == 0  # nothing was stale: nothing quarantined
        rc, got = bm.rpc_get_block_range_opened(h, key, 5000, 100)
        assert rc == BM.OK and np.array_equal(got, p[5000:5100])


def test_ranged_opened_get_during_a_layout_change(tmp_path):
    n, cap = 16, 1 << 40
    with BM.BlockManager(k=10, m=4, n_nodes=n, data_dir=str(tmp_path / "s"), batch_max_blocks=8,
                         layout=dict(zone=[0] * n, capacity=[cap] * 14 + [0, 0])) as bm:
        puts = sealed_puts(bm, SIZES, 0x6E00)
        assert bm.apply_layout([0] * n, [cap] * n)[0] == BM.OK
        assert bm.layout_versions() == [1, 2]
        puts += sealed_puts(bm, [777777], 0x6E10)
        assert_ranges(bm, puts)
        h, p, key = puts[0]
        down = bm.storage_nodes_of(h)[2]
        bm.set_node_up(down, False)
        for off, ln in ranges(p.size):
            rc, got = bm.rpc_get_block_range_opened(h, key, off, ln)
            assert rc == BM.OK and np.array_equal(got, p[off:off + ln])
        bm.set_node_up(down, True)


def test_block_under_a_previous_code_and_restart(tmp_path):
    d = str(tmp_path / "s")
    with BM.BlockManager(k=6, m=3, n_nodes=14, data_dir=d, batch_max_blocks=8) as old:
        old_puts = sealed_puts(old, SIZES, 0x6F00)
    with BM.BlockManager(k=10, m=4, n_nodes=14, data_dir=d, batch_max_blocks=8, previous_codes=[(6, 3, 0, 0)]) as bm:
        for h, p, key in old_puts:
            for off, ln in ranges(p.size):
                rc, got = bm.rpc_get_block_range_opened(h, key, off, ln)
                assert rc == BM.OK and np.array_equal(got, p[off:off + ln])
        assert bm.metrics()["legacy_gets"] > 0
        new_puts = sealed_puts(bm, SIZES, 0x6F10)
    with BM.BlockManager(k=10, m=4, n_nodes=14, data_dir=d, batch_max_blocks=8, previous_codes=[(6, 3, 0, 0)]) as bm:
        for h, p, key in new_puts:
            for off, ln in ranges(p.size):
                rc, got = bm.rpc_get_block_range_opened(h, key, off, ln)
                assert rc == BM.OK and np.array_equal(got, p[off:off + ln])
        assert bm.get_sealed_range_metrics()["fallbacks"] == 0
