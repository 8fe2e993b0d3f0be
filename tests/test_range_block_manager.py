"""Ranged GETs in the block manager (garage_bm_rpc_get_block_range): for every code the bytes equal the slice of
rpc_get_block -- healthy, with holders down, across two active layout versions and for a block still under a previous
code -- a healthy range reads only the adler8 tag spans it needs and no GPU, a flipped byte in a read span is caught,
and a BLAKE2 store reads whole touched shards."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import oracle_lib as O  # noqa: E402

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


def put(bm, sizes, seed):
    blocks = [O.fill_random(n, seed + i) for i, n in enumerate(sizes)]
    hashes = [BM.blake2sum(b) for b in blocks]
    for h, b in zip(hashes, blocks):
        assert bm.rpc_put_block(h, b) == BM.OK
    return blocks, hashes


def ranges(B, L):
    rng = np.random.default_rng(B)
    out = [(0, 1), (L - 5, 10), (B - 100, 100), (B // 3, 4096), (0, B), (L // 2 - 7, 20), (3 * L + 1000, 4096)]
    o = int(rng.integers(0, B))
    out.append((o, int(rng.integers(1, B - o + 1))))
    return [(o, n) for o, n in out if o >= 0 and n >= 1 and o + n <= B]


def assert_ranges(bm, blocks, hashes, shard_len):
    for h, b in zip(hashes, blocks):
        rc, whole = bm.rpc_get_block(h)
        assert rc == BM.OK and np.array_equal(whole, b)
        for off, n in ranges(b.size, shard_len(b.size)):
            rc, got = bm.rpc_get_block_range(h, off, n)
            assert rc == BM.OK and np.array_equal(got, b[off:off + n]), (off, n)


def L_of(kw):
    import garage_b200 as G

    with (G.GarageEc.clay(0, kw["k"], kw["m"]) if kw.get("clay") else
          G.GarageEc.piggyback(0, kw["k"], kw["m"]) if kw.get("piggyback") else G.GarageEc(0, kw["k"], kw["m"])) as ec:
        return {B: ec.code_shard_len(B) for B in SIZES}


@pytest.mark.parametrize("code", list(CODES))
def test_ranged_get_equals_the_slice(tmp_path, code):
    kw = CODES[code]
    Ls = L_of(kw)
    tot = kw["k"] + kw["m"]
    with BM.BlockManager(n_nodes=tot, data_dir=str(tmp_path / "s"), batch_max_blocks=8, **kw) as bm:
        blocks, hashes = put(bm, SIZES, 0x5A00)
        assert_ranges(bm, blocks, hashes, Ls.get)
        m0 = bm.metrics()
        assert m0["range_degraded"] == 0 and m0["corruption_counter"] == 0
        # holders down: one data shard (LRC: repaired in its group; PB: rule 1; Clay: the single-loss repair), a data
        # shard and a parity, then m holders
        # (LRC is not MDS: its m-loss pattern takes one data shard of each group and both global parities)
        worst = [0, 5, 12, 13] if kw.get("local_groups") else list(range(kw["m"]))
        for idx in ([3], [1, kw["k"]], worst):
            for h in hashes:
                for i in idx:
                    bm.set_node_up(bm.storage_nodes_of(h)[i], False)
                for b, hh in zip(blocks, hashes):
                    if hh != h:
                        continue
                    for off, n in ranges(b.size, Ls[b.size]):
                        rc, got = bm.rpc_get_block_range(h, off, n)
                        assert rc == BM.OK and np.array_equal(got, b[off:off + n]), (code, idx, off, n)
                for i in idx:
                    bm.set_node_up(bm.storage_nodes_of(h)[i], True)
        mt = bm.metrics()
        assert mt["range_degraded"] > 0 and mt["corruption_counter"] == 0
        assert mt["range_bytes_fetched"] <= mt["range_bytes_read"]
        rc, _ = bm.rpc_get_block_range(hashes[0], SIZES[0] - 1, 2)
        assert rc == -1  # GARAGE_EC_E_INVALID: past the block


def test_healthy_4k_range_reads_two_segments_and_no_gpu(tmp_path):
    with BM.BlockManager(k=10, m=4, n_nodes=14, data_dir=str(tmp_path / "s")) as bm:
        blocks, hashes = put(bm, [1 << 20], 0x5B00)
        b, h = blocks[0], hashes[0]
        L, seg = 104858, 13120
        for off in (3 * L + seg - 2000, 4 * L - 2000):  # across a segment boundary; across a shard boundary
            m0 = bm.metrics()
            rc, got = bm.rpc_get_block_range(h, off, 4096)
            m1 = bm.metrics()
            assert rc == BM.OK and np.array_equal(got, b[off:off + 4096])
            assert m1["range_bytes_read"] - m0["range_bytes_read"] <= 2 * seg
            assert m1["range_bytes_fetched"] - m0["range_bytes_fetched"] == 4096
            assert m1["range_degraded"] == m0["range_degraded"] == 0
            assert m1["reconstruct_calls"] == m0["reconstruct_calls"]
            assert m1["range_gets"] == m0["range_gets"] + 1


def test_flipped_byte_in_a_read_span_is_caught(tmp_path):
    with BM.BlockManager(k=10, m=4, n_nodes=14, data_dir=str(tmp_path / "s")) as bm:
        blocks, hashes = put(bm, [1 << 20], 0x5C00)
        b, h = blocks[0], hashes[0]
        L = 104858
        node = bm.storage_nodes_of(h)[3]
        assert bm.corrupt_shard(node, h, 1500) == 0
        m0 = bm.metrics()
        rc, got = bm.rpc_get_block_range(h, 3 * L + 1000, 4096)
        m1 = bm.metrics()
        assert rc == BM.OK and np.array_equal(got, b[3 * L + 1000:3 * L + 5096])
        assert m1["corruption_counter"] == m0["corruption_counter"] + 1
        assert m1["range_degraded"] == m0["range_degraded"] + 1
        assert m1["resync_queue_length"] >= 1
        rc, got = bm.rpc_get_block_range(h, 3 * L + 1000, 4096)  # quarantined: rebuilt again, nothing new caught
        assert rc == BM.OK and np.array_equal(got, b[3 * L + 1000:3 * L + 5096])
        assert bm.metrics()["corruption_counter"] == m1["corruption_counter"]


def test_blake2_store_reads_whole_touched_shards(tmp_path):
    with BM.BlockManager(k=10, m=4, n_nodes=14, data_dir=str(tmp_path / "s"), shard_sum_kind=BM.SUM_BLAKE2) as bm:
        blocks, hashes = put(bm, [1 << 20], 0x5D00)
        b, h = blocks[0], hashes[0]
        L = 104858
        m0 = bm.metrics()
        rc, got = bm.rpc_get_block_range(h, 2 * L + 77, 4096)
        m1 = bm.metrics()
        assert rc == BM.OK and np.array_equal(got, b[2 * L + 77:2 * L + 77 + 4096])
        assert m1["range_bytes_read"] - m0["range_bytes_read"] == L
        rc, got = bm.rpc_get_block_range(h, 3 * L - 10, 20)
        assert rc == BM.OK and np.array_equal(got, b[3 * L - 10:3 * L + 10])
        assert bm.metrics()["range_bytes_read"] - m1["range_bytes_read"] == 2 * L


def test_ranged_get_during_a_layout_change(tmp_path):
    n, cap = 16, 1 << 40
    cap14 = [cap] * 14 + [0, 0]
    with BM.BlockManager(k=10, m=4, n_nodes=n, data_dir=str(tmp_path / "s"), batch_max_blocks=8,
                         layout=dict(zone=[0] * n, capacity=cap14)) as bm:
        blocks, hashes = put(bm, SIZES, 0x5E00)
        assert bm.apply_layout([0] * n, [cap] * n)[0] == BM.OK
        assert bm.layout_versions() == [1, 2]
        more_b, more_h = put(bm, [777777], 0x5E10)
        assert_ranges(bm, blocks + more_b, hashes + more_h, lambda B: -(-B // 10))
        h = hashes[0]
        down = bm.storage_nodes_of(h)[2]  # a holder of the newest version down: its index comes from another source
        bm.set_node_up(down, False)
        for off, ln in ranges(SIZES[0], 104858):
            rc, got = bm.rpc_get_block_range(h, off, ln)
            assert rc == BM.OK and np.array_equal(got, blocks[0][off:off + ln])
        bm.set_node_up(down, True)


def test_block_under_a_previous_code_is_sliced(tmp_path):
    d = str(tmp_path / "s")
    with BM.BlockManager(k=6, m=3, n_nodes=14, data_dir=d, batch_max_blocks=8) as old:
        blocks, hashes = put(old, SIZES, 0x5F00)
    with BM.BlockManager(k=10, m=4, n_nodes=14, data_dir=d, batch_max_blocks=8, previous_codes=[(6, 3, 0, 0)]) as bm:
        for h, b in zip(hashes, blocks):
            for off, ln in ranges(b.size, -(-b.size // 10)):
                rc, got = bm.rpc_get_block_range(h, off, ln)
                assert rc == BM.OK and np.array_equal(got, b[off:off + ln])
        assert bm.metrics()["legacy_gets"] > 0
