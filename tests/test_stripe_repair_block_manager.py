"""garage_bm_stripe_repair_step on RS(10,4), LRC(10,2,2), PB(10,4), Clay(10,4) and RS(4,2) file stores with ragged
blocks: after e <= m-1 holders missed the PUTs, one sweep of the owners rebuilds every lost shard from one read of the
survivors (the rebuilt shards then serve degraded GETs and pass the deep scrub); its traffic per stripe is the code's
own plan for want = the lost shards, 1/e of the per-node resync path for RS and Clay and never more for any code; a
second sweep and the resync queues find nothing to do; min_missing orders the repair; down and read-only holders,
a corrupt survivor, an unrecoverable stripe and a stop mid-sweep; owners and resync workers running together; the
rejected calls."""
import os
import sys
import threading

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
NBLOCKS = 9
E_INVALID = -1
DOWN_ORDER = [1, 5, 9]  # the holders that miss the PUTs, first e of them


def manager(tmp_path, name, kw, **extra):
    extra.setdefault("batch_max_blocks", 4)
    return BM.BlockManager(n_nodes=kw["k"] + kw["m"], data_dir=str(tmp_path / name), **kw, **extra)


def ec_of(kw):
    import garage_b200 as G

    if kw.get("clay"):
        return G.GarageEc.clay(0, kw["k"], kw["m"])
    if kw.get("piggyback"):
        return G.GarageEc.piggyback(0, kw["k"], kw["m"])
    if kw.get("local_groups"):
        return G.GarageEc.lrc(0, kw["k"], kw["local_groups"], kw["m"] - kw["local_groups"])
    return G.GarageEc(0, kw["k"], kw["m"])


def blocks_of(seed, n=NBLOCKS):
    blocks = [O.fill_random(SIZES[i % len(SIZES)], seed + i) for i in range(n)]
    return blocks, [BM.blake2sum(b) for b in blocks]


def put_with_down(bm, blocks, hashes, down, incref=False):
    """PUT every block while the nodes `down` are down (the write quorum holds), then bring them back"""
    for d in down:
        bm.set_node_up(d, False)
    for h, b in zip(hashes, blocks):
        assert bm.rpc_put_block(h, b) == BM.OK
        if incref:
            bm.block_incref(h)  # queues a resync of h on every holder, the down ones included
    for d in down:
        bm.set_node_up(d, True)


def all_valid(bm, hashes):
    return all(bm.node_shard_index(n, h) == i for h in hashes for i, n in enumerate(bm.storage_nodes_of(h)))


def missing_of(bm, h):
    return [i for i, n in enumerate(bm.storage_nodes_of(h)) if bm.node_shard_index(n, h) != i]


def plan_bytes(ec, present, want, L):
    runs = ec.read_ranges(np.array(present, np.uint8), L, np.array(want, np.uint8))
    assert runs is not None
    return sum(n for _, _, n in runs)


def deep_scrub_clean(bm):
    m0 = bm.metrics()
    for node in range(bm.n_nodes):
        rc, _, finished, _, _ = bm.deep_scrub_step(node)
        assert rc == BM.OK and finished
    m1 = bm.metrics()
    for key in ("deep_scrub_parity_bad", "deep_scrub_content_errors", "deep_scrub_skipped"):
        assert m1[key] == m0[key], key
    return m1["deep_scrub_blocks"] - m0["deep_scrub_blocks"]


def per_node_resync(bm, down):
    """the per-node repair: each returning node enqueues and resyncs its missing shards while the other returning
    nodes' shards are still missing (as when they come back together and resync concurrently)"""
    for d in down:
        bm.set_node_up(d, False)
    done = 0
    for d in down:
        bm.set_node_up(d, True)
        bm.repair_enqueue_missing(d)
        failed, n = bm.resync_all(d)
        assert failed == 0
        done += n
        bm.set_node_up(d, False)
    for d in down:
        bm.set_node_up(d, True)
    return done


@pytest.mark.parametrize("code", list(CODES))
def test_one_sweep_rebuilds_every_lost_shard(tmp_path, code):
    kw = CODES[code]
    m = kw["m"]
    for e in range(1, m):
        blocks, hashes = blocks_of(0x7A00 + 16 * e)
        down = DOWN_ORDER[:e]
        with manager(tmp_path, "s%d" % e, kw) as bm:
            put_with_down(bm, blocks, hashes, down, incref=True)
            assert all(len(missing_of(bm, h)) == e for h in hashes)
            assert bm.stripe_repair_all() == (NBLOCKS, e * NBLOCKS)
            s = bm.stripe_repair_metrics()
            assert s["stripe_repairs"] == NBLOCKS and s["stripe_repair_shards"] == e * NBLOCKS
            assert s["stripe_repair_errors"] == 0 and s["stripe_repair_call_us"] > 0
            assert s["stripe_repair_bytes_fetched"] <= s["stripe_repair_bytes_read"]
            assert all_valid(bm, hashes)
            # m other holders down (LRC: m-1, the losses it decodes whatever their pattern): the GETs need the rebuilt
            others = [n for n in range(bm.n_nodes) if n not in down][: m - 1 if kw.get("local_groups") else m]
            for n in others:
                bm.set_node_up(n, False)
            for h, b in zip(hashes, blocks):
                rc, got = bm.rpc_get_block(h)
                assert rc == BM.OK and np.array_equal(got, b), (code, e)
            for n in others:
                bm.set_node_up(n, True)
            assert deep_scrub_clean(bm) == NBLOCKS
            # idempotence: nothing left to rebuild, and the resync queues (filled by the increfs) only drain
            m0, s0 = bm.metrics(), bm.stripe_repair_metrics()
            assert bm.stripe_repair_all() == (0, 0)
            assert bm.stripe_repair_metrics() == s0
            assert bm.metrics()["bytes_written"] == m0["bytes_written"]
            assert m0["resync_queue_length"] > 0
            for d in down:
                bm.repair_enqueue_missing(d)
                assert bm.resync_all(d) == (0, NBLOCKS)
            m1 = bm.metrics()
            for key in ("resync_counter", "resync_error_counter", "resync_recv_counter", "resync_shards_read",
                        "resync_bytes_read", "resync_bytes_fetched", "reconstruct_calls", "bytes_written"):
                assert m1[key] == m0[key], key
            assert m1["resync_queue_length"] == m0["resync_queue_length"] - len(down) * NBLOCKS


@pytest.mark.parametrize("code", list(CODES))
def test_traffic_is_the_codes_plan_once_per_stripe(tmp_path, code):
    kw = CODES[code]
    with ec_of(kw) as ec:
        for e in range(1, kw["m"]):
            blocks, hashes = blocks_of(0x7B00 + 16 * e)
            down = DOWN_ORDER[:e]
            with manager(tmp_path, "a%d" % e, kw) as bm:
                put_with_down(bm, blocks, hashes, down)
                expect = {}
                for h, b in zip(hashes, blocks):
                    present = [0 if n in down else 1 for n in bm.storage_nodes_of(h)]
                    expect[h] = plan_bytes(ec, present, [1 - p for p in present], ec.code_shard_len(b.size))
                # one block per step: each step's traffic is that stripe's plan
                seen = 0
                for node in range(bm.n_nodes):
                    cursor, finished = None, False
                    while not finished:
                        s0 = bm.stripe_repair_metrics()
                        rc, cursor, finished, rep, reb = bm.stripe_repair_step(node, cursor, max_blocks=1)
                        assert rc == BM.OK
                        if rep == 0:
                            continue
                        assert (rep, reb) == (1, e) and cursor in expect
                        s1 = bm.stripe_repair_metrics()
                        assert s1["stripe_repair_bytes_fetched"] - s0["stripe_repair_bytes_fetched"] == expect.pop(cursor)
                        seen += 1
                assert seen == NBLOCKS and not expect
                stripe = bm.stripe_repair_metrics()["stripe_repair_bytes_fetched"]
                assert all_valid(bm, hashes)
            with manager(tmp_path, "b%d" % e, kw) as bm:
                put_with_down(bm, blocks, hashes, down)
                assert per_node_resync(bm, down) == e * NBLOCKS
                per_node = bm.metrics()["resync_bytes_fetched"]
                assert all_valid(bm, hashes)
            assert stripe <= per_node, (code, e)
            if e == 1 or not (kw.get("local_groups") or kw.get("piggyback")):
                assert e * stripe == per_node, (code, e, stripe, per_node)


@pytest.mark.parametrize("code", ["rs10_4", "lrc10_2_2", "pb10_4", "clay10_4"])
def test_min_missing_repairs_the_most_degraded_first(tmp_path, code):
    kw = CODES[code]
    blocks, hashes = blocks_of(0x7C00)
    with manager(tmp_path, "s", kw) as bm:
        for h, b in zip(hashes, blocks):
            assert bm.rpc_put_block(h, b) == BM.OK
        lost = {}
        for j, h in enumerate(hashes):
            who = bm.storage_nodes_of(h)
            lost[h] = [3, 11, 7][: 1 + j % 3]
            for i in lost[h]:
                assert bm.drop_shard(who[i], h) == BM.OK
        for threshold in (4, 3, 2, 1):
            assert bm.stripe_repair_all(min_missing=threshold) == (
                (0, 0) if threshold == 4 else (NBLOCKS // 3, threshold * NBLOCKS // 3))
            for h in hashes:
                assert missing_of(bm, h) == ([] if len(lost[h]) >= threshold else sorted(lost[h])), threshold
        assert bm.stripe_repair_metrics()["stripe_repair_errors"] == 0
        assert deep_scrub_clean(bm) == NBLOCKS


def test_down_target_waits_for_a_later_sweep(tmp_path):
    kw = CODES["rs10_4"]
    blocks, hashes = blocks_of(0x7D00)
    with manager(tmp_path, "s", kw) as bm:
        put_with_down(bm, blocks, hashes, [1, 5])
        bm.set_node_up(5, False)
        assert bm.stripe_repair_all() == (NBLOCKS, NBLOCKS)
        assert bm.stripe_repair_metrics()["stripe_repair_errors"] == 0
        bm.set_node_up(5, True)
        assert all(missing_of(bm, h) == [bm.storage_nodes_of(h).index(5)] for h in hashes)
        assert bm.stripe_repair_all() == (NBLOCKS, NBLOCKS)
        assert bm.stripe_repair_metrics()["stripe_repair_errors"] == 0
        assert all_valid(bm, hashes)


@pytest.mark.parametrize("code", list(CODES))
def test_corrupt_survivor_is_quarantined_and_rebuilt(tmp_path, code):
    kw = CODES[code]
    blocks, hashes = blocks_of(0x7E00, 3)
    with ec_of(kw) as ec, manager(tmp_path, "s", kw) as bm:
        put_with_down(bm, blocks, hashes, [5])
        for h, b in zip(hashes, blocks):
            who = bm.storage_nodes_of(h)
            present = np.array([0 if n == 5 else 1 for n in who], np.uint8)
            plan = ec.read_plan(present, 1 - present) if kw.get("piggyback") else ec.read_set(present, 1 - present) * 3
            x = next(i for i in range(len(who)) if plan[i])  # a survivor the plan reads
            L = ec.code_shard_len(b.size)
            assert bm.corrupt_shard(who[x], h, 1 if plan[x] & 1 else L // 2 + 1) == BM.OK
        m0 = bm.metrics()
        assert bm.stripe_repair_all() == (3, 6)
        assert bm.metrics()["corruption_counter"] == m0["corruption_counter"] + 3
        assert bm.stripe_repair_metrics()["stripe_repair_errors"] == 0
        assert all_valid(bm, hashes)
        assert deep_scrub_clean(bm) == 3
        for h, b in zip(hashes, blocks):
            rc, got = bm.rpc_get_block(h)
            assert rc == BM.OK and np.array_equal(got, b)


def _files(root):
    out = {}
    for d, _, fs in os.walk(root):
        for f in fs:
            st = os.stat(os.path.join(d, f))
            out[os.path.join(d, f)] = (st.st_size, st.st_mtime_ns)
    return out


def test_unrecoverable_stripe_is_an_error_and_changes_no_file(tmp_path):
    kw = CODES["rs10_4"]
    blocks, hashes = blocks_of(0x7F00, 2)
    with manager(tmp_path, "s", kw) as bm:
        for h, b in zip(hashes, blocks):
            assert bm.rpc_put_block(h, b) == BM.OK
        who = bm.storage_nodes_of(hashes[0])
        for i in range(5):  # m + 1 lost
            assert bm.drop_shard(who[i], hashes[0]) == BM.OK
        before = _files(tmp_path / "s")
        assert bm.stripe_repair_all() == (0, 0)
        assert _files(tmp_path / "s") == before
        s = bm.stripe_repair_metrics()
        assert s["stripe_repair_errors"] == 1 and s["stripe_repair_bytes_written"] == 0


def test_read_only_target_is_an_error_and_the_others_are_written(tmp_path):
    kw = CODES["rs10_4"]
    blocks, hashes = blocks_of(0x8000)
    with manager(tmp_path, "s", kw) as bm:
        put_with_down(bm, blocks, hashes, [1, 5])
        assert bm.set_node_readonly(5, True) == BM.OK
        assert bm.stripe_repair_all() == (NBLOCKS, NBLOCKS)
        assert bm.stripe_repair_metrics()["stripe_repair_errors"] == NBLOCKS
        assert all(bm.node_shard_index(1, h) == bm.storage_nodes_of(h).index(1) for h in hashes)
        assert bm.set_node_readonly(5, False) == BM.OK
        assert bm.stripe_repair_all() == (NBLOCKS, NBLOCKS)
        assert bm.stripe_repair_metrics()["stripe_repair_errors"] == NBLOCKS
        assert all_valid(bm, hashes)


def test_stop_mid_sweep_resumes_from_the_cursor(tmp_path):
    kw = CODES["clay10_4"]
    blocks, hashes = blocks_of(0x8100, 24)
    with manager(tmp_path, "s", kw) as bm:
        put_with_down(bm, blocks, hashes, [1, 5])
        rebuilt, steps = 0, 0
        for node in range(bm.n_nodes):
            cursor, finished = None, False
            while not finished:
                rc, cursor, finished, _, reb = bm.stripe_repair_step(node, cursor, max_blocks=2)
                assert rc == BM.OK
                rebuilt += reb
                steps += 1
        assert rebuilt == 2 * 24 and steps > bm.n_nodes
        assert all_valid(bm, hashes)


def test_owners_and_resync_workers_together(tmp_path):
    kw = CODES["rs10_4"]
    blocks, hashes = blocks_of(0x8200, 24)
    down = [1, 5, 9]
    with manager(tmp_path, "s", kw) as bm:
        put_with_down(bm, blocks, hashes, down, incref=True)
        for d in down:
            bm.repair_enqueue_missing(d)
        errors = []

        def run(fn):
            try:
                fn()
            except Exception as ex:  # noqa: BLE001
                errors.append(ex)

        th = [threading.Thread(target=run, args=(lambda n=n: bm.stripe_repair_step(n),)) for n in range(bm.n_nodes)]
        th += [threading.Thread(target=run, args=(lambda d=d: bm.resync_all(d),)) for d in down]
        for t in th:
            t.start()
        for t in th:
            t.join()
        assert not errors
        assert bm.stripe_repair_metrics()["stripe_repair_errors"] == 0
        assert bm.metrics()["resync_error_counter"] == 0
        assert all_valid(bm, hashes)
        assert deep_scrub_clean(bm) == 24
        for h, b in zip(hashes, blocks):
            rc, got = bm.rpc_get_block(h)
            assert rc == BM.OK and np.array_equal(got, b)


def test_rejected_calls(tmp_path):
    n, cap = 16, 1 << 40
    with BM.BlockManager(k=10, m=4, n_nodes=n, data_dir=str(tmp_path / "s"), batch_max_blocks=4,
                         layout=dict(zone=[0] * n, capacity=[cap] * 14 + [0, 0])) as bm:
        blocks, hashes = blocks_of(0x8300, 2)
        for h, b in zip(hashes, blocks):
            assert bm.rpc_put_block(h, b) == BM.OK
        bm.set_node_up(3, False)
        assert bm.stripe_repair_step(3)[0] == BM.E_MESSAGE
        bm.set_node_up(3, True)
        assert bm.stripe_repair_step(3)[0] == BM.OK
        assert bm.apply_layout([0] * n, [cap] * n)[0] == BM.OK
        assert bm.stripe_repair_step(3)[0] == E_INVALID
