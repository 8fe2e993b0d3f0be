"""Scheduled resync on RS(10,4), LRC(10,2,2), PB(10,4), Clay(10,4) and RS(4,2) file stores with ragged blocks:
garage_bm_resync_step retries failed resyncs on Garage's ErrorCounter schedule (checked against a Python model of
it), reads nothing for an entry still backing off, and rebuilds every shard once the holders return; retry-now; the
queue and error table across a restart; the GC delay; garage_bm_block_info's per-index states and its recoverability
against an independent rule (k of n for RS, PB and Clay, the rank test of lrc_oracle for LRC); concurrent steps,
PUTs and resync_all; the rejected calls.  The test clock (garage_bm_debug_set_clock_ms) drives the schedule."""
import ctypes as C
import os
import sys
import threading
import time

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import clay_oracle as CO  # noqa: E402
import lrc_oracle as LO  # noqa: E402
import oracle_lib as O  # noqa: E402
import transcode_oracle as TO  # noqa: E402

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
NBLOCKS = 6
E_INVALID = -1
T0 = 1_700_000_000_000  # ms: the test clock's start
IDLE_MS = 10000  # resync_step's wait on an empty queue (Garage's IdleFor(10 s))
X = 0  # the node whose resyncs are scheduled


class ErrorCounter:
    """Garage's ErrorCounter (src/block/resync.rs): errors, last_try, delay 60 s << min(errors - 1, 6)"""

    def __init__(self):
        self.errors, self.last_try = 0, 0

    def fail(self, now):
        self.errors += 1
        self.last_try = now

    def delay(self):
        return 60000 << min(self.errors - 1, 6)

    def next_try(self):
        return self.last_try + self.delay()


def manager(tmp_path, name, kw, **extra):
    extra.setdefault("batch_max_blocks", 4)
    bm = BM.BlockManager(n_nodes=kw["k"] + kw["m"], data_dir=str(tmp_path / name), **kw, **extra)
    assert bm.debug_set_clock_ms(T0) == BM.OK
    return bm


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


def shard_path(d, node, h, ext=".shard"):
    return os.path.join(str(d), "node%d" % node, h[:1].hex(), h[1:2].hex(), h.hex() + ext)


def oracle_shards(kw, b):
    """(k+m, L) shards of block b under the store's code, from the CPU oracles (Vandermonde rows, like the manager)"""
    k, m = kw["k"], kw["m"]
    if kw.get("clay"):
        L = CO.shard_len(b.size, k, m)
        flat = np.zeros(k * L, dtype=np.uint8)
        flat[: b.size] = b
        data = flat.reshape(k, L)
        return np.concatenate([data, CO.encode(k, m, CO.build(k, m), data)])
    if kw.get("local_groups"):
        return TO.encode_block(("lrc", k, kw["local_groups"], m - kw["local_groups"]), b)
    return TO.encode_block(("pb" if kw.get("piggyback") else "rs", k, m, 0), b)


def assert_rebuilt(d, bm, kw, hashes, blocks, saved):
    """X's rebuilt shard files: the oracle's shard of X's index after the header the PUT wrote"""
    for h, b in zip(hashes, blocks):
        raw = read(shard_path(d, X, h))
        i = bm.storage_nodes_of(h).index(X)
        assert raw[:64] == saved[h][:64] and raw[6] == i
        assert raw[64:] == oracle_shards(kw, b)[i].tobytes(), i


def read(p):
    with open(p, "rb") as f:
        return f.read()


def files_of(root):
    out = {}
    for d, _, fs in os.walk(root):
        for f in fs:
            st = os.stat(os.path.join(d, f))
            out[os.path.join(d, f)] = (st.st_size, st.st_mtime_ns)
    return out


def failing_store(tmp_path, name, kw, seed):
    """NBLOCKS blocks PUT and incref'd; node X lost every shard and m+1 other holders are down, so each of X's
    resyncs reaches fewer survivors than a rebuild needs (LRC: only blocks whose lost shard the rank test says cannot
    be rebuilt -- a local group untouched by the outage would repair it).  -> (bm, blocks, hashes, X's shards, down)"""
    bm = manager(tmp_path, name, kw)
    tot = kw["k"] + kw["m"]
    down = list(range(1, kw["m"] + 2))
    blocks, hashes = [], []
    for i in range(64 * NBLOCKS):
        b = O.fill_random(SIZES[len(blocks) % len(SIZES)], seed + i)
        h = BM.blake2sum(b)
        who = bm.storage_nodes_of(h)
        present = [0 if n == X or n in down else 1 for n in who]
        if kw.get("local_groups") and rule_recoverable(kw, present, [int(n == X) for n in who]):
            continue
        blocks.append(b)
        hashes.append(h)
        if len(blocks) == NBLOCKS:
            break
    assert len(blocks) == NBLOCKS and tot == bm.n_nodes
    for h, b in zip(hashes, blocks):
        assert bm.rpc_put_block(h, b) == BM.OK
        assert bm.block_incref(h) == BM.OK  # queues a resync of h, due now, on every holder
    saved = {h: read(shard_path(tmp_path / name, X, h)) for h in hashes}
    for h in hashes:
        assert bm.drop_shard(X, h) == BM.OK
    for n in down:
        bm.set_node_up(n, False)
    return bm, blocks, hashes, saved, down


def errors_of(bm, node=-1):
    rc, errs = bm.list_resync_errors(node)
    assert rc == BM.OK
    return errs


def expect_errors(hashes, model, status=BM.E_MISSING_BLOCK, rc=1):
    return [{"node": X, "hash": h, "rc": rc, "errors": model[h].errors, "last_try_ms": model[h].last_try,
             "next_try_ms": model[h].next_try(), "last_status": status} for h in sorted(hashes)]


def step_at(bm, now, node=X, **kw):
    assert bm.debug_set_clock_ms(now) == BM.OK
    rc, ok, failed, deferred, wait = bm.resync_step(node, **kw)
    assert rc == BM.OK
    return ok, failed, deferred, wait


# ---------------------------------------------------------------- backoff schedule and recovery
@pytest.mark.parametrize("code", list(CODES))
def test_backoff_schedule_then_recovery(tmp_path, code):
    kw = CODES[code]
    bm, blocks, hashes, saved, down = failing_store(tmp_path, "s", kw, 0x9100)
    with bm:
        model = {h: ErrorCounter() for h in hashes}
        m0 = bm.metrics()
        assert step_at(bm, T0) == (0, NBLOCKS, 0, 60000)
        for h in hashes:
            model[h].fail(T0)
        assert errors_of(bm) == errors_of(bm, X) == expect_errors(hashes, model)
        m1, r1 = bm.metrics(), bm.resync_metrics()
        read_once = m1["resync_bytes_read"] - m0["resync_bytes_read"]
        assert read_once > 0 and r1["resync_failed_bytes_read"] == read_once
        assert r1["resync_error_entries"] == NBLOCKS and m1["resync_error_counter"] == NBLOCKS
        for h in hashes:
            rc, info = bm.block_info(h)
            assert rc == BM.OK
            who = info["node"]
            assert info["resync_errors"] == [1 if n == X else 0 for n in who]

        # one ms before the retry: nothing is tried and nothing is read
        assert step_at(bm, T0 + 59999) == (0, 0, 0, 1)
        # an entry queued again meanwhile (the RepairWorker) is deferred to its next try, reading nothing
        assert bm.repair_enqueue_missing(X) == NBLOCKS
        assert step_at(bm, T0 + 59999) == (0, 0, NBLOCKS, 1)
        assert bm.metrics()["resync_bytes_read"] == m1["resync_bytes_read"]
        assert bm.resync_metrics()["resync_deferred"] == NBLOCKS
        assert errors_of(bm) == expect_errors(hashes, model)

        # the retries follow the model up to the 64-minute cap
        while model[hashes[0]].errors < 9:
            nxt = model[hashes[0]].next_try()
            assert step_at(bm, nxt - 1) == (0, 0, 0, 1)
            before = bm.metrics()["resync_bytes_read"]
            ok, failed, deferred, wait = step_at(bm, nxt)
            for h in hashes:
                model[h].fail(nxt)
            assert (ok, failed, deferred, wait) == (0, NBLOCKS, 0, model[hashes[0]].delay())
            assert bm.metrics()["resync_bytes_read"] - before == read_once
            assert errors_of(bm) == expect_errors(hashes, model)
        assert model[hashes[0]].delay() == 64 * 60000

        # the holders return: the next due step rebuilds every shard byte for byte
        for n in down:
            bm.set_node_up(n, True)
        nxt = model[hashes[0]].next_try()
        assert step_at(bm, nxt - 1) == (0, 0, 0, 1)
        assert step_at(bm, nxt) == (NBLOCKS, 0, 0, IDLE_MS)
        assert_rebuilt(tmp_path / "s", bm, kw, hashes, blocks, saved)
        assert errors_of(bm) == []
        assert bm.resync_metrics()["resync_error_entries"] == 0
        assert step_at(bm, nxt + 1) == (0, 0, 0, IDLE_MS)
        for n in down[: kw["m"] - (1 if kw.get("local_groups") else 0)]:  # LRC: m-1, the losses it always decodes
            bm.set_node_up(n, False)
        for h, b in zip(hashes, blocks):
            rc, got = bm.rpc_get_block(h)
            assert rc == BM.OK and np.array_equal(got, b)


# ---------------------------------------------------------------- retry-now
@pytest.mark.parametrize("code", ["rs10_4", "clay10_4"])
def test_retry_now_one_hash_and_all(tmp_path, code):
    kw = CODES[code]
    bm, blocks, hashes, saved, down = failing_store(tmp_path, "s", kw, 0x9200)
    with bm:
        model = {h: ErrorCounter() for h in hashes}
        assert step_at(bm, T0) == (0, NBLOCKS, 0, 60000)
        for h in hashes:
            model[h].fail(T0)
        h0 = hashes[0]
        now = T0 + 5000
        assert bm.debug_set_clock_ms(now) == BM.OK
        assert bm.resync_retry_now(X, h0) == (BM.OK, 1)
        model[h0].last_try = now - model[h0].delay()  # clear_backoff keeps the count
        assert errors_of(bm) == expect_errors(hashes, model)
        assert step_at(bm, now) == (0, 1, 0, T0 + 60000 - now)
        model[h0].fail(now)
        assert errors_of(bm) == expect_errors(hashes, model)

        assert bm.resync_retry_now(X) == (BM.OK, NBLOCKS)
        assert step_at(bm, now) == (0, NBLOCKS, 0, 120000)
        for h in hashes:
            model[h].fail(now)
        assert errors_of(bm) == expect_errors(hashes, model)

        # not in an errored state: Error::Message, as Garage's clear_backoff
        assert bm.resync_retry_now(X, bytes(32))[0] == BM.E_MESSAGE
        other = bm.k + bm.m - 1
        assert bm.resync_retry_now(other, h0)[0] == BM.E_MESSAGE
        assert bm.resync_retry_now(other) == (BM.OK, 0)
        assert bm.resync_metrics()["resync_retry_nows"] == 1 + NBLOCKS

        # resync_all drains everything, backoff or not, and a success clears the error entry
        for n in down:
            bm.set_node_up(n, True)
        assert bm.resync_all(X) == (0, NBLOCKS)
        assert errors_of(bm) == []
        assert_rebuilt(tmp_path / "s", bm, kw, hashes, blocks, saved)


# ---------------------------------------------------------------- restart
@pytest.mark.parametrize("code", list(CODES))
def test_queue_and_errors_survive_a_restart(tmp_path, code):
    kw = CODES[code]
    d = tmp_path / "s"
    bm, blocks, hashes, saved, _ = failing_store(tmp_path, "s", kw, 0x9300)
    with bm:
        assert step_at(bm, T0) == (0, NBLOCKS, 0, 60000)
        assert bm.debug_set_clock_ms(T0 + 5000) == BM.OK
        assert bm.resync_retry_now(X, hashes[0]) == (BM.OK, 1)
        errs = [dict(e, rc=-1) for e in errors_of(bm)]  # the rc table is not kept across a restart: -1 after it
    image = read(os.path.join(str(d), "node%d" % X, "resync"))
    tot = kw["k"] + kw["m"]
    assert [n for n in range(tot) if os.path.exists(os.path.join(str(d), "node%d" % n, "resync"))] == [X]
    with manager(tmp_path, "s", kw) as bm:
        assert errors_of(bm) == errs
        assert bm.metrics()["resync_queue_length"] == NBLOCKS
        assert step_at(bm, T0 + 4000) == (0, 0, 0, 1000)  # the first entry is due at T0 + 5000, as before
    assert read(os.path.join(str(d), "node%d" % X, "resync")) == image
    with manager(tmp_path, "s", kw) as bm:  # every holder up again: the entry made due by retry-now is rebuilt
        assert step_at(bm, T0 + 5000) == (1, 0, 0, 55000)
        assert step_at(bm, T0 + 60000) == (NBLOCKS - 1, 0, 0, IDLE_MS)
        assert errors_of(bm) == []
        assert_rebuilt(d, bm, kw, hashes, blocks, saved)

    # a store that never used the scheduled calls writes no file, and restarts with an empty queue as before
    p = tmp_path / "plain"
    with BM.BlockManager(n_nodes=tot, data_dir=str(p), batch_max_blocks=4, **kw) as bm:
        blocks, hashes = blocks_of(0x9380)
        for h, b in zip(hashes, blocks):
            assert bm.rpc_put_block(h, b) == BM.OK
            assert bm.block_incref(h) == BM.OK
            assert bm.drop_shard(X, h) == BM.OK
        assert bm.metrics()["resync_queue_length"] == NBLOCKS * tot
    assert not any(f == "resync" for _, _, fs in os.walk(str(p)) for f in fs)
    with BM.BlockManager(n_nodes=tot, data_dir=str(p), batch_max_blocks=4, **kw) as bm:
        assert bm.metrics()["resync_queue_length"] == 0
        assert bm.repair_enqueue_missing(X) == NBLOCKS  # the RepairWorker finds what the queue lost
        assert bm.resync_all(X) == (0, NBLOCKS)


# ---------------------------------------------------------------- GC delay
def test_gc_delay_schedules_the_deletion(tmp_path):
    kw = CODES["rs4_2"]
    gc_ms = 3000
    with manager(tmp_path, "s", kw, block_gc_delay_ms=gc_ms) as bm:
        tot = kw["k"] + kw["m"]
        blocks, hashes = blocks_of(0x9400)
        for h, b in zip(hashes, blocks):
            assert bm.rpc_put_block(h, b) == BM.OK
            assert bm.block_incref(h) == BM.OK
        for n in range(tot):
            assert step_at(bm, T0, node=n) == (NBLOCKS, 0, 0, IDLE_MS)  # the shards are there: nothing to do
        for h in hashes:
            assert bm.block_decref(h) == BM.OK  # rc 0: a resync queued on every holder, to delete after the delay
        waits = []
        for n in range(tot):
            ok, failed, deferred, wait = step_at(bm, T0, node=n)
            assert (ok, failed, deferred) == (0, 0, NBLOCKS) and 0 < wait <= gc_ms
            waits.append(wait)
        d0 = bm.metrics()["delete_counter"]
        for n in range(tot):
            assert step_at(bm, T0 + min(waits) - 1, node=n)[:3] == (0, 0, 0)  # not looked at again before then
        assert bm.resync_metrics()["resync_deferred"] == NBLOCKS * tot
        assert all(bm.node_shard_index(n, h) >= 0 for n in range(tot) for h in hashes)
        time.sleep(gc_ms / 1000 + 0.3)
        for n in range(tot):
            assert step_at(bm, T0 + gc_ms, node=n) == (NBLOCKS, 0, 0, IDLE_MS)
        assert bm.metrics()["delete_counter"] == d0 + NBLOCKS * tot
        assert all(bm.node_shard_index(n, h) == -1 for n in range(tot) for h in hashes)
        assert errors_of(bm) == []


# ---------------------------------------------------------------- block_info
def rule_recoverable(kw, present, want=None):
    if kw.get("local_groups"):
        P = LO.build_lrc(kw["k"], kw["local_groups"], kw["m"] - kw["local_groups"])
        return LO.recoverable(kw["k"], P, present, want)
    return sum(present) >= kw["k"]


def check_info(kw, ec, info, states):
    tot = kw["k"] + kw["m"]
    assert info["state"] == states
    present = [1 if s == BM.SHARD_VALID else 0 for s in states]
    assert info["recoverable"] == rule_recoverable(kw, present), states
    if info["recoverable"] and not all(present):
        rs = ec.read_set(np.array(present, np.uint8))
        assert rs is not None and info["read_set"] == list(rs)
        if not (kw.get("local_groups") or kw.get("piggyback") or kw.get("clay")):  # RS: the first k valid shards
            assert info["read_set"] == [1 if i in [j for j in range(tot) if present[j]][: kw["k"]] else 0
                                        for i in range(tot)]
    else:
        assert info["read_set"] == [0] * tot


@pytest.mark.parametrize("code", list(CODES))
def test_block_info_states_and_recoverability(tmp_path, code):
    kw = CODES[code]
    k, m = kw["k"], kw["m"]
    tot = k + m
    d = tmp_path / "s"
    with ec_of(kw) as ec, manager(tmp_path, "s", kw) as bm:
        blocks, hashes = blocks_of(0x9500, 3)
        for h, b in zip(hashes, blocks):
            assert bm.rpc_put_block(h, b) == BM.OK
        h = hashes[1]
        assert bm.block_incref(h) == BM.OK
        who = bm.storage_nodes_of(h)
        rc, info = bm.block_info(h, check_tags=True)
        assert rc == BM.OK and info["rc"] == 1 and info["node"] == who
        assert info["code"] == (k, m, kw.get("local_groups", 0), int(kw.get("piggyback", False)), int(kw.get("clay", False)))
        assert info["block_len"] == blocks[1].size and info["resync_errors"] == [0] * tot
        check_info(kw, ec, info, [BM.SHARD_VALID] * tot)

        assert bm.drop_shard(who[0], h) == BM.OK
        assert bm.corrupt_shard(who[1], h, 5) == BM.OK
        assert bm.corrupt_shard_header(who[2], h, 1) == BM.OK
        assert bm.corrupt_shard(who[3], h, 7) == BM.OK
        assert bm.scrub(who[3])[2] == 1  # quarantined: only <hash>.corrupted is left on that node
        assert os.path.exists(shard_path(d, who[3], h, ".corrupted"))
        bm.set_node_up(who[4], False)
        before, m0 = files_of(str(d)), bm.metrics()
        rc, hdr = bm.block_info(h)
        assert rc == BM.OK
        rc, tagged = bm.block_info(h, check_tags=True)
        assert rc == BM.OK
        assert files_of(str(d)) == before  # read-only: the bad-tag shard is not quarantined
        m1 = bm.metrics()
        for key in ("resync_queue_length", "corruption_counter", "delete_counter", "bytes_written"):
            assert m1[key] == m0[key], key
        rest = [BM.SHARD_VALID] * (tot - 5)
        check_info(kw, ec, hdr, [BM.SHARD_ABSENT, BM.SHARD_VALID, BM.SHARD_BAD_HEADER, BM.SHARD_QUARANTINED,
                                 BM.SHARD_DOWN] + rest)
        check_info(kw, ec, tagged, [BM.SHARD_ABSENT, BM.SHARD_BAD_TAG, BM.SHARD_BAD_HEADER, BM.SHARD_QUARANTINED,
                                    BM.SHARD_DOWN] + rest)
        assert hdr["block_len"] == blocks[1].size
        bm.set_node_up(who[4], True)

        # recoverability over patterns of down holders, against the independent rule
        h = hashes[2]
        who = bm.storage_nodes_of(h)
        rng = np.random.default_rng(0x95 + k + m)
        patterns = [list(rng.choice(tot, size=e, replace=False)) for e in (m - 1, m, m + 1) for _ in range(4)]
        if kw.get("local_groups"):
            patterns.append([0, 1, 2, 3])  # k valid shards, 4 unknowns of one group behind 3 equations
        seen_k_valid_unrecoverable = False
        for pat in patterns:
            for i in pat:
                bm.set_node_up(who[i], False)
            rc, info = bm.block_info(h)
            assert rc == BM.OK
            states = [BM.SHARD_DOWN if i in pat else BM.SHARD_VALID for i in range(tot)]
            check_info(kw, ec, info, states)
            seen_k_valid_unrecoverable |= tot - len(pat) == k and not info["recoverable"]
            for i in pat:
                bm.set_node_up(who[i], True)
        assert seen_k_valid_unrecoverable == bool(kw.get("local_groups"))


def test_block_info_reports_previous_code_copies(tmp_path):
    d = str(tmp_path / "s")
    blocks, hashes = blocks_of(0x9600, 2)
    with BM.BlockManager(k=4, m=2, n_nodes=14, data_dir=d, batch_max_blocks=4) as old:
        for h, b in zip(hashes, blocks):
            assert old.rpc_put_block(h, b) == BM.OK
    with BM.BlockManager(k=10, m=4, n_nodes=14, data_dir=d, batch_max_blocks=4, previous_codes=[(4, 2, 0, 0)]) as bm:
        for h in hashes:
            rc, info = bm.block_info(h, check_tags=True)
            assert rc == BM.OK and info["rc"] == -1 and info["block_len"] == 0
            assert info["state"] == [BM.SHARD_PREVIOUS] * 6 + [BM.SHARD_ABSENT] * 8
            assert not info["recoverable"] and info["read_set"] == [0] * 14
            rc, got = bm.rpc_get_block(h)  # served from the previous code's stripe
            assert rc == BM.OK


# ---------------------------------------------------------------- concurrency and rejected calls
def test_steps_puts_and_resync_all_together(tmp_path):
    kw = CODES["rs10_4"]
    with manager(tmp_path, "s", kw) as bm:
        blocks, hashes = blocks_of(0x9700, 16)
        down = [1, 5, 9]
        for n in down:
            bm.set_node_up(n, False)
        for h, b in zip(hashes, blocks):
            assert bm.rpc_put_block(h, b) == BM.OK
            assert bm.block_incref(h) == BM.OK
        for n in down:
            bm.set_node_up(n, True)
        new_blocks, new_hashes = blocks_of(0x9780, 16)
        results, errors = [], []

        def run(fn):
            try:
                results.append(fn())
            except Exception as ex:  # noqa: BLE001
                errors.append(ex)

        jobs = [lambda n=n: bm.resync_step(n, workers=4) for n in (1, 5)]
        jobs += [lambda: bm.resync_step(5, workers=2, max_blocks=3), lambda: bm.resync_all(9)]
        jobs += [lambda h=h, b=b: bm.rpc_put_block(h, b) for h, b in zip(new_hashes, new_blocks)]
        th = [threading.Thread(target=run, args=(j,)) for j in jobs]
        for t in th:
            t.start()
        for t in th:
            t.join()
        assert not errors and len(results) == len(jobs)
        for r in results:
            if isinstance(r, int):
                assert r == BM.OK  # a PUT
            elif len(r) == 2:
                assert r[0] == 0  # resync_all: nothing failed
            else:
                assert r[0] == BM.OK and r[2] == 0  # a step: nothing failed
        for n in (1, 5):
            ok, failed, _, _ = step_at(bm, T0, node=n)
            assert failed == 0
        assert bm.metrics()["resync_error_counter"] == 0 and errors_of(bm) == []
        assert all(bm.node_shard_index(n, h) == i for h in hashes for i, n in enumerate(bm.storage_nodes_of(h)))
        for h, b in zip(hashes + new_hashes, blocks + new_blocks):
            rc, got = bm.rpc_get_block(h)
            assert rc == BM.OK and np.array_equal(got, b)


def test_rejected_calls(tmp_path):
    kw = CODES["rs4_2"]
    bm, _, hashes, _, down = failing_store(tmp_path, "s", kw, 0x9800)
    with bm:
        L, hp = bm._L, bm._h
        n_nodes = bm.n_nodes
        for node in (-1, n_nodes):
            assert bm.resync_step(node)[0] == E_INVALID
            assert bm.resync_retry_now(node)[0] == E_INVALID
        for w in (0, 9, -3):
            assert bm.resync_step(X, workers=w)[0] == E_INVALID
        assert bm.resync_step(down[0])[0] == BM.E_MESSAGE  # a down node runs no worker
        # the step's workers are threads of its own: the caller's CPU affinity (which garage_ec_bind_thread would
        # narrow to the GPU's NUMA node) is what it was, with one worker and with eight
        affinity = os.sched_getaffinity(0)
        assert step_at(bm, T0, workers=1) == (0, NBLOCKS, 0, 60000)
        assert os.sched_getaffinity(0) == affinity
        assert bm.resync_retry_now(X) == (BM.OK, NBLOCKS)
        assert step_at(bm, T0, workers=8) == (0, NBLOCKS, 0, 120000)
        assert os.sched_getaffinity(0) == affinity
        assert bm.list_resync_errors(-2)[0] == E_INVALID and bm.list_resync_errors(n_nodes)[0] == E_INVALID
        n = C.c_size_t(0)
        assert L.garage_bm_list_resync_errors(hp, -1, None, 0, None) == E_INVALID
        assert L.garage_bm_list_resync_errors(hp, -1, None, 1, C.byref(n)) == E_INVALID
        assert L.garage_bm_list_resync_errors(hp, -1, None, 0, C.byref(n)) == BM.OK and n.value == NBLOCKS  # size query
        one = (BM.ResyncError * 2)()
        assert L.garage_bm_list_resync_errors(hp, X, one, 1, C.byref(n)) == BM.OK and n.value == NBLOCKS  # cut at cap
        assert bytes(one[0].hash) == min(hashes) and one[1].errors == 0  # nothing past cap is written
        st = BM.BlockStatus()
        assert L.garage_bm_block_info(hp, None, 0, C.byref(st)) == E_INVALID
        assert L.garage_bm_block_info(hp, C.c_char_p(hashes[0]), 0, None) == E_INVALID
        assert L.garage_bm_resync_step(hp, X, 8, 0, None, None, None, None) == BM.OK  # outputs may be NULL
        assert L.garage_bm_get_resync_metrics(hp, None) is None
