"""HOST-mode ownership contract of the C ABI (include/garage_ec.h: "the library keeps no pointer
after a HOST call returns") under injected faults, lane-set concurrency, NUMA placement report
and the survivors-only upload of garage_ec_decode_blocks.

Reference convention mirrored: blocks are bytes::Bytes owned by the caller and every error is a
Result (src/util/error.rs:14-82); a Rust caller frees its Vec on Err, so a DMA that is still in
flight after an error return would be a use-after-free."""
import contextlib
import os
import sys
import threading

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import oracle_lib as O  # noqa: E402

import garage_b200 as G  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch():
    import torch as t

    assert t.cuda.is_available()
    return t


def _case(k, m, n, stride, seed):
    P = O.build_matrix(k, m, 0)
    data = O.fill_random(n * k * stride, seed)
    par = O.encode(k, m, P, data, stride, n, simd=True)
    sh = np.ascontiguousarray(np.concatenate([data.reshape(n, k, stride), par.reshape(n, m, stride)], axis=1))
    return data, par, sh


@pytest.mark.parametrize("fail_at", [0, 1, 2, 3, 5, 8, 13, 21])
def test_encode_host_fault_leaves_no_dma_in_flight(torch, fail_at):
    """n stripes over several 48 MB chunks so that copies of later chunks are queued on other
    lanes when the fault hits; after the error return the output buffer must never change again"""
    k, m, stride, n = 10, 4, 104960, 480  # 11 chunks of 48 MB
    data, par, _ = _case(k, m, n, stride, 4242)
    with G.GarageEc(0, k, m) as ec:
        out = np.zeros(n * m * stride, dtype=np.uint8)
        ec.encode(data, out, stride, n)  # lanes allocated, streams created
        assert np.array_equal(out, par)
        ec.debug_fail_after(fail_at)
        with pytest.raises(G.EcError) as ei:
            ec.encode(data, out, stride, n)
        assert ei.value.code in (G.E_CUDA, G.E_NOMEM)
        ec.debug_fail_after(-1)
        out[:] = 0xEE  # "free" the buffer: nothing may write it from now on
        torch.cuda.synchronize()
        assert (out == 0xEE).all(), "a D2H copy completed after the failed call had returned"
        # the context is still usable and correct
        ec.encode(data, out, stride, n)
        assert np.array_equal(out, par)


@pytest.mark.parametrize("fail_at", [0, 2, 4, 7, 11, 16])
def test_reconstruct_and_scrub_host_fault(torch, fail_at):
    k, m, stride, n = 6, 3, 174848, 240  # 8 chunks
    tot = k + m
    _, _, sh = _case(k, m, n, stride, 77)
    rng = np.random.default_rng(3)
    present = np.ones((n, tot), dtype=np.uint8)
    for s in range(n):
        present[s, rng.choice(tot, m, replace=False)] = 0
    with G.GarageEc(0, k, m) as ec:
        work = sh.copy()
        work[present == 0] = 0
        st = np.zeros(n, dtype=np.int32)
        ec.reconstruct(work.reshape(-1), present, stride, n, status=st)
        assert np.array_equal(work, sh)
        work[present == 0] = 0
        ec.debug_fail_after(fail_at)
        with pytest.raises(G.EcError):
            ec.reconstruct(work.reshape(-1), present, stride, n, status=st)
        ec.debug_fail_after(-1)
        work[:] = 0xEE
        st[:] = 0x5A5A5A5A
        torch.cuda.synchronize()
        assert (work == 0xEE).all() and (st == 0x5A5A5A5A).all()
        # scrub + repair sweep, same contract
        sums = np.zeros(n * tot * 32, dtype=np.uint8)
        ec.shard_sums(sh.reshape(-1), sums, stride, n, tot)
        work = sh.copy()
        work[1, 2, 5] ^= 1
        bad = np.zeros(n * tot, dtype=np.uint8)
        ec.debug_fail_after(fail_at)
        with pytest.raises(G.EcError):
            ec.scrub_repair(work.reshape(-1), sums, bad, stride, n, status=st)
        ec.debug_fail_after(-1)
        work[:] = 0xEE
        bad[:] = 0xEE
        torch.cuda.synchronize()
        assert (work == 0xEE).all() and (bad == 0xEE).all()
        work = sh.copy()
        work[1, 2, 5] ^= 1
        ec.scrub_repair(work.reshape(-1), sums, bad, stride, n, status=st)
        assert bad.sum() == 1 and bad.reshape(n, tot)[1, 2] == 1 and np.array_equal(work, sh)


def test_block_level_host_fault(torch):
    k, m = 10, 4
    tot = k + m
    blens = [1 << 20] * 70 + [12345, 1, 777777]
    blocks = [O.fill_random(b, 50 + i) for i, b in enumerate(blens)]
    n = len(blocks)
    with G.GarageEc(0, k, m) as ec:
        stride = ec.stride_for(ec.shard_len(max(blens)))
        par = np.zeros(n * m * stride, dtype=np.uint8)
        sums = np.zeros(n * tot * 32, dtype=np.uint8)
        ec.encode_blocks(blocks, par, stride, sums_out=sums)
        good_par, good_sums = par.copy(), sums.copy()
        for fail_at in (0, 3, 9, 14):
            ec.debug_fail_after(fail_at)
            with pytest.raises(G.EcError):
                ec.encode_blocks(blocks, par, stride, sums_out=sums)
            ec.debug_fail_after(-1)
            par[:] = 0xEE
            sums[:] = 0xEE
            torch.cuda.synchronize()
            assert (par == 0xEE).all() and (sums == 0xEE).all()
        ec.encode_blocks(blocks, par, stride, sums_out=sums)
        assert np.array_equal(par, good_par) and np.array_equal(sums, good_sums)
        # decode with faults
        shards = np.zeros((n, tot, stride), dtype=np.uint8)
        for s, b in enumerate(blocks):
            shards[s, :k] = O.split_block(b, k, stride).reshape(k, stride)
        shards[:, k:] = par.reshape(n, m, stride)
        present = np.ones((n, tot), dtype=np.uint8)
        rng = np.random.default_rng(9)
        for s in range(n):
            present[s, rng.choice(tot, m, replace=False)] = 0
        shards[present == 0] = 0x77  # absent shards hold garbage: they must not be read
        out = [np.zeros(b, dtype=np.uint8) for b in blens]
        st = np.zeros(n, dtype=np.int32)
        for fail_at in (0, 2, 6):
            ec.debug_fail_after(fail_at)
            with pytest.raises(G.EcError):
                ec.decode_blocks(shards.reshape(-1), present, blens, stride, out, st)
            ec.debug_fail_after(-1)
            for o in out:
                o[:] = 0xEE
            torch.cuda.synchronize()
            assert all((o == 0xEE).all() for o in out)
        assert ec.decode_blocks(shards.reshape(-1), present, blens, stride, out, st) == 0
        for s in range(n):
            assert np.array_equal(out[s], blocks[s]), s


@pytest.fixture(scope="module")
def big_case():
    """RS(10,4), 240 stripes of 14 x 104960 bytes: 8 chunks of 48 MB"""
    k, m, stride, n = 10, 4, 104960, 240
    _, _, sh = _case(k, m, n, stride, 1618)
    present = np.ones((n, k + m), dtype=np.uint8)
    rng = np.random.default_rng(21)
    for s in range(n):
        present[s, rng.choice(k + m, m, replace=False)] = 0
    return k, m, stride, n, sh, present


# Each entry: (ec, case, stack) -> (run, outputs, reset, check).  run() makes the HOST call, `outputs` are the caller's
# arrays it writes, reset() restores the inputs a run consumes and check() asserts the exact result; `stack` (an
# ExitStack) frees what the entry allocates.
def _verify_call(ec, case, stack):
    k, m, stride, n, sh, _ = case
    work = sh.copy()
    work[37, k + 1, 11] ^= 1
    mm = np.zeros(n, dtype=np.uint32)

    def check():
        assert np.flatnonzero(mm).tolist() == [37]

    return lambda: ec.verify(work.reshape(-1), mm, stride, n), [mm], lambda: None, check


def _deep_check_call(ec, case, stack):
    k, m, stride, n, sh, _ = case
    work = sh.copy()
    work[37, k + 1, 11] ^= 1
    blen = np.full(n, k * stride, dtype=np.uint32)
    hashes = np.stack([np.frombuffer(G.blake2sum(sh[s, :k].reshape(-1)), dtype=np.uint8) for s in range(n)])
    hashes[5, 0] ^= 1
    bad = np.zeros(n, dtype=np.uint8)
    mm = np.zeros(n, dtype=np.uint32)

    def check():
        assert np.flatnonzero(bad).tolist() == [5] and np.flatnonzero(mm).tolist() == [37]

    return lambda: ec.deep_check(work.reshape(-1), blen, hashes, bad, mm, stride, n), [bad, mm], lambda: None, check


def _shard_sums_call(ec, case, stack):
    k, m, stride, n, sh, _ = case
    tot = k + m
    sums = np.zeros((n, tot, 32), dtype=np.uint8)

    def check():
        for s in (0, n // 2, n - 1):
            for i in range(tot):
                assert sums[s, i].tobytes() == G.blake2sum(sh[s, i]), (s, i)

    return lambda: ec.shard_sums(sh.reshape(-1), sums, stride, n, tot), [sums], lambda: None, check


def _check_sums_call(ec, case, stack):
    k, m, stride, n, sh, _ = case
    tot = k + m
    expect = np.zeros(n * tot * 32, dtype=np.uint8)
    ec.shard_sums(sh.reshape(-1), expect, stride, n, tot)
    work = sh.copy()
    work[100, 3, 7] ^= 1
    bad = np.zeros(n * tot, dtype=np.uint8)

    def check():
        assert np.flatnonzero(bad).tolist() == [100 * tot + 3]

    return lambda: ec.check_sums(work.reshape(-1), expect, bad, stride, n, tot), [bad], lambda: None, check


def _reconstruct_stripes_call(ec, case, stack):
    k, m, stride, n, sh, present = case
    work = sh.copy()
    stripes = [work[s] for s in range(n)]
    st = np.zeros(n, dtype=np.int32)

    def reset():
        work[:] = sh
        work[present == 0] = 0

    def check():
        assert np.array_equal(work, sh) and not st.any()

    return lambda: ec.reconstruct_stripes(stripes, present, stride, status=st), [work, st], reset, check


def _reconstruct_pinned_call(ec, case, stack):
    """pinned buffer: the zero-copy reconstruct (one launch over the caller's buffer, no staging)"""
    k, m, stride, n, sh, present = case
    buf, p = ec.host_alloc(n * (k + m) * stride)
    stack.callback(ec.host_free, p)
    v = buf.reshape(n, k + m, stride)
    want = np.ones((n, k + m), dtype=np.uint8)
    lens = np.full(n, stride, dtype=np.uint32)
    st = np.zeros(n, dtype=np.int32)

    def reset():
        v[:] = sh
        v[present == 0] = 0x77

    def check():
        assert np.array_equal(v, sh) and not st.any()

    def run():
        return ec.reconstruct(buf, present, stride, n, want=want, status=st, shard_len=lens)

    return run, [buf, st], reset, check


_FAULT_CALLS = {
    "verify": _verify_call,
    "deep_check": _deep_check_call,
    "shard_sums": _shard_sums_call,
    "check_sums": _check_sums_call,
    "reconstruct_stripes": _reconstruct_stripes_call,
    "reconstruct_pinned": _reconstruct_pinned_call,
}


@pytest.mark.parametrize("fail_at", [0, 1, 3, 5])
@pytest.mark.parametrize("call", sorted(_FAULT_CALLS))
def test_host_call_fault_leaves_caller_buffers_alone(torch, big_case, call, fail_at):
    """the HOST entry points the tests above do not cover, same contract: after an injected fault's error return
    nothing writes the caller's output buffers any more, and the context still computes exact results"""
    k, m = big_case[:2]
    with G.GarageEc(0, k, m) as ec, contextlib.ExitStack() as stack:
        run, outs, reset, check = _FAULT_CALLS[call](ec, big_case, stack)
        reset()
        run()  # lanes sized, streams created
        check()
        reset()
        ec.debug_fail_after(fail_at)
        with pytest.raises(G.EcError):
            run()
        ec.debug_fail_after(-1)
        for o in outs:
            o.view(np.uint8)[...] = 0xEE
        torch.cuda.synchronize()
        assert all((o.view(np.uint8) == 0xEE).all() for o in outs), "a copy or kernel wrote after the error return"
        reset()
        run()
        check()


def test_decode_blocks_uploads_survivors_only(torch):
    """GET path: only the k shards the kernel reads cross PCIe.  Observable contract: shards that
    are absent -- or present but beyond the first k -- may hold anything, even unreadable
    garbage patterns, and the result is still exact."""
    k, m = 10, 4
    tot = k + m
    n = 24
    blens = [(1 << 20) - 3 * i for i in range(n)]
    blocks = [O.fill_random(b, 500 + i) for i, b in enumerate(blens)]
    with G.GarageEc(0, k, m) as ec:
        stride = ec.stride_for(ec.shard_len(max(blens)))
        par = np.zeros(n * m * stride, dtype=np.uint8)
        ec.encode_blocks(blocks, par, stride)
        shards = np.zeros((n, tot, stride), dtype=np.uint8)
        for s, b in enumerate(blocks):
            shards[s, :k] = O.split_block(b, k, stride).reshape(k, stride)
        shards[:, k:] = par.reshape(n, m, stride)
        present = np.ones((n, tot), dtype=np.uint8)
        rng = np.random.default_rng(11)
        for s in range(n):
            gone = rng.choice(k, int(rng.integers(1, 3)), replace=False)  # 1-2 data shards absent
            present[s, gone] = 0
            shards[s, gone] = 0xAB
            # surplus parity shards (present, but not among the first k present): poison them too
            first_k = np.flatnonzero(present[s])[:k]
            for i in range(tot):
                if present[s, i] and i not in first_k:
                    shards[s, i] = 0xCD
        out = [np.zeros(b, dtype=np.uint8) for b in blens]
        st = np.zeros(n, dtype=np.int32)
        assert ec.decode_blocks(shards.reshape(-1), present, blens, stride, out, st) == 0
        for s in range(n):
            assert np.array_equal(out[s], blocks[s]), s


def test_host_calls_from_many_threads_use_separate_lanes(torch):
    """more concurrent HOST callers than lane sets: all results exact, no deadlock"""
    k, m, stride, n = 10, 4, 104960, 40
    cases = [_case(k, m, n, stride, 1000 + i) for i in range(6)]
    with G.GarageEc(0, k, m) as ec:
        errs = []

        def work(i):
            data, par, sh = cases[i]
            try:
                for it in range(3):
                    out = np.zeros(n * m * stride, dtype=np.uint8)
                    ec.encode(data, out, stride, n)
                    if not np.array_equal(out, par):
                        errs.append(("enc", i))
                    w = sh.copy()
                    present = np.ones((n, k + m), dtype=np.uint8)
                    present[:, (i + it) % (k + m)] = 0
                    w[present == 0] = 0
                    ec.reconstruct(w.reshape(-1), present, stride, n)
                    if not np.array_equal(w, sh):
                        errs.append(("rec", i))
            except Exception as ex:  # noqa: BLE001
                errs.append(repr(ex))

        th = [threading.Thread(target=work, args=(i,)) for i in range(6)]
        [t.start() for t in th]
        [t.join(timeout=300) for t in th]
        assert not any(t.is_alive() for t in th), "deadlock in the lane-set pool"
        assert not errs, errs


def test_pinned_alloc_is_numa_local_when_topology_is_known(torch):
    with G.GarageEc(0, 10, 4) as ec:
        buf, p = ec.host_alloc(64 << 20)
        buf[:] = 1
        gpu_node, got = ec.numa_info()
        ec.host_free(p)
        if gpu_node >= 0 and got >= 0:
            assert got == gpu_node, "pinned buffer landed on node %d, the GPU hangs off node %d" % (got, gpu_node)
        # binding the calling thread is best effort and must leave the thread runnable
        before = os.sched_getaffinity(0)
        ec.bind_thread()
        assert len(os.sched_getaffinity(0)) >= 1
        os.sched_setaffinity(0, before)


def test_write_combined_pinned_buffers_work_as_upload_and_download_buffers(torch):
    """garage_ec_host_alloc_wc: upload-only / download-only landing buffers (no CPU reads on the hot path)"""
    k, m, stride, n = 10, 4, 104960, 64
    data, par, _ = _case(k, m, n, stride, 31337)
    with G.GarageEc(0, k, m) as ec:
        h_in, p1 = ec.host_alloc(n * k * stride, write_combined=True)
        h_out, p2 = ec.host_alloc(n * m * stride, write_combined=True)
        h_in[:] = data            # sequential CPU writes: what write-combined memory is for
        ec.encode(h_in, h_out, stride, n)
        assert np.array_equal(np.array(h_out), par)  # (a slow uncached read, fine in a test)
        gpu_node, got = ec.numa_info()
        if gpu_node >= 0 and got >= 0:
            assert got == gpu_node
        ec.host_free(p1)
        ec.host_free(p2)


def test_reconstruct_on_pinned_buffers_runs_in_place_over_pcie(torch):
    """HOST reconstruct on pinned (device-addressable) buffers takes the zero-copy path: the kernel reads the
    survivors from, and writes the rebuilt shards into, the caller's buffer.  Same results as the staged path,
    absent shards may hold garbage, present shards are never written, want masks and unrecoverable stripes work."""
    k, m, stride, n = 10, 4, 104960, 96
    tot = k + m
    _, _, sh = _case(k, m, n, stride, 2718)
    lens = np.full(n, 104858, dtype=np.uint32)
    rng = np.random.default_rng(5)
    present = np.ones((n, tot), dtype=np.uint8)
    for s in range(n):
        present[s, rng.choice(tot, int(rng.integers(0, m + 1)), replace=False)] = 0
    present[7, : m + 1] = 0  # unrecoverable
    want = np.ones((n, tot), dtype=np.uint8)
    want[:, k:] = 0  # GET: data shards only
    with G.GarageEc(0, k, m) as ec:
        buf, p = ec.host_alloc(n * tot * stride)
        v = buf.reshape(n, tot, stride)
        v[:] = sh
        v[present == 0] = 0x77
        st = np.zeros(n, dtype=np.int32)
        rc = ec.reconstruct(buf, present, stride, n, want=want, status=st, shard_len=lens)
        assert rc == G.E_UNRECOVERABLE and st[7] == G.E_UNRECOVERABLE and np.count_nonzero(st) == 1
        for s in range(n):
            for i in range(tot):
                got = v[s, i, :104858]
                if present[s, i] or s == 7:
                    expect = sh[s, i, :104858] if present[s, i] else np.full(104858, 0x77, dtype=np.uint8)
                elif i < k:
                    expect = sh[s, i, :104858]            # rebuilt
                else:
                    expect = np.full(104858, 0x77, dtype=np.uint8)  # absent parity, not wanted: untouched
                assert np.array_equal(got, expect), (s, i)
        # and it is the same answer the staged path gives on pageable memory
        pg = sh.copy()
        pg[present == 0] = 0x77
        st2 = np.zeros(n, dtype=np.int32)
        ec.reconstruct(pg.reshape(-1), present, stride, n, want=want, status=st2, shard_len=lens)
        assert np.array_equal(st, st2) and np.array_equal(pg[:, :, :104858], v[:, :, :104858])
        ec.host_free(p)
