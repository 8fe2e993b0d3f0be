"""A block manager on several dispatcher groups (garage_bm_create_on_devices, DESIGN.md section 5.13).  Every test runs
on two groups of device 0 ([0, 0]), and on devices 0 and 1 where two are visible: the same bytes and content addresses
as a one-device manager for every code and call, degraded reads and every repair sweep through both groups, the
routing rule, the pools' NUMA placement, and the refusals and teardown of the create call."""
import os
import sys
import threading

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
import oracle_lib as O  # noqa: E402

import garage_b200 as G  # noqa: E402
from garage_b200 import block_manager as BM  # noqa: E402

E_INVALID = -1
SIZES = [3073, 65536, 1 << 20, 777777, (1 << 20) - 1, 5]
KEY_A, KEY_B = bytes(range(32)), bytes(range(100, 132))


def _device_count():
    return int(G.load_library().garage_ec_device_count())


LISTS = [pytest.param([0, 0], id="0-0"),
         pytest.param([0, 1], id="0-1", marks=pytest.mark.skipif("_device_count() < 2", reason="one GPU visible"))]
CODES = {"rs": dict(k=10, m=4), "lrc": dict(k=10, m=4, local_groups=2), "pb": dict(k=10, m=4, piggyback=True),
         "clay": dict(k=10, m=4, clay=True)}


def _batches(bm):
    return [g["batches"] for g in bm.device_metrics()]


def _blocks(seed, sizes=SIZES):
    blocks = [O.fill_random(n, seed + i) for i, n in enumerate(sizes)]
    return blocks, [BM.blake2sum(b) for b in blocks]


def _calls(bm, blocks, hashes):
    """every PUT and GET kind on bm -> what a user sees of them (bytes, content addresses, checksums)"""
    out = []
    for h, b in zip(hashes, blocks):
        assert bm.rpc_put_block(h, b) == BM.OK
        rc, got = bm.rpc_get_block(h)
        assert rc == BM.OK
        off = len(b) // 3
        rc, part = bm.rpc_get_block_range(h, off, len(b) - off - 1 if len(b) > 2 else 1)
        assert rc == BM.OK
        out += [got.tobytes(), part.tobytes()]
    for b in blocks:  # sealed with the plaintext's CRC32C: a fresh nonce, so the address is the sealed block's hash
        rc, sh, crc = bm.rpc_put_block_sealed_crc(KEY_A, b, BM.CRC32C)
        assert rc == BM.OK
        rc, sealed = bm.rpc_get_block(sh, cap=len(b) + 8192)  # the sealed block: nonce prefix and chunk tags
        assert rc == BM.OK and BM.blake2sum(sealed) == sh
        rc, plain = bm.rpc_get_block_opened(sh, KEY_A)
        assert rc == BM.OK
        off = len(b) // 2
        rc, part = bm.rpc_get_block_range_opened(sh, KEY_A, off, len(b) - off)
        assert rc == BM.OK
        out += [crc, plain.tobytes(), part.tobytes()]
    pieces = [(hashes[0], 7, 3000), (hashes[3], 1000, 50000)]
    rc, rh, rlen, crc = bm.put_block_resealed_crc(pieces, None, KEY_B, BM.CRC32C)
    assert rc == BM.OK
    rc, plain = bm.rpc_get_block_opened(rh, KEY_B)
    assert rc == BM.OK
    out += [crc, rlen, plain.tobytes()]
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("devices", LISTS)
@pytest.mark.parametrize("code", list(CODES))
def test_same_bytes_as_one_device(code, devices):
    blocks, hashes = _blocks(0x5100)
    with BM.BlockManager(**CODES[code]) as one:
        want = _calls(one, blocks, hashes)
    with BM.BlockManager(**CODES[code], cuda_devices=devices) as bm:
        got = _calls(bm, blocks, hashes)
        # concurrent PUTs and GETs of other blocks, landing on both groups
        more, mh = _blocks(0x5200, [65536 + 4096 * i for i in range(32)])
        errs = []

        def put_get(i):
            rc = bm.rpc_put_block(mh[i], more[i])
            rc2, g = bm.rpc_get_block(mh[i])
            if rc != BM.OK or rc2 != BM.OK or not np.array_equal(g, more[i]):
                errs.append(i)

        th = [threading.Thread(target=put_get, args=(i,)) for i in range(len(more))]
        [t.start() for t in th]
        [t.join() for t in th]
        assert not errs
        dm = bm.device_metrics()
        assert [g["cuda_device"] for g in dm] == devices
        assert all(g["batches"] > 0 and g["blocks"] > 0 and g["bytes"] > 0 for g in dm), dm
        assert sum(g["routed_local"] + g["routed_remote"] for g in dm) > 0
    assert got == want
    for i, b in enumerate(blocks):
        assert got[2 * i] == b.tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize("devices", LISTS)
def test_degraded_reads_and_repairs_through_two_groups(tmp_path, devices):
    d = str(tmp_path / "store")
    blocks, hashes = _blocks(0x6100)
    with BM.BlockManager(k=10, m=4, data_dir=d, batch_max_blocks=8, cuda_devices=devices) as bm:
        for h, b in zip(hashes, blocks):
            assert bm.rpc_put_block(h, b) == BM.OK
        # degraded GETs with m holders down
        b0 = sum(_batches(bm))
        for n in range(4):
            assert bm.set_node_up(n, False) == BM.OK
        for h, b in zip(hashes, blocks):
            rc, got = bm.rpc_get_block(h)
            assert rc == BM.OK and np.array_equal(got, b)
        assert sum(_batches(bm)) > b0
        for n in range(4):
            assert bm.set_node_up(n, True) == BM.OK
        # resync of a node that lost its shards while m - 1 other holders are down: m shards of each stripe missing
        lost = 5
        for h in hashes:
            bm.drop_shard(lost, h)
        assert bm.repair_enqueue_missing(lost) == len(hashes)
        for n in range(3):
            bm.set_node_up(n, False)
        b0 = sum(_batches(bm))
        failed, done = bm.resync_all(lost, workers=4)
        assert failed == 0 and done == len(hashes) and sum(_batches(bm)) > b0
        for n in range(3):
            bm.set_node_up(n, True)
        assert all(bm.node_shard_index(lost, h) >= 0 for h in hashes if lost in bm.storage_nodes_of(h))
        # the stale-shard hunt: a data shard with a valid tag and other bytes
        h, b = hashes[2], blocks[2]
        assert bm.plant_stale_shard(bm.storage_nodes_of(h)[1], h) == BM.OK
        rc, got = bm.rpc_get_block(h)
        assert rc == BM.OK and np.array_equal(got, b)
        # deep scrub: a stale parity shard is quarantined
        h = hashes[0]
        assert bm.plant_stale_shard(bm.storage_nodes_of(h)[11], h) == BM.OK
        b0 = sum(_batches(bm))
        repaired = 0
        for n in range(bm.n_nodes):
            rc, _, _, _, rep = bm.deep_scrub_step(n)
            assert rc == BM.OK
            repaired += rep
        assert repaired >= 1 and bm.metrics()["deep_scrub_parity_bad"] >= 1 and sum(_batches(bm)) > b0
        for h, b in zip(hashes, blocks):
            rc, got = bm.rpc_get_block(h)
            assert rc == BM.OK and np.array_equal(got, b)
        assert all(x > 0 for x in _batches(bm)), bm.device_metrics()


@pytest.mark.gpu
@pytest.mark.parametrize("devices", LISTS)
def test_conversion_sweep_through_two_groups(tmp_path, devices):
    d = str(tmp_path / "store")
    blocks, hashes = _blocks(0x7100)
    with BM.BlockManager(k=6, m=3, n_nodes=14, data_dir=d, batch_max_blocks=4) as old:
        for h, b in zip(hashes, blocks):
            assert old.rpc_put_block(h, b) == BM.OK
    with BM.BlockManager(k=10, m=4, n_nodes=14, data_dir=d, batch_max_blocks=4, previous_codes=[(6, 3, 0, 0)],
                         cuda_devices=devices) as bm:
        b0 = _batches(bm)
        assert bm.convert_all() == len(blocks)
        assert bm.metrics()["convert_blocks"] == len(blocks)
        assert sum(_batches(bm)) > sum(b0)
        for h, b in zip(hashes, blocks):
            rc, got = bm.rpc_get_block(h)
            assert rc == BM.OK and np.array_equal(got, b)
        assert all(x > 0 for x in _batches(bm)), bm.device_metrics()


@pytest.mark.gpu
@pytest.mark.parametrize("devices", LISTS)
def test_layout_change_through_two_groups(tmp_path, devices):
    d = str(tmp_path / "store")
    n, dead, cap = 16, 3, 1 << 40
    cap15 = [cap] * 15 + [0]
    blocks, hashes = _blocks(0x8100)
    with BM.BlockManager(k=10, m=4, n_nodes=n, data_dir=d, batch_max_blocks=8, cuda_devices=devices,
                         layout=dict(zone=[0] * n, capacity=cap15)) as bm:
        for h, b in zip(hashes, blocks):
            assert bm.rpc_put_block(h, b) == BM.OK
        held = sum(dead in bm.storage_nodes_of(h) for h in hashes)
        assert bm.set_node_up(dead, False) == BM.OK
        assert bm.apply_layout([0] * n, [c if i != dead else 0 for i, c in enumerate(cap15)]) == (BM.OK, 2)
        b0 = sum(_batches(bm))
        bm.layout_sync_all()
        mt = bm.metrics()
        assert mt["layout_sync_errors"] == 0 and bm.layout_versions() == [2]
        if held:
            assert mt["layout_shards_rebuilt"] >= 1 and sum(_batches(bm)) > b0
        for h, b in zip(hashes, blocks):
            rc, got = bm.rpc_get_block(h)
            assert rc == BM.OK and np.array_equal(got, b)
        assert all(x > 0 for x in _batches(bm)), bm.device_metrics()


def _node_cpus(node):
    path = "/sys/devices/system/node/node%d/cpulist" % node
    if not os.path.exists(path):
        return set()
    cpus = set()
    for part in open(path).read().strip().split(","):
        if part:
            a, _, b = part.partition("-")
            cpus.update(range(int(a), int(b or a) + 1))
    return cpus & os.sched_getaffinity(0)


@pytest.mark.gpu
@pytest.mark.parametrize("devices", LISTS)
def test_a_thread_on_a_gpus_node_is_routed_locally(devices):
    blocks, hashes = _blocks(0x9100, [65536] * 8)
    with BM.BlockManager(k=10, m=4, cuda_devices=devices) as bm:
        nodes = sorted({g["numa_node"] for g in bm.device_metrics() if g["numa_node"] >= 0})
        if not nodes:
            pytest.skip("the GPUs' NUMA nodes are unknown on this host")
        for node in nodes:
            cpus = _node_cpus(node)
            if not cpus:
                continue
            before = bm.device_metrics()
            res = []

            def run():
                os.sched_setaffinity(0, cpus)  # this thread only
                for h, b in zip(hashes, blocks):
                    res.append(bm.rpc_put_block(h, b))
                    rc, got = bm.rpc_get_block(h)
                    res.append(rc if got is None or np.array_equal(got, b) else -99)

            t = threading.Thread(target=run)
            t.start()
            t.join()
            assert res and all(r == BM.OK for r in res)
            after = bm.device_metrics()
            assert sum(a["routed_remote"] - b["routed_remote"] for a, b in zip(after, before)) == 0
            for a, b in zip(after, before):  # every call went to a group on that node
                grew = a["routed_local"] - b["routed_local"]
                assert grew == 0 or a["numa_node"] == node
            assert sum(a["routed_local"] - b["routed_local"] for a, b in zip(after, before)) == 2 * len(blocks)


@pytest.mark.gpu
@pytest.mark.parametrize("devices", LISTS)
def test_each_groups_pools_are_on_its_gpus_node(devices):
    n_nodes = len([x for x in os.listdir("/sys/devices/system/node") if x.startswith("node")]) \
        if os.path.isdir("/sys/devices/system/node") else 1
    with BM.BlockManager(k=10, m=4, cuda_devices=devices) as bm:
        for dev, g in zip(devices, bm.device_metrics()):
            ec = G.GarageEc(device=dev, k=10, m=4)
            try:
                gpu_node, _ = ec.numa_info()
            finally:
                ec.close()
            assert g["numa_node"] == gpu_node
            if n_nodes > 1 and gpu_node >= 0:
                assert g["pool_numa_node"] == gpu_node, g


@pytest.mark.gpu
def test_refusals_and_teardown(tmp_path):
    n = _device_count()
    for devs in ([n], [0, n], [0] * 17, [], [-1]):
        with pytest.raises(BM.BlockManagerError) as e:
            BM.BlockManager(k=4, m=2, data_dir=str(tmp_path / "s"), cuda_devices=devs)
        assert e.value.code == E_INVALID
        assert not (tmp_path / "s").exists()

    def threads():
        return len(os.listdir("/proc/self/task"))

    BM.BlockManager(k=4, m=2, n_nodes=6, batch_max_blocks=4, cuda_devices=[0]).close()  # the driver's own threads
    base = threads()
    for devs in ([0, 0], [0, 0, 0, 0], list(range(min(n, 4)))):
        bm = BM.BlockManager(k=4, m=2, n_nodes=6, batch_max_blocks=4, cuda_devices=devs)
        assert len(bm.device_metrics()) == len(devs)
        assert threads() >= base + 2 * 3 * len(devs)  # two batchers of three dispatchers per group
        b = O.fill_random(4096, 1)
        assert bm.rpc_put_block(BM.blake2sum(b), b) == BM.OK
        bm.close()
        assert threads() == base, "destroy joins every group's threads"
