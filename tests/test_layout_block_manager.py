"""Changing the cluster layout under the block manager (DESIGN.md section 5.2): PUTs go to every active layout version,
`layout_sync_step` moves shards to their new holders (a copy from the old holder first, a GPU rebuild when that copy is
gone), old shards are deleted only once the newest stripe holds k+1, and the old version retires once every storage
node has synced.  File stores in tmp_path; a "restart" is a new manager on the same data_dir."""
import ctypes as C
import os
import shutil
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import oracle_lib as O  # noqa: E402
import transcode_oracle as TO  # noqa: E402

from garage_b200 import block_manager as BM  # noqa: E402
from garage_b200 import placement as PL  # noqa: E402

E_INVALID = -1
N = 16
CAP = 1 << 40
RS = ("rs", 10, 4)


def code_kw(code):
    if code[0] == "lrc":
        return {"k": code[1], "m": code[2] + code[3], "local_groups": code[2]}
    return {"k": code[1], "m": code[2], "piggyback": code[0] == "pb"}


def oracle_code(code):
    return code + (0,) if code[0] in ("rs", "pb") else code


def spec(capacity, **kw):
    return dict(zone=[0] * len(capacity), capacity=capacity, **kw)


def manager(d, code=RS, n=N, **kw):
    kw.setdefault("batch_max_blocks", 8)  # small pinned pools: these tests create many managers
    return BM.BlockManager(n_nodes=n, data_dir=d, **code_kw(code), **kw)


def path(d, node, h, ext):
    return os.path.join(d, "node%d" % node, h[:1].hex(), h[1:2].hex(), h.hex() + ext)


def make_blocks(sizes, seed):
    blocks = [O.fill_random(n, seed + i) for i, n in enumerate(sizes)]
    return blocks, [BM.blake2sum(b) for b in blocks]


def put_all(bm, blocks, hashes):
    for h, b in zip(hashes, blocks):
        assert bm.rpc_put_block(h, b) == BM.OK


def assert_gets(bm, blocks, hashes):
    for h, b in zip(hashes, blocks):
        rc, got = bm.rpc_get_block(h)
        assert rc == BM.OK and np.array_equal(got, b)


def files(d):
    """node -> sorted file names below it"""
    out = {}
    for name in sorted(os.listdir(d)):
        if name.startswith("node"):
            out[int(name[4:])] = sorted(n for _, _, ns in os.walk(os.path.join(d, name)) for n in ns)
    return out


def assert_placement(bm, d, code, blocks, hashes, n=N):
    """every node holds exactly the shards the newest ring gives it, each equal to the oracle's encode"""
    want = {node: [] for node in range(n)}
    for h, b in zip(hashes, blocks):
        ref = TO.encode_block(oracle_code(code), b)
        for i, node in enumerate(bm.storage_nodes_of(h)):
            want[node].append(h.hex() + ".shard")
            with open(path(d, node, h, ".shard"), "rb") as f:
                raw = f.read()
            assert raw[:4] == b"GEC1" and raw[6] == i and raw[64:] == ref[i].tobytes(), (node, i)
    got = files(d)
    for node in range(n):
        assert got.get(node, []) == sorted(want[node]), node


def moves(old_rows, new_rows):
    return sum(sum(a != b for a, b in zip(r0, r1)) for r0, r1 in zip(old_rows, new_rows))


def write_layout_file(d, n, tot, rings, synced=None):
    """<data_dir>/layout with explicit rings (one per version, 256 rows of tot nodes)"""
    s = "garage-bm-layout 1\nnodes %d shards %d\n" % (n, tot)
    for v, ring in enumerate(rings, 1):
        s += "version %d\nzone %s\ncapacity %s\nring %s\n" % (
            v, " ".join(["0"] * n), " ".join([str(CAP)] * n), bytes(x for row in ring for x in row).hex())
    s += "synced %s\n" % " ".join(str(x) for x in (synced or [0] * n))
    os.makedirs(d, exist_ok=True)
    with open(os.path.join(d, "layout"), "w") as f:
        f.write(s)


# ---------------------------------------------------------------- CPU: configuration checks
@pytest.mark.parametrize("kw", [
    spec([CAP] * 13 + [0] * 3),                          # 13 storage nodes for 14 shards
    spec([CAP] * N, max_per_zone=5),                     # a zone could lose more than m shards
    spec([CAP] * N, max_per_zone=-1),
    spec([CAP] * N, zone_redundancy=-1),
    spec([CAP] * N, zone_redundancy=2),                  # one zone: infeasible
    dict(zone=[0] * 8 + [1] * 8, capacity=[CAP] * N, max_per_zone=4),  # 14 shards in 2 zones of at most 4: infeasible
])
def test_bad_layouts_are_rejected_before_any_cuda_call(kw):
    with pytest.raises(BM.BlockManagerError) as e:
        BM.BlockManager(k=10, m=4, n_nodes=N, layout=kw)
    assert e.value.code == E_INVALID


def test_null_layout_arrays_are_rejected():
    L = BM.load_library()
    cfg = BM.Config()
    L.garage_bm_default_config(C.byref(cfg))
    assert not cfg.layout  # default: the fixed ring
    cap = (C.c_uint64 * 14)(*([CAP] * 14))
    sp = BM.LayoutSpec(None, C.cast(cap, C.POINTER(C.c_uint64)), 0, 0)
    cfg.layout = C.pointer(sp)
    h = C.c_void_p()
    assert L.garage_bm_create(C.byref(h), C.byref(cfg)) == E_INVALID and not h.value


def test_unusable_layout_file_is_rejected(tmp_path):
    d = str(tmp_path / "store")
    os.makedirs(d)
    with open(os.path.join(d, "layout"), "w") as f:
        f.write("garage-bm-layout 1\nnodes 14 shards 14\nversion 1\nzone 0\n")
    with pytest.raises(BM.BlockManagerError) as e:
        BM.BlockManager(k=10, m=4, n_nodes=14, data_dir=d)
    assert e.value.code == E_INVALID
    # two active versions and a code change at once
    ring = [[(p % 14 + i) % 14 for i in range(14)] for p in range(256)]
    write_layout_file(d, 14, 14, [ring, [r[1:] + r[:1] for r in ring]])
    with pytest.raises(BM.BlockManagerError) as e:
        BM.BlockManager(k=10, m=4, n_nodes=14, data_dir=d, previous_codes=[(6, 3, 0, 0)])
    assert e.value.code == E_INVALID


# ---------------------------------------------------------------- GPU
@pytest.mark.gpu
def test_add_nodes_copies_every_moved_shard(tmp_path):
    d = str(tmp_path / "store")
    cap14 = [CAP] * 14 + [0, 0]
    blocks, hashes = make_blocks([1 << 20, 3073, 777777, (1 << 20) - 1, 65536, 5, 1 << 20, 300001] * 2, 0x8100)
    old, new = (blocks[:8], hashes[:8]), (blocks[8:], hashes[8:])
    with manager(d, layout=spec(cap14)) as bm:
        put_all(bm, *old)
        rows1 = [bm.storage_nodes_of(h) for h in old[1]]
        assert all(max(r) < 14 for r in rows1) and bm.layout_versions() == [1]
        assert bm.apply_layout([0] * N, [CAP] * N) == (BM.OK, 2)
        assert bm.layout_versions() == [1, 2] and bm.metrics()["layout_version"] == 2
        rows2 = [bm.storage_nodes_of(h) for h in old[1]]
        l1 = PL.Layout.compute([0] * N, cap14, 14)
        l2 = PL.Layout.compute([0] * N, [CAP] * N, 14, previous=l1, version=2)
        expect = sum(len(l1.transition_to(l2, PL.partition_of(h))) for h in old[1])
        assert expect == moves(rows1, rows2) > 0
        assert rows2 == [l2.nodes_of(h) for h in old[1]]
        # the new blocks go to both versions: their old holders of a moved index delete it too
        deleted = expect + moves([l1.nodes_of(h) for h in new[1]], [l2.nodes_of(h) for h in new[1]])
        put_all(bm, *new)  # to both versions
        assert_gets(bm, blocks, hashes)
    with manager(d) as bm:  # restart: the layout file wins
        assert bm.layout_versions() == [1, 2]
        assert_gets(bm, blocks, hashes)
        moved = bm.layout_sync_all()
        mt = bm.metrics()
        assert moved == expect and mt["layout_shards_copied"] == expect and mt["layout_shards_rebuilt"] == 0
        assert mt["layout_deleted"] == deleted and mt["layout_sync_errors"] == 0 and mt["corruption_counter"] == 0
        assert bm.layout_versions() == [2]
        assert_placement(bm, d, RS, blocks, hashes)
        assert_gets(bm, blocks, hashes)
        assert bm.layout_sync_all() == 0
    with manager(d) as bm:
        assert bm.layout_versions() == [2]
        assert_gets(bm, blocks, hashes)


@pytest.mark.gpu
@pytest.mark.parametrize("code", [("rs", 10, 4), ("lrc", 10, 2, 2), ("pb", 10, 4)], ids=lambda c: "".join(map(str, c)))
def test_removing_a_dead_node_rebuilds_its_shards(tmp_path, code):
    d = str(tmp_path / "store")
    dead, k = 3, code[1]
    cap15 = [CAP] * 15 + [0]
    sizes = [1 << 20, 777777, 65536, (1 << 20) - 1, 300001, 4096]
    with manager(d, code, layout=spec(cap15)) as bm:
        # blocks whose shard on the dead node is a data shard: the cheap repairs of LRC and PB apply
        blocks, hashes, seed = [], [], 0x8200
        while len(blocks) < len(sizes):
            b = O.fill_random(sizes[len(blocks)], seed)
            h = BM.blake2sum(b)
            seed += 1
            row = bm.storage_nodes_of(h)
            if dead in row and row.index(dead) < k:
                blocks.append(b)
                hashes.append(h)
        put_all(bm, blocks, hashes)
        assert bm.set_node_up(dead, False) == BM.OK
        assert bm.apply_layout([0] * N, [c if n != dead else 0 for n, c in enumerate(cap15)]) == (BM.OK, 2)
        assert_gets(bm, blocks, hashes)
        bm.layout_sync_all()
        mt = bm.metrics()
        assert mt["layout_shards_copied"] == 0 and mt["layout_shards_rebuilt"] == len(blocks)
        assert mt["layout_sync_errors"] == 0 and bm.layout_versions() == [2]  # a removed node need not sync
        lens = [TO.shard_len(oracle_code(code), b.size) for b in blocks]
        if code[0] == "rs":
            assert mt["layout_bytes_read"] == sum(k * L for L in lens)
        elif code[0] == "lrc":
            assert mt["layout_bytes_read"] == sum(k // code[2] * L for L in lens)  # the shard's local group
        else:
            assert sum(13 * L // 2 for L in lens) <= mt["layout_bytes_read"] <= sum(14 * L // 2 for L in lens)
        shutil.rmtree(os.path.join(d, "node%d" % dead))
        os.makedirs(os.path.join(d, "node%d" % dead))
        assert_placement(bm, d, code, blocks, hashes)
        assert_gets(bm, blocks, hashes)


def rotated_store(d, code, n, blocks, hashes):
    """a store written under the fixed ring, then an explicit version 2 in which every node moves to the next index"""
    tot = TO.k_of(code) + TO.m_of(code)
    with manager(d, code, n=n) as bm:
        put_all(bm, blocks, hashes)
    ring = [[(p % n + i) % n for i in range(tot)] for p in range(256)]
    write_layout_file(d, n, tot, [ring, [r[1:] + r[:1] for r in ring]])


@pytest.mark.gpu
def test_a_node_at_two_indices_keeps_both_until_the_new_one_is_synced(tmp_path):
    d = str(tmp_path / "store")
    blocks, hashes = make_blocks([1 << 20, 12345], 0x8300)
    rotated_store(d, RS, 14, blocks[:1], hashes[:1])
    with manager(d, n=14) as bm:
        assert bm.layout_versions() == [1, 2]
        assert bm.rpc_put_block(hashes[1], blocks[1]) == BM.OK
        h = hashes[1]
        for node in range(14):  # the new block: both indices on every node, the newest one in .shard
            new_i = bm.storage_nodes_of(h).index(node)
            assert bm.node_shard_index(node, h) == new_i
            assert os.path.exists(path(d, node, h, ".legacy"))
        assert_gets(bm, blocks, hashes)
        assert bm.layout_sync_all() == 14  # the old block: every node receives its new index
        assert bm.layout_versions() == [2]
        bm.layout_sync_all()  # the old indices go once the newest stripe holds k+1
        assert bm.metrics()["layout_deleted"] == 28
        assert_placement(bm, d, RS, blocks, hashes, n=14)
        assert_gets(bm, blocks, hashes)


@pytest.mark.gpu
def test_a_corrupt_old_holder_leads_to_a_rebuild(tmp_path):
    d = str(tmp_path / "store")
    cap14 = [CAP] * 14 + [0, 0]
    blocks, hashes = make_blocks([1 << 20, 1 << 20, 1 << 20, 1 << 20], 0x8400)
    with manager(d, layout=spec(cap14)) as bm:
        put_all(bm, blocks, hashes)
        rows1 = [bm.storage_nodes_of(h) for h in hashes]
        assert bm.apply_layout([0] * N, [CAP] * N)[0] == BM.OK
        rows2 = [bm.storage_nodes_of(h) for h in hashes]
        j = next(j for j in range(len(hashes)) if rows1[j] != rows2[j])
        i = next(i for i in range(14) if rows1[j][i] != rows2[j][i])
        assert bm.corrupt_shard(rows1[j][i], hashes[j], 1000) == BM.OK
        bm.layout_sync_all()
        mt = bm.metrics()
        assert mt["layout_shards_rebuilt"] == 1 and mt["layout_shards_copied"] == moves(rows1, rows2) - 1
        assert mt["corruption_counter"] == 1
        os.remove(path(d, rows1[j][i], hashes[j], ".corrupted"))
        assert_placement(bm, d, RS, blocks, hashes)


@pytest.mark.gpu
def test_write_quorum_is_needed_in_every_version(tmp_path):
    d = str(tmp_path / "store")
    cap14 = [CAP] * 14 + [0, 0]
    cands, chashes = make_blocks([65536] * 64, 0x8500)
    with manager(d, layout=spec(cap14)) as bm:
        rows1 = {h: bm.storage_nodes_of(h) for h in chashes}
        assert bm.apply_layout([0] * N, [CAP] * N)[0] == BM.OK
        rows2 = {h: bm.storage_nodes_of(h) for h in chashes}
        # a block already stored whose new stripe has both new nodes
        j0 = next(j for j, h in enumerate(chashes) if {14, 15} <= set(rows2[h]))
        h0 = chashes[j0]
        both = [x for x in rows2[h0] if x in rows1[h0]][:2]
        ro = [14, 15] + both  # version 2 loses 4 of 14, version 1 only 2
    shutil.rmtree(d)
    with manager(d, layout=spec(cap14)) as bm:
        assert bm.rpc_put_block(h0, cands[j0]) == BM.OK
        assert bm.apply_layout([0] * N, [CAP] * N)[0] == BM.OK
        for x in ro:
            assert bm.set_node_readonly(x, True) == BM.OK
        j1 = next(j for j, h in enumerate(chashes) if j != j0 and set(ro) <= set(rows2[h]))
        assert bm.rpc_put_block(chashes[j1], cands[j1]) == BM.E_QUORUM
        bm.layout_sync_all([n for n in range(N) if n not in ro])
        mt = bm.metrics()
        assert mt["layout_deleted"] == 0 and mt["layout_shards_copied"] == 0
        for i, node in enumerate(rows1[h0]):  # every old shard is still there
            assert node in ro or bm.node_shard_index(node, h0) == i
        for x in ro:
            assert bm.set_node_readonly(x, False) == BM.OK
        assert_gets(bm, [cands[j0]], [h0])
        bm.layout_sync_all()
        bm.layout_sync_all()
        assert bm.layout_versions() == [2] and bm.metrics()["layout_deleted"] > 0
        # the PUT that missed version 2's quorum still stored version 1's stripe: its block moves like the other
        both = ([cands[j0], cands[j1]], [h0, chashes[j1]])
        assert_gets(bm, *both)
        assert_placement(bm, d, RS, *both)


@pytest.mark.gpu
def test_layout_sync_is_crash_safe_at_every_step(tmp_path):
    """stop the sync after n file operations (renames, shard writes, deletes), restart, read every block, then sync
    to the end"""
    code, n_nodes = ("rs", 4, 2), 6
    pristine = str(tmp_path / "pristine")
    blocks, hashes = make_blocks([1 << 20, 5], 0x8600)
    rotated_store(pristine, code, n_nodes, blocks, hashes)
    n, finished = 0, False
    while not finished:
        d = str(tmp_path / ("run%d" % n))
        shutil.copytree(pristine, d)
        with manager(d, code, n=n_nodes) as bm:
            bm.debug_convert_stop_after(n)
            for _ in range(2):
                bm.layout_sync_all()
            mt = bm.metrics()
            finished = mt["layout_shards_copied"] + mt["layout_shards_rebuilt"] == 12 and mt["layout_deleted"] == 12
        with manager(d, code, n=n_nodes) as bm:  # restart after the "crash"
            assert_gets(bm, blocks, hashes)
            assert bm.metrics()["corruption_counter"] == 0
            for _ in range(2):
                bm.layout_sync_all()
            assert bm.layout_versions() == [2] and bm.metrics()["layout_sync_errors"] == 0
            assert_placement(bm, d, code, blocks, hashes, n=n_nodes)
        with manager(d, code, n=n_nodes) as bm:
            assert_gets(bm, blocks, hashes)
        shutil.rmtree(d)
        n += 1
    assert n > 2 * 6 * 3  # every rename, write and delete of two blocks' moves was a stop point


@pytest.mark.gpu
def test_a_down_storage_node_stalls_retirement(tmp_path):
    d = str(tmp_path / "store")
    cap14 = [CAP] * 14 + [0, 0]
    blocks, hashes = make_blocks([1 << 20, 65536, 3073], 0x8700)
    with manager(d, layout=spec(cap14)) as bm:
        put_all(bm, blocks, hashes)
        assert bm.apply_layout([0] * N, [CAP] * N)[0] == BM.OK
        assert bm.set_node_up(15, False) == BM.OK
        bm.layout_sync_all()
        assert bm.layout_versions() == [1, 2]
        assert_gets(bm, blocks, hashes)
        assert bm.set_node_up(15, True) == BM.OK
        assert bm.layout_sync_step(15)[0] == BM.OK
        assert bm.layout_versions() == [2]
        bm.layout_sync_all()
        assert_placement(bm, d, RS, blocks, hashes)


@pytest.mark.gpu
def test_resync_alone_completes_a_move(tmp_path):
    d = str(tmp_path / "store")
    cap14 = [CAP] * 14 + [0, 0]
    blocks, hashes = make_blocks([1 << 20, 777777, 5, 65536], 0x8800)
    with manager(d, layout=spec(cap14)) as bm:
        put_all(bm, blocks, hashes)
        rows1 = [bm.storage_nodes_of(h) for h in hashes]
        assert bm.apply_layout([0] * N, [CAP] * N)[0] == BM.OK
        rows2 = [bm.storage_nodes_of(h) for h in hashes]
        for node in range(N):
            bm.repair_enqueue_missing(node)
            assert bm.resync_all(node)[0] == 0
        assert bm.metrics()["layout_shards_copied"] == moves(rows1, rows2) > 0
        for h, b, row in zip(hashes, blocks, rows2):
            ref = TO.encode_block(oracle_code(RS), b)
            for i, node in enumerate(row):
                with open(path(d, node, h, ".shard"), "rb") as f:
                    assert f.read()[64:] == ref[i].tobytes()
        assert_gets(bm, blocks, hashes)


@pytest.mark.gpu
def test_apply_layout_rejections(tmp_path):
    with BM.BlockManager(k=10, m=4, n_nodes=N, batch_max_blocks=8) as bm:  # the memory store
        assert bm.apply_layout([0] * N, [CAP] * N) == (E_INVALID, 0)
        assert bm.layout_versions() == [1]
    d = str(tmp_path / "store")
    for kw in ({"previous_codes": [(6, 3, 0, 0)]}, {"legacy_replicas": 3}):  # a code change in progress
        with manager(d, **kw) as bm:
            assert bm.apply_layout([0] * N, [CAP] * N) == (E_INVALID, 0)
            assert bm.layout_versions() == [1]
    assert not os.path.exists(os.path.join(d, "layout"))
    with manager(d) as bm:
        for bad in (spec([CAP] * N, zone_redundancy=2), spec([CAP] * 13 + [0] * 3), spec([CAP] * N, max_per_zone=5)):
            assert bm.apply_layout(**bad) == (E_INVALID, 0)
        assert not os.path.exists(os.path.join(d, "layout")) and bm.layout_versions() == [1]
        caps = [[CAP] * N, [CAP] * 15 + [0], [CAP] * 14 + [0, 0]]
        for v, cap in enumerate(caps, 2):
            assert bm.apply_layout([0] * N, cap) == (BM.OK, v)
        assert bm.layout_versions() == [1, 2, 3, 4]
        assert bm.apply_layout([0] * N, [CAP] * N) == (E_INVALID, 0)  # a fifth active version
        assert bm.layout_versions() == [1, 2, 3, 4]
    with manager(d) as bm:
        assert bm.layout_versions() == [1, 2, 3, 4]


@pytest.mark.gpu
def test_concurrent_syncs_of_every_node_finish(tmp_path):
    """one sync per node at once, with GETs alongside, on a stripe-slot pool of 4 x 2 slots: every rebuild batch
    takes its slots in one step, so no mix of callers can hold the pool between them"""
    import threading

    d = str(tmp_path / "store")
    dead = 5
    cap15 = [CAP] * 15 + [0]
    with manager(d, layout=spec(cap15), batch_max_blocks=2) as bm:
        blocks, hashes, seed = [], [], 0x8900
        while len(blocks) < 24:
            b = O.fill_random(200000 + 4099 * len(blocks), seed)
            h = BM.blake2sum(b)
            seed += 1
            if dead in bm.storage_nodes_of(h):
                blocks.append(b)
                hashes.append(h)
        put_all(bm, blocks, hashes)
        assert bm.set_node_up(dead, False) == BM.OK
        assert bm.apply_layout([0] * N, [c if n != dead else 0 for n, c in enumerate(cap15)])[0] == BM.OK
        rcs, bad = [], []

        def sync(node):
            rcs.append(bm.layout_sync_step(node)[0])

        def gets():
            for h, b in zip(hashes, blocks):
                rc, got = bm.rpc_get_block(h)
                if rc != BM.OK or not np.array_equal(got, b):
                    bad.append(h)

        th = [threading.Thread(target=sync, args=(n,), daemon=True) for n in range(N) if n != dead]
        th += [threading.Thread(target=gets, daemon=True) for _ in range(4)]
        for t in th:
            t.start()
        for t in th:
            t.join(timeout=300)
        assert not any(t.is_alive() for t in th)
        assert rcs == [BM.OK] * (N - 1) and bad == []
        mt = bm.metrics()
        assert mt["layout_shards_rebuilt"] == len(blocks) and mt["layout_sync_errors"] == 0
        assert bm.layout_versions() == [2]
        shutil.rmtree(os.path.join(d, "node%d" % dead))
        os.makedirs(os.path.join(d, "node%d" % dead))
        assert_placement(bm, d, RS, blocks, hashes)
