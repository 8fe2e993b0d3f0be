"""Changing the cluster layout under a Clay store (`clay_layout = 1`, DESIGN.md sections 5.2 and 5.3): shards move by
copy like any other code's, a removed node's shards are rebuilt from the garage_ec_read_ranges runs of the 13 others
(1/4 of each, every helper read whole from the first active version that has it), a bad helper makes way for its next
source or for k whole shards, the sync survives a stop at every file operation, and the deep scrub works across two
versions.  Without `clay_layout` a Clay store refuses every layout, as before.  File stores in tmp_path; a "restart" is
a new manager on the same data_dir."""
import ctypes as C
import os
import shutil
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import clay_oracle as CO  # noqa: E402
import oracle_lib as O  # noqa: E402

import garage_b200 as G  # noqa: E402
from garage_b200 import block_manager as BM  # noqa: E402
from garage_b200 import placement as PL  # noqa: E402

E_INVALID = -1
N = 16
CAP = 1 << 40
MIB = 1 << 20


def spec(capacity, **kw):
    return dict(zone=[0] * len(capacity), capacity=capacity, **kw)


def manager(d, n=N, k=10, m=4, **kw):
    kw.setdefault("batch_max_blocks", 8)  # small pinned pools: these tests create many managers
    kw.setdefault("clay_layout", True)
    return BM.BlockManager(k=k, m=m, n_nodes=n, data_dir=d, clay=True, **kw)


def path(d, node, h, ext):
    return os.path.join(d, "node%d" % node, h[:1].hex(), h[1:2].hex(), h.hex() + ext)


def file_of_index(d, node, h, i):
    """the node's file (.shard or .legacy) whose header names shard index i"""
    for ext in (".shard", ".legacy"):
        p = path(d, node, h, ext)
        if os.path.exists(p):
            with open(p, "rb") as f:
                if f.read(7)[6] == i:
                    return p
    return None


def flip_byte(p, off=64 + 5000):
    with open(p, "r+b") as f:
        f.seek(off)
        b = f.read(1)[0]
        f.seek(off)
        f.write(bytes([b ^ 0x40]))


def make_blocks(sizes, seed):
    blocks = [O.fill_random(n, seed + i) for i, n in enumerate(sizes)]
    return blocks, [BM.blake2sum(b) for b in blocks]


def blocks_on(bm, node, sizes, seed):
    """blocks whose row in the manager's newest layout has a shard on `node`"""
    blocks, hashes = [], []
    while len(blocks) < len(sizes):
        b = O.fill_random(sizes[len(blocks)], seed)
        h = BM.blake2sum(b)
        seed += 1
        if node in bm.storage_nodes_of(h):
            blocks.append(b)
            hashes.append(h)
    return blocks, hashes


def put_all(bm, blocks, hashes):
    for h, b in zip(hashes, blocks):
        assert bm.rpc_put_block(h, b) == BM.OK


def assert_gets(bm, blocks, hashes):
    for h, b in zip(hashes, blocks):
        rc, got = bm.rpc_get_block(h)
        assert rc == BM.OK and np.array_equal(got, b)


def clay_stripe(b, k=10, m=4):
    """the oracle's Clay(k, m) shards of a block: (k+m, L)"""
    L = CO.shard_len(b.size, k, m)
    flat = np.zeros(k * L, dtype=np.uint8)
    flat[:b.size] = b
    data = flat.reshape(k, L)
    return np.concatenate([data, CO.encode(k, m, CO.build(k, m), data)])


def files(d):
    out = {}
    for name in sorted(os.listdir(d)):
        if name.startswith("node"):
            out[int(name[4:])] = sorted(n for _, _, ns in os.walk(os.path.join(d, name)) for n in ns)
    return out


def assert_placement(bm, d, blocks, hashes, n=N, k=10, m=4):
    """every node holds exactly the shards the newest ring gives it, each equal to the oracle's Clay encode"""
    want = {node: [] for node in range(n)}
    for h, b in zip(hashes, blocks):
        ref = clay_stripe(b, k, m)
        for i, node in enumerate(bm.storage_nodes_of(h)):
            want[node].append(h.hex() + ".shard")
            with open(path(d, node, h, ".shard"), "rb") as f:
                raw = f.read()
            assert raw[:4] == b"GEC1" and raw[6] == i and raw[53] == 2 and raw[64:] == ref[i].tobytes(), (node, i)
    got = files(d)
    for node in range(n):
        assert got.get(node, []) == sorted(want[node]), node


def moves(old_rows, new_rows):
    return sum(sum(a != b for a, b in zip(r0, r1)) for r0, r1 in zip(old_rows, new_rows))


def repair_bytes(size, k=10, m=4):
    """bytes a lone lost shard's rebuild is handed: the repair runs of the k+m-1 helpers (the same for every index)"""
    L = CO.shard_len(size, k, m)
    n = (k + m - 1) * sum(ln for _, ln in CO.repair_runs(k, m, 0, L))
    assert n == (k + m - 1) * L // m
    return n


def write_layout_file(d, n, tot, rings):
    s = "garage-bm-layout 1\nnodes %d shards %d\n" % (n, tot)
    for v, ring in enumerate(rings, 1):
        s += "version %d\nzone %s\ncapacity %s\nring %s\n" % (
            v, " ".join(["0"] * n), " ".join([str(CAP)] * n), bytes(x for row in ring for x in row).hex())
    s += "synced %s\n" % " ".join(["0"] * n)
    os.makedirs(d, exist_ok=True)
    with open(os.path.join(d, "layout"), "w") as f:
        f.write(s)


# ---------------------------------------------------------------- CPU: refused before any CUDA call
@pytest.mark.parametrize("kw", [
    {"clay": False, "clay_layout": 1},                                          # clay_layout without clay
    {"clay": False, "clay_layout": 1, "layout": spec([CAP] * N)},
    {"clay": True, "clay_layout": 2},                                           # not 0 / 1
    {"clay": True, "clay_layout": -1},
    {"clay": True, "clay_layout": 0, "layout": spec([CAP] * N)},                # the refusal without the opt-in
    {"clay": True, "clay_layout": 1, "local_groups": 2},                        # still not with LRC
    {"clay": True, "clay_layout": 1, "piggyback": True},                        # nor with PB
    {"clay": True, "clay_layout": 1, "layout": spec([CAP] * 13 + [0] * 3)},     # a layout any code would refuse
    {"clay": True, "clay_layout": 1, "layout": spec([CAP] * N, max_per_zone=5)},
])
def test_bad_clay_layout_configs_are_rejected_before_any_cuda_call(kw):
    with pytest.raises(BM.BlockManagerError) as e:
        BM.BlockManager(k=10, m=4, n_nodes=N, **kw)
    assert e.value.code == E_INVALID


def test_default_config_keeps_the_refusal():
    L = BM.load_library()
    cfg = BM.Config()
    cfg.clay_layout = 7
    L.garage_bm_default_config(C.byref(cfg))
    assert cfg.clay == 0 and cfg.clay_layout == 0


@pytest.mark.parametrize("clay_layout", [0, 1])
def test_layout_file_and_a_code_change_at_once_stay_refused(tmp_path, clay_layout):
    d = str(tmp_path / "store")
    ring = [[(p % 14 + i) % 14 for i in range(14)] for p in range(256)]
    write_layout_file(d, 14, 14, [ring, [r[1:] + r[:1] for r in ring]])
    with pytest.raises(BM.BlockManagerError) as e:
        BM.BlockManager(k=10, m=4, n_nodes=14, data_dir=d, clay=True, clay_layout=clay_layout,
                        previous_codes=[(6, 3, 0, 0)])
    assert e.value.code == E_INVALID


def test_a_layout_file_is_refused_without_clay_layout(tmp_path):
    d = str(tmp_path / "store")
    ring = [[(p % 14 + i) % 14 for i in range(14)] for p in range(256)]
    write_layout_file(d, 14, 14, [ring])
    with pytest.raises(BM.BlockManagerError) as e:
        BM.BlockManager(k=10, m=4, n_nodes=14, data_dir=d, clay=True)
    assert e.value.code == E_INVALID


# ---------------------------------------------------------------- GPU
@pytest.mark.gpu
def test_add_nodes_copies_every_moved_shard_and_a_restart_resumes(tmp_path):
    d = str(tmp_path / "store")
    cap14 = [CAP] * 14 + [0, 0]
    blocks, hashes = make_blocks([MIB, 3073, 777777, MIB - 1, 65536, 5, MIB, 300001, MIB, 31, 4097, 500000], 0xCA100)
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
        deleted = expect + moves([l1.nodes_of(h) for h in new[1]], [l2.nodes_of(h) for h in new[1]])
        put_all(bm, *new)  # to both versions
        assert_gets(bm, blocks, hashes)
        copied = 0
        for node in (15, 3, 14):  # part of the sync, reads in between
            rc, _, finished, n = bm.layout_sync_step(node)
            assert rc == BM.OK and finished
            copied += n
            assert_gets(bm, blocks, hashes)
        mt = bm.metrics()
        assert mt["layout_shards_copied"] == copied > 0 and mt["layout_shards_rebuilt"] == 0
        assert mt["layout_bytes_fetched"] == mt["layout_bytes_read"] > 0  # copies are whole shards
        assert bm.layout_versions() == [1, 2]
        deleted -= mt["layout_deleted"]
    with pytest.raises(BM.BlockManagerError) as e:  # the layout file is there now: the opt-in is needed to reopen
        manager(d, clay_layout=False)
    assert e.value.code == E_INVALID
    with manager(d) as bm:  # restart: the layout file wins, the sync resumes
        assert bm.layout_versions() == [1, 2]
        assert_gets(bm, blocks, hashes)
        moved = bm.layout_sync_all()
        mt = bm.metrics()
        assert copied + moved == expect and mt["layout_shards_copied"] == moved and mt["layout_shards_rebuilt"] == 0
        assert mt["layout_sync_errors"] == 0 and mt["corruption_counter"] == 0
        assert bm.layout_versions() == [2]
        bm.layout_sync_all()
        assert bm.metrics()["layout_deleted"] == deleted  # every old holder's copy of a moved index, once
        assert_placement(bm, d, blocks, hashes)
        assert_gets(bm, blocks, hashes)
        assert bm.layout_sync_all() == 0
    with manager(d) as bm:
        assert bm.layout_versions() == [2]
        assert_gets(bm, blocks, hashes)


@pytest.mark.gpu
def test_removing_a_dead_node_rebuilds_its_shards_from_a_quarter_of_each_helper(tmp_path):
    d = str(tmp_path / "store")
    dead = 3
    cap15 = [CAP] * 15 + [0]
    sizes = [MIB, 777777, 65536, MIB - 1, 300001, 4096, MIB, 5]
    with manager(d, layout=spec(cap15)) as bm:
        blocks, hashes = blocks_on(bm, dead, sizes, 0xCA200)
        lost = [bm.storage_nodes_of(h).index(dead) for h in hashes]
        assert min(lost) < 10 <= max(lost)  # data and parity shards alike
        put_all(bm, blocks, hashes)
        assert bm.set_node_up(dead, False) == BM.OK
        assert bm.apply_layout([0] * N, [c if n != dead else 0 for n, c in enumerate(cap15)]) == (BM.OK, 2)
        assert_gets(bm, blocks, hashes)
        per_step = []
        for node in range(N):
            if node == dead:
                continue
            m0 = bm.metrics()
            rc, _, finished, n = bm.layout_sync_step(node)
            assert rc == BM.OK and finished
            m1 = bm.metrics()
            per_step.append((m1["layout_bytes_fetched"] - m0["layout_bytes_fetched"],
                             m1["layout_bytes_read"] - m0["layout_bytes_read"]))
        mt = bm.metrics()
        assert mt["layout_shards_copied"] == 0 and mt["layout_shards_rebuilt"] == len(blocks)
        assert mt["layout_sync_errors"] == 0 and bm.layout_versions() == [2]  # a removed node need not sync
        lens = [CO.shard_len(b.size, 10, 4) for b in blocks]
        assert repair_bytes(MIB) == 346112
        assert mt["layout_bytes_fetched"] == sum(repair_bytes(b.size) for b in blocks) == sum(13 * L // 4 for L in lens)
        assert mt["layout_bytes_read"] == sum(13 * L for L in lens)  # helpers check their whole shard's tag
        assert mt["layout_bytes_written"] == sum(lens)
        assert all(f * 4 == r for f, r in per_step)  # every step: a quarter of what was read
        with G.GarageEc.clay(0, 10, 4) as ec:  # and what garage_ec_read_ranges names for that loss
            runs = [ec.read_ranges(np.arange(14) != i, L) for i, L in zip(lost, lens)]
        assert mt["layout_bytes_fetched"] == sum(r[2] for rs in runs for r in rs)
        shutil.rmtree(os.path.join(d, "node%d" % dead))
        os.makedirs(os.path.join(d, "node%d" % dead))
        assert_placement(bm, d, blocks, hashes)  # byte-identical to a fresh encode
        assert_gets(bm, blocks, hashes)
    with manager(d) as bm:
        assert bm.layout_versions() == [2]
        assert_gets(bm, blocks, hashes)


@pytest.mark.gpu
def test_a_corrupt_helper_makes_way_for_its_next_source(tmp_path):
    """a block written to both versions: a moved index has two holders, and the rebuild of another index takes the
    second when the first one's tag fails -- still 13 helpers, a quarter of each"""
    d = str(tmp_path / "store")
    cap14 = [CAP] * 14 + [0, 0]
    with manager(d, layout=spec(cap14)) as bm:
        assert bm.apply_layout([0] * N, [CAP] * N)[0] == BM.OK
        l1 = PL.Layout.compute([0] * N, cap14, 14)
        seed = 0xCA300
        while True:
            b = O.fill_random(MIB, seed)
            h = BM.blake2sum(b)
            seed += 1
            r1, r2 = list(l1.nodes_of(h)), bm.storage_nodes_of(h)
            moved = [i for i in range(14) if r1[i] != r2[i]]
            kept = [i for i in range(14) if r1[i] == r2[i]]
            if moved and kept:
                break
        assert bm.rpc_put_block(h, b) == BM.OK
        i, j = moved[0], kept[0]
        assert file_of_index(d, r1[i], h, i) and file_of_index(d, r2[i], h, i)
        flip_byte(file_of_index(d, r1[i], h, i))  # the older version's holder is asked first
        os.remove(file_of_index(d, r2[j], h, j))
        m0 = bm.metrics()
        rc, _, _, n = bm.layout_sync_step(r2[j])
        m1 = bm.metrics()
        L = CO.shard_len(MIB, 10, 4)
        assert rc == BM.OK and n == 1 and m1["layout_shards_rebuilt"] - m0["layout_shards_rebuilt"] == 1
        assert m1["corruption_counter"] - m0["corruption_counter"] == 1
        assert m1["layout_bytes_fetched"] - m0["layout_bytes_fetched"] == 13 * L // 4
        assert m1["layout_bytes_read"] - m0["layout_bytes_read"] == 13 * L
        with open(file_of_index(d, r2[j], h, j), "rb") as f:
            assert f.read()[64:] == clay_stripe(b)[j].tobytes()
        assert_gets(bm, [b], [h])


@pytest.mark.gpu
def test_fallbacks_to_whole_shards_and_the_unrecoverable_case(tmp_path):
    d = str(tmp_path / "store")
    dead = 3
    cap15 = [CAP] * 15 + [0]
    L = CO.shard_len(MIB, 10, 4)
    with manager(d, layout=spec(cap15)) as bm:
        blocks, hashes = blocks_on(bm, dead, [MIB] * 3, 0xCA400)
        put_all(bm, blocks, hashes)
        rows1 = [bm.storage_nodes_of(h) for h in hashes]
        assert bm.set_node_up(dead, False) == BM.OK
        assert bm.apply_layout([0] * N, [c if n != dead else 0 for n, c in enumerate(cap15)]) == (BM.OK, 2)
        rows2 = [bm.storage_nodes_of(h) for h in hashes]
        idx = [r.index(dead) for r in rows1]
        target = [r2[x] for r2, x in zip(rows2, idx)]  # the new holders of the dead node's indices
        # helpers to damage: not on a node synced below, so that each block is rebuilt exactly once
        others = [[i for i in range(14) if i != x and r[i] not in target] for r, x in zip(rows1, idx)]
        # block 0: one helper's only copy is corrupt -> quarantined, k whole shards
        flip_byte(path(d, rows1[0][others[0][5]], hashes[0], ".shard"))
        # block 1: a second index has no source -> the whole-shard decode
        os.remove(path(d, rows1[1][others[1][2]], hashes[1], ".shard"))
        # block 2: five indices without a source -> nothing to rebuild from
        for i in others[2][:4]:
            os.remove(path(d, rows1[2][i], hashes[2], ".shard"))
        m0 = bm.metrics()
        for node in sorted(set(target)):
            assert bm.layout_sync_step(node)[0] == BM.OK
        m1 = bm.metrics()
        assert m1["corruption_counter"] - m0["corruption_counter"] == 1
        assert m1["layout_shards_rebuilt"] == 2 and m1["layout_sync_errors"] == 1 and m1["layout_deleted"] == 0
        # k whole shards, twice; the third block's 9 shards were read before it was given up
        assert m1["layout_bytes_fetched"] - m0["layout_bytes_fetched"] == (2 * 10 + 9) * L
        for j in (0, 1):
            with open(path(d, target[j], hashes[j], ".shard"), "rb") as f:
                raw = f.read()
            assert raw[6] == idx[j] and raw[64:] == clay_stripe(blocks[j])[idx[j]].tobytes()
        assert_gets(bm, blocks[:2], hashes[:2])
        assert bm.rpc_get_block(hashes[2])[0] == BM.E_MISSING_BLOCK
        assert sum(os.path.exists(path(d, n, hashes[2], ".shard")) for n in range(N)) == 10  # nothing deleted
        # the rest of the sync: the quarantined and the removed helper are lone losses now and take the repair
        m0 = bm.metrics()
        bm.layout_sync_all()
        m1 = bm.metrics()
        assert m1["layout_shards_rebuilt"] - m0["layout_shards_rebuilt"] == 2
        errors = m1["layout_sync_errors"] - m0["layout_sync_errors"]  # every node still missing a shard of block 2
        assert errors == 5 and m1["layout_deleted"] == 0
        assert m1["layout_bytes_fetched"] - m0["layout_bytes_fetched"] == 2 * 13 * L // 4 + errors * 9 * L
        assert bm.layout_versions() == [1, 2]  # block 2 keeps the sync from finishing
        for h, b in zip(hashes[:2], blocks[:2]):  # both rebuilt stripes are whole and equal to a fresh encode
            ref = clay_stripe(b)
            for i, node in enumerate(bm.storage_nodes_of(h)):
                with open(path(d, node, h, ".shard"), "rb") as f:
                    assert f.read()[64:] == ref[i].tobytes(), (node, i)
        assert_gets(bm, blocks[:2], hashes[:2])


def rotated_store(d, k, m, n, blocks, hashes):
    """a Clay store written under the fixed ring, then an explicit version 2 in which every node moves to the next
    index"""
    with manager(d, n=n, k=k, m=m) as bm:
        put_all(bm, blocks, hashes)
    ring = [[(p % n + i) % n for i in range(k + m)] for p in range(256)]
    write_layout_file(d, n, k + m, [ring, [r[1:] + r[:1] for r in ring]])


@pytest.mark.gpu
def test_clay_layout_sync_is_crash_safe_at_every_step(tmp_path):
    """stop the sync after n file operations (renames, shard writes, deletes), restart, read every block, then sync
    to the end"""
    k, m, n_nodes = 4, 2, 6
    pristine = str(tmp_path / "pristine")
    blocks, hashes = make_blocks([MIB, 5], 0xCA600)
    rotated_store(pristine, k, m, n_nodes, blocks, hashes)
    n, finished = 0, False
    while not finished:
        d = str(tmp_path / ("run%d" % n))
        shutil.copytree(pristine, d)
        with manager(d, n=n_nodes, k=k, m=m) as bm:
            bm.debug_convert_stop_after(n)
            for _ in range(2):
                bm.layout_sync_all()
            mt = bm.metrics()
            finished = mt["layout_shards_copied"] + mt["layout_shards_rebuilt"] == 12 and mt["layout_deleted"] == 12
        with manager(d, n=n_nodes, k=k, m=m) as bm:  # restart after the "crash"
            assert_gets(bm, blocks, hashes)
            assert bm.metrics()["corruption_counter"] == 0
            for _ in range(2):
                bm.layout_sync_all()
            assert bm.layout_versions() == [2] and bm.metrics()["layout_sync_errors"] == 0
            assert_placement(bm, d, blocks, hashes, n=n_nodes, k=k, m=m)
        shutil.rmtree(d)
        n += 1
    assert n > 2 * 6 * 3  # every rename, write and delete of two blocks' moves was a stop point


@pytest.mark.gpu
def test_deep_scrub_during_a_layout_change_finds_stale_parity_and_stale_data(tmp_path):
    """with two active versions the deep scrub checks the blocks whose newest stripe is whole on its own holders: two
    stale parities of one block both go before either is rebuilt, a stale data shard goes through the hunt, and a block
    with a moved index waits for the sync"""
    d = str(tmp_path / "store")
    cap14 = [CAP] * 14 + [0, 0]
    with manager(d, layout=spec(cap14)) as bm:
        assert bm.apply_layout([0] * N, [CAP] * N)[0] == BM.OK
        assert bm.layout_versions() == [1, 2]
        l1 = PL.Layout.compute([0] * N, cap14, 14)
        stay, move, seed = [], [], 0xCA700
        while len(stay) < 2 or len(move) < 1:  # blocks whose row the change leaves alone, and one it does not
            b = O.fill_random([300001, 65536, 4097][seed % 3], seed)
            h = BM.blake2sum(b)
            seed += 1
            same = list(l1.nodes_of(h)) == bm.storage_nodes_of(h)
            (stay if same else move).append((b, h))
        picked = stay[:2] + move[:1]
        blocks, hashes = [b for b, _ in picked], [h for _, h in picked]
        put_all(bm, blocks, hashes)  # to both versions
        rows = [bm.storage_nodes_of(h) for h in hashes]
        for p in (11, 13):
            assert bm.plant_stale_shard(rows[0][p], hashes[0]) == BM.OK
        assert bm.plant_stale_shard(rows[1][4], hashes[1]) == BM.OK
        checked = repaired = 0
        for node in range(N):
            rc, _, finished, c, r = bm.deep_scrub_step(node)
            assert rc == BM.OK and finished
            checked += c
            repaired += r
        mt = bm.metrics()
        assert (checked, repaired) == (2, 3) and mt["deep_scrub_skipped"] == 1
        assert mt["deep_scrub_parity_bad"] == 2 and mt["deep_scrub_content_errors"] == 0
        assert mt["corruption_counter"] == 3
        for node, h in ((rows[0][11], hashes[0]), (rows[0][13], hashes[0]), (rows[1][4], hashes[1])):
            assert bm.node_shard_index(node, h) < 0  # all three quarantined before any rebuild
        for node in (rows[0][11], rows[0][13], rows[1][4]):
            assert bm.resync_all(node)[0] == 0
        bm.layout_sync_all()
        bm.layout_sync_all()
        assert bm.layout_versions() == [2] and bm.metrics()["layout_sync_errors"] == 0
        for dirpath, _, names in os.walk(d):
            for nm in names:
                if nm.endswith(".corrupted"):
                    os.remove(os.path.join(dirpath, nm))
        assert_placement(bm, d, blocks, hashes)
        assert_gets(bm, blocks, hashes)
        for node in range(N):
            assert bm.deep_scrub_step(node)[4] == 0
