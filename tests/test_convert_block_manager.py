"""Changing a store's code in the block manager: a manager restarted with a new code and `previous_codes` (or
`legacy_replicas`) reads the blocks stored before, converts them with garage_ec_transcode in `convert_step` sweeps,
and deletes the old shards only once the new stripe holds its write quorum.  File stores in tmp_path; a "restart" is
a new manager on the same data_dir."""
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

E_INVALID = -1
N = 14  # nodes: enough for every code below
SIZES = [3073, 65536, 1 << 20, (1 << 20) - 1, 5, 777777, 1048575, 4096]  # the ragged sizes of test_block_manager.py


# ---------------------------------------------------------------- helpers
def code_kw(code):
    """("rs", k, m) / ("lrc", k, l, r) / ("pb", k, m) -> BlockManager arguments"""
    if code[0] == "lrc":
        return {"k": code[1], "m": code[2] + code[3], "local_groups": code[2]}
    return {"k": code[1], "m": code[2], "piggyback": code[0] == "pb"}


def as_previous(code):
    kw = code_kw(code)
    return (kw["k"], kw["m"], kw.get("local_groups", 0), int(kw.get("piggyback", False)))


def oracle_code(code):
    return code + (0,) if code[0] in ("rs", "pb") else code  # Vandermonde rows, like the manager's contexts


def manager(code, d, previous=(), rf=0, **kw):
    kw.setdefault("batch_max_blocks", 8)  # small pinned pools: these tests create many managers
    return BM.BlockManager(n_nodes=N, data_dir=d, previous_codes=[as_previous(c) for c in previous], legacy_replicas=rf,
                           **code_kw(code), **kw)


def ring(h, i):
    return (h[0] % N + i) % N


def path(d, node, h, ext):
    return os.path.join(d, "node%d" % node, h[:1].hex(), h[1:2].hex(), h.hex() + ext)


def write_replicas(d, h, b, rf):
    """a replicated Garage store: the block's plain bytes on the first rf nodes of its ring row"""
    for i in range(rf):
        p = path(d, ring(h, i), h, "")
        os.makedirs(os.path.dirname(p), exist_ok=True)
        with open(p, "wb") as f:
            f.write(b.tobytes())


def make_blocks(sizes, seed):
    blocks = [O.fill_random(n, seed + i) for i, n in enumerate(sizes)]
    return blocks, [BM.blake2sum(b) for b in blocks]


def store_old(src, d, blocks, hashes, rf=3):
    if src[0] == "rep":
        for h, b in zip(hashes, blocks):
            write_replicas(d, h, b, rf)
        return
    with manager(src, d) as old:
        for h, b in zip(hashes, blocks):
            assert old.rpc_put_block(h, b) == BM.OK


def legacy_files(d):
    out = []
    for root, _, names in os.walk(d):
        out += [os.path.join(root, n) for n in names if n.endswith(".legacy") or len(n) == 64]
    return out


def assert_gets(bm, blocks, hashes):
    for h, b in zip(hashes, blocks):
        rc, got = bm.rpc_get_block(h)
        assert rc == BM.OK and np.array_equal(got, b)


def assert_new_stripe(bm, d, dst, h, b, nodes_up=None):
    ref = TO.encode_block(oracle_code(dst), b)
    for i, node in enumerate(bm.storage_nodes_of(h)):
        if nodes_up is not None and node not in nodes_up:
            continue
        with open(path(d, node, h, ".shard"), "rb") as f:
            raw = f.read()
        assert raw[:4] == b"GEC1" and raw[64:] == ref[i].tobytes(), (dst, i, b.size)


# ---------------------------------------------------------------- CPU: configuration checks
@pytest.mark.parametrize("kw", [
    {"previous_codes": [(10, 4, 0, 0)]},                       # the configured code itself
    {"previous_codes": [(6, 3, 0, 0), (6, 3, 0, 0)]},          # duplicate
    {"previous_codes": [(4, 2, 0, 0), (6, 3, 0, 0), (8, 3, 0, 0), (6, 2, 0, 0), (5, 2, 0, 0)]},  # more than 4
    {"previous_codes": [(33, 2, 0, 0)]},                       # k > 32
    {"previous_codes": [(6, 0, 0, 0)]},                        # no parity
    {"previous_codes": [(10, 4, 3, 0)]},                       # LRC: k % l != 0
    {"previous_codes": [(10, 4, 4, 0)]},                       # LRC: no global parity
    {"previous_codes": [(10, 5, 0, 1)]},                       # PB: m > 4
    {"previous_codes": [(10, 4, 2, 1)]},                       # PB with LRC groups
    {"previous_codes": [(10, 4, 0, 2)]},                       # piggyback not 0 / 1
    {"previous_codes": [(6, 3, 0, 1)], "shard_sum_kind": BM.SUM_BLAKE2},  # PB needs adler8 segment tags
    {"previous_codes": [(12, 4, 0, 0)]},                       # 16 shards on 14 nodes
    {"legacy_replicas": -1},
    {"legacy_replicas": 15},
])
def test_bad_previous_codes_are_rejected_before_any_cuda_call(kw):
    with pytest.raises(BM.BlockManagerError) as e:
        BM.BlockManager(k=10, m=4, n_nodes=N, **kw)
    assert e.value.code == E_INVALID


def test_null_previous_codes_with_entries_is_rejected():
    L = BM.load_library()
    cfg = BM.Config()
    L.garage_bm_default_config(C.byref(cfg))
    assert not cfg.previous_codes and cfg.n_previous_codes == 0 and cfg.legacy_replicas == 0  # default: none
    cfg.n_previous_codes = 1
    h = C.c_void_p()
    assert L.garage_bm_create(C.byref(h), C.byref(cfg)) == E_INVALID and not h.value


# ---------------------------------------------------------------- GPU: conversions
PAIRS = [(("rs", 6, 3), ("rs", 10, 4)), (("rs", 10, 4), ("lrc", 10, 2, 2)), (("rs", 10, 4), ("pb", 10, 4)),
         (("pb", 10, 4), ("rs", 6, 3)), (("lrc", 10, 2, 2), ("rs", 10, 4)), (("rep",), ("rs", 10, 4)),
         (("rep",), ("pb", 6, 3))]


@pytest.mark.gpu
@pytest.mark.parametrize("src,dst", PAIRS, ids=lambda c: "".join(map(str, c)))
def test_conversion(tmp_path, src, dst):
    d = str(tmp_path / "store")
    blocks, hashes = make_blocks(SIZES, 0x7100)
    store_old(src, d, blocks, hashes)
    kw = {"rf": 3} if src[0] == "rep" else {"previous": [src]}
    with manager(dst, d, **kw) as bm:
        assert_gets(bm, blocks, hashes)  # served by the old code before any conversion
        mt = bm.metrics()
        assert mt["legacy_gets"] == len(blocks) and mt["corruption_counter"] == 0
        for node in range(N):  # scrub checks legacy shards' tags and replicas' content hashes
            rc, _, corrupt = bm.scrub(node)
            assert (rc, corrupt) == (BM.OK, 0)
        assert bm.convert_all() == len(blocks)
        mt = bm.metrics()
        assert mt["convert_blocks"] == len(blocks) and mt["convert_errors"] == 0 and mt["corruption_counter"] == 0
        assert mt["convert_call_us"] > 0 and mt["convert_bytes_written"] > 0
        for h, b in zip(hashes, blocks):
            assert_new_stripe(bm, d, dst, h, b)
        assert legacy_files(d) == []
        assert_gets(bm, blocks, hashes)
        assert bm.metrics()["legacy_gets"] == len(blocks)  # now from the configured stripe
        assert bm.convert_all() == 0  # nothing left
    with manager(dst, d, **kw) as bm:  # restart
        assert_gets(bm, blocks, hashes)
        assert bm.metrics()["legacy_gets"] == 0


@pytest.mark.gpu
def test_degraded_sources_are_rebuilt_and_an_unrecoverable_one_is_kept(tmp_path):
    src, dst = ("rs", 6, 3), ("rs", 10, 4)
    d = str(tmp_path / "store")
    blocks, hashes = make_blocks([1 << 20, 777777, 300001], 0x7200)
    store_old(src, d, blocks, hashes)
    with manager(src, d) as old:
        for i in (0, 2, 7):  # m_s = 3 shards of block 0: data and parity
            assert old.drop_shard(ring(hashes[0], i), hashes[0]) == BM.OK
        for i in (0, 1, 2, 3):  # 4 shards of block 2: unrecoverable
            assert old.drop_shard(ring(hashes[2], i), hashes[2]) == BM.OK
    with manager(dst, d, previous=[src]) as bm:
        assert_gets(bm, blocks[:2], hashes[:2])
        assert bm.rpc_get_block(hashes[2])[0] == BM.E_MISSING_BLOCK
        # two nodes down: block 1 loses two old shards, block 0 (three down already) none more
        row0 = {ring(hashes[0], i) for i in range(9)}
        down = set([n for n in (ring(hashes[1], i) for i in range(9)) if n not in row0][:2])
        assert len(down) == 2
        for n in down:
            bm.set_node_up(n, False)
        assert bm.convert_all() == 2
        mt = bm.metrics()
        assert mt["convert_blocks"] == 2 and mt["convert_errors"] == 1
        up = set(range(N)) - down
        for h, b in zip(hashes[:2], blocks[:2]):
            assert_new_stripe(bm, d, dst, h, b, nodes_up=up)
        for n in down:
            bm.set_node_up(n, True)
        # the nodes that were down delete their own legacy copies once they see the new stripe at quorum
        assert bm.convert_all() == 0
        assert_gets(bm, blocks[:2], hashes[:2])
        assert legacy_files(d) == []
        assert sum(os.path.exists(path(d, n, hashes[2], ".shard")) for n in range(N)) == 5  # block 2 keeps its files
        assert bm.rpc_get_block(hashes[2])[0] == BM.E_MISSING_BLOCK
        assert bm.metrics()["convert_errors"] == 2  # tried again, kept again


@pytest.mark.gpu
def test_no_legacy_copy_is_deleted_without_the_write_quorum(tmp_path):
    src, dst = ("rs", 6, 3), ("rs", 10, 4)
    d = str(tmp_path / "store")
    blocks, hashes = make_blocks([1 << 20], 0x7300)
    h = hashes[0]
    store_old(src, d, blocks, hashes)
    with manager(dst, d, previous=[src]) as bm:
        ro = [ring(h, i) for i in (10, 11, 12, 13)]  # 10 of 14 new shards can be written: k_d + 1 = 11 missed
        for n in ro:
            assert bm.set_node_readonly(n, True) == BM.OK
        assert bm.convert_all() == 0
        mt = bm.metrics()
        assert mt["convert_errors"] == 1 and mt["legacy_deleted"] == 0 and mt["convert_blocks"] == 0
        assert all(os.path.exists(path(d, ring(h, i), h, ".shard")) or os.path.exists(path(d, ring(h, i), h, ".legacy"))
                   for i in range(9))
        assert_gets(bm, blocks, hashes)
        for n in ro:
            assert bm.set_node_readonly(n, False) == BM.OK
        assert bm.convert_all() == 1
        assert_new_stripe(bm, d, dst, h, blocks[0])
        assert legacy_files(d) == [] and bm.metrics()["legacy_deleted"] == 9


@pytest.mark.gpu
def test_conversion_is_crash_safe_at_every_step(tmp_path):
    """stop the sweep after n file operations (renames, shard writes, deletes), restart, read every block, then
    sweep to the end"""
    src, dst = ("rs", 6, 3), ("rs", 10, 4)
    pristine = str(tmp_path / "pristine")
    blocks, hashes = make_blocks([1 << 20, 5], 0x7400)
    store_old(src, pristine, blocks, hashes)
    n, finished = 0, False
    while not finished:
        d = str(tmp_path / ("run%d" % n))
        shutil.copytree(pristine, d)
        with manager(dst, d, previous=[src]) as bm:
            bm.debug_convert_stop_after(n)
            bm.convert_all()
            mt = bm.metrics()
            finished = mt["convert_blocks"] == 2 and mt["legacy_deleted"] == 18
        with manager(dst, d, previous=[src]) as bm:  # restart after the "crash"
            assert_gets(bm, blocks, hashes)
            assert bm.metrics()["corruption_counter"] == 0
            bm.convert_all()
            assert legacy_files(d) == [] and bm.metrics()["convert_errors"] == 0
            for node in range(N):  # a new shard the stop left unwritten is resync's to rebuild
                bm.repair_enqueue_missing(node)
                assert bm.resync_all(node)[0] == 0
            for h, b in zip(hashes, blocks):
                assert_new_stripe(bm, d, dst, h, b)
        with manager(dst, d) as bm:  # and without the previous code at all
            assert_gets(bm, blocks, hashes)
        shutil.rmtree(d)
        n += 1
    assert n > 2 * (14 + 9)  # every stop point of two blocks' writes and deletes was visited


@pytest.mark.gpu
def test_stale_old_shard_is_caught_before_it_reaches_the_new_parity(tmp_path):
    src, dst = ("rs", 6, 3), ("rs", 10, 4)
    d = str(tmp_path / "store")
    blocks, hashes = make_blocks([900001], 0x7500)
    h = hashes[0]
    store_old(src, d, blocks, hashes)
    with manager(src, d) as old:
        assert old.plant_stale_shard(ring(h, 2), h) == BM.OK  # valid tag, other bytes
    with manager(dst, d, previous=[src]) as bm:
        assert bm.convert_all() == 1
        mt = bm.metrics()
        assert mt["corruption_counter"] == 1 and mt["convert_errors"] == 0
        assert os.path.exists(path(d, ring(h, 2), h, ".corrupted"))  # the culprit, quarantined
        assert_new_stripe(bm, d, dst, h, blocks[0])
        assert_gets(bm, blocks, hashes)


@pytest.mark.gpu
def test_a_code_not_listed_is_still_quarantined(tmp_path):
    d = str(tmp_path / "store")
    blocks, hashes = make_blocks([1 << 20], 0x7600)
    store_old(("rs", 6, 3), d, blocks, hashes)
    with manager(("rs", 10, 4), d, previous=[("rs", 4, 2)]) as bm:
        assert bm.rpc_get_block(hashes[0])[0] == BM.E_MISSING_BLOCK
        assert bm.metrics()["corruption_counter"] >= 6


@pytest.mark.gpu
def test_scrub_of_a_half_converted_store_finds_nothing(tmp_path):
    src, dst = ("rs", 6, 3), ("rs", 10, 4)
    d = str(tmp_path / "store")
    blocks, hashes = make_blocks([1 << 20, 65536], 0x7700)
    store_old(src, d, blocks, hashes)
    with manager(dst, d, previous=[src]) as bm:
        bm.debug_convert_stop_after(12)  # some .legacy renames and new shards, nothing deleted
        bm.convert_all()
    assert any(p.endswith(".legacy") for p in legacy_files(d))
    with manager(dst, d, previous=[src]) as bm:
        total = 0
        for node in range(N):
            rc, checked, corrupt = bm.scrub(node)
            assert (rc, corrupt) == (BM.OK, 0)
            total += checked
        assert total >= 2 * 9 and bm.metrics()["corruption_counter"] == 0
        assert_gets(bm, blocks, hashes)


@pytest.mark.gpu
def test_block_with_rc_zero_is_deleted_not_converted(tmp_path):
    src, dst = ("rs", 6, 3), ("rs", 10, 4)
    d = str(tmp_path / "store")
    blocks, hashes = make_blocks([400000, 1 << 20], 0x7800)
    store_old(src, d, blocks, hashes)
    with manager(dst, d, previous=[src]) as bm:
        bm.block_decref(hashes[0])  # rc 1 -> 0 (block_gc_delay_ms = 0 here)
        assert bm.get_block_rc(hashes[0]) == 0
        assert bm.convert_all() == 1  # only the referenced block
        mt = bm.metrics()
        assert mt["convert_blocks"] == 1 and mt["legacy_deleted"] == 18
        assert legacy_files(d) == []
        assert not any(os.path.exists(path(d, n, hashes[0], ".shard")) for n in range(N))
        assert_gets(bm, blocks[1:], hashes[1:])


@pytest.mark.gpu
def test_resync_converts_a_block_whose_configured_stripe_was_never_written(tmp_path):
    src, dst = ("rs", 6, 3), ("rs", 10, 4)
    d = str(tmp_path / "store")
    blocks, hashes = make_blocks([1 << 20], 0x7900)
    h = hashes[0]
    store_old(src, d, blocks, hashes)
    with manager(dst, d, previous=[src]) as bm:
        node = ring(h, 12)  # holds no old shard
        assert bm.repair_enqueue_missing(node) == 1
        assert bm.resync_all(node) == (0, 1)
        assert bm.metrics()["convert_blocks"] == 1
        assert_new_stripe(bm, d, dst, h, blocks[0])
        assert legacy_files(d) == []
        assert_gets(bm, blocks, hashes)
