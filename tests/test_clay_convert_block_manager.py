"""Clay as a previous code (DESIGN.md section 5.1): a store written as Clay(10,4) and reopened as RS(10,4), PB(10,4) or
Clay(6,3) with Clay(10,4) in `previous_codes` serves GETs from the Clay stripes (one and four shards dropped too),
converts every block with garage_ec_transcode reading k whole Clay shards per intact block, deletes the Clay shards only
once k+1 new shards are durable, and survives a stop at every file operation.  File stores in tmp_path; a "restart" is
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
import transcode_oracle as TO  # noqa: E402

from garage_b200 import block_manager as BM  # noqa: E402

E_INVALID = -1
N = 14
MIB = 1 << 20
SIZES = [3073, 65536, MIB, MIB - 1, 5, 777777, 4096]
CLAY = ("clay", 10, 4)
DSTS = [("rs", 10, 4), ("pb", 10, 4), ("clay", 6, 3)]


def code_kw(code):
    return {"k": code[1], "m": code[2], "piggyback": code[0] == "pb", "clay": code[0] == "clay"}


def as_previous(code):
    return (code[1], code[2], 0, int(code[0] == "pb"), int(code[0] == "clay"))


def manager(code, d, previous=(), **kw):
    kw.setdefault("batch_max_blocks", 8)  # small pinned pools: these tests create many managers
    return BM.BlockManager(n_nodes=N, data_dir=d, previous_codes=[as_previous(c) for c in previous], **code_kw(code), **kw)


def ring(h, i):
    return (h[0] % N + i) % N


def path(d, node, h, ext):
    return os.path.join(d, "node%d" % node, h[:1].hex(), h[1:2].hex(), h.hex() + ext)


def make_blocks(sizes, seed):
    blocks = [O.fill_random(n, seed + i) for i, n in enumerate(sizes)]
    return blocks, [BM.blake2sum(b) for b in blocks]


def store_clay(d, blocks, hashes, drop=()):
    """the blocks under Clay(10,4); drop: (block, shard index) pairs removed afterwards"""
    with manager(CLAY, d) as old:
        for h, b in zip(hashes, blocks):
            assert old.rpc_put_block(h, b) == BM.OK
        for j, i in drop:
            assert old.drop_shard(ring(hashes[j], i), hashes[j]) == BM.OK


def legacy_files(d):
    out = []
    for root, _, names in os.walk(d):
        out += [os.path.join(root, n) for n in names if n.endswith(".legacy")]
    return out


def clay_files(d):
    """shard files (.shard or .legacy) whose header names Clay(10,4)"""
    out = []
    for root, _, names in os.walk(d):
        for n in names:
            if n.endswith((".shard", ".legacy")):
                with open(os.path.join(root, n), "rb") as f:
                    hd = f.read(64)
                if hd[4] == 10 and hd[5] == 4 and hd[53] == 2:
                    out.append(os.path.join(root, n))
    return out


def assert_gets(bm, blocks, hashes):
    for h, b in zip(hashes, blocks):
        rc, got = bm.rpc_get_block(h)
        assert rc == BM.OK and np.array_equal(got, b)


def encode(code, b):
    if code[0] != "clay":
        return TO.encode_block(code + (0,), b)
    k, m = code[1], code[2]
    L = CO.shard_len(b.size, k, m)
    flat = np.zeros(k * L, dtype=np.uint8)
    flat[:b.size] = b
    data = flat.reshape(k, L)
    return np.concatenate([data, CO.encode(k, m, CO.build(k, m), data)])


def assert_new_stripe(bm, d, dst, h, b):
    ref = encode(dst, b)
    for i, node in enumerate(bm.storage_nodes_of(h)):
        with open(path(d, node, h, ".shard"), "rb") as f:
            raw = f.read()
        assert raw[:4] == b"GEC1" and raw[4] == dst[1] and raw[53] == {"rs": 0, "pb": 1, "clay": 2}[dst[0]]
        assert raw[64:] == ref[i].tobytes(), (dst, i, b.size)


# ---------------------------------------------------------------- CPU: configuration checks
@pytest.mark.parametrize("kw", [
    {"previous_codes": [(10, 4, 0, 0, 2)]},                    # clay not 0 / 1
    {"previous_codes": [(10, 5, 0, 0, 1)], "n_nodes": 15},     # Clay: m > 4
    {"previous_codes": [(1, 2, 0, 0, 1)]},                     # Clay: k < 2
    {"previous_codes": [(14, 4, 0, 0, 1)], "n_nodes": 18},     # Clay: alpha = 1024
    {"previous_codes": [(10, 4, 2, 0, 1)]},                    # Clay with LRC groups
    {"previous_codes": [(10, 4, 0, 1, 1)]},                    # Clay with PB
    {"previous_codes": [(6, 3, 0, 0, 1), (6, 3, 0, 0, 1)]},    # duplicate
    {"previous_codes": [(12, 4, 0, 0, 1)]},                    # 16 shards on 14 nodes
    {"clay": True, "previous_codes": [(10, 4, 0, 0, 1)]},      # the configured code itself
])
def test_bad_clay_previous_codes_are_rejected_before_any_cuda_call(kw):
    args = dict(k=10, m=4, n_nodes=N)
    args.update(kw)
    with pytest.raises(BM.BlockManagerError) as e:
        BM.BlockManager(**args)
    assert e.value.code == E_INVALID


def _create_rc(**fields):
    """garage_bm_create's code for the default configuration with `fields` set; with no GPU an accepted configuration
    gets as far as the first CUDA call and fails there, with another code than GARAGE_EC_E_INVALID"""
    L = BM.load_library()
    cfg = BM.Config()
    L.garage_bm_default_config(C.byref(cfg))
    prev = fields.pop("previous", [])
    arr = (BM.Code * max(1, len(prev)))(*[BM.Code(*c) for c in prev])
    if prev:
        cfg.previous_codes, cfg.n_previous_codes = C.cast(arr, C.POINTER(BM.Code)), len(prev)
    for name, v in fields.items():
        setattr(cfg, name, v)
    h = C.c_void_p()
    rc = L.garage_bm_create(C.byref(h), C.byref(cfg))
    if rc == BM.OK:
        L.garage_bm_destroy(h)
    return rc


@pytest.mark.parametrize("fields", [
    {"previous": [(10, 4, 0, 0, 1)]},                          # RS(10,4) after Clay(10,4)
    {"piggyback": 1, "previous": [(10, 4, 0, 0, 1)]},          # PB(10,4) after Clay(10,4)
    {"clay": 1, "previous": [(6, 3, 0, 0, 1)]},                # Clay(10,4) after Clay(6,3)
    {"clay": 1, "previous": [(10, 4, 0, 0, 0)]},               # Clay(10,4) after RS(10,4): equal but for `clay`
    {"previous": [(6, 3, 0, 0, 1), (6, 3, 0, 0, 0)]},          # Clay(6,3) and RS(6,3) are two codes
    {"previous": [(6, 3, 0, 0)]},                              # an entry built without the new member: clay = 0
])
def test_clay_previous_codes_pass_the_argument_checks(fields):
    assert _create_rc(**fields) != E_INVALID


def test_an_older_callers_code_and_metrics_keep_their_meaning():
    c = BM.Code(6, 3, 0, 0)  # the four members an older caller set
    assert c.clay == 0
    names = [n for n, _ in BM.Metrics._fields_]
    assert names[-1] == "layout_bytes_fetched" and names[-2] == "deep_check_call_us"  # added at the end
    assert [n for n, _ in BM.Code._fields_][-1] == "clay" and [n for n, _ in BM.Config._fields_][-1] == "clay_layout"


# ---------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("dst", DSTS, ids=lambda c: "".join(map(str, c)))
def test_conversion_from_clay(tmp_path, dst):
    d = str(tmp_path / "store")
    blocks, hashes = make_blocks(SIZES, 0xCB100)
    store_clay(d, blocks, hashes)
    with manager(dst, d, previous=[CLAY]) as bm:
        assert_gets(bm, blocks, hashes)  # served by the Clay stripes before any conversion
        mt = bm.metrics()
        assert mt["legacy_gets"] == len(blocks) and mt["corruption_counter"] == 0
        for node in range(N):  # scrub checks the Clay shards' tags
            rc, checked, corrupt = bm.scrub(node)
            assert (rc, checked, corrupt) == (BM.OK, len(blocks), 0)
        assert bm.convert_all() == len(blocks)
        mt = bm.metrics()
        assert mt["convert_blocks"] == len(blocks) and mt["convert_errors"] == 0 and mt["corruption_counter"] == 0
        assert mt["convert_bytes_read"] == sum(10 * CO.shard_len(b.size, 10, 4) for b in blocks)  # k whole shards
        assert mt["legacy_deleted"] == 14 * len(blocks)
        for h, b in zip(hashes, blocks):
            assert_new_stripe(bm, d, dst, h, b)
        assert legacy_files(d) == [] and clay_files(d) == []
        assert_gets(bm, blocks, hashes)
        assert bm.metrics()["legacy_gets"] == len(blocks)  # now from the configured stripe
        assert bm.convert_all() == 0
    with manager(dst, d) as bm:  # restart, without the previous code at all
        assert_gets(bm, blocks, hashes)
        assert bm.metrics()["legacy_gets"] == 0


@pytest.mark.gpu
@pytest.mark.parametrize("dst", DSTS, ids=lambda c: "".join(map(str, c)))
def test_degraded_clay_stripes_are_read_and_converted(tmp_path, dst):
    d = str(tmp_path / "store")
    blocks, hashes = make_blocks([MIB, 777777, 300001, 65536], 0xCB200)
    drop = [(0, 3)] + [(1, i) for i in (0, 5, 11, 13)] + [(2, 12)] + [(3, i) for i in (0, 1, 2, 3, 10)]
    store_clay(d, blocks, hashes, drop)
    with manager(dst, d, previous=[CLAY]) as bm:
        assert_gets(bm, blocks[:3], hashes[:3])  # one data shard, four shards, one parity shard dropped
        assert bm.rpc_get_block(hashes[3])[0] == BM.E_MISSING_BLOCK  # five
        assert bm.metrics()["legacy_gets"] == 3
        m0 = bm.metrics()
        assert bm.convert_all() == 3
        mt = bm.metrics()
        assert mt["convert_blocks"] == 3 and mt["convert_errors"] == 1 and mt["corruption_counter"] == 0
        Ls = [CO.shard_len(b.size, 10, 4) for b in blocks]
        # what garage_ec_read_set names, whole: the 13 others for a lone lost data shard, else the first k present;
        # the unrecoverable block's 9 shards are read before it is given up
        assert mt["convert_bytes_read"] - m0["convert_bytes_read"] == 13 * Ls[0] + 10 * Ls[1] + 10 * Ls[2] + 9 * Ls[3]
        for h, b in zip(hashes[:3], blocks[:3]):
            assert_new_stripe(bm, d, dst, h, b)
        assert_gets(bm, blocks[:3], hashes[:3])
        assert bm.metrics()["legacy_gets"] == 3
        assert bm.rpc_get_block(hashes[3])[0] == BM.E_MISSING_BLOCK
        assert len([p for p in clay_files(d) if hashes[3].hex() in p]) == 9  # the unrecoverable block keeps its files


@pytest.mark.gpu
def test_no_clay_shard_is_deleted_without_the_write_quorum(tmp_path):
    dst = ("rs", 10, 4)
    d = str(tmp_path / "store")
    blocks, hashes = make_blocks([MIB], 0xCB300)
    h = hashes[0]
    store_clay(d, blocks, hashes)
    with manager(dst, d, previous=[CLAY]) as bm:
        ro = [ring(h, i) for i in (10, 11, 12, 13)]  # 10 of 14 new shards can be written: k + 1 = 11 missed
        for n in ro:
            assert bm.set_node_readonly(n, True) == BM.OK
        assert bm.convert_all() == 0
        mt = bm.metrics()
        assert mt["convert_errors"] == 1 and mt["legacy_deleted"] == 0 and mt["convert_blocks"] == 0
        for n in ro:
            assert bm.set_node_readonly(n, False) == BM.OK
        assert len(clay_files(d)) == 14  # every Clay shard is still there, moved aside or not
        assert_gets(bm, blocks, hashes)
        assert bm.convert_all() == 1
        assert_new_stripe(bm, d, dst, h, blocks[0])
        assert legacy_files(d) == [] and clay_files(d) == [] and bm.metrics()["legacy_deleted"] == 14


@pytest.mark.gpu
def test_conversion_from_clay_is_crash_safe_at_every_step(tmp_path):
    """stop the sweep after n file operations (renames, shard writes, deletes), restart, read every block, then
    sweep to the end"""
    dst = ("rs", 10, 4)
    pristine = str(tmp_path / "pristine")
    blocks, hashes = make_blocks([MIB, 5], 0xCB400)
    store_clay(pristine, blocks, hashes)
    n, finished = 0, False
    while not finished:
        d = str(tmp_path / ("run%d" % n))
        shutil.copytree(pristine, d)
        with manager(dst, d, previous=[CLAY]) as bm:
            bm.debug_convert_stop_after(n)
            bm.convert_all()
            mt = bm.metrics()
            finished = mt["convert_blocks"] == 2 and mt["legacy_deleted"] == 28
        with manager(dst, d, previous=[CLAY]) as bm:  # restart after the "crash"
            assert_gets(bm, blocks, hashes)
            assert bm.metrics()["corruption_counter"] == 0
            bm.convert_all()
            assert legacy_files(d) == [] and clay_files(d) == [] and bm.metrics()["convert_errors"] == 0
            for node in range(N):  # a new shard the stop left unwritten is resync's to rebuild
                bm.repair_enqueue_missing(node)
                assert bm.resync_all(node)[0] == 0
            for h, b in zip(hashes, blocks):
                assert_new_stripe(bm, d, dst, h, b)
        shutil.rmtree(d)
        n += 1
    assert n > 2 * 14  # every stop point of two blocks' moves aside, writes and deletes was visited


@pytest.mark.gpu
def test_a_stale_clay_shard_is_caught_before_it_reaches_the_new_parity(tmp_path):
    dst = ("rs", 10, 4)
    d = str(tmp_path / "store")
    blocks, hashes = make_blocks([900001], 0xCB500)
    h = hashes[0]
    store_clay(d, blocks, hashes)
    with manager(CLAY, d) as old:
        assert old.plant_stale_shard(ring(h, 2), h) == BM.OK  # valid tag, other bytes
    with manager(dst, d, previous=[CLAY]) as bm:
        assert bm.convert_all() == 1
        mt = bm.metrics()
        assert mt["corruption_counter"] == 1 and mt["convert_errors"] == 0
        assert os.path.exists(path(d, ring(h, 2), h, ".corrupted"))  # the culprit, quarantined
        assert_new_stripe(bm, d, dst, h, blocks[0])
        assert_gets(bm, blocks, hashes)
