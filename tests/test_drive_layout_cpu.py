"""CPU tests of the drive layout (DESIGN.md section 5.7): a node's shard files over several data directories.

The model below is written from the rules of DESIGN.md section 5.7 alone; the C++ layout (garage_drive_layout_*, in
libgarage_block.so) must equal it exactly -- primaries and ordered secondaries -- over seeded random sequences of
init, add, remove, capacity change, read-only and drop-secondaries steps.  Also: the properties the rules promise, the
drive partition of a hash, and garage_bm_create refusing every invalid drive configuration before any CUDA call."""
import ctypes as C
import os
import random
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from garage_b200 import block_manager as BM  # noqa: E402
from garage_b200 import placement as P  # noqa: E402

NP = 1024
E_INVALID = -1


# ---------------------------------------------------------------- the model (DESIGN.md section 5.7)
def targets(cap):
    """per directory: floor(cum_after * NP / total) - floor(cum_before * NP / total); read-only (0) -> 0"""
    total, cum, out = sum(cap), 0, []
    for c in cap:
        begin = cum * NP // total
        cum += c
        out.append(cum * NP // total - begin)
    return out


def model_init(cap, non_empty):
    prim = []
    for i, t in enumerate(targets(cap)):
        prim += [i] * t
    sec = [[] for _ in range(NP)]
    for i in range(len(cap)):
        if non_empty[i]:
            for p in range(NP):
                if prim[p] != i:
                    sec[p].append(i)
    return list(cap), prim, sec


def model_update(prev, prev_index, cap, non_empty):
    pcap, pprim, psec = prev
    n = len(cap)
    if n == len(pcap) and all(prev_index[i] == i and cap[i] == pcap[i] for i in range(n)):
        return list(pcap), list(pprim), [list(s) for s in psec]
    new_of = {o: i for i, o in enumerate(prev_index) if o >= 0}
    sec = [[new_of[o] for o in s if o in new_of] for s in psec]
    owned = [[] for _ in range(n)]  # each surviving directory's primaries, in partition order
    for p, o in enumerate(pprim):
        if o in new_of:
            owned[new_of[o]].append(p)
    tgt = targets(cap)
    for i in range(n):
        while len(owned[i]) > tgt[i]:  # give up the highest-numbered, stay a secondary of it
            p = owned[i].pop()
            if i not in sec[p]:
                sec[p].append(i)
    prim = [None] * NP
    for i in range(n):
        for p in owned[i]:
            prim[p] = i
    free = [p for p in range(NP) if prim[p] is None]
    for i in range(n):  # below target, list order, highest-numbered partition first
        for _ in range(tgt[i] - len(owned[i])):
            p = free.pop()
            prim[p] = i
            sec[p] = [d for d in sec[p] if d != i]
    assert not free
    for i in range(n):
        if prev_index[i] < 0 and non_empty[i]:
            for p in range(NP):
                if prim[p] != i and i not in sec[p]:
                    sec[p].append(i)
    return list(cap), prim, sec


def model_drop(m):
    return list(m[0]), list(m[1]), [[] for _ in range(NP)]


def parse_image(b):
    """garage_drive_layout_serialize's image -> (capacities, primaries, secondaries)"""
    assert b[:4] == b"GDL1"
    n = b[4]
    cap = [int.from_bytes(b[5 + 8 * i: 13 + 8 * i], "little") for i in range(n)]
    at, prim, sec = 5 + 8 * n, [], []
    for _ in range(NP):
        prim.append(b[at])
        ns = b[at + 1]
        sec.append(list(b[at + 2: at + 2 + ns]))
        at += 2 + ns
    assert at == len(b)
    return cap, prim, sec


def snapshot(dl):
    return parse_image(dl.serialize())


# ---------------------------------------------------------------- random sequences
def random_steps(rng, n_steps):
    """a list of ("init"|"list"|"drop", dirs) steps; dirs = [(name, capacity, non_empty)], capacity 0 = read-only"""
    names = iter("d%d" % i for i in range(10 ** 6))

    def fresh():
        return [next(names), rng.choice([0, 0, 1, 2, 3, 5, 7, 10 ** 12, 2 ** 63 // 16]) if rng.random() < 0.9 else 0,
                rng.random() < 0.3]

    dirs = [fresh() for _ in range(rng.randint(1, 5))]
    if not any(d[1] for d in dirs):
        dirs[0][1] = rng.randint(1, 9)
    steps = [("init", [tuple(d) for d in dirs])]
    for _ in range(n_steps):
        op = rng.choice(["add", "add", "remove", "capacity", "read_only", "activate", "drop", "same", "shuffle"])
        if op == "add" and len(dirs) < 16:
            dirs.append(fresh())
        elif op == "remove" and len(dirs) > 1:
            dirs.pop(rng.randrange(len(dirs)))
        elif op == "capacity":
            rng.choice(dirs)[1] = rng.randint(1, 1000)
        elif op == "read_only":
            rng.choice(dirs)[1] = 0
        elif op == "activate":
            d = rng.choice(dirs)
            d[1] = d[1] or rng.randint(1, 50)
        elif op == "shuffle":
            rng.shuffle(dirs)
        if not any(d[1] for d in dirs):
            rng.choice(dirs)[1] = rng.randint(1, 9)
        for d in dirs:  # whether a directory holds files changes as the store runs
            d[2] = d[2] or rng.random() < 0.1
        steps.append(("drop" if op == "drop" else "list", [tuple(d) for d in dirs]))
    return steps


def run_sequence(seed, check_properties=True):
    rng = random.Random(seed)
    steps = random_steps(rng, rng.randint(3, 9))
    kind, dirs = steps[0]
    cap = [d[1] for d in dirs]
    dl = P.DriveLayout.init(cap, [d[2] for d in dirs])
    model = model_init(cap, [d[2] for d in dirs])
    assert snapshot(dl) == model, (seed, 0)
    check_counts(model)
    names = [d[0] for d in dirs]
    for si, (kind, dirs) in enumerate(steps[1:], 1):
        if kind == "drop":
            dl2, model2 = dl.drop_secondaries(), model_drop(model)
        else:
            prev_index = [names.index(d[0]) if d[0] in names else -1 for d in dirs]
            cap = [d[1] for d in dirs]
            ne = [d[2] for d in dirs]
            dl2 = dl.update(prev_index, cap, ne)
            model2 = model_update(model, prev_index, cap, ne)
            if check_properties:
                check_update_properties(model, model2, prev_index)
            names = [d[0] for d in dirs]
        got = snapshot(dl2)
        assert got == model2, (seed, si, kind)
        check_counts(model2)
        dl, model = dl2, model2


def check_counts(m):
    cap, prim, sec = m
    assert [prim.count(i) for i in range(len(cap))] == targets(cap)
    for p in range(NP):
        assert cap[prim[p]] > 0, "a read-only directory is never primary"
        assert prim[p] not in sec[p] and len(set(sec[p])) == len(sec[p])


def check_update_properties(old, new, prev_index):
    ocap, oprim, _ = old
    cap, prim, sec = new
    n = len(cap)
    unchanged = n == len(ocap) and all(prev_index[i] == i and cap[i] == ocap[i] for i in range(n))
    if unchanged:
        assert new == old
        return
    assert [prim.count(i) for i in range(n)] == targets(cap)
    new_of = {o: i for i, o in enumerate(prev_index) if o >= 0}
    tgt = targets(cap)
    over = {i for i in range(n) if prev_index[i] >= 0 and oprim.count(prev_index[i]) > tgt[i]}
    for p in range(NP):
        o = oprim[p]
        if o in new_of and prim[p] == new_of[o]:
            continue
        # a partition changes primary only if its directory was over target or removed
        assert o not in new_of or new_of[o] in over, p
        if o in new_of:  # and its old directory, still listed, stays a secondary
            assert new_of[o] in sec[p], p


# ---------------------------------------------------------------- tests
def test_model_equals_library_over_random_sequences():
    for seed in range(600):
        run_sequence(seed)


def test_counts_are_floor_differences_and_read_only_never_primary():
    dl = P.DriveLayout.init([3, 0, 1, 7], [0, 1, 0, 0])
    _, prim, sec = snapshot(dl)
    assert [prim.count(i) for i in range(4)] == targets([3, 0, 1, 7]) == [279, 0, 93, 652]
    assert 1 not in prim
    assert all(s == [1] for s in sec)  # the non-empty read-only directory is a secondary everywhere


def test_initial_runs_are_contiguous_in_list_order():
    _, prim, _ = snapshot(P.DriveLayout.init([1, 2, 1]))
    assert prim == [0] * 256 + [1] * 512 + [2] * 256


def test_unchanged_list_is_the_identity():
    dl = P.DriveLayout.init([1, 2, 1], [1, 0, 0])
    up = dl.update([0, 1, 2], [1, 2, 1], [1, 1, 1])
    assert up.serialize() == dl.serialize()


def test_adding_a_drive_moves_only_the_highest_partitions_and_keeps_old_secondaries():
    dl = P.DriveLayout.init([1, 1, 1, 1])
    up = dl.update([0, 1, 2, 3, -1], [1] * 5, [0, 0, 0, 0, 0])
    _, prim, sec = snapshot(up)
    _, oprim, _ = snapshot(dl)
    moved = [p for p in range(NP) if prim[p] != oprim[p]]
    assert len(moved) == prim.count(4) == targets([1] * 5)[4]
    for p in moved:
        assert prim[p] == 4 and sec[p] == [oprim[p]]
    for d in range(4):  # each drive gave up its highest-numbered partitions
        kept = [p for p in range(NP) if oprim[p] == d and prim[p] == d]
        lost = [p for p in range(NP) if oprim[p] == d and prim[p] != d]
        assert not lost or max(kept) < min(lost)


def test_drop_secondaries_keeps_primaries():
    dl = P.DriveLayout.init([1, 1], [1, 1])
    _, prim, sec = snapshot(dl)
    assert any(sec)
    _, prim2, sec2 = snapshot(dl.drop_secondaries())
    assert prim2 == prim and not any(sec2)


def test_serialize_round_trip_and_damaged_images():
    dl = P.DriveLayout.init([5, 0, 3], [1, 1, 0]).update([0, 1, 2, -1], [5, 0, 3, 4], [0, 0, 0, 1])
    img = dl.serialize()
    assert P.DriveLayout.deserialize(img).serialize() == img
    with pytest.raises(P.PlacementError):
        P.DriveLayout.deserialize(img[:-1])
    bad = bytearray(img)
    bad[5 + 8 * 4] = 1  # partition 0's primary -> the read-only directory
    with pytest.raises(P.PlacementError):
        P.DriveLayout.deserialize(bytes(bad))
    with pytest.raises(P.PlacementError):
        P.DriveLayout.deserialize(b"GDL2" + img[4:])


def test_invalid_layout_inputs():
    for cap in ([], [0], [0, 0], [1] * 17):
        with pytest.raises(P.PlacementError) as e:
            P.DriveLayout.init(cap)
        assert e.value.code == E_INVALID
    dl = P.DriveLayout.init([1, 1])
    for prev_index, cap in (([0, 0], [1, 1]), ([2], [1]), ([-2], [1]), ([0, 1], [0, 0])):
        with pytest.raises(P.PlacementError) as e:
            dl.update(prev_index, cap)
        assert e.value.code == E_INVALID


def test_drive_partition_of_worked_examples():
    def h(b2, b3, fill=0):
        return bytes([fill, fill, b2, b3]) + bytes([fill]) * 28

    assert P.drive_partition_of(h(0x12, 0x34)) == 0x1234 % 1024 == 564
    assert P.drive_partition_of(h(0xFF, 0xFF, 0xAB)) == 1023
    assert P.drive_partition_of(h(0x04, 0x00, 0xFF)) == 0
    assert P.drive_partition_of(h(0x00, 0x07)) == 7
    assert P.drive_partition_of(h(0x83, 0xFF)) == 1023


def test_drive_symbols_declared_bound_and_exported():
    import re
    import subprocess

    from garage_b200 import _build

    src = open(os.path.join(ROOT, "include", "garage_placement.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    assert sorted(set(re.findall(r"\b(garage_drive_[a-z0-9_]+)\s*\(", src))) == sorted(P.DRIVE_SYMBOLS)
    P._dlib()
    out = subprocess.run(["nm", "-D", "--defined-only", _build.BM_SO], capture_output=True, text=True).stdout
    assert set(P.DRIVE_SYMBOLS) <= set(re.findall(r"\bT (garage_[a-z0-9_]+)", out))


def _create(tmp_path, dirs, data_dir=True, n=None, null_list=False):
    """garage_bm_create_with_drives of the default config and `dirs` -> rc (a created manager is destroyed)"""
    L = BM.load_library()
    cfg = BM.Config()
    L.garage_bm_default_config(C.byref(cfg))
    keep = str(tmp_path).encode()
    cfg.data_dir = keep if data_dir else None
    arr = (BM.DataDir * max(1, len(dirs)))(*[BM.DataDir(d[0].encode(), d[1], d[2] if len(d) > 2 else 0) for d in dirs])
    h = C.c_void_p()
    rc = L.garage_bm_create_with_drives(C.byref(h), C.byref(cfg), None if null_list else arr, len(dirs) if n is None else n)
    if rc == 0:
        L.garage_bm_destroy(h)
    return rc


@pytest.mark.parametrize("case", [
    "memory_store", "null_list", "negative_count", "too_many", "duplicate", "duplicate_normalised", "zero_capacity",
    "no_active", "absolute", "escapes_node_dir", "empty_path", "bad_read_only"])
def test_create_rejects_invalid_drive_configs_before_cuda(tmp_path, case):
    good = [("d1", 1), ("d2", 1)]
    dirs = {
        "memory_store": good, "null_list": good, "negative_count": good, "too_many": [("d%d" % i, 1) for i in range(17)],
        "duplicate": [("d1", 1), ("d1", 2)], "duplicate_normalised": [(".", 1), ("d1/..", 1)],
        "zero_capacity": [("d1", 0), ("d2", 1)], "no_active": [("d1", 0, 1), ("d2", 5, 1)],
        "absolute": [("/tmp/x", 1)], "escapes_node_dir": [("../node1", 1), ("d2", 1)], "empty_path": [("", 1)],
        "bad_read_only": [("d1", 1, 2)],
    }[case]
    kw = {"memory_store": {"data_dir": False}, "null_list": {"null_list": True}, "negative_count": {"n": -1}}.get(case, {})
    assert _create(tmp_path, dirs, **kw) == E_INVALID
    assert not list(tmp_path.iterdir()), "nothing may be created before the check"


def test_valid_drive_config_passes_the_checks(tmp_path):
    import torch

    if torch.cuda.is_available():
        pytest.skip("on a GPU machine create succeeds; the block-manager tests cover that")
    rc = _create(tmp_path, [(".", 1), ("d1", 2), ("ro", 0, True)])
    assert rc not in (0, E_INVALID)  # it got as far as the GPU, which this machine lacks


def test_set_data_dirs_rejects_invalid_lists_without_a_manager():
    L = BM.load_library()
    arr, n = BM._data_dirs([("d1", 1)])
    assert L.garage_bm_set_data_dirs(None, 0, C.cast(arr, C.POINTER(BM.DataDir)), n) == E_INVALID
    assert L.garage_bm_rebalance_step(None, 0, None, 0, None, None, None) == E_INVALID
