"""garage_ec_segment_read_ranges (DESIGN.md section 2.10) on H100 contexts: the runs equal a model built from
tests/segment_oracle.py (unit_runs, unit_present) and each code's read set (RS: the first k present, LRC: lrc_oracle,
PB: pb_oracle's half-row plan), and a stripe holding only those runs -- every other byte garbage -- rebuilds to the
bytes garage_ec_reconstruct_segments gives on the whole stripe.  RS at one k per kernel class, LRC(10,2,2), PB(10,4);
ragged shard lengths from 0 to a 1 MiB block's; the refusals."""
import os
import sys
import zlib

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import lrc_oracle as LO  # noqa: E402
import pb_oracle as PO  # noqa: E402
import segment_oracle as SO  # noqa: E402
from test_segment_gpu import SENTINEL, context, damage, make_stripes, oracle_code, random_patterns  # noqa: E402

import garage_b200 as G  # noqa: E402

pytestmark = pytest.mark.gpu

GARBAGE = 0xA7


@pytest.fixture(scope="module")
def torch():
    import torch as t

    assert t.cuda.is_available()
    return t


def merge(runs):
    out = []
    for s, o, n in sorted(runs):
        if out and out[-1][0] == s and o <= out[-1][1] + out[-1][2]:
            ps, po, pn = out[-1]
            out[-1] = (ps, po, max(po + pn, o + n) - po)
        else:
            out.append((s, o, n))
    return out


def model_runs(code, sp, want, L):
    """the runs by the oracle statement, or None if a unit is unrecoverable"""
    tot = code.k + code.m
    runs = []
    for g in range(code.units):
        pres = [SO.unit_present(code, int(sp[i]), L, g) for i in range(tot)]
        if all(pres):
            continue
        ur = SO.unit_runs(code, L, g)
        if code.kind == "pb":
            ok, rows = PO.read_plan(code.k, code.m, code.P, pres, want)
            pieces = [(q >> 1, ur[q & 1]) for q in rows]
        else:
            ok, surv = LO.read_set(code.k, code.l, code.P, pres, want)
            pieces = [(i, ur[0]) for i in surv]
        if not ok:
            return None
        if any(not pres[i] and (want is None or want[i]) for i in range(tot)):
            runs += [(i, o, n) for i, (o, n) in pieces if n]
    return merge(runs)


def written_mask(code, sp, want, L, stride):
    """(k+m, stride) bool: the bytes reconstruct_segments writes -- the wanted absent units, and the zero tail of a
    shard whose last unit is rebuilt (RS / LRC)"""
    tot = code.k + code.m
    mask = np.zeros((tot, stride), dtype=bool)
    for g in range(code.units):
        for i in range(tot):
            if SO.unit_present(code, int(sp[i]), L, g) or (want is not None and not want[i]):
                continue
            runs = SO.unit_runs(code, L, g)
            for o, n in runs:
                mask[i, o:o + n] = True
            if code.kind != "pb" and runs[0][0] + runs[0][1] == L:
                mask[i, L:min(stride, -(-L // 16) * 16)] = True
    return mask


def check_batch(torch, ec, code, lens, stride, rng, seed):
    n, tot = len(lens), code.k + code.m
    sh = make_stripes(torch, ec, lens, stride, seed)
    sp, want = random_patterns(code, lens, rng)
    wants = [want[s] if s % 2 else None for s in range(n)]
    for s, L in enumerate(lens):
        damage(code, sh[s], sp[s], L)
    sparse = np.full_like(sh, GARBAGE)
    plans = []
    for s, L in enumerate(lens):
        runs = ec.segment_read_ranges(sp[s], L, want=wants[s])
        assert runs == model_runs(code, sp[s], wants[s], L), (s, L, sp[s], wants[s])
        plans.append(runs)
        for i, o, ln in runs or []:
            sparse[s, i, o:o + ln] = sh[s, i, o:o + ln]
    lens32 = np.asarray(lens, dtype=np.uint32)
    for s in range(n):  # want differs per stripe: one call each, the HOST form on both copies
        full, part = sh[s].copy(), sparse[s].copy()
        st_full, st_part = np.zeros(1, np.int32), np.zeros(1, np.int32)
        w = None if wants[s] is None else wants[s][None]
        ec.reconstruct_segments(full.reshape(-1), sp[s][None], stride, 1, want=w, status=st_full, shard_len=lens32[s:s + 1])
        ec.reconstruct_segments(part.reshape(-1), sp[s][None], stride, 1, want=w, status=st_part, shard_len=lens32[s:s + 1])
        assert st_full[0] == st_part[0] == (G.E_UNRECOVERABLE if plans[s] is None else 0)
        if plans[s] is None:
            assert np.array_equal(part, sparse[s])
            continue
        mask = written_mask(code, sp[s], wants[s], lens[s], stride)
        assert np.array_equal(part[mask], full[mask]), (s, lens[s], sp[s])
        assert np.array_equal(part[~mask], sparse[s][~mask])
    return sum(p is None for p in plans)


RS = ["rs_3_2", "rs_10_4", "rs_20_4"]  # LDG (k <= 4, 7), TMA (5..16), TMA split staging (k > 16)
NAMES = RS + ["lrc_10_2_2", "pb_10_4"]


@pytest.mark.parametrize("name", NAMES)
def test_runs_match_the_model_and_rebuild_the_same_bytes(torch, name):
    with context(name) as ec:
        code = oracle_code(ec, name)
        rng = np.random.default_rng(zlib.crc32(name.encode()))
        base = [128, 256, 384, 1152, 4096] if code.kind == "pb" else [1, 15, 16, 17, 127, 128, 129, 1000, 4096]
        lens = [base[s % len(base)] for s in range(120)]
        unrec = check_batch(torch, ec, code, lens, 4096 + 128, rng, 41)
        assert 0 < unrec < len(lens) // 2
        L = ec.code_shard_len(1 << 20)
        check_batch(torch, ec, code, [L] * 6, -(-L // 128) * 128, rng, 43)


@pytest.mark.parametrize("name", NAMES)
def test_zero_length_needs_no_runs(torch, name):
    with context(name) as ec:
        code = oracle_code(ec, name)
        rng = np.random.default_rng(3)
        for _ in range(20):
            sp = rng.integers(0, 256, code.k + code.m).astype(np.uint8)
            assert ec.segment_read_ranges(sp, 0) == [] == model_runs(code, sp, None, 0)


def test_one_bad_segment_of_a_1mib_block():
    """the bytes of the traffic table: RS(10,4) reads segment g of 10 shards, LRC(10,2,2) of a data shard's local
    group (5 shards), PB(10,4) the unit's half-plan; a whole-shard loss reads what garage_ec_read_ranges names"""
    with G.GarageEc(0, 10, 4) as ec:
        L = ec.code_shard_len(1 << 20)
        assert L == 104858
        for g in range(8):
            sp = np.full(14, 0xFF, np.uint8)
            sp[3] &= ~np.uint8(1 << g)
            runs = ec.segment_read_ranges(sp, L, want=np.eye(14, dtype=np.uint8)[3])
            assert sum(n for _, _, n in runs) == (130180 if g == 7 else 131200)
            assert [s for s, _, _ in runs] == [0, 1, 2, 4, 5, 6, 7, 8, 9, 10]
    with G.GarageEc.lrc(0, 10, 2, 2) as ec:
        sp = np.full(14, 0xFF, np.uint8)
        sp[2] = 0xFF & ~(1 << 4)
        runs = ec.segment_read_ranges(sp, ec.code_shard_len(1 << 20), want=np.eye(14, dtype=np.uint8)[2])
        assert sum(n for _, _, n in runs) == 65600 and [s for s, _, _ in runs] == [0, 1, 3, 4, 10]
    with G.GarageEc.piggyback(0, 10, 4) as ec:
        L = ec.code_shard_len(1 << 20)
        sp = np.full(14, 0xFF, np.uint8)
        sp[3] = 0xFF & ~(1 << 1)
        runs = ec.segment_read_ranges(sp, L, want=np.eye(14, dtype=np.uint8)[3])
        plan = ec.read_plan(np.array([0 if i == 3 else 1 for i in range(14)], np.uint8), np.eye(14, dtype=np.uint8)[3])
        halves = sum(bin(int(b)).count("1") for b in plan)
        assert sum(n for _, _, n in runs) == halves * L // 8


def test_refusals():
    with G.GarageEc.clay(0, 10, 4) as ec:
        with pytest.raises(G.EcError) as ei:
            ec.segment_read_ranges(np.full(14, 0xFE, np.uint8), 4096)
        assert ei.value.code == G.E_INVALID
    with G.GarageEc.piggyback(0, 10, 4) as ec:
        with pytest.raises(G.EcError) as ei:
            ec.segment_read_ranges(np.full(14, 0xFE, np.uint8), 1000)
        assert ei.value.code == G.E_INVALID
        assert ec.segment_read_ranges(np.full(14, 0xFF, np.uint8), 1024) == []
    with G.GarageEc(0, 10, 4) as ec:
        sp = np.full(14, 0xFF, np.uint8)
        sp[0] = 0xFF & ~(1 << 2)
        assert len(ec.segment_read_ranges(sp, 4096)) == 10
        with pytest.raises(G.EcError) as ei:
            ec.segment_read_ranges(sp, 4096, cap=9)
        assert ei.value.code == G.E_INVALID
        sp[:5] = 0xFF & ~(1 << 2)  # m + 1 shards without segment 2
        assert ec.segment_read_ranges(sp, 4096) is None
        sp[:5] = 0xFF
        sp[:5] &= ~np.array([1 << g for g in range(5)], np.uint8)  # five shards, five different segments
        assert len(ec.segment_read_ranges(sp, 4096)) == 14
