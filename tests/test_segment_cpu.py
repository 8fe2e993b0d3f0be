"""Reconstruct by segment (DESIGN.md section 2.10) without a GPU: the oracle's unit geometry against the library's
garage_ec_tag_span, its 0x00 / 0xFF equivalence with the whole-shard oracles, recovery of patterns with more than m
damaged shards, refusal of a unit with m+1 bad shards, and the new exports."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import garage_b200 as G  # noqa: E402
import lrc_oracle as LO  # noqa: E402
import oracle_lib as O  # noqa: E402
import pb_oracle as PO  # noqa: E402
import segment_oracle as SO  # noqa: E402

CODES = {
    "rs_4_2": lambda: SO.Code("rs", 4, 2, O.build_matrix(4, 2, 0)),
    "rs_10_4_cauchy": lambda: SO.Code("rs", 10, 4, O.build_matrix(10, 4, 1)),
    "lrc_10_2_2": lambda: SO.Code("lrc", 10, 4, LO.build_lrc(10, 2, 2), l=2),
    "pb_10_4": lambda: SO.Code("pb", 10, 4, PO.build(10, 4)),
}


def encode(code, data):
    """data (k, L) -> parity (m, L)"""
    if code.kind == "rs":
        k, L = data.shape
        return O.encode(k, code.m, code.P, np.ascontiguousarray(data).reshape(-1), L, 1).reshape(code.m, L)
    return (LO.encode if code.kind == "lrc" else PO.encode)(code.P, data)


def stripe(code, L, stride, seed):
    rng = np.random.default_rng(seed)
    data = rng.integers(0, 256, (code.k, L), dtype=np.uint8)
    sh = np.zeros((code.k + code.m, stride), dtype=np.uint8)
    sh[: code.k, :L] = data
    if L:
        sh[code.k:, :L] = encode(code, data)
    return sh


def span(L, off, n):
    a, b = C.c_uint32(), C.c_uint32()
    assert G.load_library().garage_ec_tag_span(G.SUM_ADLER8, L, off, n, C.byref(a), C.byref(b)) == 0
    return a.value, b.value


def test_segments_are_the_tag_spans():
    for L in list(range(0, 301)) + [104858, 104960, 1 << 20]:
        for o, n in SO.segments(L):
            if n:
                assert span(L, o, 1) == (o, n) and span(L, o, n) == (o, n), (L, o, n)
        assert sum(n for _, n in SO.segments(L)) == L


@pytest.mark.parametrize("name", sorted(CODES))
def test_units_of_1mib_blocks_are_tag_spans(name):
    code = CODES[name]()
    L = PO.shard_len(1 << 20, code.k) if code.kind == "pb" else -(-(1 << 20) // code.k)
    for g in range(code.units):
        runs = SO.unit_runs(code, L, g)
        segs = [g, g + 4] if code.kind == "pb" else [g]
        assert runs == [SO.segments(L)[x] for x in segs]
        for o, n in runs:
            assert span(L, o, n) == (o, n)


def whole_shard(code, sh, present, L, want=None):
    """the code's whole-shard oracle on [0, L) of every shard"""
    body = np.ascontiguousarray(sh[:, :L])
    if code.kind == "rs":
        flat = body.reshape(-1)
        _, st = O.reconstruct(code.k, code.m, code.P, flat, np.array(present, dtype=np.uint8), L, 1)
        ok = int(st[0]) == 0
        body = flat.reshape(body.shape)
    elif code.kind == "lrc":
        ok = LO.decode(code.k, code.l, code.P, body, present, want)
    else:
        ok = PO.decode(code.k, code.m, code.P, body, present, want)
    out = sh.copy()
    if ok:
        for i in range(sh.shape[0]):
            if not present[i] and (want is None or want[i]):
                out[i, :L] = body[i]
    return ok, out


@pytest.mark.parametrize("name", sorted(CODES))
def test_whole_bytes_equal_the_whole_shard_oracle(name):
    code = CODES[name]()
    tot, rng = code.k + code.m, np.random.default_rng(1)
    for L in ((128, 256, 1024) if code.kind == "pb" else (1, 15, 17, 112, 129, 300)):
        stride = -(-L // 128) * 128
        for trial in range(6):
            sh = stripe(code, L, stride, 100 * L + trial)
            present = np.ones(tot, dtype=np.uint8)
            present[rng.choice(tot, int(rng.integers(1, code.m + 2)), replace=False)] = 0
            want = None if trial % 2 else rng.integers(0, 2, tot).astype(np.uint8)
            dam = sh.copy()
            dam[present == 0] = 0x5A
            ok, want_out = whole_shard(code, dam, present, L, want)
            got = dam.copy()
            st = SO.reconstruct_stripe(code, got, np.where(present == 1, 0xFF, 0x00), L, want)
            assert (st == 0) == ok, (L, present, want)
            if ok:  # byte-identical on [0, L); the zero tail of every rebuilt shard is the only addition
                assert np.array_equal(got[:, :L], want_out[:, :L])
                assert np.array_equal(got[:, :L], np.where((present == 0)[:, None] & (
                    np.ones((tot, 1), bool) if want is None else (want != 0)[:, None]), sh[:, :L], dam[:, :L]))
            else:
                assert np.array_equal(got, dam)


def damage(code, L, n_bad, rng, bad_unit_limit):
    """seg_present of a pattern with n_bad damaged shards, each in one unit, at most bad_unit_limit per unit"""
    tot = code.k + code.m
    sp = np.full(tot, 0xFF, dtype=np.uint8)
    count = [0] * code.units
    for i in rng.choice(tot, n_bad, replace=False):
        g = int(rng.choice([u for u in range(code.units) if count[u] < bad_unit_limit]))
        count[g] += 1
        bits = (1 << g) | ((1 << (g + 4)) if code.kind == "pb" else 0)
        sp[i] &= ~np.uint8(bits & 0xFF)
    return sp


def trash(code, sh, sp, L):
    for i in range(sh.shape[0]):
        for g in range(8):
            if not (sp[i] >> g) & 1:
                o, n = SO.segments(L)[g]
                sh[i, o:o + n] ^= 0xA5


@pytest.mark.parametrize("name", sorted(CODES))
def test_recovers_more_than_m_damaged_shards(name):
    code = CODES[name]()
    tot, rng = code.k + code.m, np.random.default_rng(2)
    L = 1024 if code.kind == "pb" else 1000
    limit = 1 if code.kind == "lrc" else code.m  # LRC(10,2,2) is not MDS: one loss per unit always decodes
    for n_bad in range(code.m + 1, min(tot, limit * code.units) + 1):
        sh = stripe(code, L, 1024, n_bad)
        sp = damage(code, L, n_bad, rng, limit)
        got = sh.copy()
        trash(code, got, sp, L)
        assert SO.reconstruct_stripe(code, got, sp, L) == 0, n_bad
        assert np.array_equal(got, sh), n_bad


@pytest.mark.parametrize("name", sorted(CODES))
def test_a_unit_with_m_plus_one_bad_shards_is_unrecoverable(name):
    code = CODES[name]()
    tot, rng = code.k + code.m, np.random.default_rng(3)
    L = 1024 if code.kind == "pb" else 1000
    for trial in range(4):
        sh = stripe(code, L, 1024, 50 + trial)
        sp = np.full(tot, 0xFF, dtype=np.uint8)
        g = trial % code.units
        bits = (1 << g) | ((1 << (g + 4)) if code.kind == "pb" else 0)
        for i in rng.choice(tot, code.m + 1, replace=False):
            sp[i] &= ~np.uint8(bits & 0xFF)
        got = sh.copy()
        trash(code, got, sp, L)
        before = got.copy()
        assert SO.reconstruct_stripe(code, got, sp, L) == SO.E_UNRECOVERABLE
        assert np.array_equal(got, before)


def test_new_symbols_are_exported():
    L = G.load_library()
    out = subprocess.run(["nm", "-D", "--defined-only", G.lib_path()], capture_output=True, text=True).stdout
    for name in ("garage_ec_reconstruct_segments", "garage_ec_reconstruct_segments_stripes"):
        assert name in G.ABI_SYMBOLS and hasattr(L, name) and (" T " + name) in out


def test_a_null_context_is_refused():
    L = G.load_library()
    assert L.garage_ec_reconstruct_segments(None, None, None, None, None, None, 16, 1, 0, None) == G.E_INVALID
    assert L.garage_ec_reconstruct_segments_stripes(None, None, None, None, None, None, 16, 1) == G.E_INVALID
