"""CPU checks of the tag arithmetic of ranged reads: garage_ec_tag_span / garage_ec_check_shard_span_host against
zlib.adler32 segments (adler8) and Garage's blake2sum (whole shard), and garage_ec_check_shard_half_host, now a call of
the span check, against a model of its verdicts."""
import os
import struct
import sys
import zlib

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import garage_b200 as G  # noqa: E402

LENS = [1, 7, 15, 16, 17, 100, 127, 128, 129, 255, 1000, 4096, 4097, 13120 * 8 - 3, 104858, 106496]


def seg_bytes(L):
    return ((L + 7) // 8 + 15) // 16 * 16


def adler8(data):
    L = len(data)
    seg = seg_bytes(L)
    return b"".join(struct.pack("<I", zlib.adler32(data[j * seg:(j + 1) * seg])) for j in range(8))


def span_model(L, off, n):
    if n == 0:
        return off, 0
    seg = seg_bytes(L)
    a = off // seg * seg
    b = min(-(-(off + n) // seg) * seg, L)
    return a, b - a


@pytest.mark.parametrize("L", LENS)
def test_tag_span_is_the_covering_segments(L):
    rng = np.random.default_rng(L)
    cases = [(0, L), (0, 1), (L - 1, 1), (L, 0)]
    cases += [(int(o), int(rng.integers(0, L - o + 1))) for o in rng.integers(0, L, 40)]
    for off, n in cases:
        assert G.tag_span(G.SUM_ADLER8, L, off, n) == span_model(L, off, n), (L, off, n)
        assert G.tag_span(G.SUM_BLAKE2, L, off, n) == (0, L)
    with pytest.raises(G.EcError):
        G.tag_span(G.SUM_ADLER8, L, L, 1)
    with pytest.raises(G.EcError):
        G.tag_span(7, L, 0, 1)


@pytest.mark.parametrize("L", LENS)
def test_span_check_matches_zlib_segments(L):
    rng = np.random.default_rng(100 + L)
    shard = rng.integers(0, 256, L, dtype=np.uint8)
    tag = adler8(shard.tobytes())
    assert G.shard_sum_host(G.SUM_ADLER8, shard) == tag
    for _ in range(30):
        off = int(rng.integers(0, L))
        n = int(rng.integers(1, L - off + 1))
        a, b = G.tag_span(G.SUM_ADLER8, L, off, n)
        span = shard[a:a + b].copy()
        assert G.check_shard_span_host(G.SUM_ADLER8, span, L, a, tag) == 0
        # a flipped byte inside the span is caught
        x = int(rng.integers(0, b))
        span[x] ^= 0x40
        assert G.check_shard_span_host(G.SUM_ADLER8, span, L, a, tag) == 1
    seg = seg_bytes(L)
    if seg < L:
        # the last segment ends at the shard's end; spans that are not whole segments are refused
        assert G.check_shard_span_host(G.SUM_ADLER8, shard[seg:], L, seg, tag) == 0
        assert G.check_shard_span_host(G.SUM_ADLER8, shard[1:seg], L, 1, tag) == G.E_INVALID
        assert G.check_shard_span_host(G.SUM_ADLER8, shard[0:seg - 1], L, 0, tag) == G.E_INVALID


@pytest.mark.parametrize("L", [1, 100, 4097, 104858])
def test_blake2_span_is_the_whole_shard(L):
    rng = np.random.default_rng(200 + L)
    shard = rng.integers(0, 256, L, dtype=np.uint8)
    tag = G.blake2sum(shard.tobytes())
    assert G.check_shard_span_host(G.SUM_BLAKE2, shard, L, 0, tag) == 0
    bad = shard.copy()
    bad[L // 2] ^= 1
    assert G.check_shard_span_host(G.SUM_BLAKE2, bad, L, 0, tag) == 1
    if L > 1:
        assert G.check_shard_span_host(G.SUM_BLAKE2, shard[1:], L, 1, tag) == G.E_INVALID


def half_model(kind, half, L, which, tag):
    """the verdicts garage_ec_check_shard_half_host gave before it called the span check"""
    if kind != G.SUM_ADLER8 or L % 128 or which not in (0, 1):
        return G.E_INVALID
    seg = L // 8
    for t in range(4):
        v = zlib.adler32(bytes(half[t * seg:(t + 1) * seg])) if seg else 1
        if v != struct.unpack("<I", tag[4 * (4 * which + t):4 * (4 * which + t) + 4])[0]:
            return 1
    return 0


@pytest.mark.parametrize("L", [0, 128, 256, 1024, 104960, 106496])
def test_half_check_keeps_its_verdicts(L):
    rng = np.random.default_rng(300 + L)
    shard = rng.integers(0, 256, L, dtype=np.uint8)
    good = adler8(shard.tobytes())
    tags = [good, bytes(32), bytes(rng.integers(0, 256, 32, dtype=np.uint8))]
    flipped = bytearray(good)
    flipped[5] ^= 1
    tags.append(bytes(flipped))
    for tag in tags:
        for which in (0, 1):
            half = shard[which * (L // 2):(which + 1) * (L // 2)] if L else np.zeros(0, np.uint8)
            for kind in (G.SUM_ADLER8, G.SUM_BLAKE2):
                got = G.check_shard_half_host(kind, half, L, which, tag)
                assert got == half_model(kind, half, L, which, tag), (L, which, kind)
    assert G.check_shard_half_host(G.SUM_ADLER8, shard[:64], 129, 0, good) == G.E_INVALID
