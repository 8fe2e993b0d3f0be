"""CPU checks of ranged SSE-C opens (DESIGN.md 2.7): garage_ec_sealed_range against independent arithmetic at every
edge, and the claim it rests on -- the span's chunks, opened under their STREAM nonces with `cryptography`'s AES-GCM,
give exactly the plaintext slice of an oracle-sealed block."""
import os
import struct
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import garage_b200 as G  # noqa: E402
import sse_c_oracle as O  # noqa: E402

CH, FR = 4096, 4112


def ref_range(S, o, ln):
    """(span_off, span_len, c0, n_chunks) of plaintext bytes [o, o + ln) of a block sealed to S bytes, or an E_* code"""
    if S < 24 or 1 <= (S - 8) % FR < 16:
        return G.E_AUTH
    n = (S - 8 + FR - 1) // FR
    P = S - 8 - 16 * n
    if o + ln > P:
        return G.E_INVALID
    c0 = o // CH
    if ln == 0:
        return min(S, 8 + FR * c0), 0, c0, 0
    c1 = (o + ln - 1) // CH
    lo = 8 + FR * c0
    return lo, min(S, 8 + FR * (c1 + 1)) - lo, c0, c1 - c0 + 1


def got_range(S, o, ln):
    try:
        return G.GarageEc.sealed_range(S, o, ln)
    except G.EcError as e:
        return e.code


PLENS = [0, 1, 15, 16, 4095, 4096, 4097, 2 * 4096, 3 * 4096, 3 * 4096 + 5, 300001, (1 << 20) - 977, 1 << 20]


def _offsets(P):
    last = (max(P, 1) - 1) // CH * CH  # start of the last chunk
    return sorted({o for o in (0, 1, 4095, 4096, 4097, 8191, 8192, last, last + 1, P - 1, P - 17, P // 2, P)
                   if 0 <= o <= P})


@pytest.mark.parametrize("P", PLENS)
def test_sealed_range_matches_arithmetic(P):
    S = G.sealed_len(P)
    assert S == 8 + P + 16 * max(1, -(-P // CH))
    for o in _offsets(P):
        for ln in sorted({0, 1, 15, 16, 17, 4095, 4096, 4097, 8192, 65536, P - o, P - o + 1, P + 1}):
            if ln < 0:
                continue
            want = ref_range(S, o, ln)
            assert got_range(S, o, ln) == want, (P, o, ln)
            if isinstance(want, tuple) and ln:
                span_off, span_len, c0, nch = want
                # the span is whole sealed chunks, and the last one of the block ends at S
                assert span_off == 8 + FR * c0 and c0 == o // CH and c0 + nch - 1 == (o + ln - 1) // CH
                assert span_off + span_len <= S


def test_sealed_range_edges():
    S = G.sealed_len(1 << 20)  # 256 chunks
    assert got_range(S, 0, 4096) == (8, 4112, 0, 1)
    assert got_range(S, 4095, 2) == (8, 2 * 4112, 0, 2)
    assert got_range(S, 4096, 4096) == (8 + 4112, 4112, 1, 1)
    assert got_range(S, 4097, 4096) == (8 + 4112, 2 * 4112, 1, 2)
    assert got_range(S, (1 << 20) - 1, 1) == (8 + 255 * 4112, 4112, 255, 1)
    assert got_range(S, 0, 1 << 20) == (8, 256 * 4112, 0, 256)
    assert got_range(S, 1, 1 << 20) == G.E_INVALID
    assert got_range(S, (1 << 20) + 1, 0) == G.E_INVALID
    assert got_range(S, 1 << 20, 0) == (S, 0, 256, 0)
    # the short last chunk: its span ends at S, not at a whole frame
    S2 = G.sealed_len(2 * 4096 + 100)
    assert got_range(S2, 2 * 4096 + 50, 50) == (8 + 2 * 4112, 116, 2, 1)
    assert got_range(S2, 4000, 4292) == (8, S2 - 8, 0, 3)
    # the empty block: one empty chunk, only the empty range
    assert got_range(24, 0, 0) == (8, 0, 0, 0)
    assert got_range(24, 0, 1) == G.E_INVALID


@pytest.mark.parametrize("S", [0, 8, 23, 8 + 4112 + 8, 8 + 4112 + 1, 8 + 4112 + 15, 8 + 2 * 4112 + 7])
def test_sealed_range_malformed_length(S):
    assert got_range(S, 0, 0) == G.E_AUTH
    assert got_range(S, 0, 1) == G.E_AUTH


def test_sealed_range_rejects_null_outputs():
    L = G.load_library()
    assert L.garage_ec_sealed_range(G.sealed_len(100), 0, 10, None, None, None, None) == G.E_INVALID


def _nonce(N, c, n):
    return N + struct.pack("<I", c | ((1 << 31) if c == n - 1 else 0))


@pytest.mark.parametrize("P", [1, 4096, 3 * 4096, 300001, (1 << 20) - 977, 1 << 20])
def test_span_chunks_decrypt_to_the_slice(P):
    aead = pytest.importorskip("cryptography.hazmat.primitives.ciphers.aead")
    rng = np.random.default_rng(P)
    key, N = rng.bytes(32), rng.bytes(8)
    pt = rng.bytes(P)
    B = O.seal(key, N, pt)
    S = len(B)
    assert S == G.sealed_len(P)
    n = (S - 8 + FR - 1) // FR
    gcm = aead.AESGCM(key)
    ranges = [(0, 1), (0, P), (P - 1, 1), (max(0, P - 5000), min(P, 5000))]
    ranges += [(o, min(P - o, 4096)) for o in _offsets(P) if o < P]
    for _ in range(12):
        o = int(rng.integers(0, P))
        ranges.append((o, int(rng.integers(1, P - o + 1))))
    for o, ln in ranges:
        span_off, span_len, c0, nch = G.GarageEc.sealed_range(S, o, ln)
        span = B[span_off:span_off + span_len]
        got = b""
        for i in range(nch):
            c = c0 + i
            frame = span[i * FR:(i + 1) * FR]
            got += gcm.decrypt(_nonce(B[:8], c, n), frame, None)
        base = c0 * CH
        assert got[o - base:o - base + ln] == pt[o:o + ln], (P, o, ln)
