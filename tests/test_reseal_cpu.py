"""CPU checks of copies with re-encryption (DESIGN.md 2.8): the oracle composition the GPU tests expect -- open every
source with the scalar C oracle, cut and concatenate the pieces, seal under the new key -- against `cryptography`'s
AES-GCM on the same inputs, including pieces that cross chunks and sources; and argument rejection before any CUDA
call."""
import ctypes as C
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


def _aesgcm():
    return pytest.importorskip("cryptography.hazmat.primitives.ciphers.aead").AESGCM


def _stream_seal(key, nonce8, pt):
    """Garage's STREAM-LE31 over 4096-byte chunks, written from AES-GCM alone"""
    g = _aesgcm()(key)
    n = max(1, -(-len(pt) // 4096))
    out = [nonce8]
    for c in range(n):
        iv = nonce8 + struct.pack("<I", c | ((c == n - 1) << 31))
        out.append(g.encrypt(iv, pt[4096 * c:4096 * (c + 1)], None))
    return b"".join(out)


def _stream_open(key, b):
    g = _aesgcm()(key)
    body = b[8:]
    n = max(1, -(-len(body) // 4112))
    return b"".join(g.decrypt(b[:8] + struct.pack("<I", c | ((c == n - 1) << 31)), body[4112 * c:4112 * (c + 1)], None)
                    for c in range(n))


def reseal_oracle(sources, src_keys, pieces, piece_start, dst_keys, dst_nonces):
    """B'_d per destination: open each source with the C oracle (None: the source is plaintext), then seal Q_d"""
    plain = [O.open_(src_keys[i], b) if src_keys is not None else b for i, b in enumerate(sources)]
    out = []
    for d in range(len(piece_start) - 1):
        q = b"".join(plain[s][o:o + n] for s, o, n in pieces[piece_start[d]:piece_start[d + 1]])
        out.append((q, O.seal(dst_keys[d], dst_nonces[d], q)))
    return out


def _case(seed, keyed):
    rng = np.random.default_rng(seed)
    lens = [0, 1, 17, 4095, 4096, 4097, 8193, 40000]
    plains = [rng.bytes(n) for n in lens]
    keys = [rng.bytes(32) for _ in lens] if keyed else None
    sources = [O.seal(keys[i], rng.bytes(8), p) if keyed else p for i, p in enumerate(plains)]
    # whole blocks, a piece across chunks 0/1, tails and heads of two sources, tiny pieces, one source twice
    dests = [
        [(7, 0, 40000)],
        [(5, 4090, 7)],
        [(6, 4000, 4193), (4, 0, 4096)],
        [(7, 39990, 10), (6, 0, 5000), (2, 3, 14)],
        [(3, i, 1 + i % 17) for i in range(0, 4000, 97)],
        [(7, 12288, 4097), (7, 12288, 4097)],
        [(1, 0, 1)],
    ]
    pieces = [p for d in dests for p in d]
    piece_start = np.cumsum([0] + [len(d) for d in dests]).tolist()
    dst_keys = [rng.bytes(32) for _ in dests]
    dst_nonces = [rng.bytes(8) for _ in dests]
    return plains, keys, sources, pieces, piece_start, dst_keys, dst_nonces


@pytest.mark.parametrize("keyed", [True, False], ids=["sse_c_source", "plaintext_source"])
def test_oracle_composition_matches_cryptography(keyed):
    plains, keys, sources, pieces, piece_start, dst_keys, dst_nonces = _case(31 + keyed, keyed)
    if keyed:
        for k, b, p in zip(keys, sources, plains):
            assert _stream_open(k, b) == p
    got = reseal_oracle(sources, keys, pieces, piece_start, dst_keys, dst_nonces)
    for d, (q, b) in enumerate(got):
        want_q = b"".join(plains[s][o:o + n] for s, o, n in pieces[piece_start[d]:piece_start[d + 1]])
        assert q == want_q
        assert b == _stream_seal(dst_keys[d], dst_nonces[d], q), d
        assert len(b) == G.sealed_len(len(q))
        assert _stream_open(dst_keys[d], b) == q
        assert O.open_(keys[0] if keyed else bytes(32), b) is None  # not under any source key


def test_bad_arguments_rejected_before_touching_cuda():
    L = G.load_library()
    z = C.c_void_p(16)
    args = [z, z, z, z, None, 1, z, z, z, z, z, z, None, z, z, z, z, 16, 1]
    # no context
    assert L.garage_ec_reseal(None, *args, G.MEM_HOST, None) == G.E_INVALID
    assert L.garage_ec_reseal(None, *args, G.MEM_DEVICE, None) == G.E_INVALID
    assert L.garage_ec_reseal_stripes(None, *args) == G.E_INVALID
    # an unknown memory kind
    assert L.garage_ec_reseal(None, *args, 7, None) == G.E_INVALID
