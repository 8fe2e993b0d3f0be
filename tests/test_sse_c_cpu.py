"""CPU checks of SSE-C sealing (DESIGN.md 2.6): the scalar C oracle against FIPS-197 and the AES-256 GCM test cases of
McGrew and Viega, against `cryptography` when it is installed, the STREAM-LE31 framing against
tests/golden/sse_c_kat.json, the sealed-length arithmetic, and argument rejection before any CUDA call."""
import ctypes as C
import hashlib
import json
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

K15 = "feffe9928665731c6d6a8f9467308308feffe9928665731c6d6a8f9467308308"
P15 = ("d9313225f88406e5a55909c5aff5269a86a7a9531534f7da2e4c303d8a318a72"
       "1c3c0c95956809532fcf0e2449a6b525b16aedf5aa0de657ba637b391aafd255")
A16 = "feedfacedeadbeeffeedfacedeadbeefabaddad2"
# (key, iv, plaintext, aad, ciphertext, tag): "The Galois/Counter Mode of Operation (GCM)", test cases 13-18
GCM_CASES = [
    ("00" * 32, "00" * 12, "", "", "", "530f8afbc74536b9a963b4f1c4cb738b"),
    ("00" * 32, "00" * 12, "00" * 16, "", "cea7403d4d606b6e074ec5d3baf39d18", "d0d1c8a799996bf0265b98b5d48ab919"),
    (K15, "cafebabefacedbaddecaf888", P15, "",
     "522dc1f099567d07f47f37a32a84427d643a8cdcbfe5c0c97598a2bd2555d1aa"
     "8cb08e48590dbb3da7b08b1056828838c5f61e6393ba7a0abcc9f662898015ad", "b094dac5d93471bdec1a502270e3cc6c"),
    (K15, "cafebabefacedbaddecaf888", P15[:120], A16,
     "522dc1f099567d07f47f37a32a84427d643a8cdcbfe5c0c97598a2bd2555d1aa"
     "8cb08e48590dbb3da7b08b1056828838c5f61e6393ba7a0abcc9f662", "76fc6ece0f4e1768cddf8853bb2d551b"),
    (K15, "cafebabefacedbad", P15[:120], A16,
     "c3762df1ca787d32ae47c13bf19844cbaf1ae14d0b976afac52ff7d79bba9de0"
     "feb582d33934a4f0954cc2363bc73f7862ac430e64abe499f47c9b1f", "3a337dbf46a792c45e454913fe2ea8f2"),
    (K15, "9313225df88406e555909c5aff5269aa6a7a9538534f7da1e4c303d2a318a728"
          "c3c0c95156809539fcf0e2429a6b525416aedbf5a0de6a57a637b39b", P15[:120], A16,
     "5a8def2f0c9e53f1f75d7853659e2a20eeb2b22aafde6419a058ab4f6f746bf4"
     "0fc0c3b780f244452da3ebf1c5d82cdea2418997200ef82e44ae7e3f", "a44a8266ee1c8eb0c8b5d4cf5ae9f19a"),
]


def test_aes256_fips197_c3():
    out = O.aes256_encrypt(bytes(range(32)), bytes.fromhex("00112233445566778899aabbccddeeff"))
    assert out.hex() == "8ea2b7ca516745bfeafc49904b496089"


@pytest.mark.parametrize("case", range(len(GCM_CASES)), ids=["tc%d" % (13 + i) for i in range(len(GCM_CASES))])
def test_gcm_mcgrew_viega(case):
    k, iv, p, a, c, t = (bytes.fromhex(x) for x in GCM_CASES[case])
    assert O.gcm_seal(k, iv, p, a) == c + t


def test_oracle_matches_cryptography():
    aead = pytest.importorskip("cryptography.hazmat.primitives.ciphers.aead")
    rng = np.random.default_rng(2024)
    for _ in range(40):
        n = int(rng.choice([0, 1, 15, 16, 17, 4095, 4096, 4097, int(rng.integers(0, 20000))]))
        key, iv, p = rng.bytes(32), rng.bytes(12), rng.bytes(n)
        assert O.gcm_seal(key, iv, p) == aead.AESGCM(key).encrypt(iv, p, None), n
        nonce = rng.bytes(8)
        b = O.seal(key, nonce, p)
        chunks = max(1, -(-n // 4096))
        want = nonce + b"".join(aead.AESGCM(key).encrypt(nonce + struct.pack("<I", c | ((c == chunks - 1) << 31)),
                                                         p[4096 * c:4096 * (c + 1)], None) for c in range(chunks))
        assert b == want, n
        assert O.open_(key, b) == p


def _kat():
    with open(os.path.join(HERE, "golden", "sse_c_kat.json")) as f:
        return json.load(f)["records"]


def _kat_plain(n, seed):
    out = bytearray()
    ctr = 0
    while len(out) < n:
        out += hashlib.sha256(b"sse-c-kat %d %d" % (seed, ctr)).digest()
        ctr += 1
    return bytes(out[:n])


def test_stream_framing_matches_fixture():
    recs = _kat()
    assert [r["len"] for r in recs] == [0, 1, 15, 16, 4095, 4096, 4097, 8192, (1 << 20) - 1, 1 << 20]
    for i, r in enumerate(recs):
        key, nonce = bytes.fromhex(r["key"]), bytes.fromhex(r["nonce"])
        p = _kat_plain(r["len"], i)
        b = O.seal(key, nonce, p)
        assert len(b) == r["sealed_len"] == G.sealed_len(r["len"]) == O.sealed_len(r["len"])
        if "sealed" in r:
            assert b.hex() == r["sealed"], r["len"]
        else:
            assert hashlib.sha256(b).hexdigest() == r["sealed_sha256"], r["len"]
        assert G.blake2sum(b).hex() == r["blake2sum"]
        assert O.open_(key, b) == p


def test_oracle_open_rejects_tampering():
    rng = np.random.default_rng(5)
    key, nonce, p = rng.bytes(32), rng.bytes(8), rng.bytes(9000)
    b = bytearray(O.seal(key, nonce, p))
    assert O.open_(key, bytes(b)) == p
    for mutate in (lambda x: x.__setitem__(100, x[100] ^ 1), lambda x: x.__setitem__(8 + 4096 + 2, x[8 + 4096 + 2] ^ 1)):
        c = bytearray(b)
        mutate(c)
        assert O.open_(key, bytes(c)) is None
    swapped = b[:8] + b[8 + 4112:8 + 2 * 4112] + b[8:8 + 4112] + b[8 + 2 * 4112:]
    assert O.open_(key, bytes(swapped)) is None
    assert O.open_(key, bytes(b[:8 + 2 * 4112])) is None  # last chunk dropped: chunk 1 is not flagged last
    assert O.open_(bytes(32), bytes(b)) is None
    for bad_len in (0, 23, 8 + 4112 + 1, 8 + 4112 + 15):
        assert O.open_(key, bytes(b[:bad_len])) is None


def test_sealed_len_arithmetic_and_overflow():
    for n in (0, 1, 4095, 4096, 4097, 8192, 1 << 20, (1 << 20) - 1):
        assert G.sealed_len(n) == 8 + n + 16 * max(1, -(-n // 4096))
    assert G.sealed_len(0) == 24 and G.sealed_len(1 << 20) == 1052680
    # the longest block whose sealed form fits 32 bits: q whole chunks and a last one that ends at 2^32 - 1
    q = (0xFFFFFFFF - 8) // 4112
    rest = 0xFFFFFFFF - (8 + 4112 * q) - 16
    assert 0 < rest < 4096
    biggest = 4096 * q + rest
    assert G.sealed_len(biggest) == 0xFFFFFFFF
    L = G.load_library()
    v = C.c_uint32(0)
    assert L.garage_ec_sealed_len(biggest + 1, C.byref(v)) == G.E_INVALID
    assert L.garage_ec_sealed_len(0xFFFFFFFF, C.byref(v)) == G.E_INVALID
    assert L.garage_ec_sealed_len(0xFFF00000, C.byref(v)) == G.E_INVALID
    assert L.garage_ec_sealed_len(100, None) == G.E_INVALID


def test_seal_and_open_reject_bad_arguments_before_cuda():
    L = G.load_library()
    buf = (C.c_uint8 * 64)()
    p = C.cast(buf, C.c_void_p)
    # no context: invalid before anything else
    assert L.garage_ec_seal(None, p, 16, p, p, p, p, 128, p, None, 1, 0, None) == G.E_INVALID
    assert L.garage_ec_seal_blocks(None, p, p, p, p, p, 128, p, None, 1) == G.E_INVALID
    assert L.garage_ec_open(None, p, p, p, p, p, p, 16, p, p, p, 128, 1, 0, None) == G.E_INVALID
    assert L.garage_ec_open_stripes(None, p, p, p, p, p, p, p, p, p, 128, 1) == G.E_INVALID
