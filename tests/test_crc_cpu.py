"""CPU checks of the S3 CRC32 / CRC32C arithmetic (DESIGN.md 2.9): the oracle against the published check values
and zlib, garage_ec_crc_combine against the CRC of the concatenation, and the new entry points' refusals without a
device."""
import ctypes as C
import os
import sys
import zlib

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import crc_oracle as O  # noqa: E402
import garage_b200 as G  # noqa: E402

KINDS = (G.CRC32, G.CRC32C)


def test_check_values():
    assert O.crc(O.CRC32, b"123456789") == 0xCBF43926
    assert O.crc(O.CRC32C, b"123456789") == 0xE3069283
    for kind in KINDS:
        assert O.crc(kind, b"") == 0


def test_rfc3720_vectors():
    assert O.crc(O.CRC32C, bytes(32)) == 0x8A9136AA
    assert O.crc(O.CRC32C, b"\xff" * 32) == 0x62A8AB43
    assert O.crc(O.CRC32C, bytes(range(32))) == 0x46DD794E
    assert O.crc(O.CRC32C, bytes(range(31, -1, -1))) == 0x113FDB5C


def test_oracle_crc32_is_zlib():
    rng = np.random.default_rng(29)
    for n in [0, 1, 2, 3, 15, 16, 17, 4095, 4096, 4097] + [int(x) for x in rng.integers(0, 70000, 20)]:
        b = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        assert O.crc(O.CRC32, b) == zlib.crc32(b), n


@pytest.mark.parametrize("kind", KINDS)
def test_combine_is_crc_of_concatenation(kind):
    rng = np.random.default_rng(30 + kind)
    for _ in range(60):
        n = int(rng.integers(0, 20000))
        b = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        cut = int(rng.choice([0, n, int(rng.integers(0, n + 1))]))
        a, c = b[:cut], b[cut:]
        want = O.crc(kind, b)
        assert G.crc_combine(kind, O.crc(kind, a), O.crc(kind, c), len(c)) == want, (n, cut)
        assert O.combine(kind, O.crc(kind, a), O.crc(kind, c), len(c)) == want


@pytest.mark.parametrize("kind", KINDS)
def test_combine_long_and_empty_lengths(kind):
    rng = np.random.default_rng(40 + kind)
    for _ in range(20):
        a, b = (int(x) for x in rng.integers(0, 1 << 32, 2))
        n = int(rng.integers(0, 1 << 62))
        assert G.crc_combine(kind, a, b, n) == O.combine(kind, a, b, n), n
        assert G.crc_combine(kind, a, b, 0) == a ^ b
    assert G.crc_combine(kind, 0x1234, 0, 0) == 0x1234


def test_combine_folds_blocks_in_order():
    """what a caller does with the per-block CRCs of a sealed object: fold them, left to right"""
    rng = np.random.default_rng(41)
    blocks = [rng.integers(0, 256, int(n), dtype=np.uint8).tobytes() for n in (1 << 20, 1, 0, 12345, 4096, 77)]
    for kind in KINDS:
        acc = 0
        for b in blocks:
            acc = G.crc_combine(kind, acc, O.crc(kind, b), len(b))
        assert acc == O.crc(kind, b"".join(blocks))


def test_combine_rejects_unknown_kinds_and_null_out():
    L = G.load_library()
    v = C.c_uint32(0)
    for kind in (G.CRC_NONE, 3, 255, -1):
        assert L.garage_ec_crc_combine(kind, 1, 2, 3, C.byref(v)) == G.E_INVALID
    assert L.garage_ec_crc_combine(G.CRC32, 1, 2, 3, None) == G.E_INVALID
    with pytest.raises(G.EcError):
        G.crc_combine(3, 0, 0, 0)


def test_new_entry_points_refuse_without_a_context():
    L = G.load_library()
    kinds = (C.c_uint8 * 1)(1)
    crcs = (C.c_uint32 * 1)()
    for mem in (G.MEM_HOST, G.MEM_DEVICE):
        assert L.garage_ec_seal_crc(None, None, 16, None, None, None, None, 128, None, None, kinds, crcs, 1, mem,
                                    None) == G.E_INVALID
        assert L.garage_ec_reseal_crc(None, None, None, None, None, None, 0, None, None, None, None, None, None, None,
                                      None, None, None, None, kinds, crcs, 128, 1, mem, None) == G.E_INVALID
    assert L.garage_ec_seal_blocks_crc(None, None, None, None, None, None, 128, None, None, kinds, crcs,
                                       1) == G.E_INVALID
    assert L.garage_ec_reseal_stripes_crc(None, None, None, None, None, None, 0, None, None, None, None, None, None, None,
                                          None, None, None, None, kinds, crcs, 128, 1) == G.E_INVALID


@pytest.mark.skipif(__import__("torch").cuda.is_available(), reason="checks the no-GPU behaviour")
def test_no_device_means_error():
    with pytest.raises(G.EcError) as ei:
        G.GarageEc(device=0, k=10, m=4)
    assert ei.value.code == G.E_NODEVICE
