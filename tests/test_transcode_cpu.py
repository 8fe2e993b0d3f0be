"""Code conversion without a GPU: the byte-gather model of DESIGN.md 2.3 (tests/transcode_oracle.py) against
"reassemble + encode with the existing oracles" for RS, LRC, PB and whole-block sources and destinations on ragged
lengths, and the argument check of garage_ec_transcode that needs no context."""
import ctypes as C
import os
import sys
import zlib

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import transcode_oracle as T  # noqa: E402

import garage_b200 as G  # noqa: E402

CODES = [("rep",), ("rs", 6, 3, 0), ("rs", 10, 4, 1), ("rs", 4, 2, 0), ("lrc", 10, 2, 2), ("lrc", 12, 2, 2),
         ("pb", 10, 4, 0), ("pb", 6, 3, 1)]
LENS = [0, 1, 15, 16, 17, 511, 4095, 30001]


@pytest.mark.parametrize("src", CODES, ids=lambda c: "-".join(map(str, c)))
@pytest.mark.parametrize("dst", [c for c in CODES if c[0] != "rep"], ids=lambda c: "-".join(map(str, c)))
def test_gather_model_matches_reassemble_and_encode(src, dst):
    rng = np.random.default_rng(zlib.crc32(repr((src, dst)).encode()))
    for n in LENS:
        block = rng.integers(0, 256, n, dtype=np.uint8)
        sh = T.encode_block(src, block, stride=T.shard_len(src, n) + 16)
        assert np.array_equal(T.reassemble(src, sh, n), block)
        want = T.encode_block(dst, block)
        got = T.transcode(src, dst, sh, n)
        assert np.array_equal(got, want), (src, dst, n)
        assert np.array_equal(T.reassemble(dst, got, n), block)


def test_shard_lengths_are_the_code_lengths():
    assert T.shard_len(("rs", 6, 3, 0), 1 << 20) == 174763
    assert T.shard_len(("rs", 10, 4, 0), 1 << 20) == 104858
    assert T.shard_len(("pb", 10, 4, 0), 1 << 20) == 104960
    assert T.shard_len(("rep",), 12345) == 12345
    # the byte counts of DESIGN.md 2.3 for RS(6,3) -> RS(10,4) on 1 MiB
    assert 6 * 174763 == 1048578 and 14 * 104858 == 1468012


def test_transcode_rejects_a_missing_destination_before_touching_cuda():
    L = G.load_library()
    buf = np.zeros(64, dtype=np.uint8)
    lens = np.ones(1, dtype=np.uint32)
    p = C.c_void_p(buf.ctypes.data)
    assert L.garage_ec_transcode(None, None, p, None, C.c_void_p(lens.ctypes.data), 16, p, 16, None, None, 1,
                                 G.MEM_HOST, None) == G.E_INVALID
    assert L.garage_ec_transcode(None, None, None, None, None, 16, None, 16, None, None, 0, G.MEM_DEVICE,
                                 None) == G.E_INVALID
