"""CPU model of code conversion (DESIGN.md section 2.3).  Test infrastructure only.

A code is a tuple: ("rep",) for a whole-block replica, ("rs", k, m, kind), ("lrc", k, l, r) or ("pb", k, m, kind).
Encoding goes through the existing models (oracle/rs_oracle_np.py, tests/lrc_oracle.py, tests/pb_oracle.py).

Two statements of the transcode are kept, and the tests check that they agree:
  * `reassemble` + `encode_block`: the block is the first block_len bytes of the source data shards concatenated, the
    output is the destination code's encode of that block;
  * `transcode`: destination data byte (j, c) is source byte (o // L_s, o % L_s) with o = j*L_d + c, zero past
    block_len -- the gather the GPU kernel does.
"""
from __future__ import annotations

import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "oracle"))
import lrc_oracle as LO  # noqa: E402
import pb_oracle as PB  # noqa: E402
import rs_oracle_np as NP  # noqa: E402


def k_of(code) -> int:
    return 1 if code[0] == "rep" else code[1]


def m_of(code) -> int:
    if code[0] == "rep":
        return 0
    return code[2] + code[3] if code[0] == "lrc" else code[2]


def shard_len(code, block_len: int) -> int:
    if code[0] == "rep":
        return block_len
    if code[0] == "pb":
        return PB.shard_len(block_len, code[1])
    return -(-block_len // code[1])


def matrix(code) -> np.ndarray:
    if code[0] == "lrc":
        return LO.build_lrc(code[1], code[2], code[3])
    if code[0] == "pb":
        return PB.build(code[1], code[2], code[3])
    return NP.build_matrix(code[1], code[2], code[3])


def encode_block(code, block: np.ndarray, stride: int | None = None) -> np.ndarray:
    """(k+m, stride) shards of `block` under `code`, zero past shard_len"""
    k, m, L = k_of(code), m_of(code), shard_len(code, block.size)
    stride = L if stride is None else stride
    out = np.zeros((k + m, stride), dtype=np.uint8)
    flat = np.zeros(k * L, dtype=np.uint8)
    flat[: block.size] = block
    out[:k, :L] = flat.reshape(k, L)
    if m and L:
        enc = PB.encode if code[0] == "pb" else NP.encode
        out[k:, :L] = enc(matrix(code), out[:k, :L])
    return out


def reassemble(code, shards: np.ndarray, block_len: int) -> np.ndarray:
    """the block stored as `shards` ((k+m, >= L) array) under `code`"""
    k, L = k_of(code), shard_len(code, block_len)
    return np.ascontiguousarray(shards[:k, :L]).reshape(-1)[:block_len].copy()


def transcode(src_code, dst_code, shards: np.ndarray, block_len: int, stride: int | None = None) -> np.ndarray:
    """destination shards by the byte gather of DESIGN.md 2.3, then the destination parities"""
    Ls, Ld, kd, md = shard_len(src_code, block_len), shard_len(dst_code, block_len), k_of(dst_code), m_of(dst_code)
    stride = Ld if stride is None else stride
    out = np.zeros((kd + md, stride), dtype=np.uint8)
    o = np.arange(kd * Ld, dtype=np.int64).reshape(kd, Ld)
    valid = o < block_len
    src = np.where(valid, o // max(Ls, 1), 0), np.where(valid, o % max(Ls, 1), 0)
    out[:kd, :Ld] = np.where(valid, shards[src[0], src[1]], 0)
    if md and Ld:
        enc = PB.encode if dst_code[0] == "pb" else NP.encode
        out[kd:, :Ld] = enc(matrix(dst_code), out[:kd, :Ld])
    return out
