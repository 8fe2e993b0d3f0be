"""CPU statement of reconstruct by segment (DESIGN.md section 2.10).  Test infrastructure only.

Each stripe is cut in units: for RS and LRC the 8 adler8 segments [g*S, min(L, (g+1)*S)), S = roundup16(ceil(L/8));
for PB (L % 128 == 0) the pairs of segments g and g+4, i.e. columns [g*L/8, (g+1)*L/8) of each half.  Each unit is
handed, as a stripe of its own, to that code's whole-shard oracle -- rs_oracle.c through oracle_lib, lrc_oracle or
pb_oracle -- with the unit's presence map, and only the wanted absent units are copied back (plus the zero tail
[L, roundup16(L)) when a shard's last unit is rebuilt).  A stripe with an unrecoverable unit is left untouched.
Nothing here is shared with the library.
"""
from __future__ import annotations

import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import lrc_oracle as LO  # noqa: E402
import oracle_lib as O  # noqa: E402
import pb_oracle as PO  # noqa: E402

E_INVALID, E_UNRECOVERABLE = -1, -4


class Code:
    """kind 'rs' (k, m, P), 'lrc' (k, l, P with l + r rows) or 'pb' (k, m, P)"""

    def __init__(self, kind: str, k: int, m: int, P: np.ndarray, l: int = 0):
        self.kind, self.k, self.m, self.P, self.l = kind, k, m, np.ascontiguousarray(P, dtype=np.uint8), l

    @property
    def units(self) -> int:
        return 4 if self.kind == "pb" else 8


def seg_bytes(L: int) -> int:
    return (-(-L // 8) + 15) // 16 * 16


def segments(L: int) -> list[tuple[int, int]]:
    """the 8 adler8 segments (offset, length) of an L-byte shard"""
    S = seg_bytes(L)
    return [(min(g * S, L), max(0, min(L, (g + 1) * S) - g * S)) for g in range(8)]


def unit_runs(code: Code, L: int, g: int) -> list[tuple[int, int]]:
    """(offset, length) runs of unit g in every shard"""
    if code.kind == "pb":
        S = L // 8
        return [(g * S, S), (L // 2 + g * S, S)]
    return [segments(L)[g]]


def unit_present(code: Code, b: int, L: int, g: int) -> bool:
    if sum(n for _, n in unit_runs(code, L, g)) == 0:
        return True
    if code.kind == "pb":
        return bool((b >> g) & 1 and (b >> (g + 4)) & 1)
    return bool((b >> g) & 1)


def _decode_unit(code: Code, sub: np.ndarray, pres, want) -> bool:
    """sub (k+m, w): one unit as a stripe of its own, rebuilt in place"""
    k, m = code.k, code.m
    if code.kind == "rs":
        w = sub.shape[1]
        flat = np.ascontiguousarray(sub).reshape(-1)
        _, st = O.reconstruct(k, m, code.P, flat, np.array(pres, dtype=np.uint8), w, 1)
        sub[:] = flat.reshape(sub.shape)
        return int(st[0]) == 0
    if code.kind == "lrc":
        return LO.decode(k, code.l, code.P, sub, pres, want)
    return PO.decode(k, m, code.P, sub, pres, want)


def reconstruct_stripe(code: Code, shards: np.ndarray, seg_present, L: int, want=None) -> int:
    """shards (k+m, stride) uint8, rebuilt in place; returns the stripe's status"""
    tot, stride = shards.shape
    if L > stride or (code.kind == "pb" and L % 128):
        return E_INVALID
    out = shards.copy()
    for g in range(code.units):
        runs = unit_runs(code, L, g)
        pres = [unit_present(code, int(seg_present[i]), L, g) for i in range(tot)]
        if all(pres):
            continue
        sub = np.concatenate([shards[:, o:o + n] for o, n in runs], axis=1)
        if not _decode_unit(code, sub, pres, want):
            return E_UNRECOVERABLE
        for i in range(tot):
            if pres[i] or (want is not None and not want[i]):
                continue
            c = 0
            for o, n in runs:
                out[i, o:o + n] = sub[i, c:c + n]
                c += n
            if code.kind != "pb" and runs[0][0] + runs[0][1] == L:  # the shard's last unit: zero tail
                out[i, L:min(stride, -(-L // 16) * 16)] = 0
    shards[:] = out
    return 0


def reconstruct(code: Code, shards: np.ndarray, seg_present: np.ndarray, stride: int, n: int, shard_len=None,
                want=None) -> np.ndarray:
    """the library's flat layout: shards n*(k+m)*stride, seg_present / want n*(k+m); returns status (n,)"""
    tot = code.k + code.m
    sh = shards.reshape(n, tot, stride)
    sp = np.asarray(seg_present, dtype=np.uint8).reshape(n, tot)
    wn = None if want is None else np.asarray(want, dtype=np.uint8).reshape(n, tot)
    status = np.zeros(n, dtype=np.int32)
    for s in range(n):
        L = stride if shard_len is None else int(shard_len[s])
        status[s] = reconstruct_stripe(code, sh[s], sp[s], L, None if wn is None else wn[s])
    return status
