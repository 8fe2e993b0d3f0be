"""CPU model of the piggybacked Reed-Solomon code PB(k, m) (DESIGN.md section 2.2).  Test infrastructure only.

Arithmetic is the shift-and-xor multiplication table of oracle/rs_oracle_np.py (never log/exp), the parity rows P
are its RS(k, m) rows, and the elimination is lrc_oracle.Basis; nothing here is shared with the library.  It states
the normative parts of the code:

  * halves: shard = a-half [0, L/2) | b-half [L/2, L); groups G_1..G_{m-1} of data shards, contiguous, sizes as equal
    as possible, larger groups first;
  * encode: a-half of parity i = XOR_j P[i][j] a_j; b-half = XOR_j P[i][j] b_j, XOR (for i >= 1) XOR_{j in G_i} a_j;
  * half-rows q = 2*shard + half over the 2k half-data symbols; recoverability by rank;
  * read plan: rule 1 (lone lost data shard j of G_i, all other data and parities 0 and i present: the b-halves of
    the other data shards and of parities 0 and i, the a-halves of G_i minus j) and rule 2 (greedy rank basis of the
    present half-rows in q order).
"""
from __future__ import annotations

import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "oracle"))
import lrc_oracle as LO  # noqa: E402
import rs_oracle_np as NP  # noqa: E402


def groups(k: int, m: int) -> list[list[int]]:
    ng = m - 1
    base, rem = divmod(k, ng)
    out, j = [], 0
    for g in range(ng):
        n = base + (1 if g < rem else 0)
        out.append(list(range(j, j + n)))
        j += n
    return out


def shard_len(block_len: int, k: int) -> int:
    L = -(-block_len // k)
    return -(-L // 128) * 128


def build(k: int, m: int, kind: int = NP.VANDERMONDE) -> np.ndarray:
    assert 1 <= k <= 16 and 2 <= m <= 4
    return NP.build_matrix(k, m, kind)


def encode(P: np.ndarray, data: np.ndarray) -> np.ndarray:
    """data (k, L), L even -> parity (m, L)"""
    m, k = P.shape
    h = data.shape[1] // 2
    a, b = data[:, :h], data[:, h:]
    pa, pb = NP.encode(P, a), NP.encode(P, b)
    for i, g in enumerate(groups(k, m)[: m - 1], start=1):
        pb[i] ^= np.bitwise_xor.reduce(a[g], axis=0)
    return np.concatenate([pa, pb], axis=1)


def half_rows(k: int, m: int, P: np.ndarray) -> list[list[int]]:
    """2(k+m) generator rows over the 2k half-data symbols (column 2j + h)"""
    rows = []
    for sh in range(k + m):
        for h in range(2):
            v = [0] * (2 * k)
            if sh < k:
                v[2 * sh + h] = 1
            else:
                i = sh - k
                for j in range(k):
                    v[2 * j + h] = int(P[i, j])
                if h == 1 and i >= 1:
                    for j in groups(k, m)[i - 1]:
                        v[2 * j] = 1
            rows.append(v)
    return rows


def _wanted(k, m, present, want):
    return [o for o in range(k + m) if not present[o] and (want is None or want[o])]


def read_plan(k: int, m: int, P: np.ndarray, present, want=None):
    """(ok, sorted half-row indices q) by rules 1 and 2"""
    R = half_rows(k, m, P)
    wanted = _wanted(k, m, present, want)
    if len(wanted) == 1 and wanted[0] < k:
        j = wanted[0]
        i = next(g for g, mem in enumerate(groups(k, m), start=1) if j in mem)
        if all(present[x] for x in range(k) if x != j) and present[k] and present[k + i]:
            q = {2 * x + 1 for x in range(k) if x != j} | {2 * k + 1, 2 * (k + i) + 1}
            q |= {2 * x for x in groups(k, m)[i - 1] if x != j}
            return True, sorted(q)
    B, chosen = LO.Basis(2 * k), []
    for q in range(2 * (k + m)):
        if present[q >> 1] and len(chosen) < 2 * k and B.add(R[q]):
            chosen.append(q)
    ok = all(B.express(R[2 * o + h]) is not None for o in wanted for h in range(2))
    return ok, chosen


def recoverable(k: int, m: int, P: np.ndarray, present, want=None) -> bool:
    return read_plan(k, m, P, present, want)[0]


def decode(k: int, m: int, P: np.ndarray, shards: np.ndarray, present, want=None) -> bool:
    """shards (k+m, L), rebuilt in place from the planned halves only; False if unrecoverable"""
    R = half_rows(k, m, P)
    ok, surv = read_plan(k, m, P, present, want)
    if not ok:
        return False
    h = shards.shape[1] // 2
    half = lambda q: shards[q >> 1, (q & 1) * h:(q & 1) * h + h]  # noqa: E731
    src = [half(q).copy() for q in surv]
    B = LO.Basis(2 * k)
    for q in surv:  # both rules pick independent half-rows
        assert B.add(R[q])
    for o in _wanted(k, m, present, want):
        for hh in range(2):
            c = B.express(R[2 * o + hh])
            out = np.zeros(h, dtype=np.uint8)
            for cj, v in zip(c, src):
                if cj:
                    out ^= NP.MUL[cj][v]
            half(2 * o + hh)[:] = out
    return True
