"""CPU model of the locally repairable code LRC(k, l, r) (DESIGN.md section 2).  Test infrastructure only.

Arithmetic is the shift-and-xor multiplication table of oracle/rs_oracle_np.py (never log/exp); the
elimination below is this module's own.  It states the normative parts of the code:

  * the generator: data rows e_j, l local rows (all ones on group g = data [g*k/l, (g+1)*k/l)), then the r
    Cauchy rows P[i][j] = 1/((k+i) xor j) of RS(k, r);
  * recoverability by rank: a wanted absent shard can be rebuilt iff its generator row lies in the span of
    the present rows;
  * survivor selection: rule 1 (local repair) and rule 2 (greedy rank basis in index order), the set
    garage_ec_read_set returns and reconstruct reads.
"""
from __future__ import annotations

import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
import rs_oracle_np as NP  # noqa: E402

MULL = NP.MUL.tolist()
INV = [0] + [NP.gf_inv_scalar(a) for a in range(1, 256)]


def build_lrc(k: int, l: int, r: int) -> np.ndarray:
    """(l + r) x k parity rows: local rows, then global rows"""
    assert l >= 1 and r >= 1 and k % l == 0 and l + r <= 8 and k <= 32
    gs = k // l
    loc = np.array([[1 if j // gs == g else 0 for j in range(k)] for g in range(l)], dtype=np.uint8)
    glob = np.array([[INV[(k + i) ^ j] for j in range(k)] for i in range(r)], dtype=np.uint8)
    return np.concatenate([loc, glob], axis=0)


def generator_rows(k: int, P: np.ndarray) -> list[list[int]]:
    return [[int(i == j) for j in range(k)] for i in range(k)] + [list(map(int, row)) for row in P]


class Basis:
    """Rows kept in insertion order, each normalised at its pivot and zero at every earlier pivot; `comb[b]` gives
    row b as a combination of the inserted source rows."""

    def __init__(self, k: int):
        self.k, self.rows, self.piv, self.comb = k, [], [], []

    def reduce(self, v, c=None):
        v = list(v)
        c = [0] * self.k if c is None else list(c)
        for p, row, cb in zip(self.piv, self.rows, self.comb):
            f = v[p]
            if f:
                mf = MULL[f]
                v = [a ^ mf[b] for a, b in zip(v, row)]
                c = [a ^ mf[b] for a, b in zip(c, cb)]
        return v, c

    def add(self, v) -> bool:
        """insert v if it raises the rank"""
        c = [0] * self.k
        c[len(self.rows)] = 1
        v, c = self.reduce(v, c)
        p = next((j for j, x in enumerate(v) if x), None)
        if p is None:
            return False
        mi = MULL[INV[v[p]]]
        self.rows.append([mi[x] for x in v])
        self.comb.append([mi[x] for x in c])
        self.piv.append(p)
        return True

    def express(self, v):
        """coefficients over the inserted rows that give v, or None if v is outside the span"""
        r, c = self.reduce(v)
        return None if any(r) else c[: len(self.rows)]


def rank(k: int, rows) -> int:
    B = Basis(k)
    for v in rows:
        if len(B.rows) < k:
            B.add(v)
    return len(B.rows)


def recoverable(k: int, P: np.ndarray, present, want=None) -> bool:
    """rank test: every wanted absent row lies in the span of the present rows"""
    G = generator_rows(k, P)
    tot = len(G)
    B = Basis(k)
    for i in range(tot):
        if present[i] and len(B.rows) < k:
            B.add(G[i])
    return all(B.express(G[o]) is not None for o in range(tot)
               if not present[o] and (want is None or want[o]))


def read_set(k: int, l: int, P: np.ndarray, present, want=None):
    """(ok, sorted survivor indices) by rules 1 and 2; l = 0: RS, the first k present shards"""
    G = generator_rows(k, P)
    tot = len(G)
    wanted = [o for o in range(tot) if not present[o] and (want is None or want[o])]
    if l == 0:
        surv = [i for i in range(tot) if present[i]][:k]
        return len(surv) == k, surv
    gs = k // l

    def members(g):
        return list(range(g * gs, (g + 1) * gs)) + [k + g]

    surv, local = set(), True
    for o in wanted:
        if o >= k + l:
            local = False
            break
        mem = members(o // gs if o < k else o - k)
        if any(not present[i] for i in mem if i != o):
            local = False
            break
        surv |= {i for i in mem if i != o}
    if local:
        return True, sorted(surv)
    B, chosen = Basis(k), []
    for i in range(tot):
        if present[i] and len(chosen) < k and B.add(G[i]):
            chosen.append(i)
    ok = all(B.express(G[o]) is not None for o in wanted)
    return ok, chosen


def decode(k: int, l: int, P: np.ndarray, shards: np.ndarray, present, want=None) -> bool:
    """shards: (k+m, L) uint8, rebuilt in place from the read set only; False if unrecoverable"""
    G = generator_rows(k, P)
    ok, surv = read_set(k, l, P, present, want)
    if not ok:
        return False
    B = Basis(k)
    for i in surv:  # both rules pick independent rows
        assert B.add(G[i])
    for o in range(len(G)):
        if present[o] or (want is not None and not want[o]):
            continue
        c = B.express(G[o])
        out = np.zeros(shards.shape[1], dtype=np.uint8)
        for cj, i in zip(c, surv):
            if cj:
                out ^= NP.MUL[cj][shards[i]]
        shards[o] = out
    return True


def encode(P: np.ndarray, data: np.ndarray) -> np.ndarray:
    return NP.encode(P, data)
