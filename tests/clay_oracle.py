"""CPU model of the Clay code Clay(k, m) (DESIGN.md section 2.4).  Test infrastructure only.

Arithmetic is the multiplication table of oracle/rs_oracle_np.py and the base-code rows are its RS(k+s, m) rows;
nothing here is shared with the library.  It states the normative parts of the code, straight from the definition:

  * q = m, t = ceil((k+m)/q), n' = q*t nodes, s = n' - k - m virtual nodes, alpha = q^t layers;
  * node i sits at (x, y) = (i mod q, i div q); data shard j is node j, virtual nodes k..k+s-1 (always zero), parity
    shard j is node k+s+j;
  * layer z of a shard of length L is bytes [z*L/alpha, (z+1)*L/alpha); digit y of z is (z // q^y) % q;
  * coupling with gamma = 2: C_a = U_a ^ g*U_b, C_b = U_b ^ g*U_a for the pair a = (x, y) in layer z,
    b = (z_y, y) in layer z + (x - z_y) q^y; C = U where z_y = x;
  * every layer's U is a codeword of the systematic RS(k+s, m) with parity rows P.

Arrays of one stripe are (nodes or shards, alpha, sub) with sub = L / alpha bytes per layer.
"""
from __future__ import annotations

import itertools
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "oracle"))
import rs_oracle_np as NP  # noqa: E402

MUL = NP.MUL
GAMMA = 2
INV_GAMMA = NP.gf_inv_scalar(GAMMA)
INV_DET = NP.gf_inv_scalar(1 ^ int(MUL[GAMMA, GAMMA]))  # (1 + gamma^2)^-1


def params(k: int, m: int):
    """(q, t, n', s, alpha); ValueError for a code outside m in {2,3,4}, k >= 2, alpha <= 256"""
    if m not in (2, 3, 4) or k < 2:
        raise ValueError("Clay(%d,%d): needs m in {2,3,4} and k >= 2" % (k, m))
    q = m
    t = -(-(k + m) // q)
    alpha = q ** t
    if alpha > 256:
        raise ValueError("Clay(%d,%d): alpha = %d > 256" % (k, m, alpha))
    return q, t, q * t, q * t - k - m, alpha


def shard_len(block_len: int, k: int, m: int) -> int:
    alpha = params(k, m)[4]
    L = -(-block_len // k)
    return -(-L // (16 * alpha)) * (16 * alpha)


def build(k: int, m: int, kind: int = NP.VANDERMONDE) -> np.ndarray:
    """parity rows of the base code RS(k+s, m): m x (k+s)"""
    s = params(k, m)[3]
    return NP.build_matrix(k + s, m, kind)


def node_of_shard(k: int, m: int, i: int) -> int:
    return i if i < k else i + params(k, m)[3]


def digit(z, y: int, q: int):
    return (z // q ** y) % q


def _partner(a: int, q: int, alpha: int):
    """for node a, over all layers: (mask z_y != x, partner node b, partner layer z')"""
    x, y = a % q, a // q
    z = np.arange(alpha)
    zy = digit(z, y, q)
    return zy != x, zy + y * q, z + (x - zy) * q ** y


def _mul(c: int, a: np.ndarray) -> np.ndarray:
    return MUL[c][a]


def _base_solve(P: np.ndarray, kb: int, present_nodes, want_nodes, U: np.ndarray, layers) -> None:
    """U[want, layers] from U[present, layers] (the first kb present nodes) through RS(kb, m)"""
    m = P.shape[0]
    G = np.concatenate([np.eye(kb, dtype=np.uint8), P], axis=0)
    surv = list(present_nodes)[:kb]
    # data = inv(G[surv]) * U[surv];  U[w] = G[w] * data
    A = G[surv]
    rows = np.stack([U[i][layers] for i in surv])  # (kb, nl, sub)
    sh = rows.shape
    data = NP.gf_solve(A, rows.reshape(kb, -1))
    for w in want_nodes:
        acc = np.zeros(data.shape[1], dtype=np.uint8)
        for j in range(kb):
            if G[w, j]:
                acc ^= _mul(int(G[w, j]), data[j])
        U[w][layers] = acc.reshape(sh[1:])
    assert m == P.shape[0]


def encode(k: int, m: int, P: np.ndarray, data: np.ndarray) -> np.ndarray:
    """data (k, L) -> parity (m, L), L a multiple of alpha"""
    q, t, n, s, alpha = params(k, m)
    kb = k + s
    L = data.shape[1]
    sub = L // alpha
    C = np.zeros((n, alpha, sub), dtype=np.uint8)
    C[:k] = data.reshape(k, alpha, sub)
    U = C.copy()
    for a in range(kb):  # 1. uncouple data and virtual nodes (pairs stay inside columns y < t-1)
        mask, b, zp = _partner(a, q, alpha)
        U[a][mask] = _mul(INV_DET, C[a][mask] ^ _mul(GAMMA, C[b[mask], zp[mask]]))
    for p in range(m):  # 2. parity U layer by layer
        acc = np.zeros((alpha, sub), dtype=np.uint8)
        for j in range(kb):
            acc ^= _mul(int(P[p, j]), U[j])
        U[kb + p] = acc
    for a in range(kb, n):  # 3. couple the parity column
        mask, b, zp = _partner(a, q, alpha)
        C[a] = U[a]
        C[a][mask] = U[a][mask] ^ _mul(GAMMA, U[b[mask], zp[mask]])
    return C[kb:].reshape(m, L)


def decode(k: int, m: int, P: np.ndarray, shards: np.ndarray, present) -> np.ndarray:
    """shards (k+m, L) with any e <= m absent shards (their bytes are ignored) -> all k+m shards"""
    q, t, n, s, alpha = params(k, m)
    kb = k + s
    L = shards.shape[1]
    sub = L // alpha
    E = [node_of_shard(k, m, i) for i in range(k + m) if not present[i]]
    if len(E) > m:
        raise ValueError("more than m absent shards")
    C = np.zeros((n, alpha, sub), dtype=np.uint8)
    for i in range(k + m):
        if present[i]:
            C[node_of_shard(k, m, i)] = shards[i].reshape(alpha, sub)
    Eset = set(E)
    U = np.zeros_like(C)
    known = np.zeros((n, alpha), dtype=bool)  # U computed
    z_all = np.arange(alpha)
    score = sum((digit(z_all, e // q, q) == e % q).astype(int) for e in E) if E else np.zeros(alpha, int)
    present_nodes = [a for a in range(n) if a not in Eset]
    for sc in range(int(score.max()) + 1):
        lay = score == sc
        for a in present_nodes:
            mask, b, zp = _partner(a, q, alpha)
            sel0 = lay & ~mask
            U[a][sel0] = C[a][sel0]
            for bb in set(b[lay & mask].tolist()):
                sel = lay & mask & (b == bb)
                if bb in Eset:
                    assert known[bb, zp[sel]].all()  # decoded in a layer of lower score
                    U[a][sel] = C[a][sel] ^ _mul(GAMMA, U[bb][zp[sel]])
                else:
                    U[a][sel] = _mul(INV_DET, C[a][sel] ^ _mul(GAMMA, C[bb][zp[sel]]))
            known[a, lay] = True
        if E:
            _base_solve(P, kb, present_nodes, E, U, lay)
            known[E, :] |= lay
    out = shards.copy()
    for e in E:
        mask, b, zp = _partner(e, q, alpha)
        Ce = U[e].copy()
        Ce[mask] = U[e][mask] ^ _mul(GAMMA, U[b[mask], zp[mask]])
        i = e if e < k else e - s
        out[i] = Ce.reshape(L)
    return out


def repair_layers(k: int, m: int, f: int):
    """the layers R = {z : z_{y0} = x0} a helper sends to rebuild shard f"""
    q, t, n, s, alpha = params(k, m)
    a = node_of_shard(k, m, f)
    z = np.arange(alpha)
    return z[digit(z, a // q, q) == a % q]


def repair_runs(k: int, m: int, f: int, L: int):
    """(offset, length) byte runs of every helper shard in R: q^y0 consecutive layers, one run every q^(y0+1)"""
    q, t, n, s, alpha = params(k, m)
    a = node_of_shard(k, m, f)
    x0, y0 = a % q, a // q
    sub = L // alpha
    run = q ** y0
    return [((b * q * run + x0 * run) * sub, run * sub) for b in range(alpha // (q * run))]


def repair(k: int, m: int, P: np.ndarray, f: int, runs: dict, L: int) -> np.ndarray:
    """rebuild shard f from `runs`: {(helper shard, layer z): sub bytes} for every other shard and every z in R"""
    q, t, n, s, alpha = params(k, m)
    kb = k + s
    sub = L // alpha
    fa = node_of_shard(k, m, f)
    x0, y0 = fa % q, fa // q
    R = repair_layers(k, m, f)
    Rset = set(R.tolist())
    C = {}
    for i in range(k + m):
        if i == f:
            continue
        a = node_of_shard(k, m, i)
        for z in R:
            C[(a, int(z))] = np.frombuffer(bytes(runs[(i, int(z))]), dtype=np.uint8)
    zero = np.zeros(sub, dtype=np.uint8)
    for a in range(k, kb):
        for z in R:
            C[(a, int(z))] = zero
    G = np.concatenate([np.eye(kb, dtype=np.uint8), P], axis=0)
    col = [x + y0 * q for x in range(q)]
    others = [a for a in range(n) if a // q != y0]
    A = G[others]
    out = np.zeros((alpha, sub), dtype=np.uint8)
    for z in R:
        z = int(z)
        U = {}
        for a in others:  # uncouple every node outside column y0: its partner lies in R
            x, y = a % q, a // q
            zy = int(digit(z, y, q))
            if zy == x:
                U[a] = C[(a, z)]
            else:
                b, zp = zy + y * q, z + (x - zy) * q ** y
                assert zp in Rset
                U[a] = _mul(INV_DET, C[(a, z)] ^ _mul(GAMMA, C[(b, zp)]))
        data = NP.gf_solve(A, np.stack([U[a] for a in others]))
        Ucol = {}
        for a in col:
            acc = np.zeros(sub, dtype=np.uint8)
            for j in range(kb):
                if G[a, j]:
                    acc ^= _mul(int(G[a, j]), data[j])
            Ucol[a] = acc
        out[z] = Ucol[fa]
        for x in range(q):
            if x == x0:
                continue
            g = x + y0 * q
            zx = z + (x - x0) * q ** y0  # the layer with digit y0 = x
            Uf = _mul(INV_GAMMA, C[(g, z)] ^ Ucol[g])
            out[zx] = Uf ^ _mul(GAMMA, Ucol[g])
    return out.reshape(L)


def repair_from_shards(k: int, m: int, P: np.ndarray, shards: np.ndarray, f: int) -> np.ndarray:
    """repair() fed with exactly the runs of the other shards"""
    alpha = params(k, m)[4]
    L = shards.shape[1]
    sub = L // alpha
    runs = {(i, int(z)): shards[i, z * sub:(z + 1) * sub].tobytes()
            for i in range(k + m) if i != f for z in repair_layers(k, m, f)}
    return repair(k, m, P, f, runs, L)


# ---- linear algebra checks --------------------------------------------------------------------------------------
def generator(k: int, m: int, P: np.ndarray) -> np.ndarray:
    """((k+m)*alpha) x (k*alpha) matrix over symbols: row i*alpha + z = layer z of shard i"""
    alpha = params(k, m)[4]
    cols = []
    for c in range(k * alpha):
        d = np.zeros(k * alpha, dtype=np.uint8)
        d[c] = 1
        data = d.reshape(k, alpha)
        par = encode(k, m, P, data)
        cols.append(np.concatenate([data, par]).reshape(-1))
    return np.stack(cols, axis=1)


def rank(M: np.ndarray) -> int:
    A = np.array(M, dtype=np.uint8)
    r = 0
    rows, cols = A.shape
    for c in range(cols):
        piv = next((i for i in range(r, rows) if A[i, c]), None)
        if piv is None:
            continue
        A[[r, piv]] = A[[piv, r]]
        A[r] = MUL[NP.gf_inv_scalar(int(A[r, c])), A[r]]
        nz = np.nonzero(A[:, c])[0]
        for i in nz:
            if i != r:
                A[i] ^= MUL[int(A[i, c]), A[r]]
        r += 1
        if r == rows:
            break
    return r


def mds_every_k_subset(k: int, m: int, P: np.ndarray) -> bool:
    alpha = params(k, m)[4]
    G = generator(k, m, P)
    for sub in itertools.combinations(range(k + m), k):
        rows = np.concatenate([G[i * alpha:(i + 1) * alpha] for i in sub])
        if rank(rows) != k * alpha:
            return False
    return True


def repair_by_rank(k: int, m: int, P: np.ndarray, f: int) -> bool:
    """the helpers' rows of the layers R span every row of shard f"""
    alpha = params(k, m)[4]
    G = generator(k, m, P)
    R = repair_layers(k, m, f)
    helpers = np.stack([G[i * alpha + int(z)] for i in range(k + m) if i != f for z in R])
    r0 = rank(helpers)
    return rank(np.concatenate([helpers, G[f * alpha:(f + 1) * alpha]])) == r0
