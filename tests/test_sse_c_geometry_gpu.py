"""SSE-C seal, open and ranged open (DESIGN.md 2.6, 2.7, 4.9, 4.10) at every code geometry.

Expected values never come from the library: sealed blocks B from the scalar C oracle (tests/sse_c_oracle.py, pinned
by FIPS-197, McGrew-Viega and tests/golden/sse_c_kat.json), data shards from B framed by the code's shard length,
parity from the C oracle (RS) and the numpy models (LRC, PB, Clay; all stripes of a batch encoded as one wide stripe,
as in test_encode_geometry_gpu), content hashes and shard tags from hashlib / zlib, plaintext from the plaintext.

The geometry is where the chunk kernel does different things: L = code_shard_len(len(B)) below 8 and 16 (the nonce
prefix and one tag span several data shards), k = 1 (B is one shard), PB and Clay quanta that leave whole trailing
data shards as padding, chunk boundaries at every residue mod 16 inside a data shard, and chunk indices past 255 and
1023, where the counter word LE32(c | last << 31) uses its second byte.  Every seal and open batch has more
(block, chunk) items than the chunk kernel has warps; one ranged batch per family has more requests than the
range_pack / range_join grid has CTAs for its doubled decode batch.  The six HOST forms keep the ownership contract
of the other HOST calls under injected faults."""
import collections
import hashlib
import os
import sys
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import clay_oracle as CO  # noqa: E402
import lrc_oracle as LO  # noqa: E402
import oracle_lib as O  # noqa: E402
import pb_oracle as PB  # noqa: E402
import sse_c_oracle as SO  # noqa: E402
from test_blake2 import adler8_ref  # noqa: E402  the zlib model of the adler8 tag

import garage_b200 as G  # noqa: E402

CH, FR, PFX = 4096, 4112, 8   # plaintext chunk, sealed chunk, nonce prefix
POISON, SENT, GONE = 0xA5, 0x5A, 0x5C  # shards before a seal, outputs before an open, absent shards
PLEN_SENT = 0xA5A5A5A5  # plain_len before an open: a block that fails leaves it alone
MiB = 1 << 20
H100_SMS = 132
CHUNK_WARPS_PER_SM = 4 * 8  # the chunk kernel: min(items / 8, 4 x SMs) CTAs of 8 warps
RANGE_CTAS_PER_SM = 8       # range_pack / range_join: min(2n, 8 x SMs) CTAs for n ranged requests

RS_CASES = [("rs", k, 1 + (3 * k) % 8) for k in range(1, 33)]
PB_CASES = [("pb", k, m) for k in (1, 2, 5, 10, 16) for m in (2, 3, 4)]
LRC_CASES = [("lrc", 4, 2, 1), ("lrc", 12, 3, 2), ("lrc", 24, 6, 2), ("lrc", 32, 4, 4)]
CLAY_CASES = [("clay", k, m) for k, m in [(2, 2), (5, 2), (14, 2), (4, 3), (6, 3), (10, 4), (12, 4)]]
CASES = RS_CASES + PB_CASES + LRC_CASES + CLAY_CASES
BIG = {("rs", 32, 1), ("pb", 16, 4), ("lrc", 32, 4, 4), ("clay", 14, 2)}  # one 4 MiB + 13 block per family
GRAPH = {("rs", 32, 1), ("lrc", 24, 6, 2)}                                 # k >= 17: CUDA-graph replays
UNKEYED = {("rs", 1, 4), ("rs", 32, 1), ("pb", 1, 2), ("lrc", 24, 6, 2), ("clay", 14, 2)}
RANGE_CASES = [("rs", 32, 1), ("rs", 3, 2), ("pb", 16, 4), ("pb", 2, 3), ("lrc", 32, 4, 4), ("clay", 14, 2),
               ("clay", 4, 3)]

FIXED = [0, 1, 15, 16, 17, 4095, 4096, 4097, 8192]
LONG = [MiB - 977, MiB, MiB + 4097]  # MiB + 4097: chunks 256 and 257
BIG_LEN = 4 * MiB + 13               # chunks up to 1024
FILL = MiB + 4097                    # more blocks of it until a batch outruns the chunk kernel's warps
RANGE_SHORT = [40000, 65536 - 7]     # short blocks of the many-request ranged batch, with the FIXED ones
N_RANGE_SHORT = 1100                 # > 8 x 132: the doubled decode batch outruns range_pack / range_join


def case_id(c):
    return "-".join(map(str, c))


def r16(x):
    return (x + 15) // 16 * 16


def sealed_len(P):
    return PFX + P + 16 * max(1, -(-P // CH))


def chunks(P):
    return max(1, -(-P // CH))


class Code:
    """one case: the context it makes, its shard length model and its parity model"""

    def __init__(self, case):
        self.case = case
        self.fam, self.k = case[0], case[1]
        if self.fam == "lrc":
            self.l, self.r = case[2], case[3]
            self.m = self.l + self.r
        else:
            self.m = case[2]
        self.tot = self.k + self.m
        self.alpha = CO.params(self.k, self.m)[4] if self.fam == "clay" else 1
        self.q = {"rs": 1, "lrc": 1, "pb": 128, "clay": 16 * self.alpha}[self.fam]

    def ctx(self):
        if self.fam == "rs":
            return G.GarageEc(0, self.k, self.m)
        if self.fam == "lrc":
            return G.GarageEc.lrc(0, self.k, self.l, self.r)
        if self.fam == "pb":
            return G.GarageEc.piggyback(0, self.k, self.m)
        return G.GarageEc.clay(0, self.k, self.m)

    def shard_len(self, blen):
        L = -(-blen // self.k)
        return -(-L // self.q) * self.q

    def parity(self, datas):
        """parity (m, L) of every stripe's data shards (k, L): the stripes of a batch as one wide stripe"""
        k, m = self.k, self.m
        Ls = [d.shape[1] for d in datas]
        if self.fam in ("rs", "lrc"):
            cols = np.cumsum([0] + Ls)
            W = r16(int(cols[-1])) + 64
            wide = np.zeros((k, W), dtype=np.uint8)
            wide[:, :cols[-1]] = np.concatenate(datas, axis=1)
            if self.fam == "rs":
                par = O.encode(k, m, O.build_matrix(k, m, 0), wide.reshape(-1), W, 1, simd=True).reshape(m, W)
            else:
                par = LO.encode(LO.build_lrc(k, self.l, self.r), wide)
            return [par[:, cols[i]:cols[i + 1]] for i in range(len(datas))]
        if self.fam == "pb":
            hs = [L // 2 for L in Ls]
            a = np.concatenate([d[:, :h] for d, h in zip(datas, hs)], axis=1)
            b = np.concatenate([d[:, h:] for d, h in zip(datas, hs)], axis=1)
            par = PB.encode(PB.build(k, m), np.concatenate([a, b], axis=1))
            H, cols = a.shape[1], np.cumsum([0] + hs)
            return [np.concatenate([par[:, cols[i]:cols[i + 1]], par[:, H + cols[i]:H + cols[i + 1]]], axis=1)
                    for i in range(len(datas))]
        A = self.alpha
        wide = np.concatenate([d.reshape(k, A, -1) for d in datas], axis=2)
        par = CO.encode(k, m, CO.build(k, m), wide.reshape(k, -1)).reshape(m, A, -1)
        cols = np.cumsum([0] + [L // A for L in Ls])
        return [np.ascontiguousarray(par[:, :, cols[i]:cols[i + 1]]).reshape(m, -1) for i in range(len(datas))]


# ---------------------------------------------------------------------------------------------- case table
def small_l_lens(code):
    """plaintext lengths that give L = 7 and L = 15 (RS and LRC: B = P + 24 bytes for P <= 4096)"""
    if code.q != 1:
        return []
    return [Lt * code.k - 24 for Lt in (7, 15) if Lt * code.k >= 24]


def boundary_residues(code, P):
    """offsets mod 16 of B's chunk starts that fall inside a data shard (not at its first byte)"""
    L = code.shard_len(sealed_len(P))
    out = set()
    for c in range(chunks(P)):
        j, off = divmod(PFX + FR * c, L)
        if j < code.k and off:
            out.add(off % 16)
    return out


def residue_lens(code):
    """two-chunk lengths whose chunk boundaries fall at every residue mod 16 inside a data shard: RS and LRC with
    k >= 2 (with a quantum of 16 or more, or one shard, every boundary is 8 past a 16-byte boundary)"""
    if code.q != 1 or code.k < 2:
        return []
    got, out, P = set(), [], CH + 1
    while len(got) < 16:
        new = boundary_residues(code, P) - got
        if new:
            out.append(P)
            got |= new
        P += 1
    return out


def short_lens(code):
    """(plaintext length, key variant) of a case's short blocks; variant 1: all-0x00 key and nonce, 2: all-0xFF"""
    out = [(P, 0) for P in FIXED + small_l_lens(code) + residue_lens(code)]
    out[FIXED.index(4096)] = (4096, 1)
    out[FIXED.index(4097)] = (4097, 2)
    return out


def case_blocks(code, sms=H100_SMS):
    """the seal batch of a case: short blocks, the long ones, the family's 4 MiB block, then FILL blocks until the
    batch has more chunks than the chunk kernel has warps (with room for the blocks an open fails)"""
    out = short_lens(code) + [(LONG[0], 0), (LONG[1], 1), (LONG[2], 2)]
    if code.case in BIG:
        out.append((BIG_LEN, 0))
    v = 3
    while sum(chunks(P) for P, _ in out) <= sms * CHUNK_WARPS_PER_SM + 600:
        out.append((FILL, v))
        v += 1
    return out


def range_short_blocks(code):
    return short_lens(code)[:len(FIXED) + 2] + [(P, 0) for P in RANGE_SHORT]


def test_case_table_reaches_every_geometry():
    """RS: every k in 1..32 with m 1..8; L < 8 and L < 16 wherever the code allows them, chunk boundaries at every
    residue mod 16 inside a shard, blocks whose last data shards are all padding (PB, Clay with alpha = 256 too),
    chunk indices >= 256 in every case and >= 1024 in every family; every batch outruns the chunk kernel's warps and
    one ranged batch per family outruns the range_pack / range_join grid"""
    codes = [Code(c) for c in CASES]
    rs = [c for c in codes if c.fam == "rs"]
    assert {c.k for c in rs} == set(range(1, 33)) and {c.m for c in rs} == set(range(1, 9))
    assert {(c.k, c.m) for c in codes if c.fam == "pb"} == {(k, m) for k in (1, 2, 5, 10, 16) for m in (2, 3, 4)}
    assert 256 in {c.alpha for c in codes if c.fam == "clay"}
    reached = collections.Counter()
    for code in codes:
        Ps = [P for P, _ in case_blocks(code)]
        Ls = [code.shard_len(sealed_len(P)) for P in Ps]
        assert sum(chunks(P) for P in Ps) > H100_SMS * CHUNK_WARPS_PER_SM + 300, code.case
        assert max(chunks(P) for P in Ps) - 1 >= 257, code.case
        if code.q == 1 and code.k >= 4:
            assert any(L < 8 for L in Ls) and any(8 <= L < 16 for L in Ls), code.case
        if code.q == 1 and code.k >= 2:
            assert set().union(*[boundary_residues(code, P) for P in Ps]) == set(range(16)), code.case
        pad = [P for P, L in zip(Ps, Ls) if code.k >= 2 and sealed_len(P) <= (code.k - 1) * L]
        if code.k >= 2 and code.q > 1:  # PB and Clay: whole trailing data shards of short blocks are padding
            assert pad, code.case
        reached["L<8"] += any(L < 8 for L in Ls)
        reached["L<16"] += any(L < 16 for L in Ls)
        reached["pad-%s" % code.fam] += bool(pad)
        reached["clay256-pad"] += code.alpha == 256 and bool(pad)
        reached["chunk1024-%s" % code.fam] += max(chunks(P) for P in Ps) - 1 >= 1024
    for what in ("L<8", "L<16", "pad-rs", "pad-lrc", "pad-pb", "pad-clay", "clay256-pad", "chunk1024-rs",
                 "chunk1024-lrc", "chunk1024-pb", "chunk1024-clay"):
        assert reached[what], what
    for fam in ("rs", "lrc", "pb", "clay"):
        assert any(c[0] == fam for c in RANGE_CASES) and any(c[0] == fam for c in BIG & set(RANGE_CASES))
    assert 2 * N_RANGE_SHORT > 2 * RANGE_CTAS_PER_SM * H100_SMS
    assert all(c in CASES for c in BIG | GRAPH | UNKEYED | set(RANGE_CASES))
    assert all(c[1] >= 17 for c in GRAPH)
    # the table's shard length model is the library's (gf256.h code_shard_len), spot-checked against the models
    for code in codes:
        for P in (0, 4097, MiB):
            S = sealed_len(P)
            assert S == SO.sealed_len(P)
            if code.fam == "pb":
                assert code.shard_len(S) == PB.shard_len(S, code.k)
            if code.fam == "clay":
                assert code.shard_len(S) == CO.shard_len(S, code.k, code.m)


# ---------------------------------------------------------------------------------------------- sealed blocks
Sealed = collections.namedtuple("Sealed", "pt key nonce B")


class Pool:
    """oracle-sealed blocks by (plaintext length, key variant), each sealed once and shared by every case"""

    def __init__(self):
        self.cache = {}

    @staticmethod
    def _make(P, var):
        rng = np.random.default_rng([P, var, 0x55EC])
        pt = rng.integers(0, 256, P, dtype=np.uint8)
        if var in (1, 2):
            key = np.full(32, 0 if var == 1 else 0xFF, dtype=np.uint8)
            nonce = np.full(8, 0 if var == 1 else 0xFF, dtype=np.uint8)
        else:
            key, nonce = rng.integers(0, 256, 32, dtype=np.uint8), rng.integers(0, 256, 8, dtype=np.uint8)
        B = np.frombuffer(SO.seal(key.tobytes(), nonce.tobytes(), pt.tobytes()), dtype=np.uint8)
        return Sealed(pt, key, nonce, B)

    def get(self, items):
        todo = [x for x in dict.fromkeys(items) if x not in self.cache]
        if todo:  # the oracle is scalar: seal in parallel (ctypes releases the GIL), built once before the threads
            SO.lib()
            with ThreadPoolExecutor(os.cpu_count() or 4) as ex:
                for x, s in zip(todo, ex.map(lambda t: self._make(*t), todo)):
                    self.cache[x] = s
        return [self.cache[x] for x in items]


@pytest.fixture(scope="module")
def pool():
    return Pool()


@pytest.fixture(scope="module")
def torch():
    import torch as t

    assert t.cuda.is_available()
    return t


@pytest.fixture(scope="module")
def sms(torch):
    return torch.cuda.get_device_properties(0).multi_processor_count


def dev(torch, a):
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.int32) if a.dtype == np.uint32 else a).cuda()


def blake2(b):
    return hashlib.blake2b(bytes(b)).digest()[:32]


def expected_shards(code, Bs, stride):
    """what a seal leaves in POISON-filled shards: B framed into k shards of L bytes, the model's parity, zeros over
    [L, roundup16(L)) and POISON past it"""
    k = code.k
    Ls = [code.shard_len(b.size) for b in Bs]
    datas = []
    for b, L in zip(Bs, Ls):
        d = np.zeros(k * L, dtype=np.uint8)
        d[:b.size] = b
        datas.append(d.reshape(k, L))
    pars = code.parity(datas)
    want = np.full((len(Bs), code.tot, stride), POISON, dtype=np.uint8)
    for s, L in enumerate(Ls):
        want[s, :k, :L] = datas[s]
        want[s, k:, :L] = pars[s]
        want[s, :, L:r16(L)] = 0
    return want, Ls


def expected_tags(want, Ls, kind):
    n, tot = want.shape[:2]
    out = np.zeros((n, tot, 32), dtype=np.uint8)
    for s, L in enumerate(Ls):
        for i in range(tot):
            body = want[s, i, :L].tobytes()
            out[s, i] = np.frombuffer(blake2(body) if kind == G.SUM_BLAKE2 else adler8_ref(body), dtype=np.uint8)
    return out


def same(got, want, what):
    got = np.asarray(got).reshape(want.shape)
    if not np.array_equal(got, want):
        bad = np.argwhere(got != want)
        at = tuple(int(x) for x in bad[0])
        pytest.fail("%s: %d bytes differ, first at %s: %#x, want %#x" % (what, len(bad), at, got[at], want[at]))


def plain_rows(pts, pitch):
    rows = np.zeros((len(pts), pitch), dtype=np.uint8)
    for s, p in enumerate(pts):
        rows[s, :p.size] = p
    return rows


def present(tot, lost):
    p = np.ones(tot, dtype=np.uint8)
    p[list(lost)] = 0
    return p


def recoverable(code, ec, pr):
    lost = code.tot - int(pr.sum())
    if lost > code.m:
        return False
    if code.fam != "lrc":  # MDS: every set of m losses decodes
        return True
    return lost == 0 or ec.read_set(pr, np.arange(code.tot) < code.k) is not None


def patterns(code, ec, seed):
    """healthy, every single data shard, seeded m-sets (LRC: only those its read_set decodes; every m-set of an MDS
    code is kept)"""
    rng = np.random.default_rng(seed)
    pats = [present(code.tot, ())] + [present(code.tot, (j,)) for j in range(code.k)]
    for _ in range(6):
        pr = present(code.tot, rng.choice(code.tot, code.m, replace=False))
        if recoverable(code, ec, pr):
            pats.append(pr)
    return pats


# ---------------------------------------------------------------------------------------------- seal and open
def seal_checks(torch, code, ec, sb, stride, pitch, graph):
    n, tot = len(sb), code.tot
    pts = [x.pt for x in sb]
    keys, nonces = np.stack([x.key for x in sb]), np.stack([x.nonce for x in sb])
    Bs = [x.B for x in sb]
    want, Ls = expected_shards(code, Bs, stride)
    assert [ec.code_shard_len(b.size) for b in Bs] == Ls
    hashes = np.stack([np.frombuffer(blake2(b), dtype=np.uint8) for b in Bs])
    tags = expected_tags(want, Ls, G.SUM_BLAKE2)
    plen = np.array([p.size for p in pts], dtype=np.uint32)
    rows = plain_rows(pts, pitch)

    # DEVICE into poisoned shards, BLAKE2 shard tags
    d_rows, d_len, d_keys, d_nonces = dev(torch, rows), dev(torch, plen), dev(torch, keys), dev(torch, nonces)
    d_sh = torch.full((n * tot * stride,), POISON, dtype=torch.uint8, device="cuda")
    d_hash = torch.zeros(n * 32, dtype=torch.uint8, device="cuda")
    d_sums = torch.zeros(n * tot * 32, dtype=torch.uint8, device="cuda")
    ec.seal(d_rows, pitch, d_len, d_keys, d_nonces, d_sh, stride, d_hash, d_sums, n=n)
    torch.cuda.synchronize()
    same(d_sh.cpu().numpy(), want, "DEVICE seal shards")
    same(d_hash.cpu().numpy(), hashes, "DEVICE seal content hash")
    same(d_sums.cpu().numpy(), tags, "DEVICE seal BLAKE2 shard tags")

    if graph:
        d_sh.fill_(POISON)
        d_hash.zero_()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            ec.seal(d_rows, pitch, d_len, d_keys, d_nonces, d_sh, stride, d_hash, n=n)  # warm the pool
        torch.cuda.synchronize()
        d_sh.fill_(POISON)
        d_hash.zero_()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            ec.seal(d_rows, pitch, d_len, d_keys, d_nonces, d_sh, stride, d_hash, n=n)
        g.replay()
        torch.cuda.synchronize()
        same(d_sh.cpu().numpy(), want, "graph seal shards")
        same(d_hash.cpu().numpy(), hashes, "graph seal content hash")
    del d_sh, d_rows

    # HOST contiguous: nothing past roundup16(L) of a shard comes down
    h_sh = np.full(n * tot * stride, POISON, dtype=np.uint8)
    h_hash = np.zeros(n * 32, dtype=np.uint8)
    ec.seal(rows, pitch, plen, keys, nonces, h_sh, stride, h_hash)
    same(h_sh, want, "HOST seal shards")
    same(h_hash, hashes, "HOST seal content hash")

    # HOST seal_blocks, adler8 shard tags
    h_sh[:] = POISON
    h_sums = np.zeros(n * tot * 32, dtype=np.uint8)
    ec.set_sum_kind(G.SUM_ADLER8)
    try:
        ec.seal_blocks(pts, keys, nonces, h_sh, stride, h_hash, h_sums)
    finally:
        ec.set_sum_kind(G.SUM_BLAKE2)
    same(h_sh, want, "seal_blocks shards")
    same(h_hash, hashes, "seal_blocks content hash")
    same(h_sums, expected_tags(want, Ls, G.SUM_ADLER8), "seal_blocks adler8 shard tags")
    return want, Ls, hashes, keys


def unkeyed_checks(torch, code, ec, pts, stride, pitch):
    """B = P: the plaintext framed as it is"""
    n, tot = len(pts), code.tot
    want, Ls = expected_shards(code, pts, stride)
    hashes = np.stack([np.frombuffer(blake2(p), dtype=np.uint8) for p in pts])
    h_sh = np.full(n * tot * stride, POISON, dtype=np.uint8)
    h_hash = np.zeros(n * 32, dtype=np.uint8)
    h_sums = np.zeros(n * tot * 32, dtype=np.uint8)
    ec.seal_blocks(pts, None, None, h_sh, stride, h_hash, h_sums)
    same(h_sh, want, "unkeyed seal_blocks shards")
    same(h_hash, hashes, "unkeyed seal_blocks content hash")
    same(h_sums, expected_tags(want, Ls, G.SUM_BLAKE2), "unkeyed seal_blocks shard tags")
    plen = np.array([p.size for p in pts], dtype=np.uint32)
    d_sh = torch.full((n * tot * stride,), POISON, dtype=torch.uint8, device="cuda")
    d_hash = torch.zeros(n * 32, dtype=torch.uint8, device="cuda")
    ec.seal(dev(torch, plain_rows(pts, pitch)), pitch, dev(torch, plen), None, None, d_sh, stride, d_hash, n=n)
    torch.cuda.synchronize()
    same(d_sh.cpu().numpy(), want, "unkeyed DEVICE seal shards")
    same(d_hash.cpu().numpy(), hashes, "unkeyed DEVICE seal content hash")


def open_batch(code, ec, items, sb, want, Ls, hashes):
    """(block, present, flipped B position) per open: every block under a pattern, the patterns the blocks did not
    reach on short blocks, shard 0 of a long block and every shard holding a prefix byte absent, m + 1 losses on two
    short blocks, and tampering only these geometries allow"""
    k, tot, m = code.k, code.tot, code.m
    pats = patterns(code, ec, len(items) + k)
    n = len(items)
    short = [s for s, (P, _) in enumerate(items) if P < MiB]
    opens = [(s, pats[s % len(pats)], None) for s in range(n)]
    opens += [(short[i % len(short)], pats[i], None) for i in range(n, len(pats))]
    opens.append((items.index((MiB, 1)), present(tot, (0,)), None))
    seen = set()
    for s in short:
        if Ls[s] < 8 and Ls[s] not in seen:
            seen.add(Ls[s])
            opens += [(s, present(tot, (j,)), None) for j in range(-(-PFX // Ls[s]))]
    opens.append((items.index((4097, 2)), present(tot, range(m + 1)), None))
    opens.append((items.index((8192, 0)), present(tot, range(k - 1, k + m)), None))
    healthy = present(tot, ())
    for P in small_l_lens(code):
        s = items.index((P, 0))
        S, L = sb[s].B.size, Ls[s]
        tag0 = S - 16  # the one chunk's tag, B[S - 16, S): it spans 16 / L + 1 or more data shards
        opens.append((s, healthy, tag0 + L - tag0 % L))  # its first byte in the tag's second data shard
        if L < PFX:
            opens.append((s, healthy, L))  # a nonce byte held by data shard 1
            opens.append((s, healthy, S - 1))
    return opens


def open_checks(torch, code, ec, items, sb, want, Ls, hashes, keys, stride, pitch, sms, graph):
    n, k, tot = len(items), code.k, code.tot
    opens = open_batch(code, ec, items, sb, want, Ls, hashes)
    no = len(opens)
    sh = np.empty((no, tot, stride), dtype=np.uint8)
    pres = np.stack([p for _, p, _ in opens])
    sl = np.array([sb[s].B.size for s, _, _ in opens], dtype=np.uint32)
    hs = np.empty((no, 32), dtype=np.uint8)
    exp = np.zeros(no, dtype=np.int32)
    for i, (s, pr, flip) in enumerate(opens):
        sh[i] = want[s]
        sh[i][pr == 0] = GONE
        hs[i] = hashes[s]
        if flip is not None:
            L = Ls[s]
            sh[i, flip // L, flip % L] ^= 0x40
            B = sb[s].B.copy()
            B[flip] ^= 0x40
            hs[i] = np.frombuffer(blake2(B), dtype=np.uint8)  # only a tag can fail
            exp[i] = G.E_AUTH
        elif not recoverable(code, ec, pr):
            assert tot - pr.sum() > code.m
            exp[i] = G.E_UNRECOVERABLE
    assert (exp == G.E_UNRECOVERABLE).sum() == 2 and ((exp == G.E_AUTH).sum() > 0) == bool(small_l_lens(code))
    ok_chunks = sum(chunks(sb[s].pt.size) for i, (s, _, _) in enumerate(opens) if exp[i] == 0)
    assert ok_chunks > sms * CHUNK_WARPS_PER_SM
    okeys = np.stack([keys[s] for s, _, _ in opens])
    pts = [sb[s].pt for s, _, _ in opens]

    def check(what, status, plen, bad, row_of, zero_tail):
        assert list(status) == list(exp), "%s: status %s" % (what, [(i, int(a), int(b)) for i, (a, b) in
                                                                    enumerate(zip(status, exp)) if a != b][:8])
        for i in range(no):
            P, row = pts[i].size, row_of(i)
            if exp[i] == 0:
                assert bad[i] == 0 and plen[i] == P, (what, i, int(bad[i]), int(plen[i]), P)
                if not np.array_equal(row[:P], pts[i]):
                    x = int(np.argmax(row[:P] != pts[i]))
                    pytest.fail("%s: open %d (block %d, P %d) differs from byte %d" % (what, i, opens[i][0], P, x))
                tail = r16(P) if zero_tail else P
                assert not row[P:tail].any() and (row[tail:] == SENT).all(), (what, i, P)
            else:
                assert (row == SENT).all(), (what, "a failed block's plaintext was written", i)
                assert plen[i] == PLEN_SENT, (what, i)
                if exp[i] == G.E_AUTH:
                    assert bad[i] == 0, (what, i)

    # DEVICE: zero up to roundup16(P), nothing past it
    d_sh, d_pr, d_sl, d_hs, d_keys = (dev(torch, a) for a in (sh, pres, sl, hs, okeys))

    def run_device():
        d_plain = torch.full((no * pitch,), SENT, dtype=torch.uint8, device="cuda")
        d_plen = torch.full((no,), PLEN_SENT - (1 << 32), dtype=torch.int32, device="cuda")
        d_bad = torch.full((no,), 0x77, dtype=torch.uint8, device="cuda")
        d_st = torch.full((no,), 99, dtype=torch.int32, device="cuda")
        return d_plain, d_plen, d_bad, d_st

    outs = run_device()
    ec.open(d_sh, d_pr, d_sl, d_hs, d_keys, outs[0], pitch, outs[1], outs[2], outs[3], stride, n=no)
    torch.cuda.synchronize()
    dp = outs[0].cpu().numpy().reshape(no, pitch)
    check("DEVICE open", outs[3].cpu().numpy(), outs[1].cpu().numpy().view(np.uint32), outs[2].cpu().numpy(),
          lambda i: dp[i], True)
    del dp
    if graph:
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            ec.open(d_sh, d_pr, d_sl, d_hs, d_keys, outs[0], pitch, outs[1], outs[2], outs[3], stride, n=no)
        torch.cuda.synchronize()
        outs = run_device()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            ec.open(d_sh, d_pr, d_sl, d_hs, d_keys, outs[0], pitch, outs[1], outs[2], outs[3], stride, n=no)
        d_sh.copy_(dev(torch, sh))  # the opens so far rebuilt the absent shards in place
        g.replay()
        torch.cuda.synchronize()
        dp = outs[0].cpu().numpy().reshape(no, pitch)
        check("graph open", outs[3].cpu().numpy(), outs[1].cpu().numpy().view(np.uint32), outs[2].cpu().numpy(),
              lambda i: dp[i], True)
        del dp
    del d_sh, outs

    # HOST contiguous: exactly P bytes of each passing block come down
    h_plain = np.full((no, pitch), SENT, dtype=np.uint8)
    plen = np.full(no, PLEN_SENT, dtype=np.uint32)
    bad = np.full(no, 0x77, dtype=np.uint8)
    st = np.full(no, 99, dtype=np.int32)
    assert ec.open(sh.reshape(-1), pres, sl, hs, okeys, h_plain.reshape(-1), pitch, plen, bad, st,
                   stride) == G.E_UNRECOVERABLE
    check("HOST open", st, plen, bad, lambda i: h_plain[i], False)
    del h_plain

    # HOST gather form
    stripes = [sh[i].reshape(-1) for i in range(no)]
    plains = [np.full(pts[i].size + 32, SENT, dtype=np.uint8) for i in range(no)]
    plen[:] = PLEN_SENT
    bad[:] = 0x77
    st[:] = 99
    assert ec.open_stripes(stripes, pres, sl, hs, okeys, plains, plen, bad, st, stride) == G.E_UNRECOVERABLE
    check("open_stripes", st, plen, bad, lambda i: plains[i], False)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_seal_open_geometry(torch, sms, pool, case):
    """seal (DEVICE into poisoned shards, HOST contiguous, seal_blocks; BLAKE2 and adler8 shard tags) equals B
    framed with the model's parity; open (DEVICE, HOST, open_stripes) of those shards under erasure and tampering
    returns exactly the plaintext of every block that passes and nothing of any other"""
    code = Code(case)
    items = case_blocks(code, sms)
    sb = pool.get(items)
    assert sum(chunks(x.pt.size) for x in sb) > sms * CHUNK_WARPS_PER_SM
    pitch = r16(max(x.pt.size for x in sb))
    stride = r16(max(code.shard_len(x.B.size) for x in sb)) + 32  # poison past roundup16(L) in every shard
    with code.ctx() as ec:
        want, Ls, hashes, keys = seal_checks(torch, code, ec, sb, stride, pitch, case in GRAPH)
        if case in UNKEYED:
            unkeyed_checks(torch, code, ec, [x.pt for x in sb], stride, pitch)
        open_checks(torch, code, ec, items, sb, want, Ls, hashes, keys, stride, pitch, sms, case in GRAPH)


# ---------------------------------------------------------------------------------------------- ranged open
def plain_offset(p, P):
    """the plaintext byte at or just before B position p"""
    c, r = divmod(max(p, PFX) - PFX, FR)
    return min(c * CH + min(r, CH - 1), max(P - 1, 0))


def long_requests(code, P, L):
    """(offset, len, lost shards) over one long block"""
    k = code.k
    r = [(0, CH, ()), (3 * CH, CH, ()), (3 * CH + 100, CH, ()), (5 * CH + 4000, 300, (0,)), (P - 1, 1, ()),
         (0, P, ()), (P, 0, ()), (17, 0, ()), (P - CH - 5, CH + 5, (0,))]
    for c in (255, 256, 257, 1023, 1024, 1025):
        if c * CH + 4200 <= P:
            r += [(c * CH, CH, ()), (c * CH + 7, CH, ()), (c * CH + 4000, 200, (k - 1,))]
        elif c * CH < P:
            r.append((c * CH, P - c * CH, ()))
    for j in sorted({1, k // 2, k - 1}):  # across the edge of data shards j - 1 and j, either one absent
        if 0 < j < k and j * L < PFX + P:
            o = max(0, plain_offset(j * L, P) - 20)
            r += [(o, min(40, P - o), (j,)), (o, min(40, P - o), (j - 1,))]
    return r


def range_batch(code, ec, sb_list, reqs, stride, garbage):
    """per request a stripe holding only its open_range_plan runs, garbage everywhere else"""
    tot = code.tot
    n = len(reqs)
    shards = np.empty((n, tot, stride), dtype=np.uint8)
    pres = np.empty((n, tot), dtype=np.uint8)
    for i, (b, o, ln, lost) in enumerate(reqs):
        pr = present(tot, lost)
        runs, _ = ec.open_range_plan(pr, sb_list[b][0].B.size, o, ln)
        assert runs is not None
        shards[i] = garbage
        stripe = sb_list[b][1]
        for sh_, off, nb in runs:
            assert pr[sh_]
            shards[i, sh_, off:off + nb] = stripe[sh_, off:off + nb]
        pres[i] = pr
    return shards, pres


def range_checks(torch, code, ec, what, sb_list, reqs, stride, seed, graph):
    rng = np.random.default_rng(seed)
    garbage = rng.integers(0, 256, (code.tot, stride), dtype=np.uint8)
    shards, pres = range_batch(code, ec, sb_list, reqs, stride, garbage)
    n = len(reqs)
    sealed = np.array([sb_list[b][0].B.size for b, _, _, _ in reqs], dtype=np.uint32)
    keys = np.stack([sb_list[b][0].key for b, _, _, _ in reqs])
    offs = np.array([o for _, o, _, _ in reqs], dtype=np.uint32)
    lens = np.array([ln for _, _, ln, _ in reqs], dtype=np.uint32)
    out_stride = r16(max(int(lens.max()), 16))
    pt = [sb_list[b][0].pt for b, _, _, _ in reqs]

    def check(form, out, st, zero_tail):
        bad = np.flatnonzero(st != 0)
        assert not len(bad), (form, [(int(i), int(st[i])) for i in bad[:8]])
        for i in range(n):
            o, ln = int(offs[i]), int(lens[i])
            row = out[i]
            if not np.array_equal(row[:ln], pt[i][o:o + ln]):
                x = int(np.argmax(row[:ln] != pt[i][o:o + ln]))
                pytest.fail("%s %s: request %d (offset %d, len %d, lost %s) differs from byte %d" % (
                    what, form, i, o, ln, reqs[i][3], x))
            tail = r16(ln) if zero_tail else ln
            assert not row[ln:tail].any() and (row[tail:] == SENT).all(), (what, form, i)

    d = [dev(torch, a) for a in (shards, pres, sealed, keys, offs, lens)]
    d_out = torch.full((n * out_stride,), SENT, dtype=torch.uint8, device="cuda")
    d_st = torch.full((n,), 99, dtype=torch.int32, device="cuda")
    ec.open_range(*d, stride, d_out, out_stride, d_st)
    torch.cuda.synchronize()
    check("DEVICE", d_out.cpu().numpy().reshape(n, out_stride), d_st.cpu().numpy(), True)
    if graph:
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            ec.open_range(*d, stride, d_out, out_stride, d_st)  # warm the pool
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            ec.open_range(*d, stride, d_out, out_stride, d_st)
        d_out.fill_(SENT)
        d_st.fill_(99)
        g.replay()
        torch.cuda.synchronize()
        check("graph", d_out.cpu().numpy().reshape(n, out_stride), d_st.cpu().numpy(), True)
    del d, d_out

    h_out = np.full((n, out_stride), SENT, dtype=np.uint8)
    st = np.full(n, 99, dtype=np.int32)
    assert ec.open_range(shards.reshape(-1), pres, sealed, keys, offs, lens, stride, h_out.reshape(-1), out_stride,
                         st) == 0
    check("HOST", h_out, st, False)
    del h_out
    outs = [np.full(int(lens[i]) + 32, SENT, dtype=np.uint8) for i in range(n)]
    st[:] = 99
    assert ec.open_range_stripes([shards[i].reshape(-1) for i in range(n)], pres, sealed, keys, offs, lens, stride,
                                 outs, st) == 0
    check("stripes", outs, st, False)
    return n


def sealed_stripes(code, sb, stride):
    want, _ = expected_shards(code, [x.B for x in sb], stride)
    return [(x, want[s]) for s, x in enumerate(sb)]


@pytest.mark.gpu
@pytest.mark.parametrize("case", RANGE_CASES, ids=case_id)
def test_open_range_geometry(torch, sms, pool, case):
    """ranged opens (DEVICE into sentinel rows, HOST, open_range_stripes) of stripes that hold only the planned runs:
    4 KiB ranges on and off chunk boundaries, ranges inside chunks >= 256 and >= 1024, across data-shard edges with
    either shard absent, shard 0 absent, the last byte, whole plaintexts and empty ranges; then a batch of more than
    8 x SMs requests over short blocks (L < 8 and L < 16 among them) under every single loss and m-sets"""
    code = Code(case)
    with code.ctx() as ec:
        longs = [(LONG[2], 2), (BIG_LEN, 0) if case in BIG else (LONG[0], 0)]
        sb = pool.get(longs)
        stride = r16(max(code.shard_len(x.B.size) for x in sb)) + 16
        sbl = sealed_stripes(code, sb, stride)
        reqs = [(b, o, ln, lost) for b, x in enumerate(sb)
                for o, ln, lost in long_requests(code, x.pt.size, code.shard_len(x.B.size))]
        range_checks(torch, code, ec, "long", sbl, reqs, stride, 1, False)
        del sbl

        shorts = range_short_blocks(code)
        sb = pool.get(shorts)
        stride = r16(max(code.shard_len(x.B.size) for x in sb)) + 16
        sbl = sealed_stripes(code, sb, stride)
        pats = [np.flatnonzero(p == 0).tolist() for p in patterns(code, ec, 7)]
        rng = np.random.default_rng(zlib.crc32(case_id(case).encode()))
        reqs = []
        for i in range(N_RANGE_SHORT):
            b = i % len(sb)
            P = sb[b].pt.size
            lost = pats[(i // len(sb)) % len(pats)]
            if i % 13 == 0:
                o, ln = P, 0
            elif i % 11 == 0:
                o, ln = 0, P
            elif i % 7 == 0:
                o, ln = max(P - 1, 0), min(P, 1)
            else:
                o = int(rng.integers(0, P + 1))
                ln = int(rng.integers(0, min(P - o, 9000) + 1))
            reqs.append((b, o, ln, lost))
        n = range_checks(torch, code, ec, "short", sbl, reqs, stride, 2, case in GRAPH)
        assert 2 * n > 2 * RANGE_CTAS_PER_SM * sms


# ---------------------------------------------------------------------------------------------- HOST faults
FAULT_CASE = ("rs", 4, 2)
# (k + m) x stride > 24 MiB: a HOST pipeline chunk (48 MiB of stripe bytes) holds one block, so the five blocks are
# five chunks over the three lanes: chunk 0's retire runs when chunk 3 is issued, chunk 1's when chunk 4 is, and
# drain() retires chunks 2..4
FAULT_STRIDE = (17 << 20) // 4
FAULT_ITEMS = [(65536 + 13, 40), (40000, 41), (4097, 42), (70001, 43), (12345, 44)]
FAULT_TAMPERED = (1, 3)  # blocks with a flipped ciphertext byte in the open forms
FAULT_FORMS = ["seal", "seal_blocks", "open", "open_stripes", "open_range", "open_range_stripes"]


class Buffers:
    """caller buffers of one fault test: pageable numpy arrays, or slices of garage_ec_host_alloc buffers"""

    def __init__(self, ec, pinned):
        self.ec, self.pinned, self.ptrs = ec, pinned, []

    def __call__(self, shape, fill):
        size = int(np.prod(shape))
        if self.pinned:
            a, p = self.ec.host_alloc(max(size, 16))
            self.ptrs.append(p)
            a = a[:size].reshape(shape)
        else:
            a = np.empty(shape, dtype=np.uint8)
        a[...] = fill
        return a

    def free(self):
        for p in self.ptrs:
            self.ec.host_free(p)


def fault_call(form, code, ec, buf, sb, want):
    """(run, outputs, reset, check, never, done) for one HOST form: run() makes the call and returns its code,
    reset() fills the outputs, check() asserts the exact result, never() the outputs a failed call must not have
    written, done() lists the blocks whose plaintext a failed call had already delivered"""
    n, tot, stride = len(sb), code.tot, FAULT_STRIDE
    pts = [x.pt for x in sb]
    keys, nonces = np.stack([x.key for x in sb]), np.stack([x.nonce for x in sb])
    plen = np.array([p.size for p in pts], dtype=np.uint32)
    pitch = r16(max(plen))
    if form.startswith("seal"):
        sh = buf((n, tot, stride), POISON)
        hs, sums = np.zeros((n, 32), dtype=np.uint8), np.zeros((n, tot, 32), dtype=np.uint8)
        hashes = np.stack([np.frombuffer(blake2(x.B), dtype=np.uint8) for x in sb])
        Ls = [code.shard_len(x.B.size) for x in sb]
        tags = expected_tags(want, Ls, G.SUM_BLAKE2)
        if form == "seal":
            rows = buf((n, pitch), 0)
            rows[:] = plain_rows(pts, pitch)
            run = lambda: ec.seal(rows.reshape(-1), pitch, plen, keys, nonces, sh.reshape(-1), stride, hs, sums)  # noqa: E731
        else:
            blocks = buf((n, pitch), 0)
            blocks[:] = plain_rows(pts, pitch)
            views = [blocks[s, :plen[s]] for s in range(n)]
            run = lambda: ec.seal_blocks(views, keys, nonces, sh.reshape(-1), stride, hs, sums)  # noqa: E731

        def reset():
            sh[...] = POISON

        def check():
            same(sh, want, form + " shards")
            same(hs, hashes, form + " content hash")
            same(sums, tags, form + " shard tags")

        return run, [sh, hs, sums], reset, check, lambda: None, lambda: []

    # the open forms: two blocks tampered, their hash recorded as stored (only a tag fails)
    shards = buf((n, tot, stride), 0)
    shards[:] = want
    hashes = np.zeros((n, 32), dtype=np.uint8)
    for s, x in enumerate(sb):
        B = x.B.copy()
        if s in FAULT_TAMPERED:
            L = code.shard_len(B.size)
            B[L + 5] ^= 1  # ciphertext in data shard 1 (shard 0 is absent and rebuilt from parity)
            shards[s, 1, 5] ^= 1
        hashes[s] = np.frombuffer(blake2(B), dtype=np.uint8)
    pres = np.ones((n, tot), dtype=np.uint8)
    pres[:, 0] = 0  # the prefix and chunk 0 rebuilt from parity
    shards[:, 0] = GONE
    sl = np.array([x.B.size for x in sb], dtype=np.uint32)
    st = np.zeros(n, dtype=np.int32)
    exp = np.array([G.E_AUTH if s in FAULT_TAMPERED else 0 for s in range(n)], dtype=np.int32)
    if form.startswith("open_range"):
        offs = np.array([0 if s in FAULT_TAMPERED else plen[s] // 3 for s in range(n)], dtype=np.uint32)
        lens = np.array([plen[s] - offs[s] for s in range(n)], dtype=np.uint32)
        ost = r16(int(lens.max()))
        want_out = [pts[s][offs[s]:offs[s] + lens[s]] for s in range(n)]
        if form == "open_range":
            out = buf((n, ost), SENT)
            rows = [out[s] for s in range(n)]
            run = lambda: ec.open_range(shards.reshape(-1), pres, sl, keys, offs, lens, stride, out.reshape(-1), ost, st)  # noqa: E731,E501
            outputs = [out, st]
        else:
            big = buf((n, ost + 32), SENT)
            rows = [big[s, :lens[s] + 32] for s in range(n)]
            run = lambda: ec.open_range_stripes([shards[s].reshape(-1) for s in range(n)], pres, sl, keys, offs,  # noqa: E731,E501
                                                lens, stride, rows, st)
            outputs = [big, st]
        plen_out = bad = None
    else:
        want_out = pts
        plen_out = np.zeros(n, dtype=np.uint32)
        bad = np.zeros(n, dtype=np.uint8)
        if form == "open":
            out = buf((n, pitch), SENT)
            rows = [out[s] for s in range(n)]
            run = lambda: ec.open(shards.reshape(-1), pres, sl, hashes, keys, out.reshape(-1), pitch, plen_out, bad, st,  # noqa: E731,E501
                                  stride)
            outputs = [out, plen_out, bad, st]
        else:
            big = buf((n, pitch + 32), SENT)
            rows = [big[s, :plen[s] + 32] for s in range(n)]
            run = lambda: ec.open_stripes([shards[s].reshape(-1) for s in range(n)], pres, sl, hashes, keys, rows,  # noqa: E731,E501
                                          plen_out, bad, st, stride)
            outputs = [big, plen_out, bad, st]

    def reset():
        for o in outputs[:1]:
            o[...] = SENT
        for o in outputs[1:]:
            o[...] = 0

    def check():
        assert list(st) == list(exp), list(st)
        for s in range(n):
            w = want_out[s]
            if exp[s]:
                assert (rows[s] == SENT).all(), s
            else:
                assert np.array_equal(rows[s][:w.size], w) and (rows[s][w.size:] == SENT).all(), s
                if plen_out is not None:
                    assert plen_out[s] == w.size and bad[s] == 0, s

    def never():
        for s in FAULT_TAMPERED:
            assert (rows[s] == SENT).all(), ("plaintext of a block whose tag failed", s)

    def done():
        return [s for s in range(n) if not exp[s] and not (rows[s] == SENT).all()]

    return run, outputs, reset, check, never, done


@pytest.mark.gpu
@pytest.mark.parametrize("pinned", [False, True], ids=["pageable", "pinned"])
@pytest.mark.parametrize("form", FAULT_FORMS)
def test_sse_host_form_fault_leaves_caller_buffers_alone(torch, pool, form, pinned):
    """the contract test_host_call_fault_leaves_caller_buffers_alone asserts for the other HOST calls, for every
    SSE-C HOST form over five pipeline chunks, with the fault injected at every checked runtime call of the call in
    turn -- issue, the retire steps that decide which plaintexts come down, and drain -- until the call completes:
    the call returns an error, a failed open never wrote plaintext of a block whose tag failed, nothing writes the
    caller's outputs after the return, and the context is exact on the next call (seal forms: on every fourth, their
    outputs are large)"""
    code = Code(FAULT_CASE)
    sb = pool.get(FAULT_ITEMS)
    want, _ = expected_shards(code, [x.B for x in sb], FAULT_STRIDE)
    assert code.tot * FAULT_STRIDE > 24 << 20
    opens = not form.startswith("seal")
    with code.ctx() as ec:
        buf = Buffers(ec, pinned)
        try:
            run, outputs, reset, check, never, done = fault_call(form, code, ec, buf, sb, want)
            reset()
            run()  # lanes sized, key staging allocated
            check()
            delivered = []
            for fail_at in range(1000):
                reset()
                ec.debug_fail_after(fail_at)
                try:
                    run()
                except G.EcError as e:
                    err = e.code
                else:
                    err = None
                finally:
                    ec.debug_fail_after(-1)
                if err is None:  # past the call's last checked runtime call
                    check()
                    break
                assert err in (G.E_CUDA, G.E_NOMEM), (fail_at, err)
                never()
                delivered.append(done())
                for o in outputs:
                    o.view(np.uint8)[...] = 0xEE
                torch.cuda.synchronize()
                assert all((o.view(np.uint8) == 0xEE).all() for o in outputs), (
                    "a copy or kernel wrote after the error return", fail_at)
                if opens or fail_at % 4 == 3:
                    reset()
                    run()
                    check()
            else:
                pytest.fail("the call still failed after 1000 injected faults")
            assert fail_at >= 5 * 3, fail_at  # every chunk has several checked calls
            if opens:  # faults landed in the retire of chunk 0 and after the last retire of drain
                good = [s for s in range(len(sb)) if s not in FAULT_TAMPERED]
                assert any(d == [0] for d in delivered), delivered
                assert any(d == good for d in delivered), delivered
        finally:
            buf.free()
