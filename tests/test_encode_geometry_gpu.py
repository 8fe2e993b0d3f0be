"""Encode and verify geometry of RS, LRC, PB and Clay on the GPU, against the C oracle (RS, LRC) and the numpy models
(pb_oracle, clay_oracle).

Every compiled uniform-mode shape of each code runs in ragged batches of at least 4 x SMs x 32 work items (Clay: 4 x 16
x SMs columns), so every warp (Clay: CTA) walks several items, staged ones and empty chunks past the end of short
stripes in turn.  Shard lengths interleave short and long stripes with runs of equal ones; strides are < 512 (no
tensor map), a multiple of 512, and 512*j + 16 (every stripe's last chunk partial).  Bytes [L, stride) of every input
shard are garbage and parity outputs start as POISON: encode must equal the model over [0, L), write zeros over
[L, roundup16(L)) (RS, LRC) and nothing else.  Verify of the clean batch gives 0 words; of a corrupted batch, exactly
the rows where the model's re-encode of the corrupted data differs from the stored row.  Also: staged HOST mode
(pageable and pinned) over several pipeline chunks, encode_blocks with both tag kinds, and stripes whose shard_len
exceeds the stride.

The models encode one wide stripe per batch: every code here is column-local (DESIGN.md section 2.5), so the
concatenated PB halves, or Clay layers, of all stripes encode as one stripe; test_wide_stripe_oracle pins that."""
import hashlib
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import clay_oracle as CO  # noqa: E402
import lrc_oracle as LO  # noqa: E402
import oracle_lib as O  # noqa: E402
import pb_oracle as PB  # noqa: E402
from test_blake2 import adler8_ref  # noqa: E402  the zlib model of the adler8 tag

import garage_b200 as G  # noqa: E402

POISON = 0xA5  # parity outputs before encode
STAGE = 512    # bytes of one stage row: 32 columns of 16 bytes
MAX_WARPS = 32  # the most warps a CTA of the uniform kernels has
HOST_CHUNK = 48 << 20  # source bytes of one HOST pipeline chunk

VAND, CAUCHY = 0, 1
# RS: every k of launch_apply's GEC_CASE list; m cycles through 1..8, so two-pass m (5..8) meets small, mid and large k
RS_CASES = ([(k, 1 + (3 * k) % 8, VAND) for k in range(1, 33)]
            + [(k, m, CAUCHY) for k, m in [(1, 8), (4, 5), (7, 3), (10, 4), (12, 6), (16, 8), (23, 7), (32, 5)]])
LRC_CASES = [(4, 2, 1), (12, 3, 2), (16, 4, 2), (20, 4, 4), (24, 6, 2), (32, 4, 4)]
PB_CASES = ([(k, m, CAUCHY) for k in range(1, 17) for m in (2, 3, 4)]
            + [(k, m, VAND) for k, m in [(1, 4), (2, 4), (5, 3), (10, 4), (16, 3)]])
CLAY_CASES = [(2, 2), (3, 2), (5, 2), (13, 2), (14, 2), (4, 3), (6, 3), (11, 3), (12, 3), (2, 4), (5, 4), (10, 4),
              (12, 4)]

# RS / LRC strides: no tensor map, a multiple of 512, a 16-byte last chunk; cases rotate through them
RS_STRIDES = (496, 2048, 1552)
# PB half lengths: 1..6 stage rows, partial last chunks, last chunks of one 16-byte column
PB_HALVES = [16, 496, 512, 528, 1008, 1040, 1536, 1552, 2064, 2576, 3056, 3072]
PB_STRIDES = (6208, 6144)  # 512*12 + 64 and 512*12
CLAY_UNITS = [1, 2, 3]  # shard_len = units * 16 * alpha: 1..3 columns per layer; stride: 4 units


def rs_lens(stride):
    """any length: 1, the len & 15 tails, stage-row edges, stride - 1 and stride"""
    pool = [1, 15, 16, 17, 31, 100, 496, 511, 512, 513, 1000, 1024, 1300, 1537, stride - 1, stride]
    return sorted({x for x in pool if x <= stride})


# ---------------------------------------------------------------------------------------------- models
def pb_wide_encode(P, data, lens):
    """PB parity of stripes data (n, k, W) with shard lengths lens: the a-halves of all stripes, then their b-halves,
    encoded as one stripe and split back; (n, m, W), zero past each L"""
    n, k, W = data.shape
    hs = [int(L) // 2 for L in lens]
    a = np.concatenate([data[s, :, :hs[s]] for s in range(n)], axis=1)
    b = np.concatenate([data[s, :, hs[s]:2 * hs[s]] for s in range(n)], axis=1)
    par = PB.encode(P, np.concatenate([a, b], axis=1))
    H = a.shape[1]
    out = np.zeros((n, P.shape[0], W), dtype=np.uint8)
    o = 0
    for s in range(n):
        out[s, :, :hs[s]] = par[:, o:o + hs[s]]
        out[s, :, hs[s]:2 * hs[s]] = par[:, H + o:H + o + hs[s]]
        o += hs[s]
    return out


def clay_wide_encode(k, m, P, data, lens):
    """Clay parity: layer z of the wide stripe is layer z of every stripe, concatenated; (n, m, W), zero past L"""
    n, _, W = data.shape
    alpha = CO.params(k, m)[4]
    subs = [int(L) // alpha for L in lens]
    wide = np.concatenate([data[s, :, :int(lens[s])].reshape(k, alpha, subs[s]) for s in range(n)], axis=2)
    par = CO.encode(k, m, P, wide.reshape(k, -1)).reshape(m, alpha, -1)
    out = np.zeros((n, m, W), dtype=np.uint8)
    o = 0
    for s in range(n):
        out[s, :, :int(lens[s])] = par[:, :, o:o + subs[s]].reshape(m, -1)
        o += subs[s]
    return out


class Rs:
    family = "rs"
    unit, zero_tail = 1, True

    def __init__(self, k, m, kind, stride=1552):
        self.k, self.m, self.kind, self.tot, self.stride = k, m, kind, k + m, stride
        self.P = O.build_matrix(k, m, kind)
        self.key = ("rs", k, m, kind, stride)

    def ctx(self):
        return G.GarageEc(0, self.k, self.m, self.kind)

    def lens(self):
        return rs_lens(self.stride)

    def ips(self):
        return -(-self.stride // STAGE)

    def encode(self, data, lens):
        n, _, W = data.shape
        flat = np.ascontiguousarray(data).reshape(-1)
        return O.encode(self.k, self.m, self.P, flat, W, n, shard_len=np.asarray(lens, dtype=np.uint32),
                        simd=True).reshape(n, self.m, W)

    def flips(self, L):
        """byte 0, the tail byte L - 1, both ends of a middle chunk, a byte of the last chunk"""
        mid = L // STAGE // 2 * STAGE
        return [0, L - 1, mid, min(L, mid + STAGE) - 1, (L - 1) // STAGE * STAGE + ((L - 1) % STAGE) // 2]


class Lrc(Rs):
    family = "lrc"

    def __init__(self, k, l, r, stride=1552):
        self.k, self.l, self.r, self.m, self.tot, self.stride = k, l, r, l + r, k + l + r, stride
        self.P = LO.build_lrc(k, l, r)
        self.key = ("lrc", k, l, r, stride)

    def ctx(self):
        return G.GarageEc.lrc(0, self.k, self.l, self.r)


class Pb:
    family = "pb"
    unit, zero_tail = 32, False

    def __init__(self, k, m, kind, stride=6208):
        self.k, self.m, self.kind, self.tot, self.stride = k, m, kind, k + m, stride
        self.P = PB.build(k, m, kind)
        self.key = ("pb", k, m, kind, stride)

    def ctx(self):
        return G.GarageEc.piggyback(0, self.k, self.m, self.kind)

    def lens(self):
        return [2 * h for h in PB_HALVES if 2 * h <= self.stride]

    def ips(self):
        return (self.stride // 32 + 31) // 32

    def encode(self, data, lens):
        return pb_wide_encode(self.P, data, lens)

    def flips(self, L):
        """byte 0, the last bytes of both halves, both ends of a middle a-chunk, a byte of the last b-chunk"""
        h = L // 2
        mid = h // STAGE // 2 * STAGE
        return [0, L - 1, h - 1, mid, min(h, mid + STAGE) - 1, h + (h - 1) // STAGE * STAGE + ((h - 1) % STAGE) // 2]


class Clay:
    family = "clay"
    unit, zero_tail = None, False

    def __init__(self, k, m, kind=VAND, stride_units=4):
        self.k, self.m, self.kind, self.tot = k, m, kind, k + m
        self.alpha = CO.params(k, m)[4]
        self.unit = 16 * self.alpha
        self.stride = stride_units * self.unit
        self.P = CO.build(k, m, kind)
        self.key = ("clay", k, m, kind)

    def ctx(self):
        return G.GarageEc.clay(0, self.k, self.m, self.kind)

    def lens(self):
        return [u * self.unit for u in CLAY_UNITS]

    def ips(self):
        return -(-self.stride // self.unit)

    def encode(self, data, lens):
        return clay_wide_encode(self.k, self.m, self.P, data, lens)

    def flips(self, L):
        """byte 0, the last byte, a byte of the last layer and of a middle one"""
        sub = L // self.alpha
        return [0, L - 1, (self.alpha - 1) * sub + sub // 2, (self.alpha // 2) * sub]


def rs_case(i, k, m, kind):
    return Rs(k, m, kind, RS_STRIDES[i % 3])


def lrc_case(i, k, l, r):
    return Lrc(k, l, r, RS_STRIDES[(i + 1) % 3])


def pb_case(i, k, m, kind):
    return Pb(k, m, kind, PB_STRIDES[i % 2])


# ---------------------------------------------------------------------------------------------- batches
@pytest.fixture(scope="module")
def torch():
    import torch as t

    assert t.cuda.is_available()
    return t


@pytest.fixture(scope="module")
def sms(torch):
    return torch.cuda.get_device_properties(0).multi_processor_count


def dev(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def n_for(code, sms):
    """stripes for at least 4 x SMs x 32 work items (Clay: 4 x 16 x SMs columns)"""
    return -(-4 * sms * (16 if code.family == "clay" else MAX_WARPS) // code.ips())


def ragged(pool, n):
    """lengths of n stripes: short and long alternating, with a run of 8 equal lengths in every 32 stripes; every
    length of the pool occurs"""
    short, long_ = pool[:(len(pool) + 1) // 2], pool[(len(pool) + 1) // 2:] or pool
    out = np.zeros(n, dtype=np.uint32)
    for s in range(n):
        b = s // 8
        if b % 4 == 3:
            out[s] = pool[(b // 4) % len(pool)]
        elif s % 2:
            out[s] = long_[(s // 2 + b) % len(long_)]
        else:
            out[s] = short[(s // 2 + 3 * b) % len(short)]
    return out


def make_batch(code, n, seed):
    """(data (n, k, stride) random in full, the bytes past L garbage; lens; model parity (n, m, stride))"""
    lens = ragged(code.lens(), n)
    data = O.fill_random(n * code.k * code.stride, seed).reshape(n, code.k, code.stride)
    return data, lens, code.encode(data, lens)


def stored_shards(code, data, lens, ref, seed):
    """the shard layout of a batch: data, then the model parity with garbage past L"""
    n = data.shape[0]
    par = O.fill_random(n * code.m * code.stride, seed).reshape(n, code.m, code.stride)
    inside = np.arange(code.stride)[None, None, :] < lens[:, None, None]
    par = np.where(inside, ref, par)
    return np.ascontiguousarray(np.concatenate([data, par], axis=1))


def expected_parity(torch, code, ref, lens):
    """what encode leaves in a POISON-filled parity buffer: the model over [0, L), RS / LRC zeros up to roundup16(L)"""
    stride = ref.shape[2]
    col = torch.arange(stride, device="cuda")[None, None, :]
    L = dev(torch, lens.astype(np.int64))[:, None, None]
    exp = torch.where(col < L, dev(torch, ref), torch.full((), POISON, dtype=torch.uint8, device="cuda"))
    if code.zero_tail:
        exp = torch.where((col >= L) & (col < (L + 15) // 16 * 16), torch.zeros((), dtype=torch.uint8, device="cuda"),
                          exp)
    return exp


def assert_rows(got, exp, what):
    diff = (got != exp).any(dim=2).nonzero()
    assert not len(diff), "%s: %d parity rows differ, first (stripe, row): %s" % (what, len(diff), diff[:8].tolist())


def corrupt(code, sh, lens, seed):
    """flip 1..3 bytes of most stripes at the edges kernels get wrong, in data and parity rows (rows >= 4 too);
    the expected mismatch words from the model's re-encode of the corrupted data"""
    n, k, m = sh.shape[0], code.k, code.m
    bad = sh.copy()
    rng = np.random.default_rng(seed)
    touched = []
    for s in range(n):
        if s % 8 == 7:
            continue
        L = int(lens[s])
        pos = code.flips(L)
        for _ in range(1 + s % 3):
            row = int(rng.integers(0, k)) if rng.random() < 0.35 else k + int(rng.integers(0, m))
            bad[s, row, pos[int(rng.integers(0, len(pos)))]] ^= int(rng.integers(1, 256))
        touched.append(s)
    touched = np.array(touched)
    re = code.encode(bad[touched, :k], lens[touched])
    inside = np.arange(code.stride)[None, None, :] < lens[touched, None, None]
    diff = ((re != bad[touched, k:]) & inside).any(axis=2)
    exp = np.zeros(n, dtype=np.uint32)
    exp[touched] = (diff.astype(np.uint32) << np.arange(m, dtype=np.uint32)[None, :]).sum(axis=1).astype(np.uint32)
    return bad, exp


def verify_device(torch, ec, code, sh, lens, n):
    mm = torch.full((n,), -1, dtype=torch.int32, device="cuda")  # 0xFFFFFFFF: every word must be written
    ec.verify(dev(torch, sh).view(-1), mm, code.stride, n, shard_len=None if lens is None else dev(torch, lens.astype(np.int32)))
    return mm.cpu().numpy().view(np.uint32)


def geometry(torch, sms, code, seed):
    n = n_for(code, sms)
    data, lens, ref = make_batch(code, n, seed)
    assert len(set(lens.tolist())) == len(code.lens())
    with code.ctx() as ec:
        par = torch.full((n, code.m, code.stride), POISON, dtype=torch.uint8, device="cuda")
        ec.encode(dev(torch, data).view(-1), par.view(-1), code.stride, n, shard_len=dev(torch, lens.astype(np.int32)))
        assert_rows(par, expected_parity(torch, code, ref, lens), "%s encode" % (code.key,))
        sh = stored_shards(code, data, lens, ref, seed + 1)
        mm = verify_device(torch, ec, code, sh, lens, n)
        assert not mm.any(), "%s: clean stripes flagged at %s" % (code.key, np.nonzero(mm)[0][:8])
        bad, exp = corrupt(code, sh, lens, seed + 2)
        assert exp.any()
        mm = verify_device(torch, ec, code, bad, lens, n)
        wrong = np.nonzero(mm != exp)[0]
        assert not len(wrong), "%s: verify words %s, model %s at stripes %s" % (
            code.key, [hex(x) for x in mm[wrong[:8]]], [hex(x) for x in exp[wrong[:8]]], wrong[:8])


# ---------------------------------------------------------------------------------------------- CPU
def test_case_table_reaches_every_shape():
    """RS: every k of the GEC_CASE list with m 1..8, two-pass m with k <= 8, 9..16 and > 16, every stride class
    with the split (k > 16), TMA and LDG classes; LRC: k > 16 with m = 8; PB: every pb_apply_kernel<K>
    (k = 1..16) with m 2, 3, 4 under Cauchy, Vandermonde PB(1,4) and PB(2,4); Clay: every m, with and without
    virtual nodes, alpha up to 256; lengths hit the stage-row edges and tails"""
    rs = [rs_case(i, *c) for i, c in enumerate(RS_CASES)]
    assert {c.k for c in rs} == set(range(1, 33)) and {c.m for c in rs} == set(range(1, 9))
    for lo, hi in ((1, 8), (9, 16), (17, 32)):
        assert any(lo <= c.k <= hi and c.m > 4 for c in rs), (lo, hi)
    for st in RS_STRIDES:
        for lo, hi in ((1, 12), (13, 16), (17, 32)):
            assert any(c.stride == st and lo <= c.k <= hi for c in rs), (st, lo, hi)
    assert sum(c.kind == CAUCHY for c in rs) == 8
    assert RS_STRIDES[0] < STAGE and RS_STRIDES[1] % STAGE == 0 and RS_STRIDES[2] % STAGE == 16
    for st in RS_STRIDES:
        pool = rs_lens(st)
        assert {1, 15, 16, 17, st - 1, st} <= set(pool) and (st < 513 or {511, 512, 513} <= set(pool))
    for k, l, r in LRC_CASES:
        LO.build_lrc(k, l, r)
    assert {(4, 2, 1), (12, 3, 2), (20, 4, 4), (24, 6, 2), (32, 4, 4)} <= set(LRC_CASES)
    assert {(k, m) for k, m, kind in PB_CASES if kind == CAUCHY} == {(k, m) for k in range(1, 17) for m in (2, 3, 4)}
    assert {(1, 4), (2, 4)} <= {(k, m) for k, m, kind in PB_CASES if kind == VAND}
    rows = {-(-h // STAGE) for h in PB_HALVES}
    assert rows == {1, 2, 3, 4, 5, 6} and all(h % 16 == 0 for h in PB_HALVES)
    assert all(2 * max(PB_HALVES) <= st for st in PB_STRIDES) and PB_STRIDES[1] % STAGE == 0
    params = [CO.params(k, m) for k, m in CLAY_CASES]
    for q in (2, 3, 4):
        assert {p[3] > 0 for p in params if p[0] == q} == {False, True}
    assert {243, 256} <= {p[4] for p in params}
    # every warp walks several items with empty chunks between staged ones
    assert all(ragged(rs_lens(st), 64).tolist().count(st) for st in RS_STRIDES)


def test_wide_stripe_oracle():
    """the one-wide-stripe models equal per-stripe PB.encode / CO.encode on stripes of different lengths"""
    rng = np.random.default_rng(7)
    for k, m, kind in [(5, 3, CAUCHY), (1, 4, VAND), (16, 4, CAUCHY)]:
        P = PB.build(k, m, kind)
        lens = np.array([32, 992, 64, 6144, 1056, 32], dtype=np.uint32)
        data = rng.integers(0, 256, (len(lens), k, 6208), dtype=np.uint8)
        got = pb_wide_encode(P, data, lens)
        for s, L in enumerate(lens):
            assert np.array_equal(got[s, :, :L], PB.encode(P, data[s, :, :L])), (k, m, s)
            assert not got[s, :, L:].any()
    for k, m in [(5, 2), (4, 3), (6, 3), (5, 4)]:
        P = CO.build(k, m)
        u = 16 * CO.params(k, m)[4]
        lens = np.array([u, 3 * u, 2 * u, u, 3 * u], dtype=np.uint32)
        data = rng.integers(0, 256, (len(lens), k, 4 * u), dtype=np.uint8)
        got = clay_wide_encode(k, m, P, data, lens)
        for s, L in enumerate(lens):
            assert np.array_equal(got[s, :, :L], CO.encode(k, m, P, data[s, :, :L])), (k, m, s)
            assert not got[s, :, L:].any()


# ---------------------------------------------------------------------------------------------- geometry
@pytest.mark.gpu
@pytest.mark.parametrize("i", range(len(RS_CASES)), ids=["k%d-m%d-%s" % (k, m, "cauchy" if c else "vand")
                                                        for k, m, c in RS_CASES])
def test_rs_encode_verify_geometry(torch, sms, i):
    geometry(torch, sms, rs_case(i, *RS_CASES[i]), 0xE0C0 + 97 * i)


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(len(LRC_CASES)), ids=["%d-%d-%d" % c for c in LRC_CASES])
def test_lrc_encode_verify_geometry(torch, sms, i):
    geometry(torch, sms, lrc_case(i, *LRC_CASES[i]), 0x1EC0 + 31 * i)


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(len(PB_CASES)), ids=["k%d-m%d-%s" % (k, m, "cauchy" if c else "vand")
                                                        for k, m, c in PB_CASES])
def test_pb_encode_verify_geometry(torch, sms, i):
    geometry(torch, sms, pb_case(i, *PB_CASES[i]), 0x9BE0 + 13 * i)


@pytest.mark.gpu
@pytest.mark.parametrize("k,m", CLAY_CASES)
def test_clay_encode_verify_geometry(torch, sms, k, m):
    geometry(torch, sms, Clay(k, m), 0xC1E0 + 4 * k + m)


@pytest.mark.gpu
@pytest.mark.parametrize("code", [Rs(10, 4, VAND, 1552), Rs(20, 8, CAUCHY, 1040), Lrc(12, 3, 2, 1552),
                                  Pb(10, 4, VAND, 1568), Clay(6, 3, VAND, 3)], ids=lambda c: "-".join(map(str, c.key)))
def test_uniform_batch_at_odd_stride(torch, sms, code):
    """shard_len = NULL at a stride that is not a multiple of 512: every stripe's last chunk is partial"""
    assert code.stride % STAGE
    n = n_for(code, sms)
    data = O.fill_random(n * code.k * code.stride, 0x0DD + code.k).reshape(n, code.k, code.stride)
    lens = np.full(n, code.stride, dtype=np.uint32)
    ref = code.encode(data, lens)
    with code.ctx() as ec:
        par = torch.full((n, code.m, code.stride), POISON, dtype=torch.uint8, device="cuda")
        ec.encode(dev(torch, data).view(-1), par.view(-1), code.stride, n)
        assert_rows(par, dev(torch, ref), "%s uniform encode" % (code.key,))
        sh = np.ascontiguousarray(np.concatenate([data, ref], axis=1))
        assert not verify_device(torch, ec, code, sh, None, n).any()
        bad, exp = corrupt(code, sh, lens, 0x0DE)
        mm = verify_device(torch, ec, code, bad, None, n)
        assert np.array_equal(mm, exp), np.nonzero(mm != exp)[0][:8]


# ---------------------------------------------------------------------------------------------- HOST mode
@pytest.mark.gpu
@pytest.mark.parametrize("code", [Rs(10, 4, VAND, 4112), Rs(24, 6, CAUCHY, 2048), Lrc(12, 3, 2, 1552),
                                  Pb(10, 4, VAND, 6208), Clay(10, 4)], ids=lambda c: "-".join(map(str, c.key)))
def test_host_mode_many_chunks(torch, code):
    """staged HOST encode and verify, pageable and pinned, over five or more pipeline chunks (three lanes, so the
    lanes wrap): the same parity buffer as DEVICE, POISON past roundup16(L) included (the lane buffers hold stale
    bytes there that must never reach the caller), and the same words as DEVICE and the model"""
    k, m, stride = code.k, code.m, code.stride
    n = -(-5 * HOST_CHUNK // (k * stride))
    data, lens, ref = make_batch(code, n, 0x40E7 + k)
    sh = stored_shards(code, data, lens, ref, 0x40E8)
    bad, exp = corrupt(code, sh, lens, 0x40E9)
    with code.ctx() as ec:
        par = torch.full((n, m, stride), POISON, dtype=torch.uint8, device="cuda")
        ec.encode(dev(torch, data).view(-1), par.view(-1), stride, n, shard_len=dev(torch, lens.astype(np.int32)))
        want = expected_parity(torch, code, ref, lens)
        assert_rows(par, want, "%s DEVICE encode" % (code.key,))
        dmm = verify_device(torch, ec, code, bad, lens, n)
        assert np.array_equal(dmm, exp)
        bufs = []
        try:
            for pinned in (False, True):
                if pinned:
                    d_in, p1 = ec.host_alloc(data.size)
                    bufs.append(p1)
                    d_out, p2 = ec.host_alloc(n * m * stride)
                    bufs.append(p2)
                    s_in, p3 = ec.host_alloc(bad.size)
                    bufs.append(p3)
                    d_in[:] = data.reshape(-1)
                    s_in[:] = bad.reshape(-1)
                    d_out[:] = POISON
                else:
                    d_in, s_in = data.reshape(-1), bad.reshape(-1)
                    d_out = np.full(n * m * stride, POISON, dtype=np.uint8)
                what = "%s HOST %s" % (code.key, "pinned" if pinned else "pageable")
                ec.encode(d_in, d_out, stride, n, shard_len=lens)
                got = dev(torch, d_out).view(n, m, stride)
                assert_rows(got, want, what + " encode")
                hm = np.full(n, 0xFFFFFFFF, dtype=np.uint32)
                ec.verify(s_in, hm, stride, n, shard_len=lens)
                assert np.array_equal(hm, exp), what + " verify"
        finally:
            for p in bufs:
                ec.host_free(p)


# ---------------------------------------------------------------------------------------------- block level
@pytest.mark.gpu
@pytest.mark.parametrize("code", [Rs(10, 4, VAND), Rs(20, 8, CAUCHY), Lrc(12, 3, 2), Pb(10, 4, VAND), Pb(3, 2, CAUCHY),
                                  Clay(5, 4), Clay(6, 3)], ids=lambda c: "-".join(map(str, c.key)))
def test_encode_blocks_parity_and_tags(torch, code):
    """a few hundred blocks of mixed lengths (1 byte, blocks whose last data shards are all padding, lengths the code
    rounds up): parity equals the model's encode of the framed shards, every tag equals hashlib / zlib"""
    k, m, tot = code.k, code.m, code.tot
    rng = np.random.default_rng(0xB10C + k)
    sizes = [1, 2, k - 1, k, k + 1, 3 * k + 1, 511, 4096, 100000, 1 << 18]
    sizes += [int(x) for x in rng.integers(1, 1 << 18, 250)]
    with code.ctx() as ec:
        Ls = np.array([ec.code_shard_len(b) for b in sizes], dtype=np.uint32)
        if code.family in ("pb", "clay"):
            assert any(int(L) > -(-b // k) for L, b in zip(Ls, sizes))  # rounded up past ceil(len / k)
        stride = (int(Ls.max()) + 15) // 16 * 16
        n = len(sizes)
        blocks = [O.fill_random(b, 0xB1 + i) for i, b in enumerate(sizes)]
        data = np.zeros((n, k, stride), dtype=np.uint8)
        for s, b in enumerate(blocks):
            flat = np.zeros(k * int(Ls[s]), dtype=np.uint8)
            flat[:b.size] = b
            data[s, :, :Ls[s]] = flat.reshape(k, -1)
        assert not data[1, 2:].any()  # a 2-byte block: every data shard but the first two is padding
        ref = code.encode(data, Ls)
        for kind in (G.SUM_BLAKE2, G.SUM_ADLER8):
            ec.set_sum_kind(kind)
            par = np.zeros(n * m * stride, dtype=np.uint8)
            sums = np.zeros(n * tot * 32, dtype=np.uint8)
            ec.encode_blocks(blocks, par, stride, sums_out=sums)
            par, sums = par.reshape(n, m, stride), sums.reshape(n, tot, 32)
            for s in range(n):
                L = int(Ls[s])
                assert np.array_equal(par[s, :, :L], ref[s, :, :L]), (kind, s, sizes[s])
                for i in range(tot):
                    body = (data[s, i, :L] if i < k else par[s, i - k, :L]).tobytes()
                    tag = hashlib.blake2b(body).digest()[:32] if kind == G.SUM_BLAKE2 else adler8_ref(body)
                    assert sums[s, i].tobytes() == tag, (kind, s, i)


# ---------------------------------------------------------------------------------------------- malformed lengths
@pytest.mark.gpu
@pytest.mark.parametrize("code", [Rs(10, 4, VAND, 1552), Rs(20, 8, CAUCHY, 1552), Rs(4, 6, VAND, 496),
                                  Lrc(12, 3, 2, 1040), Pb(10, 4, VAND, 6208), Pb(16, 3, CAUCHY, 1568),
                                  Clay(6, 3, VAND, 4)], ids=lambda c: "-".join(map(str, c.key)))
def test_shard_len_past_the_stride(torch, sms, code):
    """stripes whose shard_len exceeds a stride that is not a multiple of 512, in the middle of a batch: DEVICE
    encode writes nothing of them and nothing into their neighbours, DEVICE verify sets exactly their m low bits,
    every other stripe is right; HOST encode, verify and reconstruct return E_INVALID.  Device buffers are one
    stripe longer than the batch, so a kernel that overruns shows as changed bytes"""
    k, m, tot, stride = code.k, code.m, code.tot, code.stride
    assert stride % STAGE
    n = 2 * sms + 37
    data, lens, ref = make_batch(code, n, 0xBAD + k)
    over = [stride + code.unit, stride + 16 * code.unit, stride + 97 * code.unit]  # well framed, only too long
    mal = [n // 3, n // 2, n // 2 + 1, 2 * n // 3]
    for j, s in enumerate(mal):
        lens[s] = over[j % len(over)]
    good = np.setdiff1d(np.arange(n), mal)
    ref[mal] = 0
    sh = stored_shards(code, data, np.where(lens > stride, 0, lens).astype(np.uint32), ref, 0xBAE)
    with code.ctx() as ec:
        dl = dev(torch, lens.astype(np.int32))
        d = torch.zeros((n + 1, k, stride), dtype=torch.uint8, device="cuda")
        d[:n] = dev(torch, data)
        par = torch.full((n + 1, m, stride), POISON, dtype=torch.uint8, device="cuda")
        ec.encode(d.view(-1), par.view(-1), stride, n, shard_len=dl)
        exp = expected_parity(torch, code, ref, np.where(lens > stride, 0, lens))
        exp[dev(torch, np.array(mal))] = POISON
        assert_rows(par[:n], exp, "%s DEVICE encode" % (code.key,))
        assert (par[n] == POISON).all(), "encode wrote past the batch"
        s = torch.zeros((n + 1, tot, stride), dtype=torch.uint8, device="cuda")
        s[:n] = dev(torch, sh)
        mm = torch.full((n + 1,), -1, dtype=torch.int32, device="cuda")
        ec.verify(s.view(-1), mm, stride, n, shard_len=dl)
        mm = mm.cpu().numpy().view(np.uint32)
        assert mm[n] == 0xFFFFFFFF
        assert [int(mm[x]) for x in mal] == [(1 << m) - 1] * len(mal), [hex(mm[x]) for x in mal]
        assert not mm[good].any(), good[np.nonzero(mm[good])[0][:8]]
        for call in ("encode", "verify", "reconstruct"):
            with pytest.raises(G.EcError) as e:
                if call == "encode":
                    ec.encode(data.reshape(-1), np.zeros(n * m * stride, dtype=np.uint8), stride, n, shard_len=lens)
                elif call == "verify":
                    ec.verify(sh.reshape(-1), np.zeros(n, dtype=np.uint32), stride, n, shard_len=lens)
                else:
                    present = np.ones((n, tot), dtype=np.uint8)
                    present[:, 0] = 0
                    ec.reconstruct(sh.copy().reshape(-1), present, stride, n, shard_len=lens)
            assert e.value.code == G.E_INVALID, call
