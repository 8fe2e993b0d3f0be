"""Decode geometry of LRC, PB and Clay on the GPU, against the numpy models (lrc_oracle, pb_oracle, clay_oracle).

Every compiled reconstruct shape of each code runs at per-stripe shard lengths whose shard (PB: half, Clay: layer)
spans one to six 512-byte stage rows with a partial last chunk and a one-column tail, in batches longer than twice
the SM count so the last stripes are cut into chunk ranges (Clay: more columns than the grid has CTAs).  Patterns:
every pattern of at most two losses, a seeded sample of 3..m, and m+1; want = NULL, one absent shard or the data
shards only; runs of equal patterns, and a block of one erasure pattern under changing want masks so the table
buffers are reused for equal plans and rebuilt for different ones.  Every rebuilt byte is compared with the
oracle-encoded stripe and every other byte, those past shard_len included, with what was there before.  Also: reads
limited to the host plan, staged HOST equal to DEVICE, a 4096 x 1 MiB PB(10,4) and LRC(10,2,2) decode, and
scrub_repair with adler8 tags."""
import itertools
import os
import struct
import sys
import zlib

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import clay_oracle as CO  # noqa: E402
import lrc_oracle as LO  # noqa: E402
import oracle_lib as O  # noqa: E402
import pb_oracle as PB  # noqa: E402

import garage_b200 as G  # noqa: E402

POISON = 0xA5  # absent shards, and (read-plan test) every byte outside the plan
PAST = 0x3C    # bytes [shard_len, stride) of every shard
STAGE = 512    # bytes of one stage row: 32 columns of 16 bytes

VAND, CAUCHY = 0, 1
PB_CASES = ([(k, m, CAUCHY) for k in range(1, 17) for m in (2, 3, 4)]
            + [(k, m, VAND) for k, m in [(1, 4), (2, 4), (5, 3), (8, 2), (11, 4), (16, 3)]])
LRC_CASES = [(4, 2, 1), (8, 1, 3), (12, 3, 2), (16, 4, 2), (20, 4, 4), (24, 6, 2), (32, 4, 4)]
CLAY_CASES = [(2, 2), (3, 2), (5, 2), (13, 2), (14, 2), (4, 3), (6, 3), (11, 3), (12, 3), (2, 4), (5, 4), (10, 4),
              (12, 4)]
# staged HOST mode (pageable numpy buffers) runs on these as well and must equal DEVICE byte for byte: one and
# several pipeline chunks, thousands of survivor pieces per chunk (PB halves, Clay repair runs)
HOST_CASES = {("pb", 1, 4, CAUCHY), ("pb", 16, 4, CAUCHY), ("pb", 11, 4, VAND), ("lrc", 12, 3, 2), ("lrc", 24, 6, 2),
              ("clay", 5, 4), ("clay", 13, 2)}

# PB half lengths: 1, 2, 3, 4 and 6 stage rows, partial last chunks, last chunks of one 16-byte column
PB_HALVES = [16, 496, 512, 528, 1008, 1040, 1536, 1552, 2064, 2576, 3056, 3072]
# LRC shard lengths: any length, so also the len & 15 tails
LRC_LENS = [1, 15, 16, 17, 511, 512, 513, 1000, 1024, 1300, 1537, 2063, 2591, 3072]
CLAY_UNITS = [1, 2, 3]  # shard_len = units * 16 * alpha: 1..3 columns per layer


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


def span_ok(rows, ncols, present_rows, wanted_rows):
    """rank model: every wanted generator row lies in the span of the present ones.  Rows 0..ncols-1 are the unit
    rows e_q; the present ones cover their columns, so the test runs on the other columns only.  The same answer as
    LO.recoverable / PB.recoverable (test_case_table_reaches_every_shape compares them), but it eliminates over at
    most 2m columns instead of k or 2k, which keeps the thousands of patterns per batch cheap."""
    pres = set(present_rows)
    D = [c for c in range(ncols) if c not in pres]
    B = LO.Basis(len(D))
    for q in sorted(pres):
        if q >= ncols and len(B.rows) < len(D):
            B.add([rows[q][c] for c in D])
    return all(B.express([rows[q][c] for c in D]) is not None for q in wanted_rows)


def _wanted(present, want):
    return [o for o in range(len(present)) if not present[o] and (want is None or want[o])]


class Pb:
    family = "pb"

    def __init__(self, k, m, kind):
        self.k, self.m, self.kind, self.tot = k, m, kind, k + m
        self.P = PB.build(k, m, kind)
        self.rows = PB.half_rows(k, m, self.P)
        self.lens = [2 * h for h in PB_HALVES]
        self.stride = 2 * max(PB_HALVES) + 64
        self.key = ("pb", k, m, kind)

    def ctx(self):
        return G.GarageEc.piggyback(0, self.k, self.m, self.kind)

    def encode(self, d):
        return PB.encode(self.P, d)

    def ok(self, present, want):
        pr = [q for q in range(2 * self.tot) if present[q >> 1]]
        return span_ok(self.rows, 2 * self.k, pr, [2 * o + h for o in _wanted(present, want) for h in range(2)])

    def oracle_decode(self, sh, present, want):
        out = sh.copy()
        assert PB.decode(self.k, self.m, self.P, out, present, want)
        return out

    def plan_pieces(self, ec, present, want, L):
        hv = ec.read_plan(present, want)
        return [(i, h * (L // 2), L // 2) for i in range(self.tot) for h in range(2) if (int(hv[i]) >> h) & 1]


class Lrc:
    family = "lrc"

    def __init__(self, k, l, r):
        self.k, self.l, self.r, self.m, self.tot = k, l, r, l + r, k + l + r
        self.P = LO.build_lrc(k, l, r)
        self.rows = LO.generator_rows(k, self.P)
        self.lens = list(LRC_LENS)
        self.stride = max(LRC_LENS) + 16
        self.key = ("lrc", k, l, r)

    def ctx(self):
        return G.GarageEc.lrc(0, self.k, self.l, self.r)

    def encode(self, d):
        return LO.encode(self.P, d)

    def ok(self, present, want):
        pr = [i for i in range(self.tot) if present[i]]
        return span_ok(self.rows, self.k, pr, _wanted(present, want))

    def oracle_decode(self, sh, present, want):
        out = sh.copy()
        assert LO.decode(self.k, self.l, self.P, out, present, want)
        return out

    def plan_pieces(self, ec, present, want, L):
        hv = ec.read_plan(present, want)
        assert all(int(h) in (0, 3) for h in hv)  # LRC reads whole shards
        return [(i, 0, L) for i in range(self.tot) if hv[i]]


class Clay:
    family = "clay"

    def __init__(self, k, m, kind=VAND):
        self.k, self.m, self.kind, self.tot = k, m, kind, k + m
        self.alpha = CO.params(k, m)[4]
        self.P = CO.build(k, m, kind)
        self.lens = [u * 16 * self.alpha for u in CLAY_UNITS]
        self.stride = (max(CLAY_UNITS) + 1) * 16 * self.alpha
        self.key = ("clay", k, m)

    def ctx(self):
        return G.GarageEc.clay(0, self.k, self.m, self.kind)

    def encode(self, d):
        return CO.encode(self.k, self.m, self.P, d)

    def ok(self, present, want):
        return int(np.sum(present)) >= self.k  # MDS; fewer than k present is refused even with nothing wanted

    def oracle_decode(self, sh, present, want):
        out = sh.copy()
        absent = [i for i in range(self.tot) if not present[i]]
        wanted = _wanted(present, want)
        if len(absent) == 1 and wanted:
            out[absent[0]] = CO.repair_from_shards(self.k, self.m, self.P, sh, absent[0])
        elif wanted:
            full = CO.decode(self.k, self.m, self.P, sh, present)
            out[wanted] = full[wanted]
        return out

    def plan_pieces(self, ec, present, want, L):
        return ec.read_ranges(present, L, want=want)


def make_base(code, nseeds=2, seed=0):
    """(V, tot, stride) stripes encoded by the model, one per (length, seed), PAST beyond shard_len; (V,) lengths"""
    V = len(code.lens) * nseeds
    base = np.full((V, code.tot, code.stride), PAST, dtype=np.uint8)
    vl = np.zeros(V, dtype=np.uint32)
    for v in range(V):
        L = code.lens[v % len(code.lens)]
        d = O.fill_random(code.k * L, 0xDEC0 + 97 * seed + v).reshape(code.k, L)
        base[v, :code.k, :L] = d
        base[v, code.k:, :L] = code.encode(d)
        vl[v] = L
    return base, vl


def loss_patterns(tot, m, seed):
    """() , every 1- and 2-loss pattern, a seeded sample of 3..m losses, a few of m+1"""
    pats = [()] + [c for e in (1, 2) for c in itertools.combinations(range(tot), e)]
    rng = np.random.default_rng(seed)
    for j in range(12 * (m - 2)):
        pats.append(tuple(sorted(rng.choice(tot, 3 + j % (m - 2), replace=False).tolist())))
    for _ in range(4):
        pats.append(tuple(sorted(rng.choice(tot, m + 1, replace=False).tolist())))
    return pats


def layout(code, sms, n_min, seed):
    """(lost patterns, want masks) of a batch: [A: the patterns in runs of 1, 2, 3 equal stripes, repeated up to
    n_min - 2*sms] [C: sms stripes cycling the patterns backwards] [B: sms stripes losing shards 0 and tot-1 under
    changing want masks].  C and B are the last 2*sms stripes, the ones cut into chunk ranges."""
    k, m, tot = code.k, code.m, code.tot
    pats = loss_patterns(tot, m, seed)
    run = [p for i, p in enumerate(pats) for _ in range(1 + i % 3)]
    A = list(run)
    while len(A) + 2 * sms < n_min:
        A += run
    C = [pats[-1 - (i % len(pats))] for i in range(sms)]
    lost = A + C
    want = []
    for j, ls in enumerate(lost):
        w = np.ones(tot, dtype=np.uint8)
        if len(ls) <= m:
            if j % 3 == 1 and ls:
                w[:] = 0
                w[ls[(j // 3) % len(ls)]] = 1
            elif j % 3 == 2:
                w[k:] = 0  # GET: the data shards only
        want.append(w)
    rng = np.random.default_rng(seed + 1)
    for _ in range(sms):
        lost.append((0, tot - 1))
        w = np.zeros(tot, dtype=np.uint8)
        c = int(rng.integers(0, 3))
        w[[0] if c == 0 else [tot - 1] if c == 1 else [0, tot - 1]] = 1
        want.append(w)
    present = np.ones((len(lost), tot), dtype=np.uint8)
    for s, ls in enumerate(lost):
        present[s, list(ls)] = 0
    return lost, present, np.array(want)


def model_status(code, present, want):
    cache, ok = {}, np.zeros(len(present), dtype=bool)
    for s in range(len(present)):
        key = (present[s].tobytes(), None if want is None else want[s].tobytes())
        if key not in cache:
            cache[key] = code.ok(present[s], None if want is None else want[s])
        ok[s] = cache[key]
    return ok


def check(torch, got, orig, present, rebuilt, lens, what, broken=None, chunk=256):
    """got == the input stripes (orig with absent shards POISON, or `broken`), except the rebuilt shards:
    orig in [0, shard_len), zero in [shard_len, roundup16(shard_len)), untouched beyond"""
    n, tot, stride = got.shape
    col = torch.arange(stride, device=got.device)
    zero = torch.zeros((), dtype=torch.uint8, device=got.device)
    bad, nbad = [], 0
    for a in range(0, n, chunk):
        b = min(n, a + chunk)
        L = lens[a:b].long()[:, None, None]
        if broken is None:
            exp = orig[a:b].clone()
            exp[present[a:b] == 0] = POISON
        else:
            exp = broken[a:b].clone()
        rb = rebuilt[a:b][:, :, None]
        exp = torch.where(rb & (col < L), orig[a:b], exp)
        exp = torch.where(rb & (col >= L) & (col < (L + 15) // 16 * 16), zero, exp)
        diff = (got[a:b] != exp).any(dim=2).nonzero()
        nbad += len(diff)
        bad += [(a + s, i) for s, i in diff[:8].tolist()]
    assert not nbad, "%s: %d shards differ, first (stripe, shard): %s" % (what, nbad, bad[:8])


def run_batch(torch, ec, code, stripes, present, want, lens):
    """DEVICE reconstruct of a copy of `stripes`; (result, status)"""
    n = stripes.shape[0]
    d = stripes.clone()
    st = torch.full((n,), 99, dtype=torch.int32, device="cuda")
    ec.reconstruct(d.view(-1), dev(torch, present), code.stride, n, want=None if want is None else dev(torch, want),
                   status=st, shard_len=dev(torch, lens.astype(np.int32)))
    return d, st.cpu().numpy()


def geometry(torch, sms, code, seed):
    base, vl = make_base(code, seed=seed)
    V = len(vl)
    alpha = getattr(code, "alpha", 1)
    ips = -(-code.stride // (16 * alpha))
    n_min = max(2 * sms + 40, 16 * sms // ips + 40 if code.family == "clay" else 0)
    lost, present, want = layout(code, sms, n_min, seed)
    n = len(lost)
    assert n > 2 * sms and (code.family != "clay" or n * ips > 16 * sms)
    vidx = np.array([(5 * s + s // 7) % V for s in range(n)])
    lens = vl[vidx]
    orig = dev(torch, base)[dev(torch, vidx)]
    pd = dev(torch, present)
    broken = orig.clone()
    broken[pd == 0] = POISON
    rng = np.random.default_rng(seed + 2)
    with code.ctx() as ec:
        for mode in ("want=NULL", "want"):
            w = None if mode == "want=NULL" else want
            ok = model_status(code, present, w)
            if w is None:
                assert not ok[[len(ls) > code.m for ls in lost]].any()
            got, st = run_batch(torch, ec, code, broken, present, w, lens)
            what = "%s %s" % (code.key, mode)
            assert set(np.unique(st)) <= {0, G.E_UNRECOVERABLE}, what
            bad = np.nonzero((st == 0) != ok)[0]
            assert not len(bad), "%s: status %s, model %s at stripes %s" % (what, st[bad[:8]], ok[bad[:8]], bad[:8])
            wmask = np.ones_like(present) if w is None else w
            rebuilt = (present == 0) & (wmask != 0) & ok[:, None]
            check(torch, got, orig, pd, dev(torch, rebuilt).bool(), dev(torch, lens.astype(np.int32)), what)
            # the model rebuilds the same bytes from its own plan, on a seeded sample of multi-loss stripes
            multi = [s for s in range(n) if ok[s] and rebuilt[s].any() and len(lost[s]) >= 2]
            single = [s for s in range(n) if ok[s] and rebuilt[s].any() and len(lost[s]) == 1]
            for s in [int(x) for x in rng.choice(multi, 3, replace=False)] + [int(rng.choice(single))]:
                L = int(lens[s])
                sh = broken[s, :, :L].cpu().numpy()
                ref = code.oracle_decode(sh, present[s], None if w is None else w[s])
                assert np.array_equal(ref, got[s, :, :L].cpu().numpy()), (what, s, lost[s])
            if mode == "want" and code.key in HOST_CASES:
                # staged HOST mode on a pageable copy of the same batch: the same status and every byte the same
                h = broken.cpu().numpy()
                hs = np.full(n, 99, dtype=np.int32)
                ec.reconstruct(h.reshape(-1), present, code.stride, n, want=want, status=hs, shard_len=lens)
                assert np.array_equal(hs, st), what + " HOST status"
                diff = np.nonzero((h != got.cpu().numpy()).any(axis=2))
                assert not len(diff[0]), "%s: HOST differs from DEVICE at %s" % (what, list(zip(*diff))[:8])


# ---------------------------------------------------------------------------------------------- case table (CPU)
def test_case_table_reaches_every_shape():
    """the PB cases reach every PB apply instantiation (K = 2k, k = 1..16) with every m, all Cauchy; the Clay cases
    are valid codes with every m, with and without virtual nodes, the largest t and both largest alphas; the LRC
    cases include k > 16 and m = 8 (two passes); the lengths span 1, 2, 3 and 5+ stage rows with partial and
    one-column last chunks; the rank model used for status agrees with the oracles' own"""
    assert {2 * k for k, _, _ in PB_CASES} == set(range(2, 33, 2))
    assert {(k, m) for k, m, kind in PB_CASES if kind == CAUCHY} == {(k, m) for k in range(1, 17) for m in (2, 3, 4)}
    assert {kind for _, _, kind in PB_CASES} == {VAND, CAUCHY}
    for k, l, r in LRC_CASES:
        LO.build_lrc(k, l, r)
    assert any(k > 16 for k, _, _ in LRC_CASES) and any(l + r == 8 for _, l, r in LRC_CASES)
    assert any(k > 16 and l + r == 8 for k, l, r in LRC_CASES)
    params = [CO.params(k, m) for k, m in CLAY_CASES]  # raises for an invalid code
    assert {p[0] for p in params} == {2, 3, 4}
    for q in (2, 3, 4):
        assert {p[3] > 0 for p in params if p[0] == q} == {False, True}
    assert max(p[1] for p in params) == 8 and {243, 256} <= {p[4] for p in params} and max(p[3] for p in params) == 3
    rows = {-(-h // STAGE) for h in PB_HALVES}
    assert {1, 2, 3} <= rows and max(rows) >= 5
    assert any(h % STAGE for h in PB_HALVES) and any(h % STAGE == 16 for h in PB_HALVES)
    assert all(h % 16 == 0 for h in PB_HALVES)  # PB: shard_len % 32
    assert {-(-L // STAGE) for L in LRC_LENS} >= {1, 2, 3, 5} and {L & 15 for L in LRC_LENS} > {0}
    rng = np.random.default_rng(3)
    for code in (Lrc(8, 1, 3), Lrc(12, 3, 2), Pb(4, 3, CAUCHY), Pb(1, 4, CAUCHY)):
        for _ in range(40):
            pr = (rng.random(code.tot) > 0.3).astype(np.uint8)
            w = None if rng.random() < 0.5 else (rng.random(code.tot) > 0.5).astype(np.uint8)
            if code.family == "lrc":
                exp = LO.recoverable(code.k, code.P, pr, w)
            else:
                exp = PB.recoverable(code.k, code.m, code.P, pr, w)
            assert code.ok(pr, w) == exp, (code.key, pr, w)


# ---------------------------------------------------------------------------------------------- decode geometry
@pytest.mark.gpu
@pytest.mark.parametrize("k,m,kind", PB_CASES)
def test_pb_decode_geometry(torch, sms, k, m, kind):
    geometry(torch, sms, Pb(k, m, kind), 0x9B0 + 16 * k + m + 64 * kind)


@pytest.mark.gpu
@pytest.mark.parametrize("k,l,r", LRC_CASES)
def test_lrc_decode_geometry(torch, sms, k, l, r):
    geometry(torch, sms, Lrc(k, l, r), 0x1C0 + k + l)


@pytest.mark.gpu
@pytest.mark.parametrize("k,m", CLAY_CASES)
def test_clay_decode_geometry(torch, sms, k, m):
    geometry(torch, sms, Clay(k, m), 0xC1A + 4 * k + m)


# ---------------------------------------------------------------------------------------------- read plan only
@pytest.mark.gpu
@pytest.mark.parametrize("code", [Pb(13, 4, CAUCHY), Lrc(24, 6, 2), Clay(5, 4), Clay(12, 3)],
                         ids=lambda c: "-".join(map(str, c.key)))
def test_decode_from_the_host_plan_only(torch, sms, code):
    """every byte the host plan (read_plan halves for PB and LRC, read_ranges for Clay) does not name holds poison,
    absent shards and bytes past shard_len included; the kernel, given the real present map, rebuilds the same
    bytes"""
    base, vl = make_base(code, seed=5)
    V = len(vl)
    lost, present, want = layout(code, sms, 2 * sms + 40, 0x7A)
    ok = model_status(code, present, want)
    keep_s = [s for s in range(len(lost)) if ok[s] and len(lost[s]) <= code.m]
    present, want = present[keep_s], want[keep_s]
    n = len(keep_s)
    assert n > 2 * sms
    vidx = np.array([(3 * s + s // 5) % V for s in range(n)])
    lens = vl[vidx]
    keep = np.zeros((n, code.tot, code.stride), dtype=bool)
    cache = {}
    with code.ctx() as ec:
        for s in range(n):
            key = (present[s].tobytes(), want[s].tobytes(), int(lens[s]))
            if key not in cache:
                cache[key] = code.plan_pieces(ec, present[s], want[s], int(lens[s]))
            for i, off, ln in cache[key]:
                assert present[s, i] and off + ln <= lens[s]
                keep[s, i, off:off + ln] = True
        inside = np.arange(code.stride)[None, None, :] < lens[:, None, None]
        assert (inside & (present[:, :, None] != 0) & ~keep).any()  # some present bytes are not read
        orig = dev(torch, base)[dev(torch, vidx)]
        kd = dev(torch, keep)
        broken = torch.where(kd, orig, torch.full((), POISON, dtype=torch.uint8, device="cuda"))
        del kd
        got, st = run_batch(torch, ec, code, broken, present, want, lens)
        assert not st.any()
        rebuilt = (present == 0) & (want != 0)
        check(torch, got, orig, dev(torch, present), dev(torch, rebuilt).bool(), dev(torch, lens.astype(np.int32)),
              "%s plan only" % (code.key,), broken=broken)


# ---------------------------------------------------------------------------------------------- full size
@pytest.mark.gpu
@pytest.mark.parametrize("family", ["pb", "lrc"])
def test_full_size_multi_loss_decode(torch, family):
    """4096 x 1 MiB PB(10,4) / LRC(10,2,2), 1..m random losses per stripe; every byte against the pre-erasure copy
    (LRC stripes the rank model calls unrecoverable come back untouched), parity of a sample against the model"""
    k, m, n, B = 10, 4, 4096, 1 << 20
    tot = k + m
    code = Pb(k, m, VAND) if family == "pb" else Lrc(k, 2, 2)
    with code.ctx() as ec:
        if family == "pb":
            L = ec.code_shard_len(B)
            stride = L
        else:
            L = ec.shard_len(B)
            stride = ec.stride_for(L)
        lens = torch.full((n,), L, dtype=torch.int32, device="cuda")
        data = torch.empty(n * k * stride, dtype=torch.uint8, device="cuda")
        ec.fill_random(data, data.numel(), 0xF5D0, 0)
        data.view(n, k, stride)[:, :, L:] = 0
        par = torch.zeros(n * m * stride, dtype=torch.uint8, device="cuda")
        ec.encode(data, par, stride, n, shard_len=lens)
        shards = torch.cat([data.view(n, k, stride), par.view(n, m, stride)], dim=1).contiguous()
        del data, par
        for s in (0, 1777, n - 1):
            h = shards[s, :, :L].cpu().numpy()
            assert np.array_equal(code.encode(h[:k]), h[k:]), s
        orig = shards.clone()
        rng = np.random.default_rng(0xF5)
        present = np.ones((n, tot), dtype=np.uint8)
        for s in range(n):
            present[s, rng.choice(tot, int(rng.integers(1, m + 1)), replace=False)] = 0
        ok = model_status(code, present, None)
        assert ok.all() if family == "pb" else (ok.any() and not ok.all())
        pd = dev(torch, present)
        shards[pd == 0] = POISON
        st = torch.full((n,), 99, dtype=torch.int32, device="cuda")
        ec.reconstruct(shards.view(-1), pd, stride, n, status=st, shard_len=lens)
        st = st.cpu().numpy()
        assert np.array_equal(st == 0, ok) and set(np.unique(st)) <= {0, G.E_UNRECOVERABLE}
        rebuilt = dev(torch, (present == 0) & ok[:, None]).bool()
        check(torch, shards, orig, pd, rebuilt, lens, "%s full size" % (code.key,))


# ---------------------------------------------------------------------------------------------- scrub_repair
def adler8(body):
    """GARAGE_EC_SUM_ADLER8: 8 segments of roundup16(ceil(len/8)) bytes, zlib Adler-32 of each, little endian"""
    seg = (-(-len(body) // 8) + 15) // 16 * 16
    return b"".join(struct.pack("<I", zlib.adler32(body[j * seg:(j + 1) * seg])) for j in range(8))


@pytest.mark.gpu
@pytest.mark.parametrize("code", [Pb(7, 3, CAUCHY), Lrc(12, 3, 2), Clay(4, 3)], ids=lambda c: "-".join(map(str, c.key)))
def test_scrub_repair_multi_chunk(torch, sms, code):
    """adler8 tags computed with zlib; 0..m+1 corrupt shards per stripe at multi-chunk lengths: the corrupt ones are
    reported and, where the rank model allows, rebuilt; nothing else is written"""
    base, vl = make_base(code, seed=9)
    V, tot = len(vl), code.tot
    n = 2 * sms + 57
    vidx = np.array([(5 * s + s // 3) % V for s in range(n)])
    lens = vl[vidx]
    tags = np.array([[np.frombuffer(adler8(base[v, i, :vl[v]].tobytes()), dtype=np.uint8) for i in range(tot)]
                     for v in range(V)])
    sums = tags[vidx]
    rng = np.random.default_rng(0x5C)
    orig = dev(torch, base)[dev(torch, vidx)]
    bad = np.zeros((n, tot), dtype=np.uint8)
    flips = []
    for s in range(n):
        for i in rng.choice(tot, int(rng.integers(0, code.m + 2)), replace=False):
            bad[s, i] = 1
            flips.append((s, i, int(rng.integers(0, lens[s]))))
    broken = orig.clone()
    for s, i, off in flips:
        broken[s, i, off] ^= 0xFF
    ok = model_status(code, 1 - bad, None)
    assert ok.any() and not ok.all()
    with code.ctx() as ec:
        ec.set_sum_kind(G.SUM_ADLER8)
        got = broken.clone()
        bo = torch.zeros(n * tot, dtype=torch.uint8, device="cuda")
        st = torch.full((n,), 99, dtype=torch.int32, device="cuda")
        ec.scrub_repair(got.view(-1), dev(torch, sums), bo, code.stride, n, status=st,
                        shard_len=dev(torch, lens.astype(np.int32)))
        assert np.array_equal(bo.cpu().numpy().reshape(n, tot), bad)
        st = st.cpu().numpy()
        assert np.array_equal(st == 0, ok) and set(np.unique(st)) <= {0, G.E_UNRECOVERABLE}
        rebuilt = dev(torch, (bad != 0) & ok[:, None]).bool()
        check(torch, got, orig, dev(torch, 1 - bad), rebuilt, dev(torch, lens.astype(np.int32)),
              "%s scrub" % (code.key,), broken=broken)
