"""Decode geometry of RS, LRC, PB and Clay on the GPU, against the C oracle (RS) and the numpy models (lrc_oracle,
pb_oracle, clay_oracle).

Every compiled reconstruct shape of each code runs at per-stripe shard lengths whose shard (PB: half, Clay: layer)
spans one to six 512-byte stage rows with a partial last chunk and a one-column tail, in batches longer than twice
the SM count so the last stripes are cut into chunk ranges (Clay: more columns than the grid has CTAs).  Patterns:
every pattern of at most two losses, a seeded sample of 3..m, and m+1; want = NULL, one absent shard or the data
shards only; runs of equal patterns, and a block of one erasure pattern under changing want masks so the table
buffers are reused for equal plans and rebuilt for different ones.  Every rebuilt byte is compared with the
oracle-encoded stripe and every other byte, those past shard_len included, with what was there before.  RS also
runs empty stripes and want masks naming none of the absent shards.  Also: reads limited to the host plan, staged
HOST equal to DEVICE (for RS also the pinned zero-copy form and reconstruct_stripes), 4096 x 1 MiB PB(10,4),
LRC(10,2,2) and RS(10,4) decodes and a 1024 x 1 MiB RS(20,8) one under want masks, scrub_repair with adler8 tags
(RS also BLAKE2), and stripes whose shard_len exceeds the stride."""
import hashlib
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
# RS: every k of launch_apply's GEC_CASE list (plan mode runs K = k); m cycles through 1..8, so two-pass m (5..8)
# meets small, mid and large k, and the k = 7 LDG plan path and the k > 16 split staging run
RS_CASES = ([(k, 1 + (3 * k) % 8, VAND) for k in range(1, 33)]
            + [(k, m, CAUCHY) for k, m in [(1, 8), (4, 5), (7, 3), (10, 4), (12, 6), (16, 8), (23, 7), (32, 5)]])
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
# RS shard lengths: the LRC ones and an empty stripe, at a stride of six stage rows plus one column
RS_LENS = [0] + LRC_LENS
RS_STRIDE = 6 * STAGE + 16
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


class Rs:
    family = "rs"

    def __init__(self, k, m, kind):
        self.k, self.m, self.kind, self.tot = k, m, kind, k + m
        self.P = O.build_matrix(k, m, kind)
        self.lens = list(RS_LENS)
        self.stride = RS_STRIDE
        self.key = ("rs", k, m, kind)

    def ctx(self):
        return G.GarageEc(0, self.k, self.m, self.kind)

    def encode(self, d):
        k, L = d.shape
        if not L:
            return np.zeros((self.m, 0), dtype=np.uint8)
        return O.encode(k, self.m, self.P, np.ascontiguousarray(d).reshape(-1), L, 1).reshape(self.m, L)

    def ok(self, present, want):
        return int(np.sum(present)) >= self.k  # fewer than k present is refused even with nothing wanted (gf256.h)

    def oracle_decode(self, sh, present, want):
        out = sh.copy()
        L = sh.shape[1]
        if L:
            full = sh.copy()
            _, st = O.reconstruct(self.k, self.m, self.P, full.reshape(-1), present, L, 1)
            assert not st.any()
            wanted = _wanted(present, want)
            out[wanted] = full[wanted]
        return out

    def plan_pieces(self, ec, present, want, L):
        hv = ec.read_plan(present, want)
        first_k = [i for i in range(self.tot) if present[i]][:self.k]
        assert [i for i in range(self.tot) if hv[i]] == first_k and all(int(hv[i]) == 3 for i in first_k)
        assert np.flatnonzero(ec.read_set(present, want)).tolist() == first_k
        return [(i, 0, L) for i in first_k]


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
    if code.family == "rs":
        # RS only, among the whole stripes: want masks naming none of the absent shards (none at all, or present
        # shards only).  Past m losses that is E_UNRECOVERABLE, at most m it is status 0; either way nothing is written
        rng = np.random.default_rng(seed + 3)
        X = []
        for j in range(16):
            ls = tuple(sorted(rng.choice(tot, m + 1 if j % 2 else 1 + j // 2 % m, replace=False).tolist()))
            w = np.zeros(tot, dtype=np.uint8)
            if j % 4 >= 2:
                w[[i for i in range(tot) if i not in ls]] = 1
            X.append((ls, w))
        lost[len(A):len(A)] = [ls for ls, _ in X]
        want[len(A):len(A)] = [w for _, w in X]
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
            sample = [int(x) for x in rng.choice(multi, 3, replace=False)] if multi else []  # none for m = 1
            for s in sample + [int(rng.choice(single))]:
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
    # RS: plan mode launches rs_apply_kernel<K = k>: every k of the GEC_CASE list, every m, the k = 7 LDG path, the
    # split staging of k > 16 (1-table last groups at k = 17 and 25), two passes at small, mid and large k
    assert {k for k, _, _ in RS_CASES} == set(range(1, 33)) and {m for _, m, _ in RS_CASES} == set(range(1, 9))
    for lo, hi in ((1, 8), (9, 16), (17, 32)):
        assert any(lo <= k <= hi and m > 4 for k, m, _ in RS_CASES), (lo, hi)
    assert sum(kind == CAUCHY for _, _, kind in RS_CASES) == 8
    assert {(7, 3, CAUCHY), (23, 7, CAUCHY), (32, 5, CAUCHY)} <= set(RS_CASES)
    rows = {-(-L // STAGE) for L in RS_LENS}
    assert rows == set(range(7)) and RS_STRIDE == 6 * STAGE + 16 and max(RS_LENS) < RS_STRIDE
    assert {L % STAGE for L in RS_LENS} >= {1, 15, 16, 17} and {L & 15 for L in RS_LENS} > {0}
    rng = np.random.default_rng(5)
    for code in (Rs(1, 8, CAUCHY), Rs(10, 4, VAND), Rs(23, 7, CAUCHY)):
        for _ in range(40):
            pr = (rng.random(code.tot) > rng.random()).astype(np.uint8)
            w = None if rng.random() < 0.5 else (rng.random(code.tot) > 0.5).astype(np.uint8)
            sh = O.fill_random(code.tot * 32, int(rng.integers(1 << 30)))
            _, st = O.reconstruct(code.k, code.m, code.P, sh, pr, 32, 1)
            assert code.ok(pr, w) == (st[0] == 0), (code.key, pr, w)
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
@pytest.mark.parametrize("k,m,kind", RS_CASES, ids=["k%d-m%d-%s" % (k, m, "cauchy" if c else "vand")
                                                    for k, m, c in RS_CASES])
def test_rs_decode_geometry(torch, sms, k, m, kind):
    geometry(torch, sms, Rs(k, m, kind), 0x25D0 + 16 * k + m + 512 * kind)


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
@pytest.mark.parametrize("code", [Pb(13, 4, CAUCHY), Lrc(24, 6, 2), Clay(5, 4), Clay(12, 3), Rs(7, 3, VAND),
                                  Rs(10, 4, VAND), Rs(23, 7, CAUCHY), Rs(32, 8, VAND)],
                         ids=lambda c: "-".join(map(str, c.key)))
def test_decode_from_the_host_plan_only(torch, sms, code):
    """every byte the host plan (read_plan halves for PB and LRC, the first k present shards for RS, read_ranges for
    Clay) does not name holds poison,
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


# ---------------------------------------------------------------------------------------------- HOST forms
HOST_CHUNK = 48 << 20  # source bytes of one HOST pipeline chunk


@pytest.mark.gpu
@pytest.mark.parametrize("code", [Rs(10, 4, VAND), Rs(20, 8, CAUCHY)], ids=lambda c: "-".join(map(str, c.key)))
def test_rs_host_forms_equal_device(torch, sms, code):
    """staged HOST reconstruct from pageable memory, the zero-copy in-place form on a pinned buffer, and
    reconstruct_stripes with one array per stripe, over three and a half pipeline chunks of the geometry batch:
    the same status and every byte the same as DEVICE, which matches the model"""
    tot, stride = code.tot, code.stride
    base, vl = make_base(code, seed=11)
    V = len(vl)
    lost, present, want = layout(code, sms, -(-7 * HOST_CHUNK // (2 * tot * stride)), 0x4057)
    n = len(lost)
    assert n * tot * stride > 3 * HOST_CHUNK
    vidx = np.array([(7 * s + s // 5) % V for s in range(n)])
    lens = vl[vidx]
    orig = dev(torch, base)[dev(torch, vidx)]
    pd = dev(torch, present)
    broken = orig.clone()
    broken[pd == 0] = POISON
    ok = model_status(code, present, want)
    assert ok.any() and not ok.all()
    with code.ctx() as ec:
        got, st = run_batch(torch, ec, code, broken, present, want, lens)
        assert np.array_equal(st == 0, ok) and set(np.unique(st)) <= {0, G.E_UNRECOVERABLE}
        rebuilt = (present == 0) & (want != 0) & ok[:, None]
        check(torch, got, orig, pd, dev(torch, rebuilt).bool(), dev(torch, lens.astype(np.int32)), "%s DEVICE" % (code.key,))
        exp = got.cpu().numpy()
        hb = broken.cpu().numpy()
        del orig, broken, got
        pin, handle = ec.host_alloc(hb.size)
        try:
            for form in ("pageable", "pinned", "stripes"):
                hs = np.full(n, 99, dtype=np.int32)
                if form == "pageable":
                    h = hb.copy()
                    ec.reconstruct(h.reshape(-1), present, stride, n, want=want, status=hs, shard_len=lens)
                elif form == "pinned":
                    pin[:] = hb.reshape(-1)
                    ec.reconstruct(pin, present, stride, n, want=want, status=hs, shard_len=lens)
                    h = pin.reshape(n, tot, stride)
                else:
                    arrs = [hb[s].copy() for s in range(n)]
                    ec.reconstruct_stripes(arrs, present, stride, want=want, status=hs, shard_len=lens)
                    h = np.stack(arrs)
                what = "%s HOST %s" % (code.key, form)
                assert np.array_equal(hs, st), what + " status"
                diff = np.nonzero((h != exp).any(axis=2))
                assert not len(diff[0]), "%s: differs from DEVICE at %s" % (what, list(zip(*diff))[:8])
        finally:
            ec.host_free(handle)


# ---------------------------------------------------------------------------------------------- full size
@pytest.mark.gpu
@pytest.mark.parametrize("family", ["pb", "lrc", "rs", "rs-20-8-want"])
def test_full_size_multi_loss_decode(torch, family):
    """4096 x 1 MiB PB(10,4) / LRC(10,2,2) / RS(10,4), 1..m random losses per stripe, and 1024 x 1 MiB RS(20,8) with
    1..8 losses under per-stripe want masks (two passes, split staging); every byte against the pre-erasure copy
    (LRC stripes the rank model calls unrecoverable come back untouched), parity of a sample against the model"""
    k, m, n, B = (20, 8, 1024, 1 << 20) if family == "rs-20-8-want" else (10, 4, 4096, 1 << 20)
    tot = k + m
    code = {"pb": lambda: Pb(k, m, VAND), "lrc": lambda: Lrc(k, 2, 2)}.get(family, lambda: Rs(k, m, VAND))()
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
        for s in (0, 1777 % n, n - 1):
            h = shards[s, :, :L].cpu().numpy()
            assert np.array_equal(code.encode(h[:k]), h[k:]), s
        orig = shards.clone()
        rng = np.random.default_rng(0xF5)
        present = np.ones((n, tot), dtype=np.uint8)
        for s in range(n):
            present[s, rng.choice(tot, int(rng.integers(1, m + 1)), replace=False)] = 0
        want = None
        if family == "rs-20-8-want":  # every absent shard, one of them, the data shards only, or a random subset
            want = np.ones((n, tot), dtype=np.uint8)
            for s in range(n):
                ab = np.nonzero(present[s] == 0)[0]
                if s % 4 == 1:
                    want[s] = 0
                    want[s, ab[s % len(ab)]] = 1
                elif s % 4 == 2:
                    want[s, k:] = 0
                elif s % 4 == 3:
                    want[s] = rng.random(tot) < 0.5
        ok = model_status(code, present, want)
        assert ok.all() if family != "lrc" else (ok.any() and not ok.all())
        pd = dev(torch, present)
        shards[pd == 0] = POISON
        st = torch.full((n,), 99, dtype=torch.int32, device="cuda")
        ec.reconstruct(shards.view(-1), pd, stride, n, want=None if want is None else dev(torch, want), status=st,
                       shard_len=lens)
        st = st.cpu().numpy()
        assert np.array_equal(st == 0, ok) and set(np.unique(st)) <= {0, G.E_UNRECOVERABLE}
        wmask = np.ones_like(present) if want is None else want
        rebuilt = dev(torch, (present == 0) & (wmask != 0) & ok[:, None]).bool()
        check(torch, shards, orig, pd, rebuilt, lens, "%s full size" % (code.key,))


# ---------------------------------------------------------------------------------------------- scrub_repair
def adler8(body):
    """GARAGE_EC_SUM_ADLER8: 8 segments of roundup16(ceil(len/8)) bytes, zlib Adler-32 of each, little endian"""
    seg = (-(-len(body) // 8) + 15) // 16 * 16
    return b"".join(struct.pack("<I", zlib.adler32(body[j * seg:(j + 1) * seg])) for j in range(8))


def tag(kind, body):
    return hashlib.blake2b(body).digest()[:32] if kind == G.SUM_BLAKE2 else adler8(body)


def base_tags(kind, base, vl, tot):
    """(V, tot, 32) tags of the model-encoded stripes, hashlib / zlib"""
    return np.array([[np.frombuffer(tag(kind, base[v, i, :vl[v]].tobytes()), dtype=np.uint8) for i in range(tot)]
                     for v in range(len(vl))])


@pytest.mark.gpu
@pytest.mark.parametrize("code", [Pb(7, 3, CAUCHY), Lrc(12, 3, 2), Clay(4, 3), Rs(10, 4, VAND), Rs(17, 8, VAND)],
                         ids=lambda c: "-".join(map(str, c.key)))
def test_scrub_repair_multi_chunk(torch, sms, code):
    """adler8 tags computed with zlib (RS also BLAKE2 tags from hashlib, in one batch under and one over the 24 000
    shards where the one-thread kernel takes over from the quad kernel); 0..m+1 corrupt shards per stripe at
    multi-chunk lengths: the corrupt ones are reported and, where the rank model allows, rebuilt; nothing else is
    written"""
    base, vl = make_base(code, seed=9)
    V, tot = len(vl), code.tot
    runs = [(G.SUM_ADLER8, 2 * sms + 57)]
    if code.family == "rs":
        runs += [(G.SUM_BLAKE2, 2 * sms + 57), (G.SUM_BLAKE2, 24000 // tot + 2 * sms)]
        assert runs[1][1] * tot < 24000 < runs[2][1] * tot
    for kind, n in runs:
        vidx = np.array([(5 * s + s // 3) % V for s in range(n)])
        lens = vl[vidx]
        sums = base_tags(kind, base, vl, tot)[vidx]
        rng = np.random.default_rng(0x5C)
        orig = dev(torch, base)[dev(torch, vidx)]
        bad = np.zeros((n, tot), dtype=np.uint8)
        flips = []
        for s in range(n):
            for i in rng.choice(tot, int(rng.integers(0, code.m + 2)) if lens[s] else 0, replace=False):
                bad[s, i] = 1
                flips.append((s, i, int(rng.integers(0, lens[s]))))
        broken = orig.clone()
        for s, i, off in flips:
            broken[s, i, off] ^= 0xFF
        ok = model_status(code, 1 - bad, None)
        assert ok.any() and not ok.all()
        with code.ctx() as ec:
            ec.set_sum_kind(kind)
            got = broken.clone()
            bo = torch.zeros(n * tot, dtype=torch.uint8, device="cuda")
            st = torch.full((n,), 99, dtype=torch.int32, device="cuda")
            ec.scrub_repair(got.view(-1), dev(torch, sums), bo, code.stride, n, status=st,
                            shard_len=dev(torch, lens.astype(np.int32)))
            assert np.array_equal(bo.cpu().numpy().reshape(n, tot), bad), (kind, n)
            st = st.cpu().numpy()
            assert np.array_equal(st == 0, ok) and set(np.unique(st)) <= {0, G.E_UNRECOVERABLE}, (kind, n)
            rebuilt = dev(torch, (bad != 0) & ok[:, None]).bool()
            check(torch, got, orig, dev(torch, 1 - bad), rebuilt, dev(torch, lens.astype(np.int32)),
                  "%s scrub kind %d n %d" % (code.key, kind, n), broken=broken)


# ---------------------------------------------------------------------------------------------- malformed lengths
@pytest.mark.gpu
@pytest.mark.parametrize("code", [Rs(10, 4, VAND), Rs(20, 8, CAUCHY), Lrc(12, 3, 2), Pb(10, 4, VAND), Clay(4, 3)],
                         ids=lambda c: "-".join(map(str, c.key)))
def test_shard_len_past_the_stride(torch, sms, code):
    """stripes whose shard_len exceeds the stride, in the middle of a batch and followed by intact stripes: DEVICE
    reconstruct and scrub_repair report E_INVALID for them (scrub: every shard bad) and write nothing of them or of
    their neighbours, DEVICE shard_sums leaves their tags alone and check_sums flags all their shards (adler8, and
    BLAKE2 under and over 24 000 shards); every other stripe is right.  HOST reconstruct, scrub_repair, shard_sums and
    check_sums return E_INVALID.  Lengths keep the code's framing (PB: % 32, Clay: % 16*alpha), so only the stride
    check can reject them.  Device buffers are one stripe longer than the batch: a kernel that ignores the stride reads
    and writes neighbour bytes, never outside the buffer"""
    tot, stride = code.tot, code.stride
    unit = {"pb": 32, "clay": 16 * getattr(code, "alpha", 1)}.get(code.family, 1)
    over = [stride + unit, stride + 16 * unit, stride + 97 * unit] if unit > 1 else [stride + 1, stride + 16, stride + 512]
    base, vl = make_base(code, seed=0x57)
    V = len(vl)
    n = 2 * sms + 37
    vidx = np.array([(5 * s + s // 7) % V for s in range(n)])
    lens = vl[vidx].astype(np.uint32)
    mal = [n // 3, n // 2, n // 2 + 1, 2 * n // 3]
    for j, s in enumerate(mal):
        lens[s] = over[j % len(over)]
    bad_len = np.zeros(n, dtype=bool)
    bad_len[mal] = True
    dl = dev(torch, lens.astype(np.int32))
    rng = np.random.default_rng(0x57)
    present = np.ones((n, tot), dtype=np.uint8)
    for s in range(n):
        present[s, rng.choice(tot, 1 + s % code.m, replace=False)] = 0
    ok = model_status(code, present, None)
    orig = dev(torch, base)[dev(torch, vidx)]
    GUARD = 0x5A
    with code.ctx() as ec:
        # reconstruct
        pd = dev(torch, present)
        broken = orig.clone()
        broken[pd == 0] = POISON
        d = torch.full((n + 1, tot, stride), GUARD, dtype=torch.uint8, device="cuda")
        d[:n] = broken
        st = torch.full((n + 1,), 99, dtype=torch.int32, device="cuda")
        ec.reconstruct(d.view(-1), pd, stride, n, status=st, shard_len=dl)
        st = st.cpu().numpy()
        exp_st = np.where(bad_len, G.E_INVALID, np.where(ok, 0, G.E_UNRECOVERABLE))
        assert np.array_equal(st[:n], exp_st), (st[mal], np.nonzero(st[:n] != exp_st)[0][:8])
        assert st[n] == 99 and (d[n] == GUARD).all(), "reconstruct wrote past the batch"
        rebuilt = (present == 0) & (ok & ~bad_len)[:, None]
        check(torch, d[:n], orig, pd, dev(torch, rebuilt).bool(), dl, "%s reconstruct" % (code.key,), broken=broken)

        h = broken.cpu().numpy()
        with pytest.raises(G.EcError) as e:
            ec.reconstruct(h.reshape(-1), present, stride, n, shard_len=lens)
        assert e.value.code == G.E_INVALID, "HOST reconstruct"
        del d, broken

        for kind in (G.SUM_ADLER8, G.SUM_BLAKE2):
            ec.set_sum_kind(kind)
            tags = base_tags(kind, base, vl, tot)[vidx]
            # scrub_repair: one corrupt shard per intact stripe
            flips = [(s, int(rng.integers(0, tot)), int(rng.integers(0, lens[s])))
                     for s in range(n) if lens[s] and not bad_len[s]]
            broken = orig.clone()
            exp_bad = np.zeros((n, tot), dtype=np.uint8)
            for s, i, off in flips:
                broken[s, i, off] ^= 0xFF
                exp_bad[s, i] = 1
            exp_bad[mal] = 1
            d = torch.full((n + 1, tot, stride), GUARD, dtype=torch.uint8, device="cuda")
            d[:n] = broken
            bo = torch.full(((n + 1) * tot,), 7, dtype=torch.uint8, device="cuda")
            st = torch.full((n + 1,), 99, dtype=torch.int32, device="cuda")
            ec.scrub_repair(d.view(-1), dev(torch, tags), bo, stride, n, status=st, shard_len=dl)
            what = "%s scrub kind %d" % (code.key, kind)
            bo = bo.cpu().numpy()
            assert np.array_equal(bo[:n * tot].reshape(n, tot), exp_bad), (what, bo.reshape(-1, tot)[mal])
            assert (bo[n * tot:] == 7).all(), what
            st = st.cpu().numpy()
            assert np.array_equal(st[:n], np.where(bad_len, G.E_INVALID, 0)), (what, st[mal])
            assert st[n] == 99 and (d[n] == GUARD).all(), what + ": wrote past the batch"
            rebuilt = (exp_bad != 0) & ~bad_len[:, None]
            check(torch, d[:n], orig, None, dev(torch, rebuilt).bool(), dl, what, broken=broken)
            hb = broken.cpu().numpy()
            with pytest.raises(G.EcError) as e:
                ec.scrub_repair(hb.reshape(-1), tags, np.zeros(n * tot, dtype=np.uint8), stride, n,
                                status=np.zeros(n, dtype=np.int32), shard_len=lens)
            assert e.value.code == G.E_INVALID, what + " HOST"
            del d, broken

            # shard_sums / check_sums of the clean batch, repeated past 24 000 shards for BLAKE2's one-thread kernel
            for reps in ((1, 24000 // (n * tot) + 1) if kind == G.SUM_BLAKE2 else (1,)):
                N = n * reps
                d = torch.full((N + 1, tot, stride), GUARD, dtype=torch.uint8, device="cuda")
                d[:N] = orig.repeat(reps, 1, 1)
                L = dev(torch, np.tile(lens, reps).astype(np.int32))
                mask = np.tile(bad_len, reps)
                sums = torch.full(((N + 1) * tot * 32,), POISON, dtype=torch.uint8, device="cuda")
                ec.shard_sums(d.view(-1), sums, stride, N, tot, shard_len=L)
                exp = np.tile(tags, (reps, 1, 1))
                exp[mask] = POISON
                got = sums.cpu().numpy().reshape(N + 1, tot, 32)
                wrong = np.nonzero((got[:N] != exp).any(axis=2))
                assert not len(wrong[0]), "%s sums x%d at %s" % (what, reps, list(zip(*wrong))[:8])
                assert (got[N] == POISON).all(), what
                bo = torch.full(((N + 1) * tot,), 7, dtype=torch.uint8, device="cuda")
                ec.check_sums(d.view(-1), dev(torch, np.concatenate([np.tile(tags, (reps, 1, 1)).reshape(-1),
                                                                    np.zeros(tot * 32, dtype=np.uint8)])),
                              bo, stride, N, tot, shard_len=L)
                bo = bo.cpu().numpy()
                assert np.array_equal(bo[:N * tot].reshape(N, tot), np.repeat(mask[:, None], tot, axis=1)), what
                assert (bo[N * tot:] == 7).all(), what
                del d
            h = orig.cpu().numpy()
            for call in ("shard_sums", "check_sums"):
                out = np.full(n * tot * 32 if call == "shard_sums" else n * tot, 7, dtype=np.uint8)
                with pytest.raises(G.EcError) as e:
                    if call == "shard_sums":
                        ec.shard_sums(h.reshape(-1), out, stride, n, tot, shard_len=lens)
                    else:
                        ec.check_sums(h.reshape(-1), tags, out, stride, n, tot, shard_len=lens)
                assert e.value.code == G.E_INVALID and (out == 7).all(), "%s HOST %s" % (what, call)
