"""Ranged SSE-C opens on the GPU (DESIGN.md 2.7, 4.10): plaintext ranges of oracle-sealed blocks for every code, healthy
and under erasure patterns (shard 0 absent included, so the prefix is rebuilt), with every byte outside the planned
runs overwritten with garbage; DEVICE, HOST and gather forms, CUDA graph replay, batches whose (request, chunk) items
outrun the grid; tampered chunks, tags and prefixes failing their request alone, and wrong keys."""
import itertools
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import garage_b200 as G  # noqa: E402
import sse_c_oracle as O  # noqa: E402

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

CH, FR = 4096, 4112
CODES = {
    "rs10_4": lambda: G.GarageEc(0, 10, 4),
    "rs4_2": lambda: G.GarageEc(0, 4, 2),
    "lrc10_2_2": lambda: G.GarageEc.lrc(0, 10, 2, 2),
    "pb10_4": lambda: G.GarageEc.piggyback(0, 10, 4),
    "clay10_4": lambda: G.GarageEc.clay(0, 10, 4),
}
SIZES = [1 << 20, (1 << 20) - 977, 300001]
SENT = 0x5A


def _sealed_stripe(ec, P, seed):
    """(plaintext, key, B, the context's encode of B as one stripe, stride)"""
    rng = np.random.default_rng(seed)
    pt = rng.integers(0, 256, P, dtype=np.uint8)
    key, N = rng.bytes(32), rng.bytes(8)
    B = np.frombuffer(O.seal(key, N, pt.tobytes()), dtype=np.uint8)
    L = ec.code_shard_len(B.size)
    stride = ec.stride_for(L)
    par = np.zeros(ec.m * stride, dtype=np.uint8)
    ec.encode_blocks([B.copy()], par, stride)
    stripe = np.zeros((ec.k + ec.m, stride), dtype=np.uint8)
    for j in range(ec.k):
        piece = B[j * L:(j + 1) * L]
        stripe[j, :piece.size] = piece
    stripe[ec.k:] = par.reshape(ec.m, stride)
    return pt, np.frombuffer(key, dtype=np.uint8), B, stripe, stride


def _ranges(ec, P, B, seed):
    L = ec.code_shard_len(B.size)
    r = [(0, 4096), (4096 * 3, 4096), (4000, 200), (P - 10, 10), (12345 % P, 1), (0, P), (P, 0)]
    # across a data shard edge: the plaintext byte just before B position L
    c = (L - 8) // FR
    o = c * CH + min(CH - 1, (L - 8) % FR) - 40
    r.append((max(0, o), min(100, P - max(0, o))))
    rng = np.random.default_rng(seed)
    for _ in range(3):
        a = int(rng.integers(0, P))
        r.append((a, int(rng.integers(1, min(P - a, 70000) + 1))))
    return r


def _patterns(ec, seed):
    """absent patterns the code tolerates: healthy, every single shard, shard 0 with others, and m-sets -- every
    pattern of 2..m shards when k+m <= 8 (RS(4,2)), 6 seeded m-sets otherwise (C(14,4) = 1001 patterns of a 1 MiB
    stripe each would not fit one test's budget; the decode itself is tested over every pattern in its own suites)"""
    tot = ec.k + ec.m
    rng = np.random.default_rng(seed)
    pats = [()] + [(i,) for i in range(tot)]
    pats += [tuple(range(ec.m)), (0, ec.k), tuple(range(ec.k - ec.m // 2, ec.k + (ec.m + 1) // 2))]
    if tot <= 8:
        pats += [p for r in range(2, ec.m + 1) for p in itertools.combinations(range(tot), r)]
    else:
        pats += [tuple(sorted(rng.choice(tot, ec.m, replace=False))) for _ in range(6)]
    out = []
    clay = ec.clay_info()[0] != 0  # MDS, and read_set does not plan its repairs
    for p in dict.fromkeys(pats):
        pr = np.ones(tot, dtype=np.uint8)
        pr[list(p)] = 0
        if clay or not p or ec.read_set(pr, pr ^ 1) is not None:  # LRC: some m-sets do not decode
            out.append(pr)
    return out


def _planned_copy(ec, stripe, present, S, o, ln, stride, rng):
    """a stripe that holds only the planned runs; every other byte is garbage"""
    tot = ec.k + ec.m
    runs, _ = ec.open_range_plan(present, S, o, ln)
    assert runs is not None
    got = rng.integers(0, 256, (tot, stride), dtype=np.uint8)
    for sh, off, n in runs:
        assert present[sh]
        got[sh, off:off + n] = stripe[sh, off:off + n]
    return got


def _build(ec, P, seed):
    pt, key, B, stripe, stride = _sealed_stripe(ec, P, seed)
    rng = np.random.default_rng(seed + 1)
    reqs = []
    pats = _patterns(ec, seed)
    for pi, pr in enumerate(pats):
        rs = _ranges(ec, P, B, seed + pi)
        reqs += [(pr, o, ln) for o, ln in rs]
    n = len(reqs)
    tot = ec.k + ec.m
    shards = np.stack([_planned_copy(ec, stripe, pr, B.size, o, ln, stride, rng) for pr, o, ln in reqs])
    present = np.stack([pr for pr, _, _ in reqs])
    sealed = np.full(n, B.size, dtype=np.uint32)
    offs = np.array([o for _, o, _ in reqs], dtype=np.uint32)
    lens = np.array([ln for _, _, ln in reqs], dtype=np.uint32)
    keys = np.tile(key, (n, 1))
    return pt, shards.reshape(n, tot * stride), present, sealed, keys, offs, lens, stride


def _check_out(pt, out, out_stride, offs, lens, status, zero_tail):
    for s in range(len(offs)):
        o, ln = int(offs[s]), int(lens[s])
        assert status[s] == 0, (s, o, ln, status[s])
        row = out[s * out_stride:(s + 1) * out_stride]
        assert np.array_equal(row[:ln], pt[o:o + ln]), (s, o, ln)
        r16 = (ln + 15) // 16 * 16
        if zero_tail:
            assert not row[ln:r16].any(), (s, o, ln)
            assert (row[r16:] == SENT).all(), (s, o, ln)


@pytest.mark.parametrize("P", SIZES, ids=["1MiB", "1MiB-977", "300001"])
@pytest.mark.parametrize("code", list(CODES))
def test_open_range_matches_oracle_every_form(code, P):
    ec = CODES[code]()
    pt, shards, present, sealed, keys, offs, lens, stride = _build(ec, P, 11 + P % 97)
    n = len(offs)
    out_stride = (int(lens.max()) + 15) // 16 * 16
    # the whole-plaintext requests make cmax ~ 258 chunks: n * cmax items outrun the grid's warps many times over
    assert n * (out_stride // CH + 2) > 132 * 4 * 8

    # DEVICE, into a sentinel-filled output
    d_sh = torch.from_numpy(shards.reshape(-1)).cuda()
    d_pr = torch.from_numpy(present.reshape(-1)).cuda()
    d_S = torch.from_numpy(sealed.view(np.int32)).cuda()
    d_k = torch.from_numpy(keys.reshape(-1)).cuda()
    d_o = torch.from_numpy(offs.view(np.int32)).cuda()
    d_l = torch.from_numpy(lens.view(np.int32)).cuda()
    d_out = torch.full((n * out_stride,), SENT, dtype=torch.uint8, device="cuda")
    d_st = torch.full((n,), 99, dtype=torch.int32, device="cuda")
    ec.open_range(d_sh, d_pr, d_S, d_k, d_o, d_l, stride, d_out, out_stride, d_st)
    torch.cuda.synchronize()
    _check_out(pt, d_out.cpu().numpy(), out_stride, offs, lens, d_st.cpu().numpy(), True)
    del d_out

    # HOST contiguous
    h_out = np.full(n * out_stride, SENT, dtype=np.uint8)
    st = np.full(n, 99, dtype=np.int32)
    assert ec.open_range(shards.reshape(-1), present.reshape(-1), sealed, keys, offs, lens, stride, h_out, out_stride,
                         st) == 0
    _check_out(pt, h_out, out_stride, offs, lens, st, False)

    # HOST gather form: exactly len bytes written
    stripes = [np.ascontiguousarray(shards[s]) for s in range(n)]
    outs = [np.full(int(lens[s]) + 32, SENT, dtype=np.uint8) for s in range(n)]
    st = np.full(n, 99, dtype=np.int32)
    assert ec.open_range_stripes(stripes, present.reshape(-1), sealed, keys, offs, lens, stride, outs, st) == 0
    for s in range(n):
        o, ln = int(offs[s]), int(lens[s])
        assert st[s] == 0 and np.array_equal(outs[s][:ln], pt[o:o + ln]) and (outs[s][ln:] == SENT).all(), s
    ec.close()


def test_open_range_graph_replay():
    ec = CODES["rs10_4"]()
    pt, shards, present, sealed, keys, offs, lens, stride = _build(ec, 1 << 20, 5)
    n = len(offs)
    out_stride = (int(lens.max()) + 15) // 16 * 16
    d = [torch.from_numpy(a.reshape(-1).view(np.int32) if a.dtype == np.uint32 else a.reshape(-1)).cuda()
         for a in (shards, present, sealed, keys, offs, lens)]
    d_out = torch.full((n * out_stride,), SENT, dtype=torch.uint8, device="cuda")
    d_st = torch.full((n,), 99, dtype=torch.int32, device="cuda")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        ec.open_range(d[0], d[1], d[2], d[3], d[4], d[5], stride, d_out, out_stride, d_st)  # warm the pool
    torch.cuda.synchronize()
    d_out.fill_(SENT)
    d_st.fill_(99)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        ec.open_range(d[0], d[1], d[2], d[3], d[4], d[5], stride, d_out, out_stride, d_st)
    for _ in range(2):
        d_out.fill_(SENT)
        d_st.fill_(99)
        g.replay()
        torch.cuda.synchronize()
        _check_out(pt, d_out.cpu().numpy(), out_stride, offs, lens, d_st.cpu().numpy(), True)
    ec.close()


def test_open_range_plan_bytes():
    ec = CODES["rs10_4"]()
    P = 1 << 20
    S = G.sealed_len(P)
    L = ec.code_shard_len(S)
    tot = ec.k + ec.m
    healthy = np.ones(tot, dtype=np.uint8)
    runs, gpu = ec.open_range_plan(healthy, S, 4096 * 40, 4096)
    assert sum(r[2] for r in runs) == 8 + 4112 and gpu == 0
    runs, gpu = ec.open_range_plan(healthy, S, 4096 * 40 + 7, 4096)
    assert sum(r[2] for r in runs) == 8 + 2 * 4112 and gpu == 0
    assert ec.open_range_plan(healthy, S, 10, 0) == ([], 0)
    # shard 0 absent, range in a later shard: the prefix costs its own 16-byte window in k survivors
    pr = healthy.copy()
    pr[0] = 0
    runs, gpu = ec.open_range_plan(pr, S, 4096 * 100, 4096)
    assert gpu == 1
    prefix = [r for r in runs if r[1] < 16]
    assert len(prefix) == ec.k and all(r[2] == 16 for r in prefix), runs
    assert all(r[1] + r[2] <= L for r in runs)
    with pytest.raises(G.EcError) as e:
        ec.open_range_plan(healthy, S, P, 1)
    assert e.value.code == G.E_INVALID
    with pytest.raises(G.EcError) as e:
        ec.open_range_plan(healthy, S + 1, 0, 1)
    assert e.value.code == G.E_AUTH
    pr = healthy.copy()
    pr[:ec.m + 1] = 0
    assert ec.open_range_plan(pr, S, 0, 10) == (None, 1)
    ec.close()  # now, not when the collector breaks the pytest.raises traceback cycle (maybe inside a graph capture)


def test_tampering_fails_its_request_alone():
    ec = CODES["rs10_4"]()
    P = 1 << 20
    pt, key, B, stripe, stride = _sealed_stripe(ec, P, 77)
    S = B.size
    L = ec.code_shard_len(S)
    tot = ec.k + ec.m

    def flip(pos):  # B position -> a copy of the stripe with that byte flipped
        st = stripe.copy()
        st[pos // L, pos % L] ^= 0x40
        return st

    o = 4096 * 50 + 100  # touches chunks 50 and 51
    cases = [  # (stripe, offset, len, expected status)
        (stripe, o, 5000, 0),
        (flip(8 + FR * 50 + 7), o, 5000, G.E_AUTH),          # a touched chunk's ciphertext
        (flip(8 + FR * 51 + 4096 + 3), o, 5000, G.E_AUTH),   # a touched chunk's tag
        (flip(3), o, 5000, G.E_AUTH),                        # the nonce prefix
        (flip(8 + FR * 52 + 9), o, 5000, 0),                 # an untouched chunk: the range is still served
        (flip(8 + FR * 10), 4096 * 10 + 1, 3, G.E_AUTH),
        (stripe, 0, P, 0),
    ]
    n = len(cases) + 1
    shards = np.stack([c[0] for c in cases] + [stripe]).reshape(n, tot * stride)
    present = np.ones((n, tot), dtype=np.uint8)
    present[1, 0] = 0  # the prefix is rebuilt from parity, the tampered chunk is read as it is
    sealed = np.full(n, S, dtype=np.uint32)
    keys = np.tile(key, (n, 1))
    keys[-1, 0] ^= 1  # a wrong key
    offs = np.array([c[1] for c in cases] + [o], dtype=np.uint32)
    lens = np.array([c[2] for c in cases] + [5000], dtype=np.uint32)
    want = [c[3] for c in cases] + [G.E_AUTH]
    out_stride = P
    # DEVICE
    d_out = torch.full((n * out_stride,), SENT, dtype=torch.uint8, device="cuda")
    d_st = torch.zeros(n, dtype=torch.int32, device="cuda")
    ec.open_range(torch.from_numpy(shards.reshape(-1)).cuda(), torch.from_numpy(present.reshape(-1)).cuda(),
                  torch.from_numpy(sealed.view(np.int32)).cuda(), torch.from_numpy(keys.reshape(-1)).cuda(),
                  torch.from_numpy(offs.view(np.int32)).cuda(), torch.from_numpy(lens.view(np.int32)).cuda(), stride,
                  d_out, out_stride, d_st)
    torch.cuda.synchronize()
    out, st = d_out.cpu().numpy(), d_st.cpu().numpy()
    assert list(st) == want
    for s in range(n):
        row = out[s * out_stride:(s + 1) * out_stride]
        if want[s]:
            assert (row == SENT).all(), s
        else:
            assert np.array_equal(row[:lens[s]], pt[offs[s]:offs[s] + lens[s]]), s
    # HOST
    h_out = np.full(n * out_stride, SENT, dtype=np.uint8)
    h_st = np.zeros(n, dtype=np.int32)
    assert ec.open_range(shards.reshape(-1), present.reshape(-1), sealed, keys, offs, lens, stride, h_out, out_stride,
                         h_st) == G.E_AUTH
    assert list(h_st) == want
    for s in range(n):
        if want[s]:
            assert (h_out[s * out_stride:(s + 1) * out_stride] == SENT).all(), s
    ec.close()


def test_invalid_and_malformed_requests():
    ec = CODES["rs4_2"]()
    P = 50000
    pt, key, B, stripe, stride = _sealed_stripe(ec, P, 3)
    S = B.size
    tot = ec.k + ec.m
    n = 4
    shards = np.tile(stripe.reshape(1, -1), (n, 1))
    present = np.ones((n, tot), dtype=np.uint8)
    sealed = np.array([S, S, 8 + 3 * FR + 5, S], dtype=np.uint32)  # a length the framing cannot hold
    keys = np.tile(key, (n, 1))
    offs = np.array([100, P - 5, 0, P], dtype=np.uint32)
    lens = np.array([1000, 6, 10, 0], dtype=np.uint32)  # request 1 runs past P; request 3 is empty
    out_stride = 1024
    d_out = torch.full((n * out_stride,), SENT, dtype=torch.uint8, device="cuda")
    d_st = torch.zeros(n, dtype=torch.int32, device="cuda")
    ec.open_range(torch.from_numpy(shards.reshape(-1)).cuda(), torch.from_numpy(present.reshape(-1)).cuda(),
                  torch.from_numpy(sealed.view(np.int32)).cuda(), torch.from_numpy(keys.reshape(-1)).cuda(),
                  torch.from_numpy(offs.view(np.int32)).cuda(), torch.from_numpy(lens.view(np.int32)).cuda(), stride,
                  d_out, out_stride, d_st)
    torch.cuda.synchronize()
    out = d_out.cpu().numpy()
    assert list(d_st.cpu().numpy()) == [0, G.E_INVALID, G.E_AUTH, 0]
    assert np.array_equal(out[:1000], pt[100:1100])
    assert (out[out_stride:] == SENT).all()
    # HOST: a range past P is a caller error before any GPU work; a malformed length is a verdict
    h_out = np.zeros(n * out_stride, dtype=np.uint8)
    with pytest.raises(G.EcError) as e:
        ec.open_range(shards.reshape(-1), present.reshape(-1), sealed, keys, offs, lens, stride, h_out, out_stride,
                      np.zeros(n, dtype=np.int32))
    assert e.value.code == G.E_INVALID
    lens[1] = 5
    h_st = np.zeros(n, dtype=np.int32)
    assert ec.open_range(shards.reshape(-1), present.reshape(-1), sealed, keys, offs, lens, stride, h_out, out_stride,
                         h_st) == G.E_AUTH
    assert list(h_st) == [0, 0, G.E_AUTH, 0]
    assert np.array_equal(h_out[out_stride:out_stride + 5], pt[P - 5:])
    ec.close()  # now, not when the collector breaks the pytest.raises traceback cycle (maybe inside a graph capture)
