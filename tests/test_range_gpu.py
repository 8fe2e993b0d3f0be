"""Ranged reads on the GPU (DESIGN.md section 2.5): garage_ec_range_plan names every byte garage_ec_decode_range reads,
and decode_range -- HOST, DEVICE and the gather form -- returns exactly the block's bytes [offset, offset + len), for
RS, LRC, PB and Clay, every erasure pattern of the small codes and sampled ones of the large codes, ranges at the
start, across shard, PB half and Clay layer boundaries, at the end and over the whole block.  Every shard byte outside
the planned runs is garbage, so a decode that read anything else would differ."""
import itertools
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import garage_b200 as G  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch():
    import torch as t

    assert t.cuda.is_available()
    return t


CODES = {
    "rs4_2": (lambda: G.GarageEc(0, 4, 2), True),
    "rs10_4": (lambda: G.GarageEc(0, 10, 4), False),
    "lrc10_2_2": (lambda: G.GarageEc.lrc(0, 10, 2, 2), False),
    "pb10_4": (lambda: G.GarageEc.piggyback(0, 10, 4), False),
    "clay6_3": (lambda: G.GarageEc.clay(0, 6, 3), True),
    "clay10_4": (lambda: G.GarageEc.clay(0, 10, 4), False),
}


def alpha_of(ec):
    return ec.clay_info()[2]


def is_pb(ec):
    return ec.piggyback_info()[0] > 0


def encode(ec, blocks):
    """shard layout of the blocks under ec's code: (n, k+m, stride) and the stride"""
    k, m = ec.k, ec.m
    Ls = [ec.code_shard_len(b.size) for b in blocks]
    stride = max(ec.stride_for(L) for L in Ls)
    n = len(blocks)
    par = np.zeros(n * m * stride, dtype=np.uint8)
    ec.encode_blocks(blocks, par, stride)
    sh = np.zeros((n, k + m, stride), dtype=np.uint8)
    for s, (b, L) in enumerate(zip(blocks, Ls)):
        flat = np.zeros(k * L, dtype=np.uint8)
        flat[:b.size] = b
        sh[s, :k, :L] = flat.reshape(k, L)
    sh[:, k:, :] = par.reshape(n, m, stride)
    return sh, stride


def ranges_for(ec, B):
    L = ec.code_shard_len(B)
    out = [(0, 1), (0, B), (B - 100, 100), (L - 5, 10), (2 * L - 1, 2), (B // 3, 4096)]
    if is_pb(ec):
        out += [(L // 2 - 7, 20), (L + L // 2 - 1, 3)]
    a = alpha_of(ec)
    if a > 1:
        u = L // a
        out += [(u - 3, 9), (L + 2 * u - 3, 9), (3 * u + 5, u)]
    rng = np.random.default_rng(B)
    for _ in range(2):
        o = int(rng.integers(0, B))
        out.append((o, int(rng.integers(1, B - o + 1))))
    return sorted({(o, n) for o, n in out if o >= 0 and n >= 1 and o + n <= B})


def patterns(ec, exhaustive, seed):
    tot = ec.k + ec.m
    pats = []
    if exhaustive:
        for e in range(ec.m + 1):
            pats += [set(c) for c in itertools.combinations(range(tot), e)]
        return pats
    rng = np.random.default_rng(seed)
    pats = [set(), {0}, {ec.k - 1}, {1, ec.k + 1}, set(range(ec.m))]
    if ec.code_info()[0]:  # LRC: a whole local group's data shard and its group parity
        pats += [{0, ec.k}, {2, 7}]
    if is_pb(ec):  # rule 1: one data shard; rule 2: data + parity 1
        pats += [{4}, {4, ec.k + 1}]
    for _ in range(6):
        pats.append(set(int(x) for x in rng.choice(tot, int(rng.integers(1, ec.m + 1)), replace=False)))
    return pats


def run_batch(torch, ec, sh, stride, blocks, reqs, pat, rng):
    """reqs: [(stripe, off, len)].  Every request gets its own copy of its stripe with garbage outside the planned
    runs; HOST, DEVICE and the gather form must all return the block's bytes (or status UNRECOVERABLE)."""
    tot = ec.k + ec.m
    n = len(reqs)
    present = np.ones(tot, dtype=np.uint8)
    present[list(pat)] = 0
    work = rng.integers(0, 256, (n, tot, stride), dtype=np.uint8)
    expect_status = np.zeros(n, dtype=np.int32)
    for r, (s, off, ln) in enumerate(reqs):
        B = blocks[s].size
        L = ec.code_shard_len(B)
        runs, needs = ec.range_plan(present, B, off, ln)
        touched_absent = any(not present[j] for j in range(off // L, (off + ln - 1) // L + 1))
        assert needs == int(touched_absent), (pat, off, ln)
        if runs is None:
            expect_status[r] = G.E_UNRECOVERABLE
            continue
        for (i, o, b) in runs:
            assert present[i] and o + b <= L
            work[r, i, o:o + b] = sh[s, i, o:o + b]
        if not touched_absent:
            assert runs == [(j, max(off, j * L) - j * L, min(off + ln, (j + 1) * L) - max(off, j * L))
                            for j in range(off // L, (off + ln - 1) // L + 1)]
    blen = np.array([blocks[s].size for s, _, _ in reqs], dtype=np.uint32)
    offs = np.array([o for _, o, _ in reqs], dtype=np.uint32)
    lens = np.array([ln for _, _, ln in reqs], dtype=np.uint32)
    pres = np.tile(present, (n, 1))
    ostride = (int(lens.max()) + 15) // 16 * 16

    def check(out, status, what):
        assert np.array_equal(status, expect_status), (what, pat, status, expect_status)
        for r, (s, off, ln) in enumerate(reqs):
            if expect_status[r] == 0:
                assert np.array_equal(out[r][:ln], blocks[s][off:off + ln]), (what, pat, off, ln)

    # HOST
    out = np.full((n, ostride), 0xEE, dtype=np.uint8)
    st = np.full(n, 7, dtype=np.int32)
    ec.decode_range(work.reshape(-1), pres, blen, offs, lens, stride, out.reshape(-1), ostride, status=st)
    check(out, st, "host")
    for r in np.nonzero(expect_status)[0]:
        assert (out[r] == 0xEE).all()
    # gather form
    outs = [np.full(int(ln), 0xEE, dtype=np.uint8) for ln in lens]
    st2 = np.full(n, 7, dtype=np.int32)
    ec.decode_range_stripes([work[r] for r in range(n)], pres, blen, offs, lens, stride, outs, status=st2)
    check(outs, st2, "stripes")
    # DEVICE
    d = torch.from_numpy(work.reshape(-1)).cuda()
    dout = torch.full((n * ostride,), 0xEE, dtype=torch.uint8, device="cuda")
    dst = torch.full((n,), 7, dtype=torch.int32, device="cuda")
    to_dev = lambda a: torch.from_numpy(a.view(np.int32) if a.dtype == np.uint32 else a).cuda()  # noqa: E731
    ec.decode_range(d, to_dev(pres), to_dev(blen), to_dev(offs), to_dev(lens), stride, dout, ostride, status=dst)
    torch.cuda.synchronize()
    check(dout.cpu().numpy().reshape(n, ostride), dst.cpu().numpy(), "device")
    assert torch.equal(d.cpu(), torch.from_numpy(work.reshape(-1))), "DEVICE decode_range wrote the shards"


@pytest.mark.parametrize("code", list(CODES))
def test_decode_range_equals_block_slice(torch, code):
    make, exhaustive = CODES[code]
    with make() as ec:
        sizes = [100_003, 4097, 17] if exhaustive else [1 << 20, 1_000_003, 5000]
        rng = np.random.default_rng(len(code))
        blocks = [rng.integers(0, 256, b, dtype=np.uint8) for b in sizes]
        sh, stride = encode(ec, blocks)
        reqs = [(s, o, n) for s, b in enumerate(blocks) for (o, n) in ranges_for(ec, b.size)]
        for pat in patterns(ec, exhaustive, 11):
            run_batch(torch, ec, sh, stride, blocks, reqs, pat, rng)


def test_byte_counts_follow_the_window_formulas(torch):
    B = 1 << 20
    with G.GarageEc(0, 10, 4) as ec:
        L = ec.code_shard_len(B)
        present = np.ones(14, dtype=np.uint8)
        off = 3 * L + 1000
        runs, needs = ec.range_plan(present, B, off, 4096)
        assert needs == 0 and runs == [(3, 1000, 4096)]
        # one segment boundary crossed, one shard boundary crossed: the range bytes only
        runs, needs = ec.range_plan(present, B, 4 * L - 2000, 4096)
        assert needs == 0 and sum(r[2] for r in runs) == 4096 and [r[0] for r in runs] == [3, 4]
        present[3] = 0
        runs, needs = ec.range_plan(present, B, off, 4096)
        assert needs == 1
        w = runs[0][2]
        assert w <= 4096 + 32 and w % 16 == 0 and runs[0][1] % 16 == 0
        assert [r[0] for r in runs] == [0, 1, 2, 4, 5, 6, 7, 8, 9, 10]
        assert all(r[2] == w for r in runs) and sum(r[2] for r in runs) == 10 * w
    with G.GarageEc.clay(0, 10, 4) as ec:
        L = ec.code_shard_len(B)
        present = np.ones(14, dtype=np.uint8)
        present[3] = 0
        runs, needs = ec.range_plan(present, B, 3 * L + 1000, 4096)
        assert needs == 1 and sum(r[2] for r in runs) == 346_112  # the whole-shard repair: 13 x L / 4
        assert runs == ec.read_ranges(present, L)
    with G.GarageEc.piggyback(0, 10, 4) as ec:
        L = ec.code_shard_len(B)
        present = np.ones(14, dtype=np.uint8)
        present[0] = 0
        runs, _ = ec.range_plan(present, B, 64, 4096)
        halves = ec.read_plan(present, want=np.array([1] + [0] * 13, dtype=np.uint8))
        w = 4096 + 64 - 64
        expect = []
        for i in range(14):
            if halves[i] & 1:
                expect.append((i, 64, w))
            if halves[i] & 2:
                expect.append((i, L // 2 + 64, w))
        merged = []
        for r in expect:
            if merged and merged[-1][0] == r[0] and merged[-1][1] + merged[-1][2] == r[1]:
                merged[-1] = (r[0], merged[-1][1], merged[-1][2] + r[2])
            else:
                merged.append(r)
        assert runs == merged


def test_unrecoverable_and_invalid(torch):
    B = 300_000
    rng = np.random.default_rng(5)
    blocks = [rng.integers(0, 256, B, dtype=np.uint8)]
    with G.GarageEc(0, 4, 2) as ec:
        sh, stride = encode(ec, blocks)
        L = ec.code_shard_len(B)
        # three absent: a range in shard 0 cannot be rebuilt; one in present shard 3 is served without the GPU
        run_batch(torch, ec, sh, stride, blocks, [(0, 10, 100), (0, 3 * L + 5, 100), (0, L - 1, 2)], {0, 1, 2}, rng)
        present = np.array([0, 0, 0, 1, 1, 1], dtype=np.uint8)
        assert ec.range_plan(present, B, 10, 100) == (None, 1)
        with pytest.raises(G.EcError) as ei:
            ec.range_plan(present, B, B - 1, 2)
        assert ei.value.code == G.E_INVALID
        one = lambda v: np.array([v], dtype=np.uint32)  # noqa: E731
        out = np.zeros(64, dtype=np.uint8)
        with pytest.raises(G.EcError) as ei:
            ec.decode_range(sh.reshape(-1), np.ones(6, np.uint8), one(B), one(B - 1), one(2), stride, out, 64)
        assert ei.value.code == G.E_INVALID
        d = torch.from_numpy(sh.reshape(-1)).cuda()
        dst = torch.zeros(1, dtype=torch.int32, device="cuda")
        dev = lambda a: torch.from_numpy(a.view(np.int32)).cuda()  # noqa: E731
        dout = torch.zeros(64, dtype=torch.uint8, device="cuda")
        ec.decode_range(d, torch.ones(6, dtype=torch.uint8, device="cuda"), dev(one(B)), dev(one(B - 1)), dev(one(2)),
                        stride, dout, 64, status=dst)
        torch.cuda.synchronize()
        assert int(dst[0]) == G.E_INVALID


def test_device_call_replays_in_a_cuda_graph(torch):
    B = 1 << 20
    rng = np.random.default_rng(9)
    blocks = [rng.integers(0, 256, B, dtype=np.uint8) for _ in range(4)]
    with G.GarageEc(0, 10, 4) as ec:
        sh, stride = encode(ec, blocks)
        n = len(blocks)
        present = np.ones((n, 14), dtype=np.uint8)
        present[:, [2, 11]] = 0
        ec_off = np.array([2 * 104858 - 7, 5, 700_000, 0], dtype=np.uint32)
        ec_len = np.array([65536, 4096, 300_000, B], dtype=np.uint32)
        ostride = B
        d = torch.from_numpy(sh.reshape(-1)).cuda()
        dev = lambda a: torch.from_numpy(a.view(np.int32) if a.dtype == np.uint32 else a).cuda()  # noqa: E731
        args = (d, dev(present), dev(np.full(n, B, np.uint32)), dev(ec_off), dev(ec_len), stride)
        dout = torch.zeros(n * ostride, dtype=torch.uint8, device="cuda")
        dst = torch.full((n,), 7, dtype=torch.int32, device="cuda")
        ec.decode_range(*args, dout, ostride, status=dst)  # warm-up outside the capture
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            ec.decode_range(*args, dout, ostride, status=dst)
        dout.zero_()
        dst.fill_(7)
        g.replay()
        torch.cuda.synchronize()
        assert int(dst.abs().sum()) == 0
        o = dout.cpu().numpy().reshape(n, ostride)
        for s in range(n):
            assert np.array_equal(o[s, :ec_len[s]], blocks[s][ec_off[s]:ec_off[s] + ec_len[s]])


@pytest.mark.parametrize("fail_at", [0, 2, 4, 7, 11])
def test_host_fault_leaves_caller_buffers_alone(torch, fail_at):
    """requests spread over several pipeline chunks; after a failed HOST call returns, nothing writes the output"""
    k, m, B, n = 4, 2, 1 << 19, 256
    rng = np.random.default_rng(21)
    blocks = [rng.integers(0, 256, B, dtype=np.uint8)]
    with G.GarageEc(0, k, m) as ec:
        sh, stride = encode(ec, blocks)
        work = np.ascontiguousarray(np.broadcast_to(sh[0], (n, k + m, stride)))
        present = np.ones((n, k + m), dtype=np.uint8)
        present[:, 1] = 0
        blen = np.full(n, B, np.uint32)
        offs = np.array([int(x) for x in rng.integers(0, B // 2, n)], dtype=np.uint32)
        lens = np.full(n, B // 2, np.uint32)
        ostride = B // 2
        out = np.zeros(n * ostride, dtype=np.uint8)
        ec.decode_range(work.reshape(-1), present, blen, offs, lens, stride, out, ostride)
        want = np.concatenate([blocks[0][o:o + B // 2] for o in offs])
        assert np.array_equal(out, want)
        ec.debug_fail_after(fail_at)
        with pytest.raises(G.EcError):
            ec.decode_range(work.reshape(-1), present, blen, offs, lens, stride, out, ostride)
        ec.debug_fail_after(-1)
        out[:] = 0xEE
        torch.cuda.synchronize()
        assert (out == 0xEE).all(), "a D2H copy completed after the failed call had returned"
        ec.decode_range(work.reshape(-1), present, blen, offs, lens, stride, out, ostride)
        assert np.array_equal(out, want)
