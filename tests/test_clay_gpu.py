"""Clay(k, m) contexts on the GPU, checked against the numpy model (tests/clay_oracle.py): encode / verify bit-exact,
HOST equal to DEVICE, decode of every erasure pattern in one batch, single-shard repair from the read_ranges runs
only, malformed lengths, scrub_repair, the block-level calls with a short last block, transcode to and from Clay,
and a full-size 4096 x 1 MiB Clay(10,4) round trip."""
import itertools
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import clay_oracle as CO  # noqa: E402
import oracle_lib as O  # noqa: E402

import garage_b200 as G  # noqa: E402

pytestmark = pytest.mark.gpu
POISON = 0xA5


@pytest.fixture(scope="module")
def torch():
    import torch as t

    assert t.cuda.is_available()
    return t


def dev(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def make_stripes(k, m, kind, n, stride, lens, seed):
    """(P, shards (n, k+m, stride)) encoded by the numpy model, zero past shard_len"""
    P = CO.build(k, m, kind)
    data = O.fill_random(n * k * stride, seed).reshape(n, k, stride)
    sh = np.zeros((n, k + m, stride), dtype=np.uint8)
    for s in range(n):
        L = int(lens[s])
        data[s, :, L:] = 0
        sh[s, :k] = data[s]
        sh[s, k:, :L] = CO.encode(k, m, P, data[s, :, :L])
    return P, sh


def ragged(alpha, n, units):
    q = 16 * alpha
    lens = np.array([q * (1 + (7 * i) % units) for i in range(n)], dtype=np.uint32)
    lens[0] = q * units
    return lens, q * units


@pytest.mark.parametrize("kind", [0, 1])
@pytest.mark.parametrize("k,m", [(4, 2), (6, 3), (8, 4), (10, 3), (10, 4), (12, 4)])
def test_clay_encode_verify_bit_exact(torch, k, m, kind):
    q, t, _, s_virt, alpha = CO.params(k, m)
    n = 12
    lens, stride = ragged(alpha, n, 3)
    P, ref = make_stripes(k, m, kind, n, stride, lens, 0xC1A0 + k + 64 * kind)
    with G.GarageEc.clay(0, k, m, kind) as ec:
        qq, tt, aa, ss, base = ec.clay_info()
        assert (qq, tt, aa, ss) == (q, t, alpha, s_virt) and np.array_equal(base, P)
        assert ec.code_shard_len(1 << 20) == CO.shard_len(1 << 20, k, m)
        par = torch.full((n * m * stride,), POISON, dtype=torch.uint8, device="cuda")
        ec.encode(dev(torch, ref[:, :k]), par, stride, n, shard_len=dev(torch, lens))
        got = par.cpu().numpy().reshape(n, m, stride)
        for s in range(n):
            L = int(lens[s])
            assert np.array_equal(got[s, :, :L], ref[s, k:, :L]), s
            assert (got[s, :, L:] == POISON).all(), s
        mm = torch.ones(n, dtype=torch.int32, device="cuda")
        ec.verify(dev(torch, ref), mm, stride, n, shard_len=dev(torch, lens))
        assert not mm.cpu().numpy().any()
        bad = ref.copy()
        for s in range(n):
            bad[s, k + s % m, (37 * s) % int(lens[s])] ^= 0x5A
        ec.verify(dev(torch, bad), mm, stride, n, shard_len=dev(torch, lens))
        assert [int(x) for x in mm.cpu().numpy()] == [1 << (s % m) for s in range(n)]
        hp = np.zeros(n * m * stride, dtype=np.uint8)
        ec.encode(np.ascontiguousarray(ref[:, :k]).reshape(-1), hp, stride, n, shard_len=lens)
        hp = hp.reshape(n, m, stride)
        for s in range(n):
            assert np.array_equal(hp[s, :, :int(lens[s])], ref[s, k:, :int(lens[s])])
        hm = np.ones(n, dtype=np.uint32)
        ec.verify(bad.reshape(-1), hm, stride, n, shard_len=lens)
        assert [int(x) for x in hm] == [1 << (s % m) for s in range(n)]


def _patterns(tot, m):
    return [er for e in range(1, m + 1) for er in itertools.combinations(range(tot), e)]


@pytest.mark.parametrize("k,m", [(4, 2), (6, 3), (10, 4)])
def test_clay_decode_every_pattern_in_one_batch(torch, k, m):
    tot = k + m
    alpha = CO.params(k, m)[4]
    pats = _patterns(tot, m)
    if (k, m) == (10, 4):
        assert len(pats) == 1470  # every 1..4-loss pattern of 14 shards
    n = len(pats)
    L = stride = 16 * alpha
    P = CO.build(k, m)
    data = O.fill_random(k * L * 4, 0xC1A7 + k).reshape(4, k, L)
    base = np.stack([np.concatenate([d, CO.encode(k, m, P, d)]) for d in data])
    ref = np.stack([base[i % 4] for i in range(n)])
    present = np.ones((n, tot), dtype=np.uint8)
    for s, er in enumerate(pats):
        present[s, list(er)] = 0
    broken = ref.copy()
    broken[present == 0] = POISON
    d = dev(torch, broken)
    status = torch.full((n,), 99, dtype=torch.int32, device="cuda")
    ec = G.GarageEc.clay(0, k, m)
    ec.reconstruct(d.view(-1), dev(torch, present), stride, n, status=status)
    assert not status.cpu().numpy().any()
    assert np.array_equal(d.cpu().numpy(), ref)
    # m+1 losses: unrecoverable, stripe untouched
    pr = np.ones((1, tot), dtype=np.uint8)
    pr[0, :m + 1] = 0
    one = broken[:1].copy()
    one[0, :m + 1] = POISON
    d1 = dev(torch, one)
    st1 = torch.zeros(1, dtype=torch.int32, device="cuda")
    ec.reconstruct(d1.view(-1), dev(torch, pr), stride, 1, status=st1)
    assert int(st1[0]) == G.E_UNRECOVERABLE and np.array_equal(d1.cpu().numpy(), one)
    ec.close()


@pytest.mark.parametrize("mode", ["device", "host", "stripes"])
@pytest.mark.parametrize("k,m", [(4, 2), (5, 3), (10, 4), (10, 3)])
def test_clay_repair_reads_only_the_runs(torch, k, m, mode):
    """every byte outside garage_ec_read_ranges' runs holds poison; the rebuilt shard is still exact"""
    tot = k + m
    alpha = CO.params(k, m)[4]
    L = stride = 16 * alpha * 2
    P = CO.build(k, m)
    data = O.fill_random(k * L, 0xC1AB + k).reshape(k, L)
    full = np.concatenate([data, CO.encode(k, m, P, data)])
    with G.GarageEc.clay(0, k, m) as ec:
        n = tot
        shards = np.full((n, tot, stride), POISON, dtype=np.uint8)
        present = np.ones((n, tot), dtype=np.uint8)
        want = np.zeros((n, tot), dtype=np.uint8)
        fetched = 0
        for f in range(tot):
            present[f, f] = 0
            want[f, f] = 1
            runs = ec.read_ranges(present[f], L, want=want[f])
            assert runs == [(i, off, ln) for i in range(tot) if i != f for off, ln in _merged(CO.repair_runs(k, m, f, L))]
            for i, off, ln in runs:
                shards[f, i, off:off + ln] = full[i, off:off + ln]
                fetched += ln
            assert np.array_equal(CO.repair_from_shards(k, m, P, shards[f][:, :L], f), full[f])
        assert fetched == tot * (tot - 1) * L // m
        status = np.full(n, 99, dtype=np.int32)
        if mode == "device":
            d = dev(torch, shards)
            sd = torch.full((n,), 99, dtype=torch.int32, device="cuda")
            ec.reconstruct(d.view(-1), dev(torch, present), stride, n, want=dev(torch, want), status=sd)
            got, status = d.cpu().numpy(), sd.cpu().numpy()
        elif mode == "host":
            got = shards.copy()
            ec.reconstruct(got.reshape(-1), present, stride, n, want=want, status=status)
        else:
            got = [shards[s].reshape(-1).copy() for s in range(n)]
            ec.reconstruct_stripes(got, present, stride, want=want, status=status)
            got = np.stack(got).reshape(n, tot, stride)
        assert not status.any()
        for f in range(tot):
            assert np.array_equal(got[f, f], full[f]), f


def _merged(runs):
    out = []
    for off, ln in runs:
        if out and out[-1][0] + out[-1][1] == off:
            out[-1] = (out[-1][0], out[-1][1] + ln)
        else:
            out.append((off, ln))
    return out


def test_clay_read_ranges_and_read_set(torch):
    k, m = 10, 4
    tot = k + m
    L = CO.shard_len(1 << 20, k, m)
    assert L == 106496
    with G.GarageEc.clay(0, k, m) as ec:
        for f in range(tot):
            pr = np.ones(tot, dtype=np.uint8)
            pr[f] = 0
            runs = ec.read_ranges(pr, L)
            assert sum(r[2] for r in runs) == 13 * 26624
            assert list(ec.read_set(pr)) == list(pr)
        pr = np.ones(tot, dtype=np.uint8)
        pr[[1, 12]] = 0
        assert ec.read_ranges(pr, L) == [(i, 0, L) for i in [0, 2, 3, 4, 5, 6, 7, 8, 9, 10]]
        pr[[2, 3, 4]] = 0
        assert ec.read_ranges(pr, L) is None
        with pytest.raises(G.EcError):
            ec.read_ranges(np.ones(tot, dtype=np.uint8), L + 16)
        with pytest.raises(G.EcError):
            ec.matrix()
        with pytest.raises(G.EcError):
            ec.read_plan(pr)
    with G.GarageEc(0, 10, 4) as rs:
        assert rs.clay_info()[:4] == (0, 0, 1, 0)
        pr = np.ones(tot, dtype=np.uint8)
        pr[3] = 0
        assert rs.read_ranges(pr, 1000) == [(i, 0, 1000) for i in range(tot) if i != 3][:10]
    with G.GarageEc.piggyback(0, 10, 4) as pb:
        pr = np.ones(tot, dtype=np.uint8)
        pr[3] = 0
        halves = pb.read_plan(pr)
        want = [(i, (0 if h != 2 else 64), (128 if h == 3 else 64)) for i, h in enumerate(halves) if h]
        assert pb.read_ranges(pr, 128) == want


def test_clay_host_equals_device_and_malformed(torch):
    k, m = 6, 3
    tot = k + m
    alpha = CO.params(k, m)[4]
    n = 40
    lens, stride = ragged(alpha, n, 4)
    P, ref = make_stripes(k, m, 0, n, stride, lens, 0xC1B0)
    rng = np.random.default_rng(5)
    present = np.ones((n, tot), dtype=np.uint8)
    for s in range(n):
        present[s, rng.choice(tot, 1 + s % m, replace=False)] = 0
    broken = ref.copy()
    broken[present == 0] = POISON
    with G.GarageEc.clay(0, k, m) as ec:
        d = dev(torch, broken)
        sd = torch.full((n,), 99, dtype=torch.int32, device="cuda")
        ec.reconstruct(d.view(-1), dev(torch, present), stride, n, status=sd, shard_len=dev(torch, lens))
        h = broken.copy()
        sh = np.full(n, 99, dtype=np.int32)
        ec.reconstruct(h.reshape(-1), present, stride, n, status=sh, shard_len=lens)
        assert not sd.cpu().numpy().any() and not sh.any()
        dd = d.cpu().numpy()
        for s in range(n):
            L = int(lens[s])
            assert np.array_equal(dd[s, :, :L], ref[s, :, :L]) and np.array_equal(h[s, :, :L], ref[s, :, :L]), s
        # a length that is not a multiple of 16*alpha: DEVICE reports E_INVALID for the stripe, HOST refuses the call
        badl = lens.copy()
        badl[3] -= 16
        sd.fill_(99)
        ec.reconstruct(dev(torch, broken).view(-1), dev(torch, present), stride, n, status=sd, shard_len=dev(torch, badl))
        assert int(sd[3]) == G.E_INVALID
        with pytest.raises(G.EcError):
            ec.reconstruct(broken.copy().reshape(-1), present, stride, n, shard_len=badl)
        mm = torch.zeros(n, dtype=torch.int32, device="cuda")
        ec.verify(dev(torch, ref), mm, stride, n, shard_len=dev(torch, badl))
        assert [int(x) for x in mm.cpu().numpy()] == [7 if s == 3 else 0 for s in range(n)]


def test_clay_scrub_repair(torch):
    k, m = 10, 4
    tot = k + m
    alpha = CO.params(k, m)[4]
    n = 6
    lens, stride = ragged(alpha, n, 2)
    P, ref = make_stripes(k, m, 0, n, stride, lens, 0xC1B5)
    with G.GarageEc.clay(0, k, m) as ec:
        ec.set_sum_kind(G.SUM_ADLER8)
        sums = np.zeros(n * tot * 32, dtype=np.uint8)
        ec.shard_sums(ref.reshape(-1), sums, stride, n, tot, shard_len=lens)
        broken = ref.copy()
        lost = [[0], [13], [1, 2, 3, 4], [], [5, 6, 7, 8, 9], [11, 12]]
        badmask = np.zeros((n, tot), dtype=np.uint8)
        for s, ls in enumerate(lost):
            for i in ls:
                broken[s, i, 5] ^= 0x11
                badmask[s, i] = 1
        got = broken.copy()
        bo = np.zeros(n * tot, dtype=np.uint8)
        status = np.full(n, 99, dtype=np.int32)
        ec.scrub_repair(got.reshape(-1), sums, bo, stride, n, status=status, shard_len=lens)
        assert np.array_equal(bo.reshape(n, tot), badmask)
        assert [int(x) for x in status] == [0, 0, 0, 0, G.E_UNRECOVERABLE, 0]
        for s in range(n):
            L = int(lens[s])
            exp = broken[s] if s == 4 else ref[s]
            assert np.array_equal(got[s, :, :L], exp[:, :L]), s


def test_clay_blocks_and_transcode(torch):
    """encode_blocks / decode_blocks frame with the Clay shard length (a short last block included); transcode
    RS(6,3) -> Clay(10,4), whole blocks -> Clay(10,4) and Clay(10,4) -> RS(10,4) equal the oracles' encodes"""
    k, m = 10, 4
    tot = k + m
    blocks = [O.fill_random(bl, 0xC1C0 + i) for i, bl in enumerate([1 << 20, 777777, 16384, 31, 65536])]
    n = len(blocks)
    lens = [b.size for b in blocks]
    P = CO.build(k, m)
    with G.GarageEc.clay(0, k, m) as ec:
        Ls = [ec.code_shard_len(b) for b in lens]
        assert Ls == [CO.shard_len(b, k, m) for b in lens]
        stride = max(Ls)
        parity = np.zeros(n * m * stride, dtype=np.uint8)
        ec.encode_blocks(blocks, parity, stride)
        clay = np.zeros((n, tot, stride), dtype=np.uint8)
        for s, b in enumerate(blocks):
            L = Ls[s]
            flat = np.zeros(k * L, dtype=np.uint8)
            flat[:b.size] = b
            clay[s, :k, :L] = flat.reshape(k, L)
            clay[s, k:, :L] = CO.encode(k, m, P, clay[s, :k, :L])
            assert np.array_equal(parity.reshape(n, m, stride)[s, :, :L], clay[s, k:, :L]), s
        present = np.ones((n, tot), dtype=np.uint8)
        broken = clay.copy()
        for s, lost in enumerate([[3], [0, 5, 12, 13], [9], [1], [1, 2, 3, 4, 10]]):
            present[s, lost] = 0
            broken[s, lost] = POISON
        outs = [np.zeros(b, dtype=np.uint8) for b in lens]
        status = np.full(n, 99, dtype=np.int32)
        ec.decode_blocks(broken.reshape(-1), present, lens, stride, outs, status=status)
        assert list(status) == [0, 0, 0, 0, G.E_UNRECOVERABLE]
        for s in range(4):
            assert np.array_equal(outs[s], blocks[s]), s
        # transcodes into Clay(10,4), DEVICE and HOST
        with G.GarageEc(0, 6, 3) as rs63:
            rL = [rs63.code_shard_len(b) for b in lens]
            rstride = (max(rL) + 127) // 128 * 128
            src = np.zeros((n, 9, rstride), dtype=np.uint8)
            for s, b in enumerate(blocks):
                flat = np.zeros(6 * rL[s], dtype=np.uint8)
                flat[:b.size] = b
                src[s, :6, :rL[s]] = flat.reshape(6, rL[s])
            for mode in ("device", "host"):
                dst = np.zeros((n, tot, stride), dtype=np.uint8)
                if mode == "device":
                    dd = dev(torch, dst)
                    ec.transcode(rs63, dev(torch, src).view(-1), dev(torch, np.array(lens, dtype=np.uint32)), rstride,
                                 dd.view(-1), stride, n)
                    dst = dd.cpu().numpy()
                else:
                    ec.transcode(rs63, src.reshape(-1), np.array(lens, dtype=np.uint32), rstride, dst.reshape(-1), stride, n)
                for s in range(n):
                    assert np.array_equal(dst[s, :, :Ls[s]], clay[s, :, :Ls[s]]), (mode, s)
        wstride = (max(lens) + 127) // 128 * 128
        whole = np.zeros((n, wstride), dtype=np.uint8)
        for s, b in enumerate(blocks):
            whole[s, :b.size] = b
        dst = np.zeros((n, tot, stride), dtype=np.uint8)
        ec.transcode(None, whole.reshape(-1), np.array(lens, dtype=np.uint32), wstride, dst.reshape(-1), stride, n)
        for s in range(n):
            assert np.array_equal(dst[s, :, :Ls[s]], clay[s, :, :Ls[s]]), s
        # Clay(10,4) -> RS(10,4), from a degraded Clay stripe
        with G.GarageEc(0, k, m) as rs:
            rL = [rs.code_shard_len(b) for b in lens]
            rstride = (max(rL) + 127) // 128 * 128
            pr = np.ones((n, tot), dtype=np.uint8)
            pr[0, 4] = 0
            pr[1, [0, 1, 2, 11]] = 0
            src = clay.copy()
            src[pr == 0] = POISON
            out = np.zeros((n, tot, rstride), dtype=np.uint8)
            ec_rc = rs.transcode(ec, src.reshape(-1), np.array(lens, dtype=np.uint32), stride, out.reshape(-1), rstride, n,
                                 src_present=pr)
            assert ec_rc == 0
            RP = O.build_matrix(k, m, 0)
            for s, b in enumerate(blocks):
                L = rL[s]
                flat = np.zeros(k * L, dtype=np.uint8)
                flat[:b.size] = b
                d = flat.reshape(k, L)
                assert np.array_equal(out[s, :k, :L], d), s
                par = O.encode(k, m, RP, np.ascontiguousarray(d).reshape(-1), L, 1).reshape(m, L)
                assert np.array_equal(out[s, k:, :L], par), s


def test_clay_full_size_round_trip(torch):
    """4096 x 1 MiB Clay(10,4): DEVICE encode, then a batch mixing 4-loss decodes and 1-loss repairs; 64 stripes are
    compared byte for byte with the oracle's encode"""
    k, m = 10, 4
    tot = k + m
    n, B = 4096, 1 << 20
    with G.GarageEc.clay(0, k, m) as ec:
        L = ec.code_shard_len(B)
        stride = L
        data = torch.empty((n, k, stride), dtype=torch.uint8, device="cuda")
        ec.fill_random(data, n * k * stride, 0xC1D0)
        par = torch.zeros((n, m, stride), dtype=torch.uint8, device="cuda")
        ec.encode(data.view(-1), par.view(-1), stride, n)
        sh = torch.cat([data, par], dim=1).contiguous()
        P = CO.build(k, m)
        d_np = data[:64].cpu().numpy()
        p_np = par[:64].cpu().numpy()
        for s in range(64):
            assert np.array_equal(p_np[s], CO.encode(k, m, P, d_np[s])), s
        ref = sh.clone()
        rng = np.random.default_rng(9)
        present = np.ones((n, tot), dtype=np.uint8)
        for s in range(n):
            present[s, rng.choice(tot, m if s % 2 else 1, replace=False)] = 0
        pd = dev(torch, present)
        sh[~pd.bool()] = POISON
        status = torch.full((n,), 99, dtype=torch.int32, device="cuda")
        ec.reconstruct(sh.view(-1), pd, stride, n, status=status)
        assert not status.cpu().numpy().any()
        assert torch.equal(sh, ref)
