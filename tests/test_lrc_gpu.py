"""LRC(k, l, r) contexts on the GPU: encode / verify bit-exact against the CPU oracles, reconstruct of every
erasure pattern against the rank model (tests/lrc_oracle.py), local repair that reads only the shard's group,
the survivor set garage_ec_read_set reports, scrub_repair and the block-level decode on LRC contexts."""
import hashlib
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import lrc_oracle as LO  # noqa: E402
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


def make_stripes(k, l, r, n, stride, lens, seed):
    """(P, shards (n, k+m, stride)) encoded by the C oracle with the LRC parity rows, zero past shard_len"""
    m = l + r
    P = LO.build_lrc(k, l, r)
    data = O.fill_random(n * k * stride, seed).reshape(n, k, stride)
    for s in range(n):
        data[s, :, lens[s]:] = 0
    par = O.encode(k, m, P, data.reshape(-1), stride, n, lens)
    sh = np.concatenate([data, par.reshape(n, m, stride)], axis=1)
    return P, np.ascontiguousarray(sh)


@pytest.mark.parametrize("k,l,r", [(6, 2, 2), (10, 2, 2), (12, 2, 2), (16, 4, 2), (20, 4, 4)])
def test_lrc_encode_verify_bit_exact(torch, k, l, r):
    m, n, stride = l + r, 24, 4096 + 64
    lens = np.array([1 + (977 * i) % stride for i in range(n)], dtype=np.uint32)
    lens[0] = stride
    P, ref = make_stripes(k, l, r, n, stride, lens, 0x1C0 + k)
    with G.GarageEc.lrc(0, k, l, r) as ec:
        assert np.array_equal(ec.matrix(), P)
        assert ec.code_info() == (l, r) and ec.m == m
        par = torch.zeros(n * m * stride, dtype=torch.uint8, device="cuda")
        ec.encode(dev(torch, ref[:, :k]), par, stride, n, shard_len=dev(torch, lens))
        got = par.cpu().numpy().reshape(n, m, stride)
        assert np.array_equal(got, ref[:, k:])
        gs = k // l
        for s in (0, n - 1):  # local parity = plain XOR of its group, no GF arithmetic
            for g in range(l):
                assert np.array_equal(got[s, g], np.bitwise_xor.reduce(ref[s, g * gs:(g + 1) * gs], axis=0))
        mm = torch.ones(n, dtype=torch.int32, device="cuda")
        d = dev(torch, ref)
        ec.verify(d, mm, stride, n, shard_len=dev(torch, lens))
        assert not mm.cpu().numpy().any()
        bad = ref.copy()
        for s in range(n):
            bad[s, k + s % m, int(lens[s]) // 2] ^= 0x5A
        ec.verify(dev(torch, bad), mm, stride, n, shard_len=dev(torch, lens))
        assert [int(x) for x in mm.cpu().numpy()] == [1 << (s % m) for s in range(n)]


def _patterns(tot):
    return [np.array([(p >> i) & 1 ^ 1 for i in range(tot)], dtype=np.uint8) for p in range(1 << tot)]


@pytest.mark.parametrize("k,l,r", [(6, 2, 2), (10, 2, 2)])
@pytest.mark.parametrize("single", [False, True])
def test_lrc_reconstruct_every_pattern(torch, k, l, r, single):
    """every erasure pattern; want = NULL, or each absent shard alone; status follows the rank test and the
    rebuilt bytes equal the encoded ones (and the numpy oracle's decode on a sample)"""
    m = l + r
    tot, stride = k + m, 64
    P = LO.build_lrc(k, l, r)
    G_rows = LO.generator_rows(k, P)
    present_l, want_l, ok_l = [], [], []
    for pr in _patterns(tot):
        B = LO.Basis(k)
        for i in range(tot):
            if pr[i] and len(B.rows) < k:
                B.add(G_rows[i])
        absent = [o for o in range(tot) if not pr[o]]
        if not single:
            present_l.append(pr)
            want_l.append(np.ones(tot, dtype=np.uint8))
            ok_l.append(len(B.rows) == k or all(B.express(G_rows[o]) is not None for o in absent))
        else:
            for o in absent:
                w = np.zeros(tot, dtype=np.uint8)
                w[o] = 1
                present_l.append(pr)
                want_l.append(w)
                ok_l.append(B.express(G_rows[o]) is not None)
    n = len(present_l)
    present, want, ok = np.array(present_l), np.array(want_l), np.array(ok_l)
    lens = np.array([1 + (13 * i) % stride for i in range(n)], dtype=np.uint32)
    _, orig = make_stripes(k, l, r, n, stride, lens, 0x2C0 + k + single)
    broken = orig.copy()
    broken[present == 0] = POISON
    with G.GarageEc.lrc(0, k, l, r) as ec:
        d = dev(torch, broken)
        status = torch.full((n,), 99, dtype=torch.int32, device="cuda")
        ec.reconstruct(d, dev(torch, present), stride, n, want=dev(torch, want) if single else None, status=status,
                       shard_len=dev(torch, lens))
        got = d.cpu().numpy()
        st = status.cpu().numpy()
    assert np.array_equal(st == 0, ok) and set(np.unique(st)) <= {0, G.E_UNRECOVERABLE}
    rebuilt = (present == 0) & (want != 0) & ok[:, None]
    for s in range(n):
        L = int(lens[s])
        exp = np.where(rebuilt[s][:, None], orig[s], broken[s])
        assert np.array_equal(got[s][:, :L], exp[:, :L]), (s, present[s], want[s])
    for s in range(0, n, 97):  # the numpy oracle rebuilds the same bytes from its own read set
        ref = broken[s].copy()
        if LO.decode(k, l, P, ref, present[s], want[s] if single else None):
            L = int(lens[s])
            assert np.array_equal(ref[:, :L], got[s][:, :L])


def _expected_read_set(k, l, P, pr, w):
    ok, surv = LO.read_set(k, l, P, pr, w)
    rs = np.zeros(len(pr), dtype=np.uint8)
    rs[surv] = 1
    return ok, rs


@pytest.mark.parametrize("k,l,r", [(6, 2, 2), (10, 2, 2), (6, 0, 3)])
def test_read_set_matches_model(torch, k, l, r):
    """garage_ec_read_set against the Python statement of rules 1 and 2 (l = 0: RS(k, r), first k present) for
    every pattern, with want = NULL and with each absent shard alone"""
    m = l + r
    tot = k + m
    with (G.GarageEc.lrc(0, k, l, r) if l else G.GarageEc(0, k, r)) as ec:
        P = ec.matrix()
        for pr in _patterns(tot):
            wants = [None] + [np.eye(tot, dtype=np.uint8)[o] for o in range(tot) if not pr[o]]
            for w in wants:
                ok, rs = _expected_read_set(k, l, P, pr, w)
                got = ec.read_set(pr, w)
                assert (got is not None) == ok, (pr, w)
                if ok:
                    assert np.array_equal(got, rs), (pr, w, got, rs)
                    assert int(got.sum()) <= k and not (got & (1 - pr)).any()


def test_read_set_local_repair_sizes(torch):
    with G.GarageEc.lrc(0, 10, 2, 2) as ec:
        for i in range(14):
            pr = np.ones(14, dtype=np.uint8)
            pr[i] = 0
            rs = ec.read_set(pr)
            assert int(rs.sum()) == (5 if i < 12 else 10), i
    with G.GarageEc(0, 10, 4) as ec:
        pr = np.ones(14, dtype=np.uint8)
        pr[3] = 0
        assert int(ec.read_set(pr).sum()) == 10


@pytest.mark.parametrize("mode", ["device", "host_staged", "host_zero_copy"])
def test_local_repair_reads_only_the_group(torch, mode):
    """present = the read set of one lost shard only; every other shard (absent ones included) holds poison.
    The lost shard is rebuilt exactly and nothing else is written."""
    k, l, r = 10, 2, 2
    tot, stride = 14, 8192
    cases = [(i, None) for i in range(k + l)] + [(k + l, None), (2, "two-groups")]
    n = len(cases)
    lens = np.array([stride - 16 * i - 3 for i in range(n)], dtype=np.uint32)
    _, orig = make_stripes(k, l, r, n, stride, lens, 0x3C0)
    want = np.zeros((n, tot), dtype=np.uint8)
    present = np.zeros((n, tot), dtype=np.uint8)
    with G.GarageEc.lrc(0, k, l, r) as ec:
        for s, (i, extra) in enumerate(cases):
            full = np.ones(tot, dtype=np.uint8)
            full[i] = 0
            want[s, i] = 1
            if extra:  # a second lost shard in the other group: still two local repairs
                full[7] = 0
                want[s, 7] = 1
            rs = ec.read_set(full, want[s])
            present[s] = rs
            assert int(rs.sum()) == (10 if i == k + l else 5 * int(want[s].sum())), (i, extra)
        broken = np.where(present[:, :, None] != 0, orig, np.uint8(POISON)).astype(np.uint8)
        status = np.full(n, 99, dtype=np.int32)
        if mode == "device":
            d = dev(torch, broken)
            st = torch.full((n,), 99, dtype=torch.int32, device="cuda")
            ec.reconstruct(d, dev(torch, present), stride, n, want=dev(torch, want), status=st,
                           shard_len=dev(torch, lens))
            got, status = d.cpu().numpy(), st.cpu().numpy()
        elif mode == "host_staged":
            got = broken.copy()
            ec.reconstruct(got.reshape(-1), present, stride, n, want=want, status=status, shard_len=lens)
        else:
            buf, p = ec.host_alloc(broken.size)
            try:
                buf[:] = broken.reshape(-1)
                ec.reconstruct(buf, present, stride, n, want=want, status=status, shard_len=lens)
                got = buf.copy().reshape(n, tot, stride)
            finally:
                ec.host_free(p)
    assert not status.any()
    for s in range(n):
        L = int(lens[s])
        for i in range(tot):
            exp = orig[s, i] if (present[s, i] or want[s, i]) else broken[s, i]
            assert np.array_equal(got[s, i, :L], exp[:L]), (mode, s, i)


def test_full_size_local_repair_every_stripe(torch):
    """4096 x 1 MiB LRC(10,2,2): encode, lose one data or local-parity shard per stripe, rebuild every stripe by
    local repair, compare byte for byte"""
    k, l, r, n, B = 10, 2, 2, 4096, 1 << 20
    m, tot = l + r, 14
    with G.GarageEc.lrc(0, k, l, r) as ec:
        Ls = ec.shard_len(B)
        stride = ec.stride_for(Ls)
        shards = torch.zeros(n, tot, stride, dtype=torch.uint8, device="cuda")
        data = torch.empty(n * k * stride, dtype=torch.uint8, device="cuda")
        ec.fill_random(data, data.numel(), 0x4C0, 0)
        data.view(n, k, stride)[:, :, Ls:] = 0
        lens = torch.full((n,), Ls, dtype=torch.int32, device="cuda")
        par = torch.zeros(n * m * stride, dtype=torch.uint8, device="cuda")
        ec.encode(data, par, stride, n, shard_len=lens)
        shards[:, :k] = data.view(n, k, stride)
        shards[:, k:] = par.view(n, m, stride)
        del data, par
        # spot check against the C oracle on two stripes
        P = LO.build_lrc(k, l, r)
        for s in (0, n - 1):
            h = shards[s].cpu().numpy()
            ref = O.encode(k, m, P, h[:k].reshape(-1), stride, 1, np.array([Ls], dtype=np.uint32))
            assert np.array_equal(ref.reshape(m, stride), h[k:])
        orig = shards.clone()
        lost = torch.arange(n, device="cuda") % (k + l)
        present = torch.ones(n, tot, dtype=torch.uint8, device="cuda")
        present[torch.arange(n, device="cuda"), lost] = 0
        shards[present == 0] = POISON
        status = torch.full((n,), 99, dtype=torch.int32, device="cuda")
        ec.reconstruct(shards.view(-1), present, stride, n, status=status, shard_len=lens)
        assert int(status.abs().sum()) == 0
        assert torch.equal(shards[:, :, :Ls], orig[:, :, :Ls])  # nothing is written past roundup16(shard_len)


def test_scrub_repair_on_lrc(torch):
    k, l, r = 10, 2, 2
    tot, stride, n = 14, 2048 + 128, 200
    P = LO.build_lrc(k, l, r)
    rng = np.random.default_rng(5)
    lens = rng.integers(1, stride + 1, n).astype(np.uint32)
    _, orig = make_stripes(k, l, r, n, stride, lens, 0x5C0)
    sums = np.zeros((n, tot, 32), dtype=np.uint8)
    for s in range(n):
        for i in range(tot):
            sums[s, i] = np.frombuffer(hashlib.blake2b(orig[s, i, :lens[s]].tobytes()).digest()[:32], dtype=np.uint8)
    nbad = rng.integers(0, 6, n)
    broken = orig.copy()
    badmask = np.zeros((n, tot), dtype=np.uint8)
    for s in range(n):
        for i in rng.choice(tot, int(nbad[s]), replace=False):
            broken[s, i, int(rng.integers(0, lens[s]))] ^= 0xFF
            badmask[s, i] = 1
    ok = np.array([LO.recoverable(k, P, 1 - badmask[s]) for s in range(n)])
    assert ok.any() and not ok.all()
    with G.GarageEc.lrc(0, k, l, r) as ec:
        for mode in ("device", "host"):
            if mode == "device":
                d = dev(torch, broken)
                bad_out = torch.zeros(n * tot, dtype=torch.uint8, device="cuda")
                st = torch.full((n,), 99, dtype=torch.int32, device="cuda")
                ec.scrub_repair(d, dev(torch, sums), bad_out, stride, n, status=st, shard_len=dev(torch, lens))
                got, bo, status = d.cpu().numpy(), bad_out.cpu().numpy(), st.cpu().numpy()
            else:
                got = broken.copy()
                bo = np.zeros(n * tot, dtype=np.uint8)
                status = np.full(n, 99, dtype=np.int32)
                ec.scrub_repair(got.reshape(-1), sums, bo, stride, n, status=status, shard_len=lens)
            assert np.array_equal(bo.reshape(n, tot), badmask), mode
            assert np.array_equal(status == 0, ok), mode
            for s in range(n):
                L = int(lens[s])
                exp = orig[s] if ok[s] else broken[s]
                assert np.array_equal(got[s][:, :L], exp[:, :L]), (mode, s)


def test_decode_blocks_on_lrc(torch):
    """GET of blocks that lost data shards in two groups plus an unwanted global parity (two local repairs), two
    data shards of one group (the global rule: the read set takes global parities), or too much"""
    k, l, r = 10, 2, 2
    tot = 14
    with G.GarageEc.lrc(0, k, l, r) as ec:
        blocks = [O.fill_random(bl, 0x6C0 + i) for i, bl in enumerate([1 << 20, 777777, 1 << 20, 31, 524288])]
        Ls = [ec.shard_len(b.size) for b in blocks]
        stride = ec.stride_for(max(Ls))
        n = len(blocks)
        parity = np.zeros(n * 4 * stride, dtype=np.uint8)
        ec.encode_blocks(blocks, parity, stride)
        shards = np.zeros((n, tot, stride), dtype=np.uint8)
        for s, b in enumerate(blocks):
            shards[s, :k] = O.split_block(b, k, stride).reshape(k, stride)
            shards[s, k:] = parity.reshape(n, 4, stride)[s]
        present = np.ones((n, tot), dtype=np.uint8)
        for s, lost in enumerate([[3], [0, 5, 12], [0, 1, 12], [9], [1, 2, 3, 4, 10]]):
            present[s, lost] = 0
            shards[s, lost] = POISON
        outs = [np.zeros(b.size, dtype=np.uint8) for b in blocks]
        status = np.full(n, 99, dtype=np.int32)
        ec.decode_blocks(shards.reshape(-1), present, [b.size for b in blocks], stride, outs, status=status)
        assert list(status) == [0, 0, 0, 0, G.E_UNRECOVERABLE]
        rs = ec.read_set(present[2], np.array([1] * k + [0] * 4, dtype=np.uint8))
        assert int(rs.sum()) == k and rs[10] and rs[13]  # rule 2: data 2..9, local parity 10, global parity 13
        for s in range(4):
            assert np.array_equal(outs[s], blocks[s]), s
