"""PB(k, m) contexts on the GPU: encode / verify bit-exact against the numpy model (tests/pb_oracle.py), a full-size
4096 x 1 MiB PB(10,4) encode, reconstruct of every erasure pattern, rule-1 repair from the planned halves only in
DEVICE, staged HOST and zero-copy HOST mode, malformed shard lengths, scrub_repair and the block-level calls."""
import hashlib
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import oracle_lib as O  # noqa: E402
import pb_oracle as PB  # noqa: E402

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
    P = PB.build(k, m, kind)
    data = O.fill_random(n * k * stride, seed).reshape(n, k, stride)
    sh = np.zeros((n, k + m, stride), dtype=np.uint8)
    for s in range(n):
        L = int(lens[s])
        data[s, :, L:] = 0
        sh[s, :k] = data[s]
        sh[s, k:, :L] = PB.encode(P, data[s, :, :L])
    return P, sh


@pytest.mark.parametrize("kind", [0, 1])
@pytest.mark.parametrize("k,m", [(4, 2), (6, 3), (8, 3), (10, 4), (13, 4), (16, 4)])
def test_pb_encode_verify_bit_exact(torch, k, m, kind):
    n, stride = 24, 4096 + 128
    lens = np.array([32 * (1 + (37 * i) % (stride // 32)) for i in range(n)], dtype=np.uint32)
    lens[0] = stride
    P, ref = make_stripes(k, m, kind, n, stride, lens, 0x1D0 + k + 64 * kind)
    with G.GarageEc.piggyback(0, k, m, kind) as ec:
        assert np.array_equal(ec.matrix(), P)
        groups, gof = ec.piggyback_info()
        assert groups == m - 1 and [int(g) for g in gof] == [i + 1 for i, g in enumerate(PB.groups(k, m)) for _ in g]
        par = torch.full((n * m * stride,), POISON, dtype=torch.uint8, device="cuda")
        ec.encode(dev(torch, ref[:, :k]), par, stride, n, shard_len=dev(torch, lens))
        got = par.cpu().numpy().reshape(n, m, stride)
        for s in range(n):
            L = int(lens[s])
            assert np.array_equal(got[s, :, :L], ref[s, k:, :L]), s
            assert (got[s, :, L:] == POISON).all(), s  # nothing past shard_len
        mm = torch.ones(n, dtype=torch.int32, device="cuda")
        ec.verify(dev(torch, ref), mm, stride, n, shard_len=dev(torch, lens))
        assert not mm.cpu().numpy().any()
        bad = ref.copy()
        for s in range(n):  # alternate a- and b-half corruption
            L = int(lens[s])
            bad[s, k + s % m, (L // 2) * (s & 1) + (L // 2 - 1) * ((s >> 1) & 1)] ^= 0x5A
        ec.verify(dev(torch, bad), mm, stride, n, shard_len=dev(torch, lens))
        assert [int(x) for x in mm.cpu().numpy()] == [1 << (s % m) for s in range(n)]
        # HOST mode: same bytes
        hp = np.zeros(n * m * stride, dtype=np.uint8)
        ec.encode(np.ascontiguousarray(ref[:, :k]).reshape(-1), hp, stride, n, shard_len=lens)
        hp = hp.reshape(n, m, stride)
        for s in range(n):
            assert np.array_equal(hp[s, :, :int(lens[s])], ref[s, k:, :int(lens[s])])


def test_pb_full_size_encode(torch):
    """4096 x 1 MiB PB(10,4) (shard_len 104 960): a-halves and b-halves against an RS(10,4) context run over each half
    plus the group XORs computed by torch, and two stripes byte for byte against the numpy model"""
    k, m, n, B = 10, 4, 4096, 1 << 20
    with G.GarageEc.piggyback(0, k, m) as ec, G.GarageEc(0, k, m) as rs:
        L = ec.code_shard_len(B)
        assert L == 104960 and rs.shard_len(B) == 104858
        h = L // 2
        data = torch.empty(n * k * L + L, dtype=torch.uint8, device="cuda")
        ec.fill_random(data, data.numel(), 0x4D0, 0)
        par = torch.empty(n * m * L, dtype=torch.uint8, device="cuda")
        ec.encode(data, par, L, n)
        half_len = torch.full((n,), h, dtype=torch.int32, device="cuda")
        ra = torch.empty(n * m * L, dtype=torch.uint8, device="cuda")
        rb = torch.empty(n * m * L, dtype=torch.uint8, device="cuda")
        rs.encode(data, ra, L, n, shard_len=half_len)
        rs.encode(data[h:], rb, L, n, shard_len=half_len)
        torch.cuda.synchronize()
        d3, p3 = data[: n * k * L].view(n, k, L), par.view(n, m, L)
        assert torch.equal(p3[:, :, :h], ra.view(n, m, L)[:, :, :h])
        rb3 = rb.view(n, m, L)[:, :, :h].clone()
        for i, g in enumerate(PB.groups(k, m), start=1):
            x = d3[:, g[0], :h].clone()
            for j in g[1:]:
                x ^= d3[:, j, :h]
            rb3[:, i] ^= x
        assert torch.equal(p3[:, :, h:], rb3)
        P = PB.build(k, m)
        for s in (0, n - 1):
            assert np.array_equal(PB.encode(P, d3[s].cpu().numpy()), p3[s].cpu().numpy())


def _all_patterns(tot):
    return [np.array([((p >> i) & 1) ^ 1 for i in range(tot)], dtype=np.uint8) for p in range(1 << tot)]


@pytest.mark.parametrize("k,m,single", [(6, 3, False), (6, 3, True), (10, 4, False)])
def test_pb_reconstruct_every_pattern(torch, k, m, single):
    """every erasure pattern in DEVICE mode; MDS: recoverable iff at most m shards are absent (the CPU tests check
    that against the rank model); want = NULL or each absent shard alone"""
    tot, stride = k + m, 128
    present_l, want_l = [], []
    for pr in _all_patterns(tot):
        absent = [o for o in range(tot) if not pr[o]]
        if not single:
            present_l.append(pr)
            want_l.append(np.ones(tot, dtype=np.uint8))
        else:
            for o in absent:
                present_l.append(pr)
                want_l.append(np.eye(tot, dtype=np.uint8)[o])
    n = len(present_l)
    present, want = np.array(present_l), np.array(want_l)
    ok = (present == 0).sum(axis=1) <= m
    lens = np.array([32 * (1 + i % 4) for i in range(n)], dtype=np.uint32)
    P, orig = make_stripes(k, m, 1, n, stride, lens, 0x2D0 + k + single)
    broken = orig.copy()
    broken[present == 0] = POISON
    with G.GarageEc.piggyback(0, k, m, 1) as ec:
        d = dev(torch, broken)
        status = torch.full((n,), 99, dtype=torch.int32, device="cuda")
        ec.reconstruct(d, dev(torch, present), stride, n, want=dev(torch, want) if single else None, status=status,
                       shard_len=dev(torch, lens))
        got, st = d.cpu().numpy(), status.cpu().numpy()
    assert np.array_equal(st == 0, ok) and set(np.unique(st)) <= {0, G.E_UNRECOVERABLE}
    rebuilt = (present == 0) & (want != 0) & ok[:, None]
    inside = np.arange(stride)[None, None, :] < lens[:, None, None]  # nothing is written past shard_len
    exp = np.where(rebuilt[:, :, None] & inside, orig, broken)
    assert np.array_equal(got, exp)
    for s in range(0, n, 211):  # the numpy model rebuilds the same bytes from its own plan
        ref = broken[s].copy()[:, :lens[s]]
        if PB.decode(k, m, P, ref, present[s], want[s] if single else None):
            assert np.array_equal(ref, got[s][:, :lens[s]])


@pytest.mark.parametrize("mode", ["device", "host_staged", "host_zero_copy"])
def test_rule1_repair_reads_only_the_planned_halves(torch, mode):
    """present = the shards of the read plan of one lost data shard; every half outside the plan holds poison.  The
    lost shard is rebuilt exactly and nothing else is written."""
    k, m = 10, 4
    tot, stride = 14, 8192
    n = k + 2
    lens = np.array([stride - 32 * i for i in range(n)], dtype=np.uint32)
    P, orig = make_stripes(k, m, 0, n, stride, lens, 0x3D0)
    want = np.zeros((n, tot), dtype=np.uint8)
    present = np.zeros((n, tot), dtype=np.uint8)
    broken = np.full_like(orig, POISON)
    with G.GarageEc.piggyback(0, k, m) as ec:
        for s in range(n):
            j = s % k
            full = np.ones(tot, dtype=np.uint8)
            full[j] = 0
            want[s, j] = 1
            hv = ec.read_plan(full, want[s])
            ok, surv = PB.read_plan(k, m, P, full, want[s])
            assert ok and sum(bin(int(x)).count("1") for x in hv) == len(surv) == (14 if j < 4 else 13)
            assert np.array_equal(ec.read_set(full, want[s]), (hv != 0).astype(np.uint8))
            present[s] = hv != 0
            h = int(lens[s]) // 2
            for i in range(tot):
                for half in range(2):
                    if (hv[i] >> half) & 1:
                        broken[s, i, half * h:(half + 1) * h] = orig[s, i, half * h:(half + 1) * h]
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
            exp = orig[s, i] if want[s, i] else broken[s, i]
            assert np.array_equal(got[s, i, :L], exp[:L]), (mode, s, i)


def test_malformed_shard_len(torch):
    """shard_len % 32 != 0 on a PB context: DEVICE encode writes nothing for the stripe, verify sets every mismatch
    bit, reconstruct reports GARAGE_EC_E_INVALID; the other stripes are unaffected.  HOST calls refuse the batch."""
    k, m, n, stride = 6, 3, 3, 512
    lens = np.array([512, 496, 256], dtype=np.uint32)
    good = np.array([512, 512, 256], dtype=np.uint32)
    P, ref = make_stripes(k, m, 0, n, stride, good, 0x7D0)
    with G.GarageEc.piggyback(0, k, m) as ec:
        par = torch.full((n * m * stride,), POISON, dtype=torch.uint8, device="cuda")
        ec.encode(dev(torch, ref[:, :k]), par, stride, n, shard_len=dev(torch, lens))
        got = par.cpu().numpy().reshape(n, m, stride)
        assert (got[1] == POISON).all()
        assert np.array_equal(got[0], ref[0, k:]) and np.array_equal(got[2, :, :256], ref[2, k:, :256])
        mm = torch.zeros(n, dtype=torch.int32, device="cuda")
        ec.verify(dev(torch, ref), mm, stride, n, shard_len=dev(torch, lens))
        assert [int(x) for x in mm.cpu().numpy()] == [0, 7, 0]
        present = np.ones((n, k + m), dtype=np.uint8)
        present[:, 2] = 0
        broken = ref.copy()
        broken[:, 2] = POISON
        d = dev(torch, broken)
        st = torch.full((n,), 99, dtype=torch.int32, device="cuda")
        ec.reconstruct(d, dev(torch, present), stride, n, status=st, shard_len=dev(torch, lens))
        assert [int(x) for x in st.cpu().numpy()] == [0, G.E_INVALID, 0]
        out = d.cpu().numpy()
        assert np.array_equal(out[1], broken[1]) and np.array_equal(out[0], ref[0])
        assert np.array_equal(out[2, :, :256], ref[2, :, :256])
        with pytest.raises(G.EcError) as e:
            ec.encode(np.ascontiguousarray(ref[:, :k]).reshape(-1), np.zeros(n * m * stride, np.uint8), stride, n,
                      shard_len=lens)
        assert e.value.code == G.E_INVALID
        with pytest.raises(G.EcError) as e:
            ec.reconstruct(broken.reshape(-1), present, stride, n, shard_len=lens)
        assert e.value.code == G.E_INVALID
        with pytest.raises(G.EcError) as e:
            ec.verify(ref.reshape(-1), np.zeros(n, np.uint32), 496, 1)
        assert e.value.code == G.E_INVALID


def test_scrub_repair_on_pb(torch):
    k, m = 10, 4
    tot, stride, n = 14, 2048 + 128, 120
    rng = np.random.default_rng(6)
    lens = (32 * rng.integers(1, stride // 32 + 1, n)).astype(np.uint32)
    _, orig = make_stripes(k, m, 0, n, stride, lens, 0x5D0)
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
    ok = badmask.sum(axis=1) <= m
    assert ok.any() and not ok.all()
    with G.GarageEc.piggyback(0, k, m) as ec:
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


def test_encode_and_decode_blocks_on_pb(torch):
    """the block-level calls frame blocks with the PB shard length (ceil(len/k) rounded up to 128) and decode GETs
    that lost one data shard (rule 1), four shards, or five"""
    k, m = 10, 4
    tot = 14
    with G.GarageEc.piggyback(0, k, m) as ec:
        blocks = [O.fill_random(bl, 0x6D0 + i) for i, bl in enumerate([1 << 20, 777777, 1 << 20, 31, 524288])]
        Ls = [ec.code_shard_len(b.size) for b in blocks]
        assert Ls == [PB.shard_len(b.size, k) for b in blocks] and all(L % 128 == 0 for L in Ls)
        stride = max(Ls)
        n = len(blocks)
        parity = np.zeros(n * m * stride, dtype=np.uint8)
        sums = np.zeros(n * tot * 32, dtype=np.uint8)
        ec.encode_blocks(blocks, parity, stride, sums_out=sums)
        P = PB.build(k, m)
        shards = np.zeros((n, tot, stride), dtype=np.uint8)
        for s, b in enumerate(blocks):
            L = Ls[s]
            flat = np.zeros(k * L, dtype=np.uint8)
            flat[:b.size] = b
            shards[s, :k, :L] = flat.reshape(k, L)
            shards[s, k:] = parity.reshape(n, m, stride)[s]
            assert np.array_equal(shards[s, k:, :L], PB.encode(P, shards[s, :k, :L])), s
            for i in range(tot):
                exp = np.frombuffer(hashlib.blake2b(shards[s, i, :L].tobytes()).digest()[:32], dtype=np.uint8)
                assert np.array_equal(sums.reshape(n, tot, 32)[s, i], exp), (s, i)
        present = np.ones((n, tot), dtype=np.uint8)
        for s, lost in enumerate([[3], [0, 5, 12, 13], [9], [1], [1, 2, 3, 4, 10]]):
            present[s, lost] = 0
            shards[s, lost] = POISON
        outs = [np.zeros(b.size, dtype=np.uint8) for b in blocks]
        status = np.full(n, 99, dtype=np.int32)
        ec.decode_blocks(shards.reshape(-1), present, [b.size for b in blocks], stride, outs, status=status)
        assert list(status) == [0, 0, 0, 0, G.E_UNRECOVERABLE]
        for s in range(4):
            assert np.array_equal(outs[s], blocks[s]), s
