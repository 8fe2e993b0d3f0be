"""garage_ec_reconstruct_segments on the H100 (DESIGN.md section 2.10), every output compared byte for byte with
tests/segment_oracle.py: RS at both matrix kinds and one k from each compiled kernel class, LRC(10,2,2), PB(10,4);
shard lengths with empty trailing segments and 1 MiB blocks; ragged batches larger than the grid; DEVICE == HOST ==
gather form; the 0x00 / 0xFF equivalence with garage_ec_reconstruct; CUDA graph capture; the HOST fault contract;
Clay refused; 4096 x 1 MiB RS(10,4) stripes with 5-8 damaged shards each."""
import itertools
import os
import sys
import zlib

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import oracle_lib as O  # noqa: E402
import segment_oracle as SO  # noqa: E402

import garage_b200 as G  # noqa: E402

pytestmark = pytest.mark.gpu

SENTINEL = 0xEE


@pytest.fixture(scope="module")
def torch():
    import torch as t

    assert t.cuda.is_available()
    return t


def context(name):
    kind, *a = name.split("_")
    a = [int(x) if x.isdigit() else x for x in a]
    if kind == "rs":
        return G.GarageEc(0, a[0], a[1], G.CAUCHY if a[2:] == ["c"] else G.VANDERMONDE)
    if kind == "lrc":
        return G.GarageEc.lrc(0, a[0], a[1], a[2])
    return G.GarageEc.piggyback(0, a[0], a[1])


def oracle_code(ec, name):
    kind = name.split("_")[0]
    l, _ = ec.code_info()
    return SO.Code(kind, ec.k, ec.m, ec.matrix(), l=l if kind == "lrc" else 0)


def make_stripes(torch, ec, lens, stride, seed):
    """n = len(lens) encoded stripes (n, k+m, stride); bytes past each L are the sentinel"""
    n, k, m = len(lens), ec.k, ec.m
    data = O.fill_random(n * k * stride, seed).reshape(n, k, stride)
    for s, L in enumerate(lens):
        data[s, :, L:] = 0
    par = torch.zeros(n * m * stride, dtype=torch.uint8, device="cuda")
    ec.encode(torch.from_numpy(data.reshape(-1)).cuda(), par, stride, n,
              shard_len=torch.from_numpy(np.asarray(lens, dtype=np.int32)).cuda())
    sh = np.concatenate([data, par.cpu().numpy().reshape(n, m, stride)], axis=1)
    for s, L in enumerate(lens):
        sh[s, :, L:] = SENTINEL
    return np.ascontiguousarray(sh)


def damage(code, sh, sp, L):
    for i in range(sh.shape[0]):
        for g in range(8):
            if not (int(sp[i]) >> g) & 1:
                o, n = SO.segments(L)[g]
                sh[i, o:o + n] = SENTINEL


def random_patterns(code, lens, rng, want_every=3):
    """per stripe: a pattern with m+1..k+m damaged shards spread over units (at most m per unit, LRC 1), or a random
    one (often unrecoverable), or a whole-shard one; want on every want_every-th stripe"""
    tot, n = code.k + code.m, len(lens)
    sp = np.full((n, tot), 0xFF, dtype=np.uint8)
    want = np.ones((n, tot), dtype=np.uint8)
    limit = 1 if code.kind == "lrc" else code.m
    for s in range(n):
        r = s % 3
        if r == 0:
            count = [0] * code.units
            for i in rng.choice(tot, int(rng.integers(code.m + 1, min(tot, limit * code.units) + 1)), replace=False):
                g = int(rng.choice([u for u in range(code.units) if count[u] < limit]))
                count[g] += 1
                sp[s, i] &= ~np.uint8(((1 << g) | ((1 << (g + 4)) if code.kind == "pb" else 0)) & 0xFF)
        elif r == 1:
            for i in rng.choice(tot, int(rng.integers(1, tot)), replace=False):
                sp[s, i] = rng.integers(0, 256) & ~(1 << int(rng.integers(0, 8)))
        else:
            sp[s, rng.choice(tot, int(rng.integers(1, code.m + 1)), replace=False)] = 0
        if s % want_every == 1:
            want[s] = rng.integers(0, 2, tot)
    return sp, want


def run(torch, ec, mode, sh, sp, want, lens, stride):
    n = len(lens)
    status = np.full(n, 0x5A5A, dtype=np.int32)
    lens = np.asarray(lens, dtype=np.uint32)
    if mode == "device":
        d = torch.from_numpy(sh.reshape(-1).copy()).cuda()
        ds = torch.zeros(n, dtype=torch.int32, device="cuda")
        ec.reconstruct_segments(d, torch.from_numpy(sp.reshape(-1)).cuda(), stride, n,
                                want=None if want is None else torch.from_numpy(want.reshape(-1)).cuda(), status=ds,
                                shard_len=torch.from_numpy(lens.astype(np.int32)).cuda())
        torch.cuda.synchronize()
        return d.cpu().numpy().reshape(sh.shape), ds.cpu().numpy()
    if mode == "host":
        out = sh.copy()
        ec.reconstruct_segments(out.reshape(-1), sp.reshape(-1), stride, n, want=want, status=status, shard_len=lens)
        return out, status
    bufs = [np.ascontiguousarray(sh[s]).reshape(-1) for s in range(n)]
    ec.reconstruct_segments(bufs, sp.reshape(-1), stride, n, want=want, status=status, shard_len=lens)
    return np.stack([b.reshape(sh.shape[1:]) for b in bufs]), status


def expect(code, sh, sp, want, lens, stride):
    out = sh.copy()
    st = SO.reconstruct(code, out.reshape(-1), sp.reshape(-1), stride, len(lens), lens,
                        None if want is None else want.reshape(-1))
    return out, st


CODES = ["rs_4_2", "rs_6_3", "rs_6_3_c", "rs_10_4", "rs_10_4_c", "lrc_10_2_2", "pb_10_4",
         # one k from each compiled kernel class: LDG (k <= 4, 7), TMA (5..16), TMA split staging (k > 16)
         "rs_3_2", "rs_7_3", "rs_13_4", "rs_16_4", "rs_20_4", "rs_32_4"]
RAGGED = [1, 15, 16, 17, 112, 127, 128, 129, 1000, 4096]


@pytest.mark.parametrize("name", CODES)
@pytest.mark.parametrize("mode", ["device", "host", "gather"])
def test_matches_oracle_in_ragged_batches(torch, name, mode):
    with context(name) as ec:
        code = oracle_code(ec, name)
        rng = np.random.default_rng(zlib.crc32((name + mode).encode()))
        n = 300  # more stripes than the 132 CTAs of the grid
        base = [128, 256, 384, 1152, 4096] if code.kind == "pb" else RAGGED
        lens = [base[s % len(base)] for s in range(n)]
        rng.shuffle(lens)
        stride = 4096 + 128
        sh = make_stripes(torch, ec, lens, stride, 7)
        sp, want = random_patterns(code, lens, rng)
        want = None if mode == "gather" else want
        for s, L in enumerate(lens):
            damage(code, sh[s], sp[s], L)
        got, st = run(torch, ec, mode, sh, sp, want, lens, stride)
        exp, est = expect(code, sh, sp, want, lens, stride)
        assert np.array_equal(st, est)
        assert (est == 0).sum() > n // 3 and (est == G.E_UNRECOVERABLE).sum() > 0
        for s in range(n):
            assert np.array_equal(got[s], exp[s]), (s, lens[s], sp[s], st[s])


@pytest.mark.parametrize("name", ["rs_6_3", "rs_10_4", "lrc_10_2_2", "pb_10_4"])
def test_every_subset_of_at_most_m_bad_shards_in_each_unit(torch, name):
    with context(name) as ec:
        code = oracle_code(ec, name)
        tot = code.k + code.m
        subsets = [c for r in range(code.m + 1) for c in itertools.combinations(range(tot), r)]
        n = len(subsets)
        L = 1152 if code.kind == "pb" else 1000
        stride = 1152
        lens = [L] * n
        sh = make_stripes(torch, ec, lens, stride, 11)
        sp = np.full((n, tot), 0xFF, dtype=np.uint8)
        for s in range(n):
            for g in range(code.units):  # unit g of stripe s: subset (s + 7g) mod n, so every unit sees every subset
                for i in subsets[(s + 7 * g) % n]:
                    sp[s, i] &= ~np.uint8(((1 << g) | ((1 << (g + 4)) if code.kind == "pb" else 0)) & 0xFF)
            damage(code, sh[s], sp[s], L)
        got, st = run(torch, ec, "device", sh, sp, None, lens, stride)
        exp, est = expect(code, sh, sp, None, lens, stride)
        assert np.array_equal(st, est) and np.array_equal(got, exp)
        if code.kind != "lrc":  # MDS: every such pattern is recoverable
            assert (st == 0).all()


@pytest.mark.parametrize("name", ["rs_10_4", "lrc_10_2_2", "pb_10_4"])
def test_whole_bytes_equal_reconstruct(torch, name):
    with context(name) as ec:
        tot, n = ec.k + ec.m, 200
        rng = np.random.default_rng(5)
        lens = [1152 if name.startswith("pb") else int(x) for x in rng.integers(1, 2049, n)]
        stride = 2176
        sh = make_stripes(torch, ec, lens, stride, 13)
        present = np.ones((n, tot), dtype=np.uint8)
        for s in range(n):
            present[s, rng.choice(tot, int(rng.integers(1, ec.m + 2)), replace=False)] = 0
        sh[present == 0] = SENTINEL
        want = rng.integers(0, 2, (n, tot)).astype(np.uint8)
        for w in (None, want):
            a = sh.copy()
            sa = np.zeros(n, dtype=np.int32)
            ec.reconstruct(a.reshape(-1), present, stride, n, want=w, status=sa, shard_len=np.asarray(lens, np.uint32))
            b = sh.copy()
            sb = np.zeros(n, dtype=np.int32)
            ec.reconstruct_segments(b.reshape(-1), np.where(present == 1, 0xFF, 0).astype(np.uint8), stride, n, want=w,
                                    status=sb, shard_len=np.asarray(lens, np.uint32))
            assert np.array_equal(sa, sb) and np.array_equal(a, b)


def test_clay_is_refused_before_any_cuda_call(torch):
    with G.GarageEc.clay(0, 4, 2) as ec:
        before = ec.launch_count()
        sh = torch.zeros(6 * 4096, dtype=torch.uint8, device="cuda")
        sp = torch.zeros(6, dtype=torch.uint8, device="cuda")
        with pytest.raises(G.EcError) as ei:
            ec.reconstruct_segments(sh, sp, 4096, 1)
        assert ei.value.code == G.E_INVALID and ec.launch_count() == before
        with pytest.raises(G.EcError) as ei:
            ec.reconstruct_segments(sh.cpu().numpy(), sp.cpu().numpy(), 4096, 1)
        assert ei.value.code == G.E_INVALID


def test_malformed_lengths(torch):
    with G.GarageEc.piggyback(0, 10, 4) as ec:
        lens = np.array([1024, 1000, 2048], dtype=np.uint32)  # 1000: not a multiple of 128
        stride = 1024
        sh = np.full((3, 14, stride), SENTINEL, dtype=np.uint8)
        sp = np.full((3, 14), 0xFE, dtype=np.uint8)
        sp[0] = 0xFF
        with pytest.raises(G.EcError) as ei:
            ec.reconstruct_segments(sh.reshape(-1), sp, stride, 3, shard_len=lens)
        assert ei.value.code == G.E_INVALID
        got, st = run(torch, ec, "device", sh, sp, None, lens, stride)
        assert st[1] == G.E_INVALID and st[2] == G.E_INVALID and st[0] == 0
        assert (got[1:] == SENTINEL).all()


def test_cuda_graph_capture_and_replay(torch):
    with G.GarageEc(0, 10, 4) as ec:
        code = oracle_code(ec, "rs_10_4")
        rng = np.random.default_rng(9)
        n, stride = 64, 4096
        lens = [int(x) for x in rng.integers(1, stride + 1, n)]
        sh = make_stripes(torch, ec, lens, stride, 17)
        sp, want = random_patterns(code, lens, rng)
        for s, L in enumerate(lens):
            damage(code, sh[s], sp[s], L)
        exp, est = expect(code, sh, sp, want, lens, stride)
        d = torch.from_numpy(sh.reshape(-1).copy()).cuda()
        dsp = torch.from_numpy(sp.reshape(-1)).cuda()
        dw = torch.from_numpy(want.reshape(-1)).cuda()
        dl = torch.from_numpy(np.asarray(lens, np.int32)).cuda()
        ds = torch.zeros(n, dtype=torch.int32, device="cuda")
        ec.reconstruct_segments(d, dsp, stride, n, want=dw, status=ds, shard_len=dl)  # warm-up outside capture
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            with torch.cuda.graph(g, stream=s):
                ec.reconstruct_segments(d, dsp, stride, n, want=dw, status=ds, shard_len=dl)
        for _ in range(2):
            d.copy_(torch.from_numpy(sh.reshape(-1)).cuda())
            ds.fill_(0x5A5A)
            g.replay()
            torch.cuda.synchronize()
            assert np.array_equal(ds.cpu().numpy(), est)
            assert np.array_equal(d.cpu().numpy().reshape(sh.shape), exp)


@pytest.mark.parametrize("fail_at", [0, 2, 5, 9])
def test_host_fault_leaves_caller_buffers_alone(torch, fail_at):
    with G.GarageEc(0, 6, 3) as ec:
        code = oracle_code(ec, "rs_6_3")
        rng = np.random.default_rng(fail_at)
        n, stride = 480, 174848  # several 48 MB chunks
        lens = [stride] * n
        sh = make_stripes(torch, ec, lens, stride, 23)
        sp, _ = random_patterns(code, lens, rng)
        sp[1::3] = sp[0::3][: len(sp[1::3])]  # mostly recoverable
        for s in range(n):
            damage(code, sh[s], sp[s], stride)
        st = np.zeros(n, dtype=np.int32)
        work = sh.copy()
        ec.reconstruct_segments(work.reshape(-1), sp, stride, n, status=st)  # lanes allocated
        ec.debug_fail_after(fail_at)
        work = sh.copy()
        with pytest.raises(G.EcError):
            ec.reconstruct_segments(work.reshape(-1), sp, stride, n, status=st)
        ec.debug_fail_after(-1)
        work[:] = 0x11
        st[:] = 0x5A5A5A5A
        torch.cuda.synchronize()
        assert (work == 0x11).all() and (st == 0x5A5A5A5A).all()
        work = sh.copy()
        ec.reconstruct_segments(work.reshape(-1), sp, stride, n, status=st)
        for s in range(0, n, 37):
            e = sh[s].copy()
            assert SO.reconstruct_stripe(code, e, sp[s], stride) == st[s] and np.array_equal(work[s], e)


def test_full_size_rs_10_4_with_5_to_8_damaged_shards(torch):
    """4096 x 1 MiB stripes, each with 5..8 damaged shards in disjoint segments: every byte comes back"""
    k, m, n = 10, 4, 4096
    tot = k + m
    with G.GarageEc(0, k, m) as ec:
        L = ec.shard_len(1 << 20)
        stride = ec.stride_for(L)
        sh = torch.empty(n * tot * stride, dtype=torch.uint8, device="cuda")
        v = sh.view(n, tot, stride)
        gen = torch.Generator(device="cuda").manual_seed(31)
        v[:, :k, :L] = torch.randint(0, 256, (n, k, L), dtype=torch.uint8, device="cuda", generator=gen)
        v[:, :, L:] = 0
        data = v[:, :k].contiguous().view(-1)
        par = torch.zeros(n * m * stride, dtype=torch.uint8, device="cuda")
        ec.encode(data, par, stride, n)
        v[:, k:] = par.view(n, m, stride)
        orig = sh.clone()
        rng = np.random.default_rng(1)
        sp = np.full((n, tot), 0xFF, dtype=np.uint8)
        seg = SO.segments(L)
        for s in range(n):
            bad = rng.choice(tot, 5 + s % 4, replace=False)
            units = rng.permutation(8)
            for j, i in enumerate(bad):
                g = int(units[j % 8])
                sp[s, i] &= ~np.uint8(1 << g)
                o, ln = seg[g]
                v[s, int(i), o:o + ln] = SENTINEL
        st = torch.full((n,), 0x5A5A, dtype=torch.int32, device="cuda")
        ec.reconstruct_segments(sh, torch.from_numpy(sp.reshape(-1)).cuda(), stride, n, status=st)
        torch.cuda.synchronize()
        assert int(st.abs().sum()) == 0
        assert torch.equal(sh, orig)


@pytest.mark.parametrize("mode", ["device", "host"])
def test_present_units_are_never_written(torch, mode):
    """present bytes hold the sentinel, not code bytes: the rebuilt shard's other segments and the parities outside
    the read set stay as they were, and only the rebuilt segment changes"""
    with G.GarageEc(0, 10, 4) as ec:
        code = oracle_code(ec, "rs_10_4")
        n, L, stride = 3, 1000, 1024
        lens = [L] * n
        sh = make_stripes(torch, ec, lens, stride, 29)
        orig = sh.copy()
        sp = np.full((n, 14), 0xFF, dtype=np.uint8)
        o1, n1 = SO.segments(L)[1]
        for s in range(n):
            sp[s, s] = 0xFF & ~(1 << 1)          # shard s: only segment 1 absent
            keep = sh[s, s, o1:o1 + n1].copy()
            sh[s, s, :] = SENTINEL               # its present segments: sentinel
            sh[s, s, o1:o1 + n1] = keep ^ 0x77   # its absent segment: garbage
            sh[s, 12:, :] = SENTINEL             # parities 12, 13: present, outside the first k survivors
        got, st = run(torch, ec, mode, sh, sp, None, lens, stride)
        exp, est = expect(code, sh, sp, None, lens, stride)
        assert (st == 0).all() and np.array_equal(got, exp)
        for s in range(n):
            assert np.array_equal(got[s, s, o1:o1 + n1], orig[s, s, o1:o1 + n1])
            rest = np.concatenate([got[s, s, :o1], got[s, s, o1 + n1:]])
            assert (rest == SENTINEL).all() and (got[s, 12:] == SENTINEL).all()


@pytest.mark.parametrize("name", ["lrc_10_2_2", "pb_10_4", "rs_10_4_c"])
def test_1mib_blocks_match_oracle(torch, name):
    """the shard lengths of 1 MiB blocks: units of many 32-column chunks, split across CTAs in the launch's tail"""
    with context(name) as ec:
        code = oracle_code(ec, name)
        L = ec.code_shard_len(1 << 20)
        stride = -(-L // 128) * 128
        n = 12
        lens = [L] * n
        rng = np.random.default_rng(31)
        sh = make_stripes(torch, ec, lens, stride, 37)
        sp, want = random_patterns(code, lens, rng)
        for s in range(n):
            damage(code, sh[s], sp[s], L)
        for w in (None, want):
            got, st = run(torch, ec, "device", sh, sp, w, lens, stride)
            exp, est = expect(code, sh, sp, w, lens, stride)
            assert np.array_equal(st, est) and (est == 0).any()
            assert np.array_equal(got, exp)
