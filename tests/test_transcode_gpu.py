"""garage_ec_transcode on the GPU: bit-exact against the model of DESIGN.md 2.3 (tests/transcode_oracle.py) in DEVICE
and HOST mode for RS, LRC, PB and whole-block sources and every destination kernel class, degraded sources, write
bounds, a full-size 4096 x 1 MiB RS(6,3) -> RS(10,4) batch, CUDA-graph capture, tags, and the HOST ownership
contract under injected faults."""
import itertools
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import oracle_lib as O  # noqa: E402
import transcode_oracle as T  # noqa: E402

import garage_b200 as G  # noqa: E402

pytestmark = pytest.mark.gpu
SENT = 0xA5
LENS = [1, 15, 16, 17, 511, 4095, 300001, (1 << 20) - 977, 1 << 20]


@pytest.fixture(scope="module")
def torch():
    import torch as t

    assert t.cuda.is_available()
    return t


def ctx_of(code):
    if code[0] == "rep":
        return None
    if code[0] == "lrc":
        return G.GarageEc.lrc(0, code[1], code[2], code[3])
    if code[0] == "pb":
        return G.GarageEc.piggyback(0, code[1], code[2], code[3])
    return G.GarageEc(0, code[1], code[2], code[3])


def stride_for(code, lens, slack=0):
    return -(-(max(T.shard_len(code, n) for n in lens) + slack) // 16) * 16


def make_source(code, lens, stride, seed):
    """(blocks, source shards (n, k+m, stride)); whole blocks: (n, 1, stride)"""
    rng = np.random.default_rng(seed)
    blocks = [rng.integers(0, 256, n, dtype=np.uint8) for n in lens]
    tot = T.k_of(code) + T.m_of(code)
    sh = np.zeros((len(lens), tot, stride), dtype=np.uint8)
    for s, b in enumerate(blocks):
        sh[s] = T.encode_block(code, b, stride)
    return blocks, sh


def check_dst(dst_code, blocks, got, sums=None, kind=None, skip=()):
    for s, b in enumerate(blocks):
        Ld = T.shard_len(dst_code, b.size)
        if s in skip:
            assert (got[s] == SENT).all(), s
            continue
        want = T.encode_block(dst_code, b)
        assert np.array_equal(got[s, :, :Ld], want), (dst_code, s, b.size)
        r16 = -(-Ld // 16) * 16
        assert (got[s, :, Ld:r16] == 0).all(), s
        assert (got[s, :, r16:] == SENT).all(), s  # nothing past roundup16(L_d)
        if sums is not None:
            for i in range(got.shape[1]):
                assert sums[s, i].tobytes() == G.shard_sum_host(kind, got[s, i, :Ld]), (s, i)


def run_pair(torch, src_code, dst_code, lens, seed):
    src, dst = ctx_of(src_code), ctx_of(dst_code)
    ss = stride_for(src_code, lens)
    ds = stride_for(dst_code, lens, slack=32)
    blocks, sh = make_source(src_code, lens, ss, seed)
    n, dtot = len(lens), T.k_of(dst_code) + T.m_of(dst_code)
    bl = np.array(lens, dtype=np.uint32)
    # DEVICE
    d_out = torch.full((n * dtot * ds,), SENT, dtype=torch.uint8, device="cuda")
    st = torch.full((n,), 7, dtype=torch.int32, device="cuda")
    dst.transcode(src, torch.from_numpy(sh).cuda(), torch.from_numpy(bl).cuda(), ss, d_out, ds, n, status=st)
    torch.cuda.synchronize()
    assert not st.cpu().numpy().any()
    check_dst(dst_code, blocks, d_out.cpu().numpy().reshape(n, dtot, ds))
    # HOST, with tags
    h_src = sh.copy()
    h_out = np.full((n, dtot, ds), SENT, dtype=np.uint8)
    sums = np.zeros((n, dtot, 32), dtype=np.uint8)
    hst = np.full(n, 7, dtype=np.int32)
    assert dst.transcode(src, h_src, bl, ss, h_out, ds, n, dst_sums=sums, status=hst) == 0
    assert not hst.any()
    assert np.array_equal(h_src, sh)  # HOST mode never writes the source
    check_dst(dst_code, blocks, h_out, sums, G.SUM_BLAKE2)
    for c in (src, dst):
        if c is not None:
            c.close()


PAIRS = [(("rs", 6, 3), ("rs", 10, 4)), (("rs", 10, 4), ("lrc", 10, 2, 2)), (("rs", 10, 4), ("pb", 10, 4)),
         (("pb", 10, 4), ("rs", 6, 3)), (("lrc", 12, 2, 2), ("rs", 12, 4)), (("rep",), ("rs", 10, 4)),
         (("rep",), ("pb", 6, 3))]
# destinations of every kernel class: LDG (k <= 4), TMA, tensor map (k >= 13), split staging (k > 16), m > 4
CLASSES = [(("rs", 6, 3), ("rs", k, m)) for k, m in [(4, 2), (13, 4), (16, 4), (20, 4), (32, 4), (17, 8)]]


def with_kind(code, kind):
    return code + (kind,) if code[0] in ("rs", "pb") else code


@pytest.mark.parametrize("kind", [0, 1])
@pytest.mark.parametrize("pair", PAIRS + CLASSES, ids=lambda p: "%s_to_%s" % ("-".join(map(str, p[0])), "-".join(map(str, p[1]))))
def test_transcode_bit_exact(torch, pair, kind):
    src_code, dst_code = with_kind(pair[0], kind), with_kind(pair[1], kind)
    run_pair(torch, src_code, dst_code, LENS, 0x7C0 + 17 * kind + len(str(pair)))


@pytest.mark.parametrize("src_code", [("rs", 6, 3, 0), ("pb", 6, 3, 0)])
def test_degraded_sources_every_pattern(torch, src_code):
    """every erasure pattern of up to m_s shards rebuilds exactly; a stripe with m_s + 1 erasures reports
    UNRECOVERABLE, its destination keeps the sentinel and its neighbours are exact"""
    dst_code = ("rs", 10, 4, 0)
    tot = 9
    pats = [p for r in (1, 2, 3) for p in itertools.combinations(range(tot), r)]
    bad_at = len(pats) // 2
    pats.insert(bad_at, (0, 2, 4, 6))
    n = len(pats)
    lens = [3000 + 37 * s for s in range(n)]
    src, dst = ctx_of(src_code), ctx_of(dst_code)
    ss, ds = stride_for(src_code, lens), stride_for(dst_code, lens, slack=16)
    blocks, sh = make_source(src_code, lens, ss, 0xDE6)
    present = np.ones((n, tot), dtype=np.uint8)
    work = sh.copy()
    for s, p in enumerate(pats):
        present[s, list(p)] = 0
        work[s, list(p)] = 0
    bl = np.array(lens, dtype=np.uint32)
    # HOST
    h_src = work.copy()
    out = np.full((n, 14, ds), SENT, dtype=np.uint8)
    st = np.zeros(n, dtype=np.int32)
    assert dst.transcode(src, h_src, bl, ss, out, ds, n, src_present=present, status=st) == G.E_UNRECOVERABLE
    assert [int(x) for x in np.flatnonzero(st)] == [bad_at] and st[bad_at] == G.E_UNRECOVERABLE
    assert np.array_equal(h_src, work)
    check_dst(dst_code, blocks, out, skip=(bad_at,))
    # DEVICE: the absent source data shards are overwritten with their rebuilt bytes
    d_src = torch.from_numpy(work).cuda()
    d_out = torch.full((n * 14 * ds,), SENT, dtype=torch.uint8, device="cuda")
    d_st = torch.zeros(n, dtype=torch.int32, device="cuda")
    dst.transcode(src, d_src, torch.from_numpy(bl).cuda(), ss, d_out, ds, n,
                  src_present=torch.from_numpy(present).cuda(), status=d_st)
    torch.cuda.synchronize()
    assert [int(x) for x in np.flatnonzero(d_st.cpu().numpy())] == [bad_at]
    check_dst(dst_code, blocks, d_out.cpu().numpy().reshape(n, 14, ds), skip=(bad_at,))
    rebuilt = d_src.cpu().numpy()
    for s in range(n):
        if s != bad_at:
            assert np.array_equal(rebuilt[s, :6], sh[s, :6]), s


def test_intact_batch_launches_no_reconstruct(torch):
    src_code, dst_code = ("rs", 6, 3, 0), ("rs", 10, 4, 0)
    lens = [5000] * 8
    src, dst = ctx_of(src_code), ctx_of(dst_code)
    ss, ds = stride_for(src_code, lens), stride_for(dst_code, lens)
    blocks, sh = make_source(src_code, lens, ss, 5)
    out = np.full((8, 14, ds), SENT, dtype=np.uint8)
    n0, s0 = dst.launch_count(), src.launch_count()
    dst.transcode(src, sh, np.array(lens, dtype=np.uint32), ss, out, ds, 8, src_present=np.ones((8, 9), dtype=np.uint8))
    assert src.launch_count() == s0  # the source context plans and rebuilds nothing
    assert dst.launch_count() - n0 == 3  # lengths, reframe, encode
    check_dst(dst_code, blocks, out)


@pytest.mark.parametrize("kind", [G.SUM_BLAKE2, G.SUM_ADLER8])
def test_tags_match_host_tags(torch, kind):
    src_code, dst_code = ("rs", 6, 3, 0), ("pb", 10, 4, 0)
    lens = [1, 777, 65536, 300001]
    src, dst = ctx_of(src_code), ctx_of(dst_code)
    dst.set_sum_kind(kind)
    ss, ds = stride_for(src_code, lens), stride_for(dst_code, lens)
    blocks, sh = make_source(src_code, lens, ss, 11)
    n = len(lens)
    d_out = torch.full((n * 14 * ds,), SENT, dtype=torch.uint8, device="cuda")
    d_sums = torch.zeros(n * 14 * 32, dtype=torch.uint8, device="cuda")
    dst.transcode(src, torch.from_numpy(sh).cuda(), torch.from_numpy(np.array(lens, dtype=np.uint32)).cuda(), ss, d_out,
                  ds, n, dst_sums=d_sums)
    torch.cuda.synchronize()
    check_dst(dst_code, blocks, d_out.cpu().numpy().reshape(n, 14, ds), d_sums.cpu().numpy().reshape(n, 14, 32), kind)


def test_graph_capture_replays_to_the_same_bytes(torch):
    src_code, dst_code = ("rs", 6, 3, 0), ("rs", 10, 4, 0)
    lens = [1 << 20, 300001, 17, 4095] * 4
    n = len(lens)
    src, dst = ctx_of(src_code), ctx_of(dst_code)
    ss, ds = stride_for(src_code, lens), stride_for(dst_code, lens)
    blocks, sh = make_source(src_code, lens, ss, 21)
    present = np.ones((n, 9), dtype=np.uint8)
    present[::3, 1] = 0
    work = sh.copy()
    work[present == 0] = 0
    d_src = torch.from_numpy(work).cuda()
    d_pr = torch.from_numpy(present).cuda()
    d_bl = torch.from_numpy(np.array(lens, dtype=np.uint32)).cuda()
    d_out = torch.full((n * 14 * ds,), SENT, dtype=torch.uint8, device="cuda")
    d_st = torch.zeros(n, dtype=torch.int32, device="cuda")
    dst.transcode(src, d_src, d_bl, ss, d_out, ds, n, src_present=d_pr, status=d_st)  # warm-up outside the capture
    torch.cuda.synchronize()
    d_src.copy_(torch.from_numpy(work).cuda())
    d_out.fill_(SENT)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        dst.transcode(src, d_src, d_bl, ss, d_out, ds, n, src_present=d_pr, status=d_st)
    for _ in range(2):
        d_src.copy_(torch.from_numpy(work).cuda())
        d_out.fill_(SENT)
        g.replay()
        torch.cuda.synchronize()
        assert not d_st.cpu().numpy().any()
        check_dst(dst_code, blocks, d_out.cpu().numpy().reshape(n, 14, ds))


def test_full_size_rs63_to_rs104(torch):
    """4096 x 1 MiB: every destination data byte against the reassembled blocks, every parity byte against the CPU
    oracle"""
    n, B = 4096, 1 << 20
    with G.GarageEc(0, 6, 3) as src, G.GarageEc(0, 10, 4) as dst:
        Ls, Ld = src.shard_len(B), dst.shard_len(B)
        ss, ds = src.stride_for(Ls), dst.stride_for(Ld)
        sh = torch.zeros((n, 9, ss), dtype=torch.uint8, device="cuda")
        tmp = torch.empty(n * 6 * ss, dtype=torch.uint8, device="cuda")
        src.fill_random(tmp, tmp.numel(), 0x5EED, 0)
        t3 = tmp.view(n, 6, ss)
        t3[:, :, Ls:] = 0
        t3[:, 5, Ls - (6 * Ls - B):] = 0
        sh[:, :6] = t3
        del tmp, t3  # the transcode reads only the data shards of an intact source
        out = torch.full((n, 14, ds), SENT, dtype=torch.uint8, device="cuda")
        bl = torch.full((n,), B, dtype=torch.int32, device="cuda")
        dst.transcode(src, sh.view(-1), bl, ss, out.view(-1), ds, n)
        torch.cuda.synchronize()
        blocks = sh[:, :6, :Ls].reshape(n, 6 * Ls)[:, :B]
        want = torch.zeros((n, 10 * Ld), dtype=torch.uint8, device="cuda")
        want[:, :B] = blocks
        assert torch.equal(out[:, :10, :Ld], want.view(n, 10, Ld))
        r16 = -(-Ld // 16) * 16
        assert (out[:, :, Ld:r16] == 0).all() and (out[:, :, r16:] == SENT).all()
        del want, blocks, sh
        h_data = np.ascontiguousarray(out[:, :10].cpu().numpy()).reshape(-1)
        want_par = O.encode(10, 4, O.build_matrix(10, 4, 0), h_data, ds, n, np.full(n, Ld, dtype=np.uint32), simd=True)
        got_par = out[:, 10:, :Ld].cpu().numpy()
        assert np.array_equal(got_par, want_par.reshape(n, 4, ds)[:, :, :Ld])


@pytest.mark.parametrize("fail_at", [0, 2, 5, 9, 14])
def test_host_ownership_under_injected_faults(torch, fail_at):
    src_code, dst_code = ("rs", 6, 3, 0), ("rs", 10, 4, 0)
    n, B = 400, 1 << 18  # several pipeline chunks
    lens = [B] * n
    src, dst = ctx_of(src_code), ctx_of(dst_code)
    ss, ds = stride_for(src_code, lens), stride_for(dst_code, lens)
    blocks, sh = make_source(src_code, lens[:1], ss, 3)
    sh = np.repeat(sh, n, axis=0)
    present = np.ones((n, 9), dtype=np.uint8)
    present[::2, 0] = 0
    work = sh.copy()
    work[present == 0] = 0
    bl = np.array(lens, dtype=np.uint32)
    out = np.full((n, 14, ds), SENT, dtype=np.uint8)
    sums = np.zeros((n, 14, 32), dtype=np.uint8)
    st = np.zeros(n, dtype=np.int32)
    dst.debug_fail_after(fail_at)
    with pytest.raises(G.EcError) as ei:
        dst.transcode(src, work, bl, ss, out, ds, n, src_present=present, dst_sums=sums, status=st)
    assert ei.value.code in (G.E_CUDA, G.E_NOMEM)
    dst.debug_fail_after(-1)
    out[:] = 0xEE
    sums[:] = 0xEE
    st[:] = 0x5A5A5A5A
    torch.cuda.synchronize()
    assert (out == 0xEE).all() and (sums == 0xEE).all() and (st == 0x5A5A5A5A).all()
    assert np.array_equal(work[present == 1], sh[present == 1])
    # the context is still usable and correct
    out[:] = SENT
    assert dst.transcode(src, work, bl, ss, out, ds, n, src_present=present, status=st) == 0
    check_dst(dst_code, blocks * n, out)


def test_argument_checks(torch):
    with G.GarageEc(0, 6, 3) as src, G.GarageEc(0, 10, 4) as dst:
        L = dst._L
        sh = np.zeros(9 * 1024, dtype=np.uint8)
        out = np.zeros(14 * 1024, dtype=np.uint8)
        pr = np.ones(9, dtype=np.uint8)
        p = G._ptr
        ok_len = np.array([1000], dtype=np.uint32)

        def call(dst_h, src_h, bl, s_stride, d_stride, present=None, n=1):
            return L.garage_ec_transcode(dst_h, src_h, p(sh), p(present), p(bl), s_stride, p(out), d_stride, None, None, n,
                                         G.MEM_HOST, None)

        assert call(None, src._h, ok_len, 1024, 1024) == G.E_INVALID
        assert call(dst._h, None, ok_len, 1024, 1024, present=pr) == G.E_INVALID  # whole blocks have no present
        assert call(dst._h, src._h, np.array([1 << 20], dtype=np.uint32), 1024, 1024) == G.E_INVALID  # strides too small
        assert call(dst._h, None, np.array([2000], dtype=np.uint32), 1024, 1024) == G.E_INVALID
        assert call(dst._h, src._h, ok_len, 1000, 1024) == G.E_ALIGN
        assert call(dst._h, src._h, ok_len, 1024, 1 << 29) == G.E_INVALID  # (k+m) * stride >= 4 GiB
        assert call(dst._h, src._h, ok_len, 1024, 1024) == 0
