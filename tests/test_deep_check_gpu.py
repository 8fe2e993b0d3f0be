"""garage_ec_deep_check: the blake2sum of every stripe's block, read straight from its data shards, against
hashlib.blake2b(block, digest_size=64).digest()[:32], and the parity verdict against garage_ec_verify with the code's
shard length, for RS, LRC, PB and Clay.  Every shard's bytes past L are poisoned with 0xA5, so a loader that hashes
them fails.  Also: HOST against DEVICE, a CUDA-graph replay, the argument / geometry errors and a 4096 x 1 MiB batch."""
import ctypes as C
import hashlib
import os
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import garage_b200 as G  # noqa: E402

torch = pytest.importorskip("torch")

RS_KS = (1, 2, 4, 6, 10, 12, 16, 17, 32)
CODES = [("rs", k, 2 if k == 1 else 4) for k in RS_KS] + [
    ("lrc", 10, 4), ("pb", 6, 3), ("pb", 10, 4), ("clay", 4, 2), ("clay", 6, 3), ("clay", 10, 4)]


def make_ctx(kind, k, m):
    if kind == "rs":
        return G.GarageEc(0, k, m)
    if kind == "lrc":
        return G.GarageEc.lrc(0, k, 2, m - 2)
    if kind == "pb":
        return G.GarageEc.piggyback(0, k, m)
    return G.GarageEc.clay(0, k, m)


def ragged_lens(k):
    """tiny blocks, lengths around one message block, blocks whose last data shards are pure padding (3 and 41 bytes
    for k = 10), L = 2000..2015 (every L % 16 residue, each a little short of k * L) and a 1 MiB block"""
    return [1, 3, 41, 127, 128, 129] + [k * L - (L % k) for L in range(2000, 2016)] + [1 << 20]


def build(ec, lens, seed):
    """(shards (n, k+m, stride) on the device, block_len int32 tensor, L list, expected hashes (n, 32) uint8, stride)"""
    k, m, n = ec.k, ec.m, len(lens)
    Ls = [ec.code_shard_len(x) for x in lens]
    unit = max(128, ec.code_shard_len(1))  # PB / Clay framing quantum
    stride = (max(Ls) + unit - 1) // unit * unit
    g = torch.Generator(device="cuda").manual_seed(seed)
    data = torch.zeros((n, k, stride), dtype=torch.uint8, device="cuda")
    hashes = np.zeros((n, 32), dtype=np.uint8)
    for s, (ln, L) in enumerate(zip(lens, Ls)):
        blk = torch.randint(0, 256, (k * L,), generator=g, device="cuda", dtype=torch.uint8)
        blk[ln:] = 0
        data[s, :, :L] = blk.view(k, L)
        hashes[s] = np.frombuffer(hashlib.blake2b(blk[:ln].cpu().numpy().tobytes(), digest_size=64).digest()[:32],
                                  dtype=np.uint8)
    parity = torch.zeros((n, m, stride), dtype=torch.uint8, device="cuda")
    sl = torch.tensor(Ls, dtype=torch.int32, device="cuda")
    ec.encode(data, parity, stride, n, shard_len=sl)
    sh = torch.cat([data, parity], dim=1).contiguous()
    for s, L in enumerate(Ls):
        sh[s, :, L:] = 0xA5  # not part of the block, nor of the parity
    torch.cuda.synchronize()
    return sh, torch.tensor(lens, dtype=torch.int32, device="cuda"), Ls, hashes, stride


def deep_device(ec, sh, blen, hashes, stride):
    n = blen.numel()
    bad = torch.full((n,), 7, dtype=torch.uint8, device="cuda")
    mm = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    ec.deep_check(sh, blen, torch.from_numpy(hashes).cuda(), bad, mm, stride, n)
    torch.cuda.synchronize()
    return bad.cpu().numpy(), mm.cpu().numpy().view(np.uint32)


def deep_host(ec, sh, blen, hashes, stride):
    n = blen.numel()
    bad = np.full(n, 7, dtype=np.uint8)
    mm = np.full(n, 0xFFFFFFFF, dtype=np.uint32)
    ec.deep_check(sh.cpu().numpy(), blen.cpu().numpy().view(np.uint32), hashes, bad, mm, stride, n)
    return bad, mm


def verify_ref(ec, sh, Ls, stride):
    n = len(Ls)
    mm = torch.zeros(n, dtype=torch.int32, device="cuda")
    ec.verify(sh, mm, stride, n, shard_len=torch.tensor(Ls, dtype=torch.int32, device="cuda"))
    torch.cuda.synchronize()
    return mm.cpu().numpy().view(np.uint32)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,k,m", CODES, ids=["%s%d_%d" % c for c in CODES])
def test_block_hash_and_parity_verdict(kind, k, m):
    ec = make_ctx(kind, k, m)
    lens = ragged_lens(k)
    sh, blen, Ls, hashes, stride = build(ec, lens, 0xDEE9 + k * 31 + m)
    n = len(lens)
    bad, mm = deep_device(ec, sh, blen, hashes, stride)
    assert (bad == 0).all(), [lens[s] for s in np.nonzero(bad)[0]]
    assert (mm == 0).all()
    # a wrong content address, corrupted parity rows and a corrupted data byte
    hashes2 = hashes.copy()
    hashes2[1, 5] ^= 0x10
    hashes2[n - 1, 31] ^= 0x01
    rows = {0: [0], 3: [m - 1], 7: list(range(m)), n - 2: [1 % m]}
    for s, rs in rows.items():
        for i in rs:
            sh[s, k + i, Ls[s] // 2] ^= 0x3C
    pos = lens[9] // 2  # a data byte inside the block
    sh[9, pos // Ls[9], pos % Ls[9]] ^= 0x01
    torch.cuda.synchronize()
    bad, mm = deep_device(ec, sh, blen, hashes2, stride)
    want_bad = np.zeros(n, dtype=np.uint8)
    want_bad[[1, n - 1, 9]] = 1
    assert np.array_equal(bad, want_bad)
    ref = verify_ref(ec, sh, Ls, stride)
    assert np.array_equal(mm, ref)
    for s, rs in rows.items():
        for i in rs:
            assert (mm[s] >> i) & 1, (s, i)
    hb, hm = deep_host(ec, sh, blen, hashes2, stride)
    assert np.array_equal(hb, bad) and np.array_equal(hm, mm)


@pytest.mark.gpu
def test_device_call_replays_in_a_cuda_graph():
    ec = G.GarageEc(0, 10, 4)
    lens = ragged_lens(10)
    sh, blen, Ls, hashes, stride = build(ec, lens, 0x6A9)
    n = len(lens)
    sh[4, 11, 3] ^= 0xFF
    hashes[2, 0] ^= 1
    d_hash = torch.from_numpy(hashes).cuda()
    bad = torch.zeros(n, dtype=torch.uint8, device="cuda")
    mm = torch.zeros(n, dtype=torch.int32, device="cuda")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        ec.deep_check(sh, blen, d_hash, bad, mm, stride, n)  # warm-up outside the capture
    torch.cuda.synchronize()
    want_bad, want_mm = bad.cpu().clone(), mm.cpu().clone()
    assert want_bad.tolist() == [1 if i == 2 else 0 for i in range(n)]
    assert want_mm[4].item() == 2
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ec.deep_check(sh, blen, d_hash, bad, mm, stride, n)
    for _ in range(2):
        bad.fill_(9)
        mm.fill_(-1)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(bad.cpu(), want_bad) and torch.equal(mm.cpu(), want_mm)


@pytest.mark.gpu
def test_argument_and_geometry_errors():
    ec = G.GarageEc(0, 10, 4)
    L = ec._L
    lens = [1000, 2000, 3000]
    sh, blen, Ls, hashes, stride = build(ec, lens, 0xE77)
    n = len(lens)
    d_hash = torch.from_numpy(hashes).cuda()
    bad = torch.zeros(n, dtype=torch.uint8, device="cuda")
    mm = torch.zeros(n, dtype=torch.int32, device="cuda")
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    P = G._ptr
    call = lambda *a: L.garage_ec_deep_check(ec._h, *a)  # noqa: E731
    assert call(P(sh), P(blen), P(d_hash), P(bad), P(mm), stride, n, 7, st) == G.E_INVALID
    assert L.garage_ec_deep_check(None, P(sh), P(blen), P(d_hash), P(bad), P(mm), stride, n, G.MEM_DEVICE, st) == G.E_INVALID
    for i in range(5):
        args = [P(sh), P(blen), P(d_hash), P(bad), P(mm)]
        args[i] = None
        assert call(*args, stride, n, G.MEM_DEVICE, st) == G.E_INVALID, i
    assert call(None, None, None, None, None, stride, 0, G.MEM_DEVICE, st) == G.OK
    assert call(C.c_void_p(sh.data_ptr() + 8), P(blen), P(d_hash), P(bad), P(mm), stride, n, G.MEM_DEVICE, st) == G.E_ALIGN
    assert call(P(sh), P(blen), P(d_hash), P(bad), P(mm), stride + 8, n, G.MEM_DEVICE, st) == G.E_ALIGN
    # a block whose shards do not fit the stride: DEVICE reports the stripe, HOST refuses the call
    big = blen.clone()
    big[1] = 10 * stride + 1
    bad.fill_(0)
    mm.fill_(0)
    assert call(P(sh), P(big), P(d_hash), P(bad), P(mm), stride, n, G.MEM_DEVICE, st) == G.OK
    torch.cuda.synchronize()
    assert bad.cpu().tolist() == [0, 1, 0] and mm.cpu().tolist() == [0, 0xF, 0]
    h_sh, h_big = sh.cpu().numpy(), big.cpu().numpy().view(np.uint32)
    h_bad, h_mm = np.zeros(n, dtype=np.uint8), np.zeros(n, dtype=np.uint32)
    assert L.garage_ec_deep_check(ec._h, P(h_sh), P(h_big), P(hashes), P(h_bad), P(h_mm), stride, n, G.MEM_HOST,
                                  None) == G.E_INVALID


@pytest.mark.gpu
def test_4096_one_mib_blocks_match_hashlib():
    ec = G.GarageEc(0, 10, 4)
    n, ln, k, m = 4096, 1 << 20, 10, 4
    L = ec.code_shard_len(ln)
    stride = ec.stride_for(L)
    g = torch.Generator(device="cuda").manual_seed(0x4096)
    blk = torch.randint(0, 256, (n, k * L), generator=g, device="cuda", dtype=torch.uint8)
    blk[:, ln:] = 0
    sh = torch.full((n, k + m, stride), 0xA5, dtype=torch.uint8, device="cuda")
    sh[:, :k, :L] = blk.view(n, k, L)
    host = blk[:, :ln].cpu().numpy()
    del blk
    with ThreadPoolExecutor(max(1, min(32, os.cpu_count() or 1))) as ex:
        digests = list(ex.map(lambda s: hashlib.blake2b(host[s].data, digest_size=64).digest()[:32], range(n)))
    hashes = np.frombuffer(b"".join(digests), dtype=np.uint8).reshape(n, 32).copy()
    hashes[1234, 7] ^= 0x80
    blen = torch.full((n,), ln, dtype=torch.int32, device="cuda")
    bad, _ = deep_device(ec, sh, blen, hashes, stride)
    assert np.nonzero(bad)[0].tolist() == [1234]
