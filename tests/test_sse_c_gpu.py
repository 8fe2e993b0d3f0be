"""SSE-C seal and open on the GPU (DESIGN.md 2.6, 4.9), checked against the scalar C oracle (tests/sse_c_oracle.py)
and against the context's own, separately tested encode: every code, ragged lengths, a distinct key and nonce per
block, work that outruns the grid, DEVICE == HOST, DEVICE under CUDA graph capture, every erasure pattern, and
tampered blocks failing alone."""
import ctypes as C
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

CODES = {
    "rs10_4": lambda: G.GarageEc(0, 10, 4),
    "rs6_3": lambda: G.GarageEc(0, 6, 3),
    "rs4_2": lambda: G.GarageEc(0, 4, 2),
    "lrc10_2_2": lambda: G.GarageEc.lrc(0, 10, 2, 2),
    "pb10_4": lambda: G.GarageEc.piggyback(0, 10, 4),
    "clay10_4": lambda: G.GarageEc.clay(0, 10, 4),
}
# 0, around chunk and vector edges, and a few multi-chunk blocks
LENS = [0, 1, 15, 16, 17, 4095, 4096, 4097, 8191, 8192, 8193, 12289, 3 * 4096 - 1, 40000, 100001]


def _batch(n, seed, lens=LENS):
    rng = np.random.default_rng(seed)
    ls = [lens[i % len(lens)] for i in range(n)]
    blocks = [rng.integers(0, 256, l, dtype=np.uint8) for l in ls]
    keys = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    nonces = rng.integers(0, 256, (n, 8), dtype=np.uint8)
    return blocks, keys, nonces


def _expected(ec, blocks, keys, nonces, stride):
    """B per block (oracle), the context's encode of B (HOST encode_blocks), blake2sum(B)"""
    Bs = [np.frombuffer(O.seal(keys[s].tobytes(), nonces[s].tobytes(), blocks[s]) if keys is not None
                        else blocks[s].tobytes(), dtype=np.uint8) for s in range(len(blocks))]
    tot = ec.k + ec.m
    par = np.zeros(len(Bs) * ec.m * stride, dtype=np.uint8)
    sums = np.zeros(len(Bs) * tot * 32, dtype=np.uint8)
    ec.encode_blocks([b.copy() for b in Bs], par, stride, sums_out=sums)
    want = np.zeros((len(Bs), tot, stride), dtype=np.uint8)
    for s, b in enumerate(Bs):
        L = ec.code_shard_len(b.size)
        for j in range(ec.k):
            piece = b[j * L:(j + 1) * L]
            want[s, j, :piece.size] = piece
        want[s, ec.k:] = par.reshape(len(Bs), ec.m, stride)[s]
    hashes = np.frombuffer(b"".join(G.blake2sum(b) for b in Bs), dtype=np.uint8)
    return Bs, want, hashes, sums


def _stride_for(ec, max_plain):
    return ec.stride_for(ec.code_shard_len(G.sealed_len(max_plain)))


def _plain_rows(blocks, pitch):
    rows = np.zeros(len(blocks) * pitch, dtype=np.uint8)
    for s, b in enumerate(blocks):
        rows[s * pitch:s * pitch + b.size] = b
    return rows


def _compare_shards(ec, got, want, Bs, stride):
    tot = ec.k + ec.m
    got = got.reshape(len(Bs), tot, stride)
    for s, b in enumerate(Bs):
        Lr = (ec.code_shard_len(b.size) + 15) // 16 * 16
        assert np.array_equal(got[s, :, :Lr], want[s, :, :Lr]), ("block", s, "len(B)", b.size)


@pytest.mark.parametrize("code", ["rs10_4", "rs6_3", "lrc10_2_2", "pb10_4", "clay10_4"])
def test_seal_matches_oracle_device_host_and_graph(code):
    ec = CODES[code]()
    n = 45
    blocks, keys, nonces = _batch(n, 7 + len(code))
    # the plain stride admits 300 chunks per block: n * 300 work items outrun the grid's warps several times over
    pitch = 300 * 4096
    stride = _stride_for(ec, pitch)
    tot = ec.k + ec.m
    Bs, want, hashes, sums = _expected(ec, blocks, keys, nonces, stride)
    plen = np.array([b.size for b in blocks], dtype=np.uint32)

    # HOST gather form and HOST contiguous form
    h_sh = np.zeros(n * tot * stride, dtype=np.uint8)
    h_hash = np.zeros(n * 32, dtype=np.uint8)
    h_sums = np.zeros(n * tot * 32, dtype=np.uint8)
    ec.seal_blocks(blocks, keys, nonces, h_sh, stride, h_hash, h_sums)
    _compare_shards(ec, h_sh, want, Bs, stride)
    assert np.array_equal(h_hash, hashes)
    assert np.array_equal(h_sums, sums)
    rows = _plain_rows(blocks, pitch)
    h2 = np.zeros_like(h_sh)
    h2_hash = np.zeros_like(h_hash)
    ec.seal(rows, pitch, plen, keys, nonces, h2, stride, h2_hash)
    _compare_shards(ec, h2, want, Bs, stride)
    assert np.array_equal(h2_hash, hashes)

    # DEVICE, into poisoned shards: nothing past roundup16(L) of a shard is written
    d_plain = torch.from_numpy(rows).cuda()
    d_len = torch.from_numpy(plen.view(np.int32)).cuda()
    d_keys = torch.from_numpy(keys.reshape(-1)).cuda()
    d_nonces = torch.from_numpy(nonces.reshape(-1)).cuda()
    d_sh = torch.full((n * tot * stride,), 0xA5, dtype=torch.uint8, device="cuda")
    d_hash = torch.zeros(n * 32, dtype=torch.uint8, device="cuda")
    d_sums = torch.zeros(n * tot * 32, dtype=torch.uint8, device="cuda")
    ec.seal(d_plain, pitch, d_len, d_keys, d_nonces, d_sh, stride, d_hash, d_sums, n=n)
    torch.cuda.synchronize()
    got = d_sh.cpu().numpy()
    _compare_shards(ec, got, want, Bs, stride)
    g3 = got.reshape(n, tot, stride)
    for s, b in enumerate(Bs):
        Lr = (ec.code_shard_len(b.size) + 15) // 16 * 16
        assert (g3[s, :, Lr:] == 0xA5).all(), s
    assert np.array_equal(d_hash.cpu().numpy(), hashes)
    assert np.array_equal(d_sums.cpu().numpy(), sums)

    # DEVICE inside a captured CUDA graph, replayed
    d_sh.fill_(0)
    d_hash.zero_()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            ec.seal(d_plain, pitch, d_len, d_keys, d_nonces, d_sh, stride, d_hash, n=n)
    g.replay()
    torch.cuda.synchronize()
    _compare_shards(ec, d_sh.cpu().numpy(), want, Bs, stride)
    assert np.array_equal(d_hash.cpu().numpy(), hashes)
    ec.close()


@pytest.mark.parametrize("code", ["rs10_4", "clay10_4"])
def test_seal_without_keys_is_encode_blocks(code):
    ec = CODES[code]()
    blocks, _, _ = _batch(20, 3)
    stride = _stride_for(ec, max(b.size for b in blocks))
    tot = ec.k + ec.m
    Bs, want, hashes, sums = _expected(ec, blocks, None, None, stride)
    sh = np.zeros(len(blocks) * tot * stride, dtype=np.uint8)
    hs = np.zeros(len(blocks) * 32, dtype=np.uint8)
    sm = np.zeros(len(blocks) * tot * 32, dtype=np.uint8)
    ec.seal_blocks(blocks, None, None, sh, stride, hs, sm)
    _compare_shards(ec, sh, want, Bs, stride)
    assert np.array_equal(hs, hashes) and np.array_equal(sm, sums)
    pitch = (max(b.size for b in blocks) + 15) // 16 * 16
    d_sh = torch.zeros(len(blocks) * tot * stride, dtype=torch.uint8, device="cuda")
    d_hash = torch.zeros(len(blocks) * 32, dtype=torch.uint8, device="cuda")
    plen = np.array([b.size for b in blocks], dtype=np.uint32)
    ec.seal(torch.from_numpy(_plain_rows(blocks, pitch)).cuda(), pitch, torch.from_numpy(plen.view(np.int32)).cuda(),
            None, None, d_sh, stride, d_hash, n=len(blocks))
    torch.cuda.synchronize()
    _compare_shards(ec, d_sh.cpu().numpy(), want, Bs, stride)
    assert np.array_equal(d_hash.cpu().numpy(), hashes)
    ec.close()


def _patterns(ec, rng, count):
    tot = ec.k + ec.m
    if ec.k + ec.m <= 9:  # every pattern of up to m erasures
        pats = [c for e in range(ec.m + 1) for c in itertools.combinations(range(tot), e)]
    else:
        pats = [tuple(rng.choice(tot, int(rng.integers(0, ec.m + 1)), replace=False)) for _ in range(count)]
    out = np.ones((len(pats), tot), dtype=np.uint8)
    for i, p in enumerate(pats):
        out[i, list(p)] = 0
    return out


def _sealed_stripes(ec, blocks, keys, nonces, stride):
    tot = ec.k + ec.m
    sh = np.zeros(len(blocks) * tot * stride, dtype=np.uint8)
    hs = np.zeros(len(blocks) * 32, dtype=np.uint8)
    ec.seal_blocks(blocks, keys, nonces, sh, stride, hs)
    sl = np.array([G.sealed_len(b.size) for b in blocks], dtype=np.uint32)
    return sh, hs, sl


@pytest.mark.parametrize("code", ["rs4_2", "rs6_3", "rs10_4", "lrc10_2_2", "pb10_4", "clay10_4"])
def test_open_round_trips_under_erasures(code):
    ec = CODES[code]()
    rng = np.random.default_rng(11)
    pres = _patterns(ec, rng, 60)
    n = len(pres)
    blocks, keys, nonces = _batch(n, 5 + n)
    pitch = (max(b.size for b in blocks) + 15) // 16 * 16
    stride = _stride_for(ec, pitch)
    tot = ec.k + ec.m
    sh, hs, sl = _sealed_stripes(ec, blocks, keys, nonces, stride)
    erased = sh.reshape(n, tot, stride).copy()
    erased[pres == 0] = 0x5C
    recoverable = np.array([ec.read_set(pres[s], np.arange(tot) < ec.k) is not None for s in range(n)])
    assert recoverable.any()

    # HOST gather form
    stripes = [erased[s].reshape(-1).copy() for s in range(n)]
    outs = [np.zeros(max(b.size, 1), dtype=np.uint8) for b in blocks]
    plen = np.zeros(n, dtype=np.uint32)
    bad = np.zeros(n, dtype=np.uint8)
    status = np.zeros(n, dtype=np.int32)
    ec.open_stripes(stripes, pres, sl, hs, keys, outs, plen, bad, status, stride)
    # DEVICE
    d_sh = torch.from_numpy(erased.reshape(-1).copy()).cuda()
    d_plain = torch.zeros(n * pitch, dtype=torch.uint8, device="cuda")
    d_plen = torch.zeros(n, dtype=torch.int32, device="cuda")
    d_bad = torch.zeros(n, dtype=torch.uint8, device="cuda")
    d_status = torch.zeros(n, dtype=torch.int32, device="cuda")
    ec.open(d_sh, torch.from_numpy(pres.reshape(-1)).cuda(), torch.from_numpy(sl.view(np.int32)).cuda(),
            torch.from_numpy(hs).cuda(), torch.from_numpy(keys.reshape(-1)).cuda(), d_plain, pitch, d_plen, d_bad,
            d_status, stride, n=n)
    torch.cuda.synchronize()
    dp = d_plain.cpu().numpy().reshape(n, pitch)
    for s in range(n):
        if recoverable[s]:
            assert status[s] == 0 and bad[s] == 0 and plen[s] == blocks[s].size, (s, status[s], bad[s])
            assert np.array_equal(outs[s][:blocks[s].size], blocks[s]), s
            assert int(d_status[s]) == 0 and int(d_bad[s]) == 0 and int(d_plen[s]) == blocks[s].size, s
            assert np.array_equal(dp[s, :blocks[s].size], blocks[s]), s
        else:
            assert status[s] == G.E_UNRECOVERABLE and int(d_status[s]) == G.E_UNRECOVERABLE, s
    ec.close()


@pytest.mark.parametrize("code", ["rs10_4", "pb10_4"])
def test_tampered_blocks_fail_alone(code):
    ec = CODES[code]()
    tot = ec.k + ec.m
    lens = [9000, 9000, 9000, 9000, 9000, 9000, 9000, 9000, 9000]
    n = len(lens)
    blocks, keys, nonces = _batch(n, 21, lens)
    stride = _stride_for(ec, 9000 + 4096)
    Bs = [np.frombuffer(O.seal(keys[s].tobytes(), nonces[s].tobytes(), blocks[s]), dtype=np.uint8).copy()
          for s in range(n)]
    good_hash = [G.blake2sum(b) for b in Bs]
    # 1 flipped ciphertext byte, 2 flipped tag byte, 3 chunks 0 and 1 swapped, 4 last chunk dropped, 5 wrong key,
    # 6 malformed length (8 + 4112 + 5): the hash recorded is the tampered block's, so only the tag or framing fails
    Bs[1][8 + 100] ^= 1
    Bs[2][8 + 4096 + 3] ^= 0x80
    c0, c1 = Bs[3][8:8 + 4112].copy(), Bs[3][8 + 4112:8 + 2 * 4112].copy()
    Bs[3][8:8 + 4112], Bs[3][8 + 4112:8 + 2 * 4112] = c1, c0
    Bs[4] = Bs[4][:8 + 2 * 4112].copy()
    keys = keys.copy()
    keys[5, 0] ^= 1
    Bs[6] = Bs[6][:8 + 4112 + 5].copy()
    hashes = np.frombuffer(b"".join(G.blake2sum(b) for b in Bs), dtype=np.uint8).copy()
    # 7: a modified byte under the original content hash: hash_bad and the tag both fail
    Bs[7][8 + 5000] ^= 4
    hashes[7 * 32:8 * 32] = np.frombuffer(good_hash[7], dtype=np.uint8)
    sl = np.array([b.size for b in Bs], dtype=np.uint32)
    stripes = []
    for b in Bs:
        L = ec.code_shard_len(b.size)
        st = np.zeros(tot * stride, dtype=np.uint8)
        for j in range(ec.k):
            piece = b[j * L:(j + 1) * L]
            st[j * stride:j * stride + piece.size] = piece
        stripes.append(st)
    pres = np.ones((n, tot), dtype=np.uint8)
    outs = [np.zeros(9000, dtype=np.uint8) for _ in range(n)]
    plen = np.zeros(n, dtype=np.uint32)
    bad = np.zeros(n, dtype=np.uint8)
    status = np.zeros(n, dtype=np.int32)
    rc = ec.open_stripes(stripes, pres, sl, hashes, keys, outs, plen, bad, status, stride)
    assert rc == G.E_AUTH
    assert list(status) == [0, G.E_AUTH, G.E_AUTH, G.E_AUTH, G.E_AUTH, G.E_AUTH, G.E_AUTH, G.E_AUTH, 0], list(status)
    assert list(bad) == [0, 0, 0, 0, 0, 0, 0, 1, 0], list(bad)
    for s in (0, 8):
        assert plen[s] == 9000 and np.array_equal(outs[s], blocks[s])
    for s in range(1, 8):
        assert not outs[s].any() and plen[s] == 0, s
    # DEVICE agrees
    pitch = 9008
    d_plain = torch.zeros(n * pitch, dtype=torch.uint8, device="cuda")
    d_status = torch.zeros(n, dtype=torch.int32, device="cuda")
    d_bad = torch.zeros(n, dtype=torch.uint8, device="cuda")
    d_plen = torch.zeros(n, dtype=torch.int32, device="cuda")
    ec.open(torch.from_numpy(np.concatenate(stripes)).cuda(), torch.from_numpy(pres.reshape(-1)).cuda(),
            torch.from_numpy(sl.view(np.int32)).cuda(), torch.from_numpy(hashes).cuda(),
            torch.from_numpy(keys.reshape(-1)).cuda(), d_plain, pitch, d_plen, d_bad, d_status, stride, n=n)
    torch.cuda.synchronize()
    assert list(d_status.cpu().numpy()) == list(status)
    assert list(d_bad.cpu().numpy()) == list(bad)
    dp = d_plain.cpu().numpy().reshape(n, pitch)
    for s in (0, 8):
        assert np.array_equal(dp[s, :9000], blocks[s])
    assert not dp[1:8].any()
    ec.close()


def test_seal_and_open_reject_bad_arguments_before_gpu_work():
    ec = G.GarageEc(0, 10, 4)
    L = ec._L
    n, tot = 2, 14
    stride = _stride_for(ec, 4096)
    plain = np.zeros(n * 4096 + 16, dtype=np.uint8)
    lens = np.array([4096, 100], dtype=np.uint32)
    keys = np.zeros(n * 32, dtype=np.uint8)
    nonces = np.zeros(n * 8, dtype=np.uint8)
    shards = np.zeros(n * tot * stride + 16, dtype=np.uint8)
    hashes = np.zeros(n * 32, dtype=np.uint8)
    P = lambda a, off=0: G._ptr(a) if off == 0 else a.ctypes.data + off  # noqa: E731

    def seal(plain_p=None, stride_p=4096, lens_a=lens, keys_a=keys, nonces_a=nonces, sh=None, st=stride):
        return L.garage_ec_seal(ec._h, plain_p if plain_p is not None else P(plain), stride_p, G._ptr(lens_a),
                                G._ptr(keys_a), G._ptr(nonces_a), sh if sh is not None else P(shards), st, P(hashes),
                                None, n, G.MEM_HOST, None)

    assert seal() == 0
    assert seal(keys_a=keys, nonces_a=None) == G.E_INVALID        # keys without nonces
    assert seal(keys_a=None, nonces_a=nonces) == G.E_INVALID      # nonces without keys
    assert seal(plain_p=P(plain, 8)) == G.E_ALIGN                 # misaligned plain
    assert seal(sh=P(shards, 8)) == G.E_ALIGN                     # misaligned shards
    assert seal(stride_p=4100) == G.E_INVALID                     # plain_stride not a multiple of 16
    assert seal(lens_a=np.array([4097, 1], dtype=np.uint32)) == G.E_INVALID  # plain_len > plain_stride
    small = ((ec.code_shard_len(G.sealed_len(4096)) - 1) // 16) * 16
    assert seal(st=small) == G.E_INVALID                          # L > stride (HOST)
    assert seal(st=stride + 8) == G.E_ALIGN                       # stride not a multiple of 16
    blocks = (C.c_void_p * n)(plain.ctypes.data, None)
    assert L.garage_ec_seal_blocks(ec._h, C.cast(blocks, C.c_void_p), G._ptr(lens), G._ptr(keys), G._ptr(nonces),
                                   P(shards), stride, P(hashes), None, n) == G.E_INVALID  # NULL block of length 100

    sl = np.array([G.sealed_len(4096), 24], dtype=np.uint32)
    pres = np.ones(n * tot, dtype=np.uint8)
    outp = np.zeros(n * 4096, dtype=np.uint8)
    plen, bad, status = np.zeros(n, dtype=np.uint32), np.zeros(n, dtype=np.uint8), np.zeros(n, dtype=np.int32)

    def open_(keys_a=keys, sl_a=sl, st=stride, plain_stride=4096, sh=None):
        return L.garage_ec_open(ec._h, sh if sh is not None else P(shards), G._ptr(pres), G._ptr(sl_a), P(hashes),
                                G._ptr(keys_a), P(outp), plain_stride, G._ptr(plen), G._ptr(bad), G._ptr(status), st, n,
                                G.MEM_HOST, None)

    assert open_(keys_a=None) == G.E_INVALID                      # keys are required
    assert open_(sh=P(shards, 8)) == G.E_ALIGN
    assert open_(plain_stride=4100) == G.E_INVALID
    assert open_(plain_stride=4080) == G.E_INVALID                # plaintext past plain_stride
    assert open_(st=small) == G.E_INVALID                         # L > stride (HOST)
    ec.close()
