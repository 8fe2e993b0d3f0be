"""S3 CRC32 / CRC32C checksums of the plaintext, computed by the seal and reseal chunk kernels (DESIGN.md 2.9, 4.12):
garage_ec_seal_crc, garage_ec_seal_blocks_crc, garage_ec_reseal_crc and garage_ec_reseal_stripes_crc.

Expected values never come from the library: CRC32 from zlib, CRC32C from the bitwise C oracle (tests/crc_oracle.py).
Every other output must be byte-identical to the same call without checksums.  Seal: keyed and unkeyed, every code
family, every residue mod 16 around chunk boundaries, 0 and 1 bytes, multiples of 4096, past 256 chunks, full 1 MiB
blocks and 4096 of them, mixed kinds in one batch.  Reseal: the piece lists of test_reseal_gpu (every residue mod 16,
chunk boundaries and seams), plaintext sources, every erasure pattern of RS(4,2), failed destinations.  DEVICE == HOST
== gather form, CUDA graph capture and replay, unknown kinds, and the HOST ownership contract under injected faults."""
import itertools
import os
import sys
import zlib

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import crc_oracle as CO  # noqa: E402
import garage_b200 as G  # noqa: E402
from test_reseal_gpu import CODES as RESEAL_CODES, Case, Out, dev  # noqa: E402
from test_sse_c_geometry_gpu import Code  # noqa: E402

pytestmark = pytest.mark.gpu

MiB = 1 << 20
SEAL_CODES = {"rs10_4": ("rs", 10, 4), "rs4_2": ("rs", 4, 2), "lrc10_2_2": ("lrc", 10, 2, 2), "pb10_4": ("pb", 10, 4),
              "clay10_4": ("clay", 10, 4)}
POISON = 0xA5
CRC_SENT = 0xDEADBEEF


def want_crc(kind, b):
    b = bytes(b)
    return 0 if kind == 0 else zlib.crc32(b) if kind == 1 else CO.crc(CO.CRC32C, b)


def seal_lens():
    """every residue mod 16 around the first chunk boundaries, 0 and 1, multiples of 4096, past 256 chunks, 1 MiB"""
    lens = [0, 1, 2, 15, 16, 17, 4096, 8192, 3 * 4096, MiB, MiB + 4097, MiB - 977]
    lens += [4096 * j + r for j in (1, 2) for r in range(-16, 17) if r]
    return lens


@pytest.fixture(scope="module")
def torch():
    import torch as t

    assert t.cuda.is_available()
    return t


def plain_rows(plains, pitch):
    rows = np.zeros((len(plains), pitch), dtype=np.uint8)
    for i, p in enumerate(plains):
        rows[i, :p.size] = p
    return rows


def seal_call(torch, ec, code, rows, lens, keys, nonces, stride, form, kinds=None, n_poison=POISON):
    """one seal; form: device / host / blocks.  Returns (shards, hashes, sums, crcs) as numpy arrays"""
    n, pitch = rows.shape
    tot = code.tot
    outs = dict(shards=np.full(n * tot * stride, n_poison, np.uint8), hashes=np.zeros(n * 32, np.uint8),
                sums=np.zeros(n * tot * 32, np.uint8), crcs=np.full(n, CRC_SENT, np.uint32))
    crc_args = {} if kinds is None else {"crc_kind": kinds, "crcs": outs["crcs"]}
    if form == "device":
        d = {k: dev(torch, v) for k, v in outs.items()}
        if kinds is not None:
            crc_args = {"crc_kind": dev(torch, kinds), "crcs": d["crcs"]}
        ec.seal(dev(torch, rows.reshape(-1)), pitch, dev(torch, lens), None if keys is None else dev(torch, keys),
                None if nonces is None else dev(torch, nonces), d["shards"], stride, d["hashes"], sums=d["sums"],
                **crc_args)
        torch.cuda.synchronize()
        outs = {k: v.cpu().numpy().view(outs[k].dtype) for k, v in d.items()}
    elif form == "host":
        ec.seal(rows.reshape(-1), pitch, lens, keys, nonces, outs["shards"], stride, outs["hashes"], sums=outs["sums"],
                **crc_args)
    else:
        ec.seal_blocks([rows[i, :lens[i]].copy() for i in range(n)], keys, nonces, outs["shards"], stride,
                       outs["hashes"], sums=outs["sums"], **crc_args)
    return outs


@pytest.mark.parametrize("name", list(SEAL_CODES))
def test_seal_checksums_every_geometry(torch, name):
    code = Code(SEAL_CODES[name])
    rng = np.random.default_rng(0xC5C + len(name))
    lens = np.array(seal_lens(), dtype=np.uint32)
    n = lens.size
    plains = [rng.integers(0, 256, int(x), dtype=np.uint8) for x in lens]
    pitch = (int(lens.max()) + 15) // 16 * 16
    rows = plain_rows(plains, pitch)
    for i, p in enumerate(plains):  # garbage past the plaintext: masked out of the checksum
        rows[i, p.size:min(pitch, p.size + 16)] = 0xEE
    kinds = (np.arange(n) % 3).astype(np.uint8)  # none, CRC32, CRC32C mixed in one batch
    keys = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    nonces = rng.integers(0, 256, (n, 8), dtype=np.uint8)
    with code.ctx() as ec:
        stride = max(128, -(-max(code.shard_len(G.sealed_len(int(x))) for x in lens) // 128) * 128)
        for keyed in (True, False):
            k_, n_ = (keys, nonces) if keyed else (None, None)
            base = seal_call(torch, ec, code, rows, lens, k_, n_, stride, "device")
            want = np.array([want_crc(int(kinds[i]), plains[i]) for i in range(n)], dtype=np.uint32)
            for form in ("device", "host", "blocks"):
                got = seal_call(torch, ec, code, rows, lens, k_, n_, stride, form, kinds=kinds)
                for k in ("shards", "hashes", "sums"):
                    assert np.array_equal(got[k], base[k]), (name, keyed, form, k)
                bad = np.nonzero(got["crcs"] != want)[0]
                assert bad.size == 0, (name, keyed, form, [(int(lens[i]), int(kinds[i])) for i in bad[:5]])
            # every block under each kind, so each length meets both polynomials
            for kind in (1, 2):
                got = seal_call(torch, ec, code, rows, lens, k_, n_, stride, "device",
                                kinds=np.full(n, kind, np.uint8))
                assert [int(x) for x in got["crcs"]] == [want_crc(kind, p) for p in plains], (name, keyed, kind)


def test_seal_checksums_full_size(torch):
    """4096 x 1 MiB RS(10,4), DEVICE, kinds alternating: CRC32 against zlib and CRC32C against the oracle"""
    code = Code(("rs", 10, 4))
    n, B = 4096, MiB
    with code.ctx() as ec:
        stride = -(-code.shard_len(G.sealed_len(B)) // 128) * 128
        g = torch.Generator(device="cuda").manual_seed(0xC5C0)
        plain = torch.randint(0, 256, (n, B), dtype=torch.uint8, device="cuda", generator=g)
        lens = torch.full((n,), B, dtype=torch.int32, device="cuda")
        keys = torch.randint(0, 256, (n, 32), dtype=torch.uint8, device="cuda", generator=g)
        nonces = torch.randint(0, 256, (n, 8), dtype=torch.uint8, device="cuda", generator=g)
        kinds_np = (1 + np.arange(n) % 2).astype(np.uint8)
        outs = []
        for with_crc in (False, True):
            sh = torch.zeros(n * code.tot * stride, dtype=torch.uint8, device="cuda")
            hs = torch.zeros(n * 32, dtype=torch.uint8, device="cuda")
            crcs = torch.zeros(n, dtype=torch.int32, device="cuda")
            kw = {"crc_kind": dev(torch, kinds_np), "crcs": crcs} if with_crc else {}
            ec.seal(plain.view(-1), B, lens, keys.view(-1), nonces.view(-1), sh, stride, hs, **kw)
            torch.cuda.synchronize()
            outs.append((sh, hs, crcs))
        assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
        del outs[0]
        crcs = outs[0][2].cpu().numpy().view(np.uint32)
        host = plain.cpu().numpy()
        for s in range(n):
            assert int(crcs[s]) == want_crc(int(kinds_np[s]), host[s]), s


def reseal_call(torch, ec, c, pr, form, kinds=None, src_keys="same", out=None):
    device = form == "device"
    out = out or Out(torch, c, device)
    crcs = np.full(c.n_dst, CRC_SENT, np.uint32)
    conv = (lambda a: None if a is None else dev(torch, a)) if device else (lambda a: a)
    keys = (c.src_keys if c.keyed else None) if isinstance(src_keys, str) else src_keys
    crcs_arg = conv(crcs)
    kw = {} if kinds is None else {"crc_kind": conv(kinds), "crcs": crcs_arg}
    args = [conv(pr), conv(c.src_len), conv(c.src_hashes), conv(keys), conv(c.pieces), conv(c.piece_start),
            conv(c.dst_keys), conv(c.dst_nonces), out.shards, out.hashes, out.dlen, out.bad, out.src_status,
            out.status, c.stride]
    if form == "stripes":
        rc = ec.reseal_stripes([c.src_shards[i].reshape(-1).copy() for i in range(c.n_src)], *args, dst_sums=out.sums,
                               **kw)
    else:
        src = c.src_shards.reshape(-1)
        rc = ec.reseal(conv(src) if device else src.copy(), *args, dst_sums=out.sums, n_src=c.n_src, n_dst=c.n_dst,
                       **kw)
    if device:
        torch.cuda.synchronize()
        crcs = crcs_arg.cpu().numpy().view(np.uint32) if kinds is not None else crcs
    return out.host(), crcs, rc


def dst_kinds(n):
    return (np.arange(n) % 3).astype(np.uint8)


@pytest.mark.parametrize("name", ["rs10_4", "lrc10_2_2", "pb10_4", "clay10_4"])
@pytest.mark.parametrize("keyed", [True, False])
def test_reseal_checksums(torch, name, keyed):
    code = Code(RESEAL_CODES[name])
    c = Case(code, 0xC5E + len(name), keyed=keyed)
    kinds = dst_kinds(c.n_dst)
    want = [want_crc(int(kinds[d]), c.Q[d]) for d in range(c.n_dst)]
    pr = np.ones((c.n_src, code.tot), dtype=np.uint8)
    with code.ctx() as ec:
        base, _, _ = reseal_call(torch, ec, c, pr, "device")
        for form in ("device", "host", "stripes"):
            got, crcs, rc = reseal_call(torch, ec, c, pr, form, kinds=kinds)
            for k in base:
                assert np.array_equal(got[k], base[k]), (name, keyed, form, k)
            assert (got["status"] == 0).all()
            assert [int(x) for x in crcs] == want, (name, keyed, form)
        got, crcs, _ = reseal_call(torch, ec, c, pr, "device", kinds=np.full(c.n_dst, 2, np.uint8))
        assert [int(x) for x in crcs] == [want_crc(2, q) for q in c.Q]


def test_reseal_checksums_every_erasure_pattern_rs4_2(torch):
    code = Code(("rs", 4, 2))
    lens = [2, 17, 4095, 4097, 40000]
    dests = [[(i, 0, n)] for i, n in enumerate(lens)] + [[(4, 7, 5000), (2, 1, 4000), (3, 4096, 1)]]
    c = Case(code, 0xC5F, lens=lens, dests=dests)
    kinds = np.array([1, 2, 1, 2, 1, 2], dtype=np.uint8)
    want = [want_crc(int(kinds[d]), c.Q[d]) for d in range(c.n_dst)]
    with code.ctx() as ec:
        for r in range(code.m + 1):
            for lost in itertools.combinations(range(code.tot), r):
                pr = np.ones((c.n_src, code.tot), dtype=np.uint8)
                pr[:, list(lost)] = 0
                shards = c.src_shards.copy()
                shards[:, list(lost)] = 0x5C
                c2 = Case.__new__(Case)
                c2.__dict__.update(c.__dict__)
                c2.src_shards = shards
                got, crcs, rc = reseal_call(torch, ec, c2, pr, "device", kinds=kinds)
                assert (got["status"] == 0).all(), lost
                assert [int(x) for x in crcs] == want, lost


def test_reseal_failed_destinations_are_not_reported(torch):
    """a wrong key for one source fails the destinations that name it; the others still get their checksums"""
    code = Code(("rs", 10, 4))
    c = Case(code, 0xC60)
    kinds = np.full(c.n_dst, 2, np.uint8)
    keys = c.src_keys.copy()
    keys[14] ^= 1
    with code.ctx() as ec:
        for form in ("device", "host"):
            got, crcs, rc = reseal_call(torch, ec, c, np.ones((c.n_src, code.tot), np.uint8), form, kinds=kinds,
                                        src_keys=keys)
            failed = {d for d in range(c.n_dst) if 14 in c.names(d)}
            assert failed
            for d in range(c.n_dst):
                if d in failed:
                    assert got["status"][d] == G.E_AUTH, (form, d)
                else:
                    assert got["status"][d] == 0 and int(crcs[d]) == want_crc(2, c.Q[d]), (form, d)


def test_unknown_kinds(torch):
    code = Code(("rs", 4, 2))
    rng = np.random.default_rng(0xC61)
    lens = np.array([100, 5000, 9000], dtype=np.uint32)
    plains = [rng.integers(0, 256, int(x), dtype=np.uint8) for x in lens]
    rows = plain_rows(plains, 9008)
    keys = rng.integers(0, 256, (3, 32), dtype=np.uint8)
    nonces = rng.integers(0, 256, (3, 8), dtype=np.uint8)
    kinds = np.array([1, 3, 2], dtype=np.uint8)
    with code.ctx() as ec:
        stride = 4096
        base = seal_call(torch, ec, code, rows, lens, keys, nonces, stride, "device")
        # DEVICE: block 1 is malformed -- its shards are not written -- and the others are sealed and checksummed
        got = seal_call(torch, ec, code, rows, lens, keys, nonces, stride, "device", kinds=kinds)
        sh, bsh = got["shards"].reshape(3, -1), base["shards"].reshape(3, -1)
        assert (sh[1] == POISON).all()
        assert np.array_equal(sh[[0, 2]], bsh[[0, 2]])
        assert int(got["crcs"][0]) == want_crc(1, plains[0]) and int(got["crcs"][2]) == want_crc(2, plains[2])
        # HOST: refused before any GPU work, nothing written
        for form in ("host", "blocks"):
            with pytest.raises(G.EcError) as ei:
                seal_call(torch, ec, code, rows, lens, keys, nonces, stride, form, kinds=kinds)
            assert ei.value.code == G.E_INVALID
        # reseal: DEVICE status E_INVALID for that destination, HOST refused
        c = Case(code, 0xC62, lens=[50, 6000], dests=[[(0, 0, 50)], [(1, 0, 6000)], [(1, 3, 10), (0, 1, 2)]])
        rk = np.array([2, 9, 1], dtype=np.uint8)
        pr = np.ones((c.n_src, code.tot), np.uint8)
        got, crcs, rc = reseal_call(torch, ec, c, pr, "device", kinds=rk)
        assert list(got["status"]) == [0, G.E_INVALID, 0]
        assert int(crcs[0]) == want_crc(2, c.Q[0]) and int(crcs[2]) == want_crc(1, c.Q[2])
        for form in ("host", "stripes"):
            with pytest.raises(G.EcError) as ei:
                reseal_call(torch, ec, c, pr, form, kinds=rk)
            assert ei.value.code == G.E_INVALID


def test_graph_capture_and_replay(torch):
    code = Code(("rs", 10, 4))
    rng = np.random.default_rng(0xC63)
    lens = np.array([MiB, 1, 4097, MiB + 4097, 0, 300001], dtype=np.uint32)
    n = lens.size
    plains = [rng.integers(0, 256, int(x), dtype=np.uint8) for x in lens]
    pitch = (int(lens.max()) + 15) // 16 * 16
    kinds = np.array([1, 2, 0, 2, 1, 2], dtype=np.uint8)
    want = np.array([want_crc(int(kinds[i]), plains[i]) for i in range(n)], dtype=np.uint32)
    with code.ctx() as ec:
        stride = -(-code.shard_len(G.sealed_len(int(lens.max()))) // 128) * 128
        ins = [dev(torch, a) for a in (plain_rows(plains, pitch).reshape(-1), lens,
                                       rng.integers(0, 256, (n, 32), dtype=np.uint8),
                                       rng.integers(0, 256, (n, 8), dtype=np.uint8), kinds)]
        sh = torch.zeros(n * code.tot * stride, dtype=torch.uint8, device="cuda")
        hs = torch.zeros(n * 32, dtype=torch.uint8, device="cuda")
        crcs = torch.zeros(n, dtype=torch.int32, device="cuda")

        def call():
            ec.seal(ins[0], pitch, ins[1], ins[2], ins[3], sh, stride, hs, crc_kind=ins[4], crcs=crcs)

        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            call()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        first = (sh.clone(), hs.clone())
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            call()
        for _ in range(2):
            crcs.fill_(0x5A5A5A5A)
            sh.zero_()
            g.replay()
            torch.cuda.synchronize()
            assert np.array_equal(crcs.cpu().numpy().view(np.uint32), want)
            assert torch.equal(sh, first[0]) and torch.equal(hs, first[1])
        del g

        # the reseal: every destination's checksum after each replay
        c = Case(code, 0xC64, lens=[5000, 70000], dests=[[(0, 0, 5000)], [(1, 17, 60000), (0, 3, 4000)]])
        rk = np.array([2, 1], dtype=np.uint8)
        out = Out(torch, c, True)
        d_crcs = torch.zeros(c.n_dst, dtype=torch.int32, device="cuda")
        rins = [dev(torch, a) for a in (c.src_shards.reshape(-1), np.ones((c.n_src, code.tot), np.uint8), c.src_len,
                                        c.src_hashes, c.src_keys, c.pieces, c.piece_start, c.dst_keys, c.dst_nonces,
                                        rk)]

        def rcall():
            ec.reseal(*rins[:9], out.shards, out.hashes, out.dlen, out.bad, out.src_status, out.status, c.stride,
                      dst_sums=out.sums, n_src=c.n_src, n_dst=c.n_dst, crc_kind=rins[9], crcs=d_crcs)

        with torch.cuda.stream(s):
            rcall()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            rcall()
        for _ in range(2):
            d_crcs.fill_(0x5A5A5A5A)
            g.replay()
            torch.cuda.synchronize()
            assert [int(x) for x in d_crcs.cpu().numpy().view(np.uint32)] == [want_crc(2, c.Q[0]), want_crc(1, c.Q[1])]
        del g


def test_host_fault_contract(torch):
    """an injected CUDA failure in a HOST seal or reseal with checksums: nothing writes the caller's checksums after
    the error returns, and the next call is exact"""
    code = Code(("rs", 4, 2))
    rng = np.random.default_rng(0xC65)
    lens = np.array([9000, 1, 30000, 4096], dtype=np.uint32)
    plains = [rng.integers(0, 256, int(x), dtype=np.uint8) for x in lens]
    rows = plain_rows(plains, 30000 + 16 - 30000 % 16)
    keys = rng.integers(0, 256, (4, 32), dtype=np.uint8)
    nonces = rng.integers(0, 256, (4, 8), dtype=np.uint8)
    kinds = np.array([2, 1, 2, 1], dtype=np.uint8)
    want = [want_crc(int(kinds[i]), plains[i]) for i in range(4)]
    with code.ctx() as ec:
        stride = 8192
        for fail_at in range(1000):
            crcs = np.full(4, CRC_SENT, np.uint32)
            sh = np.zeros(4 * code.tot * stride, np.uint8)
            hs = np.zeros(4 * 32, np.uint8)
            ec.debug_fail_after(fail_at)
            try:
                ec.seal(rows.reshape(-1), rows.shape[1], lens, keys, nonces, sh, stride, hs, crc_kind=kinds, crcs=crcs)
            except G.EcError as e:
                err = e.code
            else:
                err = None
            finally:
                ec.debug_fail_after(-1)
            if err is None:
                assert [int(x) for x in crcs] == want
                break
            assert err in (G.E_CUDA, G.E_NOMEM), (fail_at, err)
            crcs[...] = 0xEEEEEEEE
            torch.cuda.synchronize()
            assert (crcs == 0xEEEEEEEE).all(), ("a copy wrote the checksums after the error return", fail_at)
        else:
            pytest.fail("the call still failed after 1000 injected faults")
        assert fail_at > 0
