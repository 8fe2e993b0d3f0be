"""Copies with re-encryption on the GPU (DESIGN.md 2.8, 4.11): garage_ec_reseal and garage_ec_reseal_stripes.

Expected values never come from the library: sources and destinations are sealed by the scalar C oracle
(tests/sse_c_oracle.py), Q_d is cut from the plaintexts in numpy, parity comes from the C oracle (RS) and the numpy
models (LRC, PB, Clay) through test_sse_c_geometry_gpu's Code, and content hashes and shard tags from hashlib.

Every SSE-C code; the ragged source lengths of test_sse_c_gpu plus one source of 258 chunks; piece lists with whole
blocks, source and destination offsets at every residue mod 16, pieces across source chunk boundaries and destination
chunk seams, 230 pieces of 1..17 bytes, a source named twice and destination chunks past 255; plaintext sources;
erasures (every pattern for RS(4,2) and RS(6,3)); failures that stay with the destinations that name the failing
source; round trips through garage_ec_open; batches that outrun the chunk kernel's warps; DEVICE == HOST == gather
form; CUDA graph capture; and the HOST ownership contract under injected faults."""
import itertools
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import garage_b200 as G  # noqa: E402
import sse_c_oracle as SO  # noqa: E402
from test_sse_c_geometry_gpu import Code, blake2, expected_shards, expected_tags, patterns, same  # noqa: E402

pytestmark = pytest.mark.gpu

CODES = {"rs10_4": ("rs", 10, 4), "rs6_3": ("rs", 6, 3), "rs4_2": ("rs", 4, 2), "lrc10_2_2": ("lrc", 10, 2, 2),
         "pb10_4": ("pb", 10, 4), "clay10_4": ("clay", 10, 4)}
MiB = 1 << 20
# the ragged lengths of test_sse_c_gpu, with 2 in place of 0: every source must be named by a piece in HOST mode,
# and no piece can name an empty block
LENS = [2, 1, 15, 16, 17, 4095, 4096, 4097, 8191, 8192, 8193, 12289, 3 * 4096 - 1, 40000, 100001]
BIG = MiB + 4097        # chunks 256 and 257
POISON, GONE = 0xA5, 0x5C
CHUNK_WARPS_PER_SM = 4 * 8


def piece_lists(lens):
    """destination piece lists over sources of plaintext lengths `lens` (LENS, then BIG)"""
    dests = [[(i, 0, n)] for i, n in enumerate(lens)]  # a 1:1 rotation
    for r in range(16):  # the second piece starts at destination residue r' and source residue r
        dests.append([(13, 0, 16 + (5 * r + 3) % 16), (14, 2 * 4096 + 17 * r, 7000 + r)])
    for o in (4095, 4096, 4097):  # across source chunk boundaries
        dests.append([(11, o, 4096), (11, o - 1, 3)])
    dests.append([(14, 5, 4090), (13, 100, 12), (14, 50000, 4100), (12, 0, 12287)])  # across destination seams
    dests.append([(5 + i % 10, (37 * i) % 4000, 1 + i % 17) for i in range(230)])     # tiny pieces
    dests.append([(14, 0, 50000), (14, 10, 60000)])                                    # one source twice
    dests.append([(15, 1000, lens[15] - 1000), (14, 0, 100001)])                       # chunks past 255
    return dests


def r128(x):
    return max(1, -(-x // 128)) * 128


class Case:
    """sources sealed under their keys (or plaintext), piece lists, and the oracle's destinations"""

    def __init__(self, code, seed, keyed=True, lens=LENS + [BIG], dests=None, stride=None):
        rng = np.random.default_rng(seed)
        self.code, self.keyed = code, keyed
        self.plains = [rng.integers(0, 256, n, dtype=np.uint8) for n in lens]
        ns = self.n_src = len(lens)
        self.src_keys = rng.integers(0, 256, (ns, 32), dtype=np.uint8)
        src_nonces = rng.integers(0, 256, (ns, 8), dtype=np.uint8)
        self.B = [np.frombuffer(SO.seal(self.src_keys[i].tobytes(), src_nonces[i].tobytes(), p.tobytes()),
                                dtype=np.uint8) if keyed else p for i, p in enumerate(self.plains)]
        self.dests = piece_lists(lens) if dests is None else dests
        nd = self.n_dst = len(self.dests)
        self.pieces = np.array([p for d in self.dests for p in d], dtype=np.uint32).reshape(-1, 3)
        self.piece_start = np.cumsum([0] + [len(d) for d in self.dests]).astype(np.uint32)
        self.Q = [np.concatenate([self.plains[s][o:o + n] for s, o, n in d]) for d in self.dests]
        self.dst_keys = rng.integers(0, 256, (nd, 32), dtype=np.uint8)
        self.dst_nonces = rng.integers(0, 256, (nd, 8), dtype=np.uint8)
        self.Bd = [np.frombuffer(SO.seal(self.dst_keys[d].tobytes(), self.dst_nonces[d].tobytes(), q.tobytes()),
                                 dtype=np.uint8) for d, q in enumerate(self.Q)]
        self.stride = stride or r128(max(code.shard_len(b.size) for b in self.B + self.Bd))
        self.src_shards, _ = expected_shards(code, self.B, self.stride)
        self.want, self.Ls = expected_shards(code, self.Bd, self.stride)
        self.tags = expected_tags(self.want, self.Ls, G.SUM_BLAKE2)
        self.src_len = np.array([b.size for b in self.B], dtype=np.uint32)
        self.src_hashes = np.stack([np.frombuffer(blake2(b), dtype=np.uint8) for b in self.B])
        self.dst_hashes = np.stack([np.frombuffer(blake2(b), dtype=np.uint8) for b in self.Bd])
        self.dst_len = np.array([b.size for b in self.Bd], dtype=np.uint32)

    def names(self, d):
        return {s for s, _, _ in self.dests[d]}


def dev(torch, a):
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.int32) if a.dtype == np.uint32 else a).cuda()


class Out:
    """one call's outputs (numpy, or device tensors with .host() to read them)"""

    def __init__(self, torch, c, device):
        nd, ns, tot = c.n_dst, c.n_src, c.code.tot
        mk = (lambda shape, v, dt: torch.full(shape, v, dtype=dt, device="cuda")) if device else \
            (lambda shape, v, dt: np.full(shape, v, dtype={torch.uint8: np.uint8, torch.int32: np.int32}[dt]))
        self.device = device
        self.shards = mk((nd * tot * c.stride,), POISON, torch.uint8)
        self.hashes = mk((nd * 32,), 0, torch.uint8)
        self.sums = mk((nd * tot * 32,), 0, torch.uint8)
        self.dlen = mk((nd,), 0x5A5A5A5A, torch.int32)
        self.bad = mk((ns,), 7, torch.uint8)
        self.src_status = mk((ns,), 99, torch.int32)
        self.status = mk((nd,), 99, torch.int32)

    def host(self):
        f = (lambda x: x.cpu().numpy()) if self.device else (lambda x: x)
        return {k: f(getattr(self, k)) for k in ("shards", "hashes", "sums", "dlen", "bad", "src_status", "status")}


def run(torch, ec, c, src_shards, present, form="device", src_hashes=None, src_keys="same", out=None):
    """one reseal of case c; form: device / host / stripes.  Returns the outputs as numpy arrays and the call's code"""
    device = form == "device"
    out = out or Out(torch, c, device)
    hashes = c.src_hashes if src_hashes is None else src_hashes
    keys = (c.src_keys if c.keyed else None) if isinstance(src_keys, str) else src_keys
    conv = (lambda a: None if a is None else dev(torch, a)) if device else (lambda a: a)
    args = [conv(present), conv(c.src_len), conv(hashes), conv(keys), conv(c.pieces), conv(c.piece_start),
            conv(c.dst_keys), conv(c.dst_nonces), out.shards, out.hashes, out.dlen, out.bad, out.src_status,
            out.status, c.stride]
    if form == "stripes":
        rc = ec.reseal_stripes([src_shards[i].reshape(-1) for i in range(c.n_src)], *args, dst_sums=out.sums)
    else:
        rc = ec.reseal(conv(src_shards.reshape(-1)) if device else src_shards.reshape(-1), *args, dst_sums=out.sums,
                       n_src=c.n_src, n_dst=c.n_dst)
    if device:
        torch.cuda.synchronize()
    return out.host(), rc


def check_exact(c, got, what, failed=()):
    """every destination not in `failed` is exact; the failed ones left their shards and lengths alone"""
    tot, sh = c.code.tot, got["shards"].reshape(c.n_dst, c.code.tot, c.stride)
    for d in range(c.n_dst):
        if d in failed:
            assert (sh[d] == POISON).all(), (what, "shards of failed destination", d)
            assert got["dlen"][d] == 0x5A5A5A5A, (what, d)
            continue
        assert got["status"][d] == 0, (what, d, got["status"][d])
        same(sh[d], c.want[d], "%s: destination %d shards" % (what, d))
        assert got["dlen"][d] == c.dst_len[d], (what, d)
        same(got["hashes"].reshape(-1, 32)[d], c.dst_hashes[d], "%s: destination %d hash" % (what, d))
        same(got["sums"].reshape(-1, tot, 32)[d], c.tags[d], "%s: destination %d tags" % (what, d))


@pytest.fixture(scope="module")
def torch():
    import torch as t

    assert t.cuda.is_available()
    return t


def present_all(c):
    return np.ones((c.n_src, c.code.tot), dtype=np.uint8)


@pytest.mark.parametrize("name", list(CODES))
def test_reseal_matches_oracle_device_host_graph_and_round_trip(torch, name):
    code = Code(CODES[name])
    c = Case(code, 11 + len(name))
    with code.ctx() as ec:
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        cmax = -(-code.k * c.stride // 4096)
        assert c.n_dst * cmax > CHUNK_WARPS_PER_SM * sms  # the (destination, chunk) items outrun the grid
        assert max(-(-q.size // 4096) for q in c.Q) > 256
        pr = present_all(c)
        got, rc = run(torch, ec, c, c.src_shards, pr, "device")
        check_exact(c, got, "device")
        assert (got["src_status"] == 0).all() and (got["bad"] == 0).all()
        for form in ("host", "stripes"):
            got_h, rc = run(torch, ec, c, c.src_shards.copy(), pr, form)
            assert rc == 0
            check_exact(c, got_h, form)
            for k in got:
                assert np.array_equal(got[k], got_h[k]), (form, k)

        # CUDA graph capture and replay into fresh poisoned outputs
        out = Out(torch, c, True)
        d_src, d_pr = dev(torch, c.src_shards.reshape(-1)), dev(torch, pr)
        ins = [dev(torch, a) for a in (c.src_len, c.src_hashes, c.src_keys, c.pieces, c.piece_start, c.dst_keys,
                                       c.dst_nonces)]
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            ec.reseal(d_src, d_pr, *ins, out.shards, out.hashes, out.dlen, out.bad, out.src_status, out.status,
                      c.stride, dst_sums=out.sums, n_src=c.n_src, n_dst=c.n_dst)
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            ec.reseal(d_src, d_pr, *ins, out.shards, out.hashes, out.dlen, out.bad, out.src_status, out.status,
                      c.stride, dst_sums=out.sums, n_src=c.n_src, n_dst=c.n_dst)
        for _ in range(2):
            out.shards.fill_(POISON)
            out.hashes.zero_()
            out.sums.zero_()
            out.dlen.fill_(0x5A5A5A5A)
            g.replay()
            torch.cuda.synchronize()
            check_exact(c, out.host(), "graph replay")
        del g

        # round trip: the destinations open under their new keys to Q_d and fail under a source's key
        n, tot = c.n_dst, code.tot
        d_sh = dev(torch, got["shards"])
        pres = torch.ones(n * tot, dtype=torch.uint8, device="cuda")
        pitch = (max(q.size for q in c.Q) + 15) // 16 * 16
        for keys, ok in ((c.dst_keys, True), (np.roll(c.dst_keys, 1, axis=0), False)):
            plain = torch.zeros(n * pitch, dtype=torch.uint8, device="cuda")
            plen = torch.zeros(n, dtype=torch.int32, device="cuda")
            bad = torch.zeros(n, dtype=torch.uint8, device="cuda")
            st = torch.zeros(n, dtype=torch.int32, device="cuda")
            ec.open(d_sh, pres, dev(torch, c.dst_len), dev(torch, c.dst_hashes), dev(torch, keys), plain, pitch, plen,
                    bad, st, c.stride, n=n)
            torch.cuda.synchronize()
            st, pl = st.cpu().numpy(), plain.cpu().numpy().reshape(n, pitch)
            assert (bad.cpu().numpy() == 0).all()
            if ok:
                assert (st == 0).all(), st
                for d in range(n):
                    assert np.array_equal(pl[d, :c.Q[d].size], c.Q[d]), d
            else:
                assert (st == G.E_AUTH).all(), st


def erasure_patterns(code, ec, name):
    if name in ("rs4_2", "rs6_3"):  # every pattern of at most m losses
        return [np.array([0 if i in lost else 1 for i in range(code.tot)], dtype=np.uint8)
                for r in range(code.m + 1) for lost in itertools.combinations(range(code.tot), r)]
    return patterns(code, ec, 5)


@pytest.mark.parametrize("name", list(CODES))
def test_reseal_rebuilds_absent_source_shards(torch, name):
    """every source loses the same shards (DEVICE: overwritten with their rebuilt bytes) and every destination is
    still exact: its content hash and the tags of all k+m shards (and, for the first patterns, every byte)"""
    code = Code(CODES[name])
    c = Case(code, 23 + len(name))
    with code.ctx() as ec:
        rng = np.random.default_rng(3)
        pats = erasure_patterns(code, ec, name)
        if name in ("rs4_2", "rs6_3"):
            assert len(pats) == sum(len(list(itertools.combinations(range(code.tot), r))) for r in range(code.m + 1))
        for t, p in enumerate(pats):
            pr = np.tile(p, (c.n_src, 1))
            src = c.src_shards.copy()
            src[:, p == 0] = GONE
            # a second, random pattern on the big source, so that two patterns meet in one batch
            q = p if t % 2 else np.array(pats[int(rng.integers(len(pats)))])
            pr[-1] = q
            src[-1] = c.src_shards[-1]
            src[-1, q == 0] = GONE
            got, rc = run(torch, ec, c, src, pr, "device")
            assert (got["status"] == 0).all() and (got["src_status"] == 0).all() and (got["bad"] == 0).all(), t
            same(got["hashes"].reshape(-1, 32), c.dst_hashes, "pattern %d hashes" % t)
            same(got["sums"].reshape(-1, code.tot, 32), c.tags, "pattern %d tags" % t)
            if t < 3:
                check_exact(c, got, "pattern %d" % t)
        got, rc = run(torch, ec, c, src, pr, "host")  # HOST uploads only the read set and rebuilds the rest
        assert rc == 0
        check_exact(c, got, "host, last pattern")


@pytest.mark.parametrize("name", ["rs10_4", "lrc10_2_2", "pb10_4", "clay10_4"])
def test_reseal_plaintext_sources_into_sse_c(torch, name):
    code = Code(CODES[name])
    c = Case(code, 41, keyed=False)
    with code.ctx() as ec:
        pr = present_all(c)
        pr[3, 0] = 0  # one source rebuilds its first data shard
        src = c.src_shards.copy()
        src[3, 0] = GONE
        got, _ = run(torch, ec, c, src, pr, "device")
        check_exact(c, got, "device")
        got_h, rc = run(torch, ec, c, src, pr, "host")
        assert rc == 0
        check_exact(c, got_h, "host")


@pytest.mark.parametrize("name", ["rs10_4", "rs4_2", "lrc10_2_2", "pb10_4", "clay10_4"])
def test_reseal_failures_stay_with_the_destinations_that_name_them(torch, name):
    """a wrong source key, a tampered chunk (the block still hashes to its recorded address), a stale but
    self-consistent data shard (the block no longer hashes to its address) and more than m absent shards: only the
    destinations that name the source fail, with the specified status, and their shards stay poisoned"""
    code = Code(CODES[name])
    c = Case(code, 51)
    WRONG_KEY, TAMPERED, STALE, LOST = 13, 11, 8, 10
    with code.ctx() as ec:
        src, pr = c.src_shards.copy(), present_all(c)
        keys = c.src_keys.copy()
        keys[WRONG_KEY, 0] ^= 1
        hashes = c.src_hashes.copy()
        L = code.shard_len(c.B[TAMPERED].size)
        B = c.B[TAMPERED].copy()
        B[L + 3] ^= 0x10  # ciphertext of chunk 0 or 1, in data shard 1
        src[TAMPERED, 1, 3] ^= 0x10
        hashes[TAMPERED] = np.frombuffer(blake2(B), dtype=np.uint8)
        src[STALE, 0, 40] ^= 1
        pr[LOST, :code.m + 1] = 0
        src[LOST, :code.m + 1] = GONE
        want_dst = []
        for d in range(c.n_dst):
            nm = c.names(d)
            want_dst.append(G.E_UNRECOVERABLE if nm & {STALE, LOST} else G.E_AUTH if nm & {WRONG_KEY, TAMPERED} else 0)
        failed = {d for d in range(c.n_dst) if want_dst[d]}
        assert failed and len(failed) < c.n_dst
        for form in ("device", "host", "stripes"):
            got, rc = run(torch, ec, c, src.copy(), pr, form, src_hashes=hashes, src_keys=keys)
            assert list(got["status"]) == want_dst, (form, list(got["status"]))
            check_exact(c, got, form, failed)
            assert got["src_status"][WRONG_KEY] == G.E_AUTH and got["bad"][WRONG_KEY] == 0
            assert got["src_status"][TAMPERED] == G.E_AUTH and got["bad"][TAMPERED] == 0
            assert got["bad"][STALE] == 1
            assert got["src_status"][LOST] == G.E_UNRECOVERABLE
            for i in set(range(c.n_src)) - {WRONG_KEY, TAMPERED, STALE, LOST}:
                assert got["src_status"][i] == 0 and got["bad"][i] == 0, (form, i)
            if form != "device":
                assert rc == G.E_UNRECOVERABLE


def test_reseal_invalid_pieces(torch):
    """DEVICE: a piece past its source's plaintext, an empty piece or a source index out of range fails only its
    destination with E_INVALID; HOST refuses the call before any GPU work"""
    code = Code(CODES["rs10_4"])
    lens = [5000, 9000, 100]
    dests = [[(0, 0, 5000)], [(1, 8000, 1001)], [(0, 0, 0)], [(3, 0, 1)], [(1, 0, 9000), (2, 0, 100)]]
    c = Case(code, 61, lens=lens, dests=[[(0, 0, 5000)], [(1, 0, 9000)], [(2, 0, 100)], [(0, 0, 1)],
                                         [(1, 0, 9000), (2, 0, 100)]])
    c.pieces = np.array([p for d in dests for p in d], dtype=np.uint32).reshape(-1, 3)
    with code.ctx() as ec:
        got, _ = run(torch, ec, c, c.src_shards, present_all(c), "device")
        assert list(got["status"]) == [0, G.E_INVALID, G.E_INVALID, G.E_INVALID, 0]
        same(got["shards"].reshape(c.n_dst, code.tot, c.stride)[0], c.want[0], "valid destination 0")
        same(got["shards"].reshape(c.n_dst, code.tot, c.stride)[4], c.want[4], "valid destination 4")
        for d in (1, 2, 3):
            assert (got["shards"].reshape(c.n_dst, code.tot, c.stride)[d] == POISON).all()
        with pytest.raises(G.EcError) as e:
            run(torch, ec, c, c.src_shards, present_all(c), "host")
        assert e.value.code == G.E_INVALID
        c.pieces[:] = np.array([p for d in c.dests for p in d], dtype=np.uint32).reshape(-1, 3)
        bad_start = c.piece_start.copy()
        c.piece_start[2] = c.piece_start[1]  # destination 1 without a piece
        with pytest.raises(G.EcError) as e:
            run(torch, ec, c, c.src_shards, present_all(c), "host")
        assert e.value.code == G.E_INVALID
        c.piece_start = bad_start
        got, rc = run(torch, ec, c, c.src_shards, present_all(c), "host")
        assert rc == 0
        check_exact(c, got, "host after refusals")


def test_reseal_geometry_refusals(torch):
    """DEVICE: an L' past the stride fails its destination with E_INVALID; a source whose L is past the stride gets
    src_status E_INVALID and fails the destinations that name it; a source no piece names is still proven.  HOST
    refuses each of the three before any GPU work.  Every other destination stays exact."""
    code = Code(CODES["rs10_4"])

    def case():
        return Case(code, 81, lens=[5000, 9000, 100], dests=[[(0, 0, 5000)], [(1, 0, 9000)], [(2, 0, 100)]],
                    stride=1024)

    def refused(c):
        with pytest.raises(G.EcError) as e:
            run(torch, ec, c, c.src_shards, present_all(c), "host")
        assert e.value.code == G.E_INVALID

    with code.ctx() as ec:
        c = case()
        assert code.shard_len(G.sealed_len(14000)) > c.stride
        c.pieces = np.vstack([c.pieces, np.array([[1, 0, 9000], [0, 0, 5000]], dtype=np.uint32)])
        c.piece_start = np.append(c.piece_start, np.uint32(len(c.pieces)))
        c.dst_keys, c.dst_nonces = np.vstack([c.dst_keys, c.dst_keys[:1]]), np.vstack([c.dst_nonces, c.dst_nonces[:1]])
        c.n_dst += 1
        got, _ = run(torch, ec, c, c.src_shards, present_all(c), "device")
        assert list(got["status"]) == [0, 0, 0, G.E_INVALID]
        check_exact(c, got, "L' past the stride", failed={3})
        refused(c)

        c = case()
        c.src_len = c.src_len.copy()
        c.src_len[2] = 20000  # a stored length whose L does not fit the stride
        got, _ = run(torch, ec, c, c.src_shards, present_all(c), "device")
        assert list(got["src_status"]) == [0, 0, G.E_INVALID]
        assert list(got["status"]) == [0, 0, G.E_INVALID]
        check_exact(c, got, "source L past the stride", failed={2})
        refused(c)

        c = case()
        c.src_shards = np.concatenate([c.src_shards, c.src_shards[:1]])
        c.src_len = np.append(c.src_len, c.src_len[0])
        c.src_hashes = np.vstack([c.src_hashes, c.src_hashes[:1]])
        c.src_keys = np.vstack([c.src_keys, c.src_keys[:1]])
        c.n_src += 1
        got, _ = run(torch, ec, c, c.src_shards, present_all(c), "device")
        assert list(got["src_status"]) == [0] * 4 and list(got["bad"]) == [0] * 4
        check_exact(c, got, "a source no piece names")
        refused(c)


@pytest.mark.parametrize("pinned", [False, True], ids=["pageable", "pinned"])
def test_reseal_host_fault_leaves_caller_buffers_alone(torch, pinned):
    """the HOST ownership contract over several pipeline chunks (a stride that fits one destination per chunk), with
    the fault injected at every checked runtime call in turn until the call completes: the call returns an error,
    nothing writes the caller's outputs after the return, a destination that names a tampered source is never
    written, and the next call is exact"""
    code = Code(CODES["rs4_2"])
    lens = [40000, 100001, 5000, 12289]
    dests = [[(0, 0, 40000)], [(1, 7, 90000), (0, 3, 17)], [(2, 0, 5000)], [(3, 100, 9000)], [(1, 0, 100001)]]
    c = Case(code, 71, lens=lens, dests=dests, stride=4 * MiB)
    with code.ctx() as ec:
        src, hashes = c.src_shards.copy(), c.src_hashes.copy()
        B = c.B[2].copy()
        B[code.shard_len(B.size) + 20] ^= 4
        src[2, 1, 20] ^= 4
        hashes[2] = np.frombuffer(blake2(B), dtype=np.uint8)
        failed = {2}
        held = []

        def buf(a):
            if not pinned:
                return a
            h, p = ec.host_alloc(a.nbytes)
            held.append(p)
            v = h.view(a.dtype).reshape(a.shape)
            v[...] = a
            return v

        pr = present_all(c)
        pr[:, 0] = 0  # the nonce prefix and chunk 0 come from parity (but the tampered block's own shard 0)
        pr[2, 0] = 1
        src[pr == 0] = GONE
        src = buf(src)
        try:
            out = Out(torch, c, False)
            for k in ("shards", "hashes", "sums", "dlen", "bad", "src_status", "status"):
                setattr(out, k, buf(getattr(out, k)))

            def reset():
                out.shards[...] = POISON
                out.dlen[...] = 0x5A5A5A5A

            def call():
                return run(torch, ec, c, src, pr, "host", src_hashes=hashes, out=out)

            reset()
            got, rc = call()
            assert rc == G.E_AUTH
            check_exact(c, got, "first call", failed)
            for fail_at in range(1000):
                reset()
                ec.debug_fail_after(fail_at)
                try:
                    got, rc = call()
                except G.EcError as e:
                    err = e.code
                else:
                    err = None
                finally:
                    ec.debug_fail_after(-1)
                if err is None:
                    check_exact(c, got, "after %d faults" % fail_at, failed)
                    break
                assert err in (G.E_CUDA, G.E_NOMEM), (fail_at, err)
                assert (out.shards.reshape(c.n_dst, code.tot, c.stride)[2] == POISON).all(), fail_at
                outs = out.host()
                for o in outs.values():
                    o.view(np.uint8)[...] = 0xEE
                torch.cuda.synchronize()
                assert all((o.view(np.uint8) == 0xEE).all() for o in outs.values()), (
                    "a copy or kernel wrote after the error return", fail_at)
                if fail_at % 3 == 2:
                    reset()
                    got, rc = call()
                    check_exact(c, got, "next call after fault %d" % fail_at, failed)
            else:
                pytest.fail("the call still failed after 1000 injected faults")
            assert fail_at >= c.n_dst * 3, fail_at
        finally:
            for p in held:
                ec.host_free(p)
