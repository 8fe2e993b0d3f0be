"""PB(k, m) without a GPU: the numpy model against the frozen KATs (tests/golden/pb_kat.json) and the C oracle, the
MDS property, the rule-1 read costs, the library's half-row read plan (gf256.h, compiled here with the host compiler)
against the Python statement of rules 1 and 2, the argument checks, the per-half adler8 check, the optional "pb" wire field and the block manager's PB config
checks."""
import ctypes as C
import itertools
import json
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import oracle_lib as O  # noqa: E402
import pb_oracle as PB  # noqa: E402

import garage_b200 as G  # noqa: E402

ROOT = os.path.dirname(HERE)
KAT = json.load(open(os.path.join(HERE, "golden", "pb_kat.json")))


@pytest.mark.parametrize("name", sorted(KAT["cases"]))
def test_frozen_kats(name):
    c = KAT["cases"][name]
    k, m, kind, L = c["k"], c["m"], c["kind"], KAT["shard_len"]
    P = PB.build(k, m, kind)
    assert [bytes(r).hex() for r in P] == c["matrix_hex"]
    assert PB.groups(k, m) == c["groups"]
    data = O.fill_random(k * L, KAT["seed"]).reshape(k, L)
    assert [bytes(r).hex() for r in PB.encode(P, data)] == c["kat_parity_hex"]


@pytest.mark.parametrize("k,m,kind", [(4, 2, 0), (6, 3, 1), (10, 4, 0), (10, 4, 1), (16, 4, 0)])
def test_halves_are_rs_plus_piggyback_by_the_c_oracle(k, m, kind):
    """second arm: a-halves are the C oracle's RS(k, m) parity of the a-halves; b-halves are its parity of the
    b-halves, XOR the plain XOR of each group's a-halves for parities 1..m-1"""
    L, h = 256, 128
    P = O.build_matrix(k, m, kind)
    assert np.array_equal(P, PB.build(k, m, kind))
    data = O.fill_random(k * L, 0x9B0 + k).reshape(k, L)
    par = PB.encode(P, data)
    a = np.ascontiguousarray(data[:, :h])
    b = np.ascontiguousarray(data[:, h:])
    ra = O.encode(k, m, P, a.reshape(-1), h, 1).reshape(m, h)
    rb = O.encode(k, m, P, b.reshape(-1), h, 1).reshape(m, h)
    assert np.array_equal(par[:, :h], ra)
    for i in range(m):
        pig = np.bitwise_xor.reduce(a[PB.groups(k, m)[i - 1]], axis=0) if i else 0
        assert np.array_equal(par[i, h:], rb[i] ^ pig)


def test_group_split():
    assert PB.groups(10, 4) == [[0, 1, 2, 3], [4, 5, 6], [7, 8, 9]]
    assert PB.groups(6, 3) == [[0, 1, 2], [3, 4, 5]]
    assert PB.groups(5, 2) == [[0, 1, 2, 3, 4]]
    assert PB.groups(2, 4) == [[0], [1], []]


@pytest.mark.parametrize("k,m", [(6, 3), (10, 4)])
def test_mds_every_pattern_up_to_m(k, m):
    tot = k + m
    P = PB.build(k, m)
    for e in range(m + 1):
        for er in itertools.combinations(range(tot), e):
            pr = [0 if i in er else 1 for i in range(tot)]
            assert PB.recoverable(k, m, P, pr), er
    pr = [0] * (m + 1) + [1] * (k - 1)
    assert not PB.recoverable(k, m, P, pr)
    assert not any(PB.recoverable(k, m, P, [0 if i in er else 1 for i in range(tot)])
                   for er in itertools.combinations(range(tot), m + 1))


def test_model_decode_from_planned_halves_only():
    k, m, L = 10, 4, 64
    tot = k + m
    P = PB.build(k, m, 1)
    rng = np.random.default_rng(5)
    data = rng.integers(0, 256, (k, L), dtype=np.uint8)
    full = np.concatenate([data, PB.encode(P, data)])
    for _ in range(120):
        lost = rng.choice(tot, int(rng.integers(1, m + 1)), replace=False)
        present = np.ones(tot, dtype=np.uint8)
        present[lost] = 0
        want = None
        if rng.random() < 0.5:
            want = np.zeros(tot, dtype=np.uint8)
            want[lost[0]] = 1
        ok, surv = PB.read_plan(k, m, P, present, want)
        assert ok
        sh = np.full_like(full, 0xA5)
        for q in surv:  # only the planned halves hold data
            sh[q >> 1, (q & 1) * 32:(q & 1) * 32 + 32] = full[q >> 1, (q & 1) * 32:(q & 1) * 32 + 32]
        assert PB.decode(k, m, P, sh, present, want)
        for o in range(tot):
            if not present[o] and (want is None or want[o]):
                assert np.array_equal(sh[o], full[o]), o


@pytest.mark.parametrize("k,m,halves,ratio", [(10, 4, {0: 14, 4: 13, 9: 13}, None), (6, 3, {0: 9, 5: 9}, 0.75),
                                              (12, 4, {j: 16 for j in range(12)}, 0.67), (5, 2, {0: 10}, 1.0)])
def test_rule1_read_counts(k, m, halves, ratio):
    P = PB.build(k, m)
    L = PB.shard_len(1 << 20, k)
    for j, n in halves.items():
        pr = [1] * (k + m)
        pr[j] = 0
        ok, surv = PB.read_plan(k, m, P, pr)
        assert ok and len(surv) == n, (j, surv)
        if ratio is not None:
            assert round(n / (2 * k), 2) == ratio
    if (k, m) == (10, 4):
        assert L == 104960 and 14 * L // 2 == 734720 and 13 * L // 2 == 682240
    if (k, m) == (6, 3):
        assert L == 174848 and 9 * L // 2 == 786816
    pr = [1] * (k + m)
    pr[k + 1] = 0  # a parity shard: rule 2, both halves of the first k shards
    assert PB.read_plan(k, m, P, pr)[1] == list(range(2 * k))


_HARNESS = r"""
#include <cstdio>
#include "gf256.h"
using namespace garage_ec;
int main()
{
    int k, m, kind;
    if (scanf("%d %d %d", &k, &m, &kind) != 3) return 2;
    uint8_t P[GARAGE_EC_MAX_M_HOST * GARAGE_EC_MAX_K_HOST];
    if (!h_build_matrix(k, m, kind, P)) return 3;
    unsigned long long pm, wm;
    while (scanf("%llx %llx", &pm, &wm) == 2) {
        uint64_t hv = 0;
        const bool ok = h_read_plan(PlanCode{k, m, 0, true, P}, pm, wm, &hv);
        printf("%d %llx\n", ok ? 1 : 0, (unsigned long long)hv);
    }
    return 0;
}
"""


@pytest.fixture(scope="module")
def read_plan_harness(tmp_path_factory):
    d = tmp_path_factory.mktemp("read_plan")
    src, exe = d / "h.cpp", d / "h"
    src.write_text(_HARNESS)
    subprocess.run(["g++", "-O2", "-std=c++17", "-I", os.path.join(ROOT, "garage_b200", "csrc"), "-o", str(exe),
                    str(src)], check=True)
    return str(exe)


@pytest.mark.parametrize("k,m,kind", [(6, 3, 0), (10, 4, 1)])
def test_host_read_plan_matches_rules(read_plan_harness, k, m, kind):
    """the half-row plan the library uses (h_read_plan: garage_ec_read_plan, the HOST upload paths) against the
    Python rules for every pattern with up to 4 absent shards, want = every absent shard and each absent shard
    alone"""
    tot = k + m
    P = PB.build(k, m, kind)
    cases = []
    for e in range(5):
        for er in itertools.combinations(range(tot), e):
            pm = sum(1 << i for i in range(tot) if i not in er)
            cases.append((pm, (1 << tot) - 1))
            cases += [(pm, 1 << o) for o in er]
    inp = "%d %d %d\n" % (k, m, kind) + "".join("%x %x\n" % c for c in cases)
    out = subprocess.run([read_plan_harness], input=inp, capture_output=True, text=True, check=True).stdout.split("\n")
    for (pm, wm), line in zip(cases, out):
        present = [(pm >> i) & 1 for i in range(tot)]
        want = [(wm >> i) & 1 for i in range(tot)]
        ok, surv = PB.read_plan(k, m, P, present, want)
        got_ok, got = line.split()
        assert bool(int(got_ok)) == ok, (pm, wm)
        if ok:
            assert int(got, 16) == sum(1 << q for q in surv), (pm, wm, got, surv)


def test_create_piggyback_rejects_bad_codes_before_touching_cuda():
    L = G.load_library()
    h = C.c_void_p()
    for k, m, kind in [(0, 2, 0), (17, 4, 0), (10, 1, 0), (10, 5, 0), (10, 4, 2), (10, 4, -1), (-3, 3, 0)]:
        assert L.garage_ec_create_piggyback(C.byref(h), 0, k, m, kind) == G.E_INVALID, (k, m, kind)
        assert not h.value
    assert L.garage_ec_piggyback_info(None, None, None) == G.E_INVALID
    assert L.garage_ec_code_shard_len(None, 100, None) == G.E_INVALID
    assert L.garage_ec_read_plan(None, None, None, None) == G.E_INVALID


def _adler8(data, L):
    seg = -(-(-(-L // 8)) // 16) * 16
    tags = [zlib.adler32(bytes(data[s * seg:min(L, (s + 1) * seg)])) if s * seg < L else 1 for s in range(8)]
    return np.array(tags, dtype="<u4").view(np.uint8).tobytes()


@pytest.mark.parametrize("L", [128, 1024, 104960, 174848])
def test_half_tag_check_agrees_with_zlib(L):
    data = np.random.default_rng(L).integers(0, 256, L, dtype=np.uint8)
    tag = _adler8(data, L)
    assert tag == G.shard_sum_host(G.SUM_ADLER8, data)
    h = L // 2
    for which in (0, 1):
        half = data[which * h:(which + 1) * h].copy()
        assert G.check_shard_half_host(G.SUM_ADLER8, half, L, which, tag) == 0
        half[h // 3] ^= 1
        assert G.check_shard_half_host(G.SUM_ADLER8, half, L, which, tag) == 1
        assert G.check_shard_half_host(G.SUM_ADLER8, data[(1 - which) * h:(2 - which) * h], L, which, tag) == 1
    assert G.check_shard_half_host(G.SUM_BLAKE2, data[:h], L, 0, tag) == G.E_INVALID
    assert G.check_shard_half_host(G.SUM_ADLER8, data[:h], L + 32, 0, tag) == G.E_INVALID
    assert G.check_shard_half_host(G.SUM_ADLER8, data[:h], L, 2, tag) == G.E_INVALID


def test_wire_carries_pb_only_for_pb():
    from garage_b200 import block_manager as BM

    H, S = bytes(range(32)), bytes(range(32, 64))
    rs = BM.wire_encode(H, 0, 10, 4, 3, 1000, 100, 1, S)
    assert rs == BM.wire_encode(H, 0, 10, 4, 3, 1000, 100, 1, S, pb=0)  # RS bytes unchanged
    assert rs[8] == 0x89 and b"\xa2pb" not in rs and "pb" not in BM.wire_decode(rs)
    pb = BM.wire_encode(H, 0, 10, 4, 3, 1000, 104960, 1, S, pb=1)
    rs2 = BM.wire_encode(H, 0, 10, 4, 3, 1000, 104960, 1, S)
    assert pb[8] == 0x8A and pb[:8] == rs2[:8] and pb[9:-4] == rs2[9:] and pb.endswith(b"\xa2pb\x01")
    d = BM.wire_decode(pb)
    assert d["pb"] == 1 and d["k"] == 10 and d["m"] == 4 and d["shard_len"] == 104960 and "l" not in d
    assert BM.wire_encode(H, 0, 10, 4, 3, 1000, 100, 1, S, l=2, pb=1) == b""  # not both
    assert BM.wire_encode(H, 0, 10, 5, 3, 1000, 100, 1, S, pb=1) == b""  # m > 4
    assert BM.wire_encode(H, 0, 17, 4, 3, 1000, 100, 1, S, pb=1) == b""  # k > 16
    assert BM.wire_decode(pb[:-1] + b"\x02") is None  # "pb" is 1 or absent


def test_block_manager_rejects_bad_piggyback_configs():
    from garage_b200 import block_manager as BM

    with pytest.raises(BM.BlockManagerError):
        BM.BlockManager(k=10, m=4, piggyback=True, local_groups=2)
    with pytest.raises(BM.BlockManagerError):
        BM.BlockManager(k=10, m=4, piggyback=True, shard_sum_kind=BM.SUM_BLAKE2)
