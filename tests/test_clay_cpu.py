"""Clay(k, m) without a GPU: the numpy model (tests/clay_oracle.py) against the frozen KATs, the MDS property and the
repair property by rank, the model's decode of every pattern of up to 4 losses of Clay(10,4), the library's host read
rule (gf256.h, compiled here with the host compiler) against the Python statement, and the argument checks of
garage_ec_create_clay."""
import ctypes as C
import hashlib
import itertools
import json
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import clay_oracle as CO  # noqa: E402
import oracle_lib as O  # noqa: E402

import garage_b200 as G  # noqa: E402
from garage_b200 import block_manager as BM  # noqa: E402

ROOT = os.path.dirname(HERE)
KAT = json.load(open(os.path.join(HERE, "golden", "clay_kat.json")))


@pytest.mark.parametrize("name", sorted(KAT["cases"]))
def test_frozen_kats(name):
    c = KAT["cases"][name]
    k, m, kind, L = c["k"], c["m"], c["kind"], c["shard_len"]
    P = CO.build(k, m, kind)
    assert [bytes(r).hex() for r in P] == c["base_rows_hex"]
    data = O.fill_random(k * L, KAT["seed"]).reshape(k, L)
    par = CO.encode(k, m, P, data)
    assert hashlib.sha256(par.tobytes()).hexdigest() == c["parity_sha256"]
    assert [bytes(r[:32]).hex() for r in par] == c["parity_head_hex"]


def test_geometry():
    assert CO.params(10, 4) == (4, 4, 16, 2, 256)
    assert CO.params(6, 3) == (3, 3, 9, 0, 27)
    assert CO.params(10, 3) == (3, 5, 15, 2, 243)
    assert CO.shard_len(1 << 20, 10, 4) == 106496 and CO.shard_len(1 << 20, 6, 3) == 174960
    for k, m in [(14, 4), (16, 4), (10, 1), (10, 5), (1, 2)]:
        with pytest.raises(ValueError):
            CO.params(k, m)


@pytest.mark.parametrize("k,m", [(4, 2), (3, 2), (5, 3), (6, 3)])
def test_mds_and_repair_by_rank(k, m):
    P = CO.build(k, m)
    assert CO.mds_every_k_subset(k, m, P)
    for f in range(k + m):
        assert CO.repair_by_rank(k, m, P, f), f


def test_model_decodes_every_pattern_of_clay_10_4():
    k, m = 10, 4
    tot = k + m
    alpha = CO.params(k, m)[4]
    L = 16 * alpha
    P = CO.build(k, m)
    data = O.fill_random(k * L, 0xC1A9).reshape(k, L)
    full = np.concatenate([data, CO.encode(k, m, P, data)])
    n = 0
    for e in range(1, m + 1):
        for er in itertools.combinations(range(tot), e):
            pr = [0 if i in er else 1 for i in range(tot)]
            b = full.copy()
            b[list(er)] = 0xA5
            assert np.array_equal(CO.decode(k, m, P, b, pr), full), er
            n += 1
    assert n == 1470
    for f in range(tot):
        assert np.array_equal(CO.repair_from_shards(k, m, P, full, f), full[f]), f


_HARNESS = r"""
#include <cstdio>
#include "gf256.h"
using namespace garage_ec;
int main()
{
    int k, m;
    if (scanf("%d %d", &k, &m) != 2) return 1;
    unsigned long long pm, wm;
    while (scanf("%llx %llx", &pm, &wm) == 2) {
        uint64_t rd = 0;
        const bool ok = clay_read_set(k, m, pm, wm, &rd);
        printf("%d %llx\n", ok ? 1 : 0, (unsigned long long)rd);
    }
    return 0;
}
"""


def _rule(k, m, present, want):
    """the read rule of DESIGN.md section 2.4: (ok, shards read)"""
    tot = k + m
    absent = [i for i in range(tot) if not present[i]]
    wanted = [i for i in absent if want[i]]
    if tot - len(absent) < k:
        return False, []
    if not wanted:
        return True, []
    if len(absent) == 1:
        return True, [i for i in range(tot) if present[i]]
    return True, [i for i in range(tot) if present[i]][:k]


@pytest.mark.parametrize("k,m", [(4, 2), (10, 4)])
def test_host_read_rule(tmp_path, k, m):
    src, exe = tmp_path / "h.cpp", tmp_path / "h"
    src.write_text(_HARNESS)
    subprocess.run(["g++", "-O2", "-std=c++17", "-I", os.path.join(ROOT, "garage_b200", "csrc"), "-o", str(exe),
                    str(src)], check=True)
    tot = k + m
    cases = []
    for e in range(m + 2):
        for er in itertools.combinations(range(tot), e):
            pm = sum(1 << i for i in range(tot) if i not in er)
            cases.append((pm, (1 << tot) - 1))
            cases += [(pm, 1 << o) for o in er]
    inp = "%d %d\n" % (k, m) + "".join("%x %x\n" % c for c in cases)
    out = subprocess.run([str(exe)], input=inp, capture_output=True, text=True, check=True).stdout.split("\n")
    for (pm, wm), line in zip(cases, out):
        ok, rd = _rule(k, m, [(pm >> i) & 1 for i in range(tot)], [(wm >> i) & 1 for i in range(tot)])
        got_ok, got = line.split()
        assert bool(int(got_ok)) == ok, (pm, wm)
        if ok:
            assert int(got, 16) == sum(1 << i for i in rd), (pm, wm)


@pytest.mark.parametrize("k,m,kind", [(14, 4, 0), (16, 4, 0), (10, 1, 0), (10, 5, 0), (1, 2, 0), (0, 2, 0),
                                      (10, 4, 2), (10, 4, -1)])
def test_create_rejects_bad_codes_before_cuda(k, m, kind):
    L = G.load_library()
    h = C.c_void_p(1)
    assert L.garage_ec_create_clay(C.byref(h), 0, k, m, kind) == G.E_INVALID
    assert not h.value


def test_wire_round_trip():
    """"clay": 1 rides in the wire message only for Clay shards; RS messages keep their bytes"""
    h, s = bytes(range(32)), bytes(range(32, 64))
    rs = BM.wire_encode(h, 0, 10, 4, 3, 1 << 20, 104858, 1, s)
    clay = BM.wire_encode(h, 0, 10, 4, 3, 1 << 20, 106496, 1, s, clay=1)
    assert b"clay" in clay and b"clay" not in rs and len(clay) == len(rs) + 6
    d = BM.wire_decode(clay)
    assert d["clay"] == 1 and d["shard_len"] == 106496 and "pb" not in d
    assert "clay" not in BM.wire_decode(rs)
    assert BM.wire_encode(h, 0, 10, 4, 3, 1 << 20, 106496, 1, s, clay=1, pb=1) == b""  # not both
    assert BM.wire_encode(h, 0, 10, 5, 3, 1 << 20, 106496, 1, s, clay=1) == b""  # m > 4
