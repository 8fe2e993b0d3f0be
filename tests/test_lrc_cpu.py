"""LRC(k, l, r) without a GPU: the numpy model against the C oracle and plain XOR, the frozen KATs of
tests/golden/lrc_kat.json, the library's survivor selection (gf256.h, compiled here with the host compiler)
against the Python statement of rules 1 and 2, and garage_ec_create_lrc's argument checks."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import lrc_oracle as LO  # noqa: E402
import oracle_lib as O  # noqa: E402

import garage_b200 as G  # noqa: E402

ROOT = os.path.dirname(HERE)
KAT = json.load(open(os.path.join(HERE, "golden", "lrc_kat.json")))


@pytest.mark.parametrize("k,l,r", [(6, 2, 2), (10, 2, 2), (12, 2, 2), (12, 3, 2), (16, 4, 2), (20, 4, 4)])
def test_parity_numpy_model_equals_c_oracle_and_xor(k, l, r):
    m, n, stride = l + r, 3, 256
    P = LO.build_lrc(k, l, r)
    data = O.fill_random(n * k * stride, 0x7C0 + k)
    lens = np.array([stride, 77, 1], dtype=np.uint32)
    par = O.encode(k, m, P, data, stride, n, lens).reshape(n, m, stride)
    d3 = data.reshape(n, k, stride)
    gs = k // l
    for s in range(n):
        L = int(lens[s])
        assert np.array_equal(LO.encode(P, d3[s, :, :L]), par[s, :, :L])
        for g in range(l):  # local parity: plain XOR of the group, no GF arithmetic
            assert np.array_equal(par[s, g, :L], np.bitwise_xor.reduce(d3[s, g * gs:(g + 1) * gs, :L], axis=0))


def test_global_rows_are_the_cauchy_kats():
    P = LO.build_lrc(10, 2, 2)
    assert bytes(P[2]).hex(" ") == "dd 98 ad 9d 5d 96 3d aa 8e f4"
    assert bytes(P[3]).hex(" ") == "98 dd 9d ad 96 5d aa 3d f4 8e"
    for k, l, r in [(6, 2, 2), (12, 2, 3), (20, 4, 4)]:
        assert np.array_equal(LO.build_lrc(k, l, r)[l:], O.build_matrix(k, r, 1))  # the C oracle's Cauchy rows


@pytest.mark.parametrize("name", sorted(KAT["cases"]))
def test_frozen_kats(name):
    c = KAT["cases"][name]
    k, l, r = c["k"], c["l"], c["r"]
    P = LO.build_lrc(k, l, r)
    assert [bytes(row).hex() for row in P] == c["matrix_hex"]
    data = O.fill_random(k * 16, KAT["seed"])
    par = O.encode(k, l + r, P, data, 16, 1)
    assert [bytes(row).hex() for row in par.reshape(l + r, 16)] == c["kat_parity_hex"]
    import itertools

    tot = k + l + r
    for e, want in c["recoverable_by_erasures"].items():
        got = sum(LO.recoverable(k, P, [0 if i in er else 1 for i in range(tot)])
                  for er in itertools.combinations(range(tot), int(e)))
        assert got == want, (e, got, want)
    assert c["recoverable_by_erasures"][str(r + 1)] == len(list(itertools.combinations(range(tot), r + 1)))


def test_numpy_decode_rebuilds_from_the_read_set_only():
    k, l, r = 10, 2, 2
    tot, Ls = 14, 40
    P = LO.build_lrc(k, l, r)
    rng = np.random.default_rng(3)
    data = rng.integers(0, 256, (k, Ls), dtype=np.uint8)
    full = np.concatenate([data, LO.encode(P, data)])
    for _ in range(300):
        present = (rng.random(tot) > rng.random() * 0.5).astype(np.uint8)
        ok, surv = LO.read_set(k, l, P, present)
        assert ok == LO.recoverable(k, P, present)
        sh = np.where(present[:, None] != 0, full, 0xA5).astype(np.uint8)
        only = np.zeros(tot, dtype=np.uint8)
        only[surv] = 1
        sh[(only == 0) & (present != 0)] = 0x5A  # shards outside the read set are never read
        if LO.decode(k, l, P, sh, present):
            assert np.array_equal(sh[present == 0], full[present == 0])


_HARNESS = r"""
#include <cstdio>
#include "gf256.h"
using namespace garage_ec;
int main(int argc, char **argv)
{
    int k, m, l;
    if (scanf("%d %d %d", &k, &m, &l) != 3) return 2;
    uint8_t P[GARAGE_EC_MAX_M_HOST * GARAGE_EC_MAX_K_HOST];
    if (l ? !h_build_lrc(k, l, m - l, P) : !h_build_matrix(k, m, 0, P)) return 3;
    unsigned long long pm, wm;
    while (scanf("%llx %llx", &pm, &wm) == 2) {
        uint64_t rd = 0;
        const bool ok = h_read_plan(PlanCode{k, m, l, false, P}, pm, wm, &rd);
        printf("%d %llx\n", ok ? 1 : 0, (unsigned long long)rd);
    }
    return 0;
}
"""


@pytest.fixture(scope="module")
def read_set_harness(tmp_path_factory):
    d = tmp_path_factory.mktemp("read_set")
    src, exe = d / "h.cpp", d / "h"
    src.write_text(_HARNESS)
    subprocess.run(["g++", "-O2", "-std=c++17", "-I", os.path.join(ROOT, "garage_b200", "csrc"), "-o", str(exe),
                    str(src)], check=True)
    return str(exe)


@pytest.mark.parametrize("k,l,r", [(6, 2, 2), (10, 2, 2), (6, 0, 3)])
def test_host_read_plan_matches_rules(read_set_harness, k, l, r):
    """the survivor selection the library uses (h_read_plan: garage_ec_read_set and the HOST upload paths) against
    the Python statement of rules 1 and 2, every erasure pattern, want = every absent shard and each absent shard
    alone"""
    m = l + r
    tot = k + m
    P = LO.build_lrc(k, l, r) if l else O.build_matrix(k, m, 0)
    cases = []
    for pm in range(1 << tot):
        absent = [i for i in range(tot) if not (pm >> i) & 1]
        cases.append((pm, (1 << tot) - 1))
        cases += [(pm, 1 << o) for o in absent]
    inp = "%d %d %d\n" % (k, m, l) + "".join("%x %x\n" % c for c in cases)
    out = subprocess.run([read_set_harness], input=inp, capture_output=True, text=True, check=True).stdout.split("\n")
    for (pm, wm), line in zip(cases, out):
        present = [(pm >> i) & 1 for i in range(tot)]
        want = [(wm >> i) & 1 for i in range(tot)]
        ok, surv = LO.read_set(k, l, P, present, want)
        got_ok, got_rd = line.split()
        assert bool(int(got_ok)) == ok, (pm, wm)
        if ok:
            assert int(got_rd, 16) == sum(1 << i for i in surv), (pm, wm, got_rd, surv)


def test_create_lrc_rejects_bad_codes_before_touching_cuda():
    L = G.load_library()
    h = C.c_void_p()
    for k, l, r in [(10, 3, 2), (10, 0, 2), (10, 2, 0), (10, 5, 4), (33, 1, 1), (0, 1, 1), (10, -2, 2), (64, 2, 2)]:
        assert L.garage_ec_create_lrc(C.byref(h), 0, k, l, r) == G.E_INVALID, (k, l, r)
        assert not h.value
    assert L.garage_ec_code_info(None, None, None) == G.E_INVALID
    assert L.garage_ec_read_set(None, None, None, None) == G.E_INVALID


def _c_invertible(rows):
    M = np.ascontiguousarray(rows, dtype=np.uint8).copy()
    return O.lib().rs_oracle_invert(O._p(M), M.shape[0]) == 0


@pytest.mark.parametrize("k,l,r", [(6, 2, 2), (10, 2, 2)])
def test_recoverable_counts_by_the_c_oracle(k, l, r):
    """the pattern counts from a second arm: with want = every absent shard a pattern is recoverable iff some k of
    its present generator rows form a matrix the C oracle (log/exp Gauss-Jordan) can invert"""
    import itertools

    m = l + r
    tot = k + m
    P = LO.build_lrc(k, l, r)
    Gm = np.concatenate([np.eye(k, dtype=np.uint8), P])
    want = KAT["cases"]["lrc_%d_%d_%d" % (k, l, r)]["recoverable_by_erasures"]
    for e in range(m + 1):
        got = 0
        for er in itertools.combinations(range(tot), e):
            present = [i for i in range(tot) if i not in er]
            got += any(_c_invertible(Gm[list(sub)]) for sub in itertools.combinations(present, k))
        assert got == want[str(e)], (e, got)


def test_decode_c_oracle_agrees_with_numpy_model():
    """where the first k present shards are independent, the C oracle's decode (first k present, log/exp inverse)
    and the numpy model's (read set, own elimination) rebuild the same bytes"""
    k, l, r = 10, 2, 2
    m, tot, stride, n = 4, 14, 64, 300
    P = LO.build_lrc(k, l, r)
    Gm = np.concatenate([np.eye(k, dtype=np.uint8), P])
    rng = np.random.default_rng(9)
    lens = np.full(n, stride, dtype=np.uint32)
    data = O.fill_random(n * k * stride, 0xBC0).reshape(n, k, stride)
    par = O.encode(k, m, P, data.reshape(-1), stride, n, lens).reshape(n, m, stride)
    full = np.concatenate([data, par], axis=1)
    checked = 0
    for s in range(n):
        lost = rng.choice(tot, int(rng.integers(1, m + 1)), replace=False)
        present = np.ones(tot, dtype=np.uint8)
        present[lost] = 0
        first_k = [i for i in range(tot) if present[i]][:k]
        if not _c_invertible(Gm[first_k]):
            continue
        a = full[s].copy()
        a[present == 0] = 0
        b = a.copy()
        bad, _ = O.reconstruct(k, m, P, a.reshape(-1), present[None, :], stride, 1, lens[:1])
        assert bad == 0
        assert LO.decode(k, l, P, b, present)
        assert np.array_equal(a, b) and np.array_equal(a, full[s])
        checked += 1
    assert checked > 200
