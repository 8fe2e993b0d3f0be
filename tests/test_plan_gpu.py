"""The device planner (plan_kernel) against its host twin (garage_ec_read_plan) for RS, LRC and PB: for every erasure
pattern, with want = every absent shard and each absent shard alone, a DEVICE reconstruct whose present shards (PB:
halves) outside the host read plan hold poison rebuilds the encoded bytes, and fails exactly where the host plan
does."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import lrc_oracle as LO  # noqa: E402
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


def codewords(code, k, m, stride, lens, seed):
    """(len(lens), k+m, stride) codewords of `code` with shard_len lens[i], zero past it, and the context factory"""
    n = len(lens)
    data = O.fill_random(n * k * stride, seed).reshape(n, k, stride)
    for i in range(n):
        data[i, :, lens[i]:] = 0
    sh = np.zeros((n, k + m, stride), dtype=np.uint8)
    sh[:, :k] = data
    if code == "pb":
        P = PB.build(k, m)
        for i in range(n):
            sh[i, k:, :lens[i]] = PB.encode(P, data[i, :, :lens[i]])
        return sh, lambda: G.GarageEc.piggyback(0, k, m)
    if code == "lrc":
        P, make = LO.build_lrc(k, 2, m - 2), lambda: G.GarageEc.lrc(0, k, 2, m - 2)
    else:
        P, make = O.build_matrix(k, m, 0), lambda: G.GarageEc(0, k, m)
    sh[:, k:] = O.encode(k, m, P, data.reshape(-1), stride, n, lens).reshape(n, m, stride)
    return sh, make


@pytest.mark.parametrize("code,k,m", [("rs", 6, 3), ("lrc", 10, 4), ("pb", 6, 3)])
def test_device_plan_reads_only_the_host_read_plan(torch, code, k, m):
    tot, stride, nbase = k + m, 64, 64
    lens_base = np.array([32 * (1 + i % 2) for i in range(nbase)], dtype=np.uint32)
    base, make = codewords(code, k, m, stride, lens_base, 0x9D0 + k)
    present_l, want_l = [], []
    eye = np.eye(tot, dtype=np.uint8)
    for p in range(1 << tot):
        pr = np.array([((p >> i) & 1) ^ 1 for i in range(tot)], dtype=np.uint8)
        present_l.append(pr)
        want_l.append(np.ones(tot, dtype=np.uint8))
        for o in np.flatnonzero(pr == 0):
            present_l.append(pr)
            want_l.append(eye[o])
    n = len(present_l)
    present, want = np.array(present_l), np.array(want_l)
    idx = np.arange(n) % nbase
    orig, lens = base[idx], lens_base[idx]
    with make() as ec:
        halves = np.zeros((n, tot), dtype=np.uint8)  # bit 0: a-half read, bit 1: b-half
        ok = np.zeros(n, dtype=bool)
        for s in range(n):
            hv = ec.read_plan(present[s], want[s])
            if hv is not None:
                ok[s] = True
                halves[s] = hv
        assert ok.any() and not ok.all()
        assert ((halves != 0) <= (present != 0)).all()
        col = np.arange(stride)[None, None, :]
        half = (lens // 2)[:, None, None]
        in_a, in_b = col < half, (col >= half) & (col < 2 * half)
        keep = (in_a & ((halves & 1) != 0)[:, :, None]) | (in_b & ((halves & 2) != 0)[:, :, None])
        broken = np.where(keep | ~(in_a | in_b), orig, POISON).astype(np.uint8)
        d =torch.from_numpy(broken).cuda()
        status = torch.full((n,), 99, dtype=torch.int32, device="cuda")
        ec.reconstruct(d, torch.from_numpy(present).cuda(), stride, n, want=torch.from_numpy(want).cuda(),
                       status=status, shard_len=torch.from_numpy(lens).cuda())
        got, st = d.cpu().numpy(), status.cpu().numpy()
    assert np.array_equal(st, np.where(ok, 0, G.E_UNRECOVERABLE))
    rebuilt = (present == 0) & (want != 0) & ok[:, None]
    exp = np.where(rebuilt[:, :, None] & (in_a | in_b), orig, broken)
    assert np.array_equal(got, exp)
