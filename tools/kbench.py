#!/usr/bin/env python
"""Kernel micro-bench for tuning: times garage_ec_encode / _reconstruct / _verify (DEVICE mode)
of one .so variant on the BASELINE config-2/3 workload.  Not the contract bench (bench.py).

    python tools/kbench.py [--so path/to/libgarage_ec.so] [--k 10 --m 4 --blocks 4096 --iters 10]
    python tools/kbench.py --k 10 --lrc 2 --m 4              # LRC(10,2,2): l = 2 local groups, m = l + r
    python tools/kbench.py --k 10 --lrc 2 --m 4 --erasures 1 --local   # one lost data / local-parity shard
    python tools/kbench.py --k 10 --m 4 --pb [--erasures 1 --local]     # PB(10,4) and RS(10,4), one line each
    python tools/kbench.py --transcode 6,3:10,4 [--rounds 3]  # code conversion; also lrc:10,2,2  pb:10,4  rep
    python tools/kbench.py --k 10 --m 4 --clay [--rounds 3]   # RS, PB and Clay(10,4), alternating; m losses, then 1
Reconstruct bytes are the survivor bytes garage_ec_read_ranges names (whole shards, PB halves, Clay repair runs) plus
the shards rebuilt.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ap = argparse.ArgumentParser()
ap.add_argument("--so", default=None)
ap.add_argument("--k", type=int, default=10)
ap.add_argument("--m", type=int, default=4)
ap.add_argument("--blocks", type=int, default=4096)
ap.add_argument("--iters", type=int, default=10)
ap.add_argument("--erasures", type=int, default=None)
ap.add_argument("--same-pattern", action="store_true", help="all stripes lose the same shards")
ap.add_argument("--lrc", type=int, default=0, help="LRC with this many local groups (m = local + global parities)")
ap.add_argument("--local", action="store_true", help="erase only data / local-parity shards (LRC local repair)")
ap.add_argument("--pb", action="store_true", help="piggybacked RS PB(k, m), reported next to RS(k, m)")
ap.add_argument("--clay", action="store_true", help="Clay(k, m) next to RS(k, m) and PB(k, m), alternating rounds")
ap.add_argument("--transcode", default=None, help="SRC:DST codes: k,m | lrc:k,l,r | pb:k,m | rep (whole blocks)")
ap.add_argument("--rounds", type=int, default=3, help="--transcode: alternating rounds of the compared paths")
ap.add_argument("--tag", default="")
ap.add_argument("--stride-pad", type=int, default=0, help="extra bytes between shards (multiple of 16)")
args = ap.parse_args()

from garage_b200 import _build  # noqa: E402

if args.so:
    _build.SO = os.path.abspath(args.so)
    _build.stale = lambda: False
import torch  # noqa: E402

import garage_b200 as G  # noqa: E402

k, m, n = args.k, args.m, args.blocks
tot = k + m
ERASURES = args.erasures if args.erasures is not None else m
B = 1 << 20


def measure(ec, e):
    """encode / reconstruct / verify of one context on the workload, e erasures per stripe: (times, shard_len,
    present, ok, shards)"""
    L = ec.code_shard_len(B)
    stride = ec.stride_for(L) + args.stride_pad
    shards = torch.zeros(n * tot * stride, dtype=torch.uint8, device="cuda")
    sh3 = shards.view(n, tot, stride)
    data = torch.empty(n * k * stride, dtype=torch.uint8, device="cuda")
    ec.fill_random(data, n * k * stride, 1, 0)
    data.view(n, k, stride)[:, :, L:] = 0
    lens = torch.full((n,), L, dtype=torch.int32, device="cuda")
    parity = torch.zeros(n * m * stride, dtype=torch.uint8, device="cuda")
    ec.encode(data, parity, stride, n, shard_len=lens)
    sh3[:, :k] = data.view(n, k, stride)
    sh3[:, k:] = parity.view(n, m, stride)
    orig = shards.clone()
    g = torch.Generator().manual_seed(7)
    span = k + args.lrc if args.local else tot  # --local: erase among the data and local-parity shards
    if args.same_pattern:
        erased = torch.arange(e).repeat(n, 1)
    else:
        erased = torch.rand(n, span, generator=g).argsort(dim=1)[:, :e]
    present = torch.ones(n, tot, dtype=torch.uint8)
    if e:
        present.scatter_(1, erased, 0)
    pd = present.cuda()
    sh3[~pd.bool()] = 0
    status = torch.zeros(n, dtype=torch.int32, device="cuda")
    mm = torch.zeros(n, dtype=torch.int32, device="cuda")
    t_enc = timeit(lambda: ec.encode(data, parity, stride, n, shard_len=lens), ec)
    t_dec = timeit(lambda: ec.reconstruct(shards, pd, stride, n, status=status, shard_len=lens), ec)
    ok = torch.equal(shards, orig) and int(status.abs().sum()) == 0
    t_ver = timeit(lambda: ec.verify(shards, mm, stride, n, shard_len=lens), ec)
    ok = ok and int(mm.abs().sum()) == 0
    return (t_enc, t_dec, t_ver), L, present.numpy(), ok, orig


def timeit(fn, ctx):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ctx.set_timing(True)
    ctx.timing_read()
    for _ in range(args.iters):
        fn()
    torch.cuda.synchronize()
    ms, cnt = ctx.timing_read()
    ctx.set_timing(False)
    return ms / max(cnt, 1)


def copy_gbs(orig):
    """read+write GB/s of a plain device copy of <= 1 GiB on this GPU in this run (best of 6): the peak of the fractions"""
    cp_n = min(1 << 30, orig.numel() // 2)
    src, dst = orig[:cp_n], orig[cp_n:2 * cp_n]
    best = None
    for _ in range(6):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        dst.copy_(src)
        b.record()
        torch.cuda.synchronize()
        best = a.elapsed_time(b) if best is None else min(best, a.elapsed_time(b))
    return 2 * cp_n / (best * 1e-3) / 1e9


def power_limit():
    import subprocess

    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:
        return None


def report(ec, code, e=ERASURES):
    (t_enc, t_dec, t_ver), L, pres_np, ok, orig = measure(ec, e)
    peak = copy_gbs(orig)
    del orig
    enc_b = n * (k + m) * L
    nsurv = 0  # shards' worth of survivor bytes read
    for s in range(n):
        runs = ec.read_ranges(pres_np[s], L)
        nsurv += sum(r[2] for r in runs) / L if runs is not None else 0
    dec_b = int((nsurv + n * e) * L)
    print(json.dumps({
        "tag": args.tag or (args.so or "default"), "code": code, "k": k, "m": m, "lrc_local_groups": args.lrc,
        "blocks": n, "erasures": e, "shard_len": L,
        "local": bool(args.local), "survivors_per_stripe": round(nsurv / n, 3),
        "survivor_bytes_per_stripe": int(nsurv / n * L), "ok": bool(ok),
        "copy_GBs": round(peak, 1), "gpu": torch.cuda.get_device_name(0), "power_limit_W": power_limit(),
        "encode_ms": round(t_enc, 4), "encode_GBs": round(enc_b / t_enc / 1e6, 1), "encode_frac": round(enc_b / t_enc / 1e6 / peak, 4),
        "decode_ms": round(t_dec, 4), "decode_GBs": round(dec_b / t_dec / 1e6, 1), "decode_frac": round(dec_b / t_dec / 1e6 / peak, 4),
        "verify_ms": round(t_ver, 4), "verify_GBs": round(enc_b / t_ver / 1e6, 1), "verify_frac": round(enc_b / t_ver / 1e6 / peak, 4),
    }), flush=True)


def parse_code(t):
    if t == "rep":
        return None, "rep", 1, 0
    kind, _, nums = t.rpartition(":")
    v = [int(x) for x in nums.split(",")]
    if kind == "lrc":
        return G.GarageEc.lrc(0, *v), "LRC(%d,%d,%d)" % tuple(v), v[0], v[1] + v[2]
    if kind == "pb":
        return G.GarageEc.piggyback(0, *v), "PB(%d,%d)" % tuple(v), v[0], v[1]
    return G.GarageEc(0, *v), "RS(%d,%d)" % tuple(v), v[0], v[1]


def event_ms(fn):
    """mean device time of fn over args.iters calls, after 3 warm-up calls"""
    for _ in range(3):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(args.iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / args.iters


def transcode_bench():
    """garage_ec_transcode (reframe + the destination's encode) against torch reframe + garage_ec_encode, same batch,
    alternating; algorithmic bytes = k_s*L_s read + (k_d+m_d)*L_d written per block"""
    toks, codes = args.transcode.split(":"), []
    while toks:  # "lrc" / "pb" take the next token as their numbers
        t = toks.pop(0)
        codes.append(t + ":" + toks.pop(0) if t in ("lrc", "pb") else t)
    (src, sname, ks, ms), (dst, dname, kd, md) = (parse_code(t) for t in codes)
    Ls = src.code_shard_len(B) if src else B
    Ld = dst.code_shard_len(B)
    ss, ds = (src.stride_for(Ls) if src else (B + 15) // 16 * 16), dst.stride_for(Ld)
    st, dt = ks + ms, kd + md
    sh = torch.zeros((n, st, ss), dtype=torch.uint8, device="cuda")
    fill = torch.empty(n * ks * ss, dtype=torch.uint8, device="cuda")
    dst.fill_random(fill, fill.numel(), 3, 0)
    sh[:, :ks] = fill.view(n, ks, ss)
    del fill
    sh[:, :ks, Ls:] = 0
    out = torch.zeros((n, dt, ds), dtype=torch.uint8, device="cuda")
    bl = torch.full((n,), B, dtype=torch.int32, device="cuda")
    data = torch.zeros((n, kd, ds), dtype=torch.uint8, device="cuda")
    par = torch.zeros((n, md, ds), dtype=torch.uint8, device="cuda")
    flat = torch.zeros((n, kd * Ld), dtype=torch.uint8, device="cuda")
    lens = torch.full((n,), Ld, dtype=torch.int32, device="cuda")

    def transcode():
        dst.transcode(src, sh.view(-1), bl, ss, out.view(-1), ds, n)

    def torch_encode():
        flat[:, :B] = sh[:, :ks, :Ls].reshape(n, ks * Ls)[:, :B]
        data[:, :, :Ld] = flat.view(n, kd, Ld)
        dst.encode(data.view(-1), par.view(-1), ds, n, shard_len=lens)

    transcode()
    torch_encode()
    torch.cuda.synchronize()
    ok = torch.equal(out[:, :kd, :Ld], data[:, :, :Ld]) and torch.equal(out[:, kd:, :Ld], par[:, :, :Ld])
    peak = copy_gbs(out.view(-1))
    alg = n * (ks * Ls + dt * Ld)
    res = {"transcode_ms": [], "torch_reframe_encode_ms": []}
    for _ in range(args.rounds):
        res["transcode_ms"].append(round(event_ms(transcode), 4))
        res["torch_reframe_encode_ms"].append(round(event_ms(torch_encode), 4))
    best = {key: min(v) for key, v in res.items()}
    print(json.dumps({
        "tag": args.tag or (args.so or "default"), "transcode": "%s->%s" % (sname, dname), "blocks": n, "block_len": B,
        "ok": bool(ok), "alg_bytes": alg, "copy_GBs": round(peak, 1), "gpu": torch.cuda.get_device_name(0),
        "power_limit_W": power_limit(), **res,
        **{key.replace("_ms", "_frac"): round(alg / v / 1e6 / peak, 4) for key, v in best.items()},
    }), flush=True)


if args.transcode:
    transcode_bench()
elif args.clay:  # Clay(k, m) next to RS(k, m) and PB(k, m): m losses, then one, in alternating rounds
    for rnd in range(args.rounds):
        for erasures in (m, 1):
            for code, make in (("RS(%d,%d)" % (k, m), lambda: G.GarageEc(0, k, m)),
                               ("PB(%d,%d)" % (k, m), lambda: G.GarageEc.piggyback(0, k, m)),
                               ("Clay(%d,%d)" % (k, m), lambda: G.GarageEc.clay(0, k, m))):
                with make() as ctx:
                    report(ctx, code, erasures)
                    torch.cuda.empty_cache()
elif args.pb:  # PB(k, m) next to RS(k, m) on the same workload, one line each
    for code, make in (("RS(%d,%d)" % (k, m), lambda: G.GarageEc(0, k, m)),
                       ("PB(%d,%d)" % (k, m), lambda: G.GarageEc.piggyback(0, k, m))):
        with make() as ctx:
            report(ctx, code)
            torch.cuda.empty_cache()
elif args.lrc:
    report(G.GarageEc.lrc(0, k, args.lrc, m - args.lrc), "LRC(%d,%d,%d)" % (k, args.lrc, m - args.lrc))
else:
    report(G.GarageEc(0, k, m), "RS(%d,%d)" % (k, m))
