#!/usr/bin/env python
"""Stream-ordered compression against the synchronous device call (ZSTDB200_compressDeviceAsync / ZSTDB200_compressDevice).

  1. One 1 GiB call of bench.py's config 2 (datagen -P50, level 1): ZSTDB200_compressDevice with the NULL stream against
     the stream-ordered call followed by a synchronise.  The frames must be identical.
  2. 256 calls of 1 MiB and 256 of 16 MiB at level 1 on one context, three ways: synchronous calls; stream-ordered calls on
     one stream and one synchronise at the end; one replay per call of a CUDA graph holding one captured call.

Each figure is the median of --iters timed repetitions (host clock around work that ends in a device synchronise).  Prints
one JSON line with the card's name and power limit, read in the same run.  Needs a GPU.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

import zref  # noqa: E402
import zstd_b200  # noqa: E402

GiB, MiB = 1 << 30, 1 << 20


def _cap(n):
    return zstd_b200.ZSTD_compressBound(n) + 64


def _median_s(fn, iters):
    ts = []
    for _ in range(iters):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return statistics.median(ts)


def one_large(d_src, iters):
    n = d_src.numel()
    ctx = zstd_b200.ZSTD_CCtx()
    d_a = torch.zeros(_cap(n), dtype=torch.uint8, device="cuda")
    d_b = torch.zeros(_cap(n), dtype=torch.uint8, device="cuda")
    res = torch.zeros(1, dtype=torch.int64, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    size = {}

    def sync_call():
        size["sync"] = ctx.compress_device(d_a.data_ptr(), d_a.numel(), d_src.data_ptr(), n, 1, 0)

    def async_call():
        ctx.compress_device_async(d_b.data_ptr(), d_b.numel(), d_src.data_ptr(), n, res.data_ptr(), 1, stream)

    sync_call(); async_call()                                   # warm-up of both paths
    t_sync, t_async = [], []
    for _ in range(iters):                                      # alternated, so that both see the same card state
        t_sync.append(_median_s(sync_call, 1)); t_async.append(_median_s(async_call, 1))
    r = int(res.item())
    same = r == size["sync"] and torch.equal(d_a[:r], d_b[:r])
    ts, ta = statistics.median(t_sync), statistics.median(t_async)
    return {"bytes": n, "compressed": r, "identical": bool(same),
            "sync_GBps": round(n / ts / 1e9, 2), "async_GBps": round(n / ta / 1e9, 2),
            "sync_ms": round(1e3 * ts, 3), "async_ms": round(1e3 * ta, 3)}


def many_calls(pool, size, calls, iters):
    ctx = zstd_b200.ZSTD_CCtx()
    span = pool.numel() - size
    offs = [(i * 7919 * 4096) % span for i in range(calls)]     # distinct inputs from the pool
    cap = _cap(size)
    d_dst = torch.zeros(calls * cap, dtype=torch.uint8, device="cuda")
    res = torch.zeros(calls, dtype=torch.int64, device="cuda")
    src = pool.data_ptr()
    dst = d_dst.data_ptr()
    stream = torch.cuda.current_stream().cuda_stream

    def sync_calls():
        for i in range(calls):
            ctx.compress_device(dst + i * cap, cap, src + offs[i], size, 1, 0)

    def async_calls():
        for i in range(calls):
            ctx.compress_device_async(dst + i * cap, cap, src + offs[i], size, res.data_ptr() + 8 * i, 1, stream)

    sync_calls(); async_calls()
    gctx = zstd_b200.ZSTD_CCtx()                                # a captured call's context makes no other call while its graph lives
    gctx.compress_device_async(dst, cap, src + offs[0], size, res.data_ptr(), 1, stream)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        gctx.compress_device_async(dst, cap, src + offs[0], size, res.data_ptr(), 1, torch.cuda.current_stream().cuda_stream)

    def replays():
        for _ in range(calls):
            g.replay()

    replays()
    out = {"call_bytes": size, "calls": calls}
    for name, fn in (("sync", sync_calls), ("async", async_calls), ("graph", replays)):
        t = _median_s(fn, iters)
        out[name] = {"calls_per_s": round(calls / t, 1), "GBps": round(calls * size / t / 1e9, 2), "ms": round(1e3 * t, 3)}
    del g
    gctx.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--calls", type=int, default=256)
    ap.add_argument("--out", default=None, help="directory that also receives the JSON line (bench_async.json)")
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    src = zref.datagen(GiB, 50) if zref.have_datagen() else zref.synthetic(GiB, seed=0, match_prob=0.5)
    d_src = torch.frombuffer(bytearray(src), dtype=torch.uint8).cuda()
    del src
    rec = {"gpu": gpu, "input": "datagen -g1GB -P50" if zref.have_datagen() else "zbo_synthetic 1 GiB",
           "one_1GiB_call_level1": one_large(d_src, a.iters),
           "calls_1MiB": many_calls(d_src, MiB, a.calls, a.iters),
           "calls_16MiB": many_calls(d_src, 16 * MiB, a.calls, a.iters)}
    line = json.dumps(rec)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_async.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
