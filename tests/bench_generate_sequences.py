"""Throughput of ZSTDB200_generateSequencesDevice against ZSTDB200_compressDevice on device-resident datagen input: config 2
(1 GiB P50, level 1) and config 4 (1 GiB P90, level 3).  The two calls alternate in one process, after a warm-up of both,
each timed with CUDA events on a caller stream (one wave) and with the host clock around the NULL-stream call (the wave
streams; the call ends with its read-back).  A separate run under torch.profiler gives the export kernels' time, which is
set against the bytes they must move (K1c's packed stores and the block descriptors in, the 16-byte rows out) at the
H100 SXM's 3.35 TB/s.  Prints one JSON line per config with the card's name and power limit.  Needs a GPU.

    python tests/bench_generate_sequences.py [--mib 1024] [--iters 5] [--configs 2 4]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import zref  # noqa: E402
import zstd_b200  # noqa: E402

CONFIGS = {2: (50, 1), 4: (90, 3)}                  # datagen -P, level (BASELINE.md)
HBM_BPS = 3.35e12
BLOCK_DESC, BLOCK_META = 40, 32                      # sizeof(ZbBlock), sizeof(ZbBlockMeta): read by the scan and the export


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
    return q.stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=1024)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--configs", type=int, nargs="+", default=[2, 4])
    args = ap.parse_args()
    import torch
    n = args.mib << 20
    gib = n / (1 << 30)
    for cfg in args.configs:
        p, level = CONFIGS[cfg]
        src = zref.datagen(n, p, seed=0)
        d_src = torch.frombuffer(bytearray(src), dtype=torch.uint8).cuda()
        del src
        cap = zstd_b200.sequence_bound(n)
        d_seq = torch.empty(cap * 16, dtype=torch.uint8, device="cuda")
        fcap = zstd_b200.ZSTD_compressBound(n)
        d_dst = torch.empty(fcap, dtype=torch.uint8, device="cuda")
        ctx = zstd_b200.ZSTD_CCtx()
        ctx.set_parameter("compression_level", level)
        s = torch.cuda.Stream()
        gen = lambda st: ctx.generate_sequences_device(d_seq.data_ptr(), cap, d_src.data_ptr(), n, st)   # noqa: E731
        comp = lambda st: ctx.compress_device(d_dst.data_ptr(), fcap, d_src.data_ptr(), n, level, st)    # noqa: E731
        torch.cuda.synchronize()
        count = gen(s.cuda_stream); gen(0); comp(s.cuda_stream); comp(0)
        torch.cuda.synchronize()
        ev = {k: [] for k in ("gen", "comp")}
        host = {k: [] for k in ("gen", "comp")}
        for _ in range(args.iters):
            for k, f in (("gen", gen), ("comp", comp)):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(s)
                f(s.cuda_stream)
                b.record(s)
                b.synchronize()
                ev[k].append(a.elapsed_time(b))
                t = time.perf_counter()
                f(0)
                host[k].append(1e3 * (time.perf_counter() - t))
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            gen(s.cuda_stream)
            torch.cuda.synchronize()
        export_us = sum(e.device_time_total for e in prof.key_averages() if "seqexport" in e.key)
        nb = ctx.stats().nbBlocks
        moved = 8 * (count - nb) + 2 * (BLOCK_DESC + BLOCK_META) * nb + 16 * count + 8 * (nb + 1)
        st = {"config": cfg, "level": level, "datagen_P": p, "mib": args.mib, "gpu": card(),
              "generate_GBps_events": round(n / (min(ev["gen"]) * 1e-3) / 1e9, 2),
              "compress_GBps_events": round(n / (min(ev["comp"]) * 1e-3) / 1e9, 2),
              "generate_ms_events": [round(x, 3) for x in ev["gen"]], "compress_ms_events": [round(x, 3) for x in ev["comp"]],
              "generate_ms_null_stream": [round(x, 3) for x in host["gen"]], "compress_ms_null_stream": [round(x, 3) for x in host["comp"]],
              "sequences_per_GiB": round(count / gib), "export_ms": round(export_us / 1e3, 4),
              "export_ms_per_GiB": round(export_us / 1e3 / gib, 4),
              "export_bytes": moved, "export_share_of_hbm_peak": round(moved / HBM_BPS / (export_us * 1e-6), 3) if export_us else None}
        print(json.dumps(st), flush=True)
        del d_src, d_seq, d_dst, ctx
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
