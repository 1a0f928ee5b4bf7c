"""Cost and gain of compressing a new version of a file against the old one (ZSTDB200_CCtx_refPrefixDevice + long-distance
matching, what `zstd --patch-from` does), device-resident, level 1.  Per size (default 64 and 16 MiB): old = seeded
synthetic data, new = old with a few thousand random byte edits and one region shifted by an insertion.
  - frame size: with the prefix (LDM on), LDM on without a prefix, plain level 1;
  - GB/s of input of ZSTDB200_compressDevice for the three (median of --iters calls after one warm-up call, CUDA events
    around each call; the with-prefix call includes setting the prefix);
  - the LDM kernels of one with-prefix call by name from torch.profiler (a separate, profiled call): split (both
    segments), scans + compaction, radix sort, select, against the call's whole kernel time;
  - decoding the patch frame on the GPU with the prefix (ZSTDB200_decompressDevice_usingDict: the prefix comes from host
    memory, so the call's time includes its upload; kernel_ms is the decoder's own event time), checked against the input.
Prints one JSON line with the card's name and power limit.  Needs a GPU.

    python tests/bench_patch.py [--mib 64 16] [--iters 7] [--out DIR]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import zref  # noqa: E402
import zstd_b200  # noqa: E402


def version_pair(size: int, seed: int = 5):
    rng = np.random.default_rng(seed)
    old = np.frombuffer(zref.synthetic(size, seed=seed), dtype=np.uint8)
    new = old.copy()
    edits = max(256, size >> 14)                                   # 4096 edits in 64 MiB
    idx = rng.integers(0, size, edits)
    new[idx] = rng.integers(0, 256, edits, dtype=np.uint8)
    at, ins = size // 3, 4099                                      # everything behind `at` moves by an odd distance
    new = np.concatenate([new[:at], rng.integers(0, 256, ins, dtype=np.uint8), new[at:size - ins]])
    return old.tobytes(), new.tobytes()


def timed(torch, call, iters):
    times, size = [], 0
    for i in range(iters + 1):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        size = call()
        b.record()
        torch.cuda.synchronize()
        if i:
            times.append(a.elapsed_time(b))
    return size, float(np.median(times)), float(min(times)), float(max(times))


def ldm_kernels(torch, call):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    groups = {"split": 0.0, "scan_compact": 0.0, "radix_sort": 0.0, "select": 0.0, "all_kernels": 0.0}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        us = e.cuda_time_total if us is None else us
        if "Memcpy" in e.key or "Memset" in e.key:
            continue
        groups["all_kernels"] += us
        if "zb_ldm_split" in e.key:
            groups["split"] += us
        elif "zb_ldm_radix" in e.key:
            groups["radix_sort"] += us
        elif "zb_ldm_select" in e.key:
            groups["select"] += us
        elif "zb_ldm_scan" in e.key or "zb_ldm_compact" in e.key:
            groups["scan_compact"] += us
    return {k + "_ms": round(v / 1e3, 3) for k, v in groups.items()}


def one_size(torch, mib, iters):
    old, new = version_pair(mib << 20)
    n = len(new)
    d_old = torch.frombuffer(bytearray(old), dtype=torch.uint8).cuda()
    d_new = torch.frombuffer(bytearray(new), dtype=torch.uint8).cuda()
    cap = zstd_b200.ZSTD_compressBound(n) + 4096
    d_dst = torch.empty(cap, dtype=torch.uint8, device="cuda")
    res = {}

    def ctx(ldm):
        c = zstd_b200.ZSTD_CCtx()
        c.set_parameter("enable_long_distance_matching", 1 if ldm else 2)
        return c

    c = ctx(True)

    def patch():
        c.ref_prefix_device(d_old.data_ptr(), len(old))
        return c.compress_device(d_dst.data_ptr(), cap, d_new.data_ptr(), n, 1)

    for name, call in (("plain", lambda cc=ctx(False): cc.compress_device(d_dst.data_ptr(), cap, d_new.data_ptr(), n, 1)),
                       ("ldm", lambda cc=ctx(True): cc.compress_device(d_dst.data_ptr(), cap, d_new.data_ptr(), n, 1)),
                       ("prefix_ldm", patch)):
        size, ms, lo, hi = timed(torch, call, iters)
        res[name] = {"bytes": size, "ms": round(ms, 3), "ms_min": round(lo, 3), "ms_max": round(hi, 3), "GBps": round(n / ms / 1e6, 2)}
    frame = d_dst[:res["prefix_ldm"]["bytes"]].clone()              # the last call measured was the patch
    res["prefix_ldm"]["kernels"] = ldm_kernels(torch, patch)
    # decode on the GPU with the prefix
    L = zstd_b200.lib()
    L.ZSTDB200_decompressDevice_usingDict.restype = ctypes.c_size_t
    L.ZSTDB200_decompressDevice_usingDict.argtypes = [ctypes.c_void_p] * 2 + [ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p,
                                                      ctypes.c_size_t, ctypes.c_void_p]
    d = zstd_b200.ZSTD_DCtx()
    d_out = torch.empty(n, dtype=torch.uint8, device="cuda")
    pbuf = ctypes.create_string_buffer(old, len(old))
    times, kern = [], []
    for i in range(iters + 1):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = zstd_b200._check(L.ZSTDB200_decompressDevice_usingDict(d._h, d_out.data_ptr(), n, frame.data_ptr(), frame.numel(), pbuf, len(old), None))
        torch.cuda.synchronize()
        if i:
            times.append(1e3 * (time.perf_counter() - t0))
            kern.append(d.stats().kernel_ms)
    ok = r == n and bool(torch.equal(d_out, d_new))
    res["decode_with_prefix"] = {"call_ms": round(float(np.median(times)), 3), "kernel_ms": round(float(np.median(kern)), 3),
                                 "GBps_of_call": round(n / float(np.median(times)) / 1e6, 2), "roundtrip_ok": ok}
    return res


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, nargs="+", default=[64, 16])
    ap.add_argument("--iters", type=int, default=7)
    ap.add_argument("--out", default=None, help="directory that also receives the JSON line (bench_patch.json)")
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = {"gpu": gpu, "level": 1, "iters": a.iters}
    for mib in a.mib:
        res[f"{mib}MiB"] = one_size(torch, mib, a.iters)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_patch.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
