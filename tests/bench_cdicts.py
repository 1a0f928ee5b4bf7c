"""Config 5's records (bench.py's workload: 1 048 576 x 1 KiB of datagen -P50 and its 16 KiB ZDICT dictionary, level 1)
against K = 1, 16, 256 and 4096 dictionaries, one ZSTDB200_compressFrames_usingCDicts call per step on device buffers.
The K dictionaries are config 5's under K dictIDs (one level, one size class), so the bytes differ from K = 1 only in
the frame headers' dictID; what changes with K is where the table images and tails come from (L2 for one dictionary, HBM
for thousands).  Per K, one JSON line:
  gbps, wall_ms          the whole call (best step), host clock around a synchronous call
  kernel_ms, launches    ZSTDB200_getLastStats right after that call (kernel_ms: first to last event of the call, which
                         for a multi-wave call includes the descriptor upload)
  outside_kernels_ms     wall_ms - kernel_ms: host planning, what is enqueued before the first event, the final wait
  first_use_*            the first call with K fresh CDicts: its wall time, its launches (the image builds included) and the
                         device memory it took per CDict (torch.cuda.mem_get_info around it, on a context already warmed
                         by a call of the same shape with other CDicts; the allocation granularity blurs small K)
  single_cdict_*         K = 1 only: ZSTDB200_compressFrames_usingCDict on the same records, timed the same way
  loop_gbps              ZSTD_compress_usingCDict per record on a sample (--sample records), for comparison
with the card's name and power limit.

    python tests/bench_cdicts.py [--scale 1.0] [--steps 5] [--sample 10000] [--ks 1,16,256,4096]"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import zstd_b200  # noqa: E402
from bench import Workload  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:                                          # reported, not guessed
        return f"unknown ({e})"


def with_id(d: bytes, dict_id: int) -> bytes:
    """a zstd-format dictionary under another dictID (raw content is used as it is)"""
    return d[:4] + dict_id.to_bytes(4, "little") + d[8:] if d[:4] == b"\x37\xa4\x30\xec" else d


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--sample", type=int, default=10000)
    ap.add_argument("--ks", default="1,16,256,4096")
    a = ap.parse_args()
    import torch
    wl = Workload(5, 0, 1, a.scale)
    src, level, d = wl.src, wl.level, wl.dict
    n = len(wl.frames)
    offs, sizes = [o for o, _ in wl.frames], [s for _, s in wl.frames]
    cap = sum(zstd_b200.ZSTD_compressBound(s) + 32 for s in sizes)
    d_src = torch.frombuffer(bytearray(src), dtype=torch.uint8).cuda()
    d_dst = torch.empty(cap, dtype=torch.uint8, device="cuda")
    L = zstd_b200.lib()
    c = zstd_b200.ZSTD_CCtx()
    st = zstd_b200.Stats()
    offs_a, sizes_a = (ctypes.c_size_t * n)(*offs), (ctypes.c_size_t * n)(*sizes)
    name = card()

    def timed(fn):
        """fn() once, synchronously: (wall ms, kernel ms, launches, total)"""
        torch.cuda.synchronize()
        t = time.perf_counter()
        r = fn()
        wall = 1e3 * (time.perf_counter() - t)
        assert not L.ZSTD_isError(r), L.ZSTD_getErrorName(r)
        L.ZSTDB200_getLastStats(c._h, ctypes.byref(st))
        return wall, st.kernel_ms, st.launches, r

    def many(cds):
        arr = (ctypes.c_void_p * n)(*[cds[i % len(cds)]._h for i in range(n)])
        return lambda: L.ZSTDB200_compressFrames_usingCDicts(c._h, d_dst.data_ptr(), cap, d_src.data_ptr(), offs_a, sizes_a, n, arr,
                                                             level, None, 1, None)

    warm = [zstd_b200.ZSTD_CDict(with_id(d, 900000 + j), level) for j in range(16)]
    timed(many(warm))                                               # the context's own buffers, at this shape
    for k in [int(x) for x in a.ks.split(",")]:
        cds = [zstd_b200.ZSTD_CDict(with_id(d, 1000 + j), level) for j in range(k)]
        call = many(cds)
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        cold_wall, _, cold_launches, _ = timed(call)
        torch.cuda.synchronize()
        per_cdict = (free0 - torch.cuda.mem_get_info()[0]) / k
        runs = [timed(call) for _ in range(a.steps)]
        wall, kms, launches, total = min(runs)
        row = {"K": k, "records": n, "record_size": sizes[0], "level": level, "data": wl.desc,
               "gbps": sum(sizes) / wall / 1e6, "wall_ms": wall, "kernel_ms": kms, "outside_kernels_ms": wall - kms,
               "launches": launches, "ratio": sum(sizes) / total,
               "first_use_wall_ms": cold_wall, "first_use_launches": cold_launches, "first_use_device_bytes_per_cdict": per_cdict}
        if k == 1:
            single = lambda: L.ZSTDB200_compressFrames_usingCDict(c._h, d_dst.data_ptr(), cap, d_src.data_ptr(), offs_a, sizes_a, n,
                                                                  cds[0]._h, None, 1, None)
            s_wall, s_kms, s_launches, s_total = min(timed(single) for _ in range(a.steps))
            row.update({"single_cdict_gbps": sum(sizes) / s_wall / 1e6, "single_cdict_wall_ms": s_wall, "single_cdict_kernel_ms": s_kms,
                        "single_cdict_launches": s_launches, "single_cdict_same_total": s_total == total})
        ns = min(a.sample, n)
        t = time.perf_counter()
        for i in range(ns):
            c.compress_using_cdict(src[offs[i]:offs[i] + sizes[i]], cds[i % k])
        row.update({"loop_gbps": sum(sizes[:ns]) / (time.perf_counter() - t) / 1e9, "loop_sample": ns, "card": name})
        print(json.dumps(row), flush=True)
        for cd in cds:
            cd.close()
    for cd in warm:
        cd.close()
    c.close()


if __name__ == "__main__":
    main()
