"""Cost and gain of long-distance matching (ZSTD_c_enableLongDistanceMatching) on the GPU, device-resident inputs:
  - datagen -P50 at level 1 (config 2's input), LDM off and on;
  - a versioned input: versions of one datagen file, each 400 random byte edits away from the one before, LDM off and on,
    with the size of the reference's LDM frame for it (oracle/_ref, compiled by build()).
Per case: GB/s of ZSTDB200_compressDevice (median of --iters calls, CUDA events around each call), the size, whether the
frame decodes (GPU decoder and, where built, the reference's), and for LDM on the match phase of a one-wave call (caller
stream, events around each phase) with and without LDM: their difference over the call's kernel time is `ldm_share`, the
LDM pass plus what the 2^27 window changes in the parse.
Prints one JSON line with the card's name and power limit.  Needs a GPU.

    python tests/bench_ldm.py [--mib 1024] [--version-mib 32] [--iters 5]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ldmref  # noqa: E402
import zref  # noqa: E402
import zstd_b200  # noqa: E402


def versioned(total: int, version: int, seed: int = 3) -> bytes:
    rng = np.random.default_rng(seed)
    cur = np.frombuffer(zref.datagen(version, 50, seed), dtype=np.uint8).copy()
    out = []
    for _ in range(total // version):
        out.append(cur.tobytes())
        idx = rng.integers(0, version, 400)
        cur[idx] = rng.integers(0, 256, 400, dtype=np.uint8)
    return b"".join(out)


def run(torch, src, level, ldm, iters):
    n = len(src)
    d_src = torch.frombuffer(bytearray(src), dtype=torch.uint8).cuda()
    cap = zstd_b200.ZSTD_compressBound(n) + 4096
    d_dst = torch.empty(cap, dtype=torch.uint8, device="cuda")
    c = zstd_b200.ZSTD_CCtx()
    c.set_parameter("enable_long_distance_matching", 1 if ldm else 2)
    times, size = [], 0
    for i in range(iters + 1):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        size = c.compress_device(d_dst.data_ptr(), cap, d_src.data_ptr(), n, level)
        b.record()
        torch.cuda.synchronize()
        if i:
            times.append(a.elapsed_time(b))
    ms = float(np.median(times))
    frame = d_dst[:size].cpu().numpy().tobytes()
    ok = zstd_b200.ZSTD_DCtx().decompress(frame, n) == src             # every frame measured is decoded again on the GPU
    if zref.have_ref():
        ok = ok and zref.ref_decompress(frame, n) == src               # and by the reference decoder
    out = {"bytes": size, "ms": round(ms, 3), "GBps": round(n / ms / 1e6, 2), "roundtrip_ok": ok}
    if ldm:
        # one wave on a caller stream: the executor times the match phase (LDM pass, walk, parse, merge) with events
        s = torch.cuda.Stream()
        c.compress_device(d_dst.data_ptr(), cap, d_src.data_ptr(), n, level, s.cuda_stream)
        torch.cuda.synchronize()
        st = c.stats()
        c2 = zstd_b200.ZSTD_CCtx()
        c2.compress_device(d_dst.data_ptr(), cap, d_src.data_ptr(), n, level, s.cuda_stream)
        torch.cuda.synchronize()
        st2 = c2.stats()
        out["one_wave_kernel_ms"] = round(st.kernel_ms, 3)
        out["one_wave_match_ms"] = round(st.match_ms, 3)
        out["one_wave_match_ms_without_ldm"] = round(st2.match_ms, 3)
        out["ldm_share"] = round(max(0.0, st.match_ms - st2.match_ms) / st.kernel_ms, 3) if st.kernel_ms else None
    return out


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=1024)
    ap.add_argument("--version-mib", type=int, default=32)
    ap.add_argument("--iters", type=int, default=5)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = {"gpu": gpu, "mib": a.mib}
    src = zref.datagen(a.mib << 20, 50, seed=0)
    res["datagen_P50_l1"] = {"off": run(torch, src, 1, False, a.iters), "on": run(torch, src, 1, True, a.iters)}
    v = versioned(a.mib << 20, a.version_mib << 20)
    res["versions_l1"] = {"off": run(torch, v, 1, False, a.iters), "on": run(torch, v, 1, True, a.iters)}
    if zref.have_ref():
        res["versions_l1"]["reference_ldm_bytes"] = len(ldmref.ref_compress2(v, 1, 1))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
