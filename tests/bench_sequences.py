"""Throughput of the sequence entry points (ZSTD_compressSequences, ZSTDB200_compressSequencesDevice) on 1 GiB of datagen
P50, with the sequences the compiled reference's ZSTD_generateSequences finds at level 1, taken in 32 MiB slices (one
call over the whole input would need an output buffer of about 5.7 GB; each slice's sequences, delimiters included, are
valid for the whole input when they are laid end to end).  Prints one JSON line: device-resident GB/s, the per-kernel
split of a single-wave call (import, K2, K3, stitch) and host-buffer GB/s.  Needs oracle/_ref (built by build()) and a GPU.

    python tests/bench_sequences.py [--mib 1024] [--iters 5]
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
import seqgen  # noqa: E402
import zref  # noqa: E402
import zstd_b200  # noqa: E402

SLICE = 32 << 20


def reference_sequences(src, level=1):
    R = seqgen.ref()
    R.ZSTD_generateSequences.restype = ctypes.c_size_t
    R.ZSTD_generateSequences.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t]
    R.ZSTD_sequenceBound.restype = ctypes.c_size_t
    R.ZSTD_sequenceBound.argtypes = [ctypes.c_size_t]
    parts = []
    for p in range(0, len(src), SLICE):
        chunk = src[p:p + SLICE]
        c = seqgen._cctx(R, [(seqgen.C_LEVEL, level)])
        out = np.zeros((R.ZSTD_sequenceBound(len(chunk)), 4), np.uint32)
        n = R.ZSTD_generateSequences(c, out.ctypes.data, len(out), chunk, len(chunk))
        R.ZSTD_freeCCtx(c)
        assert not R.ZSTD_isError(n), R.ZSTD_getErrorName(n)
        parts.append(out[:n])
    return np.ascontiguousarray(np.concatenate(parts))


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=1024)
    ap.add_argument("--iters", type=int, default=5)
    a = ap.parse_args()
    src = zref.datagen(a.mib << 20, 50, seed=0)
    t = time.time()
    seqs = reference_sequences(src)
    gen_s = time.time() - t
    n = len(src)
    d_src = torch.frombuffer(bytearray(src), dtype=torch.uint8).cuda()
    d_seq = torch.from_numpy(seqs.view(np.uint8).reshape(-1)).cuda()
    cap = zstd_b200.ZSTD_compressBound(n) + 3 * (n >> 10) + 4096
    d_dst = torch.empty(cap, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()

    def ctx():
        c = zstd_b200.ZSTD_CCtx()
        c.set_parameter("compression_level", 1)
        c.set_parameter(1008, 1)
        return c

    c = ctx()
    size = c.compress_sequences_device(d_dst.data_ptr(), cap, d_seq.data_ptr(), len(seqs), d_src.data_ptr(), n)     # warm-up
    times = []
    for _ in range(a.iters):
        torch.cuda.synchronize()
        t = time.perf_counter()
        r = c.compress_sequences_device(d_dst.data_ptr(), cap, d_seq.data_ptr(), len(seqs), d_src.data_ptr(), n)
        times.append(time.perf_counter() - t)                           # the call synchronises before it returns
        assert r == size
    frame = d_dst[:size].cpu().numpy().tobytes()
    assert zref.ref_decompress(frame, n) == src
    os.environ["ZSTDB200_SERIAL"] = "1"                                 # one wave: events around every kernel stage
    cs = ctx()
    cs.compress_sequences_device(d_dst.data_ptr(), cap, d_seq.data_ptr(), len(seqs), d_src.data_ptr(), n)
    split = []
    for _ in range(a.iters):
        assert cs.compress_sequences_device(d_dst.data_ptr(), cap, d_seq.data_ptr(), len(seqs), d_src.data_ptr(), n) == size
        s = cs.stats()
        split.append((s.match_ms, s.literals_ms, s.sequences_ms, s.stitch_ms, s.kernel_ms))
    del os.environ["ZSTDB200_SERIAL"]
    ch = ctx()
    host_t = []
    for _ in range(2):
        t = time.perf_counter()
        assert len(ch.compress_sequences(seqs, src)) == size
        host_t.append(time.perf_counter() - t)
    med = np.median(np.array(split), axis=0)
    gib = n / (1 << 30)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({
        "input": f"datagen P50, {a.mib} MiB", "sequences": int(len(seqs)), "reference_generate_s": round(gen_s, 1),
        "compressed": size, "ratio": round(n / size, 3),
        "device_GBps": round(n / np.median(times) / 1e9, 2), "device_ms": round(1e3 * float(np.median(times)), 2),
        "split_ms_per_GiB": {"import": round(med[0] / gib, 3), "literals": round(med[1] / gib, 3), "sequences": round(med[2] / gib, 3),
                             "stitch": round(med[3] / gib, 3), "kernels_total": round(med[4] / gib, 3)},
        "host_GBps": round(n / min(host_t) / 1e9, 2), "gpu": q}))


if __name__ == "__main__":
    main()
