"""Batch decompression with the index in device memory, on one GPU: ZSTDB200_decompressFramesAsync (host arrays) against
ZSTDB200_decompressFramesAsync_deviceOffsets (the same values in device arrays) on the same bytes, and the size query
ZSTDB200_findDecompressedSizesAsync.  Shapes of tests/bench_decode_frames.py: 128 MiB of 1 KiB records and 1 GiB of 1 MiB
frames, datagen -P50 (synthetic data without it), level 1, frames from ZSTDB200_compressFrames.
   python tests/bench_decode_device_offsets.py
Per shape: the two calls alternated on the same context, each between CUDA events (plus a synchronise), best of 5, every
output and size checked; then, in runs of their own under torch.profiler, the check-and-pack kernel of the device-offset call
and the size-query kernel (both outputs).  Last, the size query on one 1 GiB frame of 8192 blocks as a single entry: one
thread follows its block headers, one dependent load per block.  The card's name and power limit are read in the same run."""
import ctypes, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch, zstd_b200
from bench_decode_frames import compressed, timed, walk_ms

SHAPES = (("128 MiB of 1 KiB records", 128 << 20, 1024), ("1 GiB of 1 MiB frames", 1 << 30, 1 << 20))


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(f"GPU: {q.stdout.strip() or torch.cuda.get_device_name()}", flush=True)
    dctx = zstd_b200.ZSTD_DCtx()
    L = zstd_b200.lib()
    res = torch.zeros(1, dtype=torch.int64, device="cuda")
    st = lambda: torch.cuda.current_stream().cuda_stream    # noqa: E731
    for name, n, fs in SHAPES:
        d_src, d_c, total, starts, cs, offs, sizes = compressed(n, fs)
        m = len(sizes)
        d_out = torch.empty(n, dtype=torch.uint8, device="cuda")
        d_sizes = torch.zeros(m, dtype=torch.int64, device="cuda")
        do, dc, so, ss = ((ctypes.c_size_t * m)(*a) for a in (offs, sizes, starts, cs))
        a_do, a_dc, a_so, a_ss = (torch.tensor(a, dtype=torch.int64, device="cuda") for a in (offs, sizes, starts, cs))
        cs_out, bd_out = torch.zeros(m, dtype=torch.int64, device="cuda"), torch.zeros(m, dtype=torch.int64, device="cuda")
        calls = {
            "host arrays": lambda: L.ZSTDB200_decompressFramesAsync(dctx._h, d_out.data_ptr(), n, do, dc, d_c.data_ptr(), total, so, ss, m,
                                                                    d_sizes.data_ptr(), res.data_ptr(), st()),
            "device offsets": lambda: L.ZSTDB200_decompressFramesAsync_deviceOffsets(dctx._h, d_out.data_ptr(), n, a_do.data_ptr(), a_dc.data_ptr(),
                                                                                   d_c.data_ptr(), total, a_so.data_ptr(), a_ss.data_ptr(), m,
                                                                                   d_sizes.data_ptr(), res.data_ptr(), st()),
        }
        query = lambda: L.ZSTDB200_findDecompressedSizesAsync(dctx._h, d_c.data_ptr(), total, a_so.data_ptr(), a_ss.data_ptr(), m,   # noqa: E731
                                                              cs_out.data_ptr(), bd_out.data_ptr(), st())
        for fn in calls.values():
            assert fn() == 0
        torch.cuda.synchronize()
        best = {k: [] for k in calls}
        ok = True
        want = torch.tensor(sizes, device="cuda")
        for _ in range(5):
            for k, fn in calls.items():
                d_out.zero_(); res.fill_(-1); d_sizes.zero_()
                best[k].append(timed(fn))
                ok &= torch.equal(d_out, d_src) and int(res.item()) == n and torch.equal(d_sizes, want)
        query(); torch.cuda.synchronize()
        ok &= torch.equal(cs_out, want) and torch.equal(bd_out, want)
        pack = walk_ms(calls["device offsets"], ("zbd_entries_pack_kernel",))
        qk = walk_ms(query, ("zbd_sizes_kernel",))
        fmt = lambda v: f"{min(v):.2f} (spread {min(v):.2f}-{max(v):.2f})"     # noqa: E731
        print(f"{name}: {m} frames, {total} B -> {n >> 20} MiB.  ms over 5 alternated runs: decompressFramesAsync "
              f"{fmt(best['host arrays'])}, decompressFramesAsync_deviceOffsets {fmt(best['device offsets'])}.  "
              f"check-and-pack kernel {pack * 1000:.1f} us, size-query kernel {qk * 1000:.1f} us.  ok {ok}", flush=True)
        del d_src, d_c, d_out
    d_src, d_c, total, starts, cs, offs, sizes = compressed(1 << 30, 1 << 30)
    one = torch.tensor([0, total], dtype=torch.int64, device="cuda")
    out = torch.zeros(2, dtype=torch.int64, device="cuda")
    q1 = lambda: L.ZSTDB200_findDecompressedSizesAsync(dctx._h, d_c.data_ptr(), total, one[0:].data_ptr(), one[1:].data_ptr(), 1,   # noqa: E731
                                                       out[0:].data_ptr(), out[1:].data_ptr(), st())
    q1(); torch.cuda.synchronize()
    ok = out.tolist() == [1 << 30, 1 << 30]
    t = min(timed(q1) for _ in range(5))
    print(f"one 1 GiB frame ({total} B, 8192 blocks) as one entry: size query (both outputs, two header walks) best of 5 "
          f"{t:.2f} ms, kernel {walk_ms(q1, ('zbd_sizes_kernel',)):.2f} ms.  ok {ok}", flush=True)


if __name__ == "__main__":
    main()
