"""Batch decompression timing on one GPU (ZSTDB200_decompressFrames[Async] against ZSTDB200_decompressDevice[Async] on the
same bytes), on the record shapes of tests/bench_decode_async.py: 128 MiB of 1 KiB records and 1 GiB of 1 MiB frames, datagen
-P50 (synthetic data without it), level 1, frames from ZSTDB200_compressFrames; and one 1 GiB frame as a single entry.
   python tests/bench_decode_frames.py
Per shape: the four calls alternated, each between CUDA events (the stream-ordered ones plus a synchronise), best of 5,
every output and size checked, the batch calls made through the C ABI with their host arrays built beforehand; then, in a
run of its own under torch.profiler, the header walk of the batch call (its count, scan and fill kernels) and of the single
stream-ordered call (its one-thread walk kernel).  The card's name and power limit are read in the same run."""
import ctypes, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch, zref, zstd_b200

SHAPES = (("128 MiB of 1 KiB records", 128 << 20, 1024), ("1 GiB of 1 MiB frames", 1 << 30, 1 << 20),
          ("one 1 GiB frame", 1 << 30, 1 << 30))      # one entry: one thread walks all its headers, twice
WALK = {"batch": ("zbd_entries_count_kernel", "zbd_entries_scan_kernel", "zbd_entries_fill_kernel"), "single": ("zbd_walk_kernel",)}


def compressed(n, fs):
    src = zref.datagen(n, 50) if zref.have_datagen() else zref.synthetic(n, 0, 0.5)
    d_src = torch.frombuffer(bytearray(src), dtype=torch.uint8).cuda()
    offs = list(range(0, n, fs)); sizes = [min(fs, n - o) for o in offs]
    cap = sum(zstd_b200.ZSTD_compressBound(x) + 32 for x in sizes)
    d_c = torch.empty(cap, dtype=torch.uint8, device="cuda")
    total, cs = zstd_b200.ZSTD_CCtx().compress_frames(d_c.data_ptr(), cap, d_src.data_ptr(), offs, sizes, level=1)
    starts = [0] * len(cs)
    for i in range(1, len(cs)):
        starts[i] = starts[i - 1] + cs[i - 1]
    return d_src, d_c, total, starts, cs, offs, sizes


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); fn(); e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def walk_ms(fn, names, reps=3):
    """the walk's kernels' summed mean duration over reps calls, from torch.profiler"""
    fn(); torch.cuda.synchronize()
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    us = [e.device_time for e in prof.events() if any(k in e.name for k in names)]
    return sum(us) / reps / 1000.0 if us else float("nan")


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(f"GPU: {q.stdout.strip() or torch.cuda.get_device_name()}", flush=True)
    ctx = {k: zstd_b200.ZSTD_DCtx() for k in ("device", "device_async", "frames", "frames_async")}
    res = torch.zeros(1, dtype=torch.int64, device="cuda")
    for name, n, fs in SHAPES:
        d_src, d_c, total, starts, cs, offs, sizes = compressed(n, fs)
        d_out = torch.empty(n, dtype=torch.uint8, device="cuda")
        d_sizes = torch.zeros(len(sizes), dtype=torch.int64, device="cuda")
        st = lambda: torch.cuda.current_stream().cuda_stream    # noqa: E731
        # the batch calls as a C caller makes them: the host arrays exist before the call (building them from Python lists
        # takes longer than the call itself on the record shape)
        L, m = zstd_b200.lib(), len(sizes)
        do, dc, so, ss, per = ((ctypes.c_size_t * m)(*a) for a in (offs, sizes, starts, cs, [0] * m))
        calls = {
            "device": lambda: ctx["device"].decompress_device(d_out.data_ptr(), n, d_c.data_ptr(), total),
            "device_async": lambda: ctx["device_async"].decompress_device_async(d_out.data_ptr(), n, d_c.data_ptr(), total, res.data_ptr(), st()),
            "frames": lambda: L.ZSTDB200_decompressFrames(ctx["frames"]._h, d_out.data_ptr(), n, do, dc, d_c.data_ptr(), total, so, ss, m, per, None),
            "frames_async": lambda: L.ZSTDB200_decompressFramesAsync(ctx["frames_async"]._h, d_out.data_ptr(), n, do, dc, d_c.data_ptr(), total, so, ss, m,
                                                                     d_sizes.data_ptr(), res.data_ptr(), st()),
        }
        for fn in calls.values():
            fn()
        torch.cuda.synchronize()
        best = {k: float("inf") for k in calls}
        ok = True
        for _ in range(5):
            for k, fn in calls.items():
                d_out.zero_(); res.fill_(-1)
                best[k] = min(best[k], timed(fn))
                ok &= torch.equal(d_out, d_src) and (k not in ("device_async", "frames_async") or int(res.item()) == n)
        ok &= bool((d_sizes == torch.tensor(sizes, device="cuda")).all()) and list(per) == sizes
        walk = {"batch": walk_ms(calls["frames_async"], WALK["batch"]), "single": walk_ms(calls["device_async"], WALK["single"])}
        print(f"{name}: {len(sizes)} frames, {total} B -> {n >> 20} MiB.  best of 5, ms: decompressDevice {best['device']:.2f}, "
              f"decompressDeviceAsync {best['device_async']:.2f}, decompressFrames {best['frames']:.2f}, "
              f"decompressFramesAsync {best['frames_async']:.2f}.  walk: batch (count + scan + fill) {walk['batch']:.2f} ms, "
              f"single-input stream-ordered {walk['single']:.2f} ms.  ok {ok}", flush=True)
        del d_src, d_c, d_out


if __name__ == "__main__":
    main()
