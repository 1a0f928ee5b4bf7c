"""Stream-ordered decompression timing on one GPU (ZSTDB200_decompressDeviceAsync against ZSTDB200_decompressDevice), on
the shapes of tests/bench_decode.py.
   python tests/bench_decode_async.py [--parent PATH_TO_PARENT_libzstd_b200.so]
Per shape: the synchronous call, the stream-ordered call plus a synchronise (both between CUDA events, best of 5, same
output checked), and the walk kernel alone (torch.profiler, in a run of its own).  Then 256 calls of 1 MiB and of 16 MiB:
calls/s synchronous, queued back to back, and as graph replays.  With --parent, the walk kernel of that build and of this
one are timed alternately in child processes (the synchronous call with the walk forced onto the device)."""
import argparse, json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch, zref, zstd_b200

SHAPES = (("1 GiB P50 level-1 frame", 1 << 30, 1 << 30), ("1 GiB of 1 MiB frames", 1 << 30, 1 << 20),
          ("128 MiB of 1 KiB records", 128 << 20, 1024))


def compressed(n, fs):
    src = zref.datagen(n, 50) if zref.have_datagen() else zref.synthetic(n, 0, 0.5)
    d_src = torch.frombuffer(bytearray(src), dtype=torch.uint8).cuda()
    offs = list(range(0, n, fs)); sizes = [min(fs, n - o) for o in offs]
    cap = sum(zstd_b200.ZSTD_compressBound(x) + 32 for x in sizes)
    d_c = torch.empty(cap, dtype=torch.uint8, device="cuda")
    total, _ = zstd_b200.ZSTD_CCtx().compress_frames(d_c.data_ptr(), cap, d_src.data_ptr(), offs, sizes, level=1)
    return d_src, d_c, total


def timed(fn, reps=5):
    best = None
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize()
        best = e0.elapsed_time(e1) if best is None else min(best, e0.elapsed_time(e1))
    return best


def walk_ms(fn, reps=3):
    """the walk kernel's mean duration over reps calls, from torch.profiler"""
    fn(); torch.cuda.synchronize()
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    us = [e.device_time for e in prof.events() if "zbd_walk_kernel" in e.name]
    return sum(us) / len(us) / 1000.0 if us else float("nan")


def walk_child(shape):
    """child process: the synchronous call with the walk kernel (ZSTDB200_HOSTWALK_MAX=0) of the library in ZSTDB200_LIB"""
    name, n, fs = SHAPES[shape]
    d_src, d_c, total = compressed(n, fs)
    d = zstd_b200.ZSTD_DCtx()
    d_out = torch.empty(n, dtype=torch.uint8, device="cuda")
    ms = walk_ms(lambda: d.decompress_device(d_out.data_ptr(), n, d_c.data_ptr(), total))
    print(json.dumps({"walk_ms": ms, "ok": bool(torch.equal(d_out, d_src))}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", default=None)
    ap.add_argument("--walk-child", type=int, default=None)
    a = ap.parse_args()
    if a.walk_child is not None:
        return walk_child(a.walk_child)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(f"GPU: {q.stdout.strip() or torch.cuda.get_device_name()}", flush=True)
    sd, ad = zstd_b200.ZSTD_DCtx(), zstd_b200.ZSTD_DCtx()
    res = torch.zeros(1, dtype=torch.int64, device="cuda")
    for name, n, fs in SHAPES:
        d_src, d_c, total = compressed(n, fs)
        d_out = torch.empty(n, dtype=torch.uint8, device="cuda")
        sync = lambda: sd.decompress_device(d_out.data_ptr(), n, d_c.data_ptr(), total)    # noqa: E731
        asyn = lambda: ad.decompress_device_async(d_out.data_ptr(), n, d_c.data_ptr(), total, res.data_ptr(),    # noqa: E731
                                                  torch.cuda.current_stream().cuda_stream)
        sync(); asyn(); torch.cuda.synchronize()
        t_sync = timed(sync); ok_sync = torch.equal(d_out, d_src)
        d_out.zero_()
        t_async = timed(asyn); ok_async = torch.equal(d_out, d_src) and int(res.item()) == n
        w = walk_ms(asyn)
        print(f"{name}: {total} B -> {n >> 20} MiB  sync {t_sync:.2f} ms ({n / t_sync / 1e6:.1f} GB/s)  async {t_async:.2f} ms "
              f"({n / t_async / 1e6:.1f} GB/s)  walk kernel {w:.2f} ms  ok {ok_sync and ok_async}", flush=True)
        del d_src, d_c, d_out
    for mib in (1, 16):
        n, calls = mib << 20, 256
        d_src, d_c, total = compressed(n, n)
        d_out = torch.empty(n, dtype=torch.uint8, device="cuda")
        results = torch.zeros(calls, dtype=torch.int64, device="cuda")
        def run_sync():
            for _ in range(calls):
                sd.decompress_device(d_out.data_ptr(), n, d_c.data_ptr(), total)
        def run_async(stream):
            for i in range(calls):
                ad.decompress_device_async(d_out.data_ptr(), n, d_c.data_ptr(), total, results[i:].data_ptr(), stream)
        run_sync(); run_async(torch.cuda.current_stream().cuda_stream); torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            ad.decompress_device_async(d_out.data_ptr(), n, d_c.data_ptr(), total, results.data_ptr(), torch.cuda.current_stream().cuda_stream)
        rates = {}
        for what, fn in (("sync", run_sync), ("queued", lambda: run_async(torch.cuda.current_stream().cuda_stream)),
                         ("graph", lambda: [g.replay() for _ in range(calls)])):
            torch.cuda.synchronize(); t0 = time.perf_counter(); fn(); torch.cuda.synchronize()
            rates[what] = calls / (time.perf_counter() - t0)
        ok = bool((results == n).all()) and torch.equal(d_out, d_src)
        print(f"{calls} calls of {mib} MiB: sync {rates['sync']:.0f} calls/s, queued {rates['queued']:.0f}, graph {rates['graph']:.0f}  ok {ok}", flush=True)
        del g
    if a.parent:
        here = os.path.abspath(__file__)
        mine = os.path.join(os.path.dirname(os.path.dirname(here)), "zstd_b200", "libzstd_b200.so")
        for shape, (name, _, _) in enumerate(SHAPES):
            got = {"parent": [], "this": []}
            for _ in range(2):
                for who, path in (("parent", a.parent), ("this", mine)):
                    env = dict(os.environ, ZSTDB200_LIB=path, ZSTDB200_HOSTWALK_MAX="0")
                    out = subprocess.run([sys.executable, here, "--walk-child", str(shape)], env=env, capture_output=True, text=True)
                    r = json.loads(out.stdout.strip().splitlines()[-1]) if out.returncode == 0 else {"walk_ms": float("nan"), "ok": False}
                    got[who].append(f"{r['walk_ms']:.2f}{'' if r['ok'] else ' (wrong output)'}")
            print(f"walk kernel, {name}: parent {', '.join(got['parent'])} ms; this build {', '.join(got['this'])} ms", flush=True)


if __name__ == "__main__":
    main()
