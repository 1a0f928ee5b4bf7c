"""Batch decompression with a dictionary per entry (ZSTDB200_decompressFrames_usingDDicts) on config 5's records: 1 KiB
records of datagen -P50 and its 16 KiB dictionary, written by ZSTDB200_compressFrames_usingCDicts at level 1 under K = 1,
16, 256 and 4096 dictIDs (bench_cdicts.with_id), on device buffers.  --scale 0.125 (the default) is 128 MiB of records,
the record shape of tests/bench_decode_frames.py.  Per K, one JSON line:
  wall_ms, gbps          the call between CUDA events on the context's stream, best of --steps; GB/s of output
  launches               ZSTDB200_getLastDStats after it
  first_use_ms           the first call with K fresh DDicts (host clock; the uploads and their one synchronisation)
  grouped_ms             what a caller without the call does: the entries grouped by dictionary, ZSTD_DCtx_refDDict and one
                         ZSTDB200_decompressFrames per group, between CUDA events, best of --steps
  sticky_ms              K = 1 only: ZSTDB200_decompressFrames with the one DDict as sticky dictionary, alternated with the
                         new call (every sample of both listed)
Every output is checked against the records.  The batch calls go through the C ABI with their host arrays built beforehand.
The card's name and power limit are read in the same run.
    python tests/bench_decode_ddicts.py [--scale 0.125] [--steps 5] [--ks 1,16,256,4096]"""
import argparse
import ctypes
import json
import os
import sys
import time

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import zstd_b200  # noqa: E402
from bench import Workload  # noqa: E402
from bench_cdicts import card, with_id  # noqa: E402

_sz = ctypes.c_size_t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=0.125)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--ks", default="1,16,256,4096")
    a = ap.parse_args()
    import torch
    print(json.dumps({"card": card()}), flush=True)
    wl = Workload(5, 0, 1, a.scale)
    src, d = wl.src, wl.dict
    n = len(wl.frames)
    offs, sizes = [o for o, _ in wl.frames], [s for _, s in wl.frames]
    cap = sum(zstd_b200.ZSTD_compressBound(s) + 32 for s in sizes)
    d_src = torch.frombuffer(bytearray(src), dtype=torch.uint8).cuda()
    d_c = torch.empty(cap, dtype=torch.uint8, device="cuda")
    d_out = torch.empty(len(src), dtype=torch.uint8, device="cuda")
    L = zstd_b200.lib()
    st = torch.cuda.Stream()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def events(fn):
        torch.cuda.synchronize()
        ev0.record(st)
        fn()
        ev1.record(st)
        torch.cuda.synchronize()
        return ev0.elapsed_time(ev1)

    cctx = zstd_b200.ZSTD_CCtx()
    for k in [int(x) for x in a.ks.split(",")]:
        dicts = [with_id(d, 1 + i) for i in range(k)]
        cds = [zstd_b200.ZSTD_CDict(x, wl.level) for x in dicts]
        total, cs = cctx.compress_frames_using_cdicts(d_c.data_ptr(), cap, d_src.data_ptr(), offs, sizes,
                                                      [cds[i % k] for i in range(n)], level=wl.level)
        so = [0] * n
        for i in range(1, n):
            so[i] = so[i - 1] + cs[i - 1]
        A = lambda v: (_sz * len(v))(*v)                                # noqa: E731
        c_do, c_dc, c_so, c_ss, c_sizes = A(offs), A(sizes), A(so), A(cs), (_sz * n)()

        def check():
            assert bool(torch.equal(d_out, d_src)), "output differs from the records"

        def new_call(ctx, dds):
            arr = (ctypes.c_void_p * n)(*[dds[i % k]._h for i in range(n)])

            def go():
                r = L.ZSTDB200_decompressFrames_usingDDicts(ctx._h, d_out.data_ptr(), len(src), c_do, c_dc, d_c.data_ptr(), total, c_so, c_ss,
                                                            n, arr, c_sizes, st.cuda_stream)
                assert r == len(src), zstd_b200.result_error(r)
            return go

        dctx = zstd_b200.ZSTD_DCtx()
        warm = [zstd_b200.ZSTD_DDict(x) for x in dicts]
        new_call(dctx, warm)()                                         # sizes the context
        fresh = [zstd_b200.ZSTD_DDict(x) for x in dicts]
        d_out.zero_()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        new_call(dctx, fresh)()
        first_ms = (time.perf_counter() - t0) * 1e3
        check()
        go = new_call(dctx, fresh)
        new_ms = []
        sticky_ms = []
        for _ in range(a.steps):
            d_out.zero_()
            new_ms.append(events(go))
            check()
            launches = dctx.stats().launches
            if k == 1:                                                 # the existing call on the same bytes, alternated
                dctx.ref_ddict(fresh[0])
                d_out.zero_()
                sticky_ms.append(events(lambda: L.ZSTDB200_decompressFrames(dctx._h, d_out.data_ptr(), len(src), c_do, c_dc, d_c.data_ptr(),
                                                                            total, c_so, c_ss, n, c_sizes, st.cuda_stream)))
                check()
                dctx.ref_ddict(None)
        # the grouped workaround: entries of one dictionary per call
        groups = []
        for g in range(k):
            idx = list(range(g, n, k))
            groups.append((fresh[g], len(idx), A([offs[i] for i in idx]), A([sizes[i] for i in idx]), A([so[i] for i in idx]),
                           A([cs[i] for i in idx]), (_sz * len(idx))()))

        def grouped():
            for dd, m, g_do, g_dc, g_so, g_ss, g_sizes in groups:
                L.ZSTD_DCtx_refDDict(dctx._h, dd._h)
                r = L.ZSTDB200_decompressFrames(dctx._h, d_out.data_ptr(), len(src), g_do, g_dc, d_c.data_ptr(), total, g_so, g_ss, m,
                                                g_sizes, st.cuda_stream)
                assert not zstd_b200.result_error(r), zstd_b200.result_error(r)
        grouped_ms = []
        for _ in range(a.steps):
            d_out.zero_()
            grouped_ms.append(events(grouped))
            check()
        best = min(new_ms)
        out = {"k": k, "records": n, "wall_ms": round(best, 3), "gbps": round(len(src) / best / 1e6, 2), "launches": launches,
               "samples_ms": [round(x, 3) for x in new_ms], "first_use_ms": round(first_ms, 2),
               "grouped_ms": round(min(grouped_ms), 3), "grouped_calls": k}
        if k == 1:
            out["sticky_ms"] = round(min(sticky_ms), 3)
            out["sticky_samples_ms"] = [round(x, 3) for x in sticky_ms]
        print(json.dumps(out), flush=True)
        for x in warm + fresh + cds:
            x.close()
        dctx.close()


if __name__ == "__main__":
    main()
