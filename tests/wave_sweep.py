"""Device-resident wave-executor sweep on one GPU (development tool, not the bench.py headline):
   python tests/wave_sweep.py [c2|c4] [iters]
For every (blocks per wave, waves in flight) combination: best / median total ms of
one call and a check that the output bytes equal the serial (one wave, one stream) output."""
import os, sys, statistics, zlib
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch, zref, zstd_b200


def one(d_src, n, level, env, iters):
    for k in ("ZSTDB200_SERIAL", "ZSTDB200_WAVE_BLOCKS", "ZSTDB200_WAVE_SLOTS"):
        os.environ.pop(k, None)
    os.environ.update(env)
    ctx = zstd_b200.ZSTD_CCtx()
    cap = zstd_b200.ZSTD_compressBound(n) + 32
    d_dst = torch.empty(cap, dtype=torch.uint8, device="cuda")
    ts = []
    for i in range(iters + 2):
        total = ctx.compress_device(d_dst.data_ptr(), cap, d_src.data_ptr(), n, level=level)
        if i >= 2:
            ts.append(ctx.stats().total_ms)
    crc = zlib.crc32(d_dst[:total].cpu().numpy().tobytes())
    ctx.close()
    return min(ts), statistics.median(ts), total, crc


def main():
    which = sys.argv[1] if len(sys.argv) > 1 else "c2"
    iters = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    G = 1 << 30
    src, level = (zref.datagen(G, 50), 1) if which == "c2" else (zref.datagen(G, 90), 3)
    d_src = torch.frombuffer(bytearray(src), dtype=torch.uint8).cuda()
    base = one(d_src, G, level, {"ZSTDB200_SERIAL": "1"}, iters)
    print(f"serial: best {base[0]:.2f} ms  median {base[1]:.2f} ms  {G/base[0]/1e6:.1f} GB/s  size {base[2]}", flush=True)
    for wb in (256, 512, 1024, 2048):
        for slots in (3, 4, 6, 8):
            r = one(d_src, G, level, {"ZSTDB200_WAVE_BLOCKS": str(wb), "ZSTDB200_WAVE_SLOTS": str(slots)}, iters)
            same = (r[2], r[3]) == (base[2], base[3])
            print(f"wave {wb:5d} slots {slots}: best {r[0]:.2f} ms  median {r[1]:.2f} ms  {G/r[0]/1e6:.1f} GB/s  same bytes: {same}", flush=True)


if __name__ == "__main__":
    main()
