"""Kernel time per GiB of the level-1 compression path, split by kernel name with torch.profiler (CUDA activities).
bench.py's serial-mode `parse_ms` covers the fast parse (zb_parse_kernel) and the merge after it (zb_merge_segments_kernel)
together; this script reports them apart.

    python tests/parse_split.py [--mib 1024] [--p 50] [--level 1] [--iters 3] [--out DIR]

The input is config 2's: datagen -P50, seed 0 (zbo_synthetic when the datagen binary is absent).  One untimed call warms
up, then `iters` calls run under the profiler in serial mode (one wave on one stream).  Prints one JSON line: ms per GiB
per kernel (kernels of the same name summed, averaged over the calls) and the card it ran on."""
import argparse
import collections
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=1024)
    ap.add_argument("--p", type=int, default=50)
    ap.add_argument("--level", type=int, default=1)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--out", help="also write the JSON line to DIR/parse_split.json")
    args = ap.parse_args()
    os.environ["ZSTDB200_SERIAL"] = "1"
    import torch
    from torch.profiler import ProfilerActivity, profile
    import zref
    import zstd_b200
    if not torch.cuda.is_available():
        sys.exit("parse_split.py needs a CUDA device")
    n = args.mib << 20
    src = zref.datagen(n, args.p) if zref.have_datagen() else zref.synthetic(n, 0, args.p / 100)
    t = torch.frombuffer(bytearray(src), dtype=torch.uint8).cuda()
    cap = zstd_b200.ZSTD_compressBound(n)
    out = torch.empty(cap, dtype=torch.uint8, device="cuda")
    ctx = zstd_b200.ZSTD_CCtx()
    csize = ctx.compress_device(out.data_ptr(), cap, t.data_ptr(), n, args.level)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.iters):
            ctx.compress_device(out.data_ptr(), cap, t.data_ptr(), n, args.level)
        torch.cuda.synchronize()
    ctx.close()
    per = collections.defaultdict(float)
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            per[e.name.split("(")[0].split("<")[0].replace("void ", "")] += e.device_time_total / 1000.0
    gib = n / (1 << 30)
    ms = {k: round(v / args.iters / gib, 3) for k, v in sorted(per.items(), key=lambda kv: -kv[1])}
    res = {"ms_per_gib": ms, "bytes": n, "compressed_bytes": int(csize), "level": args.level, "iters": args.iters,
           "gpu": torch.cuda.get_device_name(0), "lib": zstd_b200.LIB_PATH}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "parse_split.json"), "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
