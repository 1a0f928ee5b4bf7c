"""Time-bounded differential fuzz on a GPU box: random structured inputs, sizes clustered around the block / segment
boundaries, random levels, with and without dictionary — the GPU frame must equal the oracle's byte for byte.
   python tests/fuzz_gpu.py [seconds] [seed]"""
import os, sys, random, tempfile, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import zref, zstd_b200

budget = float(sys.argv[1]) if len(sys.argv) > 1 else 60.0
rng = random.Random(int(sys.argv[2]) if len(sys.argv) > 2 else 2024)
d = zref.golden_input("zdict-16k-synthetic-seed77")
ctx = zstd_b200.ZSTD_CCtx()
cd = {}


def gen():
    kind = rng.randrange(6)
    size = rng.choice([rng.randrange(0, 300), rng.randrange(0, 40000), rng.randrange(16000, 17000), rng.randrange(130000, 133000),
                       rng.randrange(0, 700000), rng.randrange(262100, 262200)])
    if kind == 0:
        return zref.synthetic(size, rng.randrange(1 << 30), rng.random())
    if kind == 1:
        return zref.random_bytes(size, rng.randrange(1 << 30))
    if kind == 2:
        return bytes([rng.randrange(256)]) * size
    if kind == 3:
        unit = zref.random_bytes(rng.randrange(1, 5000), rng.randrange(1 << 30))
        return (unit * (size // max(1, len(unit)) + 1))[:size]
    if kind == 4:
        a = zref.synthetic(size // 2 + 1, rng.randrange(1 << 30), 0.95)
        return (a + zref.random_bytes(size // 2 + 1, rng.randrange(1 << 30)) + a)[:size]
    return zref.synthetic(size, rng.randrange(1 << 30), 0.99)


t0, n, fails = time.time(), 0, 0
while time.time() - t0 < budget and fails < 3:
    src = gen()
    level = rng.choice([1, 2, 3, 4, -1, -3, -7, -50, 0, 9])
    mode = rng.randrange(4)
    if mode == 0:
        got, want = ctx.compress_using_dict(src, d, level), zref.oracle_compress_using_dict(src, d, level)
    elif mode == 1:
        if level not in cd:
            cd[level] = zstd_b200.ZSTD_CDict(d, level)
        got, want = ctx.compress_using_cdict(src, cd[level]), zref.oracle_compress_using_dict(src, d, level)
    else:
        got, want = ctx.compress(src, level), zref.oracle_compress(src, level)
    n += 1
    if got != want:
        fails += 1
        path = os.path.join(tempfile.gettempdir(), f"zb_fuzz_fail_{fails}.bin")
        open(path, "wb").write(src)
        print(f"MISMATCH size {len(src)} level {level} mode {mode}: gpu {len(got)} oracle {len(want)} -> {path}", flush=True)
print(f"fuzz: {n} cases in {time.time() - t0:.0f} s, {fails} mismatches")
sys.exit(1 if fails else 0)
