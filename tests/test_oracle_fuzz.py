"""Seeded differential fuzz of the oracle against the reference decoder (CPU): structured random inputs whose sizes
cluster around the 16 KiB parse-segment and 128 KiB block boundaries, all level classes, with and without a zstd-format
dictionary.  Its GPU twin is tests/fuzz_gpu.py."""
import random

import pytest

import zref

needs_ref = pytest.mark.skipif(not zref.have_ref(), reason="oracle/_ref/libzstd_ref.so not built")


def make_input(rng):
    kind = rng.randrange(6)
    size = rng.choice([rng.randrange(0, 300), rng.randrange(0, 40000), rng.randrange(16000, 17000), rng.randrange(130000, 133000),
                       rng.randrange(0, 400000)])
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


@needs_ref
@pytest.mark.parametrize("seed", [1, 2, 3, 4])
def test_oracle_frames_decode(seed):
    rng = random.Random(seed)
    d = zref.golden_input("zdict-16k-synthetic-seed77")
    for _ in range(400):
        src = make_input(rng)
        level = rng.choice([1, 2, 3, 4, -1, -3, -7, -50, 0, 9])
        if rng.random() < 0.25:
            frame = zref.oracle_compress_using_dict(src, d, level)
            assert zref.ref_decompress_using_dict(frame, d, len(src)) == src, (len(src), level)
        else:
            frame = zref.oracle_compress(src, level)
            assert zref.ref_decompress(frame, len(src)) == src, (len(src), level)
