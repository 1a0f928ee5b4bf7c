"""Paths of the fast greedy parse (K1b, zb_parse_kernel in zstd_b200/csrc/zb_match.cu), each compared whole-frame with the
oracle and decoded with the reference decoder.  The inputs are built from copy operations chosen to reach:
- table candidates at distances >= 0xFFFF (`far`, fetched only for the lane being tried) that win, and that lose to a
  lower lane with a near candidate or a repcode;
- tag false positives (random bytes: bucket collisions with equal 11-bit tags) in front of a real hit at a higher lane;
- repcode-2 right after a match; repcode-1 hits whose catch-up runs past 4 and past 32 bytes, and catch-up stopped by
  the anchor (copies that follow a copy without literals);
- matches longer than one 256-byte forward round, matches that end within 8 bytes of a block's end and matches that run
  past a segment's end (copies across 16 KiB and 128 KiB borders);
- the step sizes of levels 1, -1, -3 and -7, with and without a dictionary in front."""
import random

import pytest

import zref

SEG = 16 << 10
BLOCK = 128 << 10


def mixed(n: int, seed: int) -> bytes:
    rnd = random.Random(seed)
    out = bytearray(rnd.randbytes(256))
    reps = [1, 4, 8]
    while len(out) < n:
        op = rnd.random()
        if op < 0.22:                                             # literals, from one byte to a run that defeats the step
            out += rnd.randbytes(rnd.choice([1, 2, 5, 9, 31, 200, 700]))
            continue
        length = rnd.choice([4, 5, 7, 8, 12, 33, 64, 100, 255, 256, 257, 300, 1100])
        if op < 0.40:
            off = rnd.randint(1, min(len(out), 3000))             # near
        elif op < 0.55 and len(out) > 0x10000 + 64:
            off = rnd.randint(0xFFFF - 32, min(len(out), 0x1F000))  # far: the walk stores it in the far array
        elif op < 0.70:
            off = reps[0]                                         # repcode 1, often with matching bytes in front
            out += rnd.randbytes(rnd.choice([0, 1, 3]))
            if rnd.random() < 0.5:                                # catch-up: the copy starts before the literal gap
                for _ in range(rnd.choice([5, 6, 40])):
                    out.append(out[-off])
        elif op < 0.82:
            off = reps[1]                                         # repcode 2 right after the previous copy
        else:
            off = rnd.randint(1, min(len(out), 600))
            length = rnd.randint(300, 3 * SEG // 2)                # long: several forward rounds, across a segment end
        off = min(off, len(out))
        if off >= length:
            out += out[len(out) - off:len(out) - off + length]
        else:
            for _ in range(length):
                out.append(out[-off])
        if off != reps[0]:
            reps = [off, reps[0], reps[1]] if off != reps[1] else [off, reps[0], reps[2]]
    return bytes(out[:n])


def _sizes():
    # ends inside the last 8 bytes of a block, a block plus a few segments, two chunks (history primed), one segment
    return [3 * BLOCK - 5, BLOCK + 3 * SEG + 7, 4 * BLOCK + 2 * BLOCK + 3, SEG - 1]


@pytest.mark.gpu
@pytest.mark.parametrize("level", [1, -1, -3, -7])
@pytest.mark.parametrize("size", _sizes())
def test_parse_paths_frame(size, level):
    import zstd_b200
    src = mixed(size, 17 + size % 89 + level)
    c = zstd_b200.ZSTD_CCtx()
    try:
        got = c.compress(src, level)
    finally:
        c.close()
    assert got == zref.oracle_compress(src, level)
    if zref.have_ref():
        assert zref.ref_decompress(got, len(src)) == src


@pytest.mark.gpu
@pytest.mark.parametrize("level", [1, -3])
def test_parse_paths_behind_dictionary(level):
    """The DICT instantiation: matches into the dictionary, far ones included, and across the dictionary / frame border."""
    import zstd_b200
    d = mixed(100 << 10, 5)
    srcs = [d[-0x11000:-0x10000] + mixed(BLOCK + SEG + 9, 6), d[-5000:] + d[:3000] + mixed(20000, 7), mixed(SEG + 3, 8)]
    c = zstd_b200.ZSTD_CCtx()
    try:
        for src in srcs:
            want = zref.oracle_compress_using_dict(src, d, level)
            assert c.compress_using_dict(src, d, level) == want
            if zref.have_ref():
                assert zref.ref_decompress_using_dict(want, d, len(src)) == src
    finally:
        c.close()


def test_mixed_generator_reaches_far_and_long_copies():
    """CPU check of the generator itself: the inputs above do hold far repeats and long ones."""
    src = mixed(3 * BLOCK, 1)
    far = sum(1 for i in range(0x10000 + 4096, len(src) - 16, 4096) if src[i:i + 16] in src[:i - 0xFFFF])
    assert far > 0
    assert len(src) == 3 * BLOCK
