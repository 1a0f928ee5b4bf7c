"""Edge cases of the candidate walk (K1a, zb_walk_kernel in zstd_b200/csrc/zb_match.cu), each compared with the oracle
frame: the first chunk of a frame (no priming), histories shorter than 128 KiB (a dictionary in front), frames that end
inside a batch and inside the last 8 bytes of a batch, raw and zstd-format dictionaries (the table primed from the
dictionary's image), levels with different insertion patterns (1, -3, -7: the acceleration divides the residue) and
level 3 (the doubleFast walks at 4 and at 1 position per thread).

The CPU test checks the walk's 32-bit hash (zb_hash32 in zb_device.cuh, three 32-bit multiply-adds) and its bucket
against the reference's 64-bit hash expressions on random inputs, for every minimum match length and table size."""
import os
import random
import subprocess

import pytest

import zref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "zstd_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else "nvcc")

HASH_CHECK = r"""
#include <cstdio>
#include <cstdlib>
#include "zb_device.cuh"
/* lib/compress/zstd_compress_internal.h:815-861 with hBits = 32 */
static u32 ref_hash(u64 v, int mls)
{
    switch (mls) {
    case 4: return (u32)v * 2654435761u;
    case 5: return (u32)(((v << 24) * 889523592379ull) >> 32);
    case 6: return (u32)(((v << 16) * 227718039650203ull) >> 32);
    case 7: return (u32)(((v << 8) * 58295818150454627ull) >> 32);
    default: return (u32)((v * 0xCF1BBCDCB7A56463ull) >> 32);
    }
}
template <int MLS> static u32 new_hash(u64 v) { return zb_hash32<MLS>((u32)v, (u32)(v >> 32)); }
int main(int argc, char** argv)
{
    u64 s = strtoull(argv[1], 0, 10) | 1;
    long bad = 0, n = 0;
    for (int a = 2; a < argc; a++) {
        u32 const N = (u32)strtoul(argv[a], 0, 10);
        for (int k = 0; k < 200000; k++) {
            s ^= s << 13; s ^= s >> 7; s ^= s << 17;                       /* xorshift64 */
            u64 const v = k < 64 ? (k < 32 ? 1ull << (2 * k) : ~(1ull << (2 * k - 64))) : s;
            for (int mls = 4; mls <= 8; mls++) {
                u32 const want = ref_hash(v, mls);
                u32 const got = mls == 4 ? new_hash<4>(v) : mls == 5 ? new_hash<5>(v) : mls == 6 ? new_hash<6>(v) : mls == 7 ? new_hash<7>(v) : new_hash<8>(v);
                if (got != want || zb_mulhi(got, N) != (u32)(((u64)want * N) >> 32)) bad++;
                n++;
            }
        }
    }
    printf("%ld of %ld differ\n", bad, n);
    return bad != 0;
}
"""


def table_sizes():
    """zb_makeParams (zb_api.cu): fast tables 3 << (hl - 2) and 7 << (hl - 3) for hash logs 6..14, doubleFast short
    tables 1 << chainLog capped at 28672 buckets, long tables 1 << hashLog up to 2^14."""
    sizes = {28672}
    for hl in range(6, 15):
        sizes |= {3 << (hl - 2), 7 << (hl - 3), 1 << hl}
    return sorted(sizes)


def test_hash32_equals_64bit_form(tmp_path):
    src = tmp_path / "hash_check.cu"
    src.write_text(HASH_CHECK)
    exe = tmp_path / "hash_check"
    subprocess.check_call([NVCC, "-std=c++17", "-I", CSRC, "-o", str(exe), str(src)])
    out = subprocess.run([str(exe), "12345"] + [str(n) for n in table_sizes()], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr


BATCH = 1024
CHUNK = 4 * (128 << 10)


def _frame_sizes():
    # one chunk (no priming), two chunks (the second primed from 128 KiB), ends inside a batch and inside its last 8 bytes
    return [CHUNK - 3, CHUNK + 5 * BATCH + 517, CHUNK + 7 * BATCH + BATCH - 5, CHUNK + 2 * BATCH + BATCH - 8, 2 * CHUNK + 1, 3 * BATCH + 7]


@pytest.mark.gpu
@pytest.mark.parametrize("level", [1, -3, -7, 3])
@pytest.mark.parametrize("size", _frame_sizes())
def test_walk_frame_edges(size, level):
    import zstd_b200
    src = zref.synthetic(size, 1000 + size % 97, 0.5)
    c = zstd_b200.ZSTD_CCtx()
    try:
        got = c.compress(src, level)
    finally:
        c.close()
    assert got == zref.oracle_compress(src, level)
    if zref.have_ref():
        assert zref.ref_decompress(got, len(src)) == src


@pytest.mark.gpu
@pytest.mark.parametrize("level", [1, -7, 3])
@pytest.mark.parametrize("dict_name", ["raw-20k", "zdict-16k-synthetic-seed77"])
def test_walk_dictionary_in_front(dict_name, level):
    """A dictionary in front: the first chunk's history is the dictionary tail (shorter than 128 KiB), walked from the
    dictionary bytes (usingDict) or primed from the table image (CDict)."""
    import zstd_b200
    d = zref.synthetic(20 << 10, 321, 0.5) if dict_name == "raw-20k" else zref.golden_input(dict_name)
    rnd = random.Random(level)
    srcs = [d[-3000:-1000] + zref.synthetic(CHUNK + 3 * BATCH + 5, 9, 0.5), zref.synthetic(BATCH + 3, 8, 0.5),
            d[-(8 << 10):] + zref.synthetic(2 * BATCH - 9, 7, 0.4), bytes(rnd.getrandbits(8) for _ in range(777))]
    c = zstd_b200.ZSTD_CCtx()
    cd = zstd_b200.ZSTD_CDict(d, level)
    try:
        for src in srcs:
            want = zref.oracle_compress_using_dict(src, d, level)
            assert c.compress_using_dict(src, d, level) == want
            assert c.compress_using_cdict(src, cd) == want
            if zref.have_ref():
                assert zref.ref_decompress_using_dict(want, d, len(src)) == src
    finally:
        cd.close()
        c.close()
