"""The candidate walk (K1a, zb_walk_kernel in zstd_b200/csrc/zb_match.cu) position by position against the oracle, and
through whole frames.

Position by position: tests/walk_harness.cu runs the product's zb_launch_walk alone and returns the whole dist and far
arrays and the dictionary images.  tests/walkgen.py restates the oracle's walk batch by batch; the CPU tests prove it
equal to zbo_walkChunk, show that its inputs reach every path and that each wrong-rule switch changes some distance.  The
GPU tests hold every launch to the oracle at every position: every parameter set the planner yields, the tables no
product call uses (1 position per thread: the product's tables all take 8 or 4), every dictionary tail length and chunk
geometry, images built by zb_launch_dict_images against the restatement's tables word by word, and every word the walk
must not write.

Through frames: the first chunk of a frame (no priming), histories shorter than 128 KiB (a dictionary in front), frames
that end inside a batch and inside the last 8 bytes of a batch, raw and zstd-format dictionaries (the table primed from
the dictionary's image), levels with different insertion patterns (1, -3, -7: the acceleration divides the residue) and
level 3 (the doubleFast walks of its two tables, both at 4 positions per thread).

The CPU test checks the walk's 32-bit hash (zb_hash32 in zb_device.cuh, three 32-bit multiply-adds) and its bucket
against the reference's 64-bit hash expressions on random inputs, for every minimum match length and table size."""
import os
import random
import subprocess

import numpy as np
import pytest

import walkgen as W
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


# ------------------------------------------------------------------------------------------- position by position
HARNESS = os.path.join(ROOT, "tests", "_build", "libzb_walk_harness.so")
SENT = (0xA5, 0x3C)
GUARD = 64
_H = None


def _harness():
    global _H
    if _H is None:
        import ctypes
        H = ctypes.CDLL(HARNESS)
        H.zbh_walk.restype = ctypes.c_int
        vp, u64 = ctypes.c_void_p, ctypes.c_uint64
        H.zbh_walk.argtypes = [vp, u64, vp, vp, vp, ctypes.c_uint32, vp, u64, vp, vp, vp, vp, vp, vp, u64, vp, u64, vp]
        _H = H
    return _H


class Frame:
    """one frame of a launch: its dictionary tail (b"" = none), its bytes and its block size 1 << block_log"""
    def __init__(self, tail: bytes, data: bytes, block_log: int = 17):
        self.tail, self.data, self.block_log = tail, data, block_log

    def blocks(self):
        b = 1 << self.block_log
        return [min(b, len(self.data) - p) for p in range(0, max(1, len(self.data)), b)]


def gpu_walk(frames, mls, N, ins, image=False, image_off=0, mls_short=0, slot=0):
    """one harness launch, run twice (sentinels SENT): dist (2, rows, stride) u16, far (2, rows, stride) u32, image (2, frames,
    GUARD + image_off + N + GUARD) u32 or None"""
    src, offs = bytearray(), []
    for i, f in enumerate(frames):
        src += bytes(1 + i % 3)                                  # the frames start at every alignment
        offs.append(len(src))
        src += f.data
    tails, toffs = bytearray(), []
    for f in frames:
        toffs.append(len(tails))
        tails += f.tail
    nb = len(frames)
    rows = sum(len(f.blocks()) for f in frames)
    stride = (max(64, max(max(f.blocks()) for f in frames)) + 63) & ~63      # zb_strides of the largest block
    words = GUARD + image_off + N + GUARD
    dist = np.zeros((2, rows, stride), np.uint16)
    far = np.zeros((2, rows, stride), np.uint32)
    img = np.zeros((2, nb, words), np.uint32) if image else np.zeros(1, np.uint32)
    shape = np.zeros(2, np.uint64)
    a64 = lambda v: np.array(v, np.uint64)
    a32 = lambda v: np.array(v, np.uint32)
    fo, fs, fb, to, tl = a64(offs), a32([len(f.data) for f in frames]), a32([f.block_log for f in frames]), a64(toffs), a32([len(f.tail) for f in frames])
    prm = a32([mls, N, ins, image_off, int(image), mls_short, slot])
    sent = np.array(SENT, np.uint8)
    srcb, tailb = bytes(src) or b"\0", bytes(tails) or b"\0"
    r = _harness().zbh_walk(srcb, len(src), fo.ctypes.data, fs.ctypes.data, fb.ctypes.data, nb, tailb, len(tails), to.ctypes.data,
                            tl.ctypes.data, prm.ctypes.data, sent.ctypes.data, dist.ctypes.data, far.ctypes.data, dist.size,
                            img.ctypes.data, img.size if image else 0, shape.ctypes.data)
    assert r == 0, f"harness returned {r}"
    assert tuple(shape) == (rows, stride)
    return dist, far, (img if image else None)


def oracle_frame(pl, f: Frame, long_table=False):
    """the oracle's distances over the whole frame, chunk by chunk"""
    out = [W.oracle_walk(pl, f.tail, f.data, pos, size)[1 if long_table else 0] for pos, size in W.chunk_bounds(len(f.data), f.block_log)]
    return np.concatenate(out) if out else np.zeros(0, np.uint32)


def check_launch(frames, s, long_table=False, image=False, slot=0):
    """one launch of set s against the oracle at every position, every word it must not write, and (image) every image word
    against the restatement's table"""
    strategy, mls, N, NL, ins = s
    pl = W.plan_for(s)
    wm, wn = (8, NL) if long_table else (mls, N)
    off = N if long_table else 0
    dist, far, img = gpu_walk(frames, wm, wn, ins, image=image, image_off=off if image else (N if long_table else 0),
                              mls_short=mls if long_table else 0, slot=slot)
    s16 = [int(b) * 0x0101 for b in SENT]
    s32 = [int(b) * 0x01010101 for b in SENT]
    row = 0
    got_runs = []
    for f in frames:
        want = oracle_frame(pl, f, long_table)
        pos = 0
        for bsz in f.blocks():
            for r in range(2):
                d16 = dist[r, row, :bsz].astype(np.int64)
                fr = far[r, row, :bsz].astype(np.int64)
                got = np.where(d16 == W.FAR, fr, d16)
                bad = np.nonzero(got != want[pos:pos + bsz])[0]
                assert bad.size == 0, (f"set {s} long={long_table} image={image}: block row {row} position {bad[0]}: "
                                       f"walk {got[bad[0]]}, oracle {want[pos + bad[0]]} ({bad.size} differ)")
                assert np.all(fr[d16 != W.FAR] == s32[r]), f"far written where dist is not ZB_FAR (row {row})"
                assert np.all(dist[r, row, bsz:] == s16[r]) and np.all(far[r, row, bsz:] == s32[r]), f"row {row} written past its block"
                got_runs.append(got)
            assert np.array_equal(got_runs[-1], got_runs[-2])
            pos += bsz
            row += 1
    if image:
        for k, f in enumerate(frames):
            for r in range(2):
                w = img[r, k]
                if not f.tail:
                    assert np.all(w == s32[r]), "an image written for a frame without a dictionary"
                    continue
                assert np.all(w[:GUARD] == s32[r]) and np.all(w[GUARD + off + wn:] == s32[r]), "image guard written"
                if long_table:
                    want_s = W.image_table(mls, N, ins, f.tail).astype(np.uint32)
                    assert np.array_equal(w[GUARD:GUARD + N], want_s), "short table image differs from the restatement"
                want_t = W.image_table(wm, wn, ins, f.tail).astype(np.uint32)
                assert np.array_equal(w[GUARD + off:GUARD + off + wn], want_t), "table image differs from the restatement"


DICT_LENS = (0, 1, 1023, 1024, 1025, (8 << 10) - 3, 128 << 10)
SMALL_SIZES = tuple(range(1, 17)) + (1023, 1024, 1025)
_INPUTS = {}


def launches(mls):
    """the geometry launches of one mls: (name, frames, slotFirstBlock)"""
    if mls in _INPUTS:
        return _INPUTS[mls]
    tail = lambda n, seed: W.walk_input(n, seed, mls)
    out = []
    dicts = []
    for i, D in enumerate(DICT_LENS):                            # every dictionary tail length in front of a first chunk
        t = tail(D, 100 + i) if D else b""
        dicts.append(Frame(t, W.walk_input(70000 + 333 * i, 200 + i, mls, t)))
    out.append(("dict_tails", dicts, 0))
    t = tail(1025, 7)
    smalls = [Frame(b"", W.walk_input(n, 300 + n, mls)) for n in SMALL_SIZES]
    smalls += [Frame(t, W.walk_input(n, 400 + n, mls, t)) for n in (1, 7, 8, 9, 1023, 1025)]
    out.append(("small_chunks", smalls, 0))
    out.append(("small_chunks_slot5", smalls[::3], 5))
    big = [Frame(b"", W.walk_input((512 << 10) - 5, 500, mls)), Frame(b"", W.walk_input(512 << 10, 501, mls)),
           Frame(b"", W.walk_input((1 << 20) + 1025, 502, mls))]     # one chunk, and later chunks behind 128 KiB of history
    out.append(("big_chunks", big, 0))
    wl = [Frame(b"", W.walk_input((9 << bl) + 777, 600 + bl, mls), bl) for bl in range(10, 17)]   # windowLog 10-16: short histories
    out.append(("block_sizes", wl, 3))
    out.append(("far_max", [Frame(b"", W.far_max_input(mls))], 0))
    out.append(("incompressible", [Frame(b"", W.incompressible((1 << 20) + 3, 700 + mls)), Frame(tail(8000, 8), W.incompressible(300000, 701))], 0))
    _INPUTS[mls] = out
    return out


def product_set(level, size=1 << 20):
    pl = W.make_plan(W.oracle_cparams(level, size, 0))
    return (pl.strategy, pl.mls, pl.tableN, pl.tableNLong if pl.strategy == 2 else 0, pl.insStep)


def geometry_sets():
    """the sets every geometry launch runs: fast levels 1 and -7 (insertion step 6: the division), doubleFast level 3 (both
    tables), and the harness-only tables at 1 position per thread with every mls, and insertion steps 1024 and 1025"""
    out = [("L1", product_set(1), False), ("Lm7", product_set(-7), False), ("L3s", product_set(3), False), ("L3l", product_set(3), True)]
    for mls in range(4, 9):
        out.append((f"P1_m{mls}", (1, mls, W.N_MAX if mls % 2 else 40000, 0, 3), False))
    out += [("ins1024", (1, 5, 12345, 0, 1024), False), ("ins1025", (1, 4, 28929, 0, 1025), False), ("ins1", (1, 7, 14336, 0, 1), False)]
    return out


def _restated(s, long_table, f: Frame, cnt=None, sw=frozenset()):
    strategy, mls, N, NL, ins = s
    wm, wn = (8, NL) if long_table else (mls, N)
    return np.concatenate([W.walk_chunk(wm, wn, ins, f.tail, f.data, pos, size, sw, cnt)[0]
                           for pos, size in W.chunk_bounds(len(f.data), f.block_log)])


# the CPU cases: the geometry launches of levels 1 and 3 and of two harness-only sets
CPU_SETS = [g for g in geometry_sets() if g[0] in ("L1", "L3s", "L3l", "P1_m7", "ins1025")]
_COUNTS = {}


def _cpu_counts():
    """restatement == zbo_walkChunk at every position of every CPU case; path, zero-row and batch-kind counts over them"""
    if _COUNTS:
        return _COUNTS
    cnt = {r: 0 for r in W.ROWS + W.ZERO_ROWS}
    kinds = {r: 0 for r in W.KIND_ROWS}
    positions = 0
    for name, s, long_table in CPU_SETS:
        pl = W.plan_for(s)
        N = s[3] if long_table else s[2]
        for lname, frames, _ in launches(s[1]):
            for f in frames:
                want = oracle_frame(pl, f, long_table)
                got = _restated(s, long_table, f, cnt)
                bad = np.nonzero(got != want)[0]
                assert bad.size == 0, f"{name}/{lname}: restatement {got[bad[0]]}, oracle {want[bad[0]]} at {bad[0]} ({bad.size} differ)"
                positions += len(want)
                for pos, size in W.chunk_bounds(len(f.data), f.block_log):
                    D = len(f.tail) if pos == 0 else 0
                    H = D if pos == 0 else min(pos, W.PRIME)
                    for image in ((False, True) if D else (False,)):
                        W.batch_kinds(N, D, H, size, image, cnt=kinds)
    _COUNTS.update(cnt=cnt, kinds=kinds, positions=positions)
    return _COUNTS


def test_restatement_equals_oracle_walk():
    c = _cpu_counts()
    print(f"\nrestatement == zbo_walkChunk at {c['positions']} positions")


def test_every_path_reached():
    c = _cpu_counts()
    print("\npaths:", c["cnt"], "\nbatch kinds:", c["kinds"])
    missing = [r for r in W.ROWS if c["cnt"][r] == 0] + [r for r in W.KIND_ROWS if c["kinds"][r] == 0]
    assert not missing, f"paths never reached: {missing}"


def test_rows_that_must_stay_zero():
    c = _cpu_counts()
    assert {r: c["cnt"][r] for r in W.ZERO_ROWS} == {r: 0 for r in W.ZERO_ROWS}


def test_every_switch_changes_a_distance():
    """each wrong rule changes some position's distance on the cases of level 1 and level 3's short table"""
    changed = {k: 0 for k in W.SWITCHES}
    for name, s, long_table in CPU_SETS[:2]:
        for lname, frames, _ in launches(s[1]):
            if lname in ("big_chunks", "incompressible"):
                continue
            for f in frames:
                base = _restated(s, long_table, f)
                for k in W.SWITCHES:
                    changed[k] += int(np.count_nonzero(_restated(s, long_table, f, sw=frozenset([k])) != base))
    print("\npositions changed per switch:", changed)
    assert all(changed.values()), f"switches that change nothing: {[k for k, v in changed.items() if not v]}"


def test_inputs_deterministic():
    a = [W.walk_input(70000, 5, m, b"x" * 1025) for m in (4, 8)]
    assert a == [W.walk_input(70000, 5, m, b"x" * 1025) for m in (4, 8)]
    assert W.far_max_input(6) == W.far_max_input(6) and W.incompressible(999, 1) == W.incompressible(999, 1)


def test_parameter_sets():
    """the product's tables take 8 or 4 positions per thread, never 1; the harness-only sets reach 1 and both edges of 4"""
    ps = W.product_sets()
    assert {W.threads_p(N) for _, _, N, NL, _ in ps} | {W.threads_p(NL) for _, _, _, NL, _ in ps if NL} == {8, 4}
    hs = W.harness_sets()
    assert {W.threads_p(N) for _, _, N, _, _ in hs} == {8, 4, 1}
    assert {1023, 1024, 1025} <= {s[4] for s in ps} and max(s[4] for s in ps) == -W.MIN_CLEVEL


@pytest.mark.gpu
@pytest.mark.parametrize("name,s,long_table", geometry_sets(), ids=[g[0] for g in geometry_sets()])
def test_gpu_walk_geometry(name, s, long_table):
    """every geometry launch of the set, without and with dictionary images, against the oracle at every position"""
    for lname, frames, slot in launches(s[1]):
        check_launch(frames, s, long_table, image=False, slot=slot)
        if any(f.tail for f in frames):
            check_launch(frames, s, long_table, image=True, slot=slot)


def _sweep_groups():
    groups = {}
    for s in W.product_sets() + W.harness_sets():
        groups.setdefault(s[:4], []).append(s)
    return groups


@pytest.mark.gpu
@pytest.mark.parametrize("key", sorted(_sweep_groups()), ids=lambda k: f"s{k[0]}_m{k[1]}_N{k[2]}_L{k[3]}")
def test_gpu_walk_every_parameter_set(key):
    """every parameter set the planner yields and every harness-only set, on a launch of a dictionary frame and a frame of
    1 KiB blocks, with images, against the oracle at every position"""
    mls = key[1]
    t = W.walk_input(1025, 11, mls)
    frames = [Frame(t, W.walk_input(9000, 12, mls, t)), Frame(b"", W.walk_input(5000 + 4096 * 4, 13, mls), 10)]
    for s in _sweep_groups()[key]:
        check_launch(frames, s, False, image=True)
        if s[0] == 2:
            check_launch(frames, s, True, image=True)
