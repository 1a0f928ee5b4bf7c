"""Paths of the fast greedy parse (K1b, zb_parse_kernel in zstd_b200/csrc/zb_match.cu), which serves every negative level,
level 1 and level 2 in three of the four size classes of the parameter table.

On the CPU (runs without a GPU): a Python restatement of the oracle's fast parse (tests/fastgen.py), fed the candidates of
the oracle's own walk, is proved equal to zbo_parseBlock on every block of every input below; it then counts the path each
probe and each match takes, and every path is reached by these inputs, the blocks whose history limit the window cuts
included.  Rule switches (one neighbouring wrong rule each) each change some block's sequences: the inputs tell the rule
from its neighbours.

On the GPU: every input is compressed and compared byte for byte with the oracle's frame, and decoded with the reference
decoder: every fast row of the parameter table, frames of 1.25 MiB whose fourth block of the second chunk has its history
cut by the window, raw and zstd-format dictionaries (one with chosen repcodes) through ZSTD_compress_usingDict and
ZSTD_CDict, and batch calls on device buffers (one of frames of at most 8 KiB: one segment per row).

The older cases below (`mixed` inputs) are hand-made copies aimed at the same paths:
- table candidates at distances >= 0xFFFF (`far`, fetched only for the lane being tried) that win, and that lose to a
  lower lane with a near candidate or a repcode;
- tag false positives (random bytes: bucket collisions with equal 11-bit tags) in front of a real hit at a higher lane;
- repcode-2 right after a match; repcode-1 hits whose catch-up runs past 4 and past 32 bytes, and catch-up stopped by
  the anchor (copies that follow a copy without literals);
- matches longer than one 256-byte forward round, matches that end within 8 bytes of a block's end and matches that run
  past a segment's end (copies across 16 KiB and 128 KiB borders);
- the step sizes of levels 1, -1, -3 and -7, with and without a dictionary in front."""
import functools
import os
import random

import pytest

import dfastgen as dg
import fastgen as g
import zref

needs_oracle = pytest.mark.skipif(not os.path.exists(zref.ORACLE_SO), reason="oracle/libzb_oracle.so not built")


@functools.lru_cache(maxsize=None)
def _blocks():
    return [b for src, level, d in g.all_frames() for b in dg.frame_blocks(src, level, d)]


@functools.lru_cache(maxsize=None)
def _restated():
    counts = {}
    seqs = [g.parse_block(b, cnt=counts) for b in _blocks()]
    return seqs, counts


def _table(counts):
    return "\n".join(f"{r:18s} {counts.get(r, 0)}" for r in g.ROWS + g.NEVER)


# ------------------------------------------------------------------------------------------------------------ CPU
@needs_oracle
def test_restatement_is_the_oracle():
    blocks = _blocks()
    seqs, _ = _restated()
    assert len(blocks) > 100 and all(b.strategy == 1 for b in blocks)
    bad = [i for i, (s, b) in enumerate(zip(seqs, blocks)) if s != b.oracle_seqs]
    assert not bad, f"{len(bad)} of {len(blocks)} blocks differ from zbo_parseBlock, first: {bad[0]}"
    assert sum(len(s) for s in seqs) > 10000


@needs_oracle
def test_every_path_is_reached():
    _, counts = _restated()
    missing = [r for r in g.ROWS if counts.get(r, 0) == 0]
    print(_table(counts))
    assert not missing, f"paths not reached: {missing}\n{_table(counts)}"


@needs_oracle
def test_window_cut_blocks():
    """At a window of 2^19 the fourth block of every chunk after the first has its history limit moved from 128 KiB in
    front of the chunk to the chunk's start; the window-cut frames hold such blocks at levels 1 and -3.  Every candidate
    in front of that limit is far, and repcode-1 never reaches in front of it: those rows stay zero."""
    _, counts = _restated()
    cut = [b for b in _blocks() if b.low != b.chunk_low]
    assert len(cut) == 2 and all(b.low == b.c0 and b.be - b.c0 == g.CHUNK for b in cut)
    assert sorted(b.step_size for b in cut) == [2, 4]
    assert all(counts.get(r, 0) == 0 for r in g.NEVER), _table(counts)


@needs_oracle
@pytest.mark.parametrize("switch", sorted(g.SWITCHES))
def test_inputs_tell_the_rule_from(switch):
    """a neighbouring wrong rule changes the sequences of at least one block"""
    seqs, _ = _restated()
    changed = sum(g.parse_block(b, frozenset([switch])) != s for b, s in zip(_blocks(), seqs))
    print(f"{switch}: {changed} blocks change ({g.SWITCHES[switch]})")
    assert changed > 0, g.SWITCHES[switch]


def test_cut_input_is_deterministic_and_sized():
    a = g.cut_input(g.CUT_SIZE, 5)
    assert a == g.cut_input(g.CUT_SIZE, 5) and len(a) == g.CUT_SIZE


# ------------------------------------------------------------------------------------------------------------ GPU
def _check(got, src, level, d=None):
    want = zref.oracle_compress(src, level) if d is None else zref.oracle_compress_using_dict(src, d, level)
    assert got == want, (len(src), level, len(got), len(want))
    if zref.have_ref():
        out = zref.ref_decompress(got, len(src)) if d is None else zref.ref_decompress_using_dict(got, d, len(src))
        assert out == src


@pytest.mark.gpu
@pytest.mark.parametrize("cls,level", g.FRAME_CASES)
def test_fast_frame(cls, level):
    import zstd_b200
    src = g.frame_input(cls)
    c = zstd_b200.ZSTD_CCtx()
    try:
        got = c.compress(src, level)
    finally:
        c.close()
    _check(got, src, level)


@pytest.mark.gpu
@pytest.mark.parametrize("level", g.DICT_LEVELS)
@pytest.mark.parametrize("name", dg.DICT_NAMES)
def test_fast_dictionary(name, level):
    """the DICT instantiation: walked from the dictionary bytes (usingDict) and primed from the CDict's table image"""
    import zstd_b200
    d = dg.dictionary(name)
    c = zstd_b200.ZSTD_CCtx()
    cd = zstd_b200.ZSTD_CDict(d, level)
    try:
        for src in dg.dict_inputs(name):
            got = c.compress_using_dict(src, d, level)
            _check(got, src, level, d)
            assert c.compress_using_cdict(src, cd) == got
    finally:
        cd.close()
        c.close()


def _batch(frames, level):
    import torch
    import zstd_b200
    src = b"".join(frames)
    offs = [sum(len(f) for f in frames[:i]) for i in range(len(frames))]
    d_src = torch.frombuffer(bytearray(src), dtype=torch.uint8).cuda()
    cap = sum(zstd_b200.ZSTD_compressBound(len(f)) + 64 for f in frames)
    d_dst = torch.empty(cap, dtype=torch.uint8, device="cuda")
    c = zstd_b200.ZSTD_CCtx()
    try:
        total, csz = c.compress_frames(d_dst.data_ptr(), cap, d_src.data_ptr(), offs, [len(f) for f in frames], level=level)
    finally:
        c.close()
    out = bytes(d_dst[:total].cpu().numpy())
    assert sum(csz) == total
    pos = 0
    for f, n in zip(frames, csz):
        _check(out[pos:pos + n], f, level)
        pos += n


@pytest.mark.gpu
def test_fast_batch_small_frames():
    """frames of at most 8 KiB: the call's largest block is one segment, so one segment fills a row"""
    _batch(dg.batch_small(), g.BATCH_LEVEL)


@pytest.mark.gpu
def test_fast_batch_mixed_frames():
    """large and small frames in one call: eight segments per block, the small blocks leave segments empty"""
    _batch(dg.batch_mixed(), g.BATCH_LEVEL)


# ------------------------------------------------------------------------------------------------ hand-made cases

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
