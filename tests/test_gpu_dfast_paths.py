"""Paths of the doubleFast parse (K1b dfast, zb_parse_dfast_kernel in zstd_b200/csrc/zb_match.cu), which serves levels 2-4
and every level from 5 up.

On the CPU (runs without a GPU): a Python restatement of the oracle's doubleFast parse (tests/dfastgen.py), fed the
candidates of the oracle's own walk, is proved equal to zbo_parseBlock on every block of every input below; it then counts
the path each probe takes, and every path is reached by these inputs.  Rule switches (one neighbouring wrong rule each)
each change some block's sequences: the inputs tell the rule from its neighbours.

On the GPU: every input is compressed and compared byte for byte with the oracle's frame, and decoded with the reference
decoder: levels 2, 3, 4 and >= 5 in all four size classes of the parameter table, raw and zstd-format dictionaries (one
with chosen repcodes) through ZSTD_compress_usingDict and ZSTD_CDict, and batch calls on device buffers."""
import functools
import os

import pytest

import dfastgen as g
import zref

needs_oracle = pytest.mark.skipif(not os.path.exists(zref.ORACLE_SO), reason="oracle/libzb_oracle.so not built")


@functools.lru_cache(maxsize=None)
def _blocks():
    return [b for src, level, d in g.all_frames() for b in g.frame_blocks(src, level, d)]


@functools.lru_cache(maxsize=None)
def _restated():
    counts = {}
    seqs = [g.parse_block(b, cnt=counts) for b in _blocks()]
    return seqs, counts


def _table(counts):
    return "\n".join(f"{r:18s} {counts.get(r, 0)}" for r in g.ROWS + g.CLEARED)


# ------------------------------------------------------------------------------------------------------------ CPU
@needs_oracle
def test_restatement_is_the_oracle():
    blocks = _blocks()
    seqs, _ = _restated()
    assert len(blocks) > 100
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
def test_candidates_never_reach_in_front_of_the_window():
    """The parse clears a candidate that reaches in front of the block's history limit.  The limit is the chunk's history
    start on every block here (the window covers the frame and its dictionary), so that clearing never acts: a candidate
    of the walk always lies inside the chunk's history."""
    _, counts = _restated()
    assert all(b.low == b.chunk_low for b in _blocks())
    assert all(counts.get(r, 0) == 0 for r in g.CLEARED), _table(counts)


@needs_oracle
@pytest.mark.parametrize("switch", sorted(g.SWITCHES))
def test_inputs_tell_the_rule_from(switch):
    """a neighbouring wrong rule changes the sequences of at least one block"""
    seqs, _ = _restated()
    changed = sum(g.parse_block(b, frozenset([switch])) != s for b, s in zip(_blocks(), seqs))
    print(f"{switch}: {changed} blocks change ({g.SWITCHES[switch]})")
    assert changed > 0, g.SWITCHES[switch]


def test_no_long_candidate_has_exactly_seven_equal_bytes():
    """Why a long threshold of 7 cannot be told from 8: two 8-byte strings that differ in their last byte only never share a
    bucket of the 8-byte table (2^14 buckets or fewer: the top bits of the hash), so a long candidate that is not a
    real 8-byte match agrees in at most 6 leading bytes.  The inputs hold such 6-byte collisions (dfastgen.twin8_six)."""
    import random
    rnd = random.Random(3)
    for _ in range(2000):
        x = rnd.randbytes(8)
        h = g.hash8(int.from_bytes(x, "little"))
        for d in range(1, 256):
            y = x[:7] + bytes([(x[7] + d) & 255])
            assert g.hash8(int.from_bytes(y, "little")) >> 24 != h >> 24
        g.twin8_six(x)


def test_generator_is_deterministic_and_sized():
    a, b = g.dfast_input(40000, 9), g.dfast_input(40000, 9)
    assert a == b and len(a) == 40000
    assert len(g.dfast_input(g.SEG - 1, 2)) == g.SEG - 1


# ------------------------------------------------------------------------------------------------------------ GPU
def _check(got, src, level, d=None):
    want = zref.oracle_compress(src, level) if d is None else zref.oracle_compress_using_dict(src, d, level)
    assert got == want, (len(src), level, len(got), len(want))
    if zref.have_ref():
        out = zref.ref_decompress(got, len(src)) if d is None else zref.ref_decompress_using_dict(got, d, len(src))
        assert out == src


@pytest.mark.gpu
@pytest.mark.parametrize("cls,level", g.FRAME_CASES + [(n, lv) for n, _, lv in g.EXTRA_FRAMES])
def test_dfast_frame(cls, level):
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
@pytest.mark.parametrize("name", g.DICT_NAMES)
def test_dfast_dictionary(name, level):
    """the DICT instantiation: walked from the dictionary bytes (usingDict) and primed from the CDict's table image"""
    import zstd_b200
    d = g.dictionary(name)
    c = zstd_b200.ZSTD_CCtx()
    cd = zstd_b200.ZSTD_CDict(d, level)
    try:
        for src in g.dict_inputs(name):
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
def test_dfast_batch_small_frames():
    """frames of at most 8 KiB: one parse segment per block"""
    _batch(g.batch_small(), g.BATCH_LEVEL)


@pytest.mark.gpu
def test_dfast_batch_mixed_frames():
    """large and small frames in one call: eight segments per block, the small blocks leave segments empty"""
    _batch(g.batch_mixed(), g.BATCH_LEVEL)
