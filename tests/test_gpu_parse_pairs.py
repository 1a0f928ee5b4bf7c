"""The fast parse's pair iteration (K1b, zb_parse_kernel in zstd_b200/csrc/zb_match.cu).  One iteration probes two steps
of the rule at once, one pair of positions (p, p+1) per lane: lanes 0..15 the step at ip, lanes 16..31 the step the rule
takes next, at ip2 = ip + 16 * step with its own acceleration.  The lowest position with a real hit wins: a lane's p
before its p+1, and a position that drops out (a tag false positive, a candidate in front of the history) hands over to
the next one, which can be the same lane's p+1 or a position of the second half.

On the CPU: a Python restatement of the pair iteration, fed the candidates of the oracle's own walk, gives the same raw
sequences as the restated rule of tests/fastgen.py (which tests/test_gpu_parse_paths.py proves equal to zbo_parseBlock) on
every block of the inputs below, and counts the cases only the pair iteration has: every one is reached.
On the GPU: every input is compressed at levels 1, -1, -3 and -7, with and without a dictionary, and compared byte for
byte with the oracle's frame."""
import functools
import os

import pytest

import dfastgen as dg
import fastgen as g
import zref

needs_oracle = pytest.mark.skipif(not os.path.exists(zref.ORACLE_SO), reason="oracle/libzb_oracle.so not built")

LEVELS = [1, -1, -3, -7]
FRAMES = ["le256k", "le128k", "cut"]
DICTS = ["raw-20k", "zdict-16k-reps"]

ROWS = [
    "accel_change",         # the second half of an iteration is probed at a larger step than the first
    "second_after_tag",     # a real hit in the second half after a tag false positive in the first half
    "p1_after_p_drop",      # a hit at p+1 after p of the same lane dropped out
    "se_between",           # p < se <= p+1: p is probed, p+1 is not
    "be_between",           # p + 8 <= be < p + 9: p is probed, p+1 is not
    "rep1_window_straddle", # the repcode-1 bytes of p+1 straddle the dictionary / frame border (read byte by byte)
    "far_p1",               # a far candidate (distance >= 0xFFFF) at p+1 is tried
]
# Repcode-1 reaches the history from p+1 but not from p (p + 1 == low + rep1): never.  Repcodes start empty in every
# segment but a frame's first behind a zstd-format dictionary, whose repcodes are at most the dictionary's length, so at
# most the first position's distance to the history's start; every later rep1 is the offset of a match of the segment,
# whose source lies in the history, and every later position lies behind that match.
NEVER = ["rep1_p1_only"]


def _eq4(buf, a, b):
    return buf[a:a + 4] == buf[b:b + 4]


def pair_segment(blk: dg.Block, ss: int, se: int, bump):
    """raw sequences (match start, length, real offset) of one segment, found as the pair iteration finds them"""
    buf, dS, c0, be, low, D = blk.buf, blk.dS, blk.c0, blk.be, blk.low, blk.frame_start
    ip = anchor = ss
    rep1, rep2 = blk.start_reps if ss == D else (0, 0)
    last = min(se - 1, be - 8)                           # the last position probed: p < se and p + 8 <= be
    out = []
    while ip <= last:
        s1 = blk.step_size + ((ip - anchor) >> 7)
        ip2 = ip + 16 * s1
        s2 = blk.step_size + ((ip2 - anchor) >> 7)
        found, dropped = None, []                        # dropped: (lane, parity, why) of the positions tried before
        for lane in range(32):
            p = ip + lane * s1 if lane < 16 else ip2 + (lane - 16) * s2
            if p == se - 1 and p + 8 <= be:
                bump("se_between")
            if p == be - 8 and p < se:
                bump("be_between")
            for par in (0, 1):
                q = p + par
                if q > last:
                    break
                if par and rep1 and q >= low + rep1 and q - 1 < low + rep1:
                    bump("rep1_p1_only")
                if par and rep1 and q >= low + rep1 and D and q - rep1 < D < q - rep1 + 4:
                    bump("rep1_window_straddle")
                d = dS[q - c0]
                if lane == 0 and par == 0 and ip == anchor and rep2 and _eq4(buf, q, q - rep2):
                    found = (3, q, rep2)
                elif rep1 and q >= low + rep1 and _eq4(buf, q, q - rep1):
                    found = (2, q, rep1)
                elif d:
                    if par and d >= dg.FAR:
                        bump("far_p1")
                    if q < low + d:
                        dropped.append((lane, par, "reach"))
                    elif not _eq4(buf, q, q - d):
                        dropped.append((lane, par, "tag"))
                    else:
                        found = (1, q, d)
                if found:
                    if lane >= 16 and any(l < 16 and why == "tag" for l, _, why in dropped):
                        bump("second_after_tag")
                    if par and (lane, 0) in [(l, pr) for l, pr, _ in dropped]:
                        bump("p1_after_p_drop")
                    break
            if found:
                break
        if s1 != s2 and ip2 <= last and (found is None or lane >= 16):
            bump("accel_change")
        if found is None:
            ip = ip2 + 16 * s2
            continue
        wtype, probe, off = found
        ms, mm = probe, probe - off
        if wtype != 3:                                   # backward catch-up (zstd_fast.c:387-391)
            while ms > anchor and mm > low and buf[ms - 1] == buf[mm - 1]:
                ms -= 1
                mm -= 1
        mlen = (probe - ms) + 4 + dg._fwd(buf, probe + 4, probe + 4 - off, be)
        if wtype == 3:
            rep1, rep2 = rep2, rep1
        elif wtype == 1:
            rep1, rep2 = off, rep1
        out.append((ms, mlen, off))
        ip = anchor = ms + mlen
    return out


def _cases():
    """(src, level, dictionary or None) of every frame below"""
    out = [(g.frame_input(name), level, None) for name in FRAMES for level in LEVELS]
    for name in DICTS:
        for src in dg.dict_inputs(name):
            out += [(src, level, dg.dictionary(name)) for level in LEVELS]
    return out


@functools.lru_cache(maxsize=None)
def _counts():
    counts, bad, segs = {}, [], 0

    def bump(k):
        counts[k] = counts.get(k, 0) + 1
    for src, level, d in _cases():
        for blk in dg.frame_blocks(src, level, d):
            for ss in range(blk.bs, blk.be, dg.SEG):
                se = min(ss + dg.SEG, blk.be)
                segs += 1
                if pair_segment(blk, ss, se, bump) != g.parse_segment(blk, ss, se):
                    bad.append((level, blk.bs, ss))
    return counts, bad, segs


def _table(counts):
    return "\n".join(f"{r:22s} {counts.get(r, 0)}" for r in ROWS + NEVER)


# ------------------------------------------------------------------------------------------------------------ CPU
@needs_oracle
def test_pairs_are_the_rule():
    counts, bad, segs = _counts()
    assert segs > 100
    assert not bad, f"{len(bad)} of {segs} segments differ from the restated rule, first (level, block, segment): {bad[0]}"


@needs_oracle
def test_every_pair_case_is_reached():
    counts, _, _ = _counts()
    print(_table(counts))
    missing = [r for r in ROWS if counts.get(r, 0) == 0]
    assert not missing, f"cases not reached: {missing}\n{_table(counts)}"
    assert all(counts.get(r, 0) == 0 for r in NEVER), _table(counts)


# ------------------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("level", LEVELS)
@pytest.mark.parametrize("name", FRAMES)
def test_pairs_frame(name, level):
    import zstd_b200
    src = g.frame_input(name)
    c = zstd_b200.ZSTD_CCtx()
    try:
        got = c.compress(src, level)
    finally:
        c.close()
    assert got == zref.oracle_compress(src, level), (name, level)
    if zref.have_ref():
        assert zref.ref_decompress(got, len(src)) == src


@pytest.mark.gpu
@pytest.mark.parametrize("level", LEVELS)
@pytest.mark.parametrize("name", DICTS)
def test_pairs_dictionary(name, level):
    """the DICT instantiation of the kernel"""
    import zstd_b200
    d = dg.dictionary(name)
    c = zstd_b200.ZSTD_CCtx()
    try:
        for src in dg.dict_inputs(name):
            got = c.compress_using_dict(src, d, level)
            assert got == zref.oracle_compress_using_dict(src, d, level), (name, level, len(src))
            if zref.have_ref():
                assert zref.ref_decompress_using_dict(got, d, len(src)) == src
    finally:
        c.close()
