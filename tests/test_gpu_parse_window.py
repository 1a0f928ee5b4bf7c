"""Boundaries of the fast parse's hit path (K1b, zb_parse_kernel in zstd_b200/csrc/zb_match.cu) that the path table of
tests/test_gpu_parse_paths.py does not name, counted on the same inputs (tests/fastgen.py).  CPU only: the GPU half of
that file compresses every one of these inputs and compares the frames byte for byte with the oracle's.

A hit reads one pair of 8-byte windows per lane.  Lane 31 holds the 8 bytes in front of the probe and answers the
catch-up when it is shorter than 8 bytes; a catch-up of 8 bytes or more goes on to the cooperative 32-byte rounds.  Lane
31 reads fewer than 8 bytes where the candidate lies less than 8 bytes behind the history's start, and a candidate
window that straddles the dictionary / frame border is read byte by byte.  The rows below show the inputs reach each
side of these limits, and the lanes that are tried again after a tag collision or a far candidate out of reach."""
import functools
import os

import pytest

import dfastgen as dg
import fastgen as g
import zref

needs_oracle = pytest.mark.skipif(not os.path.exists(zref.ORACLE_SO), reason="oracle/libzb_oracle.so not built")

ROWS = [
    "catchup_in_window",    # a catch-up of 1 to 7 bytes: lane 31's window answers it
    "catchup_8",            # exactly the window's width: one cooperative round that finds nothing more
    "catchup_9",            # one byte past the window
    "window_stop_anchor",   # a catch-up of 1 to 7 bytes stopped by the anchor while the bytes in front still match
    "window_stop_offset",   # a catch-up of 1 to 7 bytes stopped by the history's start while the bytes in front match
    "window_short",         # the candidate lies less than 8 bytes behind the history's start: lane 31 reads fewer
    "window_dict_straddle", # lane 31's candidate window straddles the dictionary / frame border (read byte by byte)
    "tag_coll_next_hit",    # a tag collision, then a higher lane of the same step wins (the lane loop is re-entered)
    "far_refused",          # a far candidate that reaches in front of the history (its lane drops out the same way)
]


@functools.lru_cache(maxsize=None)
def _counts():
    """the restated parse, segment by segment, over every input: each match's probe and offset are taken where the parse
    counts forward from probe + 4, its start from the segment's raw sequences"""
    counts = {}
    real_fwd = dg._fwd
    probes = []

    def fwd(buf, a, b, end):
        probes.append(a - 4)
        return real_fwd(buf, a, b, end)

    def bump(k):
        counts[k] = counts.get(k, 0) + 1

    dg._fwd = fwd
    try:
        for src, level, d in g.all_frames():
            for blk in dg.frame_blocks(src, level, d):
                for ss in range(blk.bs, blk.be, dg.SEG):
                    del probes[:]
                    out = g.parse_segment(blk, ss, min(ss + dg.SEG, blk.be), cnt=counts)
                    assert len(out) == len(probes)
                    _rows(blk, ss, zip(probes, out), bump)
    finally:
        dg._fwd = real_fwd
    return counts


def _rows(blk, ss, matches, bump):
    buf, low, D = blk.buf, blk.low, blk.frame_start
    anchor = ss
    for probe, (ms, mlen, off) in matches:
        back, mm = probe - ms, ms - off
        if 0 < back < 8:
            bump("catchup_in_window")
            if mm > low and buf[ms - 1] == buf[mm - 1]:
                assert ms == anchor
                bump("window_stop_anchor")
            elif mm == low and low > 0 and ms > anchor and buf[ms - 1] == buf[mm - 1]:
                bump("window_stop_offset")
        elif back == 8:
            bump("catchup_8")
        elif back == 9:
            bump("catchup_9")
        if probe - off - low < 8:
            bump("window_short")
        if D and probe - off - 8 < D < probe - off + 4:
            bump("window_dict_straddle")
        anchor = ms + mlen


@needs_oracle
def test_hit_window_boundaries_are_reached():
    counts = _counts()
    table = "\n".join(f"{r:22s} {counts.get(r, 0)}" for r in ROWS)
    print(table)
    missing = [r for r in ROWS if counts.get(r, 0) == 0]
    assert not missing, f"boundaries not reached: {missing}\n{table}"
