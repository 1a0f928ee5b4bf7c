"""Inputs for the fast greedy parse (K1b, zb_parse_kernel in zstd_b200/csrc/zb_match.cu) and a Python restatement of the
oracle's fast parse (parse_fast_segment, oracle/zb_match.c) that counts which path every probe and every match takes.
TEST INFRASTRUCTURE ONLY.

Blocks come from dfastgen.frame_blocks, which drives the oracle's own walk as zbo_compress_usingDict does, and are joined by
dfastgen.parse_block; tests/test_gpu_parse_paths.py proves the restatement equal to zbo_parseBlock on every block, so its
path counts are the oracle's.  Switches replace one rule by a neighbouring wrong one: the inputs must tell each of them
apart from the rule."""
import random

import dfastgen as dg
import zref

BLOCK, FAR, WARP = dg.BLOCK, dg.FAR, dg.WARP
CHUNK = 4 * BLOCK                                            # a chunk of the walk: one hash table lives through it
PRIME = 128 << 10                                            # history primed into every chunk but the first

# rows of the path table; every one is reached by the inputs below
ROWS = [
    "rep2_anchor",        # repcode-2 at lane 0 right after a match (zstd_fast.c:410-420)
    "rep1",               # repcode-1 at the probed position
    "table",              # a table candidate with 4 equal bytes
    "rep1_over_table",    # repcode-1 wins over a table candidate of another offset that also has 4 equal bytes
    "tag_coll",           # a table candidate whose first 4 bytes differ (a hash tag collision): the next lane is tried
    "tag_coll_next_hit",  # ... and a higher lane of the same step wins
    "far_hit",            # a table hit at a distance >= 0xFFFF (the walk's far array)
    "far_refused",        # a far candidate that reaches in front of the block's history limit
    "accel_2",            # the acceleration (ip - anchor) >> 7 adds 2 or more to the step
    "accel_4",
    "accel_8",
    "step_size_2",        # matches found at a stepSize of 2 (levels 2, 1, -1), 4 (level -3) and 8 (level -7)
    "step_size_4",
    "step_size_8",
    "table_mls4",         # table hits at each minimum match length the fast rows use (the walk's hash width)
    "table_mls5",
    "table_mls6",
    "table_mls7",
    "lanes_cut_se",       # lanes at or beyond the segment's end are not probed
    "lanes_cut_be",       # lanes with p + 8 > blockEnd are not probed
    "tail_unprobed",      # the parse of a block's last segment stops with < 8 bytes left
    "back_32",            # backward catch-up of 32 bytes or more (a second cooperative round)
    "back_stop_anchor",   # catch-up stopped by the anchor while the bytes in front still match
    "back_stop_low",      # catch-up stopped by the history limit while the bytes in front still match
    "fwd_256",            # forward count of 256 bytes or more (a second cooperative round)
    "fwd_tail",           # the match ends within the last 8 bytes of the block, short of its end (the clamped last load)
    "fwd_to_be",          # the match ends exactly at the block's end
    "join_drop",          # the join drops a sequence that lies under a match run over from an earlier segment
    "join_trim",          # the join keeps the tail (>= 3 bytes) of a sequence that straddles the previous match's end
    "start_rep",          # a repcode hit with the repcodes of a zstd-format dictionary, before the segment's first match
    "dict_cross",         # a match whose source straddles the dictionary / frame border
    "dict_back_cross",    # a catch-up that crosses the dictionary / frame border
    "cut_far",            # window cut: a far candidate with 4 equal bytes in front of the cut limit, refused
    "cut_far_next_hit",   # ... and a higher lane of the same step wins
    "cut_stop_low",       # window cut: a catch-up stopped by the cut limit while the bytes in front still match
]
# Candidates that would hit but reach in front of a window-cut limit, and can never occur.  The limit is cut only in the
# fourth block of a chunk after the first at a window of 2^19 (levels <= 1, frames over 896 KiB): the limit is then the
# chunk's start, 3 blocks = 384 KiB in front of the block, so every candidate behind it is far.  Repcode-1 is an offset
# this segment's parse took at a lower position, where its source was checked against the same limit.
NEVER = ["cut_near", "cut_rep1"]

SWITCHES = {
    "accel_256": "the step grows every 256 bytes without a match instead of 128",
    "table_before_rep1": "the table candidate is tried before repcode-1",
    "rep2_every_step": "repcode-2 is tried at lane 0 of every step, not only right after a match",
    "probe_9": "positions are probed while p + 9 <= blockEnd instead of p + 8",
    "reach_gt": "a candidate's source must lie behind the history limit (p > low + d) instead of at or behind it",
    "cut_at_start": "the window cut is evaluated at the block's start instead of its end",
    "catchup_past_anchor": "the backward catch-up ignores the anchor",
    "advance_15": "a step without a hit advances by 15 * step instead of 16 * step",
}


def _eq4(buf, a, b):
    assert b >= 0
    return buf[a:a + 4] == buf[b:b + 4]


def parse_segment(blk: dg.Block, ss: int, se: int, sw=frozenset(), cnt=None):
    """parse_fast_segment (oracle/zb_match.c:211-244): raw sequences (match start, length, real offset) of one segment"""
    buf, dS, c0, be, D = blk.buf, blk.dS, blk.c0, blk.be, blk.frame_start
    low = blk.low
    if "cut_at_start" in sw:
        low = blk.bs - blk.window if blk.bs > blk.window and blk.bs - blk.window > blk.chunk_low else blk.chunk_low
    cut = low > blk.chunk_low
    shift = 8 if "accel_256" in sw else 7
    need = 9 if "probe_9" in sw else 8
    table_first = "table_before_rep1" in sw
    rep2_every = "rep2_every_step" in sw
    past_anchor = "catchup_past_anchor" in sw
    advance = 15 if "advance_15" in sw else 16
    if "reach_gt" in sw:
        def reach(p, o):
            return p > low + o
    else:
        def reach(p, o):
            return p >= low + o
    c = cnt if cnt is not None else {}

    def bump(k):
        c[k] = c.get(k, 0) + 1

    ip = anchor = ss
    rep1, rep2 = blk.start_reps if ss == D else (0, 0)
    inherited = rep1 or rep2
    out = []
    while ip < se and ip + need <= be:
        acc = (ip - anchor) >> shift
        step = blk.step_size + acc
        for k in (2, 4, 8):
            if acc >= k:
                bump(f"accel_{k}")
        found = None
        refused = None                                       # why a lower lane of this step was passed over
        for l in range(WARP):
            p = ip + (l >> 1) * step + (l & 1)
            if p >= se:
                bump("lanes_cut_se")
                break
            if p + need > be:
                bump("lanes_cut_be")
                break
            d = dS[p - c0]
            if l == 0 and (ip == anchor or rep2_every) and rep2 and _eq4(buf, p, p - rep2):
                found = (3, p, rep2)
                break
            r1 = rep1 and reach(p, rep1) and _eq4(buf, p, p - rep1)
            t_in = d and reach(p, d)
            t = t_in and _eq4(buf, p, p - d)
            if rep1 and not reach(p, rep1) and p >= rep1 and _eq4(buf, p, p - rep1):
                bump("cut_rep1")
            if d and not t_in:
                if d >= FAR:
                    bump("far_refused")
                if _eq4(buf, p, p - d):
                    bump("cut_far" if d >= FAR else "cut_near")
                    refused = refused or "cut_far"
            if r1 and not (table_first and t):
                if t and d != rep1:
                    bump("rep1_over_table")
                found = (2, p, rep1)
                break
            if t:
                found = (1, p, d)
                break
            if t_in:
                bump("tag_coll")
                refused = refused or "tag_coll"
        if found is None:
            ip += advance * step
            continue
        if refused:
            bump(refused + "_next_hit")
        wtype, probe, off = found
        bump(("table", "rep1", "rep2_anchor")[wtype - 1])
        if wtype == 1:
            bump(f"table_mls{blk.mls}")
            if off >= FAR:
                bump("far_hit")
        if wtype != 1 and inherited and not out:
            bump("start_rep")
        bump(f"step_size_{blk.step_size}")
        ms, mm = probe, probe - off
        if wtype != 3:                                       # backward catch-up (zstd_fast.c:387-391)
            bound = low if past_anchor else anchor
            while ms > bound and mm > low and buf[ms - 1] == buf[mm - 1]:
                ms -= 1
                mm -= 1
            if probe - ms >= 32:
                bump("back_32")
            if ms == anchor and mm > low and buf[ms - 1] == buf[mm - 1]:
                bump("back_stop_anchor")
            if mm == low and ms > anchor and low > 0 and buf[ms - 1] == buf[mm - 1]:
                bump("back_stop_low")
                if cut:
                    bump("cut_stop_low")
            if D and probe - off >= D > mm:
                bump("dict_back_cross")
        fwd = dg._fwd(buf, probe + 4, probe + 4 - off, be)
        mlen = (probe - ms) + 4 + fwd
        if fwd + (4 if wtype == 1 else 0) >= 256:            # what the first cooperative round counts from
            bump("fwd_256")
        end = ms + mlen
        if 0 < be - end < 8:
            bump("fwd_tail")
        if end == be:
            bump("fwd_to_be")
        if D and ms - off < D < ms - off + mlen:
            bump("dict_cross")
        if wtype == 3:
            rep1, rep2 = rep2, rep1
        elif wtype == 1:
            rep1, rep2 = off, rep1
        out.append((ms, mlen, off))
        ip = anchor = ms + mlen
    if ip < se and ip < be and ip + need > be:
        bump("tail_unprobed")
    return out


def parse_block(blk: dg.Block, sw=frozenset(), cnt=None):
    return dg.parse_block(blk, sw, cnt, segment=parse_segment)


# ------------------------------------------------------------------------------------------------------- generator
def cut_input(n: int, seed: int) -> bytes:
    """a frame of n >= 1.25 MiB for a window of 2^19 (levels <= 1).  The fourth block of the second chunk, whose history
    limit the window moves from 128 KiB in front of the chunk to the chunk's start, copies from that primed 128 KiB (every
    source far, refused) and across the chunk's start (a catch-up the limit stops).  The three blocks in between repeat a
    short period: the walk inserts nothing there, so the primed sources stay in the table.  The first chunk, the rest of
    the fourth block and the third chunk are dfastgen inputs; the last two may copy from the 128 KiB in front of them."""
    assert n >= CHUNK + 4 * BLOCK + BLOCK // 4
    rnd = random.Random(seed)
    gad = 64 * 40
    out = bytearray(dg.dfast_input(CHUNK - gad - 24, seed))
    sources = []
    while len(out) < CHUNK - 24 - 64:                        # sources: 48 random bytes each, between copies of 16
        sources.append(len(out))
        out += rnd.randbytes(48)
        o = rnd.randint(64, 4000)
        out += out[len(out) - o:len(out) - o + 16]
    out += rnd.randbytes(CHUNK - 24 - len(out))
    straddle = len(out)                                      # 24 bytes in front of the chunk's start, 40 behind it
    out += rnd.randbytes(64)
    period = rnd.randbytes(7)
    b7 = CHUNK + 3 * BLOCK
    out += (period * (b7 // 7 + 2))[:b7 - 256 - len(out)]
    out += rnd.randbytes(256)
    for s in rnd.sample(sources, len(sources)):              # far copies from the primed history
        out += out[s:s + rnd.randint(24, 48)] + rnd.randbytes(rnd.randint(4, 16))
        if rnd.random() < 0.3:
            out += out[straddle:straddle + 64] + rnd.randbytes(8)
        if rnd.random() < 0.3:                               # near: the same again from this block
            o = rnd.randint(64, 3000)
            out += out[len(out) - o:len(out) - o + rnd.randint(8, 40)] + rnd.randbytes(3)
    out += out[straddle:straddle + 64] + rnd.randbytes(8)
    rest = (b7 + BLOCK) - len(out)
    assert rest > 0
    out += dg.dfast_input(rest, seed + 1, bytes(out[-PRIME:]))
    out += dg.dfast_input(n - len(out), seed + 2, bytes(out[-PRIME:]))
    return bytes(out)


# -------------------------------------------------------------------------------------------------- the GPU cases
# (size class, level): every fast row of the parameter table -- tables 0-3 (> 256 KiB, <= 256 KiB, <= 128 KiB, <= 16 KiB)
# at level 1 and at a negative level, level 2 where it is fast (tables 0, 2 and 3; table 3 is the one fast row of minimum
# match length 4) -- and the window-cut frames at levels 1 and -3
FRAME_CASES = [("cut", 1), ("cut", -3), ("gt256k", 2), ("gt256k", -7),
               ("le256k", 1), ("le256k", -1),
               ("le128k", 1), ("le128k", 2), ("le128k", -7),
               ("le16k", 1), ("le16k", 2), ("le16k", -3)]
CUT_SIZE = CHUNK + 6 * BLOCK + 11                          # 1.25 MiB and a little: three chunks, the second one cut
DICT_LEVELS = [1, -3]
BATCH_LEVEL = 1

_cache = {}


def frame_input(name: str) -> bytes:
    if name != "cut":
        return dg.frame_input(name)
    if "cut" not in _cache:
        _cache["cut"] = cut_input(CUT_SIZE, 31)
    return _cache["cut"]


def all_frames():
    """(src, level, dictionary or None) of every frame the GPU tests compress, de-duplicated"""
    seen, out = set(), []

    def add(src, level, d):
        k = (zref.sha(src), level, zref.sha(d) if d else None)
        if k not in seen:
            seen.add(k)
            out.append((src, level, d))
    for name, level in FRAME_CASES:
        add(frame_input(name), level, None)
    for name in dg.DICT_NAMES:
        for level in DICT_LEVELS:
            for src in dg.dict_inputs(name):
                add(src, level, dg.dictionary(name))
    for f in dg.batch_small() + dg.batch_mixed():
        add(f, BATCH_LEVEL, None)
    return out
