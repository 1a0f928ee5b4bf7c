"""Inputs for long-distance matching (zb_ldm.cu: L1 split points and thinning, L2 bucket sort, L3 selection; and the overlay
zb_ldm_overlay in zb_match.cu) and a Python restatement of its rule (oracle/zb_ldm.c steps 1-5, with a prefix as
oracle/zb_prefix.c extends them) that counts which path every split point, survivor, candidate and parse match takes.
TEST INFRASTRUCTURE ONLY.

tests/test_gpu_ldm_paths.py proves each step equal to the oracle's own: steps 1-2 to zbo_ldm_survivors, steps 3-4 (fed the
oracle's survivors) to zbo_ldm_frame / zbo_ldm_frame_usingPrefix, step 5 (fed each block's zbo_parseBlock sequences, as
dfastgen.frame_blocks drives them) to zbo_ldm_overlayBlock; so its path counts are the oracle's.  Switches replace one rule
by a neighbouring wrong one: the inputs must tell each of them apart from the rule."""
import random

import numpy as np

import dfastgen as dg
import ldmref
import prefixref
import zref

BLOCK = dg.BLOCK
CHUNK = 4 * BLOCK                    # LDM runs on frames of more than one chunk
LDM_TILE = 4096                      # split points per L1 CTA (zb_ldm.cu)
OVERLAY_ROUND = 256                  # overlay entries per round of the merge kernel (MERGE_THREADS)
MERGE_TILE = 1024                    # sequences per round of the merge kernel's repcode pass (zb_merge.cuh)
SEQ_CAP = BLOCK // 4 + 8             # sd.seq of a call whose largest block is 128 KiB (zb_common.h)
M64 = (1 << 64) - 1

ROWS = [
    # steps 1-2: split points and thinning
    "thin_tie_left_kept",     # a survivor with an equal value on its left (<= on the left)
    "thin_tie_right_dropped", # a split dropped by an equal value on its right alone (< on the right)
    "thin_edge_start",        # a survivor within minMatch - 1 split points of its segment's start
    "thin_edge_end",          # ... of its segment's end
    "thin_tile_kept",         # a survivor compared with a split across a multiple of LDM_TILE split points (the L1 tile edge)
    "thin_tile_dropped",      # a split dropped by a split across such a multiple
    "hash_rate_0",            # splits hashed with hashRateLog 0: every split point fires
    "mask_low",               # splits hashed with hashRateLog > min(minMatch, 64): the stop mask in the low bits
    "xxh_stripes",            # XXH64 paths: 32-byte stripes, then the 8-, 4- and 1-byte tails
    "xxh_tail8",
    "xxh_tail4",
    "xxh_tail1",
    "passes_0",               # frames whose bucket sort takes 0, 1, 2, 3 and 4 radix passes
    "passes_1",
    "passes_2",
    "passes_3",
    "passes_4",
    # steps 3-4: buckets and selection
    "skip_anchor",            # a survivor under the anchor, skipped
    "no_earlier",             # no earlier key in the survivor's bucket
    "walk_bucket_edge",       # the candidate walk stopped by a key of another bucket
    "walk_rank",              # ... stopped by j > rank (the first key of the sorted order)
    "cand_limit",             # ... stopped after 2^bucketSizeLog candidates with more of the bucket left
    "ck_differs",             # a candidate of the bucket with another checksum
    "window_be",              # a candidate refused by q < be - W although p - q <= W
    "f_short_cap",            # f < minMatch only because the block end caps it
    "f_to_be",                # f equal to the block-end cap
    "f_seam",                 # f equal to the prefix seam (P - q)
    "f_256",                  # f >= 256: several warp rounds
    "f_tail",                 # f ends in the last 8 bytes of its cap (the byte loop)
    "b_zero",                 # b == 0
    "b_cap_anchor",           # b capped by p - anchor while the bytes in front still match
    "b_cap_q",                # b capped by q's segment: the match reaches the first byte of the frame or prefix
    "b_32",                   # b >= 32: several ballots
    "tie_nearer",             # a tie that keeps the nearer q
    "farther_longer",         # a farther candidate that wins by length
    "prefix_match",           # a selected match whose source lies in the prefix
    # step 5: overlay
    "ldm_before_parse",       # an LDM match placed before the next parse match
    "parse_unclipped",        # a parse match kept unclipped
    "clip_start_kept",        # clipped at its start, kept
    "clip_start_dropped",     # clipped at its start, < 4 bytes left, dropped
    "clip_end_kept",          # clipped at its end, kept
    "clip_end_dropped",       # clipped at its end, dropped
    "clip_both",              # clipped at both ends
    "covered",                # fully covered by an LDM match
    "span_whole",             # running over a whole LDM match, cut at its start
    "start_at_ldm_start",     # starting exactly at an LDM match's start
    "end_at_ldm_start",       # ending exactly at an LDM match's start: not clipped
    "tail3_kept",             # a 3-byte parse tail kept unclipped
    "no_parse",               # a block with LDM matches and no parse match
    "parse_256",              # more than 256 parse matches in a block (several overlay rounds)
    "ldm_256",                # more than 256 LDM matches in a block
    "merged_1024",            # more than 1024 merged sequences in a block (several merge tiles)
    "rep_from_history",       # an LDM offset coded as a repcode of the first block's history
]
# never happen, by the rule: asserted zero
NEVER = ["ldm_cross_edge", "ldm_overlap", "seq_over_cap"]

SWITCHES = {
    "thin_left_le": "thinning drops a split with an equal value on its left (<= on the left)",
    "thin_right_lt": "thinning keeps a split with an equal value on its right (< on the right)",
    "lowq_p": "the window limit is p - W instead of be - W",
    "tie_far": "a tie keeps the farther q",
    "b_no_anchor": "the backward count is not capped by the anchor",
    "anchor_p": "the anchor moves to p instead of p + f",
    "f_frame_end": "the forward count is capped at the frame end instead of the block end",
    "cand_plus1": "2^bucketSizeLog + 1 candidates",
    "keep_short3": "the overlay keeps shortened matches of 3 bytes or more",
    "keep_tail": "a parse match spanning an LDM match keeps its tail instead of its head",
    "under_strict": "'starts under an LDM match' is tested with a strict <",
    "seam_uncapped": "the forward count of a prefix candidate runs over the seam",
}
# A candidate with f >= minMatch has the survivor's minMatch bytes, so their XXH64 and its checksum are equal: the
# checksum only saves the forward count of candidates that cannot win.  A test shows it changes no block.
EQUIVALENT = {"no_checksum": "the checksum is not compared"}
THIN_SWITCHES = ("thin_left_le", "thin_right_lt")
OVERLAY_SWITCHES = ("keep_short3", "keep_tail", "under_strict")


def _bump(c, k, n=1):
    if c is not None and n:
        c[k] = c.get(k, 0) + n


# ------------------------------------------------------------------------------------------- steps 1-2 (numpy)
def _splitmix(i):
    z = (0x6C646D2D67656172 + (i + 1) * 0x9E3779B97F4A7C15) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


GEAR = np.array([_splitmix(i) for i in range(256)], dtype=np.uint64)
_U = np.uint64
P1, P2, P3, P4, P5 = (_U(0x9E3779B185EBCA87), _U(0xC2B2AE3D27D4EB4F), _U(0x165667B19E3779F9), _U(0x85EBCA77C2B2AE63),
                      _U(0x27D4EB2F165667C5))


def stop_mask(prm) -> int:
    max_bits = min(prm.minMatch, 64)
    if 0 < prm.hashRateLog <= max_bits:
        return ((1 << prm.hashRateLog) - 1) << (max_bits - prm.hashRateLog)
    return (1 << prm.hashRateLog) - 1


def _rotl(x, r):
    return (x << _U(r)) | (x >> _U(64 - r))


def _round(acc, w):
    return _rotl(acc + w * P2, 31) * P1


def xxh64(a: np.ndarray, words: np.ndarray, p: np.ndarray, n: int, cnt=None) -> np.ndarray:
    """XXH64 (seed 0) of the n bytes at every position in p; words[i] = the little-endian u64 at byte i"""
    with np.errstate(over="ignore"):
        i = 0
        if n >= 32:
            _bump(cnt, "xxh_stripes", len(p))
            v1 = np.full(len(p), (int(P1) + int(P2)) & M64, np.uint64)
            v2 = np.full(len(p), P2, np.uint64)
            v3 = np.zeros(len(p), np.uint64)
            v4 = np.full(len(p), (-int(P1)) & M64, np.uint64)
            while i + 32 <= n:
                v1, v2 = _round(v1, words[p + i]), _round(v2, words[p + i + 8])
                v3, v4 = _round(v3, words[p + i + 16]), _round(v4, words[p + i + 24])
                i += 32
            h = _rotl(v1, 1) + _rotl(v2, 7) + _rotl(v3, 12) + _rotl(v4, 18)
            for v in (v1, v2, v3, v4):
                h = (h ^ _round(_U(0), v)) * P1 + P4
        else:
            h = np.full(len(p), P5, np.uint64)
        h = h + _U(n)
        if n - i >= 8:
            _bump(cnt, "xxh_tail8", len(p))
        while i + 8 <= n:
            h = h ^ _round(_U(0), words[p + i])
            h = _rotl(h, 27) * P1 + P4
            i += 8
        if i + 4 <= n:
            _bump(cnt, "xxh_tail4", len(p))
            h = h ^ ((words[p + i] & _U(0xFFFFFFFF)) * P1)
            h = _rotl(h, 23) * P2 + P3
            i += 4
        if i < n:
            _bump(cnt, "xxh_tail1", len(p))
        while i < n:
            h = h ^ (a[p + i].astype(np.uint64) * P5)
            h = _rotl(h, 11) * P1
            i += 1
        h = h ^ (h >> _U(33))
        h = h * P2
        h = h ^ (h >> _U(29))
        h = h * P3
        return h ^ (h >> _U(32))


def survivors(src: bytes, prm, sw=frozenset(), cnt=None):
    """steps 1 and 2 on one segment: (positions, values) of the survivors, as zbo_ldm_survivors gives them"""
    mm, n = prm.minMatch, len(src)
    if n < mm:
        return np.zeros(0, np.uint64), np.zeros(0, np.uint64)
    mask = stop_mask(prm)
    a = np.frombuffer(src, np.uint8)
    nbP = n - mm + 1
    # gear hash at the byte that ends every split point; only the bits of the mask matter, so only the terms that reach
    # them (gear[byte i - k] << k for k <= the mask's top bit; carries run upwards only)
    top = mask.bit_length()
    g = GEAR[a[mm - 1:]]
    h = np.zeros(nbP, np.uint64)
    with np.errstate(over="ignore"):
        for k in range(min(top, 64)):
            if k == 0:
                h += g
            else:                                            # byte at index e - k, e = p + mm - 1; e - k >= 0
                lo = max(0, k - (mm - 1))                    # first split point whose byte e - k exists
                if lo >= nbP:
                    break
                h[lo:] += GEAR[a[lo + mm - 1 - k:n - k]] << _U(k)
    fire = np.nonzero((h & _U(mask)) == 0)[0] if mask else np.arange(nbP)
    if prm.hashRateLog == 0:
        _bump(cnt, "hash_rate_0", len(fire))
    if prm.hashRateLog > min(mm, 64):
        _bump(cnt, "mask_low", len(fire))
    padded = np.frombuffer(src + bytes(8), np.uint8)
    words = np.zeros(n, np.uint64)
    for j in range(8):
        words |= padded[j:j + n].astype(np.uint64) << _U(8 * j)
    v = xxh64(padded, words, fire, mm, cnt)
    # thinning: <= every value within mm - 1 on the left, < every value within mm - 1 on the right
    H, F = mm - 1, len(fire)
    ok = np.ones(F, bool)
    tie_l, tie_r, smaller = np.zeros(F, bool), np.zeros(F, bool), np.zeros(F, bool)
    tile_cmp, tile_kill = np.zeros(F, bool), np.zeros(F, bool)
    left_le, right_lt = "thin_left_le" in sw, "thin_right_lt" in sw
    tile = fire // LDM_TILE
    for k in range(1, F):
        w = (fire[k:] - fire[:-k]) <= H                      # pairs (j - k, j) within the window
        if not w.any():
            break
        jl, jr = np.nonzero(w)[0] + k, np.nonzero(w)[0]      # j has j - k on its left; i = j - k has j on its right
        vl, vj = v[jr], v[jl]
        cross = tile[jl] != tile[jr]
        kill_j = (vl <= vj) if left_le else (vl < vj)        # j killed by its left neighbour
        kill_i = (vj < vl) if right_lt else (vj <= vl)       # i killed by its right neighbour
        ok[jl[kill_j]] = False
        ok[jr[kill_i]] = False
        tie_l[jl[vl == vj]] = True
        tie_r[jr[vl == vj]] = True
        smaller[jl[vl < vj]] = True
        smaller[jr[vj < vl]] = True
        tile_cmp[jl[cross]] = True
        tile_cmp[jr[cross]] = True
        tile_kill[jl[cross & kill_j]] = True
        tile_kill[jr[cross & kill_i]] = True
    _bump(cnt, "thin_tie_left_kept", int(np.sum(ok & tie_l)))
    _bump(cnt, "thin_tie_right_dropped", int(np.sum(~ok & tie_r & ~smaller)))
    _bump(cnt, "thin_edge_start", int(np.sum(ok & (fire < H))))
    _bump(cnt, "thin_edge_end", int(np.sum(ok & (fire > nbP - 1 - H))))
    _bump(cnt, "thin_tile_kept", int(np.sum(ok & tile_cmp)))
    _bump(cnt, "thin_tile_dropped", int(np.sum(tile_kill)))
    return fire[ok].astype(np.uint64), v[ok]


# ------------------------------------------------------------------------------------------- steps 3-4
def _bwd(buf, a, b, lim):
    """equal bytes in front of a and of b, at most lim"""
    n, k = 0, 8
    while True:
        if n + k <= lim and buf[a - n - k:a - n] == buf[b - n - k:b - n]:
            n += k
            k = min(k * 2, 1 << 14)
        elif k > 1:
            k //= 2
        else:
            return n


def passes(prm) -> int:
    return (prm.hashLog - prm.bucketSizeLog + 7) // 8


def select(buf: bytes, P: int, pos, v, n: int, window_log: int, prm, sw=frozenset(), cnt=None):
    """steps 3 and 4 for the frame buf[P, P + n) behind P prefix bytes, fed the survivors (pos, v) of both segments in
    [prefix | frame] coordinates: per block of the frame, its matches (start in the block, length, offset)"""
    pos = np.asarray(pos, np.int64)
    v = np.asarray(v, np.uint64)
    N = len(pos)
    bits = prm.hashLog - prm.bucketSizeLog
    bucket = (v & _U((1 << bits) - 1)).astype(np.int64)
    ck = (v >> _U(32)).astype(np.int64)
    order = np.argsort(bucket, kind="stable")
    rank = np.empty(N, np.int64)
    rank[order] = np.arange(N)
    sb = bucket[order]
    run_start = np.zeros(N, np.int64)                        # sorted index where each key's bucket run starts
    if N:
        starts = np.r_[0, np.nonzero(np.diff(sb))[0] + 1]
        run_start = np.repeat(starts, np.diff(np.r_[starts, N]))
    sck, spos = ck[order], pos[order]
    nb_cand = (1 << prm.bucketSizeLog) + (1 if "cand_plus1" in sw else 0)
    W = 1 << window_log
    nb_blocks = (n + BLOCK - 1) // BLOCK
    out = []
    pos_l = pos.tolist()
    i = int(np.searchsorted(pos, P))
    for k in range(nb_blocks):
        bs = P + k * BLOCK
        be = min(bs + BLOCK, P + n)
        anchor, res, last_end = bs, [], bs
        while i < N and pos_l[i] < be:
            p = pos_l[i]
            i += 1
            if p < anchor:
                _bump(cnt, "skip_anchor")
                continue
            r = int(rank[i - 1])
            avail = r - int(run_start[r])
            if avail == 0:
                _bump(cnt, "no_earlier")
            elif avail > nb_cand:
                _bump(cnt, "cand_limit")
            elif run_start[r] > 0:
                _bump(cnt, "walk_bucket_edge")
            else:
                _bump(cnt, "walk_rank")
            walk = min(avail, nb_cand)
            if walk == 0:
                continue
            cs = slice(r - 1, r - 1 - walk if r - 1 - walk >= 0 else None, -1)
            same = sck[cs] == ck[i - 1]
            _bump(cnt, "ck_differs", int(walk - np.count_nonzero(same)))
            qs = spos[cs] if "no_checksum" in sw else spos[cs][same]
            best_len = best_q = best_b = best_f = 0
            low_q = max((p if "lowq_p" in sw else be) - W, 0)
            for q in qs.tolist():
                if q < low_q:
                    if p - q <= W:
                        _bump(cnt, "window_be")
                    continue
                fmax = (P + n if "f_frame_end" in sw else be) - p
                seam = q < P and P - q < fmax
                if seam and "seam_uncapped" not in sw:
                    fmax = P - q
                f = dg._fwd(buf, p, q, p + fmax)
                if f < prm.minMatch:
                    if f == be - p and dg._fwd(buf, p, q, len(buf)) >= prm.minMatch:
                        _bump(cnt, "f_short_cap")
                    continue
                if f == be - p:
                    _bump(cnt, "f_to_be")
                if seam and f == P - q:
                    _bump(cnt, "f_seam")
                if f >= 256:
                    _bump(cnt, "f_256")
                if f < fmax and (f // 8) * 8 + 8 > fmax:
                    _bump(cnt, "f_tail")
                qroom = q if q < P else q - P
                bmax = qroom if "b_no_anchor" in sw else min(p - anchor, qroom)
                b = _bwd(buf, p, q, bmax)
                if b == 0:
                    _bump(cnt, "b_zero")
                if b == p - anchor < qroom and buf[p - b - 1] == buf[q - b - 1]:
                    _bump(cnt, "b_cap_anchor")
                if b == qroom and b > 0:
                    _bump(cnt, "b_cap_q")
                if b >= 32:
                    _bump(cnt, "b_32")
                if f + b > best_len:
                    if best_len:
                        _bump(cnt, "farther_longer")
                    best_len, best_q, best_b, best_f = f + b, q, b, f
                elif f + b == best_len:
                    if "tie_far" in sw:
                        best_q, best_b, best_f = q, b, f
                    else:
                        _bump(cnt, "tie_nearer")
            if not best_len:
                continue
            start = p - best_b
            if start < bs or start + best_len > be:
                _bump(cnt, "ldm_cross_edge")
            if start < last_end:
                _bump(cnt, "ldm_overlap")
            if best_q < P:
                _bump(cnt, "prefix_match")
            res.append((start - bs, best_len, p - best_q))
            last_end = start + best_len
            anchor = p if "anchor_p" in sw else p + best_f
        out.append(res)
    return out


# ------------------------------------------------------------------------------------------- step 5
def _offsets(seqs, reps):
    """the real offsets of a block's final sequences: the repcode history run forward"""
    r1, r2, r3 = reps
    out, pos = [], 0
    for ob, ll, ml in seqs:
        if ob > 3:
            off = ob - 3
            r3, r2, r1 = r2, r1, off
        elif ll > 0:
            if ob == 1:
                off = r1
            elif ob == 2:
                off = r2
                r2, r1 = r1, off
            else:
                off = r3
                r3, r2, r1 = r2, r1, off
        else:
            if ob == 1:
                off = r2
                r2, r1 = r1, off
            elif ob == 2:
                off = r3
                r3, r2, r1 = r2, r1, off
            else:
                off = r1 - 1
                r3, r2, r1 = r2, r1, off
        pos += ll
        out.append((pos, ml, off))
        pos += ml
    return out


def overlay(size: int, reps, lm, seqs, sw=frozenset(), cnt=None):
    """step 5: a block's LDM matches lm [(start, length, offset)] laid over its final parse sequences, repcodes assigned
    again from reps; returns the new sequences (offBase, litLen, matchLen)"""
    P = _offsets(seqs, reps)
    nL = len(lm)
    if len(P) > OVERLAY_ROUND:
        _bump(cnt, "parse_256")
    if nL > OVERLAY_ROUND:
        _bump(cnt, "ldm_256")
    if nL and not P:
        _bump(cnt, "no_parse")
    short = 3 if "keep_short3" in sw else 4
    out, j = [], 0
    for ms0, ml, off in P:
        ms, me = ms0, ms0 + ml
        me0 = me
        cs = ce = False
        while j < nL and lm[j][0] + lm[j][1] <= ms:
            out.append(lm[j] + (True,))
            _bump(cnt, "ldm_before_parse")
            j += 1
        k = j
        if k < nL and (lm[k][0] < ms if "under_strict" in sw else lm[k][0] <= ms):
            if lm[k][0] == ms:
                _bump(cnt, "start_at_ldm_start")
            ms = lm[k][0] + lm[k][1]
            cs = True
            k += 1
        if k < nL and lm[k][0] < me:
            if lm[k][0] + lm[k][1] < me0 and not cs:
                _bump(cnt, "span_whole")
                if "keep_tail" in sw:
                    ms = lm[k][0] + lm[k][1]
                    cs = True
                else:
                    me = lm[k][0]
                    ce = True
            else:
                me = lm[k][0]
                ce = True
        elif k < nL and lm[k][0] == me:
            _bump(cnt, "end_at_ldm_start")
        clipped = cs or ce
        if me <= ms:
            _bump(cnt, "covered")
            continue
        if clipped and me - ms < short:
            _bump(cnt, "clip_both" if cs and ce else ("clip_start_dropped" if cs else "clip_end_dropped"))
            continue
        _bump(cnt, "clip_both" if cs and ce else ("clip_start_kept" if cs else ("clip_end_kept" if ce else "parse_unclipped")))
        if not clipped and me - ms == 3:
            _bump(cnt, "tail3_kept")
        while j < nL and lm[j][0] < ms:
            out.append(lm[j] + (True,))
            j += 1
        out.append((ms, me - ms, off, False))
    out.extend(m + (True,) for m in lm[j:])
    if len(out) > MERGE_TILE:
        _bump(cnt, "merged_1024")
    if len(out) > SEQ_CAP:
        _bump(cnt, "seq_over_cap")
    # zbo_parseBlock's repcode rules; `hist`: which repcodes still hold the block's starting history
    r, hist = list(reps), [True, True, True]
    res, pos = [], 0
    for ms, ml, off, is_ldm in out:
        ll = ms - pos
        if ll > 0:
            cand = [(off == r[0], 0), (off == r[1], 1), (off == r[2], 2)]
        else:
            cand = [(off == r[1], 1), (off == r[2], 2), (r[0] > 1 and off == r[0] - 1, None)]
        hit = next((slot for eq, slot in cand if eq), None)
        if is_ldm and hit is not None and hist[hit] and any(reps):
            _bump(cnt, "rep_from_history")
        if ll > 0:
            if off == r[0]:
                ob = 1
            elif off == r[1]:
                ob = 2
                r = [off, r[0], r[2]]
                hist = [hist[1], hist[0], hist[2]]
            elif off == r[2]:
                ob = 3
                r = [off, r[0], r[1]]
                hist = [hist[2], hist[0], hist[1]]
            else:
                ob = off + 3
                r = [off, r[0], r[1]]
                hist = [False, hist[0], hist[1]]
        else:
            if off == r[1]:
                ob = 1
                r = [off, r[0], r[2]]
                hist = [hist[1], hist[0], hist[2]]
            elif off == r[2]:
                ob = 2
                r = [off, r[0], r[1]]
                hist = [hist[2], hist[0], hist[1]]
            elif r[0] > 1 and off == r[0] - 1:
                ob = 3
                r = [off, r[0], r[1]]
                hist = [False, hist[0], hist[1]]
            else:
                ob = off + 3
                r = [off, r[0], r[1]]
                hist = [False, hist[0], hist[1]]
        res.append((ob, ll, ml))
        pos = ms + ml
    return res


# -------------------------------------------------------------------------------------------------- inputs
def dense(n: int, seed: int) -> bytes:
    """versions of one 96 KiB text, each with an edit every ~100 bytes: blocks with many short LDM matches among parse
    matches, which the LDM matches clip.  In front: 4000 random bytes twice"""
    rnd = random.Random(seed)
    cur = bytearray(zref.synthetic(96 << 10, seed=seed))
    r = zref.random_bytes(4000, seed=seed)
    out = bytearray(r + r)                                   # the first block's first sequence: an LDM match at offset 4000
    while len(out) < n:
        out += cur
        for _ in range(len(cur) // 100):
            at = rnd.randrange(len(cur))
            cur[at:at + 1] = bytes([rnd.randrange(256)]) if rnd.random() < 0.8 else b""
    return bytes(out[:n])


def gadgets(n: int, seed: int) -> bytes:
    """a frame of n bytes (> 1 MiB) of synthetic text with copies aimed at the selection's edges: copies against block
    edges and across them, copies of the frame's first bytes, a copy whose backward count reaches the previous match
    (the anchor), content at two earlier places (equal extensions: a tie; one extending further), content repeated more
    than 8 times, a short period (ties in the thinning), and a 160 KiB random piece copied from 1 MiB back (a block
    with no parse match)"""
    rnd = random.Random(seed)
    head = zref.random_bytes(4096, seed=seed)
    far = zref.random_bytes(160 << 10, seed=seed + 1)
    out = bytearray(head + far + zref.synthetic(CHUNK - len(head) - len(far), seed=seed + 2))
    srcs = [rnd.randrange(4096, len(out) - 8192) for _ in range(40)]

    def fill_to(x):
        if x > len(out):
            out.extend(zref.synthetic(x - len(out), seed=rnd.randrange(1 << 30)))

    # ties and a farther, longer place
    u = zref.random_bytes(3000, seed=seed + 3)
    out += u + b"tie-one" + zref.random_bytes(500, seed=seed + 4) + u + b"tie-two" + zref.random_bytes(500, seed=seed + 5)
    out += u + b"tie-" + zref.random_bytes(2000, seed=seed + 6)           # both places extend 4 bytes: a tie
    long_tail = zref.random_bytes(800, seed=seed + 7)
    out += u + long_tail + zref.random_bytes(300, seed=seed + 8)         # the farther place extends further
    out += u + b"tie-" + zref.random_bytes(600, seed=seed + 9)
    out += u + long_tail[:400] + zref.random_bytes(300, seed=seed + 10)
    # the anchor: U then W, copied from U + junk and from (U's tail + W)
    U, Wd = zref.random_bytes(2000, seed=seed + 11), zref.random_bytes(2000, seed=seed + 12)
    out += U + zref.random_bytes(300, seed=seed + 13) + U[-900:] + Wd + zref.random_bytes(300, seed=seed + 14)
    out += zref.random_bytes(100, seed=seed + 15) + U + Wd + zref.random_bytes(100, seed=seed + 16)
    # content repeated 12 times, with random bytes between
    rep = zref.random_bytes(700, seed=seed + 17)
    for t in range(12):
        out += rep + zref.random_bytes(50 + t, seed=seed + 18 + t)
    # a short period: equal hash values a few bytes apart
    out += (zref.random_bytes(7, seed=seed + 40) * 600)
    # copies against block edges: ending exactly at one, starting exactly at one, across one
    for blk in range(len(out) // BLOCK + 1, n // BLOCK - 2):
        edge = blk * BLOCK
        kind = blk % 3
        L = rnd.choice([70, 300, 1500, 5000])
        s = rnd.choice(srcs)
        at = edge - L if kind == 0 else (edge if kind == 1 else edge - L // 2)
        fill_to(at)
        del out[at:]
        out += out[s:s + L]
        fill_to(edge + BLOCK // 3)
        del out[edge + BLOCK // 3:]
        out += out[rnd.choice(srcs):][:rnd.choice([40, 64, 65, 200])]      # short ones: f near minMatch
        fill_to(edge + BLOCK // 2)                           # the frame's first bytes in the middle of the block
        del out[edge + BLOCK // 2:]
        out += head[:rnd.choice([64, 100, 3000])]
    # a block's worth of the far piece, 1 MiB behind its copy, on a block edge
    at = ((len(out) + BLOCK - 1) // BLOCK) * BLOCK
    fill_to(at)
    del out[at:]
    out += far
    fill_to(n)
    del out[n:]
    out[n - 3000:n] = out[4096 - 1000:4096 + 2000]                         # the frame's last block ends in a copy
    return bytes(out)


def window_frame() -> bytes:
    """a frame of 136 MiB, zeros but for random pieces and their copies around the window limit (W = 2^27).  Piece 0 lies
    1 MiB into the frame and its copy in the block that ends exactly W behind it: every source is inside the window.
    Pieces 1-4 lie 2, 3, 4 and 5 MiB into the frame, each copied W - 1000 bytes behind it: p - q <= W for every survivor
    of a copy, but q < be - W for those more than 1000 bytes before their block's end, so their blocks refuse them"""
    W = 1 << 27
    n = 136 << 20
    out = bytearray(n)
    for i in range(5):
        piece = zref.random_bytes(40 << 10, seed=61 + i)
        src_at = (1 + i) << 20
        out[src_at:src_at + len(piece)] = piece
        at = ((src_at + W) // BLOCK - 1) * BLOCK + 1000 if i == 0 else src_at + W - 1000
        out[at:at + len(piece)] = piece
    return bytes(out)


_cache = {}


def _c(key, fn):
    if key not in _cache:
        _cache[key] = fn()
    return _cache[key]


def frame_inputs():
    """name -> frame bytes (each > 512 KiB): the frames whose LDM steps 1-5 the restatement follows"""
    return _c("frames", lambda: {
        "dense": dense(1 << 20, 71),
        "gadgets": gadgets(1536 << 10, 72),
        "b512k1": dense(CHUNK + 1, 73),                                    # last block of 1 byte (raw)
        "tail5": gadgets(5 * BLOCK + 5, 74),                               # last block of 5 bytes (raw)
        "tail300": gadgets(5 * BLOCK + 300, 75),                           # last block: 300 bytes copied from 640 KiB back
    })


# (name, ldm parameters): the pass counts 0-4 of the bucket sort, minMatch 4, 37, 300 and 4096, hashRateLog 0, and the
# stop mask in the low bits.  hash_log 24 is above the window of these frames: hashRateLog resolves to 0 (every split
# point fires; with a large minMatch the thinning would then cost O(splits x minMatch), so those sets keep a rate).
PARAMS = [
    ("default", {}),
    ("passes0", dict(hash_log=8, bucket_size_log=8, hash_rate_log=4)),
    ("passes1", dict(hash_log=11)),
    ("passes2", dict(hash_log=12)),
    ("passes3", dict(hash_log=20, hash_rate_log=7)),
    ("passes4", dict(hash_log=30, bucket_size_log=1, hash_rate_log=7)),
    ("mm4", dict(min_match=4)),
    ("mm4_hr8", dict(min_match=4, hash_rate_log=8)),
    ("mm4_hr0", dict(min_match=4, hash_log=24)),
    ("mm37", dict(min_match=37)),
    ("mm300", dict(min_match=300, hash_rate_log=5)),
    ("mm4096", dict(min_match=4096, hash_rate_log=6)),
]
PASSES = {"passes0": 0, "passes1": 1, "passes2": 2, "passes3": 3, "passes4": 4}
ALL_PARAM_FRAMES = ("dense", "gadgets")        # every parameter set; the other frames run the defaults
PREFIX_PAIRS = ("prefix100k", "small_frame_ldm")


def cases():
    """(name, prefix, frame, level, ldm parameters) of every frame the restatement follows: each frame input with the
    default parameters, the two main ones with every set, and two prefix pairs"""
    def build():
        out = []
        for name, src in frame_inputs().items():
            for pname, prm in PARAMS:
                if pname == "default" or name in ALL_PARAM_FRAMES:
                    out.append((f"{name}/{pname}", b"", src, 1, prm))
        pairs = prefixref.pairs()
        for name in PREFIX_PAIRS:
            pfx, src = pairs[name]
            out.append((f"{name}/default", prefixref.indexed(pfx), src, 1, {}))
            out.append((f"{name}/mm37", prefixref.indexed(pfx), src, 1, dict(min_match=37)))
        return out
    return _c("cases", build)


def window_log(P: int, n: int) -> int:
    return prefixref.window_log(n, P)


def resolved(P: int, n: int, prm: dict):
    return ldmref.resolve(window_log(P, n), **prm)


def oracle_lists(P_bytes: bytes, src: bytes, prm: dict):
    """the oracle's per-block match lists (zbo_ldm_frame, or zbo_ldm_frame_usingPrefix behind a prefix)"""
    if not P_bytes:
        return ldmref.frame_lists(src, window_log(0, len(src)), **prm)
    L = prefixref.lists(src, P_bytes, window_log(len(P_bytes), len(src)), **prm)
    P = len(P_bytes)
    per = [[] for _ in range((len(src) + BLOCK - 1) // BLOCK)]
    for p, ln, off in L["matches"]:
        k = (p - P) // BLOCK
        per[k].append((p - P - k * BLOCK, ln, off))
    return per


def raw_frame(n: int, seed: int) -> bytes:
    """random bytes with a 300-byte copy from 512 KiB back in every block: LDM matches in blocks that stay raw (the copy
    saves less than the block's minimum gain)"""
    rnd = random.Random(seed)
    out = bytearray(zref.random_bytes(n, seed=seed))
    for bs in range(CHUNK, n - BLOCK + 1, BLOCK):
        at = bs + rnd.randrange(1000, BLOCK - 1000)
        out[at:at + 300] = out[at - CHUNK:at - CHUNK + 300]
    return bytes(out)


def survivor_count_frame(base: bytes, count: int, prm: dict) -> bytes:
    """the shortest prefix of base whose survivors number exactly `count` (a radix tile holds 4096 keys), at the window
    of that length"""
    lo, hi = 1, len(base)
    def n_surv(m):
        return len(ldmref.survivors(base[:m], resolved(0, m, prm)))
    assert n_surv(hi) >= count
    while lo < hi:                                           # the shortest prefix with at least `count` survivors
        mid = (lo + hi) // 2
        if n_surv(mid) >= count:
            hi = mid
        else:
            lo = mid + 1
    assert n_surv(lo) == count, (count, n_surv(lo))
    return base[:lo]


def harness_cases():
    """(name, prefix (indexed bytes), frame, ldm parameters) of every launch the harness test compares with the oracle's
    lists: the restatement's cases, the window frame, every prefix pair, the reference inputs of the LDM tests, frames
    whose split points end exactly on and one past an L1 tile (4096 split points), frames whose survivors fill whole
    radix tiles (4096 keys) and one key more, small frames, and frames whose blocks stay raw"""
    def build():
        out = [(name, pfx, src, prm) for name, pfx, src, _, prm in cases()]
        out.append(("window/default", b"", window_frame(), {}))
        for name, (pfx, src) in prefixref.pairs().items():
            if src:
                out.append((f"pair-{name}/default", prefixref.indexed(pfx), src, {}))
        for name, src in ldmref.inputs().items():
            out.append((f"ldm-{name}/default", b"", src, {}))
        d = dense(3 << 20, 76)
        for mm in (64, 300):
            for k in (100, 257):
                for extra in (0, 1):
                    n = k * LDM_TILE + mm - 1 + extra                # n - mm + 1 split points: k tiles, or one split more
                    out.append((f"tile{k}+{extra}/mm{mm}", b"", d[:n], dict(min_match=mm)))
                    out.append((f"ptile{k}+{extra}/mm{mm}", d[-n:], d[:1 << 20], dict(min_match=mm)))
        for count in (2 * 4096, 2 * 4096 + 1, 3 * 4096 - 1):
            f = survivor_count_frame(d, count, {})
            out.append((f"radix{count}/default", b"", f, {}))
        for n in (64, 1000, 4159, BLOCK + 7, 3 * BLOCK):
            out.append((f"small{n}/mm4", b"", d[:n], dict(min_match=4)))
        out.append(("raw/default", b"", raw_frame(1 << 20, 77), {}))
        return out
    return _c("harness", build)


def oracle_survivors(P_bytes: bytes, src: bytes, prm):
    """the oracle's survivors of both segments in [prefix | frame] coordinates"""
    pp, pv = ldmref.survivors_v(P_bytes, prm) if P_bytes else (np.zeros(0, np.uint64), np.zeros(0, np.uint64))
    fp, fv = ldmref.survivors_v(src, prm)
    return np.concatenate([pp, fp + np.uint64(len(P_bytes))]), np.concatenate([pv, fv])
