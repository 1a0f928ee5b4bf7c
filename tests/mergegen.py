"""The merge (K1c: zb_merge_segments_kernel / zb_merge_small_kernel in zstd_b200/csrc/zb_match.cu, zb_merge_codes in
zb_merge.cuh) restated in Python, chosen raw sequences that reach each of its paths, and wrong-rule switches.
TEST INFRASTRUCTURE ONLY.

join() is the oracle's serial loop (zbo_parseBlock, oracle/zb_match.c): the segments' raw sequences joined over the block
and the repcodes assigned; dfastgen.parse_block calls it, so the CPU tests that hold the doubleFast and fast parses equal
to zbo_parseBlock hold this code equal to it too.  The literal bytes and the meta follow from the block; with long-distance
matches the expectation is ldmgen.overlay of the joined sequences (held equal to zbo_ldm_overlayBlock elsewhere).

analyse() counts the path rows of one block while the expectation is computed: the seams of the join, the repcode outcome
at every index class the kernel's scans treat apart (thread, warp and tile edges), the literal gather's groups, the small
kernel's rounds of 32 and the LDM overlay's clips.  Raw inputs follow the parse's guarantees (check_raw); K1c never reads a
match's source bytes, so offsets are any value of the raw format's 24-bit field."""
import random

SEG = 16 << 10
BLOCK = 128 << 10
SEGS = BLOCK // SEG
SEG_SLOTS = SEG // 4              # raw sequences a segment may hold
TILE = 1024                       # sequences per round of zb_merge_codes
SMALL_ROW = 8192                  # rows of at most this many bytes (one segment) take zb_merge_small_kernel
OFF_MAX = (1 << 24) - 1           # the raw format's offset field
SEQ_OFF_MAX = (1 << 24) - 4       # the largest offset a sequence call accepts (ZB_SEQ_OFF_MAX)

OUTCOMES = ["p1", "p2", "p3", "pfull", "z1", "z2", "z3", "zfull"]     # p: litLength > 0, z: litLength = 0; code 1/2/3/full
INDEX_CLASSES = [f"mod{k}" for k in range(4)] + [f"at{i}" for i in (127, 128, 1023, 1024, 1025, 2047, 2048)]

ROWS = [
    # the join
    "raw_before_cur",      # a raw sequence that ends before cur (dropped)
    "raw_at_cur",          # one that ends exactly at cur (dropped)
    "tail1", "tail2",      # straddles cur with a tail of 1 / 2 bytes (dropped)
    "tail3",               # ... of 3 bytes (kept: the shortest match K1c emits)
    "tail_long",           # ... of more than 3 bytes (kept, trimmed)
    "ms_eq_cur",           # a survivor that starts at cur (litLength 0) after an earlier segment's match
    "seg_empty",           # a segment without raw sequences
    "seg_all_dropped",     # a segment whose every raw sequence is dropped (f == n > 0)
    "first_after_drops",   # a first survivor behind drops (f > 0)
    "seg_under_match",     # a segment that lies entirely under one match of an earlier segment
    "seg0_to_block_end",   # a match of segment 0 that runs to the end of a block of several segments
    "cur_from_pm",         # cur after a segment from its trimmed first survivor (f == n - 1)
    "cur_from_last",       # cur after a segment from its last raw sequence (f < n - 1)
    "surv_1", "surv_255", "surv_256", "surv_257", "surv_4096",    # survivors of one segment
    "last_seg_1byte",      # a block whose last segment is 1 byte (16385 bytes)
    # the repcode history
    *[f"{o}_{c}" for o in OUTCOMES for c in INDEX_CLASSES],
    "zfull_off_r1",        # litLength 0, full code, offset == r1
    "zfull_r1_is_1",       # litLength 0, r1 == 1, offset 0 (= r1 - 1, which must not be used)
    "handover_U", "handover_swap", "handover_rep", "handover_full",   # a tile's last sequence (with a tile behind it)
    "hist_148", "hist_3_17_4099", "hist_1_x_y", "hist_none",        # the history a block starts from
    "nbseq_1024", "nbseq_1025", "nbseq_32768",
    # the literal gather
    *[f"run_start_mod{k}" for k in range(8)], *[f"run_end_mod{k}" for k in range(8)],
    "zero_run_group_edge", # a zero-length run at a group edge (literal offset = 0 mod 8, inside the block's literals)
    "eight_runs_one_group",# 8 one-byte runs in one group of 8
    "tile_lit_unaligned",  # a tile after the first whose first literal is not 8-aligned
    "only_literals",       # a block without sequences
    "no_trailing",         # a block whose last match ends at its end
    "run_100k",            # a literal run of 100 KiB or more
    # the small kernel's rounds of 32 (rows of at most 8192 bytes)
    "small_31", "small_32", "small_33", "small_64", "small_65",
    # the LDM overlay
    "ldm_clip_start",      # a parse match that starts under an LDM match
    "ldm_clip_end",        # a parse match that runs into an LDM match
    "ldm_left4", "ldm_left3",   # a clipped parse match left with 4 bytes (kept) / 3 (dropped)
    "ldm_tail3_unclipped", # an unclipped 3-byte join tail (kept)
    "ldm_before_first", "ldm_after_last",   # LDM matches before the first / after the last parse match
    "ldm_nP_256", "ldm_nP_1024", "ldm_nL_256", "ldm_nL_1024",
    "ldm_nL_0",            # a block without LDM matches in an LDM launch
    "ldm_only",            # a block with LDM matches and no parse match
]
# the two expressions of cur after a segment (kernel: pm + pl when f == n - 1, else the last raw's end) never differ
ZERO_ROWS = ["cur_exprs_differ"]

SWITCHES = {
    "keep_tail4": "a straddling sequence is kept only with a tail of >= 4 bytes",
    "keep_tail2": "a straddling sequence is kept with a tail of >= 2 bytes",
    "ll0_as_llpos": "litLength 0 coded like litLength > 0",
    "first_reps_all": "every block starts from {1,4,8} (or the dictionary's repcodes), not only a frame's first",
    "reset_per_tile": "the history starts again from the block's at every tile of 1024 sequences",
    "handover_prevoff": "a tile's last sequence, U (litLength > 0, repeats r1), hands over r2 = its r1 instead of its r2",
    "lits_untrimmed": "a trimmed match's literals counted from its untrimmed start",
}
# wrong rules that no input can tell from the rule; the CPU tests prove each changes nothing on every block
EQUIVALENT = {
    "drop_lt": "drop only when ms + ml < cur: a sequence that ends at cur straddles with a tail of 0 and is dropped anyway",
    "r1m1_for_r1_1": "r1 - 1 allowed when r1 == 1: the offset 0 it matches gets code 3 and the history (0, 1, r2) either way",
}


def _bump(c, k, n=1):
    if c is not None:
        c[k] = c.get(k, 0) + n


def code(reps, off, ll, sw=frozenset()):
    """ZSTD_storeSeq's repcode rule: (offBase, new history)"""
    r1, r2, r3 = reps
    if ll > 0 or "ll0_as_llpos" in sw:
        if off == r1:
            return 1, (r1, r2, r3)
        if off == r2:
            return 2, (off, r1, r3)
        if off == r3:
            return 3, (off, r1, r2)
    else:
        if off == r2:
            return 1, (off, r1, r3)
        if off == r3:
            return 2, (off, r1, r2)
        if (r1 > 0 if "r1m1_for_r1_1" in sw else r1 > 1) and off == r1 - 1:
            return 3, (off, r1, r2)
    return off + 3, (off, r1, r2)


def join(segments, reps, base=0, sw=frozenset(), cnt=None, rows=None, size=None):
    """zbo_parseBlock's join and repcodes: segments[k] = segment k's raw sequences [(ms, mlen, off)] at positions base + ...;
    returns the block's sequences [(offBase, litLength, matchLength)].  cnt gets join_drop / join_trim (the parse tests'
    rows), rows the merge rows of the join and the history (size: the block's size, for the segment rows)."""
    cur, seqs = base, []
    first = tuple(reps)
    r = first
    tail_min = 4 if "keep_tail4" in sw else 2 if "keep_tail2" in sw else 3
    for k, seg in enumerate(segments):
        if rows is not None and size is not None:
            seg_hi = base + min((k + 1) * SEG, size)
            if not seg:
                _bump(rows, "seg_empty")
            if k > 0 and cur >= seg_hi:
                _bump(rows, "seg_under_match")
        f, kept = 0, 0
        for ms, mlen, off in seg:
            if (ms + mlen < cur) if "drop_lt" in sw else (ms + mlen <= cur):
                _bump(cnt, "join_drop")
                _bump(rows, "raw_before_cur" if ms + mlen < cur else "raw_at_cur")
                f += kept == 0
                continue
            lit_from = None
            if ms < cur:
                tail = ms + mlen - cur
                if tail < tail_min:
                    _bump(cnt, "join_drop")
                    _bump(rows, f"tail{tail}" if tail in (1, 2) else "raw_at_cur")
                    f += kept == 0
                    continue
                _bump(cnt, "join_trim")
                _bump(rows, "tail3" if tail == 3 else "tail_long")
                if "lits_untrimmed" in sw:
                    lit_from = ms
                mlen, ms = tail, cur
            elif ms == cur and k > 0 and kept == 0 and seqs:
                _bump(rows, "ms_eq_cur")
            ll = ms - cur if lit_from is None else lit_from - cur
            i = len(seqs)
            if i and i % TILE == 0 and "reset_per_tile" in sw:
                r = first
            ob, nr = code(r, off, ll, sw)
            if rows is not None:
                _history_rows(rows, r, off, ll, ob, i)
            if "handover_prevoff" in sw and i % TILE == TILE - 1 and ll > 0 and off == r[0]:
                nr = (nr[0], r[0], r[2])
            r = nr
            seqs.append((ob, ll, mlen))
            cur = ms + mlen
            kept += 1
        if rows is not None:
            n = len(seg)
            if n and f == n:
                _bump(rows, "seg_all_dropped")
            if f and f < n:
                _bump(rows, "first_after_drops")
            if kept:
                _bump(rows, f"surv_{kept}")
                lm, lml, _ = seg[-1]
                # the kernel's cur: the trimmed first survivor's end when it is the segment's last raw, else the last raw's end
                kern = (cur if f == n - 1 else lm + lml)
                _bump(rows, "cur_from_pm" if f == n - 1 else "cur_from_last")
                if kern != cur:
                    _bump(rows, "cur_exprs_differ")
                if k == 0 and size is not None and size > SEG and cur == base + size:
                    _bump(rows, "seg0_to_block_end")
    return seqs


def _history_rows(rows, r, off, ll, ob, i):
    o = ("p" if ll > 0 else "z") + (str(ob) if ob <= 3 else "full")
    if ll == 0 and r[0] == 1 and off == 0 and off not in r[1:]:
        o = "zfull"                                                # offBase 3 by the full code: off + 3
    _bump(rows, f"{o}_mod{i % 4}")
    if i in (127, 128, 1023, 1024, 1025, 2047, 2048):
        _bump(rows, f"{o}_at{i}")
    if o == "zfull" and off == r[0]:
        _bump(rows, "zfull_off_r1")
    if o == "zfull" and r[0] == 1 and off == 0:
        _bump(rows, "zfull_r1_is_1")


def literals(block: bytes, seqs):
    """the block's literal bytes: every run in front of a match, then the trailing run"""
    out, pos = bytearray(), 0
    for _, ll, ml in seqs:
        out += block[pos:pos + ll]
        pos += ll + ml
    return bytes(out + block[pos:])


def analyse(rows, block: bytes, seqs, reps, first: bool, small_row: bool):
    """the rows that follow from a block's final sequences: hand-over forms, history, counts, gather groups, small rounds"""
    n = len(seqs)
    if first:
        _bump(rows, {(1, 4, 8): "hist_148", (3, 17, 4099): "hist_3_17_4099"}.get(tuple(reps), "hist_1_x_y" if reps[0] == 1 else "hist_other"))
    else:
        _bump(rows, "hist_none")
    if n in (1024, 1025, 32768):
        _bump(rows, f"nbseq_{n}")
    if small_row and n in (31, 32, 33, 64, 65):
        _bump(rows, f"small_{n}")
    if n == 0:
        _bump(rows, "only_literals")
    if len(block) > SEG and len(block) % SEG == 1:
        _bump(rows, "last_seg_1byte")
    # hand-over: forms of every tile's last sequence with a tile behind it (the history replayed)
    r = tuple(reps) if first else (0, 0, 0)
    for i, (ob, ll, ml) in enumerate(seqs):
        off = _offset(r, ob, ll)
        if i % TILE == TILE - 1 and i + 1 < n:
            if ll > 0 and off == r[0]:
                _bump(rows, "handover_U")
            elif off == r[1]:
                _bump(rows, "handover_swap")
            elif ob <= 3:
                _bump(rows, "handover_rep")
            else:
                _bump(rows, "handover_full")
        _, r = code(r, off, ll)
    # the gather: literal runs in buffer offsets
    pos = lit = 0
    starts = []
    for i, (ob, ll, ml) in enumerate(seqs):
        starts.append((lit, ll))
        if ll:
            _bump(rows, f"run_start_mod{lit % 8}")
            _bump(rows, f"run_end_mod{(lit + ll) % 8}")
        if ll >= 100 << 10:
            _bump(rows, "run_100k")
        if i % TILE == 0 and i and lit % 8:
            _bump(rows, "tile_lit_unaligned")
        lit += ll
        pos += ll + ml
    total = lit + len(block) - pos
    if n and pos == len(block):
        _bump(rows, "no_trailing")
    for j, (s, ll) in enumerate(starts):
        if ll == 0 and s % 8 == 0 and s < total and 0 < j:
            _bump(rows, "zero_run_group_edge")
    ones = {}
    for s, ll in starts:
        if ll == 1:
            ones[s // 8] = ones.get(s // 8, 0) + 1
    if any(v == 8 for v in ones.values()):
        _bump(rows, "eight_runs_one_group")


def _offset(r, ob, ll):
    if ob > 3:
        return ob - 3
    if ll > 0:
        return r[ob - 1]
    return (r[1], r[2], r[0] - 1)[ob - 1]


def ldm_rows(rows, seqs, reps, lm):
    """the overlay's rows for one block: lm [(start, length, offset)], seqs the joined sequences"""
    P, pos = [], 0
    r = tuple(reps)
    for ob, ll, ml in seqs:
        off = _offset(r, ob, ll)
        _, r = code(r, off, ll)
        P.append((pos + ll, pos + ll + ml))
        pos += ll + ml
    nP, nL = len(P), len(lm)
    if not nL:
        _bump(rows, "ldm_nL_0")
    if nL and not nP:
        _bump(rows, "ldm_only")
    for k, lim in ((256, "256"), (1024, "1024")):
        if nP > k:
            _bump(rows, f"ldm_nP_{lim}")
        if nL > k:
            _bump(rows, f"ldm_nL_{lim}")
    if nP and nL:
        if lm[0][0] + lm[0][1] <= P[0][0]:
            _bump(rows, "ldm_before_first")
        if lm[-1][0] >= P[-1][1]:
            _bump(rows, "ldm_after_last")
    starts = [s for s, _, _ in lm]
    import bisect
    for ms, me in P:
        lo = bisect.bisect_right(starts, ms)
        clipped = False
        if lo and lm[lo - 1][0] + lm[lo - 1][1] > ms:
            ms = lm[lo - 1][0] + lm[lo - 1][1]
            clipped = True
            _bump(rows, "ldm_clip_start")
        if lo < nL and lm[lo][0] < me:
            me = lm[lo][0]
            clipped = True
            _bump(rows, "ldm_clip_end")
        if clipped and me - ms == 4:
            _bump(rows, "ldm_left4")
        if clipped and me - ms == 3:
            _bump(rows, "ldm_left3")
        if not clipped and me - ms == 3:
            _bump(rows, "ldm_tail3_unclipped")


# ------------------------------------------------------------------------------------------------------- the blocks
class Blk:
    """one block of a launch: its bytes, FIRST flag and starting history (reps of a first block: its dictionary slot's
    codeRep), the raw sequences of each of its segments (block-relative), and its LDM matches (None: no LDM launch)"""
    def __init__(self, data: bytes, segs, first=False, reps=(1, 4, 8), ldm=None, name=""):
        self.data, self.segs, self.first, self.reps, self.ldm, self.name = data, segs, first, tuple(reps), ldm, name
        check_raw(len(data), segs)

    @property
    def size(self):
        return len(self.data)

    def start_reps(self, sw=frozenset()):
        return self.reps if (self.first or "first_reps_all" in sw) else (0, 0, 0)

    def expect(self, sw=frozenset(), rows=None, small_row=False):
        """(sequences, literals) K1c must leave; rows: the path rows"""
        reps = self.start_reps(sw)
        seqs = join(self.segs, reps, 0, sw, None, rows, self.size)
        if rows is not None:
            analyse(rows, self.data, seqs, self.reps, self.first, small_row)
        if self.ldm is not None:
            import ldmgen
            if rows is not None:
                ldm_rows(rows, seqs, reps, self.ldm)
            seqs = ldmgen.overlay(self.size, reps, list(self.ldm), seqs)
        return seqs, literals(self.data, seqs)


def check_raw(size, segs):
    """the parse's guarantees: per segment, raw sequences start in it, are sorted, do not overlap, have >= 4 bytes, end
    inside the block and number at most 4096; offsets fit 24 bits"""
    nseg = (size + SEG - 1) // SEG
    assert len(segs) <= max(1, nseg) and all(not s for s in segs[nseg:])
    for k, seg in enumerate(segs):
        assert len(seg) <= SEG_SLOTS, f"segment {k}: {len(seg)} raw sequences"
        end = k * SEG
        for ms, ml, off in seg:
            assert k * SEG <= ms < min((k + 1) * SEG, size), f"segment {k}: a raw sequence starts at {ms}"
            assert ms >= end and ml >= 4 and ms + ml <= size and 0 <= off <= OFF_MAX, (k, ms, ml, off, end)
            end = ms + ml


def _pick(rnd, r, want, ll):
    """an offset that gives outcome `want` with litLength ll from history r, or None"""
    r1, r2, r3 = r
    if want == "p1":
        return r1 if r1 else None
    if want == "p2":
        return r2 if r2 and r2 != r1 else None
    if want == "p3":
        return r3 if r3 and r3 not in (r1, r2) else None
    if want == "z1":
        return r2 if r2 else None
    if want == "z2":
        return r3 if r3 and r3 != r2 else None
    if want == "z3":
        return r1 - 1 if r1 > 1 and r1 - 1 not in (r2, r3) else None
    if want == "zfull" and r1 and r1 not in (r2, r3) and rnd.random() < 0.3:
        return r1                                                  # the full code with offset == r1
    while True:
        off = rnd.choice([rnd.randint(1, 64), rnd.randint(1, 70000), rnd.randint(1, SEQ_OFF_MAX), SEQ_OFF_MAX, SEQ_OFF_MAX - 1])
        if off not in (r1, r2, r3) and off != r1 - 1:
            return off


def scripted(rnd, n, force=None, reps=(0, 0, 0), ll_max=7, ml_range=(4, 9)):
    """n sequences as [(litLength, matchLength, offset)]: outcome force[i] at index i where it can be had from the history,
    random outcomes elsewhere"""
    force = force or {}
    out, r = [], tuple(reps)
    for i in range(n):
        want = force.get(i) or rnd.choice(OUTCOMES)
        ll = 0 if want[0] == "z" else rnd.randint(1, ll_max)
        off = _pick(rnd, r, want, ll)
        if off is None:
            want = "pfull" if ll else "zfull"
            off = _pick(rnd, r, want, ll)
        ml = rnd.randint(*ml_range)
        out.append((ll, ml, off))
        _, r = code(r, off, ll)
    return out


def lay(seqs, start=0):
    """[(ll, ml, off)] laid out from `start`: raw [(ms, ml, off)] and the end"""
    raw, pos = [], start
    for ll, ml, off in seqs:
        raw.append((pos + ll, ml, off))
        pos += ll + ml
    return raw, pos


def split(raw, size):
    """raw sequences of a block to its segments by start"""
    segs = [[] for _ in range(max(1, (size + SEG - 1) // SEG))]
    for t in raw:
        segs[t[0] // SEG].append(t)
    return segs


def _bytes(rnd, n):
    return rnd.randbytes(n)


def codes_blocks():
    """the history cases: one block per outcome forced at the thread, warp and tile edges, blocks of 1024 / 1025 sequences,
    histories {1,4,8}, (3,17,4099), (1,x,y) and none, and 32768 sequences of 4 bytes in a 128 KiB block"""
    rnd = random.Random(11)
    out = []
    at = (127, 128, 1023, 1024, 1025, 2047, 2048)
    for k, o in enumerate(OUTCOMES):
        reps = [(1, 4, 8), (3, 17, 4099), (1, 700, 90000), (0, 0, 0)][k % 4]
        first = k % 4 != 3
        seqs = scripted(rnd, 2100 + k, {i: o for i in at}, reps if first else (0, 0, 0), ll_max=3, ml_range=(4, 6))
        raw, end = lay(seqs)
        size = min(BLOCK, end + rnd.randint(0, 9))
        out.append(Blk(_bytes(rnd, size), split(raw, size), first, reps if first else (1, 4, 8), name=f"codes_{o}"))
    for n, reps in ((1024, (1, 4, 8)), (1025, (3, 17, 4099)), (1023, (1, 2, 3))):
        seqs = scripted(rnd, n, {}, reps, ll_max=12)
        raw, end = lay(seqs, rnd.randint(0, 5))
        out.append(Blk(_bytes(rnd, end + 3), split(raw, end + 3), True, reps, name=f"nbseq_{n}"))
    # r1 == 1, litLength 0, offset 0: the r1 - 1 the rule must not take
    raw = [(5, 4, 1), (9, 4, 0), (20, 4, 1), (24, 5, 0), (40, 4, 7)]
    out.append(Blk(_bytes(rnd, 60), [raw], True, (1, 4, 8), name="r1_is_1"))
    # 32768 matches of 4 bytes, litLength 0: every segment full (4096 survivors each)
    seqs = [(0, 4, o) for o in _z_offsets(rnd, BLOCK // 4, (1, 4, 8))]
    raw, _ = lay(seqs)
    out.append(Blk(_bytes(rnd, BLOCK), split(raw, BLOCK), True, (1, 4, 8), name="full_4096"))
    return out


def _z_offsets(rnd, n, reps):
    """offsets of n litLength-0 sequences with random litLength-0 outcomes"""
    out, r = [], tuple(reps)
    for _ in range(n):
        want = rnd.choice(["z1", "z2", "z3", "zfull"])
        off = _pick(rnd, r, want, 0) or _pick(rnd, r, "zfull", 0)
        out.append(off)
        _, r = code(r, off, 0)
    return out


def _seam_block(rnd, name, scenarios, size=BLOCK, first=False):
    """a block whose segment k + 1 opens with scenarios[k] against the match that segment k ends with"""
    segs = [[] for _ in range((size + SEG - 1) // SEG)]
    cur = 0
    for k in range(len(segs)):
        lo, hi = k * SEG, min((k + 1) * SEG, size)
        sc = scenarios[k - 1] if 0 < k <= len(scenarios) else None
        pos = max(cur, lo)
        seg = segs[k]
        if sc == "empty":
            continue
        if sc is not None and cur > lo:
            over = cur - lo                                         # bytes of this segment under the last match (12 .. 40)
            off = rnd.randint(1, 999)
            if sc == "before":
                seg.append((lo, over - 1, off))
            elif sc == "at":
                seg.append((lo, over, off))
            elif sc in ("t1", "t2", "t3", "t7"):
                seg.append((lo, over + int(sc[1]), off))
            elif sc == "eq":
                seg.append((cur, 4, off))
            elif sc == "drops_then_eq":                            # two drops, then a first survivor at cur (f = 2)
                seg += [(lo, 4, off), (lo + 4, over - 4 + 1, off + 1), (cur + 1, 5, off + 2)]
            pos = max(cur, seg[-1][0] + seg[-1][1])
        # fill the rest of the segment, ending with a match that runs over into the next one
        while pos + 40 < hi:
            ll = rnd.randint(0, 6)
            ml = rnd.randint(4, 12)
            seg.append((pos + ll, ml, rnd.randint(1, 70000)))
            pos += ll + ml
        if pos + 4 < hi and hi < size:
            ms = pos + 1
            ml = min(size - ms, hi - ms + rnd.randint(12, 40))
            seg.append((ms, ml, rnd.randint(1, 70000)))
            pos = ms + ml
        cur = pos
    return Blk(_bytes(rnd, size), segs, first, name=name)


def join_blocks():
    """the seams: every scenario once or more against a run-over match, segments under one match, a segment-0 match to the
    block's end, survivor counts, and a 16385-byte block"""
    rnd = random.Random(12)
    out = []
    scen = ["before", "at", "t1", "t2", "t3", "t7", "eq", "empty", "drops_then_eq"]
    for i in range(3):
        rnd.shuffle(scen)
        out.append(_seam_block(rnd, f"seams_{i}", scen[:7], first=i == 0))
    # a segment whose every raw sequence lies under the match (f == n > 0), then a segment under one match, then drops
    segs = [[] for _ in range(SEGS)]
    segs[0] = [(0, 4, 9), (10, 2 * SEG + 100 - 10, 33)]
    segs[1] = [(SEG + 3, 4, 5), (SEG + 9, 6, 6), (2 * SEG - 10, 20, 7)]
    segs[2] = [(2 * SEG + 50, 52, 8), (2 * SEG + 102, 4, 9), (2 * SEG + 107, 4, 10), (2 * SEG + 200, 4, 11)]
    segs[3] = [(3 * SEG + 1, 8, 12)]
    out.append(Blk(_bytes(rnd, BLOCK), segs, False, name="under_one_match"))
    # a match of segment 0 that runs to the end of the block; later segments' raws all under it
    segs = [[(0, 5, 1), (7, BLOCK - 7, 77)]] + [[(k * SEG + 3, 9, 3)] for k in range(1, SEGS)]
    out.append(Blk(_bytes(rnd, BLOCK), segs, True, name="seg0_to_end"))
    # survivor counts 1, 255, 256, 257 per segment
    segs = [[] for _ in range(5)]
    for k, n in enumerate((1, 255, 256, 257, 4096)):
        raw, _ = lay(scripted(rnd, n, {}, (0, 0, 0), ll_max=3, ml_range=(4, 8)) if n < 4096 else [(0, 4, o) for o in _z_offsets(rnd, n, (0, 0, 0))], k * SEG)
        segs[k] = raw
    out.append(Blk(_bytes(rnd, 5 * SEG), segs, False, name="survivors"))
    # the last segment holds 1 byte
    raw, _ = lay(scripted(rnd, 1500, {}, (0, 0, 0), ll_max=5), 0)
    out.append(Blk(_bytes(rnd, SEG + 1), split([t for t in raw if t[0] + t[1] <= SEG + 1], SEG + 1), False, name="last_seg_1"))
    return out


def gather_blocks():
    """literal runs of every residue, one-byte runs, only literals, no trailing literals, runs of 100 KiB"""
    rnd = random.Random(13)
    out = []
    seqs = [(1, 4, 1 + i % 3) for i in range(40)] + [(rnd.randint(0, 17), rnd.randint(4, 9), rnd.randint(1, 500)) for _ in range(3000)]
    raw, end = lay(seqs, 3)
    out.append(Blk(_bytes(rnd, end + 11), split(raw, end + 11), True, name="runs"))
    for n in (7, 100000, BLOCK):
        out.append(Blk(_bytes(rnd, n), [[] for _ in range((n + SEG - 1) // SEG)], n == 7, name=f"only_lits_{n}"))
    raw, end = lay([(2, 5, 9), (0, 4, 10), (3, 60, 11)])
    out.append(Blk(_bytes(rnd, end), split(raw, end), True, name="no_trailing"))
    raw = [(0, 4, 5), (102400 + 5, 20, 6), (102400 + 30, BLOCK - 102430 - 10, 7)]
    out.append(Blk(_bytes(rnd, BLOCK), split(raw, BLOCK), False, name="run_100k"))
    return out


def small_blocks():
    """one-segment blocks of 31, 32, 33, 64 and 65 sequences (the small kernel's rounds of 32), and 1 .. 6-byte blocks"""
    rnd = random.Random(14)
    out = []
    for n in (31, 32, 33, 64, 65, 1, 0):
        seqs = scripted(rnd, n, {}, (1, 4, 8), ll_max=40)
        raw, end = lay(seqs, rnd.randint(0, 3))
        size = max(7, min(SMALL_ROW, end + rnd.randint(0, 30)))
        out.append(Blk(_bytes(rnd, size), [raw], n % 2 == 1, (1, 4, 8) if n != 33 else (3, 17, 4099), name=f"small_{n}"))
    return out


def raw_blocks():
    """blocks of fewer than 7 bytes: the parse writes their meta, K1c must not touch them"""
    rnd = random.Random(15)
    return [Blk(_bytes(rnd, n), [[]], True, name=f"raw_{n}") for n in (1, 6)]


def ldm_blocks():
    """blocks with long-distance matches laid over the joined sequences"""
    rnd = random.Random(16)
    out = []
    # clip start, clip end, left with 4 / 3, before the first and after the last parse match, unclipped 3-byte tail
    segs = [[] for _ in range(2)]
    segs[0] = [(100, 20, 5), (130, 10, 6), (150, 8, 7), (170, 9, 8), (200, 40, 9), (SEG - 10, 30, 10)]
    segs[1] = [(SEG + 17, 6, 11), (SEG + 30, 6, 12), (SEG + 200, 5, 13)]     # SEG + 17: a 3-byte tail at the seam
    lm = [(10, 50, 1 << 20), (116, 10, 1 << 21), (146, 7, 1 << 22), (175, 20, 1 << 23), (SEG + 100, 40, 3 << 24), (SEG + 300, 100, 5 << 20)]
    out.append(Blk(_bytes(rnd, SEG + 600), segs, True, ldm=lm, name="ldm_clips"))
    # nP and nL over 256 and 1024
    seqs = scripted(rnd, 1500, {}, (0, 0, 0), ll_max=20, ml_range=(4, 30))
    raw, end = lay(seqs)
    size = min(BLOCK, end + 50)
    lm, p = [], 5
    while p + 40 < size and len(lm) < 1300:
        s = p + rnd.randint(0, 20)
        l = rnd.randint(4, 30)
        if s + l > size:
            break
        lm.append((s, l, rnd.randint(1, (1 << 27) - 1)))
        p = s + l
    out.append(Blk(_bytes(rnd, size), split(raw, size), False, ldm=lm, name="ldm_many"))
    # LDM matches only; and no LDM match
    out.append(Blk(_bytes(rnd, 5000), [[]], False, ldm=[(0, 100, 99999), (300, 4000, 1 << 26)], name="ldm_only"))
    raw, end = lay(scripted(rnd, 50, {}, (1, 4, 8)))
    out.append(Blk(_bytes(rnd, end + 9), split(raw, end + 9), True, ldm=[], name="ldm_none"))
    return out
