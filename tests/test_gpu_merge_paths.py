"""The merge (K1c: segment join, repcodes, literal gather, meta; zb_merge_segments_kernel, its LDM variant and
zb_merge_small_kernel in zstd_b200/csrc/zb_match.cu, zb_merge_codes in zb_merge.cuh) sequence by sequence against the
oracle's serial loop, and the caller-sequence path (K1s, zb_seqimport.cu) that runs zb_merge_codes too.

tests/merge_harness.cu runs the product's zb_launch_merge on chosen raw sequences without the walk or the parse in front
of it, and K1s on chosen caller sequences.  tests/mergegen.py restates the join and the repcodes (dfastgen.parse_block
calls that restatement, so the parse tests hold it equal to zbo_parseBlock), chooses blocks that reach every seam of the
join, every repcode outcome at every thread, warp and tile edge, every shape of the literal gather, the small kernel's
rounds of 32 and the LDM overlay's clips, and holds wrong-rule switches that those blocks must tell from the rule.

CPU (no GPU needed): every row is reached, every switch changes a block, the equivalent rules change none, and the two
expressions the kernel uses for the join's cur agree.
GPU: every block of every launch (mixed sizes, blocks of fewer than 7 bytes among them) against the restatement: meta,
seq rows, literal rows, the sentinel behind the literals, untouched rows of raw blocks; the one-segment launches at rows
of at most 8192 bytes (small kernel) and of 8193-16384 (segments kernel) give identical rows; the chosen sequences
through K1s give the same rows; and the raw segment lists the doubleFast and fast parse restatements produce for every
frame of their path tests, and the LDM path frames, against zbo_parseBlock and zbo_ldm_overlayBlock."""
import ctypes
import functools
import os

import numpy as np
import pytest

import mergegen as M

HARNESS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_build", "libzb_merge_harness.so")
SENT = (0xA5, 0x3C)
META_WORDS = 8


def _one_segment(b):
    return len(b.segs) == 1 and b.size <= M.SEG


@functools.lru_cache(maxsize=None)
def launches():
    """(name, blocks, row sizes, ldm) of the chosen launches; a row size of 0 = the largest block"""
    codes, join, gather, small, raw, ldm = (M.codes_blocks(), M.join_blocks(), M.gather_blocks(), M.small_blocks(),
                                            M.raw_blocks(), M.ldm_blocks())
    mixed_small = [b for b in gather + codes if b.size <= 8192]
    return [
        ("codes", [codes[0], raw[0]] + codes[1:6] + [raw[1]] + codes[6:], (0,), False),
        ("join", [join[0], raw[1]] + join[1:] + [raw[0]] + gather, (0,), False),
        ("small", small + raw + mixed_small, (8192, 16384), False),
        ("small_7k", [b for b in small if b.size <= 7000] + raw, (7000, 8193), False),
        ("last_seg", [b for b in join if b.size == M.SEG + 1] + small[:2], (M.SEG + 1, 0), False),
        ("ldm", ldm + [raw[0]], (0,), True),
    ]


@functools.lru_cache(maxsize=None)
def _rows_and_expect():
    rows, exp = {}, {}
    for name, blocks, sizes, _ in launches():
        for row in sizes:
            small = row and row <= M.SMALL_ROW
            for b in blocks:
                if b.size >= 7:
                    exp[id(b)] = b.expect(rows=rows, small_row=bool(small and _one_segment(b)))
    return rows, exp


# ------------------------------------------------------------------------------------------------------------ CPU
def test_every_row_is_reached():
    rows, _ = _rows_and_expect()
    print("\n" + "\n".join(f"{r:24s} {rows.get(r, 0)}" for r in M.ROWS))
    missing = [r for r in M.ROWS if not rows.get(r)]
    assert not missing, f"rows never reached: {missing}"


def test_cur_expressions_agree():
    """the kernel's cur after a segment: pm + pl when the first survivor is the segment's last raw sequence, else the
    last raw's end.  They agree because a trimmed match keeps its end, and a later raw sequence of the same segment is
    never dropped (the parse's sequences of one segment do not overlap)"""
    rows, _ = _rows_and_expect()
    assert rows.get("cur_from_pm") and rows.get("cur_from_last")
    assert all(not rows.get(r) for r in M.ZERO_ROWS), {r: rows.get(r) for r in M.ZERO_ROWS}


def _all_blocks():
    seen, out = set(), []
    for _, blocks, _, _ in launches():
        for b in blocks:
            if id(b) not in seen and b.size >= 7:
                seen.add(id(b))
                out.append(b)
    return out


@pytest.mark.parametrize("switch", sorted(M.SWITCHES))
def test_inputs_tell_the_rule_from(switch):
    changed = [b.name for b in _all_blocks() if b.expect(frozenset([switch])) != b.expect()]
    print(f"\n{switch}: {len(changed)} blocks changed: {changed}")
    assert changed, f"no block tells '{M.SWITCHES[switch]}' from the rule"


@pytest.mark.parametrize("switch", sorted(M.EQUIVALENT))
def test_equivalent_rules_change_nothing(switch):
    rows, _ = _rows_and_expect()
    assert rows.get("zfull_r1_is_1") and rows.get("raw_at_cur")       # the inputs that could tell them apart exist
    assert all(b.expect(frozenset([switch])) == b.expect() for b in _all_blocks())


def test_generators_keep_the_parse_guarantees_and_are_deterministic():
    a = [(b.data, b.segs, b.ldm) for b in M.codes_blocks() + M.join_blocks() + M.ldm_blocks()]
    assert a == [(b.data, b.segs, b.ldm) for b in M.codes_blocks() + M.join_blocks() + M.ldm_blocks()]
    with pytest.raises(AssertionError):
        M.check_raw(100, [[(10, 4, 1), (12, 4, 1)]])                  # overlapping
    with pytest.raises(AssertionError):
        M.check_raw(2 * M.SEG, [[(M.SEG + 1, 4, 1)], []])             # starts outside its segment


# ------------------------------------------------------------------------------------------------------------ GPU
_H = None


def _harness():
    global _H
    if _H is None:
        H = ctypes.CDLL(HARNESS)
        vp, u64, u32 = ctypes.c_void_p, ctypes.c_uint64, ctypes.c_uint32
        H.zbh_merge.restype = ctypes.c_int
        H.zbh_merge.argtypes = [vp, u64, u32, vp, vp, vp, vp, u32, vp, vp, u64, u32, vp, vp, u64, u32, vp, vp, u64, vp, u64, vp, u64, vp]
        H.zbh_seq_convert.restype = ctypes.c_int
        H.zbh_seq_convert.argtypes = [vp, u64, vp, u32, vp, u32, vp, vp, u64, vp, u64, vp, u64, vp, vp]
        _H = H
    return _H


def _p(a):
    return a.ctypes.data


def gpu_merge(blocks, row_size=0, ldm=False, use_dicts=True):
    """one harness launch, run twice: seqs (2, rows, sd.seq) u64, lits (2, rows, sd.lit) u8, meta (2, rows, 8) u32"""
    src, offs = bytearray(), []
    for i, b in enumerate(blocks):
        src += bytes(i % 5)                                          # blocks at every alignment
        offs.append(len(src))
        src += b.data
    nb = len(blocks)
    cnt = np.zeros((nb, M.SEGS), np.uint32)
    raw, lcnt, lm = [], np.zeros(nb, np.uint32), []
    for i, b in enumerate(blocks):
        for k, seg in enumerate(b.segs):
            cnt[i, k] = len(seg)
            raw += [t for s in seg for t in s]
        if ldm:
            lcnt[i] = len(b.ldm or [])
            lm += [t for m in (b.ldm or []) for t in m]
    M_ = max(row_size or max(b.size for b in blocks), 64)
    M_ = (M_ + 63) & ~63
    seq_stride, lit_stride = M_ // 4 + 8, M_ + 256
    seqs = np.zeros((2, nb, seq_stride), np.uint64)
    lits = np.zeros((2, nb, lit_stride), np.uint8)
    meta = np.zeros((2, nb, META_WORDS), np.uint32)
    shape = np.zeros(4, np.uint64)
    a64, a32 = (lambda v: np.array(v, np.uint64)), (lambda v: np.array(v, np.uint32))
    bo, bs = a64(offs), a32([b.size for b in blocks])
    fl = a32([1 if b.first else 0 for b in blocks])
    reps = a32([r for b in blocks for r in b.reps])
    rawa, lma = a32(raw or [0]), a32(lm or [0])
    sent = np.array(SENT, np.uint8)
    r = _harness().zbh_merge(bytes(src), len(src), nb, _p(bo), _p(bs), _p(fl), _p(reps), int(use_dicts), _p(cnt), _p(rawa),
                             len(raw) // 3, int(ldm), _p(lcnt), _p(lma), len(lm) // 3, row_size, _p(sent),
                             _p(seqs), seqs.size, _p(lits), lits.size, _p(meta), meta.size, _p(shape))
    assert r == 0, f"harness returned {r}"
    assert tuple(int(x) for x in shape[:2]) == (seq_stride, lit_stride)
    return seqs, lits, meta


def pack(seqs):
    return np.array([ob | (ll << 28) | (ml << 46) for ob, ll, ml in seqs], np.uint64)


def check(blocks, seqs, lits, meta, expect, what=""):
    """every block of a launch against its expectation (both runs)"""
    for i, b in enumerate(blocks):
        for r in range(2):
            s = SENT[r]
            if b.size < 7:
                assert np.all(meta[r, i].view(np.uint8) == s), f"{what}: meta of the {b.size}-byte block {b.name} written"
                assert np.all(lits[r, i] == s) and np.all(seqs[r, i].view(np.uint8) == s), f"{what}: rows of raw block {b.name} written"
                continue
            want, wl = expect(b)
            m = meta[r, i]
            assert list(m) == [len(want), len(wl), 0, 0, 2, 0, 0, 0], f"{what}: block {b.name} meta {list(m)}, want nbSeq {len(want)} litSize {len(wl)}"
            got = seqs[r, i, :len(want)]
            wp = pack(want)
            bad = np.nonzero(got != wp)[0]
            assert bad.size == 0, (f"{what}: block {b.name} sequence {bad[0]} of {len(want)}: got "
                                   f"({int(got[bad[0]]) & 0xFFFFFFF}, {(int(got[bad[0]]) >> 28) & 0x3FFFF}, {int(got[bad[0]]) >> 46}), "
                                   f"want {want[bad[0]]} ({bad.size} differ)")
            gl = lits[r, i, :len(wl)].tobytes()
            if gl != wl:
                j = next(k for k in range(len(wl)) if gl[k] != wl[k])
                raise AssertionError(f"{what}: block {b.name} literal {j} of {len(wl)} differs")
            assert np.all(lits[r, i, len(wl):] == s), f"{what}: block {b.name} literal row written past litSize"


def _expect(b):
    return _rows_and_expect()[1][id(b)]


@pytest.mark.gpu
@pytest.mark.parametrize("name", [l[0] for l in launches()])
def test_gpu_chosen_launch(name):
    _, blocks, sizes, ldm = next(l for l in launches() if l[0] == name)
    got = []
    for row in sizes:
        seqs, lits, meta = gpu_merge(blocks, row, ldm)
        check(blocks, seqs, lits, meta, _expect, f"{name} rows {row}")
        got.append((seqs, lits, meta))
    if len(sizes) == 2:                                              # small kernel and segments kernel: identical rows
        for i, b in enumerate(blocks):
            if b.size < 7:
                continue
            n, nl = _expect(b)[0], _expect(b)[1]
            for r in range(2):
                assert np.array_equal(got[0][0][r, i, :len(n)], got[1][0][r, i, :len(n)])
                assert np.array_equal(got[0][1][r, i, :len(nl)], got[1][1][r, i, :len(nl)])
                assert np.array_equal(got[0][2][r, i], got[1][2][r, i])


@pytest.mark.gpu
def test_gpu_without_dictionary_table():
    """no dictionary table: a first block starts from {1,4,8} whatever its slot would hold"""
    blocks = [b for b in M.codes_blocks() if b.first and b.reps == (1, 4, 8)][:2] + M.small_blocks()
    seqs, lits, meta = gpu_merge(blocks, 0, False, use_dicts=False)
    check(blocks, seqs, lits, meta, lambda b: M.Blk(b.data, b.segs, b.first, (1, 4, 8)).expect(), "no dicts")


def _offsets(b, seqs):
    out, r = [], b.start_reps()
    for ob, ll, ml in seqs:
        off = M._offset(r, ob, ll)
        out.append(off)
        _, r = M.code(r, off, ll)
    return out


def _seq_frames():
    """the chosen blocks as frames of caller sequences: a first block and the non-first blocks behind it"""
    frames, cur = [], None
    for _, blocks, _, ldm in launches():
        if ldm:
            continue
        for b in blocks:
            if b.size < 7:
                continue
            want = _expect(b)[0]
            offs = _offsets(b, want)
            ok = all(1 <= o <= M.SEQ_OFF_MAX for o in offs)
            if b.first:
                cur = [] if ok else None
                if cur is not None:
                    frames.append(cur)
            if cur is not None and ok and id(b) not in {id(x) for x in cur}:
                cur.append(b)
    return [f for f in frames if f]


@pytest.mark.gpu
def test_gpu_caller_sequences_give_the_same_rows():
    """K1s: each frame's blocks as caller sequences with explicit delimiters; the rows equal the merge's"""
    H = _harness()
    for fr in _seq_frames():
        src, q = bytearray(), []
        for b in fr:
            want = _expect(b)[0]
            pos = 0
            for (ob, ll, ml), off in zip(want, _offsets(b, want)):
                q += [off, ll, ml, 0]
                pos += ll + ml
            q += [0, b.size - pos, 0, 0]
            src += b.data
        qa = np.array(q, np.uint32)
        nb = len(fr)
        seq_stride = (M.BLOCK // 3) + 8
        lit_stride = M.BLOCK + 256
        seqs = np.zeros((2, nb, seq_stride), np.uint64)
        lits = np.zeros((2, nb, lit_stride), np.uint8)
        meta = np.zeros((2, nb, META_WORDS), np.uint32)
        ctrl, shape = np.zeros(4, np.uint64), np.zeros(3, np.uint64)
        reps = np.array(fr[0].reps, np.uint32)
        r = H.zbh_seq_convert(bytes(src), len(src), _p(qa), len(q) // 4, _p(reps), 1, _p(np.array(SENT, np.uint8)),
                              _p(seqs), seqs.size, _p(lits), lits.size, _p(meta), meta.size, _p(ctrl), _p(shape))
        assert r == 0, f"harness returned {r}"
        assert int(shape[2]) == nb and int(ctrl[2]) == (1 << 64) - 1 and int(ctrl[3]) == len(src) and int(ctrl[1]) == nb
        check(fr, seqs, lits, meta, _expect, f"caller sequences ({fr[0].name} ..)")


# ------------------------------------------------------------------------------------------------- the real blocks
def _real(parse_mod, frames):
    import dfastgen as dg
    out = []
    for src, level, d in frames:
        for b in dg.frame_blocks(src, level, d):
            segs = [[(ms - b.bs, ml, off) for ms, ml, off in parse_mod.parse_segment(b, ss, min(ss + M.SEG, b.be))]
                    for ss in range(b.bs, b.be, M.SEG)]
            blk = M.Blk(b.buf[b.bs:b.be], segs, b.bs == b.frame_start, b.code_reps, name=f"L{level}@{b.bs - b.frame_start}")
            blk.oracle = b.oracle_seqs
            out.append(blk)
    return out


@functools.lru_cache(maxsize=None)
def real_blocks(kind):
    import dfastgen as dg
    import fastgen as fg
    if kind == "dfast":
        return _real(dg, dg.all_frames())
    return _real(fg, fg.all_frames())


@functools.lru_cache(maxsize=None)
def ldm_real_blocks():
    """the LDM path frames at three parameter sets: the fast parse's raw segments, the oracle's lists"""
    import dfastgen as dg
    import fastgen as fg
    import ldmgen as lg
    import ldmref
    out = []
    for name, pfx, src, level, prm in lg.cases():
        if pfx or name.split("/")[1] not in ("default", "mm4", "mm37"):
            continue
        lists = lg.oracle_lists(b"", src, prm)
        for b in dg.frame_blocks(src, 1, None, ldm=True):
            segs = [[(ms - b.bs, ml, off) for ms, ml, off in fg.parse_segment(b, ss, min(ss + M.SEG, b.be))]
                    for ss in range(b.bs, b.be, M.SEG)]
            lm = [tuple(m) for m in lists[b.index]]
            blk = M.Blk(b.buf[b.bs:b.be], segs, b.bs == b.frame_start, b.code_reps, ldm=lm, name=f"{name}#{b.index}")
            blk.oracle = ldmref.overlay_block(b.buf[b.bs:b.be], b.ldm_reps, lm, b.oracle_seqs)[0]
            out.append(blk)
    return out


def _oracle_expect(b):
    seqs = [tuple(s) for s in b.oracle]
    return seqs, M.literals(b.data, seqs)


@pytest.mark.parametrize("kind", ["dfast", "fast"])
def test_real_raw_lists_join_to_the_oracle(kind):
    """on the CPU: the restatement joins the parse's raw lists to zbo_parseBlock's sequences (what the GPU must give)"""
    blocks = real_blocks(kind)
    assert blocks and all(b.expect()[0] == [tuple(s) for s in b.oracle] for b in blocks)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["dfast", "fast"])
def test_gpu_real_blocks(kind):
    blocks = real_blocks(kind)
    for i in range(0, len(blocks), 96):
        part = blocks[i:i + 96]
        seqs, lits, meta = gpu_merge(part)
        check(part, seqs, lits, meta, _oracle_expect, f"{kind} blocks {i}..")


@pytest.mark.gpu
def test_gpu_ldm_real_blocks():
    blocks = ldm_real_blocks()
    for i in range(0, len(blocks), 64):
        part = blocks[i:i + 64]
        seqs, lits, meta = gpu_merge(part, 0, True)
        check(part, seqs, lits, meta, _oracle_expect, f"ldm blocks {i}..")
