"""Inputs for the doubleFast parse (K1b dfast, zb_parse_dfast_kernel in zstd_b200/csrc/zb_match.cu) and a Python
restatement of the oracle's doubleFast parse (parse_dfast_segment and the join of zbo_parseBlock, oracle/zb_match.c) that
counts which path every probe takes.  TEST INFRASTRUCTURE ONLY.

The restatement is fed the candidate arrays of the oracle's own walk (zbo_walkChunk) and is driven block by block as
zbo_compress_usingDict drives zbo_parseBlock (oracle/zb_frame.c); tests/test_gpu_dfast_paths.py proves it equal to
zbo_parseBlock on every block, so its path counts are the oracle's.  Switches replace one rule by a neighbouring wrong
one: the inputs must tell each of them apart from the rule.

frame_blocks and the join of parse_block serve the fast parse's restatement too (tests/fastgen.py)."""
import ctypes
import random

import numpy as np

import zref
from test_plan import OCParams, OPlan

BLOCK = 128 << 10
SEG = 16 << 10
FAR = 0xFFFF
WARP = 32
M32, M40, M64 = (1 << 32) - 1, (1 << 40) - 1, (1 << 64) - 1

# ---------------------------------------------------------------------------------------------------------- hashes
# the walk's hashes with hBits = 32 (oracle/zb_match.c zb_hash, zstd_compress_internal.h:815-861); bucket = (h * N) >> 32,
# tag = h & 0x7FF.  Each is a bijection of the bytes it reads, so an input can hold a chosen hash.
P4, P5, P8 = 2654435761, 889523592379, 0xCF1BBCDCB7A56463


def hash8(v: int) -> int:
    return ((v * P8) & M64) >> 32


def hash5(v: int) -> int:
    return (((v & M40) * P5) & M40) >> 8


def hash4(v: int) -> int:
    return ((v & M32) * P4) & M32


def with_hash8(lo: int, h: int) -> bytes:
    """8 bytes whose low 4 bytes are `lo` and whose 8-byte hash is h: hash8 = ((lo * P8 mod 2^64) >> 32) + hi * (P8 mod 2^32)."""
    hi = ((h - (((lo * P8) & M64) >> 32)) * pow(P8 & M32, -1, 1 << 32)) & M32
    return (lo | (hi << 32)).to_bytes(8, "little")


def with_hash5(h: int, low8: int) -> bytes:
    return (((((h << 8) | low8) & M40) * pow(P5, -1, 1 << 40)) & M40).to_bytes(5, "little")


def with_hash4(h: int) -> bytes:
    return ((h * pow(P4, -1, 1 << 32)) & M32).to_bytes(4, "little")


def twin_hash(h: int) -> int:
    """another 32-bit hash in the same bucket of every table the doubleFast walk uses (power-of-two tables up to 2^14 and the
    28672-bucket table: the high bits are kept) with the same 11-bit tag: a tag collision"""
    return (h + (1 << 11)) & M32 if (h >> 11) & 0x7F != 0x7F else (h - (1 << 11)) & M32


def twin8_six(x: bytes) -> bytes:
    """8 bytes equal to x in their first 6 bytes with the same bucket and tag in every long table (2^14 buckets or fewer): the
    hash moves by +-2^16, which keeps the tag and, with the carry kept inside bits 16-17, the bucket.  Bytes that agree in
    their first 7 bytes never share a bucket: changing byte 7 alone moves the hash's top 8 bits (times the odd P8 mod 2^8)."""
    h = hash8(int.from_bytes(x, "little"))
    d = 1 if (h >> 16) & 3 < 3 else -1
    hi = (int.from_bytes(x[4:], "little") + (((d * pow(P8 & M32, -1, 1 << 16)) & 0xFFFF) << 16)) & M32
    y = x[:4] + hi.to_bytes(4, "little")
    hy = hash8(int.from_bytes(y, "little"))
    assert y[:6] == x[:6] and y[6] != x[6] and hy >> 18 == h >> 18 and hy & 0x7FF == h & 0x7FF
    return y


def other_tag(h: int) -> int:
    """same bucket, a different tag: an entry with this hash evicts the one with hash h"""
    return (h & ~0x7FF) | ((h + 0x155) & 0x7FF)


# ------------------------------------------------------------------------------------------------------- generator
def dfast_input(n: int, seed: int, hist: bytes = b"", start_reps=None) -> bytes:
    """n bytes built from copy operations aimed at the doubleFast parse's paths.  `hist` is the history in front of the frame
    (a dictionary's content tail): copies may reach into it, the first ones across the dictionary / frame border.
    start_reps: the dictionary's repcodes (rep1, rep2): the frame starts with a repeat at rep2 (odd seeds: repcode-2 at the
    anchor) or, behind one literal, at rep1 (even seeds: repcode-1 at p+1)."""
    rnd = random.Random(seed)
    h0 = len(hist)
    out = bytearray(hist)
    end = h0 + n
    reps = [1, 4, 8]
    pending = []                                             # (due position, action): the second half of two-part gadgets
    rand_runs = []                                           # (start, end) of incompressible runs, sources for catch-up
    ends_done = set()

    def pos():
        return len(out) - h0

    def copy(off, length):
        off = max(1, min(off, len(out)))
        if off >= length:
            out.extend(out[len(out) - off:len(out) - off + length])
        else:
            pat = bytes(out[len(out) - off:])
            out.extend((pat * (length // off + 1))[:length])
        if off != reps[0]:
            reps[:] = [off, reps[0], reps[1]] if off != reps[1] else [off, reps[0], reps[2]]
        return off

    def differ(b):
        """one byte that is not b"""
        return (b + 1 + rnd.randrange(255)) & 255

    def lits(k):
        out.extend(rnd.randbytes(k))

    def anchor_copy():
        """a copy that ends right before the gadget that follows, so that the gadget's first byte is probed at lane 0"""
        off = copy(rnd.randint(8, min(len(out), 2000)), rnd.randint(12, 40))
        out.append(differ(out[len(out) - off]))

    # -- gadgets that need the table to hold a chosen entry: the entry, then >= one walk batch later the probe
    def near_long(kind):
        x = rnd.randbytes(8)
        lo = int.from_bytes(x[:4], "little")
        hx = hash8(int.from_bytes(x, "little"))
        lits(3)
        out.extend(x)
        lits(24)
        if kind == "coll_next":                               # other low bytes: no short candidate, the 8-byte tag collides
            y = with_hash8(int.from_bytes(rnd.randbytes(4), "little"), twin_hash(hx))
        elif kind == "f1_six":                                # 6 equal bytes at p+1, next to a short hit of 5
            y = twin8_six(x)
        else:                                                 # same 5 low bytes: the short hash is x's, the 8-byte hash collides
            y = with_hash8(lo, twin_hash(hx))
        assert kind == "coll_next" or y[:5] == x[:5]

        def probe():
            anchor_copy()
            if kind in ("f1_lt8", "f1_six"):                  # a short hit of 5 bytes at p, a long collision at p+1
                c = rnd.randbytes(1)
                out.extend(c + x[:4] + bytes([differ(x[4])]) + rnd.randbytes(30))
                lits(rnd.randint(1500, 2500))
                anchor_copy()
                out.extend(c + y + rnd.randbytes(20))
            else:
                out.extend(y + rnd.randbytes(20))
        pending.append((len(out) + rnd.randint(1100, 2000), probe))

    def near_short():
        """a tag collision in the short table, for both minimum match lengths the doubleFast rows use"""
        a = rnd.randbytes(8)
        h4, h5 = hash4(int.from_bytes(a[:4], "little")), hash5(int.from_bytes(a[:5], "little"))
        out.extend(rnd.randbytes(2) + a + rnd.randbytes(20))
        b4 = with_hash4(twin_hash(h4)) + rnd.randbytes(4)
        b5 = with_hash5(twin_hash(h5), rnd.randrange(256)) + rnd.randbytes(3)

        def probe():
            anchor_copy()
            out.extend(b4 + rnd.randbytes(20))
            anchor_copy()
            out.extend(b5 + rnd.randbytes(20))
        pending.append((len(out) + rnd.randint(1100, 2000), probe))

    def upgrade(kind, far=False):
        """a short match at p next to a match of >= 8 bytes at p+1 (zstd_double_fast.c:254-271): p = c B[0:f1] w, an earlier
        A = c B[0:k] z.  short length ml = 1 + min(k, f1) (or f1 when k = f1 - 1), long length at p+1 = f1."""
        f1 = rnd.randint(8, 40)
        if kind == "gt":
            k = rnd.choice([3, 4, 5, 6, f1 - 3]) if f1 > 10 else rnd.choice([3, 4, 5, 6])
        elif kind == "eq":
            k = f1 - 1
        else:
            k = f1 + rnd.randint(0, 8)
        bsrc = rnd.randbytes(max(f1, k) + 1)
        c = rnd.randbytes(1)
        lits(2)
        out.extend(bsrc)
        out.extend(rnd.randbytes(8))

        def place_a():
            a = c + bsrc[:k] + bytes([differ(bsrc[k])])
            lits(3)
            out.extend(a + rnd.randbytes(16))
            if k >= 7:                                        # evict A from the long table: p must find no long candidate
                ha = hash8(int.from_bytes(a[:8], "little"))
                ev = with_hash8(int.from_bytes(rnd.randbytes(4), "little"), other_tag(ha))

                def evict():
                    out.extend(rnd.randbytes(3) + ev + rnd.randbytes(16))
                    pending.append((len(out) + rnd.randint(1100, 1500), probe))
                pending.append((len(out) + rnd.randint(1100, 1500), evict))
            else:
                pending.append((len(out) + rnd.randint(1100, 1500), probe))

        def probe():
            anchor_copy()
            w = differ(bsrc[f1])
            if kind == "eq":
                w = w if w != bsrc[k - 1] else differ(w)
            out.extend(c + bsrc[:f1] + bytes([w]) + rnd.randbytes(12))
        if far:
            pending.append((len(out) + FAR + rnd.randint(64, 4000), place_a))
        else:
            pending.append((len(out) + rnd.randint(200, 1500), place_a))

    if hist and start_reps:                                  # the dictionary's repcodes start the frame's first segment
        r1, r2 = start_reps
        if seed % 2:                                         # repcode-2 at the anchor
            copy(r2, rnd.randint(6, 14))
        else:                                                # repcode-1 at p+1
            lits(1)
            copy(r1, rnd.randint(6, 14))
        lits(1)
    if hist:                                                 # copies whose sources straddle the dictionary / frame border
        for _ in range(4):
            lits(rnd.choice([1, 3, 9]))
            into = rnd.choice([1, 2, 5, 7, rnd.randint(8, min(60, h0))])   # bytes of the source in front of the border
            copy(pos() + into, into + rnd.randint(1, pos()))
        copy(pos() + rnd.randint(FAR // 4, h0 - 64) if h0 > FAR // 4 + 64 else h0, rnd.randint(20, 60))
    else:
        lits(256)

    while pos() < n:
        if pending and pending[0][0] <= len(out):
            pending.pop(0)[1]()
            pending.sort(key=lambda t: t[0])
            continue
        p = pos()
        b_end = (p // BLOCK + 1) * BLOCK
        if b_end <= n and b_end - p < 2500 and b_end not in ends_done:    # a long copy that ends 0..8 bytes before a block end
            ends_done.add(b_end)
            k = rnd.choice([0, 1, 2, 3, 5, 8, 8, -40])           # -40: runs on past the block's end
            length = b_end - k - p
            off = copy(rnd.randint(1, min(len(out), 500)), length)
            if k == 8:                                       # 8 bytes left that repeat earlier ones: never probed (p + 9 > be)
                for _ in range(64):
                    off2 = rnd.randint(9, min(len(out), 3000))
                    if out[len(out) - off2] != out[len(out) - off]:
                        break
                copy(off2, 8 + rnd.randint(4, 40))
            else:
                out.append(differ(out[len(out) - off]))
            continue
        s_end = (p // SEG + 1) * SEG
        if s_end % BLOCK and s_end < n and s_end - p < 1500 and s_end not in ends_done:
            # literals, then a copy that starts 1..6 bytes in front of a segment's start: the segment finds it at its first
            # byte (its anchor), the literal-heavy segment in front has skipped its head
            ends_done.add(s_end)
            lits(s_end - rnd.randint(1, 6) - p)
            copy(rnd.randint(1, min(len(out), 3000)), rnd.randint(20, 200))
            continue
        op = rnd.random()
        if op < 0.14:
            lits(rnd.choice([1, 2, 3, 5, 9, 31, 200]))
        elif op < 0.16:                                      # incompressible runs: the probe step reaches 2, 12, 32+
            k = rnd.choice([300, 3 << 10, 9 << 10])
            rand_runs.append((len(out), len(out) + k))
            lits(k)
        elif op < 0.28:                                      # exactly 4..7 equal bytes, then a differing one
            off = rnd.randint(1, min(len(out), 4000)) if rnd.random() < 0.7 else rnd.randint(FAR, max(FAR, min(len(out), 0x1F000)))
            off = copy(off, rnd.randint(4, 7))
            out.append(differ(out[len(out) - off]))
        elif op < 0.42:                                      # >= 8 equal bytes
            off = rnd.randint(1, min(len(out), 3000))
            copy(off, rnd.choice([8, 9, 12, 33, 64, 100, 255, 256, 257, 300]))
        elif op < 0.50 and len(out) > FAR + 64:              # far: the walk stores the distance in the far array
            copy(rnd.randint(FAR, min(len(out), 0x1F000)), rnd.choice([8, 9, 16, 40, 300]))
        elif op < 0.56:                                      # repcode-1 at p+1: one literal, then the last offset again
            lits(1)
            copy(reps[0], rnd.randint(4, 64))
        elif op < 0.62:                                      # repcode-2 at the anchor: two copies back to back
            o2 = reps[0]
            copy(rnd.randint(1, min(len(out), 3000)), rnd.randint(8, 40))
            copy(o2, rnd.randint(4, 40))
        elif op < 0.66 and rand_runs:                        # catch-up: a copy of a sparsely inserted incompressible run
            s, e = rand_runs[-1]
            if e - s >= 3 << 10:
                src = rnd.randint(s + (e - s) // 2, e - 400)
                copy(len(out) - src, rnd.randint(150, 400))
        elif op < 0.68:                                      # catch-up stopped by the anchor: the byte before both is equal
            for _ in range(64):
                off = rnd.randint(8, min(len(out), 3000))
                if out[-1] == out[len(out) - 1 - off]:
                    break
            copy(off, rnd.randint(8, 64))
        elif op < 0.70:                                      # long: several forward rounds, across segment ends
            copy(rnd.randint(1, min(len(out), 600)), rnd.randint(300, 3 * SEG // 2))
        elif op < 0.76:
            upgrade(rnd.choice(["gt", "eq", "lt"]), far=rnd.random() < 0.25)
        elif op < 0.82:
            near_long(rnd.choice(["coll_short", "coll_next", "f1_lt8", "f1_six"]))
        elif op < 0.85:
            near_short()
        else:
            copy(rnd.randint(1, min(len(out), 30000)), rnd.randint(4, 24))
    return bytes(out[h0:end])


# --------------------------------------------------------------------------------------------- oracle, through ctypes
class HufCTable(ctypes.Structure):
    _fields_ = [("nbBits", ctypes.c_uint8 * 256), ("code", ctypes.c_uint16 * 256), ("tableLog", ctypes.c_uint), ("maxSymbolValue", ctypes.c_uint)]


class FseCTable(ctypes.Structure):
    _fields_ = [("tableLog", ctypes.c_uint), ("maxSymbolValue", ctypes.c_uint), ("nextState", ctypes.c_uint16 * 512),
                ("deltaFindState", ctypes.c_int32 * 64), ("deltaNbBits", ctypes.c_uint * 64)]


class DictEntropy(ctypes.Structure):
    _fields_ = [("present", ctypes.c_uint), ("dictID", ctypes.c_uint), ("huf", HufCTable), ("hufRepeat", ctypes.c_uint),
                ("fse", FseCTable * 3), ("fseRepeat", ctypes.c_uint * 3), ("rep", ctypes.c_uint * 3)]


class ChunkCand(ctypes.Structure):
    _fields_ = [("dS", ctypes.POINTER(ctypes.c_uint)), ("dL", ctypes.POINTER(ctypes.c_uint)),
                ("low", ctypes.c_size_t), ("start", ctypes.c_size_t), ("end", ctypes.c_size_t)]


class Seq(ctypes.Structure):
    _fields_ = [("offBase", ctypes.c_uint), ("litLen", ctypes.c_uint), ("matchLen", ctypes.c_uint)]


_O = None


def _oracle():
    global _O
    if _O is None:
        O = zref.oracle()
        O.zbo_getCParams.restype = OCParams
        O.zbo_getCParams.argtypes = [ctypes.c_int, ctypes.c_ulonglong, ctypes.c_size_t]
        O.zbo_makePlan.argtypes = [ctypes.POINTER(OPlan), ctypes.POINTER(OCParams)]
        O.zbo_loadDictEntropy.restype = ctypes.c_size_t
        O.zbo_loadDictEntropy.argtypes = [ctypes.POINTER(DictEntropy), ctypes.c_char_p, ctypes.c_size_t]
        O.zbo_walkChunk.restype = None
        O.zbo_walkChunk.argtypes = [ctypes.POINTER(OPlan), ctypes.c_char_p, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_size_t,
                                    ctypes.POINTER(ChunkCand)]
        O.zbo_freeChunk.restype = None
        O.zbo_freeChunk.argtypes = [ctypes.POINTER(ChunkCand)]
        O.zbo_parseBlock.restype = ctypes.c_size_t
        O.zbo_parseBlock.argtypes = [ctypes.POINTER(OPlan), ctypes.c_char_p, ctypes.POINTER(ChunkCand), ctypes.c_size_t,
                                     ctypes.c_size_t, ctypes.POINTER(Seq), ctypes.c_char_p, ctypes.POINTER(ctypes.c_size_t)]
        _O = O
    return _O


def dict_content_offset(dict_bytes: bytes) -> int:
    """where the content of a dictionary starts, as the oracle's loader reads it (0: raw content)"""
    de = DictEntropy()
    off = _oracle().zbo_loadDictEntropy(ctypes.byref(de), dict_bytes, len(dict_bytes))
    assert off < (1 << 63), "dictionary rejected by the oracle's loader"
    return off


def patch_reps(dict_bytes: bytes, reps) -> bytes:
    """a zstd-format dictionary with its three repcodes (the 12 bytes in front of the content) replaced"""
    off = dict_content_offset(dict_bytes)
    assert off >= 12
    return dict_bytes[:off - 12] + b"".join(int(r).to_bytes(4, "little") for r in reps) + dict_bytes[off:]


class Block:
    """one block as zbo_parseBlock sees it: the buffer (dictionary tail + frame), the chunk's candidate arrays (as lists,
    index = position - chunk start), the block's bounds and its history limit"""
    __slots__ = ("buf", "dL", "dS", "c0", "low", "chunk_low", "window", "bs", "be", "frame_start", "start_reps", "code_reps",
                 "strategy", "mls", "step_size", "oracle_seqs", "index", "ldm_reps")


def frame_blocks(src: bytes, level: int, dict_bytes=None, ldm=False):
    """the blocks of one frame, driven as zbo_compress_usingDict drives the match finder (oracle/zb_frame.c:117-186); each
    carries zbo_parseBlock's own sequences.  Fast frames (strategy 1) have no long candidates: dL is None.
    ldm: a frame of more than 512 KiB with long-distance matching, driven as zbo_compress_ldm_usingDict does
    (oracle/zb_ldm.c): the LDM cParams, and each block's repcodes for the overlay in ldm_reps (the frame's codeRep in its
    first block, else none); block k of the frame has index k."""
    O = _oracle()
    use = dict_bytes is not None and len(dict_bytes) >= 8
    if ldm:
        import ldmref
        assert len(src) > 4 * BLOCK, "frames of at most one chunk are compressed as without LDM"
        cp = ldmref.cparams_ldm(level, len(src), len(dict_bytes) if use else 0)
    else:
        cp = O.zbo_getCParams(level, len(src), len(dict_bytes) if use else 0)
    plan = OPlan()
    O.zbo_makePlan(ctypes.byref(plan), ctypes.byref(cp))
    D, start_reps, code_reps, buf = 0, (0, 0), (1, 4, 8), src
    if use:
        de = DictEntropy()
        off = O.zbo_loadDictEntropy(ctypes.byref(de), dict_bytes, len(dict_bytes))
        assert off < (1 << 63)
        content = len(dict_bytes) - off
        D = min(content, plan.primeBytes)
        buf = dict_bytes[len(dict_bytes) - D:] + src
        if de.present:
            code_reps = tuple(de.rep)
            start_reps = tuple(r if r <= D else 0 for r in de.rep[:2])
    plan.frameStart = D
    plan.startRep[0], plan.startRep[1] = start_reps
    plan.codeRep[0], plan.codeRep[1], plan.codeRep[2] = code_reps
    block_max = min(1 << cp.windowLog, BLOCK)
    chunk_bytes = plan.chunkBlocks * block_max
    W = 1 << plan.windowLog
    seqs = (Seq * (BLOCK // 4 + 1))()
    lit = ctypes.create_string_buffer(BLOCK + 64)
    lsz = ctypes.c_size_t()
    cc, lists = None, None
    blocks = []
    try:
        for bs in range(0, len(src), block_max):
            bsz = min(block_max, len(src) - bs)
            if bsz < 7:                                          # a raw block (zstd_compress.c:3216)
                continue
            if cc is None or bs + D >= cc.end:
                if cc is not None:
                    O.zbo_freeChunk(ctypes.byref(cc))
                cs = bs - bs % chunk_bytes
                ce = min(cs + chunk_bytes, len(src))
                cc = ChunkCand()
                O.zbo_walkChunk(ctypes.byref(plan), buf, len(buf), cs + D, ce + D, ctypes.byref(cc))
                m = cc.end - cc.start
                lists = (np.ctypeslib.as_array(cc.dL, shape=(m,)).tolist() + [0] * 8 if plan.strategy == 2 else None,
                         np.ctypeslib.as_array(cc.dS, shape=(m,)).tolist() + [0] * 8)
            nb = O.zbo_parseBlock(ctypes.byref(plan), buf, ctypes.byref(cc), bs + D, bsz, seqs, lit, ctypes.byref(lsz))
            b = Block()
            b.buf, b.dL, b.dS, b.c0 = buf, lists[0], lists[1], cc.start
            b.bs, b.be, b.frame_start = bs + D, bs + D + bsz, D
            b.chunk_low, b.window = cc.low, W
            b.low = cc.low if not (b.be > W and b.be - W > cc.low) else b.be - W     # block_low
            b.start_reps, b.code_reps = start_reps, code_reps
            b.strategy, b.mls, b.step_size = plan.strategy, plan.mls, plan.stepSize
            b.oracle_seqs = [(seqs[i].offBase, seqs[i].litLen, seqs[i].matchLen) for i in range(nb)]
            b.index = bs // block_max
            b.ldm_reps = code_reps if bs == 0 else (0, 0, 0)
            blocks.append(b)
    finally:
        if cc is not None:
            O.zbo_freeChunk(ctypes.byref(cc))
    return blocks


# ------------------------------------------------------------------------------------------------- the restatement
# rows of the path table; every one is reached by the inputs of tests/test_gpu_dfast_paths.py
ROWS = [
    "rep2_anchor",        # repcode-2 at the anchor, lane 0 (zstd_double_fast.c:302-316)
    "rep1_p1",            # repcode-1 at p+1, the match starts at p+1 (:190-195)
    "long_hit",           # the long candidate has >= 8 equal bytes (:206-213)
    "long_coll_short",    # the long candidate is a tag collision, the same lane tries its short candidate
    "long_coll_next",     # the long candidate is a tag collision and the lane has no short candidate: next lane
    "short_hit",          # the short candidate has >= 4 equal bytes (:222-225)
    "short_coll",         # the short candidate is a tag collision
    "upgrade",            # short hit replaced by the long match at p+1 (f1 >= 8 and f1 > ml, :254-271)
    "keep_no_l1",         # short hit kept: no long candidate at p+1
    "keep_l1_coll",       # short hit kept: the long candidate at p+1 is a collision of < 4 equal bytes
    "keep_f1_lt8",        # short hit kept: the long candidate at p+1 has 4..7 equal bytes
    "keep_f1_eq",         # short hit kept: f1 >= 8 and f1 == ml
    "keep_f1_lt",         # short hit kept: f1 >= 8 and f1 < ml
    "far_long",           # long hit at a distance >= 0xFFFF (the far array)
    "far_short",          # short hit at a distance >= 0xFFFF
    "far_l1",             # a long candidate at p+1 at a distance >= 0xFFFF, weighed against a short hit
    "step_2",             # a probe step of 2 or more (1 + (ip - searchStart) >> 8, kStepIncr)
    "step_12",
    "step_32",
    "lanes_cut_se",       # lanes beyond the segment's end are not probed
    "lanes_cut_be",       # lanes with p + 9 > blockEnd are not probed
    "tail_unprobed",      # the parse of a block's last segment stops with < 9 bytes left
    "back_32",            # backward catch-up of 32 bytes or more (a second cooperative round)
    "back_stop_anchor",   # catch-up stopped by the anchor while the bytes in front still match
    "back_stop_low",      # catch-up stopped by the start of the history
    "fwd_256",            # forward count of 256 bytes or more (a second cooperative round)
    "fwd_tail",           # the match ends within the last 8 bytes of the block (the byte-wise tail of the count)
    "fwd_to_be",          # the match ends exactly at the block's end
    "join_drop",          # the join drops a sequence that lies under a match run over from an earlier segment
    "join_trim",          # the join keeps the tail (>= 3 bytes) of a sequence that straddles the previous match's end
    "start_rep",          # a repcode hit with the repcodes of a zstd-format dictionary, before the segment's first match
    "dict_cross",         # a match whose source straddles the dictionary / frame border
    "dict_back_cross",    # a catch-up that crosses the dictionary / frame border
]
# candidates the parse clears because they reach in front of the block's history (dL > p - lowLimit ...).  The walk only
# returns positions inside the chunk's history, so this happens only when the window is shorter than that history; the
# doubleFast rows never make it so (windowLog >= log2(frame + dictionary), chunk history <= 128 KiB + 512 KiB < window
# for every frame of more than one chunk).  tests/test_gpu_dfast_paths.py asserts that lowLimit is the chunk's history
# start on every block, which is why these rows stay zero.
CLEARED = ["clear_dl", "clear_ds", "clear_dl1"]

SWITCHES = {
    "f1_ge_ml": "upgrade when f1 >= ml instead of f1 > ml",
    "long_min6": "long candidates (and the upgrade) need 6 equal bytes instead of 8",
    "long_min9": "long candidates (and the upgrade) need 9 equal bytes instead of 8",
    "no_short_fallback": "a long collision ends the lane: its short candidate is not tried",
    "rep1_at_p": "repcode-1 checked at p instead of p+1",
    "step_shift7": "the probe step grows every 128 bytes instead of 256",
    "probe_9_to_8": "positions are probed while p + 8 <= blockEnd instead of p + 9",
    "rep1_after_long": "repcode-1 checked after the long candidate",
    "catchup_past_anchor": "the backward catch-up ignores the anchor",
}

# the same with 7: no input can tell it from the rule, a long candidate never has exactly 7 equal bytes (twin8_six)
EQUIVALENT = {"long_min7": "long candidates (and the upgrade) need 7 equal bytes instead of 8"}


def _fwd(buf, a, b, end):
    """ZSTD_count: equal bytes at a and b, a stopping at end"""
    n, k = 0, 8
    while True:
        if a + n + k <= end and buf[a + n:a + n + k] == buf[b + n:b + n + k]:
            n += k
            k = min(k * 2, 1 << 14)
        elif k > 1:
            k //= 2
        else:
            return n


def parse_segment(blk: Block, ss: int, se: int, sw=frozenset(), cnt=None):
    """parse_dfast_segment (oracle/zb_match.c:251-298): raw sequences (match start, length, real offset) of one segment"""
    buf, dL, dS, c0, be, low, D = blk.buf, blk.dL, blk.dS, blk.c0, blk.be, blk.low, blk.frame_start
    thr = 6 if "long_min6" in sw else (7 if "long_min7" in sw else (9 if "long_min9" in sw else 8))
    shift = 7 if "step_shift7" in sw else 8
    need = 8 if "probe_9_to_8" in sw else 9
    r1off = 0 if "rep1_at_p" in sw else 1
    rep1_late = "rep1_after_long" in sw
    no_fallback = "no_short_fallback" in sw
    f1_ge = "f1_ge_ml" in sw
    past_anchor = "catchup_past_anchor" in sw
    c = cnt if cnt is not None else {}

    def bump(k):
        c[k] = c.get(k, 0) + 1

    ip = anchor = search = ss
    rep1, rep2 = blk.start_reps if ss == blk.frame_start else (0, 0)
    inherited = rep1 or rep2
    out = []
    while ip < se and ip + need <= be:
        step = 1 + ((ip - search) >> shift)
        if step >= 2:
            bump("step_2")
        if step >= 12:
            bump("step_12")
        if step >= 32:
            bump("step_32")
        found = None
        for l in range(WARP):
            p = ip + l * step
            if p >= se:
                bump("lanes_cut_se")
                break
            if p + need > be:
                bump("lanes_cut_be")
                break
            dl, ds, dl1 = dL[p - c0], dS[p - c0], dL[p + 1 - c0]
            if dl and p < low + dl:
                dl = 0
                bump("clear_dl")
            if ds and p < low + ds:
                ds = 0
                bump("clear_ds")
            if dl1 and p + 1 < low + dl1:
                dl1 = 0
                bump("clear_dl1")
            cur = buf[p:p + 4]
            if l == 0 and ip == anchor and rep2 and buf[p - rep2:p - rep2 + 4] == cur:
                found = (3, p, rep2, 4 + _fwd(buf, p + 4, p + 4 - rep2, be), p)
                break
            q = p + r1off
            rep1_hit = rep1 and q >= low + rep1 and buf[q - rep1:q - rep1 + 4] == buf[q:q + 4]
            if rep1_hit and not rep1_late:
                found = (2, q, rep1, 4 + _fwd(buf, q + 4, q + 4 - rep1, be), q)
                break
            coll = False
            if dl:
                f = _fwd(buf, p, p - dl, be)
                if f >= thr:
                    found = (1, p, dl, f, p)
                    bump("long_hit")
                    if dl >= FAR:
                        bump("far_long")
                    break
                coll = True
                bump("long_coll_short" if ds else "long_coll_next")
            if rep1_hit:
                found = (2, q, rep1, 4 + _fwd(buf, q + 4, q + 4 - rep1, be), q)
                break
            if coll and no_fallback:
                continue
            if ds:
                if buf[p - ds:p - ds + 4] != cur:
                    bump("short_coll")
                    continue
                ml = _fwd(buf, p, p - ds, be)
                bump("short_hit")
                mp, mo = p, ds
                if dl1 and dl1 >= FAR:
                    bump("far_l1")
                if not dl1:
                    bump("keep_no_l1")
                else:
                    f1 = _fwd(buf, p + 1, p + 1 - dl1, be)
                    if f1 >= thr and (f1 >= ml if f1_ge else f1 > ml):
                        bump("upgrade")
                        mp, mo, ml = p + 1, dl1, f1
                    else:
                        bump("keep_l1_coll" if f1 < 4 else "keep_f1_lt8" if f1 < 8 else "keep_f1_eq" if f1 == ml else "keep_f1_lt")
                if mo == ds and ds >= FAR:
                    bump("far_short")
                found = (1, mp, mo, ml, mp)
                break
        if found is None:
            ip += WARP * step
            continue
        wtype, ms, off, mlen, probe = found
        if wtype == 3:
            bump("rep2_anchor")
        elif wtype == 2:
            bump("rep1_p1")
        if wtype in (2, 3) and inherited and not out:
            bump("start_rep")
        if (mlen if wtype == 1 else mlen - 4) >= 256:       # what the cooperative count measures
            bump("fwd_256")
        if wtype == 1:                                        # backward catch-up (zstd_double_fast.c:239-240, :282-283)
            mm = ms - off
            bound = low if past_anchor else anchor
            mm0 = mm
            while ms > bound and mm > low and buf[ms - 1] == buf[mm - 1]:
                ms -= 1
                mm -= 1
                mlen += 1
            if probe - ms >= 32:
                bump("back_32")
            if ms == anchor and mm > low and buf[ms - 1] == buf[mm - 1]:
                bump("back_stop_anchor")
            if mm == low and ms > anchor:
                bump("back_stop_low")
            if D and mm0 >= D > mm:
                bump("dict_back_cross")
        end = ms + mlen
        if be - end < 8:
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
        ip = anchor = search = ms + mlen
    if ip < se and ip < be and ip + need > be:
        bump("tail_unprobed")
    return out


def parse_block(blk: Block, sw=frozenset(), cnt=None, segment=None):
    """zbo_parseBlock (oracle/zb_match.c:308-352): the segments' raw sequences joined, repcodes assigned over the block
    (mergegen.join, the restatement the merge kernels are tested against).
    `segment` parses one segment (default: the doubleFast parse above; fastgen.parse_segment for the fast parse)."""
    import mergegen
    c = cnt if cnt is not None else {}
    segment = segment or parse_segment
    segs = [segment(blk, ss, min(ss + SEG, blk.be), sw, c) for ss in range(blk.bs, blk.be, SEG)]
    reps = blk.code_reps if blk.bs == blk.frame_start else (0, 0, 0)
    return mergegen.join(segs, reps, blk.bs, sw, c)


# -------------------------------------------------------------------------------------------------- the GPU cases
SIZE_CLASSES = {
    # > 256 KiB: two chunks (the second primed from 128 KiB) and a last block of 3 bytes
    "gt256k": 6 * BLOCK + 3,
    # <= 256 KiB: exactly 256 KiB, two blocks
    "le256k": 2 * BLOCK,
    # <= 128 KiB: one block that ends 5 bytes short of 128 KiB
    "le128k": BLOCK - 5,
    # <= 16 KiB: one segment minus one byte
    "le16k": SEG - 1,
}
# (size class, level): levels 3 and 4 everywhere, level 2 where it is doubleFast, one level >= 5 per class
FRAME_CASES = [("gt256k", 3), ("gt256k", 4), ("gt256k", 5),
               ("le256k", 2), ("le256k", 3), ("le256k", 4), ("le256k", 9),
               ("le128k", 3), ("le128k", 4), ("le128k", 19),
               ("le16k", 3), ("le16k", 4), ("le16k", 22)]
# one chunk without priming, and a frame of five walk batches whose window (2^13) shrinks the short table to 8192 buckets
EXTRA_FRAMES = [("one_chunk", 4 * BLOCK - 1, 3), ("small", 5000, 4)]
DICT_LEVELS = [3, 4]
DICT_NAMES = ["raw-20k", "raw-150k", "zdict-16k", "zdict-16k-reps"]
PATCHED_REPS = (3, 17, 4099)
BATCH_LEVEL = 3

_cache = {}


def frame_input(name: str) -> bytes:
    key = ("in", name)
    if key not in _cache:
        size = SIZE_CLASSES.get(name) or {n: s for n, s, _ in EXTRA_FRAMES}[name]
        _cache[key] = dfast_input(size, 1000 + size % 977)
    return _cache[key]


def dictionary(name: str) -> bytes:
    key = ("dict", name)
    if key not in _cache:
        if name == "raw-20k":
            d = dfast_input(20 << 10, 41)
        elif name == "raw-150k":
            d = dfast_input(150 << 10, 42)
        elif name == "zdict-16k":
            d = zref.golden_input("zdict-16k-synthetic-seed77")
        else:
            d = patch_reps(zref.golden_input("zdict-16k-synthetic-seed77"), PATCHED_REPS)
        _cache[key] = d
    return _cache[key]


def dict_inputs(name: str):
    """inputs compressed against a dictionary: one in each of two size classes (with the dictionary counted in), each
    starting with copies across the dictionary / frame border"""
    key = ("din", name)
    if key not in _cache:
        d = dictionary(name)
        off = dict_content_offset(d)
        tail = d[off:][-(128 << 10):]
        start = None
        if off:
            reps = [int.from_bytes(d[off - 12 + 4 * i:off - 8 + 4 * i], "little") for i in range(3)]
            start = (reps[0], reps[1])
        seed = sum(name.encode())
        _cache[key] = [dfast_input(40 << 10, seed, tail, start), dfast_input(BLOCK + 3 * SEG + 7, seed + 1, tail, start)]
    return _cache[key]


def batch_small():
    """frames of at most 8 KiB, one call: one segment per block"""
    if ("bs",) not in _cache:
        rnd = random.Random(5)
        data = dfast_input(200 << 10, 77)
        frames, p = [], 0
        for i in range(40):
            n = rnd.choice([7, 8, 9, 100, 1000, 4096, 5000, 8191, 8192]) if i % 4 else rnd.randint(10, 8192)
            frames.append(data[p:p + n])
            p += n
        _cache[("bs",)] = frames
    return _cache[("bs",)]


def batch_mixed():
    """large and small frames in one call: eight segments per block, and blocks that leave segments empty"""
    if ("bm",) not in _cache:
        big = dfast_input(3 * BLOCK + SEG + 9, 78)
        mid = dfast_input(BLOCK + 100, 79)
        small = [dfast_input(n, 80 + n) for n in (9, 777, 8192, 20000, 3 * SEG + 2)]
        _cache[("bm",)] = [small[0], big, small[1], small[2], mid, small[3], small[4]]
    return _cache[("bm",)]


def all_frames():
    """(src, level, dictionary or None) of every frame the GPU tests compress, de-duplicated"""
    seen, out = set(), []

    def add(src, level, d):
        k = (zref.sha(src), level, zref.sha(d) if d else None)
        if k not in seen:
            seen.add(k)
            out.append((src, level, d))
    for cls, level in FRAME_CASES:
        add(frame_input(cls), level, None)
    for name, _, level in EXTRA_FRAMES:
        add(frame_input(name), level, None)
    for name in DICT_NAMES:
        for level in DICT_LEVELS:
            for src in dict_inputs(name):
                add(src, level, dictionary(name))
    for f in batch_small() + batch_mixed():
        add(f, BATCH_LEVEL, None)
    return out
