"""Test helpers for frames with chosen contents: a plain LZ77 executor (the reference answer), the reference encoder's
sequence API (ZSTD_compressSequences, lib/zstd.h:1642) and advanced-parameter API (ZSTD_CCtx_setParameter,
ZSTD_compress2, ZSTD_compressStream2), and a parser of frame and block headers that lets a test assert the frame has the
shape it was built for.  Everything but execute() and frame_layout() needs oracle/_ref/libzstd_ref.so.  TEST
INFRASTRUCTURE ONLY."""
import ctypes

import numpy as np

import zref

_sz, _vp = ctypes.c_size_t, ctypes.c_void_p

# lib/zstd.h parameter numbers
C_LEVEL, C_WINDOWLOG, C_MINMATCH, C_TARGET_CBLOCK, C_LDM = 100, 101, 105, 130, 160
C_CONTENTSIZE, C_CHECKSUM = 200, 201
C_LITERAL_MODE, C_BLOCK_DELIMITERS, C_VALIDATE_SEQUENCES, C_MAX_BLOCK_SIZE, C_REPCODE_SEARCH = 1002, 1008, 1009, 1015, 1016
BT_RAW, BT_RLE, BT_COMPRESSED = 0, 1, 2


class Sequence(ctypes.Structure):
    _fields_ = [("offset", ctypes.c_uint), ("litLength", ctypes.c_uint), ("matchLength", ctypes.c_uint), ("rep", ctypes.c_uint)]


class InBuffer(ctypes.Structure):
    _fields_ = [("src", _vp), ("size", _sz), ("pos", _sz)]


class OutBuffer(ctypes.Structure):
    _fields_ = [("dst", _vp), ("size", _sz), ("pos", _sz)]


_bound = False


def ref():
    global _bound
    R = zref.ref()
    if not _bound:
        R.ZSTD_CCtx_setParameter.restype = _sz
        R.ZSTD_CCtx_setParameter.argtypes = [_vp, ctypes.c_int, ctypes.c_int]
        R.ZSTD_CCtx_loadDictionary.restype = _sz
        R.ZSTD_CCtx_loadDictionary.argtypes = [_vp, _vp, _sz]
        R.ZSTD_compressSequences.restype = _sz
        R.ZSTD_compressSequences.argtypes = [_vp, _vp, _sz, _vp, _sz, _vp, _sz]
        R.ZSTD_compress2.restype = _sz
        R.ZSTD_compress2.argtypes = [_vp, _vp, _sz, _vp, _sz]
        R.ZSTD_compressStream2.restype = _sz
        R.ZSTD_compressStream2.argtypes = [_vp, ctypes.POINTER(OutBuffer), ctypes.POINTER(InBuffer), ctypes.c_int]
        R.ZDICT_getDictHeaderSize.restype = _sz
        R.ZDICT_getDictHeaderSize.argtypes = [_vp, _sz]
        _bound = True
    return R


def _check(R, r):
    assert not R.ZSTD_isError(r), R.ZSTD_getErrorName(r).decode()
    return r


def execute(blocks, rng, dict_content=b"", alphabet=256):
    """The input a list of blocks describes.  blocks: [(sequences, trailing_literals)], a sequence is (litLength, offset,
    matchLength).  Literal bytes are drawn from rng (numpy Generator) among the first `alphabet` byte values; a match
    copies byte after byte, so it may overlap itself, and an offset beyond the output so far reads from the end of
    dict_content."""
    h = bytearray(dict_content)

    def lits(n):
        h.extend(rng.integers(0, alphabet, n, dtype="u1").tobytes())
    for seqs, trailing in blocks:
        for ll, off, ml in seqs:
            lits(ll)
            assert 0 < off <= len(h), (off, len(h))
            s = len(h) - off
            while ml:                                   # the `off` bytes in front of the match, again and again
                n = min(ml, off)
                h.extend(h[s:s + n])
                s += n
                ml -= n
        lits(trailing)
    return bytes(h[len(dict_content):])


def dict_content(d):
    """the content part of a dictionary: all of a raw one, behind the entropy tables of a zstd-format one"""
    return d[ref().ZDICT_getDictHeaderSize(d, len(d)):] if d[:4] == b"\x37\xa4\x30\xec" else d


def _cctx(R, params, dict=None):
    c = R.ZSTD_createCCtx()
    for k, v in params:
        _check(R, R.ZSTD_CCtx_setParameter(c, k, v))
    if dict is not None:
        _check(R, R.ZSTD_CCtx_loadDictionary(c, dict, len(dict)))
    return c


def ref_compress_sequences(blocks, src, level=3, dict=None, params=()):
    """ZSTD_compressSequences with explicit block delimiters: one block of the frame per entry of `blocks`, the
    sequences as given.  ZSTD_c_searchForExternalRepcodes makes the reference code an offset the history holds as a
    repcode (below level 10 it would write every offset in full)."""
    R = ref()
    arr = []
    for seqs, trailing in blocks:
        arr += [(off, ll, ml, 0) for ll, off, ml in seqs] + [(0, trailing, 0, 0)]
    seq = (Sequence * len(arr))(*arr)
    c = _cctx(R, [(C_LEVEL, level), (C_BLOCK_DELIMITERS, 1), (C_VALIDATE_SEQUENCES, 1), (C_MINMATCH, 3), (C_REPCODE_SEARCH, 1)] + list(params), dict)
    cap = R.ZSTD_compressBound(len(src)) + 4096
    dst = ctypes.create_string_buffer(cap)
    r = R.ZSTD_compressSequences(c, dst, cap, seq, len(arr), src, len(src))
    R.ZSTD_freeCCtx(c)
    return dst.raw[:_check(R, r)]


def ref_compress2(src, params, stream=False):
    """ZSTD_compress2 after ZSTD_CCtx_setParameter, or (stream=True) ZSTD_compressStream2 fed 1 MiB at a time and
    ended separately, so the frame carries no content size"""
    R = ref()
    c = _cctx(R, params)
    cap = R.ZSTD_compressBound(len(src)) + (1 << 16)
    dst = ctypes.create_string_buffer(cap)
    if not stream:
        r = R.ZSTD_compress2(c, dst, cap, src, len(src))
        R.ZSTD_freeCCtx(c)
        return dst.raw[:_check(R, r)]
    sbuf = ctypes.create_string_buffer(src, max(len(src), 1))
    base = ctypes.cast(sbuf, ctypes.c_void_p).value
    out = OutBuffer(ctypes.cast(dst, ctypes.c_void_p), cap, 0)
    for p in range(0, len(src), 1 << 20):
        n = min(1 << 20, len(src) - p)
        i = InBuffer(base + p, n, 0)
        while i.pos < i.size:
            _check(R, R.ZSTD_compressStream2(c, ctypes.byref(out), ctypes.byref(i), 0))
    i = InBuffer(base, 0, 0)
    while _check(R, R.ZSTD_compressStream2(c, ctypes.byref(out), ctypes.byref(i), 2)):
        pass
    R.ZSTD_freeCCtx(c)
    return dst.raw[:out.pos]


def ref_decompress(frames, cap, dict=None):
    """the reference decoder over one or more frames, with the dictionary if one is given; raises on an error"""
    return zref.ref_decompress_using_dict(frames, dict, cap) if dict else zref.ref_decompress(frames, cap)


def frame_layout(buf):
    """The frames of a buffer, header by header (format: "Frames", "Blocks", "Literals_Section_Header",
    "Sequences_Section_Header").  One dict per frame: skippable, single_segment, checksum, window_log (None for
    Single_Segment), content_size (None when absent), blocks = [(type, block_size, lit_type, nb_seq, nb_seq_bytes)]
    (the last three None for raw and RLE blocks) and size (compressed bytes)."""
    frames, pos = [], 0
    while pos < len(buf):
        start = pos
        magic = int.from_bytes(buf[pos:pos + 4], "little")
        if magic & 0xFFFFFFF0 == 0x184D2A50:
            pos += 8 + int.from_bytes(buf[pos + 4:pos + 8], "little")
            frames.append({"skippable": True, "size": pos - start})
            continue
        assert magic == 0xFD2FB528, hex(magic)
        fhd = buf[pos + 4]
        single, fcs_flag, did_flag = (fhd >> 5) & 1, fhd >> 6, fhd & 3
        pos += 5
        f = {"skippable": False, "single_segment": bool(single), "checksum": bool(fhd & 4), "window_log": None, "blocks": []}
        if not single:
            f["window_log"] = 10 + (buf[pos] >> 3)
            pos += 1
        pos += (0, 1, 2, 4)[did_flag]
        fcs_bytes = (single, 2, 4, 8)[fcs_flag]
        fcs = int.from_bytes(buf[pos:pos + fcs_bytes], "little") if fcs_bytes else None
        f["content_size"] = fcs + 256 if fcs_bytes == 2 else fcs
        pos += fcs_bytes
        while True:
            bh = int.from_bytes(buf[pos:pos + 3], "little")
            last, btype, bsize = bh & 1, (bh >> 1) & 3, bh >> 3
            pos += 3
            if btype == BT_COMPRESSED:
                c = buf[pos:pos + bsize]
                lt, sf = c[0] & 3, (c[0] >> 2) & 3
                if lt < 2:
                    hs = (1, 2, 1, 3)[sf]
                    regen = int.from_bytes(c[:hs], "little") >> (3 if hs == 1 else 4)
                    body = regen if lt == 0 else 1
                else:
                    hs = (3, 3, 4, 5)[sf]
                    v = int.from_bytes(c[:hs], "little") >> 4
                    bits = (10, 10, 14, 18)[sf]
                    body = v >> bits
                s = hs + body
                nb = c[s] if c[s] < 128 else (((c[s] - 128) << 8) + c[s + 1] if c[s] < 255 else c[s + 1] + (c[s + 2] << 8) + 0x7F00)
                nbb = 1 if c[s] < 128 else (2 if c[s] < 255 else 3)
                f["blocks"].append((btype, bsize, lt, nb, nbb))
            else:
                f["blocks"].append((btype, bsize, None, None, None))
            pos += 1 if btype == BT_RLE else bsize
            if last:
                break
        pos += 4 if f["checksum"] else 0
        f["size"] = pos - start
        frames.append(f)
    return frames


# ---------------------------------------------------------------------------------------------------- the cases
# Each builder returns (frames, expected input, dictionary or None) and asserts the frame has the shape it is built for:
# the reference may fall back to raw or RLE blocks, and a case that silently did would test nothing.

GRID_OFFSETS = list(range(1, 71)) + [127, 128, 129, 255, 256, 1000, 4095, 4096, 65535, 65536, 131072]
GRID_LENGTHS = [3, 4, 5, 7, 8, 9, 15, 16, 17, 31, 32, 33, 35, 36, 37, 64, 65, 200, 1000]
ZDICT = "zdict-16k-synthetic-seed77"


def _compressed(f, idx):
    for i in idx:
        assert f["blocks"][i][0] == BT_COMPRESSED and f["blocks"][i][3] > 0, (i, f["blocks"][i])


def _one(blocks, seed, level=3, dict=None, params=(), alphabet=256):
    src = execute(blocks, np.random.default_rng(seed), dict_content(dict) if dict else b"", alphabet)
    frame = ref_compress_sequences(blocks, src, level, dict, params)
    [f] = frame_layout(frame)
    assert len(f["blocks"]) == len(blocks), (len(f["blocks"]), len(blocks))
    return frame, src, f


def copy_grid():
    """every offset of GRID_OFFSETS with every length of GRID_LENGTHS, the match starting at each of the four
    positions mod 4 (with the offset: the source at each of the four too); one block per offset, behind 132 KiB of
    random history"""
    blocks, pos = [([], 131072), ([], 1000)], 132072
    for off in GRID_OFFSETS:
        seqs = []
        for ml in GRID_LENGTHS:
            for a in range(4):
                ll = 1 + (a - pos - 1) % 4
                seqs.append((ll, off, ml))
                pos += ll + ml
        blocks.append((seqs, 0))
    frame, src, f = _one(blocks, 1)
    _compressed(f, range(2, len(blocks)))
    return frame, src, None


def repcodes():
    """84 small blocks of sequences whose offsets repeat the history's on purpose: each repeat offset with and without
    literals in front, and "offset_1 - 1" behind none; the history runs through all blocks (the scan composes 32 per
    round)"""
    rng = np.random.default_rng(2)
    rep = [1, 4, 8]
    blocks, pos = [([(8, 4, 5), (0, 8, 6), (3, 1, 4), (0, 4, 9)], 2)], 34
    for s in blocks[0][0]:
        rep = _rep_update(rep, s[1], s[0])
    kinds = 0
    for b in range(84):
        seqs = []
        for i in range(8):
            ll = int(rng.choice([0, 0, 1, 2, 5]))
            k = int(rng.integers(0, 5))
            off = [rep[0], rep[1], rep[2], rep[0] - 1, int(rng.integers(16, 1500))][k]
            if off < 1 or off > pos + ll:
                off = 1 + int(rng.integers(0, pos + ll))
            ml = int(rng.integers(4, 24))
            seqs.append((ll, off, ml))
            kinds |= 1 << (k + (5 if ll == 0 else 0))
            rep = _rep_update(rep, off, ll)
            pos += ll + ml
        blocks.append((seqs, int(rng.integers(0, 3))))
        pos += blocks[-1][1]
    assert kinds == (1 << 10) - 1
    frame, src, f = _one(blocks, 3)
    _compressed(f, range(1, len(blocks)))
    return frame, src, None


def _rep_update(rep, off, ll):
    """the format's repeat offsets behind a sequence of this offset, coded as the reference codes it (ZSTD_finalizeOffBase)"""
    if ll and off == rep[0]:
        return rep
    if off == rep[1]:
        return [rep[1], rep[0], rep[2]]
    if off == rep[2]:
        return [rep[2], rep[0], rep[1]]
    return [off, rep[0], rep[1]]


def chain():
    """one block of 40 000 matches (offset 3, length 3, no literals): every match reads the one before it"""
    frame, src, f = _one([([(3, 3, 3)] + [(0, 3, 3)] * 39_999, 0)], 4)
    _compressed(f, [0])
    return frame, src, None


def chain_blocks():
    """short-offset chains that go on through block boundaries, and a match whose source is the frame's first byte
    (offset == position), at the frame's start and in a later block"""
    blocks = [([(100, 100, 50), (5, 7, 30)] + [(0, 3, 3)] * 500, 0)]
    for b in range(6):
        blocks.append(([(0, 3, 3)] * 400 + [(0, 5, 7)] * 100 + [(1, 2, 9)] * 30, 1))
    pos = sum(ll + ml for seqs, t in blocks for ll, off, ml in seqs) + sum(t for seqs, t in blocks)
    blocks.append(([(10, pos + 10, 40), (0, 6, 6)], 0))
    frame, src, f = _one(blocks, 5)
    _compressed(f, range(len(blocks)))
    return frame, src, None


def tile():
    """16 matches of 4 bytes write one 64-byte tile of the output; then 60 matches read from that tile"""
    seqs = [(64, 1000, 4)] + [(0, 1000 + 7 * k, 4) for k in range(1, 16)]
    P = 4096 + 64
    pos = P + 64
    for j in range(60):
        pos += 1
        seqs.append((1, pos - (P + j % 56), 3 + j % 6))
        pos += 3 + j % 6
    frame, src, f = _one([([], 4096), (seqs, 5)], 6)
    _compressed(f, [1])
    return frame, src, None


def block_extremes():
    """one 131 072-byte match filling a block; a block of 131 072 literals and one of 300, both without sequences"""
    blocks = [([], 5000), ([(0, 1000, 131072)], 0), ([], 131072), ([(4, 100, 50)], 10), ([], 300), ([(4, 100, 50)], 10)]
    frame, src, f = _one(blocks, 7, alphabet=16)
    _compressed(f, [1, 3, 5])
    for i in (2, 4):
        assert f["blocks"][i][0] == BT_COMPRESSED and f["blocks"][i][2] >= 2 and f["blocks"][i][3] == 0, f["blocks"][i]
    return frame, src, None


def nbseq_boundaries():
    """blocks of 127, 128, 0x7EFF and 0x7F00 sequences: the 1, 2 and 3-byte forms of the count"""
    rng = np.random.default_rng(8)
    blocks = [([], 2000)]
    for n in (127, 128, 0x7EFF, 0x7F00):
        blocks.append(([(i & 1, int(rng.integers(3, 40)), 3) for i in range(n)], 0))
    frame, src, f = _one(blocks, 9)
    assert [(b[0], b[3], b[4]) for b in f["blocks"][1:]] == [(2, 127, 1), (2, 128, 2), (2, 0x7EFF, 2), (2, 0x7F00, 3)]
    return frame, src, None


def window_1k():
    """ZSTD_c_windowLog 10: blocks of at most 1 KiB, matches at an offset equal to the window"""
    blocks = [([], 1020)] + [([(10, 1024, 100), (5, 37, 50), (0, 1024, 200), (3, 600, 300)], 100)] * 7
    frame, src, f = _one(blocks, 10, params=[(C_WINDOWLOG, 10)])
    assert f["window_log"] == 10 and max(b[1] for b in f["blocks"]) <= 1024
    _compressed(f, range(1, len(blocks)))
    return frame, src, None


def multi_frame():
    """dictated frames, an empty frame and skippable frames in one call; the matches of the second dictated frame reach
    back exactly to its first byte"""
    a, sa, fa = _one([([(20, 7, 40)] * 50, 3)], 11)
    b, sb, fb = _one([([(100, 100, 60), (0, 160, 30), (3, 193, 100)], 5), ([(2, 300, 64)], 0)], 12)
    c, sc, fc = _one([([(9, 9, 9)] * 20, 0)], 13)
    for f in (fa, fb, fc):
        _compressed(f, range(len(f["blocks"])))
    skip = bytes([0x5E, 0x2A, 0x4D, 0x18, 3, 0, 0, 0]) + b"abc"
    frames = a + zref.ref_compress(b"", 3) + skip + b + skip + c
    assert len(frame_layout(frames)) == 6
    return frames, sa + sb + sc, None


def dict_straddle(kind):
    """matches that begin in the dictionary's content and continue into the frame, at every split point, and matches
    wholly inside the content"""
    d = zref.golden_input(ZDICT) if kind == "zdict" else zref.synthetic(20_000, 5, 0.5)
    n = len(dict_content(d))
    seqs, pos = [], 0
    for ml in (4, 17, 40):
        for k in range(1, ml):
            pos += 1
            seqs.append((1, pos + k, ml))
            pos += ml
    for j in range(30):
        pos += 2
        seqs.append((2, min(pos + 20 + 97 * j, n + pos), 20))
        pos += 20
    frame, src, f = _one([(seqs, 7)], 14, dict=d)
    _compressed(f, [0])
    return frame, src, d


DICTATED = {"copy-grid": copy_grid, "repcodes": repcodes, "chain-40000": chain, "chain-blocks": chain_blocks, "tile": tile,
            "block-extremes": block_extremes, "nbseq-boundaries": nbseq_boundaries, "window-1k": window_1k,
            "multi-frame": multi_frame, "dict-straddle-raw": lambda: dict_straddle("raw"),
            "dict-straddle-zdict": lambda: dict_straddle("zdict")}


# ---------------------------------------------------------------------------------------------------- advanced parameters
# Each builder returns (frames, expected input, or the error code a decoder whose offsets are kept in 28 bits must give).
def _adv(src, params, stream=False, **shape):
    frame = ref_compress2(src, params, stream)
    fs = frame_layout(frame)
    for f in fs:
        for k, v in shape.items():
            assert f[k] == v, (k, f[k], v)
        if stream:
            assert f["content_size"] is None
    return frame, fs


def no_content_size():
    src = zref.synthetic(3 << 20, 21, 0.6)
    return _adv(src, [(C_CONTENTSIZE, 0)], content_size=None)[0], src


def streamed():
    src = zref.synthetic(3 << 20, 22, 0.6) + zref.random_bytes(100_000, 22)
    return _adv(src, [(C_LEVEL, 5)], stream=True)[0], src


def streamed_checksums():
    """three streamed frames with content checksums, none stating its size"""
    srcs = [zref.synthetic((1 << 20) + 7, 23, 0.5), zref.synthetic(2 << 20, 24, 0.8), zref.synthetic(300_001, 25, 0.3)]
    return b"".join(_adv(s, [(C_CHECKSUM, 1)], stream=True, checksum=True)[0] for s in srcs), b"".join(srcs)


def target_cblock():
    """ZSTD_c_targetCBlockSize 1340: hundreds of small blocks, tables reused many blocks later"""
    src = zref.synthetic(4 << 20, 26, 0.6)
    frame, [f] = _adv(src, [(C_TARGET_CBLOCK, 1340)])
    comp = [b for b in f["blocks"] if b[0] == BT_COMPRESSED]
    assert len(comp) > 300 and any(b[2] == 3 for b in comp), len(comp)
    return frame, src


def max_block_1k():
    src = zref.synthetic(1 << 20, 27, 0.6)
    frame, [f] = _adv(src, [(C_MAX_BLOCK_SIZE, 1024)])
    assert len(f["blocks"]) >= 1024 and max(b[1] for b in f["blocks"]) <= 1024
    return frame, src


def window_1k_streamed():
    src = zref.synthetic(1 << 20, 28, 0.7)
    return _adv(src, [(C_WINDOWLOG, 10)], stream=True, window_log=10)[0], src


def literal_mode(mode):
    """ZSTD_c_literalCompressionMode: 2 = raw literals in every compressed block, 1 = always Huffman"""
    src = zref.synthetic(2 << 20, 29, 0.5)
    frame, [f] = _adv(src, [(C_LITERAL_MODE, mode)])
    comp = [b for b in f["blocks"] if b[0] == BT_COMPRESSED]
    assert comp and all((b[2] == 0) if mode == 2 else (b[2] >= 2) for b in comp)
    return frame, src


def level22():
    src = zref.synthetic(1 << 20, 30, 0.6)
    return _adv(src, [(C_LEVEL, 22)])[0], src


def _far(x, gap):
    xs = zref.random_bytes(x, 31)
    return xs + zref.random_bytes(gap, 32) + xs


def ldm_128m(stream):
    """long-distance matching, window 2^27, on X (8 MiB) + 112 MiB random + X: offsets of about 120 MiB; one shot
    (Single_Segment) or streamed (window descriptor, no content size)"""
    src = _far(8 << 20, 112 << 20)
    shape = {"window_log": 27} if stream else {"single_segment": True}
    return _adv(src, [(C_LDM, 1), (C_WINDOWLOG, 27), (C_LEVEL, 1)], stream, **shape)[0], src


def wlog28_streamed():
    """a window descriptor of 2^28: refused with 16 (frameParameter_windowTooLarge)"""
    src = zref.synthetic(2 << 20, 33, 0.6)
    return _adv(src, [(C_WINDOWLOG, 28)], stream=True, window_log=28)[0], src


def ldm_264m_single():
    """X (4 MiB) + 256 MiB random + X with long-distance matching and window 2^29, one shot: a Single_Segment frame
    (it states no window) whose offsets need 29 bits.  Refused with 16 at the first such offset."""
    src = _far(4 << 20, 256 << 20)
    return _adv(src, [(C_LDM, 1), (C_WINDOWLOG, 29), (C_LEVEL, 1)], single_segment=True, content_size=len(src))[0], src


ADVANCED = {"no-content-size": no_content_size, "streamed": streamed, "streamed-checksums": streamed_checksums,
            "target-cblock-1340": target_cblock, "max-block-1k": max_block_1k, "window-1k-streamed": window_1k_streamed,
            "raw-literals": lambda: literal_mode(2), "huffman-literals": lambda: literal_mode(1), "level-22": level22,
            "ldm-128m": lambda: ldm_128m(False), "ldm-128m-streamed": lambda: ldm_128m(True)}
REFUSED = {"wlog28-streamed": wlog28_streamed, "ldm-264m-single": ldm_264m_single}
