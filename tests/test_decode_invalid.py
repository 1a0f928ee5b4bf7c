"""The decoder on invalid inputs, held to the compiled reference decoder's verdict.  One corpus: constructed cases, each
aimed at one check (a block that regenerates more than its frame's window, raw and RLE blocks larger than the window,
offsets that reach in front of the frame, content-size fields off by one, a failing frame among valid ones, a
destination one byte short), and a seeded corpus of bit flips, byte overwrites and truncations of frames of both encoders,
single-segment and streamed, single and concatenated, with and without the golden zstd-format dictionary.  Every input
gets the verdict of the reference's ZSTD_decompress[_usingDict], and of its ZSTD_decompressStream where that can differ.

What every input must satisfy, on every path (the CPU harness tests/host_decode.cpp; on the GPU the host call, the
device call at byte offset 1, the walk kernel, ZSTD_decompressStream in pieces):
  * the reference refuses -> this decoder refuses, with a code other than GENERIC (1: the match stage's watchdog or an
    internal failure);
  * both accept -> the bytes are equal;
  * the reference accepts and this decoder refuses -> the input is one of DIFFERENCES;
  * no byte outside [dst, dst + dstCapacity) changes;
  * all one-shot paths give the same verdict;
  * the context still decodes a valid frame afterwards.
The corpus also runs once through the harness built with -fsanitize=address,undefined."""
import collections
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

import seqgen
import zref

HERE = os.path.dirname(os.path.abspath(__file__))
needs_ref = pytest.mark.skipif(not zref.have_ref(), reason="reference library not built")
_sz, _vp = ctypes.c_size_t, ctypes.c_void_p
GUARD = 0xA5
GENERIC = 1
CORPUS_CPU, CORPUS_GPU = 2000, 600

# The reference accepts these and this decoder refuses them, on purpose:
DIFFERENCES = {
    "offset-beyond-27-bits": "offsets are kept in 28 bits: a window above 2^27, or an offset code above 27, is "
                             "frameParameter_windowTooLarge (16) whatever the header says",
    "block-over-window": "a block larger than Block_Maximum_Size = min(window, 128 KiB): a raw or RLE block of that size, "
                         "or a compressed block whose matches regenerate up to ~32 bytes more (its literal buffer lies "
                         "behind that room).  The reference's one-shot call takes them, its streaming call refuses them, "
                         "and so does this decoder (corruption_detected)",
    "huffman-start-overread": "a Huffman stream that reads past its first byte: corruption_detected",
}


# ---------------------------------------------------------------------------------------------------- decoders
@pytest.fixture(scope="module")
def build_dir(tmp_path_factory):
    """where the harness is compiled: a fresh directory, since the tree may not be writable by whoever runs the tests"""
    return str(tmp_path_factory.mktemp("hostdecode"))


@pytest.fixture(scope="module")
def H(build_dir):
    """the CPU harness: the decoder's format code, block after block"""
    so = os.path.join(build_dir, "libzb_hostdecode_invalid.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-Wall", "-Wextra", "-Werror", "-Wno-unused-function", "-x", "c++",
                           "-o", so, os.path.join(HERE, "host_decode.cpp")])
    h = ctypes.CDLL(so)
    h.zbh_decompress_usingDict.restype = _sz
    h.zbh_decompress_usingDict.argtypes = [_vp, _sz, _vp, _sz, _vp, _sz]
    return h


def _code(r):
    return (1 << 64) - r if r > (1 << 63) else None


def harness(H, buf, cap, d=None):
    """(result, zbh_refusedBy): result is the output, or ("ERR", code); zbh_refusedBy: 1 = refused at the end of a Huffman
    stream, 2 = refused a compressed block that regenerates more than its frame's window"""
    out = ctypes.create_string_buffer(bytes([GUARD]) * (cap + 16), cap + 16)
    r = H.zbh_decompress_usingDict(out, cap, buf, len(buf), d, len(d) if d else 0)
    assert out.raw[cap:] == bytes([GUARD]) * 16, "bytes behind the destination changed"
    return (("ERR", _code(r)) if _code(r) else out.raw[:r]), ctypes.c_uint.in_dll(H, "zbh_refusedBy").value


def _ref():
    R = seqgen.ref()
    R.ZSTD_getErrorCode.restype = ctypes.c_int
    R.ZSTD_getErrorCode.argtypes = [_sz]
    return R


def _bind_stream(L):
    L.ZSTD_createDStream.restype = _vp
    L.ZSTD_freeDStream.argtypes = [_vp]
    L.ZSTD_initDStream.restype = _sz
    L.ZSTD_initDStream.argtypes = [_vp]
    L.ZSTD_decompressStream.restype = _sz
    L.ZSTD_decompressStream.argtypes = [_vp, ctypes.POINTER(seqgen.OutBuffer), ctypes.POINTER(seqgen.InBuffer)]
    if hasattr(L, "ZSTD_initDStream_usingDict"):
        L.ZSTD_initDStream_usingDict.restype = _sz
        L.ZSTD_initDStream_usingDict.argtypes = [_vp, _vp, _sz]
    return L


def ref_oneshot(buf, cap, d=None, checksums=True):
    """the reference's ZSTD_decompress_usingDict; checksums=False: with ZSTD_d_forceIgnoreChecksum, the verdict for the
    paths that do not verify content checksums (the device calls and the harness)"""
    R = _ref()
    R.ZSTD_DCtx_setParameter.restype = _sz
    R.ZSTD_DCtx_setParameter.argtypes = [_vp, ctypes.c_int, ctypes.c_int]
    out = ctypes.create_string_buffer(max(cap, 1))
    dctx = R.ZSTD_createDCtx()
    if not checksums:
        assert not R.ZSTD_isError(R.ZSTD_DCtx_setParameter(dctx, 1002, 1))          # ZSTD_d_forceIgnoreChecksum
    r = R.ZSTD_decompress_usingDict(dctx, out, cap, buf, len(buf), d, len(d) if d else 0)
    R.ZSTD_freeDCtx(dctx)
    return ("ERR", R.ZSTD_getErrorCode(r)) if R.ZSTD_isError(r) else out.raw[:r]


def stream(L, buf, d=None, piece=4093, room=1 << 17):
    """ZSTD_decompressStream of library L: the input in `piece`-byte pieces, the output through a `room`-byte buffer.
    ("INCOMPLETE", None) when the input ends inside a frame."""
    zds = L.ZSTD_createDStream()
    assert not L.ZSTD_isError(L.ZSTD_initDStream_usingDict(zds, d, len(d)) if d else L.ZSTD_initDStream(zds))
    src = ctypes.create_string_buffer(buf, max(len(buf), 1))
    base = ctypes.cast(src, ctypes.c_void_p).value
    out = ctypes.create_string_buffer(room)
    got, pos, last = bytearray(), 0, 0
    try:
        while pos < len(buf):
            i = seqgen.InBuffer(base + pos, min(piece, len(buf) - pos), 0)
            while True:
                o = seqgen.OutBuffer(ctypes.cast(out, ctypes.c_void_p), room, 0)
                last = L.ZSTD_decompressStream(zds, ctypes.byref(o), ctypes.byref(i))
                if L.ZSTD_isError(last):
                    return ("ERR", L.ZSTD_getErrorCode(last))
                got += out.raw[:o.pos]
                if i.pos == i.size and o.pos < room:
                    break
            pos += i.size
    finally:
        L.ZSTD_freeDStream(zds)
    return bytes(got) if last == 0 else ("INCOMPLETE", None)


# ---------------------------------------------------------------------------------------------------- frame surgery
def layout(buf):
    """frames of a (possibly corrupt) buffer, as far as their headers can be followed: dicts of start, header (bytes),
    single_segment, window (None for Single_Segment), fcs = (offset, bytes) of the content-size field, and blocks =
    [(position of the block header, type, Block_Size)]"""
    frames, pos = [], 0
    try:
        while pos + 8 <= len(buf):
            magic = int.from_bytes(buf[pos:pos + 4], "little")
            if magic & 0xFFFFFFF0 == 0x184D2A50:
                pos += 8 + int.from_bytes(buf[pos + 4:pos + 8], "little")
                continue
            if magic != 0xFD2FB528:
                break
            fhd = buf[pos + 4]
            single, fcs_flag, did_flag = (fhd >> 5) & 1, fhd >> 6, fhd & 3
            f = {"start": pos, "single_segment": bool(single), "window": None, "blocks": []}
            p = pos + 5
            if not single:
                wl = 10 + (buf[p] >> 3)
                f["window"] = (1 << wl) + ((1 << wl) >> 3) * (buf[p] & 7)
                p += 1
            p += (0, 1, 2, 4)[did_flag]
            fcs_bytes = (single, 2, 4, 8)[fcs_flag]
            f["fcs"] = (p, fcs_bytes)
            p += fcs_bytes
            f["header"] = p - pos
            frames.append(f)
            while p + 3 <= len(buf):
                bh = int.from_bytes(buf[p:p + 3], "little")
                f["blocks"].append((p, (bh >> 1) & 3, bh >> 3))
                p += 3 + (1 if (bh >> 1) & 3 == seqgen.BT_RLE else bh >> 3)
                if bh & 1:
                    break
            pos = p + (4 if fhd & 4 else 0)
    except IndexError:
        pass
    return frames


def raw_rle_over_window(buf):
    return any(t in (seqgen.BT_RAW, seqgen.BT_RLE) and size > min(f["window"], 1 << 17)
               for f in layout(buf) if f["window"] for _, t, size in f["blocks"])


def with_window_log(frame, log):
    """a frame with a window descriptor, that descriptor set to 2^log"""
    [f] = layout(frame)
    assert f["window"] is not None
    b = bytearray(frame)
    b[5] = (log - 10) << 3
    return bytes(b)


def with_content_size(frame, delta):
    """the frame with its Frame_Content_Size field changed by delta (the field keeps its width)"""
    [f] = layout(frame)
    p, n = f["fcs"]
    v = int.from_bytes(frame[p:p + n], "little") + delta            # the 2-byte form stores size - 256: the same delta
    assert n and 0 <= v < 1 << (8 * n), (n, v)
    return frame[:p] + v.to_bytes(n, "little") + frame[p + n:]


def verdict_class(ref, results, buf, d, refused_by):
    """the verdict of one input: "both-refuse", "both-accept" or the DIFFERENCES key.  results: [(path, result)] of one
    group of paths that must agree; refused_by: the harness's zbh_refusedBy."""
    assert len({isinstance(r, tuple) for _, r in results}) == 1, ("the paths disagree", [(p, r if isinstance(r, tuple) else len(r)) for p, r in results])
    if isinstance(ref, tuple):
        for p, r in results:
            assert isinstance(r, tuple), (p, "accepted what the reference refuses", ref)
            assert r[1] != GENERIC, (p, "GENERIC", ref)
        return "both-refuse"
    got = results[0][1]
    if not isinstance(got, tuple):
        for p, r in results:
            assert r == ref, (p, "bytes differ")
        return "both-accept"
    code = got[1]
    if code == 16:
        return "offset-beyond-27-bits"
    if code == 20 and (raw_rle_over_window(buf) or refused_by == 2):
        assert stream(_bind_stream(_ref()), buf, d)[0] == "ERR", "the reference's streaming call takes it too"
        return "block-over-window"
    if code == 20 and refused_by == 1:
        return "huffman-start-overread"
    raise AssertionError(("refused what the reference accepts, and not a documented difference", results))


# ---------------------------------------------------------------------------------------------------- constructed cases
# Each builder returns [(name, buffer, dstCapacity, dictionary or None)] and asserts the shape it was built for.
W_LOGS = (10, 12, 16)


def _seq_frame(blocks, seed, d=None, params=(), alphabet=256):
    src = seqgen.execute(blocks, np.random.default_rng(seed), seqgen.dict_content(d) if d else b"", alphabet)
    return seqgen.ref_compress_sequences(blocks, src, 3, d, params), src


def window_cases(log):
    """frames without a content size (so with a window descriptor; the encoder asked for 2^17 and fits the window to the
    input) of one compressed block whose compressed size stays below 2^log while it regenerates more: only literals; a
    few literals and a long match; and exactly 2^log bytes, which must be accepted.  Their window descriptors are then
    set to 2^log."""
    w = 1 << log
    over = 4 * w if log < 16 else w + 4096
    kinds = {"lits-over": [([], over)], "matches-over": [([(64, 40, over - 64)], 0)], "at-window": [([(64, 40, w - 100)], 36)]}
    out = []
    for kind, blocks in kinds.items():
        frame, src = _seq_frame(blocks, 100 + log, params=[(seqgen.C_WINDOWLOG, 17), (seqgen.C_CONTENTSIZE, 0)], alphabet=2)
        [f] = seqgen.frame_layout(frame)
        assert f["window_log"] >= log and f["content_size"] is None and len(f["blocks"]) == 1, f
        (bt, bsize, lt, nb, _), = f["blocks"]
        assert bt == seqgen.BT_COMPRESSED and bsize < w, f
        lit = seqgen.block_layout(frame[-bsize:])["lit_size"]
        assert len(src) == (w if kind == "at-window" else over), (kind, len(src))
        assert (lit > w) == (kind == "lits-over") and (nb == 0) == (kind == "lits-over"), (kind, lit, nb)
        out.append((f"window-2^{log}-{kind}", with_window_log(frame, log), len(src), None))
    return out


def raw_rle_cases():
    """a raw block and an RLE block of 4 KiB in frames whose window descriptors say 1 KiB (written here: no encoder
    writes them)"""
    out = []
    for kind, body, bt in (("raw", zref.random_bytes(4096, 41), seqgen.BT_RAW), ("rle", b"\x07", seqgen.BT_RLE)):
        frame = (0xFD2FB528).to_bytes(4, "little") + bytes([0, 0]) + (1 | bt << 1 | 4096 << 3).to_bytes(3, "little") + body
        [f] = seqgen.frame_layout(frame)
        assert f["window_log"] == 10 and f["blocks"][0][:2] == (bt, 4096) and f["content_size"] is None, f
        out.append((f"{kind}-block-over-window", frame, 4096, None))
    return out


def front_of_frame_cases():
    """offsets that reach in front of the frame: frame(A) + frame(B), where B was written with the raw-content dictionary
    A and its first match begins 3000 bytes into A's tail, decoded without a dictionary (the bytes in front of B's frame
    are A's output, which equals the dictionary: only a check against the frame's start refuses it); B with a dictionary
    shorter than A; and first sequences whose offsets are starting repeat offsets beyond the position (8 behind
    two literals, 4 behind none)."""
    a = zref.synthetic(20_000, 42, 0.5)
    fa = zref.ref_compress(a, 3)
    fb, sb = _seq_frame([([(10, 3010, 200), (5, 40, 60)], 30)], 43, d=a)
    assert seqgen.ref_decompress(fb, len(sb), a) == sb
    out = [("prefix-frame-a-then-b-without-dict", fa + fb, len(a) + len(sb), None),
           ("prefix-b-with-shorter-dict", fb, len(sb), a[-2000:])]
    for name, seqs in (("repcode-8-at-2", [(2, 8, 20)]), ("repcode-4-at-0", [(0, 4, 20)])):
        f, s = _seq_frame([(seqs, 4)], 44, d=a)
        assert seqgen.frame_layout(f)[0]["blocks"][0][3] == 1
        out.append((f"first-{name}", f, len(s), None))
    return out


def content_size_cases():
    """Frame_Content_Size one below and one above the content, in the first, a middle and the last frame of a buffer of
    three, and in a frame of four blocks whose window is stated apart from the content size"""
    srcs = [zref.synthetic(n, 50 + n % 7, 0.6) for n in (70_000, 1000, 150)]
    frames = [zref.ref_compress(s, 3) for s in srcs]
    total = sum(map(len, srcs))
    out = []
    for k in range(3):
        for delta in (-1, 1):
            fs = list(frames)
            fs[k] = with_content_size(fs[k], delta)
            out.append((f"content-size{delta:+d}-frame-{k}", b"".join(fs), total + 64, None))
    big = zref.synthetic(450_000, 57, 0.6)
    fr = seqgen.ref_compress2(big, [(seqgen.C_WINDOWLOG, 17), (seqgen.C_LEVEL, 1)])
    [f] = seqgen.frame_layout(fr)
    assert not f["single_segment"] and f["content_size"] == len(big) and len(f["blocks"]) == 4, f
    for delta in (-1, 1):
        out.append((f"content-size{delta:+d}-multi-block", with_content_size(fr, delta), len(big) + 64, None))
    return out


def failing_frame_cases():
    """frame 1 of three fails in D4 (its block 2 has a match that begins 3000 bytes into a dictionary the call does not
    have) while frames 0 and 2 hold many matches of their own; and the same buffer with frame 1 last"""
    d = zref.synthetic(20_000, 60, 0.5)
    blocks = [([(20, 17, 40)] * 200, 10), ([(3, 100, 30)] * 300, 0)]
    pos = sum(ll + ml for seqs, t in blocks for ll, _, ml in seqs) + sum(t for _, t in blocks)
    blocks.append(([(10, pos + 10 + 3000, 50)], 5))
    bad, sbad = _seq_frame(blocks, 61, d=d)
    [f] = seqgen.frame_layout(bad)
    assert len(f["blocks"]) == 3 and all(b[0] == seqgen.BT_COMPRESSED and b[3] for b in f["blocks"]), f
    s0, s2 = zref.synthetic(1 << 20, 62, 0.7), zref.synthetic(300_000, 63, 0.9)
    f0, f2 = zref.ref_compress(s0, 1), zref.oracle_compress(s2, 1)
    n = len(s0) + len(sbad) + len(s2)
    return [("failing-frame-middle", f0 + bad + f2, n, None), ("failing-frame-last", f0 + f2 + bad, n, None)]


def capacity_cases():
    """dstCapacity one byte short of three frames' content: with content sizes, and streamed frames without"""
    srcs = [zref.synthetic(n, 70 + n % 5, 0.6) for n in (5000, 200_000, 70_000)]
    with_size = b"".join(zref.ref_compress(s, 3) for s in srcs)
    streamed = b"".join(seqgen.ref_compress2(s, [(seqgen.C_LEVEL, 3)], stream=True) for s in srcs)
    n = sum(map(len, srcs))
    return [("capacity-1-short", with_size, n - 1, None), ("capacity-1-short-streamed", streamed, n - 1, None)]


def constructed():
    out = []
    for log in W_LOGS:
        out += window_cases(log)
    return out + raw_rle_cases() + front_of_frame_cases() + content_size_cases() + failing_frame_cases() + capacity_cases()


# ---------------------------------------------------------------------------------------------------- the seeded corpus
def _bases():
    """(valid buffer, its content, dictionary or None): single-segment frames of both encoders, streamed frames with
    window descriptors and repeat-mode tables, concatenated frames, frames of the golden zstd-format dictionary"""
    zd = zref.golden_input(seqgen.ZDICT)
    srcs = [zref.synthetic(n, s, p) for n, s, p in ((300, 1, 0.5), (5000, 2, 0.7), (70_000, 3, 0.5), (200_000, 4, 0.9))] + [b"abc" * 20_000]
    out = []
    for s in srcs:
        out += [(zref.ref_compress(s, level), s, None) for level in (1, 3, 19)] + [(zref.oracle_compress(s, 1), s, None)]
    for s in srcs[1:4]:
        out += [(zref.ref_compress_using_dict(s, zd, 3), s, zd), (zref.oracle_compress_using_dict(s, zd, 1), s, zd)]
    for name in ("window-1k-streamed", "streamed-checksums"):
        f, s = seqgen.ADVANCED[name]()
        out.append((f, s, None))
    s = zref.synthetic(400_000, 5, 0.7)
    out.append((seqgen.ref_compress2(s, [(seqgen.C_WINDOWLOG, 17), (seqgen.C_LEVEL, 5)], stream=True), s, None))
    out.append((seqgen.ref_compress2(s, [(seqgen.C_WINDOWLOG, 12), (seqgen.C_LEVEL, 3)], stream=True), s, None))
    skip = bytes([0x53, 0x2A, 0x4D, 0x18, 5, 0, 0, 0]) + b"xxxxx"
    a, b, c = srcs[1], srcs[2], srcs[0]
    out.append((zref.ref_compress(a, 3) + zref.oracle_compress(b, 1) + skip + zref.ref_compress(c, 19), a + b + c, None))
    out.append((seqgen.ref_compress2(a, [(seqgen.C_WINDOWLOG, 12)], stream=True) + zref.ref_compress(c, 1)
                + seqgen.ref_compress2(b, [(seqgen.C_CHECKSUM, 1)], stream=True), a + c + b, None))
    out.append((zref.ref_compress_using_dict(a, zd, 3) + zref.oracle_compress_using_dict(b, zd, 1), a + b, zd))
    return out


def _targets(buf):
    """where a mutation is aimed half of the time: frame headers (window descriptors, content-size fields), block headers
    with the literals header behind them, and the sequences section header that holds the table modes"""
    t = []
    for f in layout(buf):
        t.append((f["start"], f["header"]))
        for p, bt, size in f["blocks"]:
            t.append((p, 8))
            if bt == seqgen.BT_COMPRESSED and size > 2:
                try:
                    L = seqgen.block_layout(buf[p + 3:p + 3 + size])
                    hs = L["lit_header"]
                    body = (L["lit_size"], 1)[L["lit_type"]] if L["lit_type"] < 2 else \
                        (int.from_bytes(buf[p + 3:p + 3 + hs], "little") >> 4) >> (10, 10, 14, 18)[(buf[p + 3] >> 2) & 3]
                    t.append((p + 3 + hs + body, 4))
                except IndexError:
                    pass
    return t


def corpus(n, seed):
    """n mutated inputs: (name, buffer, dstCapacity, dictionary or None)"""
    rng = random.Random(seed)
    bases = _bases()
    targets = [_targets(b) for b, _, _ in bases]
    out = []
    for i in range(n):
        k = rng.randrange(len(bases))
        buf, src, d = bases[k]
        kind = rng.choice(("flip", "flip", "overwrite", "truncate"))
        b = bytearray(buf)
        if kind == "truncate":
            b = b[:rng.randrange(1, len(b))]
        else:
            for _ in range(rng.choice((1, 1, 2, 3))):
                if rng.random() < 0.5:
                    p0, span = rng.choice(targets[k])
                    p = min(p0 + rng.randrange(max(span, 1)), len(b) - 1)
                else:
                    p = rng.randrange(len(b))
                if kind == "flip":
                    b[p] ^= 1 << rng.randrange(8)
                else:
                    b[p] = rng.randrange(256)
        out.append((f"corpus-{i}-{kind}-base{k}", bytes(b), len(src) + 64, d))
    return out


VALID = zref.synthetic(50_000, 80, 0.6)


# ---------------------------------------------------------------------------------------------------- CPU half
def _sanitized(cases, build_dir):
    """the harness as a program under AddressSanitizer and UndefinedBehaviorSanitizer over all cases: [(return value,
    output checksum, guard kept)]"""
    exe = os.path.join(build_dir, "zb_hostdecode_sanitized")
    subprocess.check_call(["g++", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-DZBH_CORPUS_MAIN",
                           "-Wall", "-Wextra", "-Werror", "-Wno-unused-function", "-x", "c++", "-o", exe, os.path.join(HERE, "host_decode.cpp")])
    rec = bytearray()
    for _, buf, cap, d in cases:
        d = d or b""
        rec += cap.to_bytes(8, "little") + len(d).to_bytes(8, "little") + d + len(buf).to_bytes(8, "little") + buf
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0", UBSAN_OPTIONS="print_stacktrace=1")
    p = subprocess.run([exe], input=bytes(rec), stdout=subprocess.PIPE, stderr=subprocess.PIPE, env=env)
    assert p.returncode == 0, p.stderr.decode()[-4000:]
    assert not p.stderr, p.stderr.decode()[-4000:]
    return [tuple(int(x) for x in line.split()) for line in p.stdout.decode().splitlines()]


def _checksum(b):
    a = np.frombuffer(b, dtype=np.uint8).astype(np.uint64)
    return int((a * np.arange(1, len(a) + 1, dtype=np.uint64)).sum(dtype=np.uint64)) if len(a) else 0


@needs_ref
@pytest.mark.parametrize("log", W_LOGS)
def test_window_bound(H, log):
    """a compressed block that regenerates more than its frame's window is refused with corruption_detected (20),
    whether literals alone or matches carry it over; a block of exactly the window is accepted"""
    for name, buf, cap, _ in window_cases(log):
        ref, (ours, _) = ref_oneshot(buf, cap), harness(H, buf, cap)
        if name.endswith("at-window"):
            assert not isinstance(ref, tuple) and ours == ref, name
        else:
            assert isinstance(ref, tuple) and ours == ("ERR", 20), (name, ref, ours if isinstance(ours, tuple) else len(ours))


@needs_ref
def test_raw_rle_block_over_window(H):
    """the documented difference: the reference's one-shot call takes a raw or RLE block larger than the window, its
    streaming call does not, and this decoder does not either"""
    for name, buf, cap, _ in raw_rle_cases():
        assert not isinstance(ref_oneshot(buf, cap), tuple), name
        assert isinstance(stream(_bind_stream(_ref()), buf), tuple), name
        assert harness(H, buf, cap)[0] == ("ERR", 20), name


@needs_ref
def test_invalid_inputs_harness(H, build_dir):
    """every constructed case and CORPUS_CPU corpus cases through the harness, judged against the reference; then the
    same inputs once through the harness built with sanitizers, which must report nothing and agree"""
    cases = constructed() + corpus(CORPUS_CPU, 1)
    classes, diffs, seen = collections.Counter(), collections.Counter(), []
    for i, (name, buf, cap, d) in enumerate(cases):
        ref = ref_oneshot(buf, cap, d, checksums=False)
        ours, by = harness(H, buf, cap, d)
        c = verdict_class(ref, [("harness", ours)], buf, d, by)
        classes[(name.split("-")[0] == "corpus", c)] += 1
        if c in DIFFERENCES:
            diffs[(c, name if not name.startswith("corpus") else "corpus")] += 1
        seen.append(ours)
        if not name.startswith("corpus") or i % 50 == 0:
            assert harness(H, zref.ref_compress(VALID, 3), len(VALID))[0] == VALID
    print("\nverdicts (corpus?, class):", dict(classes), "\nreference accepts, decoder refuses:", dict(diffs))
    assert classes[(True, "both-accept")] > 100 and classes[(True, "both-refuse")] > 1000
    san = _sanitized(cases, build_dir)
    assert len(san) == len(cases)
    for (name, _, cap, _), ours, (r, h, guard) in zip(cases, seen, san):
        assert guard == 1, name
        if isinstance(ours, tuple):
            assert r == (1 << 64) - ours[1], name
        else:
            assert (r, h) == (len(ours), _checksum(ours)), name


# ---------------------------------------------------------------------------------------------------- GPU half
def _lib():
    import zstd_b200
    L = _bind_stream(zstd_b200.lib())
    L.ZSTD_decompress_usingDict.restype = _sz
    L.ZSTD_decompress_usingDict.argtypes = [_vp, _vp, _sz, _vp, _sz, _vp, _sz]
    L.ZSTDB200_decompressDevice_usingDict.restype = _sz
    L.ZSTDB200_decompressDevice_usingDict.argtypes = [_vp, _vp, _sz, _vp, _sz, _vp, _sz, _vp]
    return L


@pytest.fixture(scope="module")
def dctx():
    import zstd_b200
    d = zstd_b200.ZSTD_DCtx()
    yield d
    d.close()


@pytest.fixture(scope="module")
def dctx_walk():
    """a context whose device calls walk the headers with the walk kernel"""
    import zstd_b200
    os.environ["ZSTDB200_HOSTWALK_MAX"] = "0"
    try:
        d = zstd_b200.ZSTD_DCtx()
    finally:
        del os.environ["ZSTDB200_HOSTWALK_MAX"]
    yield d
    d.close()


def gpu_host(L, dctx, buf, cap, d=None):
    out = ctypes.create_string_buffer(bytes([GUARD]) * (cap + 16), cap + 16)
    r = L.ZSTD_decompress_usingDict(dctx._h, out, cap, buf, len(buf), d, len(d) if d else 0)
    assert out.raw[cap:] == bytes([GUARD]) * 16, "bytes behind the destination changed"
    return ("ERR", L.ZSTD_getErrorCode(r)) if L.ZSTD_isError(r) else out.raw[:r]


def gpu_device(L, dctx, buf, cap, d=None, off=1):
    """the device call with source and destination `off` bytes into larger buffers; the bytes around the destination
    must keep their value whatever the verdict"""
    import torch
    d_in = torch.zeros(len(buf) + off + 8, dtype=torch.uint8, device="cuda")
    d_in[off:off + len(buf)] = torch.frombuffer(bytearray(buf), dtype=torch.uint8).cuda()
    d_out = torch.full((cap + off + 16,), GUARD, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    r = L.ZSTDB200_decompressDevice_usingDict(dctx._h, d_out.data_ptr() + off, cap, d_in.data_ptr() + off, len(buf), d, len(d) if d else 0, None)
    torch.cuda.synchronize()
    assert bool((d_out[:off] == GUARD).all()) and bool((d_out[off + cap:] == GUARD).all()), "bytes outside the destination changed"
    return ("ERR", L.ZSTD_getErrorCode(r)) if L.ZSTD_isError(r) else bytes(d_out[off:off + r].cpu().numpy())


@needs_ref
@pytest.mark.gpu
@pytest.mark.timeout(600, method="thread")
def test_invalid_inputs_gpu(H, dctx, dctx_walk):
    """every constructed case and CORPUS_GPU corpus cases on every path: the harness, the host call, the device call, the
    walk kernel (one group that must agree and is judged against the reference's one-shot call), and without a
    dictionary ZSTD_decompressStream in pieces, judged against the reference's"""
    L, R = _lib(), _bind_stream(_ref())
    valid = zref.ref_compress(VALID, 3)
    cases = constructed() + corpus(CORPUS_GPU, 1)                # the first cases of the corpus the sanitizer run saw
    classes = collections.Counter()
    for i, (name, buf, cap, d) in enumerate(cases):
        ref, ref_unchecked = ref_oneshot(buf, cap, d), ref_oneshot(buf, cap, d, checksums=False)
        ours, by = harness(H, buf, cap, d)
        host = ("host", gpu_host(L, dctx, buf, cap, d))
        paths = [("harness", ours), ("device", gpu_device(L, dctx, buf, cap, d)), ("walk-kernel", gpu_device(L, dctx_walk, buf, cap, d))]
        checksum_only = isinstance(ref, tuple) and not isinstance(ref_unchecked, tuple)
        if not checksum_only:
            paths.append(host)                                   # only content checksums (the host call's) may part them
        c = verdict_class(ref_unchecked, paths, buf, d, by)
        if checksum_only:                                        # checksum_wrong, unless the content is refused already
            h = host[1]
            assert ref[1] == 22 and (h == ("ERR", 22) if c == "both-accept" else isinstance(h, tuple) and h[1] != GENERIC), (name, c, h if isinstance(h, tuple) else len(h))
        classes[c] += 1
        if d is None:
            classes["stream-" + verdict_class(stream(R, buf), [("stream", stream(L, buf))], buf, d, by)] += 1
        if not name.startswith("corpus") or i % 50 == 0:
            assert gpu_host(L, dctx, valid, len(VALID)) == VALID, name
            assert gpu_device(L, dctx, valid, len(VALID)) == VALID, name
            assert gpu_device(L, dctx_walk, valid, len(VALID)) == VALID, name
    print("\nverdicts:", dict(classes))
