"""The host size readers ZSTD_findDecompressedSize, ZSTD_decompressBound and ZSTD_findFrameCompressedSize against the compiled
reference's, input by input: the golden frames, the reference encoder's advanced shapes (no content size, streamed,
checksums, 1 KiB blocks), skippable frames, every truncation of small multi-frame inputs, garbage tails, a reserved block
type, window descriptors of 2^28 .. 2^31 and the empty input.  No GPU needed."""
import ctypes
import glob
import os
import struct

import pytest

import seqgen
import zref
import zstd_b200
from test_decode_invalid import needs_ref

_sz, _vp = ctypes.c_size_t, ctypes.c_void_p
SKIP_MAGIC = 0x184D2A50
MAGIC = 0xFD2FB528
ERROR, UNKNOWN = 2**64 - 2, 2**64 - 1
ADVANCED = ("no-content-size", "streamed", "streamed-checksums", "max-block-1k", "window-1k-streamed", "target-cblock-1340")

_refl = None


def _ref():
    global _refl
    if _refl is None:
        R = zref.ref()
        for name in ("ZSTD_findDecompressedSize", "ZSTD_decompressBound"):
            getattr(R, name).restype = ctypes.c_ulonglong
            getattr(R, name).argtypes = [_vp, _sz]
        R.ZSTD_findFrameCompressedSize.restype = _sz
        R.ZSTD_findFrameCompressedSize.argtypes = [_vp, _sz]
        R.ZSTD_getErrorCode.restype = ctypes.c_int
        R.ZSTD_getErrorCode.argtypes = [_sz]
        _refl = R
    return _refl


def _fcs(L, b):
    r = L.ZSTD_findFrameCompressedSize(b, len(b))
    return ("ERR",) if L.ZSTD_isError(r) else r


def readings(L, b):
    """(findDecompressedSize, decompressBound, findFrameCompressedSize) of b as library L gives them; for
    findFrameCompressedSize an error counts as one outcome whatever its code (the codes of a cut-short header differ from
    the reference's in order only, and that function's behaviour is kept as it was)"""
    return L.ZSTD_findDecompressedSize(b, len(b)), L.ZSTD_decompressBound(b, len(b)), _fcs(L, b)


def same(b):
    assert readings(zstd_b200.lib(), b) == readings(_ref(), b), (len(b), b[:16].hex())


def skippable(n, magic=SKIP_MAGIC):
    return struct.pack("<II", magic, n) + bytes(range(256)) * (n // 256) + bytes(n % 256)


def header(window_byte, fcs=None, checksum=False):
    """a frame header with a window descriptor (no Single_Segment), without dictionary ID, content size fcs (8 bytes) or none"""
    fhd = (3 << 6 if fcs is not None else 0) | (4 if checksum else 0)
    return struct.pack("<IBB", MAGIC, fhd, window_byte) + (struct.pack("<Q", fcs) if fcs is not None else b"")


def block(btype, size, last, body=None):
    h = (size << 3) | (btype << 1) | int(last)
    return struct.pack("<I", h)[:3] + (body if body is not None else bytes(1 if btype == 1 else size))


def test_symbols_are_exported():
    L = zstd_b200.lib()
    for name in ("ZSTD_findDecompressedSize", "ZSTD_decompressBound", "ZSTDB200_findDecompressedSizesAsync",
                 "ZSTDB200_decompressFramesAsync_deviceOffsets"):
        assert hasattr(L, name), name


def test_python_bindings():
    f = zstd_b200.lib()
    src = zref.synthetic(5000, seed=1)
    assert zstd_b200.ZSTD_findDecompressedSize(b"") == 0 and zstd_b200.ZSTD_decompressBound(b"") == 0
    frame = header(0, None) + block(0, 100, True)
    assert zstd_b200.ZSTD_findDecompressedSize(frame) == UNKNOWN
    assert zstd_b200.ZSTD_decompressBound(frame) == 1024
    assert zstd_b200.ZSTD_findDecompressedSize(frame + b"x") == UNKNOWN          # the first frame without a size decides
    stated = header(0, 100) + block(0, 100, True)
    assert zstd_b200.ZSTD_findDecompressedSize(stated) == 100 and zstd_b200.ZSTD_findDecompressedSize(stated + b"x") == ERROR
    assert zstd_b200.ZSTD_decompressBound(frame + b"x") == ERROR
    assert f.ZSTD_findFrameCompressedSize(frame, len(frame)) == len(frame)
    assert zstd_b200.ZSTD_findDecompressedSize(skippable(len(src))) == 0


@needs_ref
def test_golden_frames():
    names = sorted(glob.glob(os.path.join(zref.GOLDEN, "decompression*", "*.zst")))
    assert len(names) >= 7
    for n in names:
        b = open(n, "rb").read()
        same(b)
        same(b + b)
        same(skippable(3) + b + skippable(0))


@needs_ref
def test_reference_encoder_shapes():
    for name in ADVANCED:
        f, src = seqgen.ADVANCED[name]()
        same(f)
        same(f + f)
        same(skippable(100) + f)
        if name in ("no-content-size", "streamed"):
            assert zstd_b200.ZSTD_findDecompressedSize(f) == UNKNOWN
            assert zstd_b200.ZSTD_decompressBound(f) >= len(src)
        for cut in (1, 3, 4, 5):
            same(f[:-cut])


@needs_ref
def test_every_truncation_of_small_multi_frame_inputs():
    a, b = zref.synthetic(300, seed=2), zref.synthetic(200_000, seed=3, match_prob=0.6)
    inputs = [zref.ref_compress(a, 3) + skippable(5) + zref.ref_compress(b"", 1),
              zref.oracle_compress(a, 1) + header(0x08, None) + block(0, 7, False) + block(1, 9, True) + zref.ref_compress(a, 19),
              header(0, None, checksum=True) + block(0, 10, True) + b"\1\2\3\4" + zref.ref_compress(b, 1)[:80]]
    for x in inputs:
        for n in range(len(x) + 1):
            same(x[:n])


@needs_ref
def test_garbage_tails_and_reserved_block_type():
    f = zref.ref_compress(zref.synthetic(10_000, seed=4), 3)
    for tail in (b"\0", b"\x28\xb5\x2f", b"\x28\xb5\x2f\xfd", b"\x28\xb5\x2f\xfd\x00", b"\x50\x2a\x4d\x18\1\0\0", b"garbage!",
                 struct.pack("<II", SKIP_MAGIC + 15, 2**32 - 1)):
        same(f + tail)
        same(tail)
    reserved = header(0x10, 5) + block(3, 5, True)
    same(reserved)
    same(f + reserved)
    same(header(0x10, None) + block(0, 5, False) + block(3, 5, True))
    same(skippable(0, SKIP_MAGIC + 7) + header(0x10, None) + block(2, 0, True, b""))
    big = header(0x00, 2**64 - 2) + block(1, 1, True)          # a content size equal to ZSTD_CONTENTSIZE_ERROR
    same(big)
    same(header(0x00, 2**63) + block(1, 1, True) + header(0x00, 2**63) + block(1, 1, True))     # the sum wraps


@needs_ref
def test_large_window_descriptors():
    for wl in range(27, 32):
        for mantissa in (0, 7):
            wd = ((wl - 10) << 3) | mantissa
            for fcs in (None, 12):
                same(header(wd, fcs) + block(0, 12, True))
                same(header(wd, fcs) + block(0, 12, False) + block(1, 200, False) + block(0, 0, True))
    same(header(32 - 10 << 3, None) + block(0, 12, True))            # windowLog 32: frameParameter_windowTooLarge


@needs_ref
def test_empty_and_tiny_inputs():
    for b in (b"", b"\x28", b"\x28\xb5\x2f\xfd", b"\x50\x2a\x4d\x18", b"\x50\x2a\x4d\x18\0\0\0\0", bytes(5)):
        same(b)
