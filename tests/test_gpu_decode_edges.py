"""GPU decompression (pytest -m gpu) of frames built to reach the stages that exist only on the GPU: the scan's offsets
and repcode histories (D3), literal placement, repcode resolution and matches that begin in the dictionary (D4), the
match copies with their dependency waits (D5), and the host driver's handling of frames without a content size.  The
frames come from tests/seqgen.py: chosen sequences written by the reference's ZSTD_compressSequences, and the
reference encoder's advanced parameters.  Every case is decoded by the host call, by the device call with source and
destination at byte offsets 1, 2 and 3 inside larger buffers (the last on a stream of the caller's), and by the
device call through the walk kernel; the plain LZ77 execution of the sequences (or the input the reference compressed)
is the answer."""
import ctypes
import os

import pytest

import seqgen
import zref
import zstd_b200

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600, method="thread")]      # a stuck kernel must fail the run, not hang it
needs_ref = pytest.mark.skipif(not zref.have_ref(), reason="reference library not built")
_sz, _vp = ctypes.c_size_t, ctypes.c_void_p
GUARD = 0xA5


def L():
    lib = zstd_b200.lib()
    lib.ZSTD_decompress_usingDict.restype = _sz
    lib.ZSTD_decompress_usingDict.argtypes = [_vp, _vp, _sz, _vp, _sz, _vp, _sz]
    lib.ZSTDB200_decompressDevice_usingDict.restype = _sz
    lib.ZSTDB200_decompressDevice_usingDict.argtypes = [_vp, _vp, _sz, _vp, _sz, _vp, _sz, _vp]
    lib.ZSTD_createDStream.restype = _vp
    lib.ZSTD_freeDStream.argtypes = [_vp]
    lib.ZSTD_initDStream.restype = _sz
    lib.ZSTD_initDStream.argtypes = [_vp]
    lib.ZSTD_decompressStream.restype = _sz
    lib.ZSTD_decompressStream.argtypes = [_vp, ctypes.POINTER(seqgen.OutBuffer), ctypes.POINTER(seqgen.InBuffer)]
    return lib


def _result(lib, r, out):
    return ("ERR", lib.ZSTD_getErrorCode(r)) if lib.ZSTD_isError(r) else out(r)


@pytest.fixture(scope="module")
def dctx():
    d = zstd_b200.ZSTD_DCtx()
    yield d
    d.close()


@pytest.fixture(scope="module")
def dctx_walk():
    """a context whose device calls walk the headers with the walk kernel (inputs beyond 512 MiB take it)"""
    os.environ["ZSTDB200_HOSTWALK_MAX"] = "0"
    try:
        d = zstd_b200.ZSTD_DCtx()
    finally:
        del os.environ["ZSTDB200_HOSTWALK_MAX"]
    yield d
    d.close()


def host(dctx, frames, n, d=None):
    """ZSTD_decompressDCtx / ZSTD_decompress_usingDict into a buffer of exactly n bytes"""
    lib = L()
    out = ctypes.create_string_buffer(max(n, 1))
    r = lib.ZSTD_decompress_usingDict(dctx._h, out, n, frames, len(frames), d, len(d) if d else 0)
    return _result(lib, r, lambda r: out.raw[:r])


def device(dctx, frames, n, off, d=None, caller_stream=False):
    """ZSTDB200_decompressDevice_usingDict with source and destination `off` bytes into larger buffers, on a stream of
    the caller's or (NULL) the context's own; the bytes around the destination must stay as they were"""
    import torch
    lib = L()
    s = torch.cuda.Stream() if caller_stream else torch.cuda.current_stream()
    with torch.cuda.stream(s):
        d_in = torch.zeros(len(frames) + off + 8, dtype=torch.uint8, device="cuda")
        d_in[off:off + len(frames)] = torch.frombuffer(bytearray(frames), dtype=torch.uint8).cuda()
        d_out = torch.full((n + off + 8,), GUARD, dtype=torch.uint8, device="cuda")
        if not caller_stream:
            torch.cuda.synchronize()                   # the context's stream is a non-blocking one: not ordered after torch's
        r = lib.ZSTDB200_decompressDevice_usingDict(dctx._h, d_out.data_ptr() + off, n, d_in.data_ptr() + off, len(frames), d, len(d) if d else 0,
                                                    s.cuda_stream if caller_stream else None)
        torch.cuda.synchronize()
        got = _result(lib, r, lambda r: bytes(d_out[off:off + r].cpu().numpy()))
        if not isinstance(got, tuple):
            assert bool((d_out[:off] == GUARD).all()) and bool((d_out[off + n:] == GUARD).all()), "bytes outside the destination changed"
    return got


def stream(frames, piece=1 << 20, room=1 << 20):
    """ZSTD_decompressStream: input in `piece`-byte pieces, output through a `room`-byte buffer"""
    lib = L()
    zds = lib.ZSTD_createDStream()
    assert not lib.ZSTD_isError(lib.ZSTD_initDStream(zds))
    src = ctypes.create_string_buffer(frames, max(len(frames), 1))
    base = ctypes.cast(src, ctypes.c_void_p).value
    buf = ctypes.create_string_buffer(room)
    out, pos, last = bytearray(), 0, None
    try:
        while pos < len(frames):
            i = seqgen.InBuffer(base + pos, min(piece, len(frames) - pos), 0)
            while True:
                o = seqgen.OutBuffer(ctypes.cast(buf, ctypes.c_void_p), room, 0)
                last = lib.ZSTD_decompressStream(zds, ctypes.byref(o), ctypes.byref(i))
                if lib.ZSTD_isError(last):
                    return ("ERR", lib.ZSTD_getErrorCode(last))
                out += buf.raw[:o.pos]
                if i.pos == i.size and o.pos < room:
                    break
            pos += i.size
    finally:
        lib.ZSTD_freeDStream(zds)
    assert last == 0
    return bytes(out)


def every_way(dctx, dctx_walk, frames, want, n, d=None):
    assert host(dctx, frames, n, d) == want
    for off in (1, 2, 3):
        assert device(dctx, frames, n, off, d, caller_stream=off == 3) == want, off
    assert device(dctx_walk, frames, n, 1, d) == want


@needs_ref
@pytest.mark.parametrize("name", sorted(seqgen.DICTATED))
def test_dictated_sequences(dctx, dctx_walk, name):
    """every copy offset, length and alignment of D5; every repcode form and histories over 85 blocks; chains of
    matches that wait for one another within and across blocks and through one tile; blocks of one match, of only
    literals, of 127 ... 0x7F00 sequences; a 1 KiB window; several frames in one call; matches that begin in the
    dictionary's content"""
    frames, src, d = seqgen.DICTATED[name]()
    assert seqgen.ref_decompress(frames, len(src), d) == src
    every_way(dctx, dctx_walk, frames, src, len(src), d)


@needs_ref
@pytest.mark.parametrize("name", sorted(seqgen.ADVANCED))
def test_advanced_parameter_frames(dctx, dctx_walk, name):
    frames, src = seqgen.ADVANCED[name]()
    assert seqgen.ref_decompress(frames, len(src)) == src
    every_way(dctx, dctx_walk, frames, src, len(src))
    if any(f["content_size"] is None for f in seqgen.frame_layout(frames)):
        assert stream(frames) == src


@needs_ref
def test_checksums_of_frames_without_size(dctx):
    """the host call verifies the checksum of frames whose size only the scan knows; one flipped byte of the middle
    frame's checksum is checksum_wrong (22)"""
    frames, src = seqgen.ADVANCED["streamed-checksums"]()
    fs = seqgen.frame_layout(frames)
    assert [f["checksum"] and f["content_size"] is None for f in fs] == [True] * 3
    bad = bytearray(frames)
    bad[fs[0]["size"] + fs[1]["size"] - 2] ^= 0x10
    with pytest.raises(ValueError, match="checksum"):
        seqgen.ref_decompress(bytes(bad), len(src))
    assert host(dctx, bytes(bad), len(src)) == ("ERR", 22)
    assert stream(bytes(bad)) == ("ERR", 22)


@needs_ref
@pytest.mark.parametrize("name", sorted(seqgen.REFUSED))
def test_offsets_beyond_28_bits_refused(dctx, dctx_walk, name):
    """frameParameter_windowTooLarge (16) for a 2^28 window descriptor and for a Single_Segment frame whose offsets
    need 29 bits, on every path, where the reference decoder takes both"""
    frames, src = seqgen.REFUSED[name]()
    assert seqgen.ref_decompress(frames, len(src)) == src
    every_way(dctx, dctx_walk, frames, ("ERR", 16), len(src))
