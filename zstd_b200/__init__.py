"""zstd_b200 — Python host-side mirror of the libzstd C API served by libzstd_b200.so.

The product is the C-ABI shared library (include/zstd_b200.h); this module is the thin ctypes
binding a Python caller (tests, bench.py, torch.distributed sharding) uses.  Function names,
argument meaning and error behaviour follow the reference's simple API
(lib/zstd.h:155 ZSTD_compress, :274 ZSTD_compressCCtx, :944 ZSTD_compress_usingDict).

There is no CPU fallback: importing works anywhere, but every compress call raises ZstdError
when the CUDA library or a CUDA device is missing.
"""
from __future__ import annotations

import ctypes
import os
from typing import Optional, Sequence, Tuple

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("ZSTDB200_LIB") or os.path.join(_HERE, "libzstd_b200.so")   # override: development variants only

_lib = None
_sz = ctypes.c_size_t
_vp = ctypes.c_void_p


class ZstdError(RuntimeError):
    """Raised with the reference's error name (lib/common/error_private.c:14-62)."""

    def __init__(self, code: int, name: str):
        super().__init__(f"zstd_b200 error {code}: {name}")
        self.code = code
        self.name = name


class Stats(ctypes.Structure):
    _fields_ = [("kernel_ms", ctypes.c_float), ("match_ms", ctypes.c_float), ("cand_ms", ctypes.c_float), ("parse_ms", ctypes.c_float), ("literals_ms", ctypes.c_float),
                ("sequences_ms", ctypes.c_float), ("stitch_ms", ctypes.c_float), ("total_ms", ctypes.c_float),
                ("launches", ctypes.c_uint), ("nbBlocks", ctypes.c_uint),
                ("h2d_bytes", _sz), ("d2h_bytes", _sz)]


class DStats(ctypes.Structure):
    _fields_ = [("kernel_ms", ctypes.c_float), ("literals_ms", ctypes.c_float), ("sequences_ms", ctypes.c_float), ("place_ms", ctypes.c_float),
                ("execute_ms", ctypes.c_float), ("launches", ctypes.c_uint), ("nbBlocks", ctypes.c_uint), ("nbFrames", ctypes.c_uint), ("h2d_bytes", _sz), ("d2h_bytes", _sz)]


def lib() -> ctypes.CDLL:
    """Load libzstd_b200.so (built in-tree by __graft_entry__.build()).  Fails loudly if absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                          "(nvcc, sm_90a). zstd_b200 has no CPU fallback.")
    L = ctypes.CDLL(LIB_PATH, mode=ctypes.RTLD_LOCAL)
    L.ZSTD_compress.restype = _sz
    L.ZSTD_compress.argtypes = [_vp, _sz, _vp, _sz, ctypes.c_int]
    L.ZSTD_createCCtx.restype = _vp
    L.ZSTD_createCCtx.argtypes = []
    L.ZSTD_freeCCtx.restype = _sz
    L.ZSTD_freeCCtx.argtypes = [_vp]
    L.ZSTD_compressCCtx.restype = _sz
    L.ZSTD_compressCCtx.argtypes = [_vp, _vp, _sz, _vp, _sz, ctypes.c_int]
    L.ZSTD_compress_usingDict.restype = _sz
    L.ZSTD_compress_usingDict.argtypes = [_vp, _vp, _sz, _vp, _sz, _vp, _sz, ctypes.c_int]
    L.ZSTD_compressBound.restype = _sz
    L.ZSTD_compressBound.argtypes = [_sz]
    L.ZSTD_isError.restype = ctypes.c_uint
    L.ZSTD_isError.argtypes = [_sz]
    L.ZSTD_getErrorName.restype = ctypes.c_char_p
    L.ZSTD_getErrorName.argtypes = [_sz]
    L.ZSTD_getErrorCode.restype = ctypes.c_int
    L.ZSTD_getErrorCode.argtypes = [_sz]
    for f in ("ZSTD_minCLevel", "ZSTD_maxCLevel", "ZSTD_defaultCLevel"):
        getattr(L, f).restype = ctypes.c_int
        getattr(L, f).argtypes = []
    L.ZSTD_versionNumber.restype = ctypes.c_uint
    L.ZSTD_versionString.restype = ctypes.c_char_p
    L.ZSTDB200_compressDevice.restype = _sz
    L.ZSTDB200_compressDevice.argtypes = [_vp, _vp, _sz, _vp, _sz, ctypes.c_int, _vp]
    L.ZSTDB200_compressFrames.restype = _sz
    L.ZSTDB200_compressFrames.argtypes = [_vp, _vp, _sz, _vp, _vp, _vp, _sz, _vp, _sz, _vp, ctypes.c_int, ctypes.c_int, _vp]
    L.ZSTDB200_getLastStats.restype = None
    L.ZSTDB200_getLastStats.argtypes = [_vp, ctypes.POINTER(Stats)]
    L.ZSTDB200_setDevice.restype = ctypes.c_int
    L.ZSTDB200_setDevice.argtypes = [ctypes.c_int]
    L.ZSTDB200_deviceAvailable.restype = ctypes.c_int
    if os.environ.get("ZSTDB200_LIB") and not hasattr(L, "ZSTD_createCDict"):      # an older development build
        _lib = L
        return L
    L.ZSTD_createCDict.restype = _vp
    L.ZSTD_createCDict.argtypes = [_vp, _sz, ctypes.c_int]
    L.ZSTD_freeCDict.restype = _sz
    L.ZSTD_freeCDict.argtypes = [_vp]
    L.ZSTD_compress_usingCDict.restype = _sz
    L.ZSTD_compress_usingCDict.argtypes = [_vp, _vp, _sz, _vp, _sz, _vp]
    L.ZSTD_getDictID_fromCDict.restype = ctypes.c_uint
    L.ZSTD_getDictID_fromCDict.argtypes = [_vp]
    L.ZSTD_getDictID_fromDict.restype = ctypes.c_uint
    L.ZSTD_getDictID_fromDict.argtypes = [_vp, _sz]
    L.ZSTD_CCtx_setParameter.restype = _sz
    L.ZSTD_CCtx_setParameter.argtypes = [_vp, ctypes.c_int, ctypes.c_int]
    L.ZSTD_CCtx_reset.restype = _sz
    L.ZSTD_CCtx_reset.argtypes = [_vp, ctypes.c_int]
    L.ZSTD_CCtx_loadDictionary.restype = _sz
    L.ZSTD_CCtx_loadDictionary.argtypes = [_vp, _vp, _sz]
    L.ZSTD_CCtx_refCDict.restype = _sz
    L.ZSTD_CCtx_refCDict.argtypes = [_vp, _vp]
    if hasattr(L, "ZSTD_CCtx_refPrefix"):                                               # absent from older development builds
        L.ZSTD_CCtx_refPrefix.restype = _sz
        L.ZSTD_CCtx_refPrefix.argtypes = [_vp, _vp, _sz]
        L.ZSTDB200_CCtx_refPrefixDevice.restype = _sz
        L.ZSTDB200_CCtx_refPrefixDevice.argtypes = [_vp, _vp, _sz]
    L.ZSTD_compress2.restype = _sz
    L.ZSTD_compress2.argtypes = [_vp, _vp, _sz, _vp, _sz]
    L.ZSTD_compressStream2.restype = _sz
    L.ZSTD_compressStream2.argtypes = [_vp, _vp, _vp, ctypes.c_int]
    L.ZSTD_compressSequences.restype = _sz
    L.ZSTD_compressSequences.argtypes = [_vp, _vp, _sz, _vp, _sz, _vp, _sz]
    L.ZSTDB200_compressSequencesDevice.restype = _sz
    L.ZSTDB200_compressSequencesDevice.argtypes = [_vp, _vp, _sz, _vp, _sz, _vp, _sz, _vp]
    L.ZSTD_sequenceBound.restype = _sz
    L.ZSTD_sequenceBound.argtypes = [_sz]
    L.ZSTD_mergeBlockDelimiters.restype = _sz
    L.ZSTD_mergeBlockDelimiters.argtypes = [_vp, _sz]
    L.ZSTD_generateSequences.restype = _sz
    L.ZSTD_generateSequences.argtypes = [_vp, _vp, _sz, _vp, _sz]
    L.ZSTDB200_generateSequencesDevice.restype = _sz
    L.ZSTDB200_generateSequencesDevice.argtypes = [_vp, _vp, _sz, _vp, _sz, _vp]
    L.ZSTDB200_generateSequencesDeviceAsync.restype = _sz
    L.ZSTDB200_generateSequencesDeviceAsync.argtypes = [_vp, _vp, _sz, _vp, _sz, _vp, _vp]
    L.ZSTDB200_compressFrames_usingCDict.restype = _sz
    L.ZSTDB200_compressFrames_usingCDict.argtypes = [_vp, _vp, _sz, _vp, _vp, _vp, _sz, _vp, _vp, ctypes.c_int, _vp]
    L.ZSTDB200_compressDeviceAsync.restype = _sz
    L.ZSTDB200_compressDeviceAsync.argtypes = [_vp, _vp, _sz, _vp, _sz, ctypes.c_int, _vp, _vp]
    L.ZSTDB200_compressFramesAsync.restype = _sz
    L.ZSTDB200_compressFramesAsync.argtypes = [_vp, _vp, _sz, _vp, _vp, _vp, _sz, _vp, ctypes.c_int, _vp, _vp, _vp]
    if hasattr(L, "ZSTDB200_compressFrames_usingCDicts"):                              # absent from older development builds
        L.ZSTDB200_compressFrames_usingCDicts.restype = _sz
        L.ZSTDB200_compressFrames_usingCDicts.argtypes = [_vp, _vp, _sz, _vp, _vp, _vp, _sz, _vp, ctypes.c_int, _vp, ctypes.c_int, _vp]
        L.ZSTDB200_compressFramesAsync_usingCDicts.restype = _sz
        L.ZSTDB200_compressFramesAsync_usingCDicts.argtypes = [_vp, _vp, _sz, _vp, _vp, _vp, _sz, _vp, ctypes.c_int, _vp, _vp, _vp]
    if hasattr(L, "ZSTD_createDCtx"):
        L.ZSTD_createDCtx.restype = _vp
        L.ZSTD_createDCtx.argtypes = []
        L.ZSTD_freeDCtx.restype = _sz
        L.ZSTD_freeDCtx.argtypes = [_vp]
        L.ZSTD_decompressDCtx.restype = _sz
        L.ZSTD_decompressDCtx.argtypes = [_vp, _vp, _sz, _vp, _sz]
        L.ZSTD_decompress.restype = _sz
        L.ZSTD_decompress.argtypes = [_vp, _sz, _vp, _sz]
        L.ZSTD_getFrameContentSize.restype = ctypes.c_ulonglong
        L.ZSTD_getFrameContentSize.argtypes = [_vp, _sz]
        L.ZSTD_findFrameCompressedSize.restype = _sz
        L.ZSTD_findFrameCompressedSize.argtypes = [_vp, _sz]
        L.ZSTDB200_decompressDevice.restype = _sz
        L.ZSTDB200_decompressDevice.argtypes = [_vp, _vp, _sz, _vp, _sz, _vp]
        if hasattr(L, "ZSTDB200_decompressDeviceAsync"):                                # absent from older development builds
            L.ZSTDB200_decompressDeviceAsync.restype = _sz
            L.ZSTDB200_decompressDeviceAsync.argtypes = [_vp, _vp, _sz, _vp, _sz, _vp, _vp]
        if hasattr(L, "ZSTDB200_decompressFrames"):                                     # absent from older development builds
            L.ZSTDB200_decompressFrames.restype = _sz
            L.ZSTDB200_decompressFrames.argtypes = [_vp, _vp, _sz, _vp, _vp, _vp, _sz, _vp, _vp, _sz, _vp, _vp]
            L.ZSTDB200_decompressFramesAsync.restype = _sz
            L.ZSTDB200_decompressFramesAsync.argtypes = [_vp, _vp, _sz, _vp, _vp, _vp, _sz, _vp, _vp, _sz, _vp, _vp, _vp]
        if hasattr(L, "ZSTDB200_decompressFrames_usingDDicts"):                         # absent from older development builds
            L.ZSTDB200_decompressFrames_usingDDicts.restype = _sz
            L.ZSTDB200_decompressFrames_usingDDicts.argtypes = [_vp, _vp, _sz, _vp, _vp, _vp, _sz, _vp, _vp, _sz, _vp, _vp, _vp]
            L.ZSTDB200_decompressFramesAsync_usingDDicts.restype = _sz
            L.ZSTDB200_decompressFramesAsync_usingDDicts.argtypes = [_vp, _vp, _sz, _vp, _vp, _vp, _sz, _vp, _vp, _sz, _vp, _vp, _vp, _vp]
        if hasattr(L, "ZSTD_findDecompressedSize"):                                     # absent from older development builds
            L.ZSTD_findDecompressedSize.restype = ctypes.c_ulonglong
            L.ZSTD_findDecompressedSize.argtypes = [_vp, _sz]
            L.ZSTD_decompressBound.restype = ctypes.c_ulonglong
            L.ZSTD_decompressBound.argtypes = [_vp, _sz]
            L.ZSTDB200_findDecompressedSizesAsync.restype = _sz
            L.ZSTDB200_findDecompressedSizesAsync.argtypes = [_vp, _vp, _sz, _vp, _vp, _sz, _vp, _vp, _vp]
            L.ZSTDB200_decompressFramesAsync_deviceOffsets.restype = _sz
            L.ZSTDB200_decompressFramesAsync_deviceOffsets.argtypes = [_vp, _vp, _sz, _vp, _vp, _vp, _sz, _vp, _vp, _sz, _vp, _vp, _vp]
        L.ZSTDB200_getLastDStats.restype = None
        L.ZSTDB200_getLastDStats.argtypes = [_vp, ctypes.POINTER(DStats)]
    if hasattr(L, "ZSTD_createDDict"):                                                  # absent from older development builds
        L.ZSTD_createDDict.restype = _vp
        L.ZSTD_createDDict.argtypes = [_vp, _sz]
        L.ZSTD_freeDDict.restype = _sz
        L.ZSTD_freeDDict.argtypes = [_vp]
        L.ZSTD_decompress_usingDDict.restype = _sz
        L.ZSTD_decompress_usingDDict.argtypes = [_vp, _vp, _sz, _vp, _sz, _vp]
        L.ZSTD_getDictID_fromDDict.restype = ctypes.c_uint
        L.ZSTD_getDictID_fromDDict.argtypes = [_vp]
        L.ZSTD_getDictID_fromFrame.restype = ctypes.c_uint
        L.ZSTD_getDictID_fromFrame.argtypes = [_vp, _sz]
        L.ZSTD_DCtx_setParameter.restype = _sz
        L.ZSTD_DCtx_setParameter.argtypes = [_vp, ctypes.c_int, ctypes.c_int]
        L.ZSTD_DCtx_reset.restype = _sz
        L.ZSTD_DCtx_reset.argtypes = [_vp, ctypes.c_int]
        L.ZSTD_DCtx_loadDictionary.restype = _sz
        L.ZSTD_DCtx_loadDictionary.argtypes = [_vp, _vp, _sz]
        L.ZSTD_DCtx_refDDict.restype = _sz
        L.ZSTD_DCtx_refDDict.argtypes = [_vp, _vp]
        L.ZSTD_DCtx_refPrefix.restype = _sz
        L.ZSTD_DCtx_refPrefix.argtypes = [_vp, _vp, _sz]
    _lib = L
    return L


def result_error(value: int) -> Optional[int]:
    """The ZSTD error code a stream-ordered call left in its result word (e.g. 70, dstSize_tooSmall), or None for a size."""
    L = lib()
    return L.ZSTD_getErrorCode(value) if L.ZSTD_isError(value) else None


def _check(code: int) -> int:
    L = lib()
    if L.ZSTD_isError(code):
        raise ZstdError(L.ZSTD_getErrorCode(code), L.ZSTD_getErrorName(code).decode())
    return code


def ZSTD_compressBound(src_size: int) -> int:
    return lib().ZSTD_compressBound(src_size)


def _buf(data) -> Tuple[ctypes.c_void_p, int, object]:
    """(pointer, nbytes, keepalive) for bytes / bytearray / memoryview / numpy arrays."""
    if isinstance(data, (bytes, bytearray)):
        keep = (ctypes.c_char * len(data)).from_buffer_copy(data) if isinstance(data, bytes) else (ctypes.c_char * len(data)).from_buffer(data)
        return ctypes.cast(keep, _vp), len(data), keep
    mv = memoryview(data).cast("B")
    keep = (ctypes.c_char * len(mv)).from_buffer(mv) if not mv.readonly else (ctypes.c_char * len(mv)).from_buffer_copy(mv)
    return ctypes.cast(keep, _vp), len(mv), keep


class ZSTD_CDict:
    """Digested dictionary (lib/zstd.h:967-995): parsed once, resident on the GPU from its first use."""

    def __init__(self, dict_bytes, level: int = 3):
        p, n, keep = _buf(dict_bytes)
        self._h = lib().ZSTD_createCDict(p, n, level)
        if not self._h:
            raise ZstdError(30, "ZSTD_createCDict failed (dictionary corrupted or out of memory)")

    @property
    def dict_id(self) -> int:
        return int(lib().ZSTD_getDictID_fromCDict(self._h))

    def close(self):
        h, self._h = getattr(self, "_h", None), None
        if h and _lib is not None:
            _lib.ZSTD_freeCDict(h)

    def __del__(self):
        try:
            self.close()
        except Exception:      # interpreter teardown
            pass


class ZSTD_CCtx:
    """Reusable compression context (lib/zstd.h:259-264): owns the device workspace and a stream."""

    def __init__(self, device: Optional[int] = None):
        L = lib()
        if device is not None:
            L.ZSTDB200_setDevice(int(device))
        self._h = L.ZSTD_createCCtx()
        if not self._h:
            raise MemoryError("ZSTD_createCCtx failed")

    def close(self):
        h, self._h = getattr(self, "_h", None), None
        if h and _lib is not None:
            _lib.ZSTD_freeCCtx(h)

    def __del__(self):
        try:
            self.close()
        except Exception:      # interpreter teardown
            pass

    # -- reference-identical calls (host buffers) --
    def compress(self, src, level: int = 3, dst_capacity: Optional[int] = None) -> bytes:
        """ZSTD_compressCCtx: one complete frame (content size in header, no checksum)."""
        p, n, keep = _buf(src)
        cap = ZSTD_compressBound(n) if dst_capacity is None else dst_capacity
        dst = ctypes.create_string_buffer(max(cap, 1))
        r = _check(lib().ZSTD_compressCCtx(self._h, dst, cap, p, n, level))
        return dst.raw[:r]

    def compress_using_dict(self, src, dict_bytes, level: int = 3) -> bytes:
        p, n, keep = _buf(src)
        dp, dn, dkeep = _buf(dict_bytes)
        cap = ZSTD_compressBound(n)
        dst = ctypes.create_string_buffer(max(cap, 1))
        r = _check(lib().ZSTD_compress_usingDict(self._h, dst, cap, p, n, dp, dn, level))
        return dst.raw[:r]

    def compress_using_cdict(self, src, cdict: "ZSTD_CDict") -> bytes:
        """ZSTD_compress_usingCDict (lib/zstd.h:987): level and dictionary come from the CDict."""
        p, n, keep = _buf(src)
        cap = ZSTD_compressBound(n)
        dst = ctypes.create_string_buffer(max(cap, 1))
        r = _check(lib().ZSTD_compress_usingCDict(self._h, dst, cap, p, n, cdict._h))
        return dst.raw[:r]

    # -- advanced one-shot API (lib/zstd.h:337-603) --
    PARAMS = {"compression_level": 100, "content_size_flag": 200, "checksum_flag": 201, "dict_id_flag": 202, "nb_workers": 400,
              "enable_long_distance_matching": 160, "ldm_hash_log": 161, "ldm_min_match": 162, "ldm_bucket_size_log": 163,
              "ldm_hash_rate_log": 164}

    def set_parameter(self, name_or_id, value: int) -> None:
        """ZSTD_CCtx_setParameter: sticky until ZSTD_CCtx_reset(parameters)."""
        pid = self.PARAMS.get(name_or_id, name_or_id)
        _check(lib().ZSTD_CCtx_setParameter(self._h, int(pid), int(value)))

    def reset(self, directive: int = 3) -> None:
        """ZSTD_CCtx_reset: 1 session only, 2 parameters, 3 both."""
        _check(lib().ZSTD_CCtx_reset(self._h, directive))

    def load_dictionary(self, dict_bytes) -> None:
        p, n, keep = (None, 0, None) if not dict_bytes else _buf(dict_bytes)
        _check(lib().ZSTD_CCtx_loadDictionary(self._h, p, n))

    def ref_cdict(self, cdict: Optional["ZSTD_CDict"]) -> None:
        _check(lib().ZSTD_CCtx_refCDict(self._h, cdict._h if cdict is not None else None))

    def ref_prefix(self, prefix) -> None:
        """ZSTD_CCtx_refPrefix: raw content for the next frame only (compress2, compress_device, the first frame of a
        stream); it replaces any dictionary, None or b"" clears it.  The context reads the bytes in place, so this object
        keeps them until the next call of this method."""
        p, n, keep = (None, 0, None) if not prefix else _buf(prefix)
        _check(lib().ZSTD_CCtx_refPrefix(self._h, p, n))
        self._prefix = keep

    def ref_prefix_device(self, d_prefix: int, size: int) -> None:
        """ZSTDB200_CCtx_refPrefixDevice: the same with the prefix in device memory (an int, e.g. torch.Tensor.data_ptr()),
        for compress_device.  The caller keeps that memory alive until the frame is made."""
        _check(lib().ZSTDB200_CCtx_refPrefixDevice(self._h, d_prefix if size else None, size))
        self._prefix = None

    def compress2(self, src) -> bytes:
        """ZSTD_compress2 with the context's sticky parameters / dictionary."""
        p, n, keep = _buf(src)
        cap = ZSTD_compressBound(n) + 8
        dst = ctypes.create_string_buffer(max(cap, 1))
        r = _check(lib().ZSTD_compress2(self._h, dst, cap, p, n))
        return dst.raw[:r]

    # -- extensions beyond the reference API --
    def compress_device(self, d_dst: int, dst_capacity: int, d_src: int, src_size: int, level: int = 3, stream: int = 0) -> int:
        """One frame, device pointers (ints, e.g. torch.Tensor.data_ptr()).  Returns compressed size."""
        return _check(lib().ZSTDB200_compressDevice(self._h, d_dst, dst_capacity, d_src, src_size, level, stream))

    def compress_device_async(self, d_dst: int, dst_capacity: int, d_src: int, src_size: int, d_result: int, level: int = 3,
                              stream: int = 0) -> None:
        """ZSTDB200_compressDeviceAsync: one frame, enqueued on `stream` (a cudaStream_t as int, e.g.
        torch.cuda.current_stream().cuda_stream; 0 = the legacy default stream).  Returns once the work is enqueued; the
        size, or an error code, lands in the 8 bytes at d_result in stream order (see result_error)."""
        _check(lib().ZSTDB200_compressDeviceAsync(self._h, d_dst, dst_capacity, d_src, src_size, level, d_result, stream))

    def compress_frames_async(self, d_dst: int, dst_capacity: int, d_src: int, offsets: Sequence[int], sizes: Sequence[int],
                              d_result: int, level: int = 3, cdict: Optional["ZSTD_CDict"] = None, d_c_sizes: int = 0,
                              stream: int = 0) -> None:
        """ZSTDB200_compressFramesAsync: many frames, enqueued on `stream`; d_c_sizes (0 = none): one u64 per frame."""
        n = len(sizes)
        offs = (_sz * n)(*offsets)
        szs = (_sz * n)(*sizes)
        _check(lib().ZSTDB200_compressFramesAsync(self._h, d_dst, dst_capacity, d_src, offs, szs, n, cdict._h if cdict else None,
                                                  level, d_c_sizes or None, d_result, stream))

    def compress_frame_part(self, d_dst: int, dst_capacity: int, d_part: int, frame_size: int, part_begin: int, part_size: int,
                            level: int = 3, stream: int = 0) -> int:
        """This rank's share of a frame several GPUs compress together (ZSTDB200_compressFramePart).  d_part: device address
        of the frame's byte part_begin - min(part_begin, halo).  Returns the bytes this share contributes."""
        L = lib()
        L.ZSTDB200_compressFramePart.restype = _sz
        L.ZSTDB200_compressFramePart.argtypes = [_vp, _vp, _sz, _vp, _sz, _sz, _sz, ctypes.c_int, _vp]
        return _check(L.ZSTDB200_compressFramePart(self._h, d_dst, dst_capacity, d_part, frame_size, part_begin, part_size, level, stream))

    def compress_frames(self, dst: int, dst_capacity: int, src: int, offsets: Sequence[int], sizes: Sequence[int],
                        level: int = 3, device_memory: bool = True, dict_bytes=None, stream: int = 0):
        """Many independent frames in one call.  Returns (total_bytes, [compressed size per frame])."""
        n = len(sizes)
        offs = (_sz * n)(*offsets)
        szs = (_sz * n)(*sizes)
        csz = (_sz * n)()
        dp, dn, dkeep = (None, 0, None) if dict_bytes is None else _buf(dict_bytes)
        r = _check(lib().ZSTDB200_compressFrames(self._h, dst, dst_capacity, src, offs, szs, n, dp, dn, csz, level,
                                                1 if device_memory else 0, stream))
        return r, list(csz)

    def compress_frames_using_cdict(self, dst: int, dst_capacity: int, src: int, offsets: Sequence[int], sizes: Sequence[int],
                                    cdict: "ZSTD_CDict", device_memory: bool = True, stream: int = 0):
        """Many independent frames against one digested dictionary.  Returns (total_bytes, [size per frame])."""
        n = len(sizes)
        offs = (_sz * n)(*offsets)
        szs = (_sz * n)(*sizes)
        csz = (_sz * n)()
        r = _check(lib().ZSTDB200_compressFrames_usingCDict(self._h, dst, dst_capacity, src, offs, szs, n, cdict._h, csz,
                                                           1 if device_memory else 0, stream))
        return r, list(csz)

    def compress_frames_using_cdicts(self, dst: int, dst_capacity: int, src: int, offsets: Sequence[int], sizes: Sequence[int],
                                     cdicts: Optional[Sequence[Optional["ZSTD_CDict"]]], level: int = 3, device_memory: bool = True,
                                     stream: int = 0):
        """Many independent frames, frame i against cdicts[i] at its level (None: no dictionary, at `level`; cdicts None:
        None for every frame).  Returns (total_bytes, [size per frame])."""
        n = len(sizes)
        offs = (_sz * n)(*offsets)
        szs = (_sz * n)(*sizes)
        csz = (_sz * n)()
        cds = _cdict_array(cdicts, n)
        r = _check(lib().ZSTDB200_compressFrames_usingCDicts(self._h, dst, dst_capacity, src, offs, szs, n, cds, level, csz,
                                                            1 if device_memory else 0, stream))
        return r, list(csz)

    def compress_frames_async_using_cdicts(self, d_dst: int, dst_capacity: int, d_src: int, offsets: Sequence[int],
                                           sizes: Sequence[int], cdicts: Optional[Sequence[Optional["ZSTD_CDict"]]], d_result: int,
                                           level: int = 3, d_c_sizes: int = 0, stream: int = 0) -> None:
        """ZSTDB200_compressFramesAsync_usingCDicts: compress_frames_using_cdicts enqueued on `stream`, its verdict at
        d_result and (d_c_sizes, 0 = none) one u64 size per frame in device memory."""
        n = len(sizes)
        offs = (_sz * n)(*offsets)
        szs = (_sz * n)(*sizes)
        cds = _cdict_array(cdicts, n)
        _check(lib().ZSTDB200_compressFramesAsync_usingCDicts(self._h, d_dst, dst_capacity, d_src, offs, szs, n, cds, level,
                                                              d_c_sizes or None, d_result, stream))

    # -- sequence API (lib/zstd.h:1555-1644) --
    def compress_sequences(self, seqs, src, dst_capacity: Optional[int] = None) -> bytes:
        """ZSTD_compressSequences: one frame from the caller's sequences (host buffers).  seqs: an (n, 4) uint32 array of
        (offset, litLength, matchLength, rep) or a list of (offset, litLength, matchLength) tuples.  The block format is
        the sticky ZSTD_c_blockDelimiters (set_parameter(1008, 0 or 1)); level, checksum and dictionary apply as for
        compress2."""
        arr = _sequences(seqs)
        p, n, keep = _buf(src)
        cap = ZSTD_compressBound(n) + 8 if dst_capacity is None else dst_capacity
        dst = ctypes.create_string_buffer(max(cap, 1))
        r = _check(lib().ZSTD_compressSequences(self._h, dst, cap, arr.ctypes.data if len(arr) else None, len(arr), p, n))
        return dst.raw[:r]

    def compress_sequences_device(self, d_dst: int, dst_capacity: int, d_seqs: int, nb_seqs: int, d_src: int, src_size: int,
                                  stream: int = 0) -> int:
        """ZSTDB200_compressSequencesDevice: sequences (nb_seqs x 16 bytes), input and output in device memory (ints, e.g.
        torch.Tensor.data_ptr()).  Returns the compressed size."""
        return _check(lib().ZSTDB200_compressSequencesDevice(self._h, d_dst, dst_capacity, d_seqs, nb_seqs, d_src, src_size, stream))

    def generate_sequences(self, src):
        """ZSTD_generateSequences: the parse of the frame compress2 writes for src, as an (n, 4) uint32 array of
        (offset, litLength, matchLength, rep), every block closed by a delimiter (0, trailing literals, 0, 0)."""
        import numpy as np
        p, n, keep = _buf(src)
        cap = sequence_bound(n)
        out = np.zeros((cap, 4), dtype=np.uint32)
        r = _check(lib().ZSTD_generateSequences(self._h, out.ctypes.data, cap, p, n))
        return out[:r].copy()

    def generate_sequences_device(self, d_out: int, capacity: int, d_src: int, src_size: int, stream: int = 0) -> int:
        """ZSTDB200_generateSequencesDevice: the same rows into device memory (d_out: capacity x 16 bytes, 4-byte aligned;
        ints, e.g. torch.Tensor.data_ptr()).  Returns the number of rows."""
        return _check(lib().ZSTDB200_generateSequencesDevice(self._h, d_out, capacity, d_src, src_size, stream))

    def generate_sequences_device_async(self, d_out: int, capacity: int, d_src: int, src_size: int, d_result: int,
                                        stream: int = 0) -> None:
        """ZSTDB200_generateSequencesDeviceAsync: generate_sequences_device enqueued on `stream` (0 = the legacy default
        stream); the number of rows, or an error code, lands in the 8 bytes at d_result in stream order."""
        _check(lib().ZSTDB200_generateSequencesDeviceAsync(self._h, d_out, capacity, d_src, src_size, d_result, stream))

    def stats(self) -> Stats:
        s = Stats()
        lib().ZSTDB200_getLastStats(self._h, ctypes.byref(s))
        return s


def _cdict_array(cdicts, n):
    """the host array of n CDict handles a per-frame-dictionary call reads (None: a NULL array)"""
    if cdicts is None:
        return None
    if len(cdicts) != n:
        raise ValueError(f"{len(cdicts)} dictionaries for {n} frames")
    return (_vp * n)(*[(cd._h if cd is not None else None) for cd in cdicts])


def _ddict_array(ddicts, n):
    """the host array of n DDict handles a per-entry-dictionary call reads (None: a NULL array)"""
    if ddicts is None:
        return None
    if len(ddicts) != n:
        raise ValueError(f"{len(ddicts)} dictionaries for {n} entries")
    return (_vp * n)(*[(dd._h if dd is not None else None) for dd in ddicts])


def _sequences(seqs):
    """an (n, 4) uint32 array (offset, litLength, matchLength, rep) from such an array or from (offset, litLength,
    matchLength) tuples"""
    import numpy as np
    a = np.asarray(seqs, dtype=np.uint32)
    if a.size == 0:
        return np.zeros((0, 4), dtype=np.uint32)
    if a.ndim != 2 or a.shape[1] not in (3, 4):
        raise ValueError("sequences: an (n, 4) array or (offset, litLength, matchLength) tuples")
    if a.shape[1] == 3:
        a = np.concatenate([a, np.zeros((len(a), 1), dtype=np.uint32)], axis=1)
    return np.ascontiguousarray(a)


def sequence_bound(src_size: int) -> int:
    """ZSTD_sequenceBound: the most sequences (delimiters included) a frame of src_size bytes can need."""
    return int(lib().ZSTD_sequenceBound(src_size))


class ZSTD_DDict:
    """Digested dictionary of the decoder (lib/zstd.h:1000-1030): parsed on the host when created, resident on the GPU from
    its first use.  Raises ZstdError(30) for a zstd-format dictionary whose entropy tables the decoder refuses."""

    def __init__(self, dict_bytes):
        p, n, keep = _buf(dict_bytes)
        self._h = lib().ZSTD_createDDict(p, n)
        if not self._h:
            raise ZstdError(30, "ZSTD_createDDict failed (dictionary corrupted or out of memory)")

    @property
    def dict_id(self) -> int:
        return int(lib().ZSTD_getDictID_fromDDict(self._h))

    def close(self):
        h, self._h = getattr(self, "_h", None), None
        if h and _lib is not None:
            _lib.ZSTD_freeDDict(h)

    def __del__(self):
        try:
            self.close()
        except Exception:      # interpreter teardown
            pass


class ZSTD_DCtx:
    """Reusable decompression context (lib/zstd.h:289-299): owns the device workspace and a stream."""

    PARAMS = {"window_log_max": 100}

    def __init__(self, device: Optional[int] = None):
        L = lib()
        if device is not None:
            L.ZSTDB200_setDevice(int(device))
        self._h = L.ZSTD_createDCtx()
        if not self._h:
            raise MemoryError("ZSTD_createDCtx failed")

    def close(self):
        h, self._h = getattr(self, "_h", None), None
        if h and _lib is not None:
            _lib.ZSTD_freeDCtx(h)

    def __del__(self):
        try:
            self.close()
        except Exception:      # interpreter teardown
            pass

    def decompress(self, frames, max_size: Optional[int] = None) -> bytes:
        """ZSTD_decompressDCtx: one or more concatenated frames (host buffers).  max_size defaults to the content size
        the first frame's header states."""
        p, n, keep = _buf(frames)
        if max_size is None:
            cs = lib().ZSTD_getFrameContentSize(p, n)
            if cs >= (1 << 64) - 2:
                raise ZstdError(72, "content size unknown: pass max_size")
            max_size = cs
        dst = ctypes.create_string_buffer(max(max_size, 1))
        r = _check(lib().ZSTD_decompressDCtx(self._h, dst, max_size, p, n))
        return dst.raw[:r]

    def decompress_using_ddict(self, frames, ddict: Optional["ZSTD_DDict"], max_size: Optional[int] = None) -> bytes:
        """ZSTD_decompress_usingDDict (lib/zstd.h:1017); max_size as for decompress."""
        p, n, keep = _buf(frames)
        if max_size is None:
            max_size = self._content_size(p, n)
        dst = ctypes.create_string_buffer(max(max_size, 1))
        r = _check(lib().ZSTD_decompress_usingDDict(self._h, dst, max_size, p, n, ddict._h if ddict is not None else None))
        return dst.raw[:r]

    @staticmethod
    def _content_size(p, n) -> int:
        cs = lib().ZSTD_getFrameContentSize(p, n)
        if cs >= (1 << 64) - 2:
            raise ZstdError(72, "content size unknown: pass max_size")
        return cs

    # -- sticky dictionary and parameters (lib/zstd.h:609-650, 1160-1210) --
    def set_parameter(self, name_or_id, value: int) -> None:
        """ZSTD_DCtx_setParameter: "window_log_max" (100) only; sticky until reset(parameters)."""
        pid = self.PARAMS.get(name_or_id, name_or_id)
        _check(lib().ZSTD_DCtx_setParameter(self._h, int(pid), int(value)))

    def reset(self, directive: int = 3) -> None:
        """ZSTD_DCtx_reset: 1 session only, 2 parameters (and dictionary), 3 both."""
        _check(lib().ZSTD_DCtx_reset(self._h, directive))

    def load_dictionary(self, dict_bytes) -> None:
        """ZSTD_DCtx_loadDictionary: a copy, sticky; None or b"" clears it."""
        p, n, keep = (None, 0, None) if not dict_bytes else _buf(dict_bytes)
        _check(lib().ZSTD_DCtx_loadDictionary(self._h, p, n))

    def ref_ddict(self, ddict: Optional["ZSTD_DDict"]) -> None:
        """ZSTD_DCtx_refDDict: borrowed (keep the DDict alive while the context uses it), sticky; None clears it."""
        self._ddict = ddict
        _check(lib().ZSTD_DCtx_refDDict(self._h, ddict._h if ddict is not None else None))

    def ref_prefix(self, prefix) -> None:
        """ZSTD_DCtx_refPrefix: raw content for the next call only.  The context reads the bytes in place, so this object
        keeps them until that call."""
        p, n, keep = (None, 0, None) if not prefix else _buf(prefix)
        _check(lib().ZSTD_DCtx_refPrefix(self._h, p, n))
        self._prefix = keep

    def decompress_device(self, d_dst: int, dst_capacity: int, d_src: int, src_size: int, stream: int = 0) -> int:
        """Frames in device memory -> device memory (ints, e.g. torch.Tensor.data_ptr()).  Returns the decompressed size."""
        return _check(lib().ZSTDB200_decompressDevice(self._h, d_dst, dst_capacity, d_src, src_size, stream))

    def decompress_device_async(self, d_dst: int, dst_capacity: int, d_src: int, src_size: int, d_result: int,
                                stream: int = 0) -> None:
        """ZSTDB200_decompressDeviceAsync: frames in device memory, decoded on `stream` (a cudaStream_t as int, e.g.
        torch.cuda.current_stream().cuda_stream; 0 = the legacy default stream).  Returns once the work is enqueued; the
        decompressed size, or an error code, lands in the 8 bytes at d_result in stream order (see result_error)."""
        _check(lib().ZSTDB200_decompressDeviceAsync(self._h, d_dst, dst_capacity, d_src, src_size, d_result, stream))

    def decompress_frames(self, d_dst: int, dst_capacity: int, dst_offsets: Sequence[int], dst_capacities: Sequence[int],
                          d_src: int, src_size: int, src_offsets: Sequence[int], src_sizes: Sequence[int], stream: int = 0):
        """ZSTDB200_decompressFrames: entry i = d_src[src_offsets[i], + src_sizes[i]) decoded into its own slot
        d_dst[dst_offsets[i], + dst_capacities[i]) (device pointers as ints).  Returns (result, [result per entry]): the sum
        of the sizes, or the error code of the lowest-index entry that failed, and each entry's size or error code (see
        result_error).  Raises ZstdError when the call is refused before any entry is decoded."""
        n = len(src_sizes)
        if not (len(src_offsets) == len(dst_offsets) == len(dst_capacities) == n):
            raise ValueError("src_offsets, src_sizes, dst_offsets and dst_capacities differ in length")
        so, ss, do, dc = ((_sz * n)(*a) for a in (src_offsets, src_sizes, dst_offsets, dst_capacities))
        sizes = (_sz * n)()
        L = lib()
        r = L.ZSTDB200_decompressFrames(self._h, d_dst, dst_capacity, do, dc, d_src, src_size, so, ss, n, sizes, stream)
        if L.ZSTD_isError(r) and not any(L.ZSTD_isError(v) for v in sizes):
            _check(r)                                       # refused: no entry holds the error
        return r, list(sizes)

    def decompress_frames_async(self, d_dst: int, dst_capacity: int, dst_offsets: Sequence[int], dst_capacities: Sequence[int],
                                d_src: int, src_size: int, src_offsets: Sequence[int], src_sizes: Sequence[int], d_result: int,
                                d_d_sizes: int = 0, stream: int = 0) -> None:
        """ZSTDB200_decompressFramesAsync: decompress_frames enqueued on `stream`; its result lands in the 8 bytes at d_result
        and (d_d_sizes, 0 = none) each entry's result in one u64 per entry, in stream order."""
        n = len(src_sizes)
        if not (len(src_offsets) == len(dst_offsets) == len(dst_capacities) == n):
            raise ValueError("src_offsets, src_sizes, dst_offsets and dst_capacities differ in length")
        so, ss, do, dc = ((_sz * n)(*a) for a in (src_offsets, src_sizes, dst_offsets, dst_capacities))
        _check(lib().ZSTDB200_decompressFramesAsync(self._h, d_dst, dst_capacity, do, dc, d_src, src_size, so, ss, n,
                                                    d_d_sizes or None, d_result, stream))

    def decompress_frames_using_ddicts(self, d_dst: int, dst_capacity: int, dst_offsets: Sequence[int],
                                       dst_capacities: Sequence[int], d_src: int, src_size: int, src_offsets: Sequence[int],
                                       src_sizes: Sequence[int], ddicts: Optional[Sequence[Optional["ZSTD_DDict"]]], stream: int = 0):
        """ZSTDB200_decompressFrames_usingDDicts: decompress_frames with entry i decoded against ddicts[i] (None: no
        dictionary; ddicts None: none for any entry) instead of the sticky dictionary.  Returns (result, [result per entry])."""
        n = len(src_sizes)
        if not (len(src_offsets) == len(dst_offsets) == len(dst_capacities) == n):
            raise ValueError("src_offsets, src_sizes, dst_offsets and dst_capacities differ in length")
        so, ss, do, dc = ((_sz * n)(*a) for a in (src_offsets, src_sizes, dst_offsets, dst_capacities))
        dds = _ddict_array(ddicts, n)
        sizes = (_sz * n)()
        L = lib()
        r = L.ZSTDB200_decompressFrames_usingDDicts(self._h, d_dst, dst_capacity, do, dc, d_src, src_size, so, ss, n, dds, sizes, stream)
        if L.ZSTD_isError(r) and not any(L.ZSTD_isError(v) for v in sizes):
            _check(r)                                       # refused: no entry holds the error
        return r, list(sizes)

    def decompress_frames_async_using_ddicts(self, d_dst: int, dst_capacity: int, dst_offsets: Sequence[int],
                                             dst_capacities: Sequence[int], d_src: int, src_size: int, src_offsets: Sequence[int],
                                             src_sizes: Sequence[int], ddicts: Optional[Sequence[Optional["ZSTD_DDict"]]],
                                             d_result: int, d_d_sizes: int = 0, stream: int = 0) -> None:
        """ZSTDB200_decompressFramesAsync_usingDDicts: decompress_frames_using_ddicts enqueued on `stream`, its results in
        device memory as for decompress_frames_async.  The DDicts are kept alive until this context's next such call."""
        n = len(src_sizes)
        if not (len(src_offsets) == len(dst_offsets) == len(dst_capacities) == n):
            raise ValueError("src_offsets, src_sizes, dst_offsets and dst_capacities differ in length")
        so, ss, do, dc = ((_sz * n)(*a) for a in (src_offsets, src_sizes, dst_offsets, dst_capacities))
        dds = _ddict_array(ddicts, n)
        _check(lib().ZSTDB200_decompressFramesAsync_usingDDicts(self._h, d_dst, dst_capacity, do, dc, d_src, src_size, so, ss, n,
                                                                dds, d_d_sizes or None, d_result, stream))
        self._batch_ddicts = list(ddicts) if ddicts is not None else None     # the kernels read them after this returns

    def decompress_frames_async_device_offsets(self, d_dst: int, dst_capacity: int, d_dst_offsets: int, d_dst_capacities: int,
                                               d_src: int, src_size: int, d_src_offsets: int, d_src_sizes: int, nb_entries: int,
                                               d_result: int, d_d_sizes: int = 0, stream: int = 0) -> None:
        """ZSTDB200_decompressFramesAsync_deviceOffsets: decompress_frames_async with the four arrays in device memory (one
        u64 per entry each, 8-byte aligned, e.g. int64 tensors' data_ptr()), read by the call's kernels in stream order.  An
        array out of bounds gives parameter_outOfBound (42) in *d_result, and nothing is written to d_dst or d_d_sizes."""
        _check(lib().ZSTDB200_decompressFramesAsync_deviceOffsets(self._h, d_dst, dst_capacity, d_dst_offsets or None,
                                                                  d_dst_capacities or None, d_src, src_size, d_src_offsets or None,
                                                                  d_src_sizes or None, nb_entries, d_d_sizes or None, d_result, stream))

    def find_decompressed_sizes_async(self, d_src: int, src_size: int, d_src_offsets: int, d_src_sizes: int, nb_entries: int,
                                      d_content_sizes: int = 0, d_bounds: int = 0, stream: int = 0) -> None:
        """ZSTDB200_findDecompressedSizesAsync: for entry i = d_src[src_offsets[i], + src_sizes[i]) (device arrays of one u64
        per entry), ZSTD_findDecompressedSize of it to d_content_sizes[i] and ZSTD_decompressBound to d_bounds[i] (0 = not
        wanted), in stream order.  A range outside [0, src_size) gets ZSTD_CONTENTSIZE_ERROR (2**64 - 2)."""
        _check(lib().ZSTDB200_findDecompressedSizesAsync(self._h, d_src, src_size, d_src_offsets or None, d_src_sizes or None,
                                                         nb_entries, d_content_sizes or None, d_bounds or None, stream))

    def stats(self) -> DStats:
        s = DStats()
        lib().ZSTDB200_getLastDStats(self._h, ctypes.byref(s))
        return s


def ZSTD_decompress(frames, max_size: Optional[int] = None) -> bytes:
    """lib/zstd.h:170 — temporary context, host buffers."""
    d = ZSTD_DCtx()
    try:
        return d.decompress(frames, max_size)
    finally:
        d.close()


def ZSTD_findDecompressedSize(frames) -> int:
    """lib/zstd.h:1437 — the content sizes of the frames in a host buffer summed (skippable frames count 0);
    ZSTD_CONTENTSIZE_UNKNOWN (2**64 - 1) when a frame states none, ZSTD_CONTENTSIZE_ERROR (2**64 - 2) for invalid input."""
    p, n, keep = _buf(frames)
    return lib().ZSTD_findDecompressedSize(p, n)


def ZSTD_decompressBound(frames) -> int:
    """lib/zstd.h:1460 — an upper bound of what the frames in a host buffer decompress to, from their headers;
    ZSTD_CONTENTSIZE_ERROR (2**64 - 2) for invalid input."""
    p, n, keep = _buf(frames)
    return lib().ZSTD_decompressBound(p, n)


def ZSTD_compress(src, level: int = 3) -> bytes:
    """lib/zstd.h:155 — temporary context, host buffers."""
    p, n, keep = _buf(src)
    cap = ZSTD_compressBound(n)
    dst = ctypes.create_string_buffer(max(cap, 1))
    r = _check(lib().ZSTD_compress(dst, cap, p, n, level))
    return dst.raw[:r]


def seek_table(c_sizes: Sequence[int], d_sizes: Sequence[int]) -> bytes:
    """ZSTDB200_writeSeekTable: the seekable-format footer for a run of frames (append it behind them)."""
    n = len(c_sizes)
    cs, ds = (_sz * n)(*c_sizes), (_sz * n)(*d_sizes)
    cap = 17 + 8 * n
    dst = ctypes.create_string_buffer(cap)
    L = lib()
    L.ZSTDB200_writeSeekTable.restype = _sz
    L.ZSTDB200_writeSeekTable.argtypes = [_vp, _sz, _vp, _vp, _sz]
    r = _check(L.ZSTDB200_writeSeekTable(dst, cap, cs, ds, n))
    return dst.raw[:r]


def device_available() -> bool:
    try:
        return bool(lib().ZSTDB200_deviceAvailable())
    except (ImportError, OSError):
        return False
