"""Prefix (ZSTD_CCtx_refPrefix) test helpers: the oracle's frame against a prefix (oracle/zb_prefix.c), its match lists, the
reference's prefix calls, and the inputs the prefix tests share.  TEST INFRASTRUCTURE ONLY."""
import ctypes

import numpy as np

import ldmref
import zref

_sz, _vp = ctypes.c_size_t, ctypes.c_void_p
INDEX_MAX = 1 << 27                   # the prefix bytes a block can reach: the LDM window
LDM_MIN = 512 << 10                   # LDM runs when indexed prefix + frame is larger


_Lists = ldmref.LdmLists              # zbo_ldm_free is bound once, for both list producers


def _o():
    O = ldmref._o()
    if not getattr(O, "_prefix_bound", False):
        O.zbo_compress_ldm_usingPrefix.restype = _sz
        O.zbo_compress_ldm_usingPrefix.argtypes = [_vp, _sz, _vp, _sz, _vp, _sz, ctypes.c_int, ctypes.POINTER(ldmref.LdmParams)]
        O.zbo_compress_usingRawDict.restype = _sz
        O.zbo_compress_usingRawDict.argtypes = [_vp, _sz, _vp, _sz, _vp, _sz, ctypes.c_int]
        O.zbo_ldm_frame_usingPrefix.restype = _Lists
        O.zbo_ldm_frame_usingPrefix.argtypes = [_vp, _sz, _vp, _sz, ctypes.c_uint, ctypes.POINTER(ldmref.LdmParams)]
        O.zbo_ldm_free.restype = None
        O.zbo_ldm_free.argtypes = [ctypes.POINTER(_Lists)]
        O._prefix_bound = True
    return O


def oracle_prefix(src: bytes, prefix: bytes, level: int, ldm: bool = True, **prm) -> bytes:
    """zbo_compress_ldm_usingPrefix: the frame the GPU must produce for src after ZSTD_CCtx_refPrefix(prefix); ldm: with
    ZSTD_c_enableLongDistanceMatching = 1 and the ldm parameters of ldmref.oracle_ldm."""
    O = _o()
    p = ldmref.LdmParams(prm.get("hash_log", 0), prm.get("min_match", 0), prm.get("bucket_size_log", 0), prm.get("hash_rate_log", 0))
    cap = O.zbo_compressBound(len(src)) + 64
    dst = ctypes.create_string_buffer(cap)
    r = O.zbo_compress_ldm_usingPrefix(dst, cap, src, len(src), prefix, len(prefix), level, ctypes.byref(p) if ldm else None)
    if r > (1 << 63):
        raise RuntimeError(f"oracle error {-(r - (1 << 64))}")
    return dst.raw[:r]


def oracle_raw_dict(src: bytes, dict_bytes: bytes, level: int) -> bytes:
    O = _o()
    cap = O.zbo_compressBound(len(src)) + 64
    dst = ctypes.create_string_buffer(cap)
    r = O.zbo_compress_usingRawDict(dst, cap, src, len(src), dict_bytes, len(dict_bytes), level)
    if r > (1 << 63):
        raise RuntimeError(f"oracle error {-(r - (1 << 64))}")
    return dst.raw[:r]


def indexed(prefix: bytes) -> bytes:
    """the part of a prefix the LDM pass indexes: nothing of a prefix shorter than 8 bytes, else its last 2^27 bytes"""
    return b"" if len(prefix) < 8 else prefix[-INDEX_MAX:]


def lists(src: bytes, prefix: bytes, window_log: int, **prm) -> dict:
    """steps 3 and 4 of the rule for src behind the indexed prefix.  P: indexed prefix bytes; nb_survivors: of both segments;
    first: per block of the frame, the index of its first survivor; matches: (p, length, offset) in [prefix | frame]
    coordinates"""
    O = _o()
    pfx = indexed(prefix)
    p = ldmref.LdmParams(prm.get("hash_log", 0), prm.get("min_match", 0), prm.get("bucket_size_log", 0), prm.get("hash_rate_log", 0))
    L = O.zbo_ldm_frame_usingPrefix(pfx if pfx else None, len(pfx), src, len(src), window_log, ctypes.byref(p))
    out = {"P": len(pfx), "nb_survivors": L.nbSurvivors, "first": [L.first[k] for k in range(L.nbBlocks)], "matches": []}
    for k in range(L.nbBlocks):
        for j in range(L.cnt[k]):
            m = L.m[L.first[k] + j]
            out["matches"].append((len(pfx) + k * (128 << 10) + m.start, m.len, m.off))
    O.zbo_ldm_free(ctypes.byref(L))
    return out


def matches(src: bytes, prefix: bytes, window_log: int, **prm):
    L = lists(src, prefix, window_log, **prm)
    return L["matches"], L["P"]


def window_log(src_size: int, prefix_size: int) -> int:
    """the window of an LDM frame: 27 clamped to the size of prefix + frame (ZSTD_adjustCParams_internal)"""
    return min(27, max(10, (src_size + prefix_size - 1).bit_length()))


def _ref_bind():
    R = zref.ref()
    R.ZSTD_CCtx_setParameter.restype = _sz
    R.ZSTD_CCtx_setParameter.argtypes = [_vp, ctypes.c_int, ctypes.c_int]
    R.ZSTD_CCtx_refPrefix.restype = _sz
    R.ZSTD_CCtx_refPrefix.argtypes = [_vp, _vp, _sz]
    R.ZSTD_compress2.restype = _sz
    R.ZSTD_compress2.argtypes = [_vp, _vp, _sz, _vp, _sz]
    R.ZSTD_DCtx_refPrefix.restype = _sz
    R.ZSTD_DCtx_refPrefix.argtypes = [_vp, _vp, _sz]
    R.ZSTD_decompressDCtx.restype = _sz
    R.ZSTD_decompressDCtx.argtypes = [_vp, _vp, _sz, _vp, _sz]
    return R


def ref_compress_prefix(src: bytes, prefix: bytes, level: int, ldm: int = 1) -> bytes:
    """the reference's ZSTD_CCtx_refPrefix + ZSTD_compress2 with ZSTD_c_enableLongDistanceMatching = ldm (what its
    --patch-from does, without the window it adds)"""
    R = _ref_bind()
    c = R.ZSTD_createCCtx()
    try:
        assert not R.ZSTD_isError(R.ZSTD_CCtx_setParameter(c, 100, level))
        assert not R.ZSTD_isError(R.ZSTD_CCtx_setParameter(c, 160, ldm))
        assert not R.ZSTD_isError(R.ZSTD_CCtx_refPrefix(c, prefix, len(prefix)))
        cap = R.ZSTD_compressBound(len(src))
        dst = ctypes.create_string_buffer(max(cap, 1))
        r = R.ZSTD_compress2(c, dst, cap, src, len(src))
        assert not R.ZSTD_isError(r), R.ZSTD_getErrorName(r)
        return dst.raw[:r]
    finally:
        R.ZSTD_freeCCtx(c)


def ref_decompress_prefix(frame: bytes, prefix: bytes, max_size: int) -> bytes:
    """the reference decoder with ZSTD_DCtx_refPrefix: raw content whatever the prefix begins with (for a prefix without
    the dictionary magic this is ZSTD_decompress_usingDict)"""
    R = _ref_bind()
    d = R.ZSTD_createDCtx()
    try:
        assert not R.ZSTD_isError(R.ZSTD_DCtx_refPrefix(d, prefix, len(prefix)))
        out = ctypes.create_string_buffer(max(max_size, 1))
        r = R.ZSTD_decompressDCtx(d, out, max_size, frame, len(frame))
        if R.ZSTD_isError(r):
            raise ValueError("reference decoder: " + R.ZSTD_getErrorName(r).decode())
        return out.raw[:r]
    finally:
        R.ZSTD_freeDCtx(d)


def version_pair(size: int = 4 << 20, edits: int = 300, insert: int = 0, seed: int = 11):
    """(old, new): new is `edits` random byte edits away from old; insert > 0 also puts that many fresh bytes in at a
    quarter of the file, which shifts everything behind them (new keeps old's size)"""
    rng = np.random.default_rng(seed)
    old = np.frombuffer(zref.synthetic(size, seed=seed), dtype=np.uint8)
    new = old.copy()
    idx = rng.integers(0, size, edits)
    new[idx] = rng.integers(0, 256, edits, dtype=np.uint8)
    if insert:
        at = size // 4
        new = np.concatenate([new[:at], rng.integers(0, 256, insert, dtype=np.uint8), new[at:size - insert]])
    return old.tobytes(), new.tobytes()


def pairs():
    """name -> (prefix, src): the inputs every prefix path is held to"""
    old, new = version_pair()
    _, shifted = version_pair(insert=12345, seed=11)
    small = zref.synthetic(300 << 10, seed=21)
    return {
        "edits": (old, new),
        "shifted": (old, shifted),
        "same": (old, old),
        "unrelated": (zref.synthetic(2 << 20, seed=12), zref.synthetic(3 << 20, seed=13)),
        "prefix1": (b"x", new[:1 << 20]),
        "prefix7": (old[:7], new[:1 << 20]),
        "prefix100k": (old[:100 << 10], old[:100 << 10] * 2 + new[:1 << 20]),
        "prefix_larger": (old, new[1 << 20:2 << 20]),
        "small_frame_ldm": (old[:400 << 10], small[:100 << 10] + old[:200 << 10]),       # n <= 512 KiB < P + n
        "small_frame_no_ldm": (old[:100 << 10], small[:150 << 10] + old[:100 << 10]),    # P + n <= 512 KiB
        "magic": (bytes.fromhex("37a430ec") + old[4:1 << 20], new[:1 << 20]),
        "empty": (old[:1 << 20], b""),
    }
