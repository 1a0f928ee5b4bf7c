"""Long-distance matching test helpers: the oracle's LDM frame (oracle/zb_ldm.c), the reference's LDM frame, the oracle's
survivors, and the inputs the LDM tests share.  TEST INFRASTRUCTURE ONLY."""
import ctypes

import numpy as np

import zref

_sz, _vp = ctypes.c_size_t, ctypes.c_void_p
PIECE = 1 << 20                       # A+B+A pieces: the copy lies beyond the parse's reach (128 KiB primed per chunk)


class LdmParams(ctypes.Structure):
    _fields_ = [("hashLog", ctypes.c_uint), ("minMatch", ctypes.c_uint), ("bucketSizeLog", ctypes.c_uint), ("hashRateLog", ctypes.c_uint)]


class LdmMatch(ctypes.Structure):     # zbo_ldm_match: start relative to its block
    _fields_ = [("start", ctypes.c_uint), ("len", ctypes.c_uint), ("off", ctypes.c_uint)]


class LdmLists(ctypes.Structure):     # zbo_ldm_lists
    _fields_ = [("nbBlocks", _sz), ("nbSurvivors", _sz), ("first", ctypes.POINTER(ctypes.c_uint64)), ("cnt", ctypes.POINTER(ctypes.c_uint)),
                ("m", ctypes.POINTER(LdmMatch))]


def _o():
    O = zref.oracle()
    if not getattr(O, "_ldm_bound", False):
        import dfastgen
        O.zbo_compress_ldm.restype = _sz
        O.zbo_compress_ldm.argtypes = [_vp, _sz, _vp, _sz, ctypes.c_int, ctypes.POINTER(LdmParams)]
        O.zbo_compress_ldm_usingDict.restype = _sz
        O.zbo_compress_ldm_usingDict.argtypes = [_vp, _sz, _vp, _sz, _vp, _sz, ctypes.c_int, ctypes.POINTER(LdmParams)]
        O.zbo_ldm_resolve.restype = LdmParams
        O.zbo_ldm_resolve.argtypes = [ctypes.POINTER(LdmParams), ctypes.c_uint]
        O.zbo_ldm_survivors.restype = _sz
        O.zbo_ldm_survivors.argtypes = [_vp, _sz, ctypes.POINTER(LdmParams), _vp, _vp]
        O.zbo_ldm_frame.restype = LdmLists
        O.zbo_ldm_frame.argtypes = [_vp, _sz, ctypes.c_uint, ctypes.POINTER(LdmParams)]
        O.zbo_ldm_free.restype = None
        O.zbo_ldm_free.argtypes = [ctypes.POINTER(LdmLists)]
        O.zbo_ldm_overlayBlock.restype = _sz
        O.zbo_ldm_overlayBlock.argtypes = [_vp, _sz, ctypes.POINTER(ctypes.c_uint * 3), ctypes.POINTER(LdmMatch), _sz,
                                           ctypes.POINTER(dfastgen.Seq), _sz, _vp, ctypes.POINTER(_sz)]
        O.zbo_getCParams_ldm.restype = dfastgen.OCParams
        O.zbo_getCParams_ldm.argtypes = [ctypes.c_int, ctypes.c_ulonglong, _sz]
        O._ldm_bound = True
    return O


def oracle_ldm(src: bytes, level: int, hash_log=0, min_match=0, bucket_size_log=0, hash_rate_log=0) -> bytes:
    """zbo_compress_ldm: the frame the GPU must produce with ZSTD_c_enableLongDistanceMatching = 1."""
    O = _o()
    prm = LdmParams(hash_log, min_match, bucket_size_log, hash_rate_log)
    cap = O.zbo_compressBound(len(src)) + 64
    dst = ctypes.create_string_buffer(cap)
    r = O.zbo_compress_ldm(dst, cap, src, len(src), level, ctypes.byref(prm))
    if r > (1 << 63):
        raise RuntimeError(f"oracle error {-(r - (1 << 64))}")
    return dst.raw[:r]


def oracle_ldm_using_dict(src: bytes, dict_bytes: bytes, level: int, hash_log=0, min_match=0, bucket_size_log=0,
                          hash_rate_log=0) -> bytes:
    """zbo_compress_ldm_usingDict: the frame the GPU must produce with LDM on against a dictionary (raw or zstd-format)"""
    O = _o()
    prm = LdmParams(hash_log, min_match, bucket_size_log, hash_rate_log)
    cap = O.zbo_compressBound(len(src)) + 64
    dst = ctypes.create_string_buffer(cap)
    r = O.zbo_compress_ldm_usingDict(dst, cap, src, len(src), dict_bytes, len(dict_bytes), level, ctypes.byref(prm))
    if r > (1 << 63):
        raise RuntimeError(f"oracle error {-(r - (1 << 64))}")
    return dst.raw[:r]


def cparams_ldm(level: int, src_size: int, dict_size: int = 0):
    """zbo_getCParams_ldm: the cParams of a frame with LDM on"""
    return _o().zbo_getCParams_ldm(level, src_size, dict_size)


def resolve(window_log: int, hash_log=0, min_match=0, bucket_size_log=0, hash_rate_log=0) -> LdmParams:
    prm = LdmParams(hash_log, min_match, bucket_size_log, hash_rate_log)
    return _o().zbo_ldm_resolve(ctypes.byref(prm), window_log)


def survivors_v(src: bytes, prm: LdmParams):
    """(positions, XXH64 values) of the split points that survive the thinning (steps 1 and 2 of the rule)"""
    cap = len(src) // prm.minMatch + 1
    pos = np.zeros(cap, dtype=np.uint64)
    v = np.zeros(cap, dtype=np.uint64)
    n = _o().zbo_ldm_survivors(src, len(src), ctypes.byref(prm), pos.ctypes.data, v.ctypes.data)
    return pos[:n], v[:n]


def survivors(src: bytes, prm: LdmParams) -> np.ndarray:
    """positions of the split points that survive the thinning (steps 1 and 2 of the rule)"""
    return survivors_v(src, prm)[0]


def frame_lists(src: bytes, window_log: int, hash_log=0, min_match=0, bucket_size_log=0, hash_rate_log=0):
    """zbo_ldm_frame (steps 3 and 4): per block of src, its matches [(start in the block, length, offset)]"""
    O = _o()
    prm = LdmParams(hash_log, min_match, bucket_size_log, hash_rate_log)
    L = O.zbo_ldm_frame(src, len(src), window_log, ctypes.byref(prm))
    try:
        return [[(L.m[L.first[k] + j].start, L.m[L.first[k] + j].len, L.m[L.first[k] + j].off) for j in range(L.cnt[k])]
                for k in range(L.nbBlocks)]
    finally:
        O.zbo_ldm_free(ctypes.byref(L))


def overlay_block(blk: bytes, reps, matches, seqs):
    """zbo_ldm_overlayBlock (step 5): a block's final parse sequences [(offBase, litLen, matchLen)] with its LDM matches
    laid over them, repcodes assigned again from `reps`; returns (sequences, literal count)"""
    import dfastgen
    O = _o()
    nL, nS = len(matches), len(seqs)
    lm = (LdmMatch * max(nL, 1))(*[LdmMatch(*m) for m in matches])
    sq = (dfastgen.Seq * (nS + nL + 1))(*[dfastgen.Seq(*s) for s in seqs])
    lit = ctypes.create_string_buffer(len(blk) + 64)
    lsz = _sz()
    rep = (ctypes.c_uint * 3)(*reps)
    n = O.zbo_ldm_overlayBlock(blk, len(blk), ctypes.byref(rep), lm, nL, sq, nS, lit, ctypes.byref(lsz))
    return [(sq[i].offBase, sq[i].litLen, sq[i].matchLen) for i in range(n)], lsz.value


def ref_compress2(src: bytes, level: int, ldm: int) -> bytes:
    """the reference's ZSTD_compress2 with ZSTD_c_enableLongDistanceMatching = ldm (1 enable, 2 disable)"""
    R = zref.ref()
    R.ZSTD_CCtx_setParameter.restype = _sz
    R.ZSTD_CCtx_setParameter.argtypes = [_vp, ctypes.c_int, ctypes.c_int]
    R.ZSTD_compress2.restype = _sz
    R.ZSTD_compress2.argtypes = [_vp, _vp, _sz, _vp, _sz]
    c = R.ZSTD_createCCtx()
    try:
        assert not R.ZSTD_isError(R.ZSTD_CCtx_setParameter(c, 100, level))
        assert not R.ZSTD_isError(R.ZSTD_CCtx_setParameter(c, 160, ldm))
        cap = R.ZSTD_compressBound(len(src))
        dst = ctypes.create_string_buffer(cap)
        r = R.ZSTD_compress2(c, dst, cap, src, len(src))
        assert not R.ZSTD_isError(r), R.ZSTD_getErrorName(r)
        return dst.raw[:r]
    finally:
        R.ZSTD_freeCCtx(c)


def aba(piece: int = PIECE) -> bytes:
    """A + B + A: the second A is a copy `2 * piece` bytes back"""
    a, b = zref.synthetic(piece, seed=1), zref.synthetic(piece, seed=2)
    return a + b + a


def versions(size: int = 256 << 10, count: int = 16, edits: int = 400, seed: int = 3) -> bytes:
    """`count` versions of one file, each `edits` random byte edits away from the one before"""
    rng = np.random.default_rng(seed)
    cur = np.frombuffer(zref.synthetic(size, seed=seed), dtype=np.uint8).copy()
    out = []
    for _ in range(count):
        out.append(cur.tobytes())
        idx = rng.integers(0, size, edits)
        cur[idx] = rng.integers(0, 256, edits, dtype=np.uint8)
    return b"".join(out)


def period(n: int = 8 << 20, p: int = 4 << 10, seed: int = 5) -> bytes:
    unit = zref.random_bytes(p, seed=seed)
    return (unit * (n // p + 1))[:n]


def inputs():
    """name -> bytes: the inputs every LDM path is held to"""
    return {
        "aba": aba(),
        "versions": versions(),
        "zeros": bytes(8 << 20),
        "random": zref.random_bytes(8 << 20, seed=4),
        "period4k": period(),
    }


# parameter corners: minMatch 4 with hashRateLog 0, bucketSizeLog 1 and 8, hashLog 6 and 30
CORNERS = [dict(min_match=4, hash_rate_log=0), dict(min_match=4, hash_rate_log=1), dict(bucket_size_log=1), dict(bucket_size_log=8),
           dict(hash_log=6), dict(hash_log=30)]
