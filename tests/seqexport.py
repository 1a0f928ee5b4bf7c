"""Helpers of the ZSTD_generateSequences tests: the repcode a frame codes each sequence with (fill_rep), a check of the
`rep` convention of ZSTD_copyBlockSequences (rep_consistent, zstd_compress.c:3411-3428), the input rebuilt from
sequences (replay), and a zstd-format dictionary's repcodes.  TEST INFRASTRUCTURE ONLY."""
import ctypes
import struct

import numpy as np

import zref

FORMAT_REP = (1, 4, 8)                               # zstd_internal.h:69


def update_rep(h, off_base, ll0):
    """ZSTD_updateRep (zstd_compress_internal.h): the history after a sequence of offBase off_base"""
    if off_base > 3:
        return (off_base - 3, h[0], h[1])
    rc = off_base - 1 + ll0
    if rc == 0:
        return h
    cur = h[0] - 1 if rc == 3 else h[rc]
    return (cur, h[0], h[2] if rc == 1 else h[1])


def _blocks(rows):
    """(first row, delimiter row) of every block of delimited rows"""
    start = 0
    for i in range(len(rows)):
        if rows[i, 0] == 0 and rows[i, 2] == 0:
            yield start, i
            start = i + 1
    assert start == len(rows), "rows do not end with a delimiter"


def fill_rep(rows, history=FORMAT_REP):
    """rows with `rep` set to the repcode the frame codes each sequence with: a history entry the offset equals, taken in
    ZSTD_storeSeq's order; the history is `history` at the first block and unknown (0, never equal) at every other"""
    out = rows.copy()
    for b, (s, e) in enumerate(_blocks(rows)):
        h = tuple(history) if b == 0 else (0, 0, 0)
        for i in range(s, e):
            off, ll = int(rows[i, 0]), int(rows[i, 1])
            if ll:
                cands = (h[0], h[1], h[2])
            else:
                cands = (h[1], h[2], h[0] - 1 if h[0] > 1 else 0)
            rep = next((k + 1 for k in range(3) if cands[k] == off), 0)
            out[i, 3] = rep
            h = update_rep(h, rep if rep else off + 3, ll == 0)
    return out


def rep_consistent(rows, history=FORMAT_REP, reset_each_block=False):
    """whether every sequence with rep != 0 has the offset that repcode stands for in the history it meets (rep 1-3 with
    literals: r1-r3; without: r2, r3, r1 - 1), the history running through the rows from `history` and, with
    reset_each_block, starting unknown (0) at every block but the first; delimiters have rep 0"""
    h = tuple(history)
    for b, (s, e) in enumerate(_blocks(rows)):
        if reset_each_block and b > 0:
            h = (0, 0, 0)
        for i in range(s, e):
            off, ll, rep = int(rows[i, 0]), int(rows[i, 1]), int(rows[i, 3])
            if rep > 3 or off == 0:
                return False
            if rep:
                want = h[rep - 1] if ll else (h[0] - 1 if rep == 3 else h[rep])
                if want != off:
                    return False
            h = update_rep(h, rep if rep else off + 3, ll == 0)
        if rows[e, 3] != 0:
            return False
    return True


def replay(rows, src, dict_content=b""):
    """the bytes the rows describe: literals taken from src at the current position, each match copied from what lies
    behind it (the dictionary's content, then the output); a match that reaches in front of the dictionary fails"""
    buf = bytearray(dict_content)
    d = len(buf)
    for off, ll, ml, _ in rows.tolist():
        pos = len(buf) - d
        buf += src[pos:pos + ll]
        if off == 0:
            continue
        start = len(buf) - off
        assert start >= 0, "match in front of the dictionary"
        for k in range(ml):                          # byte by byte: a match may overlap its own output
            buf.append(buf[start + k])
    return bytes(buf[d:])


def dict_rep(d):
    """the repcodes a zstd-format dictionary starts frames with (the 12 bytes in front of its content), or the format's
    for raw content"""
    if not d or struct.unpack_from("<I", d)[0] != 0xEC30A437:
        return FORMAT_REP
    O = zref.oracle()
    O.zbo_loadDictEntropy.restype = ctypes.c_size_t
    O.zbo_loadDictEntropy.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t]
    off = O.zbo_loadDictEntropy(ctypes.create_string_buffer(1 << 16), d, len(d))
    assert 12 <= off < len(d)
    return struct.unpack_from("<3I", d, off - 12)


def dict_content(d):
    """the content part of a dictionary (all of raw content)"""
    if not d or len(d) < 8:
        return b""
    if struct.unpack_from("<I", d)[0] != 0xEC30A437:
        return bytes(d)
    O = zref.oracle()
    O.zbo_loadDictEntropy.restype = ctypes.c_size_t
    O.zbo_loadDictEntropy.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t]
    return bytes(d[O.zbo_loadDictEntropy(ctypes.create_string_buffer(1 << 16), d, len(d)):])


def ref_generate_sequences(src, level):
    """the compiled reference's ZSTD_generateSequences at `level` (its rows, delimiters included)"""
    R = zref.ref()
    R.ZSTD_createCCtx.restype = ctypes.c_void_p
    R.ZSTD_freeCCtx.argtypes = [ctypes.c_void_p]
    R.ZSTD_CCtx_setParameter.restype = ctypes.c_size_t
    R.ZSTD_CCtx_setParameter.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
    R.ZSTD_generateSequences.restype = ctypes.c_size_t
    R.ZSTD_generateSequences.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t]
    R.ZSTD_isError.restype = ctypes.c_uint
    c = R.ZSTD_createCCtx()
    try:
        R.ZSTD_CCtx_setParameter(c, 100, level)
        cap = len(src) // 3 + len(src) // 1024 + 16
        out = np.zeros((cap, 4), np.uint32)
        n = R.ZSTD_generateSequences(c, out.ctypes.data, cap, src, len(src))
        assert not R.ZSTD_isError(n), R.ZSTD_getErrorName(n)
        return out[:n].copy()
    finally:
        R.ZSTD_freeCCtx(c)
