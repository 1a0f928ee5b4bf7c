"""Helpers of the sequence-API tests: the oracle's statement of ZSTD_compressSequences (oracle/zb_seqs.c), the frame
driver's own stores as sequences, and the chosen-sequence cases of seqgen.DICTATED with the sequences they were built
from.  TEST INFRASTRUCTURE ONLY."""
import ctypes

import numpy as np

import seqgen
import zref

_sz, _vp = ctypes.c_size_t, ctypes.c_void_p
EXTERNAL_SEQUENCES_INVALID = 107
_bound = False


def oracle():
    global _bound
    O = zref.oracle()
    if not _bound:
        O.zbo_compressSequences.restype = _sz
        O.zbo_compressSequences.argtypes = [_vp, _sz, _vp, _sz, _vp, _sz, _vp, _sz, ctypes.c_int, ctypes.c_int]
        O.zbo_frameSequences.restype = _sz
        O.zbo_frameSequences.argtypes = [_vp, _sz, _vp, _sz, _vp, _sz, ctypes.c_int]
        _bound = True
    return O


def error_code(r):
    """the zstd error code of a size_t result, 0 for a size"""
    return (1 << 64) - r if r > (1 << 64) - 121 else 0


def as_array(seqs):
    """(n, 4) uint32 array from an array or from (offset, litLength, matchLength) tuples"""
    a = np.asarray(seqs, dtype=np.uint32).reshape(-1, np.asarray(seqs).shape[-1] if len(seqs) else 4)
    if a.shape[1] == 3:
        a = np.concatenate([a, np.zeros((len(a), 1), np.uint32)], axis=1)
    return np.ascontiguousarray(a)


def compress_sequences(seqs, src, level, dict=None, explicit=True, cap=None):
    """zbo_compressSequences: the frame, or the error code (an int below 121) when the call fails"""
    a = as_array(seqs)
    cap = len(src) + (len(src) >> 8) + (128 << 10 >> 11) + 64 if cap is None else cap
    dst = ctypes.create_string_buffer(max(cap, 1))
    r = oracle().zbo_compressSequences(dst, cap, a.ctypes.data if len(a) else None, len(a), src, len(src),
                                       dict, len(dict) if dict else 0, level, 1 if explicit else 0)
    return error_code(r) or dst.raw[:r]


def frame_sequences(src, level, dict=None):
    """zbo_frameSequences: the frame driver's per-block stores, real offsets, each block closed by a delimiter"""
    cap = len(src) // 3 + len(src) // 1024 + 16
    out = np.zeros((cap, 4), np.uint32)
    r = oracle().zbo_frameSequences(out.ctypes.data, cap, src, len(src), dict, len(dict) if dict else 0, level)
    assert not error_code(r), error_code(r)
    return out[:r].copy()


def merge_delimiters(a):
    """ZSTD_mergeBlockDelimiters (zstd_compress.c:3497): the delimiters' literals move to the next sequence, the last
    delimiter's are dropped (they become the implicit trailing literals)"""
    a = a.copy()
    keep = []
    for i in range(len(a)):
        if a[i, 0] == 0 and a[i, 2] == 0:
            if i != len(a) - 1:
                a[i + 1, 1] += a[i, 1]
        else:
            keep.append(i)
    return a[keep]


def blocks_to_array(blocks):
    """seqgen's [(sequences (ll, off, ml), trailing)] as delimited ZSTD_Sequence rows"""
    rows = []
    for seqs, trailing in blocks:
        rows += [(off, ll, ml, 0) for ll, off, ml in seqs] + [(0, trailing, 0, 0)]
    return np.array(rows, dtype=np.uint32).reshape(-1, 4)


def dictated(monkeypatch, name):
    """the calls a seqgen.DICTATED builder makes to the reference's ZSTD_compressSequences: [(seqs, src, level, dict,
    reference frame)], one per frame it builds"""
    calls = []
    real = seqgen.ref_compress_sequences

    def record(blocks, src, level=3, dict=None, params=()):
        frame = real(blocks, src, level, dict, params)
        calls.append((blocks_to_array(blocks), src, level, dict, frame))
        return frame
    monkeypatch.setattr(seqgen, "ref_compress_sequences", record)
    seqgen.DICTATED[name]()
    monkeypatch.setattr(seqgen, "ref_compress_sequences", real)
    return calls
