"""ZSTD_generateSequences without a GPU: the helpers the GPU tests rely on, pinned against the compiled reference and the
oracle, and the new entry points' presence and refusal without a device."""
import ctypes

import numpy as np
import pytest

import seqexport as sx
import seqgen
import seqoracle as so
import zref
import zstd_b200

needs_ref = pytest.mark.skipif(not zref.have_ref(), reason="oracle/_ref/libzstd_ref.so not built")
SRC = zref.synthetic(300_000, 11, 0.6)


@needs_ref
@pytest.mark.parametrize("level", [1, 3, 19])
def test_rep_convention_of_the_reference(level):
    """the reference's own ZSTD_generateSequences rows, history carried from block to block, as its frame carries it"""
    rows = sx.ref_generate_sequences(SRC, level)
    assert rows[:, 3].any(), "no repcode in the reference's rows: the check would pin nothing"
    assert sx.rep_consistent(rows, reset_each_block=False)
    assert sx.replay(rows, SRC) == SRC


@pytest.mark.parametrize("level", [1, 3, -3])
def test_rep_filled_oracle_rows(level):
    """the oracle's rows with `rep` filled, history unknown at every block but the first, as this library's frames code it"""
    rows = sx.fill_rep(so.frame_sequences(SRC, level))
    assert rows[:, 3].any()
    assert sx.rep_consistent(rows, reset_each_block=True)
    assert so.compress_sequences(rows, SRC, level) == zref.oracle_compress(SRC, level)
    bad = rows.copy()                                # a repcode naming another slot of the history is caught
    i = int(np.flatnonzero(bad[:, 3] == 1)[0])
    bad[i, 3] = 2
    assert not sx.rep_consistent(bad, reset_each_block=True)


@pytest.mark.parametrize("kind", ["none", "raw", "zdict"])
def test_replay_oracle_rows(kind):
    d = None if kind == "none" else (zref.golden_input(seqgen.ZDICT) if kind == "zdict" else zref.synthetic(40_000, 3, 0.5))
    rows = sx.fill_rep(so.frame_sequences(SRC, 3, d), sx.dict_rep(d))
    assert sx.replay(rows, SRC, sx.dict_content(d)) == SRC
    assert sx.rep_consistent(rows, sx.dict_rep(d), reset_each_block=True)
    if kind == "raw":                                # its content is made by the input's own generator
        ends = np.cumsum(rows[:, 1].astype(np.int64) + rows[:, 2])
        assert (rows[:, 0] > ends - rows[:, 2]).any(), "no match reaches into the dictionary"


def test_symbols_exported():
    L = zstd_b200.lib()
    for name in ("ZSTD_generateSequences", "ZSTDB200_generateSequencesDevice", "ZSTDB200_generateSequencesDeviceAsync"):
        assert hasattr(L, name), name


@pytest.mark.skipif(zstd_b200.device_available(), reason="CUDA device present")
def test_generic_without_device():
    """no CPU fallback: every form returns GENERIC (1) without a device"""
    L = zstd_b200.lib()
    c = L.ZSTD_createCCtx()
    out = np.zeros((64, 4), np.uint32)
    src = b"abcdefgh" * 16
    result = ctypes.c_ulonglong(0)
    try:
        for r in (L.ZSTD_generateSequences(c, out.ctypes.data, 64, src, len(src)),
                  L.ZSTDB200_generateSequencesDevice(c, out.ctypes.data, 64, src, len(src), None),
                  L.ZSTDB200_generateSequencesDeviceAsync(c, out.ctypes.data, 64, src, len(src), ctypes.addressof(result), None)):
            assert L.ZSTD_getErrorCode(r) == 1
        assert not out.any()
        assert L.ZSTDB200_generateSequencesDeviceAsync(c, out.ctypes.data, 64, src, len(src), None, None) == (1 << 64) - 1
        assert L.ZSTD_generateSequences(None, out.ctypes.data, 64, src, len(src)) == (1 << 64) - 1
    finally:
        L.ZSTD_freeCCtx(c)
