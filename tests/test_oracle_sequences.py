"""The oracle's statement of ZSTD_compressSequences (oracle/zb_seqs.c) on the CPU: the frame driver's own stores give its
frames back in both block formats, every chosen-sequence case of seqgen.DICTATED decodes with the reference decoder,
invalid sequences are refused, and the library's host helpers equal the reference's."""
import ctypes

import numpy as np
import pytest

import seqgen
import seqoracle as so
import zref
import zstd_b200

needs_ref = pytest.mark.skipif(not zref.have_ref(), reason="oracle/_ref/libzstd_ref.so not built")
needs_datagen = pytest.mark.skipif(not zref.have_datagen(), reason="oracle/_ref/datagen not built")
LEVELS = [1, 3, -3, -1]
GOLDEN = ["http", "huffman-compressed-larger", "large-literal-and-match-lengths", "PR-3517-block-splitter-corruption-test"]


def _identity(src, level, d=None):
    want = zref.oracle_compress_using_dict(src, d, level) if d else zref.oracle_compress(src, level)
    seqs = so.frame_sequences(src, level, d)
    assert so.compress_sequences(seqs, src, level, d, explicit=True) == want
    merged = so.merge_delimiters(seqs)
    assert so.compress_sequences(merged, src, level, d, explicit=False) == want


@needs_datagen
@pytest.mark.parametrize("level", LEVELS)
@pytest.mark.parametrize("p,mib", [(30, 1), (50, 3), (90, 8)])
def test_identity_datagen(p, mib, level):
    _identity(zref.datagen(mib << 20, p, seed=p), level)


@pytest.mark.parametrize("level", LEVELS)
@pytest.mark.parametrize("name", GOLDEN)
def test_identity_golden(name, level):
    _identity(zref.golden_input(name), level)


@needs_ref
@pytest.mark.parametrize("level", [1, 3, -3])
@pytest.mark.parametrize("kind", ["raw", "zdict"])
def test_identity_dictionary(kind, level):
    d = zref.golden_input(seqgen.ZDICT) if kind == "zdict" else zref.synthetic(40_000, 3, 0.5)
    src = zref.synthetic(700_000, 11, 0.6)
    _identity(src, level, d)


SIZES = {}


@needs_ref
@pytest.mark.parametrize("name", list(seqgen.DICTATED))
def test_dictated_roundtrip(name, monkeypatch):
    """every frame a DICTATED builder makes with the reference, made again from its sequences in both forms"""
    ours = theirs = 0
    for seqs, src, level, d, ref_frame in so.dictated(monkeypatch, name):
        for explicit in (True, False):
            arr = seqs if explicit else so.merge_delimiters(seqs)
            f = so.compress_sequences(arr, src, level, d, explicit)
            assert isinstance(f, bytes), f"error {f}"
            assert seqgen.ref_decompress(f, len(src), d) == src
        ours += len(so.compress_sequences(seqs, src, level, d, True))
        theirs += len(ref_frame)
    SIZES[name] = (ours, theirs)
    # sizes against the reference, as first recorded: within 1 % or 16 bytes (chain-40000: 76 against 63 bytes, window-1k
    # +0.6 %), except `repcodes` (+3.1 %), whose history runs through 85 blocks of 8 sequences: unknown history at each
    # block start writes those offsets in full
    assert ours <= theirs * (1.05 if name == "repcodes" else 1.01) + 16, (name, ours, theirs)


def _seqs(*rows):
    return np.array([r if len(r) == 4 else (*r, 0) for r in rows], dtype=np.uint32).reshape(-1, 4)


SRC = zref.synthetic(300_000, 4, 0.5)


@pytest.mark.parametrize("case", ["offset0", "short-match", "offset-beyond", "past-src", "no-final-delim", "block-too-big",
                                  "nodelim-past-src", "nodelim-delimiter"])
def test_invalid(case):
    """each invalid form returns externalSequences_invalid (107)"""
    n = len(SRC)
    s, explicit = {
        "offset0": (_seqs((0, 10, 5), (0, n - 15, 0)), True),
        "short-match": (_seqs((5, 10, 2), (0, n - 12, 0)), True),
        "offset-beyond": (_seqs((11, 5, 5), (0, n - 10, 0)), True),         # offset > position behind the sequence
        "past-src": (_seqs((5, 10, 5), (0, n, 0)), True),
        "no-final-delim": (_seqs((5, 10, 5), (0, 100, 0), (5, 10, 5)), True),
        "block-too-big": (_seqs((0, 131073, 0), (0, n - 131073, 0)), True),
        "nodelim-past-src": (_seqs((5, 10, 5), (5, n, 5)), False),
        "nodelim-delimiter": (_seqs((5, 10, 5), (0, 10, 0)), False),
    }[case]
    assert so.compress_sequences(s, SRC, 3, None, explicit) == so.EXTERNAL_SEQUENCES_INVALID


def _src(blocks, n):
    return seqgen.execute(blocks, np.random.default_rng(n), alphabet=8)


EDGES = {   # name: (sequences, explicit delimiters, input they describe)
    "trailing-run-no-delimiter": (_seqs((5, 10, 5)), False, _src([([(10, 5, 5)], 300_000)], 1)),
    "empty-blocks-and-late-delimiters": (_seqs((0, 0, 0), (0, 10, 0), (0, 0, 0), (5, 10, 5), (0, 100_000, 0), (0, 0, 0)), True,
                                         _src([([], 10), ([(10, 5, 5)], 100_000)], 2)),
    "blocks-of-1-to-6-bytes": (_seqs(*[(0, 1 + k % 6, 0) for k in range(3000)]), True, _src([([], sum(1 + k % 6 for k in range(3000)))], 3)),
    "block-of-128-KiB": (_seqs((0, 131072, 0), (0, 1000, 0)), True, _src([([], 132072)], 4)),
    "match-across-block-edges": (_seqs((7, 131070, 40), (1, 0, 262144), (9, 5, 3)), False, _src([([(131070, 7, 40), (0, 1, 262144), (5, 9, 3)], 77)], 5)),
}


@pytest.mark.parametrize("name", list(EDGES))
def test_valid_edges(name):
    s, explicit, src = EDGES[name]
    f = so.compress_sequences(s, src, 3, None, explicit, cap=4 * len(src) + 1024)      # 1-byte blocks: 4 bytes each
    assert isinstance(f, bytes), f
    if zref.have_ref():
        assert zref.ref_decompress(f, len(src)) == src


def test_empty_input():
    assert so.compress_sequences(_seqs(), b"", 3) == zref.oracle_compress(b"", 3)
    assert so.compress_sequences(_seqs((0, 0, 0)), b"", 3) == zref.oracle_compress(b"", 3)


def test_sequence_bound_and_merge():
    L = zstd_b200.lib()
    for n in (0, 1, 1023, 1024, 131072, 10 ** 9):
        want = n // 3 + 1 + n // 1024 + 1
        assert L.ZSTD_sequenceBound(n) == want
        if zref.have_ref():
            R = zref.ref()
            R.ZSTD_sequenceBound.restype = ctypes.c_size_t
            R.ZSTD_sequenceBound.argtypes = [ctypes.c_size_t]
            assert R.ZSTD_sequenceBound(n) == want
    rng = np.random.default_rng(1)
    a = rng.integers(0, 50, (400, 4)).astype(np.uint32)
    a[rng.random(400) < 0.3, 0] = 0
    a[rng.random(400) < 0.5, 2] = 0
    got = a.copy()
    k = L.ZSTD_mergeBlockDelimiters(got.ctypes.data, len(got))
    want = so.merge_delimiters(a)
    assert k == len(want) and (got[:k] == want).all()
    if zref.have_ref():
        R = zref.ref()
        R.ZSTD_mergeBlockDelimiters.restype = ctypes.c_size_t
        R.ZSTD_mergeBlockDelimiters.argtypes = [ctypes.c_void_p, ctypes.c_size_t]
        r = a.copy()
        assert R.ZSTD_mergeBlockDelimiters(r.ctypes.data, len(r)) == k and (r[:k] == got[:k]).all()


def test_error_name():
    assert zstd_b200.lib().ZSTD_getErrorName((1 << 64) - 107) == b"External sequences are not valid"
