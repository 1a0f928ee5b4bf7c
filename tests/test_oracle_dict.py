"""ZSTD_compress_usingDict path of the oracle (BASELINE config 5 shape: small records + shared dictionary).
Frames must decode with the reference's ZSTD_decompress_usingDict and stay within +-0.5 % of the
reference's size for raw-content and zstd-format dictionaries; the dictionary entropy stage (treeless
literals, set_repeat tables, start repcodes) is pinned byte-for-byte against ZSTD_loadCEntropy +
ZSTD_entropyCompressSeqStore of the compiled reference."""
import ctypes
import random

import pytest

import zref
import zstd_b200
from test_host_decode import H, dec  # noqa: F401  (H: the CPU decode harness fixture)

needs_ref = pytest.mark.skipif(not zref.have_ref(), reason="oracle/_ref/libzstd_ref.so not built")
REC = 1024


def records(n, seed, p=0.5):
    data = zref.synthetic(REC * n, seed, p)
    return [data[i * REC:(i + 1) * REC] for i in range(n)]


@needs_ref
@pytest.mark.parametrize("dict_name", ["zdict-16k-synthetic-seed77", "http-dict-missing-symbols", "zero-weight-dict"])
def test_zstd_format_dictionaries_roundtrip(dict_name):
    d = zref.golden_input(dict_name)
    tot_o = tot_r = 0
    srcs = records(200, 5) + [b"", b"a", zref.golden_input("http"), zref.synthetic(300_000, 8)]
    for src in srcs:
        f = zref.oracle_compress_using_dict(src, d, 1)
        assert zref.ref_decompress_using_dict(f, d, len(src)) == src
        assert f[4] & 3, "dictID must be present in the frame header for a zstd-format dictionary"
        tot_o += len(f)
        tot_r += len(zref.ref_compress_using_dict(src, d, 1))
    if dict_name.startswith('zdict'):
        assert abs(tot_o - tot_r) / tot_r <= 0.01, (tot_o, tot_r)
    else:
        assert tot_o < tot_r * 1.03          # tiny hand-made dictionaries of the reference's test suite


@needs_ref
def test_raw_content_dictionary_size_parity():
    d = zref.synthetic(32 << 10, 123, 0.5)                 # no magic number -> raw content (zstd_compress.c:5143-5148)
    tot_o = tot_r = 0
    for src in records(400, 6):
        f = zref.oracle_compress_using_dict(src, d, 1)
        assert zref.ref_decompress_using_dict(f, d, len(src)) == src
        assert (f[4] & 3) == 0                              # no dictID for raw content (lib/zstd.h:185-186)
        tot_o += len(f)
        tot_r += len(zref.ref_compress_using_dict(src, d, 1))
    assert abs(tot_o - tot_r) / tot_r <= 0.01


@needs_ref
def test_dictionary_content_is_actually_used():
    """A record that is a verbatim slice of the dictionary must compress to almost nothing."""
    d = zref.synthetic(32 << 10, 321, 0.1)
    src = d[5000:6024]
    with_dict = zref.oracle_compress_using_dict(src, d, 1)
    without = zref.oracle_compress(src, 1)
    assert zref.ref_decompress_using_dict(with_dict, d, len(src)) == src
    assert len(with_dict) < 100 < len(without)


@needs_ref
def test_short_and_corrupted_dictionaries():
    src = zref.synthetic(5000, 1)
    assert zref.oracle_compress_using_dict(src, b"1234567", 1) == zref.oracle_compress(src, 1)      # < 8 bytes: ignored
    bad = bytes.fromhex("37a430ec01000000") + bytes(40)
    with pytest.raises(RuntimeError, match="30"):                                                     # dictionary_corrupted
        zref.oracle_compress_using_dict(src, bad, 1)


@needs_ref
@pytest.mark.parametrize("dict_name", ["zdict-16k-synthetic-seed77", "http-dict-missing-symbols", "zero-weight-dict"])
def test_dictionary_entropy_stage_byte_exact(dict_name):
    """oracle/zb_dict.c + zbo_entropyCompressBlock_prev vs the reference's ZSTD_loadCEntropy (zstd_compress.c:4987)
    + ZSTD_entropyCompressSeqStore (:3001) on randomised seqStores, through oracle/ref_shim.c."""
    import ctypes
    import numpy as np
    from test_oracle_entropy import make_seqstore
    R, O = zref.ref(), zref.oracle()
    c_sz, vp = ctypes.c_size_t, ctypes.c_void_p
    R.ref_entropyCompressBlock_dict.restype = c_sz
    R.ref_entropyCompressBlock_dict.argtypes = [vp, c_sz, vp, vp, vp, c_sz, vp, c_sz, c_sz, ctypes.c_int, ctypes.c_uint, vp, c_sz]
    O.zbo_loadDictEntropy.restype = c_sz
    O.zbo_loadDictEntropy.argtypes = [vp, vp, c_sz]
    O.zbo_entropyCompressBlock_prev.restype = c_sz
    O.zbo_entropyCompressBlock_prev.argtypes = [vp, c_sz, vp, c_sz, vp, c_sz, c_sz, ctypes.c_uint, ctypes.c_int, vp]
    d = zref.golden_input(dict_name)
    de = ctypes.create_string_buffer(16384)
    assert 8 < O.zbo_loadDictEntropy(de, d, len(d)) < len(d)
    rng = np.random.default_rng(5)
    compressed = 0
    for t in range(250):
        case = make_seqstore(rng)
        if case is None:
            continue
        offb, ll, ml, lits, block, strategy, tl = case
        if t % 2 == 0:                                             # the small-record regime (preferRepeat, set_repeat)
            k = max(1, min(len(offb), 40))
            offb, ll, ml = offb[:k], ll[:k], ml[:k]
            lits = lits[:min(len(lits), int(ll.sum()) + 50)]
            if int(ll.sum()) > len(lits):
                continue
            block = max(7, min(131072, len(lits) + int(ml.sum())))
        nseq = len(offb)
        cap = 1 << 20
        d1, d2 = ctypes.create_string_buffer(cap), ctypes.create_string_buffer(cap)
        seqs = np.ascontiguousarray(np.stack([offb, ll, ml], axis=1).astype(np.uint32)) if nseq else np.zeros((0, 3), np.uint32)
        offb, ll, ml = (np.ascontiguousarray(a, dtype=np.uint32) for a in (offb, ll, ml))
        lits = np.ascontiguousarray(lits)
        tlv = tl if strategy == 1 else 0
        r1 = R.ref_entropyCompressBlock_dict(d1, cap, offb.ctypes.data, ll.ctypes.data, ml.ctypes.data, nseq, lits.ctypes.data, len(lits), block, 1, tlv, d, len(d))
        with zref.entropy_model(0):                                 # the restatement of the reference's table builders
            r2 = O.zbo_entropyCompressBlock_prev(d2, cap, seqs.ctypes.data, nseq, lits.ctypes.data, len(lits), block, 1, 1 if tlv > 0 else 0, de)
        assert r1 == r2
        if r1 < (1 << 60):
            assert d1.raw[:r1] == d2.raw[:r2]
            compressed += r1 > 0
    assert compressed > 80


@needs_ref
@pytest.mark.skipif(not zref.have_datagen(), reason="oracle/_ref/datagen not built")
@pytest.mark.parametrize("level", [1, 3, -3])
def test_size_parity_with_reference_cdict(level):
    """ZSTD_compress_usingCDict is the production form of config 5 (SURVEY.md §8f rank 1).  The GPU CDict path
    emits the bytes of the usingDict path, so the oracle's usingDict output must sit within +-1 % of what the
    reference's ZSTD_compress_usingCDict produces on config 5's data (datagen -P50 cut into 1 KiB records,
    16 KiB ZDICT dictionary) — including level 3, where both run doubleFast over a dictionary."""
    data = zref.datagen(REC * 6000, 50)
    d = zref.train_dict(data, REC, 4000, 16 << 10)
    srcs = [data[i * REC:(i + 1) * REC] for i in range(4000, 5000)]
    ref_frames = zref.ref_compress_using_cdict(srcs, d, level)
    tot_o = 0
    for k, src in enumerate(srcs):
        f = zref.oracle_compress_using_dict(src, d, level)
        if k % 25 == 0:
            assert zref.ref_decompress_using_dict(f, d, len(src)) == src
        tot_o += len(f)
    tot_r = sum(len(f) for f in ref_frames)
    assert abs(tot_o - tot_r) / tot_r <= 0.01, (tot_o, tot_r)


def _huf_desc_len(d):
    """bytes of the Huffman tree description at d[8:] (format: "Huffman Tree Description")"""
    hb = d[8]
    return 1 + (hb - 127 + 1) // 2 if hb >= 128 else 1 + hb


def _oracle_load(d):
    """zbo_loadDictEntropy: the content offset, or an error code (> 2^63)"""
    O = zref.oracle()
    O.zbo_loadDictEntropy.restype = ctypes.c_size_t
    O.zbo_loadDictEntropy.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t]
    return O.zbo_loadDictEntropy(ctypes.create_string_buffer(16384), d, len(d))


def _cdict_decisions(dicts):
    """(product, oracle, reference) for every dictionary: accepted (True) or refused by the product's ZSTD_createCDict, the
    oracle's zbo_loadDictEntropy and the reference's ZSTD_createCDict"""
    L, R = zstd_b200.lib(), zref.ref()
    L.ZSTD_freeCDict.argtypes = [ctypes.c_void_p]
    R.ZSTD_createCDict.restype = ctypes.c_void_p
    R.ZSTD_createCDict.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.c_int]
    R.ZSTD_freeCDict.argtypes = [ctypes.c_void_p]
    out = []
    for d in dicts:
        ours = L.ZSTD_createCDict(d, len(d), 1)
        L.ZSTD_freeCDict(ours)
        ref = R.ZSTD_createCDict(d, len(d), 1)
        R.ZSTD_freeCDict(ref)
        out.append((bool(ours), _oracle_load(d) < (1 << 63), bool(ref)))
    return out


def _mutants(d, n, seed):
    """n byte flips, bit flips and truncations across the entropy header (everything in front of the content) of d"""
    end = _oracle_load(d)
    assert 8 < end < len(d)
    rng = random.Random(seed)
    out = []
    for _ in range(n):
        b = bytearray(d)
        kind = rng.random()
        if kind < 0.15:
            out.append(bytes(b[:rng.randrange(8, end + 16)]))
            continue
        for _ in range(2 if kind > 0.85 else 1):
            p = rng.randrange(8, end)
            b[p] ^= (1 << rng.randrange(8)) if kind < 0.4 else rng.randrange(1, 256)
        out.append(bytes(b))
    return out


def corrupted_dictionaries():
    """the seeded corpus: 2500 mutants of each of the three golden zstd-format dictionaries and of a trained one"""
    train = zref.train_dict(zref.synthetic(1024 * 2000, 11), 1024, 2000, 8 << 10)
    dicts = [zref.golden_input(n) for n in ("zdict-16k-synthetic-seed77", "http-dict-missing-symbols", "zero-weight-dict")] + [train]
    return [_mutants(d, 2500, k) for k, d in enumerate(dicts)]


@needs_ref
def test_corrupted_dictionaries_refused_as_the_reference_refuses():
    """the product's ZSTD_createCDict (which reads the format with the decoder's code, zb_decode_core.cuh) and the oracle
    refuse exactly the zstd-format dictionaries the reference's ZSTD_createCDict refuses"""
    for k, corpus in enumerate(corrupted_dictionaries()):
        got = _cdict_decisions(corpus)
        differ = [(i, g) for i, g in enumerate(got) if len(set(g)) > 1]
        assert not differ, (k, len(differ), [(corpus[i][:40].hex(), g) for i, g in differ[:5]])
        accepted = sum(g[0] for g in got)
        assert 100 < accepted < len(corpus) - 100, (k, accepted)


def _fse_description(norm, table_log):
    """FSE table description of normalised counts, written by the reference's FSE_writeNCount"""
    R = zref.ref()
    R.FSE_writeNCount.restype = ctypes.c_size_t
    R.FSE_writeNCount.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_uint, ctypes.c_uint]
    n = (ctypes.c_short * len(norm))(*norm)
    buf = ctypes.create_string_buffer(512)
    r = R.FSE_writeNCount(buf, 512, n, len(norm) - 1, table_log)
    assert not R.ZSTD_isError(r)
    return buf.raw[:r]


def _weights4(weights):
    """Huffman tree description with 4-bit weights"""
    w = list(weights) + [0]
    return bytes([127 + len(weights)]) + bytes(w[i] << 4 | w[i + 1] for i in range(0, len(weights), 2))


def _weightsFse(last_symbol, stream):
    """Huffman tree description with FSE-compressed weights: 32 states, symbol 1 in all but the top one, which belongs to
    last_symbol.  State 0 is the only one that reads a bit, so the stream of bytes 00 04 (initial states 0 and 0, then that
    bit) decodes to the weights 1, 1 (and the implied last weight 2)."""
    norm = [0, 31] + [0] * (last_symbol - 2) + [-1]
    nc = _fse_description(norm, 5)
    return bytes([len(nc) + len(stream)]) + nc + stream


@needs_ref
@pytest.mark.parametrize("row", [1, 2, 3, 4])
def test_rules_where_compressor_and_decoder_differ(H, row):  # noqa: F811
    """one hand-built dictionary per rule where the compressor's and the decoder's readers of a dictionary's Huffman tree
    description differ (both read it with zbd_readHufWeights, with their own limits); the tables behind it are those of a
    golden dictionary.  Accepted by the compressor, the oracle and the reference alike:
      1: weights and table log of 12 (HUF_TABLELOG_MAX); the decoder's tables stop at 11: it refuses.
      2: the weights' FSE description gives a probability to symbol 13, which no decoded weight uses.  The reference reads
         these descriptions over 256 symbols, the decoder over 13: it refuses.
    Refused by the compressor, the oracle and the reference alike:
      3: a weight bitstream shorter than its two initial states (fse_decompress.c:193); the decoder refuses it too.
      4: no weight of 1 (HUF_readStats: rank[1] >= 2); the decoder does not check, and accepts."""
    g = zref.golden_input("zdict-16k-synthetic-seed77")
    huf = {1: _weights4(range(12, 0, -1)), 2: _weightsFse(13, b"\x00\x04"), 3: _weightsFse(2, b"\x01"), 4: _weights4([2, 2, 2])}[row]
    d = g[:8] + huf + g[8 + _huf_desc_len(g):]
    [(ours, oracle, ref)] = _cdict_decisions([d])
    assert ours == oracle == ref == (row in (1, 2))
    assert dec(H, zref.ref_compress(b"", 1), 0, d) == (b"" if row == 4 else ("ERR", 30))
