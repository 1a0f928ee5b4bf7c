"""The decoder's dictionary API without a GPU: ZSTD_createDDict / ZSTD_getDictID_fromDDict / ZSTD_getDictID_fromFrame and the
return codes of the context's sticky dictionary and parameter calls, each against the compiled reference's.  None of these
calls touches the device."""
import ctypes
import glob
import os
import shutil
import subprocess

import pytest

import test_oracle_dict
import zref
import zstd_b200

needs_ref = pytest.mark.skipif(not zref.have_ref(), reason="reference library not built")
_sz, _vp = ctypes.c_size_t, ctypes.c_void_p
ZDICT = "zdict-16k-synthetic-seed77"
EXAMPLE = os.path.join(zref.ROOT, "oracle", "_ref", "examples", "dictionary_decompression.o")


def _ref():
    R = zref.ref()
    R.ZSTD_createDDict.restype = _vp
    R.ZSTD_createDDict.argtypes = [_vp, _sz]
    R.ZSTD_freeDDict.restype = _sz
    R.ZSTD_freeDDict.argtypes = [_vp]
    R.ZSTD_getDictID_fromDDict.restype = ctypes.c_uint
    R.ZSTD_getDictID_fromDDict.argtypes = [_vp]
    R.ZSTD_getDictID_fromFrame.restype = ctypes.c_uint
    R.ZSTD_getDictID_fromFrame.argtypes = [_vp, _sz]
    R.ZSTD_getDictID_fromDict.restype = ctypes.c_uint
    R.ZSTD_getDictID_fromDict.argtypes = [_vp, _sz]
    for f in ("ZSTD_DCtx_setParameter", "ZSTD_DCtx_reset", "ZSTD_DCtx_loadDictionary", "ZSTD_DCtx_refDDict", "ZSTD_DCtx_refPrefix"):
        getattr(R, f).restype = _sz
    R.ZSTD_DCtx_setParameter.argtypes = [_vp, ctypes.c_int, ctypes.c_int]
    R.ZSTD_DCtx_reset.argtypes = [_vp, ctypes.c_int]
    R.ZSTD_DCtx_loadDictionary.argtypes = [_vp, _vp, _sz]
    R.ZSTD_DCtx_refDDict.argtypes = [_vp, _vp]
    R.ZSTD_DCtx_refPrefix.argtypes = [_vp, _vp, _sz]
    R.ZSTD_getErrorCode.restype = ctypes.c_int
    R.ZSTD_getErrorCode.argtypes = [_sz]
    return R


def _code(L, r):
    return L.ZSTD_getErrorCode(r) if L.ZSTD_isError(r) else r


def _dictionaries():
    return {"zdict": zref.golden_input(ZDICT), "zero-weight": zref.golden_input("zero-weight-dict"), "raw": zref.synthetic(20_000, 5, 0.5),
            "raw-7-bytes-with-magic": bytes.fromhex("37a430ec010203"), "empty": b""}


def _header(dict_bytes_len, dict_id, single=False, fcs=None):
    """a frame header naming dict_id in a dictID field of dict_bytes_len (0, 1, 2 or 4) bytes, then one empty raw block"""
    flag = {0: 0, 1: 1, 2: 2, 4: 3}[dict_bytes_len]
    fcs_bytes = b"" if fcs is None else bytes([fcs])
    fhd = flag | (0x20 if single else 0)
    out = (0xFD2FB528).to_bytes(4, "little") + bytes([fhd]) + (b"" if single else bytes([0x08]))
    out += dict_id.to_bytes(4, "little")[:dict_bytes_len] + fcs_bytes
    return out + bytes([1, 0, 0])                                   # last block, raw, 0 bytes


def test_reference_dictionary_decompression_example_links(tmp_path):
    """examples/dictionary_decompression.c (ZSTD_createDDict, ZSTD_getDictID_fromDDict, ZSTD_getDictID_fromFrame,
    ZSTD_decompress_usingDDict), compiled unmodified against the stock lib/zstd.h, links against this library alone"""
    if not os.path.exists(EXAMPLE):
        pytest.skip("reference example object not built")
    gcc = shutil.which("gcc")
    if not gcc:
        pytest.skip("no gcc")
    libdir = os.path.join(zref.ROOT, "zstd_b200")
    exe = tmp_path / "dictionary_decompression"
    subprocess.check_call([gcc, EXAMPLE, "-o", str(exe), "-L", libdir, "-lzstd_b200", "-Wl,-rpath," + libdir,
                           "-L/usr/local/cuda/lib64", "-Wl,-rpath,/usr/local/cuda/lib64"])
    assert exe.exists()


@needs_ref
def test_dict_id_from_frame_matches_reference():
    """golden frames, frames of both encoders with and without a dictionary, dictID fields of 1, 2 and 4 bytes, skippable
    frames, and every truncation of each header"""
    L, R = zstd_b200.lib(), _ref()
    zd = zref.golden_input(ZDICT)
    frames = [open(f, "rb").read() for f in sorted(glob.glob(os.path.join(zref.GOLDEN, "decompression*", "*.zst")))]
    src = zref.synthetic(5000, 3)
    frames += [zref.ref_compress(src, 3), zref.ref_compress_using_dict(src, zd, 3), zref.oracle_compress_using_dict(src, zd, 1)]
    for n, did in ((1, 0xAB), (2, 0xBEEF), (4, 0xDEADBEEF), (4, 0), (1, 0), (2, 7)):
        frames += [_header(n, did), _header(n, did, single=True, fcs=0)]
    frames += [bytes([0x50 + k, 0x2A, 0x4D, 0x18, 3, 0, 0, 0]) + b"abc" for k in range(16)]
    frames += [b"", b"\x28", b"\x00" * 20, (0xFD2FB528).to_bytes(4, "little") + b"\x08\x00"]     # not frames; a reserved bit
    named = 0
    for f in frames:
        for n in sorted(set(range(min(len(f), 20) + 1)) | {len(f)}):
            want = R.ZSTD_getDictID_fromFrame(f[:n], n)
            assert L.ZSTD_getDictID_fromFrame(f[:n], n) == want, (f[:20].hex(), n)
            named += want != 0
    assert named > 20


@needs_ref
def test_dict_id_from_ddict():
    """ZSTD_getDictID_fromDDict equals ZSTD_getDictID_fromDict (and the reference's DDict) for zstd-format and raw
    dictionaries; a DDict is created and queried without a GPU"""
    L, R = zstd_b200.lib(), _ref()
    for name, d in _dictionaries().items():
        dd, rd = L.ZSTD_createDDict(d, len(d)), R.ZSTD_createDDict(d, len(d))
        assert dd and rd, name
        assert L.ZSTD_getDictID_fromDDict(dd) == L.ZSTD_getDictID_fromDict(d, len(d)) == R.ZSTD_getDictID_fromDDict(rd), name
        assert (L.ZSTD_getDictID_fromDDict(dd) != 0) == (name in ("zdict", "zero-weight")), name
        assert L.ZSTD_freeDDict(dd) == 0 and R.ZSTD_freeDDict(rd) == 0
    assert L.ZSTD_freeDDict(None) == 0 and L.ZSTD_getDictID_fromDDict(None) == 0
    assert zstd_b200.ZSTD_DDict(zref.golden_input(ZDICT)).dict_id == L.ZSTD_getDictID_fromDict(zref.golden_input(ZDICT), 16384)


@needs_ref
def test_create_ddict_refuses_corrupted_dictionaries_as_the_reference_does():
    """the seeded corpus of corrupted dictionaries (test_oracle_dict): ZSTD_createDDict returns NULL where the reference's
    does.  Where they differ, the reference accepts a dictionary that the compressor's reader of the same format accepts
    too (it holds the reference's limits), and the decoder's limits of a Huffman tree description refuse it: a table log
    above 11, or a weight description with a probability for a symbol above 12 (DESIGN.md section 4)."""
    L, R = zstd_b200.lib(), _ref()
    L.ZSTD_createCDict.restype = _vp
    L.ZSTD_createCDict.argtypes = [_vp, _sz, ctypes.c_int]
    for k, corpus in enumerate(test_oracle_dict.corrupted_dictionaries()):
        accepted = 0
        for d in corpus:
            ours, ref = L.ZSTD_createDDict(d, len(d)), R.ZSTD_createDDict(d, len(d))
            L.ZSTD_freeDDict(ours); R.ZSTD_freeDDict(ref)
            accepted += bool(ref)
            if bool(ours) == bool(ref):
                continue
            cd = L.ZSTD_createCDict(d, len(d), 1)
            L.ZSTD_freeCDict(cd)
            assert ref and not ours and cd, (k, d[:40].hex())
        assert 100 < accepted < len(corpus) - 100, (k, accepted)
    # the documented limits: one hand-built dictionary each (test_oracle_dict rows 1 and 2), and a golden dictionary whose
    # Huffman description is beyond them
    g = zref.golden_input(ZDICT)
    limited = [g[:8] + huf + g[8 + test_oracle_dict._huf_desc_len(g):]
               for huf in (test_oracle_dict._weights4(range(12, 0, -1)), test_oracle_dict._weightsFse(13, b"\x00\x04"))]
    for d in limited + [zref.golden_input("http-dict-missing-symbols")]:
        rd, cd = R.ZSTD_createDDict(d, len(d)), L.ZSTD_createCDict(d, len(d), 1)
        assert rd and cd and not L.ZSTD_createDDict(d, len(d))
        R.ZSTD_freeDDict(rd); L.ZSTD_freeCDict(cd)


@needs_ref
def test_sticky_calls_return_the_reference_codes():
    """ZSTD_DCtx_setParameter, ZSTD_DCtx_reset, ZSTD_DCtx_loadDictionary, ZSTD_DCtx_refDDict and ZSTD_DCtx_refPrefix on a
    context outside a stream: the same return codes as the reference's"""
    L, R = zstd_b200.lib(), _ref()
    ours, ref = L.ZSTD_createDCtx(), R.ZSTD_createDCtx()
    zd = zref.golden_input(ZDICT)
    corrupted = zd[:8] + b"\xff" * 40 + zd[48:]
    assert not R.ZSTD_createDDict(corrupted, len(corrupted))

    def both(f, *args):
        a, b = getattr(L, f)(ours, *args), getattr(R, f)(ref, *args)
        assert _code(L, a) == _code(R, b), (f, args, _code(L, a), _code(R, b))
        return _code(L, a)
    for v in (-1, 0, 9, 10, 27, 31, 32, 1 << 20):
        both("ZSTD_DCtx_setParameter", 100, v)
    for p in (0, 1, 99, 101, 999, 4000, -5):
        assert both("ZSTD_DCtx_setParameter", p, 1) == 40
    for directive in (0, 1, 2, 3, 4):
        assert both("ZSTD_DCtx_reset", directive) == 0
    for name, d in list(_dictionaries().items()) + [("corrupted", corrupted)]:
        code = both("ZSTD_DCtx_loadDictionary", d or None, len(d))
        assert code == (64 if name == "corrupted" else 0), name
        assert both("ZSTD_DCtx_refPrefix", d or None, len(d)) == 0
    both("ZSTD_DCtx_loadDictionary", None, 0)
    both("ZSTD_DCtx_loadDictionary", zd, 0)
    dd, rd = L.ZSTD_createDDict(zd, len(zd)), R.ZSTD_createDDict(zd, len(zd))
    assert L.ZSTD_DCtx_refDDict(ours, dd) == 0 == R.ZSTD_DCtx_refDDict(ref, rd)
    assert both("ZSTD_DCtx_refDDict", None) == 0
    assert both("ZSTD_DCtx_reset", 2) == 0
    L.ZSTD_freeDCtx(ours); R.ZSTD_freeDCtx(ref)
    L.ZSTD_freeDDict(dd); R.ZSTD_freeDDict(rd)


def test_python_binding_without_gpu():
    """ZSTD_DDict and the ZSTD_DCtx methods that need no device"""
    d = zstd_b200.ZSTD_DDict(zref.golden_input(ZDICT))
    raw = zstd_b200.ZSTD_DDict(b"raw content of a dictionary")
    assert d.dict_id != 0 and raw.dict_id == 0
    c = zstd_b200.ZSTD_DCtx()
    c.set_parameter("window_log_max", 20)
    with pytest.raises(zstd_b200.ZstdError) as e:
        c.set_parameter("window_log_max", 9)
    assert e.value.code == 42
    with pytest.raises(zstd_b200.ZstdError) as e:
        c.set_parameter(1000, 1)
    assert e.value.code == 40
    c.load_dictionary(zref.golden_input(ZDICT))
    c.ref_ddict(d)
    c.ref_prefix(b"a prefix")
    c.ref_ddict(None)
    c.load_dictionary(None)
    with pytest.raises(zstd_b200.ZstdError) as e:
        zstd_b200.ZSTD_DDict(zref.golden_input(ZDICT)[:8] + b"\xff" * 64)
    assert e.value.code == 30
    for directive in (1, 2, 3):
        c.reset(directive)
    c.close(); d.close(); raw.close()
