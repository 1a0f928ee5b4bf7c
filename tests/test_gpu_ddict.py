"""GPU decompression with digested dictionaries (pytest -m gpu): ZSTD_decompress_usingDDict, the context's sticky dictionary
(ZSTD_DCtx_refDDict / loadDictionary / refPrefix) through ZSTD_decompressDCtx, ZSTD_decompressStream and
ZSTDB200_decompressDevice, and ZSTD_d_windowLogMax, each held to the compiled reference decoder's output and verdict."""
import ctypes
import os
import shutil
import subprocess
import threading

import pytest

import seqgen
import test_decode_invalid
import zref
import zstd_b200

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900, method="thread"),
              pytest.mark.skipif(not zref.have_ref(), reason="reference library not built")]
_sz, _vp = ctypes.c_size_t, ctypes.c_void_p
ZDICT = "zdict-16k-synthetic-seed77"
EXAMPLE = os.path.join(zref.ROOT, "oracle", "_ref", "examples", "dictionary_decompression.o")


def _bind(L):
    """the decoder API of library L (the product or the reference) with pointer arguments"""
    for f, res, args in (("ZSTD_createDCtx", _vp, []), ("ZSTD_freeDCtx", _sz, [_vp]), ("ZSTD_createDDict", _vp, [_vp, _sz]),
                         ("ZSTD_freeDDict", _sz, [_vp]), ("ZSTD_decompressDCtx", _sz, [_vp, _vp, _sz, _vp, _sz]),
                         ("ZSTD_decompress_usingDict", _sz, [_vp, _vp, _sz, _vp, _sz, _vp, _sz]),
                         ("ZSTD_decompress_usingDDict", _sz, [_vp, _vp, _sz, _vp, _sz, _vp]),
                         ("ZSTD_DCtx_setParameter", _sz, [_vp, ctypes.c_int, ctypes.c_int]), ("ZSTD_DCtx_reset", _sz, [_vp, ctypes.c_int]),
                         ("ZSTD_DCtx_loadDictionary", _sz, [_vp, _vp, _sz]), ("ZSTD_DCtx_refDDict", _sz, [_vp, _vp]),
                         ("ZSTD_DCtx_refPrefix", _sz, [_vp, _vp, _sz]), ("ZSTD_initDStream", _sz, [_vp]),
                         ("ZSTD_decompressStream", _sz, [_vp, ctypes.POINTER(seqgen.OutBuffer), ctypes.POINTER(seqgen.InBuffer)]),
                         ("ZSTD_getErrorCode", ctypes.c_int, [_sz])):
        getattr(L, f).restype = res
        getattr(L, f).argtypes = args
    return L


@pytest.fixture(scope="module")
def libs():
    return _bind(zstd_b200.lib()), _bind(seqgen.ref())


@pytest.fixture(scope="module")
def cctx():
    c = zstd_b200.ZSTD_CCtx()
    yield c
    c.close()


def _res(L, r, out):
    return ("ERR", L.ZSTD_getErrorCode(r)) if L.ZSTD_isError(r) else out.raw[:r]


def call(L, f, ctx, buf, cap, *extra):
    """one-shot call f of library L into a buffer of cap bytes: the output, or ("ERR", code)"""
    out = ctypes.create_string_buffer(max(cap, 1))
    return _res(L, getattr(L, f)(ctx, out, cap, buf, len(buf), *extra), out)


def feed(L, zds, buf, piece, room):
    """ZSTD_decompressStream over buf in `piece`-byte pieces through a `room`-byte output buffer: the output, ("ERR", code),
    or ("INCOMPLETE", None) when the input ends inside a frame"""
    src = ctypes.create_string_buffer(buf, max(len(buf), 1))
    base = ctypes.cast(src, ctypes.c_void_p).value
    out = ctypes.create_string_buffer(room)
    got, pos, last = bytearray(), 0, 0
    while pos < len(buf):
        i = seqgen.InBuffer(base + pos, min(piece, len(buf) - pos), 0)
        while True:
            o = seqgen.OutBuffer(ctypes.cast(out, ctypes.c_void_p), room, 0)
            last = L.ZSTD_decompressStream(zds, ctypes.byref(o), ctypes.byref(i))
            if L.ZSTD_isError(last):
                return ("ERR", L.ZSTD_getErrorCode(last))
            got += out.raw[:o.pos]
            if i.pos == i.size and o.pos < room:
                break
        pos += i.size
    return bytes(got) if last == 0 else ("INCOMPLETE", None)


def _dict(kind):
    return zref.golden_input(ZDICT) if kind == "zdict" else zref.synthetic(20_000, 5, 0.5)


def _matrix(cctx, d):
    """(frames, content): the matrix of test_gpu_decode.py::test_dictionaries"""
    out = []
    for n in (0, 1, 100, 1000, 5000, 200_000):
        src = zref.synthetic(n, 31, 0.5) if n else b""
        out += [(zref.ref_compress_using_dict(src, d, level), src) for level in (1, 3, -3, 6, 19)]
        out += [(cctx.compress_using_dict(src, d, level), src) for level in (1, 3)]
    recs = [zref.synthetic(1024, 100 + i, 0.5) for i in range(300)]
    out.append((b"".join(zref.ref_compress_using_dict(r, d, 1) for r in recs), b"".join(recs)))
    return out


@pytest.mark.parametrize("kind", ["zdict", "raw"])
def test_every_dictionary_path_gives_the_reference_output(libs, cctx, kind):
    """usingDDict; refDDict, then decompressDCtx; loadDictionary, then decompressDCtx; a sticky DDict with
    ZSTDB200_decompressDevice on the context's stream and on a caller's stream"""
    import torch
    L, R = libs
    d = _dict(kind)
    dd = L.ZSTD_createDDict(d, len(d))
    a, b, c = L.ZSTD_createDCtx(), L.ZSTD_createDCtx(), L.ZSTD_createDCtx()
    assert L.ZSTD_DCtx_refDDict(b, dd) == 0 and L.ZSTD_DCtx_loadDictionary(c, d, len(d)) == 0
    side = torch.cuda.Stream()
    for frames, src in _matrix(cctx, d):
        n = len(src)
        want = zref.ref_decompress_using_dict(frames, d, n)
        assert want == src
        assert call(L, "ZSTD_decompress_usingDDict", a, frames, n, dd) == want
        assert call(L, "ZSTD_decompressDCtx", b, frames, n) == want
        assert call(L, "ZSTD_decompressDCtx", c, frames, n) == want
        d_in = torch.frombuffer(bytearray(frames), dtype=torch.uint8).cuda()
        for stream in (None, side.cuda_stream):
            d_out = torch.zeros(n + 1, dtype=torch.uint8, device="cuda")
            torch.cuda.synchronize()
            r = L.ZSTDB200_decompressDevice(b, d_out.data_ptr(), n, d_in.data_ptr(), len(frames), stream)
            torch.cuda.synchronize()
            assert r == n and bytes(d_out[:n].cpu().numpy()) == want, (n, stream)
    for ctx in (a, b, c):
        assert L.ZSTD_freeDCtx(ctx) == 0
    assert L.ZSTD_freeDDict(dd) == 0


def test_verdicts_of_the_sticky_dictionary(libs, cctx):
    """a wrong dictID; a prefix used once, then a call without it; reset(session_only) keeps the dictionary,
    reset(parameters) drops it; ZSTD_initDStream drops it"""
    L, R = libs
    zd, raw = _dict("zdict"), _dict("raw")
    src = zd[-6000:] + raw[-6000:] + zref.synthetic(40_000, 9, 0.6)          # both frames copy from their dictionary's content
    fz, fr = zref.ref_compress_using_dict(src, zd, 3), zref.ref_compress_using_dict(src, raw, 3)
    other = bytearray(zd); other[4] ^= 1; other = bytes(other)
    ctx = {lib: lib.ZSTD_createDCtx() for lib in (L, R)}
    ddo = {lib: lib.ZSTD_createDDict(other, len(other)) for lib in (L, R)}

    def verdicts(res):
        """outputs and return values as they are, a refusal as "refused": without a dictionary the reference answers a frame
        that names one with dictionary_wrong, this decoder with the error its tables meet"""
        return [r if not isinstance(r, tuple) else "refused" for r in res]

    def both(steps):
        got = []
        for lib in (L, R):
            x = ctx[lib]
            res = []
            for f, *args in steps:
                if f == "dec":
                    res.append(call(lib, "ZSTD_decompressDCtx", x, args[0], len(src)))
                elif f == "ddict":
                    res.append(call(lib, "ZSTD_decompress_usingDDict", x, args[0], len(src), ddo[lib]))
                else:
                    res.append(getattr(lib, f)(x, *args))
            got.append(res)
        assert verdicts(got[0]) == verdicts(got[1]), steps
        return got[0]
    assert both([("ddict", fz)]) == [("ERR", 32)] == [call(R, "ZSTD_decompress_usingDDict", ctx[R], fz, len(src), ddo[R])]
    res = both([("ZSTD_DCtx_refDDict", None), ("ZSTD_DCtx_refPrefix", raw, len(raw)), ("dec", fr), ("dec", fr)])
    assert res[2] == src and res[3] != src
    for directive, kept in ((1, True), (2, False), (3, False)):
        res = both([("ZSTD_DCtx_loadDictionary", zd, len(zd)), ("ZSTD_DCtx_reset", directive), ("dec", fz)])
        assert (res[2] == src) == kept, directive
    res = both([("ZSTD_DCtx_loadDictionary", zd, len(zd)), ("ZSTD_initDStream",), ("dec", fz)])
    assert res[2] != src
    for lib in (L, R):
        lib.ZSTD_freeDCtx(ctx[lib]); lib.ZSTD_freeDDict(ddo[lib])


@pytest.mark.parametrize("how", ["load", "ddict"])
def test_streaming_with_a_dictionary(libs, cctx, how):
    """the piecewise feed of test_gpu_decode.py::test_streaming_decompression, with a loaded dictionary and with a DDict"""
    L, R = libs
    d = _dict("zdict")
    a, b = zref.synthetic(300_000, 41, 0.5), zref.synthetic(70_001, 42, 0.7)
    stream = cctx.compress_using_dict(a, d, 1) + zref.ref_compress_using_dict(b, d, 5) + cctx.compress_using_dict(b"", d, 1)
    zds = L.ZSTD_createDCtx()
    dd = L.ZSTD_createDDict(d, len(d))
    assert L.ZSTD_initDStream(zds) == 5
    assert (L.ZSTD_DCtx_loadDictionary(zds, d, len(d)) if how == "load" else L.ZSTD_DCtx_refDDict(zds, dd)) == 0
    out = bytearray()
    pos = 0
    for piece in (1, 7, 100, 50_000, 3, len(stream)):
        chunk = stream[pos:pos + piece]; pos += len(chunk)
        got = feed(L, zds, chunk, len(chunk), 10_000)
        assert not (isinstance(got, tuple) and got[0] == "ERR"), got
        out += got if not isinstance(got, tuple) else b""
    # the last piece ends every frame: what was held back comes out with it
    assert bytes(out) == a + b
    L.ZSTD_freeDCtx(zds); L.ZSTD_freeDDict(dd)


def test_window_log_max(libs):
    """ZSTD_d_windowLogMax 10 .. 27 against frames written with ZSTD_c_windowLog 10 .. 27 (streamed, no content size) and
    single-segment frames: ZSTD_decompressStream's verdict in pieces and in one call equals the reference's; the one-shot
    calls ignore the limit"""
    L, R = libs
    src = zref.synthetic(300_000, 8, 0.6)
    frames = [(f"wlog{w}", seqgen.ref_compress2(src, [(seqgen.C_WINDOWLOG, w), (seqgen.C_LEVEL, 3)], stream=True), src) for w in range(10, 28)]
    frames += [(f"wlog{w}-sized", seqgen.ref_compress2(src, [(seqgen.C_WINDOWLOG, w), (seqgen.C_LEVEL, 1)]), src) for w in (10, 14, 17, 19)]
    frames += [(f"single-{n}", zref.ref_compress(zref.synthetic(n, 3), 3), zref.synthetic(n, 3)) for n in (500, 1500, 40_000, 100_000, 300_000)]
    refused = 0
    for limit in range(10, 28):
        ctx = {lib: lib.ZSTD_createDCtx() for lib in (L, R)}
        for lib in (L, R):
            assert lib.ZSTD_DCtx_setParameter(ctx[lib], 100, limit) == 0
        for name, f, s in frames:
            for piece, room in ((4093, 1 << 17), (len(f), len(s) + 64)):
                got = []
                for lib in (L, R):
                    assert lib.ZSTD_DCtx_reset(ctx[lib], 1) == 0
                    got.append(feed(lib, ctx[lib], f, piece, room))
                assert got[0] == got[1], (name, limit, piece, got[0] if isinstance(got[0], tuple) else "data", got[1] if isinstance(got[1], tuple) else "data")
                refused += isinstance(got[0], tuple)
                assert got[0] == s or got[0] == ("ERR", 16)
            assert call(L, "ZSTD_decompressDCtx", ctx[L], f, len(s)) == s
            assert call(L, "ZSTD_decompress_usingDDict", ctx[L], f, len(s), None) == s
        for lib in (L, R):
            lib.ZSTD_freeDCtx(ctx[lib])
    assert refused > 100


def test_stage_wrong_inside_a_frame(libs):
    """setting a parameter or a dictionary while a stream is inside a frame: stage_wrong (60) from both; at the frame's end
    both accept again"""
    L, R = libs
    d = _dict("zdict")
    src = zref.synthetic(100_000, 12, 0.6)
    f = zref.ref_compress_using_dict(src, d, 3)
    for lib in (L, R):
        x = lib.ZSTD_createDCtx()
        assert lib.ZSTD_DCtx_loadDictionary(x, d, len(d)) == 0
        assert feed(lib, x, f[:len(f) // 2], 1000, 1 << 17) == ("INCOMPLETE", None)
        codes = [lib.ZSTD_DCtx_setParameter(x, 100, 20), lib.ZSTD_DCtx_loadDictionary(x, d, len(d)), lib.ZSTD_DCtx_refDDict(x, None),
                 lib.ZSTD_DCtx_refPrefix(x, d, len(d)), lib.ZSTD_DCtx_reset(x, 2)]
        assert [lib.ZSTD_getErrorCode(c) for c in codes] == [60] * 5, lib
        assert not isinstance(feed(lib, x, f[len(f) // 2:], 1000, 1 << 17), tuple), lib   # the frame ends: stage init again
        assert lib.ZSTD_DCtx_setParameter(x, 100, 20) == 0 and lib.ZSTD_DCtx_reset(x, 2) == 0
        lib.ZSTD_freeDCtx(x)


def test_one_ddict_four_threads(cctx):
    """one DDict used by four contexts on four threads at once (the first use uploads it under its lock); freeing it after
    the contexts is clean"""
    d = _dict("zdict")
    dd = zstd_b200.ZSTD_DDict(d)
    recs = [zref.synthetic(3000 + 500 * i, 200 + i, 0.5) for i in range(8)]
    frames = [zref.ref_compress_using_dict(r, d, 3) for r in recs]
    errors = []

    def work(k):
        try:
            x = zstd_b200.ZSTD_DCtx()
            if k % 2:
                x.ref_ddict(dd)
            for rnd in range(10):
                for f, r in zip(frames, recs):
                    got = x.decompress(f, len(r)) if k % 2 else x.decompress_using_ddict(f, dd)
                    if got != r:
                        errors.append((k, rnd))
            x.close()
        except Exception as e:                                      # reported by the main thread
            errors.append((k, repr(e)))
    threads = [threading.Thread(target=work, args=(k,)) for k in range(4)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors[:5]
    dd.close()


def test_ddict_on_a_second_device(cctx):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU")
    d = _dict("zdict")
    f = zref.ref_compress_using_dict(b"x" * 5000, d, 3)
    dd = zstd_b200.ZSTD_DDict(d)
    assert zstd_b200.ZSTD_DCtx(device=0).decompress_using_ddict(f, dd) == b"x" * 5000
    with pytest.raises(zstd_b200.ZstdError) as e:
        zstd_b200.ZSTD_DCtx(device=1).decompress_using_ddict(f, dd)
    assert e.value.code == 40
    zstd_b200.lib().ZSTDB200_setDevice(0)


def test_corpus_through_a_ddict(libs):
    """the seeded corrupted-frame corpus of test_decode_invalid.py with a raw dictionary: a DDict of it gives the verdict
    ZSTD_decompress_usingDict gives with the same bytes"""
    L, R = libs
    raw = _dict("raw")
    dd = L.ZSTD_createDDict(raw, len(raw))
    x = L.ZSTD_createDCtx()
    kinds = set()
    for name, buf, cap, _ in test_decode_invalid.corpus(test_decode_invalid.CORPUS_GPU, 1):
        want = call(L, "ZSTD_decompress_usingDict", x, buf, cap, raw, len(raw))
        assert call(L, "ZSTD_decompress_usingDDict", x, buf, cap, dd) == want, name
        kinds.add(want[0] if isinstance(want, tuple) else "ok")
    assert kinds == {"ok", "ERR"}
    L.ZSTD_freeDCtx(x); L.ZSTD_freeDDict(dd)


def test_reference_example_decodes_a_frame_of_this_library(cctx, tmp_path):
    """examples/dictionary_decompression.c, compiled unmodified and linked against this library alone, decodes a frame this
    library wrote with a dictionary"""
    if not os.path.exists(EXAMPLE) or not shutil.which("gcc"):
        pytest.skip("reference example object (or gcc) absent")
    libdir = os.path.join(zref.ROOT, "zstd_b200")
    exe = tmp_path / "dictionary_decompression"
    subprocess.check_call(["gcc", EXAMPLE, "-o", str(exe), "-L", libdir, "-lzstd_b200", "-Wl,-rpath," + libdir,
                           "-L/usr/local/cuda/lib64", "-Wl,-rpath,/usr/local/cuda/lib64"])
    d = _dict("zdict")
    (tmp_path / "dict").write_bytes(d)
    (tmp_path / "a.zst").write_bytes(cctx.compress_using_dict(zref.synthetic(200_000, 77, 0.5), d, 1))
    (tmp_path / "b.zst").write_bytes(cctx.compress_using_dict(zref.synthetic(3000, 78, 0.5), d, 3))
    p = subprocess.run([str(exe), str(tmp_path / "a.zst"), str(tmp_path / "b.zst"), str(tmp_path / "dict")],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
    assert p.returncode == 0, p.stdout
    assert "All 2 files correctly decoded" in p.stdout
