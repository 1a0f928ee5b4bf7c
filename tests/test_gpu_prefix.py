"""Compression against a prefix on the GPU (ZSTD_CCtx_refPrefix / ZSTDB200_CCtx_refPrefixDevice, zb_ldm.cu's two segments):
byte for byte the oracle's frames (oracle/zb_prefix.c) through every call that honours a prefix, decoded again on the GPU and
by the reference with the same prefix, a frame of several waves, and the semantics of the entry points."""
import ctypes

import pytest

import ldmref
import prefixref
import zref
import zstd_b200

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pairs():
    return prefixref.pairs()


def _ctx(level, ldm=True, **prm):
    c = zstd_b200.ZSTD_CCtx()
    c.set_parameter("compression_level", level)
    if ldm:
        c.set_parameter("enable_long_distance_matching", 1)
    for k, v in prm.items():
        c.set_parameter({"hash_log": 161, "min_match": 162, "bucket_size_log": 163, "hash_rate_log": 164}[k], v)
    return c


def _dev(b):
    return torch.frombuffer(bytearray(b if b else b"\0"), dtype=torch.uint8).cuda()


def _device(c, src, level, prefix=None, device_prefix=True, stream=None):
    """compress_device of src; prefix: given to the context in device memory (device_prefix) or in host memory"""
    d_src = _dev(src)
    cap = zstd_b200.ZSTD_compressBound(len(src)) + 64
    d_dst = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    d_pfx = None
    if prefix is not None and device_prefix:
        d_pfx = _dev(prefix)
        c.ref_prefix_device(d_pfx.data_ptr(), len(prefix))
    elif prefix is not None:
        c.ref_prefix(prefix)
    torch.cuda.synchronize()
    r = c.compress_device(d_dst.data_ptr(), cap, d_src.data_ptr(), len(src), level, stream.cuda_stream if stream is not None else 0)
    torch.cuda.synchronize()
    return d_dst[:r].cpu().numpy().tobytes()


class _In(ctypes.Structure):
    _fields_ = [("src", ctypes.c_void_p), ("size", ctypes.c_size_t), ("pos", ctypes.c_size_t)]


class _Out(ctypes.Structure):
    _fields_ = [("dst", ctypes.c_void_p), ("size", ctypes.c_size_t), ("pos", ctypes.c_size_t)]


def _stream2(c, src, end_op=2, cap=None):
    cap = zstd_b200.ZSTD_compressBound(len(src)) if cap is None else cap
    sbuf = ctypes.create_string_buffer(src, max(len(src), 1))
    dbuf = ctypes.create_string_buffer(max(cap, 1))
    i, o = _In(ctypes.addressof(sbuf), len(src), 0), _Out(ctypes.addressof(dbuf), cap, 0)
    r = zstd_b200.lib().ZSTD_compressStream2(c._h, ctypes.byref(o), ctypes.byref(i), end_op)
    return r, dbuf.raw[:o.pos]


def _decode_device_using_dict(frame, prefix, size):
    L = zstd_b200.lib()
    L.ZSTDB200_decompressDevice_usingDict.restype = ctypes.c_size_t
    L.ZSTDB200_decompressDevice_usingDict.argtypes = [ctypes.c_void_p] * 2 + [ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t,
                                                      ctypes.c_void_p]
    d = zstd_b200.ZSTD_DCtx()
    d_frame = _dev(frame)
    d_out = torch.zeros(max(size, 1), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    pbuf = ctypes.create_string_buffer(prefix, len(prefix))
    r = zstd_b200._check(L.ZSTDB200_decompressDevice_usingDict(d._h, d_out.data_ptr(), size, d_frame.data_ptr(), len(frame), pbuf, len(prefix), None))
    torch.cuda.synchronize()
    return d_out[:r].cpu().numpy().tobytes()


def _check_frame(frame, prefix, src, raw_only=False):
    d = zstd_b200.ZSTD_DCtx()
    d.ref_prefix(prefix)
    assert d.decompress(frame, len(src)) == src
    if not raw_only:                                 # a prefix with the dictionary magic is raw content only through refPrefix
        assert _decode_device_using_dict(frame, prefix, len(src)) == src
    if zref.have_ref():
        assert prefixref.ref_decompress_prefix(frame, prefix, len(src)) == src


NAMES = ["edits", "shifted", "same", "unrelated", "prefix1", "prefix7", "prefix100k", "prefix_larger", "small_frame_ldm",
         "small_frame_no_ldm", "magic", "empty"]


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("level", [1, 3, -3])
def test_gpu_prefix_equals_oracle(pairs, name, level):
    prefix, src = pairs[name]
    want = prefixref.oracle_prefix(src, prefix, level)
    c = _ctx(level)
    c.ref_prefix(prefix)
    got = c.compress2(src)
    assert got == want
    c = _ctx(level)
    c.ref_prefix(prefix)
    r, streamed = _stream2(c, src)
    assert r == 0 and streamed == want
    assert _device(_ctx(level), src, level, prefix) == want                                   # device prefix, the context's streams
    assert _device(_ctx(level), src, level, prefix, stream=torch.cuda.Stream()) == want       # device prefix, a caller's stream
    assert _device(_ctx(level), src, level, prefix, device_prefix=False) == want              # host prefix, uploaded by the device call
    _check_frame(got, prefix, src, raw_only=name == "magic")


@pytest.mark.parametrize("name", ["edits", "prefix100k", "small_frame_no_ldm", "magic"])
def test_gpu_prefix_without_ldm_is_a_raw_dictionary(pairs, name):
    prefix, src = pairs[name]
    c = _ctx(1, ldm=False)
    c.ref_prefix(prefix)
    got = c.compress2(src)
    assert got == prefixref.oracle_prefix(src, prefix, 1, ldm=False)
    if name != "magic":
        assert got == zstd_b200.ZSTD_CCtx().compress_using_dict(src, prefix, 1)
    assert _device(_ctx(1, ldm=False), src, 1, prefix) == got
    _check_frame(got, prefix, src, raw_only=name == "magic")


@pytest.mark.parametrize("corner", ldmref.CORNERS, ids=lambda c: ",".join(f"{k}={v}" for k, v in c.items()))
def test_gpu_prefix_parameter_corners(pairs, corner):
    for name in ("shifted", "small_frame_ldm"):
        prefix, src = pairs[name]
        c = _ctx(1, **corner)
        c.ref_prefix(prefix)
        got = c.compress2(src)
        assert got == prefixref.oracle_prefix(src, prefix, 1, **corner)
        _check_frame(got, prefix, src)


def test_gpu_prefix_checksum_and_stats(pairs):
    prefix, src = pairs["edits"]
    c = _ctx(1)
    c.set_parameter("checksum_flag", 1)
    c.ref_prefix(prefix)
    got = c.compress2(src)
    want = prefixref.oracle_prefix(src, prefix, 1)
    assert got[:-4] == want[:4] + bytes([want[4] | 4]) + want[5:]          # Content_Checksum_flag
    assert int.from_bytes(got[-4:], "little") == zref.xxh64(src) & 0xFFFFFFFF
    assert c.stats().h2d_bytes == len(src) + len(prefix)          # the indexed prefix goes up with the input
    _check_frame(got, prefix, src)


def test_gpu_prefix_waves():
    """a 304 MiB frame against a 64 MiB prefix: the device call of several waves, the one-wave call on a caller's stream and
    the host-buffer call (48 MiB waves) give the same bytes.  Copies of the prefix's end lie across the host path's wave
    edge at 48 MiB and at 100 MiB; a piece of the prefix copied 200 MiB into the frame is out of the window's reach."""
    mib = 1 << 20
    prefix = zref.random_bytes(64 * mib, seed=61)
    a, far = prefix[56 * mib:], prefix[40 * mib:48 * mib]
    body = bytearray(zref.synthetic(304 * mib, seed=62, match_prob=0.3))
    body[44 * mib:52 * mib] = a
    body[100 * mib:108 * mib] = a[:4 * mib] + a[:4 * mib]
    body[200 * mib:208 * mib] = far
    src = bytes(body)
    del body
    multi = _device(_ctx(1), src, 1, prefix)
    single = _device(_ctx(1), src, 1, prefix, stream=torch.cuda.Stream())
    assert multi == single
    c = _ctx(1)
    c.ref_prefix(prefix)
    host = c.compress2(src)
    assert host == multi
    plain = _ctx(1).compress2(src)                   # LDM, no prefix: a is new at 44 MiB, then found in the frame; far is new
    assert len(multi) < len(plain) - 7 * mib
    assert len(multi) > 8 * mib                       # far is stored: nothing beyond the window takes from the prefix
    d = zstd_b200.ZSTD_DCtx()
    d.ref_prefix(prefix)
    assert d.decompress(multi, len(src)) == src
    if zref.have_ref():
        assert prefixref.ref_decompress_prefix(multi, prefix, len(src)) == src


def test_gpu_prefix_longer_than_the_window_indexes_its_tail():
    """a prefix of 2^27 + 1 MiB bytes: its first MiB is out of every block's reach and is not indexed"""
    mib = 1 << 20
    head = zref.random_bytes(mib, seed=71)
    prefix = head + zref.random_bytes(1 << 27, seed=72)
    src = head + prefix[-mib:] + zref.synthetic(mib, seed=73)
    got = _device(_ctx(1), src, 1, prefix)
    assert got == _device(_ctx(1), src, 1, prefix[mib:])          # the same frame as against the tail alone
    assert mib < len(got) < mib + (mib >> 1)                      # head is stored, the tail's last MiB is copied
    d = zstd_b200.ZSTD_DCtx()
    d.ref_prefix(prefix)
    assert d.decompress(got, len(src)) == src


def test_gpu_prefix_is_used_once_and_replaced_by_dictionaries(pairs):
    prefix, src = pairs["edits"]
    plain, with_prefix = ldmref.oracle_ldm(src, 1), prefixref.oracle_prefix(src, prefix, 1)
    c = _ctx(1)
    c.ref_prefix(prefix)
    assert c.compress2(src) == with_prefix
    assert c.compress2(src) == plain                                   # the next frame only
    c.ref_prefix(prefix)
    c.ref_prefix(None)                                                 # NULL clears
    assert c.compress2(src) == plain
    dict_bytes = zref.synthetic(64 << 10, seed=81)
    with_dict = None
    for setter in ("load", "cdict"):
        c = _ctx(1)
        c.ref_prefix(prefix)
        cd = zstd_b200.ZSTD_CDict(dict_bytes, 1)
        c.load_dictionary(dict_bytes) if setter == "load" else c.ref_cdict(cd)     # replaces the prefix
        got = c.compress2(src)
        with_dict = got if with_dict is None else with_dict
        assert got == with_dict and got != with_prefix and got != plain
        c.load_dictionary(None) if setter == "load" else c.ref_cdict(None)
        assert c.compress2(src) == plain                                 # clearing the dictionary does not bring the prefix back
        c.load_dictionary(dict_bytes) if setter == "load" else c.ref_cdict(cd)
        c.ref_prefix(prefix)                                             # replaces the dictionary, for good
        assert c.compress2(src) == with_prefix
        assert c.compress2(src) == plain
    c = _ctx(1)
    c.ref_prefix(prefix)
    c.reset(1)                                                         # session only: the prefix stays
    assert c.compress2(src) == with_prefix
    c.ref_prefix(prefix)
    c.reset(2)
    c.set_parameter("compression_level", 1)
    c.set_parameter("enable_long_distance_matching", 1)
    assert c.compress2(src) == plain


def test_gpu_prefix_simple_api_ignores_it(pairs):
    prefix, src = pairs["edits"]
    c = _ctx(1)
    c.ref_prefix(prefix)
    assert c.compress(src, 1) == zref.oracle_compress(src, 1)
    dict_bytes = zref.synthetic(64 << 10, seed=82)
    assert c.compress_using_dict(src, dict_bytes, 1) == zref.oracle_compress_using_dict(src, dict_bytes, 1)
    assert c.compress2(src) == prefixref.oracle_prefix(src, prefix, 1)          # still pending


def test_gpu_prefix_refused_where_it_has_no_meaning(pairs):
    prefix, src = pairs["edits"]
    src = src[:1 << 20]
    d_src, d_pfx = _dev(src), _dev(prefix)
    cap = zstd_b200.ZSTD_compressBound(len(src)) + 64
    d_dst = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    c = _ctx(1, ldm=False)
    c.ref_prefix(prefix)

    def refused(call):
        with pytest.raises(zstd_b200.ZstdError) as e:
            call()
        assert e.value.code == 40

    refused(lambda: c.compress_frames(d_dst.data_ptr(), cap, d_src.data_ptr(), [0], [len(src)], 1, True))
    refused(lambda: c.compress_frames_using_cdict(d_dst.data_ptr(), cap, d_src.data_ptr(), [0], [len(src)], zstd_b200.ZSTD_CDict(prefix[:1000], 1), True))
    refused(lambda: c.compress_frame_part(d_dst.data_ptr(), cap, d_src.data_ptr(), len(src), 0, len(src), 1))
    refused(lambda: c.compress_sequences([(0, len(src), 0)], src))
    refused(lambda: c.compress_sequences_device(d_dst.data_ptr(), cap, d_src.data_ptr(), 0, d_src.data_ptr(), len(src)))
    assert c.compress2(src) == prefixref.oracle_prefix(src, prefix, 1, ldm=False)      # the refused calls left it pending
    c.ref_prefix_device(d_pfx.data_ptr(), len(prefix))
    refused(lambda: c.compress2(src))                                                 # a device prefix needs a device call
    assert c.compress2(src) == zref.oracle_compress(src, 1)                            # and is forgotten by the call that refused it


def test_gpu_prefix_in_a_stream(pairs):
    """the first frame of a stream session takes the prefix; inside the session refPrefix is refused"""
    prefix, src = pairs["edits"]
    c = _ctx(1)
    c.ref_prefix(prefix)
    r, out = _stream2(c, src[:1 << 20], end_op=0, cap=0)              # ZSTD_e_continue: buffered
    assert out == b""
    with pytest.raises(zstd_b200.ZstdError) as e:
        c.ref_prefix(prefix)
    assert e.value.code == 60
    r, first = _stream2(c, src[1 << 20:], end_op=1, cap=zstd_b200.ZSTD_compressBound(len(src)))    # ZSTD_e_flush: the first frame
    assert r == 0 and first == prefixref.oracle_prefix(src, prefix, 1)
    r, second = _stream2(c, src, end_op=2)                             # the session's second frame has no prefix
    assert r == 0 and second == ldmref.oracle_ldm(src, 1)
    c.ref_prefix(prefix)                                               # the session is over
    assert c.compress2(src) == first
