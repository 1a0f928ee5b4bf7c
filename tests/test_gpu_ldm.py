"""Long-distance matching on the GPU (zb_ldm.cu + the K1c overlay): byte for byte the oracle's frames (oracle/zb_ldm.c)
through every call that honours ZSTD_c_enableLongDistanceMatching, waves that copy across their edges, and the calls
that refuse or ignore it."""
import ctypes

import pytest

import ldmref
import zref
import zstd_b200

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not zref.have_ref(), reason="oracle/_ref/libzstd_ref.so not built")


@pytest.fixture(scope="module")
def inputs():
    return ldmref.inputs()


def _ctx(level, **ldm):
    c = zstd_b200.ZSTD_CCtx()
    c.set_parameter("compression_level", level)
    c.set_parameter("enable_long_distance_matching", 1)
    for k, v in ldm.items():
        c.set_parameter({"hash_log": 161, "min_match": 162, "bucket_size_log": 163, "hash_rate_log": 164}[k], v)
    return c


def _check_frame(frame, src):
    if zref.have_ref():
        assert zref.ref_decompress(frame, len(src)) == src
    assert zstd_b200.ZSTD_DCtx().decompress(frame, len(src)) == src


def _device(c, src, level, stream=None):
    d_src = torch.frombuffer(bytearray(src), dtype=torch.uint8).cuda()
    cap = zstd_b200.ZSTD_compressBound(len(src)) + 64
    d_dst = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    r = c.compress_device(d_dst.data_ptr(), cap, d_src.data_ptr(), len(src), level, stream.cuda_stream if stream is not None else 0)
    torch.cuda.synchronize()
    return d_dst[:r].cpu().numpy().tobytes()


class _In(ctypes.Structure):
    _fields_ = [("src", ctypes.c_void_p), ("size", ctypes.c_size_t), ("pos", ctypes.c_size_t)]


class _Out(ctypes.Structure):
    _fields_ = [("dst", ctypes.c_void_p), ("size", ctypes.c_size_t), ("pos", ctypes.c_size_t)]


def _stream_one_shot(c, src):
    cap = zstd_b200.ZSTD_compressBound(len(src))
    sbuf = ctypes.create_string_buffer(src, len(src))
    dbuf = ctypes.create_string_buffer(cap)
    i, o = _In(ctypes.addressof(sbuf), len(src), 0), _Out(ctypes.addressof(dbuf), cap, 0)
    r = zstd_b200.lib().ZSTD_compressStream2(c._h, ctypes.byref(o), ctypes.byref(i), 2)
    assert r == 0 and i.pos == len(src)
    return dbuf.raw[:o.pos]


@pytest.mark.parametrize("name", ["aba", "versions", "zeros", "random", "period4k"])
@pytest.mark.parametrize("level", [1, 3, -3])
def test_gpu_ldm_equals_oracle(inputs, name, level):
    src = inputs[name]
    want = ldmref.oracle_ldm(src, level)
    c = _ctx(level)
    got = c.compress2(src)
    assert got == want
    assert _stream_one_shot(_ctx(level), src) == want
    assert _device(_ctx(level), src, level) == want
    _check_frame(got, src)


@pytest.mark.parametrize("corner", ldmref.CORNERS, ids=lambda c: ",".join(f"{k}={v}" for k, v in c.items()))
def test_gpu_ldm_parameter_corners(inputs, corner):
    for name in ("aba", "period4k"):
        src = inputs[name]
        got = _ctx(1, **corner).compress2(src)
        assert got == ldmref.oracle_ldm(src, 1, **corner)
        _check_frame(got, src)


def test_gpu_ldm_frames_mixed_sizes(inputs):
    """ZSTDB200_compressFrames: the large frames get LDM, the frames of at most 512 KiB are the LDM-off frames"""
    parts = [inputs["aba"], zref.synthetic(100_000, seed=41), inputs["versions"], zref.synthetic(512 << 10, seed=42), zref.synthetic(600 << 10, seed=43)]
    src = b"".join(parts)
    offs, o = [], 0
    for p in parts:
        offs.append(o)
        o += len(p)
    for device_memory in (True, False):
        c = _ctx(3)
        cap = sum(zstd_b200.ZSTD_compressBound(len(p)) + 64 for p in parts)
        if device_memory:
            d_src = torch.frombuffer(bytearray(src), dtype=torch.uint8).cuda()
            d_dst = torch.zeros(cap, dtype=torch.uint8, device="cuda")
            torch.cuda.synchronize()
            total, sizes = c.compress_frames(d_dst.data_ptr(), cap, d_src.data_ptr(), offs, [len(p) for p in parts], 3, True)
            out = d_dst[:total].cpu().numpy().tobytes()
        else:
            sbuf = ctypes.create_string_buffer(src, len(src))
            dbuf = ctypes.create_string_buffer(cap)
            total, sizes = c.compress_frames(ctypes.addressof(dbuf), cap, ctypes.addressof(sbuf), offs, [len(p) for p in parts], 3, False)
            out = dbuf.raw[:total]
        pos = 0
        for p, s in zip(parts, sizes):
            want = ldmref.oracle_ldm(p, 3) if len(p) > (512 << 10) else zref.oracle_compress(p, 3)
            assert out[pos:pos + s] == want
            pos += s


def test_gpu_ldm_waves():
    """320 MiB with copies across the 128 MiB wave edges: the multi-wave device call, the one-wave call (a caller stream)
    and the host-buffer call give the same bytes, and the frame decodes"""
    piece = 8 << 20
    a = zref.random_bytes(piece, seed=51)
    body = bytearray(zref.synthetic(320 << 20, seed=52, match_prob=0.3))
    for at in (120 << 20, 250 << 20, 300 << 20):             # copies of `a` on both sides of the wave edges at 128 and 256 MiB
        body[at:at + piece] = a
    body[4 << 20:4 << 20 | piece] = a
    src = bytes(body)
    c = _ctx(1)
    multi = _device(c, src, 1)
    s = torch.cuda.Stream()
    single = _device(_ctx(1), src, 1, stream=s)
    assert multi == single
    host = _ctx(1).compress2(src)
    assert host == multi
    assert len(multi) < len(zstd_b200.ZSTD_CCtx().compress(src, 1)) - 3 * piece // 2
    _check_frame(multi, src)


def test_gpu_ldm_frame_part_refused():
    c = _ctx(1)
    d = torch.zeros(2 << 20, dtype=torch.uint8, device="cuda")
    with pytest.raises(zstd_b200.ZstdError) as e:
        c.compress_frame_part(d.data_ptr() + (1 << 20), 1 << 20, d.data_ptr(), 1 << 20, 0, 1 << 20, 1)
    assert e.value.code == 40


def test_gpu_ldm_reset_and_simple_api(inputs):
    src = inputs["aba"]
    c = _ctx(1)
    assert c.compress2(src) == ldmref.oracle_ldm(src, 1)
    assert c.compress(src, 1) == zref.oracle_compress(src, 1)          # the simple API ignores sticky parameters
    c.reset(2)
    c.set_parameter("compression_level", 1)
    assert c.compress2(src) == zref.oracle_compress(src, 1)
    c.set_parameter("enable_long_distance_matching", 2)
    assert c.compress2(src) == zref.oracle_compress(src, 1)
