"""Stream-ordered decompression (ZSTDB200_decompressDeviceAsync): the verdict and bytes of ZSTDB200_decompressDevice on
valid and invalid input, the workspace's block capacity, no host wait behind queued work, calls on one context in the order
they are made, CUDA graph capture and freeing a context with work in flight.  The first tests need no GPU."""
import ctypes
import struct

import pytest

import zref
import zstd_b200
from test_decode_invalid import CORPUS_GPU, GUARD, _lib, constructed, corpus, needs_ref
from test_gpu_async import SLEEP_CYCLES, ZDICT, _dev, _records, _torch, _u64

SKIP_MAGIC = 0x184D2A50


# ------------------------------------------------------------------ no GPU needed
def test_symbol_is_exported():
    assert hasattr(zstd_b200.lib(), "ZSTDB200_decompressDeviceAsync")


def _raw_call(d_result):
    L = zstd_b200.lib()
    d = L.ZSTD_createDCtx()
    try:
        return L.ZSTD_getErrorCode(L.ZSTDB200_decompressDeviceAsync(d, 4096, 100, 8192, 10, d_result, None))
    finally:
        L.ZSTD_freeDCtx(d)


@pytest.mark.skipif(zstd_b200.device_available(), reason="a CUDA device is present")
def test_without_a_device_returns_generic():
    assert _raw_call(16384) == 1


def test_null_result_returns_generic():
    assert _raw_call(None) == 1


# ------------------------------------------------------------------ GPU
gpu = pytest.mark.gpu


def _skippable(n):
    return struct.pack("<II", SKIP_MAGIC, n) + bytes(n)


def _async(dctx, d_src, n, cap, stream=None, d_dst=None, off=0):
    """enqueue decompress_device_async into d_dst[off:off + cap]; returns (d_dst, d_result) to read after a synchronise"""
    torch = _torch()
    d_dst = torch.zeros(cap + off + 16, dtype=torch.uint8, device="cuda") if d_dst is None else d_dst
    res = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    s = torch.cuda.current_stream() if stream is None else stream
    s.wait_stream(torch.cuda.current_stream())              # the buffers above are made on the current stream
    dctx.decompress_device_async(d_dst.data_ptr() + off, cap, d_src.data_ptr(), n, res.data_ptr(), s.cuda_stream)
    return d_dst, res


def _verdict(d_dst, res, off=0):
    r = _u64(res)
    e = zstd_b200.result_error(r)
    return ("ERR", e) if e is not None else bytes(d_dst[off:off + r].cpu().numpy())


def _sync(dctx, d_src, n, cap):
    torch = _torch()
    d_dst = torch.zeros(cap + 16, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    r = dctx.decompress_device(d_dst.data_ptr(), cap, d_src.data_ptr(), n)
    return bytes(d_dst[:r].cpu().numpy())


def _roundtrip(frames, content, cap=None, ddict=None):
    """frames decoded by the async call on a side stream and by decompress_device: both give content"""
    torch = _torch()
    cap = len(content) if cap is None else cap
    d_src = _dev(frames)
    a, s = zstd_b200.ZSTD_DCtx(), zstd_b200.ZSTD_DCtx()
    if ddict is not None:
        a.ref_ddict(ddict); s.ref_ddict(ddict)
    d_dst, res = _async(a, d_src, len(frames), cap, stream=torch.cuda.Stream())
    torch.cuda.synchronize()
    assert _verdict(d_dst, res) == content
    assert a.stats().launches > 0 and a.stats().kernel_ms == 0.0
    assert _sync(s, d_src, len(frames), cap) == content


@pytest.fixture(scope="module")
def big():
    return zref.random_bytes(600 << 20, seed=5)


@gpu
@pytest.mark.parametrize("level", [1, 3, -5])
@pytest.mark.parametrize("n", [0, 7, 5000, (128 << 10) + 1, 3 << 20, 600 << 20])
def test_same_bytes_as_decompress_device(n, level, big):
    if n == 600 << 20 and level != 1:
        pytest.skip("one incompressible frame over the 512 MiB walk threshold is enough")
    src = big if n == 600 << 20 else zref.synthetic(n, seed=n % 997, match_prob=0.6)
    frame = zstd_b200.ZSTD_CCtx().compress(src, level)
    if n == 600 << 20:
        assert len(frame) > 512 << 20                       # the synchronous call walks it with the kernel too
    _roundtrip(frame, src)


@gpu
def test_batch_with_a_ddict():
    torch = _torch()
    data, offs, sizes = _records()
    zd = zref.golden_input(ZDICT)
    cd = zstd_b200.ZSTD_CDict(zd, 3)
    cap = sum(zstd_b200.ZSTD_compressBound(s) + 64 for s in sizes)
    d_src, d_c = _dev(data), torch.zeros(cap, dtype=torch.uint8, device="cuda")
    res = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    zstd_b200.ZSTD_CCtx().compress_frames_async(d_c.data_ptr(), cap, d_src.data_ptr(), offs, sizes, res.data_ptr(), cdict=cd)
    torch.cuda.synchronize()
    _roundtrip(bytes(d_c[:_u64(res)].cpu().numpy()), data, ddict=zstd_b200.ZSTD_DDict(zd))


@gpu
@needs_ref
def test_reference_frames():
    src = zref.synthetic(3 << 20, seed=9, match_prob=0.7)
    for level in (6, 19):
        _roundtrip(zref.ref_compress(src, level), src)
    splitter = zref.golden_input("PR-3517-block-splitter-corruption-test")
    for level in (6, 19):
        _roundtrip(zref.ref_compress(splitter, level), splitter)


@gpu
def test_concatenated_and_skippable_frames():
    parts = [zref.synthetic(n, seed=n, match_prob=0.6) for n in (5000, 200_000, 0, 70_000)]
    ctx = zstd_b200.ZSTD_CCtx()
    frames = _skippable(5) + b"".join(ctx.compress(p, 3) + _skippable(i) for i, p in enumerate(parts))
    _roundtrip(frames, b"".join(parts))
    _roundtrip(_skippable(100) + _skippable(0), b"", cap=64)


def _async_checked(L, dctx, buf, cap, off=1):
    """the async call with source and destination `off` bytes into larger buffers; the bytes around the destination keep
    their value whatever the verdict"""
    torch = _torch()
    d_in = torch.zeros(len(buf) + off + 8, dtype=torch.uint8, device="cuda")
    d_in[off:off + len(buf)] = torch.frombuffer(bytearray(buf), dtype=torch.uint8).cuda()
    d_out = torch.full((cap + off + 16,), GUARD, dtype=torch.uint8, device="cuda")
    res = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    r = L.ZSTDB200_decompressDeviceAsync(dctx._h, d_out.data_ptr() + off, cap, d_in.data_ptr() + off, len(buf), res.data_ptr(), None)
    assert r == 0, L.ZSTD_getErrorCode(r)
    torch.cuda.synchronize()
    assert bool((d_out[:off] == GUARD).all()) and bool((d_out[off + cap:] == GUARD).all()), "bytes outside the destination changed"
    return _verdict(d_out, res, off)


def _sync_checked(L, dctx, buf, cap, d, off=1):
    torch = _torch()
    d_in = torch.zeros(len(buf) + off + 8, dtype=torch.uint8, device="cuda")
    d_in[off:off + len(buf)] = torch.frombuffer(bytearray(buf), dtype=torch.uint8).cuda()
    d_out = torch.full((cap + off + 16,), GUARD, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    r = L.ZSTDB200_decompressDevice_usingDict(dctx._h, d_out.data_ptr() + off, cap, d_in.data_ptr() + off, len(buf), d, len(d) if d else 0, None)
    torch.cuda.synchronize()
    return ("ERR", L.ZSTD_getErrorCode(r)) if L.ZSTD_isError(r) else bytes(d_out[off:off + r].cpu().numpy())


@gpu
@needs_ref
@pytest.mark.timeout(900, method="thread")
def test_verdict_parity_on_invalid_inputs():
    L = _lib()
    zd = zref.golden_input(ZDICT)
    sync, plain, with_dict = zstd_b200.ZSTD_DCtx(), zstd_b200.ZSTD_DCtx(), zstd_b200.ZSTD_DCtx()
    loaded = {}
    errors = 0
    for name, buf, cap, d in constructed() + corpus(CORPUS_GPU, 1):
        for dic in (None, d if d is not None else zd):
            a = plain
            if dic is not None:
                if loaded.get("bytes") is not dic:
                    with_dict.load_dictionary(dic)
                    loaded["bytes"] = dic
                a = with_dict
            want = _sync_checked(L, sync, buf, cap, dic)
            got = _async_checked(L, a, buf, cap)
            assert got == want, (name, dic is not None, got if isinstance(got, tuple) else len(got),
                                 want if isinstance(want, tuple) else len(want))
            errors += isinstance(want, tuple)
    assert errors > 100


@gpu
def test_more_blocks_than_the_workspace_holds():
    torch = _torch()
    cap, n = 64, 2000                                        # B = srcSize / 16 + 64 / 1024 + 1024 < 2000 blocks
    frame = struct.pack("<IBB", 0xFD2FB528, 0, 0) + b"\0\0\0" * (n - 1) + b"\1\0\0"
    assert len(frame) // 16 + 1024 < n
    d_src = _dev(frame)
    dctx = zstd_b200.ZSTD_DCtx()
    d_dst = torch.full((cap + 16,), GUARD, dtype=torch.uint8, device="cuda")
    d_dst, res = _async(dctx, d_src, len(frame), cap, d_dst=d_dst)
    torch.cuda.synchronize()
    assert zstd_b200.result_error(_u64(res)) == 66
    assert bool((d_dst == GUARD).all())
    assert _sync(dctx, d_src, len(frame), cap) == b""


@gpu
def test_capacity_too_small():
    torch = _torch()
    src = zref.synthetic(400_000, seed=41, match_prob=0.6)
    d_src = _dev(zstd_b200.ZSTD_CCtx().compress(src, 3))
    n = d_src.numel()
    dctx = zstd_b200.ZSTD_DCtx()
    d_dst = torch.full((len(src) + 4096,), GUARD, dtype=torch.uint8, device="cuda")
    d_dst, res = _async(dctx, d_src, n, len(src) - 1, d_dst=d_dst)
    torch.cuda.synchronize()
    assert zstd_b200.result_error(_u64(res)) == 70
    assert bool((d_dst == GUARD).all())
    d_dst, res = _async(dctx, d_src, n, len(src))
    torch.cuda.synchronize()
    assert _verdict(d_dst, res) == src


@gpu
def test_no_host_wait_and_ordered_behind_the_producer():
    torch = _torch()
    n = 3 << 20
    ctx = zstd_b200.ZSTD_CCtx()
    old, new = zref.synthetic(n, seed=31, match_prob=0.6), zref.synthetic(n, seed=32, match_prob=0.6)
    f_old, f_new = ctx.compress(old, 1), ctx.compress(new, 1)
    size = max(len(f_old), len(f_new)) + 8
    pad = lambda f: f + _skippable(size - len(f) - 8)       # noqa: E731
    d_src, d_new = _dev(pad(f_old)), _dev(pad(f_new))
    dctx = zstd_b200.ZSTD_DCtx()
    s = torch.cuda.Stream()
    d_dst, res = _async(dctx, d_src, size, n, stream=s)     # warm-up: the context's buffers fit this shape
    torch.cuda.synchronize()
    assert _verdict(d_dst, res) == old
    e = torch.cuda.Event()
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP_CYCLES)
        e.record(s)
        d_src.copy_(d_new)                                  # the producer
        d_dst, res = _async(dctx, d_src, size, n, stream=s, d_dst=d_dst)
    assert not e.query(), "the call waited for the work queued ahead of it"
    torch.cuda.synchronize()
    assert _verdict(d_dst, res) == new


@gpu
def test_calls_run_in_the_order_they_are_made():
    torch = _torch()
    srcs = [zref.synthetic(n, seed=50 + i, match_prob=0.6) for i, n in enumerate((3 << 20, 400_000, 1 << 20, 200_000))]
    ctx = zstd_b200.ZSTD_CCtx()
    d = [_dev(ctx.compress(x, 3)) for x in srcs]
    dctx = zstd_b200.ZSTD_DCtx()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s1):
        torch.cuda._sleep(SLEEP_CYCLES)
    a = _async(dctx, d[0], d[0].numel(), len(srcs[0]), stream=s1)
    b = _async(dctx, d[1], d[1].numel(), len(srcs[1]), stream=s2)
    got_sync = _sync(dctx, d[2], d[2].numel(), len(srcs[2]))
    c = _async(dctx, d[3], d[3].numel(), len(srcs[3]), stream=s2)
    torch.cuda.synchronize()
    assert [_verdict(*a), _verdict(*b), got_sync, _verdict(*c)] == srcs


@gpu
def test_more_queued_calls_than_the_compressors_ring():
    torch = _torch()
    k = 2 * 4 + 1                                           # ZSTDB200_ASYNC_SLOTS = 4
    srcs = [zref.synthetic(100_000 + 1000 * i, seed=60 + i, match_prob=0.6) for i in range(k)]
    ctx = zstd_b200.ZSTD_CCtx()
    d = [_dev(ctx.compress(x, 1)) for x in srcs]
    dctx = zstd_b200.ZSTD_DCtx()
    _async(dctx, d[-1], d[-1].numel(), 200_000)             # sizes the context: the queued calls below make no allocation
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP_CYCLES)
    out = [_async(dctx, d[i], d[i].numel(), 200_000, stream=s) for i in range(k)]
    torch.cuda.synchronize()
    assert [_verdict(*o) for o in out] == srcs


@gpu
def test_graph_capture_and_replay():
    torch = _torch()
    n = 400_000
    ctx = zstd_b200.ZSTD_CCtx()
    srcs = [zref.synthetic(n, seed=70 + i, match_prob=0.6) for i in range(4)]
    frames = [ctx.compress(x, 1) for x in srcs]
    size = max(map(len, frames)) + 64
    padded = [f + _skippable(size - len(f) - 8) for f in frames]
    zd = zref.golden_input(ZDICT)
    recs, offs, sizes = _records(nb=200)
    cd = zstd_b200.ZSTD_CDict(zd, 3)
    rec_frames = [b"".join(ctx.compress_using_cdict(recs[o:o + s], cd) for o, s in zip(offs, sizes))]
    dctx, ddctx = zstd_b200.ZSTD_DCtx(), zstd_b200.ZSTD_DCtx()
    ddict = zstd_b200.ZSTD_DDict(zd)
    ddctx.ref_ddict(ddict)
    d_src = _dev(padded[0])
    d_rec = _dev(rec_frames[0])
    d_dst = torch.zeros(n, dtype=torch.uint8, device="cuda")
    d_dst2 = torch.zeros(len(recs), dtype=torch.uint8, device="cuda")
    res = torch.zeros(2, dtype=torch.int64, device="cuda")

    def calls(stream):
        dctx.decompress_device_async(d_dst.data_ptr(), n, d_src.data_ptr(), size, res[0:].data_ptr(), stream)
        ddctx.decompress_device_async(d_dst2.data_ptr(), len(recs), d_rec.data_ptr(), d_rec.numel(), res[1:].data_ptr(), stream)

    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    calls(s.cuda_stream)                                    # warm-up of both shapes
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        calls(torch.cuda.current_stream().cuda_stream)
    for i in range(1, 4):
        d_src.copy_(torch.frombuffer(bytearray(padded[i]), dtype=torch.uint8))
        res.fill_(-1)
        g.replay()
        torch.cuda.synchronize()
        assert _verdict(d_dst, res[0:1]) == srcs[i]
        assert _verdict(d_dst2, res[1:2]) == recs
    # a larger shape than any call before: refused under capture, before anything is enqueued
    big_src = torch.zeros(8 << 20, dtype=torch.uint8, device="cuda")
    big_dst = torch.zeros(64 << 20, dtype=torch.uint8, device="cuda")
    g2 = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g2):
        res.fill_(0)
        with pytest.raises(zstd_b200.ZstdError) as e:
            dctx.decompress_device_async(big_dst.data_ptr(), big_dst.numel(), big_src.data_ptr(), big_src.numel(), res.data_ptr(),
                                         torch.cuda.current_stream().cuda_stream)
    assert e.value.code == 60
    torch.cuda.synchronize()


@gpu
def test_pending_prefix_is_refused_and_forgotten():
    torch = _torch()
    src = zref.synthetic(5000, seed=1)
    d_src = _dev(zstd_b200.ZSTD_CCtx().compress(src, 3))
    dctx = zstd_b200.ZSTD_DCtx()
    dctx.ref_prefix(zref.synthetic(50_000, seed=2))
    with pytest.raises(zstd_b200.ZstdError) as e:
        _async(dctx, d_src, d_src.numel(), len(src))
    assert e.value.code == 40
    d_dst, res = _async(dctx, d_src, d_src.numel(), len(src))
    torch.cuda.synchronize()
    assert _verdict(d_dst, res) == src


@gpu
def test_free_with_a_call_in_flight():
    torch = _torch()
    n = 3 << 20
    src = zref.synthetic(n, seed=90, match_prob=0.6)
    d_src = _dev(zstd_b200.ZSTD_CCtx().compress(src, 3))
    dctx = zstd_b200.ZSTD_DCtx()
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP_CYCLES)
    d_dst, res = _async(dctx, d_src, d_src.numel(), n, stream=s)
    dctx.close()
    torch.cuda.synchronize()
    assert _verdict(d_dst, res) == src
