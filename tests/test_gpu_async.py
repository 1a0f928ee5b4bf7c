"""Stream-ordered compression (ZSTDB200_compressDeviceAsync / ZSTDB200_compressFramesAsync): the bytes of the synchronous
device calls, the verdict in device memory in stream order, no host wait behind queued work, calls on one context in the
order they are made, the staging ring, CUDA graph capture and freeing a context with work in flight.  The first tests need
no GPU."""
import ctypes

import pytest

import zref
import zstd_b200

ZDICT = "zdict-16k-synthetic-seed77"
SLEEP_CYCLES = 200_000_000           # torch.cuda._sleep: about 100 ms on an H100


# ------------------------------------------------------------------ no GPU needed
def test_symbols_are_exported():
    L = zstd_b200.lib()
    assert hasattr(L, "ZSTDB200_compressDeviceAsync") and hasattr(L, "ZSTDB200_compressFramesAsync")


def _raw_calls(d_result):
    L = zstd_b200.lib()
    c = L.ZSTD_createCCtx()
    try:
        offs, sizes = (ctypes.c_size_t * 1)(0), (ctypes.c_size_t * 1)(10)
        one = L.ZSTDB200_compressDeviceAsync(c, 4096, 100, 8192, 10, 3, d_result, None)
        many = L.ZSTDB200_compressFramesAsync(c, 4096, 100, 8192, offs, sizes, 1, None, 3, None, d_result, None)
        return L.ZSTD_getErrorCode(one), L.ZSTD_getErrorCode(many)
    finally:
        L.ZSTD_freeCCtx(c)


@pytest.mark.skipif(zstd_b200.device_available(), reason="a CUDA device is present")
def test_without_a_device_both_return_generic():
    assert _raw_calls(16384) == (1, 1)


def test_null_result_returns_generic():
    assert _raw_calls(None) == (1, 1)


# ------------------------------------------------------------------ GPU
gpu = pytest.mark.gpu


def _torch():
    return pytest.importorskip("torch")


def _dev(b):
    torch = _torch()
    return torch.frombuffer(bytearray(b if b else b"\0"), dtype=torch.uint8).cuda()


def _cap(n):
    return zstd_b200.ZSTD_compressBound(n) + 64


def _u64(t):
    return int(t.item()) & 0xFFFFFFFFFFFFFFFF


def _sync(ctx, src, level, d_src=None):
    """compress_device of src on ctx (NULL stream: the context's streams, behind a device synchronise)"""
    torch = _torch()
    d_src = _dev(src) if d_src is None else d_src
    torch.cuda.synchronize()
    d_dst = torch.zeros(_cap(len(src)), dtype=torch.uint8, device="cuda")
    r = ctx.compress_device(d_dst.data_ptr(), d_dst.numel(), d_src.data_ptr(), len(src), level, 0)
    return d_dst[:r].cpu().numpy().tobytes()


def _async(ctx, d_src, n, level, stream=None, cap=None, d_dst=None):
    """enqueue compress_device_async; returns (d_dst, d_result) to read after a synchronise"""
    torch = _torch()
    d_dst = torch.zeros(_cap(n), dtype=torch.uint8, device="cuda") if d_dst is None else d_dst
    res = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    s = torch.cuda.current_stream() if stream is None else stream
    s.wait_stream(torch.cuda.current_stream())              # the buffers above are made on the current stream
    ctx.compress_device_async(d_dst.data_ptr(), d_dst.numel() if cap is None else cap, d_src.data_ptr(), n, res.data_ptr(), level,
                              s.cuda_stream)
    return d_dst, res


def _frame(d_dst, res):
    r = _u64(res)
    assert zstd_b200.result_error(r) is None, zstd_b200.result_error(r)
    return d_dst[:r].cpu().numpy().tobytes()


def _input(n):
    if n == 3 << 20 and zref.have_datagen():
        return zref.datagen(n, 50)
    return zref.synthetic(n, seed=n % 997, match_prob=0.6)


@pytest.fixture(scope="module")
def big():
    return zref.synthetic(300 << 20, seed=3, match_prob=0.6)


@gpu
@pytest.mark.parametrize("level", [1, 3, -5])
@pytest.mark.parametrize("n", [0, 7, 5000, (128 << 10) + 1, 400_000, 3 << 20, 300 << 20])
def test_same_bytes_as_compress_device(n, level, big):
    torch = _torch()
    src = big if n == 300 << 20 else _input(n)
    ctx = zstd_b200.ZSTD_CCtx()
    want = _sync(ctx, src, level)
    sync_launches = ctx.stats().launches
    d_src = _dev(src)
    d_dst, res = _async(ctx, d_src, n, level, stream=torch.cuda.Stream())
    torch.cuda.synchronize()
    assert _frame(d_dst, res) == want
    assert ctx.stats().launches > 0 and ctx.stats().kernel_ms == 0.0
    assert ctx.stats().launches == sync_launches          # the same kernels, the verdict kernel included
    if level == 3 and n in (5000, 3 << 20):
        assert zstd_b200.ZSTD_DCtx().decompress(want, n) == src
        if zref.have_ref():
            assert zref.ref_decompress(want, n) == src


@gpu
@pytest.mark.parametrize("kind", ["checksum", "cdict", "prefix", "ldm"])
def test_same_bytes_with_sticky_state(kind):
    torch = _torch()
    n = (2 << 20) if kind == "ldm" else 400_000
    src = zref.synthetic(n, seed=11, match_prob=0.6)
    d_src = _dev(src)
    ctx = zstd_b200.ZSTD_CCtx()
    dict_bytes = None
    if kind == "checksum":
        ctx.set_parameter(201, 1)
    elif kind == "ldm":
        ctx.set_parameter(160, 1)
    if kind == "cdict":
        dict_bytes = zref.golden_input(ZDICT)
        cd = zstd_b200.ZSTD_CDict(dict_bytes, 3)
        ctx.ref_cdict(cd)
        d_dst = torch.zeros(_cap(n), dtype=torch.uint8, device="cuda")
        r, _ = ctx.compress_frames_using_cdict(d_dst.data_ptr(), d_dst.numel(), d_src.data_ptr(), [0], [n], cd)
        want = d_dst[:r].cpu().numpy().tobytes()
    elif kind == "prefix":
        dict_bytes = zref.synthetic(1 << 20, seed=12, match_prob=0.6)
        d_prefix = _dev(dict_bytes)
        ctx.ref_prefix_device(d_prefix.data_ptr(), len(dict_bytes))
        want = _sync(ctx, src, 3, d_src)
        ctx.ref_prefix_device(d_prefix.data_ptr(), len(dict_bytes))
    else:
        want = _sync(ctx, src, 3, d_src)
    d_dst, res = _async(ctx, d_src, n, 3, stream=torch.cuda.Stream())
    torch.cuda.synchronize()
    assert _frame(d_dst, res) == want
    dctx = zstd_b200.ZSTD_DCtx()
    if dict_bytes is None:
        assert dctx.decompress(want, n) == src
        if zref.have_ref():
            assert zref.ref_decompress(want, n) == src
    else:
        dctx.load_dictionary(dict_bytes) if kind == "cdict" else dctx.ref_prefix(dict_bytes)
        assert dctx.decompress(want, n) == src
        if zref.have_ref():
            assert zref.ref_decompress_using_dict(want, dict_bytes, n) == src


@gpu
def test_host_prefix_is_refused_and_forgotten():
    torch = _torch()
    ctx = zstd_b200.ZSTD_CCtx()
    src = zref.synthetic(5000, seed=1)
    d_src = _dev(src)
    ctx.ref_prefix(zref.synthetic(50_000, seed=2))
    with pytest.raises(zstd_b200.ZstdError) as e:
        _async(ctx, d_src, len(src), 3)
    assert e.value.code == 40
    d_dst, res = _async(ctx, d_src, len(src), 3)
    torch.cuda.synchronize()
    assert _frame(d_dst, res) == _sync(zstd_b200.ZSTD_CCtx(), src, 3)


def _records(nb=2000, size=1024):
    data = zref.synthetic(nb * size, seed=21, match_prob=0.5)
    return data, [i * size for i in range(nb)], [size] * nb


@gpu
def test_batch_with_a_cdict():
    torch = _torch()
    data, offs, sizes = _records()
    cd = zstd_b200.ZSTD_CDict(zref.golden_input(ZDICT), 3)
    ctx = zstd_b200.ZSTD_CCtx()
    d_src = _dev(data)
    cap = sum(_cap(s) for s in sizes)
    d_dst = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    r, want_sizes = ctx.compress_frames_using_cdict(d_dst.data_ptr(), cap, d_src.data_ptr(), offs, sizes, cd)
    want = d_dst[:r].cpu().numpy().tobytes()
    d_dst2 = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    res = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    c_sizes = torch.zeros(len(sizes), dtype=torch.int64, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    ctx.compress_frames_async(d_dst2.data_ptr(), cap, d_src.data_ptr(), offs, sizes, res.data_ptr(), cdict=cd,
                              d_c_sizes=c_sizes.data_ptr(), stream=s.cuda_stream)
    torch.cuda.synchronize()
    assert _u64(res) == r and c_sizes.tolist() == want_sizes
    assert d_dst2[:r].cpu().numpy().tobytes() == want


@gpu
def test_batch_without_frames_writes_zero():
    torch = _torch()
    res = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    zstd_b200.ZSTD_CCtx().compress_frames_async(0, 0, 0, [], [], res.data_ptr())
    torch.cuda.synchronize()
    assert _u64(res) == 0


@gpu
def test_no_host_wait_and_ordered_behind_the_producer():
    torch = _torch()
    n = 3 << 20
    ctx = zstd_b200.ZSTD_CCtx()
    old, new = zref.synthetic(n, seed=31, match_prob=0.6), zref.synthetic(n, seed=32, match_prob=0.6)
    d_src, d_new = _dev(old), _dev(new)
    s = torch.cuda.Stream()
    _async(ctx, d_src, n, 1, stream=s)                      # warm-up: the context's buffers fit this shape
    torch.cuda.synchronize()
    d_dst = torch.zeros(_cap(n), dtype=torch.uint8, device="cuda")
    e = torch.cuda.Event()
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP_CYCLES)
        e.record(s)
        d_src.copy_(d_new)                                  # the producer
        d_dst, res = _async(ctx, d_src, n, 1, stream=s, d_dst=d_dst)
    assert not e.query(), "the call waited for the work queued ahead of it"
    torch.cuda.synchronize()
    assert _frame(d_dst, res) == _sync(zstd_b200.ZSTD_CCtx(), new, 1)


@gpu
def test_capacity_too_small():
    torch = _torch()
    n = 400_000
    src = zref.synthetic(n, seed=41, match_prob=0.6)
    ctx = zstd_b200.ZSTD_CCtx()
    want = _sync(ctx, src, 3)
    d_src = _dev(src)
    d_dst = torch.full((len(want) + 4096,), 0xAB, dtype=torch.uint8, device="cuda")
    d_dst, res = _async(ctx, d_src, n, 3, cap=len(want) - 1, d_dst=d_dst)
    torch.cuda.synchronize()
    assert zstd_b200.result_error(_u64(res)) == 70
    assert bool((d_dst[len(want) - 1:] == 0xAB).all())
    d_dst, res = _async(ctx, d_src, n, 3)
    torch.cuda.synchronize()
    assert _frame(d_dst, res) == want


@gpu
def test_calls_run_in_the_order_they_are_made():
    torch = _torch()
    srcs = [zref.synthetic(n, seed=50 + i, match_prob=0.6) for i, n in enumerate((3 << 20, 400_000, 1 << 20))]
    want = [_sync(zstd_b200.ZSTD_CCtx(), s, 3) for s in srcs]
    d = [_dev(s) for s in srcs]
    ctx = zstd_b200.ZSTD_CCtx()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s1):
        torch.cuda._sleep(SLEEP_CYCLES)
    a = _async(ctx, d[0], len(srcs[0]), 3, stream=s1)
    b = _async(ctx, d[1], len(srcs[1]), 3, stream=s2)
    d_dst = torch.zeros(_cap(len(srcs[2])), dtype=torch.uint8, device="cuda")
    r = ctx.compress_device(d_dst.data_ptr(), d_dst.numel(), d[2].data_ptr(), len(srcs[2]), 3, 0)
    got_sync = d_dst[:r].cpu().numpy().tobytes()
    torch.cuda.synchronize()
    assert [_frame(*a), _frame(*b), got_sync] == want


@gpu
def test_more_calls_than_staging_slots():
    torch = _torch()
    k = 2 * 4 + 1                                           # ZSTDB200_ASYNC_SLOTS = 4
    srcs = [zref.synthetic(100_000 + 1000 * i, seed=60 + i, match_prob=0.6) for i in range(k)]
    d = [_dev(s) for s in srcs]
    ctx = zstd_b200.ZSTD_CCtx()
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP_CYCLES)
    out = [_async(ctx, d[i], len(srcs[i]), 1, stream=s) for i in range(k)]
    torch.cuda.synchronize()
    fresh = zstd_b200.ZSTD_CCtx()
    assert [_frame(*o) for o in out] == [_sync(fresh, x, 1) for x in srcs]


@gpu
def test_graph_capture_and_replay():
    torch = _torch()
    n = 400_000
    data, offs, sizes = _records(nb=200)
    cd = zstd_b200.ZSTD_CDict(zref.golden_input(ZDICT), 3)
    ctx = zstd_b200.ZSTD_CCtx()
    d_src = torch.zeros(n, dtype=torch.uint8, device="cuda")
    d_rec = torch.zeros(len(data), dtype=torch.uint8, device="cuda")
    d_dst = torch.zeros(_cap(n), dtype=torch.uint8, device="cuda")
    cap2 = sum(_cap(x) for x in sizes)
    d_dst2 = torch.zeros(cap2, dtype=torch.uint8, device="cuda")
    res = torch.zeros(2, dtype=torch.int64, device="cuda")
    c_sizes = torch.zeros(len(sizes), dtype=torch.int64, device="cuda")

    def calls(stream):
        ctx.compress_device_async(d_dst.data_ptr(), d_dst.numel(), d_src.data_ptr(), n, res[0:].data_ptr(), 1, stream)
        ctx.compress_frames_async(d_dst2.data_ptr(), cap2, d_rec.data_ptr(), offs, sizes, res[1:].data_ptr(), cdict=cd,
                                  d_c_sizes=c_sizes.data_ptr(), stream=stream)

    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    calls(s.cuda_stream)                                    # warm-up of both shapes
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        calls(torch.cuda.current_stream().cuda_stream)
    ref_ctx = zstd_b200.ZSTD_CCtx()
    for i in range(3):
        src = zref.synthetic(n, seed=70 + i, match_prob=0.6)
        rec = zref.synthetic(len(data), seed=80 + i, match_prob=0.5)
        d_src.copy_(torch.frombuffer(bytearray(src), dtype=torch.uint8))
        d_rec.copy_(torch.frombuffer(bytearray(rec), dtype=torch.uint8))
        res.fill_(-1)
        g.replay()
        torch.cuda.synchronize()
        assert _frame(d_dst, res[0:1]) == _sync(ref_ctx, src, 1)
        d_want = torch.zeros(cap2, dtype=torch.uint8, device="cuda")
        d_r = _dev(rec)
        torch.cuda.synchronize()
        r, want_sizes = ref_ctx.compress_frames_using_cdict(d_want.data_ptr(), cap2, d_r.data_ptr(), offs, sizes, cd)
        assert _u64(res[1:2]) == r and c_sizes.tolist() == want_sizes
        assert d_dst2[:r].cpu().numpy().tobytes() == d_want[:r].cpu().numpy().tobytes()
    # a larger shape than any call before: refused under capture, before anything is enqueued
    big = torch.zeros(8 << 20, dtype=torch.uint8, device="cuda")
    big_dst = torch.zeros(_cap(8 << 20), dtype=torch.uint8, device="cuda")
    g2 = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g2):
        res.fill_(0)
        with pytest.raises(zstd_b200.ZstdError) as e:
            ctx.compress_device_async(big_dst.data_ptr(), big_dst.numel(), big.data_ptr(), big.numel(), res.data_ptr(), 1,
                                      torch.cuda.current_stream().cuda_stream)
    assert e.value.code == 60
    torch.cuda.synchronize()


@gpu
def test_free_with_a_call_in_flight():
    torch = _torch()
    n = 3 << 20
    src = zref.synthetic(n, seed=90, match_prob=0.6)
    d_src = _dev(src)
    ctx = zstd_b200.ZSTD_CCtx()
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP_CYCLES)
    d_dst, res = _async(ctx, d_src, n, 3, stream=s)
    ctx.close()
    torch.cuda.synchronize()
    frame = _frame(d_dst, res)
    assert zstd_b200.ZSTD_DCtx().decompress(frame, n) == src
