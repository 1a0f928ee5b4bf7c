"""A dictionary per frame in one batch call (ZSTDB200_compressFrames_usingCDicts and its stream-ordered form): every frame's
bytes are those of its own single-record call, the launch count does not grow with the number of dictionaries, first use
uploads and primes new CDicts in bulk, the async form captures into a CUDA graph, refusals write nothing, and contexts on
two threads share CDicts without deadlock."""
import ctypes
import random
import threading

import pytest

import zref
import zstd_b200

gpu = pytest.mark.gpu
ZDICT = "zdict-16k-synthetic-seed77"


def _torch():
    import torch
    return torch


def _with_id(d: bytes, dict_id: int) -> bytes:
    """the golden zstd-format dictionary under another dictID"""
    return d[:4] + dict_id.to_bytes(4, "little") + d[8:]


def _dev(b: bytes):
    torch = _torch()
    return torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda() if b else torch.zeros(1, dtype=torch.uint8, device="cuda")


def _layout(sizes):
    offs = [sum(sizes[:i]) for i in range(len(sizes))]
    cap = sum(zstd_b200.ZSTD_compressBound(n) + 32 for n in sizes)
    return offs, cap


def _split(out: bytes, csz):
    pos, frames = 0, []
    for n in csz:
        frames.append(out[pos:pos + n])
        pos += n
    return frames


def _batch(c, src: bytes, sizes, cdicts, level=3, device=True):
    """one per-frame-dictionary call over device (or host) buffers: the list of frames"""
    offs, cap = _layout(sizes)
    if device:
        torch = _torch()
        d_src, d_dst = _dev(src), torch.zeros(cap, dtype=torch.uint8, device="cuda")
        total, csz = c.compress_frames_using_cdicts(d_dst.data_ptr(), cap, d_src.data_ptr(), offs, sizes, cdicts, level)
        out = bytes(d_dst[:total].cpu().numpy())
    else:
        dst, sbuf = ctypes.create_string_buffer(cap), ctypes.create_string_buffer(src, max(len(src), 1))
        total, csz = c.compress_frames_using_cdicts(ctypes.addressof(dst), cap, ctypes.addressof(sbuf), offs, sizes, cdicts, level,
                                                    device_memory=False)
        out = dst.raw[:total]
    assert sum(csz) == total
    return _split(out, csz)


def _single(c, src: bytes, sizes, cdict):
    """the single-CDict batch call (host buffers): the list of frames"""
    offs, cap = _layout(sizes)
    dst, sbuf = ctypes.create_string_buffer(cap), ctypes.create_string_buffer(src, max(len(src), 1))
    total, csz = c.compress_frames_using_cdict(ctypes.addressof(dst), cap, ctypes.addressof(sbuf), offs, sizes, cdict, device_memory=False)
    return _split(dst.raw[:total], csz)


@pytest.fixture(scope="module")
def mix():
    """a seeded mix of dictionaries: (bytes, level) per CDict"""
    g = zref.golden_input(ZDICT)
    raw = [zref.synthetic(n, 500 + n % 97, 0.5) for n in (8, 1 << 10, 16 << 10, 112 << 10)]
    specs = [(g, 1), (_with_id(g, 0x1234567), 3), (_with_id(g, 77), -1), (raw[0], 1), (raw[1], 3), (raw[2], 7), (raw[3], 1),
             (raw[3], 3), (b"tiny", 1), (g, 7)]
    cds = [zstd_b200.ZSTD_CDict(d, lv) for d, lv in specs]
    yield specs, cds
    for cd in cds:
        cd.close()


def _records(seed, n):
    rng = random.Random(seed)
    sizes = [rng.choice((0, 1, 7, 1 << 10, 4 << 10, 130 << 10, 600 << 10)) for _ in range(n)]
    return zref.synthetic(sum(sizes), seed, 0.5), sizes, rng


@gpu
@pytest.mark.parametrize("device", [True, False])
def test_frames_equal_their_single_record_calls(mix, device):
    specs, cds = mix
    src, sizes, rng = _records(11 + device, 36)
    pick = [rng.randrange(len(cds) + 2) for _ in sizes]           # the last two: no dictionary
    cdicts = [cds[k] if k < len(cds) else None for k in pick]
    c = zstd_b200.ZSTD_CCtx()
    try:
        frames = _batch(c, src, sizes, cdicts, level=1, device=device)
        offs, _ = _layout(sizes)
        for i, (cd, k) in enumerate(zip(cdicts, pick)):
            rec = src[offs[i]:offs[i] + sizes[i]]
            if cd is None:
                assert frames[i] == zref.oracle_compress(rec, 1)
                continue
            d, lv = specs[k]
            assert frames[i] == c.compress_using_cdict(rec, cd), i
            want = zref.oracle_compress(rec, lv) if len(d) < 8 else zref.oracle_compress_using_dict(rec, d, lv)
            assert frames[i] == want, i
            if zref.have_ref() and len(d) >= 8:
                assert zref.ref_decompress_using_dict(frames[i], d, len(rec)) == rec
    finally:
        c.close()


@gpu
@pytest.mark.parametrize("checksum,dict_id", [(1, 1), (0, 0), (1, 0)])
def test_sticky_frame_flags_apply_per_frame(mix, checksum, dict_id):
    """with the checksum and dictID flags set, each frame is the single-CDict batch call's frame for its record"""
    specs, cds = mix
    src, sizes, rng = _records(21 + checksum + 2 * dict_id, 24)
    cdicts = [rng.choice(cds + [None]) for _ in sizes]
    c = zstd_b200.ZSTD_CCtx()
    try:
        c.set_parameter(201, checksum)
        c.set_parameter(202, dict_id)
        frames = _batch(c, src, sizes, cdicts, level=1)
        offs, _ = _layout(sizes)
        for i, cd in enumerate(cdicts):
            rec = src[offs[i]:offs[i] + sizes[i]]
            if cd is None:
                dst, sbuf = ctypes.create_string_buffer(sizes[i] + 1024), ctypes.create_string_buffer(rec, max(len(rec), 1))
                t, _ = c.compress_frames(ctypes.addressof(dst), sizes[i] + 1024, ctypes.addressof(sbuf), [0], [sizes[i]], level=1,
                                         device_memory=False)
                assert frames[i] == dst.raw[:t], i
            else:
                assert frames[i] == _single(c, rec, [sizes[i]], cd)[0], i
    finally:
        c.close()


def _uniform(k, n=4096, rec=1 << 10, seed=5):
    g = zref.golden_input(ZDICT)
    cds = [zstd_b200.ZSTD_CDict(_with_id(g, 1000 + j), 1) for j in range(k)]
    return g, cds, zref.synthetic(n * rec, seed, 0.5), [rec] * n


@gpu
def test_launches_do_not_depend_on_the_number_of_dictionaries():
    c = zstd_b200.ZSTD_CCtx()
    launches, all_cds = {}, []
    try:
        for k in (1, 64, 1024):
            g, cds, src, sizes = _uniform(k)
            all_cds += cds
            cdicts = [cds[i % k] for i in range(len(sizes))]
            first = _batch(c, src, sizes, cdicts, level=1)          # warm-up: uploads and images
            frames = _batch(c, src, sizes, cdicts, level=1)
            launches[k] = c.stats().launches
            assert frames == first
            offs, _ = _layout(sizes)
            for i in range(0, len(sizes), 131):
                assert frames[i] == zref.oracle_compress_using_dict(src[offs[i]:offs[i] + sizes[i]], _with_id(g, 1000 + i % k), 1), (k, i)
            if k == 1:                                              # the single-CDict call on the same device buffers
                torch = _torch()
                d_src, d_dst = _dev(src), torch.zeros(_layout(sizes)[1], dtype=torch.uint8, device="cuda")
                total, csz = c.compress_frames_using_cdict(d_dst.data_ptr(), d_dst.numel(), d_src.data_ptr(), offs, sizes, cds[0])
                launches["single"] = c.stats().launches
                assert frames == _split(bytes(d_dst[:total].cpu().numpy()), csz)
        assert launches[1] == launches[64] == launches[1024] == launches["single"], launches
    finally:
        c.close()
        for cd in all_cds:
            cd.close()


@gpu
def test_first_use_uploads_and_primes_in_bulk():
    """1024 fresh CDicts: the first call makes one image-build launch for its one fast parameter group and gives the warm
    call's bytes; what the CDicts take on the device is proportional to what they hold"""
    torch = _torch()
    _, warmup, src, sizes = _uniform(1024, seed=6)
    g, cds, _, _ = _uniform(1024, seed=6)
    c = zstd_b200.ZSTD_CCtx()
    try:
        _batch(c, src, sizes, [warmup[i % 1024] for i in range(len(sizes))], level=1)   # the context's own buffers
        cdicts = [cds[i % 1024] for i in range(len(sizes))]
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        cold = _batch(c, src, sizes, cdicts, level=1)
        cold_launches = c.stats().launches
        free1 = torch.cuda.mem_get_info()[0]
        warm = _batch(c, src, sizes, cdicts, level=1)
        assert cold == warm
        assert cold_launches - c.stats().launches == 1
        # a tail of about 16 KiB and one 28 KiB table image each (the first use took 850 KB per CDict before)
        assert (free0 - free1) / 1024 < 256 << 10, (free0 - free1) / 1024
    finally:
        c.close()
        for cd in cds + warmup:
            cd.close()


@gpu
def test_async_equals_sync_and_replays_in_a_graph(mix):
    torch = _torch()
    specs, cds = mix
    rng = random.Random(31)
    sizes = [rng.choice((1 << 10, 4 << 10, 7, 130 << 10)) for _ in range(64)]
    offs, cap = _layout(sizes)
    cdicts = [rng.choice(cds + [None]) for _ in sizes]
    ctx, ref_ctx = zstd_b200.ZSTD_CCtx(), zstd_b200.ZSTD_CCtx()
    d_src = torch.zeros(sum(sizes), dtype=torch.uint8, device="cuda")
    d_dst = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    res = torch.zeros(1, dtype=torch.int64, device="cuda")
    c_sizes = torch.zeros(len(sizes), dtype=torch.int64, device="cuda")

    def call(stream):
        ctx.compress_frames_async_using_cdicts(d_dst.data_ptr(), cap, d_src.data_ptr(), offs, sizes, cdicts, res.data_ptr(),
                                               level=1, d_c_sizes=c_sizes.data_ptr(), stream=stream)

    try:
        s = torch.cuda.Stream()
        d_src.copy_(torch.frombuffer(bytearray(zref.synthetic(sum(sizes), 40, 0.5)), dtype=torch.uint8))
        torch.cuda.synchronize()
        call(s.cuda_stream)                                         # warm-up: every CDict resident, every image built
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            call(torch.cuda.current_stream().cuda_stream)
        for i in range(2):
            src = zref.synthetic(sum(sizes), 41 + i, 0.5)
            d_src.copy_(torch.frombuffer(bytearray(src), dtype=torch.uint8))
            res.fill_(-1)
            g.replay()
            torch.cuda.synchronize()
            want = _batch(ref_ctx, src, sizes, cdicts, level=1)
            total = int(res.item())
            assert total == sum(len(f) for f in want) and c_sizes.tolist() == [len(f) for f in want]
            assert bytes(d_dst[:total].cpu().numpy()) == b"".join(want)
        # one cold CDict: refused under capture before anything is enqueued
        cold = zstd_b200.ZSTD_CDict(_with_id(zref.golden_input(ZDICT), 4242), 1)
        cdicts[5] = cold
        g2 = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g2):
            with pytest.raises(zstd_b200.ZstdError) as e:
                call(torch.cuda.current_stream().cuda_stream)
        assert e.value.code == 60
        torch.cuda.synchronize()
        cold.close()
    finally:
        ctx.close()
        ref_ctx.close()


@gpu
def test_refusals_write_nothing(mix):
    torch = _torch()
    specs, cds = mix
    sizes = [4 << 10] * 8
    src = zref.synthetic(sum(sizes), 50, 0.5)
    offs, cap = _layout(sizes)
    d_src = _dev(src)
    d_dst = torch.full((cap + 64,), 0xA5, dtype=torch.uint8, device="cuda")
    c = zstd_b200.ZSTD_CCtx()
    try:
        lv7 = [cd for (d, lv), cd in zip(specs, cds) if lv == 7][0]
        zstd_b200.lib().ZSTDB200_setStrictLevels(1)
        try:
            with pytest.raises(zstd_b200.ZstdError) as e:
                c.compress_frames_using_cdicts(d_dst.data_ptr(), cap, d_src.data_ptr(), offs, sizes, [cds[0]] * 7 + [lv7], 1)
            assert e.value.code == 40
        finally:
            zstd_b200.lib().ZSTDB200_setStrictLevels(0)
        c.ref_prefix(b"some prefix bytes")
        with pytest.raises(zstd_b200.ZstdError) as e:
            c.compress_frames_using_cdicts(d_dst.data_ptr(), cap, d_src.data_ptr(), offs, sizes, [cds[0]] * 8, 1)
        assert e.value.code == 40
        c.reset(2)
        assert bool((d_dst == 0xA5).all())
        small = 3000
        with pytest.raises(zstd_b200.ZstdError) as e:
            c.compress_frames_using_cdicts(d_dst.data_ptr(), small, d_src.data_ptr(), offs, sizes, [cds[1]] * 8, 1)
        assert e.value.code == 70
        assert bool((d_dst[small:] == 0xA5).all())
    finally:
        c.close()


@gpu
def test_two_threads_share_dictionaries_in_opposite_orders():
    g = zref.golden_input(ZDICT)
    shared = [zstd_b200.ZSTD_CDict(_with_id(g, 5000 + j), 1 + j % 3) for j in range(48)]
    sizes = [1 << 10] * 480
    src = zref.synthetic(sum(sizes), 60, 0.5)
    orders = [[shared[i % 48] for i in range(len(sizes))], [shared[47 - i % 48] for i in range(len(sizes))]]
    out, errors = [None, None], []

    def work(t):
        try:
            c = zstd_b200.ZSTD_CCtx()
            out[t] = [_batch(c, src, sizes, orders[t], level=1, device=False) for _ in range(3)]
            c.close()
        except Exception as e:                                      # reported by the main thread
            errors.append(e)

    th = [threading.Thread(target=work, args=(t,)) for t in (0, 1)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=300)
    assert not any(t.is_alive() for t in th) and not errors, errors
    c = zstd_b200.ZSTD_CCtx()
    try:
        offs, _ = _layout(sizes)
        for t in (0, 1):
            assert out[t][0] == out[t][1] == out[t][2]
            for i in range(0, len(sizes), 37):
                assert out[t][0][i] == c.compress_using_cdict(src[offs[i]:offs[i] + sizes[i]], orders[t][i])
    finally:
        c.close()
        for cd in shared:
            cd.close()


@gpu
@pytest.mark.parametrize("device", [True, False])
def test_no_array_means_no_dictionary_for_any_frame(device):
    """cdicts NULL: every frame without a dictionary at the call's level, as ZSTDB200_compressFrames with dict NULL"""
    src, sizes, _ = _records(71 + device, 20)
    offs, cap = _layout(sizes)
    c = zstd_b200.ZSTD_CCtx()
    try:
        frames = _batch(c, src, sizes, None, level=-2, device=device)
        dst, sbuf = ctypes.create_string_buffer(cap), ctypes.create_string_buffer(src, max(len(src), 1))
        total, csz = c.compress_frames(ctypes.addressof(dst), cap, ctypes.addressof(sbuf), offs, sizes, level=-2, device_memory=False)
        assert frames == _split(dst.raw[:total], csz)
        assert frames[3] == zref.oracle_compress(src[offs[3]:offs[3] + sizes[3]], -2)
    finally:
        c.close()
