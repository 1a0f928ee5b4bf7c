"""Batch decompression (ZSTDB200_decompressFrames / ZSTDB200_decompressFramesAsync): every entry decoded into its own slot
with the bytes and result ZSTDB200_decompressDevice gives it alone, corrupt entries failing alone next to good ones, the
refusals, sync and stream-ordered calls agreeing, graph capture, call order on one context and a launch count that does not
depend on the number of entries.  The first tests need no GPU."""
import ctypes
import struct

import pytest

import seqgen
import zref
import zstd_b200
from test_decode_invalid import CORPUS_GPU, GUARD, _lib, constructed, corpus, needs_ref, ref_oneshot
from test_gpu_async import SLEEP_CYCLES, ZDICT, _dev, _records, _torch, _u64

SKIP_MAGIC = 0x184D2A50
GAP = 24                                                     # guard bytes between two slots


# ------------------------------------------------------------------ no GPU needed
def test_symbols_are_exported():
    L = zstd_b200.lib()
    assert hasattr(L, "ZSTDB200_decompressFrames") and hasattr(L, "ZSTDB200_decompressFramesAsync")


def _one_entry(async_call, d_result):
    L = zstd_b200.lib()
    d = L.ZSTD_createDCtx()
    one = (ctypes.c_size_t * 1)(0)
    ten = (ctypes.c_size_t * 1)(10)
    try:
        if async_call:
            r = L.ZSTDB200_decompressFramesAsync(d, 4096, 100, one, (ctypes.c_size_t * 1)(100), 8192, 10, one, ten, 1, None, d_result, None)
        else:
            r = L.ZSTDB200_decompressFrames(d, 4096, 100, one, (ctypes.c_size_t * 1)(100), 8192, 10, one, ten, 1, None, None)
        return L.ZSTD_getErrorCode(r)
    finally:
        L.ZSTD_freeDCtx(d)


@pytest.mark.skipif(zstd_b200.device_available(), reason="a CUDA device is present")
def test_without_a_device_returns_generic():
    assert _one_entry(True, 16384) == 1 and _one_entry(False, None) == 1


def test_null_result_returns_generic():
    assert _one_entry(True, None) == 1


# ------------------------------------------------------------------ GPU
gpu = pytest.mark.gpu


def _skippable(n):
    return struct.pack("<II", SKIP_MAGIC, n) + bytes(n)


def _layout(entries, caps):
    """the entries back to back in one source buffer (a byte of padding in front of each), and slots of caps[i] bytes with
    GAP guard bytes around each: (src bytes, src offsets, dst offsets, dst capacity)"""
    src, so, do, pos = bytearray(), [], [], GAP
    for e, c in zip(entries, caps):
        src += b"\x77"
        so.append(len(src)); src += e
        do.append(pos); pos += c + GAP
    return bytes(src), so, do, pos


def _slot(d_out, off, r):
    e = zstd_b200.result_error(r)
    return ("ERR", e) if e is not None else bytes(d_out[off:off + r].cpu().numpy())


def batch(dctx, entries, caps, stream=None):
    """both calls on the same bytes: [(result per entry)], where a result is the bytes or ("ERR", code).  Both calls must agree
    in bytes and sizes, keep every byte outside the slots, and give the lowest failing entry's code or the sum"""
    torch = _torch()
    src, so, do, cap = _layout(entries, caps)
    d_src = _dev(src)
    sizes = [len(e) for e in entries]
    outs = []
    for kind in ("sync", "async"):
        d_out = torch.full((cap,), GUARD, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        if kind == "sync":
            r, per = dctx.decompress_frames(d_out.data_ptr(), cap, do, caps, d_src.data_ptr(), len(src), so, sizes)
        else:
            res = torch.full((1 + len(entries),), -1, dtype=torch.int64, device="cuda")
            s = torch.cuda.Stream() if stream is None else stream
            dctx.decompress_frames_async(d_out.data_ptr(), cap, do, caps, d_src.data_ptr(), len(src), so, sizes, res.data_ptr(),
                                         res[1:].data_ptr(), s.cuda_stream)
            torch.cuda.synchronize()
            r, per = _u64(res[0]), [int(x) & (2**64 - 1) for x in res[1:].cpu().tolist()]
        mask = torch.ones(cap, dtype=torch.bool, device="cuda")
        for o, c in zip(do, caps):
            mask[o:o + c] = False
        assert bool((d_out[mask] == GUARD).all()), (kind, "bytes outside the slots changed")
        bad = [i for i, v in enumerate(per) if zstd_b200.result_error(v) is not None]
        assert r == (per[bad[0]] if bad else sum(per)), kind
        outs.append(([_slot(d_out, o, v) for o, v in zip(do, per)], d_out, do))
    (a, d_a, _), (b, d_b, _) = outs
    assert a == b, "the synchronous and the stream-ordered call differ"
    assert torch.equal(d_a, d_b)
    return a, d_a, do


def single(dctx, entry, cap):
    """ZSTDB200_decompressDevice on the entry alone (the context's sticky dictionary): (result, slot untouched)"""
    torch = _torch()
    d_in = _dev(b"\x77" + entry)
    d_out = torch.full((cap + 2 * GAP,), GUARD, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    L = zstd_b200.lib()
    r = L.ZSTDB200_decompressDevice(dctx._h, d_out.data_ptr() + GAP, cap, d_in.data_ptr() + 1, len(entry), None)
    torch.cuda.synchronize()
    untouched = bool((d_out == GUARD).all())
    return (("ERR", L.ZSTD_getErrorCode(r)) if L.ZSTD_isError(r) else bytes(d_out[GAP:GAP + r].cpu().numpy())), untouched


def _same_as_single(entries, caps, batch_ctx, single_ctx, contents=None):
    got, _, _ = batch(batch_ctx, entries, caps)
    for i, (e, c) in enumerate(zip(entries, caps)):
        want, _ = single(single_ctx, e, c)
        assert got[i] == want, (i, got[i] if isinstance(got[i], tuple) else len(got[i]), want if isinstance(want, tuple) else len(want))
        if contents is not None:
            assert got[i] == contents[i], i
    return got


def _record_frames(dict_bytes):
    torch = _torch()
    data, offs, sizes = _records(nb=3000)
    cap = sum(zstd_b200.ZSTD_compressBound(s) + 64 for s in sizes)
    d_src, d_c = _dev(data), torch.zeros(cap, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    total, cs = zstd_b200.ZSTD_CCtx().compress_frames(d_c.data_ptr(), cap, d_src.data_ptr(), offs, sizes, level=3, dict_bytes=dict_bytes)
    blob = bytes(d_c[:total].cpu().numpy())
    starts = [sum(cs[:i]) for i in range(len(cs))]
    return [blob[o:o + c] for o, c in zip(starts, cs)], [data[o:o + s] for o, s in zip(offs, sizes)]


@gpu
@needs_ref
@pytest.mark.parametrize("dictionary", ["none", "raw", "zstd"])
def test_records_match_the_single_call_and_the_reference(dictionary):
    zd = zref.golden_input(ZDICT)
    d = {"none": None, "raw": zd[8:], "zstd": zd}[dictionary]
    frames, recs = _record_frames(d)
    b, s = zstd_b200.ZSTD_DCtx(), zstd_b200.ZSTD_DCtx()
    if d is not None:
        dd = zstd_b200.ZSTD_DDict(d)
        b.ref_ddict(dd); s.ref_ddict(dd)
    got, _, _ = batch(b, frames, [len(r) for r in recs])
    assert got == recs
    for i in range(0, len(frames), 97):                      # a sample against the single call and the reference decoder
        assert single(s, frames[i], len(recs[i]))[0] == recs[i], i
        ref = zref.ref_decompress(frames[i], len(recs[i])) if d is None else zref.ref_decompress_using_dict(frames[i], d, len(recs[i]))
        assert ref == recs[i], i


@gpu
@needs_ref
def test_mixed_entries():
    ctx = zstd_b200.ZSTD_CCtx()
    srcs = [b"", b"", b"q", zref.synthetic((128 << 10) + 1, seed=3, match_prob=0.6), zref.synthetic(3 << 20, seed=4, match_prob=0.7),
            zref.synthetic(5000, seed=5, match_prob=0.5)]
    entries = [b"", ctx.compress(b"", 3), ctx.compress(b"q", 3), ctx.compress(srcs[3], 1), ctx.compress(srcs[4], 3), b""]
    entries[-1] = ctx.compress(srcs[5], -5) + _skippable(7) + zref.ref_compress(srcs[3], 3)              # concatenated + skippable
    srcs[-1] = srcs[5] + srcs[3]
    entries += [_skippable(0) + _skippable(100), zref.ref_compress(srcs[4], 19)]
    srcs += [b"", srcs[4]]
    caps = [len(x) + 16 for x in srcs]
    got = _same_as_single(entries, caps, zstd_b200.ZSTD_DCtx(), zstd_b200.ZSTD_DCtx(), srcs)
    for e, want in zip(entries, got):
        if e and not e.startswith(struct.pack("<I", SKIP_MAGIC)):
            assert ref_oneshot(e, len(want) + 16) == want


@gpu
@needs_ref
def test_frames_without_content_size_and_reference_levels():
    entries, srcs = [], []
    for name in ("no-content-size", "streamed", "window-1k-streamed", "streamed-checksums", "max-block-1k"):
        f, s = seqgen.ADVANCED[name]()
        entries.append(f); srcs.append(s)
    src = zref.synthetic(100_000, seed=8, match_prob=0.7)
    for level in range(1, 20):
        entries.append(zref.ref_compress(src, level)); srcs.append(src)
    _same_as_single(entries, [len(s) for s in srcs], zstd_b200.ZSTD_DCtx(), zstd_b200.ZSTD_DCtx(), srcs)


@gpu
@needs_ref
@pytest.mark.timeout(900, method="thread")
def test_fault_isolation():
    """the corrupt inputs of test_decode_invalid.py, each between two good entries: each bad entry's result is the single
    device call's (which that file holds to the reference's verdict with checksums ignored), every good neighbour decodes,
    and the slot of an entry refused before its output is placed keeps its guard bytes"""
    L = _lib()
    zd = zref.golden_input(ZDICT)
    good = zref.synthetic(50_000, 80, 0.6)
    good_frame = zref.ref_compress(good, 3)
    cases = constructed() + corpus(CORPUS_GPU, 1)
    groups = {}
    for n, b, c, d in cases:
        groups.setdefault(d, []).append((n, b, c, d))
    groups.setdefault(zd, []).extend((n, b, c, zd) for n, b, c, d in cases[:60] if d is None)   # decoded with a dictionary they do not name
    refused = 0
    for dic, mine in groups.items():
        b, s = zstd_b200.ZSTD_DCtx(), zstd_b200.ZSTD_DCtx()
        entries, caps = [good_frame], [len(good)]
        for _, buf, cap, _ in mine:
            entries += [buf, good_frame]; caps += [cap, len(good)]
        if dic is not None:
            b.load_dictionary(dic)
        got, d_out, do = batch(b, entries, caps)
        for i in range(0, len(entries), 2):
            assert got[i] == good, ("good neighbour", i)
        for k, (name, buf, cap, d) in enumerate(mine):
            i = 2 * k + 1
            torch = _torch()
            d_in = _dev(b"\x77" + buf)
            ref_out = torch.full((cap + 2 * GAP,), GUARD, dtype=torch.uint8, device="cuda")
            torch.cuda.synchronize()
            r = L.ZSTDB200_decompressDevice_usingDict(s._h, ref_out.data_ptr() + GAP, cap, d_in.data_ptr() + 1, len(buf), dic, len(dic) if dic else 0, None)
            torch.cuda.synchronize()
            want = ("ERR", L.ZSTD_getErrorCode(r)) if L.ZSTD_isError(r) else bytes(ref_out[GAP:GAP + r].cpu().numpy())
            assert got[i] == want, (name, got[i] if isinstance(got[i], tuple) else len(got[i]), want if isinstance(want, tuple) else len(want))
            if isinstance(want, tuple) and bool((ref_out == GUARD).all()):
                refused += 1
                assert bool((d_out[do[i]:do[i] + cap] == GUARD).all()), (name, "slot written although the entry was refused before placement")
    assert refused > 100


@gpu
def test_capacity_too_small_fails_that_entry_alone():
    ctx = zstd_b200.ZSTD_CCtx()
    srcs = [zref.synthetic(n, seed=41 + n % 7, match_prob=0.6) for n in (400_000, 70_000, 5000)]
    entries = [ctx.compress(x, 3) for x in srcs]
    got, d_out, do = batch(zstd_b200.ZSTD_DCtx(), entries, [len(srcs[0]), len(srcs[1]) - 1, len(srcs[2])])
    assert got == [srcs[0], ("ERR", 70), srcs[2]]
    assert bool((d_out[do[1]:do[1] + len(srcs[1]) - 1] == GUARD).all())


@gpu
def test_entry_past_the_workspace_fails_alone():
    """an entry of far more blocks than the workspace holds, between 1500 good entries in front and 1500 behind (chunks of
    the entry scan that fit whole, and the one admitted entry by entry): it alone gets 66, and takes no room from the
    entries behind it"""
    n = 40_000                                               # empty raw blocks: 3 bytes each, far more than B + nbEntries
    many = struct.pack("<IBB", 0xFD2FB528, 0, 0) + b"\0\0\0" * (n - 1) + b"\1\0\0"
    ctx = zstd_b200.ZSTD_CCtx()
    srcs = [zref.synthetic(64 + i % 7, seed=i, match_prob=0.6) for i in range(3000)]
    frames = [ctx.compress(x, 1) for x in srcs]
    entries = frames[:1500] + [many] + frames[1500:] + [b""]
    caps = [len(x) for x in srcs[:1500]] + [64] + [len(x) for x in srcs[1500:]] + [16]
    src_size = sum(len(e) + 1 for e in entries)
    assert src_size // 16 + sum(caps) // 1024 + 1024 + len(entries) < n          # B + nbEntries blocks
    got, d_out, do = batch(zstd_b200.ZSTD_DCtx(), entries, caps)
    assert got == srcs[:1500] + [("ERR", 66)] + srcs[1500:] + [b""]
    assert single(zstd_b200.ZSTD_DCtx(), many, 64)[0] == b""
    assert bool((d_out[do[1500]:do[1500] + 64] == GUARD).all())


@gpu
def test_refusals():
    torch = _torch()
    f = zstd_b200.ZSTD_CCtx().compress(zref.synthetic(5000, seed=1), 3)
    d_src = _dev(f)
    d_out = torch.zeros(20_000, dtype=torch.uint8, device="cuda")
    res = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    dctx = zstd_b200.ZSTD_DCtx()
    n = len(f)

    def code(do, dc, so, ss, cap=20_000):
        with pytest.raises(zstd_b200.ZstdError) as e:
            dctx.decompress_frames(d_out.data_ptr(), cap, do, dc, d_src.data_ptr(), n, so, ss)
        with pytest.raises(zstd_b200.ZstdError) as e2:
            dctx.decompress_frames_async(d_out.data_ptr(), cap, do, dc, d_src.data_ptr(), n, so, ss, res.data_ptr())
        assert e.value.code == e2.value.code
        return e.value.code

    assert code([0], [5000], [1], [n]) == 42                 # source range past srcSize
    assert code([0], [5000], [n + 1], [0]) == 42
    assert code([15_001], [5000], [0], [n]) == 42            # slot past dstCapacity
    assert code([6000, 0], [5000, 5000], [0, 0], [n, n]) == 42                 # not ascending
    assert code([0, 4999], [5000, 5000], [0, 0], [n, n]) == 42                 # overlapping
    r, per = dctx.decompress_frames(d_out.data_ptr(), 20_000, [0, 5000], [5000, 5000], d_src.data_ptr(), n, [0, 0], [n, n])
    assert per == [5000, 5000] and r == 10_000               # touching slots and a shared source are fine
    for kind in ("sync", "async"):
        dctx.ref_prefix(zref.synthetic(50_000, seed=2))
        with pytest.raises(zstd_b200.ZstdError) as e:
            if kind == "sync":
                dctx.decompress_frames(d_out.data_ptr(), 20_000, [0], [5000], d_src.data_ptr(), n, [0], [n])
            else:
                dctx.decompress_frames_async(d_out.data_ptr(), 20_000, [0], [5000], d_src.data_ptr(), n, [0], [n], res.data_ptr())
        assert e.value.code == 40
        r, per = dctx.decompress_frames(d_out.data_ptr(), 20_000, [0], [5000], d_src.data_ptr(), n, [0], [n])   # the prefix was forgotten
        assert r == 5000
    L = zstd_b200.lib()
    one = (ctypes.c_size_t * 1)
    assert L.ZSTD_getErrorCode(L.ZSTDB200_decompressFramesAsync(dctx._h, d_out.data_ptr(), 20_000, one(0), one(5000), d_src.data_ptr(), n,
                                                                one(0), one(n), 1, None, None, None)) == 1
    assert dctx.decompress_frames(d_out.data_ptr(), 20_000, [], [], d_src.data_ptr(), n, [], []) == (0, [])
    res.fill_(-1)
    dctx.decompress_frames_async(d_out.data_ptr(), 20_000, [], [], d_src.data_ptr(), n, [], [], res.data_ptr())
    torch.cuda.synchronize()
    assert _u64(res) == 0


@gpu
def test_graph_capture_and_replay():
    torch = _torch()
    ctx = zstd_b200.ZSTD_CCtx()
    k, size = 6, 30_000
    rounds = [[zref.synthetic(size, seed=100 * r + i, match_prob=0.6) for i in range(k)] for r in range(4)]
    frames = [[ctx.compress(x, 1) for x in rs] for rs in rounds]
    slot = max(len(f) for fs in frames for f in fs) + 16
    padded = [b"".join(f + _skippable(slot - len(f) - 8) for f in fs) for fs in frames]
    so, ss, do, dc = [i * slot for i in range(k)], [slot] * k, [i * (size + 8) for i in range(k)], [size] * k
    d_src = _dev(padded[0])
    d_out = torch.zeros(k * (size + 8), dtype=torch.uint8, device="cuda")
    res = torch.zeros(1 + k, dtype=torch.int64, device="cuda")
    dctx = zstd_b200.ZSTD_DCtx()

    def call(stream):
        dctx.decompress_frames_async(d_out.data_ptr(), d_out.numel(), do, dc, d_src.data_ptr(), len(padded[0]), so, ss, res.data_ptr(),
                                     res[1:].data_ptr(), stream)

    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    call(s.cuda_stream)                                      # warm-up
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        call(torch.cuda.current_stream().cuda_stream)
    for r in range(1, 4):
        d_src.copy_(torch.frombuffer(bytearray(padded[r]), dtype=torch.uint8))
        res.fill_(-1)
        g.replay()
        torch.cuda.synchronize()
        assert _u64(res[0]) == k * size and res[1:].tolist() == [size] * k
        assert [bytes(d_out[o:o + size].cpu().numpy()) for o in do] == rounds[r]
    cold = zstd_b200.ZSTD_DCtx()
    g2 = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g2):
        with pytest.raises(zstd_b200.ZstdError) as e:
            cold.decompress_frames_async(d_out.data_ptr(), d_out.numel(), do, dc, d_src.data_ptr(), len(padded[0]), so, ss, res.data_ptr(),
                                         0, torch.cuda.current_stream().cuda_stream)
    assert e.value.code == 60
    torch.cuda.synchronize()


@gpu
def test_calls_run_in_the_order_they_are_made():
    torch = _torch()
    ctx = zstd_b200.ZSTD_CCtx()
    srcs = [zref.synthetic(n, seed=50 + i, match_prob=0.6) for i, n in enumerate((3 << 20, 400_000, 1 << 20, 200_000))]
    fr = [ctx.compress(x, 3) for x in srcs]
    d = [_dev(f) for f in fr]
    dctx = zstd_b200.ZSTD_DCtx()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    outs = [torch.zeros(len(x) + 64, dtype=torch.uint8, device="cuda") for x in srcs]
    res = torch.full((4,), -1, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    with torch.cuda.stream(s1):
        torch.cuda._sleep(SLEEP_CYCLES)

    def frames_call(i, s):                                   # the frame and a 0-byte entry behind it
        dctx.decompress_frames_async(outs[i].data_ptr(), len(srcs[i]) + 64, [0, len(srcs[i])], [len(srcs[i]), 64], d[i].data_ptr(), len(fr[i]),
                                     [0, len(fr[i])], [len(fr[i]), 0], res[i:].data_ptr(), 0, s.cuda_stream)

    frames_call(0, s1)
    dctx.decompress_device_async(outs[1].data_ptr(), len(srcs[1]), d[1].data_ptr(), len(fr[1]), res[1:].data_ptr(), s2.cuda_stream)
    frames_call(2, s2)
    dctx.decompress_device_async(outs[3].data_ptr(), len(srcs[3]), d[3].data_ptr(), len(fr[3]), res[3:].data_ptr(), s1.cuda_stream)
    torch.cuda.synchronize()
    assert [int(x) for x in res.tolist()] == [len(x) for x in srcs]
    assert [bytes(o[:len(x)].cpu().numpy()) for o, x in zip(outs, srcs)] == srcs


@gpu
def test_launches_do_not_depend_on_the_number_of_entries():
    torch = _torch()
    rec = zref.synthetic(64, seed=3, match_prob=0.5)
    f = zstd_b200.ZSTD_CCtx().compress(rec, 1)
    d_src = _dev(f)
    dctx = zstd_b200.ZSTD_DCtx()
    launches = []
    for n in (1, 1024, 131_072):
        d_out = torch.zeros(n * 64, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        r, per = dctx.decompress_frames(d_out.data_ptr(), n * 64, [64 * i for i in range(n)], [64] * n, d_src.data_ptr(), len(f), [0] * n, [len(f)] * n)
        assert r == n * 64 and per == [64] * n
        assert torch.equal(d_out.view(n, 64), torch.frombuffer(bytearray(rec), dtype=torch.uint8).cuda().expand(n, 64))
        launches.append(dctx.stats().launches)
    assert launches[0] > 0 and len(set(launches)) == 1, launches
