"""Batches indexed in device memory: ZSTDB200_findDecompressedSizesAsync against the host size readers entry by entry, and
ZSTDB200_decompressFramesAsync_deviceOffsets against ZSTDB200_decompressFramesAsync with the same values as host arrays
(whole output buffer, per-entry results, verdict), the refusals made in stream order and on the host, graph replays over
layouts written into the arrays between replays, a size-query / cumsum / decode flow captured as one graph, call order
with the context's other calls, and the launch count."""
import ctypes
import glob
import os
import struct

import pytest

import seqgen
import zref
import zstd_b200
from test_decode_invalid import CORPUS_GPU, GUARD, constructed, corpus, needs_ref
from test_gpu_async import SLEEP_CYCLES, ZDICT, _dev, _torch, _u64
from test_gpu_decode_frames import GAP, _layout, _record_frames, _skippable

gpu = pytest.mark.gpu
ERROR, UNKNOWN = 2**64 - 2, 2**64 - 1
SENTINEL = -7                                                # what a per-entry result word holds before a call


def _arr(vals):
    torch = _torch()
    return torch.tensor([int(v) for v in vals] or [0], dtype=torch.int64, device="cuda")


def _words(t):
    return [int(x) & (2**64 - 1) for x in t.cpu().tolist()]


def _device_call(dctx, d_out, cap, do, dc, d_src, src_size, so, ss, res, stream):
    a = [_arr(x) for x in (do, dc, so, ss)]
    dctx.decompress_frames_async_device_offsets(d_out.data_ptr(), cap, a[0].data_ptr(), a[1].data_ptr(), d_src.data_ptr(), src_size,
                                                a[2].data_ptr(), a[3].data_ptr(), len(ss), res.data_ptr(), res[1:].data_ptr(), stream)
    return a                                                 # alive until the caller has synchronised


def both(dctx, entries, caps, layout=None):
    """the host-array and the device-offset call on the same bytes and values, each into a fresh guarded buffer: they must
    agree in the whole output buffer, every per-entry result and the verdict.  Returns (verdict, per-entry results, d_out, dst offsets)"""
    torch = _torch()
    src, so, do, cap = _layout(entries, caps) if layout is None else layout
    ss = [len(e) for e in entries]
    d_src = _dev(src)
    s = torch.cuda.Stream()
    outs = []
    for kind in ("host", "device"):
        d_out = torch.full((cap,), GUARD, dtype=torch.uint8, device="cuda")
        res = torch.full((1 + len(ss),), SENTINEL, dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        if kind == "host":
            dctx.decompress_frames_async(d_out.data_ptr(), cap, do, caps, d_src.data_ptr(), len(src), so, ss, res.data_ptr(),
                                         res[1:].data_ptr(), s.cuda_stream)
        else:
            keep = _device_call(dctx, d_out, cap, do, caps, d_src, len(src), so, ss, res, s.cuda_stream)
        torch.cuda.synchronize()
        outs.append((d_out, res))
    (h_out, h_res), (d_out, d_res) = outs
    assert torch.equal(h_out, d_out), "the output buffers differ"
    assert torch.equal(h_res, d_res), (_words(h_res)[:8], _words(d_res)[:8])
    assert dctx.stats().launches == 13
    w = _words(d_res)
    return w[0], w[1:], d_out, do


def _contents(d_out, do, per):
    return [("ERR", zstd_b200.result_error(r)) if zstd_b200.result_error(r) is not None else bytes(d_out[o:o + r].cpu().numpy())
            for o, r in zip(do, per)]


# ------------------------------------------------------------------ the size query
def _query(dctx, src, so, ss, which=("cs", "bound")):
    torch = _torch()
    d_src, a_so, a_ss = _dev(src), _arr(so), _arr(ss)
    cs = torch.full((max(len(ss), 1),), SENTINEL, dtype=torch.int64, device="cuda")
    bd = torch.full((max(len(ss), 1),), SENTINEL, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    dctx.find_decompressed_sizes_async(d_src.data_ptr(), len(src), a_so.data_ptr(), a_ss.data_ptr(), len(ss),
                                       cs.data_ptr() if "cs" in which else 0, bd.data_ptr() if "bound" in which else 0, s.cuda_stream)
    torch.cuda.synchronize()
    return _words(cs)[:len(ss)], _words(bd)[:len(ss)]


def _size_corpus():
    out = [open(n, "rb").read() for n in sorted(glob.glob(os.path.join(zref.GOLDEN, "decompression*", "*.zst")))]
    for name in ("no-content-size", "streamed", "streamed-checksums", "max-block-1k", "window-1k-streamed"):
        out.append(seqgen.ADVANCED[name]()[0])
    a = zref.synthetic(70_000, seed=5, match_prob=0.6)
    f = zref.ref_compress(a, 3)
    multi = f + _skippable(9) + zref.ref_compress(b"", 1) + zstd_b200.ZSTD_CCtx().compress(a, 1)
    out += [f + f, _skippable(0) + _skippable(300), multi, multi + b"junk", f + b"\x28\xb5\x2f\xfd",
            struct.pack("<IBB", 0xFD2FB528, 0, 31 << 3) + b"\1\0\0",        # windowLog 41: refused
            struct.pack("<IBB", 0xFD2FB528, 0, 21 << 3) + b"\x23\0\0" + b"\xab"]   # windowLog 31, one RLE block of 4
    out += [multi[:n] for n in range(0, len(multi), max(1, len(multi) // 300))]
    return out + [b"", b""]


@gpu
@needs_ref
def test_size_query_equals_the_host_readers():
    entries = _size_corpus()
    src, so, _, _ = _layout(entries, [0] * len(entries))
    ss = [len(e) for e in entries]
    # ranges outside the input: past its end, straddling it, and an offset past it with no bytes
    so += [len(src) + 1, len(src) - 3, len(src), 0]
    ss += [0, 4, 0, len(src) + 1]
    want_cs = [zstd_b200.ZSTD_findDecompressedSize(e) for e in entries] + [ERROR, ERROR, 0, ERROR]
    want_b = [zstd_b200.ZSTD_decompressBound(e) for e in entries] + [ERROR, ERROR, 0, ERROR]
    assert UNKNOWN in want_cs and ERROR in want_cs and len(set(want_b)) > 8
    dctx = zstd_b200.ZSTD_DCtx()
    cs, bd = _query(dctx, src, so, ss)
    assert cs == want_cs and bd == want_b
    assert _query(dctx, src, so, ss, ("cs",)) == (want_cs, [2**64 + SENTINEL] * len(ss))
    assert _query(dctx, src, so, ss, ("bound",)) == ([2**64 + SENTINEL] * len(ss), want_b)


@gpu
def test_size_query_refusals():
    torch = _torch()
    dctx = zstd_b200.ZSTD_DCtx()
    L = zstd_b200.lib()
    d_src, a = _dev(b"\0" * 64), _arr([0, 0, 0])
    out = torch.zeros(4, dtype=torch.int64, device="cuda")

    def code(*args):
        return L.ZSTD_getErrorCode(L.ZSTDB200_findDecompressedSizesAsync(dctx._h, d_src.data_ptr(), 64, *args, None))

    assert code(a.data_ptr(), a.data_ptr(), 3, None, None) == 1               # no output
    assert code(None, a.data_ptr(), 3, out.data_ptr(), None) == 1             # an input array NULL
    assert code(a.data_ptr() + 4, a.data_ptr(), 3, out.data_ptr(), None) == 42
    assert code(a.data_ptr(), a.data_ptr(), 3, None, out.data_ptr() + 4) == 42
    assert L.ZSTDB200_findDecompressedSizesAsync(dctx._h, d_src.data_ptr(), 64, None, None, 0, out.data_ptr(), None, None) == 0


# ------------------------------------------------------------------ the same results as the host form
@gpu
@needs_ref
@pytest.mark.parametrize("dictionary", ["none", "zstd"])
def test_records_equal_the_host_form(dictionary):
    zd = zref.golden_input(ZDICT)
    d = None if dictionary == "none" else zd
    frames, recs = _record_frames(d)
    dctx = zstd_b200.ZSTD_DCtx()
    if d is not None:
        dctx.ref_ddict(zstd_b200.ZSTD_DDict(d))
    r, per, d_out, do = both(dctx, frames, [len(x) for x in recs])
    assert r == sum(len(x) for x in recs) and _contents(d_out, do, per) == recs


@gpu
@needs_ref
def test_mixed_entries():
    ctx = zstd_b200.ZSTD_CCtx()
    a, b = zref.synthetic((128 << 10) + 1, seed=3, match_prob=0.6), zref.synthetic(3 << 20, seed=4, match_prob=0.7)
    c = zref.synthetic(5000, seed=5, match_prob=0.5)
    streamed, streamed_src = seqgen.ADVANCED["streamed-checksums"]()
    entries = [b"", ctx.compress(b"", 3), ctx.compress(b"q", 3), ctx.compress(a, 1), ctx.compress(b, 3),
               ctx.compress(c, -5) + _skippable(7) + zref.ref_compress(a, 3), _skippable(0) + _skippable(100), zref.ref_compress(b, 19),
               streamed]
    srcs = [b"", b"", b"q", a, b, c + a, b"", b, streamed_src]
    r, per, d_out, do = both(zstd_b200.ZSTD_DCtx(), entries, [len(x) + 16 for x in srcs])
    assert _contents(d_out, do, per) == srcs


@gpu
@needs_ref
@pytest.mark.timeout(900, method="thread")
def test_fault_isolation_corpus():
    zd = zref.golden_input(ZDICT)
    good = zref.synthetic(50_000, 80, 0.6)
    good_frame = zref.ref_compress(good, 3)
    cases = constructed() + corpus(CORPUS_GPU, 1)
    groups = {}
    for n, b, c, d in cases:
        groups.setdefault(d, []).append((b, c))
    failed = 0
    for dic, mine in groups.items():
        dctx = zstd_b200.ZSTD_DCtx()
        if dic is not None:
            dctx.load_dictionary(dic)
        entries, caps = [good_frame], [len(good)]
        for buf, cap in mine:
            entries += [buf, good_frame]; caps += [cap, len(good)]
        r, per, d_out, do = both(dctx, entries, caps)
        assert all(per[i] == len(good) for i in range(0, len(entries), 2))
        failed += sum(zstd_b200.result_error(v) is not None for v in per)
    assert failed > 100


@gpu
def test_capacity_and_workspace_verdicts():
    ctx = zstd_b200.ZSTD_CCtx()
    srcs = [zref.synthetic(n, seed=41 + n % 7, match_prob=0.6) for n in (400_000, 70_000, 5000)]
    r, per, _, _ = both(zstd_b200.ZSTD_DCtx(), [ctx.compress(x, 3) for x in srcs], [len(srcs[0]), len(srcs[1]) - 1, len(srcs[2])])
    assert zstd_b200.result_error(per[1]) == 70 and zstd_b200.result_error(r) == 70
    n = 40_000                                               # empty raw blocks: far more than B + nbEntries
    many = struct.pack("<IBB", 0xFD2FB528, 0, 0) + b"\0\0\0" * (n - 1) + b"\1\0\0"
    recs = [zref.synthetic(64 + i % 7, seed=i, match_prob=0.6) for i in range(3000)]
    frames = [ctx.compress(x, 1) for x in recs]
    entries = frames[:1500] + [many] + frames[1500:] + [b""]
    caps = [len(x) for x in recs[:1500]] + [64] + [len(x) for x in recs[1500:]] + [16]
    r, per, d_out, do = both(zstd_b200.ZSTD_DCtx(), entries, caps)
    assert _contents(d_out, do, per) == recs[:1500] + [("ERR", 66)] + recs[1500:] + [b""]


# ------------------------------------------------------------------ refusals
@gpu
def test_refusals_in_stream_order():
    torch = _torch()
    f = zstd_b200.ZSTD_CCtx().compress(zref.synthetic(5000, seed=1), 3)
    d_src = _dev(f)
    n = len(f)
    dctx = zstd_b200.ZSTD_DCtx()

    def verdict(do, dc, so, ss, cap=20_000):
        d_out = torch.full((cap,), GUARD, dtype=torch.uint8, device="cuda")
        res = torch.full((1 + len(ss),), SENTINEL, dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        keep = _device_call(dctx, d_out, cap, do, dc, d_src, n, so, ss, res, 0)
        torch.cuda.synchronize()
        untouched = bool((d_out == GUARD).all()) and res[1:].tolist() == [SENTINEL] * len(ss)
        return zstd_b200.result_error(_u64(res[0])), untouched

    good = ([0, 5000], [5000, 5000], [0, 0], [n, n])
    refused = (42, True)
    assert verdict([0, 5000], [5000, 5000], [0, 1], [n, n]) == refused                # a source range past srcSize
    assert verdict([0, 5000], [5000, 5000], [0, n + 1], [n, 0]) == refused
    assert verdict([0, 15_001], [5000, 5000], [0, 0], [n, n]) == refused         # a slot past dstCapacity
    assert verdict([0, 4999], [5000, 5000], [0, 0], [n, n]) == refused           # overlapping slots
    assert verdict([6000, 0], [5000, 5000], [0, 0], [n, n]) == refused           # descending slots
    assert verdict(*good) == (None, False)                                      # touching slots and a shared source are fine


@gpu
def test_refusals_on_the_host():
    torch = _torch()
    f = zstd_b200.ZSTD_CCtx().compress(zref.synthetic(5000, seed=1), 3)
    d_src, n = _dev(f), len(f)
    d_out = torch.zeros(20_000, dtype=torch.uint8, device="cuda")
    res = torch.full((2,), SENTINEL, dtype=torch.int64, device="cuda")
    a = _arr([0, 5000, 0, n])
    L = zstd_b200.lib()
    dctx = zstd_b200.ZSTD_DCtx()
    p = a.data_ptr()

    def code(do, dc, so, ss, result=res.data_ptr(), stream=None, ctx=dctx):
        return L.ZSTD_getErrorCode(L.ZSTDB200_decompressFramesAsync_deviceOffsets(ctx._h, d_out.data_ptr(), 20_000, do, dc, d_src.data_ptr(),
                                                                                 n, so, ss, 1, None, result, stream))

    torch.cuda.synchronize()
    assert code(None, p + 8, p + 16, p + 24) == 1
    assert code(p, p + 8, p + 16, None) == 1
    assert code(p, p + 8, p + 16, p + 24, result=None) == 1
    assert code(p + 4, p + 8, p + 16, p + 24) == 42
    assert code(p, p + 8, p + 20, p + 24) == 42
    dctx.ref_prefix(zref.synthetic(50_000, seed=2))
    assert code(p, p + 8, p + 16, p + 24) == 40
    assert code(p, p + 8, p + 16, p + 24) == 0                                  # the prefix was forgotten
    torch.cuda.synchronize()
    assert _u64(res[0]) == 5000
    cold = zstd_b200.ZSTD_DCtx()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        c = code(p, p + 8, p + 16, p + 24, stream=torch.cuda.current_stream().cuda_stream, ctx=cold)
    assert c == 60
    torch.cuda.synchronize()


# ------------------------------------------------------------------ capture
@gpu
def test_graph_replays_the_layout_the_arrays_hold():
    torch = _torch()
    ctx = zstd_b200.ZSTD_CCtx()
    k = 12
    recs = [zref.synthetic(20_000 + 1000 * i, seed=200 + i, match_prob=0.6) for i in range(k)]
    frames = [ctx.compress(x, 1) for x in recs]
    src, so, _, _ = _layout(frames, [0] * k)
    d_src = _dev(src)
    cap = sum(len(x) + GAP for x in recs) + GAP
    d_out = torch.full((cap,), GUARD, dtype=torch.uint8, device="cuda")
    res = torch.full((1 + k,), SENTINEL, dtype=torch.int64, device="cuda")
    a_do, a_dc, a_so, a_ss = (torch.zeros(k, dtype=torch.int64, device="cuda") for _ in range(4))
    dctx, other = zstd_b200.ZSTD_DCtx(), zstd_b200.ZSTD_DCtx()

    def layout(order, nb):
        """entries order[:nb] in slots one behind the other, then empty entries"""
        lo, ls, ldo, ldc, pos = [], [], [], [], GAP
        for j, i in enumerate(order):
            real = j < nb
            lo.append(so[i]); ls.append(len(frames[i]) if real else 0)
            ldo.append(pos); ldc.append(len(recs[i]) if real else 0)
            pos += (len(recs[i]) if real else 0) + GAP
        return ldo, ldc, lo, ls

    def write(lay):
        for t, v in zip((a_do, a_dc, a_so, a_ss), lay):
            t.copy_(torch.tensor(v, dtype=torch.int64))

    def call(stream):
        dctx.decompress_frames_async_device_offsets(d_out.data_ptr(), cap, a_do.data_ptr(), a_dc.data_ptr(), d_src.data_ptr(), len(src),
                                                    a_so.data_ptr(), a_ss.data_ptr(), k, res.data_ptr(), res[1:].data_ptr(), stream)

    write(layout(list(range(k)), k))
    torch.cuda.synchronize()
    call(torch.cuda.Stream().cuda_stream)                    # sizes the context
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        call(torch.cuda.current_stream().cuda_stream)
    perm = [5, 2, 11, 0, 7, 3, 9, 1, 10, 4, 8, 6]
    for lay in (layout([1, 3, 5, 7, 9, 11, 0, 2, 4, 6, 8, 10], 6), layout(perm, k), layout(perm, 4)):
        write(lay)
        d_out.fill_(GUARD); res.fill_(SENTINEL)
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        got_out, got_res = d_out.clone(), res.clone()
        d_out.fill_(GUARD); res.fill_(SENTINEL)
        torch.cuda.synchronize()
        other.decompress_frames_async(d_out.data_ptr(), cap, lay[0], lay[1], d_src.data_ptr(), len(src), lay[2], lay[3], res.data_ptr(),
                                      res[1:].data_ptr(), 0)
        torch.cuda.synchronize()
        assert torch.equal(got_out, d_out) and torch.equal(got_res, res)
        nb = sum(1 for x in lay[3] if x)
        assert _u64(got_res[0]) == sum(lay[1]) and nb in (4, 6, 12)
        order = [so.index(x) for x in lay[2]]
        assert [bytes(got_out[o:o + c].cpu().numpy()) for o, c in zip(lay[0], lay[1])] == [recs[i] if c else b"" for i, c in zip(order, lay[1])]


@gpu
def test_size_query_cumsum_and_decode_as_one_graph():
    """the device-only flow: sizes from the headers, slot offsets from their prefix sum, the decode; captured as one graph,
    so no host read stands between the steps"""
    torch = _torch()
    ctx = zstd_b200.ZSTD_CCtx()
    k = 300
    recs = [zref.synthetic(500 + 37 * i, seed=300 + i, match_prob=0.6) for i in range(k)]
    frames = [ctx.compress(x, 1) for x in recs]
    src, so, _, _ = _layout(frames, [0] * k)
    d_src, a_so, a_ss = _dev(src), _arr(so), _arr([len(f) for f in frames])
    cap = sum(len(x) for x in recs)
    d_out = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    sizes, offs, incl = (torch.zeros(k, dtype=torch.int64, device="cuda") for _ in range(3))
    res = torch.full((1 + k,), SENTINEL, dtype=torch.int64, device="cuda")
    dctx = zstd_b200.ZSTD_DCtx()

    def flow(stream):
        dctx.find_decompressed_sizes_async(d_src.data_ptr(), len(src), a_so.data_ptr(), a_ss.data_ptr(), k, sizes.data_ptr(), 0, stream)
        torch.cumsum(sizes, 0, out=incl)
        torch.sub(incl, sizes, out=offs)
        dctx.decompress_frames_async_device_offsets(d_out.data_ptr(), cap, offs.data_ptr(), sizes.data_ptr(), d_src.data_ptr(), len(src),
                                                    a_so.data_ptr(), a_ss.data_ptr(), k, res.data_ptr(), res[1:].data_ptr(), stream)

    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        flow(s.cuda_stream)                                  # sizes the context
    torch.cuda.synchronize()
    assert bytes(d_out.cpu().numpy()) == b"".join(recs)
    d_out.zero_(); sizes.zero_(); res.fill_(SENTINEL)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        flow(torch.cuda.current_stream().cuda_stream)
    g.replay()
    torch.cuda.synchronize()
    assert _u64(res[0]) == cap and sizes.tolist() == [len(x) for x in recs]
    assert bytes(d_out.cpu().numpy()) == b"".join(recs)


# ------------------------------------------------------------------ order and launches
@gpu
def test_calls_run_in_the_order_they_are_made():
    torch = _torch()
    ctx = zstd_b200.ZSTD_CCtx()
    srcs = [zref.synthetic(n, seed=50 + i, match_prob=0.6) for i, n in enumerate((3 << 20, 400_000, 1 << 20, 200_000, 600_000))]
    fr = [ctx.compress(x, 3) for x in srcs]
    d = [_dev(f) for f in fr]
    dctx = zstd_b200.ZSTD_DCtx()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    outs = [torch.zeros(len(x) + 64, dtype=torch.uint8, device="cuda") for x in srcs]
    res = torch.full((len(srcs) + 1,), -1, dtype=torch.int64, device="cuda")
    arrays = {i: [_arr(x) for x in ([0, len(srcs[i])], [len(srcs[i]), 64], [0, len(fr[i])], [len(fr[i]), 0])] for i in (0, 2)}
    torch.cuda.synchronize()
    with torch.cuda.stream(s1):
        torch.cuda._sleep(SLEEP_CYCLES)

    def device_call(i, s):                                   # the frame and a 0-byte entry behind it
        a = arrays[i]
        dctx.decompress_frames_async_device_offsets(outs[i].data_ptr(), len(srcs[i]) + 64, a[0].data_ptr(), a[1].data_ptr(), d[i].data_ptr(),
                                                    len(fr[i]), a[2].data_ptr(), a[3].data_ptr(), 2, res[i:].data_ptr(), 0, s.cuda_stream)

    device_call(0, s1)                                       # behind the sleep on s1
    dctx.decompress_device_async(outs[1].data_ptr(), len(srcs[1]), d[1].data_ptr(), len(fr[1]), res[1:].data_ptr(), s2.cuda_stream)
    device_call(2, s2)
    assert dctx.stats().launches == 13
    dctx.decompress_frames_async(outs[3].data_ptr(), len(srcs[3]) + 64, [0, len(srcs[3])], [len(srcs[3]), 64], d[3].data_ptr(), len(fr[3]),
                                 [0, len(fr[3])], [len(fr[3]), 0], res[3:].data_ptr(), 0, s1.cuda_stream)
    dctx.decompress_device_async(outs[4].data_ptr(), len(srcs[4]), d[4].data_ptr(), len(fr[4]), res[4:].data_ptr(), s2.cuda_stream)
    torch.cuda.synchronize()
    assert [int(x) for x in res[:len(srcs)].tolist()] == [len(x) for x in srcs]
    assert [bytes(o[:len(x)].cpu().numpy()) for o, x in zip(outs, srcs)] == srcs
