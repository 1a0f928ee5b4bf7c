"""Batch decompression with a dictionary per entry (ZSTDB200_decompressFrames[Async]_usingDDicts): every entry decoded with
the bytes and result ZSTDB200_decompressDevice gives it on a context whose sticky dictionary is that entry's DDict, each
dictionary-dependent step reading its own entry's dictionary, dictionary errors failing alone, the refusals, first use,
graph capture, two threads and a launch count that does not depend on the number of dictionaries.  The first tests need no
GPU."""
import ctypes
import threading

import pytest

import dfastgen
import zref
import zstd_b200
import seqgen
from bench_cdicts import with_id
from test_decode_invalid import GUARD, corpus, needs_ref
from test_gpu_async import ZDICT, _dev, _torch, _u64
from test_gpu_decode_frames import _layout, _slot, single


# ------------------------------------------------------------------ no GPU needed
def test_symbols_are_exported():
    L = zstd_b200.lib()
    assert hasattr(L, "ZSTDB200_decompressFrames_usingDDicts") and hasattr(L, "ZSTDB200_decompressFramesAsync_usingDDicts")


def _one_entry(async_call, d_result):
    L = zstd_b200.lib()
    d = L.ZSTD_createDCtx()
    one = (ctypes.c_size_t * 1)(0)
    ten = (ctypes.c_size_t * 1)(10)
    dds = (ctypes.c_void_p * 1)(None)
    try:
        if async_call:
            r = L.ZSTDB200_decompressFramesAsync_usingDDicts(d, 4096, 100, one, (ctypes.c_size_t * 1)(100), 8192, 10, one, ten, 1, dds,
                                                             None, d_result, None)
        else:
            r = L.ZSTDB200_decompressFrames_usingDDicts(d, 4096, 100, one, (ctypes.c_size_t * 1)(100), 8192, 10, one, ten, 1, dds, None, None)
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


def batch(dctx, entries, caps, ddicts):
    """both calls on the same bytes with ddicts: [(result per entry)], a result being the bytes or ("ERR", code).  Both calls
    agree in bytes and sizes, keep every guard byte outside the slots, and give the lowest failing entry's code or the sum"""
    torch = _torch()
    src, so, do, cap = _layout(entries, caps)
    d_src = _dev(src)
    sizes = [len(e) for e in entries]
    outs = []
    for kind in ("sync", "async"):
        d_out = torch.full((cap,), GUARD, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        if kind == "sync":
            r, per = dctx.decompress_frames_using_ddicts(d_out.data_ptr(), cap, do, caps, d_src.data_ptr(), len(src), so, sizes, ddicts)
        else:
            res = torch.full((1 + len(entries),), -1, dtype=torch.int64, device="cuda")
            s = torch.cuda.Stream()
            dctx.decompress_frames_async_using_ddicts(d_out.data_ptr(), cap, do, caps, d_src.data_ptr(), len(src), so, sizes, ddicts,
                                                      res.data_ptr(), res[1:].data_ptr(), s.cuda_stream)
            torch.cuda.synchronize()
            r, per = _u64(res[0]), [int(x) & (2**64 - 1) for x in res[1:].cpu().tolist()]
        assert dctx.stats().launches == 12
        mask = torch.ones(cap, dtype=torch.bool, device="cuda")
        for o, c in zip(do, caps):
            mask[o:o + c] = False
        assert bool((d_out[mask] == GUARD).all()), (kind, "bytes outside the slots changed")
        bad = [i for i, v in enumerate(per) if zstd_b200.result_error(v) is not None]
        assert r == (per[bad[0]] if bad else sum(per)), kind
        outs.append([_slot(d_out, o, v) for o, v in zip(do, per)])
    assert outs[0] == outs[1], "the synchronous and the stream-ordered call differ"
    return outs[0]


def _single(dctx, entry, cap, dd):
    dctx.ref_ddict(dd)
    return single(dctx, entry, cap)[0]


def _without_dict_id(frame):
    """the same frame with its Dictionary_ID field removed: it names no dictionary, so the decoder takes the one it is given"""
    fhd = frame[4]
    n = (0, 1, 2, 4)[fhd & 3]
    at = 5 + (0 if fhd & 0x20 else 1)
    return frame[:4] + bytes([fhd & ~3]) + frame[5:at] + frame[at + n:]


def _first_block(frame):
    """seqgen.block_layout of a frame's first block, None when it is not a compressed block"""
    fhd = frame[4]
    single_segment, fcs_flag = (fhd >> 5) & 1, fhd >> 6
    p = 5 + (0 if single_segment else 1) + (0, 1, 2, 4)[fhd & 3] + (single_segment, 2, 4, 8)[fcs_flag]
    bh = int.from_bytes(frame[p:p + 3], "little")
    return seqgen.block_layout(frame[p + 3:p + 3 + (bh >> 3)]) if (bh >> 1) & 3 == 2 else None


# start repcodes of the trained dictionaries, one triple each: the trainer writes the format's 1, 4, 8, which no dictionary
# would then tell apart from none
REPS = [(3001, 1307, 2203), (2711, 997, 1601), (1999, 2503, 811), (1409, 3307, 2099)]


def _entropy(d):
    """a zstd-format dictionary's Huffman tree description and its three FSE table descriptions"""
    tables = d[8:len(d) - len(seqgen.dict_content(d)) - 12]
    h = tables[0]
    huf = 1 + (h if h < 128 else (h - 127 + 1) // 2)                  # FSE-compressed weights, or 4-bit ones
    return tables[:huf], tables[huf:]


def _trained(seed, k):
    """k zstd-format dictionaries trained on different data, under their own repcodes (REPS): content, Huffman and FSE
    tables and repcodes all differ from one dictionary to the next.  Returns [(dictionary, the data it was trained on)]."""
    out = []
    for i in range(k):
        samples = zref.synthetic(600 * 1024, seed=seed + i, match_prob=0.55)
        d = dfastgen.patch_reps(with_id(zref.train_dict(samples, 1024, 600, 8192), 1000 + i), REPS[i])
        out.append((d, samples))
    huf, fse = zip(*(_entropy(d) for d, _ in out))
    assert len(set(huf)) == k and len(set(fse)) == k, "two trained dictionaries share a Huffman or an FSE description"
    return out


def _rep_frames(trained):
    """per dictionary, a frame of explicit sequences whose first three code the dictionary's repcodes (repcode 1 after
    literals, repcode 1 without literals, which is the second slot, and repcode 3), reaching into its content; the dictID
    removed.  Each is checked with the reference decoder: under the same dictionary with the format's start repcodes
    (1, 4, 8) it decodes to other bytes or fails, so its decoding depends on the dictionary's repcodes."""
    entries, contents = [], []
    for k, (d, _) in enumerate(trained):
        r = REPS[k]
        frame, src, _ = seqgen._one([([(7, r[0], 16), (0, r[1], 9), (3, r[2], 12), (5, 40, 30)], 11)], 70 + k, dict=d)
        frame = _without_dict_id(frame)
        assert zref.ref_decompress_using_dict(frame, d, len(src)) == src
        try:
            other = zref.ref_decompress_using_dict(frame, dfastgen.patch_reps(d, (1, 4, 8)), len(src))
        except ValueError:
            other = None
        assert other != src, k
        entries.append(frame)
        contents.append(src)
    return entries, contents


@gpu
@needs_ref
def test_round_trip_of_compress_frames_using_cdicts():
    """records of 1 KiB .. 1 MiB written by compressFrames_usingCDicts against zstd-format dictionaries under different
    IDs, raw-content dictionaries and none: each decodes to its record, as decompressDevice with refDDict and the
    reference's ZSTD_decompress_usingDict decode it"""
    torch = _torch()
    zd = zref.golden_input(ZDICT)
    dicts = [with_id(zd, 7000 + i) for i in range(3)] + [zref.synthetic(20_000, seed=40 + i, match_prob=0.5) for i in range(2)] + [None]
    sizes = [1024, 4096, 65536, 1 << 20, 3000, 200_000]
    recs = [zref.synthetic(s, seed=60 + i, match_prob=0.6) for i, s in enumerate(sizes * 2)]
    which = [i % len(dicts) for i in range(len(recs))]
    cds = {i: zstd_b200.ZSTD_CDict(d, 3) for i, d in enumerate(dicts) if d is not None}
    dds = {i: zstd_b200.ZSTD_DDict(d) for i, d in enumerate(dicts) if d is not None}
    blob = b"".join(recs)
    offs, pos = [], 0
    for r in recs:
        offs.append(pos)
        pos += len(r)
    cap = sum(zstd_b200.ZSTD_compressBound(len(r)) + 64 for r in recs)
    d_src, d_c = _dev(blob), torch.zeros(cap, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    cctx = zstd_b200.ZSTD_CCtx()
    total, cs = cctx.compress_frames_using_cdicts(d_c.data_ptr(), cap, d_src.data_ptr(), offs, [len(r) for r in recs],
                                                  [cds.get(w) for w in which], level=3)
    c = bytes(d_c[:total].cpu().numpy())
    frames = [c[sum(cs[:i]):sum(cs[:i + 1])] for i in range(len(cs))]
    ddicts = [dds.get(w) for w in which]
    got = batch(zstd_b200.ZSTD_DCtx(), frames, [len(r) + 5 for r in recs], ddicts)
    one = zstd_b200.ZSTD_DCtx()
    for i, (f, r) in enumerate(zip(frames, recs)):
        assert got[i] == r, i
        assert _single(one, f, len(r) + 5, ddicts[i]) == r, i
        d = dicts[which[i]]
        want = zref.ref_decompress_using_dict(f, d, len(r)) if d is not None else zref.ref_decompress(f, len(r))
        assert want == r, i


def _dict_frames(trained, per):
    """per records for each dictionary, compressed by the reference against it, the dictID removed from every frame"""
    entries, contents, owner = [], [], []
    for j in range(per):
        for k, (d, samples) in enumerate(trained):
            rec = samples[(j * 5 + 1) * 1024:(j * 5 + 2) * 1024 + 517 * j]
            entries.append(_without_dict_id(zref.ref_compress_using_dict(rec, d, 3)))
            contents.append(rec)
            owner.append(k)
    return entries, contents, owner


@gpu
@needs_ref
def test_each_step_reads_its_own_entrys_dictionary():
    """neighbouring entries against dictionaries that differ in content, Huffman and FSE tables and repcodes, in frames
    that name no dictionary: each decodes exactly with its own; with the dictionaries rotated by one, every entry comes out
    different or fails"""
    trained = _trained(300, 4)
    entries, contents, owner = _dict_frames(trained, 6)
    reps, rep_contents = _rep_frames(trained)                         # first sequences that use the dictionary's repcodes
    entries += reps; contents += rep_contents; owner += list(range(len(trained)))
    straddle, src, d = seqgen.dict_straddle("zdict")                  # matches that begin in the content and run into the frame
    entries.append(_without_dict_id(straddle)); contents.append(src)
    dds = [zstd_b200.ZSTD_DDict(t[0]) for t in trained] + [zstd_b200.ZSTD_DDict(d)]
    owner.append(len(dds) - 1)
    layouts = [f for f in map(_first_block, entries) if f is not None]
    assert any(f["lit_type"] == 3 for f in layouts), "no first block with treeless literals"
    assert any(f["modes"] and 3 in f["modes"] for f in layouts), "no first block with a repeat-mode sequence table"
    caps = [len(c) + 7 for c in contents]
    got = batch(zstd_b200.ZSTD_DCtx(), entries, caps, [dds[o] for o in owner])
    assert got == contents
    rotated = [dds[(o + 1) % len(dds)] for o in owner]
    got = batch(zstd_b200.ZSTD_DCtx(), entries, caps, rotated)
    for i, (g, c) in enumerate(zip(got, contents)):
        assert g != c, i


@gpu
@needs_ref
def test_fault_isolation():
    """frames that name another dictID (32) and corrupt entries fail alone between good entries with dictionaries"""
    trained = _trained(500, 2)
    good, contents, owner = _dict_frames(trained, 3)
    named = [zref.ref_compress_using_dict(c, trained[o][0], 3) for c, o in zip(contents, owner)]
    dds = [zstd_b200.ZSTD_DDict(t[0]) for t in trained]
    bad = corpus(len(good), 5)
    entries, caps, ddicts, want = [], [], [], []
    for i in range(len(good)):
        _, buf, cap, d = bad[i]
        entries += [named[i], buf, good[i]]
        caps += [len(contents[i]) + 3, cap, len(contents[i]) + 3]
        ddicts += [dds[(owner[i] + 1) % 2], zstd_b200.ZSTD_DDict(d) if d else None, dds[owner[i]]]
        want += [("ERR", 32), None, contents[i]]
    got = batch(zstd_b200.ZSTD_DCtx(), entries, caps, ddicts)
    one = zstd_b200.ZSTD_DCtx()
    for i, (g, w) in enumerate(zip(got, want)):
        if w is not None:
            assert g == w, i
        assert g == _single(one, entries[i], caps[i], ddicts[i]), i


def _uniform(k, n, seed=3):
    """n 1 KiB records compressed against k dictionaries (config 5's shape at a small scale): frames, records, DDicts"""
    zd = zref.golden_input(ZDICT)
    dicts = [with_id(zd, 50_000 + i) for i in range(k)]
    recs = [zref.synthetic(1024, seed=seed * 100_000 + i, match_prob=0.5) for i in range(n)]
    frames = [zref.ref_compress_using_dict(r, dicts[i % k], 1) for i, r in enumerate(recs)]
    return frames, recs, [zstd_b200.ZSTD_DDict(d) for d in dicts]


@gpu
@needs_ref
@pytest.mark.parametrize("k", [1, 64, 1024])
def test_launches_do_not_depend_on_the_number_of_dictionaries(k):
    frames, recs, dds = _uniform(k, 2048)
    got = batch(zstd_b200.ZSTD_DCtx(), frames, [1024] * len(frames), [dds[i % k] for i in range(len(frames))])
    assert got == recs


@gpu
@needs_ref
def test_first_use_uploads_all_and_a_second_call_copies_nothing():
    torch = _torch()
    frames, recs, dds = _uniform(256, 1024, seed=9)
    src, so, do, cap = _layout(frames, [1024] * len(frames))
    d_src, d_out = _dev(src), torch.zeros(cap, dtype=torch.uint8, device="cuda")
    dctx = zstd_b200.ZSTD_DCtx()
    ddicts = [dds[i % 256] for i in range(len(frames))]
    r1, _ = dctx.decompress_frames_using_ddicts(d_out.data_ptr(), cap, do, [1024] * len(frames), d_src.data_ptr(), len(src), so,
                                                [len(f) for f in frames], ddicts)
    first = dctx.stats().h2d_bytes
    r2, per = dctx.decompress_frames_using_ddicts(d_out.data_ptr(), cap, do, [1024] * len(frames), d_src.data_ptr(), len(src), so,
                                                  [len(f) for f in frames], ddicts)
    assert r1 == r2 == 1024 * len(frames)
    assert first >= 256 * len(zref.golden_input(ZDICT)), first           # every DDict once, whatever its count of entries
    assert first < 2 * 256 * len(zref.golden_input(ZDICT)), first
    assert dctx.stats().h2d_bytes == 0
    assert [bytes(d_out[o:o + 1024].cpu().numpy()) for o in do] == recs


@gpu
@needs_ref
def test_refusals_write_nothing():
    torch = _torch()
    frames, recs, dds = _uniform(4, 16, seed=11)
    src, so, do, cap = _layout(frames, [1024] * len(frames))
    d_src = _dev(src)
    ss, dc = [len(f) for f in frames], [1024] * len(frames)
    ddicts = [dds[i % 4] for i in range(len(frames))]
    L = zstd_b200.lib()
    dctx = zstd_b200.ZSTD_DCtx()
    d_out = torch.full((cap,), GUARD, dtype=torch.uint8, device="cuda")

    def raw(so_, do_, dc_, prefix=False):
        n = len(frames)
        arr = [(ctypes.c_size_t * n)(*a) for a in (do_, dc_, so_, ss)]
        sizes = (ctypes.c_size_t * n)(*([12345] * n))
        handles = (ctypes.c_void_p * n)(*[d._h for d in ddicts])
        if prefix:
            dctx.ref_prefix(b"some prefix bytes")
        r = L.ZSTDB200_decompressFrames_usingDDicts(dctx._h, d_out.data_ptr(), cap, arr[0], arr[1], d_src.data_ptr(), len(src), arr[2],
                                                    arr[3], n, handles, sizes, None)
        torch.cuda.synchronize()
        assert list(sizes) == [12345] * n
        assert bool((d_out == GUARD).all())
        return L.ZSTD_getErrorCode(r)

    assert raw(so, do, dc, prefix=True) == 40
    assert raw([len(src)] + so[1:], do, dc) == 42                      # a source range outside the input
    assert raw(so, [cap] + do[1:], dc) == 42                           # a slot outside the output
    assert raw(so, [do[1]] + do[1:], dc) == 42                         # overlapping slots
    r, per = dctx.decompress_frames_using_ddicts(d_out.data_ptr(), cap, do, dc, d_src.data_ptr(), len(src), so, ss, ddicts)
    assert r == 1024 * len(frames)                                     # the prefix was forgotten


@gpu
def test_a_ddict_on_another_device():
    torch = _torch()
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU: a DDict resident on another device cannot be made here")
    frames, recs, dds = _uniform(2, 8, seed=13)
    on1 = zstd_b200.ZSTD_DCtx(device=1)
    on1.ref_ddict(dds[0])
    with torch.cuda.device(1):
        single(on1, frames[0], 1024)
    dctx = zstd_b200.ZSTD_DCtx(device=0)
    with pytest.raises(zstd_b200.ZstdError) as e:
        batch(dctx, frames, [1024] * len(frames), [dds[i % 2] for i in range(len(frames))])
    assert e.value.code == 40


@gpu
@needs_ref
def test_graph_capture_and_replay():
    torch = _torch()
    k = 8
    zd = zref.golden_input(ZDICT)
    dicts = [with_id(zd, 60_000 + i) for i in range(k)]
    dds = [zstd_b200.ZSTD_DDict(d) for d in dicts]
    rounds = [[zref.synthetic(1024, seed=1000 * r + i, match_prob=0.5) for i in range(k)] for r in range(3)]
    frames = [[zref.ref_compress_using_dict(x, dicts[i], 1) for i, x in enumerate(rs)] for rs in rounds]
    slot = max(len(f) for fs in frames for f in fs) + 16
    padded = [b"".join(f + b"\x50\x2a\x4d\x18" + (slot - len(f) - 8).to_bytes(4, "little") + bytes(slot - len(f) - 8) for f in fs)
              for fs in frames]
    so, ss, do, dc = [i * slot for i in range(k)], [slot] * k, [i * 1032 for i in range(k)], [1024] * k
    d_src = _dev(padded[0])
    d_out = torch.zeros(k * 1032, dtype=torch.uint8, device="cuda")
    res = torch.zeros(1 + k, dtype=torch.int64, device="cuda")
    dctx = zstd_b200.ZSTD_DCtx()

    def call(ctx, stream, ddicts):
        ctx.decompress_frames_async_using_ddicts(d_out.data_ptr(), d_out.numel(), do, dc, d_src.data_ptr(), len(padded[0]), so, ss, ddicts,
                                                 res.data_ptr(), res[1:].data_ptr(), stream)

    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    call(dctx, s.cuda_stream, dds)                                   # warm-up: sizes the context, makes the DDicts resident
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        call(dctx, torch.cuda.current_stream().cuda_stream, dds)
    for r in range(1, 3):
        d_src.copy_(torch.frombuffer(bytearray(padded[r]), dtype=torch.uint8))
        res.fill_(-1)
        g.replay()
        torch.cuda.synchronize()
        assert _u64(res[0]) == k * 1024 and res[1:].tolist() == [1024] * k
        assert [bytes(d_out[o:o + 1024].cpu().numpy()) for o in do] == rounds[r]
    warm = zstd_b200.ZSTD_DCtx()
    call(warm, s.cuda_stream, dds)
    torch.cuda.synchronize()
    fresh = dds[:-1] + [zstd_b200.ZSTD_DDict(dicts[-1])]
    g2 = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g2):
        with pytest.raises(zstd_b200.ZstdError) as e:
            call(warm, torch.cuda.current_stream().cuda_stream, fresh)
    assert e.value.code == 60
    torch.cuda.synchronize()


@gpu
@needs_ref
def test_two_threads_share_ddicts_in_opposite_orders():
    """fresh DDicts: one thread names them first to last, the other last to first, each on its own context"""
    frames, recs, dds = _uniform(64, 512, seed=17)
    ddicts = [dds[i % 64] for i in range(len(frames))]
    results, errors = {}, []

    def run(name, fs, ds):
        try:
            ctx = zstd_b200.ZSTD_DCtx()
            for _ in range(3):
                results[name] = batch(ctx, fs, [1024] * len(fs), ds)
        except Exception as e:                                       # reported below
            errors.append(e)

    t = [threading.Thread(target=run, args=("a", frames, ddicts)), threading.Thread(target=run, args=("b", frames[::-1], ddicts[::-1]))]
    for x in t:
        x.start()
    for x in t:
        x.join()
    assert not errors, errors
    assert results["a"] == recs and results["b"] == recs[::-1]
