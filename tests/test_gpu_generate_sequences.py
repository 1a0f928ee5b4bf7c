"""ZSTD_generateSequences and ZSTDB200_generateSequencesDevice[Async] on the GPU: the rows are the oracle's per-block stores
(oracle/zb_seqs.c) with the repcodes the frame codes, and fed back to ZSTD_compressSequences they give ZSTD_compress2's
frame byte for byte, in every call form, wave layout, capacity and refusal."""
import functools
import os

import numpy as np
import pytest

import seqexport as sx
import seqgen
import seqoracle as so
import zref
import zstd_b200

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not zref.have_ref(), reason="oracle/_ref/libzstd_ref.so not built")

LEVELS = [1, 2, 3, 4, -1, -3, -7, 9]
DICTS = ["none", "raw", "zdict", "cdict"]
B = 128 << 10
SIZES = [0, 1, 6, 7, B, B + 1, B + 6]


def _datagen(n, p, seed):
    return zref.datagen(n, p, seed) if zref.have_datagen() else zref.synthetic(n, seed, p / 100)


@functools.lru_cache(maxsize=None)
def _input(name):
    if name.startswith("P"):
        return _datagen((1 << 20) + 12345, int(name[1:]), 5)
    if name.startswith("golden:"):
        return zref.golden_input(name[7:])
    if name == "random":
        return zref.random_bytes(300_000, 9)
    if name == "zeros":
        return bytes(300_000)
    return zref.synthetic(int(name[5:]), 13, 0.6)


INPUTS = (["P30", "P50", "P90"] + ["golden:" + f for f in sorted(os.listdir(os.path.join(zref.GOLDEN, "inputs")))]
          + ["random", "zeros"] + [f"size:{n}" for n in SIZES])


@functools.lru_cache(maxsize=None)
def _dict(kind):
    return None if kind == "none" else (zref.golden_input(seqgen.ZDICT) if kind != "raw" else zref.synthetic(40_000, 13, 0.5))


def _ctx(level, kind, checksum=False, dict_id=True):
    c = zstd_b200.ZSTD_CCtx()
    c.set_parameter("compression_level", level)
    if checksum:
        c.set_parameter("checksum_flag", 1)
    if not dict_id:
        c.set_parameter(202, 0)
    d = _dict(kind)
    if kind == "cdict":
        c._cd = zstd_b200.ZSTD_CDict(d, level)              # the CDict's level applies; the context keeps it alive
        c.ref_cdict(c._cd)
    elif d is not None:
        c.load_dictionary(d)
    return c


def _want(src, level, kind):
    d = _dict(kind)
    return sx.fill_rep(so.frame_sequences(src, level, d), sx.dict_rep(d))


def _dev(b):
    return torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda() if b else torch.zeros(1, dtype=torch.uint8, device="cuda")


GUARD = 64


def _rows(d_out, n):
    return d_out[:n * 16].cpu().numpy().view(np.uint32).reshape(-1, 4).copy()


def _device_rows(c, src, cap=None, stream=None):
    cap = zstd_b200.sequence_bound(len(src)) if cap is None else cap
    d_src = _dev(src)
    d_out = torch.full(((cap + GUARD) * 16,), 0xA5, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    err = None
    try:
        n = c.generate_sequences_device(d_out.data_ptr(), cap, d_src.data_ptr(), len(src), stream.cuda_stream if stream else 0)
    except zstd_b200.ZstdError as e:
        err = e.code
    if stream is not None:
        stream.synchronize()
    assert bool((d_out[cap * 16:] == 0xA5).all()), "rows written past the capacity"
    return err if err is not None else _rows(d_out, n)


def _async_rows(c, src, stream, cap=None):
    cap = zstd_b200.sequence_bound(len(src)) if cap is None else cap
    d_src = _dev(src)
    d_out = torch.full(((cap + GUARD) * 16,), 0xA5, dtype=torch.uint8, device="cuda")
    res = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    c.generate_sequences_device_async(d_out.data_ptr(), cap, d_src.data_ptr(), len(src), res.data_ptr(), stream.cuda_stream)
    stream.synchronize()
    r = int(res.cpu().numpy().view(np.uint64)[0])
    assert bool((d_out[cap * 16:] == 0xA5).all()), "rows written past the capacity"
    err = zstd_b200.result_error(r)
    return err if err is not None else _rows(d_out, r)


def _host(c, src):
    try:
        return c.generate_sequences(src)
    except zstd_b200.ZstdError as e:
        return e.code


def _blocks(rows):
    """rows as seqgen's [(sequences (ll, off, ml), trailing)]"""
    out, cur = [], []
    for off, ll, ml, _ in rows.tolist():
        if off == 0 and ml == 0:
            out.append((cur, ll))
            cur = []
        else:
            cur.append((ll, off, ml))
    return out


def _compress_sequences(c, rows, src, explicit):
    c.set_parameter(1008, 1 if explicit else 0)
    return c.compress_sequences(rows if explicit else so.merge_delimiters(rows), src)


@pytest.mark.parametrize("kind", DICTS)
@pytest.mark.parametrize("level", LEVELS)
@pytest.mark.parametrize("name", INPUTS)
def test_oracle_and_round_trip(name, level, kind):
    src = _input(name)
    want = _want(src, level, kind)
    got = _host(_ctx(level, kind), src)
    assert isinstance(got, np.ndarray) and got.shape == want.shape and (got == want).all()
    assert (_device_rows(_ctx(level, kind), src) == want).all()
    s = torch.cuda.Stream()
    assert (_async_rows(_ctx(level, kind), src, s) == want).all()
    for checksum, dict_id in ((False, True), (True, False)):
        c = _ctx(level, kind, checksum, dict_id)
        frame = c.compress2(src)
        assert _compress_sequences(c, got, src, True) == frame
        assert _compress_sequences(c, got, src, False) == frame


@pytest.mark.parametrize("level", [1, 3, -3, 9])
@pytest.mark.parametrize("name", ["P50", "P90", "random", "zeros", "size:7", f"size:{B + 6}"])
def test_device_round_trip(name, level):
    """generateSequencesDevice -> compressSequencesDevice gives compressDevice's frame, without leaving the device"""
    src = _input(name)
    c = _ctx(level, "none")
    cap = zstd_b200.sequence_bound(len(src))
    d_src = _dev(src)
    d_seq = torch.zeros(cap * 16 + 16, dtype=torch.uint8, device="cuda")
    fcap = zstd_b200.ZSTD_compressBound(len(src)) + 64
    d_a = torch.zeros(fcap, dtype=torch.uint8, device="cuda")
    d_b = torch.zeros(fcap, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    n = c.generate_sequences_device(d_seq.data_ptr(), cap, d_src.data_ptr(), len(src))
    c.set_parameter(1008, 1)
    r = c.compress_sequences_device(d_a.data_ptr(), fcap, d_seq.data_ptr(), n, d_src.data_ptr(), len(src))
    w = c.compress_device(d_b.data_ptr(), fcap, d_src.data_ptr(), len(src), level)
    assert r == w and bool((d_a[:r] == d_b[:w]).all())


@needs_ref
@pytest.mark.parametrize("kind", ["none", "raw", "zdict"])
@pytest.mark.parametrize("level", [1, 3, -3, 9])
@pytest.mark.parametrize("name", ["P50", "golden:http", "random", "zeros", "size:6", f"size:{B + 1}"])
def test_reference_accepts_rows(name, level, kind):
    src = _input(name)
    rows = _host(_ctx(level, kind), src)
    frame = seqgen.ref_compress_sequences(_blocks(rows), src, level, _dict(kind))
    assert seqgen.ref_decompress(frame, len(src), _dict(kind)) == src


def test_waves_of_64_blocks(monkeypatch):
    """64 MiB in waves of 64 blocks: the rows of one wave and the oracle's"""
    monkeypatch.setenv("ZSTDB200_WAVE_BLOCKS", "64")
    src = _datagen(64 << 20, 50, 3)
    waves = _device_rows(_ctx(1, "none"), src)
    monkeypatch.delenv("ZSTDB200_WAVE_BLOCKS")
    one = _device_rows(_ctx(1, "none"), src, stream=torch.cuda.Stream())
    assert waves.shape == one.shape and (waves == one).all()
    assert (waves == _want(src, 1, "none")).all()


def test_waves_on_wave_streams():
    """256 MiB with a NULL stream runs as waves on the wave streams: the rows of one wave, and compressDevice's frame back"""
    n = 256 << 20
    src = _datagen(n, 50, 4)
    c = _ctx(1, "none")
    cap = zstd_b200.sequence_bound(n)
    d_src = _dev(src)
    d_seq = torch.zeros(cap * 16, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    cnt = c.generate_sequences_device(d_seq.data_ptr(), cap, d_src.data_ptr(), n)
    assert c.stats().nbBlocks == 2048
    s = torch.cuda.Stream()
    d_one = torch.zeros(cap * 16, dtype=torch.uint8, device="cuda")
    assert c.generate_sequences_device(d_one.data_ptr(), cap, d_src.data_ptr(), n, s.cuda_stream) == cnt
    s.synchronize()
    assert bool((d_seq[:cnt * 16] == d_one[:cnt * 16]).all())
    del d_one
    fcap = zstd_b200.ZSTD_compressBound(n)
    d_a = torch.zeros(fcap, dtype=torch.uint8, device="cuda")
    d_b = torch.zeros(fcap, dtype=torch.uint8, device="cuda")
    c.set_parameter(1008, 1)
    r = c.compress_sequences_device(d_a.data_ptr(), fcap, d_seq.data_ptr(), cnt, d_src.data_ptr(), n)
    w = c.compress_device(d_b.data_ptr(), fcap, d_src.data_ptr(), n, 1)
    assert r == w and bool((d_a[:r] == d_b[:w]).all())


def test_capacity():
    src = _input("P50")
    c = _ctx(3, "zdict")
    want = _want(src, 3, "zdict")
    n = len(want)
    assert (_device_rows(c, src, cap=n) == want).all()
    assert _device_rows(c, src, cap=n - 1) == 70                      # and the guard zone behind n - 1 rows is untouched
    assert _async_rows(c, src, torch.cuda.Stream(), cap=n - 1) == 70
    L = zstd_b200.lib()
    out = np.full((n + 4, 4), 7, np.uint32)
    r = L.ZSTD_generateSequences(c._h, out.ctypes.data, n - 1, src, len(src))
    assert L.ZSTD_getErrorCode(r) == 70 and (out == 7).all()
    assert L.ZSTD_generateSequences(c._h, out.ctypes.data, n, src, len(src)) == n and (out[:n] == want).all() and (out[n:] == 7).all()
    assert c.compress2(src) == zref.oracle_compress_using_dict(src, _dict("zdict"), 3)
    assert (_host(c, src) == want).all()


def test_refusals():
    src = _input("P30")
    c = _ctx(1, "none")
    c.set_parameter(160, 1)                                 # long-distance matching
    assert _host(c, src) == 40 and _device_rows(c, src) == 40
    c.set_parameter(160, 2)
    assert (_host(c, src) == _want(src, 1, "none")).all()
    prefix = zref.synthetic(50_000, 21, 0.5)
    c.ref_prefix(prefix)
    assert _host(c, src) == 40 and _device_rows(c, src) == 40
    with_prefix = c.compress2(src)                            # still pending: this frame uses it
    p = zstd_b200.ZSTD_CCtx()
    p.set_parameter("compression_level", 1)
    p.ref_prefix(prefix)
    assert with_prefix == p.compress2(src)
    L = zstd_b200.lib()
    L.ZSTDB200_setStrictLevels(1)
    try:
        assert _host(_ctx(9, "none"), src) == 40 and _device_rows(_ctx(9, "none"), src) == 40
    finally:
        L.ZSTDB200_setStrictLevels(0)
    d_src = _dev(src)
    d_out = torch.zeros(zstd_b200.sequence_bound(len(src)) * 16 + 64, dtype=torch.uint8, device="cuda")
    with pytest.raises(zstd_b200.ZstdError) as e:
        c.generate_sequences_device(d_out.data_ptr() + 2, 1000, d_src.data_ptr(), len(src))
    assert e.value.code == 42
    with pytest.raises(zstd_b200.ZstdError) as e:
        c.generate_sequences_device(0, 1000, d_src.data_ptr(), len(src))
    assert e.value.code == 74
    # a 4-byte aligned (not 16-byte aligned) output takes the same rows
    torch.cuda.synchronize()
    k = c.generate_sequences_device(d_out.data_ptr() + 4, zstd_b200.sequence_bound(len(src)), d_src.data_ptr(), len(src))
    got = d_out[4:4 + 16 * k].cpu().numpy().view(np.uint32).reshape(-1, 4)
    assert (got == _want(src, 1, "none")).all()


def test_async_interleaved_with_compression():
    """two streams, one context: generate and compress calls interleaved, each correct"""
    srcs = [_input("P30"), _input("P90"), _input("golden:http"), _input("zeros")]
    c = _ctx(3, "none")
    ss = [torch.cuda.Stream(), torch.cuda.Stream()]
    d_src = [_dev(s) for s in srcs]
    caps = [zstd_b200.sequence_bound(len(s)) for s in srcs]
    d_seq = [torch.zeros(cap * 16, dtype=torch.uint8, device="cuda") for cap in caps]
    fcaps = [zstd_b200.ZSTD_compressBound(len(s)) + 64 for s in srcs]
    d_fr = [torch.zeros(f, dtype=torch.uint8, device="cuda") for f in fcaps]
    res = torch.zeros(2 * len(srcs), dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    for i in range(len(srcs)):
        st = ss[i % 2].cuda_stream
        c.generate_sequences_device_async(d_seq[i].data_ptr(), caps[i], d_src[i].data_ptr(), len(srcs[i]), res[2 * i:].data_ptr(), st)
        c.compress_device_async(d_fr[i].data_ptr(), fcaps[i], d_src[i].data_ptr(), len(srcs[i]), res[2 * i + 1:].data_ptr(), 3, st)
    torch.cuda.synchronize()
    r = res.cpu().numpy().view(np.uint64).tolist()
    for i, src in enumerate(srcs):
        assert (_rows(d_seq[i], r[2 * i]) == _want(src, 3, "none")).all()
        assert d_fr[i][:r[2 * i + 1]].cpu().numpy().tobytes() == zref.oracle_compress(src, 3)


def test_graph_capture():
    n = 700_000
    c = _ctx(1, "raw")
    cap = zstd_b200.sequence_bound(n)
    d_src = torch.zeros(n, dtype=torch.uint8, device="cuda")
    d_out = torch.zeros(cap * 16, dtype=torch.uint8, device="cuda")
    res = torch.zeros(1, dtype=torch.int64, device="cuda")
    cold = zstd_b200.ZSTD_CCtx()
    g0 = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.graph(g0):
        with pytest.raises(zstd_b200.ZstdError) as e:
            cold.generate_sequences_device_async(d_out.data_ptr(), cap, d_src.data_ptr(), n, res.data_ptr(),
                                                 torch.cuda.current_stream().cuda_stream)
    assert e.value.code == 60
    s = torch.cuda.Stream()
    c.generate_sequences_device_async(d_out.data_ptr(), cap, d_src.data_ptr(), n, res.data_ptr(), s.cuda_stream)   # warm call
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        c.generate_sequences_device_async(d_out.data_ptr(), cap, d_src.data_ptr(), n, res.data_ptr(),
                                          torch.cuda.current_stream().cuda_stream)
    for seed in (31, 32):
        src = zref.synthetic(n, seed, 0.6)
        d_src.copy_(torch.frombuffer(bytearray(src), dtype=torch.uint8))
        res.fill_(-1)
        g.replay()
        torch.cuda.synchronize()
        k = int(res.cpu().numpy().view(np.uint64)[0])
        assert (_rows(d_out, k) == _want(src, 1, "raw")).all()


def test_stats():
    src = _input("P50")
    c = _ctx(1, "none")
    rows = _host(c, src)
    st = c.stats()
    assert st.h2d_bytes == len(src) and st.d2h_bytes == 16 * len(rows)
    assert st.literals_ms == 0 and st.sequences_ms == 0
    _device_rows(c, src, stream=torch.cuda.Stream())
    st = c.stats()
    assert st.match_ms > 0 and st.stitch_ms > 0 and st.literals_ms == 0 and st.sequences_ms == 0 and st.nbBlocks == 9
