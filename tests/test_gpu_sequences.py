"""ZSTD_compressSequences and ZSTDB200_compressSequencesDevice on the GPU: byte for byte the oracle's frames
(oracle/zb_seqs.c), ZSTD_compress2's frames when fed that call's own stores, and the same errors."""
import numpy as np
import pytest

import seqgen
import seqoracle as so
import zref
import zstd_b200
from test_oracle_sequences import EDGES, SRC, _seqs

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not zref.have_ref(), reason="oracle/_ref/libzstd_ref.so not built")


def _ctx(level=3, explicit=True, dict=None, cdict=None, checksum=False):
    c = zstd_b200.ZSTD_CCtx()
    c.set_parameter("compression_level", level)
    c.set_parameter(1008, 1 if explicit else 0)
    c.set_parameter(1009, 1)
    if checksum:
        c.set_parameter("checksum_flag", 1)
    if dict is not None:
        c.load_dictionary(dict)
    if cdict is not None:
        c.ref_cdict(cdict)
    return c


def _device(c, seqs, src, cap=None, stream=None):
    a = so.as_array(seqs)
    d_seq = torch.from_numpy(a.view(np.uint8).reshape(-1).copy()).cuda() if len(a) else torch.zeros(16, dtype=torch.uint8, device="cuda")
    d_src = torch.frombuffer(bytearray(src), dtype=torch.uint8).cuda() if src else torch.zeros(1, dtype=torch.uint8, device="cuda")
    cap = zstd_b200.ZSTD_compressBound(len(src)) + 64 if cap is None else cap
    d_dst = torch.zeros(cap + 4096, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    h = stream.cuda_stream if stream is not None else 0
    err = None
    try:
        r = c.compress_sequences_device(d_dst.data_ptr(), cap, d_seq.data_ptr(), len(a), d_src.data_ptr(), len(src), h)
    except zstd_b200.ZstdError as e:
        err = e.code
    if stream is not None:
        stream.synchronize()
    out = d_dst.cpu().numpy().tobytes()
    assert out[cap:] == bytes(4096), "bytes written past dstCapacity"
    return err if err is not None else out[:r]


def _host(c, seqs, src, cap=None):
    try:
        return c.compress_sequences(seqs, src, cap)
    except zstd_b200.ZstdError as e:
        return e.code


def _gpu_decode(frame, n):
    return zstd_b200.ZSTD_DCtx().decompress(frame, n)


@needs_ref
@pytest.mark.parametrize("name", list(seqgen.DICTATED))
def test_dictated_against_oracle(name, monkeypatch):
    stream = torch.cuda.Stream()
    for seqs, src, level, d, _ in so.dictated(monkeypatch, name):
        for explicit in (True, False):
            arr = seqs if explicit else so.merge_delimiters(seqs)
            want = so.compress_sequences(arr, src, level, d, explicit)
            c = _ctx(level, explicit, dict=d)
            assert _host(c, arr, src) == want
            assert _device(c, arr, src) == want
            assert _device(c, arr, src, stream=stream) == want
            assert seqgen.ref_decompress(want, len(src), d) == src
            if d is None:
                assert _gpu_decode(want, len(src)) == src


@needs_ref
@pytest.mark.parametrize("level", [1, 3, -3])
@pytest.mark.parametrize("kind", ["none", "raw", "zdict"])
def test_dictionary_checksum_levels(kind, level):
    d = None if kind == "none" else (zref.golden_input(seqgen.ZDICT) if kind == "zdict" else zref.synthetic(40_000, 3, 0.5))
    src = zref.synthetic(600_000, 21, 0.6)
    seqs = so.frame_sequences(src, level, d)
    want = so.compress_sequences(seqs, src, level, d)
    assert want == (zref.oracle_compress_using_dict(src, d, level) if d else zref.oracle_compress(src, level))
    assert _host(_ctx(level, dict=d), seqs, src) == want
    if d is not None:
        cd = zstd_b200.ZSTD_CDict(d, level)
        assert _device(_ctx(level, cdict=cd), seqs, src) == want
    ck = _host(_ctx(level, dict=d, checksum=True), seqs, src)
    assert len(ck) == len(want) + 4 and seqgen.ref_decompress(ck, len(src), d) == src
    if d is None:
        assert _gpu_decode(ck, len(src)) == src


@needs_ref
@pytest.mark.parametrize("explicit", [True, False])
@pytest.mark.parametrize("level", [1, 3, -3])
def test_identity_with_compress2(level, explicit):
    src = zref.datagen(5 << 20, 50, seed=level & 0xFF) if zref.have_datagen() else zref.synthetic(5 << 20, 5)
    seqs = so.frame_sequences(src, level)
    if not explicit:
        seqs = so.merge_delimiters(seqs)
    c = _ctx(level, explicit)
    assert _host(c, seqs, src) == c.compress2(src)


@needs_ref
def test_identity_waves(monkeypatch):
    """64 MiB in waves of 64 blocks through one workspace slot"""
    monkeypatch.setenv("ZSTDB200_WAVE_BLOCKS", "64")
    src = zref.datagen(64 << 20, 50, seed=3) if zref.have_datagen() else zref.synthetic(64 << 20, 3)
    seqs = so.frame_sequences(src, 1)
    c = _ctx(1, True)
    want = c.compress2(src)
    assert _device(c, seqs, src) == want
    assert c.stats().nbBlocks == 512
    merged = so.merge_delimiters(seqs)
    c2 = _ctx(1, False)
    assert _host(c2, merged, src) == want


def test_density():
    """one block of 43 690 three-byte matches (blockMax / 3 sequences)"""
    blocks = [([(1, 1, 3)] + [(0, 3, 3)] * 43_689, 1)]
    src = seqgen.execute(blocks, np.random.default_rng(9), alphabet=4)
    seqs = so.blocks_to_array(blocks)
    want = so.compress_sequences(seqs, src, 3)
    assert _host(_ctx(3), seqs, src) == want
    assert zref.ref_decompress(want, len(src)) == src if zref.have_ref() else True


@pytest.mark.parametrize("name", list(EDGES))
def test_edges(name):
    s, explicit, src = EDGES[name]
    cap = 4 * len(src) + 1024
    want = so.compress_sequences(s, src, 3, None, explicit, cap=cap)
    assert _host(_ctx(3, explicit), s, src, cap) == want
    assert _device(_ctx(3, explicit), s, src, cap) == want


def test_empty_input():
    c = _ctx(3)
    want = c.compress2(b"")
    assert _host(c, _seqs(), b"") == want
    assert _device(c, _seqs((0, 0, 0)), b"") == want


@pytest.mark.parametrize("case", ["offset0", "short-match", "offset-beyond", "past-src", "no-final-delim", "block-too-big",
                                  "nodelim-past-src", "nodelim-delimiter"])
def test_errors_leave_context_usable(case):
    import test_oracle_sequences as t
    n = len(SRC)
    bad = {"offset0": _seqs((0, 10, 5), (0, n - 15, 0)), "short-match": _seqs((5, 10, 2), (0, n - 12, 0)),
           "offset-beyond": _seqs((11, 5, 5), (0, n - 10, 0)), "past-src": _seqs((5, 10, 5), (0, n, 0)),
           "no-final-delim": _seqs((5, 10, 5), (0, 100, 0), (5, 10, 5)), "block-too-big": _seqs((0, 131073, 0), (0, n - 131073, 0)),
           "nodelim-past-src": _seqs((5, 10, 5), (5, n, 5)), "nodelim-delimiter": _seqs((5, 10, 5), (0, 10, 0))}[case]
    explicit = not case.startswith("nodelim")
    c = _ctx(3, explicit)
    assert _host(c, bad, SRC) == 107
    assert _device(c, bad, SRC) == 107
    s, e, src = t.EDGES["trailing-run-no-delimiter"]
    c.set_parameter(1008, 0)
    assert _device(c, s, src) == so.compress_sequences(s, src, 3, None, False)


def test_dst_too_small_and_reuse():
    src = zref.synthetic(400_000, 8, 0.5)
    seqs = so.frame_sequences(src, 3)
    c = _ctx(3)
    want = so.compress_sequences(seqs, src, 3)
    assert _device(c, seqs, src, cap=len(want) - 1) == 70
    assert _host(c, seqs, src, cap=len(want) - 1) == 70
    assert _device(c, seqs, src) == want
    assert c.compress2(src) == want                                   # interleaved with ZSTD_compress2
    assert _host(c, seqs, src) == want
    assert c.compress2(src) == want


def test_parameters():
    c = zstd_b200.ZSTD_CCtx()
    for p in (1008, 1009):
        for v in (0, 1):
            c.set_parameter(p, v)
        with pytest.raises(zstd_b200.ZstdError) as e:
            c.set_parameter(p, 2)
        assert e.value.code == 40
    c.set_parameter(1008, 1)
    c.reset(2)
    s, explicit, src = EDGES["trailing-run-no-delimiter"]
    assert not explicit
    assert _host(c, s, src) == so.compress_sequences(s, src, 3, None, False)      # back to no delimiters
    assert zstd_b200.sequence_bound(1 << 20) == (1 << 20) // 3 + 1 + 1024 + 1
