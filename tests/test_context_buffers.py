"""One context through calls of different kinds and sizes: its device and page-locked buffers grow and are reused in
turn, and every call must give the bytes a fresh context gives for the same call."""
import ctypes

import pytest

import zref
import zstd_b200
from test_oracle_sequences import EDGES

torch = pytest.importorskip("torch")
pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600, method="thread")]      # a stuck kernel must fail the run, not hang it


@pytest.fixture(scope="module")
def inputs():
    far = zref.random_bytes(1 << 20, seed=12)
    return {
        "4k": zref.synthetic(4 << 10, 11, 0.5),
        "16m": zref.synthetic(16 << 20, 13, 0.5),
        "1m": zref.synthetic(1 << 20, 14, 0.5),
        "ldm": far + zref.synthetic(2 << 20, 15, 0.5) + far,           # a copy 3 MiB back: only long-distance matching finds it
        "records": [zref.synthetic(1024, 100 + i, 0.5) for i in range(2000)],
        "dict": zref.golden_input("zdict-16k-synthetic-seed77"),
    }


def _same_as_fresh(shared, make, call):
    """call(shared) and call(a new context): the same result"""
    got = call(shared)
    fresh = make()
    try:
        want = call(fresh)
    finally:
        fresh.close()
    assert got == want
    return got


def _sequences(c):
    seqs, explicit, src = EDGES["blocks-of-1-to-6-bytes"]                # 3000 blocks
    c.set_parameter("compression_level", 3)
    c.set_parameter(1008, 1 if explicit else 0)
    try:
        return c.compress_sequences(seqs, src, len(src) + 3 * 3000 + 64)  # raw blocks of a few bytes: 3 header bytes each
    finally:
        c.reset(2)


def _ldm(src):
    def call(c):
        c.set_parameter("compression_level", 1)
        c.set_parameter("enable_long_distance_matching", 1)
        try:
            return c.compress2(src)
        finally:
            c.reset(2)
    return call


def _records_with_dict(records, d):
    def call(c):
        src = b"".join(records)
        offs = [i * 1024 for i in range(len(records))]
        d_src = torch.frombuffer(bytearray(src), dtype=torch.uint8).cuda()
        cap = len(src) * 2 + 4096
        d_dst = torch.zeros(cap, dtype=torch.uint8, device="cuda")
        total, sizes = c.compress_frames(d_dst.data_ptr(), cap, d_src.data_ptr(), offs, [1024] * len(records), level=1,
                                         device_memory=True, dict_bytes=d)
        torch.cuda.synchronize()
        return d_dst[:total].cpu().numpy().tobytes(), sizes
    return call


def test_cctx_calls_of_every_kind(inputs):
    c = zstd_b200.ZSTD_CCtx()
    make = zstd_b200.ZSTD_CCtx
    small = _same_as_fresh(c, make, lambda x: x.compress(inputs["4k"], 1))
    _same_as_fresh(c, make, lambda x: x.compress(inputs["16m"], 1))      # host buffers: two waves (the last one shrinks)
    _same_as_fresh(c, make, _sequences)                                    # no segment or far arrays
    _same_as_fresh(c, make, lambda x: x.compress(inputs["1m"], 3))       # doubleFast: the second candidate arrays
    ldm = _same_as_fresh(c, make, _ldm(inputs["ldm"]))
    assert len(ldm) < len(c.compress(inputs["ldm"], 1)) - (1 << 19)       # the long-distance matches were found
    _same_as_fresh(c, make, _records_with_dict(inputs["records"], inputs["dict"]))
    assert _same_as_fresh(c, make, lambda x: x.compress(inputs["4k"], 1)) == small
    assert zstd_b200.ZSTD_decompress(small) == inputs["4k"]
    c.close()


def _decompress_using_dict(dctx, frames, d, n):
    L = zstd_b200.lib()
    L.ZSTD_decompress_usingDict.restype = ctypes.c_size_t
    L.ZSTD_decompress_usingDict.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_char_p, ctypes.c_size_t,
                                            ctypes.c_char_p, ctypes.c_size_t]
    out = ctypes.create_string_buffer(max(n, 1))
    r = L.ZSTD_decompress_usingDict(dctx._h, out, n, frames, len(frames), d, len(d))
    assert not L.ZSTD_isError(r), L.ZSTD_getErrorName(r)
    return out.raw[:r]


def _device(frames, n):
    def call(dctx):
        d_in = torch.frombuffer(bytearray(frames), dtype=torch.uint8).cuda()
        d_out = torch.zeros(n, dtype=torch.uint8, device="cuda")
        assert dctx.decompress_device(d_out.data_ptr(), n, d_in.data_ptr(), len(frames)) == n
        return d_out.cpu().numpy().tobytes()
    return call


@pytest.mark.parametrize("hostwalk", [None, "0"], ids=["host-walk", "kernel-walk"])
def test_dctx_calls_of_every_kind(inputs, monkeypatch, hostwalk):
    """the kernel walk (ZSTDB200_HOSTWALK_MAX=0, read when the context is created) sizes the descriptor arrays before the
    walk and again behind it"""
    cc = zstd_b200.ZSTD_CCtx()
    small, large = inputs["4k"], inputs["16m"][: 9 << 20]
    small_f = cc.compress(small, 1)
    large_f = cc.compress(large[: 5 << 20], 1) + cc.compress(large[5 << 20:], 3)
    recs, d = inputs["records"][:300], inputs["dict"]
    dict_f = b"".join(cc.compress_using_dict(r, d, 1) for r in recs)
    cc.close()
    if hostwalk is not None:
        monkeypatch.setenv("ZSTDB200_HOSTWALK_MAX", hostwalk)
    dc = zstd_b200.ZSTD_DCtx()
    monkeypatch.delenv("ZSTDB200_HOSTWALK_MAX", raising=False)
    make = zstd_b200.ZSTD_DCtx
    calls = [
        (lambda x: x.decompress(small_f), small),
        (lambda x: x.decompress(large_f, len(large)), large),
        (lambda x: _decompress_using_dict(x, dict_f, d, 300 * 1024), b"".join(recs)),
        (lambda x: x.decompress(small_f), small),
        (_device(large_f, len(large)), large),
        (_device(small_f, len(small)), small),
        (lambda x: x.decompress(large_f, len(large)), large),
    ]
    for call, want in calls:
        assert _same_as_fresh(dc, make, call) == want
    dc.close()
