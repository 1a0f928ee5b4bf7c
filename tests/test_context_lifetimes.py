"""Contexts and digested dictionaries are created, used and freed in every order a caller may choose: what each owns (streams,
events, device buffers, its copy of the dictionary bytes) lives exactly as long as it does, and every result equals the one
a fresh context or the oracle gives."""
import pytest

import zref
import zstd_b200

RAW = zref.synthetic(20 << 10, 7, 0.5)
ZDICT = zref.golden_input("zdict-16k-synthetic-seed77")


def test_create_and_free_without_a_device():
    """Creation, dictionary loading, referencing, resets and frees touch no device, and every free returns 0"""
    L = zstd_b200.lib()
    bad = bytearray(ZDICT)
    bad[12:40] = b"\xff" * 28                                          # entropy tables destroyed
    for _ in range(20):
        c, d = L.ZSTD_createCCtx(), L.ZSTD_createDCtx()
        assert c and d
        cds = [L.ZSTD_createCDict(x, len(x), lvl) for x, lvl in ((RAW, 1), (ZDICT, 3), (b"", 0), (b"abc", -5))]
        assert all(cds)
        assert L.ZSTD_getDictID_fromCDict(cds[0]) == 0
        assert L.ZSTD_getDictID_fromCDict(cds[1]) == L.ZSTD_getDictID_fromDict(ZDICT, len(ZDICT)) != 0
        assert not L.ZSTD_createCDict(bytes(bad), len(bad), 1)
        assert L.ZSTD_CCtx_loadDictionary(c, RAW, len(RAW)) == 0
        assert L.ZSTD_CCtx_loadDictionary(c, ZDICT, len(ZDICT)) == 0      # replaces the first one
        r = L.ZSTD_CCtx_loadDictionary(c, bytes(bad), len(bad))
        assert L.ZSTD_isError(r) and L.ZSTD_getErrorCode(r) == 30
        assert L.ZSTD_CCtx_refCDict(c, cds[1]) == 0
        assert L.ZSTD_CCtx_loadDictionary(c, RAW, len(RAW)) == 0          # drops the reference
        assert L.ZSTD_CCtx_reset(c, 2) == 0                                # drops the loaded dictionary
        assert L.ZSTD_CCtx_loadDictionary(c, ZDICT, len(ZDICT)) == 0      # left for ZSTD_freeCCtx
        assert L.ZSTD_CCtx_reset(c, 1) == 0
        assert L.ZSTD_CCtx_refCDict(c, None) == 0
        assert L.ZSTD_CCtx_loadDictionary(c, RAW, len(RAW)) == 0
        assert [L.ZSTD_freeCDict(cd) for cd in cds] == [0, 0, 0, 0]
        assert L.ZSTD_freeCCtx(c) == 0
        assert L.ZSTD_freeDCtx(d) == 0
    assert (L.ZSTD_freeCCtx(None), L.ZSTD_freeDCtx(None), L.ZSTD_freeCDict(None)) == (0, 0, 0)


@pytest.mark.parametrize("name", ["raw", "zstd-format"])
@pytest.mark.gpu
@pytest.mark.timeout(600, method="thread")
def test_cdict_shared_by_two_contexts(name):
    """One CDict serves two contexts in alternation and is freed after both; it holds its own copy of the bytes, so the
    caller's buffer may change after ZSTD_createCDict"""
    d = RAW if name == "raw" else ZDICT
    buf = bytearray(d)
    cd = zstd_b200.ZSTD_CDict(buf, 1)
    buf[:] = bytes(len(buf))
    a, b = zstd_b200.ZSTD_CCtx(), zstd_b200.ZSTD_CCtx()
    srcs = [(d[-3000:-1000] + zref.synthetic(n, 40 + n % 7, 0.5))[:n] for n in (1024, 5000, 300_000, 1024, 70_000)]
    for k, src in enumerate(srcs):
        want = zref.oracle_compress_using_dict(src, d, 1)
        assert (a if k % 2 else b).compress_using_cdict(src, cd) == want
        assert (b if k % 2 else a).compress_using_cdict(src, cd) == want
    a.close()
    assert b.compress_using_cdict(srcs[0], cd) == zref.oracle_compress_using_dict(srcs[0], d, 1)
    b.close()
    cd.close()


@pytest.mark.gpu
@pytest.mark.timeout(600, method="thread")
def test_load_dictionary_replaced():
    """ZSTD_CCtx_loadDictionary several times on one context, with a referenced CDict and no dictionary in between: each
    call uses exactly the dictionary in force"""
    src = (RAW[-2000:] + ZDICT[-2000:] + zref.synthetic(6000, 41, 0.5))[:8000]
    c = zstd_b200.ZSTD_CCtx()
    c.set_parameter("compression_level", 1)
    cd = zstd_b200.ZSTD_CDict(ZDICT, -3)
    for d in (RAW, ZDICT, RAW, None, ZDICT, "cdict", RAW):
        if d == "cdict":
            c.ref_cdict(cd)
            want = zref.oracle_compress_using_dict(src, ZDICT, -3)
        else:
            c.load_dictionary(d)
            want = zref.oracle_compress(src, 1) if d is None else zref.oracle_compress_using_dict(src, d, 1)
        assert c.compress2(src) == want
    c.close()
    cd.close()


@pytest.mark.gpu
@pytest.mark.timeout(600, method="thread")
def test_wave_events_follow_the_timeline_setting(monkeypatch):
    """Host calls of 1 to 6 waves on one context, with ZSTDB200_TIMELINE set for one of them: the wave events are recreated
    when a call needs more of them or the other kind, and each call gives the bytes and launch count of a fresh context"""
    monkeypatch.setenv("ZSTDB200_HOST_WAVE_BLOCKS", "32")             # read when a context is created: 4 MiB waves
    c = zstd_b200.ZSTD_CCtx()
    src = zref.synthetic(24 << 20, 17, 0.5)
    for mib, timeline in ((4, False), (16, False), (8, True), (16, False), (24, False), (4, True)):
        if timeline:
            monkeypatch.setenv("ZSTDB200_TIMELINE", "1")
        got = c.compress(src[:mib << 20], 1)
        st = c.stats()
        fresh = zstd_b200.ZSTD_CCtx()
        try:
            assert got == fresh.compress(src[:mib << 20], 1)
            assert (st.launches, st.nbBlocks) == (fresh.stats().launches, fresh.stats().nbBlocks)
        finally:
            fresh.close()
        monkeypatch.delenv("ZSTDB200_TIMELINE", raising=False)
    assert zstd_b200.ZSTD_decompress(got) == src[:4 << 20]
    c.close()


@pytest.mark.gpu
@pytest.mark.timeout(600, method="thread")
def test_create_use_free_cycles():
    """50 rounds of creating a compression context, a CDict and a decompression context, using each and freeing all three
    (in a different order every round)"""
    from test_context_buffers import _decompress_using_dict
    srcs = [(ZDICT[-1500:] + zref.synthetic(n, 60 + n % 5, 0.5))[:n] for n in (1000, 4096, 40_000)]
    want_plain = [zref.oracle_compress(s, 1) for s in srcs]
    want_dict = [zref.oracle_compress_using_dict(s, ZDICT, 1) for s in srcs]
    for i in range(50):
        k = i % len(srcs)
        c, cd, dc = zstd_b200.ZSTD_CCtx(), zstd_b200.ZSTD_CDict(ZDICT, 1), zstd_b200.ZSTD_DCtx()
        assert c.compress(srcs[k], 1) == want_plain[k]
        assert c.compress_using_cdict(srcs[k], cd) == want_dict[k]
        assert c.compress_using_dict(srcs[k], ZDICT, 1) == want_dict[k]
        assert dc.decompress(want_plain[k], len(srcs[k])) == srcs[k]
        assert _decompress_using_dict(dc, want_dict[k], ZDICT, len(srcs[k])) == srcs[k]
        for x in ((c, cd, dc), (cd, dc, c), (dc, c, cd))[i % 3]:
            x.close()
