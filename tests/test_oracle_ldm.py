"""Long-distance matching, CPU side: the oracle's LDM frames (oracle/zb_ldm.c) against the reference decoder and the
reference's own LDM frames, the survivor rule, the window, and the parameter interface (which needs no GPU)."""

import numpy as np
import pytest

import ldmref
import zref

needs_ref = pytest.mark.skipif(not zref.have_ref(), reason="reference library not built")


@pytest.fixture(scope="module")
def inputs():
    return ldmref.inputs()


@needs_ref
@pytest.mark.parametrize("name", ["aba", "versions", "zeros", "random", "period4k"])
@pytest.mark.parametrize("level", [1, 3, -3])
def test_oracle_ldm_frames_decode(inputs, name, level):
    src = inputs[name]
    frame = ldmref.oracle_ldm(src, level)
    assert zref.ref_decompress(frame, len(src)) == src


@needs_ref
@pytest.mark.parametrize("corner", ldmref.CORNERS, ids=lambda c: ",".join(f"{k}={v}" for k, v in c.items()))
def test_oracle_ldm_parameter_corners(inputs, corner):
    for name in ("aba", "period4k"):
        src = inputs[name]
        frame = ldmref.oracle_ldm(src, 1, **corner)
        assert zref.ref_decompress(frame, len(src)) == src


@pytest.mark.parametrize("min_match", [4, 16, 64, 300])
def test_survivors_apart_and_copied(min_match):
    a = zref.synthetic(300_000, seed=11)
    src = a + zref.random_bytes(100_000, seed=12) + a
    prm = ldmref.resolve(27, min_match=min_match, hash_rate_log=4)
    s = ldmref.survivors(src, prm).astype(np.int64)
    assert len(s) > 100
    assert np.all(np.diff(s) >= min_match)
    off = 400_000
    margin = 64 + 2 * min_match                      # the gear hash sees 64 bytes, thinning minMatch - 1 on either side
    first = s[(s >= margin) & (s < len(a) - margin)]
    copy = s[(s >= off + margin) & (s < off + len(a) - margin)] - off
    assert np.array_equal(first, copy)


def test_ldm_resolve_defaults():
    p = ldmref.resolve(27)
    assert (p.hashLog, p.bucketSizeLog, p.minMatch, p.hashRateLog) == (20, 3, 64, 7)


def test_window_edge():
    """a 4 KiB random repeat 2^27 + 4 KiB back is out of the window and stays literal; 2^27 - 4 KiB back is matched"""
    unit = zref.random_bytes(4096, seed=21)
    gap = zref.random_bytes(1 << 20, seed=22)
    for dist, matched in (((1 << 27) - 4096, True), ((1 << 27) + 4096, False)):
        filler = bytes(dist - 4096)                   # zeros: the parse makes them a few bytes, no LDM survivor lies in them
        src = unit + filler + unit + gap
        frame = ldmref.oracle_ldm(src, 1)
        if zref.have_ref():
            assert zref.ref_decompress(frame, len(src)) == src
        base = ldmref.oracle_ldm(zref.random_bytes(4096, seed=23) + filler + unit + gap, 1)
        saved = len(base) - len(frame)
        assert (saved > 3000) == matched, (dist, saved)


@needs_ref
def test_ldm_sizes(inputs):
    """LDM on against off from the oracle, and against the reference's LDM frame (measured: see DESIGN.md section 10)"""
    src = inputs["aba"]
    on, off = len(ldmref.oracle_ldm(src, 1)), len(zref.oracle_compress(src, 1))
    assert on / off <= 0.70
    assert on / len(ldmref.ref_compress2(src, 1, 1)) <= 1.10
    v = ldmref.versions(size=1 << 20, count=16)
    on, off = len(ldmref.oracle_ldm(v, 1)), len(zref.oracle_compress(v, 1))
    assert on / off <= 0.10
    assert on / len(ldmref.ref_compress2(v, 1, 1)) <= 1.25
    if zref.have_datagen():
        d = zref.datagen(16 << 20, 50, 0)
        assert len(ldmref.oracle_ldm(d, 1)) <= 1.003 * len(zref.oracle_compress(d, 1))


@pytest.mark.parametrize("size", [1000, 128 << 10, (512 << 10)])
def test_small_frames_unchanged(size):
    src = zref.synthetic(size, seed=31)
    for level in (1, 3, -3):
        assert ldmref.oracle_ldm(src, level) == zref.oracle_compress(src, level)


# ---- the parameter interface of the product (no compression happens: no GPU needed) ----
@pytest.fixture
def cctx():
    import zstd_b200
    try:
        zstd_b200.lib()
    except ImportError:
        pytest.skip("libzstd_b200.so not built")
    return zstd_b200


def _set(z, c, pid, value):
    return z.lib().ZSTD_getErrorCode(z.lib().ZSTD_CCtx_setParameter(c, pid, value))


def test_set_parameter_bounds(cctx):
    z = cctx
    c = z.lib().ZSTD_createCCtx()
    try:
        for v in (0, 1, 2):
            assert _set(z, c, 160, v) == 0
        assert _set(z, c, 160, 3) == 42
        assert _set(z, c, 160, -1) == 42
        for pid, lo, hi in ((161, 6, 30), (162, 4, 4096), (163, 1, 8), (164, 0, 25)):
            assert _set(z, c, pid, 0) == 0
            assert _set(z, c, pid, lo) == 0 and _set(z, c, pid, hi) == 0
            assert _set(z, c, pid, hi + 1) == 42
            assert _set(z, c, pid, -1) == 42
            if lo > 1:
                assert _set(z, c, pid, lo - 1) == 42
        assert _set(z, c, 101, 20) == 40                  # windowLog stays default-only
    finally:
        z.lib().ZSTD_freeCCtx(c)


def test_python_parameter_names(cctx):
    ctx = cctx.ZSTD_CCtx()
    for name in ("enable_long_distance_matching", "ldm_hash_log", "ldm_min_match", "ldm_bucket_size_log", "ldm_hash_rate_log"):
        ctx.set_parameter(name, 0)
    ctx.set_parameter("enable_long_distance_matching", 1)
    ctx.reset(2)
