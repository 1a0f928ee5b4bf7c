"""The prefix rule of oracle/zb_prefix.c (ZSTD_CCtx_refPrefix with long-distance matching over the prefix): its frames decode
with the reference decoder given the same prefix, the properties the rule states hold on its match lists, and its frames
are as small as the reference's --patch-from style frames.  CPU only."""
import pytest

import ldmref
import prefixref
import zref

needs_ref = pytest.mark.skipif(not zref.have_ref(), reason="oracle/_ref/libzstd_ref.so not built")


@pytest.fixture(scope="module")
def pairs():
    return prefixref.pairs()


NAMES = ["edits", "shifted", "same", "unrelated", "prefix1", "prefix7", "prefix100k", "prefix_larger", "small_frame_ldm",
         "small_frame_no_ldm", "magic", "empty"]


@needs_ref
@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("level", [1, 3, -3])
def test_prefix_frame_decodes_with_the_reference(pairs, name, level):
    prefix, src = pairs[name]
    for ldm in (True, False):
        frame = prefixref.oracle_prefix(src, prefix, level, ldm=ldm)
        assert prefixref.ref_decompress_prefix(frame, prefix, len(src)) == src
        if name != "magic":                      # ZSTD_decompress_usingDict would read that prefix as a zstd-format dictionary
            assert zref.ref_decompress_using_dict(frame, prefix, len(src)) == src


@needs_ref
@pytest.mark.parametrize("corner", ldmref.CORNERS, ids=lambda c: ",".join(f"{k}={v}" for k, v in c.items()))
def test_prefix_parameter_corners(pairs, corner):
    for name in ("shifted", "small_frame_ldm"):
        prefix, src = pairs[name]
        frame = prefixref.oracle_prefix(src, prefix, 1, **corner)
        assert prefixref.ref_decompress_prefix(frame, prefix, len(src)) == src


@pytest.mark.parametrize("name", ["edits", "shifted", "prefix100k", "small_frame_ldm"])
def test_frame_survivors_do_not_depend_on_the_prefix(pairs, name):
    """steps 1 and 2 run on each segment's own bytes: the survivors are the prefix's plus the frame's, and every block's
    first survivor is the one it has without a prefix, moved by the number of prefix survivors"""
    prefix, src = pairs[name]
    wl = prefixref.window_log(len(src), len(prefix))
    in_prefix = len(ldmref.survivors(prefixref.indexed(prefix), ldmref.resolve(wl)))
    alone = prefixref.lists(src, b"", wl)
    both = prefixref.lists(src, prefix, wl)
    assert in_prefix > 0 and alone["nb_survivors"] > 0
    assert both["nb_survivors"] == in_prefix + alone["nb_survivors"]
    assert [f - in_prefix for f in both["first"]] == alone["first"]


@pytest.mark.parametrize("name", ["edits", "shifted", "same", "prefix100k", "prefix_larger", "small_frame_ldm", "magic"])
def test_no_match_crosses_the_seam_and_offsets_stay_in_the_window(pairs, name):
    prefix, src = pairs[name]
    wl = prefixref.window_log(len(src), len(prefix))
    got, P = prefixref.matches(src, prefix, wl)
    assert got, "the pair shares content: the rule must find it"
    buf = prefixref.indexed(prefix) + src
    from_prefix = 0
    for p, length, off in got:
        q = p - off
        assert p >= P and q >= 0
        assert off <= min(p, 1 << wl)
        assert not (q < P < q + length), "source range runs from the prefix into the frame"
        assert buf[q:q + length] == buf[p:p + length]
        from_prefix += q < P
    assert from_prefix > 0


def test_match_lists_without_a_prefix_are_unchanged(pairs):
    """P = 0 is the rule as it was: the same frames as zbo_compress_ldm"""
    src = ldmref.aba()
    for level in (1, 3):
        assert prefixref.oracle_prefix(src, b"", level) == ldmref.oracle_ldm(src, level)
        assert prefixref.oracle_prefix(src, b"1234567", level) == ldmref.oracle_ldm(src, level)     # < 8 bytes: ignored


@pytest.mark.parametrize("name", ["edits", "prefix100k", "small_frame_no_ldm", "empty"])
@pytest.mark.parametrize("level", [1, 3])
def test_without_ldm_a_prefix_is_a_raw_dictionary(pairs, name, level):
    prefix, src = pairs[name]
    frame = prefixref.oracle_prefix(src, prefix, level, ldm=False)
    assert frame == zref.oracle_compress_using_dict(src, prefix, level)
    assert frame[4] & 3 == 0, "dictionary ID 0: no Dictionary_ID field"
    if len(prefixref.indexed(prefix)) + len(src) <= prefixref.LDM_MIN or not src:
        assert prefixref.oracle_prefix(src, prefix, level, ldm=True) == frame          # below the size LDM runs at


def test_a_prefix_with_the_dictionary_magic_is_raw_content(pairs):
    prefix, src = pairs["magic"]
    assert prefix[:4] == bytes.fromhex("37a430ec")
    for ldm in (True, False):
        frame = prefixref.oracle_prefix(src, prefix, 1, ldm=ldm)
        assert frame[4] & 3 == 0
        other = b"\x00" + prefix[1:]                 # the same content without the magic: the first byte is 1 MiB back
        assert len(frame) <= len(prefixref.oracle_prefix(src, other, 1, ldm=ldm)) + 16
    assert prefixref.oracle_prefix(src, prefix, 1, ldm=False) == prefixref.oracle_raw_dict(src, prefix, 1)


def test_prefix_beyond_the_window_is_clipped():
    """the indexed part is the prefix's last 2^27 bytes; here the clip is exercised through the window rule instead of a
    128 MiB input: with a 2^20 window, prefix survivors further than that from a block's end are no candidates"""
    old, new = prefixref.version_pair(size=2 << 20, edits=50, seed=31)
    got, P = prefixref.matches(new, old, 20)
    assert got
    for p, length, off in got:
        block_end = min(P + ((p - P) // (128 << 10) + 1) * (128 << 10), P + len(new))
        assert p - off >= max(0, block_end - (1 << 20))
    assert all(p - off >= P for p, _, off in got if p - P >= (1 << 20)), "blocks a window into the frame take nothing from the prefix"
    assert prefixref.indexed(b"a" * 7) == b"" and len(prefixref.indexed(bytes(10))) == 10


@needs_ref
@pytest.mark.parametrize("name", ["edits", "shifted", "prefix_larger"])
def test_size_against_the_reference(pairs, name):
    """the reference with the same prefix and LDM on, and the same input without the prefix"""
    prefix, src = pairs[name]
    ours = len(prefixref.oracle_prefix(src, prefix, 1))
    ref = len(prefixref.ref_compress_prefix(src, prefix, 1))
    assert ours <= 1.05 * ref + 64, (ours, ref)
    assert ours < 0.05 * len(ldmref.oracle_ldm(src, 1))
