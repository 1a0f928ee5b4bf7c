"""Long-distance matching path by path (zb_ldm.cu: split points, thinning, bucket sort, selection; the overlay in K1c).

On the CPU (runs without a GPU): a Python restatement of the rule (tests/ldmgen.py) is proved equal to the oracle step by
step on every input and parameter set below: its survivors equal zbo_ldm_survivors, its match lists (fed the oracle's
survivors) equal zbo_ldm_frame / zbo_ldm_frame_usingPrefix, and its overlay of every block (fed zbo_parseBlock's
sequences, driven by dfastgen.frame_blocks as zbo_compress_ldm_usingDict drives them) equals zbo_ldm_overlayBlock.  It
then counts the path each split point, survivor, candidate and parse match takes: every row is reached, the rows that the
rule forbids stay zero, and each neighbouring wrong rule changes some block.

On the GPU: every frame equals the oracle's byte for byte through ZSTD_compress2 (a sample also through
ZSTD_compressStream2 and a device call on a caller stream) and decodes with the reference decoder and the product's; the
frames against a prefix; the 136 MiB frame whose copies lie on both sides of the window limit; and dictionaries (raw,
zstd-format, and zstd-format with repcodes that a first-block LDM offset hits) through every call that takes one."""
import functools
import os

import numpy as np
import pytest

import dfastgen as dg
import ldmgen as g
import ldmref
import prefixref
import zref

needs_oracle = pytest.mark.skipif(not os.path.exists(zref.ORACLE_SO), reason="oracle/libzb_oracle.so not built")
LDM_MIN = 4 * g.BLOCK
DICT_NAMES = ["raw-64k", "zdict-16k", "zdict-16k-ldm-reps"]
# the parameter sets a switch of steps 1-4 is judged on (the others cost more and add no distinction)
SWITCH_PARAMS = ("default", "passes0", "mm37", "mm4")


@functools.lru_cache(maxsize=None)
def dictionary(name: str) -> bytes:
    if name == "raw-64k":
        return dg.dfast_input(64 << 10, 43)
    d = zref.golden_input("zdict-16k-synthetic-seed77")
    if name == "zdict-16k":
        return d
    # repcodes = the first three LDM offsets of the dense frame's first block behind this dictionary: its LDM matches hit them
    first = _dict_lists(g.frame_inputs()["dense"], len(d))[0]
    offs = []
    for _, _, off in first:
        if off not in offs:
            offs.append(off)
    assert len(offs) >= 3
    return dg.patch_reps(d, offs[:3])


def _dict_lists(src: bytes, dict_size: int):
    """the lists of src behind a dictionary: zbo_compress_ldm_usingDict takes them at the window of its cParams, which count
    the dictionary in (its content is not indexed)"""
    return ldmref.frame_lists(src, ldmref.cparams_ldm(1, len(src), dict_size).windowLog)


@functools.lru_cache(maxsize=None)
def _cases():
    """every case with its resolved parameters, window, the oracle's survivors and lists"""
    out = []
    for name, pfx, src, level, prm in g.cases():
        r = g.resolved(len(pfx), len(src), prm)
        pos, v = g.oracle_survivors(pfx, src, r)
        out.append(dict(name=name, pfx=pfx, src=src, level=level, prm=prm, r=r, wl=g.window_log(len(pfx), len(src)),
                        pos=pos, v=v, lists=g.oracle_lists(pfx, src, prm)))
    src = g.window_frame()
    r = g.resolved(0, len(src), {})
    pos, v = g.oracle_survivors(b"", src, r)
    out.append(dict(name="window/default", pfx=b"", src=src, level=1, prm={}, r=r, wl=g.window_log(0, len(src)), pos=pos, v=v,
                    lists=g.oracle_lists(b"", src, {})))
    return out


def _thin_cases():
    return [c for c in _cases() if not c["name"].startswith("window/")]   # 136 MiB: the oracle's survivors feed its selection


@functools.lru_cache(maxsize=None)
def _steps12(sw=frozenset()):
    """restated survivors per case (both segments, [prefix | frame] coordinates), and the counts"""
    cnt, out = {}, {}
    for c in _thin_cases():
        pp, pv = g.survivors(c["pfx"], c["r"], sw, cnt) if c["pfx"] else (np.zeros(0, np.uint64), np.zeros(0, np.uint64))
        fp, fv = g.survivors(c["src"], c["r"], sw, cnt)
        out[c["name"]] = (np.concatenate([pp, fp + np.uint64(len(c["pfx"]))]), np.concatenate([pv, fv]))
        g._bump(cnt, f"passes_{g.passes(c['r'])}")
    return out, cnt


def _select(c, sw=frozenset(), cnt=None):
    return g.select(c["pfx"] + c["src"], len(c["pfx"]), c["pos"], c["v"], len(c["src"]), c["wl"], c["r"], sw, cnt)


@functools.lru_cache(maxsize=None)
def _steps34():
    cnt = {}
    return {c["name"]: _select(c, cnt=cnt) for c in _cases()}, cnt


@functools.lru_cache(maxsize=None)
def _frame_blocks(src_name: str, dict_name):
    src = g.frame_inputs()[src_name]
    return dg.frame_blocks(src, 1, dictionary(dict_name) if dict_name else None, ldm=True)


def _overlay_units():
    """(case name, block, its LDM matches) of every block the overlay sees: the frames without a prefix at every parameter
    set, and the dense frame behind each dictionary (whose content LDM does not index) at the defaults"""
    units = []
    for c in _cases():
        if c["pfx"] or len(c["src"]) <= LDM_MIN or c["name"].startswith("window/"):
            continue
        src_name = c["name"].split("/")[0]
        for b in _frame_blocks(src_name, None):
            units.append((c["name"], b, c["lists"][b.index]))
    for d in DICT_NAMES:
        lists = _dict_lists(g.frame_inputs()["dense"], len(dictionary(d)))
        for b in _frame_blocks("dense", d):
            units.append((f"dense+{d}/default", b, lists[b.index]))
    return units


def _blk(b):
    return b.buf[b.bs:b.be]


@functools.lru_cache(maxsize=None)
def _steps5():
    cnt, got, want = {}, [], []
    for _, b, lm in _overlay_units():
        got.append(g.overlay(b.be - b.bs, b.ldm_reps, lm, b.oracle_seqs, cnt=cnt))
        want.append(ldmref.overlay_block(_blk(b), b.ldm_reps, lm, b.oracle_seqs)[0])
    return got, want, cnt


def _counts():
    c = {}
    for part in (_steps12()[1], _steps34()[1], _steps5()[2]):
        for k, v in part.items():
            c[k] = c.get(k, 0) + v
    return c


def _table(counts):
    return "\n".join(f"{r:24s} {counts.get(r, 0)}" for r in g.ROWS + g.NEVER)


# ------------------------------------------------------------------------------------------------------------ CPU
@needs_oracle
def test_parameter_sets_pin_the_pass_counts():
    """the bucket sort's pass count of each set, from the oracle's resolution, so that a default cannot move it"""
    for c in _cases():
        p = c["name"].split("/")[1]
        if p in g.PASSES:
            assert g.passes(c["r"]) == g.PASSES[p], c["name"]
        if p == "mm4_hr0":
            assert c["r"].hashRateLog == 0
        if p in ("mm4", "mm4_hr8"):
            assert c["r"].hashRateLog > c["r"].minMatch                      # the stop mask in the low bits
    assert {g.passes(c["r"]) for c in _cases()} == {0, 1, 2, 3, 4}
    assert {c["r"].minMatch for c in _cases()} >= {4, 37, 64, 300, 4096}


@needs_oracle
def test_restated_survivors_are_the_oracle():
    mine, _ = _steps12()
    bad = [c["name"] for c in _thin_cases() if not (np.array_equal(mine[c["name"]][0], c["pos"])
                                                     and np.array_equal(mine[c["name"]][1], c["v"]))]
    assert not bad, f"survivors differ from zbo_ldm_survivors: {bad}"


@needs_oracle
def test_restated_lists_are_the_oracle():
    mine, _ = _steps34()
    bad = [c["name"] for c in _cases() if mine[c["name"]] != c["lists"]]
    assert not bad, f"match lists differ from the oracle's: {bad}"
    assert sum(len(m) for c in _cases() for m in c["lists"]) > 20000


@needs_oracle
def test_restated_overlay_is_the_oracle():
    got, want, _ = _steps5()
    bad = [i for i, (a, b) in enumerate(zip(got, want)) if a != b]
    assert len(got) > 150
    assert not bad, f"{len(bad)} of {len(got)} blocks differ from zbo_ldm_overlayBlock, first: {_overlay_units()[bad[0]][0]}"


@needs_oracle
def test_every_path_is_reached():
    counts = _counts()
    print("\n" + _table(counts))
    missing = [r for r in g.ROWS if counts.get(r, 0) == 0]
    assert not missing, f"paths not reached: {missing}\n{_table(counts)}"


@needs_oracle
def test_never_rows_stay_zero():
    counts = _counts()
    assert all(counts.get(r, 0) == 0 for r in g.NEVER), _table(counts)


@needs_oracle
@pytest.mark.parametrize("switch", sorted(g.SWITCHES))
def test_inputs_tell_the_rule_from(switch):
    """a neighbouring wrong rule changes at least one block: its survivors, its match list or its overlaid sequences"""
    sw = frozenset([switch])
    changed = 0
    if switch in g.THIN_SWITCHES:
        base, _ = _steps12()
        alt = {c["name"]: g.survivors(c["src"], c["r"], sw)[0] + np.uint64(len(c["pfx"])) for c in _thin_cases() if _cheap(c)}
        for c in _thin_cases():
            if not _cheap(c):
                continue
            base_f = base[c["name"]][0]
            base_f = base_f[base_f >= len(c["pfx"])]
            a, b = set(base_f.tolist()), set(alt[c["name"]].tolist())
            changed += len({(p - len(c["pfx"])) // g.BLOCK for p in a ^ b})
    elif switch in g.OVERLAY_SWITCHES:
        got, _, _ = _steps5()
        changed = sum(g.overlay(b.be - b.bs, b.ldm_reps, lm, b.oracle_seqs, sw) != s for (_, b, lm), s in zip(_overlay_units(), got))
    else:
        mine, _ = _steps34()
        for c in _cases():
            if _cheap(c):
                changed += sum(x != y for x, y in zip(_select(c, sw), mine[c["name"]]))
    print(f"{switch}: {changed} blocks change ({g.SWITCHES[switch]})")
    assert changed > 0, g.SWITCHES[switch]


def _cheap(c):
    return c["name"].split("/")[1] in SWITCH_PARAMS


@needs_oracle
def test_checksum_is_equivalent():
    """not comparing the checksum changes no match list: a candidate that wins has the survivor's minMatch bytes"""
    mine, _ = _steps34()
    sw = frozenset(g.EQUIVALENT)
    changed = sum(sum(x != y for x, y in zip(_select(c, sw), mine[c["name"]])) for c in _cases() if _cheap(c))
    assert changed == 0


def test_inputs_are_deterministic():
    assert g.gadgets(g.CHUNK + 3 * g.BLOCK, 5) == g.gadgets(g.CHUNK + 3 * g.BLOCK, 5)
    assert g.dense(g.CHUNK + 1, 5) == g.dense(g.CHUNK + 1, 5)
    assert len(g.window_frame()) == 136 << 20


# ------------------------------------------------------------------------------------------------------------ GPU
def _ctx(level, **ldm):
    import zstd_b200
    c = zstd_b200.ZSTD_CCtx()
    c.set_parameter("compression_level", level)
    c.set_parameter("enable_long_distance_matching", 1)
    for k, v in ldm.items():
        c.set_parameter({"hash_log": 161, "min_match": 162, "bucket_size_log": 163, "hash_rate_log": 164}[k], v)
    return c


def _decodes(frame, src, d=None):
    import zstd_b200
    if zref.have_ref():
        assert (zref.ref_decompress(frame, len(src)) if d is None else zref.ref_decompress_using_dict(frame, d, len(src))) == src
    if d is None:
        assert zstd_b200.ZSTD_DCtx().decompress(frame, len(src)) == src
    else:
        dc = zstd_b200.ZSTD_DCtx()
        dc.load_dictionary(d)
        assert dc.decompress(frame, len(src)) == src


def _frame_cases():
    return [(name, src, level, prm) for name, pfx, src, level, prm in g.cases() if not pfx]


@pytest.mark.gpu
@pytest.mark.parametrize("case", [c[0] for c in _frame_cases()])
def test_gpu_frame(case):
    name, src, level, prm = next(c for c in _frame_cases() if c[0] == case)
    want = ldmref.oracle_ldm(src, level, **prm)
    got = _ctx(level, **prm).compress2(src)
    assert got == want, (case, len(got), len(want))
    _decodes(got, src)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["dense/default", "gadgets/mm4", "gadgets/passes0"])
def test_gpu_frame_stream_and_device(case):
    import torch
    import zstd_b200
    from test_gpu_ldm import _stream_one_shot
    name, src, level, prm = next(c for c in _frame_cases() if c[0] == case)
    want = ldmref.oracle_ldm(src, level, **prm)
    assert _stream_one_shot(_ctx(level, **prm), src) == want
    d_src = torch.frombuffer(bytearray(src), dtype=torch.uint8).cuda()
    cap = zstd_b200.ZSTD_compressBound(len(src)) + 64
    d_dst = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    r = _ctx(level, **prm).compress_device(d_dst.data_ptr(), cap, d_src.data_ptr(), len(src), level, s.cuda_stream)
    torch.cuda.synchronize()
    assert d_dst[:r].cpu().numpy().tobytes() == want


@pytest.mark.gpu
@pytest.mark.parametrize("case", [f"{n}/{p}" for n in g.PREFIX_PAIRS for p in ("default", "mm37")])
def test_gpu_prefix_frame(case):
    pname, p = case.split("/")
    prm = {} if p == "default" else dict(min_match=37)
    prefix, src = prefixref.pairs()[pname]
    want = prefixref.oracle_prefix(src, prefix, 1, **prm)
    c = _ctx(1, **prm)
    c.ref_prefix(prefix)
    assert c.compress2(src) == want
    if zref.have_ref():
        assert prefixref.ref_decompress_prefix(want, prefix, len(src)) == src
    import zstd_b200
    d = zstd_b200.ZSTD_DCtx()
    d.ref_prefix(prefix)
    assert d.decompress(want, len(src)) == src


@pytest.mark.gpu
def test_gpu_window_frame():
    """136 MiB: copies whose first survivors lie within 2^27 of their source, in a block whose end does not"""
    src = g.window_frame()
    want = ldmref.oracle_ldm(src, 1)
    got = _ctx(1).compress2(src)
    assert got == want, (len(got), len(want))
    _decodes(got, src)


def _dict_frames():
    dense = g.frame_inputs()["dense"]
    return [dense, dense[:300 << 10], g.frame_inputs()["b512k1"]]       # above, below and at 512 KiB + 1


def _want_dict(src, d, level=1):
    if d is None:
        return ldmref.oracle_ldm(src, level) if len(src) > LDM_MIN else zref.oracle_compress(src, level)
    return ldmref.oracle_ldm_using_dict(src, d, level) if len(src) > LDM_MIN else zref.oracle_compress_using_dict(src, d, level)


@pytest.mark.gpu
@pytest.mark.parametrize("name", DICT_NAMES)
def test_gpu_dictionary_one_frame(name):
    """ZSTD_CCtx_loadDictionary and ZSTD_CCtx_refCDict, then ZSTD_compress2"""
    import zstd_b200
    d = dictionary(name)
    cd = zstd_b200.ZSTD_CDict(d, 1)
    try:
        for src in _dict_frames():
            want = _want_dict(src, d)
            c = _ctx(1)
            c.load_dictionary(d)
            assert c.compress2(src) == want, (name, len(src))
            c = _ctx(1)
            c.ref_cdict(cd)
            assert c.compress2(src) == want, (name, len(src))
            _decodes(want, src, d)
    finally:
        cd.close()


def _batch(frames):
    src = b"".join(frames)
    offs = [sum(len(f) for f in frames[:i]) for i in range(len(frames))]
    return src, offs, [len(f) for f in frames]


def _split(out, sizes):
    res, pos = [], 0
    for s in sizes:
        res.append(out[pos:pos + s])
        pos += s
    return res


@pytest.mark.gpu
@pytest.mark.parametrize("name", DICT_NAMES)
def test_gpu_dictionary_batches(name):
    """ZSTDB200_compressFrames with a dictionary, _usingCDict, _usingCDicts (frames with and without a CDict, above and
    below 512 KiB) and its stream-ordered variant"""
    import torch
    import zstd_b200
    d = dictionary(name)
    frames = _dict_frames()
    src, offs, sizes = _batch(frames)
    cap = sum(zstd_b200.ZSTD_compressBound(n) + 64 for n in sizes)
    d_src = torch.frombuffer(bytearray(src), dtype=torch.uint8).cuda()
    d_dst = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    cd = zstd_b200.ZSTD_CDict(d, 1)
    want = [_want_dict(f, d) for f in frames]
    try:
        torch.cuda.synchronize()
        total, csz = _ctx(1).compress_frames(d_dst.data_ptr(), cap, d_src.data_ptr(), offs, sizes, 1, True, dict_bytes=d)
        assert _split(d_dst[:total].cpu().numpy().tobytes(), csz) == want
        total, csz = _ctx(1).compress_frames_using_cdict(d_dst.data_ptr(), cap, d_src.data_ptr(), offs, sizes, cd)
        assert _split(d_dst[:total].cpu().numpy().tobytes(), csz) == want
        cdicts = [cd, None, cd]
        mixed = [want[0], _want_dict(frames[1], None), want[2]]
        total, csz = _ctx(1).compress_frames_using_cdicts(d_dst.data_ptr(), cap, d_src.data_ptr(), offs, sizes, cdicts, 1)
        assert _split(d_dst[:total].cpu().numpy().tobytes(), csz) == mixed
        cdicts2 = [None, cd, None]
        mixed2 = [_want_dict(frames[0], None), want[1], _want_dict(frames[2], None)]
        res = torch.zeros(1, dtype=torch.int64, device="cuda")
        c_sizes = torch.zeros(len(sizes), dtype=torch.int64, device="cuda")
        s = torch.cuda.Stream()
        ctx = _ctx(1)
        torch.cuda.synchronize()                                     # the zero fills above ran on the default stream
        ctx.compress_frames_async_using_cdicts(d_dst.data_ptr(), cap, d_src.data_ptr(), offs, sizes, cdicts2, res.data_ptr(),
                                               level=1, d_c_sizes=c_sizes.data_ptr(), stream=s.cuda_stream)
        torch.cuda.synchronize()
        total, csz = int(res.item()), c_sizes.cpu().tolist()
        assert total == sum(csz)
        assert _split(d_dst[:total].cpu().numpy().tobytes(), csz) == mixed2
        for f, w in zip(frames, want):
            _decodes(w, f, d)
    finally:
        cd.close()


@needs_oracle
def test_dictionary_repcodes_meet_ldm_offsets():
    """the patched dictionary's repcodes are LDM offsets of the dense frame's first block, and its overlay codes one of
    them as a repcode of the dictionary's history"""
    cnt = {}
    d = dictionary("zdict-16k-ldm-reps")
    b = _frame_blocks("dense", "zdict-16k-ldm-reps")[0]
    assert b.index == 0 and b.ldm_reps == tuple(int.from_bytes(d[dg.dict_content_offset(d) - 12 + 4 * i:][:4], "little") for i in range(3))
    g.overlay(b.be - b.bs, b.ldm_reps, _dict_lists(g.frame_inputs()["dense"], len(d))[0], b.oracle_seqs, cnt=cnt)
    assert cnt.get("rep_from_history", 0) > 0


# ------------------------------------------------------------------------------- the harness: L1-L3 lists on the GPU
HARNESS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_build", "libzb_ldm_harness.so")
NONE = (1 << 64) - 1


@pytest.fixture(scope="module")
def ldm_harness():
    import ctypes
    if not os.path.exists(HARNESS):
        raise FileNotFoundError(f"{HARNESS} is missing: __graft_entry__.build() builds it")
    lib = ctypes.CDLL(HARNESS)
    vp, u64 = ctypes.c_void_p, ctypes.c_uint64
    lib.zbh_ldm.restype = ctypes.c_int
    lib.zbh_ldm.argtypes = [vp, u64, vp, u64, vp, u64, vp, u64, vp, vp]
    return lib


def _harness_lists(lib, pfx: bytes, src: bytes, prm: dict):
    """the GPU's per-block lists for src behind the indexed prefix bytes pfx; also checks that no entry outside the blocks'
    lists was written"""
    wl = g.window_log(len(pfx), len(src))
    r = ldmref.resolve(wl, **prm)
    cap = (len(pfx) + len(src)) // r.minMatch + 1
    nb = (len(src) + g.BLOCK - 1) // g.BLOCK
    match, first, cnt = np.zeros(cap, np.uint64), np.zeros(nb, np.uint64), np.zeros(nb, np.uint32)
    prm5 = np.array([r.hashLog, r.minMatch, r.bucketSizeLog, r.hashRateLog, wl], np.uint32)
    rc = lib.zbh_ldm(pfx or None, len(pfx), src, len(src), prm5.ctypes.data, g.stop_mask(r), match.ctypes.data, cap,
                     first.ctypes.data, cnt.ctypes.data)
    assert rc == 0, f"harness returned {rc}"
    used = np.zeros(cap, bool)
    out = []
    for k in range(nb):
        f, c = int(first[k]), int(cnt[k])
        assert c == 0 or f + c <= cap
        m = match[f:f + c] if c else np.zeros(0, np.uint64)
        used[f:f + c] = True
        out.append([(int(x >> np.uint64(46)), int((x >> np.uint64(28)) & np.uint64(0x3FFFF)), int(x & np.uint64(0xFFFFFFF)))
                    for x in m])
    assert np.all(match[~used] == np.uint64(NONE)), "the launch wrote match entries outside its blocks' lists"
    return out


@pytest.mark.gpu
def test_gpu_harness_lists_are_the_oracle(ldm_harness):
    """L1-L3 alone: the GPU's match lists equal the oracle's on every launch of ldmgen.harness_cases, whatever becomes of
    the frame's bytes (raw blocks, frames of any size, prefixes of any size, tile and radix edges)"""
    bad, total = [], 0
    for name, pfx, src, prm in g.harness_cases():
        want = g.oracle_lists(pfx, src, prm)
        got = _harness_lists(ldm_harness, pfx, src, prm)
        total += sum(len(m) for m in want)
        if got != want:
            k = next(i for i, (a, b) in enumerate(zip(got, want)) if a != b)
            bad.append(f"{name} block {k}")
    assert not bad, f"GPU lists differ from the oracle's: {bad}"
    assert total > 100000


@needs_oracle
def test_harness_cases_reach_their_edges():
    """the harness inputs hold what they are there for: split-point counts that end on an L1 tile and one past it, survivor
    counts that fill radix tiles and one key past, and raw blocks of the oracle's frame whose lists are not empty"""
    cases = {name: (pfx, src, prm) for name, pfx, src, prm in g.harness_cases()}
    for name, (pfx, src, prm) in cases.items():
        if name.startswith("tile"):
            mm = prm["min_match"]
            assert (len(src) - mm + 1) % g.LDM_TILE == int(name.split("+")[1][0])
        if name.startswith("radix"):
            r = g.resolved(0, len(src), prm)
            assert len(ldmref.survivors(src, r)) == int(name[5:].split("/")[0])
    src = cases["raw/default"][1]
    frame = ldmref.oracle_ldm(src, 1)
    lists = g.oracle_lists(b"", src, {})
    raw_with_matches = sum(1 for k, t in enumerate(_block_types(frame)) if t == 0 and lists[k])
    assert raw_with_matches >= 3


def _block_types(frame: bytes):
    """the block types (0 raw, 1 RLE, 2 compressed) of one frame"""
    fhd = frame[4]
    single = (fhd >> 5) & 1
    pos = 5 + (0 if single else 1) + (0, 1, 2, 4)[fhd & 3] + ((1 if single else 0), 2, 4, 8)[fhd >> 6]
    out = []
    while True:
        h = int.from_bytes(frame[pos:pos + 3], "little")
        t, size = (h >> 1) & 3, h >> 3
        out.append(t)
        pos += 3 + (1 if t == 1 else size)
        if h & 1:
            return out
