"""The GPU entropy stage (pytest -m gpu): K2 (zb_literals_kernel) and K3 (zb_sequences_kernel) on the chosen stores of
tests/entropy_cases.py, run through tests/entropy_harness.cu, which links the product's own kernel objects.  Every
block must equal, in type, size and bytes, what the oracle's model of the product's table builders gives under the
frame driver's rules; every compressed body must decode with the reference decoder to the block's bytes; and nothing
may be written behind the last block's staging area.  The stores run all together at 128 KiB strides, the small ones
again at the tight strides of a call whose largest block is 1 KiB or 4 KiB (a write past a block's stride lands in its
neighbour), and a sample one launch each.  A missing harness is an error: build() makes it."""
import ctypes
import os
from collections import defaultdict

import numpy as np
import pytest

import entropy_cases as ec
import seqgen
import zref

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600, method="thread")]
HARNESS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_build", "libzb_entropy_harness.so")
GUARD, GUARD_BYTES = 0xA5, 4096
_sz, _vp, _u32 = ctypes.c_size_t, ctypes.c_void_p, ctypes.c_uint32


class ZbBlock(ctypes.Structure):        # zb_common.h
    _fields_ = [("srcOff", ctypes.c_uint64), ("size", _u32), ("histLen", _u32), ("frame", _u32), ("flags", _u32),
                ("dictLen", _u32), ("pad", _u32)]


class ZbBlockMeta(ctypes.Structure):    # zb_common.h
    _fields_ = [(n, _u32) for n in ("nbSeq", "litSize", "litSecSize", "bodySize", "type", "forceRaw", "rleByte", "pad")]


@pytest.fixture(scope="module")
def harness():
    if not os.path.exists(HARNESS):
        raise FileNotFoundError(f"{HARNESS} is missing: __graft_entry__.build() builds it")
    lib = ctypes.CDLL(HARNESS)
    lib.zbh_entropy.restype = ctypes.c_int
    lib.zbh_entropy.argtypes = [_vp, _sz, _vp, _u32, _vp, _vp, _vp, _vp, _u32, _u32, _vp, _sz, ctypes.c_uint8,
                                _vp, _vp, _sz, ctypes.POINTER(_u32), _vp, _sz]
    return lib


@pytest.fixture(scope="module")
def want():
    """(type, payload) of every store: the oracle's model 1 under the frame driver's rules"""
    return {st.name: ec.expected(st) for st in ec.stores()}


def launch(lib, stores):
    """one K2 + K3 launch over the stores (all with one strategy, literal mode and dictionary); returns each block's
    (type, payload) and the body stride"""
    st0 = stores[0]
    assert all((s.strategy, s.lit_disabled, s.dict_name) == (st0.strategy, st0.lit_disabled, st0.dict_name) for s in stores)
    n = len(stores)
    src = b"".join(s.block for s in stores)
    blocks, off = (ZbBlock * n)(), 0
    for b, s in enumerate(stores):
        blocks[b].srcOff, blocks[b].size, blocks[b].flags = off, len(s.block), s.flags
        off += len(s.block)
    seqs = np.ascontiguousarray(np.concatenate([s.triples for s in stores]).astype(np.uint32))
    nb_seq = np.array([len(s.triples) for s in stores], np.uint32)
    lits = b"".join(s.lits for s in stores)
    lit_size = np.array([len(s.lits) for s in stores], np.uint32)
    meta = (ZbBlockMeta * n)()
    cap = n * (ec.BLOCK_MAX + 1024)
    body = ctypes.create_string_buffer(cap)
    stride = _u32(0)
    guard = ctypes.create_string_buffer(GUARD_BYTES)
    d = st0.dict
    r = lib.zbh_entropy(src, len(src), blocks, n, seqs.ctypes.data, nb_seq.ctypes.data, lits, lit_size.ctypes.data,
                        st0.strategy, st0.lit_disabled, d, len(d) if d else 0, GUARD, meta, body, cap, ctypes.byref(stride),
                        guard, GUARD_BYTES)
    assert r == 0, f"harness returned {r}"
    assert guard.raw == bytes([GUARD]) * GUARD_BYTES, "bytes behind the last block's staging area were written"
    out, raw, sd = [], body.raw, stride.value
    for b, s in enumerate(stores):
        m = meta[b]
        if m.type == seqgen.BT_COMPRESSED:
            assert m.bodySize <= sd
            out.append((m.type, raw[b * sd:b * sd + m.bodySize]))
        elif m.type == seqgen.BT_RLE:
            assert m.bodySize == 1
            out.append((m.type, bytes([m.rleByte])))
        else:
            assert m.type == seqgen.BT_RAW and m.bodySize == len(s.block), (s.name, m.type, m.bodySize)
            out.append((m.type, s.block))
    return out, sd


def groups(stores):
    g = defaultdict(list)
    for s in stores:
        g[(s.strategy, s.lit_disabled, s.dict_name or "")].append(s)
    return [g[k] for k in sorted(g)]


def differ(stores, got, want):
    """the stores whose block is not the oracle's"""
    return [f"{s.name}: type {t}, {len(p)} B (want type {want[s.name][0]}, {len(want[s.name][1])} B)"
            for s, (t, p) in zip(stores, got) if (t, p) != want[s.name]]


@pytest.mark.skipif(not zref.have_ref(), reason="reference library not built")
def test_all_stores_in_one_launch(harness, want):
    """every store, one launch per parameter set at 128 KiB strides: the oracle's bytes, and a body the reference
    decoder takes"""
    n, bad = 0, []
    for g in groups(ec.stores()):
        got, sd = launch(harness, g)
        bad += differ(g, got, want)
        for s, (t, payload) in zip(g, got):
            try:
                ok = ec.decode(s, t, payload) == s.block
            except ValueError:
                ok = False
            bad += [] if ok else [f"{s.name}: the reference decoder does not give the block's bytes"]
            n += t == seqgen.BT_COMPRESSED
    assert not bad, f"{len(bad)} blocks differ from the oracle or do not decode: " + "; ".join(bad)
    assert n > 250


@pytest.mark.parametrize("largest", [1024, 4096])
def test_tight_strides(harness, want, largest):
    """the small stores again in launches whose largest block is at most 1 KiB or 4 KiB: strides 1/128 and 1/32 of
    the 128 KiB ones, so that a write past a block's stride lands in its neighbour"""
    small = [s for s in ec.stores() if len(s.block) <= largest]
    assert len(small) > 40
    bad = []
    for g in groups(small):
        got, sd = launch(harness, g)
        m = max(len(s.block) for s in g)
        assert sd == (max(m, 64) + 63) // 64 * 64 + 1024 <= largest + 1024
        bad += differ(g, got, want)
    assert not bad, f"{len(bad)} blocks differ from the oracle: " + "; ".join(bad)


def test_single_launches(harness, want):
    """a sample of stores, each in a launch of its own: the same bytes"""
    bad = []
    for s in ec.stores()[::7]:
        got, _ = launch(harness, [s])
        bad += differ([s], got, want)
    assert not bad, f"{len(bad)} blocks differ from the oracle: " + "; ".join(bad)


def _frame(parts, size):
    """a Single_Segment frame (4-byte content size) of the given (type, payload, block size) blocks"""
    out = (0xFD2FB528).to_bytes(4, "little") + bytes([0x20 | (2 << 6)]) + size.to_bytes(4, "little")
    for k, (t, payload, n) in enumerate(parts):
        last = k == len(parts) - 1
        out += (int(last) | (t << 1) | ((n if t == seqgen.BT_RLE else len(payload)) << 3)).to_bytes(3, "little") + payload
    return out


def test_product_decoder(harness):
    """the GPU's blocks (stores without a zstd-format dictionary, and later blocks behind one), each behind its history
    sent as raw blocks, as frames of one call to the product's own decoder"""
    import zstd_b200
    stores = [s for s in ec.stores() if not (s.dict is not None and s.first)]
    frames, want = [], []
    for g in groups(stores):
        got, _ = launch(harness, g)
        for s, (t, payload) in zip(g, got):
            h = s.history
            parts = [(seqgen.BT_RAW, h[p:p + ec.BLOCK_MAX], len(h[p:p + ec.BLOCK_MAX])) for p in range(0, len(h), ec.BLOCK_MAX)]
            frames.append(_frame(parts + [(t, payload, len(s.block))], len(h) + len(s.block)))
            want.append(h + s.block)
    dctx = zstd_b200.ZSTD_DCtx()
    try:
        assert dctx.decompress(b"".join(frames), sum(len(w) for w in want)) == b"".join(want)
    finally:
        dctx.close()
