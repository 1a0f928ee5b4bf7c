"""CPU checks of the arithmetic the CUDA kernels rely on (no GPU, no product code: plain restatements).

1. K1c (zb_merge_segments_kernel, zstd_b200/csrc/zb_match.cu): the repcode history of ZSTD_storeSeq / ZSTD_updateRep
   (lib/compress/zstd_compress_internal.h:671-760) solved by two "last flagged element before me" scans per
   tile instead of a serial walk — compared here with the serial recurrence on random sequences, tile by tile with the
   history carried across tiles exactly as the kernel carries it.
2. K1a (zb_walk_kernel): key(x) = x with its offset inside the batch reversed is x ^ (BATCH - 1); the keys of a thread's P
   consecutive positions count down from the first one's; inside one batch the distance between two positions is the
   difference of their keys (what the second look of a batch uses)."""
import numpy as np
import pytest

from seqgen import serial_codes

TILE = 1024


def last_flag_before(flags):
    """1 + index of the last set flag strictly before each position (0: none): an exclusive maximum scan."""
    idx = np.where(flags, np.arange(1, len(flags) + 1), 0)
    inc = np.maximum.accumulate(idx)
    return np.concatenate(([0], inc[:-1]))


def scan_codes_tile(offs, lls, hist):
    """One tile as the kernel does it: everything below is elementwise or a scan."""
    R1, R2, R3 = hist
    offs = np.asarray(offs, dtype=np.int64); lls = np.asarray(lls, dtype=np.int64)
    n = len(offs)
    prev = np.concatenate(([R1], offs[:-1]))                      # r1 before sequence i = offset of sequence i - 1
    U = (lls > 0) & (offs == prev)                                # leaves the history alone
    m = last_flag_before(~U)                                      # last non-U sequence before i
    prev_at = lambda k: np.where(k == 0, R1, offs[np.maximum(k - 1, 0)])   # the r1 sequence k found
    r2b = np.where(m == 0, R2, prev_at(np.maximum(m - 1, 0)))
    swap = ~U & (offs == r2b)
    K = U | swap                                                  # keeps r3
    m2 = last_flag_before(~K)
    r3b = np.where(m2 == 0, R3, r2b[np.maximum(m2 - 1, 0)])
    code = offs + 3
    lit = lls > 0
    code = np.where(lit & U, 1, np.where(lit & swap, 2, np.where(lit & (offs == r3b), 3, code)))
    nolit = ~lit
    code = np.where(nolit & swap, 1, np.where(nolit & ~swap & (offs == r3b), 2,
                    np.where(nolit & ~swap & (offs != r3b) & (prev > 1) & (offs == prev - 1), 3, code)))
    last = n - 1
    new_hist = (int(offs[last]), int(r2b[last] if U[last] else prev[last]), int(r3b[last] if K[last] else r2b[last]))
    return [int(c) for c in code], new_hist


def scan_codes(offs, lls, hist):
    out = []
    for t0 in range(0, len(offs), TILE):
        c, hist = scan_codes_tile(offs[t0:t0 + TILE], lls[t0:t0 + TILE], hist)
        out += c
    return out, hist


@pytest.mark.parametrize("seed", range(12))
@pytest.mark.parametrize("hist", [(0, 0, 0), (1, 4, 8), (7, 7, 3)])
def test_repcode_scans_equal_serial_walk(seed, hist):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 3 * TILE + 17))
    # few distinct offsets (so that repcodes of every kind occur), runs of equal offsets, r1 - 1, many empty literal runs
    pool = rng.integers(1, 40, size=int(rng.integers(2, 9)))
    offs = pool[rng.integers(0, len(pool), size=n)]
    rep = rng.random(n) < 0.3
    offs[1:][rep[1:]] = offs[:-1][rep[1:]]
    dec = rng.random(n) < 0.1
    offs[1:][dec[1:]] = np.maximum(offs[:-1][dec[1:]] - 1, 1)
    lls = np.where(rng.random(n) < 0.35, 0, rng.integers(1, 50, size=n))
    want, hw = serial_codes(offs, lls, hist)
    got, hg = scan_codes(offs, lls, hist)
    assert got == want
    assert hg == hw


def test_repcode_scans_single_sequences_and_tile_edges():
    for n in (1, 2, TILE - 1, TILE, TILE + 1, 2 * TILE):
        offs = np.full(n, 5); lls = np.ones(n, dtype=np.int64)
        assert scan_codes(offs, lls, (5, 6, 7)) == serial_codes(offs, lls, (5, 6, 7))
        lls[:] = 0
        assert scan_codes(offs, lls, (5, 6, 7)) == serial_codes(offs, lls, (5, 6, 7))
        assert scan_codes(offs, lls, (6, 5, 7)) == serial_codes(offs, lls, (6, 5, 7))


def test_walk_key_identities():
    B = 1024
    x = np.arange(0, 64 * B, dtype=np.int64)
    key = (x | (B - 1)) - (x & (B - 1))                            # zb_walk_key() as written
    assert np.array_equal(key, x ^ (B - 1))
    assert np.array_equal((key | (B - 1)) - (key & (B - 1)), x)     # its own inverse
    for P in (1, 2, 4, 8, 16):
        xa = x[::P]
        for i in range(P):
            assert np.array_equal((xa + i) ^ (B - 1), (xa ^ (B - 1)) - i)      # keys of a thread's positions count down
    # inside one batch: distance = difference of the keys, and a lower position has the larger key (it wins atomicMax)
    rng = np.random.default_rng(1)
    a = rng.integers(0, B, 4096); b = rng.integers(0, B, 4096); base = rng.integers(0, 64, 4096) * B
    xa, xb = base + a, base + b
    assert np.array_equal((xb ^ (B - 1)) - (xa ^ (B - 1)), xa - xb)
    assert np.array_equal((xa < xb), ((xa ^ (B - 1)) > (xb ^ (B - 1))))
    # a later batch beats an earlier one whatever the offsets
    assert np.all(((base + B + a) ^ (B - 1)) > ((base + b) ^ (B - 1)))


def test_sequence_code_tables_match_the_format():
    """K3's shared-memory look-up tables (zbd_ll_lut_entry / zbd_ml_lut_entry, zb_sequences.cu) against the format's
    LL_bits / ML_bits and code rules (lib/common/zstd_internal.h:123-137, compress/zstd_compress_internal.h:520-549)."""
    LL_bits = [0] * 16 + [1, 1, 1, 1, 2, 2, 3, 3, 4, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16]
    ML_bits = [0] * 32 + [1, 1, 1, 1, 2, 2, 3, 3, 4, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16]
    LL_base = [0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 18, 20, 22, 24, 28, 32, 40, 48, 64, 0x80, 0x100, 0x200, 0x400,
               0x800, 0x1000, 0x2000, 0x4000, 0x8000, 0x10000]
    ML_base = [3 + v for v in list(range(32)) + [32, 34, 36, 38, 40, 44, 48, 56, 64, 80, 96, 0x80, 0x100, 0x200, 0x400, 0x800, 0x1000,
                                                 0x2000, 0x4000, 0x8000, 0x10000]]
    hb = lambda v: v.bit_length() - 1

    def ll_code(ll):
        if ll > 63: return hb(ll) + 19
        if ll < 16: return ll
        if ll < 24: return 16 + ((ll - 16) >> 1)
        if ll < 32: return 20 + ((ll - 24) >> 2)
        if ll < 48: return 22 + ((ll - 32) >> 3)
        return 24

    def ml_code(m):
        if m > 127: return hb(m) + 36
        if m < 32: return m
        if m < 40: return 32 + ((m - 32) >> 1)
        if m < 48: return 36 + ((m - 40) >> 2)
        if m < 64: return 38 + ((m - 48) >> 3)
        if m < 96: return 40 + ((m - 64) >> 4)
        return 42

    for ll in list(range(0, 300)) + [1000, 65535, 65536, 131071]:
        c = ll_code(ll)
        bits = (hb(ll) if ll > 63 else (0 if c < 16 else 1 if c < 20 else 2 if c < 22 else 3 if c < 24 else 4))
        assert bits == LL_bits[c]
        assert LL_base[c] <= ll < LL_base[c] + (1 << LL_bits[c])
    for m in list(range(0, 600)) + [1000, 65535, 65536, 131071 - 3]:
        c = ml_code(m)
        bits = (hb(m) if m > 127 else (0 if c < 32 else 1 if c < 36 else 2 if c < 38 else 3 if c < 40 else 4 if c < 42 else 5))
        assert bits == ML_bits[c]
        assert ML_base[c] <= m + 3 < ML_base[c] + (1 << ML_bits[c])
