"""A restatement of the oracle's candidate walk (walk() and zbo_walkChunk, oracle/zb_match.c) batch by batch in numpy, with
counters of the paths every position and batch takes, the batch kinds of the CUDA walk (zb_walk_kernel, K1a in
zstd_b200/csrc/zb_match.cu), switches that each replace one rule by a neighbouring wrong one, and inputs built from
hash-planted gadgets.  TEST INFRASTRUCTURE ONLY.

tests/test_gpu_walk_paths.py proves the restatement equal to zbo_walkChunk at every position, so its counts are the
oracle's; the GPU walk is then held to the oracle position by position, and its dictionary images to the restatement's
tables word by word."""
import ctypes
import random

import numpy as np

import zref
from dfastgen import ChunkCand, _oracle, other_tag, twin_hash, with_hash4, with_hash5, with_hash8
from test_plan import OPlan

BATCH = 1024
BLOCK = 128 << 10
CHUNK_BLOCKS = 4
PRIME = 128 << 10
FAR = 0xFFFF
TAG = 0x7FF
MIN_CLEVEL = -(1 << 17)                                         # ZSTD_minCLevel(): -ZSTD_TARGETLENGTH_MAX
N_MAX = 57856                                                   # 226 KiB of dynamic shared memory per walk CTA
M32, M64 = (1 << 32) - 1, (1 << 64) - 1
P6, P7 = 227718039650203, 58295818150454627
_PRIMES = {4: 2654435761, 5: 889523592379, 6: P6, 7: P7, 8: 0xCF1BBCDCB7A56463}


# ---------------------------------------------------------------------------------------------------- hash gadgets
def with_hash6(h: int, low16: int) -> bytes:
    """6 bytes whose 6-byte hash is h: hash6 = (v48 * P6 mod 2^48) >> 16, a bijection of the 6 bytes"""
    return ((((h << 16) | (low16 & 0xFFFF)) * pow(P6, -1, 1 << 48)) & ((1 << 48) - 1)).to_bytes(6, "little")


def with_hash7(h: int, low24: int) -> bytes:
    """7 bytes whose 7-byte hash is h: hash7 = (v56 * P7 mod 2^56) >> 24"""
    return ((((h << 24) | (low24 & 0xFFFFFF)) * pow(P7, -1, 1 << 56)) & ((1 << 56) - 1)).to_bytes(7, "little")


def with_hash(mls: int, h: int, rnd: random.Random) -> bytes:
    """mls bytes (8 for mls 8) whose mls-byte hash is h; the bytes the hash leaves free are random"""
    if mls == 4:
        return with_hash4(h)
    if mls == 5:
        return with_hash5(h, rnd.getrandbits(8))
    if mls == 6:
        return with_hash6(h, rnd.getrandbits(16))
    if mls == 7:
        return with_hash7(h, rnd.getrandbits(24))
    return with_hash8(rnd.getrandbits(32), h)


# ---------------------------------------------------------------------------------------------------------- inputs
DISTANCES = (1, 1023, 1024, 65534, 65535, 65536)


def walk_input(n: int, seed: int, mls: int, hist: bytes = b"") -> bytes:
    """n bytes: synthetic text, zero runs and incompressible runs, overwritten with gadgets.  Each gadget sits in zeros, which
    find their candidates and insert nothing, so its table entries live until they are looked up:
      - 16 random bytes repeated at each distance of DISTANCES;
      - a planted mls-byte hash h, and 50-900 bytes on bytes with twin_hash(h): same bucket and tag, different bytes;
      - h, then other_tag(h) (same bucket, another tag), then h again.
    `hist` is the history in front (a dictionary tail): the first copies reach into it."""
    rnd = random.Random(seed * 7919 + mls)
    out = bytearray()
    while len(out) < n:
        k = rnd.random()
        if k < 0.45:
            out += zref.synthetic(rnd.randint(2000, 30000), rnd.getrandbits(31), rnd.choice((0.3, 0.5, 0.8)))
        elif k < 0.65:
            out += bytes([rnd.choice((0, 0x61))]) * rnd.randint(500, 8000)
        else:
            out += rnd.getrandbits(8 * (m := rnd.randint(3000, 40000))).to_bytes(m, "little")
    del out[n:]
    buf = bytearray(hist) + out
    h0 = len(hist)

    def plant(p, g):
        lo, hi = max(h0 if p >= h0 else 0, p - 48), min(len(buf), p + len(g) + 48)
        if hi - lo < len(g) + 16:
            return
        buf[lo:hi] = bytes(hi - lo)
        buf[p:p + len(g)] = g

    for d in DISTANCES:
        for _ in range(3 if d > 60000 else 6):
            q = rnd.randint(h0 + 64, max(h0 + 64, len(buf) - 80))
            if q - d < 64:
                continue
            g = rnd.getrandbits(128).to_bytes(16, "little")
            if d >= 128:
                plant(q - d, g)
            plant(q, g)
            if d < 128:
                buf[q - d:q - d + 16] = g
    for _ in range(max(2, n // 20000)):
        q = rnd.randint(h0 + 64, max(h0 + 64, len(buf) - 2100))
        h = rnd.getrandbits(32)
        plant(q, with_hash(mls, h, rnd))
        if rnd.random() < 0.5:
            plant(q + rnd.randint(50, 900), with_hash(mls, twin_hash(h), rnd))
        else:
            r = q + rnd.randint(100, 900)
            plant(r, with_hash(mls, other_tag(h), rnd))
            plant(r + rnd.randint(100, 900), with_hash(mls, h, rnd))
    return bytes(buf[h0:h0 + n])


def far_max_input(mls: int) -> bytes:
    """1 MiB of zeros with the same 8 random bytes at 384 KiB and at 1 MiB - 8: the second chunk walks 128 KiB of history
    and 512 KiB, and its last active position finds the history's first, 640 KiB - 8 back (the largest distance)"""
    rnd = random.Random(mls)
    buf = bytearray(1 << 20)
    g = rnd.getrandbits(64).to_bytes(8, "little")
    buf[384 << 10:(384 << 10) + 8] = g
    buf[-8:] = g
    return bytes(buf)


def incompressible(n: int, seed: int) -> bytes:
    return random.Random(seed).getrandbits(8 * n).to_bytes(n, "little")


# --------------------------------------------------------------------------------------------------- parameters
def oracle_cparams(level: int, size: int, dict_size: int):
    return _oracle().zbo_getCParams(level, size, dict_size)


def make_plan(cp, tun=None) -> OPlan:
    """zbo_makePlan, optionally under zbo_tun overrides {field: value} (tableN, tableNLong, insStep); zbo_tun is reset after"""
    O = _oracle()
    pl = OPlan()
    t = Tun.in_dll(O, "zbo_tun")
    saved = Tun.from_buffer_copy(t)
    try:
        for k, v in (tun or {}).items():
            assert k in ("tableN", "tableNLong", "insStep")
            setattr(t, k, v)
        O.zbo_makePlan(ctypes.byref(pl), ctypes.byref(cp))
    finally:
        ctypes.memmove(ctypes.addressof(t), ctypes.addressof(saved), ctypes.sizeof(Tun))
    return pl


class Tun(ctypes.Structure):
    _fields_ = [(n, ctypes.c_uint) for n in ("tableN", "tableNLong", "tableFmt", "insStep", "primeBytes", "chunkBlocks", "batch", "spare")]


PLAN_DICTS = (0, 16 << 10, 112 << 10, 300 << 10)


def product_levels():
    """levels from ZSTD_minCLevel to 22: every level down to -1100 (insertion steps up to 1100, 1023-1025 included), and
    below that the levels where the insertion step takes its largest values"""
    return [MIN_CLEVEL, MIN_CLEVEL + 1, -65536, -4097, -2048] + list(range(-1100, 23))


def product_sets():
    """every distinct walk (mls, N, insStep) the planner yields over product_levels() x the sizes and dictionary sizes of
    tests/test_plan.py, as (strategy, mls, tableN, tableNLong, insStep); doubleFast sets carry both tables"""
    from test_plan import SIZES
    out = set()
    for level in product_levels():
        for size in SIZES:
            for ds in PLAN_DICTS:
                pl = make_plan(oracle_cparams(level, size, ds))
                out.add((pl.strategy, pl.mls, pl.tableN, pl.tableNLong if pl.strategy == 2 else 0, pl.insStep))
    return sorted(out)


def harness_sets():
    """sets no product call makes, reached in the oracle through zbo_tun: N = 14337 and 28928 (4 positions per thread at both
    ends of its range) and 14336 (8 at its top end), 28929, 40000, 57856 (1 position per thread), each with every mls; insStep 1, 1024, 1025; an odd N"""
    out = []
    for N in (14336, 14337, 28928, 28929, 40000, N_MAX):
        for mls in range(4, 9):
            out.append((1, mls, N, 0, 3))
    for ins in (1, 1024, 1025):
        out.append((1, 5, 12345, 0, ins))
    out.append((1, 6, 12345, 0, 2))
    return out


def threads_p(N: int) -> int:
    """positions per thread of the walk launch (zb_launch_walk_m): 8 up to 56 KiB of table, 4 up to 113 KiB, else 1"""
    return 8 if N * 4 <= 56 * 1024 else (4 if N * 4 <= 113 * 1024 else 1)


def plan_for(s) -> OPlan:
    """the oracle's plan of a set: the product's sets and the harness-only ones both come out of zbo_makePlan"""
    strategy, mls, N, NL, ins = s
    if strategy == 2:
        cp = oracle_cparams(3, 1 << 20, 0)
        cp.minMatch = mls
        return make_plan(cp, {"tableN": N, "tableNLong": NL, "insStep": ins})
    cp = oracle_cparams(1, 1 << 20, 0)
    cp.minMatch = mls
    return make_plan(cp, {"tableN": N, "insStep": ins})


# ---------------------------------------------------------------------------------------------------------- oracle
def oracle_walk(plan: OPlan, tail: bytes, frame: bytes, pos: int, size: int):
    """zbo_walkChunk over the chunk frame[pos, pos + size) behind the dictionary tail: (dS, dL or None) per position"""
    O = _oracle()
    plan.frameStart = len(tail)
    buf = tail + frame
    cc = ChunkCand()
    D = len(tail)
    O.zbo_walkChunk(ctypes.byref(plan), buf, len(buf), D + pos, D + pos + size, ctypes.byref(cc))
    try:
        dS = np.ctypeslib.as_array(cc.dS, shape=(size,)).copy() if size else np.zeros(0, np.uint32)
        dL = (np.ctypeslib.as_array(cc.dL, shape=(size,)).copy() if size else np.zeros(0, np.uint32)) if plan.strategy == 2 else None
    finally:
        O.zbo_freeChunk(ctypes.byref(cc))
    return dS, dL


def chunk_bounds(frame_len: int, block_log: int):
    """the chunks of a frame as the planner cuts them: (pos, size)"""
    cb = CHUNK_BLOCKS << block_log
    out, pos = [], 0
    while True:
        out.append((pos, min(cb, frame_len - pos)))
        pos += cb
        if pos >= frame_len:
            return out


# ------------------------------------------------------------------------------------------------ the restatement
ROWS = [
    "tail_inactive",        # one of the last 7 positions: its 8 bytes are not readable
    "straddle_inactive",    # its 8 bytes straddle the dictionary / frame border
    "prime_batch",          # a batch with no output (history)
    "a_cand",               # phase A: the bucket holds an entry with the position's tag
    "a_65534", "a_65535", "a_65536",
    "far",                  # a distance >= 65535 (the far array)
    "a_other_tag",          # phase A: the bucket holds an entry with another tag
    "tag_collision",        # a candidate whose mls bytes differ (the walk emits it, the parse checks the bytes)
    "multi_insert",         # a bucket that takes several insertions in one batch
    "c_cand",               # phase C: this batch's lowest insertion into the bucket serves the position
    "c_below",              # phase C: the batch's insertion into the bucket lies above the position: nothing
    "c_other_tag",          # phase C: the bucket holds this batch's entry of another tag: nothing
    "step_eq",              # a batch whose step is insStep (the residue by addition)
    "step_raised",          # a batch whose step acceleration raised (the division)
    "step_gt_batch",        # a batch whose step exceeds 1024
    "accel_reset_hit",      # a raised step that a hit resets
    "accel_reset_dict",     # a raised step reset at the frame start behind a dictionary
]
ZERO_ROWS = [
    "a_then_c",             # a position with a phase-A candidate that the kernel's phase-C formula would serve otherwise
    "c_formula",            # a phase-C result of the kernel's rotated difference that differs from the oracle's look
    "a_above",              # a phase-A entry with the position's tag at or above it (the kernel does not test for it)
    "x_ge_2_20",            # a walk coordinate >= 2^20
]
KIND_ROWS = ["slow", "interior", "steady_pair", "cut_end", "first_inside", "image_prime"]

SWITCHES = {
    "hi_wins": "the highest position of a batch wins a bucket",
    "no_second": "no second look (phase C)",
    "second_above": "the second look takes an entry above the position too",
    "no_tags": "tags ignored",
    "accel_from_start": "acceleration counted from the hit batch's start instead of its end",
    "no_dict_reset": "no acceleration reset at the frame start behind a dictionary",
    "res_from_frame": "the insertion residue taken from the frame start instead of low",
    "insert_found": "positions that found a candidate are inserted too",
    "straddle_active": "positions straddling the dictionary / frame border are active",
    "step64": "a step of 64 positions instead of 128",
}


def _words(buf: np.ndarray, lo: int, hi: int) -> np.ndarray:
    """the little-endian 8-byte words at [lo, hi), zeros past the buffer"""
    b = np.zeros(hi - lo + 8, np.uint8)
    t = buf[lo:min(len(buf), hi + 7)]
    b[:len(t)] = t
    return np.lib.stride_tricks.sliding_window_view(b, 8)[:hi - lo].copy().view("<u8")[:, 0]


def hashes(v: np.ndarray, mls: int) -> np.ndarray:
    with np.errstate(over="ignore"):
        if mls == 4:
            return ((v & np.uint64(M32)) * np.uint64(_PRIMES[4])) & np.uint64(M32)
        return ((v << np.uint64(64 - 8 * mls)) * np.uint64(_PRIMES[mls])) >> np.uint64(32)


def _keyof(x):
    return x ^ (BATCH - 1)


def _cand(c, h, x, no_tags=False, above=False):
    k = _keyof((c >> 11) - 1)
    ok = (c != 0) & (no_tags | (((c ^ h) & TAG) == 0))
    if above:
        return np.where(ok & (k != x), np.abs(x - k), 0)
    return np.where(ok & (k < x), x - k, 0)


def walk(buf: bytes, low: int, out_start: int, end: int, D: int, mls: int, N: int, ins_step: int, sw=frozenset(), cnt=None):
    """the oracle's walk() over buf[low, end) (readEnd = end): (distances of [out_start, end), the table after the last batch)"""
    b = np.frombuffer(buf, np.uint8)
    v = _words(b, low, end)
    h = hashes(v, mls).astype(np.int64)
    bkt = (h * N) >> 32
    q = np.arange(low, end, dtype=np.int64)
    shift = (BATCH - (D - low) % BATCH) % BATCH if D > low else 0
    x = q - low + shift
    straddle = (q < D) & (q + 8 > D)
    act = (q + 8 <= end) & (~straddle | ("straddle_active" in sw))
    mask = np.uint64((1 << (8 * mls)) - 1) if mls < 8 else np.uint64(M64)
    table = np.zeros(N, np.int64)
    out = np.zeros(end - out_start, np.int64)
    no_tags = "no_tags" in sw
    last_hit, s = low, low
    if cnt is not None:
        cnt["tail_inactive"] += int(np.count_nonzero(q + 8 > end))
        cnt["straddle_inactive"] += int(np.count_nonzero(straddle))
        cnt["x_ge_2_20"] += int(np.count_nonzero(x >= (1 << 20)))
    while s < end:
        e = min(s + BATCH - ((s - low + shift) % BATCH), end)
        if s == D and "no_dict_reset" not in sw:
            if cnt is not None and insstep_of(ins_step, s, last_hit, sw) > ins_step:
                cnt["accel_reset_dict"] += 1
            last_hit = D
        i0, i1 = s - low, e - low
        hb, kb, ab, xb, qb = h[i0:i1], bkt[i0:i1], act[i0:i1], x[i0:i1], q[i0:i1]
        c = table[kb]
        d_old = np.where(ab, _cand(c, hb, xb, no_tags), 0)
        step = insstep_of(ins_step, s, last_hit, sw)
        hit = bool(d_old.any())
        base = D if "res_from_frame" in sw else low
        ins = ab & ((d_old == 0) | ("insert_found" in sw)) & (((qb - base) % step) < 2)
        if hit:
            if cnt is not None and step > ins_step:
                cnt["accel_reset_hit"] += 1
            last_hit = s if "accel_from_start" in sw else e
        entry = ((_keyof(xb) + 1) << 11) | (hb & TAG)
        if "hi_wins" in sw:
            table[kb[ins]] = entry[ins]
        else:
            np.maximum.at(table, kb[ins], entry[ins])
        need = ab & (d_old == 0)
        c2 = table[kb]
        if "no_second" in sw:
            d_c = np.zeros_like(d_old)
        else:
            d_c = np.where(need, _cand(c2, hb, xb, no_tags, "second_above" in sw), 0)
        d = np.where(need, d_c, d_old)
        if e > out_start:
            o0 = max(s, out_start)
            out[o0 - out_start:e - out_start] = d[o0 - s:]
        if cnt is not None:
            _count(cnt, b, v, mask, low, s, e, out_start, ab, hb, kb, xb, c, c2, d_old, d_c, need, ins, entry, step, ins_step, d)
        s = e
    return out, table


def insstep_of(ins_step, s, last_hit, sw):
    return ins_step + ((s - last_hit) >> (6 if "step64" in sw else 7))


def _count(cnt, b, v, mask, low, s, e, out_start, ab, hb, kb, xb, c, c2, d_old, d_c, need, ins, entry, step, ins_step, d):
    if e <= out_start:
        cnt["prime_batch"] += 1
    cnt["a_cand"] += int(np.count_nonzero(d_old))
    for k in (65534, 65535, 65536):
        cnt[f"a_{k}"] += int(np.count_nonzero(d_old == k))
    if e > out_start:
        o0 = max(s, out_start) - s
        cnt["far"] += int(np.count_nonzero(d[o0:] >= FAR))
    cnt["a_other_tag"] += int(np.count_nonzero(ab & (c != 0) & (((c ^ hb) & TAG) != 0)))
    k_old = _keyof((c >> 11) - 1)
    cnt["a_above"] += int(np.count_nonzero(ab & (c != 0) & (((c ^ hb) & TAG) == 0) & (k_old >= xb)))
    hit = d != 0
    if hit.any():
        i = np.nonzero(hit)[0]
        p = s + i - low
        cnt["tag_collision"] += int(np.count_nonzero(((v[p] ^ v[p - d[i]]) & mask) != 0))
    if ins.any():
        _, counts = np.unique(kb[ins], return_counts=True)
        cnt["multi_insert"] += int(np.count_nonzero(counts > 1))
    cnt["c_cand"] += int(np.count_nonzero(d_c))
    same = (c2 != 0) & (((c2 ^ hb) & TAG) == 0)
    this_batch = (_keyof((c2 >> 11) - 1) // BATCH) == (xb // BATCH)
    cnt["c_below"] += int(np.count_nonzero(need & same & this_batch & (_keyof((c2 >> 11) - 1) > xb)))
    cnt["c_other_tag"] += int(np.count_nonzero(need & (c2 != 0) & ~same & this_batch))
    # the kernel's phase C: the rotated difference of the bucket and the position's own entry, taken when below the batch
    diff = (c2 - entry) & M32
    r = ((diff >> 11) | (diff << 21)) & M32
    gpu = np.where(ab & (r < BATCH), r, d_old)
    cnt["a_then_c"] += int(np.count_nonzero((d_old != 0) & ab & (r < BATCH)))
    cnt["c_formula"] += int(np.count_nonzero(need & (gpu != d_c)))
    cnt["step_eq"] += int(step == ins_step)
    cnt["step_raised"] += int(step > ins_step)
    cnt["step_gt_batch"] += int(step > BATCH)


def walk_chunk(plan_mls: int, N: int, ins_step: int, tail: bytes, frame: bytes, pos: int, size: int, sw=frozenset(), cnt=None):
    """zbo_walkChunk's bounds: the chunk frame[pos, pos + size) behind the tail, primed from PRIME bytes in front of it"""
    D = len(tail)
    start = D + pos
    low = start - PRIME if start > PRIME else 0
    buf = tail + frame[:pos + size]
    return walk(buf, low, start, start + size, D, plan_mls, N, ins_step, sw, cnt)


def image_table(mls: int, N: int, ins_step: int, tail: bytes) -> np.ndarray:
    """the table a walk of the dictionary tail alone leaves: what a dictionary image holds"""
    return walk(tail, 0, len(tail), len(tail), len(tail), mls, N, ins_step)[1]


def batch_kinds(N: int, D: int, H: int, size: int, from_image: bool, steady: bool = True, cnt=None):
    """the batch kinds zb_walk_kernel runs for one chunk, from its own bounds (xLow, xIntLoB, xIntHi, xEnd)"""
    P = threads_p(N)
    total = H + size
    shift = (BATCH - D % BATCH) % BATCH
    x_end = total + shift
    x_low = (D if from_image else 0) + shift
    x0 = x_low & ~(BATCH - 1)
    x_int_lo = max(D + shift, x_low)
    x_int_lo_b = (x_int_lo + BATCH - 1) & ~(BATCH - 1)
    nw = (P + 7 + 3 + 3) // 4
    x_int_hi = (x_end + P - 4 * nw) & ~(BATCH - 1) if x_end >= BATCH + 4 * nw else 0
    k = cnt if cnt is not None else {r: 0 for r in KIND_ROWS}
    k["first_inside"] += int(x_low % BATCH != 0)
    k["image_prime"] += int(from_image)

    def do_batch():
        nonlocal x0
        if x0 >= x_int_lo_b and x0 + BATCH <= x_int_hi:
            k["interior"] += 1
        else:
            k["slow"] += 1
        if x0 >= H + shift and x0 + BATCH > x_end:
            k["cut_end"] += 1
        x0 += BATCH
    while x0 < x_end:
        if steady and x0 >= x_int_lo_b and x0 + 4 * BATCH <= x_int_hi:
            while True:
                k["steady_pair"] += 1
                x0 += 2 * BATCH
                if not x0 + 4 * BATCH <= x_int_hi:
                    break
        do_batch()
        if x0 >= x_end:
            break
        do_batch()
    return k
