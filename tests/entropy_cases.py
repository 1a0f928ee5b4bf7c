"""Chosen literal and sequence stores for the entropy stage (K2 zb_literals_kernel, K3 zb_sequences_kernel), built to
reach the paths whose thresholds and table builders no whole-input test is made to reach.  Each store is one block
built from real offsets: its offBase values come from the ZSTD_storeSeq rule (seqgen.serial_codes) with the history
the decoder starts from, and its bytes from seqgen.execute.  Each names the layout it must come out with (a case that
silently fell back to raw tests nothing), checked on the body the product's table builders give (the oracle's model 1),
which the GPU must equal byte for byte.  TEST INFRASTRUCTURE ONLY."""
import ctypes
import functools
import heapq

import numpy as np

import seqgen
import zref

FIRST, DICT = 1, 4
BLOCK_MAX = 128 << 10
DICTS = ("zdict-16k-synthetic-seed77", "http-dict-missing-symbols", "zero-weight-dict")
LL_BASE = [0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 18, 20, 22, 24, 28, 32, 40, 48, 64, 0x80, 0x100, 0x200,
           0x400, 0x800, 0x1000, 0x2000, 0x4000, 0x8000, 0x10000]
ML_BASE = [3 + v for v in list(range(32)) + [32, 34, 36, 38, 40, 44, 48, 56, 64, 80, 96, 0x80, 0x100, 0x200, 0x400, 0x800, 0x1000,
                                             0x2000, 0x4000, 0x8000, 0x10000]]
_sz, _vp = ctypes.c_size_t, ctypes.c_void_p


def ll_code(ll):
    return ll if ll < 16 else max(c for c in range(36) if LL_BASE[c] <= ll)


def ml_code(ml):
    return max(c for c in range(53) if ML_BASE[c] <= ml)


class Store:
    """One block: sequences (litLength, real offset, matchLength), all its literal bytes in order (the trailing run
    last), the entropy parameters, and what it must come out as (`want`: "type" and block_layout fields)."""

    def __init__(self, name, seqs, lits, strategy=1, first=True, lit_disabled=0, dict_name=None, want=None, seed=0,
                 check_modes=None):
        self.name, self.seqs, self.lits = name, list(seqs), bytes(lits)
        self.check_modes = check_modes          # predicate on block_layout's (LL, OF, ML) modes, where a case needs one
        self.strategy, self.first, self.lit_disabled, self.dict_name = strategy, first, lit_disabled, dict_name
        self.want = dict(want or {})
        self.dict = zref.golden_input(dict_name) if dict_name else None
        if self.dict is not None:
            self.history = seqgen.dict_content(self.dict)
        else:                               # random history as far back as the furthest match reaches
            pos, need = 0, 0
            for ll, off, ml in self.seqs:
                pos += ll
                need = max(need, off - pos)
                pos += ml
            self.history = zref.random_bytes(max(need, 8), seed + 1000) if need > 0 else b""
        reps = (1, 4, 8)
        if self.dict is not None and self.first:
            reps = tuple(int.from_bytes(self.dict[k:k + 4], "little") for k in self._rep_at())
        offb, _ = seqgen.serial_codes([s[1] for s in self.seqs], [s[0] for s in self.seqs], reps)
        self.triples = np.array([(o, s[0], s[2]) for o, s in zip(offb, self.seqs)], dtype=np.uint32).reshape(-1, 3)
        trailing = len(self.lits) - sum(s[0] for s in self.seqs)
        self.block = seqgen.execute([(self.seqs, trailing)], None, self.history, literals=self.lits)
        # what the match finder guarantees and the kernels rely on: without it a case could overrun a stride
        assert trailing >= 0 and len(self.block) == len(self.lits) + sum(s[2] for s in self.seqs) <= BLOCK_MAX
        assert 7 <= len(self.block) and len(self.seqs) <= len(self.block) // 4
        assert all(ml >= 4 and ll < (1 << 18) for ll, _, ml in self.seqs)
        assert all(o < (1 << 24) for o in offb)
        assert self.lit_disabled == 0 or self.strategy == 1       # the reference disables literal compression for fast only

    def _rep_at(self):
        n = seqgen.ref().ZDICT_getDictHeaderSize(self.dict, len(self.dict))
        return (n - 12, n - 8, n - 4)

    @property
    def flags(self):
        return (FIRST if self.first else 0) | (DICT if self.dict is not None else 0)

    @property
    def decode_dict(self):
        """what the decoder needs in front of the block: the zstd-format dictionary (its tables and repeat offsets) for
        a first block behind one, else the history as raw content"""
        if self.dict is not None and self.first:
            return self.dict
        return self.history if len(self.history) >= 8 else None


# ---------------------------------------------------------------------------------------------------- the oracle and the reference
def _oracle():
    O = zref.oracle()
    O.zbo_loadDictEntropy.restype = _sz
    O.zbo_loadDictEntropy.argtypes = [_vp, _vp, _sz]
    O.zbo_entropyCompressBlock_prev.restype = _sz
    O.zbo_entropyCompressBlock_prev.argtypes = [_vp, _sz, _vp, _sz, _vp, _sz, _sz, ctypes.c_uint, ctypes.c_int, _vp]
    return O


@functools.lru_cache(maxsize=None)
def dict_entropy(name):
    """the oracle's zbo_dict_entropy of a dictionary (raw bytes of the struct)"""
    d = zref.golden_input(name)
    de = ctypes.create_string_buffer(16384)
    assert 8 < _oracle().zbo_loadDictEntropy(de, d, len(d)) < len(d)
    return de


def dict_huf_bits(name):
    """code length of every literal in the dictionary's Huffman table (0: absent); zbo_dict_entropy.huf.nbBits"""
    return list(dict_entropy(name).raw[8:264])


def dict_fse_repeat(name):
    """FSE_repeat of the dictionary's LL, OF, ML tables (2 = valid for every symbol)"""
    o = 8 + 256 + 512 + 8 + 4 + 3 * (8 + 1024 + 256 + 256)
    return [int.from_bytes(dict_entropy(name).raw[o + 4 * k:o + 4 * k + 4], "little") for k in range(3)]


def oracle_body(st, model=1):
    """zbo_entropyCompressBlock_prev on the store: model 0 = the restatement of the reference's table builders, 1 = the
    product's (oracle/zb_tables.c).  b"" = the block goes raw."""
    O = _oracle()
    cap = 1 << 20
    d = ctypes.create_string_buffer(cap)
    lits = np.frombuffer(st.lits, dtype=np.uint8) if st.lits else np.zeros(1, np.uint8)
    de = dict_entropy(st.dict_name) if (st.dict is not None and st.first) else None
    with zref.entropy_model(model):
        r = O.zbo_entropyCompressBlock_prev(d, cap, st.triples.ctypes.data, len(st.triples), lits.ctypes.data, len(st.lits),
                                            len(st.block), st.strategy, st.lit_disabled, de)
    assert r < (1 << 63), f"oracle error {(1 << 64) - r}"
    return d.raw[:r]


def ref_body(st):
    """the reference's ZSTD_entropyCompressSeqStore on the store (oracle/ref_shim.c), behind ZSTD_loadCEntropy of the
    dictionary for a first block behind a zstd-format one"""
    R = zref.ref()
    cap = 1 << 20
    d = ctypes.create_string_buffer(cap)
    offb, ll, ml = (np.ascontiguousarray(st.triples[:, k]) for k in range(3))
    lits = np.frombuffer(st.lits, dtype=np.uint8) if st.lits else np.zeros(1, np.uint8)
    tl = 3 if st.lit_disabled else 0                 # strategy fast with a target length: literal compression off
    args = (d, cap, offb.ctypes.data, ll.ctypes.data, ml.ctypes.data, len(st.triples), lits.ctypes.data, len(st.lits),
            len(st.block), st.strategy, tl)
    if st.dict is not None and st.first:
        R.ref_entropyCompressBlock_dict.restype = _sz
        R.ref_entropyCompressBlock_dict.argtypes = [_vp, _sz, _vp, _vp, _vp, _sz, _vp, _sz, _sz, ctypes.c_int, ctypes.c_uint, _vp, _sz]
        r = R.ref_entropyCompressBlock_dict(*args, st.dict, len(st.dict))
    else:
        r = R.ref_entropyCompressBlock(*args)
    assert not R.ZSTD_isError(r), R.ZSTD_getErrorName(r)
    return d.raw[:r]


def block_result(st, body):
    """(block type, payload) the frame driver makes of an entropy-stage result (oracle/zb_frame.c): raw when it is
    empty; RLE when the block is not its frame's first, the result is under 25 bytes and all the block's bytes are
    equal"""
    if not st.first and len(body) < 25 and st.block.count(st.block[:1]) == len(st.block):
        return seqgen.BT_RLE, st.block[:1]
    if not body:
        return seqgen.BT_RAW, st.block
    return seqgen.BT_COMPRESSED, body


def expected(st):
    return block_result(st, oracle_body(st, 1))


def decode(st, btype, payload):
    """the reference decoder on the block wrapped as the only block of a Single_Segment frame"""
    return seqgen.ref_decompress(seqgen.single_block_frame(btype, payload, len(st.block)), len(st.block), st.decode_dict)


def check_layout(st, btype, payload):
    """the block reached the path its case names"""
    want = dict(st.want)
    if "type" in want:
        assert btype == want.pop("type"), (st.name, btype)
    if want:
        assert btype == seqgen.BT_COMPRESSED, (st.name, btype)
        lay = seqgen.block_layout(payload)
        for k, v in want.items():
            assert lay[k] == v, (st.name, k, lay[k], v)
    if st.check_modes is not None:
        assert btype == seqgen.BT_COMPRESSED and st.check_modes(seqgen.block_layout(payload)["modes"]), st.name


# ---------------------------------------------------------------------------------------------------- literal bytes
def from_counts(counts, rng):
    """literal bytes with exactly these counts {byte: count}, in a random order"""
    a = np.concatenate([np.full(c, s, np.uint8) for s, c in counts.items()]) if counts else np.zeros(0, np.uint8)
    return rng.permutation(a).tobytes()


def skewed(n, rng, nsym=24):
    p = 1.0 / np.arange(1, nsym + 1) ** 1.3
    return rng.choice(nsym, size=n, p=p / p.sum()).astype(np.uint8).tobytes()


def huffman_depth(counts):
    """depth of a minimum-redundancy code of the counts, for counts whose tree is unique"""
    h = [(c, 0) for c in counts if c]
    heapq.heapify(h)
    while len(h) > 1:
        a, b = heapq.heappop(h), heapq.heappop(h)
        heapq.heappush(h, (a[0] + b[0], max(a[1], b[1]) + 1))
    return h[0][1]


def opt_table_log(max_log, n, max_sym, minus):
    """FSE_optimalTableLog_internal (zbd_fse_optimalTableLog): the Huffman target for n literals is this with 11, 1"""
    hb = lambda v: v.bit_length() - 1
    log = min(max_log, hb(n - 1) - minus)
    log = max(log, min(hb(n) + 1, hb(max_sym) + 2))
    return min(max(log, 5), 12)


def _lit_only(n_lits, rng, off=16):
    """one sequence in front of the trailing literals, its match as long as they are: a block whose literals go raw
    still compresses"""
    return [(min(n_lits, 4), off, min(n_lits + 64, BLOCK_MAX - n_lits))]


# ---------------------------------------------------------------------------------------------------- cases
# A builder takes (strategy, first, rng) and returns Store keyword arguments: seqs, lits, want (and lit_disabled, dict_name).
def nbseq(n):
    def b(s, first, rng):
        offs = rng.integers(1, 3000, n)
        seqs = [(0, int(o), 4) for o in offs]
        tail = min(100, BLOCK_MAX - 4 * n)
        return dict(seqs=seqs, lits=skewed(tail, rng), want={"type": 2, "nb_seq": n, "nb_seq_bytes": 2 if n < 0x7F00 else 3})
    return b


def ll_code_35(s, first, rng):
    seqs = [(70000, 5000, 40), (10, 300, 1000), (0, 7, 20)]
    assert ll_code(70000) == 35
    return dict(seqs=seqs, lits=skewed(70010 + 500, rng), want={"type": 2})


def ml_code_52(s, first, rng):
    seqs = [(20, 1000, 70000), (5, 3, 30000), (3, 50, 100)]
    assert ml_code(70000) == 52
    return dict(seqs=seqs, lits=skewed(28 + 50, rng), want={"type": 2})


def ll_codes_0_34(s, first, rng):
    seqs = [(LL_BASE[c], int(rng.integers(1, 5000)), int(rng.integers(4, 20))) for c in range(35)]
    rng.shuffle(seqs)
    assert sorted({ll_code(q[0]) for q in seqs}) == list(range(35))
    return dict(seqs=seqs, lits=skewed(sum(q[0] for q in seqs) + 3, rng), want={"type": 2})


def ml_codes_1_51(s, first, rng):
    seqs = [(int(rng.integers(0, 3)), int(rng.integers(1, 5000)), ML_BASE[c]) for c in range(1, 52)]
    rng.shuffle(seqs)
    assert sorted({ml_code(q[2]) for q in seqs}) == list(range(1, 52))
    return dict(seqs=seqs, lits=skewed(sum(q[0] for q in seqs) + 3, rng), want={"type": 2})


def of_codes_19_23(s, first, rng):
    """offsets whose codes are 19 ... 23, the largest the 24-bit offBase field holds; 8 MiB of history"""
    seqs = [(3, (1 << k) + 5, 10) for k in range(19, 24)] + [(2, int(rng.integers(1, 900)), 6) for _ in range(20)]
    rng.shuffle(seqs)
    return dict(seqs=seqs, lits=skewed(100, rng), want={"type": 2})


def ncount_zero_run(gap_to):
    """ML codes 1, 2 and gap_to, gap_to + 1 only: a run of gap_to - 3 zero probabilities in the ML table description"""
    def b(s, first, rng):
        codes = [1] * 150 + [2] * 100 + [gap_to] * 30 + [gap_to + 1] * 20
        rng.shuffle(codes)
        seqs = [(0, int(rng.integers(1, 1000)), ML_BASE[c]) for c in codes]
        return dict(seqs=seqs, lits=skewed(50, rng), want={"type": 2, "modes": (1, 2, 2)})
    return b


def seq_rle(n):
    """n identical sequences: predefined tables for 1 and 2 (mostFrequent == nbSeq <= 2), RLE for 3"""
    def b(s, first, rng):
        m = 0 if n <= 2 else 1
        return dict(seqs=[(2, 1, 40)] * n, lits=skewed(2 * n + 10, rng, 8), want={"type": 2, "modes": (m, m, m)})
    return b


def dyn_min(delta):
    """nbSeq one below (delta -1) or at (0) dynamicFse_nbSeq_min of the LL and ML streams: (64 * (10 - strategy)) >> 3"""
    def b(s, first, rng):
        n = ((64 * (10 - s)) >> 3) + delta
        llc = [0] * (n // 2) + [int(c) for c in rng.integers(1, 11, n - n // 2)]
        mlc = [1] * (n // 2) + [int(c) for c in rng.integers(2, 20, n - n // 2)]
        seqs = [(LL_BASE[a], 1 + i % 7, ML_BASE[m]) for i, (a, m) in enumerate(zip(llc, mlc))]
        mode = 2 if delta >= 0 else 0
        return dict(seqs=seqs, lits=skewed(sum(q[0] for q in seqs) + 5, rng), want={"type": 2},
                    check=lambda m: m[0] == mode and m[2] == mode)
    return b


def most_frequent(m):
    """640 sequences whose most frequent ML code occurs m times: below nbSeq >> 5 = 20 the predefined table is kept"""
    def b(s, first, rng):
        codes = [1] * m
        others = list(range(2, 43))
        k = 0
        while len(codes) < 640:
            codes.append(others[k % len(others)])
            k += 1
        assert max(codes.count(c) for c in set(codes)) == m
        rng.shuffle(codes)
        seqs = [(int(rng.integers(0, 2)), int(rng.integers(1, 64)), ML_BASE[c]) for c in codes]
        return dict(seqs=seqs, lits=skewed(sum(q[0] for q in seqs) + 5, rng), check=lambda md: md[2] == (2 if m >= 20 else 0),
                    want={"type": 2})
    return b


def lits_n(n, want, nsym=4, disabled=0, rle=False):
    def b(s, first, rng):
        lits = bytes([7]) * n if rle else skewed(n, rng, nsym)
        return dict(seqs=_lit_only(n, rng), lits=lits, want=dict(want, type=2), lit_disabled=disabled)
    return b


def _window(a, rng):
    """4096 bytes whose most frequent byte (0xEE) occurs exactly a times (the others at most 16)"""
    rest = 4096 - a
    counts = {0xEE: a}
    for k in range(255):
        sym = k if k < 0xEE else k + 1
        counts[sym] = rest // 255 + (1 if k < rest % 255 else 0)
    return from_counts(counts, rng)


def suspect(n, a, b_):
    """a literal run of n >= 40960 behind one sequence (n / nbSeq >= 20): the reference samples its first and last 4096
    bytes and stores it raw when their largest counts add up to at most 68"""
    def b(s, first, rng):
        lits = _window(a, rng) + skewed(n - 8192, rng, 8) + _window(b_, rng)
        raw = n >= 40960 and a + b_ <= 68
        return dict(seqs=_lit_only(n, rng), lits=lits, want={"type": 2, "lit_type": 0 if raw else 2})
    return b


def largest(l):
    """8192 literals whose most frequent byte occurs l times: at most (8192 >> 7) + 4 = 68 they are stored raw"""
    def b(s, first, rng):
        k, r = divmod(8192, l)
        counts = {i: l for i in range(k)}
        if r:
            counts[k] = r
        return dict(seqs=_lit_only(8192, rng), lits=from_counts(counts, rng), want={"type": 2, "lit_type": 0 if l <= 68 else 2})
    return b


def huf_depth(nsym):
    """counts 1, 2, 4, ... 2^(nsym-1): a chain whose minimum-redundancy depth is nsym - 1"""
    def b(s, first, rng):
        counts = {i: 1 << i for i in range(nsym)}
        n = sum(counts.values())
        depth, target = huffman_depth(list(counts.values())), opt_table_log(11, n, nsym - 1, 1)
        assert depth == nsym - 1 and depth > target, (depth, target)
        seqs = [] if n > BLOCK_MAX - 100 else _lit_only(n, rng)
        return dict(seqs=seqs, lits=from_counts(counts, rng), want={"type": 2, "lit_type": 2})
    return b


def huf_desc(kind):
    def b(s, first, rng):
        if kind == "distinct":       # weights 1 ... 7 of symbols 0 ... 6, the last symbol implied: maxCount == 1
            counts = {i: 2 << i for i in range(7)}
            counts[7] = 1
            want = "direct"
        elif kind == "same":         # 64 symbols of 6 bits: every weight the same, maxCount == wtSize
            counts = {i: 64 for i in range(64)}
            want = "direct"
        else:
            counts = {i: int(4000 / (i + 1) ** 1.2) + 1 for i in range(40)}
            want = "fse"
        n = sum(counts.values())
        return dict(seqs=_lit_only(n, rng), lits=from_counts(counts, rng), want={"type": 2, "lit_type": 2, "huf_desc": want})
    return b


def huf_refused(s, first, rng):
    """193 symbols: 192 of one count (8-bit codes), one of 64 times that (2 bits).  The weights of symbols 0 ... 191 are
    all equal, so the FSE form does not apply, and the 4-bit form holds at most 128: no tree description, raw literals"""
    counts = {i: 20 for i in range(192)}
    counts[192] = 64 * 20
    cnt = np.zeros(256, np.uint32)
    cnt[:193] = list(counts.values())
    nb = product_lengths(cnt, 192, opt_table_log(11, int(cnt.sum()), 192, 1))
    assert len(set(nb[:192])) == 1 and nb[192] == 2
    return dict(seqs=_lit_only(5120, rng), lits=from_counts(counts, rng), want={"type": 2, "lit_type": 0})


def min_gain(m):
    """m copies of one byte and 69 single others: the Huffman section is exactly n - ((n >> 6) + 2) bytes for m = 40
    (kept raw) and one byte under that for m = 41"""
    def b(s, first, rng):
        lits = bytes([200]) * m + bytes(range(69))
        return dict(seqs=_lit_only(len(lits), rng), lits=lits, want={"type": 2, "lit_type": 0 if m == 40 else 2})
    return b


def tiny_stream(n):
    """n sequences whose only FSE-compressed stream is the offsets' (dfast: 32 sequences are enough), 31 of them
    repeat offset 1 and the last repeat offset 2: for n = 32 its description and bit-stream take 3 bytes together, under
    the 4 the reference requires, so the block goes raw (zstd_compress.c:2987-2993); one sequence more is enough"""
    def b(s, first, rng):
        seqs = [(1, 1, 4)] * (n - 1) + [(1, 4, 4)]
        if s == 1:          # the fast strategy keeps the predefined offset table below 36 sequences
            return dict(seqs=seqs, lits=bytes([5]) * n + b"xyzxyzxyz", want={"type": 2, "modes": (1, 0, 1)})
        return dict(seqs=seqs, lits=bytes([5]) * n + b"xyzxyzxyz", want={"type": 0} if n == 32 else {"type": 2, "modes": (1, 2, 1)})
    return b


def residue(k):
    """1000 + k literals: the four streams start at every residue mod 16 over k = 0 ... 15"""
    def b(s, first, rng):
        return dict(seqs=[(3, 20, 8), (2, 9, 5)], lits=skewed(1000 + k, rng, 12), want={"type": 2, "lit_type": 2, "streams": 4})
    return b


def rle_block(s, first, rng):
    """2001 equal bytes: an RLE block, except as a frame's first block"""
    return dict(seqs=[(1, 1, 2000)], lits=b"a", want={"type": seqgen.BT_COMPRESSED if first else seqgen.BT_RLE})


def incompressible(s, first, rng):
    return dict(seqs=[(10, 100, 6), (20, 3000, 9)], lits=zref.random_bytes(6000, 9), want={"type": 0})


BUILDERS = {
    "nbseq-7eff": nbseq(0x7EFF), "nbseq-7f00": nbseq(0x7F00), "nbseq-7fff": nbseq(0x7FFF),
    "ll-code-35": ll_code_35, "ml-code-52": ml_code_52, "ll-codes-0-34": ll_codes_0_34, "ml-codes-1-51": ml_codes_1_51,
    "of-codes-19-23": of_codes_19_23,
    "ncount-zeros-25": ncount_zero_run(28), "ncount-zeros-28": ncount_zero_run(31),
    "seq-rle-1": seq_rle(1), "seq-rle-2": seq_rle(2), "seq-rle-3": seq_rle(3),
    "dyn-min-below": dyn_min(-1), "dyn-min-at": dyn_min(0),
    "most-frequent-19": most_frequent(19), "most-frequent-20": most_frequent(20),
    "lits-63": lits_n(63, {"lit_type": 0}), "lits-64": lits_n(64, {"lit_type": 2, "streams": 1}),
    "lits-255": lits_n(255, {"lit_type": 2, "streams": 1}), "lits-256": lits_n(256, {"lit_type": 2, "streams": 4}),
    "lits-1023": lits_n(1023, {"lit_type": 2, "lit_header": 3}), "lits-1024": lits_n(1024, {"lit_type": 2, "lit_header": 4}),
    "lits-16383": lits_n(16383, {"lit_type": 2, "lit_header": 4}), "lits-16384": lits_n(16384, {"lit_type": 2, "lit_header": 5}),
    "rle-lits-64": lits_n(64, {"lit_type": 1, "lit_header": 2}, rle=True),
    "rle-lits-4095": lits_n(4095, {"lit_type": 1, "lit_header": 2}, rle=True),
    "rle-lits-4096": lits_n(4096, {"lit_type": 1, "lit_header": 3}, rle=True),
    "suspect-68": suspect(40960, 34, 34), "suspect-69": suspect(40960, 34, 35), "suspect-40959": suspect(40959, 34, 34),
    "largest-68": largest(68), "largest-69": largest(69),
    "huf-depth-12": huf_depth(13), "huf-depth-16": huf_depth(17),
    "huf-desc-distinct": huf_desc("distinct"), "huf-desc-same": huf_desc("same"), "huf-desc-fse": huf_desc("fse"),
    "huf-desc-refused": huf_refused, "min-gain-at": min_gain(40), "min-gain-past": min_gain(41),
    "tiny-stream-32": tiny_stream(32), "tiny-stream-33": tiny_stream(33),
    "rle-block": rle_block, "incompressible": incompressible,
}
BUILDERS.update({f"residue-{k}": residue(k) for k in range(16)})
# literal compression disabled (fast strategy with a target length): raw literal headers of 1, 2 and 3 bytes
FAST_ONLY = {f"raw-lits-{n}": lits_n(n, {"lit_type": 0, "lit_header": h}, disabled=1) for n, h in ((31, 1), (32, 2), (4095, 2), (4096, 3))}


def _make(name, builder, s, first, seed):
    rng = np.random.default_rng(seed)
    kw = builder(s, first, rng)
    return Store(f"{name}/s{s}/{'first' if first else 'later'}", strategy=s, first=first, seed=seed,
                 check_modes=kw.pop("check", None), **kw)


def random_stores(n=48):
    """the randomised seqStores of test_oracle_entropy.make_seqstore, match lengths lifted to >= 4, offsets taken as
    real ones"""
    from test_oracle_entropy import make_seqstore
    rng = np.random.default_rng(2024)
    out = []
    while len(out) < n:
        case = make_seqstore(rng)
        if case is None:
            continue
        offb, ll, ml, lits, block, strategy, tl = case
        ml = np.maximum(ml, 4)
        if len(lits) + int(ml.sum()) > BLOCK_MAX or len(lits) + int(ml.sum()) < 7:
            continue
        seqs = [(int(a), int(o), int(m)) for a, o, m in zip(ll, offb, ml)]
        k = len(out)
        out.append(Store(f"random-{k}/s{strategy}", seqs, lits.tobytes(), strategy=strategy, first=k % 2 == 0,
                         lit_disabled=1 if (strategy == 1 and tl > 0) else 0, seed=5000 + k))
    return out


def dict_stores():
    """small records behind each zstd-format dictionary of the dictionary tests: treeless literals (preferRepeat up to
    1024 literals), a table that lacks a symbol of the block, and set_repeat tables up to 999 sequences; as a frame's
    first block (the dictionary's tables apply) and as a later one"""
    out = []
    for di, name in enumerate(DICTS):
        content = seqgen.dict_content(zref.golden_input(name))
        bits = dict_huf_bits(name)
        absent = [b for b in range(256) if not bits[b]]
        for j, (nlit, nseq, extra) in enumerate(((300, 20, None), (1024, 30, None), (1025, 30, None), (3000, 40, None),
                                                 (1024, 25, "absent"), (400, 999, None), (400, 1000, None))):
            rng = np.random.default_rng(700 + 10 * di + j)
            lits = np.frombuffer(dict_mix(name, 700 + 10 * di + j, 0.0, nlit), np.uint8).copy()
            if extra == "absent":
                if not absent:
                    continue
                lits[5] = absent[0]
            lls = [0] * nseq
            for i in range(min(nseq, nlit)):
                lls[i % nseq] += 1
            seqs = [(lls[i], int(rng.integers(1, len(content))), int(rng.integers(4, 40))) for i in range(nseq)]
            if sum(q[0] for q in seqs) > nlit:
                continue
            rep = dict_fse_repeat(name)
            for first in (True, False):
                want = {"type": 2}
                if first and nlit <= 1024:      # preferRepeat: the dictionary's table unless it lacks a literal of the block
                    want["lit_type"] = 2 if extra == "absent" else 3
                # set_repeat for a table valid for every symbol, below 1000 sequences (zstd_compress_sequences.c:187-191)
                check = (lambda m, first=first, nseq=nseq, rep=rep: all((m[k] == 3) == (first and rep[k] == 2 and nseq < 1000)
                                                                        for k in range(3))) if nseq >= 999 else None
                out.append(Store(f"{name}-{nlit}l-{nseq}s{'-' + extra if extra else ''}/{'first' if first else 'later'}", seqs,
                                 lits.tobytes(), strategy=1 + j % 2, first=first, dict_name=name, want=want, seed=900 + j,
                                 check_modes=check))
    return out


def product_lengths(cnt, maxsym, target):
    """Huffman code lengths of the product's builder (oracle/zb_tables.c) for counts cnt[256]"""
    O = zref.oracle()
    O.zbo_huf_lengths_mk.restype = _sz
    O.zbo_huf_lengths_mk.argtypes = [_vp, _vp, ctypes.c_uint, ctypes.c_uint]
    nb = np.zeros(256, np.uint8)
    O.zbo_huf_lengths_mk(nb.ctypes.data, np.ascontiguousarray(cnt, np.uint32).ctypes.data, maxsym, target)
    return nb


def old_table_margin(name, lits):
    """bytes by which the dictionary's Huffman table costs more than a fresh one with its description (K2 keeps the
    old table when this is <= 0, huf_compress.c:1415-1422), with the product's code lengths; None if a fresh table
    would not be used at all"""
    O = zref.oracle()
    O.zbo_compressLiterals.restype = _sz
    O.zbo_compressLiterals.argtypes = [_vp, _sz, _vp, _sz, ctypes.c_uint, ctypes.c_int, ctypes.c_int]
    bits = np.array(dict_huf_bits(name), np.int64)
    cnt = np.bincount(np.frombuffer(lits, np.uint8), minlength=256).astype(np.uint32)
    maxsym, n = int(np.nonzero(cnt)[0].max()), len(lits)
    d = ctypes.create_string_buffer(1 << 18)
    with zref.entropy_model(1):
        r = O.zbo_compressLiterals(d, 1 << 18, lits, n, 1, 0, 0)
    body = d.raw[:r]
    if (body[0] & 3) != 2:
        return None
    h = body[(3, 3, 4, 5)[(body[0] >> 2) & 3]]
    h_size = h + 1 if h < 128 else (h - 127 + 1) // 2 + 1
    nb = product_lengths(cnt, maxsym, opt_table_log(11, n, maxsym, 1))
    return (int((bits * cnt).sum()) >> 3) - (h_size + (int((nb.astype(np.int64) * cnt).sum()) >> 3))


def dict_mix(name, seed, a, n):
    """n literals drawn from a mix of the dictionary's own distribution (weight 1 - a) and a random one over its
    symbols (weight a)"""
    bits = np.array(dict_huf_bits(name), float)
    pd = np.where(bits > 0, 2.0 ** -bits, 0)
    pd /= pd.sum()
    rng = np.random.default_rng(seed)
    rng.integers(1100, 3000)
    po = np.where(bits > 0, rng.random(256) ** 3, 0)
    po /= po.sum()
    u = rng.random(n)
    lits = np.minimum(np.searchsorted(np.cumsum((1 - a) * pd + a * po), u), 255)
    return np.where(bits[lits] > 0, lits, np.argmax(pd)).astype(np.uint8).tobytes()


# (dictionary, seed, mix, literals) -> the old table's margin: one byte cheaper, equal, one byte dearer
OLD_TABLE = [("zdict-16k-synthetic-seed77", 0, 0.2125, 2716, -1), ("zdict-16k-synthetic-seed77", 0, 0.21, 2716, 0),
             ("zdict-16k-synthetic-seed77", 0, 0.21125, 2716, 1), ("http-dict-missing-symbols", 1, 0.19375, 1999, -1),
             ("http-dict-missing-symbols", 1, 0.2425, 1999, 0), ("http-dict-missing-symbols", 0, 0.1975, 2716, 1)]


def dict_boundaries():
    """a first block behind a zstd-format dictionary at the literal decisions its tables drive: the old table one byte
    cheaper, as cheap as, and one byte dearer than a fresh one; and, behind a dictionary whose table is valid for every
    symbol, 5 literals (below the 6 a valid table needs), 9 (the fewest its 5-bit codes make worth a treeless section)
    and 200 (treeless, one stream)"""
    out = []
    for k, (name, seed, a, n, margin) in enumerate(OLD_TABLE):
        lits = dict_mix(name, seed, a, n)
        assert old_table_margin(name, lits) == margin
        for first in (True, False):          # a later block: the fresh table the first one was weighed against
            out.append(Store(f"old-table-{margin:+d}-{name}/{'first' if first else 'later'}", [(n - 2, 40, 6), (2, 90, 5)], lits,
                             strategy=1 + k % 2, first=first, dict_name=name,
                             want={"type": 2, "lit_type": 3 if first and margin <= 0 else 2}, seed=3000 + k))
    name = DICTS[0]
    assert dict_entropy(name).raw[784] == 2                     # hufRepeat valid: every byte has a code
    for n, lt in ((5, 0), (9, 3), (200, 3)):
        rng = np.random.default_rng(n)
        lits = bytes(97 + k % 24 for k in range(n)) if n < 10 else dict_mix(name, 3, 0.0, n)    # 'a' ... 'x': 5-bit codes
        st = Store(f"treeless-{n}-{name}", [(n, int(rng.integers(1, 3000)), 300)], lits, dict_name=name,
                   want={"type": 2, "lit_type": lt} | ({"streams": 1} if lt == 3 else {}), seed=3100 + n)
        out.append(st)
    return out


@functools.lru_cache(maxsize=None)
def stores():
    out = []
    for k, (name, b) in enumerate(sorted(BUILDERS.items())):
        for s in (1, 2):
            for first in (True, False):
                out.append(_make(name, b, s, first, 100 * k + 10 * s + first))
    for k, (name, b) in enumerate(sorted(FAST_ONLY.items())):
        for first in (True, False):
            out.append(_make(name, b, 1, first, 9000 + 10 * k + first))
    return tuple(out + random_stores() + dict_stores() + dict_boundaries())
