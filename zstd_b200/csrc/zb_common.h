/* zb_common.h — shared host/device definitions of the block-parallel plan.
 *
 * Unit of work = one zstd block (<= 128 KiB, ZSTD_BLOCKSIZE_MAX, lib/zstd.h:142).
 * Every block is compressed independently of its neighbours: private hash table primed from the
 * history bytes that precede it, encoder repcodes start invalid, fresh entropy tables.  The
 * per-block state the reference carries across blocks (ZSTD_blockState_t,
 * lib/compress/zstd_compress_internal.h:263-267) therefore does not exist here.
 */
#ifndef ZB_COMMON_H
#define ZB_COMMON_H
#include <stdint.h>
#include <stddef.h>

typedef uint8_t  u8;
typedef uint16_t u16;
typedef uint32_t u32;
typedef uint64_t u64;

#define ZB_BLOCK_MAX     (128u << 10)
#define ZB_PRIME_BYTES   (128u << 10)        /* history primed into a chunk's table (ZSTDMT overlap idea, zstdmt_compress.c:1182-1227) */
#define ZB_CHUNK_BLOCKS  4u                  /* blocks per chunk: one hash table lives through a chunk */
#define ZB_BATCH         1024u               /* positions of one walk batch = threads of the walk CTA */
#define ZB_TAG_BITS      11u                 /* table entry = (position + 1) << 11 | tag, positions relative to the chunk's history start */
#define ZB_FAST_HASHLOG_MAX   14u
#ifndef ZB_DFAST_SHORT_MAX
#define ZB_DFAST_SHORT_MAX    28672u         /* buckets: 112 KiB of shared memory, two walk CTAs per SM */
#endif
#ifndef ZB_DFAST_LONGLOG_MAX
#define ZB_DFAST_LONGLOG_MAX  14u            /* 64 KiB */
#endif
#define ZB_FAR           0xFFFFu             /* dist16 value: the distance is in the far array */

/* block types, lib/common/zstd_internal.h:90 */
#define ZB_BT_RAW 0
#define ZB_BT_RLE 1
#define ZB_BT_COMPRESSED 2

#define ZB_FLAG_FIRST 1u       /* first block of its frame */
#define ZB_FLAG_LAST  2u       /* last block of its frame  */
#define ZB_FLAG_DICT  4u       /* the oldest dictLen bytes of its history are the tail of its frame's dictionary content */

/* error codes = lib/zstd_errors.h:64-101 */
#define ZB_ERR(code) ((size_t)-(long)(code))
#define ZB_error_GENERIC 1
#define ZB_error_prefix_unknown 10
#define ZB_error_dictionary_corrupted 30
#define ZB_error_dictionary_wrong 32
#define ZB_error_parameter_unsupported 40
#define ZB_error_parameter_outOfBound 42
#define ZB_error_tableLog_tooLarge 44
#define ZB_error_maxSymbolValue_tooLarge 46
#define ZB_error_stage_wrong 60
#define ZB_error_memory_allocation 64
#define ZB_error_workSpace_tooSmall 66
#define ZB_error_dstSize_tooSmall 70
#define ZB_error_srcSize_wrong 72
#define ZB_error_dstBuffer_null 74
#define ZB_error_externalSequences_invalid 107
#define ZB_error_maxCode 120

typedef struct {
    u64 srcOff;        /* block start, byte offset into the input buffer */
    u32 size;          /* block size */
    u32 histLen;       /* bytes of history a match of this block may reach back into (chunk history and window) */
    u32 frame;         /* index into ZbFrame[] */
    u32 flags;         /* ZB_FLAG_* */
    u32 dictLen;       /* the oldest dictLen bytes of that history are the tail of its frame's dictionary content (ZB_FLAG_DICT) */
    u32 dictSlot;      /* its frame's entry in the call's dictionary table (ZbDictSlot) */
} ZbBlock;

/* one chunk = up to ZB_CHUNK_BLOCKS consecutive blocks of a frame: the unit of the candidate walk */
typedef struct {
    u64 srcOff;        /* chunk start, byte offset into the input buffer */
    u32 size;          /* bytes in the chunk */
    u32 histLen;       /* bytes walked in front of the chunk to prime the table (<= ZB_PRIME_BYTES) */
    u32 dictLen;       /* the oldest dictLen of them are the dictionary content's tail (first chunk of a frame only) */
    u32 firstBlock;    /* index of the chunk's first block in the call's block array */
    u32 blockLog;      /* log2 of the frame's block size: block k of the chunk starts at k << blockLog */
    u32 dictSlot;      /* its frame's entry in the call's dictionary table */
} ZbChunk;

typedef struct {
    u64 srcOff;        /* frame input start */
    u64 srcSize;
    u32 firstBlock;    /* index of its first ZbBlock */
    u32 nbBlocks;
    u32 windowLog;
    u32 dictID;
    u32 checksum;      /* 1: Content_Checksum_flag set, 4 bytes are reserved behind the last block (filled in by the host) */
    u32 dictSlot;      /* its entry in the call's dictionary table */
} ZbFrame;

typedef struct {       /* produced on the device, one per block */
    u32 nbSeq;
    u32 litSize;       /* all literals of the block incl. the trailing run */
    u32 litSecSize;    /* bytes of the literals section written at body[0..) */
    u32 bodySize;      /* final payload size (compressed body, 1 for RLE, block size for raw) */
    u32 type;          /* ZB_BT_* */
    u32 forceRaw;      /* block too small to try (zstd_compress.c:3216) or entropy stage gave up */
    u32 rleByte;
    u32 pad;
} ZbBlockMeta;

/* FSE compression table in our own layout (the reference's is common/fse.h:249) */
typedef struct {
    u32 tableLog;
    u32 maxSymbolValue;
    u16 nextState[512];
    int deltaFindState[64];
    u32 deltaNbBits[64];
} ZbdFseCTable;

/* entropy state a zstd-format dictionary installs as the "previous block" of a frame's first block
 * (ZSTD_loadCEntropy, lib/compress/zstd_compress.c:4987-5076); built on the host (zb_dict.cu) */
typedef struct {
    u32 present;
    u32 hufRepeat;             /* HUF_repeat: 0 none, 1 check, 2 valid */
    u32 hufMaxSymbol;
    u32 fseRepeat[3];          /* FSE_repeat per stream: 0 = LL, 1 = OF, 2 = ML */
    u32 rep[3];
    u32 dictID;
    u32 hufEnc[256];           /* code | nbBits << 16 */
    ZbdFseCTable fse[3];
} ZbDictEntropy;

typedef struct {
    u32 strategy;      /* 1 = fast, 2 = dfast */
    u32 mls;           /* bytes hashed by the (short) table: 4..8 */
    u32 tableN;        /* buckets of the (short) table; bucket = (hash32 * tableN) >> 32 */
    u32 tableNLong;    /* dfast: buckets of the 8-byte-hash table */
    u32 stepSize;      /* zstd_fast.c:200 */
    u32 litDisabled;   /* zstd_compress_internal.h:621-633 */
    u32 windowLog;
    u32 insStep;       /* positions without a candidate enter the table when ((pos - low) % step) < 2, step = insStep + walked / 128 */
} ZbParams;

/* One entry of a call's dictionary table: what the kernels read of a frame's dictionary, through the dictSlot of the frame's
 * blocks and chunks, at its first chunk (walk) and first block (parse, merge, entropy stages) only.  An entry serves one
 * dictionary under one set of ZbParams (the image is that parameter group's).  A launch without a table (NULL) has no
 * dictionary in any frame: first blocks start from the format's repcodes and entropy state. */
typedef struct {
    const u8* end;               /* one past the content tail in device memory (ZB_FLAG_DICT blocks read below it) */
    const ZbDictEntropy* de;     /* a zstd-format dictionary's entropy state, else NULL */
    const u32* image;            /* the tables walked over the tail under the group's ZbParams (tableN u32, then tableNLong u32 for
                                  * doubleFast), or NULL: the walk primes them from the tail */
    u32 startRep[2];             /* repcodes the search of a frame's first segment starts with (zstd-format dictionary), 0 = none */
    u32 codeRep[3];              /* repcode history the decoder holds at a frame's first block: {1,4,8} or the dictionary's */
    u32 pad;
} ZbDictSlot;

/* Per-block strides of the workspace arrays of one call, derived from its largest block (M = that size rounded up to 64):
 * a call of 128 KiB blocks has 128 Ki dist, 32776 seq, 128 KiB + 256 lit and 128 KiB + 1 KiB body per block. */
/* fast strategy: a block is parsed in segments of ZB_PARSE_SEG bytes, one warp each (a segment behaves like a block
 * for the parse; candidates, literals and sequences stay the block's).  Per segment, for the merge kernel: */
#define ZB_PARSE_SEG   (16u << 10)
#define ZB_PARSE_SEGS  (ZB_BLOCK_MAX / ZB_PARSE_SEG)
typedef struct {
    u32 nbSeq;         /* raw sequences of the segment, stored from seq slot k * ZB_PARSE_SEG / 4 */
    u32 pad[3];
} ZbSegMeta;

typedef struct {
    u32 dist;          /* u16 per block : candidate distances (+ as many u32 of "far" distances); K3 reuses the u16 area for 3 x state records */
    u32 seq;           /* u64 per block : packed sequences */
    u32 lit;           /* bytes per block : literal bytes (multiple of 16) */
    u32 body;          /* bytes per block : compressed block body staging (multiple of 16) */
    u32 state;         /* u16 per FSE stream per block inside the dist area (3 * state <= dist) */
} ZbStrides;

#ifdef __CUDACC__
#define ZB_HD __host__ __device__
#else
#define ZB_HD
#endif
static inline ZB_HD ZbStrides zb_strides(u32 maxBlock)
{
    u32 const M = ((maxBlock < 64u ? 64u : maxBlock) + 63u) & ~63u;
    ZbStrides sd; sd.dist = M; sd.seq = M / 4u + 8u; sd.lit = M + 256u; sd.body = M + 1024u; sd.state = M / 4u;
    return sd;
}
/* Sequence calls (ZSTD_compressSequences): matches of 3 bytes allow M / 3 sequences per block, so the seq slots hold
 * M / 3 + 8 and the FSE state records (3 x state u16 inside the dist area) ceil(M / 3), rounded up to 16 bytes. */
static inline ZB_HD ZbStrides zb_seq_strides(u32 maxBlock)
{
    ZbStrides sd = zb_strides(maxBlock);
    u32 const M = sd.dist;
    sd.seq = M / 3u + 8u; sd.state = ((M + 2u) / 3u + 7u) & ~7u; sd.dist = 3u * sd.state;
    return sd;
}
/* parse segments per block row: ZbSegMeta records per block in the segmeta array (1 for calls of blocks <= 16 KiB) */
static inline ZB_HD u32 zb_segsPerRow(const ZbStrides& sd) { return (sd.dist + ZB_PARSE_SEG - 1u) / ZB_PARSE_SEG; }
#define ZB_SEQ_OFF_MAX ((1u << 24) - 4u)   /* largest offset of a sequence call (the packed sequence holds 28 bits of offBase; sequence calls keep this bound) */
/* a final sequence as the sequences kernel reads it: offBase (28 bits: long-distance offsets reach 2^27), literal length
 * (18 bits), match length (18 bits, >= 3); both lengths are <= ZB_BLOCK_MAX */
static inline ZB_HD u64 zb_pack_seq(u32 offBase, u32 litLen, u32 matchLen)
{
    return (u64)offBase | ((u64)litLen << 28) | ((u64)matchLen << 46);
}
#define ZB_SEQ_OFFBASE(q) ((u32)(q) & 0xFFFFFFFu)
#define ZB_SEQ_LL(q)      ((u32)((q) >> 28) & 0x3FFFFu)
#define ZB_SEQ_ML(q)      ((u32)((q) >> 46) & 0x3FFFFu)
/* a raw sequence, as the parse kernels (K1b) leave it for the merge (K1c): real offset (24 bits), match length (18 bits),
 * match start relative to the block above them */
static inline ZB_HD u64 zb_pack_raw(u32 off, u32 mlen, u32 msRel) { return (u64)off | ((u64)mlen << 24) | ((u64)msRel << 42); }
#define ZB_RAW_OFF(r)  ((u32)(r) & 0xFFFFFFu)
#define ZB_RAW_MLEN(r) ((u32)((r) >> 24) & 0x3FFFFu)
#define ZB_RAW_MS(r)   ((u32)((r) >> 42))

/* Long-distance matching (zb_ldm.cu; the rule: oracle/zb_ldm.c).  Frames of more than one chunk only. */
#define ZB_LDM_WINDOW_LOG 27u                                  /* ZSTD_LDM_DEFAULT_WINDOW_LOG, zstd_ldm.h:25 */
#define ZB_LDM_MIN_FRAME  (ZB_CHUNK_BLOCKS * ZB_BLOCK_MAX)
#define ZB_LDM_GEAR_SEED  0x6C646D2D67656172ull                /* gear[i] = splitmix64 output i + 1 of this seed ("ldm-gear") */
typedef struct {
    u32 hashLog, minMatch, bucketSizeLog, hashRateLog;       /* resolved (ZSTD_ldm_adjustParameters) */
    u32 windowLog, pad;
    u64 stopMask;                                            /* zstd_ldm.c:32-60 */
} ZbLdmParams;
static inline ZB_HD u64 zb_ldm_survivor_cap(u64 n, u32 minMatch) { return n / minMatch + 1u; }   /* survivors are >= minMatch apart */
/* an LDM match: offset (28 bits), length (18 bits), start relative to its block (18 bits) */
static inline ZB_HD u64 zb_pack_ldm(u64 start, u64 len, u64 off) { return off | (len << 28) | (start << 46); }
#define ZB_LDM_OFF(m)   ((u32)(m) & 0xFFFFFFFu)
#define ZB_LDM_LEN(m)   ((u32)((m) >> 28) & 0x3FFFFu)
#define ZB_LDM_START(m) ((u32)((m) >> 46))
/* what K1c reads for the blocks of one launch: match[first[b] .. first[b] + cnt[b]) of block b */
typedef struct { const u64* match; const u64* first; const u32* cnt; } ZbLdmView;

#ifdef __CUDACC__
/* host helpers of the compression and decompression drivers (zb_api.cu, zb_decode.cu) */
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <type_traits>
#include <utility>
#include <vector>

static inline bool zb_isErr(size_t c) { return c > ZB_ERR(ZB_error_maxCode); }

/* a failed CUDA call returns an error code from the enclosing function; its sticky error is cleared, so that the caller's
 * next cudaGetLastError() does not report it again */
#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { \
    if (getenv("ZSTDB200_DEBUG")) fprintf(stderr, "zstd_b200: CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); \
    cudaGetLastError(); return ZB_ERR(e_ == cudaErrorMemoryAllocation ? ZB_error_memory_allocation : ZB_error_GENERIC); } } while (0)
/* a call that returns an error code passes it on */
#define TRY(x) do { size_t const e_ = (x); if (zb_isErr(e_)) return e_; } while (0)

/* Set on a thread while a call sizes its buffers without growing them and while a call is captured into a CUDA graph
 * (ZbOrder below): every owner below then refuses to grow with ZSTD_error_stage_wrong instead. */
inline thread_local bool zb_noAlloc = false;

/* An array of T in device memory (cudaMalloc) or page-locked host memory (cudaMallocHost) that a context owns: grown on
 * demand, freed with the context.  cap counts elements. */
template <typename T, bool Pinned> struct ZbBuf {
    T* p = nullptr; size_t cap = 0;
    ZbBuf() = default;
    ZbBuf(const ZbBuf&) = delete; ZbBuf& operator=(const ZbBuf&) = delete;
    ~ZbBuf() { release(); }
    void release() { if (p) { if (Pinned) cudaFreeHost(p); else cudaFree(p); } p = nullptr; cap = 0; }
    /* room for `need` elements; a larger need frees the array (its contents are not kept), then allocates need + headroom */
    size_t ensure(size_t need, size_t headroom = 0) {
        if (need <= cap) return 0;
        if (zb_noAlloc) return ZB_ERR(ZB_error_stage_wrong);
        release();
        size_t const bytes = (need + headroom) * sizeof(T);
        CK(Pinned ? cudaMallocHost((void**)&p, bytes) : cudaMalloc((void**)&p, bytes));
        cap = need + headroom;
        return 0;
    }
    operator T*() const { return p; }
};
template <typename T> using ZbDevBuf = ZbBuf<T, false>;
template <typename T> using ZbHostBuf = ZbBuf<T, true>;

/* The compression workspace: one row per block in flight, holding what the block carries from stage to stage.
 *   meta (K1 -> K4), seqs (K1 -> K3), lits (K1 -> K2), body (K2, K3 -> K4);
 *   dist / far: candidate distances (K1a -> K1b), u16 per position, and u32 per position for those that need it (ZB_FAR);
 *   dist2 / far2: the same for doubleFast's short-hash table;
 *   segmeta: zb_segsPerRow records (K1b -> K1c).
 * Array X's row r starts r * sd.X elements in (dist, far, dist2 and far2 use sd.dist; meta 1 and segmeta
 * zb_segsPerRow(sd)).  Once K1b is done the candidate rows are free and later stages reuse them:
 *   K3: a block's FSE state records, 3 x sd.state u16, in its dist row (a sequence call's dist area exists for them);
 *   K1c with long-distance matches: the block's surviving raw sequences (at most sd.seq u64) in its far row and one u32
 *   per survivor plus one in its dist row.
 * Which arrays a call has depends on its kind. */
enum ZbWorkKind { ZB_WORK_FAST, ZB_WORK_DFAST, ZB_WORK_SEQUENCES };   /* sequences: no far or segmeta; dist2 / far2: doubleFast only */
struct ZbWorkRows {
    ZbStrides sd;
    ZbBlockMeta* meta; u64* seqs; u8* lits; u8* body; u16* dist; u32* far; u16* dist2; u32* far2; ZbSegMeta* segmeta;
    /* the view moved down by `row` rows (an array the kind does not have stays NULL) */
    ZbWorkRows at(size_t row) const {
        ZbWorkRows r = *this;
        auto down = [row](auto*& p, size_t stride) { if (p) p += row * stride; };
        down(r.meta, 1); down(r.seqs, sd.seq); down(r.lits, sd.lit); down(r.body, sd.body);
        down(r.dist, sd.dist); down(r.far, sd.dist); down(r.dist2, sd.dist); down(r.far2, sd.dist); down(r.segmeta, zb_segsPerRow(sd));
        return r;
    }
};
/* Places the arrays of `rows` rows of `kind` at the strides `sd` one behind the other from `base`, *out = the view of row 0,
 * and returns the bytes they take (base NULL: only that size).  Every array has at least 256 bytes of padding behind it and
 * starts 2 MiB into the buffer or a multiple of that, where an allocation of its own would start: with the arrays merely
 * 256-byte aligned, K3 took 2 % longer (H100 80GB HBM3 at 700 W, level 3, 2 GiB in one wave).  Strides whose candidate
 * rows cannot hold the reuse above are an error. */
static inline size_t zb_workLayout(u8* base, size_t rows, ZbWorkKind kind, const ZbStrides& sd, ZbWorkRows* out)
{
    bool const match = kind != ZB_WORK_SEQUENCES;
    if (3ull * sd.state > sd.dist) return ZB_ERR(ZB_error_GENERIC);
    if (match && ((u64)sd.seq * 8u > (u64)sd.dist * 4u || ((u64)sd.seq + 1u) * 4u > (u64)sd.dist * 2u)) return ZB_ERR(ZB_error_GENERIC);
    ZbWorkRows w = {};
    w.sd = sd;
    size_t const align = (size_t)2 << 20;
    size_t bytes = 0;
    auto place = [&](auto*& p, size_t n) {
        if (base) p = reinterpret_cast<std::remove_reference_t<decltype(p)>>(base + bytes);
        bytes = (bytes + n * sizeof(*p) + 256u + align - 1u) & ~(align - 1u);
    };
    place(w.meta, rows); place(w.seqs, rows * sd.seq); place(w.lits, rows * sd.lit); place(w.body, rows * sd.body);
    place(w.dist, rows * sd.dist);
    if (match) { place(w.far, rows * sd.dist); place(w.segmeta, rows * zb_segsPerRow(sd)); }
    if (kind == ZB_WORK_DFAST) { place(w.dist2, rows * sd.dist); place(w.far2, rows * sd.dist); }
    if (base) *out = w;
    return bytes;
}

/* A non-blocking stream that a context owns, created by ensure() and destroyed with its owner.  Move-assignable, so that a
 * context can take over a stream that was created together with its events, all or nothing. */
struct ZbStream {
    cudaStream_t s = nullptr;
    ZbStream() = default;
    ZbStream& operator=(ZbStream&& o) { std::swap(s, o.s); return *this; }
    ~ZbStream() { if (s) cudaStreamDestroy(s); }
    size_t ensure() {
        if (s) return 0;
        if (zb_noAlloc) return ZB_ERR(ZB_error_stage_wrong);
        CK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
        return 0;
    }
    operator cudaStream_t() const { return s; }
};

/* Events that a context owns, all timed or all untimed.  ensure(n, timed) keeps them until a call needs more of them or the
 * other kind; they are destroyed with their owner. */
struct ZbEvents {
    std::vector<cudaEvent_t> ev; bool timed = false;
    ZbEvents() = default;
    ZbEvents& operator=(ZbEvents&& o) { ev.swap(o.ev); std::swap(timed, o.timed); return *this; }
    ~ZbEvents() { release(); }
    void release() { for (cudaEvent_t e : ev) cudaEventDestroy(e); ev.clear(); }
    size_t ensure(size_t n, bool timing) {
        if (n <= ev.size() && timing == timed) return 0;
        if (zb_noAlloc) return ZB_ERR(ZB_error_stage_wrong);
        release();
        timed = timing;
        while (ev.size() < n) {
            cudaEvent_t e;
            CK(cudaEventCreateWithFlags(&e, timing ? cudaEventDefault : cudaEventDisableTiming));
            ev.push_back(e);
        }
        return 0;
    }
    cudaEvent_t operator[](size_t i) const { return ev[i]; }
};

/* The order of a context's calls, one rule for the compressor and the decoder (DESIGN.md section 2, "Stream-ordered calls"):
 * the `order` event, sizing without growth first, and what a call being captured into a graph may not do. */
struct ZbOrder {
    ZbEvents ev;
    size_t create() { return ev.ensure(1, false); }
    cudaError_t hostWait() const { return cudaEventSynchronize(ev[0]); }   /* every call queued so far has completed */
    struct Call {                                  /* one call's side of the rule, for the call's duration */
        const ZbOrder& o; bool capturing = false; bool const prevNoAlloc = zb_noAlloc;
        explicit Call(const ZbOrder& order) : o(order) { zb_noAlloc = false; }
        ~Call() { zb_noAlloc = prevNoAlloc; }
        size_t begin(int device, cudaStream_t st) {   /* a stream-ordered call on st; device: the context's, -1 if none yet */
            if (device >= 0) CK(cudaSetDevice(device));
            cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
            CK(cudaStreamIsCapturing(st, &cs));
            zb_noAlloc = capturing = cs != cudaStreamCaptureStatusNone;
            return capturing && device < 0 ? ZB_ERR(ZB_error_stage_wrong) : 0;
        }
        template <typename F> size_t size(F&& sizing) {
            zb_noAlloc = true; size_t r = sizing(); zb_noAlloc = capturing;
            if (r == ZB_ERR(ZB_error_stage_wrong) && !capturing) { CK(o.hostWait()); r = sizing(); }
            return r;
        }
        size_t enter(cudaStream_t st) { if (!capturing) CK(cudaStreamWaitEvent(st, o.ev[0], 0)); return 0; }
        size_t leave(cudaStream_t st) { if (!capturing) CK(cudaEventRecord(o.ev[0], st)); return 0; }
    };
};

/* restores the calling thread's current device when a call returns (a context works on the device it was created for) */
struct ZbDeviceGuard {
    int prev;
    ZbDeviceGuard() : prev(-1) { if (cudaGetDevice(&prev) != cudaSuccess) { prev = -1; cudaGetLastError(); } }
    ~ZbDeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

/* deletes a context (once the calls still queued on it have completed) or a digested dictionary on its device, where its
 * members free what they own.  One that never reached a device (device < 0) is deleted without a device switch: it holds
 * nothing there, so its deletion makes no CUDA call (but for the arrays a CDict's failed first upload left) */
template <typename T> static inline size_t zb_deleteOnDevice(T* x, const ZbOrder* order = nullptr)
{
    if (!x) return 0;
    if (x->device < 0) { delete x; return 0; }
    ZbDeviceGuard guard;
    cudaSetDevice(x->device);
    if (order) order->hostWait();
    delete x;
    return 0;
}

/* the device a new context belongs to, chosen when it is created (zb_api.cu): ZSTDB200_setDevice's value, else the calling
 * thread's current device */
int zb_contextDevice(void);
#endif

#endif
