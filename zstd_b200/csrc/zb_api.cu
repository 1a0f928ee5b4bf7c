/* zb_api.cu — host driver + C ABI of libzstd_b200.so.
 *
 * Mirrors what the reference does around the per-block hot path:
 *   ZSTD_compress / ZSTD_compressCCtx / ZSTD_compress_usingDict  (lib/compress/zstd_compress.c:5398-5440)
 *   parameter derivation   ZSTD_getCParams_internal :7123-7146 + ZSTD_adjustCParams_internal :1465-1602 (compress/clevels.h:25-130)
 *   block planning         ZSTD_compress_frameChunk :4527-4623 (here: all blocks of a call at once)
 * and hands every block to the CUDA kernels (zb_match.cu, zb_literals.cu, zb_sequences.cu,
 * zb_stitch.cu).  No compression work is done on the host; without a CUDA device every compress
 * entry point fails with ZSTD_error_GENERIC.
 */
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <vector>
#include <memory>
#include <unordered_map>
#include <unordered_set>
#include <mutex>
#include <thread>
#include <new>
#include <time.h>
#include <algorithm>
#include "../../include/zstd_b200.h"
#include "zb_common.h"
#include "zb_kernels.h"

static inline u32 hb32(u32 v) { return 31u - (u32)__builtin_clz(v); }

/* ------------------------------------------------------------------ parameters */
typedef struct { u32 windowLog, chainLog, hashLog, searchLog, minMatch, targetLength, strategy; } ZbCParams;
struct Row { u8 W, C, H, S, L, TL, strat; };
/* compress/clevels.h:25-130, rows 0..4; strategies above dfast are out of scope: a level whose
 * reference strategy is greedy or stronger is served by the strongest dfast row of its size class */
static const Row kRows[4][5] = {
    { {19,12,13,1,6,1,1}, {19,13,14,1,7,0,1}, {20,15,16,1,6,0,1}, {21,16,17,1,5,0,2}, {21,18,18,1,5,0,2} },
    { {18,12,13,1,5,1,1}, {18,13,14,1,6,0,1}, {18,14,14,1,5,0,2}, {18,16,16,1,4,0,2}, {18,16,16,1,4,0,2} },
    { {17,12,12,1,5,1,1}, {17,12,13,1,6,0,1}, {17,13,15,1,5,0,1}, {17,15,16,2,5,0,2}, {17,17,17,2,4,0,2} },
    { {14,12,13,1,5,1,1}, {14,14,15,1,5,0,1}, {14,14,15,1,4,0,1}, {14,14,15,2,4,0,2}, {14,14,15,2,4,0,2} },
};

/* ldm: long-distance matching, whose window is ZSTD_LDM_DEFAULT_WINDOW_LOG before the size adjustment (ZSTD_getCParamsFromCCtxParams,
 * zstd_compress.c:1639) */
static ZbCParams zb_getCParams(int level, u64 srcSize, size_t dictSize, bool ldm = false)
{
    u64 const rSize = srcSize + dictSize;
    u32 const tableID = (rSize <= 256u * 1024) + (rSize <= 128u * 1024) + (rSize <= 16u * 1024);
    int const r = level == 0 ? 3 : (level < 0 ? 0 : (level > 4 ? 4 : level));
    Row const x = kRows[tableID][r];
    ZbCParams cp = { x.W, x.C, x.H, x.S, x.L, x.TL, x.strat };
    if (level < 0) {
        int const minLevel = -(int)ZB_BLOCK_MAX;                 /* ZSTD_minCLevel, zstd_compress.c:7038 */
        cp.targetLength = (u32)(-(level < minLevel ? minLevel : level));
    }
    if (ldm) cp.windowLog = ZB_LDM_WINDOW_LOG;
    {   u64 const maxWindowResize = 1ull << 30;                  /* zstd_compress.c:1537-1547 */
        if (srcSize <= maxWindowResize && dictSize <= maxWindowResize) {
            u32 const tSize = (u32)(srcSize + dictSize);
            u32 const srcLog = (tSize < (1u << 6)) ? 6 : hb32(tSize - 1) + 1;
            if (cp.windowLog > srcLog) cp.windowLog = srcLog;
        }
        u32 dawl = cp.windowLog;                                  /* ZSTD_dictAndWindowLog :1432-1459 */
        if (dictSize) {
            u64 const windowSize = 1ull << cp.windowLog;
            u64 const dictAndWindowSize = dictSize + windowSize;
            if (windowSize >= dictSize + srcSize) dawl = cp.windowLog;
            else if (dictAndWindowSize >= (1ull << 31)) dawl = 31;
            else dawl = hb32((u32)dictAndWindowSize - 1) + 1;
        }
        if (cp.hashLog > dawl + 1) cp.hashLog = dawl + 1;
        if (cp.chainLog > dawl) cp.chainLog -= (cp.chainLog - dawl);
        if (cp.windowLog < 10) cp.windowLog = 10;                 /* ZSTD_WINDOWLOG_ABSOLUTEMIN */
    }
    return cp;
}

static ZbParams zb_makeParams(const ZbCParams& cp)
{
    ZbParams p; memset(&p, 0, sizeof(p));
    p.strategy = cp.strategy;
    p.windowLog = cp.windowLog;
    p.mls = cp.minMatch < 4 ? 4 : (cp.minMatch > 8 ? 8 : cp.minMatch);
    /* Table sizes and the insertion pattern are set against the reference's compressed size on datagen P30 / P50 / P90
     * (tools/exp_size.py, DESIGN.md section 5): an occurrence stays in the table until a different string takes its
     * bucket (positions that find a candidate are not inserted), so a table somewhat smaller than the reference's holds
     * as many useful candidates.  The oracle's zbo_makePlan is the same rule (tests/test_plan.py). */
    if (cp.strategy == 1) {
        u32 const hl = cp.hashLog > ZB_FAST_HASHLOG_MAX ? ZB_FAST_HASHLOG_MAX : cp.hashLog;
        p.stepSize = cp.targetLength + !cp.targetLength + 1;     /* zstd_fast.c:200 */
        if (cp.targetLength == 0) { p.tableN = 3u << (hl - 2); p.insStep = 3; }
        else                      { p.tableN = 7u << (hl - 3); p.insStep = p.stepSize >= 5u ? p.stepSize - 1u : p.stepSize; }   /* never the parse's own probe spacing from 5 on: equal periods lock the probed positions out of phase with the inserted ones (level -7: +8.6 % instead of -6.6 % on datagen -P90) */
    } else {
        p.stepSize = 1;
        p.tableN = 1u << cp.chainLog;                            /* short table (zstd_double_fast.c:116) */
        if (p.tableN > ZB_DFAST_SHORT_MAX) p.tableN = ZB_DFAST_SHORT_MAX;
        p.tableNLong = 1u << (cp.hashLog > ZB_DFAST_LONGLOG_MAX ? ZB_DFAST_LONGLOG_MAX : cp.hashLog);
        p.insStep = 2;
    }
    p.litDisabled = (cp.strategy == 1) && (cp.targetLength > 0); /* zstd_compress_internal.h:621-633 */
    return p;
}

#define ZB_MAX_IMAGES 4

/* ------------------------------------------------------------------ context */
#include <atomic>
static std::atomic<int> g_device(-1);

#define ZB_WAVE_SLOTS_MAX 14u
#define ZB_WAVE_SLOTS_DEFAULT 4u
#define ZB_HOST_WAVE_SLOTS_DEFAULT 8u   /* with 384-block waves; on the H100 no setting of tests/e2e_sweep.py was faster in every run: the upload bounds the call (DESIGN.md section 10) */
#define ZB_HOST_WAVE_BLOCKS 384u     /* 48 MiB of input per wave */
/* A dictionary's tables walked under one parameter group's ZbParams (zb_prepareDicts): allocated when first built, at the
 * size of that group's tables; ready once the build has completed */
struct ZbDictImage { ZbParams prm; ZbDevBuf<u32> img; bool ready; };
/* Digested dictionary (lib/zstd.h:979, zstd_compress.c:5477-5642), the one form in which the compressor keeps a
 * dictionary on the device: the content tail, its entropy tables and the primed hash-table images, each allocated at the
 * size it holds when first needed.  A ZSTD_createCDict object keeps them across calls and any number of contexts may use
 * it; the bytes a call passes with ZSTD_compress_usingDict or ZSTDB200_compressFrames are digested into the context's own
 * object (ZSTD_CCtx_s::callDict) on every call. */
struct ZSTD_CDict_s {
    int level;
    std::unique_ptr<u8[]> copy;    /* ZSTD_createCDict's copy of the bytes (ZSTD_dlm_byCopy) */
    const u8* content;             /* the whole dictionary: that copy, or the caller's buffer */
    bool contentOnDevice;          /* a prefix given with ZSTDB200_CCtx_refPrefixDevice: content is a device pointer */
    size_t size;
    size_t contentOff, tail;       /* entropy header size, bytes of content that blocks can see */
    ZbDictEntropy entropy;         /* parsed on the host by zb_digestDict */
    std::mutex lock;               /* guards the device state below */
    int device;                    /* -1 until the device buffers exist */
    bool resident;                 /* tail and entropy tables uploaded since the digest */
    ZbDevBuf<u8> d_dict; ZbDevBuf<ZbDictEntropy> d_de;   /* the content tail with 32 bytes of zeros on both sides; the entropy state */
    u32 nbImages; ZbDictImage images[ZB_MAX_IMAGES];
};
struct ZbCDictFree { void operator()(ZSTD_CDict* cd) const { ZSTD_freeCDict(cd); } };

struct ZbGroup { ZbParams prm; u32 b0, b1, c0, c1; u32 prmIdx; bool ldm, dict; };   /* ldm: its frames have long-distance matches; dict: some block has ZB_FLAG_DICT; prmIdx: prm in ZbPlan::prms */
/* Descriptor arrays of a plan: page-locked (so that the upload of a million frames' descriptors is a DMA at PCIe speed, not a
 * staged copy of pageable memory) and kept across calls.  Without a CUDA device (the CPU tests' ZSTDB200_describePlan)
 * ordinary memory is used. */
template <typename T> struct ZbVec {
    T* p; size_t n, cap; bool pinned;
    bool pageable;                 /* never page-locked: growing it makes no CUDA call */
    ZbVec() : p(NULL), n(0), cap(0), pinned(false), pageable(false) {}
    ~ZbVec() { release(); }
    ZbVec(const ZbVec&) = delete; ZbVec& operator=(const ZbVec&) = delete;
    void release() { if (p) { if (pinned) cudaFreeHost(p); else free(p); } p = NULL; n = cap = 0; }
    void reserve(size_t want) {
        if (want <= cap) return;
        size_t const c = want < 2 * cap ? 2 * cap : want;
        T* q = NULL; bool pin = !pageable;
        if (pin && cudaMallocHost((void**)&q, c * sizeof(T)) != cudaSuccess) { cudaGetLastError(); pin = false; }
        if (!pin) q = (T*)malloc(c * sizeof(T));
        if (n) memcpy(q, p, n * sizeof(T));
        size_t const keep = n;
        release(); p = q; n = keep; cap = c; pinned = pin;
    }
    void push_back(const T& v) { if (n == cap) reserve(cap ? 2 * cap : 64); p[n++] = v; }
    void resize(size_t m) { reserve(m); if (m > n) memset((void*)(p + n), 0, (m - n) * sizeof(T)); n = m; }
    void clear() { n = 0; }
    size_t size() const { return n; }
    T* data() { return p; }
    const T* data() const { return p; }
    T& back() { return p[n - 1]; }
    T& operator[](size_t i) { return p[i]; }
    const T& operator[](size_t i) const { return p[i]; }
};
struct ZbLdmFrame { u32 frame; ZbLdmParams prm; u64 matchBase; u64 prefix; };   /* prefix: indexed prefix bytes in front of the frame */
/* A single-block frame's descriptors, kept by the planner for the frames that follow with the same size and dictionary */
struct ZbTemplate { const ZSTD_CDict* raw; u64 size; u64 gen; u32 prmIdx; ZbFrame fr; ZbBlock b; ZbChunk ch; };
#define ZB_TEMPLATE_CACHE 16384u   /* templates of a call with many dictionaries, by (CDict, frame size): open addressing */
/* The call's dictionary table: entry s of `dicts` serves dictionary slots[s].cd (NULL: frames without one) under the
 * parameters prms[slots[s].prm]; zb_plan fills the repcodes, zb_prepareDicts the device addresses. */
struct ZbSlotInfo { ZSTD_CDict* cd; u32 prm; };
struct ZbPlan { ZbVec<ZbBlock> blocks; ZbVec<ZbChunk> chunks; ZbVec<ZbFrame> frames; std::vector<ZbGroup> groups; ZbStrides sd; bool unsupported;
                std::vector<ZbLdmFrame> ldm; u64 ldmMatches;      /* frames with long-distance matching, their share of the match list */
                u64 frameBytes, frameBlocks; u32 frameMaxBlock;   /* the whole frames, other ranks' blocks included: what decides the waves */
                ZbVec<ZbDictSlot> dicts; std::vector<ZbSlotInfo> slots; std::vector<ZbParams> prms;
                std::vector<ZSTD_CDict*> cdicts;                  /* the distinct dictionaries, in order of first use */
                std::unordered_map<u64, u32> slotOf; std::unordered_set<const ZSTD_CDict*> seen;   /* slot by (CDict, prms index); cdicts as a set */
                std::vector<ZbChunk> imageChunks;                 /* the image builds of the call, by parameters (zb_prepareDicts) */
                std::vector<u32> imageBuilds;                     /* imageChunks[imageBuilds[i] .. imageBuilds[i + 1]): builds under prms[i] */
                std::vector<ZbTemplate> tpl; u64 gen = 0;         /* the template cache, valid entries have gen == this call's */
                void reset() { blocks.clear(); chunks.clear(); frames.clear(); groups.clear(); unsupported = false; ldm.clear(); ldmMatches = 0;
                               frameBytes = frameBlocks = 0; frameMaxBlock = 0; dicts.clear(); slots.clear(); prms.clear(); cdicts.clear(); slotOf.clear(); seen.clear();
                               imageChunks.clear(); imageBuilds.clear(); gen++; } };   /* keeps its memory: a context plans call after call */

enum { EV_START, EV_K0, EV_K1, EV_K2, EV_K3, EV_MID, EV_KEND, EV_END, EV_PHASES };   /* a compression context's phase events */

struct ZSTD_CCtx_s {
    int device;                    /* -1 until the first call created the stream and events on bindDevice */
    int bindDevice;                /* device captured by ZSTD_createCCtx */
    ZbStream stream;
    ZbDevBuf<ZbChunk> d_chunks;
    ZbDevBuf<u8> d_work;           /* per-block workspace: the rows of every slot (zb_workLayout) */
    u32 devWaveBlocks;             /* device-memory calls: blocks per wave (0 = always one wave) */
    ZbStream waveStream[ZB_WAVE_SLOTS_MAX + 1];       /* one per workspace slot, then the host path's download stream */
    u32 waveSlots;                 /* waves in flight, device-memory calls */
    u32 hostWaveSlots;             /* waves in flight, host-memory calls */
    u32 hostWaveBlocks;            /* host-memory calls: blocks per wave */
    ZbDevBuf<ZbBlock> d_blocks; ZbDevBuf<ZbFrame> d_frames;
    ZbDevBuf<ZbDictSlot> d_dicts; ZbDevBuf<ZbChunk> d_imageChunks;   /* the call's dictionary table, its image builds */
    ZbDevBuf<u64> d_outOffsets;
    ZbDevBuf<u64> d_totals;        /* d_totals[w]: bytes produced up to and including wave w */
    ZbHostBuf<u64> h_totals;       /* mirror of d_totals */
    /* a synchronous call's verdict kernel writes here, [0] the total or an error code, [1 + f] frame f's size: one copy reads
     * both back into the mirror */
    ZbDevBuf<unsigned long long> d_verdict; ZbHostBuf<unsigned long long> h_verdict;
    /* host-pointer path staging */
    ZbDevBuf<u8> d_in, d_out;
    std::unique_ptr<ZSTD_CDict, ZbCDictFree> callDict;   /* digest of the dictionary bytes the current call passes; reads the caller's buffer in place */
    ZbEvents ev;                   /* EV_START .. EV_END */
    ZbEvents evH2D, evStitch, evSize, evD2H;   /* per wave: uploaded, stitched, size copied, downloaded */
    ZSTDB200_stats stats;
    /* advanced one-shot API (ZSTD_CCtx_setParameter + ZSTD_compress2, lib/zstd.h:337-603): sticky parameters */
    int advLevel, advChecksum, advNoDictID;
    int advLdm;                    /* ZSTD_c_enableLongDistanceMatching: 1 = on (0 auto and 2 disable are off) */
    u32 advLdmPrm[4];              /* ZSTD_c_ldmHashLog, ldmMinMatch, ldmBucketSizeLog, ldmHashRateLog; 0 = derived from the window */
    /* long-distance matching workspace: the call's match list and per-block (first, count), one frame's scratch */
    ZbDevBuf<u64> d_ldmMatch, d_ldmFirst; ZbDevBuf<u32> d_ldmCnt; ZbDevBuf<u8> d_ldmScratch;
    std::unique_ptr<ZSTD_CDict, ZbCDictFree> advLocalDict;   /* ZSTD_CCtx_loadDictionary: owned copy, digested at its first use */
    const ZSTD_CDict* advRefCDict; /* ZSTD_CCtx_refCDict: borrowed */
    /* ZSTD_CCtx_refPrefix / ZSTDB200_CCtx_refPrefixDevice: borrowed, for the next frame only; digested into callDict by the
     * call that consumes it */
    const u8* advPrefix; size_t advPrefixSize; bool advPrefixOnDevice;
    ZbDevBuf<u8> d_prefix;         /* host prefix with LDM on: the indexed part, uploaded ahead of the LDM pass */
    ZbPlan plan;                   /* the call's plan; its vectors are reused (a million records are 100 MB of descriptors: fresh pages cost more than filling them) */
    /* streaming front end (ZSTD_compressStream2 with ZSTD_e_continue / ZSTD_e_flush): input collected on the host, compressed
     * output waiting to be handed out */
    u8* stIn; size_t stInSize, stInCap;
    u8* stOut; size_t stOutSize, stOutPos, stOutCap;
    int stFrames;                  /* frames produced in the current session */
    /* sequence calls (ZSTD_compressSequences): sticky ZSTD_c_blockDelimiters, staging of host sequences, import scratch */
    int advDelims;
    ZbDevBuf<ZSTD_Sequence> d_seqIn;
    ZbDevBuf<u8> d_seqTile, d_seqBlk; ZbDevBuf<u64> d_seqCtrl;
    /* stream-ordered calls (ZSTDB200_compressDeviceAsync / ZSTDB200_compressFramesAsync) plan into asyncPlan (ordinary memory,
     * so that planning makes no CUDA call) and stage their descriptors in a page-locked slot of a ring: slot s is free again
     * once evStage[s], recorded behind its upload, has completed.  evJoin: one per wave stream, a wave call's join. */
    ZbOrder order; ZbEvents evStage, evJoin;
    ZbPlan asyncPlan;
    ZbHostBuf<u8> stage[ZSTDB200_ASYNC_SLOTS]; bool stageBusy[ZSTDB200_ASYNC_SLOTS]; u32 stageNext;
};

static double zb_now(void) { struct timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts); return (double)ts.tv_sec + 1e-9 * (double)ts.tv_nsec; }

extern "C" int ZSTDB200_setDevice(int device) { g_device.store(device); return 0; }
int zb_contextDevice(void)
{
    int dev = g_device.load();
    if (dev < 0) { int cur = -1; if (cudaGetDevice(&cur) == cudaSuccess) dev = cur; else cudaGetLastError(); }
    return dev;
}
extern "C" int ZSTDB200_deviceAvailable(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n > 0;
}

extern "C" ZSTD_CCtx* ZSTD_createCCtx(void)
{
    ZSTD_CCtx* c = new (std::nothrow) ZSTD_CCtx();                           /* value-initialised: every plain member is zero */
    if (!c) return NULL;
    c->device = -1;
    c->bindDevice = zb_contextDevice();
    c->advLevel = 3;                                                         /* ZSTD_CLEVEL_DEFAULT */
    c->asyncPlan.blocks.pageable = c->asyncPlan.chunks.pageable = c->asyncPlan.frames.pageable = c->asyncPlan.dicts.pageable = true;
    {   const char* s = getenv("ZSTDB200_SERIAL"); const char* w = getenv("ZSTDB200_WAVE_BLOCKS");
        c->devWaveBlocks = (s && atoi(s)) ? 0u : (w ? (u32)atoi(w) : 1024u);     /* 128 MiB waves x 4 slots: among the best on the H100, tests/wave_sweep.py (DESIGN.md section 11) */
        const char* n = getenv("ZSTDB200_WAVE_SLOTS"); const char* h = getenv("ZSTDB200_HOST_WAVE_BLOCKS");
        c->waveSlots = n ? (u32)atoi(n) : ZB_WAVE_SLOTS_DEFAULT;
        c->hostWaveSlots = n ? (u32)atoi(n) : ZB_HOST_WAVE_SLOTS_DEFAULT;
        if (c->waveSlots < 1u) c->waveSlots = 1u;
        if (c->waveSlots > ZB_WAVE_SLOTS_MAX) c->waveSlots = ZB_WAVE_SLOTS_MAX;
        if (c->hostWaveSlots < 1u) c->hostWaveSlots = 1u;
        if (c->hostWaveSlots > ZB_WAVE_SLOTS_MAX) c->hostWaveSlots = ZB_WAVE_SLOTS_MAX;
        c->hostWaveBlocks = (h && atoi(h) > 0) ? (u32)atoi(h) : ZB_HOST_WAVE_BLOCKS; }
    return c;
}

static size_t zb_ctxInit(ZSTD_CCtx* c)
{
    if (c->device >= 0) { CK(cudaSetDevice(c->device)); return 0; }
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) { cudaGetLastError(); return ZB_ERR(ZB_error_GENERIC); }
    int dev = c->bindDevice;
    if (dev < 0) { if (cudaGetDevice(&dev) != cudaSuccess) dev = 0; }
    CK(cudaSetDevice(dev));
    /* everything or nothing: the stream and events are the context's only once every step succeeded (device stays -1
     * until then); after a failure they are destroyed here */
    ZbStream st; ZbEvents ev, evStage, evJoin; ZbOrder order;
    TRY(st.ensure());
    TRY(ev.ensure(EV_PHASES, true));
    TRY(order.create()); TRY(evStage.ensure(ZSTDB200_ASYNC_SLOTS, false)); TRY(evJoin.ensure(ZB_WAVE_SLOTS_MAX, false));
    /* the predefined FSE tables live in device memory (one copy per device; re-uploading the same bytes is harmless) */
    static ZbdFseCTable defaults[3]; static std::once_flag once;
    std::call_once(once, [] { zb_buildDefaultTables(defaults); });
    CK(zb_upload_default_tables(defaults, st));
    CK(cudaStreamSynchronize(st));
    c->stream = std::move(st); c->ev = std::move(ev);
    c->order = std::move(order); c->evStage = std::move(evStage); c->evJoin = std::move(evJoin);
    c->device = dev;
    return 0;
}

extern "C" size_t ZSTD_freeCCtx(ZSTD_CCtx* c)
{
    if (!c) return 0;
    free(c->stIn); free(c->stOut);
    return zb_deleteOnDevice(c, &c->order);                     /* its dictionaries, streams, events and buffers free themselves */
}

/* descriptors (per block / per frame, small) and the per-block workspace (d_work) are sized separately:
 * the host-pointer path runs the blocks in waves that share a few workspace slots */
static size_t zb_ensureDesc(ZSTD_CCtx* c, size_t nbBlocks, size_t nbFrames, size_t nbWaves, size_t nbChunks)
{
    TRY(c->d_chunks.ensure(nbChunks));
    TRY(c->d_blocks.ensure(nbBlocks)); TRY(c->d_outOffsets.ensure(nbBlocks + 1));
    TRY(c->d_frames.ensure(nbFrames)); TRY(c->d_verdict.ensure(nbFrames + 1)); TRY(c->h_verdict.ensure(nbFrames + 1));
    TRY(c->d_totals.ensure(nbWaves)); TRY(c->h_totals.ensure(nbWaves));
    return 0;
}

/* ------------------------------------------------------------------ dictionaries (zstd_compress.c:5119-5156)
 * < 8 bytes: ignored (:5132).  No magic 0xEC30A437: raw content (:5143-5148).  With it: zstd-format
 * dictionary = magic, dictID, Huffman table, OF/ML/LL FSE tables, 3 repcodes, content (:4987-5076).
 * The CONTENT of either kind is the history of each frame's first block; a zstd-format dictionary's Huffman /
 * FSE tables are that block's "previous" entropy state (treeless literals, set_repeat sequence tables) and
 * its repcodes start the block.  Parsing: zb_dict.cu. */
/* ------------------------------------------------------------------ planning (ZSTD_compress_frameChunk, zstd_compress.c:4527) */
/* One compression call, as every entry point hands it to the executor (zb_compress) */
struct ZbCall {
    void* dst; size_t dstCapacity; const void* src;
    const size_t* frameOffsets; const size_t* frameSizes; size_t nbFrames;
    const ZSTD_CDict* cdict;                                      /* the call's dictionary, or NULL */
    int level; size_t* cSizes;                                    /* cSizes: NULL, or one compressed size per frame */
    bool deviceMemory; cudaStream_t stream;                       /* stream: the caller's, or NULL; host-memory calls ignore it */
    bool checksum, noDictID;                                      /* frame header options */
    u64 partBegin = 0, partEnd = ~0ull;                           /* ZSTDB200_compressFramePart: this rank's share of the one frame */
    const u32* ldm = nullptr;                                     /* long-distance matching: the 4 ldm parameters (0 = derived), or NULL */
    /* the part of a prefix that the LDM pass indexes (its last min(size, 2^27) bytes; the whole prefix is the call's cdict),
     * in host or device memory; one frame per call */
    const u8* prefix = nullptr; u64 prefixSize = 0; bool prefixOnDevice = false;
    /* a stream-ordered call: its total (or error code) and per-frame sizes (may be NULL) go to device-writable memory, in
     * the order of `stream`, which is then the caller's also when NULL (the legacy default stream) */
    unsigned long long* result = nullptr; unsigned long long* d_cSizes = nullptr;
    const ZSTD_CDict* const* cdicts = nullptr;                    /* a dictionary per frame in place of cdict (NULL entries: none, at `level`) */
    /* ZSTD_generateSequences: each wave ends with the export of K1's stores as ZSTD_Sequence rows into dst instead of K2..K4;
     * dstCapacity counts rows */
    bool sequences = false;
};

static int g_strictLevels = 0;
/* Levels whose reference strategy is greedy or stronger (>= 5; 4 for frames <= 256 KiB / <= 16 KiB) have no counterpart here:
 * by default they are served by the strongest doubleFast row of their size class (larger output than the reference's at
 * that level); after ZSTDB200_setStrictLevels(1) such calls fail with parameter_unsupported instead. */
extern "C" void ZSTDB200_setStrictLevels(int on) { g_strictLevels = on; }

/* ZSTD_ldm_adjustParameters (zstd_ldm.c:135) for a frame of window 2^windowLog; v = the 4 sticky values, 0 = derived */
static ZbLdmParams zb_ldmResolve(const u32* v, u32 windowLog)
{
    ZbLdmParams p; memset(&p, 0, sizeof(p));
    p.hashLog = v[0]; p.minMatch = v[1]; p.bucketSizeLog = v[2]; p.hashRateLog = v[3]; p.windowLog = windowLog;
    if (!p.bucketSizeLog) p.bucketSizeLog = 3;                                       /* LDM_BUCKET_SIZE_LOG */
    if (!p.minMatch) p.minMatch = 64;                                                /* LDM_MIN_MATCH_LENGTH */
    if (!p.hashLog) p.hashLog = windowLog > 7u + 6u ? windowLog - 7u : 6u;           /* MAX(ZSTD_HASHLOG_MIN, windowLog - LDM_HASH_RLOG) */
    if (!p.hashRateLog) p.hashRateLog = windowLog < p.hashLog ? 0u : windowLog - p.hashLog;
    if (p.bucketSizeLog > p.hashLog) p.bucketSizeLog = p.hashLog;
    u32 const maxBits = p.minMatch < 64u ? p.minMatch : 64u;                         /* ZSTD_ldm_gear_init, zstd_ldm.c:32-60 */
    p.stopMask = (p.hashRateLog > 0u && p.hashRateLog <= maxBits) ? (((1ull << p.hashRateLog) - 1ull) << (maxBits - p.hashRateLog))
                                                                   : ((1ull << p.hashRateLog) - 1ull);
    return p;
}

/* the dictionary frame f is compressed against (a CDict given with less than 8 bytes counts as none, zstd_compress.c:5130),
 * and its level: a per-frame CDict's own, else the call's */
static const ZSTD_CDict* zb_frameCDict(const ZbCall& a, size_t f) { return a.cdicts ? a.cdicts[f] : a.cdict; }
static ZSTD_CDict* zb_usable(const ZSTD_CDict* cd) { return (cd && cd->size >= 8) ? const_cast<ZSTD_CDict*>(cd) : NULL; }

/* the slot of dictionary cd (NULL: none) under prms[prmIdx]: one table entry per pair, the repcodes it starts frames with */
static u32 zb_dictSlot(ZbPlan& P, ZSTD_CDict* cd, u32 prmIdx)
{
    u64 const key = (u64)(uintptr_t)cd | ((u64)prmIdx << 48);    /* user-space addresses fit in 48 bits */
    auto const it = P.slotOf.find(key);
    if (it != P.slotOf.end()) return it->second;
    ZbDictSlot e; memset(&e, 0, sizeof(e));
    e.codeRep[0] = 1; e.codeRep[1] = 4; e.codeRep[2] = 8;          /* zstd_internal.h:69 */
    if (cd && cd->entropy.present) {                               /* a zstd-format dictionary's repcodes (zstd_compress.c:5054-5056) */
        u32 const* r = cd->entropy.rep;
        e.codeRep[0] = r[0]; e.codeRep[1] = r[1]; e.codeRep[2] = r[2];
        e.startRep[0] = r[0] <= cd->tail ? r[0] : 0u; e.startRep[1] = r[1] <= cd->tail ? r[1] : 0u;
    }
    if (cd && P.seen.insert(cd).second) P.cdicts.push_back(cd);
    P.slots.push_back(ZbSlotInfo{ cd, prmIdx });
    P.slotOf.emplace(key, (u32)P.slots.size() - 1u);
    P.dicts.push_back(e);
    return (u32)P.slots.size() - 1u;
}

/* partBegin / partEnd: only the blocks that start inside [partBegin, partEnd) of the (single) frame are planned — one rank's
 * share of a frame that several GPUs compress together (ZSTDB200_compressFramePart); the geometry is the whole frame's.
 * Every frame has its own dictionary (zb_frameCDict) and level; the dictionary table has one entry per dictionary and
 * parameter group, and stays empty when no frame has a dictionary. */
static void zb_plan(ZbPlan& P, const ZbCall& a)
{
    const size_t* const frameOffsets = a.frameOffsets; const size_t* const frameSizes = a.frameSizes;
    size_t const nbFrames = a.nbFrames;
    P.reset();
    P.frames.resize(nbFrames);
    P.blocks.reserve(nbFrames);
    P.chunks.reserve(nbFrames);
    if (a.cdicts && P.tpl.size() < ZB_TEMPLATE_CACHE) P.tpl.assign(ZB_TEMPLATE_CACHE, ZbTemplate{});
    bool anyDict = false;
    u32 maxBlock = 0;
    /* calls made of many equal, single-block frames (config 5: a million 1 KiB records): the frame before is the template;
     * with a dictionary per frame, the last frame of the same size and dictionary is (found in P.tpl) */
    ZbTemplate cur; memset((void*)&cur, 0, sizeof(cur)); cur.size = ~0ull;
    for (size_t f = 0; f < nbFrames; f++) {
        u64 const fsz = frameSizes[f];
        const ZSTD_CDict* const raw = zb_frameCDict(a, f);
        P.frameBytes += fsz;
        ZbTemplate* slotT = NULL;
        if ((fsz != cur.size || raw != cur.raw) && a.cdicts) {
            u64 h = (((u64)(uintptr_t)raw >> 4) ^ (fsz * 0xC2B2AE3D27D4EB4Full)) * 0x9E3779B97F4A7C15ull;
            for (u32 k = 0; k < 16u; k++, h += 0x10000000000000ull) {
                ZbTemplate& t = P.tpl[h >> 50];                    /* 2^14 entries */
                if (t.gen != P.gen) { slotT = &t; break; }          /* free: the place of this frame's template */
                if (t.raw == raw && t.size == fsz) { if (!P.groups.empty() && t.prmIdx == P.groups.back().prmIdx) cur = t; break; }
            }
        }
        if (fsz == cur.size && raw == cur.raw) {
            P.frameBlocks++;
            ZbFrame fr = cur.fr; fr.srcOff = frameOffsets[f]; fr.firstBlock = (u32)P.blocks.size();
            ZbBlock b = cur.b; b.srcOff = fr.srcOff; b.frame = (u32)f;
            ZbChunk ch = cur.ch; ch.srcOff = fr.srcOff; ch.firstBlock = fr.firstBlock;
            P.blocks.push_back(b);
            P.chunks.push_back(ch);
            P.frames[f] = fr;
            P.groups.back().b1 = (u32)P.blocks.size();
            P.groups.back().c1 = (u32)P.chunks.size();
            P.groups.back().dict |= (b.flags & ZB_FLAG_DICT) != 0u;
            continue;
        }
        ZSTD_CDict* const cd = zb_usable(raw);
        int const level = (a.cdicts && raw) ? raw->level : a.level;
        size_t const dictSize = cd ? cd->size : 0, dictTail = cd ? cd->tail : 0;
        u32 const dictID = (cd && cd->entropy.present) ? cd->entropy.dictID : 0u;
        if (g_strictLevels && level > 4) P.unsupported = true;
        /* a frame of one chunk is parsed whole: compressed as without LDM, unless an indexed prefix lies in front of it */
        bool const ldm = a.ldm && fsz && fsz + a.prefixSize > ZB_LDM_MIN_FRAME;
        ZbCParams cp = zb_getCParams(level, fsz, dictSize, ldm);
        ZbParams prm = zb_makeParams(cp);
        if (ldm) {
            ZbLdmFrame lf; lf.frame = (u32)f; lf.prm = zb_ldmResolve(a.ldm, cp.windowLog); lf.matchBase = P.ldmMatches; lf.prefix = a.prefixSize;
            P.ldm.push_back(lf);
            P.ldmMatches += zb_ldm_survivor_cap(fsz + a.prefixSize, lf.prm.minMatch);
        }
        u32 prmIdx = 0;
        while (prmIdx < P.prms.size() && memcmp(&P.prms[prmIdx], &prm, sizeof(prm)) != 0) prmIdx++;
        if (prmIdx == P.prms.size()) P.prms.push_back(prm);
        anyDict |= cd != NULL;
        u32 const slot = zb_dictSlot(P, cd, prmIdx);
        size_t const blockMax = ((size_t)1 << cp.windowLog) < ZB_BLOCK_MAX ? ((size_t)1 << cp.windowLog) : ZB_BLOCK_MAX;   /* zstd_compress.c:2124 */
        u64 const chunkBytes = (u64)ZB_CHUNK_BLOCKS * blockMax;
        u64 const W = 1ull << cp.windowLog;
        ZbFrame fr; fr.srcOff = frameOffsets[f]; fr.srcSize = fsz; fr.firstBlock = (u32)P.blocks.size();
        fr.windowLog = cp.windowLog; fr.dictID = a.noDictID ? 0u : dictID; fr.checksum = a.checksum; fr.dictSlot = slot;
        u32 const firstChunk = (u32)P.chunks.size();
        bool dictBlocks = false;
        u64 pos = 0;
        do {
            u64 const bsz = (fsz - pos) < blockMax ? (fsz - pos) : blockMax;
            P.frameBlocks++;
            if (bsz > P.frameMaxBlock) P.frameMaxBlock = (u32)bsz;
            if (pos < a.partBegin || pos >= a.partEnd) { pos += bsz; continue; }      /* another rank's block */
            if (pos % chunkBytes == 0) {                         /* a new chunk starts with this block */
                ZbChunk ch; memset(&ch, 0, sizeof(ch));
                ch.srcOff = fr.srcOff + pos; ch.size = (u32)((fsz - pos) < chunkBytes ? (fsz - pos) : chunkBytes);
                ch.histLen = pos == 0 ? (u32)dictTail : (u32)(pos < ZB_PRIME_BYTES ? pos : ZB_PRIME_BYTES);
                ch.dictLen = pos == 0 ? (u32)dictTail : 0u;
                ch.firstBlock = (u32)P.blocks.size(); ch.blockLog = hb32((u32)blockMax); ch.dictSlot = slot;
                P.chunks.push_back(ch);
            }
            ZbChunk const& ch = P.chunks.back();
            /* positions in [dictionary tail | frame] coordinates: the frame starts at dictTail */
            u64 const chunkPos = ch.srcOff - fr.srcOff;
            u64 const chunkLow = dictTail + chunkPos - ch.histLen;
            u64 const bsBuf = dictTail + pos, beBuf = bsBuf + bsz;
            u64 low = chunkLow;
            if (beBuf > W && beBuf - W > low) low = beBuf - W;   /* ZSTD_window_enforceMaxDist at the block's end, zstd_compress_internal.h:1173 */
            ZbBlock b; memset(&b, 0, sizeof(b));
            b.srcOff = fr.srcOff + pos; b.size = (u32)bsz;
            b.histLen = (u32)(bsBuf - low);
            b.dictLen = low < dictTail ? (u32)(dictTail - low) : 0u;
            b.frame = (u32)f; b.flags = (pos == 0 ? ZB_FLAG_FIRST : 0u) | (pos + bsz == fsz ? ZB_FLAG_LAST : 0u) | (b.dictLen ? ZB_FLAG_DICT : 0u);
            b.dictSlot = slot;
            dictBlocks |= b.dictLen != 0u;
            P.blocks.push_back(b);
            if (b.size > maxBlock) maxBlock = b.size;
            pos += bsz;
        } while (pos < fsz);
        fr.nbBlocks = (u32)P.blocks.size() - fr.firstBlock;
        P.frames[f] = fr;
        if (P.groups.empty() || P.groups.back().prmIdx != prmIdx || P.groups.back().ldm != ldm) {
            ZbGroup g; g.prm = prm; g.b0 = fr.firstBlock; g.b1 = (u32)P.blocks.size(); g.c0 = firstChunk; g.c1 = (u32)P.chunks.size(); g.prmIdx = prmIdx; g.ldm = ldm; g.dict = dictBlocks; P.groups.push_back(g);
        } else { P.groups.back().b1 = (u32)P.blocks.size(); P.groups.back().c1 = (u32)P.chunks.size(); P.groups.back().dict |= dictBlocks; }
        if (fr.nbBlocks == 1u && !ldm) {
            cur.raw = raw; cur.size = fsz; cur.gen = P.gen; cur.prmIdx = prmIdx; cur.fr = fr; cur.b = P.blocks.back(); cur.ch = P.chunks.back();
            if (slotT) *slotT = cur;
        } else cur.size = ~0ull;
    }
    if (!anyDict) { P.dicts.clear(); P.slots.clear(); }          /* no table: every first block starts from the format's state */
    P.sd = zb_strides(maxBlock);
}

/* Parses dictionary bytes into cd: the entropy tables of a zstd-format dictionary, where its content starts and the content
 * tail that blocks can see.  A new digest has nothing on the device yet: no tail, no images.  rawContent: the bytes are
 * content whatever they begin with (a prefix, ZSTD_dct_rawContent) and are not read here; onDevice: they lie in device memory. */
static size_t zb_digestDict(ZSTD_CDict* cd, const u8* dict, size_t dictSize, bool rawContent = false, bool onDevice = false)
{
    cd->content = dict; cd->size = dict ? dictSize : 0; cd->contentOnDevice = onDevice;
    cd->contentOff = 0; cd->tail = 0; cd->resident = false; cd->nbImages = 0;
    memset(&cd->entropy, 0, sizeof(cd->entropy));
    if (cd->size < 8) return 0;                                          /* ignored by zb_compress */
    size_t const off = rawContent ? 0 : zb_loadDictionary(&cd->entropy, dict, cd->size);
    if (zb_isErr(off)) return off;
    cd->contentOff = off;
    size_t const contentSize = cd->size - off;
    cd->tail = contentSize < ZB_PRIME_BYTES ? contentSize : ZB_PRIME_BYTES;
    return 0;
}

/* Long-distance matching (zb_ldm.cu): every LDM frame's matches, by block index in the call, before the first wave (a block
 * may copy from anywhere in its 2^27-byte window, i.e. from any earlier wave).  The frames run one after another on
 * `stream` through one scratch area.  zb_ldmBuffers sizes the match list and that area, zb_runLdm launches. */
static size_t zb_ldmBuffers(ZSTD_CCtx* c, const ZbPlan& P)
{
    size_t scratch = 0;
    for (size_t i = 0; i < P.ldm.size(); i++) {
        u64 const n = P.frames[P.ldm[i].frame].srcSize;
        if (zb_ldm_survivor_cap(P.ldm[i].prefix + n, P.ldm[i].prm.minMatch) >> 32) return ZB_ERR(ZB_error_memory_allocation);   /* a survivor's index is a u32 */
        size_t const b = zb_ldm_scratch_bytes(P.ldm[i].prefix, n, &P.ldm[i].prm);
        if (b > scratch) scratch = b;
    }
    size_t const nbBlocks = P.blocks.size();
    TRY(c->d_ldmMatch.ensure(P.ldmMatches));
    TRY(c->d_ldmFirst.ensure(nbBlocks));
    TRY(c->d_ldmCnt.ensure(nbBlocks));
    TRY(c->d_ldmScratch.ensure(scratch));
    return 0;
}
static size_t zb_runLdm(ZSTD_CCtx* c, const ZbPlan& P, const u8* d_src, const u8* d_prefix, cudaStream_t stream, unsigned* launches)
{
    for (size_t i = 0; i < P.ldm.size(); i++) {
        ZbLdmFrame const& lf = P.ldm[i];
        ZbFrame const& fr = P.frames[lf.frame];
        CK(zb_launch_ldm(d_prefix, lf.prefix, d_src + fr.srcOff, fr.srcSize, &lf.prm, c->d_ldmScratch, fr.nbBlocks, lf.matchBase, c->d_ldmMatch,
                         c->d_ldmFirst + fr.firstBlock, c->d_ldmCnt + fr.firstBlock, stream));
        *launches += 4u + 3u * ((lf.prm.hashLog - lf.prm.bucketSizeLog + 7u) / 8u);   /* split, scan, compact, radix passes, select */
        if (lf.prefix >= lf.prm.minMatch && fr.srcSize >= lf.prm.minMatch) *launches += 1u;   /* a split launch per segment */
    }
    return 0;
}

/* K1..K3 for blocks [b0, b1) = chunks [c0, c1), block b0 in the first of `rows`; d_dicts: the call's dictionary table, or NULL;
 * matchOnly: K1 alone */
static size_t zb_runBlocks(ZSTD_CCtx* c, const ZbPlan& P, const u8* d_src, const ZbDictSlot* d_dicts, u32 b0, u32 b1, u32 c0, u32 c1,
                           const ZbWorkRows& rows, cudaStream_t stream, bool timed, unsigned* launches, bool matchOnly)
{
    for (int phase = 0; phase < (matchOnly ? 1 : 3); phase++) {
        for (size_t g = 0; g < P.groups.size(); g++) {
            ZbGroup const& G = P.groups[g];
            u32 const lo = G.b0 > b0 ? G.b0 : b0, hi = G.b1 < b1 ? G.b1 : b1;
            u32 const clo = G.c0 > c0 ? G.c0 : c0, chi = G.c1 < c1 ? G.c1 : c1;
            if (lo >= hi) continue;
            ZbWorkRows const R = rows.at(lo - b0);
            if (phase == 0) {
                ZbLdmView lv; lv.match = c->d_ldmMatch; lv.first = c->d_ldmFirst + lo; lv.cnt = c->d_ldmCnt + lo;
                CK(zb_launch_match(d_src, d_dicts, G.dict, c->d_blocks + lo, hi - lo, c->d_chunks + clo, chi - clo, lo, &G.prm, &R,
                                   (timed && P.groups.size() == 1) ? c->ev[EV_MID] : (cudaEvent_t)0, stream, G.ldm ? &lv : nullptr));
                *launches += G.prm.strategy == 2 ? 4 : 3;       /* walk(s), parse, merge */
            } else if (phase == 1) {
                CK(zb_launch_literals(c->d_blocks + lo, hi - lo, &G.prm, &R.sd, NULL, R.lits, R.body, R.meta, stream, d_dicts));
                *launches += 1;
            } else {
                CK(zb_launch_sequences(d_src, c->d_blocks + lo, hi - lo, &G.prm, &R.sd, NULL, R.seqs, R.dist, R.body, R.meta, stream, d_dicts));
                *launches += 1;
            }
        }
        if (timed) CK(cudaEventRecord(c->ev[EV_K1 + phase], stream));
    }
    return 0;
}

/* XXH64 (lib/common/xxhash.h: XXH64_update / XXH64_digest, seed 0) of the frame's content: the frame checksum is
 * its low 32 bits (zstd_compress.c:5297-5303).  A serial recurrence over 32-byte stripes: it runs on the calling
 * host thread while the GPU works (a large checksummed frame can be bound by this pass rather than by the GPU). */
static u64 zb_xxh64(const u8* p, size_t len)
{
    u64 const P1 = 0x9E3779B185EBCA87ull, P2 = 0xC2B2AE3D27D4EB4Full, P3 = 0x165667B19E3779F9ull, P4 = 0x85EBCA77C2B2AE63ull, P5 = 0x27D4EB2F165667C5ull;
    auto rotl = [](u64 x, int r) { return (x << r) | (x >> (64 - r)); };
    auto rd64 = [](const u8* q) { u64 v; memcpy(&v, q, 8); return v; };
    auto rd32 = [](const u8* q) { u32 v; memcpy(&v, q, 4); return v; };
    auto round = [&](u64 acc, u64 in) { return rotl(acc + in * P2, 31) * P1; };
    auto merge = [&](u64 acc, u64 v) { return (acc ^ round(0, v)) * P1 + P4; };
    const u8* const end = p + len;
    u64 h;
    if (len >= 32) {
        u64 v1 = P1 + P2, v2 = P2, v3 = 0, v4 = 0 - P1;
        const u8* const limit = end - 32;
        do { v1 = round(v1, rd64(p)); v2 = round(v2, rd64(p + 8)); v3 = round(v3, rd64(p + 16)); v4 = round(v4, rd64(p + 24)); p += 32; } while (p <= limit);
        h = rotl(v1, 1) + rotl(v2, 7) + rotl(v3, 12) + rotl(v4, 18);
        h = merge(h, v1); h = merge(h, v2); h = merge(h, v3); h = merge(h, v4);
    } else h = P5;
    h += (u64)len;
    while (p + 8 <= end) { h ^= round(0, rd64(p)); h = rotl(h, 27) * P1 + P4; p += 8; }
    if (p + 4 <= end) { h ^= (u64)rd32(p) * P1; h = rotl(h, 23) * P2 + P3; p += 4; }
    while (p < end) { h ^= (u64)(*p) * P5; h = rotl(h, 11) * P1; p++; }
    h ^= h >> 33; h *= P2; h ^= h >> 29; h *= P3; h ^= h >> 32;
    return h;
}

/* ------------------------------------------------------------------ stream-ordered calls */

/* Whether a call of nbFrames frames (0: a sequence call, which walks nothing) gives dictionary cd table images: always for a
 * caller's CDict (shared: other contexts may use it, and it keeps them across calls); the context's digest of a call's bytes
 * builds its images afresh on every call, only for 8 frames or more */
static bool zb_wantImages(const ZSTD_CCtx* c, const ZSTD_CDict* cd, size_t nbFrames)
{
    return cd->tail >= 8 && nbFrames > 0 && (cd != c->callDict.get() || nbFrames >= 8);
}

/* Before anything is enqueued: every dictionary of the call belongs to the context's device (or to none yet), and under
 * capture each can be used as it stands: no first upload, no upload that synchronises, and a ready table image for every
 * parameter group that would get one (zb_prepareDicts then uploads and builds nothing). */
static size_t zb_checkDicts(const ZSTD_CCtx* c, const ZbPlan& P, size_t nbFrames, bool capturing)
{
    for (size_t s = 0; s < P.slots.size(); s++) {
        ZSTD_CDict* const cd = P.slots[s].cd;
        if (!cd) continue;
        bool const shared = cd != c->callDict.get();
        std::lock_guard<std::mutex> g(cd->lock);
        if (cd->device >= 0 && cd->device != c->device) return ZB_ERR(ZB_error_parameter_unsupported);   /* one device per CDict */
        if (!capturing) continue;
        if (cd->device != c->device || (!cd->resident && (shared || !cd->contentOnDevice))) return ZB_ERR(ZB_error_stage_wrong);
        if (!zb_wantImages(c, cd, nbFrames)) continue;
        bool found = false;
        for (u32 i = 0; i < cd->nbImages; i++) found |= cd->images[i].ready && memcmp(&cd->images[i].prm, &P.prms[P.slots[s].prm], sizeof(ZbParams)) == 0;
        if (!found && cd->nbImages < ZB_MAX_IMAGES) return ZB_ERR(ZB_error_stage_wrong);
    }
    return 0;
}

/* Copies a stream-ordered call's descriptors into the next staging slot, which its queued upload then reads: the slot is
 * taken once the upload that last read it has run (the host waits only when the ring is full of calls still queued).  Every
 * slot has room for them: the call's sizing grew the ring.  Under capture the wait needs the relaxed capture mode (the event
 * was recorded outside the graph). */
static size_t zb_stageDescriptors(ZSTD_CCtx* c, const ZbPlan& P, u32* slot, const ZbBlock** blocks, const ZbFrame** frames, const ZbChunk** chunks,
                                  const ZbDictSlot** dicts)
{
    u32 const s = c->stageNext;
    c->stageNext = (s + 1u) % ZSTDB200_ASYNC_SLOTS;
    if (c->stageBusy[s]) {
        cudaStreamCaptureMode m = cudaStreamCaptureModeRelaxed;
        CK(cudaThreadExchangeStreamCaptureMode(&m));
        cudaError_t const e = cudaEventSynchronize(c->evStage[s]);
        cudaThreadExchangeStreamCaptureMode(&m);
        CK(e);
        c->stageBusy[s] = false;
    }
    size_t const nb = P.blocks.size() * sizeof(ZbBlock), nf = P.frames.size() * sizeof(ZbFrame), nc = P.chunks.size() * sizeof(ZbChunk);
    size_t const nd = P.dicts.size() * sizeof(ZbDictSlot);
    u8* const base = c->stage[s];
    size_t const offF = (nb + 15u) & ~(size_t)15u, offC = offF + ((nf + 15u) & ~(size_t)15u), offD = offC + ((nc + 15u) & ~(size_t)15u);
    memcpy(base, P.blocks.data(), nb); memcpy(base + offF, P.frames.data(), nf); memcpy(base + offC, P.chunks.data(), nc);
    if (nd) memcpy(base + offD, P.dicts.data(), nd);
    *slot = s; *blocks = (const ZbBlock*)base; *frames = (const ZbFrame*)(base + offF); *chunks = (const ZbChunk*)(base + offC);
    *dicts = (const ZbDictSlot*)(base + offD);
    return 0;
}
static size_t zb_stageBytes(const ZbPlan& P)
{
    return ((P.blocks.size() * sizeof(ZbBlock) + 15u) & ~(size_t)15u) + ((P.frames.size() * sizeof(ZbFrame) + 15u) & ~(size_t)15u)
         + ((P.chunks.size() * sizeof(ZbChunk) + 15u) & ~(size_t)15u) + P.dicts.size() * sizeof(ZbDictSlot);
}

/* ------------------------------------------------------------------ the executor: every compression call, in waves
 * H2D copy of wave w+1 | kernels of waves w, w-1, ... (one stream + workspace slot each) | D2H of finished waves.
 * A block needs ~ms of latency end to end (one warp walks it), so several waves are kept in flight. */
struct ZbWaves {                  /* the geometry of one call */
    bool single; ZbWorkKind kind; /* single: one wave, on the upload stream */
    std::vector<u32> wb, wc;      /* wave w = blocks [wb[w], wb[w + 1]) = chunks [wc[w], wc[w + 1]) */
    u32 nbWaves, maxWaveBlocks, slots;   /* workspace slot s = rows [s * maxWaveBlocks, (s + 1) * maxWaveBlocks) */
    size_t inEnd, outCap;         /* host buffers: input bytes to upload, room of the output staging (device: dstCapacity) */
};

/* Host code only.  Device-resident input: large calls are cut into waves on several streams, so that the shared-memory
 * bound candidate walk of one wave overlaps the register-only parse / entropy kernels of another; the rule counts whole
 * frames (a rank's share of a frame goes the way the whole frame would).  Host buffers: the call ends when the LAST wave has
 * gone through every kernel, so the final waves shrink (1/2, 1/4, 1/8 of a wave): less work behind the last upload. */
static ZbWaves zb_wavePlan(const ZSTD_CCtx* c, const ZbPlan& P, const ZbCall& a)
{
    ZbWaves W{};
    u32 const nbBlocks = (u32)P.blocks.size(), nbChunks = (u32)P.chunks.size();
    bool dfast = false;
    for (size_t g = 0; g < P.groups.size(); g++) dfast |= P.groups[g].prm.strategy == 2;
    W.kind = dfast ? ZB_WORK_DFAST : ZB_WORK_FAST;
    u64 const wsBytes = zb_workLayout(NULL, P.frameBlocks, W.kind, zb_strides(P.frameMaxBlock), NULL);   /* one-wave workspace */
    W.single = a.deviceMemory && ((a.stream && !a.result) || !c->devWaveBlocks ||
                                  (P.frameBytes < 2ull * c->devWaveBlocks * ZB_BLOCK_MAX && wsBytes <= (12ull << 30)));
    u32 const waveBlocks128 = a.deviceMemory ? c->devWaveBlocks : c->hostWaveBlocks;       /* wave size in 128 KiB blocks */
    u32 const waveSlots = a.deviceMemory ? c->waveSlots : c->hostWaveSlots;
    /* a wave is sized in bytes of input (and of workspace): calls made of small blocks get proportionally more blocks per wave */
    u32 const waveBlocks = W.single ? nbBlocks : (u32)((u64)waveBlocks128 * (ZB_BLOCK_MAX / P.sd.dist) > (1u << 22) ? (1u << 22) : waveBlocks128 * (ZB_BLOCK_MAX / P.sd.dist));
    std::vector<u32> tail, target;
    u32 left = nbBlocks;
    if (!a.deviceMemory) for (u32 sz = waveBlocks / 8u; sz >= 32u && sz < waveBlocks && left > 2u * sz; sz *= 2u) { tail.push_back(sz); left -= sz; }
    for (u32 b = 0; b < left; ) { u32 const e = (left - b > waveBlocks) ? b + waveBlocks : left; target.push_back(e - b); b = e; }
    for (size_t i = tail.size(); i-- > 0; ) target.push_back(tail[i]);
    /* a chunk is never split between waves: waves are filled chunk by chunk up to their target size */
    W.wb.push_back(0); W.wc.push_back(0);
    u32 acc = 0; size_t ti = 0;
    for (u32 ci = 0; ci < nbChunks; ci++) {
        u32 const nextFirst = ci + 1u < nbChunks ? P.chunks[ci + 1u].firstBlock : nbBlocks;
        acc += nextFirst - P.chunks[ci].firstBlock;
        if (ti < target.size() && acc >= target[ti] && ci + 1u < nbChunks) { W.wb.push_back(nextFirst); W.wc.push_back(ci + 1u); acc = 0; ti++; }
    }
    W.wb.push_back(nbBlocks); W.wc.push_back(nbChunks);
    W.nbWaves = (u32)W.wb.size() - 1u;
    for (u32 w = 0; w < W.nbWaves; w++) if (W.wb[w + 1] - W.wb[w] > W.maxWaveBlocks) W.maxWaveBlocks = W.wb[w + 1] - W.wb[w];
    W.slots = W.nbWaves < waveSlots ? W.nbWaves : waveSlots;
    size_t bound = 0;
    if (!a.deviceMemory) for (size_t f = 0; f < a.nbFrames; f++) {
        if (a.frameOffsets[f] + a.frameSizes[f] > W.inEnd) W.inEnd = a.frameOffsets[f] + a.frameSizes[f];
        bound += a.sequences ? ZSTD_sequenceBound(a.frameSizes[f]) : ZSTD_compressBound(a.frameSizes[f]) + 32;
    }
    W.outCap = a.deviceMemory ? a.dstCapacity : (a.dstCapacity < bound ? a.dstCapacity : bound);
    return W;
}

/* One compression call as its stages see it: zb_compress plans it (zb_plan, zb_wavePlan), sizes its buffers, enqueues it and
 * ends it in one of two ways, by where its buffers are (DESIGN.md section 2) */
struct ZbRun {
    ZSTD_CCtx* c; const ZbCall& a; ZbPlan& P; ZbWaves W;
    cudaStream_t sCopy;                             /* descriptors, dictionaries, input */
    bool timeline;                                  /* ZSTDB200_TIMELINE: print each wave's milestones */
    ZbWorkRows work;                                /* the rows of every slot */
    u8* d_in; u8* d_out; cudaStream_t sD2H;         /* kernel input and output, download stream */
    unsigned long long *d_result, *d_sizes;         /* where the verdict kernel writes: the caller's memory, or c->d_verdict */
    unsigned launches; size_t err, prefixUp;        /* err: a launch failed; the call still finishes what it queued */
    double t0, hostEnq; std::vector<double> hostDone;   /* host clock: enqueue start and duration, each wave's size seen */
    std::vector<std::pair<ZSTD_CDict*, u32>> building;   /* images (CDict, index) this call builds; ready once built */
    /* The call's dictionaries on the device, in bulk and one CDict lock at a time (CDicts are shared between contexts on other
     * threads): the tails and entropy states not yet resident are uploaded, then the call synchronises once if a caller's CDict
     * was among them; the table gets every entry's addresses; the images it lacks are registered (allocated at the size of
     * their group's tables) and queued in P.imageChunks by parameters, for one walk launch per table (runImageBuilds).  A
     * dictionary with no free image slot for a group walks its tail per frame there, which gives the same bytes.  Two
     * contexts that upload or build the same thing at once write the same bytes; a reader waits for `resident` / `ready`. */
    size_t prepareDicts() {
        std::vector<ZSTD_CDict*> uploaded;
        for (ZSTD_CDict* cd : P.cdicts) {
            bool const shared = cd != c->callDict.get();
            std::lock_guard<std::mutex> g(cd->lock);
            if (cd->device >= 0 && cd->device != c->device) return ZB_ERR(ZB_error_parameter_unsupported);
            if (cd->resident) continue;
            /* the tail with 32 bytes of zeros on both sides; the context's own digest takes the largest tail once */
            TRY(cd->d_dict.ensure(shared ? cd->tail + 64 : ZB_PRIME_BYTES + 64));
            if (cd->entropy.present) TRY(cd->d_de.ensure(1));
            cd->device = c->device;
            CK(cudaMemsetAsync(cd->d_dict, 0, 32, sCopy)); CK(cudaMemsetAsync(cd->d_dict + 32 + cd->tail, 0, 32, sCopy));
            if (cd->tail) CK(cudaMemcpyAsync(cd->d_dict + 32, cd->content + (cd->size - cd->tail), cd->tail,
                                             cd->contentOnDevice ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, sCopy));
            if (cd->entropy.present) CK(cudaMemcpyAsync(cd->d_de, &cd->entropy, sizeof(ZbDictEntropy), cudaMemcpyHostToDevice, sCopy));
            if (shared) uploaded.push_back(cd); else cd->resident = true;
        }
        if (!uploaded.empty()) {
            CK(cudaStreamSynchronize(sCopy));
            for (ZSTD_CDict* cd : uploaded) { std::lock_guard<std::mutex> g(cd->lock); cd->resident = true; }
        }
        std::vector<std::pair<u32, u32>> builds;        /* (parameters, slot) */
        for (size_t s = 0; s < P.slots.size(); s++) {
            ZSTD_CDict* const cd = P.slots[s].cd;
            if (!cd) continue;
            ZbDictSlot& e = P.dicts[s];
            e.end = cd->d_dict.p + 32 + cd->tail; e.de = cd->entropy.present ? cd->d_de.p : NULL; e.image = NULL;
            if (!zb_wantImages(c, cd, a.nbFrames)) continue;
            ZbParams const& prm = P.prms[P.slots[s].prm];
            std::lock_guard<std::mutex> g(cd->lock);
            u32 i = 0;
            while (i < cd->nbImages && memcmp(&cd->images[i].prm, &prm, sizeof(prm)) != 0) i++;
            if (i == cd->nbImages) {
                if (i >= ZB_MAX_IMAGES) continue;
                /* a caller's CDict fills a slot once; the context's digest, re-made every call, takes the largest tables at
                 * once, so that no later call frees an image a stream-ordered call still queued may read */
                TRY(cd->images[i].img.ensure(cd != c->callDict.get() ? prm.tableN + (prm.strategy == 2 ? prm.tableNLong : 0u)
                                                                       : ZB_DFAST_SHORT_MAX + (1u << ZB_DFAST_LONGLOG_MAX)));
                cd->images[i].prm = prm; cd->images[i].ready = false; cd->nbImages++;
            }
            e.image = cd->images[i].img;
            if (!cd->images[i].ready) { builds.emplace_back(P.slots[s].prm, (u32)s); building.emplace_back(cd, i); }
        }
        std::sort(builds.begin(), builds.end());
        P.imageBuilds.assign(P.prms.size() + 1, 0u);
        for (auto const& b : builds) {
            ZbChunk ch; memset(&ch, 0, sizeof(ch));
            u32 const tail = (u32)P.slots[b.second].cd->tail;
            ch.histLen = tail; ch.dictLen = tail; ch.blockLog = 17; ch.dictSlot = b.second;
            P.imageChunks.push_back(ch);
            P.imageBuilds[b.first + 1]++;
        }
        for (size_t i = 1; i < P.imageBuilds.size(); i++) P.imageBuilds[i] += P.imageBuilds[i - 1];
        return 0;
    }
    /* the images prepareDicts queued, one launch per table of each parameter group (the table is on the device); a caller's
     * CDict's image must be complete before another context reads it: one synchronisation for all of them */
    size_t runImageBuilds() {
        if (P.imageChunks.empty()) return 0;
        CK(cudaMemcpyAsync(c->d_imageChunks, P.imageChunks.data(), P.imageChunks.size() * sizeof(ZbChunk), cudaMemcpyHostToDevice, sCopy));   /* pageable source: staged before the call returns */
        for (size_t p = 0; p + 1 < P.imageBuilds.size(); p++) {
            u32 const n = P.imageBuilds[p + 1] - P.imageBuilds[p];
            if (!n) continue;
            CK(zb_launch_dict_images(c->d_dicts, c->d_imageChunks + P.imageBuilds[p], n, &P.prms[p], sCopy));
            launches += P.prms[p].strategy == 2 ? 2u : 1u;
        }
        bool shared = false;
        for (auto const& b : building) shared |= b.first != c->callDict.get();
        if (shared) CK(cudaStreamSynchronize(sCopy));
        for (auto const& b : building) { std::lock_guard<std::mutex> g(b.first->lock); b.first->images[b.second].ready = true; }
        return 0;
    }
    /* every buffer the call needs, before its first work is enqueued (run through ZbOrder::Call::size) */
    size_t sizeBuffers() {
        TRY(zb_ensureDesc(c, P.blocks.size(), a.nbFrames, W.nbWaves, P.chunks.size()));
        size_t const bytes = zb_workLayout(NULL, (size_t)W.slots * W.maxWaveBlocks, W.kind, P.sd, NULL);
        TRY(bytes); TRY(c->d_work.ensure(bytes));
        zb_workLayout(c->d_work, (size_t)W.slots * W.maxWaveBlocks, W.kind, P.sd, &work);
        /* the wave events are created once and kept: a call creates none unless it has more waves than any call before it (or
         * ZSTDB200_TIMELINE changed, which wants timed events) */
        TRY(c->evH2D.ensure(W.nbWaves, timeline)); TRY(c->evStitch.ensure(W.nbWaves, timeline));
        TRY(c->evSize.ensure(W.nbWaves, timeline)); TRY(c->evD2H.ensure(W.nbWaves, timeline));
        /* wave streams are created on first use: every stream beyond the hardware queue count (8 by default) shares a
         * queue with another one, and a download queued behind another wave's kernels stalls the whole pipeline */
        if (!W.single) for (u32 s = 0; s < W.slots; s++) TRY(c->waveStream[s].ensure());
        if (!a.deviceMemory) { TRY(c->d_in.ensure(W.inEnd + 16)); TRY(c->d_out.ensure(W.outCap * (a.sequences ? sizeof(ZSTD_Sequence) : 1) + 16)); TRY(c->waveStream[ZB_WAVE_SLOTS_MAX].ensure()); }
        if (!P.ldm.empty()) TRY(zb_ldmBuffers(c, P));
        TRY(c->d_dicts.ensure(P.dicts.size())); TRY(c->d_imageChunks.ensure(P.cdicts.empty() ? 0 : P.slots.size()));   /* at most an image per entry */
        size_t const stageBytes = a.result ? zb_stageBytes(P) : 0;
        for (u32 s = 0; s < ZSTDB200_ASYNC_SLOTS && stageBytes; s++)
            if (c->stage[s].cap < stageBytes) { TRY(c->stage[s].ensure(stageBytes)); c->stageBusy[s] = false; }   /* every slot, so that any can serve a capture */
        return 0;
    }
    /* everything the call queues, behind the context's earlier calls, up to and including the last wave's stitch */
    size_t enqueue(ZbOrder::Call& call) {
        bool const async = a.result != nullptr, ldm = !P.ldm.empty();
        d_in = a.deviceMemory ? (u8*)a.src : c->d_in.p; d_out = a.deviceMemory ? (u8*)a.dst : c->d_out.p;
        sD2H = a.deviceMemory ? (cudaStream_t)0 : c->waveStream[ZB_WAVE_SLOTS_MAX].s;
        d_result = async ? a.result : c->d_verdict.p; d_sizes = async ? a.d_cSizes : c->d_verdict.p + 1;
        hostDone.assign(W.nbWaves, 0.0);
        t0 = zb_now();
        TRY(call.enter(sCopy));
        if (!P.cdicts.empty()) TRY(prepareDicts());
        const ZbBlock* hBlocks = P.blocks.data(); const ZbFrame* hFrames = P.frames.data(); const ZbChunk* hChunks = P.chunks.data();
        const ZbDictSlot* hDicts = P.dicts.data();
        u32 stageSlot = 0;
        if (async) TRY(zb_stageDescriptors(c, P, &stageSlot, &hBlocks, &hFrames, &hChunks, &hDicts));
        const ZbDictSlot* const d_dicts = P.dicts.size() ? c->d_dicts.p : NULL;   /* NULL: no frame has a dictionary */
        if (!W.single && !async) CK(cudaEventRecord(c->ev[EV_START], sCopy));
        CK(cudaMemcpyAsync(c->d_blocks, hBlocks, P.blocks.size() * sizeof(ZbBlock), cudaMemcpyHostToDevice, sCopy));
        CK(cudaMemcpyAsync(c->d_frames, hFrames, a.nbFrames * sizeof(ZbFrame), cudaMemcpyHostToDevice, sCopy));
        CK(cudaMemcpyAsync(c->d_chunks, hChunks, P.chunks.size() * sizeof(ZbChunk), cudaMemcpyHostToDevice, sCopy));
        if (d_dicts) CK(cudaMemcpyAsync(c->d_dicts, hDicts, P.dicts.size() * sizeof(ZbDictSlot), cudaMemcpyHostToDevice, sCopy));
        if (async && !call.capturing) { CK(cudaEventRecord(c->evStage[stageSlot], sCopy)); c->stageBusy[stageSlot] = true; }
        if (W.single && !async) CK(cudaEventRecord(c->ev[EV_K0], sCopy));   /* events around each phase of a synchronous wave */
        TRY(runImageBuilds());
        if (ldm) {
            /* host buffers: the whole input goes up first (a block may copy from any earlier wave), so this upload does not
             * overlap the kernels as the per-wave uploads do */
            if (!a.deviceMemory) CK(cudaMemcpyAsync(d_in, a.src, W.inEnd, cudaMemcpyHostToDevice, sCopy));
            const u8* d_prefix = a.prefix;                        /* the indexed prefix: in place on the device, or uploaded like the input */
            if (a.prefixSize && !a.prefixOnDevice) {
                TRY(c->d_prefix.ensure(a.prefixSize));
                CK(cudaMemcpyAsync(c->d_prefix, a.prefix, a.prefixSize, cudaMemcpyHostToDevice, sCopy));
                d_prefix = c->d_prefix; prefixUp = a.prefixSize;
            }
            err = zb_runLdm(c, P, d_in, d_prefix, sCopy, &launches);
        }
        for (u32 w = 0; w < W.nbWaves && !err; w++) {
            u32 const b0 = W.wb[w], b1 = W.wb[w + 1];
            ZbWorkRows const rows = work.at((size_t)(w % W.slots) * W.maxWaveBlocks);
            if (!a.deviceMemory && !ldm) {
                /* input bytes of the wave (frames are laid out in offset order; history was uploaded by earlier waves) */
                u64 lo = ~0ull, hi = 0;
                for (u32 b = b0; b < b1; b++) { u64 const s = P.blocks[b].srcOff, e = s + P.blocks[b].size; if (s < lo) lo = s; if (e > hi) hi = e; }
                if (hi > lo) CK(cudaMemcpyAsync(d_in + lo, (const u8*)a.src + lo, hi - lo, cudaMemcpyHostToDevice, sCopy));
            }
            cudaStream_t st = sCopy;
            if (!W.single) {
                CK(cudaEventRecord(c->evH2D[w], sCopy));
                TRY(c->waveStream[w % W.slots].ensure());
                st = c->waveStream[w % W.slots];
                CK(cudaStreamWaitEvent(st, c->evH2D[w], 0));
            }
            err = zb_runBlocks(c, P, d_in, d_dicts, b0, b1, W.wc[w], W.wc[w + 1], rows, st, W.single && !async, &launches, a.sequences);
            if (err) break;
            if (w > 0) CK(cudaStreamWaitEvent(st, c->evStitch[w - 1], 0));
            if (a.sequences)                                      /* the rows are placed as the stitch places bytes, wave after wave */
                CK(zb_launch_seqexport(c->d_blocks + b0, b1 - b0, d_dicts, &rows, c->d_outOffsets + b0, w > 0 ? c->d_totals + (w - 1) : NULL,
                                       c->d_totals + w, d_out, W.outCap, st));
            else
                CK(zb_launch_stitch(d_in, c->d_blocks + b0, b1 - b0, c->d_frames, &rows,
                                    c->d_outOffsets + b0, w > 0 ? c->d_totals + (w - 1) : NULL, c->d_totals + w, d_out, W.outCap, st));
            launches += 2;
            if (!W.single) CK(cudaEventRecord(c->evStitch[w], st));
            /* the wave's size goes to the host behind the event the next wave's stitch waits for: a store into mapped
             * host memory from inside the scan kernel would add a PCIe round trip to every link of that chain */
            if (!a.deviceMemory || timeline) {
                CK(cudaMemcpyAsync(c->h_totals + w, c->d_totals + w, sizeof(u64), cudaMemcpyDeviceToHost, st));
                CK(cudaEventRecord(c->evSize[w], st));
            }
        }
        hostEnq = zb_now() - t0;
        return 0;
    }
    /* the end of every call on device buffers: the waves join sCopy, which then runs the checksum and verdict kernels; a
     * stream-ordered call then records the context's order event, a synchronous one waits for its verdict */
    size_t finishOrdered(ZbOrder::Call& call) {
        if (!err) {
            if (!W.single) for (u32 s = 0; s < W.slots; s++) {
                CK(cudaEventRecord(c->evJoin[s], c->waveStream[s]));
                CK(cudaStreamWaitEvent(sCopy, c->evJoin[s], 0));
            }
            if (a.checksum) { CK(zb_launch_checksums(d_in, c->d_frames, (u32)a.nbFrames, c->d_outOffsets, d_out, W.outCap, sCopy)); launches++; }
            CK(zb_launch_call_result(c->d_frames, (u32)a.nbFrames, c->d_outOffsets, c->d_totals + W.nbWaves - 1, a.dstCapacity, d_sizes, d_result, sCopy));
            launches++;
        }
        if (a.result) { TRY(call.leave(sCopy)); c->stats.launches = launches; c->stats.nbBlocks = (u32)P.blocks.size(); return err; }
        CK(cudaEventRecord(c->ev[W.single ? EV_KEND : EV_END], sCopy));
        if (timeline) for (u32 w = 0; w < W.nbWaves && !err; w++) {   /* each wave's milestones, as for host buffers */
            CK(cudaEventSynchronize(c->evSize[w]));
            hostDone[w] = zb_now() - t0;
            CK(cudaEventRecord(c->evD2H[w], sCopy));
        }
        return endSync(sCopy, a.cSizes != nullptr);
    }
    /* what both synchronous ends share once the verdict kernel is queued on `st` behind all of the call's kernels: one copy
     * reads the verdict back (with every frame's size when `sizes`) and the host waits for it; then the timeline and the
     * stats.  After a failed launch the host waits for every stream instead. */
    size_t endSync(cudaStream_t st, bool sizes) {
        if (err) {
            if (!W.single) for (u32 s = 0; s < W.slots; s++) CK(cudaStreamSynchronize(c->waveStream[s]));
            CK(cudaStreamSynchronize(sCopy));
            return err;
        }
        CK(cudaMemcpyAsync(c->h_verdict, c->d_verdict, (sizes ? 1 + a.nbFrames : 1) * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        if (a.cSizes) for (size_t f = 0; f < a.nbFrames; f++) a.cSizes[f] = (size_t)c->h_verdict[1 + f];
        if (timeline) {
            fprintf(stderr, "zstd_b200 timeline (ms after the call's first enqueue; host enqueue loop took %.3f ms; %s)\n", 1e3 * hostEnq,
                    a.deviceMemory ? "device buffers" : "per-wave downloads");
            for (u32 w = 0; w < W.nbWaves; w++) {
                float up = 0, st = 0, dn = 0;
                cudaEventElapsedTime(&up, c->ev[EV_START], c->evH2D[w]); cudaEventElapsedTime(&st, c->ev[EV_START], c->evStitch[w]);
                cudaEventElapsedTime(&dn, c->ev[EV_START], c->evD2H[w]);
                fprintf(stderr, "  wave %2u blocks %5u..%5u : uploaded %7.3f  stitched %7.3f (host saw it %7.3f)  downloaded %7.3f\n",
                        w, W.wb[w], W.wb[w + 1], up, st, 1e3 * hostDone[w], dn);
            }
        }
        float ms = 0;
        if (W.single) {
            cudaEventElapsedTime(&ms, c->ev[EV_K0], c->ev[EV_KEND]); c->stats.kernel_ms = ms;
            cudaEventElapsedTime(&ms, c->ev[EV_K0], c->ev[EV_K1]); c->stats.match_ms = ms;
            if (P.groups.size() == 1) { cudaEventElapsedTime(&ms, c->ev[EV_K0], c->ev[EV_MID]); c->stats.cand_ms = ms; cudaEventElapsedTime(&ms, c->ev[EV_MID], c->ev[EV_K1]); c->stats.parse_ms = ms; }
            if (a.sequences) { cudaEventElapsedTime(&ms, c->ev[EV_K1], c->ev[EV_KEND]); c->stats.stitch_ms = ms; }   /* K1, then the export */
            else {
                cudaEventElapsedTime(&ms, c->ev[EV_K1], c->ev[EV_K2]); c->stats.literals_ms = ms;
                cudaEventElapsedTime(&ms, c->ev[EV_K2], c->ev[EV_K3]); c->stats.sequences_ms = ms;
                cudaEventElapsedTime(&ms, c->ev[EV_K3], c->ev[EV_KEND]); c->stats.stitch_ms = ms;
            }
        } else { cudaEventElapsedTime(&ms, c->ev[EV_START], c->ev[EV_END]); c->stats.kernel_ms = ms; }
        c->stats.total_ms = c->stats.kernel_ms;
        c->stats.launches = launches; c->stats.nbBlocks = (u32)P.blocks.size();
        if (!a.deviceMemory) { c->stats.h2d_bytes = W.inEnd + prefixUp; c->stats.d2h_bytes = (size_t)c->h_totals[W.nbWaves - 1]; }
        return (size_t)c->h_verdict[0];
    }
    /* a synchronous call's end on host buffers: the verdict kernel behind the last wave's stitch (host calls always run in
     * waves), XXH64 on up to 8 host threads while the GPU works, each wave downloaded as its size arrives, the checksums
     * written into the 4 bytes the size scan left free behind every frame */
    size_t finishHost() {
        const u8* const src = (const u8*)a.src; u8* const dst = (u8*)a.dst;
        cudaStream_t const last = c->waveStream[(W.nbWaves - 1u) % W.slots];   /* ordered behind every earlier wave's stitch */
        if (!err) { CK(zb_launch_call_result(c->d_frames, (u32)a.nbFrames, c->d_outOffsets, c->d_totals + W.nbWaves - 1, a.dstCapacity, d_sizes, d_result, last)); launches++; }
        if (a.sequences) {                                        /* one download of exactly the rows written, once the verdict is known */
            CK(cudaEventRecord(c->ev[EV_END], last));
            size_t const n = endSync(last, false);
            if (zb_isErr(n)) return n;
            if (n) CK(cudaMemcpyAsync(dst, d_out, n * sizeof(ZSTD_Sequence), cudaMemcpyDeviceToHost, last));
            CK(cudaStreamSynchronize(last));
            c->stats.d2h_bytes = n * sizeof(ZSTD_Sequence);
            return n;
        }
        std::vector<u64> xxh;
        if (a.checksum && !err) {
            xxh.resize(a.nbFrames);
            size_t const nt = a.nbFrames < 8 ? a.nbFrames : 8;
            if (nt <= 1) xxh[0] = zb_xxh64(src + a.frameOffsets[0], a.frameSizes[0]);
            else {
                std::vector<std::thread> th;
                for (size_t t = 0; t < nt; t++) th.emplace_back([&, t] { for (size_t f = t; f < a.nbFrames; f += nt) xxh[f] = zb_xxh64(src + a.frameOffsets[f], a.frameSizes[f]); });
                for (size_t t = 0; t < nt; t++) th[t].join();
            }
        }
        for (u64 w = 0, prev = 0; w < W.nbWaves && !err; w++) {
            CK(cudaEventSynchronize(c->evSize[w]));
            hostDone[w] = zb_now() - t0;
            u64 const total = c->h_totals[w];
            if (total <= W.outCap && total > prev) CK(cudaMemcpyAsync(dst + prev, d_out + prev, total - prev, cudaMemcpyDeviceToHost, sD2H));
            if (total <= W.outCap) prev = total;
            if (timeline) CK(cudaEventRecord(c->evD2H[w], sD2H));
        }
        CK(cudaEventRecord(c->ev[EV_END], sD2H)); CK(cudaStreamSynchronize(sD2H));
        size_t const total = endSync(last, a.cSizes || a.checksum);
        if (!zb_isErr(total) && a.checksum) for (size_t f = 0, end = 0; f < a.nbFrames; f++) {
            end += c->h_verdict[1 + f];
            if (end < 4 || end > total) break;
            u32 const ck = (u32)xxh[f];
            dst[end - 4] = (u8)ck; dst[end - 3] = (u8)(ck >> 8); dst[end - 2] = (u8)(ck >> 16); dst[end - 1] = (u8)(ck >> 24);
        }
        return total;
    }
};

static size_t zb_compress(ZSTD_CCtx* c, const ZbCall& a)
{
    bool const async = a.result != nullptr;
    if (a.nbFrames == 0 && !async) return 0;
    ZbDeviceGuard guard;
    ZbOrder::Call call(c->order);
    if (async) TRY(call.begin(c->device, a.stream));
    TRY(zb_ctxInit(c));
    memset(&c->stats, 0, sizeof(c->stats));
    if (a.nbFrames == 0) {                                        /* a batch without frames: its total, 0, in stream order */
        CK(zb_launch_call_result(NULL, 0, NULL, NULL, a.dstCapacity, NULL, a.result, a.stream));
        c->stats.launches = 1;
        return 0;
    }
    /* the dictionaries: a caller's ZSTD_CDicts, which other contexts may share (their device state is guarded by cd->lock), or
     * the context's digest of this call's bytes */
    ZbPlan& P = async ? c->asyncPlan : c->plan;
    zb_plan(P, a);
    if (P.unsupported) return ZB_ERR(ZB_error_parameter_unsupported);
    TRY(zb_checkDicts(c, P, a.nbFrames, call.capturing));
    ZbRun r{c, a, P, zb_wavePlan(c, P, a), (async || (a.deviceMemory && a.stream)) ? a.stream : c->stream};
    r.timeline = !r.W.single && !async && !a.sequences && getenv("ZSTDB200_TIMELINE") != NULL;
    TRY(call.size([&] { return r.sizeBuffers(); }));
    TRY(r.enqueue(call));
    return a.deviceMemory ? r.finishOrdered(call) : r.finishHost();
}

/* dictionary bytes passed to a call, digested into the context's callDict (*out = NULL without a dictionary) */
static size_t zb_digestCallDict(ZSTD_CCtx* c, const void* dict, size_t dictSize, const ZSTD_CDict** out)
{
    *out = NULL;
    if (!dict) return 0;
    if (!c->callDict) c->callDict.reset(ZSTD_createCDict(NULL, 0, 0));
    if (!c->callDict) return ZB_ERR(ZB_error_memory_allocation);
    TRY(zb_digestDict(c->callDict.get(), (const u8*)dict, dictSize));
    *out = c->callDict.get();
    return 0;
}

/* the sticky long-distance-matching parameters of a call that honours them, or NULL when LDM is off */
static const u32* zb_ldmArg(const ZSTD_CCtx* c) { return c->advLdm ? c->advLdmPrm : nullptr; }

/* One frame against the pending prefix (ZSTD_CCtx_refPrefix, zstd_compress.c:6272-6275): the prefix is this frame's only,
 * so it is forgotten first, whatever becomes of the call.  It is a raw-content dictionary, digested into the context's
 * callDict (a prefix of less than 8 bytes is ignored, as any dictionary that short); with LDM on its last 2^27 bytes, all
 * that a block can reach, are indexed along with the frame.  d_result: a stream-ordered call's verdict (NULL: synchronous). */
static size_t zb_compressWithPrefix(ZSTD_CCtx* c, void* dst, size_t dstCapacity, const void* src, size_t srcSize, int level,
                                    bool deviceMemory, cudaStream_t stream, unsigned long long* d_result = nullptr)
{
    const u8* const prefix = c->advPrefix; size_t const size = c->advPrefixSize; bool const onDevice = c->advPrefixOnDevice;
    c->advPrefix = NULL; c->advPrefixSize = 0;
    if (onDevice && !deviceMemory) return ZB_ERR(ZB_error_parameter_unsupported);    /* a host-buffer call uploads what it reads */
    if (!deviceMemory && dstCapacity && !dst) return ZB_ERR(ZB_error_dstBuffer_null);
    if (!deviceMemory && dstCapacity < 18) return ZB_ERR(ZB_error_dstSize_tooSmall);
    if (!c->callDict) c->callDict.reset(ZSTD_createCDict(NULL, 0, 0));
    if (!c->callDict) return ZB_ERR(ZB_error_memory_allocation);
    TRY(zb_digestDict(c->callDict.get(), prefix, size, true, onDevice));
    size_t const off = 0;
    ZbCall a = { dst, dstCapacity, src, &off, &srcSize, 1, c->callDict.get(), level, NULL, deviceMemory, stream,
                 c->advChecksum != 0, c->advNoDictID != 0 };
    a.ldm = zb_ldmArg(c); a.result = d_result;
    if (a.ldm && size >= 8) {
        u64 const reach = 1ull << ZB_LDM_WINDOW_LOG;
        a.prefixSize = size < reach ? size : reach; a.prefix = prefix + (size - a.prefixSize); a.prefixOnDevice = onDevice;
    }
    return zb_compress(c, a);
}

extern "C" size_t ZSTDB200_compressFrames(ZSTD_CCtx* c, void* dst, size_t dstCapacity,
                                          const void* src, const size_t* frameOffsets, const size_t* frameSizes,
                                          size_t nbFrames, const void* dict, size_t dictSize,
                                          size_t* cSizes, int level, int deviceMemory, void* streamv)
{
    if (!c) return ZB_ERR(ZB_error_GENERIC);
    if (c->advPrefix) return ZB_ERR(ZB_error_parameter_unsupported);            /* "the next frame only" has no meaning for a batch */
    const ZSTD_CDict* cd;
    TRY(zb_digestCallDict(c, dict, dictSize, &cd));
    ZbCall a = { dst, dstCapacity, src, frameOffsets, frameSizes, nbFrames, cd, level, cSizes, deviceMemory != 0,
                 (cudaStream_t)streamv, c->advChecksum != 0, c->advNoDictID != 0 };            /* the sticky frame parameters of ZSTD_CCtx_setParameter apply */
    a.ldm = zb_ldmArg(c);
    return zb_compress(c, a);
}

extern "C" size_t ZSTDB200_compressFrames_usingCDict(ZSTD_CCtx* c, void* dst, size_t dstCapacity,
                                                     const void* src, const size_t* frameOffsets, const size_t* frameSizes,
                                                     size_t nbFrames, const ZSTD_CDict* cdict,
                                                     size_t* cSizes, int deviceMemory, void* streamv)
{
    if (!cdict) return ZB_ERR(ZB_error_dictionary_wrong);                        /* zstd_compress.c:5753 */
    if (!c) return ZB_ERR(ZB_error_GENERIC);
    if (c->advPrefix) return ZB_ERR(ZB_error_parameter_unsupported);
    ZbCall a = { dst, dstCapacity, src, frameOffsets, frameSizes, nbFrames, cdict, cdict->level, cSizes, deviceMemory != 0,
                 (cudaStream_t)streamv, c->advChecksum != 0, c->advNoDictID != 0 };
    a.ldm = zb_ldmArg(c);
    return zb_compress(c, a);
}

/* A batch whose frames each have their own CDict (contrib/largeNbDicts/largeNbDicts.c:627-633 walks one per block): frame i
 * at cdicts[i]'s level against it, or at `level` without a dictionary where cdicts (or its entry) is NULL */
extern "C" size_t ZSTDB200_compressFrames_usingCDicts(ZSTD_CCtx* c, void* dst, size_t dstCapacity,
                                                      const void* src, const size_t* frameOffsets, const size_t* frameSizes,
                                                      size_t nbFrames, const ZSTD_CDict* const* cdicts, int level,
                                                      size_t* cSizes, int deviceMemory, void* streamv)
{
    if (!c) return ZB_ERR(ZB_error_GENERIC);
    if (c->advPrefix) return ZB_ERR(ZB_error_parameter_unsupported);
    ZbCall a = { dst, dstCapacity, src, frameOffsets, frameSizes, nbFrames, NULL, level, cSizes, deviceMemory != 0,
                 (cudaStream_t)streamv, c->advChecksum != 0, c->advNoDictID != 0 };
    a.cdicts = cdicts; a.ldm = zb_ldmArg(c);
    return zb_compress(c, a);
}

extern "C" size_t ZSTDB200_compressFramesAsync_usingCDicts(ZSTD_CCtx* c, void* d_dst, size_t dstCapacity, const void* d_src,
                                                           const size_t* frameOffsets, const size_t* frameSizes, size_t nbFrames,
                                                           const ZSTD_CDict* const* cdicts, int level, unsigned long long* d_cSizes,
                                                           unsigned long long* d_result, void* stream)
{
    if (!c || !d_result) return ZB_ERR(ZB_error_GENERIC);
    if (c->advPrefix) return ZB_ERR(ZB_error_parameter_unsupported);
    ZbCall a = { d_dst, dstCapacity, d_src, frameOffsets, frameSizes, nbFrames, NULL, level, NULL, true,
                 (cudaStream_t)stream, c->advChecksum != 0, c->advNoDictID != 0 };
    a.cdicts = cdicts; a.ldm = zb_ldmArg(c); a.result = d_result; a.d_cSizes = d_cSizes;
    return zb_compress(c, a);
}

/* ZSTD_compress_usingDict, ZSTD_compress_usingCDict, ZSTD_compress2: one frame from host buffers (c is not NULL) */
static size_t zb_compressOne(ZSTD_CCtx* c, void* dst, size_t dstCapacity, const void* src, size_t srcSize,
                             const ZSTD_CDict* cdict, int level, bool checksum, bool noDictID, const u32* ldm = nullptr)
{
    if (dstCapacity && !dst) return ZB_ERR(ZB_error_dstBuffer_null);
    if (dstCapacity < 18) return ZB_ERR(ZB_error_dstSize_tooSmall);             /* ZSTD_FRAMEHEADERSIZE_MAX, zstd_compress.c:4643 */
    size_t const off = 0;
    ZbCall a = { dst, dstCapacity, src, &off, &srcSize, 1, cdict, level, NULL, false, NULL, checksum, noDictID };
    a.ldm = ldm;
    return zb_compress(c, a);
}

/* ------------------------------------------------------------------ digested dictionaries (lib/zstd.h:967-995) */
extern "C" ZSTD_CDict* ZSTD_createCDict(const void* dict, size_t dictSize, int level)     /* zstd_compress.c:5633 */
{
    size_t const size = dict ? dictSize : 0;
    ZSTD_CDict* cd = new (std::nothrow) ZSTD_CDict();                          /* value-initialised: every plain member is zero */
    if (!cd) return NULL;
    cd->level = level == 0 ? 3 : level;                                          /* ZSTD_CLEVEL_DEFAULT, :5640 */
    cd->device = -1;
    cd->copy.reset(new (std::nothrow) u8[size]);
    if (cd->copy && size) memcpy(cd->copy.get(), dict, size);
    if (!cd->copy || zb_isErr(zb_digestDict(cd, cd->copy.get(), size))) { delete cd; return NULL; }   /* corrupted entropy tables: creation fails (:5600-5612) */
    return cd;
}

extern "C" size_t ZSTD_freeCDict(ZSTD_CDict* cd) { return zb_deleteOnDevice(cd); }           /* accepts NULL, zstd_compress.c:5655 */

extern "C" unsigned ZSTD_getDictID_fromCDict(const ZSTD_CDict* cd)                           /* zstd_compress.c:5738 */
{
    return (cd && cd->size >= 8 && cd->entropy.present) ? cd->entropy.dictID : 0u;
}

extern "C" unsigned ZSTD_getDictID_fromDict(const void* dict, size_t dictSize)              /* lib/decompress/zstd_ddict.c:227, zstd.h:1105 */
{
    const u8* d = (const u8*)dict;
    if (!d || dictSize < 8) return 0;
    if ((d[0] | (d[1] << 8) | (d[2] << 16) | ((u32)d[3] << 24)) != 0xEC30A437u) return 0;  /* ZSTD_MAGIC_DICTIONARY */
    return d[4] | (d[5] << 8) | (d[6] << 16) | ((u32)d[7] << 24);
}

extern "C" size_t ZSTD_compress_usingCDict(ZSTD_CCtx* c, void* dst, size_t dstCapacity, const void* src, size_t srcSize,
                                           const ZSTD_CDict* cdict)                          /* zstd_compress.c:5836 */
{
    if (!c) return ZB_ERR(ZB_error_GENERIC);
    if (!cdict) return ZB_ERR(ZB_error_dictionary_wrong);
    return zb_compressOne(c, dst, dstCapacity, src, srcSize, cdict, cdict->level, false, false);
}

/* One rank's share of a frame that several GPUs compress together (SURVEY.md 8e; the reference's counterpart are the jobs
 * of ZSTDMT, zstdmt_compress.c:1168-1227: a job reads an overlap of preceding input and only the first writes the frame
 * header, only the last the end mark).  Chunks are the unit: partBegin must be a multiple of ZSTDB200_framePartAlignment()
 * (512 KiB), and the bytes [partBegin - ZSTDB200_framePartHalo(), partBegin + partSize) of the frame must be resident:
 * d_part points at frame offset partBegin - min(partBegin, halo).  The ranks' outputs, concatenated in order, are byte
 * for byte the frame one GPU would have produced. */
extern "C" size_t ZSTDB200_framePartAlignment(void) { return (size_t)ZB_CHUNK_BLOCKS * ZB_BLOCK_MAX; }
extern "C" size_t ZSTDB200_framePartHalo(void) { return ZB_PRIME_BYTES; }
extern "C" size_t ZSTDB200_compressFramePart(ZSTD_CCtx* c, void* d_dst, size_t dstCapacity, const void* d_part,
                                             size_t frameSize, size_t partBegin, size_t partSize, int level, void* stream)
{
    if (!c) return ZB_ERR(ZB_error_GENERIC);
    if (partBegin % ZSTDB200_framePartAlignment() || partBegin + partSize > frameSize || (partSize == 0 && frameSize != 0)) return ZB_ERR(ZB_error_srcSize_wrong);
    if (c->advChecksum) return ZB_ERR(ZB_error_parameter_unsupported);          /* a content checksum needs the whole content in one place */
    if (c->advLdm || c->advPrefix) return ZB_ERR(ZB_error_parameter_unsupported);   /* a rank holds a halo of 128 KiB, not the LDM window or a prefix */
    size_t const halo = partBegin < ZB_PRIME_BYTES ? partBegin : ZB_PRIME_BYTES;
    const u8* const frameBase = (const u8*)d_part + halo - partBegin;          /* address frame offset 0 would have; only offsets >= partBegin - halo are touched */
    size_t const off = 0;
    ZbCall const a = { d_dst, dstCapacity, frameBase, &off, &frameSize, 1, NULL, level, NULL, true, (cudaStream_t)stream,
                       false, c->advNoDictID != 0, partBegin, frameSize ? partBegin + partSize : 1 };   /* an empty frame: its one empty block */
    return zb_compress(c, a);
}

extern "C" size_t ZSTDB200_compressDevice(ZSTD_CCtx* c, void* d_dst, size_t dstCapacity,
                                          const void* d_src, size_t srcSize, int level, void* stream)
{
    size_t const off = 0;
    if (c && c->advPrefix) return zb_compressWithPrefix(c, d_dst, dstCapacity, d_src, srcSize, level, true, (cudaStream_t)stream);
    return ZSTDB200_compressFrames(c, d_dst, dstCapacity, d_src, &off, &srcSize, 1, NULL, 0, NULL, level, 1, stream);
}

/* Stream-ordered calls: the bytes of ZSTDB200_compressDevice / ZSTDB200_compressFrames[_usingCDict] on device buffers, with
 * the verdict left in device memory.  The single-frame call honours the sticky dictionary as ZSTD_compress2 does (a
 * referenced CDict brings its level) and a device prefix; a host prefix is forgotten and refused, as a host-buffer call
 * refuses a device prefix. */
extern "C" size_t ZSTDB200_compressDeviceAsync(ZSTD_CCtx* c, void* d_dst, size_t dstCapacity, const void* d_src, size_t srcSize,
                                               int level, unsigned long long* d_result, void* stream)
{
    if (!c || !d_result) return ZB_ERR(ZB_error_GENERIC);
    if (c->advPrefix && !c->advPrefixOnDevice) { c->advPrefix = NULL; c->advPrefixSize = 0; return ZB_ERR(ZB_error_parameter_unsupported); }
    if (c->advPrefix) return zb_compressWithPrefix(c, d_dst, dstCapacity, d_src, srcSize, level, true, (cudaStream_t)stream, d_result);
    const ZSTD_CDict* const cd = c->advRefCDict ? c->advRefCDict : c->advLocalDict.get();
    size_t const off = 0;
    ZbCall a = { d_dst, dstCapacity, d_src, &off, &srcSize, 1, cd, c->advRefCDict ? c->advRefCDict->level : level, NULL, true,
                 (cudaStream_t)stream, c->advChecksum != 0, c->advNoDictID != 0 };
    a.ldm = zb_ldmArg(c); a.result = d_result;
    return zb_compress(c, a);
}

extern "C" size_t ZSTDB200_compressFramesAsync(ZSTD_CCtx* c, void* d_dst, size_t dstCapacity, const void* d_src,
                                               const size_t* frameOffsets, const size_t* frameSizes, size_t nbFrames,
                                               const ZSTD_CDict* cdict, int level, unsigned long long* d_cSizes,
                                               unsigned long long* d_result, void* stream)
{
    if (!c || !d_result) return ZB_ERR(ZB_error_GENERIC);
    if (c->advPrefix) return ZB_ERR(ZB_error_parameter_unsupported);
    ZbCall a = { d_dst, dstCapacity, d_src, frameOffsets, frameSizes, nbFrames, cdict, cdict ? cdict->level : level, NULL, true,
                 (cudaStream_t)stream, c->advChecksum != 0, c->advNoDictID != 0 };
    a.ldm = zb_ldmArg(c); a.result = d_result; a.d_cSizes = d_cSizes;
    return zb_compress(c, a);
}

/* Seek table of a run of frames, in the reference's seekable format (contrib/seekable_format/
 * zstd_seekable_compression_format.md; writer: zstdseek_compress.c:268-360): a skippable frame holding one
 * (compressed size, decompressed size) pair per frame and the 9-byte footer.  Appended behind the frames a batch or a
 * multi-GPU call produced, it makes the output randomly accessible for the reference's ZSTD_seekable_* readers.  Host
 * code, no GPU.  Returns the number of bytes written (17 + 8 * nbFrames) or an error code. */
extern "C" size_t ZSTDB200_writeSeekTable(void* dstv, size_t dstCapacity, const size_t* cSizes, const size_t* dSizes, size_t nbFrames)
{
    u8* const dst = (u8*)dstv;
    if (nbFrames > 0x8000000u) return ZB_ERR(ZB_error_srcSize_wrong);                         /* ZSTD_SEEKABLE_MAXFRAMES, zstd_seekable.h:20 */
    size_t const need = 8 + 8 * nbFrames + 9;
    if (!dst || (nbFrames && (!cSizes || !dSizes))) return ZB_ERR(ZB_error_GENERIC);
    if (dstCapacity < need) return ZB_ERR(ZB_error_dstSize_tooSmall);
    auto w32 = [](u8* p, u32 v) { p[0] = (u8)v; p[1] = (u8)(v >> 8); p[2] = (u8)(v >> 16); p[3] = (u8)(v >> 24); };
    for (size_t f = 0; f < nbFrames; f++)                           /* 32-bit fields; ZSTD_SEEKABLE_MAX_FRAME_DECOMPRESSED_SIZE = 1 GiB (zstd_seekable.h:19) */
        if (cSizes[f] > 0xFFFFFFFFull || dSizes[f] > 0x40000000ull) return ZB_ERR(ZB_error_srcSize_wrong);
    w32(dst, 0x184D2A5Eu);                                                                     /* Skippable_Magic_Number */
    w32(dst + 4, (u32)(need - 8));                                                             /* Frame_Size */
    u8* p = dst + 8;
    for (size_t f = 0; f < nbFrames; f++) { w32(p, (u32)cSizes[f]); w32(p + 4, (u32)dSizes[f]); p += 8; }
    w32(p, (u32)nbFrames); p[4] = 0;                                                           /* Number_Of_Frames, descriptor: no checksums */
    w32(p + 5, 0x8F92EAB1u);                                                                   /* Seekable_Magic_Number */
    return need;
}

/* the frame checksum's hash, exported for the CPU tests (compared with the reference's ZSTD_XXH64) */
extern "C" unsigned long long ZSTDB200_xxh64(const void* p, size_t len) { return zb_xxh64((const u8*)p, len); }

/* Host-side planning of one call, without touching a GPU (what the CPU tests compare with the oracle's plan).
 * Per frame, `out` receives 16 values: strategy, mls, tableN, tableNLong, stepSize, litDisabled, windowLog, insStep,
 * number of blocks, size of the first block, flags of the first block, history of the last block, dictionary part of
 * the first block's history, number of chunks, history walked by the last chunk, size of the last chunk.
 * Returns the total number of blocks. */
extern "C" size_t ZSTDB200_describePlan(const size_t* frameSizes, size_t nbFrames, int level, size_t dictSize, size_t dictTail, unsigned* out)
{
    std::vector<size_t> offs(nbFrames);
    size_t o = 0; for (size_t f = 0; f < nbFrames; f++) { offs[f] = o; o += frameSizes[f]; }
    ZSTD_CDict d;                                                     /* a raw-content dictionary of that size and tail, never on a device */
    d.level = level; d.content = NULL; d.contentOnDevice = false; d.size = dictSize; d.contentOff = 0; d.tail = dictTail;
    memset(&d.entropy, 0, sizeof(d.entropy)); d.device = -1; d.resident = false; d.nbImages = 0;
    ZbCall const a = { NULL, 0, NULL, offs.data(), frameSizes, nbFrames, dictSize ? &d : NULL, level };
    ZbPlan P;
    zb_plan(P, a);
    for (size_t f = 0; f < nbFrames && out; f++) {
        ZbFrame const& fr = P.frames[f];
        const ZbParams* prm = NULL;
        for (size_t g = 0; g < P.groups.size(); g++) if (P.groups[g].b0 <= fr.firstBlock && fr.firstBlock < P.groups[g].b1) prm = &P.groups[g].prm;
        ZbBlock const& b0 = P.blocks[fr.firstBlock]; ZbBlock const& bl = P.blocks[fr.firstBlock + fr.nbBlocks - 1];
        u32 nc = 0; const ZbChunk* lastChunk = NULL;
        for (size_t ci = 0; ci < P.chunks.size(); ci++) if (P.chunks[ci].firstBlock >= fr.firstBlock && P.chunks[ci].firstBlock < fr.firstBlock + fr.nbBlocks) { nc++; lastChunk = &P.chunks[ci]; }
        unsigned* r = out + f * 16;
        r[0] = prm->strategy; r[1] = prm->mls; r[2] = prm->tableN; r[3] = prm->tableNLong; r[4] = prm->stepSize; r[5] = prm->litDisabled;
        r[6] = fr.windowLog; r[7] = prm->insStep; r[8] = fr.nbBlocks; r[9] = b0.size; r[10] = b0.flags;
        r[11] = bl.histLen; r[12] = b0.dictLen; r[13] = nc; r[14] = lastChunk ? lastChunk->histLen : 0; r[15] = lastChunk ? lastChunk->size : 0;
    }
    return P.blocks.size();
}

extern "C" void ZSTDB200_getLastStats(const ZSTD_CCtx* c, ZSTDB200_stats* out) { if (c && out) *out = c->stats; }


/* ------------------------------------------------------------------ advanced one-shot API (lib/zstd.h:337-603, :1088-1102)
 * ZSTD_CCtx_setParameter + ZSTD_compress2 is how python-zstandard, zstd-jni and the zstd CLI drive the library today.
 * Supported: compressionLevel, checksumFlag (XXH64 of the content on the host), contentSizeFlag (always written),
 * dictIDFlag, nbWorkers / jobSize / overlapLog (accepted and ignored: parallelism is the GPU's), the cParams only at
 * their default 0; everything else answers parameter_unsupported.  ZSTD_compressStream2 serves the one-shot form
 * (first call, ZSTD_e_end, output room >= ZSTD_compressBound: lib/zstd.h:787) — real streaming is out of scope. */
extern "C" size_t ZSTD_CCtx_setParameter(ZSTD_CCtx* c, ZSTD_cParameter paramE, int value)                 /* zstd_compress.c:720 */
{
    if (!c) return ZB_ERR(ZB_error_GENERIC);
    int const param = (int)paramE;
    switch (param) {
    case 100: c->advLevel = value == 0 ? 3 : (value > 22 ? 22 : (value < -(int)ZB_BLOCK_MAX ? -(int)ZB_BLOCK_MAX : value)); return 0;   /* ZSTD_c_compressionLevel */
    case 200: return 0;                                                                      /* ZSTD_c_contentSizeFlag: the size is always written */
    case 201: c->advChecksum = value != 0; return 0;                                         /* ZSTD_c_checksumFlag */
    case 202: c->advNoDictID = value == 0; return 0;                                         /* ZSTD_c_dictIDFlag */
    case 400: case 401: case 402: return 0;                                                  /* nbWorkers, jobSize, overlapLog */
    case 1008: if (value != 0 && value != 1) return ZB_ERR(ZB_error_parameter_unsupported);  /* ZSTD_c_blockDelimiters */
        c->advDelims = value; return 0;
    case 1009: return (value == 0 || value == 1) ? 0 : ZB_ERR(ZB_error_parameter_unsupported);   /* ZSTD_c_validateSequences: validation always runs */
    case 101: case 102: case 103: case 104: case 105: case 106: case 107:                    /* windowLog .. strategy: default only */
        return value == 0 ? 0 : ZB_ERR(ZB_error_parameter_unsupported);
    case 160:                                                                                /* ZSTD_c_enableLongDistanceMatching: ZSTD_paramSwitch_e */
        if (value < 0 || value > 2) return ZB_ERR(ZB_error_parameter_outOfBound);
        c->advLdm = value == 1; return 0;                                                    /* auto: off (no level here is btopt or stronger, zstd_compress.c:277) */
    case 161: case 162: case 163: case 164: {                                                /* ldmHashLog, ldmMinMatch, ldmBucketSizeLog, ldmHashRateLog */
        static const int lo[4] = { 6, 4, 1, 0 }, hi[4] = { 30, 4096, 8, 25 };               /* lib/zstd.h:1267-1274; 0 = derived */
        int const i = param - 161;
        if (value != 0 && (value < lo[i] || value > hi[i])) return ZB_ERR(ZB_error_parameter_outOfBound);
        c->advLdmPrm[i] = (u32)value; return 0;
    }
    default: return ZB_ERR(ZB_error_parameter_unsupported);
    }
}

extern "C" size_t ZSTD_CCtx_setPledgedSrcSize(ZSTD_CCtx* c, unsigned long long) { return c ? 0 : ZB_ERR(ZB_error_GENERIC); }   /* one-shot calls know their size */

extern "C" size_t ZSTD_CCtx_reset(ZSTD_CCtx* c, ZSTD_ResetDirective reset)                                   /* zstd_compress.c:1390; 1 session, 2 parameters, 3 both */
{
    if (!c) return ZB_ERR(ZB_error_GENERIC);
    if (reset == 1 || reset == 3) { c->stInSize = 0; c->stOutSize = 0; c->stOutPos = 0; c->stFrames = 0; }   /* an unfinished stream is dropped */
    if (reset == 2 || reset == 3) {
        c->advLevel = 3; c->advChecksum = 0; c->advNoDictID = 0; c->advDelims = 0; c->advLdm = 0; memset(c->advLdmPrm, 0, sizeof(c->advLdmPrm));
        c->advLocalDict.reset(); c->advRefCDict = NULL; c->advPrefix = NULL; c->advPrefixSize = 0;   /* ZSTD_clearAllDicts, zstd_compress.c:1360 */
    }
    return 0;
}

extern "C" size_t ZSTD_CCtx_loadDictionary(ZSTD_CCtx* c, const void* dict, size_t dictSize)  /* zstd_compress.c:1260: copied, sticky */
{
    if (!c) return ZB_ERR(ZB_error_GENERIC);
    c->advLocalDict.reset(); c->advRefCDict = NULL; c->advPrefix = NULL; c->advPrefixSize = 0;
    if (!dict || dictSize == 0) return 0;                                                    /* NULL / 0: back to no dictionary */
    c->advLocalDict.reset(ZSTD_createCDict(dict, dictSize, c->advLevel));
    return c->advLocalDict ? 0 : ZB_ERR(ZB_error_dictionary_corrupted);
}

extern "C" size_t ZSTD_CCtx_refCDict(ZSTD_CCtx* c, const ZSTD_CDict* cdict)                  /* zstd_compress.c:1330: borrowed, sticky */
{
    if (!c) return ZB_ERR(ZB_error_GENERIC);
    c->advLocalDict.reset(); c->advPrefix = NULL; c->advPrefixSize = 0;
    c->advRefCDict = cdict;
    return 0;
}

/* zstd_compress.c:1339-1356: borrowed raw content for the next frame only; it takes the place of any dictionary, and NULL / 0
 * leaves the context without either.  Refused inside an unfinished stream. */
static size_t zb_refPrefix(ZSTD_CCtx* c, const void* prefix, size_t prefixSize, bool onDevice)
{
    if (!c) return ZB_ERR(ZB_error_GENERIC);
    if (c->stInSize || c->stOutSize || c->stFrames) return ZB_ERR(ZB_error_stage_wrong);
    c->advLocalDict.reset(); c->advRefCDict = NULL;
    bool const some = prefix && prefixSize;
    c->advPrefix = some ? (const u8*)prefix : NULL; c->advPrefixSize = some ? prefixSize : 0; c->advPrefixOnDevice = onDevice;
    return 0;
}
extern "C" size_t ZSTD_CCtx_refPrefix(ZSTD_CCtx* c, const void* prefix, size_t prefixSize) { return zb_refPrefix(c, prefix, prefixSize, false); }
extern "C" size_t ZSTDB200_CCtx_refPrefixDevice(ZSTD_CCtx* c, const void* d_prefix, size_t prefixSize) { return zb_refPrefix(c, d_prefix, prefixSize, true); }

extern "C" size_t ZSTD_compress2(ZSTD_CCtx* c, void* dst, size_t dstCapacity, const void* src, size_t srcSize)     /* zstd_compress.c:6365 */
{
    if (!c) return ZB_ERR(ZB_error_GENERIC);
    if (c->advPrefix) return zb_compressWithPrefix(c, dst, dstCapacity, src, srcSize, c->advLevel, false, NULL);
    const ZSTD_CDict* const cd = c->advRefCDict ? c->advRefCDict : c->advLocalDict.get();
    int const level = c->advRefCDict ? c->advRefCDict->level : c->advLevel;                  /* a referenced CDict brings its own level (:5836) */
    return zb_compressOne(c, dst, dstCapacity, src, srcSize, cd, level, c->advChecksum != 0, c->advNoDictID != 0, zb_ldmArg(c));
}

/* ------------------------------------------------------------------ sequence calls (lib/zstd.h:1555-1644)
 * K1s (zb_seqimport.cu) takes the place of K1: the sequences are partitioned and validated on the device, every block's
 * share is clipped to it and coded; K2 / K3 / K4 run unchanged.  One stream; more than devWaveBlocks blocks run in waves
 * over the block table, in order, through one workspace slot. */
extern "C" size_t ZSTD_sequenceBound(size_t srcSize)                                    /* zstd_compress.c:3456-3460 */
{
    return (srcSize / 3) + 1 + (srcSize / 1024) + 1;                                     /* ZSTD_MINMATCH_MIN, ZSTD_BLOCKSIZE_MAX_MIN */
}

extern "C" size_t ZSTD_mergeBlockDelimiters(ZSTD_Sequence* seqs, size_t n)               /* zstd_compress.c:3497-3511 */
{
    size_t out = 0;
    for (size_t in = 0; in < n; in++) {
        if (seqs[in].offset == 0 && seqs[in].matchLength == 0) { if (in != n - 1) seqs[in + 1].litLength += seqs[in].litLength; }
        else seqs[out++] = seqs[in];
    }
    return out;
}

static size_t zb_compressSeqs(ZSTD_CCtx* c, void* dst, size_t dstCapacity, const ZSTD_Sequence* seqs, size_t n,
                              const void* src, size_t srcSize, bool deviceMemory, cudaStream_t userStream)
{
    if (!c) return ZB_ERR(ZB_error_GENERIC);
    if (c->advPrefix) return ZB_ERR(ZB_error_parameter_unsupported);           /* the caller's sequences cannot reach into a prefix */
    if (dstCapacity && !dst) return ZB_ERR(ZB_error_dstBuffer_null);
    if (n && !seqs) return ZB_ERR(ZB_error_externalSequences_invalid);
    if (n > 0xFFFFFFF0u) return ZB_ERR(ZB_error_srcSize_wrong);
    ZbDeviceGuard guard;
    TRY(zb_ctxInit(c));
    memset(&c->stats, 0, sizeof(c->stats));
    CK(c->order.hostWait());                                      /* stream-ordered calls still queued use the buffers sized below */
    const ZSTD_CDict* const cdArg = c->advRefCDict ? c->advRefCDict : c->advLocalDict.get();
    int const level = c->advRefCDict ? c->advRefCDict->level : c->advLevel;
    ZSTD_CDict* const cd = zb_usable(cdArg);
    if (g_strictLevels && level > 4) return ZB_ERR(ZB_error_parameter_unsupported);
    bool const expl = c->advDelims != 0;
    cudaStream_t const st = (deviceMemory && userStream) ? userStream : c->stream;
    const ZbDictEntropy* const de = (cd && cd->entropy.present) ? &cd->entropy : NULL;
    ZbCParams const cp = zb_getCParams(level, srcSize, cd ? cd->size : 0);
    ZbParams prm = zb_makeParams(cp);
    /* the dictionary: made resident by the executor's own step, a one-entry table (no images: K1 does not run) */
    ZbPlan& P = c->plan;
    P.reset();
    if (cd) {
        P.prms.push_back(prm);
        zb_dictSlot(P, cd, 0);
        ZbCall const none = { NULL, 0, NULL, NULL, NULL, 0, NULL, level };
        ZbRun r{c, none, P, ZbWaves{}, st};
        TRY(r.prepareDicts());
        TRY(c->d_dicts.ensure(1));
        CK(cudaMemcpyAsync(c->d_dicts, P.dicts.data(), sizeof(ZbDictSlot), cudaMemcpyHostToDevice, st));
    }
    const ZbDictSlot* const d_dicts = cd ? c->d_dicts.p : NULL;
    u32 const blockMax = (1u << cp.windowLog) < ZB_BLOCK_MAX ? (1u << cp.windowLog) : ZB_BLOCK_MAX;      /* zstd_compress.c:2124 */
    u32 const dictFlag = (cd && cd->tail) ? ZB_FLAG_DICT : 0u;
    /* inputs on the device: the sequences need 16-byte alignment for the tile loads */
    const u8* d_src = (const u8*)src; const void* d_seqs = seqs;
    size_t const seqBytes = n * sizeof(ZSTD_Sequence);
    if (!deviceMemory) {
        TRY(c->d_in.ensure(srcSize + 16));
        if (srcSize) CK(cudaMemcpyAsync(c->d_in, src, srcSize, cudaMemcpyHostToDevice, st));
        d_src = c->d_in;
    }
    if (n && (!deviceMemory || ((uintptr_t)seqs & 15u))) {
        TRY(c->d_seqIn.ensure(n));
        CK(cudaMemcpyAsync(c->d_seqIn, seqs, seqBytes, deviceMemory ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, st));
        d_seqs = c->d_seqIn;
    }
    TRY(c->d_seqCtrl.ensure(4));
    u64 ctrl[4] = { 0, 0, ~0ull, 0 };
    CK(cudaMemcpyAsync(c->d_seqCtrl, ctrl, sizeof(ctrl), cudaMemcpyHostToDevice, st));
    CK(cudaStreamSynchronize(st));                                 /* the pageable sources above are staged */
    CK(cudaEventRecord(c->ev[EV_K0], st));
    /* K1s-a */
    u32 const nbTiles = (u32)((n + 1023) / 1024);
    TRY(c->d_seqTile.ensure((size_t)nbTiles * 12 + 16));
    u64* const d_tileLen = (u64*)c->d_seqTile.p; u32* const d_tileEnds = (u32*)(d_tileLen + nbTiles);
    CK(zb_launch_seq_partition(d_seqs, (u32)n, expl, d_tileLen, d_tileEnds, c->d_seqCtrl, st));
    u32 nbBlocks;
    if (srcSize == 0) nbBlocks = 1;                                /* the frame's one empty block */
    else if (!expl) nbBlocks = (u32)((srcSize + blockMax - 1) / blockMax);
    else {
        CK(cudaMemcpyAsync(ctrl, c->d_seqCtrl, 2 * sizeof(u64), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        if (ctrl[0] > srcSize || ctrl[1] == 0) return ZB_ERR(ZB_error_externalSequences_invalid);
        nbBlocks = (u32)ctrl[1];
    }
    TRY(zb_ensureDesc(c, nbBlocks, 1, 1, 0));
    size_t const blkBytes = (size_t)nbBlocks * 24 + 16;              /* blockFirstPos / blockEnd (u64), blockFirst / blockSeq (u32) */
    TRY(c->d_seqBlk.ensure(blkBytes));
    u64* const d_firstPos = (u64*)c->d_seqBlk.p; u64* const d_blockEnd = d_firstPos + nbBlocks;
    u32* const d_first = (u32*)(d_blockEnd + nbBlocks); u32* const d_blockSeq = d_first + nbBlocks;
    if (!expl || srcSize == 0) {                                    /* the planner's geometry */
        ZbVec<ZbBlock>& B = P.blocks;
        B.clear(); B.reserve(nbBlocks);
        for (u32 k = 0; k < nbBlocks; k++) {
            ZbBlock b; memset(&b, 0, sizeof(b));
            b.srcOff = (u64)k * blockMax; b.size = (u32)(srcSize - b.srcOff < blockMax ? srcSize - b.srcOff : blockMax);
            b.flags = (k == 0 ? ZB_FLAG_FIRST | dictFlag : 0u) | (k + 1 == nbBlocks ? ZB_FLAG_LAST : 0u);
            B.push_back(b);
        }
        CK(cudaMemcpyAsync(c->d_blocks, B.data(), nbBlocks * sizeof(ZbBlock), cudaMemcpyHostToDevice, st));
        CK(cudaMemsetAsync(d_first, 0xFF, nbBlocks * sizeof(u32), st));
    }
    u64 const dictContent = cd ? cd->size - cd->contentOff : 0;
    CK(zb_launch_seq_place(d_seqs, (u32)n, expl, d_tileLen, d_tileEnds, srcSize, 1ull << cp.windowLog, dictContent, blockMax,
                           nbBlocks, d_blockEnd, d_blockSeq, d_first, d_firstPos, c->d_seqCtrl, st));
    if (expl && srcSize) CK(zb_launch_seq_blocks(d_blockEnd, d_blockSeq, nbBlocks, blockMax, dictFlag, c->d_blocks, d_first, d_firstPos, c->d_seqCtrl, st));
    CK(cudaMemcpyAsync(ctrl, c->d_seqCtrl, sizeof(ctrl), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (ctrl[2] != ~0ull || ctrl[0] > srcSize || (expl && srcSize && ctrl[3] != srcSize)) return ZB_ERR(ZB_error_externalSequences_invalid);
    ZbFrame fr; memset(&fr, 0, sizeof(fr));
    fr.srcSize = srcSize; fr.nbBlocks = nbBlocks; fr.windowLog = cp.windowLog;
    fr.dictID = (c->advNoDictID || !de) ? 0u : de->dictID; fr.checksum = c->advChecksum != 0;
    CK(cudaMemcpyAsync(c->d_frames, &fr, sizeof(fr), cudaMemcpyHostToDevice, st));
    /* K1s-b, K2, K3, K4 in waves through one workspace slot */
    ZbStrides const sd = zb_seq_strides(blockMax);
    u32 const waveBlocks = (c->devWaveBlocks && nbBlocks > c->devWaveBlocks) ? c->devWaveBlocks : nbBlocks;
    u32 const nbWaves = (nbBlocks + waveBlocks - 1) / waveBlocks;
    TRY(zb_ensureDesc(c, nbBlocks, 1, nbWaves, 0));
    ZbWorkRows work;
    {   size_t const bytes = zb_workLayout(NULL, waveBlocks, ZB_WORK_SEQUENCES, sd, NULL);
        TRY(bytes); TRY(c->d_work.ensure(bytes));
        zb_workLayout(c->d_work, waveBlocks, ZB_WORK_SEQUENCES, sd, &work); }
    u8* d_out = (u8*)dst; size_t outCap = dstCapacity;
    if (!deviceMemory) {
        size_t const bound = srcSize + 3 * (size_t)nbBlocks + 64;      /* every block at most raw: 3 header bytes each, blocks may be tiny */
        outCap = dstCapacity < bound ? dstCapacity : bound;
        TRY(c->d_out.ensure(outCap + 16));
        d_out = c->d_out;
    }
    bool const timed = nbWaves == 1;
    unsigned launches = 2 + (n ? 2u : 0u) + (expl && srcSize ? 1u : 0u);
    for (u32 w = 0; w < nbWaves; w++) {
        u32 const b0 = w * waveBlocks, nb = (b0 + waveBlocks <= nbBlocks) ? waveBlocks : nbBlocks - b0;
        CK(zb_launch_seq_convert(d_src, c->d_blocks + b0, nb, d_first + b0, d_firstPos + b0, d_seqs, (u32)n, d_dicts, &work, st));
        if (w == 0) CK(cudaEventRecord(c->ev[EV_K1], st));
        CK(zb_launch_literals(c->d_blocks + b0, nb, &prm, &sd, NULL, work.lits, work.body, work.meta, st, d_dicts));
        if (timed) CK(cudaEventRecord(c->ev[EV_K2], st));
        CK(zb_launch_sequences(d_src, c->d_blocks + b0, nb, &prm, &sd, NULL, work.seqs, work.dist, work.body, work.meta, st, d_dicts));
        if (timed) CK(cudaEventRecord(c->ev[EV_K3], st));
        CK(zb_launch_stitch(d_src, c->d_blocks + b0, nb, c->d_frames, &work, c->d_outOffsets + b0,
                            w > 0 ? c->d_totals + (w - 1) : NULL, c->d_totals + w, d_out, outCap, st));
        launches += 5;
    }
    if (c->advChecksum) { CK(zb_launch_checksums(d_src, c->d_frames, 1, c->d_outOffsets, d_out, outCap, st)); launches++; }
    CK(cudaEventRecord(c->ev[EV_KEND], st));
    u64 total = 0;
    CK(cudaMemcpyAsync(&total, c->d_totals + nbWaves - 1, sizeof(u64), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (!deviceMemory && total <= dstCapacity) CK(cudaMemcpy(dst, d_out, total, cudaMemcpyDeviceToHost));
    float ms = 0;
    cudaEventElapsedTime(&ms, c->ev[EV_K0], c->ev[EV_KEND]); c->stats.kernel_ms = ms; c->stats.total_ms = ms;
    cudaEventElapsedTime(&ms, c->ev[EV_K0], c->ev[EV_K1]); c->stats.match_ms = ms;     /* the first wave's import */
    if (timed) {
        cudaEventElapsedTime(&ms, c->ev[EV_K1], c->ev[EV_K2]); c->stats.literals_ms = ms;
        cudaEventElapsedTime(&ms, c->ev[EV_K2], c->ev[EV_K3]); c->stats.sequences_ms = ms;
        cudaEventElapsedTime(&ms, c->ev[EV_K3], c->ev[EV_KEND]); c->stats.stitch_ms = ms;
    }
    c->stats.launches = launches; c->stats.nbBlocks = nbBlocks;
    if (!deviceMemory) { c->stats.h2d_bytes = srcSize + seqBytes; c->stats.d2h_bytes = total <= dstCapacity ? (size_t)total : 0; }
    if (total > dstCapacity) return ZB_ERR(ZB_error_dstSize_tooSmall);
    return (size_t)total;
}

extern "C" size_t ZSTD_compressSequences(ZSTD_CCtx* c, void* dst, size_t dstCapacity, const ZSTD_Sequence* seqs, size_t n,
                                         const void* src, size_t srcSize)                       /* zstd_compress.c:6858 */
{
    return zb_compressSeqs(c, dst, dstCapacity, seqs, n, src, srcSize, false, NULL);
}

/* ZSTD_generateSequences (lib/zstd.h:1594) and its device forms: the parse of the frame ZSTD_compress2 writes for src on this
 * context (sticky level, dictionary or CDict, block boundaries), run through the executor with the export as every wave's
 * tail.  d_result: a stream-ordered call's verdict (NULL: synchronous). */
static size_t zb_generateSeqs(ZSTD_CCtx* c, ZSTD_Sequence* out, size_t outCapacity, const void* src, size_t srcSize, bool deviceMemory,
                              cudaStream_t stream, unsigned long long* d_result)
{
    if (outCapacity && !out) return ZB_ERR(ZB_error_dstBuffer_null);
    if (deviceMemory && ((uintptr_t)out & 3u)) return ZB_ERR(ZB_error_parameter_outOfBound);    /* ZSTD_Sequence's alignment */
    if (c->advLdm || c->advPrefix) return ZB_ERR(ZB_error_parameter_unsupported);   /* not exported yet; the prefix stays pending */
    const ZSTD_CDict* const cd = c->advRefCDict ? c->advRefCDict : c->advLocalDict.get();
    size_t const off = 0;
    ZbCall a = { out, outCapacity, src, &off, &srcSize, 1, cd, c->advRefCDict ? c->advRefCDict->level : c->advLevel, NULL, deviceMemory,
                 stream, false, false };                          /* the frame header's flags do not change the parse */
    a.result = d_result; a.sequences = true;
    return zb_compress(c, a);
}

extern "C" size_t ZSTD_generateSequences(ZSTD_CCtx* c, ZSTD_Sequence* outSeqs, size_t outSeqsSize, const void* src, size_t srcSize)
{
    if (!c) return ZB_ERR(ZB_error_GENERIC);
    return zb_generateSeqs(c, outSeqs, outSeqsSize, src, srcSize, false, NULL, NULL);
}

extern "C" size_t ZSTDB200_generateSequencesDevice(ZSTD_CCtx* c, ZSTD_Sequence* d_outSeqs, size_t outSeqsCapacity, const void* d_src,
                                                   size_t srcSize, void* stream)
{
    if (!c) return ZB_ERR(ZB_error_GENERIC);
    return zb_generateSeqs(c, d_outSeqs, outSeqsCapacity, d_src, srcSize, true, (cudaStream_t)stream, NULL);
}

extern "C" size_t ZSTDB200_generateSequencesDeviceAsync(ZSTD_CCtx* c, ZSTD_Sequence* d_outSeqs, size_t outSeqsCapacity, const void* d_src,
                                                        size_t srcSize, unsigned long long* d_result, void* stream)
{
    if (!c || !d_result) return ZB_ERR(ZB_error_GENERIC);
    return zb_generateSeqs(c, d_outSeqs, outSeqsCapacity, d_src, srcSize, true, (cudaStream_t)stream, d_result);
}

extern "C" size_t ZSTDB200_compressSequencesDevice(ZSTD_CCtx* c, void* d_dst, size_t dstCapacity, const ZSTD_Sequence* d_seqs, size_t n,
                                                   const void* d_src, size_t srcSize, void* stream)
{
    return zb_compressSeqs(c, d_dst, dstCapacity, d_seqs, n, d_src, srcSize, true, (cudaStream_t)stream);
}

/* Streaming (lib/zstd.h:681-862).  The unit of GPU work is a whole frame, so the stream front end collects input on the
 * host and turns it into frames:
 *   ZSTD_e_continue  input is taken into the context's buffer; whenever ZB_STREAM_FRAME bytes are there they become a frame;
 *   ZSTD_e_flush     what is buffered becomes a frame now (the reference ends a block, here a frame ends: every byte given
 *                    so far is decodable from the output, which is what a flush promises);
 *   ZSTD_e_end       same, and the session is over once everything was handed out (an empty session yields an empty frame).
 * The result is a sequence of frames — a valid zstd stream that every decoder reads as the concatenation of their contents
 * (lib/zstd.h:160-162; contrib/pzstd writes the same shape) — not one frame as the reference's stream would be.
 * The first call of a session carrying everything with ZSTD_e_end and room for ZSTD_compressBound() bytes is served without
 * any buffering (the one-shot form, lib/zstd.h:787).  Return value: bytes still waiting to be handed out (0 = flushed). */
#define ZB_STREAM_FRAME ((size_t)256 << 20)
static size_t zb_streamHandOut(ZSTD_CCtx* c, ZSTD_outBuffer* out)
{
    size_t const have = c->stOutSize - c->stOutPos, room = out->size - out->pos;
    size_t const n = have < room ? have : room;
    if (n) { memcpy((u8*)out->dst + out->pos, c->stOut + c->stOutPos, n); out->pos += n; c->stOutPos += n; }
    if (c->stOutPos == c->stOutSize) { c->stOutPos = 0; c->stOutSize = 0; }
    return c->stOutSize - c->stOutPos;
}
static size_t zb_streamMakeFrame(ZSTD_CCtx* c)                        /* stIn -> one frame appended to stOut */
{
    size_t const bound = ZSTD_compressBound(c->stInSize) + 32;
    if (c->stOutSize + bound > c->stOutCap) {
        size_t const cap = c->stOutSize + bound;
        u8* const p = (u8*)realloc(c->stOut, cap);
        if (!p) return ZB_ERR(ZB_error_memory_allocation);
        c->stOut = p; c->stOutCap = cap;
    }
    size_t const r = ZSTD_compress2(c, c->stOut + c->stOutSize, bound, c->stIn ? c->stIn : (const u8*)"", c->stInSize);
    if (ZSTD_isError(r)) return r;
    c->stOutSize += r; c->stInSize = 0; c->stFrames++;
    return 0;
}
extern "C" size_t ZSTD_compressStream2(ZSTD_CCtx* c, ZSTD_outBuffer* out, ZSTD_inBuffer* in, ZSTD_EndDirective endOp)       /* zstd_compress.c:6176 */
{
    if (!c || !out || !in) return ZB_ERR(ZB_error_GENERIC);
    if (out->pos > out->size) return ZB_ERR(ZB_error_dstSize_tooSmall);
    if (in->pos > in->size) return ZB_ERR(ZB_error_srcSize_wrong);
    if ((int)endOp < 0 || (int)endOp > 2) return ZB_ERR(ZB_error_parameter_unsupported);
    size_t const n = in->size - in->pos, room = out->size - out->pos;
    bool const idle = c->stInSize == 0 && c->stOutSize == 0 && c->stFrames == 0;
    if (idle && endOp == ZSTD_e_end && room >= ZSTD_compressBound(n)) {      /* one-shot: straight from the caller's buffers */
        size_t const r = ZSTD_compress2(c, (u8*)out->dst + out->pos, room, (const u8*)in->src + in->pos, n);
        if (ZSTD_isError(r)) return r;
        in->pos = in->size; out->pos += r;
        return 0;
    }
    /* output produced earlier goes first; input is only taken while nothing is waiting */
    if (zb_streamHandOut(c, out) == 0) {
        size_t take = n;
        while (take) {
            size_t const space = ZB_STREAM_FRAME - c->stInSize;
            size_t const m = take < space ? take : space;
            if (c->stInSize + m > c->stInCap) {
                size_t cap = c->stInCap ? c->stInCap : ((size_t)1 << 20);
                while (cap < c->stInSize + m) cap *= 2;
                if (cap > ZB_STREAM_FRAME) cap = ZB_STREAM_FRAME;
                u8* const p = (u8*)realloc(c->stIn, cap);
                if (!p) return ZB_ERR(ZB_error_memory_allocation);
                c->stIn = p; c->stInCap = cap;
            }
            memcpy(c->stIn + c->stInSize, (const u8*)in->src + in->pos, m);
            c->stInSize += m; in->pos += m; take -= m;
            if (c->stInSize == ZB_STREAM_FRAME) {                           /* a full frame's worth: compress it, hand out what fits */
                size_t const e = zb_streamMakeFrame(c); if (ZSTD_isError(e)) return e;
                if (zb_streamHandOut(c, out) != 0) break;                    /* the caller has to make room before more input is taken */
            }
        }
        if (in->pos == in->size && endOp != ZSTD_e_continue && c->stOutSize == 0) {
            if (c->stInSize || (endOp == ZSTD_e_end && c->stFrames == 0)) { size_t const e = zb_streamMakeFrame(c); if (ZSTD_isError(e)) return e; }
            zb_streamHandOut(c, out);
        }
    }
    size_t const waiting = c->stOutSize - c->stOutPos;
    if (endOp == ZSTD_e_end && waiting == 0 && in->pos == in->size && c->stInSize == 0) c->stFrames = 0;   /* session over: the next call starts a new one */
    if (endOp == ZSTD_e_continue) return waiting ? waiting : (ZB_STREAM_FRAME - c->stInSize);              /* a hint for the next input size, as the reference gives one */
    return waiting + ((in->pos < in->size || c->stInSize) ? 1 : 0);                                        /* > 0 while the flush / end is incomplete */
}
/* the older streaming entry points are thin forms of the above (lib/zstd.h:832-862) */
extern "C" ZSTD_CStream* ZSTD_createCStream(void) { return ZSTD_createCCtx(); }
extern "C" size_t ZSTD_freeCStream(ZSTD_CStream* zcs) { return ZSTD_freeCCtx(zcs); }
extern "C" size_t ZSTD_initCStream(ZSTD_CStream* zcs, int level)
{
    if (!zcs) return ZB_ERR(ZB_error_GENERIC);
    ZSTD_CCtx_reset(zcs, ZSTD_reset_session_only);
    ZSTD_CCtx_refCDict(zcs, NULL);
    return ZSTD_CCtx_setParameter(zcs, ZSTD_c_compressionLevel, level);
}
extern "C" size_t ZSTD_compressStream(ZSTD_CStream* zcs, ZSTD_outBuffer* output, ZSTD_inBuffer* input) { return ZSTD_compressStream2(zcs, output, input, ZSTD_e_continue); }
extern "C" size_t ZSTD_flushStream(ZSTD_CStream* zcs, ZSTD_outBuffer* output) { ZSTD_inBuffer in = { NULL, 0, 0 }; return ZSTD_compressStream2(zcs, output, &in, ZSTD_e_flush); }
extern "C" size_t ZSTD_endStream(ZSTD_CStream* zcs, ZSTD_outBuffer* output) { ZSTD_inBuffer in = { NULL, 0, 0 }; return ZSTD_compressStream2(zcs, output, &in, ZSTD_e_end); }
extern "C" size_t ZSTD_CStreamInSize(void) { return ZB_BLOCK_MAX; }                                         /* lib/zstd.h:858 */
extern "C" size_t ZSTD_CStreamOutSize(void) { return ZSTD_compressBound(ZB_BLOCK_MAX) + 3 + 4; }            /* lib/zstd.h:859 */

/* ------------------------------------------------------------------ reference-identical entry points */
extern "C" size_t ZSTD_compress_usingDict(ZSTD_CCtx* c, void* dst, size_t dstCapacity, const void* src, size_t srcSize,
                                          const void* dict, size_t dictSize, int level)
{
    if (!c) return ZB_ERR(ZB_error_GENERIC);
    const ZSTD_CDict* cd;
    TRY(zb_digestCallDict(c, dict, dictSize, &cd));
    return zb_compressOne(c, dst, dstCapacity, src, srcSize, cd, level, false, false);   /* the simple API ignores sticky parameters (lib/zstd.h:270-273) */
}
extern "C" size_t ZSTD_compressCCtx(ZSTD_CCtx* c, void* dst, size_t dstCapacity, const void* src, size_t srcSize, int level)
{
    return ZSTD_compress_usingDict(c, dst, dstCapacity, src, srcSize, NULL, 0, level);
}
extern "C" size_t ZSTD_compress(void* dst, size_t dstCapacity, const void* src, size_t srcSize, int level)
{
    ZSTD_CCtx* c = ZSTD_createCCtx();                                            /* zstd_compress.c:5423-5440: temporary context */
    if (!c) return ZB_ERR(ZB_error_memory_allocation);
    size_t const r = ZSTD_compressCCtx(c, dst, dstCapacity, src, srcSize, level);
    ZSTD_freeCCtx(c);
    return r;
}

extern "C" size_t ZSTD_compressBound(size_t srcSize)                             /* lib/zstd.h:235 */
{
    if (srcSize >= (sizeof(size_t) == 8 ? 0xFF00FF00FF00FF00ULL : 0xFF00FF00U)) return ZB_ERR(ZB_error_srcSize_wrong);
    return srcSize + (srcSize >> 8) + ((srcSize < (128u << 10)) ? (((128u << 10) - srcSize) >> 11) : 0);
}
extern "C" unsigned ZSTD_isError(size_t code) { return code > ZB_ERR(ZB_error_maxCode); }
extern "C" int ZSTD_getErrorCode(size_t code) { return ZSTD_isError(code) ? (int)(0 - code) : 0; }
extern "C" const char* ZSTD_getErrorName(size_t code)                            /* common/error_private.c:14-62 */
{
    switch (ZSTD_getErrorCode(code)) {
    case 0: return "No error detected";
    case 1: return "Error (generic)";
    case 10: return "Unknown frame descriptor";
    case 12: return "Version not supported";
    case 14: return "Unsupported frame parameter";
    case 16: return "Frame requires too much memory for decoding";
    case 20: return "Data corruption detected";
    case 22: return "Restored data doesn't match checksum";
    case 24: return "Header of Literals' block doesn't respect format specification";
    case 30: return "Dictionary is corrupted";
    case 32: return "Dictionary mismatch";
    case 34: return "Cannot create Dictionary from provided samples";
    case 40: return "Unsupported parameter";
    case 41: return "Unsupported combination of parameters";
    case 42: return "Parameter is out of bound";
    case 44: return "tableLog requires too much memory : unsupported";
    case 46: return "Unsupported max Symbol Value : too large";
    case 48: return "Specified maxSymbolValue is too small";
    case 50: return "pledged buffer stability condition is not respected";
    case 60: return "Operation not authorized at current processing stage";
    case 62: return "Context should be init first";
    case 64: return "Allocation error : not enough memory";
    case 66: return "workSpace buffer is not large enough";
    case 70: return "Destination buffer is too small";
    case 72: return "Src size is incorrect";
    case 74: return "Operation on NULL destination buffer";
    case 80: return "Operation made no progress over multiple calls, due to output buffer being full";
    case 82: return "Operation made no progress over multiple calls, due to input being empty";
    case 107: return "External sequences are not valid";
    default: return "Unspecified error code";
    }
}
extern "C" int ZSTD_minCLevel(void) { return -(int)ZB_BLOCK_MAX; }                /* zstd_compress.c:7038 */
extern "C" int ZSTD_maxCLevel(void) { return 22; }
extern "C" int ZSTD_defaultCLevel(void) { return 3; }
extern "C" unsigned ZSTD_versionNumber(void) { return 10506; }                    /* lib/zstd.h:107-110 */
extern "C" const char* ZSTD_versionString(void) { return "1.5.6"; }
