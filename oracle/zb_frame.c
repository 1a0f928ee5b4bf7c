/* zb_frame.c — oracle frame driver (TEST INFRASTRUCTURE ONLY): parameter derivation, frame header,
 * block loop and block headers, mirroring what ZSTD_compress / ZSTD_compress_usingDict do around
 * the hot path (lib/compress/zstd_compress.c:5398-5440, :4527-4623, :4626-4672).
 */
#include <string.h>
#include <stdlib.h>
#include "zb_oracle.h"

static inline u32 hb32(u32 v) { return 31u - (u32)__builtin_clz(v); }

/* compress/clevels.h:25-130, rows 0..4 of the four size classes (strategies fast=1 / dfast=2 only;
 * rows whose reference strategy is greedy or above are served by the last dfast row of the class) */
typedef struct { u8 W, C, H, S, L, TL, strat; } row;
static const row kRows[4][5] = {
    { {19,12,13,1,6,1,1}, {19,13,14,1,7,0,1}, {20,15,16,1,6,0,1}, {21,16,17,1,5,0,2}, {21,18,18,1,5,0,2} },   /* > 256 KB */
    { {18,12,13,1,5,1,1}, {18,13,14,1,6,0,1}, {18,14,14,1,5,0,2}, {18,16,16,1,4,0,2}, {18,16,16,1,4,0,2} },   /* <= 256 KB (level 4 is greedy there -> row 3) */
    { {17,12,12,1,5,1,1}, {17,12,13,1,6,0,1}, {17,13,15,1,5,0,1}, {17,15,16,2,5,0,2}, {17,17,17,2,4,0,2} },   /* <= 128 KB */
    { {14,12,13,1,5,1,1}, {14,14,15,1,5,0,1}, {14,14,15,1,4,0,1}, {14,14,15,2,4,0,2}, {14,14,15,2,4,0,2} },   /* <= 16 KB (level 4 is greedy there -> row 3) */
};

/* zstd_compress.c:1432-1459 */
static u32 dictAndWindowLog(u32 windowLog, u64 srcSize, u64 dictSize)
{
    u64 const maxWindowSize = 1ull << 31;
    if (dictSize == 0) return windowLog;
    {   u64 const windowSize = 1ull << windowLog;
        u64 const dictAndWindowSize = dictSize + windowSize;
        if (windowSize >= dictSize + srcSize) return windowLog;
        if (dictAndWindowSize >= maxWindowSize) return 31;
        return hb32((u32)dictAndWindowSize - 1) + 1;
    }
}

/* zstd_compress.c:7123-7146 (row selection) + :1465-1602 (adjust, mode = cpm_noAttachDict) */
zbo_cparams zbo_getCParams(int level, u64 srcSize, size_t dictSize)
{
    u64 const rSize = srcSize + dictSize;
    u32 const tableID = (rSize <= 256u * 1024) + (rSize <= 128u * 1024) + (rSize <= 16u * 1024);
    int r = level == 0 ? 3 : (level < 0 ? 0 : (level > 4 ? 4 : level));
    zbo_cparams cp;
    {   row const x = kRows[tableID][r];
        cp.windowLog = x.W; cp.chainLog = x.C; cp.hashLog = x.H; cp.searchLog = x.S;
        cp.minMatch = x.L; cp.targetLength = x.TL; cp.strategy = x.strat;
    }
    if (level < 0) {
        int const minLevel = -(1 << 17);                       /* ZSTD_minCLevel, zstd_compress.c:7073 */
        int const cl = level < minLevel ? minLevel : level;
        cp.targetLength = (u32)(-cl);
    }
    {   u64 const maxWindowResize = 1ull << 30;
        if (srcSize <= maxWindowResize && dictSize <= maxWindowResize) {
            u32 const tSize = (u32)(srcSize + dictSize);
            u32 const srcLog = (tSize < (1u << 6)) ? 6 : hb32(tSize - 1) + 1;
            if (cp.windowLog > srcLog) cp.windowLog = srcLog;
        }
        {   u32 const dawl = dictAndWindowLog(cp.windowLog, srcSize, dictSize);
            u32 const cycleLog = cp.chainLog;
            if (cp.hashLog > dawl + 1) cp.hashLog = dawl + 1;
            if (cycleLog > dawl) cp.chainLog -= (cycleLog - dawl);
        }
        if (cp.windowLog < 10) cp.windowLog = 10;
    }
    return cp;
}

/* lib/zstd.h:235 */
size_t zbo_compressBound(size_t srcSize)
{
    if (srcSize >= 0xFF00FF00FF00FF00ull) return ZBO_ERR(ZBO_error_srcSize_wrong);
    return srcSize + (srcSize >> 8) + ((srcSize < (128u << 10)) ? (((128u << 10) - srcSize) >> 11) : 0);
}

/* zstd_compress.c:4626-4672 : contentSizeFlag=1, no checksum */
size_t zbo_writeFrameHeader(u8* dst, size_t cap, u32 windowLog, u64 srcSize, u32 dictID)
{
    u32 const dictIDSizeCode = (dictID > 0) + (dictID >= 256) + (dictID >= 65536);
    u64 const windowSize = 1ull << windowLog;
    u32 const singleSegment = windowSize >= srcSize;
    u8  const windowLogByte = (u8)((windowLog - 10) << 3);
    u32 const fcsCode = (srcSize >= 256) + (srcSize >= 65536 + 256) + (srcSize >= 0xFFFFFFFFu);
    size_t pos = 0;
    if (cap < 18) return ZBO_ERR(ZBO_error_dstSize_tooSmall);      /* ZSTD_FRAMEHEADERSIZE_MAX */
    dst[0] = 0x28; dst[1] = 0xB5; dst[2] = 0x2F; dst[3] = 0xFD; pos = 4;
    dst[pos++] = (u8)(dictIDSizeCode + (singleSegment << 5) + (fcsCode << 6));
    if (!singleSegment) dst[pos++] = windowLogByte;
    switch (dictIDSizeCode) {
    case 1: dst[pos++] = (u8)dictID; break;
    case 2: dst[pos++] = (u8)dictID; dst[pos++] = (u8)(dictID >> 8); break;
    case 3: dst[pos++] = (u8)dictID; dst[pos++] = (u8)(dictID >> 8); dst[pos++] = (u8)(dictID >> 16); dst[pos++] = (u8)(dictID >> 24); break;
    default: break;
    }
    switch (fcsCode) {
    case 0: if (singleSegment) dst[pos++] = (u8)srcSize; break;
    case 1: { u16 v = (u16)(srcSize - 256); dst[pos++] = (u8)v; dst[pos++] = (u8)(v >> 8); } break;
    case 2: { u32 v = (u32)srcSize; for (int i = 0; i < 4; i++) dst[pos++] = (u8)(v >> (8 * i)); } break;
    default: for (int i = 0; i < 8; i++) dst[pos++] = (u8)(srcSize >> (8 * i)); break;
    }
    return pos;
}

static int isRLE(const u8* src, size_t n)
{
    for (size_t i = 1; i < n; i++) if (src[i] != src[0]) return 0;
    return 1;
}

/* ------------------------------------------------------------------------------------------
 * Dictionaries (zstd_compress.c:5119-5156).  A dictionary shorter than 8 bytes is ignored (:5132);
 * without the magic number 0xEC30A437 it is raw content (:5143-5148); with it, it is a zstd-format
 * dictionary: magic, dictID, Huffman table, 3 FSE tables (OF, ML, LL), 3 repcodes, content
 * (ZSTD_loadCEntropy :4987-5076, restated in zb_dict.c).  The content of either kind is the history of
 * the frame's first block; a zstd-format dictionary's Huffman / FSE tables are that block's "previous"
 * entropy state (treeless literals, set_repeat sequence tables) and its repcodes start the block.
 * ---------------------------------------------------------------------------------------- */
/* One frame.  Blocks are independent (block-parallel plan); see zb_match.c. */
u64 zbo_dbg[8];
size_t zbo_compress_usingDict(void* dstv, size_t cap, const void* srcv, size_t srcSize,
                              const void* dictv, size_t dictSize, int level)
{
    u8* const dst = (u8*)dstv;
    const u8* src = (const u8*)srcv;
    const u8* const dict = (const u8*)dictv;
    int const useDict = (dict != NULL) && (dictSize >= 8);
    zbo_cparams cp = zbo_getCParams(level, srcSize, useDict ? dictSize : 0);
    zbo_plan plan;
    size_t pos;
    size_t const blockMax = ((size_t)1 << cp.windowLog) < ZB_BLOCK_MAX ? ((size_t)1 << cp.windowLog) : ZB_BLOCK_MAX;  /* zstd_compress.c:2124 */
    u32 dictID = 0;
    u8* vbuf = NULL;                 /* [dictionary content tail | src] when a dictionary is in use */
    size_t D = 0;                    /* bytes of dictionary content in front of the frame */

    zbo_makePlan(&plan, &cp);
    zbo_dict_entropy* de = NULL;
    if (useDict) {
        size_t contentOff;
        de = (zbo_dict_entropy*)malloc(sizeof(*de));
        contentOff = zbo_loadDictEntropy(de, dict, dictSize);
        if (zbo_isError(contentOff)) { free(de); return contentOff; }
        dictID = de->dictID;
        {   size_t const contentSize = dictSize - contentOff;
            D = contentSize < plan.primeBytes ? contentSize : plan.primeBytes;
            vbuf = (u8*)malloc(D + srcSize + 16);
            memcpy(vbuf, dict + contentOff + (contentSize - D), D);
            memcpy(vbuf + D, src, srcSize);
            src = vbuf + D;
        }
    }
    plan.frameStart = D;
    plan.startRep[0] = plan.startRep[1] = 0;
    plan.codeRep[0] = 1; plan.codeRep[1] = 4; plan.codeRep[2] = 8;                  /* zstd_internal.h:69 */
    if (de && de->present) { plan.codeRep[0] = de->rep[0]; plan.codeRep[1] = de->rep[1]; plan.codeRep[2] = de->rep[2];
        plan.startRep[0] = de->rep[0] <= D ? de->rep[0] : 0; plan.startRep[1] = de->rep[1] <= D ? de->rep[1] : 0; }   /* zstd_compress.c:5054-5056 */
    pos = zbo_writeFrameHeader(dst, cap, cp.windowLog, srcSize, dictID);
    if (zbo_isError(pos)) { free(vbuf); free(de); return pos; }

    if (srcSize == 0) {                                    /* zstd_compress.c:5279-5295 : empty last raw block */
        free(vbuf); free(de);
        if (cap - pos < 3) return ZBO_ERR(ZBO_error_dstSize_tooSmall);
        dst[pos++] = 1; dst[pos++] = 0; dst[pos++] = 0;
        return pos;
    }
    {   zbo_seq* seqs = (zbo_seq*)malloc((ZB_BLOCK_MAX / 4 + 1) * sizeof(zbo_seq));
        u8* lit = (u8*)malloc(ZB_BLOCK_MAX + 64);
        size_t const bodyCap = ZB_BLOCK_MAX * 4;
        u8* body = (u8*)malloc(bodyCap);
        size_t bs = 0;
        size_t err = 0;
        int first = 1;
        zbo_chunkCand cc; size_t const chunkBytes = (size_t)plan.chunkBlocks * blockMax;
        memset(&cc, 0, sizeof(cc));
        while (bs < srcSize) {
            size_t const blockSize = (srcSize - bs) < blockMax ? (srcSize - bs) : blockMax;
            u32 const lastBlock = (bs + blockSize == srcSize);
            size_t cSize = 0;
            if (blockSize >= 7) {                                    /* zstd_compress.c:3216 */
                size_t litSize = 0;
                /* the buffer handed to the matcher starts D bytes in front of the frame: only the first
                 * block's history window reaches back into the dictionary */
                size_t nbSeq;
                if (cc.dS == NULL || bs + D >= cc.end) {       /* next chunk: walk it */
                    size_t const cs = bs - bs % chunkBytes;
                    size_t const ce = cs + chunkBytes < srcSize ? cs + chunkBytes : srcSize;
                    zbo_freeChunk(&cc);
                    zbo_walkChunk(&plan, src - D, srcSize + D, cs + D, ce + D, &cc);
                }
                nbSeq = zbo_parseBlock(&plan, src - D, &cc, bs + D, blockSize, seqs, lit, &litSize);
                zbo_dbg[0] += nbSeq; zbo_dbg[1] += litSize; { size_t i; for (i = 0; i < nbSeq; i++) { zbo_dbg[2] += seqs[i].offBase <= 3; zbo_dbg[3] += seqs[i].matchLen; } }
                cSize = zbo_entropyCompressBlock_prev(body, bodyCap, seqs, nbSeq, lit, litSize, blockSize,
                                                      cp.strategy, (int)plan.litCompressionDisabled, first ? de : NULL);
                if (zbo_isError(cSize)) { err = cSize; break; }
                if (!first && cSize < 25 && isRLE(src + bs, blockSize)) { cSize = 1; body[0] = src[bs]; }   /* :4365-4376 */
            }
            if (cSize == 0) {                                          /* raw block, zstd_compress_internal.h:586 */
                if (cap - pos < 3 + blockSize) { err = ZBO_ERR(ZBO_error_dstSize_tooSmall); break; }
                {   u32 const h = lastBlock + (0u << 1) + (u32)(blockSize << 3);
                    dst[pos] = (u8)h; dst[pos + 1] = (u8)(h >> 8); dst[pos + 2] = (u8)(h >> 16); }
                memcpy(dst + pos + 3, src + bs, blockSize);
                pos += 3 + blockSize;
            } else {
                u32 const h = (cSize == 1) ? lastBlock + (1u << 1) + (u32)(blockSize << 3)
                                           : lastBlock + (2u << 1) + (u32)(cSize << 3);           /* :4586-4590 */
                if (cap - pos < 3 + cSize) { err = ZBO_ERR(ZBO_error_dstSize_tooSmall); break; }
                dst[pos] = (u8)h; dst[pos + 1] = (u8)(h >> 8); dst[pos + 2] = (u8)(h >> 16);
                memcpy(dst + pos + 3, body, cSize);
                pos += 3 + cSize;
            }
            bs += blockSize;
            first = 0;
        }
        zbo_freeChunk(&cc);
        free(seqs); free(lit); free(body); free(vbuf); free(de);
        if (err) return err;
    }
    return pos;
}

size_t zbo_compress(void* dst, size_t cap, const void* src, size_t srcSize, int level)
{
    return zbo_compress_usingDict(dst, cap, src, srcSize, NULL, 0, level);
}

/* ------------------------------------------------------------------------------------------
 * Synthetic LZ-style test data (our own generator, for tests that must run without the
 * reference's datagen binary): literals from a skewed alphabet, matches copied from the last
 * 32 KiB with probability matchProb/256, match lengths 4..~500.
 * ---------------------------------------------------------------------------------------- */
void zbo_synthetic(u8* buf, size_t n, u32 seed, u32 matchProb256)
{
    u64 s = 0x9E3779B97F4A7C15ull ^ ((u64)seed * 0xD1B54A32D192ED03ull);
    size_t pos = 0;
#define RND() (s ^= s << 13, s ^= s >> 7, s ^= s << 17, (u32)(s >> 32))
    while (pos < n) {
        u32 const r = RND();
        if (pos > 16 && (r & 255u) < matchProb256) {
            u32 const r2 = RND();
            size_t len = 4 + ((r2 & 15u) ? (r2 >> 4) % 28u : (r2 >> 4) % 500u);
            size_t const maxOff = pos < 32768 ? pos : 32768;
            size_t const off = 1 + (RND() % maxOff);
            if (len > n - pos) len = n - pos;
            for (size_t i = 0; i < len; i++) buf[pos + i] = buf[pos + i - off];
            pos += len;
        } else {
            u32 const r2 = RND();
            u32 const k = r2 & 7u;       /* skew: small symbols far more likely */
            u8 const c = (u8)(k < 5 ? (r2 >> 8) % 24u : (k < 7 ? (r2 >> 8) % 96u : (r2 >> 8)));
            buf[pos++] = (u8)('a' + c);
        }
    }
#undef RND
}
