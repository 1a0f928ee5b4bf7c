/* zb_ldm.c — oracle of the long-distance match finder (TEST INFRASTRUCTURE ONLY); the CUDA kernels of
 * zstd_b200/csrc/zb_ldm.cu produce the same matches bit for bit.
 *
 * The reference's generator (lib/compress/zstd_ldm.c:327-497) walks the input serially: it moves an anchor, skips split
 * points under the last match and resets its rolling hash behind long matches.  This is a deterministic data-parallel
 * restatement of the same idea, applied to every frame of more than one chunk (512 KiB):
 *   1. split points: a gear rolling hash h = (h << 1) + gear[byte] (it depends on the last 64 bytes only, so every
 *      position has its own) fires where (h & stopMask) == 0, with the reference's stop mask (zstd_ldm.c:32-60).  The split
 *      point is the start p of the minMatch bytes that end where it fires.  gear[] is our own table (splitmix64);
 *   2. thinning: v = XXH64 (seed 0) of the minMatch bytes at p.  A split survives iff its v is <= the v of every split in
 *      the minMatch - 1 positions before it and < the v of every split in the minMatch - 1 positions after it: survivors
 *      are at least minMatch apart, and a copy of some content has the survivors of its original away from its edges;
 *   3. buckets: bucket = the low hashLog - bucketSizeLog bits of v, checksum = its high 32 bits.  The candidates of a
 *      survivor are the 2^bucketSizeLog nearest earlier survivors of its bucket that have its checksum and lie at or after
 *      max(frame start, block end - window);
 *   4. selection, per 128 KiB block: survivors in position order from anchor = block start; p < anchor is skipped.  A
 *      candidate q counts when its forward length f (capped at the block end) is >= minMatch; b is the backward length
 *      (capped at p - anchor and at q).  The largest f + b wins, on a tie the larger q.  (p - b, f + b, p - q) is emitted
 *      and anchor = p + f: an LDM match never crosses a block edge;
 *   5. overlay onto the block's parse output: an LDM match wins; a parse match that starts under one starts again at its
 *      end, one that runs into one is cut at its start; a parse match shortened this way is kept only when at least 4 bytes
 *      remain (the parse's shortest match), so a block still holds at most blockSize / 4 + 8 sequences.
 * The dictionary content is not indexed (the reference indexes it, zstd_compress.c:4840). */
#include <stdlib.h>
#include <string.h>
#include "zb_oracle.h"

/* Everything LDM lives in this file: the rest of the oracle is the LDM-off path, untouched.  The tests reach these functions
 * through ctypes (tests/ldmref.py); zbo_compress_ldm[_usingDict] is the frame the GPU produces with LDM on. */
#define ZB_LDM_WINDOW_LOG   27u                      /* ZSTD_LDM_DEFAULT_WINDOW_LOG, zstd_ldm.h:25 */
#define ZB_LDM_MIN_FRAME    (ZB_CHUNK_BLOCKS * ZB_BLOCK_MAX)   /* LDM applies to frames of more than one chunk */
#define ZB_LDM_GEAR_SEED    0x6C646D2D67656172ull    /* "ldm-gear" */
typedef struct { u32 hashLog, minMatch, bucketSizeLog, hashRateLog; } zbo_ldm_params;   /* 0 = derived from the window */
typedef struct { u32 start, len, off; } zbo_ldm_match;                               /* start: relative to its block */
typedef struct { size_t nbBlocks, nbSurvivors; u64* first; u32* cnt; zbo_ldm_match* m; } zbo_ldm_lists;
u64            zbo_ldm_gear(u32 i);
zbo_ldm_params zbo_ldm_resolve(const zbo_ldm_params* p, u32 windowLog);
u64            zbo_ldm_stopMask(const zbo_ldm_params* p);
u64            zbo_xxh64(const u8* p, size_t len);
size_t         zbo_ldm_survivors(const u8* src, size_t n, const zbo_ldm_params* resolved, u64* pos, u64* v);
zbo_ldm_lists  zbo_ldm_frame(const u8* src, size_t n, u32 windowLog, const zbo_ldm_params* p);
void           zbo_ldm_free(zbo_ldm_lists* L);
size_t         zbo_ldm_overlayBlock(const u8* blk, size_t blockSize, const u32 rep[3], const zbo_ldm_match* lm, size_t nL,
                                    zbo_seq* seqs, size_t nbSeq, u8* lit, size_t* litSizePtr);
zbo_cparams    zbo_getCParams_ldm(int level, u64 srcSize, size_t dictSize);
size_t         zbo_compress_ldm(void* dst, size_t cap, const void* src, size_t srcSize, int level, const zbo_ldm_params* ldm);
size_t         zbo_compress_ldm_usingDict(void* dst, size_t cap, const void* src, size_t srcSize, const void* dict, size_t dictSize,
                                          int level, const zbo_ldm_params* ldm);

/* gear table: splitmix64 outputs 1..256 of the seed below */
u64 zbo_ldm_gear(u32 i)
{
    u64 z = ZB_LDM_GEAR_SEED + (u64)(i + 1u) * 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

/* ZSTD_ldm_adjustParameters (zstd_ldm.c:135) for a frame of window 2^windowLog; 0 = derived */
zbo_ldm_params zbo_ldm_resolve(const zbo_ldm_params* in, u32 windowLog)
{
    zbo_ldm_params p = *in;
    if (!p.bucketSizeLog) p.bucketSizeLog = 3;                 /* LDM_BUCKET_SIZE_LOG */
    if (!p.minMatch) p.minMatch = 64;                          /* LDM_MIN_MATCH_LENGTH */
    if (!p.hashLog) p.hashLog = windowLog > 7 + 6 ? windowLog - 7 : 6;   /* MAX(ZSTD_HASHLOG_MIN, windowLog - LDM_HASH_RLOG) */
    if (!p.hashRateLog) p.hashRateLog = windowLog < p.hashLog ? 0 : windowLog - p.hashLog;
    if (p.bucketSizeLog > p.hashLog) p.bucketSizeLog = p.hashLog;
    return p;
}

u64 zbo_ldm_stopMask(const zbo_ldm_params* p)                  /* ZSTD_ldm_gear_init, zstd_ldm.c:32-60 */
{
    u32 const maxBits = p->minMatch < 64 ? p->minMatch : 64;
    if (p->hashRateLog > 0 && p->hashRateLog <= maxBits) return (((u64)1 << p->hashRateLog) - 1) << (maxBits - p->hashRateLog);
    return ((u64)1 << p->hashRateLog) - 1;
}

static u64 rd64(const u8* p) { u64 v; memcpy(&v, p, 8); return v; }
static u32 rd32(const u8* p) { u32 v; memcpy(&v, p, 4); return v; }
static u64 rotl(u64 x, int r) { return (x << r) | (x >> (64 - r)); }
#define P1 0x9E3779B185EBCA87ull
#define P2 0xC2B2AE3D27D4EB4Full
#define P3 0x165667B19E3779F9ull
#define P4 0x85EBCA77C2B2AE63ull
#define P5 0x27D4EB2F165667C5ull
static u64 round64(u64 acc, u64 in) { return rotl(acc + in * P2, 31) * P1; }
static u64 merge64(u64 h, u64 v) { return (h ^ round64(0, v)) * P1 + P4; }
u64 zbo_xxh64(const u8* p, size_t len)                          /* seed 0 */
{
    const u8* const end = p + len;
    u64 h;
    if (len >= 32) {
        u64 v1 = P1 + P2, v2 = P2, v3 = 0, v4 = 0 - P1;
        const u8* const limit = end - 32;
        do { v1 = round64(v1, rd64(p)); v2 = round64(v2, rd64(p + 8)); v3 = round64(v3, rd64(p + 16)); v4 = round64(v4, rd64(p + 24)); p += 32; } while (p <= limit);
        h = rotl(v1, 1) + rotl(v2, 7) + rotl(v3, 12) + rotl(v4, 18);
        h = merge64(h, v1); h = merge64(h, v2); h = merge64(h, v3); h = merge64(h, v4);
    } else h = P5;
    h += (u64)len;
    while (p + 8 <= end) { h ^= round64(0, rd64(p)); h = rotl(h, 27) * P1 + P4; p += 8; }
    if (p + 4 <= end) { h ^= (u64)rd32(p) * P1; h = rotl(h, 23) * P2 + P3; p += 4; }
    while (p < end) { h ^= (u64)(*p) * P5; h = rotl(h, 11) * P1; p++; }
    h ^= h >> 33; h *= P2; h ^= h >> 29; h *= P3; h ^= h >> 32;
    return h;
}

/* steps 1 and 2: survivors of src[0, n) in position order; pos / v hold at most n / minMatch + 1 entries */
size_t zbo_ldm_survivors(const u8* src, size_t n, const zbo_ldm_params* prm, u64* pos, u64* v)
{
    u32 const mm = prm->minMatch;
    u64 const mask = zbo_ldm_stopMask(prm);
    u64 gear[256];
    u8* split; u64* hv;
    size_t i, cnt = 0, nbP;
    if (n < mm) return 0;
    nbP = n - mm + 1;                                          /* split points p in [0, nbP) */
    for (i = 0; i < 256; i++) gear[i] = zbo_ldm_gear((u32)i);
    split = (u8*)calloc(nbP, 1); hv = (u64*)malloc(nbP * sizeof(u64));
    {   u64 h = 0;
        for (i = 0; i < n; i++) {
            h = (h << 1) + gear[src[i]];
            if (i + 1 >= mm && (h & mask) == 0) { size_t const p = i + 1 - mm; split[p] = 1; hv[p] = zbo_xxh64(src + p, mm); }
        }
    }
    for (i = 0; i < nbP; i++) {
        size_t const lo = i >= mm - 1 ? i - (mm - 1) : 0, hi = i + (mm - 1) < nbP - 1 ? i + (mm - 1) : nbP - 1;
        size_t q; int ok = 1;
        if (!split[i]) continue;
        for (q = lo; q < i && ok; q++) if (split[q] && hv[q] < hv[i]) ok = 0;
        for (q = i + 1; q <= hi && ok; q++) if (split[q] && hv[q] <= hv[i]) ok = 0;
        if (ok) { pos[cnt] = i; v[cnt] = hv[i]; cnt++; }
    }
    free(split); free(hv);
    return cnt;
}

typedef struct { u32 bucket, idx; } bkey;
static int cmp_bkey(const void* a, const void* b)              /* stable: ties by position order */
{
    const bkey* x = (const bkey*)a; const bkey* y = (const bkey*)b;
    if (x->bucket != y->bucket) return x->bucket < y->bucket ? -1 : 1;
    return x->idx < y->idx ? -1 : (x->idx > y->idx);
}

static size_t count_fwd(const u8* src, size_t p, size_t q, size_t limit)
{
    size_t f = 0;
    while (f < limit && src[p + f] == src[q + f]) f++;
    return f;
}

/* steps 3 and 4 for a frame src[0, n): the matches of block k go to m[first[k] .. first[k] + cnt[k]) */
zbo_ldm_lists zbo_ldm_frame(const u8* src, size_t n, u32 windowLog, const zbo_ldm_params* prmIn)
{
    zbo_ldm_params const prm = zbo_ldm_resolve(prmIn, windowLog);
    size_t const cap = n / prm.minMatch + 1;
    size_t const nbBlocks = (n + ZB_BLOCK_MAX - 1) / ZB_BLOCK_MAX;
    u64* pos = (u64*)malloc(cap * sizeof(u64)); u64* v = (u64*)malloc(cap * sizeof(u64));
    size_t const N = zbo_ldm_survivors(src, n, &prm, pos, v);
    u32 const bucketBits = prm.hashLog - prm.bucketSizeLog;
    u32 const nbCand = 1u << prm.bucketSizeLog;
    u64 const W = (u64)1 << windowLog;
    bkey* keys = (bkey*)malloc((N + 1) * sizeof(bkey));
    u32* rank = (u32*)malloc((N + 1) * sizeof(u32));
    zbo_ldm_lists L;
    size_t i, k, si = 0;
    L.nbBlocks = nbBlocks; L.nbSurvivors = N;
    L.first = (u64*)calloc(nbBlocks + 1, sizeof(u64)); L.cnt = (u32*)calloc(nbBlocks + 1, sizeof(u32));
    L.m = (zbo_ldm_match*)malloc((N + 1) * sizeof(zbo_ldm_match));
    for (i = 0; i < N; i++) { keys[i].bucket = (u32)(v[i] & (((u64)1 << bucketBits) - 1)); keys[i].idx = (u32)i; }
    qsort(keys, N, sizeof(bkey), cmp_bkey);
    for (i = 0; i < N; i++) rank[keys[i].idx] = (u32)i;
    for (k = 0; k < nbBlocks; k++) {
        size_t const bs = k * ZB_BLOCK_MAX, be = bs + ZB_BLOCK_MAX < n ? bs + ZB_BLOCK_MAX : n;
        size_t const lowQ = be > W ? be - W : 0;
        size_t anchor = bs, out = 0;
        while (si < N && pos[si] < bs) si++;
        L.first[k] = si;
        for (i = si; i < N && pos[i] < be; i++) {
            size_t const p = pos[i];
            size_t bestLen = 0, bestQ = 0, bestB = 0, bestF = 0;
            u32 j;
            if (p < anchor) continue;
            for (j = 1; j <= nbCand && rank[i] >= j; j++) {
                bkey const c = keys[rank[i] - j];
                size_t q, f, b, bmax;
                if (c.bucket != keys[rank[i]].bucket) break;
                q = pos[c.idx];
                if ((v[c.idx] >> 32) != (v[i] >> 32) || q < lowQ) continue;
                f = count_fwd(src, p, q, be - p);
                if (f < prm.minMatch) continue;
                bmax = p - anchor < q ? p - anchor : q;
                b = 0;
                while (b < bmax && src[p - b - 1] == src[q - b - 1]) b++;
                if (f + b > bestLen || (f + b == bestLen && q > bestQ)) { bestLen = f + b; bestQ = q; bestB = b; bestF = f; }
            }
            if (!bestLen) continue;
            L.m[si + out].start = (u32)(p - bestB - bs); L.m[si + out].len = (u32)bestLen; L.m[si + out].off = (u32)(p - bestQ);
            out++;
            anchor = p + bestF;
        }
        L.cnt[k] = (u32)out;
    }
    free(pos); free(v); free(keys); free(rank);
    return L;
}

void zbo_ldm_free(zbo_ldm_lists* L) { free(L->first); free(L->cnt); free(L->m); memset(L, 0, sizeof(*L)); }

/* step 5 on a block's final sequences (as zbo_parseBlock returns them, repcodes assigned): the repcode history is run
 * forward to recover every match's offset, the LDM matches are laid over the matches, and repcodes and literals are
 * assigned again from the merged list with zbo_parseBlock's rules.  blk = the block's bytes; rep = the history at the
 * block's start ({1,4,8} / the dictionary's in a frame's first block, else 0: never matches).  Returns the new nbSeq. */
typedef struct { u32 ms, len, off; } rawm;
size_t zbo_ldm_overlayBlock(const u8* blk, size_t blockSize, const u32 rep[3], const zbo_ldm_match* lm, size_t nL,
                            zbo_seq* seqs, size_t nbSeq, u8* lit, size_t* litSizePtr)
{
    rawm* P = (rawm*)malloc((nbSeq + 1) * sizeof(rawm));
    rawm* out = (rawm*)malloc((nbSeq + nL + 1) * sizeof(rawm));
    size_t i, j = 0, n = 0, pos = 0, litSize = 0;
    u32 r1 = rep[0], r2 = rep[1], r3 = rep[2];
    for (i = 0; i < nbSeq; i++) {                              /* offsets back from the codes */
        u32 const ob = seqs[i].offBase, ll = seqs[i].litLen;
        u32 off;
        if (ob > 3) { off = ob - 3; r3 = r2; r2 = r1; r1 = off; }
        else if (ll > 0) {
            if (ob == 1) off = r1;
            else if (ob == 2) { off = r2; r2 = r1; r1 = off; }
            else { off = r3; r3 = r2; r2 = r1; r1 = off; }
        } else {
            if (ob == 1) { off = r2; r2 = r1; r1 = off; }
            else if (ob == 2) { off = r3; r3 = r2; r2 = r1; r1 = off; }
            else { off = r1 - 1; r3 = r2; r2 = r1; r1 = off; }
        }
        pos += ll;
        P[i].ms = (u32)pos; P[i].len = seqs[i].matchLen; P[i].off = off;
        pos += seqs[i].matchLen;
    }
    for (i = 0; i < nbSeq; i++) {
        u32 ms = P[i].ms, me = P[i].ms + P[i].len;
        int clipped = 0;
        while (j < nL && lm[j].start + lm[j].len <= ms) out[n++] = (rawm){ lm[j].start, lm[j].len, lm[j].off }, j++;   /* LDM matches that end before it */
        {   size_t k = j;                                      /* lm[j] is the first LDM match that ends after ms */
            if (k < nL && lm[k].start <= ms) { ms = lm[k].start + lm[k].len; clipped = 1; k++; }   /* starts under it */
            if (k < nL && lm[k].start < me) { me = lm[k].start; clipped = 1; }                      /* runs into the next */
        }
        if (me <= ms || (clipped && me - ms < 4)) continue;
        while (j < nL && lm[j].start < ms) out[n++] = (rawm){ lm[j].start, lm[j].len, lm[j].off }, j++;
        out[n].ms = ms; out[n].len = me - ms; out[n].off = P[i].off; n++;
    }
    while (j < nL) out[n++] = (rawm){ lm[j].start, lm[j].len, lm[j].off }, j++;
    r1 = rep[0]; r2 = rep[1]; r3 = rep[2];
    pos = 0;
    for (i = 0; i < n; i++) {                                  /* zbo_parseBlock's repcode rules */
        u32 const off = out[i].off, ll = out[i].ms - (u32)pos;
        u32 offBase;
        if (ll > 0) {
            if (off == r1) offBase = 1;
            else if (off == r2) { offBase = 2; r2 = r1; r1 = off; }
            else if (off == r3) { offBase = 3; r3 = r2; r2 = r1; r1 = off; }
            else { offBase = off + 3; r3 = r2; r2 = r1; r1 = off; }
        } else {
            if (off == r2) { offBase = 1; r2 = r1; r1 = off; }
            else if (off == r3) { offBase = 2; r3 = r2; r2 = r1; r1 = off; }
            else if (r1 > 1 && off == r1 - 1) { offBase = 3; r3 = r2; r2 = r1; r1 = off; }
            else { offBase = off + 3; r3 = r2; r2 = r1; r1 = off; }
        }
        memcpy(lit + litSize, blk + pos, ll); litSize += ll;
        seqs[i].offBase = offBase; seqs[i].litLen = ll; seqs[i].matchLen = out[i].len;
        pos = out[i].ms + out[i].len;
    }
    memcpy(lit + litSize, blk + pos, blockSize - pos); litSize += blockSize - pos;
    *litSizePtr = litSize;
    free(P); free(out);
    return n;
}

/* ---- frame driver ------------------------------------------------------------------------------------------------ */
static inline u32 hb32(u32 v) { return 31u - (u32)__builtin_clz(v); }

/* The cParams of a frame with LDM on: the window is ZSTD_LDM_DEFAULT_WINDOW_LOG before the size adjustment
 * (ZSTD_getCParamsFromCCtxParams, zstd_compress.c:1639), then clamped to the input as zstd_compress.c:1537-1547 does.
 * The rest is zbo_getCParams's: for a frame of more than 512 KiB its hashLog / chainLog are below the clamp of
 * ZSTD_adjustCParams_internal whatever the window (every row's hashLog and chainLog are <= 18, the window >= 20). */
zbo_cparams zbo_getCParams_ldm(int level, u64 srcSize, size_t dictSize)
{
    zbo_cparams cp = zbo_getCParams(level, srcSize, dictSize);
    cp.windowLog = ZB_LDM_WINDOW_LOG;
    if (srcSize <= (1ull << 30) && dictSize <= (1ull << 30)) {
        u32 const tSize = (u32)(srcSize + dictSize);
        u32 const srcLog = (tSize < (1u << 6)) ? 6 : hb32(tSize - 1) + 1;
        if (cp.windowLog > srcLog) cp.windowLog = srcLog;
    }
    if (cp.windowLog < 10) cp.windowLog = 10;
    return cp;
}

static int isRLE(const u8* src, size_t n)
{
    for (size_t i = 1; i < n; i++) if (src[i] != src[0]) return 0;
    return 1;
}

/* One frame with LDM: zbo_compress_usingDict's block loop (zb_frame.c) with the LDM window and the overlay of step 5
 * behind every block's parse.  Frames of at most ZB_LDM_MIN_FRAME bytes are zbo_compress_usingDict's frames.  The
 * dictionary content serves the first chunk's history as without LDM; it is not indexed for long matches. */
size_t zbo_compress_ldm_usingDict(void* dstv, size_t cap, const void* srcv, size_t srcSize, const void* dictv, size_t dictSize,
                                  int level, const zbo_ldm_params* ldm)
{
    u8* const dst = (u8*)dstv;
    const u8* src = (const u8*)srcv;
    const u8* const dict = (const u8*)dictv;
    int const useDict = (dict != NULL) && (dictSize >= 8);
    if (srcSize <= ZB_LDM_MIN_FRAME) return zbo_compress_usingDict(dstv, cap, srcv, srcSize, dictv, dictSize, level);
    zbo_cparams const cp = zbo_getCParams_ldm(level, srcSize, useDict ? dictSize : 0);
    size_t const blockMax = ZB_BLOCK_MAX;                           /* window >= 2^20 */
    zbo_plan plan;
    zbo_dict_entropy* de = NULL;
    u8* vbuf = NULL;                 /* [dictionary content tail | src] when a dictionary is in use */
    size_t D = 0, pos;
    u32 dictID = 0;
    zbo_ldm_lists lists;
    zbo_makePlan(&plan, &cp);
    if (useDict) {
        size_t contentOff, contentSize;
        de = (zbo_dict_entropy*)malloc(sizeof(*de));
        contentOff = zbo_loadDictEntropy(de, dict, dictSize);
        if (zbo_isError(contentOff)) { free(de); return contentOff; }
        dictID = de->dictID;
        contentSize = dictSize - contentOff;
        D = contentSize < plan.primeBytes ? contentSize : plan.primeBytes;
        vbuf = (u8*)malloc(D + srcSize + 16);
        memcpy(vbuf, dict + contentOff + (contentSize - D), D);
        memcpy(vbuf + D, src, srcSize);
        src = vbuf + D;
    }
    plan.frameStart = D;
    plan.startRep[0] = plan.startRep[1] = 0;
    plan.codeRep[0] = 1; plan.codeRep[1] = 4; plan.codeRep[2] = 8;                  /* zstd_internal.h:69 */
    if (de && de->present) { plan.codeRep[0] = de->rep[0]; plan.codeRep[1] = de->rep[1]; plan.codeRep[2] = de->rep[2];
        plan.startRep[0] = de->rep[0] <= D ? de->rep[0] : 0; plan.startRep[1] = de->rep[1] <= D ? de->rep[1] : 0; }   /* zstd_compress.c:5054-5056 */
    pos = zbo_writeFrameHeader(dst, cap, cp.windowLog, srcSize, dictID);
    if (zbo_isError(pos)) { free(vbuf); free(de); return pos; }
    lists = zbo_ldm_frame(src, srcSize, cp.windowLog, ldm);             /* the frame's own bytes: no dictionary content */
    {   zbo_seq* seqs = (zbo_seq*)malloc((ZB_BLOCK_MAX / 4 + 1) * sizeof(zbo_seq));
        u8* lit = (u8*)malloc(ZB_BLOCK_MAX + 64);
        size_t const bodyCap = ZB_BLOCK_MAX * 4;
        u8* body = (u8*)malloc(bodyCap);
        size_t bs = 0, err = 0;
        int first = 1;
        u32 const none[3] = { 0, 0, 0 };
        zbo_chunkCand cc; size_t const chunkBytes = (size_t)plan.chunkBlocks * blockMax;
        memset(&cc, 0, sizeof(cc));
        while (bs < srcSize) {
            size_t const blockSize = (srcSize - bs) < blockMax ? (srcSize - bs) : blockMax;
            u32 const lastBlock = (bs + blockSize == srcSize);
            size_t cSize = 0;
            if (blockSize >= 7) {                                    /* zstd_compress.c:3216 */
                size_t litSize = 0, nbSeq, k = bs / ZB_BLOCK_MAX;
                if (cc.dS == NULL || bs + D >= cc.end) {             /* next chunk: walk it */
                    size_t const cs = bs - bs % chunkBytes;
                    size_t const ce = cs + chunkBytes < srcSize ? cs + chunkBytes : srcSize;
                    zbo_freeChunk(&cc);
                    zbo_walkChunk(&plan, src - D, srcSize + D, cs + D, ce + D, &cc);
                }
                nbSeq = zbo_parseBlock(&plan, src - D, &cc, bs + D, blockSize, seqs, lit, &litSize);
                nbSeq = zbo_ldm_overlayBlock(src + bs, blockSize, first ? plan.codeRep : none, lists.m + lists.first[k], lists.cnt[k],
                                             seqs, nbSeq, lit, &litSize);
                cSize = zbo_entropyCompressBlock_prev(body, bodyCap, seqs, nbSeq, lit, litSize, blockSize,
                                                      cp.strategy, (int)plan.litCompressionDisabled, first ? de : NULL);
                if (zbo_isError(cSize)) { err = cSize; break; }
                if (!first && cSize < 25 && isRLE(src + bs, blockSize)) { cSize = 1; body[0] = src[bs]; }   /* :4365-4376 */
            }
            if (cSize == 0) {                                          /* raw block, zstd_compress_internal.h:586 */
                u32 const h = lastBlock + (0u << 1) + (u32)(blockSize << 3);
                if (cap - pos < 3 + blockSize) { err = ZBO_ERR(ZBO_error_dstSize_tooSmall); break; }
                dst[pos] = (u8)h; dst[pos + 1] = (u8)(h >> 8); dst[pos + 2] = (u8)(h >> 16);
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
        zbo_ldm_free(&lists);
        if (err) return err;
    }
    return pos;
}

size_t zbo_compress_ldm(void* dst, size_t cap, const void* src, size_t srcSize, int level, const zbo_ldm_params* ldm)
{
    return zbo_compress_ldm_usingDict(dst, cap, src, srcSize, NULL, 0, level, ldm);
}
