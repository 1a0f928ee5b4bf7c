/* zb_prefix.c — oracle of compression against a prefix, ZSTD_CCtx_refPrefix (TEST INFRASTRUCTURE ONLY); the product's
 * frames (zstd_b200/csrc/zb_api.cu, zb_ldm.cu) are the same byte for byte.
 *
 * A prefix is raw content whatever it begins with (ZSTD_dct_rawContent, zstd_compress.c:1352), used by one frame, which
 * names dictionary ID 0.  A prefix of less than 8 bytes is ignored, as every dictionary that short is (:5132).
 *
 * Without long-distance matching it is a raw-content dictionary and no more: the frame zbo_compress_usingDict (zb_frame.c)
 * makes of the same bytes when they do not begin with the dictionary magic.
 *
 * With long-distance matching the rule of zb_ldm.c (steps 1-5 there) is extended to a second segment.  Coordinates: prefix
 * bytes [0, P), frame [P, P + n), where P counts the prefix's last min(prefixSize, 2^27) bytes: no block reaches further
 * back, so no more is indexed.  The cParams take dictSize = prefixSize as the reference does.
 *   - LDM runs when the frame is not empty and P + n > 512 KiB (P = 0: the rule of zb_ldm.c); below that the frame is the
 *     raw-dictionary frame above;
 *   - steps 1 and 2 (zbo_ldm_survivors) run on the prefix and on the frame separately: the rolling hash and the thinning
 *     never look across the seam, so the frame's survivors are the ones it has without a prefix;
 *   - step 3 is one bucket order over both sets, prefix survivors first; the window rule reads q >= max(0, block end -
 *     window) in these coordinates.  That alone keeps the frame valid: a prefix candidate inside the window of a block's
 *     end means the block ends within one window of the frame's start, which is when the format still lets a frame reach
 *     its dictionary (ZSTD_checkDictValidity, zstd_compress_internal.h:1218), and every offset stays <= 2^27;
 *   - step 4: only the frame's blocks select.  For a prefix candidate f is also capped at P - q (a match does not run from
 *     the prefix into the frame's first byte) and b at q; for a frame candidate b is capped at q - P.  Ties, anchor and
 *     "never crosses a block edge" are unchanged; the offset is p - q;
 *   - step 5 (zbo_ldm_overlayBlock) and the parse are unchanged: the first chunk has the prefix's last <= 128 KiB as
 *     history, as with any raw dictionary. */
#include <stddef.h>
#include <stdlib.h>
#include <string.h>
#include "zb_oracle.h"

/* what zb_ldm.c defines and exports for the tests (it has no header of its own) */
#define ZB_LDM_WINDOW_LOG   27u
#define ZB_LDM_MIN_FRAME    (ZB_CHUNK_BLOCKS * ZB_BLOCK_MAX)
typedef struct { u32 hashLog, minMatch, bucketSizeLog, hashRateLog; } zbo_ldm_params;
typedef struct { u32 start, len, off; } zbo_ldm_match;
typedef struct { size_t nbBlocks, nbSurvivors; u64* first; u32* cnt; zbo_ldm_match* m; } zbo_ldm_lists;
zbo_ldm_params zbo_ldm_resolve(const zbo_ldm_params* p, u32 windowLog);
size_t         zbo_ldm_survivors(const u8* src, size_t n, const zbo_ldm_params* resolved, u64* pos, u64* v);
void           zbo_ldm_free(zbo_ldm_lists* L);
size_t         zbo_ldm_overlayBlock(const u8* blk, size_t blockSize, const u32 rep[3], const zbo_ldm_match* lm, size_t nL,
                                    zbo_seq* seqs, size_t nbSeq, u8* lit, size_t* litSizePtr);
zbo_cparams    zbo_getCParams_ldm(int level, u64 srcSize, size_t dictSize);

zbo_ldm_lists  zbo_ldm_frame_usingPrefix(const u8* prefix, size_t P, const u8* src, size_t n, u32 windowLog, const zbo_ldm_params* p);
size_t         zbo_compress_usingRawDict(void* dst, size_t cap, const void* src, size_t srcSize, const void* dict, size_t dictSize, int level);
size_t         zbo_compress_ldm_usingPrefix(void* dst, size_t cap, const void* src, size_t srcSize, const void* prefix, size_t prefixSize,
                                            int level, const zbo_ldm_params* ldm);              /* ldm == NULL: LDM off */

typedef struct { u32 bucket, idx; } bkey;
static int cmp_bkey(const void* a, const void* b)              /* stable: ties by position order */
{
    const bkey* x = (const bkey*)a; const bkey* y = (const bkey*)b;
    if (x->bucket != y->bucket) return x->bucket < y->bucket ? -1 : 1;
    return x->idx < y->idx ? -1 : (x->idx > y->idx);
}

/* steps 3 and 4 for a frame src[0, n) behind P indexed prefix bytes pfx[0, P) (P = 0: zbo_ldm_frame's lists): the matches of
 * the frame's block k go to m[first[k] .. first[k] + cnt[k]).  A segment of m bytes has at most m / minMatch survivors, so
 * both sets fit (P + n) / minMatch + 1 entries. */
zbo_ldm_lists zbo_ldm_frame_usingPrefix(const u8* pfx, size_t P, const u8* src, size_t n, u32 windowLog, const zbo_ldm_params* prmIn)
{
    zbo_ldm_params const prm = zbo_ldm_resolve(prmIn, windowLog);
    size_t const cap = (P + n) / prm.minMatch + 1;
    size_t const nbBlocks = (n + ZB_BLOCK_MAX - 1) / ZB_BLOCK_MAX;
    u64* pos = (u64*)malloc(cap * sizeof(u64)); u64* v = (u64*)malloc(cap * sizeof(u64));
    size_t const NP = zbo_ldm_survivors(pfx, P, &prm, pos, v);                       /* each segment on its own bytes */
    size_t const N = NP + zbo_ldm_survivors(src, n, &prm, pos + NP, v + NP);
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
    for (i = NP; i < N; i++) pos[i] += P;
    for (i = 0; i < N; i++) { keys[i].bucket = (u32)(v[i] & (((u64)1 << bucketBits) - 1)); keys[i].idx = (u32)i; }
    qsort(keys, N, sizeof(bkey), cmp_bkey);
    for (i = 0; i < N; i++) rank[keys[i].idx] = (u32)i;
    for (k = 0; k < nbBlocks; k++) {
        size_t const bs = P + k * ZB_BLOCK_MAX, be = bs + ZB_BLOCK_MAX < P + n ? bs + ZB_BLOCK_MAX : P + n;
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
                size_t q, f, b, fmax, bmax, qroom;
                const u8* pp; const u8* qq;
                if (c.bucket != keys[rank[i]].bucket) break;
                q = pos[c.idx];
                if ((v[c.idx] >> 32) != (v[i] >> 32) || q < lowQ) continue;
                pp = src + (p - P); qq = q < P ? pfx + q : src + (q - P);
                fmax = be - p;
                if (q < P && P - q < fmax) fmax = P - q;                 /* not from the prefix into the frame's first byte */
                f = 0;
                while (f < fmax && pp[f] == qq[f]) f++;
                if (f < prm.minMatch) continue;
                qroom = q < P ? q : q - P;                             /* bytes of q's own segment in front of it */
                bmax = p - anchor < qroom ? p - anchor : qroom;
                b = 0;
                while (b < bmax && pp[-(ptrdiff_t)b - 1] == qq[-(ptrdiff_t)b - 1]) b++;
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

static int isRLE(const u8* src, size_t n)
{
    for (size_t i = 1; i < n; i++) if (src[i] != src[0]) return 0;
    return 1;
}

/* One frame against a prefix: zbo_compress_usingDict's block loop (zb_frame.c) with the prefix as raw content; where LDM
 * runs, with the LDM window and the overlay of step 5 behind every block's parse, as zbo_compress_ldm_usingDict does. */
size_t zbo_compress_ldm_usingPrefix(void* dstv, size_t cap, const void* srcv, size_t srcSize, const void* prefixv, size_t prefixSize,
                                    int level, const zbo_ldm_params* ldm)
{
    u8* const dst = (u8*)dstv;
    const u8* src = (const u8*)srcv;
    const u8* const prefix = (const u8*)prefixv;
    int const usePrefix = (prefix != NULL) && (prefixSize >= 8);
    size_t const reach = (size_t)1 << ZB_LDM_WINDOW_LOG;
    size_t const P = usePrefix ? (prefixSize < reach ? prefixSize : reach) : 0;
    int const runLdm = ldm != NULL && srcSize > 0 && P + srcSize > ZB_LDM_MIN_FRAME;
    zbo_cparams const cp = runLdm ? zbo_getCParams_ldm(level, srcSize, usePrefix ? prefixSize : 0)
                                  : zbo_getCParams(level, srcSize, usePrefix ? prefixSize : 0);
    size_t const blockMax = ((size_t)1 << cp.windowLog) < ZB_BLOCK_MAX ? ((size_t)1 << cp.windowLog) : ZB_BLOCK_MAX;   /* zstd_compress.c:2124 */
    zbo_plan plan;
    u8* vbuf = NULL;                 /* [prefix tail | src] */
    size_t D = 0, pos;
    zbo_ldm_lists lists;
    memset(&lists, 0, sizeof(lists));
    zbo_makePlan(&plan, &cp);
    if (usePrefix) {
        D = prefixSize < plan.primeBytes ? prefixSize : plan.primeBytes;
        vbuf = (u8*)malloc(D + srcSize + 16);
        memcpy(vbuf, prefix + (prefixSize - D), D);
        memcpy(vbuf + D, src, srcSize);
        src = vbuf + D;
    }
    plan.frameStart = D;
    plan.startRep[0] = plan.startRep[1] = 0;
    plan.codeRep[0] = 1; plan.codeRep[1] = 4; plan.codeRep[2] = 8;                  /* zstd_internal.h:69 */
    pos = zbo_writeFrameHeader(dst, cap, cp.windowLog, srcSize, 0);
    if (zbo_isError(pos)) { free(vbuf); return pos; }
    if (srcSize == 0) {                                    /* zstd_compress.c:5279-5295 : empty last raw block */
        free(vbuf);
        if (cap - pos < 3) return ZBO_ERR(ZBO_error_dstSize_tooSmall);
        dst[pos++] = 1; dst[pos++] = 0; dst[pos++] = 0;
        return pos;
    }
    if (runLdm) lists = zbo_ldm_frame_usingPrefix(P ? prefix + (prefixSize - P) : NULL, P, src, srcSize, cp.windowLog, ldm);
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
                size_t litSize = 0, nbSeq;
                if (cc.dS == NULL || bs + D >= cc.end) {             /* next chunk: walk it */
                    size_t const cs = bs - bs % chunkBytes;
                    size_t const ce = cs + chunkBytes < srcSize ? cs + chunkBytes : srcSize;
                    zbo_freeChunk(&cc);
                    zbo_walkChunk(&plan, src - D, srcSize + D, cs + D, ce + D, &cc);
                }
                nbSeq = zbo_parseBlock(&plan, src - D, &cc, bs + D, blockSize, seqs, lit, &litSize);
                if (runLdm) {                                        /* the window is >= 2^20: blocks of ZB_BLOCK_MAX bytes */
                    size_t const k = bs / ZB_BLOCK_MAX;
                    nbSeq = zbo_ldm_overlayBlock(src + bs, blockSize, first ? plan.codeRep : none, lists.m + lists.first[k], lists.cnt[k],
                                                 seqs, nbSeq, lit, &litSize);
                }
                cSize = zbo_entropyCompressBlock_prev(body, bodyCap, seqs, nbSeq, lit, litSize, blockSize,
                                                      cp.strategy, (int)plan.litCompressionDisabled, NULL);
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
        free(seqs); free(lit); free(body); free(vbuf);
        if (runLdm) zbo_ldm_free(&lists);
        if (err) return err;
    }
    return pos;
}

/* a dictionary taken as raw content whatever it begins with: the prefix frame with LDM off */
size_t zbo_compress_usingRawDict(void* dst, size_t cap, const void* src, size_t srcSize, const void* dict, size_t dictSize, int level)
{
    return zbo_compress_ldm_usingPrefix(dst, cap, src, srcSize, dict, dictSize, level, NULL);
}
