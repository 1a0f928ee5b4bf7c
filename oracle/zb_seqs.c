/* zb_seqs.c — oracle of the sequence entry point (ZSTD_compressSequences, lib/zstd.h:1611-1644) as the product
 * implements it (TEST INFRASTRUCTURE ONLY): the caller's sequences are validated, cut into blocks, coded with the
 * product's repcode rule and handed to the same entropy stage and block decisions as the frame driver (zb_frame.c).
 *
 * Blocks, explicit delimiters: a sequence with offset == 0 && matchLength == 0 ends a block, its litLength is the
 * block's trailing run.  An empty block produces nothing; a block above blockMax, a sum of lengths above srcSize or
 * blocks that stop short of srcSize are invalid.
 * Blocks, no delimiters: the planner's geometry (consecutive blockMax blocks).  A match part that a block edge cuts
 * stays a match when at least 3 bytes of it lie in the block, else its bytes are literals; bytes behind the last
 * sequence are literals.
 * A sequence is invalid when offset == 0, matchLength < 3 (any length >= 3 is accepted whatever ZSTD_c_minMatch says),
 * offset > (pos > window ? window : pos + dictContentSize) with pos the position behind it (zstd_compress.c:6531), or
 * offset > ZBO_SEQ_OFF_MAX (an offset code has 24 bits on the device).
 * Repcodes: history {1,4,8} (or the dictionary's) at the frame's first block, unknown at every other block, updated
 * inside a block as ZSTD_storeSeq does — the rule of the frame driver, so a frame's own stores give the frame back. */
#include <string.h>
#include <stdlib.h>
#include "zb_oracle.h"

typedef struct { u32 offset, litLength, matchLength, rep; } zbo_sequence;    /* ZSTD_Sequence, lib/zstd.h:1291-1322 */
#define ZBO_error_externalSequences_invalid 107
#define ZBO_SEQ_OFF_MAX ((1u << 24) - 4u)

static u32 repCode(u32* h, u32 off, u32 ll)             /* ZSTD_storeSeq's offBase + ZSTD_updateRep */
{
    if (ll > 0) {
        if (off == h[0]) return 1;
        if (off == h[1]) { h[1] = h[0]; h[0] = off; return 2; }
        if (off == h[2]) { h[2] = h[1]; h[1] = h[0]; h[0] = off; return 3; }
    } else {
        if (off == h[1]) { h[1] = h[0]; h[0] = off; return 1; }
        if (off == h[2]) { h[2] = h[1]; h[1] = h[0]; h[0] = off; return 2; }
        if (h[0] > 1 && off == h[0] - 1) { h[2] = h[1]; h[1] = h[0]; h[0] = off; return 3; }
    }
    h[2] = h[1]; h[1] = h[0]; h[0] = off;
    return off + 3;
}

static u32 repDecode(u32* h, u32 offBase, u32 ll)      /* the real offset behind an offBase, same history update */
{
    u32 off;
    if (offBase > 3) off = offBase - 3;
    else if (ll > 0) off = h[offBase - 1];
    else off = offBase == 3 ? h[0] - 1 : h[offBase];
    repCode(h, off, ll);
    return off;
}

static int isRLE(const u8* src, size_t n)
{
    for (size_t i = 1; i < n; i++) if (src[i] != src[0]) return 0;
    return 1;
}

typedef struct {
    zbo_cparams cp; zbo_plan plan; size_t blockMax;
    zbo_dict_entropy* de; u32 dictID; size_t dictContent;
} seqFrame;

static size_t frameSetup(seqFrame* F, size_t srcSize, const u8* dict, size_t dictSize, int level)
{
    int const useDict = dict != NULL && dictSize >= 8;
    memset(F, 0, sizeof(*F));
    F->cp = zbo_getCParams(level, srcSize, useDict ? dictSize : 0);
    F->blockMax = ((size_t)1 << F->cp.windowLog) < ZB_BLOCK_MAX ? ((size_t)1 << F->cp.windowLog) : ZB_BLOCK_MAX;
    zbo_makePlan(&F->plan, &F->cp);
    F->plan.codeRep[0] = 1; F->plan.codeRep[1] = 4; F->plan.codeRep[2] = 8;
    if (useDict) {
        size_t contentOff;
        F->de = (zbo_dict_entropy*)malloc(sizeof(*F->de));
        contentOff = zbo_loadDictEntropy(F->de, dict, dictSize);
        if (zbo_isError(contentOff)) { free(F->de); F->de = NULL; return contentOff; }
        F->dictID = F->de->dictID;
        F->dictContent = dictSize - contentOff;
        if (F->de->present) { F->plan.codeRep[0] = F->de->rep[0]; F->plan.codeRep[1] = F->de->rep[1]; F->plan.codeRep[2] = F->de->rep[2]; }
    }
    return 0;
}

/* one block behind the frame driver's rules: raw below 7 bytes or without gain, RLE except in the first block */
static size_t emitBlock(u8* dst, size_t cap, size_t pos, const u8* blk, size_t blockSize, int first, int last,
                        const zbo_seq* seqs, size_t nbSeq, const u8* lit, size_t litSize, const seqFrame* F, u8* body, size_t bodyCap)
{
    size_t cSize = 0;
    if (blockSize >= 7) {
        cSize = zbo_entropyCompressBlock_prev(body, bodyCap, seqs, nbSeq, lit, litSize, blockSize, F->cp.strategy,
                                              (int)F->plan.litCompressionDisabled, first ? F->de : NULL);
        if (zbo_isError(cSize)) return cSize;
        if (!first && cSize < 25 && isRLE(blk, blockSize)) { cSize = 1; body[0] = blk[0]; }
    }
    if (cSize == 0) {
        u32 const h = (u32)last + (0u << 1) + (u32)(blockSize << 3);
        if (cap - pos < 3 + blockSize) return ZBO_ERR(ZBO_error_dstSize_tooSmall);
        dst[pos] = (u8)h; dst[pos + 1] = (u8)(h >> 8); dst[pos + 2] = (u8)(h >> 16);
        memcpy(dst + pos + 3, blk, blockSize);
        return pos + 3 + blockSize;
    }
    {   u32 const h = (cSize == 1) ? (u32)last + (1u << 1) + (u32)(blockSize << 3) : (u32)last + (2u << 1) + (u32)(cSize << 3);
        if (cap - pos < 3 + cSize) return ZBO_ERR(ZBO_error_dstSize_tooSmall);
        dst[pos] = (u8)h; dst[pos + 1] = (u8)(h >> 8); dst[pos + 2] = (u8)(h >> 16);
        memcpy(dst + pos + 3, body, cSize);
        return pos + 3 + cSize;
    }
}

/* The stores of block [B, E): sequences from index i (which starts at position p) on, as long as they start before E.
 * Every match part of >= 3 bytes inside the block is kept, every other byte is a literal. */
static size_t convertBlock(const zbo_sequence* s, size_t n, size_t i, u64 p, u64 B, u64 E, const u8* src,
                           const u32* startHist, zbo_seq* out, u8* lit, size_t* litSize)
{
    u32 h[3] = { startHist[0], startHist[1], startHist[2] };
    u64 prevEnd = B;
    size_t nb = 0, nl = 0;
    for (; i < n && p < E; i++) {
        u64 const m = p + s[i].litLength, e = m + s[i].matchLength;
        u64 const ms = m > B ? m : B, me = e < E ? e : E;
        if (me >= ms + 3) {
            u32 const ll = (u32)(ms - prevEnd);
            memcpy(lit + nl, src + prevEnd, ll); nl += ll;
            out[nb].offBase = repCode(h, s[i].offset, ll); out[nb].litLen = ll; out[nb].matchLen = (u32)(me - ms); nb++;
            prevEnd = me;
        }
        p = e;
    }
    memcpy(lit + nl, src + prevEnd, (size_t)(E - prevEnd)); nl += (size_t)(E - prevEnd);
    *litSize = nl;
    return nb;
}

size_t zbo_compressSequences(void* dstv, size_t cap, const void* seqsv, size_t n, const void* srcv, size_t srcSize,
                             const void* dict, size_t dictSize, int level, int explicitDelims)
{
    u8* const dst = (u8*)dstv;
    const u8* const src = (const u8*)srcv;
    const zbo_sequence* const s = (const zbo_sequence*)seqsv;
    static const u32 unknown[3] = { 0, 0, 0 };
    seqFrame F;
    size_t pos, err = 0;
    {   size_t const e = frameSetup(&F, srcSize, (const u8*)dict, dictSize, level); if (zbo_isError(e)) return e; }
    /* validation, and the blocks of the explicit form */
    {   u64 const W = 1ull << F.cp.windowLog;
        u64 p = 0, blockStart = 0;
        for (size_t i = 0; i < n && !err; i++) {
            int const delim = explicitDelims && s[i].offset == 0 && s[i].matchLength == 0;
            p += (u64)s[i].litLength + s[i].matchLength;
            if (p > srcSize) err = 1;
            else if (!delim) {
                u64 const bound = p > W ? W : p + F.dictContent;
                if (s[i].offset == 0 || s[i].matchLength < 3 || s[i].offset > bound || s[i].offset > ZBO_SEQ_OFF_MAX) err = 1;
            } else if (p > blockStart) {
                if (p - blockStart > F.blockMax) err = 1;
                blockStart = p;
            }
        }
        if (!err && explicitDelims && blockStart != srcSize) err = 1;
        if (err) { free(F.de); return ZBO_ERR(ZBO_error_externalSequences_invalid); }
    }
    pos = zbo_writeFrameHeader(dst, cap, F.cp.windowLog, srcSize, F.dictID);
    if (zbo_isError(pos)) { free(F.de); return pos; }
    if (srcSize == 0) {
        free(F.de);
        if (cap - pos < 3) return ZBO_ERR(ZBO_error_dstSize_tooSmall);
        dst[pos++] = 1; dst[pos++] = 0; dst[pos++] = 0;
        return pos;
    }
    {   zbo_seq* out = (zbo_seq*)malloc((ZB_BLOCK_MAX / 3 + 8) * sizeof(zbo_seq));
        u8* lit = (u8*)malloc(ZB_BLOCK_MAX + 64);
        size_t const bodyCap = ZB_BLOCK_MAX * 4;
        u8* body = (u8*)malloc(bodyCap);
        size_t i = 0;
        u64 p = 0, B = 0;
        while (B < srcSize && !err) {
            u64 E;
            size_t first = i;
            u64 pFirst = p;
            if (explicitDelims) {            /* up to the next delimiter that closes a non-empty block */
                for (;;) {
                    int const delim = s[i].offset == 0 && s[i].matchLength == 0;
                    p += (u64)s[i].litLength + s[i].matchLength; i++;
                    if (delim && p > B) break;
                    if (delim) { first = i; pFirst = p; }   /* an empty block in front: nothing to convert */
                }
                E = p;
            } else {                         /* the first sequence that ends behind B */
                E = B + F.blockMax < srcSize ? B + F.blockMax : srcSize;
                while (i < n && p + s[i].litLength + s[i].matchLength <= B) { p += (u64)s[i].litLength + s[i].matchLength; i++; }
                first = i; pFirst = p;
            }
            {   size_t const bsz = (size_t)(E - B);
                size_t nb = 0, litSize = 0, r;
                if (bsz >= 7) nb = convertBlock(s, explicitDelims ? i : n, first, pFirst, B, E, src, B == 0 ? F.plan.codeRep : unknown, out, lit, &litSize);
                r = emitBlock(dst, cap, pos, src + B, bsz, B == 0, E == srcSize, out, nb, lit, litSize, &F, body, bodyCap);
                if (zbo_isError(r)) err = r; else pos = r;
            }
            B = E;
        }
        free(out); free(lit); free(body); free(F.de);
        if (err) return err;
    }
    return pos;
}

/* The frame driver's own per-block stores (zbo_compress_usingDict's parse) as real offsets, each block closed by a
 * delimiter that carries its trailing literals; blocks below 7 bytes are one delimiter.  Returns the number of
 * sequences written (at most cap), or an error code. */
size_t zbo_frameSequences(void* outv, size_t cap, const void* srcv, size_t srcSize, const void* dictv, size_t dictSize, int level)
{
    zbo_sequence* const out = (zbo_sequence*)outv;
    const u8* src = (const u8*)srcv;
    const u8* const dict = (const u8*)dictv;
    seqFrame F;
    u8* vbuf = NULL;
    size_t D = 0, no = 0, err = 0;
    {   size_t const e = frameSetup(&F, srcSize, dict, dictSize, level); if (zbo_isError(e)) return e; }
    if (F.de) {                                       /* [dictionary content tail | src], as the frame driver lays it out */
        size_t const contentOff = dictSize - F.dictContent;
        D = F.dictContent < F.plan.primeBytes ? F.dictContent : F.plan.primeBytes;
        vbuf = (u8*)malloc(D + srcSize + 16);
        memcpy(vbuf, dict + contentOff + (F.dictContent - D), D);
        memcpy(vbuf + D, src, srcSize);
        src = vbuf + D;
        if (F.de->present) { F.plan.startRep[0] = F.de->rep[0] <= D ? F.de->rep[0] : 0; F.plan.startRep[1] = F.de->rep[1] <= D ? F.de->rep[1] : 0; }
    }
    F.plan.frameStart = D;
    {   zbo_seq* seqs = (zbo_seq*)malloc((ZB_BLOCK_MAX / 4 + 1) * sizeof(zbo_seq));
        u8* lit = (u8*)malloc(ZB_BLOCK_MAX + 64);
        size_t bs = 0;
        zbo_chunkCand cc; size_t const chunkBytes = (size_t)F.plan.chunkBlocks * F.blockMax;
        memset(&cc, 0, sizeof(cc));
        while (bs < srcSize && !err) {
            size_t const blockSize = (srcSize - bs) < F.blockMax ? (srcSize - bs) : F.blockMax;
            size_t nbSeq = 0, litSize = 0, covered = 0;
            if (blockSize >= 7) {
                u32 h[3] = { 0, 0, 0 };
                if (bs == 0) { h[0] = F.plan.codeRep[0]; h[1] = F.plan.codeRep[1]; h[2] = F.plan.codeRep[2]; }
                if (cc.dS == NULL || bs + D >= cc.end) {
                    size_t const cs = bs - bs % chunkBytes;
                    size_t const ce = cs + chunkBytes < srcSize ? cs + chunkBytes : srcSize;
                    zbo_freeChunk(&cc);
                    zbo_walkChunk(&F.plan, src - D, srcSize + D, cs + D, ce + D, &cc);
                }
                nbSeq = zbo_parseBlock(&F.plan, src - D, &cc, bs + D, blockSize, seqs, lit, &litSize);
                if (no + nbSeq + 1 > cap) { err = ZBO_ERR(ZBO_error_dstSize_tooSmall); break; }
                for (size_t k = 0; k < nbSeq; k++) {
                    out[no].offset = repDecode(h, seqs[k].offBase, seqs[k].litLen);
                    out[no].litLength = seqs[k].litLen; out[no].matchLength = seqs[k].matchLen; out[no].rep = 0; no++;
                    covered += (size_t)seqs[k].litLen + seqs[k].matchLen;
                }
            }
            if (no + 1 > cap) { err = ZBO_ERR(ZBO_error_dstSize_tooSmall); break; }
            out[no].offset = 0; out[no].litLength = (u32)(blockSize - covered); out[no].matchLength = 0; out[no].rep = 0; no++;
            bs += blockSize;
        }
        zbo_freeChunk(&cc);
        free(seqs); free(lit);
    }
    free(vbuf); free(F.de);
    return err ? err : no;
}
