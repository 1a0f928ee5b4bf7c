/* zb_match.c — oracle model of the chunk-parallel, batch-synchronous greedy match-finder
 * (TEST INFRASTRUCTURE ONLY; the CUDA kernels in zstd_b200/csrc/zb_match.cu must reproduce it bit-for-bit).
 *
 * What it restates: the greedy single-probe LZ77 parse of ZSTD_compressBlock_fast
 * (lib/compress/zstd_fast.c:192-423) and ZSTD_compressBlock_doubleFast
 * (zstd_double_fast.c:105-323): multiplicative hash of `mls` bytes (zstd_compress_internal.h:821-861), one
 * candidate per bucket, 4-byte verification, repcode-1 probe, backward catch-up (:387-391), forward count
 * (:396), immediate repcode-2 loop (:410-420), step acceleration every 128 bytes without a match
 * (:234,342-347), position pairs (p, p+1) spaced by `step` (:225-229).
 *
 * What is different by design (the data-parallel formulation):
 *   - the frame is cut into CHUNKS of `chunkBlocks` blocks.  A chunk has a private hash table that is primed
 *     from the `primeBytes` of input in front of it (the ZSTDMT overlap idea, zstdmt_compress.c:1182-1227) and
 *     then lives through all blocks of the chunk, as the reference's table lives through a frame;
 *   - candidate lookup (phase 1, "walk") is decoupled from the greedy selection (phase 2, "parse"): the walk
 *     visits every position in BATCHES of ZB_BATCH consecutive positions.  All positions of a batch first read
 *     their bucket, then the batch's insertions are applied (the LOWEST position wins a bucket), then a position
 *     that found nothing looks again: the batch's insertion into its bucket may lie below it.  A batch is what
 *     one CTA does between two barriers; batches are sequential;
 *   - which positions a batch inserts depends on the data, not on the parse: a position that found a candidate
 *     lies inside repeated content — the reference does not insert match interiors either (zstd_fast.c:403-408
 *     inserts 2 positions per match) — and is skipped; the others follow the pattern (pos % step) < 2 where
 *     step = insStep + one per 128 positions walked since the end of the last batch that saw a candidate hit
 *     (the reference's acceleration, :234,:342-347, which makes it leave the table alone inside incompressible
 *     regions);
 *   - table entries are (key + 1) << tagBits | tag: key = the position relative to the start of the chunk's
 *     history with its offset inside the batch reversed, tag = the low hash bits; a candidate whose tag differs
 *     is dropped by the walk, so the parse never loads it;
 *   - encoder repcodes start invalid in every parse segment; entropy tables are fresh per block.
 */
#include <string.h>
#include <stdlib.h>
#include "zb_oracle.h"

static inline u64 rd64(const u8* p) { u64 v; memcpy(&v, p, 8); return v; }
static inline u32 rd32(const u8* p) { u32 v; memcpy(&v, p, 4); return v; }

/* zstd_compress_internal.h:815-861 : hash of the low `mls` bytes of an 8-byte LE load */
static const u64 prime4 = 2654435761u;
static const u64 prime5 = 889523592379ull;
static const u64 prime6 = 227718039650203ull;
static const u64 prime7 = 58295818150454627ull;
static const u64 prime8 = 0xCF1BBCDCB7A56463ull;
static inline u32 zb_hash(u64 v, u32 mls, u32 hBits)
{
    switch (mls) {
    default:
    case 4: return (u32)(((u32)v * (u32)prime4) >> (32 - hBits));
    case 5: return (u32)(((v << 24) * prime5) >> (64 - hBits));
    case 6: return (u32)(((v << 16) * prime6) >> (64 - hBits));
    case 7: return (u32)(((v << 8) * prime7) >> (64 - hBits));
    case 8: return (u32)((v * prime8) >> (64 - hBits));
    }
}

/* zstd_compress_internal.h:771-795 */
static size_t zb_count(const u8* ip, const u8* match, const u8* iend)
{
    const u8* const start = ip;
    while (ip < iend && *ip == *match) { ip++; match++; }
    return (size_t)(ip - start);
}

/* experiment knobs (tools/exp_size.py only; all zero = what the product implements) */
zbo_tunables zbo_tun = { 0, 0, 0, 0, 0, 0, 0, 0 };
unsigned long long zbo_stat_hits = 0, zbo_stat_far = 0;   /* diagnostics of the last walks (tools/ only) */

void zbo_makePlan(zbo_plan* plan, const zbo_cparams* cp)
{
    memset(plan, 0, sizeof(*plan));
    plan->strategy = cp->strategy;
    plan->windowLog = cp->windowLog;
    plan->mls = cp->minMatch < 4 ? 4 : (cp->minMatch > 8 ? 8 : cp->minMatch);
    /* Table sizes and the insertion pattern are set against the reference's compressed size on datagen P30 / P50 / P90
     * (tools/exp_size.py, DESIGN.md section 5).  An occurrence stays in the table until a different string takes its
     * bucket (positions that find a candidate are not inserted), so a table somewhat smaller than the reference's
     * holds as many useful candidates. */
    if (cp->strategy == 1) {
        u32 const hl = cp->hashLog > ZB_FAST_HASHLOG_MAX ? ZB_FAST_HASHLOG_MAX : cp->hashLog;
        plan->stepSize = cp->targetLength + !cp->targetLength + 1;     /* zstd_fast.c:200 */
        if (cp->targetLength == 0) { plan->tableN = 3u << (hl - 2); plan->insStep = 3; }
        else                       { plan->tableN = 7u << (hl - 3); plan->insStep = plan->stepSize >= 5u ? plan->stepSize - 1u : plan->stepSize; }   /* see zb_api.cu: equal periods of insertion and probing lock out of phase */
        plan->tableNLong = 0;
    } else {
        plan->stepSize = 1;
        plan->tableN = 1u << cp->chainLog;                        /* short table (zstd_double_fast.c:116) */
        if (plan->tableN > ZB_DFAST_SHORT_MAX) plan->tableN = ZB_DFAST_SHORT_MAX;
        plan->tableNLong = 1u << (cp->hashLog > ZB_DFAST_LONGLOG_MAX ? ZB_DFAST_LONGLOG_MAX : cp->hashLog);
        plan->insStep = 2;
    }
    if (zbo_tun.tableN) plan->tableN = zbo_tun.tableN;
    if (zbo_tun.tableNLong) plan->tableNLong = zbo_tun.tableNLong;
    if (zbo_tun.insStep) plan->insStep = zbo_tun.insStep;
    plan->primeBytes = zbo_tun.primeBytes ? zbo_tun.primeBytes : ZB_PRIME_DEFAULT;
    plan->chunkBlocks = zbo_tun.chunkBlocks ? zbo_tun.chunkBlocks : ZB_CHUNK_BLOCKS;
    /* zstd_compress_internal.h:621-633 */
    plan->litCompressionDisabled = (cp->strategy == 1) && (cp->targetLength > 0);
}

/* ---- phase 1: batch-synchronous candidate walk over [low, end) of buf ------------------------------
 * dist[p - outStart] for p in [outStart, end) = distance to the candidate of p, 0 if none.
 * D = index of the frame's first byte in buf (a dictionary's content lies in front of it); batches are aligned
 * on frame positions.  readEnd = one past the last readable byte.  A position is active when its 8 bytes are
 * readable and do not straddle the dictionary / frame border.
 * A bucket is one u32: (position + 1) << 11 | 11 tag bits, positions relative to `low`, 0 = empty.
 * Bucket = (hash32 * N) >> 32 (N need not be a power of two), tag = the low 11 bits of hash32. */
static void walk(const u8* buf, size_t low, size_t outStart, size_t end, size_t readEnd, size_t D,
                 u32 mls, u32 N, u32 insStep, u32* dist)
{
    u32* const table = (u32*)calloc((size_t)N, sizeof(u32));
    u32 const B = zbo_tun.batch ? zbo_tun.batch : ZB_BATCH;       /* experiments: smaller batches */
    u32 hh[ZB_BATCH], dOld[ZB_BATCH];
    u8 act[ZB_BATCH], ins[ZB_BATCH];
    /* walk coordinates: x = p - low + shift, shift chosen so that batch borders (frame positions that are multiples of
     * the batch, dictionary positions counting backwards from the frame start) are multiples of B in x */
    size_t const shift = D > low ? (B - (D - low) % B) % B : 0;
    size_t lastHit = low;                 /* last position seen whose candidate was a hit (the walk's start counts as one) */
    size_t s = low;
    /* a table entry: (key + 1) << 11 | tag, key = x with its position inside the batch reversed, so that of all
     * insertions of one batch the LOWEST position has the largest key, and any batch beats the batches before it */
#define BKT(h) ((u32)(((u64)(h) * N) >> 32))
#define KEYOF(x) (((x) & ~(B - 1u)) + (B - 1u) - ((x) & (B - 1u)))
#define CAND(c, h, x) (((c) && (((c) ^ (h)) & 0x7FFu) == 0 && KEYOF(((c) >> 11) - 1u) < (x)) ? (x) - KEYOF(((c) >> 11) - 1u) : 0u)
    while (s < end) {
        size_t e, n, i;
        u32 step;
        e = s + B - ((s - low + shift) % B);
        if (e > end) e = end;
        if (s == D) lastHit = D;          /* the frame starts with a fresh acceleration state behind a dictionary */
        n = e - s;
        /* 1. every position reads its bucket (the table as the previous batch left it) */
        for (i = 0; i < n; i++) {
            size_t const q = s + i;
            act[i] = (q + 8 <= readEnd) && !(q < D && q + 8 > D);
            dOld[i] = 0; hh[i] = 0;
            if (act[i]) {
                u32 const h = zb_hash(rd64(buf + q), mls, 32);
                hh[i] = h;
                dOld[i] = CAND(table[BKT(h)], h, (u32)(q - low + shift));
            }
        }
        /* 2. positions without a candidate enter the table on the pattern ((p - low) % step) < 2,
         *    step = insStep + one per 128 positions walked since the last hit (zstd_fast.c:234,:342-347);
         *    of the batch's insertions into one bucket the lowest position stays */
        step = insStep + (u32)((s - lastHit) >> 7);
        for (i = 0; i < n; i++) {
            size_t const q = s + i;
            /* spare bit 0 (experiments only, tools/exp_size.py): also refresh a bucket whose candidate was a hit */
            ins[i] = act[i] && (dOld[i] == 0 || (zbo_tun.spare & 1u)) && ((q - low) % step) < 2;
            if (dOld[i]) lastHit = e;             /* the acceleration restarts behind a batch that saw a hit */
        }
        for (i = 0; i < n; i++) if (ins[i]) {
            u32 const x = (u32)(s + i - low + shift);
            u32 const entry = ((KEYOF(x) + 1u) << 11) | (hh[i] & 0x7FFu);
            u32* const slot = &table[BKT(hh[i])];
            if (entry > *slot) *slot = entry;
        }
        /* 3. a position that found nothing before looks again: an insertion of this batch at a lower position may serve it */
        for (i = 0; i < n; i++) {
            size_t const q = s + i;
            u32 d = dOld[i];
            if (act[i] && d == 0) d = CAND(table[BKT(hh[i])], hh[i], (u32)(q - low + shift));
            if (q >= outStart) { dist[q - outStart] = d; if (d) zbo_stat_hits++; if (d >= 0xFFFFu) zbo_stat_far++; }
        }
        s = e;
    }
    free(table);
#undef BKT
#undef KEYOF
#undef CAND
}

void zbo_walkChunk(const zbo_plan* plan, const u8* buf, size_t bufSize, size_t chunkStart, size_t chunkEnd, zbo_chunkCand* cc)
{
    size_t const D = plan->frameStart;
    size_t low = chunkStart > plan->primeBytes ? chunkStart - plan->primeBytes : 0;
    size_t const n = chunkEnd - chunkStart;
    cc->low = low; cc->start = chunkStart; cc->end = chunkEnd;
    cc->dS = (u32*)malloc((n + 8) * sizeof(u32));
    cc->dL = NULL;
    if (plan->strategy == 2) {
        cc->dL = (u32*)malloc((n + 8) * sizeof(u32));
        walk(buf, low, chunkStart, chunkEnd, chunkEnd, D, 8, plan->tableNLong, plan->insStep, cc->dL);
    }
    walk(buf, low, chunkStart, chunkEnd, chunkEnd, D, plan->mls, plan->tableN, plan->insStep, cc->dS);
    (void)bufSize;
}
void zbo_freeChunk(zbo_chunkCand* cc) { free(cc->dS); free(cc->dL); cc->dS = cc->dL = NULL; }

/* ---- phase 2: greedy selection ----------------------------------------------------------------------
 * A block is parsed in segments of ZB_PARSE_SEG bytes, each by its own warp on the GPU.  A segment owns the
 * match START positions inside it: its parse begins at the segment's first byte with an empty repcode history,
 * but a match may run past the segment's end (up to the block's end).  The segments' raw sequences
 * (literal run, match start, length, real offset) are then joined by the merge step below. */
typedef struct { u32 ms, mlen, off; } rawseq;            /* match start (absolute), length, real offset */
typedef struct { rawseq* q; size_t n; } rawlist;

/* oldest position a match of this block may reach: the chunk's history start, and the window
 * (ZSTD_window_enforceMaxDist, zstd_compress_internal.h:1173, evaluated at the block's end like the reference) */
static size_t block_low(const zbo_plan* plan, const zbo_chunkCand* cc, size_t be)
{
    size_t const W = (size_t)1 << plan->windowLog;
    size_t low = cc->low;
    /* positions are buffer positions: with a dictionary in front, frame position 0 sits at plan->frameStart and the
     * dictionary's content is reachable while the window still covers it */
    if (be > W && be - W > low) low = be - W;
    return low;
}

/* fast: 32 probe positions per step ("lanes"): pairs (p, p+1) spaced by `step` */
static void parse_fast_segment(const zbo_plan* plan, const u8* frame, const u32* dist, size_t bs, size_t be,
                               size_t ss, size_t se, size_t lowLimit, rawlist* out)
{
    size_t ip = ss, anchor = ss, searchStart = ss;
    /* repcodes of the search start empty, except at the start of a frame's first block behind a zstd-format dictionary */
    u32 rep1 = (ss == plan->frameStart) ? plan->startRep[0] : 0, rep2 = (ss == plan->frameStart) ? plan->startRep[1] : 0;
    while (ip < se && ip + 8 <= be) {
        u32 const step = plan->stepSize + (u32)((ip - searchStart) >> 7);     /* kSearchStrength = 8, zstd_fast.c:234 */
        int winner = -1, wtype = 0, l;
        size_t probe = 0; u32 offset = 0;
        /* lowest lane with a hit wins.  Per lane: repcode-2 (only at lane 0 right after a match,
         * zstd_fast.c:410-420), then repcode-1, then the table candidate (4-byte check, :102-141). */
        for (l = 0; l < (int)ZB_WARP && winner < 0; l++) {
            size_t const p = ip + (size_t)(l >> 1) * step + (size_t)(l & 1);
            u32 cur, d;
            if (p >= se || p + 8 > be) break;
            cur = rd32(frame + p);
            d = dist[p - bs];
            if (l == 0 && ip == anchor && rep2 && rd32(frame + p - rep2) == cur) { winner = l; wtype = 3; probe = p; offset = rep2; }
            else if (rep1 && p >= lowLimit + rep1 && rd32(frame + p - rep1) == cur) { winner = l; wtype = 2; probe = p; offset = rep1; }
            else if (d && p >= lowLimit + d && rd32(frame + p - d) == cur) { winner = l; wtype = 1; probe = p; offset = d; }
        }
        if (winner < 0) { ip += (size_t)(ZB_WARP / 2) * step; continue; }
        {   size_t ms = probe, mm = probe - offset, mlen;
            if (wtype != 3)           /* backward catch-up (zstd_fast.c:387-391); a repcode-2 hit starts at the anchor */
                while (ms > anchor && mm > lowLimit && frame[ms - 1] == frame[mm - 1]) { ms--; mm--; }
            mlen = (probe - ms) + 4 + zb_count(frame + probe + 4, frame + probe - offset + 4, frame + be);
            if (wtype == 3) { u32 const t = rep2; rep2 = rep1; rep1 = t; }
            else if (wtype == 1) { rep2 = rep1; rep1 = offset; }
            out->q[out->n].ms = (u32)ms; out->q[out->n].mlen = (u32)mlen; out->q[out->n].off = offset; out->n++;
            ip = ms + mlen; anchor = ip; searchStart = ip;
        }
    }
}

/* doubleFast (zstd_double_fast.c:105-323): per probe position p the reference's order is kept: repcode-1 at p+1
 * (:190-195), long match at p (8 equal bytes, :206-213), short match at p (4 equal bytes, :222-225) upgraded to the
 * long match at p+1 when that one is longer (:254-271).  32 probe positions per step, spaced by `step` (1, +1 every
 * 256 bytes without a match, kStepIncr :131), lowest lane wins; immediate repcode-2 at lane 0 right after a match
 * (:302-316). */
static void parse_dfast_segment(const zbo_plan* plan, const u8* frame, const u32* distL, const u32* distS, size_t bs, size_t be,
                                size_t ss, size_t se, size_t lowLimit, rawlist* out)
{
    size_t ip = ss, anchor = ss, searchStart = ss;
    u32 rep1 = (ss == plan->frameStart) ? plan->startRep[0] : 0, rep2 = (ss == plan->frameStart) ? plan->startRep[1] : 0;
    while (ip < se && ip + 9 <= be) {                        /* a lane reads 8 bytes at p and at p+1 */
        u32 const step = 1 + (u32)((ip - searchStart) >> 8);
        int found = 0, wtype = 0, l;
        size_t ms = 0; u32 offset = 0; size_t mlen = 0;
        for (l = 0; l < (int)ZB_WARP && !found; l++) {
            size_t const p = ip + (size_t)l * step;
            u32 dl, ds, dl1;
            if (p >= se || p + 9 > be) break;
            dl = distL[p - bs]; ds = distS[p - bs]; dl1 = distL[p + 1 - bs];
            if (dl && p < lowLimit + dl) dl = 0;
            if (ds && p < lowLimit + ds) ds = 0;
            if (dl1 && p + 1 < lowLimit + dl1) dl1 = 0;
            if (l == 0 && ip == anchor && rep2 && rd32(frame + p - rep2) == rd32(frame + p)) {
                found = 1; wtype = 3; ms = p; offset = rep2;
                mlen = 4 + zb_count(frame + p + 4, frame + p + 4 - rep2, frame + be);
            } else if (rep1 && p + 1 >= lowLimit + rep1 && rd32(frame + p + 1 - rep1) == rd32(frame + p + 1)) {
                found = 1; wtype = 2; ms = p + 1; offset = rep1;
                mlen = 4 + zb_count(frame + p + 5, frame + p + 5 - rep1, frame + be);
            } else if (dl && rd64(frame + p - dl) == rd64(frame + p)) {
                size_t mm;
                found = 1; wtype = 1; ms = p; offset = dl;
                mlen = 8 + zb_count(frame + p + 8, frame + p + 8 - offset, frame + be);
                mm = ms - offset;
                while (ms > anchor && mm > lowLimit && frame[ms - 1] == frame[mm - 1]) { ms--; mm--; mlen++; }
            } else if (ds && rd32(frame + p - ds) == rd32(frame + p)) {
                size_t mm;
                found = 1; wtype = 1; ms = p; offset = ds;
                mlen = 4 + zb_count(frame + p + 4, frame + p + 4 - offset, frame + be);
                if (dl1 && rd64(frame + p + 1 - dl1) == rd64(frame + p + 1)) {
                    size_t const l1 = 8 + zb_count(frame + p + 9, frame + p + 9 - dl1, frame + be);
                    if (l1 > mlen) { ms = p + 1; offset = dl1; mlen = l1; }
                }
                mm = ms - offset;
                while (ms > anchor && mm > lowLimit && frame[ms - 1] == frame[mm - 1]) { ms--; mm--; mlen++; }
            }
        }
        if (!found) { ip += (size_t)ZB_WARP * step; continue; }
        if (wtype == 3) { u32 const t = rep2; rep2 = rep1; rep1 = t; }
        else if (wtype == 1) { rep2 = rep1; rep1 = offset; }
        out->q[out->n].ms = (u32)ms; out->q[out->n].mlen = (u32)mlen; out->q[out->n].off = offset; out->n++;
        ip = ms + mlen; anchor = ip; searchStart = ip;
    }
}

/* ---- merge: joins the segments of a block -----------------------------------------------------------
 * `cur` = first byte not yet covered by a sequence.  A raw sequence that ends at or before `cur` (it lies under a
 * match that ran over from an earlier segment) is dropped; one that straddles `cur` keeps its tail when that is at
 * least 3 bytes (MINMATCH, zstd_internal.h:102), else it is dropped too; the others take their literals from `cur`.
 * Then the repcode history is run over the whole block (what ZSTD_storeSeq / ZSTD_updateRep do sequence by sequence
 * in the reference, zstd_compress_internal.h:671-760): it starts as {1,4,8} in the first block of a frame (zstd_internal.h:69;
 * the dictionary's repcodes behind a zstd-format dictionary) and unknown (0 = never matches) in every other block,
 * because blocks are compressed independently of each other. */
size_t zbo_parseBlock(const zbo_plan* plan, const u8* frame, const zbo_chunkCand* cc,
                      size_t bs, size_t blockSize, zbo_seq* seqs, u8* lit, size_t* litSizePtr)
{
    size_t const be = bs + blockSize;
    size_t const lowLimit = block_low(plan, cc, be);
    rawlist rl;
    size_t ss, cur = bs, nbSeq = 0, litSize = 0, i, first = 0;
    u32 r1 = 0, r2 = 0, r3 = 0;
    rl.q = (rawseq*)malloc((blockSize / 3 + 64) * sizeof(rawseq)); rl.n = 0;
    if (bs == plan->frameStart) { r1 = plan->codeRep[0]; r2 = plan->codeRep[1]; r3 = plan->codeRep[2]; }
    for (ss = bs; ss < be; ss += ZB_PARSE_SEG) {
        size_t const se = (be - ss > ZB_PARSE_SEG) ? ss + ZB_PARSE_SEG : be;
        first = rl.n;
        if (plan->strategy == 2) parse_dfast_segment(plan, frame, cc->dL + (bs - cc->start), cc->dS + (bs - cc->start), bs, be, ss, se, lowLimit, &rl);
        else                     parse_fast_segment(plan, frame, cc->dS + (bs - cc->start), bs, be, ss, se, lowLimit, &rl);
        for (i = first; i < rl.n; i++) {
            size_t ms = rl.q[i].ms, mlen = rl.q[i].mlen;
            u32 const off = rl.q[i].off;
            size_t ll;
            u32 offBase;
            if (ms + mlen <= cur) continue;
            if (ms < cur) { if (ms + mlen - cur < 3) continue; mlen = ms + mlen - cur; ms = cur; }
            ll = ms - cur;
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
            memcpy(lit + litSize, frame + cur, ll); litSize += ll;
            seqs[nbSeq].offBase = offBase; seqs[nbSeq].litLen = (u32)ll; seqs[nbSeq].matchLen = (u32)mlen; nbSeq++;
            cur = ms + mlen;
        }
    }
    /* trailing literals (zstd_compress.c:3365-3366) */
    memcpy(lit + litSize, frame + cur, be - cur); litSize += be - cur;
    *litSizePtr = litSize;
    free(rl.q);
    return nbSeq;
}
