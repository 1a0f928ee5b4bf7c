/* zb_decode.cu — GPU decompression of zstd frames (SURVEY.md 8f rank 2): the other half of the block pipeline.
 *
 * Replaces, with a block-parallel formulation, what the reference does serially per frame:
 *   ZSTD_decompress / ZSTD_decompressDCtx / ZSTD_decompressFrame  (lib/decompress/zstd_decompress.c:1011-1124)
 *   ZSTD_decodeLiteralsBlock, ZSTD_decodeSeqHeaders, ZSTD_decompressSequences_body, ZSTD_execSequence
 *                                                     (lib/decompress/zstd_decompress_block.c:343, :695, :1615, :1012)
 *   HUF_decompress4X1 / HUF_readDTableX1              (lib/decompress/huf_decompress.c:602, :383)
 * Any frame the format allows is accepted (this library's own and the reference encoder's, every level), window
 * sizes up to 128 MiB, raw-content and zstd-format dictionaries (ZSTD_decompress_usingDict, zstd_decompress.c:1133).
 * Offsets are kept in 28 bits: a frame whose offsets need more than 27 bits gets frameParameter_windowTooLarge (16)
 * whatever its header says (a window descriptor above 2^27 from the walk; a Single_Segment frame, which states no window,
 * from the first such offset code).
 * The format-level functions are in zb_decode_core.cuh.
 *
 *   D0  walker    frames and blocks of the input: block headers, section headers, which earlier block a treeless /
 *                 repeat-mode block takes its tables from.  Host code for host buffers and for device buffers up to
 *                 512 MiB (walked in a page-locked copy); one device thread per call for larger device buffers (a chain
 *                 of dependent 3-byte reads).
 *   D1  literals  one warp per block: raw / RLE copied, Huffman tree description -> decoding table in shared memory
 *                 (a block that reuses a table re-reads the description of the block that defined it: no dependency
 *                 between CTAs), the 1 or 4 streams decoded by one lane each.
 *   D2  sequences one warp per block: the three FSE decoding tables by three lanes, the interleaved bitstream by one
 *                 lane; emits packed (offset code, literal length, match length), the block's regenerated size and
 *                 its repcode history as a FUNCTION of the history at its start.
 *   D3  scan      output offset of every block (prefix sum of regenerated sizes) and the repcode history at every
 *                 block's start (composition of the blocks' functions along each frame).
 *   D4  place     one warp per block, all blocks at once: raw / RLE blocks and every literal run go to their final place,
 *                 every match becomes (destination, offset, length) with its repcode resolved.  Nothing of the output is
 *                 read, so no block waits for another.
 *   D5  matches   LZ77 copies read earlier output, which chains the matches of a frame — but a match depends only on the
 *                 few matches that wrote its source bytes.  One CTA per frame, one LANE per match, matches handed out in
 *                 order; a lane finds the writers of its source range through a tile index D4 left behind, waits for their
 *                 completion flags (block-scope fences: writer and reader share an SM), copies, raises its own.  What stays
 *                 serial is the longest chain of matches copying from one another; frames run side by side.
 */
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <vector>
#include <new>
#include "../../include/zstd_b200.h"
#include "zb_common.h"
#include "zb_decode_core.cuh"

#define ZB_FULL 0xFFFFFFFFu
#define ZBD_HOSTWALK_MAX ((size_t)512 << 20)   /* device-resident inputs up to this size have their headers walked on the host (zbd_decompress) */
#define ZBD_WARPS 4                    /* blocks per CTA in D1 / D2 / D4 */

/* per block, written by D2 and D3 */
typedef struct {
    u32 regen;             /* regenerated size of the block */
    u32 err;               /* 0 or a ZSTD error code */
    u32 sumLL;
    u32 pad;
    ZbdRep transfer;       /* history at the block's end as a function of the history at its start */
    ZbdRep start;          /* history at the block's start (D3) */
    u64 dstOff;            /* first output byte of the block (D3) */
    u64 frameOff;          /* first output byte of its frame (D3) */
} ZbdBlockOut;

/* ------------------------------------------------------------------------------------------------ D0 on the device */
__global__ void zbd_walk_kernel(const u8* __restrict__ src, u64 size, ZbdBlock* blocks, u32 capB, ZbdFrame* frames, u32 capF, u64* res, u32 dictEntropy, u32 dictID)
{
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    u32 nb = 0, nf = 0; u64 lit = 0, seq = 0;
    u32 const e = zbd_walk(src, size, blocks, capB, frames, capF, &nb, &nf, &lit, &seq, dictEntropy != 0u, dictID);
    res[0] = e; res[1] = nb; res[2] = nf; res[3] = lit; res[4] = seq;
}

/* ------------------------------------------------------------------------------------------------ D1 literals */
struct ZbdLitWork {
    u16 table[1u << ZBD_HUF_LOG_MAX];
    u16 start[256];
    u8  weights[256];
    u32 fse[64];
    short norm[16];
    u16 next[16];
    u32 nbSym, log, used;
};

__global__ void __launch_bounds__(32 * ZBD_WARPS)
zbd_literals_kernel(const u8* __restrict__ src, const ZbdBlock* __restrict__ blocks, u32 nbBlocks, u8* __restrict__ lits, ZbdBlockOut* __restrict__ bout,
                    const u8* __restrict__ dict, ZbdDictInfo di)
{
    __shared__ ZbdLitWork work[ZBD_WARPS];
    u32 const lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
    u32 const bi = blockIdx.x * ZBD_WARPS + w;
    if (bi >= nbBlocks) return;
    ZbdBlock const b = blocks[bi];
    if (lane == 0) bout[bi].err = 0;
    if (b.type != ZB_BT_COMPRESSED) return;
    ZbdLitWork& wk = work[w];
    const u8* const c = src + b.srcOff;
    u8* const out = lits + b.litPos;
    if (b.litType == 0u) { for (u32 i = lane; i < b.litRegen; i += 32u) out[i] = c[b.litHdr + i]; return; }
    if (b.litType == 1u) { u8 const v = c[b.litHdr]; for (u32 i = lane; i < b.litRegen; i += 32u) out[i] = v; return; }
    if (lane == 0) {
        u32 nbSym = 0, log = 0, dn = 0;
        const u8* const dp = zbd_hufDescription(&b, blocks, src, dict, &di, &dn);
        u32 const used = zbd_readHufWeights(wk.weights, &nbSym, &log, dp, dn, wk.fse, wk.norm, wk.next);
        if (used) zbd_hufStarts(wk.start, wk.weights, nbSym, log);
        wk.nbSym = nbSym; wk.log = log; wk.used = used;
    }
    __syncwarp();
    u32 const used = wk.used, log = wk.log, nbSym = wk.nbSym;
    if (!used) { if (lane == 0) bout[bi].err = ZBD_CORRUPT; return; }
    for (u32 s = 0; s < nbSym; s++) zbd_hufFill(wk.table, s, wk.start[s], wk.weights[s], log, lane, 32u);
    __syncwarp();
    u32 const desc = b.litType == 3u ? 0u : used;                  /* treeless: the streams follow the header directly */
    u32 err = 0;
    if (desc > b.litComp) err = ZBD_CORRUPT;
    const u8* const s = c + b.litHdr + desc;
    u32 const total = b.litComp - desc;
    if (!err) {
        if (b.litStreams == 1u) { if (lane == 0) err = zbd_hufDecodeStream(out, b.litRegen, s, total, wk.table, log); }
        else {
            u32 off[4], sz[4], cnt[4];
            err = zbd_litStreams(off, sz, cnt, s, total, b.litRegen);
            if (!err && lane < 4u) {
                u32 o = 0, n = 0, k = 0;                             /* lane k's stream, selected: no array indexed by the lane */
#pragma unroll
                for (u32 j = 0; j < 4u; j++) if (lane == j) { o = off[j]; n = sz[j]; k = cnt[j]; }
                err = zbd_hufDecodeStream(out + lane * cnt[0], k, s + o, n, wk.table, log);
            }
        }
    }
    err = __reduce_max_sync(ZB_FULL, err);
    if (err && lane == 0) bout[bi].err = err;
}

/* ------------------------------------------------------------------------------------------------ D2 sequences */
struct ZbdSeqWork {
    u32 table[3][512];     /* LL (<= 512 cells), OF (<= 256), ML (<= 512) */
    short norm[3][64];
    u16 next[3][64];
    int log[3];            /* -1: the table's description is corrupt */
};

__global__ void __launch_bounds__(32 * ZBD_WARPS)
zbd_sequences_kernel(const u8* __restrict__ src, const ZbdBlock* __restrict__ blocks, u32 nbBlocks, u64* __restrict__ seqs, ZbdBlockOut* __restrict__ bout,
                     const u8* __restrict__ dict, ZbdDictInfo di)
{
    __shared__ ZbdSeqWork work[ZBD_WARPS];
    u32 const lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
    u32 const bi = blockIdx.x * ZBD_WARPS + w;
    if (bi >= nbBlocks) return;
    ZbdBlock const b = blocks[bi];
    ZbdSeqWork& wk = work[w];
    ZbdRep ident; ident.r[0] = ZBD_SYM(0u, 0u); ident.r[1] = ZBD_SYM(1u, 0u); ident.r[2] = ZBD_SYM(2u, 0u);
    if (b.type != ZB_BT_COMPRESSED || b.nbSeq == 0u) {
        if (lane == 0) { ZbdBlockOut& o = bout[bi]; o.regen = b.type == ZB_BT_COMPRESSED ? b.litRegen : b.rawSize; o.sumLL = 0; o.transfer = ident; }
        return;
    }
    /* three lanes: one decoding table each, from the section that defined it */
    if (lane < 3u) wk.log[lane] = zbd_seqTable(wk.table[lane], wk.norm[lane], wk.next[lane], lane, &b, blocks, src, dict, &di);
    __syncwarp();
    if (lane == 0) {
        ZbdBlockOut& o = bout[bi];
        u32 e = (wk.log[0] | wk.log[1] | wk.log[2]) < 0 ? ZBD_CORRUPT : 0u;
        u32 sumLL = 0, sumML = 0; ZbdRep tr = ident;
        if (!e) {
            const u8* const sec = src + b.srcOff + b.seqOff;
            u32 const avail = b.cSize - b.seqOff;
            u32 desc[3], bitstream;
            if (zbd_locateDescriptions(&b, sec, avail, desc, &bitstream, wk.norm[0])) e = ZBD_CORRUPT;
            else e = zbd_decodeSequences(seqs + b.seqPos, b.nbSeq, sec + bitstream, avail - bitstream, wk.table[0], wk.log[0], wk.table[1], wk.log[1],
                                         wk.table[2], wk.log[2], &sumLL, &sumML, &tr);
            if (!e && (sumLL > b.litRegen || b.litRegen + sumML > ZB_BLOCK_MAX)) e = ZBD_CORRUPT;
        }
        o.regen = e ? 0u : b.litRegen + sumML; o.sumLL = sumLL; o.transfer = tr;
        if (e) o.err = e;
    }
}

/* ------------------------------------------------------------------------------------------------ D3 scan
 * One CTA.  Output offsets: prefix sum over all blocks of the call (frames are laid out back to back).  Histories: one
 * warp per frame walks its blocks, 32 transfer functions per round.  res[0] = first error, res[1] = total output bytes. */
#define SCAN_THREADS 1024
__global__ void __launch_bounds__(SCAN_THREADS)
zbd_scan_kernel(const ZbdBlock* __restrict__ blocks, u32 nbBlocks, const ZbdFrame* __restrict__ frames, u32 nbFrames, ZbdBlockOut* __restrict__ bout,
                u64 dstCapacity, u64* __restrict__ res, ZbdDictInfo di)
{
    __shared__ u64 warpSum[SCAN_THREADS / 32];
    __shared__ u64 carry;
    __shared__ u32 firstErr;
    u32 const tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    if (tid == 0) { carry = 0; firstErr = 0; }
    __syncthreads();
    for (u32 b0 = 0; b0 < nbBlocks; b0 += SCAN_THREADS) {
        u32 const i = b0 + tid;
        u64 v = 0;
        if (i < nbBlocks) { v = bout[i].regen; if (bout[i].err) atomicMax(&firstErr, bout[i].err); }
        u64 inc = v;
#pragma unroll
        for (u32 o = 1; o < 32u; o <<= 1) { u64 const x = __shfl_up_sync(ZB_FULL, inc, o); if (lane >= o) inc += x; }
        if (lane == 31u) warpSum[warp] = inc;
        __syncthreads();
        u64 base = carry;
        for (u32 k = 0; k < warp; k++) base += warpSum[k];
        if (i < nbBlocks) bout[i].dstOff = base + inc - v;
        __syncthreads();
        if (tid == SCAN_THREADS - 1u) carry = base + inc;
        __syncthreads();
    }
    u64 const total = carry;
    u32 const blockErr = firstErr;                                   /* a block that failed has no size: no content-size check over it hides its code */
    __syncthreads();
    /* per frame: content size, start offset, repcode histories */
    for (u32 f = warp; f < nbFrames; f += SCAN_THREADS / 32u) {
        ZbdFrame const fr = frames[f];
        u64 const fOff = fr.nbBlocks ? bout[fr.firstBlock].dstOff : 0;
        ZbdRep h; h.r[0] = 1u; h.r[1] = 4u; h.r[2] = 8u;            /* format: "Repeat Offsets" start values */
        if (di.entropy) { h.r[0] = di.rep[0]; h.r[1] = di.rep[1]; h.r[2] = di.rep[2]; }      /* ... or the dictionary's */
        for (u32 k0 = 0; k0 < fr.nbBlocks; k0 += 32u) {
            u32 const k = k0 + lane;
            ZbdRep tr; tr.r[0] = tr.r[1] = tr.r[2] = 0;
            if (k < fr.nbBlocks) tr = bout[fr.firstBlock + k].transfer;
            ZbdRep mine = h;
            u32 const n = min(32u, fr.nbBlocks - k0);
            for (u32 j = 0; j < n; j++) {
                if (lane == j) mine = h;                             /* history at the start of block k0 + j */
                ZbdRep t; t.r[0] = __shfl_sync(ZB_FULL, tr.r[0], (int)j); t.r[1] = __shfl_sync(ZB_FULL, tr.r[1], (int)j); t.r[2] = __shfl_sync(ZB_FULL, tr.r[2], (int)j);
                ZbdRep nx; nx.r[0] = zbd_rep_resolve(t.r[0], &h); nx.r[1] = zbd_rep_resolve(t.r[1], &h); nx.r[2] = zbd_rep_resolve(t.r[2], &h);
                h = nx;
            }
            if (k < fr.nbBlocks) { ZbdBlockOut& o = bout[fr.firstBlock + k]; o.start = mine; o.frameOff = fOff; }
        }
        if (lane == 0 && !blockErr && fr.contentSize != ZBD_CONTENTSIZE_UNKNOWN) {
            u64 const end = (fr.firstBlock + fr.nbBlocks < nbBlocks) ? bout[fr.firstBlock + fr.nbBlocks].dstOff : total;
            if (end - fOff != fr.contentSize) atomicMax(&firstErr, ZBD_CORRUPT);
        }
    }
    __syncthreads();
    if (tid == 0) {
        u32 e = firstErr;
        if (!e && total > dstCapacity) e = 70u;                      /* dstSize_tooSmall */
        res[0] = e; res[1] = total;
    }
}

/* ------------------------------------------------------------------------------------------------ D4 place
 * One warp per block, every block of the call at once: raw / RLE blocks are written; of a compressed block every literal run
 * goes to its final place and every match becomes (absolute destination, offset, length) — the repcode history runs over the
 * block's sequences from the start history D3 computed.  No byte of the output is READ here, so blocks do not depend on
 * each other.  A match that begins in the dictionary's content gets those bytes here and continues as an ordinary match
 * behind them.  seqs[g] becomes offset | length << 28, matchPos[g] the match's first output byte, and for every 64-byte
 * tile of the output tileFirst[] the first match (in the call's match order) that ends behind the tile's first byte:
 * what D5 needs to find the matches a source range depends on. */
#define ZBD_TILE_LOG 6u
__global__ void __launch_bounds__(32 * ZBD_WARPS)
zbd_place_kernel(const u8* __restrict__ src, const ZbdBlock* __restrict__ blocks, u32 nbBlocks, const u8* __restrict__ lits, u64* __restrict__ seqs,
                 u64* __restrict__ matchPos, u32* __restrict__ tileFirst, const ZbdBlockOut* __restrict__ bout, u8* __restrict__ dst,
                 const u8* __restrict__ dictContent, u32 dictContentSize, u32* __restrict__ execErr)
{
    u32 const lane = threadIdx.x & 31u;
    u32 const bi = blockIdx.x * ZBD_WARPS + (threadIdx.x >> 5);
    if (bi >= nbBlocks) return;
    ZbdBlock const b = blocks[bi];
    ZbdBlockOut const o = bout[bi];
    u8* const out = dst + o.dstOff;
    u32 const gFirst = (u32)b.seqPos;                                /* the call's match order: blocks in input order */
    u32 const gNext = gFirst + (b.type == ZB_BT_COMPRESSED ? b.nbSeq : 0u);
    /* tiles whose first byte lies in (lo, hi] of the output belong to match g */
    auto tiles = [&](u64 lo, u64 hi, u32 g) {
        for (u64 t = (lo >> ZBD_TILE_LOG) + 1u + lane; (t << ZBD_TILE_LOG) <= hi; t += 32u) tileFirst[t] = g;
    };
    if (b.type != ZB_BT_COMPRESSED) {
        if (b.type == ZB_BT_RAW) { for (u32 i = lane; i < b.rawSize; i += 32u) out[i] = src[b.srcOff + i]; }
        else { u8 const v = src[b.srcOff]; for (u32 i = lane; i < b.rawSize; i += 32u) out[i] = v; }
        if (o.dstOff == 0 && lane == 0) tileFirst[0] = gNext;
        tiles(o.dstOff, o.dstOff + o.regen, gNext);                  /* no match ends in here: the next block's first one is the first behind these tiles */
        return;
    }
    const u8* const lit = lits + b.litPos;
    u64* const sq = seqs + b.seqPos;
    u64* const mp = matchPos + b.seqPos;
    ZbdRep rep = o.start;
    u64 const inFrame = o.dstOff - o.frameOff;                       /* bytes of the frame in front of this block */
    u32 op = 0, lp = 0, err = 0, failedAt = 0;
    if (o.dstOff == 0 && lane == 0) tileFirst[0] = gFirst;
    for (u32 i0 = 0; i0 < b.nbSeq; i0 += 32u) {
        u32 const n = min(32u, b.nbSeq - i0);
        u64 const q = (lane < n) ? sq[i0 + lane] : 0ull;
        u32 const myLL = ZBD_SEQ_LL(q);
        u32 myML = ZBD_SEQ_ML(q), myOff = 0, myOp = 0, myLp = 0;
        /* the history and the positions are a serial walk (warp-uniform); lane j keeps sequence j's numbers */
        for (u32 j = 0; j < n; j++) {
            u32 const ob = __shfl_sync(ZB_FULL, ZBD_SEQ_OFF(q), (int)j), ll = __shfl_sync(ZB_FULL, myLL, (int)j), ml = __shfl_sync(ZB_FULL, myML, (int)j);
            u32 const off = zbd_rep_apply(&rep, ob, ll, false);
            if (lane == j) { myOff = off; myOp = op; myLp = lp; }
            op += ll;
            if (!err && (off == 0u || (u64)off > inFrame + op + dictContentSize)) { err = ZBD_CORRUPT; failedAt = i0 + j; }
            op += ml; lp += ll;
        }
        if (err) break;
        /* the literal runs: one after the other, 32 bytes a step */
        for (u32 j = 0; j < n; j++) {
            u32 const ll = __shfl_sync(ZB_FULL, myLL, (int)j), to = __shfl_sync(ZB_FULL, myOp, (int)j), from = __shfl_sync(ZB_FULL, myLp, (int)j);
            for (u32 k = lane; k < ll; k += 32u) out[to + k] = lit[from + k];
        }
        if (lane < n) {
            u32 mpos = myOp + myLL;                                  /* block-relative first byte of the match */
            u64 const here = inFrame + mpos;                          /* its frame position */
            if ((u64)myOff > here) {                                 /* begins in the dictionary: those bytes now, the rest is a match of the same offset */
                u32 const fromDict = (u32)((u64)myOff - here) < myML ? (u32)((u64)myOff - here) : myML;
                const u8* const dp = dictContent + dictContentSize - ((u64)myOff - here);
                for (u32 k = 0; k < fromDict; k++) out[mpos + k] = dp[k];
                mpos += fromDict; myML -= fromDict;
            }
            sq[i0 + lane] = (u64)myOff | ((u64)myML << 28);
            mp[i0 + lane] = o.dstOff + mpos;
            /* tiles that begin in (end of the match before, end of this match] */
            u64 const lo = o.dstOff + myOp, hi = o.dstOff + myOp + myLL + ZBD_SEQ_ML(q);
            for (u64 t = (lo >> ZBD_TILE_LOG) + 1u; (t << ZBD_TILE_LOG) <= hi; t++) tileFirst[t] = gFirst + i0 + lane;
        }
    }
    if (err) {                                                       /* the call fails; D5 must not follow what is left of this block */
        for (u32 i = failedAt - (failedAt % 32u) + lane; i < b.nbSeq; i += 32u) { sq[i] = 1ull; mp[i] = o.dstOff; }
        if (lane == 0) atomicMax(execErr, err);
        tiles(o.dstOff, o.dstOff + o.regen, gNext);
        return;
    }
    u32 const rest = b.litRegen - lp;
    for (u32 k = lane; k < rest; k += 32u) out[op + k] = lit[lp + k];
    tiles(o.dstOff + op, o.dstOff + o.regen, gNext);                 /* behind the block's last match */
}

/* ------------------------------------------------------------------------------------------------ D5 matches
 * LZ77 copies read earlier output, which makes a frame a chain; but a match only depends on the few matches that WROTE
 * its source bytes (literals are in place since D4).  So: one LANE per match, matches handed out in order, 32 at a time
 * per warp over a ticket counter (a match only ever waits for matches with lower numbers, which have been handed out).
 * A lane looks up, through tileFirst[], the range of matches that may have written [source, source + length), waits for
 * their completion flags, copies, raises its own flag.  Independent matches — nearly all of them when offsets exceed a
 * few hundred bytes — run in parallel across the whole GPU; what remains serial is the longest chain of matches that copy
 * from one another.  dst[p + k] = history[p - off + (k mod off)]. */
/* Hand-overs stay inside one CTA (a frame's matches are one CTA's), i.e. inside one SM and its L1: flags are read and
 * written with CTA-scope relaxed accesses (they may be served by that L1), the copied bytes with ordinary loads — a line
 * that was cached before a neighbouring warp wrote into it is updated by that write, both go through the same L1 — and
 * block-scope fences order the two.  ZBD_LD_L2 = 1 routes everything through L2 instead (development switch). */
#ifndef ZBD_LD_L2
#define ZBD_LD_L2 0
#endif
__device__ __forceinline__ u32 zbd_ld_flag(const u8* p)
{
    u32 v;
#if ZBD_LD_L2
    asm volatile("ld.volatile.global.u8 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
#else
    asm volatile("ld.relaxed.cta.global.u8 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
#endif
    return v;
}
__device__ __forceinline__ void zbd_st_flag(u8* p)
{
#if ZBD_LD_L2
    asm volatile("st.volatile.global.u8 [%0], %1;" :: "l"(p), "r"(1u) : "memory");
#else
    asm volatile("st.relaxed.cta.global.u8 [%0], %1;" :: "l"(p), "r"(1u) : "memory");
#endif
}
__device__ __forceinline__ u32 zbd_ldcg32(const u8* alignedWord)
{
#if ZBD_LD_L2
    return __ldcg(reinterpret_cast<const u32*>(alignedWord));
#else
    u32 v; asm volatile("ld.relaxed.cta.global.u32 %0, [%1];" : "=r"(v) : "l"(alignedWord) : "memory"); return v;
#endif
}
__device__ __forceinline__ u32 zbd_ld8(const u8* p)
{
#if ZBD_LD_L2
    return __ldcg(p);
#else
    u32 v; asm volatile("ld.relaxed.cta.global.u8 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v;
#endif
}

/* n bytes from `from` to `out`, the two ranges not overlapping.  Sources are read through L2 (another warp wrote them a
 * moment ago); what limits a copy is the number of DEPENDENT round trips, so loads go out in groups: the head bytes that
 * align the destination, then 32 bytes (nine aligned words) at a time, then the tail.  A source word is only loaded when it
 * holds a needed byte. */
__device__ __forceinline__ void zbd_copy_disjoint(u8* out, const u8* from, u32 n)
{
    u32 head = (4u - ((u32)(uintptr_t)out & 3u)) & 3u; head = head < n ? head : n;
    {   u32 const b0 = head > 0u ? zbd_ld8(from) : 0u, b1 = head > 1u ? zbd_ld8(from + 1) : 0u, b2 = head > 2u ? zbd_ld8(from + 2) : 0u;
        if (head > 0u) out[0] = (u8)b0; if (head > 1u) out[1] = (u8)b1; if (head > 2u) out[2] = (u8)b2; }
    u32 k = head;
    while (k + 4u <= n) {                                         /* destination word-aligned from here */
        u32 const words = (n - k) / 4u < 8u ? (n - k) / 4u : 8u;  /* this round: up to 8 words */
        const u8* const a = from + k;
        const u8* const aw = (const u8*)((uintptr_t)a & ~(uintptr_t)3);
        u32 const sh = ((u32)(uintptr_t)a & 3u) * 8u;
        u32 w[9];
#pragma unroll
        for (u32 i = 0; i < 9u; i++) w[i] = (i < words || (i == words && sh)) ? zbd_ldcg32(aw + 4u * i) : 0u;
        u32* const o = reinterpret_cast<u32*>(out + k);
#pragma unroll
        for (u32 i = 0; i < 8u; i++) if (i < words) o[i] = sh ? __funnelshift_r(w[i], w[i + 1], sh) : w[i];
        k += 4u * words;
    }
    {   u32 const t = n - k;                                       /* 0..3 tail bytes */
        u32 const b0 = t > 0u ? zbd_ld8(from + k) : 0u, b1 = t > 1u ? zbd_ld8(from + k + 1) : 0u, b2 = t > 2u ? zbd_ld8(from + k + 2) : 0u;
        if (t > 0u) out[k] = (u8)b0; if (t > 1u) out[k + 1] = (u8)b1; if (t > 2u) out[k + 2] = (u8)b2; }
}

/* One CTA per frame: the matches of a frame form a wavefront that moves through the output (a match's source lies a
 * typical offset behind it), so what decides the time of a frame is the longest chain of matches copying from one another
 * times the latency of one hand-over.  Inside one CTA a hand-over is a block-scope fence and a flag — the writer and the
 * reader share an SM — instead of a device-scope fence and a trip through L2 for every link.  Frames run side by side. */
template <int THREADS>
__global__ void __launch_bounds__(THREADS)
zbd_matches_kernel(const ZbdBlock* __restrict__ blocks, const ZbdFrame* __restrict__ frames, const u64* __restrict__ seqs, const u64* __restrict__ matchPos,
                   const u32* __restrict__ tileFirst, u64 totalOut, u8* __restrict__ dst, u8* done, u32* __restrict__ execErr)
{
    __shared__ u32 sTicket;
    u32 const lane = threadIdx.x & 31u;
    ZbdFrame const fr = frames[blockIdx.x];
    if (fr.nbBlocks == 0) return;
    ZbdBlock const bl = blocks[fr.firstBlock + fr.nbBlocks - 1u];
    u32 const g0 = (u32)blocks[fr.firstBlock].seqPos, g1 = (u32)bl.seqPos + (bl.type == ZB_BT_COMPRESSED ? bl.nbSeq : 0u);     /* the frame's matches */
    if (threadIdx.x == 0) sTicket = 0;
    __syncthreads();
    while (true) {
        u32 grp = 0;
        if (lane == 0) grp = atomicAdd(&sTicket, 1u);                /* matches are handed out in order: a lane only ever waits for matches that were handed out */
        grp = __shfl_sync(ZB_FULL, grp, 0);
        if ((u64)g0 + (u64)grp * 32u >= g1) return;
        u32 const g = g0 + grp * 32u + lane;
        u64 q = 0, pos = 0;
        if (g < g1) { q = seqs[g]; pos = matchPos[g]; }
        u32 const off = (u32)q & 0x0FFFFFFFu, ml = (u32)(q >> 28);
        bool pending = g < g1 && ml != 0u && off != 0u && (u64)off <= pos && pos + ml <= totalOut;
        if (g < g1 && !pending) zbd_st_flag(done + g);               /* nothing to copy (an empty or a refused match): nobody may wait for it */
        u64 const s = pos - off;
        u32 const span = ml < off ? ml : off;
        /* candidates for "wrote into [s, s + span)": from the first match ending behind the tile of s to the first one
         * ending behind the first tile at or past the range's end, never past g - 1; each is then tested for real overlap */
        u32 j = 0, jhi = 0;
        bool deps = false;
        if (pending && g != g0) {
            j = tileFirst[s >> ZBD_TILE_LOG];
            jhi = tileFirst[(s + span + ((1u << ZBD_TILE_LOG) - 1u)) >> ZBD_TILE_LOG];
            if (jhi >= g) jhi = g - 1u;
            if (j < g0) j = g0;                                      /* matches of earlier frames never write into this one */
            deps = j < g && j <= jhi;
        }
        long long const t0 = clock64();
        while (__any_sync(ZB_FULL, pending)) {
            /* every wait ends (see above); should that ever be wrong the call fails after ~30 s instead of hanging the device */
            if (pending && clock64() - t0 > 60000000000ll) { atomicMax(execErr, (u32)ZB_error_GENERIC); zbd_st_flag(done + g); pending = false; continue; }
            bool ready = false;
            if (pending) {
                while (deps) {
                    if (zbd_ld_flag(done + j) == 0u) {               /* unfinished: does it touch the source at all? */
                        u64 const pj = matchPos[j]; u32 const mj = (u32)(seqs[j] >> 28);
                        if (pj < s + span && pj + mj > s) break;     /* yes: wait for it */
                    }
                    j++; if (j > jhi) deps = false;
                }
                ready = !deps;
            }
            if (ready) {
                __threadfence_block();
                u8* const out = dst + pos;
                const u8* const from = dst + s;
                if (off >= ml) zbd_copy_disjoint(out, from, ml);
                else if (off < 8u) {                                 /* a short pattern: read once, written ml times over */
                    u64 pat = 0;
                    for (u32 k = 0; k < off; k++) pat |= (u64)zbd_ld8(from + k) << (8u * k);
                    u32 r = 0;
                    for (u32 k = 0; k < ml; k++) { out[k] = (u8)(pat >> (8u * r)); r++; if (r == off) r = 0; }
                } else {                                             /* the `off` bytes in front of the match, again and again: every piece a disjoint copy */
                    for (u32 k = 0; k < ml; k += off) zbd_copy_disjoint(out + k, from, ml - k < off ? ml - k : off);
                }
                __threadfence_block();
                zbd_st_flag(done + g);
                pending = false;
            }
        }
    }
}

/* ------------------------------------------------------------------------------------------------ host driver */
struct ZSTD_DCtx_s {
    int device, bindDevice;
    cudaStream_t stream;
    ZbdBlock* d_blocks; ZbdFrame* d_frames; ZbdBlockOut* d_bout; size_t capBlocks, capFrames;
    u8* d_lits; size_t capLits; u64* d_seqs; size_t capSeqs; u64* d_matchPos; size_t capMatchPos;
    u32* d_tileFirst; size_t capTiles; u8* d_done; size_t capDone;
    u8* d_in; size_t capIn; u8* d_out; size_t capOut;
    u64* d_res; u32* d_execErr;
    u64* h_res;                  /* pinned: walker / scan results */
    /* streaming front end (ZSTD_decompressStream): compressed bytes collected until a frame is complete, output waiting to be handed out */
    std::vector<u8>* dsIn; std::vector<u8>* dsOut; size_t dsOutPos;
    size_t hostWalkMax;          /* ZBD_HOSTWALK_MAX, or ZSTDB200_HOSTWALK_MAX from the environment (tests: 0 forces the kernel walk) */
    u8* h_stage; size_t capStage; /* page-locked copy of a device-resident input's compressed bytes, for the header walk */
    u8* d_dict; size_t capDict;  /* the call's dictionary, whole (header + content) */
    ZbdDictInfo di; size_t dictSize;
    cudaEvent_t ev[7];
    ZSTDB200_dstats stats;
};

/* one decompression call, as an entry point describes it */
struct ZbdCall {
    void* dst; size_t dstCapacity;
    const void* src; size_t srcSize;
    const void* dict; size_t dictSize;  /* host memory; NULL / 0: none */
    bool deviceMemory;                  /* dst and src are device memory */
    cudaStream_t stream;                /* device calls: the caller's stream, NULL for the context's */
};

extern "C" ZSTD_DCtx* ZSTD_createDCtx(void)                          /* lib/zstd.h:289 */
{
    ZSTD_DCtx* d = (ZSTD_DCtx*)calloc(1, sizeof(ZSTD_DCtx));
    if (!d) return NULL;
    d->device = -1;
    {   const char* const e = getenv("ZSTDB200_HOSTWALK_MAX"); d->hostWalkMax = e ? (size_t)strtoull(e, NULL, 10) : ZBD_HOSTWALK_MAX; }
    d->bindDevice = zb_contextDevice();
    return d;
}
extern "C" size_t ZSTD_freeDCtx(ZSTD_DCtx* d)                        /* accepts NULL, lib/zstd.h:290 */
{
    if (!d) return 0;
    if (d->device >= 0) {
        ZbDeviceGuard guard;
        cudaSetDevice(d->device);
        cudaFree(d->d_blocks); cudaFree(d->d_frames); cudaFree(d->d_bout); cudaFree(d->d_lits); cudaFree(d->d_seqs); cudaFree(d->d_matchPos); cudaFree(d->d_tileFirst); cudaFree(d->d_done);
        cudaFree(d->d_in); cudaFree(d->d_out); cudaFree(d->d_res); cudaFreeHost(d->h_res); cudaFree(d->d_dict); cudaFreeHost(d->h_stage);
        for (int i = 0; i < 7; i++) cudaEventDestroy(d->ev[i]);
        cudaStreamDestroy(d->stream);
    }
    delete d->dsIn; delete d->dsOut;
    free(d);
    return 0;
}
static size_t zbd_ctxInit(ZSTD_DCtx* d)
{
    if (d->device >= 0) { CK(cudaSetDevice(d->device)); return 0; }
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) { cudaGetLastError(); return ZB_ERR(ZB_error_GENERIC); }
    int const dev = d->bindDevice < 0 ? 0 : d->bindDevice;
    CK(cudaSetDevice(dev));
    /* everything or nothing: a partial failure leaves the context uninitialised (device stays -1) */
    cudaStream_t st = nullptr; cudaEvent_t ev[7] = {}; u64* d_res = nullptr; u64* h_res = nullptr;
    cudaError_t e = cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking);
    for (int i = 0; i < 7 && e == cudaSuccess; i++) e = cudaEventCreate(&ev[i]);
    if (e == cudaSuccess) e = cudaMalloc(&d_res, 16 * sizeof(u64));
    if (e == cudaSuccess) e = cudaMallocHost(&h_res, 16 * sizeof(u64));
    if (e != cudaSuccess) {
        for (int i = 0; i < 7; i++) if (ev[i]) cudaEventDestroy(ev[i]);
        if (st) cudaStreamDestroy(st);
        cudaFree(d_res);
        cudaGetLastError();
        return ZB_ERR(e == cudaErrorMemoryAllocation ? ZB_error_memory_allocation : ZB_error_GENERIC);
    }
    d->stream = st; memcpy(d->ev, ev, sizeof(ev));
    d->d_res = d_res; d->h_res = h_res; d->d_execErr = (u32*)(d_res + 9);
    d->device = dev;
    return 0;
}
template <typename T> static size_t zbd_grow(T** p, size_t* cap, size_t need)
{
    if (need <= *cap) return 0;
    cudaFree(*p); *p = NULL; *cap = 0;
    size_t const n = need + need / 8 + 64;
    CK(cudaMalloc(p, n * sizeof(T)));
    *cap = n;
    return 0;
}

/* D1 .. D4 over descriptors that are already on the device; returns the output size */
static size_t zbd_run(ZSTD_DCtx* d, u8* d_dst, size_t dstCapacity, const u8* d_src, u32 nb, u32 nf, u64 seqCount, cudaStream_t st)
{
    CK(cudaMemsetAsync(d->d_execErr, 0, sizeof(u32), st));
    CK(cudaEventRecord(d->ev[1], st));
    u32 const grid = (nb + ZBD_WARPS - 1u) / ZBD_WARPS;
    zbd_literals_kernel<<<grid, 32 * ZBD_WARPS, 0, st>>>(d_src, d->d_blocks, nb, d->d_lits, d->d_bout, d->d_dict, d->di);
    CK(cudaEventRecord(d->ev[2], st));
    zbd_sequences_kernel<<<grid, 32 * ZBD_WARPS, 0, st>>>(d_src, d->d_blocks, nb, d->d_seqs, d->d_bout, d->d_dict, d->di);
    CK(cudaEventRecord(d->ev[3], st));
    zbd_scan_kernel<<<1, SCAN_THREADS, 0, st>>>(d->d_blocks, nb, d->d_frames, nf, d->d_bout, (u64)dstCapacity, d->d_res, d->di);
    CK(cudaMemcpyAsync(d->h_res, d->d_res, 2 * sizeof(u64), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));                                  /* nothing is written to dst before the sizes are known to fit */
    if (d->h_res[0]) return ZB_ERR((u32)d->h_res[0]);
    size_t const total = (size_t)d->h_res[1];
    CK(cudaEventRecord(d->ev[4], st));
    u32 const dictContent = d->dictSize ? (u32)(d->dictSize - d->di.contentOff) : 0u;
    const u8* const d_dictContent = d->dictSize ? d->d_dict + d->di.contentOff : (const u8*)NULL;
    {   size_t const r = zbd_grow(&d->d_tileFirst, &d->capTiles, (total >> ZBD_TILE_LOG) + 4); if (zb_isErr(r)) return r; }
    {   size_t const r = zbd_grow(&d->d_done, &d->capDone, (size_t)seqCount + 4); if (zb_isErr(r)) return r; }
    CK(cudaMemsetAsync(d->d_tileFirst, 0xFF, ((total >> ZBD_TILE_LOG) + 4) * sizeof(u32), st));
    CK(cudaMemsetAsync(d->d_done, 0, (size_t)seqCount + 4, st));
    zbd_place_kernel<<<grid, 32 * ZBD_WARPS, 0, st>>>(d_src, d->d_blocks, nb, d->d_lits, d->d_seqs, d->d_matchPos, d->d_tileFirst, d->d_bout, d_dst,
                                                      d_dictContent, dictContent, d->d_execErr);
    CK(cudaEventRecord(d->ev[6], st));
    if (seqCount) {                                                  /* threads per frame by the matches a frame holds */
        u64 const perFrame = seqCount / (nf ? nf : 1u);
        if (perFrame >= 8192u)     zbd_matches_kernel<1024><<<nf, 1024, 0, st>>>(d->d_blocks, d->d_frames, d->d_seqs, d->d_matchPos, d->d_tileFirst, (u64)total, d_dst, d->d_done, d->d_execErr);
        else if (perFrame >= 256u) zbd_matches_kernel<128><<<nf, 128, 0, st>>>(d->d_blocks, d->d_frames, d->d_seqs, d->d_matchPos, d->d_tileFirst, (u64)total, d_dst, d->d_done, d->d_execErr);
        else                       zbd_matches_kernel<32><<<nf, 32, 0, st>>>(d->d_blocks, d->d_frames, d->d_seqs, d->d_matchPos, d->d_tileFirst, (u64)total, d_dst, d->d_done, d->d_execErr);
    }
    CK(cudaEventRecord(d->ev[5], st));
    CK(cudaMemcpyAsync(d->h_res + 2, d->d_execErr, sizeof(u32), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    CK(cudaGetLastError());
    if ((u32)d->h_res[2]) return ZB_ERR((u32)d->h_res[2]);
    {   float ms = 0;
        cudaEventElapsedTime(&ms, d->ev[1], d->ev[2]); d->stats.literals_ms = ms;
        cudaEventElapsedTime(&ms, d->ev[2], d->ev[3]); d->stats.sequences_ms = ms;
        cudaEventElapsedTime(&ms, d->ev[4], d->ev[6]); d->stats.place_ms = ms;
        cudaEventElapsedTime(&ms, d->ev[6], d->ev[5]); d->stats.execute_ms = ms;
        cudaEventElapsedTime(&ms, d->ev[1], d->ev[5]); d->stats.kernel_ms = ms;
        d->stats.nbBlocks = nb; d->stats.nbFrames = nf; d->stats.launches = 5; }
    return total;
}

static size_t zbd_ensure(ZSTD_DCtx* d, u32 nb, u32 nf, u64 litBytes, u64 seqCount)
{
    if (nb > d->capBlocks) {
        cudaFree(d->d_blocks); cudaFree(d->d_bout); d->d_blocks = NULL; d->d_bout = NULL; d->capBlocks = 0;
        size_t const n = (size_t)nb + nb / 8 + 64;
        CK(cudaMalloc(&d->d_blocks, n * sizeof(ZbdBlock))); CK(cudaMalloc(&d->d_bout, (n + 1) * sizeof(ZbdBlockOut)));
        d->capBlocks = n;
    }
    {   size_t const e = zbd_grow(&d->d_frames, &d->capFrames, (size_t)nf); if (zb_isErr(e)) return e; }
    {   size_t const e = zbd_grow(&d->d_lits, &d->capLits, (size_t)litBytes + 16); if (zb_isErr(e)) return e; }
    {   size_t const e = zbd_grow(&d->d_seqs, &d->capSeqs, (size_t)seqCount + 1); if (zb_isErr(e)) return e; }
    {   size_t const e = zbd_grow(&d->d_matchPos, &d->capMatchPos, (size_t)seqCount + 1); if (zb_isErr(e)) return e; }
    return 0;
}


/* the call's dictionary: parsed on the host (zbd_parseDict), uploaded whole; NULL / 0 = none.  A dictionary without the
 * magic number — or shorter than 8 bytes — is raw content (zstd_decompress.c:1541-1560). */
static size_t zbd_setDict(ZSTD_DCtx* d, const void* dict, size_t dictSize, cudaStream_t st)
{
    memset(&d->di, 0, sizeof(d->di)); d->dictSize = 0;
    if (!dict || dictSize == 0) return 0;
    u32 const e = zbd_parseDict(&d->di, (const u8*)dict, dictSize);
    if (e) return ZB_ERR(e);
    {   size_t const r = zbd_grow(&d->d_dict, &d->capDict, dictSize + 16); if (zb_isErr(r)) return r; }
    CK(cudaMemcpyAsync(d->d_dict, dict, dictSize, cudaMemcpyHostToDevice, st));
    CK(cudaStreamSynchronize(st));                                    /* the caller's dictionary buffer is pageable memory that may change after the call */
    d->dictSize = dictSize;
    return 0;
}

/* D0 on a host-readable copy of the compressed bytes: count the blocks and frames, then describe them into B and F */
static u32 zbd_walkHost(const ZSTD_DCtx* d, const u8* in, size_t size, std::vector<ZbdBlock>& B, std::vector<ZbdFrame>& F,
                        u32* nb, u32* nf, u64* lit, u64* seq)
{
    u32 const e = zbd_walk(in, size, NULL, 0, NULL, 0, nb, nf, lit, seq, d->di.entropy != 0, d->di.dictID);
    if (e) return e;
    B.resize(*nb ? *nb : 1); F.resize(*nf ? *nf : 1);
    return zbd_walk(in, size, B.data(), *nb, F.data(), *nf, nb, nf, lit, seq, d->di.entropy != 0, d->di.dictID);
}

/* Every decompression call.  The frame and block headers have to be followed one after the other wherever they are read:
 * one device thread pays a device-memory round trip per header, the host a cache access.  So the walk runs on the host
 * wherever a host-readable copy of the compressed bytes exists: the caller's buffer for host calls, and for device calls
 * up to hostWalkMax a page-locked copy made at PCIe speed.  Beyond that the walk is a kernel.  Host calls go through the
 * context's d_in / d_out and check the frames' content checksums; device calls do not. */
static size_t zbd_decompress(ZSTD_DCtx* d, const ZbdCall& c)
{
    if (!d) return ZB_ERR(ZB_error_GENERIC);
    if (c.srcSize == 0) return 0;                                     /* zstd_decompress.c:1093 : an empty input is an empty output */
    if (!c.deviceMemory && !c.src) return ZB_ERR(ZB_error_srcSize_wrong);
    if (!c.deviceMemory && c.dstCapacity && !c.dst) return ZB_ERR(ZB_error_dstBuffer_null);
    ZbDeviceGuard guard;
    {   size_t const e = zbd_ctxInit(d); if (zb_isErr(e)) return e; }
    memset(&d->stats, 0, sizeof(d->stats));
    cudaStream_t const st = c.stream ? c.stream : d->stream;
    {   size_t const e = zbd_setDict(d, c.dict, c.dictSize, st); if (zb_isErr(e)) return e; }
    /* D0: block and frame descriptors */
    const u8* hostIn = c.deviceMemory ? NULL : (const u8*)c.src;
    if (c.deviceMemory && c.srcSize <= d->hostWalkMax) {
        if (c.srcSize > d->capStage) {
            cudaFreeHost(d->h_stage); d->h_stage = NULL; d->capStage = 0;
            size_t const n = c.srcSize + c.srcSize / 4 + 4096;
            CK(cudaMallocHost(&d->h_stage, n));
            d->capStage = n;
        }
        CK(cudaMemcpyAsync(d->h_stage, c.src, c.srcSize, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        hostIn = d->h_stage;
    }
    std::vector<ZbdBlock> B; std::vector<ZbdFrame> F;
    u32 nb = 0, nf = 0; u64 lit = 0, seq = 0;
    if (hostIn) { u32 const e = zbd_walkHost(d, hostIn, c.srcSize, B, F, &nb, &nf, &lit, &seq); if (e) return ZB_ERR(e); }
    else {                                                            /* the walk kernel; once more if the arrays were too small */
        u32 capB = (u32)(c.srcSize / 4096u) + 1024u, capF = 1024u;
        for (int attempt = 0; attempt < 2; attempt++) {
            {   size_t const r = zbd_ensure(d, capB, capF, 0, 0); if (zb_isErr(r)) return r; }
            zbd_walk_kernel<<<1, 32, 0, st>>>((const u8*)c.src, (u64)c.srcSize, d->d_blocks, (u32)d->capBlocks, d->d_frames, (u32)d->capFrames, d->d_res, d->di.entropy, d->di.dictID);
            CK(cudaMemcpyAsync(d->h_res, d->d_res, 5 * sizeof(u64), cudaMemcpyDeviceToHost, st));
            CK(cudaStreamSynchronize(st));
            if (d->h_res[0]) return ZB_ERR((u32)d->h_res[0]);
            if (d->h_res[1] <= d->capBlocks && d->h_res[2] <= d->capFrames) break;
            capB = (u32)d->h_res[1]; capF = (u32)d->h_res[2];
            if (attempt == 1) return ZB_ERR(ZB_error_GENERIC);
        }
        nb = (u32)d->h_res[1]; nf = (u32)d->h_res[2]; lit = d->h_res[3]; seq = d->h_res[4];
    }
    if (nb == 0) return 0;
    const u8* runSrc = (const u8*)c.src; u8* runDst = (u8*)c.dst; size_t outCap = c.dstCapacity;
    if (!c.deviceMemory) {                                            /* host buffers: through the context's d_in / d_out */
        u64 known = 0; bool allKnown = true;
        for (u32 f = 0; f < nf; f++) { if (F[f].contentSize == ZBD_CONTENTSIZE_UNKNOWN) allKnown = false; else known += F[f].contentSize; }
        if (allKnown && known > c.dstCapacity) return ZB_ERR(ZB_error_dstSize_tooSmall);      /* refused before any upload */
        /* the output can not be larger than the blocks' maximum sizes */
        outCap = allKnown ? (size_t)known : (c.dstCapacity < (size_t)nb * ZB_BLOCK_MAX ? c.dstCapacity : (size_t)nb * ZB_BLOCK_MAX);
        {   size_t const r = zbd_grow(&d->d_in, &d->capIn, c.srcSize + 16); if (zb_isErr(r)) return r; }
        {   size_t const r = zbd_grow(&d->d_out, &d->capOut, outCap + 16); if (zb_isErr(r)) return r; }
        CK(cudaEventRecord(d->ev[0], st));
        CK(cudaMemcpyAsync(d->d_in, c.src, c.srcSize, cudaMemcpyHostToDevice, st));
        runSrc = d->d_in; runDst = d->d_out;
    }
    {   size_t const r = zbd_ensure(d, nb, nf, lit, seq); if (zb_isErr(r)) return r; }
    if (hostIn) {
        CK(cudaMemcpyAsync(d->d_blocks, B.data(), (size_t)nb * sizeof(ZbdBlock), cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(d->d_frames, F.data(), (size_t)nf * sizeof(ZbdFrame), cudaMemcpyHostToDevice, st));
        CK(cudaStreamSynchronize(st));                               /* B and F are pageable: the copies end before a return can free them */
    }
    size_t const total = zbd_run(d, runDst, outCap, runSrc, nb, nf, seq, st);
    if (zb_isErr(total) || c.deviceMemory) return total;
    if (total > c.dstCapacity) return ZB_ERR(ZB_error_dstSize_tooSmall);
    if (total) CK(cudaMemcpy(c.dst, d->d_out, total, cudaMemcpyDeviceToHost));
    /* frame checksums (format: "Content_Checksum"): XXH64 of the regenerated content, low 32 bits */
    {   size_t off = 0;
        for (u32 f = 0; f < nf; f++) {
            u64 size = 0;
            if (F[f].contentSize != ZBD_CONTENTSIZE_UNKNOWN) size = F[f].contentSize;
            else { /* sizes of frames without the field: from the scan */
                std::vector<ZbdBlockOut> tmp(2);
                u32 const last = F[f].firstBlock + F[f].nbBlocks;
                CK(cudaMemcpy(&tmp[0], d->d_bout + F[f].firstBlock, sizeof(ZbdBlockOut), cudaMemcpyDeviceToHost));
                u64 end = total;
                if (last < nb) { CK(cudaMemcpy(&tmp[1], d->d_bout + last, sizeof(ZbdBlockOut), cudaMemcpyDeviceToHost)); end = tmp[1].dstOff; }
                size = end - tmp[0].dstOff;
            }
            if (F[f].hasChecksum) {
                u32 const want = zbd_le(hostIn + F[f].srcOff + F[f].cSize - 4, 4);
                if ((u32)ZSTDB200_xxh64((const u8*)c.dst + off, (size_t)size) != want) return ZB_ERR(22);      /* checksum_wrong */
            }
            off += (size_t)size;
        }
    }
    d->stats.h2d_bytes = c.srcSize; d->stats.d2h_bytes = total;
    return total;
}

extern "C" size_t ZSTD_decompress_usingDict(ZSTD_DCtx* d, void* dst, size_t dstCapacity, const void* src, size_t srcSize,
                                            const void* dict, size_t dictSize)                                            /* lib/zstd.h:955 */
{
    ZbdCall const c = { dst, dstCapacity, src, srcSize, dict, dictSize, false, NULL };
    return zbd_decompress(d, c);
}
extern "C" size_t ZSTD_decompressDCtx(ZSTD_DCtx* d, void* dst, size_t dstCapacity, const void* src, size_t srcSize)      /* lib/zstd.h:299 */
{
    return ZSTD_decompress_usingDict(d, dst, dstCapacity, src, srcSize, NULL, 0);
}

extern "C" size_t ZSTD_decompress(void* dst, size_t dstCapacity, const void* src, size_t compressedSize)                  /* lib/zstd.h:170 */
{
    ZSTD_DCtx* const d = ZSTD_createDCtx();
    if (!d) return ZB_ERR(ZB_error_memory_allocation);
    size_t const r = ZSTD_decompressDCtx(d, dst, dstCapacity, src, compressedSize);
    ZSTD_freeDCtx(d);
    return r;
}

extern "C" size_t ZSTDB200_decompressDevice_usingDict(ZSTD_DCtx* d, void* d_dst, size_t dstCapacity, const void* d_src, size_t srcSize,
                                                      const void* dict, size_t dictSize, void* stream)
{
    ZbdCall const c = { d_dst, dstCapacity, d_src, srcSize, dict, dictSize, true, (cudaStream_t)stream };
    return zbd_decompress(d, c);
}
extern "C" size_t ZSTDB200_decompressDevice(ZSTD_DCtx* d, void* d_dst, size_t dstCapacity, const void* d_src, size_t srcSize, void* stream)
{
    return ZSTDB200_decompressDevice_usingDict(d, d_dst, dstCapacity, d_src, srcSize, NULL, 0, stream);
}

extern "C" void ZSTDB200_getLastDStats(const ZSTD_DCtx* d, ZSTDB200_dstats* out) { if (d && out) *out = d->stats; }

/* lib/zstd.h:205,227 : host helpers that only read headers */
extern "C" unsigned long long ZSTD_getFrameContentSize(const void* src, size_t srcSize)
{
    ZbdFrameHeader h;
    u32 const e = zbd_readFrameHeader(&h, (const u8*)src, srcSize);
    if (e) return 0ULL - 2;                                           /* ZSTD_CONTENTSIZE_ERROR */
    if (h.skippable) return 0;
    return h.contentSize == ZBD_CONTENTSIZE_UNKNOWN ? 0ULL - 1 : h.contentSize;   /* ZSTD_CONTENTSIZE_UNKNOWN */
}
extern "C" size_t ZSTD_findFrameCompressedSize(const void* src, size_t srcSize)
{
    const u8* const in = (const u8*)src;
    ZbdFrameHeader h;
    u32 const e = zbd_readFrameHeader(&h, in, srcSize);
    if (e) return ZB_ERR(e);
    if (h.skippable) return (8u + h.contentSize > srcSize) ? ZB_ERR(ZB_error_srcSize_wrong) : (size_t)(8u + h.contentSize);
    size_t p = h.headerSize;
    while (true) {
        if (p + 3 > srcSize) return ZB_ERR(ZB_error_srcSize_wrong);
        u32 const bh = zbd_le(in + p, 3);
        u32 const type = (bh >> 1) & 3u, bsz = bh >> 3;
        if (type == 3u) return ZB_ERR(ZBD_CORRUPT);
        p += 3u + (type == ZB_BT_RLE ? 1u : bsz);
        if (p > srcSize) return ZB_ERR(ZB_error_srcSize_wrong);
        if (bh & 1u) break;
    }
    if (h.hasChecksum) { p += 4; if (p > srcSize) return ZB_ERR(ZB_error_srcSize_wrong); }
    return p;
}

/* ------------------------------------------------------------------------------------------------ streaming (lib/zstd.h:880-924)
 * The GPU decodes whole frames, so the stream front end collects compressed bytes until a frame is complete
 * (ZSTD_findFrameCompressedSize), decodes it, and hands the result out as the caller makes room.  Return value as in the
 * reference: 0 when a frame has been decoded and handed out completely, else a hint (> 0) for the next input size. */
static size_t zbd_frameOutputBound(const u8* in, size_t size)          /* content size, or blocks x 128 KiB when the header does not say */
{
    ZbdFrameHeader h;
    if (zbd_readFrameHeader(&h, in, size) || h.skippable) return 0;
    if (h.contentSize != ZBD_CONTENTSIZE_UNKNOWN) return (size_t)h.contentSize;
    size_t p = h.headerSize, blocks = 0;
    while (p + 3 <= size) { u32 const bh = zbd_le(in + p, 3); blocks++; p += 3u + (((bh >> 1) & 3u) == ZB_BT_RLE ? 1u : (bh >> 3)); if (bh & 1u) break; }
    return blocks * (size_t)ZB_BLOCK_MAX;
}
extern "C" ZSTD_DStream* ZSTD_createDStream(void) { return ZSTD_createDCtx(); }
extern "C" size_t ZSTD_freeDStream(ZSTD_DStream* zds) { return ZSTD_freeDCtx(zds); }
extern "C" size_t ZSTD_initDStream(ZSTD_DStream* zds)
{
    if (!zds) return ZB_ERR(ZB_error_GENERIC);
    if (zds->dsIn) zds->dsIn->clear();
    if (zds->dsOut) zds->dsOut->clear();
    zds->dsOutPos = 0;
    return 5;                                                          /* a frame header's first bytes, as the reference suggests (ZSTD_startingInputLength) */
}
extern "C" size_t ZSTD_DStreamInSize(void) { return ZB_BLOCK_MAX + 3; }  /* lib/zstd.h:922 */
extern "C" size_t ZSTD_DStreamOutSize(void) { return ZB_BLOCK_MAX; }
extern "C" size_t ZSTD_decompressStream(ZSTD_DStream* d, ZSTD_outBuffer* out, ZSTD_inBuffer* in)
{
    if (!d || !out || !in) return ZB_ERR(ZB_error_GENERIC);
    if (out->pos > out->size) return ZB_ERR(ZB_error_dstSize_tooSmall);
    if (in->pos > in->size) return ZB_ERR(ZB_error_srcSize_wrong);
    if (!d->dsIn) { d->dsIn = new (std::nothrow) std::vector<u8>(); d->dsOut = new (std::nothrow) std::vector<u8>(); if (!d->dsIn || !d->dsOut) return ZB_ERR(ZB_error_memory_allocation); }
    auto handOut = [&]() -> size_t {
        size_t const have = d->dsOut->size() - d->dsOutPos, room = out->size - out->pos, n = have < room ? have : room;
        if (n) { memcpy((u8*)out->dst + out->pos, d->dsOut->data() + d->dsOutPos, n); out->pos += n; d->dsOutPos += n; }
        if (d->dsOutPos == d->dsOut->size()) { d->dsOut->clear(); d->dsOutPos = 0; }
        return d->dsOut->size() - d->dsOutPos;
    };
    if (handOut() != 0) return d->dsOut->size() - d->dsOutPos;           /* room first: input is only taken while nothing is waiting */
    d->dsIn->insert(d->dsIn->end(), (const u8*)in->src + in->pos, (const u8*)in->src + in->size);
    in->pos = in->size;
    bool decoded = false;
    while (!d->dsIn->empty()) {
        size_t const fs = ZSTD_findFrameCompressedSize(d->dsIn->data(), d->dsIn->size());
        if (ZSTD_isError(fs)) {
            if (ZSTD_getErrorCode(fs) == ZB_error_srcSize_wrong) break;   /* the frame is not complete yet */
            return fs;
        }
        size_t const bound = zbd_frameOutputBound(d->dsIn->data(), fs);
        size_t const base = d->dsOut->size();
        d->dsOut->resize(base + bound + 1);
        size_t const r = ZSTD_decompressDCtx(d, d->dsOut->data() + base, bound, d->dsIn->data(), fs);
        if (ZSTD_isError(r)) { d->dsOut->resize(base); return r; }
        d->dsOut->resize(base + r);
        d->dsIn->erase(d->dsIn->begin(), d->dsIn->begin() + (ptrdiff_t)fs);
        decoded = true;
    }
    size_t const waiting = handOut();
    if (waiting) return waiting;
    (void)decoded;
    if (d->dsIn->empty()) return 0;                                      /* at a frame border with everything handed out */
    return ZB_BLOCK_MAX + 3;                                             /* in the middle of a frame: more input, please */
}
