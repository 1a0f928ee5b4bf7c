/* zb_merge.cuh — the last steps of K1c (zb_match.cu), shared with K1s-b (zb_seqimport.cu): given a block's sequences as
 * (offset, litLength, matchLength) triples in its seq slots, assign the repcodes, gather the literal bytes and write the
 * block's meta.  Both kernels run it with MERGE_THREADS threads and their own shared arrays. */
#ifndef ZB_MERGE_CUH
#define ZB_MERGE_CUH
#include "zb_common.h"
#include "zb_device.cuh"

#define MERGE_THREADS 256
#define MERGE_TILE 1024u                       /* sequences scanned and gathered per round */
#define MERGE_PER (MERGE_TILE / MERGE_THREADS)  /* consecutive sequences of a tile owned by one thread */

/* The repcode history starts as (rep0, rep1, rep2) (the frame's {1,4,8} or the dictionary's) in a frame's first block and unknown
 * (0: never matches) in every other block.  Shared arrays: sPos / sLit / sLen / sOff / sR2 of MERGE_TILE, wsumL / wsumA /
 * wmaxU / wmaxK of MERGE_THREADS / 32, sRep of 3; baseL / baseA are shared scalars. */
__device__ __forceinline__ void zb_merge_codes(u32 rep0, u32 rep1, u32 rep2, bool first, u64* __restrict__ myseq, u8* __restrict__ mylit,
                                               const u8* __restrict__ in, u32 nbSeq, u32 blockSize, ZbBlockMeta* __restrict__ metaOut,
                                               u32* sPos, u32* sLit, u32* sLen, u32* sOff, u32* sR2, u32* sRep,
                                               u32* wsumL, u32* wsumA, u32* wmaxU, u32* wmaxK, u32& baseL, u32& baseA)
{
    u32 const tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    if (tid == 0) {
        baseL = 0; baseA = 0;
        sRep[0] = first ? rep0 : 0u; sRep[1] = first ? rep1 : 0u; sRep[2] = first ? rep2 : 0u;
    }
    __syncthreads();
    /* ---- 3. literals + repcodes, a tile of sequences at a time ----
     * The repcode history (r1, r2, r3) is a serial recurrence in ZSTD_updateRep's form, but its solution is not:
     *   - after any sequence r1 is that sequence's offset, so "r1 before sequence i" is the offset of sequence i-1;
     *   - a sequence leaves the history alone (U) iff it has literals and repeats r1; every other sequence sets r2 to the r1
     *     it found: "r2 before i" is the r1 found by the last non-U sequence before i;
     *   - a non-U sequence whose offset is the r2 it found swaps r1 and r2 and keeps r3 (K = U or swap); every other sets r3
     *     to the r2 it found: "r3 before i" is the r2 found by the last non-K sequence before i.
     * Two "index of the last flagged element before me" scans (maximum scans) over the tile give every sequence the history
     * it meets; its code follows from ZSTD_storeSeq's rules.  The history passes from tile to tile through sRep. */
    for (u32 t0 = 0; t0 < nbSeq; t0 += MERGE_TILE) {
        u32 const n = min(MERGE_TILE, nbSeq - t0);
        /* every thread owns MERGE_PER consecutive sequences of the tile */
        u32 ll[MERGE_PER], adv[MERGE_PER], ml[MERGE_PER], off[MERGE_PER], myL = 0, myA = 0;
#pragma unroll
        for (u32 j = 0; j < MERGE_PER; j++) {
            u32 const i = tid * MERGE_PER + j;
            u64 const q = (i < n) ? myseq[t0 + i] : 0ull;
            ll[j] = ZB_SEQ_LL(q);
            ml[j] = ZB_SEQ_ML(q);
            adv[j] = ll[j] + ml[j];
            off[j] = ZB_SEQ_OFFBASE(q);
            if (i < n) sOff[i] = off[j];
            myL += ll[j]; myA += adv[j];
        }
        u32 inL = myL, inA = myA;                                /* inclusive scan over the warp, then over the warps */
#pragma unroll
        for (u32 o = 1; o < 32u; o <<= 1) {
            u32 const a = __shfl_up_sync(ZB_FULL, inL, o), c = __shfl_up_sync(ZB_FULL, inA, o);
            if (lane >= o) { inL += a; inA += c; }
        }
        if (lane == 31u) { wsumL[warp] = inL; wsumA[warp] = inA; }
        u32 const R1 = sRep[0], R2 = sRep[1], R3 = sRep[2];      /* history at the tile's start */
        __syncthreads();
        u32 offL = baseL + inL - myL, offA = baseA + inA - myA;
        for (u32 w = 0; w < warp; w++) { offL += wsumL[w]; offA += wsumA[w]; }
#pragma unroll
        for (u32 j = 0; j < MERGE_PER; j++) {
            u32 const i = tid * MERGE_PER + j;
            if (i < n) { sPos[i] = offA; sLit[i] = offL; sLen[i] = ll[j]; }
            offL += ll[j]; offA += adv[j];
        }
        /* r1 before each of my sequences, U flags, first scan */
        u32 prevOff[MERGE_PER], r2b[MERGE_PER], r3b[MERGE_PER], bef[MERGE_PER];
        bool U[MERGE_PER], K[MERGE_PER];
        u32 run = 0;
#pragma unroll
        for (u32 j = 0; j < MERGE_PER; j++) {
            u32 const i = tid * MERGE_PER + j;
            prevOff[j] = j ? off[j - 1u] : (i == 0u ? R1 : ((i < n) ? sOff[i - 1u] : 0u));
            U[j] = ll[j] > 0u && off[j] == prevOff[j];
            bef[j] = run;                                            /* 1 + index of the last non-U sequence of mine before this one */
            if (i < n && !U[j]) run = i + 1u;
        }
        {   u32 inc = run;
#pragma unroll
            for (u32 o = 1; o < 32u; o <<= 1) { u32 const x = __shfl_up_sync(ZB_FULL, inc, o); if (lane >= o) inc = max(inc, x); }
            if (lane == 31u) wmaxU[warp] = inc;
            u32 ex = __shfl_up_sync(ZB_FULL, inc, 1); if (lane == 0u) ex = 0u;
            __syncthreads();                                         /* also: sPos / sLit / sLen / sOff of the tile are complete */
            for (u32 w = 0; w < warp; w++) ex = max(ex, wmaxU[w]);
#pragma unroll
            for (u32 j = 0; j < MERGE_PER; j++) {
                u32 const i = tid * MERGE_PER + j;
                u32 const m = max(bef[j], ex);                       /* 1 + index of the last non-U sequence before i, 0: none in this tile */
                r2b[j] = m == 0u ? R2 : (m == 1u ? R1 : sOff[m - 2u]);   /* the r1 that sequence found */
                if (i < n) sR2[i] = r2b[j];
            }
        }
        if (tid == MERGE_THREADS - 1u) { baseL = offL; baseA = offA; }     /* totals up to the end of this tile */
        run = 0;
#pragma unroll
        for (u32 j = 0; j < MERGE_PER; j++) {
            u32 const i = tid * MERGE_PER + j;
            K[j] = U[j] || off[j] == r2b[j];
            bef[j] = run;
            if (i < n && !K[j]) run = i + 1u;
        }
        {   u32 inc = run;
#pragma unroll
            for (u32 o = 1; o < 32u; o <<= 1) { u32 const x = __shfl_up_sync(ZB_FULL, inc, o); if (lane >= o) inc = max(inc, x); }
            if (lane == 31u) wmaxK[warp] = inc;
            u32 ex = __shfl_up_sync(ZB_FULL, inc, 1); if (lane == 0u) ex = 0u;
            __syncthreads();                                         /* also: sR2 of the tile is complete, every thread holds R1..R3 */
            for (u32 w = 0; w < warp; w++) ex = max(ex, wmaxK[w]);
#pragma unroll
            for (u32 j = 0; j < MERGE_PER; j++) {
                u32 const i = tid * MERGE_PER + j;
                u32 const m = max(bef[j], ex);
                r3b[j] = m == 0u ? R3 : sR2[m - 1u];                 /* the r2 that sequence found */
                bool const swp = !U[j] && off[j] == r2b[j];
                u32 c = off[j] + 3u;
                if (ll[j] > 0u) { if (U[j]) c = 1u; else if (swp) c = 2u; else if (off[j] == r3b[j]) c = 3u; }
                else            { if (swp) c = 1u; else if (off[j] == r3b[j]) c = 2u; else if (prevOff[j] > 1u && off[j] == prevOff[j] - 1u) c = 3u; }
                if (i < n) myseq[t0 + i] = zb_pack_seq(c, ll[j], ml[j]);
                if (i == n - 1u) { sRep[0] = off[j]; sRep[1] = U[j] ? r2b[j] : prevOff[j]; sRep[2] = K[j] ? r3b[j] : r2b[j]; }   /* read again only behind the tile's last barrier */
            }
        }
        /* the tile's literal bytes [L0, L1) of the block's literal buffer, 8 at a time per thread: the run that holds
         * a group's first byte is found by bisection over the runs' start offsets, later bytes step to the next
         * non-empty run; all of a thread's loads are independent of one another.  Full groups leave as one 8-byte
         * store (the buffer is 16-byte aligned), the partial groups at the tile's edges byte by byte. */
        {   u32 const L0 = sLit[0], L1 = sLit[n - 1u] + sLen[n - 1u];
            for (u32 g = (L0 >> 3) + tid; (g << 3) < L1; g += MERGE_THREADS) {
                u32 const jb = g << 3;
                u32 const j0 = jb > L0 ? jb : L0, j1 = jb + 8u < L1 ? jb + 8u : L1;
                u32 sq = 0;                                              /* largest index with sLit[sq] <= j0 (sLit[0] = L0 <= j0) */
#pragma unroll
                for (u32 stp = MERGE_TILE / 2u; stp > 0u; stp >>= 1) {
                    u32 const c = sq + stp;
                    if (c < n && sLit[c] <= j0) sq = c;
                }
                u32 runEnd = sLit[sq] + sLen[sq];
                const u8* from = in + (sPos[sq] - sLit[sq]);             /* from[j] = the literal at buffer offset j while j lies in run sq */
                u64 v = 0;
#pragma unroll
                for (u32 k = 0; k < 8u; k++) {
                    u32 const j = jb + k;
                    if (j >= j0 && j < j1) {
                        while (j >= runEnd) { sq++; runEnd = sLit[sq] + sLen[sq]; from = in + (sPos[sq] - sLit[sq]); }
                        v |= (u64)from[j] << (8u * k);
                    }
                }
                if (j1 - j0 == 8u) *reinterpret_cast<u64*>(mylit + jb) = v;
                else for (u32 j = j0; j < j1; j++) mylit[j] = (u8)(v >> (8u * (j - jb)));
            }
        }
        __syncthreads();                                             /* the shared arrays are free for the next tile, sRep is its history */
    }
    u32 const litSeq = baseL, consumed = baseA;                   /* literals in sequences, bytes covered by sequences */
    u32 const lastLits = blockSize - consumed;
    for (u32 x = tid; x < lastLits; x += MERGE_THREADS) mylit[litSeq + x] = in[consumed + x];
    /* ---- 4. meta ---- */
    if (tid == 0) {
        ZbBlockMeta m; m.nbSeq = nbSeq; m.litSize = litSeq + lastLits; m.litSecSize = 0; m.bodySize = 0;
        m.type = ZB_BT_COMPRESSED; m.forceRaw = 0; m.rleByte = 0; m.pad = 0;
        *metaOut = m;
    }
}
#endif
