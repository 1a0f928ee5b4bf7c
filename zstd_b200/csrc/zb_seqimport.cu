/* zb_seqimport.cu — K1s: caller-supplied sequences (ZSTD_Sequence, lib/zstd.h:1291-1322) instead of the match-finder.
 *
 *   K1s-a  partition + validate: one pass of tiles over the sequences (16-byte loads) sums litLength + matchLength and
 *          counts the delimiters that close a non-empty block; one CTA scans the tile sums; a second pass of tiles gives
 *          every sequence its end position, checks it and records where blocks start (the first invalid index goes
 *          through atomicMin, so the error does not depend on timing).  Explicit delimiters: the block table is built
 *          on the device.
 *   K1s-b  convert: one CTA per block clips the sequences that overlap the block to it (a match part of >= 3 bytes
 *          inside the block stays a match, every other byte is a literal), writes them as (offset, litLength,
 *          matchLength) triples into the block's seq slots and runs K1c's last steps (zb_merge.cuh: repcodes, literal
 *          gather, meta).  K2 / K3 / K4 follow unchanged.
 * The rules are stated in plain C by oracle/zb_seqs.c (tests only).
 */
#include "zb_device.cuh"
#include "zb_kernels.h"
#include "zb_merge.cuh"

#define SEQ_THREADS 256u
#define SEQ_TILE 1024u                          /* sequences per CTA of the tile passes */
#define SEQ_PER (SEQ_TILE / SEQ_THREADS)

__device__ __forceinline__ bool zb_isDelim(uint4 q, bool expl) { return expl && q.x == 0u && q.z == 0u; }

/* inclusive sums over the CTA of (u64, u32) pairs; the CTA totals through totA / totB when they are not NULL */
__device__ __forceinline__ void zb_scan2(u64& a, u32& b, u64* wa, u32* wb, u64* totA, u32* totB)
{
    u32 const lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
#pragma unroll
    for (u32 o = 1; o < 32u; o <<= 1) {
        u64 const x = __shfl_up_sync(ZB_FULL, a, o); u32 const y = __shfl_up_sync(ZB_FULL, b, o);
        if (lane >= o) { a += x; b += y; }
    }
    if (lane == 31u) { wa[warp] = a; wb[warp] = b; }
    __syncthreads();
    u64 pa = 0; u32 pb = 0;
    for (u32 w = 0; w < warp; w++) { pa += wa[w]; pb += wb[w]; }
    if (totA) { u64 ta = 0; u32 tb = 0; for (u32 w = 0; w < blockDim.x / 32u; w++) { ta += wa[w]; tb += wb[w]; } *totA = ta; *totB = tb; }
    a += pa; b += pb;
    __syncthreads();
}

/* Tiles of the sequence array.  PLACE = false: per tile, the sum of the lengths and the number of block-closing
 * delimiters.  PLACE = true (tile prefixes known): validation, and the block starts —
 *   explicit: closing delimiter number k < nbBlocks writes blockEnd[k] and blockSeq[k] = its index;
 *   otherwise: every sequence [s, e) writes itself as the first sequence of the blocks whose start lies in [s, e). */
template <bool PLACE>
__global__ void __launch_bounds__(SEQ_THREADS)
zb_seq_tiles_kernel(const uint4* __restrict__ seqs, u32 n, bool expl, u64* __restrict__ tileLen, u32* __restrict__ tileEnds,
                    u64 srcSize, u64 window, u64 dictContent, u32 blockMax, u32 nbBlocks,
                    u64* __restrict__ blockEnd, u32* __restrict__ blockSeq, u32* __restrict__ blockFirst, u64* __restrict__ blockFirstPos,
                    unsigned long long* __restrict__ errIdx)
{
    __shared__ uint4 sq[SEQ_TILE];
    __shared__ u64 wa[SEQ_THREADS / 32u]; __shared__ u32 wb[SEQ_THREADS / 32u];
    u32 const t0 = blockIdx.x * SEQ_TILE, tid = threadIdx.x;
#pragma unroll
    for (u32 k = 0; k < SEQ_PER; k++) {                        /* coalesced 16-byte loads */
        u32 const i = t0 + k * SEQ_THREADS + tid;
        sq[k * SEQ_THREADS + tid] = i < n ? seqs[i] : make_uint4(0u, 0u, 0u, 0u);
    }
    bool prevDelim = false;
    if (tid == 0 && t0 > 0) prevDelim = zb_isDelim(seqs[t0 - 1u], expl);
    __syncthreads();
    u64 len[SEQ_PER]; bool end[SEQ_PER];
    u64 a = 0; u32 c = 0;
#pragma unroll
    for (u32 k = 0; k < SEQ_PER; k++) {
        u32 const j = tid * SEQ_PER + k;
        uint4 const q = sq[j];
        bool const pd = j ? zb_isDelim(sq[j - 1u], expl) : prevDelim;
        bool const d = zb_isDelim(q, expl);
        len[k] = (u64)q.y + q.z;
        end[k] = t0 + j < n && d && (q.y > 0u || (t0 + j > 0u && !pd));
        a += len[k]; c += end[k];
    }
    u64 const myA = a; u32 const myC = c;
    if (!PLACE) {
        u64 ta; u32 tb;
        zb_scan2(a, c, wa, wb, &ta, &tb);
        if (tid == 0) { tileLen[blockIdx.x] = ta; tileEnds[blockIdx.x] = tb; }
        return;
    }
    zb_scan2(a, c, wa, wb, nullptr, nullptr);
    u64 p = tileLen[blockIdx.x] + a - myA;                      /* start of my first sequence */
    u32 k0 = tileEnds[blockIdx.x] + c - myC;                    /* index of my first closing delimiter */
    u32 bad = ~0u;
#pragma unroll
    for (u32 k = 0; k < SEQ_PER; k++) {
        u32 const j = tid * SEQ_PER + k, i = t0 + j;
        if (i >= n) break;
        uint4 const q = sq[j];
        u64 const s = p;
        p += len[k];
        if (!zb_isDelim(q, expl)) {
            u64 const bound = p > window ? window : p + dictContent;   /* zstd_compress.c:6531 */
            if (q.x == 0u || q.z < 3u || (u64)q.x > bound || q.x > ZB_SEQ_OFF_MAX) bad = min(bad, i);
        }
        if (p > srcSize) bad = min(bad, i);
        if (expl) {
            if (end[k] && k0 < nbBlocks) { blockEnd[k0] = p; blockSeq[k0] = i; }
            k0 += end[k];
        } else if (p > s && s < srcSize) {
            for (u64 b = (s + blockMax - 1u) / blockMax; b < nbBlocks && b * blockMax < p; b++) { blockFirst[b] = i; blockFirstPos[b] = s; }
        }
    }
    if (bad != ~0u) atomicMin(errIdx, (unsigned long long)bad);
}

/* exclusive scan of the tile sums in place (one CTA); ctrl[0] = sum of all lengths, ctrl[1] = closing delimiters */
__global__ void __launch_bounds__(SEQ_THREADS)
zb_seq_scan_kernel(u64* __restrict__ tileLen, u32* __restrict__ tileEnds, u32 nbTiles, u64* __restrict__ ctrl)
{
    __shared__ u64 wa[SEQ_THREADS / 32u]; __shared__ u32 wb[SEQ_THREADS / 32u];
    __shared__ u64 carryA; __shared__ u32 carryB;
    if (threadIdx.x == 0) { carryA = 0; carryB = 0; }
    __syncthreads();
    for (u32 t0 = 0; t0 < nbTiles; t0 += SEQ_THREADS) {
        u32 const i = t0 + threadIdx.x;
        u64 a = i < nbTiles ? tileLen[i] : 0ull; u32 b = i < nbTiles ? tileEnds[i] : 0u;
        u64 const myA = a; u32 const myB = b;
        u64 ta; u32 tb;
        zb_scan2(a, b, wa, wb, &ta, &tb);
        if (i < nbTiles) { tileLen[i] = carryA + a - myA; tileEnds[i] = carryB + b - myB; }
        __syncthreads();
        if (threadIdx.x == 0) { carryA += ta; carryB += tb; }
        __syncthreads();
    }
    if (threadIdx.x == 0) { ctrl[0] = carryA; ctrl[1] = carryB; }
}

/* explicit delimiters: the block table from the closing delimiters; ctrl[3] = end of the last block */
__global__ void zb_seq_blocks_kernel(const u64* __restrict__ blockEnd, const u32* __restrict__ blockSeq, u32 nbBlocks, u32 blockMax, u32 dictFlag,
                                     ZbBlock* __restrict__ blocks, u32* __restrict__ blockFirst, u64* __restrict__ blockFirstPos,
                                     u64* __restrict__ ctrl, unsigned long long* __restrict__ errIdx)
{
    u32 const k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= nbBlocks) return;
    u64 const start = k ? blockEnd[k - 1u] : 0ull, e = blockEnd[k];
    if (e - start > blockMax) atomicMin(errIdx, (unsigned long long)blockSeq[k]);
    ZbBlock b; b.srcOff = start; b.size = (u32)min(e - start, (u64)blockMax); b.histLen = 0; b.frame = 0; b.dictLen = 0; b.dictSlot = 0;
    b.flags = (k == 0u ? ZB_FLAG_FIRST | dictFlag : 0u) | (k + 1u == nbBlocks ? ZB_FLAG_LAST : 0u);
    blocks[k] = b;
    blockFirst[k] = k ? blockSeq[k - 1u] + 1u : 0u;
    blockFirstPos[k] = start;
    if (k + 1u == nbBlocks) ctrl[3] = e;
}

/* K1s-b: one CTA per block */
__global__ void __launch_bounds__(MERGE_THREADS)
zb_seq_convert_kernel(const u8* __restrict__ src, const ZbBlock* __restrict__ blocks, const u32* __restrict__ blockFirst, const u64* __restrict__ blockFirstPos,
                      const uint4* __restrict__ seqsIn, u32 n, const ZbDictSlot* __restrict__ dicts, ZbStrides sd,
                      u64* __restrict__ seqs, u8* __restrict__ lits, ZbBlockMeta* __restrict__ meta)
{
    __shared__ u32 sPos[MERGE_TILE], sLit[MERGE_TILE], sLen[MERGE_TILE], sOff[MERGE_TILE];
    __shared__ u32 wsumL[MERGE_THREADS / 32], wsumA[MERGE_THREADS / 32], wmaxU[MERGE_THREADS / 32], wmaxK[MERGE_THREADS / 32];
    __shared__ u32 sR2[MERGE_TILE], sRep[3];
    __shared__ u32 baseL, baseA;
    __shared__ u64 wa[MERGE_THREADS / 32]; __shared__ u32 wb[MERGE_THREADS / 32];
    __shared__ long long carryP; __shared__ u32 carryK, carryEnd;
    u32 const b = blockIdx.x, tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    ZbBlock const bd = blocks[b];
    if (bd.size < 7u) {                                          /* zstd_compress.c:3216, as the parse kernels write it */
        if (tid == 0) {
            ZbBlockMeta m; m.nbSeq = 0; m.litSize = bd.size; m.litSecSize = 0; m.bodySize = bd.size;
            m.type = ZB_BT_RAW; m.forceRaw = 1; m.rleByte = 0; m.pad = 0;
            meta[b] = m;
        }
        return;
    }
    u64* const myseq = seqs + (size_t)b * sd.seq;
    u8*  const mylit = lits + (size_t)b * sd.lit;
    const u8* const in = src + bd.srcOff;
    u32 const first = blockFirst[b];
    long long const E = bd.size;                                 /* positions relative to the block's start */
    if (tid == 0) { carryP = first < n ? (long long)blockFirstPos[b] - (long long)bd.srcOff : E; carryK = 0; carryEnd = 0; }
    __syncthreads();
    for (u32 i0 = first; i0 < n; i0 += MERGE_THREADS) {
        u32 const i = i0 + tid;
        uint4 const q = i < n ? seqsIn[i] : make_uint4(0u, 0u, 0u, 0u);
        long long const base = carryP;
        if (base >= E) break;                                    /* uniform: every thread read the same carry */
        u64 a = (u64)q.y + q.z; u32 unused = 0;
        u64 const myLen = a;
        zb_scan2(a, unused, wa, wb, nullptr, nullptr);
        long long const s = base + (long long)(a - myLen), m = s + q.y, e = m + q.z;
        long long const ms = m > 0 ? m : 0, me = e < E ? e : E;
        bool const keep = i < n && s < E && me >= ms + 3;
        /* compaction of the kept match parts, and the end of the last kept part in front of each */
        u32 const kb = __ballot_sync(ZB_FULL, keep);
        u32 const before = __popc(kb & ((1u << lane) - 1u));
        u32 const kEnd = keep ? (u32)me : 0u;                    /* ends grow with the index: a maximum scan finds the last one */
        u32 inc = kEnd;
#pragma unroll
        for (u32 o = 1; o < 32u; o <<= 1) { u32 const x = __shfl_up_sync(ZB_FULL, inc, o); if (lane >= o) inc = max(inc, x); }
        if (lane == 31u) { wsumL[warp] = __popc(kb); wmaxU[warp] = inc; }
        __syncthreads();
        u32 cnt = carryK, prevEnd = carryEnd;
        for (u32 w = 0; w < warp; w++) { cnt += wsumL[w]; prevEnd = max(prevEnd, wmaxU[w]); }
        u32 ex = __shfl_up_sync(ZB_FULL, inc, 1);
        if (lane > 0u) prevEnd = max(prevEnd, ex);
        if (keep) myseq[cnt + before] = zb_pack_seq(q.x, (u32)ms - prevEnd, (u32)(me - ms));
        __syncthreads();
        if (tid == MERGE_THREADS - 1u) {
            u32 tk = 0, te = carryEnd;
            for (u32 w = 0; w < MERGE_THREADS / 32u; w++) { tk += wsumL[w]; te = max(te, wmaxU[w]); }
            carryK += tk; carryEnd = te; carryP = s + (i < n ? (long long)myLen : 0ll);
            if (i + 1u >= n) carryP = E;
        }
        __syncthreads();
    }
    u32 rep[3] = { 1u, 4u, 8u };                                 /* zstd_internal.h:69, or the dictionary's */
    if (dicts && (bd.flags & ZB_FLAG_FIRST)) { rep[0] = dicts[bd.dictSlot].codeRep[0]; rep[1] = dicts[bd.dictSlot].codeRep[1]; rep[2] = dicts[bd.dictSlot].codeRep[2]; }
    zb_merge_codes(rep[0], rep[1], rep[2], (bd.flags & ZB_FLAG_FIRST) != 0u, myseq, mylit, in, carryK, bd.size, meta + b,
                   sPos, sLit, sLen, sOff, sR2, sRep, wsumL, wsumA, wmaxU, wmaxK, baseL, baseA);
}

/* ------------------------------------------------------------------------------------------------ launchers */
extern "C" cudaError_t zb_launch_seq_partition(const void* d_seqs, u32 n, int expl, u64* d_tileLen, u32* d_tileEnds, u64* d_ctrl, cudaStream_t stream)
{
    if (n == 0) return cudaSuccess;
    u32 const nbTiles = (n + SEQ_TILE - 1u) / SEQ_TILE;
    zb_seq_tiles_kernel<false><<<nbTiles, SEQ_THREADS, 0, stream>>>((const uint4*)d_seqs, n, expl != 0, d_tileLen, d_tileEnds, 0, 0, 0, 0, 0,
                                                                   nullptr, nullptr, nullptr, nullptr, nullptr);
    zb_seq_scan_kernel<<<1, SEQ_THREADS, 0, stream>>>(d_tileLen, d_tileEnds, nbTiles, d_ctrl);
    return cudaGetLastError();
}

extern "C" cudaError_t zb_launch_seq_place(const void* d_seqs, u32 n, int expl, const u64* d_tileLen, const u32* d_tileEnds,
                                           u64 srcSize, u64 window, u64 dictContent, u32 blockMax, u32 nbBlocks,
                                           u64* d_blockEnd, u32* d_blockSeq, u32* d_blockFirst, u64* d_blockFirstPos, u64* d_ctrl, cudaStream_t stream)
{
    if (n == 0) return cudaSuccess;
    u32 const nbTiles = (n + SEQ_TILE - 1u) / SEQ_TILE;
    zb_seq_tiles_kernel<true><<<nbTiles, SEQ_THREADS, 0, stream>>>((const uint4*)d_seqs, n, expl != 0, (u64*)d_tileLen, (u32*)d_tileEnds,
                                                                  srcSize, window, dictContent, blockMax, nbBlocks,
                                                                  d_blockEnd, d_blockSeq, d_blockFirst, d_blockFirstPos, (unsigned long long*)(d_ctrl + 2));
    return cudaGetLastError();
}

extern "C" cudaError_t zb_launch_seq_blocks(const u64* d_blockEnd, const u32* d_blockSeq, u32 nbBlocks, u32 blockMax, u32 dictFlag,
                                            ZbBlock* d_blocks, u32* d_blockFirst, u64* d_blockFirstPos, u64* d_ctrl, cudaStream_t stream)
{
    if (nbBlocks == 0) return cudaSuccess;
    zb_seq_blocks_kernel<<<(nbBlocks + 255u) / 256u, 256, 0, stream>>>(d_blockEnd, d_blockSeq, nbBlocks, blockMax, dictFlag, d_blocks, d_blockFirst,
                                                                      d_blockFirstPos, d_ctrl, (unsigned long long*)(d_ctrl + 2));
    return cudaGetLastError();
}

extern "C" cudaError_t zb_launch_seq_convert(const u8* d_src, const ZbBlock* d_blocks, u32 nbBlocks, const u32* d_blockFirst, const u64* d_blockFirstPos,
                                             const void* d_seqs, u32 n, const ZbDictSlot* d_dicts, const ZbWorkRows* rows, cudaStream_t stream)
{
    if (nbBlocks == 0) return cudaSuccess;
    zb_seq_convert_kernel<<<nbBlocks, MERGE_THREADS, 0, stream>>>(d_src, d_blocks, d_blockFirst, d_blockFirstPos, (const uint4*)d_seqs, n, d_dicts, rows->sd,
                                                                 rows->seqs, rows->lits, rows->meta);
    return cudaGetLastError();
}
