/* zb_seqexport.cu — the tail of a ZSTD_generateSequences wave: K1c's stores, exported as ZSTD_Sequence rows.
 *
 * The reference collects each block's seqStore in ZSTD_copyBlockSequences (lib/compress/zstd_compress.c:3370-3447): real
 * offsets, `rep` = the repcode the block codes (1-3, 0 for a direct offset), litLength == 0 shifting the repcodes, and a
 * delimiter {0, trailing literals, 0, 0} behind every block.  Here every block of the wave was parsed at once, so the rows
 * are placed by a scan of the blocks' counts (a block's sequences plus its delimiter), and every block turns its offBase
 * codes back into offsets in parallel (zb_seqexport_kernel).
 */
#include "zb_device.cuh"
#include "zb_kernels.h"

#define EXP_SCAN_THREADS 1024u
#define EXP_THREADS 256u
#define EXP_TILE 1024u                          /* sequences resolved per round */
#define EXP_PER (EXP_TILE / EXP_THREADS)        /* consecutive sequences of a tile owned by one thread */
#define EXP_HIST 3u                             /* slots 0..2: r1, r2, r3 at the tile's start; sequence i of the tile is slot 3 + i */

/* rows a block contributes: its sequences and its delimiter (a block below 7 bytes has no sequences; the empty block of an
 * empty frame has no row) */
__device__ __forceinline__ u32 zb_exportCount(const ZbBlock* blocks, const ZbBlockMeta* meta, u32 i)
{
    return blocks[i].size ? meta[i].nbSeq + 1u : 0u;
}

/* One CTA: offsets[i] = *base + rows of blocks [0, i), offsets[nbBlocks] = *total = *base + rows of the wave.  Every thread
 * sums a contiguous run of blocks; the runs' sums are scanned with warp shuffles, then across the warps. */
__global__ void __launch_bounds__(EXP_SCAN_THREADS)
zb_seqexport_scan_kernel(const ZbBlock* __restrict__ blocks, const ZbBlockMeta* __restrict__ meta, u32 nbBlocks,
                         u64* __restrict__ offsets, const u64* __restrict__ basePtr, u64* __restrict__ total)
{
    __shared__ u64 warpSum[EXP_SCAN_THREADS / 32u];
    u32 const tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    u32 const per = (nbBlocks + EXP_SCAN_THREADS - 1u) / EXP_SCAN_THREADS;
    u32 const beg = min(tid * per, nbBlocks), end = min(beg + per, nbBlocks);
    u64 mine = 0;
    for (u32 i = beg; i < end; i++) mine += zb_exportCount(blocks, meta, i);
    u64 inc = mine;
#pragma unroll
    for (u32 o = 1; o < 32u; o <<= 1) { u64 const x = __shfl_up_sync(ZB_FULL, inc, o); if (lane >= o) inc += x; }
    if (lane == 31u) warpSum[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        u64 const w = warpSum[lane];
        u64 wi = w;
#pragma unroll
        for (u32 o = 1; o < 32u; o <<= 1) { u64 const x = __shfl_up_sync(ZB_FULL, wi, o); if (lane >= o) wi += x; }
        warpSum[lane] = wi - w;                                   /* rows of the warps in front of warp `lane` */
    }
    __syncthreads();
    u64 const base = basePtr ? *basePtr : 0u;
    u64 run = base + warpSum[warp] + inc - mine;
    for (u32 i = beg; i < end; i++) { offsets[i] = run; run += zb_exportCount(blocks, meta, i); }
    if (tid == EXP_SCAN_THREADS - 1u) { offsets[nbBlocks] = run; *total = run; }
}

/* exclusive maximum of v over the threads in front of this one (scratch: EXP_THREADS / 32 u32; one barrier) */
__device__ __forceinline__ u32 zb_exportExclMax(u32 v, u32* scratch)
{
    u32 const lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    u32 inc = v;
#pragma unroll
    for (u32 o = 1; o < 32u; o <<= 1) { u32 const x = __shfl_up_sync(ZB_FULL, inc, o); if (lane >= o) inc = max(inc, x); }
    if (lane == 31u) scratch[warp] = inc;
    u32 ex = __shfl_up_sync(ZB_FULL, inc, 1); if (lane == 0u) ex = 0u;
    __syncthreads();
    for (u32 w = 0; w < warp; w++) ex = max(ex, scratch[w]);
    return ex;
}

/* One CTA per block: the block's rows at out + 4 * offsets[b] (ZSTD_Sequence = 4 u32), none at or past `capacity` rows.
 * A repcode sequence's offset is an earlier offset of the history, so it is resolved backwards along the history's
 * recurrence (the merge's, zb_merge.cuh, read the other way):
 *   - whether a sequence leaves the history alone (U: rep 1 with literals), swaps r1 and r2 (rep 2 with literals, rep 1
 *     without) or shifts it (every other) follows from (offBase, litLength) alone;
 *   - r1 before sequence i is the offset of i - 1; r2 before i is the r1 met by the last non-U sequence in front of i;
 *     r3 before i is the r2 met by the last sequence in front of i that neither leaves the history alone nor swaps;
 * so every repcode sequence names the slot (an earlier sequence of the tile, or the tile's starting history) whose offset it
 * repeats, minus 1 for rep 3 without literals.  Pointer jumping in shared memory then resolves the chains in at most 10
 * rounds per tile.  The history starts as the frame's (d_dicts' codeRep, or {1,4,8}) in a frame's first block and
 * unknown (0) in every other, as the merge starts it. */
__global__ void __launch_bounds__(EXP_THREADS)
zb_seqexport_kernel(const ZbBlock* __restrict__ blocks, const ZbDictSlot* __restrict__ dicts, const ZbBlockMeta* __restrict__ meta,
                    const u64* __restrict__ seqs, u32 seqStride, const u64* __restrict__ offsets, u32* __restrict__ out, u64 capacity)
{
    __shared__ u32 sVal[EXP_HIST + EXP_TILE];   /* a slot's offset: a direct offset or the history's, or (once resolved) any */
    __shared__ u16 sSrc[EXP_HIST + EXP_TILE];   /* the slot whose offset this one repeats; itself when it is known */
    __shared__ u16 sDel[EXP_HIST + EXP_TILE];   /* subtracted from that offset */
    __shared__ u16 sR2[EXP_TILE];                /* the slot of the r2 that sequence i meets */
    __shared__ u32 wmaxU[EXP_THREADS / 32u], wmaxK[EXP_THREADS / 32u];
    __shared__ u32 sNext[EXP_HIST];              /* the slots of the history at the tile's end */
    __shared__ u32 sCovered;
    u32 const b = blockIdx.x, tid = threadIdx.x;
    ZbBlock const bd = blocks[b];
    if (bd.size == 0u) return;
    u32 const nbSeq = meta[b].nbSeq;
    u64 const o0 = offsets[b];
    const u64* const myseq = seqs + (size_t)b * seqStride;
    bool const vec = ((uintptr_t)out & 15u) == 0u;
    if (tid < EXP_HIST) {
        u32 r = 0;
        if (bd.flags & ZB_FLAG_FIRST) r = dicts ? dicts[bd.dictSlot].codeRep[tid] : (tid == 0u ? 1u : (tid == 1u ? 4u : 8u));
        sVal[tid] = r; sSrc[tid] = (u16)tid; sDel[tid] = 0;
    }
    if (tid == 0) sCovered = 0;
    __syncthreads();
    u32 covered = 0;
    for (u32 t0 = 0; t0 < nbSeq; t0 += EXP_TILE) {
        u32 const n = min(EXP_TILE, nbSeq - t0);
        u32 code[EXP_PER], ll[EXP_PER], bef[EXP_PER], r2s[EXP_PER];
        bool U[EXP_PER], K[EXP_PER];
        u32 run = 0;
#pragma unroll
        for (u32 j = 0; j < EXP_PER; j++) {
            u32 const i = tid * EXP_PER + j;
            u64 const q = i < n ? myseq[t0 + i] : 0ull;
            code[j] = ZB_SEQ_OFFBASE(q); ll[j] = ZB_SEQ_LL(q);
            covered += ll[j] + ZB_SEQ_ML(q);
            U[j] = code[j] == 1u && ll[j] > 0u;
            K[j] = U[j] || (code[j] == 2u && ll[j] > 0u) || (code[j] == 1u && ll[j] == 0u);
            bef[j] = run;                                            /* 1 + index of the last non-U sequence of mine before this one */
            if (i < n && !U[j]) run = i + 1u;
        }
        {   u32 const ex = zb_exportExclMax(run, wmaxU);
#pragma unroll
            for (u32 j = 0; j < EXP_PER; j++) {
                u32 const i = tid * EXP_PER + j;
                u32 const m = max(bef[j], ex);                       /* 1 + index of the last non-U sequence before i, 0: none */
                r2s[j] = m == 0u ? 1u : (m == 1u ? 0u : m + 1u);     /* the r1 met by sequence m - 1: slot of m - 2, or r1 */
                if (i < n) sR2[i] = (u16)r2s[j];
            }
        }
        run = 0;
#pragma unroll
        for (u32 j = 0; j < EXP_PER; j++) {
            u32 const i = tid * EXP_PER + j;
            bef[j] = run;
            if (i < n && !K[j]) run = i + 1u;
        }
        {   u32 const ex = zb_exportExclMax(run, wmaxK);             /* its barrier also completes sR2 */
#pragma unroll
            for (u32 j = 0; j < EXP_PER; j++) {
                u32 const i = tid * EXP_PER + j;
                if (i >= n) continue;
                u32 const m = max(bef[j], ex);
                u32 const r3s = m == 0u ? 2u : sR2[m - 1u];          /* the r2 met by sequence m - 1 */
                u32 const r1s = i == 0u ? 0u : i + EXP_HIST - 1u;
                u32 const x = i + EXP_HIST;
                u32 src = x, del = 0;
                if (code[j] <= 3u) {
                    if (ll[j] > 0u) src = code[j] == 1u ? r1s : (code[j] == 2u ? r2s[j] : r3s);
                    else if (code[j] == 3u) { src = r1s; del = 1u; }
                    else src = code[j] == 1u ? r2s[j] : r3s;
                }
                sVal[x] = code[j] - 3u; sSrc[x] = (u16)src; sDel[x] = (u16)del;
                if (i == n - 1u) { sNext[0] = x; sNext[1] = U[j] ? r2s[j] : r1s; sNext[2] = K[j] ? r3s : r2s[j]; }
            }
        }
        __syncthreads();
        /* pointer jumping: every slot ends pointing at a known offset, its deltas summed on the way */
        for (;;) {
            u32 ns[EXP_PER], nd[EXP_PER];
            bool moved = false;
#pragma unroll
            for (u32 j = 0; j < EXP_PER; j++) {
                u32 const x = tid * EXP_PER + j + EXP_HIST;
                u32 const s = x < n + EXP_HIST ? sSrc[x] : x;
                ns[j] = s; nd[j] = 0;
                if (s != x && sSrc[s] != s) { ns[j] = sSrc[s]; nd[j] = sDel[x] + sDel[s]; moved = true; }
            }
            __syncthreads();
#pragma unroll
            for (u32 j = 0; j < EXP_PER; j++) {
                u32 const x = tid * EXP_PER + j + EXP_HIST;
                if (x < n + EXP_HIST && ns[j] != sSrc[x]) { sSrc[x] = (u16)ns[j]; sDel[x] = (u16)nd[j]; }
            }
            if (!__syncthreads_or(moved)) break;
        }
        {   u32 v[EXP_PER];
#pragma unroll
            for (u32 j = 0; j < EXP_PER; j++) {
                u32 const x = tid * EXP_PER + j + EXP_HIST;
                v[j] = x < n + EXP_HIST ? sVal[sSrc[x]] - sDel[x] : 0u;
            }
            __syncthreads();
#pragma unroll
            for (u32 j = 0; j < EXP_PER; j++) {
                u32 const x = tid * EXP_PER + j + EXP_HIST;
                if (x < n + EXP_HIST) { sVal[x] = v[j]; sSrc[x] = (u16)x; }
            }
            __syncthreads();
        }
        /* the tile's rows, one per thread at a time: consecutive threads write consecutive rows */
        for (u32 i = tid; i < n; i += EXP_THREADS) {
            u64 const g = o0 + t0 + i;
            if (g >= capacity) break;
            u64 const q = myseq[t0 + i];
            u32 const c = ZB_SEQ_OFFBASE(q);
            uint4 const row = make_uint4(sVal[i + EXP_HIST], ZB_SEQ_LL(q), ZB_SEQ_ML(q), c <= 3u ? c : 0u);
            u32* const p = out + 4u * g;
            if (vec) *reinterpret_cast<uint4*>(p) = row;
            else { p[0] = row.x; p[1] = row.y; p[2] = row.z; p[3] = row.w; }
        }
        u32 const h = tid < EXP_HIST ? sVal[sNext[tid]] : 0u;
        __syncthreads();
        if (tid < EXP_HIST) sVal[tid] = h;                           /* the next tile's history */
        __syncthreads();
    }
    /* the delimiter: the block's trailing literals */
#pragma unroll
    for (u32 o = 16; o > 0u; o >>= 1) covered += __shfl_down_sync(ZB_FULL, covered, o);
    if ((tid & 31u) == 0u && covered) atomicAdd(&sCovered, covered);
    __syncthreads();
    if (tid == 0) {
        u64 const g = o0 + nbSeq;
        if (g < capacity) {
            u32* const p = out + 4u * g;
            uint4 const row = make_uint4(0u, bd.size - sCovered, 0u, 0u);
            if (vec) *reinterpret_cast<uint4*>(p) = row;
            else { p[0] = row.x; p[1] = row.y; p[2] = row.z; p[3] = row.w; }
        }
    }
}

extern "C" cudaError_t zb_launch_seqexport(const ZbBlock* d_blocks, u32 nbBlocks, const ZbDictSlot* d_dicts, const ZbWorkRows* rows,
                                           u64* d_offsets, const u64* d_base, u64* d_total, void* d_out, u64 capacity, cudaStream_t stream)
{
    if (nbBlocks == 0) return cudaSuccess;
    zb_seqexport_scan_kernel<<<1, EXP_SCAN_THREADS, 0, stream>>>(d_blocks, rows->meta, nbBlocks, d_offsets, d_base, d_total);
    zb_seqexport_kernel<<<nbBlocks, EXP_THREADS, 0, stream>>>(d_blocks, d_dicts, rows->meta, rows->seqs, rows->sd.seq, d_offsets,
                                                              (u32*)d_out, capacity);
    return cudaGetLastError();
}
