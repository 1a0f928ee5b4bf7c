/* zb_sequences.cu — K3: sequences section of one block per CTA + final block-type decision.
 *
 * Replaces, for a fresh entropy state, ZSTD_buildSequencesStatistics
 * (lib/compress/zstd_compress.c:2755-2873), ZSTD_seqToCodes (:2686-2712),
 * ZSTD_selectEncodingType / ZSTD_buildCTable (zstd_compress_sequences.c:157-288),
 * ZSTD_encodeSequences_body (:291-382) and the block-level checks of
 * ZSTD_entropyCompressSeqStore (zstd_compress.c:2987-2993, :3025-3028) and
 * ZSTD_compressBlock_internal (:4365-4376).
 *
 *   1. LL/OF/ML codes + three histograms: all threads, shared-memory atomics
 *   2. per stream (one warp each): encoding type, normalised counts (largest remainders), NCount header, FSE table
 *      (zb_entropy.cuh); predefined tables are built once per device by the host and copied
 *   3. tANS state chains: state(i) depends on state(i+1) (common/fse.h:463-470), so each of the three
 *      chains is walked backwards by one lane (the three lanes share a warp); it records (bits, nbBits) per sequence
 *   4. all threads: per-sequence bit counts -> suffix sum -> bit offsets -> pack (edge words atomicOr)
 */
#include "zb_entropy.cuh"
#include "zb_kernels.h"
#include "zb_bitpack.cuh"

#define SEQ_THREADS 128
#ifndef SEQ_TILE
#define SEQ_TILE 512u                /* sequences whose chain steps are prepared at a time (3 x 2 KiB of shared memory) */
#endif
#define MaxLL 35
#define MaxML 52
#define MaxOff 31
#define DefaultMaxOff 28
#define LLFSELog 9
#define MLFSELog 9
#define OffFSELog 8

/* format constants, common/zstd_internal.h:123-168 (RFC 8878) */
__constant__ short c_LL_defaultNorm[MaxLL + 1] = { 4,3,2,2,2,2,2,2, 2,2,2,2,2,1,1,1, 2,2,2,2,2,2,2,2, 2,3,2,1,1,1,1,1, -1,-1,-1,-1 };
__constant__ short c_ML_defaultNorm[MaxML + 1] = { 1,4,3,2,2,2,2,2, 2,1,1,1,1,1,1,1, 1,1,1,1,1,1,1,1, 1,1,1,1,1,1,1,1,
                                                   1,1,1,1,1,1,1,1, 1,1,1,1,1,1,-1,-1, -1,-1,-1,-1,-1 };
__constant__ short c_OF_defaultNorm[DefaultMaxOff + 1] = { 1,1,1,1,1,1,2,2, 2,1,1,1,1,1,1,1, 1,1,1,1,1,1,1,1, -1,-1,-1,-1,-1 };

/* closed forms of the code tables in zstd_compress_internal.h:520-549 and of the extra-bit counts (LL_bits / ML_bits,
 * common/zstd_internal.h:123-137): only used to fill the CTA's look-up tables for values below 64 (LL) / 128 (ML); above
 * that the code is highbit + 19 (+ 36) and carries highbit extra bits */
__device__ __forceinline__ u32 zbd_ll_code(u32 ll)
{
    if (ll > 63u) return zb_hb32(ll) + 19u;
    if (ll < 16u) return ll;
    if (ll < 24u) return 16u + ((ll - 16u) >> 1);
    if (ll < 32u) return 20u + ((ll - 24u) >> 2);
    if (ll < 48u) return 22u + ((ll - 32u) >> 3);
    return 24u;
}
__device__ __forceinline__ u32 zbd_ml_code(u32 mlBase)
{
    if (mlBase > 127u) return zb_hb32(mlBase) + 36u;
    if (mlBase < 32u) return mlBase;
    if (mlBase < 40u) return 32u + ((mlBase - 32u) >> 1);
    if (mlBase < 48u) return 36u + ((mlBase - 40u) >> 2);
    if (mlBase < 64u) return 38u + ((mlBase - 48u) >> 3);
    if (mlBase < 96u) return 40u + ((mlBase - 64u) >> 4);
    return 42u;
}
__device__ __forceinline__ u32 zbd_ll_lut_entry(u32 ll)       /* ll < 64: code | extra bits << 8 */
{
    u32 const c = zbd_ll_code(ll);
    return c | ((c < 16u ? 0u : (c < 20u ? 1u : (c < 22u ? 2u : (c < 24u ? 3u : 4u)))) << 8);
}
__device__ __forceinline__ u32 zbd_ml_lut_entry(u32 mlBase)   /* mlBase < 128 */
{
    u32 const c = zbd_ml_code(mlBase);
    return c | ((c < 32u ? 0u : (c < 36u ? 1u : (c < 38u ? 2u : (c < 40u ? 3u : (c < 42u ? 4u : 5u))))) << 8);
}
struct ZbdCodeLut { u16 ll[64]; u16 ml[128]; };               /* shared memory, filled once per CTA: the branches of the closed forms diverge */
struct ZbdSeq { u32 offBase, litLen, mlBase, llc, ofc, mlc, llBits, mlBits; };
__device__ __forceinline__ ZbdSeq zbd_unpack(u64 q, const ZbdCodeLut& lut)
{
    ZbdSeq s;
    s.offBase = ZB_SEQ_OFFBASE(q);
    s.litLen = ZB_SEQ_LL(q);
    s.mlBase = ZB_SEQ_ML(q) - 3u;
    u32 const le = lut.ll[s.litLen < 63u ? s.litLen : 63u], lh = zb_hb32(s.litLen | 1u);
    u32 const me = lut.ml[s.mlBase < 127u ? s.mlBase : 127u], mh = zb_hb32(s.mlBase | 1u);
    bool const lBig = s.litLen > 63u, mBig = s.mlBase > 127u;
    s.llc = lBig ? lh + 19u : (le & 0xFFu);  s.llBits = lBig ? lh : (le >> 8);
    s.mlc = mBig ? mh + 36u : (me & 0xFFu);  s.mlBits = mBig ? mh : (me >> 8);
    s.ofc = zb_hb32(s.offBase);
    return s;
}

enum { set_basic = 0, set_rle = 1, set_compressed = 2, set_repeat = 3 };

/* zstd_compress_sequences.c:157-240, branch strategy < ZSTD_lazy with repeatMode == none */
__device__ __forceinline__ u32 zbd_selectEncodingType(u32 mostFrequent, u32 nbSeq, u32 defaultNormLog, bool defaultAllowed, u32 strategy, u32 prevRepeat)
{
    if (mostFrequent == nbSeq) return (defaultAllowed && nbSeq <= 2u) ? set_basic : set_rle;
    if (defaultAllowed) {
        u32 const mult = 10u - strategy;
        u32 const dynamicFse_nbSeq_min = ((1u << defaultNormLog) * mult) >> 3;
        if (prevRepeat == 2u && nbSeq < 1000u) return set_repeat;             /* :187-191 : the dictionary's table */
        if (nbSeq < dynamicFse_nbSeq_min || mostFrequent < (nbSeq >> (defaultNormLog - 1u))) return set_basic;
    }
    return set_compressed;
}

/* the three predefined tables (format "Default Distributions"), built by the host once per device (zb_dict.cu) */
__device__ ZbdFseCTable g_defaultCT[3];                          /* 0 = LL, 1 = OF, 2 = ML */
extern "C" cudaError_t zb_upload_default_tables(const ZbdFseCTable* host3, cudaStream_t stream)
{
    return cudaMemcpyToSymbolAsync(g_defaultCT, host3, 3 * sizeof(ZbdFseCTable), 0, cudaMemcpyHostToDevice, stream);
}

struct ZbdStreamWork {
    u32 count[64];
    short norm[64];
    u8  nc[136];            /* NCount bytes (or the single rle symbol) */
    u8  symAt[512];         /* table-build scratch: symbol of every cell */
    u16 cum[66];
    u32 ncSize;
    u32 type;
    u32 finalState;
    u32 err;
};

__global__ void __launch_bounds__(SEQ_THREADS)
zb_sequences_kernel(const u8* __restrict__ src, const ZbBlock* __restrict__ blocks, ZbParams prm, ZbStrides sd, const ZbDictEntropy* __restrict__ deAll,
                    const ZbDictSlot* __restrict__ dicts,
                    const u64* __restrict__ seqs, u16* __restrict__ stateBits,
                    u8* __restrict__ body, ZbBlockMeta* __restrict__ meta)
{
    __shared__ ZbdFseCTable ct[3];                 /* 0 = LL, 1 = OF, 2 = ML */
    __shared__ ZbdStreamWork wk[3];
    __shared__ u32 chunkBits[SEQ_THREADS];
    __shared__ u32 stepTile[3][SEQ_TILE + 3u];     /* per chain and sequence of a tile: deltaNbBits (20 bits, >= 0) | deltaFindState << 20 (signed), from word 1 on (word 0 is read, never used);
                                                    * odd stride: the three chains read different banks */
    __shared__ u32 sh_cSize, sh_hdrEnd, sh_streamSize;
    __shared__ ZbdCodeLut lut;

    u32 const tid = threadIdx.x;
    u32 const b = blockIdx.x;
    ZbBlockMeta const m = meta[b];
    ZbBlock const bd = blocks[b];
    if (m.forceRaw) return;
    const ZbDictEntropy* const de = (bd.flags & ZB_FLAG_FIRST) ? (dicts ? dicts[bd.dictSlot].de : deAll) : nullptr;
    u32 const nbSeq = m.nbSeq;
    const u64* const myseq = seqs + (size_t)b * sd.seq;
    u16* const myst = stateBits + (size_t)b * sd.dist;       /* the block's (dead) candidate-distance area */
    u8* const out = body + (size_t)b * sd.body;
    u32 op = m.litSecSize;

    /* nbSeq header, zstd_compress.c:2937-2947 */
    u32 const nbSeqHdr = nbSeq < 128u ? 1u : (nbSeq < 0x7F00u ? 2u : 3u);
    if (tid == 0) {
        if (nbSeq < 128u) out[op] = (u8)nbSeq;
        else if (nbSeq < 0x7F00u) { out[op] = (u8)((nbSeq >> 8) + 0x80u); out[op + 1] = (u8)nbSeq; }
        else { out[op] = 0xFF; out[op + 1] = (u8)(nbSeq - 0x7F00u); out[op + 2] = (u8)((nbSeq - 0x7F00u) >> 8); }
    }
    op += nbSeqHdr;
    u32 cSize;
    if (nbSeq == 0) {
        cSize = op;
    } else {
        /* ---- 1. codes + histograms ---- */
        for (u32 i = tid; i < 192u; i += SEQ_THREADS) wk[i >> 6].count[i & 63u] = 0;
        for (u32 i = tid; i < 192u; i += SEQ_THREADS) { if (i < 64u) lut.ll[i] = (u16)zbd_ll_lut_entry(i); else lut.ml[i - 64u] = (u16)zbd_ml_lut_entry(i - 64u); }
        __syncthreads();
        for (u32 i = tid; i < nbSeq; i += SEQ_THREADS) {
            ZbdSeq const s = zbd_unpack(myseq[i], lut);
            atomicAdd(&wk[0].count[s.llc], 1u);
            atomicAdd(&wk[1].count[s.ofc], 1u);
            atomicAdd(&wk[2].count[s.mlc], 1u);
        }
        __syncthreads();
        /* ---- 2. per-stream tables: warps 0, 1, 2 ---- */
        if (tid < 96u) {
            u32 const st = tid >> 5, lane = tid & 31u;
            ZbdStreamWork* const w = &wk[st];
            u32 const maxAll = st == 0 ? MaxLL : (st == 1 ? MaxOff : MaxML);
            u32 const c0 = w->count[lane], c1 = (lane + 32u <= maxAll) ? w->count[lane + 32u] : 0u;
            u32 const hiUsed = __ballot_sync(ZB_FULL, c1 != 0u), loUsed = __ballot_sync(ZB_FULL, c0 != 0u);
            u32 const max = hiUsed ? 63u - (u32)__clz((int)hiUsed) : 31u - (u32)__clz((int)loUsed);
            u32 mostFrequent = c0 > c1 ? c0 : c1;
#pragma unroll
            for (u32 o = 16; o > 0; o >>= 1) mostFrequent = ::max(mostFrequent, __shfl_xor_sync(ZB_FULL, mostFrequent, o));
            u32 const defLog = st == 1 ? 5u : 6u;
            bool const defAllowed = st == 1 ? (max <= DefaultMaxOff) : true;
            u32 const prevRepeat = (de != nullptr && de->present) ? de->fseRepeat[st] : 0u;
            u32 const type = zbd_selectEncodingType(mostFrequent, nbSeq, defLog, defAllowed, prm.strategy, prevRepeat);
            if (lane == 0) { w->type = type; w->err = 0; w->ncSize = 0; }
            __syncwarp();
            if (type == set_repeat || type == set_basic) {           /* a ready table: the dictionary's (zstd_compress_sequences.c:260-262) or the predefined one */
                const u32* from = reinterpret_cast<const u32*>(type == set_repeat ? &de->fse[st] : &g_defaultCT[st]);
                u32* to = reinterpret_cast<u32*>(&ct[st]);
                for (u32 i = lane; i < sizeof(ZbdFseCTable) / 4u; i += 32u) to[i] = from[i];
            } else if (type == set_rle) {                            /* zstd_compress_sequences.c:254-259 */
                if (lane == 0) {
                    ZbdSeq const first = zbd_unpack(myseq[0], lut);
                    u32 const sym = st == 0 ? first.llc : (st == 1 ? first.ofc : first.mlc);
                    zbd_fse_buildCTable_rle(&ct[st], max);
                    w->nc[0] = (u8)sym; w->ncSize = 1;
                }
            } else {
                u32 const FSELog = st == 1 ? OffFSELog : (st == 0 ? LLFSELog : MLFSELog);
                u32 nbSeq_1 = nbSeq;
                u32 const tableLog = zbd_fse_optimalTableLog(FSELog, nbSeq, max, 2);
                {   /* the last sequence's symbols start the states and cost no bits (zstd_compress_sequences.c:271-274) */
                    ZbdSeq const last = zbd_unpack(myseq[nbSeq - 1], lut);
                    u32 const lastCode = st == 0 ? last.llc : (st == 1 ? last.ofc : last.mlc);
                    if (w->count[lastCode] > 1u) { nbSeq_1--; __syncwarp(); if (lane == 0) w->count[lastCode]--; }
                    __syncwarp();
                }
                u32 const r = zbw_fse_normalize(w->norm, tableLog, w->count, nbSeq_1, max, lane);
                u32 ncs = 0;
                if (r != ZBD_ERR) { if (lane == 0) ncs = zbd_fse_writeNCount(w->nc, w->norm, max, tableLog); ncs = __shfl_sync(ZB_FULL, ncs, 0); }
                if (r == ZBD_ERR || ncs == ZBD_ERR) { if (lane == 0) w->err = 1; }
                else {
                    if (lane == 0) w->ncSize = ncs;
                    zbw_fse_buildCTable(&ct[st], w->norm, max, tableLog, w->symAt, w->cum, lane);
                }
            }
        }
        __syncthreads();
        bool const err = wk[0].err | wk[1].err | wk[2].err;
        if (err) { if (tid == 0) { meta[b].type = ZB_BT_RAW; meta[b].bodySize = bd.size; } return; }

        /* ---- 3. state chains.  The only loop-carried value of a chain is `state` (common/fse.h:463-470): everything
         * else is prepared in parallel.  The sequences are walked last to first in tiles; all threads turn a tile's
         * LL/OF/ML codes into the chains' per-step words (the symbol's deltaNbBits | deltaFindState << 20), then lanes
         * 0, 1, 2 of ONE warp walk the three chains side by side — a lane that walks alone costs a whole warp's issue
         * slot per instruction, three lanes in one warp cost the same slot once.  A step is: word of the next step
         * requested, bits shed, record stored, next-state look-up. ---- */
        {
            u32 state = 0;
            bool const chain = tid < 3u;
            u32 const st = chain ? tid : 0u;
            const u16* const ns = ct[st].nextState;
            const u32* const tw = stepTile[st] + 1;
            u16* const rec = myst + (size_t)st * sd.state;
            u32 const nbTiles = (nbSeq + SEQ_TILE - 1u) / SEQ_TILE;
            for (u32 tile = nbTiles; tile-- > 0; ) {
                u32 const t0 = tile * SEQ_TILE, t1 = min(t0 + SEQ_TILE, nbSeq);
                for (u32 i = t0 + tid; i < t1; i += SEQ_THREADS) {
                    ZbdSeq const s = zbd_unpack(myseq[i], lut);
                    stepTile[0][i - t0 + 1u] = ct[0].deltaNbBits[s.llc] | ((u32)ct[0].deltaFindState[s.llc] << 20);
                    stepTile[1][i - t0 + 1u] = ct[1].deltaNbBits[s.ofc] | ((u32)ct[1].deltaFindState[s.ofc] << 20);
                    stepTile[2][i - t0 + 1u] = ct[2].deltaNbBits[s.mlc] | ((u32)ct[2].deltaFindState[s.mlc] << 20);
                }
                __syncthreads();
                if (chain) {
                    u32 cnt = t1 - t0;                                   /* steps of this tile, last sequence first */
                    const u32* pw = tw + cnt;                            /* pw[-1] = word of the sequence in turn */
                    u16* pr = rec + t1;
                    if (t1 == nbSeq) {                                   /* last sequence: its symbols start the states and cost no bits */
                        u32 const w0 = pw[-1], dnb = w0 & 0xFFFFFu;
                        u32 const nbOut = (dnb + (1u << 15)) >> 16;
                        state = ns[(int)(((nbOut << 16) - dnb) >> nbOut) + ((int)w0 >> 20)];
                        cnt--; pw--; pr--;
                    }
                    u32 w = pw[-1];                                      /* tw[-1] exists (padding word): no guard */
                    while (cnt) {
                        cnt--; pw--; pr--;
                        u32 const wn = pw[-1];                           /* next step's word, in flight during this step */
                        u32 const nb = (state + (w & 0xFFFFFu)) >> 16;
                        *pr = (u16)((state & ((1u << nb) - 1u)) | (nb << 12));
                        state = ns[(int)(state >> nb) + ((int)w >> 20)];
                        w = wn;
                    }
                }
                __syncthreads();
            }
            if (chain) wk[st].finalState = state;
        }
        __syncthreads();

        /* ---- section header bytes: seqHead + NCounts (zstd_compress.c:2955-2966) ---- */
        u32 const ncTotal = wk[0].ncSize + wk[1].ncSize + wk[2].ncSize;
        u32 const hdrEnd = op + 1u + ncTotal;        /* first byte of the bit-stream */
        u32 lastCountSize = 0;
        if (wk[0].type == set_compressed) lastCountSize = wk[0].ncSize;
        if (wk[1].type == set_compressed) lastCountSize = wk[1].ncSize;
        if (wk[2].type == set_compressed) lastCountSize = wk[2].ncSize;

        /* ---- 4. per-sequence bit counts, suffix sums ---- */
        u32 const cs = (nbSeq + SEQ_THREADS - 1u) / SEQ_THREADS;
        u32 const cBeg = min(tid * cs, nbSeq), cEnd = min((tid + 1u) * cs, nbSeq);
        u32 bits = 0;
        for (u32 i = cBeg; i < cEnd; i++) {
            ZbdSeq const s = zbd_unpack(myseq[i], lut);
            bits += s.llBits + s.mlBits + s.ofc;
            if (i + 1u < nbSeq) bits += (myst[i] >> 12) + (myst[sd.state + i] >> 12) + (myst[2u * sd.state + i] >> 12);
        }
        chunkBits[tid] = bits;
        __syncthreads();
        u32 bitOff = 0;
        for (u32 k = tid + 1u; k < SEQ_THREADS; k++) bitOff += chunkBits[k];
        if (tid == 0) {
            u32 const totalBits = bitOff + bits + ct[2].tableLog + ct[1].tableLog + ct[0].tableLog + 1u;
            sh_streamSize = (totalBits + 7u) >> 3;
        }
        __syncthreads();
        u32 const streamSize = sh_streamSize;
        cSize = hdrEnd + streamSize;
        /* the body staging area is sd.body bytes; a block that large is emitted raw anyway */
        bool const fits = (cSize + 16u <= sd.body);
        if (fits) {
            /* zero the bit-stream words (the first may share bytes with the headers: keep those) */
            u32 const w0 = hdrEnd >> 2, w1 = (cSize + 3u) >> 2;
            u32* const ow = reinterpret_cast<u32*>(out);
            for (u32 i = w0 + 1u + tid; i < w1; i += SEQ_THREADS) ow[i] = 0;
            if (tid == 0) {
                for (u32 i = hdrEnd; i < min((w0 + 1u) << 2, cSize + 4u); i++) out[i] = 0;
                u8* p = out + op;
                *p++ = (u8)((wk[0].type << 6) + (wk[1].type << 4) + (wk[2].type << 2));
                for (u32 st = 0; st < 3; st++) for (u32 i = 0; i < wk[st].ncSize; i++) *p++ = wk[st].nc[i];
            }
            __syncthreads();
            ZbdParW pw; zbd_pw_init(&pw, ow, (u64)hdrEnd * 8u + bitOff);
            for (u32 i = cEnd; i-- > cBeg; ) {                 /* last sequence first, zstd_compress_sequences.c:311-370 */
                ZbdSeq const s = zbd_unpack(myseq[i], lut);
                if (i + 1u < nbSeq) {
                    u32 const rOF = myst[sd.state + i], rML = myst[2u * sd.state + i], rLL = myst[i];
                    zbd_pw_add(&pw, rOF & 0xFFFu, rOF >> 12);
                    zbd_pw_add(&pw, rML & 0xFFFu, rML >> 12);
                    zbd_pw_add(&pw, rLL & 0xFFFu, rLL >> 12);
                }
                u32 const llb = s.llBits, mlb = s.mlBits;
                zbd_pw_add(&pw, s.litLen & ((1u << llb) - 1u), llb);
                zbd_pw_add(&pw, s.mlBase & ((1u << mlb) - 1u), mlb);
                zbd_pw_add(&pw, s.offBase & ((1u << s.ofc) - 1u), s.ofc);
            }
            if (tid == 0) {                                    /* :372-376 + end mark */
                zbd_pw_add(&pw, wk[2].finalState & ((1u << ct[2].tableLog) - 1u), ct[2].tableLog);
                zbd_pw_add(&pw, wk[1].finalState & ((1u << ct[1].tableLog) - 1u), ct[1].tableLog);
                zbd_pw_add(&pw, wk[0].finalState & ((1u << ct[0].tableLog) - 1u), ct[0].tableLog);
                zbd_pw_add(&pw, 1u, 1u);
            }
            zbd_pw_finish(&pw);
        }
        if (!fits || (lastCountSize && (lastCountSize + streamSize) < 4u)) cSize = 0;    /* zstd_compress.c:2987-2993 */
    }

    /* ---- block-level decision (zstd_compress.c:3025-3028, :4365-4376) ---- */
    {   u32 const maxCSize = bd.size - ((bd.size >> 6) + 2u);
        if (cSize >= maxCSize) cSize = 0;
    }
    bool rle = false;
    if (!(bd.flags & ZB_FLAG_FIRST) && cSize < 25u) {
        const u8* const bsrc = src + bd.srcOff;
        u8 const v0 = bsrc[0];
        int diff = 0;
        for (u32 i = tid; i < bd.size; i += SEQ_THREADS) diff |= (bsrc[i] != v0);
        rle = !__syncthreads_or(diff);
    }
    if (tid == 0) {
        ZbBlockMeta mm = m;
        if (rle) { mm.type = ZB_BT_RLE; mm.bodySize = 1; mm.rleByte = src[bd.srcOff]; }
        else if (cSize == 0) { mm.type = ZB_BT_RAW; mm.bodySize = bd.size; }
        else { mm.type = ZB_BT_COMPRESSED; mm.bodySize = cSize; }
        meta[b] = mm;
    }
}

extern "C" cudaError_t zb_launch_sequences(const u8* d_src, const ZbBlock* d_blocks, u32 nbBlocks, const ZbParams* prm, const ZbStrides* sd, const ZbDictEntropy* d_de,
                                           const u64* d_seqs, u16* d_stateBits, u8* d_body, ZbBlockMeta* d_meta, cudaStream_t stream,
                                           const ZbDictSlot* d_dicts)
{
    if (nbBlocks == 0) return cudaSuccess;
    zb_sequences_kernel<<<nbBlocks, SEQ_THREADS, 0, stream>>>(d_src, d_blocks, *prm, *sd, d_de, d_dicts, d_seqs, d_stateBits, d_body, d_meta);
    return cudaGetLastError();
}
