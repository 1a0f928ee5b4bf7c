/* zb_literals.cu — K2: literals section of one block per CTA.
 *
 * Replaces ZSTD_compressLiterals (lib/compress/zstd_compress_literals.c:129-235)
 * and HUF_compress_internal (huf_compress.c:1333-1430) for a fresh entropy state:
 *   1. 256-bin histogram: warp w counts the bytes of Huffman stream w into its own shared-memory bins, count[] is the sum
 *      of the four (hist.c:66-133)
 *   2. raw / RLE / compressed decision with the reference's thresholds
 *   3. Huffman table + tree description: the whole CTA (zb_entropy.cuh)
 *   4. 1 or 4 streams (huf_compress.c:1056-1118, :1168-1215): a stream's size is its histogram dotted with the code
 *      lengths, so every size and offset is known before any packing; then warp s encodes stream s in one pass
 *      (zb_huf_stream).
 * Output: body[0 .. litSecSize) of the block's staging area; meta.litSecSize.
 */
#include "zb_entropy.cuh"
#include "zb_kernels.h"

#define LIT_THREADS 128               /* one warp per Huffman stream */
#ifndef LIT_MIN_CTAS
#define LIT_MIN_CTAS 12               /* 40 registers.  H100, literals per GiB of config 2: 8 CTAs (56 registers) 1.35-1.37 ms,
                                       * 10 (48) 1.39-1.40, 12 1.39-1.41, and the same wave totals; on config 5 (1 KiB blocks)
                                       * 8 took 6.52 ms against 6.36.  16 would spill at 32 registers. */
#endif
#define LIT_WARPS (LIT_THREADS / 32)
#define LIT_WIN 256u                  /* words of a warp's encoding window: a tile adds at most 512 codes x 12 bits = 192 words */

/* histogram of src[0..n) into count[256]; warp w counts the bytes [w * seg, (w + 1) * seg), seg = ceil(n / 4), into
 * whist[w]: over a literal buffer of four Huffman streams, whist[w] is stream w's histogram.  16-byte aligned vector
 * loads, bytes outside the warp's range masked. */
__device__ void zb_hist256(const u8* __restrict__ src, u32 n, u32 (*whist)[256], u32* count)
{
    u32 const tid = threadIdx.x, warp = tid >> 5, lane = tid & 31u;
    for (u32 i = tid; i < LIT_WARPS * 256; i += LIT_THREADS) (&whist[0][0])[i] = 0;
    __syncthreads();
    u32 const head = (u32)((uintptr_t)src & 15u);                      /* src[i] is byte i + head of the vectors */
    const uint4* const v4 = reinterpret_cast<const uint4*>(src - head);
    u32 const seg = (n + 3u) / 4u;
    u32 const beg = min(warp * seg, n) + head, end = min((warp + 1u) * seg, n) + head;
    if (beg < end) {
        u32 const vLo = beg >> 4, nVec = ((end - 1u) >> 4) - vLo + 1u;
        uint4 nx = lane < nVec ? __ldg(v4 + vLo + lane) : make_uint4(0, 0, 0, 0);
        for (u32 i = lane; i < nVec; i += 32u) {
            uint4 const q = nx;
            if (i + 32u < nVec) nx = __ldg(v4 + vLo + i + 32u);
            u32 const p0 = (vLo + i) << 4;
            u32 const kLo = beg > p0 ? beg - p0 : 0u, kHi = min(end - p0, 16u);     /* bytes [kLo, kHi) are the warp's */
            u32 const w[4] = { q.x, q.y, q.z, q.w };
#pragma unroll
            for (u32 k = 0; k < 16u; k++)
                if (k >= kLo && k < kHi) atomicAdd(&whist[warp][(w[k >> 2] >> (8u * (k & 3u))) & 0xFFu], 1u);
        }
    }
    __syncthreads();
    for (u32 sym = tid; sym < 256u; sym += LIT_THREADS) {
        u32 s = 0;
#pragma unroll
        for (int w = 0; w < LIT_WARPS; w++) s += whist[w][sym];
        count[sym] = s;
    }
    __syncthreads();
}

/* largest count and highest non-zero symbol of count[256] (block-wide) */
__device__ void zb_hist_stats(const u32* count, u32* red, u32* largestOut, u32* maxSymOut)
{
    u32 const tid = threadIdx.x;
    u32 c = 0, key = 0;
    for (u32 sym = tid; sym < 256u; sym += LIT_THREADS) { u32 const v = count[sym]; c = max(c, v); key = max(key, v ? sym : 0u); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        c = max(c, __shfl_xor_sync(ZB_FULL, c, o));
        key = max(key, __shfl_xor_sync(ZB_FULL, key, o));
    }
    if ((tid & 31) == 0) { red[tid >> 5] = c; red[8 + (tid >> 5)] = key; }
    __syncthreads();
    if (tid == 0) {
        u32 l = 0, m = 0;
        for (int w = 0; w < LIT_WARPS; w++) { l = max(l, red[w]); m = max(m, red[8 + w]); }
        *largestOut = l; *maxSymOut = m;
    }
    __syncthreads();
}

/* One Huffman stream, lit[beg, end) (lit 16-byte aligned, beg < end), by one warp: the symbols from the LAST to the first
 * (huf_compress.c:1056-1118), then the end mark (:973-982).  The stream's first bit is bit `bitPos` of `ow`.
 * Tiles of 32 lanes x 16 bytes, lane 0 on the highest vector, so that bit offsets grow with the lane; bytes of a vector
 * outside the stream are zero-length codes.  A warp scan over the lanes' bit counts places every lane's codes.  A lane ORs
 * them into the warp's window `win` (LIT_WIN words, zero on entry, word k of `ow` at win[k % LIT_WIN]): its first and its
 * last word may hold a neighbour's bits (shared atomicOr), the words between are its own (plain stores).  The warp then
 * stores the tile's completed words coalesced.  Only the stream's first and last word can share bytes with the headers or
 * a neighbouring stream: those two are ORed into global words the caller zeroed. */
__device__ __forceinline__ void zb_huf_stream(const u8* __restrict__ lit, u32 beg, u32 end, const u32* enc, u32* win, u32* ow,
                                              u32 bitPos, u32 lane)
{
    const uint4* const v4 = reinterpret_cast<const uint4*>(lit);
    uint4 const zero = make_uint4(0, 0, 0, 0);
    u32 const vHi = (end - 1u) >> 4, nVec = vHi - (beg >> 4) + 1u;
    u32 const firstW = bitPos >> 5;
    /* two more tiles' vectors in flight behind the one in use */
    uint4 q1 = lane < nVec ? __ldg(v4 + vHi - lane) : zero;
    uint4 q2 = lane + 32u < nVec ? __ldg(v4 + vHi - lane - 32u) : zero;
    for (u32 t = 0; t < nVec; t += 32u) {
        uint4 const q = q1;
        q1 = q2;
        q2 = t + 64u + lane < nVec ? __ldg(v4 + vHi - (t + 64u + lane)) : zero;
        u32 kLo = 0, kHi = 0;                                            /* bytes [kLo, kHi) of the vector are the stream's */
        if (t + lane < nVec) { u32 const p0 = (vHi - t - lane) << 4; kLo = beg > p0 ? beg - p0 : 0u; kHi = min(end - p0, 16u); }
        u32 const w[4] = { q.x, q.y, q.z, q.w };
        u32 nb = 0;
#pragma unroll
        for (u32 k = 0; k < 16u; k++) {
            u32 const e = enc[(w[k >> 2] >> (8u * (k & 3u))) & 0xFFu];
            nb += (k >= kLo && k < kHi) ? e >> 16 : 0u;
        }
        u32 incl = nb;
#pragma unroll
        for (u32 o = 1; o < 32u; o <<= 1) { u32 const x = __shfl_up_sync(ZB_FULL, incl, o); if (lane >= o) incl += x; }
        u32 const tileBits = __shfl_sync(ZB_FULL, incl, 31);
        {   /* the codes, last byte first; a full word is looked for once per two codes (fewer than 32 bits stay behind,
             * 32 + 2 * 12 < 64) and emitted without a branch: lanes fill their words at different moments */
            u32 const p = bitPos + incl - nb;
            u32 widx = p >> 5, nacc = p & 31u, first = 1;
            u64 acc = 0;
#pragma unroll
            for (int k = 15; k >= 0; k--) {
                u32 const e = ((u32)k >= kLo && (u32)k < kHi) ? enc[(w[k >> 2] >> (8u * (k & 3u))) & 0xFFu] : 0u;
                acc |= (u64)(e & 0xFFFFu) << nacc;
                nacc += e >> 16;
                if (k & 1) continue;
                bool const full = nacc >= 32u;
                u32* const wp = win + widx % LIT_WIN;
                if (full && first == 0u) *wp = (u32)acc;
                if (full && first != 0u) atomicOr(wp, (u32)acc);
                first = full ? 0u : first;
                widx += full ? 1u : 0u;
                acc = full ? (acc >> 32) : acc;
                nacc -= full ? 32u : 0u;
            }
            if (nacc != 0u && (u32)acc != 0u) atomicOr(win + widx % LIT_WIN, (u32)acc);
        }
        __syncwarp();
        u32 const wEnd = (bitPos + tileBits) >> 5;                       /* words below this one are complete */
        for (u32 k = (bitPos >> 5) + lane; k < wEnd; k += 32u) {
            u32 const v = win[k % LIT_WIN];
            win[k % LIT_WIN] = 0u;
            if (k == firstW) atomicOr(ow + k, v); else ow[k] = v;
        }
        __syncwarp();
        bitPos += tileBits;
    }
    if (lane == 0) atomicOr(ow + (bitPos >> 5), win[(bitPos >> 5) % LIT_WIN] | (1u << (bitPos & 31u)));  /* end mark: the last word */
}

__global__ void __launch_bounds__(LIT_THREADS, LIT_MIN_CTAS)
zb_literals_kernel(const ZbBlock* __restrict__ blocks, ZbParams prm, ZbStrides sd, const ZbDictEntropy* __restrict__ deAll,
                   const ZbDictSlot* __restrict__ dicts, const u8* __restrict__ lits, u8* __restrict__ body, ZbBlockMeta* __restrict__ meta)
{
    /* the per-warp (per-stream) histograms live until the stream sizes are known, then hold the encoding windows */
    __shared__ __align__(16) u32 whist[LIT_WARPS][256];
    __shared__ ZbdHufWksp wk;
    __shared__ u32 count[256];
    __shared__ u32 enc[256];
    __shared__ __align__(16) u8 hdr[288];                         /* the FSE form of the tree description is written before it is known to be short */
    __shared__ u32 red[16];
    __shared__ u32 sh_largest, sh_maxSym, sh_mode, sh_hSize, sh_usePrev;
    __shared__ u32 sh_bits[LIT_WARPS];

    u32 const tid = threadIdx.x, warp = tid >> 5, lane = tid & 31u;
    u32 const b = blockIdx.x;
    ZbBlockMeta const m = meta[b];
    if (m.forceRaw) return;
    u32 const n = m.litSize;
    const u8* const lit = lits + (size_t)b * sd.lit;
    u8* const out = body + (size_t)b * sd.body;
    enum { MODE_RAW = 0, MODE_RLE = 1, MODE_HUF = 2 };

    /* ---------------- decisions (zstd_compress_literals.c:129-191, huf_compress.c:1359-1420) ----------------
     * `repeat` is the HUF_repeat mode of the previous block's table: only a frame's first block behind a
     * zstd-format dictionary has one (ZSTD_loadCEntropy, zstd_compress.c:4997-5005); 0 none, 1 check, 2 valid. */
    ZbBlock const bd = blocks[b];
    const ZbDictEntropy* const de = (bd.flags & ZB_FLAG_FIRST) ? (dicts ? dicts[bd.dictSlot].de : deAll) : nullptr;
    u32 repeat = (de != nullptr && de->present) ? de->hufRepeat : 0u;
    bool const preferRepeat = (n <= 1024u);                      /* strategy < lazy, zstd_compress_literals.c:165 */
    u32 const lhSize = 3u + (n >= 1024u) + (n >= 16384u);
    u32 const nbStreams = (n < 256u || (repeat == 2u && lhSize == 3u)) ? 1u : 4u;     /* :142, :171 */
    u32 mode = MODE_HUF;
    bool usePrev = false;
    if (prm.litDisabled || n < (repeat == 2u ? 6u : 64u)) mode = MODE_RAW;   /* ZSTD_minLiteralsToCompress :114-127 */
    if (mode == MODE_HUF && preferRepeat && repeat == 2u) usePrev = true;     /* huf_compress.c:1359-1363 : no statistics at all */
    if (mode == MODE_HUF && !usePrev) {
        bool const suspect = (m.nbSeq == 0) || (n / m.nbSeq >= 20u);    /* zstd_compress.c:2915-2917 */
        if (suspect && n >= 4096u * 10u) {                               /* huf_compress.c:1367-1379 */
            u32 l1, l2;
            zb_hist256(lit, 4096u, whist, count);
            zb_hist_stats(count, red, &sh_largest, &sh_maxSym);
            l1 = sh_largest;
            __syncthreads();
            zb_hist256(lit + n - 4096u, 4096u, whist, count);
            zb_hist_stats(count, red, &sh_largest, &sh_maxSym);
            l2 = sh_largest;
            __syncthreads();
            if (l1 + l2 <= ((2u * 4096u) >> 7) + 4u) mode = MODE_RAW;
        }
    }
    /* the stream histograms are taken in the treeless case too: they give the stream sizes */
    if (mode == MODE_HUF) zb_hist256(lit, n, whist, count);
    if (mode == MODE_HUF && !usePrev) {
        zb_hist_stats(count, red, &sh_largest, &sh_maxSym);
        u32 const largest = sh_largest;
        if (largest == n) mode = MODE_RLE;
        else if (largest <= (n >> 7) + 4u) mode = MODE_RAW;
    }
    if (mode == MODE_HUF && !usePrev && repeat == 1u) {                     /* HUF_validateCTable, huf_compress.c:804, :1389-1393 */
        int bad = 0;
        for (u32 sym = tid; sym < 256u; sym += LIT_THREADS) bad |= (sym <= sh_maxSym) && count[sym] != 0u && (de->hufEnc[sym] >> 16) == 0u;
        if (__syncthreads_or(bad) || de->hufMaxSymbol < sh_maxSym) repeat = 0u;
    }
    if (mode == MODE_HUF && !usePrev && preferRepeat && repeat != 0u) usePrev = true;      /* :1395-1399 */
    if (mode == MODE_HUF && !usePrev) {
        u32 const maxSym = sh_maxSym;
        u32 const huffLog = zbd_fse_optimalTableLog(11, n, maxSym, 1);              /* huf_compress.c:1284-1287 */
        u32 const maxBits = zbc_huf_build<LIT_THREADS>(&wk, count, maxSym, huffLog, enc);
        u32 const hSizeNew = (maxBits == ZBD_ERR) ? ZBD_ERR : zbc_huf_writeHeader<LIT_THREADS>(&wk, hdr, enc, maxSym, maxBits, &sh_hSize);
        if (tid == 0) {
            u32 md = MODE_HUF, hSize = 0, prev = 0;
            if (hSizeNew == ZBD_ERR) md = MODE_RAW;
            else {
                hSize = hSizeNew;
                if (repeat != 0u) {                                        /* huf_compress.c:1415-1422 : is the old table cheaper? */
                    u32 oldBits = 0, newBits = 0;
                    for (u32 sy = 0; sy <= maxSym; sy++) { oldBits += (de->hufEnc[sy] >> 16) * count[sy]; newBits += (enc[sy] >> 16) * count[sy]; }
                    if ((oldBits >> 3) <= hSize + (newBits >> 3) || hSize + 12u >= n) prev = 1;
                }
                if (!prev && hSize + 12u >= n) md = MODE_RAW;              /* :1426 */
            }
            sh_mode = md; sh_hSize = hSize; sh_usePrev = prev;
        }
        __syncthreads();
        mode = sh_mode;
        usePrev = sh_usePrev != 0u;
    }
    if (mode == MODE_HUF && usePrev) {                                         /* treeless: encode with the dictionary's table */
        __syncthreads();
        for (u32 sym = tid; sym < 256u; sym += LIT_THREADS) enc[sym] = de->hufEnc[sym];
        if (tid == 0) sh_hSize = 0;
        __syncthreads();
    }

    /* ---------------- stream sizes: each warp's histogram against the code lengths ---------------- */
    u32 const hType = usePrev ? 3u : 2u;              /* set_repeat (treeless) : set_compressed */
    u32 const seg = (n + 3u) / 4u;                   /* huf_compress.c:1172 */
    u32 streamSize[4] = { 0u, 0u, 0u, 0u };
    u32 hSize = 0, total = 0;
    if (mode == MODE_HUF) {
        hSize = sh_hSize;
        u32 bits = 0;
        for (u32 sym = lane; sym < 256u; sym += 32u) bits += whist[warp][sym] * (enc[sym] >> 16);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) bits += __shfl_xor_sync(ZB_FULL, bits, o);
        if (lane == 0) sh_bits[warp] = bits;
        __syncthreads();
        if (nbStreams == 4u) for (u32 k = 0; k < 4u; k++) streamSize[k] = (sh_bits[k] + 1u + 7u) >> 3;   /* + end mark, huf_compress.c:973-982 */
        else streamSize[0] = (sh_bits[0] + sh_bits[1] + sh_bits[2] + sh_bits[3] + 1u + 7u) >> 3;
        u32 cSize = 0; bool tooBig = false;
#pragma unroll
        for (u32 k = 0; k < 4u; k++) { cSize += streamSize[k]; tooBig |= (streamSize[k] > 65535u); }
        if (nbStreams == 4u) cSize += 6u;
        total = hSize + cSize;
        if (nbStreams == 4u && tooBig) mode = MODE_RAW;                       /* huf_compress.c:1185 */
        else if (total >= n - 1u) mode = MODE_RAW;                            /* huf_compress.c:1232 */
        else if (total >= n - ((n >> 6) + 2u)) mode = MODE_RAW;               /* zstd_compress_literals.c:187-191 */
        else if (total == 1u) {                                               /* :193-205 : a 1-byte result is read as "single symbol" */
            int diff = 0;
            if (n < 8u) for (u32 i = tid; i < n; i += LIT_THREADS) diff |= (lit[i] != lit[0]);
            if (!__syncthreads_or(diff)) mode = MODE_RLE;
        }
    }

    /* ---------------- emit ---------------- */
    if (mode == MODE_RAW) {                                                   /* zstd_compress_literals.c:39-63 */
        u32 const flSize = 1u + (n > 31u) + (n > 4095u);
        if (tid == 0) {
            if (flSize == 1) out[0] = (u8)(0u + (n << 3));
            else if (flSize == 2) { u32 const v = 0u + (1u << 2) + (n << 4); out[0] = (u8)v; out[1] = (u8)(v >> 8); }
            else { u32 const v = 0u + (3u << 2) + (n << 4); out[0] = (u8)v; out[1] = (u8)(v >> 8); out[2] = (u8)(v >> 16); }
            meta[b].litSecSize = flSize + n;
        }
        for (u32 i = tid; i < n; i += LIT_THREADS) out[flSize + i] = lit[i];
        return;
    }
    if (mode == MODE_RLE) {                                                   /* zstd_compress_literals.c:81-108 */
        if (tid == 0) {
            u32 const flSize = 1u + (n > 31u) + (n > 4095u);
            if (flSize == 1) out[0] = (u8)(1u + (n << 3));
            else if (flSize == 2) { u32 const v = 1u + (1u << 2) + (n << 4); out[0] = (u8)v; out[1] = (u8)(v >> 8); }
            else { u32 const v = 1u + (3u << 2) + (n << 4); out[0] = (u8)v; out[1] = (u8)(v >> 8); out[2] = (u8)(v >> 16); }
            out[flSize] = lit[0];
            meta[b].litSecSize = flSize + 1u;
        }
        return;
    }

    /* compressed.  Stream k occupies bytes [sOff, sOff + streamSize[k]); its first and last word are zeroed here, the
     * headers are written behind a barrier (their bytes may share the first stream's first word), then the streams. */
    u32 sOff = lhSize + hSize + (nbStreams == 4u ? 6u : 0u), sSize = 0;
#pragma unroll
    for (u32 k = 0; k < 4u; k++) { sOff += k < warp ? streamSize[k] : 0u; sSize = k == warp ? streamSize[k] : sSize; }
    u32* const ow = reinterpret_cast<u32*>(out);
    for (u32 i = tid; i < LIT_WARPS * 256u; i += LIT_THREADS) (&whist[0][0])[i] = 0u;         /* the windows */
    if (warp < nbStreams && lane == 0) { ow[sOff >> 2] = 0u; ow[(sOff + sSize - 1u) >> 2] = 0u; }
    __syncthreads();
    if (tid == 0) {                                                           /* zstd_compress_literals.c:209-232 */
        u32 const cLitSize = total;
        if (lhSize == 3) { u32 const lhc = hType + ((nbStreams == 4u ? 1u : 0u) << 2) + (n << 4) + (cLitSize << 14);
                           out[0] = (u8)lhc; out[1] = (u8)(lhc >> 8); out[2] = (u8)(lhc >> 16); }
        else if (lhSize == 4) { u32 const lhc = hType + (2u << 2) + (n << 4) + (cLitSize << 18);
                           out[0] = (u8)lhc; out[1] = (u8)(lhc >> 8); out[2] = (u8)(lhc >> 16); out[3] = (u8)(lhc >> 24); }
        else { u32 const lhc = hType + (3u << 2) + (n << 4) + (cLitSize << 22);
                           out[0] = (u8)lhc; out[1] = (u8)(lhc >> 8); out[2] = (u8)(lhc >> 16); out[3] = (u8)(lhc >> 24);
                           out[4] = (u8)(cLitSize >> 10); }
        if (nbStreams == 4u) {
            u8* jt = out + lhSize + hSize;
            for (int k = 0; k < 3; k++) { jt[2 * k] = (u8)streamSize[k]; jt[2 * k + 1] = (u8)(streamSize[k] >> 8); }
        }
        meta[b].litSecSize = lhSize + total;
    }
    for (u32 i = tid; i < hSize; i += LIT_THREADS) out[lhSize + i] = hdr[i];
    __syncthreads();          /* byte stores above share words with the streams' first bits: order them before the ORs */
    if (warp < nbStreams) {
        u32 const beg = nbStreams == 1u ? 0u : min(warp * seg, n), end = nbStreams == 1u ? n : min((warp + 1u) * seg, n);
        zb_huf_stream(lit, beg, end, enc, whist[warp], ow, sOff * 8u, lane);
    }
}

extern "C" cudaError_t zb_launch_literals(const ZbBlock* d_blocks, u32 nbBlocks, const ZbParams* prm, const ZbStrides* sd, const ZbDictEntropy* d_de,
                                          const u8* d_lits, u8* d_body, ZbBlockMeta* d_meta, cudaStream_t stream, const ZbDictSlot* d_dicts)
{
    if (nbBlocks == 0) return cudaSuccess;
    zb_literals_kernel<<<nbBlocks, LIT_THREADS, 0, stream>>>(d_blocks, *prm, *sd, d_de, d_dicts, d_lits, d_body, d_meta);
    return cudaGetLastError();
}
