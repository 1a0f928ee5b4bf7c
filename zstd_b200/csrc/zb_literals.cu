/* zb_literals.cu — K2: literals section of one block per CTA.
 *
 * Replaces ZSTD_compressLiterals (lib/compress/zstd_compress_literals.c:129-235)
 * and HUF_compress_internal (huf_compress.c:1333-1430) for a fresh entropy state:
 *   1. 256-bin histogram: per-warp privatised bins in shared memory + merge (hist.c:66-133)
 *   2. raw / RLE / compressed decision with the reference's thresholds
 *   3. Huffman table + tree description: the whole CTA (zb_entropy.cuh)
 *   4. 1 or 4 streams (huf_compress.c:1056-1118, :1168-1215): every thread owns a contiguous run of
 *      symbols, a suffix sum over per-thread bit counts gives its bit offset (streams grow from the
 *      LAST symbol), then bits are packed straight into the output words (edge words by atomicOr).
 * Output: body[0 .. litSecSize) of the block's staging area; meta.litSecSize.
 */
#include "zb_entropy.cuh"
#include "zb_kernels.h"
#include "zb_bitpack.cuh"

#ifndef LIT_THREADS
#define LIT_THREADS 128
#endif
#ifndef LIT_MIN_CTAS
#define LIT_MIN_CTAS 12               /* 16 (32 registers) measured slower on the H100: literals 2.90 vs 2.68 ms per GiB of config 2 */
#endif
#define LIT_WARPS (LIT_THREADS / 32)
#ifndef LIT_PACK2
#define LIT_PACK2 1                   /* the stream packer looks for a full word once per two codes, without a branch */
#endif
#ifndef LIT_AHEAD
#define LIT_AHEAD 2                   /* 16-byte vectors of a thread's run requested ahead of the one in use */
#endif

/* block-wide histogram of src[0..n) into count[256]; returns nothing, count valid after the call */
__device__ void zb_hist256(const u8* __restrict__ src, u32 n, u32 (*whist)[256], u32* count)   /* whist: LIT_WARPS private histograms */
{
    u32 const tid = threadIdx.x, warp = tid >> 5;
    for (u32 i = tid; i < LIT_WARPS * 256; i += LIT_THREADS) (&whist[0][0])[i] = 0;
    __syncthreads();
    u32 const head = (u32)((16u - ((uintptr_t)src & 15u)) & 15u);       /* bytes before 16-byte alignment */
    u32 const headN = head < n ? head : n;
    if (tid < headN) atomicAdd(&whist[warp][src[tid]], 1u);
    u32 const nvec = (n - headN) / 16u;
    const uint4* v4 = reinterpret_cast<const uint4*>(src + headN);
    for (u32 i = tid; i < nvec; i += LIT_THREADS) {
        uint4 const q = __ldg(v4 + i);
        u32 w[4] = { q.x, q.y, q.z, q.w };
#pragma unroll
        for (int k = 0; k < 4; k++) {
            atomicAdd(&whist[warp][w[k] & 0xFF], 1u);
            atomicAdd(&whist[warp][(w[k] >> 8) & 0xFF], 1u);
            atomicAdd(&whist[warp][(w[k] >> 16) & 0xFF], 1u);
            atomicAdd(&whist[warp][w[k] >> 24], 1u);
        }
    }
    for (u32 i = headN + nvec * 16u + tid; i < n; i += LIT_THREADS) atomicAdd(&whist[warp][src[i]], 1u);
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


/* Visit the symbols of lit[beg, end) from the LAST to the first (the order the Huffman stream is
 * written in, huf_compress.c:1056-1118) with 16-byte aligned vector loads: a thread's run is
 * contiguous, so byte loads would cost one request per symbol. */
struct ZbNoop { __device__ __forceinline__ void operator()() const {} };
template <typename F, typename G = ZbNoop>
__device__ __forceinline__ void zb_for_each_symbol_rev(const u8* __restrict__ lit, u32 beg, u32 end, F f, G every2 = G())
{
    /* every2() runs after at most two symbols (the packer's flush point) */
    u32 const aBeg = (beg + 15u) & ~15u, aEnd = end & ~15u;
    if (aBeg >= aEnd) { for (u32 i = end; i-- > beg; ) { f(lit[i]); every2(); } return; }
    for (u32 i = end; i-- > aEnd; ) { f(lit[i]); every2(); }
    const uint4* v4 = reinterpret_cast<const uint4*>(lit);
    /* a thread's run is walked one 16-byte vector at a time, each needing the one before it consumed: the next LIT_AHEAD
     * vectors are requested before the current one is used */
    u32 k = aEnd / 16u;
    u32 const kLo = aBeg / 16u;
    uint4 nx[LIT_AHEAD];
#pragma unroll
    for (u32 a = 0; a < LIT_AHEAD; a++) nx[a] = (k >= kLo + a + 1u) ? __ldg(v4 + (k - a - 1u)) : make_uint4(0, 0, 0, 0);
    while (k > kLo) {
        k--;
        uint4 const q = nx[0];
#pragma unroll
        for (u32 a = 0; a + 1u < LIT_AHEAD; a++) nx[a] = nx[a + 1u];
        if (k >= kLo + LIT_AHEAD) nx[LIT_AHEAD - 1u] = __ldg(v4 + (k - LIT_AHEAD));
        u32 const w[4] = { q.x, q.y, q.z, q.w };
#pragma unroll
        for (int t = 3; t >= 0; t--) { f((u8)(w[t] >> 24)); f((u8)(w[t] >> 16)); every2(); f((u8)(w[t] >> 8)); f((u8)w[t]); every2(); }
    }
    for (u32 i = aBeg; i-- > beg; ) { f(lit[i]); every2(); }
}

__global__ void __launch_bounds__(LIT_THREADS, LIT_MIN_CTAS)
zb_literals_kernel(const ZbBlock* __restrict__ blocks, ZbParams prm, ZbStrides sd, const ZbDictEntropy* __restrict__ de,
                   const u8* __restrict__ lits, u8* __restrict__ body, ZbBlockMeta* __restrict__ meta)
{
    /* the per-warp histograms are dead once count[] is merged, the Huffman workspace only lives after that: one area */
    __shared__ __align__(16) u8 scratch[sizeof(ZbdHufWksp) > sizeof(u32) * LIT_WARPS * 256 ? sizeof(ZbdHufWksp) : sizeof(u32) * LIT_WARPS * 256];
    u32 (* const whist)[256] = reinterpret_cast<u32 (*)[256]>(scratch);
    ZbdHufWksp& wk = *reinterpret_cast<ZbdHufWksp*>(scratch);
    __shared__ u32 count[256];
    __shared__ u32 enc[256];
    __shared__ __align__(16) u8 hdr[288];                         /* the FSE form of the tree description is written before it is known to be short */
    __shared__ u32 red[16];
    __shared__ u32 chunkBits[LIT_THREADS];
    __shared__ u32 sh_largest, sh_maxSym, sh_mode, sh_hSize, sh_usePrev;
    __shared__ u32 sh_streamSize[4];

    u32 const tid = threadIdx.x;
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
    u32 repeat = (de != nullptr && (blocks[b].flags & ZB_FLAG_FIRST) && de->present) ? de->hufRepeat : 0u;
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
    if (mode == MODE_HUF && !usePrev) {
        zb_hist256(lit, n, whist, count);
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

    /* ---------------- stream geometry + bit counts ---------------- */
    u32 const hType = usePrev ? 3u : 2u;              /* set_repeat (treeless) : set_compressed */
    u32 const T = LIT_THREADS / nbStreams;           /* threads per stream */
    u32 const s = tid / T, j = tid % T;
    u32 const seg = (n + 3u) / 4u;                   /* huf_compress.c:1172 */
    u32 const sBeg = (nbStreams == 1u) ? 0u : s * seg;
    u32 const sEnd = (nbStreams == 1u) ? n : ((s == 3u) ? n : (s + 1u) * seg);
    u32 const sLen = sEnd - sBeg;
    u32 const cs = (sLen + T - 1u) / T;
    u32 const cBeg = sBeg + min(j * cs, sLen);
    u32 const cEnd = sBeg + min((j + 1u) * cs, sLen);
    u32 hSize = 0, total = 0, bitOff = 0;
    if (mode == MODE_HUF) {
        hSize = sh_hSize;
        u32 bits = 0;
        zb_for_each_symbol_rev(lit, cBeg, cEnd, [&](u8 sym) { bits += enc[sym] >> 16; });
        chunkBits[tid] = bits;
        __syncthreads();
        /* suffix sum inside the stream: symbols AFTER mine are written before mine */
        for (u32 k = j + 1u; k < T; k++) bitOff += chunkBits[s * T + k];
        if (j == 0) sh_streamSize[s] = (bitOff + bits + 1u + 7u) >> 3;     /* + end mark, huf_compress.c:973-982 */
        __syncthreads();
        u32 cSize = 0; bool tooBig = false;
        for (u32 k = 0; k < nbStreams; k++) { cSize += sh_streamSize[k]; tooBig |= (sh_streamSize[k] > 65535u); }
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

    /* compressed: zero the words we are going to OR into, then headers, then the packed streams */
    {   u32 const endByte = lhSize + total;
        uint4* o4 = reinterpret_cast<uint4*>(out);
        for (u32 i = tid; i < (endByte + 15u) / 16u; i += LIT_THREADS) o4[i] = make_uint4(0, 0, 0, 0);
    }
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
            for (int k = 0; k < 3; k++) { jt[2 * k] = (u8)sh_streamSize[k]; jt[2 * k + 1] = (u8)(sh_streamSize[k] >> 8); }
        }
        meta[b].litSecSize = lhSize + total;
    }
    for (u32 i = tid; i < hSize; i += LIT_THREADS) out[lhSize + i] = hdr[i];
    __syncthreads();          /* byte stores above share words with the streams' first bits: order them before the ORs */
    {
        u32 sOff = lhSize + hSize + (nbStreams == 4u ? 6u : 0u);
        for (u32 k = 0; k < s; k++) sOff += sh_streamSize[k];
        ZbdParW pw; zbd_pw_init(&pw, reinterpret_cast<u32*>(out), (u64)sOff * 8u + bitOff);
#if LIT_PACK2
        zb_for_each_symbol_rev(lit, cBeg, cEnd, [&](u8 sym) { u32 const e = enc[sym]; zbd_pw_put(&pw, e & 0xFFFFu, e >> 16); }, [&]() { zbd_pw_flush(&pw); });
#else
        zb_for_each_symbol_rev(lit, cBeg, cEnd, [&](u8 sym) { u32 const e = enc[sym]; zbd_pw_add(&pw, e & 0xFFFFu, e >> 16); });
#endif
        if (j == 0) zbd_pw_add(&pw, 1u, 1u);
        zbd_pw_finish(&pw);
    }
}

extern "C" cudaError_t zb_launch_literals(const ZbBlock* d_blocks, u32 nbBlocks, const ZbParams* prm, const ZbStrides* sd, const ZbDictEntropy* d_de,
                                          const u8* d_lits, u8* d_body, ZbBlockMeta* d_meta, cudaStream_t stream)
{
    if (nbBlocks == 0) return cudaSuccess;
    zb_literals_kernel<<<nbBlocks, LIT_THREADS, 0, stream>>>(d_blocks, *prm, *sd, d_de, d_lits, d_body, d_meta);
    return cudaGetLastError();
}
