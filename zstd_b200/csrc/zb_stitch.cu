/* zb_stitch.cu — K4: assemble frames from independently compressed blocks.
 *
 * The reference's block loop (ZSTD_compress_frameChunk, lib/compress/zstd_compress.c:4527-4623)
 * appends blocks one after the other; here all blocks of a call were compressed at once, so the
 * frame is assembled by (a) computing every block's output size (frame header for the first block
 * of a frame, :4626-4672; 3-byte block header, :4586-4590; payload), (b) an exclusive prefix sum,
 * (c) one CTA per block copying header + payload to its final place.
 */
#include "zb_device.cuh"
#include "zb_kernels.h"

/* zstd_compress.c:4626-4672, contentSizeFlag = 1.  Returns header size (<= 18). */
__device__ u32 zbd_frameHeader(u8* dst, u32 windowLog, u64 srcSize, u32 dictID, u32 checksum, bool write)
{
    u32 const dictIDSizeCode = (dictID > 0) + (dictID >= 256) + (dictID >= 65536);
    bool const singleSegment = ((u64)1 << windowLog) >= srcSize;
    u32 const fcsCode = (srcSize >= 256) + (srcSize >= 65536 + 256) + (srcSize >= 0xFFFFFFFFull);
    u8 h[18]; u32 pos = 0;
    h[pos++] = 0x28; h[pos++] = 0xB5; h[pos++] = 0x2F; h[pos++] = 0xFD;          /* ZSTD_MAGICNUMBER 0xFD2FB528 */
    h[pos++] = (u8)(dictIDSizeCode + ((checksum ? 1u : 0u) << 2) + ((singleSegment ? 1u : 0u) << 5) + (fcsCode << 6));
    if (!singleSegment) h[pos++] = (u8)((windowLog - 10u) << 3);
    if (dictIDSizeCode == 1) h[pos++] = (u8)dictID;
    else if (dictIDSizeCode == 2) { h[pos++] = (u8)dictID; h[pos++] = (u8)(dictID >> 8); }
    else if (dictIDSizeCode == 3) { for (int i = 0; i < 4; i++) h[pos++] = (u8)(dictID >> (8 * i)); }
    if (fcsCode == 0) { if (singleSegment) h[pos++] = (u8)srcSize; }
    else if (fcsCode == 1) { u32 const v = (u32)(srcSize - 256); h[pos++] = (u8)v; h[pos++] = (u8)(v >> 8); }
    else if (fcsCode == 2) { for (int i = 0; i < 4; i++) h[pos++] = (u8)(srcSize >> (8 * i)); }
    else { for (int i = 0; i < 8; i++) h[pos++] = (u8)(srcSize >> (8 * i)); }
    if (write) for (u32 i = 0; i < pos; i++) dst[i] = h[i];
    return pos;
}

#define SCAN_THREADS 1024

/* single-CTA exclusive scan over per-block output sizes (a wave is a few thousand 128 KiB blocks, or a few
 * hundred thousand blocks of a call made of short frames).  Pass 0 computes every block's size with coalesced,
 * thread-strided reads and parks it in outOffsets[i]; passes 1 and 2 then walk contiguous chunks of plain u64. */
__global__ void __launch_bounds__(SCAN_THREADS)
zb_sizes_scan_kernel(const ZbBlock* __restrict__ blocks, u32 nbBlocks, const ZbFrame* __restrict__ frames,
                     const ZbBlockMeta* __restrict__ meta, u64* __restrict__ outOffsets,
                     const u64* __restrict__ basePtr, u64* __restrict__ total)
{
    u64 const base = basePtr ? *basePtr : 0;      /* bytes produced by the waves before this one */
    __shared__ u64 part[SCAN_THREADS];
    u32 const tid = threadIdx.x;
    for (u32 i = tid; i < nbBlocks; i += SCAN_THREADS) {
        ZbBlock const bd = blocks[i];
        u64 sz = 3u + meta[i].bodySize;
        if (bd.flags & (ZB_FLAG_FIRST | ZB_FLAG_LAST)) {
            ZbFrame const f = frames[bd.frame];
            if (bd.flags & ZB_FLAG_FIRST) sz += zbd_frameHeader(nullptr, f.windowLog, f.srcSize, f.dictID, f.checksum, false);
            if ((bd.flags & ZB_FLAG_LAST) && f.checksum) sz += 4u;          /* room for the XXH64 low word, zstd_compress.c:5297-5303 */
        }
        outOffsets[i] = sz;
    }
    __syncthreads();
    u32 const per = (nbBlocks + SCAN_THREADS - 1u) / SCAN_THREADS;
    u32 const beg = min(tid * per, nbBlocks), end = min((tid + 1u) * per, nbBlocks);
    u64 sum = 0;
    for (u32 i = beg; i < end; i++) sum += outOffsets[i];
    part[tid] = sum;
    __syncthreads();
    /* Hillis-Steele inclusive scan over the 1024 partial sums */
    for (u32 off = 1; off < SCAN_THREADS; off <<= 1) {
        u64 const v = (tid >= off) ? part[tid - off] : 0;
        __syncthreads();
        part[tid] += v;
        __syncthreads();
    }
    u64 run = base + ((tid == 0) ? 0 : part[tid - 1]);
    for (u32 i = beg; i < end; i++) { u64 const sz = outOffsets[i]; outOffsets[i] = run; run += sz; }
    if (tid == SCAN_THREADS - 1) { outOffsets[nbBlocks] = base + part[SCAN_THREADS - 1]; *total = base + part[SCAN_THREADS - 1]; }
}

/* the verdict of a call, left in device memory (the caller's for a stream-ordered call, else the context's, which the host
 * reads back): each frame's size (cSizes may be NULL) and the call's total, or dstSize_tooSmall when the frames did not fit
 * in dstCapacity (K4 wrote nothing past it).  total NULL: a call without frames, whose total is 0. */
__global__ void zb_call_result_kernel(const ZbFrame* __restrict__ frames, u32 nbFrames, const u64* __restrict__ outOffsets,
                                      const u64* __restrict__ total, u64 dstCapacity, unsigned long long* cSizes, unsigned long long* result)
{
    u32 const f = blockIdx.x * blockDim.x + threadIdx.x;
    if (cSizes && f < nbFrames) {
        ZbFrame const fr = frames[f];
        cSizes[f] = outOffsets[fr.firstBlock + fr.nbBlocks] - outOffsets[fr.firstBlock];
    }
    if (f == 0) {
        u64 const t = total ? *total : 0u;
        *result = t > dstCapacity ? (unsigned long long)ZB_ERR(ZB_error_dstSize_tooSmall) : t;
    }
}

#define COPY_THREADS 256
__global__ void __launch_bounds__(COPY_THREADS)
zb_copy_kernel(const u8* __restrict__ src, const ZbBlock* __restrict__ blocks, const ZbFrame* __restrict__ frames,
               const u8* __restrict__ body, u32 bodyStride, const ZbBlockMeta* __restrict__ meta,
               const u64* __restrict__ outOffsets, u8* __restrict__ dst, u64 dstCapacity)
{
    u32 const b = blockIdx.x, tid = threadIdx.x;
    ZbBlock const bd = blocks[b];
    ZbBlockMeta const m = meta[b];
    u64 const o0 = outOffsets[b], o1 = outOffsets[b + 1];
    if (o1 > dstCapacity) return;                                   /* never write past dst + dstCapacity */
    u8* out = dst + o0;
    u32 hdr = 0;
    if (bd.flags & ZB_FLAG_FIRST) {
        ZbFrame const f = frames[bd.frame];
        hdr = zbd_frameHeader(out, f.windowLog, f.srcSize, f.dictID, f.checksum, tid == 0);
    }
    out += hdr;
    u32 const lastBlock = (bd.flags & ZB_FLAG_LAST) ? 1u : 0u;
    if (tid == 0) {                                                 /* zstd_compress.c:4586-4590, zstd_compress_internal.h:586-610 */
        u32 const h24 = (m.type == ZB_BT_COMPRESSED) ? lastBlock + (2u << 1) + (m.bodySize << 3)
                      : (m.type == ZB_BT_RLE)        ? lastBlock + (1u << 1) + (bd.size << 3)
                                                     : lastBlock + (0u << 1) + (bd.size << 3);
        out[0] = (u8)h24; out[1] = (u8)(h24 >> 8); out[2] = (u8)(h24 >> 16);
        if (m.type == ZB_BT_RLE) out[3] = (u8)m.rleByte;
    }
    out += 3;
    if (m.type == ZB_BT_RLE) return;
    const u8* const from = (m.type == ZB_BT_COMPRESSED) ? body + (size_t)b * bodyStride : src + bd.srcOff;
    u32 const n = m.bodySize;
    /* 16-byte vector body where source and destination can both be aligned: source is read through
     * unaligned 32-bit words, destination peeled to 16-byte alignment */
    u32 const head = (u32)((16u - ((uintptr_t)out & 15u)) & 15u);
    u32 const headN = head < n ? head : n;
    if (tid < headN) out[tid] = from[tid];
    u32 const nvec = (n - headN) / 16u;
    uint4* const o4 = reinterpret_cast<uint4*>(out + headN);
    const u8* const f0 = from + headN;
    if ((((uintptr_t)f0) & 15u) == 0) {
        const uint4* const f4 = reinterpret_cast<const uint4*>(f0);
        for (u32 i = tid; i < nvec; i += COPY_THREADS) o4[i] = f4[i];
    } else {
        for (u32 i = tid; i < nvec; i += COPY_THREADS) {
            const u8* p = f0 + (size_t)i * 16u;
            uint4 v; v.x = zb_ld32u(p); v.y = zb_ld32u(p + 4); v.z = zb_ld32u(p + 8); v.w = zb_ld32u(p + 12);
            o4[i] = v;
        }
    }
    for (u32 i = headN + nvec * 16u + tid; i < n; i += COPY_THREADS) out[i] = from[i];
}

/* Small blocks (calls made of many short frames, BASELINE config 5): a 256-thread CTA per block would move a
 * few hundred bytes each, so one warp takes a block — 8 blocks per CTA, bytes copied lane-strided. */
__global__ void __launch_bounds__(COPY_THREADS)
zb_copy_small_kernel(const u8* __restrict__ src, const ZbBlock* __restrict__ blocks, u32 nbBlocks, const ZbFrame* __restrict__ frames,
                     const u8* __restrict__ body, u32 bodyStride, const ZbBlockMeta* __restrict__ meta,
                     const u64* __restrict__ outOffsets, u8* __restrict__ dst, u64 dstCapacity)
{
    u32 const lane = threadIdx.x & 31u;
    u32 const b = blockIdx.x * (COPY_THREADS / 32u) + (threadIdx.x >> 5);
    if (b >= nbBlocks) return;
    ZbBlock const bd = blocks[b];
    ZbBlockMeta const m = meta[b];
    u64 const o0 = outOffsets[b], o1 = outOffsets[b + 1];
    if (o1 > dstCapacity) return;                                   /* never write past dst + dstCapacity */
    u8* out = dst + o0;
    u32 hdr = 0;
    if (bd.flags & ZB_FLAG_FIRST) {
        ZbFrame const f = frames[bd.frame];
        hdr = zbd_frameHeader(out, f.windowLog, f.srcSize, f.dictID, f.checksum, lane == 0);
    }
    out += hdr;
    u32 const lastBlock = (bd.flags & ZB_FLAG_LAST) ? 1u : 0u;
    if (lane == 0) {                                                /* zstd_compress.c:4586-4590 */
        u32 const h24 = (m.type == ZB_BT_COMPRESSED) ? lastBlock + (2u << 1) + (m.bodySize << 3)
                      : (m.type == ZB_BT_RLE)        ? lastBlock + (1u << 1) + (bd.size << 3)
                                                     : lastBlock + (0u << 1) + (bd.size << 3);
        out[0] = (u8)h24; out[1] = (u8)(h24 >> 8); out[2] = (u8)(h24 >> 16);
        if (m.type == ZB_BT_RLE) out[3] = (u8)m.rleByte;
    }
    out += 3;
    if (m.type == ZB_BT_RLE) return;
    const u8* const from = (m.type == ZB_BT_COMPRESSED) ? body + (size_t)b * bodyStride : src + bd.srcOff;
    for (u32 i = lane; i < m.bodySize; i += 32u) out[i] = from[i];
}

extern "C" cudaError_t zb_launch_stitch(const u8* d_src, const ZbBlock* d_blocks, u32 nbBlocks, const ZbFrame* d_frames, const ZbWorkRows* rows,
                                        u64* d_outOffsets, const u64* d_base, u64* d_total,
                                        u8* d_dst, u64 dstCapacity, cudaStream_t stream)
{
    if (nbBlocks == 0) return cudaSuccess;
    const u8* const d_body = rows->body; u32 const bodyStride = rows->sd.body; const ZbBlockMeta* const d_meta = rows->meta;
    zb_sizes_scan_kernel<<<1, SCAN_THREADS, 0, stream>>>(d_blocks, nbBlocks, d_frames, d_meta, d_outOffsets, d_base, d_total);
    if (bodyStride <= 8192u + 1024u)
        zb_copy_small_kernel<<<(nbBlocks + COPY_THREADS / 32u - 1u) / (COPY_THREADS / 32u), COPY_THREADS, 0, stream>>>(d_src, d_blocks, nbBlocks, d_frames, d_body, bodyStride, d_meta, d_outOffsets, d_dst, dstCapacity);
    else
        zb_copy_kernel<<<nbBlocks, COPY_THREADS, 0, stream>>>(d_src, d_blocks, d_frames, d_body, bodyStride, d_meta, d_outOffsets, d_dst, dstCapacity);
    return cudaGetLastError();
}

/* ------------------------------------------------------------------------------------------------
 * Content checksum (format: "Content_Checksum" = low 32 bits of XXH64, seed 0, of the frame's content;
 * the reference computes it chunk by chunk on the host, zstd_compress.c:4544, :5297-5303).
 * XXH64 is four serial accumulator chains per input (acc = rotl(acc + x * P2, 31) * P1 over the 8-byte words of
 * every 32-byte stripe): nothing to split inside one frame, so one warp takes a frame — all lanes load 256 bytes,
 * lanes 0..3 run the chains — and the frames of a call are hashed side by side.  The rounds are in zb_device.cuh. */

#define XXH_WARPS 4
__global__ void __launch_bounds__(32 * XXH_WARPS)
zb_checksum_kernel(const u8* __restrict__ src, const ZbFrame* __restrict__ frames, u32 nbFrames, const u64* __restrict__ outOffsets,
                   u8* __restrict__ dst, u64 dstCapacity)
{
    u32 const lane = threadIdx.x & 31u;
    u32 const f = blockIdx.x * XXH_WARPS + (threadIdx.x >> 5);
    if (f >= nbFrames) return;
    ZbFrame const fr = frames[f];
    if (!fr.checksum) return;
    const u8* const p = src + fr.srcOff;
    u64 const len = fr.srcSize;
    u64 const stripes = len >> 5;
    u64 acc = lane == 0u ? ZBX_P1 + ZBX_P2 : (lane == 1u ? ZBX_P2 : (lane == 2u ? 0ull : 0ull - ZBX_P1));
    u64 nextW = (lane < 4u * stripes) ? zb_ld64u(p + 8u * lane) : 0ull;
    for (u64 s0 = 0; s0 < stripes; s0 += 8u) {
        u64 const w = nextW;
        u64 const nx = (s0 + 8u) * 4u + lane;                        /* this lane's word of the next 256 bytes */
        nextW = (nx < 4u * stripes) ? zb_ld64u(p + 8u * nx) : 0ull;
        u32 const n = (u32)(stripes - s0 < 8u ? stripes - s0 : 8u);
        for (u32 s = 0; s < n; s++) {
            u64 const x = __shfl_sync(ZB_FULL, w, (int)(4u * s + (lane & 3u)));
            if (lane < 4u) acc = zbx_round(acc, x);
        }
    }
    u64 const v1 = __shfl_sync(ZB_FULL, acc, 0), v2 = __shfl_sync(ZB_FULL, acc, 1), v3 = __shfl_sync(ZB_FULL, acc, 2), v4 = __shfl_sync(ZB_FULL, acc, 3);
    if (lane != 0u) return;
    u64 h;
    if (len >= 32u) {
        h = zbx_rotl(v1, 1) + zbx_rotl(v2, 7) + zbx_rotl(v3, 12) + zbx_rotl(v4, 18);
        h = zbx_merge(h, v1); h = zbx_merge(h, v2); h = zbx_merge(h, v3); h = zbx_merge(h, v4);
    } else h = ZBX_P5;
    h += len;
    u64 i = stripes << 5;
    for (; i + 8u <= len; i += 8u) { h ^= zbx_round(0, zb_ld64u(p + i)); h = zbx_rotl(h, 27) * ZBX_P1 + ZBX_P4; }
    if (i + 4u <= len) { h ^= (u64)zb_ld32u(p + i) * ZBX_P1; h = zbx_rotl(h, 23) * ZBX_P2 + ZBX_P3; i += 4u; }
    for (; i < len; i++) { h ^= (u64)p[i] * ZBX_P5; h = zbx_rotl(h, 11) * ZBX_P1; }
    h ^= h >> 33; h *= ZBX_P2; h ^= h >> 29; h *= ZBX_P3; h ^= h >> 32;
    u64 const end = outOffsets[fr.firstBlock + fr.nbBlocks];          /* the frame's last 4 bytes were left free by the size scan */
    if (end > dstCapacity || end < 4u) return;
    u32 const ck = (u32)h;
    dst[end - 4u] = (u8)ck; dst[end - 3u] = (u8)(ck >> 8); dst[end - 2u] = (u8)(ck >> 16); dst[end - 1u] = (u8)(ck >> 24);
}

extern "C" cudaError_t zb_launch_checksums(const u8* d_src, const ZbFrame* d_frames, u32 nbFrames, const u64* d_outOffsets, u8* d_dst, u64 dstCapacity, cudaStream_t stream)
{
    if (nbFrames == 0) return cudaSuccess;
    zb_checksum_kernel<<<(nbFrames + XXH_WARPS - 1u) / XXH_WARPS, 32 * XXH_WARPS, 0, stream>>>(d_src, d_frames, nbFrames, d_outOffsets, d_dst, dstCapacity);
    return cudaGetLastError();
}

extern "C" cudaError_t zb_launch_call_result(const ZbFrame* d_frames, u32 nbFrames, const u64* d_outOffsets, const u64* d_total,
                                             u64 dstCapacity, unsigned long long* d_cSizes, unsigned long long* d_result, cudaStream_t stream)
{
    zb_call_result_kernel<<<nbFrames ? (nbFrames + 255) / 256 : 1, 256, 0, stream>>>(d_frames, nbFrames, d_outOffsets, d_total, dstCapacity,
                                                                                    d_cSizes, d_result);
    return cudaGetLastError();
}
