/* zb_decode.cu — GPU decompression of zstd frames (SURVEY.md 8f rank 2): the other half of the block pipeline.
 *
 * Replaces, with a block-parallel formulation, what the reference does serially per frame:
 *   ZSTD_decompress / ZSTD_decompressDCtx / ZSTD_decompressFrame  (lib/decompress/zstd_decompress.c:1011-1124)
 *   ZSTD_decodeLiteralsBlock, ZSTD_decodeSeqHeaders, ZSTD_decompressSequences_body, ZSTD_execSequence
 *                                                     (lib/decompress/zstd_decompress_block.c:343, :695, :1615, :1012)
 *   HUF_decompress4X1 / HUF_readDTableX1              (lib/decompress/huf_decompress.c:602, :383)
 * Any frame the format allows is accepted (this library's own and the reference encoder's, every level), window
 * sizes up to 128 MiB, raw-content and zstd-format dictionaries (ZSTD_decompress_usingDict, zstd_decompress.c:1133).
 * Inputs the format does not allow are refused with a ZSTD error code, as the reference's ZSTD_decompress refuses them
 * (tests/test_decode_invalid.py), except where this decoder is deliberately stricter; the reference's one-shot call
 * accepts these:
 *   - offsets are kept in 28 bits: a frame whose offsets need more than 27 bits gets frameParameter_windowTooLarge (16)
 *     whatever its header says (a window descriptor above 2^27 from the walk; a Single_Segment frame, which states no
 *     window, from the first such offset code);
 *   - every block is bounded by Block_Maximum_Size = min(window, 128 KiB): a raw or RLE block larger than that, and a
 *     compressed block that regenerates more, are corruption_detected (20), as in the reference's streaming decoder;
 *   - a Huffman stream of the literals must end exactly at its first byte (corruption_detected).
 * Device calls do not verify content checksums; host calls and ZSTD_decompressStream do.
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
#include <memory>
#include <mutex>
#include <atomic>
#include <algorithm>
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

/* Batch calls (ZSTDB200_decompressFrames): entry i's ranges as the caller gave them, uploaded ... */
typedef struct { u64 srcOff, srcSize, dstOff, dstCap; } ZbdSpan;
/* ... and what the kernels find out about it.  Entries that failed in the walk or lie past the workspace own no block and no
 * frame; the others own blocks [block, block + nb) and frames [frame, frame + nf) of the call's arrays. */
typedef struct {
    u64 lit, seq;          /* count pass: literal bytes and sequences the walk counts; scan: the entry's first of each in the workspace */
    u64 out, size;         /* D3: the offset of its output in the back-to-back sum, and its size */
    u32 nb, nf;            /* blocks and frames */
    u32 block, frame;      /* scan: its first block and frame */
    u32 status;            /* 0 or the entry's error code: the first stage that fails it writes it, later stages skip it */
    u32 pad;
} ZbdEntry;

/* A resident DDict's descriptor, written on the device behind its bytes when it becomes resident (zbd_residentDicts): what the
 * kernels need of a dictionary, found through one pointer. */
typedef struct {
    ZbdDictInfo di;
    const u8* dict;        /* the whole dictionary on the device; its content is [dict + di.contentOff, + contentSize) */
    u32 contentSize;
    u32 pad;
} ZbdDictRef;

/* Where the kernels find a block's dictionary: one reference for the whole call (NULL: none), or, in batch calls with a
 * dictionary per entry, an array of one reference per entry (a NULL reference: none), found through the frame's entry. */
typedef struct {
    const ZbdDictRef* one;
    const ZbdDictRef* const* perEntry;
} ZbdDicts;
__device__ __forceinline__ const ZbdDictRef* zbd_dictOf(ZbdDicts ds, const u32* __restrict__ frameEntry, u32 frame)
{
    return ds.perEntry ? ds.perEntry[frameEntry[frame]] : ds.one;
}

/* d_res, the call's results in device memory.  [0, 5): the walk's error, blocks, frames, literal bytes, sequences.  A
 * stream-ordered call also uses [5, 7): the blocks and frames the kernels run (0 when the walk failed or the workspace holds
 * fewer), [10, 12): D3's error and output size, [12, 15): the frames of each D5 width.  [9]: D4 / D5's error (u32).  [7]: a
 * batch call with a device-resident index, 1 when the index check refused it. */
#define ZBD_RES_RUN      5
#define ZBD_RES_REFUSED  7
#define ZBD_RES_EXEC     9
#define ZBD_RES_SCAN     10
#define ZBD_RES_CLASS    12

/* the blocks a kernel of D1 / D2 / D4 runs over: nbBlocks on the synchronous path (res NULL); on the stream-ordered path the
 * count the walk left, or 0 when it failed, and with `scanned` also when D3 refused the call (nothing is written to the
 * output before the sizes are known to fit) */
__device__ __forceinline__ u32 zbd_liveBlocks(const u64* res, u32 nbBlocks, bool scanned)
{
    if (!res) return nbBlocks;
    return scanned && res[ZBD_RES_SCAN] ? 0u : (u32)res[ZBD_RES_RUN];
}

/* ------------------------------------------------------------------------------------------------ D0 on the device
 * One thread follows the headers: a chain of dependent loads, one round trip to device memory per header if nothing helps.
 * The other warps of the CTA (one per remaining SM sub-partition, so that they take no issue slot from the walker's)
 * prefetch the lines in [cursor, cursor + ZBD_WALK_AHEAD) into L1 as the walker publishes its position: a header that
 * lies within that distance of the previous one is an L1 hit. */
#define ZBD_WALK_THREADS 128
#define ZBD_WALK_AHEAD   (16u << 10)
__global__ void __launch_bounds__(ZBD_WALK_THREADS)
zbd_walk_kernel(const u8* __restrict__ src, u64 size, ZbdBlock* blocks, u32 capB, ZbdFrame* frames, u32 capF, u64* res, u32 dictEntropy, u32 dictID)
{
    __shared__ volatile u64 cursor;
    __shared__ volatile u32 walking;
    if (threadIdx.x == 0) { cursor = 0; walking = 1; }
    __syncthreads();
    if (threadIdx.x == 0) {
        u32 nb = 0, nf = 0; u64 lit = 0, seq = 0;
        u32 const e = zbd_walk(src, size, blocks, capB, frames, capF, &nb, &nf, &lit, &seq, dictEntropy != 0u, dictID, &cursor);
        res[0] = e; res[1] = nb; res[2] = nf; res[3] = lit; res[4] = seq;
        bool const fits = e == 0u && nb <= capB && nf <= capF;
        res[ZBD_RES_RUN] = fits ? nb : 0u; res[ZBD_RES_RUN + 1] = fits ? nf : 0u;
        walking = 0;
        return;
    }
    if (threadIdx.x < 32u) return;
    u32 const t = threadIdx.x - 32u, nt = ZBD_WALK_THREADS - 32u;
    u64 done = 0;                                                     /* lines below this offset have been prefetched */
    while (walking) {
        u64 const c = cursor & ~(u64)127;
        u64 const lo = c > done ? c : done, end = c + ZBD_WALK_AHEAD < size ? c + ZBD_WALK_AHEAD : size;
        if (lo >= end) { __nanosleep(200); continue; }
        for (u64 a = lo + 128u * t; a < end; a += 128u * nt) asm volatile("prefetch.global.L1 [%0];" :: "l"(src + a));
        done = end;
    }
}

/* ------------------------------------------------------------------------------------------------ D0 for batch calls
 * The entries' header chains are independent of each other, so one thread walks each entry: a count pass, a scan that gives
 * every entry its place in the call's arrays, and a fill pass that walks again and writes the descriptors there, shifted
 * into the call's coordinates.  zbd_walk is the same function as everywhere else, with the entry's dictionary. */
#define ZBD_ENTRY_THREADS 128
#define ZBD_ENTRY_SCAN    1024        /* the one CTA of the entry scan, of the index check and of the verdict */

/* Batch calls with a device-resident index (ZSTDB200_decompressFramesAsync_deviceOffsets): the checks the host form makes in
 * its host loop, made here in stream order, and the arrays packed into the spans the count, scan and fill passes read.  One
 * CTA, because one entry out of bounds refuses the whole call: then every span is written empty, so that nothing is walked or
 * placed, and *refused = 1 tells the verdict. */
__global__ void __launch_bounds__(ZBD_ENTRY_SCAN)
zbd_entries_pack_kernel(const u64* __restrict__ srcOffsets, const u64* __restrict__ srcSizes, const u64* __restrict__ dstOffsets,
                        const u64* __restrict__ dstCapacities, u32 nbEntries, u64 srcSize, u64 dstCapacity, ZbdSpan* __restrict__ spans,
                        u64* __restrict__ refused)
{
    bool bad = false;
    for (u32 e = threadIdx.x; e < nbEntries; e += ZBD_ENTRY_SCAN) {  /* source ranges inside the input; slots inside the output, ascending and disjoint */
        u64 const so = srcOffsets[e], ss = srcSizes[e], dof = dstOffsets[e], dc = dstCapacities[e];
        bad |= so > srcSize || ss > srcSize - so || dof > dstCapacity || dc > dstCapacity - dof;
        if (e + 1u < nbEntries) bad |= dof + dc > dstOffsets[e + 1u];
    }
    bad = __syncthreads_or(bad);
    for (u32 e = threadIdx.x; e < nbEntries; e += ZBD_ENTRY_SCAN) {
        ZbdSpan s = { 0, 0, 0, 0 };
        if (!bad) { s.srcOff = srcOffsets[e]; s.srcSize = srcSizes[e]; s.dstOff = dstOffsets[e]; s.dstCap = dstCapacities[e]; }
        spans[e] = s;
    }
    if (threadIdx.x == 0) *refused = bad;
}

/* ZSTDB200_findDecompressedSizesAsync: one thread per entry, the host functions' header hop on the entry's range; a range
 * outside the input reads nothing and gets ZBD_CONTENTSIZE_ERROR */
#define ZBD_SIZES_THREADS 128
__global__ void __launch_bounds__(ZBD_SIZES_THREADS)
zbd_sizes_kernel(const u8* __restrict__ src, u64 srcSize, const u64* __restrict__ srcOffsets, const u64* __restrict__ srcSizes, u64 nbEntries,
                 u64* __restrict__ contentSizes, u64* __restrict__ bounds)
{
    u64 const e = (u64)blockIdx.x * ZBD_SIZES_THREADS + threadIdx.x;
    if (e >= nbEntries) return;
    u64 const o = srcOffsets[e], n = srcSizes[e];
    bool const inside = o <= srcSize && n <= srcSize - o;
    if (contentSizes) contentSizes[e] = inside ? zbd_findDecompressedSize(src + o, n) : ZBD_CONTENTSIZE_ERROR;
    if (bounds) bounds[e] = inside ? zbd_decompressBound(src + o, n) : ZBD_CONTENTSIZE_ERROR;
}
__global__ void __launch_bounds__(ZBD_ENTRY_THREADS)
zbd_entries_count_kernel(const u8* __restrict__ src, const ZbdSpan* __restrict__ spans, ZbdEntry* __restrict__ entries, u32 nbEntries,
                         ZbdDicts dicts)
{
    u32 const e = blockIdx.x * ZBD_ENTRY_THREADS + threadIdx.x;
    if (e >= nbEntries) return;
    ZbdSpan const s = spans[e];
    const ZbdDictRef* const r = dicts.perEntry ? dicts.perEntry[e] : dicts.one;
    u32 nb = 0, nf = 0; u64 lit = 0, seq = 0;
    u32 const err = zbd_walk(src + s.srcOff, s.srcSize, NULL, 0, NULL, 0, &nb, &nf, &lit, &seq, r && r->di.entropy, r ? r->di.dictID : 0u);
    ZbdEntry E; memset(&E, 0, sizeof(E));
    E.status = err;
    if (!err) { E.nb = nb; E.nf = nf; E.lit = lit; E.seq = seq; }
    entries[e] = E;
}

/* One CTA: the entries' places in the block, frame, literal and sequence arrays, given out in entry order.  An entry's share
 * of the literal and sequence areas is capped at what its slot allows (dstCap + 16 bytes per block, dstCap / 3); a block
 * behind the cap can only belong to an entry that fails, and the fill pass sends it to the area behind the workspace that
 * nothing reads, as the single-input path does.  An entry whose blocks or frames do not fit in what the entries in front of
 * it left of capB / capF gets workSpace_tooSmall and takes nothing, so the entries behind it keep their room.  A chunk of
 * entries that fits whole takes its places from a parallel prefix sum; one that does not is admitted entry by entry by one
 * thread, from the counts in shared memory.  res[0 .. 5) and res[ZBD_RES_RUN ..] as the walk kernel leaves them: the
 * blocks, frames, literal bytes and sequences of the entries that fit. */
#define ZBD_REFUSED (~0ull)
__global__ void __launch_bounds__(ZBD_ENTRY_SCAN)
zbd_entries_scan_kernel(const ZbdSpan* __restrict__ spans, ZbdEntry* __restrict__ entries, u32 nbEntries, u32 capB, u32 capF, u64* __restrict__ res)
{
    __shared__ u64 warpSum[4][ZBD_ENTRY_SCAN / 32];
    __shared__ u64 carry[4];
    __shared__ u64 chunk[4][ZBD_ENTRY_SCAN];                         /* a chunk admitted one by one: counts in, first places out */
    u32 const tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    if (tid < 4u) carry[tid] = 0;
    __syncthreads();
    for (u32 e0 = 0; e0 < nbEntries; e0 += ZBD_ENTRY_SCAN) {
        u32 const e = e0 + tid, n = nbEntries - e0 < ZBD_ENTRY_SCAN ? nbEntries - e0 : ZBD_ENTRY_SCAN;
        u64 v[4] = { 0, 0, 0, 0 };
        if (e < nbEntries) {
            ZbdEntry const E = entries[e];
            u64 const cap = spans[e].dstCap, litMax = (cap + 16u * (u64)E.nb + 15u) & ~15ull;
            v[0] = E.nb; v[1] = E.nf; v[2] = E.lit < litMax ? E.lit : litMax; v[3] = E.seq < cap / 3u ? E.seq : cap / 3u;
        }
        u64 inc[4], first[4], total[4];
#pragma unroll
        for (u32 k = 0; k < 4u; k++) {
            inc[k] = v[k];
#pragma unroll
            for (u32 o = 1; o < 32u; o <<= 1) { u64 const x = __shfl_up_sync(ZB_FULL, inc[k], o); if (lane >= o) inc[k] += x; }
            if (lane == 31u) warpSum[k][warp] = inc[k];
        }
        __syncthreads();
#pragma unroll
        for (u32 k = 0; k < 4u; k++) {
            first[k] = carry[k] + inc[k] - v[k]; total[k] = carry[k];
            for (u32 w = 0; w < ZBD_ENTRY_SCAN / 32u; w++) { if (w < warp) first[k] += warpSum[k][w]; total[k] += warpSum[k][w]; }
        }
        bool const whole = total[0] <= capB && total[1] <= capF;      /* the same for every thread */
        bool admitted = true;
        if (!whole) {
            for (u32 k = 0; k < 4u; k++) chunk[k][tid] = v[k];
            __syncthreads();
            if (tid == 0) {
                u64 c[4] = { carry[0], carry[1], carry[2], carry[3] };
                for (u32 j = 0; j < n; j++) {
                    u64 const nb = chunk[0][j], nf = chunk[1][j];
                    if (nb && (c[0] + nb > capB || c[1] + nf > capF)) { chunk[0][j] = ZBD_REFUSED; continue; }
                    for (u32 k = 0; k < 4u; k++) { u64 const x = chunk[k][j]; chunk[k][j] = c[k]; c[k] += x; }
                }
                for (u32 k = 0; k < 4u; k++) carry[k] = c[k];
            }
            __syncthreads();
            admitted = chunk[0][tid] != ZBD_REFUSED;
            for (u32 k = 0; k < 4u; k++) first[k] = chunk[k][tid];
        }
        if (e < nbEntries) {
            ZbdEntry& E = entries[e];
            if (!admitted) { E.status = ZB_error_workSpace_tooSmall; E.nb = 0; E.nf = 0; }
            E.block = (u32)first[0]; E.frame = (u32)first[1]; E.lit = first[2]; E.seq = first[3];
        }
        __syncthreads();                                             /* everyone has read carry and chunk */
        if (whole && tid == 0) for (u32 k = 0; k < 4u; k++) carry[k] = total[k];
        __syncthreads();
    }
    if (tid == 0) {
        res[0] = 0; res[1] = carry[0]; res[2] = carry[1]; res[3] = carry[2]; res[4] = carry[3];
        res[ZBD_RES_RUN] = carry[0]; res[ZBD_RES_RUN + 1] = carry[1];
    }
}

/* One thread per entry that fits: its descriptors at the places the scan gave it.  Offsets into the input, frame and block
 * indices (the block whose tables a treeless or repeat-mode block reuses included) and literal and sequence positions move
 * from the entry's coordinates to the call's; every frame records its entry in frameEntry. */
__global__ void __launch_bounds__(ZBD_ENTRY_THREADS)
zbd_entries_fill_kernel(const u8* __restrict__ src, const ZbdSpan* __restrict__ spans, const ZbdEntry* __restrict__ entries, u32 nbEntries,
                        ZbdBlock* __restrict__ blocks, ZbdFrame* __restrict__ frames, u32* __restrict__ frameEntry, ZbdDicts dicts,
                        u64 litCap, u64 seqCap)
{
    u32 const e = blockIdx.x * ZBD_ENTRY_THREADS + threadIdx.x;
    if (e >= nbEntries) return;
    ZbdEntry const E = entries[e];
    if (E.status || E.nb == 0) return;
    ZbdSpan const s = spans[e];
    ZbdBlock* const B = blocks + E.block;
    ZbdFrame* const F = frames + E.frame;
    const ZbdDictRef* const r = dicts.perEntry ? dicts.perEntry[e] : dicts.one;
    u32 nb = 0, nf = 0; u64 lit = 0, seq = 0;
    zbd_walk(src + s.srcOff, s.srcSize, B, E.nb, F, E.nf, &nb, &nf, &lit, &seq, r && r->di.entropy, r ? r->di.dictID : 0u);   /* the count pass's walk: it succeeds */
    u64 const litMax = s.dstCap + 16u * (u64)E.nb, seqMax = s.dstCap / 3u;
    for (u32 k = 0; k < E.nb; k++) {
        ZbdBlock& b = B[k];
        b.srcOff += s.srcOff; b.frame += E.frame;
        if (b.hufSrc < ZBD_DICT) b.hufSrc += E.block;              /* ZBD_NONE and ZBD_DICT stay */
        for (u32 t = 0; t < 3u; t++) if (b.fseSrc[t] < ZBD_DICT) b.fseSrc[t] += E.block;
        b.litPos = b.litPos + b.litRegen <= litMax ? E.lit + b.litPos : litCap;
        b.seqPos = b.seqPos + b.nbSeq <= seqMax ? E.seq + b.seqPos : seqCap;
    }
    for (u32 k = 0; k < E.nf; k++) { F[k].srcOff += s.srcOff; F[k].firstBlock += E.block; frameEntry[E.frame + k] = e; }
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

template <bool PERSISTENT>
__global__ void __launch_bounds__(32 * ZBD_WARPS, 9)             /* 9 CTAs: up to 56 registers (without it ptxas cuts <false> to 48, and its streams decode slower) */
zbd_literals_kernel(const u8* __restrict__ src, const ZbdBlock* __restrict__ blocks, u32 nbBlocks, u8* __restrict__ lits, ZbdBlockOut* __restrict__ bout,
                    ZbdDicts dicts, const u32* __restrict__ frameEntry, const u64* __restrict__ res, u64 litCap)
{
    __shared__ ZbdLitWork work[ZBD_WARPS];
    u32 const lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
    ZbdLitWork& wk = work[w];
    auto block = [&](u32 bi) {
    ZbdBlock const b = blocks[bi];
    if (lane == 0) bout[bi].err = 0;
    if (b.type != ZB_BT_COMPRESSED) return;
    const u8* const c = src + b.srcOff;
    u8* const out = !PERSISTENT || b.litPos + b.litRegen <= litCap ? lits + b.litPos : lits + litCap;
    if (b.litType == 0u) { for (u32 i = lane; i < b.litRegen; i += 32u) out[i] = c[b.litHdr + i]; return; }
    if (b.litType == 1u) { u8 const v = c[b.litHdr]; for (u32 i = lane; i < b.litRegen; i += 32u) out[i] = v; return; }
    if (lane == 0) {
        u32 nbSym = 0, log = 0, dn = 0;
        const ZbdDictRef* const r = b.hufSrc == ZBD_DICT ? zbd_dictOf(dicts, frameEntry, b.frame) : NULL;    /* the walk names ZBD_DICT only with a dictionary */
        const u8* const dp = zbd_hufDescription(&b, blocks, src, r ? r->dict : NULL, r ? &r->di : NULL, &dn);
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
    };
    if (!PERSISTENT) { u32 const bi = blockIdx.x * ZBD_WARPS + w; if (bi < nbBlocks) block(bi); return; }
    u32 const n = zbd_liveBlocks(res, nbBlocks, false);
    for (u32 bi = blockIdx.x * ZBD_WARPS + w; bi < n; bi += gridDim.x * ZBD_WARPS) { block(bi); __syncwarp(); }
}

/* ------------------------------------------------------------------------------------------------ D2 sequences */
struct ZbdSeqWork {
    u32 table[3][512];     /* LL (<= 512 cells), OF (<= 256), ML (<= 512) */
    short norm[3][64];
    u16 next[3][64];
    int log[3];            /* -1: the table's description is corrupt */
};

template <bool PERSISTENT>
__global__ void __launch_bounds__(32 * ZBD_WARPS)
zbd_sequences_kernel(const u8* __restrict__ src, const ZbdBlock* __restrict__ blocks, u32 nbBlocks, u64* __restrict__ seqs, ZbdBlockOut* __restrict__ bout,
                     ZbdDicts dicts, const u32* __restrict__ frameEntry, const u64* __restrict__ res, u64 seqCap)
{
    __shared__ ZbdSeqWork work[ZBD_WARPS];
    u32 const lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
    ZbdSeqWork& wk = work[w];
    auto block = [&](u32 bi) {
    ZbdBlock const b = blocks[bi];
    ZbdRep ident; ident.r[0] = ZBD_SYM(0u, 0u); ident.r[1] = ZBD_SYM(1u, 0u); ident.r[2] = ZBD_SYM(2u, 0u);
    if (b.type != ZB_BT_COMPRESSED || b.nbSeq == 0u) {
        if (lane == 0) { ZbdBlockOut& o = bout[bi]; o.regen = b.type == ZB_BT_COMPRESSED ? b.litRegen : b.rawSize; o.sumLL = 0; o.transfer = ident; }
        return;
    }
    /* three lanes: one decoding table each, from the section that defined it */
    if (lane < 3u) {
        bool const fromDict = b.fseSrc[0] == ZBD_DICT || b.fseSrc[1] == ZBD_DICT || b.fseSrc[2] == ZBD_DICT;
        const ZbdDictRef* const r = fromDict ? zbd_dictOf(dicts, frameEntry, b.frame) : NULL;
        wk.log[lane] = zbd_seqTable(wk.table[lane], wk.norm[lane], wk.next[lane], lane, &b, blocks, src, r ? r->dict : NULL, r ? &r->di : NULL);
    }
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
            else e = zbd_decodeSequences(!PERSISTENT || b.seqPos + b.nbSeq <= seqCap ? seqs + b.seqPos : seqs + seqCap, b.nbSeq, sec + bitstream, avail - bitstream, wk.table[0], wk.log[0], wk.table[1], wk.log[1],
                                         wk.table[2], wk.log[2], &sumLL, &sumML, &tr);
            if (!e && (sumLL > b.litRegen || b.litRegen + sumML > b.blockMax)) e = ZBD_CORRUPT;
        }
        o.regen = e ? 0u : b.litRegen + sumML; o.sumLL = sumLL; o.transfer = tr;
        if (e) o.err = e;
    }
    };
    if (!PERSISTENT) { u32 const bi = blockIdx.x * ZBD_WARPS + w; if (bi < nbBlocks) block(bi); return; }
    u32 const n = zbd_liveBlocks(res, nbBlocks, false);
    for (u32 bi = blockIdx.x * ZBD_WARPS + w; bi < n; bi += gridDim.x * ZBD_WARPS) { block(bi); __syncwarp(); }
}

/* ------------------------------------------------------------------------------------------------ D3 scan
 * One CTA.  Output offsets: prefix sum over all blocks of the call (frames are laid out back to back).  Histories: one
 * warp per frame walks its blocks, 32 transfer functions per round.  res[0] = first error, res[1] = total output bytes.
 * Stream-ordered calls (walk: the call's d_res): the counts are the walk's, and every frame with matches goes to the list
 * of the D5 width that zbd_run would pick for it (classList + k * capF, k = 0: 1024 threads, 1: 128, 2: 32; res[2 + k]
 * frames each).
 * Batch calls (ENTRIES): the sums run over the entries back to back as above, then each entry is moved to its own slot.  Block
 * errors, content sizes and the capacity are checked per entry, into the entry's status word (first error wins: an entry that
 * failed in the walk owns no block); only frames of entries still alive are listed for D5.  res[0] = 0 and res[1] =
 * dstCapacity (the whole buffer), the bound of the tile index the clear kernel resets and D5's bound on a match's end. */
#define SCAN_THREADS 1024
template <bool ENTRIES>
__global__ void __launch_bounds__(SCAN_THREADS)
zbd_scan_kernel(const ZbdBlock* __restrict__ blocks, u32 nbBlocks, const ZbdFrame* __restrict__ frames, u32 nbFrames, ZbdBlockOut* __restrict__ bout,
                u64 dstCapacity, u64* __restrict__ res, ZbdDicts dicts, const u64* __restrict__ walk, u32* __restrict__ classList, u32 capF,
                const ZbdSpan* __restrict__ spans, ZbdEntry* __restrict__ entries, const u32* __restrict__ frameEntry, u32 nbEntries)
{
    __shared__ u64 warpSum[SCAN_THREADS / 32];
    __shared__ u64 carry;
    __shared__ u32 firstErr;
    __shared__ u32 classCount[3];
    u32 const tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    if (walk) { nbBlocks = (u32)walk[ZBD_RES_RUN]; nbFrames = (u32)walk[ZBD_RES_RUN + 1]; }
    if (tid == 0) { carry = 0; firstErr = 0; classCount[0] = classCount[1] = classCount[2] = 0; }
    __syncthreads();
    for (u32 b0 = 0; b0 < nbBlocks; b0 += SCAN_THREADS) {
        u32 const i = b0 + tid;
        u64 v = 0;
        if (i < nbBlocks) {
            v = bout[i].regen;
            if (bout[i].err) atomicMax(ENTRIES ? &entries[frameEntry[blocks[i].frame]].status : &firstErr, bout[i].err);
        }
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
    /* a frame with matches goes to the list of the D5 width that zbd_run would pick for it */
    auto classify = [&](u32 f, const ZbdFrame& fr) {
        if (!fr.nbBlocks) return;
        ZbdBlock const& bl = blocks[fr.firstBlock + fr.nbBlocks - 1u];
        u64 const matches = bl.seqPos + (bl.type == ZB_BT_COMPRESSED ? bl.nbSeq : 0u) - blocks[fr.firstBlock].seqPos;
        if (matches) {
            u32 const k = matches >= 8192u ? 0u : (matches >= 256u ? 1u : 2u);
            classList[(size_t)k * capF + atomicAdd(&classCount[k], 1u)] = f;
        }
    };
    /* per frame: content size, start offset, repcode histories */
    for (u32 f = warp; f < nbFrames; f += SCAN_THREADS / 32u) {
        ZbdFrame const fr = frames[f];
        u64 const fOff = fr.nbBlocks ? bout[fr.firstBlock].dstOff : 0;
        ZbdRep h; h.r[0] = 1u; h.r[1] = 4u; h.r[2] = 8u;            /* format: "Repeat Offsets" start values */
        if (const ZbdDictRef* const r = zbd_dictOf(dicts, frameEntry, f)) {                  /* ... or the dictionary's */
            u32 const e = r->di.entropy, r0 = r->di.rep[0], r1 = r->di.rep[1], r2 = r->di.rep[2];
            if (e) { h.r[0] = r0; h.r[1] = r1; h.r[2] = r2; }
        }
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
        u32* const status = ENTRIES ? &entries[frameEntry[f]].status : &firstErr;
        if (lane == 0 && !(ENTRIES ? *(volatile u32*)status : blockErr) && fr.contentSize != ZBD_CONTENTSIZE_UNKNOWN) {
            u64 const end = (fr.firstBlock + fr.nbBlocks < nbBlocks) ? bout[fr.firstBlock + fr.nbBlocks].dstOff : total;
            if (end - fOff != fr.contentSize) atomicMax(status, ZBD_CORRUPT);
        }
        if (!ENTRIES && walk && lane == 0) classify(f, fr);
    }
    __syncthreads();
    if (ENTRIES) {
        for (u32 e = tid; e < nbEntries; e += SCAN_THREADS) {
            ZbdEntry& E = entries[e];
            E.out = 0; E.size = 0;
            if (E.status || E.nb == 0) continue;
            u64 const start = bout[E.block].dstOff, end = E.block + E.nb < nbBlocks ? bout[E.block + E.nb].dstOff : total;
            E.out = start; E.size = end - start;
            if (end - start > spans[e].dstCap) E.status = 70u;      /* dstSize_tooSmall */
        }
        __syncthreads();
        for (u32 i = tid; i < nbBlocks; i += SCAN_THREADS) {        /* into the entry's slot */
            u32 const e = frameEntry[blocks[i].frame];
            u64 const shift = spans[e].dstOff - entries[e].out;
            bout[i].dstOff += shift; bout[i].frameOff += shift;
        }
        for (u32 f = tid; f < nbFrames; f += SCAN_THREADS) {
            if (entries[frameEntry[f]].status == 0u) classify(f, frames[f]);
        }
        __syncthreads();
        if (tid == 0) { res[0] = 0; res[1] = dstCapacity; res[2] = classCount[0]; res[3] = classCount[1]; res[4] = classCount[2]; }
        return;
    }
    if (tid == 0) {
        u32 e = firstErr;
        if (!e && total > dstCapacity) e = 70u;                      /* dstSize_tooSmall */
        res[0] = e; res[1] = total;
        if (walk) { res[2] = classCount[0]; res[3] = classCount[1]; res[4] = classCount[2]; }
    }
}

/* ------------------------------------------------------------------------------------------------ D4 place
 * One warp per block, every block of the call at once: raw / RLE blocks are written; of a compressed block every literal run
 * goes to its final place and every match becomes (absolute destination, offset, length) — the repcode history runs over the
 * block's sequences from the start history D3 computed.  No byte of the output is READ here, so blocks do not depend on
 * each other.  A match that begins in the dictionary's content gets those bytes here and continues as an ordinary match
 * behind them.  seqs[g] becomes offset | length << 28, matchPos[g] the match's first output byte, and for every 64-byte
 * tile of the output tileFirst[] the first match (in the call's match order) that ends behind the tile's first byte:
 * what D5 needs to find the matches a source range depends on.
 * Batch calls (ENTRIES): blocks of entries that have failed are skipped, an error goes to the entry's status word, and an
 * entry's first block lowers the tile that holds the entry's first byte to its first match (the tile may begin in front of
 * the slot, where nothing else writes it, or in the previous entry's output: any value up to that match is right for D5,
 * which never looks below a frame's first match). */
#define ZBD_TILE_LOG 6u
template <bool PERSISTENT, bool ENTRIES>
__global__ void __launch_bounds__(32 * ZBD_WARPS, 8)             /* 8 CTAs: up to 64 registers (without it ptxas spills <false, false> down to 48) */
zbd_place_kernel(const u8* __restrict__ src, const ZbdBlock* __restrict__ blocks, u32 nbBlocks, const u8* __restrict__ lits, u64* __restrict__ seqs,
                 u64* __restrict__ matchPos, u32* __restrict__ tileFirst, const ZbdBlockOut* __restrict__ bout, u8* __restrict__ dst,
                 ZbdDicts dicts, u32* __restrict__ execErr, const u64* __restrict__ res,
                 const u32* __restrict__ frameEntry, ZbdEntry* __restrict__ entries)
{
    u32 const lane = threadIdx.x & 31u;
    auto block = [&](u32 bi, u32* errWord, bool entryFirst) {
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
        if (ENTRIES && entryFirst && lane == 0) atomicMin(&tileFirst[o.dstOff >> ZBD_TILE_LOG], gNext);
        if (!ENTRIES && o.dstOff == 0 && lane == 0) tileFirst[0] = gNext;
        tiles(o.dstOff, o.dstOff + o.regen, gNext);                 /* no match ends in here: the next block's first one is the first behind these tiles */
        return;
    }
    const u8* const lit = lits + b.litPos;
    u64* const sq = seqs + b.seqPos;
    u64* const mp = matchPos + b.seqPos;
    ZbdRep rep = o.start;
    u64 const inFrame = o.dstOff - o.frameOff;                       /* bytes of the frame in front of this block */
    const ZbdDictRef* const dict = zbd_dictOf(dicts, frameEntry, b.frame);
    u64 const reach = inFrame + (dict ? dict->contentSize : 0u);    /* offsets reach back over the frame so far and the dictionary's content */
    u32 op = 0, lp = 0, err = 0, failedAt = 0;
    if (ENTRIES && entryFirst && lane == 0) atomicMin(&tileFirst[o.dstOff >> ZBD_TILE_LOG], gFirst);
    if (!ENTRIES && o.dstOff == 0 && lane == 0) tileFirst[0] = gFirst;
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
            if (!err && (off == 0u || (u64)off > reach + op)) { err = ZBD_CORRUPT; failedAt = i0 + j; }
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
                const u8* const dp = dict->dict + dict->di.contentOff + dict->contentSize - ((u64)myOff - here);
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
        if (lane == 0) atomicMax(errWord, err);
        tiles(o.dstOff, o.dstOff + o.regen, gNext);
        return;
    }
    u32 const rest = b.litRegen - lp;
    for (u32 k = lane; k < rest; k += 32u) out[op + k] = lit[lp + k];
    tiles(o.dstOff + op, o.dstOff + o.regen, gNext);                 /* behind the block's last match */
    };
    if (!PERSISTENT) { u32 const bi = blockIdx.x * ZBD_WARPS + (threadIdx.x >> 5); if (bi < nbBlocks) block(bi, execErr, false); return; }
    u32 const n = zbd_liveBlocks(res, nbBlocks, true);
    for (u32 bi = blockIdx.x * ZBD_WARPS + (threadIdx.x >> 5); bi < n; bi += gridDim.x * ZBD_WARPS) {
        if (!ENTRIES) { block(bi, execErr, false); continue; }
        ZbdEntry* const E = entries + frameEntry[blocks[bi].frame];
        if (E->status == 0u) block(bi, &E->status, bi == E->block);
    }
}

/* Stream-ordered calls: what zbd_run clears with two memsets once it knows the output size, sized here from D3's total and
 * the walk's sequence count; nothing when the call has failed */
__global__ void zbd_clear_kernel(const u64* __restrict__ res, u32* __restrict__ tileFirst, u8* __restrict__ done)
{
    if (res[ZBD_RES_SCAN] || !res[ZBD_RES_RUN]) return;
    u64 const tiles = (res[ZBD_RES_SCAN + 1] >> ZBD_TILE_LOG) + 4u, flags = res[4] + 4u;
    u64 const stride = (u64)gridDim.x * blockDim.x;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < tiles || i < flags; i += stride) {
        if (i < tiles) tileFirst[i] = 0xFFFFFFFFu;
        if (i < flags) done[i] = 0;
    }
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
__device__ __forceinline__ void zbd_matchesFrame(u32 frame, u32* sTicket, const ZbdBlock* __restrict__ blocks, const ZbdFrame* __restrict__ frames,
                                                 const u64* __restrict__ seqs, const u64* __restrict__ matchPos, const u32* __restrict__ tileFirst,
                                                 u64 totalOut, u8* __restrict__ dst, u8* done, u32* __restrict__ execErr)
{
    u32& sTicket_ = *sTicket;
    u32 const lane = threadIdx.x & 31u;
    ZbdFrame const fr = frames[frame];
    if (fr.nbBlocks == 0) return;
    ZbdBlock const bl = blocks[fr.firstBlock + fr.nbBlocks - 1u];
    u32 const g0 = (u32)blocks[fr.firstBlock].seqPos, g1 = (u32)bl.seqPos + (bl.type == ZB_BT_COMPRESSED ? bl.nbSeq : 0u);     /* the frame's matches */
    if (threadIdx.x == 0) sTicket_ = 0;
    __syncthreads();
    while (true) {
        u32 grp = 0;
        if (lane == 0) grp = atomicAdd(&sTicket_, 1u);                /* matches are handed out in order: a lane only ever waits for matches that were handed out */
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
template <int THREADS>
__global__ void __launch_bounds__(THREADS)
zbd_matches_kernel(const ZbdBlock* __restrict__ blocks, const ZbdFrame* __restrict__ frames, const u64* __restrict__ seqs, const u64* __restrict__ matchPos,
                   const u32* __restrict__ tileFirst, u64 totalOut, u8* __restrict__ dst, u8* done, u32* __restrict__ execErr)
{
    __shared__ u32 sTicket;
    zbd_matchesFrame<THREADS>(blockIdx.x, &sTicket, blocks, frames, seqs, matchPos, tileFirst, totalOut, dst, done, execErr);
}
/* stream-ordered calls: a persistent grid over the frames D3 listed for this width (list, res[ZBD_RES_CLASS + cls] of them),
 * the ticket reset between frames; nothing when the call failed.  Batch calls (ENTRIES): a frame whose entry failed in D4 is
 * skipped, and an error goes to the entry's status word. */
template <int THREADS, bool ENTRIES>
__global__ void __launch_bounds__(THREADS)
zbd_matches_list_kernel(const ZbdBlock* __restrict__ blocks, const ZbdFrame* __restrict__ frames, const u64* __restrict__ seqs, const u64* __restrict__ matchPos,
                        const u32* __restrict__ tileFirst, u8* __restrict__ dst, u8* done, u32* __restrict__ execErr,
                        const u32* __restrict__ list, const u64* __restrict__ res, u32 cls, const u32* __restrict__ frameEntry, ZbdEntry* __restrict__ entries)
{
    __shared__ u32 sTicket;
    __shared__ u32 sFailed;
    if (res[ZBD_RES_SCAN] || !res[ZBD_RES_RUN]) return;
    u64 const n = res[ZBD_RES_CLASS + cls], totalOut = res[ZBD_RES_SCAN + 1];
    for (u64 k = blockIdx.x; k < n; k += gridDim.x) {
        u32 const f = list[k];
        if (!ENTRIES) zbd_matchesFrame<THREADS>(f, &sTicket, blocks, frames, seqs, matchPos, tileFirst, totalOut, dst, done, execErr);
        else {
            u32* const status = &entries[frameEntry[f]].status;
            if (threadIdx.x == 0) sFailed = *(volatile u32*)status;   /* one reading for the whole CTA: the frame loop below synchronises */
            __syncthreads();
            if (!sFailed) zbd_matchesFrame<THREADS>(f, &sTicket, blocks, frames, seqs, matchPos, tileFirst, totalOut, dst, done, status);
        }
        __syncthreads();                                             /* every warp is done with the frame before the ticket is reset */
    }
}

/* ------------------------------------------------------------------------------------------------ host driver */
/* Digested dictionary of the decoder (lib/zstd.h:1000-1030, zstd_ddict.c): parsed on the host when it is digested
 * (zbd_parseDict), uploaded whole (header and content) to the device of the first context that uses it, and resident there
 * from then on.  The one form in which the decoder sees a dictionary: a ZSTD_createDDict object, which any number of contexts
 * on one device may use; a context's sticky dictionary (ZSTD_DCtx_loadDictionary, ZSTD_DCtx_refPrefix); and the bytes a call
 * passes with ZSTD_decompress_usingDict, digested into the context's own object (ZSTD_DCtx_s::callDict) on every call.
 * The compressor's ZSTD_CDict_s keeps a 128 KiB tail of the content; the decoder needs all of it. */
struct ZSTD_DDict_s {
    std::unique_ptr<u8[]> copy;    /* ZSTD_createDDict's copy of the bytes (ZSTD_dlm_byCopy) */
    const u8* bytes;               /* the whole dictionary: that copy, or the caller's buffer */
    size_t size;
    ZbdDictInfo di;
    mutable std::mutex lock;       /* guards the device state below; residentOn is also read without it */
    mutable int device;            /* -1 until the device buffer exists */
    mutable std::atomic<int> residentOn;   /* the device the digest has been uploaded to, -1 until then; set once the upload completed */
    mutable ZbDevBuf<u8> d_dict;   /* the bytes, then (at zbd_refOffset) the descriptor */
    mutable ZbdDictRef ref;        /* the descriptor's host image, the source of its upload */
};
static size_t zbd_refOffset(size_t dictSize) { return (dictSize + 15) & ~(size_t)15; }
/* the device descriptor of a DDict resident on the device in question */
static const ZbdDictRef* zbd_ref(const ZSTD_DDict* dd) { return (const ZbdDictRef*)((const u8*)dd->d_dict + zbd_refOffset(dd->size)); }
struct ZbdDDictFree { void operator()(ZSTD_DDict* dd) const { ZSTD_freeDDict(dd); } };
typedef std::unique_ptr<ZSTD_DDict, ZbdDDictFree> ZbdDDictPtr;
enum ZbdDictUses { ZBD_DICT_DONT_USE, ZBD_DICT_USE_ONCE, ZBD_DICT_USE_ALWAYS };    /* ZSTD_dictUses_e, zstd_decompress_internal.h */

struct ZSTD_DCtx_s {
    int device, bindDevice;
    ZbStream stream;
    ZbDevBuf<ZbdBlock> d_blocks; ZbDevBuf<ZbdFrame> d_frames;
    ZbDevBuf<ZbdBlockOut> d_bout;  /* one more than d_blocks */
    ZbDevBuf<u8> d_lits; ZbDevBuf<u64> d_seqs, d_matchPos;
    ZbDevBuf<u32> d_tileFirst; ZbDevBuf<u8> d_done;
    ZbDevBuf<u8> d_in, d_out;
    ZbDevBuf<u64> d_res; u32* d_execErr;   /* walker / scan results; d_execErr lies in d_res[9] */
    ZbHostBuf<u64> h_res;          /* their mirror */
    /* streaming front end (ZSTD_decompressStream): compressed bytes collected until a frame is complete, output waiting to be handed out */
    std::vector<u8> dsIn, dsOut; size_t dsOutPos;
    size_t hostWalkMax;          /* ZBD_HOSTWALK_MAX, or ZSTDB200_HOSTWALK_MAX from the environment (tests: 0 forces the kernel walk) */
    ZbHostBuf<u8> h_stage;       /* copy of a device-resident input's compressed bytes, for the header walk */
    /* the sticky dictionary (zstd_decompress.c:316-322, :1178-1193): ddict is localDict or a borrowed DDict, NULL for none */
    ZbdDDictPtr localDict;       /* ZSTD_DCtx_loadDictionary's copy, or ZSTD_DCtx_refPrefix's digest of the caller's bytes */
    const ZSTD_DDict* ddict;
    int dictUses;                /* ZbdDictUses; a prefix is used by the next call (in streaming, the next frame) only */
    ZbdDDictPtr callDict;        /* digest of the dictionary bytes the current call passes; reads the caller's buffer in place */
    size_t maxWindow;            /* ZSTD_d_windowLogMax: ZSTD_decompressStream refuses frames whose window is larger */
    ZbEvents ev;
    ZSTDB200_dstats stats;
    /* stream-ordered calls (ZSTDB200_decompressDeviceAsync).  d_class: D3's frame lists per D5 width.  grid: CTAs of the
     * persistent grids (as many as resident at once) of D1, D2, D4, the clear kernel and D5 at 1024, 128 and 32 threads */
    ZbOrder order;
    ZbDevBuf<u32> d_class;
    u32 grid[7];
    /* batch calls (ZSTDB200_decompressFrames[Async]): the entries' spans are staged in a ring of page-locked slots, as the
     * compressor stages its descriptors (slot s is free again once evStage[s], recorded behind its upload, has completed);
     * d_verdict holds a synchronous call's result and sizes for its one read-back into h_verdict */
    ZbDevBuf<ZbdSpan> d_spans; ZbDevBuf<ZbdEntry> d_entries; ZbDevBuf<u32> d_frameEntry;   /* the entry of every frame */
    ZbHostBuf<ZbdSpan> stage[ZSTDB200_ASYNC_SLOTS]; bool stageBusy[ZSTDB200_ASYNC_SLOTS]; u32 stageNext; ZbEvents evStage;
    /* calls with a DDict per entry: the entries' dictionary references, staged in the same slots as the spans */
    ZbDevBuf<const ZbdDictRef*> d_refs; ZbHostBuf<const ZbdDictRef*> stageRefs[ZSTDB200_ASYNC_SLOTS];
    ZbDevBuf<unsigned long long> d_verdict; ZbHostBuf<unsigned long long> h_verdict;
};

/* one decompression call, as an entry point describes it */
struct ZbdCall {
    void* dst; size_t dstCapacity;
    const void* src; size_t srcSize;
    const void* dict; size_t dictSize;  /* bytes to digest into the context's callDict (host memory); NULL / 0: none */
    const ZSTD_DDict* ddict;            /* otherwise: a digested dictionary, or NULL for none */
    bool deviceMemory;                  /* dst and src are device memory */
    cudaStream_t stream;                /* device calls: the caller's stream, NULL for the context's */
};

#define ZBD_WINDOW_DEFAULT ((size_t)1 << 27)    /* ZSTD_WINDOWLOG_LIMIT_DEFAULT */

extern "C" ZSTD_DCtx* ZSTD_createDCtx(void)                          /* lib/zstd.h:289 */
{
    ZSTD_DCtx* d = new (std::nothrow) ZSTD_DCtx();                  /* value-initialised: every plain member is zero */
    if (!d) return NULL;
    d->device = -1;
    d->maxWindow = ZBD_WINDOW_DEFAULT;
    {   const char* const e = getenv("ZSTDB200_HOSTWALK_MAX"); d->hostWalkMax = e ? (size_t)strtoull(e, NULL, 10) : ZBD_HOSTWALK_MAX; }
    d->bindDevice = zb_contextDevice();
    return d;
}
extern "C" size_t ZSTD_freeDCtx(ZSTD_DCtx* d) { return d ? zb_deleteOnDevice(d, &d->order) : 0; }   /* accepts NULL, lib/zstd.h:290 */
static size_t zbd_ctxInit(ZSTD_DCtx* d)
{
    if (d->device >= 0) CK(cudaSetDevice(d->device));
    else {
        int n = 0;
        if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) { cudaGetLastError(); return ZB_ERR(ZB_error_GENERIC); }
        int const dev = d->bindDevice < 0 ? 0 : d->bindDevice;
        CK(cudaSetDevice(dev));
        ZbStream st; ZbEvents ev; ZbOrder order;                     /* the context's once all exist: all or nothing */
        TRY(st.ensure());
        TRY(ev.ensure(7, true));
        TRY(order.create());
        int sms = 0;
        CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
        int per[7] = { 0 };
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per[0], zbd_literals_kernel<true>, 32 * ZBD_WARPS, 0));
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per[1], zbd_sequences_kernel<true>, 32 * ZBD_WARPS, 0));
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per[2], zbd_place_kernel<true, false>, 32 * ZBD_WARPS, 0));
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per[3], zbd_clear_kernel, 256, 0));
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per[4], zbd_matches_list_kernel<1024, false>, 1024, 0));
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per[5], zbd_matches_list_kernel<128, false>, 128, 0));
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per[6], zbd_matches_list_kernel<32, false>, 32, 0));
        for (int k = 0; k < 7; k++) d->grid[k] = (u32)(per[k] > 0 ? per[k] : 1) * (u32)(sms > 0 ? sms : 1);
        d->stream = std::move(st); d->ev = std::move(ev); d->order = std::move(order);
        d->device = dev;
    }
    TRY(d->d_res.ensure(16)); TRY(d->h_res.ensure(16));
    d->d_execErr = (u32*)(d->d_res + 9);
    return 0;
}
/* the decoder's arrays are allocated with slack (an eighth more, and 64): calls of similar sizes reuse them */
template <typename T> static size_t zbd_reserve(ZbDevBuf<T>& b, size_t need) { return b.ensure(need, need / 8 + 64); }

/* the dictionary description the kernels take: dd's, or none */
static ZbdDictInfo zbd_dictInfo(const ZSTD_DDict* dd)
{
    ZbdDictInfo di;
    if (dd) di = dd->di; else memset(&di, 0, sizeof(di));
    return di;
}

/* the kernels' dictionary for a call with one: dd's descriptor (dd resident on the context's device), or none */
static ZbdDicts zbd_oneDict(const ZSTD_DDict* dd)
{
    ZbdDicts ds = { dd ? zbd_ref(dd) : NULL, NULL };
    return ds;
}

/* D1 .. D4 over descriptors that are already on the device, with the resident dictionary dd (NULL: none); returns the
 * output size */
static size_t zbd_run(ZSTD_DCtx* d, u8* d_dst, size_t dstCapacity, const u8* d_src, u32 nb, u32 nf, u64 seqCount, const ZSTD_DDict* dd,
                      cudaStream_t st)
{
    ZbdDicts const ds = zbd_oneDict(dd);
    CK(cudaMemsetAsync(d->d_execErr, 0, sizeof(u32), st));
    CK(cudaEventRecord(d->ev[1], st));
    u32 const grid = (nb + ZBD_WARPS - 1u) / ZBD_WARPS;
    zbd_literals_kernel<false><<<grid, 32 * ZBD_WARPS, 0, st>>>(d_src, d->d_blocks, nb, d->d_lits, d->d_bout, ds, NULL, NULL, 0);
    CK(cudaEventRecord(d->ev[2], st));
    zbd_sequences_kernel<false><<<grid, 32 * ZBD_WARPS, 0, st>>>(d_src, d->d_blocks, nb, d->d_seqs, d->d_bout, ds, NULL, NULL, 0);
    CK(cudaEventRecord(d->ev[3], st));
    zbd_scan_kernel<false><<<1, SCAN_THREADS, 0, st>>>(d->d_blocks, nb, d->d_frames, nf, d->d_bout, (u64)dstCapacity, d->d_res, ds, NULL, NULL, 0, NULL, NULL, NULL, 0);
    CK(cudaMemcpyAsync(d->h_res, d->d_res, 2 * sizeof(u64), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));                                  /* nothing is written to dst before the sizes are known to fit */
    if (d->h_res[0]) return ZB_ERR((u32)d->h_res[0]);
    size_t const total = (size_t)d->h_res[1];
    CK(cudaEventRecord(d->ev[4], st));
    TRY(zbd_reserve(d->d_tileFirst, (total >> ZBD_TILE_LOG) + 4));
    TRY(zbd_reserve(d->d_done, (size_t)seqCount + 4));
    CK(cudaMemsetAsync(d->d_tileFirst, 0xFF, ((total >> ZBD_TILE_LOG) + 4) * sizeof(u32), st));
    CK(cudaMemsetAsync(d->d_done, 0, (size_t)seqCount + 4, st));
    zbd_place_kernel<false, false><<<grid, 32 * ZBD_WARPS, 0, st>>>(d_src, d->d_blocks, nb, d->d_lits, d->d_seqs, d->d_matchPos, d->d_tileFirst, d->d_bout, d_dst,
                                                             ds, d->d_execErr, NULL, NULL, NULL);
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
    TRY(zbd_reserve(d->d_blocks, nb));
    TRY(d->d_bout.ensure((size_t)nb + 1, nb / 8 + 64));
    TRY(zbd_reserve(d->d_frames, nf));
    TRY(zbd_reserve(d->d_lits, (size_t)litBytes + 16));
    TRY(zbd_reserve(d->d_seqs, (size_t)seqCount + 1));
    TRY(zbd_reserve(d->d_matchPos, (size_t)seqCount + 1));
    return 0;
}


/* Digests dict[0 .. size) into dd, which reads those bytes in place.  A dictionary without the magic number, shorter than 8
 * bytes, or a prefix (rawContent) is raw content (zstd_ddict.c:95-107); a zstd-format one is parsed on the host. */
static size_t zbd_digestDict(ZSTD_DDict* dd, const u8* dict, size_t size, bool rawContent)
{
    dd->bytes = dict; dd->size = dict ? size : 0; dd->residentOn.store(-1);
    memset(&dd->di, 0, sizeof(dd->di));
    if (rawContent || dd->size == 0) return 0;
    u32 const e = zbd_parseDict(&dd->di, dict, size);
    return e ? ZB_ERR(e) : 0;
}

/* A DDict that reads dict in place (byCopy = false) or its own copy of it; NULL when the entropy tables are corrupted or
 * memory runs out */
static ZSTD_DDict* zbd_createDDict(const void* dict, size_t dictSize, bool byCopy, bool rawContent)
{
    size_t const size = dict ? dictSize : 0;
    ZSTD_DDict* dd = new (std::nothrow) ZSTD_DDict();                   /* value-initialised: every plain member is zero */
    if (!dd) return NULL;
    dd->device = -1;
    const u8* bytes = (const u8*)dict;
    if (byCopy && size) {
        dd->copy.reset(new (std::nothrow) u8[size]);
        if (!dd->copy) { delete dd; return NULL; }
        memcpy(dd->copy.get(), dict, size);
        bytes = dd->copy.get();
    }
    if (zb_isErr(zbd_digestDict(dd, bytes, size, rawContent))) { delete dd; return NULL; }
    return dd;
}

/* Makes the DDicts dds[0 .. n) resident on `device`, the compressor's rule for a CDict (ZbRun::prepareDicts): a DDict's buffer is
 * allocated on the first device that uses it (one device per DDict: another gets parameter_unsupported), its bytes and its
 * descriptor are uploaded once per digest, and the upload has completed before another context can use it.  The uploads of
 * all of them go out before one synchronisation.  Their locks are held until then, taken in address order, so that calls
 * that name the same DDicts in other orders cannot deadlock; a DDict named twice counts once.  A resident DDict costs a call
 * nothing: no copy, no synchronisation.  *uploaded (NULL: not wanted) grows by the bytes copied. */
static size_t zbd_residentDicts(const ZSTD_DDict* const* dds, size_t n, int device, cudaStream_t st, size_t* uploaded)
{
    std::vector<const ZSTD_DDict*> v(dds, dds + n);
    std::sort(v.begin(), v.end());
    v.erase(std::unique(v.begin(), v.end()), v.end());
    std::vector<std::unique_lock<std::mutex>> locks;
    locks.reserve(v.size());
    for (const ZSTD_DDict* dd : v) locks.emplace_back(dd->lock);
    std::vector<const ZSTD_DDict*> up;
    for (const ZSTD_DDict* dd : v) {
        if (dd->device >= 0 && dd->device != device) return ZB_ERR(ZB_error_parameter_unsupported);
        if (dd->residentOn.load(std::memory_order_relaxed) != device) up.push_back(dd);
    }
    if (up.empty()) return 0;
    for (const ZSTD_DDict* dd : up) {
        size_t const at = zbd_refOffset(dd->size);
        TRY(zbd_reserve(dd->d_dict, at + sizeof(ZbdDictRef)));
        dd->device = device;
        dd->ref.di = dd->di; dd->ref.dict = dd->d_dict; dd->ref.contentSize = (u32)(dd->size - dd->di.contentOff); dd->ref.pad = 0;
        CK(cudaMemcpyAsync(dd->d_dict, dd->bytes, dd->size, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(dd->d_dict + at, &dd->ref, sizeof(ZbdDictRef), cudaMemcpyHostToDevice, st));
        if (uploaded) *uploaded += dd->size + sizeof(ZbdDictRef);
    }
    CK(cudaStreamSynchronize(st));                                    /* the sources are pageable memory that may change after the call */
    for (const ZSTD_DDict* dd : up) dd->residentOn.store(device, std::memory_order_release);
    return 0;
}
static size_t zbd_residentDict(const ZSTD_DDict* dd, int device, cudaStream_t st) { return zbd_residentDicts(&dd, 1, device, st, NULL); }

/* dictionary bytes passed to a call, digested into the context's callDict */
static size_t zbd_digestCallDict(ZSTD_DCtx* d, const void* dict, size_t dictSize)
{
    if (!d->callDict) d->callDict.reset(zbd_createDDict(NULL, 0, false, false));
    if (!d->callDict) return ZB_ERR(ZB_error_memory_allocation);
    return zbd_digestDict(d->callDict.get(), (const u8*)dict, dictSize, false);
}

/* D0 on a host-readable copy of the compressed bytes: count the blocks and frames, then describe them into B and F */
static u32 zbd_walkHost(const ZbdDictInfo& di, const u8* in, size_t size, std::vector<ZbdBlock>& B, std::vector<ZbdFrame>& F,
                        u32* nb, u32* nf, u64* lit, u64* seq)
{
    u32 const e = zbd_walk(in, size, NULL, 0, NULL, 0, nb, nf, lit, seq, di.entropy != 0, di.dictID);
    if (e) return e;
    B.resize(*nb ? *nb : 1); F.resize(*nf ? *nf : 1);
    return zbd_walk(in, size, B.data(), *nb, F.data(), *nf, nb, nf, lit, seq, di.entropy != 0, di.dictID);
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
    TRY(zbd_ctxInit(d));
    CK(d->order.hostWait());                                         /* stream-ordered calls still queued use the buffers below */
    memset(&d->stats, 0, sizeof(d->stats));
    cudaStream_t const st = c.stream ? c.stream : d->stream;
    const ZSTD_DDict* dd = c.ddict;
    if (c.dict && c.dictSize) { TRY(zbd_digestCallDict(d, c.dict, c.dictSize)); dd = d->callDict.get(); }
    if (dd && dd->size == 0) dd = NULL;                               /* an empty dictionary is none */
    if (dd) TRY(zbd_residentDict(dd, d->device, st));
    ZbdDictInfo const di = zbd_dictInfo(dd);
    /* D0: block and frame descriptors */
    const u8* hostIn = c.deviceMemory ? NULL : (const u8*)c.src;
    if (c.deviceMemory && c.srcSize <= d->hostWalkMax) {
        TRY(d->h_stage.ensure(c.srcSize, c.srcSize / 4 + 4096));
        CK(cudaMemcpyAsync(d->h_stage, c.src, c.srcSize, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        hostIn = d->h_stage;
    }
    std::vector<ZbdBlock> B; std::vector<ZbdFrame> F;
    u32 nb = 0, nf = 0; u64 lit = 0, seq = 0;
    if (hostIn) { u32 const e = zbd_walkHost(di, hostIn, c.srcSize, B, F, &nb, &nf, &lit, &seq); if (e) return ZB_ERR(e); }
    else {                                                            /* the walk kernel; once more if the arrays were too small */
        u32 capB = (u32)(c.srcSize / 4096u) + 1024u, capF = 1024u;
        for (int attempt = 0; attempt < 2; attempt++) {
            TRY(zbd_ensure(d, capB, capF, 0, 0));
            zbd_walk_kernel<<<1, ZBD_WALK_THREADS, 0, st>>>((const u8*)c.src, (u64)c.srcSize, d->d_blocks, (u32)d->d_blocks.cap, d->d_frames, (u32)d->d_frames.cap, d->d_res, di.entropy, di.dictID);
            CK(cudaMemcpyAsync(d->h_res, d->d_res, 5 * sizeof(u64), cudaMemcpyDeviceToHost, st));
            CK(cudaStreamSynchronize(st));
            if (d->h_res[0]) return ZB_ERR((u32)d->h_res[0]);
            if (d->h_res[1] <= d->d_blocks.cap && d->h_res[2] <= d->d_frames.cap) break;
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
        TRY(zbd_reserve(d->d_in, c.srcSize + 16));
        TRY(zbd_reserve(d->d_out, outCap + 16));
        CK(cudaEventRecord(d->ev[0], st));
        CK(cudaMemcpyAsync(d->d_in, c.src, c.srcSize, cudaMemcpyHostToDevice, st));
        runSrc = d->d_in; runDst = d->d_out;
    }
    TRY(zbd_ensure(d, nb, nf, lit, seq));                            /* the walk kernel's descriptors fit: d_blocks and d_frames keep them */
    if (hostIn) {
        CK(cudaMemcpyAsync(d->d_blocks, B.data(), (size_t)nb * sizeof(ZbdBlock), cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(d->d_frames, F.data(), (size_t)nf * sizeof(ZbdFrame), cudaMemcpyHostToDevice, st));
        CK(cudaStreamSynchronize(st));                               /* B and F are pageable: the copies end before a return can free them */
    }
    size_t const total = zbd_run(d, runDst, outCap, runSrc, nb, nf, seq, dd, st);
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

/* ------------------------------------------------------------------------------------------------ dictionaries and parameters
 * (lib/zstd.h:1000-1030, :1160-1210; zstd_decompress.c:1697-1960) */
extern "C" ZSTD_DDict* ZSTD_createDDict(const void* dict, size_t dictSize)                  /* zstd_ddict.c:178 */
{
    return zbd_createDDict(dict, dictSize, true, false);
}
extern "C" size_t ZSTD_freeDDict(ZSTD_DDict* dd) { return zb_deleteOnDevice(dd); }           /* accepts NULL, zstd_ddict.c:212 */
extern "C" unsigned ZSTD_getDictID_fromDDict(const ZSTD_DDict* dd) { return dd ? dd->di.dictID : 0u; }      /* zstd_ddict.c:236 */
extern "C" unsigned ZSTD_getDictID_fromFrame(const void* src, size_t srcSize)               /* zstd_decompress.c:1642 */
{
    ZbdFrameHeader h;
    if (zbd_readFrameHeader(&h, (const u8*)src, srcSize) || h.skippable) return 0;
    return h.dictID;
}

static void zbd_clearDict(ZSTD_DCtx* d) { d->localDict.reset(); d->ddict = NULL; d->dictUses = ZBD_DICT_DONT_USE; }
/* the sticky dictionary for the next call (or frame); a prefix is handed out once */
static const ZSTD_DDict* zbd_getDDict(ZSTD_DCtx* d)
{
    switch (d->dictUses) {
    case ZBD_DICT_USE_ALWAYS: return d->ddict;
    case ZBD_DICT_USE_ONCE: d->dictUses = ZBD_DICT_DONT_USE; return d->ddict;
    default: zbd_clearDict(d); return NULL;
    }
}
/* ZSTD_decompressStream holds part of a frame, or output of one that is still to be handed out (streamStage != zdss_init) */
static bool zbd_midFrame(const ZSTD_DCtx* d) { return !d->dsIn.empty() || d->dsOutPos < d->dsOut.size(); }

static size_t zbd_loadDict(ZSTD_DCtx* d, const void* dict, size_t dictSize, bool byCopy, bool rawContent)
{
    if (!d) return ZB_ERR(ZB_error_GENERIC);
    if (zbd_midFrame(d)) return ZB_ERR(ZB_error_stage_wrong);
    zbd_clearDict(d);
    if (dict && dictSize) {
        d->localDict.reset(zbd_createDDict(dict, dictSize, byCopy, rawContent));
        if (!d->localDict) return ZB_ERR(ZB_error_memory_allocation);    /* corrupted entropy tables too, as in the reference (:1705-1706) */
        d->ddict = d->localDict.get(); d->dictUses = ZBD_DICT_USE_ALWAYS;
    }
    return 0;
}
extern "C" size_t ZSTD_DCtx_loadDictionary(ZSTD_DCtx* d, const void* dict, size_t dictSize)    /* :1718 */
{
    return zbd_loadDict(d, dict, dictSize, true, false);
}
extern "C" size_t ZSTD_DCtx_refPrefix(ZSTD_DCtx* d, const void* prefix, size_t prefixSize)     /* :1730 */
{
    TRY(zbd_loadDict(d, prefix, prefixSize, false, true));
    d->dictUses = ZBD_DICT_USE_ONCE;
    return 0;
}
extern "C" size_t ZSTD_DCtx_refDDict(ZSTD_DCtx* d, const ZSTD_DDict* ddict)                    /* :1778 */
{
    if (!d) return ZB_ERR(ZB_error_GENERIC);
    if (zbd_midFrame(d)) return ZB_ERR(ZB_error_stage_wrong);
    zbd_clearDict(d);
    if (ddict) { d->ddict = ddict; d->dictUses = ZBD_DICT_USE_ALWAYS; }
    return 0;
}
extern "C" size_t ZSTD_DCtx_setParameter(ZSTD_DCtx* d, ZSTD_dParameter param, int value)       /* :1904 */
{
    if (!d) return ZB_ERR(ZB_error_GENERIC);
    if (zbd_midFrame(d)) return ZB_ERR(ZB_error_stage_wrong);
    if (param != ZSTD_d_windowLogMax) return ZB_ERR(ZB_error_parameter_unsupported);
    if (value == 0) value = 27;                                          /* ZSTD_WINDOWLOG_LIMIT_DEFAULT */
    if (value < 10 || value > 31) return ZB_ERR(ZB_error_parameter_outOfBound);   /* ZSTD_WINDOWLOG_ABSOLUTEMIN, ZSTD_WINDOWLOG_MAX */
    d->maxWindow = (size_t)1 << value;
    return 0;
}
extern "C" size_t ZSTD_DCtx_reset(ZSTD_DCtx* d, ZSTD_ResetDirective reset)                     /* :1945 */
{
    if (!d) return ZB_ERR(ZB_error_GENERIC);
    if (reset == ZSTD_reset_session_only || reset == ZSTD_reset_session_and_parameters) {
        d->dsIn.clear(); d->dsOut.clear(); d->dsOutPos = 0;
    }
    if (reset == ZSTD_reset_parameters || reset == ZSTD_reset_session_and_parameters) {
        if (zbd_midFrame(d)) return ZB_ERR(ZB_error_stage_wrong);
        zbd_clearDict(d);
        d->maxWindow = ZBD_WINDOW_DEFAULT;
    }
    return 0;
}

/* ------------------------------------------------------------------------------------------------ stream-ordered calls
 * The host reads no header, so the workspace is sized from srcSize and dstCapacity alone (include/zstd_b200.h states the rule
 * and its cost).  Literals: at most dstCapacity, plus 16 bytes of alignment per block.  Sequences: at most dstCapacity / 3,
 * every match being 3 bytes or more.  A block whose literals or sequences lie past those bounds can only belong to a call
 * that fails (its blocks regenerate more than dstCapacity, or one of them is corrupt): D1 / D2 decode it into an area behind
 * the bounds, which nothing reads, so that its verdict is still the one zbd_run gives. */
#define ZBD_NBSEQ_MAX (0xFFFFu + 0x7F00u)                       /* the largest Number_of_Sequences */
static u64 zbd_asyncBlocks(size_t srcSize, size_t dstCapacity) { return (u64)srcSize / 16u + (u64)dstCapacity / 1024u + 1024u; }

/* the verdict of a stream-ordered call, with zbd_decompress's precedence: the walk, the workspace, D3, D4 / D5 */
__global__ void zbd_result_kernel(const u64* __restrict__ res, u32 capB, u32 capF, unsigned long long* result)
{
    u32 const exec = *(const u32*)(res + ZBD_RES_EXEC);
    size_t r;
    if (res[0]) r = ZB_ERR(res[0]);
    else if (res[1] > capB || res[2] > capF) r = ZB_ERR(ZB_error_workSpace_tooSmall);
    else if (res[1] == 0) r = 0;
    else if (res[ZBD_RES_SCAN]) r = ZB_ERR(res[ZBD_RES_SCAN]);
    else if (exec) r = ZB_ERR(exec);
    else r = (size_t)res[ZBD_RES_SCAN + 1];
    *result = r;
}

static bool zbd_dictResident(const ZSTD_DDict* dd, int device) { return dd->residentOn.load(std::memory_order_acquire) == device; }

/* A stream-ordered call's workspace: blocks and frames (capB, capF), literal bytes and sequences (litCap, seqCap: D1 / D2
 * decode a block whose literals or sequences lie past them into the spare area behind, which nothing reads), and the output
 * bytes the tile index covers (outMax).  Batch calls (batch) also need d_frameEntry. */
struct ZbdCaps { u32 capB, capF; u64 litCap, seqCap, outMax; };
static size_t zbd_reserveWork(ZSTD_DCtx* d, const ZbdCaps& w, bool batch)
{
    TRY(zbd_reserve(d->d_blocks, w.capB));
    TRY(d->d_bout.ensure((size_t)w.capB + 1, w.capB / 8 + 64));
    TRY(zbd_reserve(d->d_frames, w.capF));
    if (batch) TRY(zbd_reserve(d->d_frameEntry, w.capF));
    TRY(zbd_reserve(d->d_class, 3 * (size_t)w.capF));
    TRY(zbd_reserve(d->d_lits, w.litCap + ZB_BLOCK_MAX + 32));
    TRY(zbd_reserve(d->d_seqs, w.seqCap + ZBD_NBSEQ_MAX + 1));
    TRY(zbd_reserve(d->d_matchPos, w.seqCap + 1));
    TRY(zbd_reserve(d->d_done, w.seqCap + 4));
    TRY(zbd_reserve(d->d_tileFirst, (w.outMax >> ZBD_TILE_LOG) + 4));
    return 0;
}

/* D1 .. D5 of a stream-ordered call on st, behind its walk: literals, sequences, scan, clear, place and the three D5 widths,
 * ZBD_ENQUEUE_LAUNCHES kernels, persistent grids that read their counts from the walk's words in d_res and write nothing once
 * the walk or D3 has failed.  Batch calls (ENTRIES) run over the nbEntries entries in d_spans / d_entries / d_frameEntry.
 * Launch errors are the caller's to collect (cudaGetLastError). */
#define ZBD_ENQUEUE_LAUNCHES 8
template <bool ENTRIES>
static void zbd_enqueue(ZSTD_DCtx* d, const u8* src, u8* dst, size_t dstCapacity, const ZbdCaps& w, ZbdDicts ds, u32 nbEntries,
                          cudaStream_t st)
{
    u64* const res = d->d_res;
    u32* const frameEntry = ENTRIES ? (u32*)d->d_frameEntry : NULL;
    ZbdEntry* const entries = ENTRIES ? (ZbdEntry*)d->d_entries : NULL;
    const ZbdSpan* const spans = ENTRIES ? (const ZbdSpan*)d->d_spans : NULL;
    u32 const blockGrid = (w.capB + ZBD_WARPS - 1u) / ZBD_WARPS;
    auto grid = [&](int k, u32 most) { return d->grid[k] < most ? d->grid[k] : most; };
    zbd_literals_kernel<true><<<grid(0, blockGrid), 32 * ZBD_WARPS, 0, st>>>(src, d->d_blocks, w.capB, d->d_lits, d->d_bout, ds, frameEntry, res, w.litCap);
    zbd_sequences_kernel<true><<<grid(1, blockGrid), 32 * ZBD_WARPS, 0, st>>>(src, d->d_blocks, w.capB, d->d_seqs, d->d_bout, ds, frameEntry, res, w.seqCap);
    zbd_scan_kernel<ENTRIES><<<1, SCAN_THREADS, 0, st>>>(d->d_blocks, w.capB, d->d_frames, w.capF, d->d_bout, (u64)dstCapacity, res + ZBD_RES_SCAN, ds, res,
                                                         d->d_class, w.capF, spans, entries, frameEntry, nbEntries);
    zbd_clear_kernel<<<grid(3, (u32)(w.seqCap / 256u) + 1u), 256, 0, st>>>(res, d->d_tileFirst, d->d_done);
    zbd_place_kernel<true, ENTRIES><<<grid(2, blockGrid), 32 * ZBD_WARPS, 0, st>>>(src, d->d_blocks, w.capB, d->d_lits, d->d_seqs, d->d_matchPos, d->d_tileFirst,
                                                                                   d->d_bout, dst, ds, d->d_execErr, res, frameEntry, entries);
    u32* const list = d->d_class;
    zbd_matches_list_kernel<1024, ENTRIES><<<grid(4, w.capF), 1024, 0, st>>>(d->d_blocks, d->d_frames, d->d_seqs, d->d_matchPos, d->d_tileFirst, dst,
                                                                             d->d_done, d->d_execErr, list, res, 0, frameEntry, entries);
    zbd_matches_list_kernel<128, ENTRIES><<<grid(5, w.capF), 128, 0, st>>>(d->d_blocks, d->d_frames, d->d_seqs, d->d_matchPos, d->d_tileFirst, dst,
                                                                           d->d_done, d->d_execErr, list + w.capF, res, 1, frameEntry, entries);
    zbd_matches_list_kernel<32, ENTRIES><<<grid(6, w.capF), 32, 0, st>>>(d->d_blocks, d->d_frames, d->d_seqs, d->d_matchPos, d->d_tileFirst, dst,
                                                                         d->d_done, d->d_execErr, list + 2 * (size_t)w.capF, res, 2, frameEntry, entries);
}

/* D0 .. D5 and the verdict enqueued on the caller's stream, with the context's sticky dictionary, under ZbOrder's rule; a DDict's
 * first upload on the device (on the context's stream, which synchronises) is refused under capture too */
static size_t zbd_decompressAsync(ZSTD_DCtx* d, void* dst, size_t dstCapacity, const void* src, size_t srcSize,
                                  unsigned long long* result, cudaStream_t st)
{
    if (!d || !result) return ZB_ERR(ZB_error_GENERIC);
    if (d->dictUses == ZBD_DICT_USE_ONCE) { zbd_clearDict(d); return ZB_ERR(ZB_error_parameter_unsupported); }   /* a prefix is forgotten */
    ZbDeviceGuard guard;
    ZbOrder::Call call(d->order);
    TRY(call.begin(d->device, st));
    TRY(zbd_ctxInit(d));
    memset(&d->stats, 0, sizeof(d->stats));
    const ZSTD_DDict* dd = zbd_getDDict(d);
    if (dd && dd->size == 0) dd = NULL;                               /* an empty dictionary is none */
    if (dd && call.capturing && !zbd_dictResident(dd, d->device)) return ZB_ERR(ZB_error_stage_wrong);
    u64 const cap = zbd_asyncBlocks(srcSize, dstCapacity);
    if (cap > 0x7FFFFFFFull) return ZB_ERR(ZB_error_memory_allocation);
    ZbdCaps const w = { (u32)cap, (u32)cap, (u64)dstCapacity + 16u * cap, (u64)dstCapacity / 3u, (u64)dstCapacity };
    TRY(call.size([&]() { return zbd_reserveWork(d, w, false); }));
    if (dd) TRY(zbd_residentDict(dd, d->device, d->stream));           /* no copy once resident */
    ZbdDictInfo const di = zbd_dictInfo(dd);
    TRY(call.enter(st));
    const u8* const in = (const u8*)src;
    CK(cudaMemsetAsync(d->d_execErr, 0, sizeof(u32), st));
    zbd_walk_kernel<<<1, ZBD_WALK_THREADS, 0, st>>>(in, (u64)srcSize, d->d_blocks, w.capB, d->d_frames, w.capF, d->d_res, di.entropy, di.dictID);
    zbd_enqueue<false>(d, in, (u8*)dst, dstCapacity, w, zbd_oneDict(dd), 0, st);
    zbd_result_kernel<<<1, 1, 0, st>>>(d->d_res, w.capB, w.capF, result);
    CK(cudaGetLastError());
    TRY(call.leave(st));
    d->stats.launches = ZBD_ENQUEUE_LAUNCHES + 2;                     /* and the walk and the verdict */
    return 0;
}

extern "C" size_t ZSTDB200_decompressDeviceAsync(ZSTD_DCtx* d, void* d_dst, size_t dstCapacity, const void* d_src, size_t srcSize,
                                                 unsigned long long* d_result, void* stream)
{
    return zbd_decompressAsync(d, d_dst, dstCapacity, d_src, srcSize, d_result, (cudaStream_t)stream);
}

/* ------------------------------------------------------------------------------------------------ batch calls
 * ZSTDB200_decompressFrames[Async] (include/zstd_b200.h states the contract): the stream-ordered pipeline above with D0 walked
 * entry by entry and D3 .. D5 in their per-entry mode, then this verdict.  One CTA: every entry's size or error code to
 * sizes (NULL: none), and to *result the sum of the sizes, or the error code of the lowest-index entry that failed.  A call
 * whose device-resident index was refused (refused non-NULL and set) gets parameter_outOfBound, and sizes is not written. */
__global__ void __launch_bounds__(ZBD_ENTRY_SCAN)
zbd_entries_result_kernel(const ZbdEntry* __restrict__ entries, u32 nbEntries, unsigned long long* sizes, unsigned long long* result,
                          const u64* __restrict__ refused)
{
    __shared__ u32 firstBad;
    __shared__ unsigned long long total;
    if (refused && *refused) { if (threadIdx.x == 0) *result = ZB_ERR(ZB_error_parameter_outOfBound); return; }
    if (threadIdx.x == 0) { firstBad = 0xFFFFFFFFu; total = 0; }
    __syncthreads();
    u64 sum = 0;
    for (u32 e = threadIdx.x; e < nbEntries; e += ZBD_ENTRY_SCAN) {
        ZbdEntry const& E = entries[e];
        if (E.status) atomicMin(&firstBad, e); else sum += E.size;
        if (sizes) sizes[e] = E.status ? (unsigned long long)ZB_ERR(E.status) : E.size;
    }
#pragma unroll
    for (u32 o = 16; o > 0; o >>= 1) sum += __shfl_down_sync(ZB_FULL, sum, o);
    if ((threadIdx.x & 31u) == 0) atomicAdd(&total, (unsigned long long)sum);
    __syncthreads();
    if (threadIdx.x == 0) *result = firstBad != 0xFFFFFFFFu ? (unsigned long long)ZB_ERR(entries[firstBad].status) : total;
}

/* Entry i's dictionary reference for a batch call with a DDict per entry: *ref = dd's descriptor when dd is resident on
 * `device`, NULL for no dictionary (dd NULL or empty).  Returns 0, 1 when dd is not resident yet, or parameter_unsupported
 * when it is resident on another device.  No lock: residentOn is set once the upload has completed. */
static size_t zbd_entryRef(const ZSTD_DDict* dd, int device, const ZbdDictRef** ref)
{
    *ref = NULL;
    if (!dd || dd->size == 0) return 0;                               /* an empty dictionary is none */
    int const on = dd->residentOn.load(std::memory_order_acquire);
    if (on == device) { *ref = zbd_ref(dd); return 0; }
    return on >= 0 ? ZB_ERR(ZB_error_parameter_unsupported) : 1;
}

/* ownVerdict: the result and sizes go to the context's d_verdict (the synchronous call) instead of result / sizes.
 * perEntryDicts: entry i is decoded with ddicts[i] (ddicts NULL: no dictionary for any), not with the sticky dictionary.
 * deviceIndex: the four arrays are device memory; zbd_entries_pack_kernel checks them and writes the spans in stream order,
 * instead of the host loop and the staging ring (not with perEntryDicts) */
static size_t zbd_decompressFrames(ZSTD_DCtx* d, u8* dst, size_t dstCapacity, const size_t* dstOffsets, const size_t* dstCapacities,
                                   const u8* src, size_t srcSize, const size_t* srcOffsets, const size_t* srcSizes, size_t n, bool deviceIndex,
                                   bool perEntryDicts, const ZSTD_DDict* const* ddicts,
                                   unsigned long long* sizes, unsigned long long* result, bool ownVerdict, cudaStream_t st)
{
    if (!d || (!result && !ownVerdict)) return ZB_ERR(ZB_error_GENERIC);
    if (n && (!dstOffsets || !dstCapacities || !srcOffsets || !srcSizes)) return ZB_ERR(ZB_error_GENERIC);
    if (d->dictUses == ZBD_DICT_USE_ONCE) { zbd_clearDict(d); return ZB_ERR(ZB_error_parameter_unsupported); }   /* a prefix is forgotten */
    u64 sumCap = 0;
    if (deviceIndex) {                          /* the slots' sum is not known here; they lie inside the output */
        if (((uintptr_t)dstOffsets | (uintptr_t)dstCapacities | (uintptr_t)srcOffsets | (uintptr_t)srcSizes) & 7u)
            return ZB_ERR(ZB_error_parameter_outOfBound);
        sumCap = dstCapacity;
    }
    for (size_t i = 0; !deviceIndex && i < n; i++) {    /* source ranges inside the input; slots inside the output, ascending and disjoint */
        if (srcOffsets[i] > srcSize || srcSizes[i] > srcSize - srcOffsets[i]) return ZB_ERR(ZB_error_parameter_outOfBound);
        if (dstOffsets[i] > dstCapacity || dstCapacities[i] > dstCapacity - dstOffsets[i]) return ZB_ERR(ZB_error_parameter_outOfBound);
        if (i + 1 < n && dstOffsets[i] + dstCapacities[i] > dstOffsets[i + 1]) return ZB_ERR(ZB_error_parameter_outOfBound);
        sumCap += dstCapacities[i];
    }
    ZbDeviceGuard guard;
    ZbOrder::Call call(d->order);
    TRY(call.begin(d->device, st));
    TRY(zbd_ctxInit(d));
    memset(&d->stats, 0, sizeof(d->stats));
    const ZSTD_DDict* dd = perEntryDicts ? NULL : zbd_getDDict(d);    /* a call with a dictionary per entry leaves the sticky one as it is */
    if (dd && dd->size == 0) dd = NULL;                               /* an empty dictionary is none */
    if (dd && call.capturing && !zbd_dictResident(dd, d->device)) return ZB_ERR(ZB_error_stage_wrong);
    u64 const cap = zbd_asyncBlocks(srcSize, dstCapacity) + (u64)n;
    if (cap > 0x7FFFFFFFull) return ZB_ERR(ZB_error_memory_allocation);
    u32 const capB = (u32)cap, capF = (u32)cap, nbEntries = (u32)n;
    ZbdCaps const w = { capB, capF, sumCap + 32u * cap, sumCap / 3u, (u64)dstCapacity };   /* the entries' shares (zbd_entries_scan_kernel) fit */
    size_t const slots = n ? n : 1;
    TRY(call.size([&]() -> size_t {
        TRY(zbd_reserveWork(d, w, true));
        TRY(zbd_reserve(d->d_spans, slots)); TRY(zbd_reserve(d->d_entries, slots));
        if (!deviceIndex) {
            TRY(d->evStage.ensure(ZSTDB200_ASYNC_SLOTS, false));
            for (u32 s = 0; s < ZSTDB200_ASYNC_SLOTS; s++)           /* every slot, so that any can serve a capture */
                if (d->stage[s].cap < slots) { TRY(d->stage[s].ensure(slots, slots / 8 + 64)); d->stageBusy[s] = false; }
        }
        if (perEntryDicts) {
            TRY(zbd_reserve(d->d_refs, slots));
            for (u32 s = 0; s < ZSTDB200_ASYNC_SLOTS; s++)
                if (d->stageRefs[s].cap < slots) { TRY(d->stageRefs[s].ensure(slots, slots / 8 + 64)); d->stageBusy[s] = false; }
        }
        if (ownVerdict) { TRY(zbd_reserve(d->d_verdict, slots + 1)); TRY(d->h_verdict.ensure(slots + 1, slots / 8 + 64)); }
        return 0;
    }));
    if (dd) TRY(zbd_residentDict(dd, d->device, d->stream));           /* no copy once resident */
    ZbdDicts ds = zbd_oneDict(dd);
    if (ownVerdict) { result = d->d_verdict; sizes = sizes ? d->d_verdict + 1 : NULL; }
    /* the spans, into the next slot of the ring; under capture the wait needs the relaxed mode (the event was recorded outside the graph) */
    u32 slot = 0;
    if (!deviceIndex) {
        slot = d->stageNext;
        d->stageNext = (slot + 1u) % ZSTDB200_ASYNC_SLOTS;
        if (d->stageBusy[slot]) {
            cudaStreamCaptureMode m = cudaStreamCaptureModeRelaxed;
            CK(cudaThreadExchangeStreamCaptureMode(&m));
            cudaError_t const e = cudaEventSynchronize(d->evStage[slot]);
            cudaThreadExchangeStreamCaptureMode(&m);
            CK(e);
            d->stageBusy[slot] = false;
        }
        ZbdSpan* const h = d->stage[slot];
        for (size_t i = 0; i < n; i++) { h[i].srcOff = srcOffsets[i]; h[i].srcSize = srcSizes[i]; h[i].dstOff = dstOffsets[i]; h[i].dstCap = dstCapacities[i]; }
    }
    if (perEntryDicts) {
        /* the entries' references, into the same slot.  A resident DDict costs one atomic read; the DDicts that are not resident
         * yet are made resident together, with one synchronisation, then every reference is taken again. */
        const ZbdDictRef** const hr = d->stageRefs[slot];
        std::vector<const ZSTD_DDict*> cold;
        for (size_t i = 0; i < n; i++) {
            size_t const r = zbd_entryRef(ddicts ? ddicts[i] : NULL, d->device, &hr[i]);
            if (zb_isErr(r)) return r;
            if (r) cold.push_back(ddicts[i]);
        }
        if (!cold.empty()) {
            if (call.capturing) return ZB_ERR(ZB_error_stage_wrong);
            TRY(zbd_residentDicts(cold.data(), cold.size(), d->device, d->stream, &d->stats.h2d_bytes));
            for (size_t i = 0; i < n; i++) if (zbd_entryRef(ddicts[i], d->device, &hr[i])) return ZB_ERR(ZB_error_GENERIC);
        }
        ds.perEntry = d->d_refs;
    }
    TRY(call.enter(st));
    u64* const res = d->d_res;
    if (deviceIndex)
        zbd_entries_pack_kernel<<<1, ZBD_ENTRY_SCAN, 0, st>>>((const u64*)srcOffsets, (const u64*)srcSizes, (const u64*)dstOffsets, (const u64*)dstCapacities,
                                                              nbEntries, (u64)srcSize, (u64)dstCapacity, d->d_spans, res + ZBD_RES_REFUSED);
    else {
        if (n) CK(cudaMemcpyAsync(d->d_spans, d->stage[slot], n * sizeof(ZbdSpan), cudaMemcpyHostToDevice, st));
        if (n && perEntryDicts) CK(cudaMemcpyAsync(d->d_refs, d->stageRefs[slot], n * sizeof(const ZbdDictRef*), cudaMemcpyHostToDevice, st));
        if (!call.capturing) { CK(cudaEventRecord(d->evStage[slot], st)); d->stageBusy[slot] = true; }
    }
    u32 const entryGrid = (nbEntries + ZBD_ENTRY_THREADS - 1u) / ZBD_ENTRY_THREADS + (n == 0);
    zbd_entries_count_kernel<<<entryGrid, ZBD_ENTRY_THREADS, 0, st>>>(src, d->d_spans, d->d_entries, nbEntries, ds);
    zbd_entries_scan_kernel<<<1, ZBD_ENTRY_SCAN, 0, st>>>(d->d_spans, d->d_entries, nbEntries, capB, capF, res);
    zbd_entries_fill_kernel<<<entryGrid, ZBD_ENTRY_THREADS, 0, st>>>(src, d->d_spans, d->d_entries, nbEntries, d->d_blocks, d->d_frames, d->d_frameEntry,
                                                                     ds, w.litCap, w.seqCap);
    zbd_enqueue<true>(d, src, dst, dstCapacity, w, ds, nbEntries, st);
    zbd_entries_result_kernel<<<1, ZBD_ENTRY_SCAN, 0, st>>>(d->d_entries, nbEntries, sizes, result, deviceIndex ? res + ZBD_RES_REFUSED : NULL);
    CK(cudaGetLastError());
    TRY(call.leave(st));
    d->stats.launches = ZBD_ENQUEUE_LAUNCHES + (deviceIndex ? 5 : 4);   /* and count, scan, fill, the verdict, the index check */
    return 0;
}

extern "C" size_t ZSTDB200_decompressFramesAsync(ZSTD_DCtx* d, void* d_dst, size_t dstCapacity, const size_t* dstOffsets, const size_t* dstCapacities,
                                                 const void* d_src, size_t srcSize, const size_t* srcOffsets, const size_t* srcSizes,
                                                 size_t nbEntries, unsigned long long* d_dSizes, unsigned long long* d_result, void* stream)
{
    return zbd_decompressFrames(d, (u8*)d_dst, dstCapacity, dstOffsets, dstCapacities, (const u8*)d_src, srcSize, srcOffsets, srcSizes, nbEntries,
                                false, false, NULL, d_dSizes, d_result, false, (cudaStream_t)stream);
}
extern "C" size_t ZSTDB200_decompressFramesAsync_usingDDicts(ZSTD_DCtx* d, void* d_dst, size_t dstCapacity, const size_t* dstOffsets,
                                                             const size_t* dstCapacities, const void* d_src, size_t srcSize,
                                                             const size_t* srcOffsets, const size_t* srcSizes, size_t nbEntries,
                                                             const ZSTD_DDict* const* ddicts, unsigned long long* d_dSizes,
                                                             unsigned long long* d_result, void* stream)
{
    return zbd_decompressFrames(d, (u8*)d_dst, dstCapacity, dstOffsets, dstCapacities, (const u8*)d_src, srcSize, srcOffsets, srcSizes, nbEntries,
                                false, true, ddicts, d_dSizes, d_result, false, (cudaStream_t)stream);
}
extern "C" size_t ZSTDB200_decompressFramesAsync_deviceOffsets(ZSTD_DCtx* d, void* d_dst, size_t dstCapacity, const unsigned long long* d_dstOffsets,
                                                               const unsigned long long* d_dstCapacities, const void* d_src, size_t srcSize,
                                                               const unsigned long long* d_srcOffsets, const unsigned long long* d_srcSizes,
                                                               size_t nbEntries, unsigned long long* d_dSizes, unsigned long long* d_result, void* stream)
{
    static_assert(sizeof(size_t) == sizeof(unsigned long long), "the index arrays are read as size_t");
    return zbd_decompressFrames(d, (u8*)d_dst, dstCapacity, (const size_t*)d_dstOffsets, (const size_t*)d_dstCapacities, (const u8*)d_src, srcSize,
                                (const size_t*)d_srcOffsets, (const size_t*)d_srcSizes, nbEntries, true, false, NULL, d_dSizes, d_result, false,
                                (cudaStream_t)stream);
}

/* One kernel on the caller's stream; no buffer of the context is used, so the call may be captured at any time and does not
 * take part in the context's call order.  The device is chosen as zbd_ctxInit chooses it, without creating anything. */
extern "C" size_t ZSTDB200_findDecompressedSizesAsync(ZSTD_DCtx* d, const void* d_src, size_t srcSize, const unsigned long long* d_srcOffsets,
                                                      const unsigned long long* d_srcSizes, size_t nbEntries,
                                                      unsigned long long* d_contentSizes, unsigned long long* d_bounds, void* stream)
{
    if (!d || (!d_contentSizes && !d_bounds)) return ZB_ERR(ZB_error_GENERIC);
    if (nbEntries && (!d_srcOffsets || !d_srcSizes)) return ZB_ERR(ZB_error_GENERIC);
    if (((uintptr_t)d_srcOffsets | (uintptr_t)d_srcSizes | (uintptr_t)d_contentSizes | (uintptr_t)d_bounds) & 7u)
        return ZB_ERR(ZB_error_parameter_outOfBound);
    ZbDeviceGuard guard;
    int dev = d->device;
    if (dev < 0) {
        int n = 0;
        if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) { cudaGetLastError(); return ZB_ERR(ZB_error_GENERIC); }
        dev = d->bindDevice < 0 ? 0 : d->bindDevice;
    }
    CK(cudaSetDevice(dev));
    if (nbEntries == 0) return 0;
    u64 const grid = (nbEntries + ZBD_SIZES_THREADS - 1u) / ZBD_SIZES_THREADS;
    if (grid > 0x7FFFFFFFull) return ZB_ERR(ZB_error_parameter_outOfBound);
    zbd_sizes_kernel<<<(u32)grid, ZBD_SIZES_THREADS, 0, (cudaStream_t)stream>>>((const u8*)d_src, (u64)srcSize, (const u64*)d_srcOffsets,
                                                                                (const u64*)d_srcSizes, (u64)nbEntries, (u64*)d_contentSizes, (u64*)d_bounds);
    CK(cudaGetLastError());
    return 0;
}

/* the stream-ordered call on the caller's stream (NULL: the context's), then one read-back of the verdict and the sizes */
static size_t zbd_decompressFramesSync(ZSTD_DCtx* d, void* d_dst, size_t dstCapacity, const size_t* dstOffsets, const size_t* dstCapacities,
                                       const void* d_src, size_t srcSize, const size_t* srcOffsets, const size_t* srcSizes,
                                       size_t nbEntries, bool perEntryDicts, const ZSTD_DDict* const* ddicts, size_t* dSizes, void* stream)
{
    if (!d) return ZB_ERR(ZB_error_GENERIC);
    ZbDeviceGuard guard;
    TRY(zbd_ctxInit(d));
    cudaStream_t const st = stream ? (cudaStream_t)stream : (cudaStream_t)d->stream;
    unsigned long long marker = 0;                                    /* non-NULL: the sizes are wanted */
    TRY(zbd_decompressFrames(d, (u8*)d_dst, dstCapacity, dstOffsets, dstCapacities, (const u8*)d_src, srcSize, srcOffsets, srcSizes, nbEntries,
                             false, perEntryDicts, ddicts, dSizes ? &marker : NULL, NULL, true, st));
    size_t const words = 1 + (dSizes ? nbEntries : 0);
    CK(cudaMemcpyAsync(d->h_verdict, d->d_verdict, words * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    for (size_t i = 0; dSizes && i < nbEntries; i++) dSizes[i] = (size_t)d->h_verdict[1 + i];
    return (size_t)d->h_verdict[0];
}
extern "C" size_t ZSTDB200_decompressFrames(ZSTD_DCtx* d, void* d_dst, size_t dstCapacity, const size_t* dstOffsets, const size_t* dstCapacities,
                                            const void* d_src, size_t srcSize, const size_t* srcOffsets, const size_t* srcSizes,
                                            size_t nbEntries, size_t* dSizes, void* stream)
{
    return zbd_decompressFramesSync(d, d_dst, dstCapacity, dstOffsets, dstCapacities, d_src, srcSize, srcOffsets, srcSizes, nbEntries,
                                    false, NULL, dSizes, stream);
}
extern "C" size_t ZSTDB200_decompressFrames_usingDDicts(ZSTD_DCtx* d, void* d_dst, size_t dstCapacity, const size_t* dstOffsets,
                                                        const size_t* dstCapacities, const void* d_src, size_t srcSize,
                                                        const size_t* srcOffsets, const size_t* srcSizes, size_t nbEntries,
                                                        const ZSTD_DDict* const* ddicts, size_t* dSizes, void* stream)
{
    return zbd_decompressFramesSync(d, d_dst, dstCapacity, dstOffsets, dstCapacities, d_src, srcSize, srcOffsets, srcSizes, nbEntries,
                                    true, ddicts, dSizes, stream);
}

/* ------------------------------------------------------------------------------------------------ one-shot calls */
extern "C" size_t ZSTD_decompress_usingDict(ZSTD_DCtx* d, void* dst, size_t dstCapacity, const void* src, size_t srcSize,
                                            const void* dict, size_t dictSize)                                            /* lib/zstd.h:955 */
{
    ZbdCall const c = { dst, dstCapacity, src, srcSize, dict, dictSize, NULL, false, NULL };
    return zbd_decompress(d, c);
}
extern "C" size_t ZSTD_decompress_usingDDict(ZSTD_DCtx* d, void* dst, size_t dstCapacity, const void* src, size_t srcSize,
                                             const ZSTD_DDict* ddict)                                                     /* lib/zstd.h:1017 */
{
    ZbdCall const c = { dst, dstCapacity, src, srcSize, NULL, 0, ddict, false, NULL };
    return zbd_decompress(d, c);
}
extern "C" size_t ZSTD_decompressDCtx(ZSTD_DCtx* d, void* dst, size_t dstCapacity, const void* src, size_t srcSize)      /* lib/zstd.h:299 */
{
    if (!d) return ZB_ERR(ZB_error_GENERIC);
    return ZSTD_decompress_usingDDict(d, dst, dstCapacity, src, srcSize, zbd_getDDict(d));     /* zstd_decompress.c:1195 */
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
    ZbdCall const c = { d_dst, dstCapacity, d_src, srcSize, dict, dictSize, NULL, true, (cudaStream_t)stream };
    return zbd_decompress(d, c);
}
extern "C" size_t ZSTDB200_decompressDevice(ZSTD_DCtx* d, void* d_dst, size_t dstCapacity, const void* d_src, size_t srcSize, void* stream)
{
    if (!d) return ZB_ERR(ZB_error_GENERIC);
    ZbdCall const c = { d_dst, dstCapacity, d_src, srcSize, NULL, 0, zbd_getDDict(d), true, (cudaStream_t)stream };
    return zbd_decompress(d, c);
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
    ZbdFrameSizeInfo fi;
    u32 const e = zbd_frameSizeInfo(&fi, (const u8*)src, srcSize);
    return e ? ZB_ERR(e) : (size_t)fi.cSize;
}
/* lib/zstd.h:1437, :1460 */
extern "C" unsigned long long ZSTD_findDecompressedSize(const void* src, size_t srcSize) { return zbd_findDecompressedSize((const u8*)src, srcSize); }
extern "C" unsigned long long ZSTD_decompressBound(const void* src, size_t srcSize) { return zbd_decompressBound((const u8*)src, srcSize); }

/* ------------------------------------------------------------------------------------------------ streaming (lib/zstd.h:880-924)
 * The GPU decodes whole frames, so the stream front end collects compressed bytes until a frame is complete
 * (ZSTD_findFrameCompressedSize), decodes it, and hands the result out as the caller makes room.  Return value as in the
 * reference: 0 when a frame has been decoded and handed out completely, else a hint (> 0) for the next input size. */
/* the content size, capped at what the frame's blocks can regenerate (blocks x 128 KiB): a corrupt content-size field
 * must not size the output buffer */
static size_t zbd_frameOutputBound(const u8* in, size_t size)
{
    ZbdFrameHeader h;
    if (zbd_readFrameHeader(&h, in, size) || h.skippable) return 0;
    size_t p = h.headerSize, blocks = 0;
    while (p + 3 <= size) { u32 const bh = zbd_le(in + p, 3); blocks++; p += 3u + (((bh >> 1) & 3u) == ZB_BT_RLE ? 1u : (bh >> 3)); if (bh & 1u) break; }
    size_t const most = blocks * (size_t)ZB_BLOCK_MAX;
    return h.contentSize < (u64)most ? (size_t)h.contentSize : most;
}
extern "C" ZSTD_DStream* ZSTD_createDStream(void) { return ZSTD_createDCtx(); }
extern "C" size_t ZSTD_freeDStream(ZSTD_DStream* zds) { return ZSTD_freeDCtx(zds); }
extern "C" size_t ZSTD_initDStream(ZSTD_DStream* zds)
{
    if (!zds) return ZB_ERR(ZB_error_GENERIC);
    zds->dsIn.clear(); zds->dsOut.clear();
    zds->dsOutPos = 0;
    zbd_clearDict(zds);                                                /* ZSTD_DCtx_refDDict(zds, NULL), zstd_decompress.c:1752 */
    return 5;                                                         /* a frame header's first bytes, as the reference suggests (ZSTD_startingInputLength) */
}
extern "C" size_t ZSTD_DStreamInSize(void) { return ZB_BLOCK_MAX + 3; }  /* lib/zstd.h:922 */
extern "C" size_t ZSTD_DStreamOutSize(void) { return ZB_BLOCK_MAX; }
extern "C" size_t ZSTD_decompressStream(ZSTD_DStream* d, ZSTD_outBuffer* out, ZSTD_inBuffer* in)
{
    if (!d || !out || !in) return ZB_ERR(ZB_error_GENERIC);
    if (out->pos > out->size) return ZB_ERR(ZB_error_dstSize_tooSmall);
    if (in->pos > in->size) return ZB_ERR(ZB_error_srcSize_wrong);
    auto handOut = [&]() -> size_t {
        size_t const have = d->dsOut.size() - d->dsOutPos, room = out->size - out->pos, n = have < room ? have : room;
        if (n) { memcpy((u8*)out->dst + out->pos, d->dsOut.data() + d->dsOutPos, n); out->pos += n; d->dsOutPos += n; }
        if (d->dsOutPos == d->dsOut.size()) { d->dsOut.clear(); d->dsOutPos = 0; }
        return d->dsOut.size() - d->dsOutPos;
    };
    if (handOut() != 0) return d->dsOut.size() - d->dsOutPos;            /* room first: input is only taken while nothing is waiting */
    size_t carried = d->dsIn.size();                                     /* bytes that came with earlier calls */
    d->dsIn.insert(d->dsIn.end(), (const u8*)in->src + in->pos, (const u8*)in->src + in->size);
    in->pos = in->size;
    bool decoded = false;
    while (!d->dsIn.empty()) {
        size_t const fs = ZSTD_findFrameCompressedSize(d->dsIn.data(), d->dsIn.size());
        bool const incomplete = ZSTD_isError(fs) && ZSTD_getErrorCode(fs) == ZB_error_srcSize_wrong;
        if (ZSTD_isError(fs) && !incomplete) return fs;
        /* ZSTD_d_windowLogMax, decided from the header once it is complete (zstd_decompress.c:2227-2229).  As in the reference,
         * a frame that arrives whole with one call whose output buffer has room for its stated content size is decoded in
         * one pass, which does not apply the limit (:2183-2199). */
        {   ZbdFrameHeader h;
            if (!zbd_readFrameHeader(&h, d->dsIn.data(), d->dsIn.size()) && !h.skippable) {
                size_t const free = out->size - out->pos, room = free > d->dsOut.size() ? free - d->dsOut.size() : 0;   /* behind earlier frames' output */
                bool const onePass = !incomplete && carried == 0 && h.contentSize != ZBD_CONTENTSIZE_UNKNOWN && (u64)room >= h.contentSize;
                u64 const window = h.windowSize < 1024u ? 1024u : h.windowSize;
                if (!onePass && window > (u64)d->maxWindow) return ZB_ERR(16);        /* frameParameter_windowTooLarge */
            }
        }
        if (incomplete) break;                                           /* the frame is not complete yet */
        size_t const bound = zbd_frameOutputBound(d->dsIn.data(), fs);
        size_t const base = d->dsOut.size();
        try { d->dsOut.resize(base + bound + 1); }
        catch (const std::exception&) { return ZB_ERR(ZB_error_memory_allocation); }     /* no C++ exception may cross the C ABI */
        size_t const r = ZSTD_decompressDCtx(d, d->dsOut.data() + base, bound, d->dsIn.data(), fs);
        if (ZSTD_isError(r)) { d->dsOut.resize(base); return r; }
        d->dsOut.resize(base + r);
        d->dsIn.erase(d->dsIn.begin(), d->dsIn.begin() + (ptrdiff_t)fs);
        carried = carried > fs ? carried - fs : 0;
        decoded = true;
    }
    size_t const waiting = handOut();
    if (waiting) return waiting;
    (void)decoded;
    if (d->dsIn.empty()) return 0;                                       /* at a frame border with everything handed out */
    return ZB_BLOCK_MAX + 3;                                             /* in the middle of a frame: more input, please */
}
