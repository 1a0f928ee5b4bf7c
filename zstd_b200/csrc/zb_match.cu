/* zb_match.cu — K1: LZ77 match-finder ("fast" and "doubleFast" strategies) = K1a candidate walk, K1b greedy parse, K1c merge.
 *
 * Replaces the CPU loops ZSTD_compressBlock_fast_noDict_generic / _extDict_generic
 * (lib/compress/zstd_fast.c:192-423, :709-960) and ZSTD_compressBlock_doubleFast_noDict_generic
 * (zstd_double_fast.c:105-323) with a data-parallel formulation:
 *   - K1a (one CTA per CHUNK of up to 4 blocks) keeps the chunk's hash table in shared memory — primed from
 *     the <=128 KiB in front of the chunk (zstd_fast.c:53-85 does this for dictionaries, zstdmt_compress.c:1182-1227 for
 *     job overlaps), then alive through all blocks of the chunk — and visits the positions in BATCHES of 1024: every
 *     position of a batch reads its bucket, positions that found no candidate are inserted (one atomicMax each: the
 *     lowest position of a batch wins a bucket), and a position that found nothing looks once more after the batch's
 *     insertions.  Two barriers per batch, no dependent global load: the walk does not depend on the parse;
 *   - K1b (one warp per 16 KiB segment of a block) does the greedy selection: 32 probe positions per step — pairs
 *     (p, p+1) spaced by `step` as in zstd_fast.c:225-229 — lowest matching lane wins (warp ballot); backward
 *     catch-up (:387-391) and forward extension (ZSTD_count, zstd_compress_internal.h:771) are warp-cooperative:
 *     32 x 8 bytes per round, first differing lane found by ballot.  A match may run past its segment's end;
 *   - K1c (one CTA per block) joins the segments: drops what lies under a match that ran over from an earlier segment,
 *     runs the repcode history over the block's sequences and gathers the literal bytes from the input.
 * Everything is deterministic: no result depends on the order in which threads reach an atomic.
 * The bit-exact CPU model of these kernels is oracle/zb_match.c (tests only).
 */
#include "zb_device.cuh"
#include "zb_kernels.h"
#include "zb_merge.cuh"

/* matched bytes starting at rel positions (a, a - offset), never reading at or past `be` */
template <bool DICT>
__device__ __forceinline__ u32 zb_count_fwd(const ZbSeg& sg, u32 a, u32 offset, u32 be, u32 lane)
{
    u32 fwd = 0;
    while (true) {
        u32 const pa = a + fwd + 8u * lane;
        u32 m;
        if (pa + 8u <= be) {
            u64 const x = zb_seg_ld64x<DICT>(sg, pa) ^ zb_seg_ld64x<DICT>(sg, pa - offset);
            m = x ? (u32)((__ffsll((long long)x) - 1) >> 3) : 8u;
        } else {
            m = 0;
            while (pa + m < be && zb_seg_byte<DICT>(sg, pa + m) == zb_seg_byte<DICT>(sg, pa + m - offset)) m++;
        }
        u32 const inc = __ballot_sync(ZB_FULL, m != 8u);
        if (inc == 0) { fwd += 256u; continue; }
        int const f = __ffs((int)inc) - 1;
        fwd += 8u * (u32)f + __shfl_sync(ZB_FULL, m, f);
        return fwd;
    }
}

template <bool DICT>
__device__ __forceinline__ u32 zb_back_coop(const ZbSeg& sg, u32 probe, u32 offset, u32 anchor, u32 lane)
{
    u32 back = 0;
    while (true) {
        u32 const k = back + lane + 1u;                        /* compare bytes probe-k and probe-offset-k */
        bool const ok = (probe >= anchor + k) && (probe >= offset + k)
                     && (zb_seg_byte<DICT>(sg, probe - k) == zb_seg_byte<DICT>(sg, probe - offset - k));
        u32 const okb = __ballot_sync(ZB_FULL, ok);
        u32 const cnt = (okb == ZB_FULL) ? 32u : (u32)(__ffs((int)~okb) - 1);
        back += cnt;
        if (cnt < 32u) return back;
    }
}

/* ------------------------------------------------------------------------------------------------
 * K1a — candidate walk (parse-independent).  One CTA per chunk, table in shared memory.
 * dist[p] = distance from p to its candidate: the latest earlier position that was inserted into p's bucket and has
 * p's tag, 0 if none.  Distances >= 0xFFFF go to the `far` array (dist16 = ZB_FAR).
 * ---------------------------------------------------------------------------------------------- */
/* A table entry is (key + 1) << 11 | tag.  key = walk coordinate x of the position with its offset inside the batch
 * reversed: of all insertions of one batch into a bucket the LOWEST position has the largest key, and every batch beats
 * the batches before it — so one shared-memory atomicMax per insertion arbitrates a batch, whatever the thread order. */
#define ZB_TAG_MASK ((1u << ZB_TAG_BITS) - 1u)
__device__ __forceinline__ u32 zb_walk_key(u32 x) { return x ^ (ZB_BATCH - 1u); }   /* (x | B-1) - (x & B-1); its own inverse */
/* candidate distance of the position at walk coordinate x given the content c its bucket had before x's batch (0 = no
 * candidate).  Every entry then came from an earlier batch (or a dictionary image: coordinates below the frame's), so it
 * lies below x: only emptiness and the tag decide.  Coordinates stay below 2^21, so (key + 1) << TAG_BITS does not wrap. */
__device__ __forceinline__ u32 zb_walk_cand_prior(u32 c, u32 h, u32 x)
{
    u32 const px = zb_walk_key((c >> ZB_TAG_BITS) - 1u);
    return (((c ^ h) & ZB_TAG_MASK) == 0u && c != 0u) ? x - px : 0u;
}

/* which of the P consecutive positions starting at a position whose residue modulo `step` is r0 lie on the insertion
 * pattern (rel % step) < 2, as a bit mask.  step >= 3: the pair that began at or before the first position (bits 0,1
 * for r0 = 0; bit 0 for r0 = 1), then a pair every `step` positions from step - r0 on. */
template <int P>
__device__ __forceinline__ u32 zb_walk_pattern_res(u32 r0, u32 step)
{
    if (step <= 2u) return (1u << P) - 1u;
    u32 m = 3u >> (r0 < 2u ? r0 : 2u);
    u32 nxt = step - r0;
#pragma unroll
    for (int k = 0; k < (P + 2) / 3; k++) {                       /* at most ceil(P / 3) further pairs start inside P positions */
        m |= 3u << (nxt < 31u ? nxt : 31u);
        nxt += step;
    }
    return m & ((1u << P) - 1u);
}
/* residue of rel0 modulo step (rel0 < 2^22, step < 2^14: the float quotient is exact up to +-1, fixed below) */
__device__ __forceinline__ u32 zb_walk_residue(u32 rel0, u32 step)
{
    u32 const q = (u32)__fdividef((float)rel0, (float)step);
    int r = (int)rel0 - (int)(q * step);
    if (r < 0) r += (int)step; else if (r >= (int)step) r -= (int)step;
    return (u32)r;
}

/* One batch of the walk for one thread: P consecutive positions from walk coordinate xa.
 * INTERIOR: every position of the batch is walked, lies in the frame's own bytes and has its 8 bytes readable: no
 * activity predicates, bytes come from the words prefetched in wrd[].
 * Returns whether any position of the CTA found a candidate in phase A (the barrier between A and B carries the OR).
 * The walk is bound by instruction issue, not by memory (DESIGN.md section 2): the insertions are predicated, a batch
 * without output (the history that primes the table) stops after its insertions, and the far distances are handled
 * behind one warp vote. */
#define ZB_WALK_NWR(P) ((P) == 1 ? 2 : ((P) + 7 + 3) / 4)        /* realigned words that hold a thread's P + 7 bytes */
template <int MLS, int P, bool INTERIOR>
__device__ __forceinline__ bool zb_walk_batch(u32* __restrict__ table, u32 xa, const u32 (&wrd)[ZB_WALK_NWR(P)], u32 pat,
                                              u32 N, u32 shift, u32 D, u32 total, u32 xLow, u32 xEnd,
                                              const u8* fbase, const u8* dbase, bool output, u16* __restrict__ distRow, u32* __restrict__ farRow)
{
    u32 h[P], bkt[P], dOld[P];
    bool act[P];
    /* ---- A: hash, read the bucket ---- */
    {   u32 const rel0 = xa - shift;
        bool const slow = !INTERIOR && ((xa < xLow) || (D != 0u && rel0 < D && rel0 + P + 7u > D) || (rel0 + P + 7u > total));
#pragma unroll
        for (int i = 0; i < P; i++) {
            u32 const x = xa + (u32)i, rel = x - shift;
            act[i] = INTERIOR ? true : ((x >= xLow) && (rel + 8u <= total) && !(rel < D && rel + 8u > D));
            u32 lo, hi;
            if (slow) { u64 const v = act[i] ? zb_ld64u((rel < D ? dbase : fbase) + rel) : 0ull; lo = (u32)v; hi = (u32)(v >> 32); }
            else {
                constexpr int NWR = ZB_WALK_NWR(P);
                int const wi = i >> 2; u32 const sh = 8u * (u32)(i & 3);
                int const w2 = wi + 2 < NWR ? wi + 2 : NWR - 1;           /* only read when i & 3: then wi + 2 < NWR */
                lo = (i & 3) ? __funnelshift_r(wrd[wi], wrd[wi + 1], sh) : wrd[wi];
                hi = (i & 3) ? __funnelshift_r(wrd[wi + 1], wrd[w2], sh) : wrd[wi + 1];
            }
            h[i] = zb_hash32<MLS>(lo, hi);
            bkt[i] = __umulhi(h[i], N);
            dOld[i] = zb_walk_cand_prior(act[i] ? table[bkt[i]] : 0u, h[i], x);
        }
    }
    u32 anyOld = 0;
#pragma unroll
    for (int i = 0; i < P; i++) anyOld |= dOld[i];
    bool const anyHit = __syncthreads_or(anyOld != 0u) != 0;
    /* ---- B: insertions: positions that are walked, found no candidate and lie on the pattern.
     * A thread's first coordinate is a multiple of P, so the reversed in-batch offsets of its positions count down from
     * position 0's: key(xa + i) = key(xa) - i; an entry is (Y1 - i) << TAG_BITS | tag with Y1 = key(xa) + 1.
     * Every position issues its atomicMax, one that does not insert with 0 (no effect on a maximum): ptxas wraps a
     * conditional or predicated shared atomic in a divergence region of its own, which costs more issue slots than the
     * select and the extra shared-memory traffic ---- */
    u32 const Y1s = (zb_walk_key(xa) + 1u) << ZB_TAG_BITS;
    u32 e[P];
#pragma unroll
    for (int i = 0; i < P; i++) {
        e[i] = (Y1s - ((u32)i << ZB_TAG_BITS)) | (h[i] & ZB_TAG_MASK);
        atomicMax(&table[bkt[i]], (act[i] && dOld[i] == 0u && ((pat >> i) & 1u)) ? e[i] : 0u);
    }
    __syncthreads();                                              /* also orders these insertions before the next batch's A */
    if (!output) return anyHit;                                   /* CTA-uniform: priming batches only fill the table */
    /* ---- C: second look.  A position without a candidate can only have gained one from this batch's insertions (its
     * bucket held no entry with its tag before, and what was there came from earlier batches).  With equal tags the
     * bucket's entry minus the position's own is the key difference << TAG_BITS, and inside one batch the key difference
     * is the distance; unequal tags leave low bits that the rotation moves to the top.  So the rotated difference is the
     * distance exactly when it is below ZB_BATCH: an entry of an earlier batch has the smaller key, and its difference
     * wraps to 2^21 minus the keys' spread, far above ZB_BATCH (coordinates stay below 2^20).  A position that found a
     * candidate in A never finds one here: every position of its bucket with its tag found the same entry and did not
     * insert, so the look needs no test of dOld ---- */
    u32 d[P], orD = 0;
#pragma unroll
    for (int i = 0; i < P; i++) {
        u32 const c = table[bkt[i]] - e[i];
        u32 const r = __funnelshift_r(c, c, ZB_TAG_BITS);
        d[i] = (act[i] && r < ZB_BATCH) ? r : dOld[i];
        orD |= d[i];
    }
    /* ---- output.  Distances >= ZB_FAR are rare: one vote (the OR of a thread's distances is at least their maximum)
     * decides whether the warp looks at them one by one ---- */
    bool const mine = INTERIOR || xa < xEnd;
    if (__any_sync(ZB_FULL, mine && orD >= ZB_FAR)) {
#pragma unroll
        for (int i = 0; i < P; i++) if (d[i] >= ZB_FAR) { if (mine && (INTERIOR || xa + (u32)i < xEnd)) farRow[i] = d[i]; d[i] = ZB_FAR; }
    }
    if (!mine) return anyHit;
    auto pk = [&](int i) { return __byte_perm(d[i], d[i + 1], 0x5410); };   /* d[i] | d[i + 1] << 16: every d <= ZB_FAR here */
    bool vec = false;
    if constexpr (P == 16) { if (INTERIOR || xa + 16u <= xEnd) { uint4* const o4 = reinterpret_cast<uint4*>(distRow);
                                 o4[0] = make_uint4(pk(0), pk(2), pk(4), pk(6)); o4[1] = make_uint4(pk(8), pk(10), pk(12), pk(14)); vec = true; } }
    if constexpr (P == 8) { if (INTERIOR || xa + 8u <= xEnd) { *reinterpret_cast<uint4*>(distRow) = make_uint4(pk(0), pk(2), pk(4), pk(6)); vec = true; } }
    if constexpr (P == 4) { if (INTERIOR || xa + 4u <= xEnd) { *reinterpret_cast<uint2*>(distRow) = make_uint2(pk(0), pk(2)); vec = true; } }
    if constexpr (P == 2) { if (INTERIOR || xa + 2u <= xEnd) { *reinterpret_cast<u32*>(distRow) = pk(0); vec = true; } }
    if (!vec) {
#pragma unroll
        for (int i = 0; i < P; i++) if (xa + (u32)i < xEnd) distRow[i] = (u16)d[i];
    }
    return anyHit;
}

/* P consecutive positions per thread, ZB_BATCH / P threads per CTA.  Per batch:
 *   A  every position hashes its 8 bytes and reads its bucket (the table as the previous batch left it);
 *   B  positions that found no candidate and lie on the insertion pattern atomicMax their entry into the bucket;
 *   C  positions that found nothing in A look again: the batch's lowest insertion into their bucket may serve them.
 * Two barriers per batch (A|B, which also tells every thread whether the batch saw a hit, and B|C); C of one batch
 * and A of the next share a region.  The input bytes of a batch are loaded two batches ahead. */
#ifndef WALK_STEADY
#define WALK_STEADY 1            /* development switch: 0 = every batch takes the general path */
#endif
#ifndef WALK_P_SMALL
#define WALK_P_SMALL 8           /* positions per thread for tables <= 56 KiB: 128 threads per CTA (on the H100 the walk takes 2.54 ms per GiB of config 2 with 8, 2.80 with 4, 2.81 with 16; development knob: tools/build_variant.sh) */
#endif
#ifndef WALK_P_MID
#define WALK_P_MID 4             /* tables of 56 .. 113 KiB: two CTAs per SM (walk on the H100, config 4: 8.16 ms with 4 positions per thread, 9.25 with 8, 8.83 with 2 before the walk's instruction cut) */
#endif
#ifndef WALK_MINB_SMALL
#define WALK_MINB_SMALL 4        /* CTAs per SM the register allocation of that variant leaves room for */
#endif
template <int MLS, int P>
__global__ void __launch_bounds__(ZB_BATCH / P, P == WALK_P_SMALL ? WALK_MINB_SMALL : 1)
zb_walk_kernel(const u8* __restrict__ src, const ZbDictSlot* __restrict__ dicts, const ZbChunk* __restrict__ chunks, u32 insStep, u32 N, ZbStrides sd,
               u32 slotFirstBlock, u16* __restrict__ dist, u32* __restrict__ far, u32 imageOff, bool buildImage)
{
    constexpr u32 THREADS = ZB_BATCH / P;
    extern __shared__ __align__(16) u32 table[];
    u32 const t = threadIdx.x;
    ZbChunk const cd = chunks[blockIdx.x];
    u32 const D = cd.dictLen;                                     /* rel position of the frame's first byte when a dictionary is in front */
    /* the frame's dictionary (first chunk only): its tail's end and the table image of this launch's parameters (buildImage:
     * the image this CTA writes) */
    const u8* dictEnd = nullptr; const u32* imageIn = nullptr;
    if (D) { ZbDictSlot const& ds = dicts[cd.dictSlot]; dictEnd = ds.end; imageIn = ds.image ? ds.image + imageOff : nullptr; }
    u32 const H = cd.histLen;                                     /* rel position of the chunk's first byte */
    u32 const total = buildImage ? D : H + cd.size;               /* rel positions [0, total) are walked; no read at or past total */
    bool const fromImage = imageIn != nullptr && D != 0u && !buildImage;
    /* walk coordinate x = rel + shift: batch borders (frame positions that are multiples of the batch; dictionary
     * positions count backwards from the frame start) are the multiples of ZB_BATCH in x */
    u32 const shift = (ZB_BATCH - (D % ZB_BATCH)) % ZB_BATCH;
    const u8* const fbase = src + cd.srcOff - H;                  /* fbase + rel = the byte's address for rel >= D */
    const u8* const dbase = dictEnd - D;                          /* same for rel < D */

    if (fromImage) for (u32 i = t; i < N; i += THREADS) table[i] = __ldg(imageIn + i);
    else           for (u32 i = t; i < N; i += THREADS) table[i] = 0u;
    __syncthreads();

    u32 const xEnd = total + shift;
    u32 const xLow = (fromImage ? D : 0u) + shift;                /* first walked coordinate */
    u32 x0 = xLow & ~(ZB_BATCH - 1u);                             /* border of the first batch */
    /* interior batches: completely walked, completely in the frame's own bytes, all 8-byte reads inside [.., total) */
    u32 const xIntLo = ((D + shift) > xLow ? (D + shift) : xLow);
    u32 const xIntLoB = (xIntLo + ZB_BATCH - 1u) & ~(ZB_BATCH - 1u);
    /* a thread's P + 7 bytes lie in NW aligned words whatever its address modulo 4; the interior loads all NW of them */
    constexpr u32 NW = (P + 7u + 3u + 3u) / 4u;
    constexpr int NWR = ZB_WALK_NWR(P);
    u32 const xIntHi = xEnd >= (ZB_BATCH + 4u * NW) ? (xEnd + P - 4u * NW) & ~(ZB_BATCH - 1u) : 0u;     /* batches [x0, x0 + B) with x0 + B <= xIntHi are interior */

    /* the aligned words that hold the P + 7 bytes of a thread's positions, and the shift that realigns them: the words are
     * only touched (realigned) by the batch that uses them, two batches after the loads went out */
    auto fetch = [&](u32 xb, u32 (&a)[NW], u32& sh) {
        u32 const xa = xb + P * t;                                /* first coordinate of the thread */
#pragma unroll
        for (u32 k = 0; k < NW; k++) a[k] = 0u;
        sh = 0u;
        if (xb >= xIntLoB && xb + ZB_BATCH <= xIntHi) {           /* interior: no guards */
            const u8* const ad = fbase + (xa - shift);
            const u32* const p = reinterpret_cast<const u32*>((uintptr_t)ad & ~(uintptr_t)3);
            sh = ((u32)(uintptr_t)ad & 3u) * 8u;
#pragma unroll
            for (u32 k = 0; k < NW; k++) a[k] = __ldg(p + k);
            return;
        }
        if (xa + P <= xLow || xa >= xEnd) return;                 /* nothing of mine is walked */
        u32 const rel = xa - shift;
        bool const slow = (xa < xLow) || (D != 0u && rel < D && rel + P + 7u > D) || (rel + P + 7u > total);
        if (slow) return;                                         /* assembled byte-wise in the batch */
        const u8* const ad = (rel < D ? dbase : fbase) + rel;
        const u32* const p = reinterpret_cast<const u32*>((uintptr_t)ad & ~(uintptr_t)3);
        u32 const al = (u32)(uintptr_t)ad & 3u;
        sh = al * 8u;
        /* rel + P + 7 <= limit: a word is only touched when it holds one of the thread's P + 7 bytes */
#pragma unroll
        for (u32 k = 0; k < NW; k++) a[k] = (al + P + 7u > 4u * k) ? __ldg(p + k) : 0u;
    };
    u32 rawA[NW], rawB[NW], shA, shB;                             /* bytes of the next batch and of the one after it */
    fetch(x0, rawA, shA);
    fetch(x0 + ZB_BATCH, rawB, shB);
    u32 const blockMask = (1u << cd.blockLog) - 1u;
    /* insertion pattern: the residue of the thread's first position modulo insStep follows the walk by addition; only a
     * batch whose step was raised by the acceleration pays for a division */
    u32 const stepInc = ZB_BATCH % insStep;
    u32 r0 = (x0 + P * t + insStep * ZB_BATCH - shift) % insStep;
    u32 li = shift;                                               /* coordinate the acceleration counts from: the walk's start, then the end of the last batch with a hit */
    /* one batch: its words are realigned, the register set is refilled at once for the batch two ahead (no copies between
     * the sets: the loop below alternates them), then the three phases run */
    auto doBatch = [&](u32 (&raw)[NW], u32& sh) {
        u32 const xa = x0 + P * t;
        u32 cur[NWR];
#pragma unroll
        for (int k = 0; k < NWR; k++) cur[k] = __funnelshift_r(raw[k], (u32)k + 1u < NW ? raw[(u32)k + 1u < NW ? k + 1 : k] : 0u, sh);
        fetch(x0 + 2u * ZB_BATCH, raw, sh);                       /* in flight across two batches' barriers */
        if (D != 0u && x0 >= D + shift && li < D + shift) li = D + shift;   /* the frame starts with a fresh acceleration state behind a dictionary */
        u32 const sWalk = x0 > xLow ? x0 : xLow;                  /* first walked coordinate of the batch */
        u32 const step = insStep + ((sWalk - li) >> 7);
        u32 const pat = zb_walk_pattern_res<P>(step == insStep ? r0 : zb_walk_residue(xa - shift, step), step);
        bool const output = !buildImage && x0 >= H + shift;       /* H + shift is a batch border: the whole batch lies in the history or in the chunk */
        /* a batch never straddles two blocks (block sizes are multiples of the batch, or the frame is a single block) */
        u32 const qb0 = x0 - shift - H;                           /* offset of the batch in the chunk when output */
        size_t const idx = output ? (size_t)(cd.firstBlock - slotFirstBlock + (qb0 >> cd.blockLog)) * sd.dist + (qb0 & blockMask) + P * t : 0;
        bool hit;
        if (x0 >= xIntLoB && x0 + ZB_BATCH <= xIntHi)
            hit = zb_walk_batch<MLS, P, true>(table, xa, cur, pat, N, shift, D, total, xLow, xEnd, fbase, dbase, output, dist + idx, far + idx);
        else
            hit = zb_walk_batch<MLS, P, false>(table, xa, cur, pat, N, shift, D, total, xLow, xEnd, fbase, dbase, output, dist + idx, far + idx);
        if (hit) li = x0 + ZB_BATCH;
        r0 += stepInc; if (r0 >= insStep) r0 -= insStep;
        x0 += ZB_BATCH;
    };
    /* the same batch in the walk's steady state — this batch, the one whose words are requested and everything between are
     * interior batches of the frame's own bytes: none of doBatch's case distinctions apply, the words two batches ahead sit
     * 2 * ZB_BATCH bytes behind this batch's, the output row moves with the walk.  Same results as doBatch, about half
     * the instructions around the three phases. */
    const u8* const tbase = fbase + P * t - shift;                /* tbase + x0 = address of the thread's first byte in the batch at x0 */
    u16* const distT = dist + P * t;
    u32* const farT = far + P * t;
    auto steadyBatch = [&](u32 (&raw)[NW], u32 const sh) {
        u32 const xa = x0 + P * t;
        u32 cur[NWR];
#pragma unroll
        for (int k = 0; k < NWR; k++) cur[k] = __funnelshift_r(raw[k], (u32)k + 1u < NW ? raw[(u32)k + 1u < NW ? k + 1 : k] : 0u, sh);
        {   const u32* const pw = reinterpret_cast<const u32*>((uintptr_t)(tbase + x0 + 2u * ZB_BATCH) & ~(uintptr_t)3);
#pragma unroll
            for (u32 k = 0; k < NW; k++) raw[k] = __ldg(pw + k);  /* the alignment (sh) is the same in every batch: batches are 1024 bytes apart */
        }
        u32 const step = insStep + ((x0 - li) >> 7);
        u32 const pat = zb_walk_pattern_res<P>(step == insStep ? r0 : zb_walk_residue(xa - shift, step), step);
        bool const output = !buildImage && x0 >= H + shift;
        u32 const qb0 = x0 - shift - H;
        size_t const row = output ? (size_t)(cd.firstBlock - slotFirstBlock + (qb0 >> cd.blockLog)) * sd.dist + (qb0 & blockMask) : 0;
        if (zb_walk_batch<MLS, P, true>(table, xa, cur, pat, N, shift, D, total, xLow, xEnd, fbase, dbase, output, distT + row, farT + row)) li = x0 + ZB_BATCH;
        r0 += stepInc; if (r0 >= insStep) r0 -= insStep;
        x0 += ZB_BATCH;
    };
    while (x0 < xEnd) {
        /* pairs of steady-state batches (the two register sets keep their turns) */
        if (WALK_STEADY && x0 >= xIntLoB && x0 + 4u * ZB_BATCH <= xIntHi) {
            if (D != 0u && li < D + shift) li = D + shift;           /* as in doBatch: x0 >= xIntLoB >= D + shift */
            do { steadyBatch(rawA, shA); steadyBatch(rawB, shB); } while (x0 + 4u * ZB_BATCH <= xIntHi);
        }
        doBatch(rawA, shA);
        if (x0 >= xEnd) break;
        doBatch(rawB, shB);
    }
    if (buildImage) {                                             /* the image's address is read again here: not live through the walk */
        u32* const imageOut = const_cast<u32*>(dicts[chunks[blockIdx.x].dictSlot].image) + imageOff;
        __syncthreads(); for (u32 i = t; i < N; i += THREADS) imageOut[i] = table[i];
    }
}

/* ------------------------------------------------------------------------------------------------
 * K1b — greedy selection + match extension.  One warp per 16 KiB segment, no shared memory (occupancy is
 * register-bound, so the L2 latency of the candidate checks is hidden by other warps).  Per step 32 probe
 * positions: pairs (p, p+1) spaced by `step` (zstd_fast.c:225-229, step acceleration :234,:342-347).  Hit
 * priority per lane: repcode-2 (lane 0, directly after a match, :410-420), repcode-1 (:281-297), table candidate
 * with 4-byte check (:102-141).  Lowest lane wins.  A segment owns the match starts inside it; a match may run
 * past the segment's end up to the block's end (the merge kernel resolves what that covers).
 * ---------------------------------------------------------------------------------------------- */
#ifndef PARSE_WARPS
#define PARSE_WARPS 8            /* = ZB_PARSE_SEGS: the eight segments of a full block share a CTA */
#endif
#ifndef PARSE_MIN_CTAS
#define PARSE_MIN_CTAS 6         /* 48 warps per SM at 40 registers */
#endif
__device__ __forceinline__ u32 zb_dist_at(const u16* __restrict__ d16, const u32* __restrict__ far, u32 i)
{
    u32 const d = d16[i];
    return d == ZB_FAR ? far[i] : d;
}

/* zb_seg_ld64x for the hit path: the same three words, the third addressed as the word of the last byte, (p + 7) & ~3,
 * which takes three instructions where choosing between the second and third word after p takes seven */
template <bool DICT>
__device__ __forceinline__ u64 zb_hit_ld64(const ZbSeg& sg, u32 rel)
{
    if (DICT && rel < sg.split && rel + 12u > sg.split) return zb_seg_ld64x<true>(sg, rel);
    const u8* const p = zb_seg_ptr<DICT>(sg, rel);
    const u32* const w = (const u32*)((uintptr_t)p & ~(uintptr_t)3);
    u32 const sh = ((u32)(uintptr_t)p & 3u) * 8u;
    u32 const x = __ldg(w), y = __ldg(w + 1), z = __ldg((const u32*)((uintptr_t)(p + 7) & ~(uintptr_t)3));
    return ((u64)__funnelshift_r(y, z, sh) << 32) | __funnelshift_r(x, y, sh);
}

/* the 4 bytes at rel and the 4 bytes at rel + 1: the two aligned words around rel hold these 5 bytes whatever rel's
 * alignment (the second funnel shift clamps at 32: at rel % 4 == 3 the bytes at rel + 1 are the second word).  A window
 * that straddles the dictionary / frame border is read byte by byte */
template <bool DICT>
__device__ __forceinline__ void zb_ld4x2(const ZbSeg& sg, u32 rel, u32& at, u32& at1)
{
    if (DICT && rel < sg.split && rel + 5u > sg.split) {
        u64 v = 0;
#pragma unroll
        for (u32 i = 0; i < 5u; i++) v |= (u64)zb_seg_byte<true>(sg, rel + i) << (8u * i);
        at = (u32)v; at1 = (u32)(v >> 8);
        return;
    }
    const u8* const p = zb_seg_ptr<DICT>(sg, rel);
    const u32* const w = (const u32*)((uintptr_t)p & ~(uintptr_t)3);
    u32 const sh = ((u32)(uintptr_t)p & 3u) * 8u;
    u32 const x = __ldg(w), y = __ldg(w + 1);
    at = __funnelshift_r(x, y, sh);
    at1 = __funnelshift_rc(x, y, sh + 8u);
}

template <bool DICT>
__global__ void __launch_bounds__(32 * PARSE_WARPS, DICT ? (40 / PARSE_WARPS) : PARSE_MIN_CTAS)
zb_parse_kernel(const u8* __restrict__ src, const ZbDictSlot* __restrict__ dicts, const ZbBlock* __restrict__ blocks, u32 nbBlocks, ZbParams prm, ZbStrides sd,
                const u16* __restrict__ dist, const u32* __restrict__ far, u64* __restrict__ seqs, ZbBlockMeta* __restrict__ meta, ZbSegMeta* __restrict__ segmeta)
{
    u32 const lane = threadIdx.x & 31u;
    u32 const g = blockIdx.x * PARSE_WARPS + (threadIdx.x >> 5);  /* one warp per segment: the warps of a CTA share a block's history in L1/L2 */
    u32 const segs = zb_segsPerRow(sd);                            /* segments of the call's largest block (1 for calls of short frames) */
    u32 const b = g / segs, k = g % segs;
    if (b >= nbBlocks) return;
    ZbBlock const bd = blocks[b];
    const u16* const mydist = dist + (size_t)b * sd.dist;
    const u32* const myfar = far + (size_t)b * sd.dist;
    const u8* const base = src + bd.srcOff - bd.histLen;          /* base + rel addresses the frame's own bytes */
    u32 const bs = bd.histLen, blockEnd = bd.histLen + bd.size;
    ZbSeg sg; sg.hi = base; sg.lo = base; sg.split = 0;
    if (DICT && (bd.flags & ZB_FLAG_DICT)) { sg.lo = dicts[bd.dictSlot].end - bd.dictLen; sg.split = bd.dictLen; }   /* oldest history = dictionary tail */

    if (bd.size < 7u) {                                        /* zstd_compress.c:3216 */
        if (lane == 0 && k == 0) {
            ZbBlockMeta m; m.nbSeq = 0; m.litSize = bd.size; m.litSecSize = 0; m.bodySize = bd.size;
            m.type = ZB_BT_RAW; m.forceRaw = 1; m.rleByte = 0; m.pad = 0;
            meta[b] = m;
        }
        return;
    }
    u32 const ss = bs + k * ZB_PARSE_SEG;                      /* this warp owns the match starts in [ss, se) */
    if (ss >= blockEnd) {
        if (lane == 0) { ZbSegMeta z; z.nbSeq = 0; z.pad[0] = z.pad[1] = z.pad[2] = 0; segmeta[(size_t)b * segs + k] = z; }
        return;
    }
    u32 const se = min(ss + ZB_PARSE_SEG, blockEnd);
    u32 const be = blockEnd;
    int const last = min((int)se - 1, (int)be - 8);            /* the last position probed: p < se and p + 8 <= be */

    u32 ip = ss, anchor = ss;                                  /* the search restarts at the anchor: it is searchStart too */
    u32 rep1 = 0, rep2 = 0, nbSeq = 0;
    if (dicts && (bd.flags & ZB_FLAG_FIRST) && k == 0u) { rep1 = dicts[bd.dictSlot].startRep[0]; rep2 = dicts[bd.dictSlot].startRep[1]; }   /* a zstd-format dictionary's repcodes, zstd_compress.c:5054-5056 */

    /* the 4 bytes at rel position x; x + 8 <= be */
    auto ld4 = [&](u32 x) { return DICT ? (u32)zb_seg_ld64x<DICT>(sg, x) : zb_ld32w2(sg.hi + x); };
    while ((int)ip <= last) {
        /* two steps of the rule per iteration, one pair (p, p+1) per lane: lanes 0..15 hold the step at ip, lanes 16..31
         * the step the rule takes next when the first finds nothing, at ip2 with its own acceleration.  Pairs never
         * overlap (stepSize >= 2, checked at the launch), so position order is lane order, then p before p+1 */
        u32 const step = prm.stepSize + ((ip - anchor) >> 7);                /* kSearchStrength = 8 */
        u32 const ip2 = ip + 16u * step;
        u32 const step2 = prm.stepSize + ((ip2 - anchor) >> 7);
        u32 const next = ip2 + 16u * step2;                  /* where the search goes on when no position hits */
        u32 const p = lane < 16u ? ip + lane * step : ip2 + (lane - 16u) * step2;
        bool const act = (int)p <= last, act1 = (int)p < last;
        u32 const pp = act ? p : ip;                         /* a position every lane may load from (ip + 8 <= be) */
        /* one round trip per iteration: the candidate pair, the current window and both repcode windows are independent
         * loads and all go out before the first is looked at.  One window at p gives the 4 bytes at p and at p+1; one at
         * p - rep1 gives both repcode-1 compares (read at 0 where only p+1 reaches the history: p + 1 == rep1).  dist[]
         * only holds tag-verified candidates, so a step needs no random load: every window is contiguous across lanes.
         * Whether a table candidate reaches the history is checked when its position is tried, below: a far distance
         * (ZB_FAR) has its 32-bit value fetched only then.  pp + 1 < be: both entries lie in the block's row */
        const u16* const dp = mydist + (pp - bs);
        u32 const d0 = dp[0], d1 = dp[1];
        u32 const r = pp - rep1;                             /* < pp: rep1 reaches the history from p (rep1 == 0: none) */
        bool const v3 = (lane == 0u) && (ip == anchor) && (rep2 != 0u);
        bool const v2 = act && r < pp;
        bool const v21 = act1 && r + 1u <= pp;
        u32 cur, cur1, rc, rc1;
        zb_ld4x2<DICT>(sg, pp, cur, cur1);
        zb_ld4x2<DICT>(sg, r < pp ? r : 0u, rc, rc1);
        if (r >= pp) rc1 = rc;
        u32 cur3 = ~cur;
        if (ip == anchor && rep2 != 0u) cur3 = ld4(v3 ? pp - rep2 : pp);      /* warp-uniform condition */
        u32 const hit = (v3 && cur3 == cur) ? 3u : ((v2 && rc == cur) ? 2u : ((act && d0 != 0u) ? 1u : 0u));
        u32 const hit1 = (v21 && rc1 == cur1) ? 2u : ((act1 && d1 != 0u) ? 1u : 0u);
        /* what a lane hands out when one of its positions is tried: type and distance.  A position that drops out clears
         * its own; a lane tries p while hd holds a hit, then p+1 */
        u32 hd = (d0 << 2) | hit, hd1 = (d1 << 2) | hit1;
        u32 tent = __ballot_sync(ZB_FULL, (hit | hit1) != 0u);
        /* lowest position first: the lowest lane with a hit, its p before its p+1.  A table hit (type 1) is only
         * tag-verified by K1a: its bytes are checked while the match is extended; a false positive drops out and the next
         * position is tried — the result is "lowest position whose hit is real", what the oracle computes over its two
         * steps.  So does a table candidate that reaches in front of the history (a position whose repcodes had matched
         * would not be a type-1 hit). */
        u32 probe = 0, wtype = 0, offset = 0, back = 0, fwdFrom4 = 0;
        bool found = false;
        while (tent) {
            u32 const winner = (u32)__ffs((int)tent) - 1u;
            bool const odd = (hd & 3u) == 0u;                /* this lane's next position is p+1 */
            probe = __shfl_sync(ZB_FULL, odd ? p + 1u : p, winner);
            u32 const w = __shfl_sync(ZB_FULL, odd ? hd1 : hd, winner);
            wtype = w & 3u;
            offset = (wtype == 3u) ? rep2 : ((wtype == 2u) ? rep1 : w >> 2);
            /* a position that drops out clears its hit: its lane goes on to its p+1 or leaves the vote */
            auto dropOut = [&]() { if (lane == winner) { if (odd) hd1 = 0u; else hd = 0u; } tent = __ballot_sync(ZB_FULL, ((hd | hd1) & 3u) != 0u); };
            if (wtype == 1u && offset == ZB_FAR) offset = myfar[probe - bs];   /* rare: one more round trip */
            if (probe < offset) { dropOut(); continue; }     /* a table candidate in front of the history (a repcode never is) */
            /* one round trip for the first forward round and the first backward round (zstd_fast.c:387-391) together, in
             * one pair of 8-byte windows per lane.  Lanes 0..30 count forward, 248 bytes: a table hit from the probe itself
             * (its first 4 bytes are not verified yet), a repcode hit from probe + 4.  Lane 31 reads the 8 bytes in front of
             * the probe (fewer where the candidate would leave the history) and counts the catch-up from its top byte down,
             * bit-reversed so that every lane counts equal bytes from its bottom.  Only a catch-up that fills lane 31's
             * window goes on to the cooperative rounds.  A repcode-2 hit sits at the anchor: it has nothing to catch up */
            u32 const a = (wtype == 1u) ? probe : probe + 4u;
            bool const cu = lane == 31u;
            u32 const pa = a + 8u * lane;                 /* forward: this lane's 8 bytes, read at q so that no lane branches */
            u32 const db = min(8u, probe - offset);       /* catch-up bytes lane 31 may read: q - offset stays >= 0 */
            u32 const q = cu ? probe - db : min(pa, be - 8u);   /* (probe + 8 <= be, so q >= probe - db >= offset) */
            u64 const xf = zb_hit_ld64<DICT>(sg, q) ^ zb_hit_ld64<DICT>(sg, q - offset);
            u64 const xs = (cu ? __brevll(xf) : xf) >> (8u * min(cu ? 8u - db : pa - q, 7u));
            u32 const lo = (u32)xs, hi = (u32)(xs >> 32);
            u32 m = (lo ? __clz(__brev(lo)) : 32u + __clz(__brev(hi))) >> 3;          /* equal bytes from the bottom, 8 if all */
            m = min(m, cu ? min(probe - anchor, db) : (pa >= be ? 0u : be - pa));
            u32 const stop = __ballot_sync(ZB_FULL, m != 8u);
            u32 const inc = stop & (ZB_FULL >> 1);
            u32 fwd;
            if (inc == 0u) fwd = 248u + zb_count_fwd<DICT>(sg, a + 248u, offset, be, lane);
            else { int const f = __ffs((int)inc) - 1; fwd = 8u * (u32)f + __shfl_sync(ZB_FULL, m, f); }
            if (wtype == 1u && fwd < 4u) { dropOut(); continue; }           /* tag collision */
            fwdFrom4 = (wtype == 1u) ? fwd - 4u : fwd;
            back = __shfl_sync(ZB_FULL, m, 31);
            if (!(stop >> 31)) back = 8u + zb_back_coop<DICT>(sg, probe - 8u, offset, anchor, lane);
            found = true;
            break;
        }
        if (!found) { ip = next; continue; }
        u32 const ms = probe - back;
        u32 const mlen = back + 4u + fwdFrom4;
        if (wtype == 3u) { u32 const t = rep2; rep2 = rep1; rep1 = t; }
        else if (wtype == 1u) { rep2 = rep1; rep1 = offset; }
        {   u32 bb = b; asm("" : "+r"(bb));                /* the row's address is rebuilt per match: kept, it would spill */
            if (lane == 0) seqs[(size_t)bb * sd.seq + k * (ZB_PARSE_SEG / 4u) + nbSeq] = zb_pack_raw(offset, mlen, ms - bs); }
        nbSeq++;
        ip = ms + mlen; anchor = ip;
    }
    /* b * segs + k = g, recomputed: nothing of the record's address stays live through the loop */
    if (lane == 0) { ZbSegMeta z; z.nbSeq = nbSeq; z.pad[0] = z.pad[1] = z.pad[2] = 0; segmeta[blockIdx.x * PARSE_WARPS + (threadIdx.x >> 5)] = z; }
}

/* ------------------------------------------------------------------------------------------------
 * K1b (doubleFast) — the greedy selection of ZSTD_compressBlock_doubleFast_noDict_generic
 * (zstd_double_fast.c:105-323) over two candidate arrays: distL (8-byte hash) and distS (mls-byte hash).
 * Per probe position p, in the reference's order: repcode-1 at p+1 (:190-195), long match at p
 * (:206-213), short match at p (:222-225) upgraded to the long match at p+1 when longer (:254-271);
 * probes are spaced by `step` (1, +1 per 256 bytes without a match, :131); lowest lane wins; immediate
 * repcode-2 at lane 0 right after a match (:302-316).  Table candidates are tag-verified only: the
 * winning lane's bytes are checked while the match is extended, a false positive drops out.
 * ---------------------------------------------------------------------------------------------- */
template <bool DICT>
__global__ void __launch_bounds__(32 * PARSE_WARPS)
zb_parse_dfast_kernel(const u8* __restrict__ src, const ZbDictSlot* __restrict__ dicts, const ZbBlock* __restrict__ blocks, u32 nbBlocks, ZbParams prm, ZbStrides sd,
                      const u16* __restrict__ distLong, const u32* __restrict__ farLong, const u16* __restrict__ distShort, const u32* __restrict__ farShort,
                      u64* __restrict__ seqs, ZbBlockMeta* __restrict__ meta, ZbSegMeta* __restrict__ segmeta)
{
    u32 const lane = threadIdx.x & 31u;
    u32 const g = blockIdx.x * PARSE_WARPS + (threadIdx.x >> 5);  /* one warp per segment, as in zb_parse_kernel */
    u32 const segs = zb_segsPerRow(sd);
    u32 const b = g / segs, k = g % segs;
    if (b >= nbBlocks) return;
    ZbBlock const bd = blocks[b];
    u64* const myseq = seqs + (size_t)b * sd.seq + (size_t)k * (ZB_PARSE_SEG / 4u);
    const u16* const dLp = distLong + (size_t)b * sd.dist;
    const u32* const fLp = farLong + (size_t)b * sd.dist;
    const u16* const dSp = distShort + (size_t)b * sd.dist;
    const u32* const fSp = farShort + (size_t)b * sd.dist;
    const u8* const base = src + bd.srcOff - bd.histLen;
    u32 const bs = bd.histLen, blockEnd = bd.histLen + bd.size;
    ZbSeg sg; sg.hi = base; sg.lo = base; sg.split = 0;
    if (DICT && (bd.flags & ZB_FLAG_DICT)) { sg.lo = dicts[bd.dictSlot].end - bd.dictLen; sg.split = bd.dictLen; }

    if (bd.size < 7u) {                                        /* zstd_compress.c:3216 */
        if (lane == 0 && k == 0) {
            ZbBlockMeta m; m.nbSeq = 0; m.litSize = bd.size; m.litSecSize = 0; m.bodySize = bd.size;
            m.type = ZB_BT_RAW; m.forceRaw = 1; m.rleByte = 0; m.pad = 0;
            meta[b] = m;
        }
        return;
    }
    u32 const ss = bs + k * ZB_PARSE_SEG;
    if (ss >= blockEnd) {
        if (lane == 0) { ZbSegMeta z; z.nbSeq = 0; z.pad[0] = z.pad[1] = z.pad[2] = 0; segmeta[(size_t)b * segs + k] = z; }
        return;
    }
    u32 const se = min(ss + ZB_PARSE_SEG, blockEnd);
    u32 const be = blockEnd;
    u32 ip = ss, anchor = ss, searchStart = ss;
    u32 rep1 = 0, rep2 = 0, nbSeq = 0;
    if (dicts && (bd.flags & ZB_FLAG_FIRST) && k == 0u) { rep1 = dicts[bd.dictSlot].startRep[0]; rep2 = dicts[bd.dictSlot].startRep[1]; }

    while (ip < se && ip + 9u <= be) {                        /* a lane reads 8 bytes at p and at p+1 */
        u32 const step = 1u + ((ip - searchStart) >> 8);                     /* kStepIncr = 1 << kSearchStrength */
        u32 const p = ip + lane * step;
        bool const act = (p < se) && (p + 9u <= be);
        u32 const pp = act ? p : ip;
        u32 dL = act ? zb_dist_at(dLp, fLp, pp - bs) : 0u;
        u32 dS = act ? zb_dist_at(dSp, fSp, pp - bs) : 0u;
        u32 dL1 = act ? zb_dist_at(dLp, fLp, pp + 1u - bs) : 0u;
        if (dL > pp) dL = 0u;                                  /* reaches past the visible history (window) */
        if (dS > pp) dS = 0u;
        if (dL1 > pp + 1u) dL1 = 0u;
        u64 const w = zb_seg_ld64x<DICT>(sg, pp);                            /* bytes p .. p+7 */
        u32 const cur = (u32)w, cur1 = (u32)(w >> 8);
        bool const v2 = act && rep1 != 0u && (p + 1u >= rep1);
        u32 const r2 = (u32)zb_seg_ld64x<DICT>(sg, v2 ? pp + 1u - rep1 : pp);
        u32 r3 = ~cur;
        bool const v3 = (lane == 0u) && (ip == anchor) && (rep2 != 0u);
        if (ip == anchor && rep2 != 0u) r3 = (u32)zb_seg_ld64x<DICT>(sg, v3 ? pp - rep2 : pp);
        /* 3 repcode-2, 2 repcode-1 (at p+1), 1 long candidate, 4 short candidate */
        u32 hit = (v3 && r3 == cur) ? 3u : ((v2 && r2 == cur1) ? 2u : (dL ? 1u : (dS ? 4u : 0u)));
        u32 tent = __ballot_sync(ZB_FULL, hit != 0u);
        u32 ms = 0, offset = 0, mlen = 0, wtype = 0;
        bool found = false;
        while (tent) {
            int const winner = __ffs((int)tent) - 1;
            u32 const probe = __shfl_sync(ZB_FULL, p, winner);
            wtype = __shfl_sync(ZB_FULL, hit, winner);
            u32 const wL = __shfl_sync(ZB_FULL, dL, winner), wS = __shfl_sync(ZB_FULL, dS, winner), wL1 = __shfl_sync(ZB_FULL, dL1, winner);
            if (wtype == 3u) { ms = probe; offset = rep2; mlen = 4u + zb_count_fwd<DICT>(sg, probe + 4u, rep2, be, lane); found = true; break; }
            if (wtype == 2u) { ms = probe + 1u; offset = rep1; mlen = 4u + zb_count_fwd<DICT>(sg, probe + 5u, rep1, be, lane); found = true; break; }
            if (wtype == 1u) {
                u32 const f0 = zb_count_fwd<DICT>(sg, probe, wL, be, lane);
                if (f0 >= 8u) {
                    u32 const back = zb_back_coop<DICT>(sg, probe, wL, anchor, lane);
                    ms = probe - back; offset = wL; mlen = back + f0; found = true; break;
                }
                /* tag collision on the long table: the lane may still have a short candidate */
                if (lane == (u32)winner) hit = dS ? 4u : 0u;
                if (wS == 0u) { tent &= ~(1u << winner); }
                continue;
            }
            /* short candidate */
            {   u32 const f0 = zb_count_fwd<DICT>(sg, probe, wS, be, lane);
                if (f0 < 4u) { tent &= ~(1u << winner); if (lane == (u32)winner) hit = 0u; continue; }
                u32 mp = probe, mo = wS, ml = f0;
                if (wL1) {
                    u32 const f1 = zb_count_fwd<DICT>(sg, probe + 1u, wL1, be, lane);
                    if (f1 >= 8u && f1 > ml) { mp = probe + 1u; mo = wL1; ml = f1; }
                }
                u32 const back = zb_back_coop<DICT>(sg, mp, mo, anchor, lane);
                ms = mp - back; offset = mo; mlen = back + ml; wtype = 1u; found = true; break;
            }
        }
        if (!found) { ip += 32u * step; continue; }
        if (wtype == 3u) { u32 const t = rep2; rep2 = rep1; rep1 = t; }
        else if (wtype == 1u) { rep2 = rep1; rep1 = offset; }
        if (lane == 0) myseq[nbSeq] = zb_pack_raw(offset, mlen, ms - bs);
        nbSeq++;
        ip = ms + mlen; anchor = ip; searchStart = ip;
    }
    if (lane == 0) { ZbSegMeta z; z.nbSeq = nbSeq; z.pad[0] = z.pad[1] = z.pad[2] = 0; segmeta[(size_t)b * segs + k] = z; }
}

/* ------------------------------------------------------------------------------------------------
 * K1c — joins a block's segments, assigns repcodes, materialises the literals.
 * `cur` = first byte of the block not yet covered by a sequence.  A raw sequence that ends at or before `cur` lies
 * under a match that ran over from an earlier segment and is dropped; one that straddles `cur` keeps its tail when
 * that is at least 3 bytes (MINMATCH, zstd_internal.h:102); the others take their literals from `cur`.
 * The repcode history (ZSTD_storeSeq / ZSTD_updateRep, zstd_compress_internal.h:671-760) then runs over the whole
 * block: it starts as {1,4,8} (or the dictionary's) in a frame's first block and unknown in every other block.
 * ---------------------------------------------------------------------------------------------- */
struct ZbRepHist { u32 r1, r2, r3; };
__device__ __forceinline__ u32 zb_rep_code(ZbRepHist& h, u32 off, u32 ll)
{
    u32 code;
    if (ll > 0u) {
        if (off == h.r1) return 1u;
        if (off == h.r2) { code = 2u; h.r2 = h.r1; h.r1 = off; return code; }
        if (off == h.r3) { code = 3u; h.r3 = h.r2; h.r2 = h.r1; h.r1 = off; return code; }
    } else {
        if (off == h.r2) { code = 1u; h.r2 = h.r1; h.r1 = off; return code; }
        if (off == h.r3) { code = 2u; h.r3 = h.r2; h.r2 = h.r1; h.r1 = off; return code; }
        if (h.r1 > 1u && off == h.r1 - 1u) { code = 3u; h.r3 = h.r2; h.r2 = h.r1; h.r1 = off; return code; }
    }
    h.r3 = h.r2; h.r2 = h.r1; h.r1 = off;
    return off + 3u;
}

#ifndef MERGE_MIN_CTAS
#define MERGE_MIN_CTAS 6           /* 40 registers (parse + merge on the H100: 6.12 ms per GiB of config 2 against 6.22 with 5 and 6.41 with 4) */
#endif
#define SEG_SLOTS (ZB_PARSE_SEG / 4u)

/* block-wide exclusive count of `flag` over the MERGE_THREADS entries of a round: returns the entries before this thread's,
 * *total gets the round's count (wsum: MERGE_THREADS / 32 shared words) */
__device__ __forceinline__ u32 zb_block_excl(bool flag, u32* wsum, u32* total)
{
    u32 const lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    u32 const bal = __ballot_sync(ZB_FULL, flag);
    if (lane == 0u) wsum[warp] = __popc(bal);
    __syncthreads();
    u32 before = __popc(bal & ((1u << lane) - 1u)), t = 0;
    for (u32 w = 0; w < MERGE_THREADS / 32u; w++) { if (w < warp) before += wsum[w]; t += wsum[w]; }
    __syncthreads();
    *total = t;
    return before;
}

/* Overlay of a block's long-distance matches L[0, nL) (zb_pack_ldm, in position order) onto its parse output P[0, nP) (raw,
 * compacted, in position order): an LDM match wins; a parse match that starts under one starts again at its end, one that
 * runs into one is cut at its start, and a parse match shortened this way is kept only with >= 4 bytes left (the parse's
 * shortest match: a block keeps at most size / 4 + 8 sequences).  Output: (offset, litLength, matchLength) triples in
 * out[0, n), returns n.  kp: nP + 1 words of scratch.  oracle/zb_ldm.c (zbo_ldm_overlayBlock) is the same rule, serially. */
__device__ __forceinline__ void zb_ldm_clip(u32 ms, u32 me, const u64* L, u32 nL, u32* ms2, u32* me2, u32* next, bool* kept)
{
    u32 lo = 0, hi = nL;                                          /* lo = LDM matches that start at or before ms */
    while (lo < hi) { u32 const mid = (lo + hi) >> 1; if (ZB_LDM_START(L[mid]) <= ms) lo = mid + 1u; else hi = mid; }
    bool clipped = false;
    if (lo > 0u && ZB_LDM_START(L[lo - 1u]) + ZB_LDM_LEN(L[lo - 1u]) > ms) { ms = ZB_LDM_START(L[lo - 1u]) + ZB_LDM_LEN(L[lo - 1u]); clipped = true; }
    if (lo < nL && ZB_LDM_START(L[lo]) < me) { me = ZB_LDM_START(L[lo]); clipped = true; }
    *ms2 = ms; *me2 = me; *next = lo;
    *kept = me > ms && (!clipped || me - ms >= 4u);
}
__device__ u32 zb_ldm_overlay(const u64* __restrict__ P, u32 nP, const u64* __restrict__ L, u32 nL, u32* __restrict__ kp, u64* __restrict__ out,
                              u32* wsum, u32* sEnd, u32& carry)
{
    u32 const tid = threadIdx.x;
    u32 base = 0;
    for (u32 i0 = 0; i0 < nP; i0 += MERGE_THREADS) {              /* kp[i] = kept parse matches before i */
        u32 const i = i0 + tid;
        u32 ms2, me2, nx; bool kept = false;
        if (i < nP) { u64 const r = P[i]; zb_ldm_clip(ZB_RAW_MS(r), ZB_RAW_MS(r) + ZB_RAW_MLEN(r), L, nL, &ms2, &me2, &nx, &kept); }
        u32 t;
        u32 const before = zb_block_excl(kept, wsum, &t);
        if (i < nP) kp[i] = base + before;
        base += t;
    }
    if (tid == 0) kp[nP] = base;
    __syncthreads();
    for (u32 i = tid; i < nP; i += MERGE_THREADS) {               /* parse matches and LDM matches to their places, absolute */
        u64 const r = P[i];
        u32 ms2, me2, nx; bool kept;
        zb_ldm_clip(ZB_RAW_MS(r), ZB_RAW_MS(r) + ZB_RAW_MLEN(r), L, nL, &ms2, &me2, &nx, &kept);
        if (kept) out[kp[i] + nx] = zb_pack_ldm(ms2, me2 - ms2, ZB_RAW_OFF(r));
    }
    for (u32 k = tid; k < nL; k += MERGE_THREADS) {               /* kept parse matches before it = those that start before it */
        u32 const s = ZB_LDM_START(L[k]);
        u32 lo = 0, hi = nP;
        while (lo < hi) { u32 const mid = (lo + hi) >> 1; if (ZB_RAW_MS(P[mid]) < s) lo = mid + 1u; else hi = mid; }
        out[k + kp[lo]] = L[k];
    }
    u32 const n = base + nL;
    __syncthreads();
    if (tid == 0) carry = 0;
    for (u32 o0 = 0; o0 < n; o0 += MERGE_THREADS) {               /* absolute -> (offset, litLength, matchLength) */
        u32 const o = o0 + tid;
        u64 const m = o < n ? out[o] : 0ull;
        sEnd[tid] = ZB_LDM_START(m) + ZB_LDM_LEN(m);
        __syncthreads();
        u32 const prevEnd = tid ? sEnd[tid - 1u] : carry;
        if (o < n) out[o] = zb_pack_seq(ZB_LDM_OFF(m), ZB_LDM_START(m) - prevEnd, ZB_LDM_LEN(m));
        __syncthreads();
        if (tid == MERGE_THREADS - 1u) carry = sEnd[tid];
        __syncthreads();
    }
    return n;
}

/* LDM: the variant that lays the block's long-distance matches over the parse output (ldm: rows of this launch; farScratch /
 * distScratch: the candidate arrays, dead once the parse is done).  Without LDM the instruction stream is the kernel's own. */
template <bool LDM>
__global__ void __launch_bounds__(MERGE_THREADS, MERGE_MIN_CTAS)
zb_merge_segments_kernel(const u8* __restrict__ src, const ZbDictSlot* __restrict__ dicts, const ZbBlock* __restrict__ blocks, ZbStrides sd, const ZbSegMeta* __restrict__ segmeta,
                         u64* __restrict__ seqs, u8* __restrict__ lits, ZbBlockMeta* __restrict__ meta,
                         ZbLdmView ldm, u32* __restrict__ farScratch, u16* __restrict__ distScratch)
{
    __shared__ u32 sPos[MERGE_TILE], sLit[MERGE_TILE], sLen[MERGE_TILE], sOff[MERGE_TILE];
    __shared__ u32 wsumL[MERGE_THREADS / 32], wsumA[MERGE_THREADS / 32], wmaxU[MERGE_THREADS / 32], wmaxK[MERGE_THREADS / 32];
    __shared__ u32 sR2[MERGE_TILE], sRep[3];
    __shared__ u32 baseL, baseA, carryEnd;
    __shared__ u32 gFirst[ZB_PARSE_SEGS], gCnt[ZB_PARSE_SEGS], gBase[ZB_PARSE_SEGS], gCur[ZB_PARSE_SEGS], gPm[ZB_PARSE_SEGS], gPl[ZB_PARSE_SEGS];
    __shared__ u32 gTotal;
    u32 const b = blockIdx.x, tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    ZbBlock const bd = blocks[b];
    if (bd.size < 7u) return;                                    /* raw block: meta written by the parse kernel */
    u64* const myseq = seqs + (size_t)b * sd.seq;
    u8*  const mylit = lits + (size_t)b * sd.lit;
    const u8* const in = src + bd.srcOff;                        /* literals always lie inside the block itself */
    u32 const segs = (bd.size + ZB_PARSE_SEG - 1u) / ZB_PARSE_SEG;
    u32 const segStride = zb_segsPerRow(sd);
    /* ---- 1. which raw sequences survive (warp 0; positions are relative to the block) ---- */
    if (warp == 0u) {
        u32 nb = 0; u64 r0 = 0, rl = 0;
        if (lane < segs) {
            nb = segmeta[(size_t)b * segStride + lane].nbSeq;
            if (nb) { r0 = myseq[(size_t)lane * SEG_SLOTS]; rl = myseq[(size_t)lane * SEG_SLOTS + nb - 1u]; }
        }
        u32 cur = 0, total = 0;
        for (u32 k = 0; k < segs; k++) {
            u32 const n = __shfl_sync(ZB_FULL, nb, (int)k);
            u64 r = __shfl_sync(ZB_FULL, r0, (int)k);
            u64 const last = __shfl_sync(ZB_FULL, rl, (int)k);
            u32 f = 0, pm = 0, pl = 0;
            while (f < n) {
                u32 const ms = ZB_RAW_MS(r), ml = ZB_RAW_MLEN(r);
                if (ms + ml <= cur || (ms < cur && ms + ml - cur < 3u)) { f++; if (f < n) r = myseq[(size_t)k * SEG_SLOTS + f]; continue; }
                if (ms < cur) { pm = cur; pl = ms + ml - cur; } else { pm = ms; pl = ml; }
                break;
            }
            if (lane == 0u) { gFirst[k] = f; gCnt[k] = n - f; gBase[k] = total; gCur[k] = cur; gPm[k] = pm; gPl[k] = pl; }
            if (f < n) { cur = (f == n - 1u) ? pm + pl : ZB_RAW_MS(last) + ZB_RAW_MLEN(last); total += n - f; }
        }
        if (lane == 0u) gTotal = total;
    }
    __syncthreads();
    u32 nbSeq;
    if constexpr (LDM) {
        /* ---- 2'. survivors (raw) to the scratch, then the overlay writes the triples ---- */
        u64* const P = reinterpret_cast<u64*>(farScratch + (size_t)b * sd.dist);
#pragma unroll 1
        for (u32 k = 0; k < segs; k++) {
            u32 const f = gFirst[k], cnt = gCnt[k];
            const u64* const sfrom = myseq + (size_t)k * SEG_SLOTS + f;
            for (u32 i = tid; i < cnt; i += MERGE_THREADS) {
                u64 r = sfrom[i];
                if (i == 0u) r = zb_pack_raw(ZB_RAW_OFF(r), gPl[k], gPm[k]);
                P[gBase[k] + i] = r;
            }
        }
        __syncthreads();
        nbSeq = zb_ldm_overlay(P, gTotal, ldm.match + ldm.first[b], ldm.cnt[b], reinterpret_cast<u32*>(distScratch + (size_t)b * sd.dist), myseq,
                               wsumA, sPos, carryEnd);
        __syncthreads();
    } else {
    /* ---- 2. survivors move down to be contiguous (in place: a destination never lies above its source) and become
     *         (offset, litLength, matchLength) ---- */
#pragma unroll 1
    for (u32 k = 0; k < segs; k++) {
        u32 const f = gFirst[k], cnt = gCnt[k];
        const u64* const sfrom = myseq + (size_t)k * SEG_SLOTS + f;
        u64* const sto = myseq + gBase[k];
        for (u32 c0 = 0; c0 < cnt; c0 += MERGE_THREADS) {
            u32 const i = c0 + tid;
            u64 r = 0; u32 ms = 0, ml = 0;
            if (i < cnt) { r = sfrom[i]; ms = ZB_RAW_MS(r); ml = ZB_RAW_MLEN(r); if (i == 0u) { ms = gPm[k]; ml = gPl[k]; } }
            u32 const myEnd = ms + ml;
            u32 prevEnd = __shfl_up_sync(ZB_FULL, myEnd, 1);
            if (lane == 31u) wsumL[warp] = myEnd;
            __syncthreads();
            if (lane == 0u) prevEnd = warp ? wsumL[warp - 1u] : (c0 ? carryEnd : gCur[k]);
            __syncthreads();
            if (i < cnt) sto[i] = zb_pack_seq(ZB_RAW_OFF(r), ms - prevEnd, ml);
            if (tid == MERGE_THREADS - 1u) carryEnd = myEnd;
            __syncthreads();
        }
    }
    nbSeq = gTotal;
    }
    u32 rep[3] = { 1u, 4u, 8u };                                 /* zstd_internal.h:69, or the frame's dictionary's */
    if (dicts && (bd.flags & ZB_FLAG_FIRST)) { rep[0] = dicts[bd.dictSlot].codeRep[0]; rep[1] = dicts[bd.dictSlot].codeRep[1]; rep[2] = dicts[bd.dictSlot].codeRep[2]; }
    zb_merge_codes(rep[0], rep[1], rep[2], (bd.flags & ZB_FLAG_FIRST) != 0u, myseq, mylit, in, nbSeq, bd.size, meta + b,
                   sPos, sLit, sLen, sOff, sR2, sRep, wsumL, wsumA, wmaxU, wmaxK, baseL, baseA);
}

/* K1c for calls made of short frames (one segment per block: nothing to join): one warp per block, 8 blocks per CTA;
 * every lane converts and gathers the literals of its own sequences, the repcode history runs through the warp. */
__global__ void __launch_bounds__(MERGE_THREADS)
zb_merge_small_kernel(const u8* __restrict__ src, const ZbDictSlot* __restrict__ dicts, const ZbBlock* __restrict__ blocks, u32 nbBlocks, ZbStrides sd, const ZbSegMeta* __restrict__ segmeta,
                      u64* __restrict__ seqs, u8* __restrict__ lits, ZbBlockMeta* __restrict__ meta)
{
    u32 const lane = threadIdx.x & 31u;
    u32 const b = blockIdx.x * (MERGE_THREADS / 32u) + (threadIdx.x >> 5);
    if (b >= nbBlocks) return;
    ZbBlock const bd = blocks[b];
    if (bd.size < 7u) return;
    u64* const myseq = seqs + (size_t)b * sd.seq;
    u8* const mylit = lits + (size_t)b * sd.lit;
    const u8* const in = src + bd.srcOff;
    u32 const nbSeq = segmeta[b].nbSeq;
    ZbRepHist hist; hist.r1 = 0; hist.r2 = 0; hist.r3 = 0;
    if (bd.flags & ZB_FLAG_FIRST) {                              /* zstd_internal.h:69, or the frame's dictionary's */
        hist.r1 = 1u; hist.r2 = 4u; hist.r3 = 8u;
        if (dicts) { hist.r1 = dicts[bd.dictSlot].codeRep[0]; hist.r2 = dicts[bd.dictSlot].codeRep[1]; hist.r3 = dicts[bd.dictSlot].codeRep[2]; }
    }
    u32 posL = 0, posA = 0;
    for (u32 t0 = 0; t0 < nbSeq; t0 += 32u) {
        u32 const i = t0 + lane;
        u64 const r = (i < nbSeq) ? myseq[i] : 0ull;
        u32 const ms = ZB_RAW_MS(r), ml = ZB_RAW_MLEN(r), off = ZB_RAW_OFF(r);
        u32 const myEnd = (i < nbSeq) ? ms + ml : 0u;
        u32 prevEnd = __shfl_up_sync(ZB_FULL, myEnd, 1);
        if (lane == 0u) prevEnd = posA;
        u32 const ll = (i < nbSeq) ? ms - prevEnd : 0u;
        u32 const adv = ll + ((i < nbSeq) ? ml : 0u);
        u32 inL = ll;
#pragma unroll
        for (u32 o = 1; o < 32u; o <<= 1) { u32 const x = __shfl_up_sync(ZB_FULL, inL, o); if (lane >= o) inL += x; }
        /* repcodes: the history is uniform across the warp, lane j keeps sequence j's code */
        u32 code = 0;
        u32 const cnt = min(32u, nbSeq - t0);
        for (u32 j = 0; j < cnt; j++) {
            u32 const o = __shfl_sync(ZB_FULL, off, (int)j), l = __shfl_sync(ZB_FULL, ll, (int)j);
            u32 const c = zb_rep_code(hist, o, l);
            if (lane == j) code = c;
        }
        if (i < nbSeq) {
            const u8* const from = in + prevEnd;
            u8* const to = mylit + posL + inL - ll;
            for (u32 x = 0; x < ll; x++) to[x] = from[x];
            myseq[i] = zb_pack_seq(code, ll, ml);
        }
        posL += __shfl_sync(ZB_FULL, inL, 31);
        posA = __shfl_sync(ZB_FULL, myEnd, (int)(cnt - 1u));
        (void)adv;
    }
    u32 const lastLits = bd.size - posA;
    for (u32 x = lane; x < lastLits; x += 32u) mylit[posL + x] = in[posA + x];
    if (lane == 0) {
        ZbBlockMeta m; m.nbSeq = nbSeq; m.litSize = posL + lastLits; m.litSecSize = 0; m.bodySize = 0;
        m.type = ZB_BT_COMPRESSED; m.forceRaw = 0; m.rleByte = 0; m.pad = 0;
        meta[b] = m;
    }
}

/* ------------------------------------------------------------------------------------------------ launchers */
/* Positions per thread (P) follow the table size: the table decides how many walk CTAs fit an SM (227 KiB of shared
 * memory), and ZB_BATCH / P threads per CTA keep about 32 warps resident in every case — fast tables (<= 56 KiB): 4 CTAs of
 * 256 threads; <= 113 KiB: 2 CTAs of 512; the doubleFast tables (128 / 200 KiB): one CTA of 1024.  The result does not
 * depend on P (a batch is ZB_BATCH positions whatever the thread count). */
template <int MLS, int P>
static cudaError_t zb_launch_walk_p(const u8* d_src, const ZbDictSlot* d_dicts, const ZbChunk* d_chunks, u32 nbChunks, u32 N, u32 insStep, const ZbStrides& sd,
                                    u32 slotFirstBlock, u16* d_dist, u32* d_far, u32 imageOff, bool build, cudaStream_t stream)
{
    cudaError_t const e = cudaFuncSetAttribute(zb_walk_kernel<MLS, P>, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024);
    if (e != cudaSuccess) return e;
    zb_walk_kernel<MLS, P><<<nbChunks, ZB_BATCH / P, (size_t)N * 4u, stream>>>(d_src, d_dicts, d_chunks, insStep, N, sd, slotFirstBlock, d_dist, d_far, imageOff, build);
    return cudaGetLastError();
}
template <int MLS>
static cudaError_t zb_launch_walk_m(const u8* d_src, const ZbDictSlot* d_dicts, const ZbChunk* d_chunks, u32 nbChunks, u32 N, u32 insStep, const ZbStrides& sd,
                                    u32 slotFirstBlock, u16* d_dist, u32* d_far, u32 imageOff, bool build, cudaStream_t stream)
{
    size_t const smem = (size_t)N * 4u;
    if (smem <= 56u * 1024u)  return zb_launch_walk_p<MLS, WALK_P_SMALL>(d_src, d_dicts, d_chunks, nbChunks, N, insStep, sd, slotFirstBlock, d_dist, d_far, imageOff, build, stream);
    if (smem <= 113u * 1024u) return zb_launch_walk_p<MLS, WALK_P_MID>(d_src, d_dicts, d_chunks, nbChunks, N, insStep, sd, slotFirstBlock, d_dist, d_far, imageOff, build, stream);
    return zb_launch_walk_p<MLS, 1>(d_src, d_dicts, d_chunks, nbChunks, N, insStep, sd, slotFirstBlock, d_dist, d_far, imageOff, build, stream);
}
extern "C" cudaError_t zb_launch_walk(const u8* d_src, const ZbDictSlot* d_dicts, const ZbChunk* d_chunks, u32 nbChunks, u32 mls, u32 N, u32 insStep, const ZbStrides& sd,
                                      u32 slotFirstBlock, u16* d_dist, u32* d_far, u32 imageOff, bool build, cudaStream_t stream)
{
    switch (mls) {
    case 4: return zb_launch_walk_m<4>(d_src, d_dicts, d_chunks, nbChunks, N, insStep, sd, slotFirstBlock, d_dist, d_far, imageOff, build, stream);
    case 5: return zb_launch_walk_m<5>(d_src, d_dicts, d_chunks, nbChunks, N, insStep, sd, slotFirstBlock, d_dist, d_far, imageOff, build, stream);
    case 6: return zb_launch_walk_m<6>(d_src, d_dicts, d_chunks, nbChunks, N, insStep, sd, slotFirstBlock, d_dist, d_far, imageOff, build, stream);
    case 7: return zb_launch_walk_m<7>(d_src, d_dicts, d_chunks, nbChunks, N, insStep, sd, slotFirstBlock, d_dist, d_far, imageOff, build, stream);
    default: return zb_launch_walk_m<8>(d_src, d_dicts, d_chunks, nbChunks, N, insStep, sd, slotFirstBlock, d_dist, d_far, imageOff, build, stream);
    }
}

/* the table images of nbImages dictionaries under one ZbParams, one CTA per image: image i walks the tail of
 * d_dicts[d_imageChunks[i].dictSlot] and stores the table(s) in that entry's image: prm->tableN u32 of the (short) table,
 * followed for doubleFast (a second launch) by prm->tableNLong u32 of the 8-byte-hash table */
extern "C" cudaError_t zb_launch_dict_images(const ZbDictSlot* d_dicts, const ZbChunk* d_imageChunks, u32 nbImages, const ZbParams* prm, cudaStream_t stream)
{
    if (nbImages == 0) return cudaSuccess;
    ZbStrides const sd = zb_strides(ZB_BLOCK_MAX);               /* unused: no block row is written */
    cudaError_t e = zb_launch_walk(nullptr, d_dicts, d_imageChunks, nbImages, prm->mls, prm->tableN, prm->insStep, sd, 0, nullptr, nullptr, 0, true, stream);
    if (e == cudaSuccess && prm->strategy == 2)
        e = zb_launch_walk(nullptr, d_dicts, d_imageChunks, nbImages, 8, prm->tableNLong, prm->insStep, sd, 0, nullptr, nullptr, prm->tableN, true, stream);
    return e;
}

extern "C" cudaError_t zb_launch_match(const u8* d_src, const ZbDictSlot* d_dicts, bool dict, const ZbBlock* d_blocks, u32 nbBlocks,
                                       const ZbChunk* d_chunks, u32 nbChunks, u32 slotFirstBlock, const ZbParams* prm, const ZbWorkRows* rows,
                                       cudaEvent_t evMid, cudaStream_t stream, const ZbLdmView* ldm)
{
    if (nbBlocks == 0) return cudaSuccess;
    ZbStrides const sd = rows->sd;
    u16* const d_dist = rows->dist; u32* const d_far = rows->far; u16* const d_dist2 = rows->dist2; u32* const d_far2 = rows->far2;
    u64* const d_seqs = rows->seqs; ZbBlockMeta* const d_meta = rows->meta; ZbSegMeta* const d_segmeta = rows->segmeta;
    cudaError_t e;
    u32 const segs = zb_segsPerRow(sd);
    u32 const sgrid = (u32)(((u64)nbBlocks * segs + PARSE_WARPS - 1) / PARSE_WARPS);                       /* one warp per segment */
    if (prm->strategy == 2) {
        /* doubleFast: one candidate walk per table */
        e = zb_launch_walk(d_src, d_dicts, d_chunks, nbChunks, 8, prm->tableNLong, prm->insStep, sd, slotFirstBlock, d_dist, d_far, prm->tableN, false, stream); if (e != cudaSuccess) return e;
        e = zb_launch_walk(d_src, d_dicts, d_chunks, nbChunks, prm->mls, prm->tableN, prm->insStep, sd, slotFirstBlock, d_dist2, d_far2, 0, false, stream); if (e != cudaSuccess) return e;
        if (evMid) cudaEventRecord(evMid, stream);
        if (dict) zb_parse_dfast_kernel<true><<<sgrid, 32 * PARSE_WARPS, 0, stream>>>(d_src, d_dicts, d_blocks, nbBlocks, *prm, sd, d_dist, d_far, d_dist2, d_far2, d_seqs, d_meta, d_segmeta);
        else      zb_parse_dfast_kernel<false><<<sgrid, 32 * PARSE_WARPS, 0, stream>>>(d_src, d_dicts, d_blocks, nbBlocks, *prm, sd, d_dist, d_far, d_dist2, d_far2, d_seqs, d_meta, d_segmeta);
    } else {
        if (prm->stepSize < 2u) return cudaErrorInvalidValue;    /* zb_parse_kernel's pairs (p, p+1) must not overlap */
        e = zb_launch_walk(d_src, d_dicts, d_chunks, nbChunks, prm->mls, prm->tableN, prm->insStep, sd, slotFirstBlock, d_dist, d_far, 0, false, stream); if (e != cudaSuccess) return e;
        if (evMid) cudaEventRecord(evMid, stream);
        if (dict) zb_parse_kernel<true><<<sgrid, 32 * PARSE_WARPS, 0, stream>>>(d_src, d_dicts, d_blocks, nbBlocks, *prm, sd, d_dist, d_far, d_seqs, d_meta, d_segmeta);
        else      zb_parse_kernel<false><<<sgrid, 32 * PARSE_WARPS, 0, stream>>>(d_src, d_dicts, d_blocks, nbBlocks, *prm, sd, d_dist, d_far, d_seqs, d_meta, d_segmeta);
    }
    return zb_launch_merge(d_src, d_dicts, d_blocks, nbBlocks, rows, ldm, stream);
}

extern "C" cudaError_t zb_launch_merge(const u8* d_src, const ZbDictSlot* d_dicts, const ZbBlock* d_blocks, u32 nbBlocks, const ZbWorkRows* rows,
                                       const ZbLdmView* ldm, cudaStream_t stream)
{
    if (nbBlocks == 0) return cudaSuccess;
    ZbStrides const sd = rows->sd;
    u32 const segs = zb_segsPerRow(sd);
    if (segs == 1u && sd.dist <= 8192u)
        zb_merge_small_kernel<<<(nbBlocks + MERGE_THREADS / 32u - 1u) / (MERGE_THREADS / 32u), MERGE_THREADS, 0, stream>>>(d_src, d_dicts, d_blocks, nbBlocks, sd, rows->segmeta, rows->seqs, rows->lits, rows->meta);
    else if (ldm)                                                /* scratch in the dead candidate rows: far, then dist (zb_workLayout) */
        zb_merge_segments_kernel<true><<<nbBlocks, MERGE_THREADS, 0, stream>>>(d_src, d_dicts, d_blocks, sd, rows->segmeta, rows->seqs, rows->lits, rows->meta, *ldm, rows->far, rows->dist);
    else
        zb_merge_segments_kernel<false><<<nbBlocks, MERGE_THREADS, 0, stream>>>(d_src, d_dicts, d_blocks, sd, rows->segmeta, rows->seqs, rows->lits, rows->meta, ZbLdmView(), nullptr, nullptr);
    return cudaGetLastError();
}
