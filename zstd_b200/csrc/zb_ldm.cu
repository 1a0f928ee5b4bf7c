/* zb_ldm.cu — long-distance match finder (ZSTD_c_enableLongDistanceMatching): the pass that runs in front of the parse of
 * every frame of more than one chunk, so that a block can copy from anywhere in its window (up to 2^27 bytes back), not
 * only from the 128 KiB primed in front of its chunk.  A frame compressed against a prefix (ZSTD_CCtx_refPrefix) has two
 * segments: the prefix's last P bytes at positions [0, P) and the frame at [P, P + n), each in its own buffer.  L1 runs
 * over each segment by itself (no hash or thinning across the seam) into one set of slots, the scan, compaction and sort
 * run once over both, and L3 selects for the frame's blocks only, picking a candidate's buffer by q < P (the rule with a
 * prefix, in plain C: oracle/zb_prefix.c).
 *
 * The rule is stated once, in plain C, in oracle/zb_ldm.c; these kernels produce the same matches bit for bit:
 *   L1  (one CTA per tile of LDM_TILE split points) gear rolling hash, split test, XXH64 of the minMatch bytes of every
 *       split, thinning against the splits within minMatch - 1 positions on either side; the survivors of a tile go to
 *       the tile's slots in position order.  Survivors are >= minMatch apart, so a tile has at most LDM_TILE / minMatch + 1;
 *   scan + compact: the tiles' survivors become one array in position order, with a sort key (bucket << 32 | index);
 *   L2  stable LSD radix sort of the keys by bucket, 8-bit digits (one pass per 8 bits of hashLog - bucketSizeLog), one
 *       warp per tile of RADIX_TILE keys ranking them with __match_any_sync.  Input in position order: every bucket comes
 *       out sorted by position, and the last pass writes each survivor's sorted rank;
 *   L3  (one warp per 128 KiB block) the selection: survivors of the block in position order, the 2^bucketSizeLog
 *       preceding keys of their bucket as candidates, warp-cooperative forward (32 x 8 bytes) and backward (32 bytes)
 *       counts.  The block's matches go to the match array at its first survivor's index (a block has at most one
 *       match per survivor), with their number in ldmCnt.
 * Workspace of P + n bytes (zb_ldm_scratch_bytes): 36 bytes per survivor for (P + n) / minMatch + 1 survivors, 16 bytes per L1
 * slot (about as many) and the radix counts; 8 bytes per survivor for the match list (the executor's, kept for the call). */
#include "zb_device.cuh"
#include "zb_kernels.h"

#define LDM_TILE        4096u            /* split points per L1 CTA */
#define LDM_THREADS     256u
#define RADIX_TILE      4096u            /* keys per radix warp */
#define RADIX_WARPS     4u
#define SCAN_THREADS_L  1024u
#define L3_WARPS        4u

__device__ __forceinline__ u64 zbl_gear(u32 i)                   /* splitmix64 output i + 1 of ZB_LDM_GEAR_SEED */
{
    u64 z = ZB_LDM_GEAR_SEED + (u64)(i + 1u) * 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

/* XXH64, seed 0, of len bytes (one thread) */
__device__ __forceinline__ u64 zbl_xxh64(const u8* p, u32 len)
{
    u32 i = 0;
    u64 h;
    if (len >= 32u) {
        u64 v1 = ZBX_P1 + ZBX_P2, v2 = ZBX_P2, v3 = 0, v4 = 0ull - ZBX_P1;
        for (; i + 32u <= len; i += 32u) {
            v1 = zbx_round(v1, zb_ld64u(p + i)); v2 = zbx_round(v2, zb_ld64u(p + i + 8u));
            v3 = zbx_round(v3, zb_ld64u(p + i + 16u)); v4 = zbx_round(v4, zb_ld64u(p + i + 24u));
        }
        h = zbx_rotl(v1, 1) + zbx_rotl(v2, 7) + zbx_rotl(v3, 12) + zbx_rotl(v4, 18);
        h = zbx_merge(h, v1); h = zbx_merge(h, v2); h = zbx_merge(h, v3); h = zbx_merge(h, v4);
    } else h = ZBX_P5;
    h += len;
    for (; i + 8u <= len; i += 8u) { h ^= zbx_round(0, zb_ld64u(p + i)); h = zbx_rotl(h, 27) * ZBX_P1 + ZBX_P4; }
    if (i + 4u <= len) { h ^= (u64)zb_ld32u(p + i) * ZBX_P1; h = zbx_rotl(h, 23) * ZBX_P2 + ZBX_P3; i += 4u; }
    for (; i < len; i++) { h ^= (u64)p[i] * ZBX_P5; h = zbx_rotl(h, 11) * ZBX_P1; }
    h ^= h >> 33; h *= ZBX_P2; h ^= h >> 29; h *= ZBX_P3; h ^= h >> 32;
    return h;
}

/* ---- L1: splits, hashes, thinning of one segment src[0, n), whose first byte is position posBase and whose tiles own the
 * slots from tileBase on.  Shared: v[LDM_TILE + 2H] then flags[LDM_TILE + 2H], H = minMatch - 1 ---- */
__global__ void __launch_bounds__(LDM_THREADS)
zb_ldm_split_kernel(const u8* __restrict__ src, u64 n, u64 posBase, u32 tileBase, ZbLdmParams prm, u64* __restrict__ slotPos, u64* __restrict__ slotV,
                    u32 slotCap, u32* __restrict__ tileCnt)
{
    extern __shared__ u64 sV[];
    __shared__ u64 gear[256];
    __shared__ u32 wsum[LDM_THREADS / 32u];
    u32 const tid = threadIdx.x, mm = prm.minMatch, H = mm - 1u;
    u64 const nbP = n - mm + 1u;                                   /* split points p in [0, nbP) */
    u32 const span = LDM_TILE + 2u * H;
    u8* const sF = (u8*)(sV + span);
    long long const w0 = (long long)blockIdx.x * LDM_TILE - (long long)H;   /* split point of window slot 0 */
    for (u32 i = tid; i < 256u; i += LDM_THREADS) gear[i] = zbl_gear(i);
    __syncthreads();
    /* every thread a run of consecutive split points: the hash of the byte that ends split point p is the sum of
     * gear[byte] << k over the 64 bytes behind it, so a run starts 63 bytes early and rolls */
    u32 const per = (span + LDM_THREADS - 1u) / LDM_THREADS;
    u32 const j0 = tid * per, j1 = min(span, j0 + per);
    if (j0 < j1) {
        long long const p0 = w0 + j0;
        long long const e0 = p0 + mm - 1;                           /* byte that ends split point p0 */
        long long i = e0 - 63 > 0 ? e0 - 63 : 0;
        u64 h = 0;
        for (; i < e0 && i < (long long)n; i++) h = (h << 1) + gear[src[i]];
        for (u32 j = j0; j < j1; j++) {
            long long const p = w0 + j, e = p + mm - 1;
            if (e >= 0 && e < (long long)n) h = (h << 1) + gear[src[e]];
            bool const fire = p >= 0 && (u64)p < nbP && (h & prm.stopMask) == 0ull;
            sF[j] = fire;
            sV[j] = fire ? zbl_xxh64(src + p, mm) : 0ull;
        }
    }
    __syncthreads();
    /* thinning, LDM_TILE / LDM_THREADS consecutive split points per thread, then an ordered compaction */
    u32 const PER = LDM_TILE / LDM_THREADS;
    u32 keep = 0;
    for (u32 k = 0; k < PER; k++) {
        u32 const j = H + tid * PER + k;
        if (!sF[j]) continue;
        u64 const v = sV[j];
        bool ok = true;
        for (u32 q = j - H; q < j && ok; q++) if (sF[q] && sV[q] < v) ok = false;
        for (u32 q = j + 1u; q <= j + H && ok; q++) if (sF[q] && sV[q] <= v) ok = false;
        if (ok) keep |= 1u << k;
    }
    u32 const lane = tid & 31u, warp = tid >> 5;
    u32 const c = __popc(keep);
    u32 inc = c;
#pragma unroll
    for (u32 o = 1; o < 32u; o <<= 1) { u32 const x = __shfl_up_sync(ZB_FULL, inc, o); if (lane >= o) inc += x; }
    if (lane == 31u) wsum[warp] = inc;
    __syncthreads();
    u32 base = inc - c, total = 0;
    for (u32 w = 0; w < LDM_THREADS / 32u; w++) { if (w < warp) base += wsum[w]; total += wsum[w]; }
    u32 const tile = tileBase + blockIdx.x;
    u64* const op = slotPos + (size_t)tile * slotCap; u64* const ov = slotV + (size_t)tile * slotCap;
    for (u32 k = 0; k < PER; k++) if (keep & (1u << k)) {
        u32 const j = H + tid * PER + k;
        op[base] = posBase + (u64)(w0 + j); ov[base] = sV[j]; base++;
    }
    if (tid == 0) tileCnt[tile] = total;
}

/* exclusive scan of in[0, m) into out[0, m], out[m] = total (one CTA; in and out may be the same array) */
__global__ void __launch_bounds__(SCAN_THREADS_L)
zb_ldm_scan_kernel(const u32* in, u32* out, u32 m)
{
    __shared__ u32 wsum[SCAN_THREADS_L / 32u];
    u32 const tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    u32 const per = (m + SCAN_THREADS_L - 1u) / SCAN_THREADS_L;
    u32 const a = min(m, tid * per), b = min(m, a + per);
    u32 s = 0;
    for (u32 i = a; i < b; i++) s += in[i];
    u32 inc = s;
#pragma unroll
    for (u32 o = 1; o < 32u; o <<= 1) { u32 const x = __shfl_up_sync(ZB_FULL, inc, o); if (lane >= o) inc += x; }
    if (lane == 31u) wsum[warp] = inc;
    __syncthreads();
    u32 run = inc - s, total = 0;
    for (u32 w = 0; w < SCAN_THREADS_L / 32u; w++) { if (w < warp) run += wsum[w]; total += wsum[w]; }
    __syncthreads();                                               /* in == out: every read above is done */
    for (u32 i = a; i < b; i++) { u32 const x = in[i]; out[i] = run; run += x; }
    if (tid == 0) out[m] = total;
}

/* the tiles' survivors -> pos / v / keys in position order (one CTA per L1 tile) */
__global__ void zb_ldm_compact_kernel(const u64* __restrict__ slotPos, const u64* __restrict__ slotV, u32 slotCap, const u32* __restrict__ tileOff,
                                      u32 bucketBits, u64* __restrict__ pos, u64* __restrict__ v, u64* __restrict__ keys, u32* __restrict__ rank, bool identity)
{
    u32 const t = blockIdx.x, cnt = tileOff[t + 1] - tileOff[t];
    for (u32 k = threadIdx.x; k < cnt; k += blockDim.x) {
        u32 const idx = tileOff[t] + k;
        u64 const vv = slotV[(size_t)t * slotCap + k];
        pos[idx] = slotPos[(size_t)t * slotCap + k]; v[idx] = vv;
        keys[idx] = ((vv & ((1ull << bucketBits) - 1ull)) << 32) | idx;
        if (identity) rank[idx] = idx;                             /* one bucket: position order is the sorted order */
    }
}

/* ---- L2: one LSD pass.  Counts are digit-major (count[d * nbTiles + tile]): their exclusive scan is every (digit, tile)
 * pair's first destination ---- */
__global__ void __launch_bounds__(32 * RADIX_WARPS)
zb_ldm_radix_hist_kernel(const u64* __restrict__ keys, const u32* __restrict__ nPtr, u32 shift, u32 nbTiles, u32* __restrict__ count)
{
    __shared__ u32 hist[RADIX_WARPS][256];
    u32 const lane = threadIdx.x & 31u, warp = threadIdx.x >> 5, tile = blockIdx.x * RADIX_WARPS + warp;
    for (u32 d = lane; d < 256u; d += 32u) hist[warp][d] = 0;
    __syncwarp();
    if (tile >= nbTiles) return;
    u32 const n = *nPtr;
    u64 const t0 = (u64)tile * RADIX_TILE;
    for (u32 i = lane; i < RADIX_TILE; i += 32u)
        if (t0 + i < n) atomicAdd(&hist[warp][(u32)(keys[t0 + i] >> shift) & 255u], 1u);
    __syncwarp();
    for (u32 d = lane; d < 256u; d += 32u) count[(size_t)d * nbTiles + tile] = hist[warp][d];
}

__global__ void __launch_bounds__(32 * RADIX_WARPS)
zb_ldm_radix_scatter_kernel(const u64* __restrict__ in, u64* __restrict__ out, const u32* __restrict__ nPtr, u32 shift, u32 nbTiles,
                            const u32* __restrict__ base, u32* __restrict__ rank)
{
    __shared__ u32 run[RADIX_WARPS][256];
    u32 const lane = threadIdx.x & 31u, warp = threadIdx.x >> 5, tile = blockIdx.x * RADIX_WARPS + warp;
    if (tile >= nbTiles) return;
    for (u32 d = lane; d < 256u; d += 32u) run[warp][d] = base[(size_t)d * nbTiles + tile];
    __syncwarp();
    u32 const n = *nPtr;
    u64 const t0 = (u64)tile * RADIX_TILE;
    for (u32 r = 0; r < RADIX_TILE && t0 + r < n; r += 32u) {
        bool const act = t0 + r + lane < n;
        u64 const e = act ? in[t0 + r + lane] : 0ull;
        u32 const d = act ? (u32)(e >> shift) & 255u : 256u + lane;  /* inactive lanes form groups of their own */
        u32 const grp = __match_any_sync(ZB_FULL, d);
        u32 const before = __popc(grp & ((1u << lane) - 1u));
        if (act) {
            u32 const dst = run[warp][d] + before;
            out[dst] = e;
            if (rank) rank[(u32)e] = dst;
        }
        __syncwarp();
        if (act && before == 0u) run[warp][d] += __popc(grp);
        __syncwarp();
    }
}

/* ---- L3: selection, one warp per block ---- */
__device__ __forceinline__ u32 zbl_count_fwd(const u8* a, const u8* b, u32 limit, u32 lane)
{
    u32 f = 0;
    while (true) {
        u32 const o = f + 8u * lane;
        u32 m;
        if (o + 8u <= limit) {
            u64 const x = zb_ld64u(a + o) ^ zb_ld64u(b + o);
            m = x ? (u32)((__ffsll((long long)x) - 1) >> 3) : 8u;
        } else {
            m = 0;
            while (o + m < limit && a[o + m] == b[o + m]) m++;
        }
        u32 const inc = __ballot_sync(ZB_FULL, m != 8u);
        if (inc == 0) { f += 256u; continue; }
        int const l = __ffs((int)inc) - 1;
        return f + 8u * (u32)l + __shfl_sync(ZB_FULL, m, l);
    }
}
__device__ __forceinline__ u32 zbl_count_back(const u8* a, const u8* b, u32 limit, u32 lane)   /* bytes a[-k] == b[-k], k = 1.. */
{
    u32 back = 0;
    while (true) {
        u32 const k = back + lane + 1u;
        bool const ok = k <= limit && a[-(long long)k] == b[-(long long)k];
        u32 const okb = __ballot_sync(ZB_FULL, ok);
        u32 const cnt = okb == ZB_FULL ? 32u : (u32)(__ffs((int)~okb) - 1);
        back += cnt;
        if (cnt < 32u) return back;
    }
}

/* Positions: prefix [0, P), frame [P, P + n); block k of the frame spans [P + k * ZB_BLOCK_MAX, ...).  All lanes of a warp
 * work on one candidate, so the choice of its buffer does not diverge. */
__global__ void __launch_bounds__(32 * L3_WARPS)
zb_ldm_select_kernel(const u8* __restrict__ pfx, u64 P, const u8* __restrict__ src, u64 n, ZbLdmParams prm, const u64* __restrict__ pos, const u64* __restrict__ v,
                     const u64* __restrict__ sorted, const u32* __restrict__ rank, const u32* __restrict__ nPtr, u32 nbBlocks,
                     u64 matchBase, u64* __restrict__ match, u64* __restrict__ ldmFirst, u32* __restrict__ ldmCnt)
{
    u32 const lane = threadIdx.x & 31u, k = blockIdx.x * L3_WARPS + (threadIdx.x >> 5);
    if (k >= nbBlocks) return;
    u32 const N = *nPtr;
    u64 const bs = P + (u64)k * ZB_BLOCK_MAX, be = bs + ZB_BLOCK_MAX < P + n ? bs + ZB_BLOCK_MAX : P + n;
    u64 const W = 1ull << prm.windowLog, lowQ = be > W ? be - W : 0;
    u32 lo = 0, hi = N;                                            /* first survivor at or after bs */
    while (lo < hi) { u32 const mid = (lo + hi) >> 1; if (pos[mid] < bs) lo = mid + 1u; else hi = mid; }
    u32 const nbCand = 1u << prm.bucketSizeLog;
    u64 anchor = bs;
    u32 out = 0;
    for (u32 i = lo; i < N; i++) {
        u64 const p = pos[i];
        if (p >= be) break;
        if (p < anchor) continue;
        u32 const r = rank[i];
        u32 const bucket = (u32)(sorted[r] >> 32), ck = (u32)(v[i] >> 32);
        u64 bestLen = 0, bestQ = 0, bestF = 0, bestB = 0;
        for (u32 j = 1; j <= nbCand && j <= r; j++) {
            u64 const c = sorted[r - j];
            if ((u32)(c >> 32) != bucket) break;
            u32 const ci = (u32)c;
            u64 const q = pos[ci];
            if ((u32)(v[ci] >> 32) != ck || q < lowQ) continue;
            bool const inPfx = q < P;                                /* a prefix candidate: no match runs over the seam */
            const u8* const pp = src + (p - P); const u8* const qq = inPfx ? pfx + q : src + (q - P);
            u64 const fmax = (inPfx && P - q < be - p) ? P - q : be - p;
            u32 const f = zbl_count_fwd(pp, qq, (u32)fmax, lane);
            if (f < prm.minMatch) continue;
            u64 const qroom = inPfx ? q : q - P;
            u64 const bmax = (p - anchor) < qroom ? (p - anchor) : qroom;
            u32 const b = zbl_count_back(pp, qq, (u32)bmax, lane);
            if (f + b > bestLen || (f + b == bestLen && q > bestQ)) { bestLen = f + b; bestQ = q; bestF = f; bestB = b; }
        }
        if (!bestLen) continue;
        if (lane == 0) match[matchBase + lo + out] = zb_pack_ldm(p - bestB - bs, bestLen, p - bestQ);
        out++;
        anchor = p + bestF;
    }
    if (lane == 0) { ldmFirst[k] = matchBase + lo; ldmCnt[k] = out; }
}

/* ------------------------------------------------------------------------------------------------ host */
struct ZbLdmScratch { u64 nbTiles, slotCap, cap, nbRadixTiles; };
static u64 zbl_tiles(u64 n, u32 minMatch) { return n >= minMatch ? (n - minMatch + 1u + LDM_TILE - 1u) / LDM_TILE : 0u; }   /* L1 CTAs of a segment */
static ZbLdmScratch zbl_geometry(u64 P, u64 n, const ZbLdmParams* p)
{
    ZbLdmScratch g;
    g.nbTiles = zbl_tiles(P, p->minMatch) + zbl_tiles(n, p->minMatch);
    g.slotCap = LDM_TILE / p->minMatch + 1u;
    g.cap = zb_ldm_survivor_cap(P + n, p->minMatch);               /* a segment of m bytes has at most m / minMatch survivors */
    g.nbRadixTiles = (g.cap + RADIX_TILE - 1u) / RADIX_TILE;
    return g;
}
static size_t zbl_align(size_t x) { return (x + 255u) & ~(size_t)255u; }

/* slots (2 x u64 per slot), tile counts / offsets (the last one is the survivor count), pos / v / keys x 2 (4 x u64 per survivor),
 * rank (u32 per survivor), radix counts */
extern "C" size_t zb_ldm_scratch_bytes(u64 P, u64 n, const ZbLdmParams* p)
{
    ZbLdmScratch const g = zbl_geometry(P, n, p);
    return zbl_align(g.nbTiles * g.slotCap * 16u) + zbl_align((g.nbTiles + 1u) * 4u) + zbl_align(g.cap * 32u) + zbl_align(g.cap * 4u) + zbl_align((256u * g.nbRadixTiles + 1u) * 4u);
}

extern "C" cudaError_t zb_launch_ldm(const u8* d_prefix, u64 P, const u8* d_frame, u64 n, const ZbLdmParams* prm, void* d_scratch, u32 nbBlocks,
                                     u64 matchBase, u64* d_match, u64* d_ldmFirst, u32* d_ldmCnt, cudaStream_t stream)
{
    ZbLdmScratch const g = zbl_geometry(P, n, prm);
    if (g.nbTiles == 0) return cudaMemsetAsync(d_ldmCnt, 0, nbBlocks * sizeof(u32), stream);
    u8* s = (u8*)d_scratch;
    auto take = [&](size_t bytes) { u8* const r = s; s += zbl_align(bytes); return (void*)r; };
    u64* const slotPos = (u64*)take(g.nbTiles * g.slotCap * 16u); u64* const slotV = slotPos + g.nbTiles * g.slotCap;
    u32* const tileOff = (u32*)take((g.nbTiles + 1u) * 4u);
    u64* const pos = (u64*)take(g.cap * 32u); u64* const v = pos + g.cap; u64* const keyA = v + g.cap; u64* const keyB = keyA + g.cap;
    u32* const rank = (u32*)take(g.cap * 4u);
    u32* const count = (u32*)take((256u * g.nbRadixTiles + 1u) * 4u);
    u32 const span = LDM_TILE + 2u * (prm->minMatch - 1u);
    size_t const smem = (size_t)span * 9u;
    cudaError_t e = cudaFuncSetAttribute(zb_ldm_split_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    u32 const tilesP = (u32)zbl_tiles(P, prm->minMatch), tilesF = (u32)g.nbTiles - tilesP;
    if (tilesP) zb_ldm_split_kernel<<<tilesP, LDM_THREADS, smem, stream>>>(d_prefix, P, 0, 0, *prm, slotPos, slotV, (u32)g.slotCap, tileOff);
    if (tilesF) zb_ldm_split_kernel<<<tilesF, LDM_THREADS, smem, stream>>>(d_frame, n, P, tilesP, *prm, slotPos, slotV, (u32)g.slotCap, tileOff);
    zb_ldm_scan_kernel<<<1, SCAN_THREADS_L, 0, stream>>>(tileOff, tileOff, (u32)g.nbTiles);
    u32 const* const nPtr = tileOff + g.nbTiles;
    u32 const bucketBits = prm->hashLog - prm->bucketSizeLog;
    u32 const passes = (bucketBits + 7u) / 8u;
    zb_ldm_compact_kernel<<<(u32)g.nbTiles, 128, 0, stream>>>(slotPos, slotV, (u32)g.slotCap, tileOff, bucketBits, pos, v, keyA, rank, passes == 0);
    u64* in = keyA; u64* out = keyB;
    u32 const rgrid = (u32)((g.nbRadixTiles + RADIX_WARPS - 1u) / RADIX_WARPS);
    for (u32 ps = 0; ps < passes; ps++) {
        u32 const shift = 32u + 8u * ps;
        zb_ldm_radix_hist_kernel<<<rgrid, 32 * RADIX_WARPS, 0, stream>>>(in, nPtr, shift, (u32)g.nbRadixTiles, count);
        zb_ldm_scan_kernel<<<1, SCAN_THREADS_L, 0, stream>>>(count, count, (u32)(256u * g.nbRadixTiles));
        zb_ldm_radix_scatter_kernel<<<rgrid, 32 * RADIX_WARPS, 0, stream>>>(in, out, nPtr, shift, (u32)g.nbRadixTiles, count, ps + 1u == passes ? rank : (u32*)0);
        u64* const t = in; in = out; out = t;
    }
    zb_ldm_select_kernel<<<(nbBlocks + L3_WARPS - 1u) / L3_WARPS, 32 * L3_WARPS, 0, stream>>>(d_prefix, P, d_frame, n, *prm, pos, v, in, rank, nPtr, nbBlocks,
                                                                                           matchBase, d_match, d_ldmFirst, d_ldmCnt);
    return cudaGetLastError();
}
