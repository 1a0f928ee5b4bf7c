/* zb_entropy.cuh — device-side entropy table builders (Huffman + FSE), written for a warp / a CTA.
 *
 * The format fixes what a table must BE (a complete prefix code with lengths <= tableLog whose weights the tree
 * description can carry, doc/zstd_compression_format.md "Huffman Tree Description"; a normalised distribution summing
 * to 1 << tableLog, "FSE Table Description"), not how an encoder arrives at it.  The reference's way is
 * HUF_buildCTable_wksp (lib/compress/huf_compress.c:756) and FSE_normalizeCount / FSE_buildCTable_wksp
 * (lib/compress/fse_compress.c:465, :68); the algorithms here are different ones, chosen because they spread over
 * the lanes of a warp:
 *   - FSE normalisation: largest remainders (rank by remainder, one extra slot each);
 *   - FSE compression table: a symbol's cells come from the spread rule's closed form (cell = occurrence * step
 *     mod size, the table holds no low-probability symbols), state numbers from a stable per-symbol count over
 *     the cells, 32 cells per round;
 *   - Huffman lengths: rank sort across the CTA, Moffat-Katajainen in-place code lengths, deflate-style length
 *     limiting on the histogram of lengths, lengths dealt back by rank, canonical codes by counting.
 * oracle/zb_tables.c is the plain-C statement of the same algorithms (tests only).
 */
#ifndef ZB_ENTROPY_CUH
#define ZB_ENTROPY_CUH
#include "zb_device.cuh"

#define ZBD_ERR 0xFFFFFFFFu           /* "could not build" -> caller falls back to raw/basic */

/* ------------------------------------------------------------------ serial LE bit writer (one lane) */
struct ZbdBitW { u8* out; u32 pos; u64 acc; u32 nacc; };
__device__ __forceinline__ void zbd_bw_init(ZbdBitW* w, u8* out) { w->out = out; w->pos = 0; w->acc = 0; w->nacc = 0; }
__device__ __forceinline__ void zbd_bw_add(ZbdBitW* w, u32 value, u32 nbBits)
{
    if (!nbBits) return;
    w->acc |= (u64)(value & ((1u << nbBits) - 1u)) << w->nacc;       /* nbBits <= 16 here */
    w->nacc += nbBits;
    while (w->nacc >= 8) { w->out[w->pos++] = (u8)w->acc; w->acc >>= 8; w->nacc -= 8; }
}
__device__ __forceinline__ u32 zbd_bw_close(ZbdBitW* w)              /* a set bit ends a stream, then zero padding */
{
    zbd_bw_add(w, 1, 1);
    if (w->nacc) w->out[w->pos++] = (u8)w->acc;
    return w->pos;
}

/* ------------------------------------------------------------------ FSE */
/* ZbdFseCTable: zb_common.h.  Encoding with it (format: "FSE", state in [size, 2 * size)):
 *   nbBitsOut = (state + deltaNbBits[sym]) >> 16; emit the low nbBitsOut bits of state;
 *   state = nextState[(state >> nbBitsOut) + deltaFindState[sym]]. */

/* accuracy for srcSize symbols over an alphabet ending at maxSymbolValue: enough states for the alphabet and for the
 * source, not more than the source can fill (same value as FSE_optimalTableLog_internal, fse_compress.c:357-374) */
__device__ __forceinline__ u32 zbd_fse_optimalTableLog(u32 maxTableLog, u32 srcSize, u32 maxSymbolValue, u32 minus)
{
    u32 const fromSource = zb_hb32(srcSize - 1u) - minus;
    u32 const needSrc = zb_hb32(srcSize) + 1u, needAlphabet = zb_hb32(maxSymbolValue) + 2u;
    u32 const floorLog = needSrc < needAlphabet ? needSrc : needAlphabet;
    u32 log = maxTableLog < fromSource ? maxTableLog : fromSource;
    if (log < floorLog) log = floorLog;
    return log < 5u ? 5u : (log > 12u ? 12u : log);
}

/* Normalisation by largest remainders, one warp, up to 64 symbols (lane l owns symbols l and l + 32).
 * norm[s] = max(1, floor(count[s] << tableLog / total)) for present symbols; if that sums short of the table size
 * the largest remainders get one more (ties: lower symbol), if it overshoots the largest entry gives one back.
 * Returns tableLog, or ZBD_ERR. */
__device__ inline u32 zbw_fse_normalize(short* norm, u32 tableLog, const u32* count, u32 total, u32 maxSymbolValue, u32 lane)
{
    u32 const T = 1u << tableLog;
    u32 base[2], rem[2]; bool present[2];
#pragma unroll
    for (u32 k = 0; k < 2u; k++) {
        u32 const s = lane + 32u * k;
        u32 const c = s <= maxSymbolValue ? count[s] : 0u;
        present[k] = c != 0u; base[k] = 0; rem[k] = 0;
        if (c) {
            u64 const x = (u64)c << tableLog;
            u32 const q = (u32)(x / total);
            if (q == 0u) base[k] = 1u; else { base[k] = q; rem[k] = (u32)(x - (u64)q * total); }
        }
    }
    u32 sum = base[0] + base[1];
#pragma unroll
    for (u32 o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(ZB_FULL, sum, o);
    if (sum < T) {
        u32 const need = T - sum;
        u32 rank[2] = { 0u, 0u };
        for (u32 j = 0; j < 64u; j++) {                          /* every present symbol against every other */
            u32 const rj = __shfl_sync(ZB_FULL, (j < 32u) ? rem[0] : rem[1], (int)(j & 31u));
            bool const pj = __shfl_sync(ZB_FULL, (j < 32u) ? (int)present[0] : (int)present[1], (int)(j & 31u)) != 0;
#pragma unroll
            for (u32 k = 0; k < 2u; k++) {
                u32 const s = lane + 32u * k;
                rank[k] += (pj && (rj > rem[k] || (rj == rem[k] && j < s))) ? 1u : 0u;
            }
        }
        u32 nbPresent = __popc(__ballot_sync(ZB_FULL, present[0])) + __popc(__ballot_sync(ZB_FULL, present[1]));
        if (need > nbPresent) return ZBD_ERR;
#pragma unroll
        for (u32 k = 0; k < 2u; k++) if (present[k] && rank[k] < need) base[k]++;
    } else {
        for (u32 over = sum - T; over > 0u; over--) {
            u32 bestV = base[0], bestS = lane;
            if (base[1] > bestV) { bestV = base[1]; bestS = lane + 32u; }
#pragma unroll
            for (u32 o = 16; o > 0; o >>= 1) {
                u32 const v = __shfl_xor_sync(ZB_FULL, bestV, o), s2 = __shfl_xor_sync(ZB_FULL, bestS, o);
                if (v > bestV || (v == bestV && s2 < bestS)) { bestV = v; bestS = s2; }
            }
            if (bestV < 2u) return ZBD_ERR;
            if ((bestS & 31u) == lane) { if (bestS >> 5) base[1]--; else base[0]--; }   /* a select: an indexed base[] would live in local memory */
        }
    }
#pragma unroll
    for (u32 k = 0; k < 2u; k++) { u32 const s = lane + 32u * k; if (s <= maxSymbolValue) norm[s] = (short)base[k]; }
    __syncwarp();
    return tableLog;
}

/* Table description (format: "FSE Table Description"; the decoder's side is FSE_readNCount, lib/common/entropy_common.c:42):
 * 4 bits of accuracy, then every probability as value = prob + 1 in a field whose width follows the points still to
 * be distributed; small values use one bit less; a zero probability is followed by a 2-bit count of further zeros
 * (3 = "three more and another count", sixteen set bits = 24 more).  One lane.  Returns the size in bytes. */
__device__ inline u32 zbd_fse_writeNCount(u8* dst, const short* norm, u32 maxSymbolValue, u32 tableLog)
{
    ZbdBitW w; zbd_bw_init(&w, dst);
    zbd_bw_add(&w, tableLog - 5u, 4);
    int left = (int)(1u << tableLog) + 1;                        /* points to distribute, plus one */
    int limit = (int)(1u << tableLog);
    u32 width = tableLog + 1u;
    u32 s = 0;
    bool afterZero = false;
    while (s <= maxSymbolValue && left > 1) {
        if (afterZero) {
            u32 z = 0;
            while (s + z <= maxSymbolValue && norm[s + z] == 0) z++;
            if (s + z > maxSymbolValue) break;                   /* nothing but zeros left: cannot happen for a full distribution */
            s += z;
            while (z >= 24u) { zbd_bw_add(&w, 0xFFFFu, 16); z -= 24u; }
            while (z >= 3u) { zbd_bw_add(&w, 3u, 2); z -= 3u; }
            zbd_bw_add(&w, z, 2);
        }
        int const p = norm[s++];
        int const small = 2 * limit - 1 - left;                  /* values below this one take width - 1 bits */
        left -= p < 0 ? -p : p;
        int v = p + 1;
        if (v >= limit) v += small;
        zbd_bw_add(&w, (u32)v, width - (v < small ? 1u : 0u));
        afterZero = (p == 0);
        while (left < limit) { width--; limit >>= 1; }
    }
    if (left != 1) return ZBD_ERR;
    if (w.nacc) w.out[w.pos++] = (u8)w.acc;
    return w.pos;
}

/* Compression table of a distribution without low-probability (-1) symbols, one warp.
 * Cells: the spread rule visits cell (k * step) mod size for the k-th table occurrence (step = size/2 + size/8 + 3,
 * format "FSE decoding table"), occurrences are handed out symbol after symbol.  A symbol's cells, in ascending
 * cell order, are its sub-states n, n+1, ... (n = its probability); nextState[] lists, symbol after symbol, the
 * table states of those sub-states.  symAt: size bytes, cum: 66 u16, both shared memory scratch. */
__device__ inline void zbw_fse_buildCTable(ZbdFseCTable* ct, const short* norm, u32 maxSymbolValue, u32 tableLog, u8* symAt, u16* cum, u32 lane)
{
    u32 const T = 1u << tableLog, mask = T - 1u, step = (T >> 1) + (T >> 3) + 3u;
    u16* const run = cum + 65;                                   /* not used: kept for layout clarity */
    (void)run;
    /* exclusive prefix sums of the probabilities: lane l owns symbols 2l and 2l+1 */
    u32 const n0 = (2u * lane <= maxSymbolValue) ? (u32)norm[2u * lane] : 0u;
    u32 const n1 = (2u * lane + 1u <= maxSymbolValue) ? (u32)norm[2u * lane + 1u] : 0u;
    u32 inc = n0 + n1;
#pragma unroll
    for (u32 o = 1; o < 32u; o <<= 1) { u32 const x = __shfl_up_sync(ZB_FULL, inc, o); if (lane >= o) inc += x; }
    u32 const ex = inc - n0 - n1;
    cum[2u * lane] = (u16)ex; cum[2u * lane + 1u] = (u16)(ex + n0);
    if (lane == 31u) cum[64] = (u16)inc;
    if (lane == 0u) { ct->tableLog = tableLog; ct->maxSymbolValue = maxSymbolValue; }
    /* per-symbol transform: how many bits a state sheds before it lands in [n, 2n), and where its sub-states start */
#pragma unroll
    for (u32 k = 0; k < 2u; k++) {
        u32 const s = 2u * lane + k;
        if (s <= maxSymbolValue) {
            u32 const n = k ? n1 : n0, c = k ? ex + n0 : ex;
            if (n == 0u) { ct->deltaNbBits[s] = ((tableLog + 1u) << 16) - T; ct->deltaFindState[s] = 0; }
            else {
                u32 const shed = n == 1u ? tableLog : tableLog - zb_hb32(n - 1u);   /* bits shed by the smallest states of the symbol's range */
                ct->deltaNbBits[s] = (shed << 16) - (n << shed);
                ct->deltaFindState[s] = (int)c - (int)n;
            }
        }
    }
    __syncwarp();
    /* which symbol owns each cell */
    u32 const nbSym = maxSymbolValue + 1u;
    for (u32 k0 = 0; k0 < T; k0 += 32u) {
        u32 const k = k0 + lane;
        if (k < T) {
            u32 lo = 0, hi = nbSym;                               /* largest s with cum[s] <= k */
            while (hi - lo > 1u) { u32 const mid = (lo + hi) >> 1; if (cum[mid] <= k) lo = mid; else hi = mid; }
            symAt[(k * step) & mask] = (u8)lo;
        }
    }
    __syncwarp();
    /* state numbers: cells in ascending order, a stable count per symbol (32 cells a round) */
    u32 seen0 = 0, seen1 = 0;                                    /* cells already numbered for symbols 2l, 2l+1 (lane-owned counters) */
    for (u32 u0 = 0; u0 < T; u0 += 32u) {
        u32 const u = u0 + lane;
        u32 const s = (u < T) ? symAt[u] : 0xFFu;
        u32 pending = __ballot_sync(ZB_FULL, u < T);
        while (pending) {
            int const leader = __ffs((int)pending) - 1;
            u32 const ls = __shfl_sync(ZB_FULL, s, leader);
            u32 const grp = __ballot_sync(ZB_FULL, s == ls);
            u32 const owner = ls >> 1;
            u32 const before = __shfl_sync(ZB_FULL, (ls & 1u) ? seen1 : seen0, (int)owner);
            if (s == ls) ct->nextState[cum[ls] + before + (u32)__popc(grp & ((1u << lane) - 1u))] = (u16)(T + u);
            if (lane == owner) { if (ls & 1u) seen1 += (u32)__popc(grp); else seen0 += (u32)__popc(grp); }
            pending &= ~grp;
        }
    }
    __syncwarp();
}

/* format "FSE": a single-symbol (RLE) table: zero bits per symbol */
__device__ inline void zbd_fse_buildCTable_rle(ZbdFseCTable* ct, u32 symbol)
{
    ct->tableLog = 0; ct->maxSymbolValue = symbol;
    ct->nextState[0] = 0; ct->nextState[1] = 0;
    ct->deltaNbBits[symbol] = 0; ct->deltaFindState[symbol] = 0;
}

/* first state of a stream: the symbol's smallest-cost sub-state (the first symbol costs no bits) */
__device__ __forceinline__ u32 zbd_fse_initState2(const ZbdFseCTable* ct, u32 symbol)
{
    u32 const dnb = ct->deltaNbBits[symbol];
    u32 const nbBitsOut = (dnb + (1u << 15)) >> 16;
    u32 const value = (nbBitsOut << 16) - dnb;
    return ct->nextState[(int)(value >> nbBitsOut) + ct->deltaFindState[symbol]];
}
/* returns next state; *bits / *nb receive the emitted field */
__device__ __forceinline__ u32 zbd_fse_step(const ZbdFseCTable* ct, u32 state, u32 symbol, u32* bits, u32* nb)
{
    u32 const nbBitsOut = (state + ct->deltaNbBits[symbol]) >> 16;
    *nb = nbBitsOut;
    *bits = state & ((1u << nbBitsOut) - 1u);
    return ct->nextState[(int)(state >> nbBitsOut) + ct->deltaFindState[symbol]];
}

/* ------------------------------------------------------------------ Huffman */
struct ZbdHufWksp {
    u32 A[256];                      /* ascending weights, then parents, then depths (in place) */
    u16 rankSym[256];                /* symbol of rank r (count descending, symbol ascending) */
    u8  len[256];                    /* code length per symbol */
    u8  weights[256];
    u32 nl[16];                      /* symbols per code length */
    u32 firstCode[16];               /* first code value of each length */
    u32 wcount[16];                  /* histogram of the weights */
    short wnorm[16];
    u8  symAt[64];
    u16 cum[66];
    u32 maxLen, nz;
    ZbdFseCTable wct;                /* FSE table for the weights */
};

/* Code lengths <= target for count[0..maxSymbolValue] and canonical codes; the whole CTA (HUF_THREADS threads) calls it,
 * at least two symbols are present.  enc[s] = code | nbBits << 16 (0 for absent symbols).  Returns the longest
 * length in use, or ZBD_ERR. */
template <int HUF_THREADS>
__device__ inline u32 zbc_huf_build(ZbdHufWksp* w, const u32* count, u32 maxSymbolValue, u32 target, u32* enc)
{
    u32 const tid = threadIdx.x;
    if (tid == 0) w->nz = 0;
    __syncthreads();
    /* 1. rank of every present symbol = how many present symbols come before it (count descending, symbol ascending) */
    {   u32 mine = 0;
        for (u32 s = tid; s < 256u; s += HUF_THREADS) {
            u32 const c = s <= maxSymbolValue ? count[s] : 0u;
            w->len[s] = 0;
            if (c) {
                u32 r = 0;
                for (u32 j = 0; j <= maxSymbolValue; j++) { u32 const cj = count[j]; r += (cj > c || (cj == c && j < s)) ? 1u : 0u; }
                w->rankSym[r] = (u16)s;
                mine++;
            }
        }
        if (mine) atomicAdd(&w->nz, mine);
    }
    __syncthreads();
    u32 const nz = w->nz;
    for (u32 i = tid; i < nz; i += HUF_THREADS) w->A[i] = count[w->rankSym[nz - 1u - i]];      /* ascending weights */
    __syncthreads();
    /* 2. minimum-redundancy code lengths in place (Moffat & Katajainen 1995): a serial recurrence over <= 256 nodes */
    if (tid == 0) {
        u32* const A = w->A;
        u32 root = 0, leaf = 2, next;
        A[0] += A[1];
        for (next = 1; next + 1u < nz; next++) {                 /* A[k] becomes the parent of internal node k */
            if (leaf >= nz || A[root] < A[leaf]) { A[next] = A[root]; A[root++] = next; } else A[next] = A[leaf++];
            if (leaf >= nz || (root < next && A[root] < A[leaf])) { A[next] += A[root]; A[root++] = next; } else A[next] += A[leaf++];
        }
        A[nz - 2u] = 0;
        for (next = nz - 2u; next-- > 0u; ) A[next] = A[A[next]] + 1u;      /* depths of the internal nodes */
        {   int avbl = 1, used = 0, depth = 0;
            int rt = (int)nz - 2, nx = (int)nz - 1;
            while (avbl > 0) {                                   /* depths of the leaves, deepest first */
                while (rt >= 0 && (int)A[rt] == depth) { used++; rt--; }
                while (avbl > used) { A[nx--] = (u32)depth; avbl--; }
                avbl = 2 * used; depth++; used = 0;
            }
        }
        for (u32 l = 0; l < 16u; l++) w->nl[l] = 0;
    }
    __syncthreads();
    /* 3. histogram of lengths (lengths above 15 are counted at 15: they are lifted to `target` anyway) */
    u32 const deepest = w->A[0];
    for (u32 i = tid; i < nz; i += HUF_THREADS) { u32 const l = w->A[i]; atomicAdd(&w->nl[l < 15u ? l : 15u], 1u); }
    __syncthreads();
    if (tid == 0) {
        u32* const nl = w->nl;
        u32 maxLen = deepest;
        if (maxLen > target) {
            /* lift what is too deep, then repair the Kraft sum: per unit of excess the deepest leaf above the bottom level
             * goes one level down together with one leaf from the bottom level */
            u32 K = 0;
            for (u32 l = target + 1u; l < 16u; l++) { nl[target] += nl[l]; nl[l] = 0; }
            for (u32 l = 1; l <= target; l++) K += nl[l] << (target - l);
            for (u32 E = K - (1u << target); E > 0u; E--) {
                u32 b = target - 1u;
                while (nl[b] == 0u) b--;
                nl[b]--; nl[b + 1u] += 2u; nl[target]--;
            }
            maxLen = target;
        }
        while (nl[maxLen] == 0u) maxLen--;
        w->maxLen = maxLen;
        /* first code of every length: the longest codes start at 0, a shorter length continues where the longer one
         * stopped, one bit shorter (format "Huffman Tree Description": weights order the prefix ranges) */
        u32 v = 0;
        for (u32 l = maxLen; l > 0u; l--) { w->firstCode[l] = v; v = (v + nl[l]) >> 1; }
    }
    __syncthreads();
    /* 4. lengths dealt out by rank: the nl[1] most frequent symbols get 1 bit, the next nl[2] get 2, ... */
    u32 const maxLen = w->maxLen;
    for (u32 r = tid; r < nz; r += HUF_THREADS) {
        u32 l = 1, acc = w->nl[1];
        while (r >= acc) { l++; acc += w->nl[l]; }
        w->len[w->rankSym[r]] = (u8)l;
    }
    __syncthreads();
    /* 5. canonical codes: within a length, ascending symbol order */
    for (u32 s = tid; s < 256u; s += HUF_THREADS) {
        u32 const l = w->len[s];
        u32 e = 0;
        if (l) {
            u32 idx = 0;
            for (u32 j = 0; j < s; j++) idx += (w->len[j] == l) ? 1u : 0u;
            e = (w->firstCode[l] + idx) | (l << 16);
        }
        enc[s] = e;
    }
    __syncthreads();
    return maxLen;
}

/* Tree description (format "Huffman Tree Description"): weights = maxLen + 1 - length (0 = absent) of symbols
 * 0 .. maxSymbolValue-1 (the last one is implied), FSE-compressed with two interleaved states when that is smaller
 * than half a byte per weight, else 4 bits each (only possible up to 128 weights).  Called by the whole CTA; the
 * FSE part runs on warp 0.  Returns the header size, or ZBD_ERR. */
template <int HUF_THREADS>
__device__ inline u32 zbc_huf_writeHeader(ZbdHufWksp* w, u8* dst, const u32* enc, u32 maxSymbolValue, u32 huffLog, u32* sh_result)
{
    u32 const tid = threadIdx.x, lane = tid & 31u;
    u8* const wt = w->weights;
    u32 const wtSize = maxSymbolValue;
    if (tid < 16u) w->wcount[tid] = 0;
    __syncthreads();
    for (u32 n = tid; n < wtSize; n += HUF_THREADS) {
        u32 const nb = enc[n] >> 16;
        u32 const v = nb ? huffLog + 1u - nb : 0u;
        wt[n] = (u8)v;
        atomicAdd(&w->wcount[v], 1u);
    }
    if (tid == 0) wt[wtSize] = 0;
    __syncthreads();
    if (tid < 32u) {
        u32 hSize = 0;                                           /* size of the FSE form, 0 = not usable */
        if (wtSize > 2u) {
            u32 const c = lane < 13u ? w->wcount[lane] : 0u;
            u32 const used = __ballot_sync(ZB_FULL, c != 0u);
            u32 const maxSym = 31u - (u32)__clz((int)used);
            u32 maxCount = c;
#pragma unroll
            for (u32 o = 16; o > 0; o >>= 1) maxCount = max(maxCount, __shfl_xor_sync(ZB_FULL, maxCount, o));
            if (maxCount != wtSize && maxCount != 1u) {          /* one repeated weight, or all distinct: the 4-bit form is used */
                u32 const tableLog = zbd_fse_optimalTableLog(6, wtSize, maxSym, 2);
                u32 ok = zbw_fse_normalize(w->wnorm, tableLog, w->wcount, wtSize, maxSym, lane);
                u32 nc = 0;
                if (ok != ZBD_ERR) {
                    if (lane == 0) nc = zbd_fse_writeNCount(dst + 1, w->wnorm, maxSym, tableLog);
                    nc = __shfl_sync(ZB_FULL, nc, 0);
                    if (nc == ZBD_ERR) ok = ZBD_ERR;
                }
                if (ok != ZBD_ERR) {
                    zbw_fse_buildCTable(&w->wct, w->wnorm, maxSym, tableLog, w->symAt, w->cum, lane);
                    if (lane == 0) {
                        /* two interleaved states, last weight first (format "FSE" bitstream, read backwards) */
                        ZbdBitW bw; zbd_bw_init(&bw, dst + 1 + nc);
                        const u8* ip = wt + wtSize;
                        u32 s1, s2, bits, nb;
                        if (wtSize & 1u) {
                            s1 = zbd_fse_initState2(&w->wct, *--ip);
                            s2 = zbd_fse_initState2(&w->wct, *--ip);
                            s1 = zbd_fse_step(&w->wct, s1, *--ip, &bits, &nb); zbd_bw_add(&bw, bits, nb);
                        } else {
                            s2 = zbd_fse_initState2(&w->wct, *--ip);
                            s1 = zbd_fse_initState2(&w->wct, *--ip);
                        }
                        while (ip > wt) {
                            s2 = zbd_fse_step(&w->wct, s2, *--ip, &bits, &nb); zbd_bw_add(&bw, bits, nb);
                            s1 = zbd_fse_step(&w->wct, s1, *--ip, &bits, &nb); zbd_bw_add(&bw, bits, nb);
                        }
                        zbd_bw_add(&bw, s2, tableLog);
                        zbd_bw_add(&bw, s1, tableLog);
                        hSize = nc + zbd_bw_close(&bw);
                    }
                } else if (lane == 0) hSize = ZBD_ERR;
            } else if (maxCount == wtSize) hSize = 1;
        }
        if (lane == 0) {
            u32 res;
            if (hSize == ZBD_ERR) res = ZBD_ERR;
            else if (hSize > 1u && hSize < maxSymbolValue / 2u) { dst[0] = (u8)hSize; res = hSize + 1u; }
            else if (maxSymbolValue > 128u) res = ZBD_ERR;
            else {
                dst[0] = (u8)(128u + (maxSymbolValue - 1u));
                for (u32 n = 0; n < maxSymbolValue; n += 2u) dst[(n / 2u) + 1u] = (u8)((wt[n] << 4) + wt[n + 1u]);
                res = ((maxSymbolValue + 1u) / 2u) + 1u;
            }
            *sh_result = res;
        }
    }
    __syncthreads();
    return *sh_result;
}
#endif
