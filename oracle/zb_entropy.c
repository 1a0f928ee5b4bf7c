/* zb_entropy.c — oracle restatement of the reference entropy stage (TEST INFRASTRUCTURE ONLY).
 *
 * Every function names the reference lines it restates (paths relative to the reference's lib/).
 * Output is meant to be byte-identical with the reference for the same (sequences, literals)
 * when the reference starts from a fresh entropy state (no repeat / treeless modes).
 */
#include <string.h>
#include <stdlib.h>
#include "zb_oracle.h"

static inline u32 hb32(u32 v) { return 31u - (u32)__builtin_clz(v); }   /* common/bits.h:177 */

/* ------------------------------------------------------------------------------------------
 * LE bit writer: value occupies [pos, pos+nbBits), LSB first (common/bitstream.h:179-241)
 * ---------------------------------------------------------------------------------------- */
typedef struct { u8* start; size_t cap; u64 acc; u32 nacc; size_t pos; int overflow; } bitw;
static void bw_init(bitw* w, u8* dst, size_t cap) { w->start = dst; w->cap = cap; w->acc = 0; w->nacc = 0; w->pos = 0; w->overflow = 0; }
static void bw_flush(bitw* w)
{
    while (w->nacc >= 8) {
        if (w->pos < w->cap) w->start[w->pos] = (u8)w->acc; else w->overflow = 1;
        w->pos++; w->acc >>= 8; w->nacc -= 8;
    }
}
static void bw_add(bitw* w, u64 value, u32 nbBits)
{
    if (nbBits == 0) return;
    value &= (nbBits >= 64) ? ~0ull : ((1ull << nbBits) - 1);
    w->acc |= value << w->nacc;
    w->nacc += nbBits;
    bw_flush(w);
}
/* end mark + byte size (bitstream.h:235-241).  0 on overflow. */
static size_t bw_close(bitw* w)
{
    bw_add(w, 1, 1);
    if (w->nacc) {
        if (w->pos < w->cap) w->start[w->pos] = (u8)w->acc; else w->overflow = 1;
        w->pos++;
    }
    return w->overflow ? 0 : w->pos;
}

/* ------------------------------------------------------------------------------------------
 * histogram (compress/hist.c:29-54) : returns largest count, trims *maxSymbolPtr
 * ---------------------------------------------------------------------------------------- */
u32 zbo_hist(const u8* src, size_t n, u32* count, u32* maxSymbolPtr)
{
    u32 maxSym = *maxSymbolPtr, largest = 0, s;
    memset(count, 0, (maxSym + 1) * sizeof(u32));
    if (n == 0) { *maxSymbolPtr = 0; return 0; }
    for (size_t i = 0; i < n; i++) count[src[i]]++;
    while (!count[maxSym]) maxSym--;
    *maxSymbolPtr = maxSym;
    for (s = 0; s <= maxSym; s++) if (count[s] > largest) largest = count[s];
    return largest;
}

/* ------------------------------------------------------------------------------------------
 * FSE
 * ---------------------------------------------------------------------------------------- */
#define FSE_MIN_TABLELOG 5
#define FSE_MAX_TABLELOG 12
#define FSE_DEFAULT_TABLELOG 11

/* fse_compress.c:347-355 */
static u32 fse_minTableLog(size_t srcSize, u32 maxSymbolValue)
{
    u32 const minBitsSrc = hb32((u32)srcSize) + 1;
    u32 const minBitsSymbols = hb32(maxSymbolValue) + 2;
    return minBitsSrc < minBitsSymbols ? minBitsSrc : minBitsSymbols;
}

/* fse_compress.c:357-374 */
u32 zbo_fse_optimalTableLog(u32 maxTableLog, size_t srcSize, u32 maxSymbolValue, u32 minus)
{
    u32 const maxBitsSrc = hb32((u32)(srcSize - 1)) - minus;
    u32 tableLog = maxTableLog;
    u32 const minBits = fse_minTableLog(srcSize, maxSymbolValue);
    if (tableLog == 0) tableLog = FSE_DEFAULT_TABLELOG;
    if (maxBitsSrc < tableLog) tableLog = maxBitsSrc;
    if (minBits > tableLog) tableLog = minBits;
    if (tableLog < FSE_MIN_TABLELOG) tableLog = FSE_MIN_TABLELOG;
    if (tableLog > FSE_MAX_TABLELOG) tableLog = FSE_MAX_TABLELOG;
    return tableLog;
}

/* fse_compress.c:379-463 : fallback normalisation */
static size_t fse_normalizeM2(int16_t* norm, u32 tableLog, const u32* count, size_t total, u32 maxSymbolValue, int16_t lowProbCount)
{
    int16_t const NOT_YET = -2;
    u32 s, distributed = 0, toDistribute;
    u32 const lowThreshold = (u32)(total >> tableLog);
    u32 lowOne = (u32)((total * 3) >> (tableLog + 1));

    for (s = 0; s <= maxSymbolValue; s++) {
        if (count[s] == 0) { norm[s] = 0; continue; }
        if (count[s] <= lowThreshold) { norm[s] = lowProbCount; distributed++; total -= count[s]; continue; }
        if (count[s] <= lowOne) { norm[s] = 1; distributed++; total -= count[s]; continue; }
        norm[s] = NOT_YET;
    }
    toDistribute = (1u << tableLog) - distributed;
    if (toDistribute == 0) return 0;

    if ((total / toDistribute) > lowOne) {
        lowOne = (u32)((total * 3) / (toDistribute * 2));
        for (s = 0; s <= maxSymbolValue; s++) {
            if (norm[s] == NOT_YET && count[s] <= lowOne) { norm[s] = 1; distributed++; total -= count[s]; }
        }
        toDistribute = (1u << tableLog) - distributed;
    }
    if (distributed == maxSymbolValue + 1) {
        u32 maxV = 0, maxC = 0;
        for (s = 0; s <= maxSymbolValue; s++) if (count[s] > maxC) { maxV = s; maxC = count[s]; }
        norm[maxV] += (int16_t)toDistribute;
        return 0;
    }
    if (total == 0) {
        for (s = 0; toDistribute > 0; s = (s + 1) % (maxSymbolValue + 1))
            if (norm[s] > 0) { toDistribute--; norm[s]++; }
        return 0;
    }
    {   u64 const vStepLog = 62 - tableLog;
        u64 const mid = (1ull << (vStepLog - 1)) - 1;
        u64 const rStep = ((((u64)1 << vStepLog) * toDistribute) + mid) / (u32)total;
        u64 tmpTotal = mid;
        for (s = 0; s <= maxSymbolValue; s++) {
            if (norm[s] == NOT_YET) {
                u64 const end = tmpTotal + (count[s] * rStep);
                u32 const sStart = (u32)(tmpTotal >> vStepLog);
                u32 const sEnd = (u32)(end >> vStepLog);
                u32 const weight = sEnd - sStart;
                if (weight < 1) return ZBO_ERR(ZBO_error_GENERIC);
                norm[s] = (int16_t)weight;
                tmpTotal = end;
            }
        }
    }
    return 0;
}

/* fse_compress.c:465-525 */
size_t zbo_fse_normalize(int16_t* norm, u32 tableLog, const u32* count, size_t total, u32 maxSymbolValue, u32 useLowProbCount)
{
    static const u32 rtb[8] = { 0, 473195, 504333, 520860, 550000, 700000, 750000, 830000 };
    if (tableLog == 0) tableLog = FSE_DEFAULT_TABLELOG;
    if (tableLog < FSE_MIN_TABLELOG) return ZBO_ERR(ZBO_error_GENERIC);
    if (tableLog > FSE_MAX_TABLELOG) return ZBO_ERR(44);
    if (tableLog < fse_minTableLog(total, maxSymbolValue)) return ZBO_ERR(ZBO_error_GENERIC);
    if (zbo_entropy_model) return zbo_fse_normalize_lr(norm, tableLog, count, total, maxSymbolValue);    /* the product's own normalisation, zb_tables.c */
    {
        int16_t const lowProbCount = useLowProbCount ? -1 : 1;
        u64 const scale = 62 - tableLog;
        u64 const step = ((u64)1 << 62) / (u32)total;
        u64 const vStep = 1ull << (scale - 20);
        int stillToDistribute = 1 << tableLog;
        u32 s, largest = 0;
        int16_t largestP = 0;
        u32 const lowThreshold = (u32)(total >> tableLog);

        for (s = 0; s <= maxSymbolValue; s++) {
            if (count[s] == total) return 0;     /* rle */
            if (count[s] == 0) { norm[s] = 0; continue; }
            if (count[s] <= lowThreshold) {
                norm[s] = lowProbCount;
                stillToDistribute--;
            } else {
                int16_t proba = (int16_t)((count[s] * step) >> scale);
                if (proba < 8) {
                    u64 const restToBeat = vStep * rtb[proba];
                    proba += (count[s] * step) - ((u64)proba << scale) > restToBeat;
                }
                if (proba > largestP) { largestP = proba; largest = s; }
                norm[s] = proba;
                stillToDistribute -= proba;
            }
        }
        if (-stillToDistribute >= (norm[largest] >> 1)) {
            size_t const e = fse_normalizeM2(norm, tableLog, count, total, maxSymbolValue, lowProbCount);
            if (zbo_isError(e)) return e;
        } else norm[largest] += (int16_t)stillToDistribute;
    }
    return tableLog;
}

/* fse_compress.c:234-327 (capacity assumed ample: the "safe" variant) */
size_t zbo_fse_writeNCount(u8* dst, size_t cap, const int16_t* norm, u32 maxSymbolValue, u32 tableLog)
{
    u8* out = dst;
    u8* const oend = dst + cap;
    int nbBits;
    int const tableSize = 1 << tableLog;
    int remaining, threshold;
    u32 bitStream = 0;
    int bitCount = 0;
    u32 symbol = 0;
    u32 const alphabetSize = maxSymbolValue + 1;
    int previousIs0 = 0;

    if (tableLog > FSE_MAX_TABLELOG) return ZBO_ERR(44);
    if (tableLog < FSE_MIN_TABLELOG) return ZBO_ERR(ZBO_error_GENERIC);

    bitStream += (tableLog - FSE_MIN_TABLELOG) << bitCount;
    bitCount += 4;
    remaining = tableSize + 1;
    threshold = tableSize;
    nbBits = (int)tableLog + 1;

#define NC_OUT16() do { if (out > oend - 2) return ZBO_ERR(ZBO_error_dstSize_tooSmall); \
        out[0] = (u8)bitStream; out[1] = (u8)(bitStream >> 8); out += 2; bitStream >>= 16; } while (0)

    while (symbol < alphabetSize && remaining > 1) {
        if (previousIs0) {
            u32 start = symbol;
            while (symbol < alphabetSize && !norm[symbol]) symbol++;
            if (symbol == alphabetSize) break;
            while (symbol >= start + 24) {
                start += 24;
                bitStream += 0xFFFFu << bitCount;
                NC_OUT16();
            }
            while (symbol >= start + 3) {
                start += 3;
                bitStream += 3u << bitCount;
                bitCount += 2;
            }
            bitStream += (symbol - start) << bitCount;
            bitCount += 2;
            if (bitCount > 16) { NC_OUT16(); bitCount -= 16; }
        }
        {   int count = norm[symbol++];
            int const max = (2 * threshold - 1) - remaining;
            remaining -= count < 0 ? -count : count;
            count++;
            if (count >= threshold) count += max;
            bitStream += (u32)count << bitCount;
            bitCount += nbBits;
            bitCount -= (count < max);
            previousIs0 = (count == 1);
            if (remaining < 1) return ZBO_ERR(ZBO_error_GENERIC);
            while (remaining < threshold) { nbBits--; threshold >>= 1; }
        }
        if (bitCount > 16) { NC_OUT16(); bitCount -= 16; }
    }
    if (remaining != 1) return ZBO_ERR(ZBO_error_GENERIC);
    if (out > oend - 2) return ZBO_ERR(ZBO_error_dstSize_tooSmall);
    out[0] = (u8)bitStream;
    out[1] = (u8)(bitStream >> 8);
    out += (bitCount + 7) / 8;
#undef NC_OUT16
    return (size_t)(out - dst);
}

/* fse_compress.c:68-214.  Symbol spreading uses the generic (low-prob aware) walk; the
 * reference's 8-byte "no low-prob" fast path lands every symbol on the same slots. */
size_t zbo_fse_buildCTable(zbo_fse_ctable* ct, const int16_t* norm, u32 maxSymbolValue, u32 tableLog)
{
    u32 const tableSize = 1u << tableLog;
    u32 const tableMask = tableSize - 1;
    u32 const step = (tableSize >> 1) + (tableSize >> 3) + 3;      /* common/fse.h:632 */
    u32 const maxSV1 = maxSymbolValue + 1;
    u16 cumul[64 + 2];
    u8  tableSymbol[512];
    u32 highThreshold = tableSize - 1;
    u32 u;

    if (tableLog > 9 || maxSymbolValue > 63) return ZBO_ERR(44);
    ct->tableLog = tableLog;
    ct->maxSymbolValue = maxSymbolValue;

    cumul[0] = 0;
    for (u = 1; u <= maxSV1; u++) {
        if (norm[u - 1] == -1) {
            cumul[u] = cumul[u - 1] + 1;
            tableSymbol[highThreshold--] = (u8)(u - 1);
        } else {
            cumul[u] = cumul[u - 1] + (u16)norm[u - 1];
        }
    }
    cumul[maxSV1] = (u16)(tableSize + 1);

    {   u32 position = 0, symbol;
        for (symbol = 0; symbol < maxSV1; symbol++) {
            int i, freq = norm[symbol];
            for (i = 0; i < freq; i++) {
                tableSymbol[position] = (u8)symbol;
                position = (position + step) & tableMask;
                while (position > highThreshold) position = (position + step) & tableMask;
            }
        }
    }
    for (u = 0; u < tableSize; u++) {
        u8 const s = tableSymbol[u];
        ct->nextState[cumul[s]++] = (u16)(tableSize + u);
    }
    {   u32 total = 0, s;
        for (s = 0; s <= maxSymbolValue; s++) {
            switch (norm[s]) {
            case 0:
                ct->deltaNbBits[s] = ((tableLog + 1) << 16) - (1u << tableLog);
                ct->deltaFindState[s] = 0;
                break;
            case -1:
            case 1:
                ct->deltaNbBits[s] = (tableLog << 16) - (1u << tableLog);
                ct->deltaFindState[s] = (int32_t)(total - 1);
                total++;
                break;
            default: {
                u32 const maxBitsOut = tableLog - hb32((u32)norm[s] - 1);
                u32 const minStatePlus = (u32)norm[s] << maxBitsOut;
                ct->deltaNbBits[s] = (maxBitsOut << 16) - minStatePlus;
                ct->deltaFindState[s] = (int32_t)(total - (u32)norm[s]);
                total += (u32)norm[s];
            } }
        }
    }
    return 0;
}

/* fse_compress.c:528-549 */
void zbo_fse_buildCTable_rle(zbo_fse_ctable* ct, u8 symbol)
{
    memset(ct, 0, sizeof(*ct));
    ct->tableLog = 0;
    ct->maxSymbolValue = symbol;
    ct->nextState[0] = 0; ct->nextState[1] = 0;
    ct->deltaNbBits[symbol & 63] = 0;
    ct->deltaFindState[symbol & 63] = 0;
}

/* common/fse.h:452-476 */
typedef struct { u32 value; const zbo_fse_ctable* ct; } fse_cstate;
static void fse_initState2(fse_cstate* st, const zbo_fse_ctable* ct, u32 symbol)
{
    u32 const dnb = ct->deltaNbBits[symbol];
    u32 const nbBitsOut = (dnb + (1u << 15)) >> 16;
    st->ct = ct;
    st->value = (nbBitsOut << 16) - dnb;
    st->value = ct->nextState[(int32_t)(st->value >> nbBitsOut) + ct->deltaFindState[symbol]];
}
static void fse_encode(bitw* w, fse_cstate* st, u32 symbol)
{
    u32 const nbBitsOut = (st->value + st->ct->deltaNbBits[symbol]) >> 16;
    bw_add(w, st->value, nbBitsOut);
    st->value = st->ct->nextState[(int32_t)(st->value >> nbBitsOut) + st->ct->deltaFindState[symbol]];
}
static void fse_flushState(bitw* w, const fse_cstate* st) { bw_add(w, st->value, st->ct->tableLog); }

/* fse_compress.c:551-608 : two interleaved states, symbols walked last -> first */
static size_t fse_compress2(u8* dst, size_t cap, const u8* src, size_t n, const zbo_fse_ctable* ct)
{
    bitw w; fse_cstate s1, s2;
    const u8* ip = src + n;
    if (n <= 2) return 0;
    if (cap <= 8) return 0;
    bw_init(&w, dst, cap);
    if (n & 1) {
        fse_initState2(&s1, ct, *--ip);
        fse_initState2(&s2, ct, *--ip);
        fse_encode(&w, &s1, *--ip);
    } else {
        fse_initState2(&s2, ct, *--ip);
        fse_initState2(&s1, ct, *--ip);
    }
    /* after the inits the remaining symbol count is even; the reference's unrolled loops all
     * reduce to strict alternation state2, state1, ... */
    while (ip > src) {
        fse_encode(&w, &s2, *--ip);
        fse_encode(&w, &s1, *--ip);
    }
    fse_flushState(&w, &s2);
    fse_flushState(&w, &s1);
    return bw_close(&w);
}

/* ------------------------------------------------------------------------------------------
 * Huffman
 * ---------------------------------------------------------------------------------------- */
#define HUF_TABLELOG_MAX 12
#define HUF_SYMBOLVALUE_MAX 255
typedef struct { u32 count; u16 parent; u8 byte; u8 nbBits; } hnode;

/* huf_compress.c:524-545 */
#define RANK_TABLE 192
#define RANK_LOG_BEGIN 158
#define RANK_DISTINCT_CUTOFF 166
static u32 huf_bucket(u32 count) { return count < RANK_DISTINCT_CUTOFF ? count : hb32(count) + RANK_LOG_BEGIN; }

/* huf_compress.c:564-615 : the exact (unstable) sort matters for ties -> restated as is */
static void huf_swap(hnode* a, hnode* b) { hnode t = *a; *a = *b; *b = t; }
static void huf_insertionSort(hnode* arr, int low, int high)
{
    int const size = high - low + 1;
    arr += low;
    for (int i = 1; i < size; i++) {
        hnode const key = arr[i];
        int j = i - 1;
        while (j >= 0 && arr[j].count < key.count) { arr[j + 1] = arr[j]; j--; }
        arr[j + 1] = key;
    }
}
static int huf_partition(hnode* arr, int low, int high)
{
    u32 const pivot = arr[high].count;
    int i = low - 1;
    for (int j = low; j < high; j++) if (arr[j].count > pivot) { i++; huf_swap(&arr[i], &arr[j]); }
    huf_swap(&arr[i + 1], &arr[high]);
    return i + 1;
}
static void huf_quickSort(hnode* arr, int low, int high)
{
    if (high - low < 8) { huf_insertionSort(arr, low, high); return; }
    while (low < high) {
        int const idx = huf_partition(arr, low, high);
        if (idx - low < high - idx) { huf_quickSort(arr, low, idx - 1); low = idx + 1; }
        else { huf_quickSort(arr, idx + 1, high); high = idx - 1; }
    }
}

/* huf_compress.c:620-668 */
static void huf_sort(hnode* node, const u32* count, u32 maxSymbolValue)
{
    struct { u16 base, curr; } rp[RANK_TABLE];
    u32 n; u32 const maxSV1 = maxSymbolValue + 1;
    memset(rp, 0, sizeof(rp));
    for (n = 0; n < maxSV1; n++) rp[huf_bucket(count[n])].base++;
    for (n = RANK_TABLE - 1; n > 0; n--) { rp[n - 1].base += rp[n].base; rp[n - 1].curr = rp[n - 1].base; }
    for (n = 0; n < maxSV1; n++) {
        u32 const c = count[n];
        u32 const r = huf_bucket(c) + 1;
        u32 const pos = rp[r].curr++;
        node[pos].count = c;
        node[pos].byte = (u8)n;
    }
    for (n = RANK_DISTINCT_CUTOFF; n < RANK_TABLE - 1; n++) {
        int const bucketSize = rp[n].curr - rp[n].base;
        if (bucketSize > 1) huf_quickSort(node + rp[n].base, 0, bucketSize - 1);
    }
}

/* huf_compress.c:376-497 */
static u32 huf_setMaxHeight(hnode* node, u32 lastNonNull, u32 targetNbBits)
{
    u32 const largestBits = node[lastNonNull].nbBits;
    if (largestBits <= targetNbBits) return largestBits;
    {   int totalCost = 0;
        u32 const baseCost = 1u << (largestBits - targetNbBits);
        int n = (int)lastNonNull;
        while (node[n].nbBits > targetNbBits) {
            totalCost += (int)(baseCost - (1u << (largestBits - node[n].nbBits)));
            node[n].nbBits = (u8)targetNbBits;
            n--;
        }
        while (node[n].nbBits == targetNbBits) --n;
        totalCost >>= (largestBits - targetNbBits);
        {   u32 const noSymbol = 0xF0F0F0F0;
            u32 rankLast[HUF_TABLELOG_MAX + 2];
            memset(rankLast, 0xF0, sizeof(rankLast));
            {   u32 currentNbBits = targetNbBits;
                for (int pos = n; pos >= 0; pos--) {
                    if (node[pos].nbBits >= currentNbBits) continue;
                    currentNbBits = node[pos].nbBits;
                    rankLast[targetNbBits - currentNbBits] = (u32)pos;
                }
            }
            while (totalCost > 0) {
                u32 nBitsToDecrease = hb32((u32)totalCost) + 1;
                for (; nBitsToDecrease > 1; nBitsToDecrease--) {
                    u32 const highPos = rankLast[nBitsToDecrease];
                    u32 const lowPos = rankLast[nBitsToDecrease - 1];
                    if (highPos == noSymbol) continue;
                    if (lowPos == noSymbol) break;
                    {   u32 const highTotal = node[highPos].count;
                        u32 const lowTotal = 2 * node[lowPos].count;
                        if (highTotal <= lowTotal) break;
                    }
                }
                while (nBitsToDecrease <= HUF_TABLELOG_MAX && rankLast[nBitsToDecrease] == noSymbol) nBitsToDecrease++;
                totalCost -= 1 << (nBitsToDecrease - 1);
                node[rankLast[nBitsToDecrease]].nbBits++;
                if (rankLast[nBitsToDecrease - 1] == noSymbol) rankLast[nBitsToDecrease - 1] = rankLast[nBitsToDecrease];
                if (rankLast[nBitsToDecrease] == 0) rankLast[nBitsToDecrease] = noSymbol;
                else {
                    rankLast[nBitsToDecrease]--;
                    if (node[rankLast[nBitsToDecrease]].nbBits != targetNbBits - nBitsToDecrease)
                        rankLast[nBitsToDecrease] = noSymbol;
                }
            }
            while (totalCost < 0) {
                if (rankLast[1] == noSymbol) {
                    while (node[n].nbBits == targetNbBits) n--;
                    node[n + 1].nbBits--;
                    rankLast[1] = (u32)(n + 1);
                    totalCost++;
                    continue;
                }
                node[rankLast[1] + 1].nbBits--;
                rankLast[1]++;
                totalCost++;
            }
        }
    }
    return targetNbBits;
}

/* huf_compress.c:756-791 (sort :620, tree :681-723, limit :376, canonical codes :730-753) */
size_t zbo_huf_buildCTable(zbo_huf_ctable* ct, const u32* count, u32 maxSymbolValue, u32 maxNbBits)
{
    hnode table[2 * (HUF_SYMBOLVALUE_MAX + 1) + 1];
    hnode* const node = table + 1;         /* node[-1] is the sentinel of huf_compress.c:695 */
    int const STARTNODE = HUF_SYMBOLVALUE_MAX + 1;
    int nonNullRank, lowS, lowN, nodeNb = STARTNODE, nodeRoot, n;

    if (maxNbBits == 0) maxNbBits = 11;
    if (maxSymbolValue > HUF_SYMBOLVALUE_MAX) return ZBO_ERR(46);
    if (zbo_entropy_model) {                                     /* the product's own code lengths (zb_tables.c) + the format's canonical codes */
        u16 nbPerRank[HUF_TABLELOG_MAX + 2] = {0};
        u16 valPerRank[HUF_TABLELOG_MAX + 2] = {0};
        size_t const ml = zbo_huf_lengths_mk(ct->nbBits, count, maxSymbolValue, maxNbBits);
        if (ml == 0 || ml > HUF_TABLELOG_MAX) return ZBO_ERR(ZBO_error_GENERIC);
        for (n = 0; n <= (int)maxSymbolValue; n++) nbPerRank[ct->nbBits[n]]++;
        {   u16 min = 0;
            for (n = (int)ml; n > 0; n--) { valPerRank[n] = min; min += nbPerRank[n]; min >>= 1; }
        }
        memset(ct->code, 0, sizeof(ct->code));
        for (n = 0; n <= (int)maxSymbolValue; n++) if (ct->nbBits[n]) ct->code[n] = valPerRank[ct->nbBits[n]]++;
        ct->tableLog = (u32)ml;
        ct->maxSymbolValue = maxSymbolValue;
        return ml;
    }
    memset(table, 0, sizeof(table));
    huf_sort(node, count, maxSymbolValue);

    nonNullRank = (int)maxSymbolValue;
    while (node[nonNullRank].count == 0) nonNullRank--;
    lowS = nonNullRank; nodeRoot = nodeNb + lowS - 1; lowN = nodeNb;
    node[nodeNb].count = node[lowS].count + node[lowS - 1].count;
    node[lowS].parent = node[lowS - 1].parent = (u16)nodeNb;
    nodeNb++; lowS -= 2;
    for (n = nodeNb; n <= nodeRoot; n++) node[n].count = 1u << 30;
    node[-1].count = 1u << 31;
    while (nodeNb <= nodeRoot) {
        int const n1 = (node[lowS].count < node[lowN].count) ? lowS-- : lowN++;
        int const n2 = (node[lowS].count < node[lowN].count) ? lowS-- : lowN++;
        node[nodeNb].count = node[n1].count + node[n2].count;
        node[n1].parent = node[n2].parent = (u16)nodeNb;
        nodeNb++;
    }
    node[nodeRoot].nbBits = 0;
    for (n = nodeRoot - 1; n >= STARTNODE; n--) node[n].nbBits = node[node[n].parent].nbBits + 1;
    for (n = 0; n <= nonNullRank; n++) node[n].nbBits = node[node[n].parent].nbBits + 1;

    maxNbBits = huf_setMaxHeight(node, (u32)nonNullRank, maxNbBits);
    if (maxNbBits > HUF_TABLELOG_MAX) return ZBO_ERR(ZBO_error_GENERIC);

    {   u16 nbPerRank[HUF_TABLELOG_MAX + 1] = {0};
        u16 valPerRank[HUF_TABLELOG_MAX + 1] = {0};
        int const alphabetSize = (int)(maxSymbolValue + 1);
        for (n = 0; n <= nonNullRank; n++) nbPerRank[node[n].nbBits]++;
        {   u16 min = 0;
            for (n = (int)maxNbBits; n > 0; n--) { valPerRank[n] = min; min += nbPerRank[n]; min >>= 1; }
        }
        memset(ct->nbBits, 0, sizeof(ct->nbBits));
        memset(ct->code, 0, sizeof(ct->code));
        for (n = 0; n < alphabetSize; n++) ct->nbBits[node[n].byte] = node[n].nbBits;
        for (n = 0; n < alphabetSize; n++) ct->code[n] = valPerRank[ct->nbBits[n]]++;
        for (n = 0; n < alphabetSize; n++) if (ct->nbBits[n] == 0) ct->code[n] = 0;
    }
    ct->tableLog = maxNbBits;
    ct->maxSymbolValue = maxSymbolValue;
    return maxNbBits;
}

/* huf_compress.c:147-186 : FSE-compress the weight vector */
static size_t huf_compressWeights(u8* dst, size_t cap, const u8* weights, size_t wtSize)
{
    u8* op = dst;
    u8* const oend = dst + cap;
    u32 maxSymbolValue = HUF_TABLELOG_MAX;
    u32 tableLog = 6;
    u32 count[HUF_TABLELOG_MAX + 1];
    int16_t norm[HUF_TABLELOG_MAX + 1];
    zbo_fse_ctable ct;

    if (wtSize <= 1) return 0;
    {   u32 const maxCount = zbo_hist(weights, wtSize, count, &maxSymbolValue);
        if (maxCount == wtSize) return 1;
        if (maxCount == 1) return 0;
    }
    tableLog = zbo_fse_optimalTableLog(tableLog, wtSize, maxSymbolValue, 2);
    {   size_t const e = zbo_fse_normalize(norm, tableLog, count, wtSize, maxSymbolValue, 0);
        if (zbo_isError(e)) return e; }
    {   size_t const h = zbo_fse_writeNCount(op, (size_t)(oend - op), norm, maxSymbolValue, tableLog);
        if (zbo_isError(h)) return h;
        op += h; }
    {   size_t const e = zbo_fse_buildCTable(&ct, norm, maxSymbolValue, tableLog);
        if (zbo_isError(e)) return e; }
    {   size_t const c = fse_compress2(op, (size_t)(oend - op), weights, wtSize, &ct);
        if (zbo_isError(c)) return c;
        if (c == 0) return 0;
        op += c; }
    return (size_t)(op - dst);
}

/* huf_compress.c:248-289 */
size_t zbo_huf_writeCTable(u8* dst, size_t cap, const zbo_huf_ctable* ct)
{
    u8 huffWeight[HUF_SYMBOLVALUE_MAX + 1];
    u32 const maxSymbolValue = ct->maxSymbolValue, huffLog = ct->tableLog;
    u32 n;
    for (n = 0; n < maxSymbolValue; n++) huffWeight[n] = ct->nbBits[n] ? (u8)(huffLog + 1 - ct->nbBits[n]) : 0;
    if (cap < 1) return ZBO_ERR(ZBO_error_dstSize_tooSmall);
    {   size_t const hSize = huf_compressWeights(dst + 1, cap - 1, huffWeight, maxSymbolValue);
        if (zbo_isError(hSize)) return hSize;
        if ((hSize > 1) & (hSize < maxSymbolValue / 2)) { dst[0] = (u8)hSize; return hSize + 1; }
    }
    if (maxSymbolValue > (256 - 128)) return ZBO_ERR(ZBO_error_GENERIC);
    if (((maxSymbolValue + 1) / 2) + 1 > cap) return ZBO_ERR(ZBO_error_dstSize_tooSmall);
    dst[0] = (u8)(128 + (maxSymbolValue - 1));
    huffWeight[maxSymbolValue] = 0;
    for (n = 0; n < maxSymbolValue; n += 2) dst[(n / 2) + 1] = (u8)((huffWeight[n] << 4) + huffWeight[n + 1]);
    return ((maxSymbolValue + 1) / 2) + 1;
}

/* huf_compress.c:1056-1118 : symbols last -> first into a forward LE bit-stream, closed by a 1 */
size_t zbo_huf_encode1X(u8* dst, size_t cap, const u8* src, size_t n, const zbo_huf_ctable* ct)
{
    bitw w;
    if (cap < 8) return 0;
    bw_init(&w, dst, cap);
    for (size_t i = n; i-- > 0; ) bw_add(&w, ct->code[src[i]], ct->nbBits[src[i]]);
    return bw_close(&w);
}

/* huf_compress.c:1168-1215 */
size_t zbo_huf_encode4X(u8* dst, size_t cap, const u8* src, size_t n, const zbo_huf_ctable* ct)
{
    size_t const segmentSize = (n + 3) / 4;
    const u8* ip = src;
    u8* op = dst;
    u8* const oend = dst + cap;
    if (cap < 6 + 1 + 1 + 1 + 8) return 0;
    if (n < 12) return 0;
    op += 6;
    for (int s = 0; s < 4; s++) {
        size_t const len = (s < 3) ? segmentSize : (size_t)((src + n) - ip);
        size_t const c = zbo_huf_encode1X(op, (size_t)(oend - op), ip, len, ct);
        if (c == 0 || c > 65535) return 0;
        if (s < 3) { dst[2 * s] = (u8)c; dst[2 * s + 1] = (u8)(c >> 8); }
        op += c; ip += len;
    }
    return (size_t)(op - dst);
}

/* encode with a given table: huf_compress.c:1218-1233 (HUF_compressCTable_internal); `already` = header bytes in front */
static size_t huf_encodeWith(u8* dst, u8* op, size_t capLeft, const u8* src, size_t n, int fourStreams, const zbo_huf_ctable* ct)
{
    size_t const c = fourStreams ? zbo_huf_encode4X(op, capLeft, src, n, ct) : zbo_huf_encode1X(op, capLeft, src, n, ct);
    if (c == 0) return 0;
    op += c;
    if ((size_t)(op - dst) >= n - 1) return 0;
    return (size_t)(op - dst);
}
static size_t huf_estimate(const zbo_huf_ctable* ct, const u32* count, u32 maxSymbolValue)      /* huf_compress.c:793 */
{
    size_t nbBits = 0;
    for (u32 s = 0; s <= maxSymbolValue; s++) nbBits += (size_t)ct->nbBits[s] * count[s];
    return nbBits >> 3;
}
static int huf_validate(const zbo_huf_ctable* ct, const u32* count, u32 maxSymbolValue)          /* huf_compress.c:804 */
{
    int bad = 0;
    if (ct->maxSymbolValue < maxSymbolValue) return 0;
    for (u32 s = 0; s <= maxSymbolValue; s++) bad |= (count[s] != 0) & (ct->nbBits[s] == 0);
    return !bad;
}

/* huf_compress.c:1333-1430.  prev/repeatPtr describe the previous block's table (NULL / 0 = none);
 * on return *repeatPtr != 0 means the previous table was used (treeless literals). */
static size_t huf_compress_internal(u8* dst, size_t cap, const u8* src, size_t n, int fourStreams, int suspectUncompressible,
                                    const zbo_huf_ctable* prev, u32* repeatPtr, int preferRepeat)
{
    u32 count[256];
    u32 maxSymbolValue = HUF_SYMBOLVALUE_MAX;
    u32 huffLog = 11;                                  /* LitHufLog, common/zstd_internal.h:105 */
    zbo_huf_ctable ct;
    u8* op = dst;
    u8* const oend = dst + cap;
    u32 repeat = (prev && repeatPtr) ? *repeatPtr : 0;

    if (!n || !cap) return 0;
    if (n > ZB_BLOCK_MAX) return ZBO_ERR(ZBO_error_srcSize_wrong);

    if (preferRepeat && repeat == 2)                                            /* :1359-1363 */
        return huf_encodeWith(dst, op, cap, src, n, fourStreams, prev);

    if (suspectUncompressible && n >= 4096 * 10) {            /* :1367-1379 */
        size_t largestTotal = 0;
        u32 m1 = maxSymbolValue, m2 = maxSymbolValue;
        largestTotal += zbo_hist(src, 4096, count, &m1);
        largestTotal += zbo_hist(src + n - 4096, 4096, count, &m2);
        if (largestTotal <= ((2 * 4096) >> 7) + 4) return 0;
    }
    {   u32 const largest = zbo_hist(src, n, count, &maxSymbolValue);   /* :1382-1385 */
        if (largest == n) { *dst = src[0]; return 1; }
        if (largest <= (n >> 7) + 4) return 0;
    }
    if (repeat == 1 && !huf_validate(prev, count, maxSymbolValue)) { repeat = 0; *repeatPtr = 0; }     /* :1389-1393 */
    if (preferRepeat && repeat != 0)                                             /* :1395-1399 */
        return huf_encodeWith(dst, op, cap, src, n, fourStreams, prev);

    huffLog = zbo_fse_optimalTableLog(huffLog, n, maxSymbolValue, 1);   /* :1402 -> :1284-1287 */
    {   size_t const maxBits = zbo_huf_buildCTable(&ct, count, maxSymbolValue, huffLog);
        if (zbo_isError(maxBits)) return maxBits;
        huffLog = (u32)maxBits;
    }
    {   size_t const hSize = zbo_huf_writeCTable(op, cap, &ct);            /* :1412 */
        if (zbo_isError(hSize)) return hSize;
        if (repeat != 0) {                                                   /* :1415-1422 */
            size_t const oldSize = huf_estimate(prev, count, maxSymbolValue);
            size_t const newSize = huf_estimate(&ct, count, maxSymbolValue);
            if (oldSize <= hSize + newSize || hSize + 12 >= n)
                return huf_encodeWith(dst, op, cap, src, n, fourStreams, prev);
        }
        if (hSize + 12ul >= n) return 0;
        op += hSize;
        if (repeatPtr) *repeatPtr = 0;
    }
    return huf_encodeWith(dst, op, (size_t)(oend - op), src, n, fourStreams, &ct);
}

/* zstd_compress_literals.c:39-63 */
static size_t lit_raw(u8* dst, size_t cap, const u8* src, size_t n)
{
    u32 const flSize = 1 + (n > 31) + (n > 4095);
    if (n + flSize > cap) return ZBO_ERR(ZBO_error_dstSize_tooSmall);
    switch (flSize) {
    case 1: dst[0] = (u8)(0 + (n << 3)); break;
    case 2: { u16 v = (u16)(0 + (1 << 2) + (n << 4)); dst[0] = (u8)v; dst[1] = (u8)(v >> 8); } break;
    default: { u32 v = (u32)(0 + (3 << 2) + (n << 4)); dst[0] = (u8)v; dst[1] = (u8)(v >> 8); dst[2] = (u8)(v >> 16); } break;
    }
    memcpy(dst + flSize, src, n);
    return n + flSize;
}
/* zstd_compress_literals.c:81-108 */
static size_t lit_rle(u8* dst, const u8* src, size_t n)
{
    u32 const flSize = 1 + (n > 31) + (n > 4095);
    switch (flSize) {
    case 1: dst[0] = (u8)(1 + (n << 3)); break;
    case 2: { u16 v = (u16)(1 + (1 << 2) + (n << 4)); dst[0] = (u8)v; dst[1] = (u8)(v >> 8); } break;
    default: { u32 v = (u32)(1 + (3 << 2) + (n << 4)); dst[0] = (u8)v; dst[1] = (u8)(v >> 8); dst[2] = (u8)(v >> 16); } break;
    }
    dst[flSize] = src[0];
    return flSize + 1;
}

/* zstd_compress_literals.c:129-235.  prev == NULL : previous table absent (HUF_repeat_none) */
static size_t compressLiterals_prev(u8* dst, size_t cap, const u8* lit, size_t n,
                                    u32 strategy, int disableLiteralCompression, int suspectUncompressible,
                                    const zbo_huf_ctable* prev, u32 prevRepeat)
{
    size_t const lhSize = 3 + (n >= 1024) + (n >= 16384);
    u32 singleStream = n < 256;
    u32 hType = 2;                                         /* set_compressed */
    size_t cLitSize;
    u32 repeat = prev ? prevRepeat : 0;

    if (disableLiteralCompression) return lit_raw(dst, cap, lit, n);
    {   /* :114-127 */
        int const shift = (9 - (int)strategy) < 3 ? (9 - (int)strategy) : 3;
        size_t const mintc = (repeat == 2) ? 6 : (size_t)8 << shift;
        if (n < mintc) return lit_raw(dst, cap, lit, n);
    }
    if (cap < lhSize + 1) return ZBO_ERR(ZBO_error_dstSize_tooSmall);
    {   int const preferRepeat = (strategy < 4 /* ZSTD_lazy */) && (n <= 1024);            /* :165 */
        if (repeat == 2 && lhSize == 3) singleStream = 1;                                  /* :171 */
        cLitSize = huf_compress_internal(dst + lhSize, cap - lhSize, lit, n, !singleStream, suspectUncompressible,
                                         prev, &repeat, preferRepeat);
        if (repeat != 0) hType = 3;                         /* set_repeat: reused the existing table */
    }
    {   size_t const minGain = (n >> 6) + 2;             /* zstd_compress_internal.h:613 */
        if (cLitSize == 0 || zbo_isError(cLitSize) || cLitSize >= n - minGain) return lit_raw(dst, cap, lit, n);
    }
    if (cLitSize == 1) {                                    /* :193-205 */
        int same = 1;
        if (n < 8) for (size_t i = 1; i < n; i++) if (lit[i] != lit[0]) same = 0;
        if (n >= 8 || same) return lit_rle(dst, lit, n);
    }
    switch (lhSize) {
    case 3: { u32 const lhc = hType + ((u32)(!singleStream) << 2) + ((u32)n << 4) + ((u32)cLitSize << 14);
              dst[0] = (u8)lhc; dst[1] = (u8)(lhc >> 8); dst[2] = (u8)(lhc >> 16); } break;
    case 4: { u32 const lhc = hType + (2 << 2) + ((u32)n << 4) + ((u32)cLitSize << 18);
              dst[0] = (u8)lhc; dst[1] = (u8)(lhc >> 8); dst[2] = (u8)(lhc >> 16); dst[3] = (u8)(lhc >> 24); } break;
    default:{ u32 const lhc = hType + (3 << 2) + ((u32)n << 4) + ((u32)cLitSize << 22);
              dst[0] = (u8)lhc; dst[1] = (u8)(lhc >> 8); dst[2] = (u8)(lhc >> 16); dst[3] = (u8)(lhc >> 24);
              dst[4] = (u8)(cLitSize >> 10); } break;
    }
    return lhSize + cLitSize;
}
size_t zbo_compressLiterals(u8* dst, size_t cap, const u8* lit, size_t n,
                            u32 strategy, int disableLiteralCompression, int suspectUncompressible)
{
    return compressLiterals_prev(dst, cap, lit, n, strategy, disableLiteralCompression, suspectUncompressible, NULL, 0);
}

/* ------------------------------------------------------------------------------------------
 * Sequences section
 * ---------------------------------------------------------------------------------------- */
#define MaxLL 35
#define MaxML 52
#define MaxOff 31
#define DefaultMaxOff 28
#define LLFSELog 9
#define MLFSELog 9
#define OffFSELog 8
#define LONGNBSEQ 0x7F00

/* format constants: common/zstd_internal.h:123-168 (RFC 8878 tables) */
static const u8 LL_bits[MaxLL + 1] = { 0,0,0,0,0,0,0,0, 0,0,0,0,0,0,0,0, 1,1,1,1,2,2,3,3, 4,6,7,8,9,10,11,12, 13,14,15,16 };
static const u8 ML_bits[MaxML + 1] = { 0,0,0,0,0,0,0,0, 0,0,0,0,0,0,0,0, 0,0,0,0,0,0,0,0, 0,0,0,0,0,0,0,0,
                                       1,1,1,1,2,2,3,3, 4,4,5,7,8,9,10,11, 12,13,14,15,16 };
static const int16_t LL_defaultNorm[MaxLL + 1] = { 4,3,2,2,2,2,2,2, 2,2,2,2,2,1,1,1, 2,2,2,2,2,2,2,2, 2,3,2,1,1,1,1,1, -1,-1,-1,-1 };
static const int16_t ML_defaultNorm[MaxML + 1] = { 1,4,3,2,2,2,2,2, 2,1,1,1,1,1,1,1, 1,1,1,1,1,1,1,1, 1,1,1,1,1,1,1,1,
                                                   1,1,1,1,1,1,1,1, 1,1,1,1,1,1,-1,-1, -1,-1,-1,-1,-1 };
static const int16_t OF_defaultNorm[DefaultMaxOff + 1] = { 1,1,1,1,1,1,2,2, 2,1,1,1,1,1,1,1, 1,1,1,1,1,1,1,1, -1,-1,-1,-1,-1 };

/* zstd_compress_internal.h:520-549 : the tables there are the closed forms below */
static u32 ll_code(u32 litLength)
{
    if (litLength > 63) return hb32(litLength) + 19;
    if (litLength < 16) return litLength;
    if (litLength < 24) return 16 + ((litLength - 16) >> 1);
    if (litLength < 32) return 20 + ((litLength - 24) >> 2);
    if (litLength < 48) return 22 + ((litLength - 32) >> 3);
    return 24;
}
static u32 ml_code(u32 mlBase)
{
    if (mlBase > 127) return hb32(mlBase) + 36;
    if (mlBase < 32) return mlBase;
    if (mlBase < 40) return 32 + ((mlBase - 32) >> 1);
    if (mlBase < 48) return 36 + ((mlBase - 40) >> 2);
    if (mlBase < 64) return 38 + ((mlBase - 48) >> 3);
    if (mlBase < 96) return 40 + ((mlBase - 64) >> 4);
    return 42;
}

enum { set_basic = 0, set_rle = 1, set_compressed = 2, set_repeat = 3 };

/* zstd_compress_sequences.c:157-240, branch strategy < ZSTD_lazy; prevRepeat = FSE_repeat of the previous table (2 = valid) */
static int seq_selectEncodingType(u32 mostFrequent, size_t nbSeq, u32 defaultNormLog, int isDefaultAllowed, u32 strategy, u32 prevRepeat)
{
    if (mostFrequent == nbSeq) {
        if (isDefaultAllowed && nbSeq <= 2) return set_basic;
        return set_rle;
    }
    if (isDefaultAllowed) {
        size_t const mult = 10 - strategy;
        size_t const dynamicFse_nbSeq_min = (((size_t)1 << defaultNormLog) * mult) >> 3;
        if (prevRepeat == 2 && nbSeq < 1000) return set_repeat;                     /* :187-191 */
        if ((nbSeq < dynamicFse_nbSeq_min) || (mostFrequent < (nbSeq >> (defaultNormLog - 1)))) return set_basic;
    }
    return set_compressed;
}

/* zstd_compress_sequences.c:242-288 */
static size_t seq_buildCTable(u8* dst, size_t cap, zbo_fse_ctable* ct, u32 FSELog, int type,
                              u32* count, u32 max, const u8* codeTable, size_t nbSeq,
                              const int16_t* defaultNorm, u32 defaultNormLog, u32 defaultMax)
{
    switch (type) {
    case set_repeat:
        return 0;                                   /* caller already points at the previous table, :260-262 */
    case set_rle:
        zbo_fse_buildCTable_rle(ct, (u8)max);
        if (cap == 0) return ZBO_ERR(ZBO_error_dstSize_tooSmall);
        *dst = codeTable[0];
        return 1;
    case set_basic:
        return zbo_fse_buildCTable(ct, defaultNorm, defaultMax, defaultNormLog);
    default: {
        int16_t norm[MaxML + 1];
        size_t nbSeq_1 = nbSeq;
        u32 const tableLog = zbo_fse_optimalTableLog(FSELog, nbSeq, max, 2);
        if (count[codeTable[nbSeq - 1]] > 1) { count[codeTable[nbSeq - 1]]--; nbSeq_1--; }   /* :271-274 */
        {   size_t const e = zbo_fse_normalize(norm, tableLog, count, nbSeq_1, max, nbSeq_1 >= 2048);  /* :57-64 */
            if (zbo_isError(e)) return e; }
        {   size_t const nc = zbo_fse_writeNCount(dst, cap, norm, max, tableLog);
            if (zbo_isError(nc)) return nc;
            {   size_t const e = zbo_fse_buildCTable(ct, norm, max, tableLog);
                if (zbo_isError(e)) return e; }
            return nc;
        }
    } }
}

/* zstd_compress.c:2881-2999 + :3001-3035 (fresh entropy state) */
size_t zbo_entropyCompressBlock(u8* dst, size_t cap,
                                const zbo_seq* seqs, size_t nbSeq,
                                const u8* lit, size_t litSize,
                                size_t blockSrcSize, u32 strategy, int disableLiteralCompression)
{
    return zbo_entropyCompressBlock_prev(dst, cap, seqs, nbSeq, lit, litSize, blockSrcSize, strategy, disableLiteralCompression, NULL);
}

size_t zbo_entropyCompressBlock_prev(u8* dst, size_t cap,
                                const zbo_seq* seqs, size_t nbSeq,
                                const u8* lit, size_t litSize,
                                size_t blockSrcSize, u32 strategy, int disableLiteralCompression,
                                const zbo_dict_entropy* prev)
{
    u8* op = dst;
    u8* const oend = dst + cap;
    size_t lastCountSize = 0;
    u8 *llCode = NULL, *ofCode = NULL, *mlCode = NULL;
    size_t result = 0;

    {   int const suspect = (nbSeq == 0) || (litSize / nbSeq >= 20);          /* :2915-2917 */
        size_t const c = compressLiterals_prev(op, cap, lit, litSize, strategy, disableLiteralCompression, suspect,
                                               (prev && prev->present) ? &prev->huf : NULL, (prev && prev->present) ? prev->hufRepeat : 0);
        if (zbo_isError(c)) return (c == ZBO_ERR(ZBO_error_dstSize_tooSmall) && blockSrcSize <= cap) ? 0 : c;
        op += c;
    }
    if ((oend - op) < 3 + 1) return 0;
    if (nbSeq < 128) *op++ = (u8)nbSeq;                                          /* :2937-2947 */
    else if (nbSeq < LONGNBSEQ) { op[0] = (u8)((nbSeq >> 8) + 0x80); op[1] = (u8)nbSeq; op += 2; }
    else { op[0] = 0xFF; op[1] = (u8)(nbSeq - LONGNBSEQ); op[2] = (u8)((nbSeq - LONGNBSEQ) >> 8); op += 3; }
    if (nbSeq == 0) { result = (size_t)(op - dst); goto check; }

    llCode = (u8*)malloc(3 * nbSeq); ofCode = llCode + nbSeq; mlCode = ofCode + nbSeq;
    for (size_t i = 0; i < nbSeq; i++) {                                           /* :2686-2712 */
        llCode[i] = (u8)ll_code(seqs[i].litLen);
        ofCode[i] = (u8)hb32(seqs[i].offBase);
        mlCode[i] = (u8)ml_code(seqs[i].matchLen - 3);
    }
    {   u8* const seqHead = op++;
        zbo_fse_ctable ctLL, ctOF, ctML;
        u32 count[MaxML + 1];
        int LLtype, Offtype, MLtype;
        u32 const rLL = (prev && prev->present) ? prev->fseRepeat[0] : 0, rOF = (prev && prev->present) ? prev->fseRepeat[1] : 0,
                  rML = (prev && prev->present) ? prev->fseRepeat[2] : 0;
        {   u32 max = MaxLL;
            u32 const mostFrequent = zbo_hist(llCode, nbSeq, count, &max);
            LLtype = seq_selectEncodingType(mostFrequent, nbSeq, 6, 1, strategy, rLL);
            if (LLtype == set_repeat) ctLL = prev->fse[0];
            size_t const cs = seq_buildCTable(op, (size_t)(oend - op), &ctLL, LLFSELog, LLtype, count, max, llCode, nbSeq, LL_defaultNorm, 6, MaxLL);
            if (zbo_isError(cs)) { result = cs; goto done; }
            if (LLtype == set_compressed) lastCountSize = cs;
            op += cs;
        }
        {   u32 max = MaxOff;
            u32 const mostFrequent = zbo_hist(ofCode, nbSeq, count, &max);
            int const defaultAllowed = (max <= DefaultMaxOff);
            Offtype = seq_selectEncodingType(mostFrequent, nbSeq, 5, defaultAllowed, strategy, rOF);
            if (Offtype == set_repeat) ctOF = prev->fse[1];
            size_t const cs = seq_buildCTable(op, (size_t)(oend - op), &ctOF, OffFSELog, Offtype, count, max, ofCode, nbSeq, OF_defaultNorm, 5, DefaultMaxOff);
            if (zbo_isError(cs)) { result = cs; goto done; }
            if (Offtype == set_compressed) lastCountSize = cs;
            op += cs;
        }
        {   u32 max = MaxML;
            u32 const mostFrequent = zbo_hist(mlCode, nbSeq, count, &max);
            MLtype = seq_selectEncodingType(mostFrequent, nbSeq, 6, 1, strategy, rML);
            if (MLtype == set_repeat) ctML = prev->fse[2];
            size_t const cs = seq_buildCTable(op, (size_t)(oend - op), &ctML, MLFSELog, MLtype, count, max, mlCode, nbSeq, ML_defaultNorm, 6, MaxML);
            if (zbo_isError(cs)) { result = cs; goto done; }
            if (MLtype == set_compressed) lastCountSize = cs;
            op += cs;
        }
        *seqHead = (u8)((LLtype << 6) + (Offtype << 4) + (MLtype << 2));           /* :2963 */

        /* zstd_compress_sequences.c:291-382 */
        {   bitw w; fse_cstate stML, stOF, stLL;
            size_t n = nbSeq - 1;
            if ((size_t)(oend - op) <= 8) { result = 0; goto done; }
            bw_init(&w, op, (size_t)(oend - op));
            fse_initState2(&stML, &ctML, mlCode[n]);
            fse_initState2(&stOF, &ctOF, ofCode[n]);
            fse_initState2(&stLL, &ctLL, llCode[n]);
            bw_add(&w, seqs[n].litLen, LL_bits[llCode[n]]);
            bw_add(&w, seqs[n].matchLen - 3, ML_bits[mlCode[n]]);
            bw_add(&w, seqs[n].offBase, ofCode[n]);
            while (n-- > 0) {
                fse_encode(&w, &stOF, ofCode[n]);
                fse_encode(&w, &stML, mlCode[n]);
                fse_encode(&w, &stLL, llCode[n]);
                bw_add(&w, seqs[n].litLen, LL_bits[llCode[n]]);
                bw_add(&w, seqs[n].matchLen - 3, ML_bits[mlCode[n]]);
                bw_add(&w, seqs[n].offBase, ofCode[n]);
            }
            fse_flushState(&w, &stML);
            fse_flushState(&w, &stOF);
            fse_flushState(&w, &stLL);
            {   size_t const streamSize = bw_close(&w);
                if (streamSize == 0) { result = 0; goto done; }                 /* dstSize_tooSmall -> raw */
                op += streamSize;
                if (lastCountSize && (lastCountSize + streamSize) < 4) { result = 0; goto done; }  /* :2987-2993 */
            }
        }
    }
    result = (size_t)(op - dst);
done:
    free(llCode);
check:
    if (zbo_isError(result) || result == 0) return (zbo_isError(result) && result != ZBO_ERR(ZBO_error_dstSize_tooSmall)) ? result : 0;
    {   size_t const maxCSize = blockSrcSize - ((blockSrcSize >> 6) + 2);            /* :3025-3028 */
        if (result >= maxCSize) return 0;
    }
    return result;
}
