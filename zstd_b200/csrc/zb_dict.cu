/* zb_dict.cu — host side: parsing a dictionary (no device code here).
 * Replaces ZSTD_compress_insertDictionary / ZSTD_loadZstdDictionary / ZSTD_loadCEntropy
 * (lib/compress/zstd_compress.c:5119-5156, :5087-5115, :4987-5076) for the simple API:
 *   < 8 bytes                -> ignored (:5132)
 *   no magic 0xEC30A437      -> raw content (:5143-5148)
 *   magic                    -> dictID, Huffman table (HUF_readCTable huf_compress.c:292, HUF_readStats
 *                               common/entropy_common.c:236 incl. FSE-decoded weights), OF/ML/LL FSE tables
 *                               (FSE_readNCount entropy_common.c:42, FSE_buildCTable fse_compress.c:68),
 *                               repeat modes (ZSTD_dictNCountRepeat :4973), 3 repcodes, then content.
 */
#include <string.h>
#include "zb_common.h"
#include "zb_kernels.h"

static inline u32 hb32(u32 v) { return 31u - (u32)__builtin_clz(v); }

namespace {
struct FBits {                                            /* little-endian forward bit reader */
    const u8* p; size_t avail, pos = 0; u64 bits = 0; u32 nb = 0; size_t used = 0;
    FBits(const u8* p_, size_t a) : p(p_), avail(a) {}
    void need(u32 k) { while (nb < k) { u64 const byte = pos < avail ? p[pos] : 0; bits |= byte << nb; nb += 8; pos++; } }
    void take(u32 k) { bits >>= k; nb -= k; used += k; }
};

/* doc/zstd_compression_format.md:1063 ; returns bytes read, 0 if malformed */
size_t readNCount(short* norm, u32* maxSymbolPtr, u32* tableLogPtr, const u8* p, size_t avail)
{
    FBits b(p, avail);
    u32 const maxSymbol = *maxSymbolPtr;
    u32 symbol = 0;
    memset(norm, 0, (maxSymbol + 1) * sizeof(short));
    b.need(4); u32 const tableLog = (u32)(b.bits & 15) + 5; b.take(4);
    if (tableLog > 15) return 0;
    *tableLogPtr = tableLog;
    int remaining = (1 << tableLog) + 1, threshold = 1 << tableLog, nbBits = (int)tableLog + 1;
    while (remaining > 1 && symbol <= maxSymbol) {
        int const max = (2 * threshold - 1) - remaining;
        int count;
        b.need((u32)nbBits);
        if ((int)(b.bits & (u32)(threshold - 1)) < max) { count = (int)(b.bits & (u32)(threshold - 1)); b.take((u32)nbBits - 1); }
        else { count = (int)(b.bits & (u32)(2 * threshold - 1)); if (count >= threshold) count -= max; b.take((u32)nbBits); }
        count--;
        remaining -= count < 0 ? -count : count;
        norm[symbol++] = (short)count;
        if (count == 0) { for (;;) { b.need(2); u32 const r = (u32)(b.bits & 3); b.take(2); symbol += r; if (r != 3) break; } }
        while (remaining < threshold && threshold > 1) { nbBits--; threshold >>= 1; }
    }
    if (remaining != 1 || symbol > maxSymbol + 1) return 0;
    *maxSymbolPtr = symbol - 1;
    size_t const bytes = (b.used + 7) / 8;
    return bytes <= avail ? bytes : 0;
}

/* Compression table of a normalised distribution that may hold low-probability (-1) symbols: dictionaries and the
 * format's predefined distributions have them (format "FSE decoding table": such a symbol owns one cell at the top of
 * the table, the spread walk steps over that area).  Host code; the kernels build the tables of fresh distributions,
 * which never hold -1, with zbw_fse_buildCTable (zb_entropy.cuh).  The reference's builder is FSE_buildCTable_wksp
 * (lib/compress/fse_compress.c:68). */
void buildCTable(ZbdFseCTable* ct, const short* norm, u32 maxSymbolValue, u32 tableLog)
{
    u32 const size = 1u << tableLog, mask = size - 1u, step = (size >> 1) + (size >> 3) + 3u;
    u32 const nbSym = maxSymbolValue + 1u;
    u8 owner[512];                      /* symbol of every cell */
    u32 weight[64], first[65];
    memset(ct, 0, sizeof(*ct));
    ct->tableLog = tableLog; ct->maxSymbolValue = maxSymbolValue;
    /* cells a symbol owns, and where its sub-states start in nextState[] */
    first[0] = 0;
    for (u32 s = 0; s < nbSym; s++) { weight[s] = norm[s] == -1 ? 1u : (u32)norm[s]; first[s + 1] = first[s] + weight[s]; }
    /* low-probability symbols: the top cells, highest first, in symbol order */
    u32 top = size;
    for (u32 s = 0; s < nbSym; s++) if (norm[s] == -1) owner[--top] = (u8)s;
    /* the walk: every cell below `top` exactly once (step is odd), handed to the other symbols occurrence by occurrence */
    {   u32 cell = 0, s = 0, left = 0;
        for (u32 visited = 0; visited < top; ) {
            while (left == 0) { left = norm[s] > 0 ? (u32)norm[s] : 0u; if (left == 0) s++; }
            if (cell < top) { owner[cell] = (u8)s; visited++; if (--left == 0) s++; }
            cell = (cell + step) & mask;
        }
    }
    /* sub-states in ascending cell order */
    {   u32 given[64];
        for (u32 s = 0; s < nbSym; s++) given[s] = 0;
        for (u32 cell = 0; cell < size; cell++) { u32 const s = owner[cell]; ct->nextState[first[s] + given[s]++] = (u16)(size + cell); }
    }
    /* per-symbol transform: bits shed before a state lands in [weight, 2 * weight), offset of the sub-states */
    for (u32 s = 0; s < nbSym; s++) {
        u32 const n = weight[s];
        if (n == 0) { ct->deltaNbBits[s] = ((tableLog + 1u) << 16) - size; ct->deltaFindState[s] = 0; continue; }
        u32 const shed = n == 1u ? tableLog : tableLog - hb32(n - 1u);
        ct->deltaNbBits[s] = (shed << 16) - (n << shed);
        ct->deltaFindState[s] = (int)first[s] - (int)n;
    }
}

/* Huffman weights compressed with FSE: two interleaved states, stream read backwards (common/fse_decompress.c) */
size_t decodeWeights(u8* out, size_t maxOut, const u8* src, size_t srcSize)
{
    short norm[256]; u32 maxSym = 255, tableLog;
    size_t const hdr = readNCount(norm, &maxSym, &tableLog, src, srcSize);
    struct { u8 sym, nbBits; u16 newState; } dt[64];
    if (hdr == 0 || tableLog > 6) return 0;
    {   u32 const size = 1u << tableLog, mask = size - 1, step = (size >> 1) + (size >> 3) + 3;
        u16 next[256]; u8 spread[64]; u32 high = size - 1, pos = 0;
        for (u32 s = 0; s <= maxSym; s++) { if (norm[s] == -1) { spread[high--] = (u8)s; next[s] = 1; } else next[s] = (u16)norm[s]; }
        for (u32 s = 0; s <= maxSym; s++) for (int i = 0; i < norm[s]; i++) { spread[pos] = (u8)s; do { pos = (pos + step) & mask; } while (pos > high); }
        if (pos != 0) return 0;
        for (u32 u = 0; u < size; u++) {
            u8 const sym = spread[u]; u32 const ns = next[sym]++;
            dt[u].sym = sym; dt[u].nbBits = (u8)(tableLog - hb32(ns)); dt[u].newState = (u16)((ns << dt[u].nbBits) - size);
        }
    }
    const u8* const bs = src + hdr; size_t const n = srcSize - hdr;
    if (n == 0 || bs[n - 1] == 0) return 0;
    long bitpos = (long)(n - 1) * 8 + (long)hb32(bs[n - 1]);
    auto rd = [&](u32 k) { u32 v = 0; for (u32 i = 0; i < k; i++) { long const bp = bitpos - (long)k + (long)i; if (bp >= 0) v |= (u32)((bs[bp >> 3] >> (bp & 7)) & 1) << i; } bitpos -= (long)k; return v; };
    size_t op = 0;
    u32 s1 = rd(tableLog), s2 = rd(tableLog);
    for (;;) {
        if (op + 2 > maxOut) return 0;
        out[op++] = dt[s1].sym; s1 = dt[s1].newState + rd(dt[s1].nbBits);
        if (bitpos < 0) { out[op++] = dt[s2].sym; break; }
        if (op + 2 > maxOut) return 0;
        out[op++] = dt[s2].sym; s2 = dt[s2].newState + rd(dt[s2].nbBits);
        if (bitpos < 0) { out[op++] = dt[s1].sym; break; }
    }
    return op;
}
}   /* namespace */

/* Returns the offset of the dictionary content inside `dict` (0 for raw content / ignored dictionaries:
 * then de->present == 0), or a zstd error code (dictionary_corrupted). */
/* the format's predefined distributions (doc/zstd_compression_format.md "Default Distributions"; RFC 8878 3.1.1.3.2.2):
 * literal lengths and match lengths with 64 states, offsets with 32.  out[0] = LL, out[1] = OF, out[2] = ML. */
extern "C" void zb_buildDefaultTables(ZbdFseCTable* out)
{
    static const short ll[36] = { 4,3,2,2,2,2,2,2, 2,2,2,2,2,1,1,1, 2,2,2,2,2,2,2,2, 2,3,2,1,1,1,1,1, -1,-1,-1,-1 };
    static const short of[29] = { 1,1,1,1,1,1,2,2, 2,1,1,1,1,1,1,1, 1,1,1,1,1,1,1,1, -1,-1,-1,-1,-1 };
    static const short ml[53] = { 1,4,3,2,2,2,2,2, 2,1,1,1,1,1,1,1, 1,1,1,1,1,1,1,1, 1,1,1,1,1,1,1,1,
                                  1,1,1,1,1,1,1,1, 1,1,1,1,1,1,-1,-1, -1,-1,-1,-1,-1 };
    buildCTable(&out[0], ll, 35, 6);
    buildCTable(&out[1], of, 28, 5);
    buildCTable(&out[2], ml, 52, 6);
}

extern "C" size_t zb_loadDictionary(ZbDictEntropy* de, const u8* dict, size_t dictSize)
{
    size_t const corrupted = ZB_ERR(ZB_error_dictionary_corrupted);
    memset(de, 0, sizeof(*de));
    if (!dict || dictSize < 8 || !(dict[0] == 0x37 && dict[1] == 0xA4 && dict[2] == 0x30 && dict[3] == 0xEC)) return 0;
    size_t pos = 8;
    de->dictID = (u32)dict[4] | ((u32)dict[5] << 8) | ((u32)dict[6] << 16) | ((u32)dict[7] << 24);
    {   u8 w[256]; u32 rank[16] = {0}; size_t oSize, iSize; u32 weightTotal = 0;
        if (pos >= dictSize) return corrupted;
        iSize = dict[pos];
        if (iSize >= 128) {
            oSize = iSize - 127; iSize = (oSize + 1) / 2;
            if (pos + 1 + iSize > dictSize || oSize >= 256) return corrupted;
            for (u32 n = 0; n < oSize; n += 2) { w[n] = dict[pos + 1 + n / 2] >> 4; w[n + 1] = dict[pos + 1 + n / 2] & 15; }
        } else {
            if (pos + 1 + iSize > dictSize) return corrupted;
            oSize = decodeWeights(w, 255, dict + pos + 1, iSize);
            if (oSize == 0) return corrupted;
        }
        for (u32 n = 0; n < oSize; n++) { if (w[n] > 12) return corrupted; rank[w[n]]++; weightTotal += (1u << w[n]) >> 1; }
        if (weightTotal == 0) return corrupted;
        u32 const tableLog = hb32(weightTotal) + 1;
        if (tableLog > 12) return corrupted;
        {   u32 const rest = (1u << tableLog) - weightTotal, last = hb32(rest) + 1;
            if ((1u << hb32(rest)) != rest) return corrupted;
            w[oSize] = (u8)last; rank[last]++; }
        if (rank[1] < 2 || (rank[1] & 1)) return corrupted;
        u32 const nbSymbols = (u32)oSize + 1;
        u16 nbPerRank[14] = {0}, valPerRank[14] = {0};
        u8 nbBits[256] = {0};
        for (u32 n = 0; n < nbSymbols; n++) { nbBits[n] = w[n] ? (u8)(tableLog + 1 - w[n]) : 0; nbPerRank[nbBits[n]]++; }
        {   u16 min = 0; for (u32 n = tableLog; n > 0; n--) { valPerRank[n] = min; min += nbPerRank[n]; min >>= 1; } }
        for (u32 n = 0; n < nbSymbols; n++) de->hufEnc[n] = nbBits[n] ? ((u32)valPerRank[nbBits[n]]++ | ((u32)nbBits[n] << 16)) : 0u;
        de->hufMaxSymbol = nbSymbols - 1;
        de->hufRepeat = (rank[0] == 0 && nbSymbols == 256) ? 2u : 1u;          /* zstd_compress.c:4997-5005 */
        pos += iSize + 1;
    }
    {   short ofN[32], mlN[53], llN[36]; u32 ofMax = 31, mlMax = 52, llMax = 35, ofLog, mlLog, llLog; size_t n;
        n = readNCount(ofN, &ofMax, &ofLog, dict + pos, dictSize - pos);
        if (n == 0 || ofLog > 8) return corrupted;
        pos += n;
        buildCTable(&de->fse[1], ofN, 31, ofLog);                               /* all offset symbols, :5020-5026 */
        n = readNCount(mlN, &mlMax, &mlLog, dict + pos, dictSize - pos);
        if (n == 0 || mlLog > 9) return corrupted;
        pos += n;
        buildCTable(&de->fse[2], mlN, mlMax, mlLog);
        {   bool ok = (mlMax >= 52); for (u32 s = 0; ok && s <= 52; s++) if (mlN[s] == 0) ok = false; de->fseRepeat[2] = ok ? 2u : 1u; }
        n = readNCount(llN, &llMax, &llLog, dict + pos, dictSize - pos);
        if (n == 0 || llLog > 9) return corrupted;
        pos += n;
        buildCTable(&de->fse[0], llN, llMax, llLog);
        {   bool ok = (llMax >= 35); for (u32 s = 0; ok && s <= 35; s++) if (llN[s] == 0) ok = false; de->fseRepeat[0] = ok ? 2u : 1u; }
        if (pos + 12 > dictSize) return corrupted;
        size_t const contentSize = dictSize - (pos + 12);
        u32 offcodeMax = 31;
        if (contentSize <= 0xFFFFFFFFu - (128u << 10)) { offcodeMax = hb32((u32)contentSize + (128u << 10)); if (offcodeMax > 31) offcodeMax = 31; }
        {   bool ok = (ofMax >= offcodeMax); for (u32 s = 0; ok && s <= offcodeMax; s++) if (ofN[s] == 0) ok = false; de->fseRepeat[1] = ok ? 2u : 1u; }
        for (int r = 0; r < 3; r++) {
            de->rep[r] = (u32)dict[pos + 4 * r] | ((u32)dict[pos + 4 * r + 1] << 8) | ((u32)dict[pos + 4 * r + 2] << 16) | ((u32)dict[pos + 4 * r + 3] << 24);
            if (de->rep[r] == 0 || de->rep[r] > contentSize) return corrupted;
        }
        pos += 12;
    }
    de->present = 1;
    return pos;
}
