/* zb_dict.c — oracle: loading a zstd-format dictionary's entropy tables (TEST INFRASTRUCTURE ONLY).
 * Restates ZSTD_loadCEntropy (lib/compress/zstd_compress.c:4987-5076): Huffman table
 * (HUF_readCTable huf_compress.c:292-340, HUF_readStats common/entropy_common.c:236-330 incl. the FSE
 * decoding of the weights, common/fse_decompress.c), three FSE tables (FSE_readNCount
 * entropy_common.c:42-188, FSE_buildCTable), repeat modes (ZSTD_dictNCountRepeat :4973-4985) and the
 * three start repcodes.
 */
#include <string.h>
#include "zb_oracle.h"

static inline u32 hb32(u32 v) { return 31u - (u32)__builtin_clz(v); }

/* little-endian forward bit reader */
typedef struct { const u8* p; size_t avail, pos; u64 bits; u32 nb; size_t used; } fbits;
static void fb_need(fbits* b, u32 k) { while (b->nb < k) { u64 const byte = b->pos < b->avail ? b->p[b->pos] : 0; b->bits |= byte << b->nb; b->nb += 8; b->pos++; } }
static void fb_take(fbits* b, u32 k) { b->bits >>= k; b->nb -= k; b->used += k; }

/* normalised counts of an FSE table description (doc/zstd_compression_format.md:1063).  Returns bytes read, 0 if malformed. */
size_t zbo_readNCount(int16_t* norm, u32* maxSymbolPtr, u32* tableLogPtr, const u8* p, size_t avail)
{
    fbits b = { p, avail, 0, 0, 0, 0 };
    u32 const maxSymbol = *maxSymbolPtr;
    u32 tableLog, symbol = 0;
    int remaining, threshold, nbBits;
    memset(norm, 0, (maxSymbol + 1) * sizeof(norm[0]));
    fb_need(&b, 4); tableLog = (u32)(b.bits & 15) + 5; fb_take(&b, 4);
    if (tableLog > 15) return 0;
    *tableLogPtr = tableLog;
    remaining = (1 << tableLog) + 1; threshold = 1 << tableLog; nbBits = (int)tableLog + 1;
    while (remaining > 1 && symbol <= maxSymbol) {
        int const max = (2 * threshold - 1) - remaining;
        int count;
        fb_need(&b, (u32)nbBits);
        if ((int)(b.bits & (u32)(threshold - 1)) < max) { count = (int)(b.bits & (u32)(threshold - 1)); fb_take(&b, (u32)nbBits - 1); }
        else { count = (int)(b.bits & (u32)(2 * threshold - 1)); if (count >= threshold) count -= max; fb_take(&b, (u32)nbBits); }
        count--;
        remaining -= count < 0 ? -count : count;
        norm[symbol++] = (int16_t)count;
        if (count == 0) {
            while (1) { u32 r; fb_need(&b, 2); r = (u32)(b.bits & 3); fb_take(&b, 2); symbol += r; if (r != 3) break; }
        }
        while (remaining < threshold && threshold > 1) { nbBits--; threshold >>= 1; }
    }
    if (remaining != 1 || symbol > maxSymbol + 1) return 0;
    *maxSymbolPtr = symbol - 1;
    {   size_t const bytes = (b.used + 7) / 8;
        return bytes <= avail ? bytes : 0; }
}

/* FSE decoding of the Huffman weights: two interleaved states, stream read backwards
 * (common/fse_decompress.c:FSE_buildDTable_internal, FSE_decompress_usingDTable_generic). */
static size_t fse_decodeWeights(u8* out, size_t maxOut, const u8* src, size_t srcSize)
{
    int16_t norm[256]; u32 maxSym = 255, tableLog;
    size_t const hdr = zbo_readNCount(norm, &maxSym, &tableLog, src, srcSize);
    struct { u8 sym; u8 nbBits; u16 newState; } dt[64];
    if (hdr == 0 || tableLog > 6) return 0;
    {   u32 const size = 1u << tableLog, mask = size - 1, step = (size >> 1) + (size >> 3) + 3;
        u16 next[256]; u8 spread[64]; u32 high = size - 1, pos = 0, s, u;
        for (s = 0; s <= maxSym; s++) { if (norm[s] == -1) { spread[high--] = (u8)s; next[s] = 1; } else next[s] = (u16)norm[s]; }
        for (s = 0; s <= maxSym; s++) for (int i = 0; i < norm[s]; i++) { spread[pos] = (u8)s; do { pos = (pos + step) & mask; } while (pos > high); }
        if (pos != 0) return 0;
        for (u = 0; u < size; u++) {
            u8 const sym = spread[u]; u32 const ns = next[sym]++;
            dt[u].sym = sym; dt[u].nbBits = (u8)(tableLog - hb32(ns)); dt[u].newState = (u16)((ns << dt[u].nbBits) - size);
        }
    }
    {   const u8* const bs = src + hdr; size_t const n = srcSize - hdr;
        long bitpos; size_t op = 0; u32 s1, s2;
        if (n == 0 || bs[n - 1] == 0) return 0;
        bitpos = (long)(n - 1) * 8 + (long)hb32(bs[n - 1]);          /* bits below the end mark */
#define RD(k) ({ u32 v_ = 0; for (u32 i_ = 0; i_ < (k); i_++) { long const bp_ = bitpos - (long)(k) + (long)i_; if (bp_ >= 0) v_ |= (u32)((bs[bp_ >> 3] >> (bp_ & 7)) & 1) << i_; } bitpos -= (long)(k); v_; })
        s1 = RD(tableLog); s2 = RD(tableLog);
        if (bitpos < 0) return 0;                                         /* shorter than its two initial states (fse_decompress.c:193) */
        while (1) {
            if (op + 2 > maxOut) return 0;
            out[op++] = dt[s1].sym; s1 = dt[s1].newState + RD(dt[s1].nbBits);
            if (bitpos < 0) { out[op++] = dt[s2].sym; break; }
            if (op + 2 > maxOut) return 0;
            out[op++] = dt[s2].sym; s2 = dt[s2].newState + RD(dt[s2].nbBits);
            if (bitpos < 0) { out[op++] = dt[s1].sym; break; }
        }
#undef RD
        return op;
    }
}

/* returns the offset of the dictionary content (> 0), 0 for "raw content / no dictionary", or an error */
size_t zbo_loadDictEntropy(zbo_dict_entropy* de, const u8* dict, size_t dictSize)
{
    size_t pos = 8;
    memset(de, 0, sizeof(*de));
    if (dictSize < 8 || !(dict[0] == 0x37 && dict[1] == 0xA4 && dict[2] == 0x30 && dict[3] == 0xEC)) return 0;
    de->dictID = (u32)dict[4] | ((u32)dict[5] << 8) | ((u32)dict[6] << 16) | ((u32)dict[7] << 24);
    /* ---- Huffman table ---- */
    {   u8 w[256]; u32 rank[16] = {0}; size_t oSize, iSize; u32 weightTotal = 0, tableLog, n;
        if (pos >= dictSize) return ZBO_ERR(ZBO_error_dictionary_corrupted);
        iSize = dict[pos];
        if (iSize >= 128) {
            oSize = iSize - 127; iSize = (oSize + 1) / 2;
            if (pos + 1 + iSize > dictSize || oSize >= 256) return ZBO_ERR(ZBO_error_dictionary_corrupted);
            for (n = 0; n < oSize; n += 2) { w[n] = dict[pos + 1 + n / 2] >> 4; w[n + 1] = dict[pos + 1 + n / 2] & 15; }
        } else {
            if (pos + 1 + iSize > dictSize) return ZBO_ERR(ZBO_error_dictionary_corrupted);
            oSize = fse_decodeWeights(w, 255, dict + pos + 1, iSize);
            if (oSize == 0) return ZBO_ERR(ZBO_error_dictionary_corrupted);
        }
        for (n = 0; n < oSize; n++) { if (w[n] > 12) return ZBO_ERR(ZBO_error_dictionary_corrupted); rank[w[n]]++; weightTotal += (1u << w[n]) >> 1; }
        if (weightTotal == 0) return ZBO_ERR(ZBO_error_dictionary_corrupted);
        tableLog = hb32(weightTotal) + 1;
        if (tableLog > 12) return ZBO_ERR(ZBO_error_dictionary_corrupted);
        {   u32 const rest = (1u << tableLog) - weightTotal, last = hb32(rest) + 1;
            if ((1u << hb32(rest)) != rest) return ZBO_ERR(ZBO_error_dictionary_corrupted);
            w[oSize] = (u8)last; rank[last]++; }
        if (rank[1] < 2 || (rank[1] & 1)) return ZBO_ERR(ZBO_error_dictionary_corrupted);
        {   u32 const nbSymbols = (u32)oSize + 1;
            u16 nbPerRank[14] = {0}, valPerRank[14] = {0};
            de->huf.tableLog = tableLog; de->huf.maxSymbolValue = nbSymbols - 1;
            for (n = 0; n < nbSymbols; n++) { de->huf.nbBits[n] = w[n] ? (u8)(tableLog + 1 - w[n]) : 0; nbPerRank[de->huf.nbBits[n]]++; }
            {   u16 min = 0; for (n = tableLog; n > 0; n--) { valPerRank[n] = min; min += nbPerRank[n]; min >>= 1; } }
            for (n = 0; n < nbSymbols; n++) de->huf.code[n] = de->huf.nbBits[n] ? valPerRank[de->huf.nbBits[n]]++ : 0;
            de->hufRepeat = (rank[0] == 0 && nbSymbols == 256) ? 2 : 1;          /* zstd_compress.c:4997-5005 */
        }
        pos += iSize + 1;
    }
    /* ---- FSE tables: offsets, match lengths, literal lengths ---- */
    {   int16_t ofN[32], mlN[53], llN[36]; u32 ofMax = 31, mlMax = 52, llMax = 35, ofLog, mlLog, llLog; size_t n;
        n = zbo_readNCount(ofN, &ofMax, &ofLog, dict + pos, dictSize - pos);
        if (n == 0 || ofLog > 8) return ZBO_ERR(ZBO_error_dictionary_corrupted);
        pos += n;
        zbo_fse_buildCTable(&de->fse[1], ofN, 31, ofLog);                           /* all offset symbols, :5020-5026 */
        n = zbo_readNCount(mlN, &mlMax, &mlLog, dict + pos, dictSize - pos);
        if (n == 0 || mlLog > 9) return ZBO_ERR(ZBO_error_dictionary_corrupted);
        pos += n;
        zbo_fse_buildCTable(&de->fse[2], mlN, mlMax, mlLog);
        {   u32 s, ok = (mlMax >= 52); for (s = 0; ok && s <= 52; s++) if (mlN[s] == 0) ok = 0; de->fseRepeat[2] = ok ? 2 : 1; }
        n = zbo_readNCount(llN, &llMax, &llLog, dict + pos, dictSize - pos);
        if (n == 0 || llLog > 9) return ZBO_ERR(ZBO_error_dictionary_corrupted);
        pos += n;
        zbo_fse_buildCTable(&de->fse[0], llN, llMax, llLog);
        {   u32 s, ok = (llMax >= 35); for (s = 0; ok && s <= 35; s++) if (llN[s] == 0) ok = 0; de->fseRepeat[0] = ok ? 2 : 1; }
        if (pos + 12 > dictSize) return ZBO_ERR(ZBO_error_dictionary_corrupted);
        {   size_t const contentSize = dictSize - (pos + 12);
            u32 offcodeMax = 31, s, ok;
            if (contentSize <= 0xFFFFFFFFu - (128u << 10)) { offcodeMax = hb32((u32)contentSize + (128u << 10)); if (offcodeMax > 31) offcodeMax = 31; }
            ok = (ofMax >= offcodeMax); for (s = 0; ok && s <= offcodeMax; s++) if (ofN[s] == 0) ok = 0;
            de->fseRepeat[1] = ok ? 2 : 1;
            for (int r = 0; r < 3; r++) {
                de->rep[r] = (u32)dict[pos + 4 * r] | ((u32)dict[pos + 4 * r + 1] << 8) | ((u32)dict[pos + 4 * r + 2] << 16) | ((u32)dict[pos + 4 * r + 3] << 24);
                if (de->rep[r] == 0 || de->rep[r] > contentSize) return ZBO_ERR(ZBO_error_dictionary_corrupted);
            }
        }
        pos += 12;
    }
    de->present = 1;
    return pos;
}
