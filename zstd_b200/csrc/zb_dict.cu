/* zb_dict.cu — host side: parsing a dictionary (no device code here).
 * Replaces ZSTD_compress_insertDictionary / ZSTD_loadZstdDictionary / ZSTD_loadCEntropy
 * (lib/compress/zstd_compress.c:5119-5156, :5087-5115, :4987-5076) for the simple API:
 *   < 8 bytes                -> ignored (:5132)
 *   no magic 0xEC30A437      -> raw content (:5143-5148)
 *   magic                    -> dictID, Huffman table (HUF_readCTable huf_compress.c:292), OF/ML/LL FSE tables
 *                               (FSE_buildCTable fse_compress.c:68), repeat modes (ZSTD_dictNCountRepeat :4973),
 *                               3 repcodes, then content.
 * The format itself (layout, table descriptions, Huffman weights) is read by the decoder's zbd_parseDict,
 * zbd_readHufWeights and zbd_readNCount (zb_decode_core.cuh), with the compressor's limits; this file turns what they
 * read into compression tables.
 */
#include <string.h>
#include "zb_common.h"
#include "zb_kernels.h"
#include "zb_decode_core.cuh"

namespace {
/* the compressor's limits of a Huffman tree description: weights and table log up to HUF_TABLELOG_MAX (huf.h), and the
 * weights' FSE description over all 256 symbols (fse_decompress.c:252) */
constexpr u32 HUF_LOG_MAX = 12u, HUF_WEIGHT_FSE_MAXSYM = 255u;

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
        u32 const shed = n == 1u ? tableLog : tableLog - zbd_hb(n - 1u);
        ct->deltaNbBits[s] = (shed << 16) - (n << shed);
        ct->deltaFindState[s] = (int)first[s] - (int)n;
    }
}

/* FSE_repeat of a dictionary's table (ZSTD_dictNCountRepeat, zstd_compress.c:4973): valid when every symbol up to
 * maxSymbolValue may be encoded with it, else check */
u32 fseRepeat(const short* norm, u32 tableMaxSym, u32 maxSymbolValue)
{
    if (tableMaxSym < maxSymbolValue) return 1u;
    for (u32 s = 0; s <= maxSymbolValue; s++) if (norm[s] == 0) return 1u;
    return 2u;
}
}   /* namespace */

/* the format's predefined distributions (zbd_defaultNorm): literal lengths and match lengths with 64 states, offsets
 * with 32.  out[0] = LL, out[1] = OF, out[2] = ML. */
extern "C" void zb_buildDefaultTables(ZbdFseCTable* out)
{
    u32 const log[3] = { ZBD_LL_DEFAULT_LOG, ZBD_OF_DEFAULT_LOG, ZBD_ML_DEFAULT_LOG };
    u32 const maxSym[3] = { ZBD_LL_MAXSYM, ZBD_OF_DEFAULT_MAXSYM, ZBD_ML_MAXSYM };
    for (u32 st = 0; st < 3u; st++) {
        short norm[ZBD_ML_MAXSYM + 1];
        for (u32 s = 0; s <= maxSym[st]; s++) norm[s] = zbd_defaultNorm(st, s);
        buildCTable(&out[st], norm, maxSym[st], log[st]);
    }
}

/* Returns the offset of the dictionary content inside `dict` (0 for raw content / ignored dictionaries:
 * then de->present == 0), or a zstd error code (dictionary_corrupted). */
extern "C" size_t zb_loadDictionary(ZbDictEntropy* de, const u8* dict, size_t dictSize)
{
    size_t const corrupted = ZB_ERR(ZB_error_dictionary_corrupted);
    memset(de, 0, sizeof(*de));
    if (!dict) return 0;
    ZbdDictInfo di;
    if (zbd_parseDict(&di, dict, dictSize, HUF_LOG_MAX, HUF_WEIGHT_FSE_MAXSYM)) return corrupted;
    if (!di.entropy) return 0;
    de->dictID = di.dictID;
    /* zbd_parseDict has read every section below with the same limits: reading them again cannot fail */
    {   u8 w[256]; u32 nbSymbols, tableLog, fse[64]; short norm[256]; u16 next[256]; u32 rank[HUF_LOG_MAX + 1] = {0};
        zbd_readHufWeights(w, &nbSymbols, &tableLog, dict + di.hufOff, di.hufLen, fse, norm, next, HUF_LOG_MAX, HUF_WEIGHT_FSE_MAXSYM);
        for (u32 n = 0; n < nbSymbols; n++) rank[w[n]]++;
        if (rank[1] < 2 || (rank[1] & 1)) return corrupted;                  /* HUF_readStats, entropy_common.c */
        u16 nbPerRank[HUF_LOG_MAX + 2] = {0}, valPerRank[HUF_LOG_MAX + 2] = {0};
        u8 nbBits[256] = {0};
        for (u32 n = 0; n < nbSymbols; n++) { nbBits[n] = w[n] ? (u8)(tableLog + 1 - w[n]) : 0; nbPerRank[nbBits[n]]++; }
        {   u16 min = 0; for (u32 n = tableLog; n > 0; n--) { valPerRank[n] = min; min += nbPerRank[n]; min >>= 1; } }
        for (u32 n = 0; n < nbSymbols; n++) de->hufEnc[n] = nbBits[n] ? ((u32)valPerRank[nbBits[n]]++ | ((u32)nbBits[n] << 16)) : 0u;
        de->hufMaxSymbol = nbSymbols - 1;
        de->hufRepeat = (rank[0] == 0 && nbSymbols == 256) ? 2u : 1u;          /* zstd_compress.c:4997-5005 */
    }
    size_t const contentSize = dictSize - di.contentOff;
    u32 offcodeMax = 31;
    if (contentSize <= 0xFFFFFFFFu - (128u << 10)) { offcodeMax = zbd_hb((u32)contentSize + (128u << 10)); if (offcodeMax > 31) offcodeMax = 31; }
    for (u32 st = 0; st < 3u; st++) {
        short norm[ZBD_ML_MAXSYM + 1]; u32 maxSym, log;
        zbd_readNCount(norm, &maxSym, &log, zbd_seqMaxSym(st), zbd_seqMaxLog(st), dict + di.fseOff[st], di.fseLen[st]);
        if (st == 1u) {
            buildCTable(&de->fse[1], norm, ZBD_OF_MAXSYM, log);              /* all offset symbols, :5020-5026 */
            de->fseRepeat[1] = fseRepeat(norm, maxSym, offcodeMax);
        } else {
            buildCTable(&de->fse[st], norm, maxSym, log);
            de->fseRepeat[st] = fseRepeat(norm, maxSym, zbd_seqMaxSym(st));
        }
    }
    for (u32 r = 0; r < 3u; r++) de->rep[r] = di.rep[r];
    de->present = 1;
    return di.contentOff;
}
