/* zb_decode_core.cuh — format-level pieces of the decompressor, written from the format specification
 * (doc/zstd_compression_format.md) as host+device functions: frame / block / section headers, the two
 * bit readers, FSE table descriptions and decoding tables, Huffman tree descriptions and decoding tables, the sequence
 * bitstream.  The CUDA kernels of zb_decode.cu call them per warp / per lane; tests/host_decode.cpp compiles the same
 * functions for the CPU so that this logic is checked against the reference encoder's frames without a GPU (the
 * reference's counterparts: lib/decompress/zstd_decompress.c, zstd_decompress_block.c, huf_decompress.c,
 * lib/common/entropy_common.c, fse_decompress.c — none of their code is used here).
 */
#ifndef ZB_DECODE_CORE_CUH
#define ZB_DECODE_CORE_CUH
#include "zb_common.h"
#include <string.h>

#ifdef __CUDACC__
#define ZBD_HD __host__ __device__ __forceinline__
#define ZBD_HDN static __host__ __device__        /* internal linkage: more than one .cu file includes this header */
#else
#define ZBD_HD static inline
#define ZBD_HDN static
#endif

#define ZBD_OK 0u
#define ZBD_CORRUPT 20u                /* ZSTD_error_corruption_detected */
#define ZBD_NONE 0xFFFFFFFFu
#define ZBD_DICT 0xFFFFFFFEu            /* "the table the dictionary brings" where a block index is expected */

#define ZBD_MAGIC 0xFD2FB528u
#define ZBD_MAGIC_SKIPPABLE 0x184D2A50u   /* .. 0x184D2A5F */
#define ZBD_HUF_LOG_MAX 11u
#define ZBD_HUF_WEIGHT_MAXSYM 12u       /* largest symbol the FSE description of Huffman weights may hold */
#define ZBD_LL_LOG_MAX 9u
#define ZBD_OF_LOG_MAX 8u
#define ZBD_ML_LOG_MAX 9u
#define ZBD_LL_MAXSYM 35u
#define ZBD_OF_MAXSYM 31u
#define ZBD_ML_MAXSYM 52u

ZBD_HD u32 zbd_hb(u32 v)               /* index of the highest set bit, v != 0 */
{
#ifdef __CUDA_ARCH__
    return 31u - (u32)__clz((int)v);
#else
    return 31u - (u32)__builtin_clz(v);
#endif
}

/* ---- byte access that never leaves [p, p + n): the compressed input has no padding ---- */
ZBD_HD u32 zbd_le(const u8* p, u32 n) { u32 v = 0; for (u32 i = 0; i < n; i++) v |= (u32)p[i] << (8u * i); return v; }
/* up to 8 bytes at p[idx ..), bytes at or past `size` read as zero */
ZBD_HD u64 zbd_load64(const u8* p, u32 idx, u32 size)
{
    u64 v = 0;
#ifdef __CUDA_ARCH__
    if (idx + 8u <= size) {
        const u8* const a = p + idx;
        const u32* q = (const u32*)((uintptr_t)a & ~(uintptr_t)3);
        u32 const sh = ((u32)(uintptr_t)a & 3u) * 8u;
        u32 const w0 = q[0], w1 = q[1], w2 = sh ? q[2] : 0u;      /* the third word only when it holds a requested byte */
        return ((u64)__funnelshift_r(w1, w2, sh) << 32) | __funnelshift_r(w0, w1, sh);
    }
#else
    if (idx + 8u <= size) { memcpy(&v, p + idx, 8); return v; }
#endif
    for (u32 i = 0; i < 8u && idx + i < size; i++) v |= (u64)p[idx + i] << (8u * i);
    return v;
}

/* ---- backward bit reader (format: "Bitstream" — Huffman streams and the sequence section are written forward and
 * read from their last byte, whose highest set bit marks the end).  pos = unread bits; bits below position 0 read
 * as zero and make pos negative, which the callers treat as the format says (end of an FSE weight stream, else
 * corruption). ---- */
typedef struct { const u8* base; u32 size; int pos; u64 win; int winLo; } ZbdBack;
ZBD_HD u32 zbd_back_init(ZbdBack* b, const u8* base, u32 size)
{
    b->base = base; b->size = size; b->win = 0; b->winLo = 0x40000000; b->pos = 0;
    if (size == 0) return ZBD_CORRUPT;
    u32 const last = base[size - 1];
    if (last == 0) return ZBD_CORRUPT;
    b->pos = (int)(8u * (size - 1u) + zbd_hb(last));
    return ZBD_OK;
}
/* the next n bits (n <= 32) without consuming them */
ZBD_HD u32 zbd_back_peek(ZbdBack* b, u32 n)
{
    int const lo = b->pos - (int)n;                               /* lowest wanted bit */
    if (lo < 0) {                                                 /* fewer than n bits left: zeros are appended */
        if (b->pos <= 0) return 0;
        u64 const w = zbd_load64(b->base, 0, b->size);
        u32 const have = (u32)b->pos;
        u32 const v = (u32)(w & ((have >= 32u) ? 0xFFFFFFFFull : ((1ull << have) - 1ull)));
        return (v << (n - have)) & (n >= 32u ? 0xFFFFFFFFu : ((1u << n) - 1u));
    }
    if (lo < b->winLo || b->pos > b->winLo + 64) {                /* window does not cover [lo, pos) */
        int wl = b->pos - 57; if (wl < 0) wl = 0;
        wl &= ~7;
        b->winLo = wl;
        b->win = zbd_load64(b->base, (u32)wl >> 3, b->size);
    }
    u64 const v = b->win >> (u32)(lo - b->winLo);
    return (u32)v & (n >= 32u ? 0xFFFFFFFFu : ((1u << n) - 1u));
}
ZBD_HD u32 zbd_back_read(ZbdBack* b, u32 n) { if (n == 0) return 0; u32 const v = zbd_back_peek(b, n); b->pos -= (int)n; return v; }

/* ---- forward bit reader (FSE table descriptions) ---- */
typedef struct { const u8* base; u32 size; u32 pos; } ZbdFwd;
ZBD_HD u32 zbd_fwd_peek(const ZbdFwd* f, u32 n)
{
    u64 const w = zbd_load64(f->base, f->pos >> 3, f->size);
    return (u32)(w >> (f->pos & 7u)) & ((1u << n) - 1u);          /* n <= 16 */
}

/* ---- frame header (format: "Frame_Header") ---- */
typedef struct {
    u32 headerSize;        /* magic + descriptor + optional fields */
    u32 windowLog;         /* 0 when Single_Segment (the window is the content) */
    u64 windowSize;
    u64 contentSize;       /* ~0 when absent */
    u32 dictID;
    u32 hasChecksum;
    u32 skippable;         /* a skippable frame: headerSize = 8, contentSize = its payload size */
} ZbdFrameHeader;
#define ZBD_CONTENTSIZE_UNKNOWN 0xFFFFFFFFFFFFFFFFull

/* returns 0, ZBD_CORRUPT, 10 (prefix_unknown) or 72 (srcSize_wrong: truncated) */
ZBD_HDN u32 zbd_readFrameHeader(ZbdFrameHeader* h, const u8* src, u64 size)
{
    memset(h, 0, sizeof(*h));
    if (size < 5) return size < 4 ? 72u : (zbd_le(src, 4) == ZBD_MAGIC ? 72u : ((zbd_le(src, 4) & 0xFFFFFFF0u) == ZBD_MAGIC_SKIPPABLE ? 72u : 10u));
    u32 const magic = zbd_le(src, 4);
    if ((magic & 0xFFFFFFF0u) == ZBD_MAGIC_SKIPPABLE) {
        if (size < 8) return 72u;
        h->skippable = 1; h->headerSize = 8; h->contentSize = zbd_le(src + 4, 4);
        return ZBD_OK;
    }
    if (magic != ZBD_MAGIC) return 10u;
    u32 const fhd = src[4];
    u32 const fcsFlag = fhd >> 6, single = (fhd >> 5) & 1u, dictFlag = fhd & 3u;
    if (fhd & 0x08u) return 14u;                                  /* reserved bit: frameParameter_unsupported */
    u32 const dictBytes = dictFlag == 3u ? 4u : dictFlag;
    u32 const fcsBytes = fcsFlag == 0u ? single : (fcsFlag == 1u ? 2u : (fcsFlag == 2u ? 4u : 8u));
    u32 const hs = 5u + (single ? 0u : 1u) + dictBytes + fcsBytes;
    if (size < hs) return 72u;
    u32 p = 5;
    h->hasChecksum = (fhd >> 2) & 1u;
    if (!single) {
        u32 const wd = src[p++];
        u32 const wl = 10u + (wd >> 3);
        if (wl > 31u) return 16u;                                 /* frameParameter_windowTooLarge */
        u64 const base = 1ull << wl;
        h->windowLog = wl; h->windowSize = base + (base >> 3) * (wd & 7u);
    }
    h->dictID = dictBytes ? zbd_le(src + p, dictBytes) : 0u; p += dictBytes;
    h->contentSize = ZBD_CONTENTSIZE_UNKNOWN;
    if (fcsBytes == 1u) h->contentSize = src[p];
    else if (fcsBytes == 2u) h->contentSize = (u64)zbd_le(src + p, 2) + 256u;
    else if (fcsBytes == 4u) h->contentSize = zbd_le(src + p, 4);
    else if (fcsBytes == 8u) h->contentSize = (u64)zbd_le(src + p, 4) | ((u64)zbd_le(src + p + 4, 4) << 32);
    if (single) h->windowSize = h->contentSize;
    h->headerSize = hs;
    return ZBD_OK;
}

/* ---- one frame's sizes from its frame and block headers alone (the reference's ZSTD_findFrameSizeInfo,
 * zstd_decompress.c:732-790): nothing behind a block header is read, no block size is checked against the window, and
 * windows up to 2^31 are read although the decoder refuses those above 2^27. ---- */
#define ZBD_CONTENTSIZE_ERROR 0xFFFFFFFFFFFFFFFEull
typedef struct {
    u64 cSize;             /* bytes of the frame incl. header and checksum */
    u64 contentSize;       /* the header's content size (ZBD_CONTENTSIZE_UNKNOWN if absent), 0 for a skippable frame,
                              ZBD_CONTENTSIZE_ERROR when the header cannot be read */
    u64 bound;             /* the content size if stated, else nbBlocks x min(window, 128 KiB); 0 for a skippable frame */
} ZbdFrameSizeInfo;
/* returns 0 or the error code of ZSTD_findFrameCompressedSize: those of zbd_readFrameHeader, 20 for a reserved block type,
 * 72 (srcSize_wrong) for a frame cut short.  A skippable frame that states 0xFFFFFFF8 bytes or more gets contentSize and
 * bound ZBD_CONTENTSIZE_ERROR: the reference's 32-bit frame size wraps there and its size readers refuse the frame. */
ZBD_HDN u32 zbd_frameSizeInfo(ZbdFrameSizeInfo* fi, const u8* src, u64 size)
{
    fi->cSize = 0; fi->contentSize = ZBD_CONTENTSIZE_ERROR; fi->bound = 0;
    ZbdFrameHeader h;
    u32 const e = zbd_readFrameHeader(&h, src, size);
    if (e) return e;
    if (h.skippable) {
        bool const wraps = h.contentSize > 0xFFFFFFF7ull;
        fi->contentSize = fi->bound = wraps ? ZBD_CONTENTSIZE_ERROR : 0u;
        if (8u + h.contentSize > size) return 72u;
        fi->cSize = 8u + h.contentSize;
        return ZBD_OK;
    }
    fi->contentSize = h.contentSize;
    u64 p = h.headerSize, nbBlocks = 0;
    while (true) {
        if (p + 3u > size) return 72u;
        u32 const bh = zbd_le(src + p, 3);
        u32 const type = (bh >> 1) & 3u;
        if (type == 3u) return ZBD_CORRUPT;
        p += 3u + (type == ZB_BT_RLE ? 1u : (bh >> 3));
        if (p > size) return 72u;
        nbBlocks++;
        if (bh & 1u) break;
    }
    if (h.hasChecksum) { p += 4u; if (p > size) return 72u; }
    u64 const blockMax = h.windowSize < ZB_BLOCK_MAX ? h.windowSize : ZB_BLOCK_MAX;
    fi->cSize = p;
    fi->bound = h.contentSize != ZBD_CONTENTSIZE_UNKNOWN ? h.contentSize : nbBlocks * blockMax;
    return ZBD_OK;
}

/* the reference's ZSTD_findDecompressedSize (zstd_decompress.c:641-678): the content sizes of the frames in src[0, size)
 * summed, skippable frames 0; ZBD_CONTENTSIZE_UNKNOWN at the first frame that states none; ZBD_CONTENTSIZE_ERROR for a bad
 * header or block-header chain, trailing bytes, or a sum past 2^64 */
ZBD_HDN u64 zbd_findDecompressedSize(const u8* src, u64 size)
{
    u64 total = 0;
    while (size >= 5u) {
        ZbdFrameSizeInfo fi;
        u32 const e = zbd_frameSizeInfo(&fi, src, size);
        if (fi.contentSize >= ZBD_CONTENTSIZE_ERROR) return fi.contentSize;      /* the header decides before the blocks do */
        if (total + fi.contentSize < total) return ZBD_CONTENTSIZE_ERROR;
        total += fi.contentSize;
        if (e) return ZBD_CONTENTSIZE_ERROR;
        src += fi.cSize; size -= fi.cSize;
    }
    return size ? ZBD_CONTENTSIZE_ERROR : total;
}

/* the reference's ZSTD_decompressBound (zstd_decompress.c:805-834): the frames' bounds summed (modulo 2^64, as there) */
ZBD_HDN u64 zbd_decompressBound(const u8* src, u64 size)
{
    u64 bound = 0;
    while (size > 0) {
        ZbdFrameSizeInfo fi;
        if (zbd_frameSizeInfo(&fi, src, size) || fi.bound == ZBD_CONTENTSIZE_ERROR) return ZBD_CONTENTSIZE_ERROR;
        src += fi.cSize; size -= fi.cSize;
        bound += fi.bound;
    }
    return bound;
}

/* ---- one block as the walker describes it to the kernels ---- */
typedef struct {
    u64 srcOff;            /* first byte of the block's content (behind its 3-byte header) in the compressed input */
    u32 cSize;             /* bytes of content (1 for an RLE block) */
    u32 type;              /* ZB_BT_RAW / ZB_BT_RLE / ZB_BT_COMPRESSED */
    u32 rawSize;           /* regenerated size of a raw / RLE block */
    u32 frame;
    u32 flags;             /* ZB_FLAG_FIRST / ZB_FLAG_LAST */
    /* literals section (compressed blocks) */
    u32 litType;           /* 0 raw, 1 RLE, 2 compressed, 3 treeless */
    u32 litRegen, litComp; /* regenerated / stored size */
    u32 litHdr;            /* bytes of the section header */
    u32 litStreams;        /* 1 or 4 */
    u32 hufSrc;            /* block whose tree description the literals use (itself for type 2), ZBD_NONE if none */
    /* sequences section */
    u32 seqOff;            /* from srcOff to the section's first byte */
    u32 seqHdr;            /* bytes of Number_of_Sequences + the modes byte */
    u32 nbSeq;
    u32 mode[3];           /* 0 = LL, 1 = OF, 2 = ML: 0 predefined, 1 RLE, 2 compressed, 3 repeat */
    u32 eff[3];            /* what a stream finally uses once repeat chains are resolved: 0 predefined, 1 RLE, 2 compressed */
    u32 fseSrc[3];         /* block whose sequences section holds that RLE byte / table description (itself unless repeat) */
    u32 blockMax;          /* Block_Maximum_Size of its frame, min(window, 128 KiB): bounds the block's regenerated size */
    u64 litPos;            /* where the block's literals go in the literal workspace (multiples of 16) */
    u64 seqPos;            /* index of its first decoded sequence in the sequence workspace */
} ZbdBlock;

typedef struct {
    u64 srcOff;            /* first byte of the frame (its magic number) */
    u64 cSize;             /* bytes of the whole frame incl. header and checksum */
    u64 contentSize;       /* from the header, ZBD_CONTENTSIZE_UNKNOWN if absent */
    u64 windowSize;
    u32 firstBlock, nbBlocks;
    u32 hasChecksum;       /* the 4 bytes behind the last block */
    u32 dictID;
} ZbdFrame;

/* literals section header (format: "Literals_Section_Header") at p[0 .. avail) */
ZBD_HD u32 zbd_readLitHeader(ZbdBlock* b, const u8* p, u32 avail)
{
    if (avail < 1) return ZBD_CORRUPT;
    u32 const b0 = p[0], type = b0 & 3u, fmt = (b0 >> 2) & 3u;
    b->litType = type; b->litStreams = 1;
    if (type < 2u) {
        u32 const hs = (fmt & 1u) == 0u ? 1u : (fmt == 1u ? 2u : 3u);
        if (avail < hs) return ZBD_CORRUPT;
        b->litRegen = hs == 1u ? (b0 >> 3) : (zbd_le(p, hs) >> 4);
        b->litComp = type == 0u ? b->litRegen : 1u;
        b->litHdr = hs;
    } else {
        u32 const hs = fmt < 2u ? 3u : (fmt == 2u ? 4u : 5u);
        if (avail < hs) return ZBD_CORRUPT;
        u32 const v = zbd_le(p, hs > 4u ? 4u : hs);
        if (hs == 3u) { b->litRegen = (v >> 4) & 0x3FFu; b->litComp = (v >> 14) & 0x3FFu; }
        else if (hs == 4u) { b->litRegen = (v >> 4) & 0x3FFFu; b->litComp = v >> 18; }
        else { b->litRegen = (v >> 4) & 0x3FFFFu; b->litComp = (v >> 22) + ((u32)p[4] << 10); }
        b->litStreams = fmt == 0u ? 1u : 4u;
        b->litHdr = hs;
    }
    if (b->litRegen > ZB_BLOCK_MAX) return ZBD_CORRUPT;
    if (b->litHdr + b->litComp > avail) return ZBD_CORRUPT;
    return ZBD_OK;
}

/* sequences section header (format: "Sequences_Section_Header") at p[0 .. avail) */
ZBD_HD u32 zbd_readSeqHeader(ZbdBlock* b, const u8* p, u32 avail)
{
    if (avail < 1) return ZBD_CORRUPT;
    u32 const b0 = p[0];
    b->mode[0] = b->mode[1] = b->mode[2] = 0;
    u32 hs;
    if (b0 < 128u) { b->nbSeq = b0; hs = 1; }
    else if (b0 < 255u) { if (avail < 2) return ZBD_CORRUPT; b->nbSeq = ((b0 - 128u) << 8) + p[1]; hs = 2; }
    else { if (avail < 3) return ZBD_CORRUPT; b->nbSeq = (u32)p[1] + ((u32)p[2] << 8) + 0x7F00u; hs = 3; }
    if (b->nbSeq == 0) { b->seqHdr = hs; return avail == hs ? ZBD_OK : ZBD_CORRUPT; }   /* zero may be written in two bytes; nothing may follow it */
    if (avail < hs + 1u) return ZBD_CORRUPT;
    u32 const m = p[hs];
    if (m & 3u) return ZBD_CORRUPT;
    b->mode[0] = m >> 6; b->mode[1] = (m >> 4) & 3u; b->mode[2] = (m >> 2) & 3u;
    b->seqHdr = hs + 1u;
    return ZBD_OK;
}

/* ---- FSE table description (format: "FSE Table Description"): normalised counts, -1 = "less than one".
 * Returns the bytes consumed (> 0), or 0 on corruption. ---- */
ZBD_HDN u32 zbd_readNCount(short* norm, u32* maxSymPtr, u32* logPtr, u32 maxSym, u32 maxLog, const u8* p, u32 avail)
{
    ZbdFwd f; f.base = p; f.size = avail; f.pos = 0;
    if (avail < 1) return 0;
    u32 const log = (zbd_fwd_peek(&f, 4)) + 5u; f.pos += 4;
    if (log > maxLog) return 0;
    int left = (1 << log) + 1;                                    /* points still to distribute, plus one */
    int limit = 1 << log;                                         /* field values below 2 * limit */
    u32 width = log + 1u;
    u32 s = 0;
    bool afterZero = false;
    while (left > 1 && s <= maxSym) {
        if (afterZero) {                                          /* 2-bit counts of further zeros, 3 = "and another count" */
            while (true) {
                if ((f.pos >> 3) >= avail) return 0;
                u32 const r = zbd_fwd_peek(&f, 2); f.pos += 2;
                for (u32 k = 0; k < r; k++) { if (s > maxSym) return 0; norm[s++] = 0; }
                if (r != 3u) break;
            }
            if (s > maxSym) break;
        }
        if ((f.pos >> 3) >= avail) return 0;
        int const small = 2 * limit - 1 - left;                   /* values below it take width - 1 bits */
        u32 const bits = zbd_fwd_peek(&f, width);
        int v;
        if ((int)(bits & (u32)(limit - 1)) < small) { v = (int)(bits & (u32)(limit - 1)); f.pos += width - 1u; }
        else { v = (int)(bits & (u32)(2 * limit - 1)); if (v >= limit) v -= small; f.pos += width; }
        int const p1 = v - 1;                                     /* probability; -1 = less than one */
        left -= p1 < 0 ? -p1 : p1;
        norm[s++] = (short)p1;
        afterZero = (p1 == 0);
        while (left < limit) { width--; limit >>= 1; }
    }
    if (left != 1) return 0;
    u32 const used = (f.pos + 7u) >> 3;
    if (used > avail) return 0;
    for (u32 k = s; k <= maxSym; k++) norm[k] = 0;
    *maxSymPtr = s - 1u; *logPtr = log;
    return used;
}

/* ---- FSE decoding table (format: "FSE decoding table"): entry = symbol | nbBits << 8 | baseline << 16 ----
 * next[] is scratch for maxSym + 1 counters. */
ZBD_HDN void zbd_buildFseTable(u32* table, const short* norm, u32 maxSym, u32 log, u16* next)
{
    u32 const size = 1u << log, mask = size - 1u, step = (size >> 1) + (size >> 3) + 3u;
    u32 high = size - 1u;
    for (u32 s = 0; s <= maxSym; s++) {
        if (norm[s] == -1) { table[high--] = s; next[s] = 1; }
        else next[s] = (u16)norm[s];
    }
    u32 pos = 0;
    for (u32 s = 0; s <= maxSym; s++) {
        for (int i = 0; i < norm[s]; i++) {
            table[pos] = s;
            do { pos = (pos + step) & mask; } while (pos > high);
        }
    }
    for (u32 u = 0; u < size; u++) {
        u32 const s = table[u];
        u32 const x = next[s]++;
        u32 const nb = log - zbd_hb(x);
        table[u] = s | (nb << 8) | (((x << nb) - size) << 16);
    }
}
ZBD_HD void zbd_buildFseTableRle(u32* table, u32 symbol) { table[0] = symbol; }   /* one state, zero bits */
#define ZBD_FSE_SYM(e)  ((e) & 0xFFu)
#define ZBD_FSE_NB(e)   (((e) >> 8) & 0xFFu)
#define ZBD_FSE_BASE(e) ((e) >> 16)

/* ---- code tables of the sequence section (format: "Sequence codes") ---- */
ZBD_HD u32 zbd_llBits(u32 c) { return c < 16u ? 0u : (c < 20u ? 1u : (c < 22u ? 2u : (c < 24u ? 3u : (c == 24u ? 4u : c - 19u)))); }
ZBD_HD u32 zbd_llBase(u32 c)
{
    if (c < 16u) return c;
    if (c < 20u) return 16u + 2u * (c - 16u);
    if (c < 22u) return 24u + 4u * (c - 20u);
    if (c < 24u) return 32u + 8u * (c - 22u);
    if (c == 24u) return 48u;
    return 1u << (c - 19u);                                       /* 25 -> 64 ... 35 -> 65536 */
}
ZBD_HD u32 zbd_mlBits(u32 c)
{
    if (c < 32u) return 0u;
    if (c < 36u) return 1u;
    if (c < 38u) return 2u;
    if (c < 40u) return 3u;
    if (c < 42u) return 4u;
    if (c == 42u) return 5u;
    return c - 36u;                                               /* 43 -> 7 ... 52 -> 16 */
}
ZBD_HD u32 zbd_mlBase(u32 c)
{
    if (c < 32u) return c + 3u;
    if (c < 36u) return 35u + 2u * (c - 32u);
    if (c < 38u) return 43u + 4u * (c - 36u);
    if (c < 40u) return 51u + 8u * (c - 38u);
    if (c < 42u) return 67u + 16u * (c - 40u);
    if (c == 42u) return 99u;
    return (1u << (c - 36u)) + 3u;                                /* 43 -> 131 ... 52 -> 65539 */
}

/* predefined distributions (format: "Default Distributions") */
#define ZBD_LL_DEFAULT_LOG 6u
#define ZBD_OF_DEFAULT_LOG 5u
#define ZBD_ML_DEFAULT_LOG 6u
#define ZBD_OF_DEFAULT_MAXSYM 28u
ZBD_HD short zbd_defaultNorm(u32 stream, u32 s)
{
    if (stream == 0u) {                                           /* literal lengths */
        if (s == 0u) return 4;
        if (s == 1u || s == 25u) return 3;
        if (s < 13u || (s >= 16u && s < 25u) || s == 26u) return 2;
        if (s < 16u || (s >= 27u && s < 32u)) return 1;
        return -1;
    }
    if (stream == 1u) {                                           /* offsets */
        if (s >= 6u && s <= 8u) return 2;
        if (s < 24u) return 1;
        return -1;
    }
    if (s == 0u) return 1;                                        /* match lengths */
    if (s == 1u) return 4;
    if (s == 2u) return 3;
    if (s < 9u) return 2;
    if (s < 46u) return 1;
    return -1;
}

/* ---- Huffman tree description (format: "Huffman Tree Description") ----
 * weights[0 .. *nbSym) receive every symbol's weight incl. the implied last one.  fseTable / norm / next are scratch (64
 * u32, fseMaxSym + 1 short and u16).  maxLog: the largest weight and table log taken; fseMaxSym: the largest symbol the
 * weights' FSE description may hold.  The defaults are the decoder's; the compressor reads dictionaries with the
 * reference's limits (zb_dict.cu).  Returns the bytes of the description (> 0), or 0 on corruption. */
ZBD_HDN u32 zbd_readHufWeights(u8* weights, u32* nbSymPtr, u32* logPtr, const u8* p, u32 avail, u32* fseTable, short* norm, u16* next,
                               u32 maxLog = ZBD_HUF_LOG_MAX, u32 fseMaxSym = ZBD_HUF_WEIGHT_MAXSYM)
{
    if (avail < 1) return 0;
    u32 const hb = p[0];
    u32 n = 0, used;
    if (hb >= 128u) {                                             /* 4 bits per weight */
        n = hb - 127u;
        used = 1u + (n + 1u) / 2u;
        if (used > avail) return 0;
        for (u32 i = 0; i < n; i++) { u32 const v = p[1u + i / 2u]; weights[i] = (u8)((i & 1u) ? (v & 15u) : (v >> 4)); }
    } else {                                                      /* FSE-compressed weights, two interleaved states */
        used = 1u + hb;
        if (hb == 0 || used > avail) return 0;
        u32 maxSym = 0, log = 0;
        u32 const nc = zbd_readNCount(norm, &maxSym, &log, fseMaxSym, 6u, p + 1, hb);
        if (nc == 0 || nc >= hb) return 0;
        zbd_buildFseTable(fseTable, norm, maxSym, log, next);
        ZbdBack bs;
        if (zbd_back_init(&bs, p + 1u + nc, hb - nc) != ZBD_OK) return 0;
        u32 s1 = zbd_back_read(&bs, log), s2 = zbd_back_read(&bs, log);
        if (bs.pos < 0) return 0;
        while (true) {
            if (n > 253u) return 0;
            u32 e = fseTable[s1]; weights[n++] = (u8)ZBD_FSE_SYM(e);
            s1 = ZBD_FSE_BASE(e) + zbd_back_read(&bs, ZBD_FSE_NB(e));
            if (bs.pos < 0) { weights[n++] = (u8)ZBD_FSE_SYM(fseTable[s2]); break; }
            if (n > 253u) return 0;
            e = fseTable[s2]; weights[n++] = (u8)ZBD_FSE_SYM(e);
            s2 = ZBD_FSE_BASE(e) + zbd_back_read(&bs, ZBD_FSE_NB(e));
            if (bs.pos < 0) { weights[n++] = (u8)ZBD_FSE_SYM(fseTable[s1]); break; }
        }
    }
    /* the last weight completes the sum of 2^(w-1) to a power of two */
    u32 total = 0;
    for (u32 i = 0; i < n; i++) { if (weights[i] > maxLog) return 0; total += weights[i] ? (1u << (weights[i] - 1u)) : 0u; }
    if (total == 0) return 0;
    u32 const log = zbd_hb(total) + 1u;
    if (log > maxLog) return 0;
    u32 const rest = (1u << log) - total;
    if (rest & (rest - 1u)) return 0;                             /* not a power of two */
    weights[n++] = (u8)(zbd_hb(rest) + 1u);
    *nbSymPtr = n; *logPtr = log;
    return used;
}

/* first cell of every symbol in the decoding table (format: "Huffman codes": weights ascending, then symbol order;
 * a symbol of weight w owns 2^(w-1) cells).  Serial form used by the host model; the kernel spreads it over a warp. */
ZBD_HDN void zbd_hufStarts(u16* start, const u8* weights, u32 nbSym, u32 log)
{
    u32 rank[ZBD_HUF_LOG_MAX + 2];
    for (u32 w = 0; w <= log + 1u; w++) rank[w] = 0;
    for (u32 s = 0; s < nbSym; s++) rank[weights[s]]++;
    u32 nextStart = 0;
    for (u32 w = 1; w <= log; w++) { u32 const c = rank[w]; rank[w] = nextStart; nextStart += c << (w - 1u); }
    for (u32 s = 0; s < nbSym; s++) { u32 const w = weights[s]; if (w) { start[s] = (u16)rank[w]; rank[w] += 1u << (w - 1u); } else start[s] = 0; }
}
/* entry = symbol | nbBits << 8 */
ZBD_HD void zbd_hufFill(u16* table, u32 s, u32 start, u32 w, u32 log, u32 lane, u32 lanes)
{
    if (!w) return;
    u32 const len = 1u << (w - 1u);
    u16 const e = (u16)(s | ((log + 1u - w) << 8));
    for (u32 i = lane; i < len; i += lanes) table[start + i] = e;
}

/* one Huffman stream of `count` symbols into out[]; returns 0 or ZBD_CORRUPT.  Symbols are stored four at a time once
 * out is word-aligned (one lane writes a whole stream: byte stores would be one memory transaction each). */
ZBD_HDN u32 zbd_hufDecodeStream(u8* out, u32 count, const u8* p, u32 size, const u16* table, u32 log)
{
    ZbdBack bs;
    if (zbd_back_init(&bs, p, size) != ZBD_OK) return ZBD_CORRUPT;
    u32 i = 0;
    while (i < count && (((uintptr_t)(out + i)) & 3u)) {
        u32 const e = table[zbd_back_peek(&bs, log)];
        out[i++] = (u8)e; bs.pos -= (int)(e >> 8);
    }
    /* fast path: while at least 64 unread bits remain, one 8-byte load serves four symbols (4 x 11 bits <= the 57 bits a
     * byte-aligned window is sure to hold below `pos`) — no underflow or refill tests inside */
    u32 const mask = (1u << log) - 1u;
    while (i + 4u <= count && bs.pos >= 64) {
        int const wl = (bs.pos - 57) & ~7;
        u64 const win = zbd_load64(p, (u32)wl >> 3, size);
        u32 have = (u32)(bs.pos - wl);                            /* 57 .. 64 window bits lie below pos */
        u32 w = 0;
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
        for (u32 k = 0; k < 4u; k++) {
            u32 const e = table[(u32)(win >> (have - log)) & mask];
            w |= (e & 0xFFu) << (8u * k); have -= e >> 8;
        }
        *(u32*)(out + i) = w;
        bs.pos = wl + (int)have;
        i += 4u;
    }
    bs.winLo = 0x40000000;                                        /* the generic reader below starts with a fresh window */
    for (; i + 4u <= count; i += 4u) {
        u32 w = 0;
        for (u32 k = 0; k < 4u; k++) {
            u32 const e = table[zbd_back_peek(&bs, log)];
            w |= (e & 0xFFu) << (8u * k); bs.pos -= (int)(e >> 8);
        }
        *(u32*)(out + i) = w;
    }
    for (; i < count; i++) {
        u32 const e = table[zbd_back_peek(&bs, log)];
        out[i] = (u8)e; bs.pos -= (int)(e >> 8);
    }
    return bs.pos == 0 ? ZBD_OK : ZBD_CORRUPT;
}

/* ---- repcode history as a function of the history at the block's start (format: "Repeat Offsets").
 * A slot holds either a known offset or (1 + k) << 28 | delta: "offset k of the start history minus delta". ---- */
#define ZBD_SYM(k, delta) (((1u + (k)) << 28) | (delta))
#define ZBD_IS_SYM(v) ((v) >> 28)
typedef struct { u32 r[3]; } ZbdRep;
ZBD_HD u32 zbd_rep_minus1(u32 v) { return v - 1u; }              /* known: offset - 1; symbolic: delta + 1 is encoded the other way round below */
/* one sequence: offBase (1..3 repcode, else offset + 3), literal length -> the offset in the same representation */
ZBD_HD u32 zbd_rep_apply(ZbdRep* h, u32 offBase, u32 ll, bool symbolic)
{
    u32 off;
    if (offBase > 3u) { off = offBase - 3u; h->r[2] = h->r[1]; h->r[1] = h->r[0]; h->r[0] = off; return off; }
    u32 const idx = offBase - 1u + (ll == 0u ? 1u : 0u);          /* 0, 1, 2, or 3 = "first offset minus one" */
    if (idx == 0u) return h->r[0];
    if (idx == 3u) off = (symbolic && ZBD_IS_SYM(h->r[0])) ? h->r[0] + 1u : h->r[0] - 1u;     /* symbolic: the low 28 bits count what is subtracted */
    else { off = h->r[1]; if (idx == 2u) off = h->r[2]; }              /* selected, not indexed: h stays in registers */
    if (idx != 1u) h->r[2] = h->r[1];
    h->r[1] = h->r[0]; h->r[0] = off;
    return off;
}
/* value of a slot given the concrete start history */
ZBD_HD u32 zbd_rep_resolve(u32 v, const ZbdRep* start)
{
    u32 const k = ZBD_IS_SYM(v);
    u32 const r = k == 1u ? start->r[0] : (k == 2u ? start->r[1] : start->r[2]);      /* selected, not indexed: the history stays in registers */
    return k ? r - (v & 0x0FFFFFFFu) : v;
}

/* decoded sequence: offBase (28 bits) | litLength (18 bits) << 28 | matchLength (18 bits) << 46 */
ZBD_HD u64 zbd_packSeq(u32 offBase, u32 ll, u32 ml) { return (u64)offBase | ((u64)ll << 28) | ((u64)ml << 46); }
#define ZBD_SEQ_OFF(q) ((u32)(q) & 0x0FFFFFFFu)
#define ZBD_SEQ_LL(q)  ((u32)((q) >> 28) & 0x3FFFFu)
#define ZBD_SEQ_ML(q)  ((u32)((q) >> 46))

/* ---- the sequence bitstream (format: "Sequences_Section", "Sequence Execution" reads these in order) ----
 * tables: LL / OF / ML decoding tables with their accuracy logs (0 for an RLE table).  Writes nbSeq packed sequences;
 * *sumLL / *sumML their totals; *transfer the repcode history at the block's end as a function of its start.
 * Returns 0, ZBD_CORRUPT, or 16 (frameParameter_windowTooLarge) for an offset code above 27. */
ZBD_HDN u32 zbd_decodeSequences(u64* seqs, u32 nbSeq, const u8* p, u32 size, const u32* llT, u32 llLog, const u32* ofT, u32 ofLog,
                                const u32* mlT, u32 mlLog, u32* sumLL, u32* sumML, ZbdRep* transfer)
{
    ZbdBack bs;
    if (zbd_back_init(&bs, p, size) != ZBD_OK) return ZBD_CORRUPT;
    u32 sl = zbd_back_read(&bs, llLog), so = zbd_back_read(&bs, ofLog), sm = zbd_back_read(&bs, mlLog);
    u32 tl = 0, tm = 0;
    ZbdRep h; h.r[0] = ZBD_SYM(0u, 0u); h.r[1] = ZBD_SYM(1u, 0u); h.r[2] = ZBD_SYM(2u, 0u);
    for (u32 i = 0; i < nbSeq; i++) {
        u32 const el = llT[sl], eo = ofT[so], em = mlT[sm];
        u32 const lc = ZBD_FSE_SYM(el), oc = ZBD_FSE_SYM(eo), mc = ZBD_FSE_SYM(em);
        if (oc > ZBD_OF_MAXSYM || lc > ZBD_LL_MAXSYM || mc > ZBD_ML_MAXSYM) return ZBD_CORRUPT;
        if (oc > 27u) return 16u;                                 /* an offset of 2^28 or more: a window this decoder does not take, whatever the header says (frameParameter_windowTooLarge) */
        u32 const offBase = (1u << oc) + zbd_back_read(&bs, oc);
        u32 const ml = zbd_mlBase(mc) + zbd_back_read(&bs, zbd_mlBits(mc));
        u32 const ll = zbd_llBase(lc) + zbd_back_read(&bs, zbd_llBits(lc));
        if (bs.pos < 0) return ZBD_CORRUPT;
        tl += ll; tm += ml;
        if (tl > ZB_BLOCK_MAX || tm > ZB_BLOCK_MAX) return ZBD_CORRUPT;
        seqs[i] = zbd_packSeq(offBase, ll, ml);
        zbd_rep_apply(&h, offBase, ll, true);
        if (i + 1u < nbSeq) {                                     /* state updates: LL, ML, OF */
            sl = ZBD_FSE_BASE(el) + zbd_back_read(&bs, ZBD_FSE_NB(el));
            sm = ZBD_FSE_BASE(em) + zbd_back_read(&bs, ZBD_FSE_NB(em));
            so = ZBD_FSE_BASE(eo) + zbd_back_read(&bs, ZBD_FSE_NB(eo));
            if (bs.pos < 0) return ZBD_CORRUPT;
        }
    }
    if (bs.pos != 0) return ZBD_CORRUPT;
    *sumLL = tl; *sumML = tm; *transfer = h;
    return ZBD_OK;
}


/* ---- the walker: frames and blocks of a compressed buffer (format: "Frames", "Blocks").  Writes at most capB block and
 * capF frame descriptors but counts all of them (*nbB, *nbF): a caller whose arrays were too small calls again.
 * Skippable frames are stepped over.  Returns 0 or a ZSTD error code (10 prefix_unknown, 20 corruption_detected,
 * 72 srcSize_wrong, 14 / 16 frame parameter errors). ---- */
/* dictEntropy: the call's dictionary is a zstd-format one — a frame's first blocks may reuse its Huffman / FSE tables
 * (format: "Dictionary Format"); dictID: its ID (0 = raw content or none): a frame that names another one is refused (32).
 * cursor (NULL on the host): the walk's position in src, published at every frame and block header, for the threads that
 * load the bytes ahead of it (zbd_walk_kernel). */
ZBD_HDN u32 zbd_walk(const u8* src, u64 size, ZbdBlock* blocks, u32 capB, ZbdFrame* frames, u32 capF, u32* nbB, u32* nbF, u64* litBytes, u64* seqCount,
                     bool dictEntropy = false, u32 dictID = 0, volatile u64* cursor = NULL)
{
    u64 pos = 0, litPos = 0, seqPos = 0;
    u32 nb = 0, nf = 0;
    while (pos < size) {
        if (cursor) *cursor = pos;
        ZbdFrameHeader fh;
        u32 const e = zbd_readFrameHeader(&fh, src + pos, size - pos);
        if (e) return (nf > 0 && e == 10u) ? 72u : e;             /* garbage behind a valid frame: srcSize_wrong, as the reference reports it */
        if (fh.skippable) {
            if (fh.contentSize + 8u > size - pos) return 72u;
            pos += 8u + fh.contentSize;
            continue;
        }
        if (fh.windowLog > 27u) return 16u;                       /* offsets are kept in 28 bits.  A Single_Segment frame states no window: any content size passes here, and an offset that needs more than 27 bits gets the same 16 from zbd_decodeSequences */
        ZbdFrame fr; memset(&fr, 0, sizeof(fr));
        fr.srcOff = pos; fr.contentSize = fh.contentSize; fr.windowSize = fh.windowSize; fr.firstBlock = nb;
        fr.hasChecksum = fh.hasChecksum; fr.dictID = fh.dictID;
        u64 const blockMax = fh.windowSize < ZB_BLOCK_MAX ? fh.windowSize : ZB_BLOCK_MAX;
        u64 p = pos + fh.headerSize;
        if (fh.dictID && dictID && fh.dictID != dictID) return 32u;   /* dictionary_wrong */
        u32 lastHuf = ZBD_NONE, lastEff[3] = { ZBD_NONE, ZBD_NONE, ZBD_NONE }, lastSrc[3] = { ZBD_NONE, ZBD_NONE, ZBD_NONE };
        if (dictEntropy) { lastHuf = ZBD_DICT; for (u32 s = 0; s < 3u; s++) { lastEff[s] = 2u; lastSrc[s] = ZBD_DICT; } }
        bool first = true;
        while (true) {
            if (cursor) *cursor = p;
            if (p + 3u > size) return 72u;
            u32 const bh = zbd_le(src + p, 3);
            u32 const last = bh & 1u, type = (bh >> 1) & 3u, bsz = bh >> 3;
            if (type == 3u) return ZBD_CORRUPT;
            u32 const csz = type == ZB_BT_RLE ? 1u : bsz;
            if (bsz > blockMax) return ZBD_CORRUPT;               /* Block_Maximum_Size = min(window, 128 KiB) */
            if (p + 3u + csz > size) return 72u;
            ZbdBlock b; memset(&b, 0, sizeof(b));
            b.srcOff = p + 3u; b.cSize = csz; b.type = type; b.rawSize = type == ZB_BT_COMPRESSED ? 0u : bsz; b.frame = nf; b.blockMax = (u32)blockMax;
            b.flags = (first ? ZB_FLAG_FIRST : 0u) | (last ? ZB_FLAG_LAST : 0u);
            b.hufSrc = ZBD_NONE; b.fseSrc[0] = b.fseSrc[1] = b.fseSrc[2] = ZBD_NONE;
            if (type == ZB_BT_COMPRESSED) {
                const u8* const c = src + p + 3u;
                if (csz < 2u) return ZBD_CORRUPT;
                if (zbd_readLitHeader(&b, c, csz)) return ZBD_CORRUPT;
                if (b.litRegen > blockMax) return ZBD_CORRUPT;   /* the whole regenerated size, literals + matches: D2 */
                if (b.litType == 2u) lastHuf = nb;
                if (b.litType >= 2u) { if (lastHuf == ZBD_NONE) return ZBD_CORRUPT; b.hufSrc = lastHuf; }
                b.seqOff = b.litHdr + b.litComp;
                if (zbd_readSeqHeader(&b, c + b.seqOff, csz - b.seqOff)) return ZBD_CORRUPT;
                if (b.nbSeq) {
                    for (u32 s = 0; s < 3u; s++) {
                        if (b.mode[s] == 3u) {
                            if (lastEff[s] == ZBD_NONE) return ZBD_CORRUPT;
                            b.eff[s] = lastEff[s]; b.fseSrc[s] = lastSrc[s];
                        } else { b.eff[s] = b.mode[s]; b.fseSrc[s] = b.mode[s] ? nb : ZBD_NONE; }
                        lastEff[s] = b.eff[s]; lastSrc[s] = b.fseSrc[s];
                    }
                }
            }
            b.litPos = litPos; b.seqPos = seqPos;
            if (type == ZB_BT_COMPRESSED) { litPos += ((u64)b.litRegen + 15u) & ~15ull; seqPos += b.nbSeq; }
            if (nb < capB) blocks[nb] = b;
            nb++; first = false;
            p += 3u + csz;
            if (last) break;
        }
        if (fh.hasChecksum) { if (p + 4u > size) return 72u; p += 4u; }
        fr.cSize = p - pos; fr.nbBlocks = nb - fr.firstBlock;
        if (nf < capF) frames[nf] = fr;
        nf++;
        pos = p;
    }
    *nbB = nb; *nbF = nf; *litBytes = litPos; *seqCount = seqPos;
    return ZBD_OK;
}

/* ---- dictionary (format: "Dictionary Format"): magic 0xEC30A437, ID, Huffman tree description, FSE table descriptions of
 * offsets, match lengths, literal lengths (in this order), three repeat offsets, content.  Anything else is raw content. ---- */
typedef struct {
    u32 entropy;           /* 1: a zstd-format dictionary */
    u32 dictID;
    u32 hufOff, hufLen;    /* tree description */
    u32 fseOff[3], fseLen[3];   /* 0 = LL, 1 = OF, 2 = ML (the order of the kernels' streams, not of the file) */
    u32 rep[3];
    u32 contentOff;
    u32 pad;
} ZbdDictInfo;
#define ZBD_MAGIC_DICT 0xEC30A437u
/* hufMaxLog / hufFseMaxSym (<= 255): the limits of the Huffman tree description, as zbd_readHufWeights takes them (the
 * defaults are the decoder's).
 * Returns 0, or 30 (dictionary_corrupted). */
ZBD_HDN u32 zbd_parseDict(ZbdDictInfo* di, const u8* dict, u64 size, u32 hufMaxLog = ZBD_HUF_LOG_MAX, u32 hufFseMaxSym = ZBD_HUF_WEIGHT_MAXSYM)
{
    memset(di, 0, sizeof(*di));
    if (size < 8 || zbd_le(dict, 4) != ZBD_MAGIC_DICT) return ZBD_OK;          /* raw content */
    di->entropy = 1; di->dictID = zbd_le(dict + 4, 4);
    u32 p = 8;
    {   u8 weights[256]; u32 nbSym, log; u32 fse[64]; short norm[256]; u16 next[256];
        u32 const used = zbd_readHufWeights(weights, &nbSym, &log, dict + p, (u32)(size - p > 0xFFFFu ? 0xFFFFu : size - p), fse, norm, next,
                                            hufMaxLog, hufFseMaxSym);
        if (!used) return 30u;
        di->hufOff = p; di->hufLen = used; p += used; }
    u32 const order[3] = { 1u, 2u, 0u };                                        /* the file holds OF, ML, LL */
    u32 const maxSym[3] = { ZBD_LL_MAXSYM, ZBD_OF_MAXSYM, ZBD_ML_MAXSYM }, maxLog[3] = { ZBD_LL_LOG_MAX, ZBD_OF_LOG_MAX, ZBD_ML_LOG_MAX };
    for (u32 k = 0; k < 3u; k++) {
        u32 const st = order[k];
        short norm[64]; u32 ms, lg;
        if (p >= size) return 30u;
        u32 const used = zbd_readNCount(norm, &ms, &lg, maxSym[st], maxLog[st], dict + p, (u32)(size - p > 0xFFFFu ? 0xFFFFu : size - p));
        if (!used) return 30u;
        di->fseOff[st] = p; di->fseLen[st] = used; p += used;
    }
    if ((u64)p + 12u > size) return 30u;
    for (u32 k = 0; k < 3u; k++) { di->rep[k] = zbd_le(dict + p + 4u * k, 4); }
    p += 12u;
    di->contentOff = p;
    u64 const contentSize = size - p;
    for (u32 k = 0; k < 3u; k++) if (di->rep[k] == 0 || di->rep[k] > contentSize) return 30u;
    return ZBD_OK;
}

/* offsets of the three table descriptions inside a block's sequences section (LL, OF, ML in this order, each 0 bytes for
 * predefined / repeat, 1 byte for RLE, an FSE table description otherwise).  sec = the section's first byte.  desc[s] =
 * offset of stream s's description from sec; *bitstream = offset of the sequence bitstream.  Returns 0 or ZBD_CORRUPT.
 * norm is scratch for 53 shorts. */
ZBD_HDN u32 zbd_locateDescriptions(const ZbdBlock* b, const u8* sec, u32 avail, u32* desc, u32* bitstream, short* norm)
{
    u32 off = b->seqHdr;
    u32 const maxSym[3] = { ZBD_LL_MAXSYM, ZBD_OF_MAXSYM, ZBD_ML_MAXSYM }, maxLog[3] = { ZBD_LL_LOG_MAX, ZBD_OF_LOG_MAX, ZBD_ML_LOG_MAX };
    for (u32 s = 0; s < 3u; s++) {
        desc[s] = off;
        if (b->mode[s] == 1u) { if (off + 1u > avail) return ZBD_CORRUPT; off += 1u; }
        else if (b->mode[s] == 2u) {
            u32 ms, lg;
            u32 const n = zbd_readNCount(norm, &ms, &lg, maxSym[s], maxLog[s], sec + off, avail - off);
            if (!n) return ZBD_CORRUPT;
            off += n;
        }
    }
    if (off > avail) return ZBD_CORRUPT;
    *bitstream = off;
    return ZBD_OK;
}

/* ---- per-block steps of the literals and sequences kernels (zb_decode.cu D1 / D2), run block after block by the CPU
 * harness.  Per-stream limits are selected, not indexed: a stream index that is a lane number would put an array into
 * local memory. ---- */
ZBD_HD u32 zbd_seqMaxSym(u32 st) { return st == 0u ? ZBD_LL_MAXSYM : (st == 1u ? ZBD_OF_MAXSYM : ZBD_ML_MAXSYM); }
ZBD_HD u32 zbd_seqMaxLog(u32 st) { return st == 0u ? ZBD_LL_LOG_MAX : (st == 1u ? ZBD_OF_LOG_MAX : ZBD_ML_LOG_MAX); }

/* the Huffman tree description the literals of block b use: that of the block that defined the table (b->hufSrc: b itself
 * unless treeless), or the dictionary's.  src = the compressed input; *len = the bytes the description may occupy. */
ZBD_HD const u8* zbd_hufDescription(const ZbdBlock* b, const ZbdBlock* blocks, const u8* src, const u8* dict, const ZbdDictInfo* di, u32* len)
{
    if (b->hufSrc == ZBD_DICT) { *len = di->hufLen; return dict + di->hufOff; }
    const ZbdBlock* const sb = blocks + b->hufSrc;
    *len = sb->litComp;
    return src + sb->srcOff + sb->litHdr;
}

/* the four Huffman streams of a literals section (format: "Jump_Table"): s[0 .. total) = jump table + streams, regen = the
 * symbols they decode to.  off[k] / size[k]: stream k's bytes from s; count[k]: its symbols, which go to k * count[0].
 * Returns 0 or ZBD_CORRUPT. */
ZBD_HD u32 zbd_litStreams(u32* off, u32* size, u32* count, const u8* s, u32 total, u32 regen)
{
    if (total < 6u) return ZBD_CORRUPT;
    u32 const s1 = zbd_le(s, 2), s2 = zbd_le(s + 2, 2), s3 = zbd_le(s + 4, 2);
    u32 const seg = (regen + 3u) / 4u;
    if (6u + s1 + s2 + s3 > total || 3u * seg > regen) return ZBD_CORRUPT;
    off[0] = 6u; off[1] = 6u + s1; off[2] = 6u + s1 + s2; off[3] = 6u + s1 + s2 + s3;
    size[0] = s1; size[1] = s2; size[2] = s3; size[3] = total - off[3];
    count[0] = count[1] = count[2] = seg; count[3] = regen - 3u * seg;
    return ZBD_OK;
}

/* decoding table of sequence stream st (0 LL, 1 OF, 2 ML) of block b into table[] (up to 512 cells), as b->eff[st] and
 * b->fseSrc[st] say: predefined, the dictionary's, one RLE symbol, or a table description in the sequences section of the
 * block that defined it.  norm / next are scratch for 64 entries each.  Returns the table's log (0 for RLE), or -1 on
 * corruption. */
ZBD_HD int zbd_seqTable(u32* table, short* norm, u16* next, u32 st, const ZbdBlock* b, const ZbdBlock* blocks, const u8* src,
                        const u8* dict, const ZbdDictInfo* di)
{
    u32 const maxSym = zbd_seqMaxSym(st);
    u32 ms = 0, log = 0;
    if (b->eff[st] == 0u) {
        log = st == 0u ? ZBD_LL_DEFAULT_LOG : (st == 1u ? ZBD_OF_DEFAULT_LOG : ZBD_ML_DEFAULT_LOG);
        ms = st == 1u ? ZBD_OF_DEFAULT_MAXSYM : maxSym;
        for (u32 s = 0; s <= ms; s++) norm[s] = zbd_defaultNorm(st, s);
        zbd_buildFseTable(table, norm, ms, log, next);
        return (int)log;
    }
    const u8* p; u32 avail;
    if (b->fseSrc[st] == ZBD_DICT) { p = dict + di->fseOff[st]; avail = di->fseLen[st]; }
    else {
        const ZbdBlock* const sb = blocks + b->fseSrc[st];
        const u8* const sec = src + sb->srcOff + sb->seqOff;
        u32 const secLen = sb->cSize - sb->seqOff;
        u32 desc[3], bitstream;
        if (zbd_locateDescriptions(sb, sec, secLen, desc, &bitstream, norm)) return -1;
        p = sec + desc[st]; avail = secLen - desc[st];
        if (b->eff[st] == 1u) {
            if (p[0] > maxSym) return -1;
            zbd_buildFseTableRle(table, p[0]);
            return 0;
        }
    }
    if (!zbd_readNCount(norm, &ms, &log, maxSym, zbd_seqMaxLog(st), p, avail)) return -1;
    zbd_buildFseTable(table, norm, ms, log, next);
    return (int)log;
}

#endif
