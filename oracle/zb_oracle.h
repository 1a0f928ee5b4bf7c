/* zb_oracle.h — CPU oracle for the zstd_b200 hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing in the product (zstd_b200/) may include, link or call this.
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg use it, and only as the
 * checker.  It is a plain-C restatement of
 *   (1) the reference's entropy stage (Huffman literals + FSE sequences), byte-exact with
 *       lib/compress/{huf_compress.c,fse_compress.c,zstd_compress_literals.c,
 *       zstd_compress_sequences.c,zstd_compress.c:2881-3035} given the same seqStore, and
 *   (2) the block-parallel "warp-batch" greedy match-finder the CUDA kernels implement (a
 *       deterministic data-parallel re-formulation of zstd_fast.c:192-423 /
 *       zstd_double_fast.c:105-323; the parse differs from the serial CPU parse by design,
 *       the compressed size must stay within +-0.5 % and every frame must decode with the
 *       reference ZSTD_decompress).
 * Parity pins (tests/test_oracle_*.py): (1) is compared byte-for-byte with the compiled reference
 * (oracle/_ref/libzstd_ref.so + oracle/_ref/libref_shim.so); (2) is pinned by round-trip through
 * the reference decoder and by size against the reference at the same level.
 */
#ifndef ZB_ORACLE_H
#define ZB_ORACLE_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef uint8_t  u8;
typedef uint16_t u16;
typedef uint32_t u32;
typedef uint64_t u64;

/* ---- error codes: same numbering as lib/zstd_errors.h:64-101 ---- */
#define ZBO_ERR(code)            ((size_t)-(long)(code))
#define ZBO_error_GENERIC            1
#define ZBO_error_dictionary_corrupted 30
#define ZBO_error_parameter_unsupported 40
#define ZBO_error_memory_allocation 64
#define ZBO_error_dstSize_tooSmall  70
#define ZBO_error_srcSize_wrong     72
#define ZBO_error_maxCode          120
static inline int zbo_isError(size_t c) { return c > ZBO_ERR(ZBO_error_maxCode); }

/* ---- compression parameters (lib/zstd.h:ZSTD_compressionParameters) ---- */
typedef struct {
    u32 windowLog, chainLog, hashLog, searchLog, minMatch, targetLength, strategy; /* 1=fast 2=dfast */
} zbo_cparams;
zbo_cparams zbo_getCParams(int level, u64 srcSize, size_t dictSize);

/* ---- one sequence, as the match-finder emits it ---- */
typedef struct { u32 offBase; u32 litLen; u32 matchLen; } zbo_seq;   /* matchLen = real length (>=3) */

/* ---- block-parallel plan constants (shared with the CUDA side; see DESIGN.md) ---- */
#define ZB_BLOCK_MAX      (128u << 10)     /* ZSTD_BLOCKSIZE_MAX, lib/zstd.h:142 */
#define ZB_PRIME_DEFAULT  (128u << 10)     /* history primed into a chunk's private table */
#define ZB_CHUNK_BLOCKS   4u               /* blocks per chunk (one table lives through a chunk) */
#define ZB_BATCH          1024u            /* positions of one walk batch (= threads of the walk CTA) */
#define ZB_BATCH_MAX      4096u
#define ZB_FAST_HASHLOG_MAX  14u           /* fast: <= 12288 u32 buckets = 48 KiB of shared memory */
#define ZB_DFAST_SHORT_MAX 28672u          /* dfast short table: 28672 x u32 = 112 KiB of shared memory */
#define ZB_DFAST_LONGLOG_MAX  14u          /* dfast long table: 16384 x u32 = 64 KiB */
#define ZB_WARP           32u
#define ZB_PARSE_SEG      (16u << 10)      /* fast strategy: bytes of a block parsed by one warp (8 segments per 128 KiB block) */

typedef struct {
    u32 mls;          /* bytes hashed (cParams.minMatch clamped to 4..8; short hash for dfast) */
    u32 tableN;       /* buckets of the (short) table */
    u32 tableNLong;   /* dfast only: buckets of the 8-byte-hash table, else 0 */
    u32 stepSize;     /* targetLength + !targetLength + 1 (zstd_fast.c:200); dfast: 1 */
    u32 insStep;      /* positions without a candidate enter the table when ((pos - low) % step) < 2, step = insStep + walked/128 */
    u32 chunkBlocks;  /* blocks per chunk */
    u32 startRep[2];  /* repcodes the search of the frame's first segment starts with (a zstd-format dictionary's), 0 = none */
    u32 codeRep[3];   /* repcode history the decoder holds at the frame's first block: {1,4,8} or the dictionary's */
    size_t frameStart;/* index of the frame's first byte inside the buffer handed to the matcher (dictionary tail in front) */
    u32 primeBytes;   /* history window primed before a chunk */
    u32 strategy;     /* 1 fast, 2 dfast */
    u32 windowLog;
    u32 litCompressionDisabled; /* zstd_compress_internal.h:621-633 */
} zbo_plan;
void zbo_makePlan(zbo_plan* plan, const zbo_cparams* cp);

/* ---- entropy primitives (exported so tests can pin each against the reference) ---- */
u32    zbo_hist(const u8* src, size_t n, u32* count, u32* maxSymbolPtr);  /* hist.c:29 */
u32    zbo_fse_optimalTableLog(u32 maxTableLog, size_t srcSize, u32 maxSymbolValue, u32 minus); /* fse_compress.c:357 */
size_t zbo_fse_normalize(int16_t* norm, u32 tableLog, const u32* count, size_t total, u32 maxSymbolValue, u32 useLowProbCount); /* fse_compress.c:465 */
size_t zbo_fse_writeNCount(u8* dst, size_t cap, const int16_t* norm, u32 maxSymbolValue, u32 tableLog); /* fse_compress.c:234 */

typedef struct {           /* our own layout of an FSE compression table (fse.h:249 holds the reference's) */
    u32 tableLog;
    u32 maxSymbolValue;
    u16 nextState[512];    /* sorted by symbol; value = tableSize + slot   (fse_compress.c:170-173) */
    int32_t deltaFindState[64];
    u32 deltaNbBits[64];
} zbo_fse_ctable;
size_t zbo_fse_buildCTable(zbo_fse_ctable* ct, const int16_t* norm, u32 maxSymbolValue, u32 tableLog); /* fse_compress.c:68 */
void   zbo_fse_buildCTable_rle(zbo_fse_ctable* ct, u8 symbol);   /* fse_compress.c:528 */

typedef struct { u8 nbBits[256]; u16 code[256]; u32 tableLog; u32 maxSymbolValue; } zbo_huf_ctable;
size_t zbo_huf_buildCTable(zbo_huf_ctable* ct, const u32* count, u32 maxSymbolValue, u32 maxNbBits); /* huf_compress.c:756 */
size_t zbo_huf_writeCTable(u8* dst, size_t cap, const zbo_huf_ctable* ct);    /* huf_compress.c:248 */
size_t zbo_huf_encode1X(u8* dst, size_t cap, const u8* src, size_t n, const zbo_huf_ctable* ct); /* huf_compress.c:1056 */
size_t zbo_huf_encode4X(u8* dst, size_t cap, const u8* src, size_t n, const zbo_huf_ctable* ct); /* huf_compress.c:1168 */

/* entropy state a zstd-format dictionary installs as "previous block" (zstd_compress.c:4987-5076) */
typedef struct {
    u32 present, dictID;
    zbo_huf_ctable huf; u32 hufRepeat;          /* 0 none, 1 check, 2 valid (HUF_repeat) */
    zbo_fse_ctable fse[3]; u32 fseRepeat[3];     /* 0 = LL, 1 = OF, 2 = ML ; FSE_repeat */
    u32 rep[3];
} zbo_dict_entropy;
size_t zbo_readNCount(int16_t* norm, u32* maxSymbolPtr, u32* tableLogPtr, const u8* p, size_t avail);  /* entropy_common.c:42 */
size_t zbo_loadDictEntropy(zbo_dict_entropy* de, const u8* dict, size_t dictSize);

/* the product's own table builders (zb_tables.c); zbo_entropy_model selects them (1, default) or the restatement of the
 * reference's (0: what tests/test_oracle_entropy.py pins byte-for-byte against the compiled reference) inside
 * zbo_fse_normalize / zbo_huf_buildCTable and everything built on them */
extern int zbo_entropy_model;
size_t zbo_fse_normalize_lr(int16_t* norm, u32 tableLog, const u32* count, size_t total, u32 maxSymbolValue);
size_t zbo_huf_lengths_mk(u8* nbBits, const u32* count, u32 maxSymbolValue, u32 target);

/* literals section, fresh tables (no repeat/treeless): zstd_compress_literals.c:129 */
size_t zbo_compressLiterals(u8* dst, size_t cap, const u8* lit, size_t litSize,
                            u32 strategy, int disableLiteralCompression, int suspectUncompressible);

/* whole compressed-block body (literals + sequences sections) with fresh entropy state:
 * zstd_compress.c:2881-3035.  Returns 0 when the block must be emitted raw. */
size_t zbo_entropyCompressBlock(u8* dst, size_t cap,
                                const zbo_seq* seqs, size_t nbSeq,
                                const u8* lit, size_t litSize,
                                size_t blockSrcSize, u32 strategy, int disableLiteralCompression);
/* same with a dictionary's tables as the previous block's entropy state (prev may be NULL) */
size_t zbo_entropyCompressBlock_prev(u8* dst, size_t cap,
                                const zbo_seq* seqs, size_t nbSeq,
                                const u8* lit, size_t litSize,
                                size_t blockSrcSize, u32 strategy, int disableLiteralCompression,
                                const zbo_dict_entropy* prev);

/* ---- match-finder model ---- */
/* candidates of one chunk [start, end) of buf (phase 1); dS/dL indexed by position - start */
typedef struct { u32* dS; u32* dL; size_t low, start, end; } zbo_chunkCand;
void zbo_walkChunk(const zbo_plan* plan, const u8* buf, size_t bufSize, size_t chunkStart, size_t chunkEnd, zbo_chunkCand* cc);
void zbo_freeChunk(zbo_chunkCand* cc);
/* Parses block [blockStart, blockStart+blockSize) of its chunk (phase 2).  Emits sequences + literal bytes.
 * Returns nbSeq; *litSizePtr gets the total literal count (including the trailing literals). */
size_t zbo_parseBlock(const zbo_plan* plan, const u8* buf, const zbo_chunkCand* cc,
                      size_t blockStart, size_t blockSize,
                      zbo_seq* seqs, u8* lit, size_t* litSizePtr);
/* experiment knobs (0 = default), only set by tools/ scripts */
typedef struct { u32 tableN, tableNLong, tableFmt, insStep, primeBytes, chunkBlocks, batch, spare; } zbo_tunables;
extern zbo_tunables zbo_tun;

/* ---- frame level: mirrors ZSTD_compress / ZSTD_compress_usingDict (lib/zstd.h:155,944) ---- */
size_t zbo_compressBound(size_t srcSize);                             /* lib/zstd.h:235 */
size_t zbo_compress(void* dst, size_t cap, const void* src, size_t srcSize, int level);
size_t zbo_compress_usingDict(void* dst, size_t cap, const void* src, size_t srcSize,
                              const void* dict, size_t dictSize, int level);
/* per-block compressed sizes of the last zbo_compress call on this thread (diagnostics) */
size_t zbo_writeFrameHeader(u8* dst, size_t cap, u32 windowLog, u64 srcSize, u32 dictID); /* zstd_compress.c:4626 */
void   zbo_synthetic(u8* buf, size_t n, u32 seed, u32 matchProb256);   /* test data generator (ours) */

#ifdef __cplusplus
}
#endif
#endif
