/* zstd_b200.h — C ABI of libzstd_b200.so: the H100-native drop-in for zstd's per-block
 * compression hot path (fast / doubleFast match-finder + Huffman literals + FSE sequences).
 *
 * Section 1 re-declares, with identical names, signatures, argument meaning and error
 * behaviour, the reference entry points this library replaces (a language binding that
 * dlopen()s libzstd for these symbols can be pointed at libzstd_b200.so unchanged).
 * Section 2 adds device-pointer and many-frame entry points that have no reference
 * counterpart (the reference has no device memory and no batch call); they are what the
 * benchmark's device-resident `value` and the multi-GPU sharding use.
 *
 * All compression work is done by sm_90a CUDA kernels (H100).  There is no CPU fallback: when no
 * CUDA device is usable every compress call returns ZSTD_error_GENERIC (code 1).
 */
#ifndef ZSTD_B200_H
#define ZSTD_B200_H
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#  define ZSTDB200_API __attribute__((visibility("default")))
#else
#  define ZSTDB200_API
#endif

/* =====================  1. reference-identical entry points  ===================== */

typedef struct ZSTD_CCtx_s ZSTD_CCtx;                 /* opaque, lib/zstd.h:262 */

/* lib/zstd.h:155 — one call = one complete frame, content size in the header, no checksum.
 * Returns compressed size, or an error code testable with ZSTD_isError(). */
ZSTDB200_API size_t ZSTD_compress(void* dst, size_t dstCapacity, const void* src, size_t srcSize, int compressionLevel);

/* lib/zstd.h:263-264 — context lifecycle; ZSTD_freeCCtx accepts NULL. */
ZSTDB200_API ZSTD_CCtx* ZSTD_createCCtx(void);
ZSTDB200_API size_t     ZSTD_freeCCtx(ZSTD_CCtx* cctx);

/* lib/zstd.h:274 — same as ZSTD_compress with an explicit, reusable context. */
ZSTDB200_API size_t ZSTD_compressCCtx(ZSTD_CCtx* cctx, void* dst, size_t dstCapacity,
                                      const void* src, size_t srcSize, int compressionLevel);

/* lib/zstd.h:944 — compression with a (raw-content or zstd-format) dictionary. */
ZSTDB200_API size_t ZSTD_compress_usingDict(ZSTD_CCtx* ctx, void* dst, size_t dstCapacity,
                                            const void* src, size_t srcSize,
                                            const void* dict, size_t dictSize, int compressionLevel);

/* lib/zstd.h:967-995 — digested dictionary: the dictionary is parsed once, its content tail, entropy tables
 * and primed match-finder tables stay resident on the GPU across calls (the reference's CDict keeps the
 * same things in host memory, zstd_compress.c:5477-5642).  A CDict may be shared by any number of contexts
 * on one device.  ZSTD_createCDict returns NULL for a zstd-format dictionary whose entropy tables are
 * corrupted; ZSTD_freeCDict accepts NULL.  ZSTD_compress_usingCDict compresses at the CDict's level
 * (zstd_compress.c:5836) and produces the bytes ZSTD_compress_usingDict produces for the same inputs. */
typedef struct ZSTD_CDict_s ZSTD_CDict;
ZSTDB200_API ZSTD_CDict* ZSTD_createCDict(const void* dictBuffer, size_t dictSize, int compressionLevel);
ZSTDB200_API size_t      ZSTD_freeCDict(ZSTD_CDict* cdict);
ZSTDB200_API size_t      ZSTD_compress_usingCDict(ZSTD_CCtx* cctx, void* dst, size_t dstCapacity,
                                                  const void* src, size_t srcSize, const ZSTD_CDict* cdict);
/* lib/zstd.h:1099-1111 */
ZSTDB200_API unsigned    ZSTD_getDictID_fromCDict(const ZSTD_CDict* cdict);
ZSTDB200_API unsigned    ZSTD_getDictID_fromDict(const void* dict, size_t dictSize);

/* lib/zstd.h:337-603 — the advanced one-shot API most bindings use today: sticky parameters on the context, then
 * ZSTD_compress2.  Honoured: ZSTD_c_compressionLevel, ZSTD_c_checksumFlag (XXH64 of the content: a serial recurrence per
 * frame — hashed by host threads while the GPU compresses when the input is in host memory; by one
 * warp per frame on the device for device buffers, all frames of a call side by side),
 * ZSTD_c_dictIDFlag, ZSTD_c_contentSizeFlag (the size is always written).  Accepted and ignored: ZSTD_c_nbWorkers,
 * ZSTD_c_jobSize, ZSTD_c_overlapLog.  windowLog .. strategy only at 0 (ZSTD_c_windowLog = 20 answers 40 even with long
 * distance matching on); anything else returns ZSTD_error_parameter_unsupported (40).  ZSTD_CCtx_loadDictionary copies and
 * digests the dictionary (lib/zstd.h:1088); ZSTD_CCtx_refCDict borrows a CDict, whose level then applies (:1102).
 * Long-distance matching (zstd --long): ZSTD_c_enableLongDistanceMatching takes 0 auto (= off: the reference enables it
 * only for btopt and stronger), 1 enable, 2 disable, anything else 42 (parameter_outOfBound).  ZSTD_c_ldmHashLog [6, 30],
 * ZSTD_c_ldmMinMatch [4, 4096], ZSTD_c_ldmBucketSizeLog [1, 8] and ZSTD_c_ldmHashRateLog [0, 25] are honoured (0 = derived
 * from the frame's window as ZSTD_ldm_adjustParameters does: 20, 64, 3 and 7 for a 2^27 window; outside the bounds 42).  All
 * are sticky until ZSTD_CCtx_reset(ZSTD_reset_parameters).  With LDM on, a frame of more than ZSTDB200_framePartAlignment()
 * (512 KiB) has a 2^27-byte window (before the adjustment to its size) and its blocks may copy from anywhere in it; smaller
 * frames are compressed exactly as with LDM off.  Honoured by ZSTD_compress2, ZSTD_compressStream2,
 * ZSTDB200_compressFrames[_usingCDict] and ZSTDB200_compressDevice; ignored by the simple API and the sequence calls;
 * ZSTDB200_compressFramePart returns 40.  A prefix (ZSTD_CCtx_refPrefix, below) is searched for long matches; unlike the
 * reference, the content of a loaded dictionary or CDict is not (it still serves the first chunk's history).  Host-buffer
 * calls upload their whole input before the first kernel.
 *
 * ZSTD_CCtx_refPrefix (lib/zstd.h:1104-1125) — compress the next frame against a prefix, e.g. the previous version of a file
 * (what `zstd --patch-from` does); the decoder needs the same bytes (ZSTD_DCtx_refPrefix, ZSTD_decompress_usingDict).  As in
 * the reference: the bytes are borrowed, not copied, and must stay valid until that frame is made; they are raw content
 * even when they begin with the dictionary magic; the frame names dictionary ID 0; the prefix serves the NEXT FRAME ONLY
 * and is then forgotten (also when that call fails); NULL / 0 clears it; it replaces a loaded dictionary or referenced
 * CDict and those replace it; inside an unfinished stream it returns ZSTD_error_stage_wrong (60).
 * ZSTD_CCtx_reset(ZSTD_reset_session_only) keeps a pending prefix, the directives that reset parameters drop it.  A prefix of
 * less than 8 bytes is ignored, as every dictionary that short.
 * Honoured by ZSTD_compress2, ZSTD_compressStream2 (the first frame the session emits; frames the front end cuts later
 * have none) and ZSTDB200_compressDevice; the simple API ignores it (it stays pending); ZSTDB200_compressFrames[_usingCDict],
 * ZSTDB200_compressFramePart and the sequence calls return 40 while one is pending.
 * Without LDM the prefix is a raw-content dictionary: its last 128 KiB are the first chunk's history.  With
 * ZSTD_c_enableLongDistanceMatching = 1 and more than 512 KiB of prefix and input together, the prefix's last 2^27 bytes are
 * indexed along with the frame and every block that ends within the window (2^27 bytes, less when prefix + input are
 * smaller) of a prefix position may copy from it.  Matches are found in the prefix and in the frame, never across the seam
 * between them; blocks beyond 2^27 bytes into the frame take nothing from the prefix (the format's window), and prefix bytes
 * more than 2^27 from its end are never used.  Cost per call with P = min(prefixSize, 2^27) indexed bytes, n input bytes and
 * m = ZSTD_c_ldmMinMatch (64): the LDM workspace grows from about 36 (n / m + 1) + 16 (n / 4096 + 1)(4096 / m + 1) bytes to the
 * same of P + n, the match list from 8 (n / m + 1) to 8 ((P + n) / m + 1) bytes; a host prefix is uploaded (P bytes of device
 * memory and of PCIe traffic, counted in h2d_bytes), a device prefix (ZSTDB200_CCtx_refPrefixDevice) is read in place. */
typedef enum {
    ZSTD_c_compressionLevel = 100, ZSTD_c_windowLog = 101, ZSTD_c_hashLog = 102, ZSTD_c_chainLog = 103, ZSTD_c_searchLog = 104,
    ZSTD_c_minMatch = 105, ZSTD_c_targetLength = 106, ZSTD_c_strategy = 107,
    ZSTD_c_enableLongDistanceMatching = 160, ZSTD_c_ldmHashLog = 161, ZSTD_c_ldmMinMatch = 162, ZSTD_c_ldmBucketSizeLog = 163,
    ZSTD_c_ldmHashRateLog = 164,
    ZSTD_c_contentSizeFlag = 200, ZSTD_c_checksumFlag = 201, ZSTD_c_dictIDFlag = 202,
    ZSTD_c_nbWorkers = 400, ZSTD_c_jobSize = 401, ZSTD_c_overlapLog = 402,
    ZSTD_c_blockDelimiters = 1008, ZSTD_c_validateSequences = 1009     /* lib/zstd.h:2123-2149, see ZSTD_compressSequences */
} ZSTD_cParameter;
typedef enum { ZSTD_reset_session_only = 1, ZSTD_reset_parameters = 2, ZSTD_reset_session_and_parameters = 3 } ZSTD_ResetDirective;
ZSTDB200_API size_t ZSTD_CCtx_setParameter(ZSTD_CCtx* cctx, ZSTD_cParameter param, int value);
ZSTDB200_API size_t ZSTD_CCtx_setPledgedSrcSize(ZSTD_CCtx* cctx, unsigned long long pledgedSrcSize);
ZSTDB200_API size_t ZSTD_CCtx_reset(ZSTD_CCtx* cctx, ZSTD_ResetDirective reset);
ZSTDB200_API size_t ZSTD_CCtx_loadDictionary(ZSTD_CCtx* cctx, const void* dict, size_t dictSize);
ZSTDB200_API size_t ZSTD_CCtx_refCDict(ZSTD_CCtx* cctx, const ZSTD_CDict* cdict);
ZSTDB200_API size_t ZSTD_CCtx_refPrefix(ZSTD_CCtx* cctx, const void* prefix, size_t prefixSize);
ZSTDB200_API size_t ZSTD_compress2(ZSTD_CCtx* cctx, void* dst, size_t dstCapacity, const void* src, size_t srcSize);

/* lib/zstd.h:681-862 — streaming.  The GPU works on whole frames, so the stream front end collects input in the context
 * and emits FRAMES: ZSTD_e_continue buffers (256 MiB of input become a frame of their own), ZSTD_e_flush turns what is
 * buffered into a frame now, ZSTD_e_end does the same and ends the session.  The output is therefore a sequence of frames —
 * every zstd decoder reads it as the concatenation of their contents (lib/zstd.h:160-162) — where the reference writes one
 * frame; ZSTD_getFrameContentSize() of such output describes its first frame only.  A session's first call that brings
 * everything with ZSTD_e_end and room for ZSTD_compressBound(size) bytes is compressed straight from the caller's buffers.
 * Return value as in the reference: > 0 while output is still waiting (call again with more room), 0 when flushed / ended;
 * with ZSTD_e_continue a hint for the next input size. */
typedef struct ZSTD_inBuffer_s  { const void* src; size_t size; size_t pos; } ZSTD_inBuffer;
typedef struct ZSTD_outBuffer_s { void* dst; size_t size; size_t pos; } ZSTD_outBuffer;
typedef enum { ZSTD_e_continue = 0, ZSTD_e_flush = 1, ZSTD_e_end = 2 } ZSTD_EndDirective;
ZSTDB200_API size_t ZSTD_compressStream2(ZSTD_CCtx* cctx, ZSTD_outBuffer* output, ZSTD_inBuffer* input, ZSTD_EndDirective endOp);
typedef ZSTD_CCtx ZSTD_CStream;                       /* lib/zstd.h:822: the same object */
ZSTDB200_API ZSTD_CStream* ZSTD_createCStream(void);
ZSTDB200_API size_t ZSTD_freeCStream(ZSTD_CStream* zcs);
ZSTDB200_API size_t ZSTD_initCStream(ZSTD_CStream* zcs, int compressionLevel);
ZSTDB200_API size_t ZSTD_compressStream(ZSTD_CStream* zcs, ZSTD_outBuffer* output, ZSTD_inBuffer* input);
ZSTDB200_API size_t ZSTD_flushStream(ZSTD_CStream* zcs, ZSTD_outBuffer* output);
ZSTDB200_API size_t ZSTD_endStream(ZSTD_CStream* zcs, ZSTD_outBuffer* output);
ZSTDB200_API size_t ZSTD_CStreamInSize(void);
ZSTDB200_API size_t ZSTD_CStreamOutSize(void);

/* lib/zstd.h:1291-1322, 1555-1644 — compression of sequences the caller found (an external or GPU match finder, a format
 * transcoder): zstd does the entropy stage and the framing only.  `rep` is ignored, as in the reference.
 * ZSTD_c_blockDelimiters (0 or 1, sticky, reset by ZSTD_reset_parameters):
 *   ZSTD_sf_explicitBlockDelimiters: a sequence with offset == 0 && matchLength == 0 ends a block, its litLength being the
 *     block's trailing literals.  A block larger than min(128 KiB, window), sequences that run past srcSize or that stop
 *     before srcSize is covered (no final delimiter) are invalid; an empty block produces no block, delimiters behind
 *     the last byte are ignored.
 *   ZSTD_sf_noBlockDelimiters: blocks of min(128 KiB, window) bytes, as ZSTD_compress2 cuts a frame; bytes beyond the sum of
 *     the sequences are literals.  A sequence that crosses a block edge is split there: its literals go to the block they
 *     fall in; a part of its match that is at least 3 bytes long stays a match (the part behind the edge with
 *     litLength 0 and the same offset), a shorter part becomes literals.  The reference's splitter may cut other
 *     blocks; both give valid frames.
 * A sequence is invalid when offset == 0 (and it is not a delimiter), matchLength < 3, or offset > (pos > window ? window :
 * pos + dictionary content size) with pos its end (zstd_compress.c:6531), or offset > 2^24 - 4.  Matches of 3 bytes are
 * accepted whatever ZSTD_c_minMatch says (the reference rejects them unless minMatch is 3; minMatch is default-only here).
 * Invalid sequences return ZSTD_error_externalSequences_invalid (107).  Validation always runs (on the GPU: it costs a few
 * compares in a pass that reads every sequence, and the kernels rely on the lengths it checks), so ZSTD_c_validateSequences
 * (0 or 1) is accepted and has no effect.
 * Repcodes: the history is {1,4,8} (or the dictionary's) at the frame's first block and unknown at every other block; inside
 * a block it runs as the reference runs it.  Feeding back the sequences of one of this library's frames, with its level,
 * dictionary and block boundaries, gives that frame again byte for byte.
 * Level, checksum flag, dictID flag and the dictionary (ZSTD_CCtx_loadDictionary / ZSTD_CCtx_refCDict) apply as for
 * ZSTD_compress2, window and strategy come from the level and srcSize.  The call writes one frame. */
typedef struct { unsigned int offset, litLength, matchLength, rep; } ZSTD_Sequence;
typedef enum { ZSTD_sf_noBlockDelimiters = 0, ZSTD_sf_explicitBlockDelimiters = 1 } ZSTD_sequenceFormat_e;
ZSTDB200_API size_t ZSTD_sequenceBound(size_t srcSize);                                       /* zstd_compress.c:3456 */
ZSTDB200_API size_t ZSTD_mergeBlockDelimiters(ZSTD_Sequence* sequences, size_t seqsSize);   /* zstd_compress.c:3497, host code */
ZSTDB200_API size_t ZSTD_compressSequences(ZSTD_CCtx* cctx, void* dst, size_t dstSize, const ZSTD_Sequence* inSeqs, size_t inSeqsSize,
                                           const void* src, size_t srcSize);
/* lib/zstd.h:1594 — the parse of the frame ZSTD_compress2 writes for src on this context: the sticky level, the loaded
 * dictionary or referenced CDict (whose level then applies) and the same blocks of min(128 KiB, window) bytes.  For every
 * block of that frame, in order: its sequences, then a delimiter {offset 0, litLength = the block's trailing literals,
 * matchLength 0, rep 0}.  A sequence's offset is the real distance (it may reach into the dictionary's content); rep is the
 * repcode 1-3 the frame codes it with, 0 for a directly coded offset, with the reference's convention (a sequence without
 * literals shifts the repcodes, zstd_compress.c:3411-3428).  The repcode history is {1,4,8} (or the dictionary's) at the
 * frame's first block and unknown at every other, as for ZSTD_compressSequences, so rep is non-zero only where this frame
 * really uses a repcode.  Feeding the output back to ZSTD_compressSequences with ZSTD_sf_explicitBlockDelimiters (or, after
 * ZSTD_mergeBlockDelimiters, with ZSTD_sf_noBlockDelimiters) and the same level, dictionary and flags gives ZSTD_compress2's
 * frame byte for byte.  Checksum, dictID and content-size flags do not change the output; nbWorkers is ignored as
 * everywhere here.  An empty input gives 0 sequences; ZSTD_sequenceBound(srcSize) rows always suffice.
 * Returns the number of sequences written, or an error code: dstSize_tooSmall (70) when they do not fit in outSeqsSize,
 * dstBuffer_null (74) for a NULL outSeqs with a non-zero size, parameter_unsupported (40) with long-distance matching on,
 * with a prefix pending (it stays pending) or for a level above 4 under ZSTDB200_setStrictLevels(1), GENERIC (1) without a
 * device.  The GPU runs the match finder; only the input goes up and only the rows written come back.
 * Two deliberate differences from the reference, which marks its version "for debugging only": a block below 7 bytes is
 * one delimiter carrying its size (the reference fails there with sequenceProducer_failed), and on dstSize_tooSmall
 * outSeqs is left untouched (the reference writes a prefix). */
ZSTDB200_API size_t ZSTD_generateSequences(ZSTD_CCtx* cctx, ZSTD_Sequence* outSeqs, size_t outSeqsSize, const void* src, size_t srcSize);

/* lib/zstd.h:236,242-246,114-120 ; lib/zstd_errors.h:106 */
ZSTDB200_API size_t      ZSTD_compressBound(size_t srcSize);
ZSTDB200_API unsigned    ZSTD_isError(size_t code);
ZSTDB200_API const char* ZSTD_getErrorName(size_t code);
ZSTDB200_API int         ZSTD_getErrorCode(size_t functionResult);     /* ZSTD_ErrorCode as int */
ZSTDB200_API int         ZSTD_minCLevel(void);
ZSTDB200_API int         ZSTD_maxCLevel(void);
ZSTDB200_API int         ZSTD_defaultCLevel(void);
ZSTDB200_API unsigned    ZSTD_versionNumber(void);
ZSTDB200_API const char* ZSTD_versionString(void);

/* lib/zstd.h:170-299 — decompression (SURVEY.md 8f rank 2).  Every frame the format allows is accepted: this library's
 * own and the reference encoder's at any level, concatenated frames, skippable frames, frames without a content size,
 * window sizes up to 128 MiB (the reference decoder's default limit, ZSTD_WINDOWLOG_LIMIT_DEFAULT = 27), raw-content
 * and zstd-format dictionaries (ZSTD_decompress_usingDict, lib/zstd.h:955: the dictionary's content is the history in front
 * of every frame, its entropy tables and repeat offsets what a frame's first blocks may reuse; dictionary_wrong = 32 when a
 * frame names another dictionary ID).
 * The content checksum of a frame that carries one is verified (host buffers; checksum_wrong = 22).
 * All decoding work is done by CUDA kernels (zb_decode.cu); no CPU fallback. */
typedef struct ZSTD_DCtx_s ZSTD_DCtx;
ZSTDB200_API size_t     ZSTD_decompress(void* dst, size_t dstCapacity, const void* src, size_t compressedSize);
ZSTDB200_API ZSTD_DCtx* ZSTD_createDCtx(void);
ZSTDB200_API size_t     ZSTD_freeDCtx(ZSTD_DCtx* dctx);                                    /* accepts NULL */
ZSTDB200_API size_t     ZSTD_decompressDCtx(ZSTD_DCtx* dctx, void* dst, size_t dstCapacity, const void* src, size_t srcSize);
ZSTDB200_API size_t     ZSTD_decompress_usingDict(ZSTD_DCtx* dctx, void* dst, size_t dstCapacity, const void* src, size_t srcSize,
                                                  const void* dict, size_t dictSize);
/* lib/zstd.h:195-227 — header readers (host code).  ZSTD_CONTENTSIZE_UNKNOWN = (0ULL - 1), ZSTD_CONTENTSIZE_ERROR = (0ULL - 2). */
ZSTDB200_API unsigned long long ZSTD_getFrameContentSize(const void* src, size_t srcSize);
ZSTDB200_API size_t     ZSTD_findFrameCompressedSize(const void* src, size_t srcSize);
/* lib/zstd.h:1437-1473 — what the frames in src[0, srcSize) decompress to, read from frame and block headers alone; both
 * return what the reference returns for every input.  Skippable frames count 0.  Windows up to 2^31 are read, although
 * the decoder refuses windows above 2^27; legacy (pre-v0.8) frames are not supported and give ZSTD_CONTENTSIZE_ERROR.
 * ZSTD_findDecompressedSize: the frames' content sizes summed; ZSTD_CONTENTSIZE_UNKNOWN at the first frame that states
 * none; ZSTD_CONTENTSIZE_ERROR for a bad frame header or block-header chain, bytes behind the last frame, or a sum past
 * 2^64.  ZSTD_decompressBound: the same sum, with a frame that states no content size counted as its number of blocks
 * times min(window, 128 KiB); ZSTD_CONTENTSIZE_ERROR for invalid input. */
ZSTDB200_API unsigned long long ZSTD_findDecompressedSize(const void* src, size_t srcSize);
ZSTDB200_API unsigned long long ZSTD_decompressBound(const void* src, size_t srcSize);
/* lib/zstd.h:1120 — the dictionary ID a frame names (host code): 0 when it names none, for a skippable frame, and when the
 * header can not be read (too short, not a frame). */
ZSTDB200_API unsigned   ZSTD_getDictID_fromFrame(const void* src, size_t srcSize);

/* lib/zstd.h:1000-1030 — digested dictionary of the decoder.  ZSTD_createDDict copies and parses the dictionary on the host
 * (no GPU is needed to create or query one); its first use uploads it whole (header and content) to the device of the
 * context using it, where it stays resident: later calls with it make no copy and no synchronisation for the dictionary.
 * Any number of contexts on that one device may use it; a context on another device gets ZSTD_error_parameter_unsupported
 * (40).  ZSTD_createDDict returns NULL for a zstd-format dictionary with corrupted entropy tables, and also where this
 * decoder refuses more than the reference: a Huffman tree description with a table log above 11 (the reference's limit is
 * 12), or whose weights' FSE description gives a probability to a symbol above 12; it accepts Huffman weights with fewer
 * than two 1s, which the reference refuses (DESIGN.md section 4).  ZSTD_freeDDict
 * accepts NULL.  ZSTD_decompress_usingDDict with NULL decodes without a dictionary. */
typedef struct ZSTD_DDict_s ZSTD_DDict;
ZSTDB200_API ZSTD_DDict* ZSTD_createDDict(const void* dictBuffer, size_t dictSize);
ZSTDB200_API size_t      ZSTD_freeDDict(ZSTD_DDict* ddict);
ZSTDB200_API size_t      ZSTD_decompress_usingDDict(ZSTD_DCtx* dctx, void* dst, size_t dstCapacity, const void* src, size_t srcSize,
                                                    const ZSTD_DDict* ddict);
ZSTDB200_API unsigned    ZSTD_getDictID_fromDDict(const ZSTD_DDict* ddict);                  /* lib/zstd.h:1113 */

/* lib/zstd.h:609-650, 1160-1210 (zstd_decompress.c:1697-1960) — the context's sticky dictionary and parameters, used by
 * ZSTD_decompressDCtx (hence ZSTD_decompressStream) and ZSTDB200_decompressDevice.  ZSTD_DCtx_loadDictionary copies and
 * digests the dictionary (a corrupted one returns ZSTD_error_memory_allocation, 64, as in the reference), ZSTD_DCtx_refDDict
 * borrows a DDict (NULL: none); both are sticky.  ZSTD_DCtx_refPrefix borrows raw content for the next call only (in
 * streaming: the next frame).  Each replaces what was there.
 * ZSTD_d_windowLogMax: 0 means the default 27; [10, 31], else ZSTD_error_parameter_outOfBound (42).  As in the reference it
 * applies to ZSTD_decompressStream only, which refuses a frame whose window (at least 1 KiB; a Single_Segment frame's is
 * its content size) is larger with ZSTD_error_frameParameter_windowTooLarge (16), decided from its header.  A frame that
 * arrives whole with one call whose output buffer has room for its content size is decoded in one pass, without the limit,
 * as the reference does.  Windows above 2^27 stay refused everywhere.  Other parameters return
 * ZSTD_error_parameter_unsupported (40).
 * ZSTD_DCtx_reset: ZSTD_reset_session_only drops an unfinished stream and keeps dictionary and parameters;
 * ZSTD_reset_parameters drops both.  ZSTD_initDStream drops the dictionary too.  Setting a parameter or a dictionary (or
 * resetting parameters) while ZSTD_decompressStream is inside a frame returns ZSTD_error_stage_wrong (60). */
typedef enum { ZSTD_d_windowLogMax = 100 } ZSTD_dParameter;
ZSTDB200_API size_t ZSTD_DCtx_setParameter(ZSTD_DCtx* dctx, ZSTD_dParameter param, int value);
ZSTDB200_API size_t ZSTD_DCtx_reset(ZSTD_DCtx* dctx, ZSTD_ResetDirective reset);
ZSTDB200_API size_t ZSTD_DCtx_loadDictionary(ZSTD_DCtx* dctx, const void* dict, size_t dictSize);
ZSTDB200_API size_t ZSTD_DCtx_refDDict(ZSTD_DCtx* dctx, const ZSTD_DDict* ddict);
ZSTDB200_API size_t ZSTD_DCtx_refPrefix(ZSTD_DCtx* dctx, const void* prefix, size_t prefixSize);

/* lib/zstd.h:880-924 — streaming decompression.  Whole frames are decoded on the GPU: compressed bytes are collected in
 * the context until a frame is complete, then decoded and handed out as the caller makes room.  Returns 0 when a frame has
 * been decoded and handed out completely, else a hint (> 0) for the next call, or an error code. */
typedef ZSTD_DCtx ZSTD_DStream;
ZSTDB200_API ZSTD_DStream* ZSTD_createDStream(void);
ZSTDB200_API size_t ZSTD_freeDStream(ZSTD_DStream* zds);
ZSTDB200_API size_t ZSTD_initDStream(ZSTD_DStream* zds);
ZSTDB200_API size_t ZSTD_decompressStream(ZSTD_DStream* zds, ZSTD_outBuffer* output, ZSTD_inBuffer* input);
ZSTDB200_API size_t ZSTD_DStreamInSize(void);
ZSTDB200_API size_t ZSTD_DStreamOutSize(void);

/* =====================  2. Extensions (no reference counterpart)  ===================== */

/* Decompress frames whose bytes are in device memory into device memory.  The frame / block headers are a chain that has to
 * be followed in order: for inputs of up to 512 MiB the compressed bytes are copied to a page-locked host buffer and walked
 * there, beyond that one device thread follows them (1.3-1.4 us per block on an H100 80GB HBM3 at 700 W); everything else is block-parallel.  Content
 * checksums are not verified on this path.  `stream`: as for ZSTDB200_compressDevice.  Returns the decompressed size. */
ZSTDB200_API size_t ZSTDB200_decompressDevice(ZSTD_DCtx* dctx, void* d_dst, size_t dstCapacity, const void* d_src, size_t srcSize, void* stream);
/* same with a dictionary (host memory; uploaded by the call) */
ZSTDB200_API size_t ZSTDB200_decompressDevice_usingDict(ZSTD_DCtx* dctx, void* d_dst, size_t dstCapacity, const void* d_src, size_t srcSize,
                                                        const void* dict, size_t dictSize, void* stream);
typedef struct {
    float kernel_ms;         /* literals kernel start -> match kernel end */
    float literals_ms, sequences_ms, place_ms, execute_ms;       /* D1, D2, D4 (literal placement), D5 (match copies) */
    unsigned launches, nbBlocks, nbFrames;
    size_t h2d_bytes, d2h_bytes;
} ZSTDB200_dstats;
ZSTDB200_API void ZSTDB200_getLastDStats(const ZSTD_DCtx* dctx, ZSTDB200_dstats* out);

/* Stream-ordered decompression: the call enqueues the whole decompression on `stream` and returns without waiting for the
 * GPU; the verdict lands in device memory, so the consumer of the decompressed bytes can be queued behind it, and the call
 * can be captured into a CUDA graph.  The header walk runs on the device (one thread, fed from L1 by the rest of its CTA),
 * so no compressed byte crosses PCIe.
 * `stream` is the caller's cudaStream_t; NULL is the legacy default stream — unlike ZSTDB200_decompressDevice.
 * Return value: 0 once the work is enqueued, or an error code decided before anything is enqueued: ZSTD_error_GENERIC (1)
 * without a device or with d_result NULL, parameter_unsupported (40) while a ZSTD_DCtx_refPrefix is pending (the prefix is
 * forgotten), memory_allocation (64), stage_wrong (60) under capture (below).
 * *d_result (8 bytes of device, managed or mapped page-locked memory) is written by the call's last kernel, in stream order:
 * the decompressed size, or an error code as size_t (ZSTD_isError is true for it).  For the same bytes, capacity and sticky
 * dictionary it is what ZSTDB200_decompressDevice returns (content checksums are not verified either), but for inputs of
 * more blocks or frames than the workspace below holds: those get workSpace_tooSmall (66), and ZSTDB200_decompressDevice
 * decodes them.  Nothing is written outside [d_dst, d_dst + dstCapacity); with an error found before the output is placed
 * (a corrupt header or block, a content size that does not match, dstSize_tooSmall (70)) nothing is written to d_dst.
 * Workspace.  The host reads no header, so the context's buffers are sized from srcSize and dstCapacity alone, for up to
 *   B = srcSize / 16 + dstCapacity / 1024 + 1024
 * blocks and as many frames: any input whose blocks hold, on average, 16 compressed bytes or 1 KiB of content (every frame
 * this library or the reference encoder writes of 8 bytes of content or more, and up to 1024 blocks of anything).  That
 * costs about 7 bytes per byte of dstCapacity (literals, sequences, match positions, tiles) plus about 16 bytes per byte
 * of srcSize (block and frame descriptors), a few GiB for a call of 1 GiB.  Buffers only grow; a context keeps them.
 * Dictionaries: the sticky one (ZSTD_DCtx_refDDict, ZSTD_DCtx_loadDictionary) is honoured.  Its first use on a device
 * uploads it and synchronises with the context's own stream; from then on it costs a call nothing.
 * No host wait: once an earlier call has sized the context for this (srcSize, dstCapacity) or larger, a call neither
 * synchronises, nor allocates, nor copies synchronously or from pageable memory.  A call that has to grow a buffer waits for
 * the context's earlier calls; it never waits for the producer of d_src.
 * Ordering: the calls made on one context run on the GPU in the order they are made, whatever stream they name; synchronous
 * calls wait for the stream-ordered ones queued before them, and ZSTD_freeDCtx waits for them.  d_src must stay valid
 * until the work ran.
 * CUDA graphs: a call made while `stream` is capturing becomes part of the graph, and every replay decodes whatever bytes
 * lie at d_src then.  Precondition: a completed call with the same (srcSize, dstCapacity) or larger on the same context
 * before the capture, and a resident dictionary; otherwise the call returns stage_wrong (60) before enqueuing anything.
 * While such a graph lives, its context makes no other call and is not freed: replays use its workspace.
 * ZSTDB200_getLastDStats after a stream-ordered call fills launches only (reading the times would synchronise). */
ZSTDB200_API size_t ZSTDB200_decompressDeviceAsync(ZSTD_DCtx* dctx, void* d_dst, size_t dstCapacity,
                                                   const void* d_src, size_t srcSize,
                                                   unsigned long long* d_result, void* stream);

/* Decompress a batch of independent entries in one call (the counterpart of ZSTDB200_compressFrames): each entry into its
 * own slot of the output, each with its own result, the entries' headers walked side by side on the GPU.
 * Buffers and arrays.  d_src and d_dst are device memory.  srcOffsets, srcSizes, dstOffsets and dstCapacities are host
 * arrays of nbEntries values, read before the call returns.
 * Entry i is d_src[srcOffsets[i], + srcSizes[i]).  It may hold anything ZSTDB200_decompressDevice accepts: one or more frames,
 * skippable frames.  Its result equals what ZSTDB200_decompressDevice(dctx, d_dst + dstOffsets[i], dstCapacities[i],
 * d_src + srcOffsets[i], srcSizes[i], ...) returns with the same sticky dictionary: the decompressed size or an error code.
 * Content checksums are not verified, as on that call.  An entry of 0 bytes gives 0.
 * Writes.  Nothing is written outside an entry's slot d_dst[dstOffsets[i], + dstCapacities[i]).  An error found before an
 * entry's output is placed (a corrupt header or block, a content size that does not match, dstSize_tooSmall (70)) leaves its
 * slot untouched.
 * Per-entry results.  dSizes[i] (host array) or d_dSizes[i] (device, managed or mapped page-locked memory) receives entry i's
 * result; either may be NULL.
 * Return value.  ZSTDB200_decompressFrames returns the sum of the entries' sizes when every entry decoded, otherwise the error
 * code of the lowest-index entry that failed: ZSTD_isError on it says "look at the sizes".  ZSTDB200_decompressFramesAsync
 * returns 0 once the work is enqueued, and *d_result receives that same value in stream order.
 * Refusals, decided before anything is enqueued (dSizes is then not written): ZSTD_error_GENERIC (1) without a device, with
 * d_result NULL or an array NULL; parameter_unsupported (40) while a ZSTD_DCtx_refPrefix is pending (the prefix is forgotten);
 * parameter_outOfBound (42) when a source range lies outside [0, srcSize), a slot outside [0, dstCapacity), or the slots are
 * not ascending and disjoint (dstOffsets[i] + dstCapacities[i] <= dstOffsets[i + 1]; overlapping slots would race); checked
 * in O(nbEntries); memory_allocation (64); stage_wrong (60) under capture, as below.  nbEntries = 0 gives 0.
 * Workspace.  Sized from host-known numbers, as for ZSTDB200_decompressDeviceAsync, so the host reads no header: up to
 * B + nbEntries blocks and as many frames, B = srcSize / 16 + dstCapacity / 1024 + 1024, literals and sequences sized from
 * the sum of dstCapacities.  An entry whose blocks or frames fall past that bound gets workSpace_tooSmall (66); the others
 * still decode.  The workspace is given out in entry order, and an entry that gets 66 takes none of it.
 * Ordering, capture and stats: as for ZSTDB200_decompressDeviceAsync.  The calls made on one context run in the order they
 * are made; a context sized by an earlier call of the same shape or a larger one neither synchronises nor allocates; a CUDA
 * graph captured after such a call replays on whatever bytes lie at d_src, with the offsets and capacities of the captured
 * call.  The offset arrays are staged in a ring of ZSTDB200_ASYNC_SLOTS page-locked slots (the host waits when the next
 * slot's call has not uploaded them yet).  ZSTDB200_getLastDStats fills launches, which does not depend on nbEntries.
 * ZSTDB200_decompressFrames is the stream-ordered call plus one read-back of the verdict and the sizes; a NULL stream
 * means the context's own stream, as for ZSTDB200_decompressDevice. */
ZSTDB200_API size_t ZSTDB200_decompressFrames(ZSTD_DCtx* dctx,
        void* d_dst, size_t dstCapacity, const size_t* dstOffsets, const size_t* dstCapacities,
        const void* d_src, size_t srcSize, const size_t* srcOffsets, const size_t* srcSizes,
        size_t nbEntries, size_t* dSizes, void* stream);
ZSTDB200_API size_t ZSTDB200_decompressFramesAsync(ZSTD_DCtx* dctx,
        void* d_dst, size_t dstCapacity, const size_t* dstOffsets, const size_t* dstCapacities,
        const void* d_src, size_t srcSize, const size_t* srcOffsets, const size_t* srcSizes,
        size_t nbEntries, unsigned long long* d_dSizes, unsigned long long* d_result, void* stream);

/* The same calls with one digested dictionary per entry (the decoder's counterpart of ZSTDB200_compressFrames_usingCDicts):
 * a batch written against many dictionaries is read back in one launch sequence.  Everything stated above holds (slots,
 * writes, per-entry results, return value, refusals, workspace, ordering, the staging ring, capture, launches); only where
 * each entry's dictionary comes from differs.
 * Entry i's bytes and result are what ZSTDB200_decompressDevice gives for it on a context whose sticky dictionary is ddicts[i]
 * (ZSTD_DCtx_refDDict): a frame that names another dictionary ID gets dictionary_wrong (32), and fails alone.  A NULL entry,
 * a NULL ddicts, or a DDict of size 0 means no dictionary for that entry.  ddicts is a host array read before the call
 * returns; the same DDict may appear any number of times.  The DDicts must stay alive until the work ran.
 * The context's sticky dictionary is not used and is left as it is; a pending ZSTD_DCtx_refPrefix still gets
 * parameter_unsupported (40) and is forgotten.
 * More refusals, decided before anything is enqueued (dSizes is then not written): parameter_unsupported (40) for a DDict
 * resident on another device, as ZSTD_decompress_usingDDict gives it; under capture, stage_wrong (60) for any DDict not yet
 * resident on the context's device.
 * Dictionaries.  A DDict becomes resident on its first use: the call uploads every DDict it names that is not resident yet,
 * then synchronises once with the context's own stream.  From then on a DDict costs a call one reference in the staging
 * slot (8 bytes per entry); the kernels find each block's dictionary through it.  DDicts may be shared by contexts on one
 * device and by threads.  ZSTDB200_getLastDStats fills launches (12, whatever the number of entries and dictionaries) and
 * h2d_bytes, the dictionary bytes the call uploaded (0 when all were resident). */
ZSTDB200_API size_t ZSTDB200_decompressFrames_usingDDicts(ZSTD_DCtx* dctx,
        void* d_dst, size_t dstCapacity, const size_t* dstOffsets, const size_t* dstCapacities,
        const void* d_src, size_t srcSize, const size_t* srcOffsets, const size_t* srcSizes,
        size_t nbEntries, const ZSTD_DDict* const* ddicts, size_t* dSizes, void* stream);
ZSTDB200_API size_t ZSTDB200_decompressFramesAsync_usingDDicts(ZSTD_DCtx* dctx,
        void* d_dst, size_t dstCapacity, const size_t* dstOffsets, const size_t* dstCapacities,
        const void* d_src, size_t srcSize, const size_t* srcOffsets, const size_t* srcSizes,
        size_t nbEntries, const ZSTD_DDict* const* ddicts,
        unsigned long long* d_dSizes, unsigned long long* d_result, void* stream);

/* ZSTDB200_decompressFramesAsync with the batch's index in device memory, for a GPU reader that finds its pages' offsets and
 * sizes in a kernel: no copy to the host and no synchronisation stand between that kernel and the decode.  The contract of
 * ZSTDB200_decompressFramesAsync holds word for word (slots, writes, per-entry results, return value, the sticky dictionary,
 * ordering, "no host wait once sized"), but for these points.
 * Arrays.  d_dstOffsets, d_dstCapacities, d_srcOffsets and d_srcSizes are device (or managed) arrays of nbEntries values,
 * 8-byte aligned; otherwise the call returns parameter_outOfBound (42) before enqueuing anything.  The call's kernels read
 * them in stream order, so a kernel that writes them may be queued on `stream` just before the call; they must stay valid
 * until the work ran.  No descriptor crosses PCIe and the staging ring is not used.
 * Checks in stream order.  The checks the host form makes in its host loop (source ranges inside [0, srcSize), slots inside
 * [0, dstCapacity), ascending and disjoint) are made on the device.  A violation makes the whole call's verdict
 * parameter_outOfBound (42) in *d_result; nothing is then written to d_dst or d_dSizes.  Decided on the host, before
 * enqueuing: ZSTD_error_GENERIC (1) without a device, with d_result NULL or an array NULL while nbEntries > 0;
 * parameter_unsupported (40) for a pending prefix; stage_wrong (60) under capture on a context not sized; memory_allocation (64).
 * Workspace.  The sum of the slots is not known on the host, so literals and sequences are sized from dstCapacity; blocks and
 * frames as for the host form (B + nbEntries).  An entry's admission depends only on the block and frame bounds, so for the
 * same values the bytes and results equal ZSTDB200_decompressFramesAsync's, workSpace_tooSmall (66) and dstSize_tooSmall (70)
 * included.
 * CUDA graphs.  A replay reads the arrays at replay time: one graph decodes whatever batch of at most nbEntries entries the
 * arrays describe then.  Pad a smaller batch with empty entries (an entry of 0 bytes gives 0).
 * ZSTDB200_getLastDStats fills launches: 13, the host form's 12 and the kernel that checks and packs the arrays.
 * Per-entry DDicts and a synchronous form are not offered. */
ZSTDB200_API size_t ZSTDB200_decompressFramesAsync_deviceOffsets(ZSTD_DCtx* dctx,
        void* d_dst, size_t dstCapacity, const unsigned long long* d_dstOffsets, const unsigned long long* d_dstCapacities,
        const void* d_src, size_t srcSize, const unsigned long long* d_srcOffsets, const unsigned long long* d_srcSizes,
        size_t nbEntries, unsigned long long* d_dSizes, unsigned long long* d_result, void* stream);

/* Each entry's decompressed size on the device, to size the slots of a batch without reading headers on the host:
 * d_contentSizes[i] = ZSTD_findDecompressedSize(d_src + d_srcOffsets[i], d_srcSizes[i]) and d_bounds[i] =
 * ZSTD_decompressBound(...) of the same range.  Either output may be NULL, not both (ZSTD_error_GENERIC).  An entry whose
 * range lies outside [0, srcSize) gets ZSTD_CONTENTSIZE_ERROR in both; no byte outside the input is read.
 * One kernel, one thread per entry, following the entry's frame and block headers (one dependent load per block: a 1 GiB
 * entry of 128 KiB blocks is a chain of 8192).  The call uses none of the context's buffers (the context names the device),
 * enqueues on `stream` (NULL: the legacy default stream) without joining the context's call order, and may be captured at
 * any time.  Every array is 8-byte aligned, otherwise parameter_outOfBound (42) before enqueuing.  Returns 0 once enqueued;
 * ZSTD_error_GENERIC without a device or with an input array NULL while nbEntries > 0. */
ZSTDB200_API size_t ZSTDB200_findDecompressedSizesAsync(ZSTD_DCtx* dctx, const void* d_src, size_t srcSize,
        const unsigned long long* d_srcOffsets, const unsigned long long* d_srcSizes, size_t nbEntries,
        unsigned long long* d_contentSizes, unsigned long long* d_bounds, void* stream);


/* Compress one frame whose input and output already live in device memory (HBM).  The call returns when the frame is
 * complete (it synchronises to read the size).
 * `stream` is a cudaStream_t.  Non-NULL: all work of the call is enqueued on that stream, behind whatever the caller
 * queued there before (the way to compress the output of a kernel that is still running).  NULL: the context's own
 * NON-BLOCKING streams are used — they are NOT ordered after the legacy default stream or any other stream, so the
 * producer of d_src must have completed (e.g. cudaStreamSynchronize) before the call.  Large NULL-stream calls run as
 * several waves on several streams.  d_src needs no padding: no byte outside [d_src, d_src + srcSize) is read. */
ZSTDB200_API size_t ZSTDB200_compressDevice(ZSTD_CCtx* cctx, void* d_dst, size_t dstCapacity,
                                            const void* d_src, size_t srcSize, int compressionLevel, void* stream);

/* Stream-ordered compression: the call enqueues the whole compression on `stream` and returns without waiting for the GPU;
 * the verdict lands in device memory, so the consumer of the compressed bytes (a copy, a send, the next kernel) can be
 * queued behind it, and the call can be captured into a CUDA graph.
 * Output: byte for byte what ZSTDB200_compressDevice produces (single frame), or ZSTDB200_compressFrames with deviceMemory = 1
 * (ZSTDB200_compressFrames_usingCDict when cdict is not NULL) for the same inputs and context state.
 * `stream` is the caller's cudaStream_t; NULL is the legacy default stream (PyTorch's default stream) — unlike
 * ZSTDB200_compressDevice, where NULL selects the context's own streams.  Inputs of 256 MiB or more run as the same waves as
 * a NULL-stream ZSTDB200_compressDevice call, on the context's wave streams, forked from and joined back into `stream`.
 * Return value: 0 once the work is enqueued, or an error code decided before anything is enqueued: ZSTD_error_GENERIC (1)
 * without a device or with d_result NULL, parameter_unsupported (40) for strict levels (ZSTDB200_setStrictLevels) or a
 * pending prefix as below, memory_allocation (64), stage_wrong (60) under capture (below).
 * *d_result (8 bytes of device, managed or mapped page-locked memory) is written by the call's last kernel, in stream order:
 * the total compressed size, or an error code as size_t (ZSTD_isError is true for it): dstSize_tooSmall (70) when the frames
 * do not fit, in which case nothing is written past d_dst + dstCapacity.  d_cSizes (batch call, may be NULL; same kinds of
 * memory): the size of each frame.  frameOffsets / frameSizes are host arrays, read before the call returns.
 * Parameters.  ZSTDB200_compressDeviceAsync honours the sticky checksum flag, dictID flag, long-distance matching and its
 * parameters, the dictionary of ZSTD_CCtx_loadDictionary (at compressionLevel) or ZSTD_CCtx_refCDict (at the CDict's level,
 * as ZSTD_compress2), and a device prefix (ZSTDB200_CCtx_refPrefixDevice); a pending host prefix returns 40 and is
 * forgotten.  ZSTDB200_compressFramesAsync applies compressionLevel without a CDict and the CDict's level with one, and
 * returns 40 while a prefix is pending.  The input, the dictionary's bytes and a CDict must stay valid until the work ran.
 * No host wait: once an earlier call of the same or a larger shape has sized the context's buffers, made the dictionary
 * resident and built its table images, a call neither synchronises, nor copies synchronously or from pageable memory, nor
 * allocates or frees.  A call that has to do one of those may synchronise with the context's earlier calls.  The
 * descriptors of a call are staged in a ring of ZSTDB200_ASYNC_SLOTS page-locked slots; the host waits when the next slot's
 * call has not yet uploaded them (more than that many calls queued behind unfinished work).
 * Ordering: the calls made on one context run on the GPU in the order they are made, whatever stream they name and whether
 * they are stream-ordered or not (they share the context's workspace); ZSTD_freeCCtx waits for them.
 * CUDA graphs: a call made while `stream` is capturing (cudaStreamCaptureModeGlobal or weaker, e.g. torch.cuda.graph) becomes
 * part of the graph, and every replay compresses whatever bytes lie at d_src then.  Precondition: a call of the same shape
 * (sizes, level, parameters, dictionary) on the same context before the capture, completed when the capture starts.  A call
 * that would have to allocate, upload a dictionary or build a table image returns stage_wrong (60) before enqueuing
 * anything.  While such a graph lives, its context must make no other call and must not be freed: replays use its workspace
 * and descriptor slot.
 * ZSTDB200_getLastStats after a stream-ordered call fills launches and nbBlocks only (reading the times would synchronise). */
#define ZSTDB200_ASYNC_SLOTS 4
ZSTDB200_API size_t ZSTDB200_compressDeviceAsync(ZSTD_CCtx* cctx, void* d_dst, size_t dstCapacity, const void* d_src, size_t srcSize,
                                                 int compressionLevel, unsigned long long* d_result, void* stream);
ZSTDB200_API size_t ZSTDB200_compressFramesAsync(ZSTD_CCtx* cctx, void* d_dst, size_t dstCapacity, const void* d_src,
                                                 const size_t* frameOffsets, const size_t* frameSizes, size_t nbFrames,
                                                 const ZSTD_CDict* cdict, int compressionLevel,
                                                 unsigned long long* d_cSizes, unsigned long long* d_result, void* stream);

/* ZSTD_CCtx_refPrefix with the prefix in device memory, for ZSTDB200_compressDevice: nothing of it crosses PCIe and no copy
 * is made (the kernels read it where it lies; it need not be adjacent to the input).  With a NULL stream the producer of
 * d_prefix must have completed before the compression call, as for d_src.  A host-buffer call (ZSTD_compress2,
 * ZSTD_compressStream2) that finds a device prefix pending returns 40 and forgets it.  A host prefix (ZSTD_CCtx_refPrefix)
 * followed by ZSTDB200_compressDevice is fine: the call uploads it. */
ZSTDB200_API size_t ZSTDB200_CCtx_refPrefixDevice(ZSTD_CCtx* cctx, const void* d_prefix, size_t prefixSize);

/* ZSTD_compressSequences with sequences, input and output in device memory (a match finder on the GPU hands its sequences
 * over without a round trip through the host).  d_seqs: nbSeqs ZSTD_Sequence.  `stream`: as for ZSTDB200_compressDevice.
 * Inputs of more than 1024 blocks run in waves of blocks on the one stream.  ZSTDB200_getLastStats: match_ms is the time of
 * the sequence import (partition, validation, conversion). */
ZSTDB200_API size_t ZSTDB200_compressSequencesDevice(ZSTD_CCtx* cctx, void* d_dst, size_t dstCapacity,
                                                     const ZSTD_Sequence* d_seqs, size_t nbSeqs,
                                                     const void* d_src, size_t srcSize, void* stream);

/* ZSTD_generateSequences with input and output in device memory: the parse of the GPU match finder, handed over without a
 * round trip through the host.  d_outSeqs must be 4-byte aligned (parameter_outOfBound (42) otherwise); no row at or past
 * outSeqsCapacity is written.  The Async form follows ZSTDB200_compressDeviceAsync's contract word for word (stream
 * semantics with NULL = the legacy default stream, waves for inputs of 256 MiB or more, ordering with the context's other
 * calls, no host wait once sized, the staging ring, the capture precondition and stage_wrong (60)): *d_result receives the
 * number of rows or an error code (dstSize_tooSmall (70) when they do not fit), in stream order.  The other form is that
 * call plus one read-back of the verdict; its NULL stream means the context's own streams, as for ZSTDB200_compressDevice.
 * Both refuse as ZSTD_generateSequences does, before anything is enqueued.  ZSTDB200_getLastStats: match_ms is the match
 * finder, stitch_ms the export, literals_ms and sequences_ms are 0. */
ZSTDB200_API size_t ZSTDB200_generateSequencesDevice(ZSTD_CCtx* cctx, ZSTD_Sequence* d_outSeqs, size_t outSeqsCapacity,
                                                     const void* d_src, size_t srcSize, void* stream);
ZSTDB200_API size_t ZSTDB200_generateSequencesDeviceAsync(ZSTD_CCtx* cctx, ZSTD_Sequence* d_outSeqs, size_t outSeqsCapacity,
                                                          const void* d_src, size_t srcSize, unsigned long long* d_result, void* stream);

/* One frame compressed by several GPUs (the reference's counterpart: the jobs of ZSTDMT, zstdmt_compress.c:1168-1227 —
 * every job reads an overlap of the input in front of it, only the first writes the frame header, only the last the end
 * mark).  Each rank calls this for its share [partBegin, partBegin + partSize) of a frame of frameSize bytes; partBegin must
 * be a multiple of ZSTDB200_framePartAlignment() and d_part must point at the frame's byte partBegin - min(partBegin,
 * ZSTDB200_framePartHalo()): the rank needs that much of the preceding input.  The ranks' outputs, concatenated in
 * order, are byte for byte the frame a single ZSTDB200_compressDevice call produces (zstd_b200/sharding.py gathers them).
 * No content checksum (ZSTD_c_checksumFlag must be off). */
ZSTDB200_API size_t ZSTDB200_framePartAlignment(void);
ZSTDB200_API size_t ZSTDB200_framePartHalo(void);
ZSTDB200_API size_t ZSTDB200_compressFramePart(ZSTD_CCtx* cctx, void* d_dst, size_t dstCapacity, const void* d_part,
                                               size_t frameSize, size_t partBegin, size_t partSize, int compressionLevel, void* stream);

/* Compress nbFrames independent inputs src[frameOffsets[i] .. +frameSizes[i]) into nbFrames
 * complete frames written back to back into dst (the decoder accepts the concatenation,
 * lib/zstd.h:160-162).  cSizes[i] (host array, may be NULL) receives each frame's size.
 * With dict != NULL every frame is compressed as ZSTD_compress_usingDict would (config 5).
 * `deviceMemory` != 0: src/dst are device pointers (dict and the offset arrays stay on the host).
 * The context's sticky ZSTD_c_checksumFlag / ZSTD_c_dictIDFlag apply to every frame of the call (level and dictionary are arguments). */
ZSTDB200_API size_t ZSTDB200_compressFrames(ZSTD_CCtx* cctx, void* dst, size_t dstCapacity,
                                            const void* src, const size_t* frameOffsets, const size_t* frameSizes,
                                            size_t nbFrames, const void* dict, size_t dictSize,
                                            size_t* cSizes, int compressionLevel, int deviceMemory, void* stream);

/* Same with a digested dictionary (level = the CDict's): what a record store calling
 * ZSTD_compress_usingCDict in a loop would batch (contrib/largeNbDicts/largeNbDicts.c:553). */
ZSTDB200_API size_t ZSTDB200_compressFrames_usingCDict(ZSTD_CCtx* cctx, void* dst, size_t dstCapacity,
                                            const void* src, const size_t* frameOffsets, const size_t* frameSizes,
                                            size_t nbFrames, const ZSTD_CDict* cdict,
                                            size_t* cSizes, int deviceMemory, void* stream);

/* Same with a dictionary per frame, as a record store with one dictionary per table, column, tenant or file uses them
 * (contrib/largeNbDicts/largeNbDicts.c:627-633 walks one CDict per block).  cdicts is a host array of nbFrames pointers,
 * read before the call returns; a CDict may appear any number of times.  Frame i is byte for byte what
 * ZSTD_compress_usingCDict(cctx, ..., cdicts[i]) produces for that record, at that CDict's level, with the sticky
 * checksum, dictID and long-distance-matching parameters as for ZSTDB200_compressFrames_usingCDict; a NULL entry (or
 * cdicts NULL: every entry) compresses the frame without a dictionary at compressionLevel, as ZSTDB200_compressFrames
 * does.  Output layout, cSizes, deviceMemory, stream and the return value are those of
 * ZSTDB200_compressFrames_usingCDict.  The number of kernel launches does not depend on the number of dictionaries:
 * consecutive frames whose parameters are equal share them, whichever dictionary each has.  A CDict's first use uploads
 * it and builds its table images for the call's parameter groups, in bulk for all of the call's new CDicts.  Fails with
 * parameter_unsupported (40) when a frame's level is above 4 under ZSTDB200_setStrictLevels(1), while a prefix is
 * pending, or when a CDict belongs to another device; dstSize_tooSmall (70) when the output does not fit; GENERIC (1)
 * without a device.  A refused call writes nothing. */
ZSTDB200_API size_t ZSTDB200_compressFrames_usingCDicts(ZSTD_CCtx* cctx, void* dst, size_t dstCapacity,
                                            const void* src, const size_t* frameOffsets, const size_t* frameSizes,
                                            size_t nbFrames, const ZSTD_CDict* const* cdicts, int compressionLevel,
                                            size_t* cSizes, int deviceMemory, void* stream);
/* The stream-ordered form, with ZSTDB200_compressFramesAsync's contract (device buffers, verdict and sizes in device
 * memory, ordered with the context's other calls, capturable in a CUDA graph).  Under capture every CDict of the call must
 * already be resident on the device and hold the table images its frames need (a warm call made them so); otherwise the
 * call returns stage_wrong (60) before it enqueues anything. */
ZSTDB200_API size_t ZSTDB200_compressFramesAsync_usingCDicts(ZSTD_CCtx* cctx, void* d_dst, size_t dstCapacity,
                                            const void* d_src, const size_t* frameOffsets, const size_t* frameSizes,
                                            size_t nbFrames, const ZSTD_CDict* const* cdicts, int compressionLevel,
                                            unsigned long long* d_cSizes, unsigned long long* d_result, void* stream);

/* Timing / evidence of the last call on this context (CUDA events on the launching stream). */
typedef struct {
    float  kernel_ms;        /* first kernel start -> last kernel end */
    float  match_ms;         /* K1a candidate walk + K1b parse */
    float  cand_ms, parse_ms; /* K1a, K1b separately (single parameter group only, else 0) */
    float  literals_ms;      /* K2 */
    float  sequences_ms;     /* K3 */
    float  stitch_ms;        /* K4 scan + copy */
    float  total_ms;         /* including host<->device copies, when the call made any */
    unsigned launches;       /* kernels launched by the call */
    unsigned nbBlocks;       /* 128 KiB blocks processed */
    size_t h2d_bytes, d2h_bytes;
} ZSTDB200_stats;
ZSTDB200_API void ZSTDB200_getLastStats(const ZSTD_CCtx* cctx, ZSTDB200_stats* out);

/* Seek table for the frames of a ZSTDB200_compressFrames call (or of several ranks' outputs laid end to end): the
 * reference's seekable format (contrib/seekable_format/zstd_seekable_compression_format.md; its writer is
 * ZSTD_seekable_writeSeekTable, zstdseek_compress.c:297).  Append the bytes behind the frames and the reference's
 * ZSTD_seekable_* readers can decompress any range.  cSizes / dSizes: compressed and decompressed size of every frame
 * (compressed < 4 GiB, decompressed <= 1 GiB each: the format's limit, zstd_seekable.h:19).  Host code.  Returns 17 + 8 * nbFrames, or an error code. */
ZSTDB200_API size_t ZSTDB200_writeSeekTable(void* dst, size_t dstCapacity, const size_t* cSizes, const size_t* dSizes, size_t nbFrames);

/* XXH64 (seed 0) as used for the frame checksum (lib/common/xxhash.h); host code, no GPU (test hook). */
ZSTDB200_API unsigned long long ZSTDB200_xxh64(const void* data, size_t size);

/* The host planner's view of a call, computed without a GPU (test hook: tests/test_plan.py compares it with the
 * oracle's plan).  out: nbFrames x 16 unsigned = strategy, mls, tableN, tableNLong, stepSize, litDisabled, windowLog,
 * insStep, blocks of the frame, first block's size and flags, last block's history reach, dictionary part of the first
 * block's history, chunks of the frame, history walked by the last chunk, size of the last chunk.
 * Returns the total number of blocks. */
ZSTDB200_API size_t ZSTDB200_describePlan(const size_t* frameSizes, size_t nbFrames, int compressionLevel,
                                          size_t dictSize, size_t dictTail, unsigned* out);

/* COMPRESSION LEVELS.  This library implements the reference's `fast` and `doubleFast` strategies, i.e. negative
 * levels and levels 1-4 (clevels.h:25-50; level 4 only for inputs > 256 KiB).  A level whose reference strategy is
 * greedy or stronger (5 ... 22) is NOT implemented: by default such a call is served by the strongest doubleFast row
 * of its size class and returns a valid frame that is LARGER (typically 20-40 %) than what the reference produces at
 * that level.  ZSTDB200_setStrictLevels(1) turns that into ZSTD_error_parameter_unsupported for the whole process. */
ZSTDB200_API void ZSTDB200_setStrictLevels(int on);

/* Which CUDA device contexts created FROM NOW ON belong to (default: the creating thread's current device).  A context
 * keeps the device it was created for; every call restores the calling thread's current device before it returns. */
ZSTDB200_API int  ZSTDB200_setDevice(int device);
ZSTDB200_API int  ZSTDB200_deviceAvailable(void);

#ifdef __cplusplus
}
#endif
#endif /* ZSTD_B200_H */
