/* zb_kernels.h — launch shims of the CUDA kernels (C linkage, called by the host driver zb_api.cu). */
#ifndef ZB_KERNELS_H
#define ZB_KERNELS_H
#include <cuda_runtime.h>
#include "zb_common.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Every launch of K1..K4 works on the workspace rows [0, nbBlocks) (zb_workLayout, zb_common.h), one per block of the
 * launch: K1, K1s-b and K4 take them as `rows`.
 * d_dicts: the call's dictionary table (ZbDictSlot, zb_common.h), indexed by the dictSlot of a frame's first chunk and
 * first block; NULL when no frame of the launch has a dictionary.
 * K1: match-finder = K1a candidate walk (one CTA per chunk) + K1b greedy parse (one warp per 16 KiB segment) + K1c merge.
 * d_blocks / d_chunks point at the first block / chunk of the launch; slotFirstBlock = index (in the call's block array)
 * of the block that owns row 0.  Writes meta, seqs and lits; dist, far, segmeta (and doubleFast's dist2, far2) are its
 * own scratch.
 * Chunks / blocks with dictLen > 0 take the oldest dictLen bytes of their history from in front of their dictionary
 * entry's end; a first chunk starts from the entry's image when it has one (built by zb_launch_dict_images under the
 * same ZbParams).  dict: some block of the launch has ZB_FLAG_DICT (the parse's variant that reads two buffers).
 * zb_launch_dict_images: one CTA per image, image i walks the tail of d_dicts[d_imageChunks[i].dictSlot] (a chunk of
 * size 0 whose history is that tail) into that entry's image. */
cudaError_t zb_launch_dict_images(const ZbDictSlot* d_dicts, const ZbChunk* d_imageChunks, u32 nbImages, const ZbParams* prm, cudaStream_t stream);
/* K1a alone, one table (zb_launch_match runs it once per table; the walk test harness, tests/walk_harness.cu, on its own):
 * one CTA per chunk walks the chunk's history and bytes with `mls`-byte hashes into a table of N buckets (N * 4 bytes of
 * shared memory, at most 226 KiB).  build = false: writes dist (u16, ZB_FAR = see far) and far (u32, only where dist is
 * ZB_FAR) at [0, size) of row firstBlock - slotFirstBlock + k of block k of each chunk (rows sd.dist apart), and nothing
 * else.  build = true (d_src NULL): walks each chunk's dictionary tail and writes the table to d_dicts[dictSlot].image +
 * imageOff (N u32), and nothing else.  A first chunk whose dictionary entry has an image starts from image + imageOff. */
cudaError_t zb_launch_walk(const u8* d_src, const ZbDictSlot* d_dicts, const ZbChunk* d_chunks, u32 nbChunks, u32 mls, u32 N, u32 insStep,
                           const ZbStrides& sd, u32 slotFirstBlock, u16* d_dist, u32* d_far, u32 imageOff, bool build, cudaStream_t stream);
cudaError_t zb_launch_match(const u8* d_src, const ZbDictSlot* d_dicts, bool dict, const ZbBlock* d_blocks, u32 nbBlocks,
                            const ZbChunk* d_chunks, u32 nbChunks, u32 slotFirstBlock, const ZbParams* prm, const ZbWorkRows* rows,
                            cudaEvent_t evMid, cudaStream_t stream, const ZbLdmView* ldm = nullptr);
/* ldm (K1c): the launch's blocks' long-distance matches (zb_launch_ldm), laid over the parse output; NULL = none */
/* K1c alone (zb_launch_match runs it behind the parse; the merge test harness, tests/merge_harness.cu, on its own): joins
 * each block's parse segments, assigns the repcodes and gathers the literals.  zb_merge_small_kernel (one warp per block)
 * when the rows hold one segment of at most 8192 bytes, else zb_merge_segments_kernel (one CTA per block), its LDM variant
 * when ldm is given.  Reads, for each block b of at least 7 bytes: rows->segmeta (zb_segsPerRow records of row b), the
 * raw sequences (zb_pack_raw) of segment k at seq slot k * ZB_PARSE_SEG / 4 of row b, d_src at the block, d_blocks[b],
 * d_dicts[dictSlot].codeRep of a first block (d_dicts NULL: {1,4,8}) and, for LDM, ldm->match[first[b], + cnt[b]).
 * Writes seqs[0, nbSeq) (zb_pack_seq: offBase, litLength, matchLength), lits[0, litSize) and meta of those blocks, and
 * for LDM the block's far and dist rows as scratch; blocks of fewer than 7 bytes (meta written by the parse) not at all. */
cudaError_t zb_launch_merge(const u8* d_src, const ZbDictSlot* d_dicts, const ZbBlock* d_blocks, u32 nbBlocks, const ZbWorkRows* rows,
                            const ZbLdmView* ldm, cudaStream_t stream);

/* Long-distance matching of one frame of n bytes at d_frame behind P indexed prefix bytes at d_prefix (P = 0: none; the two
 * need not be adjacent) (zb_ldm.cu): nbBlocks blocks of ZB_BLOCK_MAX bytes, the frame's; block k's matches go to
 * d_match[d_ldmFirst[k] .. + d_ldmCnt[k]), inside d_match[matchBase, matchBase + zb_ldm_survivor_cap(P + n, minMatch)).
 * d_scratch: zb_ldm_scratch_bytes(P, n, prm) bytes, free again when the stream reaches the end of the launch. */
size_t zb_ldm_scratch_bytes(u64 P, u64 n, const ZbLdmParams* prm);
cudaError_t zb_launch_ldm(const u8* d_prefix, u64 P, const u8* d_frame, u64 n, const ZbLdmParams* prm, void* d_scratch, u32 nbBlocks,
                          u64 matchBase, u64* d_match, u64* d_ldmFirst, u32* d_ldmCnt, cudaStream_t stream);

/* K1s: caller-supplied sequences (ZSTD_Sequence[n], 16-byte aligned, device memory) in place of K1 (zb_seqimport.cu).
 * partition: per-tile sums (d_tileLen / d_tileEnds: one per 1024 sequences), scanned; d_ctrl[0] = sum of the lengths,
 * d_ctrl[1] = delimiters that close a non-empty block (expl != 0).  place: validation (d_ctrl[2] = first invalid index,
 * to be preset to ~0) and the block starts: explicit delimiters -> d_blockEnd / d_blockSeq per closing delimiter, else
 * d_blockFirst / d_blockFirstPos of the nbBlocks blocks of blockMax bytes (preset d_blockFirst to ~0).  blocks (explicit
 * only): the ZbBlock table, d_blockFirst / d_blockFirstPos, d_ctrl[3] = end of the last block.  convert (K1s-b): the
 * blocks' triples, literals and meta into the workspace rows (ZB_WORK_SEQUENCES, strides zb_seq_strides). */
cudaError_t zb_launch_seq_partition(const void* d_seqs, u32 n, int expl, u64* d_tileLen, u32* d_tileEnds, u64* d_ctrl, cudaStream_t stream);
cudaError_t zb_launch_seq_place(const void* d_seqs, u32 n, int expl, const u64* d_tileLen, const u32* d_tileEnds,
                                u64 srcSize, u64 window, u64 dictContent, u32 blockMax, u32 nbBlocks,
                                u64* d_blockEnd, u32* d_blockSeq, u32* d_blockFirst, u64* d_blockFirstPos, u64* d_ctrl, cudaStream_t stream);
cudaError_t zb_launch_seq_blocks(const u64* d_blockEnd, const u32* d_blockSeq, u32 nbBlocks, u32 blockMax, u32 dictFlag,
                                 ZbBlock* d_blocks, u32* d_blockFirst, u64* d_blockFirstPos, u64* d_ctrl, cudaStream_t stream);
cudaError_t zb_launch_seq_convert(const u8* d_src, const ZbBlock* d_blocks, u32 nbBlocks, const u32* d_blockFirst, const u64* d_blockFirstPos,
                                  const void* d_seqs, u32 n, const ZbDictSlot* d_dicts, const ZbWorkRows* rows, cudaStream_t stream);

/* host: the format's predefined FSE tables (zb_dict.cu), and their upload to the current device (zb_sequences.cu) */
void zb_buildDefaultTables(ZbdFseCTable* out3);
cudaError_t zb_upload_default_tables(const ZbdFseCTable* host3, cudaStream_t stream);

/* host: parse a dictionary (zb_dict.cu).  Returns the content offset, 0 for raw content, or an error code */
size_t zb_loadDictionary(ZbDictEntropy* de, const u8* dict, size_t dictSize);

/* K2 and K3 take their arrays one by one: the entropy test harness (tests/entropy_harness.cu) runs them over allocations
 * of its own.  The driver passes the workspace rows of the launch (K3's d_stateBits: the dist rows, see zb_workLayout). */
/* K2: literals section (histogram, Huffman table, 1/4-stream encode).  One CTA per block.
 * The entropy state a frame's first block starts from: its dictionary entry's when d_dicts is given (the driver), else d_de
 * (NULL: none) for every first block (the entropy harness). */
cudaError_t zb_launch_literals(const ZbBlock* d_blocks, u32 nbBlocks, const ZbParams* prm, const ZbStrides* sd, const ZbDictEntropy* d_de,
                               const u8* d_lits, u8* d_body, ZbBlockMeta* d_meta, cudaStream_t stream, const ZbDictSlot* d_dicts = nullptr);

/* K3: sequences section (codes, histograms, FSE tables, tANS bit-stream) + block-type decision. */
cudaError_t zb_launch_sequences(const u8* d_src, const ZbBlock* d_blocks, u32 nbBlocks, const ZbParams* prm, const ZbStrides* sd, const ZbDictEntropy* d_de,
                                const u64* d_seqs, u16* d_stateBits, u8* d_body, ZbBlockMeta* d_meta, cudaStream_t stream,
                                const ZbDictSlot* d_dicts = nullptr);

/* K4: stitch — per-block output sizes -> exclusive scan -> frame/block headers + payload copy, for
 * one wave of blocks, from the body and meta rows.  d_blocks/d_outOffsets point at the wave's first block;
 * d_outOffsets gets nbBlocks+1 absolute offsets, starting at *d_base (NULL = 0); *d_total receives
 * the running total after this wave (even past dstCapacity: nothing is written past dst+dstCapacity). */
cudaError_t zb_launch_stitch(const u8* d_src, const ZbBlock* d_blocks, u32 nbBlocks, const ZbFrame* d_frames, const ZbWorkRows* rows,
                             u64* d_outOffsets, const u64* d_base, u64* d_total,
                             u8* d_dst, u64 dstCapacity, cudaStream_t stream);
cudaError_t zb_launch_checksums(const u8* d_src, const ZbFrame* d_frames, u32 nbFrames, const u64* d_outOffsets, u8* d_dst, u64 dstCapacity, cudaStream_t stream);
/* The tail of a ZSTD_generateSequences wave in place of K2..K4 (zb_seqexport.cu): K1c's stores of the wave's blocks, from the
 * seqs and meta rows, as ZSTD_Sequence rows at d_out (4-byte aligned): each block's sequences with real offsets and the
 * repcode the block codes them with (history: d_dicts[dictSlot].codeRep at a frame's first block, {1,4,8} without a
 * table, unknown elsewhere), then its delimiter {0, trailing literals, 0, 0}.  d_offsets gets nbBlocks + 1 row indices,
 * starting at *d_base (NULL = 0); *d_total the running count after this wave.  No row at or past `capacity` is written. */
cudaError_t zb_launch_seqexport(const ZbBlock* d_blocks, u32 nbBlocks, const ZbDictSlot* d_dicts, const ZbWorkRows* rows,
                                u64* d_offsets, const u64* d_base, u64* d_total, void* d_out, u64 capacity, cudaStream_t stream);
/* the last kernel of a call: d_cSizes[f] (d_cSizes may be NULL) and *d_result = *d_total, or dstSize_tooSmall
 * when *d_total > dstCapacity; d_total NULL (no frames): 0 */
cudaError_t zb_launch_call_result(const ZbFrame* d_frames, u32 nbFrames, const u64* d_outOffsets, const u64* d_total,
                                  u64 dstCapacity, unsigned long long* d_cSizes, unsigned long long* d_result, cudaStream_t stream);

#ifdef __cplusplus
}
#endif
#endif
