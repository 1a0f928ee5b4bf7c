/* merge_harness.cu — TEST INFRASTRUCTURE ONLY.  Runs the product's merge, zb_launch_merge (K1c: segment join, repcodes,
 * literal gather, meta; its LDM variant lays a block's long-distance matches over the joined sequences), on chosen raw
 * sequences without the walk or the parse in front of it, and the caller-sequence path K1s (zb_launch_seq_partition,
 * _place, _blocks, _convert) on chosen sequences.  Linked against the product's own zb_match.o and zb_seqimport.o
 * (zstd_b200/csrc/Makefile, target `harness`), so the kernels under test are the ones the library ships.  Used by
 * tests/test_gpu_merge_paths.py. */
#include <string.h>
#include <vector>
#include "../zstd_b200/csrc/zb_common.h"
#include "../zstd_b200/csrc/zb_kernels.h"

#define ZBH_PAD 64u              /* zero bytes in front of and behind the source */
#define ZBH_SEG_SLOTS (ZB_PARSE_SEG / 4u)

/* One K1c launch over nbBlocks blocks.  Block b is src[blockOff[b], + blockSize[b]), flags[b] its ZB_FLAG_* (FIRST: the
 * repcode history starts from codeRep[3b .. 3b + 3), held in dictionary slot b; useDicts = 0 passes no dictionary table,
 * and first blocks start from {1,4,8}).  Its segment k (k < ZB_PARSE_SEGS) has segCnt[b * ZB_PARSE_SEGS + k] raw
 * sequences, taken in order from raw (u32 triples: match start relative to the block, match length, offset), packed with
 * zb_pack_raw into seq slot k * ZB_PARSE_SEG / 4 of row b.  ldm = 1: the LDM variant, block b's matches are ldmCnt[b] u32
 * triples (start, length, offset) taken in order from ldmM, packed with zb_pack_ldm.
 *   rowSize: the rows' strides are zb_strides(rowSize) (0: the largest block); rowSize <= 8192 with one segment per row
 *            takes zb_merge_small_kernel
 *   sent:    two sentinel bytes.  The launch runs twice; before run r the raw sequences are loaded again and the seq, lit,
 *            meta, far and dist rows are filled with sent[r] (the seq rows first, then the raw sequences over them)
 *   seqs, lits, meta: 2 x rows x sd.seq u64, 2 x rows x sd.lit bytes, 2 x rows ZbBlockMeta (8 u32), run r at r x rows x that
 *   shape:   sd.seq, sd.lit, sd.dist, zb_segsPerRow (written first, also when the capacities are too small)
 * Returns 0, a CUDA error code, or a negative value for bad arguments.  Every allocation is freed before it returns. */
extern "C" __attribute__((visibility("default")))
int zbh_merge(const u8* src, u64 srcLen, u32 nbBlocks, const u64* blockOff, const u32* blockSize, const u32* flags, const u32* codeRep,
              u32 useDicts, const u32* segCnt, const u32* raw, u64 nbRaw, u32 ldm, const u32* ldmCnt, const u32* ldmM, u64 nbLdm,
              u32 rowSize, const u8* sent, u64* seqs, u64 seqCap, u8* lits, u64 litCap, u32* meta, u64 metaCap, u64* shape)
{
    if (nbBlocks == 0 || ldm > 1 || useDicts > 1) return -1;
    u32 maxBlock = 0;
    for (u32 b = 0; b < nbBlocks; b++) {
        if (blockSize[b] == 0 || blockSize[b] > ZB_BLOCK_MAX || blockOff[b] > srcLen || blockSize[b] > srcLen - blockOff[b]) return -1;
        if (blockSize[b] > maxBlock) maxBlock = blockSize[b];
    }
    if (rowSize && rowSize < maxBlock) return -1;
    ZbStrides const sd = zb_strides(rowSize ? rowSize : maxBlock);
    u32 const segStride = zb_segsPerRow(sd);
    shape[0] = sd.seq; shape[1] = sd.lit; shape[2] = sd.dist; shape[3] = segStride;
    u64 const seqCells = (u64)nbBlocks * sd.seq, litCells = (u64)nbBlocks * sd.lit;
    if (seqCap < 2 * seqCells || litCap < 2 * litCells || metaCap < 2ull * nbBlocks * 8u) return -2;
    /* the rows as the parse leaves them */
    std::vector<u64> hostSeq(seqCells, 0);
    std::vector<ZbSegMeta> hostSeg((size_t)nbBlocks * segStride);
    std::vector<u64> hostLdm, ldmFirst(nbBlocks, 0);
    std::vector<ZbDictSlot> slots(nbBlocks);
    memset(hostSeg.data(), 0, hostSeg.size() * sizeof(ZbSegMeta));
    u64 ri = 0, li = 0;
    for (u32 b = 0; b < nbBlocks; b++) {
        u32 const segs = (blockSize[b] + ZB_PARSE_SEG - 1u) / ZB_PARSE_SEG;
        u64 total = 0;
        for (u32 k = 0; k < ZB_PARSE_SEGS; k++) {
            u32 const c = segCnt[(size_t)b * ZB_PARSE_SEGS + k];
            if (c && (k >= segs || k >= segStride || c > ZBH_SEG_SLOTS || (u64)k * ZBH_SEG_SLOTS + c > sd.seq || ri + c > nbRaw)) return -1;
            if (k < segStride) hostSeg[(size_t)b * segStride + k].nbSeq = c;
            for (u32 i = 0; i < c; i++, ri++) {
                u32 const ms = raw[3 * ri], ml = raw[3 * ri + 1], off = raw[3 * ri + 2];
                if (ms >= blockSize[b] || ml > blockSize[b] - ms || ml >= (1u << 18) || off >= (1u << 24)) return -1;
                hostSeq[(size_t)b * sd.seq + (size_t)k * ZBH_SEG_SLOTS + i] = zb_pack_raw(off, ml, ms);
            }
            total += c;
        }
        if (ldm) {
            ldmFirst[b] = hostLdm.size();
            if (li + ldmCnt[b] > nbLdm || total + ldmCnt[b] > sd.seq) return -1;
            for (u32 i = 0; i < ldmCnt[b]; i++, li++) {
                u32 const s = ldmM[3 * li], l = ldmM[3 * li + 1], off = ldmM[3 * li + 2];
                if (s >= blockSize[b] || l > blockSize[b] - s || off >= (1u << 28)) return -1;
                hostLdm.push_back(zb_pack_ldm(s, l, off));
            }
        }
        memset(&slots[b], 0, sizeof(ZbDictSlot));
        slots[b].codeRep[0] = codeRep[3 * b]; slots[b].codeRep[1] = codeRep[3 * b + 1]; slots[b].codeRep[2] = codeRep[3 * b + 2];
    }
    if (ri != nbRaw || (ldm && li != nbLdm)) return -1;
    std::vector<ZbBlock> blocks(nbBlocks);
    for (u32 b = 0; b < nbBlocks; b++) {
        memset(&blocks[b], 0, sizeof(ZbBlock));
        blocks[b].srcOff = ZBH_PAD + blockOff[b]; blocks[b].size = blockSize[b]; blocks[b].flags = flags[b]; blocks[b].dictSlot = b;
    }
    size_t const workBytes = zb_workLayout(nullptr, nbBlocks, ZB_WORK_FAST, sd, nullptr);
    if (zb_isErr(workBytes)) return -1;

    u8 *d_src = nullptr, *d_work = nullptr; ZbBlock* d_blocks = nullptr; ZbDictSlot* d_dicts = nullptr;
    u64 *d_ldm = nullptr, *d_ldmFirst = nullptr; u32* d_ldmCnt = nullptr;
    ZbWorkRows w; ZbLdmView view;
    cudaStream_t st = nullptr;
    cudaError_t e;
#define HK(x) do { if ((e = (x)) != cudaSuccess) goto out; } while (0)
    HK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    HK(cudaMalloc(&d_src, srcLen + 2 * ZBH_PAD));
    HK(cudaMalloc(&d_work, workBytes));
    HK(cudaMalloc(&d_blocks, nbBlocks * sizeof(ZbBlock)));
    HK(cudaMalloc(&d_dicts, nbBlocks * sizeof(ZbDictSlot)));
    HK(cudaMalloc(&d_ldm, (hostLdm.size() + 1) * sizeof(u64)));
    HK(cudaMalloc(&d_ldmFirst, nbBlocks * sizeof(u64)));
    HK(cudaMalloc(&d_ldmCnt, nbBlocks * sizeof(u32)));
    zb_workLayout(d_work, nbBlocks, ZB_WORK_FAST, sd, &w);
    view.match = d_ldm; view.first = d_ldmFirst; view.cnt = d_ldmCnt;
    HK(cudaMemsetAsync(d_src, 0, srcLen + 2 * ZBH_PAD, st));
    HK(cudaMemcpyAsync(d_src + ZBH_PAD, src, srcLen, cudaMemcpyHostToDevice, st));
    HK(cudaMemcpyAsync(d_blocks, blocks.data(), nbBlocks * sizeof(ZbBlock), cudaMemcpyHostToDevice, st));
    HK(cudaMemcpyAsync(d_dicts, slots.data(), nbBlocks * sizeof(ZbDictSlot), cudaMemcpyHostToDevice, st));
    if (!hostLdm.empty()) HK(cudaMemcpyAsync(d_ldm, hostLdm.data(), hostLdm.size() * sizeof(u64), cudaMemcpyHostToDevice, st));
    HK(cudaMemcpyAsync(d_ldmFirst, ldmFirst.data(), nbBlocks * sizeof(u64), cudaMemcpyHostToDevice, st));
    if (ldm) HK(cudaMemcpyAsync(d_ldmCnt, ldmCnt, nbBlocks * sizeof(u32), cudaMemcpyHostToDevice, st));
    HK(cudaMemcpyAsync(w.segmeta, hostSeg.data(), hostSeg.size() * sizeof(ZbSegMeta), cudaMemcpyHostToDevice, st));
    for (int r = 0; r < 2; r++) {
        HK(cudaMemsetAsync(w.lits, sent[r], litCells, st));
        HK(cudaMemsetAsync(w.meta, sent[r], nbBlocks * sizeof(ZbBlockMeta), st));
        HK(cudaMemsetAsync(w.far, sent[r], (size_t)nbBlocks * sd.dist * sizeof(u32), st));
        HK(cudaMemsetAsync(w.dist, sent[r], (size_t)nbBlocks * sd.dist * sizeof(u16), st));
        HK(cudaMemsetAsync(w.seqs, sent[r], seqCells * sizeof(u64), st));
        for (u32 b = 0; b < nbBlocks; b++)                       /* the raw sequences of every segment, around them the sentinel */
            for (u32 k = 0; k < segStride; k++) {
                u32 const c = hostSeg[(size_t)b * segStride + k].nbSeq;
                size_t const at = (size_t)b * sd.seq + (size_t)k * ZBH_SEG_SLOTS;
                if (c) HK(cudaMemcpyAsync(w.seqs + at, hostSeq.data() + at, c * sizeof(u64), cudaMemcpyHostToDevice, st));
            }
        HK(zb_launch_merge(d_src, useDicts ? d_dicts : nullptr, d_blocks, nbBlocks, &w, ldm ? &view : nullptr, st));
        HK(cudaMemcpyAsync(seqs + r * seqCells, w.seqs, seqCells * sizeof(u64), cudaMemcpyDeviceToHost, st));
        HK(cudaMemcpyAsync(lits + r * litCells, w.lits, litCells, cudaMemcpyDeviceToHost, st));
        HK(cudaMemcpyAsync(meta + (size_t)r * nbBlocks * 8u, w.meta, nbBlocks * sizeof(ZbBlockMeta), cudaMemcpyDeviceToHost, st));
    }
    HK(cudaStreamSynchronize(st));
    HK(cudaGetLastError());
#undef HK
out:
    cudaFree(d_src); cudaFree(d_work); cudaFree(d_blocks); cudaFree(d_dicts); cudaFree(d_ldm); cudaFree(d_ldmFirst); cudaFree(d_ldmCnt);
    if (st) cudaStreamDestroy(st);
    return (int)e;
}

/* One frame of caller sequences through K1s: n ZSTD_Sequence records (u32 x 4: offset, litLength, matchLength, rep) with
 * explicit block delimiters over src[0, srcLen), blocks of at most ZB_BLOCK_MAX bytes, offsets valid up to the
 * product's bound (dictContent = 2^24 bytes of history assumed in front of the frame).  useDict = 1: the frame's first
 * block starts from codeRep[0..3) (a dictionary table of one entry), else from {1,4,8}.  Rows are zb_seq_strides of
 * ZB_BLOCK_MAX.  The launch runs twice, with the seq, lit and meta rows filled with sent[r] before run r.
 *   seqs, lits, meta: 2 x nbBlocks x sd.seq u64, x sd.lit bytes, x 8 u32 (nbBlocks = the closing delimiters)
 *   ctrl: 4 u64 as K1s leaves them (sum of lengths, closing delimiters, first invalid index or ~0, end of the last block)
 *   shape: sd.seq, sd.lit, nbBlocks (written first, also when the capacities are too small)
 * Returns 0, a CUDA error code, or a negative value for bad arguments (-2: capacities, -3: no closing delimiter).  Every
 * allocation is freed before it returns. */
extern "C" __attribute__((visibility("default")))
int zbh_seq_convert(const u8* src, u64 srcLen, const u32* seqIn, u32 n, const u32* codeRep, u32 useDict, const u8* sent,
                    u64* seqs, u64 seqCap, u8* lits, u64 litCap, u32* meta, u64 metaCap, u64* ctrlOut, u64* shape)
{
    if (n == 0 || srcLen == 0 || useDict > 1) return -1;
    ZbStrides const sd = zb_seq_strides(ZB_BLOCK_MAX);
    u32 const nbTiles = (n + 1023u) / 1024u;
    u64 ctrl[4] = { 0, 0, ~0ull, 0 };
    u32 nbBlocks = 0;
    size_t workBytes = 0;
    ZbDictSlot slot;
    memset(&slot, 0, sizeof(slot));
    slot.codeRep[0] = codeRep[0]; slot.codeRep[1] = codeRep[1]; slot.codeRep[2] = codeRep[2];
    shape[0] = sd.seq; shape[1] = sd.lit; shape[2] = 0;
    u8 *d_src = nullptr, *d_work = nullptr, *d_blk = nullptr; void* d_seqs = nullptr; u64 *d_tile = nullptr, *d_ctrl = nullptr;
    ZbBlock* d_blocks = nullptr; ZbDictSlot* d_dicts = nullptr;
    u64 *d_firstPos = nullptr, *d_blockEnd = nullptr; u32 *d_first = nullptr, *d_blockSeq = nullptr;
    ZbWorkRows w;
    u64 seqCells = 0, litCells = 0;
    cudaStream_t st = nullptr;
    cudaError_t e;
    int bad = 0;
#define HK(x) do { if ((e = (x)) != cudaSuccess) goto out; } while (0)
#define HB(c, v) do { if (c) { bad = (v); e = cudaSuccess; goto out; } } while (0)
    HK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    HK(cudaMalloc(&d_src, srcLen + 2 * ZBH_PAD));
    HK(cudaMalloc(&d_seqs, (size_t)n * 16u));
    HK(cudaMalloc(&d_tile, (size_t)nbTiles * 12u + 16u));
    HK(cudaMalloc(&d_ctrl, sizeof(ctrl)));
    HK(cudaMalloc(&d_dicts, sizeof(ZbDictSlot)));
    HK(cudaMemsetAsync(d_src, 0, srcLen + 2 * ZBH_PAD, st));
    HK(cudaMemcpyAsync(d_src + ZBH_PAD, src, srcLen, cudaMemcpyHostToDevice, st));
    HK(cudaMemcpyAsync(d_seqs, seqIn, (size_t)n * 16u, cudaMemcpyHostToDevice, st));
    HK(cudaMemcpyAsync(d_ctrl, ctrl, sizeof(ctrl), cudaMemcpyHostToDevice, st));
    HK(cudaMemcpyAsync(d_dicts, &slot, sizeof(slot), cudaMemcpyHostToDevice, st));
    HK(zb_launch_seq_partition(d_seqs, n, 1, d_tile, (u32*)(d_tile + nbTiles), d_ctrl, st));
    HK(cudaMemcpyAsync(ctrl, d_ctrl, 2 * sizeof(u64), cudaMemcpyDeviceToHost, st));
    HK(cudaStreamSynchronize(st));
    HB(ctrl[1] == 0, -3);
    nbBlocks = (u32)ctrl[1];
    shape[2] = nbBlocks;
    seqCells = (u64)nbBlocks * sd.seq; litCells = (u64)nbBlocks * sd.lit;
    HB(seqCap < 2 * seqCells || litCap < 2 * litCells || metaCap < 2ull * nbBlocks * 8u, -2);
    workBytes = zb_workLayout(nullptr, nbBlocks, ZB_WORK_SEQUENCES, sd, nullptr);
    HB(zb_isErr(workBytes), -1);
    HK(cudaMalloc(&d_work, workBytes));
    HK(cudaMalloc(&d_blocks, nbBlocks * sizeof(ZbBlock)));
    HK(cudaMalloc(&d_blk, (size_t)nbBlocks * 24u + 16u));
    zb_workLayout(d_work, nbBlocks, ZB_WORK_SEQUENCES, sd, &w);
    d_firstPos = (u64*)d_blk; d_blockEnd = d_firstPos + nbBlocks; d_first = (u32*)(d_blockEnd + nbBlocks); d_blockSeq = d_first + nbBlocks;
    HK(zb_launch_seq_place(d_seqs, n, 1, d_tile, (u32*)(d_tile + nbTiles), srcLen, 1ull << ZB_LDM_WINDOW_LOG, 1ull << 24, ZB_BLOCK_MAX,
                           nbBlocks, d_blockEnd, d_blockSeq, d_first, d_firstPos, d_ctrl, st));
    HK(zb_launch_seq_blocks(d_blockEnd, d_blockSeq, nbBlocks, ZB_BLOCK_MAX, 0u, d_blocks, d_first, d_firstPos, d_ctrl, st));
    for (int r = 0; r < 2; r++) {
        HK(cudaMemsetAsync(w.seqs, sent[r], seqCells * sizeof(u64), st));
        HK(cudaMemsetAsync(w.lits, sent[r], litCells, st));
        HK(cudaMemsetAsync(w.meta, sent[r], nbBlocks * sizeof(ZbBlockMeta), st));
        HK(zb_launch_seq_convert(d_src + ZBH_PAD, d_blocks, nbBlocks, d_first, d_firstPos, d_seqs, n, useDict ? d_dicts : nullptr, &w, st));
        HK(cudaMemcpyAsync(seqs + r * seqCells, w.seqs, seqCells * sizeof(u64), cudaMemcpyDeviceToHost, st));
        HK(cudaMemcpyAsync(lits + r * litCells, w.lits, litCells, cudaMemcpyDeviceToHost, st));
        HK(cudaMemcpyAsync(meta + (size_t)r * nbBlocks * 8u, w.meta, nbBlocks * sizeof(ZbBlockMeta), cudaMemcpyDeviceToHost, st));
    }
    HK(cudaMemcpyAsync(ctrlOut, d_ctrl, sizeof(ctrl), cudaMemcpyDeviceToHost, st));
    HK(cudaStreamSynchronize(st));
    HK(cudaGetLastError());
#undef HK
#undef HB
out:
    cudaFree(d_src); cudaFree(d_work); cudaFree(d_blk); cudaFree(d_seqs); cudaFree(d_tile); cudaFree(d_ctrl); cudaFree(d_blocks); cudaFree(d_dicts);
    if (st) cudaStreamDestroy(st);
    return bad ? bad : (int)e;
}
