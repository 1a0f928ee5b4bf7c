/* entropy_harness.cu — TEST INFRASTRUCTURE ONLY.  Runs the product's entropy stage, K2 (zb_launch_literals) and K3
 * (zb_launch_sequences), on chosen sequences and literals, without the match finder in front of it.  Linked against the
 * product's own zb_literals.o, zb_sequences.o and zb_dict.o (zstd_b200/csrc/Makefile, target `harness`), so the kernels
 * under test are the ones the library ships.  Used by tests/test_gpu_entropy.py. */
#include <string.h>
#include <vector>
#include "../zstd_b200/csrc/zb_common.h"
#include "../zstd_b200/csrc/zb_kernels.h"

/* One launch of K2 then K3 over nbBlocks blocks on one stream, workspace strides derived from the largest block.
 *   src / srcSize:     the blocks' bytes; blocks[b].srcOff, .size and .flags (ZB_FLAG_FIRST, ZB_FLAG_DICT) describe block b
 *   seqs:              (offBase, litLen, matchLen) triples of all blocks, block after block; nbSeq[b] of them for block b
 *   lits:              the literal bytes of all blocks, block after block; litSize[b] of them for block b
 *   dict / dictSize:   a dictionary (NULL: none); a zstd-format one gives FIRST blocks its entropy tables
 * Out: meta[b]; body[b * bodyStride ...] holds block b's staging area (bodyCap >= nbBlocks * bodyStride);
 *   guard[guardSize]: the bytes behind the last block's area; the whole area and these were `guardByte` before the launch.
 * Returns 0, or a CUDA error code (negative: bad arguments). */
extern "C" __attribute__((visibility("default")))
int zbh_entropy(const u8* src, size_t srcSize, const ZbBlock* blocks, u32 nbBlocks, const u32* seqs, const u32* nbSeq,
                const u8* lits, const u32* litSize, u32 strategy, u32 litDisabled, const u8* dict, size_t dictSize,
                u8 guardByte, ZbBlockMeta* meta, u8* body, size_t bodyCap, u32* bodyStride, u8* guard, size_t guardSize)
{
    u32 maxBlock = 0;
    for (u32 b = 0; b < nbBlocks; b++) maxBlock = blocks[b].size > maxBlock ? blocks[b].size : maxBlock;
    ZbStrides const sd = zb_strides(maxBlock);
    *bodyStride = sd.body;
    if (nbBlocks == 0 || bodyCap < (size_t)nbBlocks * sd.body) return -1;

    std::vector<u64> hseq((size_t)nbBlocks * sd.seq, 0);
    std::vector<u8> hlit((size_t)nbBlocks * sd.lit, 0);
    std::vector<ZbBlockMeta> hmeta(nbBlocks);
    size_t sq = 0, lt = 0;
    for (u32 b = 0; b < nbBlocks; b++) {
        if (nbSeq[b] > sd.seq - 8u || litSize[b] > sd.lit - 256u || blocks[b].srcOff + blocks[b].size > srcSize) return -2;
        for (u32 i = 0; i < nbSeq[b]; i++, sq++)
            hseq[(size_t)b * sd.seq + i] = zb_pack_seq(seqs[3 * sq], seqs[3 * sq + 1], seqs[3 * sq + 2]);
        memcpy(&hlit[(size_t)b * sd.lit], lits + lt, litSize[b]);
        lt += litSize[b];
        memset(&hmeta[b], 0, sizeof(ZbBlockMeta));
        hmeta[b].nbSeq = nbSeq[b]; hmeta[b].litSize = litSize[b]; hmeta[b].forceRaw = 0;
    }
    ZbDictEntropy de;
    if (zb_isErr(zb_loadDictionary(&de, dict, dictSize))) return -3;
    ZbParams prm;
    memset(&prm, 0, sizeof(prm));
    prm.strategy = strategy; prm.litDisabled = litDisabled;

    /* the predefined FSE tables, once per device */
    static bool uploaded[64];
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return (int)e;
    if (dev < 64 && !uploaded[dev]) {
        static ZbdFseCTable defaults[3];
        zb_buildDefaultTables(defaults);
        if ((e = zb_upload_default_tables(defaults, 0)) != cudaSuccess || (e = cudaDeviceSynchronize()) != cudaSuccess) return (int)e;
        uploaded[dev] = true;
    }

    size_t const bodyBytes = (size_t)nbBlocks * sd.body;
    u8 *d_src = nullptr, *d_lits = nullptr, *d_body = nullptr; u64* d_seqs = nullptr; u16* d_state = nullptr;
    ZbBlock* d_blocks = nullptr; ZbBlockMeta* d_meta = nullptr; ZbDictEntropy* d_de = nullptr;
    cudaStream_t st = nullptr;
#define HK(x) do { if ((e = (x)) != cudaSuccess) goto out; } while (0)
    HK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    HK(cudaMalloc(&d_src, srcSize ? srcSize : 1));
    HK(cudaMalloc(&d_lits, hlit.size()));
    HK(cudaMalloc(&d_seqs, hseq.size() * sizeof(u64)));
    HK(cudaMalloc(&d_state, (size_t)nbBlocks * sd.dist * sizeof(u16)));
    HK(cudaMalloc(&d_body, bodyBytes + guardSize));
    HK(cudaMalloc(&d_blocks, nbBlocks * sizeof(ZbBlock)));
    HK(cudaMalloc(&d_meta, nbBlocks * sizeof(ZbBlockMeta)));
    HK(cudaMalloc(&d_de, sizeof(ZbDictEntropy)));
    HK(cudaMemcpyAsync(d_src, src, srcSize, cudaMemcpyHostToDevice, st));
    HK(cudaMemcpyAsync(d_lits, hlit.data(), hlit.size(), cudaMemcpyHostToDevice, st));
    HK(cudaMemcpyAsync(d_seqs, hseq.data(), hseq.size() * sizeof(u64), cudaMemcpyHostToDevice, st));
    HK(cudaMemcpyAsync(d_blocks, blocks, nbBlocks * sizeof(ZbBlock), cudaMemcpyHostToDevice, st));
    HK(cudaMemcpyAsync(d_meta, hmeta.data(), nbBlocks * sizeof(ZbBlockMeta), cudaMemcpyHostToDevice, st));
    HK(cudaMemcpyAsync(d_de, &de, sizeof(ZbDictEntropy), cudaMemcpyHostToDevice, st));
    HK(cudaMemsetAsync(d_body, guardByte, bodyBytes + guardSize, st));
    HK(zb_launch_literals(d_blocks, nbBlocks, &prm, &sd, d_de, d_lits, d_body, d_meta, st));
    HK(zb_launch_sequences(d_src, d_blocks, nbBlocks, &prm, &sd, d_de, d_seqs, d_state, d_body, d_meta, st));
    HK(cudaMemcpyAsync(meta, d_meta, nbBlocks * sizeof(ZbBlockMeta), cudaMemcpyDeviceToHost, st));
    HK(cudaMemcpyAsync(body, d_body, bodyBytes, cudaMemcpyDeviceToHost, st));
    HK(cudaMemcpyAsync(guard, d_body + bodyBytes, guardSize, cudaMemcpyDeviceToHost, st));
    HK(cudaStreamSynchronize(st));
#undef HK
out:
    cudaFree(d_src); cudaFree(d_lits); cudaFree(d_seqs); cudaFree(d_state); cudaFree(d_body);
    cudaFree(d_blocks); cudaFree(d_meta); cudaFree(d_de);
    if (st) cudaStreamDestroy(st);
    return (int)e;
}
