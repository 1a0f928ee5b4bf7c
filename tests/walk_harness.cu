/* walk_harness.cu — TEST INFRASTRUCTURE ONLY.  Runs the product's candidate walk, zb_launch_walk (K1a), on chosen frames without
 * the parse behind it, and hands back the whole dist and far arrays and the dictionary table images.  Linked against the
 * product's own zb_match.o (zstd_b200/csrc/Makefile, target `harness`), so the kernel under test is the one the library
 * ships.  Used by tests/test_gpu_walk_paths.py. */
#include <string.h>
#include <vector>
#include "../zstd_b200/csrc/zb_common.h"
#include "../zstd_b200/csrc/zb_kernels.h"

#define ZBH_GUARD 64u            /* u32 words of guard on both sides of every image */
#define ZBH_PAD 64u              /* zero bytes around the frames and around every dictionary tail */
#define ZBH_N_MAX 57856u         /* 226 KiB of dynamic shared memory: what the walk launch asks for */

/* One launch over nbFrames frames.  Frame f is src[frameOff[f], + frameSize[f]) with blocks of 1 << blockLog[f] bytes (one
 * block when the frame is smaller) and, when tailLen[f] > 0, the dictionary tail tails[tailOff[f], + tailLen[f]) in front of
 * it.  The chunk descriptors are the planner's (zb_plan in zb_api.cu): chunks of ZB_CHUNK_BLOCKS blocks, a first chunk's
 * history is the tail, a later chunk's the min(pos, ZB_PRIME_BYTES) frame bytes in front of it; block k of the launch owns
 * row k, its chunk's firstBlock is slotFirstBlock + its index.  Row strides: zb_strides of the launch's largest block.
 *   prm:   mls, N, insStep, imageOff, imageMode, mlsShort, slotFirstBlock
 *          imageMode 1: zb_launch_dict_images first builds every tail's image (imageOff = 0: strategy 1 with mls and N;
 *          imageOff > 0: strategy 2, a short table of imageOff buckets with mlsShort, then the long table of N buckets, whose
 *          walk must hash 8 bytes), and the walk of each first chunk starts from its image
 *   sent:  two sentinel bytes.  The launch runs twice; before run r the dist, far and image buffers are filled with sent[r]
 *   dist, far: 2 x rows x stride u16 / u32 (rows = blocks of the launch, stride = zb_strides(largest block).dist), run r at r x
 *          rows x stride.  image: 2 x nbFrames x (ZBH_GUARD + imageOff + N + ZBH_GUARD) u32 (imageMode only), frame f's at
 *          f x that, run r at r x nbFrames x that
 *   shape: rows, stride (written first, also when the capacities are too small)
 * Returns 0, a CUDA error code, or a negative value for bad arguments.  Every allocation is freed before it returns. */
extern "C" __attribute__((visibility("default")))
int zbh_walk(const u8* src, u64 srcLen, const u64* frameOff, const u32* frameSize, const u32* blockLog, u32 nbFrames,
             const u8* tails, u64 tailsLen, const u64* tailOff, const u32* tailLen, const u32* prm, const u8* sent,
             u16* dist, u32* far, u64 distCap, u32* image, u64 imageCap, u64* shape)
{
    u32 const mls = prm[0], N = prm[1], insStep = prm[2], imageOff = prm[3], imageMode = prm[4], mlsShort = prm[5], slotFirstBlock = prm[6];
    if (nbFrames == 0 || mls < 4 || mls > 8 || N == 0 || N > ZBH_N_MAX || insStep == 0 || imageMode > 1) return -1;
    if (imageMode && imageOff && (mls != 8 || mlsShort < 4 || mlsShort > 8 || imageOff > ZBH_N_MAX)) return -1;
    std::vector<ZbChunk> chunks, imageChunks;
    std::vector<u64> tailDev(nbFrames);
    u32 rows = 0, maxBlock = 0; u64 tailBytes = ZBH_PAD;
    for (u32 f = 0; f < nbFrames; f++) {
        u64 const fsz = frameSize[f];
        if (blockLog[f] < 10 || blockLog[f] > 17 || frameOff[f] > srcLen || fsz > srcLen - frameOff[f]) return -1;   /* blocks are whole batches */
        if (tailLen[f] > ZB_PRIME_BYTES || (tailLen[f] && (tailOff[f] > tailsLen || tailLen[f] > tailsLen - tailOff[f]))) return -1;
        u64 const blockMax = 1ull << blockLog[f], chunkBytes = ZB_CHUNK_BLOCKS * blockMax;
        tailDev[f] = tailBytes; tailBytes += tailLen[f] + ZBH_PAD;
        u64 pos = 0;
        do {
            u64 const bsz = (fsz - pos) < blockMax ? (fsz - pos) : blockMax;
            if (pos % chunkBytes == 0) {
                ZbChunk ch; memset(&ch, 0, sizeof(ch));
                ch.srcOff = ZBH_PAD + frameOff[f] + pos; ch.size = (u32)((fsz - pos) < chunkBytes ? (fsz - pos) : chunkBytes);
                ch.histLen = pos == 0 ? tailLen[f] : (u32)(pos < ZB_PRIME_BYTES ? pos : ZB_PRIME_BYTES);
                ch.dictLen = pos == 0 ? tailLen[f] : 0u;
                ch.firstBlock = slotFirstBlock + rows; ch.blockLog = blockLog[f]; ch.dictSlot = f;
                chunks.push_back(ch);
            }
            if (bsz > maxBlock) maxBlock = (u32)bsz;
            rows++;
            pos += bsz;
        } while (pos < fsz);
        if (imageMode && tailLen[f]) {
            ZbChunk ch; memset(&ch, 0, sizeof(ch));
            ch.histLen = tailLen[f]; ch.dictLen = tailLen[f]; ch.blockLog = 17; ch.dictSlot = f;
            imageChunks.push_back(ch);
        }
    }
    ZbStrides const sd = zb_strides(maxBlock);
    shape[0] = rows; shape[1] = sd.dist;
    u64 const cells = (u64)rows * sd.dist;
    u64 const imgWords = ZBH_GUARD + (u64)imageOff + N + ZBH_GUARD;
    if (distCap < 2 * cells || (imageMode && imageCap < 2 * nbFrames * imgWords)) return -2;

    u8 *d_src = nullptr, *d_tails = nullptr; u16* d_dist = nullptr; u32 *d_far = nullptr, *d_image = nullptr;
    ZbChunk *d_chunks = nullptr, *d_imageChunks = nullptr; ZbDictSlot* d_dicts = nullptr;
    std::vector<ZbDictSlot> slots(nbFrames);
    cudaStream_t st = nullptr;
    cudaError_t e;
#define HK(x) do { if ((e = (x)) != cudaSuccess) goto out; } while (0)
    HK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    HK(cudaMalloc(&d_src, srcLen + 2 * ZBH_PAD));
    HK(cudaMalloc(&d_tails, tailBytes));
    HK(cudaMalloc(&d_dist, cells * sizeof(u16)));
    HK(cudaMalloc(&d_far, cells * sizeof(u32)));
    HK(cudaMalloc(&d_chunks, chunks.size() * sizeof(ZbChunk)));
    HK(cudaMalloc(&d_dicts, nbFrames * sizeof(ZbDictSlot)));
    if (imageMode) HK(cudaMalloc(&d_image, nbFrames * imgWords * sizeof(u32)));
    if (!imageChunks.empty()) HK(cudaMalloc(&d_imageChunks, imageChunks.size() * sizeof(ZbChunk)));
    for (u32 f = 0; f < nbFrames; f++) {
        memset(&slots[f], 0, sizeof(ZbDictSlot));
        slots[f].end = d_tails + tailDev[f] + tailLen[f];
        slots[f].image = (imageMode && tailLen[f]) ? d_image + f * imgWords + ZBH_GUARD : nullptr;
    }
    HK(cudaMemsetAsync(d_src, 0, srcLen + 2 * ZBH_PAD, st));
    HK(cudaMemcpyAsync(d_src + ZBH_PAD, src, srcLen, cudaMemcpyHostToDevice, st));
    HK(cudaMemsetAsync(d_tails, 0, tailBytes, st));
    for (u32 f = 0; f < nbFrames; f++)
        if (tailLen[f]) HK(cudaMemcpyAsync(d_tails + tailDev[f], tails + tailOff[f], tailLen[f], cudaMemcpyHostToDevice, st));
    HK(cudaMemcpyAsync(d_chunks, chunks.data(), chunks.size() * sizeof(ZbChunk), cudaMemcpyHostToDevice, st));
    HK(cudaMemcpyAsync(d_dicts, slots.data(), nbFrames * sizeof(ZbDictSlot), cudaMemcpyHostToDevice, st));
    if (!imageChunks.empty()) HK(cudaMemcpyAsync(d_imageChunks, imageChunks.data(), imageChunks.size() * sizeof(ZbChunk), cudaMemcpyHostToDevice, st));
    for (int r = 0; r < 2; r++) {
        HK(cudaMemsetAsync(d_dist, sent[r], cells * sizeof(u16), st));
        HK(cudaMemsetAsync(d_far, sent[r], cells * sizeof(u32), st));
        if (imageMode) {
            HK(cudaMemsetAsync(d_image, sent[r], nbFrames * imgWords * sizeof(u32), st));
            ZbParams ip; memset(&ip, 0, sizeof(ip));
            ip.strategy = imageOff ? 2u : 1u; ip.mls = imageOff ? mlsShort : mls; ip.tableN = imageOff ? imageOff : N; ip.tableNLong = N;
            ip.insStep = insStep;
            HK(zb_launch_dict_images(d_dicts, d_imageChunks, (u32)imageChunks.size(), &ip, st));
        }
        HK(zb_launch_walk(d_src, d_dicts, d_chunks, (u32)chunks.size(), mls, N, insStep, sd, slotFirstBlock, d_dist, d_far, imageOff, false, st));
        HK(cudaMemcpyAsync(dist + r * cells, d_dist, cells * sizeof(u16), cudaMemcpyDeviceToHost, st));
        HK(cudaMemcpyAsync(far + r * cells, d_far, cells * sizeof(u32), cudaMemcpyDeviceToHost, st));
        if (imageMode) HK(cudaMemcpyAsync(image + r * nbFrames * imgWords, d_image, nbFrames * imgWords * sizeof(u32), cudaMemcpyDeviceToHost, st));
    }
    HK(cudaStreamSynchronize(st));
    HK(cudaGetLastError());
#undef HK
out:
    cudaFree(d_src); cudaFree(d_tails); cudaFree(d_dist); cudaFree(d_far); cudaFree(d_image);
    cudaFree(d_chunks); cudaFree(d_imageChunks); cudaFree(d_dicts);
    if (st) cudaStreamDestroy(st);
    return (int)e;
}
