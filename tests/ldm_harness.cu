/* ldm_harness.cu — TEST INFRASTRUCTURE ONLY.  Runs the product's long-distance match finder, zb_launch_ldm (L1 split points
 * and thinning, scan and compaction, L2 bucket sort, L3 selection), on a chosen prefix and frame of any size, without the
 * parse or the overlay behind it.  Linked against the product's own zb_ldm.o (zstd_b200/csrc/Makefile, target `harness`),
 * so the kernels under test are the ones the library ships.  Used by tests/test_gpu_ldm_paths.py. */
#include <string.h>
#include "../zstd_b200/csrc/zb_common.h"
#include "../zstd_b200/csrc/zb_kernels.h"

/* One launch over the frame src[0, n) behind the prefix bytes prefix[0, P) (P = 0: none).
 *   prm:       hashLog, minMatch, bucketSizeLog, hashRateLog (resolved), windowLog; stopMask: the split test's mask
 *   match:     matchCap >= zb_ldm_survivor_cap(P + n, minMatch) packed matches (zb_pack_ldm); entries the launch does not
 *              write keep the value 0xFF..FF they have before it
 *   first/cnt: per block of the frame (ceil(n / ZB_BLOCK_MAX) blocks): its matches are match[first[k] .. + cnt[k]); first[k]
 *              is meaningful where cnt[k] > 0
 * Returns 0, a CUDA error code, or a negative value for bad arguments.  Every allocation is freed before it returns. */
extern "C" __attribute__((visibility("default")))
int zbh_ldm(const u8* prefix, u64 P, const u8* src, u64 n, const u32* prm5, u64 stopMask, u64* match, u64 matchCap,
            u64* first, u32* cnt)
{
    ZbLdmParams prm;
    memset(&prm, 0, sizeof(prm));
    prm.hashLog = prm5[0]; prm.minMatch = prm5[1]; prm.bucketSizeLog = prm5[2]; prm.hashRateLog = prm5[3]; prm.windowLog = prm5[4];
    prm.stopMask = stopMask;
    u32 const nbBlocks = (u32)((n + ZB_BLOCK_MAX - 1) / ZB_BLOCK_MAX);
    u64 const cap = zb_ldm_survivor_cap(P + n, prm.minMatch);
    if (n == 0 || prm.minMatch < 4 || prm.bucketSizeLog > prm.hashLog || matchCap < cap) return -1;
    size_t const scratch = zb_ldm_scratch_bytes(P, n, &prm);
    u8 *d_prefix = nullptr, *d_src = nullptr, *d_scratch = nullptr; u64 *d_match = nullptr, *d_first = nullptr; u32* d_cnt = nullptr;
    cudaStream_t st = nullptr;
    cudaError_t e;
#define HK(x) do { if ((e = (x)) != cudaSuccess) goto out; } while (0)
    HK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    HK(cudaMalloc(&d_prefix, P ? P : 1));
    HK(cudaMalloc(&d_src, n));
    HK(cudaMalloc(&d_scratch, scratch ? scratch : 1));
    HK(cudaMalloc(&d_match, cap * sizeof(u64)));
    HK(cudaMalloc(&d_first, nbBlocks * sizeof(u64)));
    HK(cudaMalloc(&d_cnt, nbBlocks * sizeof(u32)));
    if (P) HK(cudaMemcpyAsync(d_prefix, prefix, P, cudaMemcpyHostToDevice, st));
    HK(cudaMemcpyAsync(d_src, src, n, cudaMemcpyHostToDevice, st));
    HK(cudaMemsetAsync(d_match, 0xFF, cap * sizeof(u64), st));
    HK(cudaMemsetAsync(d_first, 0xFF, nbBlocks * sizeof(u64), st));
    HK(zb_launch_ldm(d_prefix, P, d_src, n, &prm, d_scratch, nbBlocks, 0, d_match, d_first, d_cnt, st));
    HK(cudaMemcpyAsync(match, d_match, cap * sizeof(u64), cudaMemcpyDeviceToHost, st));
    HK(cudaMemcpyAsync(first, d_first, nbBlocks * sizeof(u64), cudaMemcpyDeviceToHost, st));
    HK(cudaMemcpyAsync(cnt, d_cnt, nbBlocks * sizeof(u32), cudaMemcpyDeviceToHost, st));
    HK(cudaStreamSynchronize(st));
    HK(cudaGetLastError());
#undef HK
out:
    cudaFree(d_prefix); cudaFree(d_src); cudaFree(d_scratch); cudaFree(d_match); cudaFree(d_first); cudaFree(d_cnt);
    if (st) cudaStreamDestroy(st);
    return (int)e;
}
