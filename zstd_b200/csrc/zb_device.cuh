/* zb_device.cuh — small device helpers shared by the kernels. */
#ifndef ZB_DEVICE_CUH
#define ZB_DEVICE_CUH
#include <cuda_runtime.h>
#include "zb_common.h"

#define ZB_FULL 0xFFFFFFFFu

/* Unaligned little-endian loads built from aligned 32-bit words.  Only words that contain a
 * requested byte are dereferenced, so a load never leaves the 4-byte word of the last byte. */
__device__ __forceinline__ u32 zb_ld32u(const u8* p)
{
    const u32* q = (const u32*)((uintptr_t)p & ~(uintptr_t)3);
    u32 const sh = ((u32)(uintptr_t)p & 3u) * 8u;
    u32 const a = __ldg(q);
    u32 const b = __ldg(sh ? q + 1 : q);                  /* select the address, not the load: no branch */
    return __funnelshift_r(a, b, sh);
}
__device__ __forceinline__ u64 zb_ld64u(const u8* p)
{
    const u32* q = (const u32*)((uintptr_t)p & ~(uintptr_t)3);
    u32 const sh = ((u32)(uintptr_t)p & 3u) * 8u;
    u32 const a = __ldg(q);
    u32 const b = __ldg(q + 1);
    u32 const c = __ldg(sh ? q + 2 : q + 1);
    u32 const lo = __funnelshift_r(a, b, sh);
    u32 const hi = __funnelshift_r(b, c, sh);
    return ((u64)hi << 32) | lo;
}

/* Branch-free variants: always touch 2 (resp. 3) words, so several of them can be in flight at
 * once (the predicated forms above make ptxas fence each load in its own reconvergence region).
 * Caller guarantees p + 8 (resp. p + 12 rounded down to a word) stays inside the input. */
__device__ __forceinline__ u32 zb_ld32w2(const u8* p)
{
    const u32* q = (const u32*)((uintptr_t)p & ~(uintptr_t)3);
    u32 const sh = ((u32)(uintptr_t)p & 3u) * 8u;
    return __funnelshift_r(__ldg(q), __ldg(q + 1), sh);
}
__device__ __forceinline__ u64 zb_ld64w3(const u8* p)
{
    const u32* q = (const u32*)((uintptr_t)p & ~(uintptr_t)3);
    u32 const sh = ((u32)(uintptr_t)p & 3u) * 8u;
    u32 const a = __ldg(q), b = __ldg(q + 1), c = __ldg(q + 2);
    return ((u64)__funnelshift_r(b, c, sh) << 32) | __funnelshift_r(a, b, sh);
}
/* ---- two-segment addressing (dictionary content in front of a frame, zstd_compress_internal.h:797
 * ZSTD_count_2segments is the reference's counterpart): rel positions < split live in `lo`, the rest
 * in `hi`; both pointers are pre-biased so that ptr + rel is the byte's address. ---- */
struct ZbSeg { const u8* lo; const u8* hi; u32 split; };

template <bool DICT> __device__ __forceinline__ const u8* zb_seg_ptr(const ZbSeg& s, u32 rel)
{
    if (DICT) return (rel < s.split ? s.lo : s.hi) + rel;
    return s.hi + rel;
}
template <bool DICT> __device__ __forceinline__ u8 zb_seg_byte(const ZbSeg& s, u32 rel) { return *zb_seg_ptr<DICT>(s, rel); }

/* 8 bytes at rel (3-word form: the caller guarantees rel + 12 stays inside the input) */
template <bool DICT> __device__ __forceinline__ u64 zb_seg_ld64(const ZbSeg& s, u32 rel)
{
    if (DICT && rel < s.split && rel + 12u > s.split) {          /* straddles the dictionary / frame boundary */
        u64 v = 0;
#pragma unroll
        for (u32 i = 0; i < 8u; i++) v |= (u64)zb_seg_byte<true>(s, rel + i) << (8u * i);
        return v;
    }
    return zb_ld64w3(zb_seg_ptr<DICT>(s, rel));
}
/* exact 8-byte load that never touches a byte past rel+7 (match extension up to the block end) */
template <bool DICT> __device__ __forceinline__ u64 zb_seg_ld64x(const ZbSeg& s, u32 rel)
{
    if (DICT && rel < s.split && rel + 12u > s.split) {
        u64 v = 0;
#pragma unroll
        for (u32 i = 0; i < 8u; i++) v |= (u64)zb_seg_byte<true>(s, rel + i) << (8u * i);
        return v;
    }
    return zb_ld64u(zb_seg_ptr<DICT>(s, rel));
}
template <bool DICT> __device__ __forceinline__ u32 zb_seg_ld32(const ZbSeg& s, u32 rel) { return (u32)zb_seg_ld64<DICT>(s, rel); }
/* The 4 bytes at rel position x (`cur`) and the 4 bytes in front of it (`pre`, byte x-1 in the top byte;
 * bytes in front of position 0 are undefined and must be masked by the caller's limits). */
template <bool DICT> __device__ __forceinline__ void zb_seg_pre_cur(const ZbSeg& sg, u32 x, u32* pre, u32* cur)
{
    u32 const s = x >= 4u ? 0u : 4u - x;
    u64 const w = zb_seg_ld64<DICT>(sg, x + s - 4u);
    *pre = (u32)(w << (8u * s));
    *cur = (u32)(w >> (32u - 8u * s));
}

__host__ __device__ __forceinline__ u32 zb_mulhi(u32 a, u32 b)
{
#ifdef __CUDA_ARCH__
    return __umulhi(a, b);
#else
    return (u32)(((u64)a * b) >> 32);
#endif
}

/* The 32-bit hash of the MLS bytes at a position (lib/compress/zstd_compress_internal.h:815-861 with hBits = 32) from the
 * position's 8 bytes v = hi:lo.  For MLS 5..8 the reference keeps the top 32 bits of the 64-bit product (v << (64 - 8 MLS))
 * * prime: the shift moves into the constant (C = prime << (64 - 8 MLS), the bytes past MLS then only reach bits >= 64),
 * and of the 32 x 32 partial products only lo * C.lo (its high half), lo * C.hi and hi * C.lo reach the kept bits.
 * Three multiply-adds instead of a 64-bit product; tests/test_gpu_walk_paths.py compares it with the 64-bit form. */
template <int MLS>
__host__ __device__ __forceinline__ u32 zb_hash32(u32 lo, u32 hi)
{
    static_assert(MLS >= 4 && MLS <= 8, "minimum match length 4..8");
    if (MLS == 4) return lo * 2654435761u;
    constexpr u64 C = MLS == 5 ? 889523592379ull << 24 : MLS == 6 ? 227718039650203ull << 16
                    : MLS == 7 ? 58295818150454627ull << 8 : 0xCF1BBCDCB7A56463ull;
    return zb_mulhi(lo, (u32)C) + lo * (u32)(C >> 32) + hi * (u32)C;
}

__device__ __forceinline__ u32 zb_hb32(u32 v) { return 31u - (u32)__clz((int)v); }

/* XXH64 rounds (lib/common/xxhash.h; XXH64 spec): the frame checksum (zb_stitch.cu) and the LDM split hash (zb_ldm.cu) */
__device__ __forceinline__ u64 zbx_rotl(u64 x, int r) { return (x << r) | (x >> (64 - r)); }
#define ZBX_P1 0x9E3779B185EBCA87ull
#define ZBX_P2 0xC2B2AE3D27D4EB4Full
#define ZBX_P3 0x165667B19E3779F9ull
#define ZBX_P4 0x85EBCA77C2B2AE63ull
#define ZBX_P5 0x27D4EB2F165667C5ull
__device__ __forceinline__ u64 zbx_round(u64 acc, u64 in) { return zbx_rotl(acc + in * ZBX_P2, 31) * ZBX_P1; }
__device__ __forceinline__ u64 zbx_merge(u64 h, u64 v) { return (h ^ zbx_round(0, v)) * ZBX_P1 + ZBX_P4; }

#endif
