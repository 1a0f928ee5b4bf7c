/* zb_bitpack.cuh — parallel bit packing into a little-endian bit-stream.
 *
 * Each thread knows (from a prefix sum over bit counts) the absolute bit position at which its
 * run of fields starts, accumulates fields in a 64-bit register and emits whole 32-bit words.
 * Words that may be shared with a neighbouring thread (the first and the last one it touches) are
 * merged with atomicOr into pre-zeroed memory; interior words are plain stores.
 * Bit order is that of BIT_addBits (lib/common/bitstream.h:179-188): a field
 * occupies [pos, pos+nbBits), least significant bit first.
 */
#ifndef ZB_BITPACK_CUH
#define ZB_BITPACK_CUH
#include "zb_device.cuh"

struct ZbdParW { u32* words; u64 acc; u32 nacc; u32 widx; u32 first; };

__device__ __forceinline__ void zbd_pw_init(ZbdParW* w, u32* words, u64 bitPos)
{
    w->words = words; w->acc = 0; w->nacc = (u32)(bitPos & 31u); w->widx = (u32)(bitPos >> 5); w->first = 1;
}
/* value must already be < 2^nbBits ; nbBits <= 31 */
__device__ __forceinline__ void zbd_pw_add(ZbdParW* w, u32 value, u32 nbBits)
{
    w->acc |= (u64)value << w->nacc;
    w->nacc += nbBits;
    if (w->nacc >= 32u) {
        u32 const lo = (u32)w->acc;
        if (w->first) { if (lo) atomicOr(&w->words[w->widx], lo); w->first = 0; }
        else w->words[w->widx] = lo;
        w->widx++;
        w->acc >>= 32;
        w->nacc -= 32u;
    }
}
__device__ __forceinline__ void zbd_pw_finish(ZbdParW* w)
{
    u32 const lo = (u32)w->acc;
    if (w->nacc && lo) atomicOr(&w->words[w->widx], lo);
}

#endif
