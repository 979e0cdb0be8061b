// The 16-byte vector codec of the NHWC kernels: a uint4 holds 4 x f32, 8 x f16 or 16 x s8 / u8 (VecKind), and 8-bit
// codes are written by one rounding rule, cvt_q8.
#pragma once
#include <cuda_fp16.h>
#include <stdint.h>

#include "common.cuh"

namespace b200 {

template <int K> constexpr int vec_lanes = K == VK_F32 ? 4 : (K == VK_F16 ? 8 : 16);

// cvt.rni.sat: round to nearest even, saturate to the 8-bit range; returns the code's byte
__device__ __forceinline__ uint32_t cvt_q8(float f, bool to_unsigned) {
    uint32_t c;
    if (to_unsigned) asm("cvt.rni.sat.u8.f32 %0, %1;" : "=r"(c) : "f"(f));
    else asm("cvt.rni.sat.s8.f32 %0, %1;" : "=r"(c) : "f"(f));
    return c & 0xffu;
}

// E4M3 (OCP e4m3fn: no infinities, max finite 448, smallest subnormal 2^-9). Encoding rounds to nearest even and
// saturates to +-448; decoding is exact. `lo` lands in the low byte of the pair, `hi` in the high byte.
__device__ __forceinline__ uint32_t enc_e4m3x2(float lo, float hi) {
    uint16_t c;
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(c) : "f"(hi), "f"(lo));
    return c;
}
// the two codes in the low 16 bits of `pair` -> (low byte's value, high byte's value)
__device__ __forceinline__ float2 dec_e4m3x2(uint32_t pair) {
    uint32_t h;
    asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(h) : "h"(static_cast<uint16_t>(pair)));
    return __half22float2(*reinterpret_cast<const __half2*>(&h));
}
// four codes of a word -> four values, byte order
__device__ __forceinline__ void dec_e4m3x4(uint32_t w, float* f) {
    const float2 a = dec_e4m3x2(w), b = dec_e4m3x2(w >> 16);
    f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y;
}
__device__ __forceinline__ uint32_t enc_e4m3x4(float a, float b, float c, float d) {
    return enc_e4m3x2(a, b) | (enc_e4m3x2(c, d) << 16);
}

template <int K>
__device__ __forceinline__ void unpack_vec(const uint4& v, float (&f)[vec_lanes<K>]) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    if constexpr (K == VK_F32) {
#pragma unroll
        for (int i = 0; i < 4; ++i) f[i] = __uint_as_float(w[i]);
    } else if constexpr (K == VK_F16) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float2 q = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
            f[2 * i] = q.x;
            f[2 * i + 1] = q.y;
        }
    } else {
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            const uint32_t b = (w[i >> 2] >> (8 * (i & 3))) & 0xffu;
            f[i] = K == VK_U8 ? static_cast<float>(b) : static_cast<float>(static_cast<int8_t>(b));
        }
    }
}

// Packs lane values f(0), f(1), ... in lane order (computing each value next to its conversion keeps the depthwise
// epilogues' register use where it was). f16 rounds to nearest even; the 8-bit kinds go through cvt_q8, to_unsigned
// choosing the code (the depthwise kernels write s8 or u8 from one instance).
template <int K, typename F>
__device__ __forceinline__ uint4 pack_vec(F f, bool to_unsigned = K == VK_U8) {
    uint32_t w[4];
    if constexpr (K == VK_F32) {
#pragma unroll
        for (int i = 0; i < 4; ++i) w[i] = __float_as_uint(f(i));
    } else if constexpr (K == VK_F16) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float lo = f(2 * i), hi = f(2 * i + 1);
            const __half2 h = __floats2half2_rn(lo, hi);
            w[i] = *reinterpret_cast<const uint32_t*>(&h);
        }
    } else {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            w[i] = 0;
#pragma unroll
            for (int j = 0; j < 4; ++j) w[i] |= cvt_q8(f(4 * i + j), to_unsigned) << (8 * j);
        }
    }
    return make_uint4(w[0], w[1], w[2], w[3]);
}
template <int K>
__device__ __forceinline__ uint4 pack_vec(const float (&f)[vec_lanes<K>], bool to_unsigned = K == VK_U8) {
    return pack_vec<K>([&](int i) { return f[i]; }, to_unsigned);
}

}  // namespace b200
