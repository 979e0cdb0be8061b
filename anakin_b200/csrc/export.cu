// Interior-tensor export (include/b200_saber.h has the contract): one NHWC edge tensor -- 8-bit codes, f16 or f32,
// channel-padded -- written as the dense fp32 NCHW tensor a caller of Net::get_tensor_from_edge expects. The Net
// launches it right behind the producer of an exported edge, inside its captured prediction.
//
// An NHWC -> NCHW transpose is a bandwidth kernel, so both sides are coalesced: a CTA stages kPix pixels x kCh
// channels in shared memory, reading each pixel's channel run with 16-byte loads and writing each channel's pixel run
// with 16-byte stores when h*w is a multiple of 4 (the row starts are then 16-byte aligned). A 1 x 1 tensor (a global
// pooling, the logits) is already [n][c]: it is a row-by-row conversion without the transpose.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

#include "../../include/b200_saber.h"
#include "common.cuh"
#include "ptx.cuh"
#include "vec.cuh"

namespace b200 {

namespace {

constexpr int kThreads = 256;
constexpr int kPix = 32;    // pixels per tile (the output row segment of one channel)
constexpr int kCh = 64;     // channels per tile (the input row segment of one pixel)

// The oracle's as_float, one code: s8 q * scale; u8 (q * scale) * (127 / 255), two fp32 roundings; f16 widening; f32
// the value itself. __fmul_rn keeps the compiler from contracting anything.
template <int K>
__device__ __forceinline__ float decode(uint32_t bits, float scale) {
    if constexpr (K == VK_S8) return __fmul_rn(static_cast<float>(static_cast<int8_t>(bits & 0xffu)), scale);
    else if constexpr (K == VK_U8)
        return __fmul_rn(__fmul_rn(static_cast<float>(bits & 0xffu), scale), static_cast<float>(127.0 / 255.0));
    else if constexpr (K == VK_F16) return __half2float(__ushort_as_half(static_cast<unsigned short>(bits)));
    else return __uint_as_float(bits);
}

// Lane j of a 16-byte vector of kind K, as raw bits.
template <int K>
__device__ __forceinline__ uint32_t lane_bits(const uint4& v, int j) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    if constexpr (K == VK_F32) return w[j];
    else if constexpr (K == VK_F16) return (w[j >> 1] >> (16 * (j & 1))) & 0xffffu;
    else return (w[j >> 2] >> (8 * (j & 3))) & 0xffu;
}

template <int K>
__device__ __forceinline__ uint32_t load_bits(const void* x, long long i) {
    if constexpr (K == VK_F32) return __ldg(static_cast<const uint32_t*>(x) + i);
    else if constexpr (K == VK_F16) return __ldg(static_cast<const unsigned short*>(x) + i);
    else return __ldg(static_cast<const uint8_t*>(x) + i);
}

// x: [n][hw][ld] of kind K, out: fp32 [n][c][hw]. Grid (hw tiles, channel tiles, n). VEC_IN: ld * sizeof(element) is
// a multiple of 16 and x is 16-byte aligned; VEC_OUT: hw % 4 == 0 and out is 16-byte aligned.
template <int K, bool VEC_IN, bool VEC_OUT>
__global__ void __launch_bounds__(kThreads) export_nchw_kernel(const void* __restrict__ x, float* __restrict__ out,
                                                               int c, int ld, int hw, float scale) {
    __shared__ float tile[kCh][kPix + 1];
    pdl_enter();      // the producer of x has finished
    const int n = blockIdx.z, px0 = blockIdx.x * kPix, c0 = blockIdx.y * kCh;
    const long long row0 = static_cast<long long>(n) * hw;
    if constexpr (VEC_IN) {
        constexpr int L = vec_lanes<K>, V = kCh / L;          // 16-byte vectors per pixel of the tile
        for (int i = threadIdx.x; i < kPix * V; i += kThreads) {
            const int p = i / V, v = i - p * V, ch = c0 + v * L;
            if (px0 + p >= hw || ch >= c) continue;       // (ld is a multiple of L: the vector is inside the row)
            const char* src = static_cast<const char*>(x) + ((row0 + px0 + p) * ld + ch) * (16 / L);
            const uint4 q = __ldg(reinterpret_cast<const uint4*>(src));
#pragma unroll
            for (int j = 0; j < L; ++j) tile[v * L + j][p] = decode<K>(lane_bits<K>(q, j), scale);
        }
    } else {
        for (int i = threadIdx.x; i < kPix * kCh; i += kThreads) {
            const int p = i / kCh, j = i - p * kCh;
            if (px0 + p < hw && c0 + j < c) tile[j][p] = decode<K>(load_bits<K>(x, (row0 + px0 + p) * ld + c0 + j), scale);
        }
    }
    __syncthreads();
    float* dst = out + (static_cast<long long>(n) * c + c0) * hw + px0;
    if constexpr (VEC_OUT) {
        constexpr int Q = kPix / 4;                      // float4 per channel row of the tile
        for (int i = threadIdx.x; i < kCh * Q; i += kThreads) {
            const int j = i / Q, q = i - j * Q, p = 4 * q;
            if (c0 + j >= c || px0 + p >= hw) continue;   // (hw % 4 == 0: the float4 is inside the row)
            const float4 f = make_float4(tile[j][p], tile[j][p + 1], tile[j][p + 2], tile[j][p + 3]);
            *reinterpret_cast<float4*>(dst + static_cast<long long>(j) * hw + p) = f;
        }
    } else {
        for (int i = threadIdx.x; i < kCh * kPix; i += kThreads) {
            const int j = i / kPix, p = i - j * kPix;
            if (c0 + j < c && px0 + p < hw) dst[static_cast<long long>(j) * hw + p] = tile[j][p];
        }
    }
}

// h = w = 1: x [rows][ld] -> out [rows][c], one thread per 4 outputs (a float4 store when c % 4 == 0).
template <int K, bool VEC_OUT>
__global__ void __launch_bounds__(kThreads) export_rows_kernel(const void* __restrict__ x, float* __restrict__ out,
                                                               long long rows, int c, int ld, float scale) {
    pdl_enter();
    const int groups = (c + 3) / 4;
    const long long total = rows * groups;
    for (long long i = static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x; i < total;
         i += static_cast<long long>(gridDim.x) * kThreads) {
        const long long r = i / groups;
        const int ch = static_cast<int>(i - r * groups) * 4;
        float f[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) f[j] = ch + j < c ? decode<K>(load_bits<K>(x, r * ld + ch + j), scale) : 0.f;
        float* dst = out + r * c + ch;
        if constexpr (VEC_OUT) {
            *reinterpret_cast<float4*>(dst) = make_float4(f[0], f[1], f[2], f[3]);
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (ch + j < c) dst[j] = f[j];
        }
    }
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

}  // namespace

}  // namespace b200

using namespace b200;

extern "C" {

int b200_export_run(const void* x, int32_t dtype, int32_t n, int32_t h, int32_t w, int32_t c, int32_t c_stored,
                    float scale, float* out, void* stream) {
    if (!x || !out || n < 1 || h < 1 || w < 1 || c < 1 || c_stored < c) return B200_INVALID_VALUE;
    if (dtype != B200_FLOAT && dtype != B200_HALF && dtype != B200_INT8 && dtype != B200_UINT8) return B200_INVALID_VALUE;
    const long long hw = static_cast<long long>(h) * w;
    if (hw > (1ll << 30)) return B200_INVALID_VALUE;
    if (!device_is_sm90()) return B200_WRONG_DEVICE;
    return with_vec_kind(dtype, [&](auto kind) -> int {
        constexpr int K = decltype(kind)::value;
        if (hw == 1) {
            const long long total = static_cast<long long>(n) * ((c + 3) / 4);
            const unsigned grid = static_cast<unsigned>(std::min<long long>((total + kThreads - 1) / kThreads, 65535));
            const bool vout = c % 4 == 0 && aligned16(out);
            return launch("export", Pdl::On, vout ? export_rows_kernel<K, true> : export_rows_kernel<K, false>, grid,
                          kThreads, 0, stream, dim3(1), x, out, (long long)n, c, c_stored, scale);
        }
        const dim3 grid(static_cast<unsigned>((hw + kPix - 1) / kPix), (c + kCh - 1) / kCh, n);
        const bool vin = (static_cast<long long>(c_stored) * (16 / vec_lanes<K>)) % 16 == 0 && aligned16(x);
        const bool vout = hw % 4 == 0 && aligned16(out);
        auto go = [&](auto kern) {
            return launch("export", Pdl::On, kern, grid, kThreads, 0, stream, dim3(1), x, out, c, c_stored,
                          static_cast<int>(hw), scale);
        };
        if (vin && vout) return go(export_nchw_kernel<K, true, true>);
        if (vin) return go(export_nchw_kernel<K, true, false>);
        if (vout) return go(export_nchw_kernel<K, false, true>);
        return go(export_nchw_kernel<K, false, false>);
    });
}

}  // extern "C"
