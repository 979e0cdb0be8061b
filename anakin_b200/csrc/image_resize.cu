// Resize + centre crop of 8-bit images of any size to the image input's H x W, on the GPU (include/b200_saber.h has
// the geometry and the arithmetic). The per-image sizes live in a device table the host fills per request, so the
// launch depends only on (n, c, H, W) and the op is captured once into the Net's CUDA graph.
//
// Replaces (reference): the host-side preprocessing of test/framework/net/classification_accuracy.cpp and the x86
// BILINEAR_NO_ALIGN resize, saber/funcs/impl/x86/saber_resize.cpp:103-153 (resize_bilinear_no_align_kernel), whose
// fp32 result this kernel reproduces bit for bit before rounding to 8 bits.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/b200_saber.h"
#include "common.cuh"
#include "ptx.cuh"

namespace b200 {

namespace {

constexpr int kResizeThreads = 256;
constexpr int kPixelsPerThread = 4;         // a run of 4 output pixels of one row: 4*C bytes, C 32-bit words
constexpr long long kMaxResized = 1ll << 23;

// One axis of the source coordinate: f = max(scale * ((float)r + 0.5f) - 0.5f, 0), taps i0, i1 and the fraction
// f - i0; every fp32 step rounded on its own, as the reference computes it without contraction.
struct Axis {
    int i0, i1;
    float f;
};
__device__ __forceinline__ Axis resize_axis(float scale, int r, int size) {
    float f = __fsub_rn(__fmul_rn(scale, __fadd_rn(static_cast<float>(r), 0.5f)), 0.5f);
    f = f < 0.f ? 0.f : f;
    Axis a;
    a.i0 = static_cast<int>(f);
    a.i1 = a.i0 + (a.i0 < size - 1 ? 1 : 0);
    a.f = __fsub_rn(f, static_cast<float>(a.i0));
    return a;
}

__device__ __forceinline__ uint32_t cvt_u8_sat(float v) {
    uint32_t c;
    asm("cvt.rni.sat.u8.f32 %0, %1;" : "=r"(c) : "f"(v));
    return c & 0xffu;
}

// Thread = kPixelsPerThread consecutive output pixels of one row of one image. The row's source taps and weights are
// computed once; the 4 taps x C channels of each pixel are read through the read-only path. VEC (out_w % 4 == 0):
// the run is C aligned 32-bit words, stored as one 4-, 8-, 12- or 16-byte write; otherwise byte stores.
template <int C, bool VEC>
__global__ void __launch_bounds__(kResizeThreads) image_resize_kernel(const uint8_t* __restrict__ src,
                                                                      const b200_image_resize_entry_t* __restrict__ table,
                                                                      uint8_t* __restrict__ out, int out_h, int out_w,
                                                                      int runs, long long total) {
    pdl_launch_dependents();
    pdl_wait_prior_grid();      // the previous request's readers of `out` are done
    const long long t = blockIdx.x * 1ll * blockDim.x + threadIdx.x;
    if (t >= total) return;
    const int run = static_cast<int>(t % runs);
    const long long row = t / runs;
    const int y = static_cast<int>(row % out_h);
    const int img = static_cast<int>(row / out_h);
    const long long offset = __ldg(&table[img].offset);
    const int h = __ldg(&table[img].h), w = __ldg(&table[img].w);
    const int rh = __ldg(&table[img].rh), rw = __ldg(&table[img].rw);
    const int top = __ldg(&table[img].top), left = __ldg(&table[img].left);

    const Axis ay = resize_axis(__fdiv_rn(static_cast<float>(h), static_cast<float>(rh)), y + top, h);
    const double ry = __dsub_rn(1.0, static_cast<double>(ay.f));
    const uint8_t* r0 = src + offset + static_cast<long long>(ay.i0) * w * C;
    const uint8_t* r1 = src + offset + static_cast<long long>(ay.i1) * w * C;
    const float sx = __fdiv_rn(static_cast<float>(w), static_cast<float>(rw));
    const int x_begin = run * kPixelsPerThread;
    uint8_t* o = out + ((static_cast<long long>(img) * out_h + y) * out_w + x_begin) * C;

    uint32_t words[C];
#pragma unroll
    for (int i = 0; i < C; ++i) words[i] = 0;
#pragma unroll
    for (int p = 0; p < kPixelsPerThread; ++p) {
        if (!VEC && x_begin + p >= out_w) break;
        const Axis ax = resize_axis(sx, x_begin + p + left, w);
        const double rx = __dsub_rn(1.0, static_cast<double>(ax.f));
        const float w00 = __double2float_rn(__dmul_rn(ry, rx));
        const float w01 = __double2float_rn(__dmul_rn(static_cast<double>(ax.f), ry));
        const float w10 = __double2float_rn(__dmul_rn(static_cast<double>(ay.f), rx));
        const float w11 = __double2float_rn(__dmul_rn(static_cast<double>(ax.f), static_cast<double>(ay.f)));
#pragma unroll
        for (int ch = 0; ch < C; ++ch) {
            const float p00 = __ldg(r0 + ax.i0 * C + ch), p01 = __ldg(r0 + ax.i1 * C + ch);
            const float p10 = __ldg(r1 + ax.i0 * C + ch), p11 = __ldg(r1 + ax.i1 * C + ch);
            float v = __fadd_rn(__fmul_rn(w00, p00), __fmul_rn(w01, p01));
            v = __fadd_rn(v, __fmul_rn(w10, p10));
            v = __fadd_rn(v, __fmul_rn(w11, p11));
            const uint32_t b = cvt_u8_sat(v);
            if constexpr (VEC) {
                const int byte = p * C + ch;
                words[byte >> 2] |= b << (8 * (byte & 3));
            } else {
                o[p * C + ch] = static_cast<uint8_t>(b);
            }
        }
    }
    if constexpr (VEC) {
        if constexpr (C == 4) *reinterpret_cast<uint4*>(o) = make_uint4(words[0], words[1], words[2], words[3]);
        else if constexpr (C == 2) *reinterpret_cast<uint2*>(o) = make_uint2(words[0], words[1]);
        else if constexpr (C == 3) {
            uint32_t* o32 = reinterpret_cast<uint32_t*>(o);
            o32[0] = words[0]; o32[1] = words[1]; o32[2] = words[2];
        } else *reinterpret_cast<uint32_t*>(o) = words[0];
    }
}

template <int C>
int launch_resize(const b200_image_resize_desc_t* d, const uint8_t* src, const void* table, uint8_t* out,
                  cudaStream_t stream) {
    const int runs = (d->out_w + kPixelsPerThread - 1) / kPixelsPerThread;
    const long long total = 1ll * d->n * d->out_h * runs;
    const unsigned grid = static_cast<unsigned>((total + kResizeThreads - 1) / kResizeThreads);
    const auto* tab = static_cast<const b200_image_resize_entry_t*>(table);
    cudaError_t e;
    if (d->out_w % kPixelsPerThread == 0)
        e = launch_kernel(image_resize_kernel<C, true>, grid, kResizeThreads, 0, stream, dim3(1), src, tab, out,
                          d->out_h, d->out_w, runs, total);
    else
        e = launch_kernel(image_resize_kernel<C, false>, grid, kResizeThreads, 0, stream, dim3(1), src, tab, out,
                          d->out_h, d->out_w, runs, total);
    count_launch();
    if (e != cudaSuccess) {
        fprintf(stderr, "[b200_saber] image_resize launch failed: %s\n", cudaGetErrorString(e));
        return B200_UNKNOWN_ERROR;
    }
    return B200_SUCCESS;
}

}  // namespace
}  // namespace b200

extern "C" {

int b200_image_resize_geometry(int32_t h, int32_t w, int32_t resize_short, int32_t out_h, int32_t out_w, int32_t* rh,
                               int32_t* rw, int32_t* top, int32_t* left) {
    using b200::kMaxResized;
    if (!rh || !rw || !top || !left) return B200_INVALID_VALUE;
    if (h < 1 || w < 1 || out_h < 1 || out_w < 1 || h > kMaxResized || w > kMaxResized || resize_short < 0)
        return B200_INVALID_VALUE;
    long long sh, sw;
    if (resize_short == 0) {
        sh = out_h;
        sw = out_w;
    } else {
        if (resize_short < (out_h > out_w ? out_h : out_w)) return B200_INVALID_VALUE;
        const long long s = resize_short;
        if (h <= w) { sh = s; sw = s * w / h; }
        else { sw = s; sh = s * h / w; }
    }
    if (sh > kMaxResized || sw > kMaxResized) return B200_INVALID_VALUE;
    *rh = static_cast<int32_t>(sh);
    *rw = static_cast<int32_t>(sw);
    *top = static_cast<int32_t>((sh - out_h) / 2);
    *left = static_cast<int32_t>((sw - out_w) / 2);
    return B200_SUCCESS;
}

int b200_image_resize_run(const b200_image_resize_desc_t* d, const uint8_t* src, const void* table_dev, uint8_t* out,
                          void* stream) {
    if (!d || !src || !table_dev || !out) return B200_INVALID_VALUE;
    if (d->n < 1 || d->c < 1 || d->c > 4 || d->out_h < 1 || d->out_w < 1) return B200_INVALID_VALUE;
    if (!b200::device_is_sm90()) return B200_WRONG_DEVICE;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    switch (d->c) {
        case 1: return b200::launch_resize<1>(d, src, table_dev, out, s);
        case 2: return b200::launch_resize<2>(d, src, table_dev, out, s);
        case 3: return b200::launch_resize<3>(d, src, table_dev, out, s);
        default: return b200::launch_resize<4>(d, src, table_dev, out, s);
    }
}

}  // extern "C"
