// Bandwidth-bound Saber ops on NHWC tensors: pooling, softmax, eltwise, activation,
// scale and the layout / precision transforms at graph boundaries.  All are 128-bit
// vectorised, grid sized to the data, judged against the HBM roofline only.
//
// Replaces (reference, all under saber/funcs/impl/cuda/base/cuda_c/):
//   saber_pooling.cu:20-229 + vender_pooling.cpp (cuDNN) -> pool_kernel
//   saber_softmax.cu:10-430  (one *thread* per row)      -> softmax_rows_kernel (one warp per row)
//   saber_eltwise.cu:6-360                                -> eltwise_*_kernel
//   saber_activation.cu:11-420                            -> activation_kernel
//   saber_scale.cu:8-70                                   -> scale_kernel
//   calibrate.cu:10-700, reorder.cu                       -> nchw_to_nhwc_kernel / nhwc_to_nchw_kernel
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <type_traits>

#include "../../include/b200_saber.h"
#include "common.cuh"
#include "ptx.cuh"
#include "softmax.cuh"
#include "vec.cuh"

namespace b200 {

// ------------------------------------------------------------------ pooling
struct PoolP {
    int n, h, w, c, oh, ow;
    int wh, ww, ph, pw, sh, sw;
    int type;
};

// Window of output pixel (oh, ow) clipped to the image: rows [sh, eh), columns [sw, ew). The padding is never
// negative (b200_pool_out_hw), so this one rule is the reference's for every kind
// (test/saber/test_saber_pooling.cpp:14-104, test/saber/conv_func_helper.h:29-100).
// The clipped window can be empty, with eh - sh or ew - sw equal to 0 or even -1: in ceil mode with no padding and
// stride > window the last row / column starts at or past the edge, and with pad >= window the first lies wholly in
// the padding. Such a window has no taps (pool_taps); its MAX is 0, as in the references.
struct PoolWin {
    int sh, eh, sw, ew;
};
__device__ __forceinline__ PoolWin pool_window(const PoolP& p, int oh, int ow) {
    const int y = oh * p.sh - p.ph, x = ow * p.sw - p.pw;
    return {max(y, 0), min(y + p.wh, p.h), max(x, 0), min(x + p.ww, p.w)};
}
// Taps of a window read in row-major order by the kernels that flatten it: rows x ww columns, 0 when either extent is
// empty (two negative extents must not multiply to a positive count).
__device__ __forceinline__ int pool_taps(const PoolWin& w, int& ww) {
    ww = max(w.ew - w.sw, 0);
    return max(w.eh - w.sh, 0) * ww;
}

// AVG divisor (1 for MAX). The include-padding rules of the two references differ: the float kinds count the window
// clipped to the padded extent, the 8-bit kinds the whole window_h x window_w (pool_basic_check_int8).
template <bool kQ8>
__device__ __forceinline__ float pool_divisor(const PoolP& p, const PoolWin& w) {
    if (p.type == B200_POOL_AVG_EXCLUDE_PAD) return static_cast<float>((w.ew - w.sw) * (w.eh - w.sh));
    if (p.type != B200_POOL_AVG_INCLUDE_PAD) return 1.f;
    if (kQ8) return static_cast<float>(p.wh * p.ww);
    int bh = p.wh, bw = p.ww;
    if (w.ew == p.w) bw = min(w.sw + p.ww, p.w + p.pw) - w.sw;
    if (w.eh == p.h) bh = min(w.sh + p.wh, p.h + p.ph) - w.sh;
    return static_cast<float>(bh * bw);
}

// one tap into a running MAX / sum (fp32, the reference's (kh, kw) order); the window's first tap starts it
__device__ __forceinline__ float pool_fold(float r, float x, bool first, int type) {
    if (first) return x;
    return type == B200_POOL_MAX ? (r >= x ? r : x) : __fadd_rn(r, x);
}

// Small windows, float kinds: one thread = one output vector.
template <int K>
__global__ void pool_thread_kernel(const uint4* __restrict__ in, uint4* __restrict__ out, PoolP p) {
    pdl_enter();
    constexpr int VEC = vec_lanes<K>;
    const int cv = p.c / VEC;
    const long long total = 1ll * p.n * p.oh * p.ow * cv;
    for (long long idx = blockIdx.x * 1ll * blockDim.x + threadIdx.x; idx < total;
         idx += 1ll * gridDim.x * blockDim.x) {
        const int v = static_cast<int>(idx % cv);
        long long t = idx / cv;
        const int ow = static_cast<int>(t % p.ow); t /= p.ow;
        const int oh = static_cast<int>(t % p.oh);
        const int n = static_cast<int>(t / p.oh);
        const PoolWin win = pool_window(p, oh, ow);
        float r[VEC];
#pragma unroll
        for (int i = 0; i < VEC; ++i) r[i] = 0.f;
        for (int kh = win.sh; kh < win.eh; ++kh) {
            for (int kw = win.sw; kw < win.ew; ++kw) {
                float f[VEC];
                unpack_vec<K>(__ldg(in + ((1ll * n * p.h + kh) * p.w + kw) * cv + v), f);
                const bool first = kh == win.sh && kw == win.sw;
#pragma unroll
                for (int i = 0; i < VEC; ++i) r[i] = pool_fold(r[i], f[i], first, p.type);
            }
        }
        if (p.type != B200_POOL_MAX) {
            const float d = pool_divisor<false>(p, win);
#pragma unroll
            for (int i = 0; i < VEC; ++i) r[i] = __fdiv_rn(r[i], d);
        }
        out[((1ll * n * p.oh + oh) * p.ow + ow) * cv + v] = pack_vec<K>(r);
    }
}

// ---- int8 / uint8 pooling with SIMD-in-register integer arithmetic.
// Sums of 8-bit codes are exact in any order (taps * 255 < 2^16 for up to 257 taps), so the float
// reference (sum in fp32, divide, nearbyintf, saturate) is reproduced bit-exactly from integer
// partial sums: bytes are accumulated as packed 16-bit lanes (even / odd bytes of each word), max
// uses the byte-wise video instructions. s8 codes are biased by 0x80 to unsigned and un-biased at
// the end. LANES threads cooperate on one 16-channel output vector (1 for small windows, 8 for
// global pooling) and combine through xor-shuffles.
template <int K, int LANES>
__global__ void pool_q8_simd_kernel(const uint4* __restrict__ in, uint4* __restrict__ out, PoolP p) {
    pdl_enter();
    constexpr bool kUnsigned = K == VK_U8;
    const int cv = p.c >> 4;
    const long long total = 1ll * p.n * p.oh * p.ow * cv;
    const long long tid0 = blockIdx.x * 1ll * blockDim.x + threadIdx.x;
    const int sub = static_cast<int>(tid0 % LANES);
    const long long nthreads = 1ll * gridDim.x * blockDim.x;
    // all 32 lanes of a warp run the same number of iterations (the shuffles below use the full
    // mask); groups past the end just carry zero taps and skip the store
    const long long warp_first = (tid0 - (threadIdx.x & 31)) / LANES;
    for (long long it = 0; warp_first + it * (nthreads / LANES) < total; ++it) {
        const long long idx = tid0 / LANES + it * (nthreads / LANES);
        const bool valid = idx < total;
        const long long cidx = valid ? idx : 0;
        const int v = static_cast<int>(cidx % cv);
        long long t = cidx / cv;
        const int ow = static_cast<int>(t % p.ow); t /= p.ow;
        const int oh = static_cast<int>(t % p.oh);
        const int n = static_cast<int>(t / p.oh);
        const PoolWin win = pool_window(p, oh, ow);
        int ww;
        const int taps = valid ? pool_taps(win, ww) : 0;
        uint32_t mx[4] = {0u, 0u, 0u, 0u};                    // biased-unsigned byte max
        uint32_t se[4] = {0, 0, 0, 0}, so[4] = {0, 0, 0, 0};  // packed 16-bit sums of even / odd bytes
        const bool is_max = p.type == B200_POOL_MAX;
#pragma unroll 4
        for (int tp = sub; tp < taps; tp += LANES) {
            const int kh = win.sh + tp / ww, kw = win.sw + tp % ww;
            const uint4 x = __ldg(in + ((1ll * n * p.h + kh) * p.w + kw) * cv + v);
            uint32_t w[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                if (!kUnsigned) w[i] ^= 0x80808080u;
                if (is_max) {
                    mx[i] = __vmaxu4(mx[i], w[i]);
                } else {
                    se[i] += w[i] & 0x00FF00FFu;
                    so[i] += (w[i] >> 8) & 0x00FF00FFu;
                }
            }
        }
#pragma unroll
        for (int o = LANES >> 1; o > 0; o >>= 1) {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                mx[i] = __vmaxu4(mx[i], __shfl_xor_sync(0xffffffffu, mx[i], o));
                se[i] += __shfl_xor_sync(0xffffffffu, se[i], o);
                so[i] += __shfl_xor_sync(0xffffffffu, so[i], o);
            }
        }
        if (sub != 0 || !valid) continue;
        uint4 o;
        if (is_max) {
            // an empty window's max stays at the biased minimum: write code 0 instead (s8 -128 otherwise)
            const uint32_t flip = kUnsigned || taps == 0 ? 0u : 0x80808080u;
            o = make_uint4(mx[0] ^ flip, mx[1] ^ flip, mx[2] ^ flip, mx[3] ^ flip);
        } else {
            const float d = pool_divisor<true>(p, win);
            const int unbias = kUnsigned ? 0 : 128 * taps;
            o = pack_vec<K>([&](int l) {   // byte l of the vector: byte l % 4 of word l / 4
                const uint32_t s2 = (l & 1) ? so[l >> 2] : se[l >> 2];
                return __fdiv_rn(static_cast<float>(static_cast<int>((l & 2) ? s2 >> 16 : s2 & 0xFFFFu) - unbias), d);
            });
        }
        out[((1ll * n * p.oh + oh) * p.ow + ow) * cv + v] = o;
    }
}

// Large windows (global average pooling: 7x7 = 49 taps): one WARP per output vector. The lanes
// fetch 32 window taps at a time in parallel (the thread-per-output kernel above serialises 49
// dependent L2 round trips), then every lane folds them in the reference's (kh, kw) order through
// shuffles, so the result is bit-identical to the sequential kernels.
template <int K>
__global__ void pool_warp_kernel(const uint4* __restrict__ in, uint4* __restrict__ out, PoolP p) {
    pdl_enter();
    constexpr int VEC = vec_lanes<K>;
    const int cv = p.c / VEC;
    const long long total = 1ll * p.n * p.oh * p.ow * cv;
    const int lane = threadIdx.x & 31;
    const long long warp0 = (blockIdx.x * 1ll * blockDim.x + threadIdx.x) >> 5;
    const long long nwarps = (1ll * gridDim.x * blockDim.x) >> 5;
    for (long long idx = warp0; idx < total; idx += nwarps) {
        const int v = static_cast<int>(idx % cv);
        long long t = idx / cv;
        const int ow = static_cast<int>(t % p.ow); t /= p.ow;
        const int oh = static_cast<int>(t % p.oh);
        const int n = static_cast<int>(t / p.oh);
        const PoolWin win = pool_window(p, oh, ow);
        int ww;
        const int taps = pool_taps(win, ww);
        float r[VEC];
#pragma unroll
        for (int i = 0; i < VEC; ++i) r[i] = 0.f;
        for (int base = 0; base < taps; base += 32) {
            const int mine = base + lane;
            uint4 x = make_uint4(0, 0, 0, 0);
            if (mine < taps) {
                const int kh = win.sh + mine / ww, kw = win.sw + mine % ww;
                x = __ldg(in + ((1ll * n * p.h + kh) * p.w + kw) * cv + v);
            }
            const int cnt = min(32, taps - base);
            for (int i = 0; i < cnt; ++i) {
                uint4 y;
                y.x = __shfl_sync(0xffffffffu, x.x, i); y.y = __shfl_sync(0xffffffffu, x.y, i);
                y.z = __shfl_sync(0xffffffffu, x.z, i); y.w = __shfl_sync(0xffffffffu, x.w, i);
                float f[VEC];
                unpack_vec<K>(y, f);
                const bool first = (base + i) == 0;
#pragma unroll
                for (int j = 0; j < VEC; ++j) r[j] = pool_fold(r[j], f[j], first, p.type);
            }
        }
        if (lane == 0) {
            if (p.type != B200_POOL_MAX) {
                const float d = pool_divisor<(K >= VK_S8)>(p, win);
#pragma unroll
                for (int j = 0; j < VEC; ++j) r[j] = __fdiv_rn(r[j], d);
            }
            out[((1ll * n * p.oh + oh) * p.ow + ow) * cv + v] = pack_vec<K>(r);
        }
    }
}

// ------------------------------------------------------------------ softmax
// inner == 1: one 256-thread CTA per row (the reference uses one thread per row).
__global__ void __launch_bounds__(SOFTMAX_THREADS) softmax_rows_kernel(const float* __restrict__ in, float* __restrict__ out,
                                                                     int rows, int len, int in_pitch, int out_pitch) {
    __shared__ float red[SOFTMAX_THREADS / 32];
    pdl_enter();
    const int row = blockIdx.x;
    if (row >= rows) return;
    softmax_row_block(in + 1ll * row * in_pitch, out + 1ll * row * out_pitch, len, red);
}
// inner > 1 (softmax over a non-innermost axis): one thread per (outer, inner) column.
__global__ void softmax_strided_kernel(const float* __restrict__ in, float* __restrict__ out,
                                       int outer, int len, int inner) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= outer * inner) return;
    const int o = idx / inner, i = idx % inner;
    const float* x = in + (1ll * o * len) * inner + i;
    float* y = out + (1ll * o * len) * inner + i;
    float mx = -3.402823466e+38f;
    for (int a = 0; a < len; ++a) mx = fmaxf(mx, x[1ll * a * inner]);
    float sum = 0.f;
    for (int a = 0; a < len; ++a) { const float e = expf(x[1ll * a * inner] - mx); y[1ll * a * inner] = e; sum += e; }
    for (int a = 0; a < len; ++a) y[1ll * a * inner] = __fdiv_rn(y[1ll * a * inner], sum);
}

// ------------------------------------------------------------------ eltwise
__device__ __forceinline__ float elt_op(int op, float a, float b, float c0, float c1) {
    if (op == B200_ELT_SUM) return __fadd_rn(__fmul_rn(c0, a), __fmul_rn(c1, b));
    if (op == B200_ELT_PROD) return __fmul_rn(a, b);
    return a > b ? a : b;
}
__global__ void eltwise_f32_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                   float* __restrict__ out, size_t count, int op, float c0, float c1,
                                   int relu) {
    const size_t nv = count >> 2;
    const size_t tid = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t i = tid; i < nv; i += stride) {
        const float4 x = __ldg(reinterpret_cast<const float4*>(a) + i);
        const float4 y = __ldg(reinterpret_cast<const float4*>(b) + i);
        float4 r;
        r.x = elt_op(op, x.x, y.x, c0, c1); r.y = elt_op(op, x.y, y.y, c0, c1);
        r.z = elt_op(op, x.z, y.z, c0, c1); r.w = elt_op(op, x.w, y.w, c0, c1);
        if (relu) { r.x = fmaxf(r.x, 0.f); r.y = fmaxf(r.y, 0.f); r.z = fmaxf(r.z, 0.f); r.w = fmaxf(r.w, 0.f); }
        reinterpret_cast<float4*>(out)[i] = r;
    }
    for (size_t i = (nv << 2) + tid; i < count; i += stride) {
        float r = elt_op(op, a[i], b[i], c0, c1);
        out[i] = relu ? fmaxf(r, 0.f) : r;
    }
}
__global__ void eltwise_f16_kernel(const __half* __restrict__ a, const __half* __restrict__ b,
                                   __half* __restrict__ out, size_t count, int op, float c0, float c1,
                                   int relu) {
    const size_t tid = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t i = tid; i < count; i += stride) {
        float r = elt_op(op, __half2float(a[i]), __half2float(b[i]), c0, c1);
        out[i] = __float2half_rn(relu ? fmaxf(r, 0.f) : r);
    }
}
// int8 sum (x86 semantics, reference saber/funcs/impl/x86/saber_eltwise.cpp:72-111):
//   tmp = a*sa + b*sb; relu; saturate(roundf(tmp))   (roundf = half away from zero)
__global__ void eltwise_q8_kernel(const uint8_t* __restrict__ a, int a_unsigned,
                                  const uint8_t* __restrict__ b, int b_unsigned,
                                  uint8_t* __restrict__ out, int out_unsigned, size_t count, float sa,
                                  float sb, int relu) {
    const size_t tid = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    const size_t nv = count >> 4;
    for (size_t i = tid; i < nv; i += stride) {
        const uint4 x = __ldg(reinterpret_cast<const uint4*>(a) + i);
        const uint4 y = __ldg(reinterpret_cast<const uint4*>(b) + i);
        const uint32_t xs[4] = {x.x, x.y, x.z, x.w}, ys[4] = {y.x, y.y, y.z, y.w};
        uint32_t o[4] = {0, 0, 0, 0};
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            const uint32_t xb = (xs[j >> 2] >> (8 * (j & 3))) & 0xffu, yb = (ys[j >> 2] >> (8 * (j & 3))) & 0xffu;
            const float fa = a_unsigned ? static_cast<float>(xb) : static_cast<float>(static_cast<int8_t>(xb));
            const float fb = b_unsigned ? static_cast<float>(yb) : static_cast<float>(static_cast<int8_t>(yb));
            float f = __fadd_rn(__fmul_rn(fa, sa), __fmul_rn(fb, sb));
            if (relu) f = f > 0.f ? f : 0.f;
            float r = roundf(f);
            r = out_unsigned ? fminf(fmaxf(r, 0.f), 255.f) : fminf(fmaxf(r, -128.f), 127.f);
            o[j >> 2] |= (static_cast<uint32_t>(static_cast<int32_t>(r)) & 0xffu) << (8 * (j & 3));
        }
        reinterpret_cast<uint4*>(out)[i] = make_uint4(o[0], o[1], o[2], o[3]);
    }
    for (size_t i = (nv << 4) + tid; i < count; i += stride) {
        const float fa = a_unsigned ? static_cast<float>(a[i]) : static_cast<float>(static_cast<int8_t>(a[i]));
        const float fb = b_unsigned ? static_cast<float>(b[i]) : static_cast<float>(static_cast<int8_t>(b[i]));
        float f = __fadd_rn(__fmul_rn(fa, sa), __fmul_rn(fb, sb));
        if (relu) f = f > 0.f ? f : 0.f;
        float r = roundf(f);
        r = out_unsigned ? fminf(fmaxf(r, 0.f), 255.f) : fminf(fmaxf(r, -128.f), 127.f);
        out[i] = static_cast<uint8_t>(static_cast<int32_t>(r) & 0xff);
    }
}

// ------------------------------------------------------------------ activation / scale
__device__ __forceinline__ float act_op(int act, float x, float slope, float coef) {
    switch (act) {
        case B200_ACT_RELU: return x > 0.f ? x : __fmul_rn(x, slope);
        case B200_ACT_SIGMOID: return __fdiv_rn(1.0f, expf(-x) + 1.0f);
        case B200_ACT_TANH: return tanhf(x);
        case B200_ACT_CLIPPED_RELU: { float y = x > 0.f ? x : 0.f; return y < coef ? y : coef; }
        case B200_ACT_ELU: return x > 0.f ? x : __fmul_rn(coef, expf(x) - 1.f);
        default: return x;
    }
}
__global__ void activation_f32_kernel(const float* __restrict__ in, float* __restrict__ out,
                                      size_t count, int act, float slope, float coef) {
    const size_t tid = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    const size_t nv = count >> 2;
    for (size_t i = tid; i < nv; i += stride) {
        const float4 x = __ldg(reinterpret_cast<const float4*>(in) + i);
        reinterpret_cast<float4*>(out)[i] = make_float4(act_op(act, x.x, slope, coef), act_op(act, x.y, slope, coef),
                                                        act_op(act, x.z, slope, coef), act_op(act, x.w, slope, coef));
    }
    for (size_t i = (nv << 2) + tid; i < count; i += stride) out[i] = act_op(act, in[i], slope, coef);
}
__global__ void activation_f16_kernel(const __half* __restrict__ in, __half* __restrict__ out,
                                      size_t count, int act, float slope, float coef) {
    const size_t tid = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t i = tid; i < count; i += stride)
        out[i] = __float2half_rn(act_op(act, __half2float(in[i]), slope, coef));
}
template <typename T>  // float | __half
__global__ void scale_kernel(const T* __restrict__ in, T* __restrict__ out, size_t pixels, int c,
                             const float* __restrict__ w, const float* __restrict__ b) {
    constexpr bool kHalf = std::is_same<T, __half>::value;
    const size_t total = pixels * c;
    const size_t tid = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t i = tid; i < total; i += stride) {
        const int ch = static_cast<int>(i % c);
        float x;
        if constexpr (kHalf) x = __half2float(in[i]);
        else x = in[i];
        float y = __fmul_rn(x, __ldg(w + ch));
        if (b) y = __fadd_rn(y, __ldg(b + ch));
        if constexpr (kHalf) out[i] = __float2half_rn(y);
        else out[i] = y;
    }
}

// ------------------------------------------------------------------ layout / precision transforms
// Graph-input quantisation (reference x86_utils.h:318-372): s8 = secur_cast2char(x * inv), i.e. roundf, then clamp;
// u8 = static_cast<unsigned char>(x * inv), i.e. truncation, then clamp.
template <int K>
__device__ __forceinline__ int quant_input(float x, float inv_scale) {
    const float t = __fmul_rn(x, inv_scale);
    if constexpr (K == VK_U8) return static_cast<int>(fminf(fmaxf(t, 0.f), 255.f));
    else return static_cast<int>(fminf(fmaxf(roundf(t), -128.f), 127.f));
}

// NCHW fp32 -> NHWC (c padded to c_pad with zeros) of vector kind K; a 32x32 smem transpose of
// the (c, hw) plane keeps both the read (along hw) and the write (along c) coalesced.
template <int K>
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ in, void* __restrict__ out, int c,
                                    int hw, int c_pad, float inv_scale) {
    __shared__ float tile[32][33];
    const int n = blockIdx.z;
    const int hw0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    for (int j = threadIdx.y; j < 32; j += blockDim.y) {
        const int ch = c0 + j, px = hw0 + threadIdx.x;
        tile[j][threadIdx.x] = (ch < c && px < hw) ? __ldg(in + (1ll * n * c + ch) * hw + px) : 0.f;
    }
    __syncthreads();
    for (int j = threadIdx.y; j < 32; j += blockDim.y) {
        const int px = hw0 + j, ch = c0 + threadIdx.x;
        if (px >= hw || ch >= c_pad) continue;
        const float x = tile[threadIdx.x][j];
        const long long o = (1ll * n * hw + px) * c_pad + ch;
        if constexpr (K == VK_F32) static_cast<float*>(out)[o] = x;
        else if constexpr (K == VK_F16) static_cast<__half*>(out)[o] = __float2half_rn(x);
        else static_cast<uint8_t*>(out)[o] = static_cast<uint8_t>(quant_input<K>(x, inv_scale));
    }
}
// Graph inputs have C <= 4 (RGB): one thread per pixel reads C planes (coalesced along hw) and
// writes its whole padded pixel with 16-byte stores.
template <int K>
__global__ void nchw_to_nhwc_smallc_kernel(const float* __restrict__ in, void* __restrict__ out, int n, int c,
                                           int hw, int c_pad, float inv_scale) {
    const long long total = 1ll * n * hw;
    for (long long idx = blockIdx.x * 1ll * blockDim.x + threadIdx.x; idx < total;
         idx += 1ll * gridDim.x * blockDim.x) {
        const int b = static_cast<int>(idx / hw);
        const int px = static_cast<int>(idx - 1ll * b * hw);
        float x[4] = {0.f, 0.f, 0.f, 0.f};
        for (int ch = 0; ch < c; ++ch) x[ch] = __ldg(in + (1ll * b * c + ch) * hw + px);
        if constexpr (K == VK_F32) {
            float4* o = reinterpret_cast<float4*>(static_cast<float*>(out) + idx * c_pad);
            o[0] = make_float4(x[0], x[1], x[2], x[3]);
            for (int q = 1; q < c_pad / 4; ++q) o[q] = make_float4(0.f, 0.f, 0.f, 0.f);
        } else if constexpr (K == VK_F16) {
            uint4* o = reinterpret_cast<uint4*>(static_cast<__half*>(out) + idx * c_pad);
            __half2 a = __floats2half2_rn(x[0], x[1]), bq = __floats2half2_rn(x[2], x[3]);
            o[0] = make_uint4(*reinterpret_cast<uint32_t*>(&a), *reinterpret_cast<uint32_t*>(&bq), 0, 0);
            for (int q = 1; q < c_pad / 8; ++q) o[q] = make_uint4(0, 0, 0, 0);
        } else {
            uint32_t w = 0;
            for (int ch = 0; ch < 4; ++ch) w |= (static_cast<uint32_t>(quant_input<K>(x[ch], inv_scale)) & 0xffu) << (8 * ch);
            uint4* o = reinterpret_cast<uint4*>(static_cast<uint8_t*>(out) + idx * c_pad);
            o[0] = make_uint4(w, 0, 0, 0);
            for (int q = 1; q < c_pad / 16; ++q) o[q] = make_uint4(0, 0, 0, 0);
        }
    }
}

// The 8-bit image counterpart of nchw_to_nhwc_smallc_kernel: one thread per pixel reads its c interleaved bytes,
// normalises them (image_norm, channel order of the descriptor) and writes the padded pixel with the same conversion
// / quantisation -- 16-byte stores when a pixel is a 16-byte multiple (VEC), element stores otherwise.
template <int K, bool VEC>
__global__ void image_to_nhwc_kernel(const uint8_t* __restrict__ in, void* __restrict__ out, long long pixels, int c,
                                     int c_pad, float inv_scale, const b200_image_desc_t img) {
    for (long long idx = blockIdx.x * 1ll * blockDim.x + threadIdx.x; idx < pixels; idx += 1ll * gridDim.x * blockDim.x) {
        const uint8_t* px = in + idx * c;
        float x[4];
#pragma unroll
        for (int ch = 0; ch < 4; ++ch) x[ch] = ch < c ? image_norm(__ldg(px + img.src_channel[ch]), img.mean[ch], img.scale[ch]) : 0.f;
        if constexpr (!VEC) {
            for (int ch = 0; ch < c_pad; ++ch) {
                const float v = ch < 4 ? x[ch] : 0.f;
                const long long o = idx * c_pad + ch;
                if constexpr (K == VK_F32) static_cast<float*>(out)[o] = v;
                else if constexpr (K == VK_F16) static_cast<__half*>(out)[o] = __float2half_rn(v);
                else static_cast<uint8_t*>(out)[o] = static_cast<uint8_t>(quant_input<K>(v, inv_scale));
            }
        } else if constexpr (K == VK_F32) {
            float4* o = reinterpret_cast<float4*>(static_cast<float*>(out) + idx * c_pad);
            o[0] = make_float4(x[0], x[1], x[2], x[3]);
            for (int q = 1; q < c_pad / 4; ++q) o[q] = make_float4(0.f, 0.f, 0.f, 0.f);
        } else if constexpr (K == VK_F16) {
            uint4* o = reinterpret_cast<uint4*>(static_cast<__half*>(out) + idx * c_pad);
            __half2 a = __floats2half2_rn(x[0], x[1]), bq = __floats2half2_rn(x[2], x[3]);
            o[0] = make_uint4(*reinterpret_cast<uint32_t*>(&a), *reinterpret_cast<uint32_t*>(&bq), 0, 0);
            for (int q = 1; q < c_pad / 8; ++q) o[q] = make_uint4(0, 0, 0, 0);
        } else {
            uint32_t w = 0;
            for (int ch = 0; ch < 4; ++ch) w |= (static_cast<uint32_t>(quant_input<K>(x[ch], inv_scale)) & 0xffu) << (8 * ch);
            uint4* o = reinterpret_cast<uint4*>(static_cast<uint8_t*>(out) + idx * c_pad);
            o[0] = make_uint4(w, 0, 0, 0);
            for (int q = 1; q < c_pad / 16; ++q) o[q] = make_uint4(0, 0, 0, 0);
        }
    }
}

template <int K>
__global__ void nhwc_to_nchw_kernel(const void* __restrict__ in, float* __restrict__ out, int c, int hw,
                                    int c_pad, float scale) {
    __shared__ float tile[32][33];
    const int n = blockIdx.z;
    const int hw0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    for (int j = threadIdx.y; j < 32; j += blockDim.y) {
        const int px = hw0 + j, ch = c0 + threadIdx.x;
        float x = 0.f;
        if (px < hw && ch < c) {
            const long long i = (1ll * n * hw + px) * c_pad + ch;
            if constexpr (K == VK_F32) x = static_cast<const float*>(in)[i];
            else if constexpr (K == VK_F16) x = __half2float(static_cast<const __half*>(in)[i]);
            else if constexpr (K == VK_S8) x = static_cast<float>(static_cast<const int8_t*>(in)[i]);
            else x = static_cast<float>(static_cast<const uint8_t*>(in)[i]);
        }
        tile[j][threadIdx.x] = x;
    }
    __syncthreads();
    for (int j = threadIdx.y; j < 32; j += blockDim.y) {
        const int ch = c0 + j, px = hw0 + threadIdx.x;
        if (ch < c && px < hw) out[(1ll * n * c + ch) * hw + px] = __fmul_rn(tile[threadIdx.x][j], scale);
    }
}

// ------------------------------------------------------------------ depthwise conv
// 128-bit vectorised depthwise convolution (saber_depthwiseconv_act.cu:84-295): one thread = one output pixel x 16
// bytes of channels (4 fp32 | 8 fp16 | 16 int8). Consecutive threads take consecutive channel groups of a pixel, so
// every tap is one coalesced 16-byte load per thread of the input and of the [r][s][c] weights (L1-resident).
// The kernels are instantiated for VK_F32, VK_F16 and VK_S8; the 8-bit instance reads s8 or u8 and writes s8 or u8,
// chosen at run time. The three kernels differ in their schedules only: dw_mac and dw_finish are their arithmetic.
template <int K> using dw_acc_t = std::conditional_t<K == VK_S8, int, float>;

// One tap (one 16-byte input / weight pair) into the accumulators of the vector's channels:
//   f32 / f16 : fp32 FMA (the f16 products are exact in fp32)
//   int8      : exact s32 accumulation, dp4a against the weight word masked to one byte = one channel's product
template <int K>
__device__ __forceinline__ void dw_mac(dw_acc_t<K> (&acc)[vec_lanes<K>], const uint4& xq, const uint4& wq, int in_unsigned) {
    const uint32_t xw[4] = {xq.x, xq.y, xq.z, xq.w}, ww[4] = {wq.x, wq.y, wq.z, wq.w};
    if constexpr (K == VK_F32) {
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[i] = __fmaf_rn(__uint_as_float(xw[i]), __uint_as_float(ww[i]), acc[i]);
    } else if constexpr (K == VK_F16) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&xw[i]));
            const float2 c2 = __half22float2(*reinterpret_cast<const __half2*>(&ww[i]));
            acc[2 * i] = __fmaf_rn(a.x, c2.x, acc[2 * i]);
            acc[2 * i + 1] = __fmaf_rn(a.y, c2.y, acc[2 * i + 1]);
        }
    } else {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const uint32_t wm = ww[i] & (0xFFu << (8 * j));
                int& a = acc[4 * i + j];
                if (in_unsigned) asm("dp4a.u32.s32 %0, %1, %2, %0;" : "+r"(a) : "r"(xw[i]), "r"(wm));
                else asm("dp4a.s32.s32 %0, %1, %2, %0;" : "+r"(a) : "r"(xw[i]), "r"(wm));
            }
        }
    }
}

// Epilogue of one output vector; bias(i) and scale(i) are channel i's (each kernel loads them its own way).
//   f32 / f16 : acc + bias, relu(neg_slope), one rounding at the store -- the arithmetic of dwconv_kernel
//   int8      : the x86 Saber epilogue of the conv kernels: f = (acc + bias) * scale, relu, rne + saturate
template <int K, typename Bias, typename Scale>
__device__ __forceinline__ uint4 dw_finish(const dw_acc_t<K> (&acc)[vec_lanes<K>], Bias bias, Scale scale, int relu,
                                           float slope, int out_dtype) {
    return pack_vec<K>(
        [&](int i) {
            float y;
            if constexpr (K == VK_S8) {
                y = __fmul_rn(__fadd_rn(__int2float_rn(acc[i]), bias(i)), scale(i));
                if (relu) y = fmaxf(y, 0.f);
            } else {
                y = acc[i] + bias(i);
                if (relu) y = y > 0.f ? y : y * slope;
            }
            return y;
        },
        out_dtype == B200_UINT8);
}

// bias / scale of channel c0 + i read from global memory; `none` when the pointer is null
__device__ __forceinline__ auto dw_param(const float* p, int c0, float none) {
    return [=](int i) { return p ? __ldg(p + c0 + i) : none; };
}

template <int K>
__global__ void __launch_bounds__(256)
dwconv_vec_kernel(const uint4* __restrict__ in, const uint4* __restrict__ wgt, const float* __restrict__ bias,
                  const float* __restrict__ scale, uint4* __restrict__ out, int n, int h, int w, int cv, int oh, int ow,
                  int r, int s, int ph, int pw, int sh, int sw, int dh, int dw, int relu, float slope, int in_unsigned,
                  int out_dtype) {
    pdl_enter();
    constexpr int NCH = vec_lanes<K>;
    const long long total = 1ll * n * oh * ow * cv;
    for (long long idx = blockIdx.x * 1ll * blockDim.x + threadIdx.x; idx < total; idx += 1ll * gridDim.x * blockDim.x) {
        const int v = static_cast<int>(idx % cv);
        long long t = idx / cv;
        const int x0 = static_cast<int>(t % ow); t /= ow;
        const int y0 = static_cast<int>(t % oh);
        const int b = static_cast<int>(t / oh);
        dw_acc_t<K> acc[NCH];
#pragma unroll
        for (int i = 0; i < NCH; ++i) acc[i] = 0;
        for (int kr = 0; kr < r; ++kr) {
            const int iy = y0 * sh - ph + kr * dh;
            if (iy < 0 || iy >= h) continue;
            for (int ks = 0; ks < s; ++ks) {
                const int ix = x0 * sw - pw + ks * dw;
                if (ix < 0 || ix >= w) continue;
                dw_mac<K>(acc, __ldg(in + ((1ll * b * h + iy) * w + ix) * cv + v), __ldg(wgt + (1ll * kr * s + ks) * cv + v),
                          in_unsigned);
            }
        }
        const int c0 = v * NCH;
        out[((1ll * b * oh + y0) * ow + x0) * cv + v] =
            dw_finish<K>(acc, dw_param(bias, c0, 0.f), dw_param(scale, c0, 1.f), relu, slope, out_dtype);
    }
}

// Same arithmetic, XP adjacent output pixels of one row per thread (filter width S, horizontal stride SW, dilation 1 --
// the MobileNet 3x3 layers): the (XP-1)*SW + S input columns of a filter row are loaded once and shared by the XP outputs,
// the S weight vectors of the row once per thread -- 2.2x fewer instructions and loads per output than one pixel per
// thread. Per output the taps are still accumulated in (r, s) order (a padding tap adds an exact 0), so the results are
// bit-identical to dwconv_vec_kernel.
template <int K, int XP, int S, int SW>
__global__ void __launch_bounds__(256)
dwconv_row_kernel(const uint4* __restrict__ in, const uint4* __restrict__ wgt, const float* __restrict__ bias,
                  const float* __restrict__ scale, uint4* __restrict__ out, int n, int h, int w, int cv, int oh, int ow,
                  int r, int ph, int pw, int sh, int dh, int relu, float slope, int in_unsigned, int out_dtype) {
    pdl_enter();
    constexpr int NCH = vec_lanes<K>;
    constexpr int SPAN = (XP - 1) * SW + S;
    const int xgroups = (ow + XP - 1) / XP;
    const long long total = 1ll * n * oh * xgroups * cv;
    for (long long idx = blockIdx.x * 1ll * blockDim.x + threadIdx.x; idx < total; idx += 1ll * gridDim.x * blockDim.x) {
        const int v = static_cast<int>(idx % cv);
        long long t = idx / cv;
        const int xg = static_cast<int>(t % xgroups); t /= xgroups;
        const int y0 = static_cast<int>(t % oh);
        const int b = static_cast<int>(t / oh);
        const int x0 = xg * XP;
        dw_acc_t<K> acc[XP][NCH];
#pragma unroll
        for (int p = 0; p < XP; ++p) {
#pragma unroll
            for (int i = 0; i < NCH; ++i) acc[p][i] = 0;
        }
        for (int kr = 0; kr < r; ++kr) {
            const int iy = y0 * sh - ph + kr * dh;
            if (iy < 0 || iy >= h) continue;
            uint4 wv[S];
#pragma unroll
            for (int ks = 0; ks < S; ++ks) wv[ks] = __ldg(wgt + (1ll * kr * S + ks) * cv + v);
            const uint4* rowp = in + (1ll * b * h + iy) * w * cv + v;
            uint4 xv[SPAN];
#pragma unroll
            for (int col = 0; col < SPAN; ++col) {
                const int ix = x0 * SW - pw + col;
                xv[col] = (ix >= 0 && ix < w) ? __ldg(rowp + 1ll * ix * cv) : make_uint4(0, 0, 0, 0);
            }
#pragma unroll
            for (int p = 0; p < XP; ++p) {
#pragma unroll
                for (int ks = 0; ks < S; ++ks) dw_mac<K>(acc[p], xv[p * SW + ks], wv[ks], in_unsigned);
            }
        }
        const int c0 = v * NCH;
#pragma unroll
        for (int p = 0; p < XP; ++p) {
            if (x0 + p >= ow) break;
            out[((1ll * b * oh + y0) * ow + x0 + p) * cv + v] =
                dw_finish<K>(acc[p], dw_param(bias, c0, 0.f), dw_param(scale, c0, 1.f), relu, slope, out_dtype);
        }
    }
}

// Shared-memory tiled 3x3 / stride-1 / dilation-1 depthwise conv (the big MobileNet layers). dwconv_row_kernel re-reads
// every input vector ~4.5 times from L1/L2 (3 filter rows x 1.5 for the column overlap of neighbouring threads), which is
// what bounds it at a third of the HBM rate; here a block stages the (8 + 2) x (TW + 2) pixel halo tile of CVB channel
// vectors once (cp.async, zero-filled outside the image) and every tap comes from shared memory: 1.4x halo re-read.
// Thread = (channel vector, 4 adjacent outputs of one row), 256 threads = 8 rows x (32 / CVB) groups x CVB vectors, so a
// tile is 8 x (128 / CVB) output pixels. The row pitch is congruent to CVB * 16 modulo 128 and 8 / CVB rows interleave
// inside a quarter warp, which makes every 16-byte shared load conflict-free. Arithmetic and tap order (r, s) are those of
// dwconv_vec_kernel (a padding tap adds an exact zero): results are bit-identical for INT8, equal for the float kinds.
// One tile per block, three blocks per SM (two for INT8). Measured and dropped (DESIGN section 9): a two-buffer walk over the
// tiles (next tile streaming in under the arithmetic) and a 2 x 2-pixel patch per thread with packed fp32x2 FMAs.
template <int K, int CVB>
__global__ void __launch_bounds__(256, K == VK_S8 ? 2 : 3)
dwconv_tile_kernel(const uint4* __restrict__ in, const uint4* __restrict__ wgt, const float* __restrict__ bias,
                   const float* __restrict__ scale, uint4* __restrict__ out, int h, int w, int cv, int oh, int ow,
                   int ph, int pw, int relu, float slope, int in_unsigned, int out_dtype, int tiles_x, int tiles_y, int cblocks) {
    constexpr int NCH = vec_lanes<K>;
    constexpr int TH = 8, XP = 4, XG = 32 / CVB, TW = XG * XP, IH = TH + 2, IW = TW + 2, YSUB = 8 / CVB;
    constexpr int RAW = IW * CVB * 16;
    constexpr int PITCH = RAW + ((CVB * 16 - RAW % 128) + 128) % 128;
    static_assert(PITCH % 128 == (CVB * 16) % 128 && PITCH % 16 == 0, "row pitch");
    __shared__ __align__(128) uint8_t tile[IH * PITCH];
    pdl_enter();
    const int tid = threadIdx.x;
    // tile index -> (image, tile row, tile column, channel block); channel blocks vary fastest
    auto decode = [&](int ti, int& b, int& ty, int& tx, int& cb) {
        unsigned t = static_cast<unsigned>(ti);
        cb = static_cast<int>(t % static_cast<unsigned>(cblocks)); t /= static_cast<unsigned>(cblocks);
        tx = static_cast<int>(t % static_cast<unsigned>(tiles_x)); t /= static_cast<unsigned>(tiles_x);
        ty = static_cast<int>(t % static_cast<unsigned>(tiles_y));
        b = static_cast<int>(t / static_cast<unsigned>(tiles_y));
    };
    // stage the halo tile of tile `ti` (one cp.async group)
    auto stage = [&](int ti) {
        int b, ty, tx, cb;
        decode(ti, b, ty, tx, cb);
        const int iy0 = ty * TH - ph, ix0 = tx * TW - pw;
        const uint4* img = in + 1ll * b * h * w * cv + cb * CVB;
        const uint32_t tile_s = static_cast<uint32_t>(__cvta_generic_to_shared(tile));
        for (int i = tid; i < IH * IW * CVB; i += 256) {
            const int v = i % CVB, col = (i / CVB) % IW, row = i / (CVB * IW);
            const int iy = iy0 + row, ix = ix0 + col;
            const bool ok = iy >= 0 && iy < h && ix >= 0 && ix < w;
            const uint4* src = ok ? img + (1ll * iy * w + ix) * cv + v : img;
            const uint32_t dst = tile_s + row * PITCH + (col * CVB + v) * 16;
            const int bytes = ok ? 16 : 0;      // src-size 0: the 16 bytes are zero-filled, nothing is read
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(bytes) : "memory");
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    const int v = tid & (CVB - 1);
    const int ysub = (tid / CVB) & (YSUB - 1);
    const int xg = (tid >> 3) & (XG - 1);
    const int y = (tid >> 3) / XG * YSUB + ysub;
    const int ti = blockIdx.x;
    stage(ti);
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();
    {
        int b, ty, tx, cb;
        decode(ti, b, ty, tx, cb);
        const uint8_t* cur = tile;
        const int oy = ty * TH + y, ox0 = tx * TW + xg * XP;
        if (oy < oh && ox0 < ow) {
            const int vg = cb * CVB + v;
            dw_acc_t<K> acc[XP][NCH];
#pragma unroll
            for (int p = 0; p < XP; ++p) {
#pragma unroll
                for (int i = 0; i < NCH; ++i) acc[p][i] = 0;
            }
#pragma unroll
            for (int kr = 0; kr < 3; ++kr) {
                uint4 wv[3];
#pragma unroll
                for (int ks = 0; ks < 3; ++ks) wv[ks] = __ldg(wgt + (kr * 3 + ks) * cv + vg);
                const uint8_t* rowp = cur + (y + kr) * PITCH + (xg * XP * CVB + v) * 16;
                uint4 xv[XP + 2];
#pragma unroll
                for (int col = 0; col < XP + 2; ++col) xv[col] = *reinterpret_cast<const uint4*>(rowp + col * CVB * 16);
#pragma unroll
                for (int p = 0; p < XP; ++p) {
#pragma unroll
                    for (int ks = 0; ks < 3; ++ks) dw_mac<K>(acc[p], xv[p + ks], wv[ks], in_unsigned);
                }
            }
            // ---- epilogue, bias / scale as 16-byte loads
            const int c0 = vg * NCH;
            float bv[NCH], sv[K == VK_S8 ? NCH : 1];
#pragma unroll
            for (int i = 0; i < NCH / 4; ++i) {
                const float4 b4 = bias ? __ldg(reinterpret_cast<const float4*>(bias + c0) + i) : make_float4(0.f, 0.f, 0.f, 0.f);
                bv[4 * i] = b4.x; bv[4 * i + 1] = b4.y; bv[4 * i + 2] = b4.z; bv[4 * i + 3] = b4.w;
                if constexpr (K == VK_S8) {
                    const float4 s4 = scale ? __ldg(reinterpret_cast<const float4*>(scale + c0) + i) : make_float4(1.f, 1.f, 1.f, 1.f);
                    sv[4 * i] = s4.x; sv[4 * i + 1] = s4.y; sv[4 * i + 2] = s4.z; sv[4 * i + 3] = s4.w;
                }
            }
            uint4* orow = out + ((1ll * b * oh + oy) * ow + ox0) * cv + vg;
#pragma unroll
            for (int p = 0; p < XP; ++p) {
                if (ox0 + p >= ow) break;
                orow[1ll * p * cv] = dw_finish<K>(acc[p], [&](int i) { return bv[i]; }, [&](int i) { return sv[i]; }, relu, slope,
                                                  out_dtype);
            }
        }
    }
}

static unsigned grid_for(long long total, int block) {
    long long g = (total + block - 1) / block;
    const long long cap = static_cast<long long>(sm_count()) * 16;
    if (g > cap) g = cap;
    if (g < 1) g = 1;
    return static_cast<unsigned>(g);
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200_pool_out_hw(const b200_pool_desc_t* d, int32_t* ho, int32_t* wo) {
    if (!d || d->h <= 0 || d->w <= 0) return B200_INVALID_VALUE;
    int oh, ow;
    if (d->global_pooling) {
        oh = ow = 1;
    } else {
        if (d->stride_h <= 0 || d->stride_w <= 0 || d->window_h <= 0 || d->window_w <= 0 || d->pad_h < 0 || d->pad_w < 0)
            return B200_INVALID_VALUE;
        if (d->floor_as_conv) {
            oh = static_cast<int>(static_cast<float>(d->h + 2 * d->pad_h - d->window_h) / d->stride_h) + 1;
            ow = static_cast<int>(static_cast<float>(d->w + 2 * d->pad_w - d->window_w) / d->stride_w) + 1;
            if (oh <= 0) oh = 1;
            if (ow <= 0) ow = 1;
        } else {
            oh = static_cast<int>(ceilf(static_cast<float>(d->h + 2 * d->pad_h - d->window_h) / d->stride_h)) + 1;
            ow = static_cast<int>(ceilf(static_cast<float>(d->w + 2 * d->pad_w - d->window_w) / d->stride_w)) + 1;
        }
        if (d->pad_h > 0 || d->pad_w > 0) {
            if ((oh - 1) * d->stride_h >= d->h + d->pad_h) --oh;
            if ((ow - 1) * d->stride_w >= d->w + d->pad_w) --ow;
        }
    }
    if (ho) *ho = oh;
    if (wo) *wo = ow;
    return B200_SUCCESS;
}

int b200_pool_run(const b200_pool_desc_t* d, const void* in, void* out, void* stream) {
    if (!d || !in || !out) return B200_INVALID_VALUE;
    if (!device_is_sm90()) return B200_WRONG_DEVICE;
    PoolP p;
    int32_t oh, ow;
    int st = b200_pool_out_hw(d, &oh, &ow);
    if (st != B200_SUCCESS) return st;
    p.n = d->n; p.h = d->h; p.w = d->w; p.c = d->c; p.oh = oh; p.ow = ow;
    if (d->global_pooling) {
        p.wh = d->h; p.ww = d->w; p.ph = p.pw = 0; p.sh = d->h; p.sw = d->w;
    } else {
        p.wh = d->window_h; p.ww = d->window_w; p.ph = d->pad_h; p.pw = d->pad_w;
        p.sh = d->stride_h; p.sw = d->stride_w;
    }
    p.type = d->type;
    if (p.type < B200_POOL_MAX || p.type > B200_POOL_AVG_EXCLUDE_PAD) return B200_INVALID_VALUE;
    const int block = 256;
    const int taps = p.wh * p.ww;
    const uint4* src = static_cast<const uint4*>(in);
    uint4* dst = static_cast<uint4*>(out);
    return with_vec_kind(d->dtype, [&](auto kind) -> int {
        constexpr int K = decltype(kind)::value;
        if (d->c % vec_lanes<K>) return B200_INVALID_VALUE;
        const long long total = 1ll * p.n * oh * ow * (d->c / vec_lanes<K>);
        const bool big_window = taps >= 16;
        if constexpr (K < VK_S8) {
            if (big_window)
                return launch("pool", Pdl::On, pool_warp_kernel<K>, grid_for(total * 32, block), block, 0, stream, dim3(1),
                              src, dst, p);
            return launch("pool", Pdl::On, pool_thread_kernel<K>, grid_for(total, block), block, 0, stream, dim3(1), src,
                          dst, p);
        } else if (taps > 256) {   // beyond the exact range of the SIMD kernel's 16-bit sums
            return launch("pool", Pdl::On, pool_warp_kernel<K>, grid_for(total * 32, block), block, 0, stream, dim3(1), src,
                          dst, p);
        } else if (big_window) {
            // the grid covers (outputs x LANES) threads, rounded so that LANES-groups never straddle the loop bound
            return launch("pool", Pdl::On, pool_q8_simd_kernel<K, 8>, grid_for(total * 8, block), block, 0, stream, dim3(1),
                          src, dst, p);
        } else {
            return launch("pool", Pdl::On, pool_q8_simd_kernel<K, 1>, grid_for(total, block), block, 0, stream, dim3(1),
                          src, dst, p);
        }
    });
}

int b200_softmax_rows(const float* in, float* out, int32_t rows, int32_t len, int32_t in_pitch,
                      int32_t out_pitch, void* stream) {
    if (!in || !out || rows <= 0 || len <= 0 || in_pitch < len || out_pitch < len) return B200_INVALID_VALUE;
    if (!device_is_sm90()) return B200_WRONG_DEVICE;
    return launch("softmax", Pdl::On, softmax_rows_kernel, static_cast<unsigned>(rows), SOFTMAX_THREADS, 0, stream, dim3(1),
                  in, out, rows, len, in_pitch, out_pitch);
}

int b200_softmax_run(const float* in, float* out, int32_t outer, int32_t axis_size, int32_t inner,
                     void* stream) {
    if (!in || !out || outer <= 0 || axis_size <= 0 || inner <= 0) return B200_INVALID_VALUE;
    if (!device_is_sm90()) return B200_WRONG_DEVICE;
    if (inner == 1) return b200_softmax_rows(in, out, outer, axis_size, axis_size, axis_size, stream);
    const int block = 128;
    return launch("softmax", Pdl::Off, softmax_strided_kernel, (outer * inner + block - 1) / block, block, 0, stream,
                  dim3(1), in, out, outer, axis_size, inner);
}

int b200_eltwise_run(int32_t dtype_a, int32_t dtype_b, int32_t dtype_out, int32_t op, const void* a,
                     const void* b, void* out, size_t count, float c0, float c1, int32_t relu,
                     void* stream) {
    if (!a || !b || !out || count == 0) return B200_INVALID_VALUE;
    if (!device_is_sm90()) return B200_WRONG_DEVICE;
    if (op < B200_ELT_PROD || op > B200_ELT_MAX) return B200_UNIMPL_ERROR;
    const int block = 256;
    if (dtype_a == B200_FLOAT && dtype_b == B200_FLOAT && dtype_out == B200_FLOAT)
        return launch("eltwise", Pdl::Off, eltwise_f32_kernel, grid_for((count + 3) / 4, block), block, 0, stream, dim3(1),
                      static_cast<const float*>(a), static_cast<const float*>(b), static_cast<float*>(out), count, op, c0,
                      c1, relu);
    if (dtype_a == B200_HALF && dtype_b == B200_HALF && dtype_out == B200_HALF)
        return launch("eltwise", Pdl::Off, eltwise_f16_kernel, grid_for(count, block), block, 0, stream, dim3(1),
                      static_cast<const __half*>(a), static_cast<const __half*>(b), static_cast<__half*>(out), count, op,
                      c0, c1, relu);
    auto q8 = [](int dt) { return dt == B200_INT8 || dt == B200_UINT8; };
    if (!q8(dtype_a) || !q8(dtype_b) || !q8(dtype_out) || op != B200_ELT_SUM) return B200_UNIMPL_ERROR;
    return launch("eltwise", Pdl::Off, eltwise_q8_kernel, grid_for((count + 15) / 16, block), block, 0, stream, dim3(1),
                  static_cast<const uint8_t*>(a), dtype_a == B200_UINT8, static_cast<const uint8_t*>(b),
                  dtype_b == B200_UINT8, static_cast<uint8_t*>(out), dtype_out == B200_UINT8, count, c0, c1, relu);
}

int b200_activation_run(int32_t dtype, int32_t act, const void* in, void* out, size_t count,
                        float neg_slope, float coef, void* stream) {
    if (!in || !out || count == 0) return B200_INVALID_VALUE;
    if (!device_is_sm90()) return B200_WRONG_DEVICE;
    const int block = 256;
    if (dtype == B200_FLOAT)
        return launch("activation", Pdl::Off, activation_f32_kernel, grid_for((count + 3) / 4, block), block, 0, stream,
                      dim3(1), static_cast<const float*>(in), static_cast<float*>(out), count, act, neg_slope, coef);
    if (dtype == B200_HALF)
        return launch("activation", Pdl::Off, activation_f16_kernel, grid_for(count, block), block, 0, stream, dim3(1),
                      static_cast<const __half*>(in), static_cast<__half*>(out), count, act, neg_slope, coef);
    return B200_UNIMPL_ERROR;
}

int b200_scale_run(int32_t dtype, const void* in, void* out, size_t pixels, int32_t c, const float* w,
                   const float* b, void* stream) {
    if (!in || !out || !w || pixels == 0 || c <= 0) return B200_INVALID_VALUE;
    if (!device_is_sm90()) return B200_WRONG_DEVICE;
    const int block = 256;
    if (dtype == B200_FLOAT)
        return launch("scale", Pdl::Off, scale_kernel<float>, grid_for(pixels * c, block), block, 0, stream, dim3(1),
                      static_cast<const float*>(in), static_cast<float*>(out), pixels, c, w, b);
    if (dtype == B200_HALF)
        return launch("scale", Pdl::Off, scale_kernel<__half>, grid_for(pixels * c, block), block, 0, stream, dim3(1),
                      static_cast<const __half*>(in), static_cast<__half*>(out), pixels, c, w, b);
    return B200_UNIMPL_ERROR;
}

int b200_nchw_to_nhwc(const float* in, void* out, int32_t out_dtype, int32_t n, int32_t c, int32_t h,
                      int32_t w, int32_t c_pad, float inv_scale, void* stream) {
    if (!in || !out || n <= 0 || c <= 0 || h <= 0 || w <= 0 || c_pad < c) return B200_INVALID_VALUE;
    if (!device_is_sm90()) return B200_WRONG_DEVICE;
    const int hw = h * w;
    return with_vec_kind(out_dtype, [&](auto kind) {
        constexpr int K = decltype(kind)::value;
        if (c <= 4 && c_pad * (16 / vec_lanes<K>) % 16 == 0)
            return launch("nchw_to_nhwc", Pdl::Off, nchw_to_nhwc_smallc_kernel<K>, grid_for(1ll * n * hw, 256), 256, 0,
                          stream, dim3(1), in, out, n, c, hw, c_pad, inv_scale);
        const dim3 grid((hw + 31) / 32, (c_pad + 31) / 32, n), block(32, 8);
        return launch("nchw_to_nhwc", Pdl::Off, nchw_to_nhwc_kernel<K>, grid, block, 0, stream, dim3(1), in, out, c, hw,
                      c_pad, inv_scale);
    });
}

int b200_image_to_nhwc(const b200_image_desc_t* img, const uint8_t* in, void* out, int32_t out_dtype, int32_t n,
                       int32_t c, int32_t h, int32_t w, int32_t c_pad, float inv_scale, void* stream) {
    if (!img || !in || !out || n <= 0 || h <= 0 || w <= 0 || c_pad < c) return B200_INVALID_VALUE;
    if (!b200_image_desc_valid(img, c)) return B200_INVALID_VALUE;
    if (!device_is_sm90()) return B200_WRONG_DEVICE;
    const long long pixels = 1ll * n * h * w;
    return with_vec_kind(out_dtype, [&](auto kind) {
        constexpr int K = decltype(kind)::value;
        const bool vec = c_pad * (16 / vec_lanes<K>) % 16 == 0;
        return launch("image_to_nhwc", Pdl::Off, vec ? image_to_nhwc_kernel<K, true> : image_to_nhwc_kernel<K, false>,
                      grid_for(pixels, 256), 256, 0, stream, dim3(1), in, out, pixels, c, c_pad, inv_scale, *img);
    });
}

int b200_nhwc_to_nchw(const void* in, int32_t in_dtype, float* out, int32_t n, int32_t c, int32_t h,
                      int32_t w, int32_t c_pad, float scale, void* stream) {
    if (!in || !out || n <= 0 || c <= 0 || h <= 0 || w <= 0 || c_pad < c) return B200_INVALID_VALUE;
    if (!device_is_sm90()) return B200_WRONG_DEVICE;
    const int hw = h * w;
    const dim3 grid((hw + 31) / 32, (c + 31) / 32, n), block(32, 8);
    return with_vec_kind(in_dtype, [&](auto kind) {
        return launch("nhwc_to_nchw", Pdl::Off, nhwc_to_nchw_kernel<decltype(kind)::value>, grid, block, 0, stream, dim3(1),
                      in, out, c, hw, c_pad, scale);
    });
}

int b200_dwconv_run(const b200_conv_desc_t* d, const void* in, const void* weights_rsc,
                    const float* bias, const float* scale, void* out, void* stream) {
    if (!d || !in || !weights_rsc || !out) return B200_INVALID_VALUE;
    if (!device_is_sm90()) return B200_WRONG_DEVICE;
    if (d->k != d->c) return B200_INVALID_VALUE;
    const int oh = (d->h + 2 * d->pad_h - (d->dil_h * (d->r - 1) + 1)) / d->stride_h + 1;
    const int ow = (d->w + 2 * d->pad_w - (d->dil_w * (d->s - 1) + 1)) / d->stride_w + 1;
    if (oh <= 0 || ow <= 0) return B200_INVALID_VALUE;
    // the float kinds keep their dtype; the 8-bit kernels read s8 | u8 and write s8 | u8
    const bool q8_in = d->in_dtype == B200_INT8 || d->in_dtype == B200_UINT8;
    const bool q8_out = d->out_dtype == B200_INT8 || d->out_dtype == B200_UINT8;
    if (q8_in ? !q8_out : d->out_dtype != d->in_dtype) return B200_UNIMPL_ERROR;
    const int block = 256;
    const uint4* in4 = static_cast<const uint4*>(in);
    const uint4* w4 = static_cast<const uint4*>(weights_rsc);
    uint4* out4 = static_cast<uint4*>(out);
    const int in_unsigned = d->in_dtype == B200_UINT8 ? 1 : 0;
    return with_vec_kind(d->in_dtype, [&](auto kind) -> int {
        constexpr int K = decltype(kind)::value == VK_U8 ? VK_S8 : decltype(kind)::value;
        if (d->c % vec_lanes<K>) return B200_INVALID_VALUE;
        const int cv = d->c / vec_lanes<K>;
        // big 3x3 / stride-1 layers: the shared-memory tiled kernel, where the tile is not mostly halo and idle lanes
        const int cvb = cv % 8 == 0 ? 8 : (cv == 4 ? 4 : (cv == 2 ? 2 : 0));
        if (cvb && d->r == 3 && d->s == 3 && d->stride_h == 1 && d->stride_w == 1 && d->dil_h == 1 && d->dil_w == 1 &&
            d->pad_h <= 1 && d->pad_w <= 1) {
            const int tw = 128 / cvb;
            const int tiles_x = (ow + tw - 1) / tw, tiles_y = (oh + 7) / 8, cblocks = cv / cvb;
            const double util = static_cast<double>(oh) * ow / (static_cast<double>(tiles_y) * 8 * tiles_x * tw);
            const long long blocks = 1ll * d->n * tiles_y * tiles_x * cblocks;
            // INT8 (its row kernel keeps only 2 outputs per thread): from 7 x 7 up (MobileNet-v1 INT8 b16 in-net 12.97 -> 7.32 us
            // per 14 x 14 layer); float kinds: from 28 x 28 (at 14 x 14 the row kernel is 0.4 us faster per layer)
            const bool take = K == VK_S8 ? util >= 0.35 : (util >= 0.6 && oh * ow >= 28 * 28);
            if (blocks < (1ll << 31) && take) {
                auto tile = [&](auto vecs) {
                    return launch("dwconv", Pdl::On, dwconv_tile_kernel<K, decltype(vecs)::value>,
                                  static_cast<unsigned>(blocks), block, 0, stream, dim3(1), in4, w4, bias, scale, out4, d->h,
                                  d->w, cv, oh, ow, d->pad_h, d->pad_w, d->relu, d->neg_slope, in_unsigned, d->out_dtype,
                                  tiles_x, tiles_y, cblocks);
                };
                if (cvb == 8) return tile(Int<8>());
                if (cvb == 4) return tile(Int<4>());
                return tile(Int<2>());
            }
        }
        if (d->s == 3 && d->dil_w == 1 && (d->stride_w == 1 || d->stride_w == 2)) {
            // 3-wide filters: several adjacent outputs per thread (dwconv_row_kernel)
            constexpr int XP = K == VK_S8 ? 2 : 4;
            const unsigned g = grid_for(1ll * d->n * oh * ((ow + XP - 1) / XP) * cv, block);
            auto row = [&](auto sw) {
                return launch("dwconv", Pdl::On, dwconv_row_kernel<K, XP, 3, decltype(sw)::value>, g, block, 0, stream,
                              dim3(1), in4, w4, bias, scale, out4, d->n, d->h, d->w, cv, oh, ow, d->r, d->pad_h, d->pad_w,
                              d->stride_h, d->dil_h, d->relu, d->neg_slope, in_unsigned, d->out_dtype);
            };
            return d->stride_w == 1 ? row(Int<1>()) : row(Int<2>());
        }
        return launch("dwconv", Pdl::On, dwconv_vec_kernel<K>, grid_for(1ll * d->n * oh * ow * cv, block), block, 0, stream,
                      dim3(1), in4, w4, bias, scale, out4, d->n, d->h, d->w, cv, oh, ow, d->r, d->s, d->pad_h, d->pad_w,
                      d->stride_h, d->stride_w, d->dil_h, d->dil_w, d->relu, d->neg_slope, in_unsigned, d->out_dtype);
    });
}

}  // extern "C"
