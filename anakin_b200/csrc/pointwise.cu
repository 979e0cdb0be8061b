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
#include <stdio.h>

#include "../../include/b200_saber.h"
#include "common.cuh"
#include "softmax.cuh"

namespace b200 {

static inline cudaStream_t S(void* s) { return static_cast<cudaStream_t>(s); }

// Programmatic dependent launch for the pointwise kernels that sit between tensor-core convs: the
// kernel signals its dependents at once and waits for its predecessor before touching memory, so
// launch latency and the neighbours' prologues overlap along the whole chain.
__device__ __forceinline__ void pdl_enter() {
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    asm volatile("griddepcontrol.wait;" ::: "memory");
}

template <typename Kern, typename... Args>
static void launch_pdl(Kern kern, unsigned grid, unsigned block, cudaStream_t stream, Args... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(block);
    cfg.dynamicSmemBytes = 0;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    cudaLaunchKernelEx(&cfg, kern, args...);
}

template <typename Kern, typename... Args>
static void launch_pdl_smem(Kern kern, unsigned grid, unsigned block, size_t smem, cudaStream_t stream, Args... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(block);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    cudaLaunchKernelEx(&cfg, kern, args...);
}

static int check_launch(const char* what) {
    count_launch();
    cudaError_t e = cudaPeekAtLastError();
    if (e != cudaSuccess) {
        fprintf(stderr, "[b200_saber] %s launch failed: %s\n", what, cudaGetErrorString(e));
        return B200_UNKNOWN_ERROR;
    }
    return B200_SUCCESS;
}

// ------------------------------------------------------------------ pooling
struct PoolP {
    int n, h, w, c, oh, ow;
    int wh, ww, ph, pw, sh, sw;
    int type;
};

// One thread = one output pixel x 4 fp32 channels.
// Window logic = reference test/saber/test_saber_pooling.cpp:14-104 (incl. the
// include-padding divisor rule).
__global__ void pool_f32_kernel(const float4* __restrict__ in, float4* __restrict__ out, PoolP p) {
    pdl_enter();
    const int cv = p.c >> 2;
    const long long total = 1ll * p.n * p.oh * p.ow * cv;
    for (long long idx = blockIdx.x * 1ll * blockDim.x + threadIdx.x; idx < total;
         idx += 1ll * gridDim.x * blockDim.x) {
        const int v = static_cast<int>(idx % cv);
        long long t = idx / cv;
        const int ow = static_cast<int>(t % p.ow); t /= p.ow;
        const int oh = static_cast<int>(t % p.oh);
        const int n = static_cast<int>(t / p.oh);
        int sh = oh * p.sh, eh = sh + p.wh;
        sh = (sh - p.ph) < 0 ? 0 : sh - p.ph;
        eh = (eh - p.ph) > p.h ? p.h : eh - p.ph;
        int sw = ow * p.sw, ew = sw + p.ww;
        sw = (sw - p.pw) < 0 ? 0 : sw - p.pw;
        ew = (ew - p.pw) > p.w ? p.w : ew - p.pw;
        float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int kh = sh; kh < eh; ++kh) {
            for (int kw = sw; kw < ew; ++kw) {
                const float4 x = __ldg(in + ((1ll * n * p.h + kh) * p.w + kw) * cv + v);
                if (kh == sh && kw == sw) {
                    r = x;
                } else if (p.type == B200_POOL_MAX) {
                    r.x = r.x >= x.x ? r.x : x.x; r.y = r.y >= x.y ? r.y : x.y;
                    r.z = r.z >= x.z ? r.z : x.z; r.w = r.w >= x.w ? r.w : x.w;
                } else {
                    r.x = __fadd_rn(r.x, x.x); r.y = __fadd_rn(r.y, x.y);
                    r.z = __fadd_rn(r.z, x.z); r.w = __fadd_rn(r.w, x.w);
                }
            }
        }
        if (p.type == B200_POOL_AVG_INCLUDE_PAD) {
            int bh = p.wh, bw = p.ww;
            if (ew == p.w) { bw = (sw + p.ww >= p.w + p.pw) ? p.w + p.pw : sw + p.ww; bw -= sw; }
            if (eh == p.h) { bh = (sh + p.wh >= p.h + p.ph) ? p.h + p.ph : sh + p.wh; bh -= sh; }
            const float d = static_cast<float>(bh * bw);
            r.x = __fdiv_rn(r.x, d); r.y = __fdiv_rn(r.y, d); r.z = __fdiv_rn(r.z, d); r.w = __fdiv_rn(r.w, d);
        } else if (p.type == B200_POOL_AVG_EXCLUDE_PAD) {
            const float d = static_cast<float>((ew - sw) * (eh - sh));
            r.x = __fdiv_rn(r.x, d); r.y = __fdiv_rn(r.y, d); r.z = __fdiv_rn(r.z, d); r.w = __fdiv_rn(r.w, d);
        }
        out[((1ll * n * p.oh + oh) * p.ow + ow) * cv + v] = r;
    }
}

// fp16: 8 channels per thread, accumulate in fp32.
__global__ void pool_f16_kernel(const uint4* __restrict__ in, uint4* __restrict__ out, PoolP p) {
    pdl_enter();
    const int cv = p.c >> 3;
    const long long total = 1ll * p.n * p.oh * p.ow * cv;
    for (long long idx = blockIdx.x * 1ll * blockDim.x + threadIdx.x; idx < total;
         idx += 1ll * gridDim.x * blockDim.x) {
        const int v = static_cast<int>(idx % cv);
        long long t = idx / cv;
        const int ow = static_cast<int>(t % p.ow); t /= p.ow;
        const int oh = static_cast<int>(t % p.oh);
        const int n = static_cast<int>(t / p.oh);
        int sh = oh * p.sh, eh = sh + p.wh;
        sh = (sh - p.ph) < 0 ? 0 : sh - p.ph;
        eh = (eh - p.ph) > p.h ? p.h : eh - p.ph;
        int sw = ow * p.sw, ew = sw + p.ww;
        sw = (sw - p.pw) < 0 ? 0 : sw - p.pw;
        ew = (ew - p.pw) > p.w ? p.w : ew - p.pw;
        float r[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) r[i] = 0.f;
        for (int kh = sh; kh < eh; ++kh) {
            for (int kw = sw; kw < ew; ++kw) {
                const uint4 x = __ldg(in + ((1ll * n * p.h + kh) * p.w + kw) * cv + v);
                const __half2* hx = reinterpret_cast<const __half2*>(&x);
                float f[8];
#pragma unroll
                for (int i = 0; i < 4; ++i) { float2 q = __half22float2(hx[i]); f[2 * i] = q.x; f[2 * i + 1] = q.y; }
                const bool first = (kh == sh && kw == sw);
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    if (first) r[i] = f[i];
                    else if (p.type == B200_POOL_MAX) r[i] = r[i] >= f[i] ? r[i] : f[i];
                    else r[i] = __fadd_rn(r[i], f[i]);
                }
            }
        }
        float d = 1.f;
        if (p.type == B200_POOL_AVG_INCLUDE_PAD) {
            int bh = p.wh, bw = p.ww;
            if (ew == p.w) { bw = (sw + p.ww >= p.w + p.pw) ? p.w + p.pw : sw + p.ww; bw -= sw; }
            if (eh == p.h) { bh = (sh + p.wh >= p.h + p.ph) ? p.h + p.ph : sh + p.wh; bh -= sh; }
            d = static_cast<float>(bh * bw);
        } else if (p.type == B200_POOL_AVG_EXCLUDE_PAD) {
            d = static_cast<float>((ew - sw) * (eh - sh));
        }
        uint4 o;
        __half2* ho = reinterpret_cast<__half2*>(&o);
#pragma unroll
        for (int i = 0; i < 4; ++i)
            ho[i] = __floats2half2_rn(__fdiv_rn(r[2 * i], d), __fdiv_rn(r[2 * i + 1], d));
        out[((1ll * n * p.oh + oh) * p.ow + ow) * cv + v] = o;
    }
}

// int8 / uint8 NHWC: 16 channels per thread. Semantics = reference
// test/saber/conv_func_helper.h:29-100 (pool_basic_check_int8): float sum of the raw
// codes, avg-incl divides by window_h*window_w, nearbyintf (RNE), saturate.
template <bool kUnsigned>
__global__ void pool_q8_kernel(const uint4* __restrict__ in, uint4* __restrict__ out, PoolP p) {
    pdl_enter();
    const int cv = p.c >> 4;
    const long long total = 1ll * p.n * p.oh * p.ow * cv;
    for (long long idx = blockIdx.x * 1ll * blockDim.x + threadIdx.x; idx < total;
         idx += 1ll * gridDim.x * blockDim.x) {
        const int v = static_cast<int>(idx % cv);
        long long t = idx / cv;
        const int ow = static_cast<int>(t % p.ow); t /= p.ow;
        const int oh = static_cast<int>(t % p.oh);
        const int n = static_cast<int>(t / p.oh);
        int sh = oh * p.sh, eh = sh + p.wh;
        if (p.ph > 0) {
            sh = (sh - p.ph) < 0 ? 0 : sh - p.ph;
            eh = (eh - p.ph) > p.h ? p.h : eh - p.ph;
        }
        if (eh > p.h) eh = p.h;
        int sw = ow * p.sw, ew = sw + p.ww;
        if (p.pw > 0) {
            sw = (sw - p.pw) < 0 ? 0 : sw - p.pw;
            ew = (ew - p.pw) > p.w ? p.w : ew - p.pw;
        }
        if (ew > p.w) ew = p.w;
        float r[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) r[i] = 0.f;
        for (int kh = sh; kh < eh; ++kh) {
            for (int kw = sw; kw < ew; ++kw) {
                const uint4 x = __ldg(in + ((1ll * n * p.h + kh) * p.w + kw) * cv + v);
                const uint32_t wds[4] = {x.x, x.y, x.z, x.w};
                const bool first = (kh == sh && kw == sw);
#pragma unroll
                for (int i = 0; i < 16; ++i) {
                    const uint32_t b = (wds[i >> 2] >> (8 * (i & 3))) & 0xffu;
                    const float f = kUnsigned ? static_cast<float>(b)
                                              : static_cast<float>(static_cast<int8_t>(b));
                    if (first) r[i] = f;
                    else if (p.type == B200_POOL_MAX) r[i] = r[i] >= f ? r[i] : f;
                    else r[i] = __fadd_rn(r[i], f);
                }
            }
        }
        float d = 1.f;
        if (p.type == B200_POOL_AVG_INCLUDE_PAD) d = static_cast<float>(p.wh * p.ww);
        else if (p.type == B200_POOL_AVG_EXCLUDE_PAD) d = static_cast<float>((ew - sw) * (eh - sh));
        uint32_t o[4] = {0, 0, 0, 0};
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            const float q = (p.type == B200_POOL_MAX) ? r[i] : __fdiv_rn(r[i], d);
            uint32_t code;
            if (kUnsigned) asm("cvt.rni.sat.u8.f32 %0, %1;" : "=r"(code) : "f"(q));
            else { int32_t sc; asm("cvt.rni.sat.s8.f32 %0, %1;" : "=r"(sc) : "f"(q)); code = static_cast<uint32_t>(sc) & 0xffu; }
            o[i >> 2] |= (code & 0xffu) << (8 * (i & 3));
        }
        out[((1ll * n * p.oh + oh) * p.ow + ow) * cv + v] = make_uint4(o[0], o[1], o[2], o[3]);
    }
}

// ---- int8 / uint8 pooling with SIMD-in-register integer arithmetic.
// Sums of 8-bit codes are exact in any order (taps * 255 < 2^16 for up to 257 taps), so the float
// reference (sum in fp32, divide, nearbyintf, saturate) is reproduced bit-exactly from integer
// partial sums: bytes are accumulated as packed 16-bit lanes (even / odd bytes of each word), max
// uses the byte-wise video instructions. s8 codes are biased by 0x80 to unsigned and un-biased at
// the end. LANES threads cooperate on one 16-channel output vector (1 for small windows, 8 for
// global pooling) and combine through xor-shuffles.
template <bool kUnsigned, int LANES>
__global__ void pool_q8_simd_kernel(const uint4* __restrict__ in, uint4* __restrict__ out, PoolP p) {
    pdl_enter();
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
        int sh = oh * p.sh, eh = sh + p.wh;
        int sw = ow * p.sw, ew = sw + p.ww;
        if (p.ph > 0) { sh = (sh - p.ph) < 0 ? 0 : sh - p.ph; eh = (eh - p.ph) > p.h ? p.h : eh - p.ph; }
        if (p.pw > 0) { sw = (sw - p.pw) < 0 ? 0 : sw - p.pw; ew = (ew - p.pw) > p.w ? p.w : ew - p.pw; }
        if (eh > p.h) eh = p.h;
        if (ew > p.w) ew = p.w;
        const int ww = ew - sw, taps = valid ? (eh - sh) * ww : 0;
        uint32_t mx[4] = {0u, 0u, 0u, 0u};                    // biased-unsigned byte max
        uint32_t se[4] = {0, 0, 0, 0}, so[4] = {0, 0, 0, 0};  // packed 16-bit sums of even / odd bytes
        const bool is_max = p.type == B200_POOL_MAX;
#pragma unroll 4
        for (int tp = sub; tp < taps; tp += LANES) {
            const int kh = sh + tp / ww, kw = sw + tp % ww;
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
        uint32_t ow_[4];
        if (is_max) {
#pragma unroll
            for (int i = 0; i < 4; ++i) ow_[i] = kUnsigned ? mx[i] : (mx[i] ^ 0x80808080u);
        } else {
            const float d = (p.type == B200_POOL_AVG_INCLUDE_PAD) ? static_cast<float>(p.wh * p.ww)
                                                                  : static_cast<float>((ew - sw) * (eh - sh));
            const int unbias = kUnsigned ? 0 : 128 * taps;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int s0 = static_cast<int>(se[i] & 0xFFFFu) - unbias, s2 = static_cast<int>(se[i] >> 16) - unbias;
                const int s1 = static_cast<int>(so[i] & 0xFFFFu) - unbias, s3 = static_cast<int>(so[i] >> 16) - unbias;
                const float q0 = __fdiv_rn(static_cast<float>(s0), d), q1 = __fdiv_rn(static_cast<float>(s1), d);
                const float q2 = __fdiv_rn(static_cast<float>(s2), d), q3 = __fdiv_rn(static_cast<float>(s3), d);
                uint32_t c0, c1, c2, c3;
                if (kUnsigned) {
                    asm("cvt.rni.sat.u8.f32 %0, %1;" : "=r"(c0) : "f"(q0)); asm("cvt.rni.sat.u8.f32 %0, %1;" : "=r"(c1) : "f"(q1));
                    asm("cvt.rni.sat.u8.f32 %0, %1;" : "=r"(c2) : "f"(q2)); asm("cvt.rni.sat.u8.f32 %0, %1;" : "=r"(c3) : "f"(q3));
                } else {
                    int32_t t0, t1, t2, t3;
                    asm("cvt.rni.sat.s8.f32 %0, %1;" : "=r"(t0) : "f"(q0)); asm("cvt.rni.sat.s8.f32 %0, %1;" : "=r"(t1) : "f"(q1));
                    asm("cvt.rni.sat.s8.f32 %0, %1;" : "=r"(t2) : "f"(q2)); asm("cvt.rni.sat.s8.f32 %0, %1;" : "=r"(t3) : "f"(q3));
                    c0 = t0 & 0xff; c1 = t1 & 0xff; c2 = t2 & 0xff; c3 = t3 & 0xff;
                }
                ow_[i] = (c0 & 0xffu) | ((c1 & 0xffu) << 8) | ((c2 & 0xffu) << 16) | ((c3 & 0xffu) << 24);
            }
        }
        out[((1ll * n * p.oh + oh) * p.ow + ow) * cv + v] = make_uint4(ow_[0], ow_[1], ow_[2], ow_[3]);
    }
}

// Large windows (global average pooling: 7x7 = 49 taps): one WARP per output vector. The lanes
// fetch 32 window taps at a time in parallel (the thread-per-output kernel above serialises 49
// dependent L2 round trips), then every lane folds them in the reference's (kh, kw) order through
// shuffles, so the result is bit-identical to the sequential kernels.
template <int MODE>  // 0 f32 (4 ch), 1 f16 (8 ch), 2 s8 (16 ch), 3 u8 (16 ch)
__global__ void pool_warp_kernel(const uint4* __restrict__ in, uint4* __restrict__ out, PoolP p) {
    pdl_enter();
    constexpr int VEC = MODE == 0 ? 4 : (MODE == 1 ? 8 : 16);
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
        int sh = oh * p.sh, eh = sh + p.wh;
        int sw = ow * p.sw, ew = sw + p.ww;
        if (MODE < 2 || p.ph > 0) { sh = (sh - p.ph) < 0 ? 0 : sh - p.ph; eh = (eh - p.ph) > p.h ? p.h : eh - p.ph; }
        if (MODE < 2 || p.pw > 0) { sw = (sw - p.pw) < 0 ? 0 : sw - p.pw; ew = (ew - p.pw) > p.w ? p.w : ew - p.pw; }
        if (eh > p.h) eh = p.h;
        if (ew > p.w) ew = p.w;
        const int ww = ew - sw, taps = (eh - sh) * ww;
        float r[VEC];
#pragma unroll
        for (int i = 0; i < VEC; ++i) r[i] = 0.f;
        for (int base = 0; base < taps; base += 32) {
            const int mine = base + lane;
            uint4 x = make_uint4(0, 0, 0, 0);
            if (mine < taps) {
                const int kh = sh + mine / ww, kw = sw + mine % ww;
                x = __ldg(in + ((1ll * n * p.h + kh) * p.w + kw) * cv + v);
            }
            const int cnt = min(32, taps - base);
            for (int i = 0; i < cnt; ++i) {
                uint4 y;
                y.x = __shfl_sync(0xffffffffu, x.x, i); y.y = __shfl_sync(0xffffffffu, x.y, i);
                y.z = __shfl_sync(0xffffffffu, x.z, i); y.w = __shfl_sync(0xffffffffu, x.w, i);
                float f[VEC];
                if (MODE == 0) {
                    f[0] = __uint_as_float(y.x); f[1] = __uint_as_float(y.y);
                    f[2] = __uint_as_float(y.z); f[3] = __uint_as_float(y.w);
                } else if (MODE == 1) {
                    const __half2* h = reinterpret_cast<const __half2*>(&y);
#pragma unroll
                    for (int j = 0; j < 4; ++j) { float2 q = __half22float2(h[j]); f[2 * j] = q.x; f[2 * j + 1] = q.y; }
                } else {
                    const uint32_t w[4] = {y.x, y.y, y.z, y.w};
#pragma unroll
                    for (int j = 0; j < VEC; ++j) {
                        const uint32_t b = (w[j >> 2] >> (8 * (j & 3))) & 0xffu;
                        f[j] = MODE == 3 ? static_cast<float>(b) : static_cast<float>(static_cast<int8_t>(b));
                    }
                }
                const bool first = (base + i) == 0;
#pragma unroll
                for (int j = 0; j < VEC; ++j) {
                    if (first) r[j] = f[j];
                    else if (p.type == B200_POOL_MAX) r[j] = r[j] >= f[j] ? r[j] : f[j];
                    else r[j] = __fadd_rn(r[j], f[j]);
                }
            }
        }
        float d = 1.f;
        if (p.type == B200_POOL_AVG_INCLUDE_PAD) {
            if (MODE < 2) {
                int bh = p.wh, bw = p.ww;
                if (ew == p.w) { bw = (sw + p.ww >= p.w + p.pw) ? p.w + p.pw : sw + p.ww; bw -= sw; }
                if (eh == p.h) { bh = (sh + p.wh >= p.h + p.ph) ? p.h + p.ph : sh + p.wh; bh -= sh; }
                d = static_cast<float>(bh * bw);
            } else {
                d = static_cast<float>(p.wh * p.ww);
            }
        } else if (p.type == B200_POOL_AVG_EXCLUDE_PAD) {
            d = static_cast<float>((ew - sw) * (eh - sh));
        }
        if (lane == 0) {
            uint4 o = make_uint4(0, 0, 0, 0);
            if (MODE == 0) {
                const bool avg = p.type != B200_POOL_MAX;
                o.x = __float_as_uint(avg ? __fdiv_rn(r[0], d) : r[0]); o.y = __float_as_uint(avg ? __fdiv_rn(r[1], d) : r[1]);
                o.z = __float_as_uint(avg ? __fdiv_rn(r[2], d) : r[2]); o.w = __float_as_uint(avg ? __fdiv_rn(r[3], d) : r[3]);
            } else if (MODE == 1) {
                __half2* ho = reinterpret_cast<__half2*>(&o);
#pragma unroll
                for (int j = 0; j < 4; ++j) ho[j] = __floats2half2_rn(__fdiv_rn(r[2 * j], d), __fdiv_rn(r[2 * j + 1], d));
            } else {
                uint32_t w[4] = {0, 0, 0, 0};
#pragma unroll
                for (int j = 0; j < VEC; ++j) {
                    const float q = (p.type == B200_POOL_MAX) ? r[j] : __fdiv_rn(r[j], d);
                    uint32_t code;
                    if (MODE == 3) asm("cvt.rni.sat.u8.f32 %0, %1;" : "=r"(code) : "f"(q));
                    else { int32_t sc; asm("cvt.rni.sat.s8.f32 %0, %1;" : "=r"(sc) : "f"(q)); code = static_cast<uint32_t>(sc) & 0xffu; }
                    w[j >> 2] |= (code & 0xffu) << (8 * (j & 3));
                }
                o = make_uint4(w[0], w[1], w[2], w[3]);
            }
            out[((1ll * n * p.oh + oh) * p.ow + ow) * cv + v] = o;
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
__global__ void scale_f32_kernel(const float* __restrict__ in, float* __restrict__ out, size_t pixels,
                                 int c, const float* __restrict__ w, const float* __restrict__ b) {
    const size_t total = pixels * c;
    const size_t tid = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t i = tid; i < total; i += stride) {
        const int ch = static_cast<int>(i % c);
        float y = __fmul_rn(in[i], __ldg(w + ch));
        if (b) y = __fadd_rn(y, __ldg(b + ch));
        out[i] = y;
    }
}
__global__ void scale_f16_kernel(const __half* __restrict__ in, __half* __restrict__ out, size_t pixels,
                                 int c, const float* __restrict__ w, const float* __restrict__ b) {
    const size_t total = pixels * c;
    const size_t tid = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t i = tid; i < total; i += stride) {
        const int ch = static_cast<int>(i % c);
        float y = __fmul_rn(__half2float(in[i]), __ldg(w + ch));
        if (b) y = __fadd_rn(y, __ldg(b + ch));
        out[i] = __float2half_rn(y);
    }
}

// ------------------------------------------------------------------ layout / precision transforms
// NCHW fp32 -> NHWC (c padded to c_pad with zeros) in out_dtype; a 32x32 smem transpose of
// the (c, hw) plane keeps both the read (along hw) and the write (along c) coalesced.
template <int OUT>  // 0 f32, 1 f16, 2 s8, 3 u8
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
        if (OUT == 0) {
            static_cast<float*>(out)[o] = x;
        } else if (OUT == 1) {
            static_cast<__half*>(out)[o] = __float2half_rn(x);
        } else if (OUT == 2) {
            // secur_cast2char(x * inv): roundf + clamp (reference x86_utils.h:318-347)
            float t = roundf(__fmul_rn(x, inv_scale));
            t = fminf(fmaxf(t, -128.f), 127.f);
            static_cast<int8_t*>(out)[o] = static_cast<int8_t>(static_cast<int>(t));
        } else {
            // static_cast<unsigned char>(x * inv): truncation (reference x86_utils.h:360-372)
            float t = __fmul_rn(x, inv_scale);
            t = fminf(fmaxf(t, 0.f), 255.f);
            static_cast<uint8_t*>(out)[o] = static_cast<uint8_t>(static_cast<int>(t));
        }
    }
}
// Graph inputs have C <= 4 (RGB): one thread per pixel reads C planes (coalesced along hw) and
// writes its whole padded pixel with 16-byte stores.
template <int OUT>  // 0 f32, 1 f16, 2 s8, 3 u8
__global__ void nchw_to_nhwc_smallc_kernel(const float* __restrict__ in, void* __restrict__ out, int n, int c,
                                           int hw, int c_pad, float inv_scale) {
    const long long total = 1ll * n * hw;
    for (long long idx = blockIdx.x * 1ll * blockDim.x + threadIdx.x; idx < total;
         idx += 1ll * gridDim.x * blockDim.x) {
        const int b = static_cast<int>(idx / hw);
        const int px = static_cast<int>(idx - 1ll * b * hw);
        float x[4] = {0.f, 0.f, 0.f, 0.f};
        for (int ch = 0; ch < c; ++ch) x[ch] = __ldg(in + (1ll * b * c + ch) * hw + px);
        if (OUT == 0) {
            float4* o = reinterpret_cast<float4*>(static_cast<float*>(out) + idx * c_pad);
            o[0] = make_float4(x[0], x[1], x[2], x[3]);
            for (int q = 1; q < c_pad / 4; ++q) o[q] = make_float4(0.f, 0.f, 0.f, 0.f);
        } else if (OUT == 1) {
            uint4* o = reinterpret_cast<uint4*>(static_cast<__half*>(out) + idx * c_pad);
            __half2 a = __floats2half2_rn(x[0], x[1]), bq = __floats2half2_rn(x[2], x[3]);
            o[0] = make_uint4(*reinterpret_cast<uint32_t*>(&a), *reinterpret_cast<uint32_t*>(&bq), 0, 0);
            for (int q = 1; q < c_pad / 8; ++q) o[q] = make_uint4(0, 0, 0, 0);
        } else {
            uint32_t w = 0;
            for (int ch = 0; ch < 4; ++ch) {
                float t = __fmul_rn(x[ch], inv_scale);
                int code;
                if (OUT == 2) { t = fminf(fmaxf(roundf(t), -128.f), 127.f); code = static_cast<int>(t); }
                else { t = fminf(fmaxf(t, 0.f), 255.f); code = static_cast<int>(t); }
                w |= (static_cast<uint32_t>(code) & 0xffu) << (8 * ch);
            }
            uint4* o = reinterpret_cast<uint4*>(static_cast<uint8_t*>(out) + idx * c_pad);
            o[0] = make_uint4(w, 0, 0, 0);
            for (int q = 1; q < c_pad / 16; ++q) o[q] = make_uint4(0, 0, 0, 0);
        }
    }
}

// Stem pack: the first conv of a CNN has C <= 4 input channels, so an NHWC pixel is far below
// the 16-byte TMA / 32-byte MMA granules. This kernel turns the fp32 NCHW graph input into
//   X2[n][h + 2*pad_h][wo][taps][4]      (taps = filter width rounded up to 4 or 8)
// i.e. for every (padded) input row and every OUTPUT column the S horizontal taps x 4 channels the
// filter row touches, already quantised / converted. The R x S conv then runs on the tensor-core
// kernel as an R x 1 conv over X2 with c = taps*4, stride_w = 1, no padding.
// One block per (image, padded input row): the row's pixels are read (coalesced), quantised / converted ONCE
// into a shared-memory line of 4-channel pixels, then the overlapping tap windows are emitted as 16-byte
// stores that are contiguous across the block.
template <int OUT>  // 0 f32, 1 f16, 2 s8, 3 u8
__global__ void stem_pack_kernel(const float* __restrict__ in, void* __restrict__ out, int n, int c, int h,
                                 int w, int pad_h, int pad_w, int s, int stride_w, int taps, int wo,
                                 float inv_scale) {
    pdl_enter();
    constexpr int PX = OUT == 0 ? 16 : (OUT == 1 ? 8 : 4);   // bytes per 4-channel pixel
    constexpr int TP = 16 / PX;                              // taps per 16-byte store
    extern __shared__ __align__(16) uint8_t line[];          // (w + 2*pad_w + taps) pixels
    const int hp = h + 2 * pad_h;
    const int row = blockIdx.x;
    const int b = row / hp;
    const int y = row - b * hp - pad_h;
    const bool row_ok = y >= 0 && y < h;
    const int wp = w + 2 * pad_w + taps;
    for (int xp = threadIdx.x; xp < wp; xp += blockDim.x) {
        const int x = xp - pad_w;
        float v[4] = {0.f, 0.f, 0.f, 0.f};
        if (row_ok && x >= 0 && x < w)
            for (int ch = 0; ch < c; ++ch) v[ch] = __ldg(in + ((1ll * b * c + ch) * h + y) * w + x);
        if (OUT == 0) {
            reinterpret_cast<float4*>(line)[xp] = make_float4(v[0], v[1], v[2], v[3]);
        } else if (OUT == 1) {
            __half2 a = __floats2half2_rn(v[0], v[1]), bq = __floats2half2_rn(v[2], v[3]);
            reinterpret_cast<uint2*>(line)[xp] = make_uint2(*reinterpret_cast<uint32_t*>(&a), *reinterpret_cast<uint32_t*>(&bq));
        } else {
            uint32_t wd = 0;
            for (int ch = 0; ch < 4; ++ch) {
                float f = __fmul_rn(v[ch], inv_scale);
                int code;
                if (OUT == 2) { f = fminf(fmaxf(roundf(f), -128.f), 127.f); code = static_cast<int>(f); }
                else { f = fminf(fmaxf(f, 0.f), 255.f); code = static_cast<int>(f); }
                wd |= (static_cast<uint32_t>(code) & 0xffu) << (8 * ch);
            }
            reinterpret_cast<uint32_t*>(line)[xp] = wd;
        }
    }
    __syncthreads();
    const int groups = taps / TP;   // 16-byte stores per output column
    uint4* dst = reinterpret_cast<uint4*>(out) + 1ll * row * wo * groups;
    for (int i = threadIdx.x; i < wo * groups; i += blockDim.x) {
        const int q = i / groups, g = i - q * groups;
        const int tap0 = g * TP;
        const int xp0 = q * stride_w + tap0;   // x = q*stride_w - pad_w + tap  ->  xp = x + pad_w
        uint4 val;
        if (OUT == 0) {
            val = tap0 < s ? reinterpret_cast<const uint4*>(line)[xp0] : make_uint4(0, 0, 0, 0);
        } else if (OUT == 1) {
            const uint2 p0 = tap0 < s ? reinterpret_cast<const uint2*>(line)[xp0] : make_uint2(0, 0);
            const uint2 p1 = tap0 + 1 < s ? reinterpret_cast<const uint2*>(line)[xp0 + 1] : make_uint2(0, 0);
            val = make_uint4(p0.x, p0.y, p1.x, p1.y);
        } else {
            const uint32_t* l = reinterpret_cast<const uint32_t*>(line);
            val = make_uint4(tap0 < s ? l[xp0] : 0u, tap0 + 1 < s ? l[xp0 + 1] : 0u, tap0 + 2 < s ? l[xp0 + 2] : 0u,
                             tap0 + 3 < s ? l[xp0 + 3] : 0u);
        }
        dst[i] = val;
    }
}

template <int IN>  // 0 f32, 1 f16, 2 s8, 3 u8
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
            if (IN == 0) x = static_cast<const float*>(in)[i];
            else if (IN == 1) x = __half2float(static_cast<const __half*>(in)[i]);
            else if (IN == 2) x = static_cast<float>(static_cast<const int8_t*>(in)[i]);
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
//   f32 / f16 : fp32 FMA in (r, s) order, + bias, relu(neg_slope)  -- the arithmetic of dwconv_kernel
//   int8      : exact s32 accumulation (dp4a against the weight word masked to one byte = one channel's product),
//               then the x86 Saber epilogue of the conv kernels: f = (acc + bias) * scale, relu, rne + saturate
template <int MODE>   // 0 f32, 1 f16, 2 int8
__global__ void __launch_bounds__(256)
dwconv_vec_kernel(const uint4* __restrict__ in, const uint4* __restrict__ wgt, const float* __restrict__ bias,
                  const float* __restrict__ scale, uint4* __restrict__ out, int n, int h, int w, int cv, int oh, int ow,
                  int r, int s, int ph, int pw, int sh, int sw, int dh, int dw, int relu, float slope, int in_unsigned,
                  int out_dtype) {
    pdl_enter();
    constexpr int NCH = MODE == 0 ? 4 : (MODE == 1 ? 8 : 16);
    const long long total = 1ll * n * oh * ow * cv;
    for (long long idx = blockIdx.x * 1ll * blockDim.x + threadIdx.x; idx < total; idx += 1ll * gridDim.x * blockDim.x) {
        const int v = static_cast<int>(idx % cv);
        long long t = idx / cv;
        const int x0 = static_cast<int>(t % ow); t /= ow;
        const int y0 = static_cast<int>(t % oh);
        const int b = static_cast<int>(t / oh);
        float facc[MODE == 2 ? 1 : NCH];
        int iacc[MODE == 2 ? NCH : 1];
#pragma unroll
        for (int i = 0; i < (MODE == 2 ? 1 : NCH); ++i) facc[i] = 0.f;
#pragma unroll
        for (int i = 0; i < (MODE == 2 ? NCH : 1); ++i) iacc[i] = 0;
        for (int kr = 0; kr < r; ++kr) {
            const int iy = y0 * sh - ph + kr * dh;
            if (iy < 0 || iy >= h) continue;
            for (int ks = 0; ks < s; ++ks) {
                const int ix = x0 * sw - pw + ks * dw;
                if (ix < 0 || ix >= w) continue;
                const uint4 xv = __ldg(in + ((1ll * b * h + iy) * w + ix) * cv + v);
                const uint4 wv = __ldg(wgt + (1ll * kr * s + ks) * cv + v);
                const uint32_t xw[4] = {xv.x, xv.y, xv.z, xv.w}, ww[4] = {wv.x, wv.y, wv.z, wv.w};
                if constexpr (MODE == 0) {
#pragma unroll
                    for (int i = 0; i < 4; ++i) facc[i] = __fmaf_rn(__uint_as_float(xw[i]), __uint_as_float(ww[i]), facc[i]);
                } else if constexpr (MODE == 1) {
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&xw[i]));
                        const float2 c2 = __half22float2(*reinterpret_cast<const __half2*>(&ww[i]));
                        facc[2 * i] = __fmaf_rn(a.x, c2.x, facc[2 * i]);
                        facc[2 * i + 1] = __fmaf_rn(a.y, c2.y, facc[2 * i + 1]);
                    }
                } else {
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            const uint32_t wm = ww[i] & (0xFFu << (8 * j));
                            int& a = iacc[4 * i + j];
                            if (in_unsigned) asm("dp4a.u32.s32 %0, %1, %2, %0;" : "+r"(a) : "r"(xw[i]), "r"(wm));
                            else asm("dp4a.s32.s32 %0, %1, %2, %0;" : "+r"(a) : "r"(xw[i]), "r"(wm));
                        }
                    }
                }
            }
        }
        const int c0 = v * NCH;
        const long long o = ((1ll * b * oh + y0) * ow + x0) * cv + v;
        if constexpr (MODE == 2) {
            float f[16];
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                f[i] = __fmul_rn(__fadd_rn(__int2float_rn(iacc[i]), bias ? __ldg(bias + c0 + i) : 0.f),
                                 scale ? __ldg(scale + c0 + i) : 1.f);
                if (relu) f[i] = fmaxf(f[i], 0.f);
            }
            uint32_t q[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                uint32_t wd = 0;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    uint32_t code;
                    if (out_dtype == B200_UINT8) asm("cvt.rni.sat.u8.f32 %0, %1;" : "=r"(code) : "f"(f[4 * i + j]));
                    else asm("cvt.rni.sat.s8.f32 %0, %1;" : "=r"(code) : "f"(f[4 * i + j]));
                    wd |= (code & 0xffu) << (8 * j);
                }
                q[i] = wd;
            }
            out[o] = make_uint4(q[0], q[1], q[2], q[3]);
        } else {
            float y[NCH];
#pragma unroll
            for (int i = 0; i < NCH; ++i) {
                y[i] = facc[i] + (bias ? __ldg(bias + c0 + i) : 0.f);
                if (relu) y[i] = y[i] > 0.f ? y[i] : y[i] * slope;
            }
            if constexpr (MODE == 0) {
                out[o] = make_uint4(__float_as_uint(y[0]), __float_as_uint(y[1]), __float_as_uint(y[2]), __float_as_uint(y[3]));
            } else {
                uint32_t q[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const __half2 hh = __halves2half2(static_cast<__half>(y[2 * i]), static_cast<__half>(y[2 * i + 1]));
                    q[i] = *reinterpret_cast<const uint32_t*>(&hh);
                }
                out[o] = make_uint4(q[0], q[1], q[2], q[3]);
            }
        }
    }
}

// Same arithmetic, XP adjacent output pixels of one row per thread (filter width S, horizontal stride SW, dilation 1 --
// the MobileNet 3x3 layers): the (XP-1)*SW + S input columns of a filter row are loaded once and shared by the XP outputs,
// the S weight vectors of the row once per thread -- 2.2x fewer instructions and loads per output than one pixel per
// thread. Per output the taps are still accumulated in (r, s) order (a padding tap adds an exact 0), so the results are
// bit-identical to dwconv_vec_kernel.
template <int MODE, int XP, int S, int SW>
__global__ void __launch_bounds__(256)
dwconv_row_kernel(const uint4* __restrict__ in, const uint4* __restrict__ wgt, const float* __restrict__ bias,
                  const float* __restrict__ scale, uint4* __restrict__ out, int n, int h, int w, int cv, int oh, int ow,
                  int r, int ph, int pw, int sh, int dh, int relu, float slope, int in_unsigned, int out_dtype) {
    pdl_enter();
    constexpr int NCH = MODE == 0 ? 4 : (MODE == 1 ? 8 : 16);
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
        float facc[XP][MODE == 2 ? 1 : NCH];
        int iacc[XP][MODE == 2 ? NCH : 1];
#pragma unroll
        for (int p = 0; p < XP; ++p) {
#pragma unroll
            for (int i = 0; i < (MODE == 2 ? 1 : NCH); ++i) facc[p][i] = 0.f;
#pragma unroll
            for (int i = 0; i < (MODE == 2 ? NCH : 1); ++i) iacc[p][i] = 0;
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
                for (int ks = 0; ks < S; ++ks) {
                    const uint4 xq = xv[p * SW + ks], wq = wv[ks];
                    const uint32_t xw[4] = {xq.x, xq.y, xq.z, xq.w}, ww[4] = {wq.x, wq.y, wq.z, wq.w};
                    if constexpr (MODE == 0) {
#pragma unroll
                        for (int i = 0; i < 4; ++i) facc[p][i] = __fmaf_rn(__uint_as_float(xw[i]), __uint_as_float(ww[i]), facc[p][i]);
                    } else if constexpr (MODE == 1) {
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                            const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&xw[i]));
                            const float2 c2 = __half22float2(*reinterpret_cast<const __half2*>(&ww[i]));
                            facc[p][2 * i] = __fmaf_rn(a.x, c2.x, facc[p][2 * i]);
                            facc[p][2 * i + 1] = __fmaf_rn(a.y, c2.y, facc[p][2 * i + 1]);
                        }
                    } else {
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
#pragma unroll
                            for (int j = 0; j < 4; ++j) {
                                const uint32_t wm = ww[i] & (0xFFu << (8 * j));
                                int& a = iacc[p][4 * i + j];
                                if (in_unsigned) asm("dp4a.u32.s32 %0, %1, %2, %0;" : "+r"(a) : "r"(xw[i]), "r"(wm));
                                else asm("dp4a.s32.s32 %0, %1, %2, %0;" : "+r"(a) : "r"(xw[i]), "r"(wm));
                            }
                        }
                    }
                }
            }
        }
        const int c0 = v * NCH;
#pragma unroll
        for (int p = 0; p < XP; ++p) {
            if (x0 + p >= ow) break;
            const long long o = ((1ll * b * oh + y0) * ow + x0 + p) * cv + v;
            if constexpr (MODE == 2) {
                uint32_t q[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    uint32_t wd = 0;
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        float f = __fmul_rn(__fadd_rn(__int2float_rn(iacc[p][4 * i + j]), bias ? __ldg(bias + c0 + 4 * i + j) : 0.f),
                                            scale ? __ldg(scale + c0 + 4 * i + j) : 1.f);
                        if (relu) f = fmaxf(f, 0.f);
                        uint32_t code;
                        if (out_dtype == B200_UINT8) asm("cvt.rni.sat.u8.f32 %0, %1;" : "=r"(code) : "f"(f));
                        else asm("cvt.rni.sat.s8.f32 %0, %1;" : "=r"(code) : "f"(f));
                        wd |= (code & 0xffu) << (8 * j);
                    }
                    q[i] = wd;
                }
                out[o] = make_uint4(q[0], q[1], q[2], q[3]);
            } else {
                float y[NCH];
#pragma unroll
                for (int i = 0; i < NCH; ++i) {
                    y[i] = facc[p][i] + (bias ? __ldg(bias + c0 + i) : 0.f);
                    if (relu) y[i] = y[i] > 0.f ? y[i] : y[i] * slope;
                }
                if constexpr (MODE == 0) {
                    out[o] = make_uint4(__float_as_uint(y[0]), __float_as_uint(y[1]), __float_as_uint(y[2]), __float_as_uint(y[3]));
                } else {
                    uint32_t q[4];
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const __half2 hh = __halves2half2(static_cast<__half>(y[2 * i]), static_cast<__half>(y[2 * i + 1]));
                        q[i] = *reinterpret_cast<const uint32_t*>(&hh);
                    }
                    out[o] = make_uint4(q[0], q[1], q[2], q[3]);
                }
            }
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
template <int MODE, int CVB>
__global__ void __launch_bounds__(256, MODE == 2 ? 2 : 3)
dwconv_tile_kernel(const uint4* __restrict__ in, const uint4* __restrict__ wgt, const float* __restrict__ bias,
                   const float* __restrict__ scale, uint4* __restrict__ out, int h, int w, int cv, int oh, int ow,
                   int ph, int pw, int relu, float slope, int in_unsigned, int out_dtype, int tiles_x, int tiles_y, int cblocks) {
    constexpr int NCH = MODE == 0 ? 4 : (MODE == 1 ? 8 : 16);
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
            float facc[XP][MODE == 2 ? 1 : NCH];
            int iacc[XP][MODE == 2 ? NCH : 1];
#pragma unroll
            for (int p = 0; p < XP; ++p) {
#pragma unroll
                for (int i = 0; i < (MODE == 2 ? 1 : NCH); ++i) facc[p][i] = 0.f;
#pragma unroll
                for (int i = 0; i < (MODE == 2 ? NCH : 1); ++i) iacc[p][i] = 0;
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
                    for (int ks = 0; ks < 3; ++ks) {
                        const uint4 xq = xv[p + ks], wq = wv[ks];
                        const uint32_t xw[4] = {xq.x, xq.y, xq.z, xq.w}, ww[4] = {wq.x, wq.y, wq.z, wq.w};
                        if constexpr (MODE == 0) {
#pragma unroll
                            for (int i = 0; i < 4; ++i) facc[p][i] = __fmaf_rn(__uint_as_float(xw[i]), __uint_as_float(ww[i]), facc[p][i]);
                        } else if constexpr (MODE == 1) {
#pragma unroll
                            for (int i = 0; i < 4; ++i) {
                                const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&xw[i]));
                                const float2 c2 = __half22float2(*reinterpret_cast<const __half2*>(&ww[i]));
                                facc[p][2 * i] = __fmaf_rn(a.x, c2.x, facc[p][2 * i]);
                                facc[p][2 * i + 1] = __fmaf_rn(a.y, c2.y, facc[p][2 * i + 1]);
                            }
                        } else {
#pragma unroll
                            for (int i = 0; i < 4; ++i) {
#pragma unroll
                                for (int j = 0; j < 4; ++j) {
                                    const uint32_t wm = ww[i] & (0xFFu << (8 * j));
                                    int& a = iacc[p][4 * i + j];
                                    if (in_unsigned) asm("dp4a.u32.s32 %0, %1, %2, %0;" : "+r"(a) : "r"(xw[i]), "r"(wm));
                                    else asm("dp4a.s32.s32 %0, %1, %2, %0;" : "+r"(a) : "r"(xw[i]), "r"(wm));
                                }
                            }
                        }
                    }
                }
            }
            // ---- epilogue (that of dwconv_vec_kernel), bias / scale as 16-byte loads
            const int c0 = vg * NCH;
            float bv[NCH], sv[MODE == 2 ? NCH : 1];
#pragma unroll
            for (int i = 0; i < NCH / 4; ++i) {
                const float4 b4 = bias ? __ldg(reinterpret_cast<const float4*>(bias + c0) + i) : make_float4(0.f, 0.f, 0.f, 0.f);
                bv[4 * i] = b4.x; bv[4 * i + 1] = b4.y; bv[4 * i + 2] = b4.z; bv[4 * i + 3] = b4.w;
                if constexpr (MODE == 2) {
                    const float4 s4 = scale ? __ldg(reinterpret_cast<const float4*>(scale + c0) + i) : make_float4(1.f, 1.f, 1.f, 1.f);
                    sv[4 * i] = s4.x; sv[4 * i + 1] = s4.y; sv[4 * i + 2] = s4.z; sv[4 * i + 3] = s4.w;
                }
            }
            uint4* orow = out + ((1ll * b * oh + oy) * ow + ox0) * cv + vg;
#pragma unroll
            for (int p = 0; p < XP; ++p) {
                if (ox0 + p >= ow) break;
                uint32_t q[4];
                if constexpr (MODE == 2) {
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        uint32_t wd = 0;
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            float f = __fmul_rn(__fadd_rn(__int2float_rn(iacc[p][4 * i + j]), bv[4 * i + j]), sv[4 * i + j]);
                            if (relu) f = fmaxf(f, 0.f);
                            uint32_t code;
                            if (out_dtype == B200_UINT8) asm("cvt.rni.sat.u8.f32 %0, %1;" : "=r"(code) : "f"(f));
                            else asm("cvt.rni.sat.s8.f32 %0, %1;" : "=r"(code) : "f"(f));
                            wd |= (code & 0xffu) << (8 * j);
                        }
                        q[i] = wd;
                    }
                } else {
                    float yv[NCH];
#pragma unroll
                    for (int i = 0; i < NCH; ++i) {
                        yv[i] = facc[p][i] + bv[i];
                        if (relu) yv[i] = yv[i] > 0.f ? yv[i] : yv[i] * slope;
                    }
                    if constexpr (MODE == 0) {
#pragma unroll
                        for (int i = 0; i < 4; ++i) q[i] = __float_as_uint(yv[i]);
                    } else {
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                            const __half2 hh = __halves2half2(static_cast<__half>(yv[2 * i]), static_cast<__half>(yv[2 * i + 1]));
                            q[i] = *reinterpret_cast<const uint32_t*>(&hh);
                        }
                    }
                }
                orow[1ll * p * cv] = make_uint4(q[0], q[1], q[2], q[3]);
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
        if (d->stride_h <= 0 || d->stride_w <= 0 || d->window_h <= 0 || d->window_w <= 0)
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
    const bool big_window = p.wh * p.ww >= 16;
    if (d->dtype == B200_FLOAT) {
        if (d->c % 4) return B200_INVALID_VALUE;
        const long long total = 1ll * p.n * oh * ow * (d->c / 4);
        if (big_window)
            launch_pdl(pool_warp_kernel<0>, grid_for(total * 32, block), block, S(stream),
                       static_cast<const uint4*>(in), static_cast<uint4*>(out), p);
        else
            launch_pdl(pool_f32_kernel, grid_for(total, block), block, S(stream),
                       static_cast<const float4*>(in), static_cast<float4*>(out), p);
    } else if (d->dtype == B200_HALF) {
        if (d->c % 8) return B200_INVALID_VALUE;
        const long long total = 1ll * p.n * oh * ow * (d->c / 8);
        if (big_window)
            launch_pdl(pool_warp_kernel<1>, grid_for(total * 32, block), block, S(stream),
                       static_cast<const uint4*>(in), static_cast<uint4*>(out), p);
        else
            launch_pdl(pool_f16_kernel, grid_for(total, block), block, S(stream),
                       static_cast<const uint4*>(in), static_cast<uint4*>(out), p);
    } else if (d->dtype == B200_INT8 || d->dtype == B200_UINT8) {
        if (d->c % 16) return B200_INVALID_VALUE;
        const long long total = 1ll * p.n * oh * ow * (d->c / 16);
        if (p.wh * p.ww <= 256) {
            // grid covers (outputs x LANES) threads, rounded so that LANES-groups never straddle the loop bound
            if (big_window) {
                const unsigned g = grid_for(total * 8, block);
                if (d->dtype == B200_UINT8) launch_pdl(pool_q8_simd_kernel<true, 8>, g, block, S(stream), static_cast<const uint4*>(in), static_cast<uint4*>(out), p);
                else launch_pdl(pool_q8_simd_kernel<false, 8>, g, block, S(stream), static_cast<const uint4*>(in), static_cast<uint4*>(out), p);
            } else {
                const unsigned g = grid_for(total, block);
                if (d->dtype == B200_UINT8) launch_pdl(pool_q8_simd_kernel<true, 1>, g, block, S(stream), static_cast<const uint4*>(in), static_cast<uint4*>(out), p);
                else launch_pdl(pool_q8_simd_kernel<false, 1>, g, block, S(stream), static_cast<const uint4*>(in), static_cast<uint4*>(out), p);
            }
        } else if (big_window) {
            if (d->dtype == B200_UINT8)
                launch_pdl(pool_warp_kernel<3>, grid_for(total * 32, block), block, S(stream),
                           static_cast<const uint4*>(in), static_cast<uint4*>(out), p);
            else
                launch_pdl(pool_warp_kernel<2>, grid_for(total * 32, block), block, S(stream),
                           static_cast<const uint4*>(in), static_cast<uint4*>(out), p);
        } else if (d->dtype == B200_UINT8) {
            launch_pdl(pool_q8_kernel<true>, grid_for(total, block), block, S(stream),
                       static_cast<const uint4*>(in), static_cast<uint4*>(out), p);
        } else {
            launch_pdl(pool_q8_kernel<false>, grid_for(total, block), block, S(stream),
                       static_cast<const uint4*>(in), static_cast<uint4*>(out), p);
        }
    } else {
        return B200_UNIMPL_ERROR;
    }
    return check_launch("pool");
}

int b200_softmax_rows(const float* in, float* out, int32_t rows, int32_t len, int32_t in_pitch,
                      int32_t out_pitch, void* stream) {
    if (!in || !out || rows <= 0 || len <= 0 || in_pitch < len || out_pitch < len) return B200_INVALID_VALUE;
    if (!device_is_sm90()) return B200_WRONG_DEVICE;
    launch_pdl(softmax_rows_kernel, static_cast<unsigned>(rows), SOFTMAX_THREADS, S(stream), in, out, rows, len, in_pitch,
               out_pitch);
    return check_launch("softmax");
}

int b200_softmax_run(const float* in, float* out, int32_t outer, int32_t axis_size, int32_t inner,
                     void* stream) {
    if (!in || !out || outer <= 0 || axis_size <= 0 || inner <= 0) return B200_INVALID_VALUE;
    if (!device_is_sm90()) return B200_WRONG_DEVICE;
    if (inner == 1) {
        return b200_softmax_rows(in, out, outer, axis_size, axis_size, axis_size, stream);
    } else {
        const int block = 128;
        softmax_strided_kernel<<<(outer * inner + block - 1) / block, block, 0, S(stream)>>>(
            in, out, outer, axis_size, inner);
    }
    return check_launch("softmax");
}

int b200_eltwise_run(int32_t dtype_a, int32_t dtype_b, int32_t dtype_out, int32_t op, const void* a,
                     const void* b, void* out, size_t count, float c0, float c1, int32_t relu,
                     void* stream) {
    if (!a || !b || !out || count == 0) return B200_INVALID_VALUE;
    if (!device_is_sm90()) return B200_WRONG_DEVICE;
    if (op < B200_ELT_PROD || op > B200_ELT_MAX) return B200_UNIMPL_ERROR;
    const int block = 256;
    if (dtype_a == B200_FLOAT && dtype_b == B200_FLOAT && dtype_out == B200_FLOAT) {
        eltwise_f32_kernel<<<grid_for((count + 3) / 4, block), block, 0, S(stream)>>>(
            static_cast<const float*>(a), static_cast<const float*>(b), static_cast<float*>(out), count,
            op, c0, c1, relu);
    } else if (dtype_a == B200_HALF && dtype_b == B200_HALF && dtype_out == B200_HALF) {
        eltwise_f16_kernel<<<grid_for(count, block), block, 0, S(stream)>>>(
            static_cast<const __half*>(a), static_cast<const __half*>(b), static_cast<__half*>(out),
            count, op, c0, c1, relu);
    } else {
        auto q8 = [](int dt) { return dt == B200_INT8 || dt == B200_UINT8; };
        if (!q8(dtype_a) || !q8(dtype_b) || !q8(dtype_out) || op != B200_ELT_SUM) return B200_UNIMPL_ERROR;
        eltwise_q8_kernel<<<grid_for((count + 15) / 16, block), block, 0, S(stream)>>>(
            static_cast<const uint8_t*>(a), dtype_a == B200_UINT8, static_cast<const uint8_t*>(b),
            dtype_b == B200_UINT8, static_cast<uint8_t*>(out), dtype_out == B200_UINT8, count, c0, c1,
            relu);
    }
    return check_launch("eltwise");
}

int b200_activation_run(int32_t dtype, int32_t act, const void* in, void* out, size_t count,
                        float neg_slope, float coef, void* stream) {
    if (!in || !out || count == 0) return B200_INVALID_VALUE;
    if (!device_is_sm90()) return B200_WRONG_DEVICE;
    const int block = 256;
    if (dtype == B200_FLOAT)
        activation_f32_kernel<<<grid_for((count + 3) / 4, block), block, 0, S(stream)>>>(
            static_cast<const float*>(in), static_cast<float*>(out), count, act, neg_slope, coef);
    else if (dtype == B200_HALF)
        activation_f16_kernel<<<grid_for(count, block), block, 0, S(stream)>>>(
            static_cast<const __half*>(in), static_cast<__half*>(out), count, act, neg_slope, coef);
    else
        return B200_UNIMPL_ERROR;
    return check_launch("activation");
}

int b200_scale_run(int32_t dtype, const void* in, void* out, size_t pixels, int32_t c, const float* w,
                   const float* b, void* stream) {
    if (!in || !out || !w || pixels == 0 || c <= 0) return B200_INVALID_VALUE;
    if (!device_is_sm90()) return B200_WRONG_DEVICE;
    const int block = 256;
    if (dtype == B200_FLOAT)
        scale_f32_kernel<<<grid_for(pixels * c, block), block, 0, S(stream)>>>(
            static_cast<const float*>(in), static_cast<float*>(out), pixels, c, w, b);
    else if (dtype == B200_HALF)
        scale_f16_kernel<<<grid_for(pixels * c, block), block, 0, S(stream)>>>(
            static_cast<const __half*>(in), static_cast<__half*>(out), pixels, c, w, b);
    else
        return B200_UNIMPL_ERROR;
    return check_launch("scale");
}

int b200_nchw_to_nhwc(const float* in, void* out, int32_t out_dtype, int32_t n, int32_t c, int32_t h,
                      int32_t w, int32_t c_pad, float inv_scale, int32_t split_hi_lo, void* stream) {
    if (!in || !out || n <= 0 || c <= 0 || h <= 0 || w <= 0 || c_pad < c) return B200_INVALID_VALUE;
    if (split_hi_lo) return B200_UNIMPL_ERROR;
    if (!device_is_sm90()) return B200_WRONG_DEVICE;
    const int hw = h * w;
    const int es = out_dtype == B200_FLOAT ? 4 : (out_dtype == B200_HALF ? 2 : 1);
    if (c <= 4 && (c_pad * es) % 16 == 0 && (out_dtype == B200_FLOAT || out_dtype == B200_HALF ||
                                             out_dtype == B200_INT8 || out_dtype == B200_UINT8)) {
        const long long total = 1ll * n * hw;
        const unsigned g = grid_for(total, 256);
        switch (out_dtype) {
            case B200_FLOAT: nchw_to_nhwc_smallc_kernel<0><<<g, 256, 0, S(stream)>>>(in, out, n, c, hw, c_pad, inv_scale); break;
            case B200_HALF: nchw_to_nhwc_smallc_kernel<1><<<g, 256, 0, S(stream)>>>(in, out, n, c, hw, c_pad, inv_scale); break;
            case B200_INT8: nchw_to_nhwc_smallc_kernel<2><<<g, 256, 0, S(stream)>>>(in, out, n, c, hw, c_pad, inv_scale); break;
            default: nchw_to_nhwc_smallc_kernel<3><<<g, 256, 0, S(stream)>>>(in, out, n, c, hw, c_pad, inv_scale); break;
        }
        return check_launch("nchw_to_nhwc");
    }
    dim3 grid((hw + 31) / 32, (c_pad + 31) / 32, n), block(32, 8);
    switch (out_dtype) {
        case B200_FLOAT: nchw_to_nhwc_kernel<0><<<grid, block, 0, S(stream)>>>(in, out, c, hw, c_pad, inv_scale); break;
        case B200_HALF: nchw_to_nhwc_kernel<1><<<grid, block, 0, S(stream)>>>(in, out, c, hw, c_pad, inv_scale); break;
        case B200_INT8: nchw_to_nhwc_kernel<2><<<grid, block, 0, S(stream)>>>(in, out, c, hw, c_pad, inv_scale); break;
        case B200_UINT8: nchw_to_nhwc_kernel<3><<<grid, block, 0, S(stream)>>>(in, out, c, hw, c_pad, inv_scale); break;
        default: return B200_UNIMPL_ERROR;
    }
    return check_launch("nchw_to_nhwc");
}

int b200_stem_pack(const float* in, void* out, int32_t out_dtype, int32_t n, int32_t c, int32_t h, int32_t w,
                   int32_t pad_h, int32_t pad_w, int32_t s, int32_t stride_w, int32_t taps, float inv_scale,
                   void* stream) {
    if (!in || !out || n <= 0 || c <= 0 || c > 4 || h <= 0 || w <= 0 || s <= 0 || s > taps || stride_w <= 0 ||
        (taps != 4 && taps != 8) || pad_h < 0 || pad_w < 0)
        return B200_INVALID_VALUE;
    if (!device_is_sm90()) return B200_WRONG_DEVICE;
    const int wo = (w + 2 * pad_w - s) / stride_w + 1;
    if (wo <= 0) return B200_INVALID_VALUE;
    const unsigned g = static_cast<unsigned>(n * (h + 2 * pad_h));
    const int px = out_dtype == B200_FLOAT ? 16 : (out_dtype == B200_HALF ? 8 : 4);
    const size_t smem = static_cast<size_t>(w + 2 * pad_w + taps) * px;
    if (smem > 48 * 1024) return B200_UNIMPL_ERROR;
    switch (out_dtype) {
        case B200_FLOAT: launch_pdl_smem(stem_pack_kernel<0>, g, 128, smem, S(stream), in, out, n, c, h, w, pad_h, pad_w, s, stride_w, taps, wo, inv_scale); break;
        case B200_HALF: launch_pdl_smem(stem_pack_kernel<1>, g, 128, smem, S(stream), in, out, n, c, h, w, pad_h, pad_w, s, stride_w, taps, wo, inv_scale); break;
        case B200_INT8: launch_pdl_smem(stem_pack_kernel<2>, g, 128, smem, S(stream), in, out, n, c, h, w, pad_h, pad_w, s, stride_w, taps, wo, inv_scale); break;
        case B200_UINT8: launch_pdl_smem(stem_pack_kernel<3>, g, 128, smem, S(stream), in, out, n, c, h, w, pad_h, pad_w, s, stride_w, taps, wo, inv_scale); break;
        default: return B200_UNIMPL_ERROR;
    }
    return check_launch("stem_pack");
}

int b200_nhwc_to_nchw(const void* in, int32_t in_dtype, float* out, int32_t n, int32_t c, int32_t h,
                      int32_t w, int32_t c_pad, float scale, void* stream) {
    if (!in || !out || n <= 0 || c <= 0 || h <= 0 || w <= 0 || c_pad < c) return B200_INVALID_VALUE;
    if (!device_is_sm90()) return B200_WRONG_DEVICE;
    const int hw = h * w;
    dim3 grid((hw + 31) / 32, (c + 31) / 32, n), block(32, 8);
    switch (in_dtype) {
        case B200_FLOAT: nhwc_to_nchw_kernel<0><<<grid, block, 0, S(stream)>>>(in, out, c, hw, c_pad, scale); break;
        case B200_HALF: nhwc_to_nchw_kernel<1><<<grid, block, 0, S(stream)>>>(in, out, c, hw, c_pad, scale); break;
        case B200_INT8: nhwc_to_nchw_kernel<2><<<grid, block, 0, S(stream)>>>(in, out, c, hw, c_pad, scale); break;
        case B200_UINT8: nhwc_to_nchw_kernel<3><<<grid, block, 0, S(stream)>>>(in, out, c, hw, c_pad, scale); break;
        default: return B200_UNIMPL_ERROR;
    }
    return check_launch("nhwc_to_nchw");
}

int b200_dwconv_run(const b200_conv_desc_t* d, const void* in, const void* weights_rsc,
                    const float* bias, const float* scale, void* out, void* stream) {
    if (!d || !in || !weights_rsc || !out) return B200_INVALID_VALUE;
    if (!device_is_sm90()) return B200_WRONG_DEVICE;
    if (d->k != d->c) return B200_INVALID_VALUE;
    const int oh = (d->h + 2 * d->pad_h - (d->dil_h * (d->r - 1) + 1)) / d->stride_h + 1;
    const int ow = (d->w + 2 * d->pad_w - (d->dil_w * (d->s - 1) + 1)) / d->stride_w + 1;
    if (oh <= 0 || ow <= 0) return B200_INVALID_VALUE;
    const int block = 256;
    const uint4* in4 = static_cast<const uint4*>(in);
    const uint4* w4 = static_cast<const uint4*>(weights_rsc);
    uint4* out4 = static_cast<uint4*>(out);
    int mode, nch;
    if (d->in_dtype == B200_FLOAT && d->out_dtype == B200_FLOAT) { mode = 0; nch = 4; }
    else if (d->in_dtype == B200_HALF && d->out_dtype == B200_HALF) { mode = 1; nch = 8; }
    else if ((d->in_dtype == B200_INT8 || d->in_dtype == B200_UINT8) && (d->out_dtype == B200_INT8 || d->out_dtype == B200_UINT8)) { mode = 2; nch = 16; }
    else return B200_UNIMPL_ERROR;
    if (d->c % nch) return B200_INVALID_VALUE;
    const int cv = d->c / nch;
    // big 3x3 / stride-1 layers: the shared-memory tiled kernel. B200_SABER_DW_TILE: 0 never, 2 whenever the shape fits
    // (default: feature maps of at least 28 x 28, below that the tile would be mostly halo and idle lanes)
    static const int tile_mode = [] { const char* e = getenv("B200_SABER_DW_TILE"); return e ? atoi(e) : 1; }();
    const int cvb = cv % 8 == 0 ? 8 : (cv == 4 ? 4 : (cv == 2 ? 2 : 0));
    if (tile_mode > 0 && cvb && d->r == 3 && d->s == 3 && d->stride_h == 1 && d->stride_w == 1 && d->dil_h == 1 && d->dil_w == 1 &&
        d->pad_h <= 1 && d->pad_w <= 1) {
        const int tw = 128 / cvb;
        const int tiles_x = (ow + tw - 1) / tw, tiles_y = (oh + 7) / 8, cblocks = cv / cvb;
        const double util = static_cast<double>(oh) * ow / (static_cast<double>(tiles_y) * 8 * tiles_x * tw);
        const long long blocks = 1ll * d->n * tiles_y * tiles_x * cblocks;
        // INT8 (its row kernel keeps only 2 outputs per thread): from 7 x 7 up (MobileNet-v1 INT8 b16 in-net 12.97 -> 7.32 us
        // per 14 x 14 layer); float kinds: from 28 x 28 (at 14 x 14 the row kernel is 0.4 us faster per layer)
        const bool take = tile_mode >= 2 ? util >= 0.5 : (mode == 2 ? util >= 0.35 : (util >= 0.6 && oh * ow >= 28 * 28));
        if (blocks < (1ll << 31) && take) {
            const unsigned g = static_cast<unsigned>(blocks);
#define B200_DWT_ARGS in4, w4, bias, scale, out4, d->h, d->w, cv, oh, ow, d->pad_h, d->pad_w, d->relu, d->neg_slope, \
                      d->in_dtype == B200_UINT8 ? 1 : 0, d->out_dtype, tiles_x, tiles_y, cblocks
#define B200_DWT_LAUNCH(M)                                                                              \
            do {                                                                                        \
                if (cvb == 8) launch_pdl(dwconv_tile_kernel<M, 8>, g, block, S(stream), B200_DWT_ARGS); \
                else if (cvb == 4) launch_pdl(dwconv_tile_kernel<M, 4>, g, block, S(stream), B200_DWT_ARGS); \
                else launch_pdl(dwconv_tile_kernel<M, 2>, g, block, S(stream), B200_DWT_ARGS);          \
            } while (0)
            if (mode == 0) B200_DWT_LAUNCH(0);
            else if (mode == 1) B200_DWT_LAUNCH(1);
            else B200_DWT_LAUNCH(2);
#undef B200_DWT_LAUNCH
#undef B200_DWT_ARGS
            return check_launch("dwconv");
        }
    }
    if (d->s == 3 && d->dil_w == 1 && (d->stride_w == 1 || d->stride_w == 2)) {
        // 3-wide filters: several adjacent outputs per thread (dwconv_row_kernel)
        const int xp = mode == 2 ? 2 : 4;
        const long long items = 1ll * d->n * oh * ((ow + xp - 1) / xp) * cv;
        const unsigned g = grid_for(items, block);
#define B200_DWR_ARGS in4, w4, bias, scale, out4, d->n, d->h, d->w, cv, oh, ow, d->r, d->pad_h, d->pad_w, d->stride_h, d->dil_h, \
                      d->relu, d->neg_slope, d->in_dtype == B200_UINT8 ? 1 : 0, d->out_dtype
        if (d->stride_w == 1) {
            if (mode == 0) launch_pdl(dwconv_row_kernel<0, 4, 3, 1>, g, block, S(stream), B200_DWR_ARGS);
            else if (mode == 1) launch_pdl(dwconv_row_kernel<1, 4, 3, 1>, g, block, S(stream), B200_DWR_ARGS);
            else launch_pdl(dwconv_row_kernel<2, 2, 3, 1>, g, block, S(stream), B200_DWR_ARGS);
        } else {
            if (mode == 0) launch_pdl(dwconv_row_kernel<0, 4, 3, 2>, g, block, S(stream), B200_DWR_ARGS);
            else if (mode == 1) launch_pdl(dwconv_row_kernel<1, 4, 3, 2>, g, block, S(stream), B200_DWR_ARGS);
            else launch_pdl(dwconv_row_kernel<2, 2, 3, 2>, g, block, S(stream), B200_DWR_ARGS);
        }
#undef B200_DWR_ARGS
        return check_launch("dwconv");
    }
    const long long total = 1ll * d->n * oh * ow * cv;
    const unsigned grid = grid_for(total, block);
#define B200_DW_ARGS in4, w4, bias, scale, out4, d->n, d->h, d->w, cv, oh, ow, d->r, d->s, d->pad_h, d->pad_w, d->stride_h, \
                     d->stride_w, d->dil_h, d->dil_w, d->relu, d->neg_slope, d->in_dtype == B200_UINT8 ? 1 : 0, d->out_dtype
    if (mode == 0) launch_pdl(dwconv_vec_kernel<0>, grid, block, S(stream), B200_DW_ARGS);
    else if (mode == 1) launch_pdl(dwconv_vec_kernel<1>, grid, block, S(stream), B200_DW_ARGS);
    else launch_pdl(dwconv_vec_kernel<2>, grid, block, S(stream), B200_DW_ARGS);
#undef B200_DW_ARGS
    return check_launch("dwconv");
}

}  // extern "C"
