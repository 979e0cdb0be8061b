// Stem convolution: the first conv of a CNN (C <= 4 input channels, fp32 NCHW graph input) with its activation and
// -- optionally -- the max pooling that follows it, in ONE launch on Hopper tensor cores (wgmma, sm_90a).
//
// Replaces, for the graph-input layer, the reference's fused conv + pooling path
//   SaberConv2DPooling<NV,*>::{create,dispatch}             saber/funcs/impl/cuda/saber_conv_pooling.cpp:36-130
//   winograd_conv_relu_pooling / direct_conv_bias_relu_maxpool2k2s0p_*   third-party/sass/include/sass_funcs.h:54-427
//   the input quantisation inside conv (conv_calibrate_fp32_int8_c4)     saber/funcs/impl/cuda/saber_conv.cpp:341-381
// and this library's own three-launch sequence stem_pack -> conv plan -> pool (a 6.6 MB packed tensor and a 6.4 MB
// conv output written and re-read at ResNet-50 batch 8).
//
// A CTA owns a ch x cw rectangle of ONE image's conv output (ch*cw <= 128 GEMM rows; with pooling fused the
// rectangle is exactly what a ph x pw tile of pooled pixels needs, halo included):
//   1. the fp32 input patch is read once (coalesced along w), quantised / converted (x86 Saber rule: roundf + clamp)
//      into a shared-memory line buffer of 4-channel pixels;
//   2. the A operand is built in shared memory, one "plane" per input-row parity (stride_h planes): row (k, j) of a
//      plane holds the 8 horizontal taps x 4 channels that output column j reads from input row k*stride_h + par --
//      a 32/64/128-byte K-major row written with the SWIZZLE_32/64/128B pattern the tensor core expects. Filter row
//      r = a*stride_h + par is then ONE MMA (K = 32 bytes per slice) whose A descriptor starts a*cw rows into plane
//      par: the swizzle is a function of the absolute address, so a row-shifted view of the plane is a valid operand
//      (as in conv_slab.cu);
//   3. R (x row slices) wgmma accumulate the 128 x BN tile in the registers of the CTA's warpgroup (two 64-row halves);
//   4. the fused epilogue of the other conv kernels (bias, per-channel scale, relu, requantise; conv_common.cuh) stages
//      the tile in shared memory, and the CTA max-pools it there (packed byte / half2 / float max) and writes only the
//      pooled pixels, 16 bytes per thread, NHWC.
// Results are bit-identical to conv plan -> pool: same accumulation (exact for int8), same epilogue code, and max
// commutes with the monotone requantisation (it is applied to the already requantised bytes anyway).
#include <cuda_fp16.h>
#include <stdio.h>
#include <string.h>

#include <atomic>

#include "conv_common.cuh"

namespace b200 {

constexpr int STEM_THREADS = 128;   // one warpgroup: issues the MMAs of both 64-row halves, then runs the epilogue
constexpr int STEM_TAPS = 8;

// n / d for small non-negative n by one multiply-high (m = ceil(2^32 / d); exact for n * d < 2^32)
struct FastDiv {
    uint32_t m, d;
    __host__ void set(uint32_t div) { d = div; m = div <= 1 ? 0u : static_cast<uint32_t>(0xFFFFFFFFu / div) + 1u; }
    __device__ __forceinline__ uint32_t quot(uint32_t n) const { return d <= 1 ? n : __umulhi(n, m); }
};

struct StemParams {
    const float* in;      // [n][c][h][w] fp32
    const uint8_t* w;     // packed [k][R][ROWB] (X3: the low image follows the high image)
    void* out;            // NHWC [n][OH][OW][ldc]
    int32_t n, c, h, w_in;
    int32_t k, ldc;
    int32_t R, stride_h, stride_w, pad_h, pad_w;
    int32_t Ho, Wo;       // conv output
    int32_t OH, OW;       // what is stored: the pooled size when pooling is fused, else Ho x Wo
    int32_t ch, cw;       // conv rectangle of a CTA
    int32_t pool;         // 0 none, 1 max
    int32_t pk_h, pk_w, ps_h, ps_w, pp_h, pp_w;
    int32_t ph, pw;       // pooled tile of a CTA
    int32_t tiles_h, tiles_w;
    int32_t bn;           // output channels per CTA (16 | 32 | 64)
    int32_t qrows, qcols; // line buffer extent (input rows / columns of the patch)
    int32_t krows;        // rows (k) per plane that carry data = ch + (R-1)/stride_h
    int32_t plane_bytes, wt_stride;
    int32_t off_planes, off_stage, off_tail;
    int32_t tiles_img, tiles_total;      // tiles per image, tiles in all (walked by gridDim.x persistent CTAs)
    int32_t cpp, store_tw, store_items;  // store phase: 16-byte chunks per pixel, tile width, items per tile
    int32_t pairs_row;                   // stride_w == 2: pixel pairs per patch row
    int32_t pool_on_acc;                 // pool the raw accumulators, epilogue on the pooled pixels only (monotone epilogue)
    int32_t groups, pool_items, off_pool_stage;   // 16-channel groups per tile, (pooled pixel, group) items, their staging rows
    FastDiv div_bn, div_tiles_img, div_tiles_w, div_qcols, div_sh, div_sw, div_cpp, div_tw, div_pairs, div_groups;
    float inv_scale;
    ConvKParams kp;       // epilogue parameters (relu, dtypes, tables)
};

template <int KIND>
struct StemElem {
    static constexpr int ES = KIND == KIND_I8 ? 1 : (KIND == KIND_F16 ? 2 : 4);
    static constexpr int PXB = 4 * ES;               // one 4-channel pixel
    static constexpr int ROWB = STEM_TAPS * PXB;     // one K-major operand row: 32 | 64 | 128 bytes
    static constexpr int LG = ES == 1 ? 5 : (ES == 2 ? 6 : 7);
    static constexpr int C16 = ROWB / 16;
};

__device__ __forceinline__ uint32_t swz16(int row, int lg) { return (row >> (7 - lg)) & ((1 << (lg - 4)) - 1); }

// One 4-channel pixel in operand precision: `hi` holds PXB bytes (1 | 2 | 4 words), `lo` the low plane of the 3xTF32 split.
template <int MK, bool X3>
__device__ __forceinline__ void stem_convert(float v0, float v1, float v2, float v3, float inv_scale, uint32_t (&hi)[4],
                                             uint32_t (&lo)[4]) {
    if constexpr (MK == KIND_I8) {
        const float v[4] = {v0, v1, v2, v3};
        uint32_t wd = 0;
#pragma unroll
        for (int cch = 0; cch < 4; ++cch) {
            // secur_cast2char(x * inv): roundf + clamp (reference x86_utils.h:318-347)
            float f = roundf(__fmul_rn(v[cch], inv_scale));
            f = fminf(fmaxf(f, -128.f), 127.f);
            wd |= (static_cast<uint32_t>(static_cast<int>(f)) & 0xffu) << (8 * cch);
        }
        hi[0] = wd;
    } else if constexpr (MK == KIND_F16) {
        __half2 a = __floats2half2_rn(v0, v1), b = __floats2half2_rn(v2, v3);
        hi[0] = *reinterpret_cast<uint32_t*>(&a); hi[1] = *reinterpret_cast<uint32_t*>(&b);
    } else {
        const uint32_t w[4] = {__float_as_uint(v0), __float_as_uint(v1), __float_as_uint(v2), __float_as_uint(v3)};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            if constexpr (X3) {   // x = hi + lo, hi = top 19 bits (exact split)
                hi[i] = w[i] & 0xFFFFE000u;
                lo[i] = __float_as_uint(__fsub_rn(__uint_as_float(w[i]), __uint_as_float(hi[i])));
            } else {
                hi[i] = w[i];
            }
        }
    }
}

// max over raw accumulators: s32 for the int8 kind, fp32 bit patterns otherwise (r >= x ? r : x)
template <int MK>
__device__ __forceinline__ uint32_t acc_max(uint32_t a, uint32_t b) {
    if constexpr (MK == KIND_I8) return static_cast<uint32_t>(max(static_cast<int32_t>(a), static_cast<int32_t>(b)));
    else return __uint_as_float(a) >= __uint_as_float(b) ? a : b;
}

template <int KIND, int BN>
__global__ void __launch_bounds__(STEM_THREADS)
conv_stem_kernel(const StemParams p, const uint32_t idesc) {
    constexpr bool X3 = (KIND == KIND_TF32X3);
    constexpr int MK = X3 ? KIND_TF32 : KIND;
    constexpr int PL = X3 ? 2 : 1;
    using E = StemElem<MK>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
    uint8_t* wt = smem;                           // [PL][R][wt_stride], loaded once per CTA
    uint8_t* planes = smem + p.off_planes;        // [stride_h][PL][plane_bytes]
    uint8_t* stage = smem + p.off_stage;          // epilogue staging tile [128][bn * out_es]
    float* bias_s = reinterpret_cast<float*>(smem + p.off_tail);
    float* scale_s = bias_s + 64;

    const int tid = threadIdx.x;
    const int warp_idx = tid >> 5;
    const int lane = tid & 31;
    const int n0 = blockIdx.y * p.bn;

    // ---- weights (independent of the previous kernel), once per CTA: packed [k][R][ROWB] -> R swizzled [bn][ROWB] tiles
    // as asynchronous 16-byte copies that land while the first input patch is read and converted
    {
        const int per_plane = p.R * p.bn * E::C16;
        for (int i = tid; i < PL * per_plane; i += STEM_THREADS) {
            const int pl = i >= per_plane ? 1 : 0;
            uint32_t e = i - pl * per_plane;
            const uint32_t c16 = e % E::C16; e /= E::C16;      // compile-time divisor
            const uint32_t r = p.div_bn.quot(e), oc = e - r * p.bn;
            const uint32_t dst = smem_u32(wt + (pl * p.R + r) * p.wt_stride + oc * E::ROWB + ((c16 ^ swz16(oc, E::LG)) << 4));
            if (n0 + static_cast<int>(oc) < p.k) {
                const uint8_t* src = p.w + (static_cast<size_t>(pl) * p.k + n0 + oc) * p.R * E::ROWB +
                                     static_cast<size_t>(r) * E::ROWB + c16 * 16;
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
            } else {
                sts128(dst, make_uint4(0, 0, 0, 0));
            }
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
        for (int i = tid; i < p.bn; i += STEM_THREADS) {
            const bool ok = n0 + i < p.k;
            bias_s[i] = (p.kp.bias != nullptr && ok) ? __ldg(p.kp.bias + n0 + i) : 0.f;
            scale_s[i] = (p.kp.scale != nullptr && ok) ? __ldg(p.kp.scale + n0 + i) : 1.f;
        }
    }
    pdl_launch_dependents();
    pdl_wait_prior_grid();

    auto lg2 = [](int pw) { return pw == 128 ? 7 : (pw == 64 ? 6 : (pw == 32 ? 5 : 4)); };
    const int lg_out = lg2(p.kp.out_pw);
    const uint32_t stage_sa = smem_u32(stage);
    const uint32_t planes_sa = smem_u32(planes);
    const size_t plane = static_cast<size_t>(p.h) * p.w_in;
    const int npx = p.qrows * p.qcols;
    bool first_tile = true;
    uint32_t acc[2][BN / 2];   // GEMM rows [0, 64) and [64, 128)

    // ---- persistent walk over the CTA's tiles (tile = one ch x cw conv rectangle of one image)
    for (int tile = blockIdx.x; tile < p.tiles_total; tile += gridDim.x) {
        const uint32_t n_img = p.div_tiles_img.quot(tile);
        const uint32_t t_in = tile - n_img * p.tiles_img;
        const uint32_t ti = p.div_tiles_w.quot(t_in), tj = t_in - ti * p.tiles_w;
        // conv-output origin of the rectangle (negative rows / columns exist with a padded pooling window: they are
        // computed from zero input and never read)
        const int i0 = p.pool ? static_cast<int>(ti) * p.ph * p.ps_h - p.pp_h : static_cast<int>(ti) * p.ch;
        const int j0 = p.pool ? static_cast<int>(tj) * p.pw * p.ps_w - p.pp_w : static_cast<int>(tj) * p.cw;

        // ---- 1. input patch -> operand planes. Pixel (qr, qc) of the patch is input (h0 + qr, w0 + qc); quantised /
        // converted once, it is stored at every (output column j, tap t) with j * stride_w + t == qc of row
        // k = qr / stride_h of plane qr % stride_h of the swizzled K-major operand.
        {
            const int h0 = i0 * p.stride_h - p.pad_h, w0 = j0 * p.stride_w - p.pad_w;
            const float* img = p.in + static_cast<size_t>(n_img) * p.c * plane;
            if (p.stride_w == 2) {
                // stride 2: the pixel PAIR (qc, qc + 1), qc even, is taps (2u, 2u + 1) of output column qc/2 - u: one
                // 8 / 16 / 32-byte store per column instead of two half-sized ones
                constexpr int NB = 3;    // pairs in flight per thread: all their loads are issued before the first use
                const int npair = p.qrows * p.pairs_row;
                for (int base = tid; base < npair; base += NB * STEM_THREADS) {
                    float va[NB][4], vb[NB][4];
#pragma unroll
                    for (int u = 0; u < NB; ++u) {
                        const int i = base + u * STEM_THREADS;
                        const uint32_t qr = p.div_pairs.quot(i), pi = i - qr * p.pairs_row;
                        const int y = h0 + static_cast<int>(qr), x = w0 + 2 * static_cast<int>(pi);
                        const bool oky = i < npair && y >= 0 && y < p.h;
                        const bool ok0 = oky && x >= 0 && x < p.w_in, ok1 = oky && x + 1 >= 0 && x + 1 < p.w_in;
                        const float* px = img + static_cast<size_t>(oky ? y : 0) * p.w_in + x;
#pragma unroll
                        for (int cch = 0; cch < 4; ++cch) {
                            va[u][cch] = (ok0 && cch < p.c) ? __ldg(px + cch * plane) : 0.f;
                            vb[u][cch] = (ok1 && cch < p.c) ? __ldg(px + cch * plane + 1) : 0.f;
                        }
                    }
#pragma unroll
                    for (int u = 0; u < NB; ++u) {
                        const int i = base + u * STEM_THREADS;
                        if (i >= npair) break;
                        const uint32_t qr = p.div_pairs.quot(i), pi = i - qr * p.pairs_row;
                        const uint32_t k = p.div_sh.quot(qr), par = qr - k * p.stride_h;
                        uint32_t ha[4], la[4], hb[4], lb[4];
                        stem_convert<MK, X3>(va[u][0], va[u][1], va[u][2], va[u][3], p.inv_scale, ha, la);
                        stem_convert<MK, X3>(vb[u][0], vb[u][1], vb[u][2], vb[u][3], p.inv_scale, hb, lb);
                        const uint32_t plane_sa = planes_sa + par * PL * p.plane_bytes;
#pragma unroll
                        for (int q = 0; q < STEM_TAPS / 2; ++q) {
                            const int jj = static_cast<int>(pi) - q;
                            if (jj < 0 || jj >= p.cw) continue;
                            const uint32_t row = k * p.cw + jj;
                            const uint32_t boff = 2 * q * E::PXB;      // taps (2q, 2q + 1)
                            const uint32_t a = plane_sa + row * E::ROWB + ((((boff >> 4) ^ swz16(row, E::LG))) << 4) + (boff & 15u);
                            if constexpr (MK == KIND_I8) {
                                asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(a), "r"(ha[0]), "r"(hb[0]) : "memory");
                            } else if constexpr (MK == KIND_F16) {
                                sts128(a, make_uint4(ha[0], ha[1], hb[0], hb[1]));
                            } else {
                                // two 16-byte chunks: a pixel each (the pair straddles chunks boff/16 and boff/16 + 1)
                                const uint32_t a2 = plane_sa + row * E::ROWB + (((((boff >> 4) + 1) ^ swz16(row, E::LG))) << 4);
                                sts128(a, make_uint4(ha[0], ha[1], ha[2], ha[3]));
                                sts128(a2, make_uint4(hb[0], hb[1], hb[2], hb[3]));
                                if constexpr (X3) {
                                    sts128(a + p.plane_bytes, make_uint4(la[0], la[1], la[2], la[3]));
                                    sts128(a2 + p.plane_bytes, make_uint4(lb[0], lb[1], lb[2], lb[3]));
                                }
                            }
                        }
                    }
                }
            } else {
                constexpr int NB = 4;
                for (int base = tid; base < npx; base += NB * STEM_THREADS) {
                    float vv[NB][4];
#pragma unroll
                    for (int u = 0; u < NB; ++u) {
                        const int i = base + u * STEM_THREADS;
                        const uint32_t qr = p.div_qcols.quot(i), qc = i - qr * p.qcols;
                        const int y = h0 + static_cast<int>(qr), x = w0 + static_cast<int>(qc);
                        const bool ok = i < npx && y >= 0 && y < p.h && x >= 0 && x < p.w_in;
                        const float* px = img + static_cast<size_t>(ok ? y : 0) * p.w_in + (ok ? x : 0);
#pragma unroll
                        for (int cch = 0; cch < 4; ++cch) vv[u][cch] = (ok && cch < p.c) ? __ldg(px + cch * plane) : 0.f;
                    }
#pragma unroll
                    for (int u = 0; u < NB; ++u) {
                        const int i = base + u * STEM_THREADS;
                        if (i >= npx) break;
                        const uint32_t qr = p.div_qcols.quot(i), qc = i - qr * p.qcols;
                        const uint32_t k = p.div_sh.quot(qr), par = qr - k * p.stride_h;
                        const uint32_t j = p.div_sw.quot(qc);
                        uint32_t t = qc - j * p.stride_w;
                        uint32_t hw[4], lw[4];
                        stem_convert<MK, X3>(vv[u][0], vv[u][1], vv[u][2], vv[u][3], p.inv_scale, hw, lw);
                        const uint32_t plane_sa = planes_sa + par * PL * p.plane_bytes;
                        int jj = static_cast<int>(j);
#pragma unroll 1
                        for (; t < STEM_TAPS && jj >= 0; t += p.stride_w, --jj) {
                            if (jj >= p.cw) continue;
                            const uint32_t row = k * p.cw + jj;
                            const uint32_t boff = t * E::PXB;
                            const uint32_t a = plane_sa + row * E::ROWB + ((((boff >> 4) ^ swz16(row, E::LG))) << 4) + (boff & 15u);
                            if constexpr (MK == KIND_I8) {
                                asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(hw[0]) : "memory");
                            } else if constexpr (MK == KIND_F16) {
                                asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(a), "r"(hw[0]), "r"(hw[1]) : "memory");
                            } else {
                                sts128(a, make_uint4(hw[0], hw[1], hw[2], hw[3]));
                                if constexpr (X3) sts128(a + p.plane_bytes, make_uint4(lw[0], lw[1], lw[2], lw[3]));
                            }
                        }
                    }
                }
            }
        }
        if (first_tile) asm volatile("cp.async.wait_group 0;" ::: "memory");   // this thread's weight copies have landed
        first_tile = false;
        fence_proxy_async_smem();   // generic-proxy writes -> visible to the tensor core's shared-memory reads
        __syncthreads();

        // ---- 2. R filter rows x (ROWB / 32) K slices into the register accumulators
        {
            const bool a_signed = idesc_a_signed(idesc);
            const uint32_t lt = layout_type_for_chunk(E::ROWB);
            const uint32_t hi = ((8u * E::ROWB) >> 4) | (lt << 29);   // SBO = 8 rows, swizzle
            const uint32_t lbo = 1u << 16;
            const uint32_t planes16 = planes_sa >> 4, wt16 = smem_u32(wt) >> 4;
            const uint32_t plane16 = static_cast<uint32_t>(p.plane_bytes) >> 4, wts16 = static_cast<uint32_t>(p.wt_stride) >> 4;
            const uint32_t shift16 = static_cast<uint32_t>(p.cw * E::ROWB) >> 4;   // one conv row of the rectangle
            const uint32_t half16 = (64u * E::ROWB) >> 4;                           // GEMM rows 64..127
            auto mma = [&](uint32_t a_lo, uint32_t b_lo) {
                const uint64_t bd = desc64((b_lo & 0x3FFFu) | lbo, hi);
                wgmma<MK, BN>(acc[0], desc64((a_lo & 0x3FFFu) | lbo, hi), bd, a_signed, 1u);
                wgmma<MK, BN>(acc[1], desc64(((a_lo + half16) & 0x3FFFu) | lbo, hi), bd, a_signed, 1u);
            };
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int i = 0; i < BN / 2; ++i) acc[h][i] = 0u;
            wgmma_fence();
            int par = 0, a = 0;
#pragma unroll 1
            for (int r = 0; r < p.R; ++r) {
                const uint32_t a_hi_pl = planes16 + par * PL * plane16 + a * shift16;
                const uint32_t b_hi_pl = wt16 + r * wts16;
#pragma unroll
                for (uint32_t q = 0; q < 2u * (E::ROWB / 32); q += 2) {
                    mma(a_hi_pl + q, b_hi_pl + q);
                    if (X3) {
                        mma(a_hi_pl + plane16 + q, b_hi_pl + q);
                        mma(a_hi_pl + q, b_hi_pl + p.R * wts16 + q);
                    }
                }
                if (++par == p.stride_h) { par = 0; ++a; }
            }
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_acc(acc[0]);
            wgmma_fence_acc(acc[1]);
        }
        // GEMM row of this thread in each 64-row half (acc_row16), and the column groups of 32
        const int row0 = 16 * warp_idx + acc_row16_row(lane);
        constexpr int GROUPS = (BN + 31) / 32;

        const uint32_t bias_sa = smem_u32(bias_s), scale_sa = smem_u32(scale_s);
        const int oi0 = p.pool ? static_cast<int>(ti) * p.ph : i0, oj0 = p.pool ? static_cast<int>(tj) * p.pw : j0;
        const int es = p.kp.out_es;
        uint8_t* out = static_cast<uint8_t*>(p.out);
        if (p.pool_on_acc) {
            // ---- 3a. MAX pooling on the RAW accumulators: the epilogue (acc + bias) * scale [relu] -> rne + saturate is
            // monotone non-decreasing in acc for a positive scale (float kinds: + bias, relu with a non-negative slope),
            // so max commutes with it EXACTLY and only the pooled pixels -- a fifth of the tile for 3x3/s2 -- pay for it.
            // Accumulators go registers -> a 16-byte-chunk-swizzled [128][bn] s32 tile in shared memory.
            const uint32_t raw_sa = stage_sa;
            const uint32_t nchunk = static_cast<uint32_t>(p.bn) >> 2;          // 16-byte chunks per row (4 | 8 | 16)
            // (the planes are dead: every thread's MMAs have retired -- but not yet every other thread's)
            __syncthreads();
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const uint32_t row = 64 * h + row0;
                const uint32_t row_sa = raw_sa + row * p.bn * 4;
                const uint32_t sw = row & (nchunk - 1);
#pragma unroll
                for (int g = 0; g < GROUPS; ++g) {
                    uint32_t v0[16];
                    acc_row16<BN>(acc[h], g, v0);
                    const int c0 = acc_row16_col(lane, g);
                    if (c0 >= BN || n0 + c0 >= p.k) continue;
#pragma unroll
                    for (int q = 0; q < 4; ++q)
                        sts128(row_sa + ((((c0 >> 2) + q) ^ sw) << 4), make_uint4(v0[4 * q], v0[4 * q + 1], v0[4 * q + 2], v0[4 * q + 3]));
                }
            }
            __syncthreads();
            // ---- 4a. item = (pooled pixel, 16 channels): window max, epilogue, 16 * out_es bytes to HBM
            const uint32_t pst_sa = smem_u32(smem + p.off_pool_stage);
            for (int it = tid; it < p.pool_items; it += STEM_THREADS) {
                const uint32_t e = p.div_groups.quot(it), g = it - e * p.groups;
                const uint32_t oi = p.div_tw.quot(e), oj = e - oi * p.store_tw;
                const int gi = oi0 + static_cast<int>(oi), gj = oj0 + static_cast<int>(oj);
                if (gi >= p.OH || gj >= p.OW || n0 + static_cast<int>(g) * 16 >= p.k) continue;
                const int hs = max(gi * p.ps_h - p.pp_h, 0), he = min(gi * p.ps_h - p.pp_h + p.pk_h, p.Ho);
                const int ws = max(gj * p.ps_w - p.pp_w, 0), we = min(gj * p.ps_w - p.pp_w + p.pk_w, p.Wo);
                uint32_t v[16];
                bool first = true;
                for (int y = hs; y < he; ++y) {
                    uint32_t m = (y - i0) * p.cw + (ws - j0);
                    for (int x = ws; x < we; ++x, ++m) {
                        const uint32_t rsa = raw_sa + m * p.bn * 4, sw = m & (nchunk - 1);
#pragma unroll
                        for (int q = 0; q < 4; ++q) {
                            const uint4 t4 = lds128(rsa + (((g * 4 + q) ^ sw) << 4));
                            if (first) { v[4 * q] = t4.x; v[4 * q + 1] = t4.y; v[4 * q + 2] = t4.z; v[4 * q + 3] = t4.w; }
                            else {
                                v[4 * q] = acc_max<MK>(v[4 * q], t4.x); v[4 * q + 1] = acc_max<MK>(v[4 * q + 1], t4.y);
                                v[4 * q + 2] = acc_max<MK>(v[4 * q + 2], t4.z); v[4 * q + 3] = acc_max<MK>(v[4 * q + 3], t4.w);
                            }
                        }
                        first = false;
                    }
                }
                if (first) continue;                                   // (an empty window cannot happen: defensive)
                // the conv kernels' epilogue on the pooled accumulators, staged in this item's own row, then stored
                const PanelRow prow = make_panel_row(pst_sa, lg_out, e);
                epilogue16<MK>(p.kp, v, g * 16, bias_sa, scale_sa, prow, prow);
                const size_t o = ((static_cast<size_t>(n_img) * p.OH + gi) * p.OW + gj) * p.ldc * es + static_cast<size_t>(n0 + g * 16) * es;
                for (int q = 0; q < es; ++q) {
                    if ((n0 + static_cast<int>(g) * 16) * es + q * 16 + 16 > p.k * es) break;      // (ragged last group)
                    *reinterpret_cast<uint4*>(out + o + q * 16) = lds128(panel_addr(prow, g * 16 * es + q * 16));
                }
            }
        } else {
        // ---- 3. fused epilogue into the staging tile (GEMM row m = i*cw + j <-> one thread)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const PanelRow out_row = make_panel_row(stage_sa, lg_out, 64 * h + row0);
            const PanelRow res_row = out_row;   // no residual
#pragma unroll
            for (int g = 0; g < GROUPS; ++g) {
                uint32_t v0[16];
                acc_row16<BN>(acc[h], g, v0);
                const int c0 = acc_row16_col(lane, g);
                if (c0 >= BN || n0 + c0 >= p.k) continue;
                epilogue16<MK>(p.kp, v0, c0, bias_sa, scale_sa, res_row, out_row);
            }
        }
        __syncthreads();

        // ---- 4. (max pool +) store: 16 bytes per thread and item, NHWC
        {
            const int out_dt = p.kp.out_dtype;
            for (int it = tid; it < p.store_items; it += STEM_THREADS) {
                const uint32_t e = p.div_cpp.quot(it), c16 = it - e * p.cpp;
                const uint32_t oi = p.div_tw.quot(e), oj = e - oi * p.store_tw;
                const int gi = oi0 + static_cast<int>(oi), gj = oj0 + static_cast<int>(oj);
                const int byte = c16 * 16;
                if (gi >= p.OH || gj >= p.OW || n0 * es + byte + 16 > p.k * es) continue;   // (ragged last n-tile)
                uint4 acc;
                if (!p.pool) {
                    acc = lds128(panel_addr(make_panel_row(stage_sa, lg_out, oi * p.cw + oj), byte));
                } else {
                    // window in conv coordinates, clipped to the conv output (padding cells never take part)
                    const int hs = max(gi * p.ps_h - p.pp_h, 0), he = min(gi * p.ps_h - p.pp_h + p.pk_h, p.Ho);
                    const int ws = max(gj * p.ps_w - p.pp_w, 0), we = min(gj * p.ps_w - p.pp_w + p.pk_w, p.Wo);
                    bool first = true;
                    acc = make_uint4(0, 0, 0, 0);
                    for (int y = hs; y < he; ++y) {
                        int m = (y - i0) * p.cw + (ws - j0);
                        for (int x = ws; x < we; ++x, ++m) {
                            const uint4 v = lds128(panel_addr(make_panel_row(stage_sa, lg_out, m), byte));
                            if (first) { acc = v; first = false; continue; }
                            if (out_dt == B200_UINT8) {
                                acc.x = __vmaxu4(acc.x, v.x); acc.y = __vmaxu4(acc.y, v.y); acc.z = __vmaxu4(acc.z, v.z); acc.w = __vmaxu4(acc.w, v.w);
                            } else if (out_dt == B200_INT8) {
                                acc.x = __vmaxs4(acc.x, v.x); acc.y = __vmaxs4(acc.y, v.y); acc.z = __vmaxs4(acc.z, v.z); acc.w = __vmaxs4(acc.w, v.w);
                            } else if (out_dt == B200_HALF) {
                                // r >= x ? r : x on every lane, as the stand-alone pooling kernel
                                uint32_t* a = &acc.x; const uint32_t* b = &v.x;
#pragma unroll
                                for (int q = 0; q < 4; ++q) {
                                    const __half2 ha = *reinterpret_cast<const __half2*>(a + q), hb = *reinterpret_cast<const __half2*>(b + q);
                                    const float2 fa = __half22float2(ha), fb = __half22float2(hb);
                                    const __half2 r = __halves2half2(fa.x >= fb.x ? __low2half(ha) : __low2half(hb),
                                                                     fa.y >= fb.y ? __high2half(ha) : __high2half(hb));
                                    a[q] = *reinterpret_cast<const uint32_t*>(&r);
                                }
                            } else {
                                float* a = reinterpret_cast<float*>(&acc.x); const float* b = reinterpret_cast<const float*>(&v.x);
#pragma unroll
                                for (int q = 0; q < 4; ++q) a[q] = a[q] >= b[q] ? a[q] : b[q];
                            }
                        }
                    }
                }
                const size_t o = ((static_cast<size_t>(n_img) * p.OH + gi) * p.OW + gj) * p.ldc * es + static_cast<size_t>(n0) * es + byte;
                *reinterpret_cast<uint4*>(out + o) = acc;
            }
        }
        }
        // the next tile rewrites the planes and the staging tile
        __syncthreads();
    }
    if (first_tile) asm volatile("cp.async.wait_group 0;" ::: "memory");   // a CTA without a tile
}

namespace {

struct StemPlan {
    StemParams p;
    uint32_t idesc;
    int smem_bytes;
    dim3 grid;
    int kind;
};

int stem_elem_size(int math) { return math == B200_MATH_I8 ? 1 : (math == B200_MATH_F16 ? 2 : 4); }

// Geometry, tiling and shared-memory carve-up for one descriptor. Returns a B200 status.
int stem_plan(const b200_stem_desc_t* d, StemPlan* P) {
    if (!d) return B200_INVALID_VALUE;
    if (d->math != B200_MATH_I8 && d->math != B200_MATH_F16 && d->math != B200_MATH_TF32 && d->math != B200_MATH_TF32X3)
        return B200_UNIMPL_ERROR;
    if (d->n <= 0 || d->c <= 0 || d->c > 4 || d->h <= 0 || d->w <= 0 || d->k <= 0 || d->r <= 0 || d->s <= 0 ||
        d->stride_h <= 0 || d->stride_w <= 0 || d->pad_h < 0 || d->pad_w < 0)
        return B200_INVALID_VALUE;
    if (d->s > STEM_TAPS || d->r > 16 || d->stride_h > 4 || d->stride_w > 4) return B200_UNIMPL_ERROR;
    const int es = stem_elem_size(d->math);
    const bool x3 = d->math == B200_MATH_TF32X3;
    const int out_es = dtype_size(d->out_dtype);
    if (d->math == B200_MATH_I8 && !(d->out_dtype == B200_INT8 || d->out_dtype == B200_UINT8 || d->out_dtype == B200_FLOAT))
        return B200_INVALID_VALUE;
    if (d->math == B200_MATH_F16 && !(d->out_dtype == B200_HALF || d->out_dtype == B200_FLOAT)) return B200_INVALID_VALUE;
    if ((d->math == B200_MATH_TF32 || x3) && d->out_dtype != B200_FLOAT) return B200_INVALID_VALUE;
    if (d->ldc < d->k || (static_cast<int64_t>(d->ldc) * out_es) % 16 || (static_cast<int64_t>(d->k) * out_es) % 16)
        return B200_UNIMPL_ERROR;
    StemParams& p = P->p;
    memset(&p, 0, sizeof(p));
    p.n = d->n; p.c = d->c; p.h = d->h; p.w_in = d->w; p.k = d->k; p.ldc = d->ldc;
    p.R = d->r; p.stride_h = d->stride_h; p.stride_w = d->stride_w; p.pad_h = d->pad_h; p.pad_w = d->pad_w;
    p.Ho = (d->h + 2 * d->pad_h - d->r) / d->stride_h + 1;
    p.Wo = (d->w + 2 * d->pad_w - d->s) / d->stride_w + 1;
    if (p.Ho <= 0 || p.Wo <= 0) return B200_INVALID_VALUE;
    p.inv_scale = d->in_inv_scale;
    p.pool = 0;
    p.OH = p.Ho; p.OW = p.Wo;
    if (d->fuse_pool) {
        if (d->pool_type != B200_POOL_MAX || d->pool_global) return B200_UNIMPL_ERROR;
        b200_pool_desc_t pd;
        memset(&pd, 0, sizeof(pd));
        pd.dtype = d->out_dtype; pd.type = d->pool_type; pd.n = d->n; pd.h = p.Ho; pd.w = p.Wo; pd.c = d->k;
        pd.window_h = d->pool_window_h; pd.window_w = d->pool_window_w; pd.pad_h = d->pool_pad_h; pd.pad_w = d->pool_pad_w;
        pd.stride_h = d->pool_stride_h; pd.stride_w = d->pool_stride_w; pd.floor_as_conv = d->pool_floor_as_conv;
        int32_t oh, ow;
        int st = b200_pool_out_hw(&pd, &oh, &ow);
        if (st != B200_SUCCESS) return st;
        p.pool = 1;
        p.pk_h = pd.window_h; p.pk_w = pd.window_w; p.ps_h = pd.stride_h; p.ps_w = pd.stride_w;
        p.pp_h = pd.pad_h; p.pp_w = pd.pad_w;
        p.OH = oh; p.OW = ow;
        if (p.pk_h * p.pk_w > BLOCK_M) return B200_UNIMPL_ERROR;
    }
    // ---- tile: fewest CTAs per image; ties go to the wider tile (longer coalesced runs of the input rows)
    int best_tiles = 1 << 30, bt_h = 0, bt_w = 0;
    const int oh = p.OH, ow = p.OW;
    for (int tw = 1; tw <= ow && tw <= BLOCK_M; ++tw) {
        const int cwid = p.pool ? (tw - 1) * p.ps_w + p.pk_w : tw;
        if (cwid > BLOCK_M) break;
        int th_max = p.pool ? ((BLOCK_M / cwid - p.pk_h) / p.ps_h + 1) : BLOCK_M / cwid;
        if (p.pool && BLOCK_M / cwid < p.pk_h) th_max = 0;
        if (th_max < 1) continue;
        if (th_max > oh) th_max = oh;
        const int tiles_h = (oh + th_max - 1) / th_max;
        const int th = (oh + tiles_h - 1) / tiles_h;      // equal-height tiles
        const int tiles = tiles_h * ((ow + tw - 1) / tw);
        if (tiles < best_tiles || (tiles == best_tiles && tw > bt_w)) { best_tiles = tiles; bt_h = th; bt_w = tw; }
    }
    if (bt_h == 0) return B200_UNIMPL_ERROR;
    if (p.pool) {
        p.ph = bt_h; p.pw = bt_w;
        p.ch = (bt_h - 1) * p.ps_h + p.pk_h; p.cw = (bt_w - 1) * p.ps_w + p.pk_w;
    } else {
        p.ch = bt_h; p.cw = bt_w;
    }
    p.tiles_h = (oh + bt_h - 1) / bt_h;
    p.tiles_w = (ow + bt_w - 1) / bt_w;
    const int amax = (p.R - 1) / p.stride_h;
    p.krows = p.ch + amax;
    p.qrows = (p.ch - 1) * p.stride_h + p.R;
    p.qcols = (p.cw - 1) * p.stride_w + STEM_TAPS;
    const int rowb = STEM_TAPS * 4 * es;
    const int planes_n = x3 ? 2 : 1;
    int prow = p.krows * p.cw;
    if (prow < amax * p.cw + BLOCK_M) prow = amax * p.cw + BLOCK_M;   // the MMA reads 128 rows from the shifted start
    p.plane_bytes = ((prow + 7) / 8 * 8 * rowb + 1023) & ~1023;
    // ---- output channels per CTA: as many (<= 64) as shared memory allows
    const int kr = d->k <= 16 ? 16 : (d->k <= 32 ? 32 : 64);
    for (int bn = kr; bn >= 16; bn >>= 1) {
        p.bn = bn;
        p.wt_stride = (bn * rowb + 1023) & ~1023;
        p.off_planes = planes_n * p.R * p.wt_stride;
        p.off_stage = p.off_planes + p.stride_h * planes_n * p.plane_bytes;      // (1024-aligned: every part is)
        // pooling on the raw accumulators needs the [128][bn] s32 tile and one staged row per pooled pixel
        p.pool_on_acc = (p.pool && d->monotone_epilogue) ? 1 : 0;
        if (p.pool_on_acc) {
            // the raw tile reuses the planes (dead once the MMAs have retired; the next tile rewrites them after the
            // barrier that ends this one); a single-panel pooled staging tile only needs the pooled pixels' rows
            const int planes_bytes = p.stride_h * planes_n * p.plane_bytes, raw_bytes = BLOCK_M * bn * 4;
            p.off_stage = p.off_planes;
            p.off_pool_stage = p.off_planes + (planes_bytes > raw_bytes ? planes_bytes : raw_bytes);
            const int pooled_rows = bn * out_es <= 128 ? ((p.ph * p.pw + 7) & ~7) : BLOCK_M;
            p.off_tail = (p.off_pool_stage + pooled_rows * bn * out_es + 1023) & ~1023;
        } else {
            p.off_pool_stage = p.off_stage + BLOCK_M * bn * out_es;
            p.off_tail = p.off_pool_stage;
        }
        P->smem_bytes = p.off_tail + 2 * 64 * 4 + 16 + 1024;
        if (P->smem_bytes <= MAX_SMEM) break;
        if (bn == 16) return B200_OUT_OF_MEM;
    }
    p.tiles_img = p.tiles_h * p.tiles_w;
    p.tiles_total = d->n * p.tiles_img;
    p.cpp = (d->k < p.bn ? d->k : p.bn) * out_es / 16;   // (a ragged last n-tile stores fewer: guarded by the kernel)
    p.store_tw = p.pool ? p.pw : p.cw;
    p.store_items = (p.pool ? p.ph * p.pw : p.ch * p.cw) * p.cpp;
    p.div_bn.set(p.bn); p.div_tiles_img.set(p.tiles_img); p.div_tiles_w.set(p.tiles_w); p.div_qcols.set(p.qcols);
    p.div_sh.set(p.stride_h); p.div_sw.set(p.stride_w); p.div_cpp.set(p.cpp); p.div_tw.set(p.store_tw);
    p.pairs_row = p.qcols / 2;        // (qcols is even whenever stride_w is)
    p.div_pairs.set(p.pairs_row);
    p.groups = p.bn / 16;
    p.pool_items = p.pool ? p.ph * p.pw * p.groups : 0;
    p.div_groups.set(p.groups);
    ConvKParams& kp = p.kp;
    kp.K = d->k;
    kp.relu = d->relu; kp.neg_slope = d->neg_slope; kp.sum_scale = 1.f;
    kp.out_dtype = d->out_dtype; kp.res_dtype = -1;
    kp.out_es = out_es;
    kp.epi_bn = p.bn;
    kp.out_pw = p.bn * out_es >= 128 ? 128 : p.bn * out_es;
    kp.out_panels = p.bn * out_es / kp.out_pw;
    kp.res_es = 0; kp.res_pw = 0; kp.res_panels = 0;
    kp.split = 1;
    uint32_t a_fmt = 0, b_fmt = 0, c_fmt = 1;
    if (d->math == B200_MATH_I8) { a_fmt = 1u; b_fmt = 1u; c_fmt = 2u; }       // the graph input quantises to s8
    else if (d->math != B200_MATH_F16) { a_fmt = b_fmt = 2u; }
    P->idesc = make_idesc(c_fmt, a_fmt, b_fmt, BLOCK_M, p.bn);
    // persistent CTAs: a few per SM (they hide each other's serial phases), each walking its share of the tiles with the
    // weights and tables set up once
    {
        const int n_tiles_n = (d->k + p.bn - 1) / p.bn;
        int per_sm = (MAX_SMEM + 1024) / (P->smem_bytes + 1024);
        if (per_sm > 4) per_sm = 4;
        if (per_sm < 1) per_sm = 1;
        int ctas = sm_count() * per_sm / n_tiles_n;
        if (ctas < 1) ctas = 1;
        if (ctas > p.tiles_total) ctas = p.tiles_total;
        P->grid = dim3(ctas, n_tiles_n, 1);
    }
    P->kind = d->math == B200_MATH_I8 ? KIND_I8 : (d->math == B200_MATH_F16 ? KIND_F16 : (x3 ? KIND_TF32X3 : KIND_TF32));
    return B200_SUCCESS;
}

template <int KIND, int BN>
void launch_stem_bn(const StemPlan& P, cudaStream_t stream) {
    auto kern = conv_stem_kernel<KIND, BN>;
    static std::atomic<bool> opted_in[kMaxDevices];
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev >= 0 && dev < kMaxDevices && !opted_in[dev].load(std::memory_order_acquire)) {
        cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, MAX_SMEM);
        // several small CTAs per SM hide each other's serial phases: ask for the whole shared-memory carveout
        cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        opted_in[dev].store(true, std::memory_order_release);
    }
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = P.grid;
    cfg.blockDim = dim3(STEM_THREADS);
    cfg.dynamicSmemBytes = P.smem_bytes;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    cudaLaunchKernelEx(&cfg, kern, P.p, P.idesc);
    count_launch();
}

template <int KIND>
void launch_stem(const StemPlan& P, cudaStream_t stream) {
    switch (P.p.bn) {
        case 16: launch_stem_bn<KIND, 16>(P, stream); break;
        case 32: launch_stem_bn<KIND, 32>(P, stream); break;
        default: launch_stem_bn<KIND, 64>(P, stream); break;
    }
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" {

int b200_stem_conv_out_hw(const b200_stem_desc_t* d, int32_t* oh, int32_t* ow) {
    StemPlan P;
    int st = stem_plan(d, &P);
    if (st != B200_SUCCESS) return st;
    if (oh) *oh = P.p.OH;
    if (ow) *ow = P.p.OW;
    return B200_SUCCESS;
}

size_t b200_stem_packed_weight_bytes(const b200_stem_desc_t* d) {
    if (!d || d->k <= 0 || d->r <= 0) return 0;
    const int es = stem_elem_size(d->math);
    return static_cast<size_t>(d->k) * d->r * STEM_TAPS * 4 * es * (d->math == B200_MATH_TF32X3 ? 2 : 1);
}

int b200_stem_pack_weights(const b200_stem_desc_t* d, const void* src_kcrs, void* dst_packed) {
    if (!d || !src_kcrs || !dst_packed || d->s > STEM_TAPS || d->c > 4 || d->c <= 0) return B200_INVALID_VALUE;
    const int es = stem_elem_size(d->math);
    const size_t rowb = STEM_TAPS * 4 * es;
    const size_t image = static_cast<size_t>(d->k) * d->r * rowb;
    memset(dst_packed, 0, b200_stem_packed_weight_bytes(d));
    const uint8_t* src = static_cast<const uint8_t*>(src_kcrs);
    uint8_t* dst = static_cast<uint8_t*>(dst_packed);
    for (int oc = 0; oc < d->k; ++oc)
        for (int ch = 0; ch < d->c; ++ch)
            for (int r = 0; r < d->r; ++r)
                for (int s = 0; s < d->s; ++s) {
                    const size_t so = (((static_cast<size_t>(oc) * d->c + ch) * d->r + r) * d->s + s) * es;
                    const size_t doff = (static_cast<size_t>(oc) * d->r + r) * rowb + (static_cast<size_t>(s) * 4 + ch) * es;
                    if (d->math == B200_MATH_TF32X3) {
                        uint32_t u;
                        memcpy(&u, src + so, 4);
                        const uint32_t hu = u & 0xFFFFE000u;
                        float x, h;
                        memcpy(&x, &u, 4);
                        memcpy(&h, &hu, 4);
                        const float l = x - h;
                        memcpy(dst + doff, &h, 4);
                        memcpy(dst + image + doff, &l, 4);
                    } else {
                        memcpy(dst + doff, src + so, es);
                    }
                }
    return B200_SUCCESS;
}

int b200_stem_conv_info(const b200_stem_desc_t* d, int32_t* tile_h, int32_t* tile_w, int32_t* block_n, int32_t* ctas,
                        int32_t* smem_bytes) {
    StemPlan P;
    int st = stem_plan(d, &P);
    if (st != B200_SUCCESS) return st;
    if (tile_h) *tile_h = P.p.ch;
    if (tile_w) *tile_w = P.p.cw;
    if (block_n) *block_n = P.p.bn;
    if (ctas) *ctas = static_cast<int32_t>(P.grid.x * P.grid.y);
    if (smem_bytes) *smem_bytes = P.smem_bytes;
    return B200_SUCCESS;
}

int b200_stem_conv_run(const b200_stem_desc_t* d, const float* in_nchw, const void* packed_weights_dev, const float* bias_dev,
                       const float* scale_dev, void* out, void* stream) {
    if (!d || !in_nchw || !packed_weights_dev || !out) return B200_INVALID_VALUE;
    if (!device_is_sm90()) return B200_WRONG_DEVICE;
    StemPlan P;
    int st = stem_plan(d, &P);
    if (st != B200_SUCCESS) return st;
    P.p.in = in_nchw;
    P.p.w = static_cast<const uint8_t*>(packed_weights_dev);
    P.p.out = out;
    P.p.kp.bias = bias_dev;
    P.p.kp.scale = scale_dev;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    switch (P.kind) {
        case KIND_I8: launch_stem<KIND_I8>(P, s); break;
        case KIND_F16: launch_stem<KIND_F16>(P, s); break;
        case KIND_TF32X3: launch_stem<KIND_TF32X3>(P, s); break;
        default: launch_stem<KIND_TF32>(P, s); break;
    }
    cudaError_t e = cudaPeekAtLastError();
    if (e != cudaSuccess) {
        fprintf(stderr, "[b200_saber] stem conv launch failed: %s\n", cudaGetErrorString(e));
        return B200_UNKNOWN_ERROR;
    }
    return B200_SUCCESS;
}

}  // extern "C"
