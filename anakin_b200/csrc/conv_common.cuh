// Shared between the convolution kernels (conv_igemm.cu: TMA-im2col implicit GEMM; conv_slab.cu: slab-staged
// stride-1 RxS convolution): kernel parameters, the swizzled-panel epilogue helpers, geometry and the plan object.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>

#include <type_traits>

#include "../../include/b200_saber.h"
#include "common.cuh"
#include "ptx.cuh"

namespace b200 {

constexpr int BLOCK_M = 128;
constexpr int STAGE_K_BYTES = 128;  // K bytes per pipeline stage (4 MMAs of 32 B)
constexpr int A_STAGE_BYTES = BLOCK_M * STAGE_K_BYTES;
constexpr int MAX_STAGES = 12;
constexpr int EPI_WARPS = 8;                       // two consumer warpgroups: 64 GEMM rows each (wgmma M = 64)
constexpr int EPI_THREADS = 32 * EPI_WARPS;
constexpr int EPI_TID0 = 128;                      // warpgroup 0 holds the TMA producer (warp 0, one lane)
constexpr int NUM_THREADS = EPI_TID0 + EPI_THREADS;
constexpr int MAX_SMEM = 227 * 1024;

struct ConvKParams {
    int32_t M_total, HoWo, Wo;
    int32_t pad_h, pad_w, stride_h, stride_w, dil_h, dil_w;
    int32_t R, S;
    int32_t CC;        // channel chunks per filter tap
    int32_t chunk;     // bytes per chunk (16|32|64|128)
    int32_t chunk_el;  // elements per chunk
    int32_t KS;        // k-steps issued (KS_real rounded up to even when chunk==16)
    int32_t KS_real;   // R*S*CC
    int32_t K;         // output channels
    int32_t relu;
    float neg_slope;
    float sum_scale;
    int32_t out_dtype, res_dtype;
    int32_t stages;      // depth of the operand ring
    int32_t out_es;      // bytes per output element
    int32_t epi_bn;      // channels of the tile this CTA finishes and stores (BN, or BN/split with split-K)
    int32_t out_pw;      // output panel width in bytes (16|32|64|128) = TMA-store box inner extent
    int32_t out_panels;  // epi_bn*out_es / out_pw
    int32_t res_es, res_pw, res_panels;  // same for the residual tile (0 panels = no residual)
    int32_t split;       // split-K factor = cluster size along z (1, 2 or 4)
    const float* bias;
    const float* scale;
};

// Tiling of the slab-staged stride-1 R x S convolution (conv_slab.cu). A CTA owns a th x tw rectangle of one
// image's output; per input-channel chunk it stages the (th+R-1) x (tw+S-1) input rectangle ONCE (one tiled 4-D TMA
// box, halo zero-filled) as rows of `chunk` bytes -- the "slab" -- and issues the R*S filter taps as MMAs whose A
// descriptors start (r*PW + s) rows into it. GEMM row m = i*PW + j is output pixel (p0+i, q0+j); rows with
// j >= tw or i >= th are computed and dropped.
struct SlabParams {
    int32_t th, tw, PW;            // tile rows / columns, slab pitch = tw + S - 1
    int32_t tiles_h, tiles_w;      // tiles per image
    int32_t Ho, Wo;
    int32_t slab_bytes;            // one slab slot (rows allocated x chunk, multiple of 1024)
    int32_t slab_box_bytes;        // bytes one slab load delivers = (th+R-1) * PW * chunk
    int32_t SA, SB;                // slab slots, weight-tile slots
    int32_t btile_bytes;           // BN * chunk
    int32_t mma_per_tap;           // chunk / 32
    int32_t a_off, b_off, epi_off; // smem carve-up: slab ring, weight ring (staging reuses the front), residual tile
    int32_t step_h, step_w;        // conv-output distance between neighbouring tiles (= th, tw unless pooling is fused)
    int32_t org_h, org_w;          // conv-output origin of tile (0, 0): 0, or -pool_pad with a padded pooling window
    // fused MAX pooling (b200_conv_desc_t::fuse_pool): the CTA's th x tw conv rectangle is what a ph x pw tile of pooled
    // pixels needs (neighbouring rectangles overlap when the window exceeds the stride); the pooled pixels are written
    // straight from the staging tile, 16 bytes per thread
    int32_t pool, pk, ps, pp;      // fused pooling: window, stride, padding (square)
    int32_t ph, pw, PHo, PWo;      // pooled tile of a CTA, pooled size
    int32_t out_ld_bytes;          // pooled tensor: bytes per pixel row pitch
    void* out_ptr;                 // pooled tensor (bound per run)
};

// Shared memory carve-up (1024-B aligned base):
//   [ stages x (A 16 KiB + B BN*128 B) ]  operand ring; reused as the output staging tile
//   [ residual tile 128 x BN x res_es ]   TMA-prefetched during the main loop
//   [ bias BN f32 | scale BN f32 ]        epilogue tables
//   [ full[MAX] empty[MAX] conv[MAX] res_full part | spare ]
// x3 = error-compensated fp32: every stage also holds the A-low tile and the W-low tile.
__host__ __device__ constexpr int stage_bytes(int bn, bool x3 = false) {
    return (x3 ? 2 : 1) * (A_STAGE_BYTES + bn * STAGE_K_BYTES);
}
__host__ __device__ constexpr int tail_bytes(int bn) { return 2 * bn * 4 + (3 * MAX_STAGES + 3) * 8 + 16; }

__device__ __forceinline__ uint32_t layout_type_for_chunk(int chunk) {
    return chunk == 128 ? 2u : (chunk == 64 ? 4u : (chunk == 32 ? 6u : 0u));
}

// ----------------------------------------------------------------- swizzled panel access
// A panel is [128 rows x pw bytes] (pw = 1 << lg, 32|64|128) written / read by TMA with
// SWIZZLE_{32,64,128}B: the 16-byte chunk index is XOR-ed with address bits [7, 7+lg-4).
struct PanelRow {       // everything about one thread's row of a panelled tile, precomputed once
    uint32_t base;      // shared-space address of the tile + row * pw
    int lg;             // log2(panel width in bytes)
    int sw;             // swizzle XOR of this row
};
__device__ __forceinline__ PanelRow make_panel_row(uint32_t tile_saddr, int lg, int row) {
    PanelRow r;
    r.lg = lg;
    r.base = tile_saddr + (static_cast<uint32_t>(row) << lg);
    r.sw = (row >> (7 - lg)) & ((1 << (lg - 4)) - 1);
    return r;
}
__device__ __forceinline__ uint32_t panel_addr(const PanelRow& r, int byte_in_row) {
    const int panel = byte_in_row >> r.lg;
    const int c16 = (byte_in_row & ((1 << r.lg) - 1)) >> 4;
    return r.base + (static_cast<uint32_t>(panel) << (7 + r.lg)) + (static_cast<uint32_t>(c16 ^ r.sw) << 4);
}
__device__ __forceinline__ uint4 lds128(uint32_t saddr) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(saddr));
    return v;
}
__device__ __forceinline__ void sts128(uint32_t saddr, uint4 v) {
    asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(saddr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ void lds_f32x16(uint32_t saddr, float (&f)[16]) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const uint4 t = lds128(saddr + q * 16);
        f[4 * q] = __uint_as_float(t.x); f[4 * q + 1] = __uint_as_float(t.y);
        f[4 * q + 2] = __uint_as_float(t.z); f[4 * q + 3] = __uint_as_float(t.w);
    }
}

// ---- int8 epilogue arithmetic kept off the conversion pipe (I2F.U8 / F2I issue at a quarter of the fp32 rate and
// made the epilogue of wide tiles conversion-bound), in pairs of round-to-nearest fp32 operations.
struct F2 { float x, y; };
__device__ __forceinline__ F2 add2(F2 a, F2 b) { return F2{__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)}; }
__device__ __forceinline__ F2 mul2(F2 a, F2 b) { return F2{__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)}; }
__device__ __forceinline__ F2 fma2(F2 a, F2 b, F2 c) { return F2{__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)}; }
// byte `lane` of w -> float, exactly: splice the byte under the exponent of 2^23 and subtract 2^23
// (+128 for int8 residuals, whose words were xor-ed with 0x80808080 first)
__device__ __forceinline__ float byte_as_biased_float(uint32_t w, int lane) {
    uint32_t t;
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(t) : "r"(w), "r"(0x4B000000u), "r"(0x7650u + lane));
    return __uint_as_float(t);
}
// Quantise four lanes: clamp to the integer range [lo, hi], add 1.5 * 2^23 -- the fp32 add rounds to
// nearest-even exactly as cvt.rni / vcvtps2dq do -- and gather the low bytes. round(clamp(x)) == clamp(round(x))
// for integer bounds, so this equals cvt.rni.sat.{s8,u8}.f32 on every finite input.
__device__ __forceinline__ uint32_t pack4_q8(F2 a, F2 b, float lo, float hi) {
    const F2 magic = {12582912.f, 12582912.f};
    a.x = fminf(fmaxf(a.x, lo), hi); a.y = fminf(fmaxf(a.y, lo), hi);
    b.x = fminf(fmaxf(b.x, lo), hi); b.y = fminf(fmaxf(b.y, lo), hi);
    a = add2(a, magic);
    b = add2(b, magic);
    uint32_t l, h, w;
    asm("prmt.b32 %0, %1, %2, 0x0040;" : "=r"(l) : "r"(__float_as_uint(a.x)), "r"(__float_as_uint(a.y)));
    asm("prmt.b32 %0, %1, %2, 0x0040;" : "=r"(h) : "r"(__float_as_uint(b.x)), "r"(__float_as_uint(b.y)));
    asm("prmt.b32 %0, %1, %2, 0x5410;" : "=r"(w) : "r"(l), "r"(h));
    return w;
}

// One thread, one output row, 16 consecutive channels starting at tile-local column cl.
// int8 nets: x86 Saber epilogue (acc + bias) * scale, [relu], [+ res * sum_scale], [relu], rne + saturate; the
// residual is s8 | u8 and the output s8 | u8 | f32 (the fc feeding softmax).
__device__ __forceinline__ void epilogue16_i8(const ConvKParams& p, const uint32_t (&v)[16], int cl, uint32_t bias_sa,
                                              uint32_t scale_sa, const PanelRow& res_row, const PanelRow& out_row) {
    F2 f[8];
    {
        float bias[16], scale[16];
        lds_f32x16(bias_sa + cl * 4, bias);
        lds_f32x16(scale_sa + cl * 4, scale);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const F2 a = {__int2float_rn(static_cast<int32_t>(v[2 * i])), __int2float_rn(static_cast<int32_t>(v[2 * i + 1]))};
            f[i] = mul2(add2(a, F2{bias[2 * i], bias[2 * i + 1]}), F2{scale[2 * i], scale[2 * i + 1]});
        }
    }
    if (p.res_panels > 0) {
        const uint4 t = lds128(panel_addr(res_row, cl));
        const bool rs = p.res_dtype == B200_INT8;
        const uint32_t flip = rs ? 0x80808080u : 0u;
        const float off = rs ? -8388736.f : -8388608.f;     // -(2^23 [+ 128])
        const uint32_t w[4] = {t.x ^ flip, t.y ^ flip, t.z ^ flip, t.w ^ flip};
        const bool unit = p.sum_scale == 1.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const F2 r = add2(F2{byte_as_biased_float(w[i >> 1], (2 * i) & 3), byte_as_biased_float(w[i >> 1], (2 * i + 1) & 3)},
                              F2{off, off});
            f[i] = unit ? add2(f[i], r) : fma2(r, F2{p.sum_scale, p.sum_scale}, f[i]);
        }
    }
    if (p.out_dtype == B200_FLOAT) {
        if (p.relu) {
#pragma unroll
            for (int i = 0; i < 8; ++i) { f[i].x = fmaxf(f[i].x, 0.f); f[i].y = fmaxf(f[i].y, 0.f); }
        }
#pragma unroll
        for (int q = 0; q < 4; ++q)
            sts128(panel_addr(out_row, cl * 4 + q * 16),
                   make_uint4(__float_as_uint(f[2 * q].x), __float_as_uint(f[2 * q].y),
                              __float_as_uint(f[2 * q + 1].x), __float_as_uint(f[2 * q + 1].y)));
    } else {
        // relu (it is the last step whenever it is set: relu-before-sum only exists without a sum) folds into
        // the lower clamp bound; u8 saturates at 0 anyway
        const bool u = p.out_dtype == B200_UINT8;
        const float lo = (u || p.relu) ? 0.f : -128.f, hi = u ? 255.f : 127.f;
        sts128(panel_addr(out_row, cl), make_uint4(pack4_q8(f[0], f[1], lo, hi), pack4_q8(f[2], f[3], lo, hi),
                                                   pack4_q8(f[4], f[5], lo, hi), pack4_q8(f[6], f[7], lo, hi)));
    }
}

// float nets carry and write their own type (or f32): acc (+ beta * res) + bias, relu(neg_slope)
template <int KIND>
__device__ __forceinline__ void epilogue16(const ConvKParams& p, const uint32_t (&v)[16], int cl, uint32_t bias_sa,
                                           uint32_t scale_sa, const PanelRow& res_row, const PanelRow& out_row) {
    if constexpr (KIND == KIND_I8) {
        epilogue16_i8(p, v, cl, bias_sa, scale_sa, res_row, out_row);
        return;
    }
    float f[16], r[16];
    const bool has_res = p.res_panels > 0;
    if (has_res) {
        if (p.res_dtype == B200_FLOAT) {
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const uint4 t = lds128(panel_addr(res_row, cl * 4 + q * 16));
                r[4 * q] = __uint_as_float(t.x); r[4 * q + 1] = __uint_as_float(t.y);
                r[4 * q + 2] = __uint_as_float(t.z); r[4 * q + 3] = __uint_as_float(t.w);
            }
        } else if (KIND == KIND_F16 && p.res_dtype == B200_HALF) {
#pragma unroll
            for (int q = 0; q < 2; ++q) {
                const uint4 t = lds128(panel_addr(res_row, cl * 2 + q * 16));
                const __half2* h = reinterpret_cast<const __half2*>(&t);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const float2 x = __half22float2(h[i]);
                    r[8 * q + 2 * i] = x.x; r[8 * q + 2 * i + 1] = x.y;
                }
            }
        }
    }
    float bias[16];
    lds_f32x16(bias_sa + cl * 4, bias);
#pragma unroll
    for (int i = 0; i < 16; ++i) {
        float x = __uint_as_float(v[i]);
        if (has_res) x = __fmaf_rn(p.sum_scale, r[i], x);
        x = __fadd_rn(x, bias[i]);
        if (p.relu) x = x > 0.f ? x : __fmul_rn(x, p.neg_slope);
        f[i] = x;
    }
    // ---- stage into the swizzled output tile
    if (p.out_dtype == B200_FLOAT) {
#pragma unroll
        for (int q = 0; q < 4; ++q)
            sts128(panel_addr(out_row, cl * 4 + q * 16),
                   make_uint4(__float_as_uint(f[4 * q]), __float_as_uint(f[4 * q + 1]),
                              __float_as_uint(f[4 * q + 2]), __float_as_uint(f[4 * q + 3])));
    } else if (KIND == KIND_F16 && p.out_dtype == B200_HALF) {
#pragma unroll
        for (int q = 0; q < 2; ++q) {
            uint32_t w[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                __half2 h = __floats2half2_rn(f[8 * q + 2 * i], f[8 * q + 2 * i + 1]);
                w[i] = *reinterpret_cast<uint32_t*>(&h);
            }
            sts128(panel_addr(out_row, cl * 2 + q * 16), make_uint4(w[0], w[1], w[2], w[3]));
        }
    }
}

// log2 of a panel width in bytes (16 | 32 | 64 | 128)
__device__ __forceinline__ int panel_lg(int pw) { return pw == 128 ? 7 : (pw == 64 ? 6 : (pw == 32 ? 5 : 4)); }

// Epilogue tables of the n channels from n0, filled by threads t of NT: bias (0 past K or without one) and per-channel
// scale (1 past K or without one).
template <int NT>
__device__ __forceinline__ void fill_epilogue_tables(const ConvKParams& p, int n0, int n, int t, float* bias_s, float* scale_s) {
    for (int i = t; i < n; i += NT) {
        const bool ok = (n0 + i) < p.K;
        bias_s[i] = (p.bias != nullptr && ok) ? __ldg(p.bias + n0 + i) : 0.f;
        scale_s[i] = (p.scale != nullptr && ok) ? __ldg(p.scale + n0 + i) : 1.f;
    }
}

// 3xTF32: split a landed fp32 operand tile of nvec 16-byte vectors in place, hi = top 19 bits, and write
// lo = x - hi (exact in fp32) to the low plane; then make both visible to the tensor core and wait for every consumer
// thread (etid of EPI_THREADS).
__device__ __forceinline__ void split_tf32x3(uint4* hi, uint4* lo, int nvec, int etid) {
    for (int i = etid; i < nvec; i += EPI_THREADS) {
        uint4 x = hi[i], h, l;
        h.x = x.x & 0xFFFFE000u; h.y = x.y & 0xFFFFE000u; h.z = x.z & 0xFFFFE000u; h.w = x.w & 0xFFFFE000u;
        l.x = __float_as_uint(__fsub_rn(__uint_as_float(x.x), __uint_as_float(h.x)));
        l.y = __float_as_uint(__fsub_rn(__uint_as_float(x.y), __uint_as_float(h.y)));
        l.z = __float_as_uint(__fsub_rn(__uint_as_float(x.z), __uint_as_float(h.z)));
        l.w = __float_as_uint(__fsub_rn(__uint_as_float(x.w), __uint_as_float(h.w)));
        hi[i] = h;
        lo[i] = l;
    }
    fence_proxy_async_smem();  // generic-proxy writes -> visible to the tensor core's smem reads
    asm volatile("bar.sync 1, %0;" ::"n"(EPI_THREADS) : "memory");
}

// MAX of two 16-byte runs of staged output channels of dtype dt, as the stand-alone pooling kernel computes it: packed
// bytes (u8 | s8), half lanes compared through float (r >= x ? r : x), floats (r >= x ? r : x).
__device__ __forceinline__ uint4 max16(uint4 acc, uint4 v, int dt) {
    if (dt == B200_UINT8) {
        acc.x = __vmaxu4(acc.x, v.x); acc.y = __vmaxu4(acc.y, v.y); acc.z = __vmaxu4(acc.z, v.z); acc.w = __vmaxu4(acc.w, v.w);
    } else if (dt == B200_INT8) {
        acc.x = __vmaxs4(acc.x, v.x); acc.y = __vmaxs4(acc.y, v.y); acc.z = __vmaxs4(acc.z, v.z); acc.w = __vmaxs4(acc.w, v.w);
    } else if (dt == B200_HALF) {
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
    return acc;
}

// ----------------------------------------------------------------- phase timeline (debug builds only)
// -DB200_TIMELINE (tools/timeline.py builds it into anakin_b200/lib_tl) records per-CTA SM-clock stamps of
// the pipeline phases; the shipped library compiles all of it out.
#ifdef B200_TIMELINE
struct TlRec {
    unsigned long long gt0, gt1;
    long long clk[8];
    uint32_t bx, by, bz, smid, K, KS, bn, stages;
};
constexpr unsigned TL_CAP = 1u << 15;
static __device__ TlRec g_tl[TL_CAP];   // one array per translation unit (no -rdc)
static __device__ unsigned g_tl_n;
__device__ __forceinline__ unsigned long long tl_globaltimer() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
#define TL(slot) do { g_tl[tl_idx].clk[slot] = clock64(); } while (0)
#else
#define TL(slot) do { } while (0)
#endif


// ----------------------------------------------------------------- host-side geometry
static inline int elem_size(int math) { return math == B200_MATH_I8 ? 1 : (math == B200_MATH_F16 ? 2 : 4); }
static inline int dtype_size(int dt) {
    switch (dt) {
        case B200_HALF: return 2;
        case B200_FLOAT: return 4;
        case B200_INT32: return 4;
        default: return 1;
    }
}
// dtype of the operands a math kind reads (int8 activations move as bytes, signed or not)
static inline int operand_dtype(int math) {
    return math == B200_MATH_I8 ? B200_UINT8 : (math == B200_MATH_F16 ? B200_HALF : B200_FLOAT);
}
// Largest chunk (bytes) in {128,64,32,16} that divides the per-pixel channel bytes.
static inline int pick_chunk(int c_bytes) {
    if (c_bytes % 128 == 0) return 128;
    if (c_bytes % 64 == 0) return 64;
    if (c_bytes % 32 == 0) return 32;
    if (c_bytes % 16 == 0) return 16;
    return 0;
}

struct Geometry {
    int es, chunk, chunk_el, CC, KS_real, KS, ho, wo;
    int64_t M_total;
    bool ok;
};

static inline Geometry make_geometry(const b200_conv_desc_t* d) {
    Geometry g{};
    g.es = elem_size(d->math);
    g.chunk = pick_chunk(d->c * g.es);
    g.ok = g.chunk != 0 && d->n > 0 && d->h > 0 && d->w > 0 && d->k > 0 && d->r > 0 && d->s > 0 &&
           d->stride_h > 0 && d->stride_w > 0 && d->dil_h > 0 && d->dil_w > 0;
    if (!g.ok) return g;
    g.chunk_el = g.chunk / g.es;
    g.CC = d->c * g.es / g.chunk;
    g.KS_real = d->r * d->s * g.CC;
    g.KS = (g.chunk == 16) ? ((g.KS_real + 1) & ~1) : g.KS_real;
    g.ho = (d->h + 2 * d->pad_h - (d->dil_h * (d->r - 1) + 1)) / d->stride_h + 1;
    g.wo = (d->w + 2 * d->pad_w - (d->dil_w * (d->s - 1) + 1)) / d->stride_w + 1;
    g.M_total = static_cast<int64_t>(d->n) * g.ho * g.wo;
    g.ok = g.ho > 0 && g.wo > 0 && g.M_total < (1ll << 31);
    return g;
}

// ----------------------------------------------------------------- host-side kernel selection
static inline int kind_for_math(int math) {
    return math == B200_MATH_I8 ? KIND_I8
                                : (math == B200_MATH_F16 ? KIND_F16 : (math == B200_MATH_TF32X3 ? KIND_TF32X3 : KIND_TF32));
}
// Instruction descriptor of a 128 x bn MMA: int8 activations are signed or unsigned as in_dtype says, int8 weights signed.
static inline uint32_t conv_idesc(int math, int in_dtype, int bn) {
    if (math == B200_MATH_I8) return make_idesc(2u, in_dtype == B200_INT8 ? 1u : 0u, 1u, BLOCK_M, bn);
    if (math == B200_MATH_F16) return make_idesc(1u, 0u, 0u, BLOCK_M, bn);
    return make_idesc(1u, 2u, 2u, BLOCK_M, bn);
}

using ConvLaunch = void (*)(b200_conv_plan*, void* stream);
// Calls f(Int<KIND>(), Int<BN>()) for the run-time kind and tile width bn, BN one of BNS, and returns its result (the
// launch function of that kernel instance), or a null one when bn is not among BNS. The kernel instances that exist
// are the ones the f of a call site names.
template <int... BNS, typename F>
auto bind_kind_bn(int kind, int bn, F f) {
    decltype(f(Int<KIND_I8>(), Int<32>())) r{};
    auto by_bn = [&](auto k) { ((bn == BNS ? (void)(r = f(k, Int<BNS>())) : void()), ...); };
    switch (kind) {
        case KIND_I8: by_bn(Int<KIND_I8>()); break;
        case KIND_F16: by_bn(Int<KIND_F16>()); break;
        case KIND_TF32: by_bn(Int<KIND_TF32>()); break;
        case KIND_TF32X3: by_bn(Int<KIND_TF32X3>()); break;
    }
    return r;
}

// ----------------------------------------------------------------- planner cost model
// The constants -- per-MMA cost in SM clocks (K = 32 bytes, M = 128), the L2 ingest of one SM, the epilogue and fixed
// clocks of conv_slab.cu's estimate -- and the thresholds built on them were measured on the earlier sm_100 version of
// these kernels and have NOT been re-measured on the H100. They only rank plans of the same layer against each other.
constexpr double L2_INGEST_BYTES_PER_CLK = 38.7;
static inline double mma_clk(int bn) { return bn / 2.0 > 32.0 + bn / 4.0 ? bn / 2.0 : 32.0 + bn / 4.0; }
// widest tile: keeps an fp32 staging (or residual) tile <= 64 KiB
static inline int max_bn_for(int out_es, int res_es) { return (out_es == 4 || res_es == 4) ? 128 : 256; }
// B200_SABER_FORCE_BN (tuning experiments only): the forced tile width, or 0 when unset or not a width up to max_bn
static inline int forced_bn(int max_bn) {
    const char* e = getenv("B200_SABER_FORCE_BN");
    if (!e) return 0;
    const int fb = atoi(e);
    return ((fb == 32 || fb == 64 || fb == 128 || fb == 256) && fb <= max_bn) ? fb : 0;
}

// ----------------------------------------------------------------- tensor maps (tensor_map.cu)
// False when the driver does not export the tensor-map encoders.
bool tensor_maps_available();
// 2-D map over a row-major [m_total][ldc] activation matrix, box = one swizzled panel of BLOCK_M rows.
int encode_tile_map(CUtensorMap* map, const void* ptr, int dtype, int k_valid, int64_t m_total, int ldc, int panel_bytes);
// 4-D tiled map over an NHWC tensor [n][h][w][ldc] of which `c_valid` channels exist; box {box_c, box_w, box_h, 1}.
int encode_nhwc_map(CUtensorMap* map, const void* ptr, int dtype, int c_valid, int ldc, int w, int h, int n, int box_c,
                    int box_w, int box_h, int swizzle_bytes);
// im2col map of the plan's activation tensor `in` (pl->map_a).
int encode_im2col_map(b200_conv_plan* pl, const void* in);
// weights map of the plan (pl->map_b) for tile width bn.
int encode_weights_map(b200_conv_plan* pl, int bn);

}  // namespace b200

struct b200_conv_plan {
    b200_conv_desc_t desc;
    b200::Geometry g;
    int bn;
    dim3 grid;
    int smem_bytes;
    uint32_t idesc;
    b200::ConvKParams kp;
    const void* weights;
    CUtensorMap map_b;
    CUtensorMap map_a, map_out, map_res;
    const void* map_a_ptr;    // pointers the activation / output / residual maps were encoded for
    const void* map_out_ptr;
    const void* map_res_ptr;
    b200::ConvLaunch launch;
    // persistent tile-pipelined variant (conv_persistent.cu): grid.x x grid.y tiles walked by persistent_ctas CTAs
    bool persistent = false;
    int persistent_ctas = 0;
    // slab-staged variant (conv_slab.cu): 4-D tiled maps, its own tiling
    bool slab = false;
    b200::SlabParams sp;
};
