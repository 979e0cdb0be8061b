// Weight-streaming fully-connected layer for small row counts, and the fused classifier head.
//
// Replaces SaberFc<NV,*> (saber/funcs/impl/cuda/base/cuda_c/saber_fc.cu:17-195, ker_gemm.cu:8-186, cuBLAS sgemm) for
// m <= 16 rows: with a handful of rows an inner-product layer is a stream of its weights (VGG16 fc6: 411 MB of fp32)
// past a few vectors, so the right machine is the load path, not the tensor core -- a 128-row MMA tile would carry 4
// live rows and the error-compensated fp32 tensor path would read the weights twice. Every weight byte is read exactly
// once, 16 bytes per lane, by warps that each keep R output rows x 8 input rows of accumulators in registers; the input
// rows are staged per K chunk in shared memory and shared by the CTA's 8 warps.
//   int8 : dp4a (u8|s8 x s8 -> s32), exact, then the x86 Saber epilogue of the conv kernels
//          (f = (acc + bias) * scale, relu, rne + saturate) -- bit-identical to the wgmma path.
//   f16  : fp32 accumulation of exact products;   f32: FFMA.
//
// b200_head_run: global pooling + inner product + softmax of an INT8 classification head in ONE launch (k-split
// integer reduction, last CTA finishes), replacing three dependent launches
// (saber_pooling.cu, saber_fc.cu, saber_softmax.cu) at the latency-critical end of every request.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <atomic>

#include "../../include/b200_saber.h"
#include "common.cuh"
#include "softmax.cuh"
#include "ptx.cuh"

namespace b200 {

constexpr int FC_THREADS = 256;
constexpr int FC_WARPS = FC_THREADS / 32;
constexpr int FC_MT = 8;                  // input rows handled per pass
constexpr int FC_X_BYTES = 16 * 1024;     // one staged input chunk (two buffers): up to FC_MT rows x its K elements

struct FcParams {
    const void* x;        // [m][ldx] operand dtype
    const void* w;        // [n][k] operand dtype, k contiguous (k = ldx: stored-K order, zero weights on padding)
    const float* bias;    // [n] or null
    const float* scale;   // [n] (int8) or null
    void* out;            // [m][ldo]
    int m, k, n, ldx, ldo;
    int in_unsigned;      // int8: x is u8
    int out_dtype;        // B200_FLOAT | B200_HALF | B200_INT8 | B200_UINT8
    int relu;
    float neg_slope;
};

__device__ __forceinline__ uint4 ldg_stream(const uint4* p) {
    uint4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}
__device__ __forceinline__ int dp4a_us(uint32_t a_u8, uint32_t b_s8, int c) {
    int d;
    asm("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a_u8), "r"(b_s8), "r"(c));
    return d;
}
__device__ __forceinline__ int dp4a_ss(uint32_t a_s8, uint32_t b_s8, int c) {
    int d;
    asm("dp4a.s32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a_s8), "r"(b_s8), "r"(c));
    return d;
}

// MODE 0: int8 (accumulate s32), 1: f16 (accumulate f32), 2: f32.
template <int MODE>
struct FcAcc { typedef float type; };
template <>
struct FcAcc<0> { typedef int type; };

template <int MODE>
__device__ __forceinline__ void fc_dot(typename FcAcc<MODE>::type& acc, const uint4& xv, const uint4& wv, bool x_unsigned) {
    if constexpr (MODE == 0) {
        if (x_unsigned) {
            acc = dp4a_us(xv.x, wv.x, acc); acc = dp4a_us(xv.y, wv.y, acc);
            acc = dp4a_us(xv.z, wv.z, acc); acc = dp4a_us(xv.w, wv.w, acc);
        } else {
            acc = dp4a_ss(xv.x, wv.x, acc); acc = dp4a_ss(xv.y, wv.y, acc);
            acc = dp4a_ss(xv.z, wv.z, acc); acc = dp4a_ss(xv.w, wv.w, acc);
        }
    } else if constexpr (MODE == 1) {
        const __half2* xh = reinterpret_cast<const __half2*>(&xv);
        const __half2* wh = reinterpret_cast<const __half2*>(&wv);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float2 a = __half22float2(xh[i]), b = __half22float2(wh[i]);
            acc = __fmaf_rn(a.x, b.x, acc);
            acc = __fmaf_rn(a.y, b.y, acc);
        }
    } else {
        acc = __fmaf_rn(__uint_as_float(xv.x), __uint_as_float(wv.x), acc);
        acc = __fmaf_rn(__uint_as_float(xv.y), __uint_as_float(wv.y), acc);
        acc = __fmaf_rn(__uint_as_float(xv.z), __uint_as_float(wv.z), acc);
        acc = __fmaf_rn(__uint_as_float(xv.w), __uint_as_float(wv.w), acc);
    }
}

template <int MODE>
__device__ __forceinline__ void fc_store(const FcParams& p, int mi, int row, typename FcAcc<MODE>::type acc) {
    float f;
    if constexpr (MODE == 0) {
        // x86 Saber int8 epilogue, as epilogue16_i8 of the conv kernels: add, then multiply, each rounded
        f = __fmul_rn(__fadd_rn(__int2float_rn(acc), p.bias ? __ldg(p.bias + row) : 0.f), p.scale ? __ldg(p.scale + row) : 1.f);
        if (p.relu) f = fmaxf(f, 0.f);
    } else {
        f = __fadd_rn(acc, p.bias ? __ldg(p.bias + row) : 0.f);
        if (p.relu) f = f > 0.f ? f : __fmul_rn(f, p.neg_slope);
    }
    const size_t o = static_cast<size_t>(mi) * p.ldo + row;
    if (p.out_dtype == B200_FLOAT) {
        static_cast<float*>(p.out)[o] = f;
    } else if (p.out_dtype == B200_HALF) {
        static_cast<__half*>(p.out)[o] = __float2half_rn(f);
    } else if (p.out_dtype == B200_UINT8) {
        uint32_t c;
        asm("cvt.rni.sat.u8.f32 %0, %1;" : "=r"(c) : "f"(f));
        static_cast<uint8_t*>(p.out)[o] = static_cast<uint8_t>(c);
    } else {
        int32_t c;
        asm("cvt.rni.sat.s8.f32 %0, %1;" : "=r"(c) : "f"(f));
        static_cast<int8_t*>(p.out)[o] = static_cast<int8_t>(c);
    }
}

// The inner-product body: CTA `cta` of `ncta` takes the row blocks cta, cta + ncta, ... ; each of its 8 warps owns
// R consecutive output rows of the block. smem_x: 2 x FC_X_BYTES bytes -- the input rows are staged per K chunk with
// cp.async, chunk c+1 while chunk c is being multiplied, so the weight stream never waits for them.
template <int MODE, int R>
__device__ __forceinline__ void fc_body(const FcParams& p, uint8_t* smem_x, int cta, int ncta) {
    constexpr int ES = MODE == 0 ? 1 : (MODE == 1 ? 2 : 4);
    constexpr int VEC = 16 / ES;                     // elements per 16-byte vector
    typedef typename FcAcc<MODE>::type acc_t;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int rows_per_block = FC_WARPS * R;
    const int nblocks = (p.n + rows_per_block - 1) / rows_per_block;
    for (int m0 = 0; m0 < p.m; m0 += FC_MT) {
        const int mt = min(FC_MT, p.m - m0);
        // chunk length: the staged rows fill one buffer (more rows -> shorter chunks), whole 16-byte vectors
        const int kc_len = (FC_X_BYTES / (mt * 16)) * VEC;
        const int nchunks = (p.k + kc_len - 1) / kc_len;
        const int row_vecs = kc_len / VEC;           // vectors per staged row
        auto stage = [&](int buf, int c) {
            const int kc = c * kc_len;
            const int nv = min(kc_len, p.k - kc) / VEC;
            const uint32_t dst0 = static_cast<uint32_t>(__cvta_generic_to_shared(smem_x + buf * FC_X_BYTES));
            for (int i = threadIdx.x; i < mt * nv; i += FC_THREADS) {
                const int mi = i / nv, v = i - mi * nv;
                const void* src = static_cast<const uint8_t*>(p.x) + (static_cast<size_t>(m0 + mi) * p.ldx + kc) * ES + v * 16;
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst0 + (mi * row_vecs + v) * 16), "l"(src) : "memory");
            }
            asm volatile("cp.async.commit_group;" ::: "memory");
        };
        for (int blk = cta; blk < nblocks; blk += ncta) {
            const int row0 = blk * rows_per_block + warp * R;
            acc_t acc[FC_MT][R];
#pragma unroll
            for (int mi = 0; mi < FC_MT; ++mi)
#pragma unroll
                for (int r = 0; r < R; ++r) acc[mi][r] = 0;
            __syncthreads();                              // both buffers are free
            stage(0, 0);
            for (int c = 0; c < nchunks; ++c) {
                if (c + 1 < nchunks) {
                    stage((c + 1) & 1, c + 1);
                    asm volatile("cp.async.wait_group 1;" ::: "memory");
                } else {
                    asm volatile("cp.async.wait_group 0;" ::: "memory");
                }
                __syncthreads();                          // chunk c has landed for everybody
                const int kc = c * kc_len;
                const int nv = min(kc_len, p.k - kc) / VEC;
                const uint4* xs = reinterpret_cast<const uint4*>(smem_x + (c & 1) * FC_X_BYTES);
                if (row0 < p.n) {
                    const uint4* wrow[R];
#pragma unroll
                    for (int r = 0; r < R; ++r)
                        wrow[r] = reinterpret_cast<const uint4*>(static_cast<const uint8_t*>(p.w) +
                                                                 (static_cast<size_t>(min(row0 + r, p.n - 1)) * p.k + kc) * ES);
                    // U vectors per row in flight per lane before any arithmetic: the layer is a stream, and what
                    // streams it at HBM speed is bytes in flight (R x U x 512 B per warp), not issue rate
                    constexpr int U = 8 / R;
                    int v = lane;
                    for (; v + 32 * (U - 1) < nv; v += 32 * U) {
                        uint4 wv[R][U];
#pragma unroll
                        for (int r = 0; r < R; ++r)
#pragma unroll
                            for (int u = 0; u < U; ++u) wv[r][u] = ldg_stream(wrow[r] + v + 32 * u);
#pragma unroll
                        for (int u = 0; u < U; ++u)
#pragma unroll
                            for (int mi = 0; mi < FC_MT; ++mi) {
                                if (mi < mt) {
                                    const uint4 xv = xs[mi * row_vecs + v + 32 * u];
#pragma unroll
                                    for (int r = 0; r < R; ++r) fc_dot<MODE>(acc[mi][r], xv, wv[r][u], p.in_unsigned != 0);
                                }
                            }
                    }
                    if (v < nv) {
                        // the rest of the row (all of it for rows below U x 512 bytes -- MobileNet's fc7, the INT8 heads):
                        // still every load in flight before the first use, each guarded; same per-lane order as above
                        uint4 wv[R][U];
#pragma unroll
                        for (int r = 0; r < R; ++r)
#pragma unroll
                            for (int u = 0; u < U; ++u)
                                wv[r][u] = (v + 32 * u < nv) ? ldg_stream(wrow[r] + v + 32 * u) : make_uint4(0, 0, 0, 0);
#pragma unroll
                        for (int u = 0; u < U; ++u) {
                            if (v + 32 * u < nv) {
#pragma unroll
                                for (int mi = 0; mi < FC_MT; ++mi) {
                                    if (mi < mt) {
                                        const uint4 xv = xs[mi * row_vecs + v + 32 * u];
#pragma unroll
                                        for (int r = 0; r < R; ++r) fc_dot<MODE>(acc[mi][r], xv, wv[r][u], p.in_unsigned != 0);
                                    }
                                }
                            }
                        }
                    }
                }
                __syncthreads();                          // chunk c is consumed: its buffer may be refilled
            }
            // lanes hold partial sums over their k vectors: butterfly, then lane 0 finishes the R x mt outputs
            if (row0 < p.n) {
#pragma unroll
                for (int mi = 0; mi < FC_MT; ++mi)
#pragma unroll
                    for (int r = 0; r < R; ++r) {
                        acc_t a = acc[mi][r];
#pragma unroll
                        for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
                        acc[mi][r] = a;
                    }
                if (lane == 0) {
#pragma unroll
                    for (int mi = 0; mi < FC_MT; ++mi)
#pragma unroll
                        for (int r = 0; r < R; ++r)
                            if (mi < mt && row0 + r < p.n) fc_store<MODE>(p, m0 + mi, row0 + r, acc[mi][r]);
                }
            }
        }
    }
}

template <int MODE, int R>
__global__ void __launch_bounds__(FC_THREADS) fc_stream_kernel(const FcParams p) {
    __shared__ __align__(16) uint8_t smem_x[2 * FC_X_BYTES];
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    asm volatile("griddepcontrol.wait;" ::: "memory");
    fc_body<MODE, R>(p, smem_x, blockIdx.x, gridDim.x);
}

// ------------------------------------------------------------------------------------------------ fused head
// INT8 classifier head: global pooling + inner product in ONE launch, softmax in a second one (instead of three
// dependent launches of 4-8 us each). One CLUSTER of m CTAs per slice of the output neurons: CTA r of a cluster pools
// image r (hw x c bytes, exact packed 16-bit integer sums or byte maxima) into its own shared memory; after one cluster
// barrier every CTA gathers the m pooled rows through distributed shared memory and computes its own neurons for all m
// images -- a warp per neuron, 16 weight bytes per lane and step, dp4a, xor-shuffle fold, then the x86 Saber epilogue
// (acc + bias) * scale. Pooling is repeated by every cluster (m x hw x c bytes from L2 each, ~0.8 MB for ResNet-50):
// cheaper than a grid-wide dependency. Same arithmetic as b200_pool_run -> b200_fc_stream_run, bit for bit.
struct HeadParams {
    const uint8_t* in;    // NHWC [m][hw][c]  u8 | s8
    uint8_t* pooled;      // [m][c]           same dtype (the pooling op's output tensor)
    const int8_t* w;      // [n][c]
    const float* bias;
    const float* scale;
    float* logits;        // [m][ldo]
    int m, hw, c, n, ldo;
    int in_unsigned, pool_max;
    int n_cluster, n_cta; // neurons per cluster / per CTA
};

constexpr int HEAD_THREADS = 512;
constexpr int HEAD_MAX_M = 8;
constexpr int HEAD_MAX_C = 4096;
constexpr int HEAD_LOADS = 16;      // pooling loads in flight per thread (the stage is pure load latency otherwise)
constexpr int HEAD_PRE_ROWS = 2;    // neurons per warp whose weights are fetched before anything else
constexpr int HEAD_PRE_VECS = 4;    // ... when a row is at most 4 x 32 vectors (c <= 2048)

__global__ void __launch_bounds__(HEAD_THREADS) head_pool_fc_kernel(const HeadParams h) {
    extern __shared__ __align__(16) uint8_t head_smem[];
    uint8_t* xs = head_smem;                                      // [c] this CTA's pooled row
    uint8_t* xall = head_smem + h.c;                              // [m][c]
    uint32_t* part = reinterpret_cast<uint32_t*>(xall + static_cast<size_t>(h.m) * h.c);   // [pg][cv][8]
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int rank = static_cast<int>(cluster_ctarank());
    const int cid = blockIdx.x / h.m;
    const int cv = h.c >> 4;                                      // 16-byte vectors per pixel
    const int row_begin = cid * h.n_cluster + rank * h.n_cta;
    const int row_end = min(min(row_begin + h.n_cta, (cid + 1) * h.n_cluster), h.n);
    // The weights do not depend on the previous kernel: the first HEAD_PRE_ROWS neurons of every warp are on their way
    // before the grid dependency resolves (PDL), so their DRAM / L2 latency is off the pool -> gather -> dot chain.
    uint4 wpre[HEAD_PRE_ROWS][HEAD_PRE_VECS];
    const bool prefetched = cv <= 32 * HEAD_PRE_VECS;
    if (prefetched) {
#pragma unroll
        for (int pr = 0; pr < HEAD_PRE_ROWS; ++pr) {
            const int row = row_begin + warp + pr * (HEAD_THREADS / 32);
#pragma unroll
            for (int j = 0; j < HEAD_PRE_VECS; ++j) {
                const int v = lane + 32 * j;
                wpre[pr][j] = (row < row_end && v < cv) ? ldg_stream(reinterpret_cast<const uint4*>(h.w + static_cast<size_t>(row) * h.c) + v)
                                                        : make_uint4(0, 0, 0, 0);
            }
        }
    }
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    asm volatile("griddepcontrol.wait;" ::: "memory");
    const uint32_t flip = h.in_unsigned ? 0u : 0x80808080u;       // s8 -> biased u8
    // ---- 1. pool image `rank`: thread (pg, v) folds pixels pg, pg + PG, ... of channel vector v
    const int PG = HEAD_THREADS / cv > 0 ? HEAD_THREADS / cv : 1;
    for (int v = tid % cv, pg = tid / cv; pg < PG && v < cv; v += HEAD_THREADS) {   // (cv <= 256: one trip)
        const uint4* src = reinterpret_cast<const uint4*>(h.in) + static_cast<size_t>(rank) * h.hw * cv + v;
        uint32_t a[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) a[j] = 0u;
        for (int t0 = pg; t0 < h.hw; t0 += PG * HEAD_LOADS) {
            uint4 y[HEAD_LOADS];
#pragma unroll
            for (int u = 0; u < HEAD_LOADS; ++u) {
                const int t = t0 + u * PG;
                // (a missing pixel contributes the neutral element of both folds: biased 0)
                y[u] = t < h.hw ? __ldg(src + static_cast<size_t>(t) * cv) : make_uint4(flip, flip, flip, flip);
            }
#pragma unroll
            for (int u = 0; u < HEAD_LOADS; ++u) {
                const uint32_t w4[4] = {y[u].x ^ flip, y[u].y ^ flip, y[u].z ^ flip, y[u].w ^ flip};
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    if (h.pool_max) {
                        a[j] = __vmaxu4(a[j], w4[j]);
                    } else {      // bytes 0, 2 and bytes 1, 3 as two pairs of 16-bit lanes (255 * hw < 65536)
                        a[2 * j] += w4[j] & 0x00FF00FFu;
                        a[2 * j + 1] += (w4[j] >> 8) & 0x00FF00FFu;
                    }
                }
            }
        }
        uint32_t* dst = part + (static_cast<size_t>(pg) * cv + v) * 8;
#pragma unroll
        for (int j = 0; j < 8; ++j) dst[j] = a[j];
    }
    __syncthreads();
    for (int v = tid; v < cv; v += HEAD_THREADS) {
        uint32_t a[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) a[j] = 0u;
        for (int pg = 0; pg < PG; ++pg) {
            const uint32_t* src = part + (static_cast<size_t>(pg) * cv + v) * 8;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                if (h.pool_max) { if (j < 4) a[j] = __vmaxu4(a[j], src[j]); }
                else a[j] += src[j];
            }
        }
        uint32_t codes[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            uint32_t wd = 0;
#pragma unroll
            for (int b = 0; b < 4; ++b) {
                uint32_t code;
                if (h.pool_max) {
                    code = ((a[j] >> (8 * b)) & 0xffu) ^ (h.in_unsigned ? 0u : 0x80u);
                } else {
                    // byte b of word j: even bytes live in a[2j], odd ones in a[2j + 1]; low / high 16-bit lane
                    const uint32_t lanes = a[2 * j + (b & 1)];
                    const int32_t sum = static_cast<int32_t>((b & 2) ? (lanes >> 16) : (lanes & 0xffffu)) - (h.in_unsigned ? 0 : 128 * h.hw);
                    // saber_pooling int8: fp32 sum (exact here) / window, rounded to nearest even, saturated
                    const float q = __fdiv_rn(static_cast<float>(sum), static_cast<float>(h.hw));
                    if (h.in_unsigned) asm("cvt.rni.sat.u8.f32 %0, %1;" : "=r"(code) : "f"(q));
                    else { int32_t sc; asm("cvt.rni.sat.s8.f32 %0, %1;" : "=r"(sc) : "f"(q)); code = static_cast<uint32_t>(sc) & 0xffu; }
                }
                wd |= code << (8 * b);
            }
            codes[j] = wd;
        }
        const uint4 cq = make_uint4(codes[0], codes[1], codes[2], codes[3]);
        reinterpret_cast<uint4*>(xs)[v] = cq;
        if (cid == 0) reinterpret_cast<uint4*>(h.pooled + static_cast<size_t>(rank) * h.c)[v] = cq;   // the pooling op's tensor
    }
    // ---- 2. every CTA of the cluster gathers the m pooled rows
    cluster_sync_all();
    {
        const uint32_t xs_sa = smem_u32(xs);
        for (int i = tid; i < h.m * cv; i += HEAD_THREADS) {
            const int mi = i / cv, v = i - mi * cv;
            uint4 t;
            const uint32_t ra = map_to_cta(xs_sa + v * 16, mi);
            asm volatile("ld.shared::cluster.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(t.x), "=r"(t.y), "=r"(t.z), "=r"(t.w) : "r"(ra));
            reinterpret_cast<uint4*>(xall)[i] = t;
        }
    }
    cluster_sync_all();       // nobody's pooled row is read after this: CTAs may finish at their own pace
    // ---- 3. this CTA's neurons: a warp each, all m images at once
    int pr_idx = 0;
    for (int row = row_begin + warp; row < row_end; row += HEAD_THREADS / 32, ++pr_idx) {
        const uint4* wr = reinterpret_cast<const uint4*>(h.w + static_cast<size_t>(row) * h.c);
        int acc[HEAD_MAX_M];
#pragma unroll
        for (int mi = 0; mi < HEAD_MAX_M; ++mi) acc[mi] = 0;
        // all weight vectors of the neuron in flight at once (cv <= 256: at most 8 per lane); the first rows of the warp
        // were fetched at kernel entry
        uint4 wvs[HEAD_MAX_C / 16 / 32];
        const bool pre = prefetched && pr_idx < HEAD_PRE_ROWS;
#pragma unroll
        for (int j = 0; j < HEAD_MAX_C / 16 / 32; ++j) {
            const int v = lane + 32 * j;
            if (pre) wvs[j] = j < HEAD_PRE_VECS ? (pr_idx == 0 ? wpre[0][j < HEAD_PRE_VECS ? j : 0] : wpre[1][j < HEAD_PRE_VECS ? j : 0]) : make_uint4(0, 0, 0, 0);
            else wvs[j] = v < cv ? ldg_stream(wr + v) : make_uint4(0, 0, 0, 0);
        }
#pragma unroll
        for (int j = 0; j < HEAD_MAX_C / 16 / 32; ++j) {
            const int v = lane + 32 * j;
            if (v >= cv) break;
            const uint4 wv = wvs[j];
#pragma unroll
            for (int mi = 0; mi < HEAD_MAX_M; ++mi) {
                if (mi < h.m) {
                    const uint4 xv = reinterpret_cast<const uint4*>(xall)[mi * cv + v];
                    int a = acc[mi];
                    if (h.in_unsigned) {
                        a = dp4a_us(xv.x, wv.x, a); a = dp4a_us(xv.y, wv.y, a); a = dp4a_us(xv.z, wv.z, a); a = dp4a_us(xv.w, wv.w, a);
                    } else {
                        a = dp4a_ss(xv.x, wv.x, a); a = dp4a_ss(xv.y, wv.y, a); a = dp4a_ss(xv.z, wv.z, a); a = dp4a_ss(xv.w, wv.w, a);
                    }
                    acc[mi] = a;
                }
            }
        }
#pragma unroll
        for (int mi = 0; mi < HEAD_MAX_M; ++mi) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) acc[mi] += __shfl_xor_sync(0xffffffffu, acc[mi], o);
        }
        // x86 Saber int8 epilogue, as epilogue16_i8 of the conv kernels: add, then multiply, each rounded
        const float bs = h.bias ? __ldg(h.bias + row) : 0.f, sc = h.scale ? __ldg(h.scale + row) : 1.f;
#pragma unroll
        for (int mi = 0; mi < HEAD_MAX_M; ++mi)
            if (mi < h.m && lane == mi) h.logits[static_cast<size_t>(mi) * h.ldo + row] = __fmul_rn(__fadd_rn(__int2float_rn(acc[mi]), bs), sc);
    }
}

static int fc_mode(int math) { return math == B200_MATH_I8 ? 0 : (math == B200_MATH_F16 ? 1 : 2); }

// rows per warp: two CTAs per SM first (bytes in flight), then fewer input re-stagings
static int fc_rows_per_warp(int n) {
    const int sms = sm_count();
    if (n >= FC_WARPS * 4 * 2 * sms) return 4;
    if (n >= FC_WARPS * 2 * 2 * sms) return 2;
    return 1;
}

template <int MODE>
static void launch_fc(const FcParams& p, int r, unsigned grid, cudaStream_t stream) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(FC_THREADS);
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    if (r == 4) cudaLaunchKernelEx(&cfg, fc_stream_kernel<MODE, 4>, p);
    else if (r == 2) cudaLaunchKernelEx(&cfg, fc_stream_kernel<MODE, 2>, p);
    else cudaLaunchKernelEx(&cfg, fc_stream_kernel<MODE, 1>, p);
}

static bool fc_args_ok(const b200_fc_stream_desc_t* d) {
    if (!d || d->m <= 0 || d->k <= 0 || d->n_out <= 0 || d->ldx < d->k || d->ldo < d->n_out) return false;
    const int es = d->math == B200_MATH_I8 ? 1 : (d->math == B200_MATH_F16 ? 2 : 4);
    if ((static_cast<int64_t>(d->k) * es) % 16 != 0 || (static_cast<int64_t>(d->ldx) * es) % 16 != 0) return false;
    if (d->math == B200_MATH_I8 && !(d->in_dtype == B200_INT8 || d->in_dtype == B200_UINT8)) return false;
    if (d->math == B200_MATH_F16 && d->in_dtype != B200_HALF) return false;
    if ((d->math == B200_MATH_TF32 || d->math == B200_MATH_TF32X3) && d->in_dtype != B200_FLOAT) return false;
    return true;
}

static FcParams make_fc_params(const b200_fc_stream_desc_t* d, const void* x, const void* w, const float* bias, const float* scale,
                               void* out) {
    FcParams p{};
    p.x = x; p.w = w; p.bias = bias; p.scale = scale; p.out = out;
    p.m = d->m; p.k = d->k; p.n = d->n_out; p.ldx = d->ldx; p.ldo = d->ldo;
    p.in_unsigned = d->in_dtype == B200_UINT8 ? 1 : 0;
    p.out_dtype = d->out_dtype;
    p.relu = d->relu; p.neg_slope = d->neg_slope;
    return p;
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200_fc_stream_max_rows(void) { return 2 * FC_MT; }

int b200_fc_stream_run(const b200_fc_stream_desc_t* d, const void* x, const void* w_plain, const float* bias, const float* scale,
                       void* out, void* stream) {
    if (!fc_args_ok(d) || !x || !w_plain || !out) return B200_INVALID_VALUE;
    if (!device_is_sm90()) return B200_WRONG_DEVICE;
    const FcParams p = make_fc_params(d, x, w_plain, bias, scale, out);
    const int r = fc_rows_per_warp(p.n);
    const int nblocks = (p.n + FC_WARPS * r - 1) / (FC_WARPS * r);
    static const int grid_mult = [] { const char* e = getenv("B200_FC_GRID_MULT"); const int v = e ? atoi(e) : 0; return v > 0 ? v : 4; }();
    const unsigned grid = static_cast<unsigned>(nblocks < grid_mult * sm_count() ? nblocks : grid_mult * sm_count());
    const int mode = fc_mode(d->math);
    if (mode == 0) launch_fc<0>(p, r, grid, static_cast<cudaStream_t>(stream));
    else if (mode == 1) launch_fc<1>(p, r, grid, static_cast<cudaStream_t>(stream));
    else launch_fc<2>(p, r, grid, static_cast<cudaStream_t>(stream));
    count_launch();
    cudaError_t e = cudaPeekAtLastError();
    if (e != cudaSuccess) {
        fprintf(stderr, "[b200_saber] fc_stream launch failed: %s\n", cudaGetErrorString(e));
        return B200_UNKNOWN_ERROR;
    }
    return B200_SUCCESS;
}

size_t b200_head_workspace_bytes(const b200_head_desc_t* hd) {
    (void)hd;
    return 16;      // (kept for the ABI: the two-launch head needs no scratch)
}

int b200_head_run(const b200_head_desc_t* hd, const void* in, void* pooled, const void* w_plain, const float* bias,
                  const float* scale, void* logits, float* prob, void* workspace, void* stream) {
    (void)workspace;
    if (!hd || !in || !pooled || !w_plain || !logits) return B200_INVALID_VALUE;
    const b200_fc_stream_desc_t* d = &hd->fc;
    if (!fc_args_ok(d) || hd->hw <= 0 || d->ldx != d->k) return B200_INVALID_VALUE;
    // int8 nets only (float heads keep the three separate ops), fp32 logits out, at most 8 rows = one cluster
    if (d->math != B200_MATH_I8 || d->out_dtype != B200_FLOAT || d->m > HEAD_MAX_M || d->relu || d->k > HEAD_MAX_C ||
        (!hd->pool_max && hd->hw > 256))
        return B200_UNIMPL_ERROR;
    if (!device_is_sm90()) return B200_WRONG_DEVICE;
    HeadParams h{};
    h.in = static_cast<const uint8_t*>(in);
    h.pooled = static_cast<uint8_t*>(pooled);
    h.w = static_cast<const int8_t*>(w_plain);
    h.bias = bias; h.scale = scale;
    h.logits = static_cast<float*>(logits);
    h.m = d->m; h.hw = hd->hw; h.c = d->k; h.n = d->n_out; h.ldo = d->ldo;
    h.in_unsigned = d->in_dtype == B200_UINT8 ? 1 : 0;
    h.pool_max = hd->pool_max;
    // Every cluster pools all m images again, and clusters that read the same lines at the same time queue up at the L2
    // slices (18 clusters: 15 us; tools/bench_head.py): as few clusters as keep a CTA's weight slice around 64 KB
    int clusters = static_cast<int>((static_cast<int64_t>(d->n_out) * d->k + static_cast<int64_t>(d->m) * 65536 - 1) /
                                    (static_cast<int64_t>(d->m) * 65536));
    if (const char* e = getenv("B200_HEAD_CLUSTERS")) { if (atoi(e) > 0) clusters = atoi(e); }   // tuning experiments only
    if (clusters > sm_count() / d->m) clusters = sm_count() / d->m;
    if (clusters < 1) clusters = 1;
    if (clusters > d->n_out) clusters = d->n_out;
    h.n_cluster = (d->n_out + clusters - 1) / clusters;
    clusters = (d->n_out + h.n_cluster - 1) / h.n_cluster;
    h.n_cta = (h.n_cluster + d->m - 1) / d->m;
    const int cv = d->k / 16;
    const int pg = HEAD_THREADS / cv > 0 ? HEAD_THREADS / cv : 1;
    const size_t smem = static_cast<size_t>(d->k) * (1 + d->m) + static_cast<size_t>(pg) * cv * 32;
    static std::atomic<bool> opted_in[64];
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev >= 0 && dev < 64 && !opted_in[dev].load(std::memory_order_acquire)) {
        cudaFuncSetAttribute(head_pool_fc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
        opted_in[dev].store(true, std::memory_order_release);
    }
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(static_cast<unsigned>(clusters * d->m));
    cfg.blockDim = dim3(HEAD_THREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = static_cast<cudaStream_t>(stream);
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
    attr[1].id = cudaLaunchAttributeClusterDimension;
    attr[1].val.clusterDim.x = static_cast<unsigned>(d->m);
    attr[1].val.clusterDim.y = 1;
    attr[1].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 2;
    cudaError_t e = cudaLaunchKernelEx(&cfg, head_pool_fc_kernel, h);
    count_launch();
    if (e == cudaSuccess) e = cudaPeekAtLastError();
    if (e != cudaSuccess) {
        fprintf(stderr, "[b200_saber] head launch failed: %s\n", cudaGetErrorString(e));
        return B200_UNKNOWN_ERROR;
    }
    if (prob != nullptr) return b200_softmax_rows(h.logits, prob, d->m, d->n_out, d->ldo, hd->ldp, stream);
    return B200_SUCCESS;
}

}  // extern "C"
