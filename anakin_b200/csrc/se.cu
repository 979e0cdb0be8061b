// Squeeze-and-excitation blocks (SENet): the Axpy operator and the fused excitation gate. include/b200_saber.h has the
// contracts; oracle restatements: tests/se_oracle.py.
//
//   b200_axpy_run     out = act(g[n,c] * x + y) over NHWC           reference saber_axpy.cu:9-16 (fp32), + fp16 / int8
//   b200_se_gate_run  g = sigmoid(W2 relu(W1 mean_hw(x) + b1) + b2)  the reference's Pooling -> Convolution -> ReLU ->
//                                                                    Convolution -> Activation(Sigmoid) chain, one launch
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
constexpr int kWarps = kThreads / 32;
constexpr int kAxpyVecsPerThread = 4;
constexpr int kGateCluster = 8;   // CTAs of the cluster that runs the two inner products

// ------------------------------------------------------------------ Axpy
struct AxpyP {
    int hw, c, ld, ldg;      // pixels per image, real channels, stored channels of x / y / out, gate row pitch
    int gate_half;           // gate stored as f16 (an FP16 net whose gate chain is not fused)
    int relu;
    float neg_slope, ay;     // ay: 8-bit y factor (see b200_axpy_desc_t)
    float ax;
    int y_unsigned, out_unsigned;
};

// Grid (vector blocks, n). The gate row of image blockIdx.y (times ax for the 8-bit kinds) is staged once per CTA.
template <int KX>
__global__ void __launch_bounds__(kThreads) axpy_kernel(const void* __restrict__ gate, const uint4* __restrict__ x,
                                                        const uint4* __restrict__ y, uint4* __restrict__ out, AxpyP p) {
    constexpr int L = vec_lanes<KX>;
    constexpr bool kQ8 = KX >= VK_S8;
    extern __shared__ float gs[];
    pdl_enter();
    const int n = blockIdx.y;
    for (int c = threadIdx.x; c < p.ld; c += kThreads) {
        float g = 0.f;
        if (c < p.c) {
            g = p.gate_half ? __half2float(static_cast<const __half*>(gate)[static_cast<long long>(n) * p.ldg + c])
                            : static_cast<const float*>(gate)[static_cast<long long>(n) * p.ldg + c];
            if (kQ8) g = __fmul_rn(g, p.ax);
        }
        gs[c] = g;
    }
    __syncthreads();
    const int nv = p.ld / L;
    const long long per_image = static_cast<long long>(p.hw) * nv;
    const long long base = static_cast<long long>(n) * per_image;
    const long long v0 = static_cast<long long>(blockIdx.x) * kThreads * kAxpyVecsPerThread + threadIdx.x;
#pragma unroll
    for (int it = 0; it < kAxpyVecsPerThread; ++it) {
        const long long v = v0 + static_cast<long long>(it) * kThreads;
        if (v >= per_image) break;
        const int c0 = static_cast<int>(v % nv) * L;
        float fx[L], fy[L];
        unpack_vec<KX>(__ldg(x + base + v), fx);
        const uint4 yv = __ldg(y + base + v);
        if constexpr (kQ8) {
            if (p.y_unsigned) unpack_vec<VK_U8>(yv, fy);
            else unpack_vec<VK_S8>(yv, fy);
        } else {
            unpack_vec<KX>(yv, fy);
        }
        float r[L];
#pragma unroll
        for (int j = 0; j < L; ++j) {
            float t;
            if constexpr (kQ8) {
                // (g * ax) * qx + qy * ay, each product and the sum rounded on its own
                t = __fadd_rn(__fmul_rn(gs[c0 + j], fx[j]), __fmul_rn(fy[j], p.ay));
                if (p.relu) t = t > 0.f ? t : 0.f;
            } else {
                t = __fmaf_rn(gs[c0 + j], fx[j], fy[j]);
                if (p.relu) t = t > 0.f ? t : __fmul_rn(t, p.neg_slope);
            }
            r[j] = c0 + j < p.c ? t : 0.f;
        }
        out[base + v] = pack_vec<KX>(r, p.out_unsigned);
    }
}

// ------------------------------------------------------------------ SE gate
// fp32 sigmoid by an explicit sequence (every step rounded on its own, no library call): e = exp(-|z|) by a
// Cody-Waite reduction and a degree-7 Taylor polynomial on |r| <= ln2/2, scaled by 2^k in one or two exact-or-final
// multiplies; sigmoid = 1 / (1 + e) for z >= 0, e / (1 + e) otherwise.
// The constants are given by their bits (float32 nearest to 1/7!, ..., 1/3!, log2(e), and the split ln2 = C1 + C2).
__device__ __forceinline__ float se_sigmoid(float z) {
    const float a = fminf(fabsf(z), 126.f);
    const float t = -a;
    const float k = rintf(__fmul_rn(t, __int_as_float(0x3fb8aa3b)));
    float r = __fsub_rn(t, __fmul_rn(k, __int_as_float(0x3f318000)));
    r = __fsub_rn(r, __fmul_rn(k, __int_as_float(0xb95e8083)));
    float q = __int_as_float(0x39500d01);
    q = __fadd_rn(__fmul_rn(q, r), __int_as_float(0x3ab60b61));
    q = __fadd_rn(__fmul_rn(q, r), __int_as_float(0x3c088889));
    q = __fadd_rn(__fmul_rn(q, r), __int_as_float(0x3d2aaaab));
    q = __fadd_rn(__fmul_rn(q, r), __int_as_float(0x3e2aaaab));
    q = __fadd_rn(__fmul_rn(q, r), 0.5f);
    q = __fadd_rn(__fmul_rn(q, r), 1.f);
    q = __fadd_rn(__fmul_rn(q, r), 1.f);
    const int ki = static_cast<int>(k);
    float e;
    if (ki >= -126) e = __fmul_rn(q, __int_as_float((ki + 127) << 23));
    else e = __fmul_rn(__fmul_rn(q, __int_as_float((ki + 64 + 127) << 23)), __int_as_float(0x1f800000));   // 2^-64
    const float den = __fadd_rn(1.f, e);
    return z >= 0.f ? __fdiv_rn(1.f, den) : __fdiv_rn(e, den);
}

struct GateP {
    int n, hw, c, ld, r, ldg;
    int chunk;               // pixels pooled by one CTA of a cluster
    float scale;             // 8-bit input: edge scale
    int w2_vec;              // W2 rows can be read as float4 (r % 4 == 0, 16-byte aligned)
};

// Workspace: part [n][kGateCluster][c] (int32 or fp32 partial sums), hidden [n][r] (fp32).
struct GateWs {
    void* part;
    float* hidden;
};

// One cluster of kGateCluster CTAs per image (images strided over the clusters of the grid). Per image: every CTA pools
// an eighth of the pixels; after a cluster barrier every CTA forms the whole mean vector from the eight partial sums (in
// rank order) in its shared memory; the cluster's 64 warps share the squeeze rows, its 2048 threads the excitation
// outputs, with one more barrier between the two. No CTA waits for another cluster.
template <int K>
__global__ void __launch_bounds__(kThreads) se_gate_kernel(const uint4* __restrict__ x, const float* __restrict__ w1,
                                                            const float* __restrict__ b1, const float* __restrict__ w2,
                                                            const float* __restrict__ b2, float* __restrict__ gate,
                                                            GateWs ws, GateP p) {
    constexpr int L = vec_lanes<K>;
    constexpr bool kQ8 = K >= VK_S8;
    typedef typename std::conditional<kQ8, int, float>::type Acc;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    Acc* red = reinterpret_cast<Acc*>(smem_raw);           // pooling: [slots][ld]
    float* mean = reinterpret_cast<float*>(smem_raw);      // then: mean [c], hidden [r]
    float* hid = mean + p.c;
    pdl_enter();

    const int rank = static_cast<int>(cluster_ctarank());
    const int clusters = gridDim.x / kGateCluster;
    const int lane = threadIdx.x & 31;
    const int gwarp = rank * kWarps + (threadIdx.x >> 5);
    const int gtid = rank * kThreads + threadIdx.x;
    const int nv = p.ld / L;
    const int slots = nv >= kThreads ? 1 : kThreads / nv;
    const int s = nv >= kThreads ? 0 : threadIdx.x / nv;
    const int vb = nv >= kThreads ? threadIdx.x : threadIdx.x % nv;
    const bool active = nv >= kThreads || threadIdx.x < slots * nv;
    for (int img = blockIdx.x / kGateCluster; img < p.n; img += clusters) {
        // ---- 1. this CTA's pixels [px0, px1): exact integer sums (8-bit) or fixed-order fp32 sums (float kinds)
        const int px0 = min(rank * p.chunk, p.hw), px1 = min(px0 + p.chunk, p.hw);
        const uint4* xi = x + static_cast<long long>(img) * p.hw * nv;
        for (int v = vb; active && v < nv; v += (nv >= kThreads ? kThreads : nv)) {
            Acc acc[L];
#pragma unroll
            for (int j = 0; j < L; ++j) acc[j] = 0;
            for (int px = px0 + s; px < px1; px += slots) {
                float f[L];
                unpack_vec<K>(__ldg(xi + static_cast<long long>(px) * nv + v), f);
#pragma unroll
                for (int j = 0; j < L; ++j) {
                    if constexpr (kQ8) acc[j] += static_cast<int>(f[j]);
                    else acc[j] = __fadd_rn(acc[j], f[j]);
                }
            }
#pragma unroll
            for (int j = 0; j < L; ++j) red[s * p.ld + v * L + j] = acc[j];
        }
        __syncthreads();
        Acc* part = static_cast<Acc*>(ws.part) + static_cast<long long>(img) * kGateCluster * p.c;
        for (int c = threadIdx.x; c < p.c; c += kThreads) {
            Acc t = red[c];
            for (int q = 1; q < slots; ++q) {
                if constexpr (kQ8) t += red[q * p.ld + c];
                else t = __fadd_rn(t, red[q * p.ld + c]);
            }
            part[rank * p.c + c] = t;
        }
        __threadfence();
        cluster_sync_all();

        // ---- 2. mean: the eight partials in rank order (written by peers: read through L2); 8-bit:
        //         ((float)S * scale [* 127/255]) / hw in fp32 steps
        for (int c = threadIdx.x; c < p.c; c += kThreads) {
            Acc t = __ldcg(part + c);
#pragma unroll
            for (int q = 1; q < kGateCluster; ++q) {
                if constexpr (kQ8) t += __ldcg(part + q * p.c + c);
                else t = __fadd_rn(t, __ldcg(part + q * p.c + c));
            }
            float m;
            if constexpr (kQ8) {
                m = __fmul_rn(static_cast<float>(t), p.scale);
                if constexpr (K == VK_U8) m = __fmul_rn(m, static_cast<float>(127.0 / 255.0));
            } else {
                m = t;
            }
            mean[c] = __fdiv_rn(m, static_cast<float>(p.hw));
        }
        __syncthreads();

        // ---- 3. squeeze: hidden[j] = relu(b1[j] + W1[j] . mean); one warp per j, lane l sums c = l, l+32, ... in
        //         order, then a butterfly over the 32 lane sums (xor 16, 8, 4, 2, 1)
        float* hg = ws.hidden + static_cast<long long>(img) * p.r;
        for (int j = gwarp; j < p.r; j += kGateCluster * kWarps) {
            const float* wr = w1 + static_cast<long long>(j) * p.c;
            float sum = 0.f;
#pragma unroll 16
            for (int c = lane; c < p.c; c += 32) sum = __fadd_rn(sum, __fmul_rn(__ldg(wr + c), mean[c]));
#pragma unroll
            for (int o = 16; o >= 1; o >>= 1) sum = __fadd_rn(sum, __shfl_xor_sync(0xffffffffu, sum, o));
            if (lane == 0) {
                const float h = __fadd_rn(sum, __ldg(b1 + j));
                hg[j] = h > 0.f ? h : 0.f;
            }
        }
        __threadfence();
        cluster_sync_all();

        // ---- 4. excitation: g[c] = sigmoid(b2[c] + W2[c] . hidden), the dot product summed k = 0, 1, ... in order
        for (int k = threadIdx.x; k < p.r; k += kThreads) hid[k] = __ldcg(hg + k);
        __syncthreads();
        for (int c = gtid; c < p.c; c += kGateCluster * kThreads) {
            const float* wr = w2 + static_cast<long long>(c) * p.r;
            float sum = 0.f;
            if (p.w2_vec) {
#pragma unroll 8
                for (int k = 0; k < p.r; k += 4) {
                    const float4 w = __ldg(reinterpret_cast<const float4*>(wr + k));
                    sum = __fadd_rn(sum, __fmul_rn(w.x, hid[k]));
                    sum = __fadd_rn(sum, __fmul_rn(w.y, hid[k + 1]));
                    sum = __fadd_rn(sum, __fmul_rn(w.z, hid[k + 2]));
                    sum = __fadd_rn(sum, __fmul_rn(w.w, hid[k + 3]));
                }
            } else {
                for (int k = 0; k < p.r; ++k) sum = __fadd_rn(sum, __fmul_rn(__ldg(wr + k), hid[k]));
            }
            gate[static_cast<long long>(img) * p.ldg + c] = se_sigmoid(__fadd_rn(sum, __ldg(b2 + c)));
        }
        __syncthreads();      // the next image's pooling reuses this CTA's shared memory
    }
}

size_t align256(size_t b) { return (b + 255) / 256 * 256; }

// Shared memory of the gate kernel: the pooling slots, then (reused) the mean vector and the hidden activations.
size_t gate_smem_bytes(const b200_se_gate_desc_t* d) {
    const int L = d->dtype == B200_FLOAT ? 4 : (d->dtype == B200_HALF ? 8 : 16);
    const int nv = d->ld / L;
    const int slots = nv >= kThreads ? 1 : kThreads / nv;
    return std::max(static_cast<size_t>(slots) * d->ld, static_cast<size_t>(d->c) + d->r) * 4;
}
constexpr size_t kGateSmemMax = 200 * 1024;

bool gate_desc_ok(const b200_se_gate_desc_t* d) {
    if (!d || d->n < 1 || d->hw < 1 || d->c < 1 || d->r < 1 || d->ld < d->c || d->ldg < d->c) return false;
    if (d->hw > (1 << 24) / 255) return false;   // 8-bit sums stay exact in an fp32 (and in an int32)
    const int es = d->dtype == B200_FLOAT ? 4 : (d->dtype == B200_HALF ? 2 : 1);
    if (d->dtype != B200_FLOAT && d->dtype != B200_HALF && d->dtype != B200_INT8 && d->dtype != B200_UINT8) return false;
    if ((static_cast<long long>(d->ld) * es) % 16 != 0) return false;
    return gate_smem_bytes(d) <= kGateSmemMax;
}

}  // namespace

}  // namespace b200

using namespace b200;

extern "C" {

int b200_axpy_run(const b200_axpy_desc_t* d, const void* gate, const void* x, const void* y, void* out, void* stream) {
    if (!d || !gate || !x || !y || !out || d->n < 1 || d->hw < 1 || d->c < 1 || d->ld < d->c || d->ldg < d->c)
        return B200_INVALID_VALUE;
    if (d->gate_dtype != B200_FLOAT && d->gate_dtype != B200_HALF) return B200_INVALID_VALUE;
    const bool q8 = d->x_dtype == B200_INT8 || d->x_dtype == B200_UINT8;
    if (q8) {
        const bool ok = (d->y_dtype == B200_INT8 || d->y_dtype == B200_UINT8) &&
                        (d->out_dtype == B200_INT8 || d->out_dtype == B200_UINT8);
        if (!ok) return B200_UNIMPL_ERROR;
    } else if (d->y_dtype != d->x_dtype || d->out_dtype != d->x_dtype ||
               (d->x_dtype != B200_FLOAT && d->x_dtype != B200_HALF)) {
        return B200_UNIMPL_ERROR;
    }
    if (!device_is_sm90()) return B200_WRONG_DEVICE;
    AxpyP p;
    p.hw = d->hw; p.c = d->c; p.ld = d->ld; p.ldg = d->ldg;
    p.gate_half = d->gate_dtype == B200_HALF;
    p.relu = d->relu; p.neg_slope = d->neg_slope;
    p.ax = d->ax; p.ay = d->ay;
    p.y_unsigned = d->y_dtype == B200_UINT8; p.out_unsigned = d->out_dtype == B200_UINT8;
    const size_t smem = static_cast<size_t>(d->ld) * sizeof(float);
    return with_vec_kind(d->x_dtype, [&](auto kind) -> int {
        constexpr int K = decltype(kind)::value;
        if (d->ld % vec_lanes<K>) return B200_INVALID_VALUE;
        const long long per_image = static_cast<long long>(d->hw) * (d->ld / vec_lanes<K>);
        const long long blocks = (per_image + kThreads * kAxpyVecsPerThread - 1) / (kThreads * kAxpyVecsPerThread);
        if (blocks > 0x7fffffffll || d->n > 65535 || smem > 48 * 1024) return B200_INVALID_VALUE;
        return launch("axpy", Pdl::On, axpy_kernel<K>, dim3(static_cast<unsigned>(blocks), d->n), dim3(kThreads), smem,
                      stream, dim3(1), gate, static_cast<const uint4*>(x), static_cast<const uint4*>(y),
                      static_cast<uint4*>(out), p);
    });
}

size_t b200_se_gate_workspace_bytes(const b200_se_gate_desc_t* d) {
    if (!gate_desc_ok(d)) return 0;
    return align256(static_cast<size_t>(d->n) * kGateCluster * d->c * 4) + align256(static_cast<size_t>(d->n) * d->r * 4);
}

int b200_se_gate_run(const b200_se_gate_desc_t* d, const void* x, const float* w1, const float* b1, const float* w2,
                     const float* b2, float* gate, void* workspace, void* stream) {
    if (!gate_desc_ok(d) || !x || !w1 || !b1 || !w2 || !b2 || !gate || !workspace) return B200_INVALID_VALUE;
    if (!device_is_sm90()) return B200_WRONG_DEVICE;
    GateP p;
    p.n = d->n; p.hw = d->hw; p.c = d->c; p.ld = d->ld; p.r = d->r; p.ldg = d->ldg; p.scale = d->scale;
    p.chunk = (d->hw + kGateCluster - 1) / kGateCluster;
    p.w2_vec = d->r % 4 == 0 && (reinterpret_cast<uintptr_t>(w2) & 15u) == 0;
    // one cluster per image, at most as many clusters as fit the SMs once
    const int clusters = std::max(1, std::min<int>(d->n, sm_count() / kGateCluster));
    char* w = static_cast<char*>(workspace);
    GateWs ws;
    ws.part = w;
    ws.hidden = reinterpret_cast<float*>(w + align256(static_cast<size_t>(d->n) * kGateCluster * d->c * 4));
    const size_t smem = gate_smem_bytes(d);
    return with_vec_kind(d->dtype, [&](auto kind) -> int {
        constexpr int K = decltype(kind)::value;
        opt_in_smem<se_gate_kernel<K>>(static_cast<int>(kGateSmemMax));
        return launch("se_gate", Pdl::On, se_gate_kernel<K>, dim3(static_cast<unsigned>(clusters * kGateCluster)),
                      dim3(kThreads), smem, stream, dim3(kGateCluster), static_cast<const uint4*>(x), w1, b1, w2, b2, gate,
                      ws, p);
    });
}

}  // extern "C"
