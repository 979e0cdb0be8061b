// INT8 calibration statistics on the GPU (include/b200_saber.h has the contract).
//
// Replaces (reference): the host loops of framework/core/net/entropy_calibrator.cpp -- get_max_values / get_histgrams
// (the max |x| and the 2048-bin histogram of |x| of every edge tensor) and get_kl_threshold:300-346 with
// get_ref_q / expand_to_q / get_kl_divergence:24-130 -- as restated, with the arg-min the reference meant, by
// anakin_b200/calibrate.py::kl_threshold. The statistics kernel runs right behind each producer inside the Net's
// captured prediction; the threshold search runs once over all histograms.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/b200_saber.h"
#include "common.cuh"
#include "ptx.cuh"

namespace b200 {

namespace {

constexpr int kBins = B200_CALIB_BINS;
constexpr int kLevels = 128;                // quantised levels of the KL search (QUANT_LEVELS)
constexpr int kFirstCandidate = kLevels + 1;
constexpr int kStatsThreads = 256;
constexpr int kStatsVecPerThread = 16;      // float4 loads per thread before another CTA is worth its flush
constexpr int kKlWarps = 16;
constexpr int kPairwiseBlock = 128;         // numpy's PW_BLOCKSIZE

__device__ __forceinline__ double inf_f64() { return __longlong_as_double(0x7ff0000000000000ll); }

// ------------------------------------------------------------------------------------------------ edge statistics
// Element e of the [rows][ld] tensor counts when its column e % ld is below c (PADDED), else always.
template <bool PADDED>
__device__ __forceinline__ bool counts(long long e, int c, int ld) {
    if constexpr (PADDED) return static_cast<int>(e % ld) < c;
    else return true;
}

// |x| bin of the histogram: numpy's (|x| / step).astype(int64) clipped to kBins - 1, step = max / kBins, with the
// division correctly rounded in fp32 (no reciprocal).
__device__ __forceinline__ int bin_of(float v, float step) {
    const float q = __fdiv_rn(fabsf(v), step);
    return q >= static_cast<float>(kBins - 1) ? kBins - 1 : static_cast<int>(q);
}

// One pass over a tensor, the mode word chooses the statistic: 0 folds max |x| into *max_bits (non-negative floats
// order like their bit patterns), 1 adds |x| to the slot's bins. Every thread of a CTA runs the same number of loop
// trips (warp ballots below); VEC: 16-byte loads (x 16-byte aligned, ld % 4 == 0).
template <bool PADDED, bool VEC>
__global__ void __launch_bounds__(kStatsThreads) calib_stats_kernel(const float* __restrict__ x, long long count,
                                                                    int c, int ld, const int32_t* __restrict__ mode,
                                                                    uint32_t* __restrict__ max_bits,
                                                                    unsigned long long* __restrict__ hist) {
    __shared__ uint32_t sbins[kBins];
    __shared__ uint32_t smax[kStatsThreads / 32];
    pdl_enter();      // the producer of x has finished
    const int m = *mode;
    if (m != 0 && m != 1) return;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long items = VEC ? count / 4 : count;
    const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
    float step = 0.f;
    if (m == 1) {
        const uint32_t mx = *max_bits;
        if (mx == 0) return;    // max <= 0: no histogram (the host skips such a tensor)
        step = __fdiv_rn(__uint_as_float(mx), static_cast<float>(kBins));
        for (int b = threadIdx.x; b < kBins; b += blockDim.x) sbins[b] = 0;
        __syncthreads();
    }
    uint32_t best = 0;
    for (long long base = static_cast<long long>(blockIdx.x) * blockDim.x; base < items; base += stride) {
        const long long i = base + threadIdx.x;
        const bool in = i < items;
        float v[4] = {0.f, 0.f, 0.f, 0.f};
        bool ok[4] = {false, false, false, false};
        if constexpr (VEC) {
            if (in) {
                const float4 f = __ldg(reinterpret_cast<const float4*>(x) + i);
                v[0] = f.x; v[1] = f.y; v[2] = f.z; v[3] = f.w;
#pragma unroll
                for (int j = 0; j < 4; ++j) ok[j] = counts<PADDED>(4 * i + j, c, ld);
            }
        } else {
            if (in) { v[0] = __ldg(x + i); ok[0] = counts<PADDED>(i, c, ld); }
        }
#pragma unroll
        for (int j = 0; j < (VEC ? 4 : 1); ++j) {
            if (m == 0) {
                if (ok[j]) best = max(best, __float_as_uint(v[j]) & 0x7fffffffu);
            } else {
                const int b = ok[j] ? bin_of(v[j], step) : -1;
                // bin 0 holds most of a post-ReLU tensor: one shared atomic per warp for it
                const uint32_t zeros = __ballot_sync(0xffffffffu, b == 0);
                if (lane == 0 && zeros) atomicAdd(&sbins[0], static_cast<uint32_t>(__popc(zeros)));
                if (b > 0) atomicAdd(&sbins[b], 1u);
            }
        }
    }
    if (m == 0) {
        best = __reduce_max_sync(0xffffffffu, best);
        if (lane == 0) smax[warp] = best;
        __syncthreads();
        if (threadIdx.x == 0) {
            for (int w = 1; w < kStatsThreads / 32; ++w) best = max(best, smax[w]);
            if (best) atomicMax(max_bits, best);
        }
        return;
    }
    __syncthreads();
    for (int b = threadIdx.x; b < kBins; b += blockDim.x)
        if (sbins[b]) atomicAdd(hist + b, static_cast<unsigned long long>(sbins[b]));
}

// ------------------------------------------------------------------------------------------------ KL search
// Shared memory of one CTA (one histogram): prefix sums of the counts and of the empty bins, and per warp the expanded
// distribution q of its current candidate, the 128 quantised counts and their spreading denominators.
struct KlShared {
    long long prefix[kBins + 1];       // prefix[m] = hist[0] + ... + hist[m - 1]
    int zeros[kBins + 1];              // zeros[m] = number of empty bins among hist[0 .. m - 1]
    float q[kKlWarps][kBins];
    float ref_q[kKlWarps][kLevels];
    float dis[kKlWarps][kLevels];
    float leaf[kKlWarps][32];
    double best_kl[kKlWarps];
    int best_i[kKlWarps];
};

// The clipped distribution of candidate i: ref_p[k] = hist[k + 1], its last bin (k = i - 1) also holds every count
// beyond bin i (`ref_p[i - 1] += total - start_num`).
struct RefP {
    const KlShared* s;
    int i;
    long long tail;                    // total - start_num = hist[i] + ... + hist[kBins - 1]
    __device__ long long at(int k) const {
        const long long h = s->prefix[k + 2] - s->prefix[k + 1];
        return k == i - 1 ? h + tail : h;
    }
    __device__ long long sum(int a, int b) const {   // ref_p[a:b].sum()
        if (a >= b) return 0;
        long long v = s->prefix[b + 1] - s->prefix[a + 1];
        if (a <= i - 1 && i - 1 < b) v += tail;
        return v;
    }
    __device__ int zero_count(int a, int b) const {  // np.count_nonzero(ref_p[a:b] == 0)
        if (a >= b) return 0;
        int z = s->zeros[b + 1] - s->zeros[a + 1];
        if (a <= i - 1 && i - 1 < b) z += (at(i - 1) == 0) - (s->prefix[i + 1] == s->prefix[i]);
        return z;
    }
};

// `count + f * ref_p[k]` of _get_ref_q: float32 x int64 is a float64 product under numpy's promotion, the python int
// joins in float64 and int() truncates.
__device__ __forceinline__ long long ref_q_step(long long count, float f, long long p) {
    const double prod = __dmul_rn(static_cast<double>(f), __ll2double_rn(p));
    return __double2ll_rz(__dadd_rn(__ll2double_rn(count), prod));
}

// numpy's float32 pairwise sum (PW_BLOCKSIZE 128): a block of n <= 128 elements, 8 interleaved accumulators.
__device__ float pairwise_leaf(const float* a, int n) {
    if (n < 8) {
        float res = 0.f;
        for (int t = 0; t < n; ++t) res = __fadd_rn(res, a[t]);
        return res;
    }
    float r[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = a[j];
    int t = 8;
    for (; t < n - (n % 8); t += 8) {
#pragma unroll
        for (int j = 0; j < 8; ++j) r[j] = __fadd_rn(r[j], a[t + j]);
    }
    float res = __fadd_rn(__fadd_rn(__fadd_rn(r[0], r[1]), __fadd_rn(r[2], r[3])),
                          __fadd_rn(__fadd_rn(r[4], r[5]), __fadd_rn(r[6], r[7])));
    for (; t < n; ++t) res = __fadd_rn(res, a[t]);
    return res;
}

// The leaves of the pairwise split of n elements, in order: `idx` counts them; the one numbered `want` is returned in
// (off, len). Above 128 elements the split is at n / 2 rounded down to a multiple of 8. D bounds the depth: n <= 2048
// reaches leaves in at most 5 splits.
template <int D>
__device__ void pairwise_find_leaf(int off, int n, int& idx, int want, int& leaf_off, int& leaf_len) {
    if constexpr (D > 0) {
        if (n > kPairwiseBlock) {
            int n2 = n / 2;
            n2 -= n2 % 8;
            pairwise_find_leaf<D - 1>(off, n2, idx, want, leaf_off, leaf_len);
            pairwise_find_leaf<D - 1>(off + n2, n - n2, idx, want, leaf_off, leaf_len);
            return;
        }
    }
    if (idx == want) { leaf_off = off; leaf_len = n; }
    ++idx;
}

// Combines the leaf sums in the order of the pairwise recursion.
template <int D>
__device__ float pairwise_combine(int n, int& idx, const float* leaf) {
    if constexpr (D > 0) {
        if (n > kPairwiseBlock) {
            int n2 = n / 2;
            n2 -= n2 % 8;
            const float a = pairwise_combine<D - 1>(n2, idx, leaf);
            const float b = pairwise_combine<D - 1>(n - n2, idx, leaf);
            return __fadd_rn(a, b);
        }
    }
    return leaf[idx++];
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = __dadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// KL(hist || q) of candidate i (_get_ref_q, _expand_to_q, _kl_divergence), computed by one warp. Every integer and
// float32 step is the restatement's, in its order; only the float64 log2 and the float64 sums of the KL terms may
// round differently.
__device__ double candidate_kl(KlShared& s, int warp, int lane, int i) {
    const RefP rp{&s, i, s.prefix[kBins] - s.prefix[i]};
    float* q = s.q[warp];
    float* ref_q = s.ref_q[warp];
    float* dis = s.dis[warp];
    const float coeff = __fdiv_rn(static_cast<float>(i), static_cast<float>(kLevels));   // = step of _get_ref_q
    for (int j = lane; j < kLevels; j += 32) {
        const float start = __fmul_rn(coeff, static_cast<float>(j));
        const float end = __fmul_rn(coeff, static_cast<float>(j + 1));
        const int s_f = static_cast<int>(floorf(start)), e_f = static_cast<int>(floorf(end));
        const int s_c = static_cast<int>(ceilf(start));
        // _get_ref_q
        long long count = rp.sum(s_c, e_f);
        count = ref_q_step(count, __fsub_rn(static_cast<float>(s_c), start), rp.at(s_f));
        if (e_f < i) count = ref_q_step(count, __fsub_rn(end, static_cast<float>(e_f)), rp.at(e_f));
        ref_q[j] = __double2float_rn(__ll2double_rn(count));    // python int -> float64 -> float32 element
        // _expand_to_q's denominator: the python float count turns float32 at its first fractional addition
        float zero_num = static_cast<float>(rp.zero_count(s_c, e_f));
        if (rp.at(s_f) == 0) zero_num = __fadd_rn(zero_num, __fsub_rn(static_cast<float>(s_c), start));
        if (e_f < i && rp.at(e_f) == 0) zero_num = __fadd_rn(zero_num, __fsub_rn(end, static_cast<float>(e_f)));
        dis[j] = __fsub_rn(coeff, zero_num);
    }
    __syncwarp();
    // _expand_to_q, one element at a time: the quantised bins j that touch bin k add to it in the loop's order (j
    // ascending; within one j the partial first bin, the whole bins, the partial last bin).
    for (int k = lane; k < i; k += 32) {
        float acc = 0.f;
        if (rp.at(k) != 0) {
            const int jlo = max(0, static_cast<int>(static_cast<float>(k) / coeff) - 2);
            const int jhi = min(kLevels - 1, static_cast<int>(static_cast<float>(k + 1) / coeff) + 1);
            for (int j = jlo; j <= jhi; ++j) {
                const float d = dis[j];
                if (!(d > 0.f)) continue;
                const float start = __fmul_rn(coeff, static_cast<float>(j));
                const float end = __fmul_rn(coeff, static_cast<float>(j + 1));
                const int s_f = static_cast<int>(floorf(start)), e_f = static_cast<int>(floorf(end));
                const int s_c = static_cast<int>(ceilf(start));
                if (k == s_f)
                    acc = __fadd_rn(acc, __fmul_rn(__fdiv_rn(__fsub_rn(static_cast<float>(s_c), start), d), ref_q[j]));
                if (s_c <= k && k < e_f) acc = __fadd_rn(acc, __fmul_rn(__fdiv_rn(1.f, d), ref_q[j]));
                if (k == e_f)
                    acc = __fadd_rn(acc, __fmul_rn(__fdiv_rn(__fsub_rn(end, static_cast<float>(e_f)), d), ref_q[j]));
            }
        }
        q[k] = acc;
    }
    __syncwarp();
    // sum_q = float(int(q.sum())): the leaves of numpy's pairwise sum on their own lanes, combined on lane 0
    {
        int idx = 0, off = 0, len = 0;
        pairwise_find_leaf<6>(0, i, idx, lane, off, len);
        if (lane < idx) s.leaf[warp][lane] = pairwise_leaf(q + off, len);
    }
    __syncwarp();
    float total_q = 0.f;
    if (lane == 0) {
        int idx = 0;
        total_q = __fadd_rn(0.f, pairwise_combine<6>(i, idx, s.leaf[warp]));   // add.reduce starts from 0
    }
    total_q = __shfl_sync(0xffffffffu, total_q, 0);
    const double sum_p = __ll2double_rn(s.prefix[kBins]);
    const float sum_q_f = truncf(total_q);
    const double sum_q = static_cast<double>(sum_q_f);
    double kl;
    if (sum_p <= 0.0 || sum_q <= 0.0) {
        kl = inf_f64();
    } else {
        // q_prob = q / sum_q is float32 (a python float divisor is weak); p_prob = hist / sum_p is float64
        const double tail_q = __ddiv_rn(__ddiv_rn(static_cast<double>(q[i - 1]), sum_q), static_cast<double>(kBins - i + 1));
        double head = 0.0, tail = 0.0;
        for (int k = lane; k < kBins; k += 32) {
            const long long h = s.prefix[k + 1] - s.prefix[k];
            if (h == 0) continue;
            const double p = __ddiv_rn(__ll2double_rn(h), sum_p);
            if (k < i - 1) {
                if (q[k] != 0.f) {
                    const double qp = static_cast<double>(__fdiv_rn(q[k], sum_q_f));
                    head = __dadd_rn(head, __dmul_rn(p, log2(__ddiv_rn(p, qp))));
                }
            } else if (h > 0) {
                tail = __dadd_rn(tail, __dmul_rn(p, log2(__ddiv_rn(p, tail_q))));
            }
        }
        head = warp_sum(head);
        tail = warp_sum(tail);
        const bool tail_any = s.prefix[kBins] - s.prefix[i - 1] > 0;   // (counts are non-negative)
        if (tail_any && !(tail_q > 0.0)) kl = inf_f64();
        else kl = __dadd_rn(head, tail_any ? tail : 0.0);
    }
    __syncwarp();   // q, ref_q and dis are rewritten by the next candidate
    return kl;
}

__global__ void __launch_bounds__(kKlWarps * 32) calib_kl_kernel(const unsigned long long* __restrict__ hists,
                                                                 int32_t* __restrict__ thresh, double* __restrict__ kl_out) {
    extern __shared__ __align__(16) unsigned char kl_smem[];
    KlShared& s = *reinterpret_cast<KlShared*>(kl_smem);
    pdl_enter();
    const int h = blockIdx.x;
    const unsigned long long* hist = hists + static_cast<size_t>(h) * kBins;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int k = threadIdx.x; k < kBins; k += blockDim.x) {
        s.prefix[k + 1] = static_cast<long long>(__ldg(hist + k));
        if (kl_out && (k < kFirstCandidate || k >= kBins - 1))
            kl_out[static_cast<size_t>(h) * kBins + k] = __longlong_as_double(0x7ff8000000000000ll);   // NaN
    }
    if (threadIdx.x == 0) { s.prefix[0] = 0; s.zeros[0] = 0; }
    __syncthreads();
    // inclusive scans in chunks of 32: warp 0 the counts (in place), warp 1 the empty bins (read from global memory)
    if (warp < 2) {
        long long carry = 0;
        for (int base = 0; base < kBins; base += 32) {
            long long v = warp == 0 ? s.prefix[base + lane + 1] : static_cast<long long>(__ldg(hist + base + lane) == 0);
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const long long u = __shfl_up_sync(0xffffffffu, v, o);
                if (lane >= o) v += u;
            }
            if (warp == 0) s.prefix[base + lane + 1] = carry + v;
            else s.zeros[base + lane + 1] = static_cast<int>(carry + v);
            carry += __shfl_sync(0xffffffffu, v, 31);
        }
    }
    __syncthreads();
    // candidates i = 129 .. kBins - 2 round-robin over the warps; each warp keeps its first strict minimum
    double best = inf_f64();
    int best_i = 0;
    for (int i = kFirstCandidate + warp; i < kBins - 1; i += kKlWarps) {
        const double kl = candidate_kl(s, warp, lane, i);
        if (lane == 0 && kl_out) kl_out[static_cast<size_t>(h) * kBins + i] = kl;
        if (kl < best) { best = kl; best_i = i; }
    }
    if (lane == 0) { s.best_kl[warp] = best; s.best_i[warp] = best_i; }
    __syncthreads();
    if (threadIdx.x == 0) {
        // the restatement's `if kl < best` over ascending i: the smallest i among equal minima
        double b = inf_f64();
        int bi = 0;
        for (int w = 0; w < kKlWarps; ++w)
            if (s.best_i[w] && (s.best_kl[w] < b || (s.best_kl[w] == b && s.best_i[w] < bi))) {
                b = s.best_kl[w];
                bi = s.best_i[w];
            }
        thresh[h] = bi > 0 ? bi : kBins;
    }
}

template <bool PADDED, bool VEC>
int launch_stats(const float* x, long long count, int c, int ld, const int32_t* mode, uint32_t* max_bits,
                 unsigned long long* hist, void* stream) {
    const long long items = VEC ? count / 4 : count;
    const long long per_cta = static_cast<long long>(kStatsThreads) * kStatsVecPerThread;
    long long grid = (items + per_cta - 1) / per_cta;
    const long long cap = 2ll * sm_count();
    if (grid > cap) grid = cap;
    if (grid < 1) grid = 1;
    return launch("calib_stats", Pdl::On, calib_stats_kernel<PADDED, VEC>, dim3(static_cast<unsigned>(grid)),
                  dim3(kStatsThreads), 0, stream, dim3(1), x, count, c, ld, mode, max_bits, hist);
}

}  // namespace
}  // namespace b200

extern "C" {

int b200_calib_stats_run(const float* x, int64_t rows, int32_t c, int32_t ld, const int32_t* mode_dev,
                         uint32_t* max_bits_dev, uint64_t* hist_dev, void* stream) {
    if (!x || !mode_dev || !max_bits_dev || !hist_dev) return B200_INVALID_VALUE;
    if (rows < 1 || c < 1 || ld < c) return B200_INVALID_VALUE;
    if (!b200::device_is_sm90()) return B200_WRONG_DEVICE;
    const long long count = rows * static_cast<long long>(ld);
    auto* hist = reinterpret_cast<unsigned long long*>(hist_dev);
    const bool padded = c < ld;
    // 16-byte loads need an aligned base and, for a padded layout, rows of whole vectors
    const bool vec = (reinterpret_cast<uintptr_t>(x) & 15) == 0 && (padded ? ld % 4 == 0 : count % 4 == 0);
    if (padded)
        return vec ? b200::launch_stats<true, true>(x, count, c, ld, mode_dev, max_bits_dev, hist, stream)
                   : b200::launch_stats<true, false>(x, count, c, ld, mode_dev, max_bits_dev, hist, stream);
    return vec ? b200::launch_stats<false, true>(x, count, c, ld, mode_dev, max_bits_dev, hist, stream)
               : b200::launch_stats<false, false>(x, count, c, ld, mode_dev, max_bits_dev, hist, stream);
}

int b200_calib_kl_run(const uint64_t* hists, int32_t n, int32_t* thresh, double* kl, void* stream) {
    if (!hists || !thresh || n < 0) return B200_INVALID_VALUE;
    if (n == 0) return B200_SUCCESS;
    if (!b200::device_is_sm90()) return B200_WRONG_DEVICE;
    constexpr int smem = static_cast<int>(sizeof(b200::KlShared));
    b200::opt_in_smem<b200::calib_kl_kernel>(smem);
    return b200::launch("calib_kl", b200::Pdl::On, b200::calib_kl_kernel, dim3(static_cast<unsigned>(n)),
                        dim3(b200::kKlWarps * 32), smem, stream, dim3(1), reinterpret_cast<const unsigned long long*>(hists),
                        thresh, kl);
}

}  // extern "C"
