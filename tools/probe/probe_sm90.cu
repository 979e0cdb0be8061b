// Micro-probes behind the conv planner's cost model on the H100 (sm_90a). Stand-alone: one executable, run on the GPU
// by tools/probe/run_probe.sh, which writes profiles/probe_sm90.txt.
//   1. wgmma cost per 32-byte k slice: two consumer warpgroups of 64 rows (the conv kernels' shape), N = 32..256,
//      s8 / f16 / tf32, both operands in shared memory
//   2. TMA ingest from L2: a tiled 128-row x 128 B box and a 3x3 im2col walk, at grids of 1, 66, 132 and 264 CTAs,
//      and the same loads multicast over clusters of 2 and 4 (each CTA fetches 1/cn of every box, receives all of it,
//      and a ring slot is refilled only after every CTA of the cluster has released it -- the conv kernels' protocol)
//   3. fixed cost of one split-K reduce-scatter through distributed shared memory (128 x 64 int32 partial tile)
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o probe_sm90 probe_sm90.cu -lcuda
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "../../anakin_b200/csrc/ptx.cuh"

using namespace b200;

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); exit(1); } } while (0)

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
typedef CUresult (*PFN_encodeIm2col)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                     const cuuint64_t*, const int*, const int*, cuuint32_t, cuuint32_t,
                                     const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                     CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static PFN_encodeTiled g_tiled;
static PFN_encodeIm2col g_im2col;

// ------------------------------------------------------------------------------------------------ 1. wgmma cost
// 256 threads = two warpgroups, each D[64 x N] += A[64 x 32 B] * B[N x 32 B]^T in groups of four k slices (one
// pipeline stage), committed and waited one group behind, as the conv main loops do. Operands: SW128 K-major tiles.
template <int MK, int N>
__global__ void __launch_bounds__(256, 1) mma_cost_kernel(int n_groups, long long* out, uint32_t* sink) {
    constexpr int NI = N < 128 ? N : 128;
    constexpr int NB = N / NI;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    for (int i = threadIdx.x; i < (128 + N) * 128 / 16; i += 256) reinterpret_cast<uint4*>(smem)[i] = make_uint4(0, 0, 0, 0);
    fence_proxy_async_smem();
    __syncthreads();
    const int wg = threadIdx.x >> 7;
    const uint32_t hi = ((8u * 128) >> 4) | (2u << 29);
    const uint32_t a16 = (smem_u32(smem) >> 4) + wg * (64 * 128 >> 4), b16 = (smem_u32(smem) + 128 * 128) >> 4;
    uint32_t acc[NB][NI / 2];
#pragma unroll
    for (int nb = 0; nb < NB; ++nb)
#pragma unroll
        for (int i = 0; i < NI / 2; ++i) acc[nb][i] = 0u;
    long long t0 = clock64();
    for (int g = 0; g < n_groups; ++g) {
        wgmma_fence();
#pragma unroll
        for (int m = 0; m < 4; ++m)
#pragma unroll
            for (int nb = 0; nb < NB; ++nb)
                wgmma<MK, NI>(acc[nb], desc64(((a16 + 2 * m) & 0x3FFFu) | (1u << 16), hi),
                              desc64(((b16 + nb * (NI * 128 >> 4) + 2 * m) & 0x3FFFu) | (1u << 16), hi), false, 1u);
        wgmma_commit();
        wgmma_wait<1>();
    }
    wgmma_wait<0>();
#pragma unroll
    for (int nb = 0; nb < NB; ++nb) wgmma_fence_acc(acc[nb]);
    const long long t1 = clock64();
    if ((threadIdx.x & 127) == 0) out[blockIdx.x * 2 + wg] = t1 - t0;
    uint32_t s = 0;
#pragma unroll
    for (int nb = 0; nb < NB; ++nb)
#pragma unroll
        for (int i = 0; i < NI / 2; ++i) s += acc[nb][i];
    if (s == 0x12345678u) sink[0] = s;   // keeps the MMAs alive
}

template <int MK, int N>
static void mma_cost_row(const char* kind, int grid, long long* d_out, uint32_t* d_sink) {
    const int n_groups = 512;
    const int smem = (128 + N) * 128 + 1024;
    auto kern = mma_cost_kernel<MK, N>;
    CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    for (int rep = 0; rep < 2; ++rep) {
        kern<<<grid, 256, smem>>>(n_groups, d_out, d_sink);
        CK(cudaDeviceSynchronize());
    }
    std::vector<long long> h(2 * grid);
    CK(cudaMemcpy(h.data(), d_out, h.size() * 8, cudaMemcpyDeviceToHost));
    std::sort(h.begin(), h.end());
    printf("%-6s %-5d %-6d %12.1f %12.1f\n", kind, N, grid, double(h[h.size() / 2]) / (4.0 * n_groups),
           double(h.back()) / (4.0 * n_groups));
}

static void run_mma_cost() {
    printf("== 1. wgmma cost: SM clocks per 32-byte k slice of a 128 x N tile (two warpgroups of 64 rows), median / max over warpgroups\n");
    printf("%-6s %-5s %-6s %12s %12s\n", "kind", "N", "grid", "clk med", "clk max");
    long long* d_out;
    uint32_t* d_sink;
    CK(cudaMalloc(&d_out, 2 * 264 * sizeof(long long)));
    CK(cudaMalloc(&d_sink, 4));
    for (int grid : {1, 132}) {
        mma_cost_row<KIND_I8, 32>("s8", grid, d_out, d_sink);
        mma_cost_row<KIND_I8, 64>("s8", grid, d_out, d_sink);
        mma_cost_row<KIND_I8, 128>("s8", grid, d_out, d_sink);
        mma_cost_row<KIND_I8, 256>("s8", grid, d_out, d_sink);
        mma_cost_row<KIND_F16, 32>("f16", grid, d_out, d_sink);
        mma_cost_row<KIND_F16, 64>("f16", grid, d_out, d_sink);
        mma_cost_row<KIND_F16, 128>("f16", grid, d_out, d_sink);
        mma_cost_row<KIND_F16, 256>("f16", grid, d_out, d_sink);
        mma_cost_row<KIND_TF32, 32>("tf32", grid, d_out, d_sink);
        mma_cost_row<KIND_TF32, 64>("tf32", grid, d_out, d_sink);
        mma_cost_row<KIND_TF32, 128>("tf32", grid, d_out, d_sink);
        mma_cost_row<KIND_TF32, 256>("tf32", grid, d_out, d_sink);
    }
    cudaFree(d_out);
    cudaFree(d_sink);
}

// ------------------------------------------------------------------------------------------------ 2. TMA ingest
struct IngestParams {
    int iters, depth, im2col;
    int cn;                      // cluster size: every box is fetched in cn parts, one per CTA, multicast to all
    int tiles_total;             // box index wrap
    int HoWo, Wo;                // im2col geometry (56 x 56, pad 1)
};

__global__ void __launch_bounds__(128) ingest_kernel(const __grid_constant__ CUtensorMap map, const IngestParams p, long long* out) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    __shared__ uint64_t full[16], empty[16];
    const uint32_t rank = p.cn > 1 ? cluster_ctarank() : 0;
    if (threadIdx.x == 0) {
        for (int i = 0; i < p.depth; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], p.cn); }
        fence_mbar_init();
        tma_prefetch_desc(&map);
    }
    __syncthreads();
    if (p.cn > 1) cluster_sync_all();
    constexpr int tile_bytes = 128 * 128;
    const int part_rows = 128 / p.cn;
    if (threadIdx.x == 0) {
        const int cluster_id = blockIdx.x / p.cn;
        const uint32_t smem_sa = smem_u32(smem), full_sa = smem_u32(full), empty_sa = smem_u32(empty);
        const uint16_t mask = static_cast<uint16_t>((1u << p.cn) - 1);
        auto issue = [&](int i) {
            const int st = i % p.depth;
            mbar_arrive_expect_tx_sa(full_sa + 8 * st, tile_bytes);
            const uint32_t dst = smem_sa + st * tile_bytes + rank * part_rows * 128;
            if (!p.im2col) {
                const int row = ((cluster_id * 977 + i) % p.tiles_total) * 128 + rank * part_rows;
                if (p.cn == 1) tma_load_2d_sa(&map, full_sa + 8 * st, dst, 0, row);
                else tma_load_2d_mc_sa(&map, full_sa + 8 * st, dst, 0, row, mask);
            } else {
                // 3x3 pad-1 walk: consecutive loads = the 9 taps of one 128-pixel tile; this CTA's part starts
                // rank * 128 / cn pixels into it
                const int t = (cluster_id * 977 + i / 9) % p.tiles_total, tap = i % 9;
                const int m0 = t * 128 + rank * part_rows;
                const int n = m0 / p.HoWo, rem = m0 - n * p.HoWo, p0 = rem / p.Wo, q0 = rem - p0 * p.Wo;
                if (p.cn == 1)
                    tma_load_im2col_4d_sa(&map, full_sa + 8 * st, dst, 0, q0 - 1, p0 - 1, n, static_cast<uint16_t>(tap % 3),
                                          static_cast<uint16_t>(tap / 3));
                else
                    tma_load_im2col_4d_mc_sa(&map, full_sa + 8 * st, dst, 0, q0 - 1, p0 - 1, n, static_cast<uint16_t>(tap % 3),
                                             static_cast<uint16_t>(tap / 3), mask);
            }
        };
        const long long t0 = clock64();
        for (int i = 0; i < p.depth && i < p.iters; ++i) issue(i);
        for (int i = 0; i < p.iters; ++i) {
            const int st = i % p.depth;
            const uint32_t ph = (i / p.depth) & 1;
            mbar_wait_sa(full_sa + 8 * st, ph);
            // release the slot to every producer that writes into it
            for (int r = 0; r < p.cn; ++r) mbar_arrive_cluster(map_to_cta(empty_sa + 8 * st, r));
            if (i + p.depth < p.iters) {
                mbar_wait_sa(empty_sa + 8 * st, ph);
                issue(i + p.depth);
            }
        }
        out[blockIdx.x] = clock64() - t0;
    }
    __syncthreads();
    if (p.cn > 1) cluster_sync_all();   // no CTA exits while a peer may still arrive on its barriers
}

static void run_ingest() {
    printf("== 2. TMA ingest from L2: bytes/clk received per CTA (median, min over CTAs), whole-grid time, and the grid's\n"
           "      received and L2-fetched rates (fetched = received / cn). 16 KiB per box, 4- or 8-deep ring, 360 boxes per CTA.\n");
    const size_t bytes = 32u << 20;   // L2-resident on the 50 MB L2
    uint8_t* buf;
    CK(cudaMalloc(&buf, bytes));
    CK(cudaMemset(buf, 1, bytes));
    long long* d_out;
    CK(cudaMalloc(&d_out, 512 * sizeof(long long)));
    CK(cudaFuncSetAttribute(ingest_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 8 * 16 * 1024 + 1024));
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    printf("%-10s %-4s %-5s %-5s %10s %10s %10s %12s %12s\n", "mode", "cn", "depth", "grid", "B/clk med", "B/clk min", "grid us",
           "recv GB/s", "fetch GB/s");
    auto run = [&](int im2col, int cn, int grid, int depth) {
        CUtensorMap map;
        IngestParams p{};
        p.iters = 360; p.depth = depth; p.im2col = im2col; p.cn = cn;
        if (im2col) {
            const int H = 56, W = 56, C = 128, N = static_cast<int>(bytes / (size_t(H) * W * C) * 3 / 4);
            cuuint64_t dims[4] = {cuuint64_t(C), cuuint64_t(W), cuuint64_t(H), cuuint64_t(N)};
            cuuint64_t strides[3] = {cuuint64_t(C), cuuint64_t(W) * C, cuuint64_t(H) * W * C};
            int lower[2] = {-1, -1}, upper[2] = {-1, -1};
            cuuint32_t estr[4] = {1, 1, 1, 1};
            CUresult r = g_im2col(&map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 4, buf, dims, strides, lower, upper, C, 128 / cn, estr,
                                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            if (r != CUDA_SUCCESS) { printf("im2col encode failed %d\n", int(r)); return; }
            p.HoWo = H * W; p.Wo = W; p.tiles_total = N * H * W / 128 - 1;
        } else {
            const size_t rows = bytes / 128;
            cuuint64_t dims[2] = {128, cuuint64_t(rows)};
            cuuint64_t strides[1] = {128};
            cuuint32_t box[2] = {128, cuuint32_t(128 / cn)};
            cuuint32_t estr[2] = {1, 1};
            CUresult r = g_tiled(&map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, buf, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                 CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            if (r != CUDA_SUCCESS) { printf("tiled encode failed %d\n", int(r)); return; }
            p.tiles_total = static_cast<int>(rows / 128);
        }
        cudaLaunchConfig_t cfg{};
        cfg.gridDim = dim3(grid); cfg.blockDim = dim3(128);
        cfg.dynamicSmemBytes = depth * 128 * 128 + 1024;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim.x = cn; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
        cfg.attrs = attr; cfg.numAttrs = 1;
        CK(cudaLaunchKernelEx(&cfg, ingest_kernel, map, p, d_out));   // warms L2
        CK(cudaDeviceSynchronize());
        const int reps = 5;
        CK(cudaEventRecord(e0));
        for (int rep = 0; rep < reps; ++rep) CK(cudaLaunchKernelEx(&cfg, ingest_kernel, map, p, d_out));
        CK(cudaEventRecord(e1));
        CK(cudaDeviceSynchronize());
        float ms = 0;
        CK(cudaEventElapsedTime(&ms, e0, e1));
        const double us = ms * 1e3 / reps;
        std::vector<long long> h(grid);
        CK(cudaMemcpy(h.data(), d_out, h.size() * 8, cudaMemcpyDeviceToHost));
        std::vector<double> bpc(grid);
        for (int i = 0; i < grid; ++i) bpc[i] = double(p.iters) * 128 * 128 / double(h[i]);
        std::sort(bpc.begin(), bpc.end());
        const double recv = double(grid) * p.iters * 128 * 128;
        printf("%-10s %-4d %-5d %-5d %10.1f %10.1f %10.1f %12.0f %12.0f\n", im2col ? "im2col3x3" : "tiled", cn, depth, grid, bpc[grid / 2],
               bpc[0], us, recv / us / 1e3, recv / cn / us / 1e3);
    };
    for (int im2col : {0, 1})
        for (int cn : {1, 2, 4})
            for (int depth : {4, 8})
                for (int grid : {1, 66, 132, 264}) run(im2col, cn, grid < cn ? cn : grid / cn * cn, depth);   // whole clusters
    cudaFree(buf);
    cudaFree(d_out);
}

// ------------------------------------------------------------------------------------------------ 3. split-K exchange
// A cluster of `split` CTAs, 256 threads each holding one row's 64 int32 partial sums per 128-row tile: every CTA sends
// the slices it does not own to their owners with st.async (completing on the owner's mbarrier) and waits for its own.
// Timed from the cluster barrier that opens the exchange to the owner's barrier completing.
__global__ void __launch_bounds__(256, 1) exchange_kernel(int split, long long* out) {
    constexpr int BN = 64;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    __shared__ uint64_t part_bar;
    const int rank = static_cast<int>(cluster_ctarank());
    const int epi_bn = BN / split;
    const uint32_t slice_bytes = 128 * epi_bn * 4;
    if (threadIdx.x == 0) {
        mbar_init(&part_bar, 1);
        mbar_arrive_expect_tx(&part_bar, (split - 1) * slice_bytes);
        fence_mbar_init();
    }
    __syncthreads();
    cluster_sync_all();
    const long long t0 = clock64();
    const int row = threadIdx.x >> 1, half = threadIdx.x & 1;   // two threads per row, 32 columns each
    const uint32_t part_sa = smem_u32(smem), bar_sa = smem_u32(&part_bar);
    for (int g = 0; g < 2; ++g) {
        const int c0 = half * 32 + g * 16;
        const int owner = c0 / epi_bn;
        if (owner == rank) continue;
        const int slot = rank - (rank > owner ? 1 : 0);
        const uint32_t d = map_to_cta(part_sa + slot * slice_bytes + static_cast<uint32_t>(((c0 - owner * epi_bn) >> 4) * 128 + row) * 64, owner);
        const uint32_t bar = map_to_cta(bar_sa, owner);
        for (int q = 0; q < 4; ++q) st_async_v4(d + q * 16, bar, c0, row, q, rank);
    }
    mbar_wait(&part_bar, 0);
    const long long t1 = clock64();
    if (threadIdx.x == 0) out[blockIdx.x] = t1 - t0;
    __syncthreads();
    cluster_sync_all();
}

static void run_exchange() {
    printf("== 3. split-K reduce-scatter of a 128 x 64 int32 tile through DSMEM: SM clocks from the opening cluster barrier\n"
           "      to the last partial slice landing (median / max over CTAs), and one cluster barrier alone\n");
    long long* d_out;
    CK(cudaMalloc(&d_out, 512 * sizeof(long long)));
    CK(cudaFuncSetAttribute(exchange_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    printf("%-6s %-5s %10s %10s\n", "split", "grid", "clk med", "clk max");
    for (int split : {2, 4}) {
        for (int grid : {split, 128}) {
            cudaLaunchConfig_t cfg{};
            cfg.gridDim = dim3(grid); cfg.blockDim = dim3(256);
            cfg.dynamicSmemBytes = 3 * 128 * 32 * 4 + 1024;
            cudaLaunchAttribute attr[1];
            attr[0].id = cudaLaunchAttributeClusterDimension;
            attr[0].val.clusterDim.x = split; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
            cfg.attrs = attr; cfg.numAttrs = 1;
            for (int rep = 0; rep < 3; ++rep) CK(cudaLaunchKernelEx(&cfg, exchange_kernel, split, d_out));
            CK(cudaDeviceSynchronize());
            std::vector<long long> h(grid);
            CK(cudaMemcpy(h.data(), d_out, h.size() * 8, cudaMemcpyDeviceToHost));
            std::sort(h.begin(), h.end());
            printf("%-6d %-5d %10lld %10lld\n", split, grid, h[grid / 2], h.back());
        }
    }
    cudaFree(d_out);
}

int main(int argc, char** argv) {
    cudaDriverEntryPointQueryResult q;
    void* fn = nullptr;
    CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q));
    g_tiled = reinterpret_cast<PFN_encodeTiled>(fn);
    CK(cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &fn, cudaEnableDefault, &q));
    g_im2col = reinterpret_cast<PFN_encodeIm2col>(fn);
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    int clk_khz = 0;
    CK(cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, 0));
    printf("device %s, %d SMs, max SM clock %d kHz\n", prop.name, prop.multiProcessorCount, clk_khz);
    const char* which = argc > 1 ? argv[1] : "all";
    if (!strcmp(which, "all") || !strcmp(which, "mma")) run_mma_cost();
    if (!strcmp(which, "all") || !strcmp(which, "ingest")) run_ingest();
    if (!strcmp(which, "all") || !strcmp(which, "exchange")) run_exchange();
    return 0;
}
