// Persistent, tile-pipelined variant of the TMA-im2col implicit-GEMM convolution (conv_igemm.cu) for grids of several
// waves (large batches, the 112 x 112 stem, the 56 x 56 stage): one CTA per SM walks the tile list
//     tile t = (n-tile t / tiles_m, m-tile t % tiles_m),  t = blockIdx.x, blockIdx.x + gridDim.x, ...
//   * warp 0 (one lane): TMA producer -- the operand ring never drains between tiles: the next tile's operands load
//     while the consumers finish the current one, no tile pays the first-load latency again, and the prologue
//     (barrier init, descriptor prefetch) is paid once;
//   * warps 4..11 (two warpgroups, 64 GEMM rows each): wgmma main loop with the accumulator in registers, then the
//     epilogue (bias / scale / residual / relu / requantise -> swizzled staging tile in its OWN shared memory -> TMA
//     store, which completes while the next tile's main loop runs).
// Same arithmetic, same epilogue code (conv_common.cuh) and same tensor maps as the per-tile kernel: results are
// bit-identical. Reference loop being replaced: one SASS / cuDNN launch per layer with one CTA per tile
// (saber/funcs/impl/cuda/saber_conv.cpp:17-585, sass_funcs.h:481-555).
#include <stdio.h>
#include <string.h>

#include "conv_common.cuh"

namespace b200 {

// smem: [ring: stages x (A 16 KiB + B BN*128 B)][staging 128 x BN x out_es][residual 128 x BN x res_es]
//       [bias | scale][full[MAX] empty[MAX] (4 spare) res_full res_empty][spare]
__host__ __device__ constexpr int persistent_tail_bytes(int bn) { return 2 * bn * 4 + (2 * MAX_STAGES + 6) * 8 + 16; }

template <int KIND, int BN>
__global__ void __launch_bounds__(NUM_THREADS, 1)
conv_persistent_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                       const __grid_constant__ CUtensorMap map_out, const __grid_constant__ CUtensorMap map_res,
                       const ConvKParams p, const uint32_t idesc, const int tiles_m, const int tiles_total) {
    constexpr int SB = stage_bytes(BN, false);
    constexpr int B_OFF = A_STAGE_BYTES;
    constexpr int NI = BN < 128 ? BN : 128;                          // wgmma N
    constexpr int NB = BN / NI;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>(
        (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
    uint8_t* out_tile = smem + p.stages * SB;
    uint8_t* res_tile = out_tile + BLOCK_M * BN * p.out_es;
    float* bias_s = reinterpret_cast<float*>(res_tile + p.res_panels * BLOCK_M * p.res_pw);
    float* scale_s = bias_s + BN;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(scale_s + BN);
    uint64_t* empty_bar = full_bar + MAX_STAGES;
    uint64_t* res_full_bar = empty_bar + MAX_STAGES + 4;
    uint64_t* res_empty_bar = res_full_bar + 1;

    const int warp_idx = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int subs_per_stage = STAGE_K_BYTES / p.chunk;
    const int num_stage_iters = (p.KS + subs_per_stage - 1) / subs_per_stage;

    if (warp_idx == 0 && lane == 0) {
        tma_prefetch_desc(&map_a);
        tma_prefetch_desc(&map_b);
        tma_prefetch_desc(&map_out);
        if (p.res_panels > 0) tma_prefetch_desc(&map_res);
        for (int i = 0; i < p.stages; ++i) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], EPI_WARPS);
        }
        mbar_init(res_full_bar, 1);
        mbar_init(res_empty_bar, EPI_THREADS);
        fence_mbar_init();
    }
    __syncthreads();

    pdl_launch_dependents();

    if (warp_idx == 0) {
        if (lane == 0) {
            // ===================== TMA producer =====================
            const uint32_t b_sub_bytes = BN * p.chunk;
            const uint32_t a_sub_bytes = BLOCK_M * p.chunk;
            const uint32_t tx_per_sub = a_sub_bytes + b_sub_bytes;
            const uint32_t ring_sa = smem_u32(smem), full_sa0 = smem_u32(full_bar), empty_sa0 = smem_u32(empty_bar);
            const int res_cols_per_panel = p.res_panels > 0 ? p.res_pw / p.res_es : 0;
            int stage = 0;
            uint32_t phase = 0, stage_sa = ring_sa, full_sa = full_sa0, empty_sa = empty_sa0;
            uint32_t res_phase = 1;       // parity to wait on res_empty: the first use finds the buffer free
            pdl_wait_prior_grid();
            for (int tile = blockIdx.x; tile < tiles_total; tile += gridDim.x) {
                const int nt = tile / tiles_m, mt = tile - nt * tiles_m;
                const int m0 = mt * BLOCK_M, n0 = nt * BN;
                const int n_img = m0 / p.HoWo;
                const int rem = m0 - n_img * p.HoWo;
                const int p0 = rem / p.Wo;
                const int q0 = rem - p0 * p.Wo;
                const int base_w = q0 * p.stride_w - p.pad_w;
                const int base_h = p0 * p.stride_h - p.pad_h;
                int ks = 0, cc = 0, r = 0, s = 0;
                int c_coord = 0, k_coord = 0, off_w = 0, off_h = 0;
                for (int it = 0; it < num_stage_iters; ++it) {
                    // always a full stage: k-steps past KS_real re-read tap (0,0) against zero weights (the weight map
                    // zero-fills k beyond its extent)
                    mbar_wait_sa(empty_sa, phase ^ 1);
                    mbar_arrive_expect_tx_sa(full_sa, subs_per_stage * tx_per_sub);
                    uint32_t a_dst = stage_sa, b_dst = stage_sa + B_OFF;
#pragma unroll 1
                    for (int j = 0; j < subs_per_stage; ++j) {
                        const bool pad_step = ks >= p.KS_real;
                        tma_load_im2col_4d_sa(&map_a, full_sa, a_dst, pad_step ? 0 : c_coord, base_w, base_h, n_img,
                                              static_cast<uint16_t>(pad_step ? 0 : off_w),
                                              static_cast<uint16_t>(pad_step ? 0 : off_h));
                        tma_load_2d_sa(&map_b, full_sa, b_dst, k_coord, n0);
                        a_dst += a_sub_bytes; b_dst += b_sub_bytes;
                        ++ks;
                        k_coord += p.chunk_el;
                        c_coord += p.chunk_el;
                        if (++cc == p.CC) {
                            cc = 0; c_coord = 0;
                            off_w += p.dil_w;
                            if (++s == p.S) { s = 0; off_w = 0; ++r; off_h += p.dil_h; }
                        }
                    }
                    stage_sa += SB; full_sa += 8; empty_sa += 8;
                    if (++stage == p.stages) { stage = 0; phase ^= 1; stage_sa = ring_sa; full_sa = full_sa0; empty_sa = empty_sa0; }
                    if (it == 0 && p.res_panels > 0) {
                        // the residual tile of this output tile: into the single residual buffer once the epilogue of
                        // the previous tile has read it out
                        mbar_wait(res_empty_bar, res_phase);
                        res_phase ^= 1;
                        mbar_arrive_expect_tx(res_full_bar, p.res_panels * BLOCK_M * p.res_pw);
                        for (int j = 0; j < p.res_panels; ++j)
                            tma_load_2d(&map_res, res_full_bar, res_tile + j * BLOCK_M * p.res_pw, n0 + j * res_cols_per_panel, m0);
                    }
                }
            }
        }
    } else if (warp_idx >= EPI_TID0 / 32) {
        // ===================== consumer warpgroups =====================
        const int etid = threadIdx.x - EPI_TID0;
        const int cwg = etid >> 7;
        const int row = 64 * cwg + 16 * ((etid >> 5) & 3) + acc_row16_row(lane);
        const PanelRow out_row = make_panel_row(smem_u32(out_tile), panel_lg(p.out_pw), row);
        const PanelRow res_row = make_panel_row(smem_u32(res_tile), panel_lg(p.res_pw ? p.res_pw : 128), row);
        const uint32_t bias_sa = smem_u32(bias_s), scale_sa = smem_u32(scale_s);
        const bool storer = etid == 0;
        const int cols_per_panel = p.out_pw / p.out_es;
        // descriptors as (lo, hi) words (conv_igemm.cu)
        const bool a_signed = idesc_a_signed(idesc);
        const uint32_t lt = layout_type_for_chunk(p.chunk);
        const uint32_t a_sub16 = (BLOCK_M * p.chunk) >> 4, b_sub16 = (BN * p.chunk) >> 4;
        const bool swz = p.chunk >= 32;
        const uint32_t hi = (swz ? (8u * p.chunk) >> 4 : 128u >> 4) | (lt << 29);
        const uint32_t a_lbo = (swz ? 1u : a_sub16) << 16, b_lbo = (swz ? 1u : b_sub16) << 16;
        const uint32_t a_wg16 = (64u * p.chunk * cwg) >> 4, nb16 = (NI * p.chunk) >> 4;
        const uint32_t ring16 = smem_u32(smem) >> 4;
        // 16-byte offsets of the four 32-byte K slices of a stage (STAGE_K_BYTES = 4 MMAs). Every stage is full -- the
        // producer pads the last one with zero-weight k-steps -- so the MMAs are issued by a loop of fixed length:
        // a loop with a runtime trip count around wgmma makes ptxas serialise the MMAs.
        uint32_t a_off[4], b_off[4];
#pragma unroll
        for (int m = 0; m < 4; ++m) {
            const uint32_t j = swz ? m / (p.chunk >> 5) : 2 * m, q = swz ? m % (p.chunk >> 5) : 0;
            a_off[m] = j * a_sub16 + 2 * q;
            b_off[m] = j * b_sub16 + 2 * q;
        }
        int stage = 0;
        uint32_t phase = 0, res_phase = 0;
        int n0_loaded = -1;
        for (int tile = blockIdx.x; tile < tiles_total; tile += gridDim.x) {
            const int nt = tile / tiles_m, mt = tile - nt * tiles_m;
            const int m0 = mt * BLOCK_M, n0 = nt * BN;
            uint32_t acc[NB][NI / 2];
#pragma unroll
            for (int nb = 0; nb < NB; ++nb)
#pragma unroll
                for (int i = 0; i < NI / 2; ++i) acc[nb][i] = 0u;
            int prev = -1;
            for (int it = 0; it < num_stage_iters; ++it) {
                mbar_wait(&full_bar[stage], phase);
                const uint32_t st16 = ring16 + stage * (SB >> 4);
                const uint32_t a16 = st16 + a_wg16, b16 = st16 + (B_OFF >> 4);
                wgmma_fence();
#pragma unroll
                for (int m = 0; m < 4; ++m) {
                    const uint64_t ad = desc64(((a16 + a_off[m]) & 0x3FFFu) | a_lbo, hi);
#pragma unroll
                    for (int nb = 0; nb < NB; ++nb)
                        wgmma<KIND, NI>(acc[nb], ad, desc64(((b16 + nb * nb16 + b_off[m]) & 0x3FFFu) | b_lbo, hi), a_signed, 1u);
                }
                wgmma_commit();
                wgmma_wait<1>();
                if (prev >= 0) {
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&empty_bar[prev]);
                }
                prev = stage;
                if (++stage == p.stages) { stage = 0; phase ^= 1; }
            }
            wgmma_wait<0>();
#pragma unroll
            for (int nb = 0; nb < NB; ++nb) wgmma_fence_acc(acc[nb]);
            if (prev >= 0) {
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty_bar[prev]);
            }
            // the staging tile is free once the previous tile's TMA store has read it; the tables follow the n-tile
            if (storer) tma_store_wait_read();
            if (n0 != n0_loaded) {
                asm volatile("bar.sync 1, %0;" ::"n"(EPI_THREADS) : "memory");   // nobody still reads the old tables
                fill_epilogue_tables<EPI_THREADS>(p, n0, BN, etid, bias_s, scale_s);
                n0_loaded = n0;
            }
            asm volatile("bar.sync 1, %0;" ::"n"(EPI_THREADS) : "memory");
            if (p.res_panels > 0) { mbar_wait(res_full_bar, res_phase); res_phase ^= 1; }
#pragma unroll
            for (int g = 0; g < BN / 32; ++g) {
                uint32_t v0[16];
                acc_row16<NI>(acc[g / (NI / 32)], g % (NI / 32), v0);
                const int c0 = acc_row16_col(lane, g);
                if (n0 + c0 >= p.K) continue;
                epilogue16<KIND>(p, v0, c0, bias_sa, scale_sa, res_row, out_row);
            }
            // the residual buffer is read out: hand it back before the store
            if (p.res_panels > 0) mbar_arrive(res_empty_bar);
            fence_proxy_async_smem();
            asm volatile("bar.sync 1, %0;" ::"n"(EPI_THREADS) : "memory");
            if (storer) {
                for (int j = 0; j < p.out_panels; ++j) {
                    if (n0 + j * cols_per_panel >= p.K) break;
                    tma_store_2d(&map_out, out_tile + j * BLOCK_M * p.out_pw, n0 + j * cols_per_panel, m0);
                }
                tma_store_commit();
            }
        }
        if (storer) tma_store_wait_read();
    }

    __syncthreads();
}

template <int KIND, int BN>
static void launch_persistent(b200_conv_plan* pl, void* stream) {
    constexpr auto kern = conv_persistent_kernel<KIND, BN>;
    opt_in_smem<kern>(MAX_SMEM);
    launch_kernel(kern, dim3(pl->persistent_ctas), dim3(NUM_THREADS), pl->smem_bytes, static_cast<cudaStream_t>(stream),
                  dim3(1), pl->map_a, pl->map_b, pl->map_out, pl->map_res, pl->kp, pl->idesc, static_cast<int>(pl->grid.x),
                  static_cast<int>(pl->grid.x * pl->grid.y));
    count_launch();
}

// Turn a finished per-tile im2col plan into the persistent variant when its grid spans several waves. Keeps BN, the
// tensor maps and the epilogue parameters; recomputes the ring depth for one CTA per SM with a dedicated staging tile.
bool persistent_plan_setup(b200_conv_plan* pl) {
    const b200_conv_desc_t& d = pl->desc;
    const char* env = getenv("B200_SABER_PERSISTENT");
    if (env && env[0] == '0') return false;
    if (d.math == B200_MATH_TF32X3 || pl->kp.split != 1) return false;
    const int sms = sm_count();
    const int tiles = static_cast<int>(pl->grid.x * pl->grid.y);
    const bool force = env && env[0] == '2';
    // worth it once every SM gets more than the two tiles that co-resident CTAs already overlap ...
    if (!force && tiles <= 2 * sms) return false;
    const int bn = pl->bn;
    {
        // ... and the tile is not epilogue-dominated: the walker's consumer warps run each tile's epilogue after its main
        // loop (only the producer keeps loading meanwhile), while two co-resident per-tile CTAs overlap one's epilogue with
        // the other's main loop. Cost model and thresholds: conv_common.cuh (epilogue clocks per channel below).
        const double k_bytes = static_cast<double>(pl->g.KS) * pl->g.chunk;
        const double ingest = (BLOCK_M + bn) * k_bytes / L2_INGEST_BYTES_PER_CLK;
        const double mma = k_bytes / 32.0 * mma_clk(bn);
        const double loop = mma > ingest ? mma : ingest;
        const double epi = bn * (pl->kp.res_es ? 11.0 : 9.0);
        // With many tiles per SM (>= 6) the per-tile CTAs pay their prologue / barrier setup / drain once per tile, so the
        // walker is taken further into epilogue-bound territory from 6 tiles per SM.
        static const double epi_env = [] { const char* e = getenv("B200_SABER_PERSISTENT_EPI"); const double v = e ? atof(e) : 0.0; return v > 0.0 ? v : 0.0; }();
        const double epi_ratio = epi_env > 0.0 ? epi_env : (tiles >= 6 * sms ? 2.5 : 1.5);
        if (!force && epi > epi_ratio * loop) return false;
    }
    const int sb = stage_bytes(bn, false);
    const int staging = BLOCK_M * bn * pl->kp.out_es;
    const int res_bytes = BLOCK_M * bn * pl->kp.res_es;
    const int fixed = staging + res_bytes + persistent_tail_bytes(bn) + 1024;
    int stages = (MAX_SMEM - fixed) / sb;
    if (stages > MAX_STAGES) stages = MAX_STAGES;
    if (stages < 2) return false;
    // (no 3xTF32 walker: excluded above)
    const ConvLaunch l = bind_kind_bn<32, 64, 128, 256>(kind_for_math(d.math), bn, [](auto K, auto N) -> ConvLaunch {
        if constexpr (K == KIND_TF32X3) return nullptr;
        else return launch_persistent<K, N>;
    });
    if (!l) return false;
    pl->launch = l;
    pl->kp.stages = stages;
    pl->smem_bytes = stages * sb + fixed;
    pl->persistent_ctas = tiles < sms ? tiles : sms;
    pl->persistent = true;
    return true;
}

}  // namespace b200
