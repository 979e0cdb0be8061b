// Implicit-GEMM convolution on Hopper tensor cores (wgmma, sm_90a).
//
// Replaces the reference's NV conv family: SaberConv2D / SaberConvEltwise /
// SaberGemmLikeConv / SaberDirectConv / SaberWinogradConv dispatchers
// (reference saber/funcs/impl/cuda/saber_conv.cpp:17-585,
//  saber_conv_eltwise.cpp:32-318, saber_conv_gemmlike.cpp:38-168,
//  saber_conv_direct.cpp:40-220) and the closed SASS kernels behind them
// (third-party/sass/include/sass_funcs.h:54-935).
//
// GEMM view:  D[M x N] = A[M x Kg] * B[N x Kg]^T
//   M  = n*ho*wo output pixels (NHWC rows), N = output channels,
//   Kg = r*s*c, ordered (r, s, c) with c innermost.
// A is never materialised: one TMA *im2col* load fetches, for a filter tap
// (r,s) and a channel chunk, the [128 pixels x chunk bytes] operand tile straight
// from the NHWC activation tensor into swizzled shared memory (zero-filling the
// padding halo).  B (packed weights) arrives through a tiled TMA load.  Two
// consumer warpgroups issue wgmma on 64 rows each, accumulating in registers.
//
// Epilogue: the residual tile is TMA-prefetched into swizzled shared memory while
// the main loop runs, bias / scale tables are staged in shared memory, the consumer
// warps regroup their accumulator fragments into 16-column runs of one row
// (acc_row16), apply bias / per-channel scale / residual / relu / requantise in
// registers, write the result tile into swizzled shared memory (the freed operand
// ring) and one thread hands it to TMA for a fully coalesced store (which also
// clips the ragged M / N edges).
//
// Warp roles (384 threads): warp 0 = TMA producer (warps 1..3 idle),
// warps 4..11 = two consumer warpgroups (main loop + epilogue).
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdio.h>
#include <string.h>

#include <new>

#include "conv_common.cuh"

namespace b200 {

// ----------------------------------------------------------------- the kernel
// Two CTAs per SM for narrow tiles (85 registers a thread); split-K grids fit in one wave by construction and wide tiles
// hold BN / 2 accumulator registers a thread: one CTA per SM.
template <int KIND, int BN, bool SPLITK>
__global__ void __launch_bounds__(NUM_THREADS, (BN <= 64 && !SPLITK) ? 2 : 1)
conv_igemm_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                  const __grid_constant__ CUtensorMap map_out, const __grid_constant__ CUtensorMap map_res,
                  const ConvKParams p, const uint32_t idesc) {
    // KIND_TF32X3: fp32 operands split as x = hi + lo (hi = top 19 bits); D += Ahi*Whi + Alo*Whi + Ahi*Wlo
    // keeps ~fp32 accuracy on the tf32 tensor pipe. The consumer warps split each landed A tile in shared
    // memory before they issue its MMAs; W is split on the host at pack time.
    constexpr bool X3 = (KIND == KIND_TF32X3);
    constexpr int MK = X3 ? KIND_TF32 : KIND;
    constexpr int SB = stage_bytes(BN, X3);
    constexpr int A_LO_OFF = A_STAGE_BYTES;                          // X3 only
    constexpr int B_OFF = X3 ? 2 * A_STAGE_BYTES : A_STAGE_BYTES;
    constexpr int B_LO_OFF = B_OFF + BN * STAGE_K_BYTES;             // X3 only
    constexpr int NI = BN < 128 ? BN : 128;                          // wgmma N
    constexpr int NB = BN / NI;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>(
        (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
    // split-K: the `split` CTAs of a cluster (along z) each take a contiguous range of the k loop, then
    // reduce-scatter: rank r receives everyone's partial sums for channel slice r (epi_bn = BN/split
    // channels) through distributed shared memory, finishes and stores that slice.
    // (compiled out of the SPLITK = false instantiations, which most layers use)
    const int split = SPLITK ? p.split : 1;
    const int rank = SPLITK ? static_cast<int>(cluster_ctarank()) : 0;
    const int epi_bn = SPLITK ? p.epi_bn : BN;
    const uint32_t slice_bytes = BLOCK_M * epi_bn * 4;    // one rank's raw 32-bit partial sums of a slice
    // [ring][split-K: (split-1) partial slices, written by the other ranks][residual][tables][barriers]
    uint8_t* part_tile = smem + p.stages * SB;
    uint8_t* res_tile = part_tile + (SPLITK ? (split - 1) * slice_bytes : 0u);
    float* bias_s = reinterpret_cast<float*>(res_tile + p.res_panels * BLOCK_M * p.res_pw);
    float* scale_s = bias_s + BN;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(scale_s + BN);
    uint64_t* empty_bar = full_bar + MAX_STAGES;
    uint64_t* res_full_bar = empty_bar + 2 * MAX_STAGES;
    uint64_t* part_bar = res_full_bar + 1;         // split-K: the other ranks' partial sums have landed
    uint32_t* spare_smem = reinterpret_cast<uint32_t*>(part_bar + 1);
    (void)spare_smem;

    const int warp_idx = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
#ifdef B200_TIMELINE
    uint32_t& tl_idx = spare_smem[1];
    if (threadIdx.x == 0) {
        tl_idx = atomicAdd(&g_tl_n, 1u) & (TL_CAP - 1);
        TlRec& r = g_tl[tl_idx];
        r.gt0 = tl_globaltimer();
        r.clk[0] = clock64();
        r.bx = blockIdx.x; r.by = blockIdx.y; r.bz = blockIdx.z;
        asm volatile("mov.u32 %0, %%smid;" : "=r"(r.smid));
        r.K = p.K; r.KS = p.KS; r.bn = BN; r.stages = p.stages;
    }
#endif
    const int subs_per_stage = STAGE_K_BYTES / p.chunk;
    const int num_stage_iters = (p.KS + subs_per_stage - 1) / subs_per_stage;
    const int m0 = blockIdx.x * BLOCK_M;
    const int n0 = blockIdx.y * BN;
    const int n0_epi = n0 + rank * epi_bn;     // first channel of the slice this CTA finishes
    // 16-channel groups of that slice which hold real channels (0: nothing to finish or store)
    const int own_groups = max(0, min(epi_bn, p.K - n0_epi) + 15) >> 4;
    const int it_begin = SPLITK ? num_stage_iters * rank / split : 0;
    const int it_end = SPLITK ? num_stage_iters * (rank + 1) / split : num_stage_iters;

    if (warp_idx == 0 && lane == 0) {
        tma_prefetch_desc(&map_a);
        tma_prefetch_desc(&map_b);
        tma_prefetch_desc(&map_out);
        if (p.res_panels > 0) tma_prefetch_desc(&map_res);
        for (int i = 0; i < p.stages; ++i) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], EPI_WARPS);   // one arrival per consumer warp once the slot's MMAs retired
        }
        mbar_init(res_full_bar, 1);
        if (SPLITK) {
            mbar_init(part_bar, 1);
            // every other rank sends 128 rows x 64 bytes per 16-channel group of this CTA's slice
            mbar_arrive_expect_tx(part_bar, (split - 1) * own_groups * BLOCK_M * 64);
        }
        fence_mbar_init();
    }
    __syncthreads();
    // rank 0's barrier must exist before a peer can complete bytes on it; this runs before the
    // grid-dependency wait, i.e. under the previous kernel's tail
    if (SPLITK) cluster_sync_all();
    if (threadIdx.x == 0) TL(1);

    // PDL: let the next kernel start its own prologue now; everything that reads the previous
    // kernel's outputs (activations, residual) happens after the wait below.
    pdl_launch_dependents();

    if (warp_idx == 0) {
        if (lane == 0) {
            // ===================== TMA producer =====================
            const uint32_t b_sub_bytes = BN * p.chunk;
            const uint32_t tx_per_sub = BLOCK_M * p.chunk + (X3 ? 2 : 1) * b_sub_bytes;
            // Weights do not depend on the previous kernel: the first trip round the ring gets its B tiles
            // (and the whole stage's expect_tx) before the grid-dependency wait, so their HBM / L2 latency
            // overlaps the previous kernel's tail. Only this thread reads the prior grid's output.
            const int npre = min(p.stages, it_end - it_begin);
            {
                int ks = it_begin * subs_per_stage;
                uint32_t full_sa = smem_u32(full_bar), b_dst0 = smem_u32(smem) + B_OFF;
#pragma unroll 1
                for (int i = 0; i < npre; ++i) {
                    // always a full stage: k-steps past KS_real re-read tap (0,0) against zero weights (the weight
                    // map zero-fills k beyond its extent)
                    mbar_arrive_expect_tx_sa(full_sa, subs_per_stage * tx_per_sub);
                    uint32_t b_dst = b_dst0;
#pragma unroll 1
                    for (int j = 0; j < subs_per_stage; ++j) {
                        tma_load_2d_sa(&map_b, full_sa, b_dst, ks * p.chunk_el, n0);
                        if (X3) tma_load_2d_sa(&map_b, full_sa, b_dst + (B_LO_OFF - B_OFF), ks * p.chunk_el, p.K + n0);
                        b_dst += b_sub_bytes;
                        ++ks;
                    }
                    full_sa += 8; b_dst0 += SB;
                }
            }
            // (all coordinate arithmetic happens before the wait too: nothing but TMA issues follow it)
            const int n_img = m0 / p.HoWo;
            const int rem = m0 - n_img * p.HoWo;
            const int p0 = rem / p.Wo;
            const int q0 = rem - p0 * p.Wo;
            const int base_w = q0 * p.stride_w - p.pad_w;
            const int base_h = p0 * p.stride_h - p.pad_h;
            const uint32_t a_sub_bytes = BLOCK_M * p.chunk;
            // lean single-thread loop: 32-bit shared addresses and running coordinates only
            const uint32_t ring_sa = smem_u32(smem), full_sa0 = smem_u32(full_bar), empty_sa0 = smem_u32(empty_bar);
            int ks = it_begin * subs_per_stage;
            int cc = ks % p.CC;
            const int tap0 = ks / p.CC;
            int r = tap0 / p.S, s = tap0 - r * p.S;
            int c_coord = cc * p.chunk_el, k_coord = ks * p.chunk_el;
            int off_w = s * p.dil_w, off_h = r * p.dil_h;
            int stage = 0;
            uint32_t phase = 0, stage_sa = ring_sa, full_sa = full_sa0, empty_sa = empty_sa0;
            const int res_cols_per_panel = p.res_panels > 0 ? p.res_pw / p.res_es : 0;
            int pre_left = npre;
            pdl_wait_prior_grid();
            TL(2);
            for (int it = it_begin; it < it_end; ++it) {
                const bool pre = pre_left > 0;   // first trip: slot free, B + expect_tx already issued
                --pre_left;
                if (!pre) {
                    mbar_wait_sa(empty_sa, phase ^ 1);
                    mbar_arrive_expect_tx_sa(full_sa, subs_per_stage * tx_per_sub);
                }
                uint32_t a_dst = stage_sa, b_dst = stage_sa + B_OFF, bl_dst = stage_sa + B_LO_OFF;
#pragma unroll 1
                for (int j = 0; j < subs_per_stage; ++j) {
                    // padding k-steps (ks >= KS_real) re-read tap (0,0); their weights are zero
                    const bool pad_step = ks >= p.KS_real;
                    tma_load_im2col_4d_sa(&map_a, full_sa, a_dst, pad_step ? 0 : c_coord, base_w, base_h, n_img,
                                          static_cast<uint16_t>(pad_step ? 0 : off_w),
                                          static_cast<uint16_t>(pad_step ? 0 : off_h));
                    if (!pre) {
                        tma_load_2d_sa(&map_b, full_sa, b_dst, k_coord, n0);
                        if (X3)  // the W-low image follows the W-high image (row offset K)
                            tma_load_2d_sa(&map_b, full_sa, bl_dst, k_coord, p.K + n0);
                    }
                    a_dst += a_sub_bytes; b_dst += b_sub_bytes; bl_dst += b_sub_bytes;
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
                if (it == it_begin && p.res_panels > 0 && own_groups > 0) {
                    // the residual tile is only needed by the epilogue: after the first operand stage is on its way
                    mbar_arrive_expect_tx(res_full_bar, p.res_panels * BLOCK_M * p.res_pw);
                    for (int j = 0; j < p.res_panels; ++j)
                        tma_load_2d(&map_res, res_full_bar, res_tile + j * BLOCK_M * p.res_pw,
                                    n0_epi + j * res_cols_per_panel, m0);
                }
            }
        }
    } else if (warp_idx >= EPI_TID0 / 32) {
        // ===================== consumer warpgroups: wgmma main loop, then the epilogue =====================
        const int etid = threadIdx.x - EPI_TID0;
        const int cwg = etid >> 7;                                    // GEMM rows [64 cwg, 64 cwg + 64)
        const int row = 64 * cwg + 16 * ((etid >> 5) & 3) + acc_row16_row(lane);
        // bias / scale tables (weights-side constants)
        fill_epilogue_tables<EPI_THREADS>(p, n0_epi, epi_bn, etid, bias_s, scale_s);
        uint32_t acc[NB][NI / 2];
#pragma unroll
        for (int nb = 0; nb < NB; ++nb)
#pragma unroll
            for (int i = 0; i < NI / 2; ++i) acc[nb][i] = 0u;
        {
            // descriptors as (lo, hi) words: lo = addr>>4 | LBO>>4 << 16, hi = SBO>>4 | layout << 30;
            // between MMAs only `lo` moves, by 32-bit adds
            const bool a_signed = idesc_a_signed(idesc);
            const uint32_t lt = layout_type_for_chunk(p.chunk);
            const uint32_t a_sub16 = (BLOCK_M * p.chunk) >> 4, b_sub16 = (BN * p.chunk) >> 4;
            const bool swz = p.chunk >= 32;
            const uint32_t hi = (swz ? (8u * p.chunk) >> 4 : 128u >> 4) | (lt << 29);
            const uint32_t a_lbo = (swz ? 1u : a_sub16) << 16, b_lbo = (swz ? 1u : b_sub16) << 16;
            // (16-byte chunks: one K=32B MMA spans two sub-tiles, LBO = sub-tile)
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
            int stage = 0, prev = -1;
            uint32_t phase = 0;
            for (int it = it_begin; it < it_end; ++it) {
                if (prev == stage) {   // single-stage ring: the slot must go back before it can refill
                    wgmma_wait<0>();
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&empty_bar[prev]);
                    prev = -1;
                }
                mbar_wait(&full_bar[stage], phase);
#ifdef B200_TIMELINE
                if (it == it_begin && etid == 0) TL(3);
#endif
                if (X3)   // split the landed fp32 A tile: hi in place, lo behind it
                    split_tf32x3(reinterpret_cast<uint4*>(smem + stage * SB), reinterpret_cast<uint4*>(smem + stage * SB + A_LO_OFF),
                                 A_STAGE_BYTES / 16, etid);
                const uint32_t st16 = ring16 + stage * (SB >> 4);
                const uint32_t a16 = st16 + a_wg16, b16 = st16 + (B_OFF >> 4);
                wgmma_fence();
#pragma unroll
                for (int m = 0; m < 4; ++m) {
                    const uint64_t ad = desc64(((a16 + a_off[m]) & 0x3FFFu) | a_lbo, hi);
#pragma unroll
                    for (int nb = 0; nb < NB; ++nb) {
                        const uint64_t bd = desc64(((b16 + nb * nb16 + b_off[m]) & 0x3FFFu) | b_lbo, hi);
                        wgmma<MK, NI>(acc[nb], ad, bd, a_signed, 1u);
                        if (X3) {
                            const uint64_t al = desc64(((a16 + (A_LO_OFF >> 4) + a_off[m]) & 0x3FFFu) | a_lbo, hi);
                            const uint64_t bl = desc64(((b16 + ((B_LO_OFF - B_OFF) >> 4) + nb * nb16 + b_off[m]) & 0x3FFFu) | b_lbo, hi);
                            wgmma<MK, NI>(acc[nb], al, bd, a_signed, 1u);
                            wgmma<MK, NI>(acc[nb], ad, bl, a_signed, 1u);
                        }
                    }
                }
                wgmma_commit();
                wgmma_wait<1>();   // the previous stage's MMAs have retired: its slot goes back to the producer
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
        }
        // every MMA of both warpgroups retired: the operand ring is free for the staging tile
        asm volatile("bar.sync 1, %0;" ::"n"(EPI_THREADS) : "memory");
        if (etid == 0) TL(5);

        if (SPLITK) {
            // scatter: every 16-channel group of this CTA's accumulators goes to the rank that owns its slice, as
            // asynchronous stores completing on that rank's mbarrier. Layout at the receiver:
            // [sender slot][16-channel group][row][16 x 32 bit], 64 contiguous bytes per thread.
            const uint32_t part_sa = smem_u32(part_tile), bar_sa = smem_u32(part_bar);
#pragma unroll
            for (int g = 0; g < BN / 32; ++g) {
                uint32_t v[16];
                acc_row16<NI>(acc[g / (NI / 32)], g % (NI / 32), v);
                const int c0 = acc_row16_col(lane, g);
                if (n0 + c0 >= p.K) continue;
                const int owner = c0 / epi_bn;
                if (owner == rank) continue;
                const int slot = rank - (rank > owner ? 1 : 0);
                const int grp = (c0 - owner * epi_bn) >> 4;
                const uint32_t d = map_to_cta(part_sa + slot * slice_bytes + (static_cast<uint32_t>(grp * BLOCK_M + row) << 6), owner);
                const uint32_t bar = map_to_cta(bar_sa, owner);
#pragma unroll
                for (int q4 = 0; q4 < 4; ++q4)
                    st_async_v4(d + q4 * 16, bar, v[4 * q4], v[4 * q4 + 1], v[4 * q4 + 2], v[4 * q4 + 3]);
            }
        }

        if (own_groups > 0) {
            if (p.res_panels > 0) mbar_wait(res_full_bar, 0);
            const PanelRow out_row = make_panel_row(smem_u32(smem), panel_lg(p.out_pw), row);
            const PanelRow res_row = make_panel_row(smem_u32(res_tile), panel_lg(p.res_pw ? p.res_pw : 128), row);
            const uint32_t bias_sa = smem_u32(bias_s), scale_sa = smem_u32(scale_s);
            const uint32_t part_sa = smem_u32(part_tile);
            if (SPLITK) mbar_wait(part_bar, 0);
            uint8_t* out_tile = smem;
            // fold the other ranks' partial sums into 16 accumulator columns (slot order: deterministic)
            auto add_partials = [&](uint32_t (&v)[16], int c0) {
                for (int sl = 0; sl < split - 1; ++sl) {
                    const uint32_t src = part_sa + sl * slice_bytes + (static_cast<uint32_t>((c0 >> 4) * BLOCK_M + row) << 6);
#pragma unroll
                    for (int q4 = 0; q4 < 4; ++q4) {
                        const uint4 t = lds128(src + q4 * 16);
                        if (MK == KIND_I8) {
                            v[4 * q4] += t.x; v[4 * q4 + 1] += t.y; v[4 * q4 + 2] += t.z; v[4 * q4 + 3] += t.w;
                        } else {
                            v[4 * q4] = __float_as_uint(__fadd_rn(__uint_as_float(v[4 * q4]), __uint_as_float(t.x)));
                            v[4 * q4 + 1] = __float_as_uint(__fadd_rn(__uint_as_float(v[4 * q4 + 1]), __uint_as_float(t.y)));
                            v[4 * q4 + 2] = __float_as_uint(__fadd_rn(__uint_as_float(v[4 * q4 + 2]), __uint_as_float(t.z)));
                            v[4 * q4 + 3] = __float_as_uint(__fadd_rn(__uint_as_float(v[4 * q4 + 3]), __uint_as_float(t.w)));
                        }
                    }
                }
            };
#pragma unroll
            for (int g = 0; g < BN / 32; ++g) {
                uint32_t v0[16];
                acc_row16<NI>(acc[g / (NI / 32)], g % (NI / 32), v0);
                const int c0 = acc_row16_col(lane, g) - (SPLITK ? rank * epi_bn : 0);   // column within the slice
                if (c0 < 0 || c0 >= epi_bn || n0_epi + c0 >= p.K) continue;   // TMA clips the unwritten columns
                if (SPLITK) add_partials(v0, c0);
                epilogue16<MK>(p, v0, c0, bias_sa, scale_sa, res_row, out_row);
            }
            fence_proxy_async_smem();                                          // staged tile -> visible to the TMA engine
            asm volatile("bar.sync 1, %0;" ::"n"(EPI_THREADS) : "memory");    // the consumer warps only
            if (etid == 0) {
                TL(6);
                const int cols_per_panel = p.out_pw / p.out_es;
                for (int j = 0; j < p.out_panels; ++j) {
                    if (n0_epi + j * cols_per_panel >= p.K) break;
                    tma_store_2d(&map_out, out_tile + j * BLOCK_M * p.out_pw, n0_epi + j * cols_per_panel, m0);
                }
                tma_store_commit();
                tma_store_wait_read();  // smem may be released once the engine has read it; the writes
                                        // complete before the grid is reported complete
#ifdef B200_TIMELINE
                TL(7);
                g_tl[tl_idx].gt1 = tl_globaltimer();
#endif
            }
        }
    }

    __syncthreads();
    // no CTA of the cluster exits while its asynchronous stores may still be in flight towards rank 0
    if (SPLITK) cluster_sync_all();
}

// ----------------------------------------------------------------- host side
template <int KIND, int BN, bool SPLITK>
static void launch_conv(b200_conv_plan* pl, void* stream) {
    constexpr auto kern = conv_igemm_kernel<KIND, BN, SPLITK>;
    opt_in_smem<kern>(MAX_SMEM);
    // split-K: the z-CTAs of one tile form a cluster
    launch_kernel(kern, pl->grid, dim3(NUM_THREADS), pl->smem_bytes, static_cast<cudaStream_t>(stream),
                  dim3(1, 1, pl->kp.split), pl->map_a, pl->map_b, pl->map_out, pl->map_res, pl->kp, pl->idesc);
    count_launch();
}

// conv_slab.cu, conv_persistent.cu
bool slab_plan_setup(b200_conv_plan* pl);
bool persistent_plan_setup(b200_conv_plan* pl);
int slab_bind_maps(b200_conv_plan* pl, const void* in, const void* res, void* out);
#ifdef B200_TIMELINE
int slab_debug_timeline(void* out, int max_recs);
#endif

}  // namespace b200

using namespace b200;

extern "C" {

int b200_conv_out_hw(const b200_conv_desc_t* d, int32_t* ho, int32_t* wo) {
    if (!d) return B200_INVALID_VALUE;
    Geometry g = make_geometry(d);
    if (!g.ok) return B200_INVALID_VALUE;
    if (ho) *ho = g.ho;
    if (wo) *wo = g.wo;
    return B200_SUCCESS;
}

int b200_conv_pooled_hw(const b200_conv_desc_t* d, int32_t* ho, int32_t* wo) {
    if (!d) return B200_INVALID_VALUE;
    Geometry g = make_geometry(d);
    if (!g.ok) return B200_INVALID_VALUE;
    int32_t oh = g.ho, ow = g.wo;
    if (d->fuse_pool) {
        b200_pool_desc_t pd;
        memset(&pd, 0, sizeof(pd));
        pd.dtype = d->out_dtype; pd.type = B200_POOL_MAX; pd.n = d->n; pd.h = g.ho; pd.w = g.wo; pd.c = d->k;
        pd.window_h = pd.window_w = d->fuse_pool;
        pd.stride_h = pd.stride_w = d->pool_stride > 0 ? d->pool_stride : 2;
        pd.pad_h = pd.pad_w = d->pool_pad;
        pd.floor_as_conv = d->pool_floor_as_conv;
        int st = b200_pool_out_hw(&pd, &oh, &ow);
        if (st != B200_SUCCESS) return st;
    }
    if (ho) *ho = oh;
    if (wo) *wo = ow;
    return B200_SUCCESS;
}

size_t b200_conv_packed_weight_bytes(const b200_conv_desc_t* d) {
    if (!d) return 0;
    Geometry g = make_geometry(d);
    if (!g.ok) return 0;
    return static_cast<size_t>(d->k) * g.KS * g.chunk * (d->math == B200_MATH_TF32X3 ? 2 : 1);
}

int b200_conv_pack_weights(const b200_conv_desc_t* d, const void* src_kcrs, int32_t c_real, void* dst_packed) {
    if (!d || !src_kcrs || !dst_packed) return B200_INVALID_VALUE;
    Geometry g = make_geometry(d);
    if (!g.ok || c_real > d->c || c_real <= 0) return B200_INVALID_VALUE;
    const size_t row_bytes = static_cast<size_t>(g.KS) * g.chunk;
    memset(dst_packed, 0, row_bytes * d->k * (d->math == B200_MATH_TF32X3 ? 2 : 1));
    const int es = g.es;
    const uint8_t* src = static_cast<const uint8_t*>(src_kcrs);
    uint8_t* dst = static_cast<uint8_t*>(dst_packed);
    const int RS = d->r * d->s;
    for (int ko = 0; ko < d->k; ++ko) {
        for (int rs = 0; rs < RS; ++rs) {
            for (int c = 0; c < c_real; ++c) {
                const size_t s_off = ((static_cast<size_t>(ko) * c_real + c) * RS + rs) * es;
                const size_t d_off = ko * row_bytes + (static_cast<size_t>(rs) * d->c + c) * es;
                if (d->math == B200_MATH_TF32X3) {
                    // W = hi + lo, hi = top 19 bits; the low image follows the high image
                    uint32_t u;
                    memcpy(&u, src + s_off, 4);
                    const uint32_t hu = u & 0xFFFFE000u;
                    float x, h;
                    memcpy(&x, &u, 4);
                    memcpy(&h, &hu, 4);
                    const float l = x - h;
                    memcpy(dst + d_off, &h, 4);
                    memcpy(dst + row_bytes * d->k + d_off, &l, 4);
                } else {
                    memcpy(dst + d_off, src + s_off, es);
                }
            }
        }
    }
    return B200_SUCCESS;
}

int b200_conv_plan_create(const b200_conv_desc_t* d, const void* packed_weights_dev, const float* bias_dev,
                          const float* scale_dev, b200_conv_plan_t** plan_out) {
    if (!d || !packed_weights_dev || !plan_out) return B200_INVALID_VALUE;
    if (!device_is_sm90()) return B200_WRONG_DEVICE;
    if (d->math != B200_MATH_I8 && d->math != B200_MATH_F16 && d->math != B200_MATH_TF32 &&
        d->math != B200_MATH_TF32X3)
        return B200_UNIMPL_ERROR;
    if (d->fuse_pool < 0 || d->pool_stride < 0 || d->pool_pad < 0) return B200_INVALID_VALUE;
    // fused pooling lives in the slab kernel's epilogue (a CTA owns a rectangle of the output): stride-1 r x s filters
    if (d->fuse_pool != 0 && (d->res_dtype >= 0 || d->r * d->s < 2 || d->stride_h != 1 || d->stride_w != 1 ||
                              d->dil_h != 1 || d->dil_w != 1 || (d->k * dtype_size(d->out_dtype)) % 16 != 0))
        return B200_UNIMPL_ERROR;
    if (!tensor_maps_available()) return B200_NOT_INITIALIZED;
    Geometry g = make_geometry(d);
    if (!g.ok) return B200_INVALID_VALUE;
    // operand / epilogue dtype consistency
    if (d->math == B200_MATH_I8 && !(d->in_dtype == B200_INT8 || d->in_dtype == B200_UINT8)) return B200_INVALID_VALUE;
    if (d->math == B200_MATH_F16 && d->in_dtype != B200_HALF) return B200_INVALID_VALUE;
    if ((d->math == B200_MATH_TF32 || d->math == B200_MATH_TF32X3) && d->in_dtype != B200_FLOAT) return B200_INVALID_VALUE;
    if (d->ldc < d->k) return B200_INVALID_VALUE;
    const int out_es = dtype_size(d->out_dtype);
    const int res_es = d->res_dtype >= 0 ? dtype_size(d->res_dtype) : 0;
    // the output / residual tiles move by TMA: row pitch must be a 16-byte multiple
    if ((static_cast<int64_t>(d->ldc) * out_es) % 16 != 0) return B200_INVALID_VALUE;
    if (res_es && (static_cast<int64_t>(d->ldc) * res_es) % 16 != 0) return B200_INVALID_VALUE;
    // TMA im2col hardware limits (corner and offset field widths for 2 spatial dims)
    const int up_w = d->pad_w - (d->s - 1) * d->dil_w, up_h = d->pad_h - (d->r - 1) * d->dil_h;
    if (d->pad_w > 127 || d->pad_h > 127 || up_w < -128 || up_h < -128 || up_w > 127 || up_h > 127 ||
        (d->s - 1) * d->dil_w > 254 || (d->r - 1) * d->dil_h > 254 || d->stride_w > 8 || d->stride_h > 8)
        return B200_UNIMPL_ERROR;

    b200_conv_plan* pl = new (std::nothrow) b200_conv_plan();
    if (!pl) return B200_MEM_ALLOC_FAILED;
    pl->desc = *d;
    pl->g = g;
    pl->weights = packed_weights_dev;
    pl->map_a_ptr = pl->map_out_ptr = pl->map_res_ptr = nullptr;

    // ---- tile-N heuristic: widest tile that still yields >= ~1 wave of CTAs
    const int tiles_m = static_cast<int>((g.M_total + BLOCK_M - 1) / BLOCK_M);
    const int kr32 = (d->k + 31) / 32 * 32;
    const int sms = sm_count();
    const int max_bn = max_bn_for(out_es, res_es);
    int bn = 32;
    bool found = false;
    const int cands[4] = {256, 128, 64, 32};
    for (int i = 0; i < 4 && !found; ++i) {
        if (cands[i] > max_bn) continue;
        if (cands[i] > kr32 && cands[i] != 32) continue;
        const int ctas = tiles_m * ((d->k + cands[i] - 1) / cands[i]);
        if (ctas >= sms) { bn = cands[i]; found = true; }
    }
    if (!found) {
        // not enough work for a full wave: maximise the CTA count, but keep N >= 64 when free
        bn = 32;
        if (kr32 >= 64 && tiles_m * ((d->k + 63) / 64) == tiles_m * ((d->k + 31) / 32)) bn = 64;
        // fp32 operands: a k-iteration is 4 (tf32) or 12 (3xtf32) MMAs whose cost barely depends on N below 64, and
        // the long k loops of these layers are split over a cluster anyway: the wider tile halves the MMA count per
        // output (a choice carried over from the sm_100 version, not re-measured on the H100)
        if ((d->math == B200_MATH_TF32 || d->math == B200_MATH_TF32X3) && kr32 >= 64 &&
            static_cast<int64_t>(g.KS) * g.chunk >= 2048)
            bn = 64;
    }
    if (const int fb = forced_bn(max_bn)) bn = fb;
    pl->bn = bn;
    pl->grid = dim3(tiles_m, (d->k + bn - 1) / bn, 1);
    const int ctas = tiles_m * static_cast<int>(pl->grid.y);

    const int kind = kind_for_math(d->math);
    pl->launch = bind_kind_bn<32, 64, 128, 256>(kind, bn, [](auto K, auto N) -> ConvLaunch { return launch_conv<K, N, false>; });
    if (!pl->launch) { delete pl; return B200_UNIMPL_ERROR; }
    pl->idesc = conv_idesc(d->math, d->in_dtype, bn);

    if (encode_weights_map(pl, bn) != B200_SUCCESS) { delete pl; return B200_INVALID_VALUE; }

    ConvKParams& kp = pl->kp;
    memset(&kp, 0, sizeof(kp));
    kp.M_total = static_cast<int32_t>(g.M_total);
    kp.HoWo = g.ho * g.wo;
    kp.Wo = g.wo;
    kp.pad_h = d->pad_h; kp.pad_w = d->pad_w;
    kp.stride_h = d->stride_h; kp.stride_w = d->stride_w;
    kp.dil_h = d->dil_h; kp.dil_w = d->dil_w;
    kp.R = d->r; kp.S = d->s;
    kp.CC = g.CC; kp.chunk = g.chunk; kp.chunk_el = g.chunk_el;
    kp.KS = g.KS; kp.KS_real = g.KS_real;
    kp.K = d->k;
    kp.relu = d->relu; kp.neg_slope = d->neg_slope; kp.sum_scale = d->sum_scale;
    kp.out_dtype = d->out_dtype; kp.res_dtype = d->res_dtype;
    kp.bias = bias_dev; kp.scale = scale_dev;
    kp.out_es = out_es;
    kp.res_es = res_es;

    // ---- pipeline depth: as deep as the k loop needs, within the shared-memory budget. A grid that
    // exceeds one wave keeps two CTAs per SM resident (epilogue of one overlaps the main loop of the
    // other); a sub-wave grid takes the whole SM for latency hiding on its long k loop.
    const int sb = stage_bytes(bn, d->math == B200_MATH_TF32X3);
    const int subs = STAGE_K_BYTES / g.chunk;
    const int k_iters = (g.KS + subs - 1) / subs;
    // split-K for sub-wave grids with a long k loop (deep 3x3 / wide 1x1 layers on small feature maps):
    // one SM's TMA engine cannot feed such a loop fast enough, so 2 or 4 CTAs (a cluster) share it.
    int split = 1;
    static const bool split_enabled = [] { const char* e = getenv("B200_SABER_SPLITK"); return !(e && e[0] == '0'); }();
    // Splitting pays only for long k loops on grids that stay within one wave: the cluster barriers and the DSMEM
    // exchange cost a fixed time. Float kinds split from 16 iterations (their k loops move 2-4x the bytes per MAC), int8
    // from 24. These thresholds were tuned on the earlier sm_100 version of this kernel and have NOT been re-measured on
    // the H100.
    static const int split_min_env = [] { const char* e = getenv("B200_SABER_SPLIT_MIN_ITERS"); const int v = e ? atoi(e) : 0; return v > 0 ? v : 0; }();
    const int split_min_iters = split_min_env ? split_min_env : (d->math == B200_MATH_I8 ? 24 : 16);
    if (split_enabled && k_iters >= split_min_iters && ctas * 2 <= sms) {
        split = 2;
        if (k_iters >= 32 && ctas * 4 <= sms) split = 4;
    }
    if (const char* e = getenv("B200_SABER_FORCE_SPLIT")) {   // tuning experiments only
        const int fs = atoi(e);
        if ((fs == 1 || fs == 2 || fs == 4 || fs == 8) && k_iters >= fs) split = fs;
    }
    while (split > 1 && (bn / split) % 16) split >>= 1;      // a slice is whole 16-channel groups
    if (split > 1) {
        // split-K instantiations exist for the narrow tiles only (the heuristic never splits wide ones)
        const ConvLaunch l = bind_kind_bn<32, 64, 128>(kind, bn, [](auto K, auto N) -> ConvLaunch { return launch_conv<K, N, true>; });
        if (l) pl->launch = l;
        else split = 1;   // wide tile: no split variant
    }
    kp.split = split;
    // each rank of a split cluster finishes and stores a slice of epi_bn channels (reduce-scatter)
    const int epi_bn = bn / split;
    kp.epi_bn = epi_bn;
    kp.out_pw = epi_bn * out_es >= 128 ? 128 : epi_bn * out_es;
    kp.out_panels = epi_bn * out_es / kp.out_pw;
    kp.res_pw = res_es ? (epi_bn * res_es >= 128 ? 128 : epi_bn * res_es) : 0;
    kp.res_panels = res_es ? epi_bn * res_es / kp.res_pw : 0;
    const int res_bytes = BLOCK_M * epi_bn * res_es;
    const int fixed = res_bytes + tail_bytes(bn) + 1024;
    const int staging = BLOCK_M * epi_bn * out_es;
    const int part_bytes = (split - 1) * BLOCK_M * epi_bn * 4;   // the other ranks' partial sums of this slice
    pl->grid.z = split;
    const int k_iters_local = (k_iters + split - 1) / split;
    // Every CTA keeps to half of the SM's shared memory so that two CTAs are always co-resident: the next
    // kernel's prologue + weight prefetch (PDL) and the kernels of other streams (the Worker serves several
    // requests at once) overlap this one instead of queueing behind it. Measured on ResNet-50 INT8 b8: one
    // stream 354 -> 348 us, six Worker streams 24.4k -> 40.8k img/s. B200_SABER_SMEM_FULL=1 restores the deep
    // ring for sub-wave grids (slightly better for a single batch-1 stream).
    static const bool smem_full = [] { const char* e = getenv("B200_SABER_SMEM_FULL"); return e && e[0] == '1'; }();
    const int fixed_all = fixed + part_bytes;
    const int half_budget = MAX_SMEM / 2 - 2048;
    int budget = half_budget;
    if (ctas * split <= sms) {
        // a sub-wave grid may take the whole SM when half of it cannot hold a useful ring (wide int8 tiles with a
        // long k loop, and every 3xTF32 tile, whose stages are twice as large): 2 stages would serialise TMA and MMA
        const int stages_half = (half_budget - fixed_all) / sb;
        if (smem_full || stages_half < (k_iters_local < 4 ? k_iters_local : 4)) budget = MAX_SMEM;
    }
    int stages = (budget - fixed_all) / sb;
    if (stages > k_iters_local) stages = k_iters_local;
    if (stages > MAX_STAGES) stages = MAX_STAGES;
    const int min_stages = (staging + sb - 1) / sb;   // the ring doubles as the output staging tile
    if (stages < min_stages) stages = min_stages;
    if (stages < 1) stages = 1;
    if (stages < 2 && k_iters >= 2 && 2 * sb + fixed_all <= MAX_SMEM) stages = 2;  // never serialise load / MMA
    if (stages * sb + fixed_all > MAX_SMEM) { delete pl; return B200_OUT_OF_MEM; }
    kp.stages = stages;
    pl->smem_bytes = stages * sb + fixed_all;
    // ---- stride-1 R x S layers: the slab-staged kernel (conv_slab.cu) when it applies and its estimate beats this plan's
    static const bool verbose = [] { const char* e = getenv("B200_SABER_VERBOSE"); return e && e[0] == '1'; }();
    if (slab_plan_setup(pl)) {
        if (verbose)
            fprintf(stderr, "[b200_saber] plan slab  n%d %dx%d c%d k%d %dx%d | tile %dx%d (pitch %d) BN %d grid %ux%u slabs %d groups %d smem %d\n",
                    d->n, d->h, d->w, d->c, d->k, d->r, d->s, pl->sp.th, pl->sp.tw, pl->sp.PW, pl->bn, pl->grid.x, pl->grid.y,
                    pl->sp.SA, pl->sp.SB, pl->smem_bytes);
        *plan_out = pl;
        return B200_SUCCESS;
    }
    if (d->fuse_pool != 0) { delete pl; return B200_UNIMPL_ERROR; }   // no rectangle tiling holds this window
    const bool persistent = persistent_plan_setup(pl);
    if (verbose && persistent)
        fprintf(stderr, "[b200_saber] plan persistent: %u x %u tiles on %d CTAs, stages %d smem %d\n", pl->grid.x, pl->grid.y,
                pl->persistent_ctas, pl->kp.stages, pl->smem_bytes);
    if (verbose)
        fprintf(stderr, "[b200_saber] plan im2col n%d %dx%d c%d k%d %dx%d s%d | BN %d split %d grid %ux%u stages %d smem %d\n",
                d->n, d->h, d->w, d->c, d->k, d->r, d->s, d->stride_h, bn, split, pl->grid.x, pl->grid.y, stages, pl->smem_bytes);
    *plan_out = pl;
    return B200_SUCCESS;
}

int b200_conv_plan_run(b200_conv_plan_t* pl, const void* in, const void* res, void* out, void* stream) {
    if (!pl || !in || !out) return B200_INVALID_VALUE;
    const b200_conv_desc_t& d = pl->desc;
    if (d.res_dtype >= 0 && !res) return B200_INVALID_VALUE;
    if (pl->slab) {
        int st = slab_bind_maps(pl, in, res, out);
        if (st != B200_SUCCESS) return st;
        pl->launch(pl, stream);
        cudaError_t e = cudaPeekAtLastError();
        if (e != cudaSuccess) {
            fprintf(stderr, "[b200_saber] conv (slab) launch failed: %s\n", cudaGetErrorString(e));
            return B200_UNKNOWN_ERROR;
        }
        return B200_SUCCESS;
    }
    if (in != pl->map_a_ptr) {
        int st = encode_im2col_map(pl, in);
        if (st != B200_SUCCESS) return st;
    }
    if (out != pl->map_out_ptr) {
        int st = encode_tile_map(&pl->map_out, out, d.out_dtype, d.k, pl->g.M_total, d.ldc, pl->kp.out_pw);
        if (st != B200_SUCCESS) return st;
        pl->map_out_ptr = out;
    }
    if (d.res_dtype >= 0 && res != pl->map_res_ptr) {
        int st = encode_tile_map(&pl->map_res, res, d.res_dtype, d.k, pl->g.M_total, d.ldc, pl->kp.res_pw);
        if (st != B200_SUCCESS) return st;
        pl->map_res_ptr = res;
    } else if (d.res_dtype < 0 && pl->map_res_ptr == nullptr) {
        pl->map_res = pl->map_out;  // placeholder: never dereferenced when res_panels == 0
    }
    pl->launch(pl, stream);
    cudaError_t e = cudaPeekAtLastError();
    if (e != cudaSuccess) {
        fprintf(stderr, "[b200_saber] conv launch failed: %s\n", cudaGetErrorString(e));
        return B200_UNKNOWN_ERROR;
    }
    return B200_SUCCESS;
}

void b200_conv_plan_destroy(b200_conv_plan_t* pl) {
    delete pl;
}

int b200_conv_plan_info(const b200_conv_plan_t* pl, int32_t* block_n, int32_t* grid_x, int32_t* grid_y,
                        int32_t* k_steps, int32_t* smem_bytes) {
    if (!pl) return B200_INVALID_VALUE;
    if (block_n) *block_n = pl->bn;
    if (grid_x) *grid_x = pl->grid.x;
    if (grid_y) *grid_y = pl->grid.y;
    if (k_steps) *k_steps = pl->g.KS;
    if (smem_bytes) *smem_bytes = pl->smem_bytes;
    return B200_SUCCESS;
}

int b200_conv_plan_split(const b200_conv_plan_t* pl) { return pl ? static_cast<int>(pl->grid.z) : 0; }

int b200_conv_plan_is_slab(const b200_conv_plan_t* pl) { return pl && pl->slab ? 1 : 0; }

int b200_conv_plan_is_persistent(const b200_conv_plan_t* pl) { return pl && pl->persistent ? 1 : 0; }

int b200_fc_desc(b200_conv_desc_t* d, int32_t math, int32_t in_dtype, int32_t out_dtype, int32_t m, int32_t k_in,
                 int32_t n_out) {
    if (!d) return B200_INVALID_VALUE;
    memset(d, 0, sizeof(*d));
    d->math = math; d->in_dtype = in_dtype; d->out_dtype = out_dtype; d->res_dtype = -1;
    d->n = m; d->h = 1; d->w = 1; d->c = k_in; d->k = n_out; d->ldc = n_out;
    d->r = d->s = 1; d->stride_h = d->stride_w = 1; d->dil_h = d->dil_w = 1;
    d->sum_scale = 1.f;
    return B200_SUCCESS;
}

}  // extern "C"

#ifdef B200_TIMELINE
// debug only: copy out and reset the phase timeline (record layout = TlRec, 112 bytes)
extern "C" B200_API int b200_debug_timeline(void* out, int max_recs) {
    unsigned n = 0;
    cudaDeviceSynchronize();
    cudaMemcpyFromSymbol(&n, b200::g_tl_n, sizeof(n));
    if (n > b200::TL_CAP) n = b200::TL_CAP;
    if (static_cast<int>(n) > max_recs) n = max_recs;
    if (out && n) cudaMemcpyFromSymbol(out, b200::g_tl, n * sizeof(b200::TlRec));
    const unsigned zero = 0;
    cudaMemcpyToSymbol(b200::g_tl_n, &zero, sizeof(zero));
    // records of the slab kernel live in its own translation unit
    const int more = b200::slab_debug_timeline(out ? static_cast<char*>(out) + n * sizeof(b200::TlRec) : nullptr,
                                               max_recs - static_cast<int>(n));
    return static_cast<int>(n) + more;
}
#endif
