// Slab-staged stride-1 R x S convolution on Hopper tensor cores (wgmma, sm_90a).
//
// The TMA-im2col kernel (conv_igemm.cu) fetches the A operand once per filter tap: a 3x3 layer pulls every input
// pixel through the SM's L2 port nine times, and that port is what bounds a convolution at inference batch sizes. Here a CTA owns a th x tw rectangle of one image's output. Per input-channel
// chunk it stages the (th+R-1) x (tw+S-1) input rectangle ONCE -- one tiled 4-D TMA box, halo zero-filled by the
// engine -- as rows of `chunk` bytes (the slab), and the R*S taps are MMAs whose A descriptors simply start
// (r*PW + s) rows further into the slab: the shared-memory swizzle is a function of the absolute address
// (the wgmma descriptor carries no base offset), so a row-shifted view of a TMA-written tile is a
// valid K-major operand. GEMM row m = i*PW + j is output pixel (p0+i, q0+j); the S-1 extra columns per row are
// computed and dropped.
//
// Replaces the same reference entry points as conv_igemm.cu for 3x3 / 5x5 / 7x7 stride-1 layers
// (saber/funcs/impl/cuda/saber_conv.cpp:17-585, sass winograd_conv* / direct_conv* families,
//  third-party/sass/include/sass_funcs.h:54-427).
//
// Pipelines: slab slots (full_a / empty_a) and weight-tile slots (full_b / empty_b) are separate mbarrier rings fed
// by one producer thread that issues whichever load has a free slot; two consumer warpgroups (warps 4..11, 64 GEMM
// rows each) issue the wgmma main loop with the accumulator in registers and then run the same fused epilogue as the im2col kernel, compacting the dropped columns while they stage the tile, and one
// thread stores it with a 4-D TMA box (which also clips the ragged image edges).
#include <stdio.h>
#include <string.h>

#include "conv_common.cuh"

namespace b200 {

constexpr int SLAB_MAX_A = 4;    // slab slots
constexpr int SLAB_MAX_B = 16;   // weight-tile slots

// smem: [slab ring][weight ring][residual tile][bias | scale][barriers: full_a, empty_a, full_b, empty_b,
//       (spare), res_full][spare]
__host__ __device__ constexpr int slab_tail_bytes(int bn) {
    return 2 * bn * 4 + (3 * SLAB_MAX_A + 2 * SLAB_MAX_B + 2) * 8 + 16;
}

template <int KIND, int BN>
__global__ void __launch_bounds__(NUM_THREADS, BN <= 64 ? 2 : 1)
conv_slab_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                 const __grid_constant__ CUtensorMap map_out, const __grid_constant__ CUtensorMap map_res,
                 const ConvKParams p, const SlabParams sp, const uint32_t idesc) {
    // KIND_TF32X3: fp32 operands split as x = hi + lo (hi = top 19 bits); D += Ahi*Whi + Alo*Whi + Ahi*Wlo keeps
    // ~fp32 accuracy on the tf32 tensor pipe. The consumer warps split every landed slab into a high plane (in place)
    // and a low plane (behind it) before they issue its MMAs; W is split on the host at pack time.
    constexpr bool X3 = (KIND == KIND_TF32X3);
    constexpr int MK = X3 ? KIND_TF32 : KIND;
    constexpr int PL = X3 ? 2 : 1;
    constexpr int NI = BN < 128 ? BN : 128;                          // wgmma N
    constexpr int NB = BN / NI;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>(
        (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
    uint8_t* slab_ring = smem + sp.a_off;
    uint8_t* b_ring = smem + sp.b_off;
    uint8_t* res_tile = smem + sp.epi_off;
    float* bias_s = reinterpret_cast<float*>(res_tile + p.res_panels * BLOCK_M * p.res_pw);
    float* scale_s = bias_s + BN;
    uint64_t* full_a = reinterpret_cast<uint64_t*>(scale_s + BN);
    uint64_t* empty_a = full_a + SLAB_MAX_A;
    uint64_t* full_b = empty_a + 2 * SLAB_MAX_A;
    uint64_t* empty_b = full_b + SLAB_MAX_B;
    uint64_t* res_full_bar = empty_b + SLAB_MAX_B + 1;
    uint32_t* spare_smem = reinterpret_cast<uint32_t*>(res_full_bar + 1);
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
        r.bx = blockIdx.x; r.by = blockIdx.y; r.bz = 0;
        asm volatile("mov.u32 %0, %%smid;" : "=r"(r.smid));
        r.K = p.K; r.KS = p.CC * p.R * p.S; r.bn = BN; r.stages = sp.SA * 100 + sp.SB;
    }
#endif

    // tile of this CTA
    int t = blockIdx.x;
    const int tj = t % sp.tiles_w; t /= sp.tiles_w;
    const int ti = t % sp.tiles_h;
    const int n_img = t / sp.tiles_h;
    const int p0 = ti * sp.step_h + sp.org_h, q0 = tj * sp.step_w + sp.org_w;
    const int n0 = blockIdx.y * BN;
    const int own_groups = max(0, min(BN, p.K - n0) + 15) >> 4;

    if (warp_idx == 0 && lane == 0) {
        tma_prefetch_desc(&map_a);
        tma_prefetch_desc(&map_b);
        tma_prefetch_desc(&map_out);
        if (p.res_panels > 0) tma_prefetch_desc(&map_res);
        for (int i = 0; i < sp.SA; ++i) { mbar_init(&full_a[i], 1); mbar_init(&empty_a[i], EPI_WARPS); }
        for (int i = 0; i < sp.SB; ++i) { mbar_init(&full_b[i], 1); mbar_init(&empty_b[i], EPI_WARPS); }
        mbar_init(res_full_bar, 1);
        fence_mbar_init();
    }
    __syncthreads();
    if (threadIdx.x == 0) TL(1);

    pdl_launch_dependents();
    uint32_t acc[NB][NI / 2];

    if (warp_idx == 0) {
        if (lane == 0) {
            // ===================== TMA producer =====================
            // Two rings, one thread: slab slots (one input-channel chunk each) and weight-group slots (the S taps of
            // one filter row of one chunk, S tiled loads on one barrier). All ring state is carried incrementally --
            // no division in the loop -- and whichever ring has a free slot is fed first.
            const uint32_t full_a_sa = smem_u32(full_a), empty_a_sa = smem_u32(empty_a);
            const uint32_t full_b_sa = smem_u32(full_b), empty_b_sa = smem_u32(empty_b);
            const uint32_t slab_sa = smem_u32(slab_ring), bring_sa = smem_u32(b_ring);
            const int total_g = p.CC * p.R;                    // weight groups, consumed in (cc, r) order
            const uint32_t plane_bytes = static_cast<uint32_t>(sp.btile_bytes) * p.S;   // the S tiles of one plane
            const uint32_t group_bytes = PL * plane_bytes;
            const uint32_t slot_a_bytes = PL * static_cast<uint32_t>(sp.slab_bytes);
            const int k_tap = p.CC * p.chunk_el;               // k distance between consecutive taps (tap-major packing)
            // weight group state
            int gb = 0, g_slot = 0, g_r = 0;
            uint32_t g_phase = 1;                              // parity to wait on the empty barrier (first trip: free)
            int g_k = 0;                                       // k coordinate of (cc, r, s = 0)
            int g_kcc = 0;                                     // cc * chunk_el
            auto issue_group = [&]() {
                const uint32_t bar = full_b_sa + 8 * g_slot;
                mbar_arrive_expect_tx_sa(bar, group_bytes);
                uint32_t dst = bring_sa + g_slot * group_bytes;
                int k = g_k;
                for (int s2 = 0; s2 < p.S; ++s2) {
                    tma_load_2d_sa(&map_b, bar, dst, k, n0);
                    if (X3) tma_load_2d_sa(&map_b, bar, dst + plane_bytes, k, p.K + n0);   // the W-low image follows the W-high one
                    dst += sp.btile_bytes;
                    k += k_tap;
                }
                ++gb;
                if (++g_slot == sp.SB) { g_slot = 0; g_phase ^= 1; }
                if (++g_r == p.R) { g_r = 0; g_kcc += p.chunk_el; g_k = g_kcc; }
                else g_k += p.S * k_tap;
            };
            // weights do not depend on the previous kernel: the first ring trip goes out before the grid dependency
            const int npre = min(sp.SB, total_g);
            for (int i = 0; i < npre; ++i) issue_group();
            pdl_wait_prior_grid();
            TL(2);
            int ia = 0, a_slot = 0;
            uint32_t a_phase = 1;
            int a_c = 0;
            while (ia < p.CC || gb < total_g) {
                if (ia < p.CC && (ia < sp.SA || mbar_try_wait_sa(empty_a_sa + 8 * a_slot, a_phase))) {
                    mbar_arrive_expect_tx_sa(full_a_sa + 8 * a_slot, sp.slab_box_bytes);
                    tma_load_4d_sa(&map_a, full_a_sa + 8 * a_slot, slab_sa + a_slot * slot_a_bytes, a_c, q0 - p.pad_w,
                                   p0 - p.pad_h, n_img);
                    if (ia == 0 && p.res_panels > 0 && own_groups > 0) {
                        // the residual tile is only needed by the epilogue: after the first slab is on its way
                        const int cols = p.res_pw / p.res_es;
                        mbar_arrive_expect_tx(res_full_bar, p.res_panels * sp.th * sp.tw * p.res_pw);
#pragma unroll 1
                        for (int j = 0; j < p.res_panels; ++j)
                            tma_load_4d_sa(&map_res, smem_u32(res_full_bar), smem_u32(res_tile) + j * BLOCK_M * p.res_pw,
                                           n0 + j * cols, q0, p0, n_img);
                    }
                    ++ia;
                    a_c += p.chunk_el;
                    if (++a_slot == sp.SA) { a_slot = 0; a_phase ^= 1; }
                }
                if (gb < total_g && (gb < sp.SB || mbar_try_wait_sa(empty_b_sa + 8 * g_slot, g_phase))) issue_group();
            }
        }
    } else if (warp_idx >= EPI_TID0 / 32) {
        // ===================== consumer warpgroups: wgmma main loop =====================
        const int etid = threadIdx.x - EPI_TID0;
        fill_epilogue_tables<EPI_THREADS>(p, n0, BN, etid, bias_s, scale_s);
#pragma unroll
        for (int nb = 0; nb < NB; ++nb)
#pragma unroll
            for (int i = 0; i < NI / 2; ++i) acc[nb][i] = 0u;
        const bool a_signed = idesc_a_signed(idesc);
        const uint32_t lt = layout_type_for_chunk(p.chunk);
        const uint32_t hi = ((8u * p.chunk) >> 4) | (lt << 29);   // SBO = 8 rows, swizzle
        const uint32_t lbo = 1u << 16;
        const uint32_t row16 = static_cast<uint32_t>(p.chunk) >> 4;            // one slab row in 16-byte units
        // this warpgroup's 64 GEMM rows start 64 rows into every tap view
        const uint32_t slab_d0 = (smem_u32(slab_ring) >> 4) + 64u * row16 * (etid >> 7), bring_d0 = smem_u32(b_ring) >> 4;
        const uint32_t slab16 = static_cast<uint32_t>(sp.slab_bytes) >> 4;
        const uint32_t btile16 = static_cast<uint32_t>(sp.btile_bytes) >> 4;
        const uint32_t pw16 = static_cast<uint32_t>(sp.PW) * row16;
        const uint32_t nb16 = NI * row16;
        const uint32_t plane16 = btile16 * p.S;            // X3: the low-plane tiles sit one plane behind the high ones
        const uint32_t group16 = PL * plane16;
        const uint32_t slot_a16 = PL * slab16;
        auto mma = [&](uint32_t a_lo, uint32_t b_lo) {
#pragma unroll
            for (int nb = 0; nb < NB; ++nb)
                wgmma<MK, NI>(acc[nb], desc64(((a_lo) & 0x3FFFu) | lbo, hi), desc64(((b_lo + nb * nb16) & 0x3FFFu) | lbo, hi),
                              a_signed, 1u);
        };
        // a weight group's slot (and, after the last filter row of a chunk, the slab slot) goes back to the producer once
        // the group's MMAs have retired: one group behind the issue -- or at once when the next wait is for that very
        // slot (single-slot rings)
        int a_slot = 0, b_slot = 0, prev_b = -1, prev_a = -1;
        uint32_t a_phase = 0, b_phase = 0;
        auto release_prev = [&]() {
            if (prev_b < 0) return;
            __syncwarp();
            if (lane == 0) {
                mbar_arrive(&empty_b[prev_b]);
                if (prev_a >= 0) mbar_arrive(&empty_a[prev_a]);
            }
            prev_b = prev_a = -1;
        };
#pragma unroll 1
        for (int cc = 0; cc < p.CC; ++cc) {
            if (prev_a == a_slot) { wgmma_wait<0>(); release_prev(); }
            mbar_wait(&full_a[a_slot], a_phase);
#ifdef B200_TIMELINE
            if (cc == 0 && etid == 0) TL(3);
#endif
            if (X3)   // split the landed fp32 slab: high plane in place, low plane behind it
                split_tf32x3(reinterpret_cast<uint4*>(slab_ring + a_slot * PL * sp.slab_bytes),
                             reinterpret_cast<uint4*>(slab_ring + a_slot * PL * sp.slab_bytes + sp.slab_bytes), sp.slab_box_bytes >> 4,
                             etid);
            uint32_t a_row = slab_d0 + a_slot * slot_a16;      // descriptor of tap (r, 0)
#pragma unroll 1
            for (int r = 0; r < p.R; ++r) {
                if (prev_b == b_slot) { wgmma_wait<0>(); release_prev(); }
                mbar_wait(&full_b[b_slot], b_phase);
                uint32_t a_tap = a_row, b_tile = bring_d0 + b_slot * group16;
                wgmma_fence();
#pragma unroll 1
                for (int s2 = 0; s2 < p.S; ++s2) {
                    // the 32-byte k slices of one chunk: descriptors differ by 2 (x 16 B)
#pragma unroll 1
                    for (uint32_t q = 0; q < 2u * sp.mma_per_tap; q += 2) {
                        mma(a_tap + q, b_tile + q);
                        if (X3) {
                            mma(a_tap + slab16 + q, b_tile + q);
                            mma(a_tap + q, b_tile + plane16 + q);
                        }
                    }
                    a_tap += row16;
                    b_tile += btile16;
                }
                wgmma_commit();
                wgmma_wait<1>();
                release_prev();
                prev_b = b_slot;
                prev_a = r == p.R - 1 ? a_slot : -1;
                if (++b_slot == sp.SB) { b_slot = 0; b_phase ^= 1; }
                a_row += pw16;
            }
            if (++a_slot == sp.SA) { a_slot = 0; a_phase ^= 1; }
        }
        wgmma_wait<0>();
#pragma unroll
        for (int nb = 0; nb < NB; ++nb) wgmma_fence_acc(acc[nb]);
        // every MMA of both warpgroups retired: both operand rings are free for the staging tile
        asm volatile("bar.sync 1, %0;" ::"n"(EPI_THREADS) : "memory");
        if (etid == 0) TL(5);
    }

    if (warp_idx >= EPI_TID0 / 32 && own_groups > 0) {
        const int etid = threadIdx.x - EPI_TID0;
        const int m = 64 * (etid >> 7) + 16 * ((etid >> 5) & 3) + acc_row16_row(lane);
        // GEMM row -> staging row: kept pixels are compacted to i*tw + j (the dense [th][tw] order the store box
        // reads); dropped rows go to the unused rows behind them, one each, so every thread runs the same code
        const int i = m / sp.PW, j = m - i * sp.PW;
        int row;
        if (i < sp.th && j < sp.tw) row = i * sp.tw + j;
        else if (i < sp.th) row = sp.th * sp.tw + i * (sp.PW - sp.tw) + (j - sp.tw);
        else row = m;
        if (p.res_panels > 0) mbar_wait(res_full_bar, 0);
        uint8_t* out_tile = smem;   // the operand rings, all consumed
        const PanelRow out_row = make_panel_row(smem_u32(out_tile), panel_lg(p.out_pw), row);
        const PanelRow res_row = make_panel_row(smem_u32(res_tile), panel_lg(p.res_pw ? p.res_pw : 128), row);
        const uint32_t bias_sa = smem_u32(bias_s), scale_sa = smem_u32(scale_s);
#pragma unroll
        for (int g = 0; g < BN / 32; ++g) {
            uint32_t v0[16];
            acc_row16<NI>(acc[g / (NI / 32)], g % (NI / 32), v0);
            const int c0 = acc_row16_col(lane, g);
            if (n0 + c0 >= p.K) continue;
            epilogue16<MK>(p, v0, c0, bias_sa, scale_sa, res_row, out_row);
        }
        fence_proxy_async_smem();
        asm volatile("bar.sync 1, %0;" ::"n"(EPI_THREADS) : "memory");
        if (sp.pool) {
            // fused MAX pooling: (pooled pixel, 16-byte channel group) items over the 256 epilogue threads; windows are
            // clipped to the conv output, so padding cells and the garbage rows of the rectangle never take part
            const int es = p.out_es;
            const int cpp = min(BN, p.K - n0) * es / 16;
            const int lgo = panel_lg(p.out_pw);
            const uint32_t stage_sa = smem_u32(out_tile);
            uint8_t* outp = static_cast<uint8_t*>(sp.out_ptr);
            for (int it = etid; it < sp.ph * sp.pw * cpp; it += EPI_THREADS) {
                const int c16 = it % cpp;
                const int e = it / cpp;
                const int oj = e % sp.pw, oi = e / sp.pw;
                const int gi = ti * sp.ph + oi, gj = tj * sp.pw + oj;
                if (gi >= sp.PHo || gj >= sp.PWo) continue;
                const int hs = max(gi * sp.ps - sp.pp, 0), he = min(gi * sp.ps - sp.pp + sp.pk, sp.Ho);
                const int ws = max(gj * sp.ps - sp.pp, 0), we = min(gj * sp.ps - sp.pp + sp.pk, sp.Wo);
                uint4 acc = make_uint4(0, 0, 0, 0);
                bool first = true;
                for (int y = hs; y < he; ++y) {
                    for (int x = ws; x < we; ++x) {
                        const uint4 v = lds128(panel_addr(make_panel_row(stage_sa, lgo, (y - p0) * sp.tw + (x - q0)), c16 * 16));
                        if (first) { acc = v; first = false; continue; }
                        acc = max16(acc, v, p.out_dtype);
                    }
                }
                const size_t o = ((static_cast<size_t>(n_img) * sp.PHo + gi) * sp.PWo + gj) * sp.out_ld_bytes +
                                 static_cast<size_t>(n0) * es + c16 * 16;
                *reinterpret_cast<uint4*>(outp + o) = acc;
            }
        } else if (etid == 0) {
            TL(6);
            const int cols_per_panel = p.out_pw / p.out_es;
            for (int jp = 0; jp < p.out_panels; ++jp) {
                if (n0 + jp * cols_per_panel >= p.K) break;
                tma_store_4d(&map_out, smem_u32(out_tile) + jp * BLOCK_M * p.out_pw, n0 + jp * cols_per_panel, q0, p0,
                             n_img);
            }
            tma_store_commit();
            tma_store_wait_read();
#ifdef B200_TIMELINE
            TL(7);
            g_tl[tl_idx].gt1 = tl_globaltimer();
#endif
        }
    }

    __syncthreads();
}

// ----------------------------------------------------------------- host side
template <int KIND, int BN>
static void launch_slab(b200_conv_plan* pl, void* stream) {
    constexpr auto kern = conv_slab_kernel<KIND, BN>;
    opt_in_smem<kern>(MAX_SMEM);
    launch_kernel(kern, pl->grid, dim3(NUM_THREADS), pl->smem_bytes, static_cast<cudaStream_t>(stream), dim3(1), pl->map_a,
                  pl->map_b, pl->map_out, pl->map_res, pl->kp, pl->sp, pl->idesc);
    count_launch();
}

// Whole-kernel time estimate (SM clocks) both conv kernels are compared with: a CTA costs its main loop (the slower
// of MMA issue and L2 ingest) + its epilogue + ~6000 clk of fixed latencies (prologue, first TMA round trip,
// accumulator read-out, store); CTAs beyond one per SM run in turns, two co-resident CTAs overlapping each other's
// fixed parts at the price of a shared SM. Cost model: conv_common.cuh.
static double conv_time_estimate(int ctas, double loop_clk, int bn, int out_es, bool two_per_sm) {
    const int sms = sm_count();
    const double cta = loop_clk + bn * (out_es == 4 ? 12.0 : 9.0) + 6000.0;
    if (ctas <= sms) return cta;
    const int r = two_per_sm ? 2 : 1;
    const double turns = static_cast<double>((ctas + sms * r - 1) / (sms * r));
    return turns * cta * (r == 2 ? 1.25 : 1.0);
}

namespace {
struct SlabLayout {
    SlabParams sp;
    int bn, smem_bytes, out_pw, out_panels, res_pw, res_panels;
    bool two_per_sm;
    double est_clk;
};

// Shared-memory layout of one (tile, BN) candidate; false when it cannot fit.
struct PoolTiling { int pk, ps, pp, ph, pw, PHo, PWo; };   // fused pooling: th x tw is the rectangle a ph x pw pooled tile needs

bool slab_layout(const b200_conv_desc_t& d, const Geometry& g, int th, int tw, int bn, SlabLayout* L,
                 const PoolTiling* pool = nullptr) {
    const bool x3 = d.math == B200_MATH_TF32X3;
    const int planes = x3 ? 2 : 1;
    const int out_es = dtype_size(d.out_dtype);
    const int res_es = d.res_dtype >= 0 ? dtype_size(d.res_dtype) : 0;
    SlabParams sp{};
    sp.Ho = g.ho; sp.Wo = g.wo;
    sp.th = th; sp.tw = tw; sp.PW = tw + d.s - 1;
    if (sp.th * sp.PW > BLOCK_M || sp.th + d.r - 1 > 256 || sp.PW > 256) return false;
    sp.tiles_h = (g.ho + th - 1) / th;
    sp.tiles_w = (g.wo + tw - 1) / tw;
    sp.step_h = th; sp.step_w = tw; sp.org_h = 0; sp.org_w = 0;
    if (pool) {
        sp.pool = 1; sp.pk = pool->pk; sp.ps = pool->ps; sp.pp = pool->pp;
        sp.ph = pool->ph; sp.pw = pool->pw; sp.PHo = pool->PHo; sp.PWo = pool->PWo;
        sp.tiles_h = (pool->PHo + pool->ph - 1) / pool->ph;
        sp.tiles_w = (pool->PWo + pool->pw - 1) / pool->pw;
        sp.step_h = pool->ph * pool->ps; sp.step_w = pool->pw * pool->ps;
        sp.org_h = sp.org_w = -pool->pp;
        sp.out_ld_bytes = d.ldc * dtype_size(d.out_dtype);
    }
    const int rows_alloc = ((BLOCK_M + (d.r - 1) * sp.PW + (d.s - 1)) + 7) & ~7;
    sp.slab_bytes = (rows_alloc * g.chunk + 1023) & ~1023;   // rows of `chunk` bytes; 8 rows = one swizzle period
    sp.slab_box_bytes = (th + d.r - 1) * sp.PW * g.chunk;
    sp.mma_per_tap = g.chunk / 32;
    sp.btile_bytes = bn * g.chunk;
    L->bn = bn;
    L->out_pw = bn * out_es >= 128 ? 128 : bn * out_es;
    L->out_panels = bn * out_es / L->out_pw;
    L->res_pw = res_es ? (bn * res_es >= 128 ? 128 : bn * res_es) : 0;
    L->res_panels = res_es ? bn * res_es / L->res_pw : 0;
    const int staging = BLOCK_M * bn * out_es;
    const int fixed = BLOCK_M * bn * res_es + slab_tail_bytes(bn) + 1024;
    const int slot_a = planes * sp.slab_bytes;                       // x3: the low plane follows the high plane
    const int slot_b = planes * d.s * sp.btile_bytes;                // one group: the S taps of a filter row (x3: hi + lo)
    const int total_groups = g.CC * d.r;
    auto fits = [&](int sa, int sb, int budget) { return sa * slot_a + sb * slot_b + fixed <= budget; };
    const int half_budget = MAX_SMEM / 2 - 2048;
    int sa = g.CC < 2 ? 1 : 2;
    int sb = total_groups < 3 ? total_groups : 3;
    int budget = half_budget;
    if (!fits(sa, sb, budget)) {
        budget = MAX_SMEM;
        while (sb > 2 && !fits(sa, sb, budget)) --sb;
        if (!fits(sa, sb, budget) && sa > 1) sa = 1;
        while (sb > 1 && !fits(sa, sb, budget)) --sb;
        if (!fits(sa, sb, budget)) return false;
    }
    // what is left of the budget: a deeper weight ring first (it hides the L2 latency of the k loop), then slabs
    while (sb < SLAB_MAX_B && sb < total_groups && fits(sa, sb + 1, budget)) ++sb;
    while (sa < SLAB_MAX_A && sa < g.CC && fits(sa + 1, sb, budget)) ++sa;
    int ring = sa * slot_a + sb * slot_b;
    if (ring < staging) {   // the staging tile must fit in the rings it reuses
        const int extra = (staging - ring + slot_b - 1) / slot_b;
        if (sb + extra > SLAB_MAX_B || !fits(sa, sb + extra, MAX_SMEM)) return false;
        sb += extra;
        ring = sa * slot_a + sb * slot_b;
        if (ring + fixed > half_budget) budget = MAX_SMEM;
    }
    sp.SA = sa; sp.SB = sb;
    sp.a_off = 0;
    sp.b_off = sa * slot_a;
    sp.epi_off = ring;
    L->smem_bytes = ring + fixed;
    if (L->smem_bytes > MAX_SMEM) return false;
    L->two_per_sm = L->smem_bytes <= half_budget + 2048;
    L->sp = sp;

    // ---- estimated time (SM clocks)
    const int RS = d.r * d.s;
    const int ctas = d.n * sp.tiles_h * sp.tiles_w * ((d.k + bn - 1) / bn);
    const double mma = static_cast<double>(g.CC) * RS * sp.mma_per_tap * (x3 ? 3 : 1) * mma_clk(bn);
    const double ingest =
        static_cast<double>(g.CC) * (sp.slab_box_bytes + static_cast<double>(planes) * RS * bn * g.chunk) / L2_INGEST_BYTES_PER_CLK;
    double loop = mma > ingest ? mma : ingest;
    if ((sa < 2 && g.CC > 1) || sb < 2) loop = mma + ingest;          // no double buffering: load and MMA serialise
    L->est_clk = conv_time_estimate(ctas, loop, bn, out_es, L->two_per_sm);
    return true;
}
}  // namespace

// Decide whether the slab variant serves this convolution and set the plan up for it (tile, BN, ring depths, smem).
// Returns false to leave the plan to the im2col kernel.
bool slab_plan_setup(b200_conv_plan* pl) {
    const b200_conv_desc_t& d = pl->desc;
    const Geometry& g = pl->g;
    // B200_SABER_SLAB: 0 never, 2 whenever it applies (tests), default: when its time estimate beats the im2col plan's
    const char* slab_env = getenv("B200_SABER_SLAB");
    if (!d.fuse_pool) {   // (a fused pooling has no other kernel to fall back to)
        if (slab_env && slab_env[0] == '0') return false;
        if (const char* e = getenv("B200_SABER_FORCE_SPLIT")) { if (atoi(e) > 1) return false; }   // split-K experiments
    }
    if (d.r * d.s < 2 || d.stride_h != 1 || d.stride_w != 1 || d.dil_h != 1 || d.dil_w != 1) return false;
    if (g.chunk < 32 || d.s > 16 || d.r > 16) return false;
    const int out_es = dtype_size(d.out_dtype);
    const int res_es = d.res_dtype >= 0 ? dtype_size(d.res_dtype) : 0;

    // ---- candidates: tile width = the row (or an equal part of it), tile height = what fits 128 GEMM rows, every
    // tile width of the kernel; the estimate weighs halo re-reads, weight re-reads per tile, MMA width and waves
    const int kr32 = (d.k + 31) / 32 * 32;
    const int max_bn = max_bn_for(out_es, res_es);
    const int force_bn = forced_bn(max_bn);
    SlabLayout best{};
    bool have = false;
    // Alternative rule (B200_SABER_SLAB_BN_RULE=1): the widest tile (<= 128) that still leaves >= 64 CTAs, the narrowest one
    // when no width reaches 64 CTAs. The wider tiles take the whole SM's shared memory, so the next layer's CTAs cannot
    // become resident early and its prologue + weight prefetch no longer hide under this layer (PDL); the estimate-driven
    // choice stays the default (decided on the sm_100 version, not re-measured on the H100).
    SlabLayout pick{};
    bool have_pick = false;
    auto consider = [&](const SlabLayout& L) {
        if (!have || L.est_clk < best.est_clk) { best = L; have = true; }
        if (L.bn > 128) return;
        const int ctas = d.n * L.sp.tiles_h * L.sp.tiles_w * ((d.k + L.bn - 1) / L.bn);
        const int pick_ctas = have_pick ? d.n * pick.sp.tiles_h * pick.sp.tiles_w * ((d.k + pick.bn - 1) / pick.bn) : 0;
        bool better;
        if (!have_pick) better = true;
        else if ((ctas >= 64) != (pick_ctas >= 64)) better = ctas >= 64;
        else if (ctas >= 64) better = L.bn > pick.bn || (L.bn == pick.bn && L.est_clk < pick.est_clk);
        else better = L.bn < pick.bn || (L.bn == pick.bn && L.est_clk < pick.est_clk);
        if (better) { pick = L; have_pick = true; }
    };
    const int parts[8] = {1, 2, 3, 4, 6, 8, 12, 16};
    if (d.fuse_pool) {
        // pooled tilings: a ph x pw tile of pooled pixels, its conv rectangle th x tw = ((ph-1)*ps + pk) x ((pw-1)*ps + pk)
        PoolTiling pt{};
        pt.pk = d.fuse_pool; pt.ps = d.pool_stride > 0 ? d.pool_stride : 2; pt.pp = d.pool_pad;
        int32_t pho = 0, pwo = 0;
        if (b200_conv_pooled_hw(&d, &pho, &pwo) != B200_SUCCESS) return false;
        pt.PHo = pho; pt.PWo = pwo;
        for (int pi = 0; pi < 8; ++pi) {
            const int pw = (pwo + parts[pi] - 1) / parts[pi];
            const int tw = (pw - 1) * pt.ps + pt.pk;
            const int PW = tw + d.s - 1;
            if (PW > BLOCK_M) continue;
            if (pi > 0 && pw < 2) break;
            const int rows = BLOCK_M / PW;                    // conv rows that fit
            if (rows < pt.pk) continue;
            int ph_max = (rows - pt.pk) / pt.ps + 1;
            if (ph_max > pho) ph_max = pho;
            const int tiles_h = (pho + ph_max - 1) / ph_max;
            pt.ph = (pho + tiles_h - 1) / tiles_h;
            pt.pw = pw;
            const int th = (pt.ph - 1) * pt.ps + pt.pk;
            const int cands[4] = {32, 64, 128, 256};
            for (int ci = 0; ci < 4; ++ci) {
                const int bn = cands[ci];
                if (force_bn ? bn != force_bn : (bn > max_bn || (bn > kr32 && bn != 32))) continue;
                SlabLayout L{};
                if (!slab_layout(d, g, th, tw, bn, &L, &pt)) continue;
                consider(L);
            }
        }
        if (!have) return false;
    }
    for (int pi = 0; pi < 8 && !d.fuse_pool; ++pi) {
        const int tw = (g.wo + parts[pi] - 1) / parts[pi];
        const int PW = tw + d.s - 1;
        if (PW > BLOCK_M) continue;
        if (pi > 0 && tw < 8) break;
        const int th_max = BLOCK_M / PW < g.ho ? BLOCK_M / PW : g.ho;
        if (th_max < 1) continue;
        const int tiles_h = (g.ho + th_max - 1) / th_max;
        const int th = (g.ho + tiles_h - 1) / tiles_h;          // equal-height tiles
        const int cands[4] = {32, 64, 128, 256};
        for (int ci = 0; ci < 4; ++ci) {
            const int bn = cands[ci];
            if (force_bn ? bn != force_bn : (bn > max_bn || (bn > kr32 && bn != 32))) continue;
            SlabLayout L{};
            if (!slab_layout(d, g, th, tw, bn, &L)) continue;
            consider(L);
        }
    }
    if (!have) return false;
    if (!d.fuse_pool) {
        // the complete im2col plan (pl->bn, grid, stages, smem): A is fetched once per tap; a ring of fewer than three
        // stages cannot overlap loads and MMAs
        const bool x3 = d.math == B200_MATH_TF32X3;
        const double k_bytes = static_cast<double>(g.KS) * g.chunk;
        const int bn0 = pl->bn;
        const double mma0 = k_bytes / 32.0 * (x3 ? 3 : 1) * mma_clk(bn0);
        const double ingest0 = (BLOCK_M + (x3 ? 2.0 : 1.0) * bn0) * k_bytes / L2_INGEST_BYTES_PER_CLK;
        double loop0 = mma0 > ingest0 ? mma0 : ingest0;
        if (pl->kp.stages < 3) loop0 = mma0 + ingest0;
        const int split0 = static_cast<int>(pl->grid.z);           // split-K cluster: the k loop is shared, plus the exchange
        if (split0 > 1) loop0 = loop0 / split0 + 2500.0;
        const double est0 = conv_time_estimate(static_cast<int>(pl->grid.x * pl->grid.y * pl->grid.z), loop0, bn0, out_es,
                                               pl->smem_bytes <= MAX_SMEM / 2);
        const bool force = slab_env && slab_env[0] == '2';
        if (!force && !force_bn && est0 <= best.est_clk) return false;
    }

    static const bool bn_rule = [] { const char* e = getenv("B200_SABER_SLAB_BN_RULE"); return e && e[0] == '1'; }();
    if (have_pick && bn_rule && !force_bn) best = pick;
    ConvKParams& kp = pl->kp;
    kp.epi_bn = best.bn;
    kp.split = 1;
    kp.out_es = out_es;
    kp.res_es = res_es;
    kp.out_pw = best.out_pw; kp.out_panels = best.out_panels;
    kp.res_pw = best.res_pw; kp.res_panels = best.res_panels;
    pl->smem_bytes = best.smem_bytes;
    const SlabParams& sp = best.sp;
    const int bn = best.bn;
    pl->bn = bn;
    pl->grid = dim3(d.n * sp.tiles_h * sp.tiles_w, (d.k + bn - 1) / bn, 1);
    pl->launch = bind_kind_bn<32, 64, 128, 256>(kind_for_math(d.math), bn,
                                                [](auto K, auto N) -> ConvLaunch { return launch_slab<K, N>; });
    if (!pl->launch) return false;
    if (encode_weights_map(pl, bn) != B200_SUCCESS) return false;   // the weight box follows THIS kernel's tile width
    pl->idesc = conv_idesc(d.math, d.in_dtype, bn);
    pl->sp = sp;
    pl->slab = true;
    return true;
}

// (re)encode the activation / output / residual maps of a slab plan for the buffers of this run
int slab_bind_maps(b200_conv_plan* pl, const void* in, const void* res, void* out) {
    const b200_conv_desc_t& d = pl->desc;
    const Geometry& g = pl->g;
    const SlabParams& sp = pl->sp;
    if (in != pl->map_a_ptr) {
        int st = encode_nhwc_map(&pl->map_a, in, operand_dtype(d.math), d.c, d.c, d.w, d.h, d.n, g.chunk_el, sp.PW,
                                 sp.th + d.r - 1, g.chunk);
        if (st != B200_SUCCESS) return st;
        pl->map_a_ptr = in;
    }
    if (sp.pool) {
        pl->sp.out_ptr = out;       // the pooled pixels are written with plain 16-byte stores
        if (pl->map_out_ptr == nullptr) { pl->map_out = pl->map_a; pl->map_out_ptr = out; }   // placeholder, never used
    } else if (out != pl->map_out_ptr) {
        int st = encode_nhwc_map(&pl->map_out, out, d.out_dtype, d.k, d.ldc, g.wo, g.ho, d.n,
                                 pl->kp.out_pw / pl->kp.out_es, sp.tw, sp.th, pl->kp.out_pw);
        if (st != B200_SUCCESS) return st;
        pl->map_out_ptr = out;
    }
    if (d.res_dtype >= 0 && res != pl->map_res_ptr) {
        int st = encode_nhwc_map(&pl->map_res, res, d.res_dtype, d.k, d.ldc, g.wo, g.ho, d.n,
                                 pl->kp.res_pw / pl->kp.res_es, sp.tw, sp.th, pl->kp.res_pw);
        if (st != B200_SUCCESS) return st;
        pl->map_res_ptr = res;
    } else if (d.res_dtype < 0 && pl->map_res_ptr == nullptr) {
        pl->map_res = pl->map_out;
    }
    return B200_SUCCESS;
}

#ifdef B200_TIMELINE
int slab_debug_timeline(void* out, int max_recs) {
    unsigned n = 0;
    cudaMemcpyFromSymbol(&n, g_tl_n, sizeof(n));
    if (n > TL_CAP) n = TL_CAP;
    if (max_recs < 0) max_recs = 0;
    if (static_cast<int>(n) > max_recs) n = max_recs;
    if (out && n) cudaMemcpyFromSymbol(out, g_tl, n * sizeof(TlRec));
    const unsigned zero = 0;
    cudaMemcpyToSymbol(g_tl_n, &zero, sizeof(zero));
    return static_cast<int>(n);
}
#endif

}  // namespace b200
