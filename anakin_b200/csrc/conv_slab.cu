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
#include "conv_common.cuh"

namespace b200 {

// Filter-row shape a main loop is compiled for: S taps of Q 32-byte k slices each (0: read from the plan at run time).
template <int S_, int Q_>
struct RowShape {
    static constexpr int S = S_, Q = Q_;
};

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

    const int warp_idx = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

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
        // The main loop, once per A signedness and row shape. A filter row is S taps x mma_per_tap k slices; with both
        // fixed at compile time (RowShape<S, Q>) the row's MMAs are one straight run, and ptxas issues them back to back.
        // RowShape<0, 0> reads both from the plan and loops over them: 3xTF32, and 5x5 / 7x7 filters or 32-byte chunks,
        // which no zoo net's slab plan uses (tests/test_cpu_conv_sass.py checks the recorded plans).
        auto main_loop = [&](auto sg, auto shape) {
            constexpr int FS = decltype(shape)::S, FQ = decltype(shape)::Q;
            auto mma = [&](uint32_t a_lo, uint32_t b_lo) {
#pragma unroll
                for (int nb = 0; nb < NB; ++nb)
                    wgmma<MK, NI>(acc[nb], desc64(((a_lo) & 0x3FFFu) | lbo, hi), desc64(((b_lo + nb * nb16) & 0x3FFFu) | lbo, hi),
                                  sg, 1u);
            };
            // k slice q of the tap whose descriptors are given: the 32-byte k slices of one chunk differ by 2 (x 16 B)
            auto slice = [&](uint32_t a_tap, uint32_t b_tile, uint32_t q) {
                mma(a_tap + q, b_tile + q);
                if (X3) {
                    mma(a_tap + slab16 + q, b_tile + q);
                    mma(a_tap + q, b_tile + plane16 + q);
                }
            };
#pragma unroll 1
            for (int cc = 0; cc < p.CC; ++cc) {
                if (prev_a == a_slot) { wgmma_wait<0>(); release_prev(); }
                mbar_wait(&full_a[a_slot], a_phase);
                if (X3)   // split the landed fp32 slab: high plane in place, low plane behind it
                    split_tf32x3(reinterpret_cast<uint4*>(slab_ring + a_slot * PL * sp.slab_bytes),
                                 reinterpret_cast<uint4*>(slab_ring + a_slot * PL * sp.slab_bytes + sp.slab_bytes), sp.slab_box_bytes >> 4,
                                 etid);
                uint32_t a_row = slab_d0 + a_slot * slot_a16;      // descriptor of tap (r, 0)
#pragma unroll 1
                for (int r = 0; r < p.R; ++r) {
                    if (prev_b == b_slot) { wgmma_wait<0>(); release_prev(); }
                    mbar_wait(&full_b[b_slot], b_phase);
                    const uint32_t b_row = bring_d0 + b_slot * group16;
                    wgmma_fence();
                    if constexpr (FS > 0) {
#pragma unroll
                        for (int s2 = 0; s2 < FS; ++s2)
#pragma unroll
                            for (uint32_t q = 0; q < 2u * FQ; q += 2) slice(a_row + s2 * row16, b_row + s2 * btile16, q);
                    } else {
                        uint32_t a_tap = a_row, b_tile = b_row;
#pragma unroll 1
                        for (int s2 = 0; s2 < p.S; ++s2) {
#pragma unroll 1
                            for (uint32_t q = 0; q < 2u * sp.mma_per_tap; q += 2) slice(a_tap, b_tile, q);
                            a_tap += row16;
                            b_tile += btile16;
                        }
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
            wgmma_wait<0>();   // (inside: no MMA may be in flight where the copies of the loop join)
        };
        with_a_sign<MK>(idesc_a_signed(idesc), [&](auto sg) {
            if constexpr (!X3) {   // (3xTF32 issues three MMAs per k slice: its rows unrolled would not fit the registers)
                if (p.S == 3 && sp.mma_per_tap == 2) return main_loop(sg, RowShape<3, 2>{});   // 64-byte chunks
                if (p.S == 3 && sp.mma_per_tap == 4) return main_loop(sg, RowShape<3, 4>{});   // 128-byte chunks
            }
            main_loop(sg, RowShape<0, 0>{});
        });
#pragma unroll
        for (int nb = 0; nb < NB; ++nb) wgmma_fence_acc(acc[nb]);
        // every MMA of both warpgroups retired: both operand rings are free for the staging tile
        asm volatile("bar.sync 1, %0;" ::"n"(EPI_THREADS) : "memory");
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
                        acc = max16<KIND>(acc, v, p.out_dtype);
                    }
                }
                const size_t o = ((static_cast<size_t>(n_img) * sp.PHo + gi) * sp.PWo + gj) * sp.out_ld_bytes +
                                 static_cast<size_t>(n0) * es + c16 * 16;
                *reinterpret_cast<uint4*>(outp + o) = acc;
            }
        } else if (etid == 0) {
            const int cols_per_panel = p.out_pw / p.out_es;
            for (int jp = 0; jp < p.out_panels; ++jp) {
                if (n0 + jp * cols_per_panel >= p.K) break;
                tma_store_4d(&map_out, smem_u32(out_tile) + jp * BLOCK_M * p.out_pw, n0 + jp * cols_per_panel, q0, p0,
                             n_img);
            }
            tma_store_commit();
            tma_store_wait_read();
        }
    }

    __syncthreads();
}

// ----------------------------------------------------------------- host side
template <int KIND, int BN>
static int launch_slab(b200_conv_plan* pl, void* stream) {
    constexpr auto kern = conv_slab_kernel<KIND, BN>;
    opt_in_smem<kern>(MAX_SMEM);
    const ConvPlanChoice& c = pl->choice;
    return launch("conv (slab)", Pdl::On, kern, dim3(c.grid_x, c.grid_y), dim3(NUM_THREADS), c.smem_bytes, stream, dim3(1),
                  pl->map_a, pl->map_b, pl->map_out, pl->map_res, pl->kp, c.sp, pl->idesc);
}

ConvLaunch slab_launch(int kind, int bn) {
    return bind_kind_bn<32, 64, 128, 256>(kind, bn, [](auto K, auto N) -> ConvLaunch { return launch_slab<K, N>; });
}

// (re)encode the activation / output / residual maps of a slab plan for the buffers of this run
int slab_bind_maps(b200_conv_plan* pl, const void* in, const void* res, void* out) {
    const b200_conv_desc_t& d = pl->desc;
    const Geometry& g = pl->g;
    const SlabParams& sp = pl->choice.sp;
    if (in != pl->map_a_ptr) {
        int st = encode_nhwc_map(&pl->map_a, in, math_kind(d.math)->operand_dtype, d.c, d.c, d.w, d.h, d.n, g.chunk_el, sp.PW,
                                 sp.th + d.r - 1, g.chunk);
        if (st != B200_SUCCESS) return st;
        pl->map_a_ptr = in;
    }
    if (sp.pool) {
        pl->choice.sp.out_ptr = out;       // the pooled pixels are written with plain 16-byte stores
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

}  // namespace b200
