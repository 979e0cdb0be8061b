// The conv planner: kernel, tile width, split-K factor, ring depth, shared memory, grid and slab tiling as a function
// of the descriptor, the planner switches and the SM count alone, with no CUDA call (b200_conv_plan_choose). Order:
// the per-tile im2col candidate, then the slab kernel against its estimate, then the persistent walker on the im2col
// candidate; a fused pooling takes the slab kernel or is refused.
#include <stdio.h>
#include <stdlib.h>

#include <new>

#include "conv_common.cuh"

namespace b200 {

// Planner switches, read from the environment on every plan (tuning experiments and tests).
struct PlanKnobs {
    bool splitk = true;   // B200_SABER_SPLITK=0: never split the k loop
    int force_bn = 0;     // B200_SABER_FORCE_BN: tile width (32 | 64 | 128 | 256 up to the widest allowed, else ignored)
    int force_split = 0;  // B200_SABER_FORCE_SPLIT: split-K factor (1 | 2 | 4 | 8 up to the k iterations, else ignored)
    char slab = 0;        // B200_SABER_SLAB: '0' never the slab kernel, '2' whenever it applies
    char persistent = 0;  // B200_SABER_PERSISTENT: '0' never the persistent walker, '2' whenever it applies
    bool verbose = false; // B200_SABER_VERBOSE=1: print every plan
};

// ----------------------------------------------------------------- cost model
// The constants -- per-MMA cost in SM clocks (K = 32 bytes, M = 128), the L2 ingest of one SM, the epilogue and fixed
// clocks of conv_time_estimate -- and the thresholds built on them were measured on the earlier sm_100 version of
// these kernels. They only rank plans of the same layer against each other, and now only for the float kinds, whose
// plans (and k summation order) they keep as they were; int8 plans follow rules measured on the H100 instead (below).
// On the H100, tools/probe/probe_sm90.cu measures a 128 x N wgmma k slice at max(48, N) clocks for s8, f16 and tf32
// alike (profiles/probe_sm90.txt).
// The e4m3 kind moves the int8 kind's bytes through the same 32-byte k slices (same boxes, chunks, swizzles and slab
// tilings) at the data sheet's same dense rate, so it is planned as the int8 kind is: every rule below that names the
// 8-bit kinds gives both the same plan at every shape.
static bool eight_bit(int math) { return math_kind(math)->es == 1; }
constexpr double L2_INGEST_BYTES_PER_CLK = 38.7;
static double mma_clk(int bn) { return bn / 2.0 > 32.0 + bn / 4.0 ? bn / 2.0 : 32.0 + bn / 4.0; }
// widest tile: keeps an fp32 staging (or residual) tile <= 64 KiB
static int max_bn_for(int out_es, int res_es) { return (out_es == 4 || res_es == 4) ? 128 : 256; }
// B200_SABER_FORCE_BN (tuning experiments only): the forced tile width, or 0 when unset or not a width up to max_bn
static int forced_bn(const PlanKnobs& knobs, int max_bn) {
    const int fb = knobs.force_bn;
    return ((fb == 32 || fb == 64 || fb == 128 || fb == 256) && fb <= max_bn) ? fb : 0;
}

// Whole-kernel time estimate (SM clocks) both conv kernels are compared with: a CTA costs its main loop (the slower
// of MMA issue and L2 ingest) + its epilogue + ~6000 clk of fixed latencies (prologue, first TMA round trip,
// accumulator read-out, store); CTAs beyond one per SM run in turns, two co-resident CTAs overlapping each other's
// fixed parts at the price of a shared SM.
static double conv_time_estimate(int ctas, double loop_clk, int bn, int out_es, bool two_per_sm, int sms) {
    const double cta = loop_clk + bn * (out_es == 4 ? 12.0 : 9.0) + 6000.0;
    if (ctas <= sms) return cta;
    const int r = two_per_sm ? 2 : 1;
    const double turns = static_cast<double>((ctas + sms * r - 1) / (sms * r));
    return turns * cta * (r == 2 ? 1.25 : 1.0);
}

static PlanKnobs plan_knobs_from_env() {
    auto env = [](const char* name) { const char* e = getenv(name); return e ? e : ""; };
    PlanKnobs k;
    k.splitk = env("B200_SABER_SPLITK")[0] != '0';
    k.force_bn = atoi(env("B200_SABER_FORCE_BN"));
    k.force_split = atoi(env("B200_SABER_FORCE_SPLIT"));
    k.slab = env("B200_SABER_SLAB")[0];
    k.persistent = env("B200_SABER_PERSISTENT")[0];
    k.verbose = env("B200_SABER_VERBOSE")[0] == '1';
    return k;
}

// Epilogue of a CTA that finishes and stores epi_bn channels: output / residual tiles as TMA panels of up to 128 bytes.
static void set_epilogue_panels(ConvKParams& kp, int epi_bn) {
    kp.epi_bn = epi_bn;
    kp.out_pw = epi_bn * kp.out_es >= 128 ? 128 : epi_bn * kp.out_es;
    kp.out_panels = epi_bn * kp.out_es / kp.out_pw;
    kp.res_pw = kp.res_es ? (epi_bn * kp.res_es >= 128 ? 128 : epi_bn * kp.res_es) : 0;
    kp.res_panels = kp.res_es ? epi_bn * kp.res_es / kp.res_pw : 0;
}

// ----------------------------------------------------------------- slab-staged kernel (conv_slab.cu)
namespace {
struct SlabLayout {
    SlabParams sp;
    int bn, smem_bytes;
    bool two_per_sm;
    double est_clk;
};

// Shared-memory layout of one (tile, BN) candidate; false when it cannot fit.
struct PoolTiling { int pk, ps, pp, ph, pw, PHo, PWo; };   // fused pooling: th x tw is the rectangle a ph x pw pooled tile needs

bool slab_layout(const b200_conv_desc_t& d, const Geometry& g, int th, int tw, int bn, int sms, SlabLayout* L,
                 const PoolTiling* pool = nullptr) {
    const int planes = g.planes;
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
    const int mmas = 2 * planes - 1;   // per k slice: 3xTF32 issues Ahi*Whi, Alo*Whi and Ahi*Wlo
    const double mma = static_cast<double>(g.CC) * RS * sp.mma_per_tap * mmas * mma_clk(bn);
    const double ingest =
        static_cast<double>(g.CC) * (sp.slab_box_bytes + static_cast<double>(planes) * RS * bn * g.chunk) / L2_INGEST_BYTES_PER_CLK;
    double loop = mma > ingest ? mma : ingest;
    if ((sa < 2 && g.CC > 1) || sb < 2) loop = mma + ingest;          // no double buffering: load and MMA serialise
    L->est_clk = conv_time_estimate(ctas, loop, bn, out_es, L->two_per_sm, sms);
    return true;
}

// The slab kernel for this convolution when it applies and its estimate beats the im2col candidate c (a fused pooling
// takes it whenever one of its tilings holds): replaces c and returns true. Returns false to leave c as it is.
bool choose_slab(const b200_conv_desc_t& d, const Geometry& g, const PlanKnobs& knobs, int sms, ConvPlanChoice& c) {
    // B200_SABER_SLAB: 0 never, 2 whenever it applies (tests), default: when its time estimate beats the im2col plan's
    // (a fused pooling has no other kernel to fall back to; a forced split-K is an im2col experiment)
    if (!d.fuse_pool && (knobs.slab == '0' || knobs.force_split > 1)) return false;
    if (d.r * d.s < 2 || d.stride_h != 1 || d.stride_w != 1 || d.dil_h != 1 || d.dil_w != 1) return false;
    if (g.chunk < 32 || d.s > 16 || d.r > 16) return false;
    const int out_es = c.kp.out_es, res_es = c.kp.res_es;

    // ---- candidates: tile width = the row (or an equal part of it), tile height = what fits 128 GEMM rows, every
    // tile width of the kernel; the estimate weighs halo re-reads, weight re-reads per tile, MMA width and waves
    const int kr32 = (d.k + 31) / 32 * 32;
    const int max_bn = max_bn_for(out_es, res_es);
    const int force_bn = forced_bn(knobs, max_bn);
    // int8 without a fused pooling, when 64-wide tiles make half a wave to one wave: 64-wide tiles. In the ResNet-50 b8
    // sweep (profiles/README.md) the 64-wide slab beat 32 and 128 on all four 3x3 layers (res2..res5: 6.9 / 6.6 / 8.5 /
    // 13.2 us), which the estimate below does not see. Other grids keep the estimate (at b1 the 32-wide slab was faster).
    const bool i8 = eight_bit(d.math);
    const int i8_bn = kr32 >= 64 ? 64 : 32;
    SlabLayout best{};
    bool have = false;
    auto consider = [&](const SlabLayout& L) {
        if (!have || L.est_clk < best.est_clk) { best = L; have = true; }
    };
    const int parts[8] = {1, 2, 3, 4, 6, 8, 12, 16};
    const int cands[4] = {32, 64, 128, 256};
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
            for (int ci = 0; ci < 4; ++ci) {
                const int bn = cands[ci];
                if (force_bn ? bn != force_bn : (bn > max_bn || (bn > kr32 && bn != 32))) continue;
                SlabLayout L{};
                if (!slab_layout(d, g, th, tw, bn, sms, &L, &pt)) continue;
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
        for (int ci = 0; ci < 4; ++ci) {
            const int bn = cands[ci];
            const int ctas64 = d.n * tiles_h * ((g.wo + tw - 1) / tw) * ((d.k + i8_bn - 1) / i8_bn);
            const bool i8_rule = i8 && ctas64 >= sms * 15 / 32 && ctas64 <= sms;
            if (force_bn ? bn != force_bn : (bn > max_bn || (bn > kr32 && bn != 32) || (i8_rule && bn != i8_bn))) continue;
            SlabLayout L{};
            if (!slab_layout(d, g, th, tw, bn, sms, &L)) continue;
            consider(L);
        }
    }
    if (!have) return false;
    if (!d.fuse_pool) {
        // the complete im2col plan (bn, grid, stages, smem): A is fetched once per tap; a ring of fewer than three
        // stages cannot overlap loads and MMAs
        const double k_bytes = static_cast<double>(g.KS) * g.chunk;
        const int bn0 = c.bn;
        const int mmas = 2 * g.planes - 1;   // per k slice: 3xTF32 issues Ahi*Whi, Alo*Whi and Ahi*Wlo
        const double mma0 = k_bytes / 32.0 * mmas * mma_clk(bn0);
        const double ingest0 = (BLOCK_M + static_cast<double>(g.planes) * bn0) * k_bytes / L2_INGEST_BYTES_PER_CLK;
        double loop0 = mma0 > ingest0 ? mma0 : ingest0;
        if (c.kp.stages < 3) loop0 = mma0 + ingest0;
        const int split0 = c.kp.split;           // split-K cluster: the k loop is shared, plus the exchange
        if (split0 > 1) loop0 = loop0 / split0 + 2500.0;
        const double est0 = conv_time_estimate(c.ctas, loop0, bn0, out_es, c.smem_bytes <= MAX_SMEM / 2, sms);
        const bool force = knobs.slab == '2';
        // int8 (the b8 regime above): the slab kernel unless the im2col plan splits its k loop. Measured on the H100 (ResNet-50 b8), the slab
        // won every 3x3 layer the im2col plan runs unsplit and lost the one it splits (res5: 13.2 against 10.6 us); the
        // estimate still decides for the float kinds, whose plans (and k summation order) are kept as they were.
        const bool i8_rule = i8 && best.bn == i8_bn && c.ctas <= 2 * sms;
        const bool im2col_wins = i8_rule ? split0 > 1 : est0 <= best.est_clk;
        if (!force && !force_bn && im2col_wins) return false;
    }

    const SlabParams& sp = best.sp;
    const int bn = best.bn;
    c.kernel = B200_CONV_KERNEL_SLAB;
    c.bn = bn;
    c.grid_x = d.n * sp.tiles_h * sp.tiles_w;
    c.grid_y = (d.k + bn - 1) / bn;
    c.ctas = c.grid_x * c.grid_y;
    c.smem_bytes = best.smem_bytes;
    c.sp = sp;
    c.kp.stages = 0;   // the slab kernel's rings are sp.SA and sp.SB
    c.kp.split = 1;
    set_epilogue_panels(c.kp, bn);
    return true;
}

// ----------------------------------------------------------------- persistent walker (conv_persistent.cu)
// Turns the per-tile im2col candidate c into the persistent variant when its grid spans several waves. Keeps BN and the
// epilogue parameters; recomputes the ring depth for one CTA per SM with a dedicated staging tile.
void choose_persistent(const b200_conv_desc_t& d, const Geometry& g, const PlanKnobs& knobs, int sms, ConvPlanChoice& c) {
    if (knobs.persistent == '0') return;
    if (g.planes != 1 || c.kp.split != 1) return;   // (no 3xTF32 walker)
    const int tiles = c.grid_x * c.grid_y;
    const bool force = knobs.persistent == '2';
    // worth it once every SM gets more than the two tiles that co-resident CTAs already overlap ...
    if (!force && tiles <= 2 * sms) return;
    const int bn = c.bn;
    // ... and the tile is not epilogue-dominated: the walker's consumer warps run each tile's epilogue after its main
    // loop (only the producer keeps loading meanwhile), while two co-resident per-tile CTAs overlap one's epilogue with
    // the other's main loop. Epilogue clocks per channel below.
    const double k_bytes = static_cast<double>(g.KS) * g.chunk;
    const double ingest = (BLOCK_M + bn) * k_bytes / L2_INGEST_BYTES_PER_CLK;
    const double mma = k_bytes / 32.0 * mma_clk(bn);
    const double loop = mma > ingest ? mma : ingest;
    const double epi = bn * (c.kp.res_es ? 11.0 : 9.0);
    // With many tiles per SM (>= 6) the per-tile CTAs pay their prologue / barrier setup / drain once per tile, so the
    // walker is taken further into epilogue-bound territory from 6 tiles per SM.
    const double epi_ratio = tiles >= 6 * sms ? 2.5 : 1.5;
    if (!force && epi > epi_ratio * loop) return;
    const int sb = stage_bytes(bn, false);
    const int staging = BLOCK_M * bn * c.kp.out_es;
    const int res_bytes = BLOCK_M * bn * c.kp.res_es;
    const int fixed = staging + res_bytes + persistent_tail_bytes(bn) + 1024;
    int stages = (MAX_SMEM - fixed) / sb;
    if (stages > MAX_STAGES) stages = MAX_STAGES;
    if (stages < 2) return;
    c.kernel = B200_CONV_KERNEL_PERSISTENT;
    c.kp.stages = stages;
    c.smem_bytes = stages * sb + fixed;
    c.ctas = tiles < sms ? tiles : sms;
}
}  // namespace

// ----------------------------------------------------------------- the plan
static ConvPlanChoice choose_conv_plan(const b200_conv_desc_t& desc, const PlanKnobs& knobs, int sms) {
    const b200_conv_desc_t* d = &desc;
    ConvPlanChoice c{};
    auto refuse = [&c](int status) { c.status = status; return c; };
    const MathKind* mk = math_kind(d->math);
    if (!mk) return refuse(B200_UNIMPL_ERROR);
    if (d->fuse_pool < 0 || d->pool_stride < 0 || d->pool_pad < 0) return refuse(B200_INVALID_VALUE);
    // fused pooling lives in the slab kernel's epilogue (a CTA owns a rectangle of the output): stride-1 r x s filters
    if (d->fuse_pool != 0 && (d->res_dtype >= 0 || d->r * d->s < 2 || d->stride_h != 1 || d->stride_w != 1 ||
                              d->dil_h != 1 || d->dil_w != 1 || (d->k * dtype_size(d->out_dtype)) % 16 != 0))
        return refuse(B200_UNIMPL_ERROR);
    const Geometry g = make_geometry(d);
    if (!g.ok) return refuse(B200_INVALID_VALUE);
    // operand / epilogue dtype consistency: the epilogues read and write only the kind's types (epilogue16 /
    // epilogue16_i8 would skip any other one and leave the staging tile or the residual registers unset)
    if (!dtype_in(mk->in_dtypes, d->in_dtype) || !dtype_in(mk->out_dtypes, d->out_dtype) ||
        (d->res_dtype >= 0 && !dtype_in(mk->res_dtypes, d->res_dtype)))
        return refuse(B200_INVALID_VALUE);
    if (d->ldc < d->k) return refuse(B200_INVALID_VALUE);
    const int out_es = dtype_size(d->out_dtype);
    const int res_es = d->res_dtype >= 0 ? dtype_size(d->res_dtype) : 0;
    // the output / residual tiles move by TMA: row pitch must be a 16-byte multiple
    if ((static_cast<int64_t>(d->ldc) * out_es) % 16 != 0) return refuse(B200_INVALID_VALUE);
    if (res_es && (static_cast<int64_t>(d->ldc) * res_es) % 16 != 0) return refuse(B200_INVALID_VALUE);
    // TMA im2col hardware limits (corner and offset field widths for 2 spatial dims)
    const int up_w = d->pad_w - (d->s - 1) * d->dil_w, up_h = d->pad_h - (d->r - 1) * d->dil_h;
    if (d->pad_w > 127 || d->pad_h > 127 || up_w < -128 || up_h < -128 || up_w > 127 || up_h > 127 ||
        (d->s - 1) * d->dil_w > 254 || (d->r - 1) * d->dil_h > 254 || d->stride_w > 8 || d->stride_h > 8)
        return refuse(B200_UNIMPL_ERROR);

    // ---- tile-N heuristic: widest tile that still yields >= ~1 wave of CTAs
    const int tiles_m = static_cast<int>((g.M_total + BLOCK_M - 1) / BLOCK_M);
    const int kr32 = (d->k + 31) / 32 * 32;
    const bool i8 = eight_bit(d->math);
    // split-K threshold: float kinds split from 16 k iterations (their k loops move 2-4x the bytes per MAC), int8 from 24
    const int split_min_iters = i8 ? 24 : 16;
    const int k_iters = (g.KS + STAGE_K_BYTES / g.chunk - 1) / (STAGE_K_BYTES / g.chunk);
    // int8 sub-wave grids whose 64-wide split-2 grid still fills about half of the SMs (ResNet-50 res5 3x3 at b8; at b1
    // the 32-wide split-4 plans of the sm_100 rules measured faster and stay)
    const bool i8_split64 = i8 && kr32 >= 64 && k_iters >= split_min_iters && 2 * tiles_m * ((d->k + 63) / 64) >= sms * 15 / 32;
    int bn = 32;
    bool found = false;
    const int cands[4] = {256, 128, 64, 32};
    auto widest = [&](int max_bn, int wave) {
        for (int i = 0; i < 4 && !found; ++i) {
            if (cands[i] > max_bn) continue;
            if (cands[i] > kr32 && cands[i] != 32) continue;
            const int ctas = tiles_m * ((d->k + cands[i] - 1) / cands[i]);
            if (ctas >= wave) { bn = cands[i]; found = true; }
        }
    };
    widest(max_bn_for(out_es, res_es), sms);
    // int8 grids of up to two CTAs per SM: tiles at most 64 wide, and 64 once it leaves a wave less a few SMs. A 128 x N
    // wgmma k slice costs max(48, N) clocks on the H100, so 128- and 256-wide tiles are MMA-bound where 64-wide ones are
    // not, and 64 over 32 halves the A re-fetch. (ResNet-50 INT8 b8 layer sweep, profiles/README.md: 64 is at or within
    // noise of the best per-tile width on every 1x1 layer with >= 128 CTAs at 64, up to 22% faster than the widths
    // chosen before. Larger grids were not measured per layer and keep the widest-tile rule.)
    if (i8 && found && tiles_m * ((d->k + bn - 1) / bn) <= 2 * sms) {
        found = false;
        widest(64, sms - sms / 32);
    }
    if (!found) {
        // not enough work for a full wave: maximise the CTA count, but keep N >= 64 when free
        bn = 32;
        if (kr32 >= 64 && tiles_m * ((d->k + 63) / 64) == tiles_m * ((d->k + 31) / 32)) bn = 64;
        // int8 k loops long enough to be split over a cluster: the 64-wide tile halves the A traffic of the shared loop
        // (res5 3x3 512, b8: 64-wide split 2 10.6 us against 32-wide split 2 13.3 us)
        if (i8_split64) bn = 64;
        // fp32 operands: a k-iteration is 12 3xTF32 MMAs whose cost barely depends on N below 64, and the long k loops
        // of these layers are split over a cluster anyway: the wider tile halves the MMA count per output (a choice
        // carried over from the sm_100 version, not re-measured on the H100)
        if (mk->kind == KIND_TF32X3 && kr32 >= 64 && static_cast<int64_t>(g.KS) * g.chunk >= 2048)
            bn = 64;
    }
    if (const int fb = forced_bn(knobs, max_bn_for(out_es, res_es))) bn = fb;
    const int grid_y = (d->k + bn - 1) / bn;
    const int ctas = tiles_m * grid_y;

    // ---- pipeline depth: as deep as the k loop needs, within the shared-memory budget. A grid that
    // exceeds one wave keeps two CTAs per SM resident (epilogue of one overlaps the main loop of the
    // other); a sub-wave grid takes the whole SM for latency hiding on its long k loop.
    const int sb = stage_bytes(bn, g.planes == 2);
    // split-K for sub-wave grids with a long k loop (deep 3x3 / wide 1x1 layers on small feature maps):
    // one SM's TMA engine cannot feed such a loop fast enough, so 2 or 4 CTAs (a cluster) share it.
    int split = 1;
    // Splitting pays only for long k loops on grids that stay within one wave: the cluster barriers and the DSMEM
    // exchange cost a fixed time. The thresholds were tuned on the earlier sm_100 version of this kernel; float plans keep
    // them, and with them their k summation order. On the H100 a split of 4 of the 64-wide int8 tiles above lost to a
    // split of 2 on every layer of the ResNet-50 b8 sweep (res4 / res5 3x3: 16.1 / 18.1 us against 9.5 / 10.6 us).
    if (knobs.splitk && k_iters >= split_min_iters && ctas * 2 <= sms) {
        split = 2;
        if (!i8_split64 && k_iters >= 32 && ctas * 4 <= sms) split = 4;
    }
    {   // B200_SABER_FORCE_SPLIT: tuning experiments only
        const int fs = knobs.force_split;
        if ((fs == 1 || fs == 2 || fs == 4 || fs == 8) && k_iters >= fs) split = fs;
    }
    while (split > 1 && (bn / split) % 16) split >>= 1;      // a slice is whole 16-channel groups
    if (bn > 128) split = 1;   // split-K instances exist for the narrow tiles only (the heuristic never splits wide ones)
    // each rank of a split cluster finishes and stores a slice of epi_bn channels (reduce-scatter)
    const int epi_bn = bn / split;
    ConvKParams& kp = c.kp;
    kp.split = split;
    kp.out_es = out_es;
    kp.res_es = res_es;
    set_epilogue_panels(kp, epi_bn);
    const int res_bytes = BLOCK_M * epi_bn * res_es;
    const int fixed = res_bytes + tail_bytes(bn) + 1024;
    const int staging = BLOCK_M * epi_bn * out_es;
    const int part_bytes = (split - 1) * BLOCK_M * epi_bn * 4;   // the other ranks' partial sums of this slice
    const int k_iters_local = (k_iters + split - 1) / split;
    // Every CTA keeps to half of the SM's shared memory so that two CTAs are always co-resident: the next
    // kernel's prologue + weight prefetch (PDL) and the kernels of other streams (the Worker serves several
    // requests at once) overlap this one instead of queueing behind it. Measured on ResNet-50 INT8 b8: one
    // stream 354 -> 348 us, six Worker streams 24.4k -> 40.8k img/s.
    const int fixed_all = fixed + part_bytes;
    const int half_budget = MAX_SMEM / 2 - 2048;
    int budget = half_budget;
    if (ctas * split <= sms) {
        // a sub-wave grid may take the whole SM when half of it cannot hold a useful ring (wide int8 tiles with a
        // long k loop, and every 3xTF32 tile, whose stages are twice as large): 2 stages would serialise TMA and MMA
        const int stages_half = (half_budget - fixed_all) / sb;
        if (stages_half < (k_iters_local < 4 ? k_iters_local : 4)) budget = MAX_SMEM;
    }
    int stages = (budget - fixed_all) / sb;
    if (stages > k_iters_local) stages = k_iters_local;
    if (stages > MAX_STAGES) stages = MAX_STAGES;
    const int min_stages = (staging + sb - 1) / sb;   // the ring doubles as the output staging tile
    if (stages < min_stages) stages = min_stages;
    if (stages < 1) stages = 1;
    if (stages < 2 && k_iters >= 2 && 2 * sb + fixed_all <= MAX_SMEM) stages = 2;  // never serialise load / MMA
    if (stages * sb + fixed_all > MAX_SMEM) return refuse(B200_OUT_OF_MEM);
    kp.stages = stages;
    c.kernel = B200_CONV_KERNEL_TILE;
    c.bn = bn;
    c.grid_x = tiles_m;
    c.grid_y = grid_y;
    c.ctas = ctas * split;
    c.smem_bytes = stages * sb + fixed_all;
    c.tile_stages = stages;

    // ---- stride-1 R x S layers: the slab-staged kernel when it applies and its estimate beats this plan's
    if (!choose_slab(*d, g, knobs, sms, c)) {
        if (d->fuse_pool != 0) return refuse(B200_UNIMPL_ERROR);   // no rectangle tiling holds this window
        choose_persistent(*d, g, knobs, sms, c);
    }
    c.status = B200_SUCCESS;
    return c;
}

// B200_SABER_VERBOSE=1: one line per plan (the persistent walker also prints the im2col candidate it replaces)
static void print_conv_plan(const b200_conv_desc_t& d, const ConvPlanChoice& c) {
    const unsigned gx = static_cast<unsigned>(c.grid_x), gy = static_cast<unsigned>(c.grid_y);
    if (c.kernel == B200_CONV_KERNEL_SLAB) {
        fprintf(stderr, "[b200_saber] plan slab  n%d %dx%d c%d k%d %dx%d | tile %dx%d (pitch %d) BN %d grid %ux%u slabs %d groups %d smem %d\n",
                d.n, d.h, d.w, d.c, d.k, d.r, d.s, c.sp.th, c.sp.tw, c.sp.PW, c.bn, gx, gy, c.sp.SA, c.sp.SB, c.smem_bytes);
        return;
    }
    if (c.kernel == B200_CONV_KERNEL_PERSISTENT)
        fprintf(stderr, "[b200_saber] plan persistent: %u x %u tiles on %d CTAs, stages %d smem %d\n", gx, gy, c.ctas,
                c.kp.stages, c.smem_bytes);
    fprintf(stderr, "[b200_saber] plan im2col n%d %dx%d c%d k%d %dx%d s%d | BN %d split %d grid %ux%u stages %d smem %d\n",
            d.n, d.h, d.w, d.c, d.k, d.r, d.s, d.stride_h, c.bn, c.kp.split, gx, gy, c.tile_stages, c.smem_bytes);
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200_conv_plan_create(const b200_conv_desc_t* d, const void* packed_weights_dev, const float* bias_dev,
                          const float* scale_dev, b200_conv_plan_t** plan_out) {
    if (!d || !packed_weights_dev || !plan_out) return B200_INVALID_VALUE;
    if (!device_is_sm90()) return B200_WRONG_DEVICE;
    if (!tensor_maps_available()) return B200_NOT_INITIALIZED;
    const PlanKnobs knobs = plan_knobs_from_env();
    const ConvPlanChoice c = choose_conv_plan(*d, knobs, sm_count());
    if (c.status != B200_SUCCESS) return c.status;

    b200_conv_plan* pl = new (std::nothrow) b200_conv_plan();
    if (!pl) return B200_MEM_ALLOC_FAILED;
    const Geometry g = make_geometry(d);
    pl->desc = *d;
    pl->g = g;
    pl->choice = c;
    pl->weights = packed_weights_dev;   // (value-initialised: no map is bound yet)
    const MathKind& mk = *math_kind(d->math);
    pl->idesc = conv_idesc(mk, d->in_dtype, c.bn);
    ConvKParams& kp = pl->kp;
    kp = c.kp;
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

    pl->launch = c.kernel == B200_CONV_KERNEL_SLAB         ? slab_launch(mk.kind, c.bn)
                 : c.kernel == B200_CONV_KERNEL_PERSISTENT ? persistent_launch(mk.kind, c.bn)
                                                           : tile_launch(mk.kind, c.bn, c.kp.split > 1);
    if (!pl->launch) { delete pl; return B200_UNIMPL_ERROR; }
    // the weight box follows the tile width of the kernel that runs
    if (encode_weights_map(pl, c.bn) != B200_SUCCESS) { delete pl; return B200_INVALID_VALUE; }
    if (knobs.verbose) print_conv_plan(*d, c);
    *plan_out = pl;
    return B200_SUCCESS;
}

int b200_conv_plan_choose(const b200_conv_desc_t* d, int32_t sm_count, b200_conv_plan_choice_t* out) {
    if (!d || !out || sm_count <= 0) return B200_INVALID_VALUE;
    const ConvPlanChoice c = choose_conv_plan(*d, plan_knobs_from_env(), sm_count);
    *out = b200_conv_plan_choice_t{};
    if (c.status != B200_SUCCESS) return c.status;
    const bool slab = c.kernel == B200_CONV_KERNEL_SLAB;
    *out = {c.kernel, c.bn, c.kp.split, c.kp.stages, c.smem_bytes, c.grid_x, c.grid_y, make_geometry(d).KS, c.ctas,
            slab ? c.sp.th : 0, slab ? c.sp.tw : 0};
    return B200_SUCCESS;
}

}  // extern "C"
