// ConvEngine: host-side preparation of one fused convolution for the C-ABI wgmma plan.
// Replaces, for target NV, the host halves of the reference's
//   SaberConv2D<NV,*>::{init,create,dispatch,trans_weights}  saber/funcs/impl/cuda/saber_conv.cpp:17-585
//   SaberConvEltwise / SaberConv2DPooling / SaberFc           saber_conv_eltwise.cpp, saber_conv_pooling.cpp, saber_fc.cu
// INT8 numerics follow the x86 Saber path (the designated oracle, SURVEY.md section 8c):
//   weights   per-output-channel s_w = max|w|/127, truncating cast   x86_utils.h:293-323
//   scales    kernel/jit_avx512_core_x8s8s32x_conv.cpp:226-255 (scale), :55-62 (bias), :174-192 (sum)
#include "saber_funcs.h"

#include <cuda_fp16.h>

#include <algorithm>
#include <map>
#include <mutex>

namespace anakin {
namespace saber {

// ---------------------------------------------------------------------------------------------------------
// WeightArena: one packed device image per (device, host weight block, packing signature), shared by every
// ConvEngine that asks for it -- the per-thread Nets of a Worker all point at the same device weights, as the
// reference's Nets share the PBlocks of the process-wide GraphGlobalMem (framework/graph/graph_global_mem.h:78-250,
// framework/core/net/worker.cpp:10-53). Entries are reference counted and freed with their last user.
struct DevWeights {
    DeviceBuffer w, bias, scale;   // w: wgmma-packed image, or the plain [n][k] image of a weight-streaming fc
    int device = 0;
};
namespace {
std::mutex g_arena_mu;
std::map<std::string, std::weak_ptr<DevWeights>> g_arena;
std::vector<std::weak_ptr<DevWeights>> g_arena_order;   // creation order: identical on every replica of one graph
bool g_arena_receive = false;                            // allocate images without building them (see below)
size_t g_arena_hits = 0, g_arena_misses = 0;
constexpr size_t kFlatAlign = 256;
size_t flat_pad(size_t n) { return (n + kFlatAlign - 1) / kFlatAlign * kFlatAlign; }

template <typename T>
void key_add(std::string& k, const T& v) { k.append(reinterpret_cast<const char*>(&v), sizeof(T)); }
}  // namespace

size_t weight_arena_stats(size_t* entries, size_t* hits, size_t* misses) {
    std::lock_guard<std::mutex> lk(g_arena_mu);
    size_t bytes = 0, n = 0;
    for (auto it = g_arena.begin(); it != g_arena.end();) {
        if (auto p = it->second.lock()) { bytes += p->w.bytes + p->bias.bytes + p->scale.bytes; ++n; ++it; }
        else it = g_arena.erase(it);
    }
    g_arena_order.erase(std::remove_if(g_arena_order.begin(), g_arena_order.end(),
                                       [](const std::weak_ptr<DevWeights>& w) { return w.expired(); }), g_arena_order.end());
    if (entries) *entries = n;
    if (hits) *hits = g_arena_hits;
    if (misses) *misses = g_arena_misses;
    return bytes;
}

// ---------------------------------------------------------------------------------------------------------
// Replicas on other GPUs (one process per GPU) need not fold, quantise and pack the weights again: the rank that built
// them exports every image of its arena, in creation order, into ONE contiguous device buffer; that buffer travels by a
// single NCCL broadcast over NVLink (bench.py / anakin_b200/dist.py), and the other ranks -- which built their Nets in
// "receive" mode: same plans, same buffer sizes, no host-side packing -- import it. The reference has nothing of the
// kind (its Worker replicates on one device, worker.cpp:10-53); SURVEY.md section 8e asks for NCCL-broadcast weights.
void weight_arena_set_receive(bool on) {
    std::lock_guard<std::mutex> lk(g_arena_mu);
    g_arena_receive = on;
}
static std::vector<std::shared_ptr<DevWeights>> arena_entries_of(int device) {
    std::vector<std::shared_ptr<DevWeights>> v;
    for (auto& w : g_arena_order)
        if (auto p = w.lock()) if (p->device == device) v.push_back(p);
    return v;
}
size_t weight_arena_flat_bytes(int device) {
    std::lock_guard<std::mutex> lk(g_arena_mu);
    size_t n = 0;
    for (auto& p : arena_entries_of(device)) n += flat_pad(p->w.bytes) + flat_pad(p->bias.bytes) + flat_pad(p->scale.bytes);
    return n;
}
static SaberStatus arena_copy(int device, void* flat, size_t cap, bool to_flat) {
    std::lock_guard<std::mutex> lk(g_arena_mu);
    size_t off = 0;
    for (auto& p : arena_entries_of(device)) {
        DeviceBuffer* bufs[3] = {&p->w, &p->bias, &p->scale};
        for (DeviceBuffer* b : bufs) {
            if (b->bytes == 0) continue;
            if (off + b->bytes > cap) return SaberInvalidValue;
            uint8_t* f = static_cast<uint8_t*>(flat) + off;
            if (cudaMemcpy(to_flat ? static_cast<void*>(f) : b->ptr, to_flat ? b->ptr : static_cast<void*>(f), b->bytes,
                           cudaMemcpyDeviceToDevice) != cudaSuccess)
                return SaberUnKownError;
            off += flat_pad(b->bytes);
        }
    }
    return SaberSuccess;
}
SaberStatus weight_arena_export(int device, void* flat_dev, size_t cap) { return arena_copy(device, flat_dev, cap, true); }
SaberStatus weight_arena_import(int device, const void* flat_dev, size_t bytes) {
    return arena_copy(device, const_cast<void*>(flat_dev), bytes, false);
}

struct ConvEngine::Impl {
    Spec spec;
    bool ready = false;
    // change detection
    Shape in_shape, out_shape;
    DataType in_dtype = AK_INVALID, out_dtype = AK_INVALID, res_dtype = AK_INVALID;
    std::vector<float> in_scale, out_scale;
    float res_scale = 0.f;
    const void* weights_id = nullptr;

    b200_conv_desc_t desc;
    b200_conv_plan_t* plan = nullptr;
    std::shared_ptr<DevWeights> dw;   // packed weights / bias / scale tables, shared through the WeightArena
    bool need_in_transform = false;
    bool stem = false;       // input transform = stem pack (R x S conv over RGB -> R x 1 conv over X2)
    int stem_taps = 0;
    bool stem_fused = false; // graph-input conv (+ max pool) in one launch straight from the fp32 NCHW tensor (conv_stem.cu)
    bool stem_pool_fused = false;
    bool pool_fused = false;  // NHWC conv whose plan runs the following MAX pooling in its epilogue (fuse_pool)
    b200_stem_desc_t stem_desc;
    Tensor<NV> in_scratch;
    float in_inv_scale = 1.f;
    bool depthwise = false;
    bool fc_stream = false;           // inner product with few rows: b200_fc_stream_run on the plain weight image
    b200_fc_stream_desc_t fc_desc;
    Tensor<NV> conv_out_scratch;
    b200_pool_desc_t pool_desc;

    ~Impl() {
        if (plan) b200_conv_plan_destroy(plan);
    }
};

ConvEngine::ConvEngine() : _p(new Impl()) {}
const void* ConvEngine::weight_device_ptr() const { return _p->dw ? _p->dw->w.ptr : nullptr; }
bool ConvEngine::fc_stream_info(b200_fc_stream_desc_t* d, const void** w, const float** bias, const float** scale) const {
    if (!_p->ready || !_p->fc_stream || _p->need_in_transform) return false;
    *d = _p->fc_desc;
    *w = _p->dw->w.ptr;
    *bias = static_cast<const float*>(_p->dw->bias.ptr);
    *scale = _p->spec.op_dtype == AK_INT8 ? static_cast<const float*>(_p->dw->scale.ptr) : nullptr;
    return true;
}
ConvEngine::~ConvEngine() { delete _p; }

b200_pool_desc_t make_pool_desc(const Tensor<NV>& in, const PoolingParam<NV>& p) {
    b200_pool_desc_t d;
    memset(&d, 0, sizeof(d));
    d.dtype = in.get_dtype();
    d.type = p.pooling_type;
    d.n = in.num(); d.h = in.height(); d.w = in.width(); d.c = in.channel_stored();
    d.window_h = p.window_h; d.window_w = p.window_w;
    d.pad_h = p.pad_h; d.pad_w = p.pad_w;
    d.stride_h = p.stride_h; d.stride_w = p.stride_w;
    d.global_pooling = p.global_pooling ? 1 : 0;
    d.floor_as_conv = p.cmp_out_shape_floor_as_conv ? 1 : 0;
    return d;
}

static SaberStatus upload(DeviceBuffer& buf, const void* src, size_t bytes) {
    if (buf.re_alloc(bytes, false) != SaberSuccess) return SaberOutOfMem;
    if (bytes && cudaMemcpy(buf.ptr, src, bytes, cudaMemcpyHostToDevice) != cudaSuccess) return SaberUnKownError;
    return SaberSuccess;
}

SaberStatus ConvEngine::prepare(const Spec& spec, const Tensor<NV>& in, const Tensor<NV>* residual,
                                Tensor<NV>& out, Context<NV>& ctx) {
    Impl& P = *_p;
    const float res_scale = spec.residual_scale;
    const DataType res_dt = residual ? residual->get_dtype() : AK_INVALID;
    if (P.ready && P.in_shape == in.valid_shape() && P.out_shape == out.valid_shape() &&
        P.in_dtype == in.get_dtype() && P.out_dtype == out.get_dtype() && P.res_dtype == res_dt &&
        P.in_scale == in.get_scale() && P.out_scale == out.get_scale() && P.res_scale == res_scale &&
        P.weights_id == spec.weights->data() && P.spec.relu == spec.relu && P.spec.neg_slope == spec.neg_slope)
        return SaberSuccess;
    P.ready = false;
    P.spec = spec;
    if (P.plan) { b200_conv_plan_destroy(P.plan); P.plan = nullptr; }

    const DataType op = spec.op_dtype;
    // FP32 runs as error-compensated 3xTF32 (fp32-grade accuracy: the reference pins FP32 results at
    // 1e-3 against exact-fp32 oracles); B200_SABER_FP32_MATH=tf32 selects the single-pass kind.
    static const bool fp32_single_pass = [] {
        const char* e = getenv("B200_SABER_FP32_MATH");
        return e && strcmp(e, "tf32") == 0;
    }();
    const int math = op == AK_INT8 ? B200_MATH_I8
                                   : (op == AK_HALF ? B200_MATH_F16
                                                    : (fp32_single_pass ? B200_MATH_TF32 : B200_MATH_TF32X3));

    // ---- 1. the tensor the conv kernel reads (NHWC in the op's operand type)
    const Tensor<NV>* cin = &in;
    P.need_in_transform = false;
    P.stem = false;
    if (in.get_layout() == Layout_NCHW && !(in.height() == 1 && in.width() == 1 && in.get_dtype() != AK_FLOAT)) {
        if (in.get_dtype() != AK_FLOAT) return SaberUnImplError;
        // graph-input case: fp32 NCHW -> NHWC operand type (the reference quantises inside conv too:
        // saber_conv.cpp:341-381 conv_calibrate_fp32_int8_c4 / x86_utils.h:325-347)
        DataType sdt = op == AK_INT8 ? AK_INT8 : (op == AK_HALF ? AK_HALF : AK_FLOAT);
        Shape s = in.valid_shape();
        s.set_layout(Layout_NHWC);
        // RGB stem: pack S taps x 4 channels per output column (see b200_stem_pack)
        static const bool stem_enabled = [] { const char* e = getenv("B200_SABER_STEM_PACK"); return !(e && e[0] == '0'); }();
        P.stem = stem_enabled && !spec.is_fc && spec.group == 1 && in.channel() <= 4 && spec.s > 1 && spec.s <= 8 &&
                 spec.dil_w == 1 && spec.dil_h == 1;
        // ... and when the output is a plain 16-byte-multiple NHWC pixel, the whole layer (quantise, conv, epilogue and a
        // following MAX pooling) is one launch that reads the fp32 NCHW tensor itself (b200_stem_conv_run)
        static const bool stem_fused_enabled = [] { const char* e = getenv("B200_SABER_STEM_FUSED"); return !(e && e[0] == '0'); }();
        P.stem_fused = false;
        if (P.stem && stem_fused_enabled && !residual) {
            b200_stem_desc_t& sd = P.stem_desc;
            memset(&sd, 0, sizeof(sd));
            sd.math = math;
            sd.n = in.num(); sd.c = in.channel(); sd.h = in.height(); sd.w = in.width();
            sd.k = spec.k;
            sd.r = spec.r; sd.s = spec.s; sd.stride_h = spec.stride_h; sd.stride_w = spec.stride_w;
            sd.pad_h = spec.pad_h; sd.pad_w = spec.pad_w;
            sd.relu = spec.relu ? 1 : 0; sd.neg_slope = spec.neg_slope;
            sd.in_inv_scale = 1.f;
            if (op == AK_INT8) {
                if (in.get_scale().empty()) return SaberInvalidValue;
                sd.in_inv_scale = 1.f / in.get_scale()[0];
            }
            sd.out_dtype = out.get_dtype();
            sd.ldc = out.channel_stored();
            P.stem_pool_fused = false;
            if (spec.has_pool && spec.pool.pooling_type == Pooling_max && !spec.pool.global_pooling) {
                sd.fuse_pool = 1; sd.pool_type = B200_POOL_MAX;
                sd.pool_window_h = spec.pool.window_h; sd.pool_window_w = spec.pool.window_w;
                sd.pool_pad_h = spec.pool.pad_h; sd.pool_pad_w = spec.pool.pad_w;
                sd.pool_stride_h = spec.pool.stride_h; sd.pool_stride_w = spec.pool.stride_w;
                sd.pool_floor_as_conv = spec.pool.cmp_out_shape_floor_as_conv ? 1 : 0;
                P.stem_pool_fused = true;
            }
            int32_t oh = 0, ow = 0;
            int st = b200_stem_conv_out_hw(&sd, &oh, &ow);
            if (st != B200_SUCCESS && P.stem_pool_fused) {     // this pooling does not fuse: conv here, pooling after it
                sd.fuse_pool = 0;
                P.stem_pool_fused = false;
                st = b200_stem_conv_out_hw(&sd, &oh, &ow);
            }
            const bool direct = !spec.has_pool || P.stem_pool_fused;
            P.stem_fused = st == B200_SUCCESS && (!direct || (oh == out.height() && ow == out.width())) &&
                           (out.get_layout() == Layout_NHWC || (out.height() == 1 && out.width() == 1));
        }
        if (P.stem_fused) {
            P.in_inv_scale = P.stem_desc.in_inv_scale;
            s = Shape({1, 4, 1, 1}, Layout_NHWC);        // no packed tensor exists; the dtype bookkeeping below stays
        } else if (P.stem) {
            P.stem_taps = spec.s <= 4 ? 4 : 8;
            const int wo = conv_out_size(in.width(), spec.pad_w, 1, spec.s, spec.stride_w);
            s = Shape({in.num(), P.stem_taps * 4, in.height() + 2 * spec.pad_h, wo}, Layout_NHWC);
        }
        if (P.in_scratch.re_alloc(s, sdt) != SaberSuccess) return SaberOutOfMem;
        CUDA_CHECK(cudaMemsetAsync(P.in_scratch.mutable_data(), 0, P.in_scratch.storage_bytes(), ctx.get_compute_stream()));
        if (P.stem_fused) {
            if (op == AK_INT8) P.in_scratch.set_scale(in.get_scale());
        } else if (op == AK_INT8) {
            if (in.get_scale().empty()) return SaberInvalidValue;
            P.in_inv_scale = 1.f / in.get_scale()[0];
            P.in_scratch.set_scale(in.get_scale());
        } else {
            P.in_inv_scale = 1.f;
        }
        P.need_in_transform = true;
        cin = &P.in_scratch;
    }
    const DataType cin_dt = cin->get_dtype();
    if (op == AK_INT8 && !(cin_dt == AK_INT8 || cin_dt == AK_UINT8)) return SaberUnImplError;
    if (op == AK_HALF && cin_dt != AK_HALF) return SaberUnImplError;
    if (op == AK_FLOAT && cin_dt != AK_FLOAT) return SaberUnImplError;
    if (out.get_layout() != Layout_NHWC && !(out.height() == 1 && out.width() == 1)) return SaberInvalidValue;

    // ---- 2. geometry
    b200_conv_desc_t& d = P.desc;
    memset(&d, 0, sizeof(d));
    d.math = math;
    d.in_dtype = cin_dt;
    d.res_dtype = residual ? residual->get_dtype() : -1;
    d.relu = spec.relu ? 1 : 0;
    d.neg_slope = spec.neg_slope;
    d.sum_scale = 1.f;
    const int cs = cin->channel_stored();
    int c_real;                 // real input channels per filter tap as the weights see them
    std::vector<int> col_map;   // fc: weight column (NCHW flatten) for every stored K position, -1 = pad
    if (spec.is_fc) {
        const int H = cin->height(), W = cin->width(), C = cin->channel();
        d.n = cin->num(); d.h = 1; d.w = 1; d.c = H * W * cs;
        d.r = d.s = 1; d.stride_h = d.stride_w = 1; d.dil_h = d.dil_w = 1;
        c_real = d.c;
        if (spec.c_per_group != C * H * W) return SaberInvalidValue;
        col_map.assign(d.c, -1);
        for (int y = 0; y < H; ++y)
            for (int x = 0; x < W; ++x)
                for (int c = 0; c < C; ++c) col_map[(y * W + x) * cs + c] = (c * H + y) * W + x;
    } else if (P.need_in_transform && P.stem_fused) {
        // bookkeeping in the X2 view (8 taps x 4 channels per output column): the weight image is the same
        d.n = in.num(); d.h = in.height() + 2 * spec.pad_h;
        d.w = conv_out_size(in.width(), spec.pad_w, 1, spec.s, spec.stride_w);
        d.c = 32;
        d.r = spec.r; d.s = 1;
        d.pad_h = 0; d.pad_w = 0;
        d.stride_h = spec.stride_h; d.stride_w = 1;
        d.dil_h = 1; d.dil_w = 1;
        c_real = 32;
    } else if (P.need_in_transform && P.stem) {
        d.n = cin->num(); d.h = cin->height(); d.w = cin->width(); d.c = cs;   // X2: c = taps*4
        d.r = spec.r; d.s = 1;
        d.pad_h = 0; d.pad_w = 0;
        d.stride_h = spec.stride_h; d.stride_w = 1;
        d.dil_h = 1; d.dil_w = 1;
        c_real = cs;
    } else {
        d.n = cin->num(); d.h = cin->height(); d.w = cin->width(); d.c = cs;
        d.r = spec.r; d.s = spec.s;
        d.pad_h = spec.pad_h; d.pad_w = spec.pad_w;
        d.stride_h = spec.stride_h; d.stride_w = spec.stride_w;
        d.dil_h = spec.dil_h; d.dil_w = spec.dil_w;
        c_real = spec.c_per_group;
    }
    const bool stem = P.need_in_transform && P.stem;
    d.k = spec.k;
    P.depthwise = !spec.is_fc && spec.group > 1 && spec.group == cin->channel() && spec.c_per_group == 1 &&
                  spec.k == spec.group;
    if (spec.group != 1 && !P.depthwise) return SaberUnImplError;
    if (!spec.is_fc && !P.depthwise && !stem && c_real != cin->channel()) return SaberInvalidValue;

    // ---- 3. where the conv writes
    Tensor<NV>* cout = &out;
    // conv + MAX pooling in one launch (the conv plan's fuse_pool) when the window is square; the plan decides
    static const bool pool_fusion_enabled = [] { const char* e = getenv("B200_SABER_FUSE_POOL"); return !(e && e[0] == '0'); }();
    P.pool_fused = pool_fusion_enabled && spec.has_pool && !P.need_in_transform && !spec.is_fc && !residual &&
                   spec.group == 1 && spec.pool.pooling_type == Pooling_max && !spec.pool.global_pooling &&
                   spec.pool.window_h == spec.pool.window_w && spec.pool.stride_h == spec.pool.stride_w &&
                   spec.pool.pad_h == spec.pool.pad_w && out.get_layout() == Layout_NHWC;
    auto setup_pool_scratch = [&]() -> SaberStatus {
        Shape s({d.n, spec.k, conv_out_size(d.h, d.pad_h, d.dil_h, d.r, d.stride_h),
                 conv_out_size(d.w, d.pad_w, d.dil_w, d.s, d.stride_w)}, Layout_NHWC);
        if (P.conv_out_scratch.re_alloc(s, out.get_dtype()) != SaberSuccess) return SaberOutOfMem;
        CUDA_CHECK(cudaMemsetAsync(P.conv_out_scratch.mutable_data(), 0, P.conv_out_scratch.storage_bytes(), ctx.get_compute_stream()));
        P.conv_out_scratch.set_scale(out.get_scale());
        P.pool_desc = make_pool_desc(P.conv_out_scratch, spec.pool);
        return SaberSuccess;
    };
    if (P.pool_fused) {
        d.fuse_pool = spec.pool.window_h;
        d.pool_stride = spec.pool.stride_h;
        d.pool_pad = spec.pool.pad_h;
        d.pool_floor_as_conv = spec.pool.cmp_out_shape_floor_as_conv ? 1 : 0;
    } else if (spec.has_pool && !(P.stem_fused && P.stem_pool_fused)) {
        Shape s({d.n, spec.k, conv_out_size(d.h, d.pad_h, d.dil_h, d.r, d.stride_h),
                 conv_out_size(d.w, d.pad_w, d.dil_w, d.s, d.stride_w)}, Layout_NHWC);
        if (P.conv_out_scratch.re_alloc(s, out.get_dtype()) != SaberSuccess) return SaberOutOfMem;
        CUDA_CHECK(cudaMemsetAsync(P.conv_out_scratch.mutable_data(), 0, P.conv_out_scratch.storage_bytes(), ctx.get_compute_stream()));
        P.conv_out_scratch.set_scale(out.get_scale());
        cout = &P.conv_out_scratch;
        P.pool_desc = make_pool_desc(P.conv_out_scratch, spec.pool);
    }
    d.out_dtype = cout->get_dtype();
    d.ldc = cout->channel_stored();
    if (residual && residual->channel_stored() != d.ldc) return SaberInvalidValue;

    // ---- 4. weights, bias, scales: looked up in / built into the WeightArena
    const bool wq8 = spec.weights->get_dtype() == AK_INT8;   // model file carries int8 codes + per-channel scales
    const float* w = wq8 ? nullptr : static_cast<const float*>(spec.weights->data());
    const int8_t* wq = wq8 ? static_cast<const int8_t*>(spec.weights->data()) : nullptr;
    const std::vector<float>& wq_scale = spec.weights->get_scale();
    if (wq8 && wq_scale.empty()) return SaberInvalidValue;
    auto wq_scale_of = [&](int oc) { return wq_scale[static_cast<size_t>(oc) < wq_scale.size() ? oc : wq_scale.size() - 1]; };
    const size_t per_k = static_cast<size_t>(spec.is_fc ? spec.c_per_group : spec.c_per_group * spec.r * spec.s);
    const bool has_bias = spec.bias && spec.bias->valid_size() >= spec.k && spec.bias->data();
    const float* b = has_bias ? static_cast<const float*>(spec.bias->data()) : nullptr;
    const DataType odt = cout->get_dtype();
    float in_scale = 1.f, out_scale = 1.f;
    if (op == AK_INT8) {
        if (cin->get_scale().empty()) return SaberInvalidValue;
        in_scale = cin->get_scale()[0];
        if (odt != AK_FLOAT) {
            if (cout->get_scale().empty()) return SaberInvalidValue;
            out_scale = cout->get_scale()[0];
        }
    }
    if (P.stem_fused) {
        // the fused pooling may run on the raw accumulators when the epilogue is non-decreasing in them
        bool pos = spec.neg_slope >= 0.f;
        if (op == AK_INT8) {
            pos = pos && in_scale > 0.f && out_scale > 0.f;
            for (float sc : wq_scale) pos = pos && sc > 0.f;
        }
        P.stem_desc.monotone_epilogue = pos ? 1 : 0;
    }
    if (P.depthwise) { d.c = cs; d.k = cs; d.ldc = cout->channel_stored(); }
    {
        const char* e = getenv("B200_SABER_FC_STREAM");
        P.fc_stream = spec.is_fc && !(e && e[0] == '0') && d.n <= b200_fc_stream_max_rows() && !residual && !spec.has_pool;
    }

    // everything the device image depends on
    std::string key;
    {
        int dev = 0;
        cudaGetDevice(&dev);
        key_add(key, dev);
        key_add(key, spec.weights->data());
        key_add(key, b);
        const int32_t sig[] = {math, d.c, d.k, d.r, d.s, static_cast<int32_t>(cin_dt), static_cast<int32_t>(odt), c_real,
                               spec.is_fc ? 1 : 0, stem ? 1 : 0, P.depthwise ? 1 : 0, spec.c_per_group, spec.r, spec.s,
                               P.fc_stream ? 1 : 0};
        key_add(key, sig);
        key_add(key, in_scale);
        key_add(key, out_scale);
    }
    {
        std::lock_guard<std::mutex> lk(g_arena_mu);
        auto it = g_arena.find(key);
        if (it != g_arena.end()) P.dw = it->second.lock();
        else P.dw.reset();
        if (P.dw) ++g_arena_hits;
    }
    bool receive;
    { std::lock_guard<std::mutex> lk(g_arena_mu); receive = g_arena_receive; }
    if (!P.dw && receive) {
        // receive mode: the image arrives by broadcast (weight_arena_import); only its buffers are made here
        std::shared_ptr<DevWeights> dw = std::make_shared<DevWeights>();
        cudaGetDevice(&dw->device);
        const int es = op == AK_INT8 ? 1 : (op == AK_HALF ? 2 : 4);
        size_t w_bytes, n_tab;
        if (P.depthwise) {
            w_bytes = static_cast<size_t>(spec.r) * spec.s * cs * es;
            n_tab = cs;
        } else if (P.fc_stream) {
            w_bytes = static_cast<size_t>(spec.k) * d.c * es;
            n_tab = spec.k;
        } else {
            w_bytes = b200_conv_packed_weight_bytes(&d);
            n_tab = spec.k;
        }
        if (w_bytes == 0 || dw->w.re_alloc(w_bytes, false) != SaberSuccess || dw->bias.re_alloc(n_tab * sizeof(float), false) != SaberSuccess ||
            (op == AK_INT8 && dw->scale.re_alloc(n_tab * sizeof(float), false) != SaberSuccess))
            return SaberOutOfMem;
        std::lock_guard<std::mutex> lk(g_arena_mu);
        g_arena[key] = dw;
        g_arena_order.push_back(dw);
        P.dw = dw;
        ++g_arena_misses;
    }
    if (!P.dw) {
        std::shared_ptr<DevWeights> dw = std::make_shared<DevWeights>();
        cudaGetDevice(&dw->device);
        std::vector<float> bias_f(spec.k, 0.f), scale_f;
        // INT8 epilogue tables from the per-output-channel weight scales (jit_avx512_core_x8s8s32x_conv.cpp:55-62,226-255)
        auto int8_tables = [&](const std::vector<float>& w_scale, int count) {
            const float u = 127.f / 255.f;
            scale_f.assign(count, 1.f);
            bias_f.assign(count, 0.f);
            for (int i = 0; i < spec.k; ++i) {
                float sc;
                if (cin_dt == AK_INT8 && odt == AK_INT8) sc = (w_scale[i] * in_scale) / out_scale;
                else if (cin_dt == AK_UINT8 && odt == AK_UINT8) sc = (w_scale[i] * in_scale * u) / (out_scale * u);
                else if (cin_dt == AK_UINT8 && odt == AK_INT8) sc = (w_scale[i] * in_scale * u) / out_scale;
                else if (cin_dt == AK_UINT8 && odt == AK_FLOAT) sc = w_scale[i] * in_scale * u;
                else if (cin_dt == AK_INT8 && odt == AK_UINT8) sc = (w_scale[i] * in_scale) / (out_scale * u);
                else sc = w_scale[i] * in_scale;
                scale_f[i] = sc;
                const float inv = (cin_dt == AK_UINT8) ? (1.f / (w_scale[i] * in_scale * u))
                                                       : (1.f / (w_scale[i] * in_scale));
                bias_f[i] = b ? b[i] * inv : 0.f;
            }
        };
        if (P.depthwise && op == AK_INT8) {
            // weights [c][1][r][s] -> int8 [r][s][c_stored], one scale per channel (x86_utils.h:293-323: max|w|/127,
            // truncating cast); SaberDepthWiseConv's INT8 arm (saber_depthwiseconv_act.cu:84-295)
            if (odt != AK_INT8 && odt != AK_UINT8) return SaberUnImplError;
            const int RS = spec.r * spec.s;
            std::vector<int8_t> ww(static_cast<size_t>(RS) * cs, 0);
            std::vector<float> w_scale(spec.k, 1.f);
            for (int c = 0; c < spec.k; ++c) {
                float sw = 1.f;
                if (wq8) {
                    sw = wq_scale_of(c);
                } else {
                    float mx = 0.f;
                    for (int i = 0; i < RS; ++i) { const float a = fabsf(w[c * RS + i]); mx = a > mx ? a : mx; }
                    sw = mx / 127.f;
                    if (sw == 0.f) sw = 1.f;
                }
                w_scale[c] = sw;
                for (int i = 0; i < RS; ++i)
                    ww[static_cast<size_t>(i) * cs + c] = wq8 ? wq[c * RS + i] : static_cast<int8_t>(w[c * RS + i] / sw);
            }
            if (upload(dw->w, ww.data(), ww.size()) != SaberSuccess) return SaberOutOfMem;
            int8_tables(w_scale, cs);
            if (upload(dw->scale, scale_f.data(), scale_f.size() * sizeof(float)) != SaberSuccess) return SaberOutOfMem;
            if (upload(dw->bias, bias_f.data(), bias_f.size() * sizeof(float)) != SaberSuccess) return SaberOutOfMem;
        } else if (P.depthwise) {
            // weights [c][1][r][s] -> [r][s][c_stored]
            const int RS = spec.r * spec.s;
            auto wv = [&](int c, int i) { return wq8 ? wq[c * RS + i] * wq_scale_of(c) : w[c * RS + i]; };
            if (op == AK_HALF) {
                std::vector<__half> ww(static_cast<size_t>(RS) * cs, __float2half(0.f));
                for (int c = 0; c < spec.k; ++c)
                    for (int i = 0; i < RS; ++i) ww[static_cast<size_t>(i) * cs + c] = __float2half(wv(c, i));
                if (upload(dw->w, ww.data(), ww.size() * sizeof(__half)) != SaberSuccess) return SaberOutOfMem;
            } else {
                std::vector<float> ww(static_cast<size_t>(RS) * cs, 0.f);
                for (int c = 0; c < spec.k; ++c)
                    for (int i = 0; i < RS; ++i) ww[static_cast<size_t>(i) * cs + c] = wv(c, i);
                if (upload(dw->w, ww.data(), ww.size() * sizeof(float)) != SaberSuccess) return SaberOutOfMem;
            }
            std::vector<float> bb(cs, 0.f);
            for (int i = 0; i < spec.k; ++i) bb[i] = b ? b[i] : 0.f;
            if (upload(dw->bias, bb.data(), bb.size() * sizeof(float)) != SaberSuccess) return SaberOutOfMem;
        } else {
            // operand-typed KCRS image (fc: permuted into the stored-K order), then the wgmma pack
            const int es = op == AK_INT8 ? 1 : (op == AK_HALF ? 2 : 4);
            const int c_img = spec.is_fc ? d.c : c_real;
            const int RS = spec.is_fc ? 1 : (stem ? spec.r : spec.r * spec.s);
            std::vector<uint8_t> img(static_cast<size_t>(spec.k) * c_img * RS * es, 0);
            std::vector<float> w_scale(spec.k, 1.f);
            for (int oc = 0; oc < spec.k; ++oc) {
                const size_t row = static_cast<size_t>(oc) * per_k;
                float sw = 1.f;
                if (op == AK_INT8) {
                    if (wq8) {
                        sw = wq_scale_of(oc);     // codes are used as stored (model_io.cpp:204-216)
                    } else {
                        float mx = 0.f;
                        for (size_t i = 0; i < per_k; ++i) { float a = fabsf(w[row + i]); mx = a > mx ? a : mx; }
                        sw = mx / 127.f;
                        if (sw == 0.f) sw = 1.f;
                    }
                    w_scale[oc] = sw;
                }
                const float deq = wq8 ? wq_scale_of(oc) : 1.f;
                for (int ci = 0; ci < c_img; ++ci) {
                    for (int rs = 0; rs < RS; ++rs) {
                        size_t idx;
                        if (spec.is_fc) {
                            const int col = col_map[ci];
                            if (col < 0) continue;
                            idx = row + col;
                        } else if (stem) {
                            // ci = tap*4 + ch, rs = filter row: w[oc][ch][r][tap]
                            const int tap = ci >> 2, ch = ci & 3;
                            if (tap >= spec.s || ch >= spec.c_per_group) continue;
                            idx = row + (static_cast<size_t>(ch) * spec.r + rs) * spec.s + tap;
                        } else {
                            idx = row + static_cast<size_t>(ci) * RS + rs;
                        }
                        const size_t o = (static_cast<size_t>(oc) * c_img + ci) * RS + rs;
                        if (op == AK_INT8) {
                            reinterpret_cast<int8_t*>(img.data())[o] = wq8 ? wq[idx] : static_cast<int8_t>(w[idx] / sw);
                        } else {
                            const float v = wq8 ? wq[idx] * deq : w[idx];
                            if (op == AK_HALF) reinterpret_cast<__half*>(img.data())[o] = __float2half(v);
                            else reinterpret_cast<float*>(img.data())[o] = v;
                        }
                    }
                }
            }
            if (P.fc_stream) {
                // [n][k] in the stored order of the input row: exactly `img`
                if (upload(dw->w, img.data(), img.size()) != SaberSuccess) return SaberOutOfMem;
            } else {
                const size_t pbytes = b200_conv_packed_weight_bytes(&d);
                if (pbytes == 0) return SaberInvalidValue;
                std::vector<uint8_t> packed(pbytes);
                SaberStatus st = static_cast<SaberStatus>(b200_conv_pack_weights(&d, img.data(), c_img, packed.data()));
                if (st != SaberSuccess) return st;
                if (upload(dw->w, packed.data(), pbytes) != SaberSuccess) return SaberOutOfMem;
            }

            if (op == AK_INT8) {
                int8_tables(w_scale, spec.k);
                if (upload(dw->scale, scale_f.data(), scale_f.size() * sizeof(float)) != SaberSuccess) return SaberOutOfMem;
            } else {
                for (int i = 0; i < spec.k; ++i) bias_f[i] = b ? b[i] : 0.f;
            }
            if (upload(dw->bias, bias_f.data(), bias_f.size() * sizeof(float)) != SaberSuccess) return SaberOutOfMem;
        }
        std::lock_guard<std::mutex> lk(g_arena_mu);
        auto it = g_arena.find(key);
        std::shared_ptr<DevWeights> other = it != g_arena.end() ? it->second.lock() : nullptr;
        if (other) {
            P.dw = other;          // another thread built the same image meanwhile: keep one
        } else {
            g_arena[key] = dw;
            g_arena_order.push_back(dw);
            P.dw = dw;
            ++g_arena_misses;
        }
    }
    d.sum_scale = 1.f;  // float: eltwise coeff 1 (ConvEltwise fuses only Add with coeff {1,1})
    if (op == AK_INT8 && residual) {
        const DataType rdt = residual->get_dtype();
        if (rdt == AK_INT8 && odt == AK_UINT8) d.sum_scale = res_scale * (255.f / 127.f) / out_scale;
        else if (rdt == AK_UINT8 && odt == AK_INT8) d.sum_scale = res_scale * (127.f / 255.f) / out_scale;
        else d.sum_scale = res_scale / out_scale;
    }
    if (P.fc_stream) {
        b200_fc_stream_desc_t& f = P.fc_desc;
        memset(&f, 0, sizeof(f));
        f.math = math; f.in_dtype = cin_dt; f.out_dtype = odt;
        f.m = d.n; f.k = d.c; f.ldx = d.c; f.n_out = spec.k; f.ldo = d.ldc;
        f.relu = d.relu; f.neg_slope = d.neg_slope;
    } else if (!P.depthwise && !P.stem_fused) {
        SaberStatus pst = static_cast<SaberStatus>(b200_conv_plan_create(
            &d, P.dw->w.ptr, static_cast<const float*>(P.dw->bias.ptr),
            op == AK_INT8 ? static_cast<const float*>(P.dw->scale.ptr) : nullptr, &P.plan));
        if (pst == SaberUnImplError && P.pool_fused) {
            // this pooling does not fuse into this conv: conv into a scratch tensor, pooling after it
            P.pool_fused = false;
            d.fuse_pool = 0; d.pool_stride = 0; d.pool_pad = 0; d.pool_floor_as_conv = 0;
            SaberStatus sst = setup_pool_scratch();
            if (sst != SaberSuccess) return sst;
            d.out_dtype = P.conv_out_scratch.get_dtype();
            d.ldc = P.conv_out_scratch.channel_stored();
            pst = static_cast<SaberStatus>(b200_conv_plan_create(
                &d, P.dw->w.ptr, static_cast<const float*>(P.dw->bias.ptr),
                op == AK_INT8 ? static_cast<const float*>(P.dw->scale.ptr) : nullptr, &P.plan));
        }
        if (pst != SaberSuccess) return pst;
    }

    P.in_shape = in.valid_shape();
    P.out_shape = out.valid_shape();
    P.in_dtype = in.get_dtype();
    P.out_dtype = out.get_dtype();
    P.res_dtype = res_dt;
    P.in_scale = in.get_scale();
    P.out_scale = out.get_scale();
    P.res_scale = res_scale;
    P.weights_id = spec.weights->data();
    P.ready = true;
    return SaberSuccess;
}

SaberStatus ConvEngine::run(const Tensor<NV>& in, const Tensor<NV>* residual, Tensor<NV>& out,
                            cudaStream_t stream) {
    Impl& P = *_p;
    if (!P.ready) return SaberNotInitialized;
    const void* src = in.data();
    if (P.need_in_transform && P.stem_fused) {
        const bool pool_after = P.spec.has_pool && !P.stem_pool_fused;
        void* dst = pool_after ? P.conv_out_scratch.mutable_data() : out.mutable_data();
        SaberStatus st = static_cast<SaberStatus>(b200_stem_conv_run(
            &P.stem_desc, static_cast<const float*>(in.data()), P.dw->w.ptr, static_cast<const float*>(P.dw->bias.ptr),
            P.spec.op_dtype == AK_INT8 ? static_cast<const float*>(P.dw->scale.ptr) : nullptr, dst, stream));
        if (st != SaberSuccess) return st;
        if (pool_after)
            st = static_cast<SaberStatus>(b200_pool_run(&P.pool_desc, P.conv_out_scratch.data(), out.mutable_data(), stream));
        return st;
    }
    if (P.need_in_transform && P.stem) {
        SaberStatus st = static_cast<SaberStatus>(b200_stem_pack(
            static_cast<const float*>(in.data()), P.in_scratch.mutable_data(), P.in_scratch.get_dtype(), in.num(),
            in.channel(), in.height(), in.width(), P.spec.pad_h, P.spec.pad_w, P.spec.s, P.spec.stride_w,
            P.stem_taps, P.in_inv_scale, stream));
        if (st != SaberSuccess) return st;
        src = P.in_scratch.data();
    } else if (P.need_in_transform) {
        SaberStatus st = static_cast<SaberStatus>(b200_nchw_to_nhwc(
            static_cast<const float*>(in.data()), P.in_scratch.mutable_data(), P.in_scratch.get_dtype(), in.num(),
            in.channel(), in.height(), in.width(), P.in_scratch.channel_stored(), P.in_inv_scale, 0, stream));
        if (st != SaberSuccess) return st;
        src = P.in_scratch.data();
    }
    const bool pool_after = P.spec.has_pool && !P.pool_fused;
    void* dst = pool_after ? P.conv_out_scratch.mutable_data() : out.mutable_data();
    SaberStatus st;
    if (P.fc_stream) {
        st = static_cast<SaberStatus>(b200_fc_stream_run(
            &P.fc_desc, src, P.dw->w.ptr, static_cast<const float*>(P.dw->bias.ptr),
            P.spec.op_dtype == AK_INT8 ? static_cast<const float*>(P.dw->scale.ptr) : nullptr, dst, stream));
    } else if (P.depthwise) {
        st = static_cast<SaberStatus>(b200_dwconv_run(
            &P.desc, src, P.dw->w.ptr, static_cast<const float*>(P.dw->bias.ptr),
            P.spec.op_dtype == AK_INT8 ? static_cast<const float*>(P.dw->scale.ptr) : nullptr, dst, stream));
    } else {
        st = static_cast<SaberStatus>(b200_conv_plan_run(P.plan, src, residual ? residual->data() : nullptr, dst, stream));
    }
    if (st != SaberSuccess) return st;
    if (pool_after)
        st = static_cast<SaberStatus>(b200_pool_run(&P.pool_desc, P.conv_out_scratch.data(), out.mutable_data(), stream));
    return st;
}

}  // namespace saber
}  // namespace anakin
