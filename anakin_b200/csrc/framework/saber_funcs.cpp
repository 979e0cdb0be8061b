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


// The live arena entry under `key`, or a new one made by `fill(dw, receive)`: it allocates the buffers and, unless in
// receive mode, writes the image. `fill` runs outside the lock, so engines packing different images do not wait for each
// other.
template <typename Fill>
static SaberStatus arena_acquire(const std::string& key, std::shared_ptr<DevWeights>& dw, Fill fill) {
    auto live = [&]() -> std::shared_ptr<DevWeights> {   // g_arena_mu held
        auto it = g_arena.find(key);
        return it != g_arena.end() ? it->second.lock() : nullptr;
    };
    bool receive;
    {
        std::lock_guard<std::mutex> lk(g_arena_mu);
        dw = live();
        if (dw) { ++g_arena_hits; return SaberSuccess; }
        receive = g_arena_receive;
    }
    std::shared_ptr<DevWeights> made = std::make_shared<DevWeights>();
    cudaGetDevice(&made->device);
    const SaberStatus st = fill(*made, receive);
    if (st != SaberSuccess) return st;
    std::lock_guard<std::mutex> lk(g_arena_mu);
    dw = live();
    if (dw) return SaberSuccess;   // another thread built the same image meanwhile: keep one
    g_arena[key] = made;
    g_arena_order.push_back(made);
    dw = made;
    ++g_arena_misses;
    return SaberSuccess;
}

// ---------------------------------------------------------------------------------------------------------
// What a conv-family op's operand kind (Spec::op_dtype) implies: one row per kind.
struct OperandKind {
    DataType op;                 // Spec::op_dtype
    int math;                    // b200_conv_desc_t::math
    size_t es;                   // operand element bytes
    DataType graph_in;           // the operand dtype a graph input is converted to
    bool (*accepts)(DataType);   // the input dtypes the kernels read
    // INT8: per-channel weight scales, the epilogue scale table, and the input and output scales are required
    bool quantised;
    // writes weight idx of output channel oc (weight scale sc) to element o of the operand-typed image; one of w (fp32)
    // and wq (int8 codes, used as stored: model_io.cpp:204-216) is given. fp32 weights are quantised with a truncating
    // cast.
    void (*put)(uint8_t* img, size_t o, const float* w, const int8_t* wq, size_t idx, float sc);
};

static const OperandKind* operand_kind(DataType op) {
    // FP32 runs as error-compensated 3xTF32 (fp32-grade accuracy: the reference pins FP32 results at
    // 1e-3 against exact-fp32 oracles).
    static const OperandKind kinds[] = {
        {AK_INT8, B200_MATH_I8, 1, AK_INT8, [](DataType d) { return d == AK_INT8 || d == AK_UINT8; }, true,
         [](uint8_t* img, size_t o, const float* w, const int8_t* wq, size_t idx, float sc) {
             reinterpret_cast<int8_t*>(img)[o] = wq ? wq[idx] : static_cast<int8_t>(w[idx] / sc);
         }},
        {AK_HALF, B200_MATH_F16, 2, AK_HALF, [](DataType d) { return d == AK_HALF; }, false,
         [](uint8_t* img, size_t o, const float* w, const int8_t* wq, size_t idx, float sc) {
             reinterpret_cast<__half*>(img)[o] = __float2half(wq ? wq[idx] * sc : w[idx]);
         }},
        {AK_FLOAT, B200_MATH_TF32X3, 4, AK_FLOAT, [](DataType d) { return d == AK_FLOAT; }, false,
         [](uint8_t* img, size_t o, const float* w, const int8_t* wq, size_t idx, float sc) {
             reinterpret_cast<float*>(img)[o] = wq ? wq[idx] * sc : w[idx];
         }},
    };
    for (const OperandKind& k : kinds)
        if (k.op == op) return &k;
    return nullptr;
}

struct ConvEngine::Impl {
    // How the conv's operand is made from the input tensor; ConvEngine::run has one launch sequence for each.
    enum class InputPath {
        Direct,       // the input is the operand
        NchwToNhwc,   // fp32 NCHW -> NHWC operand in in_scratch (b200_nchw_to_nhwc)
        ImageToNhwc,  // 8-bit image -> NHWC operand in in_scratch (b200_image_to_nhwc)
        Stem,         // RGB stem (+ MAX pooling) in one launch that reads the fp32 NCHW tensor or the image (conv_stem.cu)
    };
    // Where the MAX pooling of a ConvPooling runs.
    enum class PoolPath {
        None,    // no pooling
        Plan,    // in the conv plan's epilogue (fuse_pool)
        Stem,    // in the stem kernel (stem_desc.fuse_pool)
        After,   // b200_pool_run over conv_out_scratch, which holds the whole conv output
    };

    Spec spec;
    const OperandKind* kind = nullptr;   // of spec.op_dtype
    bool ready = false;

    b200_conv_desc_t desc;
    b200_conv_plan_t* plan = nullptr;
    std::shared_ptr<DevWeights> dw;   // packed weights / bias / scale tables, shared through the WeightArena
    InputPath in_path = InputPath::Direct;
    PoolPath pool = PoolPath::None;
    b200_stem_desc_t stem_desc;
    Tensor<NV> in_scratch;            // the operand written by NchwToNhwc and ImageToNhwc
    float in_inv_scale = 1.f;
    bool depthwise = false;
    bool fc_stream = false;           // inner product with few rows: b200_fc_stream_run on the plain weight image
    b200_fc_stream_desc_t fc_desc;
    Tensor<NV> conv_out_scratch;
    b200_pool_desc_t pool_desc;

    SaberStatus choose_input_path(const Tensor<NV>& in, const Tensor<NV>* residual, const Tensor<NV>& out, int math);
    SaberStatus pool_after(const Tensor<NV>& out, cudaStream_t stream);

    ~Impl() {
        if (plan) b200_conv_plan_destroy(plan);
    }
};

ConvEngine::ConvEngine() : _p(new Impl()) {}
const void* ConvEngine::weight_device_ptr() const { return _p->dw ? _p->dw->w.ptr : nullptr; }
bool ConvEngine::fc_stream_info(b200_fc_stream_desc_t* d, const void** w, const float** bias, const float** scale) const {
    if (!_p->ready || !_p->fc_stream || _p->in_path != Impl::InputPath::Direct) return false;
    *d = _p->fc_desc;
    *w = _p->dw->w.ptr;
    *bias = static_cast<const float*>(_p->dw->bias.ptr);
    *scale = _p->kind->quantised ? static_cast<const float*>(_p->dw->scale.ptr) : nullptr;
    return true;
}
ConvEngine::~ConvEngine() { delete _p; }

// Sets in_path; for InputPath::Stem also stem_desc. A graph input (fp32 NCHW, or an 8-bit image) is turned into the
// operand with in_inv_scale. An image takes the fp32 input's path with its own readers: b200_stem_conv_run_image where
// the fp32 input takes the fused stem, b200_image_to_nhwc where it takes b200_nchw_to_nhwc.
SaberStatus ConvEngine::Impl::choose_input_path(const Tensor<NV>& in, const Tensor<NV>* residual, const Tensor<NV>& out,
                                                int math) {
    in_path = InputPath::Direct;
    const bool image = in.is_image();
    if (!image && !(in.get_layout() == Layout_NCHW && !(in.height() == 1 && in.width() == 1 && in.get_dtype() != AK_FLOAT)))
        return SaberSuccess;
    if (!image && in.get_dtype() != AK_FLOAT) return SaberUnImplError;
    // graph-input case: fp32 NCHW -> NHWC operand type (the reference quantises inside conv too:
    // saber_conv.cpp:341-381 conv_calibrate_fp32_int8_c4 / x86_utils.h:325-347)
    in_inv_scale = 1.f;
    if (kind->quantised) {
        if (in.get_scale().empty()) return SaberInvalidValue;
        in_inv_scale = 1.f / in.get_scale()[0];
    }
    // RGB stem whose output is a plain 16-byte-multiple NHWC pixel: the whole layer (quantise, conv, epilogue and a
    // following MAX pooling) is one launch that reads the fp32 NCHW tensor itself (b200_stem_conv_run)
    if (!residual && !spec.is_fc && spec.group == 1 && in.channel() <= 4 && spec.s > 1 && spec.s <= 8 && spec.dil_w == 1 &&
        spec.dil_h == 1) {
        b200_stem_desc_t& sd = stem_desc;
        memset(&sd, 0, sizeof(sd));
        sd.math = math;
        sd.n = in.num(); sd.c = in.channel(); sd.h = in.height(); sd.w = in.width();
        sd.k = spec.k;
        sd.r = spec.r; sd.s = spec.s; sd.stride_h = spec.stride_h; sd.stride_w = spec.stride_w;
        sd.pad_h = spec.pad_h; sd.pad_w = spec.pad_w;
        sd.relu = spec.relu ? 1 : 0; sd.neg_slope = spec.neg_slope;
        sd.in_inv_scale = in_inv_scale;
        sd.out_dtype = out.get_dtype();
        sd.ldc = out.channel_stored();
        if (spec.has_pool && spec.pool.type == B200_POOL_MAX && !spec.pool.global_pooling) {
            sd.fuse_pool = 1; sd.pool_type = B200_POOL_MAX;
            sd.pool_window_h = spec.pool.window_h; sd.pool_window_w = spec.pool.window_w;
            sd.pool_pad_h = spec.pool.pad_h; sd.pool_pad_w = spec.pool.pad_w;
            sd.pool_stride_h = spec.pool.stride_h; sd.pool_stride_w = spec.pool.stride_w;
            sd.pool_floor_as_conv = spec.pool.floor_as_conv;
        }
        int32_t oh = 0, ow = 0;
        int st = b200_stem_conv_out_hw(&sd, &oh, &ow);
        if (st != B200_SUCCESS && sd.fuse_pool) {     // this pooling does not fuse: conv here, pooling after it
            sd.fuse_pool = 0;
            st = b200_stem_conv_out_hw(&sd, &oh, &ow);
        }
        const bool direct = !spec.has_pool || sd.fuse_pool;
        if (st == B200_SUCCESS && (!direct || (oh == out.height() && ow == out.width())) &&
            (out.get_layout() == Layout_NHWC || (out.height() == 1 && out.width() == 1))) {
            in_path = InputPath::Stem;
            return SaberSuccess;
        }
    }
    in_path = image ? InputPath::ImageToNhwc : InputPath::NchwToNhwc;
    return SaberSuccess;
}

// Switches to PoolPath::After: the conv writes its whole output into conv_out_scratch, b200_pool_run pools it into `out`.
SaberStatus ConvEngine::Impl::pool_after(const Tensor<NV>& out, cudaStream_t stream) {
    b200_conv_desc_t& d = desc;
    Shape s({d.n, spec.k, conv_out_size(d.h, d.pad_h, d.dil_h, d.r, d.stride_h),
             conv_out_size(d.w, d.pad_w, d.dil_w, d.s, d.stride_w)}, Layout_NHWC);
    if (conv_out_scratch.re_alloc(s, out.get_dtype()) != SaberSuccess) return SaberOutOfMem;
    CUDA_CHECK(cudaMemsetAsync(conv_out_scratch.mutable_data(), 0, conv_out_scratch.storage_bytes(), stream));
    conv_out_scratch.set_scale(out.get_scale());
    pool_desc = make_pool_desc(conv_out_scratch, spec.pool);
    pool = PoolPath::After;
    d.fuse_pool = 0; d.pool_stride = 0; d.pool_pad = 0; d.pool_floor_as_conv = 0;
    d.ldc = conv_out_scratch.channel_stored();
    return SaberSuccess;
}

// Allocates `bytes` of (zeroed) device memory and copies `src` into it when given.
static SaberStatus upload(DeviceBuffer& buf, const void* src, size_t bytes) {
    if (buf.re_alloc(bytes, false) != SaberSuccess) return SaberOutOfMem;
    if (src && bytes && cudaMemcpy(buf.ptr, src, bytes, cudaMemcpyHostToDevice) != cudaSuccess) return SaberUnKownError;
    return SaberSuccess;
}

// ---------------------------------------------------------------------------------------------------------
// Device weight images. An engine's image is its weights in the layout its kernel reads, an fp32 bias table and, for
// INT8, the epilogue scale table.
enum class WeightLayout {
    Packed,      // b200_conv_pack_weights of the operand-typed KCRS image: dense conv, fc
    Stem,        // b200_stem_pack_weights of the operand-typed KCRS image: the fused stem
    Plain,       // the operand-typed [n][k] image in the stored order of the input row: fc-stream
    Depthwise,   // [r][s][c_stored]
};
struct ImageSizes { size_t w, bias, scale; };   // bytes
struct HostImage { std::vector<uint8_t> w; std::vector<float> bias, scale; };

// The bytes of each buffer of an image (d: the conv in the kernel's view; sd: the fused stem's, for Stem). Receive mode
// allocates these without building the image; build_weight_image fails if what it builds has other sizes, so an
// imported image always fits.
static ImageSizes weight_image_sizes(WeightLayout layout, const b200_conv_desc_t& d, const b200_stem_desc_t& sd,
                                     const OperandKind& kind) {
    const size_t es = kind.es;
    size_t w = 0, n_tab = d.k;
    switch (layout) {
        case WeightLayout::Packed: w = b200_conv_packed_weight_bytes(&d); break;
        case WeightLayout::Stem: w = b200_stem_packed_weight_bytes(&sd); break;
        case WeightLayout::Plain: w = static_cast<size_t>(d.k) * d.c * es; break;
        case WeightLayout::Depthwise: w = static_cast<size_t>(d.r) * d.s * d.c * es; n_tab = d.c; break;
    }
    return {w, n_tab * sizeof(float), kind.quantised ? n_tab * sizeof(float) : 0};
}

static const float* spec_bias(const ConvEngine::Spec& spec) {
    const bool has_bias = spec.bias && spec.bias->valid_size() >= spec.k && spec.bias->data();
    return has_bias ? static_cast<const float*>(spec.bias->data()) : nullptr;
}

// Per-output-channel INT8 weight scale over the channel's per_k weights: the stored scale of int8 codes, else
// max|w|/127 with 0 -> 1 (x86_utils.h:293-323).
static float int8_weight_scale(const Tensor<NVHX86>& wt, int oc, size_t per_k) {
    const std::vector<float>& stored = wt.get_scale();
    if (wt.get_dtype() == AK_INT8) return stored[static_cast<size_t>(oc) < stored.size() ? oc : stored.size() - 1];
    const float* w = static_cast<const float*>(wt.data()) + static_cast<size_t>(oc) * per_k;
    float mx = 0.f;
    for (size_t i = 0; i < per_k; ++i) { const float a = fabsf(w[i]); mx = a > mx ? a : mx; }
    const float sw = mx / 127.f;
    return sw == 0.f ? 1.f : sw;
}

// Builds the host bytes of an image of sizes `sz`. d is the conv in the kernel's view, sd the fused stem's (for Stem);
// col_map gives an fc's weight column (NCHW flatten) for every stored K position, -1 = pad.
static SaberStatus build_weight_image(const ConvEngine::Spec& spec, const OperandKind& kind, WeightLayout layout,
                                      const b200_conv_desc_t& d, const b200_stem_desc_t& sd, const ImageSizes& sz,
                                      const std::vector<int>& col_map, DataType cin_dt, DataType odt, float in_scale,
                                      float out_scale, HostImage& img) {
    const Tensor<NVHX86>& wt = *spec.weights;
    const bool wq8 = wt.get_dtype() == AK_INT8;   // model file carries int8 codes + per-channel scales
    const float* w = wq8 ? nullptr : static_cast<const float*>(wt.data());
    const int8_t* wq = wq8 ? static_cast<const int8_t*>(wt.data()) : nullptr;
    const size_t es = kind.es;
    const size_t per_k = static_cast<size_t>(spec.is_fc ? spec.c_per_group : spec.c_per_group * spec.r * spec.s);
    // the per-output-channel scale: INT8 quantisation, or the dequantisation of int8 codes for fp16 / fp32
    std::vector<float> w_scale(spec.k, 1.f);
    for (int oc = 0; oc < spec.k; ++oc)
        if (kind.quantised || wq8) w_scale[oc] = int8_weight_scale(wt, oc, per_k);
    auto put = [&](size_t o, size_t idx, int oc) { kind.put(img.w.data(), o, w, wq, idx, w_scale[oc]); };
    if (layout == WeightLayout::Depthwise) {
        // weights [c][1][r][s] -> [r][s][c_stored]; INT8 is SaberDepthWiseConv's INT8 arm (saber_depthwiseconv_act.cu:84-295)
        if (kind.quantised && odt != AK_INT8 && odt != AK_UINT8) return SaberUnImplError;
        const int RS = spec.r * spec.s;
        img.w.assign(static_cast<size_t>(RS) * d.c * es, 0);
        for (int c = 0; c < spec.k; ++c)
            for (int i = 0; i < RS; ++i) put(static_cast<size_t>(i) * d.c + c, static_cast<size_t>(c) * RS + i, c);
    } else {
        // operand-typed KCRS image (fc: permuted into the stored-K order); Packed and Stem then pack it for wgmma
        const int c_img = spec.is_fc ? d.c : spec.c_per_group;
        const int RS = spec.is_fc ? 1 : spec.r * spec.s;
        img.w.assign(static_cast<size_t>(spec.k) * c_img * RS * es, 0);
        for (int oc = 0; oc < spec.k; ++oc) {
            const size_t row = static_cast<size_t>(oc) * per_k;
            for (int ci = 0; ci < c_img; ++ci) {
                for (int rs = 0; rs < RS; ++rs) {
                    size_t idx;
                    if (spec.is_fc) {
                        const int col = col_map[ci];
                        if (col < 0) continue;
                        idx = row + col;
                    } else {
                        idx = row + static_cast<size_t>(ci) * RS + rs;
                    }
                    put((static_cast<size_t>(oc) * c_img + ci) * RS + rs, idx, oc);
                }
            }
        }
        if (layout != WeightLayout::Plain) {
            std::vector<uint8_t> packed(sz.w);
            const SaberStatus st = static_cast<SaberStatus>(
                layout == WeightLayout::Stem ? b200_stem_pack_weights(&sd, img.w.data(), packed.data())
                                             : b200_conv_pack_weights(&d, img.w.data(), c_img, packed.data()));
            if (st != SaberSuccess) return st;
            img.w.swap(packed);
        }
    }
    // one table entry per channel the kernel writes (depthwise: per stored channel)
    const size_t n_tab = layout == WeightLayout::Depthwise ? d.c : spec.k;
    const float* b = spec_bias(spec);
    img.bias.assign(n_tab, 0.f);
    if (kind.quantised) {
        // INT8 epilogue tables from the per-output-channel weight scales (jit_avx512_core_x8s8s32x_conv.cpp:55-62,226-255)
        const float u = 127.f / 255.f;
        img.scale.assign(n_tab, 1.f);
        for (int i = 0; i < spec.k; ++i) {
            float sc;
            if (cin_dt == AK_INT8 && odt == AK_INT8) sc = (w_scale[i] * in_scale) / out_scale;
            else if (cin_dt == AK_UINT8 && odt == AK_UINT8) sc = (w_scale[i] * in_scale * u) / (out_scale * u);
            else if (cin_dt == AK_UINT8 && odt == AK_INT8) sc = (w_scale[i] * in_scale * u) / out_scale;
            else if (cin_dt == AK_UINT8 && odt == AK_FLOAT) sc = w_scale[i] * in_scale * u;
            else if (cin_dt == AK_INT8 && odt == AK_UINT8) sc = (w_scale[i] * in_scale) / (out_scale * u);
            else sc = w_scale[i] * in_scale;
            img.scale[i] = sc;
            const float inv = (cin_dt == AK_UINT8) ? (1.f / (w_scale[i] * in_scale * u))
                                                   : (1.f / (w_scale[i] * in_scale));
            img.bias[i] = b ? b[i] * inv : 0.f;
        }
    } else {
        for (int i = 0; i < spec.k; ++i) img.bias[i] = b ? b[i] : 0.f;
    }
    if (img.w.size() != sz.w || img.bias.size() * sizeof(float) != sz.bias || img.scale.size() * sizeof(float) != sz.scale)
        return SaberUnKownError;
    return SaberSuccess;
}

SaberStatus weight_arena_floats(const void* id, const std::string& tag, const std::vector<float>& w,
                                const std::vector<float>& b, std::shared_ptr<DevWeights>& dw, const float** w_dev,
                                const float** b_dev) {
    std::string key;
    int dev = 0;
    cudaGetDevice(&dev);
    key_add(key, dev);
    key_add(key, id);
    key_add(key, w.size());
    key_add(key, b.size());
    key += tag;
    const SaberStatus st = arena_acquire(key, dw, [&](DevWeights& d, bool receive) -> SaberStatus {
        if (upload(d.w, receive ? nullptr : w.data(), w.size() * sizeof(float)) != SaberSuccess ||
            upload(d.bias, receive ? nullptr : b.data(), b.size() * sizeof(float)) != SaberSuccess)
            return SaberOutOfMem;
        return SaberSuccess;
    });
    if (st != SaberSuccess) return st;
    *w_dev = static_cast<const float*>(dw->w.ptr);
    *b_dev = static_cast<const float*>(dw->bias.ptr);
    return SaberSuccess;
}

SaberStatus ConvEngine::prepare(const Spec& spec, const Tensor<NV>& in, const Tensor<NV>* residual,
                                Tensor<NV>& out, Context<NV>& ctx) {
    using InputPath = Impl::InputPath;
    using PoolPath = Impl::PoolPath;
    Impl& P = *_p;
    const float res_scale = spec.residual_scale;
    P.spec = spec;
    P.kind = operand_kind(spec.op_dtype);
    if (!P.kind) return SaberUnImplError;
    const OperandKind& kind = *P.kind;
    const int math = kind.math;

    // ---- 1. the tensor the conv kernel reads (NHWC in the op's operand type)
    SaberStatus st = P.choose_input_path(in, residual, out, math);
    if (st != SaberSuccess) return st;
    const DataType cin_dt = P.in_path == InputPath::Direct ? in.get_dtype() : kind.graph_in;
    const Tensor<NV>* cin = &in;   // the fused stem reads `in` itself
    if (P.in_path == InputPath::NchwToNhwc || P.in_path == InputPath::ImageToNhwc) {
        Shape s = in.valid_shape();
        s.set_layout(Layout_NHWC);
        if (P.in_scratch.re_alloc(s, cin_dt) != SaberSuccess) return SaberOutOfMem;
        CUDA_CHECK(cudaMemsetAsync(P.in_scratch.mutable_data(), 0, P.in_scratch.storage_bytes(), ctx.get_compute_stream()));
        cin = &P.in_scratch;
    }
    if (!kind.accepts(cin_dt)) return SaberUnImplError;
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
    } else {
        d.n = cin->num(); d.h = cin->height(); d.w = cin->width(); d.c = cs;
        d.r = spec.r; d.s = spec.s;
        d.pad_h = spec.pad_h; d.pad_w = spec.pad_w;
        d.stride_h = spec.stride_h; d.stride_w = spec.stride_w;
        d.dil_h = spec.dil_h; d.dil_w = spec.dil_w;
        c_real = spec.c_per_group;
    }
    d.k = spec.k;
    P.depthwise = !spec.is_fc && spec.group > 1 && spec.group == cin->channel() && spec.c_per_group == 1 &&
                  spec.k == spec.group;
    if (spec.group != 1 && !P.depthwise) return SaberUnImplError;
    if (!spec.is_fc && !P.depthwise && c_real != cin->channel()) return SaberInvalidValue;

    // ---- 3. where the conv writes, and where its MAX pooling runs
    const DataType odt = out.get_dtype();
    d.out_dtype = odt;
    d.ldc = out.channel_stored();
    P.pool = PoolPath::None;
    // conv + MAX pooling in one launch (the conv plan's fuse_pool) when the window is square; the plan decides
    if (spec.has_pool) {
        if (P.in_path == InputPath::Stem && P.stem_desc.fuse_pool) {
            P.pool = PoolPath::Stem;
        } else if (P.in_path == InputPath::Direct && !spec.is_fc && !residual && spec.group == 1 &&
                   spec.pool.type == B200_POOL_MAX && !spec.pool.global_pooling &&
                   spec.pool.window_h == spec.pool.window_w && spec.pool.stride_h == spec.pool.stride_w &&
                   spec.pool.pad_h == spec.pool.pad_w && out.get_layout() == Layout_NHWC) {
            P.pool = PoolPath::Plan;
            d.fuse_pool = spec.pool.window_h;
            d.pool_stride = spec.pool.stride_h;
            d.pool_pad = spec.pool.pad_h;
            d.pool_floor_as_conv = spec.pool.floor_as_conv;
        } else if ((st = P.pool_after(out, ctx.get_compute_stream())) != SaberSuccess) {
            return st;
        }
    }
    if (residual && residual->channel_stored() != d.ldc) return SaberInvalidValue;

    // ---- 4. weights, bias, scales: looked up in / built into the WeightArena
    const std::vector<float>& wq_scale = spec.weights->get_scale();
    if (spec.weights->get_dtype() == AK_INT8 && wq_scale.empty()) return SaberInvalidValue;
    float in_scale = 1.f, out_scale = 1.f;
    if (kind.quantised) {
        if (in.get_scale().empty()) return SaberInvalidValue;
        in_scale = in.get_scale()[0];
        if (odt != AK_FLOAT) {
            if (out.get_scale().empty()) return SaberInvalidValue;
            out_scale = out.get_scale()[0];
        }
    }
    if (P.in_path == InputPath::Stem) {
        // the fused pooling may run on the raw accumulators when the epilogue is non-decreasing in them
        bool pos = spec.neg_slope >= 0.f;
        if (kind.quantised) {
            pos = pos && in_scale > 0.f && out_scale > 0.f;
            for (float sc : wq_scale) pos = pos && sc > 0.f;
        }
        P.stem_desc.monotone_epilogue = pos ? 1 : 0;
    }
    if (P.depthwise) { d.c = cs; d.k = cs; }
    P.fc_stream = spec.is_fc && d.n <= b200_fc_stream_max_rows() && !residual && !spec.has_pool;
    const WeightLayout layout = P.in_path == InputPath::Stem ? WeightLayout::Stem
                                : P.depthwise                ? WeightLayout::Depthwise
                                : P.fc_stream                ? WeightLayout::Plain
                                                             : WeightLayout::Packed;

    // everything the device image depends on
    std::string key;
    {
        int dev = 0;
        cudaGetDevice(&dev);
        key_add(key, dev);
        key_add(key, spec.weights->data());
        key_add(key, spec_bias(spec));
        const int32_t sig[] = {math, d.c, d.k, d.r, d.s, static_cast<int32_t>(cin_dt), static_cast<int32_t>(odt), c_real,
                               spec.is_fc ? 1 : 0, static_cast<int32_t>(layout), spec.c_per_group, spec.r, spec.s};
        key_add(key, sig);
        key_add(key, in_scale);
        key_add(key, out_scale);
    }
    st = arena_acquire(key, P.dw, [&](DevWeights& dw, bool receive) -> SaberStatus {
        const ImageSizes sz = weight_image_sizes(layout, d, P.stem_desc, kind);
        if (sz.w == 0) return SaberInvalidValue;
        // receive mode: the image arrives by broadcast (weight_arena_import); only its buffers are made here
        HostImage img;
        if (!receive) {
            const SaberStatus bst = build_weight_image(spec, kind, layout, d, P.stem_desc, sz, col_map, cin_dt, odt,
                                                       in_scale, out_scale, img);
            if (bst != SaberSuccess) return bst;
        }
        if (upload(dw.w, receive ? nullptr : img.w.data(), sz.w) != SaberSuccess ||
            upload(dw.bias, receive ? nullptr : img.bias.data(), sz.bias) != SaberSuccess ||
            upload(dw.scale, receive ? nullptr : img.scale.data(), sz.scale) != SaberSuccess)
            return SaberOutOfMem;
        return SaberSuccess;
    });
    if (st != SaberSuccess) return st;

    d.sum_scale = 1.f;  // float: eltwise coeff 1 (ConvEltwise fuses only Add with coeff {1,1})
    if (kind.quantised && residual) {
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
    } else if (!P.depthwise && P.in_path != InputPath::Stem) {
        auto create_plan = [&] {
            return static_cast<SaberStatus>(b200_conv_plan_create(
                &d, P.dw->w.ptr, static_cast<const float*>(P.dw->bias.ptr),
                kind.quantised ? static_cast<const float*>(P.dw->scale.ptr) : nullptr, &P.plan));
        };
        st = create_plan();
        if (st == SaberUnImplError && P.pool == PoolPath::Plan) {
            // this pooling does not fuse into this conv: conv into a scratch tensor, pooling after it
            st = P.pool_after(out, ctx.get_compute_stream());
            if (st == SaberSuccess) st = create_plan();
        }
        if (st != SaberSuccess) return st;
    }

    P.ready = true;
    return SaberSuccess;
}

SaberStatus ConvEngine::run(const Tensor<NV>& in, const Tensor<NV>* residual, Tensor<NV>& out,
                            cudaStream_t stream) {
    using InputPath = Impl::InputPath;
    Impl& P = *_p;
    if (!P.ready) return SaberNotInitialized;
    const float* bias = static_cast<const float*>(P.dw->bias.ptr);
    const float* scale = P.kind->quantised ? static_cast<const float*>(P.dw->scale.ptr) : nullptr;
    const bool pool_after = P.pool == Impl::PoolPath::After;
    void* dst = pool_after ? P.conv_out_scratch.mutable_data() : out.mutable_data();
    Tensor<NV>& x = P.in_scratch;
    SaberStatus st = SaberSuccess;
    switch (P.in_path) {
        case InputPath::Direct:
            break;
        case InputPath::NchwToNhwc:
            st = static_cast<SaberStatus>(b200_nchw_to_nhwc(
                static_cast<const float*>(in.data()), x.mutable_data(), x.get_dtype(), in.num(), in.channel(),
                in.height(), in.width(), x.channel_stored(), P.in_inv_scale, stream));
            break;
        case InputPath::ImageToNhwc:
            st = static_cast<SaberStatus>(b200_image_to_nhwc(
                &in.image_desc(), static_cast<const uint8_t*>(in.data()), x.mutable_data(), x.get_dtype(), in.num(),
                in.channel(), in.height(), in.width(), x.channel_stored(), P.in_inv_scale, stream));
            break;
        case InputPath::Stem:   // the whole conv, reading the graph input: an 8-bit image or fp32 NCHW
            st = static_cast<SaberStatus>(
                in.is_image()
                    ? b200_stem_conv_run_image(&P.stem_desc, &in.image_desc(), static_cast<const uint8_t*>(in.data()),
                                               P.dw->w.ptr, bias, scale, dst, stream)
                    : b200_stem_conv_run(&P.stem_desc, static_cast<const float*>(in.data()), P.dw->w.ptr, bias, scale,
                                         dst, stream));
            break;
    }
    if (st != SaberSuccess) return st;
    if (P.in_path != InputPath::Stem) {
        const void* src = P.in_path == InputPath::Direct ? in.data() : x.data();
        if (P.fc_stream)
            st = static_cast<SaberStatus>(b200_fc_stream_run(&P.fc_desc, src, P.dw->w.ptr, bias, scale, dst, stream));
        else if (P.depthwise)
            st = static_cast<SaberStatus>(b200_dwconv_run(&P.desc, src, P.dw->w.ptr, bias, scale, dst, stream));
        else
            st = static_cast<SaberStatus>(b200_conv_plan_run(P.plan, src, residual ? residual->data() : nullptr, dst, stream));
        if (st != SaberSuccess) return st;
    }
    if (pool_after)
        st = static_cast<SaberStatus>(b200_pool_run(&P.pool_desc, P.conv_out_scratch.data(), out.mutable_data(), stream));
    return st;
}

}  // namespace saber
}  // namespace anakin
