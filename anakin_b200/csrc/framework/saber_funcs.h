// The host side of the convolution family over the C ABI: ConvEngine (one fused conv or inner product
// on the wgmma plan), the weight arena it packs into, and the conv / pooling output-size rules.
//   reference saber/funcs/{conv,conv_eltwise,conv_pooling,fc}.h and saber/funcs/impl/cuda/saber_conv*.cpp
#pragma once
#include "saber.h"

namespace anakin {
namespace saber {

// Conv output size: saber/funcs/funcs_utils.h:41-51.
inline int conv_out_size(int in, int pad, int dil, int k, int stride) {
    return (in + 2 * pad - (dil * (k - 1) + 1)) / stride + 1;
}

// One fused convolution (conv | conv+act | conv+eltwise | conv+pool | fc) bound to the
// wgmma plan of the C ABI. Owns the packed weights, bias / scale tables and any scratch.
class ANAKIN_EXPORT ConvEngine {
public:
    ConvEngine();
    ~ConvEngine();
    ConvEngine(const ConvEngine&) = delete;
    ConvEngine& operator=(const ConvEngine&) = delete;

    struct Spec {
        DataType op_dtype = AK_FLOAT;      // AK_FLOAT (3xTF32) | AK_HALF | AK_INT8
        const Tensor<NVHX86>* weights = nullptr;  // fp32 [k][c/g][r][s] (fc: [n_out][K])
        const Tensor<NVHX86>* bias = nullptr;     // fp32 [k] or null / empty
        int k = 0, c_per_group = 0, r = 1, s = 1, group = 1;
        int pad_h = 0, pad_w = 0, stride_h = 1, stride_w = 1, dil_h = 1, dil_w = 1;
        bool relu = false;
        float neg_slope = 0.f;
        float residual_scale = 1.f;        // scale of the residual tensor (the reference's ConvParam::beta)
        bool is_fc = false;                // input flattened in NCHW order (saber_fc.cu:27-35)
        bool has_pool = false;
        b200_pool_desc_t pool{};           // the pooling's type and window; prepare fills in the tensor fields
    };

    // Builds everything that depends on the shapes, dtypes and scales of the tensors; once per engine.
    SaberStatus prepare(const Spec& spec, const Tensor<NV>& in, const Tensor<NV>* residual, Tensor<NV>& out,
                        Context<NV>& ctx);
    SaberStatus run(const Tensor<NV>& in, const Tensor<NV>* residual, Tensor<NV>& out, cudaStream_t stream);
    // device address of the packed weight image this engine runs on (shared between engines through the arena)
    const void* weight_device_ptr() const;
    // the engine is a weight-streaming inner product (few rows): its C-ABI descriptor and device tables, for the
    // fused classifier head
    bool fc_stream_info(b200_fc_stream_desc_t* d, const void** w, const float** bias, const float** scale) const;

private:
    struct Impl;
    Impl* _p;
};

// Live packed-weight images of this process: total device bytes; optionally entry count and how many
// ConvEngine::prepare calls found their image already built (hits) or had to build it (misses).
ANAKIN_EXPORT size_t weight_arena_stats(size_t* entries, size_t* hits, size_t* misses);
// Multi-GPU replicas: export / import the whole arena of a device as one contiguous device buffer (one NCCL broadcast);
// in receive mode ConvEngine::prepare allocates the images without building them. See saber_funcs.cpp.
ANAKIN_EXPORT void weight_arena_set_receive(bool on);
ANAKIN_EXPORT size_t weight_arena_flat_bytes(int device);
ANAKIN_EXPORT SaberStatus weight_arena_export(int device, void* flat_dev, size_t cap);
ANAKIN_EXPORT SaberStatus weight_arena_import(int device, const void* flat_dev, size_t bytes);
// An image of two plain fp32 arrays (weights, bias) in the arena, keyed by (device, id, tag): ops outside the conv family
// whose weights are used as given (the SE gate's inner products). *w_dev / *b_dev point into the entry `dw` holds.
struct DevWeights;
ANAKIN_EXPORT SaberStatus weight_arena_floats(const void* id, const std::string& tag, const std::vector<float>& w,
                                              const std::vector<float>& b, std::shared_ptr<DevWeights>& dw,
                                              const float** w_dev, const float** b_dev);

// Pooling output size: saber/funcs/pooling.h:69-132.
inline void pool_out_size(const b200_pool_desc_t& pool, int in_h, int in_w, int* oh, int* ow) {
    b200_pool_desc_t d = pool;
    d.h = in_h; d.w = in_w;
    int32_t a = 1, b = 1;
    b200_pool_out_hw(&d, &a, &b);
    *oh = a; *ow = b;
}

// The pooling `pool` (type, window, padding, stride, flags) over the tensor `in`: the descriptor b200_pool_run takes.
inline b200_pool_desc_t make_pool_desc(const Tensor<NV>& in, b200_pool_desc_t pool) {
    pool.dtype = in.get_dtype();
    pool.n = in.num(); pool.h = in.height(); pool.w = in.width(); pool.c = in.channel_stored();
    return pool;
}

}  // namespace saber
}  // namespace anakin
