// Saber funcs + impls for target NV over the C ABI (see saber.h for the mapping).
//   reference saber/funcs/{conv,conv_eltwise,conv_pooling,fc,pooling,softmax,eltwise,
//   activation,scale}.h  and  saber/funcs/impl/cuda/saber_*.{cpp,cu}
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
        DataType op_dtype = AK_FLOAT;      // AK_FLOAT (tf32) | AK_HALF | AK_INT8
        const Tensor<NVHX86>* weights = nullptr;  // fp32 [k][c/g][r][s] (fc: [n_out][K])
        const Tensor<NVHX86>* bias = nullptr;     // fp32 [k] or null / empty
        int k = 0, c_per_group = 0, r = 1, s = 1, group = 1;
        int pad_h = 0, pad_w = 0, stride_h = 1, stride_w = 1, dil_h = 1, dil_w = 1;
        bool relu = false;
        float neg_slope = 0.f;
        bool has_residual = false;
        float residual_scale = 1.f;        // scale of the residual tensor (ConvParam::beta)
        bool is_fc = false;                // input flattened in NCHW order (saber_fc.cu:27-35)
        bool has_pool = false;
        PoolingParam<NV> pool;
    };

    // (Re)build everything that depends on shapes / scales; cheap when nothing changed.
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

// ------------------------------------------------------------------------------------- conv
template <typename T, DataType OpDtype>
class SaberConv2D : public ImplBase<ConvParam<T>> {
public:
    typedef typename ImplBase<ConvParam<T>>::TensorVec TensorVec;
    SaberStatus init(const TensorVec& in, TensorVec& out, ConvParam<T>& p, Context<NV>& ctx) override {
        this->_ctx = &ctx;
        return create(in, out, p, ctx);
    }
    SaberStatus create(const TensorVec& in, TensorVec& out, ConvParam<T>& p, Context<NV>& ctx) override {
        this->_ctx = &ctx;
        return _eng.prepare(make_spec(p, OpDtype), *in[0], nullptr, *out[0], ctx);
    }
    SaberStatus dispatch(const TensorVec& in, TensorVec& out, ConvParam<T>& p) override {
        return _eng.run(*in[0], nullptr, *out[0], this->_ctx->get_compute_stream());
    }
    static ConvEngine::Spec make_spec(const ConvParam<T>& p, DataType op) {
        ConvEngine::Spec s;
        s.op_dtype = op;
        s.weights = p.weight_tensor;
        s.bias = p.bias_tensor;
        s.k = p.weight_tensor->num();
        s.c_per_group = p.weight_tensor->channel();
        s.r = p.weight_tensor->height();
        s.s = p.weight_tensor->width();
        s.group = p.group;
        s.pad_h = p.pad_h; s.pad_w = p.pad_w;
        s.stride_h = p.stride_h; s.stride_w = p.stride_w;
        s.dil_h = p.dilation_h; s.dil_w = p.dilation_w;
        s.relu = p.activation_param.has_active && p.activation_param.active == Active_relu;
        s.neg_slope = p.activation_param.negative_slope;
        return s;
    }

    const ConvEngine& engine() const { return _eng; }

private:
    ConvEngine _eng;
};

// conv + eltwise-sum (+relu): residual = in[1] when given, else the output buffer itself
// (beta = 1 accumulate, saber_conv_eltwise.cpp:113-125).
template <typename T, DataType OpDtype>
class SaberConvEltwise : public ImplBase<ConvEltwiseParam<T>> {
public:
    typedef typename ImplBase<ConvEltwiseParam<T>>::TensorVec TensorVec;
    SaberStatus init(const TensorVec& in, TensorVec& out, ConvEltwiseParam<T>& p, Context<NV>& ctx) override {
        this->_ctx = &ctx;
        return create(in, out, p, ctx);
    }
    SaberStatus create(const TensorVec& in, TensorVec& out, ConvEltwiseParam<T>& p, Context<NV>& ctx) override {
        this->_ctx = &ctx;
        ConvEngine::Spec s = SaberConv2D<T, OpDtype>::make_spec(p.conv_param, OpDtype);
        if (p.eltwise_param.operation != Eltwise_sum) return SaberUnImplError;
        s.has_residual = true;
        s.residual_scale = p.conv_param.beta;
        // the activation after the sum lives in the eltwise param (conv_eltwise.cpp:154-176)
        if (p.eltwise_param.activation_param.has_active) {
            s.relu = p.eltwise_param.activation_param.active == Active_relu;
            s.neg_slope = p.eltwise_param.activation_param.negative_slope;
        }
        const Tensor<NV>* res = in.size() > 1 ? in[1] : out[0];
        return _eng.prepare(s, *in[0], res, *out[0], ctx);
    }
    SaberStatus dispatch(const TensorVec& in, TensorVec& out, ConvEltwiseParam<T>& p) override {
        const Tensor<NV>* res = in.size() > 1 ? in[1] : out[0];
        return _eng.run(*in[0], res, *out[0], this->_ctx->get_compute_stream());
    }

    const ConvEngine& engine() const { return _eng; }

private:
    ConvEngine _eng;
};

template <typename T, DataType OpDtype>
class SaberConv2DPooling : public ImplBase<ConvPoolingParam<T>> {
public:
    typedef typename ImplBase<ConvPoolingParam<T>>::TensorVec TensorVec;
    SaberStatus init(const TensorVec& in, TensorVec& out, ConvPoolingParam<T>& p, Context<NV>& ctx) override {
        this->_ctx = &ctx;
        return create(in, out, p, ctx);
    }
    SaberStatus create(const TensorVec& in, TensorVec& out, ConvPoolingParam<T>& p, Context<NV>& ctx) override {
        this->_ctx = &ctx;
        ConvEngine::Spec s = SaberConv2D<T, OpDtype>::make_spec(p.conv_param, OpDtype);
        s.has_pool = true;
        s.pool = p.pooling_param;
        return _eng.prepare(s, *in[0], nullptr, *out[0], ctx);
    }
    SaberStatus dispatch(const TensorVec& in, TensorVec& out, ConvPoolingParam<T>& p) override {
        return _eng.run(*in[0], nullptr, *out[0], this->_ctx->get_compute_stream());
    }

    const ConvEngine& engine() const { return _eng; }

private:
    ConvEngine _eng;
};

// fc: out[m][n] = in[m][k] * W[n][k]^T + b  (saber_fc.cu:17-195) on the same wgmma plan.
template <typename T, DataType OpDtype>
class SaberFc : public ImplBase<FcParam<T>> {
public:
    typedef typename ImplBase<FcParam<T>>::TensorVec TensorVec;
    SaberStatus init(const TensorVec& in, TensorVec& out, FcParam<T>& p, Context<NV>& ctx) override {
        this->_ctx = &ctx;
        return create(in, out, p, ctx);
    }
    SaberStatus create(const TensorVec& in, TensorVec& out, FcParam<T>& p, Context<NV>& ctx) override {
        this->_ctx = &ctx;
        if (p.is_transpose_weights) return SaberUnImplError;
        ConvEngine::Spec s;
        s.op_dtype = OpDtype;
        s.weights = p.weights;
        s.bias = p.bias;
        s.k = p.num_output;
        s.c_per_group = static_cast<int>(in[0]->count_valid(p.axis, 4));
        s.is_fc = true;
        s.relu = p.activation_param.has_active && p.activation_param.active == Active_relu;
        s.neg_slope = p.activation_param.negative_slope;
        return _eng.prepare(s, *in[0], nullptr, *out[0], ctx);
    }
    SaberStatus dispatch(const TensorVec& in, TensorVec& out, FcParam<T>& p) override {
        return _eng.run(*in[0], nullptr, *out[0], this->_ctx->get_compute_stream());
    }

    const ConvEngine& engine() const { return _eng; }

private:
    ConvEngine _eng;
};

// ------------------------------------------------------------------------------------- pointwise impls
ANAKIN_EXPORT b200_pool_desc_t make_pool_desc(const Tensor<NV>& in, const PoolingParam<NV>& p);

template <typename T, DataType OpDtype>
class SaberPooling : public ImplBase<PoolingParam<T>> {
public:
    typedef typename ImplBase<PoolingParam<T>>::TensorVec TensorVec;
    SaberStatus init(const TensorVec& in, TensorVec& out, PoolingParam<T>& p, Context<NV>& ctx) override {
        return create(in, out, p, ctx);
    }
    SaberStatus create(const TensorVec& in, TensorVec& out, PoolingParam<T>& p, Context<NV>& ctx) override {
        this->_ctx = &ctx;
        if (in[0]->get_layout() != Layout_NHWC || out[0]->get_layout() != Layout_NHWC) return SaberInvalidValue;
        if (in[0]->get_dtype() != out[0]->get_dtype()) return SaberInvalidValue;
        // int8 pooling passes its input scale through (reference x86 saber_pooling.cpp:583-584)
        out[0]->set_scale(in[0]->get_scale());
        return SaberSuccess;
    }
    SaberStatus dispatch(const TensorVec& in, TensorVec& out, PoolingParam<T>& p) override {
        b200_pool_desc_t d = make_pool_desc(*in[0], p);
        return static_cast<SaberStatus>(
            b200_pool_run(&d, in[0]->data(), out[0]->mutable_data(), this->_ctx->get_compute_stream()));
    }
};

template <typename T, DataType OpDtype>
class SaberSoftmax : public ImplBase<SoftmaxParam<T>> {
public:
    typedef typename ImplBase<SoftmaxParam<T>>::TensorVec TensorVec;
    SaberStatus init(const TensorVec& in, TensorVec& out, SoftmaxParam<T>& p, Context<NV>& ctx) override {
        return create(in, out, p, ctx);
    }
    SaberStatus create(const TensorVec& in, TensorVec& out, SoftmaxParam<T>& p, Context<NV>& ctx) override {
        this->_ctx = &ctx;
        const Tensor<NV>& x = *in[0];
        if (x.get_dtype() != AK_FLOAT || out[0]->get_dtype() != AK_FLOAT) return SaberUnImplError;
        // logical NCHW axes -> (outer, axis, inner) of the stored layout
        const bool flat = x.height() == 1 && x.width() == 1;
        _in_pitch = _out_pitch = 0;
        if (p.axis == 1 && (flat || x.get_layout() == Layout_NHWC)) {
            // channels are innermost: one row per pixel, row pitch = stored (padded) channels
            _outer = x.num() * x.height() * x.width();
            _len = x.channel();
            _inner = 1;
            _in_pitch = x.channel_stored();
            _out_pitch = out[0]->channel_stored();
        } else if (x.get_layout() == Layout_NCHW) {
            _outer = static_cast<int>(x.count_valid(0, p.axis));
            _len = x.valid_shape()[p.axis];
            _inner = static_cast<int>(x.count_valid(p.axis + 1, 4));
        } else {
            return SaberUnImplError;
        }
        return SaberSuccess;
    }
    SaberStatus dispatch(const TensorVec& in, TensorVec& out, SoftmaxParam<T>& p) override {
        if (_in_pitch)
            return static_cast<SaberStatus>(b200_softmax_rows(static_cast<const float*>(in[0]->data()),
                                                              static_cast<float*>(out[0]->mutable_data()), _outer,
                                                              _len, _in_pitch, _out_pitch,
                                                              this->_ctx->get_compute_stream()));
        return static_cast<SaberStatus>(b200_softmax_run(static_cast<const float*>(in[0]->data()),
                                                         static_cast<float*>(out[0]->mutable_data()), _outer,
                                                         _len, _inner, this->_ctx->get_compute_stream()));
    }

private:
    int _outer = 0, _len = 0, _inner = 1, _in_pitch = 0, _out_pitch = 0;
};

template <typename T, DataType OpDtype>
class SaberEltwise : public ImplBase<EltwiseParam<T>> {
public:
    typedef typename ImplBase<EltwiseParam<T>>::TensorVec TensorVec;
    SaberStatus init(const TensorVec& in, TensorVec& out, EltwiseParam<T>& p, Context<NV>& ctx) override {
        return create(in, out, p, ctx);
    }
    SaberStatus create(const TensorVec& in, TensorVec& out, EltwiseParam<T>& p, Context<NV>& ctx) override {
        this->_ctx = &ctx;
        if (in.size() != 2) return SaberUnImplError;
        if (in[0]->storage_bytes() != in[1]->storage_bytes()) return SaberInvalidValue;
        _c0 = p.coeff.size() > 0 ? p.coeff[0] : 1.f;
        _c1 = p.coeff.size() > 1 ? p.coeff[1] : 1.f;
        const DataType d0 = in[0]->get_dtype(), d1 = in[1]->get_dtype(), dout = out[0]->get_dtype();
        auto q8 = [](DataType d) { return d == AK_INT8 || d == AK_UINT8; };
        if (q8(d0)) {
            // x86 int8 eltwise (saber_eltwise.cpp:72-111): tmp = sum coeff*code*scale, rescaled to
            // the output code space; u8 tensors carry scale*127/255.
            if (!q8(d1) || !q8(dout) || in[0]->get_scale().empty() || in[1]->get_scale().empty() ||
                out[0]->get_scale().empty())
                return SaberInvalidValue;
            const float u = 127.f / 255.f;
            const float f0 = in[0]->get_scale()[0] * (d0 == AK_UINT8 ? u : 1.f);
            const float f1 = in[1]->get_scale()[0] * (d1 == AK_UINT8 ? u : 1.f);
            const float fo = out[0]->get_scale()[0] * (dout == AK_UINT8 ? u : 1.f);
            _c0 = _c0 * (f0 / fo);
            _c1 = _c1 * (f1 / fo);
        }
        return SaberSuccess;
    }
    SaberStatus dispatch(const TensorVec& in, TensorVec& out, EltwiseParam<T>& p) override {
        const size_t count = in[0]->storage_bytes() / type_length(in[0]->get_dtype());
        const int relu = p.activation_param.has_active && p.activation_param.active == Active_relu;
        return static_cast<SaberStatus>(b200_eltwise_run(
            in[0]->get_dtype(), in[1]->get_dtype(), out[0]->get_dtype(), p.operation, in[0]->data(), in[1]->data(),
            out[0]->mutable_data(), count, _c0, _c1, relu, this->_ctx->get_compute_stream()));
    }

private:
    float _c0 = 1.f, _c1 = 1.f;
};

template <typename T, DataType OpDtype>
class SaberActivation : public ImplBase<ActivationParam<T>> {
public:
    typedef typename ImplBase<ActivationParam<T>>::TensorVec TensorVec;
    SaberStatus init(const TensorVec& in, TensorVec& out, ActivationParam<T>& p, Context<NV>& ctx) override {
        return create(in, out, p, ctx);
    }
    SaberStatus create(const TensorVec& in, TensorVec& out, ActivationParam<T>& p, Context<NV>& ctx) override {
        this->_ctx = &ctx;
        return SaberSuccess;
    }
    SaberStatus dispatch(const TensorVec& in, TensorVec& out, ActivationParam<T>& p) override {
        const size_t count = in[0]->storage_bytes() / type_length(in[0]->get_dtype());
        return static_cast<SaberStatus>(b200_activation_run(in[0]->get_dtype(), p.active, in[0]->data(),
                                                            out[0]->mutable_data(), count, p.negative_slope, p.coef,
                                                            this->_ctx->get_compute_stream()));
    }
};

template <typename T, DataType OpDtype>
class SaberScale : public ImplBase<ScaleParam<T>> {
public:
    typedef typename ImplBase<ScaleParam<T>>::TensorVec TensorVec;
    SaberStatus init(const TensorVec& in, TensorVec& out, ScaleParam<T>& p, Context<NV>& ctx) override {
        return create(in, out, p, ctx);
    }
    SaberStatus create(const TensorVec& in, TensorVec& out, ScaleParam<T>& p, Context<NV>& ctx) override;
    SaberStatus dispatch(const TensorVec& in, TensorVec& out, ScaleParam<T>& p) override {
        const size_t pixels = static_cast<size_t>(in[0]->num()) * in[0]->height() * in[0]->width();
        return static_cast<SaberStatus>(b200_scale_run(
            in[0]->get_dtype(), in[0]->data(), out[0]->mutable_data(), pixels, in[0]->channel_stored(),
            static_cast<const float*>(_w.ptr), p.bias_term ? static_cast<const float*>(_b.ptr) : nullptr,
            this->_ctx->get_compute_stream()));
    }

private:
    DeviceBuffer _w, _b;
};

template <typename T, DataType D>
SaberStatus SaberScale<T, D>::create(const TensorVec& in, TensorVec& out, ScaleParam<T>& p, Context<NV>& ctx) {
    this->_ctx = &ctx;
    if (p.axis != 1 || p.num_axes != 1) return SaberUnImplError;
    if (in[0]->get_layout() != Layout_NHWC) return SaberInvalidValue;
    const int cs = in[0]->channel_stored();
    std::vector<float> w(cs, 0.f), b(cs, 0.f);
    for (int i = 0; i < in[0]->channel() && i < static_cast<int>(p.scale_w.size()); ++i) w[i] = p.scale_w[i];
    for (int i = 0; i < in[0]->channel() && i < static_cast<int>(p.scale_b.size()); ++i) b[i] = p.scale_b[i];
    if (_w.re_alloc(cs * sizeof(float), false) != SaberSuccess) return SaberOutOfMem;
    if (_b.re_alloc(cs * sizeof(float), false) != SaberSuccess) return SaberOutOfMem;
    CUDA_CHECK(cudaMemcpy(_w.ptr, w.data(), cs * sizeof(float), cudaMemcpyHostToDevice));
    CUDA_CHECK(cudaMemcpy(_b.ptr, b.data(), cs * sizeof(float), cudaMemcpyHostToDevice));
    return SaberSuccess;
}

// ------------------------------------------------------------------------------------- funcs (front ends)
template <typename T, DataType D>
class Conv : public BaseFunc<SaberConv2D<T, D>, ConvParam<T>> {
public:
    typedef std::vector<Tensor<NV>*> V;
    SaberStatus compute_output_shape(const V& in, V& out, ConvParam<T>& p) override {
        Shape s = out[0]->valid_shape();
        s.set_num(in[0]->num());
        s.set_channel(p.weight_tensor->num());
        s.set_height(conv_out_size(in[0]->height(), p.pad_h, p.dilation_h, p.weight_tensor->height(), p.stride_h));
        s.set_width(conv_out_size(in[0]->width(), p.pad_w, p.dilation_w, p.weight_tensor->width(), p.stride_w));
        return out[0]->set_shape(s);
    }
};

template <typename T, DataType D>
class ConvEltwise : public BaseFunc<SaberConvEltwise<T, D>, ConvEltwiseParam<T>> {
public:
    typedef std::vector<Tensor<NV>*> V;
    SaberStatus compute_output_shape(const V& in, V& out, ConvEltwiseParam<T>& pe) override {
        ConvParam<T>& p = pe.conv_param;
        Shape s = out[0]->valid_shape();
        s.set_num(in[0]->num());
        s.set_channel(p.weight_tensor->num());
        s.set_height(conv_out_size(in[0]->height(), p.pad_h, p.dilation_h, p.weight_tensor->height(), p.stride_h));
        s.set_width(conv_out_size(in[0]->width(), p.pad_w, p.dilation_w, p.weight_tensor->width(), p.stride_w));
        return out[0]->set_shape(s);
    }
};

// Pooling output size: saber/funcs/pooling.h:69-132.
inline void pool_out_size(const PoolingParam<NV>& p, int in_h, int in_w, int* oh, int* ow) {
    b200_pool_desc_t d;
    memset(&d, 0, sizeof(d));
    d.h = in_h; d.w = in_w;
    d.window_h = p.window_h; d.window_w = p.window_w; d.pad_h = p.pad_h; d.pad_w = p.pad_w;
    d.stride_h = p.stride_h; d.stride_w = p.stride_w;
    d.global_pooling = p.global_pooling; d.floor_as_conv = p.cmp_out_shape_floor_as_conv;
    int32_t a = 1, b = 1;
    b200_pool_out_hw(&d, &a, &b);
    *oh = a; *ow = b;
}

template <typename T, DataType D>
class ConvPooling : public BaseFunc<SaberConv2DPooling<T, D>, ConvPoolingParam<T>> {
public:
    typedef std::vector<Tensor<NV>*> V;
    SaberStatus compute_output_shape(const V& in, V& out, ConvPoolingParam<T>& pp) override {
        ConvParam<T>& p = pp.conv_param;
        const int ch = conv_out_size(in[0]->height(), p.pad_h, p.dilation_h, p.weight_tensor->height(), p.stride_h);
        const int cw = conv_out_size(in[0]->width(), p.pad_w, p.dilation_w, p.weight_tensor->width(), p.stride_w);
        int oh, ow;
        pool_out_size(pp.pooling_param, ch, cw, &oh, &ow);
        Shape s = out[0]->valid_shape();
        s.set_num(in[0]->num());
        s.set_channel(p.weight_tensor->num());
        s.set_height(oh);
        s.set_width(ow);
        return out[0]->set_shape(s);
    }
};

template <typename T, DataType D>
class Fc : public BaseFunc<SaberFc<T, D>, FcParam<T>> {
public:
    typedef std::vector<Tensor<NV>*> V;
    SaberStatus compute_output_shape(const V& in, V& out, FcParam<T>& p) override {
        Shape s = out[0]->valid_shape();
        s.set_num(static_cast<int>(in[0]->count_valid(0, p.axis)));
        s.set_channel(p.num_output);
        s.set_height(1);
        s.set_width(1);
        return out[0]->set_shape(s);
    }
};

template <typename T, DataType D>
class Pooling : public BaseFunc<SaberPooling<T, D>, PoolingParam<T>> {
public:
    typedef std::vector<Tensor<NV>*> V;
    SaberStatus compute_output_shape(const V& in, V& out, PoolingParam<T>& p) override {
        int oh, ow;
        pool_out_size(p, in[0]->height(), in[0]->width(), &oh, &ow);
        Shape s = out[0]->valid_shape();
        s.set_num(in[0]->num());
        s.set_channel(in[0]->channel());
        s.set_height(oh);
        s.set_width(ow);
        return out[0]->set_shape(s);
    }
};

template <typename Impl, typename Param>
class SameShapeFunc : public BaseFunc<Impl, Param> {
public:
    typedef std::vector<Tensor<NV>*> V;
    SaberStatus compute_output_shape(const V& in, V& out, Param&) override {
        Shape s = in[0]->valid_shape();
        s.set_layout(out[0]->get_layout());
        return out[0]->set_shape(s);
    }
};
template <typename T, DataType D> class Softmax : public SameShapeFunc<SaberSoftmax<T, D>, SoftmaxParam<T>> {};
template <typename T, DataType D> class Eltwise : public SameShapeFunc<SaberEltwise<T, D>, EltwiseParam<T>> {};
template <typename T, DataType D> class Activation : public SameShapeFunc<SaberActivation<T, D>, ActivationParam<T>> {};
template <typename T, DataType D> class Scale : public SameShapeFunc<SaberScale<T, D>, ScaleParam<T>> {};

}  // namespace saber
}  // namespace anakin
