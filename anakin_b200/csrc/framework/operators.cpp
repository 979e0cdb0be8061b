// Operator implementations for the CNN classification path (22 operator names).
//   reference framework/operators/{convolution,dense,pooling,softmax,eltwise_op,relu,activation,
//             batch_norm,scale,input,output,split,flatten}.cpp and fusion_ops/{conv_relu,
//             conv_batchnorm_scale,conv_batchnorm_scale_relu,conv_batchnorm_scale_relu_pool,
//             conv_relu_pool,conv_eltwise,eltwise_relu}.cpp
#include "operators.h"

#include <map>
#include <mutex>

namespace anakin {
namespace ops {

using namespace saber;
using graph::Node;

#define GET_PARAMETER(type, name) (_node->get_attr<type>(#name))
// In Init() a failing Saber call is reported through Status (with node name and SaberStatus text)
// instead of aborting; operator() keeps the reference's SABER_CHECK abort.
#define SABER_INIT_CHECK(call)                                                                     \
    do {                                                                                           \
        ::anakin::saber::SaberStatus _s = static_cast<::anakin::saber::SaberStatus>(call);         \
        if (_s != ::anakin::saber::SaberSuccess)                                                   \
            return Status::ANAKINFAIL(std::string(#call) + " -> " + b200_status_string(_s) +      \
                                      " (node " + _node->name + ", op " + _node->op + ")");       \
    } while (0)

namespace {

PBlockPtr clone_block(const PBlockPtr& src) {
    PBlockPtr b = std::make_shared<PBlock>();
    const DataType dt = src->is_int8() ? AK_INT8 : AK_FLOAT;
    b->h.re_alloc(src->h.valid_shape(), dt);
    memcpy(b->h.mutable_data(), src->h.data(),
           static_cast<size_t>(src->h.valid_size()) * (dt == AK_INT8 ? 1 : sizeof(float)));
    b->h.set_scale(src->h.get_scale());
    return b;
}

PBlockPtr zero_block(int n) {
    PBlockPtr b = std::make_shared<PBlock>();
    b->h.re_alloc(Shape({1, n, 1, 1}), AK_FLOAT);
    memset(b->h.mutable_data(), 0, static_cast<size_t>(n) * sizeof(float));
    return b;
}

std::vector<float> block_vector(const PBlockPtr& b) {
    const float* p = b->data();
    return std::vector<float>(p, p + b->count());
}

// WeightsFusion<float>::update_weights, framework/utils/parameter_fusion.cpp:86-131:
//   f = bn_scale_factor==0 ? 1 : 1/bn_scale_factor
//   alpha = 1/sqrt(var*f + eps); beta = -(mean*f)*alpha; alpha *= gamma; beta = beta*gamma (+ beta_s)
//   w[i,:] *= alpha; b[i] = b[i]*alpha + beta
void fold_bn_scale(PBlock& w, PBlock& bias, int n, float bn_scale_factor, float eps, const std::vector<float>& mean,
                   const std::vector<float>& var, const std::vector<float>& scale_w, const std::vector<float>& scale_b,
                   bool scale_bias_term) {
    float* wp = w.mutable_data();
    float* bp = bias.mutable_data();
    const long long chw = w.count() / n;
    bn_scale_factor = (bn_scale_factor == 0) ? 1.f : 1.f / bn_scale_factor;
    for (int i = 0; i < n; ++i) {
        float alpha = var[i] * bn_scale_factor + eps;
        alpha = 1.f / sqrtf(alpha);
        float beta = -1.f * (mean[i] * bn_scale_factor);
        beta = beta * alpha;
        alpha = scale_w[i] * alpha;
        if (scale_bias_term) beta = beta * scale_w[i] + scale_b[i];
        else beta = beta * scale_w[i];
        for (long long j = 0; j < chw; ++j) wp[i * chw + j] *= alpha;
        bp[i] *= alpha;
        bp[i] += beta;
    }
}

// WeightsFusion<char>::update_weights, framework/utils/parameter_fusion.cpp:406-456: quantised weights keep their
// codes; the per-output-channel weight scale absorbs alpha (a negative alpha flips the channel's codes), the bias
// is updated as in the float case.
void fold_bn_scale_q8(PBlock& w, PBlock& bias, int n, float bn_scale_factor, float eps, const std::vector<float>& mean,
                      const std::vector<float>& var, const std::vector<float>& scale_w, const std::vector<float>& scale_b,
                      bool scale_bias_term) {
    int8_t* wp = w.mutable_data_q8();
    float* bp = bias.mutable_data();
    std::vector<float> w_scale = w.h.get_scale();
    if (static_cast<int>(w_scale.size()) < n) w_scale.resize(n, w_scale.empty() ? 1.f : w_scale.back());
    const long long chw = w.count() / n;
    bn_scale_factor = (bn_scale_factor == 0) ? 1.f : 1.f / bn_scale_factor;
    for (int i = 0; i < n; ++i) {
        float alpha = var[i] * bn_scale_factor + eps;
        alpha = 1.f / sqrtf(alpha);
        float beta = -1.f * (mean[i] * bn_scale_factor);
        beta = beta * alpha;
        alpha = scale_w[i] * alpha;
        if (scale_bias_term) beta = beta * scale_w[i] + scale_b[i];
        else beta = beta * scale_w[i];
        w_scale[i] *= alpha;
        if (w_scale[i] < 0) {
            w_scale[i] = fabsf(w_scale[i]);
            for (long long j = 0; j < chw; ++j) wp[i * chw + j] = static_cast<int8_t>(-wp[i * chw + j]);
        }
        bp[i] *= alpha;
        bp[i] += beta;
    }
    w.h.set_scale(w_scale);
}

// Folded weight / bias blocks are a function of the graph node alone: every Net built from one Graph (the
// per-thread Nets of a Worker, worker.cpp:10-53) shares them, and through them the packed device image
// (saber_funcs.cpp WeightArena) -- the role of the reference's process-wide GraphGlobalMem
// (framework/graph/graph_global_mem.h:78-250). Entries die with their last Net.
struct FoldedBlocks {
    PBlockPtr w, b;
    bool folded = false;   // BatchNorm / Scale already applied (by the first Net that used the node)
};
std::mutex g_fold_mu;
std::map<std::pair<const PBlock*, std::string>, std::weak_ptr<FoldedBlocks>> g_fold_cache;

PoolingParam<NV> parse_pooling(const Node& n, const std::string& pre) {
    auto pool_size = n.get_attr<PTuple<int>>(pre + "pool_size");
    auto strides = n.get_attr<PTuple<int>>(pre + "strides");
    auto padding = n.get_attr<PTuple<int>>(pre + "padding");
    auto method = n.get_attr<std::string>(pre + "method");
    bool global_pooling = n.get_attr_or<bool>(pre + "global_pooling", false);
    bool floor_as_conv = n.get_attr_or<bool>(pre + "cmp_out_shape_floor_as_conv", false);
    PoolingType t;
    if (method == "MAX") t = Pooling_max;
    else if (method == "AVG") t = Pooling_average_include_padding;
    else if (method == "AVGEXC") t = Pooling_average_exclude_padding;
    else { fprintf(stderr, "[FATAL] pooling method %s not supported\n", method.c_str()); abort(); }
    return PoolingParam<NV>(pool_size[0], pool_size[1], padding[0], padding[1], strides[0], strides[1], t,
                            global_pooling, floor_as_conv);
}

// ------------------------------------------------------------------ structural ops
class InputOp : public OperatorBase {
public:
    Status InitParam() override {
        _shape = GET_PARAMETER(PTuple<int>, input_shape);
        const int st = graph::node_image_format(*_node, &_image_desc);
        if (st < 0) return Status::ANAKINFAIL("malformed image input format on Input " + _node->name);
        _image = st == 1;
        return Status::OK();
    }
    Status InferShape(const TensorVec&, TensorVec& outs) override {
        // Input holds a user-facing fp32 NCHW tensor (input.cpp:17-40), or -- an image input -- the caller's 8-bit
        // interleaved images, normalised by the convolutions that read them
        std::vector<int> s = _shape;
        while (s.size() < 4) s.push_back(1);
        for (auto* o : outs) {
            if (_image) o->re_alloc_image(Shape(s, Layout_NHWC), _image_desc);
            else o->re_alloc(Shape(s, Layout_NCHW), AK_FLOAT);
        }
        return Status::OK();
    }
    Status Init(OpContext<NV>&, const TensorVec&, TensorVec&) override { return Status::OK(); }
    void operator()(OpContext<NV>&, const TensorVec&, TensorVec&) override {}
    bool is_alias() const override { return true; }

private:
    PTuple<int> _shape;
    bool _image = false;
    b200_image_desc_t _image_desc{};
};

class AliasOp : public OperatorBase {  // Output, Split, Flatten: zero-copy bookkeeping (split.cpp, output.cpp)
public:
    Status InitParam() override { return Status::OK(); }
    Status InferShape(const TensorVec&, TensorVec&) override { return Status::OK(); }
    Status Init(OpContext<NV>&, const TensorVec&, TensorVec&) override { return Status::OK(); }
    void operator()(OpContext<NV>&, const TensorVec&, TensorVec&) override {}
    bool is_alias() const override { return true; }
    int output_signedness() const override { return -1; }
};

// ------------------------------------------------------------------ conv family
template <DataType D>
class ConvFamilyOp : public OperatorBase {
public:
    Status InitParam() override {
        const Node& n = *_node;
        std::string flavour = n.op;
        _is_eltwise = n.op == "ConvEltwise";
        if (_is_eltwise) flavour = n.get_attr_or<std::string>("conv_eltwise_base_op", "Convolution");
        const bool has_bn = flavour.find("Batchnorm") != std::string::npos;
        const bool has_scale = flavour.find("Scale") != std::string::npos;
        const bool has_relu = flavour.find("Relu") != std::string::npos;
        _has_pool = flavour.find("Pool") != std::string::npos;

        auto group = GET_PARAMETER(int, group);
        auto bias_term = GET_PARAMETER(bool, bias_term);
        auto padding = GET_PARAMETER(PTuple<int>, padding);
        auto strides = GET_PARAMETER(PTuple<int>, strides);
        auto dilation_rate = GET_PARAMETER(PTuple<int>, dilation_rate);
        auto filter_num = GET_PARAMETER(int, filter_num);
        auto weights = GET_PARAMETER(PBlockPtr, weight_1);
        if (weights->h.num() != filter_num) return Status::ANAKINFAIL("weight_1 shape does not match filter_num");

        // folded copies, one per graph node: the graph's blocks stay pristine, and every Net built from this
        // Graph (Worker threads, multi-GPU replicas) shares the same folded host blocks (SURVEY.md app. C.5)
        _has_bias = bias_term || has_bn || has_scale;
        std::lock_guard<std::mutex> fold_lock(g_fold_mu);
        const auto fold_key = std::make_pair(static_cast<const PBlock*>(weights.get()), n.name);
        if (auto hit = g_fold_cache[fold_key].lock()) {
            _folded = hit;
        } else {
            _folded = std::make_shared<FoldedBlocks>();
            _folded->w = clone_block(weights);
            _folded->b = bias_term ? clone_block(GET_PARAMETER(PBlockPtr, weight_2)) : zero_block(filter_num);
            g_fold_cache[fold_key] = _folded;
        }
        _w = _folded->w;
        _b = _folded->b;
        if ((has_bn || has_scale) && !_folded_done()) {
            std::vector<float> mean(filter_num, 0.f), var(filter_num, 1.f), gamma(filter_num, 1.f), beta_s(filter_num, 0.f);
            float factor = 1.f, eps = 0.f;
            bool scale_bias = false;
            if (has_bn) {
                eps = GET_PARAMETER(float, batchnorm_0_epsilon);
                mean = block_vector(GET_PARAMETER(PBlockPtr, batchnorm_0_weight_1));
                var = block_vector(GET_PARAMETER(PBlockPtr, batchnorm_0_weight_2));
                factor = block_vector(GET_PARAMETER(PBlockPtr, batchnorm_0_weight_3))[0];
            } else {
                // conv + scale only: alpha = gamma, beta = beta_s (var=1, eps=0, mean=0)
                eps = 0.f;
            }
            if (has_scale) {
                scale_bias = GET_PARAMETER(bool, scale_0_bias_term);
                gamma = block_vector(GET_PARAMETER(PBlockPtr, scale_0_weight_1));
                if (scale_bias) beta_s = block_vector(GET_PARAMETER(PBlockPtr, scale_0_weight_2));
            }
            if (static_cast<int>(mean.size()) < filter_num || static_cast<int>(var.size()) < filter_num ||
                static_cast<int>(gamma.size()) < filter_num)
                return Status::ANAKINFAIL("batchnorm/scale parameter size mismatch in " + n.name);
            if (_w->is_int8()) fold_bn_scale_q8(*_w, *_b, filter_num, factor, eps, mean, var, gamma, beta_s, scale_bias);
            else fold_bn_scale(*_w, *_b, filter_num, factor, eps, mean, var, gamma, beta_s, scale_bias);
        }
        _folded->folded = true;
        ActivationParam<NV> act;
        if (has_relu) act = ActivationParam<NV>(Active_relu, n.get_attr_or<float>("relu_0_alpha", 0.f));
        _relu_out = has_relu;
        _conv = ConvParam<NV>(group, padding[0], padding[1], strides[0], strides[1], dilation_rate[0],
                              dilation_rate[1], &_w->h, _has_bias ? &_b->h : nullptr, act);
        if (_is_eltwise) {
            if (!n.has("merge_type")) return Status::ANAKINFAIL("ConvEltwise Op must have been merged eltwise");
            auto type = GET_PARAMETER(std::string, merge_type);
            auto coeff = n.get_attr_or<PTuple<float>>("merge_coeff", {1.f, 1.f});
            EltwiseType et = type == "Add" ? Eltwise_sum : (type == "Max" ? Eltwise_max : Eltwise_prod);
            if (n.has("merge_relu_0_alpha")) {
                ActivationParam<NV> a(Active_relu, n.get_attr_or<float>("merge_relu_0_alpha", 0.f));
                _elt = EltwiseParam<NV>(et, coeff, a);
                _relu_out = true;
            } else {
                _elt = EltwiseParam<NV>(et, coeff);
            }
            _conv_elt = ConvEltwiseParam<NV>(_conv, _elt);
        } else if (_has_pool) {
            _pool = parse_pooling(n, "pooling_0_");
            _conv_pool = ConvPoolingParam<NV>(_conv, _pool);
        }
        return Status::OK();
    }

    Status InferShape(const TensorVec& ins, TensorVec& outs) override {
        SaberStatus st;
        if (_is_eltwise) st = _f_elt.compute_output_shape(ins, outs, _conv_elt);
        else if (_has_pool) st = _f_pool.compute_output_shape(ins, outs, _conv_pool);
        else st = _f_conv.compute_output_shape(ins, outs, _conv);
        return st == SaberSuccess ? Status::OK() : Status::ANAKINFAIL("conv InferShape failed");
    }

    Status Init(OpContext<NV>& ctx, const TensorVec& ins, TensorVec& outs) override {
        if (_is_eltwise) {
            if (ins.size() < 2) return Status::ANAKINFAIL("ConvEltwise needs the residual as second input");
            // beta = scale of the residual edge, beta_type its dtype (fusion_ops/conv_eltwise.cpp:182-188)
            _conv_elt.conv_param.beta = ins[1]->get_scale().empty() ? 1.f : ins[1]->get_scale()[0];
            _conv_elt.conv_param.beta_type = ins[1]->get_dtype();
            SABER_INIT_CHECK(_f_elt.init(ins, outs, _conv_elt, SPECIFY, SABER_IMPL, ctx));
        } else if (_has_pool) {
            SABER_INIT_CHECK(_f_pool.init(ins, outs, _conv_pool, SPECIFY, SABER_IMPL, ctx));
        } else {
            SABER_INIT_CHECK(_f_conv.init(ins, outs, _conv, SPECIFY, SABER_IMPL, ctx));
        }
        return Status::OK();
    }

    void operator()(OpContext<NV>& ctx, const TensorVec& ins, TensorVec& outs) override {
        TensorVec o = outs;
        if (_is_eltwise) SABER_CHECK(_f_elt(ins, o, _conv_elt, ctx));
        else if (_has_pool) SABER_CHECK(_f_pool(ins, o, _conv_pool, ctx));
        else SABER_CHECK(_f_conv(ins, o, _conv, ctx));
    }
    int output_signedness() const override { return _relu_out ? 1 : 0; }
    const void* weight_device_ptr() const override {
        if (_is_eltwise) return const_cast<saber::ConvEltwise<NV, D>&>(_f_elt).impl().engine().weight_device_ptr();
        if (_has_pool) return const_cast<saber::ConvPooling<NV, D>&>(_f_pool).impl().engine().weight_device_ptr();
        return const_cast<saber::Conv<NV, D>&>(_f_conv).impl().engine().weight_device_ptr();
    }

private:
    bool _folded_done() const { return _folded && _folded->folded; }
    bool _is_eltwise = false, _has_pool = false, _has_bias = false, _relu_out = false;
    std::shared_ptr<FoldedBlocks> _folded;
    PBlockPtr _w, _b;
    ConvParam<NV> _conv;
    EltwiseParam<NV> _elt;
    PoolingParam<NV> _pool;
    ConvEltwiseParam<NV> _conv_elt;
    ConvPoolingParam<NV> _conv_pool;
    saber::Conv<NV, D> _f_conv;
    saber::ConvEltwise<NV, D> _f_elt;
    saber::ConvPooling<NV, D> _f_pool;
};

// ------------------------------------------------------------------ dense (dense.cpp:20-90)
template <DataType D>
class DenseOp : public OperatorBase {
public:
    Status InitParam() override {
        auto axis = GET_PARAMETER(int, axis);
        auto out_dim = _node->get_attr_or<int>("out_dim", 0);
        auto bias_term = GET_PARAMETER(bool, bias_term);
        _w = GET_PARAMETER(PBlockPtr, weight_1);
        _b = bias_term ? GET_PARAMETER(PBlockPtr, weight_2) : nullptr;
        _param = FcParam<NV>(&_w->h, _b ? &_b->h : nullptr, out_dim, axis);
        return Status::OK();
    }
    Status InferShape(const TensorVec& ins, TensorVec& outs) override {
        return _f.compute_output_shape(ins, outs, _param) == SaberSuccess ? Status::OK()
                                                                            : Status::ANAKINFAIL("Dense InferShape");
    }
    Status Init(OpContext<NV>& ctx, const TensorVec& ins, TensorVec& outs) override {
        SABER_INIT_CHECK(_f.init(ins, outs, _param, SPECIFY, SABER_IMPL, ctx));
        return Status::OK();
    }
    void operator()(OpContext<NV>& ctx, const TensorVec& ins, TensorVec& outs) override {
        TensorVec o = outs;
        SABER_CHECK(_f(ins, o, _param, ctx));
    }
    const void* weight_device_ptr() const override {
        return const_cast<saber::Fc<NV, D>&>(_f).impl().engine().weight_device_ptr();
    }
    bool head_fc_info(b200_fc_stream_desc_t* d, const void** w, const float** bias, const float** scale) const override {
        if (_param.activation_param.has_active) return false;
        return const_cast<saber::Fc<NV, D>&>(_f).impl().engine().fc_stream_info(d, w, bias, scale);
    }

private:
    PBlockPtr _w, _b;
    FcParam<NV> _param;
    saber::Fc<NV, D> _f;
};

// ------------------------------------------------------------------ pointwise ops
template <typename Func, typename Param>
class SimpleOp : public OperatorBase {
public:
    Status InferShape(const TensorVec& ins, TensorVec& outs) override {
        return _f.compute_output_shape(ins, outs, _param) == SaberSuccess ? Status::OK()
                                                                            : Status::ANAKINFAIL("InferShape failed");
    }
    Status Init(OpContext<NV>& ctx, const TensorVec& ins, TensorVec& outs) override {
        SABER_INIT_CHECK(_f.init(ins, outs, _param, SPECIFY, SABER_IMPL, ctx));
        return Status::OK();
    }
    void operator()(OpContext<NV>& ctx, const TensorVec& ins, TensorVec& outs) override {
        TensorVec o = outs;
        SABER_CHECK(_f(ins, o, _param, ctx));
    }

protected:
    Param _param;
    Func _f;
};

class PoolingOp : public SimpleOp<saber::Pooling<NV, AK_FLOAT>, PoolingParam<NV>> {
public:
    Status InitParam() override { _param = parse_pooling(*_node, ""); return Status::OK(); }
    int output_signedness() const override { return -1; }
    bool head_pool_info(int* is_max) const override {
        if (!_param.global_pooling || _param.pad_h != 0 || _param.pad_w != 0) return false;
        *is_max = _param.pooling_type == Pooling_max ? 1 : 0;
        return true;
    }
};

class SoftmaxOp : public SimpleOp<saber::Softmax<NV, AK_FLOAT>, SoftmaxParam<NV>> {
public:
    Status InitParam() override { _param = SoftmaxParam<NV>(GET_PARAMETER(int, axis)); return Status::OK(); }
    bool head_softmax_info(int* axis) const override { *axis = _param.axis; return true; }
};

class EltwiseOp : public SimpleOp<saber::Eltwise<NV, AK_FLOAT>, EltwiseParam<NV>> {
public:
    Status InitParam() override {
        auto type = GET_PARAMETER(std::string, type);
        auto coeff = _node->get_attr_or<PTuple<float>>("coeff", {1.f, 1.f});
        EltwiseType et;
        if (type == "Add") et = Eltwise_sum;
        else if (type == "Max") et = Eltwise_max;
        else et = Eltwise_prod;
        if (coeff.empty()) coeff = {1.f, 1.f};
        if (_node->op == "EltwiseRelu") {
            ActivationParam<NV> a(Active_relu, _node->get_attr_or<float>("relu_0_alpha", 0.f));
            _param = EltwiseParam<NV>(et, coeff, a);
            _relu = true;
        } else {
            _param = EltwiseParam<NV>(et, coeff);
        }
        return Status::OK();
    }
    int output_signedness() const override { return _relu ? 1 : 0; }

private:
    bool _relu = false;
};

class ActivationOp : public SimpleOp<saber::Activation<NV, AK_FLOAT>, ActivationParam<NV>> {
public:
    Status InitParam() override {
        if (_node->op == "ReLU") {
            _param = ActivationParam<NV>(Active_relu, GET_PARAMETER(float, alpha));
            _relu = true;
        } else {
            auto type = GET_PARAMETER(std::string, type);
            if (type == "TanH") _param = ActivationParam<NV>(Active_tanh);
            else if (type == "Sigmoid") _param = ActivationParam<NV>(Active_sigmoid);
            else if (type == "ClippedRelu") _param = ActivationParam<NV>(Active_clipped_relu, 0.f, _node->get_attr_or<float>("clip_relu_num", 0.f));
            else return Status::ANAKINFAIL("activation type " + type + " not supported");
        }
        return Status::OK();
    }
    int output_signedness() const override { return _relu ? 1 : 0; }

private:
    bool _relu = false;
};

// un-fused BatchNorm / Scale: y = x*w[c] + b[c] (batch_norm.cpp:36-60, scale.cpp:41-60)
class ScaleLikeOp : public SimpleOp<saber::Scale<NV, AK_FLOAT>, ScaleParam<NV>> {
public:
    Status InitParam() override {
        if (_node->op == "BatchNorm") {
            auto eps = GET_PARAMETER(float, epsilon);
            auto mean = block_vector(GET_PARAMETER(PBlockPtr, weight_1));
            auto var = block_vector(GET_PARAMETER(PBlockPtr, weight_2));
            float factor = block_vector(GET_PARAMETER(PBlockPtr, weight_3))[0];
            factor = factor == 0 ? 1.f : 1.f / factor;
            std::vector<float> w(mean.size()), b(mean.size());
            for (size_t i = 0; i < mean.size(); ++i) {
                float alpha = 1.f / sqrtf(var[i] * factor + eps);
                w[i] = alpha;
                b[i] = -1.f * (mean[i] * factor) * alpha;
            }
            _param = ScaleParam<NV>(w, b, true, 1, 1);
        } else {
            auto bias_term = GET_PARAMETER(bool, bias_term);
            auto w = block_vector(GET_PARAMETER(PBlockPtr, weight_1));
            std::vector<float> b;
            if (bias_term) b = block_vector(GET_PARAMETER(PBlockPtr, weight_2));
            _param = ScaleParam<NV>(w, b, bias_term, GET_PARAMETER(int, axis), GET_PARAMETER(int, num_axes));
        }
        return Status::OK();
    }
};

template <typename OpT>
OperatorBase* make() { return new OpT(); }

}  // namespace

namespace {
const char* const kConvNames[] = {"Convolution", "ConvRelu", "ConvBatchnorm", "ConvBatchnormScale",
                                  "ConvBatchnormScaleRelu", "ConvScale", "ConvScaleRelu", "ConvEltwise",
                                  "ConvReluPool", "ConvBatchnormScaleReluPool"};
}  // namespace

bool is_conv_family(const std::string& op_name) {
    for (const char* nm : kConvNames)
        if (op_name == nm) return true;
    return false;
}

void register_all_operators() {
    static std::once_flag once;
    std::call_once(once, [] {
        auto& f32 = OpFactory<NV, Precision::FP32>::Global();
        auto& f16 = OpFactory<NV, Precision::FP16>::Global();
        auto& i8 = OpFactory<NV, Precision::INT8>::Global();
        for (const char* nm : kConvNames) {
            f32.Register(nm, make<ConvFamilyOp<AK_FLOAT>>);
            f16.Register(nm, make<ConvFamilyOp<AK_HALF>>);
            i8.Register(nm, make<ConvFamilyOp<AK_INT8>>);
        }
        f32.Register("Dense", make<DenseOp<AK_FLOAT>>);
        f16.Register("Dense", make<DenseOp<AK_HALF>>);
        i8.Register("Dense", make<DenseOp<AK_INT8>>);
        // precision-agnostic ops: the kernels key on the tensor dtype
        for (OpFactoryCore* f : {static_cast<OpFactoryCore*>(&f32), static_cast<OpFactoryCore*>(&f16),
                                 static_cast<OpFactoryCore*>(&i8)}) {
            f->Register("Input", make<InputOp>);
            f->Register("Output", make<AliasOp>);
            f->Register("Split", make<AliasOp>);
            f->Register("Gather", make<AliasOp>);   // framework/operators/gather.cpp: launches nothing
            f->Register("Pooling", make<PoolingOp>);
            f->Register("Eltwise", make<EltwiseOp>);
            f->Register("EltwiseRelu", make<EltwiseOp>);
        }
        for (OpFactoryCore* f : {static_cast<OpFactoryCore*>(&f32), static_cast<OpFactoryCore*>(&f16)}) {
            f->Register("Softmax", make<SoftmaxOp>);
            f->Register("ReLU", make<ActivationOp>);
            f->Register("Activation", make<ActivationOp>);
            f->Register("BatchNorm", make<ScaleLikeOp>);
            f->Register("Scale", make<ScaleLikeOp>);
            f->Register("Flatten", make<AliasOp>);
        }
    });
}

OperatorBase* create_operator(const std::string& op_name, Precision p) {
    register_all_operators();
    OperatorBase* op = nullptr;
    switch (p) {
        case Precision::INT8: op = OpFactory<NV, Precision::INT8>::Global()[op_name]; break;
        case Precision::FP16: op = OpFactory<NV, Precision::FP16>::Global()[op_name]; break;
        default: op = OpFactory<NV, Precision::FP32>::Global()[op_name]; break;
    }
    return op;
}

}  // namespace ops
}  // namespace anakin
