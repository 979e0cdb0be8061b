// Operator implementations for the CNN classification path (27 operator names, listed in kOps).
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
#define SABER_INIT_CHECK(call)                                                             \
    do {                                                                                   \
        ::anakin::saber::SaberStatus _s = static_cast<::anakin::saber::SaberStatus>(call); \
        if (_s != ::anakin::saber::SaberSuccess) return init_fail(*_node, #call, _s);      \
    } while (0)

namespace {

typedef OperatorBase::TensorVec TensorVec;

// Init's failure of node n: what failed, the SaberStatus text, the node and its op
Status init_fail(const Node& n, const std::string& what, SaberStatus st) {
    return Status::ANAKINFAIL(what + " -> " + b200_status_string(st) + " (node " + n.name + ", op " + n.op + ")");
}

// The last step of every InferShape: the output takes shape s (and storage for it).
Status set_out_shape(Tensor<NV>& out, const Shape& s) {
    return out.set_shape(s) == SaberSuccess ? Status::OK() : Status::ANAKINFAIL("cannot allocate the output");
}

// The output of an op that keeps its input's shape: in[0]'s dims in out[0]'s layout.
Status infer_same_shape(const TensorVec& ins, TensorVec& outs) {
    Shape s = ins[0]->valid_shape();
    s.set_layout(outs[0]->get_layout());
    return set_out_shape(*outs[0], s);
}

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

b200_pool_desc_t parse_pooling(const Node& n, const std::string& pre) {
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
    b200_pool_desc_t d{};
    d.type = t;
    d.window_h = pool_size[0]; d.window_w = pool_size[1];
    d.pad_h = padding[0]; d.pad_w = padding[1];
    d.stride_h = strides[0]; d.stride_w = strides[1];
    d.global_pooling = global_pooling ? 1 : 0;
    d.floor_as_conv = floor_as_conv ? 1 : 0;
    return d;
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
        const bool has_bias = bias_term || has_bn || has_scale;
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
        if ((has_bn || has_scale) && !_folded->folded) {
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

        const Tensor<NVHX86>& w = _w->h;
        _spec.op_dtype = D;
        _spec.weights = &w;
        _spec.bias = has_bias ? &_b->h : nullptr;
        _spec.k = w.num(); _spec.c_per_group = w.channel(); _spec.r = w.height(); _spec.s = w.width();
        _spec.group = group;
        _spec.pad_h = padding[0]; _spec.pad_w = padding[1];
        _spec.stride_h = strides[0]; _spec.stride_w = strides[1];
        _spec.dil_h = dilation_rate[0]; _spec.dil_w = dilation_rate[1];
        _spec.relu = has_relu;
        _spec.neg_slope = has_relu ? n.get_attr_or<float>("relu_0_alpha", 0.f) : 0.f;
        if (_is_eltwise) {
            if (!n.has("merge_type")) return Status::ANAKINFAIL("ConvEltwise Op must have been merged eltwise");
            _merge_add = GET_PARAMETER(std::string, merge_type) == "Add";
            // the activation after the sum replaces the conv's own (conv_eltwise.cpp:154-176)
            if (n.has("merge_relu_0_alpha")) {
                _spec.relu = true;
                _spec.neg_slope = n.get_attr_or<float>("merge_relu_0_alpha", 0.f);
            }
        } else if (flavour.find("Pool") != std::string::npos) {
            _spec.has_pool = true;
            _spec.pool = parse_pooling(n, "pooling_0_");
        }
        return Status::OK();
    }

    Status InferShape(const TensorVec& ins, TensorVec& outs) override {
        const Tensor<NV>& in = *ins[0];
        Shape s = outs[0]->valid_shape();
        s.set_num(in.num());
        s.set_channel(_spec.k);
        s.set_height(conv_out_size(in.height(), _spec.pad_h, _spec.dil_h, _spec.r, _spec.stride_h));
        s.set_width(conv_out_size(in.width(), _spec.pad_w, _spec.dil_w, _spec.s, _spec.stride_w));
        if (_spec.has_pool) {
            int oh, ow;
            pool_out_size(_spec.pool, s.height(), s.width(), &oh, &ow);
            s.set_height(oh);
            s.set_width(ow);
        }
        return set_out_shape(*outs[0], s);
    }

    Status Init(OpContext<NV>& ctx, const TensorVec& ins, TensorVec& outs) override {
        if (_is_eltwise) {
            if (ins.size() < 2) return Status::ANAKINFAIL("ConvEltwise needs the residual as second input");
            if (!_merge_add) return init_fail(*_node, "ConvEltwise fuses only an Add", SaberUnImplError);
            // the residual edge's scale (fusion_ops/conv_eltwise.cpp:182-188)
            _spec.residual_scale = ins[1]->get_scale().empty() ? 1.f : ins[1]->get_scale()[0];
        }
        SABER_INIT_CHECK(_eng.prepare(_spec, *ins[0], residual(ins), *outs[0], ctx));
        return Status::OK();
    }

    void operator()(OpContext<NV>& ctx, const TensorVec& ins, TensorVec& outs) override {
        SABER_CHECK(_eng.run(*ins[0], residual(ins), *outs[0], ctx.get_compute_stream()));
    }
    int output_signedness() const override { return _spec.relu ? 1 : 0; }
    const void* weight_device_ptr() const override { return _eng.weight_device_ptr(); }

private:
    const Tensor<NV>* residual(const TensorVec& ins) const { return _is_eltwise ? ins[1] : nullptr; }
    bool _is_eltwise = false, _merge_add = false;
    std::shared_ptr<FoldedBlocks> _folded;
    PBlockPtr _w, _b;
    ConvEngine::Spec _spec;
    ConvEngine _eng;
};

// ------------------------------------------------------------------ dense (dense.cpp:20-90)
// out[m][n] = in[m][k] * W[n][k]^T + b (saber_fc.cu:17-195) on the conv family's engine
template <DataType D>
class DenseOp : public OperatorBase {
public:
    Status InitParam() override {
        _axis = GET_PARAMETER(int, axis);
        auto bias_term = GET_PARAMETER(bool, bias_term);
        _w = GET_PARAMETER(PBlockPtr, weight_1);
        _b = bias_term ? GET_PARAMETER(PBlockPtr, weight_2) : nullptr;
        _spec.op_dtype = D;
        _spec.weights = &_w->h;
        _spec.bias = _b ? &_b->h : nullptr;
        _spec.k = _node->get_attr_or<int>("out_dim", 0);
        _spec.is_fc = true;
        return Status::OK();
    }
    Status InferShape(const TensorVec& ins, TensorVec& outs) override {
        Shape s = outs[0]->valid_shape();
        s.set_num(static_cast<int>(ins[0]->count_valid(0, _axis)));
        s.set_channel(_spec.k);
        s.set_height(1);
        s.set_width(1);
        return set_out_shape(*outs[0], s);
    }
    Status Init(OpContext<NV>& ctx, const TensorVec& ins, TensorVec& outs) override {
        _spec.c_per_group = static_cast<int>(ins[0]->count_valid(_axis, 4));
        SABER_INIT_CHECK(_eng.prepare(_spec, *ins[0], nullptr, *outs[0], ctx));
        return Status::OK();
    }
    void operator()(OpContext<NV>& ctx, const TensorVec& ins, TensorVec& outs) override {
        SABER_CHECK(_eng.run(*ins[0], nullptr, *outs[0], ctx.get_compute_stream()));
    }
    const void* weight_device_ptr() const override { return _eng.weight_device_ptr(); }
    bool head_fc_info(b200_fc_stream_desc_t* d, const void** w, const float** bias, const float** scale) const override {
        return _eng.fc_stream_info(d, w, bias, scale);
    }

private:
    int _axis = 1;
    PBlockPtr _w, _b;
    ConvEngine::Spec _spec;
    ConvEngine _eng;
};

// ------------------------------------------------------------------ pointwise ops
class PoolingOp : public OperatorBase {
public:
    Status InitParam() override { _d = parse_pooling(*_node, ""); return Status::OK(); }
    Status InferShape(const TensorVec& ins, TensorVec& outs) override {
        int oh, ow;
        pool_out_size(_d, ins[0]->height(), ins[0]->width(), &oh, &ow);
        Shape s = outs[0]->valid_shape();
        s.set_num(ins[0]->num());
        s.set_channel(ins[0]->channel());
        s.set_height(oh);
        s.set_width(ow);
        return set_out_shape(*outs[0], s);
    }
    Status Init(OpContext<NV>&, const TensorVec& ins, TensorVec& outs) override {
        if (ins[0]->get_layout() != Layout_NHWC || outs[0]->get_layout() != Layout_NHWC)
            return init_fail(*_node, "Pooling needs NHWC tensors", SaberInvalidValue);
        if (ins[0]->get_dtype() != outs[0]->get_dtype())
            return init_fail(*_node, "Pooling keeps its input's dtype", SaberInvalidValue);
        // int8 pooling passes its input scale through (reference x86 saber_pooling.cpp:583-584)
        outs[0]->set_scale(ins[0]->get_scale());
        _d = make_pool_desc(*ins[0], _d);
        return Status::OK();
    }
    void operator()(OpContext<NV>& ctx, const TensorVec& ins, TensorVec& outs) override {
        SABER_CHECK(b200_pool_run(&_d, ins[0]->data(), outs[0]->mutable_data(), ctx.get_compute_stream()));
    }
    int output_signedness() const override { return -1; }
    bool head_pool_info(int* is_max) const override {
        if (!_d.global_pooling || _d.pad_h != 0 || _d.pad_w != 0) return false;
        *is_max = _d.type == Pooling_max ? 1 : 0;
        return true;
    }

private:
    b200_pool_desc_t _d{};   // the node's pooling; Init fills in the input's fields
};

class SoftmaxOp : public OperatorBase {
public:
    Status InitParam() override { _axis = GET_PARAMETER(int, axis); return Status::OK(); }
    Status InferShape(const TensorVec& ins, TensorVec& outs) override { return infer_same_shape(ins, outs); }
    Status Init(OpContext<NV>&, const TensorVec& ins, TensorVec& outs) override {
        const Tensor<NV>& x = *ins[0];
        if (x.get_dtype() != AK_FLOAT || outs[0]->get_dtype() != AK_FLOAT)
            return init_fail(*_node, "Softmax runs on fp32 tensors", SaberUnImplError);
        // logical NCHW axes -> (outer, axis, inner) of the stored layout
        const bool flat = x.height() == 1 && x.width() == 1;
        if (_axis == 1 && (flat || x.get_layout() == Layout_NHWC)) {
            // channels are innermost: one row per pixel, row pitch = stored (padded) channels
            _outer = x.num() * x.height() * x.width();
            _len = x.channel();
            _inner = 1;
            _in_pitch = x.channel_stored();
            _out_pitch = outs[0]->channel_stored();
        } else if (x.get_layout() == Layout_NCHW) {
            _outer = static_cast<int>(x.count_valid(0, _axis));
            _len = x.valid_shape()[_axis];
            _inner = static_cast<int>(x.count_valid(_axis + 1, 4));
        } else {
            return init_fail(*_node, "Softmax over axis " + std::to_string(_axis) + " of this layout", SaberUnImplError);
        }
        return Status::OK();
    }
    void operator()(OpContext<NV>& ctx, const TensorVec& ins, TensorVec& outs) override {
        const float* x = static_cast<const float*>(ins[0]->data());
        float* y = static_cast<float*>(outs[0]->mutable_data());
        if (_in_pitch) SABER_CHECK(b200_softmax_rows(x, y, _outer, _len, _in_pitch, _out_pitch, ctx.get_compute_stream()));
        else SABER_CHECK(b200_softmax_run(x, y, _outer, _len, _inner, ctx.get_compute_stream()));
    }
    bool head_softmax_info(int* axis) const override { *axis = _axis; return true; }

private:
    int _axis = 1;
    int _outer = 0, _len = 0, _inner = 1, _in_pitch = 0, _out_pitch = 0;
};

class EltwiseOp : public OperatorBase {
public:
    Status InitParam() override {
        auto type = GET_PARAMETER(std::string, type);
        auto coeff = _node->get_attr_or<PTuple<float>>("coeff", {1.f, 1.f});
        if (type == "Add") _op = Eltwise_sum;
        else if (type == "Max") _op = Eltwise_max;
        else _op = Eltwise_prod;
        _c0 = coeff.size() > 0 ? coeff[0] : 1.f;
        _c1 = coeff.size() > 1 ? coeff[1] : 1.f;
        _relu = _node->op == "EltwiseRelu";
        return Status::OK();
    }
    Status InferShape(const TensorVec& ins, TensorVec& outs) override { return infer_same_shape(ins, outs); }
    Status Init(OpContext<NV>&, const TensorVec& ins, TensorVec& outs) override {
        if (ins.size() != 2) return init_fail(*_node, "Eltwise takes 2 inputs", SaberUnImplError);
        if (ins[0]->storage_bytes() != ins[1]->storage_bytes())
            return init_fail(*_node, "Eltwise inputs differ in size", SaberInvalidValue);
        const Tensor<NV>& a = *ins[0];
        const Tensor<NV>& b = *ins[1];
        const Tensor<NV>& o = *outs[0];
        auto q8 = [](DataType d) { return d == AK_INT8 || d == AK_UINT8; };
        if (q8(a.get_dtype())) {
            // x86 int8 eltwise (saber_eltwise.cpp:72-111): tmp = sum coeff*code*scale, rescaled to
            // the output code space; u8 tensors carry scale*127/255.
            if (!q8(b.get_dtype()) || !q8(o.get_dtype()) || a.get_scale().empty() || b.get_scale().empty() ||
                o.get_scale().empty())
                return init_fail(*_node, "8-bit Eltwise needs 8-bit operands with calibrated scales", SaberInvalidValue);
            const float u = 127.f / 255.f;
            const float f0 = a.get_scale()[0] * (a.get_dtype() == AK_UINT8 ? u : 1.f);
            const float f1 = b.get_scale()[0] * (b.get_dtype() == AK_UINT8 ? u : 1.f);
            const float fo = o.get_scale()[0] * (o.get_dtype() == AK_UINT8 ? u : 1.f);
            _c0 = _c0 * (f0 / fo);
            _c1 = _c1 * (f1 / fo);
        }
        return Status::OK();
    }
    void operator()(OpContext<NV>& ctx, const TensorVec& ins, TensorVec& outs) override {
        const size_t count = ins[0]->storage_bytes() / type_length(ins[0]->get_dtype());
        SABER_CHECK(b200_eltwise_run(ins[0]->get_dtype(), ins[1]->get_dtype(), outs[0]->get_dtype(), _op, ins[0]->data(),
                                     ins[1]->data(), outs[0]->mutable_data(), count, _c0, _c1, _relu ? 1 : 0,
                                     ctx.get_compute_stream()));
    }
    int output_signedness() const override { return _relu ? 1 : 0; }

private:
    EltwiseType _op = Eltwise_sum;
    float _c0 = 1.f, _c1 = 1.f;   // the node's coefficients; an 8-bit Init folds the operand scales in
    bool _relu = false;
};

class ActivationOp : public OperatorBase {
public:
    Status InitParam() override {
        if (_node->op == "ReLU") {
            _act = Active_relu;
            _slope = GET_PARAMETER(float, alpha);
        } else {
            auto type = GET_PARAMETER(std::string, type);
            if (type == "TanH") _act = Active_tanh;
            else if (type == "Sigmoid") _act = Active_sigmoid;
            else if (type == "ClippedRelu") { _act = Active_clipped_relu; _coef = _node->get_attr_or<float>("clip_relu_num", 0.f); }
            else return Status::ANAKINFAIL("activation type " + type + " not supported");
        }
        return Status::OK();
    }
    Status InferShape(const TensorVec& ins, TensorVec& outs) override { return infer_same_shape(ins, outs); }
    Status Init(OpContext<NV>&, const TensorVec&, TensorVec&) override { return Status::OK(); }
    void operator()(OpContext<NV>& ctx, const TensorVec& ins, TensorVec& outs) override {
        const size_t count = ins[0]->storage_bytes() / type_length(ins[0]->get_dtype());
        SABER_CHECK(b200_activation_run(ins[0]->get_dtype(), _act, ins[0]->data(), outs[0]->mutable_data(), count, _slope,
                                        _coef, ctx.get_compute_stream()));
    }
    int output_signedness() const override { return _act == Active_relu ? 1 : 0; }

private:
    ActiveType _act = Active_unknow;
    float _slope = 0.f, _coef = 1.f;
};

// un-fused BatchNorm / Scale: y = x*w[c] + b[c] (batch_norm.cpp:36-60, scale.cpp:41-60)
class ScaleLikeOp : public OperatorBase {
public:
    Status InitParam() override {
        if (_node->op == "BatchNorm") {
            auto eps = GET_PARAMETER(float, epsilon);
            auto mean = block_vector(GET_PARAMETER(PBlockPtr, weight_1));
            auto var = block_vector(GET_PARAMETER(PBlockPtr, weight_2));
            float factor = block_vector(GET_PARAMETER(PBlockPtr, weight_3))[0];
            factor = factor == 0 ? 1.f : 1.f / factor;
            _scale_w.resize(mean.size());
            _scale_b.resize(mean.size());
            for (size_t i = 0; i < mean.size(); ++i) {
                float alpha = 1.f / sqrtf(var[i] * factor + eps);
                _scale_w[i] = alpha;
                _scale_b[i] = -1.f * (mean[i] * factor) * alpha;
            }
            _bias_term = true;
        } else {
            _bias_term = GET_PARAMETER(bool, bias_term);
            _scale_w = block_vector(GET_PARAMETER(PBlockPtr, weight_1));
            if (_bias_term) _scale_b = block_vector(GET_PARAMETER(PBlockPtr, weight_2));
            _axis = GET_PARAMETER(int, axis);
            _num_axes = GET_PARAMETER(int, num_axes);
        }
        return Status::OK();
    }
    Status InferShape(const TensorVec& ins, TensorVec& outs) override { return infer_same_shape(ins, outs); }
    Status Init(OpContext<NV>&, const TensorVec& ins, TensorVec&) override {
        if (_axis != 1 || _num_axes != 1) return init_fail(*_node, "Scale runs over the channel axis only", SaberUnImplError);
        if (ins[0]->get_layout() != Layout_NHWC) return init_fail(*_node, "Scale needs an NHWC input", SaberInvalidValue);
        const int cs = ins[0]->channel_stored();
        std::vector<float> w(cs, 0.f), b(cs, 0.f);
        for (int i = 0; i < ins[0]->channel() && i < static_cast<int>(_scale_w.size()); ++i) w[i] = _scale_w[i];
        for (int i = 0; i < ins[0]->channel() && i < static_cast<int>(_scale_b.size()); ++i) b[i] = _scale_b[i];
        SABER_INIT_CHECK(_w.re_alloc(cs * sizeof(float), false));
        SABER_INIT_CHECK(_b.re_alloc(cs * sizeof(float), false));
        CUDA_CHECK(cudaMemcpy(_w.ptr, w.data(), cs * sizeof(float), cudaMemcpyHostToDevice));
        CUDA_CHECK(cudaMemcpy(_b.ptr, b.data(), cs * sizeof(float), cudaMemcpyHostToDevice));
        return Status::OK();
    }
    void operator()(OpContext<NV>& ctx, const TensorVec& ins, TensorVec& outs) override {
        const size_t pixels = static_cast<size_t>(ins[0]->num()) * ins[0]->height() * ins[0]->width();
        SABER_CHECK(b200_scale_run(ins[0]->get_dtype(), ins[0]->data(), outs[0]->mutable_data(), pixels,
                                   ins[0]->channel_stored(), static_cast<const float*>(_w.ptr),
                                   _bias_term ? static_cast<const float*>(_b.ptr) : nullptr, ctx.get_compute_stream()));
    }

private:
    std::vector<float> _scale_w, _scale_b;
    bool _bias_term = false;
    int _axis = 1, _num_axes = 1;
    DeviceBuffer _w, _b;
};

// ------------------------------------------------------------------ squeeze-and-excitation
// Axpy (framework/operators/axpy.cpp:63-68): out = gate[n,c] * x + y; inputs 0 = gate [n,C,1,1], 1 = x, 2 = y.
// AxpyRelu is Axpy + ReLU fused (this build's pattern; the reference has none). The kernel keys on the dtypes.
class AxpyOp : public OperatorBase {
public:
    Status InitParam() override {
        _relu = _node->op == "AxpyRelu";
        _slope = _relu ? _node->get_attr_or<float>("relu_0_alpha", 0.f) : 0.f;
        return Status::OK();
    }
    Status InferShape(const TensorVec& ins, TensorVec& outs) override {
        if (ins.size() != 3) return Status::ANAKINFAIL("Axpy takes 3 inputs (gate, x, y), got " + std::to_string(ins.size()));
        const Tensor<NV>& g = *ins[0];
        const Tensor<NV>& x = *ins[1];
        const Tensor<NV>& y = *ins[2];
        if (x.num() != y.num() || x.channel() != y.channel() || x.height() != y.height() || x.width() != y.width())
            return Status::ANAKINFAIL("Axpy: x and y differ in shape");
        if (g.num() != x.num() || g.channel() != x.channel() || g.height() != 1 || g.width() != 1)
            return Status::ANAKINFAIL("Axpy: the gate must be [n, C, 1, 1] of x's n and C");
        Shape s = x.valid_shape();
        s.set_layout(outs[0]->get_layout());
        return outs[0]->set_shape(s) == SaberSuccess ? Status::OK() : Status::ANAKINFAIL("Axpy InferShape");
    }
    Status Init(OpContext<NV>&, const TensorVec& ins, TensorVec& outs) override {
        const Tensor<NV>& g = *ins[0];
        const Tensor<NV>& x = *ins[1];
        const Tensor<NV>& y = *ins[2];
        const Tensor<NV>& o = *outs[0];
        if (x.get_layout() != Layout_NHWC || y.get_layout() != Layout_NHWC || o.get_layout() != Layout_NHWC ||
            y.channel_stored() != x.channel_stored() || o.channel_stored() != x.channel_stored())
            return Status::ANAKINFAIL("Axpy (node " + _node->name + "): x, y and out must be NHWC of one channel pitch");
        memset(&_d, 0, sizeof(_d));
        _d.x_dtype = x.get_dtype(); _d.y_dtype = y.get_dtype(); _d.out_dtype = o.get_dtype(); _d.gate_dtype = g.get_dtype();
        _d.n = x.num(); _d.hw = x.height() * x.width(); _d.c = x.channel(); _d.ld = x.channel_stored();
        _d.ldg = g.channel_stored();
        _d.relu = _relu ? 1 : 0;
        _d.neg_slope = _slope;
        auto q8 = [](DataType d) { return d == AK_INT8 || d == AK_UINT8; };
        if (q8(x.get_dtype()) && _relu && _slope != 0.f)
            return Status::ANAKINFAIL("AxpyRelu (node " + _node->name + "): the 8-bit Axpy runs a plain ReLU, relu_0_alpha " +
                                      std::to_string(_slope) + " is not supported");
        if (q8(x.get_dtype())) {
            if (x.get_scale().empty() || y.get_scale().empty() || o.get_scale().empty())
                return Status::ANAKINFAIL("Axpy (node " + _node->name + "): 8-bit x, y and out need calibrated scales");
            // the u8 factor 127/255 as the INT8 eltwise carries it (EltwiseOp above)
            const float u = 127.f / 255.f;
            const float fx = x.get_scale()[0] * (x.get_dtype() == AK_UINT8 ? u : 1.f);
            const float fy = y.get_scale()[0] * (y.get_dtype() == AK_UINT8 ? u : 1.f);
            const float fo = o.get_scale()[0] * (o.get_dtype() == AK_UINT8 ? u : 1.f);
            _d.ax = fx / fo;
            _d.ay = fy / fo;
        }
        return Status::OK();
    }
    void operator()(OpContext<NV>& ctx, const TensorVec& ins, TensorVec& outs) override {
        SABER_CHECK(static_cast<SaberStatus>(b200_axpy_run(&_d, ins[0]->data(), ins[1]->data(), ins[2]->data(),
                                                           outs[0]->mutable_data(), ctx.get_compute_stream())));
    }
    int output_signedness() const override { return _relu ? 1 : 0; }

private:
    bool _relu = false;
    float _slope = 0.f;
    b200_axpy_desc_t _d;
};

// SqueezeExcite (Graph::Optimize's fusion of global AVE Pooling -> ConvRelu 1x1 -> Convolution 1x1 ->
// Activation(Sigmoid)): the excitation gate [n, C, 1, 1], fp32 in every precision, in one launch (b200_se_gate_run).
// The pooling's attributes stay unprefixed; the followers' carry conv_0_, conv_1_ and act_0_.
class SqueezeExciteOp : public OperatorBase {
public:
    Status InitParam() override {
        const Node& n = *_node;
        const std::string what = "SqueezeExcite (node " + n.name + "): ";
        if (n.get_attr_or<std::string>("method", "") != "AVG" || !n.get_attr_or<bool>("global_pooling", false))
            return Status::ANAKINFAIL(what + "the pooling must be a global AVG pooling");
        if (n.get_attr_or<std::string>("act_0_type", "") != "Sigmoid") return Status::ANAKINFAIL(what + "the activation must be a Sigmoid");
        if (n.get_attr_or<float>("conv_0_relu_0_alpha", 0.f) != 0.f) return Status::ANAKINFAIL(what + "the squeeze ReLU must be plain");
        PBlockPtr w1 = n.get_attr<PBlockPtr>("conv_0_weight_1"), w2 = n.get_attr<PBlockPtr>("conv_1_weight_1");
        if (!w1 || !w2 || w1->is_int8() || w2->is_int8()) return Status::ANAKINFAIL(what + "fp32 weights are needed");
        _r = w1->h.num();
        _c = w1->h.channel();
        if (w1->h.height() != 1 || w1->h.width() != 1 || w2->h.num() != _c || w2->h.channel() != _r ||
            w2->h.height() != 1 || w2->h.width() != 1 || n.get_attr_or<int>("conv_0_group", 1) != 1 ||
            n.get_attr_or<int>("conv_1_group", 1) != 1)
            return Status::ANAKINFAIL(what + "the two convolutions must be 1x1, C -> r -> C, ungrouped");
        for (const char* pre : {"conv_0_", "conv_1_"}) {
            PTuple<int> pad = n.get_attr_or<PTuple<int>>(std::string(pre) + "padding", {0, 0});
            for (int v : pad) if (v != 0) return Status::ANAKINFAIL(what + "the convolutions must be unpadded");
        }
        _w.assign(w1->data(), w1->data() + w1->count());
        _w.insert(_w.end(), w2->data(), w2->data() + w2->count());
        _b.assign(static_cast<size_t>(_r + _c), 0.f);
        if (n.get_attr_or<bool>("conv_0_bias_term", false)) {
            PBlockPtr b = n.get_attr<PBlockPtr>("conv_0_weight_2");
            if (!b || b->count() < _r) return Status::ANAKINFAIL(what + "short squeeze bias");
            std::copy(b->data(), b->data() + _r, _b.begin());
        }
        if (n.get_attr_or<bool>("conv_1_bias_term", false)) {
            PBlockPtr b = n.get_attr<PBlockPtr>("conv_1_weight_2");
            if (!b || b->count() < _c) return Status::ANAKINFAIL(what + "short excitation bias");
            std::copy(b->data(), b->data() + _c, _b.begin() + _r);
        }
        _key = w1.get();
        return Status::OK();
    }
    Status InferShape(const TensorVec& ins, TensorVec& outs) override {
        if (ins.size() != 1 || ins[0]->channel() != _c)
            return Status::ANAKINFAIL("SqueezeExcite: the input must have the " + std::to_string(_c) + " channels of the weights");
        Shape s = outs[0]->valid_shape();
        s.set_num(ins[0]->num());
        s.set_channel(_c);
        s.set_height(1);
        s.set_width(1);
        return outs[0]->set_shape(s) == SaberSuccess ? Status::OK() : Status::ANAKINFAIL("SqueezeExcite InferShape");
    }
    Status Init(OpContext<NV>&, const TensorVec& ins, TensorVec& outs) override {
        const Tensor<NV>& x = *ins[0];
        const std::string what = "SqueezeExcite (node " + _node->name + "): ";
        if (x.get_layout() != Layout_NHWC || outs[0]->get_dtype() != AK_FLOAT)
            return Status::ANAKINFAIL(what + "NHWC input and an fp32 gate are needed");
        memset(&_d, 0, sizeof(_d));
        _d.dtype = x.get_dtype();
        _d.n = x.num(); _d.hw = x.height() * x.width(); _d.c = _c; _d.ld = x.channel_stored(); _d.r = _r;
        _d.ldg = outs[0]->channel_stored();
        _d.scale = 1.f;
        if (x.get_dtype() == AK_INT8 || x.get_dtype() == AK_UINT8) {
            if (x.get_scale().empty()) return Status::ANAKINFAIL(what + "the 8-bit input has no calibrated scale");
            _d.scale = x.get_scale()[0];
        }
        const size_t ws = b200_se_gate_workspace_bytes(&_d);
        if (ws == 0) return Status::ANAKINFAIL(what + "unsupported geometry or dtype");
        if (_ws.re_alloc(ws, false) != SaberSuccess) return Status::ANAKINFAIL(what + "cannot allocate the workspace");
        SABER_INIT_CHECK(weight_arena_floats(_key, "se_gate", _w, _b, _dw, &_w_dev, &_b_dev));
        return Status::OK();
    }
    void operator()(OpContext<NV>& ctx, const TensorVec& ins, TensorVec& outs) override {
        SABER_CHECK(static_cast<SaberStatus>(b200_se_gate_run(&_d, ins[0]->data(), _w_dev, _b_dev,
                                                              _w_dev + static_cast<size_t>(_r) * _c, _b_dev + _r,
                                                              static_cast<float*>(outs[0]->mutable_data()), _ws.ptr,
                                                              ctx.get_compute_stream())));
    }
    bool output_fp32() const override { return true; }
    const void* weight_device_ptr() const override { return _w_dev; }

private:
    int _r = 0, _c = 0;
    std::vector<float> _w, _b;     // [W1 | W2], [b1 | b2]
    const void* _key = nullptr;
    b200_se_gate_desc_t _d;
    DeviceBuffer _ws;
    std::shared_ptr<DevWeights> _dw;
    const float* _w_dev = nullptr;
    const float* _b_dev = nullptr;
};

template <typename OpT>
OperatorBase* make() { return new OpT(); }

// Every operator of this build: its name, the factory of each precision it runs in (null: it does not) and whether it
// is a convolution. In an INT8 Net a node runs INT8 when its op has an INT8 factory and the node is marked INT8 or left
// unmarked (SURVEY.md appendix A, ANAKIN_REGISTER_OP_HELPER(..., INT8)); every other node of an INT8 Net runs FP32.
// Output launches nothing and has no INT8 factory: in an INT8 Net it is an FP32 node.
struct OpRow {
    const char* name;
    OperatorBase* (*fp32)();
    OperatorBase* (*fp16)();
    OperatorBase* (*int8)();
    bool conv_family;
};
// one class per precision
template <template <DataType> class Op>
constexpr OpRow typed(const char* name, bool conv_family = false) {
    return {name, make<Op<AK_FLOAT>>, make<Op<AK_HALF>>, make<Op<AK_INT8>>, conv_family};
}
// one class in every precision: its kernels key on the tensor dtype
template <typename Op>
constexpr OpRow any(const char* name) { return {name, make<Op>, make<Op>, make<Op>, false}; }
template <typename Op>
constexpr OpRow float_only(const char* name) { return {name, make<Op>, make<Op>, nullptr, false}; }

constexpr OpRow kOps[] = {
    typed<ConvFamilyOp>("Convolution", true),
    typed<ConvFamilyOp>("ConvRelu", true),
    typed<ConvFamilyOp>("ConvBatchnorm", true),
    typed<ConvFamilyOp>("ConvBatchnormScale", true),
    typed<ConvFamilyOp>("ConvBatchnormScaleRelu", true),
    typed<ConvFamilyOp>("ConvScale", true),
    typed<ConvFamilyOp>("ConvScaleRelu", true),
    typed<ConvFamilyOp>("ConvEltwise", true),
    typed<ConvFamilyOp>("ConvReluPool", true),
    typed<ConvFamilyOp>("ConvBatchnormScaleReluPool", true),
    typed<DenseOp>("Dense"),
    any<InputOp>("Input"),
    float_only<AliasOp>("Output"),
    any<AliasOp>("Split"),
    any<AliasOp>("Gather"),   // framework/operators/gather.cpp: launches nothing
    any<PoolingOp>("Pooling"),
    any<EltwiseOp>("Eltwise"),
    any<EltwiseOp>("EltwiseRelu"),
    any<AxpyOp>("Axpy"),
    any<AxpyOp>("AxpyRelu"),
    any<SqueezeExciteOp>("SqueezeExcite"),
    float_only<SoftmaxOp>("Softmax"),
    float_only<ActivationOp>("ReLU"),
    float_only<ActivationOp>("Activation"),
    float_only<ScaleLikeOp>("BatchNorm"),
    float_only<ScaleLikeOp>("Scale"),
    float_only<AliasOp>("Flatten"),
};

const OpRow* find_op(const std::string& op_name) {
    for (const OpRow& r : kOps)
        if (op_name == r.name) return &r;
    return nullptr;
}

}  // namespace

bool is_conv_family(const std::string& op_name) {
    const OpRow* r = find_op(op_name);
    return r && r->conv_family;
}

bool has_int8(const std::string& op_name) {
    const OpRow* r = find_op(op_name);
    return r && r->int8;
}

OperatorBase* create_operator(const std::string& op_name, Precision p) {
    const OpRow* r = find_op(op_name);
    if (!r) return nullptr;
    OperatorBase* (*const make_op)() = p == Precision::INT8 ? r->int8 : (p == Precision::FP16 ? r->fp16 : r->fp32);
    return make_op ? make_op() : nullptr;
}

}  // namespace ops
}  // namespace anakin
