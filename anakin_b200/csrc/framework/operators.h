// Operators: bind graph node attributes to Saber params and launch the Saber funcs.
//   reference framework/core/operator/operator.h:38-318 (Operator, OperatorHelper, OpFactory,
//             ANAKIN_REGISTER_OP[_HELPER]), framework/operators/*.cpp + fusion_ops/*.cpp
// One class per operator family carries both the reference's Operator (operator()) and
// OperatorHelper (InitParam / InferShape / Init) roles; OpFactory<NV, Precision> keeps the
// by-name registry the Net uses (calibrator_factory.h:155-174 picks the precision per node).
#pragma once
#include <functional>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "graph.h"
#include "saber_funcs.h"

namespace anakin {

template <typename Ttype>
using Tensor4dPtr = saber::Tensor<Ttype>*;
template <typename Ttype>
using OpContext = saber::Context<Ttype>;

namespace ops {

class ANAKIN_EXPORT OperatorBase {
public:
    typedef std::vector<saber::Tensor<saber::NV>*> TensorVec;
    virtual ~OperatorBase() {}
    void BindParam(const graph::NodePtr& node) { _node = node; }
    virtual Status InitParam() = 0;                                        // attrs -> saber Param
    virtual Status InferShape(const TensorVec& ins, TensorVec& outs) = 0;  // compute_output_shape
    virtual Status Init(OpContext<saber::NV>& ctx, const TensorVec& ins, TensorVec& outs) = 0;
    virtual void operator()(OpContext<saber::NV>& ctx, const TensorVec& ins, TensorVec& outs) = 0;
    // INT8 edge typing (docs/Manual/int8_design_ch.md): ops ending in relu emit u8.
    // 1 = unsigned, 0 = signed, -1 = same as input 0.
    virtual int output_signedness() const { return 0; }
    // true when the op launches nothing and its outputs alias its first input
    virtual bool is_alias() const { return false; }
    // device address of the op's packed weights (null for weightless ops); Nets built from one Graph on one
    // device report the same address (WeightArena)
    virtual const void* weight_device_ptr() const { return nullptr; }
    // Hooks for the Net's fused classifier head (global pooling -> inner product -> softmax in one launch,
    // b200_head_run): each op reports whether -- after Init -- it is the plain form the fused kernel implements.
    virtual bool head_pool_info(int* is_max) const { (void)is_max; return false; }
    virtual bool head_fc_info(b200_fc_stream_desc_t* d, const void** w, const float** bias, const float** scale) const {
        (void)d; (void)w; (void)bias; (void)scale;
        return false;
    }
    virtual bool head_softmax_info(int* axis) const { (void)axis; return false; }
    const graph::NodePtr& node() const { return _node; }

protected:
    graph::NodePtr _node;
};
typedef std::shared_ptr<OperatorBase> OperatorPtr;

// OpFactory<Ttype, Ptype>::Global()[name] -> new operator (operator.h:210-257)
class ANAKIN_EXPORT OpFactoryCore {
public:
    typedef std::function<OperatorBase*()> Creator;
    void Register(const std::string& name, Creator c) { _creators[name] = c; }
    OperatorBase* operator[](const std::string& name) const {
        auto it = _creators.find(name);
        return it == _creators.end() ? nullptr : it->second();
    }
    bool has(const std::string& name) const { return _creators.count(name) != 0; }
    std::vector<std::string> get_list_op_name() const {
        std::vector<std::string> v;
        for (auto& kv : _creators) v.push_back(kv.first);
        return v;
    }

private:
    std::map<std::string, Creator> _creators;
};

template <typename Ttype, Precision Ptype>
class OpFactory : public OpFactoryCore {
public:
    static OpFactory& Global() {
        static OpFactory f;
        return f;
    }
};

// Registers every operator of this build into the three precision factories (static-init in the
// reference via ANAKIN_REGISTER_OP_HELPER; explicit and idempotent here).
ANAKIN_EXPORT void register_all_operators();

// precision -> factory lookup with the reference's fallback (an INT8 net may hold fp32 nodes)
ANAKIN_EXPORT OperatorBase* create_operator(const std::string& op_name, Precision p);
// true for the convolution-family operator names (Convolution and its fused forms): the only readers of an image input
bool is_conv_family(const std::string& op_name);

}  // namespace ops
}  // namespace anakin
