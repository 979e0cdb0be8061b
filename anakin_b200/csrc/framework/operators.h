// Operators: turn graph node attributes into ConvEngine specs and C-ABI descriptors, and launch them.
//   reference framework/core/operator/operator.h:38-318 (Operator, OperatorHelper, OpFactory,
//             ANAKIN_REGISTER_OP[_HELPER]), framework/operators/*.cpp + fusion_ops/*.cpp
// One class per operator family carries both the reference's Operator (operator()) and
// OperatorHelper (InitParam / InferShape / Init) roles; one table in operators.cpp holds the
// by-name registry the Net uses (calibrator_factory.h:155-174 picks the precision per node).
#pragma once
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
    virtual Status InitParam() = 0;                                        // the node's attributes
    virtual Status InferShape(const TensorVec& ins, TensorVec& outs) = 0;  // the output's shape
    // once, after the memory plan: checks the tensors and builds what the launch needs
    virtual Status Init(OpContext<saber::NV>& ctx, const TensorVec& ins, TensorVec& outs) = 0;
    // launches on ctx's compute stream
    virtual void operator()(OpContext<saber::NV>& ctx, const TensorVec& ins, TensorVec& outs) = 0;
    // INT8 edge typing (docs/Manual/int8_design_ch.md): ops ending in relu emit u8.
    // 1 = unsigned, 0 = signed, -1 = same as input 0.
    virtual int output_signedness() const { return 0; }
    // true when the op writes an fp32 tensor in every precision, whatever its readers are (the SE gate)
    virtual bool output_fp32() const { return false; }
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

// A new operator of the named op at precision p, or null when the op does not run at p. The operator table and the
// per-node precision rule are in operators.cpp.
ANAKIN_EXPORT OperatorBase* create_operator(const std::string& op_name, Precision p);
// true for the ops with an INT8 operator: the nodes of an INT8 Net that run INT8 unless marked otherwise
bool has_int8(const std::string& op_name);
// true for the convolution-family operator names (Convolution and its fused forms): the only readers of an image input
bool is_conv_family(const std::string& op_name);

}  // namespace ops
}  // namespace anakin
