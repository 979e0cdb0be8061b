// Graph, Node, Edge, PBlock: host-side mirror of Anakin's framework/graph for the CNN
// classification path.
//   reference framework/graph/{graph.h:36-226, node.h, arc.h, graph_global_mem.h:78-250}
//             framework/core/parameter.h:62,191-316 (PTuple, PBlock)
//             framework/core/types.h:25-39 (Precision, OpRunType)
// Kept: load / save of *.anakin.bin, ResetBatchSize / Reshape, Optimize(with_fusion) with
// the fusion patterns of llvm/fusion/fusion_op_register.cpp:45-175 (merged attrs renamed
// "<patternNode>_<attr>", graph.cpp:588-762), the ConvEltwise scheduler
// (llvm/optimizer/conv_elewise_fusion_scheduler.cpp:31-136) and execution ordering.
#pragma once
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <variant>
#include <vector>

#include "saber.h"

namespace anakin {

enum class Precision : int { INT4 = -10, INT8 = -2, FP16 = -1, FP32 = 0, FP64 };
enum class OpRunType : int { SYNC, ASYNC };

// framework/core/base.h:27-48
class ANAKIN_EXPORT Status {
public:
    Status() : _ok(true) {}
    Status(bool ok, const std::string& msg) : _ok(ok), _msg(msg) {}
    static Status OK() { return Status(); }
    static Status ANAKINFAIL(const std::string& msg) { return Status(false, msg); }
    operator bool() const { return _ok; }
    const char* info() const { return _msg.c_str(); }

private:
    bool _ok;
    std::string _msg;
};

template <typename T>
using PTuple = std::vector<T>;

// Weight block: host tensor (4-D), fp32 -- or int8 codes with per-output-channel scales when the model file
// stores quantised weights (model_io.cpp:204-216). The device image is built by the consuming op (packed for
// wgmma) once per device and shared by every Net that uses the block (saber_funcs.cpp, WeightArena).
struct PBlock {
    saber::Tensor<saber::NVHX86> h;
    saber::Tensor<saber::NVHX86>& h_tensor() { return h; }
    bool is_int8() const { return h.get_dtype() == saber::AK_INT8; }
    const float* data() const { return static_cast<const float*>(h.data()); }
    float* mutable_data() { return static_cast<float*>(h.mutable_data()); }
    const int8_t* data_q8() const { return static_cast<const int8_t*>(h.data()); }
    int8_t* mutable_data_q8() { return static_cast<int8_t*>(h.mutable_data()); }
    long long count() const { return h.valid_size(); }
};
typedef std::shared_ptr<PBlock> PBlockPtr;

namespace graph {

typedef std::variant<std::string, int, float, bool, PTuple<int>, PTuple<float>, PTuple<bool>,
                     PTuple<std::string>, PBlockPtr>
    AttrValue;

struct Node {
    std::string name;
    std::string op;                      // operator name (OpProto.name)
    std::vector<std::string> ins, outs;  // producer / consumer node names, ordered
    std::map<std::string, AttrValue> attrs;
    saber::DataType bit_type = saber::AK_INVALID;  // NodeProto.bit_type
    int lane = 0;
    bool need_wait = false;
    std::map<std::string, std::string> share_pairs;  // attr key -> node that owns the shared weight (node.h set_share_pair)

    template <typename T>
    bool has_attr(const std::string& k) const {
        auto it = attrs.find(k);
        return it != attrs.end() && std::holds_alternative<T>(it->second);
    }
    bool has(const std::string& k) const { return attrs.count(k) != 0; }
    template <typename T>
    const T& get_attr(const std::string& k) const {
        auto it = attrs.find(k);
        if (it == attrs.end() || !std::holds_alternative<T>(it->second)) {
            fprintf(stderr, "[FATAL] node %s (%s): missing or mistyped attr '%s'\n", name.c_str(), op.c_str(), k.c_str());
            abort();
        }
        return std::get<T>(it->second);
    }
    template <typename T>
    T get_attr_or(const std::string& k, const T& dflt) const {
        auto it = attrs.find(k);
        if (it == attrs.end() || !std::holds_alternative<T>(it->second)) return dflt;
        return std::get<T>(it->second);
    }
    template <typename T>
    void set_attr(const std::string& k, const T& v) { attrs[k] = v; }
};
typedef std::shared_ptr<Node> NodePtr;

struct Edge {
    std::string bottom, top;
    std::vector<float> scale;  // calibrated activation scale of `bottom`'s output (TargetProto.scale)
    bool shared = false;
    std::string share_from;
    std::string name() const { return bottom + "_" + top; }
};

class ANAKIN_EXPORT GraphCore {
public:
    GraphCore() {}
    const std::string& name() const { return _name; }
    void set_name(const std::string& n) { _name = n; }

    Status load(const std::string& model_path);
    Status load(const char* buffer, size_t len);
    Status save(const std::string& model_path);

    void Reshape(const std::string& in_name, std::vector<int> shape);
    void ResetBatchSize(const std::string& in_name, int batch_size);
    Status Optimize(bool with_fusion = true);
    bool is_optimized() const { return _optimized; }

    // manual construction (graph.h:62-75)
    Status AddOp(const std::string& name, const std::string& type, const std::vector<std::string>& ins,
                 const std::vector<std::string>& outs);
    template <typename T>
    Status AddOpAttr(const std::string& op_name, const std::string& attr_name, const T& v) {
        auto it = _nodes.find(op_name);
        if (it == _nodes.end()) return Status::ANAKINFAIL("no such op " + op_name);
        it->second->set_attr(attr_name, v);
        return Status::OK();
    }
    Status Freeze();

    std::vector<std::string>& get_ins() { return _ins; }
    std::vector<std::string>& get_outs() { return _outs; }
    const std::vector<std::string>& get_nodes_in_order() const { return _order; }
    NodePtr operator[](const std::string& n) const {
        auto it = _nodes.find(n);
        return it == _nodes.end() ? nullptr : it->second;
    }
    bool has_node(const std::string& n) const { return _nodes.count(n) != 0; }
    // scale of the edge bottom->top (empty when not calibrated)
    std::vector<float> edge_scale(const std::string& bottom, const std::string& top) const;
    std::vector<float> node_out_scale(const std::string& node) const;
    size_t node_count() const { return _nodes.size(); }

protected:
    friend class GraphIO;
    void add_node(const NodePtr& n);
    void remove_node(const std::string& n);
    void rebuild_edges_from_nodes();
    Status topo_sort();
    void fuse_in_order_patterns();
    void fuse_conv_eltwise();

    std::string _name;
    std::map<std::string, NodePtr> _nodes;
    std::vector<std::string> _order;   // file order before Optimize, execution order after
    std::vector<std::string> _ins, _outs;
    std::map<std::string, Edge> _edges;  // key = Edge::name()
    bool _optimized = false;
    std::mutex _mut;
};

// Typed facade with the reference's template signature: Graph<NV, Precision::INT8> etc.
template <typename Ttype, Precision Ptype>
class Graph : public GraphCore {
public:
    static constexpr Precision precision = Ptype;
};

}  // namespace graph
}  // namespace anakin
