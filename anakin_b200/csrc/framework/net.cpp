// Net / Worker implementation -- see net.h for the reference mapping.
#include "net.h"

#include <algorithm>
#include <stdexcept>
#include <set>

namespace anakin {

using namespace saber;
using graph::GraphCore;
using graph::NodePtr;

NetCore::NetCore() {}

NetCore::~NetCore() {
    drop_cuda_graph();
    _exec.clear();
    _resize.clear();
    _owned.clear();
    if (_fork_ev) cudaEventDestroy(_fork_ev);
    if (_join_ev) cudaEventDestroy(_join_ev);
    if (_side_stream) cudaStreamDestroy(_side_stream);
    if (_stream) cudaStreamDestroy(_stream);
}

void NetCore::drop_cuda_graph() {
    if (_graph_exec) { cudaGraphExecDestroy(_graph_exec); _graph_exec = nullptr; }
    if (_graph) { cudaGraphDestroy(_graph); _graph = nullptr; }
}

void NetCore::set_use_cuda_graph(bool v) {
    _use_cuda_graph = v;
    if (!v) drop_cuda_graph();
}

namespace {

bool op_supports_int8(const std::string& op) {
    // who gets an INT8 kernel at all (SURVEY.md appendix A, ANAKIN_REGISTER_OP_HELPER(..., INT8))
    static const std::set<std::string> s = {
        "Convolution", "ConvRelu", "ConvBatchnorm", "ConvBatchnormScale", "ConvBatchnormScaleRelu", "ConvScale",
        "ConvScaleRelu", "ConvEltwise", "ConvReluPool", "ConvBatchnormScaleReluPool", "Dense", "Pooling", "Eltwise", "EltwiseRelu", "Split", "Gather", "Input"};
    return s.count(op) != 0;
}

// The exec entry `<input>:ImageResize`: resizes the request's staged images into the image input tensor. It has no
// graph node; Net::init puts it first, so it is captured into the CUDA graph and timed by profile_ops like any op.
class ImageResizeOp : public ops::OperatorBase {
public:
    explicit ImageResizeOp(const NetCore::ImageResizeState* s) : _s(s) {}
    Status InitParam() override { return Status::OK(); }
    Status InferShape(const TensorVec&, TensorVec&) override { return Status::OK(); }
    Status Init(OpContext<NV>&, const TensorVec&, TensorVec&) override { return Status::OK(); }
    void operator()(OpContext<NV>& ctx, const TensorVec&, TensorVec& outs) override {
        SABER_CHECK(static_cast<SaberStatus>(b200_image_resize_run(
            &_s->desc, static_cast<const uint8_t*>(_s->staging.ptr), _s->table.ptr,
            static_cast<uint8_t*>(outs[0]->mutable_data()), ctx.get_compute_stream())));
    }

private:
    const NetCore::ImageResizeState* _s;
};

}  // namespace

NetCore::ImageResizeState::~ImageResizeState() {
    if (table_uploaded) cudaEventDestroy(table_uploaded);
    if (host_table) cudaFreeHost(host_table);
}

// Staging memory and the ImageResize exec entry of every image input with on-device resize.
Status NetCore::plan_image_resize(GraphCore& graph) {
    for (auto& nm : _in_names) {
        NodePtr node = graph[nm];
        graph::ImageResize cfg;
        const int st = node ? graph::node_image_resize(*node, &cfg) : 0;
        if (st == 0) continue;
        if (st < 0) return Status::ANAKINFAIL("malformed image resize attributes on Input " + nm);
        DTensor* t = _node_tensor[nm];
        if (!t || !t->is_image())
            return Status::ANAKINFAIL("input " + nm + " has image resize attributes but is not an image input");
        const int H = t->height(), W = t->width(), c = t->channel();
        if (cfg.resize_short != 0 && cfg.resize_short < std::max(H, W))
            return Status::ANAKINFAIL("input " + nm + ": image_resize_short " + std::to_string(cfg.resize_short) +
                                      " must be 0 or at least max(H, W) = " + std::to_string(std::max(H, W)) +
                                      " of the " + std::to_string(H) + " x " + std::to_string(W) + " input");
        auto s = std::make_unique<ImageResizeState>();
        s->cfg = cfg;
        s->tensor = t;
        s->desc.n = t->num(); s->desc.c = c; s->desc.out_h = H; s->desc.out_w = W;
        const size_t staging = static_cast<size_t>(t->num()) * cfg.max_h * cfg.max_w * c;
        const size_t table = static_cast<size_t>(t->num()) * sizeof(b200_image_resize_entry_t);
        if (s->staging.re_alloc(staging, false) != SaberSuccess || s->table.re_alloc(table, false) != SaberSuccess)
            return Status::ANAKINFAIL("input " + nm + ": cannot allocate " + std::to_string(staging) +
                                      " bytes of image staging memory");
        CUDA_CHECK(cudaMallocHost(reinterpret_cast<void**>(&s->host_table), table));
        CUDA_CHECK(cudaEventCreateWithFlags(&s->table_uploaded, cudaEventDisableTiming));
        // until the first request the table reads as 1 x 1 images at offset 0 (the zeroed staging buffer)
        for (int i = 0; i < t->num(); ++i) {
            b200_image_resize_entry_t& e = s->host_table[i];
            e.offset = 0; e.h = e.w = 1; e.rh = H; e.rw = W; e.top = e.left = 0;
        }
        CUDA_CHECK(cudaMemcpyAsync(s->table.ptr, s->host_table, table, cudaMemcpyHostToDevice, _stream));
        CUDA_CHECK(cudaEventRecord(s->table_uploaded, _stream));
        ExecOp e;
        e.name = nm;
        e.op_name = "ImageResize";
        e.op = std::make_shared<ImageResizeOp>(s.get());
        e.outs.push_back(t);
        _exec.insert(_exec.begin(), e);
        _resize[nm] = std::move(s);
    }
    return Status::OK();
}

Status NetCore::set_input_images(const std::string& in_name, const uint8_t* pixels, size_t bytes, const int32_t* hw,
                                 size_t count) {
    auto it = _resize.find(in_name);
    if (it == _resize.end()) {
        DTensor* t = get_in(in_name);
        if (!t) return Status::ANAKINFAIL("no input " + in_name);
        return Status::ANAKINFAIL("input " + in_name + (t->is_image() ? " is a fixed-size image input (no on-device resize): use set_input_image"
                                                                       : " is not an image input"));
    }
    ImageResizeState& s = *it->second;
    if (!pixels || !hw) return Status::ANAKINFAIL("set_input_images(" + in_name + "): null pixels or sizes");
    if (count != static_cast<size_t>(s.desc.n))
        return Status::ANAKINFAIL("set_input_images(" + in_name + "): " + std::to_string(count) + " images, the batch is " +
                                  std::to_string(s.desc.n));
    std::vector<b200_image_resize_entry_t> tab(count);
    size_t total = 0;
    for (size_t i = 0; i < count; ++i) {
        const int32_t h = hw[2 * i], w = hw[2 * i + 1];
        const std::string which = "set_input_images(" + in_name + "): image " + std::to_string(i) + " is " +
                                  std::to_string(h) + " x " + std::to_string(w);
        if (h < 1 || h > s.cfg.max_h || w < 1 || w > s.cfg.max_w)
            return Status::ANAKINFAIL(which + ", outside 1..max (" + std::to_string(s.cfg.max_h) + " x " +
                                      std::to_string(s.cfg.max_w) + ")");
        b200_image_resize_entry_t& e = tab[i];
        if (b200_image_resize_geometry(h, w, s.cfg.resize_short, s.desc.out_h, s.desc.out_w, &e.rh, &e.rw, &e.top,
                                       &e.left) != B200_SUCCESS)
            return Status::ANAKINFAIL(which + ": no valid resize geometry for resize_short " +
                                      std::to_string(s.cfg.resize_short));
        e.offset = static_cast<int64_t>(total);
        e.h = h; e.w = w;
        total += static_cast<size_t>(h) * w * s.desc.c;
    }
    if (bytes != total)
        return Status::ANAKINFAIL("set_input_images(" + in_name + "): " + std::to_string(bytes) + " pixel bytes, the sizes need " +
                                  std::to_string(total));
    cudaSetDevice(_device);
    // the pinned table may still be in flight from the previous request
    CUDA_CHECK(cudaEventSynchronize(s.table_uploaded));
    memcpy(s.host_table, tab.data(), count * sizeof(b200_image_resize_entry_t));
    CUDA_CHECK(cudaMemcpyAsync(s.table.ptr, s.host_table, count * sizeof(b200_image_resize_entry_t),
                               cudaMemcpyHostToDevice, _stream));
    CUDA_CHECK(cudaEventRecord(s.table_uploaded, _stream));
    CUDA_CHECK(cudaMemcpyAsync(s.staging.ptr, pixels, bytes, cudaMemcpyHostToDevice, _stream));
    return Status::OK();
}

Status NetCore::init(GraphCore& graph, Precision precision, int device) {
    if (device >= 0) {
        if (cudaSetDevice(device) != cudaSuccess) return Status::ANAKINFAIL("cudaSetDevice failed");
        _device = device;
    } else {
        cudaGetDevice(&_device);
    }
    if (!b200_device_ok(_device))
        return Status::ANAKINFAIL("device is not an sm_90 (H100) GPU: no kernel of this build can run (no CPU fallback)");
    if (!graph.is_optimized()) {
        Status st = graph.Optimize();
        if (!st) return st;
    }
    _precision = precision;
    if (!_stream) CUDA_CHECK(cudaStreamCreateWithFlags(&_stream, cudaStreamNonBlocking));
    if (!_side_stream) {
        CUDA_CHECK(cudaStreamCreateWithFlags(&_side_stream, cudaStreamNonBlocking));
        CUDA_CHECK(cudaEventCreateWithFlags(&_fork_ev, cudaEventDisableTiming));
        CUDA_CHECK(cudaEventCreateWithFlags(&_join_ev, cudaEventDisableTiming));
    }
    _ctx = Context<NV>(_device, _stream);
    _side_ctx = Context<NV>(_device, _side_stream);
    drop_cuda_graph();
    _exec.clear(); _resize.clear(); _owned.clear(); _node_tensor.clear(); _eager_runs = 0;
    _in_names = graph.get_ins();
    _out_names = graph.get_outs();
    const char* env = getenv("B200_ANAKIN_CUDA_GRAPH");
    if (env && env[0] == '0') _use_cuda_graph = false;
    env = getenv("B200_ANAKIN_SHARE_ACTIVATIONS");
    if (env && env[0] == '0') _share_activations = false;

    // ---- 1. operators, precision per node (net.cpp:230-288, calibrator_factory.h:155-174)
    struct Built {
        NodePtr node;
        ops::OperatorPtr op;
        bool int8 = false;
    };
    std::vector<Built> built;
    std::map<std::string, size_t> index;
    for (auto& nm : graph.get_nodes_in_order()) {
        NodePtr node = graph[nm];
        Precision p = precision;
        if (precision == Precision::INT8) {
            const bool wants_int8 = node->bit_type == AK_INT8 || (node->bit_type == AK_INVALID && op_supports_int8(node->op));
            p = wants_int8 && op_supports_int8(node->op) ? Precision::INT8 : Precision::FP32;
        }
        ops::OperatorBase* raw = ops::create_operator(node->op, p);
        if (!raw && p == Precision::INT8) { p = Precision::FP32; raw = ops::create_operator(node->op, p); }
        if (!raw) return Status::ANAKINFAIL("operator " + node->op + " (node " + nm + ") is not supported by this build");
        Built b;
        b.node = node;
        b.op.reset(raw);
        b.int8 = (p == Precision::INT8);
        b.op->BindParam(node);
        Status st = b.op->InitParam();
        if (!st) return Status::ANAKINFAIL("InitParam(" + nm + "): " + st.info());
        index[nm] = built.size();
        built.push_back(b);
    }

    // ---- 2. one tensor per producing node; alias ops share their input's tensor
    auto real_consumers = [&](const std::string& nm) {
        std::vector<size_t> out;
        std::vector<std::string> stack = {nm};
        while (!stack.empty()) {
            std::string cur = stack.back(); stack.pop_back();
            for (auto& t : built[index[cur]].node->outs) {
                const Built& c = built[index[t]];
                if (c.op->is_alias() && c.node->op != "Output") stack.push_back(t);
                else out.push_back(index[t]);
            }
        }
        return out;
    };
    // an image input is normalised by the convolutions that read it (conv_stem.cu / b200_image_to_nhwc): every real
    // consumer must be one, reading it as its main input (not as a ConvEltwise residual)
    for (auto& b : built) {
        if (b.node->op != "Input" || graph::node_image_format(*b.node, nullptr) != 1) continue;
        const std::string& nm = b.node->name;
        for (size_t ci : real_consumers(nm)) {
            const graph::Node& c = *built[ci].node;
            std::string src = c.ins.empty() ? std::string() : c.ins[0];
            while (index.count(src) && built[index[src]].op->is_alias() && built[index[src]].node->op != "Input")
                src = built[index[src]].node->ins.empty() ? std::string() : built[index[src]].node->ins[0];
            if (!ops::is_conv_family(c.op) || src != nm)
                return Status::ANAKINFAIL("image input " + nm + " is read by node " + c.name + " (op " + c.op +
                                          "): an image input can only be the input of a convolution");
        }
    }
    for (auto& b : built) {
        const std::string& nm = b.node->name;
        if (b.op->is_alias() && b.node->op != "Input") {
            if (b.node->ins.empty()) return Status::ANAKINFAIL("alias op without input: " + nm);
            _node_tensor[nm] = _node_tensor[b.node->ins[0]];
            continue;
        }
        auto t = std::make_shared<DTensor>();
        // dtype / layout / scale of the edge (net.h:228-260, calibrator_parse.cpp:82-128)
        DataType dt = AK_FLOAT;
        LayoutType layout = b.node->op == "Input" ? Layout_NCHW : Layout_NHWC;
        std::vector<size_t> cons = real_consumers(nm);
        bool consumer_needs_float = false;
        bool all_cons_int8 = !cons.empty();
        for (size_t ci : cons) {
            const std::string& cop = built[ci].node->op;
            if (cop == "Softmax" || cop == "Output") consumer_needs_float = true;
            if (!built[ci].int8 || cop == "Output") all_cons_int8 = false;
        }
        if (b.node->op == "Input") {
            dt = AK_FLOAT;
        } else if (precision == Precision::INT8 && b.int8 && all_cons_int8) {
            int sgn = b.op->output_signedness();
            if (sgn < 0) {
                DTensor* in0 = _node_tensor[b.node->ins[0]];
                dt = in0->get_dtype();
                if (dt != AK_INT8 && dt != AK_UINT8) dt = AK_INT8;
            } else {
                dt = sgn ? AK_UINT8 : AK_INT8;
            }
        } else if (precision == Precision::FP16 && !consumer_needs_float) {
            dt = AK_HALF;
        }
        Shape s({1, 1, 1, 1}, layout);
        t->re_alloc(s, dt);
        t->set_scale(graph.node_out_scale(nm));
        _owned[nm] = t;
        _node_tensor[nm] = t.get();
    }

    // ---- 3. shapes for every edge, then memory, then init (weights packed once per device, see WeightArena)
    std::vector<ExecOp> all;
    for (auto& b : built) {
        ExecOp e;
        e.name = b.node->name;
        e.op_name = b.node->op;
        e.op = b.op;
        for (auto& in : b.node->ins) e.ins.push_back(_node_tensor[in]);
        e.outs.push_back(_node_tensor[b.node->name]);
        Status st = b.op->InferShape(e.ins, e.outs);
        if (!st) return Status::ANAKINFAIL("InferShape(" + e.name + "): " + st.info());
        all.push_back(e);
    }
    plan_side_ops(all);
    plan_activation_memory(all);
    for (auto& kv : _owned)
        if (kv.second->storage_bytes())
            CUDA_CHECK(cudaMemsetAsync(kv.second->mutable_data(), 0, kv.second->storage_bytes(), _stream));
    for (auto& e : all) {
        if (e.op->is_alias()) continue;
        Status st = e.op->Init(e.side_join >= 0 ? _side_ctx : _ctx, e.ins, e.outs);
        if (!st) return Status::ANAKINFAIL("Init(" + e.name + "): " + st.info());
        _exec.push_back(e);
    }
    plan_fused_head();
    Status rst = plan_image_resize(graph);
    if (!rst) return rst;
    // weight uploads and the zero fills above used synchronous copies / this stream: nothing is pending after this
    CUDA_CHECK(cudaStreamSynchronize(_stream));
    CUDA_CHECK(cudaDeviceSynchronize());
    return Status::OK();
}

// Classifier head: global pooling -> inner product -> softmax, three dependent launches of a few microseconds each at
// the end of every request (saber_pooling.cu, saber_fc.cu, saber_softmax.cu), run as ONE cooperative launch
// (b200_head_run). Every edge tensor of the three ops is still written, so the fusion is invisible to readers.
void NetCore::plan_fused_head() {
    _head.on = false;
    // On by default (B200_ANAKIN_FUSED_HEAD=0 keeps the three ops): pooling + inner product are one cluster launch, the
    // softmax a second one. (A first version that split the reduction dimension over the CTAs and combined them with
    // integer atomics took 37 us on ResNet-50 INT8 b8 -- slower than the ~17 us of the three ops -- and was replaced.)
    const char* env = getenv("B200_ANAKIN_FUSED_HEAD");
    if (env && env[0] == '0') return;
    for (size_t i = 0; i + 2 < _exec.size(); ++i) {
        ExecOp &ep = _exec[i], &ef = _exec[i + 1], &es = _exec[i + 2];
        int is_max = 0, axis = 0;
        b200_fc_stream_desc_t fd;
        const void* w; const float *bias, *scale;
        if (ep.side_join >= 0 || ef.side_join >= 0 || es.side_join >= 0 || ef.wait_side || es.wait_side) continue;
        if (!ep.op->head_pool_info(&is_max) || !ef.op->head_fc_info(&fd, &w, &bias, &scale) || !es.op->head_softmax_info(&axis)) continue;
        if (ef.ins.empty() || ef.ins[0] != ep.outs[0] || es.ins.empty() || es.ins[0] != ef.outs[0]) continue;
        DTensor *in = ep.ins[0], *pooled = ep.outs[0], *logits = ef.outs[0], *prob = es.outs[0];
        if (in->get_layout() != Layout_NHWC || pooled->get_layout() != Layout_NHWC || in->get_dtype() != pooled->get_dtype()) continue;
        if (pooled->height() != 1 || pooled->width() != 1 || fd.m > 8 || fd.k != pooled->channel_stored() ||
            fd.in_dtype != pooled->get_dtype() || fd.out_dtype != B200_FLOAT || logits->get_dtype() != AK_FLOAT ||
            prob->get_dtype() != AK_FLOAT || axis != 1 || logits->height() != 1 || logits->width() != 1)
            continue;
        _head.desc.fc = fd;
        _head.desc.hw = in->height() * in->width();
        _head.desc.pool_max = is_max;
        _head.desc.ldp = prob->channel_stored();
        _head.w = w; _head.bias = bias; _head.scale = scale;
        _head.in = in; _head.pooled = pooled; _head.logits = logits; _head.prob = prob;
        if (fd.math != B200_MATH_I8) continue;                           // float heads keep the three ops
        if (_head.barrier.re_alloc(b200_head_workspace_bytes(&_head.desc), false) != SaberSuccess) return;   // zero-filled
        ep.head = 1; ef.head = 2; es.head = 2;
        _head.on = true;
        return;
    }
}

// Off-chain ops (the reference's ParallScheduler gives such nodes their own lane / stream,
// framework/graph/llvm/scheduler.cpp + net.cpp:430-444,480-492): an op whose result is not read by the op that
// follows it -- the projection shortcut `resXa_branch1`, read only by `branch2c` three ops later -- runs on a second
// stream, forked after the ops before it and joined in front of its first reader. Inside the captured CUDA graph
// this is a parallel branch, so the shortcut convolution leaves the critical path of the request.
void NetCore::plan_side_ops(std::vector<ExecOp>& all) {
    const char* env = getenv("B200_ANAKIN_SIDE_STREAM");
    if (env && env[0] == '0') return;
    std::vector<ExecOp*> run;
    for (auto& e : all) if (!e.op->is_alias()) run.push_back(&e);
    std::set<DTensor*> outs;
    for (auto& n : _out_names) outs.insert(_node_tensor[n]);
    int busy_until = -1;   // one side stream: do not stack side ops
    for (size_t i = 0; i + 2 < run.size(); ++i) {
        ExecOp& e = *run[i];
        if (static_cast<int>(i) <= busy_until || e.outs.size() != 1 || outs.count(e.outs[0])) continue;
        if (e.op_name.compare(0, 4, "Conv") != 0) continue;
        int first_reader = -1;
        for (size_t j = i + 1; j < run.size() && first_reader < 0; ++j)
            for (DTensor* t : run[j]->ins) if (t == e.outs[0]) first_reader = static_cast<int>(j);
        if (first_reader <= static_cast<int>(i) + 1) continue;
        // nothing in between may touch the tensors this op writes or reads-and-shares (in-place ops do not exist here)
        e.side_join = first_reader;
        run[first_reader]->wait_side = true;
        busy_until = first_reader;
    }
}

// Activation memory (the reference's MemoryScheduler pass + Net::init_memory, framework/graph/llvm/optimizer/
// memory_scheduler.cpp, framework/core/net/net.cpp:812-898): an edge tensor is live from the op that writes it to
// the last op that reads it (through alias nodes); tensors whose live ranges do not overlap share one buffer.
// Greedy best-fit over the execution order. Kept out of the pool: graph inputs / outputs (the user reads and
// writes them between predictions) and tensors with channel padding (their never-written padding must stay 0).
void NetCore::plan_activation_memory(const std::vector<ExecOp>& all) {
    _act_bytes = 0;
    _act_bytes_unshared = 0;
    for (auto& kv : _owned) _act_bytes_unshared += kv.second->storage_bytes();
    if (!_share_activations) { _act_bytes = _act_bytes_unshared; return; }
    std::map<DTensor*, int> def, last;
    std::vector<const ExecOp*> run;
    for (auto& e : all) if (!e.op->is_alias()) run.push_back(&e);
    for (size_t i = 0; i < run.size(); ++i) {
        for (DTensor* t : run[i]->outs) if (!def.count(t)) def[t] = static_cast<int>(i);
        // a side-stream op may still be reading its inputs until the op that joins it
        const int until = run[i]->side_join >= 0 ? std::max(run[i]->side_join, static_cast<int>(i)) : static_cast<int>(i);
        for (DTensor* t : run[i]->ins) last[t] = std::max(last.count(t) ? last[t] : 0, until);
    }
    std::set<DTensor*> pinned;
    for (auto& n : _in_names) pinned.insert(_node_tensor[n]);
    for (auto& n : _out_names) pinned.insert(_node_tensor[n]);
    struct Slot { size_t bytes = 0; int free_at = -1; std::vector<DTensor*> users; };
    std::vector<Slot> slots;
    std::vector<std::pair<int, DTensor*>> order;
    for (auto& kv : _owned) {
        DTensor* t = kv.second.get();
        if (pinned.count(t) || !def.count(t) || t->storage_bytes() == 0 ||
            (t->get_layout() == Layout_NHWC && t->channel_stored() != t->channel())) {
            _act_bytes += t->storage_bytes();
            continue;
        }
        order.push_back({def[t], t});
    }
    std::sort(order.begin(), order.end());
    for (auto& od : order) {
        DTensor* t = od.second;
        const int d0 = od.first;
        const int l0 = std::max(last.count(t) ? last[t] : d0, d0);
        const size_t need = t->storage_bytes();
        int best = -1;
        for (size_t i = 0; i < slots.size(); ++i) {
            if (slots[i].free_at >= d0) continue;   // still read by the op that defines t (or later)
            if (best < 0) { best = static_cast<int>(i); continue; }
            const bool fit_i = slots[i].bytes >= need, fit_b = slots[best].bytes >= need;
            if (fit_i && (!fit_b || slots[i].bytes < slots[best].bytes)) best = static_cast<int>(i);
            else if (!fit_i && !fit_b && slots[i].bytes > slots[best].bytes) best = static_cast<int>(i);
        }
        if (best < 0) { slots.emplace_back(); best = static_cast<int>(slots.size()) - 1; }
        slots[best].bytes = std::max(slots[best].bytes, need);
        slots[best].free_at = l0;
        slots[best].users.push_back(t);
    }
    for (auto& sl : slots) {
        DTensor backing;
        backing.re_alloc(Shape({1, 1, 1, static_cast<int>((sl.bytes + 15) / 16 * 4)}, Layout_NCHW), AK_FLOAT);
        for (DTensor* t : sl.users) t->share_from(backing);
        _act_bytes += sl.bytes;
    }
}

void NetCore::run_eager() {
    size_t ev = 0;
    for (auto& e : _exec) {
        if (e.wait_side) CUDA_CHECK(cudaStreamWaitEvent(_stream, _join_ev, 0));
        if (e.head == 2) continue;
        if (e.head == 1) {
            SABER_CHECK(static_cast<SaberStatus>(b200_head_run(
                &_head.desc, _head.in->data(), _head.pooled->mutable_data(), _head.w, _head.bias, _head.scale,
                _head.logits->mutable_data(), static_cast<float*>(_head.prob->mutable_data()),
                _head.barrier.ptr, _stream)));
            continue;
        }
        if (e.side_join >= 0) {
            (void)ev;
            CUDA_CHECK(cudaEventRecord(_fork_ev, _stream));
            CUDA_CHECK(cudaStreamWaitEvent(_side_stream, _fork_ev, 0));
            (*e.op)(_side_ctx, e.ins, e.outs);
            CUDA_CHECK(cudaEventRecord(_join_ev, _side_stream));
        } else {
            (*e.op)(_ctx, e.ins, e.outs);
        }
    }
}

void NetCore::prediction() {
    cudaSetDevice(_device);
    if (_graph_exec) {
        CUDA_CHECK(cudaGraphLaunch(_graph_exec, _stream));
        return;
    }
    if (_use_cuda_graph && _eager_runs >= 1) {
        // static shapes: capture the whole op sequence once (one eager run has already built
        // every plan / tensor map), then replay it.
        cudaError_t e = cudaStreamBeginCapture(_stream, cudaStreamCaptureModeThreadLocal);
        if (e == cudaSuccess) {
            run_eager();
            e = cudaStreamEndCapture(_stream, &_graph);
            if (e == cudaSuccess) e = cudaGraphInstantiate(&_graph_exec, _graph, 0);
            if (e == cudaSuccess) {
                CUDA_CHECK(cudaGraphLaunch(_graph_exec, _stream));
                return;
            }
        }
        fprintf(stderr, "[anakin_b200] CUDA graph capture failed (%s); staying eager\n", cudaGetErrorString(e));
        (void)cudaGetLastError();
        drop_cuda_graph();
        _use_cuda_graph = false;
    }
    run_eager();
    ++_eager_runs;
}

std::vector<float> NetCore::profile_ops(int iters, int reps) {
    cudaSetDevice(_device);
    const size_t n = _exec.size();
    if (reps < 1) reps = 1;
    std::vector<cudaEvent_t> ev(2 * n);
    for (auto& e : ev) CUDA_CHECK(cudaEventCreate(&e));
    std::vector<float> ms(n, 0.f);
    iters = iters * 1;
    for (int it = 0; it < iters + 1; ++it) {  // first pass is a warm-up
        for (size_t i = 0; i < n; ++i) {
            CUDA_CHECK(cudaEventRecord(ev[2 * i], _stream));
            for (int r = 0; r < reps; ++r) {   // all on one stream here
                if (_exec[i].head == 2) continue;       // covered by the fused head launch timed at the pooling op
                if (_exec[i].head == 1)
                    SABER_CHECK(static_cast<SaberStatus>(b200_head_run(
                        &_head.desc, _head.in->data(), _head.pooled->mutable_data(), _head.w, _head.bias, _head.scale,
                        _head.logits->mutable_data(), static_cast<float*>(_head.prob->mutable_data()),
                        _head.barrier.ptr, _stream)));
                else
                    (*_exec[i].op)(_ctx, _exec[i].ins, _exec[i].outs);
            }
            CUDA_CHECK(cudaEventRecord(ev[2 * i + 1], _stream));
        }
        CUDA_CHECK(cudaStreamSynchronize(_stream));
        if (it == 0) continue;
        for (size_t i = 0; i < n; ++i) {
            float t = 0.f;
            CUDA_CHECK(cudaEventElapsedTime(&t, ev[2 * i], ev[2 * i + 1]));
            ms[i] += t / iters / reps;
        }
    }
    for (auto& e : ev) cudaEventDestroy(e);
    return ms;
}

std::vector<const void*> NetCore::weight_device_ptrs() const {
    std::vector<const void*> v;
    for (auto& e : _exec)
        if (const void* p = e.op->weight_device_ptr()) v.push_back(p);
    return v;
}

void NetCore::sync() { CUDA_CHECK(cudaStreamSynchronize(_stream)); }

NetCore::DTensor* NetCore::get_in(const std::string& in_name) { return get_tensor_from_node(in_name); }
NetCore::DTensor* NetCore::get_out(const std::string& out_name) { return get_tensor_from_node(out_name); }

NetCore::DTensor* NetCore::get_tensor_from_node(const std::string& node_name) {
    auto it = _node_tensor.find(node_name);
    return it == _node_tensor.end() ? nullptr : it->second;
}

std::vector<NetCore::DTensor*> NetCore::get_in_list() {
    std::vector<DTensor*> v;
    for (auto& n : _in_names) v.push_back(get_in(n));
    return v;
}
std::vector<NetCore::DTensor*> NetCore::get_out_list() {
    std::vector<DTensor*> v;
    for (auto& n : _out_names) v.push_back(get_out(n));
    return v;
}

std::vector<std::string> NetCore::get_exec_order() const {
    std::vector<std::string> v;
    for (auto& e : _exec) v.push_back(e.name + ":" + e.op_name);
    return v;
}

// ---------------------------------------------------------------------------------------------
WorkerCore::WorkerCore(const std::string& model_path, Precision precision, int thread_num)
    : _model_path(model_path), _precision(precision), _thread_num(thread_num) {}

WorkerCore::~WorkerCore() {
    {
        std::lock_guard<std::mutex> lk(_mu);
        _stop = true;
    }
    _cv.notify_all();
    for (auto& t : _threads) if (t.joinable()) t.join();
}

void WorkerCore::launch() {
    for (int i = 0; i < _thread_num; ++i) _threads.emplace_back([this, i] { thread_main(i); });
}

void WorkerCore::thread_main(int tid) {
    const int device = _devices.empty() ? -1 : _devices[tid % _devices.size()];
    NetCore net;
    struct ReadyMark {   // counted on every exit path of the init block
        WorkerCore* w;
        ~ReadyMark() {
            { std::lock_guard<std::mutex> lk(w->_mu); ++w->_ready; }
            w->_ready_cv.notify_all();
        }
    };
    bool init_failed = false;
    {
        ReadyMark mark{this};
        // first thread loads + optimises the graph, every thread builds its own Net (worker.cpp:13-39)
        std::lock_guard<std::mutex> lk(_graph_mu);
        if (!_graph) {
            auto g = std::make_shared<graph::GraphCore>();
            Status st = g->load(_model_path);
            if (st) {
                for (auto& kv : _reshape) g->Reshape(kv.first, kv.second);
                st = g->Optimize();
            }
            if (!st) { _init_errors.push_back(st.info()); init_failed = true; }
            else _graph = g;
        }
        if (!init_failed) {
            Status st = net.init(*_graph, _precision, device);
            if (!st) { _init_errors.push_back(st.info()); init_failed = true; }
        }
        if (!init_failed) {
            if (_inputs.empty()) _inputs = net.get_in_names();
            if (_outputs.empty()) _outputs = net.get_out_names();
        }
    }
    if (init_failed) {
        // a thread without a Net still drains the queue, completing every request with the init error: callers
        // blocked in sync_prediction().get() / async_get_result() return instead of waiting forever
        std::string why;
        { std::lock_guard<std::mutex> lk(_graph_mu); why = _init_errors.empty() ? "Net init failed" : _init_errors.front(); }
        while (true) {
            std::shared_ptr<Task> task;
            {
                std::unique_lock<std::mutex> lk(_mu);
                _cv.wait(lk, [this] { return _stop || !_tasks.empty(); });
                if (_stop && _tasks.empty()) return;
                task = _tasks.front();
                _tasks.pop_front();
            }
            task->done.set_exception(std::make_exception_ptr(std::runtime_error("Worker: " + why)));
        }
    }
    while (true) {
        std::shared_ptr<Task> task;
        {
            std::unique_lock<std::mutex> lk(_mu);
            _cv.wait(lk, [this] { return _stop || !_tasks.empty(); });
            if (_stop && _tasks.empty()) return;
            task = _tasks.front();
            _tasks.pop_front();
        }
        std::vector<std::vector<float>> outs;
        try {
            // the request's form must match the input's: the marker decides, not the byte count
            NetCore::DTensor* in0 = _inputs.empty() ? nullptr : net.get_in(_inputs[0]);
            if (!in0 && (task->image || task->in_view)) throw std::runtime_error("Worker: the model has no input");
            if (in0 && task->image != in0->is_image())
                throw std::runtime_error("Worker: input " + _inputs[0] +
                                         (task->image ? " is an fp32 input, not an image input" : " is an image input: use the image prediction calls"));
            if (in0 && task->image && task->resize != net.resizes_input(_inputs[0]))
                throw std::runtime_error("Worker: input " + _inputs[0] +
                                         (task->resize ? " is a fixed-size image input: use the *_prediction_image calls"
                                                       : " resizes on the GPU: use the *_prediction_images calls"));
            if (task->resize) {
                Status st = net.set_input_images(_inputs[0], task->image_in, task->image_bytes, task->hw, task->image_count);
                if (!st) throw std::runtime_error(std::string("Worker: ") + st.info());
            } else if (task->image) {
                if (task->image_bytes != in0->storage_bytes())
                    throw std::runtime_error("Worker: image request of " + std::to_string(task->image_bytes) + " bytes, input " +
                                             _inputs[0] + " holds " + std::to_string(in0->storage_bytes()));
                CUDA_CHECK(cudaMemcpyAsync(in0->mutable_data(), task->image_in, task->image_bytes, cudaMemcpyHostToDevice, net.stream()));
            }
            if (task->in_view || (task->image && task->out_view)) {
                if (task->in_view) {
                    const size_t ib = std::min(in0->storage_bytes(), task->in_count * sizeof(float));
                    CUDA_CHECK(cudaMemcpyAsync(in0->mutable_data(), task->in_view, ib, cudaMemcpyHostToDevice, net.stream()));
                }
                net.prediction();
                NetCore::DTensor* o = net.get_out(_outputs[0]);
                const size_t ob = std::min(o->storage_bytes(), task->out_count * sizeof(float));
                CUDA_CHECK(cudaMemcpyAsync(task->out_view, o->data(), ob, cudaMemcpyDeviceToHost, net.stream()));
                net.sync();
                task->done.set_value(std::move(outs));
                continue;
            }
            for (size_t i = 0; !task->image && i < _inputs.size() && i < task->ins.size(); ++i) {
                NetCore::DTensor* d = net.get_in(_inputs[i]);
                if (d->is_image()) throw std::runtime_error("Worker: input " + _inputs[i] + " is an image input");
                const size_t bytes = std::min(d->storage_bytes(), task->ins[i].size() * sizeof(float));
                CUDA_CHECK(cudaMemcpyAsync(d->mutable_data(), task->ins[i].data(), bytes, cudaMemcpyHostToDevice, net.stream()));
            }
            net.prediction();
            for (auto& on : _outputs) {
                NetCore::DTensor* d = net.get_out(on);
                std::vector<float> h(d->storage_bytes() / sizeof(float));
                CUDA_CHECK(cudaMemcpyAsync(h.data(), d->data(), d->storage_bytes(), cudaMemcpyDeviceToHost, net.stream()));
                outs.push_back(std::move(h));
            }
            net.sync();
            task->done.set_value(std::move(outs));
        } catch (...) {
            task->done.set_exception(std::current_exception());
        }
    }
}

std::future<std::vector<std::vector<float>>> WorkerCore::sync_prediction(const std::vector<std::vector<float>>& host_ins) {
    auto task = std::make_shared<Task>();
    task->ins = host_ins;
    auto fut = task->done.get_future();
    {
        std::lock_guard<std::mutex> lk(_mu);
        _tasks.push_back(task);
    }
    _cv.notify_one();
    return fut;
}

void WorkerCore::async_prediction_view(const float* in, size_t in_count, float* out, size_t out_count) {
    auto task = std::make_shared<Task>();
    task->in_view = in; task->in_count = in_count;
    task->out_view = out; task->out_count = out_count;
    auto fut = task->done.get_future();
    {
        std::lock_guard<std::mutex> lk(_mu);
        _tasks.push_back(task);
        _async_que.push_back(std::move(fut));
    }
    _cv.notify_one();
}

std::future<std::vector<std::vector<float>>> WorkerCore::sync_prediction_image(const uint8_t* in, size_t in_bytes) {
    auto task = std::make_shared<Task>();
    task->image = true;
    task->image_copy.assign(in, in + in_bytes);
    task->image_in = task->image_copy.data();
    task->image_bytes = in_bytes;
    auto fut = task->done.get_future();
    {
        std::lock_guard<std::mutex> lk(_mu);
        _tasks.push_back(task);
    }
    _cv.notify_one();
    return fut;
}

void WorkerCore::async_prediction_image_view(const uint8_t* in, size_t in_bytes, float* out, size_t out_count) {
    auto task = std::make_shared<Task>();
    task->image = true;
    task->image_in = in; task->image_bytes = in_bytes;
    task->out_view = out; task->out_count = out_count;
    auto fut = task->done.get_future();
    {
        std::lock_guard<std::mutex> lk(_mu);
        _tasks.push_back(task);
        _async_que.push_back(std::move(fut));
    }
    _cv.notify_one();
}

std::future<std::vector<std::vector<float>>> WorkerCore::sync_prediction_images(const uint8_t* pixels, size_t bytes,
                                                                                 const int32_t* hw, size_t count) {
    auto task = std::make_shared<Task>();
    task->image = task->resize = true;
    task->image_copy.assign(pixels, pixels + bytes);
    task->image_in = task->image_copy.data();
    task->image_bytes = bytes;
    task->hw_copy.assign(hw, hw + 2 * count);
    task->hw = task->hw_copy.data();
    task->image_count = count;
    auto fut = task->done.get_future();
    {
        std::lock_guard<std::mutex> lk(_mu);
        _tasks.push_back(task);
    }
    _cv.notify_one();
    return fut;
}

void WorkerCore::async_prediction_images_view(const uint8_t* pixels, size_t bytes, const int32_t* hw, size_t count,
                                              float* out, size_t out_count) {
    auto task = std::make_shared<Task>();
    task->image = task->resize = true;
    task->image_in = pixels; task->image_bytes = bytes;
    task->hw = hw; task->image_count = count;
    task->out_view = out; task->out_count = out_count;
    auto fut = task->done.get_future();
    {
        std::lock_guard<std::mutex> lk(_mu);
        _tasks.push_back(task);
        _async_que.push_back(std::move(fut));
    }
    _cv.notify_one();
}

std::string WorkerCore::wait_ready() {
    std::unique_lock<std::mutex> lk(_mu);
    _ready_cv.wait(lk, [this] { return _ready >= _thread_num; });
    return _init_errors.empty() ? std::string() : _init_errors.front();
}

void WorkerCore::async_prediction(const std::vector<std::vector<float>>& host_ins) {
    auto fut = sync_prediction(host_ins);
    std::lock_guard<std::mutex> lk(_mu);
    _async_que.push_back(std::move(fut));
}

std::vector<std::vector<float>> WorkerCore::async_get_result() {
    std::future<std::vector<std::vector<float>>> fut;
    {
        std::lock_guard<std::mutex> lk(_mu);
        if (_async_que.empty()) return {};
        fut = std::move(_async_que.front());
        _async_que.pop_front();
    }
    return fut.get();
}

bool WorkerCore::empty() {
    std::lock_guard<std::mutex> lk(_mu);
    return _async_que.empty();
}

}  // namespace anakin
