// Net / Worker: the executor.  reference framework/core/net/{net.h:35-328, net.cpp:215-509,
// worker.h:69-190, worker.cpp:10-213}
//   Net::init(graph)   creates one operator per node of the optimised graph (precision per node,
//                      calibrator_factory.h:155-174), types every edge tensor (dtype / scale /
//                      layout: net.h:228-260, calibrator_parse.cpp:82-128,180-192), infers shapes,
//                      initialises the ops (weights packed once) and allocates edge memory.
//   Net::prediction()  the hot loop (net.cpp:417-509): launches every op on the compute stream;
//                      B200-first it is captured once into a CUDA graph (static shapes) and
//                      replayed, with programmatic dependent launch between the conv kernels.
//   Worker             a pool of per-thread Nets behind sync / async prediction; each thread can
//                      be pinned to its own GPU (the reference keeps all replicas on one device).
#pragma once
#include <condition_variable>
#include <deque>
#include <future>
#include <map>
#include <memory>
#include <string>
#include <thread>
#include <vector>

#include "graph.h"
#include "operators.h"

namespace anakin {

class ANAKIN_EXPORT NetCore {
public:
    typedef saber::Tensor<saber::NV> DTensor;
    NetCore();
    virtual ~NetCore();
    NetCore(const NetCore&) = delete;
    NetCore& operator=(const NetCore&) = delete;

    // device < 0: keep the current CUDA device
    Status init(graph::GraphCore& graph, Precision precision, int device = -1);
    void prediction();
    void sync();  // wait for the compute stream

    DTensor* get_in(const std::string& in_name);
    DTensor* get_out(const std::string& out_name);
    std::vector<DTensor*> get_in_list();
    std::vector<DTensor*> get_out_list();
    const std::vector<std::string>& get_in_names() const { return _in_names; }
    const std::vector<std::string>& get_out_names() const { return _out_names; }
    // tensor produced by (or aliased to) a node of the optimised graph -- parity tests read
    // intermediate edges through this
    DTensor* get_tensor_from_node(const std::string& node_name);
    std::vector<std::string> get_exec_order() const;  // "name:op" of every launched op
    size_t launched_op_count() const { return _exec.size() - (_head.on ? 2 : 0); }
    cudaStream_t stream() const { return _stream; }
    int device() const { return _device; }
    Precision precision() const { return _precision; }
    void set_use_cuda_graph(bool v);
    bool cuda_graph_active() const { return _graph_exec != nullptr; }
    // device bytes held by edge tensors after buffer sharing / what one buffer per edge would take
    size_t activation_bytes() const { return _act_bytes; }
    size_t activation_bytes_unshared() const { return _act_bytes_unshared; }
    // false: every edge keeps its own buffer, so intermediate tensors stay readable after prediction()
    // (parity tests); default true, or B200_ANAKIN_SHARE_ACTIVATIONS=0. Call before init().
    void set_share_activations(bool v) { _share_activations = v; }
    // device pointers of the packed weights of every launched op that has some (arena sharing is visible here)
    std::vector<const void*> weight_device_ptrs() const;
    // Per-op device time (ms), averaged over `iters` eager runs with a CUDA-event pair around every
    // op on the compute stream (the reference's -DENABLE_OP_TIMER, net.cpp:445-449,494-506).
    // reps > 1: each op is launched `reps` times back to back inside its event pair, which hides the
    // host's launch rate and gives the op's steady-state device time.
    std::vector<float> profile_ops(int iters, int reps = 1);

    // Image inputs with on-device resize (Graph::set_input_image_resize). One request is `count` images, image i
    // being h_i * w_i * c bytes (hw[2i] = h_i, hw[2i + 1] = w_i, rows unpadded), packed back to back in batch order.
    // Everything is checked before any copy: count == the batch, 1 <= h_i <= max_h, 1 <= w_i <= max_w, bytes == the
    // sum, and a valid geometry (b200_image_resize_geometry). The pixels and the per-image table are then copied H2D
    // on the net's stream; the next prediction() resizes them into the input tensor (op `<input>:ImageResize`, the
    // first launch).
    Status set_input_images(const std::string& in_name, const uint8_t* pixels, size_t bytes, const int32_t* hw,
                            size_t count);
    // true when `in_name` is an image input with on-device resize
    bool resizes_input(const std::string& in_name) const { return _resize.count(in_name) != 0; }

    // The staging memory of one resizing input: raw pixels of a request, the geometry table on the device and a
    // pinned host copy that is rewritten only once the previous table upload has completed.
    struct ImageResizeState {
        graph::ImageResize cfg;
        b200_image_resize_desc_t desc{};
        saber::DeviceBuffer staging, table;
        b200_image_resize_entry_t* host_table = nullptr;
        cudaEvent_t table_uploaded = nullptr;
        DTensor* tensor = nullptr;
        ~ImageResizeState();
    };

private:
    Status plan_image_resize(graph::GraphCore& graph);
    struct ExecOp {
        std::string name, op_name;
        ops::OperatorPtr op;
        std::vector<DTensor*> ins, outs;
        int side_join = -1;       // >= 0: runs on the side stream, joined in front of exec op `side_join`
        bool wait_side = false;   // first reader of a side op's result
        int head = 0;             // 1: this pooling op launches the fused head (pool + fc + softmax); 2: covered by it
    };
    void run_eager();
    void drop_cuda_graph();
    void plan_activation_memory(const std::vector<ExecOp>& all);
    void plan_side_ops(std::vector<ExecOp>& all);
    void plan_fused_head();
    struct FusedHead {
        b200_head_desc_t desc;
        const void* w = nullptr;
        const float* bias = nullptr;
        const float* scale = nullptr;
        DTensor *in = nullptr, *pooled = nullptr, *logits = nullptr, *prob = nullptr;
        saber::DeviceBuffer barrier;   // zeroed workspace of b200_head_run (s32 accumulator + ticket)
        bool on = false;
    } _head;

    Precision _precision = Precision::FP32;
    int _device = 0;
    cudaStream_t _stream = nullptr, _side_stream = nullptr;
    cudaEvent_t _fork_ev = nullptr, _join_ev = nullptr;
    saber::Context<saber::NV> _ctx, _side_ctx;
    std::map<std::string, std::unique_ptr<ImageResizeState>> _resize;   // resizing input -> its staging memory
    std::vector<ExecOp> _exec;
    std::map<std::string, std::shared_ptr<DTensor>> _owned;  // producer node -> tensor
    std::map<std::string, DTensor*> _node_tensor;            // every node -> its (possibly aliased) output
    std::vector<std::string> _in_names, _out_names;
    bool _use_cuda_graph = true;
    int _eager_runs = 0;
    cudaGraph_t _graph = nullptr;
    cudaGraphExec_t _graph_exec = nullptr;
    size_t _act_bytes = 0, _act_bytes_unshared = 0;
    bool _share_activations = true;
};

template <typename Ttype, Precision Ptype, OpRunType RunType = OpRunType::ASYNC>
class Net : public NetCore {
public:
    Net() {}
    explicit Net(graph::Graph<Ttype, Ptype>& g, int device = -1) { init(g, device); }
    Status init(graph::Graph<Ttype, Ptype>& g, int device = -1) { return NetCore::init(g, Ptype, device); }
    void prediction() {
        NetCore::prediction();
        if (RunType == OpRunType::SYNC) sync();
    }
};

// ---------------------------------------------------------------------------------------------
// Worker (worker.h:69-190): thread pool, one Net per thread.
class ANAKIN_EXPORT WorkerCore {
public:
    typedef saber::Tensor<saber::NVHX86> HTensor;
    WorkerCore(const std::string& model_path, Precision precision, int thread_num);
    ~WorkerCore();
    void Reshape(const std::string& in_name, std::vector<int> shape) { _reshape[in_name] = shape; }
    void register_inputs(const std::vector<std::string>& names) { _inputs = names; }
    void register_outputs(const std::vector<std::string>& names) { _outputs = names; }
    // pin thread i to device devices[i % size]; empty = current device for every thread
    void set_devices(const std::vector<int>& devices) { _devices = devices; }
    void launch();
    // inputs: fp32 NCHW host tensors in registered-input order; returns fp32 host outputs
    std::future<std::vector<std::vector<float>>> sync_prediction(const std::vector<std::vector<float>>& host_ins);
    void async_prediction(const std::vector<std::vector<float>>& host_ins);
    std::vector<std::vector<float>> async_get_result();
    // Zero-copy flavour for serving loops: `in` (fp32 NCHW of the first registered input) and `out` (first
    // registered output) are caller-owned -- ideally pinned -- host buffers that stay valid until the matching
    // async_get_result() returns; the worker thread copies H2D, runs prediction() and copies D2H on its own
    // stream, so with >= 2 threads one request's transfers overlap another's kernels.
    void async_prediction_view(const float* in, size_t in_count, float* out, size_t out_count);
    // The same two calls for a first input declared an 8-bit image input (Graph::set_input_image): `in` holds exactly
    // the input's uint8 [n][h][w][c] bytes. The fp32 calls fail on an image input and these fail on an fp32 input.
    std::future<std::vector<std::vector<float>>> sync_prediction_image(const uint8_t* in, size_t in_bytes);
    void async_prediction_image_view(const uint8_t* in, size_t in_bytes, float* out, size_t out_count);
    // The same for a first input with on-device resize (Graph::set_input_image_resize): one request is the images of
    // NetCore::set_input_images (`pixels`, `bytes`, `hw`, `count`). The sync form copies them; the async form is
    // zero-copy, and pixels / hw stay caller-owned until the matching async_get_result(). A malformed request fails
    // alone. The fixed-size image calls fail on such an input and these fail on any other.
    std::future<std::vector<std::vector<float>>> sync_prediction_images(const uint8_t* pixels, size_t bytes,
                                                                        const int32_t* hw, size_t count);
    void async_prediction_images_view(const uint8_t* pixels, size_t bytes, const int32_t* hw, size_t count, float* out,
                                      size_t out_count);
    // blocks until every thread has built its Net (or failed); returns the first init error, if any
    std::string wait_ready();
    bool empty();
    int thread_num() const { return _thread_num; }

private:
    struct Task {
        std::vector<std::vector<float>> ins;
        const float* in_view = nullptr;
        float* out_view = nullptr;
        size_t in_count = 0, out_count = 0;
        bool image = false;                 // the first input is given as 8-bit image bytes
        std::vector<uint8_t> image_copy;    // sync_prediction_image: the request's own copy of them
        const uint8_t* image_in = nullptr;  // the bytes (image_copy or the caller's buffer)
        size_t image_bytes = 0;
        bool resize = false;                // image_in holds images of their own sizes, given by hw
        std::vector<int32_t> hw_copy;       // sync_prediction_images: the request's own copy of hw
        const int32_t* hw = nullptr;
        size_t image_count = 0;
        std::promise<std::vector<std::vector<float>>> done;
    };
    void thread_main(int tid);
    std::string _model_path;
    Precision _precision;
    int _thread_num;
    std::vector<int> _devices;
    std::map<std::string, std::vector<int>> _reshape;
    std::vector<std::string> _inputs, _outputs;
    std::vector<std::thread> _threads;
    std::deque<std::shared_ptr<Task>> _tasks;
    std::deque<std::future<std::vector<std::vector<float>>>> _async_que;
    std::mutex _mu, _graph_mu;
    std::condition_variable _cv;
    bool _stop = false;
    int _ready = 0;
    std::condition_variable _ready_cv;
    std::shared_ptr<graph::GraphCore> _graph;  // loaded + optimised once, shared by all threads
    std::vector<std::string> _init_errors;
};

template <typename Ttype, Precision Ptype, OpRunType RunType = OpRunType::ASYNC>
class Worker : public WorkerCore {
public:
    Worker(const std::string& model_path, int thread_num) : WorkerCore(model_path, Ptype, thread_num) {}
};

}  // namespace anakin
