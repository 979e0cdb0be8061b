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
#include <atomic>
#include <chrono>
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
    // How each op of get_exec_order is launched: `join` is the exec index of the op that waits for a side-stream op
    // (-1: the op runs on the main stream); `head` is 1 for the fused head's launch (pooling, inner product and
    // softmax as one), 2 for an op it covers, 0 otherwise.
    struct ScheduleEntry { int join, head; };
    std::vector<ScheduleEntry> get_schedule() const;
    size_t launched_op_count() const {   // what run_eager launches: every entry the fused head does not cover, and taps
        size_t n = _input_taps.size();
        for (auto& e : _exec) n += (e.head != 2) + e.taps.size();
        return n;
    }
    cudaStream_t stream() const { return _stream; }
    int device() const { return _device; }
    Precision precision() const { return _precision; }
    void set_use_cuda_graph(bool v);
    bool cuda_graph_active() const { return _graph_exec != nullptr; }
    // device bytes held by edge tensors after buffer sharing / what one buffer per edge would take
    size_t activation_bytes() const { return _act_bytes; }
    size_t activation_bytes_unshared() const { return _act_bytes_unshared; }
    // false (default true): one buffer per edge, so edge tensors stay readable after prediction(). Call before init().
    void set_share_activations(bool v) { _share_activations = v; }
    // device pointers of the packed weights of every launched op that has some (arena sharing is visible here)
    std::vector<const void*> weight_device_ptrs() const;
    // Per-op device time (ms), averaged over `iters` eager runs with a CUDA-event pair around every
    // op on the compute stream (the reference's -DENABLE_OP_TIMER, net.cpp:445-449,494-506).
    // reps > 1: each op is launched `reps` times back to back inside its event pair, which hides the
    // host's launch rate and gives the op's steady-state device time.
    std::vector<float> profile_ops(int iters, int reps = 1);

    // The input setters: each checks the request against the input's kind and size, then copies it H2D on the net's
    // stream (asynchronously: `host` must stay valid until the next sync). A failed copy returns the CUDA error.
    // fp32 input: `count` must equal the input tensor's elements.
    Status set_input(const std::string& in_name, const float* host, size_t count);
    // Fixed-size 8-bit image input (Graph::set_input_image): `bytes` must equal its uint8 [n][h][w][c] storage.
    Status set_input_image(const std::string& in_name, const uint8_t* host, size_t bytes);
    // Image inputs with on-device resize (Graph::set_input_image_resize). One request is `count` images, image i
    // being h_i * w_i * c bytes (hw[2i] = h_i, hw[2i + 1] = w_i, rows unpadded), or an h_i * w_i * 3 / 2 byte frame for
    // an NV12 / I420 input (Graph::set_input_image_pixel_format), packed back to back in batch order.
    // Everything is checked before any copy: count == the batch, 1 <= h_i <= max_h, 1 <= w_i <= max_w (both even for
    // a YUV frame), bytes == the sum, and a valid geometry (b200_image_resize_geometry_ex for the input's filter). The pixels and the per-image
    // table are then copied H2D on the net's stream; the next prediction() resizes them into the input tensor (op
    // `<input>:ImageResize`, the first launches).
    Status set_input_images(const std::string& in_name, const uint8_t* pixels, size_t bytes, const int32_t* hw,
                            size_t count);
    // true when `in_name` is an image input with on-device resize
    bool resizes_input(const std::string& in_name) const { return _resize.count(in_name) != 0; }
    // Slot-range forms of the three setters: stage k images into slots [first, first + k) of the input's batch, with
    // the same checks and the same stream ordering; sizes are per-image multiples (count = k x the elements of one
    // image, bytes = k x its bytes). The whole-batch setters above are the first = 0, k = batch case. The fp32 and
    // image forms leave the other slots as they are.
    Status set_input_slots(const std::string& in_name, const float* host, size_t count, int first, int k);
    Status set_input_image_slots(const std::string& in_name, const uint8_t* host, size_t bytes, int first, int k);
    // Resize form: k = count, table entries [first, first + count) come from hw and every later entry repeats the last
    // of them, so the launch over the whole batch stays valid without copying pixels for the unfilled slots. The
    // pixels go to the staging memory of slot `first` onwards (each slot holds the largest image of the format).
    Status set_input_images_slots(const std::string& in_name, const uint8_t* pixels, size_t bytes, const int32_t* hw,
                                  size_t count, int first);
    // The checks of set_input_images_slots on a request of `count` images, without copying anything
    Status check_input_images(const std::string& in_name, size_t bytes, const int32_t* hw, size_t count) const;
    // Boxes cropped out of frames on an input with on-device resize (b200_image_crop_resize_run): `frame_count` frames
    // packed as set_input_images packs images (frames, bytes, hw), and `count` boxes, int32 [count][5] of (frame, top,
    // left, height, width). Box i becomes image i of the batch: the input's resize and crop applied to
    // frame[top:top+height, left:left+width]. Everything is checked before any copy: count == the batch,
    // 1 <= frame_count <= count, every frame as set_input_images checks an image, and every box names a frame in
    // range, lies inside it (never clamped) and has a valid geometry. set_input_images is the case of one whole-frame
    // box per image.
    Status set_input_crops(const std::string& in_name, const uint8_t* frames, size_t bytes, const int32_t* hw,
                           size_t frame_count, const int32_t* boxes, size_t count);
    // Slot-range form: the boxes fill table entries [first, first + count), later entries repeat the last of them, and
    // the frames go to the staging memory of slots [first, first + frame_count).
    Status set_input_crops_slots(const std::string& in_name, const uint8_t* frames, size_t bytes, const int32_t* hw,
                                 size_t frame_count, const int32_t* boxes, size_t count, int first);
    // The checks of set_input_crops_slots on a request of `count` boxes, without copying anything
    Status check_input_crops(const std::string& in_name, size_t bytes, const int32_t* hw, size_t frame_count,
                             const int32_t* boxes, size_t count) const;

    // INT8 calibration statistics (the reference's EntropyCalibrator passes, entropy_calibrator.cpp), computed inside
    // prediction() of an FP32 net: call set_calib_stats(true) before init(). One slot per graph input (launched first)
    // and one per launched op's output, in exec order; each slot's b200_calib_stats_run goes right behind its producer,
    // on the producer's stream, so it is captured into the CUDA graph with the rest. The pass lives in a device word:
    // switching passes records no new graph. Without the flag nothing of this exists.
    void set_calib_stats(bool v) { _calib.on = v; }
    size_t calib_count() const { return _calib.slots.size(); }
    const std::string& calib_name(size_t i) const { return _calib.slots[i].name; }
    Status calib_reset();                          // zero every maximum and bin (stream-ordered)
    Status calib_set_pass(int pass);               // 0: maxima, 1: histograms (stream-ordered)
    // waits for the stream; max: float[count] (or NULL), hist: uint64[count][B200_CALIB_BINS] (or NULL)
    Status calib_read(float* max, uint64_t* hist);
    // entropy thresholds of the accumulated histograms (b200_calib_kl_run on the stream), int32[count]; waits
    Status calib_kl(int32_t* thresh);

    // Interior-tensor exports (the reference's Net::get_tensor_from_edge, Worker::register_interior_edges): call
    // register_exports before init(). Each name is a node of the optimised graph (an alias node -- Split, Flatten,
    // Gather -- stands for its producer's tensor); init() refuses an unknown name, an Input, a name given twice and a
    // graph output. Every prediction then writes each export as a dense fp32 [n][c][h][w] copy into a buffer of its
    // own (b200_export_run), launched right behind the producer on the producer's stream and captured into the CUDA
    // graph. Edge dtypes, plans, fusions, exec order and the shared activation memory are those of the same net
    // without exports; only launched_op_count() grows, by the number of exports.
    void register_exports(const std::vector<std::string>& names) { _export_names = names; }
    size_t export_count() const { return _exports.size(); }
    const std::string& export_name(size_t i) const { return _exports[i]->name; }
    int export_index(const std::string& name) const;   // -1 when `name` is not an export
    const int32_t* export_dims(size_t i) const { return _exports[i]->nchw; }   // n, c, h, w
    size_t export_elements(size_t i) const;
    const float* export_device_ptr(size_t i) const { return static_cast<const float*>(_exports[i]->buf.ptr); }
    size_t export_bytes() const;                       // device bytes of all export buffers
    // waits for the stream, then copies export i: `count` must equal its n*c*h*w
    Status read_export(size_t i, float* host, size_t count);

    // The staging memory of one resizing input: raw pixels of a request, the crop table on the device (one
    // b200_image_crop_entry_t per slot) and a pinned host copy that is rewritten only once the previous table upload
    // has completed.
    struct ImageResizeState {
        graph::ImageResize cfg;
        b200_image_resize_desc_t desc{};
        saber::DeviceBuffer staging, table;
        saber::DeviceBuffer workspace;      // a Pillow filter: b200_image_resize_workspace bytes
        b200_image_crop_entry_t* host_table = nullptr;
        cudaEvent_t table_uploaded = nullptr;
        DTensor* tensor = nullptr;
        ~ImageResizeState();
    };

private:
    Status plan_image_resize(graph::GraphCore& graph);
    Status crop_table(const std::string& in_name, const ImageResizeState& s, size_t bytes, const int32_t* hw,
                      size_t frame_count, const int32_t* boxes, size_t count, size_t base,
                      b200_image_crop_entry_t* tab) const;
    Status check_crops(const std::string& in_name, bool crops, size_t bytes, const int32_t* hw, size_t frame_count,
                       const int32_t* boxes, size_t count) const;
    Status stage_crops(const std::string& in_name, bool crops, const uint8_t* frames, size_t bytes, const int32_t* hw,
                       size_t frame_count, const int32_t* boxes, size_t count, int first);
    // Taps: launches that read a producer's output -- calibration statistics, then exports -- each right behind the
    // producer, on the producer's stream, so before its first reader can run and before a side op's join is recorded.
    // plan_activation_memory hands a tensor's buffer to another tensor only after its last reader (for a side op's
    // inputs, only after the op that joins it), so every op that could overwrite the tapped tensor is ordered after
    // the tap, and sharing stays on. The taps of the fused head's pooled rows and logits run behind the head launch.
    struct Taps {
        std::vector<int> calib, exports;   // slots of _calib.slots / _exports
        size_t size() const { return calib.size() + exports.size(); }
    };
    struct ExecOp {
        std::string name, op_name;
        ops::OperatorPtr op;
        std::vector<DTensor*> ins, outs;
        bool side = false;        // runs on the side stream, joined in front of side_join()
        bool wait_side = false;   // first reader of a side op's result
        int head = 0;             // 1: `op` is the fused head (pool + fc + softmax); 2: covered by it, launches nothing
        Taps taps;
    };
    int side_join(size_t i) const;
    ExecOp& tap_owner(size_t i);
    void launch(ExecOp& e, saber::Context<saber::NV>& ctx);
    void launch_taps(const Taps& t, cudaStream_t stream);
    Taps _input_taps;             // the graph inputs' statistics, launched before the first entry
    struct ExportSlot {
        std::string name;
        DTensor* t = nullptr;
        int32_t nchw[4] = {0, 0, 0, 0};
        saber::DeviceBuffer buf;  // fp32 [n][c][h][w], outside the activation planner
    };
    std::vector<std::string> _export_names;
    std::vector<std::unique_ptr<ExportSlot>> _exports;
    Status plan_exports(graph::GraphCore& graph);
    struct CalibSlot {
        std::string name;
        DTensor* t = nullptr;
        int64_t rows = 0;
        int32_t c = 0, ld = 0;    // first c of every ld floats count (b200_calib_stats_run)
    };
    struct CalibStats {
        bool on = false;
        std::vector<CalibSlot> slots;
        saber::DeviceBuffer mode, max_bits, hist, thresh;
    } _calib;
    Status plan_calib_stats();
    void run_eager();
    void drop_cuda_graph();
    void plan_activation_memory();
    void plan_side_ops();
    void plan_fused_head();
    static bool head_chain(const ExecOp& ep, const ExecOp& ef, const ExecOp& es);

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
// The packing decision of a batching Worker (WorkerCore::set_max_delay_us); it makes no CUDA call. The queue holds n
// requests in FIFO order: request i carries sizes[i] images (0..batch; 0 for a malformed request, which takes no slot
// and fails alone) and arrived at arrive_us[i]. The batch is the longest prefix whose sizes sum to at most `batch`:
// requests are never split or reordered, so one that does not fit waits for the next batch. The batch closes now when
// it is full, when a request is left behind it, or once now_us reaches arrive_us[0] + max_delay_us; until then the
// gatherer waits for that deadline or the next arrival, and plans again.
struct BatchPlan {
    size_t take = 0;          // the first `take` queued requests form the batch
    bool close = false;       // run it now
    int64_t deadline_us = 0;  // arrive_us[0] + max_delay_us
};
ANAKIN_EXPORT BatchPlan plan_batch(const int* sizes, const int64_t* arrive_us, size_t n, int batch,
                                   int64_t max_delay_us, int64_t now_us);

// Worker (worker.h:69-190): thread pool, one Net per thread.
class ANAKIN_EXPORT WorkerCore {
public:
    typedef saber::Tensor<saber::NVHX86> HTensor;
    WorkerCore(const std::string& model_path, Precision precision, int thread_num);
    ~WorkerCore();
    void Reshape(const std::string& in_name, std::vector<int> shape) { _reshape[in_name] = shape; }
    void register_inputs(const std::vector<std::string>& names) { _inputs = names; }
    // Names that are not graph outputs become exports (NetCore::register_exports) of every thread's Net, in order.
    void register_outputs(const std::vector<std::string>& names) { _outputs = names; }
    // Export the tensor on the edge bottom -> top of the optimised graph (worker.h:100-105), after the exports named
    // by register_outputs, in call order. A Net init fails when no such edge exists. Call before launch().
    void register_interior_edges(const std::string& bottom, const std::string& top) { _edges.push_back({bottom, top}); }
    // Export the tensor of a node of the optimised graph, in call order with register_interior_edges.
    void register_export(const std::string& node) { _edges.push_back({node, std::string()}); }
    // Results carry the graph outputs first, then every export as fp32 [n][c][h][w]: the sync calls return one vector
    // each, and with exports registered the *_view calls fill `out` with graph output 0 then every export, back to
    // back, and fail a request whose out_count is not exactly that total. Blocks until the threads are ready; 0 when
    // a Net failed to build.
    size_t output_count();
    // pin thread i to device devices[i % size]; empty = current device for every thread
    void set_devices(const std::vector<int>& devices) { _devices = devices; }
    // Batching (call before launch(); < 0, the default, leaves it off): a request then carries k images, 1 <= k <=
    // the batch, in any form -- in_count / in_bytes are k x one image's, an images or crops request's count is k, and a
    // view's out_count is k x image_view_floats(). The thread that takes the first queued request gathers the requests behind
    // it in FIFO order while they fit in the batch (plan_batch), waiting at most max_delay_us from that request's
    // arrival (0: only what is already queued); one thread gathers at a time. Every gathered request is checked before
    // any is staged, so a malformed one fails alone; the others go H2D straight into their slots (the NetCore *_slots
    // setters), the Net runs its built batch once, and each request gets its own rows of graph output 0 and of every
    // export. Slots no request filled are computed and dropped. A graph with more than one input is refused.
    void set_max_delay_us(int64_t us) { _max_delay_us = us; }
    int64_t max_delay_us() const { return _max_delay_us; }
    // Per-image sizes once the threads are ready (0 when a Net failed to build): the batch, one image of the first
    // input (floats of an fp32 input, bytes of a fixed-size image input or of a resizing input's resized tensor) and
    // one image's floats of a view result (graph output 0 as stored plus every export).
    int batch();
    size_t image_input_size();
    size_t image_view_floats();
    // batching: predictions run so far and the images of the requests they served
    void batch_stats(uint64_t* predictions, uint64_t* images) const { *predictions = _batches_run; *images = _images_run; }
    void launch();
    // Every request is staged through the Net's input setter for its form (NetCore::set_input, set_input_image,
    // set_input_images) with the same checks; a request they refuse fails alone, and the Worker keeps serving.
    // inputs: fp32 NCHW host tensors, one per registered input in order, each exactly the input's element count;
    // returns fp32 host outputs
    std::future<std::vector<std::vector<float>>> sync_prediction(const std::vector<std::vector<float>>& host_ins);
    void async_prediction(const std::vector<std::vector<float>>& host_ins);
    std::vector<std::vector<float>> async_get_result();
    // Zero-copy flavour for serving loops: `in` (fp32 NCHW of the first registered input, exactly its element count)
    // and `out` (first registered output) are caller-owned -- ideally pinned -- host buffers that stay valid until the
    // matching async_get_result() returns; the worker thread copies H2D, runs prediction() and copies D2H on its own
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
    // The same for boxes cropped out of frames: one request is the frames and boxes of NetCore::set_input_crops, and
    // its k is `count`, the number of boxes. The sync form copies the three arrays; the async form is zero-copy, and
    // frames / hw / boxes stay caller-owned until the matching async_get_result(). A malformed request fails alone.
    std::future<std::vector<std::vector<float>>> sync_prediction_crops(const uint8_t* frames, size_t bytes,
                                                                       const int32_t* hw, size_t frame_count,
                                                                       const int32_t* boxes, size_t count);
    void async_prediction_crops_view(const uint8_t* frames, size_t bytes, const int32_t* hw, size_t frame_count,
                                     const int32_t* boxes, size_t count, float* out, size_t out_count);
    // blocks until every thread has built its Net (or failed); returns the first init error, if any
    std::string wait_ready();
    bool empty();
    int thread_num() const { return _thread_num; }

private:
    typedef std::vector<std::vector<float>> Result;
    // One request. Its form names the NetCore setter that stages the first input.
    struct Request {
        enum Form { FP32, IMAGE, IMAGES, CROPS } form;
        const void* in;                   // the first input: floats (FP32) or bytes; FP32 and null: every input from ins
        size_t size;                      // floats or bytes of `in`
        float* out;                       // view: graph output 0, then every export; null: one vector per result
        size_t out_count;
        const int32_t* hw = nullptr;      // IMAGES: int32 [count][2] image sizes; CROPS: [frame_count][2] frame sizes
        size_t count = 0;                 // IMAGES: images; CROPS: boxes
        const int32_t* boxes = nullptr;   // CROPS: int32 [count][5]
        size_t frame_count = 0;
        std::vector<std::vector<float>> ins;   // the sync forms' own copies of their inputs
        std::vector<uint8_t> bytes;
        std::vector<int32_t> hw_copy, boxes_copy;
        std::promise<Result> done;
        int64_t arrive_us = 0;            // batching: when it was queued (steady clock)
        Request(Form f, const void* in, size_t size, float* out = nullptr, size_t out_count = 0)
            : form(f), in(in), size(size), out(out), out_count(out_count) {}
    };
    std::future<Result> enqueue(std::shared_ptr<Request> r, bool async);
    Status check_form(NetCore& net, const Request& r) const;
    Status stage(NetCore& net, const Request& r) const;
    void thread_main(int tid);
    // batching
    size_t request_images(const Request& r) const;   // k of a request; 0 when it is not a whole number of images
    Status check_request(NetCore& net, const Request& r, size_t k) const;
    Status stage_slots(NetCore& net, const Request& r, int first, int k) const;
    void serve_batches(NetCore& net, const std::string& why);
    void run_batch(NetCore& net, std::vector<std::shared_ptr<Request>>& batch);
    static int64_t now_us();   // steady clock
    int64_t _max_delay_us = -1;
    bool _gathering = false;             // a thread is gathering a batch (under _mu)
    int _batch = 0;                      // the first input's N
    size_t _image_in = 0, _image_view = 0;   // one image: of the first input, of a view result
    std::atomic<uint64_t> _batches_run{0}, _images_run{0};
    std::string _model_path;
    Precision _precision;
    int _thread_num;
    std::vector<int> _devices;
    std::map<std::string, std::vector<int>> _reshape;
    std::vector<std::string> _inputs, _outputs;
    std::vector<std::pair<std::string, std::string>> _edges;  // register_interior_edges / register_export (top "")
    std::vector<std::string> _exports;   // resolved once the graph is loaded: every Net registers these
    bool _io_planned = false;
    size_t _view_count = 0;              // floats of one *_view result: graph output 0, then every export
    std::vector<std::thread> _threads;
    std::deque<std::shared_ptr<Request>> _tasks;
    std::deque<std::future<Result>> _async_que;
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
