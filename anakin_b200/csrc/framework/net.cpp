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

// The exec entry `<input>:ImageResize`: resizes the request's staged images into the image input tensor. It has no
// graph node; Net::init puts it first, so it is captured into the CUDA graph and timed by profile_ops like any op.
class ImageResizeOp : public ops::OperatorBase {
public:
    explicit ImageResizeOp(const NetCore::ImageResizeState* s) : _s(s) {}
    Status InitParam() override { return Status::OK(); }
    Status InferShape(const TensorVec&, TensorVec&) override { return Status::OK(); }
    Status Init(OpContext<NV>&, const TensorVec&, TensorVec&) override { return Status::OK(); }
    void operator()(OpContext<NV>& ctx, const TensorVec&, TensorVec& outs) override {
        const auto* src = static_cast<const uint8_t*>(_s->staging.ptr);
        auto* out = static_cast<uint8_t*>(outs[0]->mutable_data());
        SABER_CHECK(static_cast<SaberStatus>(b200_image_crop_resize_run(
            &_s->desc, _s->cfg.filter, _s->cfg.pixel_format, _s->cfg.max_h, _s->cfg.max_w, _s->cfg.resize_short, src,
            _s->table.ptr, _s->workspace.ptr, out, ctx.get_compute_stream())));
    }

private:
    const NetCore::ImageResizeState* _s;
};

// The fused classifier head: the exec entries global pooling -> inner product -> softmax run as ONE cooperative launch
// (b200_head_run). plan_fused_head installs it as the op of the pooling entry; the other two entries launch nothing.
// Every edge tensor of the three ops is still written, so the fusion is invisible to readers.
class FusedHeadOp : public ops::OperatorBase {
public:
    Status InitParam() override { return Status::OK(); }
    Status InferShape(const TensorVec&, TensorVec&) override { return Status::OK(); }
    Status Init(OpContext<NV>&, const TensorVec&, TensorVec&) override { return Status::OK(); }
    void operator()(OpContext<NV>& ctx, const TensorVec&, TensorVec&) override {
        SABER_CHECK(static_cast<SaberStatus>(b200_head_run(
            &desc, in->data(), pooled->mutable_data(), w, bias, scale, logits->mutable_data(),
            static_cast<float*>(prob->mutable_data()), barrier.ptr, ctx.get_compute_stream())));
    }

    b200_head_desc_t desc{};
    const void* w = nullptr;
    const float *bias = nullptr, *scale = nullptr;
    Tensor<NV> *in = nullptr, *pooled = nullptr, *logits = nullptr, *prob = nullptr;
    DeviceBuffer barrier;   // zeroed workspace of b200_head_run (s32 accumulator + ticket)
};

}  // namespace

NetCore::ImageResizeState::~ImageResizeState() {
    if (table_uploaded) cudaEventDestroy(table_uploaded);
    if (host_table) cudaFreeHost(host_table);
}

static const char* pixel_format_name(int f) {
    return f == B200_IMAGE_YUV_NV12 ? "nv12" : f == B200_IMAGE_YUV_I420 ? "i420" : "interleaved";
}

// Bytes of one h x w request image: h * w * c interleaved, h * w * 3 / 2 for a YUV 4:2:0 frame
static size_t image_bytes(const NetCore::ImageResizeState& s, int h, int w) {
    const size_t px = static_cast<size_t>(h) * w;
    return s.cfg.pixel_format == graph::ImageResize::kInterleaved ? px * s.desc.c : px * 3 / 2;
}

// Staging bytes of one slot: the largest image of the input's format (YUV frames have even sides)
static size_t slot_bytes(const NetCore::ImageResizeState& s) {
    const bool yuv = s.cfg.pixel_format != graph::ImageResize::kInterleaved;
    return image_bytes(s, yuv ? s.cfg.max_h & ~1 : s.cfg.max_h, yuv ? s.cfg.max_w & ~1 : s.cfg.max_w);
}

// Staging memory and the ImageResize exec entry of every image input with on-device resize.
Status NetCore::plan_image_resize(GraphCore& graph) {
    for (auto& nm : _in_names) {
        NodePtr node = graph[nm];
        graph::ImageResize cfg;
        const int st = node ? graph::node_image_resize(*node, &cfg) : 0;
        if (st == 0) continue;
        if (st < 0)
            return Status::ANAKINFAIL("malformed image resize attributes on Input " + nm +
                                      " (image_max_h / image_max_w in 1..16384, image_resize_short >= 0, "
                                      "image_resize_filter 0, 1, 3 or 5, image_pixel_format 0, 1 or 2)");
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
        const size_t staging = static_cast<size_t>(t->num()) * slot_bytes(*s);
        const size_t table = static_cast<size_t>(t->num()) * sizeof(b200_image_crop_entry_t);
        if (s->staging.re_alloc(staging, false) != SaberSuccess || s->table.re_alloc(table, false) != SaberSuccess)
            return Status::ANAKINFAIL("input " + nm + ": cannot allocate " + std::to_string(staging) +
                                      " bytes of image staging memory");
        if (cfg.filter != B200_IMAGE_RESIZE_REFERENCE) {     // a Pillow filter's tap records and intermediates (cv2's: 0)
            size_t ws = 0;
            if (b200_image_resize_workspace(&s->desc, cfg.filter, cfg.max_h, cfg.max_w, cfg.resize_short, &ws) !=
                B200_SUCCESS)
                return Status::ANAKINFAIL("input " + nm + ": no Pillow resize workspace for this geometry");
            if (s->workspace.re_alloc(ws, false) != SaberSuccess)
                return Status::ANAKINFAIL("input " + nm + ": cannot allocate " + std::to_string(ws) +
                                          " bytes of image resize workspace");
        }
        CUDA_CHECK(cudaMallocHost(reinterpret_cast<void**>(&s->host_table), table));
        CUDA_CHECK(cudaEventCreateWithFlags(&s->table_uploaded, cudaEventDisableTiming));
        // until the first request the table reads as the whole of the smallest image of the format (1 x 1, or a 2 x 2
        // YUV frame) at offset 0 of the staging buffer
        const int side = cfg.pixel_format == graph::ImageResize::kInterleaved ? 1 : 2;
        for (int i = 0; i < t->num(); ++i) {
            b200_image_crop_entry_t& e = s->host_table[i];
            e.r.offset = 0; e.r.h = e.r.w = side; e.r.rh = H; e.r.rw = W; e.r.top = e.r.left = 0;
            e.frame_h = e.frame_w = side; e.box_top = e.box_left = 0;
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

// "" for the whole batch, " slots [first, first + k) of" otherwise: the setters' messages name the slots they fill
static std::string slots_of(int first, int k, int n) {
    return first == 0 && k == n ? std::string()
                                : " slots [" + std::to_string(first) + ", " + std::to_string(first + k) + ") of";
}

static Status slot_range(const std::string& in_name, int first, int k, int n) {
    if (first < 0 || k < 1 || first + k > n)
        return Status::ANAKINFAIL("input " + in_name + ": slots [" + std::to_string(first) + ", " +
                                  std::to_string(first + k) + ") outside its batch of " + std::to_string(n));
    return Status::OK();
}

Status NetCore::set_input(const std::string& in_name, const float* host, size_t count) {
    DTensor* t = get_in(in_name);
    return set_input_slots(in_name, host, count, 0, t ? t->num() : 0);
}

Status NetCore::set_input_slots(const std::string& in_name, const float* host, size_t count, int first, int k) {
    if (!host) return Status::ANAKINFAIL("null argument");
    DTensor* t = get_in(in_name);
    if (!t) return Status::ANAKINFAIL("no input " + in_name);
    if (t->is_image()) return Status::ANAKINFAIL("input " + in_name + " is an image input: use anakin_net_set_input_image");
    Status st = slot_range(in_name, first, k, t->num());
    if (!st) return st;
    const size_t image = t->storage_bytes() / t->num();
    if (count * sizeof(float) != k * image)
        return Status::ANAKINFAIL("input element count does not match" + slots_of(first, k, t->num()) +
                                  " the input tensor");
    cudaSetDevice(_device);
    cudaError_t e = cudaMemcpyAsync(static_cast<char*>(t->mutable_data()) + first * image, host, k * image,
                                    cudaMemcpyHostToDevice, _stream);
    return e == cudaSuccess ? Status::OK() : Status::ANAKINFAIL(cudaGetErrorString(e));
}

Status NetCore::set_input_image(const std::string& in_name, const uint8_t* host, size_t bytes) {
    DTensor* t = get_in(in_name);
    return set_input_image_slots(in_name, host, bytes, 0, t ? t->num() : 0);
}

Status NetCore::set_input_image_slots(const std::string& in_name, const uint8_t* host, size_t bytes, int first, int k) {
    if (!host) return Status::ANAKINFAIL("null argument");
    DTensor* t = get_in(in_name);
    if (!t) return Status::ANAKINFAIL("no input " + in_name);
    if (!t->is_image()) return Status::ANAKINFAIL("input " + in_name + " is not an image input");
    if (resizes_input(in_name))
        return Status::ANAKINFAIL("input " + in_name + " resizes images on the GPU: use anakin_net_set_input_images");
    Status st = slot_range(in_name, first, k, t->num());
    if (!st) return st;
    const size_t image = t->storage_bytes() / t->num();
    if (bytes != k * image)
        return Status::ANAKINFAIL("image of " + std::to_string(bytes) + " bytes," + slots_of(first, k, t->num()) +
                                  " input " + in_name + (first == 0 && k == t->num() ? " holds " : " hold ") +
                                  std::to_string(k * image));
    cudaSetDevice(_device);
    cudaError_t e = cudaMemcpyAsync(static_cast<uint8_t*>(t->mutable_data()) + first * image, host, bytes,
                                    cudaMemcpyHostToDevice, _stream);
    return e == cudaSuccess ? Status::OK() : Status::ANAKINFAIL(cudaGetErrorString(e));
}

Status NetCore::set_input_images(const std::string& in_name, const uint8_t* pixels, size_t bytes, const int32_t* hw,
                                 size_t count) {
    auto it = _resize.find(in_name);
    if (it != _resize.end() && pixels && hw && count != static_cast<size_t>(it->second->desc.n))
        return Status::ANAKINFAIL("set_input_images(" + in_name + "): " + std::to_string(count) + " images, the batch is " +
                                  std::to_string(it->second->desc.n));
    return set_input_images_slots(in_name, pixels, bytes, hw, count, 0);
}

// The crop table of a request of `frame_count` frames (hw) whose pixels start `base` bytes into the staging memory,
// and of its `count` boxes (int32 [count][5]), after every check of the request: frame sizes, boxes, geometry, the
// pixel bytes. boxes == null is an images request: one whole-frame box per image, and messages that name images.
Status NetCore::crop_table(const std::string& in_name, const ImageResizeState& s, size_t bytes, const int32_t* hw,
                           size_t frame_count, const int32_t* boxes, size_t count, size_t base,
                           b200_image_crop_entry_t* tab) const {
    const std::string what = std::string(boxes ? "set_input_crops(" : "set_input_images(") + in_name + "): ";
    auto size_of = [](int32_t h, int32_t w) { return std::to_string(h) + " x " + std::to_string(w); };
    std::vector<int64_t> offset(frame_count);
    size_t total = 0;
    for (size_t i = 0; i < frame_count; ++i) {
        const int32_t h = hw[2 * i], w = hw[2 * i + 1];
        const std::string which = what + (boxes ? "frame " : "image ") + std::to_string(i) + " is " + size_of(h, w);
        if (h < 1 || h > s.cfg.max_h || w < 1 || w > s.cfg.max_w)
            return Status::ANAKINFAIL(which + ", outside 1..max (" + size_of(s.cfg.max_h, s.cfg.max_w) + ")");
        if (s.cfg.pixel_format != graph::ImageResize::kInterleaved && ((h | w) & 1))
            return Status::ANAKINFAIL(which + ": " + pixel_format_name(s.cfg.pixel_format) +
                                      " frames need an even height and width");
        offset[i] = static_cast<int64_t>(base + total);
        total += image_bytes(s, h, w);
    }
    for (size_t j = 0; j < count; ++j) {
        int32_t whole[5] = {static_cast<int32_t>(j), 0, 0, 0, 0};
        if (!boxes) { whole[3] = hw[2 * j]; whole[4] = hw[2 * j + 1]; }
        const int32_t* b = boxes ? boxes + 5 * j : whole;
        const int32_t f = b[0], top = b[1], left = b[2], bh = b[3], bw = b[4];
        const std::string which =
            boxes ? what + "box " + std::to_string(j) + " (frame " + std::to_string(f) + ", top " + std::to_string(top) +
                        ", left " + std::to_string(left) + ", " + size_of(bh, bw) + ")"
                  : what + "image " + std::to_string(j) + " is " + size_of(bh, bw);
        if (f < 0 || static_cast<size_t>(f) >= frame_count)
            return Status::ANAKINFAIL(which + ": no frame " + std::to_string(f) + " among the request's " +
                                      std::to_string(frame_count));
        const int32_t h = hw[2 * f], w = hw[2 * f + 1];
        if (top < 0 || left < 0 || bh < 1 || bw < 1 || top > h - bh || left > w - bw)
            return Status::ANAKINFAIL(which + " is not inside frame " + std::to_string(f) + " (" + size_of(h, w) + ")");
        b200_image_crop_entry_t& e = tab[j];
        if (b200_image_resize_geometry_ex(bh, bw, s.cfg.resize_short, s.desc.out_h, s.desc.out_w, s.cfg.filter,
                                          &e.r.rh, &e.r.rw, &e.r.top, &e.r.left) != B200_SUCCESS)
            return Status::ANAKINFAIL(which + ": no valid resize geometry for resize_short " +
                                      std::to_string(s.cfg.resize_short));
        e.r.offset = offset[f];
        e.r.h = bh; e.r.w = bw;
        e.frame_h = h; e.frame_w = w;
        e.box_top = top; e.box_left = left;
    }
    if (bytes != total)
        return Status::ANAKINFAIL(what + std::to_string(bytes) + " pixel bytes, the sizes need " + std::to_string(total));
    return Status::OK();
}

// The resizing input's state, or the refusal of an input that is not one
static Status resize_state(const std::map<std::string, std::unique_ptr<NetCore::ImageResizeState>>& resize,
                           NetCore::DTensor* t, const std::string& in_name, const NetCore::ImageResizeState** s) {
    auto it = resize.find(in_name);
    if (it != resize.end()) { *s = it->second.get(); return Status::OK(); }
    if (!t) return Status::ANAKINFAIL("no input " + in_name);
    return Status::ANAKINFAIL("input " + in_name + (t->is_image() ? " is a fixed-size image input (no on-device resize): use set_input_image"
                                                                   : " is not an image input"));
}

// The counts of a request: boxes within the batch, 1 <= frames <= boxes (an images request: frames = boxes = count)
static Status request_counts(const std::string& in_name, const NetCore::ImageResizeState& s, bool crops,
                             size_t frame_count, size_t count) {
    const std::string what = std::string(crops ? "set_input_crops(" : "set_input_images(") + in_name + "): ";
    if (count < 1 || count > static_cast<size_t>(s.desc.n))
        return Status::ANAKINFAIL(what + std::to_string(count) + (crops ? " boxes" : " images") + ", the batch is " +
                                  std::to_string(s.desc.n));
    if (frame_count < 1 || frame_count > count)
        return Status::ANAKINFAIL(what + std::to_string(frame_count) + " frames for " + std::to_string(count) +
                                  " boxes: a request needs 1 to (boxes) frames");
    return Status::OK();
}

static std::string null_arrays(const std::string& in_name, bool crops) {
    return crops ? "set_input_crops(" + in_name + "): null frames, sizes or boxes"
                 : "set_input_images(" + in_name + "): null pixels or sizes";
}

Status NetCore::check_crops(const std::string& in_name, bool crops, size_t bytes, const int32_t* hw,
                            size_t frame_count, const int32_t* boxes, size_t count) const {
    const ImageResizeState* s = nullptr;
    auto t = _node_tensor.find(in_name);
    Status st = resize_state(_resize, t == _node_tensor.end() ? nullptr : t->second, in_name, &s);
    if (!st) return st;
    if (!hw || (crops && !boxes)) return Status::ANAKINFAIL(null_arrays(in_name, crops));
    st = request_counts(in_name, *s, crops, frame_count, count);
    if (!st) return st;
    std::vector<b200_image_crop_entry_t> tab(count);
    return crop_table(in_name, *s, bytes, hw, frame_count, boxes, count, 0, tab.data());
}

Status NetCore::check_input_images(const std::string& in_name, size_t bytes, const int32_t* hw, size_t count) const {
    return check_crops(in_name, false, bytes, hw, count, nullptr, count);
}

Status NetCore::check_input_crops(const std::string& in_name, size_t bytes, const int32_t* hw, size_t frame_count,
                                  const int32_t* boxes, size_t count) const {
    return check_crops(in_name, true, bytes, hw, frame_count, boxes, count);
}

Status NetCore::stage_crops(const std::string& in_name, bool crops, const uint8_t* frames, size_t bytes,
                            const int32_t* hw, size_t frame_count, const int32_t* boxes, size_t count, int first) {
    const ImageResizeState* cs = nullptr;
    Status st = resize_state(_resize, get_in(in_name), in_name, &cs);
    if (!st) return st;
    ImageResizeState& s = *_resize[in_name];
    if (!frames || !hw || (crops && !boxes)) return Status::ANAKINFAIL(null_arrays(in_name, crops));
    const int n = s.desc.n;
    st = slot_range(in_name, first, static_cast<int>(std::min<size_t>(count, n + 1)), n);
    if (!st) return st;
    st = request_counts(in_name, s, crops, frame_count, count);
    if (!st) return st;
    // every slot's staging holds one frame of up to max_h x max_w: a request's frames (no more than its boxes) fit from
    // its first slot on
    const size_t base = static_cast<size_t>(first) * slot_bytes(s);
    std::vector<b200_image_crop_entry_t> tab(n - first);
    st = crop_table(in_name, s, bytes, hw, frame_count, boxes, count, base, tab.data());
    if (!st) return st;
    for (size_t i = count; i < tab.size(); ++i) tab[i] = tab[count - 1];
    cudaSetDevice(_device);
    // the pinned table may still be in flight from the previous request
    CUDA_CHECK(cudaEventSynchronize(s.table_uploaded));
    memcpy(s.host_table + first, tab.data(), tab.size() * sizeof(b200_image_crop_entry_t));
    CUDA_CHECK(cudaMemcpyAsync(static_cast<b200_image_crop_entry_t*>(s.table.ptr) + first, s.host_table + first,
                               tab.size() * sizeof(b200_image_crop_entry_t), cudaMemcpyHostToDevice, _stream));
    CUDA_CHECK(cudaEventRecord(s.table_uploaded, _stream));
    CUDA_CHECK(cudaMemcpyAsync(static_cast<uint8_t*>(s.staging.ptr) + base, frames, bytes, cudaMemcpyHostToDevice,
                               _stream));
    return Status::OK();
}

Status NetCore::set_input_images_slots(const std::string& in_name, const uint8_t* pixels, size_t bytes,
                                       const int32_t* hw, size_t count, int first) {
    return stage_crops(in_name, false, pixels, bytes, hw, count, nullptr, count, first);
}

Status NetCore::set_input_crops(const std::string& in_name, const uint8_t* frames, size_t bytes, const int32_t* hw,
                                size_t frame_count, const int32_t* boxes, size_t count) {
    auto it = _resize.find(in_name);
    if (it != _resize.end() && frames && hw && boxes && count != static_cast<size_t>(it->second->desc.n))
        return Status::ANAKINFAIL("set_input_crops(" + in_name + "): " + std::to_string(count) + " boxes, the batch is " +
                                  std::to_string(it->second->desc.n));
    return set_input_crops_slots(in_name, frames, bytes, hw, frame_count, boxes, count, 0);
}

Status NetCore::set_input_crops_slots(const std::string& in_name, const uint8_t* frames, size_t bytes,
                                      const int32_t* hw, size_t frame_count, const int32_t* boxes, size_t count,
                                      int first) {
    return stage_crops(in_name, true, frames, bytes, hw, frame_count, boxes, count, first);
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
    if (_calib.on && precision != Precision::FP32)
        return Status::ANAKINFAIL("calibration statistics need an FP32 net: an INT8 table is built from the fp32 "
                                  "activations, and an FP16 or INT8 net does not compute them");
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
    _calib.slots.clear(); _input_taps = Taps();
    _exports.clear();
    _in_names = graph.get_ins();
    _out_names = graph.get_outs();

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
        // in an INT8 Net: INT8 where the op has an INT8 operator and the node is not marked otherwise (operators.cpp)
        const bool int8 = ops::has_int8(node->op) && (node->bit_type == AK_INT8 || node->bit_type == AK_INVALID);
        const Precision p = precision == Precision::INT8 && !int8 ? Precision::FP32 : precision;
        ops::OperatorBase* raw = ops::create_operator(node->op, p);
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
    // An INT8 Axpy reads an fp32 gate only from the fused SqueezeExcite: the un-fused gate chain would be an fp32
    // island inside the INT8 net, which this build does not run
    if (precision == Precision::INT8) {
        for (auto& b : built) {
            if ((b.node->op != "Axpy" && b.node->op != "AxpyRelu") || !b.int8 || b.node->ins.empty()) continue;
            const std::string& g = b.node->ins[0];
            if (graph[g] && graph[g]->op != "SqueezeExcite")
                return Status::ANAKINFAIL("node " + b.node->name + " (" + b.node->op + "): its gate " + g + " (op " +
                                          graph[g]->op + ") is not a fused SqueezeExcite; an fp32 gate chain inside an "
                                          "INT8 net is not supported");
        }
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
    // YUV frames are converted to RGB by the resize: only a 3-channel image input with on-device resize takes them
    for (auto& b : built) {
        const int f = b.node->op == "Input" ? graph::node_image_pixel_format(*b.node) : graph::ImageResize::kInterleaved;
        if (f == graph::ImageResize::kInterleaved || f < 0) continue;   // a bad value fails with the resize attributes
        const std::string& nm = b.node->name;
        graph::ImageResize cfg;
        if (graph::node_image_resize(*b.node, &cfg) != 1)
            return Status::ANAKINFAIL("input " + nm + ": image_pixel_format " + std::to_string(f) +
                                      " needs an image input with on-device resize (set_input_image_resize)");
        const PTuple<int> shape = b.node->get_attr_or<PTuple<int>>("input_shape", {});
        const int c = shape.size() >= 2 ? shape[1] : 1;
        if (c != 3 || cfg.max_h < 2 || cfg.max_w < 2)
            return Status::ANAKINFAIL("input " + nm + ": " + pixel_format_name(f) +
                                      " frames need 3 channels and max_h, max_w >= 2, the input has " +
                                      std::to_string(c) + " channels and max " + std::to_string(cfg.max_h) + " x " +
                                      std::to_string(cfg.max_w));
    }
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
        if (b.node->op == "Input" || b.op->output_fp32()) {
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

    // ---- 3. shapes for every edge; the non-alias ops in graph order are the exec entries. Memory is planned before
    // init: conv plans bake buffer addresses into their tensor maps (weights packed once per device, see WeightArena)
    for (auto& b : built) {
        ExecOp e;
        e.name = b.node->name;
        e.op_name = b.node->op;
        e.op = b.op;
        for (auto& in : b.node->ins) e.ins.push_back(_node_tensor[in]);
        e.outs.push_back(_node_tensor[b.node->name]);
        Status st = b.op->InferShape(e.ins, e.outs);
        if (!st) return Status::ANAKINFAIL("InferShape(" + e.name + "): " + st.info());
        if (!b.op->is_alias()) _exec.push_back(e);
    }
    plan_side_ops();
    plan_activation_memory();
    for (auto& kv : _owned)
        if (kv.second->storage_bytes())
            CUDA_CHECK(cudaMemsetAsync(kv.second->mutable_data(), 0, kv.second->storage_bytes(), _stream));
    for (auto& e : _exec) {
        Status st = e.op->Init(e.side ? _side_ctx : _ctx, e.ins, e.outs);
        if (!st) return Status::ANAKINFAIL("Init(" + e.name + "): " + st.info());
    }
    plan_fused_head();
    Status rst = plan_image_resize(graph);
    if (!rst) return rst;
    if (_calib.on) {
        Status cst = plan_calib_stats();
        if (!cst) return cst;
    }
    Status xst = plan_exports(graph);
    if (!xst) return xst;
    // weight uploads and the zero fills above used synchronous copies / this stream: nothing is pending after this
    CUDA_CHECK(cudaStreamSynchronize(_stream));
    CUDA_CHECK(cudaDeviceSynchronize());
    return Status::OK();
}

// Classifier head: global pooling -> inner product -> softmax, three dependent launches of a few microseconds each at
// the end of every request (saber_pooling.cu, saber_fc.cu, saber_softmax.cu), run as one FusedHeadOp.
void NetCore::plan_fused_head() {
    // Pooling + inner product are one cluster launch, the softmax a second one. (A first version that split the
    // reduction dimension over the CTAs and combined them with integer atomics took 37 us on ResNet-50 INT8 b8 -- slower
    // than the ~17 us of the three ops -- and was replaced.)
    for (size_t i = 0; i + 2 < _exec.size(); ++i) {
        ExecOp &ep = _exec[i], &ef = _exec[i + 1], &es = _exec[i + 2];
        int is_max = 0, axis = 0;
        b200_fc_stream_desc_t fd;
        const void* w; const float *bias, *scale;
        if (!head_chain(ep, ef, es)) continue;
        if (!ep.op->head_pool_info(&is_max) || !ef.op->head_fc_info(&fd, &w, &bias, &scale) || !es.op->head_softmax_info(&axis)) continue;
        DTensor *in = ep.ins[0], *pooled = ep.outs[0], *logits = ef.outs[0], *prob = es.outs[0];
        if (in->get_layout() != Layout_NHWC || pooled->get_layout() != Layout_NHWC || in->get_dtype() != pooled->get_dtype()) continue;
        if (pooled->height() != 1 || pooled->width() != 1 || fd.m > 8 || fd.k != pooled->channel_stored() ||
            fd.in_dtype != pooled->get_dtype() || fd.out_dtype != B200_FLOAT || logits->get_dtype() != AK_FLOAT ||
            prob->get_dtype() != AK_FLOAT || axis != 1 || logits->height() != 1 || logits->width() != 1)
            continue;
        if (fd.math != B200_MATH_I8) continue;                           // float heads keep the three ops
        auto head = std::make_shared<FusedHeadOp>();
        head->desc.fc = fd;
        head->desc.hw = in->height() * in->width();
        head->desc.pool_max = is_max;
        head->desc.ldp = prob->channel_stored();
        head->w = w; head->bias = bias; head->scale = scale;
        head->in = in; head->pooled = pooled; head->logits = logits; head->prob = prob;
        if (head->barrier.re_alloc(b200_head_workspace_bytes(&head->desc), false) != SaberSuccess) return;  // zeroed
        ep.op = head;
        ep.head = 1; ef.head = 2; es.head = 2;
        return;
    }
}

// Three consecutive main-stream ops global pooling -> op reading the pooled rows -> softmax reading its output: the
// chain plan_fused_head may run as one launch. The memory plan, made before the ops are initialised, protects every
// such chain; plan_fused_head fuses at most one, once the initialised ops show that the head kernel can run it.
bool NetCore::head_chain(const ExecOp& ep, const ExecOp& ef, const ExecOp& es) {
    int is_max = 0, axis = 0;
    if (ep.side || ef.side || es.side || ef.wait_side || es.wait_side) return false;
    if (!ep.op->head_pool_info(&is_max) || !es.op->head_softmax_info(&axis)) return false;
    return !ef.ins.empty() && ef.ins[0] == ep.outs[0] && !es.ins.empty() && es.ins[0] == ef.outs[0];
}

// Off-chain ops (the reference's ParallScheduler gives such nodes their own lane / stream,
// framework/graph/llvm/scheduler.cpp + net.cpp:430-444,480-492): an op whose result is not read by the op that
// follows it -- the projection shortcut `resXa_branch1`, read only by `branch2c` three ops later -- runs on a second
// stream, forked after the ops before it and joined in front of its first reader. Inside the captured CUDA graph
// this is a parallel branch, so the shortcut convolution leaves the critical path of the request.
void NetCore::plan_side_ops() {
    std::set<DTensor*> outs;
    for (auto& n : _out_names) outs.insert(_node_tensor[n]);
    int busy_until = -1;   // one side stream: do not stack side ops
    for (size_t i = 0; i + 2 < _exec.size(); ++i) {
        ExecOp& e = _exec[i];
        if (static_cast<int>(i) <= busy_until || e.outs.size() != 1 || outs.count(e.outs[0])) continue;
        if (e.op_name.compare(0, 4, "Conv") != 0) continue;
        int first_reader = -1;
        for (size_t j = i + 1; j < _exec.size() && first_reader < 0; ++j)
            for (DTensor* t : _exec[j].ins) if (t == e.outs[0]) first_reader = static_cast<int>(j);
        if (first_reader <= static_cast<int>(i) + 1) continue;
        // nothing in between may touch the tensors this op writes or reads-and-shares (in-place ops do not exist here)
        e.side = true;
        _exec[first_reader].wait_side = true;
        busy_until = first_reader;
    }
}

// The entry that joins side op i: the next one that waits for the side stream (side ops do not overlap); -1 for an
// entry on the main stream.
int NetCore::side_join(size_t i) const {
    for (size_t j = i + 1; _exec[i].side && j < _exec.size(); ++j)
        if (_exec[j].wait_side) return static_cast<int>(j);
    return -1;
}

// Activation memory (the reference's MemoryScheduler pass + Net::init_memory, framework/graph/llvm/optimizer/
// memory_scheduler.cpp, framework/core/net/net.cpp:812-898): an edge tensor is live from the op that writes it to
// the last op that reads it (through alias nodes); tensors whose live ranges do not overlap share one buffer.
// Greedy best-fit over the execution order. Kept out of the pool: graph inputs / outputs (the user reads and
// writes them between predictions) and tensors with channel padding (their never-written padding must stay 0).
void NetCore::plan_activation_memory() {
    _act_bytes = 0;
    _act_bytes_unshared = 0;
    for (auto& kv : _owned) _act_bytes_unshared += kv.second->storage_bytes();
    if (!_share_activations) { _act_bytes = _act_bytes_unshared; return; }
    std::map<DTensor*, int> def, last;
    for (size_t i = 0; i < _exec.size(); ++i) {
        for (DTensor* t : _exec[i].outs) if (!def.count(t)) def[t] = static_cast<int>(i);
        // a side-stream op may still be reading its inputs until the op that joins it
        const int until = std::max(side_join(i), static_cast<int>(i));
        for (DTensor* t : _exec[i].ins) last[t] = std::max(last.count(t) ? last[t] : 0, until);
    }
    // A fused head reads its input and writes the pooled rows, the logits and the probabilities in any of its three
    // steps (one cluster's logits may be stored while another cluster still pools the input): the chain is one step
    for (size_t i = 0; i + 2 < _exec.size(); ++i) {
        if (!head_chain(_exec[i], _exec[i + 1], _exec[i + 2])) continue;
        const int p = static_cast<int>(i);
        last[_exec[i].ins[0]] = std::max(last[_exec[i].ins[0]], p + 2);
        for (size_t k = 0; k < 3; ++k) {
            DTensor* t = _exec[i + k].outs[0];
            def[t] = p;
            last[t] = std::max(last.count(t) ? last[t] : 0, p + 2);
        }
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

// Calibration statistics slots, taps (see Taps): the graph inputs, then the output of every exec entry in exec order --
// the tensors the calibration table names.
Status NetCore::plan_calib_stats() {
    auto add = [&](const std::string& name, DTensor* t) -> Status {
        if (!t || t->get_dtype() != AK_FLOAT || t->num() < 1)
            return Status::ANAKINFAIL("calibration statistics: the tensor of " + name + " is not an fp32 tensor");
        CalibSlot s;
        s.name = name;
        s.t = t;
        if (t->get_layout() == Layout_NHWC) {
            s.rows = static_cast<int64_t>(t->num()) * t->height() * t->width();
            s.c = t->channel();
            s.ld = t->channel_stored();
        } else {   // the unpadded NCHW graph input
            s.rows = t->num();
            s.c = s.ld = static_cast<int32_t>(t->storage_bytes() / sizeof(float) / t->num());
        }
        _calib.slots.push_back(s);
        return Status::OK();
    };
    for (auto& nm : _in_names) {
        DTensor* t = _node_tensor[nm];
        if (t && t->is_image())
            return Status::ANAKINFAIL("calibration statistics need an fp32 graph input: " + nm +
                                      " is an 8-bit image input, whose normalised fp32 tensor is never materialised");
        _input_taps.calib.push_back(static_cast<int>(_calib.slots.size()));
        Status st = add(nm, t);
        if (!st) return st;
    }
    for (size_t i = 0; i < _exec.size(); ++i) {
        if (_exec[i].outs.empty()) continue;
        tap_owner(i).taps.calib.push_back(static_cast<int>(_calib.slots.size()));
        Status st = add(_exec[i].name, _exec[i].outs[0]);
        if (!st) return st;
    }
    const size_t n = _calib.slots.size();
    if (_calib.mode.re_alloc(sizeof(int32_t), false) != SaberSuccess ||
        _calib.max_bits.re_alloc(n * sizeof(uint32_t), false) != SaberSuccess ||
        _calib.hist.re_alloc(n * B200_CALIB_BINS * sizeof(uint64_t), false) != SaberSuccess ||
        _calib.thresh.re_alloc(n * sizeof(int32_t), false) != SaberSuccess)
        return Status::ANAKINFAIL("calibration statistics: cannot allocate the statistics of " + std::to_string(n) +
                                  " tensors");
    return calib_reset();
}

Status NetCore::calib_reset() {
    if (!_calib.on || _calib.slots.empty()) return Status::ANAKINFAIL("the net was not created with calibration statistics");
    cudaSetDevice(_device);
    CUDA_CHECK(cudaMemsetAsync(_calib.max_bits.ptr, 0, _calib.max_bits.bytes, _stream));
    CUDA_CHECK(cudaMemsetAsync(_calib.hist.ptr, 0, _calib.hist.bytes, _stream));
    return Status::OK();
}

Status NetCore::calib_set_pass(int pass) {
    if (!_calib.on || _calib.slots.empty()) return Status::ANAKINFAIL("the net was not created with calibration statistics");
    if (pass != 0 && pass != 1) return Status::ANAKINFAIL("calibration pass " + std::to_string(pass) + ": 0 (maxima) or 1 (histograms)");
    cudaSetDevice(_device);
    // (a pageable source is staged before the call returns)
    const int32_t word = pass;
    CUDA_CHECK(cudaMemcpyAsync(_calib.mode.ptr, &word, sizeof(word), cudaMemcpyHostToDevice, _stream));
    return Status::OK();
}

Status NetCore::calib_read(float* max, uint64_t* hist) {
    if (!_calib.on || _calib.slots.empty()) return Status::ANAKINFAIL("the net was not created with calibration statistics");
    cudaSetDevice(_device);
    CUDA_CHECK(cudaStreamSynchronize(_stream));
    if (max) {
        std::vector<uint32_t> bits(_calib.slots.size());
        CUDA_CHECK(cudaMemcpy(bits.data(), _calib.max_bits.ptr, bits.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost));
        memcpy(max, bits.data(), bits.size() * sizeof(uint32_t));
    }
    if (hist) CUDA_CHECK(cudaMemcpy(hist, _calib.hist.ptr, _calib.hist.bytes, cudaMemcpyDeviceToHost));
    return Status::OK();
}

Status NetCore::calib_kl(int32_t* thresh) {
    if (!_calib.on || _calib.slots.empty()) return Status::ANAKINFAIL("the net was not created with calibration statistics");
    if (!thresh) return Status::ANAKINFAIL("calib_kl: null output");
    cudaSetDevice(_device);
    const int n = static_cast<int>(_calib.slots.size());
    const int st = b200_calib_kl_run(static_cast<const uint64_t*>(_calib.hist.ptr), n,
                                     static_cast<int32_t*>(_calib.thresh.ptr), nullptr, _stream);
    if (st != B200_SUCCESS) return Status::ANAKINFAIL(std::string("calib_kl: ") + b200_status_string(st));
    CUDA_CHECK(cudaMemcpyAsync(thresh, _calib.thresh.ptr, n * sizeof(int32_t), cudaMemcpyDeviceToHost, _stream));
    CUDA_CHECK(cudaStreamSynchronize(_stream));
    return Status::OK();
}

// Export slots, taps (see Taps): nothing has to be pinned. The exported tensor keeps its dtype: an Output node on the
// edge would make it fp32 (NetCore::init, step 2), re-quantise its INT8 readers and break the fused head, changing the
// probabilities served next to the export.
Status NetCore::plan_exports(GraphCore& graph) {
    std::set<std::string> seen;
    std::set<DTensor*> ins, outs;
    for (auto& nm : _in_names) ins.insert(_node_tensor[nm]);
    for (auto& nm : _out_names) outs.insert(_node_tensor[nm]);
    for (auto& nm : _export_names) {
        const std::string what = "export " + nm + ": ";
        auto it = _node_tensor.find(nm);
        NodePtr node = graph[nm];
        if (!node || it == _node_tensor.end() || !it->second)
            return Status::ANAKINFAIL(what + "no node of that name in the optimised graph (the value of a fused chain "
                                      "is exported under the fused node's name)");
        if (!seen.insert(nm).second) return Status::ANAKINFAIL(what + "registered twice");
        DTensor* t = it->second;
        if (node->op == "Input" || ins.count(t)) return Status::ANAKINFAIL(what + "is a graph input");
        if (outs.count(t)) return Status::ANAKINFAIL(what + "is a graph output, already served by get_out");
        int at = -1;
        for (size_t i = 0; i < _exec.size(); ++i)
            if (!_exec[i].outs.empty() && _exec[i].outs[0] == t) at = static_cast<int>(i);
        if (at < 0) return Status::ANAKINFAIL(what + "no launched op writes its tensor");
        if (t->get_layout() != Layout_NHWC || t->num() < 1)
            return Status::ANAKINFAIL(what + "its tensor is not an NHWC edge tensor");
        const DataType dt = t->get_dtype();
        if (dt != AK_FLOAT && dt != AK_HALF && dt != AK_INT8 && dt != AK_UINT8)
            return Status::ANAKINFAIL(what + "its tensor's dtype cannot be exported");
        if ((dt == AK_INT8 || dt == AK_UINT8) && t->get_scale().empty())
            return Status::ANAKINFAIL(what + "its 8-bit tensor has no calibrated scale");
        auto s = std::make_unique<ExportSlot>();
        s->name = nm;
        s->t = t;
        s->nchw[0] = t->num(); s->nchw[1] = t->channel(); s->nchw[2] = t->height(); s->nchw[3] = t->width();
        const size_t bytes = static_cast<size_t>(s->nchw[0]) * s->nchw[1] * s->nchw[2] * s->nchw[3] * sizeof(float);
        if (s->buf.re_alloc(bytes, false) != SaberSuccess)
            return Status::ANAKINFAIL(what + "cannot allocate " + std::to_string(bytes) + " bytes");
        tap_owner(at).taps.exports.push_back(static_cast<int>(_exports.size()));
        _exports.push_back(std::move(s));
    }
    return Status::OK();
}

// The entry whose launch writes entry i's output: i itself, or the fused head's pooling entry for an entry it covers.
NetCore::ExecOp& NetCore::tap_owner(size_t i) {
    while (i > 0 && _exec[i].head == 2) --i;
    return _exec[i];
}

void NetCore::launch_taps(const Taps& taps, cudaStream_t stream) {
    for (int i : taps.calib) {
        const CalibSlot& s = _calib.slots[i];
        SABER_CHECK(static_cast<SaberStatus>(b200_calib_stats_run(
            static_cast<const float*>(s.t->data()), s.rows, s.c, s.ld, static_cast<const int32_t*>(_calib.mode.ptr),
            static_cast<uint32_t*>(_calib.max_bits.ptr) + i,
            static_cast<uint64_t*>(_calib.hist.ptr) + static_cast<size_t>(i) * B200_CALIB_BINS, stream)));
    }
    for (int i : taps.exports) {
        const ExportSlot& s = *_exports[i];
        const float scale = s.t->get_scale().empty() ? 1.f : s.t->get_scale()[0];
        SABER_CHECK(static_cast<SaberStatus>(b200_export_run(s.t->data(), s.t->get_dtype(), s.nchw[0], s.nchw[2],
                                                             s.nchw[3], s.nchw[1], s.t->channel_stored(), scale,
                                                             static_cast<float*>(s.buf.ptr), stream)));
    }
}

int NetCore::export_index(const std::string& name) const {
    for (size_t i = 0; i < _exports.size(); ++i)
        if (_exports[i]->name == name) return static_cast<int>(i);
    return -1;
}

size_t NetCore::export_elements(size_t i) const {
    const int32_t* d = _exports[i]->nchw;
    return static_cast<size_t>(d[0]) * d[1] * d[2] * d[3];
}

size_t NetCore::export_bytes() const {
    size_t b = 0;
    for (size_t i = 0; i < _exports.size(); ++i) b += export_elements(i) * sizeof(float);
    return b;
}

Status NetCore::read_export(size_t i, float* host, size_t count) {
    if (i >= _exports.size()) return Status::ANAKINFAIL("read_export: no export " + std::to_string(i));
    if (!host) return Status::ANAKINFAIL("read_export(" + _exports[i]->name + "): null output");
    const size_t need = export_elements(i);
    if (count != need)
        return Status::ANAKINFAIL("read_export(" + _exports[i]->name + "): " + std::to_string(count) +
                                  " floats, the export holds " + std::to_string(need));
    cudaSetDevice(_device);
    CUDA_CHECK(cudaMemcpyAsync(host, _exports[i]->buf.ptr, need * sizeof(float), cudaMemcpyDeviceToHost, _stream));
    CUDA_CHECK(cudaStreamSynchronize(_stream));
    return Status::OK();
}

// Launches exec entry e's op on ctx's stream; an entry covered by the fused head launches nothing.
void NetCore::launch(ExecOp& e, Context<NV>& ctx) {
    if (e.head != 2) (*e.op)(ctx, e.ins, e.outs);
}

void NetCore::run_eager() {
    launch_taps(_input_taps, _stream);
    for (auto& e : _exec) {
        if (e.wait_side) CUDA_CHECK(cudaStreamWaitEvent(_stream, _join_ev, 0));
        if (e.side) {
            CUDA_CHECK(cudaEventRecord(_fork_ev, _stream));
            CUDA_CHECK(cudaStreamWaitEvent(_side_stream, _fork_ev, 0));
        }
        Context<NV>& ctx = e.side ? _side_ctx : _ctx;
        launch(e, ctx);
        launch_taps(e.taps, ctx.get_compute_stream());
        if (e.side) CUDA_CHECK(cudaEventRecord(_join_ev, _side_stream));
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
    for (int it = 0; it < iters + 1; ++it) {  // first pass is a warm-up
        for (size_t i = 0; i < n; ++i) {
            CUDA_CHECK(cudaEventRecord(ev[2 * i], _stream));
            for (int r = 0; r < reps; ++r) launch(_exec[i], _ctx);   // all on one stream here
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

std::vector<NetCore::ScheduleEntry> NetCore::get_schedule() const {
    std::vector<ScheduleEntry> v;
    for (size_t i = 0; i < _exec.size(); ++i) v.push_back({side_join(i), _exec[i].head});
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
    size_t view_count = 0;   // floats of one *_view result of this thread's Net
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
        if (!init_failed && !_io_planned) {
            // registered names that are not graph outputs, then the interior edges, become every Net's exports
            const std::vector<std::string>& gouts = _graph->get_outs();
            std::vector<std::string> outs;
            for (auto& o : _outputs)
                (std::find(gouts.begin(), gouts.end(), o) != gouts.end() ? outs : _exports).push_back(o);
            for (auto& e : _edges) {
                NodePtr b = (*_graph)[e.first];
                if (!e.second.empty() && (!b || std::find(b->outs.begin(), b->outs.end(), e.second) == b->outs.end())) {
                    _init_errors.push_back("register_interior_edges(" + e.first + ", " + e.second + "): no edge " +
                                           e.first + " -> " + e.second + " in the optimised graph");
                    init_failed = true;
                    break;
                }
                _exports.push_back(e.first);
            }
            _outputs = outs;
            _io_planned = true;
        }
        if (!init_failed && _max_delay_us >= 0 && _graph->get_ins().size() != 1) {
            _init_errors.push_back("a batching Worker serves graphs of one input; this graph has " +
                                   std::to_string(_graph->get_ins().size()));
            init_failed = true;
        }
        if (!init_failed) {
            net.register_exports(_exports);
            Status st = net.init(*_graph, _precision, device);
            if (!st) { _init_errors.push_back(st.info()); init_failed = true; }
        }
        if (!init_failed) {
            if (_inputs.empty()) _inputs = net.get_in_names();
            if (_outputs.empty()) _outputs = net.get_out_names();
            view_count = net.get_out(_outputs[0])->storage_bytes() / sizeof(float);
            for (size_t i = 0; i < net.export_count(); ++i) view_count += net.export_elements(i);
            const NetCore::DTensor* in0 = net.get_in(_inputs[0]);
            const int n = in0->num();
            // batching hands out rows: every result must hold one row per slot of the input
            std::string rows;
            for (auto& o : _outputs)
                if (net.get_out(o)->num() != n) rows = "graph output " + o;
            for (size_t i = 0; i < net.export_count(); ++i)
                if (net.export_dims(i)[0] != n) rows = "export " + net.export_name(i);
            if (_max_delay_us >= 0 && !rows.empty()) {
                _init_errors.push_back("a batching Worker needs one row per image: " + rows + " has another batch");
                init_failed = true;
            }
            std::lock_guard<std::mutex> lk2(_mu);
            _view_count = view_count;
            if (!_batch) {   // the same for every thread's Net; written once, read by the serving threads
                _batch = n;
                _image_in = in0->storage_bytes() / n / (in0->is_image() ? 1 : sizeof(float));
                _image_view = view_count / n;
            }
        }
    }
    if (_max_delay_us >= 0) {
        std::string why;
        if (init_failed) {
            std::lock_guard<std::mutex> lk(_graph_mu);
            why = _init_errors.empty() ? "Net init failed" : _init_errors.front();
        }
        serve_batches(net, why);
        return;
    }
    // a thread without a Net still serves the queue, failing every request with the init error: callers blocked in
    // sync_prediction().get() / async_get_result() return instead of waiting forever
    std::string why;
    if (init_failed) {
        std::lock_guard<std::mutex> lk(_graph_mu);
        why = _init_errors.empty() ? "Net init failed" : _init_errors.front();
    }
    while (true) {
        std::shared_ptr<Request> r;
        {
            std::unique_lock<std::mutex> lk(_mu);
            _cv.wait(lk, [this] { return _stop || !_tasks.empty(); });
            if (_stop && _tasks.empty()) return;
            r = _tasks.front();
            _tasks.pop_front();
        }
        try {
            if (init_failed) throw std::runtime_error("Worker: " + why);
            // with exports, a view result is graph output 0 and every export: a buffer of another size is refused
            // before anything runs
            const size_t nx = net.export_count();
            if (r->out && nx && r->out_count != view_count)
                throw std::runtime_error("Worker: out_count " + std::to_string(r->out_count) + ", the result is " +
                                         std::to_string(view_count) + " floats (graph output 0 and " +
                                         std::to_string(nx) + " exports)");
            Status st = stage(net, *r);
            if (!st) throw std::runtime_error(std::string("Worker: ") + st.info());
            net.prediction();
            // a view gets graph output 0 (at most out_count floats), then every export, back to back; otherwise each
            // graph output, then each export, goes to a vector of its own
            std::vector<std::pair<const void*, size_t>> parts;   // device source, floats
            for (size_t i = 0; i < (r->out ? 1 : _outputs.size()); ++i) {
                NetCore::DTensor* d = net.get_out(_outputs[i]);
                parts.push_back({d->data(), d->storage_bytes() / sizeof(float)});
            }
            if (r->out) parts[0].second = std::min(parts[0].second, r->out_count);
            for (size_t i = 0; i < nx; ++i) parts.push_back({net.export_device_ptr(i), net.export_elements(i)});
            Result outs;
            float* at = r->out;
            for (auto& p : parts) {
                if (!r->out) { outs.emplace_back(p.second); at = outs.back().data(); }
                CUDA_CHECK(cudaMemcpyAsync(at, p.first, p.second * sizeof(float), cudaMemcpyDeviceToHost, net.stream()));
                at += p.second;
            }
            net.sync();
            r->done.set_value(std::move(outs));
        } catch (...) {
            r->done.set_exception(std::current_exception());
        }
    }
}

// Checks the request's form against the first input's kind -- the marker decides, not the byte count.
Status WorkerCore::check_form(NetCore& net, const Request& r) const {
    if (_inputs.empty()) return Status::ANAKINFAIL("the model has no input");
    const std::string& in0 = _inputs[0];
    const NetCore::DTensor* t = net.get_in(in0);
    const bool image = r.form != Request::FP32, resize = r.form == Request::IMAGES || r.form == Request::CROPS;
    if (t && image != t->is_image())
        return Status::ANAKINFAIL("input " + in0 + (image ? " is an fp32 input, not an image input"
                                                          : " is an image input: use the image prediction calls"));
    if (t && image && resize != net.resizes_input(in0))
        return Status::ANAKINFAIL("input " + in0 + (resize ? " is a fixed-size image input: use the *_prediction_image calls"
                                                           : " resizes on the GPU: use the *_prediction_images calls"));
    return Status::OK();
}

// Checks the request's form, then stages it through the NetCore setter of that form.
Status WorkerCore::stage(NetCore& net, const Request& r) const {
    Status st = check_form(net, r);
    if (!st) return st;
    const std::string& in0 = _inputs[0];
    const bool image = r.form != Request::FP32;
    const auto* bytes = static_cast<const uint8_t*>(r.in);
    if (r.form == Request::CROPS) return net.set_input_crops(in0, bytes, r.size, r.hw, r.frame_count, r.boxes, r.count);
    if (r.form == Request::IMAGES) return net.set_input_images(in0, bytes, r.size, r.hw, r.count);
    if (image) return net.set_input_image(in0, bytes, r.size);
    if (r.in) return net.set_input(in0, static_cast<const float*>(r.in), r.size);
    if (r.ins.size() < _inputs.size())
        return Status::ANAKINFAIL(std::to_string(r.ins.size()) + " input vectors, the model has " +
                                  std::to_string(_inputs.size()) + " inputs");
    for (size_t i = 0; i < _inputs.size(); ++i) {
        Status st = net.set_input(_inputs[i], r.ins[i].data(), r.ins[i].size());
        if (!st) return st;
    }
    return Status::OK();
}

// The one way onto the queue; an async request's future goes to _async_que in the same critical section, so results
// come back in submission order.
std::future<WorkerCore::Result> WorkerCore::enqueue(std::shared_ptr<Request> r, bool async) {
    std::future<Result> fut = r->done.get_future();
    if (_max_delay_us >= 0) r->arrive_us = now_us();
    {
        std::lock_guard<std::mutex> lk(_mu);
        _tasks.push_back(std::move(r));
        if (async) _async_que.push_back(std::move(fut));
    }
    // batching: the gathering thread waits on _cv as well, and must see every arrival
    if (_max_delay_us >= 0) _cv.notify_all();
    else _cv.notify_one();
    return fut;
}

// ---------------------------------------------------------------------------------------------
// Batching

BatchPlan plan_batch(const int* sizes, const int64_t* arrive_us, size_t n, int batch, int64_t max_delay_us,
                     int64_t now_us) {
    BatchPlan p;
    if (n == 0) return p;
    int used = 0;
    while (p.take < n && used + sizes[p.take] <= batch) used += sizes[p.take++];
    p.deadline_us = arrive_us[0] + max_delay_us;
    p.close = used >= batch || p.take < n || now_us >= p.deadline_us;
    return p;
}

int64_t WorkerCore::now_us() {
    return std::chrono::duration_cast<std::chrono::microseconds>(
               std::chrono::steady_clock::now().time_since_epoch()).count();
}

size_t WorkerCore::request_images(const Request& r) const {
    if (r.form == Request::IMAGES || r.form == Request::CROPS) return r.count;
    const size_t n = r.in ? r.size : (r.ins.size() == 1 ? r.ins[0].size() : 0);
    return _image_in && n % _image_in == 0 ? n / _image_in : 0;
}

// Everything a request of a gathered batch is checked for before any request of it is staged.
Status WorkerCore::check_request(NetCore& net, const Request& r, size_t k) const {
    Status st = check_form(net, r);
    if (!st) return st;
    if (r.form == Request::IMAGES || r.form == Request::CROPS) {
        st = r.form == Request::IMAGES ? net.check_input_images(_inputs[0], r.size, r.hw, r.count)
                                       : net.check_input_crops(_inputs[0], r.size, r.hw, r.frame_count, r.boxes, r.count);
        if (!st) return st;
    } else if (k < 1 || k > static_cast<size_t>(_batch)) {
        const bool image = r.form == Request::IMAGE;
        if (!r.in && r.ins.size() != 1)
            return Status::ANAKINFAIL(std::to_string(r.ins.size()) + " input vectors, the model has 1 input");
        const size_t n = r.in ? r.size : r.ins[0].size();
        return Status::ANAKINFAIL("request of " + std::to_string(n) + (image ? " bytes" : " floats") +
                                  ": not 1.." + std::to_string(_batch) + " images of " + std::to_string(_image_in) +
                                  (image ? " bytes" : " floats") + " each");
    }
    if (r.out && r.out_count != k * _image_view)
        return Status::ANAKINFAIL("out_count " + std::to_string(r.out_count) + ", the result of " + std::to_string(k) +
                                  " images is " + std::to_string(k * _image_view) + " floats (" +
                                  std::to_string(_image_view) + " per image: graph output 0 and " +
                                  std::to_string(net.export_count()) + " exports)");
    return Status::OK();
}

Status WorkerCore::stage_slots(NetCore& net, const Request& r, int first, int k) const {
    const std::string& in0 = _inputs[0];
    const auto* bytes = static_cast<const uint8_t*>(r.in);
    if (r.form == Request::IMAGES) return net.set_input_images_slots(in0, bytes, r.size, r.hw, r.count, first);
    if (r.form == Request::CROPS)
        return net.set_input_crops_slots(in0, bytes, r.size, r.hw, r.frame_count, r.boxes, r.count, first);
    if (r.form == Request::IMAGE) return net.set_input_image_slots(in0, bytes, r.size, first, k);
    if (r.in) return net.set_input_slots(in0, static_cast<const float*>(r.in), r.size, first, k);
    return net.set_input_slots(in0, r.ins[0].data(), r.ins[0].size(), first, k);
}

// The batching thread loop: gather (one thread at a time), then run the batch with _mu released.
void WorkerCore::serve_batches(NetCore& net, const std::string& why) {
    std::vector<int> sizes;
    std::vector<int64_t> arrive;
    while (true) {
        std::vector<std::shared_ptr<Request>> batch;
        {
            std::unique_lock<std::mutex> lk(_mu);
            _cv.wait(lk, [this] { return (_stop && _tasks.empty()) || (!_tasks.empty() && !_gathering); });
            if (_stop && _tasks.empty()) return;
            _gathering = true;
            size_t take = 1;   // a thread without a Net fails the requests one by one
            while (why.empty()) {
                sizes.clear();
                arrive.clear();
                for (auto& r : _tasks) {
                    const size_t k = request_images(*r);
                    sizes.push_back(k <= static_cast<size_t>(_batch) ? static_cast<int>(k) : 0);
                    arrive.push_back(r->arrive_us);
                }
                const BatchPlan p = plan_batch(sizes.data(), arrive.data(), sizes.size(), _batch, _max_delay_us,
                                               now_us());
                take = p.take;
                if (p.close || _stop) break;
                _cv.wait_until(lk, std::chrono::steady_clock::time_point(std::chrono::microseconds(p.deadline_us)));
            }
            for (size_t i = 0; i < take; ++i) {
                batch.push_back(_tasks.front());
                _tasks.pop_front();
            }
            _gathering = false;
        }
        _cv.notify_all();   // another thread may gather what is left
        if (!why.empty()) {
            batch[0]->done.set_exception(std::make_exception_ptr(std::runtime_error("Worker: " + why)));
            continue;
        }
        run_batch(net, batch);
    }
}

// Checks every request, stages the valid ones into consecutive slots, runs the Net once and copies each request its
// own rows of graph output 0 (the view forms) or of every graph output (the sync forms), then of every export.
void WorkerCore::run_batch(NetCore& net, std::vector<std::shared_ptr<Request>>& batch) {
    auto fail = [](Request& r, const Status& st) {
        r.done.set_exception(std::make_exception_ptr(std::runtime_error(std::string("Worker: ") + st.info())));
    };
    struct Placed { Request* r; int first, k; };
    std::vector<Placed> placed;
    int used = 0;
    for (auto& r : batch) {
        const size_t k = request_images(*r);
        Status st = check_request(net, *r, k);
        if (!st) { fail(*r, st); continue; }
        placed.push_back({r.get(), used, static_cast<int>(k)});
        used += static_cast<int>(k);
    }
    std::vector<Placed> staged;
    for (auto& p : placed) {
        Status st = stage_slots(net, *p.r, p.first, p.k);
        if (!st) fail(*p.r, st);
        else staged.push_back(p);
    }
    if (staged.empty()) return;
    net.prediction();
    ++_batches_run;
    for (auto& p : staged) _images_run += p.k;
    const size_t nx = net.export_count();
    std::vector<Result> results(staged.size());
    for (size_t j = 0; j < staged.size(); ++j) {
        const Placed& p = staged[j];
        // device source of every part's rows, and the floats of one row
        std::vector<std::pair<const float*, size_t>> parts;
        for (size_t i = 0; i < (p.r->out ? 1 : _outputs.size()); ++i) {
            NetCore::DTensor* d = net.get_out(_outputs[i]);
            parts.push_back({static_cast<const float*>(d->data()), d->storage_bytes() / sizeof(float) / _batch});
        }
        for (size_t i = 0; i < nx; ++i) parts.push_back({net.export_device_ptr(i), net.export_elements(i) / _batch});
        float* at = p.r->out;
        for (auto& part : parts) {
            const size_t n = part.second * p.k;
            if (!p.r->out) { results[j].emplace_back(n); at = results[j].back().data(); }
            CUDA_CHECK(cudaMemcpyAsync(at, part.first + part.second * p.first, n * sizeof(float),
                                       cudaMemcpyDeviceToHost, net.stream()));
            at += n;
        }
    }
    net.sync();
    for (size_t j = 0; j < staged.size(); ++j) staged[j].r->done.set_value(std::move(results[j]));
}

int WorkerCore::batch() {
    if (!wait_ready().empty()) return 0;
    std::lock_guard<std::mutex> lk(_mu);
    return _batch;
}

size_t WorkerCore::image_input_size() {
    if (!wait_ready().empty()) return 0;
    std::lock_guard<std::mutex> lk(_mu);
    return _image_in;
}

size_t WorkerCore::image_view_floats() {
    if (!wait_ready().empty()) return 0;
    std::lock_guard<std::mutex> lk(_mu);
    return _image_view;
}

std::future<std::vector<std::vector<float>>> WorkerCore::sync_prediction(const std::vector<std::vector<float>>& host_ins) {
    auto r = std::make_shared<Request>(Request::FP32, nullptr, 0);
    r->ins = host_ins;
    return enqueue(r, false);
}

void WorkerCore::async_prediction(const std::vector<std::vector<float>>& host_ins) {
    auto r = std::make_shared<Request>(Request::FP32, nullptr, 0);
    r->ins = host_ins;
    enqueue(r, true);
}

void WorkerCore::async_prediction_view(const float* in, size_t in_count, float* out, size_t out_count) {
    enqueue(std::make_shared<Request>(Request::FP32, in, in_count, out, out_count), true);
}

std::future<std::vector<std::vector<float>>> WorkerCore::sync_prediction_image(const uint8_t* in, size_t in_bytes) {
    auto r = std::make_shared<Request>(Request::IMAGE, nullptr, in_bytes);
    r->bytes.assign(in, in + in_bytes);
    r->in = r->bytes.data();
    return enqueue(r, false);
}

void WorkerCore::async_prediction_image_view(const uint8_t* in, size_t in_bytes, float* out, size_t out_count) {
    enqueue(std::make_shared<Request>(Request::IMAGE, in, in_bytes, out, out_count), true);
}

std::future<std::vector<std::vector<float>>> WorkerCore::sync_prediction_images(const uint8_t* pixels, size_t bytes,
                                                                                 const int32_t* hw, size_t count) {
    auto r = std::make_shared<Request>(Request::IMAGES, nullptr, bytes);
    r->bytes.assign(pixels, pixels + bytes);
    r->hw_copy.assign(hw, hw + 2 * count);
    r->in = r->bytes.data();
    r->hw = r->hw_copy.data(); r->count = count;
    return enqueue(r, false);
}

void WorkerCore::async_prediction_images_view(const uint8_t* pixels, size_t bytes, const int32_t* hw, size_t count,
                                              float* out, size_t out_count) {
    auto r = std::make_shared<Request>(Request::IMAGES, pixels, bytes, out, out_count);
    r->hw = hw; r->count = count;
    enqueue(r, true);
}

std::future<std::vector<std::vector<float>>> WorkerCore::sync_prediction_crops(const uint8_t* frames, size_t bytes,
                                                                                const int32_t* hw, size_t frame_count,
                                                                                const int32_t* boxes, size_t count) {
    auto r = std::make_shared<Request>(Request::CROPS, nullptr, bytes);
    r->bytes.assign(frames, frames + bytes);
    r->hw_copy.assign(hw, hw + 2 * frame_count);
    r->boxes_copy.assign(boxes, boxes + 5 * count);
    r->in = r->bytes.data();
    r->hw = r->hw_copy.data(); r->frame_count = frame_count;
    r->boxes = r->boxes_copy.data(); r->count = count;
    return enqueue(r, false);
}

void WorkerCore::async_prediction_crops_view(const uint8_t* frames, size_t bytes, const int32_t* hw,
                                             size_t frame_count, const int32_t* boxes, size_t count, float* out,
                                             size_t out_count) {
    auto r = std::make_shared<Request>(Request::CROPS, frames, bytes, out, out_count);
    r->hw = hw; r->frame_count = frame_count;
    r->boxes = boxes; r->count = count;
    enqueue(r, true);
}

std::string WorkerCore::wait_ready() {
    std::unique_lock<std::mutex> lk(_mu);
    _ready_cv.wait(lk, [this] { return _ready >= _thread_num; });
    return _init_errors.empty() ? std::string() : _init_errors.front();
}

size_t WorkerCore::output_count() {
    if (!wait_ready().empty()) return 0;
    std::lock_guard<std::mutex> lk(_mu);
    return _view_count;
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
