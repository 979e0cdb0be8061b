// C ABI over Graph / Net / Worker (include/anakin_b200.h); replaces the reference's
// framework/c_api/anakin_runner.{h,cpp}.
#include "../../../include/anakin_b200.h"

#include <sstream>

#include "net.h"

using namespace anakin;

struct anakin_graph { graph::GraphCore g; };
struct anakin_net { NetCore net; std::vector<std::string> ins, outs; };
struct anakin_worker { std::unique_ptr<WorkerCore> w; };

static thread_local std::string g_err;
static int fail(const std::string& m) { g_err = m; return 1; }
static Precision to_precision(int p) {
    return p == ANAKIN_INT8 ? Precision::INT8 : (p == ANAKIN_FP16 ? Precision::FP16 : Precision::FP32);
}
static size_t emit(const std::string& s, char* buf, size_t cap) {
    if (buf && cap) {
        size_t n = s.size() < cap - 1 ? s.size() : cap - 1;
        memcpy(buf, s.data(), n);
        buf[n] = 0;
    }
    return s.size() + 1;
}

extern "C" {

const char* anakin_last_error(void) { return g_err.c_str(); }

int anakin_graph_load(const char* model_path, anakin_graph_t** out) {
    if (!model_path || !out) return fail("null argument");
    auto* g = new anakin_graph();
    Status st = g->g.load(std::string(model_path));
    if (!st) { std::string m = st.info(); delete g; return fail(m); }
    *out = g;
    return 0;
}

int anakin_graph_load_buffer(const void* buf, size_t len, anakin_graph_t** out) {
    if (!buf || !out) return fail("null argument");
    auto* g = new anakin_graph();
    Status st = g->g.load(static_cast<const char*>(buf), len);
    if (!st) { std::string m = st.info(); delete g; return fail(m); }
    *out = g;
    return 0;
}

int anakin_graph_reset_batch_size(anakin_graph_t* g, const char* in_name, int batch) {
    if (!g || !in_name) return fail("null argument");
    if (!g->g.has_node(in_name)) return fail(std::string("no input node ") + in_name);
    g->g.ResetBatchSize(in_name, batch);
    return 0;
}

int anakin_graph_reshape(anakin_graph_t* g, const char* in_name, const int* nchw) {
    if (!g || !in_name || !nchw) return fail("null argument");
    if (!g->g.has_node(in_name)) return fail(std::string("no input node ") + in_name);
    g->g.Reshape(in_name, {nchw[0], nchw[1], nchw[2], nchw[3]});
    return 0;
}

int anakin_graph_input_shape(anakin_graph_t* g, const char* in_name, int* nchw) {
    if (!g || !in_name || !nchw) return fail("null argument");
    auto n = g->g[in_name];
    if (!n || n->op != "Input") return fail(std::string("no input node ") + in_name);
    const auto s = n->get_attr_or<PTuple<int>>("input_shape", {});
    for (int i = 0; i < 4; ++i) nchw[i] = i < static_cast<int>(s.size()) ? s[i] : 1;
    return 0;
}

int anakin_graph_optimize(anakin_graph_t* g, int with_fusion) {
    if (!g) return fail("null argument");
    Status st = g->g.Optimize(with_fusion != 0);
    return st ? 0 : fail(st.info());
}

int anakin_graph_save(anakin_graph_t* g, const char* model_path) {
    if (!g || !model_path) return fail("null argument");
    Status st = g->g.save(std::string(model_path));
    return st ? 0 : fail(st.info());
}

static_assert(sizeof(anakin_image_format_t) == sizeof(b200_image_desc_t), "image format layouts differ");

int anakin_graph_set_input_image(anakin_graph_t* g, const char* in_name, const anakin_image_format_t* fmt) {
    if (!g || !in_name || !fmt) return fail("null argument");
    b200_image_desc_t d;
    memcpy(&d, fmt, sizeof(d));
    Status st = g->g.set_input_image(in_name, d);
    return st ? 0 : fail(st.info());
}

int anakin_graph_input_image(anakin_graph_t* g, const char* in_name, anakin_image_format_t* out) {
    if (!g || !in_name) return 0;
    b200_image_desc_t d;
    if (!g->g.input_image(in_name, &d)) return 0;
    const auto s = g->g[in_name]->get_attr_or<PTuple<int>>("image_src_channel", {});
    for (size_t i = s.size(); i < 4; ++i) d.src_channel[i] = -1;   // past the channel count
    if (out) memcpy(out, &d, sizeof(d));
    return 1;
}

int anakin_graph_set_input_image_resize(anakin_graph_t* g, const char* in_name, int max_h, int max_w, int resize_short) {
    if (!g || !in_name) return fail("null argument");
    Status st = g->g.set_input_image_resize(in_name, max_h, max_w, resize_short);
    return st ? 0 : fail(st.info());
}

int anakin_graph_input_image_resize(anakin_graph_t* g, const char* in_name, int* max_h, int* max_w, int* resize_short) {
    if (!g || !in_name) return 0;
    graph::ImageResize r;
    if (!g->g.input_image_resize(in_name, &r)) return 0;
    if (max_h) *max_h = r.max_h;
    if (max_w) *max_w = r.max_w;
    if (resize_short) *resize_short = r.resize_short;
    return 1;
}

size_t anakin_graph_describe(anakin_graph_t* g, char* buf, size_t cap) {
    if (!g) return 0;
    std::ostringstream os;
    for (auto& nm : g->g.get_nodes_in_order()) {
        auto n = g->g[nm];
        os << n->name << "|" << n->op << "|";
        for (size_t i = 0; i < n->ins.size(); ++i) os << (i ? "," : "") << n->ins[i];
        os << "|";
        for (size_t i = 0; i < n->outs.size(); ++i) os << (i ? "," : "") << n->outs[i];
        os << "\n";
    }
    return emit(os.str(), buf, cap);
}

void anakin_graph_destroy(anakin_graph_t* g) { delete g; }

int anakin_net_create(anakin_graph_t* g, int precision, int device, anakin_net_t** out) {
    return anakin_net_create_ex(g, precision, device, 0, out);
}

int anakin_net_create_ex(anakin_graph_t* g, int precision, int device, int flags, anakin_net_t** out) {
    if (!g || !out) return fail("null argument");
    auto* n = new anakin_net();
    if (flags & ANAKIN_NET_KEEP_EDGES) n->net.set_share_activations(false);
    Status st = n->net.init(g->g, to_precision(precision), device);
    if (!st) { std::string m = st.info(); delete n; return fail(m); }
    n->ins = n->net.get_in_names();
    n->outs = n->net.get_out_names();
    *out = n;
    return 0;
}

int anakin_net_num_inputs(anakin_net_t* n) { return n ? static_cast<int>(n->ins.size()) : 0; }
int anakin_net_num_outputs(anakin_net_t* n) { return n ? static_cast<int>(n->outs.size()) : 0; }
const char* anakin_net_input_name(anakin_net_t* n, int idx) {
    return (n && idx >= 0 && idx < static_cast<int>(n->ins.size())) ? n->ins[idx].c_str() : nullptr;
}
const char* anakin_net_output_name(anakin_net_t* n, int idx) {
    return (n && idx >= 0 && idx < static_cast<int>(n->outs.size())) ? n->outs[idx].c_str() : nullptr;
}

int anakin_net_tensor_info(anakin_net_t* n, const char* node, int* dims4, int* c_stored, int* layout, int* dtype,
                           float* scale, size_t* bytes) {
    if (!n || !node) return fail("null argument");
    auto* t = n->net.get_tensor_from_node(node);
    if (!t) return fail(std::string("no tensor for node ") + node);
    if (dims4) { dims4[0] = t->num(); dims4[1] = t->channel(); dims4[2] = t->height(); dims4[3] = t->width(); }
    if (c_stored) *c_stored = t->channel_stored();
    if (layout) *layout = t->get_layout();
    if (dtype) *dtype = t->get_dtype();
    if (scale) *scale = t->get_scale().empty() ? 0.f : t->get_scale()[0];
    if (bytes) *bytes = t->storage_bytes();
    return 0;
}

void* anakin_net_tensor_device_ptr(anakin_net_t* n, const char* node) {
    if (!n || !node) return nullptr;
    auto* t = n->net.get_tensor_from_node(node);
    return t ? t->mutable_data() : nullptr;
}

int anakin_net_set_input(anakin_net_t* n, const char* in_name, const float* host, size_t count) {
    if (!n || !in_name || !host) return fail("null argument");
    auto* t = n->net.get_in(in_name);
    if (!t) return fail(std::string("no input ") + in_name);
    if (t->is_image()) return fail(std::string("input ") + in_name + " is an image input: use anakin_net_set_input_image");
    if (count * sizeof(float) != t->storage_bytes()) return fail("input element count does not match the input tensor");
    cudaSetDevice(n->net.device());
    cudaError_t e = cudaMemcpyAsync(t->mutable_data(), host, t->storage_bytes(), cudaMemcpyHostToDevice, n->net.stream());
    return e == cudaSuccess ? 0 : fail(cudaGetErrorString(e));
}

int anakin_net_set_input_image(anakin_net_t* n, const char* in_name, const uint8_t* host, size_t bytes) {
    if (!n || !in_name || !host) return fail("null argument");
    auto* t = n->net.get_in(in_name);
    if (!t) return fail(std::string("no input ") + in_name);
    if (!t->is_image()) return fail(std::string("input ") + in_name + " is not an image input");
    if (n->net.resizes_input(in_name))
        return fail(std::string("input ") + in_name + " resizes images on the GPU: use anakin_net_set_input_images");
    if (bytes != t->storage_bytes())
        return fail("image of " + std::to_string(bytes) + " bytes, input " + in_name + " holds " + std::to_string(t->storage_bytes()));
    cudaSetDevice(n->net.device());
    cudaError_t e = cudaMemcpyAsync(t->mutable_data(), host, bytes, cudaMemcpyHostToDevice, n->net.stream());
    return e == cudaSuccess ? 0 : fail(cudaGetErrorString(e));
}

int anakin_net_set_input_images(anakin_net_t* n, const char* in_name, const uint8_t* pixels, size_t bytes,
                                const int32_t* hw, size_t count) {
    if (!n || !in_name || !pixels || !hw) return fail("null argument");
    Status st = n->net.set_input_images(in_name, pixels, bytes, hw, count);
    return st ? 0 : fail(st.info());
}

int anakin_net_prediction(anakin_net_t* n) {
    if (!n) return fail("null argument");
    n->net.prediction();
    return 0;
}

int anakin_net_sync(anakin_net_t* n) {
    if (!n) return fail("null argument");
    cudaError_t e = cudaStreamSynchronize(n->net.stream());
    return e == cudaSuccess ? 0 : fail(cudaGetErrorString(e));
}

int anakin_net_read_tensor(anakin_net_t* n, const char* node, void* host, size_t bytes) {
    if (!n || !node || !host) return fail("null argument");
    auto* t = n->net.get_tensor_from_node(node);
    if (!t) return fail(std::string("no tensor for node ") + node);
    if (bytes > t->storage_bytes()) bytes = t->storage_bytes();
    cudaSetDevice(n->net.device());
    cudaError_t e = cudaMemcpyAsync(host, t->data(), bytes, cudaMemcpyDeviceToHost, n->net.stream());
    if (e == cudaSuccess) e = cudaStreamSynchronize(n->net.stream());
    return e == cudaSuccess ? 0 : fail(cudaGetErrorString(e));
}

void* anakin_net_stream(anakin_net_t* n) { return n ? n->net.stream() : nullptr; }
int anakin_net_launched_ops(anakin_net_t* n) { return n ? static_cast<int>(n->net.launched_op_count()) : 0; }
int anakin_net_cuda_graph_active(anakin_net_t* n) { return n && n->net.cuda_graph_active() ? 1 : 0; }
int anakin_net_set_cuda_graph(anakin_net_t* n, int enable) {
    if (!n) return fail("null argument");
    n->net.set_use_cuda_graph(enable != 0);
    return 0;
}
size_t anakin_net_exec_order(anakin_net_t* n, char* buf, size_t cap) {
    if (!n) return 0;
    std::string s;
    for (auto& e : n->net.get_exec_order()) s += e + "\n";
    return emit(s, buf, cap);
}
int anakin_net_profile_ops(anakin_net_t* n, int iters, int reps, float* ms, int cap) {
    if (!n || !ms || iters <= 0) return fail("bad argument");
    std::vector<float> v = n->net.profile_ops(iters, reps);
    for (int i = 0; i < cap && i < static_cast<int>(v.size()); ++i) ms[i] = v[i];
    return 0;
}
size_t anakin_net_activation_bytes(anakin_net_t* n) { return n ? n->net.activation_bytes() : 0; }
size_t anakin_net_activation_bytes_unshared(anakin_net_t* n) { return n ? n->net.activation_bytes_unshared() : 0; }
int anakin_net_weight_ptrs(anakin_net_t* n, const void** out, int cap) {
    if (!n) return 0;
    std::vector<const void*> v = n->net.weight_device_ptrs();
    for (int i = 0; out && i < cap && i < static_cast<int>(v.size()); ++i) out[i] = v[i];
    return static_cast<int>(v.size());
}
size_t anakin_weight_arena_stats(size_t* entries, size_t* hits, size_t* misses) {
    return saber::weight_arena_stats(entries, hits, misses);
}
void anakin_weight_arena_set_receive(int on) { saber::weight_arena_set_receive(on != 0); }
size_t anakin_weight_arena_flat_bytes(int device) { return saber::weight_arena_flat_bytes(device); }
int anakin_weight_arena_export(int device, void* flat_dev, size_t cap) {
    return saber::weight_arena_export(device, flat_dev, cap) == saber::SaberSuccess ? 0 : fail("weight arena export failed");
}
int anakin_weight_arena_import(int device, const void* flat_dev, size_t bytes) {
    return saber::weight_arena_import(device, flat_dev, bytes) == saber::SaberSuccess ? 0 : fail("weight arena import failed");
}
void anakin_net_destroy(anakin_net_t* n) { delete n; }

int anakin_worker_create(const char* model_path, int precision, int threads, const int* devices, int n_devices,
                         int batch, anakin_worker_t** out) {
    if (!model_path || !out || threads <= 0) return fail("bad argument");
    auto* w = new anakin_worker();
    w->w.reset(new WorkerCore(model_path, to_precision(precision), threads));
    if (devices && n_devices > 0) w->w->set_devices(std::vector<int>(devices, devices + n_devices));
    if (batch > 0) {
        // the model's input is assumed to be the classification input [N,3,H,W]; read H,W from the file
        graph::GraphCore g;
        Status st = g.load(std::string(model_path));
        if (!st) { std::string m = st.info(); delete w; return fail(m); }
        for (auto& in : g.get_ins()) {
            auto s = g[in]->get_attr<PTuple<int>>("input_shape");
            s[0] = batch;
            w->w->Reshape(in, s);
        }
    }
    w->w->launch();
    *out = w;
    return 0;
}

int anakin_worker_sync_prediction(anakin_worker_t* w, const float* in, size_t in_count, float* out, size_t out_count) {
    if (!w || !in || !out) return fail("null argument");
    std::vector<std::vector<float>> ins(1, std::vector<float>(in, in + in_count));
    try {
        auto res = w->w->sync_prediction(ins).get();
        if (res.empty()) return fail("worker produced no output");
        size_t n = res[0].size() < out_count ? res[0].size() : out_count;
        memcpy(out, res[0].data(), n * sizeof(float));
    } catch (const std::exception& e) {
        return fail(e.what());
    }
    return 0;
}

int anakin_worker_wait_ready(anakin_worker_t* w) {
    if (!w) return fail("null argument");
    const std::string err = w->w->wait_ready();
    return err.empty() ? 0 : fail(err);
}

int anakin_worker_async_prediction(anakin_worker_t* w, const float* in, size_t in_count, float* out, size_t out_count) {
    if (!w || !in || !out) return fail("null argument");
    w->w->async_prediction_view(in, in_count, out, out_count);
    return 0;
}

int anakin_worker_async_get_result(anakin_worker_t* w) {
    if (!w) return fail("null argument");
    if (w->w->empty()) return fail("no request in flight");
    try {
        w->w->async_get_result();
    } catch (const std::exception& e) {
        return fail(e.what());
    }
    return 0;
}

int anakin_worker_sync_prediction_image(anakin_worker_t* w, const uint8_t* in, size_t in_bytes, float* out, size_t out_count) {
    if (!w || !in || !out) return fail("null argument");
    try {
        auto res = w->w->sync_prediction_image(in, in_bytes).get();
        if (res.empty()) return fail("worker produced no output");
        size_t n = res[0].size() < out_count ? res[0].size() : out_count;
        memcpy(out, res[0].data(), n * sizeof(float));
    } catch (const std::exception& e) {
        return fail(e.what());
    }
    return 0;
}

int anakin_worker_async_prediction_image(anakin_worker_t* w, const uint8_t* in, size_t in_bytes, float* out,
                                         size_t out_count) {
    if (!w || !in || !out) return fail("null argument");
    w->w->async_prediction_image_view(in, in_bytes, out, out_count);
    return 0;
}

int anakin_worker_sync_prediction_images(anakin_worker_t* w, const uint8_t* pixels, size_t bytes, const int32_t* hw,
                                         size_t count, float* out, size_t out_count) {
    if (!w || !pixels || !hw || !out) return fail("null argument");
    try {
        auto res = w->w->sync_prediction_images(pixels, bytes, hw, count).get();
        if (res.empty()) return fail("worker produced no output");
        size_t n = res[0].size() < out_count ? res[0].size() : out_count;
        memcpy(out, res[0].data(), n * sizeof(float));
    } catch (const std::exception& e) {
        return fail(e.what());
    }
    return 0;
}

int anakin_worker_async_prediction_images(anakin_worker_t* w, const uint8_t* pixels, size_t bytes, const int32_t* hw,
                                          size_t count, float* out, size_t out_count) {
    if (!w || !pixels || !hw || !out) return fail("null argument");
    w->w->async_prediction_images_view(pixels, bytes, hw, count, out, out_count);
    return 0;
}

void anakin_worker_destroy(anakin_worker_t* w) { delete w; }

}  // extern "C"
