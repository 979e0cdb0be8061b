/*
 * anakin_b200.h -- C ABI of the host framework (libanakin_b200.so): Graph load / Optimize /
 * save and the Net executor, for callers that cannot include the C++ headers
 * (anakin_b200/csrc/framework/{graph,net}.h mirror the reference's C++ API directly).
 *
 * Replaces the reference's dlopen-able runner, framework/c_api/anakin_runner.h:9-58
 * (get_anakinrun_instance -> AnakinRunerInterface::{load_model, get_input_number,
 * get_input_tensor, get_output_tensor, prediction} and AnakinRunerTensorInterface::
 * {get_dev_shape, get_dev_data, copy_data_host_2_dev, copy_data_dev_2_host}) with plain
 * C entry points; the reference's version returns C++ virtual interfaces through
 * extern "C", which no FFI can bind.
 *
 * Return codes: 0 = ok, non-zero = failure (anakin_last_error() has the text).
 * Precision codes = reference framework/core/types.h:25-31: FP32 0, FP16 -1, INT8 -2.
 */
#ifndef ANAKIN_B200_H
#define ANAKIN_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define ANAKIN_API __attribute__((visibility("default")))
#else
#define ANAKIN_API
#endif

#define ANAKIN_FP32 0
#define ANAKIN_FP16 (-1)
#define ANAKIN_INT8 (-2)

typedef struct anakin_graph anakin_graph_t;
typedef struct anakin_net anakin_net_t;
typedef struct anakin_worker anakin_worker_t;

ANAKIN_API const char* anakin_last_error(void);

/* ---- Graph (reference framework/graph/graph.h:36-226) */
ANAKIN_API int anakin_graph_load(const char* model_path, anakin_graph_t** out);            /* Graph::load */
ANAKIN_API int anakin_graph_load_buffer(const void* buf, size_t len, anakin_graph_t** out);
ANAKIN_API int anakin_graph_reset_batch_size(anakin_graph_t* g, const char* in_name, int batch); /* ResetBatchSize */
ANAKIN_API int anakin_graph_reshape(anakin_graph_t* g, const char* in_name, const int* nchw);    /* Reshape */
/* the input_shape (N,C,H,W; missing trailing dims read 1) of Input node in_name */
ANAKIN_API int anakin_graph_input_shape(anakin_graph_t* g, const char* in_name, int* nchw);
ANAKIN_API int anakin_graph_optimize(anakin_graph_t* g, int with_fusion);                 /* Optimize */
ANAKIN_API int anakin_graph_save(anakin_graph_t* g, const char* model_path);              /* save */
/* 8-bit image input (b200_image_desc_t of include/b200_saber.h, same layout): the Input node then takes uint8
 * [n][h][w][c] interleaved pixels (c = its channel count, 1..4, no row padding) and the network sees
 *     x[n][i][y][x] = ((float)img[n][y][x][src_channel[i]] - mean[i]) * scale[i]      (fp32, no FMA)
 * computed by the convolutions that read it; only convolutions may read an image input. Entries i >= c are ignored.
 * The format is stored on the Input node, so it survives save / load, Reshape and ResetBatchSize. */
typedef struct {
    int32_t src_channel[4]; /* network channel i reads image channel src_channel[i]; {2,1,0}: BGR -> RGB */
    float mean[4], scale[4];
} anakin_image_format_t;
/* Fails for an unknown name, a node that is not an Input, c outside 1..4, a src_channel that is not a permutation of
 * 0..c-1, or a non-finite mean / scale. */
ANAKIN_API int anakin_graph_set_input_image(anakin_graph_t* g, const char* in_name, const anakin_image_format_t* fmt);
/* 1 (and *out filled when out != NULL) if in_name is an image input, else 0. Entries i >= c of *out read
 * src_channel -1, mean 0, scale 0. */
ANAKIN_API int anakin_graph_input_image(anakin_graph_t* g, const char* in_name, anakin_image_format_t* out);
/* On-device resize of an image input: requests then carry images of any size up to max_h x max_w (1..16384 each),
 * which the Net resizes and centre-crops on the GPU, inside its CUDA graph, to the Input's H x W before the image
 * path above (b200_image_resize_run of include/b200_saber.h: short side to resize_short, then centre crop; 0 =
 * stretch to H x W; bilinear, no antialiasing). Needs set_input_image first. Stored on the Input node (image_max_h /
 * image_max_w / image_resize_short), so it survives save / load, Reshape and ResetBatchSize. Fails for an unknown
 * name, a node that is not an image Input, max_* outside 1..16384 or resize_short < 0; Net creation fails unless
 * resize_short is 0 or at least max(H, W). */
ANAKIN_API int anakin_graph_set_input_image_resize(anakin_graph_t* g, const char* in_name, int max_h, int max_w,
                                                   int resize_short);
/* 1 (and the non-NULL outputs filled) if in_name is an image input with on-device resize, else 0. */
ANAKIN_API int anakin_graph_input_image_resize(anakin_graph_t* g, const char* in_name, int* max_h, int* max_w,
                                               int* resize_short);
/* Text dump "name|op|in1,in2|out1,out2\n" per node in execution order; returns bytes needed. */
ANAKIN_API size_t anakin_graph_describe(anakin_graph_t* g, char* buf, size_t cap);
ANAKIN_API void anakin_graph_destroy(anakin_graph_t* g);

/* ---- Net (reference framework/core/net/net.h:35-328) */
/* Net<NV, precision>::init(graph) on `device` (-1 = current). */
ANAKIN_API int anakin_net_create(anakin_graph_t* g, int precision, int device, anakin_net_t** out);
/* flags: ANAKIN_NET_KEEP_EDGES = one buffer per edge tensor instead of the MemoryScheduler-style sharing
 * (framework/graph/llvm/optimizer/memory_scheduler.cpp), so that intermediate tensors stay readable after
 * prediction() -- parity tests and debugging only. */
#define ANAKIN_NET_KEEP_EDGES 1
ANAKIN_API int anakin_net_create_ex(anakin_graph_t* g, int precision, int device, int flags, anakin_net_t** out);
ANAKIN_API int anakin_net_num_inputs(anakin_net_t* n);
ANAKIN_API int anakin_net_num_outputs(anakin_net_t* n);
ANAKIN_API const char* anakin_net_input_name(anakin_net_t* n, int idx);
ANAKIN_API const char* anakin_net_output_name(anakin_net_t* n, int idx);
/* info of the tensor produced by a node of the optimised graph (inputs / outputs included):
 * dims = logical N,C,H,W; c_stored = channels as laid out (NHWC padding); layout 8 NCHW / 9 NHWC;
 * dtype = reference DataType; scale = calibrated scale or 0. */
ANAKIN_API int anakin_net_tensor_info(anakin_net_t* n, const char* node, int* dims4, int* c_stored, int* layout,
                                      int* dtype, float* scale, size_t* bytes);
ANAKIN_API void* anakin_net_tensor_device_ptr(anakin_net_t* n, const char* node);
/* get_in(name)->copy_from(host): fp32 NCHW host -> device input, async on the net stream.
 * `pinned` != 0 promises the host buffer is page-locked. */
ANAKIN_API int anakin_net_set_input(anakin_net_t* n, const char* in_name, const float* host, size_t count);
/* The image-input counterpart: `bytes` must equal the input tensor's storage (n*h*w*c). anakin_net_set_input fails on
 * an image input and this fails on an fp32 input. The input's tensor_info reads dtype 7 (UINT8), layout 9 (NHWC),
 * c_stored = c. */
ANAKIN_API int anakin_net_set_input_image(anakin_net_t* n, const char* in_name, const uint8_t* host, size_t bytes);
/* A request on an input with on-device resize: `count` (= the batch) images, image i h_i * w_i * c uint8 bytes
 * (interleaved, rows unpadded), packed back to back in batch order; hw = int32 [count][2] of (h_i, w_i). Checked
 * before any copy: count, 1 <= h_i <= max_h, 1 <= w_i <= max_w, bytes == the sum, a valid geometry. The pixels and
 * the size table are copied H2D asynchronously on the net stream, so `pixels` must stay valid until the next sync.
 * The next prediction resizes them into the input tensor (exec op "<input>:ImageResize"), whose tensor_info /
 * read_tensor then give the resized bytes. anakin_net_set_input_image fails on such an input and this on any other. */
ANAKIN_API int anakin_net_set_input_images(anakin_net_t* n, const char* in_name, const uint8_t* pixels, size_t bytes,
                                           const int32_t* hw, size_t count);
/* Net::prediction(): enqueue the whole network on the net's stream (asynchronous). */
ANAKIN_API int anakin_net_prediction(anakin_net_t* n);
ANAKIN_API int anakin_net_sync(anakin_net_t* n);
/* D2H of a node's raw tensor storage (then stream-synchronise). */
ANAKIN_API int anakin_net_read_tensor(anakin_net_t* n, const char* node, void* host, size_t bytes);
ANAKIN_API void* anakin_net_stream(anakin_net_t* n);
ANAKIN_API int anakin_net_launched_ops(anakin_net_t* n);      /* kernels-launching ops per prediction */
ANAKIN_API int anakin_net_cuda_graph_active(anakin_net_t* n);
ANAKIN_API int anakin_net_set_cuda_graph(anakin_net_t* n, int enable);
ANAKIN_API size_t anakin_net_exec_order(anakin_net_t* n, char* buf, size_t cap); /* "name:op\n" per launched op */
ANAKIN_API size_t anakin_net_activation_bytes(anakin_net_t* n);          /* device bytes of edge tensors, after sharing */
ANAKIN_API size_t anakin_net_activation_bytes_unshared(anakin_net_t* n); /* one buffer per edge */
/* device addresses of the packed weights of every launched op that has some; returns their count. Nets built
 * from one Graph on one device share them (the reference's GraphGlobalMem, graph_global_mem.h:78-250). */
ANAKIN_API int anakin_net_weight_ptrs(anakin_net_t* n, const void** out, int cap);
/* live packed-weight images of this process: total device bytes (+ entries, lookups that hit / missed) */
ANAKIN_API size_t anakin_weight_arena_stats(size_t* entries, size_t* hits, size_t* misses);
/* Replicas on other GPUs (one process per GPU): the rank that built the weights exports the whole arena of `device` as one
 * contiguous DEVICE buffer (creation order, 256-byte aligned images), that buffer is broadcast once with NCCL, and ranks
 * whose Nets were initialised in receive mode (same plans and buffers, no fold / quantise / pack on the host) import it.
 * SURVEY.md section 8e: "NCCL-broadcast weights over NVLink". Returns 0 on success. */
ANAKIN_API void anakin_weight_arena_set_receive(int on);
ANAKIN_API size_t anakin_weight_arena_flat_bytes(int device);
ANAKIN_API int anakin_weight_arena_export(int device, void* flat_dev, size_t cap);
ANAKIN_API int anakin_weight_arena_import(int device, const void* flat_dev, size_t bytes);
/* Per-op device time in ms (same order as anakin_net_exec_order), mean of `iters` eager runs with a
 * CUDA-event pair around every op -- the reference's ENABLE_OP_TIMER (net.cpp:445-449,494-506).
 * reps > 1 launches each op `reps` times back to back inside its pair (steady-state device time). */
ANAKIN_API int anakin_net_profile_ops(anakin_net_t* n, int iters, int reps, float* ms, int cap);
ANAKIN_API void anakin_net_destroy(anakin_net_t* n);

/* ---- Worker (reference framework/core/net/worker.h:69-190): thread pool of per-thread Nets.
 * devices: thread i runs on devices[i % n_devices]; n_devices == 0 keeps the current device. */
ANAKIN_API int anakin_worker_create(const char* model_path, int precision, int threads, const int* devices,
                                    int n_devices, int batch, anakin_worker_t** out);
/* sync_prediction: one fp32 NCHW input, one fp32 output (first registered in / out). */
ANAKIN_API int anakin_worker_sync_prediction(anakin_worker_t* w, const float* in, size_t in_count, float* out,
                                             size_t out_count);
/* Worker::async_prediction / async_get_result (framework/core/worker.h:77-92), zero-copy: `in` / `out` are
 * caller-owned (ideally pinned) host buffers that stay valid until the matching get_result returns. Results
 * come back in submission order. With threads >= 2 one request's H2D / D2H copies overlap another's kernels. */
ANAKIN_API int anakin_worker_wait_ready(anakin_worker_t* w);
ANAKIN_API int anakin_worker_async_prediction(anakin_worker_t* w, const float* in, size_t in_count, float* out,
                                              size_t out_count);
ANAKIN_API int anakin_worker_async_get_result(anakin_worker_t* w);
/* The same for a first input that is an image input: `in` holds exactly its uint8 [n][h][w][c] bytes. The async form is
 * zero-copy like anakin_worker_async_prediction and is collected by anakin_worker_async_get_result. The float calls
 * fail on an image input, these on an fp32 input. */
ANAKIN_API int anakin_worker_sync_prediction_image(anakin_worker_t* w, const uint8_t* in, size_t in_bytes, float* out,
                                                   size_t out_count);
ANAKIN_API int anakin_worker_async_prediction_image(anakin_worker_t* w, const uint8_t* in, size_t in_bytes, float* out,
                                                    size_t out_count);
/* The same for a first input with on-device resize: one request as anakin_net_set_input_images. The async form is
 * zero-copy: pixels and hw stay caller-owned until anakin_worker_async_get_result. A malformed request fails alone
 * (its result reports the error) and the Worker keeps serving. */
ANAKIN_API int anakin_worker_sync_prediction_images(anakin_worker_t* w, const uint8_t* pixels, size_t bytes,
                                                    const int32_t* hw, size_t count, float* out, size_t out_count);
ANAKIN_API int anakin_worker_async_prediction_images(anakin_worker_t* w, const uint8_t* pixels, size_t bytes,
                                                     const int32_t* hw, size_t count, float* out, size_t out_count);
ANAKIN_API void anakin_worker_destroy(anakin_worker_t* w);

#ifdef __cplusplus
}
#endif
#endif /* ANAKIN_B200_H */
