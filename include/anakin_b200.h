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
 * stretch to H x W; bilinear, no antialiasing, unless anakin_graph_set_input_image_resize_filter picks Pillow's).
 * Needs set_input_image first. Stored on the Input node (image_max_h / image_max_w / image_resize_short), so it survives save / load, Reshape and ResetBatchSize. Fails for an unknown
 * name, a node that is not an image Input, max_* outside 1..16384 or resize_short < 0; Net creation fails unless
 * resize_short is 0 or at least max(H, W). */
ANAKIN_API int anakin_graph_set_input_image_resize(anakin_graph_t* g, const char* in_name, int max_h, int max_w,
                                                   int resize_short);
/* The resize filter of an image input with on-device resize (anakin_graph_set_input_image_resize first):
 * 0 (B200_IMAGE_RESIZE_REFERENCE, the default) the bilinear resize above; 1 (B200_IMAGE_RESIZE_PIL) Pillow's
 * antialiased BILINEAR with torchvision's centre crop, the bytes of CenterCrop(H, W)(Resize(resize_short)(img)) on a
 * PIL image (b200_image_resize_pil_run); 3 (B200_IMAGE_RESIZE_PIL_BICUBIC) the same with Pillow's antialiased BICUBIC,
 * the bytes of CenterCrop(H, W)(Resize(resize_short, interpolation=BICUBIC)(img)); 5 (B200_IMAGE_RESIZE_CV2_LINEAR)
 * OpenCV's INTER_LINEAR, the bytes of cv2.resize(img, (rw, rh))[top:top + H, left:left + W] with the sizes and floor
 * offsets of filter 0. Every filter runs on interleaved images, NV12 / I420 frames and crop boxes alike
 * (b200_image_crop_resize_run). Stored as the Input attribute image_resize_filter (absent = 0), so it survives save /
 * load, Reshape and ResetBatchSize. Fails for a name that is not such an input or a filter other than 0, 1, 3 or 5. */
ANAKIN_API int anakin_graph_set_input_image_resize_filter(anakin_graph_t* g, const char* in_name, int filter);
/* The filter of an image input with on-device resize, or -1 when in_name is not one. */
ANAKIN_API int anakin_graph_input_image_resize_filter(anakin_graph_t* g, const char* in_name);
/* The pixel layout of the requests of an image input with on-device resize (anakin_graph_set_input_image_resize
 * first): 0 (the default) interleaved h x w x c bytes per image; 1 (B200_IMAGE_YUV_NV12) or 2 (B200_IMAGE_YUV_I420)
 * YUV 4:2:0 frames of even h and w, h*w*3/2 bytes each, that the Net converts to RGB exactly as OpenCV's
 * cvtColor(COLOR_YUV2RGB_NV12 / _I420) while it resizes them with either filter (b200_image_resize_yuv_run). Stored as
 * the Input attribute image_pixel_format (absent = 0), so it survives save / load, Reshape and ResetBatchSize. Fails
 * for a name that is not such an input or a format other than 0 / 1 / 2; Net creation fails for a YUV format unless
 * the input has 3 channels. */
ANAKIN_API int anakin_graph_set_input_image_pixel_format(anakin_graph_t* g, const char* in_name, int format);
/* The pixel format of an image input with on-device resize, or -1 when in_name is not one. */
ANAKIN_API int anakin_graph_input_image_pixel_format(anakin_graph_t* g, const char* in_name);
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
/* ANAKIN_NET_CALIB_STATS = INT8 calibration statistics computed inside every prediction (see anakin_net_calib_*
 * below). FP32 nets with fp32 graph inputs only: creation fails on an FP16 / INT8 net or an 8-bit image input. */
#define ANAKIN_NET_CALIB_STATS 2
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
 * (interleaved, rows unpadded) or, for an NV12 / I420 input, an h_i * w_i * 3 / 2 byte frame, packed back to back in
 * batch order; hw = int32 [count][2] of (h_i, w_i). Checked before any copy: count, 1 <= h_i <= max_h,
 * 1 <= w_i <= max_w (both even for a YUV frame), bytes == the sum, a valid geometry. The pixels and
 * the size table are copied H2D asynchronously on the net stream, so `pixels` must stay valid until the next sync.
 * The next prediction resizes them into the input tensor (exec op "<input>:ImageResize"), whose tensor_info /
 * read_tensor then give the resized bytes. anakin_net_set_input_image fails on such an input and this on any other. */
ANAKIN_API int anakin_net_set_input_images(anakin_net_t* n, const char* in_name, const uint8_t* pixels, size_t bytes,
                                           const int32_t* hw, size_t count);
/* A request of boxes cropped out of frames on an input with on-device resize (b200_image_crop_resize_run of
 * include/b200_saber.h): frame_count frames packed and sized as anakin_net_set_input_images packs images (hw = int32
 * [frame_count][2]), and boxes = int32 [count][5] of (frame, top, left, height, width), count = the batch. Box i becomes
 * image i of the batch: the input's resize and centre crop of frame[top:top+height, left:left+width], taps clipped at
 * the box. Any box inside its frame is allowed, odd offsets and sizes of YUV frames included; boxes are never clamped.
 * Checked before any copy: 1 <= frame_count <= count, every frame as an image of anakin_net_set_input_images, every
 * box names a frame in range, lies inside it and has a valid geometry; the message names the box. Copied H2D
 * asynchronously like anakin_net_set_input_images, so all three arrays must stay valid until the next sync. */
ANAKIN_API int anakin_net_set_input_crops(anakin_net_t* n, const char* in_name, const uint8_t* frames, size_t bytes,
                                          const int32_t* hw, size_t frame_count, const int32_t* boxes, size_t count);
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
/* How each op of anakin_net_exec_order is launched, for the first `cap` ops (either array may be NULL); returns the op
 * count. join[i] = exec index of the op that waits for op i on the side stream, or -1 when op i runs on the main
 * stream. head[i] = 1: op i launches the fused head (pooling, inner product and softmax as one), 2: the head covers
 * op i, which launches nothing, 0: neither. */
ANAKIN_API int anakin_net_schedule(anakin_net_t* n, int* join, int* head, int cap);
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
/* INT8 calibration statistics of a net created with ANAKIN_NET_CALIB_STATS (the reference's EntropyCalibrator passes,
 * entropy_calibrator.cpp). The net keeps one slot per graph input and one per launched op's output, in
 * anakin_net_exec_order order after the inputs; anakin_net_calib_name(i) names slot i's node. Every prediction
 * launches b200_calib_stats_run (include/b200_saber.h) on each slot right behind its producer, inside the CUDA graph
 * (the launch count grows by the slot count; exec order, profile_ops and activation memory are unchanged).
 *   set_pass 0: fold max |x| into each slot's running maximum; 1: add |x| to its 2048 bins of width max / 2048 (the
 *     maximum of pass 0). The pass is a device word, so both passes replay one captured graph. Stream-ordered.
 *   reset: zero every maximum and bin (stream-ordered; creation starts zeroed, in pass 0).
 *   read: wait for the net stream, then copy float max[count] and / or uint64 hist[count][2048] (either may be NULL).
 *   kl: the entropy thresholds of the accumulated histograms (b200_calib_kl_run on the net stream): int32 thresh[count].
 * The calls fail on a net created without the flag. */
ANAKIN_API int anakin_net_calib_count(anakin_net_t* n);
ANAKIN_API const char* anakin_net_calib_name(anakin_net_t* n, int i);
ANAKIN_API int anakin_net_calib_reset(anakin_net_t* n);
ANAKIN_API int anakin_net_calib_set_pass(anakin_net_t* n, int pass);
ANAKIN_API int anakin_net_calib_read(anakin_net_t* n, float* max, uint64_t* hist);
ANAKIN_API int anakin_net_calib_kl(anakin_net_t* n, int32_t* thresh);
/* Interior-tensor exports (the reference's Net::get_tensor_from_edge, net.h:209): anakin_net_create_ex plus n node
 * names of the optimised graph (as anakin_graph_describe lists them after Optimize; an alias node -- Split, Flatten,
 * Gather -- stands for its producer's tensor) whose output tensors every prediction also writes as dense fp32
 * [n][c][h][w] into buffers the net owns (b200_export_run of include/b200_saber.h, launched right behind each
 * producer inside the CUDA graph). 8-bit edges are dequantised as codes x scale (x 127/255 for uint8 codes), f16
 * edges widened, channel padding dropped. The network is unchanged: edge dtypes, plans, the fused INT8 head, exec
 * order, profile_ops and activation bytes are those of the same net without exports; anakin_net_launched_ops grows
 * by n. Fails for n < 0 or a null array or entry (before any device is touched), and for an unknown name (a node that
 * fusion absorbed is exported under the fused node's name), an Input, a name given twice or a graph output. */
ANAKIN_API int anakin_net_create_exports(anakin_graph_t* g, int precision, int device, int flags,
                                         const char* const* nodes, int n, anakin_net_t** out);
ANAKIN_API int anakin_net_num_exports(anakin_net_t* n);
ANAKIN_API const char* anakin_net_export_name(anakin_net_t* n, int i);   /* registration order */
/* nchw = int[4]: the export's N, C, H, W (it holds N*C*H*W floats). */
ANAKIN_API int anakin_net_export_info(anakin_net_t* n, const char* node, int* nchw);
/* Waits for the net stream, then copies the export: count must equal its N*C*H*W. */
ANAKIN_API int anakin_net_read_export(anakin_net_t* n, const char* node, float* host, size_t count);
/* Device address of the export's fp32 buffer (NULL when node is not an export), valid for the net's lifetime; it is
 * rewritten by every prediction, in the net stream's order. */
ANAKIN_API const float* anakin_net_export_device_ptr(anakin_net_t* n, const char* node);
ANAKIN_API size_t anakin_net_export_bytes(anakin_net_t* n);   /* device bytes of all export buffers */
ANAKIN_API void anakin_net_destroy(anakin_net_t* n);

/* ---- Worker (reference framework/core/net/worker.h:69-190): thread pool of per-thread Nets.
 * devices: thread i runs on devices[i % n_devices]; n_devices == 0 keeps the current device. */
ANAKIN_API int anakin_worker_create(const char* model_path, int precision, int threads, const int* devices,
                                    int n_devices, int batch, anakin_worker_t** out);
/* sync_prediction: one fp32 NCHW input, one fp32 output (first registered in / out). Every Worker request is checked
 * as anakin_net_set_input* checks it: in_count must equal the input's elements, and a refused request fails alone. */
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
/* The same for a request of boxes as anakin_net_set_input_crops; its k (batching) is count, the number of boxes. The
 * async form is zero-copy: frames, hw and boxes stay caller-owned until anakin_worker_async_get_result. A malformed
 * request fails alone (its result reports the error) and the Worker keeps serving. */
ANAKIN_API int anakin_worker_sync_prediction_crops(anakin_worker_t* w, const uint8_t* frames, size_t bytes,
                                                   const int32_t* hw, size_t frame_count, const int32_t* boxes,
                                                   size_t count, float* out, size_t out_count);
ANAKIN_API int anakin_worker_async_prediction_crops(anakin_worker_t* w, const uint8_t* frames, size_t bytes,
                                                    const int32_t* hw, size_t frame_count, const int32_t* boxes,
                                                    size_t count, float* out, size_t out_count);
/* anakin_worker_create with exports on every thread's Net (anakin_net_create_exports): each of the n entries names a
 * node of the optimised graph, or an edge as "bottom->top" (Worker::register_interior_edges, worker.h:100-105:
 * bottom's tensor, once the edge is found). Waits until every thread has built its Net and fails with the first
 * error (an unknown edge or a refused export). With exports the sync calls copy graph output 0; the view calls
 * (anakin_worker_async_prediction*) fill `out` with graph output 0 as stored, then every export as fp32
 * [n][c][h][w], in registration order, back to back. Their out_count must then equal anakin_worker_output_count
 * exactly; otherwise that request alone fails with both numbers and the worker keeps serving. n < 0 or a null array
 * or entry fails before anything is loaded. */
ANAKIN_API int anakin_worker_create_exports(const char* model_path, int precision, int threads, const int* devices,
                                            int n_devices, int batch, const char* const* nodes, int n,
                                            anakin_worker_t** out);
/* Floats of one view result: graph output 0 (as stored) plus every export; waits for the threads; 0 on failure. */
ANAKIN_API size_t anakin_worker_output_count(anakin_worker_t* w);
/* Server-side batching: anakin_worker_create_exports (n = 0 for no exports) whose requests may carry k images,
 * 1 <= k <= the batch, through every request entry point above. in_count / in_bytes are then k x one image's, an
 * images or crops request's count is k, a view request's out_count is exactly k x out_per_image
 * (anakin_worker_image_sizes), and each request gets its own k rows: graph output 0 (the sync calls) or output 0 then
 * every export (the view calls).
 * The thread that takes the first queued request gathers the requests behind it in FIFO order while they fit in the
 * batch, waiting at most max_delay_us microseconds from that request's arrival (0: only what is already queued); a
 * request is never split, one that does not fit waits for the next batch, and one thread gathers at a time. Every
 * gathered request is checked before any is staged: a malformed one fails alone and the rest of its batch runs. The Net
 * runs its built batch, with the same plans and CUDA graph; slots no request filled are computed and dropped. Fails
 * for max_delay_us < 0 before anything is loaded, and for a graph with more than one input. */
ANAKIN_API int anakin_worker_create_batching(const char* model_path, int precision, int threads, const int* devices,
                                             int n_devices, int batch, const char* const* nodes, int n,
                                             int64_t max_delay_us, anakin_worker_t** out);
/* Per-image sizes of any Worker once its threads are ready (any pointer may be NULL): the batch, one image of the first
 * input (floats of an fp32 input; bytes of an 8-bit image input, or of the resized tensor of one with on-device resize)
 * and one image's floats of a view result (graph output 0 as stored plus every export). */
ANAKIN_API int anakin_worker_image_sizes(anakin_worker_t* w, int* batch, size_t* in_per_image, size_t* out_per_image);
/* A batching Worker's predictions run so far and the images of the requests they served (their ratio is the mean
 * batch fill). */
ANAKIN_API int anakin_worker_batch_stats(anakin_worker_t* w, uint64_t* predictions, uint64_t* images);
/* The packing decision of a batching Worker, without a device: n queued requests in FIFO order, request i of sizes[i]
 * images (0..batch; 0 = a malformed request, which takes no slot) that arrived at arrive_us[i]. Returns how many
 * leading requests form the batch (the longest prefix that fits), with *close = 1 when it runs now (full, a request
 * left behind it, or now_us >= *deadline_us = arrive_us[0] + max_delay_us), else 0: wait for the deadline or the next
 * arrival and plan again. -1 for n < 0, batch < 1, max_delay_us < 0 or a size outside 0..batch. */
ANAKIN_API int anakin_worker_plan_batch(const int* sizes, const int64_t* arrive_us, int n, int batch,
                                        int64_t max_delay_us, int64_t now_us, int* close, int64_t* deadline_us);
ANAKIN_API void anakin_worker_destroy(anakin_worker_t* w);

#ifdef __cplusplus
}
#endif
#endif /* ANAKIN_B200_H */
