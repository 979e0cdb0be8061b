/*
 * b200_saber.h -- C ABI of the sm_90a device layer that sits behind Anakin's
 * Saber operator surface (SaberConv2D / SaberConvEltwise / SaberConv2DPooling /
 * SaberFc / SaberPooling / SaberSoftmax / SaberEltwise / SaberActivation /
 * SaberScale for target NV).
 *
 * The reference has no C plugin ABI: the boundary is the C++ virtual interface
 *     ImplBase<NV, Dtype, Param>::{init, create, dispatch}
 * (reference saber/funcs/impl/impl_base.h:33-69) plus Conv::trans_weights
 * (saber/funcs/conv.h:103-119).  Each entry point below names the reference
 * interface it replaces; the C++ shims in anakin_b200/csrc/saber/ map the
 * reference's Param structs onto these calls (see INTEGRATION.md).
 *
 * Conventions
 *  - plain C types only; device pointers are void*; streams are cudaStream_t
 *    passed as void* so the header needs no CUDA include.
 *  - status codes are the reference's SaberStatus values
 *    (saber/saber_types.h:223-233): success is -1 (!).
 *  - enum values for dtypes / pooling / eltwise / activation mirror
 *    saber/saber_types.h:205-319 so a shim can pass them through.
 *  - activations are NHWC (channels innermost), channel count padded as
 *    documented per op; all launches are asynchronous on the given stream.
 *  - no CPU fallback exists: on a machine without an sm_90 device every
 *    compute entry point returns B200_WRONG_DEVICE.
 */
#ifndef B200_SABER_H
#define B200_SABER_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_SABER_ABI_VERSION 1

#if defined(__GNUC__)
#define B200_API __attribute__((visibility("default")))
#else
#define B200_API
#endif

/* SaberStatus (saber/saber_types.h:223-233) */
typedef enum {
    B200_SUCCESS = -1,
    B200_NOT_INITIALIZED = 1,
    B200_INVALID_VALUE = 3,
    B200_MEM_ALLOC_FAILED = 7,
    B200_UNKNOWN_ERROR = 15,
    B200_OUT_OF_AUTHORITY = 31,
    B200_OUT_OF_MEM = 63,
    B200_UNIMPL_ERROR = 127,
    B200_WRONG_DEVICE = 255
} b200_status_t;

/* DataType (saber/saber_types.h:205-222) */
typedef enum {
    B200_HALF = 0,
    B200_FLOAT = 1,
    B200_INT8 = 3,
    B200_INT32 = 5,
    B200_UINT8 = 7
} b200_dtype_t;

/* PoolingType (saber/saber_types.h:283-289) */
typedef enum {
    B200_POOL_MAX = 1,
    B200_POOL_AVG_INCLUDE_PAD = 2,
    B200_POOL_AVG_EXCLUDE_PAD = 3
} b200_pool_t;

/* EltwiseType (saber/saber_types.h:290-297) */
typedef enum { B200_ELT_PROD = 1, B200_ELT_SUM = 2, B200_ELT_MAX = 3 } b200_eltwise_t;

/* ActiveType (saber/saber_types.h:259-272) */
typedef enum {
    B200_ACT_NONE = 0,
    B200_ACT_SIGMOID = 1,
    B200_ACT_RELU = 2,
    B200_ACT_TANH = 3,
    B200_ACT_CLIPPED_RELU = 4,
    B200_ACT_ELU = 5,
    B200_ACT_IDENTITY = 6
} b200_act_t;

/* Tensor-core arithmetic kind of a conv / fc plan. */
typedef enum {
    B200_MATH_I8 = 0,   /* u8|s8 x s8 -> s32 (wgmma .s32.u8|s8.s8)                     */
    B200_MATH_F16 = 1,  /* f16 x f16 -> f32 (wgmma .f32.f16.f16)                     */
    B200_MATH_TF32 = 2, /* f32 operands, tf32 multiply, f32 accumulate (wgmma .tf32) */
    B200_MATH_TF32X3 = 3 /* f32 via 3-term error-compensated tf32 split (hi/lo planes) */
} b200_math_t;

B200_API const char* b200_status_string(int status);
B200_API int b200_abi_version(void);
/* 1 if device 0..n-1 has an sm_90 GPU the kernels can run on, else 0. */
B200_API int b200_device_ok(int device);

/* ------------------------------------------------------------------------
 * Convolution family.  Replaces SaberConv2D<NV,*>, SaberConvEltwise<NV,*>,
 * SaberConv2DPooling<NV,*>::{init,create,dispatch}
 * (saber/funcs/impl/cuda/saber_conv.cpp:17-188,190-585,
 *  saber_conv_eltwise.cpp:32-318, saber_conv_pooling.cpp:36-130) and the
 * closed SASS kernels they call (third-party/sass/include/sass_funcs.h:54-935).
 *
 * One plan = one fused op:  out = act( alpha-scaled conv(in) + bias [+ beta*res] )
 * as implicit GEMM on wgmma with TMA-im2col operand staging.
 *
 *   in   NHWC  [n, h, w, c_in_stored]   dtype in_dtype
 *   out  NHWC  [n, ho, wo, ldc]  (first k channels written)  dtype out_dtype
 *   res  same geometry as out, dtype res_dtype (B200 dtype or -1 for none)
 *
 * INT8 epilogue (x86 Saber semantics, reference
 * saber/funcs/impl/x86/kernel/jit_avx512_core_x8s8s32x_conv_kernel.cpp:137-215):
 *   f = (float)acc + bias[oc]; f *= scale[oc]; if (relu && !res) f = max(f,0);
 *   if (res) f = (sum_scale==1) ? f + (float)res : fmaf((float)res, sum_scale, f);
 *   if (relu && res) f = max(f,0);  out = f (fp32) | sat_s8(rne(f)) | sat_u8(rne(f))
 * Float epilogue (saber/funcs/impl/x86/saber_im2col_conv.cpp:161-214,
 * test/saber/conv_func_helper.h:196-264):
 *   f = acc; if (res) f += beta*res; f += bias[oc]; relu with negative slope.
 * ------------------------------------------------------------------------ */
typedef struct {
    int32_t math;     /* b200_math_t */
    int32_t in_dtype; /* B200_INT8|B200_UINT8 (I8), B200_HALF (F16), B200_FLOAT (TF32*) */
    int32_t out_dtype;
    int32_t res_dtype; /* -1: no residual */
    int32_t n, h, w;   /* input geometry */
    int32_t c;         /* stored input channels (multiple of 16 bytes worth) */
    int32_t k;         /* output channels */
    int32_t ldc;       /* output / residual row pitch in elements (>= k) */
    int32_t r, s;      /* filter */
    int32_t pad_h, pad_w, stride_h, stride_w, dil_h, dil_w;
    int32_t relu;      /* 0/1 */
    float neg_slope;   /* float paths only */
    float sum_scale;   /* I8: residual multiplier; float: beta */
    int32_t fuse_pool;  /* 0, or the window w of a w x w MAX pooling fused behind the activation (ConvPooling,
                           saber_conv_pooling.cpp:36-130): `out` is then the POOLED tensor [n, ph, pw, ldc]
                           (b200_conv_pooled_hw). Stride-1 r x s convolutions with r*s > 1, no residual,
                           k * sizeof(out) a 16-byte multiple; anything else: B200_UNIMPL_ERROR from plan_create */
    int32_t pool_stride; /* fused pooling: stride (0 = 2), padding, PoolingParam::cmp_out_shape_floor_as_conv */
    int32_t pool_pad;
    int32_t pool_floor_as_conv;
} b200_conv_desc_t;

typedef struct b200_conv_plan b200_conv_plan_t;

/* Output spatial size per saber/funcs/funcs_utils.h:41-51. */
B200_API int b200_conv_out_hw(const b200_conv_desc_t* d, int32_t* ho, int32_t* wo);
/* Size of what the plan stores: the pooled size (saber/funcs/pooling.h:69-132) when d->fuse_pool, else the conv size. */
B200_API int b200_conv_pooled_hw(const b200_conv_desc_t* d, int32_t* ho, int32_t* wo);

/* Bytes of the packed (wgmma K-major, k-step ordered) weight image. */
B200_API size_t b200_conv_packed_weight_bytes(const b200_conv_desc_t* d);
/* Host-side pack (replaces Conv::trans_weights, saber_conv.cpp:382-585):
 * src is KCRS ([k][c_real][r][s]) in the operand element type (int8 / fp16 bits / fp32);
 * c_real <= d->c, missing channels are zero. dst is host memory. */
B200_API int b200_conv_pack_weights(const b200_conv_desc_t* d, const void* src_kcrs, int32_t c_real,
                           void* dst_packed);

/* bias / scale: device float[k] (may be NULL: bias 0 / scale 1). Pointers must
 * stay valid for the plan's lifetime. */
B200_API int b200_conv_plan_create(const b200_conv_desc_t* d, const void* packed_weights_dev,
                          const float* bias_dev, const float* scale_dev,
                          b200_conv_plan_t** plan);
B200_API int b200_conv_plan_run(b200_conv_plan_t* plan, const void* in, const void* res, void* out,
                       void* stream);
B200_API void b200_conv_plan_destroy(b200_conv_plan_t* plan);
/* Introspection for tests / roofline: tile shape and grid the plan chose. */
B200_API int b200_conv_plan_info(const b200_conv_plan_t* plan, int32_t* block_n, int32_t* grid_x,
                        int32_t* grid_y, int32_t* k_steps, int32_t* smem_bytes);
/* split-K factor of the plan (= cluster size along z; 1 when the k loop is not split), 0 for a null plan. */
B200_API int b200_conv_plan_split(const b200_conv_plan_t* plan);
/* 1 when the plan runs the slab-staged stride-1 R x S kernel (the input rectangle of a tile is staged once per
 * channel chunk and the filter taps are row-shifted views of it) instead of the TMA-im2col kernel. */
B200_API int b200_conv_plan_is_slab(const b200_conv_plan_t* plan);
/* 1 when the plan runs the persistent tile-pipelined kernel (one CTA per SM walks the tile list, register accumulators:
 * the epilogue of a tile overlaps the main loop of the next) -- chosen for grids of more than two tiles per SM. */
B200_API int b200_conv_plan_is_persistent(const b200_conv_plan_t* plan);

/* ------------------------------------------------------------------------
 * Depthwise convolution (MobileNet). Replaces SaberDepthWiseConv
 * (saber/funcs/impl/cuda/base/cuda_c/saber_depthwiseconv_act.cu:10-295).
 * weights: device [r][s][c] in out math type (float / half / int8).
 * ------------------------------------------------------------------------ */
B200_API int b200_dwconv_run(const b200_conv_desc_t* d, const void* in, const void* weights_rsc,
                    const float* bias, const float* scale, void* out, void* stream);

/* ------------------------------------------------------------------------
 * Fully connected. Replaces SaberFc<NV,*> (saber/funcs/impl/cuda/base/cuda_c/
 * saber_fc.cu:17-195): out[m][n] = sum_k in[m][k]*W[n][k] + b[n].
 * Implemented on the conv plan (1x1 conv over an [m,1,1,k] tensor); this is a
 * convenience wrapper that fills the descriptor.
 * ------------------------------------------------------------------------ */
B200_API int b200_fc_desc(b200_conv_desc_t* d, int32_t math, int32_t in_dtype, int32_t out_dtype, int32_t m,
                 int32_t k_in, int32_t n_out);

/* ------------------------------------------------------------------------
 * Weight-streaming inner product for m <= b200_fc_stream_max_rows() rows. Replaces SaberFc<NV,*>::dispatch
 * (saber/funcs/impl/cuda/base/cuda_c/saber_fc.cu:17-195, ker_gemm.cu:8-186 / cuBLAS) where the layer is a stream of
 * its weights past a few input rows: every weight byte is read once.
 *   x        [m][ldx]      operand dtype (u8|s8 for I8, f16 for F16, f32 for TF32 / TF32X3 -- computed in plain fp32)
 *   w_plain  [n_out][k]    operand dtype, k contiguous, in the STORED order of x's row (k = ldx; zero on padding)
 *   out      [m][ldo]      out_dtype;  int8 epilogue f = (acc + bias) * scale, relu, rne + saturate (as the conv plan)
 * ------------------------------------------------------------------------ */
typedef struct {
    int32_t math;       /* b200_math_t */
    int32_t in_dtype, out_dtype;
    int32_t m, k, ldx;  /* rows, reduction length, input row pitch (elements); k*es and ldx*es multiples of 16 bytes */
    int32_t n_out, ldo; /* output columns, output row pitch (elements) */
    int32_t relu;
    float neg_slope;
} b200_fc_stream_desc_t;
B200_API int b200_fc_stream_max_rows(void);
B200_API int b200_fc_stream_run(const b200_fc_stream_desc_t* d, const void* x, const void* w_plain, const float* bias,
                                const float* scale, void* out, void* stream);

/* INT8 classification head in one launch: global pooling over hw pixels of an NHWC tensor [m][hw][k]
 * (saber_pooling.cu; AVG divides by hw, rounds to nearest even and saturates), the inner product above on the pooled
 * rows, and -- when prob is given -- a row softmax of the fp32 logits (saber_softmax.cu). The reduction dimension is
 * split over the CTAs and combined with integer atomics (exact, order-free); the last CTA applies the epilogue and the
 * softmax. The pooled rows and the logits are written to their own tensors exactly as the three separate ops would
 * write them. `workspace`: b200_head_workspace_bytes(d) bytes of ZEROED device memory owned by the caller, one per
 * concurrently running stream (the kernel leaves it zeroed). math I8, fp32 logits, m <= 8; anything else returns
 * B200_UNIMPL_ERROR and the caller runs the three ops. */
typedef struct {
    b200_fc_stream_desc_t fc; /* ldx == k == stored channels of the pooled tensor */
    int32_t hw;               /* pixels pooled per row */
    int32_t pool_max;         /* 1 max, 0 average */
    int32_t ldp;              /* prob row pitch (elements) */
} b200_head_desc_t;
B200_API size_t b200_head_workspace_bytes(const b200_head_desc_t* d);
B200_API int b200_head_run(const b200_head_desc_t* d, const void* in, void* pooled, const void* w_plain, const float* bias,
                           const float* scale, void* logits, float* prob, void* workspace, void* stream);

/* ------------------------------------------------------------------------
 * Pooling. Replaces SaberPooling<NV,*> / VenderPooling
 * (saber/funcs/impl/cuda/base/cuda_c/saber_pooling.cu:20-229, vender_pooling.cpp).
 * NHWC in/out, c multiple of (16 / sizeof(elem)).
 * Output size rule: saber/funcs/pooling.h:69-132 (b200_pool_out_hw). Negative padding: B200_INVALID_VALUE.
 * ------------------------------------------------------------------------ */
typedef struct {
    int32_t dtype; /* B200_FLOAT | B200_HALF | B200_INT8 | B200_UINT8 */
    int32_t type;  /* b200_pool_t */
    int32_t n, h, w, c;
    int32_t window_h, window_w, pad_h, pad_w, stride_h, stride_w;
    int32_t global_pooling;
    int32_t floor_as_conv; /* PoolingParam::cmp_out_shape_floor_as_conv */
    int32_t reserved[2];
} b200_pool_desc_t;
B200_API int b200_pool_out_hw(const b200_pool_desc_t* d, int32_t* ho, int32_t* wo);
B200_API int b200_pool_run(const b200_pool_desc_t* d, const void* in, void* out, void* stream);

/* ------------------------------------------------------------------------
 * Softmax over the innermost `axis_size` elements of [outer][axis_size] fp32
 * rows. Replaces SaberSoftmax<NV,AK_FLOAT>
 * (saber/funcs/impl/cuda/base/cuda_c/saber_softmax.cu:175-430) for inner == 1,
 * and the strided form for inner > 1.
 * ------------------------------------------------------------------------ */
B200_API int b200_softmax_run(const float* in, float* out, int32_t outer, int32_t axis_size, int32_t inner,
                     void* stream);
/* Row softmax with explicit row pitches (elements): NHWC tensors whose channel count is padded. */
B200_API int b200_softmax_rows(const float* in, float* out, int32_t rows, int32_t len, int32_t in_pitch,
                      int32_t out_pitch, void* stream);

/* ------------------------------------------------------------------------
 * Eltwise (2 inputs) with optional fused relu. Replaces SaberEltwise<NV,*>
 * (saber/funcs/impl/cuda/base/cuda_c/saber_eltwise.cu:6-360).
 * float: out = c0*a + c1*b | a*b | max(a,b), then relu.
 * int8 (x86 EltwiseRelu semantics): out = sat(rne(a*sa + b*sb)) with sa,sb the
 * per-input rescale factors, optional relu.
 * ------------------------------------------------------------------------ */
B200_API int b200_eltwise_run(int32_t dtype_a, int32_t dtype_b, int32_t dtype_out, int32_t op,
                     const void* a, const void* b, void* out, size_t count, float c0, float c1,
                     int32_t relu, void* stream);

/* Pointwise activation (SaberActivation<NV,*>, saber_activation.cu:11-420). fp32/fp16. */
B200_API int b200_activation_run(int32_t dtype, int32_t act, const void* in, void* out, size_t count,
                        float neg_slope, float coef, void* stream);

/* Per-channel scale y = x*w[c] (+ b[c]) on NHWC (SaberScale<NV,*>, saber_scale.cu:8-70). */
B200_API int b200_scale_run(int32_t dtype, const void* in, void* out, size_t pixels, int32_t c,
                   const float* w, const float* b, void* stream);

/* ------------------------------------------------------------------------
 * Layout / precision transforms at graph boundaries. Replaces calibrate.cu
 * (saber/funcs/impl/cuda/base/cuda_c/calibrate.cu:10-700) and reorder.cu.
 *   nchw_to_nhwc: fp32 NCHW [n,c,h,w] -> NHWC [n,h,w,c_pad] in out_dtype.
 *      FLOAT: copy (zero pad). HALF: rn convert.
 *      INT8:  secur_cast2char(x * inv_scale) = clamp(roundf(.)) (x86_utils.h:325-347)
 *      UINT8: truncation of x*inv_scale (x86_utils.h:360-372)
 *      split_hi_lo != 0 (FLOAT only): write [hi | lo] tf32 planes, c_pad each.
 *   nhwc_to_nchw: NHWC in_dtype -> fp32 NCHW, multiply by scale (dequantise).
 * ------------------------------------------------------------------------ */
B200_API int b200_nchw_to_nhwc(const float* in, void* out, int32_t out_dtype, int32_t n, int32_t c, int32_t h,
                      int32_t w, int32_t c_pad, float inv_scale, int32_t split_hi_lo, void* stream);
/* Stem pack for the first conv (C <= 4, filter width s <= 8, dilation 1): fp32 NCHW ->
 *   X2[n][h + 2*pad_h][wo][taps][4] in out_dtype  (taps = 4 or 8 >= s, wo = conv output width)
 * so that the R x S conv becomes an R x 1 conv over X2 with c = taps*4, stride_w 1, pad 0 on the
 * tensor-core plan (weights laid out [k][tap*4+ch][r]). Quantisation as in b200_nchw_to_nhwc. */
B200_API int b200_stem_pack(const float* in, void* out, int32_t out_dtype, int32_t n, int32_t c, int32_t h,
                   int32_t w, int32_t pad_h, int32_t pad_w, int32_t s, int32_t stride_w, int32_t taps,
                   float inv_scale, void* stream);
B200_API int b200_nhwc_to_nchw(const void* in, int32_t in_dtype, float* out, int32_t n, int32_t c, int32_t h,
                      int32_t w, int32_t c_pad, float scale, void* stream);

/* ------------------------------------------------------------------------
 * Stem convolution: the graph-input conv (fp32 NCHW input with c <= 4 channels, filter width <= 8, dilation 1),
 * its bias / scale / relu epilogue and -- with fuse_pool = 1 -- the MAX pooling that follows it, in one launch.
 * Replaces SaberConv2DPooling<NV,*>::{create,dispatch} (saber/funcs/impl/cuda/saber_conv_pooling.cpp:36-130; the SASS
 * winograd_conv_relu_pooling / direct_conv_bias_relu_maxpool2k2s0p_* entry points, sass_funcs.h:54-427) and the input
 * quantisation the reference's conv runs on its own input (saber_conv.cpp:341-381) for that layer: the input is
 * quantised (INT8: clamp(roundf(x * in_inv_scale)), x86_utils.h:318-347) / converted in shared memory, never in HBM.
 *   in   fp32 NCHW [n, c, h, w]
 *   out  NHWC [n, oh, ow, ldc] out_dtype, first k channels written; (oh, ow) = the pooled size when fuse_pool,
 *        else the conv size (b200_stem_conv_out_hw)
 *   weights: b200_stem_pack_weights of the operand-typed KCRS image ([k][c][r][s] int8 / fp16 bits / fp32)
 * Epilogue numerics are the conv plan's (see above); pooling is applied to the requantised values, so the result is
 * bit-identical to conv plan -> b200_pool_run. Pooling other than MAX, or k * sizeof(out) not a 16-byte multiple,
 * returns B200_UNIMPL_ERROR (the caller runs the separate ops).
 * ------------------------------------------------------------------------ */
typedef struct {
    int32_t math;      /* b200_math_t */
    int32_t out_dtype;
    int32_t n, c, h, w;
    int32_t k, ldc;
    int32_t r, s, stride_h, stride_w, pad_h, pad_w;
    int32_t relu;
    float neg_slope;
    float in_inv_scale; /* INT8: 1 / input scale */
    int32_t fuse_pool;  /* 0 | 1 */
    int32_t pool_type;  /* a b200_pool_t value: B200_POOL_MAX is what fuses */
    int32_t pool_window_h, pool_window_w, pool_pad_h, pool_pad_w, pool_stride_h, pool_stride_w;
    int32_t pool_global, pool_floor_as_conv;
    int32_t monotone_epilogue; /* caller's promise: every scale[] entry is > 0 (INT8) and neg_slope >= 0, i.e. the
                                  epilogue is non-decreasing in the accumulator. The fused pooling then runs on the raw
                                  accumulators and only pooled pixels pay for the epilogue -- same bits, less work */
    int32_t reserved[1];
} b200_stem_desc_t;
B200_API int b200_stem_conv_out_hw(const b200_stem_desc_t* d, int32_t* oh, int32_t* ow);
B200_API size_t b200_stem_packed_weight_bytes(const b200_stem_desc_t* d);
B200_API int b200_stem_pack_weights(const b200_stem_desc_t* d, const void* src_kcrs, void* dst_packed);
/* tile the kernel chose: conv rectangle per CTA, output channels per CTA, CTA count, shared memory */
B200_API int b200_stem_conv_info(const b200_stem_desc_t* d, int32_t* tile_h, int32_t* tile_w, int32_t* block_n,
                                 int32_t* ctas, int32_t* smem_bytes);
B200_API int b200_stem_conv_run(const b200_stem_desc_t* d, const float* in_nchw, const void* packed_weights_dev,
                                const float* bias_dev, const float* scale_dev, void* out, void* stream);

/* ------------------------------------------------------------------------
 * 8-bit image graph input: uint8 pixels, interleaved HWC, images contiguous ([n][h][w][c], 1 <= c <= 4, no row
 * padding). The network sees the fp32 tensor
 *     x[n][i][y][x] = ((float)img[n][y][x][src_channel[i]] - mean[i]) * scale[i]
 * with both operations rounded to fp32 (no fused multiply-add): bit for bit numpy's
 * (u.astype(np.float32) - mean) * scale in float32. Convolution zero padding applies to x (an out-of-image tap is
 * 0.0, not the normalised value of a zero byte); then quantisation / conversion are those of the fp32 input.
 * Entries i >= c are ignored. B200_INVALID_VALUE for c outside 1..4, a src_channel that is not a permutation of
 * 0..c-1, a non-finite mean or scale, or a null pointer.
 * ------------------------------------------------------------------------ */
typedef struct {
    int32_t src_channel[4]; /* network channel i reads image channel src_channel[i]; {2,1,0} swaps BGR <-> RGB */
    float mean[4], scale[4]; /* x = ((float)u - mean[i]) * scale[i], no FMA */
} b200_image_desc_t;
/* b200_stem_conv_run on an 8-bit image: same descriptor (n, c, h, w are the image's), same output, the input
 * normalised while the patch is staged in shared memory. */
B200_API int b200_stem_conv_run_image(const b200_stem_desc_t* d, const b200_image_desc_t* img, const uint8_t* in_nhwc,
                                      const void* packed_weights_dev, const float* bias_dev, const float* scale_dev,
                                      void* out, void* stream);
/* b200_nchw_to_nhwc (split_hi_lo = 0) on an 8-bit image: normalised image -> NHWC [n,h,w,c_pad] in out_dtype, with
 * the same conversion / quantisation rules; channels c..c_pad-1 are written as zero. Any c_pad >= c is accepted. */
B200_API int b200_image_to_nhwc(const b200_image_desc_t* img, const uint8_t* in, void* out, int32_t out_dtype, int32_t n,
                                int32_t c, int32_t h, int32_t w, int32_t c_pad, float inv_scale, void* stream);

/* ------------------------------------------------------------------------
 * Resize and centre-crop of 8-bit images of any size to the image input's out_h x out_w (classification
 * preprocessing: short side to S, centre crop). Image i (h x w) is resized to rh x rw and the crop starts at
 * (top, left) of the resized image:
 *   S == 0: (rh, rw) = (out_h, out_w), top = left = 0 (stretch);
 *   S  > 0: the short side becomes S -- h <= w: rh = S, rw = floor(S*w/h); else rw = S, rh = floor(S*h/w) (64-bit
 *           integers) -- and top = (rh - out_h) / 2, left = (rw - out_w) / 2 (floor). S must be >= max(out_h, out_w).
 * Output pixel (y, x), channel j, is the reference's BILINEAR_NO_ALIGN resize (x86 saber_resize.cpp,
 * resize_bilinear_no_align_kernel) evaluated at resized coordinates (y + top, x + left):
 *   fh = ((float)h / (float)rh) * ((float)(y + top) + 0.5f) - 0.5f, every step rounded to fp32, no FMA; fh = max(fh, 0)
 *   y0 = (int)fh, y1 = y0 + (y0 < h - 1), fh -= y0                       (x likewise with w, rw, left)
 *   w00 = (float)((1.0 - fh) * (1.0 - fw)), w01 = (float)(fw * (1.0 - fh)), w10 = (float)(fh * (1.0 - fw)),
 *   w11 = (float)(fw * fh)                                                (double products, rounded once)
 *   v = ((w00 * p[y0][x0] + w01 * p[y0][x1]) + w10 * p[y1][x0]) + w11 * p[y1][x1]   (fp32, no FMA)
 *   out = saturate(rint(v))                                                (round half to even)
 * No antialiasing: a downscale samples 2 x 2 source pixels per output pixel.
 * ------------------------------------------------------------------------ */
typedef struct {
    int32_t n, c;         /* images, channels (1..4) */
    int32_t out_h, out_w; /* the image input's H x W */
} b200_image_resize_desc_t;
/* One entry per image of the device table b200_image_resize_run reads (filled on the host with
 * b200_image_resize_geometry). */
typedef struct {
    int64_t offset;         /* byte offset of the image's pixels (h*w*c bytes, rows unpadded) in `src` */
    int32_t h, w;           /* source size */
    int32_t rh, rw;         /* resized size */
    int32_t top, left;      /* crop offsets in the resized image */
} b200_image_resize_entry_t;
/* The geometry above (host only, no device needed): B200_INVALID_VALUE for h, w, out_h or out_w < 1, h or w above
 * 2^23, S < 0, 0 < S < max(out_h, out_w), or rh / rw above 2^23 (pixel-centre coordinates stop being exact in fp32);
 * B200_SUCCESS otherwise, with *rh, *rw, *top, *left filled. */
B200_API int b200_image_resize_geometry(int32_t h, int32_t w, int32_t resize_short, int32_t out_h, int32_t out_w,
                                        int32_t* rh, int32_t* rw, int32_t* top, int32_t* left);
/* Resize + crop of d->n images into out = uint8 [n][out_h][out_w][c] (the image input tensor). table_dev: device
 * array of n b200_image_resize_entry_t. The launch depends only on *d; every per-image size is read from the table,
 * so one captured CUDA graph serves requests of any sizes. B200_INVALID_VALUE for a null pointer, n < 1, c outside
 * 1..4 or out_h / out_w < 1 (checked before the device check). */
B200_API int b200_image_resize_run(const b200_image_resize_desc_t* d, const uint8_t* src, const void* table_dev,
                                   uint8_t* out, void* stream);

/* Kernel-launch counter (every launch made through this library). */
B200_API uint64_t b200_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* B200_SABER_H */
