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

#define B200_SABER_ABI_VERSION 2

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
    B200_UINT8 = 7,
    B200_FP8E4M3 = 32 /* OCP e4m3fn codes (no reference counterpart; a value no DataType uses) */
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
    /* 2: retired (single-pass tf32, ABI version 1); refused with B200_UNIMPL_ERROR */
    B200_MATH_TF32X3 = 3, /* f32 via 3-term error-compensated tf32 split (hi/lo planes) */
    B200_MATH_E4M3 = 4   /* e4m3 x e4m3 -> f32 (wgmma .f32.e4m3.e4m3)                  */
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
 * E4M3 epilogue (math B200_MATH_E4M3; in, weights and residual are B200_FP8E4M3 codes, out FP8E4M3 or fp32).
 *   Codec: OCP e4m3fn, no infinities, max finite +-448, smallest subnormal 2^-9. enc rounds to nearest even and
 *   saturates to +-448; dec is exact. An edge holds e = enc(x / sigma), one sigma per tensor; weights
 *   w_e = enc(w / sigma_w[k]) per output channel. The tensor cores sum the exact products in fp32 (or narrower);
 *   split-K partials are fp32, summed in rank order. Then, with acc the sum of dec(x_e) * dec(w_e):
 *   f = (acc + bias[oc]) * scale[oc]; if (res) f = fmaf(dec(res), sum_scale, f); if (relu) f = f > 0 ? f : +0;
 *   out = enc(f) (FP8E4M3) | f (fp32), each step rounded to fp32 on its own. The caller's tables are
 *   bias = b / (sigma_w * sigma_in), scale = sigma_w * sigma_in / sigma_out, sum_scale = sigma_res / sigma_out
 *   (sigma_out = 1 for an fp32 output). A fused MAX pooling compares decoded values and keeps the codes.
 * Float epilogue (saber/funcs/impl/x86/saber_im2col_conv.cpp:161-214,
 * test/saber/conv_func_helper.h:196-264):
 *   f = acc; if (res) f += beta*res; f += bias[oc]; relu with negative slope.
 * ------------------------------------------------------------------------ */
typedef struct {
    int32_t math;     /* b200_math_t */
    int32_t in_dtype; /* B200_INT8|B200_UINT8 (I8), B200_HALF (F16), B200_FLOAT (TF32*), B200_FP8E4M3 (E4M3) */
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

/* Kernel of a conv plan. */
typedef enum {
    B200_CONV_KERNEL_TILE = 0,       /* TMA-im2col implicit GEMM, one CTA (or split-K cluster) per tile */
    B200_CONV_KERNEL_PERSISTENT = 1, /* the same kernel as a persistent walker over the tile list */
    B200_CONV_KERNEL_SLAB = 2        /* slab-staged stride-1 r x s kernel (see b200_conv_plan_is_slab) */
} b200_conv_kernel_t;

/* The plan b200_conv_plan_create would build for a descriptor, as chosen on a device with sm_count SMs. */
typedef struct {
    int32_t kernel;         /* b200_conv_kernel_t */
    int32_t block_n;        /* tile width (output channels per tile) */
    int32_t split;          /* split-K factor (cluster size along z), 1 when the k loop is not split */
    int32_t stages;         /* operand ring depth of the im2col kernels; 0 for the slab kernel */
    int32_t smem_bytes;     /* dynamic shared memory per CTA */
    int32_t grid_x, grid_y; /* tiles along M (slab: output rectangles) and along N */
    int32_t k_steps;        /* k steps of the packed weights (b200_conv_plan_info) */
    int32_t ctas;           /* CTAs launched: grid_x * grid_y * split, or the persistent walker's count */
    int32_t tile_h, tile_w; /* slab kernel: output rectangle of a CTA; 0 otherwise */
} b200_conv_plan_choice_t;
/* Device-free planning: fills *out with the plan b200_conv_plan_create would build on a device of sm_count SMs, under
 * the same B200_SABER_* switches, and returns the status it would return (B200_WRONG_DEVICE and B200_NOT_INITIALIZED
 * apart). *out is zeroed when the descriptor is refused. */
B200_API int b200_conv_plan_choose(const b200_conv_desc_t* d, int32_t sm_count, b200_conv_plan_choice_t* out);

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
 *   nhwc_to_nchw: NHWC in_dtype -> fp32 NCHW, multiply by scale (dequantise).
 * ------------------------------------------------------------------------ */
B200_API int b200_nchw_to_nhwc(const float* in, void* out, int32_t out_dtype, int32_t n, int32_t c, int32_t h,
                      int32_t w, int32_t c_pad, float inv_scale, void* stream);
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
/* b200_nchw_to_nhwc on an 8-bit image: normalised image -> NHWC [n,h,w,c_pad] in out_dtype, with
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

/* ------------------------------------------------------------------------
 * The Pillow filter: torchvision's Resize(S) + CenterCrop on PIL images, bit for bit (Pillow's antialiased 8-bit
 * BILINEAR resampler, modes L / RGB / RGBX / CMYK; not RGBA / LA, which Pillow premultiplies).
 * Sizes as above; the crop offsets round half to even: top = round((rh - out_h) / 2), left likewise.
 * Per axis (source size in, resized size out, output coordinate o = y + top or x + left), in IEEE double, each step
 * rounded on its own (Pillow's precompute_coeffs):
 *   scale = in / out; support = max(scale, 1.0); ss = 1.0 / support; center = (o + 0.5) * scale
 *   xmin = max((int)(center - support + 0.5), 0); xmax = min((int)(center + support + 0.5), in) - xmin
 *   w[t] = tri(((double)(t + xmin) - center + 0.5) * ss), t < xmax, tri(x) = |x| < 1 ? 1 - |x| : 0
 *   ww = w[0] + w[1] + ... (left to right); w[t] = ww != 0 ? w[t] / ww : w[t]
 *   k[t] = (int32)(w[t] * 2^22 + 0.5)   (w[t] * 2^22 - 0.5 when negative; truncation)
 * A pass computes clamp((2^21 + sum_t p[xmin + t] * k[t]) >> 22, 0, 255) per channel in int32 and stores uint8.
 * Passes run horizontal then vertical, except for an image with h > 100 * w and rh < h, which Pillow's Image.resize
 * runs vertical first; the order changes the 8-bit intermediate, so it is kept.
 *
 * Pillow's BICUBIC (B200_IMAGE_RESIZE_PIL_BICUBIC; torchvision's Resize(S, interpolation=BICUBIC) + CenterCrop):
 * the same sizes, crop offsets, bounds, normalisation, passes and pass order, with the cubic convolution filter of
 * a = -0.5 and support 2 in place of the triangle. Per axis, in IEEE double, each step rounded on its own:
 *   filterscale = max(in / out, 1.0); support = 2.0 * filterscale; ss = 1.0 / filterscale (not 1.0 / support)
 *   w[t] = cubic(((double)(t + xmin) - center + 0.5) * ss), with x = |x| and
 *   cubic(x) = ((1.5 * x - 2.5) * x) * x + 1                 for x < 1
 *              (((x - 5) * x + 8) * x - 4) * (-0.5)          for 1 <= x < 2
 *              0                                             otherwise
 * Taps can be negative (rounded away from zero as above), and a pass's sum can leave [0, 255 * 2^22] near sharp
 * edges, where the clamp to 0..255 applies. These are the bytes of x86-64 Pillow, which evaluates the filter
 * without contraction into fused multiply-adds.
 *
 * OpenCV's INTER_LINEAR (B200_IMAGE_RESIZE_CV2_LINEAR): the bytes of cv2.resize(img, (rw, rh)) with the default
 * interpolation on 8-bit images, cropped as img[top:top + out_h, left:left + out_w] with the floor offsets above (those
 * of the reference filter). Bit for bit OpenCV 4.13 on x86-64. No antialiasing: a shrink reads 2 x 2 source pixels per
 * output pixel. Per axis (source size in, resized size out, output coordinate d = y + top or x + left):
 *   scale = 1.0 / ((double)out / in)                     (double; in / out gives other bytes)
 *   f = (float)((d + 0.5) * scale - 0.5);  s = floor(f);  f -= s                   (f - s in fp32)
 *   columns: s < 0 -> s = 0, f = 0;  s + 1 >= in -> s = in - 1, f = 0;  taps s, s + 1
 *   rows:    taps clamp(s, 0, in - 1) and clamp(s + 1, 0, in - 1), f unchanged (an upscale's first and last rows
 *            weight one row by both coefficients)
 *   a0 = rint((1.0f - f) * 2048),  a1 = rint(f * 2048)  (fp32, half to even; column weights a, row weights b)
 * Per channel, in int32, with arithmetic shifts:
 *   S0 = p[y0][x0] * a0 + p[y0][x1] * a1,  S1 = p[y1][x0] * a0 + p[y1][x1] * a1       (exact)
 *   v = (((S0 >> 4) * b0) >> 16) + (((S1 >> 4) * b1) >> 16);  out = (v + 2) >> 2     (v <= 1020)
 * Equal sizes give a copy and every exact 2x shrink the rounded mean of each 2 x 2 block, (sum + 2) >> 2, both as
 * cv2 computes them. One exception: for c = 2 shrunk exactly 2x on both axes (h = 2 * rh, w = 2 * rw) cv2 uses its
 * float area filter, which rounds half to even: out = (v + 1 + ((v >> 2) & 1)) >> 2, v the block's sum. No case is
 * refused beyond the geometry's own limits.
 * ------------------------------------------------------------------------ */
enum {
    B200_IMAGE_RESIZE_REFERENCE = 0,   /* b200_image_resize_run: the reference's BILINEAR_NO_ALIGN, no antialiasing */
    B200_IMAGE_RESIZE_PIL = 1,         /* b200_image_resize_pil_run: Pillow's BILINEAR, antialiased */
    B200_IMAGE_RESIZE_PIL_BICUBIC = 3, /* b200_image_crop_resize_run: Pillow's BICUBIC, antialiased (2 is unused) */
    B200_IMAGE_RESIZE_CV2_LINEAR = 5   /* b200_image_crop_resize_run: OpenCV's INTER_LINEAR (4 is unused) */
};
/* b200_image_resize_geometry for a filter: the same sizes and, for both Pillow filters, the half-to-even crop
 * offsets (floor offsets for the reference filter and B200_IMAGE_RESIZE_CV2_LINEAR). B200_INVALID_VALUE for an unknown
 * filter or where b200_image_resize_geometry refuses. */
B200_API int b200_image_resize_geometry_ex(int32_t h, int32_t w, int32_t resize_short, int32_t out_h, int32_t out_w,
                                           int32_t filter, int32_t* rh, int32_t* rw, int32_t* top, int32_t* left);
/* *bytes of device workspace the resize of `filter` needs for images up to max_h x max_w resized with resize_short.
 * The reference filter and B200_IMAGE_RESIZE_CV2_LINEAR need none (0 bytes; max_h, max_w and resize_short are
 * ignored). A Pillow filter needs the tap
 * records of every cropped row and column (2 + kmax int32 each) and one uint8 intermediate per image, sized for
 * whichever pass order needs more. kmax = 2 * ceil(f * largest scale) + 1, at least 2 * f + 1, for the filter's
 * support f: 1 for B200_IMAGE_RESIZE_PIL, 2 for B200_IMAGE_RESIZE_PIL_BICUBIC (at max 16384 -> 224, 149 and 295).
 * B200_INVALID_VALUE for a null pointer, an unknown filter, a desc b200_image_resize_run refuses, and for a Pillow
 * filter max_h / max_w outside 1..2^23, S < 0 or 0 < S < max(out_h, out_w). */
B200_API int b200_image_resize_workspace(const b200_image_resize_desc_t* d, int32_t filter, int32_t max_h,
                                         int32_t max_w, int32_t resize_short, size_t* bytes);
/* b200_image_resize_workspace(d, B200_IMAGE_RESIZE_PIL, max_h, max_w, resize_short, bytes). */
B200_API int b200_image_resize_pil_workspace(const b200_image_resize_desc_t* d, int32_t max_h, int32_t max_w,
                                             int32_t resize_short, size_t* bytes);
/* The Pillow filter's resize + crop of d->n images into out = uint8 [n][out_h][out_w][c]: three launches (taps,
 * first pass, second pass), all computed on the device from table_dev (entries filled with
 * b200_image_resize_geometry_ex(..., B200_IMAGE_RESIZE_PIL, ...), every h <= max_h and w <= max_w). The launches
 * depend only on the arguments, so one captured CUDA graph serves requests of any sizes. `workspace` holds
 * b200_image_resize_pil_workspace bytes. Argument errors (B200_INVALID_VALUE) are checked before the device.
 * BILINEAR only, as is b200_image_resize_pil_yuv_run; b200_image_crop_resize_run runs either Pillow filter. */
B200_API int b200_image_resize_pil_run(const b200_image_resize_desc_t* d, int32_t max_h, int32_t max_w,
                                       int32_t resize_short, const uint8_t* src, const void* table_dev,
                                       void* workspace, uint8_t* out, void* stream);

/* ------------------------------------------------------------------------
 * YUV 4:2:0 sources (video decoders, camera pipelines) for either filter, c = 3. A frame is h x w with h and w even,
 * h*w*3/2 bytes at its table entry's offset, rows unpadded:
 *   B200_IMAGE_YUV_NV12: the h x w Y plane, then h/2 rows of w bytes of interleaved U,V;
 *   B200_IMAGE_YUV_I420: the h x w Y plane, then the (h/2) x (w/2) U plane, then the V plane.
 * The image the filters resize is OpenCV's cvtColor(frame, COLOR_YUV2RGB_NV12 / COLOR_YUV2RGB_I420), channels R, G, B:
 * pixel (y, x) takes the chroma sample (y/2, x/2) (no chroma interpolation) and BT.601 limited range in int32,
 *   yy = max(Y - 16, 0) * 1220542;  u = U - 128;  v = V - 128;  half = 1 << 19
 *   R = sat8((yy + half + 1673527*v) >> 20)
 *   G = sat8((yy + half - 852492*v - 409993*u) >> 20)
 *   B = sat8((yy + half + 2116026*u) >> 20)                  (>> arithmetic, sat8 clamps to 0..255)
 * Each source tap is converted as it is read, so the output is, byte for byte, the filter applied to the converted
 * image (the Pillow filter's 8-bit intermediate and pass order included). The table, the geometry and the launches are
 * those of the interleaved entry points; the Pillow filter's workspace is b200_image_resize_pil_workspace of *d.
 * ------------------------------------------------------------------------ */
enum {
    B200_IMAGE_INTERLEAVED = 0, /* h x w x c interleaved bytes (b200_image_crop_resize_run's pixel_format) */
    B200_IMAGE_YUV_NV12 = 1,
    B200_IMAGE_YUV_I420 = 2
};
/* b200_image_resize_run on YUV frames of `format`. B200_INVALID_VALUE for d->c != 3, an unknown format or whatever
 * b200_image_resize_run refuses (checked before the device check). */
B200_API int b200_image_resize_yuv_run(const b200_image_resize_desc_t* d, int32_t format, const uint8_t* src,
                                       const void* table_dev, uint8_t* out, void* stream);
/* b200_image_resize_pil_run on YUV frames of `format`. B200_INVALID_VALUE for d->c != 3, an unknown format or whatever
 * b200_image_resize_pil_run refuses (checked before the device check). */
B200_API int b200_image_resize_pil_yuv_run(const b200_image_resize_desc_t* d, int32_t format, int32_t max_h,
                                           int32_t max_w, int32_t resize_short, const uint8_t* src,
                                           const void* table_dev, void* workspace, uint8_t* out, void* stream);

/* ------------------------------------------------------------------------
 * Crop boxes out of frames (a detector's regions, classified one by one), for either filter and every layout above.
 *   A box is (frame, top, left, height, width) in int32 pixels of its frame.
 *   A box lies inside its frame: top, left >= 0, height, width >= 1, top + height <= h, left + width <= w. Boxes are
 *   never clamped.
 *   The image a box gives is the image above for the array frame[top:top+height, left:left+width]: that array is the
 *   "image" of b200_image_resize_geometry_ex, with the same filter, geometry, pass-order rule (judged on the box) and
 *   crop offsets. With B200_IMAGE_RESIZE_PIL this is torchvision's
 *   CenterCrop((out_h, out_w))(Resize(S)(img.crop((left, top, left + width, top + height)))), and
 *   torchvision.transforms.functional.resized_crop(img, top, left, height, width, (out_h, out_w)) when S = 0.
 *   Taps are clipped at the box's edges, never the frame's: no pixel outside the box influences the result.
 *   In a YUV frame any offset and size is allowed, odd ones included: box pixel (y, x) converts with chroma sample
 *   ((top + y) / 2, (left + x) / 2) of the frame, so the box is cut from the frame's cvtColor. Frames keep even sizes.
 * ------------------------------------------------------------------------ */
typedef struct {
    b200_image_resize_entry_t r; /* offset: the frame's; h, w: the box's size; rh, rw, top, left: the box's geometry */
    int32_t frame_h, frame_w;    /* the frame's size */
    int32_t box_top, box_left;   /* the box's origin in the frame */
} b200_image_crop_entry_t;
/* Resize + crop of d->n boxes into out = uint8 [n][out_h][out_w][c]: table_dev is a device array of n
 * b200_image_crop_entry_t, `filter` a B200_IMAGE_RESIZE_* and pixel_format B200_IMAGE_INTERLEAVED (c = 1..4) or
 * B200_IMAGE_YUV_NV12 / _I420 (c = 3). The launches are those of the whole-image entry points (one for the reference
 * filter, three for Pillow's; one for B200_IMAGE_RESIZE_CV2_LINEAR, which only this entry point runs) and depend only
 * on the arguments, so one captured CUDA graph serves any mix of frames and boxes. B200_IMAGE_RESIZE_PIL and
 * _PIL_BICUBIC need b200_image_resize_workspace(d, filter, max_h, max_w, resize_short) bytes of workspace with every
 * frame within max_h x max_w; the reference filter and _CV2_LINEAR ignore max_h, max_w, resize_short and workspace.
 * B200_INVALID_VALUE (checked before the device check) for an unknown filter or format,
 * c != 3 with a YUV format, a null pointer, whatever b200_image_resize_run refuses, or, for a Pillow filter, whatever
 * b200_image_resize_workspace refuses. */
B200_API int b200_image_crop_resize_run(const b200_image_resize_desc_t* d, int32_t filter, int32_t pixel_format,
                                        int32_t max_h, int32_t max_w, int32_t resize_short, const uint8_t* src,
                                        const void* table_dev, void* workspace, uint8_t* out, void* stream);

/* ------------------------------------------------------------------------
 * INT8 calibration statistics. Replaces the host loops of the reference's EntropyCalibrator
 * (framework/core/net/entropy_calibrator.cpp: get_max_values, get_histgrams, get_kl_threshold:300-346) with kernels
 * that run inside the FP32 Net's prediction.
 *
 * b200_calib_stats_run: one fp32 tensor of `rows` rows of `ld` floats, of which the first c count (NHWC edges:
 * rows = n*h*w, c = channels, ld = stored channels, so zero padding never reaches a bin; an unpadded NCHW tensor:
 * c = ld). The device word *mode_dev picks the statistic, so one captured CUDA graph serves both passes:
 *   0  *max_bits_dev = max(*max_bits_dev, bits of max |x|): the running maximum as the bit pattern of a non-negative
 *      float (such floats order like their bits); equals numpy's float(np.abs(t).max()), maximised over launches.
 *   1  hist_dev[bin] += number of x in bin, bin = min(trunc(|x| / step), B200_CALIB_BINS - 1),
 *      step = max / B200_CALIB_BINS with max the float of *max_bits_dev; both divisions correctly rounded in fp32
 *      (numpy's (np.abs(t) / step).astype(np.int64)). Nothing is added while the max is 0. uint64 counters.
 *   anything else: no effect.
 * B200_INVALID_VALUE for a null pointer, rows < 1, c < 1 or ld < c.
 *
 * b200_calib_kl_run: the entropy threshold of each of n histograms hists[n][B200_CALIB_BINS] (uint64), with the
 * semantics of anakin_b200/calibrate.py::kl_threshold: the candidate bin i = 129 .. B200_CALIB_BINS - 2 of smallest
 * KL divergence (the smallest i among equal minima), B200_CALIB_BINS when every candidate is infinite. Every int64 and
 * float32 step of the restatement is reproduced in its order, with numpy 2 promotion (the float32 x int64 products of
 * the bin shrinking are float64; q.sum() is numpy's float32 pairwise sum); only the float64 log2 and the float64 sums
 * of the KL terms may round differently. thresh: device int32[n]. kl: NULL or device double[n][B200_CALIB_BINS],
 * filled with the KL value of every candidate (NaN outside the candidate range). One CTA per histogram.
 * ------------------------------------------------------------------------ */
#define B200_CALIB_BINS 2048
B200_API int b200_calib_stats_run(const float* x, int64_t rows, int32_t c, int32_t ld, const int32_t* mode_dev,
                                  uint32_t* max_bits_dev, uint64_t* hist_dev, void* stream);
B200_API int b200_calib_kl_run(const uint64_t* hists, int32_t n, int32_t* thresh, double* kl, void* stream);

/* ------------------------------------------------------------------------
 * Interior-tensor export: one NHWC edge tensor x = [n][h][w][c_stored] (c_stored >= c channels per pixel, the first
 * c of them real) written as the dense fp32 tensor out = [n][c][h][w], channel padding dropped. Per element, with
 * `scale` the edge's calibrated scale (oracle/model_walker.py, as_float):
 *   B200_INT8   (float)q * scale
 *   B200_UINT8  ((float)q * scale) * (float)(127.0 / 255.0)   two fp32 roundings in that order, no FMA
 *   B200_HALF   exact widening                                 (scale unused)
 *   B200_FLOAT  the value, bit for bit                         (scale unused)
 * It waits on the prior grid (programmatic dependent launch) before reading x, so it can sit right behind x's
 * producer in a PDL chain. B200_INVALID_VALUE for a null pointer, n, h, w or c < 1, c_stored < c, h * w above 2^30 or
 * another dtype (checked before the device check).
 * ------------------------------------------------------------------------ */
B200_API int b200_export_run(const void* x, int32_t dtype, int32_t n, int32_t h, int32_t w, int32_t c,
                             int32_t c_stored, float scale, float* out, void* stream);

/* ------------------------------------------------------------------------
 * Squeeze-and-excitation (SENet). Replaces the reference's SaberAxpy<NV, AK_FLOAT>
 * (saber/funcs/impl/cuda/base/cuda_c/saber_axpy.cu:9-16) and, for the gate chain global AVE Pooling -> 1x1
 * Convolution + ReLU -> 1x1 Convolution -> Activation(Sigmoid), the four launches it takes there.
 *
 * b200_axpy_run: out[n][p][c] = act(g[n][c] * x[n][p][c] + y[n][p][c]) over NHWC [n][hw][ld] tensors (first c
 * channels real, channels c..ld-1 written as 0); the gate is [n][ldg], fp32 (or f16). ld * sizeof(x) a 16-byte
 * multiple. It waits on the prior grid (programmatic dependent launch) before reading.
 *   B200_FLOAT  t = fmaf(g, x, y); relu: t > 0 ? t : t * neg_slope
 *   B200_HALF   the same in fp32 on the widened operands, one round-half-even store
 *   8-bit       x s8|u8, y s8|u8, out s8|u8 (u8 after a relu): with f_t = scale_t * (127/255 if t is u8)
 *               the caller passes ax = f_x / f_out and ay = f_y / f_out (fp32 divisions); then
 *               t = (g * ax) * qx + qy * ay, each product and the sum rounded on its own (no FMA);
 *               relu: t = max(t, 0); out = saturate(round half to even(t))
 *
 * b200_se_gate_run: gate[n][c] = sigmoid(b2[c] + W2[c] . relu(b1 + W1 . m[n])), m[n][c] the mean of x over the hw
 * pixels, all in fp32, for every input dtype. x NHWC [n][hw][ld] (f32, f16, s8 or u8), W1 [r][c], b1 [r], W2 [c][r],
 * b2 [c] fp32 device arrays. Every step has a fixed order, so the result is reproducible bit for bit:
 *   m      8-bit: S = exact integer sum of the codes; m = ((float)S * scale [* (float)(127/255) for u8]) / hw
 *          float kinds: fp32 sums in a fixed order (per pixel chunk, then the chunks in order); m = S / hw
 *   hidden for each j: lane l (0..31) sums W1[j][c] * m[c] for c = l, l+32, ... in order (products and sums rounded
 *          on their own); the 32 lane sums are combined by s += shfl_xor(s, o) for o = 16, 8, 4, 2, 1;
 *          h = max(s + b1[j], 0)
 *   z      s = sum over k = 0 .. r-1 in order of W2[c][k] * h[k]; z = s + b2[c]
 *   g      the explicit fp32 sigmoid of se.cu (Cody-Waite exp and a degree-7 polynomial, no library call)
 * One cluster of 8 CTAs per image (images strided over up to sm_count / 8 clusters): each CTA pools an eighth of the
 * image's pixels (the float kinds' "chunks" are these eighths, summed in CTA rank order), then the cluster shares the
 * image's squeeze rows and excitation outputs; no CTA waits for another cluster. The weights are read from L2 once per
 * image. workspace: b200_se_gate_workspace_bytes(d) bytes of device memory (partial sums and hidden activations), one per
 * concurrently running stream. B200_INVALID_VALUE (and a workspace size of 0) for a descriptor whose shared-memory need
 * (max(pooling slots, c + r) floats) exceeds 200 KB.
 * ------------------------------------------------------------------------ */
typedef struct {
    int32_t x_dtype, y_dtype, out_dtype, gate_dtype;
    int32_t n, hw, c, ld, ldg;
    int32_t relu;
    float neg_slope;     /* float kinds */
    float ax, ay;        /* 8-bit kinds */
} b200_axpy_desc_t;
B200_API int b200_axpy_run(const b200_axpy_desc_t* d, const void* gate, const void* x, const void* y, void* out,
                           void* stream);

typedef struct {
    int32_t dtype;       /* of x */
    int32_t n, hw, c, ld;
    int32_t r;           /* squeezed channels */
    int32_t ldg;         /* gate row pitch (elements) */
    float scale;         /* 8-bit x: the edge scale */
} b200_se_gate_desc_t;
B200_API size_t b200_se_gate_workspace_bytes(const b200_se_gate_desc_t* d);
B200_API int b200_se_gate_run(const b200_se_gate_desc_t* d, const void* x, const float* w1, const float* b1,
                              const float* w2, const float* b2, float* gate, void* workspace, void* stream);

/* Kernel-launch counter (every launch made through this library). */
B200_API uint64_t b200_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* B200_SABER_H */
