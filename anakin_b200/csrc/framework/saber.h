// Host-side mirror of Anakin's Saber layer for target NV, re-expressed over the C ABI
// (include/b200_saber.h).  Same names / argument meaning / status conventions as the
// reference so that operator code and tests read like the reference's:
//   saber/saber_types.h            -> enums below (values identical)
//   saber/core/{shape,tensor,context}.h -> Shape, Tensor<T>, Context<T>
//   saber/saber_funcs_param.h      -> ActivationParam .. SoftmaxParam (field names kept)
//   saber/funcs/base.h, impl/impl_base.h -> BaseFunc-style funcs with
//        compute_output_shape / init / operator() and impls with init / create / dispatch
// Differences that are deliberate (B200-first): device activations are NHWC with channels
// padded to a 16-byte multiple (Layout_NHWC); one target (NV) and no Vender/Saber impl
// choice -- every op is a hand-written sm_90a kernel behind b200_*; FP32 NCHW tensors are
// accepted only at graph inputs and converted by the consuming op.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "../../../include/b200_saber.h"

// C++ classes that user code links against are exported from libanakin_b200.so explicitly
// (the library is built with -fvisibility=hidden).
#define ANAKIN_EXPORT __attribute__((visibility("default")))

namespace anakin {
namespace saber {

// ---------------------------------------------------------------- types (saber_types.h:205-319)
enum DataType { AK_INVALID = -1, AK_HALF = 0, AK_FLOAT = 1, AK_INT8 = 3, AK_INT32 = 5, AK_UINT8 = 7 };
enum LayoutType { Layout_invalid = 0, Layout_NCHW = 8, Layout_NHWC = 9 };
typedef enum {
    SaberSuccess = -1,
    SaberNotInitialized = 1,
    SaberInvalidValue = 3,
    SaberMemAllocFailed = 7,
    SaberUnKownError = 15,
    SaberOutOfAuthority = 31,
    SaberOutOfMem = 63,
    SaberUnImplError = 127,
    SaberWrongDevice = 255
} SaberStatus;
typedef enum { STATIC = 1, RUNTIME = 2, SPECIFY = 3, UNKNOWN = 4 } SaberImplStrategy;
enum ImplEnum { VENDER_IMPL = 0, SABER_IMPL };
typedef enum {
    Active_unknow = 0, Active_sigmoid = 1, Active_relu = 2, Active_tanh = 3, Active_clipped_relu = 4,
    Active_elu = 5, Active_identity = 6
} ActiveType;
typedef enum {
    Pooling_unknow = 0, Pooling_max = 1, Pooling_average_include_padding = 2,
    Pooling_average_exclude_padding = 3
} PoolingType;
typedef enum { Eltwise_unknow = 0, Eltwise_prod = 1, Eltwise_sum = 2, Eltwise_max = 3 } EltwiseType;

struct NV {};        // device target
struct NVHX86 {};    // pinned host target
struct X86 {};

inline size_t type_length(DataType t) {
    switch (t) {
        case AK_HALF: return 2;
        case AK_FLOAT: case AK_INT32: return 4;
        default: return 1;
    }
}

// SABER_CHECK (saber/core/common.h:36-40): abort on any status but SaberSuccess.
#define SABER_CHECK(cond)                                                                   \
    do {                                                                                    \
        ::anakin::saber::SaberStatus _st = static_cast<::anakin::saber::SaberStatus>(cond); \
        if (_st != ::anakin::saber::SaberSuccess) {                                         \
            fprintf(stderr, "[FATAL] %s:%d SABER_CHECK(%s) = %s\n", __FILE__, __LINE__, #cond, \
                    b200_status_string(_st));                                               \
            abort();                                                                        \
        }                                                                                   \
    } while (0)
#define CUDA_CHECK(cond)                                                                  \
    do {                                                                                  \
        cudaError_t _e = (cond);                                                          \
        if (_e != cudaSuccess) {                                                          \
            fprintf(stderr, "[FATAL] %s:%d CUDA %s\n", __FILE__, __LINE__, cudaGetErrorString(_e)); \
            abort();                                                                      \
        }                                                                                 \
    } while (0)

// ---------------------------------------------------------------- Shape (saber/core/shape.h)
// Logical dims are always kept in N,C,H,W order; the layout tag says how memory is laid out.
class Shape {
public:
    Shape() : _layout(Layout_NCHW) { _d[0] = _d[1] = _d[2] = _d[3] = 0; }
    Shape(std::vector<int> nchw, LayoutType layout = Layout_NCHW) : _layout(layout) {
        for (int i = 0; i < 4; ++i) _d[i] = i < static_cast<int>(nchw.size()) ? nchw[i] : 1;
    }
    int num() const { return _d[0]; }
    int channel() const { return _d[1]; }
    int height() const { return _d[2]; }
    int width() const { return _d[3]; }
    void set_num(int v) { _d[0] = v; }
    void set_channel(int v) { _d[1] = v; }
    void set_height(int v) { _d[2] = v; }
    void set_width(int v) { _d[3] = v; }
    int dims() const { return 4; }
    int& operator[](int i) { return _d[i]; }
    int operator[](int i) const { return _d[i]; }
    long long count() const { return 1ll * _d[0] * _d[1] * _d[2] * _d[3]; }
    long long count(int start, int end) const {
        long long c = 1;
        for (int i = start; i < end && i < 4; ++i) c *= _d[i];
        return c;
    }
    LayoutType get_layout() const { return _layout; }
    void set_layout(LayoutType l) { _layout = l; }
    bool operator==(const Shape& o) const {
        return _d[0] == o._d[0] && _d[1] == o._d[1] && _d[2] == o._d[2] && _d[3] == o._d[3] &&
               _layout == o._layout;
    }
    bool operator!=(const Shape& o) const { return !(*this == o); }

private:
    int _d[4];
    LayoutType _layout;
};

// ---------------------------------------------------------------- Buffer + Tensor (saber/core/tensor.h)
struct DeviceBuffer {
    void* ptr = nullptr;
    size_t bytes = 0;
    bool host = false;  // host tensors (weights, PBlocks) live in ordinary pageable memory
    ~DeviceBuffer() { release(); }
    void release() {
        if (ptr) {
            if (host) free(ptr); else cudaFree(ptr);
        }
        ptr = nullptr;
        bytes = 0;
    }
    SaberStatus re_alloc(size_t n, bool on_host) {
        if (n <= bytes && on_host == host && ptr) return SaberSuccess;
        release();
        host = on_host;
        if (n == 0) return SaberSuccess;
        if (on_host) {
            ptr = calloc(1, n);
            if (!ptr) return SaberOutOfMem;
        } else {
            // device buffers start zeroed: NHWC channel padding is never written by any kernel and
            // must read as 0 (a NaN there would poison 0-weight products in the float convs)
            if (cudaMalloc(&ptr, n) != cudaSuccess) { ptr = nullptr; (void)cudaGetLastError(); return SaberOutOfMem; }
            // (the fill runs on the legacy default stream, which does not order against the Nets' non-blocking streams:
            // wait for it here -- allocation time only -- so that no later kernel can race with a late memset)
            if (cudaMemset(ptr, 0, n) != cudaSuccess || cudaStreamSynchronize(cudaStreamLegacy) != cudaSuccess) { (void)cudaGetLastError(); }
        }
        bytes = n;
        return SaberSuccess;
    }
};

template <typename TargetType>
class Tensor {
public:
    static constexpr bool kHost = !std::is_same<TargetType, NV>::value;
    Tensor() : _dtype(AK_FLOAT), _c_pad(0), _buf(std::make_shared<DeviceBuffer>()) {}
    explicit Tensor(const Shape& s, DataType dt = AK_FLOAT) : Tensor() { _dtype = dt; re_alloc(s, dt); }

    // channels as stored: NHWC tensors pad C so that a pixel is a multiple of 16 bytes
    static int padded_channels(int c, DataType dt, LayoutType l) {
        if (l != Layout_NHWC) return c;
        const int q = 16 / static_cast<int>(type_length(dt));
        return (c + q - 1) / q * q;
    }
    SaberStatus re_alloc(const Shape& s, DataType dt) {
        _shape = s;
        _dtype = dt;
        _c_pad = padded_channels(s.channel(), dt, s.get_layout());
        return _buf->re_alloc(storage_bytes(), kHost);
    }
    SaberStatus reshape(const Shape& s) { return re_alloc(s, _dtype); }
    SaberStatus set_shape(const Shape& s) { return reshape(s); }
    SaberStatus set_dtype(DataType dt) { return re_alloc(_shape, dt); }
    // Share the storage of another tensor (reference Tensor::share_from, tensor.h).
    SaberStatus share_from(const Tensor& o) { _buf = o._buf; return SaberSuccess; }

    size_t storage_bytes() const {
        return static_cast<size_t>(_shape.num()) * _shape.height() * _shape.width() * _c_pad * type_length(_dtype);
    }
    const Shape& valid_shape() const { return _shape; }
    const Shape& shape() const { return _shape; }
    long long valid_size() const { return _shape.count(); }
    long long size() const { return _shape.count(); }
    int num() const { return _shape.num(); }
    int channel() const { return _shape.channel(); }
    int height() const { return _shape.height(); }
    int width() const { return _shape.width(); }
    int channel_stored() const { return _c_pad; }
    int dims() const { return 4; }
    long long count_valid(int s, int e) const { return _shape.count(s, e); }
    DataType get_dtype() const { return _dtype; }
    LayoutType get_layout() const { return _shape.get_layout(); }
    void set_layout(LayoutType l) { Shape s = _shape; s.set_layout(l); re_alloc(s, _dtype); }
    const std::vector<float>& get_scale() const { return _scale; }
    void set_scale(const std::vector<float>& s) { _scale = s; }
    void* mutable_data() { return _buf->ptr; }
    const void* data() const { return _buf->ptr; }

    // H2D / D2H / D2D copy of the raw storage; shapes, dtype and layout must match.
    template <typename Other>
    SaberStatus copy_from(const Tensor<Other>& o, cudaStream_t stream = nullptr) {
        if (o.storage_bytes() != storage_bytes()) return SaberInvalidValue;
        if (storage_bytes() == 0) return SaberSuccess;
        cudaError_t e = cudaMemcpyAsync(_buf->ptr, o.data(), storage_bytes(), cudaMemcpyDefault, stream);
        if (e == cudaSuccess && (kHost || Tensor<Other>::kHost)) e = cudaStreamSynchronize(stream);
        return e == cudaSuccess ? SaberSuccess : SaberUnKownError;
    }

private:
    Shape _shape;
    DataType _dtype;
    int _c_pad;
    std::vector<float> _scale;
    std::shared_ptr<DeviceBuffer> _buf;
};

// ---------------------------------------------------------------- Context (saber/core/context.h:29-201)
template <typename TargetType>
class Context {
public:
    Context() : _device_id(0), _stream(nullptr) {}
    Context(int device_id, cudaStream_t compute) : _device_id(device_id), _stream(compute) {}
    int get_device_id() const { return _device_id; }
    cudaStream_t get_compute_stream() const { return _stream; }
    cudaStream_t get_data_stream() const { return _stream; }
    void set_compute_stream(cudaStream_t s) { _stream = s; }

private:
    int _device_id;
    cudaStream_t _stream;
};

// ---------------------------------------------------------------- Params (saber/saber_funcs_param.h)
template <typename T>
struct ActivationParam {  // :48
    ActivationParam() : active(Active_unknow), negative_slope(0.f), coef(1.f), has_active(false) {}
    ActivationParam(ActiveType act, float n_slope = 0.f, float co = 1.f)
        : active(act), negative_slope(n_slope), coef(co), has_active(true) {}
    bool operator==(const ActivationParam& o) const {
        return active == o.active && negative_slope == o.negative_slope && coef == o.coef &&
               has_active == o.has_active;
    }
    ActiveType active;
    float negative_slope;
    float coef;
    bool has_active;
};

template <typename T>
struct ConvParam {  // :470
    ConvParam() : group(1), pad_h(0), pad_w(0), stride_h(1), stride_w(1), dilation_h(1), dilation_w(1),
                  weight_tensor(nullptr), bias_tensor(nullptr), alpha(1.f), beta(0.f),
                  beta_type(AK_FLOAT) {}
    ConvParam(int group_in, int pad_h_in, int pad_w_in, int stride_h_in, int stride_w_in, int dilation_h_in,
              int dilation_w_in, Tensor<NVHX86>* weight, Tensor<NVHX86>* bias,
              ActivationParam<T> act = ActivationParam<T>(), float alpha_in = 1.f, float beta_in = 0.f,
              DataType beta_type_in = AK_FLOAT)
        : group(group_in), pad_h(pad_h_in), pad_w(pad_w_in), stride_h(stride_h_in), stride_w(stride_w_in),
          dilation_h(dilation_h_in), dilation_w(dilation_w_in), weight_tensor(weight), bias_tensor(bias),
          activation_param(act), alpha(alpha_in), beta(beta_in), beta_type(beta_type_in) {}
    bool operator==(const ConvParam& o) const {
        return group == o.group && pad_h == o.pad_h && pad_w == o.pad_w && stride_h == o.stride_h &&
               stride_w == o.stride_w && dilation_h == o.dilation_h && dilation_w == o.dilation_w &&
               weight_tensor == o.weight_tensor && bias_tensor == o.bias_tensor &&
               activation_param == o.activation_param && alpha == o.alpha && beta == o.beta;
    }
    Tensor<NVHX86>* weight() const { return weight_tensor; }
    Tensor<NVHX86>* bias() const { return bias_tensor; }
    int group, pad_h, pad_w, stride_h, stride_w, dilation_h, dilation_w;
    // Non-owning: KCRS fp32 weights [k][c/g][r][s] and bias [k] in HOST memory, owned by the
    // graph's PBlock arena.  (The reference points at device copies; here the device image is the
    // wgmma-packed form built once by trans_weights.)
    Tensor<NVHX86>* weight_tensor;
    Tensor<NVHX86>* bias_tensor;
    ActivationParam<T> activation_param;
    float alpha, beta;
    DataType beta_type;  // dtype of the residual ("be-added") tensor for ConvEltwise
};

template <typename T>
struct EltwiseParam {  // :1077
    EltwiseParam() : operation(Eltwise_unknow), has_eltwise(false) {}
    EltwiseParam(EltwiseType op, std::vector<float> coeff_in = std::vector<float>({1.f, 1.f}),
                 ActivationParam<T> act = ActivationParam<T>())
        : operation(op), coeff(coeff_in), activation_param(act), has_eltwise(true) {}
    bool operator==(const EltwiseParam& o) const {
        return operation == o.operation && coeff == o.coeff && activation_param == o.activation_param;
    }
    EltwiseType operation;
    std::vector<float> coeff;
    ActivationParam<T> activation_param;
    bool has_eltwise;
};

template <typename T>
struct ConvEltwiseParam {  // :586
    ConvEltwiseParam() {}
    ConvEltwiseParam(ConvParam<T>& c, EltwiseParam<T>& e) : conv_param(c), eltwise_param(e) {}
    bool operator==(const ConvEltwiseParam& o) const {
        return conv_param == o.conv_param && eltwise_param == o.eltwise_param;
    }
    ConvParam<T> conv_param;
    EltwiseParam<T> eltwise_param;
};

template <typename T>
struct PoolingParam {  // :2087
    PoolingParam() : window_h(1), window_w(1), pad_h(0), pad_w(0), stride_h(1), stride_w(1),
                     pooling_type(Pooling_unknow), global_pooling(false), cmp_out_shape_floor_as_conv(false) {}
    PoolingParam(int window_h_in, int window_w_in, int pad_h_in, int pad_w_in, int stride_h_in, int stride_w_in,
                 PoolingType type, bool global_pooling_in = false, bool cmp_out_shape_floor_as_conv_in = false)
        : window_h(window_h_in), window_w(window_w_in), pad_h(pad_h_in), pad_w(pad_w_in), stride_h(stride_h_in),
          stride_w(stride_w_in), pooling_type(type), global_pooling(global_pooling_in),
          cmp_out_shape_floor_as_conv(cmp_out_shape_floor_as_conv_in) {}
    bool operator==(const PoolingParam& o) const {
        return window_h == o.window_h && window_w == o.window_w && pad_h == o.pad_h && pad_w == o.pad_w &&
               stride_h == o.stride_h && stride_w == o.stride_w && pooling_type == o.pooling_type &&
               global_pooling == o.global_pooling && cmp_out_shape_floor_as_conv == o.cmp_out_shape_floor_as_conv;
    }
    bool pooling_padded() const { return pad_h || pad_w; }
    int window_h, window_w, pad_h, pad_w, stride_h, stride_w;
    PoolingType pooling_type;
    bool global_pooling;
    bool cmp_out_shape_floor_as_conv;
};

template <typename T>
struct ConvPoolingParam {  // :647
    ConvPoolingParam() {}
    ConvPoolingParam(ConvParam<T>& c, PoolingParam<T>& p) : conv_param(c), pooling_param(p) {}
    bool operator==(const ConvPoolingParam& o) const {
        return conv_param == o.conv_param && pooling_param == o.pooling_param;
    }
    ConvParam<T> conv_param;
    PoolingParam<T> pooling_param;
};

template <typename T>
struct FcParam {  // :1236
    FcParam() : weights(nullptr), bias(nullptr), num_output(0), axis(1), is_transpose_weights(false) {}
    FcParam(Tensor<NVHX86>* w, Tensor<NVHX86>* b, int num_output_in, int axis_in = 1, bool trans = false)
        : weights(w), bias(b), num_output(num_output_in), axis(axis_in), is_transpose_weights(trans) {}
    bool operator==(const FcParam& o) const {
        return weights == o.weights && bias == o.bias && num_output == o.num_output && axis == o.axis &&
               is_transpose_weights == o.is_transpose_weights;
    }
    Tensor<NVHX86>* weights;  // [num_output][K] row-major fp32, host
    Tensor<NVHX86>* bias;
    int num_output;
    int axis;
    bool is_transpose_weights;
    ActivationParam<T> activation_param;  // fused relu (DenseRelu); extension, default off
};

template <typename T>
struct SoftmaxParam {  // :2859
    SoftmaxParam() : axis(1) {}
    explicit SoftmaxParam(int axis_in) : axis(axis_in) {}
    bool operator==(const SoftmaxParam& o) const { return axis == o.axis; }
    int axis;
};

template <typename T>
struct ScaleParam {  // :2599
    ScaleParam() : axis(1), num_axes(1), bias_term(false) {}
    ScaleParam(std::vector<float> w, std::vector<float> b, bool bias_term_in, int axis_in = 1, int num_axes_in = 1)
        : axis(axis_in), num_axes(num_axes_in), bias_term(bias_term_in), scale_w(w), scale_b(b) {}
    bool operator==(const ScaleParam& o) const {
        return axis == o.axis && num_axes == o.num_axes && bias_term == o.bias_term && scale_w == o.scale_w &&
               scale_b == o.scale_b;
    }
    int axis, num_axes;
    bool bias_term;
    std::vector<float> scale_w, scale_b;
};

// ---------------------------------------------------------------- impl / func base (impl_base.h:30-69, base.h:32-252)
template <typename Param>
class ImplBase {
public:
    typedef std::vector<Tensor<NV>*> TensorVec;
    virtual ~ImplBase() {}
    virtual SaberStatus init(const TensorVec& in, TensorVec& out, Param& p, Context<NV>& ctx) = 0;    // once; may alloc
    virtual SaberStatus create(const TensorVec& in, TensorVec& out, Param& p, Context<NV>& ctx) = 0;  // on shape/param change
    virtual SaberStatus dispatch(const TensorVec& in, TensorVec& out, Param& p) = 0;                  // hot, async on ctx stream
protected:
    Context<NV>* _ctx = nullptr;
};

inline std::vector<Shape> shapes_of(const std::vector<Tensor<NV>*>& v) {
    std::vector<Shape> s;
    for (auto* t : v) s.push_back(t->valid_shape());
    return s;
}

// BaseFunc: shape inference + plan cache keyed on (param, input shapes)  (base.h:85-162).
template <typename Impl, typename Param>
class BaseFunc {
public:
    typedef std::vector<Tensor<NV>*> Input_v;
    typedef std::vector<Tensor<NV>*> Output_v;
    virtual ~BaseFunc() {}
    virtual SaberStatus compute_output_shape(const Input_v& in, Output_v& out, Param& p) = 0;
    SaberStatus init(const Input_v& in, Output_v& out, Param& p, SaberImplStrategy, ImplEnum, Context<NV>& ctx) {
        _ctx = ctx;
        _param = p;
        _in_shapes = shapes_of(in);
        SaberStatus st = _impl.init(in, out, p, _ctx);
        _inited = (st == SaberSuccess);
        return st;
    }
    SaberStatus operator()(const Input_v& in, Output_v& out, Param& p, Context<NV>& ctx) {
        if (!_inited) return SaberNotInitialized;
        if (!(p == _param) || shapes_of(in) != _in_shapes || ctx.get_compute_stream() != _ctx.get_compute_stream()) {
            _ctx = ctx;
            _param = p;
            _in_shapes = shapes_of(in);
            SaberStatus st = compute_output_shape(in, out, p);
            if (st != SaberSuccess) return st;
            st = _impl.create(in, out, p, _ctx);
            if (st != SaberSuccess) return st;
        }
        return _impl.dispatch(in, out, p);
    }
    Impl& impl() { return _impl; }

protected:
    Impl _impl;
    Param _param;
    Context<NV> _ctx;
    std::vector<Shape> _in_shapes;
    bool _inited = false;
};

}  // namespace saber
}  // namespace anakin
