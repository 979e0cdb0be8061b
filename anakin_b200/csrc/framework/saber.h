// Host-side mirror of Anakin's Saber core types for target NV, over the C ABI
// (include/b200_saber.h).  Same names / argument meaning / status conventions as the
// reference so that operator code and tests read like the reference's:
//   saber/saber_types.h            -> enums below (values identical)
//   saber/core/{shape,tensor,context}.h -> Shape, Tensor<T>, Context<T>
// The reference's Param structs and func / impl layers have no counterpart: the operators
// (operators.cpp) build ConvEngine specs and C-ABI descriptors from their attributes directly.
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
        _image = false;
        return _buf->re_alloc(storage_bytes(), kHost);
    }
    // An 8-bit image graph input: uint8 [n][h][w][c] with c stored unpadded (it is the caller's buffer), read through
    // the normalisation `d`. Only the marker says so: a u8 NHWC tensor is otherwise an INT8 (post-ReLU) activation.
    SaberStatus re_alloc_image(const Shape& s, const b200_image_desc_t& d) {
        Shape hwc = s;
        hwc.set_layout(Layout_NHWC);
        _shape = hwc;
        _dtype = AK_UINT8;
        _c_pad = s.channel();
        _image = true;
        _image_desc = d;
        return _buf->re_alloc(storage_bytes(), kHost);
    }
    bool is_image() const { return _image; }
    const b200_image_desc_t& image_desc() const { return _image_desc; }
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
    bool _image = false;
    b200_image_desc_t _image_desc{};
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

}  // namespace saber
}  // namespace anakin
