// Small host-side helpers shared by every translation unit of libb200saber.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <type_traits>
#include <utility>

#include "../../include/b200_saber.h"
#include "image_desc.h"
#include "ptx.cuh"

namespace b200 {

constexpr int kMaxDevices = 64;

template <int V> using Int = std::integral_constant<int, V>;

// A set of dtypes, one bit per b200_dtype_t value.
constexpr uint64_t dtype_bit(int dt) { return 1ull << dt; }
constexpr bool dtype_in(uint64_t set, int dt) { return dt >= 0 && dt < 64 && (set & dtype_bit(dt)); }

// One math kind (b200_math_t) of the conv, stem and fc_stream entry points: the kernel kind it compiles to, its operands
// and the edge dtypes its epilogues read and write.
struct MathKind {
    int math;               // B200_MATH_*
    int kind;               // KIND_* of the kernel instances
    int es;                 // operand element bytes
    int operand_dtype;      // dtype of the operands (int8 activations move as bytes, signed or not)
    uint64_t in_dtypes;     // input dtypes the kernels read
    uint64_t out_dtypes;    // output dtypes the epilogues write
    uint64_t res_dtypes;    // residual dtypes the epilogues read
    int planes;             // operand and weight planes: 2 for 3xTF32 (hi, then lo = x - hi)
    uint32_t c_fmt, a_fmt, b_fmt;   // conv_idesc type codes (a signed int8 input sets a_fmt to 1)
};

inline constexpr MathKind kMathKinds[] = {
    {B200_MATH_I8, KIND_I8, 1, B200_UINT8, dtype_bit(B200_INT8) | dtype_bit(B200_UINT8),
     dtype_bit(B200_INT8) | dtype_bit(B200_UINT8) | dtype_bit(B200_FLOAT), dtype_bit(B200_INT8) | dtype_bit(B200_UINT8),
     1, 2u, 0u, 1u},
    {B200_MATH_F16, KIND_F16, 2, B200_HALF, dtype_bit(B200_HALF), dtype_bit(B200_HALF) | dtype_bit(B200_FLOAT),
     dtype_bit(B200_HALF) | dtype_bit(B200_FLOAT), 1, 1u, 0u, 0u},
    {B200_MATH_TF32X3, KIND_TF32X3, 4, B200_FLOAT, dtype_bit(B200_FLOAT), dtype_bit(B200_FLOAT), dtype_bit(B200_FLOAT),
     2, 1u, 2u, 2u},
    {B200_MATH_E4M3, KIND_E4M3, 1, B200_FP8E4M3, dtype_bit(B200_FP8E4M3), dtype_bit(B200_FP8E4M3) | dtype_bit(B200_FLOAT),
     dtype_bit(B200_FP8E4M3), 1, 1u, 2u, 2u},
};

// The row of math kind `math`; null for a value with none (B200_UNIMPL_ERROR at every entry point).
inline const MathKind* math_kind(int math) {
    for (const MathKind& k : kMathKinds)
        if (k.math == math) return &k;
    return nullptr;
}

// Kinds of the 16-byte vectors the NHWC kernels load and store: 4 x f32, 8 x f16, 16 x s8 or 16 x u8.
enum VecKind : int { VK_F32 = 0, VK_F16 = 1, VK_S8 = 2, VK_U8 = 3 };

// Calls f(Int<K>()) with the vector kind K of dtype and returns its result; B200_UNIMPL_ERROR for any other dtype.
template <typename F>
inline int with_vec_kind(int dtype, F&& f) {
    switch (dtype) {
        case B200_FLOAT: return f(Int<VK_F32>());
        case B200_HALF: return f(Int<VK_F16>());
        case B200_INT8: return f(Int<VK_S8>());
        case B200_UINT8: return f(Int<VK_U8>());
        default: return B200_UNIMPL_ERROR;
    }
}

// True when the current device is a compute-capability 9.x (sm_90, Hopper) part.
bool device_is_sm90();
int sm_count();

inline unsigned div_up(size_t a, size_t b) { return static_cast<unsigned>((a + b - 1) / b); }

// One channel of an 8-bit image input (b200_image_desc_t): (u - mean) * scale, each step rounded to fp32 on its own
// (no contraction into an FMA), so that it equals the host's fp32 normalisation bit for bit.
__device__ __forceinline__ float image_norm(uint8_t u, float mean, float scale) {
    return __fmul_rn(__fsub_rn(static_cast<float>(u), mean), scale);
}

// Whether a launch is a programmatic dependent launch (PDL).
enum class Pdl : bool { Off, On };

// Counts a launch (b200_launch_count) whether or not it succeeded and checks its status e, then
// cudaPeekAtLastError(): B200_SUCCESS, or "[b200_saber] <what> launch failed: <error>" on stderr and
// B200_UNKNOWN_ERROR. Only launch() calls it.
int launch_status(const char* what, cudaError_t e);

// Every kernel of the library is launched, counted and checked here; `what` names it in the error message.
// Pdl::On makes a programmatic dependent launch: the kernel may start while its predecessor on the stream is still
// running, so it must execute griddepcontrol.wait (pdl_wait_prior_grid, pdl_enter) before it reads its predecessor's
// output. Pdl::Off is a plain launch. Unless `cluster` is a single CTA, the CTAs run as thread-block clusters of that
// shape.
template <typename... Params, typename... Args>
inline int launch(const char* what, Pdl pdl, void (*kern)(Params...), dim3 grid, dim3 block, size_t smem, void* stream,
                  dim3 cluster, Args&&... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = static_cast<cudaStream_t>(stream);
    cudaLaunchAttribute attr[2];
    cfg.attrs = attr;
    cfg.numAttrs = 0;
    if (pdl == Pdl::On) {
        cudaLaunchAttribute& a = attr[cfg.numAttrs++];
        a.id = cudaLaunchAttributeProgrammaticStreamSerialization;
        a.val.programmaticStreamSerializationAllowed = 1;
    }
    if (cluster.x * cluster.y * cluster.z > 1) {
        cudaLaunchAttribute& a = attr[cfg.numAttrs++];
        a.id = cudaLaunchAttributeClusterDimension;
        a.val.clusterDim.x = cluster.x;
        a.val.clusterDim.y = cluster.y;
        a.val.clusterDim.z = cluster.z;
    }
    return launch_status(what, cudaLaunchKernelEx(&cfg, kern, std::forward<Args>(args)...));
}

// Lets KERN use `bytes` of dynamic shared memory (and, on request, the whole shared-memory carveout) on the current
// device. Function attributes are per device, and a Worker may drive several GPUs from one process: this runs once
// per kernel and device.
template <auto KERN>
inline void opt_in_smem(int bytes, bool max_carveout = false) {
    static std::atomic<bool> opted_in[kMaxDevices];
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev >= 0 && dev < kMaxDevices && !opted_in[dev].load(std::memory_order_acquire)) {
        cudaFuncSetAttribute(KERN, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
        if (max_carveout)
            cudaFuncSetAttribute(KERN, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        opted_in[dev].store(true, std::memory_order_release);
    }
}

}  // namespace b200
