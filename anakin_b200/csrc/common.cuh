// Small host-side helpers shared by every translation unit of libb200saber.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <type_traits>
#include <utility>

#include "../../include/b200_saber.h"
#include "image_desc.h"

namespace b200 {

constexpr int kMaxDevices = 64;

template <int V> using Int = std::integral_constant<int, V>;

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
// Programmatic dependent launch (overlap a kernel's prologue with its
// predecessor's tail). On by default; B200_SABER_PDL=0 disables.
bool pdl_enabled();
void count_launch();

inline unsigned div_up(size_t a, size_t b) { return static_cast<unsigned>((a + b - 1) / b); }

// One channel of an 8-bit image input (b200_image_desc_t): (u - mean) * scale, each step rounded to fp32 on its own
// (no contraction into an FMA), so that it equals the host's fp32 normalisation bit for bit.
__device__ __forceinline__ float image_norm(uint8_t u, float mean, float scale) {
    return __fmul_rn(__fsub_rn(static_cast<float>(u), mean), scale);
}

// Launches kern with programmatic dependent launch (when pdl_enabled()) and, unless `cluster` is a single CTA, as
// thread-block clusters of that shape. The caller counts the launch (count_launch).
template <typename... Params, typename... Args>
inline cudaError_t launch_kernel(void (*kern)(Params...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                                 dim3 cluster, Args&&... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    if (cluster.x * cluster.y * cluster.z > 1) {
        attr[1].id = cudaLaunchAttributeClusterDimension;
        attr[1].val.clusterDim.x = cluster.x;
        attr[1].val.clusterDim.y = cluster.y;
        attr[1].val.clusterDim.z = cluster.z;
        cfg.numAttrs = 2;
    }
    return cudaLaunchKernelEx(&cfg, kern, std::forward<Args>(args)...);
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
