// Small host-side helpers shared by every translation unit of libb200saber.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <utility>

namespace b200 {

constexpr int kMaxDevices = 64;

// True when the current device is a compute-capability 9.x (sm_90, Hopper) part.
bool device_is_sm90();
int sm_count();
// Programmatic dependent launch (overlap a kernel's prologue with its
// predecessor's tail). On by default; B200_SABER_PDL=0 disables.
bool pdl_enabled();
void count_launch();

inline unsigned div_up(size_t a, size_t b) { return static_cast<unsigned>((a + b - 1) / b); }

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
