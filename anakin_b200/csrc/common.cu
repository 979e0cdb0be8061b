// Library-wide state: device probe, launch counter, status strings.
#include <stdlib.h>
#include <string.h>

#include <atomic>
#include <mutex>

#include "../../include/b200_saber.h"
#include "common.cuh"

namespace b200 {

static std::atomic<uint64_t> g_launches{0};

struct DevInfo {
    bool probed = false;
    bool sm90 = false;
    int sms = 132;
};
static DevInfo g_dev[64];
static std::mutex g_dev_mu;

static DevInfo& probe_current() {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) {
        (void)cudaGetLastError();
        static DevInfo none;
        return none;
    }
    std::lock_guard<std::mutex> lk(g_dev_mu);
    DevInfo& d = g_dev[dev];
    if (!d.probed) {
        cudaDeviceProp prop;
        if (cudaGetDeviceProperties(&prop, dev) == cudaSuccess) {
            d.sm90 = (prop.major == 9);
            d.sms = prop.multiProcessorCount;
        } else {
            (void)cudaGetLastError();
        }
        d.probed = true;
    }
    return d;
}

bool device_is_sm90() { return probe_current().sm90; }
int sm_count() { return probe_current().sms; }

bool pdl_enabled() {
    static int v = -1;
    if (v < 0) {
        const char* e = getenv("B200_SABER_PDL");
        v = (e && e[0] == '0') ? 0 : 1;
    }
    return v == 1;
}

void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

}  // namespace b200

extern "C" {

const char* b200_status_string(int status) {
    switch (status) {
        case B200_SUCCESS: return "SaberSuccess";
        case B200_NOT_INITIALIZED: return "SaberNotInitialized";
        case B200_INVALID_VALUE: return "SaberInvalidValue";
        case B200_MEM_ALLOC_FAILED: return "SaberMemAllocFailed";
        case B200_UNKNOWN_ERROR: return "SaberUnKownError";
        case B200_OUT_OF_AUTHORITY: return "SaberOutOfAuthority";
        case B200_OUT_OF_MEM: return "SaberOutOfMem";
        case B200_UNIMPL_ERROR: return "SaberUnImplError";
        case B200_WRONG_DEVICE: return "SaberWrongDevice";
    }
    return "unknown";
}

int b200_abi_version(void) { return B200_SABER_ABI_VERSION; }

int b200_device_ok(int device) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        (void)cudaGetLastError();
        return 0;
    }
    if (device < 0 || device >= n) return 0;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) {
        (void)cudaGetLastError();
        return 0;
    }
    return prop.major == 9 ? 1 : 0;
}

uint64_t b200_launch_count(void) { return b200::g_launches.load(std::memory_order_relaxed); }

}  // extern "C"
