// Small host-side helpers shared by every translation unit of libb200saber.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200 {

// True when the current device is a compute-capability 9.x (sm_90, Hopper) part.
bool device_is_sm90();
int sm_count();
// Programmatic dependent launch (overlap a kernel's prologue with its
// predecessor's tail). On by default; B200_SABER_PDL=0 disables.
bool pdl_enabled();
void count_launch();

inline unsigned div_up(size_t a, size_t b) { return static_cast<unsigned>((a + b - 1) / b); }

}  // namespace b200
