// Validation of an 8-bit image input format (b200_image_desc_t), shared by the kernels' entry points
// (conv_stem.cu, pointwise.cu) and the framework (Graph::set_input_image, InputOp).
#pragma once
#include <math.h>

#include "../../include/b200_saber.h"

// c channels in 1..4, src_channel[0..c) a permutation of 0..c-1, mean[0..c) and scale[0..c) finite
inline bool b200_image_desc_valid(const b200_image_desc_t* d, int c) {
    if (!d || c < 1 || c > 4) return false;
    bool seen[4] = {false, false, false, false};
    for (int i = 0; i < c; ++i) {
        const int s = d->src_channel[i];
        if (s < 0 || s >= c || seen[s]) return false;
        seen[s] = true;
        if (!isfinite(d->mean[i]) || !isfinite(d->scale[i])) return false;
    }
    return true;
}
