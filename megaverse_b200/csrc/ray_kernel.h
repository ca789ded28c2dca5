// Ray sensors (ray_kernel.cu): every agent casts the same fan of R camera-space rays against its env's instance list -- the rows and counts
// the rasteriser draws -- and reports the distance and segmentation tag of the nearest front face.  The hit definition, operation by
// operation, is in DESIGN.md section 3 ("Ray sensors"); tests/oracle_seg/orc_rays.cpp restates it on the CPU.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "mv_types.h"

namespace mvray {

struct RayParams {
    const MvInstance *instances;  // [E][instStride], draw order
    const int32_t *instCounts;    // [E][8]; [1] is the number of entries drawn
    const float *views;           // [E * A][16] world-to-camera matrices
    const float *dirs;            // [R][3] camera-space directions
    const uint8_t *envMask;       // [E] or null: envs whose byte is 0 are not cast (their rows keep what they hold)
    float *dist;                  // [E * A][R]
    uint16_t *tag;                // [E * A][R]
    int instStride, E, A, R;
    float maxDist;
};

// one launch on `stream`: one CTA per env
cudaError_t castRays(const RayParams &p, cudaStream_t stream);

}  // namespace mvray
