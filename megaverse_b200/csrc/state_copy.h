// Row copy between the engine's per-env device arrays and a state store (mv_states_save / mv_states_load).  The kernel lives in its
// own translation unit (state_copy.cu): NVVM optimises per module, and a kernel added to engine.cu could change the code generated for
// the step and raster kernels.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>

namespace mvs {

constexpr int kMaxSlabs = 17;

// one per-env array: row r of it starts at base + r * pitch and holds rowBytes bytes
struct Slab {
    const uint8_t *src;
    uint8_t *dst;
    size_t rowBytes, srcPitch, dstPitch;
};

// for every pair (x, y) of dPairs (device memory) and every slab: copy row x of src to row y of dst.  One launch on `stream`.
cudaError_t copyRows(const Slab *slabs, int nSlabs, const int2 *dPairs, int nPairs, cudaStream_t stream);

}  // namespace mvs
