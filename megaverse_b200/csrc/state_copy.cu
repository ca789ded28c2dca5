// State-store row copy (state_copy.h): one launch moves every per-env array of a list of (source row, destination row) pairs.
//
// Grid: y walks the pairs, x the flattened (slab, 16-byte chunk) index of one env row.  Chunks are aligned to the DESTINATION address,
// so a whole chunk is one 16-byte store; its load is one 128-bit load when the source row has the same alignment mod 16, else two
// 64-bit / four 32-bit / sixteen byte loads.  Rows whose size is not a multiple of 16 bytes (dones: 1 byte per env, A x 264-byte agent
// rows) start and end with a partial chunk that is copied byte by byte.
#include "state_copy.h"

namespace mvs {
namespace {

struct Table {
    Slab slab[kMaxSlabs];
    uint32_t chunkBase[kMaxSlabs + 1];  // prefix sums of the chunks per row of each slab
    int n;
};

constexpr int kThreads = 256;
constexpr int kChunksPerThread = 4;  // per pair: about this many chunks per thread before x wraps

__host__ __device__ inline uint32_t chunksPerRow(size_t rowBytes) { return uint32_t((rowBytes + 30) / 16); }  // the row may start mid-chunk

__device__ inline void copyChunk(const uint8_t *src, uint8_t *dst, size_t rowBytes, uint32_t c) {
    const long long lo = (long long)c * 16 - (long long)(reinterpret_cast<uintptr_t>(dst) & 15);
    const size_t b = size_t(lo < 0 ? 0 : lo), e = size_t(lo + 16 < (long long)rowBytes ? lo + 16 : (long long)rowBytes);
    if (b >= e) return;
    const uint8_t *s = src + b;
    uint8_t *d = dst + b;
    if (e - b < 16) {
        for (size_t i = 0; i < e - b; ++i) d[i] = s[i];
        return;
    }
    const uintptr_t mis = reinterpret_cast<uintptr_t>(s) & 15;  // d is 16-byte aligned here
    uint4 v;
    if (mis == 0) {
        v = *reinterpret_cast<const uint4 *>(s);
    } else if ((mis & 7) == 0) {
        const uint2 a = reinterpret_cast<const uint2 *>(s)[0], z = reinterpret_cast<const uint2 *>(s)[1];
        v = make_uint4(a.x, a.y, z.x, z.y);
    } else if ((mis & 3) == 0) {
        const uint32_t *w = reinterpret_cast<const uint32_t *>(s);
        v = make_uint4(w[0], w[1], w[2], w[3]);
    } else {
        uint8_t t[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) t[i] = s[i];
        v = make_uint4(t[0] | t[1] << 8 | t[2] << 16 | uint32_t(t[3]) << 24, t[4] | t[5] << 8 | t[6] << 16 | uint32_t(t[7]) << 24,
                       t[8] | t[9] << 8 | t[10] << 16 | uint32_t(t[11]) << 24, t[12] | t[13] << 8 | t[14] << 16 | uint32_t(t[15]) << 24);
    }
    *reinterpret_cast<uint4 *>(d) = v;
}

__global__ void __launch_bounds__(kThreads) stateCopyKernel(const __grid_constant__ Table t, const int2 *__restrict__ pairs, int nPairs) {
    const uint32_t perPair = t.chunkBase[t.n];
    for (int p = blockIdx.y; p < nPairs; p += gridDim.y) {
        const int2 pr = pairs[p];
        int s = 0;
        for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < perPair; i += gridDim.x * kThreads) {
            while (i >= t.chunkBase[s + 1]) ++s;  // i only grows
            const Slab &sl = t.slab[s];
            copyChunk(sl.src + size_t(pr.x) * sl.srcPitch, sl.dst + size_t(pr.y) * sl.dstPitch, sl.rowBytes, i - t.chunkBase[s]);
        }
    }
}

}  // namespace

cudaError_t copyRows(const Slab *slabs, int nSlabs, const int2 *dPairs, int nPairs, cudaStream_t stream) {
    if (nSlabs < 1 || nSlabs > kMaxSlabs || nPairs < 1) return cudaErrorInvalidValue;
    Table t = {};
    t.n = nSlabs;
    size_t total = 0;
    for (int i = 0; i < nSlabs; ++i) {
        t.slab[i] = slabs[i];
        t.chunkBase[i] = uint32_t(total);
        total += chunksPerRow(slabs[i].rowBytes);
    }
    if (total >= (size_t(1) << 32)) return cudaErrorInvalidValue;
    t.chunkBase[nSlabs] = uint32_t(total);
    const dim3 grid(unsigned((total + kThreads * kChunksPerThread - 1) / (kThreads * kChunksPerThread)), unsigned(nPairs < 65535 ? nPairs : 65535));
    stateCopyKernel<<<grid, kThreads, 0, stream>>>(t, dPairs, nPairs);
    return cudaGetLastError();
}

}  // namespace mvs
