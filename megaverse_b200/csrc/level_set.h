// Level sets (option "level_set"): which level of the set an env plays next when nobody named one.  Defined once for both sides: the
// step kernel calls it at an episode end, the host exports it as mv_level_set_pick so that a caller can predict or check the sequence.
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define MV_HOST_DEVICE __host__ __device__
#else
#define MV_HOST_DEVICE
#endif

// A counter-based hash: the level of episode `episode` of the env whose pick seed is `seed`, uniform over [0, count).  No state besides
// the two counters, so a saved env replays its later levels and any episode's level can be computed out of order.  Two rounds of the
// murmur3 finaliser with the episode mixed in between (so that neither consecutive seeds nor consecutive episodes walk the set with a
// fixed stride), then the high word of hash * count (no modulo bias pattern in the low bits).
MV_HOST_DEVICE inline uint32_t mvLevelSetPick(uint32_t seed, int32_t episode, int32_t count) {
    if (count <= 1) return 0u;
    uint32_t h = seed + 0x9E3779B9u;
    h ^= h >> 16; h *= 0x85EBCA6Bu; h ^= h >> 13; h *= 0xC2B2AE35u; h ^= h >> 16;
    h ^= uint32_t(episode) * 0x9E3779B1u + 0x7F4A7C15u;
    h ^= h >> 16; h *= 0x85EBCA6Bu; h ^= h >> 13; h *= 0xC2B2AE35u; h ^= h >> 16;
    return uint32_t((uint64_t(h) * uint64_t(uint32_t(count))) >> 32);
}
