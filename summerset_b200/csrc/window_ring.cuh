// window_ring.cuh -- the 64-slot instance window shared by the leader engine (engine.cu) and the acceptor (acceptor.cu).
// Group g holds absolute slots [window_base[g], window_base[g] + 64); per-slot bits live in ring words (bit s & 63).
#pragma once
#include "device_common.cuh"

namespace ssb {

// ring word (bit p = absolute slot with s & 63 == p) <-> window word (bit i = absolute slot base + i), r = base & 63
__device__ __forceinline__ uint64_t ring_to_window(uint64_t x, uint32_t r) { return (x >> r) | (x << ((64u - r) & 63u)); }
__device__ __forceinline__ uint64_t window_to_ring(uint64_t x, uint32_t r) { return (x << r) | (x >> ((64u - r) & 63u)); }

// ring positions that stay after the first k (1..64) window positions of a window at base are retired
__device__ __forceinline__ uint64_t ring_keep_after(uint64_t k, uint64_t base) {
    return window_to_ring(k == 64ull ? 0ull : ~0ull << k, static_cast<uint32_t>(base & 63u));
}

}  // namespace ssb
