// wire_common.cuh -- device helpers shared by the wire kernels (wire_kernels.cu), the acceptor (acceptor.cu) and the
// CRaft calls: 16-byte region rounding, bincode 2 standard-config u64 varints and warp-cooperative byte copies.
#pragma once
#include "device_common.cuh"

namespace ssb {

// a region's bytes: every record and frame region starts 16-byte aligned
__device__ __forceinline__ uint64_t round16(uint64_t x) { return (x + 15u) & ~15ull; }

__device__ __forceinline__ int wv_put(uint8_t *p, uint64_t v) {
    if (v < 251ull) { p[0] = static_cast<uint8_t>(v); return 1; }
    int nb; uint8_t tag;
    if (v < (1ull << 16)) { nb = 2; tag = 251; }
    else if (v < (1ull << 32)) { nb = 4; tag = 252; }
    else { nb = 8; tag = 253; }
    p[0] = tag;
    for (int i = 0; i < nb; ++i) p[1 + i] = static_cast<uint8_t>(v >> (8 * i));
    return 1 + nb;
}
__device__ __forceinline__ int wv_len(uint64_t v) { return v < 251ull ? 1 : v < (1ull << 16) ? 3 : v < (1ull << 32) ? 5 : 9; }

// returns bytes consumed (0: truncated or not a u64 varint)
__device__ __forceinline__ uint32_t wv_get(const uint8_t *p, uint64_t avail, uint64_t &v) {
    if (avail < 1) return 0;
    const uint8_t t = p[0];
    if (t < 251) { v = t; return 1; }
    const uint32_t nb = t == 251 ? 2u : t == 252 ? 4u : t == 253 ? 8u : 0u;
    if (nb == 0u || avail < 1u + nb) return 0;
    uint64_t x = 0;
    for (uint32_t i = 0; i < nb; ++i) x |= static_cast<uint64_t>(p[1 + i]) << (8 * i);
    v = x;
    return 1u + nb;
}

// warp-cooperative copy of n bytes: src 16-byte aligned (a padded shard slot), dst at any alignment
__device__ __forceinline__ void warp_copy_bytes(uint8_t *dst, const uint8_t *__restrict__ src, uint32_t n, uint32_t lane) {
    uint32_t head = (16u - (static_cast<uint32_t>(reinterpret_cast<uintptr_t>(dst)) & 15u)) & 15u;
    if (head > n) head = n;
    if (lane < head) dst[lane] = src[lane];
    const uint32_t nvec = (n - head) >> 4;
    for (uint32_t v = lane; v < nvec; v += 32u) {
        // aligned 16-byte destination vector <- the (generally misaligned) 16 source bytes that belong there
        const uint4 x = head == 0u ? dev::ldg128(src + v * 16u) : dev::load16(src + head + v * 16u, 16);
        dev::stg128_cs(dst + head + v * 16u, x);
    }
    const uint32_t done = head + nvec * 16u, rem = n - done;
    if (lane < rem) dst[done + lane] = src[done + lane];
}

// the same copy with src at any alignment too (bytes out of a receive buffer): aligned 128-bit stores, each fed by the
// two aligned loads around its 16 source bytes
__device__ __forceinline__ void warp_copy_unaligned(uint8_t *dst, const uint8_t *__restrict__ src, uint64_t n, uint32_t lane) {
    uint64_t head = (16u - (static_cast<uint32_t>(reinterpret_cast<uintptr_t>(dst)) & 15u)) & 15u;
    if (head > n) head = n;
    if (lane < head) dst[lane] = src[lane];
    const uint64_t nvec = (n - head) >> 4;
    for (uint64_t v = lane; v < nvec; v += 32u) dev::stg128_cs(dst + head + v * 16u, dev::load16(src + head + v * 16u, 16));
    const uint64_t done = head + nvec * 16u, rem = n - done;
    if (lane < rem) dst[done + lane] = src[done + lane];
}

}  // namespace ssb
