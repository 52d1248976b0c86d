// wire_common.cuh -- device helpers shared by the wire kernels (wire_kernels.cu), the acceptor (acceptor.cu) and the
// CRaft calls: 16-byte region rounding, bincode 2 standard-config u64 varints, the frame head every decoder starts with
// and warp-cooperative byte copies.
#pragma once
#include "device_common.cuh"
#include "ss_internal.hpp"

namespace ssb {

constexpr uint32_t kPending = 0xfffffffeu;                  // a decoder's "well formed so far": the caller's checks follow
constexpr uint32_t kVariantLimit = 1u << 16;                // no enum of the protocol has this many variants: malformed
constexpr uint64_t kMaxFrameBody = 0xffffffffull - 64u;     // the cap of the decoders whose record lengths must fit a u32

// a region's bytes: every record and frame region starts 16-byte aligned
__device__ __forceinline__ uint64_t round16(uint64_t x) { return (x + 15u) & ~15ull; }

// the 8-byte big-endian length every frame and WAL record starts with (utils/safetcp.rs:30-88, server/storage.rs:333-337)
__device__ __forceinline__ uint64_t get_be64(const uint8_t *p) {
    uint64_t v = 0;
    for (int k = 0; k < 8; ++k) v = (v << 8) | p[k];
    return v;
}
__device__ __forceinline__ void put_be64(uint8_t *p, uint64_t v) {
    for (int k = 0; k < 8; ++k) p[k] = static_cast<uint8_t>(v >> (8 * (7 - k)));
}

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

// the varint at body position n of b[0..len) into v, n past it; false: truncated or not a u64 varint
__device__ __forceinline__ bool wv_next(const uint8_t *b, uint64_t len, uint64_t &n, uint64_t &v) {
    const uint32_t c = wv_get(b + n, len - n, v);
    n += c;
    return c != 0u;
}

// the length prefix of the frame or WAL record at buf + off: false when the prefix or the len-byte body b runs past
// buf_len, or len > max_body
__device__ __forceinline__ bool frame_body(const uint8_t *buf, uint64_t buf_len, uint64_t off, uint64_t max_body, const uint8_t *&b,
                                           uint64_t &len) {
    if (off > buf_len || buf_len - off < 8u) return false;                  // off + 8 would wrap near 2^64
    len = get_be64(buf + off);
    if (len > buf_len - off - 8u || len > max_body) return false;
    b = buf + off + 8u;
    return true;
}

// The head of a peer frame: the length prefix (frame_body), PeerMessage::Msg and the PeerMsg variant.  true: the frame
// is PeerMsg `variant`, with b / len / n past it.  false: kind = the verdict, 0x80000000 | v for another PeerMessage
// variant (LeaseMsg / Leave / LeaveReply), v for another PeerMsg (the host's business), SS_FRAME_KIND_MALFORMED for a
// bad head or, when cap_variant, a variant >= kVariantLimit.  (Without the cap any u32 can be a verdict, so the "it is
// the message" answer is the return value rather than a reserved kind.)
__device__ __forceinline__ bool msg_head(const uint8_t *buf, uint64_t buf_len, uint64_t off, uint32_t variant, uint64_t max_body,
                                         bool cap_variant, const uint8_t *&b, uint64_t &len, uint64_t &n, uint32_t &kind) {
    kind = SS_FRAME_KIND_MALFORMED;
    uint64_t v = 0;
    n = 0;
    if (!frame_body(buf, buf_len, off, max_body, b, len) || !wv_next(b, len, n, v)) return false;
    if (v != 0u) {
        if (!cap_variant || v < kVariantLimit) kind = 0x80000000u | static_cast<uint32_t>(v);
        return false;
    }
    if (!wv_next(b, len, n, v)) return false;
    if (v != variant) {
        if (!cap_variant || v < kVariantLimit) kind = static_cast<uint32_t>(v);
        return false;
    }
    return true;
}

// msg_head with the variant cap, then the element count of the Vec or HashMap the message starts with (Reconstruct,
// ReconstructReply): kPending with b / len / n past cnt, else the verdict
__device__ __forceinline__ uint32_t msg_head_count(const uint8_t *buf, uint64_t buf_len, uint64_t off, uint32_t variant, uint64_t max_body,
                                                   const uint8_t *&b, uint64_t &len, uint64_t &n, uint64_t &cnt) {
    uint32_t kind;
    if (!msg_head(buf, buf_len, off, variant, max_body, true, b, len, n, kind)) return kind;
    return wv_next(b, len, n, cnt) ? kPending : SS_FRAME_KIND_MALFORMED;
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
