// codeword_wire.cuh -- the bincode RSCodeword on the device: the warp copies of its shards into padded store slots, shared
// by the acceptor (acceptor.cu) and the CRaft follower (follower.cu), and the follower's codeword parser.
#pragma once
#include "device_common.cuh"
#include "ss_internal.hpp"
#include "wire_common.cuh"

namespace ssb {

// one shard of L bytes at src (any alignment) into its padded store slot at dst (16-byte aligned): aligned 128-bit
// stores, each fed by dev::load16, bytes L..round_up(L, 16) zero
__device__ __forceinline__ void warp_fill_slot(uint8_t *dst, const uint8_t *src, uint64_t L, uint32_t lane) {
    const uint64_t nvec = (L + 15u) >> 4;
    for (uint64_t v = lane; v < nvec; v += 32u) {
        const uint64_t left = L - v * 16u;
        dev::stg128_cs(dst + v * 16u, dev::load16(src + v * 16u, left < 16u ? static_cast<int>(left) : 16));
    }
}

// the T shard Options of a bincode RSCodeword starting at tags (Option tag, length varint, bytes): the shards of `take`
// (a subset of the present ones, `present`) go to their padded slots of the region at dst: one after the other, or with
// a dst_mask, shard j at its rank among the shards of dst_mask
__device__ __forceinline__ void warp_fill_shards(uint8_t *dst, const uint8_t *tags, uint32_t T, uint32_t present, uint32_t take,
                                                 uint32_t L, uint32_t lane, uint64_t dst_mask = ~0ull) {
    const uint64_t pitch = SS_CW_SLOT_PITCH(L);
    uint64_t at = 0;
    uint32_t k = 0;
    for (uint32_t j = 0; j < T; ++j) {
        if (!((present >> j) & 1u)) { at += 1u; continue; }
        // Some tag, then the shard length as the frame spells it: a non-minimal varint is as valid as the header pass
        // found it, so its width comes from its own tag byte
        const uint8_t t = tags[at + 1u];
        const uint64_t some_len = 1u + (t < 251u ? 1u : t == 251u ? 3u : t == 252u ? 5u : 9u);
        if ((take >> j) & 1u) {
            const uint64_t slot = dst_mask == ~0ull ? k++ : static_cast<uint64_t>(__popc(static_cast<uint32_t>(dst_mask) & ((1u << j) - 1u)));
            warp_fill_slot(dst + slot * pitch, tags + at + some_len, L, lane);
        }
        at += some_len + static_cast<uint64_t>(L);
    }
}

// An RSCodeword of the code (d, T) in the body b[0..len) from position n on (rscoding.rs:43-72), checked by the rules of
// the acceptor's decode_frame (which keeps its own inline copy: calling this function from there changes the SASS of
// acceptor_header_kernel): num_data_shards and
// num_parity_shards as raw bytes, data_len < 2^32, shard_len = ceil(data_len / d) (rscoding.rs:177-181), exactly T shard
// Options each present one shard_len bytes, data_copy None.  On success n is past data_copy, tags_at is the position
// of shard 0's Option tag counted from the frame's start (8 + the body position), held the
// present shards, v is scratch; false: malformed or truncated (the outputs are then unspecified).
__device__ __forceinline__ bool cw_parse(const uint8_t *b, uint64_t len, uint64_t &n, uint32_t d, uint32_t T, uint64_t &dl,
                                         uint64_t &sl, uint32_t &tags_at, uint32_t &held, uint64_t &v) {
    uint32_t c;
    if (len - n < 2u || b[n] != d || b[n + 1] != T - d) return false;      // num_data_shards, num_parity_shards
    n += 2;
    if (!(c = wv_get(b + n, len - n, dl))) return false;
    n += c;
    if (!(c = wv_get(b + n, len - n, sl))) return false;
    n += c;
    if (!(c = wv_get(b + n, len - n, v))) return false;
    n += c;
    if (dl > 0xffffffffull || v != T || sl != (dl + d - 1u) / d) return false;
    tags_at = static_cast<uint32_t>(8u + n);
    held = 0;
    for (uint32_t j = 0; j < T; ++j) {
        if (n >= len) return false;
        const uint8_t tag = b[n++];
        if (tag == 0u) continue;
        if (tag != 1u) return false;
        if (!(c = wv_get(b + n, len - n, v))) return false;
        n += c;
        if (v != sl || len - n < sl) return false;
        held |= 1u << j;
        n += sl;
    }
    return n < len && b[n++] == 0u;                                         // data_copy: None
}

}  // namespace ssb
