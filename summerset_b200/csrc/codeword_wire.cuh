// codeword_wire.cuh -- the bincode RSCodeword on the device, for every call that reads or writes one (the acceptor, the
// CRaft follower, leader and reconstruct calls, the PrepareReply parser): its parser, its size, its warp writer, and the
// warp copies of its shards into padded store slots.
#pragma once
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

// A present shard's Some tag plus its length varint, from the varint's tag byte t: a non-minimal varint is as valid as
// cw_parse found it, so its width comes from its own tag byte
__device__ __forceinline__ uint64_t some_len(uint8_t t) { return 1u + (t < 251u ? 1u : t == 251u ? 3u : t == 252u ? 5u : 9u); }

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
        const uint64_t sl = some_len(tags[at + 1u]);
        if ((take >> j) & 1u) {
            const uint64_t slot = dst_mask == ~0ull ? k++ : static_cast<uint64_t>(__popc(static_cast<uint32_t>(dst_mask) & ((1u << j) - 1u)));
            warp_fill_slot(dst + slot * pitch, tags + at + sl, L, lane);
        }
        at += sl + static_cast<uint64_t>(L);
    }
}

// An RSCodeword of the code (d, T) in the body b[0..len) from position n on (rscoding.rs:43-72): num_data_shards and
// num_parity_shards as raw bytes, data_len < 2^32, shard_len = ceil(data_len / d) (rscoding.rs:177-181), exactly T shard
// Options each present one shard_len bytes, then data_copy: None, or with kSomeCopy also Some(data_len bytes).  On
// success n is past data_copy, tags_at is the body position of shard 0's Option tag and held the present shards;
// false: malformed or truncated (the outputs are then unspecified).
template <bool kSomeCopy>
__device__ __forceinline__ bool cw_parse(const uint8_t *b, uint64_t len, uint64_t &n, uint32_t d, uint32_t T, uint64_t &dl,
                                         uint64_t &sl, uint64_t &tags_at, uint32_t &held) {
    uint64_t v = 0;
    if (len - n < 2u || b[n] != d || b[n + 1] != T - d) return false;      // num_data_shards, num_parity_shards
    n += 2;
    if (!wv_next(b, len, n, dl) || !wv_next(b, len, n, sl) || !wv_next(b, len, n, v)) return false;
    if (dl > 0xffffffffull || v != T || sl != (dl + d - 1u) / d) return false;
    tags_at = n;
    held = 0;
    for (uint32_t j = 0; j < T; ++j) {
        if (n >= len) return false;
        const uint8_t tag = b[n++];
        if (tag == 0u) continue;
        if (tag != 1u || !wv_next(b, len, n, v) || v != sl || len - n < sl) return false;
        held |= 1u << j;
        n += sl;
    }
    if (n >= len) return false;
    const uint8_t tag = b[n++];                                             // data_copy
    if (kSomeCopy && tag == 1u) {
        if (len - n < dl) return false;
        n += dl;
        return true;
    }
    return tag == 0u;
}

// bytes of a bincode RSCodeword of data_len dl under the code (d, T) carrying k shards: d, p, data_len, shard_len, T,
// T shard Options, data_copy None
__device__ __forceinline__ uint64_t cw_bytes(uint64_t dl, uint32_t d, uint32_t T, uint32_t k) {
    const uint64_t L = (dl + d - 1u) / d;
    return 2u + wv_len(dl) + wv_len(L) + wv_len(T) + T + static_cast<uint64_t>(k) * (wv_len(L) + L) + 1u;
}

// shard j of a codeword whose shards sit in planes: src + j * plane_stride
struct Planes {
    const uint8_t *src;
    uint64_t stride;
    __device__ __forceinline__ const uint8_t *operator()(uint32_t j) const { return src + static_cast<uint64_t>(j) * stride; }
};

// That codeword carrying the shards `mask`, written by a warp at p (any alignment): lane 0 writes the varints and the
// Option tags, the warp copies shard j from shard(j), a 16-byte aligned address: a store slot by rank (the follower's
// reconstruct serve passes a lambda) or a plane (Planes).  Returns its bytes.
template <typename Src>
__device__ __forceinline__ uint64_t warp_put_cw(uint8_t *p, uint32_t d, uint32_t T, uint64_t dl, uint32_t mask, Src &&shard,
                                                uint32_t lane) {
    const uint64_t L = (dl + d - 1u) / d;
    const uint32_t wl = static_cast<uint32_t>(wv_len(L));
    if (lane == 0u) {
        p[0] = static_cast<uint8_t>(d);
        p[1] = static_cast<uint8_t>(T - d);
        uint64_t m = 2u;
        m += wv_put(p + m, dl);
        m += wv_put(p + m, L);
        wv_put(p + m, T);
    }
    uint64_t m = 2u + wv_len(dl) + wl + wv_len(T);
    for (uint32_t j = 0; j < T; ++j) {
        if ((mask >> j) & 1u) {
            if (lane == 0u) {
                p[m] = 1u;
                wv_put(p + m + 1u, L);
            }
            m += 1u + wl;
            warp_copy_bytes(p + m, shard(j), static_cast<uint32_t>(L), lane);
            m += L;
        } else {
            if (lane == 0u) p[m] = 0u;
            m += 1u;
        }
    }
    if (lane == 0u) p[m] = 0u;                                            // data_copy: None
    return m + 1u;
}

// PeerMessage::Msg{PrepareReply{slot, trigger_slot, endprep_slot, ballot, voted}} at buf + off, with the codeword checked
// as ss_acceptor_absorb checks one; the shards stay where they are (shards_at).  Shared by ss_prepare_reply_parse_dev
// and ss_engine_prepare_absorb.
__device__ __forceinline__ ss_prepare_reply_rec prepare_reply_decode(const uint8_t *buf, uint64_t buf_len, uint64_t off, uint32_t d,
                                                                     uint32_t T, uint32_t variant) {
    ss_prepare_reply_rec r{};
    r.kind = SS_FRAME_KIND_MALFORMED;
    r.shards_at = ~0ull;
    do {
        const uint8_t *b;
        uint64_t len, n, f0 = 0, f1 = 0, f2 = 0, f3 = 0, vb = 0, dl = 0, sl = 0, at = ~0ull;
        uint32_t mask = 0;
        if (!msg_head(buf, buf_len, off, variant, ~0ull, true, b, len, n, r.kind)) break;
        if (!wv_next(b, len, n, f0) || !wv_next(b, len, n, f1) || !wv_next(b, len, n, f2) || !wv_next(b, len, n, f3) || n >= len)
            break;
        const uint8_t tag = b[n++];
        if (tag == 1u) {
            uint64_t tags_at = 0;
            if (!wv_next(b, len, n, vb) || !cw_parse<true>(b, len, n, d, T, dl, sl, tags_at, mask)) break;
            at = off + 8u + tags_at;
        } else if (tag != 0u) {
            break;
        }
        if (n != len) break;
        r.slot = f0; r.trigger_slot = f1; r.endprep_slot = f2; r.ballot = f3;
        r.vote_bal = vb; r.vote_mask = mask; r.data_len = static_cast<uint32_t>(dl); r.shards_at = at;
        r.kind = variant;
    } while (false);
    return r;
}

}  // namespace ssb
