// acceptor_state.hpp -- the RSPaxos / Crossword acceptor handle (ss_acceptor_*) and the Accept body decoder, shared by
// acceptor.cu and the WAL replay (acceptor_recover.cu).
#pragma once
#include "codeword_wire.cuh"
#include "ss_internal.hpp"
#include "wire_common.cuh"

namespace ssb {

// one decoded Accept frame (ss_acceptor_accept) or WAL record (ss_acceptor_recover)
struct FrameHdr {
    uint64_t slot, ballot;
    uint64_t end;                   // frame bytes: 8-byte length prefix + body
    uint32_t kind;                  // verdict so far
    uint32_t held, dlen, L;
    uint32_t slot_at;               // offset of the `slot` varint inside the frame
    uint32_t tags_at;               // offset of shard 0's Option tag
    uint32_t asg;                   // Crossword: assignment[me]
    uint32_t asg_at;                // Crossword: offset of assignment[0] inside the frame
};

}  // namespace ssb

struct ss_acceptor {
    ss_ctx *ctx = nullptr;
    ss_acceptor_config cfg{};
    uint64_t G = 0;
    uint64_t *window_base = nullptr, *bal_max_seen = nullptr, *inst_bal = nullptr, *accepting = nullptr, *shard_addr = nullptr;
    uint32_t *held = nullptr, *data_len = nullptr, *assignment = nullptr;
    uint8_t *source = nullptr;
    uint64_t *committed = nullptr, *commit_bar = nullptr, *exec_bar = nullptr;
    // Prepare: Status::Preparing (ring word), inst.voted = (voted_bal, voted_mask), replica_bk's trigger_slot and
    // endprep_slot - trigger_slot
    uint64_t *preparing = nullptr, *voted_bal = nullptr, *prep_trigger = nullptr;
    uint32_t *voted_mask = nullptr;
    uint8_t *prep_span = nullptr;
    // Crossword follower gossip: the instance's whole assignment ([G*64][population] rows) and gossip_bar ([G])
    uint32_t *assign_rows = nullptr;
    uint64_t *gossip_bar = nullptr;
    uint8_t *matrix = nullptr;      // [T*d] the coder's coding matrix (gf256.hpp), row-major
    uint64_t *ex_cnt = nullptr, *ex_bytes = nullptr, *ex_partials = nullptr, *ex_n = nullptr;   // execute scratch
    // per-call scratch, grow-only
    uint64_t cap_frames = 0;
    ssb::FrameHdr *hdr = nullptr;
    uint32_t *keys = nullptr;       // [2][cap]: sort keys in / out
    uint32_t *idx = nullptr;        // [2][cap]: frame indices in / out
    uint64_t *partials = nullptr;   // [scan_tiles(cap)]
    uint64_t *fcnt = nullptr;       // [cap]: ss_acceptor_prepare's per-frame record counts, then their scan
    void *sort_tmp = nullptr;
    size_t sort_tmp_bytes = 0;
    uint64_t *totals = nullptr;     // [2] when the caller passes none
};

namespace ssb {

constexpr int kAccThreads = 256;
// WAL records in the window that are not AcceptData (ss_acceptor_recover)
constexpr uint32_t kPendingPrepareBal = 0xfffffffdu;
constexpr uint32_t kPendingCommitSlot = 0xfffffffcu;

// grows the per-call scratch to n frames: headers, sort keys and indices, scan partials, per-frame counts (acceptor.cu)
int acc_scratch(ss_acceptor *a, uint64_t n);

__device__ __forceinline__ uint64_t store_bytes(const FrameHdr &h) {
    return static_cast<uint64_t>(__popc(h.held)) * SS_CW_SLOT_PITCH(h.L);
}

// Decodes frame i as ssor_decode_accept reads it, plus the acceptor's own checks (code, shard_len, assignment shape).
// kWal = false: A is ss_acceptor_accept's arguments and frame i a PeerMessage::Msg{Accept{...}}.  kWal = true: A is
// ss_acceptor_recover's and frame i a WalEntry: AcceptData (A.wal_variant) is the Accept body from `slot` on, PrepareBal
// {slot, ballot} and CommitSlot{slot} come back with kind kPendingPrepareBal / kPendingCommitSlot, any other variant is
// malformed.  Both end with the window filters.
template <bool kWal, typename Args>
__device__ __forceinline__ FrameHdr decode_frame(const Args &A, uint64_t i) {
    FrameHdr h{};
    h.kind = SS_FRAME_KIND_MALFORMED;
    const uint32_t grp = A.frame_group[i];
    const uint64_t off = A.frame_off[i];
    if (grp >= A.G) return h;
    const uint8_t *b;
    uint64_t len, n = 0, v = 0;
    if constexpr (kWal) {
        if (!frame_body(A.buf, A.buf_len, off, kMaxFrameBody, b, len) || !wv_next(b, len, n, v)) return h;
        if (v != A.wal_variant) {
            if (v != A.prepare_variant && v != A.commit_variant) return h;
            h.slot_at = static_cast<uint32_t>(8u + n);
            if (!wv_next(b, len, n, h.slot)) return h;
            if (v == A.prepare_variant && !wv_next(b, len, n, h.ballot)) return h;
            if (n != len) return h;
            h.end = 8u + len;
            const uint64_t base = A.window_base[grp];
            h.kind = h.slot < base                ? SS_ACCEPT_VERDICT_STALE_SLOT
                     : h.slot - base >= 64u       ? SS_ACCEPT_VERDICT_BEYOND_WINDOW
                     : v == A.prepare_variant     ? kPendingPrepareBal
                                                  : kPendingCommitSlot;
            return h;
        }
    } else {
        if (!msg_head(A.buf, A.buf_len, off, A.accept_variant, kMaxFrameBody, true, b, len, n, h.kind)) return h;
    }
    h.slot_at = static_cast<uint32_t>(8u + n);
    if (!wv_next(b, len, n, h.slot) || !wv_next(b, len, n, h.ballot)) return h;
    uint64_t dl = 0, sl = 0, tags_at = 0;
    uint32_t held = 0;
    if (!cw_parse<false>(b, len, n, A.d, A.T, dl, sl, tags_at, held)) return h;
    h.tags_at = static_cast<uint32_t>(8u + tags_at);
    if (A.crossword) {                                                      // assignment: Vec<Bitmap>, one row per replica
        if (!wv_next(b, len, n, v) || v != A.population) return h;
        h.asg_at = static_cast<uint32_t>(8u + n);
        for (uint32_t r = 0; r < A.population; ++r) {
            uint64_t sz = 0, nb = 0, blk = 0;
            if (!wv_next(b, len, n, sz) || !wv_next(b, len, n, nb) || sz != A.T || nb != 1u) return h;
            if (!wv_next(b, len, n, blk) || (blk >> A.T)) return h;
            if (r == A.me) h.asg = static_cast<uint32_t>(blk);
        }
    }
    if (n != len) return h;
    h.end = 8u + len;
    h.held = held;
    h.dlen = static_cast<uint32_t>(dl);
    h.L = static_cast<uint32_t>(sl);
    const uint64_t base = A.window_base[grp];
    h.kind = h.slot < base ? SS_ACCEPT_VERDICT_STALE_SLOT : h.slot - base >= 64u ? SS_ACCEPT_VERDICT_BEYOND_WINDOW : kPending;
    return h;
}

// WalEntry::PrepareBal{slot, ballot} as the 32-byte cell at dst (16-byte aligned): 8-byte big-endian length, the bincode
// body (at most 21 bytes with wal_variant < 2^16), zero to the end of the cell.  Written by ss_acceptor_prepare and
// ss_acceptor_step_up.
__device__ __forceinline__ void put_prepare_bal_cell(uint8_t *dst, uint32_t wal_variant, uint64_t slot, uint64_t ballot) {
    uint8_t cell[32];
#pragma unroll
    for (int b = 0; b < 32; ++b) cell[b] = 0u;
    uint32_t m = 8u;
    m += wv_put(cell + m, wal_variant);
    m += wv_put(cell + m, slot);
    m += wv_put(cell + m, ballot);
    cell[7] = static_cast<uint8_t>(m - 8u);                                  // the body is < 256 bytes
    uint4 lo, hi;
    memcpy(&lo, cell, 16);
    memcpy(&hi, cell + 16, 16);
    uint4 *d = reinterpret_cast<uint4 *>(dst);
    d[0] = lo;
    d[1] = hi;
}

// the whole assignment of a frame whose rows decode_frame validated, from rb = the frame + asg_at, lim = end - asg_at
// bytes on: row r into rows[first + r]
__device__ __forceinline__ void read_assign_rows(const uint8_t *rb, uint64_t lim, uint32_t population, uint32_t *rows, uint64_t first) {
    uint64_t q = 0, sz = 0, nb = 0, blk = 0;
    for (uint32_t r = 0; r < population; ++r) {
        q += wv_get(rb + q, lim - q, sz);
        q += wv_get(rb + q, lim - q, nb);
        q += wv_get(rb + q, lim - q, blk);
        rows[first + r] = static_cast<uint32_t>(blk);
    }
}

}  // namespace ssb
