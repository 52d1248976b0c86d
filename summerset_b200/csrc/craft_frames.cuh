// craft_frames.cuh -- the device decoders of the four CRaft messages that carry a term, shared by the calls that take
// them (follower.cu: AppendEntries and the leader's AppendEntriesReply parser; craft_election.cu: RequestVote and
// RequestVoteReply) and by the step-down's check_term over a batch of them (craft_stepdown.cu).
#pragma once
#include "codeword_wire.cuh"
#include "engine_state.hpp"
#include "ss_internal.hpp"
#include "wire_common.cuh"

namespace ssb {

// ---- AppendEntries (the follower's decoder) ------------------------------------------------------------------------
// one decoded AppendEntries frame
struct FolHdr {
    uint64_t term, prev, prev_term, n_ent, commit, snap;
    uint64_t store_sz, wal_sz;      // the regions the frame reserves
    uint32_t ents_at;               // offset of entry 0 inside the frame
    uint32_t kind;                  // verdict so far
    uint64_t first_k;               // replay: index of the first appended entry (n_ent: none appended)
};

// one LogEntry inside a frame; offsets count from the frame's start
struct Ent {
    uint64_t term, dl, sl;
    uint32_t held, tags_at, start, ext_end, next;
};

struct FolArgs {
    const uint8_t *buf;
    uint64_t buf_len;
    const uint64_t *frame_off;
    const uint32_t *frame_group;
    const uint8_t *frame_peer;
    uint64_t n, G;
    uint32_t d, T, W, me, population, append_variant, reply_variant, meta_variant, log_variant;
    uint64_t *start_slot, *log_end, *curr_term, *last_commit, *last_snap;
    uint8_t *leader;
    uint64_t *term, *shard_addr;
    uint32_t *held, *data_len;
    FolHdr *hdr;
    uint32_t *key_in, *idx_in;
    const uint32_t *key, *idx;
    uint64_t *cut, *abs_cursor, *tot;
    uint8_t *store;
    uint64_t store_cap, *store_off;
    uint8_t *wal;
    uint64_t wal_cap, *wal_off, *wal_len;
    uint8_t *meta;
    uint32_t *meta_len;
    uint8_t *replies;
    uint32_t *reply_len;
    uint8_t *reply_dst;
    uint64_t *trunc_slot;
    uint32_t *verdict, *status;
};

// entry at frame offset `at` of a frame whose body is fr[8 .. end): term, the codeword, external (a raw bool byte),
// log_offset
__device__ __forceinline__ bool ent_parse(const uint8_t *fr, uint64_t end, uint64_t at, uint32_t d, uint32_t T, Ent &e) {
    const uint8_t *b = fr + 8;
    const uint64_t len = end - 8u;
    uint64_t n = at - 8u, v = 0, term = 0, dl = 0, sl = 0, tags_at = 0;
    uint32_t held = 0;
    if (!wv_next(b, len, n, term) || !cw_parse<false>(b, len, n, d, T, dl, sl, tags_at, held)) return false;
    if (n >= len || b[n] > 1u) return false;                                // external: bool
    const uint32_t ext_end = static_cast<uint32_t>(8u + n + 1u);
    ++n;
    if (!wv_next(b, len, n, v)) return false;                               // log_offset, dropped
    e.term = term; e.dl = dl; e.sl = sl; e.held = held; e.tags_at = static_cast<uint32_t>(8u + tags_at);
    e.start = static_cast<uint32_t>(at); e.ext_end = ext_end; e.next = static_cast<uint32_t>(8u + n);
    return true;
}

__device__ __forceinline__ uint64_t ent_store_bytes(const Ent &e) {
    return static_cast<uint64_t>(__popc(e.held)) * SS_CW_SLOT_PITCH(e.sl);
}
__device__ __forceinline__ uint64_t ent_rec_len(const Ent &e, uint32_t log_variant) {
    return 8u + static_cast<uint64_t>(wv_len(log_variant)) + (e.ext_end - e.start) + 1u;
}

// decodes frame i: PeerMessage::Msg{AppendEntries{term, prev_slot, prev_term, entries, leader_commit, last_snap}}
__device__ __forceinline__ FolHdr fol_decode(const FolArgs &A, uint64_t i) {
    FolHdr h{};
    h.kind = SS_FRAME_KIND_MALFORMED;
    const uint32_t grp = A.frame_group[i];
    const uint64_t off = A.frame_off[i];
    if (grp >= A.G || A.frame_peer[i] == A.me || A.frame_peer[i] >= A.population) return h;
    const uint8_t *b;
    uint64_t len, n;
    if (!msg_head(A.buf, A.buf_len, off, A.append_variant, kMaxFrameBody, true, b, len, n, h.kind)) return h;
    const uint8_t *fr = b - 8;
    uint64_t term = 0, prev = 0, prev_term = 0, n_ent = 0;
    if (!wv_next(b, len, n, term) || !wv_next(b, len, n, prev) || !wv_next(b, len, n, prev_term) || !wv_next(b, len, n, n_ent))
        return h;
    const uint64_t ents_at = 8u + n;
    uint64_t sz = 0, wz = 0;
    for (uint64_t k = 0; k < n_ent; ++k) {
        Ent e;
        if (!ent_parse(fr, 8u + len, 8u + n, A.d, A.T, e)) return h;
        sz += ent_store_bytes(e);
        wz += round16(ent_rec_len(e, A.log_variant));
        n = e.next - 8u;
    }
    uint64_t commit = 0, snap = 0;
    if (!wv_next(b, len, n, commit) || !wv_next(b, len, n, snap) || n != len) return h;
    h.term = term; h.prev = prev; h.prev_term = prev_term; h.n_ent = n_ent; h.commit = commit; h.snap = snap;
    h.store_sz = sz; h.wal_sz = wz;
    h.ents_at = static_cast<uint32_t>(ents_at);
    h.first_k = n_ent;
    // every entry inside [start_slot, start_slot + window): the ring holds them
    const uint64_t start = A.start_slot[grp];
    const bool beyond = n_ent != 0u && (prev + n_ent < prev || prev + n_ent >= start + A.W);
    h.kind = beyond ? SS_FOLLOWER_VERDICT_BEYOND_WINDOW : kPending;
    return h;
}

// ---- AppendEntriesReply (the leader's parser) ----------------------------------------------------------------------
// PeerMessage::Msg{AppendEntriesReply{term, end_slot, conflict}} at buf + off for group grp: the record kind of
// ss_append_reply_parse_dev against curr_term[grp] (SS_APPEND_REPLY_*: the frame decoded, its fields set), or another
// message's variant index (0x80000000 | k for PeerMessage variants) or SS_FRAME_KIND_MALFORMED
__device__ __forceinline__ uint32_t reply_parse(const uint8_t *buf, uint64_t buf_len, uint64_t off, uint32_t grp, uint64_t G,
                                                uint32_t reply_variant, const uint32_t *curr_term, uint64_t &term, uint64_t &end,
                                                uint64_t &c_term, uint64_t &c_slot) {
    uint32_t kind = SS_FRAME_KIND_MALFORMED;
    do {
        const uint8_t *b;
        uint64_t len, n;
        if (grp >= G || !msg_head(buf, buf_len, off, reply_variant, ~0ull, true, b, len, n, kind)) break;
        if (!wv_next(b, len, n, term) || !wv_next(b, len, n, end)) break;
        if (n >= len) break;
        const uint8_t tag = b[n++];
        if (tag == 1u) {
            if (!wv_next(b, len, n, c_term) || !wv_next(b, len, n, c_slot)) break;
        } else if (tag != 0u) {
            break;
        }
        if (n != len) break;
        // check_term first (messages.rs:272-274): a higher term makes the leader step down and drop the reply
        kind = term > curr_term[grp] ? SS_APPEND_REPLY_HIGHER_TERM
             : tag == 1u             ? SS_APPEND_REPLY_CONFLICT
             : end > 0xffffffffull   ? SS_APPEND_REPLY_END_RANGE
                                     : SS_APPEND_REPLY_INGEST;
    } while (false);
    return kind;
}

// ---- RequestVote and RequestVoteReply (the election decoders) -------------------------------------------------------
constexpr uint8_t kNone = 0xffu;                 // ReplicaId::MAX: voted_for None, leader None
constexpr uint32_t kMetaCell = 32u;

// DurEntry::Metadata{curr_term, voted_for} into a 32-byte cell (at most 8 + 3 + 9 + 1 bytes), zero to its end
__device__ __forceinline__ uint32_t el_put_meta(uint8_t *cell, uint32_t variant, uint64_t term, uint8_t voted_for) {
    uint32_t m = 8u;
    m += wv_put(cell + m, variant);
    m += wv_put(cell + m, term);
    cell[m++] = voted_for;
    put_be64(cell, m - 8u);
    for (uint32_t q = m; q < kMetaCell; ++q) cell[q] = 0u;
    return m;
}

struct ElectArgs {
    const uint8_t *buf;
    uint64_t buf_len;
    const uint64_t *frame_off;
    const uint32_t *frame_group;
    const uint8_t *frame_peer;
    uint64_t n, G;
    uint32_t W, me, population, majority, variant, reply_variant, meta_variant;
    const uint64_t *log_end, *term;
    uint64_t *curr_term;
    uint8_t *leader;
    uint64_t *vote_term, *role_term;
    uint8_t *voted_for, *role;
    uint32_t *votes;
    uint32_t *key_in, *idx_in;
    const uint32_t *key, *idx;
    uint8_t *meta;
    uint32_t *meta_len;
    uint8_t *replies;               // vote only
    uint32_t *reply_len;
    uint8_t *reply_dst;
    uint32_t *verdict;
    uint64_t *won_flag;             // tally only: [n] per sorted frame, then its exclusive scan
    const uint64_t *n_won;
    uint32_t *won_group;
    uint64_t *won_term;
};

// Frame i: PeerMessage::Msg{RequestVote{term, last_slot, last_term}} (kReply false) or
// PeerMessage::Msg{RequestVoteReply{term, granted}} (kReply true: f1 = granted).  kPending when it is one, else its
// verdict: another message's variant index (0x80000000 | k for PeerMessage variants) or SS_FRAME_KIND_MALFORMED
template <bool kReply>
__device__ __forceinline__ uint32_t el_decode(const ElectArgs &A, uint64_t i, uint64_t &f0, uint64_t &f1, uint64_t &f2) {
    const uint32_t g = A.frame_group[i];
    const uint64_t off = A.frame_off[i];
    const uint8_t peer = A.frame_peer[i];
    if (g >= A.G || peer == A.me || peer >= A.population) return SS_FRAME_KIND_MALFORMED;
    const uint8_t *b;
    uint64_t len, n;
    uint32_t kind;
    if (!msg_head(A.buf, A.buf_len, off, A.variant, ~0ull, true, b, len, n, kind)) return kind;
    if (!wv_next(b, len, n, f0)) return SS_FRAME_KIND_MALFORMED;
    if (kReply) {
        if (n >= len || b[n] > 1u) return SS_FRAME_KIND_MALFORMED;  // bool
        f1 = b[n++];
        f2 = 0u;
    } else if (!wv_next(b, len, n, f1) || !wv_next(b, len, n, f2)) {
        return SS_FRAME_KIND_MALFORMED;
    }
    return n == len ? kPending : SS_FRAME_KIND_MALFORMED;
}

}  // namespace ssb
