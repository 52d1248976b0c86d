// acceptor.cu -- the follower side of the RSPaxos / Crossword accept path behind the C ABI (ss_acceptor_*).
//
// What a follower does for every Accept (SURVEY 3.2 step 4): handle_msg_accept (rspaxos/messages.rs:329-392,
// crossword/messages.rs:403-470) with check_leader's bal_max_seen update (rspaxos/leadership.rs:11-17), the
// WalEntry::AcceptData it logs, and the AcceptReply it sends once the record is durable (rspaxos/durability.rs:101-118,
// crossword/durability.rs:96-125) -- for a batch of frames of many groups at once:
//
//   acceptor_header_kernel   a thread per frame: walks the varints, validates, keeps the fields, the held mask and the
//                            offsets of `slot` and of the first shard tag; slot / window filters; region sizes
//   (CUB radix sort)         frame indices stably sorted by group: each group's frames in frame order
//   acceptor_ballot_kernel   a thread per group segment: check_leader's running maximum, replayed in frame order
//   (engine.cu's scan)       store and WAL regions: exclusive scans in frame order
//   acceptor_place_kernel    a thread per group segment, backwards: capacity, the final verdicts, the last accepted
//                            frame of each (group, slot) defines the instance, bal_max_seen = max of the accepted
//   acceptor_copy_kernel     a warp per accepted frame: the AcceptData record (length, wal_variant, the frame from `slot`
//                            on, verbatim), the held shards into their padded store slots, the AcceptReply cell
//
// Frames sit in a receive buffer at any byte alignment; every 128-bit store is aligned, its 16 source bytes come from
// the two aligned loads around them (dev::load16).
//
// What the follower does next: the commit half of heard_heartbeat (rspaxos/leadership.rs:222-311,
// crossword/leadership.rs:260-359) and, once the CommitSlot records are durable, handle_logged_commit_slot's execution
// walk (rspaxos/durability.rs:125-186, crossword/durability.rs:142-206):
//
//   heartbeat_keys_kernel    a thread per record: sort keys (the records are then stably sorted by group as above)
//   heartbeat_walk_kernel    a thread per group segment: check_leader, the ballot / exec_bar filters and the commit walk
//                            of every record of the group in record order
//   (exec_walk.cuh, AccLog)  a thread per group: how many instances the walk executes, their payload bytes, then the
//                            records and commit_bar; a warp per executed instance: get_data's bytes, with
//                            reconstruct_data's regeneration of missing data shards from the first d held shards
//                            (Gauss-Jordan on the device, then packed GF(2^8) Horner rows on the byte stream)
//
// Reconstruct reads, for the instances the follower cannot execute from its own shards: handle_msg_reconstruct
// (rspaxos/messages.rs:468-516, crossword/messages.rs:577-632) and handle_msg_reconstruct_reply
// (rspaxos/messages.rs:519-594, crossword/messages.rs:635-722):
//
//   serve_count_kernel       a warp per Reconstruct frame: filters, refusals, one entry per slot, reply bytes
//   (engine.cu's scan)       reply regions
//   serve_copy_kernel        a warp per frame: capacity, the ReconstructReply with entries in the order of their defining
//                            occurrences, shards from the store slots
//   absorb_decode_kernel     a thread per ReconstructReply frame: validates, notes a slot repeated in the window
//   (CUB radix sort)         frames by group, as above
//   absorb_plan_kernel       a warp per group segment: the entries in frame, then wire order; bytes of the growing regions
//   (engine.cu's scan)       group region offsets
//   absorb_copy_kernel       a warp per group segment: capacity, old and new shards into the new regions, held /
//                            shard_addr, per-frame counts and verdicts
// Stated differences from the reference: include/summerset_b200.h at ss_acceptor_reconstruct_serve.
//
// The follower half of leader fail-over: handle_msg_prepare (rspaxos/messages.rs:13-84, crossword/messages.rs:63-136)
// and, once the PrepareBal records are durable, the follower branch of handle_logged_prepare_bal
// (rspaxos/durability.rs:10-79, crossword/durability.rs:9-79):
//
//   prepare_header_kernel    a thread per Prepare frame: decode, window filters, sort keys
//   (CUB radix sort)         frames by group, as above
//   prepare_walk_kernel      a thread per group segment: check_leader and each frame's [trigger_slot, endprep_slot],
//                            replayed in frame order over the group's state words held in registers; writes no state
//   (engine.cu's scan)       record numbers: exclusive scan of the per-frame counts in frame order
//   prepare_apply_kernel     a thread per group segment, last frame first: the capacity suffix, verdicts, state words,
//                            bal_max_seen, and the positions each applied frame defines
//   prepare_write_kernel     a warp per applied frame: the PrepareBal cells, the per-slot arrays of the defined positions
//   prep_reply_size_kernel   a thread per record: PrepareReply bytes
//   (engine.cu's scan)       reply regions
//   prep_reply_copy_kernel   a warp per record: capacity, the PrepareReply with the voted shards (the RSCodeword writer
//                            serve_copy_kernel uses)
//
// Reconstruct requests for the instances this follower cannot execute: Crossword's trigger_gossiping with
// gossip_targets_excl (crossword/gossiping.rs:35-192) and become_a_leader's recon_slots (rspaxos/leadership.rs:99-172,
// crossword/leadership.rs:105-190):
//
//   request_size_kernel      a warp per listed group: the walk, each lane's two instances planned (gossip_walk.cuh),
//                            per destination the entries' bytes, frames and region bytes
//   (engine.cu's scan)       frame numbers and regions per listed group
//   request_write_kernel     a warp per listed group: the per-group capacity cut, the same plan again, frame headers and
//                            entries, gossip_bar
#include <cub/device/device_radix_sort.cuh>

#include <cstring>
#include <new>

#include "acceptor_state.hpp"
#include "codeword_wire.cuh"
#include "device_common.cuh"
#include "exec_walk.cuh"
#include "gf256.hpp"
#include "ss_internal.hpp"
#include "gossip_walk.cuh"
#include "window_ring.cuh"
#include "wire_common.cuh"

namespace ssb {

// one decoded ReconstructReply frame (ss_acceptor_absorb); it lives in the FrameHdr scratch, which is at least as large
struct ReplyHdr {
    uint64_t count;                 // map entries
    uint64_t entries_at;            // offset of the first entry inside the body
    uint64_t body_len;              // bytes after the 8-byte length prefix
    uint32_t kind;                  // verdict so far
    uint32_t repeated;              // a slot inside the window appears twice: its last value counts
};
static_assert(sizeof(ReplyHdr) <= sizeof(FrameHdr) && alignof(ReplyHdr) <= alignof(FrameHdr), "ReplyHdr reuses FrameHdr scratch");

// one decoded Prepare frame (ss_acceptor_prepare), also in the FrameHdr scratch
struct PrepHdr {
    uint64_t trigger, ballot;
    uint64_t endprep;               // the walk's endprep_slot, for the frames that pass
    uint64_t define;                // ring positions for which this frame is the last applied frame covering them
    uint64_t fresh;                 // of those, the ones null before the call: their vote becomes None
    uint32_t kind;                  // verdict so far
    uint32_t pad;
};
static_assert(sizeof(PrepHdr) <= sizeof(FrameHdr) && alignof(PrepHdr) <= alignof(FrameHdr), "PrepHdr reuses FrameHdr scratch");
static_assert(kAccThreads == kExecThreads, "the warp kernels run kExecWarps warps per kAccThreads-thread CTA");

struct AccArgs {
    const uint8_t *buf;
    uint64_t buf_len;
    const uint64_t *frame_off;
    const uint32_t *frame_group;
    const uint8_t *frame_peer;
    uint64_t n, G;
    uint32_t d, T, population, me, accept_variant, wal_variant, reply_variant, crossword;
    // state
    uint64_t *window_base, *bal_max_seen, *inst_bal, *accepting, *shard_addr, *committed;
    uint32_t *held, *data_len, *assignment, *assign_rows;
    uint8_t *source;
    uint64_t *preparing, *voted_bal, *prep_trigger;
    uint32_t *voted_mask;
    uint8_t *prep_span;
    // scratch
    FrameHdr *hdr;
    uint32_t *key_in, *idx_in;
    const uint32_t *key, *idx;      // sorted
    // outputs
    uint8_t *store;
    uint64_t store_cap;
    uint64_t *store_off;
    uint8_t *wal;
    uint64_t wal_cap;
    uint64_t *wal_off;
    uint32_t *wal_len;
    uint8_t *replies;
    uint32_t *reply_len;
    uint8_t *reply_dst;
    uint32_t *verdict;
    uint32_t *status;
};

__device__ __forceinline__ uint64_t wal_bytes(const FrameHdr &h, uint32_t wal_variant) {
    return 8u + static_cast<uint64_t>(wv_len(wal_variant)) + (h.end - h.slot_at);
}

// 1. a thread per frame: decode, filter, region sizes (0 for frames that cannot be accepted), sort keys
__global__ void __launch_bounds__(kAccThreads) acceptor_header_kernel(const __grid_constant__ AccArgs A) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kAccThreads;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kAccThreads + threadIdx.x; i < A.n; i += stride) {
        const FrameHdr h = decode_frame<false>(A, i);
        A.hdr[i] = h;
        const bool pending = h.kind == kPending;
        A.store_off[i] = pending ? store_bytes(h) : 0ull;
        A.wal_off[i] = pending ? round16(wal_bytes(h, A.wal_variant)) : 0ull;
        const uint32_t grp = A.frame_group[i];
        A.key_in[i] = grp < A.G ? grp : static_cast<uint32_t>(A.G);
        A.idx_in[i] = static_cast<uint32_t>(i);
    }
}

__device__ __forceinline__ bool segment_head(const AccArgs &A, uint64_t t) { return t == 0u || A.key[t] != A.key[t - 1]; }

// 2. a thread per group segment (the group's frames in frame order): a frame inside the window passes when its ballot
//    is at least the running maximum, which it then raises (check_leader); the others are stale and take no room
__global__ void __launch_bounds__(kAccThreads) acceptor_ballot_kernel(const __grid_constant__ AccArgs A) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kAccThreads;
    for (uint64_t t = static_cast<uint64_t>(blockIdx.x) * kAccThreads + threadIdx.x; t < A.n; t += stride) {
        if (!segment_head(A, t)) continue;
        const uint32_t g = A.key[t];
        if (g >= A.G) continue;
        uint64_t run = A.bal_max_seen[g];
        for (uint64_t k = t; k < A.n && A.key[k] == g; ++k) {
            const uint32_t i = A.idx[k];
            if (A.hdr[i].kind != kPending) continue;
            const uint64_t bal = A.hdr[i].ballot;
            if (bal < run) {
                A.hdr[i].kind = SS_ACCEPT_VERDICT_STALE_BALLOT;
                A.store_off[i] = 0ull;
                A.wal_off[i] = 0ull;
            } else {
                A.hdr[i].kind = SS_ACCEPT_VERDICT_ACCEPTED;            // subject to capacity
                run = bal;
            }
        }
    }
}

// 3. a thread per group segment, last frame first: store_off / wal_off hold the scanned region starts.  A frame whose
//    region ends past the capacity changes nothing; of the accepted frames of one slot the last defines the instance.
__global__ void __launch_bounds__(kAccThreads) acceptor_place_kernel(const __grid_constant__ AccArgs A) {
    bool store_full = false, wal_full = false;
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kAccThreads;
    for (uint64_t t = static_cast<uint64_t>(blockIdx.x) * kAccThreads + threadIdx.x; t < A.n; t += stride) {
        if (!segment_head(A, t)) continue;
        const uint32_t g = A.key[t];
        const bool known = g < A.G;
        uint64_t e = t + 1u;
        while (e < A.n && A.key[e] == g) ++e;
        uint64_t seen = 0ull, mx = known ? A.bal_max_seen[g] : 0ull;
        for (uint64_t k = e; k-- > t;) {
            const uint32_t i = A.idx[k];
            const FrameHdr h = A.hdr[i];
            uint32_t kind = h.kind;
            if (kind == SS_ACCEPT_VERDICT_ACCEPTED) {
                const uint64_t so = A.store_off[i], sz = store_bytes(h), wo = A.wal_off[i];
                const uint64_t wl = wal_bytes(h, A.wal_variant);
                if (so > A.store_cap || sz > A.store_cap - so) {
                    kind = SS_ACCEPT_VERDICT_STORE_FULL;
                    store_full = true;
                } else if (wo > A.wal_cap || round16(wl) > A.wal_cap - wo) {
                    kind = SS_ACCEPT_VERDICT_WAL_FULL;
                    wal_full = true;
                } else {
                    A.wal_len[i] = static_cast<uint32_t>(wl);
                    mx = h.ballot > mx ? h.ballot : mx;
                    const uint32_t pos = static_cast<uint32_t>(h.slot & 63u);
                    if (!((seen >> pos) & 1ull)) {                     // the last accepted frame of this slot
                        seen |= 1ull << pos;
                        const uint64_t at = static_cast<uint64_t>(g) * 64u + pos;
                        A.inst_bal[at] = h.ballot;
                        A.source[at] = A.frame_peer[i];
                        A.held[at] = h.held;
                        A.data_len[at] = h.dlen;
                        A.shard_addr[at] = reinterpret_cast<uint64_t>(A.store + so);
                        if (A.assignment != nullptr) {
                            A.assignment[at] = h.asg;
                            // the whole assignment, re-read from the rows the header pass validated
                            read_assign_rows(A.buf + A.frame_off[i] + h.asg_at, h.end - h.asg_at, A.population, A.assign_rows, at * A.population);
                        }
                        A.voted_bal[at] = h.ballot;                     // inst.voted = (ballot, reqs_cw as accepted)
                        A.voted_mask[at] = h.held;
                        A.prep_trigger[at] = 0u;                        // replica_bk = {source, 0, 0}
                        A.prep_span[at] = 0u;
                    }
                }
            }
            if (kind != SS_ACCEPT_VERDICT_ACCEPTED) {
                A.store_off[i] = ~0ull;
                A.wal_off[i] = ~0ull;
                A.wal_len[i] = 0u;
                A.reply_len[i] = 0u;
                A.reply_dst[i] = 0xffu;
            }
            A.verdict[i] = kind;
        }
        if (known) {
            A.accepting[g] |= seen;                                     // Status::Accepting, also for a committed slot
            A.committed[g] &= ~seen;                                    // (rspaxos/messages.rs:363)
            A.preparing[g] &= ~seen;
            A.bal_max_seen[g] = mx;
        }
    }
    if (store_full) atomicOr(A.status, SS_DEV_STATUS_STORE_FULL);
    if (wal_full) atomicOr(A.status, SS_DEV_STATUS_FRAME_OVERFLOW);
}

// 4. a warp per accepted frame: AcceptData record, held shards into the store, AcceptReply cell
__global__ void __launch_bounds__(kAccThreads) acceptor_copy_kernel(const __grid_constant__ AccArgs A) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = (static_cast<uint64_t>(blockIdx.x) * kAccThreads + threadIdx.x) >> 5;
    const uint64_t nwarps = (static_cast<uint64_t>(gridDim.x) * kAccThreads) >> 5;
    for (uint64_t i = warp; i < A.n; i += nwarps) {
        if (A.verdict[i] != SS_ACCEPT_VERDICT_ACCEPTED) continue;
        const FrameHdr h = A.hdr[i];
        const uint8_t *fr = A.buf + A.frame_off[i];
        // WalEntry::AcceptData: length, wal_variant, then the Accept body from `slot` on as it came
        uint8_t *rec = A.wal + A.wal_off[i];
        const uint32_t wvl = static_cast<uint32_t>(wv_len(A.wal_variant));
        const uint64_t tail = h.end - h.slot_at;
        if (lane == 0u) {
            put_be64(rec, wvl + tail);
            wv_put(rec + 8, A.wal_variant);
        }
        warp_copy_unaligned(rec + 8u + wvl, fr + h.slot_at, tail, lane);
        // held shards in index order, each in a SS_CW_SLOT_PITCH(L) slot, zero up to round_up(L, 16)
        warp_fill_shards(A.store + A.store_off[i], fr + h.tags_at, A.T, h.held, h.held, h.L, lane);
        // AcceptReply of the instance as the whole call left it
        if (lane == 0u) {
            const uint32_t g = A.frame_group[i];
            const uint64_t at_s = static_cast<uint64_t>(g) * 64u + (h.slot & 63u);
            uint8_t *cell = A.replies + i * 48u;
            uint32_t m = 8u;
            m += wv_put(cell + m, 0u);                                   // PeerMessage::Msg
            m += wv_put(cell + m, A.reply_variant);
            m += wv_put(cell + m, h.slot);
            m += wv_put(cell + m, A.inst_bal[at_s]);
            if (A.crossword) {                                           // size, reply_ts: None
                const uint64_t size = static_cast<uint64_t>(__popc(A.assignment[at_s])) * (static_cast<uint64_t>(A.data_len[at_s]) / A.d + 1u);
                m += wv_put(cell + m, size);
                cell[m++] = 0u;
            }
            put_be64(cell, m - 8u);
            A.reply_len[i] = m;
            A.reply_dst[i] = A.source[at_s];
        }
    }
}

// retire window prefixes: k = clamp(upto - base, 0, 64) positions leave Preparing, Accepting and Committed, the base
// moves on
__global__ void __launch_bounds__(kAccThreads)
acceptor_advance_kernel(const uint64_t *__restrict__ upto, uint64_t G, uint64_t *__restrict__ window_base, uint64_t *__restrict__ accepting,
                        uint64_t *__restrict__ committed, uint64_t *__restrict__ preparing) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kAccThreads;
    for (uint64_t g = static_cast<uint64_t>(blockIdx.x) * kAccThreads + threadIdx.x; g < G; g += stride) {
        const uint64_t base = window_base[g], u = upto[g];
        const uint64_t k = u <= base ? 0ull : (u - base < 64u ? u - base : 64ull);
        if (k == 0ull) continue;
        const uint64_t keep = ring_keep_after(k, base);
        accepting[g] &= keep;
        committed[g] &= keep;
        preparing[g] &= keep;
        window_base[g] = base + k;
    }
}

// ---- commit (heartbeat) -----------------------------------------------------------------------------------------
struct HbArgs {
    const uint32_t *group;
    const uint8_t *peer;
    const uint64_t *ballot, *hb_commit_bar, *hb_exec_bar;
    uint64_t n, G;
    uint32_t me;
    const uint64_t *window_base, *inst_bal, *commit_bar, *exec_bar;
    uint64_t *bal_max_seen, *accepting, *committed, *newly;
    uint32_t *key_in, *idx_in;
    const uint32_t *key, *idx;      // sorted
};

__global__ void __launch_bounds__(kAccThreads) heartbeat_keys_kernel(const __grid_constant__ HbArgs A) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kAccThreads;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kAccThreads + threadIdx.x; i < A.n; i += stride) {
        const uint32_t grp = A.group[i];
        A.key_in[i] = grp < A.G ? grp : static_cast<uint32_t>(A.G);
        A.idx_in[i] = static_cast<uint32_t>(i);
    }
}

// a thread per group segment, records in record order: heard_heartbeat's check_leader, its two filters and its commit
// walk over [max(commit_bar, window_base), min(hb commit_bar, window_base + 64)).  commit_bar does not move here (only
// execution moves it), so every record of the call walks from the same start.
__global__ void __launch_bounds__(kAccThreads) heartbeat_walk_kernel(const __grid_constant__ HbArgs A) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kAccThreads;
    for (uint64_t t = static_cast<uint64_t>(blockIdx.x) * kAccThreads + threadIdx.x; t < A.n; t += stride) {
        if (t != 0u && A.key[t] == A.key[t - 1]) continue;
        const uint32_t g = A.key[t];
        if (g >= A.G) continue;
        const uint64_t base = A.window_base[g], cb = A.commit_bar[g], eb = A.exec_bar[g];
        const uint64_t start = cb > base ? cb : base, wend = base + 64u;
        const uint64_t *ib = A.inst_bal + static_cast<uint64_t>(g) * 64u;
        uint64_t bmax = A.bal_max_seen[g], acc = A.accepting[g], com = A.committed[g], nw = 0ull;
        for (uint64_t k = t; k < A.n && A.key[k] == g; ++k) {
            const uint32_t i = A.idx[k];
            const uint64_t bal = A.ballot[i];
            if (A.peer[i] != A.me && bal > bmax) bmax = bal;           // check_leader
            if (bal < bmax || A.hb_exec_bar[i] < eb) continue;          // outdated heartbeat; exec_bar behind ours
            const uint64_t hcb = A.hb_commit_bar[i], stop = hcb < wend ? hcb : wend;
            for (uint64_t s = start; s < stop; ++s) {
                const uint64_t bit = 1ull << (s & 63u);
                if (ib[s & 63u] < bal || !((acc | com) & bit)) break;   // inst.bal < ballot, status < Accepting
                if (com & bit) continue;
                com |= bit;                                            // Status::Committed, a CommitSlot record
                acc &= ~bit;
                nw |= bit;
            }
        }
        A.bal_max_seen[g] = bmax;
        A.accepting[g] = acc;
        A.committed[g] = com;
        if (A.newly != nullptr) A.newly[g] = ring_to_window(nw, static_cast<uint32_t>(base & 63u));
    }
}

// ---- execute -----------------------------------------------------------------------------------------------------
// handle_logged_commit_slot's walk (exec_walk.cuh) over the 64-slot window, from max(commit_bar, window_base): stop past
// the window, at an instance not committed, or at fewer than d shards (postponed); stop at a null codeword, which
// get_data and reconstruct_data both refuse (rscoding.rs:495-497, 581-583).  A held shard of rank k is at shard_addr +
// k * pitch, the store slots.
struct AccLog {
    uint32_t d;
    const uint64_t *window_base, *committed, *shard_addr;
    const uint32_t *held, *data_len;
    uint64_t *commit_bar;

    struct Walk { uint64_t s, base, com; };
    static constexpr bool kTables = true, kByIndex = false;

    __device__ __forceinline__ bool live(uint64_t) const { return true; }
    __device__ __forceinline__ Walk start(uint64_t g) const {
        const uint64_t base = window_base[g], com = committed[g], cb = commit_bar[g];
        return {cb > base ? cb : base, base, com};
    }
    __device__ __forceinline__ uint32_t next(const Walk &w, uint64_t g, uint64_t s, uint32_t *dlen) const {
        if (s - w.base >= 64u || !((w.com >> (s & 63u)) & 1u)) return kExecStop;
        const uint64_t at = g * 64u + (s & 63u);
        if (static_cast<uint32_t>(__popc(held[at])) < d) return kExecStop;
        *dlen = data_len[at];
        return *dlen == 0u ? kExecNull : kExecRun;
    }
    __device__ __forceinline__ void finish(uint64_t g, uint64_t s) const { commit_bar[g] = s; }
    __device__ __forceinline__ ExecSrc source(uint64_t g, uint64_t s, uint32_t dlen) const {
        const uint64_t at = g * 64u + (s & 63u);
        return {held[at], reinterpret_cast<const uint8_t *>(shard_addr[at]), SS_CW_SLOT_PITCH((dlen + d - 1u) / d)};
    }
};

// ---- reconstruct reads ---------------------------------------------------------------------------------------------
struct RecArgs {
    const uint8_t *buf;
    uint64_t buf_len;
    const uint64_t *frame_off;
    const uint32_t *frame_group;
    uint64_t n, G;
    uint32_t d, T, variant, reply_variant, crossword;
    // state
    const uint64_t *window_base, *inst_bal, *accepting, *committed, *exec_bar;
    const uint32_t *data_len;
    uint64_t *shard_addr;
    uint32_t *held;
    // serve
    uint8_t *out;
    uint64_t out_cap;
    uint64_t *reply_off, *reply_len;
    // absorb
    ReplyHdr *rhdr;
    uint32_t *key_in, *idx_in;
    const uint32_t *key, *idx;      // sorted
    uint64_t *grp_bytes;            // [G] region bytes per group, then their exclusive scan
    uint8_t *store;
    uint64_t store_cap;
    uint32_t *absorbed;
    uint32_t *verdict;
    uint32_t *status;
};

// Per-warp scratch of the walks below.  Every lane of a warp runs the same walk over the same frame bytes (the loads
// broadcast), so the warp stays converged and copies the shards of an entry together; lane 0 writes the arrays and
// __syncwarp publishes them.
struct RecWarp {
    uint32_t mask[64];              // serve: the defining entry's shards; absorb: the instance's mask as the walk goes
    uint32_t last[64];              // occurrence index of the defining (last) entry of each ring position
    uint32_t fin[64];               // absorb: the instance's final mask
    uint64_t off[64];               // serve: entry offsets in the reply; absorb: new region offsets (~0: unchanged)
};

// the 8-byte length, PeerMessage::Msg and the PeerMsg variant of frame i; kPending with b / len / n past the entry count
// (cnt) when it is `variant`
__device__ __forceinline__ uint32_t rec_head(const RecArgs &A, uint64_t i, const uint8_t *&b, uint64_t &len, uint64_t &n, uint64_t &cnt) {
    if (A.frame_group[i] >= A.G) return SS_FRAME_KIND_MALFORMED;
    return msg_head_count(A.buf, A.buf_len, A.frame_off[i], A.variant, kMaxFrameBody, b, len, n, cnt);
}

__device__ __forceinline__ uint64_t ring_slot(uint64_t base, uint32_t pos) { return base + ((pos - base) & 63u); }

// Reconstruct{slots} (RSPaxos) or Reconstruct{slots_excl} (Crossword) of frame i, walked as handle_msg_reconstruct
// walks it (rspaxos/messages.rs:468-516, crossword/messages.rs:577-632).  Returns kPending when the frame is well formed
// and refused nothing, and *nz = the ring positions with an entry: W.mask the defining entry's shards, W.last its
// occurrence index (HashMap::insert keeps the last value).  Warp-uniform.
__device__ uint32_t serve_walk(const RecArgs &A, uint64_t i, RecWarp &W, uint32_t lane, uint64_t *nz) {
    *nz = 0ull;
    const uint8_t *b;
    uint64_t len, n, cnt;
    const uint32_t kind = rec_head(A, i, b, len, n, cnt);
    if (kind != kPending) return kind;
    const uint32_t g = A.frame_group[i];
    const uint64_t base = A.window_base[g], live = A.accepting[g] | A.committed[g];
    const uint64_t T = A.T;
    uint32_t err = 0u;
    for (uint64_t e = 0; e < cnt; ++e) {
        uint64_t slot = 0;
        if (!wv_next(b, len, n, slot)) return SS_FRAME_KIND_MALFORMED;
        uint32_t sel = 0xffffffffu;
        bool range_bad = false;
        if (A.crossword) {
            // Bitmap::decode: size, then any number of u64 blocks, padded with zeros or cut to the size (bitmap.rs:32-40).
            // subset_copy walks subset.iter() (rscoding.rs:264-275), which stops at Bitmap::size() = size as u8
            // (bitmap.rs:103-105, 258-270), so only bits [0, size mod 256) take part.  flip() selects the ones the
            // exclusion leaves clear, and one at index >= T makes subset_copy fail: every bit of [T, size mod 256) must
            // be set.
            uint64_t sz = 0, nb = 0, blk = 0, lo = 0;
            if (!wv_next(b, len, n, sz) || !wv_next(b, len, n, nb)) return SS_FRAME_KIND_MALFORMED;
            const uint64_t walk = sz & 255u;
            for (uint64_t k = 0; k < nb; ++k) {
                if (!wv_next(b, len, n, blk)) return SS_FRAME_KIND_MALFORMED;
                if (k == 0u) lo = blk;
                const uint64_t b0 = 64u * k, from = T > b0 ? T : b0, to = walk < b0 + 64u ? walk : b0 + 64u;
                if (from < to) {
                    const uint64_t w = to - from, m = (w == 64u ? ~0ull : (1ull << w) - 1u) << (from - b0);
                    if ((blk & m) != m) range_bad = true;
                }
            }
            const uint64_t pad_from = T > 64u * nb ? T : 64u * nb;
            if (walk > pad_from) range_bad = true;                              // zero-padded blocks
            const uint64_t w = walk < T ? walk : T;
            sel = ~static_cast<uint32_t>(lo) & (w >= 32u ? 0xffffffffu : (1u << w) - 1u);
        }
        if (err != 0u || slot < base || slot - base >= 64u) continue;           // below start_slot; a padded null instance
        const uint32_t pos = static_cast<uint32_t>(slot & 63u);
        if (!((live >> pos) & 1u)) continue;                                    // status < Accepting
        const uint64_t at = static_cast<uint64_t>(g) * 64u + pos;
        if (A.crossword) {
            if (A.data_len[at] == 0u) { err = SS_RECON_VERDICT_NULL_CODEWORD; continue; }
            if (range_bad) { err = SS_RECON_VERDICT_SHARD_RANGE; continue; }
        }
        const uint32_t m = A.held[at] & sel;                                    // RSPaxos: reqs_cw.clone()
        if (m == 0u) continue;
        if (lane == 0u) { W.mask[pos] = m; W.last[pos] = static_cast<uint32_t>(e); }
        *nz |= 1ull << pos;
    }
    __syncwarp();
    if (n != len) return SS_FRAME_KIND_MALFORMED;
    return err != 0u ? err : kPending;
}

// the codeword of cw_bytes at e (any alignment): lane 0 writes the header, the Option tags and the shard lengths; the
// warp copies shard j of m from its padded slot in the instance's store region at src, rank popcount(held & below j).
// Not inlined: inlined into serve_copy_kernel it made that kernel spill; the call costs one per entry.  It keeps its own
// loop rather than warp_put_cw's, whose lane-0 writes between the shard copies made ss_acceptor_reconstruct_serve 3-5 %
// slower on an H100.
__device__ __noinline__ void warp_put_codeword(uint8_t *e, uint32_t d, uint32_t T, uint64_t dl, uint32_t m, uint32_t held, const uint8_t *src,
                                               uint32_t lane) {
    const uint64_t L = (dl + d - 1u) / d, pitch = SS_CW_SLOT_PITCH(L);
    const uint64_t h0 = 2u + wv_len(dl) + wv_len(L) + wv_len(T), some = 1u + wv_len(L);
    if (lane == 0u) {
        uint64_t q = 0;
        e[q++] = static_cast<uint8_t>(d);
        e[q++] = static_cast<uint8_t>(T - d);
        q += wv_put(e + q, dl);
        q += wv_put(e + q, L);
        q += wv_put(e + q, T);
        for (uint32_t j = 0; j < T; ++j) {
            if ((m >> j) & 1u) {
                e[q] = 1u;
                wv_put(e + q + 1u, L);
                q += some + L;
            } else {
                e[q++] = 0u;
            }
        }
        e[q] = 0u;                                                           // data_copy: None
    }
    for (uint32_t rest_j = m; rest_j != 0u; rest_j &= rest_j - 1u) {
        const uint32_t j = static_cast<uint32_t>(__ffs(rest_j)) - 1u;
        const uint32_t below = (1u << j) - 1u;
        const uint64_t sel_before = static_cast<uint64_t>(__popc(m & below));
        const uint64_t at_j = h0 + (j - sel_before) + sel_before * (some + L) + some;
        warp_copy_unaligned(e + at_j, src + static_cast<uint64_t>(__popc(held & below)) * pitch, L, lane);
    }
}

// bytes of one (slot, (inst.bal, RSCodeword)) map entry carrying the shards m of instance `at`
__device__ __forceinline__ uint64_t serve_entry_bytes(const RecArgs &A, uint64_t slot, uint64_t at, uint32_t m) {
    return wv_len(slot) + wv_len(A.inst_bal[at]) + cw_bytes(A.data_len[at], A.d, A.T, __popc(m));
}

__device__ __forceinline__ uint64_t warp_sum(uint64_t x) {
    for (int s = 16; s > 0; s >>= 1) x += __shfl_xor_sync(0xffffffffu, x, s);
    return x;
}

// 1. a warp per frame: verdict, reply bytes (8-byte length, Msg, variant, map length, entries)
__global__ void __launch_bounds__(kAccThreads) serve_count_kernel(const __grid_constant__ RecArgs A) {
    __shared__ RecWarp Ws[kExecWarps];
    const uint32_t lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
    RecWarp &W = Ws[w];
    const uint64_t nwarps = static_cast<uint64_t>(gridDim.x) * kExecWarps;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kExecWarps + w; i < A.n; i += nwarps) {
        uint64_t nz;
        uint32_t kind = serve_walk(A, i, W, lane, &nz);
        uint64_t bytes = 0;
        if (kind == kPending) {
            kind = SS_ACCEPT_VERDICT_ACCEPTED;
            if (nz != 0u) {
                const uint32_t g = A.frame_group[i];
                const uint64_t base = A.window_base[g];
                for (uint32_t p = lane; p < 64u; p += 32u)
                    if ((nz >> p) & 1u) bytes += serve_entry_bytes(A, ring_slot(base, p), static_cast<uint64_t>(g) * 64u + p, W.mask[p]);
                bytes = warp_sum(bytes) + 9u + wv_len(A.reply_variant) + wv_len(__popcll(nz));
            }
        }
        if (lane == 0u) {
            A.verdict[i] = kind;
            A.reply_len[i] = bytes;
            A.reply_off[i] = round16(bytes);
        }
        __syncwarp();                   // the next frame's walk overwrites W
    }
}

// 2. a warp per frame with a reply: capacity, then the ReconstructReply, entries in the order of their defining
//    occurrences; every shard is copied from its 16-byte aligned store slot
__global__ void __launch_bounds__(kAccThreads) serve_copy_kernel(const __grid_constant__ RecArgs A) {
    __shared__ RecWarp Ws[kExecWarps];
    const uint32_t lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
    RecWarp &W = Ws[w];
    bool full = false;
    const uint64_t nwarps = static_cast<uint64_t>(gridDim.x) * kExecWarps;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kExecWarps + w; i < A.n; i += nwarps) {
        const uint64_t len = A.reply_len[i], off = A.reply_off[i];
        if (A.verdict[i] != SS_ACCEPT_VERDICT_ACCEPTED || len == 0u || off > A.out_cap || round16(len) > A.out_cap - off) {
            if (lane == 0u) {
                if (len != 0u) {
                    A.verdict[i] = SS_RECON_VERDICT_OUT_FULL;
                    A.reply_len[i] = 0u;
                }
                A.reply_off[i] = ~0ull;
            }
            full |= len != 0u;
            continue;
        }
        uint64_t nz;
        serve_walk(A, i, W, lane, &nz);
        const uint32_t g = A.frame_group[i];
        const uint64_t base = A.window_base[g];
        const uint64_t cnt = static_cast<uint64_t>(__popcll(nz)), head = 9u + wv_len(A.reply_variant) + wv_len(cnt);
        uint64_t mine[2] = {0u, 0u};
        for (uint32_t r = 0; r < 2u; ++r) {
            const uint32_t p = lane + 32u * r;
            if ((nz >> p) & 1u) mine[r] = serve_entry_bytes(A, ring_slot(base, p), static_cast<uint64_t>(g) * 64u + p, W.mask[p]);
        }
        if (lane == 0u) for (uint32_t p = 0; p < 64u; ++p) W.off[p] = 0u;
        __syncwarp();
        for (uint32_t r = 0; r < 2u; ++r) if (mine[r]) W.off[lane + 32u * r] = mine[r];
        __syncwarp();
        for (uint32_t r = 0; r < 2u; ++r) {                                      // offsets: sizes of the earlier entries
            const uint32_t p = lane + 32u * r;
            if (!((nz >> p) & 1u)) continue;
            uint64_t o = head;
            for (uint32_t q = 0; q < 64u; ++q)
                if (((nz >> q) & 1u) && W.last[q] < W.last[p]) o += W.off[q];
            mine[r] = o;
        }
        __syncwarp();
        for (uint32_t r = 0; r < 2u; ++r) if ((nz >> (lane + 32u * r)) & 1u) W.off[lane + 32u * r] = mine[r];
        __syncwarp();
        uint8_t *dst = A.out + off;
        if (lane == 0u) {
            put_be64(dst, len - 8u);
            uint32_t m = 8u;
            m += wv_put(dst + m, 0u);                                            // PeerMessage::Msg
            m += wv_put(dst + m, A.reply_variant);
            wv_put(dst + m, cnt);
        }
        for (uint64_t rest = nz; rest != 0u; rest &= rest - 1u) {
            const uint32_t p = static_cast<uint32_t>(__ffsll(static_cast<long long>(rest))) - 1u;
            const uint64_t at = static_cast<uint64_t>(g) * 64u + p, slot = ring_slot(base, p);
            const uint64_t bal = A.inst_bal[at];
            uint8_t *e = dst + W.off[p];
            if (lane == 0u) wv_put(e + wv_put(e, slot), bal);                 // (slot, (bal, RSCodeword))
            warp_put_codeword(e + wv_len(slot) + wv_len(bal), A.d, A.T, A.data_len[at], W.mask[p], A.held[at],
                              reinterpret_cast<const uint8_t *>(A.shard_addr[at]), lane);
        }
        __syncwarp();
    }
    if (full && lane == 0u) atomicOr(A.status, SS_DEV_STATUS_FRAME_OVERFLOW);
}

// one (slot, (ballot, RSCodeword)) of a ReconstructReply at b + n: the codeword must carry the acceptor's code,
// shard_len = ceil(data_len / d), T shard Options of shard_len bytes each, and data_copy None or Some(data_len bytes)
struct RecEntry {
    uint64_t slot, bal, tags_at;
    uint32_t dlen, L, mask;
};
__device__ __forceinline__ bool absorb_entry(const RecArgs &A, const uint8_t *b, uint64_t len, uint64_t &n, RecEntry &E) {
    uint64_t dl = 0, sl = 0;
    if (!wv_next(b, len, n, E.slot) || !wv_next(b, len, n, E.bal) || !cw_parse<true>(b, len, n, A.d, A.T, dl, sl, E.tags_at, E.mask))
        return false;
    E.dlen = static_cast<uint32_t>(dl);
    E.L = static_cast<uint32_t>(sl);
    return true;
}

// 1. a thread per frame: decode the whole ReconstructReply, note a slot repeated in the window, sort keys
__global__ void __launch_bounds__(kAccThreads) absorb_decode_kernel(const __grid_constant__ RecArgs A) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kAccThreads;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kAccThreads + threadIdx.x; i < A.n; i += stride) {
        const uint8_t *b = nullptr;
        uint64_t len = 0, n = 0, cnt = 0;
        uint32_t kind = rec_head(A, i, b, len, n, cnt);
        ReplyHdr h{};
        if (kind == kPending) {
            const uint64_t base = A.window_base[A.frame_group[i]];
            h.entries_at = n;
            h.count = cnt;
            uint64_t seen = 0;
            RecEntry E;
            kind = SS_ACCEPT_VERDICT_ACCEPTED;
            for (uint64_t e = 0; e < cnt; ++e) {
                if (!absorb_entry(A, b, len, n, E)) { kind = SS_FRAME_KIND_MALFORMED; break; }
                if (E.slot < base || E.slot - base >= 64u) continue;
                const uint64_t bit = 1ull << (E.slot & 63u);
                h.repeated |= (seen & bit) ? 1u : 0u;
                seen |= bit;
            }
            if (n != len) kind = SS_FRAME_KIND_MALFORMED;
            h.body_len = len;
        }
        h.kind = kind;
        A.rhdr[i] = h;
        A.verdict[i] = kind;
        A.absorbed[i] = 0u;
        A.key_in[i] = kind == SS_ACCEPT_VERDICT_ACCEPTED ? A.frame_group[i] : static_cast<uint32_t>(A.G);
        A.idx_in[i] = static_cast<uint32_t>(i);
    }
}

// The entries of group g's frames (sorted positions [t, e)) in frame order, then wire order, through
// handle_msg_reconstruct_reply's filters (rspaxos/messages.rs:519-594, crossword/messages.rs:635-722); a slot repeated
// inside one frame counts once, with its last value (a HashMap decode keeps the last insert).  W.mask starts at the held
// masks; an entry that passes adds the shards the instance does not hold yet (absorb_other, rscoding.rs:337-343), and
// on_entry(b, E, pos, contribution) runs for each entry that adds any; on_frame(i) runs after each frame.  Warp-uniform.
template <typename FE, typename FF>
__device__ void absorb_replay(const RecArgs &A, uint64_t t, uint64_t e, uint32_t g, RecWarp &W, uint32_t lane, FE &&on_entry,
                              FF &&on_frame) {
    const uint64_t base = A.window_base[g], live = A.accepting[g] | A.committed[g], eb = A.exec_bar[g];
    const uint64_t row = static_cast<uint64_t>(g) * 64u;
    W.mask[lane] = A.held[row + lane];
    W.mask[lane + 32u] = A.held[row + lane + 32u];
    __syncwarp();
    for (uint64_t k = t; k < e; ++k) {
        const uint32_t i = A.idx[k];
        const ReplyHdr h = A.rhdr[i];
        const uint8_t *b = A.buf + A.frame_off[i] + 8u;
        RecEntry E;
        uint64_t n = h.entries_at;
        if (h.repeated) {                                                             // a repeated slot: find its last value
            __syncwarp();
            for (uint64_t q = 0; q < h.count; ++q) {
                absorb_entry(A, b, h.body_len, n, E);
                if (E.slot >= base && E.slot - base < 64u && lane == 0u) W.last[E.slot & 63u] = static_cast<uint32_t>(q);
            }
            __syncwarp();
            n = h.entries_at;
        }
        for (uint64_t q = 0; q < h.count; ++q) {
            absorb_entry(A, b, h.body_len, n, E);
            if (E.slot < base || E.slot - base >= 64u) continue;                 // outdated; beyond the window
            const uint32_t pos = static_cast<uint32_t>(E.slot & 63u);
            if (h.repeated && W.last[pos] != q) continue;
            const uint64_t at = row + pos;
            if (!((live >> pos) & 1u) || E.slot < eb || E.bal < A.inst_bal[at]) continue;   // status, Executed, ballot
            const uint32_t dl = A.data_len[at];
            if (dl == 0u || E.dlen != dl) continue;                              // null instance; absorb_other's checks
            const uint32_t cur = W.mask[pos], add = E.mask & ~cur;
            if (add == 0u) continue;
            __syncwarp();
            if (lane == 0u) W.mask[pos] = cur | add;
            __syncwarp();
            on_entry(b, E, pos, add);
        }
        on_frame(i);
    }
}

__device__ __forceinline__ uint64_t segment_end(const RecArgs &A, uint64_t t) {
    uint64_t e = t + 1u;
    while (e < A.n && A.key[e] == A.key[t]) ++e;
    return e;
}

// 2. a warp per group segment: the final masks, and the bytes of the regions of the instances that grow
__global__ void __launch_bounds__(kAccThreads) absorb_plan_kernel(const __grid_constant__ RecArgs A) {
    __shared__ RecWarp Ws[kExecWarps];
    const uint32_t lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
    RecWarp &W = Ws[w];
    const uint64_t nwarps = static_cast<uint64_t>(gridDim.x) * kExecWarps;
    for (uint64_t t = static_cast<uint64_t>(blockIdx.x) * kExecWarps + w; t < A.n; t += nwarps) {
        if (t != 0u && A.key[t] == A.key[t - 1]) continue;
        const uint32_t g = A.key[t];
        if (g >= A.G) continue;
        absorb_replay(A, t, segment_end(A, t), g, W, lane, [](const uint8_t *, const RecEntry &, uint32_t, uint32_t) {}, [](uint32_t) {});
        uint64_t bytes = 0;
        for (uint32_t p = lane; p < 64u; p += 32u) {
            const uint64_t at = static_cast<uint64_t>(g) * 64u + p;
            if (W.mask[p] != A.held[at]) bytes += static_cast<uint64_t>(__popc(W.mask[p])) * SS_CW_SLOT_PITCH((A.data_len[at] + A.d - 1u) / A.d);
        }
        bytes = warp_sum(bytes);
        if (lane == 0u) A.grp_bytes[g] = bytes;
        __syncwarp();
    }
}

// 3. a warp per group segment: regions in slot order from the group's scanned offset, capacity, the old shards and
//    then the new ones into the new regions, held / shard_addr, per-frame counts and verdicts
__global__ void __launch_bounds__(kAccThreads) absorb_copy_kernel(const __grid_constant__ RecArgs A) {
    __shared__ RecWarp Ws[kExecWarps];
    const uint32_t lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
    RecWarp &W = Ws[w];
    bool full = false;
    const uint64_t nwarps = static_cast<uint64_t>(gridDim.x) * kExecWarps;
    for (uint64_t t = static_cast<uint64_t>(blockIdx.x) * kExecWarps + w; t < A.n; t += nwarps) {
        if (t != 0u && A.key[t] == A.key[t - 1]) continue;
        const uint32_t g = A.key[t];
        if (g >= A.G) continue;
        const uint64_t e = segment_end(A, t), row = static_cast<uint64_t>(g) * 64u, base = A.window_base[g];
        absorb_replay(A, t, e, g, W, lane, [](const uint8_t *, const RecEntry &, uint32_t, uint32_t) {}, [](uint32_t) {});
        W.fin[lane] = W.mask[lane];
        W.fin[lane + 32u] = W.mask[lane + 32u];
        __syncwarp();
        // region offsets in window order: lane r takes positions base + r and base + 32 + r
        uint64_t sz[2], pre[2];
        for (uint32_t h = 0; h < 2u; ++h) {
            const uint32_t p = static_cast<uint32_t>((base + 32u * h + lane) & 63u);
            const uint32_t old = A.held[row + p], nw = W.fin[p];
            sz[h] = nw != old ? static_cast<uint64_t>(__popc(nw)) * SS_CW_SLOT_PITCH((A.data_len[row + p] + A.d - 1u) / A.d) : 0u;
            uint64_t x = sz[h];
            for (int s = 1; s < 32; s <<= 1) {
                const uint64_t y = __shfl_up_sync(0xffffffffu, x, s);
                if (lane >= static_cast<uint32_t>(s)) x += y;
            }
            pre[h] = x - sz[h];
        }
        pre[1] += __shfl_sync(0xffffffffu, pre[0] + sz[0], 31);
        const uint64_t goff = A.grp_bytes[g];
        for (uint32_t h = 0; h < 2u; ++h) {
            const uint32_t p = static_cast<uint32_t>((base + 32u * h + lane) & 63u);
            const uint32_t old = A.held[row + p];
            const uint64_t o = goff + pre[h];
            const bool grows = W.fin[p] != old, placed = o <= A.store_cap && sz[h] <= A.store_cap - o;
            W.off[p] = grows && placed ? o : ~0ull;
            full |= grows && !placed;
        }
        __syncwarp();
        // the shards the instance held, into their ranks of the new mask
        for (uint32_t p = 0; p < 64u; ++p) {
            if (W.off[p] == ~0ull) continue;
            const uint32_t old = A.held[row + p], nw = W.fin[p];
            const uint64_t L = (A.data_len[row + p] + A.d - 1u) / A.d, pitch = SS_CW_SLOT_PITCH(L);
            const uint8_t *src = reinterpret_cast<const uint8_t *>(A.shard_addr[row + p]);
            uint8_t *dst = A.store + W.off[p];
            uint32_t k = 0;
            for (uint32_t rest = old; rest != 0u; rest &= rest - 1u, ++k) {
                const uint32_t j = static_cast<uint32_t>(__ffs(rest)) - 1u;
                warp_fill_slot(dst + static_cast<uint64_t>(__popc(nw & ((1u << j) - 1u))) * pitch, src + k * pitch, L, lane);
            }
        }
        // the new shards, each from the first entry that carries it
        uint32_t taken = 0u;
        bool frame_full = false;
        absorb_replay(
            A, t, e, g, W, lane,
            [&](const uint8_t *b, const RecEntry &E, uint32_t pos, uint32_t add) {
                if (W.off[pos] == ~0ull) { frame_full = true; return; }
                warp_fill_shards(A.store + W.off[pos], b + E.tags_at, A.T, E.mask, add, E.L, lane, W.fin[pos]);
                ++taken;
            },
            [&](uint32_t i) {
                if (lane == 0u) {
                    A.absorbed[i] = taken;
                    if (frame_full) A.verdict[i] = SS_ACCEPT_VERDICT_STORE_FULL;
                }
                taken = 0u;
                frame_full = false;
            });
        for (uint32_t p = lane; p < 64u; p += 32u) {
            if (W.off[p] == ~0ull) continue;
            A.held[row + p] = W.fin[p];
            A.shard_addr[row + p] = reinterpret_cast<uint64_t>(A.store + W.off[p]);
        }
        __syncwarp();
    }
    if (full) atomicOr(A.status, SS_DEV_STATUS_STORE_FULL);
}

// ---- prepare -----------------------------------------------------------------------------------------------------
struct PrepArgs {
    const uint8_t *buf;
    uint64_t buf_len;
    const uint64_t *frame_off;
    const uint32_t *frame_group;
    const uint8_t *frame_peer;
    uint64_t n, G;
    uint32_t me, variant, wal_variant;
    // state
    const uint64_t *window_base;
    uint64_t *bal_max_seen, *inst_bal, *accepting, *committed, *preparing, *voted_bal, *prep_trigger;
    uint32_t *voted_mask;
    uint8_t *source, *prep_span;
    // scratch
    PrepHdr *hdr;
    uint32_t *key_in, *idx_in;
    const uint32_t *key, *idx;      // sorted
    uint64_t *cnt;                  // [n] records per frame, then their exclusive scan (the first record's number)
    uint64_t *totals;               // [2]: [0] the scan's total, [1] its WAL bytes
    uint64_t cap;                   // min(rec_capacity, wal_capacity / 32)
    // outputs
    uint8_t *wal;
    uint32_t *rec_group;
    uint64_t *rec_slot;
    uint32_t *rec_frame;
    uint32_t *verdict;
    uint32_t *status;
};

// PeerMessage::Msg{Prepare{trigger_slot, ballot}}, then the window filters; a Prepare from `me` is malformed
// (check_leader debug-asserts peer != me)
__device__ __forceinline__ PrepHdr decode_prepare(const PrepArgs &A, uint64_t i) {
    PrepHdr h{};
    h.kind = SS_FRAME_KIND_MALFORMED;
    const uint32_t grp = A.frame_group[i];
    const uint64_t off = A.frame_off[i];
    if (grp >= A.G) return h;
    const uint8_t *b;
    uint64_t len, n, trig = 0, bal = 0;
    if (!msg_head(A.buf, A.buf_len, off, A.variant, kMaxFrameBody, true, b, len, n, h.kind)) return h;
    if (!wv_next(b, len, n, trig) || !wv_next(b, len, n, bal)) return h;
    if (n != len || A.frame_peer[i] == A.me) return h;
    h.trigger = trig;
    h.ballot = bal;
    const uint64_t base = A.window_base[grp];
    h.kind = trig < base ? SS_ACCEPT_VERDICT_STALE_SLOT : trig - base >= 64u ? SS_ACCEPT_VERDICT_BEYOND_WINDOW : kPending;
    return h;
}

// 1. a thread per frame
__global__ void __launch_bounds__(kAccThreads) prepare_header_kernel(const __grid_constant__ PrepArgs A) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kAccThreads;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kAccThreads + threadIdx.x; i < A.n; i += stride) {
        A.hdr[i] = decode_prepare(A, i);
        A.cnt[i] = 0u;
        const uint32_t grp = A.frame_group[i];
        A.key_in[i] = grp < A.G ? grp : static_cast<uint32_t>(A.G);
        A.idx_in[i] = static_cast<uint32_t>(i);
    }
}

// window positions [lo, hi] (0 <= lo <= hi < 64) as a ring word of a window at base
__device__ __forceinline__ uint64_t window_range_ring(uint64_t lo, uint64_t hi, uint64_t base) {
    const uint64_t w = hi - lo + 1u;
    return window_to_ring((w == 64u ? ~0ull : (1ull << w) - 1u) << lo, static_cast<uint32_t>(base & 63u));
}

// 2. a thread per group segment, frames in frame order: check_leader, then endprep_slot = max(the last window position
//    that is not null, trigger_slot) over the state as the earlier frames of the call left it; [trigger, endprep]
//    becomes Preparing.  Only the per-frame verdict, endprep and record count are written.
__global__ void __launch_bounds__(kAccThreads) prepare_walk_kernel(const __grid_constant__ PrepArgs A) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kAccThreads;
    for (uint64_t t = static_cast<uint64_t>(blockIdx.x) * kAccThreads + threadIdx.x; t < A.n; t += stride) {
        if (t != 0u && A.key[t] == A.key[t - 1]) continue;
        const uint32_t g = A.key[t];
        if (g >= A.G) continue;
        const uint64_t base = A.window_base[g];
        const uint32_t r = static_cast<uint32_t>(base & 63u);
        uint64_t bmax = A.bal_max_seen[g], prep = A.preparing[g], acc = A.accepting[g], com = A.committed[g];
        for (uint64_t k = t; k < A.n && A.key[k] == g; ++k) {
            const uint32_t i = A.idx[k];
            if (A.hdr[i].kind != kPending) continue;
            const uint64_t bal = A.hdr[i].ballot, tw = A.hdr[i].trigger - base;
            if (bal < bmax) {
                A.hdr[i].kind = SS_ACCEPT_VERDICT_STALE_BALLOT;
                continue;
            }
            bmax = bal;
            const uint64_t live = ring_to_window(prep | acc | com, r);       // rposition(status > Null)
            const uint64_t hi = live != 0u ? 63u - static_cast<uint64_t>(__clzll(static_cast<long long>(live))) : 0u;
            const uint64_t ew = hi > tw ? hi : tw;
            const uint64_t m = window_range_ring(tw, ew, base);
            prep |= m;
            acc &= ~m;
            com &= ~m;
            A.hdr[i].kind = SS_ACCEPT_VERDICT_ACCEPTED;                       // subject to capacity
            A.hdr[i].endprep = base + ew;
            A.cnt[i] = ew - tw + 1u;
        }
    }
}

// 3. a thread per group segment, last frame first.  cnt holds the scanned record numbers, so frame j's records end at
//    cnt[j + 1] (the total for the last frame), monotone in frame order: the first frame whose records end past the
//    capacity is found by bisection, and it and every later frame whose verdict came from the replay get WAL_FULL.
//    The applied frames are then a prefix in frame order, so each group's applied frames are a prefix of its frames and
//    the ranges the walk computed for them stay exact.
__global__ void __launch_bounds__(kAccThreads) prepare_apply_kernel(const __grid_constant__ PrepArgs A) {
    const uint64_t total = A.totals[0];
    if (blockIdx.x == 0u && threadIdx.x == 0u) A.totals[1] = total * 32u;
    uint64_t cut = A.n;
    if (total > A.cap) {
        uint64_t lo = 0, hi = A.n;
        while (lo < hi) {
            const uint64_t mid = (lo + hi) >> 1, end = mid + 1u < A.n ? A.cnt[mid + 1u] : total;
            if (end > A.cap) hi = mid; else lo = mid + 1u;
        }
        cut = lo;
    }
    bool full = false;
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kAccThreads;
    for (uint64_t t = static_cast<uint64_t>(blockIdx.x) * kAccThreads + threadIdx.x; t < A.n; t += stride) {
        if (t != 0u && A.key[t] == A.key[t - 1]) continue;
        const uint32_t g = A.key[t];
        const bool known = g < A.G;
        uint64_t e = t + 1u;
        while (e < A.n && A.key[e] == g) ++e;
        const uint64_t base = known ? A.window_base[g] : 0u;
        const uint64_t null0 = known ? ~(A.preparing[g] | A.accepting[g] | A.committed[g]) : 0u;
        uint64_t seen = 0u, mx = known ? A.bal_max_seen[g] : 0u;
        for (uint64_t k = e; k-- > t;) {
            const uint32_t i = A.idx[k];
            uint32_t kind = A.hdr[i].kind;
            if ((kind == SS_ACCEPT_VERDICT_ACCEPTED || kind == SS_ACCEPT_VERDICT_STALE_BALLOT) && i >= cut) {
                kind = SS_ACCEPT_VERDICT_WAL_FULL;
                full = true;
            }
            if (kind == SS_ACCEPT_VERDICT_ACCEPTED) {
                const PrepHdr h = A.hdr[i];
                mx = h.ballot > mx ? h.ballot : mx;
                const uint64_t m = window_range_ring(h.trigger - base, h.endprep - base, base), def = m & ~seen;
                seen |= m;
                A.hdr[i].define = def;
                A.hdr[i].fresh = def & null0;
            }
            A.verdict[i] = kind;
        }
        if (known) {
            A.preparing[g] |= seen;                                           // Status::Preparing, also over Committed
            A.accepting[g] &= ~seen;
            A.committed[g] &= ~seen;
            A.bal_max_seen[g] = mx;
        }
    }
    if (full) atomicOr(A.status, SS_DEV_STATUS_FRAME_OVERFLOW);
}

// 4. a warp per applied frame: its WalEntry::PrepareBal{slot, ballot} cells (8-byte big-endian length + bincode, zero to
//    32 bytes) and, at the positions it defines, inst.bal, replica_bk and -- for a position that was null -- voted None
__global__ void __launch_bounds__(kAccThreads) prepare_write_kernel(const __grid_constant__ PrepArgs A) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = (static_cast<uint64_t>(blockIdx.x) * kAccThreads + threadIdx.x) >> 5;
    const uint64_t nwarps = (static_cast<uint64_t>(gridDim.x) * kAccThreads) >> 5;
    for (uint64_t i = warp; i < A.n; i += nwarps) {
        if (A.verdict[i] != SS_ACCEPT_VERDICT_ACCEPTED) continue;
        const PrepHdr h = A.hdr[i];
        const uint32_t g = A.frame_group[i];
        const uint64_t first = A.cnt[i], count = h.endprep - h.trigger + 1u;
        for (uint64_t q = lane; q < count; q += 32u) {
            const uint64_t k = first + q, slot = h.trigger + q;
            put_prepare_bal_cell(A.wal + k * 32u, A.wal_variant, slot, h.ballot);
            A.rec_group[k] = g;
            A.rec_slot[k] = slot;
            A.rec_frame[k] = static_cast<uint32_t>(i);
        }
        for (uint32_t p = lane; p < 64u; p += 32u) {
            if (!((h.define >> p) & 1u)) continue;
            const uint64_t at = static_cast<uint64_t>(g) * 64u + p;
            A.inst_bal[at] = h.ballot;
            A.source[at] = A.frame_peer[i];
            A.prep_trigger[at] = h.trigger;
            A.prep_span[at] = static_cast<uint8_t>(h.endprep - h.trigger);
            if ((h.fresh >> p) & 1u) {                                        // a fresh null_instance(): voted (0, null)
                A.voted_bal[at] = 0u;
                A.voted_mask[at] = 0u;
            }
        }
    }
}

// ---- prepare replies ----------------------------------------------------------------------------------------------
struct PrepReplyArgs {
    const uint32_t *rec_group;
    const uint64_t *rec_slot;
    uint64_t n, G;
    uint32_t d, T, variant;
    const uint64_t *window_base, *preparing, *accepting, *committed, *inst_bal, *voted_bal, *prep_trigger, *shard_addr;
    const uint32_t *voted_mask, *held, *data_len;
    const uint8_t *source, *prep_span;
    uint8_t *out;
    uint64_t out_cap;
    uint64_t *reply_off, *reply_len;
    uint8_t *reply_dst;
    uint32_t *status;
};

// PrepareReply bytes of record k (0: no reply), *at its instance
__device__ __forceinline__ uint64_t prep_reply_bytes(const PrepReplyArgs &A, uint64_t k, uint64_t *at) {
    const uint32_t g = A.rec_group[k];
    if (g >= A.G) return 0u;
    const uint64_t s = A.rec_slot[k], base = A.window_base[g];
    if (s < base || s - base >= 64u) return 0u;
    const uint32_t p = static_cast<uint32_t>(s & 63u);
    if (!(((A.preparing[g] | A.accepting[g] | A.committed[g]) >> p) & 1u)) return 0u;   // null: no replica_bk
    *at = static_cast<uint64_t>(g) * 64u + p;
    const uint64_t trig = A.prep_trigger[*at], vb = A.voted_bal[*at];
    uint64_t len = 9u + wv_len(A.variant) + wv_len(s) + wv_len(trig) + wv_len(trig + A.prep_span[*at]) + wv_len(A.inst_bal[*at]) + 1u;
    if (vb > 0u) len += wv_len(vb) + cw_bytes(A.data_len[*at], A.d, A.T, __popc(A.voted_mask[*at]));
    return len;
}

// 1. a thread per record: the reply's bytes and its 16-byte region
__global__ void __launch_bounds__(kAccThreads) prep_reply_size_kernel(const __grid_constant__ PrepReplyArgs A) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kAccThreads;
    for (uint64_t k = static_cast<uint64_t>(blockIdx.x) * kAccThreads + threadIdx.x; k < A.n; k += stride) {
        uint64_t at = 0;
        const uint64_t len = prep_reply_bytes(A, k, &at);
        A.reply_len[k] = len;
        A.reply_off[k] = round16(len);
    }
}

// 2. a warp per record: capacity, then PeerMessage::Msg{PrepareReply{slot, trigger_slot, endprep_slot, ballot, voted}}
__global__ void __launch_bounds__(kAccThreads) prep_reply_copy_kernel(const __grid_constant__ PrepReplyArgs A) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = (static_cast<uint64_t>(blockIdx.x) * kAccThreads + threadIdx.x) >> 5;
    const uint64_t nwarps = (static_cast<uint64_t>(gridDim.x) * kAccThreads) >> 5;
    bool full = false;
    for (uint64_t k = warp; k < A.n; k += nwarps) {
        const uint64_t len = A.reply_len[k], off = A.reply_off[k];
        if (len == 0u || off > A.out_cap || round16(len) > A.out_cap - off) {
            full |= len != 0u;
            if (lane == 0u) {
                A.reply_off[k] = ~0ull;
                A.reply_dst[k] = 0xffu;
            }
            continue;
        }
        uint64_t at = 0;
        prep_reply_bytes(A, k, &at);
        const uint64_t s = A.rec_slot[k], trig = A.prep_trigger[at], vb = A.voted_bal[at];
        uint8_t *dst = A.out + off;
        uint64_t q = 8u;
        q += wv_len(0u) + wv_len(A.variant) + wv_len(s) + wv_len(trig) + wv_len(trig + A.prep_span[at]) + wv_len(A.inst_bal[at]) + 1u;
        if (vb > 0u) q += wv_len(vb);
        if (lane == 0u) {
            put_be64(dst, len - 8u);
            uint64_t m = 8u;
            m += wv_put(dst + m, 0u);                                           // PeerMessage::Msg
            m += wv_put(dst + m, A.variant);
            m += wv_put(dst + m, s);
            m += wv_put(dst + m, trig);
            m += wv_put(dst + m, trig + A.prep_span[at]);
            m += wv_put(dst + m, A.inst_bal[at]);
            dst[m++] = vb > 0u ? 1u : 0u;                                       // voted: Option
            if (vb > 0u) wv_put(dst + m, vb);
            A.reply_dst[k] = A.source[at];
        }
        if (vb > 0u)
            warp_put_codeword(dst + q, A.d, A.T, A.data_len[at], A.voted_mask[at], A.held[at],
                              reinterpret_cast<const uint8_t *>(A.shard_addr[at]), lane);
    }
    if (full && lane == 0u) atomicOr(A.status, SS_DEV_STATUS_FRAME_OVERFLOW);
}

// ---- reconstruct requests ----------------------------------------------------------------------------------------
struct ReqArgs {
    const uint32_t *groups;         // the listed groups; nullptr: entry i is group i
    const uint32_t *peer_alive;     // [G] peer masks; nullptr: every peer is alive
    uint64_t n, G, tail, batch;     // batch <= 64: no destination gets more than 64 entries of one group
    uint32_t me, population, d, T, variant, crossword, step_up;
    const uint64_t *window_base, *accepting, *committed, *preparing, *exec_bar;
    const uint32_t *held, *assign_rows;
    const uint8_t *source;
    uint64_t *gossip_bar;
    uint64_t *bar0;                 // [n] gossip_bar of entry i's group as the size pass read it
    uint64_t *cnt, *bytes;          // [n] frames and region bytes of entry i, then their exclusive scans
    const uint64_t *totals;         // [2] the two scans' totals
    uint8_t *out;
    uint64_t out_cap;
    uint32_t *frame_group;
    uint8_t *frame_dst;
    uint64_t *frame_off;
    uint32_t *frame_len;
    uint64_t frame_cap;
    uint32_t *status;
};

// per-warp scratch of one destination's entries
struct ReqWarp {
    uint32_t pre[65];               // pre[k]: bytes of the destination's first k entries
    uint64_t off[64];               // write pass: the frame offset of each chunk
};

__device__ __forceinline__ uint64_t warp_incl_scan(uint64_t x, uint32_t lane) {
    for (int s = 1; s < 32; s <<= 1) {
        const uint64_t y = __shfl_up_sync(0xffffffffu, x, s);
        if (lane >= static_cast<uint32_t>(s)) x += y;
    }
    return x;
}

// The walk of group g from gossip_bar = bar0, warp-uniform.  Returns the window positions with an entry (bit w: slot
// base + w, committed with fewer than d shards held); *bar = gossip_bar after the walk.
//   gossip (trigger_gossiping, crossword/gossiping.rs:88-192): slots [max(bar0, base), until), until = log_end minus
//     tail_ignores, log_end = base + 1 + the last window position that is Preparing, Accepting or Committed; a slot
//     below exec_bar is Executed and passed, the first other slot that is not committed stops the walk; the last slot
//     visited (the stop included) is slot_up_to, and the bar moves to max(bar0, slot_up_to)
//   step-up (become_a_leader's recon_slots, rspaxos/leadership.rs:99-172, crossword/leadership.rs:105-190): every slot
//     of [max(exec_bar, base), base + 64), no stop
__device__ __forceinline__ uint64_t request_walk(const ReqArgs &A, uint32_t g, uint64_t bar0, uint32_t lane, uint64_t *bar) {
    const uint64_t base = A.window_base[g], eb = A.exec_bar[g];
    const uint32_t r = static_cast<uint32_t>(base & 63u);
    const uint64_t com = ring_to_window(A.committed[g], r);
    const uint64_t exec_w = eb <= base ? 0ull : eb - base >= 64u ? ~0ull : (1ull << (eb - base)) - 1u;
    uint64_t walk = 0u;
    *bar = bar0;
    if (A.step_up) {
        walk = com & ~exec_w;
    } else {
        const uint64_t live = ring_to_window(A.preparing[g] | A.accepting[g] | A.committed[g], r);
        const uint64_t log_end = base + (live == 0u ? 0u : 64u - static_cast<uint64_t>(__clzll(static_cast<long long>(live))));
        const uint64_t until = log_end > A.tail ? log_end - A.tail : 0u;
        const uint64_t start = bar0 > base ? bar0 : base;
        if (start < until) {                                                    // lo < hi <= 64
            const uint64_t lo = start - base, hi = until - base;
            const uint64_t range = (hi == 64u ? ~0ull : (1ull << hi) - 1u) & ~((1ull << lo) - 1u);
            const uint64_t stop = range & ~exec_w & ~com;
            const uint64_t first = stop != 0u ? static_cast<uint64_t>(__ffsll(static_cast<long long>(stop))) - 1u : 64u;
            walk = range & ~exec_w & com & (first == 64u ? ~0ull : (1ull << first) - 1u);
            const uint64_t up_to = base + (first != 64u ? first : hi - 1u);
            *bar = up_to > bar0 ? up_to : bar0;
        }
    }
    const uint64_t row = static_cast<uint64_t>(g) * 64u;
    bool need[2];
    for (uint32_t h = 0; h < 2u; ++h) {
        const uint32_t w = lane + 32u * h;
        need[h] = ((walk >> w) & 1u) && static_cast<uint32_t>(__popc(A.held[row + ((r + w) & 63u)])) < A.d;
    }
    return static_cast<uint64_t>(__ballot_sync(0xffffffffu, need[0])) | static_cast<uint64_t>(__ballot_sync(0xffffffffu, need[1])) << 32;
}

// gossip_targets_excl for the instance at `at`: the selected peers; *excl = the exclusion of peer q when it is selected
__device__ __forceinline__ uint32_t request_targets(const ReqArgs &A, uint64_t at, uint32_t alive, uint32_t q, uint32_t *excl) {
    const uint32_t *rows = A.assign_rows + at * A.population;
    return gossip_walk(A.me, A.population, A.d, A.source[at], A.held[at], alive, [&](uint32_t p) { return rows[p]; },
                       [&](uint32_t p, uint32_t avail) { if (p == q) *excl = avail; });
}

// one entry: slot (RSPaxos), or (slot, Bitmap{size T, one block: excl}) as ssor_bitmap_encode writes it (Crossword)
__device__ __forceinline__ uint32_t request_entry_bytes(const ReqArgs &A, uint64_t slot, uint32_t excl) {
    return static_cast<uint32_t>(wv_len(slot)) + (A.crossword ? static_cast<uint32_t>(wv_len(A.T) + 1 + wv_len(excl)) : 0u);
}

// frame c of a destination with cnt entries: 8-byte length, PeerMessage::Msg, the variant, the entry count, the entries
__device__ __forceinline__ uint64_t request_frame_len(const ReqArgs &A, const ReqWarp &W, uint32_t c, uint32_t cnt) {
    const uint32_t b = static_cast<uint32_t>(A.batch), k0 = c * b, m = cnt - k0 < b ? cnt - k0 : b;
    return 9u + wv_len(A.variant) + wv_len(m) + (W.pre[k0 + m] - W.pre[k0]);
}

// The destinations of group g in order (gossip: peers 0..population-1, step-up: one broadcast list), each with its
// entries in slot order.  For each destination with entries: W.pre holds the entry byte prefix, and
// per_dst(q, cnt, sel, k, excl) runs on the whole warp (this lane's positions: sel[h], entry index k[h], exclusion).
template <typename F>
__device__ void request_plan(const ReqArgs &A, uint32_t g, uint64_t need, uint32_t lane, ReqWarp &W, F &&per_dst) {
    const uint64_t base = A.window_base[g];
    const uint32_t alive = A.peer_alive != nullptr ? A.peer_alive[g] : 0xffffffffu;
    uint64_t at[2];
    uint32_t t[2] = {0u, 0u};
    for (uint32_t h = 0; h < 2u; ++h) {
        const uint32_t w = lane + 32u * h;
        at[h] = static_cast<uint64_t>(g) * 64u + ((base + w) & 63u);
        if ((need >> w) & 1u) t[h] = A.step_up ? 1u : request_targets(A, at[h], alive, 32u, nullptr);
    }
    const uint32_t ndst = A.step_up ? 1u : A.population;
    const uint32_t below = (1u << lane) - 1u;
    for (uint32_t q = 0; q < ndst; ++q) {
        bool sel[2];
        uint32_t b[2];
        for (uint32_t h = 0; h < 2u; ++h) {
            sel[h] = (t[h] >> q) & 1u;
            b[h] = __ballot_sync(0xffffffffu, sel[h]);
        }
        const uint32_t cnt = static_cast<uint32_t>(__popc(b[0]) + __popc(b[1]));
        if (cnt == 0u) continue;
        const uint32_t k[2] = {static_cast<uint32_t>(__popc(b[0] & below)), static_cast<uint32_t>(__popc(b[0]) + __popc(b[1] & below))};
        uint32_t ex[2] = {0u, 0u}, e[2] = {0u, 0u};
        for (uint32_t h = 0; h < 2u; ++h) {
            if (!sel[h]) continue;
            if (A.step_up) ex[h] = A.held[at[h]];
            else request_targets(A, at[h], alive, q, &ex[h]);
            e[h] = request_entry_bytes(A, base + lane + 32u * h, ex[h]);
        }
        const uint64_t s0 = warp_incl_scan(e[0], lane), s1 = warp_incl_scan(e[1], lane) + __shfl_sync(0xffffffffu, s0, 31);
        __syncwarp();                   // the previous destination's readers of W are done
        if (lane == 0u) W.pre[0] = 0u;
        if (sel[0]) W.pre[k[0] + 1u] = static_cast<uint32_t>(s0);
        if (sel[1]) W.pre[k[1] + 1u] = static_cast<uint32_t>(s1);
        __syncwarp();
        per_dst(q, cnt, sel, k, ex);
    }
    __syncwarp();
}

__device__ __forceinline__ uint32_t request_group(const ReqArgs &A, uint64_t i) { return A.groups != nullptr ? A.groups[i] : static_cast<uint32_t>(i); }

// 1. a warp per listed group: the walk, the plan, the frames and region bytes it asks for
__global__ void __launch_bounds__(kAccThreads) request_size_kernel(const __grid_constant__ ReqArgs A) {
    __shared__ ReqWarp Ws[kExecWarps];
    const uint32_t lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
    ReqWarp &W = Ws[w];
    const uint64_t nwarps = static_cast<uint64_t>(gridDim.x) * kExecWarps;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kExecWarps + w; i < A.n; i += nwarps) {
        const uint32_t g = request_group(A, i);
        uint64_t frames = 0u, bytes = 0u;
        if (g < A.G) {
            const uint64_t bar0 = A.gossip_bar[g];
            uint64_t bar;
            const uint64_t need = request_walk(A, g, bar0, lane, &bar);
            request_plan(A, g, need, lane, W, [&](uint32_t, uint32_t cnt, const bool *, const uint32_t *, const uint32_t *) {
                const uint32_t nc = (cnt + static_cast<uint32_t>(A.batch) - 1u) / static_cast<uint32_t>(A.batch);
                uint64_t b = 0u;
                for (uint32_t c = lane; c < nc; c += 32u) b += round16(request_frame_len(A, W, c, cnt));
                frames += nc;
                bytes += warp_sum(b);
            });
            if (lane == 0u) A.bar0[i] = bar0;
        }
        if (lane == 0u) {
            A.cnt[i] = frames;
            A.bytes[i] = bytes;
        }
    }
}

// 2. a warp per listed group: capacity, then the same plan again from the same bar, written: frame headers by the lane
//    of each chunk, entries by the lane of their slot; gossip_bar of the placed groups
__global__ void __launch_bounds__(kAccThreads) request_write_kernel(const __grid_constant__ ReqArgs A) {
    __shared__ ReqWarp Ws[kExecWarps];
    const uint32_t lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
    ReqWarp &W = Ws[w];
    bool full = false;
    const uint64_t nwarps = static_cast<uint64_t>(gridDim.x) * kExecWarps;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kExecWarps + w; i < A.n; i += nwarps) {
        const uint32_t g = request_group(A, i);
        if (g >= A.G) continue;
        const uint64_t f0 = A.cnt[i], o0 = A.bytes[i];
        const uint64_t f1 = i + 1u < A.n ? A.cnt[i + 1u] : A.totals[0], o1 = i + 1u < A.n ? A.bytes[i + 1u] : A.totals[1];
        if (f1 > A.frame_cap || o1 > A.out_cap) {                              // the ends are monotone: a suffix is cut
            full = true;
            for (uint64_t f = f0 + lane; f < f1 && f < A.frame_cap; f += 32u) {
                A.frame_group[f] = g;
                A.frame_dst[f] = 0xffu;
                A.frame_off[f] = ~0ull;
                A.frame_len[f] = 0u;
            }
            continue;
        }
        const uint64_t bar0 = A.bar0[i], base = A.window_base[g];
        uint64_t bar;
        const uint64_t need = request_walk(A, g, bar0, lane, &bar);
        uint64_t fr = f0, ob = o0;
        const uint32_t B = static_cast<uint32_t>(A.batch), vl = static_cast<uint32_t>(wv_len(A.variant));
        request_plan(A, g, need, lane, W, [&](uint32_t q, uint32_t cnt, const bool *sel, const uint32_t *k, const uint32_t *ex) {
            const uint32_t nc = (cnt + B - 1u) / B;
            for (uint32_t c0 = 0; c0 < nc; c0 += 32u) {
                const uint32_t c = c0 + lane;
                const uint64_t len = c < nc ? request_frame_len(A, W, c, cnt) : 0u, reg = round16(len);
                const uint64_t incl = warp_incl_scan(reg, lane), o = ob + incl - reg;
                if (c < nc) {
                    W.off[c] = o;
                    const uint64_t f = fr + c;
                    A.frame_group[f] = g;
                    A.frame_dst[f] = A.step_up ? 0xffu : static_cast<uint8_t>(q);
                    A.frame_off[f] = o;
                    A.frame_len[f] = static_cast<uint32_t>(len);
                    uint8_t *dst = A.out + o;
                    put_be64(dst, len - 8u);
                    uint32_t m = 8u;
                    m += wv_put(dst + m, 0u);                                   // PeerMessage::Msg
                    m += wv_put(dst + m, A.variant);
                    wv_put(dst + m, cnt - c * B < B ? cnt - c * B : B);
                }
                ob += __shfl_sync(0xffffffffu, incl, 31);
            }
            fr += nc;
            __syncwarp();
            for (uint32_t h = 0; h < 2u; ++h) {
                if (!sel[h]) continue;
                const uint32_t c = k[h] / B, m = cnt - c * B < B ? cnt - c * B : B;
                uint8_t *e = A.out + W.off[c] + 9u + vl + wv_len(m) + (W.pre[k[h]] - W.pre[c * B]);
                e += wv_put(e, base + lane + 32u * h);
                if (A.crossword) {                                              // Bitmap: size, one block
                    e += wv_put(e, A.T);
                    e += wv_put(e, 1u);
                    wv_put(e, ex[h]);
                }
            }
        });
        if (!A.step_up && lane == 0u) A.gossip_bar[g] = bar;
    }
    if (full && lane == 0u) atomicOr(A.status, SS_DEV_STATUS_FRAME_OVERFLOW);
}

int acc_scratch(ss_acceptor *a, uint64_t n) {
    if (n <= a->cap_frames) return SS_OK;
    ss_ctx *ctx = a->ctx;
    SS_CUDA(cudaStreamSynchronize(ctx->stream));
    void *old[] = {a->hdr, a->keys, a->idx, a->partials, a->fcnt, a->sort_tmp};
    for (void *b : old)
        if (b) cudaFree(b);
    a->hdr = nullptr; a->keys = nullptr; a->idx = nullptr; a->partials = nullptr; a->fcnt = nullptr; a->sort_tmp = nullptr;
    a->cap_frames = 0;
    // the header pass writes hdr, key_in and idx_in (and fcnt) of every frame, the sort the rest, the scan its partials
    SS_TRY(dalloc(ctx, &a->hdr, n, false));
    SS_TRY(dalloc(ctx, &a->keys, 2 * n, false));
    SS_TRY(dalloc(ctx, &a->idx, 2 * n, false));
    SS_TRY(dalloc(ctx, &a->partials, scan_tiles(n), false));
    SS_TRY(dalloc(ctx, &a->fcnt, n, false));
    size_t bytes = 0;
    SS_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, bytes, a->keys, a->keys + n, a->idx, a->idx + n, static_cast<int>(n), 0,
                                            key_bits(a->G), ctx->stream));
    SS_CUDA(cudaMalloc(&a->sort_tmp, bytes ? bytes : 1));
    a->sort_tmp_bytes = bytes;
    a->cap_frames = n;
    return SS_OK;
}

}  // namespace ssb

using namespace ssb;

extern "C" {

int ss_acceptor_destroy(ss_acceptor *a) {
    if (a == nullptr) return SS_OK;
    if (a->ctx) {
        cudaSetDevice(a->ctx->device);
        cudaStreamSynchronize(a->ctx->stream);
    }
    void *bufs[] = {a->window_base, a->bal_max_seen, a->inst_bal, a->accepting, a->shard_addr, a->held, a->data_len, a->assignment,
                    a->source, a->committed, a->commit_bar, a->exec_bar, a->preparing, a->voted_bal, a->voted_mask,
                    a->prep_trigger, a->prep_span, a->assign_rows, a->gossip_bar, a->matrix, a->ex_cnt, a->ex_bytes,
                    a->ex_partials, a->ex_n, a->hdr,
                    a->keys, a->idx, a->partials, a->fcnt, a->sort_tmp, a->totals};
    for (void *b : bufs)
        if (b) cudaFree(b);
    if (a->ctx) ctx_release(a->ctx);
    delete a;
    return SS_OK;
}

int ss_acceptor_create(ss_ctx *ctx, const ss_acceptor_config *cfg, uint64_t G, ss_acceptor **out) {
    if (out == nullptr) return set_error(SS_ERR_INVALID_ARG, "null out pointer");
    *out = nullptr;
    if (cfg == nullptr || G == 0) return set_error(SS_ERR_INVALID_ARG, "null config or zero groups");
    if (G > 0xffffffffull) return set_error(SS_ERR_INVALID_ARG, "at most 2^32 - 1 groups");
    if (cfg->protocol != SS_PROTO_RSPAXOS && cfg->protocol != SS_PROTO_CROSSWORD)
        return set_error(SS_ERR_INVALID_ARG, "the acceptor serves RSPaxos and Crossword, not protocol %u", cfg->protocol);
    if (cfg->population == 0 || cfg->population > 32 || cfg->me >= cfg->population)
        return set_error(SS_ERR_INVALID_ARG, "bad population %u / me %u", cfg->population, cfg->me);
    if (cfg->data_shards == 0 || cfg->data_shards > cfg->total_shards || cfg->total_shards > 32)
        return set_error(SS_ERR_INVALID_ARG, "shard counts must satisfy 1 <= d <= T <= 32 (d=%u, T=%u)", cfg->data_shards,
                         cfg->total_shards);
    if (ctx == nullptr) {
        int count = 0;
        const cudaError_t e = cudaGetDeviceCount(&count);
        cudaGetLastError();
        if (e != cudaSuccess || count == 0) return set_error(SS_ERR_NO_DEVICE, "no CUDA device available; this library has no CPU fallback");
        return set_error(SS_ERR_INVALID_ARG, "null context");
    }
    SS_TRY(ctx_bind(ctx));
    ss_acceptor *a = new (std::nothrow) ss_acceptor();
    if (!a) return set_error(SS_ERR_OUT_OF_MEMORY, "host allocation failed");
    a->ctx = ctx; a->cfg = *cfg; a->G = G;
    ctx_retain(ctx);
    int rc = SS_OK;
    if ((rc = dalloc(ctx, &a->window_base, G)) || (rc = dalloc(ctx, &a->bal_max_seen, G)) ||
        (rc = dalloc(ctx, &a->inst_bal, G * 64)) || (rc = dalloc(ctx, &a->accepting, G)) ||
        (rc = dalloc(ctx, &a->shard_addr, G * 64)) || (rc = dalloc(ctx, &a->held, G * 64)) ||
        (rc = dalloc(ctx, &a->data_len, G * 64)) || (rc = dalloc(ctx, &a->source, G * 64)) || (rc = dalloc(ctx, &a->totals, 2)) ||
        (cfg->protocol == SS_PROTO_CROSSWORD && (rc = dalloc(ctx, &a->assignment, G * 64))) ||
        (cfg->protocol == SS_PROTO_CROSSWORD && (rc = dalloc(ctx, &a->assign_rows, G * 64 * cfg->population))) ||
        (rc = dalloc(ctx, &a->gossip_bar, G)) ||
        (rc = dalloc(ctx, &a->committed, G)) || (rc = dalloc(ctx, &a->commit_bar, G)) || (rc = dalloc(ctx, &a->exec_bar, G)) ||
        (rc = dalloc(ctx, &a->preparing, G)) || (rc = dalloc(ctx, &a->voted_bal, G * 64)) ||
        (rc = dalloc(ctx, &a->voted_mask, G * 64)) || (rc = dalloc(ctx, &a->prep_trigger, G * 64)) ||
        (rc = dalloc(ctx, &a->prep_span, G * 64)) ||
        (rc = dalloc(ctx, &a->ex_cnt, G, false)) || (rc = dalloc(ctx, &a->ex_bytes, G, false)) ||
        (rc = dalloc(ctx, &a->ex_partials, scan_tiles(G), false)) || (rc = dalloc(ctx, &a->ex_n, 1, false)) ||
        (rc = dalloc(ctx, &a->matrix, size_t(cfg->total_shards) * cfg->data_shards, false))) {
        ss_acceptor_destroy(a);
        return rc;
    }
    // the coder's matrix, whose rows ss_acceptor_execute inverts on the device; a pageable source is staged before the
    // call returns
    const gf::Matrix m = gf::coding_matrix(static_cast<int>(cfg->data_shards), static_cast<int>(cfg->total_shards - cfg->data_shards));
    if (cudaMemcpyAsync(a->matrix, m.v.data(), m.v.size(), cudaMemcpyHostToDevice, ctx->stream) != cudaSuccess) {
        ss_acceptor_destroy(a);
        return set_error(SS_ERR_CUDA, "coding matrix upload failed");
    }
    *out = a;
    return SS_OK;
}

int ss_acceptor_commit_view_get(ss_acceptor *a, ss_acceptor_commit_view *v) {
    if (a == nullptr || v == nullptr) return set_error(SS_ERR_INVALID_ARG, "null argument");
    memset(v, 0, sizeof(*v));
    v->n_groups = a->G;
    v->committed = a->committed; v->commit_bar = a->commit_bar; v->exec_bar = a->exec_bar;
    return SS_OK;
}

int ss_acceptor_heartbeat(ss_acceptor *a, const uint32_t *hb_group, const uint8_t *hb_peer, const uint64_t *hb_ballot,
                          const uint64_t *hb_commit_bar, const uint64_t *hb_exec_bar, uint64_t n, uint64_t *newly) {
    if (a == nullptr) return set_error(SS_ERR_INVALID_ARG, "null acceptor");
    ss_ctx *ctx = a->ctx;
    SS_TRY(ctx_bind(ctx));
    if (newly != nullptr) SS_CUDA(cudaMemsetAsync(newly, 0, a->G * 8, ctx->stream));
    if (n == 0) return SS_OK;
    if (!hb_group || !hb_peer || !hb_ballot || !hb_commit_bar || !hb_exec_bar) return set_error(SS_ERR_INVALID_ARG, "null buffer");
    if (n > 0x7fffffffull) return set_error(SS_ERR_INVALID_ARG, "at most 2^31 - 1 records per call");
    SS_TRY(acc_scratch(a, n));
    HbArgs H{};
    H.group = hb_group; H.peer = hb_peer; H.ballot = hb_ballot; H.hb_commit_bar = hb_commit_bar; H.hb_exec_bar = hb_exec_bar;
    H.n = n; H.G = a->G; H.me = a->cfg.me;
    H.window_base = a->window_base; H.inst_bal = a->inst_bal; H.commit_bar = a->commit_bar; H.exec_bar = a->exec_bar;
    H.bal_max_seen = a->bal_max_seen; H.accepting = a->accepting; H.committed = a->committed; H.newly = newly;
    H.key_in = a->keys; H.idx_in = a->idx; H.key = a->keys + n; H.idx = a->idx + n;
    const uint32_t grid = launch_grid(ctx, n, kAccThreads);
    heartbeat_keys_kernel<<<grid, kAccThreads, 0, ctx->stream>>>(H);
    SS_TRY(launched(ctx));
    size_t bytes = a->sort_tmp_bytes;
    SS_CUDA(cub::DeviceRadixSort::SortPairs(a->sort_tmp, bytes, a->keys, a->keys + n, a->idx, a->idx + n, static_cast<int>(n), 0,
                                            key_bits(a->G), ctx->stream));
    SS_TRY(launched(ctx));
    heartbeat_walk_kernel<<<grid, kAccThreads, 0, ctx->stream>>>(H);
    return launched(ctx);
}

int ss_acceptor_execute(ss_acceptor *a, uint8_t *out, uint64_t out_capacity, uint32_t *rec_group, uint64_t *rec_slot,
                        uint64_t *rec_off, uint32_t *rec_len, uint64_t rec_capacity, uint64_t *totals) {
    if (a == nullptr) return set_error(SS_ERR_INVALID_ARG, "null acceptor");
    if (!out || !rec_group || !rec_slot || !rec_off || !rec_len) return set_error(SS_ERR_INVALID_ARG, "null buffer");
    if (reinterpret_cast<uintptr_t>(out) & 15u) return set_error(SS_ERR_INVALID_ARG, "out must be 16-byte aligned");
    ss_ctx *ctx = a->ctx;
    SS_TRY(ctx_bind(ctx));
    const ExecOut o{a->matrix, a->ex_cnt, a->ex_bytes, a->ex_n, out, out_capacity, rec_group, rec_slot, rec_off,
                    rec_len, rec_capacity, ctx->dev_status};
    const AccLog log{a->cfg.data_shards, a->window_base, a->committed, a->shard_addr, a->held, a->data_len, a->commit_bar};
    return launch_execute(ctx, o, log, log, a->G, a->G * 64u, a->ex_partials, totals != nullptr ? totals : a->totals);
}

int ss_acceptor_view_get(ss_acceptor *a, ss_acceptor_view *v) {
    if (a == nullptr || v == nullptr) return set_error(SS_ERR_INVALID_ARG, "null argument");
    memset(v, 0, sizeof(*v));
    v->n_groups = a->G; v->protocol = a->cfg.protocol; v->population = a->cfg.population; v->me = a->cfg.me;
    v->data_shards = a->cfg.data_shards; v->total_shards = a->cfg.total_shards;
    v->window_base = a->window_base; v->bal_max_seen = a->bal_max_seen; v->inst_bal = a->inst_bal; v->accepting = a->accepting;
    v->shard_addr = a->shard_addr; v->held = a->held; v->data_len = a->data_len; v->assignment = a->assignment; v->source = a->source;
    return SS_OK;
}

int ss_acceptor_window_get(ss_acceptor *a, uint64_t **window_base) {
    if (a == nullptr || window_base == nullptr) return set_error(SS_ERR_INVALID_ARG, "null argument");
    *window_base = a->window_base;
    return SS_OK;
}

int ss_acceptor_advance(ss_acceptor *a, const uint64_t *upto) {
    if (a == nullptr || upto == nullptr) return set_error(SS_ERR_INVALID_ARG, "null acceptor or upto");
    ss_ctx *ctx = a->ctx;
    SS_TRY(ctx_bind(ctx));
    acceptor_advance_kernel<<<launch_grid(ctx, a->G, kAccThreads), kAccThreads, 0, ctx->stream>>>(upto, a->G, a->window_base, a->accepting,
                                                                                               a->committed, a->preparing);
    return launched(ctx);
}

int ss_acceptor_accept(ss_acceptor *a, const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off, const uint32_t *frame_group,
                       const uint8_t *frame_peer, uint64_t n, uint8_t *store, uint64_t store_capacity, uint64_t *store_off,
                       uint8_t *wal, uint64_t wal_capacity, uint64_t *wal_off, uint32_t *wal_len, uint8_t *replies,
                       uint32_t *reply_len, uint8_t *reply_dst, uint32_t *verdict, uint64_t *totals) {
    if (a == nullptr) return set_error(SS_ERR_INVALID_ARG, "null acceptor");
    ss_ctx *ctx = a->ctx;
    SS_TRY(ctx_bind(ctx));
    if (n == 0) {
        if (totals != nullptr) SS_CUDA(cudaMemsetAsync(totals, 0, 16, ctx->stream));
        return SS_OK;
    }
    if (!buf || !frame_off || !frame_group || !frame_peer || !store || !store_off || !wal || !wal_off || !wal_len || !replies ||
        !reply_len || !reply_dst || !verdict)
        return set_error(SS_ERR_INVALID_ARG, "null buffer");
    if ((reinterpret_cast<uintptr_t>(store) | reinterpret_cast<uintptr_t>(wal)) & 15u)
        return set_error(SS_ERR_INVALID_ARG, "store and wal must be 16-byte aligned");
    if (n > 0x7fffffffull) return set_error(SS_ERR_INVALID_ARG, "at most 2^31 - 1 frames per call");
    SS_TRY(acc_scratch(a, n));
    uint64_t *tot = totals != nullptr ? totals : a->totals;
    AccArgs A{};
    A.buf = buf; A.buf_len = buf_len; A.frame_off = frame_off; A.frame_group = frame_group; A.frame_peer = frame_peer;
    A.n = n; A.G = a->G;
    A.d = a->cfg.data_shards; A.T = a->cfg.total_shards; A.population = a->cfg.population; A.me = a->cfg.me;
    A.accept_variant = a->cfg.accept_variant; A.wal_variant = a->cfg.wal_variant; A.reply_variant = a->cfg.reply_variant;
    A.crossword = a->cfg.protocol == SS_PROTO_CROSSWORD ? 1u : 0u;
    A.window_base = a->window_base; A.bal_max_seen = a->bal_max_seen; A.inst_bal = a->inst_bal; A.accepting = a->accepting;
    A.shard_addr = a->shard_addr; A.held = a->held; A.data_len = a->data_len; A.assignment = a->assignment; A.source = a->source;
    A.assign_rows = a->assign_rows; A.committed = a->committed;
    A.preparing = a->preparing; A.voted_bal = a->voted_bal; A.voted_mask = a->voted_mask; A.prep_trigger = a->prep_trigger;
    A.prep_span = a->prep_span;
    A.hdr = a->hdr; A.key_in = a->keys; A.idx_in = a->idx; A.key = a->keys + n; A.idx = a->idx + n;
    A.store = store; A.store_cap = store_capacity; A.store_off = store_off;
    A.wal = wal; A.wal_cap = wal_capacity; A.wal_off = wal_off; A.wal_len = wal_len;
    A.replies = replies; A.reply_len = reply_len; A.reply_dst = reply_dst; A.verdict = verdict; A.status = ctx->dev_status;
    const uint32_t grid_t = launch_grid(ctx, n, kAccThreads);
    acceptor_header_kernel<<<grid_t, kAccThreads, 0, ctx->stream>>>(A);
    SS_TRY(launched(ctx));
    size_t bytes = a->sort_tmp_bytes;
    SS_CUDA(cub::DeviceRadixSort::SortPairs(a->sort_tmp, bytes, a->keys, a->keys + n, a->idx, a->idx + n, static_cast<int>(n), 0,
                                            key_bits(a->G), ctx->stream));
    SS_TRY(launched(ctx));
    acceptor_ballot_kernel<<<grid_t, kAccThreads, 0, ctx->stream>>>(A);
    SS_TRY(launched(ctx));
    SS_TRY(launch_exclusive_scan_u64(ctx, store_off, n, a->partials, tot));
    SS_TRY(launch_exclusive_scan_u64(ctx, wal_off, n, a->partials, tot + 1));
    acceptor_place_kernel<<<grid_t, kAccThreads, 0, ctx->stream>>>(A);
    SS_TRY(launched(ctx));
    acceptor_copy_kernel<<<launch_grid(ctx, n, kAccThreads / 32), kAccThreads, 0, ctx->stream>>>(A);
    return launched(ctx);
}

static RecArgs rec_args(ss_acceptor *a, const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off, const uint32_t *frame_group,
                        uint64_t n, uint32_t variant) {
    RecArgs R{};
    R.buf = buf; R.buf_len = buf_len; R.frame_off = frame_off; R.frame_group = frame_group; R.n = n; R.G = a->G;
    R.d = a->cfg.data_shards; R.T = a->cfg.total_shards; R.variant = variant;
    R.crossword = a->cfg.protocol == SS_PROTO_CROSSWORD ? 1u : 0u;
    R.window_base = a->window_base; R.inst_bal = a->inst_bal; R.accepting = a->accepting; R.committed = a->committed;
    R.exec_bar = a->exec_bar; R.data_len = a->data_len; R.shard_addr = a->shard_addr; R.held = a->held;
    R.status = a->ctx->dev_status;
    return R;
}

int ss_acceptor_reconstruct_serve(ss_acceptor *a, const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off,
                                  const uint32_t *frame_group, const uint8_t *frame_peer, uint64_t n, uint32_t reconstruct_variant,
                                  uint32_t reply_variant, uint8_t *out, uint64_t out_capacity, uint64_t *reply_off,
                                  uint64_t *reply_len, uint32_t *verdict, uint64_t *total) {
    if (a == nullptr) return set_error(SS_ERR_INVALID_ARG, "null acceptor");
    ss_ctx *ctx = a->ctx;
    SS_TRY(ctx_bind(ctx));
    if (n == 0) {
        if (total != nullptr) SS_CUDA(cudaMemsetAsync(total, 0, 8, ctx->stream));
        return SS_OK;
    }
    if (!buf || !frame_off || !frame_group || !frame_peer || !out || !reply_off || !reply_len || !verdict)
        return set_error(SS_ERR_INVALID_ARG, "null buffer");
    if (reinterpret_cast<uintptr_t>(out) & 15u) return set_error(SS_ERR_INVALID_ARG, "out must be 16-byte aligned");
    if (n > 0x7fffffffull) return set_error(SS_ERR_INVALID_ARG, "at most 2^31 - 1 frames per call");
    SS_TRY(acc_scratch(a, n));
    RecArgs R = rec_args(a, buf, buf_len, frame_off, frame_group, n, reconstruct_variant);
    R.reply_variant = reply_variant; R.out = out; R.out_cap = out_capacity; R.reply_off = reply_off; R.reply_len = reply_len;
    R.verdict = verdict;
    const uint32_t grid_w = launch_grid(ctx, n, kExecWarps);
    serve_count_kernel<<<grid_w, kAccThreads, 0, ctx->stream>>>(R);
    SS_TRY(launched(ctx));
    SS_TRY(launch_exclusive_scan_u64(ctx, reply_off, n, a->partials, total != nullptr ? total : a->totals));
    serve_copy_kernel<<<grid_w, kAccThreads, 0, ctx->stream>>>(R);
    return launched(ctx);
}

int ss_acceptor_absorb(ss_acceptor *a, const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off, const uint32_t *frame_group,
                       const uint8_t *frame_peer, uint64_t n, uint32_t reply_variant, uint8_t *store, uint64_t store_capacity,
                       uint32_t *absorbed, uint32_t *verdict, uint64_t *total) {
    if (a == nullptr) return set_error(SS_ERR_INVALID_ARG, "null acceptor");
    ss_ctx *ctx = a->ctx;
    SS_TRY(ctx_bind(ctx));
    if (n == 0) {
        if (total != nullptr) SS_CUDA(cudaMemsetAsync(total, 0, 8, ctx->stream));
        return SS_OK;
    }
    if (!buf || !frame_off || !frame_group || !frame_peer || !store || !absorbed || !verdict) return set_error(SS_ERR_INVALID_ARG, "null buffer");
    if (reinterpret_cast<uintptr_t>(store) & 15u) return set_error(SS_ERR_INVALID_ARG, "store must be 16-byte aligned");
    if (n > 0x7fffffffull) return set_error(SS_ERR_INVALID_ARG, "at most 2^31 - 1 frames per call");
    SS_TRY(acc_scratch(a, n));
    RecArgs R = rec_args(a, buf, buf_len, frame_off, frame_group, n, reply_variant);
    R.rhdr = reinterpret_cast<ReplyHdr *>(a->hdr);   // the accept pass's per-frame header scratch, reused
    R.key_in = a->keys; R.idx_in = a->idx; R.key = a->keys + n; R.idx = a->idx + n;
    R.grp_bytes = a->ex_bytes;      // execute's per-group scratch: both calls are ordered on the context's stream
    R.store = store; R.store_cap = store_capacity; R.absorbed = absorbed; R.verdict = verdict;
    absorb_decode_kernel<<<launch_grid(ctx, n, kAccThreads), kAccThreads, 0, ctx->stream>>>(R);
    SS_TRY(launched(ctx));
    size_t bytes = a->sort_tmp_bytes;
    SS_CUDA(cub::DeviceRadixSort::SortPairs(a->sort_tmp, bytes, a->keys, a->keys + n, a->idx, a->idx + n, static_cast<int>(n), 0,
                                            key_bits(a->G), ctx->stream));
    SS_TRY(launched(ctx));
    SS_CUDA(cudaMemsetAsync(a->ex_bytes, 0, a->G * 8, ctx->stream));
    const uint32_t grid_w = launch_grid(ctx, n, kExecWarps);
    absorb_plan_kernel<<<grid_w, kAccThreads, 0, ctx->stream>>>(R);
    SS_TRY(launched(ctx));
    SS_TRY(launch_exclusive_scan_u64(ctx, a->ex_bytes, a->G, a->ex_partials, total != nullptr ? total : a->totals));
    absorb_copy_kernel<<<grid_w, kAccThreads, 0, ctx->stream>>>(R);
    return launched(ctx);
}

int ss_acceptor_prepare_view_get(ss_acceptor *a, ss_acceptor_prepare_view *v) {
    if (a == nullptr || v == nullptr) return set_error(SS_ERR_INVALID_ARG, "null argument");
    memset(v, 0, sizeof(*v));
    v->n_groups = a->G;
    v->preparing = a->preparing; v->voted_bal = a->voted_bal; v->voted_mask = a->voted_mask;
    v->prep_trigger = a->prep_trigger; v->prep_span = a->prep_span;
    return SS_OK;
}

int ss_acceptor_prepare(ss_acceptor *a, const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off, const uint32_t *frame_group,
                        const uint8_t *frame_peer, uint64_t n, uint32_t prepare_variant, uint32_t wal_variant, uint8_t *wal,
                        uint64_t wal_capacity, uint32_t *rec_group, uint64_t *rec_slot, uint32_t *rec_frame, uint64_t rec_capacity,
                        uint32_t *verdict, uint64_t *totals) {
    if (a == nullptr) return set_error(SS_ERR_INVALID_ARG, "null acceptor");
    if (wal_variant >= kVariantLimit) return set_error(SS_ERR_INVALID_ARG, "wal_variant must be below 2^16");
    ss_ctx *ctx = a->ctx;
    SS_TRY(ctx_bind(ctx));
    if (n == 0) {
        if (totals != nullptr) SS_CUDA(cudaMemsetAsync(totals, 0, 16, ctx->stream));
        return SS_OK;
    }
    if (!buf || !frame_off || !frame_group || !frame_peer || !wal || !rec_group || !rec_slot || !rec_frame || !verdict)
        return set_error(SS_ERR_INVALID_ARG, "null buffer");
    if (reinterpret_cast<uintptr_t>(wal) & 15u) return set_error(SS_ERR_INVALID_ARG, "wal must be 16-byte aligned");
    if (n > 0x7fffffffull) return set_error(SS_ERR_INVALID_ARG, "at most 2^31 - 1 frames per call");
    SS_TRY(acc_scratch(a, n));
    PrepArgs P{};
    P.buf = buf; P.buf_len = buf_len; P.frame_off = frame_off; P.frame_group = frame_group; P.frame_peer = frame_peer;
    P.n = n; P.G = a->G; P.me = a->cfg.me; P.variant = prepare_variant; P.wal_variant = wal_variant;
    P.window_base = a->window_base; P.bal_max_seen = a->bal_max_seen; P.inst_bal = a->inst_bal; P.accepting = a->accepting;
    P.committed = a->committed; P.preparing = a->preparing; P.voted_bal = a->voted_bal; P.prep_trigger = a->prep_trigger;
    P.voted_mask = a->voted_mask; P.source = a->source; P.prep_span = a->prep_span;
    P.hdr = reinterpret_cast<PrepHdr *>(a->hdr);
    P.key_in = a->keys; P.idx_in = a->idx; P.key = a->keys + n; P.idx = a->idx + n;
    P.cnt = a->fcnt; P.totals = totals != nullptr ? totals : a->totals;
    const uint64_t wal_cells = wal_capacity / 32u;
    P.cap = rec_capacity < wal_cells ? rec_capacity : wal_cells;
    P.wal = wal; P.rec_group = rec_group; P.rec_slot = rec_slot; P.rec_frame = rec_frame; P.verdict = verdict;
    P.status = ctx->dev_status;
    const uint32_t grid_t = launch_grid(ctx, n, kAccThreads);
    prepare_header_kernel<<<grid_t, kAccThreads, 0, ctx->stream>>>(P);
    SS_TRY(launched(ctx));
    size_t bytes = a->sort_tmp_bytes;
    SS_CUDA(cub::DeviceRadixSort::SortPairs(a->sort_tmp, bytes, a->keys, a->keys + n, a->idx, a->idx + n, static_cast<int>(n), 0,
                                            key_bits(a->G), ctx->stream));
    SS_TRY(launched(ctx));
    prepare_walk_kernel<<<grid_t, kAccThreads, 0, ctx->stream>>>(P);
    SS_TRY(launched(ctx));
    SS_TRY(launch_exclusive_scan_u64(ctx, a->fcnt, n, a->partials, P.totals));
    prepare_apply_kernel<<<grid_t, kAccThreads, 0, ctx->stream>>>(P);
    SS_TRY(launched(ctx));
    prepare_write_kernel<<<launch_grid(ctx, n, kAccThreads / 32), kAccThreads, 0, ctx->stream>>>(P);
    return launched(ctx);
}

int ss_acceptor_prepare_reply(ss_acceptor *a, const uint32_t *rec_group, const uint64_t *rec_slot, uint64_t n, uint32_t reply_variant,
                              uint8_t *out, uint64_t out_capacity, uint64_t *reply_off, uint64_t *reply_len, uint8_t *reply_dst,
                              uint64_t *total) {
    if (a == nullptr) return set_error(SS_ERR_INVALID_ARG, "null acceptor");
    ss_ctx *ctx = a->ctx;
    SS_TRY(ctx_bind(ctx));
    if (n == 0) {
        if (total != nullptr) SS_CUDA(cudaMemsetAsync(total, 0, 8, ctx->stream));
        return SS_OK;
    }
    if (!rec_group || !rec_slot || !out || !reply_off || !reply_len || !reply_dst) return set_error(SS_ERR_INVALID_ARG, "null buffer");
    if (reinterpret_cast<uintptr_t>(out) & 15u) return set_error(SS_ERR_INVALID_ARG, "out must be 16-byte aligned");
    if (n > 0x7fffffffull) return set_error(SS_ERR_INVALID_ARG, "at most 2^31 - 1 records per call");
    SS_TRY(acc_scratch(a, n));
    PrepReplyArgs R{};
    R.rec_group = rec_group; R.rec_slot = rec_slot; R.n = n; R.G = a->G;
    R.d = a->cfg.data_shards; R.T = a->cfg.total_shards; R.variant = reply_variant;
    R.window_base = a->window_base; R.preparing = a->preparing; R.accepting = a->accepting; R.committed = a->committed;
    R.inst_bal = a->inst_bal; R.voted_bal = a->voted_bal; R.prep_trigger = a->prep_trigger; R.shard_addr = a->shard_addr;
    R.voted_mask = a->voted_mask; R.held = a->held; R.data_len = a->data_len; R.source = a->source; R.prep_span = a->prep_span;
    R.out = out; R.out_cap = out_capacity; R.reply_off = reply_off; R.reply_len = reply_len; R.reply_dst = reply_dst;
    R.status = ctx->dev_status;
    prep_reply_size_kernel<<<launch_grid(ctx, n, kAccThreads), kAccThreads, 0, ctx->stream>>>(R);
    SS_TRY(launched(ctx));
    SS_TRY(launch_exclusive_scan_u64(ctx, reply_off, n, a->partials, total != nullptr ? total : a->totals));
    prep_reply_copy_kernel<<<launch_grid(ctx, n, kExecWarps), kAccThreads, 0, ctx->stream>>>(R);
    return launched(ctx);
}

int ss_acceptor_gossip_view_get(ss_acceptor *a, ss_acceptor_gossip_view *v) {
    if (a == nullptr || v == nullptr) return set_error(SS_ERR_INVALID_ARG, "null argument");
    memset(v, 0, sizeof(*v));
    v->n_groups = a->G; v->population = a->cfg.population;
    v->assign_rows = a->assign_rows; v->gossip_bar = a->gossip_bar;
    return SS_OK;
}

}  // extern "C"

// the two request calls: size pass, scans of frames and bytes over the listed groups, write pass
static int acceptor_requests(ss_acceptor *a, bool step_up, const uint32_t *groups, uint64_t n_listed, const uint32_t *peer_alive,
                             uint64_t tail_ignores, uint64_t batch, uint32_t variant, uint8_t *out, uint64_t out_capacity,
                             uint32_t *frame_group, uint8_t *frame_dst, uint64_t *frame_off, uint32_t *frame_len,
                             uint64_t frame_capacity, uint64_t *totals) {
    if (a == nullptr) return set_error(SS_ERR_INVALID_ARG, "null acceptor");
    if (!step_up && a->cfg.protocol != SS_PROTO_CROSSWORD) return set_error(SS_ERR_INVALID_ARG, "gossip is Crossword's");
    if (batch == 0) return set_error(SS_ERR_INVALID_ARG, "batch / chunk size must be at least 1");
    ss_ctx *ctx = a->ctx;
    SS_TRY(ctx_bind(ctx));
    const uint64_t n = groups != nullptr ? n_listed : a->G;
    if (n == 0) {
        if (totals != nullptr) SS_CUDA(cudaMemsetAsync(totals, 0, 16, ctx->stream));
        return SS_OK;
    }
    if (!out || !frame_group || !frame_dst || !frame_off || !frame_len) return set_error(SS_ERR_INVALID_ARG, "null buffer");
    if (reinterpret_cast<uintptr_t>(out) & 15u) return set_error(SS_ERR_INVALID_ARG, "out must be 16-byte aligned");
    if (n > 0x7fffffffull) return set_error(SS_ERR_INVALID_ARG, "at most 2^31 - 1 listed groups per call");
    SS_TRY(acc_scratch(a, n));
    ReqArgs R{};
    R.groups = groups; R.peer_alive = peer_alive; R.n = n; R.G = a->G; R.tail = tail_ignores; R.batch = batch < 64u ? batch : 64u;
    R.me = a->cfg.me; R.population = a->cfg.population; R.d = a->cfg.data_shards; R.T = a->cfg.total_shards; R.variant = variant;
    R.crossword = a->cfg.protocol == SS_PROTO_CROSSWORD ? 1u : 0u; R.step_up = step_up ? 1u : 0u;
    R.window_base = a->window_base; R.accepting = a->accepting; R.committed = a->committed; R.preparing = a->preparing;
    R.exec_bar = a->exec_bar; R.held = a->held; R.assign_rows = a->assign_rows; R.source = a->source; R.gossip_bar = a->gossip_bar;
    // per-entry scratch: the header pass's FrameHdr cells (6 words each) hold bytes and bar0, fcnt the frame counts
    uint64_t *words = reinterpret_cast<uint64_t *>(a->hdr);
    R.bytes = words; R.bar0 = words + n; R.cnt = a->fcnt;
    uint64_t *tot = totals != nullptr ? totals : a->totals;
    R.totals = tot;
    R.out = out; R.out_cap = out_capacity; R.frame_group = frame_group; R.frame_dst = frame_dst; R.frame_off = frame_off;
    R.frame_len = frame_len; R.frame_cap = frame_capacity; R.status = ctx->dev_status;
    const uint32_t grid_w = launch_grid(ctx, n, kExecWarps);
    request_size_kernel<<<grid_w, kAccThreads, 0, ctx->stream>>>(R);
    SS_TRY(launched(ctx));
    SS_TRY(launch_exclusive_scan_u64(ctx, R.cnt, n, a->partials, tot));
    SS_TRY(launch_exclusive_scan_u64(ctx, R.bytes, n, a->partials, tot + 1));
    request_write_kernel<<<grid_w, kAccThreads, 0, ctx->stream>>>(R);
    return launched(ctx);
}

extern "C" {

int ss_acceptor_gossip(ss_acceptor *a, const uint32_t *groups, uint64_t n_listed, const uint32_t *peer_alive, uint64_t tail_ignores,
                       uint64_t batch_size, uint32_t reconstruct_variant, uint8_t *out, uint64_t out_capacity, uint32_t *frame_group,
                       uint8_t *frame_dst, uint64_t *frame_off, uint32_t *frame_len, uint64_t frame_capacity, uint64_t *totals) {
    return acceptor_requests(a, false, groups, n_listed, peer_alive, tail_ignores, batch_size, reconstruct_variant, out, out_capacity,
                             frame_group, frame_dst, frame_off, frame_len, frame_capacity, totals);
}

int ss_acceptor_step_up_reads(ss_acceptor *a, const uint32_t *groups, uint64_t n_listed, uint64_t chunk_size,
                              uint32_t reconstruct_variant, uint8_t *out, uint64_t out_capacity, uint32_t *frame_group,
                              uint8_t *frame_dst, uint64_t *frame_off, uint32_t *frame_len, uint64_t frame_capacity, uint64_t *totals) {
    return acceptor_requests(a, true, groups, n_listed, nullptr, 0u, chunk_size, reconstruct_variant, out, out_capacity, frame_group,
                             frame_dst, frame_off, frame_len, frame_capacity, totals);
}

}  // extern "C"
