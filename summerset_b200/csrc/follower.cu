// follower.cu -- the CRaft follower behind the C ABI (ss_follower_*), and the leader's AppendEntriesReply parser.
//
// What a CRaft follower does for every AppendEntries: handle_msg_append_entries (craft/messages.rs:14-252) with
// check_term (craft/leadership.rs:16-75), the DurEntry::LogEntry records it appends, and the AppendEntriesReply it sends
// straight away or once those records are durable (craft/durability.rs:129-160) -- for a batch of frames of many groups:
//
//   follower_header_kernel   a thread per frame: decode and validate every entry, the window filter, the store and WAL
//                            regions the frame reserves (every entry as if appended), sort keys
//   (CUB radix sort)         frame indices stably sorted by group: each group's frames in frame order
//   (engine.cu's scan)       store and WAL regions: exclusive scans in frame order
//   follower_cut_kernel      a thread per frame: the first frame in frame order whose region ends past a capacity
//   follower_replay_kernel   a thread per group segment: handle_msg_append_entries replayed in frame order over the
//                            group's state (term check, rejection and its conflict walk, truncation, appends, absorbs,
//                            commit walk); Metadata cells and reply cells
//   follower_copy_kernel     a warp per frame that appended: the LogEntry records, the shards into their padded store
//                            slots, the entries' store addresses
//
// A batch costs its largest per-group run of frames in the replay (a follower catching up on one group replays that
// group's frames serially on one thread); the copies take a warp per frame whatever the grouping.
//
//   append_reply_parse_kernel  a thread per AppendEntriesReply frame: the records ss_engine_raft_ingest takes
//
// Execution of the committed entries (the walk in handle_msg_append_entries, craft/messages.rs:198-240):
//
//   (exec_walk.cuh, FolLog)  a thread per group: the entries the walk executes, their payload bytes, then the records
//                            and last_exec; a warp per record: get_data's bytes from the held shards, a missing data
//                            shard regenerated from the first d held ones
//
// Serving a new leader's Reconstruct reads (ss_follower_reconstruct_serve) is in craft_recon.cu; campaigns, votes and
// their tally (ss_follower_campaign / _vote / _tally) are in craft_election.cu.
#include <cub/device/device_radix_sort.cuh>

#include <cstring>
#include <new>

#include "codeword_wire.cuh"
#include "craft_frames.cuh"
#include "device_common.cuh"
#include "exec_walk.cuh"
#include "follower_state.hpp"
#include "gf256.hpp"
#include "ss_internal.hpp"
#include "wire_common.cuh"

namespace ssb {

constexpr int kFolThreads = 256;
constexpr uint64_t kTag = 1ull << 63;          // shard_addr of an entry appended by this call: its frame and shard tags

__global__ void __launch_bounds__(kFolThreads) follower_header_kernel(const __grid_constant__ FolArgs A) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kFolThreads;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kFolThreads + threadIdx.x; i < A.n; i += stride) {
        const FolHdr h = fol_decode(A, i);
        A.hdr[i] = h;
        const bool pending = h.kind == kPending;
        A.store_off[i] = pending ? h.store_sz : 0ull;
        A.wal_off[i] = pending ? h.wal_sz : 0ull;
        const uint32_t grp = A.frame_group[i];
        A.key_in[i] = grp < A.G ? grp : static_cast<uint32_t>(A.G);
        A.idx_in[i] = static_cast<uint32_t>(i);
    }
}

// the capacity cut: key = 2 * (first frame whose region ends past a capacity) + (1 when only its WAL region does)
__global__ void __launch_bounds__(kFolThreads) follower_cut_kernel(const __grid_constant__ FolArgs A) {
    if (blockIdx.x == 0 && threadIdx.x == 0) *A.abs_cursor = A.tot[0];    // absorbed entries go after every region
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kFolThreads;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kFolThreads + threadIdx.x; i < A.n; i += stride) {
        const FolHdr &h = A.hdr[i];
        if (h.kind != kPending) continue;
        const uint64_t so = A.store_off[i], wo = A.wal_off[i];
        const bool s_over = so > A.store_cap || h.store_sz > A.store_cap - so;
        const bool w_over = wo > A.wal_cap || h.wal_sz > A.wal_cap - wo;
        if (s_over || w_over)
            atomicMin(reinterpret_cast<unsigned long long *>(A.cut), static_cast<unsigned long long>(2u * i + (s_over ? 0u : 1u)));
    }
}

// PeerMessage::Msg{AppendEntriesReply{term, end_slot, conflict}} into a 48-byte cell (at most 47 bytes)
__device__ __forceinline__ uint32_t put_reply(uint8_t *cell, uint32_t variant, uint64_t term, uint64_t end_slot, bool conflict,
                                              uint64_t c_term, uint64_t c_slot) {
    uint32_t m = 8u;
    m += wv_put(cell + m, 0u);
    m += wv_put(cell + m, variant);
    m += wv_put(cell + m, term);
    m += wv_put(cell + m, end_slot);
    cell[m++] = conflict ? 1u : 0u;
    if (conflict) {
        m += wv_put(cell + m, c_term);
        m += wv_put(cell + m, c_slot);
    }
    put_be64(cell, m - 8u);
    return m;
}

// the bytes of shard j (present in `present`) among the T shard Options starting at tags
__device__ __forceinline__ const uint8_t *shard_in_frame(const uint8_t *tags, uint32_t j, uint32_t present, uint64_t L) {
    uint64_t at = 0;
    for (uint32_t q = 0; q <= j; ++q) {
        if (!((present >> q) & 1u)) { at += 1u; continue; }
        const uint64_t sl = some_len(tags[at + 1u]);
        if (q == j) return tags + at + sl;
        at += sl + L;
    }
    return nullptr;
}

// absorb_other (messages.rs:143-154) on one thread: the union of the held shards and the frame's into a new region at
// dst (shard j at its rank in the union, bytes L..round_up(L,16) zero).  The held shards come from the caller's store,
// or -- for an entry this call appended, whose slots the copy pass has not written yet -- from its own frame.
__device__ void absorb_copy(const FolArgs &A, uint8_t *dst, uint64_t old_addr, uint32_t old_held, const uint8_t *new_tags,
                            uint32_t new_held, uint64_t L) {
    const uint64_t pitch = SS_CW_SLOT_PITCH(L), padded = round16(L);
    const uint32_t uni = old_held | new_held;
    const uint8_t *old_tags = nullptr;
    if (old_addr & kTag) {
        const uint64_t fi = (old_addr >> 32) & 0x7fffffffull;
        old_tags = A.buf + A.frame_off[fi] + (old_addr & 0xffffffffull);
    }
    for (uint32_t j = 0; j < A.T; ++j) {
        if (!((uni >> j) & 1u)) continue;
        uint8_t *out = dst + static_cast<uint64_t>(__popc(uni & ((1u << j) - 1u))) * pitch;
        const uint8_t *src;
        if ((old_held >> j) & 1u)
            src = old_tags != nullptr ? shard_in_frame(old_tags, j, old_held, L)
                                      : reinterpret_cast<const uint8_t *>(old_addr) + static_cast<uint64_t>(__popc(old_held & ((1u << j) - 1u))) * pitch;
        else
            src = shard_in_frame(new_tags, j, new_held, L);
        for (uint64_t q = 0; q < L; ++q) out[q] = src[q];
        for (uint64_t q = L; q < padded; ++q) out[q] = 0u;
    }
}

// a thread per group segment: every frame of the group in frame order, as handle_msg_append_entries meets them
__global__ void __launch_bounds__(kFolThreads) follower_replay_kernel(const __grid_constant__ FolArgs A) {
    bool abs_full = false, cut_store = false, cut_wal = false;
    const uint64_t cut = *A.cut, cut_i = cut >> 1;
    const uint32_t cut_kind = (cut & 1u) ? SS_FOLLOWER_VERDICT_WAL_FULL : SS_FOLLOWER_VERDICT_STORE_FULL;
    const uint32_t dmask = A.d >= 32u ? 0xffffffffu : (1u << A.d) - 1u;
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kFolThreads;
    for (uint64_t t = static_cast<uint64_t>(blockIdx.x) * kFolThreads + threadIdx.x; t < A.n; t += stride) {
        if (t != 0u && A.key[t] == A.key[t - 1]) continue;
        const uint32_t g = A.key[t];
        uint64_t e_end = t + 1u;
        while (e_end < A.n && A.key[e_end] == g) ++e_end;
        const bool known = g < A.G;
        const uint64_t row = static_cast<uint64_t>(known ? g : 0u) * A.W, wm = A.W - 1u;
        uint64_t start = 0, le = 0, ct = 0, lc = 0, ls = 0;
        uint32_t ldr = 0xffu;
        if (known) {
            start = A.start_slot[g]; le = A.log_end[g]; ct = A.curr_term[g]; lc = A.last_commit[g]; ls = A.last_snap[g];
            ldr = A.leader[g];
        }
        for (uint64_t k = t; k < e_end; ++k) {
            const uint32_t i = A.idx[k];
            FolHdr h = A.hdr[i];
            uint32_t kind = h.kind;
            A.meta_len[i] = 0u;
            A.reply_len[i] = 0u;
            A.reply_dst[i] = 0xffu;
            A.trunc_slot[i] = ~0ull;
            A.wal_len[i] = 0u;
            if (kind == kPending && i >= cut_i) {
                kind = cut_kind;
                cut_store |= kind == SS_FOLLOWER_VERDICT_STORE_FULL;
                cut_wal |= kind == SS_FOLLOWER_VERDICT_WAL_FULL;
            }
            if (kind != kPending) {
                A.verdict[i] = kind;
                A.store_off[i] = ~0ull;
                A.wal_off[i] = ~0ull;
                continue;
            }
            const uint8_t peer = A.frame_peer[i];
            // check_term: a higher term is adopted (voted_for None) and made durable before anything else
            if (h.term > ct) {
                ct = h.term;
                uint8_t *cell = A.meta + static_cast<uint64_t>(i) * 32u;
                uint32_t m = 8u;
                m += wv_put(cell + m, A.meta_variant);
                m += wv_put(cell + m, ct);
                cell[m++] = 0xffu;                                           // voted_for: None = ReplicaId::MAX
                put_be64(cell, m - 8u);
                for (uint32_t q = m; q < 32u; ++q) cell[q] = 0u;
                A.meta_len[i] = m;
                ldr = peer;
            }
            if (h.term == ct) ldr = peer;                                   // messages.rs:86-97
            const uint64_t end_slot = h.prev + h.n_ent;
            if (h.term < ct || h.prev < start || h.prev >= le || A.term[row + (h.prev & wm)] != h.prev_term) {
                // messages.rs:47-78: the conflicting entry's term and the first slot of that term
                const bool inside = h.prev >= start && h.prev < le;
                const uint64_t c_term = inside ? A.term[row + (h.prev & wm)] : 0ull;
                uint64_t c_slot = h.prev;
                while (c_term > 0u && c_slot > start && A.term[row + ((c_slot - 1u) & wm)] == c_term) --c_slot;
                A.reply_len[i] = put_reply(A.replies + static_cast<uint64_t>(i) * 48u, A.reply_variant, ct, end_slot, true, c_term, c_slot);
                A.reply_dst[i] = peer;
                A.verdict[i] = SS_FOLLOWER_VERDICT_REJECTED;
                A.store_off[i] = ~0ull;
                A.wal_off[i] = ~0ull;
                if (h.snap > ls) ls = h.snap;
                continue;
            }
            // accepted: truncate at the first conflicting entry, append from there, absorb matching entries' shards
            const uint8_t *fr = A.buf + A.frame_off[i];
            const uint64_t fend = 8u + [&] { uint64_t x = 0; for (int b = 0; b < 8; ++b) x = (x << 8) | fr[b]; return x; }();
            uint64_t at = h.ents_at, wl = 0, first_k = h.n_ent;
            for (uint64_t q = 0; q < h.n_ent; ++q) {
                Ent e;
                ent_parse(fr, fend, at, A.d, A.T, e);
                const uint64_t s = h.prev + 1u + q, pos = row + (s & wm);
                if (first_k == h.n_ent) {
                    if (s < le && A.term[pos] != e.term) {
                        A.trunc_slot[i] = s;                                 // LogAction::Truncate at this slot's offset
                        le = s;
                    }
                    if (s >= le) first_k = q;
                }
                if (first_k != h.n_ent) {
                    A.term[pos] = e.term;
                    A.held[pos] = e.held;
                    A.data_len[pos] = static_cast<uint32_t>(e.dl);
                    A.shard_addr[pos] = kTag | (static_cast<uint64_t>(i) << 32) | e.tags_at;
                    le = s + 1u;
                    wl += round16(ent_rec_len(e, A.log_variant));
                } else {
                    const uint32_t oh = A.held[pos];
                    if (static_cast<uint32_t>(__popc(oh & dmask)) < A.d && A.data_len[pos] == e.dl && oh != e.held) {
                        const uint64_t bytes = static_cast<uint64_t>(__popc(oh | e.held)) * SS_CW_SLOT_PITCH(e.sl);
                        const uint64_t ao = atomicAdd(reinterpret_cast<unsigned long long *>(A.abs_cursor), static_cast<unsigned long long>(bytes));
                        if (ao > A.store_cap || bytes > A.store_cap - ao) {
                            abs_full = true;                                 // the entry keeps the shards it holds
                        } else {
                            absorb_copy(A, A.store + ao, A.shard_addr[pos], oh, fr + e.tags_at, e.held, e.sl);
                            A.held[pos] = oh | e.held;
                            A.shard_addr[pos] = reinterpret_cast<uint64_t>(A.store + ao);
                        }
                    }
                }
                at = e.next;
            }
            A.hdr[i].first_k = first_k;
            A.verdict[i] = SS_FOLLOWER_VERDICT_ACCEPTED;
            if (first_k == h.n_ent) {                                       // nothing appended: the reply goes now
                A.store_off[i] = ~0ull;
                A.wal_off[i] = ~0ull;
                A.reply_dst[i] = peer;
            } else {
                A.wal_len[i] = wl;
            }
            A.reply_len[i] = put_reply(A.replies + static_cast<uint64_t>(i) * 48u, A.reply_variant, ct, end_slot, false, 0u, 0u);
            // commit walk (messages.rs:198-244): stops at an entry holding fewer than majority shards.  Its cap is
            // prev_slot + entries.len() after the append loop drained entries[first_new - prev_slot - 1 ..], i.e.
            // first_new - 1: the last slot the frame matched, never one it appended (prev_slot when nothing was appended)
            if (h.commit > lc) {
                const uint64_t cap = h.prev + (first_k == h.n_ent ? 0u : first_k);
                uint64_t nc = h.commit < cap ? h.commit : cap;
                nc = nc < le - 1u ? nc : le - 1u;
                for (uint64_t s = lc + 1u; s <= nc; ++s) {
                    if (static_cast<uint32_t>(__popc(A.held[row + (s & wm)])) < A.d) break;
                    lc = s;
                }
            }
            if (h.snap > ls) ls = h.snap;
        }
        if (!known) continue;
        // the success replies go to the leader as the whole call left it
        for (uint64_t k = t; k < e_end; ++k) {
            const uint32_t i = A.idx[k];
            if (A.verdict[i] == SS_FOLLOWER_VERDICT_ACCEPTED && A.wal_len[i] != 0u) A.reply_dst[i] = ldr;
        }
        A.log_end[g] = le; A.curr_term[g] = ct; A.last_commit[g] = lc; A.last_snap[g] = ls; A.leader[g] = ldr;
    }
    if (abs_full || cut_store) atomicOr(A.status, SS_DEV_STATUS_STORE_FULL);
    if (cut_wal) atomicOr(A.status, SS_DEV_STATUS_FRAME_OVERFLOW);
}

// a warp per frame that appended: its LogEntry records one after the other from wal_off, its shards one entry after the
// other from store_off, and the entries' store addresses
__global__ void __launch_bounds__(kFolThreads) follower_copy_kernel(const __grid_constant__ FolArgs A) {
    if (blockIdx.x == 0 && threadIdx.x == 0) A.tot[0] = *A.abs_cursor;    // the store bytes asked for, absorbs included
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = (static_cast<uint64_t>(blockIdx.x) * kFolThreads + threadIdx.x) >> 5;
    const uint64_t nwarps = (static_cast<uint64_t>(gridDim.x) * kFolThreads) >> 5;
    const uint32_t wvl = static_cast<uint32_t>(wv_len(A.log_variant));
    for (uint64_t i = warp; i < A.n; i += nwarps) {
        if (A.verdict[i] != SS_FOLLOWER_VERDICT_ACCEPTED || A.wal_len[i] == 0u) continue;
        const FolHdr h = A.hdr[i];
        const uint8_t *fr = A.buf + A.frame_off[i];
        uint64_t fend = 0;
        for (int b = 0; b < 8; ++b) fend = (fend << 8) | fr[b];
        fend += 8u;
        const uint64_t row = static_cast<uint64_t>(A.frame_group[i]) * A.W, wm = A.W - 1u;
        uint64_t at = h.ents_at, wo = A.wal_off[i], so = A.store_off[i];
        for (uint64_t q = 0; q < h.n_ent; ++q) {
            Ent e;
            ent_parse(fr, fend, at, A.d, A.T, e);
            if (q >= h.first_k) {
                // DurEntry::LogEntry: length, log_variant, the entry from term through external as it came, log_offset 0
                uint8_t *rec = A.wal + wo;
                const uint64_t body = ent_rec_len(e, A.log_variant) - 8u, span = e.ext_end - e.start;
                if (lane == 0u) {
                    put_be64(rec, body);
                    wv_put(rec + 8, A.log_variant);
                    rec[8u + wvl + span] = 0u;
                }
                warp_copy_unaligned(rec + 8u + wvl, fr + e.start, span, lane);
                warp_fill_shards(A.store + so, fr + e.tags_at, A.T, e.held, e.held, static_cast<uint32_t>(e.sl), lane);
                const uint64_t pos = row + ((h.prev + 1u + q) & wm);
                if (lane == 0u && A.shard_addr[pos] == (kTag | (i << 32) | e.tags_at))
                    A.shard_addr[pos] = reinterpret_cast<uint64_t>(A.store + so);
                wo += round16(8u + body);
                so += ent_store_bytes(e);
            }
            at = e.next;
        }
    }
}

// snapshot start_slot move: k = clamp(upto - start_slot, 0, last_commit - start_slot)
__global__ void __launch_bounds__(kFolThreads)
follower_advance_kernel(const uint64_t *__restrict__ upto, uint64_t G, uint64_t *__restrict__ start_slot,
                        const uint64_t *__restrict__ last_commit) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kFolThreads;
    for (uint64_t g = static_cast<uint64_t>(blockIdx.x) * kFolThreads + threadIdx.x; g < G; g += stride) {
        const uint64_t s = start_slot[g], u = upto[g], lc = last_commit[g];
        const uint64_t lim = lc > s ? lc : s;
        start_slot[g] = u <= s ? s : (u < lim ? u : lim);
    }
}

// ---- execution -----------------------------------------------------------------------------------------------------
// the walk in handle_msg_append_entries (exec_walk.cuh), from max(last_exec + 1, start_slot): stop past last_commit, or
// at fewer than d shards held, which the commit walk already excludes but state a host installed may hold; stop at a
// null entry, which get_data refuses (rscoding.rs:581-583).  A held shard of rank k is at shard_addr + k *
// SS_CW_SLOT_PITCH(L), the store layout of the append.
struct FolLog {
    uint32_t W, d;
    const uint64_t *start_slot, *last_commit, *shard_addr;
    const uint32_t *held, *data_len;
    uint64_t *last_exec;

    struct Walk { uint64_t s; };
    static constexpr bool kTables = true, kByIndex = false;

    __device__ __forceinline__ bool live(uint64_t) const { return true; }
    __device__ __forceinline__ Walk start(uint64_t g) const {
        const uint64_t s = last_exec[g] + 1u, st = start_slot[g];
        return {s > st ? s : st};
    }
    __device__ __forceinline__ uint32_t next(const Walk &, uint64_t g, uint64_t s, uint32_t *dlen) const {
        if (s > last_commit[g]) return kExecStop;
        const uint64_t pos = g * W + (s & (W - 1u));
        if (static_cast<uint32_t>(__popc(held[pos])) < d) return kExecStop;
        *dlen = data_len[pos];
        return *dlen == 0u ? kExecNull : kExecRun;
    }
    __device__ __forceinline__ void finish(uint64_t g, uint64_t s) const { last_exec[g] = s - 1u; }
    __device__ __forceinline__ ExecSrc source(uint64_t g, uint64_t s, uint32_t dlen) const {
        const uint64_t pos = g * W + (s & (W - 1u));
        return {held[pos], reinterpret_cast<const uint8_t *>(shard_addr[pos]), SS_CW_SLOT_PITCH((dlen + d - 1u) / d)};
    }
};

// the leader's side: PeerMessage::Msg{AppendEntriesReply{term, end_slot, conflict}} frames -> ingest records
struct ReplyParseArgs {
    const uint8_t *buf;
    uint64_t buf_len;
    const uint64_t *frame_off;
    const uint32_t *frame_group;
    const uint8_t *frame_peer;
    const uint32_t *curr_term;
    uint64_t n, G;
    uint32_t reply_variant;
    uint32_t *rec_group;
    uint8_t *rec_peer;
    uint32_t *rec_end_slot;
    uint64_t *rec_term, *rec_conflict_term, *rec_conflict_slot;
    uint32_t *rec_kind;
};

__global__ void __launch_bounds__(kFolThreads) append_reply_parse_kernel(const __grid_constant__ ReplyParseArgs A) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kFolThreads;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kFolThreads + threadIdx.x; i < A.n; i += stride) {
        uint64_t term = 0, end = 0, c_term = 0, c_slot = 0;
        const uint32_t grp = A.frame_group[i];
        const uint64_t off = A.frame_off[i];
        const uint32_t kind = reply_parse(A.buf, A.buf_len, off, grp, A.G, A.reply_variant, A.curr_term, term, end, c_term, c_slot);
        if (kind < SS_APPEND_REPLY_INGEST || kind > SS_APPEND_REPLY_END_RANGE) term = end = c_term = c_slot = 0u;   // not decoded
        const bool ok = kind == SS_APPEND_REPLY_INGEST;
        A.rec_group[i] = ok ? grp : 0xffffffffu;
        A.rec_peer[i] = ok ? A.frame_peer[i] : 0xffu;
        A.rec_end_slot[i] = ok ? static_cast<uint32_t>(end) : 0u;
        A.rec_term[i] = term;
        A.rec_conflict_term[i] = c_term;
        A.rec_conflict_slot[i] = c_slot;
        A.rec_kind[i] = kind;
    }
}

int fol_scratch(ss_follower *f, uint64_t n) {
    if (n <= f->cap_frames) return SS_OK;
    ss_ctx *ctx = f->ctx;
    SS_CUDA(cudaStreamSynchronize(ctx->stream));
    void *old[] = {f->hdr, f->keys, f->idx, f->partials, f->sort_tmp};
    for (void *b : old)
        if (b) cudaFree(b);
    f->hdr = nullptr; f->keys = nullptr; f->idx = nullptr; f->partials = nullptr; f->sort_tmp = nullptr;
    f->cap_frames = 0;
    SS_TRY(dalloc(ctx, &f->hdr, n, false));
    SS_TRY(dalloc(ctx, &f->keys, 2 * n, false));
    SS_TRY(dalloc(ctx, &f->idx, 2 * n, false));
    SS_TRY(dalloc(ctx, &f->partials, scan_tiles(n), false));
    size_t bytes = 0;
    SS_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, bytes, f->keys, f->keys + n, f->idx, f->idx + n, static_cast<int>(n), 0,
                                            key_bits(f->G), ctx->stream));
    SS_CUDA(cudaMalloc(&f->sort_tmp, bytes ? bytes : 1));
    f->sort_tmp_bytes = bytes;
    f->cap_frames = n;
    return SS_OK;
}

// one group's state at creation: recovery's slot-0 null entry (craft/recovery.rs:99-125), no leader
__global__ void follower_init_kernel(uint64_t G, uint64_t *log_end, uint8_t *leader) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
    for (uint64_t g = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; g < G; g += stride) {
        log_end[g] = 1u;
        leader[g] = 0xffu;
    }
}

}  // namespace ssb

using namespace ssb;

extern "C" {

int ss_follower_destroy(ss_follower *f) {
    if (f == nullptr) return SS_OK;
    if (f->ctx) {
        cudaSetDevice(f->ctx->device);
        cudaStreamSynchronize(f->ctx->stream);
    }
    void *bufs[] = {f->start_slot, f->log_end, f->curr_term, f->last_commit, f->last_snap, f->leader, f->term, f->shard_addr,
                    f->held, f->data_len, f->last_exec, f->matrix, f->ex_cnt, f->ex_bytes, f->ex_partials, f->ex_words, f->hdr,
                    f->keys, f->idx, f->partials, f->sort_tmp, f->words, f->vote_term, f->role_term, f->voted_for, f->role,
                    f->votes, f->won_flag};
    for (void *b : bufs)
        if (b) cudaFree(b);
    if (f->ctx) ctx_release(f->ctx);
    delete f;
    return SS_OK;
}

int ss_follower_create(ss_ctx *ctx, const ss_follower_config *cfg, uint64_t G, ss_follower **out) {
    if (out == nullptr) return set_error(SS_ERR_INVALID_ARG, "null out pointer");
    *out = nullptr;
    if (cfg == nullptr || G == 0) return set_error(SS_ERR_INVALID_ARG, "null config or zero groups");
    if (G > 0xffffffffull) return set_error(SS_ERR_INVALID_ARG, "at most 2^32 - 1 groups");
    if (cfg->protocol != SS_PROTO_CRAFT) return set_error(SS_ERR_INVALID_ARG, "the follower serves CRaft, not protocol %u", cfg->protocol);
    if (cfg->population == 0 || cfg->population > 32 || cfg->me >= cfg->population)
        return set_error(SS_ERR_INVALID_ARG, "bad population %u / me %u", cfg->population, cfg->me);
    // a ring of one entry holds only start_slot, so no entry could ever be appended: the window filter refuses every slot
    // past start_slot, nothing commits, and start_slot can never move
    const uint32_t W = cfg->window ? cfg->window : 64u;
    if (W < 2u || (W & (W - 1u)) || W > 4096u)
        return set_error(SS_ERR_INVALID_ARG, "window must be a power of two in 2..4096 (got %u)", cfg->window);
    // a reply is at most 8 + 1 + wv_len(reply_variant) + 9 + 9 + 1 + 9 + 9 bytes: one-byte variants fill at most 47 of its
    // 48-byte cell; a Metadata record at most 8 + 3 + 9 + 1 of its 32
    if (cfg->reply_variant >= 251u || cfg->meta_variant >= 65536u || cfg->append_variant >= 65536u || cfg->log_variant >= 65536u)
        return set_error(SS_ERR_INVALID_ARG, "reply_variant must be < 251, the other variants < 2^16");
    if (ctx == nullptr) {
        int count = 0;
        const cudaError_t e = cudaGetDeviceCount(&count);
        cudaGetLastError();
        if (e != cudaSuccess || count == 0) return set_error(SS_ERR_NO_DEVICE, "no CUDA device available; this library has no CPU fallback");
        return set_error(SS_ERR_INVALID_ARG, "null context");
    }
    SS_TRY(ctx_bind(ctx));
    ss_follower *f = new (std::nothrow) ss_follower();
    if (!f) return set_error(SS_ERR_OUT_OF_MEMORY, "host allocation failed");
    f->ctx = ctx; f->cfg = *cfg; f->G = G; f->W = W;
    f->d = cfg->population / 2u + 1u;                                       // craft/mod.rs:527-536: (majority, n - majority)
    f->T = cfg->population;
    ctx_retain(ctx);
    int rc = SS_OK;
    if ((rc = dalloc(ctx, &f->start_slot, G)) || (rc = dalloc(ctx, &f->log_end, G)) || (rc = dalloc(ctx, &f->curr_term, G)) ||
        (rc = dalloc(ctx, &f->last_commit, G)) || (rc = dalloc(ctx, &f->last_snap, G)) || (rc = dalloc(ctx, &f->leader, G)) ||
        (rc = dalloc(ctx, &f->term, G * W)) || (rc = dalloc(ctx, &f->shard_addr, G * W)) ||
        (rc = dalloc(ctx, &f->held, G * W)) || (rc = dalloc(ctx, &f->data_len, G * W)) || (rc = dalloc(ctx, &f->words, 4)) ||
        (rc = dalloc(ctx, &f->last_exec, G)) || (rc = dalloc(ctx, &f->matrix, size_t(f->T) * f->d, false)) ||
        (rc = dalloc(ctx, &f->ex_cnt, G, false)) || (rc = dalloc(ctx, &f->ex_bytes, G, false)) ||
        (rc = dalloc(ctx, &f->ex_partials, scan_tiles(G), false)) || (rc = dalloc(ctx, &f->ex_words, 3, false))) {
        ss_follower_destroy(f);
        return rc;
    }
    // the coder's matrix, whose rows ss_follower_execute inverts on the device; a pageable source is staged before the
    // call returns
    const gf::Matrix m = gf::coding_matrix(static_cast<int>(f->d), static_cast<int>(f->T - f->d));
    if (cudaMemcpyAsync(f->matrix, m.v.data(), m.v.size(), cudaMemcpyHostToDevice, ctx->stream) != cudaSuccess) {
        ss_follower_destroy(f);
        return set_error(SS_ERR_CUDA, "coding matrix upload failed");
    }
    follower_init_kernel<<<launch_grid(ctx, G, kFolThreads), kFolThreads, 0, ctx->stream>>>(G, f->log_end, f->leader);
    if ((rc = launched(ctx)) != SS_OK) {
        ss_follower_destroy(f);
        return rc;
    }
    *out = f;
    return SS_OK;
}

int ss_follower_view_get(ss_follower *f, ss_follower_view *v) {
    if (f == nullptr || v == nullptr) return set_error(SS_ERR_INVALID_ARG, "null argument");
    memset(v, 0, sizeof(*v));
    v->n_groups = f->G; v->protocol = f->cfg.protocol; v->population = f->cfg.population; v->me = f->cfg.me;
    v->data_shards = f->d; v->total_shards = f->T; v->window = f->W;
    v->start_slot = f->start_slot; v->log_end = f->log_end; v->curr_term = f->curr_term; v->last_commit = f->last_commit;
    v->last_snap = f->last_snap; v->leader = f->leader; v->term = f->term; v->shard_addr = f->shard_addr; v->held = f->held;
    v->data_len = f->data_len;
    return SS_OK;
}

int ss_follower_advance(ss_follower *f, const uint64_t *upto) {
    if (f == nullptr || upto == nullptr) return set_error(SS_ERR_INVALID_ARG, "null follower or upto");
    ss_ctx *ctx = f->ctx;
    SS_TRY(ctx_bind(ctx));
    follower_advance_kernel<<<launch_grid(ctx, f->G, kFolThreads), kFolThreads, 0, ctx->stream>>>(upto, f->G, f->start_slot, f->last_commit);
    return launched(ctx);
}

int ss_follower_exec_view_get(ss_follower *f, ss_follower_exec_view *v) {
    if (f == nullptr || v == nullptr) return set_error(SS_ERR_INVALID_ARG, "null argument");
    memset(v, 0, sizeof(*v));
    v->n_groups = f->G;
    v->last_exec = f->last_exec;
    return SS_OK;
}

int ss_follower_execute(ss_follower *f, uint8_t *out, uint64_t out_capacity, uint32_t *rec_group, uint64_t *rec_slot, uint64_t *rec_off,
                        uint32_t *rec_len, uint64_t rec_capacity, uint64_t *totals) {
    if (f == nullptr) return set_error(SS_ERR_INVALID_ARG, "null follower");
    if (!out || !rec_group || !rec_slot || !rec_off || !rec_len) return set_error(SS_ERR_INVALID_ARG, "null buffer");
    if (reinterpret_cast<uintptr_t>(out) & 15u) return set_error(SS_ERR_INVALID_ARG, "out must be 16-byte aligned");
    ss_ctx *ctx = f->ctx;
    SS_TRY(ctx_bind(ctx));
    const ExecOut o{f->matrix, f->ex_cnt, f->ex_bytes, f->ex_words, out, out_capacity, rec_group, rec_slot, rec_off, rec_len,
                    rec_capacity, ctx->dev_status};
    const FolLog log{f->W, f->d, f->start_slot, f->last_commit, f->shard_addr, f->held, f->data_len, f->last_exec};
    return launch_execute(ctx, o, log, log, f->G, f->G * f->W, f->ex_partials, totals != nullptr ? totals : f->ex_words + 1);
}

int ss_follower_append(ss_follower *f, const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off, const uint32_t *frame_group,
                       const uint8_t *frame_peer, uint64_t n, uint8_t *store, uint64_t store_capacity, uint64_t *store_off,
                       uint8_t *wal, uint64_t wal_capacity, uint64_t *wal_off, uint64_t *wal_len, uint8_t *meta, uint32_t *meta_len,
                       uint8_t *replies, uint32_t *reply_len, uint8_t *reply_dst, uint64_t *trunc_slot, uint32_t *verdict,
                       uint64_t *commit_lo, uint64_t *totals) {
    if (f == nullptr) return set_error(SS_ERR_INVALID_ARG, "null follower");
    ss_ctx *ctx = f->ctx;
    SS_TRY(ctx_bind(ctx));
    if (n == 0) {
        if (totals != nullptr) SS_CUDA(cudaMemsetAsync(totals, 0, 16, ctx->stream));
        if (commit_lo != nullptr) SS_CUDA(cudaMemcpyAsync(commit_lo, f->last_commit, f->G * 8, cudaMemcpyDeviceToDevice, ctx->stream));
        return SS_OK;
    }
    if (!buf || !frame_off || !frame_group || !frame_peer || !store || !store_off || !wal || !wal_off || !wal_len || !meta ||
        !meta_len || !replies || !reply_len || !reply_dst || !trunc_slot || !verdict)
        return set_error(SS_ERR_INVALID_ARG, "null buffer");
    if ((reinterpret_cast<uintptr_t>(store) | reinterpret_cast<uintptr_t>(wal)) & 15u)
        return set_error(SS_ERR_INVALID_ARG, "store and wal must be 16-byte aligned");
    if (n > 0x7fffffffull) return set_error(SS_ERR_INVALID_ARG, "at most 2^31 - 1 frames per call");
    SS_TRY(fol_scratch(f, n));
    if (commit_lo != nullptr) SS_CUDA(cudaMemcpyAsync(commit_lo, f->last_commit, f->G * 8, cudaMemcpyDeviceToDevice, ctx->stream));
    uint64_t *tot = totals != nullptr ? totals : f->words + 2;
    FolArgs A{};
    A.buf = buf; A.buf_len = buf_len; A.frame_off = frame_off; A.frame_group = frame_group; A.frame_peer = frame_peer;
    A.n = n; A.G = f->G; A.d = f->d; A.T = f->T; A.W = f->W; A.me = f->cfg.me; A.population = f->cfg.population;
    A.append_variant = f->cfg.append_variant; A.reply_variant = f->cfg.reply_variant; A.meta_variant = f->cfg.meta_variant;
    A.log_variant = f->cfg.log_variant;
    A.start_slot = f->start_slot; A.log_end = f->log_end; A.curr_term = f->curr_term; A.last_commit = f->last_commit;
    A.last_snap = f->last_snap; A.leader = f->leader; A.term = f->term; A.shard_addr = f->shard_addr; A.held = f->held;
    A.data_len = f->data_len;
    A.hdr = f->hdr; A.key_in = f->keys; A.idx_in = f->idx; A.key = f->keys + n; A.idx = f->idx + n;
    A.cut = f->words; A.abs_cursor = f->words + 1; A.tot = tot;
    A.store = store; A.store_cap = store_capacity; A.store_off = store_off;
    A.wal = wal; A.wal_cap = wal_capacity; A.wal_off = wal_off; A.wal_len = wal_len;
    A.meta = meta; A.meta_len = meta_len; A.replies = replies; A.reply_len = reply_len; A.reply_dst = reply_dst;
    A.trunc_slot = trunc_slot; A.verdict = verdict; A.status = ctx->dev_status;
    const uint32_t grid_t = launch_grid(ctx, n, kFolThreads);
    SS_CUDA(cudaMemsetAsync(f->words, 0xff, 8, ctx->stream));
    follower_header_kernel<<<grid_t, kFolThreads, 0, ctx->stream>>>(A);
    SS_TRY(launched(ctx));
    size_t bytes = f->sort_tmp_bytes;
    SS_CUDA(cub::DeviceRadixSort::SortPairs(f->sort_tmp, bytes, f->keys, f->keys + n, f->idx, f->idx + n, static_cast<int>(n), 0,
                                            key_bits(f->G), ctx->stream));
    SS_TRY(launched(ctx));
    SS_TRY(launch_exclusive_scan_u64(ctx, store_off, n, f->partials, tot));
    SS_TRY(launch_exclusive_scan_u64(ctx, wal_off, n, f->partials, tot + 1));
    follower_cut_kernel<<<grid_t, kFolThreads, 0, ctx->stream>>>(A);
    SS_TRY(launched(ctx));
    follower_replay_kernel<<<grid_t, kFolThreads, 0, ctx->stream>>>(A);
    SS_TRY(launched(ctx));
    follower_copy_kernel<<<launch_grid(ctx, n, kFolThreads / 32), kFolThreads, 0, ctx->stream>>>(A);
    return launched(ctx);
}

int ss_append_reply_parse_dev(ss_ctx *ctx, const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off, const uint32_t *frame_group,
                              const uint8_t *frame_peer, const uint32_t *curr_term, uint64_t n_frames, uint64_t n_groups,
                              uint32_t reply_variant, uint32_t *rec_group, uint8_t *rec_peer, uint32_t *rec_end_slot,
                              uint64_t *rec_term, uint64_t *rec_conflict_term, uint64_t *rec_conflict_slot, uint32_t *rec_kind) {
    // a frame's variant >= 2^16 is malformed, so no index from there on can name the reply (ss_engine_craft_backoff, which
    // takes the same reply_variant, refuses it too)
    if (reply_variant >= kVariantLimit) return set_error(SS_ERR_INVALID_ARG, "reply_variant must be < 2^16");
    if (ctx == nullptr) return set_error(SS_ERR_INVALID_ARG, "null context");
    SS_TRY(ctx_bind(ctx));
    if (n_frames == 0) return SS_OK;
    if (!buf || !frame_off || !frame_group || !frame_peer || !curr_term || !rec_group || !rec_peer || !rec_end_slot || !rec_term ||
        !rec_conflict_term || !rec_conflict_slot || !rec_kind)
        return set_error(SS_ERR_INVALID_ARG, "null buffer");
    ReplyParseArgs A;
    A.buf = buf; A.buf_len = buf_len; A.frame_off = frame_off; A.frame_group = frame_group; A.frame_peer = frame_peer;
    A.curr_term = curr_term; A.n = n_frames; A.G = n_groups; A.reply_variant = reply_variant;
    A.rec_group = rec_group; A.rec_peer = rec_peer; A.rec_end_slot = rec_end_slot; A.rec_term = rec_term;
    A.rec_conflict_term = rec_conflict_term; A.rec_conflict_slot = rec_conflict_slot; A.rec_kind = rec_kind;
    append_reply_parse_kernel<<<launch_grid(ctx, n_frames, kFolThreads), kFolThreads, 0, ctx->stream>>>(A);
    return launched(ctx);
}

}  // extern "C"
