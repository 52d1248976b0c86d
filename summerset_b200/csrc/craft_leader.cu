// craft_leader.cu -- the CRaft leader's log behind the C ABI (ss_engine_craft_*, ss_frame_append_pack_dev): request
// batches coded into the leader's log, AppendEntries frames out, conflict replies backed off.
//
//   ss_engine_craft_propose   handle_req_batch (craft/request.rs:70-116) for every group with a batch:
//     craft_propose_prepare_kernel  a thread per group: window check, slot pitch and WAL record length
//     (engine.cu's scan)            shard slots and WAL regions: exclusive scans in group order
//     craft_propose_commit_kernel   a thread per group: the capacity cuts, then the entry at log_end in curr_term
//     (ragged RS encoder)           from_data + compute_parity, one launch, into the caller's planes
//     craft_propose_wal_kernel      a warp per proposing group: its DurEntry::LogEntry record
//   ss_frame_append_pack_dev  handle_logged_leader_append (craft/durability.rs:12-127) or bcast_heartbeats
//                             (craft/leadership.rs:249-279) for every (peer, group) pair:
//     append_plan_kernel            a warp per pair: what goes out, its frames and region bytes (lanes over chunks)
//     (engine.cu's scan)            frame indices and byte offsets: exclusive scans in (peer, group) order
//     append_place_kernel           a warp per pair: the capacity cut, try_next, and each frame's offset and length
//     append_write_kernel           a warp per frame (its pair from frame_peer / frame_group): header varints, then each
//                                   entry with its shards copied from the store with 128-bit loads
//   ss_engine_craft_backoff   the conflict branch of handle_msg_append_entries_reply (craft/messages.rs:386-406):
//     backoff_key_kernel            a thread per reply frame: conflicts keyed by (group, peer)
//     (CUB radix sort)              stable: each pair's conflicts in frame order
//     backoff_walk_kernel           a thread per pair: the walk-back over the terms ring, try_next and want_end
//   ss_engine_craft_execute   the execution half of handle_msg_append_entries_reply's success branch (craft/messages.rs:316-359):
//     (exec_walk.cuh, CraftLog)     a thread per group: the entries the walk executes, their payload bytes, then the
//                                   records and last_exec
//     (exec_walk.cuh, CraftShards)  a warp per record: get_data's bytes gathered from the planes; after a step-up, a
//                                   missing data shard regenerated from the first d held ones
// Step-up, reconstruct reads and absorb, which fill the held masks below, are in craft_recon.cu.
//   ss_engine_craft_advance   the snapshot's start_slot move (craft/snapshot.rs:142,184)
#include <cub/device/device_radix_sort.cuh>

#include <cstring>
#include <new>

#include "codeword_wire.cuh"
#include "device_common.cuh"
#include "engine_state.hpp"
#include "exec_walk.cuh"
#include "gf256.hpp"
#include "ss_internal.hpp"
#include "wire_common.cuh"

namespace ssb {

constexpr int kClThreads = 256;
constexpr uint32_t kLogEntryVariant = 1u;          // DurEntry::LogEntry (craft/mod.rs:148-159: Metadata 0, LogEntry 1)

// one status write per warp, not one per flagged item
__device__ __forceinline__ void cl_warp_status(bool flag, uint32_t bit, uint32_t *status) {
    const unsigned any = __ballot_sync(__activemask(), flag);
    if (flag && (threadIdx.x & 31u) == static_cast<unsigned>(__ffs(static_cast<int>(any)) - 1)) atomicOr(status, bit);
}

// ---- propose -------------------------------------------------------------------------------------------------------
struct ProposeArgs {
    uint64_t G;
    uint32_t W, d, T, me, majority, full_copy;
    const uint32_t *data_len;
    const uint64_t *log_offset;
    uint8_t *shards;
    uint64_t plane_stride, wal_capacity;
    uint64_t *shard_off, *slot_out, *wal_off, *wal_len;
    uint8_t *wal;
    const uint64_t *log_start;
    uint32_t *log_end, *terms;
    const uint32_t *curr_term;
    uint32_t *ent_len, *held;
    uint64_t *ent_addr, *ent_log_offset;
    uint32_t *eff;
    uint64_t *rec_len;
    uint32_t *status;
    const uint8_t *led;             // read by the kLed instances only (ss_engine_craft_role_view)
};

__device__ __forceinline__ uint32_t own_mask(uint32_t full_copy, uint32_t majority, uint32_t replica) {
    return full_copy ? (1u << majority) - 1u : 1u << replica;
}

// the record of an entry of term t: length, DurEntry::LogEntry, term, the codeword, external, log_offset 0
__device__ __forceinline__ uint64_t wal_rec_len(uint32_t t, uint64_t dl, uint32_t d, uint32_t T, uint32_t nsh) {
    return 8u + wv_len(kLogEntryVariant) + wv_len(t) + cw_bytes(dl, d, T, nsh) + 2u;
}

// kLed: a group the engine does not lead is refused as a full window is, under SS_DEV_STATUS_NOT_LEADER
template <bool kLed>
__global__ void __launch_bounds__(kClThreads) craft_propose_prepare_kernel(const __grid_constant__ ProposeArgs A) {
    bool full = false, fenced = false;
    const uint32_t nsh = A.full_copy ? A.majority : 1u;
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kClThreads;
    for (uint64_t g = static_cast<uint64_t>(blockIdx.x) * kClThreads + threadIdx.x; g < A.G; g += stride) {
        uint32_t len = A.data_len[g];
        if (kLed && len != 0u && A.led[g] == 0u) {
            fenced = true;
            len = 0u;
        }
        // every slot of [log_start, log_end] must stay in the ring: the packer reads the terms of lagging peers' entries
        if (len != 0u && static_cast<uint64_t>(A.log_end[g]) + 1u - A.log_start[g] > A.W) {
            full = true;
            len = 0u;
        }
        A.eff[g] = len;
        A.shard_off[g] = len == 0u ? 0ull : SS_CW_SLOT_PITCH((static_cast<uint64_t>(len) + A.d - 1u) / A.d);
        const uint64_t rl = len == 0u ? 0ull : wal_rec_len(A.curr_term[g], len, A.d, A.T, nsh);
        A.rec_len[g] = rl;
        A.wal_off[g] = round16(rl);
    }
    cl_warp_status(full, SS_DEV_STATUS_RAFT_WINDOW_FULL, A.status);
    if (kLed) cl_warp_status(fenced, SS_DEV_STATUS_NOT_LEADER, A.status);
}

__global__ void __launch_bounds__(kClThreads) craft_propose_commit_kernel(const __grid_constant__ ProposeArgs A) {
    bool s_full = false, w_full = false;
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kClThreads;
    for (uint64_t g = static_cast<uint64_t>(blockIdx.x) * kClThreads + threadIdx.x; g < A.G; g += stride) {
        const uint32_t len = A.eff[g];
        const uint64_t off = A.shard_off[g], wo = A.wal_off[g], rl = A.rec_len[g];
        const uint64_t pitch = SS_CW_SLOT_PITCH((static_cast<uint64_t>(len) + A.d - 1u) / A.d);
        const bool s_over = len != 0u && (off > A.plane_stride || pitch > A.plane_stride - off);
        const bool w_over = len != 0u && (wo > A.wal_capacity || round16(rl) > A.wal_capacity - wo);
        if (len == 0u || s_over || w_over) {
            s_full |= s_over;
            w_full |= w_over;
            A.eff[g] = 0u;                                                  // the encode and the WAL pass skip it
            A.shard_off[g] = ~0ull;
            A.slot_out[g] = ~0ull;
            A.wal_off[g] = ~0ull;
            A.wal_len[g] = 0ull;
            continue;
        }
        // log.push at start_slot + log.len() in curr_term (request.rs:110-116)
        const uint32_t s = A.log_end[g];
        const uint64_t pos = g * A.W + (s & (A.W - 1u));
        A.terms[pos] = A.curr_term[g];
        A.ent_len[pos] = len;
        if (A.held != nullptr) A.held[pos] = A.T >= 32u ? 0xffffffffu : (1u << A.T) - 1u;   // every shard: the encode writes them all
        A.ent_addr[pos] = reinterpret_cast<uint64_t>(A.shards + off);
        A.ent_log_offset[pos] = A.log_offset != nullptr ? A.log_offset[g] : 0ull;
        A.log_end[g] = s + 1u;
        A.slot_out[g] = s;
        A.wal_len[g] = rl;
    }
    cl_warp_status(s_full, SS_DEV_STATUS_STORE_FULL, A.status);
    cl_warp_status(w_full, SS_DEV_STATUS_FRAME_OVERFLOW, A.status);
}

// a warp per proposing group: DurEntry::LogEntry{term, reqs_cw: subset_copy({me}) or {0..majority}, external: true,
// log_offset: 0} (request.rs:79-104)
__global__ void __launch_bounds__(kClThreads) craft_propose_wal_kernel(const __grid_constant__ ProposeArgs A) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = (static_cast<uint64_t>(blockIdx.x) * kClThreads + threadIdx.x) >> 5;
    const uint64_t nwarps = (static_cast<uint64_t>(gridDim.x) * kClThreads) >> 5;
    const uint32_t mask = own_mask(A.full_copy, A.majority, A.me);
    for (uint64_t g = warp; g < A.G; g += nwarps) {
        const uint32_t len = A.eff[g];
        if (len == 0u) continue;
        uint8_t *rec = A.wal + A.wal_off[g];
        const uint32_t t = A.curr_term[g];
        const uint64_t rl = A.wal_len[g];
        if (lane == 0u) {
            put_be64(rec, rl - 8u);
            const int m = 8 + wv_put(rec + 8, kLogEntryVariant);
            wv_put(rec + m, t);
        }
        const uint64_t m = 8u + wv_len(kLogEntryVariant) + wv_len(t);
        const uint64_t c = warp_put_cw(rec + m, A.d, A.T, len, mask, Planes{A.shards + A.shard_off[g], A.plane_stride}, lane);
        if (lane == 0u) {
            rec[m + c] = 1u;                                                // external: true
            rec[m + c + 1u] = 0u;                                           // log_offset: 0
        }
    }
}

// ---- AppendEntries packer ------------------------------------------------------------------------------------------
struct PackArgs {
    uint64_t G, PG;
    uint32_t P, W, d, T, me, majority, variant, chunk, full_copy, heartbeat;
    const uint64_t *want_end;
    const uint32_t *next_slot, *log_end, *curr_term, *terms, *last_commit, *last_snap;
    uint32_t *try_next;
    const uint64_t *log_start;
    const uint32_t *ent_len;
    const uint32_t *held;           // read by the kHeld instances only (after a step-up or the recon view)
    const uint64_t *ent_addr, *ent_log_offset;
    uint64_t plane_stride;
    uint8_t *out;
    uint64_t out_capacity, max_frames;
    uint64_t *frame_off, *frame_len;
    uint32_t *frame_group;
    uint8_t *frame_peer;
    uint64_t *n_frames, *total;
    uint32_t *pair_status;
    uint64_t *pk_frames, *pk_bytes, *pk_range, *frames_total;
    uint32_t *status;
    const uint8_t *led;             // read by the kLed instances only (ss_engine_craft_role_view)
};

// what goes to pair p = q*G + g: SENT with entries [lo, hi] (hi = lo - 1: a heartbeat), NOTHING or SNAPSHOTTED
struct PairPlan {
    uint32_t status, try_slot;
    uint64_t lo, hi, nf;
};

__device__ __forceinline__ uint32_t pair_try(const PackArgs &A, uint64_t p) {
    const uint32_t t = A.try_next[p], ns = A.next_slot[p];
    return t > ns ? t : ns;
}

__device__ __forceinline__ PairPlan plan_pair(const PackArgs &A, uint64_t p) {
    PairPlan r{SS_APPEND_PAIR_NOTHING, 0u, 0ull, 0ull, 0ull};
    const uint64_t g = p % A.G;
    const uint32_t t = pair_try(A, p);
    r.try_slot = t;
    const uint64_t le = A.log_end[g], ls = A.log_start[g];
    if (A.heartbeat) {
        // bcast_heartbeats: prev_slot = min(try_next_slot - 1, log end - 1)
        const uint64_t tm1 = t == 0u ? 0ull : t - 1ull;
        const uint64_t prev = tm1 < le - 1u ? tm1 : le - 1u;
        if (prev < ls) { r.status = SS_APPEND_PAIR_SNAPSHOTTED; return r; }
        r.status = SS_APPEND_PAIR_SENT;
        r.lo = prev + 1u;
        r.hi = prev;
        r.nf = 1u;
        return r;
    }
    uint64_t end = le - 1u;
    if (A.want_end != nullptr) {
        const uint64_t w = A.want_end[p];
        if (w == ~0ull) return r;
        end = w < end ? w : end;
    }
    if (t < 1u) return r;
    const uint64_t prev = t - 1ull;
    if (prev < ls) { r.status = SS_APPEND_PAIR_SNAPSHOTTED; return r; }
    if (prev >= le || end < t) return r;
    r.status = SS_APPEND_PAIR_SENT;
    r.lo = t;
    r.hi = end;
    r.nf = (end - t + A.chunk) / A.chunk;
    return r;
}

// the shards peer q's entries carry, before the held mask cuts them (subset_copy, rscoding.rs:255-293): the peer's
// own, or 0..majority in full copy
__device__ __forceinline__ uint32_t peer_want(const PackArgs &A, uint64_t q) {
    const uint32_t r = static_cast<uint32_t>(q) < A.me ? static_cast<uint32_t>(q) : static_cast<uint32_t>(q) + 1u;
    return own_mask(A.full_copy, A.majority, r);
}

// the shards of `want` the entry at ring position pos carries.  kHeld false: every entry holds every shard (a log that
// was never stepped up), and the pack kernels compile without the held loads
template <bool kHeld>
__device__ __forceinline__ uint32_t pack_mask(const PackArgs &A, uint64_t pos, uint32_t want) {
    return kHeld ? want & A.held[pos] : want;
}

// an entry's bytes; nsh: its shard count when every shard is held
template <bool kHeld>
__device__ __forceinline__ uint64_t ent_bytes(const PackArgs &A, uint64_t row, uint64_t s, uint32_t want, uint32_t nsh) {
    const uint64_t pos = row + (s & (A.W - 1u));
    if (kHeld) nsh = static_cast<uint32_t>(__popc(pack_mask<kHeld>(A, pos, want)));
    return wv_len(A.terms[pos]) + cw_bytes(A.ent_len[pos], A.d, A.T, nsh) + 1u + wv_len(A.ent_log_offset[pos]);
}

// chunk c of a plan: its first slot and entry count
__device__ __forceinline__ void chunk_span(const PackArgs &A, uint64_t lo, uint64_t hi, uint64_t c, uint64_t &first, uint64_t &n) {
    first = lo + c * A.chunk;
    const uint64_t last = hi < first + A.chunk - 1u ? hi : first + A.chunk - 1u;
    n = hi + 1u > first ? last + 1u - first : 0u;
}

// PeerMessage::Msg{AppendEntries{term, prev_slot, prev_term, entries, leader_commit, last_snap}} behind its length
template <bool kHeld>
__device__ __forceinline__ uint64_t frame_bytes(const PackArgs &A, uint64_t g, uint64_t first, uint64_t n, uint32_t want) {
    const uint64_t row = g * A.W, prev = first - 1u;
    const uint32_t nsh = A.full_copy ? A.majority : 1u;
    uint64_t b = 8u + 1u + wv_len(A.variant) + wv_len(A.curr_term[g]) + wv_len(prev) + wv_len(A.terms[row + (prev & (A.W - 1u))]) +
                 wv_len(n) + wv_len(A.last_commit[g]) + wv_len(A.last_snap[g]);
    for (uint64_t k = 0; k < n; ++k) b += ent_bytes<kHeld>(A, row, first + k, want, nsh);
    return b;
}

__device__ __forceinline__ uint64_t warp_sum(uint64_t v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// kLed: the pairs of a group the engine does not lead send nothing (SS_APPEND_PAIR_NOT_LEADER)
template <bool kHeld, bool kLed>
__global__ void __launch_bounds__(kClThreads) append_plan_kernel(const __grid_constant__ PackArgs A) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = (static_cast<uint64_t>(blockIdx.x) * kClThreads + threadIdx.x) >> 5;
    const uint64_t nwarps = (static_cast<uint64_t>(gridDim.x) * kClThreads) >> 5;
    for (uint64_t p = warp; p < A.PG; p += nwarps) {
        const PairPlan r = kLed && A.led[p % A.G] == 0u ? PairPlan{SS_APPEND_PAIR_NOT_LEADER, 0u, 0ull, 0ull, 0ull} : plan_pair(A, p);
        const uint64_t g = p % A.G;
        const uint32_t want = kHeld ? peer_want(A, p / A.G) : 0u;
        uint64_t bytes = 0;
        for (uint64_t c = lane; c < r.nf; c += 32u) {
            uint64_t first, n;
            chunk_span(A, r.lo, r.hi, c, first, n);
            bytes += round16(frame_bytes<kHeld>(A, g, first, n, want));
        }
        bytes = warp_sum(bytes);
        if (lane == 0u) {
            A.pk_frames[p] = r.nf;
            A.pk_bytes[p] = bytes;
            A.pk_range[p] = r.lo | (r.hi << 32);
            A.pair_status[p] = r.status;
        }
    }
}

// the cut, try_next, and the frame arrays of every pair written; a NOT_LEADER pair keeps its try_next
template <bool kHeld, bool kLed>
__global__ void __launch_bounds__(kClThreads) append_place_kernel(const __grid_constant__ PackArgs A) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = (static_cast<uint64_t>(blockIdx.x) * kClThreads + threadIdx.x) >> 5;
    const uint64_t nwarps = (static_cast<uint64_t>(gridDim.x) * kClThreads) >> 5;
    bool over = false;
    for (uint64_t p = warp; p < A.PG; p += nwarps) {
        const uint32_t st = A.pair_status[p];
        const uint32_t t = pair_try(A, p);
        if (st != SS_APPEND_PAIR_SENT) {
            if (lane == 0u && !(kLed && st == SS_APPEND_PAIR_NOT_LEADER)) A.try_next[p] = t;   // try_next >= next_slot from here on
            continue;
        }
        const uint64_t base = A.pk_frames[p], off = A.pk_bytes[p];
        const uint64_t nf_end = p + 1u < A.PG ? A.pk_frames[p + 1u] : *A.frames_total;
        const uint64_t end = p + 1u < A.PG ? A.pk_bytes[p + 1u] : *A.total;
        if (end > A.out_capacity || nf_end > A.max_frames) {
            over = true;
            if (lane == 0u) {
                A.pair_status[p] = SS_APPEND_PAIR_OVERFLOW;
                atomicMin(reinterpret_cast<unsigned long long *>(A.n_frames), static_cast<unsigned long long>(base));
            }
            continue;
        }
        const uint64_t rng = A.pk_range[p], lo = rng & 0xffffffffull, hi = rng >> 32;
        const uint64_t g = p % A.G;
        const uint32_t want = kHeld ? peer_want(A, p / A.G) : 0u;
        if (lane == 0u) A.try_next[p] = A.heartbeat ? t : static_cast<uint32_t>(hi + 1u);   // durability.rs:124-125
        uint64_t run = off;
        for (uint64_t c0 = 0; c0 < nf_end - base; c0 += 32u) {
            const uint64_t c = c0 + lane;
            uint64_t len = 0;
            if (c < nf_end - base) {
                uint64_t first, n;
                chunk_span(A, lo, hi, c, first, n);
                len = frame_bytes<kHeld>(A, g, first, n, want);
            }
            const uint64_t r = round16(len);
            uint64_t x = r;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint64_t y = __shfl_up_sync(0xffffffffu, x, o);
                if (lane >= static_cast<uint32_t>(o)) x += y;
            }
            if (c < nf_end - base) {
                A.frame_off[base + c] = run + x - r;
                A.frame_len[base + c] = len;
                A.frame_group[base + c] = static_cast<uint32_t>(g);
                A.frame_peer[base + c] = static_cast<uint8_t>(p / A.G);
            }
            run += __shfl_sync(0xffffffffu, x, 31);
        }
    }
    cl_warp_status(over, SS_DEV_STATUS_FRAME_OVERFLOW, A.status);
}

// a warp per written frame
template <bool kHeld>
__global__ void __launch_bounds__(kClThreads) append_write_kernel(const __grid_constant__ PackArgs A) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = (static_cast<uint64_t>(blockIdx.x) * kClThreads + threadIdx.x) >> 5;
    const uint64_t nwarps = (static_cast<uint64_t>(gridDim.x) * kClThreads) >> 5;
    const uint64_t nfr = *A.n_frames;
    for (uint64_t f = warp; f < nfr; f += nwarps) {
        // the place kernel wrote the frame's pair as (frame_peer, frame_group)
        const uint64_t g = A.frame_group[f], q = A.frame_peer[f], p = q * A.G + g;
        const uint64_t rng = A.pk_range[p], c = f - A.pk_frames[p];
        uint64_t first, n;
        chunk_span(A, rng & 0xffffffffull, rng >> 32, c, first, n);
        const uint64_t row = g * A.W, wm = A.W - 1u, prev = first - 1u;
        const uint32_t ct = A.curr_term[g], pt = A.terms[row + (prev & wm)];
        const uint32_t want = peer_want(A, q);
        uint8_t *fr = A.out + A.frame_off[f];
        if (lane == 0u) {
            put_be64(fr, A.frame_len[f] - 8u);
            uint64_t m = 8u;
            m += wv_put(fr + m, 0u);                                        // PeerMessage::Msg
            m += wv_put(fr + m, A.variant);
            m += wv_put(fr + m, ct);
            m += wv_put(fr + m, prev);
            m += wv_put(fr + m, pt);
            wv_put(fr + m, n);
        }
        uint64_t m = 9u + wv_len(A.variant) + wv_len(ct) + wv_len(prev) + wv_len(pt) + wv_len(n);
        for (uint64_t k = 0; k < n; ++k) {
            // LogEntry{term, reqs_cw: subset_copy({peer}) or {0..majority}, external: false, log_offset}; a shard the
            // leader does not hold goes out as None
            const uint64_t pos = row + ((first + k) & wm);
            const uint32_t et = A.terms[pos];
            const uint64_t lof = A.ent_log_offset[pos];
            if (lane == 0u) wv_put(fr + m, et);
            m += wv_len(et);
            m += warp_put_cw(fr + m, A.d, A.T, A.ent_len[pos], pack_mask<kHeld>(A, pos, want),
                             Planes{reinterpret_cast<const uint8_t *>(A.ent_addr[pos]), A.plane_stride}, lane);
            if (lane == 0u) {
                fr[m] = 0u;
                wv_put(fr + m + 1u, lof);
            }
            m += 1u + wv_len(lof);
        }
        if (lane == 0u) {
            m += wv_put(fr + m, A.last_commit[g]);
            wv_put(fr + m, A.last_snap[g]);
        }
    }
}

// ---- conflict back-off ---------------------------------------------------------------------------------------------
// PeerMessage::Msg{AppendEntriesReply{term, end_slot, conflict: Some((conflict_term, conflict_slot))}}
__device__ __forceinline__ bool conflict_decode(const uint8_t *buf, uint64_t buf_len, uint64_t off, uint32_t variant, uint64_t &end,
                                                uint64_t &c_term, uint64_t &c_slot) {
    const uint8_t *b;
    uint64_t len, n, term = 0;
    uint32_t kind;
    if (!msg_head(buf, buf_len, off, variant, ~0ull, true, b, len, n, kind)) return false;
    if (!wv_next(b, len, n, term) || !wv_next(b, len, n, end) || n >= len || b[n] != 1u) return false;
    ++n;
    return wv_next(b, len, n, c_term) && wv_next(b, len, n, c_slot) && n == len;
}

struct BackoffArgs {
    const uint8_t *buf;
    uint64_t buf_len;
    const uint64_t *frame_off;
    const uint32_t *frame_group;
    const uint8_t *frame_peer;
    const uint32_t *rec_kind;
    uint64_t n, G, PG;
    uint32_t P, W, variant;
    uint32_t *key_in, *idx_in;
    const uint32_t *key, *idx;
    uint32_t *next_slot, *try_next;
    const uint32_t *terms;
    const uint64_t *log_start;
    uint64_t *want_end;
};

__global__ void __launch_bounds__(kClThreads) backoff_key_kernel(const __grid_constant__ BackoffArgs A) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kClThreads;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kClThreads + threadIdx.x; i < A.n; i += stride) {
        uint64_t key = A.PG, end, ct, cs;
        const uint32_t g = A.frame_group[i], q = A.frame_peer[i];
        if (A.rec_kind[i] == SS_APPEND_REPLY_CONFLICT && g < A.G && q < A.P &&
            conflict_decode(A.buf, A.buf_len, A.frame_off[i], A.variant, end, ct, cs))
            key = static_cast<uint64_t>(g) * A.P + q;
        A.key_in[i] = static_cast<uint32_t>(key);
        A.idx_in[i] = static_cast<uint32_t>(i);
    }
}

// a thread per (group, peer) segment of the sorted conflicts, applied in frame order (messages.rs:386-406)
__global__ void __launch_bounds__(kClThreads) backoff_walk_kernel(const __grid_constant__ BackoffArgs A) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kClThreads;
    for (uint64_t t = static_cast<uint64_t>(blockIdx.x) * kClThreads + threadIdx.x; t < A.n; t += stride) {
        const uint32_t key = A.key[t];
        if (key >= A.PG || (t != 0u && A.key[t - 1u] == key)) continue;
        const uint64_t g = key / A.P, q = key % A.P, at = q * A.G + g;
        const uint64_t row = g * A.W, wm = A.W - 1u, ls = A.log_start[g];
        uint32_t ns = A.next_slot[at], tn = A.try_next[at];
        uint64_t we = ~0ull;
        for (uint64_t k = t; k < A.n && A.key[k] == key; ++k) {
            uint64_t end = 0, ct = 0, cs = 0;
            conflict_decode(A.buf, A.buf_len, A.frame_off[A.idx[k]], A.variant, end, ct, cs);
            if (ns == 1u) {                                                 // cannot move backward any more
                tn = 1u;
                we = ~0ull;
                continue;
            }
            --ns;
            while (ns > ls && A.terms[row + (ns & wm)] == ct && ns >= cs && ns > 1u) --ns;
            tn = ns;
            we = end;
        }
        A.next_slot[at] = ns;
        A.try_next[at] = tn;
        A.want_end[at] = we;
    }
}

// ---- execution -----------------------------------------------------------------------------------------------------
// the log's ring as the execution walk (exec_walk.cuh) reads it
struct CraftRing {
    uint32_t W, d;
    uint64_t plane_stride;
    const uint32_t *last_commit, *ent_len;
    const uint32_t *held;           // nullptr while every entry holds every shard (no step-up, no recon view)
    const uint64_t *log_start, *ent_addr;
    uint64_t *last_exec;
    const uint8_t *led;             // read by the kLed instances only: a group the engine does not lead is skipped
};

// the walk from max(last_exec + 1, log_start): stop past last_commit, or at fewer than d shards held (an entry a step-up
// took over that no absorb has completed yet); stop at a null entry, which get_data refuses (rscoding.rs:581-583)
template <bool kLed>
struct CraftLog : CraftRing {
    struct Walk { uint64_t s; };

    __device__ __forceinline__ bool live(uint64_t g) const { return !(kLed && led[g] == 0u); }
    __device__ __forceinline__ Walk start(uint64_t g) const {
        const uint64_t s = last_exec[g] + 1u, ls = log_start[g];
        return {s > ls ? s : ls};
    }
    __device__ __forceinline__ uint32_t next(const Walk &, uint64_t g, uint64_t s, uint32_t *dlen) const {
        if (s > last_commit[g]) return kExecStop;
        const uint64_t pos = g * W + (s & (W - 1u));
        if (held != nullptr && static_cast<uint32_t>(__popc(held[pos])) < d) return kExecStop;
        *dlen = ent_len[pos];
        return *dlen == 0u ? kExecNull : kExecRun;
    }
    __device__ __forceinline__ void finish(uint64_t g, uint64_t s) const { last_exec[g] = s - 1u; }
};

// shard j at ent_addr + j * plane_stride.  kRegen = false while every entry holds every shard (a log that was never
// stepped up): the gather never regenerates one and needs neither the coder's matrix nor the GF(2^8) tables.  kRegen
// once a held mask may lack shards (after a step-up): a missing data shard regenerated from the first d held ones.
template <bool kRegen>
struct CraftShards : CraftRing {
    static constexpr bool kTables = kRegen, kByIndex = kRegen;

    __device__ __forceinline__ ExecSrc source(uint64_t g, uint64_t s, uint32_t) const {
        const uint64_t pos = g * W + (s & (W - 1u));
        return {kRegen ? held[pos] : (1u << d) - 1u, reinterpret_cast<const uint8_t *>(ent_addr[pos]), plane_stride};
    }
};

// start_slot moves by clamp(upto - log_start, 0, min(last_snap, last_commit) - log_start)
__global__ void __launch_bounds__(kClThreads)
craft_advance_kernel(const uint64_t *__restrict__ upto, uint64_t G, uint64_t *__restrict__ log_start,
                     const uint32_t *__restrict__ last_snap, const uint32_t *__restrict__ last_commit) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kClThreads;
    for (uint64_t g = static_cast<uint64_t>(blockIdx.x) * kClThreads + threadIdx.x; g < G; g += stride) {
        const uint64_t s = log_start[g], u = upto[g];
        const uint64_t sn = last_snap[g], lc = last_commit[g];
        const uint64_t lim = sn < lc ? sn : lc;
        if (u > s && lim > s) log_start[g] = u < lim ? u : lim;
    }
}

void craft_log_free(ss_engine *e) {
    void *bufs[] = {e->log_start, e->try_next, e->ent_len, e->ent_addr, e->ent_log_offset, e->cl_partials, e->cl_words, e->cl_eff,
                    e->cl_wal, e->pk_frames, e->pk_bytes, e->pk_range, e->last_exec, e->ex_cnt, e->ex_bytes, e->ex_words, e->bo_keys,
                    e->bo_idx, e->bo_sort_tmp, e->held, e->last_recon, e->matrix, e->rc_words, e->led};
    for (void *b : bufs)
        if (b) cudaFree(b);
}

// the configuration checks every log call makes
int craft_check(ss_engine *e) {
    if (e == nullptr) return set_error(SS_ERR_INVALID_ARG, "null engine");
    if (e->cfg.protocol != SS_PROTO_CRAFT) return set_error(SS_ERR_INVALID_ARG, "the leader's log serves CRaft engines only");
    if (e->raft_appended) return set_error(SS_ERR_INVALID_ARG, "ss_engine_raft_append ran on this engine: its entries have no codeword");
    if (e->n < 3) return set_error(SS_ERR_INVALID_ARG, "the CRaft code needs a parity shard: population >= 3");
    return SS_OK;
}

// the coder's matrix, whose rows execute inverts on the device; a pageable source is staged before the call returns
static int upload_matrix(ss_engine *e) {
    const gf::Matrix m = gf::coding_matrix(static_cast<int>(e->majority), static_cast<int>(e->n - e->majority));
    SS_CUDA(cudaMemcpyAsync(e->matrix, m.v.data(), m.v.size(), cudaMemcpyHostToDevice, e->ctx->stream));
    return SS_OK;
}

// every ring position: every shard
__global__ void __launch_bounds__(kClThreads) craft_held_fill_kernel(uint32_t *held, uint64_t n, uint32_t all) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kClThreads;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kClThreads + threadIdx.x; i < n; i += stride) held[i] = all;
}

int craft_held_in_use(ss_engine *e) {
    if (e->held_partial) return SS_OK;
    // until now every entry was proposed, so it holds every shard: the masks start full
    ss_ctx *ctx = e->ctx;
    const uint64_t n = e->G * e->W;
    craft_held_fill_kernel<<<launch_grid(ctx, n, kClThreads), kClThreads, 0, ctx->stream>>>(e->held, n, e->n >= 32u ? 0xffffffffu : (1u << e->n) - 1u);
    SS_TRY(launched(ctx));
    e->held_partial = true;
    return SS_OK;
}

// takes the log into use: its state, scratch and coder on the first call
int craft_log_init(ss_engine *e) {
    ss_ctx *ctx = e->ctx;
    SS_TRY(ctx_bind(ctx));
    if (e->log_in_use) return SS_OK;
    const uint64_t G = e->G, PG = uint64_t(e->n_peers) * G, GW = G * e->W;
    if (e->coder == nullptr) SS_TRY(ss_rs_coder_create(ctx, static_cast<int>(e->majority), static_cast<int>(e->n - e->majority), &e->coder));
    int rc = SS_OK;
    if ((rc = dalloc(ctx, &e->try_next, PG, true)) || (rc = dalloc(ctx, &e->ent_len, GW, true)) ||
        (rc = dalloc(ctx, &e->ent_addr, GW, true)) || (rc = dalloc(ctx, &e->ent_log_offset, GW, true)) ||
        (rc = dalloc(ctx, &e->cl_partials, scan_tiles(PG > G ? PG : G), false)) || (rc = dalloc(ctx, &e->cl_words, 4, false)) ||
        (rc = dalloc(ctx, &e->cl_eff, G, false)) || (rc = dalloc(ctx, &e->cl_wal, G, false)) ||
        (rc = dalloc(ctx, &e->pk_frames, PG, false)) || (rc = dalloc(ctx, &e->pk_bytes, PG, false)) ||
        (rc = dalloc(ctx, &e->pk_range, PG, false)) || (rc = dalloc(ctx, &e->log_start, G, true)) ||
        (rc = dalloc(ctx, &e->last_exec, G, true)) || (rc = dalloc(ctx, &e->ex_cnt, G, false)) ||
        (rc = dalloc(ctx, &e->ex_bytes, G, false)) || (rc = dalloc(ctx, &e->ex_words, 3, false)) ||
        (rc = dalloc(ctx, &e->held, GW, true)) || (rc = dalloc(ctx, &e->last_recon, G, true)) ||
        (rc = dalloc(ctx, &e->matrix, size_t(e->n) * e->majority, false)) || (rc = upload_matrix(e))) {
        // nothing half-built stays behind: a later call starts over, and raft_append stays allowed
        cudaStreamSynchronize(ctx->stream);
        craft_log_free(e);
        e->log_start = nullptr; e->try_next = nullptr; e->ent_len = nullptr; e->ent_addr = nullptr; e->ent_log_offset = nullptr;
        e->cl_partials = nullptr; e->cl_words = nullptr; e->cl_eff = nullptr; e->cl_wal = nullptr;
        e->pk_frames = nullptr; e->pk_bytes = nullptr; e->pk_range = nullptr;
        e->last_exec = nullptr; e->ex_cnt = nullptr; e->ex_bytes = nullptr; e->ex_words = nullptr;
        e->bo_keys = nullptr; e->bo_idx = nullptr; e->bo_sort_tmp = nullptr; e->bo_cap = 0;
        e->held = nullptr; e->last_recon = nullptr; e->matrix = nullptr; e->rc_words = nullptr; e->rc_cap = 0; e->led = nullptr;
        return rc;
    }
    e->log_in_use = true;
    return SS_OK;
}

int backoff_scratch(ss_engine *e, uint64_t n, int bits) {
    if (n <= e->bo_cap) return SS_OK;
    ss_ctx *ctx = e->ctx;
    SS_CUDA(cudaStreamSynchronize(ctx->stream));
    void *old[] = {e->bo_keys, e->bo_idx, e->bo_sort_tmp};
    for (void *b : old)
        if (b) cudaFree(b);
    e->bo_keys = nullptr; e->bo_idx = nullptr; e->bo_sort_tmp = nullptr;
    e->bo_cap = 0;
    SS_TRY(dalloc(ctx, &e->bo_keys, 2 * n, false));
    SS_TRY(dalloc(ctx, &e->bo_idx, 2 * n, false));
    size_t bytes = 0;
    SS_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, bytes, e->bo_keys, e->bo_keys + n, e->bo_idx, e->bo_idx + n, static_cast<int>(n), 0, bits,
                                            ctx->stream));
    SS_CUDA(cudaMalloc(&e->bo_sort_tmp, bytes ? bytes : 1));
    e->bo_sort_bytes = bytes;
    e->bo_cap = n;
    return SS_OK;
}

}  // namespace ssb

using namespace ssb;

extern "C" {

int ss_engine_craft_log_view_get(ss_engine *e, ss_engine_craft_log_view *v) {
    if (v == nullptr) return set_error(SS_ERR_INVALID_ARG, "null view");
    SS_TRY(craft_check(e));
    SS_TRY(craft_log_init(e));
    memset(v, 0, sizeof(*v));
    v->n_groups = e->G; v->population = e->n; v->raft_window = e->W; v->data_shards = e->majority; v->total_shards = e->n;
    v->plane_stride = e->log_plane_stride;
    v->log_start = e->log_start; v->try_next = e->try_next; v->data_len = e->ent_len; v->shard_addr = e->ent_addr;
    v->log_offset = e->ent_log_offset;
    return SS_OK;
}

int ss_engine_craft_propose(ss_engine *e, uint32_t me, const uint8_t *arena, const uint64_t *data_off, const uint32_t *data_len,
                            uint8_t *shards, uint64_t plane_stride, uint64_t *shard_off, uint64_t *slot_out, uint64_t *need,
                            const uint64_t *log_offset, uint8_t *wal, uint64_t wal_capacity, uint64_t *wal_off, uint64_t *wal_len,
                            int full_copy) {
    if ((plane_stride & 31u) || plane_stride == 0) return set_error(SS_ERR_INVALID_ARG, "plane_stride must be a non-zero multiple of 32");
    if ((reinterpret_cast<uintptr_t>(shards) | reinterpret_cast<uintptr_t>(wal)) & 15u)
        return set_error(SS_ERR_INVALID_ARG, "the shard store and the WAL buffer must be 16-byte aligned");
    SS_TRY(craft_check(e));
    if (me >= e->n) return set_error(SS_ERR_INVALID_ARG, "me %u >= population %u", me, e->n);
    if (e->log_plane_stride != 0 && plane_stride != e->log_plane_stride)
        return set_error(SS_ERR_INVALID_ARG, "plane_stride %llu differs from the log's %llu", (unsigned long long)plane_stride,
                         (unsigned long long)e->log_plane_stride);
    if (!arena || !data_off || !data_len || !shards || !shard_off || !slot_out || !wal || !wal_off || !wal_len)
        return set_error(SS_ERR_INVALID_ARG, "null buffer");
    SS_TRY(craft_log_init(e));
    e->log_plane_stride = plane_stride;
    ss_ctx *ctx = e->ctx;
    ProposeArgs A{};
    A.G = e->G; A.W = e->W; A.d = e->majority; A.T = e->n; A.me = me; A.majority = e->majority; A.full_copy = full_copy ? 1u : 0u;
    A.data_len = data_len; A.log_offset = log_offset; A.shards = shards; A.plane_stride = plane_stride; A.wal_capacity = wal_capacity;
    A.shard_off = shard_off; A.slot_out = slot_out; A.wal_off = wal_off; A.wal_len = wal_len; A.wal = wal;
    A.log_start = e->log_start; A.log_end = e->log_end; A.terms = e->terms; A.curr_term = e->curr_term;
    A.ent_len = e->ent_len; A.held = e->held_partial ? e->held : nullptr; A.ent_addr = e->ent_addr; A.ent_log_offset = e->ent_log_offset;
    A.eff = e->cl_eff;
    A.rec_len = e->cl_wal;
    A.status = ctx->dev_status;
    A.led = e->led;
    const uint32_t grid = launch_grid(ctx, e->G, kClThreads);
    if (e->led != nullptr) craft_propose_prepare_kernel<true><<<grid, kClThreads, 0, ctx->stream>>>(A);
    else craft_propose_prepare_kernel<false><<<grid, kClThreads, 0, ctx->stream>>>(A);
    SS_TRY(launched(ctx));
    SS_TRY(launch_exclusive_scan_u64(ctx, shard_off, e->G, e->cl_partials, need != nullptr ? need : e->cl_words + 2));
    SS_TRY(launch_exclusive_scan_u64(ctx, wal_off, e->G, e->cl_partials, e->cl_words + 1));
    craft_propose_commit_kernel<<<grid, kClThreads, 0, ctx->stream>>>(A);
    SS_TRY(launched(ctx));
    // RSCodeword::from_data(batch, majority, population - majority) + compute_parity (craft/request.rs:70-77): data shards
    // into planes 0..d-1, parity into planes d..T-1, each at the group's slot
    SS_TRY(ss_rs_encode_batch_dev(e->coder, arena, data_off, e->cl_eff, e->G, shards + uint64_t(e->majority) * plane_stride, plane_stride,
                                  shard_off, SS_RS_OUT_PADDED16 | SS_RS_EMIT_DATA));
    craft_propose_wal_kernel<<<launch_grid(ctx, e->G, kClThreads / 32), kClThreads, 0, ctx->stream>>>(A);
    return launched(ctx);
}

int ss_frame_append_pack_dev(ss_engine *e, const ss_append_pack_spec *spec, const uint64_t *want_end, uint8_t *out, uint64_t out_capacity,
                             uint64_t *frame_off, uint64_t *frame_len, uint32_t *frame_group, uint8_t *frame_peer, uint64_t max_frames,
                             uint64_t *n_frames, uint32_t *pair_status, uint64_t *total) {
    if (spec == nullptr) return set_error(SS_ERR_INVALID_ARG, "null spec");
    if (spec->msg_chunk_size == 0) return set_error(SS_ERR_INVALID_ARG, "msg_chunk_size must be >= 1");
    if (spec->append_variant >= kVariantLimit) return set_error(SS_ERR_INVALID_ARG, "append_variant must be < 2^16");
    if (reinterpret_cast<uintptr_t>(out) & 15u) return set_error(SS_ERR_INVALID_ARG, "out must be 16-byte aligned");
    SS_TRY(craft_check(e));
    if (spec->me >= e->n) return set_error(SS_ERR_INVALID_ARG, "me %u >= population %u", spec->me, e->n);
    if (!out || !frame_off || !frame_len || !frame_group || !frame_peer || !n_frames || !pair_status)
        return set_error(SS_ERR_INVALID_ARG, "null buffer");
    SS_TRY(craft_log_init(e));
    ss_ctx *ctx = e->ctx;
    PackArgs A{};
    A.G = e->G; A.P = e->n_peers; A.PG = uint64_t(e->n_peers) * e->G; A.W = e->W; A.d = e->majority; A.T = e->n; A.me = spec->me;
    A.majority = e->majority; A.variant = spec->append_variant; A.chunk = spec->msg_chunk_size; A.full_copy = spec->full_copy ? 1u : 0u;
    A.heartbeat = spec->heartbeat ? 1u : 0u;
    A.want_end = spec->heartbeat ? nullptr : want_end;
    A.next_slot = e->next_slot; A.log_end = e->log_end; A.curr_term = e->curr_term; A.terms = e->terms; A.last_commit = e->last_commit;
    A.last_snap = e->last_snap; A.try_next = e->try_next; A.log_start = e->log_start; A.ent_len = e->ent_len;
    A.held = e->held_partial ? e->held : nullptr; A.ent_addr = e->ent_addr;
    A.ent_log_offset = e->ent_log_offset; A.plane_stride = e->log_plane_stride;
    A.out = out; A.out_capacity = out_capacity; A.max_frames = max_frames; A.frame_off = frame_off; A.frame_len = frame_len;
    A.frame_group = frame_group; A.frame_peer = frame_peer; A.n_frames = n_frames; A.total = total != nullptr ? total : e->cl_words + 3;
    A.pair_status = pair_status; A.pk_frames = e->pk_frames; A.pk_bytes = e->pk_bytes; A.pk_range = e->pk_range;
    A.frames_total = e->cl_words; A.status = ctx->dev_status; A.led = e->led;
    const uint32_t grid_w = launch_grid(ctx, A.PG, kClThreads / 32);
    const bool held = e->held_partial, led = e->led != nullptr;
    if (held && led) append_plan_kernel<true, true><<<grid_w, kClThreads, 0, ctx->stream>>>(A);
    else if (held) append_plan_kernel<true, false><<<grid_w, kClThreads, 0, ctx->stream>>>(A);
    else if (led) append_plan_kernel<false, true><<<grid_w, kClThreads, 0, ctx->stream>>>(A);
    else append_plan_kernel<false, false><<<grid_w, kClThreads, 0, ctx->stream>>>(A);
    SS_TRY(launched(ctx));
    SS_TRY(launch_exclusive_scan_u64(ctx, e->pk_frames, A.PG, e->cl_partials, e->cl_words));
    SS_TRY(launch_exclusive_scan_u64(ctx, e->pk_bytes, A.PG, e->cl_partials, A.total));
    SS_CUDA(cudaMemcpyAsync(n_frames, e->cl_words, 8, cudaMemcpyDeviceToDevice, ctx->stream));
    if (held && led) append_place_kernel<true, true><<<grid_w, kClThreads, 0, ctx->stream>>>(A);
    else if (held) append_place_kernel<true, false><<<grid_w, kClThreads, 0, ctx->stream>>>(A);
    else if (led) append_place_kernel<false, true><<<grid_w, kClThreads, 0, ctx->stream>>>(A);
    else append_place_kernel<false, false><<<grid_w, kClThreads, 0, ctx->stream>>>(A);
    SS_TRY(launched(ctx));
    const uint32_t grid_f = launch_grid(ctx, max_frames, kClThreads / 32);
    if (held) append_write_kernel<true><<<grid_f, kClThreads, 0, ctx->stream>>>(A);
    else append_write_kernel<false><<<grid_f, kClThreads, 0, ctx->stream>>>(A);
    return launched(ctx);
}

int ss_engine_craft_backoff(ss_engine *e, const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off, const uint32_t *frame_group,
                            const uint8_t *frame_peer, const uint32_t *rec_kind, uint64_t n_frames, uint32_t reply_variant,
                            uint64_t *want_end) {
    if (reply_variant >= kVariantLimit) return set_error(SS_ERR_INVALID_ARG, "reply_variant must be < 2^16");
    SS_TRY(craft_check(e));
    if (want_end == nullptr) return set_error(SS_ERR_INVALID_ARG, "null want_end");
    const uint64_t PG = uint64_t(e->n_peers) * e->G;
    if (PG >= 0xffffffffull) return set_error(SS_ERR_INVALID_ARG, "back-off keys need (population - 1) * n_groups < 2^32 - 1");
    if (n_frames > 0x7fffffffull) return set_error(SS_ERR_INVALID_ARG, "at most 2^31 - 1 frames per call");
    if (n_frames != 0 && (!buf || !frame_off || !frame_group || !frame_peer || !rec_kind)) return set_error(SS_ERR_INVALID_ARG, "null buffer");
    SS_TRY(craft_log_init(e));
    ss_ctx *ctx = e->ctx;
    SS_CUDA(cudaMemsetAsync(want_end, 0xff, PG * 8, ctx->stream));
    if (n_frames == 0) return SS_OK;
    SS_TRY(backoff_scratch(e, n_frames, key_bits(PG)));
    BackoffArgs A{};
    A.buf = buf; A.buf_len = buf_len; A.frame_off = frame_off; A.frame_group = frame_group; A.frame_peer = frame_peer; A.rec_kind = rec_kind;
    A.n = n_frames; A.G = e->G; A.PG = PG; A.P = e->n_peers; A.W = e->W; A.variant = reply_variant;
    A.key_in = e->bo_keys; A.idx_in = e->bo_idx; A.key = e->bo_keys + n_frames; A.idx = e->bo_idx + n_frames;
    A.next_slot = e->next_slot; A.try_next = e->try_next; A.terms = e->terms; A.log_start = e->log_start; A.want_end = want_end;
    const uint32_t grid = launch_grid(ctx, n_frames, kClThreads);
    backoff_key_kernel<<<grid, kClThreads, 0, ctx->stream>>>(A);
    SS_TRY(launched(ctx));
    size_t bytes = e->bo_sort_bytes;
    SS_CUDA(cub::DeviceRadixSort::SortPairs(e->bo_sort_tmp, bytes, e->bo_keys, e->bo_keys + n_frames, e->bo_idx, e->bo_idx + n_frames,
                                            static_cast<int>(n_frames), 0, key_bits(PG), ctx->stream));
    SS_TRY(launched(ctx));
    backoff_walk_kernel<<<grid, kClThreads, 0, ctx->stream>>>(A);
    return launched(ctx);
}

int ss_engine_craft_exec_view_get(ss_engine *e, ss_engine_craft_exec_view *v) {
    if (v == nullptr) return set_error(SS_ERR_INVALID_ARG, "null view");
    SS_TRY(craft_check(e));
    SS_TRY(craft_log_init(e));
    memset(v, 0, sizeof(*v));
    v->n_groups = e->G;
    v->last_exec = e->last_exec;
    return SS_OK;
}

int ss_engine_craft_execute(ss_engine *e, uint8_t *out, uint64_t out_capacity, uint32_t *rec_group, uint64_t *rec_slot,
                            uint64_t *rec_off, uint32_t *rec_len, uint64_t rec_capacity, uint64_t *totals) {
    if (!out || !rec_group || !rec_slot || !rec_off || !rec_len) return set_error(SS_ERR_INVALID_ARG, "null buffer");
    if (reinterpret_cast<uintptr_t>(out) & 15u) return set_error(SS_ERR_INVALID_ARG, "out must be 16-byte aligned");
    SS_TRY(craft_check(e));
    SS_TRY(craft_log_init(e));
    ss_ctx *ctx = e->ctx;
    const ExecOut o{e->matrix, e->ex_cnt, e->ex_bytes, e->ex_words, out, out_capacity, rec_group, rec_slot, rec_off, rec_len,
                    rec_capacity, ctx->dev_status};
    const CraftRing ring{e->W, e->majority, e->log_plane_stride, e->last_commit, e->ent_len, e->held_partial ? e->held : nullptr, e->log_start,
                         e->ent_addr, e->last_exec, e->led};
    uint64_t *tot = totals != nullptr ? totals : e->ex_words + 1;
    const auto run = [&](auto log, auto shards) { return launch_execute(ctx, o, log, shards, e->G, e->G * e->W, e->cl_partials, tot); };
    const bool led = e->led != nullptr;
    if (e->held_partial) return led ? run(CraftLog<true>{ring}, CraftShards<true>{ring}) : run(CraftLog<false>{ring}, CraftShards<true>{ring});
    return led ? run(CraftLog<true>{ring}, CraftShards<false>{ring}) : run(CraftLog<false>{ring}, CraftShards<false>{ring});
}

int ss_engine_craft_set_full_copy(ss_engine *e, int full_copy) {
    if (e == nullptr) return set_error(SS_ERR_INVALID_ARG, "null engine");
    if (e->cfg.protocol != SS_PROTO_CRAFT) return set_error(SS_ERR_INVALID_ARG, "the full-copy threshold serves CRaft engines only");
    // craft/messages.rs:300-310: majority in full-copy mode, majority + fault_tolerance otherwise
    e->threshold = full_copy ? e->majority : e->majority + e->cfg.fault_tolerance;
    return SS_OK;
}

int ss_engine_craft_advance(ss_engine *e, const uint64_t *upto) {
    SS_TRY(craft_check(e));
    if (upto == nullptr) return set_error(SS_ERR_INVALID_ARG, "null upto");
    SS_TRY(craft_log_init(e));
    ss_ctx *ctx = e->ctx;
    craft_advance_kernel<<<launch_grid(ctx, e->G, kClThreads), kClThreads, 0, ctx->stream>>>(upto, e->G, e->log_start, e->last_snap,
                                                                                      e->last_commit);
    return launched(ctx);
}

}  // extern "C"
