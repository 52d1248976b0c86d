// craft_recon.cu -- CRaft leader fail-over on the device: a follower's log taken over by the new leader, the Reconstruct
// reads for the entries it cannot execute, the followers' replies and the leader absorbing them.
//
//   ss_engine_craft_step_up   the log half of become_the_leader (craft/leadership.rs:212-246) for the listed groups:
//     stepup_first_kernel           a thread per listing: the first listing of each group
//     stepup_size_kernel            a thread per listing: verdicts, and the plane slots of the group's non-null entries
//     (engine.cu's scan)            plane regions in listing order
//     stepup_commit_kernel          a thread per listing: the capacity cut, then the engine's words, rings and peers
//     stepup_copy_kernel            a warp per (listing, ring entry): the held shards into their planes, 128-bit copies
//   ss_engine_craft_reconstruct_reads   the recon half of handle_msg_append_entries_reply's success branch
//                                       (craft/messages.rs:316-371):
//     recon_size_kernel             a thread per listing: the walk, its frames and region bytes
//     (engine.cu's scan)            frame indices and byte offsets in listing order
//     recon_write_kernel            a thread per listing: the capacity cut, the frames, last_recon
//   ss_follower_reconstruct_serve handle_msg_reconstruct (craft/messages.rs:621-662):
//     serve_size_kernel             a thread per frame: decode, verdict, reply bytes
//     (engine.cu's scan)            reply regions in frame order
//     serve_write_kernel            a warp per frame with a reply: capacity, the ReconstructReply, shards copied by the warp
//   ss_engine_craft_absorb    handle_msg_reconstruct_reply (craft/messages.rs:664-744) without its execution loop:
//     absorb_head_kernel            a thread per frame: decode and check the whole frame, sort keys
//     (CUB radix sort)              stable: each group's frames in frame order
//     absorb_apply_kernel           a warp per group segment: entries in frame order, then wire order, each missing shard
//                                   into its reserved plane slot
#include <cub/device/device_radix_sort.cuh>

#include <cstring>

#include "codeword_wire.cuh"
#include "craft_frames.cuh"
#include "device_common.cuh"
#include "engine_state.hpp"
#include "follower_state.hpp"
#include "ss_internal.hpp"
#include "wire_common.cuh"

namespace ssb {

constexpr int kRcThreads = 256;

// ---- step-up -------------------------------------------------------------------------------------------------------
struct StepUpArgs {
    const uint32_t *groups;
    const uint64_t *term;
    uint64_t n, G;
    uint32_t W, FW, d, P, wshift;   // wshift: log2(W)
    // the follower, read only
    const uint64_t *f_start, *f_log_end, *f_curr_term, *f_last_commit, *f_last_snap, *f_last_exec, *f_term, *f_addr;
    const uint32_t *f_held, *f_len;
    // outputs and scratch
    uint64_t *first;                // [G] the first listing of each group
    uint8_t *shards;
    uint64_t plane_stride;
    uint64_t *shard_off;
    const uint64_t *need;
    uint32_t *verdict;
    // the engine
    uint64_t *log_start, *last_exec, *ent_addr, *ent_log_offset;
    uint32_t *log_end, *last_commit, *last_snap, *curr_term, *terms, *ent_len, *held, *match, *next_slot, *try_next;
    uint32_t *status;
};

__global__ void __launch_bounds__(kRcThreads) stepup_first_kernel(const __grid_constant__ StepUpArgs A) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kRcThreads;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kRcThreads + threadIdx.x; i < A.n; i += stride) {
        const uint32_t g = A.groups[i];
        if (g < A.G) atomicMin(reinterpret_cast<unsigned long long *>(A.first + g), static_cast<unsigned long long>(i));
    }
}

__global__ void __launch_bounds__(kRcThreads) stepup_size_kernel(const __grid_constant__ StepUpArgs A) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kRcThreads;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kRcThreads + threadIdx.x; i < A.n; i += stride) {
        const uint32_t g = A.groups[i];
        uint32_t v = SS_STEPUP_VERDICT_DONE;
        uint64_t bytes = 0;
        if (g >= A.G || A.first[g] != i) {
            v = SS_STEPUP_VERDICT_IGNORED;
        } else {
            const uint64_t st = A.f_start[g], le = A.f_log_end[g], t = A.term[i], row = static_cast<uint64_t>(g) * A.FW;
            if (le - st > A.W) {
                v = SS_STEPUP_VERDICT_WINDOW;
            } else {
                bool range = le > 0xffffffffull || t > 0xffffffffull || A.f_last_snap[g] > 0xffffffffull;
                for (uint64_t s = st; s < le && !range; ++s) range = A.f_term[row + (s & (A.FW - 1u))] > 0xffffffffull;
                if (range) {
                    v = SS_STEPUP_VERDICT_RANGE;
                } else if (t < A.f_curr_term[g]) {
                    v = SS_STEPUP_VERDICT_STALE_TERM;
                } else {
                    for (uint64_t s = st; s < le; ++s) {
                        const uint32_t dl = A.f_len[row + (s & (A.FW - 1u))];
                        if (dl != 0u) bytes += SS_CW_SLOT_PITCH((dl + A.d - 1u) / A.d);
                    }
                }
            }
        }
        A.verdict[i] = v;
        A.shard_off[i] = bytes;
    }
}

__global__ void __launch_bounds__(kRcThreads) stepup_commit_kernel(const __grid_constant__ StepUpArgs A) {
    bool full = false;
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kRcThreads;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kRcThreads + threadIdx.x; i < A.n; i += stride) {
        // shard_off is only read here: the next listing's offset is this one's end (UINT64_MAX goes in with the copies)
        if (A.verdict[i] != SS_STEPUP_VERDICT_DONE) continue;
        const uint64_t off = A.shard_off[i], end = i + 1u < A.n ? A.shard_off[i + 1u] : *A.need;
        if (end > A.plane_stride) {                                         // the offsets are monotone: a suffix is cut
            full = true;
            A.verdict[i] = SS_STEPUP_VERDICT_STORE_FULL;
            continue;
        }
        const uint32_t g = A.groups[i];
        const uint64_t st = A.f_start[g], le = A.f_log_end[g], frow = static_cast<uint64_t>(g) * A.FW, row = static_cast<uint64_t>(g) * A.W;
        uint64_t at = off;
        for (uint64_t s = st; s < le; ++s) {
            const uint64_t fp = frow + (s & (A.FW - 1u)), ep = row + (s & (A.W - 1u));
            const uint32_t dl = A.f_len[fp];
            A.terms[ep] = static_cast<uint32_t>(A.f_term[fp]);
            A.ent_len[ep] = dl;
            A.held[ep] = A.f_held[fp];
            A.ent_addr[ep] = dl != 0u ? reinterpret_cast<uint64_t>(A.shards + at) : 0ull;
            A.ent_log_offset[ep] = 0u;
            if (dl != 0u) at += SS_CW_SLOT_PITCH((dl + A.d - 1u) / A.d);
        }
        A.log_start[g] = st;
        A.log_end[g] = static_cast<uint32_t>(le);
        A.last_commit[g] = static_cast<uint32_t>(A.f_last_commit[g]);
        A.last_snap[g] = static_cast<uint32_t>(A.f_last_snap[g]);
        A.last_exec[g] = A.f_last_exec[g];
        A.curr_term[g] = static_cast<uint32_t>(A.term[i]);
        for (uint32_t q = 0; q < A.P; ++q) {                                // leadership.rs:225-234
            const uint64_t p = static_cast<uint64_t>(q) * A.G + g;
            A.next_slot[p] = static_cast<uint32_t>(le);
            A.try_next[p] = static_cast<uint32_t>(le);
            A.match[p] = 0u;
        }
    }
    if (full) atomicOr(A.status, SS_DEV_STATUS_STORE_FULL);
}

// a warp per (listing i, entry k of its span): the held shard of rank r (follower store, SS_CW_SLOT_PITCH(L) apart) into
// plane j at the slot the commit pass gave the entry; round_up(L, 16) bytes, the zero pad included.  A listing not
// stepped up gets shard_off UINT64_MAX here.
__global__ void __launch_bounds__(kRcThreads, 1) stepup_copy_kernel(const __grid_constant__ StepUpArgs A) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = (static_cast<uint64_t>(blockIdx.x) * kRcThreads + threadIdx.x) >> 5;
    const uint64_t nwarps = (static_cast<uint64_t>(gridDim.x) * kRcThreads) >> 5;
    const uint64_t items = A.n * A.W;
    for (uint64_t it = warp; it < items; it += nwarps) {
        const uint64_t i = it >> A.wshift, k = it & (A.W - 1u);
        if (A.verdict[i] != SS_STEPUP_VERDICT_DONE) {
            if (k == 0u && lane == 0u) A.shard_off[i] = ~0ull;
            continue;
        }
        const uint32_t g = A.groups[i];
        const uint64_t s = A.f_start[g] + k;
        if (s >= A.f_log_end[g]) continue;
        const uint64_t fp = static_cast<uint64_t>(g) * A.FW + (s & (A.FW - 1u)), ep = static_cast<uint64_t>(g) * A.W + (s & (A.W - 1u));
        const uint32_t dl = A.f_len[fp];
        if (dl == 0u) continue;
        const uint64_t L = (dl + A.d - 1u) / A.d, pitch = SS_CW_SLOT_PITCH(L), nvec = (L + 15u) >> 4;
        const uint8_t *src = reinterpret_cast<const uint8_t *>(A.f_addr[fp]);
        uint8_t *dst = reinterpret_cast<uint8_t *>(A.ent_addr[ep]);
        uint32_t r = 0;
        for (uint32_t rest = A.f_held[fp]; rest != 0u; rest &= rest - 1u, ++r) {
            const uint32_t j = static_cast<uint32_t>(__ffs(static_cast<int>(rest))) - 1u;
            const uint8_t *sj = src + r * pitch;
            uint8_t *dj = dst + j * A.plane_stride;
            for (uint64_t v = lane; v < nvec; v += 32u) dev::stg128_cs(dj + v * 16u, dev::ldg128(sj + v * 16u));
        }
    }
}

// ---- reconstruct reads ---------------------------------------------------------------------------------------------
struct ReadsArgs {
    const uint32_t *groups;         // nullptr: listing i is group i
    uint64_t n, G, chunk;
    uint32_t W, d, variant;
    const uint64_t *log_start, *last_exec;
    const uint32_t *last_commit, *terms, *held;
    uint64_t *last_recon;
    uint64_t *recon0;               // [n] last_recon of listing i's group as the size pass read it
    uint64_t *cnt, *bytes;          // [n] frames and region bytes of listing i, then their exclusive scans
    const uint64_t *totals;
    uint8_t *out;
    uint64_t out_cap;
    uint32_t *frame_group;
    uint8_t *frame_dst;
    uint64_t *frame_off;
    uint32_t *frame_len;
    uint64_t frame_cap;
    uint32_t *status;
    const uint8_t *led;             // read by the kLed instances only: a group the engine does not lead lists nothing
};

__device__ __forceinline__ uint32_t reads_group(const ReadsArgs &A, uint64_t i) { return A.groups != nullptr ? A.groups[i] : static_cast<uint32_t>(i); }

// the walk of group g past last_recon = lr0: calls f(slot, term) for every listed slot, in slot order
template <typename F>
__device__ __forceinline__ void reads_walk(const ReadsArgs &A, uint32_t g, uint64_t lr0, F &&f) {
    const uint64_t ex = A.last_exec[g] + 1u, ls = A.log_start[g];
    uint64_t s = ex > ls ? ex : ls;
    if (s <= lr0) s = lr0 + 1u;
    const uint64_t lc = A.last_commit[g], row = static_cast<uint64_t>(g) * A.W;
    for (; s <= lc; ++s) {
        const uint64_t pos = row + (s & (A.W - 1u));
        if (static_cast<uint32_t>(__popc(A.held[pos])) < A.d) f(s, A.terms[pos]);
    }
}

// frame bytes: 8-byte length, PeerMessage::Msg, the variant, the entry count, the (slot, term) entries
__device__ __forceinline__ uint64_t reads_frame_len(const ReadsArgs &A, uint64_t m, uint64_t ebytes) {
    return 9u + wv_len(A.variant) + wv_len(m) + ebytes;
}

template <bool kLed>
__global__ void __launch_bounds__(kRcThreads) recon_size_kernel(const __grid_constant__ ReadsArgs A) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kRcThreads;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kRcThreads + threadIdx.x; i < A.n; i += stride) {
        const uint32_t g = reads_group(A, i);
        uint64_t frames = 0, bytes = 0;
        if (g < A.G && !(kLed && A.led[g] == 0u)) {
            const uint64_t lr0 = A.last_recon[g];
            uint64_t m = 0, eb = 0;
            reads_walk(A, g, lr0, [&](uint64_t s, uint32_t t) {
                eb += wv_len(s) + wv_len(t);
                if (++m == A.chunk) {
                    bytes += round16(reads_frame_len(A, m, eb));
                    ++frames;
                    m = eb = 0;
                }
            });
            if (m != 0u) {
                bytes += round16(reads_frame_len(A, m, eb));
                ++frames;
            }
            A.recon0[i] = lr0;
        }
        A.cnt[i] = frames;
        A.bytes[i] = bytes;
    }
}

template <bool kLed>
__global__ void __launch_bounds__(kRcThreads) recon_write_kernel(const __grid_constant__ ReadsArgs A) {
    bool full = false;
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kRcThreads;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kRcThreads + threadIdx.x; i < A.n; i += stride) {
        const uint32_t g = reads_group(A, i);
        if (g >= A.G || (kLed && A.led[g] == 0u)) continue;
        const uint64_t f0 = A.cnt[i], o0 = A.bytes[i];
        const uint64_t f1 = i + 1u < A.n ? A.cnt[i + 1u] : A.totals[0], o1 = i + 1u < A.n ? A.bytes[i + 1u] : A.totals[1];
        if (f1 > A.frame_cap || o1 > A.out_cap) {                          // the ends are monotone: a suffix is cut
            full |= f1 != f0;
            for (uint64_t f = f0; f < f1 && f < A.frame_cap; ++f) {
                A.frame_group[f] = g;
                A.frame_dst[f] = 0xffu;
                A.frame_off[f] = ~0ull;
                A.frame_len[f] = 0u;
            }
            continue;
        }
        // the count walk gives each frame's entry count; the write walk puts a frame's header in at its first entry and
        // its length once its last entry is written: two passes over the group's span in all
        const uint64_t lr0 = A.recon0[i];
        uint64_t total = 0;
        reads_walk(A, g, lr0, [&](uint64_t, uint32_t) { ++total; });
        uint64_t f = f0, o = o0, k = 0, m = 0, last = lr0, at = 0;
        uint8_t *fr = nullptr;
        reads_walk(A, g, lr0, [&](uint64_t s, uint32_t t) {
            if (k % A.chunk == 0u) {                                        // a new frame: Msg, the variant, its entry count
                m = total - k < A.chunk ? total - k : A.chunk;
                fr = A.out + o;
                at = 8u;
                at += wv_put(fr + at, 0u);                                  // PeerMessage::Msg
                at += wv_put(fr + at, A.variant);
                at += wv_put(fr + at, m);
            }
            at += wv_put(fr + at, s);
            at += wv_put(fr + at, t);
            ++k;
            last = s;
            if (k % A.chunk == 0u || k == total) {                          // its last entry: the length and the records
                put_be64(fr, at - 8u);
                A.frame_group[f] = g;
                A.frame_dst[f] = 0xffu;
                A.frame_off[f] = o;
                A.frame_len[f] = static_cast<uint32_t>(at);
                ++f;
                o += round16(at);
            }
        });
        if (total != 0u) A.last_recon[g] = last;
    }
    if (full) atomicOr(A.status, SS_DEV_STATUS_FRAME_OVERFLOW);
}

// ---- serve on the follower -----------------------------------------------------------------------------------------
struct ServeArgs {
    const uint8_t *buf;
    uint64_t buf_len;
    const uint64_t *frame_off;
    const uint32_t *frame_group;
    uint64_t n, G;
    uint32_t d, T, FW, variant, reply_variant;
    const uint64_t *start_slot, *log_end, *term, *shard_addr;
    const uint32_t *held, *data_len;
    uint8_t *out;
    uint64_t out_cap;
    uint64_t *reply_off, *reply_len;
    uint32_t *verdict, *status;
};

// The Reconstruct{slots: Vec<(usize, Term)>} of frame i walked as handle_msg_reconstruct walks it: f(slot, ring
// position) for each entry the reply carries -- inside [start_slot, log_end) with the ring's term, and not an earlier
// entry's (slot, term) again (the map keeps one entry per slot; entries follow their first occurrence).  Returns
// kPending for a well-formed frame, else its verdict.
template <typename F>
__device__ __forceinline__ uint32_t serve_walk(const ServeArgs &A, uint64_t i, F &&f) {
    const uint8_t *b = nullptr;
    uint64_t len = 0, n = 0, cnt = 0;
    const uint32_t g = A.frame_group[i];
    if (g >= A.G) return SS_FRAME_KIND_MALFORMED;
    const uint32_t kind = msg_head_count(A.buf, A.buf_len, A.frame_off[i], A.variant, ~0ull, b, len, n, cnt);
    if (kind != kPending) return kind;
    const uint64_t st = A.start_slot[g], le = A.log_end[g], row = static_cast<uint64_t>(g) * A.FW;
    const uint64_t n0 = n;
    bool rising = true;                                                     // slots strictly rising: no entry repeats
    for (uint64_t e = 0, prev = 0; e < cnt; ++e) {
        uint64_t slot = 0, t = 0;
        if (!wv_next(b, len, n, slot) || !wv_next(b, len, n, t)) return SS_FRAME_KIND_MALFORMED;
        rising &= e == 0u || slot > prev;
        prev = slot;
    }
    if (n != len) return SS_FRAME_KIND_MALFORMED;
    n = n0;
    for (uint64_t e = 0; e < cnt; ++e) {
        uint64_t slot = 0, t = 0;
        n += wv_get(b + n, len - n, slot);
        n += wv_get(b + n, len - n, t);
        if (slot < st || slot >= le) continue;
        const uint64_t pos = row + (slot & (A.FW - 1u));
        if (A.term[pos] != t) continue;
        bool seen = false;
        for (uint64_t q = 0, m = n0; !rising && q < e && !seen; ++q) {
            uint64_t s2 = 0, t2 = 0;
            m += wv_get(b + m, len - m, s2);
            m += wv_get(b + m, len - m, t2);
            seen = s2 == slot && t2 == t;
        }
        if (!seen) f(slot, pos);
    }
    return kPending;
}

__global__ void __launch_bounds__(kRcThreads) serve_size_kernel(const __grid_constant__ ServeArgs A) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kRcThreads;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kRcThreads + threadIdx.x; i < A.n; i += stride) {
        uint64_t cnt = 0, bytes = 0;
        uint32_t kind = serve_walk(A, i, [&](uint64_t slot, uint64_t pos) {
            ++cnt;
            bytes += wv_len(slot) + cw_bytes(A.data_len[pos], A.d, A.T, __popc(A.held[pos]));
        });
        if (kind == kPending) kind = SS_ACCEPT_VERDICT_ACCEPTED;
        if (kind != SS_ACCEPT_VERDICT_ACCEPTED || cnt == 0u) bytes = 0;
        else bytes += 9u + wv_len(A.reply_variant) + wv_len(cnt);
        A.verdict[i] = kind;
        A.reply_len[i] = bytes;
        A.reply_off[i] = round16(bytes);
    }
}

// a warp per frame with a reply: PeerMessage::Msg{ReconstructReply{slots_data: HashMap<usize, RSCodeword>}}; every lane
// walks the frame (the loads broadcast), lane 0 writes the varints and tags, the warp copies each held shard from its
// 16-byte aligned store slot
__global__ void __launch_bounds__(kRcThreads, 1) serve_write_kernel(const __grid_constant__ ServeArgs A) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = (static_cast<uint64_t>(blockIdx.x) * kRcThreads + threadIdx.x) >> 5;
    const uint64_t nwarps = (static_cast<uint64_t>(gridDim.x) * kRcThreads) >> 5;
    bool full = false;
    for (uint64_t i = warp; i < A.n; i += nwarps) {
        const uint64_t len = A.reply_len[i], off = A.reply_off[i];
        if (len == 0u || off > A.out_cap || round16(len) > A.out_cap - off) {
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
        uint64_t cnt = 0;
        serve_walk(A, i, [&](uint64_t, uint64_t) { ++cnt; });
        uint8_t *dst = A.out + off;
        uint64_t at = 8u + 1u + wv_len(A.reply_variant) + wv_len(cnt);
        if (lane == 0u) {
            put_be64(dst, len - 8u);
            uint64_t m = 8u;
            m += wv_put(dst + m, 0u);                                       // PeerMessage::Msg
            m += wv_put(dst + m, A.reply_variant);
            wv_put(dst + m, cnt);
        }
        serve_walk(A, i, [&](uint64_t slot, uint64_t pos) {
            const uint32_t held = A.held[pos];
            const uint64_t dl = A.data_len[pos], pitch = SS_CW_SLOT_PITCH((dl + A.d - 1u) / A.d);
            const uint8_t *src = reinterpret_cast<const uint8_t *>(A.shard_addr[pos]);
            if (lane == 0u) wv_put(dst + at, slot);
            at += wv_len(slot);
            at += warp_put_cw(dst + at, A.d, A.T, dl, held, [&](uint32_t j) {
                return src + static_cast<uint64_t>(__popc(held & ((1u << j) - 1u))) * pitch;
            }, lane);
        });
        __syncwarp();
    }
    if (full && lane == 0u) atomicOr(A.status, SS_DEV_STATUS_FRAME_OVERFLOW);
}

// ---- absorb on the leader ------------------------------------------------------------------------------------------
struct AbsorbArgs {
    const uint8_t *buf;
    uint64_t buf_len;
    const uint64_t *frame_off;
    const uint32_t *frame_group;
    uint64_t n, G;
    uint32_t W, d, T, variant;
    uint64_t plane_stride;
    const uint64_t *log_start, *ent_addr;
    const uint32_t *log_end, *ent_len;
    uint32_t *held;
    uint64_t *fr_at;                // [n] body offset of entry 0 (past the map length), [n] the entry count, [n] 1 when
                                    // the slots do not strictly rise (a key may repeat)
    uint32_t *key_in, *idx_in;
    const uint32_t *key, *idx;
    uint32_t *absorbed, *verdict;
};

// one (slot, RSCodeword) at b + n: this code, shard_len = ceil(data_len / d), exactly T shard Options of shard_len
// bytes, data_copy None or Some(data_len bytes); tags_at = body offset of shard 0's Option tag
struct AbsEntry {
    uint64_t slot, dl, L, tags_at;
    uint32_t mask;
};

__device__ __forceinline__ bool abs_entry(const uint8_t *b, uint64_t len, uint64_t &n, uint32_t d, uint32_t T, AbsEntry &E) {
    return wv_next(b, len, n, E.slot) && cw_parse<true>(b, len, n, d, T, E.dl, E.L, E.tags_at, E.mask);
}

__global__ void __launch_bounds__(kRcThreads) absorb_head_kernel(const __grid_constant__ AbsorbArgs A) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kRcThreads;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kRcThreads + threadIdx.x; i < A.n; i += stride) {
        const uint8_t *b = nullptr;
        uint64_t len = 0, n = 0, cnt = 0;
        const uint32_t g = A.frame_group[i];
        uint32_t kind = g >= A.G ? SS_FRAME_KIND_MALFORMED : msg_head_count(A.buf, A.buf_len, A.frame_off[i], A.variant, ~0ull, b, len, n, cnt);
        if (kind == kPending) {
            A.fr_at[i] = n;
            A.fr_at[A.n + i] = cnt;
            AbsEntry E;
            kind = SS_ACCEPT_VERDICT_ACCEPTED;
            bool rising = true;
            for (uint64_t e = 0, prev = 0; e < cnt; ++e) {
                if (!abs_entry(b, len, n, A.d, A.T, E)) { kind = SS_FRAME_KIND_MALFORMED; break; }
                rising &= e == 0u || E.slot > prev;
                prev = E.slot;
            }
            A.fr_at[2u * A.n + i] = rising ? 0u : 1u;
            if (n != len) kind = SS_FRAME_KIND_MALFORMED;
        }
        A.verdict[i] = kind;
        A.absorbed[i] = 0u;
        A.key_in[i] = kind == SS_ACCEPT_VERDICT_ACCEPTED ? g : static_cast<uint32_t>(A.G);
        A.idx_in[i] = static_cast<uint32_t>(i);
    }
}

// a warp per group segment: its frames in frame order, each frame's entries in wire order; an entry whose slot comes
// again later in the frame is passed (a HashMap decode keeps the last insert).  Warp-uniform: every lane decodes the
// same bytes; lane 0 updates held after the warp has copied the shards.
__global__ void __launch_bounds__(kRcThreads, 1) absorb_apply_kernel(const __grid_constant__ AbsorbArgs A) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = (static_cast<uint64_t>(blockIdx.x) * kRcThreads + threadIdx.x) >> 5;
    const uint64_t nwarps = (static_cast<uint64_t>(gridDim.x) * kRcThreads) >> 5;
    for (uint64_t t = warp; t < A.n; t += nwarps) {
        const uint32_t g = A.key[t];
        if (g >= A.G || (t != 0u && A.key[t - 1u] == g)) continue;
        const uint64_t ls = A.log_start[g], le = A.log_end[g], row = static_cast<uint64_t>(g) * A.W;
        for (uint64_t k = t; k < A.n && A.key[k] == g; ++k) {
            const uint32_t i = A.idx[k];
            const uint8_t *fr = A.buf + A.frame_off[i];
            const uint64_t len = get_be64(fr);
            const uint8_t *b = fr + 8;
            const uint64_t cnt = A.fr_at[A.n + i];
            const bool may_repeat = A.fr_at[2u * A.n + i] != 0u;
            uint64_t n = A.fr_at[i];
            uint32_t taken = 0;
            AbsEntry E, E2;
            for (uint64_t e = 0; e < cnt; ++e) {
                abs_entry(b, len, n, A.d, A.T, E);
                bool later = false;
                for (uint64_t q = e + 1u, m = n; may_repeat && q < cnt && !later; ++q) {
                    abs_entry(b, len, m, A.d, A.T, E2);
                    later = E2.slot == E.slot;
                }
                if (later || E.slot < ls || E.slot >= le) continue;
                const uint64_t pos = row + (E.slot & (A.W - 1u));
                const uint32_t dl = A.ent_len[pos];
                if (dl == 0u || E.dl != dl) continue;                       // a null entry; absorb_other's data_len check
                const uint32_t add = E.mask & ~A.held[pos];
                __syncwarp();
                if (add == 0u) continue;
                uint8_t *dst = reinterpret_cast<uint8_t *>(A.ent_addr[pos]);
                const uint8_t *tags = b + E.tags_at;
                uint64_t at = 0;
                for (uint32_t j = 0; j < A.T; ++j) {
                    if (!((E.mask >> j) & 1u)) { at += 1u; continue; }
                    const uint64_t sl = some_len(tags[at + 1u]);
                    if ((add >> j) & 1u) warp_fill_slot(dst + j * A.plane_stride, tags + at + sl, E.L, lane);
                    at += sl + E.L;
                }
                __syncwarp();
                if (lane == 0u) A.held[pos] |= add;
                __syncwarp();
                ++taken;
            }
            if (lane == 0u) A.absorbed[i] = taken;
        }
    }
}

// the engine's recon scratch, grow-only: `words` u64
int rc_scratch(ss_engine *e, uint64_t words) {
    if (words <= e->rc_cap) return SS_OK;
    SS_CUDA(cudaStreamSynchronize(e->ctx->stream));
    if (e->rc_words) cudaFree(e->rc_words);
    e->rc_words = nullptr;
    e->rc_cap = 0;
    SS_CUDA(cudaMalloc(reinterpret_cast<void **>(&e->rc_words), words * 8));
    e->rc_cap = words;
    return SS_OK;
}

}  // namespace ssb

using namespace ssb;

extern "C" {

int ss_engine_craft_recon_view_get(ss_engine *e, ss_engine_craft_recon_view *v) {
    if (v == nullptr) return set_error(SS_ERR_INVALID_ARG, "null view");
    SS_TRY(craft_check(e));
    SS_TRY(craft_log_init(e));
    memset(v, 0, sizeof(*v));
    v->n_groups = e->G; v->raft_window = e->W; v->total_shards = e->n;
    v->held = e->held; v->last_recon = e->last_recon;
    SS_TRY(craft_held_in_use(e));                                           // the host may clear held bits through the view
    return SS_OK;
}

int ss_engine_craft_step_up(ss_engine *e, const ss_follower *f, const uint32_t *groups, uint64_t n_listed, const uint64_t *term,
                            uint8_t *shards, uint64_t plane_stride, uint64_t *shard_off, uint64_t *need, uint32_t *verdict) {
    if (f == nullptr) return set_error(SS_ERR_INVALID_ARG, "null follower");
    if ((plane_stride & 31u) || plane_stride == 0) return set_error(SS_ERR_INVALID_ARG, "plane_stride must be a non-zero multiple of 32");
    if (reinterpret_cast<uintptr_t>(shards) & 15u) return set_error(SS_ERR_INVALID_ARG, "the shard planes must be 16-byte aligned");
    SS_TRY(craft_check(e));
    if (f->cfg.protocol != e->cfg.protocol) return set_error(SS_ERR_INVALID_ARG, "the follower's protocol differs from the engine's");
    if (f->cfg.population != e->n) return set_error(SS_ERR_INVALID_ARG, "the follower's population %u differs from the engine's %u", f->cfg.population, e->n);
    if (f->G != e->G) return set_error(SS_ERR_INVALID_ARG, "the follower's n_groups differs from the engine's");
    if (f->ctx != e->ctx) return set_error(SS_ERR_INVALID_ARG, "the follower and the engine must share a context");
    if (e->log_plane_stride != 0 && plane_stride != e->log_plane_stride)
        return set_error(SS_ERR_INVALID_ARG, "plane_stride %llu differs from the log's %llu", (unsigned long long)plane_stride,
                         (unsigned long long)e->log_plane_stride);
    if (n_listed > 0x7fffffffull) return set_error(SS_ERR_INVALID_ARG, "at most 2^31 - 1 listed groups per call");
    SS_TRY(craft_log_init(e));
    ss_ctx *ctx = e->ctx;
    if (n_listed == 0) {
        if (need != nullptr) SS_CUDA(cudaMemsetAsync(need, 0, 8, ctx->stream));
        return SS_OK;
    }
    if (!groups || !term || !shards || !shard_off || !verdict) return set_error(SS_ERR_INVALID_ARG, "null buffer");
    SS_TRY(rc_scratch(e, e->G + scan_tiles(n_listed) + 1u));
    e->log_plane_stride = plane_stride;
    SS_TRY(craft_held_in_use(e));
    StepUpArgs A{};
    A.groups = groups; A.term = term; A.n = n_listed; A.G = e->G; A.W = e->W; A.FW = f->W; A.d = e->majority; A.P = e->n_peers;
    while ((1u << A.wshift) < A.W) ++A.wshift;
    A.f_start = f->start_slot; A.f_log_end = f->log_end; A.f_curr_term = f->curr_term; A.f_last_commit = f->last_commit;
    A.f_last_snap = f->last_snap; A.f_last_exec = f->last_exec; A.f_term = f->term; A.f_addr = f->shard_addr; A.f_held = f->held;
    A.f_len = f->data_len;
    A.first = e->rc_words; A.shards = shards; A.plane_stride = plane_stride; A.shard_off = shard_off;
    uint64_t *partials = e->rc_words + e->G, *tot = need != nullptr ? need : partials + scan_tiles(n_listed);
    A.need = tot; A.verdict = verdict;
    A.log_start = e->log_start; A.last_exec = e->last_exec; A.ent_addr = e->ent_addr; A.ent_log_offset = e->ent_log_offset;
    A.log_end = e->log_end; A.last_commit = e->last_commit; A.last_snap = e->last_snap; A.curr_term = e->curr_term; A.terms = e->terms;
    A.ent_len = e->ent_len; A.held = e->held; A.match = e->match; A.next_slot = e->next_slot; A.try_next = e->try_next;
    A.status = ctx->dev_status;
    const uint32_t grid = launch_grid(ctx, n_listed, kRcThreads);
    SS_CUDA(cudaMemsetAsync(e->rc_words, 0xff, e->G * 8, ctx->stream));
    stepup_first_kernel<<<grid, kRcThreads, 0, ctx->stream>>>(A);
    SS_TRY(launched(ctx));
    stepup_size_kernel<<<grid, kRcThreads, 0, ctx->stream>>>(A);
    SS_TRY(launched(ctx));
    SS_TRY(launch_exclusive_scan_u64(ctx, shard_off, n_listed, partials, tot));
    stepup_commit_kernel<<<grid, kRcThreads, 0, ctx->stream>>>(A);
    SS_TRY(launched(ctx));
    stepup_copy_kernel<<<launch_grid(ctx, n_listed * e->W, kRcThreads / 32), kRcThreads, 0, ctx->stream>>>(A);
    SS_TRY(launched(ctx));
    return craft_led_mark(e, groups, verdict, n_listed);                   // a stepped-up group is led again
}

int ss_engine_craft_reconstruct_reads(ss_engine *e, const uint32_t *groups, uint64_t n_listed, uint64_t chunk_size,
                                      uint32_t reconstruct_variant, uint8_t *out, uint64_t out_capacity, uint32_t *frame_group,
                                      uint8_t *frame_dst, uint64_t *frame_off, uint32_t *frame_len, uint64_t frame_capacity,
                                      uint64_t *totals) {
    if (chunk_size == 0) return set_error(SS_ERR_INVALID_ARG, "chunk_size must be at least 1");
    if (reconstruct_variant >= kVariantLimit) return set_error(SS_ERR_INVALID_ARG, "reconstruct_variant must be < 2^16");
    SS_TRY(craft_check(e));
    SS_TRY(craft_log_init(e));
    SS_TRY(craft_held_in_use(e));                                           // it reads held
    ss_ctx *ctx = e->ctx;
    const uint64_t n = groups != nullptr ? n_listed : e->G;
    if (n == 0) {
        if (totals != nullptr) SS_CUDA(cudaMemsetAsync(totals, 0, 16, ctx->stream));
        return SS_OK;
    }
    if (!out || !frame_group || !frame_dst || !frame_off || !frame_len) return set_error(SS_ERR_INVALID_ARG, "null buffer");
    if (reinterpret_cast<uintptr_t>(out) & 15u) return set_error(SS_ERR_INVALID_ARG, "out must be 16-byte aligned");
    if (n > 0x7fffffffull) return set_error(SS_ERR_INVALID_ARG, "at most 2^31 - 1 listed groups per call");
    SS_TRY(rc_scratch(e, 3u * n + scan_tiles(n) + 2u));
    ReadsArgs A{};
    A.groups = groups; A.n = n; A.G = e->G; A.chunk = chunk_size; A.W = e->W; A.d = e->majority; A.variant = reconstruct_variant;
    A.log_start = e->log_start; A.last_exec = e->last_exec; A.last_commit = e->last_commit; A.terms = e->terms; A.held = e->held;
    A.last_recon = e->last_recon;
    A.cnt = e->rc_words; A.bytes = e->rc_words + n; A.recon0 = e->rc_words + 2u * n;
    uint64_t *partials = e->rc_words + 3u * n, *tot = totals != nullptr ? totals : partials + scan_tiles(n);
    A.totals = tot;
    A.out = out; A.out_cap = out_capacity; A.frame_group = frame_group; A.frame_dst = frame_dst; A.frame_off = frame_off;
    A.frame_len = frame_len; A.frame_cap = frame_capacity; A.status = ctx->dev_status; A.led = e->led;
    const uint32_t grid = launch_grid(ctx, n, kRcThreads);
    if (e->led != nullptr) recon_size_kernel<true><<<grid, kRcThreads, 0, ctx->stream>>>(A);
    else recon_size_kernel<false><<<grid, kRcThreads, 0, ctx->stream>>>(A);
    SS_TRY(launched(ctx));
    SS_TRY(launch_exclusive_scan_u64(ctx, A.cnt, n, partials, tot));
    SS_TRY(launch_exclusive_scan_u64(ctx, A.bytes, n, partials, tot + 1));
    if (e->led != nullptr) recon_write_kernel<true><<<grid, kRcThreads, 0, ctx->stream>>>(A);
    else recon_write_kernel<false><<<grid, kRcThreads, 0, ctx->stream>>>(A);
    return launched(ctx);
}

int ss_follower_reconstruct_serve(ss_follower *f, const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off,
                                  const uint32_t *frame_group, const uint8_t *frame_peer, uint64_t n, uint32_t reconstruct_variant,
                                  uint32_t reply_variant, uint8_t *out, uint64_t out_capacity, uint64_t *reply_off,
                                  uint64_t *reply_len, uint32_t *verdict, uint64_t *total) {
    if (f == nullptr) return set_error(SS_ERR_INVALID_ARG, "null follower");
    if (reconstruct_variant >= kVariantLimit || reply_variant >= kVariantLimit)
        return set_error(SS_ERR_INVALID_ARG, "the variants must be < 2^16");
    ss_ctx *ctx = f->ctx;
    SS_TRY(ctx_bind(ctx));
    if (n == 0) {
        if (total != nullptr) SS_CUDA(cudaMemsetAsync(total, 0, 8, ctx->stream));
        return SS_OK;
    }
    if (!buf || !frame_off || !frame_group || !frame_peer || !out || !reply_off || !reply_len || !verdict)
        return set_error(SS_ERR_INVALID_ARG, "null buffer");
    if (reinterpret_cast<uintptr_t>(out) & 15u) return set_error(SS_ERR_INVALID_ARG, "out must be 16-byte aligned");
    if (n > 0x7fffffffull) return set_error(SS_ERR_INVALID_ARG, "at most 2^31 - 1 frames per call");
    SS_TRY(fol_scratch(f, n));
    ServeArgs A{};
    A.buf = buf; A.buf_len = buf_len; A.frame_off = frame_off; A.frame_group = frame_group; A.n = n; A.G = f->G;
    A.d = f->d; A.T = f->T; A.FW = f->W; A.variant = reconstruct_variant; A.reply_variant = reply_variant;
    A.start_slot = f->start_slot; A.log_end = f->log_end; A.term = f->term; A.shard_addr = f->shard_addr; A.held = f->held;
    A.data_len = f->data_len;
    A.out = out; A.out_cap = out_capacity; A.reply_off = reply_off; A.reply_len = reply_len; A.verdict = verdict;
    A.status = ctx->dev_status;
    serve_size_kernel<<<launch_grid(ctx, n, kRcThreads), kRcThreads, 0, ctx->stream>>>(A);
    SS_TRY(launched(ctx));
    SS_TRY(launch_exclusive_scan_u64(ctx, reply_off, n, f->partials, total != nullptr ? total : f->words + 2));
    serve_write_kernel<<<launch_grid(ctx, n, kRcThreads / 32), kRcThreads, 0, ctx->stream>>>(A);
    return launched(ctx);
}

int ss_engine_craft_absorb(ss_engine *e, const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off, const uint32_t *frame_group,
                           const uint8_t *frame_peer, uint64_t n, uint32_t reply_variant, uint32_t *absorbed, uint32_t *verdict) {
    if (reply_variant >= kVariantLimit) return set_error(SS_ERR_INVALID_ARG, "reply_variant must be < 2^16");
    SS_TRY(craft_check(e));
    if (n > 0x7fffffffull) return set_error(SS_ERR_INVALID_ARG, "at most 2^31 - 1 frames per call");
    if (n != 0 && (!buf || !frame_off || !frame_group || !frame_peer || !absorbed || !verdict)) return set_error(SS_ERR_INVALID_ARG, "null buffer");
    SS_TRY(craft_log_init(e));
    SS_TRY(craft_held_in_use(e));                                           // it reads held
    if (n == 0) return SS_OK;
    ss_ctx *ctx = e->ctx;
    // keys run 0..G; the sort scratch is the back-off's, sized for its (population - 1) * G keys
    const int bits = key_bits(uint64_t(e->n_peers) * e->G);
    SS_TRY(rc_scratch(e, 3u * n));                                          // each frame's entry offset, count, repeat flag
    SS_TRY(backoff_scratch(e, n, bits));
    AbsorbArgs A{};
    A.buf = buf; A.buf_len = buf_len; A.frame_off = frame_off; A.frame_group = frame_group; A.n = n; A.G = e->G;
    A.W = e->W; A.d = e->majority; A.T = e->n; A.variant = reply_variant; A.plane_stride = e->log_plane_stride;
    A.log_start = e->log_start; A.ent_addr = e->ent_addr; A.log_end = e->log_end; A.ent_len = e->ent_len; A.held = e->held;
    A.fr_at = e->rc_words; A.key_in = e->bo_keys; A.idx_in = e->bo_idx; A.key = e->bo_keys + n; A.idx = e->bo_idx + n;
    A.absorbed = absorbed; A.verdict = verdict;
    absorb_head_kernel<<<launch_grid(ctx, n, kRcThreads), kRcThreads, 0, ctx->stream>>>(A);
    SS_TRY(launched(ctx));
    size_t bytes = e->bo_sort_bytes;
    SS_CUDA(cub::DeviceRadixSort::SortPairs(e->bo_sort_tmp, bytes, e->bo_keys, e->bo_keys + n, e->bo_idx, e->bo_idx + n, static_cast<int>(n), 0,
                                            bits, ctx->stream));
    SS_TRY(launched(ctx));
    absorb_apply_kernel<<<launch_grid(ctx, n, kRcThreads / 32), kRcThreads, 0, ctx->stream>>>(A);
    return launched(ctx);
}

}  // extern "C"
