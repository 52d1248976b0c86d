// engine.cu -- the batched multi-group consensus engine behind the C ABI (ss_engine_*).
//
// One handle holds the leader-side state of G independent replica groups as a struct of arrays in HBM and advances
// all of them together; the host (the Rust shim of INTEGRATION.md, or summerset_b200/engine.py) calls
//
//   ss_engine_propose   RSCodeword::from_data + compute_parity + per-peer subset_copy for every group's new instance
//   ss_engine_propose_next  (multipaxos/request.rs:112-221, rspaxos/request.rs:72-142, crossword/request.rs:82-185): the
//                       RS encode kernel writes the shard planes, one bookkeeping kernel moves the instance -- at a given
//                       window position, or at the group's first Null slot (rspaxos/mod.rs:434-442) -- to Accepting
//                       under the group's prepared ballot with an empty ack set
//   ss_engine_ingest    handle_msg_accept_reply's filters over a batch of AcceptReply records
//                       (multipaxos/messages.rs:377-409, rspaxos/messages.rs:402-437, crossword/messages.rs:489-530)
//   ss_engine_tick      the commit decision for every Accepting instance and the commit_bar advance, ONE kernel:
//                         MultiPaxos  accept_acks.count() >= quorum_cnt              (multipaxos/messages.rs:412-413)
//                         RSPaxos     count() >= majority + fault_tolerance          (rspaxos/messages.rs:438-440)
//                         Crossword   #acks >= majority && coverage_under_faults >= d (crossword/messages.rs:535-542)
//                       committed |= newly, accepting &= ~newly (a committed instance drops later replies, :394-399),
//                       commit_bar = committed prefix (multipaxos/durability.rs:161-170)
//   ss_engine_advance   retire a committed prefix: window_base moves forward (start_slot, multipaxos/snapshot.rs:121-171)
//   Raft / CRaft        ss_engine_raft_append (leader appends entries in its term), ss_engine_raft_ingest (successful
//                       AppendEntriesReply: next_slot / match_slot update, raft/messages.rs:243-252), ss_engine_tick
//                       (commit scan :254-275,295 and last_snap :298-309; CRaft thresholds craft/messages.rs:300-308)
//
// Paxos-family window: group g holds the absolute slots [window_base[g], window_base[g] + 64).  Every per-slot array is
// a ring: absolute slot s lives at position s & 63 (bit s & 63 of the ack planes, accepting and committed; entry
// g*64 + (s & 63) of inst_bal and policy_idx).  commit_bar and the tick's newly words are window-relative (bit i =
// slot window_base + i): ring words are rotated right by window_base & 63.  At window_base == 0 both orders coincide.
//
// No tally, filter or shard byte is computed on the host, and nothing here is a torch op.
#include <cstring>
#include <new>

#include "device_common.cuh"
#include "engine_state.hpp"
#include "ss_internal.hpp"
#include "window_ring.cuh"

namespace ssb {

constexpr int kEngThreads = 256;

static inline uint32_t eng_grid(ss_ctx *ctx, uint64_t items) {
    uint64_t ctas = (items + kEngThreads - 1) / kEngThreads;
    const uint64_t cap = static_cast<uint64_t>(ctx->sm_count) * 8ull * 4ull;
    if (ctas > cap) ctas = cap;
    if (ctas == 0) ctas = 1;
    return static_cast<uint32_t>(ctas);
}

// ---- propose bookkeeping: one new instance per group enters Accepting --------------------------------------------
// window position of the group's first Null slot (rspaxos/mod.rs:434-442); 64 = the window is full
__device__ __forceinline__ uint32_t first_null(uint64_t acc, uint64_t cm, uint64_t base) {
    return dev::commit_prefix(ring_to_window(acc | cm, static_cast<uint32_t>(base & 63u)));
}

// one status write per warp, not one per flagged group
__device__ __forceinline__ void warp_status(bool flag, uint32_t bit, uint32_t *status) {
    const unsigned any = __ballot_sync(__activemask(), flag);
    if (flag && (threadIdx.x & 31u) == static_cast<unsigned>(__ffs(static_cast<int>(any)) - 1)) atomicOr(status, bit);
}

// slot < 64: at window position `slot`; slot == kProposeNext: at the group's first Null slot, which a full window does
// not have -- then slot_out = UINT64_MAX, the status bit is set and the group is left as is.
constexpr uint32_t kProposeNext = 64;
__global__ void __launch_bounds__(kEngThreads)
engine_propose_kernel(uint64_t *__restrict__ planes, uint32_t R, uint64_t G, uint32_t slot, const uint64_t *__restrict__ window_base,
                      const uint64_t *__restrict__ bal_prepared, uint64_t *__restrict__ inst_bal, uint64_t *__restrict__ accepting,
                      uint64_t *__restrict__ committed, uint8_t *__restrict__ policy_idx, const uint8_t *__restrict__ new_policy,
                      ss_cw_loc *__restrict__ cw_loc, const uint8_t *store, uint64_t shard_stride, uint64_t plane_stride,
                      uint32_t data_len, uint64_t *__restrict__ slot_out, uint32_t *status) {
    bool full = false;
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kEngThreads;
    for (uint64_t g = static_cast<uint64_t>(blockIdx.x) * kEngThreads + threadIdx.x; g < G; g += stride) {
        const uint64_t base = window_base[g];
        const uint64_t acc = accepting[g], cm = committed[g];
        uint32_t rel = slot;
        if (slot == kProposeNext) {
            rel = first_null(acc, cm, base);
            if (rel == 64u) {
                full = true;
                if (slot_out != nullptr) slot_out[g] = ~0ull;
                continue;
            }
        }
        const uint64_t s = base + rel;
        enter_accepting(g, s, acc, cm, planes, R, G, bal_prepared, inst_bal, accepting, committed, policy_idx, new_policy, cw_loc,
                        store + g * shard_stride, plane_stride, data_len);
        if (slot_out != nullptr) slot_out[g] = s;
    }
    warp_status(full, SS_DEV_STATUS_WINDOW_FULL, status);
}

// ---- ragged proposals (ss_engine_propose_ragged) ------------------------------------------------------------------
// 1. prepare: a group proposes when it has a batch (data_len > 0) and its window a Null slot; its effective length is
//    then data_len, its pitch SS_CW_SLOT_PITCH(ceil(data_len / d)), else both are 0.  The pitches go to shard_off, which
//    the scan then turns into slot offsets in place.
__global__ void __launch_bounds__(kEngThreads)
engine_ragged_prepare_kernel(const uint32_t *__restrict__ data_len, uint64_t G, uint32_t d, const uint64_t *__restrict__ window_base,
                             const uint64_t *__restrict__ accepting, const uint64_t *__restrict__ committed,
                             uint32_t *__restrict__ eff_len, uint64_t *__restrict__ pitch, uint32_t *status) {
    bool full = false;
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kEngThreads;
    for (uint64_t g = static_cast<uint64_t>(blockIdx.x) * kEngThreads + threadIdx.x; g < G; g += stride) {
        uint32_t len = data_len[g];
        if (len != 0u && first_null(accepting[g], committed[g], window_base[g]) == 64u) {
            full = true;
            len = 0u;
        }
        eff_len[g] = len;
        pitch[g] = len == 0u ? 0ull : SS_CW_SLOT_PITCH((static_cast<uint64_t>(len) + d - 1u) / d);
    }
    warp_status(full, SS_DEV_STATUS_WINDOW_FULL, status);
}

// 3. clamp + bookkeeping: shard_off holds the exclusive prefix of the pitches.  A proposing group whose slot ends past
//    the plane capacity is dropped (effective length 0, status bit); the others enter Accepting at their first Null slot.
//    Groups that do not propose get shard_off = slot_out = UINT64_MAX.
__global__ void __launch_bounds__(kEngThreads)
engine_ragged_commit_kernel(uint32_t *__restrict__ eff_len, uint64_t *__restrict__ shard_off, uint64_t capacity, uint32_t d,
                            uint64_t *__restrict__ planes, uint32_t R, uint64_t G, const uint64_t *__restrict__ window_base,
                            const uint64_t *__restrict__ bal_prepared, uint64_t *__restrict__ inst_bal,
                            uint64_t *__restrict__ accepting, uint64_t *__restrict__ committed, uint8_t *__restrict__ policy_idx,
                            const uint8_t *__restrict__ new_policy, ss_cw_loc *__restrict__ cw_loc, const uint8_t *shards,
                            uint64_t *__restrict__ slot_out, uint32_t *status) {
    bool over = false;
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kEngThreads;
    for (uint64_t g = static_cast<uint64_t>(blockIdx.x) * kEngThreads + threadIdx.x; g < G; g += stride) {
        const uint32_t len = eff_len[g];
        const uint64_t off = shard_off[g];
        const uint64_t pitch = SS_CW_SLOT_PITCH((static_cast<uint64_t>(len) + d - 1u) / d);
        if (len == 0u || off > capacity || pitch > capacity - off) {
            if (len != 0u) {
                over = true;
                eff_len[g] = 0u;                               // the encode skips it
            }
            shard_off[g] = ~0ull;
            slot_out[g] = ~0ull;
            continue;
        }
        const uint64_t base = window_base[g];
        const uint64_t acc = accepting[g], cm = committed[g];
        const uint64_t s = base + first_null(acc, cm, base);   // not full: the prepare kernel checked the same words
        enter_accepting(g, s, acc, cm, planes, R, G, bal_prepared, inst_bal, accepting, committed, policy_idx, new_policy, cw_loc,
                        shards + off, capacity, len);
        slot_out[g] = s;
    }
    warp_status(over, SS_DEV_STATUS_STORE_FULL, status);
}

// ---- exclusive scan of u64 values, in place: reduce / scan / add ------------------------------------------------------
// Tiles of kScanTile values: the first pass writes each tile's sum, one CTA scans the sums (and writes the total), the
// last pass scans each tile again from its base.  Integer sums in a fixed order: the result is exactly numpy's
// cumsum shifted by one, on every run.
constexpr int kScanThreads = 256, kScanItems = 8, kScanTile = kScanThreads * kScanItems;

// exclusive scan of one value per thread across the CTA; *total (shared) receives the CTA's sum
__device__ __forceinline__ uint64_t cta_exclusive_scan(uint64_t v, uint64_t *warp_sums, uint64_t *total) {
    const uint32_t lane = threadIdx.x & 31u, wid = threadIdx.x >> 5;
    uint64_t x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint64_t y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= static_cast<uint32_t>(o)) x += y;
    }
    if (lane == 31u) warp_sums[wid] = x;
    __syncthreads();
    if (wid == 0) {
        uint64_t w = lane < kScanThreads / 32 ? warp_sums[lane] : 0ull;
#pragma unroll
        for (int o = 1; o < kScanThreads / 32; o <<= 1) {
            const uint64_t y = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= static_cast<uint32_t>(o)) w += y;
        }
        if (lane < kScanThreads / 32) warp_sums[lane] = w;           // inclusive over warps
        if (lane == kScanThreads / 32 - 1) *total = w;
    }
    __syncthreads();
    const uint64_t before = wid == 0 ? 0ull : warp_sums[wid - 1];
    const uint64_t r = before + x - v;
    __syncthreads();                                                 // warp_sums / total may be reused by the caller
    return r;
}

__global__ void __launch_bounds__(kScanThreads) scan_tile_sum_kernel(const uint64_t *__restrict__ x, uint64_t n,
                                                                     uint64_t *__restrict__ partials) {
    __shared__ uint64_t warp_sums[kScanThreads / 32], total;
    const uint64_t t0 = static_cast<uint64_t>(blockIdx.x) * kScanTile;
    uint64_t s = 0;
#pragma unroll
    for (int i = 0; i < kScanItems; ++i) {
        const uint64_t k = t0 + static_cast<uint64_t>(i) * kScanThreads + threadIdx.x;
        if (k < n) s += x[k];
    }
    cta_exclusive_scan(s, warp_sums, &total);
    if (threadIdx.x == 0) partials[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kScanThreads) scan_partials_kernel(uint64_t *__restrict__ partials, uint64_t tiles,
                                                                     uint64_t *__restrict__ total_out) {
    __shared__ uint64_t warp_sums[kScanThreads / 32], total;
    uint64_t carry = 0;
    for (uint64_t c = 0; c < tiles; c += kScanThreads) {
        const uint64_t k = c + threadIdx.x;
        const uint64_t v = k < tiles ? partials[k] : 0ull;
        const uint64_t e = cta_exclusive_scan(v, warp_sums, &total);
        if (k < tiles) partials[k] = carry + e;
        carry += total;
        __syncthreads();
    }
    if (threadIdx.x == 0 && total_out != nullptr) *total_out = carry;
}

__global__ void __launch_bounds__(kScanThreads) scan_tile_apply_kernel(uint64_t *__restrict__ x, uint64_t n,
                                                                       const uint64_t *__restrict__ partials) {
    __shared__ uint64_t tile[kScanTile + kScanTile / 32];            // one pad word per 32: the per-thread runs avoid bank conflicts
    __shared__ uint64_t warp_sums[kScanThreads / 32], total;
    auto at = [](uint32_t i) { return i + (i >> 5); };
    const uint64_t t0 = static_cast<uint64_t>(blockIdx.x) * kScanTile;
#pragma unroll
    for (int i = 0; i < kScanItems; ++i) {
        const uint32_t j = static_cast<uint32_t>(i) * kScanThreads + threadIdx.x;
        tile[at(j)] = t0 + j < n ? x[t0 + j] : 0ull;
    }
    __syncthreads();
    uint64_t v[kScanItems], s = 0;
#pragma unroll
    for (int i = 0; i < kScanItems; ++i) { v[i] = tile[at(threadIdx.x * kScanItems + i)]; s += v[i]; }
    uint64_t run = partials[blockIdx.x] + cta_exclusive_scan(s, warp_sums, &total);
#pragma unroll
    for (int i = 0; i < kScanItems; ++i) { tile[at(threadIdx.x * kScanItems + i)] = run; run += v[i]; }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < kScanItems; ++i) {
        const uint32_t j = static_cast<uint32_t>(i) * kScanThreads + threadIdx.x;
        if (t0 + j < n) x[t0 + j] = tile[at(j)];
    }
}

// ---- retire the committed prefix up to upto[g] (all of it when upto is NULL) ---------------------------------------
// multipaxos/snapshot.rs:121-171 moves start_slot past the executed prefix.  The retired ring positions are cleared in
// every per-slot bit word, so that a later proposal there starts with no acks and the tick's prefix does not see them.
__global__ void __launch_bounds__(kEngThreads)
engine_advance_kernel(const uint64_t *__restrict__ upto, uint64_t *__restrict__ planes, uint32_t R, uint64_t G,
                      uint64_t *__restrict__ window_base, uint64_t *__restrict__ accepting, uint64_t *__restrict__ committed,
                      uint32_t *__restrict__ commit_bar) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kEngThreads;
    for (uint64_t g = static_cast<uint64_t>(blockIdx.x) * kEngThreads + threadIdx.x; g < G; g += stride) {
        const uint64_t base = window_base[g];
        const uint64_t cm = committed[g];
        const uint32_t r = static_cast<uint32_t>(base & 63u);
        // only committed instances can be retired: the prefix of the committed word itself, so a commit_bar left stale
        // by a re-proposal at a committed position never retires an uncommitted instance
        const uint32_t bar = dev::commit_prefix(ring_to_window(cm, r));
        uint64_t k = bar;
        if (upto != nullptr) {
            const uint64_t u = upto[g];
            k = u <= base ? 0ull : (u - base < k ? u - base : k);
        }
        if (k == 0ull) continue;
        const uint64_t keep = ring_keep_after(k, base);
        committed[g] = cm & keep;
        accepting[g] &= keep;
        for (uint32_t q = 0; q < R; ++q) planes[static_cast<uint64_t>(q) * G + g] &= keep;
        window_base[g] = base + k;
        commit_bar[g] = bar - static_cast<uint32_t>(k);
    }
}

// ---- fused tick, threshold protocols: two groups per thread, 128-bit accesses ------------------------------------
// WIN = false: no base can be non-zero yet (the engine never advanced nor handed out window_base), so the ring is the
// window and the tick skips the 8 B/group load of window_base
template <int RT, bool WIN>
__global__ void __launch_bounds__(kEngThreads)
engine_tick_x2_kernel(const ulonglong2 *__restrict__ planes, uint32_t R, uint64_t G2, uint32_t threshold,
                      const ulonglong2 *__restrict__ window_base, ulonglong2 *__restrict__ accepting,
                      ulonglong2 *__restrict__ committed, uint2 *__restrict__ commit_bar, ulonglong2 *__restrict__ newly_out) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kEngThreads;
    for (uint64_t g = static_cast<uint64_t>(blockIdx.x) * kEngThreads + threadIdx.x; g < G2; g += stride) {
        uint64_t a[5] = {0, 0, 0, 0, 0}, b[5] = {0, 0, 0, 0, 0};
        auto add = [&](const ulonglong2 &x) {
            uint64_t c = x.x, t;
            t = a[0] & c; a[0] ^= c; c = t;
            t = a[1] & c; a[1] ^= c; c = t;
            t = a[2] & c; a[2] ^= c; c = t;
            t = a[3] & c; a[3] ^= c; c = t;
            a[4] ^= c;
            c = x.y;
            t = b[0] & c; b[0] ^= c; c = t;
            t = b[1] & c; b[1] ^= c; c = t;
            t = b[2] & c; b[2] ^= c; c = t;
            t = b[3] & c; b[3] ^= c; c = t;
            b[4] ^= c;
        };
        const ulonglong2 acc = accepting[g];
        ulonglong2 cm = committed[g];
        if constexpr (RT > 0) {
            ulonglong2 v[RT];
#pragma unroll
            for (int r = 0; r < RT; ++r) v[r] = __ldg(planes + static_cast<uint64_t>(r) * G2 + g);
#pragma unroll
            for (int r = 0; r < RT; ++r) add(v[r]);
        } else {
            for (uint32_t r = 0; r < R; ++r) add(__ldg(planes + static_cast<uint64_t>(r) * G2 + g));
        }
        auto ge = [&](const uint64_t (&cb)[5]) -> uint64_t {
            if (threshold == 0u) return ~0ull;
            if (threshold > 31u) return 0ull;
            uint64_t lt = 0ull, eq = ~0ull;
#pragma unroll
            for (int bb = 4; bb >= 0; --bb) {
                const uint64_t tb = ((threshold >> bb) & 1u) ? ~0ull : 0ull;
                lt |= eq & ~cb[bb] & tb;
                eq &= ~(cb[bb] ^ tb);
            }
            return ~lt;
        };
        ulonglong2 newly;
        newly.x = ge(a) & acc.x;                // only instances in Accepting can commit
        newly.y = ge(b) & acc.y;
        cm.x |= newly.x; cm.y |= newly.y;
        committed[g] = cm;
        accepting[g] = make_ulonglong2(acc.x & ~newly.x, acc.y & ~newly.y);
        const ulonglong2 base = WIN ? window_base[g] : make_ulonglong2(0ull, 0ull);
        const uint32_t rx = static_cast<uint32_t>(base.x & 63u), ry = static_cast<uint32_t>(base.y & 63u);
        commit_bar[g] = make_uint2(dev::commit_prefix(ring_to_window(cm.x, rx)), dev::commit_prefix(ring_to_window(cm.y, ry)));
        if (newly_out != nullptr) newly_out[g] = make_ulonglong2(ring_to_window(newly.x, rx), ring_to_window(newly.y, ry));
    }
}

template <bool WIN>
__global__ void __launch_bounds__(kEngThreads)
engine_tick_kernel(const uint64_t *__restrict__ planes, uint32_t R, uint64_t G, uint32_t threshold,
                   const uint64_t *__restrict__ window_base, uint64_t *__restrict__ accepting, uint64_t *__restrict__ committed,
                   uint32_t *__restrict__ commit_bar, uint64_t *__restrict__ newly_out) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kEngThreads;
    for (uint64_t g = static_cast<uint64_t>(blockIdx.x) * kEngThreads + threadIdx.x; g < G; g += stride) {
        const uint64_t acc = accepting[g];
        const uint64_t newly = dev::tally_word(planes, R, G, g, threshold) & acc;
        const uint64_t cm = committed[g] | newly;
        committed[g] = cm;
        accepting[g] = acc & ~newly;
        const uint32_t r = WIN ? static_cast<uint32_t>(window_base[g] & 63u) : 0u;
        commit_bar[g] = dev::commit_prefix(ring_to_window(cm, r));
        if (newly_out != nullptr) newly_out[g] = ring_to_window(newly, r);
    }
}

// ---- fused tick, Crossword: coverage look-up per Accepting instance ------------------------------------------------
template <bool WIN>
__global__ void __launch_bounds__(kEngThreads)
engine_tick_crossword_kernel(const uint64_t *__restrict__ planes, uint32_t R, uint64_t G, const uint8_t *__restrict__ policy_idx,
                             const uint32_t *__restrict__ lut_bits, uint32_t lut_words, uint32_t n_policies,
                             const uint64_t *__restrict__ window_base, uint64_t *__restrict__ accepting,
                             uint64_t *__restrict__ committed, uint32_t *__restrict__ commit_bar, uint64_t *__restrict__ newly_out) {
    extern __shared__ uint32_t lut[];
    for (uint32_t i = threadIdx.x; i < lut_words; i += kEngThreads) lut[i] = lut_bits[i];
    __syncthreads();
    const uint32_t nmask = 1u << R;
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kEngThreads;
    for (uint64_t g = static_cast<uint64_t>(blockIdx.x) * kEngThreads + threadIdx.x; g < G; g += stride) {
        const uint64_t acc = accepting[g];
        uint64_t newly = 0ull;
        if (acc != 0ull) {
            uint64_t pl[12];
#pragma unroll
            for (int r = 0; r < 12; ++r) pl[r] = static_cast<uint32_t>(r) < R ? __ldg(planes + static_cast<uint64_t>(r) * G + g) : 0ull;
            uint64_t rem = acc;
            while (rem) {
                const int s = __ffsll(static_cast<long long>(rem)) - 1;
                rem &= rem - 1ull;
                uint32_t ack = 0;
#pragma unroll
                for (int r = 0; r < 12; ++r) ack |= static_cast<uint32_t>((pl[r] >> s) & 1ull) << r;
                const uint32_t k = policy_idx[g * 64 + s];
                if (k < n_policies) {
                    const uint32_t e = k * nmask + ack;
                    if ((lut[e >> 5] >> (e & 31u)) & 1u) newly |= 1ull << s;
                }
            }
        }
        const uint64_t cm = committed[g] | newly;
        committed[g] = cm;
        accepting[g] = acc & ~newly;
        const uint32_t r = WIN ? static_cast<uint32_t>(window_base[g] & 63u) : 0u;
        commit_bar[g] = dev::commit_prefix(ring_to_window(cm, r));
        if (newly_out != nullptr) newly_out[g] = ring_to_window(newly, r);
    }
}

// ---- Raft ----------------------------------------------------------------------------------------------------------
// leader appends n_new[g] entries in its current term (raft/request.rs: log.push(LogEntry{term: curr_term, ..}))
__global__ void __launch_bounds__(kEngThreads)
engine_raft_append_kernel(const uint32_t *__restrict__ n_new, uint64_t G, uint32_t W, const uint32_t *__restrict__ curr_term,
                          const uint32_t *__restrict__ last_commit, uint32_t *__restrict__ log_end, uint32_t *__restrict__ terms,
                          uint32_t *status) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kEngThreads;
    for (uint64_t g = static_cast<uint64_t>(blockIdx.x) * kEngThreads + threadIdx.x; g < G; g += stride) {
        const uint32_t k = n_new[g];
        if (k == 0u) continue;
        const uint32_t le = log_end[g], ct = curr_term[g];
        // the ring holds the terms of slots last_commit+1 .. log_end-1: appending past W uncommitted entries would
        // overwrite one that the scan still needs
        if (le + k - last_commit[g] - 1u > W) { atomicOr(status, 2u); continue; }
        for (uint32_t i = 0; i < k; ++i) terms[g * W + ((le + i) & (W - 1u))] = ct;
        log_end[g] = le + k;
    }
}

// successful AppendEntriesReply (raft/messages.rs:243-252): ignored when next_slot[peer] > end_slot + 1, else
// next_slot = end_slot + 1 and match_slot = end_slot.  next only ever holds accepted end_slot + 1 values, so within a
// batch the outcome is the maximum in any order: atomicMax models it exactly.
__global__ void __launch_bounds__(kEngThreads)
engine_raft_ingest_kernel(const uint32_t *__restrict__ rec_group, const uint8_t *__restrict__ rec_peer,
                          const uint32_t *__restrict__ rec_end_slot, uint64_t n_rec, uint32_t P, uint64_t G,
                          uint32_t *next_slot, uint32_t *match, uint8_t *touched) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kEngThreads;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kEngThreads + threadIdx.x; i < n_rec; i += stride) {
        const uint64_t g = rec_group[i];
        const uint32_t peer = rec_peer[i], end = rec_end_slot[i];
        if (g >= G || peer >= P) continue;
        const uint64_t at = static_cast<uint64_t>(peer) * G + g;
        const uint32_t old = atomicMax(next_slot + at, end + 1u);
        if (old > end + 1u) continue;                          // :245-247
        atomicMax(match + at, end);
        touched[g] = 1;
    }
}

// last_snap advance (raft/messages.rs:298-309): after an accepted reply, the last slot every server stores
template <int NP>
__global__ void __launch_bounds__(kEngThreads)
engine_raft_snap_kernel(const uint32_t *__restrict__ match, uint32_t P, uint64_t G, uint8_t *__restrict__ touched,
                        uint32_t *__restrict__ last_snap) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kEngThreads;
    for (uint64_t g = static_cast<uint64_t>(blockIdx.x) * kEngThreads + threadIdx.x; g < G; g += stride) {
        if (!touched[g]) continue;
        touched[g] = 0;
        uint32_t mn = 0xffffffffu;
#pragma unroll
        for (int q = 0; q < NP; ++q)
            if (static_cast<uint32_t>(q) < P) { const uint32_t v = __ldg(match + static_cast<uint64_t>(q) * G + g); mn = v < mn ? v : mn; }
        if (P != 0u && mn > last_snap[g]) last_snap[g] = mn;
    }
}

uint64_t scan_tiles(uint64_t n) { return (n + kScanTile - 1) / kScanTile; }

int launch_exclusive_scan_u64(ss_ctx *ctx, uint64_t *x, uint64_t n, uint64_t *partials, uint64_t *total) {
    const uint64_t tiles = scan_tiles(n);
    if (tiles == 0) {
        if (total != nullptr) SS_CUDA(cudaMemsetAsync(total, 0, 8, ctx->stream));
        return SS_OK;
    }
    if (tiles > 0x7fffffffull) return set_error(SS_ERR_INVALID_ARG, "scan of %llu values is too long", (unsigned long long)n);
    const uint32_t grid = static_cast<uint32_t>(tiles);
    scan_tile_sum_kernel<<<grid, kScanThreads, 0, ctx->stream>>>(x, n, partials);
    scan_partials_kernel<<<1, kScanThreads, 0, ctx->stream>>>(partials, tiles, total);
    scan_tile_apply_kernel<<<grid, kScanThreads, 0, ctx->stream>>>(x, n, partials);
    SS_CUDA(cudaGetLastError());
    ctx->launches += 3;
    return SS_OK;
}

}  // namespace ssb

using namespace ssb;

extern "C" {

int ss_engine_destroy(ss_engine *e) {
    if (e == nullptr) return SS_OK;
    if (e->ctx) {
        cudaSetDevice(e->ctx->device);
        cudaStreamSynchronize(e->ctx->stream);
    }
    void *bufs[] = {e->planes, e->bal_prepared, e->inst_bal, e->accepting, e->committed, e->window_base, e->commit_bar, e->shards, e->policy_idx,
                    e->policies, e->lut_bits, e->match, e->next_slot, e->last_commit, e->log_end, e->curr_term, e->terms,
                    e->last_snap, e->touched, e->rg_len, e->rg_partials, e->rg_need, e->cw_loc};
    for (void *b : bufs)
        if (b) cudaFree(b);
    craft_log_free(e);
    prepare_free(e);
    fallback_free(e);
    if (e->coder) ss_rs_coder_destroy(e->coder);
    if (e->ctx) ctx_release(e->ctx);
    delete e;
    return SS_OK;
}

int ss_engine_create(ss_ctx *ctx, const ss_engine_config *cfg, uint64_t G, ss_engine **out) {
    if (out == nullptr) return set_error(SS_ERR_INVALID_ARG, "null out pointer");
    *out = nullptr;
    SS_TRY(ctx_bind(ctx));
    if (cfg == nullptr || G == 0) return set_error(SS_ERR_INVALID_ARG, "null config or zero groups");
    const uint32_t n = cfg->population;
    if (n == 0 || n > 12) return set_error(SS_ERR_INVALID_ARG, "population must be 1..12, got %u", n);
    const uint32_t majority = n / 2 + 1;
    if (cfg->protocol > SS_PROTO_CRAFT) return set_error(SS_ERR_INVALID_ARG, "unknown protocol %u", cfg->protocol);
    // fault_tolerance <= population - majority (rspaxos/mod.rs:599-605, crossword/mod.rs:752-760)
    if (cfg->protocol != SS_PROTO_MULTIPAXOS && cfg->protocol != SS_PROTO_RAFT && cfg->fault_tolerance > n - majority)
        return set_error(SS_ERR_INVALID_ARG, "invalid fault_tolerance %u for population %u", cfg->fault_tolerance, n);
    ss_engine *e = new (std::nothrow) ss_engine();
    if (!e) return set_error(SS_ERR_OUT_OF_MEMORY, "host allocation failed");
    e->ctx = ctx; e->cfg = *cfg; e->G = G; e->n = n; e->majority = majority;
    ctx_retain(ctx);
    int rc = SS_OK;
    auto fail = [&](int code) { ss_engine_destroy(e); return code; };
    const bool raft = cfg->protocol == SS_PROTO_RAFT || cfg->protocol == SS_PROTO_CRAFT;
    if (raft) {
        e->n_peers = n - 1;
        e->W = cfg->raft_window ? cfg->raft_window : 64;
        if ((e->W & (e->W - 1)) || e->W > 4096) return fail(set_error(SS_ERR_INVALID_ARG, "raft_window must be a power of two <= 4096"));
        // quorum_cnt (raft/mod.rs), or CRaft's majority + f (craft/messages.rs:300-308; full-copy mode = plain Raft)
        e->threshold = cfg->protocol == SS_PROTO_CRAFT ? majority + cfg->fault_tolerance : majority;
        if ((rc = dalloc(ctx, &e->match, size_t(e->n_peers) * G)) || (rc = dalloc(ctx, &e->next_slot, size_t(e->n_peers) * G)) ||
            (rc = dalloc(ctx, &e->last_commit, G)) || (rc = dalloc(ctx, &e->log_end, G)) || (rc = dalloc(ctx, &e->curr_term, G)) ||
            (rc = dalloc(ctx, &e->terms, G * e->W)) || (rc = dalloc(ctx, &e->last_snap, G)) || (rc = dalloc(ctx, &e->touched, G)))
            return fail(rc);
        // slot 0 is the sentinel entry (raft/mod.rs: log starts with a dummy entry): next_slot = 1, log_end = 1
        // on the context's stream, after the zeroing above; `ones` lives until the copies have completed
        std::vector<uint32_t> ones(size_t(e->n_peers) * G > G ? size_t(e->n_peers) * G : G, 1u);
        cudaError_t ce = cudaMemcpyAsync(e->next_slot, ones.data(), size_t(e->n_peers) * G * 4, cudaMemcpyHostToDevice, ctx->stream);
        if (ce == cudaSuccess) ce = cudaMemcpyAsync(e->log_end, ones.data(), G * 4, cudaMemcpyHostToDevice, ctx->stream);
        if (ce == cudaSuccess) ce = cudaStreamSynchronize(ctx->stream);
        if (ce != cudaSuccess) return fail(cuda_error(ce, "initialise Raft state", __FILE__, __LINE__));
        *out = e;
        return SS_OK;
    }
    // ---- Paxos family ----
    switch (cfg->protocol) {
        case SS_PROTO_MULTIPAXOS: e->threshold = majority; e->d = 1; e->T = 1; break;                     // quorum_cnt (multipaxos/mod.rs:774)
        case SS_PROTO_RSPAXOS: e->threshold = majority + cfg->fault_tolerance; e->d = majority; e->T = n; break;
        default: {                                                                                       // crossword/mod.rs:805-830
            e->T = cfg->rs_total_shards ? cfg->rs_total_shards : n;
            e->d = cfg->rs_data_shards ? cfg->rs_data_shards : majority;
            if (e->T < n) e->T = n;
            if (e->d < majority) e->d = majority;
            if (e->T % n != 0 || e->d >= e->T || e->T > 32)
                return fail(set_error(SS_ERR_INVALID_ARG, "invalid Crossword code (T=%u, d=%u, n=%u)", e->T, e->d, n));
            e->threshold = 0;
        }
    }
    if ((rc = dalloc(ctx, &e->planes, size_t(n) * G)) || (rc = dalloc(ctx, &e->bal_prepared, G)) || (rc = dalloc(ctx, &e->inst_bal, G * 64)) ||
        (rc = dalloc(ctx, &e->accepting, G)) || (rc = dalloc(ctx, &e->committed, G)) || (rc = dalloc(ctx, &e->window_base, G)) ||
        (rc = dalloc(ctx, &e->commit_bar, G)))
        return fail(rc);
    if (cfg->protocol != SS_PROTO_MULTIPAXOS) {
        if (cfg->data_len == 0) return fail(set_error(SS_ERR_INVALID_ARG, "data_len must be > 0 for an RS-coded protocol"));
        if ((rc = ss_rs_coder_create(ctx, static_cast<int>(e->d), static_cast<int>(e->T - e->d), &e->coder))) return fail(rc);
        e->L = (cfg->data_len + e->d - 1) / e->d;
        e->ds = (e->L + 15u) & ~15u;
        const uint32_t keep = cfg->keep_slots ? cfg->keep_slots : 1;
        e->cfg.keep_slots = keep;
        if ((rc = dalloc(ctx, &e->shards, size_t(keep) * e->T * G * e->ds))) return fail(rc);
    }
    if (cfg->protocol == SS_PROTO_CROSSWORD) {
        if (G * e->ds >= kCwLocStrideLimit)
            return fail(set_error(SS_ERR_INVALID_ARG, "a Crossword engine's shard plane (n_groups * shard_stride) must be below 2^36 bytes"));
        if ((rc = dalloc(ctx, &e->policy_idx, G * 64)) || (rc = dalloc(ctx, &e->cw_loc, G * 64))) return fail(rc);
    }
    *out = e;
    return SS_OK;
}

int ss_engine_view_get(ss_engine *e, ss_engine_view *v) {
    if (e == nullptr || v == nullptr) return set_error(SS_ERR_INVALID_ARG, "null argument");
    memset(v, 0, sizeof(*v));
    v->n_groups = e->G; v->population = e->n; v->threshold = e->threshold; v->data_shards = e->d; v->total_shards = e->T;
    v->shard_len = e->L; v->shard_stride = e->ds; v->plane_stride = e->G * e->ds; v->slot_stride = uint64_t(e->T) * e->G * e->ds;
    v->planes = e->planes; v->bal_prepared = e->bal_prepared; v->inst_bal = e->inst_bal; v->accepting = e->accepting;
    v->committed = e->committed; v->commit_bar = e->commit_bar; v->shards = e->shards; v->policy_idx = e->policy_idx;
    v->match = e->match; v->next_slot = e->next_slot; v->last_commit = e->last_commit; v->log_end = e->log_end;
    v->curr_term = e->curr_term; v->terms = e->terms; v->last_snap = e->last_snap; v->raft_window = e->W;
    return SS_OK;
}

int ss_engine_set_prepared_ballots(ss_engine *e, const uint64_t *ballots_dev) {
    if (e == nullptr || ballots_dev == nullptr) return set_error(SS_ERR_INVALID_ARG, "null argument");
    if (e->bal_prepared == nullptr) return set_error(SS_ERR_INVALID_ARG, "not a Paxos-family engine");
    SS_TRY(ctx_bind(e->ctx));
    SS_CUDA(cudaMemcpyAsync(e->bal_prepared, ballots_dev, e->G * 8, cudaMemcpyDeviceToDevice, e->ctx->stream));
    return SS_OK;
}

int ss_engine_set_policies(ss_engine *e, const uint32_t *policies_host, uint32_t n_policies, int balanced) {
    if (e == nullptr || policies_host == nullptr) return set_error(SS_ERR_INVALID_ARG, "null argument");
    if (e->cfg.protocol != SS_PROTO_CROSSWORD) return set_error(SS_ERR_INVALID_ARG, "not a Crossword engine");
    if (n_policies == 0 || n_policies > 16) return set_error(SS_ERR_INVALID_ARG, "n_policies must be 1..16");
    ss_ctx *ctx = e->ctx;
    SS_TRY(ctx_bind(ctx));
    SS_CUDA(cudaStreamSynchronize(ctx->stream));
    if (e->policies) { cudaFree(e->policies); e->policies = nullptr; }
    if (e->lut_bits) { cudaFree(e->lut_bits); e->lut_bits = nullptr; }
    const uint32_t entries = n_policies << e->n;
    e->lut_words = (entries + 31) / 32;
    e->n_policies = n_policies;
    e->balanced = balanced;
    SS_TRY(dalloc(ctx, &e->policies, size_t(n_policies) * e->n, false));
    SS_TRY(dalloc(ctx, &e->lut_bits, e->lut_words));
    // stream-ordered before the table kernel; from pageable memory the call returns once the bytes are staged
    SS_CUDA(cudaMemcpyAsync(e->policies, policies_host, size_t(n_policies) * e->n * 4, cudaMemcpyHostToDevice, ctx->stream));
    return launch_crossword_lut(ctx, e->policies, n_policies, e->n, e->T, e->d, e->majority, e->cfg.fault_tolerance, balanced,
                                e->lut_bits);
}

// both propose calls: encode into shard store `store`, then the bookkeeping kernel at window position `slot`
// (kProposeNext: the first Null slot)
static int engine_propose(ss_engine *e, uint32_t store, uint32_t slot, const uint8_t *payloads, uint64_t payload_stride,
                          const uint8_t *policy, uint64_t *slot_out, uint8_t **shard_planes) {
    ss_ctx *ctx = e->ctx;
    SS_TRY(ctx_bind(ctx));
    if (e->cfg.protocol == SS_PROTO_CROSSWORD && e->lut_bits == nullptr)
        return set_error(SS_ERR_INVALID_ARG, "ss_engine_set_policies must be called before proposing");
    if (e->coder != nullptr) {
        if (payloads == nullptr) return set_error(SS_ERR_INVALID_ARG, "null payloads");
        uint8_t *base = e->shards + uint64_t(store) * e->T * e->G * e->ds;
        // from_data + compute_parity + the per-peer packed buffers of subset_copy: data shards into planes 0..d-1,
        // parity into planes d..T-1 (rspaxos/request.rs:72-77,127-142)
        SS_TRY(ss_rs_encode_uniform_dev(e->coder, payloads, payload_stride, e->cfg.data_len, e->G, base + uint64_t(e->d) * e->G * e->ds,
                                        e->G * e->ds, e->ds, SS_RS_OUT_PADDED16 | SS_RS_EMIT_DATA));
        if (shard_planes) *shard_planes = base;
    } else if (shard_planes) {
        *shard_planes = nullptr;                  // MultiPaxos sends the full batch to every peer: nothing to code
    }
    engine_propose_kernel<<<eng_grid(ctx, e->G), kEngThreads, 0, ctx->stream>>>(e->planes, e->n, e->G, slot, e->window_base,
                                                                             e->bal_prepared, e->inst_bal, e->accepting, e->committed,
                                                                             e->policy_idx, policy, e->cw_loc, e->shards + uint64_t(store) * e->T * e->G * e->ds,
                                                                             e->ds, e->G * e->ds, e->cfg.data_len, slot_out, ctx->dev_status);
    return launched(ctx);
}

int ss_engine_propose(ss_engine *e, uint32_t slot, const uint8_t *payloads, uint64_t payload_stride, const uint8_t *policy,
                      uint8_t **shard_planes) {
    if (e == nullptr) return set_error(SS_ERR_INVALID_ARG, "null engine");
    if (e->planes == nullptr) return set_error(SS_ERR_INVALID_ARG, "not a Paxos-family engine");
    if (slot >= 64) return set_error(SS_ERR_INVALID_ARG, "slot %u outside the 64-slot window", slot);
    const uint32_t store = e->coder != nullptr ? slot % e->cfg.keep_slots : 0;
    return engine_propose(e, store, slot, payloads, payload_stride, policy, nullptr, shard_planes);
}

int ss_engine_propose_next(ss_engine *e, uint32_t store, const uint8_t *payloads, uint64_t payload_stride, const uint8_t *policy,
                           uint64_t *slot_out, uint8_t **shard_planes) {
    if (e == nullptr) return set_error(SS_ERR_INVALID_ARG, "null engine");
    if (e->planes == nullptr) return set_error(SS_ERR_INVALID_ARG, "not a Paxos-family engine");
    const uint32_t keep = e->cfg.keep_slots ? e->cfg.keep_slots : 1;
    if (store >= keep) return set_error(SS_ERR_INVALID_ARG, "shard store %u >= keep_slots %u", store, keep);
    return engine_propose(e, store, kProposeNext, payloads, payload_stride, policy, slot_out, shard_planes);
}

int ss_engine_propose_ragged(ss_engine *e, const uint8_t *arena, const uint64_t *data_off, const uint32_t *data_len,
                             const uint8_t *policy, uint8_t *shards, uint64_t plane_stride, uint64_t *shard_off,
                             uint64_t *slot_out, uint64_t *need) {
    if (e == nullptr) return set_error(SS_ERR_INVALID_ARG, "null engine");
    if (e->planes == nullptr || e->coder == nullptr) return set_error(SS_ERR_INVALID_ARG, "ragged proposals need an RSPaxos or Crossword engine");
    if (!arena || !data_off || !data_len || !shards || !shard_off || !slot_out) return set_error(SS_ERR_INVALID_ARG, "null buffer");
    if ((plane_stride & 31u) || plane_stride == 0) return set_error(SS_ERR_INVALID_ARG, "plane_stride must be a non-zero multiple of 32");
    if (reinterpret_cast<uintptr_t>(shards) & 15u) return set_error(SS_ERR_INVALID_ARG, "the shard store must be 16-byte aligned");
    if (e->cfg.protocol == SS_PROTO_CROSSWORD && e->lut_bits == nullptr)
        return set_error(SS_ERR_INVALID_ARG, "ss_engine_set_policies must be called before proposing");
    if (e->cw_loc != nullptr && plane_stride >= kCwLocStrideLimit)
        return set_error(SS_ERR_INVALID_ARG, "a Crossword engine's plane_stride must be below 2^36");
    ss_ctx *ctx = e->ctx;
    SS_TRY(ctx_bind(ctx));
    if (e->rg_len == nullptr) SS_TRY(dalloc(ctx, &e->rg_len, e->G, false));
    if (e->rg_partials == nullptr) SS_TRY(dalloc(ctx, &e->rg_partials, scan_tiles(e->G), false));
    if (e->rg_need == nullptr) SS_TRY(dalloc(ctx, &e->rg_need, 1, false));
    const uint32_t grid = eng_grid(ctx, e->G);
    engine_ragged_prepare_kernel<<<grid, kEngThreads, 0, ctx->stream>>>(data_len, e->G, e->d, e->window_base, e->accepting, e->committed,
                                                                      e->rg_len, shard_off, ctx->dev_status);
    SS_TRY(launched(ctx));
    SS_TRY(launch_exclusive_scan_u64(ctx, shard_off, e->G, e->rg_partials, need != nullptr ? need : e->rg_need));
    engine_ragged_commit_kernel<<<grid, kEngThreads, 0, ctx->stream>>>(e->rg_len, shard_off, plane_stride, e->d, e->planes, e->n, e->G,
                                                                     e->window_base, e->bal_prepared, e->inst_bal, e->accepting,
                                                                     e->committed, e->policy_idx, policy, e->cw_loc, shards, slot_out,
                                                                     ctx->dev_status);
    SS_TRY(launched(ctx));
    // from_data + compute_parity + subset_copy's per-peer buffers for every proposing group, one launch: data shards into
    // planes 0..d-1, parity into planes d..T-1, each at the group's slot (rspaxos/request.rs:72-77,127-142,
    // crossword/request.rs:82-87,164-185)
    return ss_rs_encode_batch_dev(e->coder, arena, data_off, e->rg_len, e->G, shards + uint64_t(e->d) * plane_stride, plane_stride,
                                  shard_off, SS_RS_OUT_PADDED16 | SS_RS_EMIT_DATA);
}

int ss_engine_ingest(ss_engine *e, const uint32_t *rec_group, const uint8_t *rec_slot, const uint8_t *rec_peer,
                     const uint64_t *rec_ballot, uint64_t n_records) {
    if (e == nullptr) return set_error(SS_ERR_INVALID_ARG, "null engine");
    if (e->planes == nullptr) return set_error(SS_ERR_INVALID_ARG, "not a Paxos-family engine");
    if (n_records == 0) return SS_OK;
    if (!rec_group || !rec_slot || !rec_peer || !rec_ballot) return set_error(SS_ERR_INVALID_ARG, "null buffer");
    return launch_ack_ingest(e->ctx, rec_group, rec_slot, rec_peer, rec_ballot, n_records, e->bal_prepared, e->inst_bal,
                             e->accepting, e->windowed ? e->window_base : nullptr, e->n, e->G, e->planes);
}

int ss_engine_advance(ss_engine *e, const uint64_t *upto) {
    if (e == nullptr) return set_error(SS_ERR_INVALID_ARG, "null engine");
    if (e->planes == nullptr) return set_error(SS_ERR_INVALID_ARG, "not a Paxos-family engine");
    ss_ctx *ctx = e->ctx;
    SS_TRY(ctx_bind(ctx));
    e->windowed = true;
    engine_advance_kernel<<<eng_grid(ctx, e->G), kEngThreads, 0, ctx->stream>>>(upto, e->planes, e->n, e->G, e->window_base,
                                                                             e->accepting, e->committed, e->commit_bar);
    return launched(ctx);
}

int ss_engine_window_get(ss_engine *e, uint64_t **window_base) {
    if (e == nullptr || window_base == nullptr) return set_error(SS_ERR_INVALID_ARG, "null argument");
    if (e->planes == nullptr) return set_error(SS_ERR_INVALID_ARG, "not a Paxos-family engine");
    *window_base = e->window_base;
    e->windowed = true;                       // the host may install bases through the pointer
    return SS_OK;
}

int ss_engine_tick(ss_engine *e, uint64_t *newly) {
    if (e == nullptr) return set_error(SS_ERR_INVALID_ARG, "null engine");
    ss_ctx *ctx = e->ctx;
    SS_TRY(ctx_bind(ctx));
    if (e->planes == nullptr) {
        // Raft / CRaft: commit scan in place (new_commit -> last_commit), then last_snap for the groups that ingested
        SS_TRY(launch_raft_scan_ring(ctx, e->match, e->n_peers, e->G, e->last_commit, e->log_end, e->curr_term, e->terms, e->W,
                                     e->threshold, e->last_commit));
        const uint32_t grid = eng_grid(ctx, e->G);
        if (e->n_peers <= 4) engine_raft_snap_kernel<4><<<grid, kEngThreads, 0, ctx->stream>>>(e->match, e->n_peers, e->G, e->touched, e->last_snap);
        else if (e->n_peers <= 8) engine_raft_snap_kernel<8><<<grid, kEngThreads, 0, ctx->stream>>>(e->match, e->n_peers, e->G, e->touched, e->last_snap);
        else engine_raft_snap_kernel<16><<<grid, kEngThreads, 0, ctx->stream>>>(e->match, e->n_peers, e->G, e->touched, e->last_snap);
        return launched(ctx);
    }
    if (e->cfg.protocol == SS_PROTO_CROSSWORD) {
        if (e->lut_bits == nullptr) return set_error(SS_ERR_INVALID_ARG, "ss_engine_set_policies must be called first");
        auto *k = e->windowed ? engine_tick_crossword_kernel<true> : engine_tick_crossword_kernel<false>;
        k<<<eng_grid(ctx, e->G), kEngThreads, e->lut_words * 4, ctx->stream>>>(e->planes, e->n, e->G, e->policy_idx, e->lut_bits, e->lut_words,
                                                                             e->n_policies, e->window_base, e->accepting, e->committed,
                                                                             e->commit_bar, newly);
    } else if ((e->G & 1ull) == 0ull && (newly == nullptr || (reinterpret_cast<uintptr_t>(newly) & 15u) == 0u)) {
        const uint64_t G2 = e->G / 2;
        const uint32_t grid = static_cast<uint32_t>((G2 + kEngThreads - 1) / kEngThreads);
        const ulonglong2 *p2 = reinterpret_cast<const ulonglong2 *>(e->planes);
        const ulonglong2 *w2 = reinterpret_cast<const ulonglong2 *>(e->window_base);
        ulonglong2 *a2 = reinterpret_cast<ulonglong2 *>(e->accepting), *c2 = reinterpret_cast<ulonglong2 *>(e->committed);
        uint2 *b2 = reinterpret_cast<uint2 *>(e->commit_bar);
        ulonglong2 *n2 = reinterpret_cast<ulonglong2 *>(newly);
        const bool w = e->windowed;
        auto *k = e->n == 5 ? (w ? engine_tick_x2_kernel<5, true> : engine_tick_x2_kernel<5, false>)
                : e->n == 3 ? (w ? engine_tick_x2_kernel<3, true> : engine_tick_x2_kernel<3, false>)
                : e->n == 7 ? (w ? engine_tick_x2_kernel<7, true> : engine_tick_x2_kernel<7, false>)
                            : (w ? engine_tick_x2_kernel<0, true> : engine_tick_x2_kernel<0, false>);
        k<<<grid, kEngThreads, 0, ctx->stream>>>(p2, e->n, G2, e->threshold, w2, a2, c2, b2, n2);
    } else {
        auto *k = e->windowed ? engine_tick_kernel<true> : engine_tick_kernel<false>;
        k<<<eng_grid(ctx, e->G), kEngThreads, 0, ctx->stream>>>(e->planes, e->n, e->G, e->threshold, e->window_base, e->accepting,
                                                             e->committed, e->commit_bar, newly);
    }
    return launched(ctx);
}

int ss_engine_raft_append(ss_engine *e, const uint32_t *n_new) {
    if (e == nullptr || n_new == nullptr) return set_error(SS_ERR_INVALID_ARG, "null argument");
    if (e->match == nullptr) return set_error(SS_ERR_INVALID_ARG, "not a Raft engine");
    if (e->log_in_use) return set_error(SS_ERR_INVALID_ARG, "the CRaft log is in use: an entry without a codeword cannot be sent");
    ss_ctx *ctx = e->ctx;
    SS_TRY(ctx_bind(ctx));
    e->raft_appended = true;
    engine_raft_append_kernel<<<eng_grid(ctx, e->G), kEngThreads, 0, ctx->stream>>>(n_new, e->G, e->W, e->curr_term, e->last_commit,
                                                                                 e->log_end, e->terms, ctx->dev_status);
    return launched(ctx);
}

int ss_engine_raft_ingest(ss_engine *e, const uint32_t *rec_group, const uint8_t *rec_peer, const uint32_t *rec_end_slot,
                          uint64_t n_records) {
    if (e == nullptr) return set_error(SS_ERR_INVALID_ARG, "null engine");
    if (e->match == nullptr) return set_error(SS_ERR_INVALID_ARG, "not a Raft engine");
    if (n_records == 0) return SS_OK;
    if (!rec_group || !rec_peer || !rec_end_slot) return set_error(SS_ERR_INVALID_ARG, "null buffer");
    ss_ctx *ctx = e->ctx;
    SS_TRY(ctx_bind(ctx));
    engine_raft_ingest_kernel<<<eng_grid(ctx, n_records), kEngThreads, 0, ctx->stream>>>(rec_group, rec_peer, rec_end_slot, n_records,
                                                                                      e->n_peers, e->G, e->next_slot, e->match, e->touched);
    return launched(ctx);
}

}  // extern "C"
