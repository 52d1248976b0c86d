// acceptor_stepup.cu -- a new RSPaxos / Crossword leader's step-up on its own acceptor (ss_acceptor_step_up): what
// become_a_leader (rspaxos/leadership.rs:45-185, crossword/leadership.rs:47-190) does to the replica's instances, the
// WalEntry::PrepareBal records it logs and the Prepare it broadcasts, for a list of groups at once:
//
//   stepup_header_kernel     a thread per listed entry: sort keys, the entry's defaults (ignored, no records, no frame)
//   (CUB radix sort)         entry indices stably sorted by group: each group's entries in list order
//   stepup_walk_kernel       a thread per group segment: trigger_slot, endprep_slot and the positions to prepare from the
//                            group's state words, then make_greater_ballot once per entry in list order
//   (engine.cu's scan)       record and frame numbers: exclusive scans in list order
//   stepup_apply_kernel      a thread per group segment: the capacity cut, verdicts, state words, bal_max_seen; the last
//                            applied entry of the group defines the instances
//   stepup_write_kernel      a warp per applied entry: its PrepareBal cells, its Prepare frame and, for the defining
//                            entry, the per-slot arrays
//
// The leader's own vote then comes out of ss_acceptor_prepare_reply, unchanged: the marked instances have source = me.
// Stated differences from the reference: include/summerset_b200.h at ss_acceptor_step_up.
#include <cub/device/device_radix_sort.cuh>

#include "acceptor_state.hpp"
#include "ss_internal.hpp"
#include "window_ring.cuh"
#include "wire_common.cuh"

namespace ssb {

// one listed entry, in the FrameHdr scratch
struct StepHdr {
    uint64_t ballot, trigger, endprep;
    uint64_t marked;                // window positions the step-up makes Preparing
    uint64_t fresh;                 // the defining entry: ring positions that were null before the call
    uint32_t kind;                  // verdict so far
    uint32_t define;                // the last applied entry of its group
};
static_assert(sizeof(StepHdr) + sizeof(uint64_t) <= sizeof(FrameHdr) && alignof(StepHdr) <= alignof(FrameHdr),
              "StepHdr and a frame count per entry reuse the FrameHdr scratch");

struct StepArgs {
    const uint32_t *groups;         // nullptr: entry i is group i
    uint64_t n, G;
    uint32_t me, population, prepare_variant, wal_variant;
    // state
    const uint64_t *window_base, *exec_bar, *committed;
    uint64_t *bal_max_seen, *inst_bal, *accepting, *preparing, *voted_bal, *prep_trigger;
    uint32_t *held, *data_len, *voted_mask, *assignment, *assign_rows;
    uint8_t *source, *prep_span;
    // scratch
    StepHdr *hdr;
    uint32_t *key_in, *idx_in;
    const uint32_t *key, *idx;      // sorted
    uint64_t *rcnt, *fcnt;          // [n] records and frames per entry, then their exclusive scans
    uint64_t *totals;               // the caller's [4] (records, WAL bytes, frames, frame bytes), may be nullptr
    uint64_t rec_cap, frame_cap;    // min(rec_capacity, wal_capacity / 32), min(frame_capacity, out_capacity / 32)
    uint64_t frame_capacity;        // the frame records
    // outputs
    uint8_t *wal;
    uint32_t *rec_group;
    uint64_t *rec_slot;
    uint8_t *out;
    uint32_t *frame_group;
    uint8_t *frame_dst;
    uint64_t *frame_off;
    uint32_t *frame_len;
    uint32_t *verdict;
    uint64_t *ballot, *trigger_slot, *endprep_slot;
    uint32_t *status;
};

__device__ __forceinline__ uint32_t step_group(const StepArgs &A, uint64_t i) { return A.groups != nullptr ? A.groups[i] : static_cast<uint32_t>(i); }

// make_greater_ballot (rspaxos/mod.rs:446-454), in u64 as the reference computes it
__device__ __forceinline__ uint64_t greater_ballot(uint64_t bal, uint32_t me) { return (((bal >> 8) + 1u) << 8) | (me + 1u); }

// 1. a thread per listed entry
__global__ void __launch_bounds__(kAccThreads) stepup_header_kernel(const __grid_constant__ StepArgs A) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kAccThreads;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kAccThreads + threadIdx.x; i < A.n; i += stride) {
        const uint32_t g = step_group(A, i);
        StepHdr h{};
        h.kind = SS_FRAME_KIND_MALFORMED;
        A.hdr[i] = h;
        A.rcnt[i] = 0u;
        A.fcnt[i] = 0u;
        A.key_in[i] = g < A.G ? g : static_cast<uint32_t>(A.G);
        A.idx_in[i] = static_cast<uint32_t>(i);
    }
}

// 2. a thread per group segment.  In window terms: log_end = 1 + the last position that is Preparing, Accepting or
//    Committed; a position is done when it is Committed or below exec_bar; trigger = the first position of [0, log_end)
//    that is not done (log_end when there is none: the null instance the reference pushes), endprep = the last one
//    (trigger when there is none).  The positions of [max(exec_bar - base, 0), endprep] that are not Committed are marked.
//    A repeated step-up of the group finds the same trigger, endprep and marks, so only the ballot changes per entry.
__global__ void __launch_bounds__(kAccThreads) stepup_walk_kernel(const __grid_constant__ StepArgs A) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kAccThreads;
    for (uint64_t t = static_cast<uint64_t>(blockIdx.x) * kAccThreads + threadIdx.x; t < A.n; t += stride) {
        if (t != 0u && A.key[t] == A.key[t - 1]) continue;
        const uint32_t g = A.key[t];
        if (g >= A.G) continue;
        const uint64_t base = A.window_base[g], eb = A.exec_bar[g];
        const uint32_t r = static_cast<uint32_t>(base & 63u);
        const uint64_t com = ring_to_window(A.committed[g], r);
        const uint64_t live = ring_to_window(A.preparing[g] | A.accepting[g] | A.committed[g], r);
        const uint64_t end = live == 0u ? 0u : 64u - static_cast<uint64_t>(__clzll(static_cast<long long>(live)));
        const uint64_t lo = eb <= base ? 0u : eb - base >= 64u ? 64u : eb - base;
        const uint64_t below_end = end == 64u ? ~0ull : (1ull << end) - 1u;
        const uint64_t open = below_end & ~com & (lo == 64u ? 0ull : ~0ull << lo);
        const uint64_t trig = open != 0u ? static_cast<uint64_t>(__ffsll(static_cast<long long>(open))) - 1u : end;
        const uint64_t endp = open != 0u ? 63u - static_cast<uint64_t>(__clzll(static_cast<long long>(open))) : trig;
        const bool beyond = trig == 64u;
        uint64_t marked = 0u;
        if (!beyond && lo <= endp) marked = (endp == 63u ? ~0ull : (1ull << (endp + 1u)) - 1u) & ~((1ull << lo) - 1u) & ~com;
        const uint64_t recs = static_cast<uint64_t>(__popcll(marked));
        uint64_t bal = A.bal_max_seen[g];
        for (uint64_t k = t; k < A.n && A.key[k] == g; ++k) {
            const uint32_t i = A.idx[k];
            StepHdr h{};
            h.ballot = greater_ballot(bal, A.me);
            h.trigger = base + trig;
            h.endprep = base + endp;
            h.marked = marked;
            h.kind = beyond ? SS_ACCEPT_VERDICT_BEYOND_WINDOW : SS_ACCEPT_VERDICT_ACCEPTED;   // subject to capacity
            A.hdr[i] = h;
            if (!beyond) {
                bal = h.ballot;
                A.rcnt[i] = recs;
                A.fcnt[i] = 1u;
            }
        }
    }
}

// 3. a thread per group segment.  The record and frame ends are monotone in list order, so the entries cut by the
//    capacities are a suffix of the list and each group's applied entries a prefix of its entries; the last of them
//    defines the instances and bal_max_seen.
__global__ void __launch_bounds__(kAccThreads) stepup_apply_kernel(const __grid_constant__ StepArgs A) {
    if (A.totals != nullptr && blockIdx.x == 0u && threadIdx.x == 0u) {
        A.totals[1] = A.totals[0] * 32u;
        A.totals[3] = A.totals[2] * 32u;
    }
    bool full = false;
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kAccThreads;
    for (uint64_t t = static_cast<uint64_t>(blockIdx.x) * kAccThreads + threadIdx.x; t < A.n; t += stride) {
        if (t != 0u && A.key[t] == A.key[t - 1]) continue;
        const uint32_t g = A.key[t];
        uint64_t last = ~0ull;
        for (uint64_t k = t; k < A.n && A.key[k] == g; ++k) {
            const uint32_t i = A.idx[k];
            const StepHdr h = A.hdr[i];
            uint32_t kind = h.kind;
            if (kind == SS_ACCEPT_VERDICT_ACCEPTED) {
                if (A.rcnt[i] + __popcll(h.marked) > A.rec_cap || A.fcnt[i] + 1u > A.frame_cap) {
                    kind = SS_ACCEPT_VERDICT_WAL_FULL;
                    full = true;
                } else {
                    last = i;
                }
            }
            A.verdict[i] = kind;
            A.ballot[i] = h.ballot;
            A.trigger_slot[i] = h.trigger;
            A.endprep_slot[i] = h.endprep;
        }
        if (last == ~0ull) continue;
        const StepHdr h = A.hdr[last];
        const uint64_t m = window_to_ring(h.marked, static_cast<uint32_t>(A.window_base[g] & 63u));
        A.hdr[last].define = 1u;
        A.hdr[last].fresh = m & ~(A.preparing[g] | A.accepting[g] | A.committed[g]);
        A.preparing[g] |= m;                                                    // Status::Preparing, Accepting cleared
        A.accepting[g] &= ~m;
        A.bal_max_seen[g] = h.ballot;
    }
    if (full) atomicOr(A.status, SS_DEV_STATUS_FRAME_OVERFLOW);
}

// PeerMessage::Msg{Prepare{trigger_slot, ballot}} as the 32-byte cell at dst (16-byte aligned): 8-byte big-endian
// length, the bincode body (at most 22 bytes with variant < 2^16), zero to the end of the cell -> the frame's bytes
__device__ __forceinline__ uint32_t put_prepare_cell(uint8_t *dst, uint32_t variant, uint64_t trigger, uint64_t ballot) {
    uint8_t cell[32];
#pragma unroll
    for (int b = 0; b < 32; ++b) cell[b] = 0u;
    uint32_t m = 8u;
    m += wv_put(cell + m, 0u);                                                  // PeerMessage::Msg
    m += wv_put(cell + m, variant);
    m += wv_put(cell + m, trigger);
    m += wv_put(cell + m, ballot);
    put_be64(cell, m - 8u);
    uint4 lo, hi;
    memcpy(&lo, cell, 16);
    memcpy(&hi, cell + 16, 16);
    uint4 *d = reinterpret_cast<uint4 *>(dst);
    d[0] = lo;
    d[1] = hi;
    return m;
}

// 4. a warp per listed entry: an applied one writes its records (lane of each marked position), its frame (lane 0) and,
//    if it defines its group, the per-slot arrays; one cut by the capacities marks its frame slot as not written
__global__ void __launch_bounds__(kAccThreads) stepup_write_kernel(const __grid_constant__ StepArgs A) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = (static_cast<uint64_t>(blockIdx.x) * kAccThreads + threadIdx.x) >> 5;
    const uint64_t nwarps = (static_cast<uint64_t>(gridDim.x) * kAccThreads) >> 5;
    for (uint64_t i = warp; i < A.n; i += nwarps) {
        const uint32_t v = A.verdict[i];
        if (v != SS_ACCEPT_VERDICT_ACCEPTED && v != SS_ACCEPT_VERDICT_WAL_FULL) continue;
        const uint32_t g = step_group(A, i);
        const uint64_t f = A.fcnt[i];
        if (v == SS_ACCEPT_VERDICT_WAL_FULL) {
            if (lane == 0u && f < A.frame_capacity) {
                A.frame_group[f] = g;
                A.frame_dst[f] = 0xffu;
                A.frame_off[f] = ~0ull;
                A.frame_len[f] = 0u;
            }
            continue;
        }
        const StepHdr h = A.hdr[i];
        const uint64_t base = A.window_base[g], row = static_cast<uint64_t>(g) * 64u, first = A.rcnt[i];
        for (uint32_t w = lane; w < 64u; w += 32u) {
            if (!((h.marked >> w) & 1u)) continue;
            const uint64_t k = first + static_cast<uint64_t>(__popcll(h.marked & ((1ull << w) - 1u))), slot = base + w;
            put_prepare_bal_cell(A.wal + k * 32u, A.wal_variant, slot, h.ballot);
            A.rec_group[k] = g;
            A.rec_slot[k] = slot;
            if (!h.define) continue;
            const uint32_t p = static_cast<uint32_t>(slot & 63u);
            const uint64_t at = row + p;
            A.inst_bal[at] = h.ballot;
            A.source[at] = static_cast<uint8_t>(A.me);
            A.prep_trigger[at] = h.trigger;
            A.prep_span[at] = static_cast<uint8_t>(h.endprep - h.trigger);
            if ((h.fresh >> p) & 1u) {                                          // a fresh null_instance()
                A.held[at] = 0u;
                A.data_len[at] = 0u;
                A.voted_bal[at] = 0u;
                A.voted_mask[at] = 0u;
                if (A.assignment != nullptr) {
                    A.assignment[at] = 0u;
                    for (uint32_t q = 0; q < A.population; ++q) A.assign_rows[at * A.population + q] = 0u;
                }
            }
        }
        if (lane == 0u) {
            A.frame_len[f] = put_prepare_cell(A.out + f * 32u, A.prepare_variant, h.trigger, h.ballot);
            A.frame_group[f] = g;
            A.frame_dst[f] = 0xffu;
            A.frame_off[f] = f * 32u;
        }
    }
}

}  // namespace ssb

using namespace ssb;

extern "C" int ss_acceptor_step_up(ss_acceptor *a, const uint32_t *groups, uint64_t n_listed, uint32_t prepare_variant,
                                   uint32_t wal_variant, uint8_t *wal, uint64_t wal_capacity, uint32_t *rec_group,
                                   uint64_t *rec_slot, uint64_t rec_capacity, uint8_t *out, uint64_t out_capacity,
                                   uint32_t *frame_group, uint8_t *frame_dst, uint64_t *frame_off, uint32_t *frame_len,
                                   uint64_t frame_capacity, uint32_t *verdict, uint64_t *ballot, uint64_t *trigger_slot,
                                   uint64_t *endprep_slot, uint64_t *totals) {
    if (prepare_variant >= kVariantLimit || wal_variant >= kVariantLimit)
        return set_error(SS_ERR_INVALID_ARG, "prepare_variant and wal_variant must be below 2^16");
    if (a == nullptr) return set_error(SS_ERR_INVALID_ARG, "null acceptor");
    ss_ctx *ctx = a->ctx;
    SS_TRY(ctx_bind(ctx));
    const uint64_t n = groups != nullptr ? n_listed : a->G;
    if (n == 0) {
        if (totals != nullptr) SS_CUDA(cudaMemsetAsync(totals, 0, 32, ctx->stream));
        return SS_OK;
    }
    if (!wal || !rec_group || !rec_slot || !out || !frame_group || !frame_dst || !frame_off || !frame_len || !verdict || !ballot ||
        !trigger_slot || !endprep_slot)
        return set_error(SS_ERR_INVALID_ARG, "null buffer");
    if ((reinterpret_cast<uintptr_t>(wal) | reinterpret_cast<uintptr_t>(out)) & 15u)
        return set_error(SS_ERR_INVALID_ARG, "wal and out must be 16-byte aligned");
    if (n > 0x7fffffffull) return set_error(SS_ERR_INVALID_ARG, "at most 2^31 - 1 listed groups per call");
    SS_TRY(acc_scratch(a, n));
    StepArgs S{};
    S.groups = groups; S.n = n; S.G = a->G;
    S.me = a->cfg.me; S.population = a->cfg.population; S.prepare_variant = prepare_variant; S.wal_variant = wal_variant;
    S.window_base = a->window_base; S.exec_bar = a->exec_bar; S.committed = a->committed;
    S.bal_max_seen = a->bal_max_seen; S.inst_bal = a->inst_bal; S.accepting = a->accepting; S.preparing = a->preparing;
    S.voted_bal = a->voted_bal; S.prep_trigger = a->prep_trigger; S.held = a->held; S.data_len = a->data_len;
    S.voted_mask = a->voted_mask; S.assignment = a->assignment; S.assign_rows = a->assign_rows; S.source = a->source;
    S.prep_span = a->prep_span;
    // per-entry scratch: the FrameHdr cells hold a StepHdr each and, past them, the frame counts; fcnt the record counts
    S.hdr = reinterpret_cast<StepHdr *>(a->hdr);
    S.key_in = a->keys; S.idx_in = a->idx; S.key = a->keys + n; S.idx = a->idx + n;
    S.rcnt = a->fcnt;
    S.fcnt = reinterpret_cast<uint64_t *>(S.hdr + n);
    S.totals = totals;
    const uint64_t wal_cells = wal_capacity / 32u, out_cells = out_capacity / 32u;
    S.rec_cap = rec_capacity < wal_cells ? rec_capacity : wal_cells;
    S.frame_cap = frame_capacity < out_cells ? frame_capacity : out_cells;
    S.frame_capacity = frame_capacity;
    S.wal = wal; S.rec_group = rec_group; S.rec_slot = rec_slot; S.out = out; S.frame_group = frame_group; S.frame_dst = frame_dst;
    S.frame_off = frame_off; S.frame_len = frame_len; S.verdict = verdict; S.ballot = ballot; S.trigger_slot = trigger_slot;
    S.endprep_slot = endprep_slot; S.status = ctx->dev_status;
    const uint32_t grid_t = launch_grid(ctx, n, kAccThreads);
    stepup_header_kernel<<<grid_t, kAccThreads, 0, ctx->stream>>>(S);
    SS_TRY(launched(ctx));
    size_t bytes = a->sort_tmp_bytes;
    SS_CUDA(cub::DeviceRadixSort::SortPairs(a->sort_tmp, bytes, a->keys, a->keys + n, a->idx, a->idx + n, static_cast<int>(n), 0,
                                            key_bits(a->G), ctx->stream));
    SS_TRY(launched(ctx));
    stepup_walk_kernel<<<grid_t, kAccThreads, 0, ctx->stream>>>(S);
    SS_TRY(launched(ctx));
    SS_TRY(launch_exclusive_scan_u64(ctx, S.rcnt, n, a->partials, totals != nullptr ? totals : a->totals));
    SS_TRY(launch_exclusive_scan_u64(ctx, S.fcnt, n, a->partials, totals != nullptr ? totals + 2 : a->totals + 1));
    stepup_apply_kernel<<<grid_t, kAccThreads, 0, ctx->stream>>>(S);
    SS_TRY(launched(ctx));
    stepup_write_kernel<<<launch_grid(ctx, n, kAccThreads / 32), kAccThreads, 0, ctx->stream>>>(S);
    return launched(ctx);
}
