// acceptor_recover.cu -- WAL recovery on the RSPaxos / Crossword acceptor (ss_acceptor_recover): recover_apply_entry
// and recover_from_wal (rspaxos/recovery.rs:10-181, crossword/recovery.rs:10-186) for the PrepareBal, AcceptData and
// CommitSlot records the acceptor wrote, for a batch of records of many groups at once:
//
//   recover_header_kernel    a thread per record: decode_frame reached from the WalEntry tag (acceptor_state.hpp),
//                            window filters, sort keys
//   (CUB radix sort)         record indices stably sorted by group: each group's records in WAL order
//   recover_walk_kernel      a thread per group segment: the verdicts in WAL order (the log ends at the first malformed
//                            record, the replay stops at the first record beyond the window), then backwards: the last
//                            applied AcceptData of each slot defines the instance; the group's store bytes
//   (engine.cu's scan)       group regions: exclusive scan over the groups
//   recover_apply_kernel     a thread per group segment: the capacity cut, then every applied record in WAL order over
//                            the group's state words held in registers; the defined instances' regions in window order
//   recover_copy_kernel      a warp per defining AcceptData: its shards into the padded store slots (the accept copy),
//                            Crossword: its assignment rows
//
// Stated differences from the reference: include/summerset_b200.h at ss_acceptor_recover.
#include <cub/device/device_radix_sort.cuh>

#include "acceptor_state.hpp"
#include "codeword_wire.cuh"
#include "ss_internal.hpp"
#include "window_ring.cuh"
#include "wire_common.cuh"

namespace ssb {

constexpr uint32_t kDefining = 0xfffffffbu;         // an applied AcceptData, the last of its (group, slot)

struct RcvArgs {
    const uint8_t *buf;
    uint64_t buf_len;
    const uint64_t *frame_off;      // rec_off
    const uint32_t *frame_group;    // rec_group
    uint64_t n, G;
    uint32_t d, T, population, me, wal_variant, prepare_variant, commit_variant, crossword;
    // state
    const uint64_t *window_base;
    uint64_t *bal_max_seen, *inst_bal, *accepting, *committed, *preparing, *shard_addr, *voted_bal, *prep_trigger;
    uint32_t *held, *data_len, *assignment, *assign_rows, *voted_mask;
    uint8_t *source, *prep_span;
    // scratch
    FrameHdr *hdr;
    uint32_t *key_in, *idx_in;
    const uint32_t *key, *idx;      // sorted
    uint64_t *grp_off;              // [G] store bytes per group, then their exclusive scan
    const uint64_t *total;          // the scan's total
    // outputs
    uint8_t *store;
    uint64_t store_cap;
    uint32_t *verdict;
    uint32_t *status;
};

// 1. a thread per record
__global__ void __launch_bounds__(kAccThreads) recover_header_kernel(const __grid_constant__ RcvArgs A) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kAccThreads;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kAccThreads + threadIdx.x; i < A.n; i += stride) {
        A.hdr[i] = decode_frame<true>(A, i);
        const uint32_t grp = A.frame_group[i];
        A.key_in[i] = grp < A.G ? grp : static_cast<uint32_t>(A.G);
        A.idx_in[i] = static_cast<uint32_t>(i);
    }
}

__device__ __forceinline__ uint64_t rcv_segment_end(const RcvArgs &A, uint64_t t) {
    uint64_t e = t + 1u;
    while (e < A.n && A.key[e] == A.key[t]) ++e;
    return e;
}

// 2. a thread per group segment, records in WAL order: the log ends at a malformed record (the reference's read loop
//    stops there and truncates), the replay at the first record beyond the window; the records before either are
//    applied or stale.  Then backwards over those: the last AcceptData of each slot defines the instance and takes
//    store room.
__global__ void __launch_bounds__(kAccThreads) recover_walk_kernel(const __grid_constant__ RcvArgs A) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kAccThreads;
    for (uint64_t t = static_cast<uint64_t>(blockIdx.x) * kAccThreads + threadIdx.x; t < A.n; t += stride) {
        if (t != 0u && A.key[t] == A.key[t - 1]) continue;
        const uint32_t g = A.key[t];
        const uint64_t e = rcv_segment_end(A, t);
        if (g >= A.G) {                                                        // no such group: each record alone
            for (uint64_t k = t; k < e; ++k) A.verdict[A.idx[k]] = SS_FRAME_KIND_MALFORMED;
            continue;
        }
        uint64_t stop = e;
        bool cut = false, ended = false;
        for (uint64_t k = t; k < e; ++k) {
            const uint32_t i = A.idx[k];
            uint32_t v = A.hdr[i].kind;
            if (v != SS_FRAME_KIND_MALFORMED && v != SS_ACCEPT_VERDICT_STALE_SLOT && v != SS_ACCEPT_VERDICT_BEYOND_WINDOW)
                v = SS_ACCEPT_VERDICT_ACCEPTED;
            if (ended) {
                v = SS_RECOVER_VERDICT_AFTER_END;
            } else if (v == SS_FRAME_KIND_MALFORMED) {
                ended = true;
            } else if (cut || v == SS_ACCEPT_VERDICT_BEYOND_WINDOW) {
                v = SS_ACCEPT_VERDICT_BEYOND_WINDOW;
                cut = true;
            }
            if (stop == e && v != SS_ACCEPT_VERDICT_ACCEPTED && v != SS_ACCEPT_VERDICT_STALE_SLOT) stop = k;
            A.verdict[i] = v;
        }
        uint64_t seen = 0u, bytes = 0u;
        for (uint64_t k = stop; k-- > t;) {
            const uint32_t i = A.idx[k];
            const FrameHdr h = A.hdr[i];
            if (h.kind != kPending) continue;                                  // PrepareBal, CommitSlot, stale
            const uint64_t bit = 1ull << (h.slot & 63u);
            if (seen & bit) continue;
            seen |= bit;
            A.hdr[i].kind = kDefining;
            bytes += store_bytes(h);
        }
        A.grp_off[g] = bytes;
    }
}

// 3. a thread per group segment: a group whose region ends past the capacity applies nothing; the others replay their
//    applied records in WAL order as recover_apply_entry does, then place the defined instances' shards in window order
//    from the group's offset
__global__ void __launch_bounds__(kAccThreads) recover_apply_kernel(const __grid_constant__ RcvArgs A) {
    bool full = false;
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kAccThreads;
    for (uint64_t t = static_cast<uint64_t>(blockIdx.x) * kAccThreads + threadIdx.x; t < A.n; t += stride) {
        if (t != 0u && A.key[t] == A.key[t - 1]) continue;
        const uint32_t g = A.key[t];
        if (g >= A.G) continue;
        const uint64_t e = rcv_segment_end(A, t);
        const uint64_t off = A.grp_off[g], end = g + 1u < A.G ? A.grp_off[g + 1u] : *A.total;
        if (end > A.store_cap) {                                               // the ends are monotone: a suffix of groups
            for (uint64_t k = t; k < e; ++k) {
                const uint32_t i = A.idx[k];
                if (A.verdict[i] != SS_ACCEPT_VERDICT_ACCEPTED) continue;
                A.verdict[i] = SS_ACCEPT_VERDICT_STORE_FULL;
                full = true;
            }
            continue;
        }
        const uint64_t base = A.window_base[g], row = static_cast<uint64_t>(g) * 64u;
        uint64_t prep = A.preparing[g], acc = A.accepting[g], com = A.committed[g], mx = A.bal_max_seen[g], def = 0u;
        for (uint64_t k = t; k < e; ++k) {
            const uint32_t i = A.idx[k];
            if (A.verdict[i] != SS_ACCEPT_VERDICT_ACCEPTED) continue;
            const FrameHdr h = A.hdr[i];
            const uint64_t bit = 1ull << (h.slot & 63u), at = row + (h.slot & 63u);
            if (!((prep | acc | com) & bit)) {                                 // a fresh null_instance(): no bal, shards, vote
                A.inst_bal[at] = 0u;
                A.held[at] = 0u;
                A.data_len[at] = 0u;
                A.voted_bal[at] = 0u;
                A.voted_mask[at] = 0u;
                if (A.assignment != nullptr) {
                    A.assignment[at] = 0u;
                    for (uint32_t r = 0; r < A.population; ++r) A.assign_rows[at * A.population + r] = 0u;
                }
            }
            A.source[at] = 0xffu;                                              // replica_bk: None
            A.prep_trigger[at] = 0u;
            A.prep_span[at] = 0u;
            if (h.kind == kPendingCommitSlot) {                                // Status::Committed
                com |= bit;
                acc &= ~bit;
                prep &= ~bit;
                continue;
            }
            A.inst_bal[at] = h.ballot;
            mx = h.ballot > mx ? h.ballot : mx;
            if (h.kind == kPendingPrepareBal) {                                // Status::Preparing
                prep |= bit;
                acc &= ~bit;
                com &= ~bit;
                continue;
            }
            acc |= bit;                                                        // AcceptData: Status::Accepting
            prep &= ~bit;
            com &= ~bit;
            if (h.kind == kDefining) {                                         // no later AcceptData of this slot:
                def |= bit;                                                    // the final reqs_cw, voted, assignment
                A.held[at] = h.held;
                A.data_len[at] = h.dlen;
                A.voted_bal[at] = h.ballot;
                A.voted_mask[at] = h.held;
                if (A.assignment != nullptr) A.assignment[at] = h.asg;   // the rows: recover_copy_kernel
            }
        }
        A.preparing[g] = prep;
        A.accepting[g] = acc;
        A.committed[g] = com;
        A.bal_max_seen[g] = mx;
        uint64_t o = off;
        for (uint64_t rest = ring_to_window(def, static_cast<uint32_t>(base & 63u)); rest != 0u; rest &= rest - 1u) {
            const uint64_t w = static_cast<uint64_t>(__ffsll(static_cast<long long>(rest))) - 1u;
            const uint64_t at = row + ((base + w) & 63u);
            A.shard_addr[at] = reinterpret_cast<uint64_t>(A.store + o);
            // L as decode_frame computed it for recover_walk_kernel's sizes: in 64 bits, data_len + d - 1 may pass 2^32
            const uint64_t L = (static_cast<uint64_t>(A.data_len[at]) + A.d - 1u) / A.d;
            o += static_cast<uint64_t>(__popc(A.held[at])) * SS_CW_SLOT_PITCH(L);
        }
    }
    if (full) atomicOr(A.status, SS_DEV_STATUS_STORE_FULL);
}

// 4. a warp per defining AcceptData of a placed group: its held shards into the instance's store slots; Crossword: its
//    whole assignment into assign_rows
__global__ void __launch_bounds__(kAccThreads) recover_copy_kernel(const __grid_constant__ RcvArgs A) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = (static_cast<uint64_t>(blockIdx.x) * kAccThreads + threadIdx.x) >> 5;
    const uint64_t nwarps = (static_cast<uint64_t>(gridDim.x) * kAccThreads) >> 5;
    for (uint64_t i = warp; i < A.n; i += nwarps) {
        if (A.verdict[i] != SS_ACCEPT_VERDICT_ACCEPTED || A.hdr[i].kind != kDefining) continue;
        const FrameHdr h = A.hdr[i];
        const uint64_t at = static_cast<uint64_t>(A.frame_group[i]) * 64u + (h.slot & 63u);
        const uint8_t *fr = A.buf + A.frame_off[i];
        warp_fill_shards(reinterpret_cast<uint8_t *>(A.shard_addr[at]), fr + h.tags_at, A.T, h.held, h.held, h.L, lane);
        if (A.assignment != nullptr && lane == 0u)
            read_assign_rows(fr + h.asg_at, h.end - h.asg_at, A.population, A.assign_rows, at * A.population);
    }
}

}  // namespace ssb

using namespace ssb;

extern "C" int ss_acceptor_recover(ss_acceptor *a, const uint8_t *buf, uint64_t buf_len, const uint64_t *rec_off,
                                   const uint32_t *rec_group, uint64_t n, uint32_t prepare_variant, uint32_t commit_variant,
                                   uint8_t *store, uint64_t store_capacity, uint32_t *verdict, uint64_t *total) {
    if (a == nullptr) return set_error(SS_ERR_INVALID_ARG, "null acceptor");
    const uint32_t wal_variant = a->cfg.wal_variant;
    if (prepare_variant == commit_variant || prepare_variant == wal_variant || commit_variant == wal_variant)
        return set_error(SS_ERR_INVALID_ARG, "the PrepareBal, AcceptData and CommitSlot variants must differ (%u, %u, %u)",
                         prepare_variant, wal_variant, commit_variant);
    ss_ctx *ctx = a->ctx;
    SS_TRY(ctx_bind(ctx));
    if (n == 0) {
        if (total != nullptr) SS_CUDA(cudaMemsetAsync(total, 0, 8, ctx->stream));
        return SS_OK;
    }
    if (!buf || !rec_off || !rec_group || !store || !verdict) return set_error(SS_ERR_INVALID_ARG, "null buffer");
    if (reinterpret_cast<uintptr_t>(store) & 15u) return set_error(SS_ERR_INVALID_ARG, "store must be 16-byte aligned");
    if (n > 0x7fffffffull) return set_error(SS_ERR_INVALID_ARG, "at most 2^31 - 1 records per call");
    SS_TRY(acc_scratch(a, n));
    uint64_t *tot = total != nullptr ? total : a->totals;
    RcvArgs R{};
    R.buf = buf; R.buf_len = buf_len; R.frame_off = rec_off; R.frame_group = rec_group; R.n = n; R.G = a->G;
    R.d = a->cfg.data_shards; R.T = a->cfg.total_shards; R.population = a->cfg.population; R.me = a->cfg.me;
    R.wal_variant = wal_variant; R.prepare_variant = prepare_variant; R.commit_variant = commit_variant;
    R.crossword = a->cfg.protocol == SS_PROTO_CROSSWORD ? 1u : 0u;
    R.window_base = a->window_base; R.bal_max_seen = a->bal_max_seen; R.inst_bal = a->inst_bal; R.accepting = a->accepting;
    R.committed = a->committed; R.preparing = a->preparing; R.shard_addr = a->shard_addr; R.voted_bal = a->voted_bal;
    R.prep_trigger = a->prep_trigger; R.held = a->held; R.data_len = a->data_len; R.assignment = a->assignment;
    R.assign_rows = a->assign_rows; R.voted_mask = a->voted_mask; R.source = a->source; R.prep_span = a->prep_span;
    R.hdr = a->hdr; R.key_in = a->keys; R.idx_in = a->idx; R.key = a->keys + n; R.idx = a->idx + n;
    R.grp_off = a->ex_bytes;        // execute's per-group scratch: both calls are ordered on the context's stream
    R.total = tot;
    R.store = store; R.store_cap = store_capacity; R.verdict = verdict; R.status = ctx->dev_status;
    const uint32_t grid_t = launch_grid(ctx, n, kAccThreads);
    recover_header_kernel<<<grid_t, kAccThreads, 0, ctx->stream>>>(R);
    SS_TRY(launched(ctx));
    size_t bytes = a->sort_tmp_bytes;
    SS_CUDA(cub::DeviceRadixSort::SortPairs(a->sort_tmp, bytes, a->keys, a->keys + n, a->idx, a->idx + n, static_cast<int>(n), 0,
                                            key_bits(a->G), ctx->stream));
    SS_TRY(launched(ctx));
    SS_CUDA(cudaMemsetAsync(a->ex_bytes, 0, a->G * 8, ctx->stream));
    recover_walk_kernel<<<grid_t, kAccThreads, 0, ctx->stream>>>(R);
    SS_TRY(launched(ctx));
    SS_TRY(launch_exclusive_scan_u64(ctx, a->ex_bytes, a->G, a->ex_partials, tot));
    recover_apply_kernel<<<grid_t, kAccThreads, 0, ctx->stream>>>(R);
    SS_TRY(launched(ctx));
    recover_copy_kernel<<<launch_grid(ctx, n, kAccThreads / 32), kAccThreads, 0, ctx->stream>>>(R);
    return launched(ctx);
}
