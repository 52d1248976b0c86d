// engine_fallback.cu -- Crossword's soft fallback on the leader (ss_engine_fallback_redo): fallback_redo_accepts
// (crossword/leadership.rs:389-550) in window terms for a list of groups.  Every Accepting instance whose assignment is
// not responsive for the group's live peers is re-assigned the host's policy, loses its acks and has its full codeword
// copied out of the location the engine recorded when it entered Accepting, for ss_frame_accept_pack_ragged_dev.
//
//   fb_mark_kernel    a thread per listed entry: the first entry of each group (atomicMin)
//   fb_count_kernel   a warp per listed entry, lane l keeping window positions l and l + 32: the positions it redoes and
//                     the decided records and store bytes they add
//   (engine.cu's scan) their exclusive scans in list order
//   fb_apply_kernel   a warp per listed entry: the per-entry capacity cut, the engine's words and the decided list
//   fb_copy_kernel    a warp per decided record: the codeword's T shards into its store slot; the store cursor
//
// Stated differences from the reference: include/summerset_b200.h at ss_engine_fallback_redo.
#include "device_common.cuh"
#include "engine_state.hpp"
#include "ss_internal.hpp"
#include "window_ring.cuh"

namespace ssb {

constexpr int kFbThreads = 256;

struct FbArgs {
    const uint32_t *groups;
    uint64_t n, G;
    uint32_t n_pop, pop_mask, d, T, majority, f, n_policies;
    int balanced;
    const uint32_t *peer_alive;     // [G] or nullptr: every replica alive
    const uint8_t *policy;          // [G]
    const uint32_t *policies;       // [n_policies][n_pop]
    const ss_cw_loc *cw_loc;
    const uint64_t *window_base, *accepting, *committed, *bal_prepared;
    uint64_t *planes, *inst_bal;
    uint8_t *policy_idx;
    uint32_t *first;                // [G]
    uint64_t *mask;                 // [n] redone ring positions
    uint64_t *c_rec, *c_store;      // [n] records and store bytes per entry, then their exclusive scans
    const uint64_t *tot;            // [2] the scans' totals
    uint64_t *words;                // [2] applied store bytes and records (atomicMax)
    const uint64_t *store_used;
    uint64_t *store_used_out;
    uint64_t store_cap, dec_cap;
    uint8_t *shards;
    uint64_t *dec_slot, *dec_ballot, *dec_off;
    uint32_t *dec_len, *dec_group;
    uint8_t *dec_policy;
    uint32_t *verdict, *status;
};

__device__ __forceinline__ uint64_t below(uint32_t w) { return w >= 64u ? ~0ull : (1ull << w) - 1u; }

__device__ __forceinline__ uint64_t cw_pitch(uint32_t data_len, uint32_t d) {
    return SS_CW_SLOT_PITCH((static_cast<uint64_t>(data_len) + d - 1u) / d);
}

// min_shards_per_replica (adaptive.rs:98-106) in the reference's u8 arithmetic, where (majority + f + 1 - alive) would
// underflow: then 0, so every balanced instance is responsive
__device__ __forceinline__ uint32_t min_spr(uint32_t majority, uint32_t f, uint32_t alive, uint32_t d) {
    const uint32_t top = majority + f + 1u;
    return alive > top ? 0u : ((top - alive) * (d / majority)) & 0xffu;
}

// a policy index whose assignment is responsive for the group's live peers: the engine is balanced and replica 0 of
// the assignment holds at least min_spr shards; an index >= n_policies never is
__device__ __forceinline__ bool responsive(const FbArgs &A, uint32_t k, uint32_t spr) {
    return A.balanced && k < A.n_policies && static_cast<uint32_t>(__popc(A.policies[static_cast<uint64_t>(k) * A.n_pop])) >= spr;
}

// 1. a thread per listed entry
__global__ void __launch_bounds__(kFbThreads) fb_mark_kernel(const __grid_constant__ FbArgs A) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kFbThreads;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kFbThreads + threadIdx.x; i < A.n; i += stride) {
        const uint32_t g = A.groups[i];
        if (g < A.G) atomicMin(A.first + g, static_cast<uint32_t>(i));
    }
}

// 2. a warp per listed entry.  Every entry reads the state before the call.  The first entry of a group redoes R0, the
//    Accepting, uncommitted positions whose policy is not responsive (and that have a recorded codeword); they then hold
//    policy[g], so a later entry of the group redoes R0 again when policy[g] is not responsive either, and nothing when it
//    is -- what a second reference call would do.  A cut entry cuts every later one, so a later entry only applies after
//    the first did.
__global__ void __launch_bounds__(kFbThreads) fb_count_kernel(const __grid_constant__ FbArgs A) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = (static_cast<uint64_t>(blockIdx.x) * kFbThreads + threadIdx.x) >> 5;
    const uint64_t nwarps = (static_cast<uint64_t>(gridDim.x) * kFbThreads) >> 5;
    for (uint64_t i = warp; i < A.n; i += nwarps) {
        const uint32_t g = A.groups[i];
        uint64_t redo = 0, bytes = 0;
        if (g < A.G) {
            const uint64_t row = static_cast<uint64_t>(g) * 64u;
            const uint32_t r = static_cast<uint32_t>(A.window_base[g] & 63u);
            const uint64_t open = A.accepting[g] & ~A.committed[g];
            const uint32_t alive = static_cast<uint32_t>(__popc((A.peer_alive != nullptr ? A.peer_alive[g] : ~0u) & A.pop_mask));
            const uint32_t spr = min_spr(A.majority, A.f, alive, A.d);
            const bool later = A.first[g] != static_cast<uint32_t>(i);
            const bool again = !later || !responsive(A, A.policy[g], spr);
            for (uint32_t h = 0; h < 2u; ++h) {
                const uint32_t p = (lane + 32u * h + r) & 63u;
                bool take = false;
                if (again && ((open >> p) & 1u)) {
                    const ss_cw_loc loc = A.cw_loc[row + p];
                    take = loc.addr != 0u && !responsive(A, A.policy_idx[row + p], spr);
                    if (take) bytes += cw_pitch(loc.data_len, A.d);
                }
                redo |= static_cast<uint64_t>(__ballot_sync(0xffffffffu, take)) << (32u * h);
            }
            for (int o = 16; o > 0; o >>= 1) bytes += __shfl_xor_sync(0xffffffffu, bytes, o);
            redo = window_to_ring(redo, r);
        }
        if (lane == 0u) {
            A.mask[i] = redo;
            A.c_rec[i] = static_cast<uint64_t>(__popcll(redo));
            A.c_store[i] = bytes;
        }
    }
}

// 3. a warp per listed entry: the cut, then inst_bal = bal_prepared, the acks cleared, policy_idx = policy[g] and one
//    decided record per redone position in slot order.  Two entries of one group write the same values to the engine's
//    words, so their warps may run in either order.
__global__ void __launch_bounds__(kFbThreads) fb_apply_kernel(const __grid_constant__ FbArgs A) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = (static_cast<uint64_t>(blockIdx.x) * kFbThreads + threadIdx.x) >> 5;
    const uint64_t nwarps = (static_cast<uint64_t>(gridDim.x) * kFbThreads) >> 5;
    bool store_full = false, list_full = false;
    for (uint64_t i = warp; i < A.n; i += nwarps) {
        const uint32_t g = A.groups[i];
        if (g >= A.G) {
            if (lane == 0u) A.verdict[i] = SS_FRAME_KIND_MALFORMED;
            continue;
        }
        const uint64_t r_end = i + 1u < A.n ? A.c_rec[i + 1u] : A.tot[0];
        const uint64_t s_end = i + 1u < A.n ? A.c_store[i + 1u] : A.tot[1];
        const uint64_t used = (*A.store_used + 31u) & ~31ull;                // slots start 32-byte aligned
        const bool sf = used > A.store_cap || s_end > A.store_cap - used;
        const bool lf = r_end > A.dec_cap;
        if (lane == 0u) A.first[g] = ~0u;                               // ready for the next call
        if (sf || lf) {                                                 // the per-entry cut: nothing of it applies
            store_full |= sf;
            list_full |= lf && !sf;
            if (lane == 0u) A.verdict[i] = sf ? SS_ACCEPT_VERDICT_STORE_FULL : SS_ACCEPT_VERDICT_WAL_FULL;
            continue;
        }
        if (lane == 0u) {
            A.verdict[i] = SS_ACCEPT_VERDICT_ACCEPTED;
            atomicMax(reinterpret_cast<unsigned long long *>(A.words), static_cast<unsigned long long>(s_end));
            atomicMax(reinterpret_cast<unsigned long long *>(A.words + 1), static_cast<unsigned long long>(r_end));
        }
        const uint64_t redo = A.mask[i];
        if (redo == 0u) continue;
        const uint64_t row = static_cast<uint64_t>(g) * 64u, base = A.window_base[g], bp = A.bal_prepared[g];
        const uint32_t r = static_cast<uint32_t>(base & 63u);
        const uint8_t k = A.policy[g];
        const uint64_t redo_w = ring_to_window(redo, r);
        if (lane < A.n_pop) A.planes[static_cast<uint64_t>(lane) * A.G + g] &= ~redo;   // accept_acks.clear()
        // slot pitches in window order: a warp scan over positions 0..31, then 32..63 after them
        uint64_t at = used + A.c_store[i];
        const uint64_t rec0 = A.c_rec[i];
        for (uint32_t h = 0; h < 2u; ++h) {
            const uint32_t w = lane + 32u * h, p = (w + r) & 63u;
            const bool mine = (redo_w >> w) & 1u;
            const uint32_t len = mine ? A.cw_loc[row + p].data_len : 0u;
            const uint64_t pitch = mine ? cw_pitch(len, A.d) : 0u;
            uint64_t incl = pitch;
            for (int o = 1; o < 32; o <<= 1) {
                const uint64_t y = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= static_cast<uint32_t>(o)) incl += y;
            }
            if (mine) {
                const uint64_t kd = rec0 + static_cast<uint64_t>(__popcll(redo_w & below(w)));
                A.inst_bal[row + p] = bp;                               // inst.bal = bal_prepared
                A.policy_idx[row + p] = k;
                A.dec_slot[kd] = base + w;
                A.dec_ballot[kd] = bp;
                A.dec_off[kd] = at + incl - pitch;
                A.dec_len[kd] = len;
                A.dec_group[kd] = g;
                if (A.dec_policy != nullptr) A.dec_policy[kd] = k;
            }
            at += __shfl_sync(0xffffffffu, incl, 31);
        }
    }
    if (lane == 0u) {
        if (store_full) atomicOr(A.status, SS_DEV_STATUS_STORE_FULL);
        if (list_full) atomicOr(A.status, SS_DEV_STATUS_FRAME_OVERFLOW);
    }
}

// 4. a warp per decided record: shard j from its recorded location into plane j at the record's slot, 128-bit copies,
//    bytes shard_len..round_up(shard_len, 16) zero; then the store cursor
__global__ void __launch_bounds__(kFbThreads) fb_copy_kernel(const __grid_constant__ FbArgs A, uint64_t plane_stride) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = (static_cast<uint64_t>(blockIdx.x) * kFbThreads + threadIdx.x) >> 5;
    const uint64_t nwarps = (static_cast<uint64_t>(gridDim.x) * kFbThreads) >> 5;
    const uint64_t n_rec = A.words[1];
    for (uint64_t k = warp; k < n_rec; k += nwarps) {
        const ss_cw_loc loc = A.cw_loc[static_cast<uint64_t>(A.dec_group[k]) * 64u + (A.dec_slot[k] & 63u)];
        const uint64_t L = (static_cast<uint64_t>(loc.data_len) + A.d - 1u) / A.d, nvec = (L + 15u) >> 4;
        const uint64_t src_stride = static_cast<uint64_t>(loc.stride16) << 4, off = A.dec_off[k];
        for (uint32_t j = 0; j < A.T; ++j) {
            const uint4 *src = reinterpret_cast<const uint4 *>(loc.addr + j * src_stride);
            uint4 *dst = reinterpret_cast<uint4 *>(A.shards + j * plane_stride + off);
            for (uint64_t v = lane; v < nvec; v += 32u) {
                uint4 x = src[v];
                const uint64_t left = L - v * 16u;
                if (left < 16u) {                                       // the padding of the last vector
                    uint32_t w[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const int keep = static_cast<int>(left) - 4 * q;
                        w[q] = keep >= 4 ? w[q] : keep <= 0 ? 0u : w[q] & ((1u << (8 * keep)) - 1u);
                    }
                    x = make_uint4(w[0], w[1], w[2], w[3]);
                }
                dst[v] = x;
            }
        }
    }
    if (blockIdx.x == 0 && threadIdx.x == 0 && A.words[0] != 0u) *A.store_used_out = ((*A.store_used_out + 31u) & ~31ull) + A.words[0];
}

void fallback_free(ss_engine *e) {
    void *bufs[] = {e->fb_first, e->fb_mask, e->fb_cnt, e->fb_partials, e->fb_words};
    for (void *b : bufs)
        if (b) cudaFree(b);
}

// fb_first on first use (every entry UINT32_MAX), per-entry scratch grow-only
static int fallback_scratch(ss_engine *e, uint64_t n) {
    ss_ctx *ctx = e->ctx;
    if (e->fb_first == nullptr) {
        SS_TRY(dalloc(ctx, &e->fb_first, e->G, false));
        SS_CUDA(cudaMemsetAsync(e->fb_first, 0xff, e->G * 4, ctx->stream));
        SS_TRY(dalloc(ctx, &e->fb_words, 4));
    }
    if (n > e->fb_cap) {
        SS_CUDA(cudaStreamSynchronize(ctx->stream));
        void *old[] = {e->fb_mask, e->fb_cnt, e->fb_partials};
        for (void *b : old)
            if (b) cudaFree(b);
        e->fb_mask = nullptr; e->fb_cnt = nullptr; e->fb_partials = nullptr; e->fb_cap = 0;
        SS_TRY(dalloc(ctx, &e->fb_mask, n, false)); SS_TRY(dalloc(ctx, &e->fb_cnt, 2 * n, false));
        SS_TRY(dalloc(ctx, &e->fb_partials, scan_tiles(n), false));
        e->fb_cap = n;
    }
    return SS_OK;
}

}  // namespace ssb

using namespace ssb;

extern "C" int ss_engine_fallback_redo(ss_engine *e, const uint32_t *groups, uint64_t n_listed, const uint32_t *peer_alive,
                                       const uint8_t *policy, uint8_t *shards, uint64_t plane_stride, uint64_t *store_used,
                                       uint64_t *dec_slot, uint64_t *dec_ballot, uint64_t *dec_shard_off, uint32_t *dec_data_len,
                                       uint8_t *dec_policy, uint32_t *dec_group, uint64_t dec_capacity, uint32_t *verdict,
                                       uint64_t *totals) {
    if (e == nullptr) return set_error(SS_ERR_INVALID_ARG, "null engine");
    if (e->cfg.protocol != SS_PROTO_CROSSWORD) return set_error(SS_ERR_INVALID_ARG, "the soft fallback serves Crossword engines only");
    if (e->lut_bits == nullptr) return set_error(SS_ERR_INVALID_ARG, "ss_engine_set_policies must be called first");
    if (!policy || !shards || !store_used || !dec_slot || !dec_ballot || !dec_shard_off || !dec_data_len || !dec_group ||
        (n_listed != 0 && (!groups || !verdict)))
        return set_error(SS_ERR_INVALID_ARG, "null buffer");
    if ((plane_stride & 31u) || plane_stride == 0 || plane_stride >= kCwLocStrideLimit)
        return set_error(SS_ERR_INVALID_ARG, "plane_stride must be a non-zero multiple of 32 below 2^36");
    if (reinterpret_cast<uintptr_t>(shards) & 15u) return set_error(SS_ERR_INVALID_ARG, "the shard store must be 16-byte aligned");
    if (n_listed > 0x7fffffffull) return set_error(SS_ERR_INVALID_ARG, "at most 2^31 - 1 listed groups per call");
    ss_ctx *ctx = e->ctx;
    SS_TRY(ctx_bind(ctx));
    SS_TRY(fallback_scratch(e, n_listed));
    FbArgs A{};
    A.groups = groups; A.n = n_listed; A.G = e->G;
    A.n_pop = e->n; A.pop_mask = e->n >= 32u ? ~0u : (1u << e->n) - 1u; A.d = e->d; A.T = e->T; A.majority = e->majority;
    A.f = e->cfg.fault_tolerance; A.n_policies = e->n_policies; A.balanced = e->balanced;
    A.peer_alive = peer_alive; A.policy = policy; A.policies = e->policies; A.cw_loc = e->cw_loc;
    A.window_base = e->window_base; A.accepting = e->accepting; A.committed = e->committed; A.bal_prepared = e->bal_prepared;
    A.planes = e->planes; A.inst_bal = e->inst_bal; A.policy_idx = e->policy_idx;
    A.first = e->fb_first; A.mask = e->fb_mask; A.c_rec = e->fb_cnt; A.c_store = e->fb_cnt + n_listed;
    uint64_t *tot = totals != nullptr ? totals : e->fb_words + 2;
    A.tot = tot; A.words = e->fb_words;
    A.store_used = store_used; A.store_used_out = store_used; A.store_cap = plane_stride; A.dec_cap = dec_capacity;
    A.shards = shards; A.dec_slot = dec_slot; A.dec_ballot = dec_ballot; A.dec_off = dec_shard_off; A.dec_len = dec_data_len;
    A.dec_group = dec_group; A.dec_policy = dec_policy; A.verdict = verdict; A.status = ctx->dev_status;
    SS_CUDA(cudaMemsetAsync(e->fb_words, 0, 16, ctx->stream));
    if (n_listed == 0) {
        if (totals != nullptr) SS_CUDA(cudaMemsetAsync(totals, 0, 16, ctx->stream));
        return SS_OK;
    }
    const uint32_t grid_t = launch_grid(ctx, n_listed, kFbThreads), grid_w = launch_grid(ctx, n_listed, kFbThreads / 32);
    fb_mark_kernel<<<grid_t, kFbThreads, 0, ctx->stream>>>(A);
    SS_TRY(launched(ctx));
    fb_count_kernel<<<grid_w, kFbThreads, 0, ctx->stream>>>(A);
    SS_TRY(launched(ctx));
    for (int c = 0; c < 2; ++c) SS_TRY(launch_exclusive_scan_u64(ctx, e->fb_cnt + c * n_listed, n_listed, e->fb_partials, tot + c));
    fb_apply_kernel<<<grid_w, kFbThreads, 0, ctx->stream>>>(A);
    SS_TRY(launched(ctx));
    fb_copy_kernel<<<launch_grid(ctx, dec_capacity, kFbThreads / 32), kFbThreads, 0, ctx->stream>>>(A, plane_stride);
    return launched(ctx);
}
