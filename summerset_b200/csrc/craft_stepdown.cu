// craft_stepdown.cu -- CRaft step-down on the device: check_term (craft/leadership.rs:16-75) for the groups this replica's
// engine leads, over a batch of incoming frames, and the deposed leader's log handed back to its follower.
//
//   ss_engine_craft_step_down
//     sd_head_kernel       a thread per frame: decode by the rules of the call that takes it (craft_frames.cuh), and the
//                          first frame of each led group that carries a higher term (atomicMin)
//     sd_size_kernel       a thread per frame: verdict; a deposing frame walks its group's span for the store bytes and
//                          the entries it copies
//     (engine.cu's scan)   store regions and copy items in frame order
//     sd_commit_kernel     a thread per deposing frame: the capacity cut, then the follower's ring and words, the
//                          Metadata cell, the engine's words, the copy items
//     sd_copy_kernel       a warp per copied entry: its held shards from the engine's planes into the store, 128-bit
//                          copies; then UINT64_MAX into store_off of the frames that took no region
//   ss_engine_craft_role_view_get   the led bytes; craft_led_mark sets them after a step-up
#include <cstring>

#include "craft_frames.cuh"
#include "device_common.cuh"
#include "engine_state.hpp"
#include "follower_state.hpp"
#include "ss_internal.hpp"
#include "wire_common.cuh"

namespace ssb {

constexpr int kSdThreads = 256;
constexpr uint32_t kSdTerm = 0xfffffffdu;         // decoded, carries a term
constexpr uint32_t kSdNoVariant = 0xffffffffu;    // msg_head_count's variant that no frame has: it returns the frame's

struct StepDownArgs {
    FolArgs fa;                     // the append decoder's view (frames, follower window and start_slot)
    ElectArgs ev, er;               // the RequestVote and RequestVoteReply decoders' views
    uint32_t reply_variant;
    uint64_t n, G;
    uint32_t W, FW, d, T, P, meta_variant;
    uint32_t all;                   // every shard: the held mask while the engine's masks are not in use
    // scratch: [G] first deposing frame, [n] kind, [n] term, [n] copy items then their scan, items
    uint64_t *first, *kind, *term, *cnt, *items;
    const uint64_t *n_items;
    uint64_t *need;
    uint8_t *store;
    uint64_t store_cap, *store_off;
    uint8_t *meta;
    uint32_t *meta_len, *verdict, *status;
    uint64_t plane_stride;
    // the follower
    uint64_t *f_start, *f_log_end, *f_curr_term, *f_last_commit, *f_last_snap, *f_last_exec, *f_term, *f_addr;
    uint8_t *f_leader;
    uint32_t *f_held, *f_len;
    // the engine
    const uint64_t *log_start, *last_exec, *ent_addr;
    const uint32_t *log_end, *last_commit, *last_snap, *terms, *ent_len, *held;   // held: nullptr while not in use
    uint32_t *curr_term, *match;
    uint8_t *led;
};

// frame i: kSdTerm with its term, SS_STEPDOWN_VERDICT_PASS for a PeerMsg that carries none, or the verdict of the
// call that takes it (another message's variant index, SS_FRAME_KIND_MALFORMED)
__device__ __forceinline__ uint32_t sd_decode(const StepDownArgs &A, uint64_t i, uint64_t &term) {
    if (A.fa.frame_group[i] >= A.G) return SS_FRAME_KIND_MALFORMED;
    const uint8_t *b = nullptr;
    uint64_t len = 0, n = 0, cnt = 0;
    const uint32_t v = msg_head_count(A.fa.buf, A.fa.buf_len, A.fa.frame_off[i], kSdNoVariant, ~0ull, b, len, n, cnt);
    if (v == SS_FRAME_KIND_MALFORMED || (v & 0x80000000u)) return v;
    uint32_t kind;
    if (v == A.fa.append_variant) {
        const FolHdr h = fol_decode(A.fa, i);
        // a frame past the follower's window still carries its term
        kind = h.kind == kPending || h.kind == SS_FOLLOWER_VERDICT_BEYOND_WINDOW ? kPending : h.kind;
        term = h.term;
    } else if (v == A.reply_variant) {
        // the reply parser's rules, and a sender that is a peer: it becomes the follower's leader
        const uint8_t peer = A.fa.frame_peer[i];
        if (peer == A.fa.me || peer >= A.fa.population) return SS_FRAME_KIND_MALFORMED;
        uint64_t end = 0, c_term = 0, c_slot = 0;
        const uint32_t r = reply_parse(A.fa.buf, A.fa.buf_len, A.fa.frame_off[i], A.fa.frame_group[i], A.G, A.reply_variant,
                                       A.curr_term, term, end, c_term, c_slot);
        kind = r >= SS_APPEND_REPLY_INGEST && r <= SS_APPEND_REPLY_END_RANGE ? kPending : r;
    } else if (v == A.ev.variant) {
        uint64_t f1 = 0, f2 = 0;
        kind = el_decode<false>(A.ev, i, term, f1, f2) == kPending ? kPending : SS_FRAME_KIND_MALFORMED;
    } else if (v == A.er.variant) {
        uint64_t f1 = 0, f2 = 0;
        kind = el_decode<true>(A.er, i, term, f1, f2) == kPending ? kPending : SS_FRAME_KIND_MALFORMED;
    } else {
        return SS_STEPDOWN_VERDICT_PASS;                                    // Reconstruct, ReconstructReply
    }
    return kind == kPending ? kSdTerm : kind;
}

__global__ void __launch_bounds__(kSdThreads) sd_head_kernel(const __grid_constant__ StepDownArgs A) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kSdThreads;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kSdThreads + threadIdx.x; i < A.n; i += stride) {
        uint64_t term = 0;
        const uint32_t kind = sd_decode(A, i, term);
        A.kind[i] = kind;
        A.term[i] = term;
        const uint32_t g = A.fa.frame_group[i];
        if (kind == kSdTerm && A.led[g] != 0u && term > A.curr_term[g] && term <= 0xffffffffull)
            atomicMin(reinterpret_cast<unsigned long long *>(A.first + g), static_cast<unsigned long long>(i));
    }
}

// the deposed span [max(start_slot, log_start), log_end) of group g; f(slot, follower pos, engine pos, data_len, held,
// reused) for each slot
template <typename F>
__device__ __forceinline__ void sd_walk(const StepDownArgs &A, uint32_t g, F &&f) {
    const uint64_t fs = A.f_start[g], ole = A.f_log_end[g], ls = A.log_start[g], le = A.log_end[g];
    const uint64_t frow = static_cast<uint64_t>(g) * A.FW, erow = static_cast<uint64_t>(g) * A.W;
    for (uint64_t s = fs > ls ? fs : ls; s < le; ++s) {
        const uint64_t fp = frow + (s & (A.FW - 1u)), ep = erow + (s & (A.W - 1u));
        const uint32_t dl = A.ent_len[ep], h = A.held != nullptr ? A.held[ep] : A.all;
        // Log Matching: the same slot and term in the follower's old span hold the same entry, so the same shard bytes
        const bool reused = dl != 0u && s >= fs && s < ole && A.f_term[fp] == A.terms[ep] && A.f_len[fp] == dl && A.f_held[fp] == h;
        f(s, fp, ep, dl, h, reused);
    }
}

__device__ __forceinline__ uint64_t sd_entry_bytes(uint32_t dl, uint32_t held, uint32_t d) {
    return static_cast<uint64_t>(__popc(held)) * SS_CW_SLOT_PITCH((static_cast<uint64_t>(dl) + d - 1u) / d);
}

__global__ void __launch_bounds__(kSdThreads) sd_size_kernel(const __grid_constant__ StepDownArgs A) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kSdThreads;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kSdThreads + threadIdx.x; i < A.n; i += stride) {
        const uint32_t kind = static_cast<uint32_t>(A.kind[i]);
        uint32_t v = kind;
        uint64_t bytes = 0, items = 0;
        if (kind == kSdTerm) {
            const uint32_t g = A.fa.frame_group[i];
            const uint64_t t = A.term[i], first = A.first[g];
            v = SS_STEPDOWN_VERDICT_PASS;
            if (A.led[g] == 0u || first < i || t <= A.curr_term[g]) {
            } else if (t > 0xffffffffull) {
                v = SS_STEPDOWN_VERDICT_RANGE;
            } else {                                                        // first == i
                v = SS_STEPDOWN_VERDICT_DEPOSED;
                sd_walk(A, g, [&](uint64_t, uint64_t, uint64_t, uint32_t dl, uint32_t h, bool reused) {
                    if (dl != 0u && !reused) {
                        bytes += sd_entry_bytes(dl, h, A.d);
                        ++items;
                    }
                });
            }
        }
        A.verdict[i] = v;
        A.meta_len[i] = 0u;
        A.store_off[i] = bytes;
        A.cnt[i] = items;
    }
}

__global__ void __launch_bounds__(kSdThreads) sd_commit_kernel(const __grid_constant__ StepDownArgs A) {
    bool full = false;
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kSdThreads;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kSdThreads + threadIdx.x; i < A.n; i += stride) {
        if (A.verdict[i] != SS_STEPDOWN_VERDICT_DEPOSED) continue;
        // store_off is only read here: the next frame's offset is this one's end (UINT64_MAX goes in with the copies)
        const uint64_t off = A.store_off[i], end = i + 1u < A.n ? A.store_off[i + 1u] : *A.need;
        const uint64_t c0 = A.cnt[i], c1 = i + 1u < A.n ? A.cnt[i + 1u] : *A.n_items;
        if (end > A.store_cap) {                                            // the offsets are monotone: a suffix is cut
            full = true;
            A.verdict[i] = SS_STEPDOWN_VERDICT_STORE_FULL;
            for (uint64_t c = c0; c < c1; ++c) A.items[c] = ~0ull;
            continue;
        }
        const uint32_t g = A.fa.frame_group[i];
        const uint64_t t = A.term[i];
        uint64_t at = off, c = c0;
        sd_walk(A, g, [&](uint64_t s, uint64_t fp, uint64_t ep, uint32_t dl, uint32_t h, bool reused) {
            A.f_term[fp] = A.terms[ep];
            A.f_len[fp] = dl;
            A.f_held[fp] = h;
            if (dl == 0u) {
                A.f_addr[fp] = 0u;
            } else if (!reused) {
                A.f_addr[fp] = reinterpret_cast<uint64_t>(A.store + at);
                at += sd_entry_bytes(dl, h, A.d);
                A.items[c++] = (static_cast<uint64_t>(g) << 32) | s;
            }
        });
        const uint64_t fs = A.f_start[g], ls = A.log_start[g];
        A.f_start[g] = fs > ls ? fs : ls;
        A.f_log_end[g] = A.log_end[g];
        const uint64_t lc = A.last_commit[g], sn = A.last_snap[g], ex = A.last_exec[g];
        if (lc > A.f_last_commit[g]) A.f_last_commit[g] = lc;
        if (sn > A.f_last_snap[g]) A.f_last_snap[g] = sn;
        if (ex > A.f_last_exec[g]) A.f_last_exec[g] = ex;
        if (t > A.f_curr_term[g]) {                                         // check_term: durable before anything else
            A.f_curr_term[g] = t;
            A.meta_len[i] = el_put_meta(A.meta + i * kMetaCell, A.meta_variant, t, kNone);
        }
        A.f_leader[g] = A.fa.frame_peer[i];
        A.led[g] = 0u;
        A.curr_term[g] = static_cast<uint32_t>(t);
        for (uint32_t q = 0; q < A.P; ++q) A.match[static_cast<uint64_t>(q) * A.G + g] = 0u;
    }
    if (full) atomicOr(A.status, SS_DEV_STATUS_STORE_FULL);
}

// a warp per copied entry: held shard j (plane j of the engine's slot) to rank r of its store region, round_up(L, 16)
// bytes, the zero pad included; then, per frame: a term-carrying frame after its group's cut deposing frame is
// STORE_FULL too (the group still leads, so none of them may reach its handler), and store_off is UINT64_MAX for every
// frame that took no region
__global__ void __launch_bounds__(kSdThreads) sd_copy_kernel(const __grid_constant__ StepDownArgs A) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = (static_cast<uint64_t>(blockIdx.x) * kSdThreads + threadIdx.x) >> 5;
    const uint64_t nwarps = (static_cast<uint64_t>(gridDim.x) * kSdThreads) >> 5;
    const uint64_t total = *A.n_items;
    for (uint64_t it = warp; it < total; it += nwarps) {
        const uint64_t item = A.items[it];
        if (item == ~0ull) continue;                                        // its frame was cut
        const uint64_t g = item >> 32, s = item & 0xffffffffull;
        const uint64_t fp = g * A.FW + (s & (A.FW - 1u)), ep = g * A.W + (s & (A.W - 1u));
        const uint64_t L = (A.f_len[fp] + A.d - 1u) / A.d, pitch = SS_CW_SLOT_PITCH(L), nvec = (L + 15u) >> 4;
        const uint8_t *src = reinterpret_cast<const uint8_t *>(A.ent_addr[ep]);
        uint8_t *dst = reinterpret_cast<uint8_t *>(A.f_addr[fp]);
        uint32_t r = 0;
        for (uint32_t rest = A.f_held[fp]; rest != 0u; rest &= rest - 1u, ++r) {
            const uint32_t j = static_cast<uint32_t>(__ffs(static_cast<int>(rest))) - 1u;
            const uint8_t *sj = src + j * A.plane_stride;
            uint8_t *dj = dst + r * pitch;
            for (uint64_t v = lane; v < nvec; v += 32u) dev::stg128_cs(dj + v * 16u, dev::ldg128(sj + v * 16u));
        }
    }
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kSdThreads;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kSdThreads + threadIdx.x; i < A.n; i += stride) {
        const uint32_t v = A.verdict[i];
        if (v == SS_STEPDOWN_VERDICT_PASS && A.kind[i] == kSdTerm) {
            const uint64_t f = A.first[A.fa.frame_group[i]];
            if (f < i && A.verdict[f] == SS_STEPDOWN_VERDICT_STORE_FULL) A.verdict[i] = SS_STEPDOWN_VERDICT_STORE_FULL;
        }
        if (v != SS_STEPDOWN_VERDICT_DEPOSED) A.store_off[i] = ~0ull;
    }
}

__global__ void __launch_bounds__(kSdThreads) led_mark_kernel(const uint32_t *groups, const uint32_t *verdict, uint64_t n, uint64_t G,
                                                              uint8_t *led) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kSdThreads;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kSdThreads + threadIdx.x; i < n; i += stride)
        if (verdict[i] == SS_STEPUP_VERDICT_DONE && groups[i] < G) led[groups[i]] = 1u;
}

int craft_led_in_use(ss_engine *e) {
    if (e->led != nullptr) return SS_OK;
    ss_ctx *ctx = e->ctx;
    SS_CUDA(cudaMalloc(reinterpret_cast<void **>(&e->led), e->G));
    SS_CUDA(cudaMemsetAsync(e->led, 1, e->G, ctx->stream));                // the engine led every group until now
    return SS_OK;
}

int craft_led_mark(ss_engine *e, const uint32_t *groups, const uint32_t *verdict, uint64_t n) {
    if (e->led == nullptr || n == 0) return SS_OK;
    ss_ctx *ctx = e->ctx;
    led_mark_kernel<<<launch_grid(ctx, n, kSdThreads), kSdThreads, 0, ctx->stream>>>(groups, verdict, n, e->G, e->led);
    return launched(ctx);
}

}  // namespace ssb

using namespace ssb;

extern "C" {

int ss_engine_craft_role_view_get(ss_engine *e, ss_engine_craft_role_view *v) {
    if (v == nullptr) return set_error(SS_ERR_INVALID_ARG, "null view");
    SS_TRY(craft_check(e));
    SS_TRY(craft_log_init(e));
    SS_TRY(craft_led_in_use(e));
    memset(v, 0, sizeof(*v));
    v->n_groups = e->G;
    v->led = e->led;
    return SS_OK;
}

int ss_engine_craft_step_down(ss_engine *e, ss_follower *f, const ss_step_down_spec *spec, const uint8_t *buf, uint64_t buf_len,
                              const uint64_t *frame_off, const uint32_t *frame_group, const uint8_t *frame_peer, uint64_t n,
                              uint8_t *store, uint64_t store_capacity, uint64_t *store_off, uint8_t *meta, uint32_t *meta_len,
                              uint32_t *verdict, uint64_t *need) {
    if (f == nullptr) return set_error(SS_ERR_INVALID_ARG, "null follower");
    if (spec == nullptr) return set_error(SS_ERR_INVALID_ARG, "null spec");
    const uint32_t vs[4] = {spec->append_variant, spec->append_reply_variant, spec->request_vote_variant, spec->vote_reply_variant};
    for (int a = 0; a < 4; ++a) {
        if (vs[a] >= kVariantLimit) return set_error(SS_ERR_INVALID_ARG, "the variants must be < 2^16");
        for (int b = 0; b < a; ++b)
            if (vs[a] == vs[b]) return set_error(SS_ERR_INVALID_ARG, "the four variants must differ");
    }
    if (reinterpret_cast<uintptr_t>(store) & 15u) return set_error(SS_ERR_INVALID_ARG, "store must be 16-byte aligned");
    SS_TRY(craft_check(e));
    if (f->cfg.protocol != e->cfg.protocol) return set_error(SS_ERR_INVALID_ARG, "the follower's protocol differs from the engine's");
    if (f->cfg.population != e->n) return set_error(SS_ERR_INVALID_ARG, "the follower's population %u differs from the engine's %u", f->cfg.population, e->n);
    if (f->G != e->G) return set_error(SS_ERR_INVALID_ARG, "the follower's n_groups differs from the engine's");
    if (f->ctx != e->ctx) return set_error(SS_ERR_INVALID_ARG, "the follower and the engine must share a context");
    if (f->W < e->W) return set_error(SS_ERR_INVALID_ARG, "the follower's window %u is smaller than the engine's raft_window %u", f->W, e->W);
    if (n > 0x7fffffffull) return set_error(SS_ERR_INVALID_ARG, "at most 2^31 - 1 frames per call");
    SS_TRY(craft_log_init(e));
    SS_TRY(craft_led_in_use(e));
    ss_ctx *ctx = e->ctx;
    if (n == 0) {
        if (need != nullptr) SS_CUDA(cudaMemsetAsync(need, 0, 8, ctx->stream));
        return SS_OK;
    }
    if (!buf || !frame_off || !frame_group || !frame_peer || !store || !store_off || !meta || !meta_len || !verdict)
        return set_error(SS_ERR_INVALID_ARG, "null buffer");
    const uint64_t G = e->G, span = (n < G ? n : G) * e->W, tiles = scan_tiles(n);
    SS_TRY(rc_scratch(e, G + 3u * n + tiles + 2u + span));
    StepDownArgs A{};
    A.fa.buf = buf; A.fa.buf_len = buf_len; A.fa.frame_off = frame_off; A.fa.frame_group = frame_group; A.fa.frame_peer = frame_peer;
    A.fa.n = n; A.fa.G = G; A.fa.d = f->d; A.fa.T = f->T; A.fa.W = f->W; A.fa.me = f->cfg.me; A.fa.population = f->cfg.population;
    A.fa.append_variant = spec->append_variant; A.fa.log_variant = f->cfg.log_variant; A.fa.start_slot = f->start_slot;
    A.ev.buf = buf; A.ev.buf_len = buf_len; A.ev.frame_off = frame_off; A.ev.frame_group = frame_group; A.ev.frame_peer = frame_peer;
    A.ev.n = n; A.ev.G = G; A.ev.me = f->cfg.me; A.ev.population = f->cfg.population;
    A.er = A.ev;
    A.ev.variant = spec->request_vote_variant;
    A.er.variant = spec->vote_reply_variant;
    A.reply_variant = spec->append_reply_variant;
    A.n = n; A.G = G; A.W = e->W; A.FW = f->W; A.d = e->majority; A.T = e->n; A.P = e->n_peers; A.meta_variant = f->cfg.meta_variant;
    A.all = e->n >= 32u ? 0xffffffffu : (1u << e->n) - 1u;
    uint64_t *w = e->rc_words;
    A.first = w; A.kind = w + G; A.term = w + G + n; A.cnt = w + G + 2u * n;
    uint64_t *partials = w + G + 3u * n, *tot = partials + tiles;
    A.items = tot + 2u;
    A.need = need != nullptr ? need : tot;
    A.n_items = tot + 1u;
    A.store = store; A.store_cap = store_capacity; A.store_off = store_off; A.meta = meta; A.meta_len = meta_len; A.verdict = verdict;
    A.status = ctx->dev_status; A.plane_stride = e->log_plane_stride;
    A.f_start = f->start_slot; A.f_log_end = f->log_end; A.f_curr_term = f->curr_term; A.f_last_commit = f->last_commit;
    A.f_last_snap = f->last_snap; A.f_last_exec = f->last_exec; A.f_term = f->term; A.f_addr = f->shard_addr; A.f_leader = f->leader;
    A.f_held = f->held; A.f_len = f->data_len;
    A.log_start = e->log_start; A.last_exec = e->last_exec; A.ent_addr = e->ent_addr; A.log_end = e->log_end;
    A.last_commit = e->last_commit; A.last_snap = e->last_snap; A.terms = e->terms; A.ent_len = e->ent_len;
    A.held = e->held_partial ? e->held : nullptr; A.curr_term = e->curr_term; A.match = e->match; A.led = e->led;
    const uint32_t grid = launch_grid(ctx, n, kSdThreads);
    SS_CUDA(cudaMemsetAsync(A.first, 0xff, G * 8, ctx->stream));
    sd_head_kernel<<<grid, kSdThreads, 0, ctx->stream>>>(A);
    SS_TRY(launched(ctx));
    sd_size_kernel<<<grid, kSdThreads, 0, ctx->stream>>>(A);
    SS_TRY(launched(ctx));
    SS_TRY(launch_exclusive_scan_u64(ctx, store_off, n, partials, A.need));
    SS_TRY(launch_exclusive_scan_u64(ctx, A.cnt, n, partials, tot + 1u));
    sd_commit_kernel<<<grid, kSdThreads, 0, ctx->stream>>>(A);
    SS_TRY(launched(ctx));
    // a warp per entry the deposed spans can copy, up to the grid cap; warps past the copied count return at once
    sd_copy_kernel<<<launch_grid(ctx, span > n ? span : n, kSdThreads / 32), kSdThreads, 0, ctx->stream>>>(A);
    return launched(ctx);
}

}  // extern "C"
