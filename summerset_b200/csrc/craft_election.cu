// craft_election.cu -- CRaft elections on the follower: campaigns, RequestVote frames answered, votes tallied.
//
//   ss_follower_campaign   become_a_candidate (craft/leadership.rs:143-209) for the listed groups:
//     campaign_key_kernel      a thread per listing: sort keys
//     (CUB radix sort)         stable: each group's listings in listing order, the first one at the head
//     campaign_kernel          a thread per listing: verdict; the first listing of a group runs the campaign, its
//                              Metadata cell and its RequestVote frame
//   ss_follower_vote       handle_msg_request_vote (craft/messages.rs:499-591):
//     vote_head_kernel         a thread per frame: decode and check the frame, sort keys; outputs of the frames that
//                              take no part
//     (CUB radix sort)         stable: each group's frames in frame order
//     vote_replay_kernel       a thread per group segment: check_term, the grant rule, Metadata and reply cells
//   ss_follower_tally      handle_msg_request_vote_reply (craft/messages.rs:593-619):
//     tally_head_kernel        as vote_head_kernel
//     (CUB radix sort)
//     tally_replay_kernel      a thread per group segment: check_term, the vote set, the majority; a flag per segment
//                              head for the groups the call elected
//     (engine.cu's scan)       the elected groups' places, in group order
//     tally_won_kernel         a thread per segment head: won_group / won_term
//
// The election state sits beside the follower's and is read through curr_term and leader, so ss_follower_append is
// unchanged: a vote counts while vote_term == curr_term, a candidacy or election while role_term == curr_term and
// leader == me.  A term raise in the append's check_term, or a same-term AppendEntries setting leader to its sender,
// ends both without the append touching these arrays.
#include <cub/device/device_radix_sort.cuh>

#include <cstring>

#include "craft_frames.cuh"
#include "device_common.cuh"
#include "engine_state.hpp"
#include "follower_state.hpp"
#include "ss_internal.hpp"
#include "wire_common.cuh"

namespace ssb {

constexpr int kElThreads = 256;
constexpr uint32_t kVoteCell = 48u, kReplyCell = 32u;

// ---- campaign ------------------------------------------------------------------------------------------------------
struct CampaignArgs {
    const uint32_t *groups;
    const uint8_t *timeout_source;  // nullptr: no check
    uint64_t n, G;
    uint32_t W, me, variant, meta_variant;
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
    uint8_t *frames;
    uint32_t *frame_len;
    uint8_t *frame_dst;
    uint32_t *verdict;
};

__global__ void __launch_bounds__(kElThreads) campaign_key_kernel(const __grid_constant__ CampaignArgs A) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kElThreads;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kElThreads + threadIdx.x; i < A.n; i += stride) {
        const uint32_t g = A.groups[i];
        A.key_in[i] = g < A.G ? g : static_cast<uint32_t>(A.G);
        A.idx_in[i] = static_cast<uint32_t>(i);
    }
}

// a thread per sorted listing: only the head of a group's run (its first listing) may campaign
__global__ void __launch_bounds__(kElThreads) campaign_kernel(const __grid_constant__ CampaignArgs A) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kElThreads;
    for (uint64_t t = static_cast<uint64_t>(blockIdx.x) * kElThreads + threadIdx.x; t < A.n; t += stride) {
        const uint32_t i = A.idx[t], g = A.key[t];
        A.meta_len[i] = 0u;
        A.frame_len[i] = 0u;
        A.frame_dst[i] = kNone;
        if (g >= A.G || (t != 0u && A.key[t - 1u] == g)) {
            A.verdict[i] = SS_CAMPAIGN_VERDICT_IGNORED;
            continue;
        }
        const uint64_t ct = A.curr_term[g];
        const uint8_t ldr = A.leader[g];
        if (A.role_term[g] == ct && ldr == A.me && A.role[g] != SS_FOLLOWER_ROLE_FOLLOWER) {
            A.verdict[i] = SS_CAMPAIGN_VERDICT_NOT_FOLLOWER;
        } else if (A.timeout_source != nullptr && ldr != kNone && ldr != A.timeout_source[i]) {
            A.verdict[i] = SS_CAMPAIGN_VERDICT_OTHER_LEADER;
        } else if (ct >= 0xffffffffull) {
            A.verdict[i] = SS_CAMPAIGN_VERDICT_RANGE;
        } else {
            const uint64_t nt = ct + 1u;
            const uint8_t me = static_cast<uint8_t>(A.me);
            A.curr_term[g] = nt;
            A.leader[g] = me;
            A.vote_term[g] = nt;
            A.voted_for[g] = me;
            A.role_term[g] = nt;
            A.role[g] = SS_FOLLOWER_ROLE_CANDIDATE;
            A.votes[g] = 1u << A.me;
            A.meta_len[i] = el_put_meta(A.meta + static_cast<uint64_t>(i) * kMetaCell, A.meta_variant, nt, me);
            // PeerMessage::Msg{RequestVote{term, last_slot, last_term}}: the same bytes for every peer
            const uint64_t last = A.log_end[g] - 1u;
            uint8_t *cell = A.frames + static_cast<uint64_t>(i) * kVoteCell;
            uint32_t m = 8u;
            m += wv_put(cell + m, 0u);
            m += wv_put(cell + m, A.variant);
            m += wv_put(cell + m, nt);
            m += wv_put(cell + m, last);
            m += wv_put(cell + m, A.term[static_cast<uint64_t>(g) * A.W + (last & (A.W - 1u))]);
            put_be64(cell, m - 8u);
            for (uint32_t q = m; q < kVoteCell; ++q) cell[q] = 0u;
            A.frame_len[i] = m;
            A.verdict[i] = SS_CAMPAIGN_VERDICT_DONE;
        }
    }
}

// ---- vote and tally ------------------------------------------------------------------------------------------------
// ElectArgs and el_decode are in craft_frames.cuh, beside the other term-carrying messages' decoders
template <bool kReply>
__device__ __forceinline__ void el_head(const ElectArgs &A) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kElThreads;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kElThreads + threadIdx.x; i < A.n; i += stride) {
        uint64_t f0 = 0, f1 = 0, f2 = 0;
        const uint32_t kind = el_decode<kReply>(A, i, f0, f1, f2);
        A.meta_len[i] = 0u;
        if (!kReply) {
            A.reply_len[i] = 0u;
            A.reply_dst[i] = kNone;
        }
        if (kind != kPending) A.verdict[i] = kind;
        A.key_in[i] = kind == kPending ? A.frame_group[i] : static_cast<uint32_t>(A.G);
        A.idx_in[i] = static_cast<uint32_t>(i);
    }
}

__global__ void __launch_bounds__(kElThreads) vote_head_kernel(const __grid_constant__ ElectArgs A) { el_head<false>(A); }
__global__ void __launch_bounds__(kElThreads) tally_head_kernel(const __grid_constant__ ElectArgs A) { el_head<true>(A); }

// PeerMessage::Msg{RequestVoteReply{term, granted}} into a 32-byte cell (at most 8 + 1 + 3 + 9 + 1 bytes)
__device__ __forceinline__ uint32_t el_put_reply(uint8_t *cell, uint32_t variant, uint64_t term, bool granted) {
    uint32_t m = 8u;
    m += wv_put(cell + m, 0u);
    m += wv_put(cell + m, variant);
    m += wv_put(cell + m, term);
    cell[m++] = granted ? 1u : 0u;
    put_be64(cell, m - 8u);
    for (uint32_t q = m; q < kReplyCell; ++q) cell[q] = 0u;
    return m;
}

// a thread per group segment: the group's RequestVote frames in frame order, as handle_msg_request_vote meets them
__global__ void __launch_bounds__(kElThreads) vote_replay_kernel(const __grid_constant__ ElectArgs A) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kElThreads;
    for (uint64_t t = static_cast<uint64_t>(blockIdx.x) * kElThreads + threadIdx.x; t < A.n; t += stride) {
        const uint32_t g = A.key[t];
        if (g >= A.G || (t != 0u && A.key[t - 1u] == g)) continue;
        const uint64_t le = A.log_end[g], my_last_term = A.term[static_cast<uint64_t>(g) * A.W + ((le - 1u) & (A.W - 1u))];
        uint64_t ct = A.curr_term[g];
        uint8_t ldr = A.leader[g], vf = A.vote_term[g] == ct ? A.voted_for[g] : kNone;
        bool wrote = false;
        for (uint64_t k = t; k < A.n && A.key[k] == g; ++k) {
            const uint32_t i = A.idx[k];
            uint64_t term = 0, last_slot = 0, last_term = 0;
            el_decode<false>(A, i, term, last_slot, last_term);
            const uint8_t cand = A.frame_peer[i];
            bool meta = false;
            if (term > ct) {                                                // check_term: durable before the reply
                ct = term;
                vf = kNone;
                ldr = cand;
                meta = true;
            }
            uint32_t v;
            if (term < ct) {
                A.reply_len[i] = el_put_reply(A.replies + static_cast<uint64_t>(i) * kReplyCell, A.reply_variant, ct, false);
                A.reply_dst[i] = cand;
                v = SS_VOTE_VERDICT_DENIED_STALE;
            } else if ((vf == kNone || vf == cand) && (last_term >= my_last_term || (last_term == ct && last_slot >= le - 1u))) {
                vf = cand;
                meta = true;
                A.reply_len[i] = el_put_reply(A.replies + static_cast<uint64_t>(i) * kReplyCell, A.reply_variant, ct, true);
                A.reply_dst[i] = cand;
                v = SS_VOTE_VERDICT_GRANTED;
            } else {
                v = SS_VOTE_VERDICT_NO_REPLY;
            }
            if (meta) A.meta_len[i] = el_put_meta(A.meta + static_cast<uint64_t>(i) * kMetaCell, A.meta_variant, ct, vf);
            wrote |= meta;
            A.verdict[i] = v;
        }
        if (wrote) {
            A.curr_term[g] = ct;
            A.leader[g] = ldr;
            A.vote_term[g] = ct;
            A.voted_for[g] = vf;
        }
    }
}

// a thread per group segment: the group's RequestVoteReply frames in frame order, as handle_msg_request_vote_reply meets
// them; won_flag[t] = 1 at the head of a group this call elected and that is still elected at its end
__global__ void __launch_bounds__(kElThreads) tally_replay_kernel(const __grid_constant__ ElectArgs A) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kElThreads;
    for (uint64_t t = static_cast<uint64_t>(blockIdx.x) * kElThreads + threadIdx.x; t < A.n; t += stride) {
        A.won_flag[t] = 0u;
        const uint32_t g = A.key[t];
        if (g >= A.G || (t != 0u && A.key[t - 1u] == g)) continue;
        uint64_t ct = A.curr_term[g];
        uint8_t ldr = A.leader[g], role = A.role_term[g] == ct && ldr == A.me ? A.role[g] : static_cast<uint8_t>(SS_FOLLOWER_ROLE_FOLLOWER);
        uint32_t votes = A.votes[g];
        uint8_t counted_role = SS_FOLLOWER_ROLE_CANDIDATE;          // the role the last counted vote left
        bool raised = false, counted = false, won = false;
        for (uint64_t k = t; k < A.n && A.key[k] == g; ++k) {
            const uint32_t i = A.idx[k];
            uint64_t term = 0, granted = 0, unused = 0;
            el_decode<true>(A, i, term, granted, unused);
            const uint8_t peer = A.frame_peer[i];
            uint32_t v;
            if (term > ct) {                                                // check_term: the group steps down
                ct = term;
                ldr = peer;
                role = SS_FOLLOWER_ROLE_FOLLOWER;
                raised = true;
                won = false;
                A.meta_len[i] = el_put_meta(A.meta + static_cast<uint64_t>(i) * kMetaCell, A.meta_variant, ct, kNone);
                v = SS_TALLY_VERDICT_HIGHER_TERM;
            } else if (role == SS_FOLLOWER_ROLE_ELECTED) {
                v = SS_TALLY_VERDICT_ELECTED_ALREADY;
            } else if (role != SS_FOLLOWER_ROLE_CANDIDATE) {
                v = SS_TALLY_VERDICT_NOT_CANDIDATE;
            } else if (term < ct) {
                v = SS_TALLY_VERDICT_STALE_TERM;
            } else if (granted == 0u) {
                v = SS_TALLY_VERDICT_DENIED;
            } else if ((votes >> peer) & 1u) {
                v = SS_TALLY_VERDICT_DUPLICATE;
            } else {
                votes |= 1u << peer;
                counted = true;
                if (static_cast<uint32_t>(__popc(votes)) >= A.majority) {
                    role = counted_role = SS_FOLLOWER_ROLE_ELECTED;
                    won = true;
                    v = SS_TALLY_VERDICT_WON;
                } else {
                    v = SS_TALLY_VERDICT_COUNTED;
                }
            }
            A.verdict[i] = v;
        }
        if (counted) {                                                      // role only changes when a vote counts
            A.votes[g] = votes;
            A.role[g] = counted_role;
        }
        if (raised) {
            A.curr_term[g] = ct;
            A.leader[g] = ldr;
            A.vote_term[g] = ct;
            A.voted_for[g] = kNone;
        }
        A.won_flag[t] = won ? 1u : 0u;
    }
}

__global__ void __launch_bounds__(kElThreads) tally_won_kernel(const __grid_constant__ ElectArgs A) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kElThreads;
    for (uint64_t t = static_cast<uint64_t>(blockIdx.x) * kElThreads + threadIdx.x; t < A.n; t += stride) {
        const uint64_t at = A.won_flag[t], end = t + 1u < A.n ? A.won_flag[t + 1u] : *A.n_won;
        if (end == at) continue;
        const uint32_t g = A.key[t];
        A.won_group[at] = g;
        A.won_term[at] = A.curr_term[g];
    }
}

// the election arrays, allocated on first use: no vote, no candidacy
int el_state(ss_follower *f) {
    if (f->vote_term != nullptr) return SS_OK;
    ss_ctx *ctx = f->ctx;
    const uint64_t G = f->G;
    uint64_t *vt = nullptr, *rt = nullptr;
    uint8_t *vf = nullptr, *role = nullptr;
    uint32_t *votes = nullptr;
    if (cudaMalloc(reinterpret_cast<void **>(&vt), G * 8) != cudaSuccess || cudaMalloc(reinterpret_cast<void **>(&rt), G * 8) != cudaSuccess ||
        cudaMalloc(reinterpret_cast<void **>(&vf), G) != cudaSuccess || cudaMalloc(reinterpret_cast<void **>(&role), G) != cudaSuccess ||
        cudaMalloc(reinterpret_cast<void **>(&votes), G * 4) != cudaSuccess) {
        cudaGetLastError();
        void *bufs[] = {vt, rt, vf, role, votes};
        for (void *b : bufs)
            if (b) cudaFree(b);
        return set_error(SS_ERR_OUT_OF_MEMORY, "election state allocation failed");
    }
    f->vote_term = vt; f->role_term = rt; f->voted_for = vf; f->role = role; f->votes = votes;
    SS_CUDA(cudaMemsetAsync(vt, 0, G * 8, ctx->stream));
    SS_CUDA(cudaMemsetAsync(rt, 0, G * 8, ctx->stream));
    SS_CUDA(cudaMemsetAsync(vf, 0xff, G, ctx->stream));
    SS_CUDA(cudaMemsetAsync(role, 0, G, ctx->stream));
    SS_CUDA(cudaMemsetAsync(votes, 0, G * 4, ctx->stream));
    return SS_OK;
}

// the tally's won flags, grow-only
static int el_won_scratch(ss_follower *f, uint64_t n) {
    if (n <= f->won_cap) return SS_OK;
    SS_CUDA(cudaStreamSynchronize(f->ctx->stream));
    if (f->won_flag) cudaFree(f->won_flag);
    f->won_flag = nullptr;
    f->won_cap = 0;
    SS_CUDA(cudaMalloc(reinterpret_cast<void **>(&f->won_flag), (n + 1u) * 8));
    f->won_cap = n;
    return SS_OK;
}

static void el_fill(ElectArgs &A, ss_follower *f, uint64_t n) {
    A.n = n; A.G = f->G; A.W = f->W; A.me = f->cfg.me; A.population = f->cfg.population; A.majority = f->d;
    A.meta_variant = f->cfg.meta_variant;
    A.log_end = f->log_end; A.term = f->term; A.curr_term = f->curr_term; A.leader = f->leader;
    A.vote_term = f->vote_term; A.role_term = f->role_term; A.voted_for = f->voted_for; A.role = f->role; A.votes = f->votes;
    A.key_in = f->keys; A.idx_in = f->idx; A.key = f->keys + n; A.idx = f->idx + n;
}

static int el_sort(ss_follower *f, uint64_t n) {
    size_t bytes = f->sort_tmp_bytes;
    SS_CUDA(cub::DeviceRadixSort::SortPairs(f->sort_tmp, bytes, f->keys, f->keys + n, f->idx, f->idx + n, static_cast<int>(n), 0,
                                            key_bits(f->G), f->ctx->stream));
    return launched(f->ctx);
}

}  // namespace ssb

using namespace ssb;

extern "C" {

int ss_follower_vote_view_get(ss_follower *f, ss_follower_vote_view *v) {
    if (f == nullptr || v == nullptr) return set_error(SS_ERR_INVALID_ARG, "null argument");
    SS_TRY(ctx_bind(f->ctx));
    SS_TRY(el_state(f));
    memset(v, 0, sizeof(*v));
    v->n_groups = f->G;
    v->vote_term = f->vote_term; v->voted_for = f->voted_for; v->role_term = f->role_term; v->role = f->role; v->votes = f->votes;
    return SS_OK;
}

int ss_follower_campaign(ss_follower *f, const uint32_t *groups, uint64_t n_listed, const uint8_t *timeout_source,
                         uint32_t request_vote_variant, uint8_t *meta, uint32_t *meta_len, uint8_t *frames, uint32_t *frame_len,
                         uint8_t *frame_dst, uint32_t *verdict) {
    if (request_vote_variant >= kVariantLimit) return set_error(SS_ERR_INVALID_ARG, "request_vote_variant must be < 2^16");
    if (f == nullptr) return set_error(SS_ERR_INVALID_ARG, "null follower");
    ss_ctx *ctx = f->ctx;
    SS_TRY(ctx_bind(ctx));
    if (n_listed == 0) return SS_OK;
    if (!groups || !meta || !meta_len || !frames || !frame_len || !frame_dst || !verdict) return set_error(SS_ERR_INVALID_ARG, "null buffer");
    if (n_listed > 0x7fffffffull) return set_error(SS_ERR_INVALID_ARG, "at most 2^31 - 1 listed groups per call");
    SS_TRY(el_state(f));
    SS_TRY(fol_scratch(f, n_listed));
    CampaignArgs A{};
    A.groups = groups; A.timeout_source = timeout_source; A.n = n_listed; A.G = f->G; A.W = f->W; A.me = f->cfg.me;
    A.variant = request_vote_variant; A.meta_variant = f->cfg.meta_variant;
    A.log_end = f->log_end; A.term = f->term; A.curr_term = f->curr_term; A.leader = f->leader;
    A.vote_term = f->vote_term; A.role_term = f->role_term; A.voted_for = f->voted_for; A.role = f->role; A.votes = f->votes;
    A.key_in = f->keys; A.idx_in = f->idx; A.key = f->keys + n_listed; A.idx = f->idx + n_listed;
    A.meta = meta; A.meta_len = meta_len; A.frames = frames; A.frame_len = frame_len; A.frame_dst = frame_dst; A.verdict = verdict;
    const uint32_t grid = launch_grid(ctx, n_listed, kElThreads);
    campaign_key_kernel<<<grid, kElThreads, 0, ctx->stream>>>(A);
    SS_TRY(launched(ctx));
    SS_TRY(el_sort(f, n_listed));
    campaign_kernel<<<grid, kElThreads, 0, ctx->stream>>>(A);
    return launched(ctx);
}

int ss_follower_vote(ss_follower *f, const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off, const uint32_t *frame_group,
                     const uint8_t *frame_peer, uint64_t n, uint32_t request_vote_variant, uint32_t reply_variant, uint8_t *meta,
                     uint32_t *meta_len, uint8_t *replies, uint32_t *reply_len, uint8_t *reply_dst, uint32_t *verdict) {
    if (request_vote_variant >= kVariantLimit || reply_variant >= kVariantLimit)
        return set_error(SS_ERR_INVALID_ARG, "the variants must be < 2^16");
    if (f == nullptr) return set_error(SS_ERR_INVALID_ARG, "null follower");
    ss_ctx *ctx = f->ctx;
    SS_TRY(ctx_bind(ctx));
    if (n == 0) return SS_OK;
    if (!buf || !frame_off || !frame_group || !frame_peer || !meta || !meta_len || !replies || !reply_len || !reply_dst || !verdict)
        return set_error(SS_ERR_INVALID_ARG, "null buffer");
    if (n > 0x7fffffffull) return set_error(SS_ERR_INVALID_ARG, "at most 2^31 - 1 frames per call");
    SS_TRY(el_state(f));
    SS_TRY(fol_scratch(f, n));
    ElectArgs A{};
    el_fill(A, f, n);
    A.buf = buf; A.buf_len = buf_len; A.frame_off = frame_off; A.frame_group = frame_group; A.frame_peer = frame_peer;
    A.variant = request_vote_variant; A.reply_variant = reply_variant;
    A.meta = meta; A.meta_len = meta_len; A.replies = replies; A.reply_len = reply_len; A.reply_dst = reply_dst; A.verdict = verdict;
    const uint32_t grid = launch_grid(ctx, n, kElThreads);
    vote_head_kernel<<<grid, kElThreads, 0, ctx->stream>>>(A);
    SS_TRY(launched(ctx));
    SS_TRY(el_sort(f, n));
    vote_replay_kernel<<<grid, kElThreads, 0, ctx->stream>>>(A);
    return launched(ctx);
}

int ss_follower_tally(ss_follower *f, const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off, const uint32_t *frame_group,
                      const uint8_t *frame_peer, uint64_t n, uint32_t reply_variant, uint8_t *meta, uint32_t *meta_len, uint32_t *verdict,
                      uint32_t *won_group, uint64_t *won_term, uint64_t *n_won) {
    if (reply_variant >= kVariantLimit) return set_error(SS_ERR_INVALID_ARG, "reply_variant must be < 2^16");
    if (f == nullptr) return set_error(SS_ERR_INVALID_ARG, "null follower");
    ss_ctx *ctx = f->ctx;
    SS_TRY(ctx_bind(ctx));
    if (!won_group || !won_term) return set_error(SS_ERR_INVALID_ARG, "null won_group or won_term");
    if (n != 0 && (!buf || !frame_off || !frame_group || !frame_peer || !meta || !meta_len || !verdict))
        return set_error(SS_ERR_INVALID_ARG, "null buffer");
    if (n > 0x7fffffffull) return set_error(SS_ERR_INVALID_ARG, "at most 2^31 - 1 frames per call");
    SS_CUDA(cudaMemsetAsync(won_group, 0xff, f->G * 4, ctx->stream));
    SS_CUDA(cudaMemsetAsync(won_term, 0, f->G * 8, ctx->stream));
    if (n == 0) {
        if (n_won != nullptr) SS_CUDA(cudaMemsetAsync(n_won, 0, 8, ctx->stream));
        return SS_OK;
    }
    SS_TRY(el_state(f));
    SS_TRY(fol_scratch(f, n));
    SS_TRY(el_won_scratch(f, n));
    ElectArgs A{};
    el_fill(A, f, n);
    A.buf = buf; A.buf_len = buf_len; A.frame_off = frame_off; A.frame_group = frame_group; A.frame_peer = frame_peer;
    A.variant = reply_variant;
    A.meta = meta; A.meta_len = meta_len; A.verdict = verdict;
    uint64_t *tot = n_won != nullptr ? n_won : f->won_flag + n;
    A.won_flag = f->won_flag; A.n_won = tot; A.won_group = won_group; A.won_term = won_term;
    const uint32_t grid = launch_grid(ctx, n, kElThreads);
    tally_head_kernel<<<grid, kElThreads, 0, ctx->stream>>>(A);
    SS_TRY(launched(ctx));
    SS_TRY(el_sort(f, n));
    tally_replay_kernel<<<grid, kElThreads, 0, ctx->stream>>>(A);
    SS_TRY(launched(ctx));
    SS_TRY(launch_exclusive_scan_u64(ctx, f->won_flag, n, f->partials, tot));
    tally_won_kernel<<<grid, kElThreads, 0, ctx->stream>>>(A);
    return launched(ctx);
}

}  // extern "C"
