// craft_recover.cu -- WAL recovery on the CRaft follower (ss_follower_recover): recover_from_wal
// (craft/recovery.rs:11-165) for the DurEntry::Metadata and DurEntry::LogEntry records a replica wrote, for a batch of
// records of many groups at once:
//
//   frecover_header_kernel   a thread per record: the Metadata fields, or the LogEntry decoded by ent_parse (the
//                            follower's entry rules, craft_frames.cuh); sort keys
//   (CUB radix sort)         record indices stably sorted by group: each group's records in WAL order
//   frecover_walk_kernel     a thread per group segment: the verdicts in WAL order (Metadata first, then LogEntry
//                            records; the log ends at the first record that breaks this), the entries against the
//                            window, the group's store bytes
//   (engine.cu's scan)       group regions: exclusive scan over the groups
//   frecover_apply_kernel    a thread per group segment: the capacity cut, then the term and vote words and the whole
//                            ring of the group; each entry's region from the group's offset
//   frecover_copy_kernel     a warp per applied LogEntry: its shards into the padded store slots (the append's copy)
//
// Stated differences from the reference: include/summerset_b200.h at ss_follower_recover.
#include <cub/device/device_radix_sort.cuh>

#include "codeword_wire.cuh"
#include "craft_frames.cuh"
#include "follower_state.hpp"
#include "ss_internal.hpp"
#include "wire_common.cuh"

namespace ssb {

constexpr int kFrThreads = 256;
constexpr uint32_t kFrMeta = 0xfffffffdu;           // decoded kinds, before the walk gives the verdicts
constexpr uint32_t kFrLog = 0xfffffffcu;

// one decoded record; lives in the follower's header scratch (FolHdr-sized slots)
struct FrHdr {
    uint64_t term;                  // Metadata: curr_term; LogEntry: the entry's term
    uint64_t so;                    // LogEntry: its store offset (frecover_apply_kernel)
    uint32_t dl, sl, held, tags_at; // LogEntry: data_len, shard_len, present shards, shard 0's Option tag from the record start
    uint32_t kind;                  // kFrMeta, kFrLog or SS_FRAME_KIND_MALFORMED
    uint8_t voted_for;              // Metadata
};
static_assert(sizeof(FrHdr) <= sizeof(FolHdr) && alignof(FrHdr) <= alignof(FolHdr), "FrHdr reuses the follower's FolHdr scratch");

struct FrArgs {
    const uint8_t *buf;
    uint64_t buf_len;
    const uint64_t *rec_off;
    const uint32_t *rec_group;
    uint64_t n, G;
    uint32_t d, T, W, meta_variant, log_variant;
    // state
    const uint64_t *start_slot;
    uint64_t *log_end, *curr_term;
    uint8_t *leader;
    uint64_t *term, *shard_addr;
    uint32_t *held, *data_len;
    uint64_t *vote_term;
    uint8_t *voted_for;
    // scratch
    FrHdr *hdr;
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

// record i: 8-byte big-endian length, then DurEntry::Metadata{curr_term, voted_for} (a raw ReplicaId byte) or
// DurEntry::LogEntry{entry} whose entry is decoded as ss_follower_append decodes one (log_offset read and dropped)
__device__ __forceinline__ FrHdr fr_decode(const FrArgs &A, uint64_t i) {
    FrHdr h{};
    h.kind = SS_FRAME_KIND_MALFORMED;
    const uint64_t off = A.rec_off[i];
    const uint8_t *b;
    uint64_t len, v = 0, n = 0;
    if (!frame_body(A.buf, A.buf_len, off, kMaxFrameBody, b, len) || !wv_next(b, len, n, v)) return h;
    const uint8_t *fr = b - 8;
    if (v == A.meta_variant) {
        uint64_t ct = 0;
        if (!wv_next(b, len, n, ct) || len - n != 1u) return h;            // voted_for, then the end
        h.term = ct;
        h.voted_for = b[n];
        h.kind = kFrMeta;
    } else if (v == A.log_variant) {
        Ent e;
        if (!ent_parse(fr, 8u + len, 8u + n, A.d, A.T, e) || e.next != 8u + len) return h;
        h.term = e.term; h.dl = static_cast<uint32_t>(e.dl); h.sl = static_cast<uint32_t>(e.sl); h.held = e.held;
        h.tags_at = e.tags_at;
        h.kind = kFrLog;
    }
    return h;
}

// 1. a thread per record
__global__ void __launch_bounds__(kFrThreads) frecover_header_kernel(const __grid_constant__ FrArgs A) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kFrThreads;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kFrThreads + threadIdx.x; i < A.n; i += stride) {
        A.hdr[i] = fr_decode(A, i);
        const uint32_t grp = A.rec_group[i];
        A.key_in[i] = grp < A.G ? grp : static_cast<uint32_t>(A.G);
        A.idx_in[i] = static_cast<uint32_t>(i);
    }
}

__device__ __forceinline__ uint64_t fr_segment_end(const FrArgs &A, uint64_t t) {
    uint64_t e = t + 1u;
    while (e < A.n && A.key[e] == A.key[t]) ++e;
    return e;
}

// 2. a thread per group segment, records in WAL order: Metadata first, LogEntry records after it; the log ends at the
//    first record that is neither (the reference's read loop stops at an entry it cannot decode and truncates).  A log
//    of more than W entries refuses the whole group: a shorter log could lose an acknowledged entry.
__global__ void __launch_bounds__(kFrThreads) frecover_walk_kernel(const __grid_constant__ FrArgs A) {
    bool over = false;
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kFrThreads;
    for (uint64_t t = static_cast<uint64_t>(blockIdx.x) * kFrThreads + threadIdx.x; t < A.n; t += stride) {
        if (t != 0u && A.key[t] == A.key[t - 1]) continue;
        const uint32_t g = A.key[t];
        const uint64_t e = fr_segment_end(A, t);
        if (g >= A.G) {                                                        // no such group: each record alone
            for (uint64_t k = t; k < e; ++k) A.verdict[A.idx[k]] = SS_FRAME_KIND_MALFORMED;
            continue;
        }
        uint64_t cnt = 0u, bytes = 0u;
        bool ended = false;
        for (uint64_t k = t; k < e; ++k) {
            const uint32_t i = A.idx[k];
            const FrHdr h = A.hdr[i];
            uint32_t v;
            if (ended) {
                v = SS_RECOVER_VERDICT_AFTER_END;
            } else if (h.kind == (k == t ? kFrMeta : kFrLog)) {
                v = SS_FOLLOWER_VERDICT_ACCEPTED;
                if (k != t) {
                    ++cnt;
                    bytes += static_cast<uint64_t>(__popc(h.held)) * SS_CW_SLOT_PITCH(h.sl);
                }
            } else {
                v = SS_FRAME_KIND_MALFORMED;
                ended = true;
            }
            A.verdict[i] = v;
        }
        if (cnt > A.W) {
            for (uint64_t k = t; k < e; ++k) A.verdict[A.idx[k]] = SS_FOLLOWER_VERDICT_BEYOND_WINDOW;
            bytes = 0u;
            over = true;
        }
        A.grp_off[g] = bytes;
    }
    if (over) atomicOr(A.status, SS_DEV_STATUS_FRAME_OVERFLOW);
}

// 3. a thread per group segment: a group whose region ends past the capacity applies nothing; a group whose Metadata
//    applied takes its term and vote, and, when an entry applied, a whole new ring: entry k at slot start_slot + k with
//    its region at the group's offset plus the regions before it, every other position zero
__global__ void __launch_bounds__(kFrThreads) frecover_apply_kernel(const __grid_constant__ FrArgs A) {
    bool full = false;
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kFrThreads;
    for (uint64_t t = static_cast<uint64_t>(blockIdx.x) * kFrThreads + threadIdx.x; t < A.n; t += stride) {
        if (t != 0u && A.key[t] == A.key[t - 1]) continue;
        const uint32_t g = A.key[t];
        if (g >= A.G) continue;
        const uint64_t e = fr_segment_end(A, t);
        const uint64_t off = A.grp_off[g], end = g + 1u < A.G ? A.grp_off[g + 1u] : *A.total;
        if (end > A.store_cap) {                                               // the ends are monotone: a suffix of groups
            for (uint64_t k = t; k < e; ++k) {
                const uint32_t i = A.idx[k];
                if (A.verdict[i] != SS_FOLLOWER_VERDICT_ACCEPTED) continue;
                A.verdict[i] = SS_FOLLOWER_VERDICT_STORE_FULL;
                full = true;
            }
            continue;
        }
        const uint32_t i0 = A.idx[t];
        if (A.verdict[i0] != SS_FOLLOWER_VERDICT_ACCEPTED) continue;           // no Metadata first, or refused
        const uint64_t ct = A.hdr[i0].term;
        A.curr_term[g] = ct;
        A.leader[g] = kNone;
        A.vote_term[g] = ct;
        A.voted_for[g] = A.hdr[i0].voted_for;
        const uint64_t start = A.start_slot[g], row = static_cast<uint64_t>(g) * A.W, wm = A.W - 1u;
        uint64_t o = off, cnt = 0u;
        for (uint64_t k = t + 1u; k < e; ++k, ++cnt) {                         // the applied entries are a prefix
            const uint32_t i = A.idx[k];
            if (A.verdict[i] != SS_FOLLOWER_VERDICT_ACCEPTED) break;
            const FrHdr &h = A.hdr[i];
            const uint64_t pos = row + ((start + cnt) & wm);
            A.term[pos] = h.term;
            A.held[pos] = h.held;
            A.data_len[pos] = h.dl;
            A.shard_addr[pos] = reinterpret_cast<uint64_t>(A.store + o);
            A.hdr[i].so = o;
            o += static_cast<uint64_t>(__popc(h.held)) * SS_CW_SLOT_PITCH(h.sl);
        }
        if (cnt == 0u) continue;
        A.log_end[g] = start + cnt;
        for (; cnt < A.W; ++cnt) {
            const uint64_t pos = row + ((start + cnt) & wm);
            A.term[pos] = 0u;
            A.held[pos] = 0u;
            A.data_len[pos] = 0u;
            A.shard_addr[pos] = 0u;
        }
    }
    if (full) atomicOr(A.status, SS_DEV_STATUS_STORE_FULL);
}

// 4. a warp per applied LogEntry holding shards: its shards into their padded store slots
__global__ void __launch_bounds__(kFrThreads) frecover_copy_kernel(const __grid_constant__ FrArgs A) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = (static_cast<uint64_t>(blockIdx.x) * kFrThreads + threadIdx.x) >> 5;
    const uint64_t nwarps = (static_cast<uint64_t>(gridDim.x) * kFrThreads) >> 5;
    for (uint64_t i = warp; i < A.n; i += nwarps) {
        if (A.verdict[i] != SS_FOLLOWER_VERDICT_ACCEPTED) continue;
        const FrHdr h = A.hdr[i];
        if (h.kind != kFrLog || h.held == 0u) continue;
        warp_fill_shards(A.store + h.so, A.buf + A.rec_off[i] + h.tags_at, A.T, h.held, h.held, h.sl, lane);
    }
}

}  // namespace ssb

using namespace ssb;

extern "C" int ss_follower_recover(ss_follower *f, const uint8_t *buf, uint64_t buf_len, const uint64_t *rec_off,
                                   const uint32_t *rec_group, uint64_t n, uint8_t *store, uint64_t store_capacity,
                                   uint32_t *verdict, uint64_t *total) {
    if (f == nullptr) return set_error(SS_ERR_INVALID_ARG, "null follower");
    if (f->cfg.meta_variant == f->cfg.log_variant)
        return set_error(SS_ERR_INVALID_ARG, "the Metadata and LogEntry variants must differ (both %u)", f->cfg.log_variant);
    ss_ctx *ctx = f->ctx;
    SS_TRY(ctx_bind(ctx));
    if (n == 0) {
        if (total != nullptr) SS_CUDA(cudaMemsetAsync(total, 0, 8, ctx->stream));
        return SS_OK;
    }
    if (!buf || !rec_off || !rec_group || !store || !verdict) return set_error(SS_ERR_INVALID_ARG, "null buffer");
    if (reinterpret_cast<uintptr_t>(store) & 15u) return set_error(SS_ERR_INVALID_ARG, "store must be 16-byte aligned");
    if (n > 0x7fffffffull) return set_error(SS_ERR_INVALID_ARG, "at most 2^31 - 1 records per call");
    SS_TRY(el_state(f));
    SS_TRY(fol_scratch(f, n));
    uint64_t *tot = total != nullptr ? total : f->words + 2;
    FrArgs R{};
    R.buf = buf; R.buf_len = buf_len; R.rec_off = rec_off; R.rec_group = rec_group; R.n = n; R.G = f->G;
    R.d = f->d; R.T = f->T; R.W = f->W; R.meta_variant = f->cfg.meta_variant; R.log_variant = f->cfg.log_variant;
    R.start_slot = f->start_slot; R.log_end = f->log_end; R.curr_term = f->curr_term; R.leader = f->leader;
    R.term = f->term; R.shard_addr = f->shard_addr; R.held = f->held; R.data_len = f->data_len;
    R.vote_term = f->vote_term; R.voted_for = f->voted_for;
    R.hdr = reinterpret_cast<FrHdr *>(f->hdr); R.key_in = f->keys; R.idx_in = f->idx; R.key = f->keys + n; R.idx = f->idx + n;
    R.grp_off = f->ex_bytes;        // execute's per-group scratch: both calls are ordered on the context's stream
    R.total = tot;
    R.store = store; R.store_cap = store_capacity; R.verdict = verdict; R.status = ctx->dev_status;
    const uint32_t grid_t = launch_grid(ctx, n, kFrThreads);
    frecover_header_kernel<<<grid_t, kFrThreads, 0, ctx->stream>>>(R);
    SS_TRY(launched(ctx));
    size_t bytes = f->sort_tmp_bytes;
    SS_CUDA(cub::DeviceRadixSort::SortPairs(f->sort_tmp, bytes, f->keys, f->keys + n, f->idx, f->idx + n, static_cast<int>(n), 0,
                                            key_bits(f->G), ctx->stream));
    SS_TRY(launched(ctx));
    SS_CUDA(cudaMemsetAsync(f->ex_bytes, 0, f->G * 8, ctx->stream));
    frecover_walk_kernel<<<grid_t, kFrThreads, 0, ctx->stream>>>(R);
    SS_TRY(launched(ctx));
    SS_TRY(launch_exclusive_scan_u64(ctx, f->ex_bytes, f->G, f->ex_partials, tot));
    frecover_apply_kernel<<<grid_t, kFrThreads, 0, ctx->stream>>>(R);
    SS_TRY(launched(ctx));
    frecover_copy_kernel<<<launch_grid(ctx, n, kFrThreads / 32), kFrThreads, 0, ctx->stream>>>(R);
    return launched(ctx);
}
