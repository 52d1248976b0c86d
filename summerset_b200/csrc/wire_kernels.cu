// wire_kernels.cu -- the steps either side of the hot path (SURVEY 8f-2, 8f-4), batched on the device so that what the
// kernels produce can be handed to an unmodified TransportHub / StorageHub, and what those deliver can feed the kernels:
//
//   frame_pack_kernel           PeerMessage::Msg{PeerMsg::Accept{slot, ballot, reqs_cw[, assignment]}} frames for one
//                               destination peer, or WalEntry::AcceptData{slot, ballot, reqs_cw} records -- 8-byte
//                               big-endian length (utils/safetcp.rs:30-88, server/storage.rs:333-337) + bincode body, the
//                               codeword carrying exactly the shards of the peer's assignment (subset_copy(.., false),
//                               rspaxos/request.rs:127-142, crossword/request.rs:164-185; encoding utils/rscoding.rs:43-72,
//                               assignment Vec<Bitmap> utils/bitmap.rs:20-30)
//   frame_size_ragged_kernel    the same frames for ragged codewords (data_len per codeword), packed back to back:
//   frame_pack_ragged_kernel    exact sizes, an exclusive scan of the 16-byte regions (engine.cu), then the frames;
//                               both share frame_layout / frame_write with frame_pack_kernel
//   accept_reply_parse_kernel   AcceptReply frames -> (group, window slot, peer, ballot) records for ss_ack_ingest_dev /
//                               ss_engine_ingest (rspaxos/mod.rs:290-291, crossword/mod.rs:365-373)
//   prepare_reply_parse_kernel  PrepareReply frames -> (slot, trigger, endprep, ballot, vote ballot / shards) records for
//                               the new leader's ss_prepare_merge_dev (rspaxos/messages.rs:88-196)
//   wal_commit_pack_kernel      newly committed instances -> WalEntry::CommitSlot{slot} records (rspaxos/mod.rs:231)
//   reconstruct_serve_kernel    Reconstruct serving: reply shards = held & flip(exclude) per requested instance, packed
//                               (crossword/messages.rs:577-632, rspaxos/messages.rs:468-517)
//
// bincode 2 standard config facts are from knowledge of the crate (unpinned against the reference, DESIGN.md section 4);
// every kernel is tested byte for byte against oracle/ss_wire.c.
#include "codeword_wire.cuh"
#include "device_common.cuh"
#include "ss_internal.hpp"
#include "wire_common.cuh"

namespace ssb {

constexpr int kWireThreads = 256;

struct PackArgs {
    const uint8_t *planes;          // shard j of codeword g at planes + j*plane_stride + g*shard_stride (16-byte aligned slots)
    uint64_t plane_stride, shard_stride;
    uint32_t d, p, data_len, L;
    uint32_t kind;                  // SS_FRAME_PEER_ACCEPT / SS_FRAME_WAL_ACCEPT_DATA
    uint32_t variant;
    const uint32_t *policies;       // [n_policies][population] shard bitmasks
    const uint8_t *policy_idx;      // [n] or nullptr (policy 0)
    uint32_t n_policies, population, peer;
    uint32_t with_assignment, assign_size;
    const uint64_t *slot, *ballot;
    uint64_t n;
    uint8_t *out;
    uint64_t frame_stride;          // uniform: frame g inside out[g*frame_stride ..)
    uint64_t *frame_off;
    uint32_t *frame_len;
    uint32_t *status;               // context's device status word
    // ragged: shard j of codeword g at planes + j*plane_stride + shard_off[g], data_len[g] bytes; packed regions in out
    const uint64_t *shard_off;
    const uint32_t *lens;
    uint64_t capacity;
};

// where the bytes of frame g go, known before a byte is written
struct FrameLayout {
    const uint32_t *pol;            // the codeword's policy row
    uint32_t mask;                  // shards carried for this peer
    uint32_t h;                     // fixed fields after the length prefix
    uint32_t some_len;              // Some tag + byte length of one carried shard
    uint32_t pad;                   // bytes before the frame that put its first carried shard on a 16-byte boundary
    uint64_t len;                   // frame bytes: 8-byte length prefix + body
};

__device__ __forceinline__ FrameLayout frame_layout(const PackArgs &A, uint64_t g, uint32_t data_len, uint32_t L) {
    FrameLayout F;
    const uint32_t T = A.d + A.p;
    uint32_t k = A.policy_idx != nullptr ? A.policy_idx[g] : 0u;
    if (k >= A.n_policies) k = 0u;
    F.pol = A.policies + static_cast<uint64_t>(k) * A.population;
    F.mask = __ldg(F.pol + A.peer) & (T >= 32u ? 0xffffffffu : ((1u << T) - 1u));
    F.h = (A.kind == SS_FRAME_PEER_ACCEPT ? 1u : 0u) + static_cast<uint32_t>(wv_len(A.variant) + wv_len(__ldg(A.slot + g)) +
          wv_len(__ldg(A.ballot + g))) + 2u + static_cast<uint32_t>(wv_len(data_len) + wv_len(L) + wv_len(T));
    F.some_len = 1u + static_cast<uint32_t>(wv_len(L));
    // bytes before the first carried shard's payload decide the padding that makes that payload 16-byte aligned
    const uint32_t first = F.mask ? static_cast<uint32_t>(__ffs(F.mask) - 1) : T;
    const uint32_t pre = 8u + F.h + first + (F.mask ? F.some_len : 0u);
    F.pad = (16u - (pre & 15u)) & 15u;
    uint32_t asg_len = 0;
    if (A.with_assignment) {
        const uint32_t nblocks = (A.assign_size + 63u) / 64u;
        asg_len = static_cast<uint32_t>(wv_len(A.population));
        for (uint32_t r = 0; r < A.population; ++r)
            asg_len += static_cast<uint32_t>(wv_len(A.assign_size) + wv_len(nblocks) + wv_len(F.pol[r])) + (nblocks > 1u ? nblocks - 1u : 0u);
    }
    const uint32_t carried = static_cast<uint32_t>(__popc(F.mask));
    F.len = 8u + static_cast<uint64_t>(F.h) + (T - carried) + static_cast<uint64_t>(carried) * (F.some_len + L) + 1u + asg_len;
    return F;
}

// one warp writes frame g at f (its length prefix first); shard j is read from shards + j*plane_stride
__device__ __forceinline__ void frame_write(const PackArgs &A, const FrameLayout &F, uint64_t g, uint32_t data_len, uint32_t L,
                                            const uint8_t *shards, uint8_t *f, uint32_t lane) {
    const uint32_t T = A.d + A.p;
    if (lane == 0u) {                                                            // fixed fields (at most 41 bytes)
        uint32_t w = 8u;
        if (A.kind == SS_FRAME_PEER_ACCEPT) f[w++] = 0;                          // PeerMessage::Msg
        w += wv_put(f + w, A.variant);
        w += wv_put(f + w, __ldg(A.slot + g));
        w += wv_put(f + w, __ldg(A.ballot + g));
        f[w++] = static_cast<uint8_t>(A.d);
        f[w++] = static_cast<uint8_t>(A.p);
        w += wv_put(f + w, data_len);
        w += wv_put(f + w, L);
        wv_put(f + w, T);
    }
    uint32_t at = 8u + F.h;                                                      // running offset inside the frame
    for (uint32_t j = 0; j < T; ++j) {
        if (!((F.mask >> j) & 1u)) {
            if (lane == 0u) f[at] = 0;                                           // None
            at += 1u;
            continue;
        }
        if (lane == 0u) { f[at] = 1; wv_put(f + at + 1u, L); }                   // Some(bytes): tag, length
        at += F.some_len;
        warp_copy_bytes(f + at, shards + static_cast<uint64_t>(j) * A.plane_stride, L, lane);
        at += L;
    }
    if (lane == 0u) f[at] = 0;                                                   // data_copy: None
    at += 1u;
    if (A.with_assignment && lane == 0u) {                                       // assignment: Vec<Bitmap>
        uint32_t w = at;
        w += wv_put(f + w, A.population);
        const uint32_t nblocks = (A.assign_size + 63u) / 64u;
        for (uint32_t r = 0; r < A.population; ++r) {
            w += wv_put(f + w, A.assign_size);
            w += wv_put(f + w, nblocks);
            for (uint32_t b = 0; b < nblocks; ++b) w += wv_put(f + w, b == 0u ? F.pol[r] : 0u);
        }
    }
    const uint64_t body = F.len - 8u;
    if (lane < 8u) f[lane] = static_cast<uint8_t>(body >> (8u * (7u - lane)));
}

__global__ void __launch_bounds__(kWireThreads) frame_pack_kernel(const __grid_constant__ PackArgs A) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = (static_cast<uint64_t>(blockIdx.x) * kWireThreads + threadIdx.x) >> 5;
    const uint64_t nwarps = (static_cast<uint64_t>(gridDim.x) * kWireThreads) >> 5;
    for (uint64_t g = warp; g < A.n; g += nwarps) {
        const FrameLayout F = frame_layout(A, g, A.data_len, A.L);
        // the frame must fit its slot
        if (F.pad + F.len > A.frame_stride) {
            if (lane == 0u) {
                A.frame_off[g] = g * A.frame_stride;
                A.frame_len[g] = 0;                                              // nothing written for this codeword
                atomicOr(A.status, SS_DEV_STATUS_FRAME_OVERFLOW);
            }
            continue;
        }
        frame_write(A, F, g, A.data_len, A.L, A.planes + g * A.shard_stride, A.out + g * A.frame_stride + F.pad, lane);
        if (lane == 0u) {
            A.frame_off[g] = g * A.frame_stride + F.pad;
            A.frame_len[g] = static_cast<uint32_t>(F.len);
        }
    }
}

// ragged, pass 1 (a thread per codeword): each frame's region round_up(pad + len, 16) into frame_off (the scan's input)
// and its length into frame_len; 0 for the frames that are not written
__global__ void __launch_bounds__(kWireThreads) frame_size_ragged_kernel(const __grid_constant__ PackArgs A) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kWireThreads;
    for (uint64_t g = static_cast<uint64_t>(blockIdx.x) * kWireThreads + threadIdx.x; g < A.n; g += stride) {
        const uint32_t len = __ldg(A.lens + g);
        uint64_t region = 0;
        uint32_t flen = 0;
        if (len != 0u && __ldg(A.slot + g) != ~0ull) {
            const FrameLayout F = frame_layout(A, g, len, (len + A.d - 1u) / A.d);
            region = (F.pad + F.len + 15u) & ~15ull;
            flen = static_cast<uint32_t>(F.len);
        }
        A.frame_off[g] = region;
        A.frame_len[g] = flen;
    }
}

// ragged, pass 2 (a warp per codeword): frame_off now holds the region's start
__global__ void __launch_bounds__(kWireThreads) frame_pack_ragged_kernel(const __grid_constant__ PackArgs A) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = (static_cast<uint64_t>(blockIdx.x) * kWireThreads + threadIdx.x) >> 5;
    const uint64_t nwarps = (static_cast<uint64_t>(gridDim.x) * kWireThreads) >> 5;
    bool over = false;
    for (uint64_t g = warp; g < A.n; g += nwarps) {
        if (A.frame_len[g] == 0u) continue;                                      // skipped codeword
        const uint32_t len = __ldg(A.lens + g), L = (len + A.d - 1u) / A.d;
        const FrameLayout F = frame_layout(A, g, len, L);
        const uint64_t off = A.frame_off[g], region = (F.pad + F.len + 15u) & ~15ull;
        __syncwarp();                                                            // every lane has read frame_off / frame_len
        if (off > A.capacity || region > A.capacity - off) {
            over = true;
            if (lane == 0u) A.frame_len[g] = 0;                                  // nothing written for this codeword
            continue;
        }
        frame_write(A, F, g, len, L, A.planes + __ldg(A.shard_off + g), A.out + off + F.pad, lane);
        if (lane == 0u) A.frame_off[g] = off + F.pad;
    }
    if (over && lane == 0u) atomicOr(A.status, SS_DEV_STATUS_FRAME_OVERFLOW);
}

struct ParseArgs {
    const uint8_t *buf;
    uint64_t buf_len;
    const uint64_t *frame_off;
    const uint32_t *frame_group;
    const uint8_t *frame_peer;
    const uint64_t *window_base;    // [G]: absolute slot of window position 0 (start_slot of the group's in-memory log)
    uint64_t n_frames, G;
    uint32_t reply_variant, with_size;
    uint32_t *rec_group;
    uint8_t *rec_slot, *rec_peer;
    uint64_t *rec_ballot;
    uint32_t *rec_kind;
};

// one frame per thread: these frames are a dozen bytes; the work is the varint walk
__global__ void __launch_bounds__(kWireThreads) accept_reply_parse_kernel(const __grid_constant__ ParseArgs A) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kWireThreads;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kWireThreads + threadIdx.x; i < A.n_frames; i += stride) {
        uint32_t kind = SS_FRAME_KIND_MALFORMED;
        uint8_t wslot = 0xff;
        uint64_t ballot = 0;
        const uint32_t grp = A.frame_group[i];
        const uint64_t off = A.frame_off[i];
        do {
            const uint8_t *b;
            uint64_t len, n, v = 0, slot = 0;
            // every variant index is reported as such: no cap
            if (!msg_head(A.buf, A.buf_len, off, A.reply_variant, ~0ull, false, b, len, n, kind)) break;
            if (!wv_next(b, len, n, slot) || !wv_next(b, len, n, ballot)) break;
            if (A.with_size) {                                                        // crossword: size, reply_ts
                if (!wv_next(b, len, n, v) || n >= len) break;
                const uint8_t tag = b[n++];
                if (tag == 1) {
                    if (!wv_next(b, len, n, v) || !wv_next(b, len, n, v)) break;
                } else if (tag != 0) break;
            }
            if (n != len) break;
            kind = A.reply_variant;
            // `slot < start_slot` is ignored by the handler (messages.rs:377); beyond the window cannot be an instance
            if (grp < A.G) {
                const uint64_t base = A.window_base[grp];
                if (slot >= base && slot - base < 64u) wslot = static_cast<uint8_t>(slot - base);
            }
        } while (false);
        A.rec_group[i] = grp;
        A.rec_slot[i] = wslot;                        // 0xff: dropped by the ingest kernel (slot >= 64)
        A.rec_peer[i] = A.frame_peer[i];
        A.rec_ballot[i] = ballot;
        A.rec_kind[i] = kind;
    }
}

struct PrepParseArgs {
    const uint8_t *buf;
    uint64_t buf_len;
    const uint64_t *frame_off;
    uint64_t n_frames;
    uint32_t d, T, reply_variant;
    ss_prepare_reply_rec *rec;
};

// a thread per frame: PrepareReply{slot, trigger_slot, endprep_slot, ballot, voted} (prepare_reply_decode)
__global__ void __launch_bounds__(kWireThreads) prepare_reply_parse_kernel(const __grid_constant__ PrepParseArgs A) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kWireThreads;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kWireThreads + threadIdx.x; i < A.n_frames; i += stride)
        A.rec[i] = prepare_reply_decode(A.buf, A.buf_len, A.frame_off[i], A.d, A.T, A.reply_variant);
}

// newly committed instances -> CommitSlot records (24-byte cells: the record is at most 8 + 1 + 9 bytes)
__global__ void __launch_bounds__(kWireThreads)
wal_commit_pack_kernel(const uint64_t *__restrict__ newly, const uint64_t *__restrict__ window_base, uint64_t G, uint32_t variant,
                       uint8_t *__restrict__ entries, uint32_t *__restrict__ entry_group, uint32_t *__restrict__ entry_len,
                       uint64_t capacity, unsigned long long *counter) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kWireThreads;
    for (uint64_t g = static_cast<uint64_t>(blockIdx.x) * kWireThreads + threadIdx.x; g < G; g += stride) {
        uint64_t w = __ldg(newly + g);
        if (w == 0ull) continue;
        const unsigned long long first = atomicAdd(counter, static_cast<unsigned long long>(__popcll(w)));
        uint64_t e = first;
        while (w) {
            const int s = __ffsll(static_cast<long long>(w)) - 1;
            w &= w - 1ull;
            if (e < capacity) {
                uint8_t *cell = entries + e * 24u;
                int n = 0;
                n += wv_put(cell + 8 + n, variant);
                n += wv_put(cell + 8 + n, window_base[g] + static_cast<uint64_t>(s));
                for (int b = 0; b < 8; ++b) cell[b] = b == 7 ? static_cast<uint8_t>(n) : 0;
                entry_group[e] = static_cast<uint32_t>(g);
                entry_len[e] = static_cast<uint32_t>(8 + n);
            }
            ++e;
        }
    }
}

struct ServeArgs {
    const uint8_t *planes;
    uint64_t plane_stride, shard_stride;
    uint32_t T, L;
    const uint32_t *req_group, *req_held, *req_excl;
    const uint8_t *req_status;
    const uint64_t *reply_off;
    uint64_t n;
    uint32_t *reply_mask;
    uint8_t *out;
};

// a warp per request: reply = held & flip(exclude) when the instance is at least Accepting; the selected shards are
// copied back to back (padded slots) at reply_off[i]
__global__ void __launch_bounds__(kWireThreads) reconstruct_serve_kernel(const __grid_constant__ ServeArgs A) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = (static_cast<uint64_t>(blockIdx.x) * kWireThreads + threadIdx.x) >> 5;
    const uint64_t nwarps = (static_cast<uint64_t>(gridDim.x) * kWireThreads) >> 5;
    const uint32_t all = A.T >= 32u ? 0xffffffffu : ((1u << A.T) - 1u);
    const uint32_t vpc = (A.L + 15u) >> 4;
    for (uint64_t i = warp; i < A.n; i += nwarps) {
        uint32_t m = 0;
        if (A.req_status[i] >= 2u)                                       // Status::Accepting (messages.rs:606-608)
            m = __ldg(A.req_held + i) & ~__ldg(A.req_excl + i) & all;    // subset.flip(); subset_copy(&subset, false)
        if (lane == 0u) A.reply_mask[i] = m;                             // 0: no entry in the reply (:611-613)
        if (m == 0u) continue;
        const uint64_t g = __ldg(A.req_group + i);
        uint8_t *dst = A.out + __ldg(A.reply_off + i);
        uint32_t rem = m;
        while (rem) {
            const uint32_t j = static_cast<uint32_t>(__ffs(rem) - 1);
            rem &= rem - 1u;
            const uint8_t *src = A.planes + static_cast<uint64_t>(j) * A.plane_stride + g * A.shard_stride;
            for (uint32_t v = lane; v < vpc; v += 32u) dev::stg128_cs(dst + v * 16u, dev::ldg128(src + v * 16u));
            dst += static_cast<uint64_t>(vpc) * 16u;
        }
    }
}

}  // namespace ssb

using namespace ssb;

extern "C" {

uint64_t ss_frame_accept_max_len(const ss_frame_spec *s, uint32_t max_shards_per_frame) {
    if (s == nullptr) return 0;
    const uint64_t T = uint64_t(s->data_shards) + s->parity_shards;
    const uint64_t L = s->data_shards ? (uint64_t(s->data_len) + s->data_shards - 1) / s->data_shards : 0;
    uint64_t n = 8 + 44 + T + uint64_t(max_shards_per_frame) * (5 + L) + 1;
    if (s->with_assignment) n += 5 + uint64_t(s->population) * (5 + 5 + 9);
    return (n + 15 + 15) & ~uint64_t(15);            // + the alignment pad, rounded up to the stride granule
}

int ss_frame_accept_pack_dev(ss_ctx *ctx, const ss_frame_spec *s, const uint8_t *shard_planes, uint64_t plane_stride,
                             uint64_t shard_stride, const uint32_t *policies, uint32_t n_policies, const uint8_t *policy_idx,
                             uint32_t peer, const uint64_t *slot, const uint64_t *ballot, uint64_t n, uint8_t *out,
                             uint64_t frame_stride, uint64_t *frame_off, uint32_t *frame_len) {
    if (ctx == nullptr || s == nullptr) return set_error(SS_ERR_INVALID_ARG, "null context or spec");
    SS_TRY(ctx_bind(ctx));
    if (n == 0) return SS_OK;
    if (!shard_planes || !policies || !slot || !ballot || !out || !frame_off || !frame_len) return set_error(SS_ERR_INVALID_ARG, "null buffer");
    const uint32_t T = s->data_shards + s->parity_shards;
    if (s->data_shards == 0 || T > 32) return set_error(SS_ERR_INVALID_ARG, "shard counts must satisfy 1 <= d, d+p <= 32");
    if (s->kind != SS_FRAME_PEER_ACCEPT && s->kind != SS_FRAME_WAL_ACCEPT_DATA) return set_error(SS_ERR_INVALID_ARG, "unknown frame kind %u", s->kind);
    if (s->data_len == 0) return set_error(SS_ERR_INVALID_ARG, "null codeword cannot be framed");
    if (s->population == 0 || s->population > 32 || peer >= s->population || n_policies == 0)
        return set_error(SS_ERR_INVALID_ARG, "bad population / peer / policy table");
    if (s->with_assignment && (s->assign_size == 0 || s->assign_size > 64)) return set_error(SS_ERR_INVALID_ARG, "assignment bitmaps must have 1..64 bits");
    if ((frame_stride & 15u) || ((reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(shard_planes) | plane_stride | shard_stride) & 15u))
        return set_error(SS_ERR_INVALID_ARG, "frame_stride, buffers and strides must be 16-byte aligned");
    PackArgs A;
    A.status = ctx->dev_status;     // a frame that does not fit frame_stride is skipped (frame_len 0) and reported there
    A.planes = shard_planes; A.plane_stride = plane_stride; A.shard_stride = shard_stride;
    A.d = s->data_shards; A.p = s->parity_shards; A.data_len = s->data_len; A.L = (s->data_len + s->data_shards - 1) / s->data_shards;
    A.kind = s->kind; A.variant = s->msg_variant; A.policies = policies; A.policy_idx = policy_idx; A.n_policies = n_policies;
    A.population = s->population; A.peer = peer; A.with_assignment = s->with_assignment; A.assign_size = s->assign_size;
    A.slot = slot; A.ballot = ballot; A.n = n; A.out = out; A.frame_stride = frame_stride; A.frame_off = frame_off; A.frame_len = frame_len;
    if (shard_stride < ((uint64_t(A.L) + 15) & ~uint64_t(15))) return set_error(SS_ERR_INVALID_ARG, "shard_stride shorter than a padded shard");
    frame_pack_kernel<<<launch_grid(ctx, n, kWireThreads / 32), kWireThreads, 0, ctx->stream>>>(A);
    return launched(ctx);
}

int ss_frame_accept_pack_ragged_dev(ss_ctx *ctx, const ss_frame_spec *s, const uint8_t *shard_planes, uint64_t plane_stride,
                                    const uint64_t *shard_off, const uint32_t *data_len, const uint32_t *policies,
                                    uint32_t n_policies, const uint8_t *policy_idx, uint32_t peer, const uint64_t *slot,
                                    const uint64_t *ballot, uint64_t n, uint8_t *out, uint64_t out_capacity,
                                    uint64_t *frame_off, uint32_t *frame_len, uint64_t *total) {
    if (ctx == nullptr || s == nullptr) return set_error(SS_ERR_INVALID_ARG, "null context or spec");
    SS_TRY(ctx_bind(ctx));
    if (n == 0) {
        if (total != nullptr) SS_CUDA(cudaMemsetAsync(total, 0, 8, ctx->stream));
        return SS_OK;
    }
    if (!shard_planes || !shard_off || !data_len || !policies || !slot || !ballot || !out || !frame_off || !frame_len)
        return set_error(SS_ERR_INVALID_ARG, "null buffer");
    const uint32_t T = s->data_shards + s->parity_shards;
    if (s->data_shards == 0 || T > 32) return set_error(SS_ERR_INVALID_ARG, "shard counts must satisfy 1 <= d, d+p <= 32");
    if (s->kind != SS_FRAME_PEER_ACCEPT && s->kind != SS_FRAME_WAL_ACCEPT_DATA) return set_error(SS_ERR_INVALID_ARG, "unknown frame kind %u", s->kind);
    if (s->population == 0 || s->population > 32 || peer >= s->population || n_policies == 0)
        return set_error(SS_ERR_INVALID_ARG, "bad population / peer / policy table");
    if (s->with_assignment && (s->assign_size == 0 || s->assign_size > 64)) return set_error(SS_ERR_INVALID_ARG, "assignment bitmaps must have 1..64 bits");
    if ((reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(shard_planes) | plane_stride) & 15u)
        return set_error(SS_ERR_INVALID_ARG, "buffers and plane_stride must be 16-byte aligned");
    PackArgs A{};
    A.status = ctx->dev_status;
    A.planes = shard_planes; A.plane_stride = plane_stride;
    A.d = s->data_shards; A.p = s->parity_shards;
    A.kind = s->kind; A.variant = s->msg_variant; A.policies = policies; A.policy_idx = policy_idx; A.n_policies = n_policies;
    A.population = s->population; A.peer = peer; A.with_assignment = s->with_assignment; A.assign_size = s->assign_size;
    A.slot = slot; A.ballot = ballot; A.n = n; A.out = out; A.frame_off = frame_off; A.frame_len = frame_len;
    A.shard_off = shard_off; A.lens = data_len; A.capacity = out_capacity;
    void *scr = nullptr;
    SS_TRY(ctx_scratch(ctx, scan_tiles(n) * 8, &scr));
    frame_size_ragged_kernel<<<launch_grid(ctx, n, kWireThreads), kWireThreads, 0, ctx->stream>>>(A);
    SS_TRY(launched(ctx));
    SS_TRY(launch_exclusive_scan_u64(ctx, frame_off, n, static_cast<uint64_t *>(scr), total));
    frame_pack_ragged_kernel<<<launch_grid(ctx, n, kWireThreads / 32), kWireThreads, 0, ctx->stream>>>(A);
    return launched(ctx);
}

int ss_accept_reply_parse_dev(ss_ctx *ctx, const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off, const uint32_t *frame_group,
                              const uint8_t *frame_peer, const uint64_t *window_base, uint64_t n_frames, uint64_t n_groups,
                              uint32_t reply_variant, int with_size, uint32_t *rec_group, uint8_t *rec_slot, uint8_t *rec_peer,
                              uint64_t *rec_ballot, uint32_t *rec_kind) {
    if (ctx == nullptr) return set_error(SS_ERR_INVALID_ARG, "null context");
    SS_TRY(ctx_bind(ctx));
    if (n_frames == 0) return SS_OK;
    if (!buf || !frame_off || !frame_group || !frame_peer || !window_base || !rec_group || !rec_slot || !rec_peer || !rec_ballot || !rec_kind)
        return set_error(SS_ERR_INVALID_ARG, "null buffer");
    ParseArgs A;
    A.buf = buf; A.buf_len = buf_len; A.frame_off = frame_off; A.frame_group = frame_group; A.frame_peer = frame_peer;
    A.window_base = window_base; A.n_frames = n_frames; A.G = n_groups; A.reply_variant = reply_variant; A.with_size = with_size ? 1u : 0u;
    A.rec_group = rec_group; A.rec_slot = rec_slot; A.rec_peer = rec_peer; A.rec_ballot = rec_ballot; A.rec_kind = rec_kind;
    accept_reply_parse_kernel<<<launch_grid(ctx, n_frames, kWireThreads), kWireThreads, 0, ctx->stream>>>(A);
    return launched(ctx);
}

int ss_prepare_reply_parse_dev(ss_ctx *ctx, const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off, uint64_t n_frames,
                               uint32_t data_shards, uint32_t total_shards, uint32_t reply_variant, ss_prepare_reply_rec *rec) {
    if (ctx == nullptr) return set_error(SS_ERR_INVALID_ARG, "null context");
    if (data_shards == 0 || data_shards > total_shards || total_shards > 32)
        return set_error(SS_ERR_INVALID_ARG, "shard counts must satisfy 1 <= d <= T <= 32 (d=%u, T=%u)", data_shards, total_shards);
    SS_TRY(ctx_bind(ctx));
    if (n_frames == 0) return SS_OK;
    if (!buf || !frame_off || !rec) return set_error(SS_ERR_INVALID_ARG, "null buffer");
    PrepParseArgs A;
    A.buf = buf; A.buf_len = buf_len; A.frame_off = frame_off; A.n_frames = n_frames;
    A.d = data_shards; A.T = total_shards; A.reply_variant = reply_variant; A.rec = rec;
    prepare_reply_parse_kernel<<<launch_grid(ctx, n_frames, kWireThreads), kWireThreads, 0, ctx->stream>>>(A);
    return launched(ctx);
}

int ss_wal_commit_pack_dev(ss_ctx *ctx, const uint64_t *newly, const uint64_t *window_base, uint64_t n_groups, uint32_t commit_variant,
                           uint8_t *entries, uint32_t *entry_group, uint32_t *entry_len, uint64_t capacity, uint64_t *n_entries) {
    if (ctx == nullptr) return set_error(SS_ERR_INVALID_ARG, "null context");
    SS_TRY(ctx_bind(ctx));
    if (!newly || !window_base || !entries || !entry_group || !entry_len || !n_entries) return set_error(SS_ERR_INVALID_ARG, "null buffer");
    SS_CUDA(cudaMemsetAsync(n_entries, 0, 8, ctx->stream));
    if (n_groups == 0) return SS_OK;
    wal_commit_pack_kernel<<<launch_grid(ctx, n_groups, kWireThreads), kWireThreads, 0, ctx->stream>>>(
        newly, window_base, n_groups, commit_variant, entries, entry_group, entry_len, capacity, reinterpret_cast<unsigned long long *>(n_entries));
    return launched(ctx);
}

int ss_reconstruct_serve_dev(ss_ctx *ctx, const uint8_t *shard_planes, uint64_t plane_stride, uint64_t shard_stride, uint32_t total_shards,
                             uint32_t shard_len, const uint32_t *req_group, const uint32_t *req_held, const uint32_t *req_excl,
                             const uint8_t *req_status, const uint64_t *reply_off, uint64_t n_requests, uint32_t *reply_mask, uint8_t *out) {
    if (ctx == nullptr) return set_error(SS_ERR_INVALID_ARG, "null context");
    SS_TRY(ctx_bind(ctx));
    if (n_requests == 0) return SS_OK;
    if (!shard_planes || !req_group || !req_held || !req_excl || !req_status || !reply_off || !reply_mask || !out)
        return set_error(SS_ERR_INVALID_ARG, "null buffer");
    if (total_shards == 0 || total_shards > 32 || shard_len == 0) return set_error(SS_ERR_INVALID_ARG, "bad shard geometry");
    if (((reinterpret_cast<uintptr_t>(shard_planes) | reinterpret_cast<uintptr_t>(out) | plane_stride | shard_stride) & 15u) ||
        shard_stride < ((uint64_t(shard_len) + 15) & ~uint64_t(15)))
        return set_error(SS_ERR_INVALID_ARG, "reconstruct serving needs 16-byte aligned, padded shard slots");
    ServeArgs A;
    A.planes = shard_planes; A.plane_stride = plane_stride; A.shard_stride = shard_stride; A.T = total_shards; A.L = shard_len;
    A.req_group = req_group; A.req_held = req_held; A.req_excl = req_excl; A.req_status = req_status; A.reply_off = reply_off;
    A.n = n_requests; A.reply_mask = reply_mask; A.out = out;
    reconstruct_serve_kernel<<<launch_grid(ctx, n_requests, kWireThreads / 32), kWireThreads, 0, ctx->stream>>>(A);
    return launched(ctx);
}

}  // extern "C"
