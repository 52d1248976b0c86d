// exec_walk.cuh -- the execution walk shared by the acceptor (acceptor.cu), the CRaft follower (follower.cu) and the
// CRaft leader (craft_leader.cu): per group, the committed entries from where the last call stopped, as request batch
// records into the caller's buffers, each batch's bytes written by one warp (get_data, rscoding.rs:490-537, 581-683).
//
//   exec_count_kernel<Log>    a thread per group: the entries the walk executes, and their payload bytes
//   (engine.cu's scan)        record indices and payload regions
//   exec_place_kernel<Log>    a thread per group: capacities, the records, the group's bar
//   exec_payload_kernel<Log>  a warp per record: warp_exec_payload with the entry's held mask and the address rule of
//                             its shards, chosen at compile time: by rank (the default), held shard j of rank k (k-th set
//                             bit of held) is at src + k * stride -- the acceptor and the follower keep only their held
//                             shards in padded store slots (stride SS_CW_SLOT_PITCH(L)); by index, shard j is at src +
//                             j * stride -- the leader's planes (stride plane_stride), where a stepped-up leader reserves
//                             a slot for every shard and holds some of them.
//
// A Log policy is a struct of device pointers (with the owner's ring layout), the code's d (the CRaft policies keep it
// beside the ring size W: the kernels load the two as one 64-bit constant), and
//   bool live(g)                          the group is walked
//   Walk start(g)                         what the walk reads once per group, its first slot in .s
//   uint32_t next(w, g, s, &dlen)         at slot s: kExecStop, kExecRun (*dlen = its data_len) or kExecNull
//   void finish(g, s)                     the walk executed up to slot s - 1
//   ExecSrc source(g, slot, dlen)         a record's held mask and shards
//   kTables, kByIndex                     the payload kernel builds the GF(2^8) tables and passes the coder's matrix
//                                         (without them every record must hold its d data shards); the address rule
#pragma once
#include <cstdint>

#include "device_common.cuh"
#include "ss_internal.hpp"
#include "wire_common.cuh"

namespace ssb {

constexpr int kExecThreads = 256;
constexpr int kExecWarps = kExecThreads / 32;
constexpr int kChunk = 4;           // sources per Horner pass: their loads are issued together

struct ExecShared {
    uint8_t exp[512], log[256];
    uint8_t a[kExecWarps][32][32];  // Gauss-Jordan: lane r owns row r of M[sources] ...
    uint8_t inv[kExecWarps][32][32];   // ... and of the identity it turns into the inverse
    uint8_t piv[kExecWarps][32];    // piv[c]: the row that took column c as its pivot
};

__device__ __forceinline__ uint32_t gmul(const ExecShared &S, uint32_t a, uint32_t b) {
    return (a != 0u && b != 0u) ? S.exp[S.log[a] + S.log[b]] : 0u;
}

// x * 2 in GF(2^8) on 16 packed bytes
__device__ __forceinline__ uint4 xtime16(uint4 v) {
    return make_uint4(dev::xtime4(v.x), dev::xtime4(v.y), dev::xtime4(v.z), dev::xtime4(v.w));
}

// v moved up by k (1..15) byte positions: bytes [16-k, 32-k) of the 32-byte window {0, v}
__device__ __forceinline__ uint4 shift_up(const uint4 &v, uint32_t k) { return dev::funnel16(make_uint4(0u, 0u, 0u, 0u), v, 16u - k); }

// the GF(2^8) exp / log tables of the CTA (blockDim.x == kExecThreads); ends with __syncthreads
__device__ __forceinline__ void exec_tables_init(ExecShared &S) {
    for (uint32_t i = threadIdx.x; i < 256u; i += kExecThreads) {
        uint32_t v = 1u;
        for (uint32_t k = 0; k < i; ++k) v = (v << 1) ^ ((v & 0x80u) ? 0x11Du : 0u);   // 2^i, i < 255
        if (i < 255u) { S.exp[i] = static_cast<uint8_t>(v); S.exp[i + 255u] = static_cast<uint8_t>(v); S.log[v] = static_cast<uint8_t>(i); }
    }
    if (threadIdx.x < 2u) S.exp[510u + threadIdx.x] = S.exp[threadIdx.x];
    __syncthreads();
}

// Output-stationary: lane v writes payload bytes [16v, 16v + 16) of dst with one aligned 128-bit store (zero past dlen).
// Data shard i is payload bytes [i*L, (i+1)*L); a held one is read at src + rank(i)*stride (kByIndex: src + i*stride),
// a missing one is the
// GF(2^8) combination of the first d held shards (ranks 0..d-1) with row i of inverse(M[sources]), reconstruct_data's
// choice of sources (rscoding.rs:490-537).  matrix: the coder's [T*d] coding matrix; held has at least d bits below T.
// Ends with __syncwarp: the warp's next record may overwrite the rows this one read.
template <bool kByIndex = false>
__device__ __forceinline__ void warp_exec_payload(ExecShared &S, uint32_t w, uint32_t lane, uint32_t d, uint32_t held, uint32_t dlen,
                                                  const uint8_t *matrix, const uint8_t *src, uint64_t stride, uint8_t *dst) {
    uint8_t (*ra)[32] = S.a[w];
    uint8_t (*ri)[32] = S.inv[w];
    uint8_t *piv = S.piv[w];
    const uint32_t L = (dlen + d - 1u) / d;
    const uint32_t dmask = d == 32u ? 0xffffffffu : (1u << d) - 1u;
    const uint32_t missing = ~held & dmask;
    if (missing != 0u) {
        // Gauss-Jordan on M[sources] (d x d, invertible for any d distinct rows of the coder's matrix): lane k owns
        // row k, whose source is the k-th held shard; pivots are taken in column order, rows are never swapped
        if (lane < d) {
            uint32_t h = held;
            for (uint32_t q = 0; q < lane; ++q) h &= h - 1u;
            const uint32_t row = static_cast<uint32_t>(__ffs(h)) - 1u;
            for (uint32_t c = 0; c < d; ++c) {
                ra[lane][c] = matrix[row * d + c];
                ri[lane][c] = c == lane ? 1u : 0u;
            }
        }
        __syncwarp();
        uint32_t used = 0u;
        for (uint32_t c = 0; c < d; ++c) {
            const uint32_t f = lane < d ? ra[lane][c] : 0u;
            const uint32_t cand = __ballot_sync(0xffffffffu, f != 0u && !((used >> lane) & 1u));
            if (cand == 0u) break;
            const uint32_t p = static_cast<uint32_t>(__ffs(cand)) - 1u;
            used |= 1u << p;
            if (lane == p) {
                const uint32_t sc = S.exp[255u - S.log[f]];
                piv[c] = static_cast<uint8_t>(p);
                for (uint32_t k = c; k < d; ++k) ra[p][k] = static_cast<uint8_t>(gmul(S, ra[p][k], sc));
                for (uint32_t k = 0; k < d; ++k) ri[p][k] = static_cast<uint8_t>(gmul(S, ri[p][k], sc));
            }
            __syncwarp();
            if (lane < d && lane != p && f != 0u) {
                for (uint32_t k = c; k < d; ++k) ra[lane][k] ^= static_cast<uint8_t>(gmul(S, f, ra[p][k]));
                for (uint32_t k = 0; k < d; ++k) ri[lane][k] ^= static_cast<uint8_t>(gmul(S, f, ri[p][k]));
            }
            __syncwarp();
        }
    }
    // bytes [o, o + c) of data shard i (c <= 16) as the low c bytes of a uint4, the rest zero
    auto shard16 = [&](uint32_t i, uint32_t o, int c) -> uint4 {
        if ((held >> i) & 1u) {
            if (kByIndex) return dev::load16(src + i * stride + o, c);
            return dev::load16(src + __popc(held & ((1u << i) - 1u)) * stride + o, c);
        }
        const uint8_t *coef = ri[piv[i]];
        uint4 acc = make_uint4(0u, 0u, 0u, 0u);
        uint32_t rest = held;                                          // kByIndex: the held shards not yet a source
        for (uint32_t q0 = 0; q0 < d; q0 += kChunk) {
            uint32_t cq[kChunk], top = 0u;
            dev::Raw16 raw[kChunk];
#pragma unroll
            for (int q = 0; q < kChunk; ++q) {
                const bool in = q0 + q < d;
                cq[q] = in ? coef[q0 + q] : 0u;
                top |= cq[q];
                uint32_t at = q0 + q;                                  // source q0 + q
                if (kByIndex) {
                    at = in ? static_cast<uint32_t>(__ffs(static_cast<int>(rest))) - 1u : 0u;
                    if (in) rest &= rest - 1u;
                }
                raw[q] = dev::raw16_issue(src + at * stride + o, in && cq[q] != 0u ? c : 0);
            }
            uint4 x[kChunk];
#pragma unroll
            for (int q = 0; q < kChunk; ++q) x[q] = dev::raw16_finish(raw[q], c);
            // Horner from the top coefficient bit down: part = part * 2 ^ (XOR of the x_q whose c_q has bit k)
            uint4 part = make_uint4(0u, 0u, 0u, 0u);
            for (int k = top == 0u ? -1 : 31 - __clz(top); k >= 0; --k) {
                part = xtime16(part);
#pragma unroll
                for (int q = 0; q < kChunk; ++q) {
                    const uint32_t m = 0u - ((cq[q] >> k) & 1u);
                    part.x ^= x[q].x & m; part.y ^= x[q].y & m; part.z ^= x[q].z & m; part.w ^= x[q].w & m;
                }
            }
            acc.x ^= part.x; acc.y ^= part.y; acc.z ^= part.z; acc.w ^= part.w;
        }
        return acc;
    };
    const uint32_t ncol = (dlen + 15u) >> 4;
    for (uint32_t v = lane; v < ncol; v += 32u) {
        uint32_t pos = v * 16u;
        const uint32_t end = dlen - pos < 16u ? dlen : pos + 16u;
        const uint32_t i = pos / L, o = pos - i * L;
        uint4 out;
        if (o + 16u <= L) {
            out = shard16(i, o, static_cast<int>(end - pos));           // the column lies in one shard
        } else {                                                       // it spans shards (always for L < 16)
            out = make_uint4(0u, 0u, 0u, 0u);
            for (uint32_t filled = 0u; pos < end;) {
                const uint32_t j = pos / L, oj = pos - j * L;
                const uint32_t c = L - oj < end - pos ? L - oj : end - pos;
                uint4 piece = shard16(j, oj, static_cast<int>(c));
                if (filled != 0u) piece = shift_up(piece, filled);
                out.x |= piece.x; out.y |= piece.y; out.z |= piece.z; out.w |= piece.w;
                filled += c;
                pos += c;
            }
        }
        dev::stg128_cs(dst + static_cast<uint64_t>(v) * 16u, out);
    }
    __syncwarp();                       // the next record's Gauss-Jordan overwrites the rows this one read
}

// ---- the walk ------------------------------------------------------------------------------------------------------
enum : uint32_t { kExecStop = 0u, kExecRun = 1u, kExecNull = 2u };

// what every walk writes, its scratch, and the coder's matrix
struct ExecOut {
    const uint8_t *matrix;          // [T*d]
    uint64_t *cnt, *bytes;          // [G] per group: records, payload bytes; then their exclusive scans
    uint64_t *n_exec;               // records written (a prefix: the offsets are monotone)
    uint8_t *out;
    uint64_t out_cap;
    uint32_t *rec_group;
    uint64_t *rec_slot, *rec_off;
    uint32_t *rec_len;
    uint64_t rec_cap;
    uint32_t *status;
};

template <class Log>
struct ExecArgs {
    uint64_t G;
    Log log;
    ExecOut o;
};

// a record's shards: held mask, shard 0's address, the stride warp_exec_payload steps by
struct ExecSrc {
    uint32_t held;
    const uint8_t *base;
    uint64_t stride;
};

template <class Log>
__global__ void __launch_bounds__(kExecThreads) exec_count_kernel(const __grid_constant__ ExecArgs<Log> A) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kExecThreads;
    for (uint64_t g = static_cast<uint64_t>(blockIdx.x) * kExecThreads + threadIdx.x; g < A.G; g += stride) {
        uint64_t n = 0u, b = 0u;
        uint32_t dl = 0u;
        if (A.log.live(g)) {
            const typename Log::Walk w = A.log.start(g);
            for (uint64_t s = w.s; A.log.next(w, g, s, &dl) == kExecRun; ++s, ++n) b += round16(dl);
        }
        A.o.cnt[g] = n;
        A.o.bytes[g] = b;
    }
}

template <class Log>
__global__ void __launch_bounds__(kExecThreads) exec_place_kernel(const __grid_constant__ ExecArgs<Log> A) {
    const ExecOut &o = A.o;
    bool full = false, null_ent = false;
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kExecThreads;
    for (uint64_t g = static_cast<uint64_t>(blockIdx.x) * kExecThreads + threadIdx.x; g < A.G; g += stride) {
        if (!A.log.live(g)) continue;
        const typename Log::Walk w = A.log.start(g);
        uint64_t ro = o.cnt[g], bo = o.bytes[g], s = w.s;
        uint32_t dl = 0u, r;
        while ((r = A.log.next(w, g, s, &dl)) == kExecRun) {
            const uint64_t sz = round16(dl);
            if (ro >= o.rec_cap || bo > o.out_cap || sz > o.out_cap - bo) { full = true; break; }
            o.rec_group[ro] = static_cast<uint32_t>(g);
            o.rec_slot[ro] = s;
            o.rec_off[ro] = bo;
            o.rec_len[ro] = dl;
            ++ro;
            bo += sz;
            ++s;
        }
        null_ent |= r == kExecNull;
        if (s != w.s) {
            A.log.finish(g, s);
            atomicMax(reinterpret_cast<unsigned long long *>(o.n_exec), static_cast<unsigned long long>(ro));
        }
    }
    if (full) atomicOr(o.status, SS_DEV_STATUS_EXEC_FULL);
    if (null_ent) atomicOr(o.status, SS_DEV_STATUS_EXEC_NULL);
}

template <class Log>
__global__ void __launch_bounds__(kExecThreads) exec_payload_kernel(const __grid_constant__ ExecArgs<Log> A) {
    __shared__ ExecShared S;
    if (Log::kTables) exec_tables_init(S);
    const uint32_t lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
    const uint64_t n = *A.o.n_exec;
    const uint64_t nwarps = static_cast<uint64_t>(gridDim.x) * kExecWarps;
    for (uint64_t r = static_cast<uint64_t>(blockIdx.x) * kExecWarps + w; r < n; r += nwarps) {
        const uint32_t dlen = A.o.rec_len[r];
        const ExecSrc src = A.log.source(A.o.rec_group[r], A.o.rec_slot[r], dlen);
        warp_exec_payload<Log::kByIndex>(S, w, lane, A.log.d, src.held, dlen, Log::kTables ? A.o.matrix : nullptr, src.base, src.stride,
                                         A.o.out + A.o.rec_off[r]);
    }
}

// One execution call: count and place walk the groups with `log`, the payload warps read the shards through `src` (the
// same policy but for the CRaft leader, whose walk and shard layout vary apart).  The payload grid has a warp per entry
// the ring can hold (ring_entries), up to the grid cap; warps past the executed count return at once.  partials: the
// scans' scratch; totals: the sums of the record counts and payload bytes.
template <class Log, class Src>
int launch_execute(ss_ctx *ctx, const ExecOut &o, const Log &log, const Src &src, uint64_t groups, uint64_t ring_entries,
                   uint64_t *partials, uint64_t *totals) {
    const ExecArgs<Log> A{groups, log, o};
    const uint32_t grid = launch_grid(ctx, groups, kExecThreads);
    SS_CUDA(cudaMemsetAsync(o.n_exec, 0, 8, ctx->stream));
    exec_count_kernel<Log><<<grid, kExecThreads, 0, ctx->stream>>>(A);
    SS_TRY(launched(ctx));
    SS_TRY(launch_exclusive_scan_u64(ctx, o.cnt, groups, partials, totals));
    SS_TRY(launch_exclusive_scan_u64(ctx, o.bytes, groups, partials, totals + 1));
    exec_place_kernel<Log><<<grid, kExecThreads, 0, ctx->stream>>>(A);
    SS_TRY(launched(ctx));
    exec_payload_kernel<Src><<<launch_grid(ctx, ring_entries, kExecWarps), kExecThreads, 0, ctx->stream>>>(ExecArgs<Src>{groups, src, o});
    return launched(ctx);
}

}  // namespace ssb
