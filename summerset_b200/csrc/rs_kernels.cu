// rs_kernels.cu -- Reed-Solomon GF(2^8) shard encode / reconstruct kernels for sm_90a.
//
// What they replace (reference, josehu07/summerset @ 1daf80aa):
//   RSCodeword::from_data split + compute_parity  src/utils/rscoding.rs:165-243,447-486
//     -> crate ReedSolomon::encode (rscoding.rs:484): parity_j = sum_i M[d+j][i] * data_i
//   RSCodeword::reconstruct_data / reconstruct_all src/utils/rscoding.rs:490-537
//     -> crate ReedSolomon::reconstruct{,_data} (rscoding.rs:515,517)
// executed for millions of codewords per launch instead of one per event-loop turn
// (rspaxos/request.rs:72-77, crossword/request.rs:82-87, rspaxos/durability.rs:146-159).
//
// This is HBM-bound byte work: no tensor cores.  Design points:
//   * a thread owns 16-byte "columns" of a codeword: it reads the 16 bytes at the same offset of each of the d source
//     shards (128-bit loads; the shards of a contiguous split are generally misaligned w.r.t. 16 bytes: two aligned
//     loads + a byte funnel shift, the second load being an L1 hit on the neighbour lane's sectors) and writes 16
//     bytes of each output shard with one 128-bit streaming store;
//   * GF multiplication works on four packed field elements per 32-bit register with prmt / lop3 / imad only -- no
//     table, no shared-memory gathers.  Every product is a Horner evaluation in x over the coefficient bits:
//       - RS(3,2), the code of every 5-replica RSPaxos / Crossword / CRaft deployment, is specialised with its
//         coefficients folded in: parity0 = a^b^c, parity1 = (((a^b)*x ^ (a^c))*x ^ (a^c))*x ^ a;
//       - other codes with d <= 8 and all reconstructions use run-time coefficient programs (one per erasure
//         pattern, built on the host at coder creation): per bit level one packed xtime of the accumulator and one
//         lop3 per source.  d > 8 falls back to the bit-plane form (sources expanded into byte masks).
//   * kernels, by geometry:
//       rs32_encode_row_kernel            uniform codewords up to 256 columns, 16-byte-aligned stride: a CTA walks
//                                         codewords, thread = column, kernel-uniform funnel, masked tail handled by
//                                         whichever warp has the last column block this iteration (rotating), the
//                                         fused tally (after the codeword when the planes are local, else as a
//                                         coalesced prologue), optional stores into peer GPUs
//       rs32_accept_bulk_kernel           the same geometry when the parity goes to local planes (the accept step):
//                                         payload rows staged in shared memory by bulk async copies, parity rows
//                                         written back with bulk stores, tally by a warp of its own
//       rs32_encode_uniform_kernel        any uniform geometry: flat thread <-> column index, general masked loads
//       rs32_encode_ragged_kernel         ragged batches: a warp per codeword, two columns per lane on long ones
//       rs32_crossword_distribute_kernel  ragged encode + per-replica shard placement (config 4)
//       horner_* / generic_*              other codes; rs_reconstruct_small_kernel / horner_reconstruct_kernel
#include <cstring>

#include "device_common.cuh"
#include "ss_internal.hpp"
#include "static_codes.hpp"
#include "rs32_decode.cuh"
#include "horner_row_kernels.cuh"

namespace ssb {

using dev::funnel16;
using dev::keep_bytes;
using dev::load16;
using dev::msb_mask;
using dev::store16;
using dev::xtime4;

constexpr int kThreads = 256;

// ------------------------------------------------------------------------------------------------
// compute cores
// ------------------------------------------------------------------------------------------------

// RS(3,2): parity rows {01 01 01}, {0f 08 06} (checked on the host against the coder's matrix).
__device__ __forceinline__ void rs32_word(uint32_t a, uint32_t b, uint32_t c, uint32_t &p0,
                                          uint32_t &p1) {
    const uint32_t t = a ^ b;
    const uint32_t u = a ^ c;
    p0 = t ^ c;
    uint32_t r = xtime4(t) ^ u;
    r = xtime4(r) ^ u;
    p1 = xtime4(r) ^ a;
}

__device__ __forceinline__ void rs32_column(const uint8_t *src, uint32_t len, uint32_t L, uint32_t k,
                                            uint8_t *out, uint64_t plane_stride, bool padded, bool emit_data) {
    const int64_t rem = static_cast<int64_t>(len) - static_cast<int64_t>(k);
    auto nv = [](int64_t r) { return r > 16 ? 16 : (r < 0 ? 0 : static_cast<int>(r)); };
    // all loads issued before any of the data is touched
    const dev::Raw16 ra = dev::raw16_issue(src + k, nv(rem));
    const dev::Raw16 rb = dev::raw16_issue(src + static_cast<uint64_t>(L) + k, nv(rem - L));
    const dev::Raw16 rc = dev::raw16_issue(src + 2ull * L + k, nv(rem - 2ll * L));
    const uint4 a = dev::raw16_finish(ra, nv(rem));
    const uint4 b = dev::raw16_finish(rb, nv(rem - L));
    const uint4 c = dev::raw16_finish(rc, nv(rem - 2ll * L));
    uint4 p0, p1;
    rs32_word(a.x, b.x, c.x, p0.x, p1.x);
    rs32_word(a.y, b.y, c.y, p0.y, p1.y);
    rs32_word(a.z, b.z, c.z, p0.z, p1.z);
    rs32_word(a.w, b.w, c.w, p0.w, p1.w);
    const int onv = static_cast<int>(L - k) > 16 ? 16 : static_cast<int>(L - k);
    store16(out + k, p0, onv, padded);
    store16(out + plane_stride + k, p1, onv, padded);
    if (emit_data) {   // data shards copied into planes 0..2 of the shard store (pack-for-send, rscoding.rs:255-293)
        store16(out - 3 * plane_stride + k, a, onv, padded);
        store16(out - 2 * plane_stride + k, b, onv, padded);
        store16(out - 1 * plane_stride + k, c, onv, padded);
    }
}

// Generic bit-plane core: acc[j] ^= sum over bits k of (mask_k(x_i) & splat(c_ji * 2^k)).
template <int P>
__device__ __forceinline__ void bitplane_accumulate(const uint4 &x, const uint32_t *__restrict__ splat_i,
                                                    int d, int n_out, uint4 (&acc)[P]) {
    // splat_i points at splat[(0*d + i)*8]; output j is at + j*d*8
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int sh = 7 - k;
        const uint4 m = make_uint4(msb_mask(x.x << sh), msb_mask(x.y << sh), msb_mask(x.z << sh),
                                   msb_mask(x.w << sh));
#pragma unroll
        for (int j = 0; j < P; ++j) {
            if (j < n_out) {
                const uint32_t c = __ldg(splat_i + j * d * 8 + k);
                acc[j].x ^= m.x & c;
                acc[j].y ^= m.y & c;
                acc[j].z ^= m.z & c;
                acc[j].w ^= m.w & c;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// encode kernels
// ------------------------------------------------------------------------------------------------
struct EncUniform {
    const uint8_t *data;
    uint64_t data_stride;
    uint32_t len, L, vpc;
    uint8_t *parity;
    uint64_t plane_stride, shard_stride;
    uint64_t n;
    uint32_t total;   // n * vpc (host guarantees it fits 32 bits per launch)
    uint32_t padded;  // bit0: SS_RS_OUT_PADDED16, bit1: SS_RS_EMIT_DATA
    // fused tally (planes == nullptr: none)
    const uint64_t *planes;
    uint32_t R, threshold;
    uint64_t G;
    uint64_t *committed;
    uint32_t *commit_bar;
};

__global__ void __launch_bounds__(kThreads) rs32_encode_uniform_kernel(const __grid_constant__ EncUniform P) {
    const uint32_t t = blockIdx.x * kThreads + threadIdx.x;
    if (P.planes != nullptr && t < P.G) {
        const uint64_t w = dev::tally_word(P.planes, P.R, P.G, t, P.threshold);
        P.committed[t] = w;
        if (P.commit_bar != nullptr) P.commit_bar[t] = dev::commit_prefix(w);
    }
    if (t >= P.total) return;
    const uint32_t g = t / P.vpc;
    const uint32_t k = (t - g * P.vpc) * 16u;
    rs32_column(P.data + static_cast<uint64_t>(g) * P.data_stride, P.len, P.L, k,
                P.parity + static_cast<uint64_t>(g) * P.shard_stride, P.plane_stride, (P.padded & 1u) != 0u,
                (P.padded & 2u) != 0u);
}


// ------------------------------------------------------------------------------------------------
// RS(3,2) "row" kernel for uniform geometry (the BASELINE config-3 hot kernel)
// ------------------------------------------------------------------------------------------------
// A CTA of round_up(vpc,32) threads walks codewords g = blockIdx.x, + gridDim.x, ...; thread v owns
// column v of every codeword it visits, so there is no per-thread index division and all address
// arithmetic is a per-iteration pointer bump.  With a 16-byte-aligned payload stride the misalignment of
// shard 1 and shard 2 w.r.t. 16 bytes is the same for every codeword: the byte funnel (prmt selector and
// word offset) is kernel-uniform, hoisted out of the loop, and its branches are uniform.  Only the last
// column(s) of a codeword (partial output vector / zero-padded payload tail) take the masked general path.
// Lanes beyond vpc in the last warp would idle; lane vpc tallies the group's 64-slot ack window instead.
struct Enc32Row {
    const uint8_t *data;
    uint64_t data_stride;
    uint8_t *plane[5];        // base of shard plane j (local memory, or a peer GPU's memory mapped over NVLink);
                              // planes 0..2 (data shards) are only written when emit_data is set
    uint64_t shard_stride;
    uint32_t n, len, L, vpc;
    uint32_t fast_cols;       // columns [0, fast_cols) need no masking
    uint32_t s1, s2;          // (L & 15), (2L & 15): misalignment of shards 1 and 2
    uint32_t emit_data;
    uint32_t chunk;           // 0: codewords g = blockIdx.x + i*gridDim.x ; else CTA b owns [b*chunk, (b+1)*chunk)
    uint32_t st_mode;         // cache operator of the plane stores in replicate mode (tuning)
    uint32_t rotate;          // 1: rotate the warp -> column-block assignment per codeword (default)
    uint32_t tally_last;      // 1: the fused tally runs after the CTA's encode loop instead of before it
    const uint64_t *planes;   // fused tally (nullptr: none); G == n
    uint32_t R, threshold;
    uint64_t *committed;
    uint32_t *commit_bar;
    dev::FlagWait wait;       // replicate mode: every CTA first waits for the followers' ack flags (flags == nullptr: no wait)
};

// one Horner step r*x ^ u on four packed field elements: shift on the FMA pipe (imad), then
// prmt (sign mask) + two lop3 on the ALU pipe.
__device__ __forceinline__ uint32_t horner_step(uint32_t r, uint32_t u) {
    const uint32_t m = msb_mask(r);
    const uint32_t r2 = r * 2u;
    const uint32_t t = (r2 & 0xfefefefeu) ^ u;
    return t ^ (m & 0x1d1d1d1du);
}
__device__ __forceinline__ void rs32_word_fast(uint32_t a, uint32_t b, uint32_t c, uint32_t &p0, uint32_t &p1) {
    const uint32_t t = a ^ b;
    const uint32_t u = a ^ c;
    p0 = a ^ b ^ c;
    uint32_t r = horner_step(t, u);
    r = horner_step(r, u);
    p1 = horner_step(r, a);
}

// one column of the row kernel.  MASKED: this warp owns the codeword's last column(s): inputs past data_len
// are zeroed, outputs past L are zeroed, and a second aligned load is issued only when it holds a valid byte.
template <bool EMIT, bool MASKED, bool PF = false>
__device__ __forceinline__ void rs32_row_column(const uint8_t *__restrict__ src, uint8_t *const (&out)[5],
                                                uint32_t k, uint32_t o1, uint32_t o2,
                                                uint32_t s0, uint32_t s1, uint32_t s2, int nva, int nvb, int nvc,
                                                int onv, uint32_t st_mode = 0u) {
    // `src` is the 16-byte-aligned address at or below the payload (payload = src + s0); o1/o2 are aligned
    // offsets from src.  Loads first (pairs adjacent so the second one hits the sectors the first just
    // brought into L1), then the byte funnels.  PF: the loads carry the L2 256-byte prefetch hint.
    auto ldg = [](const uint8_t *q) { return PF ? dev::ldg128_pf256(q) : dev::ldg128(q); };
    const uint4 a0 = ldg(src + k);
    // the second-load registers start as zeros, never as a copy of the first load: a copy would be issued right
    // behind the load and stall every later load of this column until that one has landed
    uint4 a1 = make_uint4(0u, 0u, 0u, 0u);
    if (s0 != 0u && (!MASKED || static_cast<int>(s0) + nva > 16)) a1 = ldg(src + k + 16u);
    uint4 b0 = make_uint4(0u, 0u, 0u, 0u);
    if (!MASKED || nvb > 0) b0 = ldg(src + o1);   // a window entirely in the zero padding is never read
    uint4 b1 = make_uint4(0u, 0u, 0u, 0u);
    if (s1 != 0u && (!MASKED || static_cast<int>(s1) + nvb > 16)) b1 = ldg(src + o1 + 16u);
    uint4 c0 = make_uint4(0u, 0u, 0u, 0u);
    if (!MASKED || nvc > 0) c0 = ldg(src + o2);
    uint4 c1 = make_uint4(0u, 0u, 0u, 0u);
    if (s2 != 0u && (!MASKED || static_cast<int>(s2) + nvc > 16)) c1 = ldg(src + o2 + 16u);
    uint4 a = s0 != 0u ? funnel16(a0, a1, s0) : a0;
    uint4 b = s1 != 0u ? funnel16(b0, b1, s1) : b0;
    uint4 c = s2 != 0u ? funnel16(c0, c1, s2) : c0;
    if (MASKED) {
        a = keep_bytes(a, nva);
        b = keep_bytes(b, nvb);
        c = keep_bytes(c, nvc);
    }
    uint4 p0, p1;
    rs32_word_fast(a.x, b.x, c.x, p0.x, p1.x);
    rs32_word_fast(a.y, b.y, c.y, p0.y, p1.y);
    rs32_word_fast(a.z, b.z, c.z, p0.z, p1.z);
    rs32_word_fast(a.w, b.w, c.w, p0.w, p1.w);
    if (MASKED) {
        p0 = keep_bytes(p0, onv);
        p1 = keep_bytes(p1, onv);
    }
    if (EMIT) {   // all five planes (possibly peer memory): data shards too -- the pack-for-send of subset_copy
        dev::stg128_mode(out[3] + k, p0, st_mode);
        dev::stg128_mode(out[4] + k, p1, st_mode);
        dev::stg128_mode(out[0] + k, MASKED ? keep_bytes(a, onv) : a, st_mode);
        dev::stg128_mode(out[1] + k, MASKED ? keep_bytes(b, onv) : b, st_mode);
        dev::stg128_mode(out[2] + k, MASKED ? keep_bytes(c, onv) : c, st_mode);
    } else {
        dev::stg128_cs(out[3] + k, p0);
        dev::stg128_cs(out[4] + k, p1);
    }
}

// two unmasked columns (k and k + 512 bytes) of one codeword with all ten loads in flight before any compute:
// doubles the memory-level parallelism of a warp that walks a long codeword alone (ragged geometry)
__device__ __forceinline__ void rs32_row_pair(const uint8_t *__restrict__ src, uint8_t *out3, uint8_t *out4, uint32_t k,
                                              uint32_t o1, uint32_t o2, uint32_t s0, uint32_t s1, uint32_t s2) {
    const uint32_t D2 = 512u;
    const uint4 a0 = dev::ldg128(src + k), A0 = dev::ldg128(src + k + D2);
    uint4 a1 = make_uint4(0u, 0u, 0u, 0u), A1 = a1;      // zeros, not copies of the loads (see rs32_row_column)
    if (s0 != 0u) { a1 = dev::ldg128(src + k + 16u); A1 = dev::ldg128(src + k + D2 + 16u); }
    const uint4 b0 = dev::ldg128(src + o1), B0 = dev::ldg128(src + o1 + D2);
    uint4 b1 = make_uint4(0u, 0u, 0u, 0u), B1 = b1;
    if (s1 != 0u) { b1 = dev::ldg128(src + o1 + 16u); B1 = dev::ldg128(src + o1 + D2 + 16u); }
    const uint4 c0 = dev::ldg128(src + o2), C0 = dev::ldg128(src + o2 + D2);
    uint4 c1 = make_uint4(0u, 0u, 0u, 0u), C1 = c1;
    if (s2 != 0u) { c1 = dev::ldg128(src + o2 + 16u); C1 = dev::ldg128(src + o2 + D2 + 16u); }
    {
        const uint4 a = s0 != 0u ? funnel16(a0, a1, s0) : a0;
        const uint4 b = s1 != 0u ? funnel16(b0, b1, s1) : b0;
        const uint4 c = s2 != 0u ? funnel16(c0, c1, s2) : c0;
        uint4 p0, p1;
        rs32_word_fast(a.x, b.x, c.x, p0.x, p1.x);
        rs32_word_fast(a.y, b.y, c.y, p0.y, p1.y);
        rs32_word_fast(a.z, b.z, c.z, p0.z, p1.z);
        rs32_word_fast(a.w, b.w, c.w, p0.w, p1.w);
        dev::stg128_cs(out3 + k, p0);
        dev::stg128_cs(out4 + k, p1);
    }
    {
        const uint4 a = s0 != 0u ? funnel16(A0, A1, s0) : A0;
        const uint4 b = s1 != 0u ? funnel16(B0, B1, s1) : B0;
        const uint4 c = s2 != 0u ? funnel16(C0, C1, s2) : C0;
        uint4 p0, p1;
        rs32_word_fast(a.x, b.x, c.x, p0.x, p1.x);
        rs32_word_fast(a.y, b.y, c.y, p0.y, p1.y);
        rs32_word_fast(a.z, b.z, c.z, p0.z, p1.z);
        rs32_word_fast(a.w, b.w, c.w, p0.w, p1.w);
        dev::stg128_cs(out3 + k + D2, p0);
        dev::stg128_cs(out4 + k + D2, p1);
    }
}

template <bool EMIT, int MAXT, int MINB, bool SEG = false, bool PF = false>
__global__ void __launch_bounds__(MAXT, MINB) rs32_encode_row_kernel(const __grid_constant__ Enc32Row P) {
    const uint32_t lane = threadIdx.x & 31u, wid = threadIdx.x >> 5, nblk = blockDim.x >> 5;
    const uint32_t s1 = P.s1, s2 = P.s2;
    auto clamp16 = [](int64_t r) { return r > 16 ? 16 : (r < 0 ? 0 : static_cast<int>(r)); };

    // replicate mode only: the ack planes tallied below are written by peer GPUs; wait for their step flags
    if constexpr (EMIT) dev::cta_wait_flags(P.wait);

    // ---- fused tally: this CTA's contiguous slice of groups, coalesced (one pass, before the encode loop, or after
    //      it when tally_last is set) ----
    auto tally = [&] {
        if (P.planes == nullptr) return;
        const uint32_t per = (P.n + gridDim.x - 1) / gridDim.x;
        const uint32_t lo = blockIdx.x * per;
        const uint32_t hi = lo + per < P.n ? lo + per : P.n;
        for (uint32_t g = lo + threadIdx.x; g < hi; g += blockDim.x) {
            const uint64_t w = dev::tally_word(P.planes, P.R, P.n, g, P.threshold);
            P.committed[g] = w;
            if (P.commit_bar != nullptr) P.commit_bar[g] = dev::commit_prefix(w);
        }
    };
    if (!P.tally_last) tally();

    // The CTA's warps work on the same codeword, each on one 32-column block.  The block that holds the codeword's
    // last column runs the (longer) masked variant; with a fixed warp->block assignment that warp is the CTA's
    // critical path and the other warps idle at the end (measured: 10 % of the whole kernel).  So the assignment
    // ROTATES: on its i-th codeword warp w takes block (w + i) mod nblk, and every warp does every block type
    // equally often.
    if constexpr (SEG) {
        // Codewords wider than the CTA (more than 256 columns: payloads above 12 KB, up to one multi-megabyte codeword):
        // the work items are (codeword, 256-column segment) pairs, so that a single large codeword still fills the GPU
        // (benches/rse_bench.rs sizes 16 KB .. 4 MB).
        const uint32_t nseg = (P.vpc + blockDim.x - 1u) / blockDim.x;
        const uint64_t items = static_cast<uint64_t>(P.n) * nseg;
#pragma unroll 1
        for (uint64_t it = blockIdx.x; it < items; it += gridDim.x) {
            const uint32_t g = static_cast<uint32_t>(it / nseg), seg = static_cast<uint32_t>(it - static_cast<uint64_t>(g) * nseg);
            const uint32_t vb = seg * blockDim.x + wid * 32u;
            const uint32_t v = vb + lane, k = v * 16u;
            if (v >= P.vpc) continue;
            const bool masked = vb + 32u > P.fast_cols;                 // warp-uniform
            const uint32_t o1 = P.L + k - s1, o2 = 2u * P.L + k - s2;
            const uint64_t so = static_cast<uint64_t>(g) * P.shard_stride;
            uint8_t *const out[5] = {EMIT ? P.plane[0] + so : nullptr, EMIT ? P.plane[1] + so : nullptr,
                                     EMIT ? P.plane[2] + so : nullptr, P.plane[3] + so, P.plane[4] + so};
            const uint8_t *src = P.data + static_cast<uint64_t>(g) * P.data_stride;
            if (!masked) {
                rs32_row_column<EMIT, false>(src, out, k, o1, o2, 0u, s1, s2, 16, 16, 16, 16, P.st_mode);
            } else {
                rs32_row_column<EMIT, true>(src, out, k, o1, o2, 0u, s1, s2, clamp16(static_cast<int64_t>(P.len) - k),
                                            clamp16(static_cast<int64_t>(P.len) - P.L - k),
                                            clamp16(static_cast<int64_t>(P.len) - 2ll * P.L - k),
                                            clamp16(static_cast<int64_t>(P.L) - k), P.st_mode);
            }
        }
        return;
    }
    const uint32_t g_begin = P.chunk ? blockIdx.x * P.chunk : blockIdx.x;
    const uint32_t g_step = P.chunk ? 1u : gridDim.x;
    const uint32_t g_end = P.chunk ? (g_begin + P.chunk < P.n ? g_begin + P.chunk : P.n) : P.n;
    uint32_t wb = wid;
#pragma unroll 1
    for (uint32_t g = g_begin; g < g_end; g += g_step) {
        const uint32_t v = wb * 32u + lane;
        const uint32_t k = v * 16u;
        const bool masked = wb * 32u + 32u > P.fast_cols;           // warp-uniform
        if (P.rotate) wb = (wb + 1u == nblk) ? 0u : wb + 1u;
        if (v >= P.vpc) continue;
        // aligned in-codeword offsets of the vectors that cover shard 1 / shard 2 at column v
        const uint32_t o1 = P.L + k - s1, o2 = 2u * P.L + k - s2;
        const uint64_t so = static_cast<uint64_t>(g) * P.shard_stride;
        uint8_t *const out[5] = {EMIT ? P.plane[0] + so : nullptr, EMIT ? P.plane[1] + so : nullptr,
                                 EMIT ? P.plane[2] + so : nullptr, P.plane[3] + so, P.plane[4] + so};
        const uint8_t *src = P.data + static_cast<uint64_t>(g) * P.data_stride;
        if (!masked) {
            rs32_row_column<EMIT, false, PF>(src, out, k, o1, o2, 0u, s1, s2, 16, 16, 16, 16, P.st_mode);
        } else {
            rs32_row_column<EMIT, true, PF>(src, out, k, o1, o2, 0u, s1, s2, clamp16(static_cast<int64_t>(P.len) - k),
                                        clamp16(static_cast<int64_t>(P.len) - P.L - k),
                                        clamp16(static_cast<int64_t>(P.len) - 2ll * P.L - k),
                                        clamp16(static_cast<int64_t>(P.L) - k), P.st_mode);
        }
    }
    if (P.tally_last) tally();
}

// ------------------------------------------------------------------------------------------------
// RS(3,2) accept step fed by bulk async copies (the BASELINE config-3 hot kernel)
// ------------------------------------------------------------------------------------------------
// The row kernel above has every thread issue its own five 128-bit loads per column, wait for them, compute and store:
// all of its memory-level parallelism comes from resident warps, each with one load batch in flight.  This kernel
// moves whole rows instead.  A persistent CTA owns a contiguous range of codewords (sequential DRAM streams);
//   * thread 0 streams payload rows, round_up(len,16) bytes each, into a ring of `nin` shared-memory stages with
//     cp.async.bulk (one mbarrier per stage counts the bytes in), keeping up to nin rows per CTA in flight;
//   * the encode warps (one thread per 16-byte column) read the three shards from the stage -- aligned 16-byte reads
//     and the kernel-uniform byte funnel -- apply the row kernel's masking, and write both parity vectors into one of
//     kOut output stages;
//   * after a proxy fence and a barrier of the encode warps, thread 0 writes the two parity rows out with bulk stores
//     (vpc*16 bytes each) and refills the stage just consumed with the payload row nin codewords ahead;
//   * the last warp tallies the CTA's groups while the encode pipeline runs.
// One barrier per codeword is the whole synchronisation: an input stage is refilled only after every encode thread has
// passed the barrier that follows its reads of it, and an output stage is written again only after thread 0 has seen,
// before an earlier barrier, that the bulk store that read it last has finished reading (cp.async.bulk.wait_group.read).
struct Enc32Bulk {
    const uint8_t *data;
    uint64_t data_stride;
    uint8_t *par0, *par1;       // parity planes 0 and 1 (16-byte aligned, padded shard slots)
    uint64_t shard_stride;
    uint32_t n, len, L, vpc;
    uint32_t fast_cols;         // columns [0, fast_cols) need no masking
    uint32_t s1, s2;            // (L & 15), (2L & 15): misalignment of shards 1 and 2
    uint32_t chunk;             // CTA b tallies groups [b*chunk, min(n, (b+1)*chunk)) (and encodes them if !interleave)
    uint32_t interleave;        // 1: CTA b encodes codewords b, b + gridDim.x, ...
    uint32_t in_bytes;         // bytes copied per payload row: round_up(len, 16)
    uint32_t in_pitch;          // bytes per input stage: in_bytes + room for the funnel's reads past the row, 128-aligned
    uint32_t nin;               // input stages
    const uint64_t *planes;     // fused tally (nullptr: none); G == n
    uint32_t R, threshold;
    uint64_t *committed;
    uint32_t *commit_bar;
};

constexpr uint32_t kBulkOut = 4;          // output stages: a bulk store has two codewords' time to read its stage
constexpr uint32_t kBulkHeader = 128;     // the input stages' mbarriers, ahead of the stages

namespace bulk {
__device__ __forceinline__ uint32_t smem_addr(const void *p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@!p bra WAIT_%=;\n}" ::"r"(bar), "r"(parity) : "memory");
}
// global -> shared, completion counted in bytes on the mbarrier
__device__ __forceinline__ void load_row(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
// shared -> global, tracked by bulk groups
__device__ __forceinline__ void store_row(void *dst, uint32_t src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wait_group_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void wait_group_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
// generic-proxy writes to shared memory become visible to the bulk copies issued after the next barrier
__device__ __forceinline__ void fence_async_shared() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void encode_barrier(uint32_t nthreads) { asm volatile("bar.sync 1, %0;" ::"r"(nthreads) : "memory"); }
}  // namespace bulk

__global__ void __launch_bounds__(288) rs32_accept_bulk_kernel(const __grid_constant__ Enc32Bulk P) {
    extern __shared__ __align__(128) uint8_t s_bulk[];
    const uint32_t tid = threadIdx.x, lane = tid & 31u, wid = tid >> 5;
    const uint32_t nenc = blockDim.x - 32u;             // encode threads; the last warp tallies
    const uint32_t lo = blockIdx.x * P.chunk;
    const uint32_t hi = lo + P.chunk < P.n ? lo + P.chunk : P.n;
    // codewords encoded here: lo + i*step (interleaved: step = gridDim.x from blockIdx.x; contiguous: step 1 from lo)
    const uint32_t first = P.interleave ? blockIdx.x : lo;
    const uint32_t step = P.interleave ? gridDim.x : 1u;
    const uint32_t cnt = P.interleave ? (P.n - blockIdx.x + gridDim.x - 1u) / gridDim.x : hi - lo;
    const uint32_t bar0 = bulk::smem_addr(s_bulk);
    uint8_t *const in_base = s_bulk + kBulkHeader;
    uint8_t *const out_base = in_base + static_cast<uint64_t>(P.nin) * P.in_pitch;
    const uint32_t out_pitch = 2u * P.vpc * 16u;        // parity row 0, then parity row 1

    if (tid == 0) {
        for (uint32_t s = 0; s < P.nin; ++s) bulk::mbar_init(bar0 + 8u * s, 1u);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (wid * 32u == nenc) {
        // ---- tally warp: this CTA's groups, coalesced, alongside the encode pipeline ----
        if (P.planes == nullptr) return;
        for (uint32_t g = lo + lane; g < hi; g += 32u) {
            const uint64_t w = dev::tally_word(P.planes, P.R, P.n, g, P.threshold);
            P.committed[g] = w;
            if (P.commit_bar != nullptr) P.commit_bar[g] = dev::commit_prefix(w);
        }
        return;
    }

    auto load = [&](uint32_t dst, uint32_t g, uint32_t bar) {
        bulk::mbar_expect_tx(bar, P.in_bytes);
        bulk::load_row(dst, P.data + static_cast<uint64_t>(g) * P.data_stride, P.in_bytes, bar);
    };
    auto store = [&](uint8_t *dst, uint32_t src) { bulk::store_row(dst, src, P.vpc * 16u); };

    // ---- prologue: fill the ring ----
    if (tid == 0) {
        const uint32_t pre = cnt < P.nin ? cnt : P.nin;
        for (uint32_t i = 0; i < pre; ++i)
            load(bulk::smem_addr(in_base + static_cast<uint64_t>(i) * P.in_pitch), first + i * step, bar0 + 8u * i);
    }

    auto clamp16 = [](int64_t r) { return r > 16 ? 16 : (r < 0 ? 0 : static_cast<int>(r)); };
    const uint32_t v = tid, k = v * 16u;
    const bool active = v < P.vpc;
    const bool masked = v >= P.fast_cols;
    const uint32_t s1 = P.s1, s2 = P.s2;
    const uint32_t o1 = P.L + k - s1, o2 = 2u * P.L + k - s2;   // aligned in-row offsets of the shard 1 / 2 windows
    const int nva = clamp16(static_cast<int64_t>(P.len) - k);
    const int nvb = clamp16(static_cast<int64_t>(P.len) - P.L - k);
    const int nvc = clamp16(static_cast<int64_t>(P.len) - 2ll * P.L - k);
    const int onv = clamp16(static_cast<int64_t>(P.L) - k);
    uint32_t s = 0, phase = 0, o = 0;
#pragma unroll 1
    for (uint32_t i = 0; i < cnt; ++i) {
        bulk::mbar_wait(bar0 + 8u * s, phase);
        const uint8_t *in = in_base + static_cast<uint64_t>(s) * P.in_pitch;
        uint8_t *out = out_base + static_cast<uint64_t>(o) * out_pitch;
        if (active) {
            const uint4 a0 = *reinterpret_cast<const uint4 *>(in + k);
            const uint4 b0 = *reinterpret_cast<const uint4 *>(in + o1);
            const uint4 c0 = *reinterpret_cast<const uint4 *>(in + o2);
            uint4 b = b0, c = c0;
            if (s1 != 0u) b = funnel16(b0, *reinterpret_cast<const uint4 *>(in + o1 + 16u), s1);
            if (s2 != 0u) c = funnel16(c0, *reinterpret_cast<const uint4 *>(in + o2 + 16u), s2);
            uint4 a = a0;
            if (masked) {
                a = keep_bytes(a, nva);
                b = keep_bytes(b, nvb);
                c = keep_bytes(c, nvc);
            }
            uint4 p0, p1;
            rs32_word_fast(a.x, b.x, c.x, p0.x, p1.x);
            rs32_word_fast(a.y, b.y, c.y, p0.y, p1.y);
            rs32_word_fast(a.z, b.z, c.z, p0.z, p1.z);
            rs32_word_fast(a.w, b.w, c.w, p0.w, p1.w);
            if (masked) {
                p0 = keep_bytes(p0, onv);
                p1 = keep_bytes(p1, onv);
            }
            *reinterpret_cast<uint4 *>(out + k) = p0;
            *reinterpret_cast<uint4 *>(out + P.vpc * 16u + k) = p1;
        }
        bulk::fence_async_shared();
        // thread 0: the bulk store that last read the output stage of codeword i + 1 has finished reading it
        if (tid == 0) bulk::wait_group_read<kBulkOut - 2>();
        bulk::encode_barrier(nenc);
        if (tid == 0) {
            const uint64_t so = static_cast<uint64_t>(first + i * step) * P.shard_stride;
            const uint32_t src = bulk::smem_addr(out);
            store(P.par0 + so, src);
            store(P.par1 + so, src + P.vpc * 16u);
            bulk::commit_group();
            // every encode thread is past its reads of stage s: refill it
            if (i + P.nin < cnt) load(bulk::smem_addr(in), first + (i + P.nin) * step, bar0 + 8u * s);
        }
        if (++s == P.nin) { s = 0; phase ^= 1u; }
        if (++o == kBulkOut) o = 0;
    }
    if (tid == 0) bulk::wait_group_all();
}

struct EncRagged {
    const uint8_t *data;
    const uint64_t *data_off;
    const uint32_t *data_len;
    uint8_t *parity;
    uint64_t plane_stride;
    const uint64_t *par_off;
    uint64_t n;
    uint32_t padded;
};

__global__ void __launch_bounds__(kThreads, 3) rs32_encode_ragged_kernel(const __grid_constant__ EncRagged P) {
    // a warp per codeword; the byte-funnel parameters are per-codeword, hence warp-uniform
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = (static_cast<uint64_t>(blockIdx.x) * kThreads + threadIdx.x) >> 5;
    const uint64_t nwarps = (static_cast<uint64_t>(gridDim.x) * kThreads) >> 5;
    const bool padded = (P.padded & 1u) != 0u, emit = (P.padded & 2u) != 0u;
    auto clamp16 = [](int64_t r) { return r > 16 ? 16 : (r < 0 ? 0 : static_cast<int>(r)); };
    // metadata of the next codeword is fetched while the current one is being encoded
    uint32_t nx_len = 0; uint64_t nx_off = 0, nx_poff = 0;
    if (warp < P.n) { nx_len = __ldg(P.data_len + warp); nx_off = __ldg(P.data_off + warp); nx_poff = __ldg(P.par_off + warp); }
    for (uint64_t g = warp; g < P.n; g += nwarps) {
        const uint32_t len = nx_len;
        const uint8_t *pay = P.data + nx_off;
        uint8_t *out = P.parity + nx_poff;
        if (g + nwarps < P.n) {
            nx_len = __ldg(P.data_len + g + nwarps); nx_off = __ldg(P.data_off + g + nwarps); nx_poff = __ldg(P.par_off + g + nwarps);
        }
        if (len == 0u) continue;                      // null codeword (rscoding.rs:451-453)
        const uint32_t L = (len + 2u) / 3u;           // rscoding.rs:177-181 with d = 3
        const uint32_t vpc = (L + 15u) >> 4;
        if (!padded || emit) {                        // byte-exact outputs / emit: general masked path
            for (uint32_t v = lane; v < vpc; v += 32u)
                rs32_column(pay, len, L, v * 16u, out, P.plane_stride, padded, emit);
            continue;
        }
        const uint32_t s0 = static_cast<uint32_t>(reinterpret_cast<uintptr_t>(pay)) & 15u;
        const uint8_t *src = pay - s0;
        const uint32_t s1 = (s0 + L) & 15u, s2 = (s0 + 2u * L) & 15u;
        const uint32_t fast_cols = len >= 2u * L ? (((len - 2u * L) < L ? (len - 2u * L) : L) / 16u) : 0u;
        uint32_t v0 = 0;
        // long codewords: two columns per lane per iteration while both are interior
        for (; v0 + 64u <= fast_cols; v0 += 64u) {
            const uint32_t k = (v0 + lane) * 16u;
            rs32_row_pair(src, out, out + P.plane_stride, k, s0 + L + k - s1, s0 + 2u * L + k - s2, s0, s1, s2);
        }
        for (; v0 < vpc; v0 += 32u) {
            const uint32_t v = v0 + lane;
            if (v >= vpc) break;
            const uint32_t k = v * 16u;
            const uint32_t o1 = s0 + L + k - s1, o2 = s0 + 2u * L + k - s2;
            uint8_t *const outs[5] = {nullptr, nullptr, nullptr, out, out + P.plane_stride};
            if (v0 + 32u <= fast_cols) {
                rs32_row_column<false, false>(src, outs, k, o1, o2, s0, s1, s2, 16, 16, 16, 16);
            } else {
                rs32_row_column<false, true>(src, outs, k, o1, o2, s0, s1, s2,
                                             clamp16(static_cast<int64_t>(len) - k),
                                             clamp16(static_cast<int64_t>(len) - L - k),
                                             clamp16(static_cast<int64_t>(len) - 2ll * L - k),
                                             clamp16(static_cast<int64_t>(L) - k));
            }
        }
    }
}

// generic encode from the payload arena (any d <= 32, p <= P)
struct GenArgs {
    const uint32_t *prog;     // ProgHeader + splats (encode: single program)
    int d;
};

template <int P>
__device__ __forceinline__ void generic_payload_column(const uint8_t *src, uint32_t len, uint32_t L,
                                                       uint32_t k, uint8_t *out, uint64_t plane_stride,
                                                       uint32_t oflags, const uint32_t *prog, int d, int p) {
    const bool padded = (oflags & 1u) != 0u, emit_data = (oflags & 2u) != 0u;
    const int onv = static_cast<int>(L - k) > 16 ? 16 : static_cast<int>(L - k);
    const uint32_t *splat = prog + sizeof(ProgHeader) / 4;
    uint4 acc[P];
#pragma unroll
    for (int j = 0; j < P; ++j) acc[j] = make_uint4(0u, 0u, 0u, 0u);
    for (int i = 0; i < d; ++i) {
        const int64_t pos = static_cast<int64_t>(i) * L + k;
        const int64_t rem = static_cast<int64_t>(len) - pos;
        const int nv = rem > 16 ? 16 : (rem < 0 ? 0 : static_cast<int>(rem));
        const uint4 x = load16(src + pos, nv);        // nv == 0: zeros, no memory access
        if (emit_data)
            store16(out - static_cast<uint64_t>(d - i) * plane_stride + k, x, onv, padded);
        if (nv == 0) continue;                        // all-zero padding contributes nothing
        bitplane_accumulate<P>(x, splat + i * 8, d, p, acc);
    }
#pragma unroll
    for (int j = 0; j < P; ++j)
        if (j < p) store16(out + static_cast<uint64_t>(j) * plane_stride + k, acc[j], onv, padded);
}

template <int P>
__global__ void __launch_bounds__(kThreads)
generic_encode_uniform_kernel(const __grid_constant__ EncUniform E, const uint32_t *__restrict__ prog, int d, int p) {
    const uint32_t t = blockIdx.x * kThreads + threadIdx.x;
    if (E.planes != nullptr && t < E.G) {
        const uint64_t w = dev::tally_word(E.planes, E.R, E.G, t, E.threshold);
        E.committed[t] = w;
        if (E.commit_bar != nullptr) E.commit_bar[t] = dev::commit_prefix(w);
    }
    if (t >= E.total) return;
    const uint32_t g = t / E.vpc;
    const uint32_t k = (t - g * E.vpc) * 16u;
    generic_payload_column<P>(E.data + static_cast<uint64_t>(g) * E.data_stride, E.len, E.L, k,
                              E.parity + static_cast<uint64_t>(g) * E.shard_stride, E.plane_stride,
                              E.padded, prog, d, p);
}

template <int P>
__global__ void __launch_bounds__(kThreads)
generic_encode_ragged_kernel(const __grid_constant__ EncRagged E, const uint32_t *__restrict__ prog, int d, int p) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = (static_cast<uint64_t>(blockIdx.x) * kThreads + threadIdx.x) >> 5;
    const uint64_t nwarps = (static_cast<uint64_t>(gridDim.x) * kThreads) >> 5;
    for (uint64_t g = warp; g < E.n; g += nwarps) {
        const uint32_t len = __ldg(E.data_len + g);
        if (len == 0u) continue;
        const uint32_t L = (len + static_cast<uint32_t>(d) - 1u) / static_cast<uint32_t>(d);
        const uint32_t vpc = (L + 15u) >> 4;
        const uint8_t *src = E.data + __ldg(E.data_off + g);
        uint8_t *out = E.parity + __ldg(E.par_off + g);
        for (uint32_t v = lane; v < vpc; v += 32u)
            generic_payload_column<P>(src, len, L, v * 16u, out, E.plane_stride, E.padded, prog, d, p);
    }
}

// ------------------------------------------------------------------------------------------------
// reconstruct kernel: shards in planes, one coefficient program per erasure pattern
// ------------------------------------------------------------------------------------------------
struct DecArgs {
    uint8_t *shards;
    uint64_t plane_stride;
    const uint64_t *off;
    const uint32_t *data_len;
    const uint32_t *present;
    uint64_t n;
    int32_t *status;
    const uint8_t *progs;     // 2^(d+p) programs of prog_stride bytes
    uint32_t prog_stride;
    uint32_t pattern_mask;
    int d;
    uint32_t padded;
    uint32_t hmask_off;       // words from the splat table to the Horner mask table (p*d*8)
    uint32_t need_mask;       // shards that must be present for a codeword to need no work (data only, or all)
    const uint8_t *fast_progs; // d <= 4: compact programs
    uint32_t fast_stride, fast_bytes;
};

template <int P>
__global__ void __launch_bounds__(kThreads) generic_reconstruct_kernel(const __grid_constant__ DecArgs A) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = (static_cast<uint64_t>(blockIdx.x) * kThreads + threadIdx.x) >> 5;
    const uint64_t nwarps = (static_cast<uint64_t>(gridDim.x) * kThreads) >> 5;
    const int d = A.d;
    for (uint64_t g = warp; g < A.n; g += nwarps) {
        const uint32_t len = __ldg(A.data_len + g);
        if (len == 0u) {                              // null codeword: rscoding.rs:495-497
            if (lane == 0u) A.status[g] = SS_ERR_INVALID_ARG;
            continue;
        }
        const uint32_t pat = __ldg(A.present + g) & A.pattern_mask;
        const uint8_t *prog = A.progs + static_cast<uint64_t>(pat) * A.prog_stride;
        const ProgHeader *hdr = reinterpret_cast<const ProgHeader *>(prog);
        const int valid = hdr->valid;
        const int n_out = hdr->n_out;
        if (lane == 0u) A.status[g] = valid ? SS_OK : SS_ERR_TOO_FEW_SHARDS_PRESENT;
        if (!valid || n_out == 0) continue;           // never partial output
        const uint32_t *splat = reinterpret_cast<const uint32_t *>(prog + sizeof(ProgHeader));
        const uint32_t L = (len + static_cast<uint32_t>(d) - 1u) / static_cast<uint32_t>(d);
        const uint32_t vpc = (L + 15u) >> 4;
        uint8_t *base = A.shards + __ldg(A.off + g);
        for (uint32_t v = lane; v < vpc; v += 32u) {
            const uint32_t k = v * 16u;
            const int nv = static_cast<int>(L - k) > 16 ? 16 : static_cast<int>(L - k);
            uint4 acc[P];
#pragma unroll
            for (int j = 0; j < P; ++j) acc[j] = make_uint4(0u, 0u, 0u, 0u);
            for (int i = 0; i < d; ++i) {
                const uint4 x = load16(base + static_cast<uint64_t>(hdr->src[i]) * A.plane_stride + k, nv);
                bitplane_accumulate<P>(x, splat + i * 8, d, n_out, acc);
            }
#pragma unroll
            for (int j = 0; j < P; ++j)
                if (j < n_out)
                    store16(base + static_cast<uint64_t>(hdr->dst[j]) * A.plane_stride + k, acc[j], nv,
                            A.padded != 0u);
        }
    }
}


// ------------------------------------------------------------------------------------------------
// Horner core for arbitrary (run-time) coefficients, d <= D sources held in registers.
//   out_j = sum_i c_ji * x_i = sum_k x^k * ( XOR of the x_i whose c_ji has bit k set )
// evaluated from the top bit down: acc = acc*x ^ (XOR_i x_i & hmask[j][i][k]).  Per output word that is
// (top+1) * d lop3 + top packed-xtime steps -- 2-3x fewer ALU ops than the bit-plane form, which matters
// because reconstruction is otherwise ALU-bound rather than HBM-bound.
// ------------------------------------------------------------------------------------------------
template <int D>
__device__ __forceinline__ uint4 horner_row(const uint4 (&x)[D], int d, const uint32_t *__restrict__ hm_j, int top) {
    uint4 acc = make_uint4(0u, 0u, 0u, 0u);
    for (int k = top; k >= 0; --k) {
        if (k != top) {
            const uint4 m = make_uint4(msb_mask(acc.x), msb_mask(acc.y), msb_mask(acc.z), msb_mask(acc.w));
            acc.x = ((acc.x * 2u) & 0xfefefefeu) ^ (m.x & 0x1d1d1d1du);
            acc.y = ((acc.y * 2u) & 0xfefefefeu) ^ (m.y & 0x1d1d1d1du);
            acc.z = ((acc.z * 2u) & 0xfefefefeu) ^ (m.z & 0x1d1d1d1du);
            acc.w = ((acc.w * 2u) & 0xfefefefeu) ^ (m.w & 0x1d1d1d1du);
        }
#pragma unroll
        for (int i = 0; i < D; ++i) {
            if (i < d) {
                const uint32_t hm = __ldg(hm_j + i * 8 + k);
                acc.x ^= x[i].x & hm;
                acc.y ^= x[i].y & hm;
                acc.z ^= x[i].z & hm;
                acc.w ^= x[i].w & hm;
            }
        }
    }
    return acc;
}

// Horner row for d <= 4 with the transposed mask table: one 128-bit load per bit level brings the masks of
// all inputs (hmT[(j*8 + k)*4 + i]).
template <int D, bool SMEM>
__device__ __forceinline__ uint4 horner_row_t(const uint4 (&x)[D], const uint4 *__restrict__ hmT_j, int top) {
    uint4 acc = make_uint4(0u, 0u, 0u, 0u);
    for (int k = top; k >= 0; --k) {
        const uint4 hm = SMEM ? hmT_j[k] : __ldg(hmT_j + k);
        if (k != top) {
            const uint4 m = make_uint4(msb_mask(acc.x), msb_mask(acc.y), msb_mask(acc.z), msb_mask(acc.w));
            acc.x = ((acc.x * 2u) & 0xfefefefeu) ^ (m.x & 0x1d1d1d1du);
            acc.y = ((acc.y * 2u) & 0xfefefefeu) ^ (m.y & 0x1d1d1d1du);
            acc.z = ((acc.z * 2u) & 0xfefefefeu) ^ (m.z & 0x1d1d1d1du);
            acc.w = ((acc.w * 2u) & 0xfefefefeu) ^ (m.w & 0x1d1d1d1du);
        }
        const uint32_t hmi[4] = {hm.x, hm.y, hm.z, hm.w};
#pragma unroll
        for (int i = 0; i < D; ++i) {
            acc.x ^= x[i].x & hmi[i];
            acc.y ^= x[i].y & hmi[i];
            acc.z ^= x[i].z & hmi[i];
            acc.w ^= x[i].w & hmi[i];
        }
    }
    return acc;
}

template <int D>
__global__ void __launch_bounds__(kThreads, D <= 4 ? 4 : 2) horner_reconstruct_kernel(const __grid_constant__ DecArgs A) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = (static_cast<uint64_t>(blockIdx.x) * kThreads + threadIdx.x) >> 5;
    const uint64_t nwarps = (static_cast<uint64_t>(gridDim.x) * kThreads) >> 5;
    const int d = A.d;
    uint32_t nx_len = 0, nx_pat = 0;
    if (warp < A.n) { nx_len = __ldg(A.data_len + warp); nx_pat = __ldg(A.present + warp); }
    for (uint64_t g = warp; g < A.n; g += nwarps) {
        const uint32_t len = nx_len;
        const uint32_t pat = nx_pat & A.pattern_mask;
        if (g + nwarps < A.n) { nx_len = __ldg(A.data_len + g + nwarps); nx_pat = __ldg(A.present + g + nwarps); }
        if (len == 0u) {                              // null codeword: rscoding.rs:495-497
            if (lane == 0u) A.status[g] = SS_ERR_INVALID_ARG;
            continue;
        }
        if ((pat & A.need_mask) == A.need_mask) {     // nothing to regenerate: no table look-up at all
            if (lane == 0u) A.status[g] = SS_OK;
            continue;
        }
        const uint8_t *prog = A.progs + static_cast<uint64_t>(pat) * A.prog_stride;
        const ProgHeader *hdr = reinterpret_cast<const ProgHeader *>(prog);
        const int valid = hdr->valid;
        const int n_out = hdr->n_out;
        if (lane == 0u) A.status[g] = valid ? SS_OK : SS_ERR_TOO_FEW_SHARDS_PRESENT;
        if (!valid || n_out == 0) continue;           // never partial output
        const uint32_t *hmask = reinterpret_cast<const uint32_t *>(prog + sizeof(ProgHeader)) + A.hmask_off;
        const uint32_t L = (len + static_cast<uint32_t>(d) - 1u) / static_cast<uint32_t>(d);
        const uint32_t vpc = (L + 15u) >> 4;
        uint8_t *base = A.shards + __ldg(A.off + g);
        for (uint32_t v = lane; v < vpc; v += 32u) {
            const uint32_t k = v * 16u;
            const int nv = static_cast<int>(L - k) > 16 ? 16 : static_cast<int>(L - k);
            uint4 x[D];
            dev::Raw16 raw[D];
            // every source load of the column is issued before any loaded byte is touched
#pragma unroll
            for (int i = 0; i < D; ++i) {
                raw[i].lo = make_uint4(0u, 0u, 0u, 0u); raw[i].hi = raw[i].lo; raw[i].s = 0u;
                if (i < d) {
                    const uint8_t *sp = base + static_cast<uint64_t>(hdr->src[i]) * A.plane_stride + k;
                    // padded layout: every shard slot is 16-byte aligned -> one aligned 128-bit load
                    if (A.padded != 0u) raw[i].lo = dev::ldg128(sp);
                    else raw[i] = dev::raw16_issue(sp, nv);
                }
            }
#pragma unroll
            for (int i = 0; i < D; ++i) x[i] = dev::raw16_finish(raw[i], nv);
            for (int j = 0; j < n_out; ++j) {
                const uint4 acc = horner_row<D>(x, d, hmask + j * d * 8, hdr->top[j]);
                store16(base + static_cast<uint64_t>(hdr->dst[j]) * A.plane_stride + k, acc, nv, A.padded != 0u);
            }
        }
    }
}


// ------------------------------------------------------------------------------------------------
// reconstruct for small codes (d <= 4, i.e. every 3/5/7-replica deployment): compact per-pattern programs
// staged in shared memory (no dependent global look-ups between a codeword's metadata and its shard loads),
// Horner rows from one 128-bit mask word per bit level, XOR chain for the second of two missing data shards.
// ------------------------------------------------------------------------------------------------
template <int D, bool SMEM, bool PADDED, bool PAIR>
__global__ void __launch_bounds__(kThreads, PAIR ? 3 : 4) rs_reconstruct_small_kernel(const __grid_constant__ DecArgs A) {
    extern __shared__ uint4 s_prog[];
    const uint8_t *table = A.fast_progs;
    if (SMEM) {
        const uint4 *gsrc = reinterpret_cast<const uint4 *>(A.fast_progs);
        for (uint32_t i = threadIdx.x; i < A.fast_bytes / 16u; i += kThreads) s_prog[i] = __ldg(gsrc + i);
        __syncthreads();
        table = reinterpret_cast<const uint8_t *>(s_prog);
    }
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = (static_cast<uint64_t>(blockIdx.x) * kThreads + threadIdx.x) >> 5;
    const uint64_t nwarps = (static_cast<uint64_t>(gridDim.x) * kThreads) >> 5;
    const int d = A.d;
    constexpr bool padded = PADDED;
    uint32_t nx_len = 0, nx_pat = 0; uint64_t nx_off = 0;
    if (warp < A.n) { nx_len = __ldg(A.data_len + warp); nx_pat = __ldg(A.present + warp); nx_off = __ldg(A.off + warp); }
    for (uint64_t g = warp; g < A.n; g += nwarps) {
        const uint32_t len = nx_len;
        const uint32_t pat = nx_pat & A.pattern_mask;
        uint8_t *base = A.shards + nx_off;
        if (g + nwarps < A.n) {
            nx_len = __ldg(A.data_len + g + nwarps); nx_pat = __ldg(A.present + g + nwarps); nx_off = __ldg(A.off + g + nwarps);
        }
        if (len == 0u) {                              // null codeword: rscoding.rs:495-497
            if (lane == 0u) A.status[g] = SS_ERR_INVALID_ARG;
            continue;
        }
        if ((pat & A.need_mask) == A.need_mask) {     // nothing to regenerate
            if (lane == 0u) A.status[g] = SS_OK;
            continue;
        }
        const uint8_t *prog = table + pat * A.fast_stride;
        const FastProgHeader *hdr = reinterpret_cast<const FastProgHeader *>(prog);
        const int valid = hdr->valid;
        const int n_out = hdr->n_out;
        if (lane == 0u) A.status[g] = valid ? SS_OK : SS_ERR_TOO_FEW_SHARDS_PRESENT;
        if (!valid || n_out == 0) continue;           // never partial output
        const uint4 *hmT = reinterpret_cast<const uint4 *>(prog + sizeof(FastProgHeader));
        const uint32_t L = (len + static_cast<uint32_t>(d) - 1u) / static_cast<uint32_t>(d);
        const uint32_t vpc = (L + 15u) >> 4;
        const uint8_t *sp[D];
#pragma unroll
        for (int i = 0; i < D; ++i) sp[i] = base + static_cast<uint64_t>(hdr->src[i < d ? i : 0]) * A.plane_stride;
        const int top0 = hdr->top[0], top1 = hdr->top[1];
        const bool chain1 = hdr->chain1 != 0;
        uint8_t *dp0 = base + static_cast<uint64_t>(hdr->dst[0]) * A.plane_stride;
        uint8_t *dp1 = base + static_cast<uint64_t>(hdr->dst[1]) * A.plane_stride;
        // one column: Horner rows of the missing shards from the d source vectors
        auto emit = [&](const uint4 (&x)[D], uint32_t k, int nv) {
            const uint4 y0 = horner_row_t<D, SMEM>(x, hmT, top0);
            store16(dp0 + k, y0, nv, padded);
            if (n_out > 1) {
                uint4 y1 = horner_row_t<D, SMEM>(x, hmT + 8, top1);
                if (chain1) { y1.x ^= y0.x; y1.y ^= y0.y; y1.z ^= y0.z; y1.w ^= y0.w; }
                store16(dp1 + k, y1, nv, padded);
            }
            for (int j = 2; j < n_out; ++j)
                store16(base + static_cast<uint64_t>(hdr->dst[j]) * A.plane_stride + k,
                        horner_row_t<D, SMEM>(x, hmT + j * 8, hdr->top[j]), nv, padded);
        };
        if constexpr (PADDED && PAIR) {
            // Two columns (v and v + 32) per lane and pass: all 2d source loads are issued before any loaded byte is
            // touched, so a warp that walks its codeword alone keeps twice the bytes in flight.
            for (uint32_t v = lane; v < vpc; v += 64u) {
                const uint32_t k0 = v * 16u, k1 = k0 + 512u;
                const bool two = v + 32u < vpc;
                const int nv0 = static_cast<int>(L - k0) > 16 ? 16 : static_cast<int>(L - k0);
                const int nv1 = two ? (static_cast<int>(L - k1) > 16 ? 16 : static_cast<int>(L - k1)) : 0;
                uint4 x[D], y[D];
#pragma unroll
                for (int i = 0; i < D; ++i) {
                    x[i] = make_uint4(0u, 0u, 0u, 0u);
                    y[i] = x[i];
                    if (i < d) {
                        x[i] = dev::ldg128(sp[i] + k0);
                        if (two) y[i] = dev::ldg128(sp[i] + k1);
                    }
                }
                if (nv0 < 16) {
#pragma unroll
                    for (int i = 0; i < D; ++i) x[i] = keep_bytes(x[i], nv0);
                }
                if (two && nv1 < 16) {
#pragma unroll
                    for (int i = 0; i < D; ++i) y[i] = keep_bytes(y[i], nv1);
                }
                emit(x, k0, nv0);
                if (two) emit(y, k1, nv1);
            }
        } else {
            for (uint32_t v = lane; v < vpc; v += 32u) {
                const uint32_t k = v * 16u;
                const int nv = static_cast<int>(L - k) > 16 ? 16 : static_cast<int>(L - k);
                uint4 x[D];
                // every source load of the column is issued before any loaded byte is touched
                if constexpr (PADDED) {
#pragma unroll
                    for (int i = 0; i < D; ++i) {
                        x[i] = make_uint4(0u, 0u, 0u, 0u);
                        if (i < d) x[i] = dev::ldg128(sp[i] + k);
                    }
                    if (nv < 16) {
#pragma unroll
                        for (int i = 0; i < D; ++i) x[i] = keep_bytes(x[i], nv);
                    }
                } else {
                    dev::Raw16 raw[D];
#pragma unroll
                    for (int i = 0; i < D; ++i) {
                        raw[i].lo = make_uint4(0u, 0u, 0u, 0u); raw[i].hi = raw[i].lo; raw[i].s = 0u;
                        if (i < d) raw[i] = dev::raw16_issue(sp[i] + k, nv);
                    }
#pragma unroll
                    for (int i = 0; i < D; ++i) x[i] = dev::raw16_finish(raw[i], nv);
                }
                emit(x, k, nv);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// RS(3,2) reconstruct, uniform geometry: the row structure of the encode kernel.  A CTA walks codewords, thread = 16-byte
// column; the codeword's present mask is CTA-uniform, so one switch per codeword selects the pattern's COMPILE-TIME
// column routine (rs32_decode.cuh): three aligned source loads, a fully unrolled Horner row per missing shard (XOR chain
// where the all-ones parity row allows), one or two 128-bit stores.  Intact codewords cost one 4-byte read (prefetched an
// iteration ahead) and a status write; nothing is looked up in memory between a codeword's mask and its shard loads.
// ------------------------------------------------------------------------------------------------
struct Dec32Row {
    uint8_t *shards;
    uint64_t plane_stride, shard_stride;
    const uint32_t *present;
    int32_t *status;
    uint32_t n, L, vpc;
};

template <uint32_t PAT, bool DATA_ONLY>
__device__ __forceinline__ void rs32_dec_column(uint8_t *__restrict__ base, uint64_t plane_stride, int nv) {
    constexpr rs32::Decode D = rs32::make_decode(PAT, DATA_ONLY);
    const uint4 x0 = dev::ldg128(base + D.src[0] * plane_stride);
    const uint4 x1 = dev::ldg128(base + D.src[1] * plane_stride);
    const uint4 x2 = dev::ldg128(base + D.src[2] * plane_stride);
    uint4 y0, y1 = make_uint4(0u, 0u, 0u, 0u);
    rs32::decode_column<PAT, DATA_ONLY>(x0, x1, x2, y0, y1);
    dev::stg128_cs(base + D.dst[0] * plane_stride, nv < 16 ? keep_bytes(y0, nv) : y0);
    if constexpr (D.n_out == 2) dev::stg128_cs(base + D.dst[1] * plane_stride, nv < 16 ? keep_bytes(y1, nv) : y1);
}

template <bool DATA_ONLY, int MAXT, int MINB>
__global__ void __launch_bounds__(MAXT, MINB) rs32_reconstruct_row_kernel(const __grid_constant__ Dec32Row P) {
    uint32_t g = blockIdx.x;
    uint32_t nx_pat = g < P.n ? __ldg(P.present + g) : 0u;
#pragma unroll 1
    for (; g < P.n; g += gridDim.x) {
        const uint32_t pat = nx_pat & 31u;
        if (g + gridDim.x < P.n) nx_pat = __ldg(P.present + g + gridDim.x);     // next codeword's mask, one iteration ahead
        const bool enough = __popc(pat) >= 3;                                   // crate: Error::TooFewShardsPresent
        if (threadIdx.x == 0u) P.status[g] = enough ? SS_OK : SS_ERR_TOO_FEW_SHARDS_PRESENT;
        if (!enough || !rs32::needs_work(pat, DATA_ONLY)) continue;             // never partial output
        uint8_t *cw = P.shards + static_cast<uint64_t>(g) * P.shard_stride;
        for (uint32_t v = threadIdx.x; v < P.vpc; v += blockDim.x) {
            const int nv = static_cast<int>(P.L - v * 16u) > 16 ? 16 : static_cast<int>(P.L - v * 16u);
            // a switch the compiler turns into a jump table over the pattern-specialised column routines
            switch (pat) {
#define SS_DEC_CASE(PT) case PT: if constexpr (rs32::make_decode(PT, DATA_ONLY).valid && rs32::needs_work(PT, DATA_ONLY)) \
                                     rs32_dec_column<PT, DATA_ONLY>(cw + v * 16u, P.plane_stride, nv); break;
                SS_DEC_CASE(7) SS_DEC_CASE(11) SS_DEC_CASE(13) SS_DEC_CASE(14) SS_DEC_CASE(15) SS_DEC_CASE(19) SS_DEC_CASE(21)
                SS_DEC_CASE(22) SS_DEC_CASE(23) SS_DEC_CASE(25) SS_DEC_CASE(26) SS_DEC_CASE(27) SS_DEC_CASE(28) SS_DEC_CASE(29)
                SS_DEC_CASE(30) SS_DEC_CASE(31)
#undef SS_DEC_CASE
                default: break;
            }
        }
    }
}

// off[g] = g * stride, len[g] = data_len: lets the ragged kernels serve a uniform batch of any code
__global__ void uniform_meta_kernel(uint64_t *off, uint32_t *len, uint64_t n, uint64_t stride, uint32_t data_len) {
    const uint64_t step = static_cast<uint64_t>(gridDim.x) * blockDim.x;
    for (uint64_t g = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; g < n; g += step) {
        off[g] = g * stride;
        len[g] = data_len;
    }
}

template <int D>
__device__ __forceinline__ void horner_payload_column(const uint8_t *src, uint32_t len, uint32_t L, uint32_t k,
                                                      uint8_t *out, uint64_t plane_stride, uint32_t oflags,
                                                      const uint32_t *prog, int d, int p) {
    const bool padded = (oflags & 1u) != 0u, emit_data = (oflags & 2u) != 0u;
    const int onv = static_cast<int>(L - k) > 16 ? 16 : static_cast<int>(L - k);
    const ProgHeader *hdr = reinterpret_cast<const ProgHeader *>(prog);
    const uint32_t *hmask = prog + sizeof(ProgHeader) / 4 + p * d * 8;
    uint4 x[D];
    dev::Raw16 raw[D];
    // every source load of the column is issued before any loaded byte is touched
#pragma unroll
    for (int i = 0; i < D; ++i) {
        raw[i].lo = make_uint4(0u, 0u, 0u, 0u); raw[i].hi = raw[i].lo; raw[i].s = 0u;
        if (i < d) {
            const int64_t pos = static_cast<int64_t>(i) * L + k;
            const int64_t rem = static_cast<int64_t>(len) - pos;
            raw[i] = dev::raw16_issue(src + pos, rem > 16 ? 16 : (rem < 0 ? 0 : static_cast<int>(rem)));
        }
    }
#pragma unroll
    for (int i = 0; i < D; ++i) {
        if (i < d) {
            const int64_t rem = static_cast<int64_t>(len) - (static_cast<int64_t>(i) * L + k);
            x[i] = dev::raw16_finish(raw[i], rem > 16 ? 16 : (rem < 0 ? 0 : static_cast<int>(rem)));
            if (emit_data) store16(out - static_cast<uint64_t>(d - i) * plane_stride + k, x[i], onv, padded);
        } else {
            x[i] = make_uint4(0u, 0u, 0u, 0u);
        }
    }
    for (int j = 0; j < p; ++j) {
        const uint4 acc = horner_row<D>(x, d, hmask + j * d * 8, hdr->top[j]);
        store16(out + static_cast<uint64_t>(j) * plane_stride + k, acc, onv, padded);
    }
}

template <int D>
__global__ void __launch_bounds__(kThreads)
horner_encode_uniform_kernel(const __grid_constant__ EncUniform E, const uint32_t *__restrict__ prog, int d, int p) {
    const uint32_t t = blockIdx.x * kThreads + threadIdx.x;
    if (E.planes != nullptr && t < E.G) {
        const uint64_t w = dev::tally_word(E.planes, E.R, E.G, t, E.threshold);
        E.committed[t] = w;
        if (E.commit_bar != nullptr) E.commit_bar[t] = dev::commit_prefix(w);
    }
    if (t >= E.total) return;
    const uint32_t g = t / E.vpc;
    const uint32_t k = (t - g * E.vpc) * 16u;
    horner_payload_column<D>(E.data + static_cast<uint64_t>(g) * E.data_stride, E.len, E.L, k,
                             E.parity + static_cast<uint64_t>(g) * E.shard_stride, E.plane_stride, E.padded, prog, d, p);
}

template <int D>
__global__ void __launch_bounds__(kThreads)
horner_encode_ragged_kernel(const __grid_constant__ EncRagged E, const uint32_t *__restrict__ prog, int d, int p) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = (static_cast<uint64_t>(blockIdx.x) * kThreads + threadIdx.x) >> 5;
    const uint64_t nwarps = (static_cast<uint64_t>(gridDim.x) * kThreads) >> 5;
    for (uint64_t g = warp; g < E.n; g += nwarps) {
        const uint32_t len = __ldg(E.data_len + g);
        if (len == 0u) continue;
        const uint32_t L = (len + static_cast<uint32_t>(d) - 1u) / static_cast<uint32_t>(d);
        const uint32_t vpc = (L + 15u) >> 4;
        const uint8_t *src = E.data + __ldg(E.data_off + g);
        uint8_t *out = E.parity + __ldg(E.par_off + g);
        for (uint32_t v = lane; v < vpc; v += 32u)
            horner_payload_column<D>(src, len, L, v * 16u, out, E.plane_stride, E.padded, prog, d, p);
    }
}


int match_static_code(int d, int p, const uint8_t *matrix) {
    for (int c = 0; c < kNumStaticCodes; ++c) {
        if (static_code_d(c) != d || static_code_p(c) != p) continue;
        bool same = true;
        for (int j = 0; j < p && same; ++j)
            for (int i = 0; i < d; ++i)
                if (matrix[static_cast<size_t>(d + j) * d + i] != static_code_coef(c, j, i)) { same = false; break; }
        if (same) return c;
    }
    return -1;
}

// smallest instantiated register capacity >= d (0: use the bit-plane kernels)
template <typename F>
static int dispatch_d(int d, F &&f) {
    if (d <= 2) return f(std::integral_constant<int, 2>{});
    if (d == 3) return f(std::integral_constant<int, 3>{});
    if (d == 4) return f(std::integral_constant<int, 4>{});
    if (d <= 6) return f(std::integral_constant<int, 6>{});
    return f(std::integral_constant<int, 8>{});
}

// ------------------------------------------------------------------------------------------------
// host launchers
// ------------------------------------------------------------------------------------------------
static inline uint32_t ragged_grid(ss_ctx *ctx, uint64_t n) {
    // persistent-ish grid: enough warps to fill the machine several times over, capped by n
    const uint64_t warps_per_cta = kThreads / 32;
    uint64_t ctas = (n + warps_per_cta - 1) / warps_per_cta;
    const uint64_t cap = static_cast<uint64_t>(ctx->sm_count) * 8ull * 4ull;  // 8 CTAs/SM resident x 4 waves
    if (ctas > cap) ctas = cap;
    if (ctas == 0) ctas = 1;
    return static_cast<uint32_t>(ctas);
}

template <typename F>
static int dispatch_p(int p, F &&f) {
    switch (p) {
        case 1: return f(std::integral_constant<int, 1>{});
        case 2: return f(std::integral_constant<int, 2>{});
        case 3: return f(std::integral_constant<int, 3>{});
        case 4: return f(std::integral_constant<int, 4>{});
        case 5: case 6: return f(std::integral_constant<int, 6>{});
        case 7: case 8: return f(std::integral_constant<int, 8>{});
        default: return set_error(SS_ERR_UNSUPPORTED, "batched kernels support at most %d outputs, got %d", kMaxP, p);
    }
}

// f(integral_constant<D>, integral_constant<Code>): a compile-time cluster code at its exact width, any other code
// (kCodeGeneric) at dispatch_d's capacity for d.  The NVRTC code (kCodeJit) is launched by the callers themselves.
template <typename F>
static int dispatch_code(int sc, int d, F &&f) {
    auto fixed = [&](auto CC) { return f(std::integral_constant<int, static_code_d(decltype(CC)::value)>{}, CC); };
    switch (sc) {
        case kCode21: return fixed(std::integral_constant<int, kCode21>{});
        case kCode43: return fixed(std::integral_constant<int, kCode43>{});
        case kCode54: return fixed(std::integral_constant<int, kCode54>{});
        case kCode42: return fixed(std::integral_constant<int, kCode42>{});
        case kCode31: return fixed(std::integral_constant<int, kCode31>{});
        default: return dispatch_d(d, [&](auto DC) { return f(DC, std::integral_constant<int, kCodeGeneric>{}); });
    }
}

// the fused-tally fields of an encode kernel's parameters (t == nullptr: no tally)
template <typename Args>
static void set_tally(Args &a, const TallyArgs *t) {
    const TallyArgs none;
    if (t == nullptr) t = &none;
    a.planes = t->planes; a.R = t->R; a.threshold = t->threshold; a.committed = t->committed; a.commit_bar = t->commit_bar;
}

// base of shard plane j of a uniform batch: the caller's explicit plane bases, or parity plane j - d
static uint8_t *out_plane(const EncGeom &g, int d, int j) {
    if (g.plane_ptrs != nullptr) return g.plane_ptrs[j];
    return g.parity + (static_cast<int64_t>(j) - d) * static_cast<int64_t>(g.plane_stride);
}


// ------------------------------------------------------------------------------------------------
// Crossword distribute (BASELINE config 4, n = 5 replicas, RS(3,2), T = 5 total shards, dj = 1):
// encode a ragged batch and write, for every codeword g, the spr[g] shards of replica r --
// shards {(r + k) mod 5 : k < spr} (balanced round-robin assignment, crossword/mod.rs:866-888) -- into
// replica r's log at rep_off[g] + k * round_up(L_g,32).  The five log bases may be local memory or peer
// GPUs' HBM (CUDA IPC): this is crossword/request.rs:137-185 (subset_copy per peer + send_msg) for a
// whole batch, with the NVLink transfer done by the encode kernel's own stores.
// ------------------------------------------------------------------------------------------------
struct CwDistribute {
    const uint8_t *data;
    const uint64_t *data_off;
    const uint32_t *data_len;
    const uint8_t *spr;        // shards per replica of codeword g (1..3)
    const uint64_t *rep_off;   // byte offset of codeword g's slots inside every replica log
    uint8_t *rep[5];           // replica log bases
    uint64_t n;
    unsigned long long *next_cw;   // dynamic kernels: the next codeword nobody has taken yet (zeroed before the launch)
};

// raw aligned vectors covering one unmasked column of the three data shards
struct Raw6 { uint4 a0, a1, b0, b1, c0, c1; };
__device__ __forceinline__ void rs32_issue_loads(const uint8_t *__restrict__ src, uint32_t k, uint32_t o1, uint32_t o2,
                                                 uint32_t s0, uint32_t s1, uint32_t s2, Raw6 &r) {
    r.a0 = dev::ldg128(src + k);
    r.a1 = make_uint4(0u, 0u, 0u, 0u);       // zeros, not copies of the loads (see rs32_row_column)
    if (s0 != 0u) r.a1 = dev::ldg128(src + k + 16u);
    r.b0 = dev::ldg128(src + o1);
    r.b1 = make_uint4(0u, 0u, 0u, 0u);
    if (s1 != 0u) r.b1 = dev::ldg128(src + o1 + 16u);
    r.c0 = dev::ldg128(src + o2);
    r.c1 = make_uint4(0u, 0u, 0u, 0u);
    if (s2 != 0u) r.c1 = dev::ldg128(src + o2 + 16u);
}
__device__ __forceinline__ void rs32_shards_from_raw(const Raw6 &r, uint32_t s0, uint32_t s1, uint32_t s2, uint4 (&sh)[5]) {
    sh[0] = s0 != 0u ? funnel16(r.a0, r.a1, s0) : r.a0;
    sh[1] = s1 != 0u ? funnel16(r.b0, r.b1, s1) : r.b0;
    sh[2] = s2 != 0u ? funnel16(r.c0, r.c1, s2) : r.c0;
    rs32_word_fast(sh[0].x, sh[1].x, sh[2].x, sh[3].x, sh[4].x);
    rs32_word_fast(sh[0].y, sh[1].y, sh[2].y, sh[3].y, sh[4].y);
    rs32_word_fast(sh[0].z, sh[1].z, sh[2].z, sh[3].z, sh[4].z);
    rs32_word_fast(sh[0].w, sh[1].w, sh[2].w, sh[3].w, sh[4].w);
}
// replica r, slot kk holds shard (r + kk) mod 5
__device__ __forceinline__ void distribute_store(const CwDistribute &P, uint64_t ro, uint32_t k, uint32_t Lpad, uint32_t spr,
                                                 const uint4 (&sh)[5]) {
#pragma unroll
    for (int r = 0; r < 5; ++r) {
        uint8_t *dst = P.rep[r] + ro + k;
#pragma unroll
        for (int kk = 0; kk < 3; ++kk)
            if (static_cast<uint32_t>(kk) < spr) dev::stg128_cs(dst + static_cast<uint64_t>(kk) * Lpad, sh[(r + kk) % 5]);
    }
}

// one column (masked when it touches the payload tail / the last partial vector) of codeword geometry (len, L, s0)
__device__ __forceinline__ void cw_column(const CwDistribute &P, const uint8_t *__restrict__ src, uint32_t len, uint32_t L, uint32_t v,
                                          uint32_t s0, uint32_t s1, uint32_t s2, bool fast, uint64_t ro, uint32_t Lpad, uint32_t spr) {
    auto clamp16 = [](int64_t r) { return r > 16 ? 16 : (r < 0 ? 0 : static_cast<int>(r)); };
    const uint32_t k = v * 16u;
    const uint32_t o1 = s0 + L + k - s1, o2 = s0 + 2u * L + k - s2;
    uint4 sh[5];
    if (fast) {
        Raw6 r1;
        rs32_issue_loads(src, k, o1, o2, s0, s1, s2, r1);
        rs32_shards_from_raw(r1, s0, s1, s2, sh);
    } else {
        const int nva = clamp16(static_cast<int64_t>(len) - k);
        const int nvb = clamp16(static_cast<int64_t>(len) - L - k);
        const int nvc = clamp16(static_cast<int64_t>(len) - 2ll * L - k);
        const int onv = clamp16(static_cast<int64_t>(L) - k);
        uint4 a0 = make_uint4(0u, 0u, 0u, 0u), a1 = a0;    // the all-padding column of an odd-length slot reads nothing
        if (nva > 0) a0 = dev::ldg128(src + k);
        if (s0 != 0u && static_cast<int>(s0) + nva > 16) a1 = dev::ldg128(src + k + 16u);
        uint4 b0 = make_uint4(0u, 0u, 0u, 0u), c0 = make_uint4(0u, 0u, 0u, 0u);
        if (nvb > 0) b0 = dev::ldg128(src + o1);
        uint4 b1 = make_uint4(0u, 0u, 0u, 0u);
        if (s1 != 0u && static_cast<int>(s1) + nvb > 16) b1 = dev::ldg128(src + o1 + 16u);
        if (nvc > 0) c0 = dev::ldg128(src + o2);
        uint4 c1 = make_uint4(0u, 0u, 0u, 0u);
        if (s2 != 0u && static_cast<int>(s2) + nvc > 16) c1 = dev::ldg128(src + o2 + 16u);
        sh[0] = keep_bytes(s0 != 0u ? funnel16(a0, a1, s0) : a0, nva < onv ? nva : onv);
        sh[1] = keep_bytes(s1 != 0u ? funnel16(b0, b1, s1) : b0, nvb < onv ? nvb : onv);
        sh[2] = keep_bytes(s2 != 0u ? funnel16(c0, c1, s2) : c0, nvc < onv ? nvc : onv);
        rs32_word_fast(sh[0].x, sh[1].x, sh[2].x, sh[3].x, sh[4].x);
        rs32_word_fast(sh[0].y, sh[1].y, sh[2].y, sh[3].y, sh[4].y);
        rs32_word_fast(sh[0].z, sh[1].z, sh[2].z, sh[3].z, sh[4].z);
        rs32_word_fast(sh[0].w, sh[1].w, sh[2].w, sh[3].w, sh[4].w);
        sh[3] = keep_bytes(sh[3], onv);
        sh[4] = keep_bytes(sh[4], onv);
    }
    distribute_store(P, ro, k, Lpad, spr, sh);
}

// A warp takes a RUN of codewords (RUN consecutive ones from a shared counter when DYN, else one at a fixed stride) and
// walks it in two phases:
//   A  every codeword of 64 unmasked columns or more (payloads from 3 KB): its interior in blocks of 64 columns, two
//      columns per lane, all loads in flight before any compute, then its own trailing columns;
//   B  the SHORT codewords of the run, pooled into one column sequence dealt 32 lanes at a time, each lane looking up
//      which codeword its column is in (lane j of the warp holds the geometry of codeword j of the run).
// Why the pooling: walked alone, a payload of 256 B costs a full pass of ~400 warp instructions for 6 useful lanes; a batch
// of such payloads runs several times faster pooled.  In the cfg-4 mix the short codewords carry 3 % of the bytes and the
// pooling does not pay for the coarser unit of work, so RUN = 1 stays the default there.
// The next run is fetched one run ahead, so the counter's latency hides behind the current run.
template <int RUN, bool DYN>
__global__ void __launch_bounds__(kThreads, 3) rs32_crossword_distribute_kernel(const __grid_constant__ CwDistribute P) {
    static_assert(RUN >= 1 && RUN <= 32, "a lane per codeword of the run");
    constexpr uint32_t kFull = 0xffffffffu;
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = (static_cast<uint64_t>(blockIdx.x) * kThreads + threadIdx.x) >> 5;
    const uint64_t nwarps = (static_cast<uint64_t>(gridDim.x) * kThreads) >> 5;
    auto take = [&]() -> uint64_t {
        unsigned long long v = 0;
        if (lane == 0u) v = atomicAdd(P.next_cw, static_cast<unsigned long long>(RUN));
        return __shfl_sync(kFull, v, 0);
    };
    auto shfl64 = [&](uint64_t v, uint32_t from) -> uint64_t {
        const uint32_t lo = __shfl_sync(kFull, static_cast<uint32_t>(v), from), hi = __shfl_sync(kFull, static_cast<uint32_t>(v >> 32), from);
        return (static_cast<uint64_t>(hi) << 32) | lo;
    };
    // column bookkeeping of a codeword of `len` bytes: shard length, columns, unmasked columns, columns phase A covers
    auto cols_of = [](uint32_t len, uint32_t &L, uint32_t &vpc, uint32_t &fast_cols, uint32_t &done) {
        L = (len + 2u) / 3u;
        vpc = ((L + 31u) >> 5) << 1;                       // 16-byte columns of a slot: the slot pitch is round_up(L, 32)
        fast_cols = len >= 2u * L ? (((len - 2u * L) < L ? (len - 2u * L) : L) / 16u) : 0u;
        done = fast_cols & ~63u;
    };
    uint64_t base = DYN ? take() : warp * RUN, ahead = DYN ? take() : (warp + nwarps) * RUN;
    while (base < P.n) {
        const uint64_t rb = base;
        base = ahead;
        ahead = DYN ? take() : ahead + nwarps * RUN;
        // lane j < RUN holds codeword rb + j: one gather of the four geometry arrays per run
        uint32_t m_len = 0, m_spr = 0;
        uint64_t m_off = 0, m_ro = 0;
        if (lane < static_cast<uint32_t>(RUN) && rb + lane < P.n) {
            m_len = __ldg(P.data_len + rb + lane); m_spr = __ldg(P.spr + rb + lane);
            m_off = __ldg(P.data_off + rb + lane); m_ro = __ldg(P.rep_off + rb + lane);
        }
        uint32_t mL, mvpc, mfast, mdone;
        cols_of(m_len, mL, mvpc, mfast, mdone);
        uint32_t pool_end = mdone == 0u ? mvpc : 0u;       // inclusive prefix sum of the pooled column counts over the run
#pragma unroll
        for (uint32_t d = 1; d < static_cast<uint32_t>(RUN); d <<= 1) {
            const uint32_t up = __shfl_up_sync(kFull, pool_end, d);
            if (lane >= d) pool_end += up;
        }
        const uint32_t pool_total = __shfl_sync(kFull, pool_end, RUN - 1);
        // ---- phase A ----
#pragma unroll 1
        for (uint32_t j = 0; j < static_cast<uint32_t>(RUN); ++j) {
            const uint32_t len = __shfl_sync(kFull, m_len, j);
            uint32_t L, vpc, fast_cols, done;
            cols_of(len, L, vpc, fast_cols, done);
            if (done == 0u) continue;                      // uniform: every lane sees the same len
            const uint32_t spr = __shfl_sync(kFull, m_spr, j);
            const uint8_t *pay = P.data + shfl64(m_off, j);
            const uint64_t ro = shfl64(m_ro, j);
            const uint32_t Lpad = vpc * 16u;
            const uint32_t s0 = static_cast<uint32_t>(reinterpret_cast<uintptr_t>(pay)) & 15u;
            const uint8_t *src = pay - s0;
            const uint32_t s1 = (s0 + L) & 15u, s2 = (s0 + 2u * L) & 15u;
            for (uint32_t v0 = 0; v0 < done; v0 += 64u) {
                const uint32_t k = (v0 + lane) * 16u, k2 = k + 512u;
                Raw6 r1, r2;
                rs32_issue_loads(src, k, s0 + L + k - s1, s0 + 2u * L + k - s2, s0, s1, s2, r1);
                rs32_issue_loads(src, k2, s0 + L + k2 - s1, s0 + 2u * L + k2 - s2, s0, s1, s2, r2);
                uint4 sh[5];
                rs32_shards_from_raw(r1, s0, s1, s2, sh);
                distribute_store(P, ro, k, Lpad, spr, sh);
                rs32_shards_from_raw(r2, s0, s1, s2, sh);
                distribute_store(P, ro, k2, Lpad, spr, sh);
            }
            // its own < 64 + 2 trailing columns: whole passes are unmasked or masked together
            for (uint32_t v0 = done; v0 < vpc; v0 += 32u)
                if (v0 + lane < vpc) cw_column(P, src, len, L, v0 + lane, s0, s1, s2, v0 + 32u <= fast_cols, ro, Lpad, spr);
        }
        // ---- phase B ----
#pragma unroll 1
        for (uint32_t t0 = 0; t0 < pool_total; t0 += 32u) {
            const uint32_t t = t0 + lane;
            uint32_t mine = 0;                             // how many codewords of the run end at or before pooled column t
#pragma unroll
            for (uint32_t j = 0; j + 1 < static_cast<uint32_t>(RUN); ++j) mine += __shfl_sync(kFull, pool_end, j) <= t ? 1u : 0u;
            const uint32_t len = __shfl_sync(kFull, m_len, mine), spr = __shfl_sync(kFull, m_spr, mine);
            const uint32_t end = __shfl_sync(kFull, pool_end, mine);
            const uint64_t off = shfl64(m_off, mine), ro = shfl64(m_ro, mine);
            if (t < pool_total) {
                uint32_t L, vpc, fast_cols, done;
                cols_of(len, L, vpc, fast_cols, done);
                const uint32_t v = vpc - (end - t);        // column of codeword `mine`, all of whose columns are pooled
                const uint8_t *pay = P.data + off;
                const uint32_t s0 = static_cast<uint32_t>(reinterpret_cast<uintptr_t>(pay)) & 15u;
                cw_column(P, pay - s0, len, L, v, s0, (s0 + L) & 15u, (s0 + 2u * L) & 15u, v < fast_cols, ro, vpc * 16u, spr);
            }
        }
    }
}

// General Crossword distribute: any code with d <= 8, p <= 8 and any population n with T = d + p a multiple of n
// (crossword/mod.rs:805-830).  Replica r holds shards {(r*dj + k) mod T : k < spr}, dj = T / n (balanced round-robin,
// crossword/mod.rs:866-888).  A warp per codeword; every column's T shards live in registers (d source vectors, p Horner
// rows with the coder's run-time masks) and each is stored into the slot of every replica that holds it.
struct CwDistributeGen {
    const uint8_t *data;
    const uint64_t *data_off;
    const uint32_t *data_len;
    const uint8_t *spr;
    const uint64_t *rep_off;
    uint8_t *rep[16];
    uint64_t n;
    uint32_t d, p, n_rep, dj;
    const uint32_t *prog;      // encode program: ProgHeader + splats + Horner masks
};

template <int CODE, int D, int... Js>
__device__ __forceinline__ void static_parity_all(const uint4 (&x)[D], uint4 (&par)[kMaxP], int onv, std::integer_sequence<int, Js...>) {
    ((par[Js] = keep_bytes(static_parity_row<CODE, Js, D>(x), onv)), ...);
}

// CODE != kCodeGeneric: the coder's matrix is one of the compile-time cluster codes (RS(2,1), (4,3), (5,4), (4,2), (3,1) --
// the 3-, 7- and 9-replica deployments), parity rows are unrolled from the table instead of read from the mask program
template <int D, int CODE>
__global__ void __launch_bounds__(kThreads, 2) crossword_distribute_generic_kernel(const __grid_constant__ CwDistributeGen P) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = (static_cast<uint64_t>(blockIdx.x) * kThreads + threadIdx.x) >> 5;
    const uint64_t nwarps = (static_cast<uint64_t>(gridDim.x) * kThreads) >> 5;
    const int d = static_cast<int>(P.d), p = static_cast<int>(P.p);
    const uint32_t T = P.d + P.p;
    const ProgHeader *hdr = reinterpret_cast<const ProgHeader *>(P.prog);
    const uint32_t *hmask = P.prog + sizeof(ProgHeader) / 4 + p * d * 8;
    for (uint64_t g = warp; g < P.n; g += nwarps) {
        const uint32_t len = __ldg(P.data_len + g);
        if (len == 0u) continue;
        const uint32_t spr = __ldg(P.spr + g);
        const uint32_t L = (len + P.d - 1u) / P.d, vpc = ((L + 31u) >> 5) << 1, Lpad = vpc * 16u;   // slot pitch round_up(L, 32)
        const uint8_t *src = P.data + __ldg(P.data_off + g);
        const uint64_t ro = __ldg(P.rep_off + g);
        for (uint32_t v = lane; v < vpc; v += 32u) {
            const uint32_t k = v * 16u;
            const int onv = k >= L ? 0 : (L - k > 16u ? 16 : static_cast<int>(L - k));      // 0: the padding column of an odd-length slot
            uint4 x[D], par[kMaxP];
            dev::Raw16 raw[D];
#pragma unroll
            for (int i = 0; i < D; ++i) {
                raw[i].lo = make_uint4(0u, 0u, 0u, 0u); raw[i].hi = raw[i].lo; raw[i].s = 0u;
                if (i < d) {
                    const int64_t rem = static_cast<int64_t>(len) - (static_cast<int64_t>(i) * L + k);
                    const int nv = rem > onv ? onv : (rem < 0 ? 0 : static_cast<int>(rem));
                    raw[i] = dev::raw16_issue(src + static_cast<uint64_t>(i) * L + k, nv);
                }
            }
#pragma unroll
            for (int i = 0; i < D; ++i) {
                const int64_t rem = static_cast<int64_t>(len) - (static_cast<int64_t>(i) * L + k);
                const int nv = rem > onv ? onv : (rem < 0 ? 0 : static_cast<int>(rem));
                x[i] = i < d ? dev::raw16_finish(raw[i], nv) : make_uint4(0u, 0u, 0u, 0u);
            }
            if constexpr (CODE != kCodeGeneric) {
                static_parity_all<CODE>(x, par, onv, std::make_integer_sequence<int, static_code_p(CODE)>{});
            } else {
#pragma unroll
                for (int j = 0; j < kMaxP; ++j)
                    par[j] = j < p ? keep_bytes(horner_row<D>(x, d, hmask + j * d * 8, hdr->top[j]), onv) : make_uint4(0u, 0u, 0u, 0u);
            }
            // shard js goes to replica r's slot kk when (js - r*dj) mod T = kk < spr
            auto place = [&](uint32_t js, const uint4 &val) {
                // kk = (js - r*dj) mod T without a division: js < T and r*dj < T
                uint32_t first = 0;                                   // r * dj
                for (uint32_t r = 0; r < P.n_rep; ++r, first += P.dj) {
                    const uint32_t kk = js >= first ? js - first : js + T - first;
                    if (kk < spr) dev::stg128_cs(P.rep[r] + ro + static_cast<uint64_t>(kk) * Lpad + k, val);
                }
            };
#pragma unroll
            for (int i = 0; i < D; ++i)
                if (i < d) place(static_cast<uint32_t>(i), x[i]);
#pragma unroll
            for (int j = 0; j < kMaxP; ++j)
                if (j < p) place(P.d + static_cast<uint32_t>(j), par[j]);
        }
    }
}

int launch_crossword_distribute(ss_rs_coder *coder, const uint8_t *data, const uint64_t *data_off,
                                const uint32_t *data_len, const uint8_t *spr, const uint64_t *rep_off, uint64_t n,
                                uint8_t *const *replica_logs, uint32_t n_replicas) {
    ss_ctx *ctx = coder->ctx;
    SS_TRY(ctx_bind(ctx));
    const uint32_t T = static_cast<uint32_t>(coder->d + coder->p);
    // crossword/mod.rs:805-830: rs_total_shards must be a multiple of the population
    if (n_replicas == 0 || n_replicas > 16 || T % n_replicas != 0)
        return set_error(SS_ERR_INVALID_ARG, "total shards (%u) must be a multiple of the population (%u <= 16)", T, n_replicas);
    if (n == 0) return SS_OK;
    for (uint32_t r = 0; r < n_replicas; ++r)
        if (replica_logs[r] == nullptr || (reinterpret_cast<uintptr_t>(replica_logs[r]) & 15u))
            return set_error(SS_ERR_INVALID_ARG, "replica log %u is null or not 16-byte aligned", r);
    if (!(coder->is_rs32 && n_replicas == 5) || (coder->variant & 15) == 4) {
        // any other (T, d, n): the general kernel (variant 4 forces it for RS(3,2) / n = 5 as well)
        if (coder->d > 8 || !coder->batch_ok)
            return set_error(SS_ERR_UNSUPPORTED, "crossword distribute needs d <= 8 data shards (coder is %d,%d)", coder->d, coder->p);
        CwDistributeGen Gp;
        Gp.data = data; Gp.data_off = data_off; Gp.data_len = data_len; Gp.spr = spr; Gp.rep_off = rep_off; Gp.n = n;
        Gp.d = static_cast<uint32_t>(coder->d); Gp.p = static_cast<uint32_t>(coder->p); Gp.n_rep = n_replicas; Gp.dj = T / n_replicas;
        Gp.prog = static_cast<const uint32_t *>(coder->enc_prog);
        for (uint32_t r = 0; r < 16; ++r) Gp.rep[r] = r < n_replicas ? replica_logs[r] : nullptr;
        const uint32_t grid = ragged_grid(ctx, n);
        const int sc = ((coder->variant >> 11) & 1) ? kCodeGeneric : coder->static_code;
        SS_TRY(dispatch_code(sc, coder->d, [&](auto DC, auto CC) {
            crossword_distribute_generic_kernel<decltype(DC)::value, decltype(CC)::value><<<grid, kThreads, 0, ctx->stream>>>(Gp);
            return SS_OK;
        }));
        coder->last_kernel = sc != kCodeGeneric ? "crossword_distribute_generic_kernel<static>" : "crossword_distribute_generic_kernel";
        return launched(ctx);
    }
    CwDistribute P;
    P.data = data; P.data_off = data_off; P.data_len = data_len; P.spr = spr; P.rep_off = rep_off; P.n = n;
    for (int r = 0; r < 5; ++r) P.rep[r] = replica_logs[r];
    // variant bits 0-3 (tuning; tools/distribute_ab.py compares them): default = a codeword per warp at a fixed stride;
    // 6 / 7 = runs of 8 / 4 codewords from a shared counter with the short ones pooled -- for the cfg-4 mix a run of long
    // codewords is a coarse unit of work, but batches of payloads under 1 KB run several times faster, for callers that
    // know their batch is like that
    const int vk = coder->variant & 15;
    P.next_cw = reinterpret_cast<unsigned long long *>(ctx->dev_status + 32);
    if (vk != 6 && vk != 7) {
        rs32_crossword_distribute_kernel<1, false><<<ragged_grid(ctx, n), kThreads, 0, ctx->stream>>>(P);
        coder->last_kernel = "rs32_crossword_distribute_kernel<1>";
    } else {
        // one CTA per resident slot (3 per SM at 80 registers), never more warps than runs
        SS_CUDA(cudaMemsetAsync(P.next_cw, 0, sizeof(unsigned long long), ctx->stream));
        const uint64_t run = vk == 7 ? 4 : 8;
        uint64_t ctas = static_cast<uint64_t>(ctx->sm_count) * 3ull;
        const uint64_t need = (n + run * (kThreads / 32) - 1) / (run * (kThreads / 32));
        if (ctas > need) ctas = need;
        if (vk == 7) rs32_crossword_distribute_kernel<4, true><<<static_cast<uint32_t>(ctas), kThreads, 0, ctx->stream>>>(P);
        else rs32_crossword_distribute_kernel<8, true><<<static_cast<uint32_t>(ctas), kThreads, 0, ctx->stream>>>(P);
        coder->last_kernel = vk == 7 ? "rs32_crossword_distribute_kernel<4,dynamic>" : "rs32_crossword_distribute_kernel<8,dynamic>";
    }
    return launched(ctx);
}

// ---- batched encode: launch_rs_encode validates a batch and routes it to one of the four kernel families below ----

// RS(3,2) in the row geometry: the bulk-copy accept kernel (variant bit 18), the segmented row kernel for codewords over
// 256 columns, else the row kernel
static int encode_rs32_row(ss_rs_coder *coder, const EncGeom &g, const TallyArgs *tally, uint32_t len, uint32_t L,
                           uint32_t vpc) {
    ss_ctx *ctx = coder->ctx;
    cudaStream_t st = ctx->stream;
    Enc32Row Rw;
    Rw.data = g.data; Rw.data_stride = g.data_stride; Rw.shard_stride = g.shard_stride;
    for (int j = 0; j < 5; ++j) Rw.plane[j] = out_plane(g, 3, j);
    Rw.n = static_cast<uint32_t>(g.n); Rw.len = len; Rw.L = L; Rw.vpc = vpc;
    const uint32_t lim = (len - 2u * L) < L ? (len - 2u * L) : L;     // bytes of shard 2 inside the payload
    Rw.fast_cols = len >= 2u * L ? lim / 16u : 0u;
    Rw.s1 = L & 15u; Rw.s2 = (2u * L) & 15u;
    Rw.emit_data = ((g.flags & SS_RS_EMIT_DATA) || g.plane_ptrs != nullptr) ? 1u : 0u;
    set_tally(Rw, tally);
    Rw.wait = g.wait;
    // The accept step proper (parity to local planes, no replication) on the bulk-copy kernel: variant bit 18
    // selects it.  It is not the default: on an H100 it measured 2-3 % slower than the row kernel (DESIGN.md 3.1).
    const uint32_t in_bytes = (len + 15u) & ~15u;
    if (vpc <= 256u && !Rw.emit_data && ((coder->variant >> 18) & 1) && g.data_stride >= in_bytes) {
        int smem_sm = 0, smem_blk = 0, smem_rsv = 0;
        SS_CUDA(cudaDeviceGetAttribute(&smem_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, ctx->device));
        SS_CUDA(cudaDeviceGetAttribute(&smem_blk, cudaDevAttrMaxSharedMemoryPerBlockOptin, ctx->device));
        SS_CUDA(cudaDeviceGetAttribute(&smem_rsv, cudaDevAttrReservedSharedMemoryPerBlock, ctx->device));
        Enc32Bulk B;
        B.data = g.data; B.data_stride = g.data_stride; B.par0 = Rw.plane[3]; B.par1 = Rw.plane[4];
        B.shard_stride = g.shard_stride; B.n = Rw.n; B.len = len; B.L = L; B.vpc = vpc;
        B.fast_cols = Rw.fast_cols; B.s1 = Rw.s1; B.s2 = Rw.s2;
        B.in_bytes = in_bytes;
        B.in_pitch = (in_bytes + 48u + 127u) & ~127u;
        set_tally(B, tally);
        // Resident CTAs per SM (variant bits 19-20, tuning): 4 by default.  The SM's shared memory is split
        // evenly between them; each CTA keeps kBulkOut output stages and as many input stages as fit, at most
        // 8 -- at cfg3 (4096 B rows) that is 8 stages, up to 4 x 7 x 4 KB = 112 KB of payload in flight per SM.
        static const uint32_t kCtasPerSm[4] = {4, 2, 3, 6};
        const uint32_t out_bytes = kBulkOut * 2u * vpc * 16u;
        uint32_t cps = kCtasPerSm[(coder->variant >> 19) & 3], nin = 0;
        for (; cps >= 1; --cps) {
            int64_t room = static_cast<int64_t>(smem_sm) / cps - smem_rsv;
            if (room > smem_blk) room = smem_blk;
            room -= kBulkHeader + out_bytes;
            nin = room > 0 ? static_cast<uint32_t>(room / B.in_pitch) : 0u;
            if (nin > 8u) nin = 8u;
            if (nin >= 2u) break;
        }
        if (nin < 2u) return set_error(SS_ERR_UNSUPPORTED, "accept step: no room for two %u-byte stages", B.in_pitch);
        B.nin = nin;
        uint64_t ctas = static_cast<uint64_t>(ctx->sm_count) * cps;
        if (ctas > g.n) ctas = g.n;
        B.chunk = static_cast<uint32_t>((g.n + ctas - 1) / ctas);
        ctas = (g.n + B.chunk - 1) / B.chunk;
        B.interleave = ((coder->variant >> 21) & 1) ? 1u : 0u;       // bit 21 (tuning): interleaved codewords
        const uint32_t smem = kBulkHeader + nin * B.in_pitch + out_bytes;
        SS_CUDA(cudaFuncSetAttribute(rs32_accept_bulk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     static_cast<int>(smem)));
        const uint32_t threads = ((vpc + 31u) & ~31u) + 32u;      // a thread per column + the tally warp
        rs32_accept_bulk_kernel<<<static_cast<uint32_t>(ctas), threads, smem, st>>>(B);
        coder->last_kernel = B.planes ? "rs32_accept_bulk_kernel+tally" : "rs32_accept_bulk_kernel";
        return launched(ctx);
    }
    const uint32_t threads = vpc > 256u ? 256u : ((vpc + 31u) & ~31u);
    if (vpc > 256u) {
        // wide codewords: (codeword, 256-column segment) work items
        const uint64_t items = g.n * ((vpc + 255u) / 256u);
        uint64_t ctas = static_cast<uint64_t>(ctx->sm_count) * 8ull * 16ull;
        if (ctas > items) ctas = items;
        Rw.chunk = 0; Rw.st_mode = static_cast<uint32_t>((coder->variant >> 8) & 3); Rw.rotate = 0; Rw.tally_last = 0;
        if (Rw.emit_data) rs32_encode_row_kernel<true, 256, 4, true><<<static_cast<uint32_t>(ctas), 256, 0, st>>>(Rw);
        else rs32_encode_row_kernel<false, 256, 4, true><<<static_cast<uint32_t>(ctas), 256, 0, st>>>(Rw);
        coder->last_kernel = Rw.planes ? "rs32_encode_row_kernel<segmented>+tally" : "rs32_encode_row_kernel<segmented>";
        return launched(ctx);
    }
    // resident CTAs per SM (2048 threads, 32 CTAs) x a few waves; every CTA strides over codewords
    uint32_t per_sm = 2048u / threads; if (per_sm > 32u) per_sm = 32u;
    const int vr = coder->variant & 15, vchunk = (coder->variant >> 4) & 1, vw = (coder->variant >> 5) & 7;
    static const uint64_t kWaves[8] = {64, 1, 32, 4, 16, 256, 128, 8};   // [0] = default, rest: tuning
    // Local planes (the accept step): by default a CTA per codeword.  The block scheduler then hands codewords
    // out in order, so the whole GPU reads and writes one narrow, advancing window of memory; on an H100 that
    // measured 2.6 % faster than 64 or 256 waves of CTAs striding over the batch (DESIGN.md 3.1).
    const uint64_t waves = (vw == 0 && !Rw.emit_data) ? (1ull << 32) : kWaves[vw];
    uint64_t ctas = static_cast<uint64_t>(ctx->sm_count) * per_sm * waves;
    if (ctas > g.n) ctas = g.n;
    if (ctas > 0x7fffffffull) ctas = 0x7fffffffull;
    Rw.chunk = 0;
    Rw.st_mode = static_cast<uint32_t>((coder->variant >> 8) & 3);
    Rw.rotate = ((coder->variant >> 10) & 1) ? 0u : 1u;
    // local planes: the tally goes after the CTA's codeword, so its first loads are the payload's
    Rw.tally_last = Rw.emit_data ? 0u : 1u;
    if (vchunk) { Rw.chunk = static_cast<uint32_t>((g.n + ctas - 1) / ctas); ctas = (g.n + Rw.chunk - 1) / Rw.chunk; }
    const uint32_t grid = static_cast<uint32_t>(ctas);
    // Register budget: 40/thread (12 CTAs of <= 128 threads per SM; the kernel needs ~47 unconstrained and fits
    // 40 without spilling); a CTA per codeword for local planes, 64 waves of CTAs otherwise.  The other budgets
    // (variant bits 0-3: 3 = 32 regs, 6 = 64, 7 = 56) and wave counts stay selectable for tuning.
    if (threads > 128) {
        if (Rw.emit_data) rs32_encode_row_kernel<true, 256, 4><<<grid, threads, 0, st>>>(Rw);
        else rs32_encode_row_kernel<false, 256, 4><<<grid, threads, 0, st>>>(Rw);
    } else if (Rw.emit_data) rs32_encode_row_kernel<true, 128, 8><<<grid, threads, 0, st>>>(Rw);
    else if (vr == 3) rs32_encode_row_kernel<false, 128, 16><<<grid, threads, 0, st>>>(Rw);   // 32 regs
    else if (vr == 6) rs32_encode_row_kernel<false, 128, 8><<<grid, threads, 0, st>>>(Rw);    // 64 regs cap
    else if (vr == 7) rs32_encode_row_kernel<false, 128, 9><<<grid, threads, 0, st>>>(Rw);    // 56 regs cap
    else rs32_encode_row_kernel<false, 128, 12, false, true><<<grid, threads, 0, st>>>(Rw);    // 40 regs, L2 prefetch
    coder->last_kernel = Rw.planes ? "rs32_encode_row_kernel+tally" : "rs32_encode_row_kernel";
    return launched(ctx);
}

// Other codes with d <= 8 in the row geometry: the packed or the row layout, each as a compile-time cluster code, the
// coder's own NVRTC specialisation or with run-time coefficient masks
static int encode_horner_row(ss_rs_coder *coder, const EncGeom &g, const TallyArgs *tally, uint32_t len, uint32_t L,
                             uint32_t vpc) {
    ss_ctx *ctx = coder->ctx;
    cudaStream_t st = ctx->stream;
    const int d = coder->d, p = coder->p;
    EncRowGen Rg;
    Rg.data = g.data; Rg.data_stride = g.data_stride;
    for (int j = 0; j < 16; ++j) Rg.plane[j] = j < d + p ? out_plane(g, d, j) : nullptr;
    Rg.emit_data = ((g.flags & SS_RS_EMIT_DATA) || g.plane_ptrs != nullptr) ? 1u : 0u;
    Rg.wait = g.wait;
    Rg.shard_stride = g.shard_stride; Rg.n = static_cast<uint32_t>(g.n); Rg.len = len; Rg.L = L; Rg.vpc = vpc;
    // columns whose every source window lies inside the payload and whose output vector is complete
    const uint64_t last_shard_bytes = static_cast<uint64_t>(len) >= static_cast<uint64_t>(d - 1) * L
                                          ? static_cast<uint64_t>(len) - static_cast<uint64_t>(d - 1) * L : 0;
    Rg.fast_cols = static_cast<uint32_t>((last_shard_bytes < L ? last_shard_bytes : L) / 16u);
    Rg.d = static_cast<uint32_t>(d); Rg.p = static_cast<uint32_t>(p);
    Rg.hmT8 = static_cast<const uint32_t *>(coder->enc_hmT8);
    for (int j = 0; j < kMaxP; ++j) Rg.top[j] = coder->enc_top[j];
    set_tally(Rg, tally);
    // which flavour of the kernels: a compile-time cluster code, the coder's own NVRTC specialisation (any other
    // matrix; compiled on first use), or run-time coefficient masks (variant bit 11 forces them, bit 17 skips NVRTC)
    int sc = ((coder->variant >> 11) & 1) ? kCodeGeneric : coder->static_code;
    const bool jit_allowed = sc == kCodeGeneric && !((coder->variant >> 11) & 1) && !((coder->variant >> 17) & 1);
    auto launch_jit = [&](int which, uint32_t grid_x, uint32_t block_x) -> int {
        void *args[] = {&Rg};
        SS_CUDA(cudaLaunchKernel(reinterpret_cast<const void *>(coder->jit_kernel[which]), dim3(grid_x), dim3(block_x), args, 0, st));
        return SS_OK;
    };
    // Packed flavour when the one-codeword-per-pass layout would idle or mask a good part of the lanes
    // (bit 13 forces it off, bit 14 forces it on).
    const uint32_t fc = Rg.fast_cols;
    const uint32_t row_threads = vpc > 256u ? 256u : ((vpc + 31u) & ~31u);    // wider codewords: 256-column segments
    bool packed = (fc != vpc || row_threads != vpc) && vpc <= 256u;
    if ((coder->variant >> 13) & 1) packed = false;
    if ((coder->variant >> 14) & 1) packed = true;
    // software-pipelined main loop: always when every shard is 16-byte aligned; bit 15 selects it for unaligned too
    const bool pipe = (L & 15u) == 0u || ((coder->variant >> 15) & 1);
    if (jit_allowed) {
        // the one instance this geometry needs (compiled by NVRTC on first use, ~1 s; then cached in the coder)
        const int which = packed ? ((L & 15u) == 0u ? 2 : pipe ? 3 : 4) : (row_threads > 128u ? 1 : 0);
        if (jit_ensure(coder, which) == SS_OK) sc = kCodeJit;
    }
    if (packed) {
        // threads: the multiple of 32 (<= 256) that wastes the fewest lanes; ties go to the larger CTA
        uint32_t T = 256, m = fc ? 256u / fc : 0u;
        if (fc) {
            double best = -1.0;
            for (uint32_t t = 256; t >= 64; t -= 32) {
                const uint32_t mm = t / fc;
                const double eff = static_cast<double>(mm * fc) / t;
                if (eff > best + 1e-9) { best = eff; T = t; m = mm; }
            }
        }
        Rg.pack_m = m;
        Rg.ntail = vpc - fc;
        const uint64_t tail_items = g.n * Rg.ntail;
        const uint64_t tail_ctas = (tail_items + T - 1) / T;
        uint64_t main_ctas = 0;
        if (m) {
            const uint32_t dcap = d <= 2 ? 2 : d == 3 ? 3 : d == 4 ? 4 : d <= 6 ? 6 : 8;      // dispatch_d's capacity
            const uint32_t dt = sc != kCodeGeneric ? static_cast<uint32_t>(d) : dcap;       // static and NVRTC kernels are exact-width
            const uint32_t reg_need = 4u * dt + ((L & 15u) == 0u ? 4u * dt : 8u * dt - 4u) + 22u;
            uint32_t rb = 65536u / (256u * reg_need); rb = rb > 6u ? 6u : (rb < 1u ? 1u : rb);
            if (!pipe) rb = dt <= 3 ? 6u : dt <= 5 ? 5u : dt <= 6 ? 4u : 3u;
            const uint32_t resident_threads = 256u * rb;
            main_ctas = static_cast<uint64_t>(ctx->sm_count) * (resident_threads / T) * 64ull;
            const uint64_t need = (g.n + m - 1) / m;
            if (main_ctas > need) main_ctas = need;
        }
        if (tail_ctas + main_ctas <= 0x7fffffffull) {
            Rg.tail_ctas = static_cast<uint32_t>(tail_ctas);
            const uint32_t grid = static_cast<uint32_t>(tail_ctas + main_ctas);
            if (sc == kCodeJit) SS_TRY(launch_jit((L & 15u) == 0u ? 2 : pipe ? 3 : 4, grid, T));
            else SS_TRY(dispatch_code(sc, d, [&](auto DC, auto CC) {
                constexpr int kD = decltype(DC)::value, kC = decltype(CC)::value;
                if ((L & 15u) == 0u) horner_encode_packed_kernel<kD, kC, true, true><<<grid, T, 0, st>>>(Rg);
                else if (pipe) horner_encode_packed_kernel<kD, kC, false, true><<<grid, T, 0, st>>>(Rg);
                else horner_encode_packed_kernel<kD, kC, false, false><<<grid, T, 0, st>>>(Rg);
                return SS_OK;
            }));
            if (sc == kCodeJit)
                coder->last_kernel = Rg.planes ? "horner_encode_packed_kernel<nvrtc>+tally" : "horner_encode_packed_kernel<nvrtc>";
            else if (sc != kCodeGeneric)
                coder->last_kernel = Rg.planes ? "horner_encode_packed_kernel<static code>+tally" : "horner_encode_packed_kernel<static code>";
            else
                coder->last_kernel = Rg.planes ? "horner_encode_packed_kernel+tally" : "horner_encode_packed_kernel";
            return launched(ctx);
        }
    }
    Rg.pack_m = 0; Rg.tail_ctas = 0; Rg.ntail = 0;
    const uint32_t threads = row_threads;
    if (sc == kCodeJit && jit_ensure(coder, threads > 128u ? 1 : 0) != SS_OK) sc = kCodeGeneric;   // (packed grid did not fit)
    uint32_t per_sm = 2048u / threads; if (per_sm > 32u) per_sm = 32u;
    uint64_t ctas = static_cast<uint64_t>(ctx->sm_count) * per_sm * 64ull;
    if (ctas > g.n) ctas = g.n;
    const uint32_t grid = static_cast<uint32_t>(ctas);
    // register budget (variant bits 0-3): threads <= 128: 0 = 12 CTAs/SM (40 regs), 2 = 10 (48), 3 = 8 (64), 4 = 6 (80)
    const int vbits = coder->variant & 15;
    if (sc == kCodeJit) SS_TRY(launch_jit(threads > 128 ? 1 : 0, grid, threads));
    else SS_TRY(dispatch_code(sc, d, [&](auto DC, auto CC) {
        constexpr int kD = decltype(DC)::value, kC = decltype(CC)::value;
        // default budget by width: spill-free at 40 registers up to d = 4, 48 for 5, 64 for 6, 80 beyond
        const int vdef = kD <= 4 ? 0 : kD == 5 ? 2 : kD == 6 ? 3 : 4;
        const int vb = (vbits >= 2 && vbits <= 4) ? vbits : vdef;      // other values select other kernels' knobs
        if (threads > 128) horner_encode_row_kernel<kD, kC, 256, 3><<<grid, threads, 0, st>>>(Rg);
        else if (vb == 2) horner_encode_row_kernel<kD, kC, 128, 10><<<grid, threads, 0, st>>>(Rg);
        else if (vb == 3) horner_encode_row_kernel<kD, kC, 128, 8><<<grid, threads, 0, st>>>(Rg);
        else if (vb == 4) horner_encode_row_kernel<kD, kC, 128, 6><<<grid, threads, 0, st>>>(Rg);
        else horner_encode_row_kernel<kD, kC, 128, 12><<<grid, threads, 0, st>>>(Rg);
        return SS_OK;
    }));
    if (sc == kCodeJit)
        coder->last_kernel = Rg.planes ? "horner_encode_row_kernel<nvrtc>+tally" : "horner_encode_row_kernel<nvrtc>";
    else if (sc != kCodeGeneric)
        coder->last_kernel = Rg.planes ? "horner_encode_row_kernel<static code>+tally" : "horner_encode_row_kernel<static code>";
    else
        coder->last_kernel = Rg.planes ? "horner_encode_row_kernel+tally" : "horner_encode_row_kernel";
    return launched(ctx);
}

// Any uniform geometry, a thread per flat column index; chunked so that a launch's n_chunk * vpc fits in 32 bits.  The
// fused tally rides on the first launch.
static int encode_flat(ss_rs_coder *coder, const EncGeom &g, const TallyArgs *tally, uint32_t len, uint32_t L,
                       uint32_t vpc) {
    ss_ctx *ctx = coder->ctx;
    const int d = coder->d, p = coder->p;
    const uint64_t max_cw = vpc ? (0xffffff00ull / vpc) : g.n;
    uint64_t done = 0;
    bool tally_pending = tally != nullptr;
    do {
        const uint64_t nc = (g.n - done) < max_cw ? (g.n - done) : max_cw;
        EncUniform E;
        E.data = g.data + done * g.data_stride;
        E.data_stride = g.data_stride;
        E.len = len; E.L = L; E.vpc = vpc;
        E.parity = g.parity + done * g.shard_stride;
        E.plane_stride = g.plane_stride; E.shard_stride = g.shard_stride;
        E.n = nc;
        E.total = static_cast<uint32_t>(nc * vpc);
        E.padded = ((g.flags & SS_RS_OUT_PADDED16) ? 1u : 0u) | ((g.flags & SS_RS_EMIT_DATA) ? 2u : 0u);
        set_tally(E, tally_pending ? tally : nullptr);
        E.G = 0;
        uint64_t threads = E.total;
        if (tally_pending) {
            if (tally->G > 0xffffff00ull) return set_error(SS_ERR_INVALID_ARG, "too many groups for one fused launch");
            E.G = tally->G;
            if (threads < tally->G) threads = tally->G;
            tally_pending = false;
        }
        if (threads == 0) break;
        const uint32_t grid = static_cast<uint32_t>((threads + kThreads - 1) / kThreads);
        const uint32_t *prog = static_cast<const uint32_t *>(coder->enc_prog);
        if (coder->is_rs32) {
            rs32_encode_uniform_kernel<<<grid, kThreads, 0, ctx->stream>>>(E);
            coder->last_kernel = E.planes ? "rs32_encode_uniform_kernel+tally" : "rs32_encode_uniform_kernel";
        } else if (d <= 8 && (coder->variant & 15) != 5) {
            SS_TRY(dispatch_d(d, [&](auto DC) {
                horner_encode_uniform_kernel<decltype(DC)::value><<<grid, kThreads, 0, ctx->stream>>>(E, prog, d, p);
                return SS_OK;
            }));
            coder->last_kernel = "horner_encode_uniform_kernel";
        } else {
            SS_TRY(dispatch_p(p, [&](auto PC) {
                generic_encode_uniform_kernel<decltype(PC)::value><<<grid, kThreads, 0, ctx->stream>>>(E, prog, d, p);
                return SS_OK;
            }));
            coder->last_kernel = "generic_encode_uniform_kernel";
        }
        SS_TRY(launched(ctx));
        done += nc;
    } while (done < g.n);
    return SS_OK;
}

// Ragged batches, a warp per codeword; the fused tally is a launch of its own
static int encode_ragged(ss_rs_coder *coder, const EncGeom &g, const TallyArgs *tally) {
    ss_ctx *ctx = coder->ctx;
    const int d = coder->d, p = coder->p;
    if (g.n == 0) return SS_OK;
    if (g.data_len == nullptr || g.par_off == nullptr)
        return set_error(SS_ERR_INVALID_ARG, "ragged encode needs data_off, data_len and par_off");
    EncRagged E;
    E.data = g.data; E.data_off = g.data_off; E.data_len = g.data_len;
    E.parity = g.parity; E.plane_stride = g.plane_stride; E.par_off = g.par_off;
    E.n = g.n; E.padded = ((g.flags & SS_RS_OUT_PADDED16) ? 1u : 0u) | ((g.flags & SS_RS_EMIT_DATA) ? 2u : 0u);
    const uint32_t grid = ragged_grid(ctx, g.n);
    const uint32_t *prog = static_cast<const uint32_t *>(coder->enc_prog);
    if (coder->is_rs32) {
        rs32_encode_ragged_kernel<<<grid, kThreads, 0, ctx->stream>>>(E);
        coder->last_kernel = "rs32_encode_ragged_kernel";
    } else if (d <= 8 && (coder->variant & 15) != 5) {
        SS_TRY(dispatch_d(d, [&](auto DC) {
            horner_encode_ragged_kernel<decltype(DC)::value><<<grid, kThreads, 0, ctx->stream>>>(E, prog, d, p);
            return SS_OK;
        }));
        coder->last_kernel = "horner_encode_ragged_kernel";
    } else {
        SS_TRY(dispatch_p(p, [&](auto PC) {
            generic_encode_ragged_kernel<decltype(PC)::value><<<grid, kThreads, 0, ctx->stream>>>(E, prog, d, p);
            return SS_OK;
        }));
        coder->last_kernel = "generic_encode_ragged_kernel";
    }
    SS_TRY(launched(ctx));
    if (tally == nullptr) return SS_OK;
    return launch_tally_planes(ctx, tally->planes, tally->R, tally->G, tally->threshold, tally->committed, tally->commit_bar);
}

int launch_rs_encode(ss_rs_coder *coder, const EncGeom &g, const TallyArgs *tally) {
    SS_TRY(ctx_bind(coder->ctx));
    if (!coder->batch_ok)
        return set_error(SS_ERR_UNSUPPORTED, "batched encode needs d <= %d, p <= %d (coder is %d,%d)", kMaxD,
                         kMaxP, coder->d, coder->p);
    const bool padded = (g.flags & SS_RS_OUT_PADDED16) != 0u;
    if (padded && ((reinterpret_cast<uintptr_t>(g.parity) | g.plane_stride) & 15u))
        return set_error(SS_ERR_INVALID_ARG, "SS_RS_OUT_PADDED16 needs 16-byte aligned parity base and plane_stride");
    if (tally != nullptr && tally->planes == nullptr) tally = nullptr;     // no ack planes: nothing to tally
    if (g.data_off != nullptr) return encode_ragged(coder, g, tally);

    // uniform geometry
    const uint32_t len = g.uni_len;
    if ((len == 0u || g.n == 0u) && tally == nullptr) return SS_OK;
    if (len >= 0x7fffffffu) return set_error(SS_ERR_INVALID_ARG, "data_len too large");
    const uint32_t d = static_cast<uint32_t>(coder->d);
    const uint32_t L = len == 0u ? 0u : (len + d - 1u) / d;
    const uint32_t vpc = (L + 15u) >> 4;
    if (padded && (g.shard_stride & 15u))
        return set_error(SS_ERR_INVALID_ARG, "SS_RS_OUT_PADDED16 needs shard_stride %% 16 == 0");
    if (padded && g.shard_stride < static_cast<uint64_t>(vpc) * 16u)
        return set_error(SS_ERR_INVALID_ARG, "shard_stride %llu < padded shard length %u",
                         (unsigned long long)g.shard_stride, vpc * 16u);
    // The row kernels take 16-byte aligned payload rows into padded shard slots, codewords of at least one column,
    // a batch whose size fits 32 bits, and a fused tally over exactly the batch's groups.  Variant bits 0-3 = 1 select
    // the flat kernels instead, 5 the bit-plane ones.
    const int vk = coder->variant & 15;
    const bool row_geometry = padded && vpc >= 1 && g.n <= 0xffffffffull &&
                              ((reinterpret_cast<uintptr_t>(g.data) | g.data_stride) & 15u) == 0u &&
                              (tally == nullptr || tally->G == g.n);
    const bool rs32_row = coder->is_rs32 && vk != 1 && row_geometry;
    const bool horner_row = !coder->is_rs32 && d <= 8 && coder->enc_hmT8 != nullptr && vk != 5 && vk != 1 && row_geometry;
    if (rs32_row) return encode_rs32_row(coder, g, tally, len, L, vpc);
    if (horner_row) return encode_horner_row(coder, g, tally, len, L, vpc);
    return encode_flat(coder, g, tally, len, L, vpc);
}

int launch_rs_reconstruct(ss_rs_coder *coder, uint8_t *shards, uint64_t plane_stride, const uint64_t *off,
                          const uint32_t *data_len, const uint32_t *present, uint64_t n, int data_only,
                          int32_t *status, uint32_t flags) {
    ss_ctx *ctx = coder->ctx;
    SS_TRY(ctx_bind(ctx));
    if (!coder->batch_ok || !coder->dec_ok)
        return set_error(SS_ERR_UNSUPPORTED, "batched reconstruct needs d+p <= 12 (coder is %d,%d)", coder->d, coder->p);
    if (n == 0) return SS_OK;
    const bool padded = (flags & SS_RS_OUT_PADDED16) != 0u;
    if (padded && ((reinterpret_cast<uintptr_t>(shards) | plane_stride) & 15u))
        return set_error(SS_ERR_INVALID_ARG, "SS_RS_OUT_PADDED16 needs 16-byte aligned shard base and plane_stride");
    DecArgs A;
    A.shards = shards; A.plane_stride = plane_stride; A.off = off; A.data_len = data_len; A.present = present;
    A.n = n; A.status = status;
    A.progs = static_cast<const uint8_t *>(data_only ? coder->dec_progs_data : coder->dec_progs);
    A.prog_stride = static_cast<uint32_t>(coder->prog_stride);
    A.pattern_mask = (1u << (coder->d + coder->p)) - 1u;
    A.d = coder->d;
    A.padded = padded ? 1u : 0u;
    A.hmask_off = static_cast<uint32_t>(coder->p * coder->d * 8);
    A.need_mask = data_only ? ((1u << coder->d) - 1u) : A.pattern_mask;
    const uint32_t grid = ragged_grid(ctx, n);
    A.fast_progs = static_cast<const uint8_t *>(data_only ? coder->fast_progs_data : coder->fast_progs);
    A.fast_stride = static_cast<uint32_t>(coder->fast_stride);
    A.fast_bytes = static_cast<uint32_t>(coder->fast_stride << (coder->d + coder->p));
    if (coder->d <= 4 && A.fast_progs != nullptr && (coder->variant & 15) != 5 && (coder->variant & 15) != 8) {
        const bool smem = A.fast_bytes <= 40u * 1024u;
        const size_t sb = smem ? A.fast_bytes : 0;
        const bool pair = A.padded && ((coder->variant >> 16) & 1);    // bit 16: two columns per lane and pass
        auto small = [&](auto DC) {
            constexpr int kD = decltype(DC)::value;
            if (smem && pair) rs_reconstruct_small_kernel<kD, true, true, true><<<grid, kThreads, sb, ctx->stream>>>(A);
            else if (smem && A.padded) rs_reconstruct_small_kernel<kD, true, true, false><<<grid, kThreads, sb, ctx->stream>>>(A);
            else if (smem) rs_reconstruct_small_kernel<kD, true, false, false><<<grid, kThreads, sb, ctx->stream>>>(A);
            else if (pair) rs_reconstruct_small_kernel<kD, false, true, true><<<grid, kThreads, 0, ctx->stream>>>(A);
            else if (A.padded) rs_reconstruct_small_kernel<kD, false, true, false><<<grid, kThreads, 0, ctx->stream>>>(A);
            else rs_reconstruct_small_kernel<kD, false, false, false><<<grid, kThreads, 0, ctx->stream>>>(A);
        };
        if (coder->d <= 2) small(std::integral_constant<int, 2>{});
        else if (coder->d == 3) small(std::integral_constant<int, 3>{});
        else small(std::integral_constant<int, 4>{});
        coder->last_kernel = smem ? "rs_reconstruct_small_kernel(smem programs)" : "rs_reconstruct_small_kernel";
    } else if (coder->d <= 8 && (coder->variant & 15) != 5) {
        SS_TRY(dispatch_d(coder->d, [&](auto DC) {
            horner_reconstruct_kernel<decltype(DC)::value><<<grid, kThreads, 0, ctx->stream>>>(A);
            return SS_OK;
        }));
        coder->last_kernel = "horner_reconstruct_kernel";
    } else {
        SS_TRY(dispatch_p(coder->p, [&](auto PC) {
            generic_reconstruct_kernel<decltype(PC)::value><<<grid, kThreads, 0, ctx->stream>>>(A);
            return SS_OK;
        }));
        coder->last_kernel = "generic_reconstruct_kernel";
    }
    return launched(ctx);
}

int launch_rs_reconstruct_uniform(ss_rs_coder *coder, uint8_t *shards, uint64_t plane_stride, uint64_t shard_stride,
                                  uint32_t data_len, const uint32_t *present, uint64_t n, int data_only, int32_t *status) {
    ss_ctx *ctx = coder->ctx;
    SS_TRY(ctx_bind(ctx));
    if (n == 0) return SS_OK;
    if (data_len == 0) return set_error(SS_ERR_INVALID_ARG, "null codewords cannot be reconstructed (rscoding.rs:495-497)");
    const uint32_t d = static_cast<uint32_t>(coder->d);
    const uint32_t L = (data_len + d - 1u) / d, vpc = (L + 15u) >> 4;
    if (((reinterpret_cast<uintptr_t>(shards) | plane_stride | shard_stride) & 15u) || shard_stride < static_cast<uint64_t>(vpc) * 16u)
        return set_error(SS_ERR_INVALID_ARG, "uniform reconstruct needs 16-byte aligned, padded shard slots (shard_stride >= round_up(L,16))");
    if (coder->is_rs32 && (coder->variant & 15) != 8 && (coder->variant & 15) != 5 && n <= 0xffffffffull) {
        Dec32Row P;
        P.shards = shards; P.plane_stride = plane_stride; P.shard_stride = shard_stride; P.present = present; P.status = status;
        P.n = static_cast<uint32_t>(n); P.L = L; P.vpc = vpc;
        uint32_t threads = (vpc + 31u) & ~31u;
        if (threads > 256u) threads = 256u;
        uint32_t per_sm = 2048u / threads; if (per_sm > 32u) per_sm = 32u;
        static const uint64_t kWaves[8] = {16, 1, 32, 4, 64, 256, 128, 8};   // variant bits 5-7 (tuning); [0] = default
        uint64_t ctas = static_cast<uint64_t>(ctx->sm_count) * per_sm * kWaves[(coder->variant >> 5) & 7];
        if (ctas > n) ctas = n;
        const uint32_t grid = static_cast<uint32_t>(ctas);
        if (threads > 128u) {
            if (data_only) rs32_reconstruct_row_kernel<true, 256, 5><<<grid, threads, 0, ctx->stream>>>(P);
            else rs32_reconstruct_row_kernel<false, 256, 5><<<grid, threads, 0, ctx->stream>>>(P);
        } else {
            if (data_only) rs32_reconstruct_row_kernel<true, 128, 12><<<grid, threads, 0, ctx->stream>>>(P);
            else rs32_reconstruct_row_kernel<false, 128, 12><<<grid, threads, 0, ctx->stream>>>(P);
        }
        coder->last_kernel = "rs32_reconstruct_row_kernel";
        return launched(ctx);
    }
    // any other code: the per-pattern program kernels over synthesised offsets
    void *scr = nullptr;
    SS_TRY(ctx_scratch(ctx, n * 12 + 256, &scr));
    uint64_t *off = static_cast<uint64_t *>(scr);
    uint32_t *len = reinterpret_cast<uint32_t *>(off + n);
    uint64_t mg = (n + 255) / 256; if (mg > 4096) mg = 4096;
    uniform_meta_kernel<<<static_cast<uint32_t>(mg), 256, 0, ctx->stream>>>(off, len, n, shard_stride, data_len);
    SS_TRY(launched(ctx));
    return launch_rs_reconstruct(coder, shards, plane_stride, off, len, present, n, data_only, status, SS_RS_OUT_PADDED16);
}

}  // namespace ssb
