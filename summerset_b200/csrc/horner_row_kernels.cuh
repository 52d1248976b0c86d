// horner_row_kernels.cuh -- the "row" and "packed" encode kernels for any Reed-Solomon code with d <= 8 data shards.
//
// This header is compiled twice:
//   * by nvcc into the library (rs_kernels.cu), instantiated for the compile-time cluster codes of static_codes.hpp
//     (RS(2,1), RS(4,3), RS(5,4), RS(4,2), RS(3,1)) and for CODE = kCodeGeneric (coefficient masks read at run time);
//   * at RUN time by NVRTC (jit.cu), once per coder whose matrix is none of the compile-time tables: the coder's parity
//     rows are #defined into the translation unit (SS_JIT_D / SS_JIT_P / SS_JIT_COEFS -> CODE = kCodeJit), so an
//     arbitrary code -- Crossword's RS(6,4), RS(9,6) ... (crossword/mod.rs:805-830) -- runs the SAME fully unrolled
//     kernels as the cluster codes, with its coefficients as instruction immediates instead of masks fetched per bit.
// It therefore depends only on device_common.cuh and static_codes.hpp and uses no host-side or libc++ facilities.
#pragma once
#include "device_common.cuh"
#include "static_codes.hpp"

namespace ssb {

using dev::funnel16;
using dev::keep_bytes;
using dev::msb_mask;

#ifndef SS_KMAXP
#define SS_KMAXP 8
#endif

// ------------------------------------------------------------------------------------------------
// Generic "row" encode kernel for any code with d <= 8 (RS(2,1), RS(4,3), RS(5,4), RS(6,4) ...): the structure of
// rs32_encode_row_kernel -- a CTA walks codewords, thread = column, kernel-uniform byte funnels, rotating block
// assignment, coalesced tally prologue -- with the parity rows evaluated by run-time Horner programs.
// hmT8[(j*8 + k)*8 + i] = all-ones if bit k of coefficient M[d+j][i] is set.
// ------------------------------------------------------------------------------------------------
struct EncRowGen {
    const uint8_t *data;
    uint64_t data_stride;
    uint8_t *plane[16];       // base of shard plane j, j < d + p (local memory, or a peer GPU's memory mapped over NVLink);
                              // planes 0..d-1 (data shards) are only written when emit_data is set
    uint64_t shard_stride;
    uint32_t emit_data;
    dev::FlagWait wait;       // replicate mode: wait for the followers' ack flags before the tally (flags == nullptr: none)
    uint32_t n, len, L, vpc, fast_cols;
    uint32_t d, p;
    uint32_t pack_m, tail_ctas, ntail;   // packed kernel: codewords per CTA pass, CTAs that do tail columns, tail columns per codeword
    const uint32_t *hmT8;
    uint8_t top[SS_KMAXP];
    const uint64_t *planes;   // fused tally (nullptr: none); G == n
    uint32_t R, threshold;
    uint64_t *committed;
    uint32_t *commit_bar;
};

// multiply four packed field elements by x: shift on the FMA pipe, prmt sign mask + two lop3 on the ALU pipe.
// (A flavour that took the reduction term from a high multiply -- 1 ALU + 3 FMA-pipe instructions -- was no faster and
// was dropped.)
__device__ __forceinline__ uint32_t xtime_word(uint32_t x) { return ((x * 2u) & 0xfefefefeu) ^ (msb_mask(x) & 0x1d1d1d1du); }

// the d source vectors of column k of one codeword, funnelled to shard alignment and masked to the payload
template <int D, bool MASKED, bool EXACT>
__device__ __forceinline__ int row_load_column(const EncRowGen &P, const uint8_t *__restrict__ src, uint32_t k, uint4 (&x)[D]) {
    auto clamp16 = [](int64_t r) { return r > 16 ? 16 : (r < 0 ? 0 : static_cast<int>(r)); };
    const int d = EXACT ? D : static_cast<int>(P.d);            // EXACT: the code's width is the template's
    uint4 lo[D], hi[D];
#pragma unroll
    for (int i = 0; i < D; ++i) {
        lo[i] = make_uint4(0u, 0u, 0u, 0u);
        hi[i] = lo[i];
        if (i < d) {
            const uint32_t pos = static_cast<uint32_t>(i) * P.L + k;
            const uint32_t s = (static_cast<uint32_t>(i) * P.L) & 15u;      // kernel-uniform (k is a multiple of 16)
            const int nv = MASKED ? clamp16(static_cast<int64_t>(P.len) - pos) : 16;
            if (!MASKED || nv > 0) lo[i] = dev::ldg128(src + pos - s);
            // hi stays zero when unused: copying lo here would make every later load wait for this one to land
            if (s != 0u && (!MASKED || static_cast<int>(s) + nv > 16)) hi[i] = dev::ldg128(src + pos - s + 16u);
        }
    }
    const int onv = MASKED ? clamp16(static_cast<int64_t>(P.L) - k) : 16;
#pragma unroll
    for (int i = 0; i < D; ++i) {
        x[i] = lo[i];
        if (i < d) {
            const uint32_t s = (static_cast<uint32_t>(i) * P.L) & 15u;
            if (s != 0u) x[i] = funnel16(lo[i], hi[i], s);
            if (MASKED) {
                const int nv = clamp16(static_cast<int64_t>(P.len) - (static_cast<uint32_t>(i) * P.L + k));
                x[i] = keep_bytes(x[i], nv < onv ? nv : onv);
            }
        }
    }
    return onv;
}

// parity row j of a compile-time code from the column's source vectors: Horner over the coefficient bits, fully unrolled
template <int CODE, int J, int D>
__device__ __forceinline__ uint4 static_parity_row(const uint4 (&x)[D]) {
    static_assert(D == static_code_d(CODE), "static code width");
    constexpr int top = static_code_top(CODE, J);
    uint4 acc = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
    for (int kk = 7; kk >= 0; --kk) {
        if (kk > top) continue;
        if (kk != top) {
            acc.x = xtime_word(acc.x); acc.y = xtime_word(acc.y);
            acc.z = xtime_word(acc.z); acc.w = xtime_word(acc.w);
        }
#pragma unroll
        for (int i = 0; i < D; ++i)
            if ((static_code_coef(CODE, J, i) >> kk) & 1u) {
                acc.x ^= x[i].x; acc.y ^= x[i].y; acc.z ^= x[i].z; acc.w ^= x[i].w;
            }
    }
    return acc;
}

// the p parity vectors of one column from its d source vectors x[], stored at plane[d + j] + out_off (and, with
// emit_data, the source vectors themselves at plane[i] + out_off: the pack-for-send of subset_copy, rscoding.rs:255-293)
template <int D, int CODE, bool MASKED>
__device__ __forceinline__ void parity_rows(const EncRowGen &P, const uint4 (&x)[D], int onv, uint64_t out_off) {
    if (P.emit_data) {        // kernel-uniform; x[] is already masked to the output vector in MASKED columns
#pragma unroll
        for (int i = 0; i < D; ++i)
            if (CODE != kCodeGeneric || static_cast<uint32_t>(i) < P.d) dev::stg128_cs(P.plane[i] + out_off, x[i]);
    }
    if constexpr (CODE != kCodeGeneric) {
        static_assert(D == static_code_d(CODE), "static code width");
#pragma unroll
        for (int j = 0; j < static_code_p(CODE); ++j) {
            const int top = static_code_top(CODE, j);
            uint4 acc = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
            for (int kk = 7; kk >= 0; --kk) {
                if (kk > top) continue;
                if (kk != top) {
                    acc.x = xtime_word(acc.x); acc.y = xtime_word(acc.y);
                    acc.z = xtime_word(acc.z); acc.w = xtime_word(acc.w);
                }
#pragma unroll
                for (int i = 0; i < D; ++i)
                    if ((static_code_coef(CODE, j, i) >> kk) & 1u) {
                        acc.x ^= x[i].x; acc.y ^= x[i].y; acc.z ^= x[i].z; acc.w ^= x[i].w;
                    }
            }
            if (MASKED) acc = keep_bytes(acc, onv);
            dev::stg128_cs(P.plane[D + j] + out_off, acc);
        }
    } else {
        for (uint32_t j = 0; j < P.p; ++j) {
            const uint4 *hm = reinterpret_cast<const uint4 *>(P.hmT8 + j * 64u);
            uint4 acc = make_uint4(0u, 0u, 0u, 0u);
            const int top = P.top[j];
            for (int kk = top; kk >= 0; --kk) {
                const uint4 m0 = __ldg(hm + kk * 2);
                const uint4 m1 = D > 4 ? __ldg(hm + kk * 2 + 1) : make_uint4(0u, 0u, 0u, 0u);
                const uint32_t mk[8] = {m0.x, m0.y, m0.z, m0.w, m1.x, m1.y, m1.z, m1.w};
                if (kk != top) {
                    acc.x = xtime_word(acc.x); acc.y = xtime_word(acc.y);
                    acc.z = xtime_word(acc.z); acc.w = xtime_word(acc.w);
                }
#pragma unroll
                for (int i = 0; i < D; ++i) {
                    acc.x ^= x[i].x & mk[i];
                    acc.y ^= x[i].y & mk[i];
                    acc.z ^= x[i].z & mk[i];
                    acc.w ^= x[i].w & mk[i];
                }
            }
            if (MASKED) acc = keep_bytes(acc, onv);
            dev::stg128_cs(P.plane[P.d + j] + out_off, acc);
        }
    }
}

template <int D, int CODE, bool MASKED>
__device__ __forceinline__ void horner_row_column(const EncRowGen &P, const uint8_t *__restrict__ src, uint64_t out_off, uint32_t k) {
    uint4 x[D];
    const int onv = row_load_column<D, MASKED, CODE != kCodeGeneric>(P, src, k, x);
    parity_rows<D, CODE, MASKED>(P, x, onv, out_off + k);
}

// Split load for the software-pipelined packed kernel (complete columns only): issue the aligned 128-bit loads of one
// column into raw registers, and later funnel them to shard alignment.  Shard 0 always starts 16-byte aligned; with
// ALIGNED (shard_len % 16 == 0) every shard does and no second load exists.
template <int D, bool ALIGNED>
struct RawColumn {
    uint4 lo[D];
    uint4 hi[ALIGNED ? 1 : D];
};
template <int D, bool ALIGNED, bool EXACT>
__device__ __forceinline__ void raw_issue(const EncRowGen &P, const uint8_t *__restrict__ src, uint32_t k, RawColumn<D, ALIGNED> &r) {
    const int d = EXACT ? D : static_cast<int>(P.d);
#pragma unroll
    for (int i = 0; i < D; ++i) {
        if (i < d) {
            const uint32_t pos = static_cast<uint32_t>(i) * P.L + k;
            const uint32_t s = ALIGNED ? 0u : (static_cast<uint32_t>(i) * P.L) & 15u;
            r.lo[i] = dev::ldg128(src + pos - s);
            if constexpr (!ALIGNED) {
                if (i > 0) {
                    r.hi[i] = make_uint4(0u, 0u, 0u, 0u);       // never a copy of lo: that would wait for the load
                    if (s != 0u) r.hi[i] = dev::ldg128(src + pos - s + 16u);
                }
            }
        } else {
            r.lo[i] = make_uint4(0u, 0u, 0u, 0u);
        }
    }
}
template <int D, bool ALIGNED, bool EXACT>
__device__ __forceinline__ void raw_finish(const EncRowGen &P, const RawColumn<D, ALIGNED> &r, uint4 (&x)[D]) {
    const int d = EXACT ? D : static_cast<int>(P.d);
#pragma unroll
    for (int i = 0; i < D; ++i) {
        x[i] = r.lo[i];
        if constexpr (!ALIGNED) {
            if (i > 0 && i < d) {
                const uint32_t s = (static_cast<uint32_t>(i) * P.L) & 15u;
                if (s != 0u) x[i] = funnel16(r.lo[i], r.hi[i], s);
            }
        }
    }
}

template <int D, int CODE, int MAXT, int MINB>
__global__ void __launch_bounds__(MAXT, MINB) horner_encode_row_kernel(const __grid_constant__ EncRowGen P) {
    const uint32_t lane = threadIdx.x & 31u, wid = threadIdx.x >> 5, nblk = blockDim.x >> 5;
    if (P.emit_data) dev::cta_wait_flags(P.wait);       // kernel-uniform; the ack planes tallied below come from peer GPUs
    if (P.planes != nullptr) {
        const uint32_t per = (P.n + gridDim.x - 1) / gridDim.x;
        const uint32_t lo = blockIdx.x * per;
        const uint32_t hi = lo + per < P.n ? lo + per : P.n;
        for (uint32_t g = lo + threadIdx.x; g < hi; g += blockDim.x) {
            const uint64_t w = dev::tally_word(P.planes, P.R, P.n, g, P.threshold);
            P.committed[g] = w;
            if (P.commit_bar != nullptr) P.commit_bar[g] = dev::commit_prefix(w);
        }
    }
    uint32_t wb = wid;
#pragma unroll 1
    for (uint32_t g = blockIdx.x; g < P.n; g += gridDim.x) {
        const uint8_t *src = P.data + static_cast<uint64_t>(g) * P.data_stride;
        const uint64_t out_off = static_cast<uint64_t>(g) * P.shard_stride;
        // codewords wider than the CTA are walked in segments of blockDim.x columns (one pass for the usual sizes)
        for (uint32_t vb = 0; vb < P.vpc; vb += blockDim.x) {
            const uint32_t v = vb + wb * 32u + lane;
            const bool masked = vb + wb * 32u + 32u > P.fast_cols;       // warp-uniform
            if (v >= P.vpc) continue;
            if (!masked) horner_row_column<D, CODE, false>(P, src, out_off, v * 16u);
            else horner_row_column<D, CODE, true>(P, src, out_off, v * 16u);
        }
        wb = (wb + 1u == nblk) ? 0u : wb + 1u;                       // rotate the warp -> block assignment
    }
}

// Packed flavour of the row kernel, for shard lengths whose column count is not a multiple of 32.  The complete
// columns (every source window inside the payload, full 16-byte output) of pack_m consecutive codewords are laid side by
// side over the CTA's threads with a FIXED thread -> (codeword, column) map -- one division per thread for the whole
// kernel -- so nearly every lane does unmasked work (RS(5,4) on 4 KB: 5 x 51 columns on 256 threads instead of 52 on 64).
// The incomplete columns (normally one per codeword) go to the first tail_ctas CTAs, one column per thread, masked.
// resident 256-thread CTAs per SM for the packed kernel: the pipelined main loop holds one column being computed
// (4D registers) and the next one in flight (4D aligned, 8D-4 otherwise)
template <int D, bool ALIGNED, bool PIPE>
SSB_HD constexpr int packed_min_blocks() {
    if (!PIPE) return D <= 3 ? 6 : D <= 5 ? 5 : D <= 6 ? 4 : 3;          // 40 / 48 / 64 / 80 registers
    constexpr int need = 4 * D + (ALIGNED ? 4 * D : 8 * D - 4) + 22;
    constexpr int b = 65536 / (256 * need);
    return b > 6 ? 6 : (b < 1 ? 1 : b);
}

template <int D, int CODE, bool ALIGNED, bool PIPE>
__global__ void __launch_bounds__(256, packed_min_blocks<D, ALIGNED, PIPE>()) horner_encode_packed_kernel(const __grid_constant__ EncRowGen P) {
    if (P.emit_data) dev::cta_wait_flags(P.wait);
    if (P.planes != nullptr) {
        const uint32_t per = (P.n + gridDim.x - 1) / gridDim.x;
        const uint32_t lo = blockIdx.x * per;
        const uint32_t hi = lo + per < P.n ? lo + per : P.n;
        for (uint32_t g = lo + threadIdx.x; g < hi; g += blockDim.x) {
            const uint64_t w = dev::tally_word(P.planes, P.R, P.n, g, P.threshold);
            P.committed[g] = w;
            if (P.commit_bar != nullptr) P.commit_bar[g] = dev::commit_prefix(w);
        }
    }
    if (blockIdx.x < P.tail_ctas) {
        const uint64_t item = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
        const uint64_t g = P.ntail == 1u ? item : item / P.ntail;
        if (g >= P.n) return;
        const uint32_t col = P.fast_cols + static_cast<uint32_t>(item - g * P.ntail);
        horner_row_column<D, CODE, true>(P, P.data + g * P.data_stride, g * P.shard_stride, col * 16u);
        return;
    }
    const uint32_t cg = threadIdx.x / P.fast_cols;               // fast_cols >= 1 whenever main CTAs exist
    const uint32_t k = (threadIdx.x - cg * P.fast_cols) * 16u;
    if (cg >= P.pack_m) return;
    const uint64_t step = static_cast<uint64_t>(gridDim.x - P.tail_ctas) * P.pack_m;
    uint64_t g = static_cast<uint64_t>(blockIdx.x - P.tail_ctas) * P.pack_m + cg;
    if (g >= P.n) return;
    if constexpr (!PIPE) {
#pragma unroll 1
        for (; g < P.n; g += step)
            horner_row_column<D, CODE, false>(P, P.data + g * P.data_stride, g * P.shard_stride, k);
        return;
    }
    // software pipeline: the loads of this thread's next column are in flight while the current one is computed
    RawColumn<D, ALIGNED> raw;
    raw_issue<D, ALIGNED, CODE != kCodeGeneric>(P, P.data + g * P.data_stride, k, raw);
#pragma unroll 1
    while (true) {
        uint4 x[D];
        raw_finish<D, ALIGNED, CODE != kCodeGeneric>(P, raw, x);
        const uint64_t gn = g + step;
        if (gn < P.n) raw_issue<D, ALIGNED, CODE != kCodeGeneric>(P, P.data + gn * P.data_stride, k, raw);
        parity_rows<D, CODE, false>(P, x, 16, g * P.shard_stride + k);
        if (gn >= P.n) break;
        g = gn;
    }
}


}  // namespace ssb
