// device_common.cuh -- device-side helpers shared by the kernel files (sm_90a).
#pragma once
#ifndef __CUDACC_RTC__
#include <cuda_runtime.h>

#include <cstdint>
#else
// NVRTC (run-time specialisation, jit.cu): no host headers; the fixed-width types are spelled out
typedef unsigned char uint8_t;
typedef unsigned short uint16_t;
typedef unsigned int uint32_t;
typedef int int32_t;
typedef unsigned long long uint64_t;
typedef long long int64_t;
typedef unsigned long long uintptr_t;
#endif

namespace ssb {
namespace dev {

// ---- byte permute / packed GF(2^8) arithmetic on four bytes per 32-bit register -------------
__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel) {
    uint32_t r;
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(sel));
    return r;
}

// 0xff in every byte whose top bit is set, 0x00 elsewhere (prmt sign-replicate mode): one ALU op.
__device__ __forceinline__ uint32_t msb_mask(uint32_t x) { return prmt(x, 0u, 0xba98u); }

// multiply each of the four packed field elements by x (i.e. by 2) modulo 0x11D
__device__ __forceinline__ uint32_t xtime4(uint32_t x) {
    return ((x & 0x7f7f7f7fu) << 1) ^ (msb_mask(x) & 0x1d1d1d1du);
}

// ---- memory -----------------------------------------------------------------------------------
__device__ __forceinline__ uint4 ldg128(const void *p) {
    uint4 r;
    asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}

// the same load with an L2 prefetch-size hint: the L2 fetches the whole 256-byte block around the address from DRAM
__device__ __forceinline__ uint4 ldg128_pf256(const void *p) {
    uint4 r;
    asm volatile("ld.global.nc.L2::256B.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}

// streaming 128-bit store (written once, not re-read by this kernel)
__device__ __forceinline__ void stg128_cs(void *p, const uint4 &v) {
    asm volatile("st.global.cs.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
                 "r"(v.w)
                 : "memory");
}

// 128-bit store with a run-time cache operator (tuning knob for stores that land in a peer GPU's memory):
// 0 = .cs (streaming), 1 = default write-back, 2 = .cg, 3 = .wt
__device__ __forceinline__ void stg128_mode(void *p, const uint4 &v, uint32_t mode) {
    if (mode == 0u) { stg128_cs(p, v); return; }
    if (mode == 1u)
        asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
    else if (mode == 2u)
        asm volatile("st.global.cg.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
    else
        asm volatile("st.global.wt.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// keep the first nvalid (0..16) bytes of v, zero the rest
__device__ __forceinline__ uint4 keep_bytes(uint4 v, int nvalid) {
    if (nvalid >= 16) return v;
    uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int nv = nvalid - 4 * i;
        const uint32_t m = nv >= 4 ? 0xffffffffu : (nv <= 0 ? 0u : ((1u << (8 * nv)) - 1u));
        w[i] &= m;
    }
    return make_uint4(w[0], w[1], w[2], w[3]);
}

// Bytes [p, p+16) of global memory, for any alignment of p, as a little-endian uint4; bytes at
// index >= nvalid come back as zero and are never dereferenced beyond the aligned 16-byte block
// that holds the last valid byte.  nvalid <= 0 returns zeros without touching memory.
// Two aligned 128-bit loads + a byte funnel shift; neighbouring lanes hit the same sectors in L1.
//
// Split in two so that a thread that needs several vectors can ISSUE all their loads before it TOUCHES any of the
// data: a warp issues in order, so the first instruction that reads a load's destination stalls everything behind
// it -- including the next vector's loads -- until that load has landed.
struct Raw16 {
    uint4 lo, hi;
    uint32_t s;
};
__device__ __forceinline__ Raw16 raw16_issue(const uint8_t *p, int nvalid) {
    Raw16 r;
    r.lo = make_uint4(0u, 0u, 0u, 0u);
    r.hi = r.lo;
    r.s = 0u;
    if (nvalid <= 0) return r;
    const uintptr_t a = reinterpret_cast<uintptr_t>(p);
    r.s = static_cast<uint32_t>(a) & 15u;
    const uint4 *q = reinterpret_cast<const uint4 *>(a - r.s);
    r.lo = ldg128(q);
    if (r.s != 0u && static_cast<int>(16u - r.s) < nvalid) r.hi = ldg128(q + 1);
    return r;
}
__device__ __forceinline__ uint4 raw16_finish(const Raw16 &r, int nvalid) {
    const uint4 &lo = r.lo, &hi = r.hi;
    const uint32_t s = r.s;
    uint4 o;
    if (s == 0u) {
        o = lo;
    } else {
        const uint32_t sel = 0x3210u + 0x1111u * (s & 3u);
        switch (s >> 2) {
            case 0:
                o = make_uint4(prmt(lo.x, lo.y, sel), prmt(lo.y, lo.z, sel), prmt(lo.z, lo.w, sel),
                               prmt(lo.w, hi.x, sel));
                break;
            case 1:
                o = make_uint4(prmt(lo.y, lo.z, sel), prmt(lo.z, lo.w, sel), prmt(lo.w, hi.x, sel),
                               prmt(hi.x, hi.y, sel));
                break;
            case 2:
                o = make_uint4(prmt(lo.z, lo.w, sel), prmt(lo.w, hi.x, sel), prmt(hi.x, hi.y, sel),
                               prmt(hi.y, hi.z, sel));
                break;
            default:
                o = make_uint4(prmt(lo.w, hi.x, sel), prmt(hi.x, hi.y, sel), prmt(hi.y, hi.z, sel),
                               prmt(hi.z, hi.w, sel));
                break;
        }
    }
    return keep_bytes(o, nvalid);
}
__device__ __forceinline__ uint4 load16(const uint8_t *p, int nvalid) { return raw16_finish(raw16_issue(p, nvalid), nvalid); }

// bytes [s, s+16) of the 32-byte window {lo, hi}; s is kernel-uniform
__device__ __forceinline__ uint4 funnel16(const uint4 &lo, const uint4 &hi, uint32_t s) {
    const uint32_t sel = 0x3210u + 0x1111u * (s & 3u);
    switch (s >> 2) {
        case 0:
            return make_uint4(prmt(lo.x, lo.y, sel), prmt(lo.y, lo.z, sel), prmt(lo.z, lo.w, sel),
                              prmt(lo.w, hi.x, sel));
        case 1:
            return make_uint4(prmt(lo.y, lo.z, sel), prmt(lo.z, lo.w, sel), prmt(lo.w, hi.x, sel),
                              prmt(hi.x, hi.y, sel));
        case 2:
            return make_uint4(prmt(lo.z, lo.w, sel), prmt(lo.w, hi.x, sel), prmt(hi.x, hi.y, sel),
                              prmt(hi.y, hi.z, sel));
        default:
            return make_uint4(prmt(lo.w, hi.x, sel), prmt(hi.x, hi.y, sel), prmt(hi.y, hi.z, sel),
                              prmt(hi.z, hi.w, sel));
    }
}

// Store the first nvalid (1..16) bytes of v at p.  padded: p is 16-byte aligned with 16 bytes of
// capacity, and the bytes past nvalid are written as zeros (one 128-bit store).  Otherwise exact.
__device__ __forceinline__ void store16(uint8_t *p, uint4 v, int nvalid, bool padded) {
    if (padded) {
        stg128_cs(p, keep_bytes(v, nvalid));
        return;
    }
    if (nvalid >= 16 && (reinterpret_cast<uintptr_t>(p) & 15u) == 0u) {
        stg128_cs(p, v);
        return;
    }
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    const int nb = nvalid < 16 ? nvalid : 16;
#pragma unroll
    for (int b = 0; b < 16; ++b)
        if (b < nb) p[b] = static_cast<uint8_t>(w[b >> 2] >> (8 * (b & 3)));
}

// ---- cross-GPU step flags (multi-GPU accept step; DESIGN.md section 6) -------------------------------
// A flag is a u64 step counter in some GPU's memory.  Producers publish with st.release.sys after their data
// stores are visible system-wide; consumers poll with ld.acquire.sys.  Waits are bounded: on time-out bit 0 of the
// context's device status word is set and the kernel carries on (a wrong result that the host can see, not a hang).
__device__ __forceinline__ uint64_t ld_acquire_sys(const uint64_t *p) {
    uint64_t v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_sys(uint64_t *p, uint64_t v) {
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ uint64_t globaltimer_ns() {
    uint64_t t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
struct FlagWait {
    const uint64_t *flags;    // n counters in LOCAL memory (written by peers), nullptr: no wait
    uint32_t n;               // <= 32
    uint64_t value;           // proceed once every flags[i] >= value
    uint64_t timeout_ns;
    uint32_t *status;         // context's device status word
};
// the first n threads of the CTA poll one flag each, then the CTA barrier releases everybody
__device__ __forceinline__ void cta_wait_flags(const FlagWait &w) {
    if (w.flags == nullptr) return;
    if (threadIdx.x < w.n) {
        const uint64_t t0 = globaltimer_ns();
        while (ld_acquire_sys(w.flags + threadIdx.x) < w.value) {
            if (globaltimer_ns() - t0 > w.timeout_ns) { atomicOr(w.status, 1u); break; }
            __nanosleep(100);
        }
    }
    __syncthreads();
}

// ---- bit-sliced quorum tally of one 64-slot window ------------------------------------------
// planes[r*G + g] holds replica r's ack bits for the 64 slots of group g.  The per-slot count of
// set planes is kept bit-sliced in five 64-bit words (counts up to 31), then compared against the
// threshold with a bit-sliced comparator: 64 slots are tallied with ~4 logic ops per replica.
// This is Bitmap::count() >= threshold (src/utils/bitmap.rs:111-113;
// multipaxos/messages.rs:412-413) for 64 instances at once.
__device__ __forceinline__ uint64_t tally_word(const uint64_t *__restrict__ planes, uint32_t R,
                                               uint64_t G, uint64_t g, uint32_t threshold) {
    uint64_t c0 = 0, c1 = 0, c2 = 0, c3 = 0, c4 = 0;
    for (uint32_t r = 0; r < R; ++r) {
        uint64_t carry = __ldg(planes + static_cast<uint64_t>(r) * G + g);
        uint64_t t;
        t = c0 & carry; c0 ^= carry; carry = t;
        t = c1 & carry; c1 ^= carry; carry = t;
        t = c2 & carry; c2 ^= carry; carry = t;
        t = c3 & carry; c3 ^= carry; carry = t;
        c4 ^= carry;
    }
    if (threshold == 0u) return ~0ull;
    if (threshold > 31u) return 0ull;
    // lt = (count < threshold), most-significant bit first
    const uint64_t cb[5] = {c0, c1, c2, c3, c4};
    uint64_t lt = 0ull, eq = ~0ull;
#pragma unroll
    for (int b = 4; b >= 0; --b) {
        const uint64_t tb = ((threshold >> b) & 1u) ? ~0ull : 0ull;
        lt |= eq & ~cb[b] & tb;
        eq &= ~(cb[b] ^ tb);
    }
    return ~lt;
}

// length of the committed prefix of the window (multipaxos/durability.rs:161-170)
__device__ __forceinline__ uint32_t commit_prefix(uint64_t w) {
    return w == ~0ull ? 64u : static_cast<uint32_t>(__ffsll(static_cast<long long>(~w)) - 1);
}

}  // namespace dev
}  // namespace ssb
