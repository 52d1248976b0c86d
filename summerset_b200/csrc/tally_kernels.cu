// tally_kernels.cu -- quorum vote tallies, ack ingest, Crossword coverage predicate and the Raft
// match-index commit scan, batched over millions of independent (group, slot) instances (sm_90a).
//
// What they replace (reference, josehu07/summerset @ 1daf80aa) -- work the reference does one
// message at a time inside the replica's event loop:
//   handle_msg_accept_reply    multipaxos/messages.rs:370-443, rspaxos/messages.rs:395-465,
//                              crossword/messages.rs:481-574 (+ coverage_under_faults :15-62)
//   commit_bar advance         multipaxos/durability.rs:161-170
//   AppendEntriesReply scan    raft/messages.rs:256-275, craft/messages.rs:288-314
// All of it is HBM-bound integer/bit work: coalesced 64/128-bit loads, no shared-memory staging
// needed except for the Crossword look-up table.
#include "device_common.cuh"
#include "gossip_walk.cuh"
#include "prepare_rule.cuh"
#include "ss_internal.hpp"

namespace ssb {

constexpr int kTallyThreads = 256;

// ------------------------------------------------------------------------------------------------
// bit-plane tally: one thread per group (64 slots per thread)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kTallyThreads)
tally_planes_kernel(const uint64_t *__restrict__ planes, uint32_t R, uint64_t G, uint32_t threshold,
                    uint64_t *__restrict__ committed, uint32_t *__restrict__ commit_bar) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kTallyThreads;
    for (uint64_t g = static_cast<uint64_t>(blockIdx.x) * kTallyThreads + threadIdx.x; g < G; g += stride) {
        const uint64_t w = dev::tally_word(planes, R, G, g, threshold);
        committed[g] = w;
        if (commit_bar != nullptr) commit_bar[g] = dev::commit_prefix(w);
    }
}

// two adjacent groups per thread: 128-bit loads/stores (G even, planes 16-byte aligned)
__device__ __forceinline__ uint64_t ge_threshold(const uint64_t (&cb)[5], uint32_t threshold) {
    if (threshold == 0u) return ~0ull;
    if (threshold > 31u) return 0ull;
    uint64_t lt = 0ull, eq = ~0ull;
#pragma unroll
    for (int b = 4; b >= 0; --b) {
        const uint64_t tb = ((threshold >> b) & 1u) ? ~0ull : 0ull;
        lt |= eq & ~cb[b] & tb;
        eq &= ~(cb[b] ^ tb);
    }
    return ~lt;
}

template <int RT>   // RT > 0: replica count known at compile time (loads fully unrolled and issued up front)
__global__ void __launch_bounds__(kTallyThreads)
tally_planes_x2_kernel(const ulonglong2 *__restrict__ planes, uint32_t R, uint64_t G2, uint32_t threshold,
                       ulonglong2 *__restrict__ committed, uint2 *__restrict__ commit_bar) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kTallyThreads;
    for (uint64_t g = static_cast<uint64_t>(blockIdx.x) * kTallyThreads + threadIdx.x; g < G2; g += stride) {
        uint64_t a[5] = {0, 0, 0, 0, 0}, b[5] = {0, 0, 0, 0, 0};
        auto add = [&](const ulonglong2 &x) {
            uint64_t c = x.x, t;
            t = a[0] & c; a[0] ^= c; c = t;
            t = a[1] & c; a[1] ^= c; c = t;
            t = a[2] & c; a[2] ^= c; c = t;
            t = a[3] & c; a[3] ^= c; c = t;
            a[4] ^= c;
            c = x.y;
            t = b[0] & c; b[0] ^= c; c = t;
            t = b[1] & c; b[1] ^= c; c = t;
            t = b[2] & c; b[2] ^= c; c = t;
            t = b[3] & c; b[3] ^= c; c = t;
            b[4] ^= c;
        };
        if constexpr (RT > 0) {
            ulonglong2 v[RT];
#pragma unroll
            for (int r = 0; r < RT; ++r) v[r] = __ldg(planes + static_cast<uint64_t>(r) * G2 + g);
#pragma unroll
            for (int r = 0; r < RT; ++r) add(v[r]);
        } else {
            for (uint32_t r = 0; r < R; ++r) add(__ldg(planes + static_cast<uint64_t>(r) * G2 + g));
        }
        ulonglong2 w;
        w.x = ge_threshold(a, threshold);
        w.y = ge_threshold(b, threshold);
        committed[g] = w;
        if (commit_bar != nullptr) commit_bar[g] = make_uint2(dev::commit_prefix(w.x), dev::commit_prefix(w.y));
    }
}

// ------------------------------------------------------------------------------------------------
// per-instance vote masks: SWAR popcount of 16 one-byte Bitmaps per 128-bit load
// ------------------------------------------------------------------------------------------------
// per-byte population count of four packed bytes
__device__ __forceinline__ uint32_t popc_bytes(uint32_t x) {
    x = x - ((x >> 1) & 0x55555555u);
    x = (x & 0x33333333u) + ((x >> 2) & 0x33333333u);
    return (x + (x >> 4)) & 0x0f0f0f0fu;
}
// 4-bit result: bit b = (byte b of cnt >= thr), cnt bytes <= 8, 1 <= thr <= 127
__device__ __forceinline__ uint32_t ge_nibble(uint32_t cnt, uint32_t thr) {
    const uint32_t v = (cnt + (0x80u - thr) * 0x01010101u) & 0x80808080u;   // msb set where cnt >= thr
    return (((v >> 7) * 0x01020408u) >> 24) & 0xfu;
}

__global__ void __launch_bounds__(kTallyThreads)
tally_masks8_kernel(const uint8_t *__restrict__ masks, uint64_t n, uint32_t threshold,
                    uint16_t *__restrict__ commit16) {
    // thread i handles instances [16i, 16i+16) -> 16 commit bits
    const uint64_t nvec = ((n + 63) / 64) * 4;     // whole 64-bit output words
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kTallyThreads;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kTallyThreads + threadIdx.x; i < nvec; i += stride) {
        const uint64_t first = i * 16;
        const int nv = first >= n ? 0 : ((n - first) >= 16 ? 16 : static_cast<int>(n - first));
        const uint4 v = dev::load16(masks + first, nv);    // masks is 16-byte aligned in practice
        uint32_t bits;
        if (threshold == 0u) bits = 0xffffu;
        else if (threshold > 8u) bits = 0u;
        else
            bits = ge_nibble(popc_bytes(v.x), threshold) | (ge_nibble(popc_bytes(v.y), threshold) << 4) |
                   (ge_nibble(popc_bytes(v.z), threshold) << 8) | (ge_nibble(popc_bytes(v.w), threshold) << 12);
        if (nv < 16) bits &= (1u << nv) - 1u;   // nv == 0 -> 0
        commit16[i] = static_cast<uint16_t>(bits);
    }
}

__global__ void __launch_bounds__(kTallyThreads)
tally_masks16_kernel(const uint16_t *__restrict__ masks, uint64_t n, uint32_t threshold,
                     uint8_t *__restrict__ commit8) {
    // thread i handles instances [8i, 8i+8) -> 8 commit bits
    const uint64_t nvec = ((n + 63) / 64) * 8;     // whole 64-bit output words
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kTallyThreads;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kTallyThreads + threadIdx.x; i < nvec; i += stride) {
        const uint64_t first = i * 8;
        const int nv = first >= n ? 0 : ((n - first) >= 8 ? 8 : static_cast<int>(n - first));
        const uint4 v = dev::load16(reinterpret_cast<const uint8_t *>(masks + first), nv * 2);
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
        uint32_t bits = 0;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            bits |= (static_cast<uint32_t>(__popc(w[j] & 0xffffu)) >= threshold ? 1u : 0u) << (2 * j);
            bits |= (static_cast<uint32_t>(__popc(w[j] >> 16)) >= threshold ? 1u : 0u) << (2 * j + 1);
        }
        if (nv < 8) bits &= (1u << nv) - 1u;
        commit8[i] = static_cast<uint8_t>(bits);
    }
}

// ------------------------------------------------------------------------------------------------
// ack ingest: record stream -> planes, with the handler's filters
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kTallyThreads)
ack_ingest_kernel(const uint32_t *__restrict__ rec_group, const uint8_t *__restrict__ rec_slot,
                  const uint8_t *__restrict__ rec_peer, const uint64_t *__restrict__ rec_ballot, uint64_t n_records,
                  const uint64_t *__restrict__ bal_prepared, const uint64_t *__restrict__ inst_bal,
                  const uint64_t *__restrict__ accepting, const uint64_t *__restrict__ window_base, uint32_t R, uint64_t G,
                  uint64_t *planes) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kTallyThreads;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kTallyThreads + threadIdx.x; i < n_records; i += stride) {
        const uint64_t g = rec_group[i];
        uint32_t s = rec_slot[i];
        const uint32_t peer = rec_peer[i];
        if (g >= G || s >= 64u || peer >= R) continue;            // Bitmap::get -> Err (bitmap.rs:89-97)
        // window-relative slot -> ring position of absolute slot window_base + s (the engine's ring layout)
        if (window_base != nullptr) s = static_cast<uint32_t>(__ldg(window_base + g) + s) & 63u;
        const uint64_t ballot = rec_ballot[i];
        if (ballot != __ldg(bal_prepared + g)) continue;          // multipaxos/messages.rs:388
        if (((__ldg(accepting + g) >> s) & 1ull) == 0ull) continue; // :394-399 status != Accepting
        if (ballot < __ldg(inst_bal + g * 64 + s)) continue;      // :394-399 ballot < inst.bal
        // :404-409 -- duplicates are idempotent, so an atomic OR is an exact model
        atomicOr(reinterpret_cast<unsigned long long *>(planes + static_cast<uint64_t>(peer) * G + g), 1ull << s);
    }
}

// ------------------------------------------------------------------------------------------------
// Crossword: look-up table over (policy, ack mask), then a streaming look-up kernel
// ------------------------------------------------------------------------------------------------
// one thread per (policy, ack_mask): evaluates the reference predicate verbatim
__global__ void crossword_lut_kernel(const uint32_t *__restrict__ policies, uint32_t n_policies, uint32_t n,
                                     uint32_t T, uint32_t d, uint32_t majority, uint32_t f, int balanced,
                                     uint32_t *__restrict__ lut_bits /* n_policies * 2^n bits, zeroed */) {
    const uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t nmask = 1u << n;
    if (idx >= n_policies * nmask) return;
    const uint32_t k = idx / nmask, ack = idx % nmask;
    const uint32_t *asg = policies + k * n;
    const uint32_t nacks = __popc(ack);
    uint32_t coverage;
    if (nacks <= f) {
        coverage = 0;                                             // crossword/messages.rs:22-24
    } else if (balanced) {
        // :28-33 -- spr read from "an" entry; balanced => all equal, take the lowest acked replica
        const uint32_t first = __ffs(ack) - 1;
        coverage = (nacks - f - 1u) * (T / n) + __popc(asg[first]);
    } else {
        // :35-61 -- min over all (nacks - f)-subsets of the union of their shards
        const uint32_t cnt = nacks - f;
        coverage = T;
        for (uint32_t sub = ack; ; sub = (sub - 1u) & ack) {      // all sub-masks of ack
            if (static_cast<uint32_t>(__popc(sub)) == cnt) {
                uint32_t cov = 0;
                for (uint32_t r = 0; r < n; ++r)
                    if ((sub >> r) & 1u) cov |= asg[r];
                const uint32_t c = __popc(cov);
                if (c < coverage) coverage = c;
            }
            if (sub == 0u) break;
        }
    }
    if (nacks >= majority && coverage >= d)                       // :535-542
        atomicOr(lut_bits + (idx >> 5), 1u << (idx & 31u));
}

template <typename MaskT>
__global__ void __launch_bounds__(kTallyThreads)
tally_crossword_kernel(const MaskT *__restrict__ masks, const uint8_t *__restrict__ policy_idx, uint64_t n_inst,
                       const uint32_t *__restrict__ lut_bits, uint32_t lut_words, uint32_t n_policies, uint32_t n,
                       uint8_t *__restrict__ commit8) {
    extern __shared__ uint32_t lut[];
    for (uint32_t i = threadIdx.x; i < lut_words; i += kTallyThreads) lut[i] = lut_bits[i];
    __syncthreads();
    const uint32_t nmask = 1u << n;
    const uint64_t nvec = ((n_inst + 63) / 64) * 8;   // whole 64-bit output words
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kTallyThreads;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kTallyThreads + threadIdx.x; i < nvec; i += stride) {
        const uint64_t first = i * 8;
        const int nv = first >= n_inst ? 0 : ((n_inst - first) >= 8 ? 8 : static_cast<int>(n_inst - first));
        uint32_t bits = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            if (j < nv) {
                const uint32_t ack = static_cast<uint32_t>(masks[first + j]) & (nmask - 1u);
                uint32_t k = policy_idx[first + j];
                if (k < n_policies) {
                    const uint32_t e = k * nmask + ack;
                    bits |= ((lut[e >> 5] >> (e & 31u)) & 1u) << j;
                }
            }
        }
        commit8[i] = static_cast<uint8_t>(bits);
    }
}

// ------------------------------------------------------------------------------------------------
// Raft / CRaft commit scan: a warp walks 32 groups; lanes own groups for the scalar part and
// cooperate on each group's term window (coalesced 128-byte rows + ballot).
// ------------------------------------------------------------------------------------------------
constexpr int kRaftMaxPeers = 16;

template <int NP>   // NP >= n_peers: compile-time bound so the match values stay in registers
__global__ void __launch_bounds__(kTallyThreads)
raft_scan_kernel(const uint32_t *__restrict__ match, uint32_t n_peers, uint64_t G,
                 const uint32_t *__restrict__ last_commit, const uint32_t *__restrict__ log_end,
                 const uint32_t *__restrict__ curr_term, const uint32_t *__restrict__ terms, uint32_t W,
                 uint32_t threshold, uint32_t *new_commit, uint32_t *__restrict__ window_overflow, uint32_t ring) {
    // ring != 0 (engine state): the term of slot s sits at terms[g*W + (s & (W-1))] (W a power of two) instead of at the
    // window-relative offset s - last_commit - 1; new_commit may then alias last_commit (each lane reads its group's
    // last_commit before anything is written).
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = (static_cast<uint64_t>(blockIdx.x) * kTallyThreads + threadIdx.x) >> 5;
    const uint64_t nwarps = (static_cast<uint64_t>(gridDim.x) * kTallyThreads) >> 5;
    const uint64_t nbatches = (G + 31) / 32;
    for (uint64_t b = warp; b < nbatches; b += nwarps) {
        const uint64_t g = b * 32 + lane;
        const bool live = g < G;
        // ---- per-lane scalar part: highest slot the peers' match indices allow ----
        uint32_t lc = 0, le = 0, ct = 0, upper = 0;
        bool any = false;
        if (live) {
            lc = __ldg(last_commit + g);
            le = __ldg(log_end + g);
            ct = __ldg(curr_term + g);
            // match_cnt(slot) = 1 + #{p: match[p] >= slot} >= threshold  <=>  slot <= m, where m is
            // the (threshold-1)-th largest peer match (raft/messages.rs:266-271).
            const uint32_t need = threshold > 0u ? threshold - 1u : 0u;   // peers required
            if (need == 0u) {
                upper = 0xffffffffu; any = true;
            } else if (need <= n_peers) {
                uint32_t mv[NP];
#pragma unroll
                for (int q = 0; q < NP; ++q)
                    mv[q] = (static_cast<uint32_t>(q) < n_peers) ? __ldg(match + static_cast<uint64_t>(q) * G + g) : 0u;
                // need-th largest: the value with exactly (need-1) elements ranked above it
                uint32_t kth = 0;
#pragma unroll
                for (int q = 0; q < NP; ++q) {
                    if (static_cast<uint32_t>(q) < n_peers) {
                        uint32_t rank = 0;
#pragma unroll
                        for (int r = 0; r < NP; ++r)
                            if (static_cast<uint32_t>(r) < n_peers)
                                rank += (mv[r] > mv[q] || (mv[r] == mv[q] && r < q)) ? 1u : 0u;
                        if (rank == need - 1u) kth = mv[q];
                    }
                }
                upper = kth; any = true;
            }
            // slots scanned: last_commit+1 .. log_end-1 (raft/messages.rs:256-258)
            if (any && le > 0u) { if (upper > le - 1u) upper = le - 1u; }
            else any = false;
            if (any && upper <= lc) any = false;
            // precondition log_end - last_commit - 1 <= window violated: candidates beyond the window cannot be
            // examined, the result is then a LOWER bound of raft/messages.rs:256-275 -- counted so the host can tell
            if (any && upper - lc > W && window_overflow != nullptr) atomicAdd(window_overflow, 1u);
        }
        uint32_t result = lc;
        // ---- probe: the highest candidate slot usually IS a current-term entry (a leader appends in its own
        //      term), so each lane first checks terms[upper] for its own group: one 4-byte load instead of the
        //      whole window.  Only groups whose top candidate is an older-term entry take the cooperative scan.
        if (live && any) {
            const uint32_t o = upper - lc - 1u;
            if (o < W && __ldg(terms + g * W + (ring ? (upper & (W - 1u)) : o)) == ct) { result = upper; any = false; }
        }
        // ---- the rest: the last slot in (lc, upper) whose term equals curr_term (raft/messages.rs:261-263,271-274: last one
        //      wins).  Each lane walks ITS OWN group's window from the top, four terms per 128-bit load (the window rows are
        //      16-byte aligned when W % 4 == 0): a dozen instructions per step instead of a warp-wide ballot per 32 entries
        //      and group -- the scan was issue-bound, not bandwidth-bound.  Windows whose
        //      size is not a multiple of four, or unaligned term arrays, take the cooperative walk below. ----
        const bool vec_ok = (W & 3u) == 0u && (reinterpret_cast<uintptr_t>(terms) & 15u) == 0u;
        if (vec_ok) {
            if (live && any) {
                // positions: ring -> absolute slot numbers, else window offsets; candidates are lo_p .. hi_p
                const uint32_t span = upper - lc;                                  // offsets 0 .. span-1; span-1 was the probe
                const uint32_t lim = span < W ? span : W;
                if (lim >= 2u || (lim == 1u && span > W)) {
                    const uint32_t top_o = (span <= W) ? lim - 2u : lim - 1u;       // highest offset not probed yet
                    const uint32_t base_p = ring ? lc + 1u : 0u;                    // position of offset 0
                    const uint32_t *row = terms + g * W;
                    int64_t p = static_cast<int64_t>(base_p) + top_o;
                    const int64_t lo_p = base_p;
                    bool found = false;
                    while (p >= lo_p && !found) {
                        const uint32_t pb = static_cast<uint32_t>(p) & ~3u;         // chunk of four positions
                        const uint32_t idx = ring ? (pb & (W - 1u)) : pb;
                        const uint4 t4 = __ldg(reinterpret_cast<const uint4 *>(row + idx));
                        const uint32_t tv[4] = {t4.x, t4.y, t4.z, t4.w};
#pragma unroll
                        for (int e = 3; e >= 0; --e) {
                            const int64_t pe = static_cast<int64_t>(pb) + e;
                            if (!found && pe <= p && pe >= lo_p && tv[e] == ct) {
                                result = lc + 1u + static_cast<uint32_t>(pe - lo_p);
                                found = true;
                            }
                        }
                        p = static_cast<int64_t>(pb) - 1;
                    }
                }
            }
            if (live) new_commit[g] = result;
            continue;
        }
        // ---- cooperative part: for each remaining group of the batch, find the last slot in (lc, upper]
        //      whose term equals curr_term (raft/messages.rs:261-263,271-274: last one wins) ----
        const uint32_t todo = __ballot_sync(0xffffffffu, live && any);
        uint32_t rem = todo;
        while (rem) {
            const int src = __ffs(rem) - 1;
            rem &= rem - 1u;
            const uint32_t s_lc = __shfl_sync(0xffffffffu, lc, src);
            const uint32_t s_up = __shfl_sync(0xffffffffu, upper, src);
            const uint32_t s_ct = __shfl_sync(0xffffffffu, ct, src);
            const uint64_t sg = b * 32 + static_cast<uint64_t>(src);
            const uint32_t span = s_up - s_lc;                    // window offsets 0 .. span-1 are candidates
            const uint32_t *row = terms + sg * W;
            uint32_t found = 0xffffffffu;
            // walk the window from the top in 32-entry chunks
            const uint32_t limit = span < W ? span : W;
            for (int base = static_cast<int>((limit - 1u) & ~31u); base >= 0; base -= 32) {
                const uint32_t o = static_cast<uint32_t>(base) + lane;
                const bool hit = o < limit && __ldg(row + (ring ? ((s_lc + 1u + o) & (W - 1u)) : o)) == s_ct;
                const uint32_t m = __ballot_sync(0xffffffffu, hit);
                if (m) { found = static_cast<uint32_t>(base) + (31u - __clz(m)); break; }
            }
            if (lane == static_cast<uint32_t>(src) && found != 0xffffffffu) result = s_lc + 1u + found;
        }
        if (live) new_commit[g] = result;
    }
}

// k-th largest peer match per group: CRaft's shadow_last_commit (craft/messages.rs:677-690) with
// k = threshold - 1; also Raft's last_snap bound with k = n_peers (raft/messages.rs:298-309).
template <int NP>
__global__ void __launch_bounds__(kTallyThreads)
kth_match_kernel(const uint32_t *__restrict__ match, uint32_t n_peers, uint64_t G, uint32_t k, uint32_t *__restrict__ out) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kTallyThreads;
    for (uint64_t g = static_cast<uint64_t>(blockIdx.x) * kTallyThreads + threadIdx.x; g < G; g += stride) {
        uint32_t mv[NP];
#pragma unroll
        for (int q = 0; q < NP; ++q) mv[q] = (static_cast<uint32_t>(q) < n_peers) ? __ldg(match + static_cast<uint64_t>(q) * G + g) : 0u;
        uint32_t kth = 0;
#pragma unroll
        for (int q = 0; q < NP; ++q) {
            if (static_cast<uint32_t>(q) < n_peers) {
                uint32_t rank = 0;
#pragma unroll
                for (int r = 0; r < NP; ++r)
                    if (static_cast<uint32_t>(r) < n_peers) rank += (mv[r] > mv[q] || (mv[r] == mv[q] && r < q)) ? 1u : 0u;
                if (rank == k - 1u) kth = mv[q];
            }
        }
        out[g] = kth;
    }
}

// Prepare-phase shard merge + decision, one instance per thread (rspaxos/messages.rs:182-259,
// crossword/messages.rs:233-312): keep the shards voted at the highest ballot (the union over the replies
// carrying that ballot is what the chain of absorb_other calls leaves in inst.reqs_cw, in any arrival order),
// then decide use / null / wait and whether reconstruct_data and compute_parity are needed.  A reply votes iff its
// ballot is non-zero (rspaxos/durability.rs, crossword/durability.rs: `voted = if inst.voted.0 > 0`): a vote with no
// shards still raises the ballot and discards the shards gathered at lower ones.
__global__ void __launch_bounds__(kTallyThreads)
prepare_merge_kernel(const uint64_t *__restrict__ vote_bal, const uint32_t *__restrict__ vote_mask, uint32_t R, uint64_t N,
                     const uint8_t *__restrict__ acks_cnt, uint32_t d, uint32_t population, uint32_t f,
                     uint64_t *__restrict__ max_bal, uint32_t *__restrict__ merged, uint8_t *__restrict__ action) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kTallyThreads;
    const uint32_t data_mask = d >= 32u ? 0xffffffffu : ((1u << d) - 1u);
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kTallyThreads + threadIdx.x; i < N; i += stride) {
        uint64_t mb = 0;              // prepare_max_bal starts at 0
        uint32_t cw = 0;
        for (uint32_t r = 0; r < R; ++r) {
            const uint64_t b = __ldg(vote_bal + static_cast<uint64_t>(r) * N + i);
            if (b == 0ull) continue;  // voted == None
            const uint32_t m = __ldg(vote_mask + static_cast<uint64_t>(r) * N + i);
            if (b > mb) { mb = b; cw = m; }
            else if (b == mb) cw |= m;
        }
        max_bal[i] = mb;
        merged[i] = cw;
        action[i] = static_cast<uint8_t>(prepare_action(cw, [&] { return static_cast<uint32_t>(acks_cnt[i]); }, d, data_mask, population, f));
    }
}

// ------------------------------------------------------------------------------------------------
// Accept-frame packer (SURVEY 8f-2): turns one shard plane into the exact byte frames an unmodified Summerset
// peer decodes -- 8-byte big-endian length (utils/safetcp.rs) + bincode(PeerMessage::Msg{PeerMsg::Accept{slot,
// ballot, reqs_cw}}) where reqs_cw carries the single shard of the destination replica and data_copy = None
// (rspaxos/request.rs:127-142, utils/rscoding.rs:54-71).  A warp per frame; the frame is placed inside its
// fixed-stride slot so that the SHARD BYTES land 16-byte aligned: the bulk of the work is an aligned 128-bit copy.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ int put_varint(uint8_t *p, uint64_t v) {
    if (v < 251ull) { p[0] = static_cast<uint8_t>(v); return 1; }
    int nb; uint8_t tag;
    if (v < (1ull << 16)) { nb = 2; tag = 251; }
    else if (v < (1ull << 32)) { nb = 4; tag = 252; }
    else { nb = 8; tag = 253; }
    p[0] = tag;
    for (int i = 0; i < nb; ++i) p[1 + i] = static_cast<uint8_t>(v >> (8 * i));
    return 1 + nb;
}

struct FrameArgs {
    const uint8_t *plane;      // shard `shard_idx` of codeword g at plane + g*shard_stride (16-byte aligned)
    uint64_t shard_stride;
    uint32_t shard_idx, d, p, data_len, L;
    uint32_t msg_variant;      // PeerMsg::Accept variant index (2 for RSPaxos)
    const uint64_t *slot, *ballot;
    uint64_t n;
    uint8_t *out;
    uint64_t frame_stride;
    uint64_t *frame_off;
    uint32_t *frame_len;
};

__global__ void __launch_bounds__(kTallyThreads) frame_accept_kernel(const __grid_constant__ FrameArgs A) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = (static_cast<uint64_t>(blockIdx.x) * kTallyThreads + threadIdx.x) >> 5;
    const uint64_t nwarps = (static_cast<uint64_t>(gridDim.x) * kTallyThreads) >> 5;
    for (uint64_t g = warp; g < A.n; g += nwarps) {
        // body header: PeerMessage::Msg (0), PeerMsg::Accept, slot, ballot, d, p, data_len, shard_len, #shards -- the fixed
        // fields (at most 39 bytes) -- then `shard_idx` None tags, the Some tag and the shard's byte length.  Only the
        // fixed fields and the Some tag + length go through thread-local arrays; the None runs (up to d+p-1 bytes on
        // either side of the shard) are written straight into the frame by lane-strided loops.
        uint8_t hdr[40], some[8];
        int h = 0;
        hdr[h++] = 0;
        h += put_varint(hdr + h, A.msg_variant);
        h += put_varint(hdr + h, __ldg(A.slot + g));
        h += put_varint(hdr + h, __ldg(A.ballot + g));
        hdr[h++] = static_cast<uint8_t>(A.d);
        hdr[h++] = static_cast<uint8_t>(A.p);
        h += put_varint(hdr + h, A.data_len);
        h += put_varint(hdr + h, A.L);
        h += put_varint(hdr + h, A.d + A.p);
        int hs = 0;
        some[hs++] = 1;
        hs += put_varint(some + hs, A.L);
        const uint32_t lead = A.shard_idx;                                // None tags before the shard
        const uint32_t tail = (A.d + A.p - 1u - A.shard_idx) + 1u;       // remaining Nones + data_copy None
        const uint32_t hb = static_cast<uint32_t>(h) + lead + static_cast<uint32_t>(hs);   // body bytes before the shard
        const uint64_t body = static_cast<uint64_t>(hb) + A.L + tail;
        const uint32_t pre = 8u + hb;                                    // bytes before the shard payload
        const uint32_t pad = (16u - (pre & 15u)) & 15u;                  // so that the payload is 16-byte aligned
        uint8_t *slot_base = A.out + g * A.frame_stride;
        uint8_t *f = slot_base + pad;
        if (lane == 0u) {
            for (int i = 0; i < 8; ++i) f[i] = static_cast<uint8_t>(body >> (8 * (7 - i)));
            for (int i = 0; i < h; ++i) f[8 + i] = hdr[i];
            for (int i = 0; i < hs; ++i) f[8u + static_cast<uint32_t>(h) + lead + i] = some[i];
            A.frame_off[g] = g * A.frame_stride + pad;
            A.frame_len[g] = static_cast<uint32_t>(8u + body);
        }
        for (uint32_t t = lane; t < lead; t += 32u) f[8u + static_cast<uint32_t>(h) + t] = 0;
        uint8_t *pay = f + pre;
        const uint8_t *src = A.plane + g * A.shard_stride;
        const uint32_t full = A.L >> 4;
        for (uint32_t v = lane; v < full; v += 32u) dev::stg128_cs(pay + v * 16u, dev::ldg128(src + v * 16u));
        const uint32_t rem = A.L & 15u;
        if (lane < rem) pay[full * 16u + lane] = src[full * 16u + lane];
        for (uint32_t t = lane; t < tail; t += 32u) pay[A.L + t] = 0;
    }
}

// Crossword follower gossip planning, one instance per thread (crossword/gossiping.rs:35-84): greedy walk over the
// peers after `me`; selected peers get the availability map of that moment as their exclusion set.
__global__ void __launch_bounds__(kTallyThreads)
gossip_plan_kernel(uint32_t me, uint32_t population, uint32_t d, const uint8_t *__restrict__ src_peer,
                   const uint32_t *__restrict__ avail_in, const uint8_t *__restrict__ policy_idx,
                   const uint32_t *__restrict__ policies, uint32_t n_policies, uint32_t peer_alive, uint64_t N,
                   uint32_t *__restrict__ targets, uint32_t *__restrict__ excl /* [population][N] */) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kTallyThreads;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kTallyThreads + threadIdx.x; i < N; i += stride) {
        uint32_t k = policy_idx[i];
        if (k >= n_policies) k = 0;
        const uint32_t *asg = policies + k * population;
        targets[i] = gossip_walk(me, population, d, src_peer[i], __ldg(avail_in + i), peer_alive,
                                 [&](uint32_t peer) { return __ldg(asg + peer); },
                                 [&](uint32_t peer, uint32_t avail) { excl[static_cast<uint64_t>(peer) * N + i] = avail; });
    }
}

// ------------------------------------------------------------------------------------------------
// multi-GPU step: flag signal + the simulated followers' ack (DESIGN.md section 6)
// ------------------------------------------------------------------------------------------------
struct SignalArgs {
    uint64_t *flag[32];
    uint32_t n;
    uint64_t value;
};
// Launched right behind the kernel whose stores it publishes: a kernel boundary orders those stores (local and peer)
// before this one, and each lane then releases one flag at system scope.
__global__ void flag_signal_kernel(const __grid_constant__ SignalArgs A) {
    if (threadIdx.x < A.n) {
        __threadfence_system();
        dev::st_release_sys(A.flag[threadIdx.x], A.value);
    }
}

// stand-alone wait: one warp polls the flags; later work on the stream starts when they are all there
__global__ void flag_wait_kernel(const __grid_constant__ dev::FlagWait W) { dev::cta_wait_flags(W); }

struct AckArgs {
    const uint64_t *src;      // [R][G] local
    uint64_t *dst[16];        // per replica: G words in the leader GPU's memory (local or peer), or nullptr
    uint32_t R;
    uint64_t G;
    dev::FlagWait wait;
};
// rspaxos/durability.rs:101-118 for a whole batch: the follower has the shard in its log (the leader's kernel stored
// it there), so it replies -- its ack bit-plane goes into the leader's ack buffer with plain (possibly NVLink) stores.
__global__ void __launch_bounds__(kTallyThreads) follower_ack_kernel(const __grid_constant__ AckArgs A) {
    dev::cta_wait_flags(A.wait);
    const uint64_t G2 = A.G / 2;                       // 128-bit vectors (G even, checked on the host)
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kTallyThreads;
    for (uint32_t r = 0; r < A.R; ++r) {
        if (A.dst[r] == nullptr) continue;
        const uint4 *s = reinterpret_cast<const uint4 *>(A.src + static_cast<uint64_t>(r) * A.G);
        uint4 *d = reinterpret_cast<uint4 *>(A.dst[r]);
        for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kTallyThreads + threadIdx.x; i < G2; i += stride)
            dev::stg128_mode(d + i, dev::ldg128(s + i), 1u);
    }
}

// ------------------------------------------------------------------------------------------------
// host launchers
// ------------------------------------------------------------------------------------------------
int launch_flag_signal(ss_ctx *ctx, const ss_step_sync *sync) {
    if (sync == nullptr || sync->n_signal == 0) return SS_OK;
    SS_TRY(ctx_bind(ctx));
    SignalArgs A;
    A.n = sync->n_signal; A.value = sync->signal_value;
    for (uint32_t i = 0; i < 32; ++i) A.flag[i] = i < A.n ? sync->signal_flags[i] : nullptr;
    for (uint32_t i = 0; i < A.n; ++i)
        if (A.flag[i] == nullptr || (reinterpret_cast<uintptr_t>(A.flag[i]) & 7u))
            return set_error(SS_ERR_INVALID_ARG, "signal flag %u is null or not 8-byte aligned", i);
    flag_signal_kernel<<<1, 32, 0, ctx->stream>>>(A);
    return launched(ctx);
}

int launch_flag_wait(ss_ctx *ctx, const dev::FlagWait &w) {
    if (w.flags == nullptr) return SS_OK;
    SS_TRY(ctx_bind(ctx));
    flag_wait_kernel<<<1, 32, 0, ctx->stream>>>(w);
    return launched(ctx);
}

int launch_follower_ack(ss_ctx *ctx, const uint64_t *ack_src, uint64_t *const *ack_dst, uint32_t R, uint64_t G,
                        const dev::FlagWait &wait) {
    SS_TRY(ctx_bind(ctx));
    if (G == 0) return SS_OK;
    if ((G & 1ull) || (reinterpret_cast<uintptr_t>(ack_src) & 15u))
        return set_error(SS_ERR_INVALID_ARG, "follower ack needs an even group count and 16-byte aligned planes");
    AckArgs A;
    A.src = ack_src; A.R = R; A.G = G; A.wait = wait;
    for (uint32_t r = 0; r < 16; ++r) {
        A.dst[r] = r < R ? ack_dst[r] : nullptr;
        if (A.dst[r] != nullptr && (reinterpret_cast<uintptr_t>(A.dst[r]) & 15u))
            return set_error(SS_ERR_INVALID_ARG, "ack destination %u is not 16-byte aligned", r);
    }
    uint64_t ctas = (G / 2 + kTallyThreads - 1) / kTallyThreads;
    const uint64_t cap = static_cast<uint64_t>(ctx->sm_count) * 2ull;     // small, latency-bound: two CTAs per SM are plenty
    if (ctas > cap) ctas = cap;
    follower_ack_kernel<<<static_cast<uint32_t>(ctas), kTallyThreads, 0, ctx->stream>>>(A);
    return launched(ctx);
}

static inline uint32_t stream_grid(ss_ctx *ctx, uint64_t items) {
    uint64_t ctas = (items + kTallyThreads - 1) / kTallyThreads;
    const uint64_t cap = static_cast<uint64_t>(ctx->sm_count) * 8ull * 4ull;
    if (ctas > cap) ctas = cap;
    if (ctas == 0) ctas = 1;
    return static_cast<uint32_t>(ctas);
}

int launch_tally_planes(ss_ctx *ctx, const uint64_t *planes, uint32_t R, uint64_t G, uint32_t thr,
                        uint64_t *committed, uint32_t *commit_bar) {
    SS_TRY(ctx_bind(ctx));
    if (R == 0 || R > 16) return set_error(SS_ERR_INVALID_ARG, "n_replicas must be 1..16, got %u", R);
    if (G == 0) return SS_OK;
    const bool al16 = ((reinterpret_cast<uintptr_t>(planes) | reinterpret_cast<uintptr_t>(committed)) & 15u) == 0u &&
                      (reinterpret_cast<uintptr_t>(commit_bar) & 7u) == 0u;
    if ((G & 1ull) == 0ull && al16) {
        const uint64_t G2 = G / 2;
        const uint32_t grid = static_cast<uint32_t>((G2 + kTallyThreads - 1) / kTallyThreads);
        const ulonglong2 *p2 = reinterpret_cast<const ulonglong2 *>(planes);
        ulonglong2 *c2 = reinterpret_cast<ulonglong2 *>(committed);
        uint2 *b2 = reinterpret_cast<uint2 *>(commit_bar);
        if (R == 5) tally_planes_x2_kernel<5><<<grid, kTallyThreads, 0, ctx->stream>>>(p2, R, G2, thr, c2, b2);
        else if (R == 3) tally_planes_x2_kernel<3><<<grid, kTallyThreads, 0, ctx->stream>>>(p2, R, G2, thr, c2, b2);
        else if (R == 7) tally_planes_x2_kernel<7><<<grid, kTallyThreads, 0, ctx->stream>>>(p2, R, G2, thr, c2, b2);
        else tally_planes_x2_kernel<0><<<grid, kTallyThreads, 0, ctx->stream>>>(p2, R, G2, thr, c2, b2);
        return launched(ctx);
    }
    tally_planes_kernel<<<stream_grid(ctx, G), kTallyThreads, 0, ctx->stream>>>(planes, R, G, thr, committed, commit_bar);
    return launched(ctx);
}

int launch_tally_masks(ss_ctx *ctx, const void *masks, uint32_t mask_bytes, uint64_t n, uint32_t thr,
                       uint64_t *commit_bits) {
    SS_TRY(ctx_bind(ctx));
    if (n == 0) return SS_OK;
    if (mask_bytes == 1) {
        tally_masks8_kernel<<<stream_grid(ctx, ((n + 63) / 64) * 4), kTallyThreads, 0, ctx->stream>>>(
            static_cast<const uint8_t *>(masks), n, thr, reinterpret_cast<uint16_t *>(commit_bits));
    } else if (mask_bytes == 2) {
        tally_masks16_kernel<<<stream_grid(ctx, ((n + 63) / 64) * 8), kTallyThreads, 0, ctx->stream>>>(
            static_cast<const uint16_t *>(masks), n, thr, reinterpret_cast<uint8_t *>(commit_bits));
    } else {
        return set_error(SS_ERR_INVALID_ARG, "mask_bytes must be 1 or 2, got %u", mask_bytes);
    }
    return launched(ctx);
}

int launch_ack_ingest(ss_ctx *ctx, const uint32_t *rec_group, const uint8_t *rec_slot, const uint8_t *rec_peer,
                      const uint64_t *rec_ballot, uint64_t n_records, const uint64_t *bal_prepared,
                      const uint64_t *inst_bal, const uint64_t *accepting, const uint64_t *window_base, uint32_t R, uint64_t G,
                      uint64_t *planes) {
    SS_TRY(ctx_bind(ctx));
    if (R == 0 || R > 16) return set_error(SS_ERR_INVALID_ARG, "n_replicas must be 1..16, got %u", R);
    if (n_records == 0) return SS_OK;
    ack_ingest_kernel<<<stream_grid(ctx, n_records), kTallyThreads, 0, ctx->stream>>>(
        rec_group, rec_slot, rec_peer, rec_ballot, n_records, bal_prepared, inst_bal, accepting, window_base, R, G, planes);
    return launched(ctx);
}

int launch_tally_crossword(ss_ctx *ctx, const void *masks, uint32_t mask_bytes, const uint8_t *policy_idx,
                           uint64_t n, const uint32_t *policies_host, uint32_t n_policies, uint32_t n_replicas,
                           uint32_t T, uint32_t d, uint32_t majority, uint32_t f, int balanced,
                           uint64_t *commit_bits) {
    SS_TRY(ctx_bind(ctx));
    if (n_replicas == 0 || n_replicas > 12) return set_error(SS_ERR_INVALID_ARG, "n_replicas must be 1..12, got %u", n_replicas);
    if (n_policies == 0 || n_policies > 16) return set_error(SS_ERR_INVALID_ARG, "n_policies must be 1..16, got %u", n_policies);
    if (T == 0 || T > 32) return set_error(SS_ERR_INVALID_ARG, "total_shards must be 1..32, got %u", T);
    if (mask_bytes != 1 && mask_bytes != 2) return set_error(SS_ERR_INVALID_ARG, "mask_bytes must be 1 or 2");
    if (mask_bytes == 1 && n_replicas > 8) return set_error(SS_ERR_INVALID_ARG, "n_replicas > 8 needs 2-byte masks");
    if (n == 0) return SS_OK;
    const uint32_t entries = n_policies << n_replicas;
    const uint32_t lut_words = (entries + 31) / 32;
    const size_t pol_bytes = sizeof(uint32_t) * n_policies * n_replicas;
    const size_t pol_slot = (pol_bytes + 255) & ~size_t(255);
    void *scratch = nullptr;
    SS_TRY(ctx_scratch(ctx, pol_slot + lut_words * 4, &scratch));
    uint32_t *d_pol = static_cast<uint32_t *>(scratch);
    uint32_t *d_lut = reinterpret_cast<uint32_t *>(static_cast<uint8_t *>(scratch) + pol_slot);
    SS_CUDA(cudaMemcpyAsync(d_pol, policies_host, pol_bytes, cudaMemcpyHostToDevice, ctx->stream));
    // policies_host may be pageable and reused by the caller right after we return
    SS_CUDA(cudaStreamSynchronize(ctx->stream));
    SS_CUDA(cudaMemsetAsync(d_lut, 0, lut_words * 4, ctx->stream));
    crossword_lut_kernel<<<(entries + 127) / 128, 128, 0, ctx->stream>>>(d_pol, n_policies, n_replicas, T, d, majority,
                                                                         f, balanced, d_lut);
    SS_TRY(launched(ctx));
    const uint32_t grid = stream_grid(ctx, ((n + 63) / 64) * 8);
    const size_t smem = lut_words * 4;
    if (mask_bytes == 1)
        tally_crossword_kernel<uint8_t><<<grid, kTallyThreads, smem, ctx->stream>>>(
            static_cast<const uint8_t *>(masks), policy_idx, n, d_lut, lut_words, n_policies, n_replicas,
            reinterpret_cast<uint8_t *>(commit_bits));
    else
        tally_crossword_kernel<uint16_t><<<grid, kTallyThreads, smem, ctx->stream>>>(
            static_cast<const uint16_t *>(masks), policy_idx, n, d_lut, lut_words, n_policies, n_replicas,
            reinterpret_cast<uint8_t *>(commit_bits));
    return launched(ctx);
}

int launch_raft_scan(ss_ctx *ctx, const uint32_t *match, uint32_t n_peers, uint64_t G, const uint32_t *last_commit,
                     const uint32_t *log_end, const uint32_t *curr_term, const uint32_t *terms, uint32_t window,
                     uint32_t threshold, uint32_t *new_commit, uint32_t *window_overflow, uint32_t ring) {
    SS_TRY(ctx_bind(ctx));
    if (ring && (window & (window - 1u))) return set_error(SS_ERR_INVALID_ARG, "ring term windows need a power-of-two size");
    if (n_peers > kRaftMaxPeers) return set_error(SS_ERR_INVALID_ARG, "n_peers must be <= %d, got %u", kRaftMaxPeers, n_peers);
    if (G == 0) return SS_OK;
    const uint64_t warps = (G + 31) / 32;
    uint64_t ctas = (warps + (kTallyThreads / 32) - 1) / (kTallyThreads / 32);
    const uint64_t cap = static_cast<uint64_t>(ctx->sm_count) * 8ull * 4ull;
    if (ctas > cap) ctas = cap;
    const uint32_t grid = static_cast<uint32_t>(ctas);
#define SS_RAFT_LAUNCH(NP) raft_scan_kernel<NP><<<grid, kTallyThreads, 0, ctx->stream>>>( \
        match, n_peers, G, last_commit, log_end, curr_term, terms, window, threshold, new_commit, window_overflow, ring)
    if (n_peers <= 2) SS_RAFT_LAUNCH(2);
    else if (n_peers <= 4) SS_RAFT_LAUNCH(4);
    else if (n_peers <= 6) SS_RAFT_LAUNCH(6);
    else if (n_peers <= 8) SS_RAFT_LAUNCH(8);
    else SS_RAFT_LAUNCH(16);
#undef SS_RAFT_LAUNCH
    return launched(ctx);
}

int launch_raft_scan_ring(ss_ctx *ctx, const uint32_t *match, uint32_t n_peers, uint64_t G, const uint32_t *last_commit,
                          const uint32_t *log_end, const uint32_t *curr_term, const uint32_t *terms, uint32_t window,
                          uint32_t threshold, uint32_t *new_commit) {
    return launch_raft_scan(ctx, match, n_peers, G, last_commit, log_end, curr_term, terms, window, threshold, new_commit, nullptr, 1u);
}

int launch_crossword_lut(ss_ctx *ctx, const uint32_t *d_policies, uint32_t n_policies, uint32_t n_replicas, uint32_t T, uint32_t d,
                         uint32_t majority, uint32_t f, int balanced, uint32_t *d_lut_bits) {
    SS_TRY(ctx_bind(ctx));
    const uint32_t entries = n_policies << n_replicas;
    SS_CUDA(cudaMemsetAsync(d_lut_bits, 0, ((entries + 31) / 32) * 4, ctx->stream));
    crossword_lut_kernel<<<(entries + 127) / 128, 128, 0, ctx->stream>>>(d_policies, n_policies, n_replicas, T, d, majority, f,
                                                                         balanced, d_lut_bits);
    return launched(ctx);
}

int launch_kth_match(ss_ctx *ctx, const uint32_t *match, uint32_t n_peers, uint64_t G, uint32_t k, uint32_t *out) {
    SS_TRY(ctx_bind(ctx));
    if (n_peers == 0 || n_peers > kRaftMaxPeers) return set_error(SS_ERR_INVALID_ARG, "n_peers must be 1..%d, got %u", kRaftMaxPeers, n_peers);
    if (k == 0 || k > n_peers) return set_error(SS_ERR_INVALID_ARG, "k must be 1..n_peers, got %u", k);
    if (G == 0) return SS_OK;
    const uint32_t grid = stream_grid(ctx, G);
    if (n_peers <= 2) kth_match_kernel<2><<<grid, kTallyThreads, 0, ctx->stream>>>(match, n_peers, G, k, out);
    else if (n_peers <= 4) kth_match_kernel<4><<<grid, kTallyThreads, 0, ctx->stream>>>(match, n_peers, G, k, out);
    else if (n_peers <= 6) kth_match_kernel<6><<<grid, kTallyThreads, 0, ctx->stream>>>(match, n_peers, G, k, out);
    else if (n_peers <= 8) kth_match_kernel<8><<<grid, kTallyThreads, 0, ctx->stream>>>(match, n_peers, G, k, out);
    else kth_match_kernel<16><<<grid, kTallyThreads, 0, ctx->stream>>>(match, n_peers, G, k, out);
    return launched(ctx);
}

int launch_prepare_merge(ss_ctx *ctx, const uint64_t *vote_bal, const uint32_t *vote_mask, uint32_t R, uint64_t N,
                         const uint8_t *acks_cnt, uint32_t d, uint32_t population, uint32_t f, uint64_t *max_bal,
                         uint32_t *merged, uint8_t *action) {
    SS_TRY(ctx_bind(ctx));
    if (R == 0 || R > 32) return set_error(SS_ERR_INVALID_ARG, "n_replicas must be 1..32, got %u", R);
    if (f > population) return set_error(SS_ERR_INVALID_ARG, "fault_tolerance > population");
    if (N == 0) return SS_OK;
    prepare_merge_kernel<<<stream_grid(ctx, N), kTallyThreads, 0, ctx->stream>>>(vote_bal, vote_mask, R, N, acks_cnt, d,
                                                                                population, f, max_bal, merged, action);
    return launched(ctx);
}

int launch_frame_accept(ss_ctx *ctx, const uint8_t *plane, uint64_t shard_stride, uint32_t shard_idx, uint32_t d, uint32_t p,
                        uint32_t data_len, uint32_t msg_variant, const uint64_t *slot, const uint64_t *ballot, uint64_t n,
                        uint8_t *out, uint64_t frame_stride, uint64_t *frame_off, uint32_t *frame_len) {
    SS_TRY(ctx_bind(ctx));
    if (d == 0 || shard_idx >= d + p || d + p > 250) return set_error(SS_ERR_INVALID_ARG, "bad shard geometry");
    if (data_len == 0) return set_error(SS_ERR_INVALID_ARG, "null codeword cannot be framed");
    const uint32_t L = (data_len + d - 1) / d;
    if (frame_stride < static_cast<uint64_t>(L) + 96u + (d + p) || (frame_stride & 15u) ||
        ((reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(plane) | shard_stride) & 15u))
        return set_error(SS_ERR_INVALID_ARG, "frame_stride must be a multiple of 16 and >= shard_len + 96 + d + p; buffers 16-byte aligned");
    if (n == 0) return SS_OK;
    FrameArgs A;
    A.plane = plane; A.shard_stride = shard_stride; A.shard_idx = shard_idx; A.d = d; A.p = p; A.data_len = data_len; A.L = L;
    A.msg_variant = msg_variant; A.slot = slot; A.ballot = ballot; A.n = n; A.out = out; A.frame_stride = frame_stride;
    A.frame_off = frame_off; A.frame_len = frame_len;
    const uint64_t warps = n;
    uint64_t ctas = (warps + (kTallyThreads / 32) - 1) / (kTallyThreads / 32);
    const uint64_t cap = static_cast<uint64_t>(ctx->sm_count) * 8ull * 8ull;
    if (ctas > cap) ctas = cap;
    frame_accept_kernel<<<static_cast<uint32_t>(ctas), kTallyThreads, 0, ctx->stream>>>(A);
    return launched(ctx);
}

int launch_gossip_plan(ss_ctx *ctx, uint32_t me, uint32_t population, uint32_t d, const uint8_t *src_peer,
                       const uint32_t *avail, const uint8_t *policy_idx, const uint32_t *policies_host, uint32_t n_policies,
                       uint32_t peer_alive, uint64_t N, uint32_t *targets, uint32_t *excl) {
    SS_TRY(ctx_bind(ctx));
    if (population == 0 || population > 32 || me >= population) return set_error(SS_ERR_INVALID_ARG, "bad me/population");
    if (n_policies == 0 || n_policies > 16) return set_error(SS_ERR_INVALID_ARG, "n_policies must be 1..16");
    if (N == 0) return SS_OK;
    const size_t pol_bytes = sizeof(uint32_t) * n_policies * population;
    void *scratch = nullptr;
    SS_TRY(ctx_scratch(ctx, pol_bytes, &scratch));
    SS_CUDA(cudaMemcpyAsync(scratch, policies_host, pol_bytes, cudaMemcpyHostToDevice, ctx->stream));
    SS_CUDA(cudaStreamSynchronize(ctx->stream));       // policies_host may be reused by the caller
    gossip_plan_kernel<<<stream_grid(ctx, N), kTallyThreads, 0, ctx->stream>>>(
        me, population, d, src_peer, avail, policy_idx, static_cast<const uint32_t *>(scratch), n_policies, peer_alive, N,
        targets, excl);
    return launched(ctx);
}

}  // namespace ssb
