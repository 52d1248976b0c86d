// engine_prepare.cu -- the new RSPaxos / Crossword leader's PrepareReply absorb (ss_engine_prepare_absorb):
// handle_msg_prepare_reply (rspaxos/messages.rs:88-326, crossword/messages.rs:140-400) for a batch of PrepareReply frames
// over many groups.  The Prepare-phase bookkeeping (prepare_acks, prepare_max_bal and the gathered codeword) is the
// engine's, the leader's state; the replica's acceptor is read for the Preparing positions and written only where the
// reference writes the shared instance while it is Preparing (the external fill).
//
//   pa_decode_kernel       a thread per frame: prepare_reply_decode (codeword_wire.cuh), the sort keys
//   (CUB radix sort)       frame indices stably sorted by group: each group's frames in frame order
//   pa_walk_kernel<false>  a warp per group segment, lane l keeping ring positions l and l + 32: the frames replayed in
//                          order (filters, external fill, vote merge, acks, decision points); per frame the store
//                          bytes, PrepareBal cells and decided records it adds
//   (engine.cu's scan)     their exclusive scans in group order
//   pa_walk_kernel<true>   the same walk for the groups that fit the capacities, now writing: the engine's window rebuild
//                          and Accepting instances, the decided list, the zero NULL codewords, the per-position
//                          bookkeeping and each frame's fill and copy target
//   pa_write_kernel        a warp per frame: its fill's PrepareBal cells and fresh acceptor instances, and the shards it
//                          adds to a gathered codeword that is still current
//   pa_finish_kernel       pending, the store cursor, the decided list's unused tail
//   (ss_rs_reconstruct_batch_dev)  one launch over the decided list: the missing shards of the USE codewords
//
// Stated differences from the reference: include/summerset_b200.h at ss_engine_prepare_absorb.
#include <cub/device/device_radix_sort.cuh>

#include "acceptor_state.hpp"
#include "codeword_wire.cuh"
#include "device_common.cuh"
#include "engine_state.hpp"
#include "prepare_rule.cuh"
#include "ss_internal.hpp"
#include "window_ring.cuh"
#include "wire_common.cuh"

namespace ssb {

constexpr int kPaThreads = 256;
constexpr uint64_t kNullPitch = SS_CW_SLOT_PITCH(1);        // the NULL codeword's slot: shard_len 1

struct PaArgs {
    const uint8_t *buf;
    uint64_t buf_len;
    const uint64_t *frame_off;
    const uint32_t *frame_group;
    const uint8_t *frame_peer;
    uint64_t n, G;
    uint32_t d, T, population, majority, f, me, variant, wal_variant, data_mask, all_mask;
    const uint64_t *bps;            // [G] bal_prep_sent
    const uint8_t *policy;          // Crossword [G], may be nullptr
    // acceptor
    const uint64_t *a_base, *a_accepting, *a_committed;
    uint64_t *a_preparing, *a_inst_bal, *a_voted_bal, *a_prep_trigger;
    uint32_t *a_held, *a_data_len, *a_voted_mask, *a_assignment, *a_assign_rows;
    uint8_t *a_source, *a_prep_span;
    // engine
    uint64_t *planes, *bal_prepared, *inst_bal, *accepting, *committed, *window_base;
    uint32_t *commit_bar;
    uint8_t *policy_idx;
    ss_cw_loc *cw_loc;              // Crossword [G*64], else nullptr
    uint64_t *pa_ballot, *pa_done, *pa_max_bal, *pa_off;
    uint32_t *pa_acks, *pa_mask, *pa_len;
    // scratch
    ss_prepare_reply_rec *rec;
    uint32_t *key_in, *idx_in;
    const uint32_t *key, *idx;
    uint64_t *c_dec, *c_cell, *c_store;     // [n] by sorted position: decided records, cells, store bytes; then their scans
    const uint64_t *tot;                    // [3] the scans' totals
    uint64_t *words;                        // [2] applied store bytes and decided records (atomicMax)
    uint64_t *dst;                          // [n] by frame: the slot offset its shards go to (UINT64_MAX: none)
    uint32_t *take;                         // [n] by frame: the shards it adds there
    uint64_t *fill;                         // [n] by frame: the window positions its external fill covers
    uint32_t *present;                      // [dec_cap] shards each decided codeword holds before the reconstruct
    // capacities and outputs
    const uint64_t *store_used;
    uint64_t *store_used_out;
    uint64_t store_cap, cell_cap, dec_cap;
    uint8_t *shards;
    uint64_t plane_stride;
    uint8_t *wal;
    uint32_t *rec_group;
    uint64_t *rec_slot;
    uint64_t *dec_slot, *dec_ballot, *dec_off;
    uint32_t *dec_len, *dec_group;
    uint8_t *dec_policy;
    uint64_t *pending;
    uint32_t *verdict, *status;
};

__device__ __forceinline__ uint64_t below(uint32_t w) { return w >= 64u ? ~0ull : (1ull << w) - 1u; }

// 1. a thread per frame
__global__ void __launch_bounds__(kPaThreads) pa_decode_kernel(const __grid_constant__ PaArgs A) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kPaThreads;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kPaThreads + threadIdx.x; i < A.n; i += stride) {
        const uint32_t g = A.frame_group[i];
        ss_prepare_reply_rec r = prepare_reply_decode(A.buf, A.buf_len, A.frame_off[i], A.d, A.T, A.variant);
        if (g >= A.G || (r.kind == A.variant && A.frame_peer[i] >= A.population)) {
            r = ss_prepare_reply_rec{};
            r.kind = SS_FRAME_KIND_MALFORMED;
            r.shards_at = ~0ull;
        }
        A.rec[i] = r;
        A.key_in[i] = g < A.G ? g : static_cast<uint32_t>(A.G);
        A.idx_in[i] = static_cast<uint32_t>(i);
    }
}

// 2. / 4. a warp per group segment.  kApply = false counts what each frame adds; kApply = true cuts the groups that do
//    not fit and replays the others again, writing.  Both passes read the same acceptor state (its per-slot words are
//    read only at positions the walk has not filled, and the fill is written afterwards), so they decide the same.
template <bool kApply>
__global__ void __launch_bounds__(kPaThreads, 1) pa_walk_kernel(const __grid_constant__ PaArgs A) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = (static_cast<uint64_t>(blockIdx.x) * kPaThreads + threadIdx.x) >> 5;
    const uint64_t nwarps = (static_cast<uint64_t>(gridDim.x) * kPaThreads) >> 5;
    bool store_full = false, wal_full = false;
    for (uint64_t t = warp; t < A.n; t += nwarps) {
        if (t != 0u && A.key[t] == A.key[t - 1]) continue;
        const uint32_t g = A.key[t];
        uint64_t k_end = t + 1u;
        while (k_end < A.n && A.key[k_end] == g) ++k_end;
        if (g >= A.G) {                                                 // malformed: nothing to add
            for (uint64_t k = t + lane; k < k_end; k += 32u) {
                if (kApply) {
                    A.verdict[A.idx[k]] = SS_FRAME_KIND_MALFORMED;
                    A.dst[A.idx[k]] = ~0ull;
                    A.fill[A.idx[k]] = 0u;
                } else {
                    A.c_dec[k] = 0u; A.c_cell[k] = 0u; A.c_store[k] = 0u;
                }
            }
            continue;
        }
        uint64_t d_at = 0, c_at = 0, s_at = 0;
        if (kApply) {
            const uint64_t d_end = k_end < A.n ? A.c_dec[k_end] : A.tot[0];
            const uint64_t c_end = k_end < A.n ? A.c_cell[k_end] : A.tot[1];
            const uint64_t s_end = k_end < A.n ? A.c_store[k_end] : A.tot[2];
            const uint64_t used = (*A.store_used + 31u) & ~31ull;            // slots start 32-byte aligned
            const bool sf = used > A.store_cap || s_end > A.store_cap - used;
            const bool wf = c_end > A.cell_cap || d_end > A.dec_cap;
            if (sf || wf) {                                             // the per-group cut: nothing of g applies
                store_full |= sf;
                wal_full |= wf && !sf;
                for (uint64_t k = t + lane; k < k_end; k += 32u) {
                    const uint32_t i = A.idx[k], kind = A.rec[i].kind;
                    A.verdict[i] = kind != A.variant ? kind : sf ? SS_ACCEPT_VERDICT_STORE_FULL : SS_ACCEPT_VERDICT_WAL_FULL;
                    A.dst[i] = ~0ull;
                    A.fill[i] = 0u;
                }
                continue;
            }
            d_at = A.c_dec[t]; c_at = A.c_cell[t]; s_at = used + A.c_store[t];
            if (lane == 0u) {
                atomicMax(reinterpret_cast<unsigned long long *>(A.words), static_cast<unsigned long long>(s_end));
                atomicMax(reinterpret_cast<unsigned long long *>(A.words + 1), static_cast<unsigned long long>(d_end));
            }
        }
        const uint64_t bps = A.bps[g], row = static_cast<uint64_t>(g) * 64u;
        const bool reset = A.pa_ballot[g] != bps;                       // a new step-up: fresh bookkeeping
        uint32_t acks = reset ? 0u : A.pa_acks[g];
        uint64_t done = reset ? 0ull : A.pa_done[g];
        const uint64_t base = A.a_base[g];
        const uint32_t r = static_cast<uint32_t>(base & 63u);
        const uint64_t settled = A.a_accepting[g] | A.a_committed[g];
        uint64_t prep = A.a_preparing[g], filled = 0u;
        // this lane's two ring positions, lo = lane and hi = lane + 32
        uint64_t mb_lo = 0u, mb_hi = 0u, of_lo = ~0ull, of_hi = ~0ull;
        uint32_t mk_lo = 0u, mk_hi = 0u, ln_lo = 0u, ln_hi = 0u;
        if (!reset) {
            mb_lo = A.pa_max_bal[row + lane]; mb_hi = A.pa_max_bal[row + lane + 32u];
            of_lo = A.pa_off[row + lane]; of_hi = A.pa_off[row + lane + 32u];
            mk_lo = A.pa_mask[row + lane]; mk_hi = A.pa_mask[row + lane + 32u];
            ln_lo = A.pa_len[row + lane]; ln_hi = A.pa_len[row + lane + 32u];
        }
        uint64_t d_run = 0, c_run = 0, s_run = 0;
        for (uint64_t k = t; k < k_end; ++k) {
            const uint32_t i = A.idx[k];
            const ss_prepare_reply_rec R = A.rec[i];
            uint32_t v = SS_PREP_VERDICT_IGNORED, take = 0u;
            uint64_t nd = 0, nc = 0, ns = 0, dst = ~0ull, fill = 0u;
            if (R.kind != A.variant) {
                v = R.kind;
            } else if (R.slot < base) {
                v = SS_ACCEPT_VERDICT_STALE_SLOT;
            } else if (bps == 0u || R.ballot != bps || R.trigger_slot < base || R.trigger_slot - base >= 64u ||
                       ((filled >> (R.trigger_slot & 63u)) & 1u) || A.a_source[row + (R.trigger_slot & 63u)] != A.me) {
                // not this leader's Prepare at this ballot; a position the call filled is past the leader's endprep, so
                // never its trigger (and its replica_bk is written only after the walk)
                v = SS_PREP_VERDICT_IGNORED;
            } else if (R.slot - base >= 64u) {
                v = SS_ACCEPT_VERDICT_BEYOND_WINDOW;
            } else {
                const uint32_t w = static_cast<uint32_t>(R.slot - base), p = static_cast<uint32_t>(R.slot & 63u);
                const uint32_t tw = static_cast<uint32_t>(R.trigger_slot - base);
                // external fill (messages.rs:127-170): every position from the log end through the slot
                const uint64_t live = ring_to_window(prep | settled, r);
                const uint32_t end = live == 0u ? 0u : 64u - static_cast<uint32_t>(__clzll(static_cast<long long>(live)));
                if (w >= end) {
                    const uint64_t fw = below(w + 1u) & ~below(end), fm = window_to_ring(fw, r);
                    nc = static_cast<uint64_t>(__popcll(fw));
                    fill = fw;
                    filled |= fm;
                    prep |= fm;
                }
                const uint64_t bit = 1ull << p;
                const uint64_t ib = ((filled >> p) & 1u) ? bps : A.a_inst_bal[row + p];
                if (((prep & ~done) & bit) && R.ballot >= ib) {
                    // vote merge on the lane that keeps position p (ss_prepare_merge_dev's rule, one reply at a time)
                    const uint32_t owner = p & 31u;
                    uint32_t vv = SS_ACCEPT_VERDICT_ACCEPTED, tk = 0u;
                    uint64_t sv = 0u, dv = ~0ull;
                    if (lane == owner && R.vote_bal != 0u) {
                        const bool hi = p >= 32u;
                        uint64_t mb = hi ? mb_hi : mb_lo, of = hi ? of_hi : of_lo;
                        uint32_t mk = hi ? mk_hi : mk_lo, ln = hi ? ln_hi : ln_lo;
                        if (R.vote_bal > mb) {                           // a higher ballot: a new gathered codeword
                            mb = R.vote_bal; mk = R.vote_mask; ln = R.data_len;
                            sv = SS_CW_SLOT_PITCH((static_cast<uint64_t>(ln) + A.d - 1u) / A.d);
                            of = s_at + s_run;
                            tk = mk; dv = of;
                        } else if (R.vote_bal == mb) {
                            if (R.data_len != ln) {                      // absorb_other's error: this reply alone
                                vv = SS_PREP_VERDICT_DATA_LEN;
                            } else {
                                tk = R.vote_mask & ~mk; mk |= R.vote_mask; dv = of;
                            }
                        }
                        if (hi) { mb_hi = mb; of_hi = of; mk_hi = mk; ln_hi = ln; }
                        else { mb_lo = mb; of_lo = of; mk_lo = mk; ln_lo = ln; }
                    }
                    v = __shfl_sync(0xffffffffu, vv, owner);
                    take = __shfl_sync(0xffffffffu, tk, owner);
                    ns = __shfl_sync(0xffffffffu, sv, owner);
                    dst = __shfl_sync(0xffffffffu, dv, owner);
                    if (v == SS_ACCEPT_VERDICT_ACCEPTED && R.slot == R.endprep_slot) {
                        // the sender joins the quorum (messages.rs:197-323); every reply that leaves it at a majority
                        // is a decision point for the Preparing positions from the trigger on
                        const uint32_t before = static_cast<uint32_t>(__popc(acks));
                        acks |= 1u << A.frame_peer[i];
                        const uint32_t cnt = static_cast<uint32_t>(__popc(acks));
                        if (cnt >= A.majority) {
                            if (kApply && lane == 0u && before < A.majority) {
                                // the first quorum of the ballot: the engine's window is rebuilt from the acceptor
                                const uint64_t cm = A.a_committed[g];
                                A.window_base[g] = base;
                                A.committed[g] = cm;
                                A.commit_bar[g] = dev::commit_prefix(ring_to_window(cm, r));
                                A.accepting[g] = 0u;
                                for (uint32_t q = 0; q < A.population; ++q) A.planes[static_cast<uint64_t>(q) * A.G + g] = 0u;
                                A.bal_prepared[g] = bps;
                            }
                            const uint64_t cand = window_to_ring(ring_to_window(prep & ~done, r) & ~below(tw), r);
                            const auto cnt_f = [&] { return cnt; };
                            const uint32_t a_lo = ((cand >> lane) & 1u) ? prepare_action(mk_lo, cnt_f, A.d, A.data_mask, A.population, A.f) : 0u;
                            const uint32_t a_hi = ((cand >> (lane + 32u)) & 1u) ? prepare_action(mk_hi, cnt_f, A.d, A.data_mask, A.population, A.f) : 0u;
                            const uint64_t dec = static_cast<uint64_t>(__ballot_sync(0xffffffffu, a_lo != 0u)) |
                                                 (static_cast<uint64_t>(__ballot_sync(0xffffffffu, a_hi != 0u)) << 32);
                            const uint64_t nul = static_cast<uint64_t>(__ballot_sync(0xffffffffu, (a_lo & SS_PM_NULL) != 0u)) |
                                                 (static_cast<uint64_t>(__ballot_sync(0xffffffffu, (a_hi & SS_PM_NULL) != 0u)) << 32);
                            const uint64_t dec_w = ring_to_window(dec, r), nul_w = ring_to_window(nul, r);
                            const uint64_t null_at = s_at + s_run + ns;   // after the frame's own new slot, in slot order
                            nd = static_cast<uint64_t>(__popcll(dec));
                            ns += kNullPitch * static_cast<uint64_t>(__popcll(nul));
                            if (kApply) {
                                for (uint32_t h = 0; h < 2u; ++h) {
                                    const uint32_t q = lane + 32u * h;
                                    if (!((dec >> q) & 1u)) continue;
                                    const uint32_t qw = (q - r) & 63u;
                                    const uint64_t kd = d_at + d_run + static_cast<uint64_t>(__popcll(dec_w & below(qw)));
                                    uint64_t off = h ? of_hi : of_lo;
                                    uint32_t len = h ? ln_hi : ln_lo, pres = h ? mk_hi : mk_lo;
                                    if ((nul >> q) & 1u) {                  // RSCodeword::from_data(ReqBatch::new(), d, p)
                                        off = null_at + kNullPitch * static_cast<uint64_t>(__popcll(nul_w & below(qw)));
                                        len = 1u;
                                        pres = A.all_mask;
                                        for (uint32_t j = 0; j < A.T; ++j) {
                                            uint4 *z = reinterpret_cast<uint4 *>(A.shards + static_cast<uint64_t>(j) * A.plane_stride + off);
                                            z[0] = make_uint4(0u, 0u, 0u, 0u);    // shard_len 1, padded to 16
                                        }
                                        if (h) { of_hi = off; ln_hi = len; } else { of_lo = off; ln_lo = len; }
                                    }
                                    A.dec_slot[kd] = base + qw;
                                    A.dec_ballot[kd] = bps;
                                    A.dec_off[kd] = off;
                                    A.dec_len[kd] = len;
                                    A.dec_group[kd] = g;
                                    if (A.dec_policy != nullptr) A.dec_policy[kd] = A.policy != nullptr ? A.policy[g] : 0u;
                                    A.present[kd] = pres;
                                    if (A.cw_loc != nullptr) put_cw_loc(A.cw_loc, row + q, A.shards + off, A.plane_stride, len);
                                }
                                if (lane == 0u && dec != 0u) {
                                    uint64_t acc = A.accepting[g], cm = A.committed[g];
                                    for (uint64_t m = dec; m != 0u; m &= m - 1u) {
                                        const uint32_t q = static_cast<uint32_t>(__ffsll(static_cast<long long>(m)) - 1);
                                        enter_accepting(g, base + ((q - r) & 63u), acc, cm, A.planes, A.population, A.G, A.bal_prepared,
                                                        A.inst_bal, A.accepting, A.committed, A.policy_idx, A.policy, nullptr, nullptr, 0u,
                                                        0u);   // the owning lanes recorded the locations above
                                        acc |= 1ull << q;
                                        cm &= ~(1ull << q);
                                    }
                                }
                            }
                            done |= dec;
                        }
                    }
                }
            }
            if (kApply) {
                if (lane == 0u) {
                    A.verdict[i] = v;
                    A.dst[i] = v == SS_ACCEPT_VERDICT_ACCEPTED && take != 0u ? dst : ~0ull;
                    A.take[i] = take;
                    A.fill[i] = fill;
                }
            } else if (lane == 0u) {
                A.c_dec[k] = nd; A.c_cell[k] = nc; A.c_store[k] = ns;
            }
            d_run += nd; c_run += nc; s_run += ns;
        }
        if (kApply) {
            A.pa_max_bal[row + lane] = mb_lo; A.pa_max_bal[row + lane + 32u] = mb_hi;
            A.pa_off[row + lane] = of_lo; A.pa_off[row + lane + 32u] = of_hi;
            A.pa_mask[row + lane] = mk_lo; A.pa_mask[row + lane + 32u] = mk_hi;
            A.pa_len[row + lane] = ln_lo; A.pa_len[row + lane + 32u] = ln_hi;
            if (lane == 0u) {
                A.pa_ballot[g] = bps;
                A.pa_acks[g] = acks;
                A.pa_done[g] = done;
                A.a_preparing[g] = prep;
            }
        }
    }
    if (kApply && lane == 0u) {
        if (store_full) atomicOr(A.status, SS_DEV_STATUS_STORE_FULL);
        if (wal_full) atomicOr(A.status, SS_DEV_STATUS_FRAME_OVERFLOW);
    }
}

// 5. a warp per frame, in group order: its external fill (the PrepareBal cells and the acceptor's fresh instances) and
//    the shards it added, when the codeword they went to is still the position's (a later reply at a higher ballot, or
//    a NULL decision, abandons it)
__global__ void __launch_bounds__(kPaThreads) pa_write_kernel(const __grid_constant__ PaArgs A) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = (static_cast<uint64_t>(blockIdx.x) * kPaThreads + threadIdx.x) >> 5;
    const uint64_t nwarps = (static_cast<uint64_t>(gridDim.x) * kPaThreads) >> 5;
    for (uint64_t k = warp; k < A.n; k += nwarps) {
        const uint32_t i = A.idx[k];
        const uint64_t fw = A.fill[i], dst = A.dst[i];
        if (fw == 0u && dst == ~0ull) continue;
        const uint32_t g = A.key[k];
        const uint64_t row = static_cast<uint64_t>(g) * 64u;
        const ss_prepare_reply_rec R = A.rec[i];
        if (fw != 0u) {                                                 // external fill (messages.rs:127-170)
            const uint64_t base = A.a_base[g];
            const uint32_t r = static_cast<uint32_t>(base & 63u);
            const uint8_t span = A.a_prep_span[row + (R.trigger_slot & 63u)];
            for (uint32_t qw = lane; qw < 64u; qw += 32u) {
                if (!((fw >> qw) & 1u)) continue;
                const uint64_t cell = A.c_cell[k] + static_cast<uint64_t>(__popcll(fw & below(qw)));
                put_prepare_bal_cell(A.wal + cell * 32u, A.wal_variant, base + qw, R.ballot);
                A.rec_group[cell] = g;
                A.rec_slot[cell] = base + qw;
                const uint64_t at = row + ((qw + r) & 63u);             // a fresh null_instance(), Preparing at the ballot
                A.a_inst_bal[at] = R.ballot;
                A.a_source[at] = static_cast<uint8_t>(A.me);
                A.a_prep_trigger[at] = R.trigger_slot;
                A.a_prep_span[at] = span;
                A.a_held[at] = 0u;
                A.a_data_len[at] = 0u;
                A.a_voted_bal[at] = 0u;
                A.a_voted_mask[at] = 0u;
                if (A.a_assignment != nullptr) {
                    A.a_assignment[at] = 0u;
                    for (uint32_t m = 0; m < A.population; ++m) A.a_assign_rows[at * A.population + m] = 0u;
                }
            }
        }
        if (dst == ~0ull || A.pa_off[row + (R.slot & 63u)] != dst) continue;
        const uint32_t take = A.take[i];
        const uint64_t L = (static_cast<uint64_t>(R.data_len) + A.d - 1u) / A.d;
        const uint8_t *tags = A.buf + R.shards_at;
        uint64_t at = 0;
        for (uint32_t j = 0; j < A.T; ++j) {
            if (!((R.vote_mask >> j) & 1u)) { at += 1u; continue; }
            const uint64_t sl = some_len(tags[at + 1u]);
            if ((take >> j) & 1u) warp_fill_slot(A.shards + static_cast<uint64_t>(j) * A.plane_stride + dst, tags + at + sl, L, lane);
            at += sl + L;
        }
    }
}

// 6. a thread per group (and per decided record): pending, the store cursor, data_len 0 past the decided records so the
//    reconstruct launch over the whole capacity passes them by
__global__ void __launch_bounds__(kPaThreads) pa_finish_kernel(const __grid_constant__ PaArgs A, uint64_t items) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kPaThreads;
    const uint64_t n_dec = A.words[1];
    for (uint64_t x = static_cast<uint64_t>(blockIdx.x) * kPaThreads + threadIdx.x; x < items; x += stride) {
        if (x < A.G) {
            const uint64_t bps = A.bps[x];
            A.pending[x] = bps == 0u ? 0u : A.a_preparing[x] & ~(A.pa_ballot[x] == bps ? A.pa_done[x] : 0u);
        }
        if (x < A.dec_cap && x >= n_dec) A.dec_len[x] = 0u;
        if (x == 0u && A.words[0] != 0u) *A.store_used_out = ((*A.store_used_out + 31u) & ~31ull) + A.words[0];
    }
}

}  // namespace ssb

using namespace ssb;

namespace ssb {

void prepare_free(ss_engine *e) {
    void *bufs[] = {e->pa_ballot, e->pa_acks, e->pa_done, e->pa_max_bal, e->pa_off, e->pa_mask, e->pa_len, e->pa_rec, e->pa_cnt,
                    e->pa_dst, e->pa_fill, e->pa_take, e->pa_partials, e->pa_words, e->pa_present, e->pa_status};
    for (void *b : bufs)
        if (b) cudaFree(b);
}

// per-group and per-position bookkeeping on first use, per-frame and per-record scratch grow-only
static int prepare_scratch(ss_engine *e, uint64_t n, uint64_t dec_cap) {
    ss_ctx *ctx = e->ctx;
    const uint64_t G = e->G;
    if (e->pa_ballot == nullptr) {
        SS_TRY(dalloc(ctx, &e->pa_ballot, G)); SS_TRY(dalloc(ctx, &e->pa_acks, G)); SS_TRY(dalloc(ctx, &e->pa_done, G));
        SS_TRY(dalloc(ctx, &e->pa_max_bal, G * 64)); SS_TRY(dalloc(ctx, &e->pa_off, G * 64)); SS_TRY(dalloc(ctx, &e->pa_mask, G * 64));
        SS_TRY(dalloc(ctx, &e->pa_len, G * 64)); SS_TRY(dalloc(ctx, &e->pa_words, 5));
    }
    if (n > e->pa_cap) {
        SS_CUDA(cudaStreamSynchronize(ctx->stream));
        void *old[] = {e->pa_rec, e->pa_cnt, e->pa_dst, e->pa_fill, e->pa_take, e->pa_partials};
        for (void *b : old)
            if (b) cudaFree(b);
        e->pa_rec = nullptr; e->pa_cnt = nullptr; e->pa_dst = nullptr; e->pa_fill = nullptr; e->pa_take = nullptr; e->pa_partials = nullptr; e->pa_cap = 0;
        SS_TRY(dalloc(ctx, &e->pa_rec, n, false)); SS_TRY(dalloc(ctx, &e->pa_cnt, 3 * n, false)); SS_TRY(dalloc(ctx, &e->pa_dst, n, false));
        SS_TRY(dalloc(ctx, &e->pa_fill, n, false));
        SS_TRY(dalloc(ctx, &e->pa_take, n, false)); SS_TRY(dalloc(ctx, &e->pa_partials, scan_tiles(n), false));
        e->pa_cap = n;
    }
    if (dec_cap > e->pa_dec_cap) {
        SS_CUDA(cudaStreamSynchronize(ctx->stream));
        if (e->pa_present) cudaFree(e->pa_present);
        if (e->pa_status) cudaFree(e->pa_status);
        e->pa_present = nullptr; e->pa_status = nullptr; e->pa_dec_cap = 0;
        SS_TRY(dalloc(ctx, &e->pa_present, dec_cap, false)); SS_TRY(dalloc(ctx, &e->pa_status, dec_cap, false));
        e->pa_dec_cap = dec_cap;
    }
    return SS_OK;
}

}  // namespace ssb

extern "C" int ss_engine_prepare_absorb(ss_engine *e, ss_acceptor *a, const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off,
                                        const uint32_t *frame_group, const uint8_t *frame_peer, uint64_t n_frames,
                                        uint32_t reply_variant, uint32_t wal_variant, const uint64_t *bal_prep_sent,
                                        const uint8_t *policy, uint8_t *shards, uint64_t plane_stride, uint64_t *store_used,
                                        uint8_t *wal, uint64_t wal_capacity, uint32_t *rec_group, uint64_t *rec_slot,
                                        uint64_t rec_capacity, uint64_t *dec_slot, uint64_t *dec_ballot, uint64_t *dec_shard_off,
                                        uint32_t *dec_data_len, uint8_t *dec_policy, uint32_t *dec_group, uint64_t dec_capacity,
                                        uint64_t *pending, uint32_t *verdict, uint64_t *totals) {
    if (e == nullptr || a == nullptr) return set_error(SS_ERR_INVALID_ARG, "null engine or acceptor");
    if (e->cfg.protocol != SS_PROTO_RSPAXOS && e->cfg.protocol != SS_PROTO_CROSSWORD)
        return set_error(SS_ERR_INVALID_ARG, "the PrepareReply absorb serves RSPaxos and Crossword engines only");
    if (e->ctx != a->ctx || e->cfg.protocol != a->cfg.protocol || e->G != a->G || e->n != a->cfg.population ||
        e->d != a->cfg.data_shards || e->T != a->cfg.total_shards)
        return set_error(SS_ERR_INVALID_ARG, "the engine and the acceptor must share context, protocol, groups, population and code");
    if (reply_variant >= kVariantLimit || wal_variant >= kVariantLimit)
        return set_error(SS_ERR_INVALID_ARG, "reply_variant and wal_variant must be below 2^16");
    if (!e->coder->batch_ok || !e->coder->dec_ok)
        return set_error(SS_ERR_UNSUPPORTED, "the batched reconstruct needs d+p <= 12 (code is %u,%u)", e->d, e->T - e->d);
    if (!bal_prep_sent || !shards || !store_used || !wal || !rec_group || !rec_slot || !dec_slot || !dec_ballot || !dec_shard_off ||
        !dec_data_len || !dec_group || !pending || (n_frames != 0 && (!buf || !frame_off || !frame_group || !frame_peer || !verdict)))
        return set_error(SS_ERR_INVALID_ARG, "null buffer");
    if ((plane_stride & 31u) || plane_stride == 0) return set_error(SS_ERR_INVALID_ARG, "plane_stride must be a non-zero multiple of 32");
    if ((reinterpret_cast<uintptr_t>(shards) | reinterpret_cast<uintptr_t>(wal)) & 15u)
        return set_error(SS_ERR_INVALID_ARG, "the shard store and wal must be 16-byte aligned");
    if (n_frames > 0x7fffffffull) return set_error(SS_ERR_INVALID_ARG, "at most 2^31 - 1 frames per call");
    if (e->cw_loc != nullptr && plane_stride >= kCwLocStrideLimit)
        return set_error(SS_ERR_INVALID_ARG, "a Crossword engine's plane_stride must be below 2^36");
    ss_ctx *ctx = e->ctx;
    SS_TRY(ctx_bind(ctx));
    SS_TRY(prepare_scratch(e, n_frames, dec_capacity));
    PaArgs A{};
    A.buf = buf; A.buf_len = buf_len; A.frame_off = frame_off; A.frame_group = frame_group; A.frame_peer = frame_peer;
    A.n = n_frames; A.G = e->G; A.d = e->d; A.T = e->T; A.population = e->n; A.majority = e->majority; A.f = e->cfg.fault_tolerance;
    A.me = a->cfg.me; A.variant = reply_variant; A.wal_variant = wal_variant;
    A.data_mask = e->d >= 32u ? 0xffffffffu : (1u << e->d) - 1u;
    A.all_mask = e->T >= 32u ? 0xffffffffu : (1u << e->T) - 1u;
    A.bps = bal_prep_sent; A.policy = policy;
    A.a_base = a->window_base; A.a_accepting = a->accepting; A.a_committed = a->committed; A.a_preparing = a->preparing;
    A.a_inst_bal = a->inst_bal; A.a_voted_bal = a->voted_bal; A.a_prep_trigger = a->prep_trigger; A.a_held = a->held;
    A.a_data_len = a->data_len; A.a_voted_mask = a->voted_mask; A.a_assignment = a->assignment; A.a_assign_rows = a->assign_rows;
    A.a_source = a->source; A.a_prep_span = a->prep_span;
    A.planes = e->planes; A.bal_prepared = e->bal_prepared; A.inst_bal = e->inst_bal; A.accepting = e->accepting;
    A.committed = e->committed; A.window_base = e->window_base; A.commit_bar = e->commit_bar; A.policy_idx = e->policy_idx;
    A.cw_loc = e->cw_loc;
    A.pa_ballot = e->pa_ballot; A.pa_done = e->pa_done; A.pa_max_bal = e->pa_max_bal; A.pa_off = e->pa_off; A.pa_acks = e->pa_acks;
    A.pa_mask = e->pa_mask; A.pa_len = e->pa_len;
    A.rec = e->pa_rec;
    A.c_dec = e->pa_cnt; A.c_cell = e->pa_cnt + n_frames; A.c_store = e->pa_cnt + 2 * n_frames;
    uint64_t *tot = totals != nullptr ? totals : e->pa_words + 2;
    A.tot = tot; A.words = e->pa_words; A.dst = e->pa_dst; A.fill = e->pa_fill; A.take = e->pa_take; A.present = e->pa_present;
    A.store_used = store_used; A.store_used_out = store_used; A.store_cap = plane_stride;
    const uint64_t wal_cells = wal_capacity / 32u;
    A.cell_cap = rec_capacity < wal_cells ? rec_capacity : wal_cells;
    A.dec_cap = dec_capacity;
    A.shards = shards; A.plane_stride = plane_stride; A.wal = wal; A.rec_group = rec_group; A.rec_slot = rec_slot;
    A.dec_slot = dec_slot; A.dec_ballot = dec_ballot; A.dec_off = dec_shard_off; A.dec_len = dec_data_len; A.dec_group = dec_group;
    A.dec_policy = dec_policy; A.pending = pending; A.verdict = verdict; A.status = ctx->dev_status;
    SS_CUDA(cudaMemsetAsync(e->pa_words, 0, 16, ctx->stream));
    if (n_frames != 0) {
        SS_TRY(backoff_scratch(e, n_frames, key_bits(e->G)));
        A.key_in = e->bo_keys; A.idx_in = e->bo_idx; A.key = e->bo_keys + n_frames; A.idx = e->bo_idx + n_frames;
        const uint32_t grid_t = launch_grid(ctx, n_frames, kPaThreads), grid_w = launch_grid(ctx, n_frames, kPaThreads / 32);
        pa_decode_kernel<<<grid_t, kPaThreads, 0, ctx->stream>>>(A);
        SS_TRY(launched(ctx));
        size_t bytes = e->bo_sort_bytes;
        SS_CUDA(cub::DeviceRadixSort::SortPairs(e->bo_sort_tmp, bytes, e->bo_keys, e->bo_keys + n_frames, e->bo_idx, e->bo_idx + n_frames,
                                                static_cast<int>(n_frames), 0, key_bits(e->G), ctx->stream));
        SS_TRY(launched(ctx));
        pa_walk_kernel<false><<<grid_w, kPaThreads, 0, ctx->stream>>>(A);
        SS_TRY(launched(ctx));
        for (int c = 0; c < 3; ++c) SS_TRY(launch_exclusive_scan_u64(ctx, e->pa_cnt + c * n_frames, n_frames, e->pa_partials, tot + c));
        pa_walk_kernel<true><<<grid_w, kPaThreads, 0, ctx->stream>>>(A);
        SS_TRY(launched(ctx));
        pa_write_kernel<<<grid_w, kPaThreads, 0, ctx->stream>>>(A);
        SS_TRY(launched(ctx));
    } else if (totals != nullptr) {
        SS_CUDA(cudaMemsetAsync(totals, 0, 24, ctx->stream));
    }
    const uint64_t items = e->G > dec_capacity ? e->G : dec_capacity;
    pa_finish_kernel<<<launch_grid(ctx, items, kPaThreads), kPaThreads, 0, ctx->stream>>>(A, items);
    SS_TRY(launched(ctx));
    if (n_frames == 0) return SS_OK;
    e->windowed = true;                                                 // a quorum's rebuild installs the acceptor's bases
    if (dec_capacity == 0) return SS_OK;
    // USE codewords: the shards they lack regenerated in place, parity included; NULL ones are intact (present = all).
    // No record can lack shards (a USE codeword holds at least d), so the per-record status is not read: a non-zero one
    // is only the null-codeword status of the entries past the decided count (data_len 0), which nothing packs.
    return ss_rs_reconstruct_batch_dev(e->coder, shards, plane_stride, dec_shard_off, dec_data_len, e->pa_present, dec_capacity, 0,
                                       e->pa_status, SS_RS_OUT_PADDED16);
}
