/*
 * ss_oracle.h -- CPU ORACLE for the Summerset quorum-tally + Reed-Solomon hot path.
 *
 * THIS IS TEST INFRASTRUCTURE, NOT THE PRODUCT.  Only tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline / --impl reference legs may load it.  The product
 * (summerset_b200/csrc, libsummerset_b200.so) never links, imports or calls it.
 *
 * It is a plain-C restatement of the reference's Rust path (josehu07/summerset @ 1daf80aa;
 * paths relative to the reference tree's root):
 *   src/utils/rscoding.rs            RSCodeword geometry / encode / reconstruct / verify
 *   src/utils/bitmap.rs              Bitmap (replica-id / shard-id bitset)
 *   src/protocols/multipaxos/messages.rs:370-443   MultiPaxos accept-reply tally
 *   src/protocols/rspaxos/messages.rs:395-465      RSPaxos tally (majority + fault_tolerance)
 *   src/protocols/crossword/messages.rs:15-62,481-574  coverage_under_faults + tally
 *   src/protocols/crossword/adaptive.rs:98-106, mod.rs:866-888  balanced round-robin assignment
 *   src/protocols/multipaxos/durability.rs:148-218 commit_bar advance
 *   src/protocols/raft/messages.rs:243-309         match-index commit scan
 *   src/protocols/craft/messages.rs:288-314        CRaft thresholds
 * and of the un-vendored crate `reed-solomon-erasure ^6.0` (Cargo.toml:43; Cargo.lock is
 * git-ignored so no exact version is pinned) -- galois_8 field, Backblaze-style
 * Vandermonde-derived systematic matrix.
 *
 * PINNING STATUS (see DESIGN.md "Oracle"):
 *   - pinned against every assertion of the reference's own unit tests for this path
 *     (rscoding.rs:685-877, bitmap.rs:312-420): geometry, null codeword, subset/absorb,
 *     verify-after-encode, reconstruct under erasures, error cases.
 *   - PARITY-BYTE VALUES AND COMMIT BITMAPS: **parity unpinned** by the reference tree --
 *     the reference holds no golden parity bytes and no handler unit tests, and it cannot be
 *     compiled here (no cargo/rustc, no network).  They are anchored instead on the published
 *     algorithm of the crate (Backblaze JavaReedSolomon construction) and its upstream
 *     known-answer tests (recalled, labelled as such in tests/test_oracle_kat.py).
 */
#ifndef SS_ORACLE_H
#define SS_ORACLE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* error codes mirroring reed_solomon_erasure::Error (crate enum order) */
enum {
    SSOR_OK = 0,
    SSOR_ERR_TOO_FEW_SHARDS = -1,
    SSOR_ERR_TOO_MANY_SHARDS = -2,
    SSOR_ERR_TOO_FEW_DATA_SHARDS = -3,
    SSOR_ERR_TOO_MANY_DATA_SHARDS = -4,
    SSOR_ERR_TOO_FEW_PARITY_SHARDS = -5,
    SSOR_ERR_TOO_MANY_PARITY_SHARDS = -6,
    SSOR_ERR_INCORRECT_SHARD_SIZE = -9,
    SSOR_ERR_TOO_FEW_SHARDS_PRESENT = -10,
    SSOR_ERR_EMPTY_SHARD = -11,
    SSOR_ERR_INVALID_ARG = -20,
    SSOR_ERR_SINGULAR = -21
};

/* ---- GF(2^8), poly 0x11D, generator 2 (crate galois_8) ---- */
uint8_t ssor_gf_mul(uint8_t a, uint8_t b);
uint8_t ssor_gf_div(uint8_t a, uint8_t b);          /* b != 0 */
uint8_t ssor_gf_exp(uint8_t a, unsigned n);
uint8_t ssor_gf_log(uint8_t a);                     /* a != 0 */
uint8_t ssor_gf_exp_table(unsigned i);              /* EXP[i], i < 510 */

/* ---- coding matrix: (d+p) x d, row-major; top d x d is identity ---- */
int ssor_rs_build_matrix(int d, int p, uint8_t *out);
/* invert an n x n matrix in GF(2^8) (row-major, in -> out) */
int ssor_gf_matrix_invert(int n, const uint8_t *in, uint8_t *out);
/* decode rows for the given present mask: picks the first d present shards (index order),
 * writes their indices to src_idx[d] and the d x d inverse (row r = coefficients that
 * regenerate data shard r from those d sources) to dec. */
int ssor_rs_decode_matrix(int d, int p, const uint8_t *present, int *src_idx, uint8_t *dec);

/* ---- single-codeword coder ops (crate: encode / reconstruct / reconstruct_data / verify) ----
 * shards: array of d+p pointers to shard_len bytes each. */
int ssor_rs_encode(int d, int p, uint8_t *const *shards, size_t shard_len);
int ssor_rs_reconstruct(int d, int p, uint8_t *const *shards, uint8_t *present,
                        size_t shard_len, int data_only);
int ssor_rs_verify(int d, int p, const uint8_t *const *shards, size_t shard_len, int *ok);

/* ---- RSCodeword geometry (rscoding.rs:165-220) ---- */
size_t ssor_cw_shard_len(size_t data_len, int d);
/* copy + zero-pad `data` into d contiguous data shards of shard_len bytes: out[d*shard_len] */
void ssor_cw_split(const uint8_t *data, size_t data_len, int d, uint8_t *out);

/* ---- batched CPU path (baseline + parity checker for the GPU batch API) ----
 * codeword g: payload bytes data[data_off[g] .. +data_len[g]); L_g = ceil(len/d).
 * parity shard j of codeword g is written to parity[j*plane_stride + par_off[g] .. +L_g).
 * mode: 0 = scalar MUL_TABLE loops (crate default), 1 = AVX2 vpshufb nibble tables
 * (what the crate's simd-accel gives), falls back to 0 if the CPU lacks AVX2.
 * threads: OpenMP threads (<=0: all).  mode | SSOR_MODE_STATIC: one contiguous block of codewords per thread
 * instead of dynamic chunks of 256 (uniform batches on NUMA hosts: see ssor_first_touch_fill). */
#define SSOR_MODE_STATIC 0x100
int ssor_rs_encode_batch(int d, int p, const uint8_t *data, const uint64_t *data_off,
                         const uint32_t *data_len, uint64_t n, uint8_t *parity,
                         uint64_t plane_stride, const uint64_t *par_off, int mode, int threads);
/* shards laid out as shard j of codeword g at shards[j*plane_stride + off[g] .. +L_g);
 * present[g] bitmask (bit j = shard j available). Regenerates missing data shards (and
 * missing parity when !data_only) in place; status[g] = 0 / SSOR_ERR_TOO_FEW_SHARDS_PRESENT. */
int ssor_rs_reconstruct_batch(int d, int p, uint8_t *shards, uint64_t plane_stride,
                              const uint64_t *off, const uint32_t *data_len,
                              const uint32_t *present, uint64_t n, int data_only,
                              int32_t *status, int mode, int threads);
void ssor_first_touch_fill(uint8_t *buf, uint64_t n_items, uint64_t item_bytes, uint64_t item_stride,
                           uint64_t seed, int zero, int threads);
int ssor_have_avx2(void);
int ssor_max_threads(void);

/* ---- quorum tallies ---- */
/* Incremental per-ack restatement of handle_msg_accept_reply
 * (multipaxos/messages.rs:370-443; rspaxos/messages.rs:395-465 with another threshold).
 * State (caller-allocated, S slots per group): bal_prepared[g], inst_bal[g*S+s],
 * status[g*S+s] (SSOR_ST_*), acks[g*S+s] (bitmask over replica ids).
 * Records i: group rec_g[i], slot rec_s[i], peer rec_p[i], ballot rec_b[i]. */
enum { SSOR_ST_NULL = 0, SSOR_ST_PREPARING = 1, SSOR_ST_ACCEPTING = 2,
       SSOR_ST_COMMITTED = 3, SSOR_ST_EXECUTED = 4 };
void ssor_tally_stream(const uint32_t *rec_g, const uint8_t *rec_s, const uint8_t *rec_p,
                       const uint64_t *rec_b, uint64_t n_rec, uint32_t S, uint32_t population,
                       uint32_t threshold, const uint64_t *bal_prepared, const uint64_t *inst_bal,
                       uint8_t *status, uint16_t *acks);
/* batch (bit-plane) form: planes[r*G+g] bit s = valid ack of replica r for slot s. */
void ssor_tally_planes(const uint64_t *planes, uint32_t R, uint64_t G, uint32_t threshold,
                       uint64_t *committed, uint32_t *commit_bar, int threads);
/* per-instance vote-mask form: masks[i] = Bitmap of acks (bit r), count() >= threshold */
void ssor_tally_masks(const uint16_t *masks, uint64_t n, uint32_t threshold, uint8_t *commit);
/* commit_bar = length of committed prefix of the 64-slot window (durability.rs:148-218) */
void ssor_tally_stream_crossword(const uint32_t *rec_g, const uint8_t *rec_s, const uint8_t *rec_p,
                                 const uint64_t *rec_b, uint64_t n_rec, uint32_t S, uint32_t population,
                                 uint32_t T, uint32_t d, uint32_t majority, uint32_t f, int balanced,
                                 const uint32_t *policies, uint32_t n_policies, const uint8_t *policy_idx,
                                 const uint64_t *bal_prepared, const uint64_t *inst_bal, uint8_t *status,
                                 uint16_t *acks);
uint32_t ssor_commit_bar(uint64_t committed_word);

/* ---- Crossword ---- */
/* balanced round-robin assignment (crossword/mod.rs:866-888): replica r holds shards
 * {(r*dj + k) mod T : k in [0,spr)}, dj = T/n.  out[r] = bitmask over shard ids. */
void ssor_cw_brr_assignment(uint32_t n, uint32_t T, uint32_t spr, uint32_t *out);
/* min_shards_per_replica (crossword/adaptive.rs:98-106) */
uint32_t ssor_cw_min_spr(uint32_t d, uint32_t majority, uint32_t f, uint32_t alive);
/* coverage_under_faults (crossword/messages.rs:15-62). ack_mask: replicas that acked;
 * assignment[r]: shard bitmask of replica r. */
uint32_t ssor_cw_coverage(uint32_t T, uint32_t n, uint32_t ack_mask, const uint32_t *assignment,
                          uint32_t f, int balanced);
/* commit predicate (crossword/messages.rs:535-542) */
int ssor_cw_committed(uint32_t T, uint32_t n, uint32_t d, uint32_t majority, uint32_t f,
                      uint32_t ack_mask, const uint32_t *assignment, int balanced);

/* ---- Raft / CRaft match-index scan (raft/messages.rs:256-275) ----
 * match[p] for the npeers = population-1 peers (self excluded); log entries
 * last_commit+1 .. log_end-1 have terms terms[slot - (last_commit+1)].
 * threshold = quorum_cnt (Raft) or majority+f / majority (CRaft). */
uint32_t ssor_raft_scan(const uint32_t *match, uint32_t npeers, uint32_t last_commit,
                        uint32_t log_end, uint32_t curr_term, const uint32_t *terms,
                        uint32_t threshold);
/* last_snap scan (raft/messages.rs:298-309): match_cnt == population */
uint32_t ssor_raft_snap_scan(const uint32_t *match, uint32_t npeers, uint32_t last_snap,
                             uint32_t end_slot);
void ssor_raft_scan_batch(const uint32_t *match, uint32_t npeers, uint64_t G,
                          const uint32_t *last_commit, const uint32_t *log_end,
                          const uint32_t *curr_term, const uint32_t *terms, uint32_t W,
                          uint32_t threshold, uint32_t *new_commit, int threads);

/* ---- CRaft (SURVEY 8f-1) ----
 * commit threshold (craft/messages.rs:300-308): full_copy_mode ? majority : majority + fault_tolerance */
void ssor_raft_reply_stream(const uint32_t *rec_g, const uint8_t *rec_peer, const uint32_t *rec_end,
                            uint64_t n_rec, uint32_t npeers, uint32_t threshold, uint64_t G, uint32_t *next_slot,
                            uint32_t *match, uint32_t *last_commit, uint32_t *last_snap, const uint32_t *log_end,
                            const uint32_t *curr_term, const uint32_t *terms, uint32_t W);
uint32_t ssor_craft_threshold(uint32_t majority, uint32_t fault_tolerance, int full_copy_mode);
/* shadow_last_commit (craft/messages.rs:677-690): peers' match slots sorted descending, element
 * [threshold - 2]; i.e. the (threshold-1)-th largest peer match */
uint32_t ssor_craft_shadow_last_commit(const uint32_t *match, uint32_t npeers, uint32_t threshold);

/* ---- prepare-phase shard merge (SURVEY 8f-3) ----
 * Incremental restatement of the PrepareReply bookkeeping (rspaxos/messages.rs:182-196,
 * crossword/messages.rs:233-248) for ONE instance: replies i = 0..n_rep-1 in arrival order, reply i
 * has_vote[i] ? (bal[i], shard mask[i]) : None.  Outputs the final prepare_max_bal and the shard set
 * held by inst.reqs_cw (absorb_other keeps what is already there, so the set is the union). */
void ssor_prepare_merge_stream(const uint8_t *has_vote, const uint64_t *bal, const uint32_t *mask,
                               uint32_t n_rep, uint64_t *max_bal, uint32_t *merged);
/* decision once prepare_acks_cnt >= majority (rspaxos/messages.rs:227-259, crossword/messages.rs:279-312):
 * bit0 USE (>= d shards of the highest ballot), bit1 NULL (fewer, but acks >= n - f), neither = wait;
 * bit2 needs reconstruct_data (avail data shards < d), bit3 needs compute_parity (avail shards <
 * POPULATION -- the reference compares with population, not rs_total_shards; SURVEY 8a.10). */
enum { SSOR_PM_USE = 1, SSOR_PM_NULL = 2, SSOR_PM_RECONSTRUCT = 4, SSOR_PM_PARITY = 8 };
uint32_t ssor_prepare_decide(uint32_t merged, uint32_t acks_cnt, uint32_t data_shards, uint32_t population,
                             uint32_t fault_tolerance);

/* ---- Crossword follower gossip planning (SURVEY 8f-4; crossword/gossiping.rs:35-84) ----
 * gossip_targets_excl for ONE instance: greedily walk peers me+1, me+2, ... (mod n), skipping the source peer and
 * peers not alive; a peer is selected when its assigned shards include one not yet available/asked for; the
 * exclusion set sent to it is the availability map at that moment.  Stops once >= d shards are covered.
 * assignment[r] = shard bitmask of replica r.  Returns the selected-peer bitmask; excl[peer] is written for the
 * selected peers (others left untouched). */
uint32_t ssor_gossip_targets_excl(uint32_t me, uint32_t population, uint32_t data_shards, uint32_t src_peer,
                                  uint32_t avail, const uint32_t *assignment, uint32_t peer_alive, uint32_t *excl);


/* ---- wire / WAL byte formats and reconstruct serving (ss_wire.c; SURVEY 8f-2, 8f-4) ---- */
size_t ssor_varint_put(uint8_t *out, uint64_t v);
size_t ssor_varint_get(const uint8_t *in, size_t avail, uint64_t *v);
size_t ssor_bitmap_encode(uint32_t size, uint64_t bits, uint8_t *out);
size_t ssor_rscodeword_encode(uint32_t d, uint32_t p, uint64_t data_len, uint64_t shard_len,
                              const uint8_t *const *shards, uint8_t *out);
size_t ssor_frame_accept(uint32_t accept_variant, uint64_t slot, uint64_t ballot, uint32_t d, uint32_t p,
                         uint64_t data_len, uint64_t shard_len, const uint8_t *const *shards,
                         const uint32_t *assignment, uint32_t n_assign, uint32_t assign_size, uint8_t *out);
size_t ssor_frame_accept_reply(uint32_t reply_variant, uint64_t slot, uint64_t ballot, int with_size, uint64_t size,
                               uint8_t *out);
long ssor_parse_accept_reply(const uint8_t *frame, size_t avail, uint32_t reply_variant, int with_size,
                             uint64_t *slot, uint64_t *ballot, uint64_t *size, uint32_t *kind);
size_t ssor_wal_accept_data(uint64_t slot, uint64_t ballot, uint32_t d, uint32_t p, uint64_t data_len,
                            uint64_t shard_len, const uint8_t *const *shards, uint8_t *out);
size_t ssor_wal_commit_slot(uint64_t slot, uint8_t *out);
long ssor_decode_accept(const uint8_t *frame, size_t avail, int kind, uint32_t *variant, uint64_t *slot, uint64_t *ballot,
                        uint32_t *d, uint32_t *p, uint64_t *data_len, uint64_t *shard_len, uint64_t *shard_at,
                        uint32_t max_shards, int with_assignment, uint32_t *assignment, uint32_t *n_assign,
                        uint32_t *assign_size);
uint32_t ssor_reconstruct_serve_mask(uint32_t held, uint32_t exclude, uint32_t total_shards, int status);

#ifdef __cplusplus
}
#endif
#endif
