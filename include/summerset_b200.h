/*
 * summerset_b200.h -- C ABI of libsummerset_b200.so
 *
 * The H100 (sm_90a) implementation of Summerset's quorum-tally + Reed-Solomon hot path.
 * Plain C: pointers and sizes only, no torch / C++ types.  This is the boundary a Rust
 * `extern "C"` block (INTEGRATION.md) binds; the GenericReplica / SmrProtocol surface
 * (src/server/replica.rs:15-42, src/protocols/mod.rs:118-215) is untouched by it.
 *
 * The reference has no FFI for this path (SURVEY.md 8b).  Each entry point states the reference
 * interface it replaces (path:line relative to the reference tree, josehu07/summerset @ 1daf80aa).
 *
 * Conventions
 *   - Ownership: the caller owns every buffer.  The library never frees or retains caller
 *     memory (rscoding.rs:479-484, :515-517 -- encode/reconstruct mutate caller slices in place).
 *   - Errors: `int` return, 0 = ok, negative = error.  Codes -1..-13 mirror the variants of
 *     `reed_solomon_erasure::Error`, which the reference converts into `SummersetError(String)`
 *     (src/utils/error.rs:6-14,59); ss_last_error() gives the message text for that conversion.
 *   - Threading: every call may come from a different OS thread (the replica's run() task
 *     migrates across tokio worker threads, summerset_server/src/main.rs:45-47,133-137).  No
 *     thread-local CUDA state is assumed: each call binds its handle's device.  Calls on ONE
 *     handle must be serialised by the caller (the reference calls from a single task).
 *   - `_dev` entry points take DEVICE pointers and are asynchronous on the context's stream;
 *     the others take HOST pointers, copy in/out and return when the result is in host memory.
 *   - No CPU fallback: every compute entry point fails with SS_ERR_NO_DEVICE / SS_ERR_CUDA when
 *     no sm_90 device is usable.
 */
#ifndef SUMMERSET_B200_H
#define SUMMERSET_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SS_VERSION 200 /* 0.2.0: engine, step flags, wire formats, uniform reconstruct; several round-1 signatures gained a parameter */

/* ---- error codes ---------------------------------------------------------------------------
 * -1..-13: reed_solomon_erasure::Error variants in declaration order. */
enum {
    SS_OK = 0,
    SS_ERR_TOO_FEW_SHARDS = -1,
    SS_ERR_TOO_MANY_SHARDS = -2,
    SS_ERR_TOO_FEW_DATA_SHARDS = -3,
    SS_ERR_TOO_MANY_DATA_SHARDS = -4,
    SS_ERR_TOO_FEW_PARITY_SHARDS = -5,
    SS_ERR_TOO_MANY_PARITY_SHARDS = -6,
    SS_ERR_TOO_FEW_BUFFER_SHARDS = -7,
    SS_ERR_TOO_MANY_BUFFER_SHARDS = -8,
    SS_ERR_INCORRECT_SHARD_SIZE = -9,
    SS_ERR_TOO_FEW_SHARDS_PRESENT = -10,
    SS_ERR_EMPTY_SHARD = -11,
    SS_ERR_INVALID_SHARD_FLAGS = -12,
    SS_ERR_INVALID_INDEX = -13,
    /* library-level */
    SS_ERR_INVALID_ARG = -20,
    SS_ERR_UNSUPPORTED = -21,
    SS_ERR_OUT_OF_MEMORY = -22,
    SS_ERR_NO_DEVICE = -30,   /* no CUDA device / not sm_90: there is NO CPU fallback */
    SS_ERR_CUDA = -31
};

typedef struct ss_ctx ss_ctx;           /* device + stream + scratch */
typedef struct ss_rs_coder ss_rs_coder; /* replaces reed_solomon_erasure::galois_8::ReedSolomon */

int ss_version(void);
/* Text of the most recent error raised on the CALLING thread (one buffer per OS thread; the pointer stays valid until
 * the next failing call on that thread).  Read it right after the failing call, before yielding: two replicas driven
 * from two tokio worker threads never see each other's text.  Maps to SummersetError::msg (src/utils/error.rs:6-14). */
const char *ss_last_error(void);
const char *ss_strerror(int code);

/* ---- context ------------------------------------------------------------------------------- */
/* Creates a context on `device` with its own non-blocking stream. */
int ss_ctx_create(int device, ss_ctx **out);
/* Same, but launches on a caller-owned cudaStream_t (e.g. torch's current stream). */
int ss_ctx_create_on_stream(int device, void *cuda_stream, ss_ctx **out);
/* Coders / engines created on a context keep it alive: destroying the context before them only marks it closed and the
 * last handle's destroy call frees it (either order is safe). */
int ss_ctx_destroy(ss_ctx *ctx);
int ss_ctx_sync(ss_ctx *ctx);               /* cudaStreamSynchronize on the context's stream */
void *ss_ctx_stream(ss_ctx *ctx);           /* the cudaStream_t */
int ss_ctx_sm_count(ss_ctx *ctx);
/* number of kernels this context has launched so far (bench.py's gpu_launches claim) */
uint64_t ss_ctx_launch_count(ss_ctx *ctx);

/* device / pinned-host memory helpers for non-CUDA callers (Rust shim) */
int ss_dev_alloc(ss_ctx *ctx, size_t bytes, void **dptr);
int ss_dev_free(ss_ctx *ctx, void *dptr);
int ss_dev_memset(ss_ctx *ctx, void *dptr, int value, size_t bytes);      /* async */
int ss_host_alloc(ss_ctx *ctx, size_t bytes, void **hptr);                /* pinned */
/* write-combined pinned memory: for buffers the CPU only WRITES and the GPU reads (payload staging); faster H2D on
 * some hosts, very slow for CPU reads */
int ss_host_alloc_wc(ss_ctx *ctx, size_t bytes, void **hptr);
int ss_host_free(ss_ctx *ctx, void *hptr);
int ss_copy_h2d(ss_ctx *ctx, void *dst_dev, const void *src_host, size_t bytes); /* async */
int ss_copy_d2h(ss_ctx *ctx, void *dst_host, const void *src_dev, size_t bytes); /* async */

int ss_copy_d2d(ss_ctx *ctx, void *dst_dev, const void *src_dev, size_t bytes);  /* async; dst/src may be peer memory */

/* ---- cross-process peer memory (one process per GPU, NVLink) ---------------------------------
 * ss_ipc_export gives a 64-byte handle for a buffer obtained from ss_dev_alloc; another process on the same
 * box turns it into a device pointer with ss_ipc_open (peer access is enabled on first use).  The pointers
 * can be passed to ss_accept_step_replicate_dev / ss_copy_d2d: kernels then store straight into the peer
 * GPU's HBM over NVLink -- the replacement for TransportHub::send_msg of a shard (server/transport.rs:258-345,
 * rspaxos/request.rs:127-142) when the simulated replicas of a group live on the GPUs of one box. */
#define SS_IPC_HANDLE_BYTES 64
int ss_ipc_export(ss_ctx *ctx, void *dptr, uint8_t handle[SS_IPC_HANDLE_BYTES]);
int ss_ipc_open(ss_ctx *ctx, const uint8_t handle[SS_IPC_HANDLE_BYTES], void **dptr);
int ss_ipc_close(ss_ctx *ctx, void *dptr);

/* ---- Reed-Solomon coder --------------------------------------------------------------------
 * Replaces ReedSolomon::new(d, p) (constructors at rspaxos/mod.rs:606, crossword/mod.rs:827,
 * craft/mod.rs:534, benches/rse_bench.rs:51).  GF(2^8) poly 0x11D; systematic matrix
 * M = vandermonde(d+p, d) * inverse(top d x d) -- bit-identical to the crate's.
 * Errors: d == 0 -> TOO_FEW_DATA_SHARDS, p == 0 -> TOO_FEW_PARITY_SHARDS, d+p > 256 ->
 * TOO_MANY_SHARDS (the crate's behaviour; Summerset special-cases p == 0 before touching the
 * coder, rscoding.rs:454-456,498-507).  Any such code gets a coder, but the kernels cover less:
 *   encode (ss_rs_encode, ss_rs_verify and every batched encode / accept step) needs d <= 32 and p <= 8,
 *     so up to 40 shards;
 *   reconstruct (ss_rs_reconstruct, ss_rs_reconstruct_data, ss_rs_reconstruct_batch_dev and
 *     ss_rs_reconstruct_uniform_dev) needs d + p <= 12 as well.
 * Past those limits the calls return SS_ERR_UNSUPPORTED and write nothing, except where no work is
 * left: a single-codeword reconstruct with every shard it would regenerate already present returns
 * SS_OK for any code. */
int ss_rs_coder_create(ss_ctx *ctx, int data_shards, int parity_shards, ss_rs_coder **out);
int ss_rs_coder_destroy(ss_rs_coder *coder);
int ss_rs_data_shard_count(const ss_rs_coder *coder);    /* rscoding.rs:428 */
int ss_rs_parity_shard_count(const ss_rs_coder *coder);  /* rscoding.rs:434 */
int ss_rs_total_shard_count(const ss_rs_coder *coder);
/* copies the (d+p) x d coding matrix, row-major, into out */
int ss_rs_coder_matrix(const ss_rs_coder *coder, uint8_t *out);

/* -- one codeword, HOST slices: the four crate methods RSCodeword calls ----------------------
 * shards: n_shards (= d+p) pointers to shard_len bytes each.
 * ss_rs_encode            replaces rs.encode(slices)             (rscoding.rs:484)
 * ss_rs_reconstruct       replaces rs.reconstruct(&mut shards)   (rscoding.rs:517)
 * ss_rs_reconstruct_data  replaces rs.reconstruct_data(..)       (rscoding.rs:515)
 * ss_rs_verify            replaces rs.verify(&slices)            (rscoding.rs:575)
 * present[j] != 0 <=> shards[j] is Some(..); missing entries must still point at a
 * shard_len-byte buffer to fill (the crate allocates it; here the caller does).  On success
 * present[] is updated for the regenerated shards.  ss_rs_reconstruct_data neither reads nor
 * writes missing parity entries (they may all alias one scratch buffer) and leaves their present[]
 * at 0.  Fewer than d present -> SS_ERR_TOO_FEW_SHARDS_PRESENT and no output is written (never
 * partial). */
int ss_rs_encode(ss_rs_coder *coder, uint8_t *const *shards, size_t n_shards, size_t shard_len);
int ss_rs_reconstruct(ss_rs_coder *coder, uint8_t *const *shards, uint8_t *present,
                      size_t n_shards, size_t shard_len);
int ss_rs_reconstruct_data(ss_rs_coder *coder, uint8_t *const *shards, uint8_t *present,
                           size_t n_shards, size_t shard_len);
int ss_rs_verify(ss_rs_coder *coder, const uint8_t *const *shards, size_t n_shards,
                 size_t shard_len, int *ok);

/* -- batched, device-resident log of codewords ------------------------------------------------
 * Codeword g: payload bytes data[data_off[g] .. +data_len[g]) = the bincode-serialised request
 * batch RSCodeword::from_data produces (rscoding.rs:223-243).  Geometry is the reference's
 * (rscoding.rs:177-199): L_g = ceil(data_len/d); data shard i = payload bytes [i*L, (i+1)*L),
 * zero-padded past data_len; a contiguous split, so data shards are VIEWS of the payload.
 * Parity shard j of codeword g is written to parity[j*plane_stride + par_off[g] .. +L_g).
 * One launch = RSCodeword::from_data's split + compute_parity (rspaxos/request.rs:72-77,
 * crossword/request.rs:82-87) for n codewords; plane j is at the same time the packed
 * per-destination send buffer subset_copy builds one codeword at a time (rscoding.rs:255-293,
 * rspaxos/request.rs:127-142).  data_len[g] == 0 (null codeword) is skipped.
 *
 * flags:
 *   SS_RS_OUT_PADDED16  every parity slot starts 16-byte aligned and has capacity
 *                       round_up(L_g,16); bytes [L_g, round_up) are written as zeros.  This is
 *                       the fast path (128-bit stores).  Without it stores are byte-exact.
 *                       16-byte alignment is what correctness needs; where the layout is yours to choose,
 *                       prefer 32-byte multiples for par_off / shard_stride: write-heavy kernels lose ~7 %
 *                       when rows start in the middle of a DRAM sector (see SS_CW_SLOT_PITCH).
 *   SS_RS_EMIT_DATA     `parity` is plane d of a (d+p)-plane shard store with the same plane_stride:
 *                       the kernel ALSO copies data shard i into plane i (parity - (d-i)*plane_stride),
 *                       so all d+p planes are packed per-destination send buffers after one pass.
 * The payload arena must be a CUDA allocation (the kernel issues aligned 16-byte loads that may
 * cover up to 15 bytes either side of a payload, inside the allocation's 256-byte granule). */
#define SS_RS_OUT_PADDED16 1u
#define SS_RS_EMIT_DATA 2u
int ss_rs_encode_batch_dev(ss_rs_coder *coder, const uint8_t *data, const uint64_t *data_off,
                           const uint32_t *data_len, uint64_t n, uint8_t *parity,
                           uint64_t plane_stride, const uint64_t *par_off, uint32_t flags);
/* uniform geometry: data_off[g] = g*data_stride, data_len[g] = data_len, par_off[g] = g*shard_stride */
int ss_rs_encode_uniform_dev(ss_rs_coder *coder, const uint8_t *data, uint64_t data_stride,
                             uint32_t data_len, uint64_t n, uint8_t *parity,
                             uint64_t plane_stride, uint64_t shard_stride, uint32_t flags);

/* Batched reconstruct (rscoding.rs:490-537 over n codewords; callers rspaxos/durability.rs:146-159,
 * crossword/durability.rs:163-179).  Shard j of codeword g lives at
 * shards[j*plane_stride + off[g] .. +L_g), L_g = ceil(data_len[g]/d).  present[g] bit j =
 * shard j available; bits d+p and above are ignored.  Missing DATA shards are regenerated in place (and missing parity too when
 * data_only == 0).  status[g] = 0, SS_ERR_TOO_FEW_SHARDS_PRESENT (nothing written for g), or
 * SS_ERR_INVALID_ARG for a null codeword (data_len == 0; rscoding.rs:495-497). */
int ss_rs_reconstruct_batch_dev(ss_rs_coder *coder, uint8_t *shards, uint64_t plane_stride,
                                const uint64_t *off, const uint32_t *data_len,
                                const uint32_t *present, uint64_t n, int data_only,
                                int32_t *status, uint32_t flags);

/* uniform geometry: every codeword has data_len bytes and its shard j sits at shards + j*plane_stride + g*shard_stride
 * (16-byte aligned slots of capacity round_up(L,16), the layout ss_rs_encode_uniform_dev writes with
 * SS_RS_OUT_PADDED16; regenerated shards get zero padding).  For RS(3,2) -- every 5-replica deployment -- this runs
 * the pattern-specialised row kernel (compile-time decode rows per present mask); other codes go through the kernels of
 * the ragged call.  present[g] and status as above (present bits d+p and above are ignored). */
int ss_rs_reconstruct_uniform_dev(ss_rs_coder *coder, uint8_t *shards, uint64_t plane_stride, uint64_t shard_stride,
                                  uint32_t data_len, const uint32_t *present, uint64_t n, int data_only,
                                  int32_t *status);

/* host-buffer forms of the two batch calls (H2D, kernel, D2H inside; chunked + overlapped) */
int ss_rs_encode_uniform(ss_rs_coder *coder, const uint8_t *data, uint64_t data_stride,
                         uint32_t data_len, uint64_t n, uint8_t *parity, uint64_t plane_stride,
                         uint64_t shard_stride);

/* ---- quorum tallies ------------------------------------------------------------------------
 * Bit-plane form.  planes[r*G + g] bit s = a VALID AcceptReply from replica r for slot s of
 * group g (the leader's own WAL ack is one of the planes, multipaxos/durability.rs:99-103).
 * committed[g] bit s = (count of set planes >= threshold) -- the end state of
 * handle_msg_accept_reply on that ack set (multipaxos/messages.rs:404-413 with
 * threshold = quorum_cnt; rspaxos/messages.rs:438-440 with majority + fault_tolerance).
 * commit_bar[g] (may be NULL) = length of the committed prefix of the 64-slot window
 * (multipaxos/durability.rs:161-170).  R <= 16. */
int ss_tally_planes_dev(ss_ctx *ctx, const uint64_t *planes, uint32_t n_replicas, uint64_t n_groups,
                        uint32_t threshold, uint64_t *committed, uint32_t *commit_bar);
int ss_tally_planes(ss_ctx *ctx, const uint64_t *planes, uint32_t n_replicas, uint64_t n_groups,
                    uint32_t threshold, uint64_t *committed, uint32_t *commit_bar);

/* Per-instance vote-mask form: masks[i] = the instance's accept_acks Bitmap (bit r = replica r,
 * src/utils/bitmap.rs:17; LeaderBookkeeping.accept_acks, multipaxos/mod.rs:181-197), one
 * mask_bytes-wide (1 or 2) little-endian integer per instance.  commit_bits word i/64 bit i%64 =
 * Bitmap::count() >= threshold (bitmap.rs:111-113). */
int ss_tally_masks_dev(ss_ctx *ctx, const void *masks, uint32_t mask_bytes, uint64_t n_instances,
                       uint32_t threshold, uint64_t *commit_bits);

/* Ack ingest: applies the filters of handle_msg_accept_reply to a record stream and ORs the
 * surviving acks into the planes (multipaxos/messages.rs:388 ballot == bal_prepared;
 * :394-399 status == Accepting && ballot >= inst.bal; :404-406 duplicates are idempotent).
 * accepting[g] bit s = instance (g,s) is in Status::Accepting; inst_bal[g*64+s] its ballot.
 * Records with peer >= n_replicas or slot >= 64 are dropped (Bitmap::get -> Err, bitmap.rs:89-97). */
int ss_ack_ingest_dev(ss_ctx *ctx, const uint32_t *rec_group, const uint8_t *rec_slot,
                      const uint8_t *rec_peer, const uint64_t *rec_ballot, uint64_t n_records,
                      const uint64_t *bal_prepared, const uint64_t *inst_bal,
                      const uint64_t *accepting, uint32_t n_replicas, uint64_t n_groups,
                      uint64_t *planes);

/* Crossword commit predicate (crossword/messages.rs:15-62 coverage_under_faults, :535-542).
 * policies[k*n_replicas + r] = shard bitmask (over T = total_shards ids) replica r holds under
 * assignment policy k (Instance.assignment, crossword/mod.rs:260; balanced round-robin policies
 * crossword/mod.rs:866-888, or the single init_assignment when unbalanced, adaptive.rs:129-131).
 * policy_idx[i] selects instance i's policy; masks[i] = which replicas acked.
 * balanced != 0 uses the reference's closed form (:28-33), else the subset enumeration (:35-61).
 * commit iff #acks >= majority && coverage >= data_shards.  n_replicas <= 12, n_policies <= 16.
 * An instance with policy_idx[i] >= n_policies never commits. */
int ss_tally_crossword_dev(ss_ctx *ctx, const void *masks, uint32_t mask_bytes,
                           const uint8_t *policy_idx, uint64_t n_instances,
                           const uint32_t *policies_host, uint32_t n_policies, uint32_t n_replicas,
                           uint32_t total_shards, uint32_t data_shards, uint32_t majority,
                           uint32_t fault_tolerance, int balanced, uint64_t *commit_bits);

/* Raft / CRaft match-index commit scan (raft/messages.rs:256-275; craft/messages.rs:288-314).
 * match[p*G + g] for the n_peers = population-1 peers (self excluded, raft/mod.rs:560-562);
 * entries last_commit+1 .. log_end-1 of group g have terms terms[g*window + (slot-last_commit-1)]
 * (log_end - last_commit - 1 <= window).  new_commit[g] = the LAST slot in that range with
 * term == curr_term and 1 + #{p: match[p] >= slot} >= threshold, else last_commit[g].
 * threshold = quorum_cnt (Raft), majority+f or majority (CRaft full-copy).
 * window_overflow (device u32, may be NULL): incremented once per group whose candidate range exceeds `window`
 * entries (precondition violated); for such a group new_commit is a lower bound of the reference's result (candidates
 * beyond the window cannot be examined) and the host should rescan it with a larger window. */
int ss_raft_commit_scan_dev(ss_ctx *ctx, const uint32_t *match, uint32_t n_peers, uint64_t n_groups,
                            const uint32_t *last_commit, const uint32_t *log_end,
                            const uint32_t *curr_term, const uint32_t *terms, uint32_t window,
                            uint32_t threshold, uint32_t *new_commit, uint32_t *window_overflow);

/* k-th largest peer match per group.  k = threshold - 1 gives CRaft's shadow_last_commit
 * (craft/messages.rs:677-690: match slots sorted descending, element [threshold-2], threshold =
 * majority + fault_tolerance, or majority in full-copy mode); k = n_peers gives the bound of Raft's
 * last_snap scan (raft/messages.rs:298-309: every server has the entry). */
int ss_raft_kth_match_dev(ss_ctx *ctx, const uint32_t *match, uint32_t n_peers, uint64_t n_groups, uint32_t k,
                          uint32_t *out);

/* Prepare-phase shard merge + decision for n_instances recovering instances (leader fail-over;
 * rspaxos/messages.rs:182-259, crossword/messages.rs:233-312).  vote_bal[r*N+i] / vote_mask[r*N+i] = the
 * (ballot, shards carried) of replica r's PrepareReply vote for instance i; vote_bal == 0 means "no vote", as the
 * reply's `voted = if inst.voted.0 > 0 { Some(..) } else { None }` (rspaxos/durability.rs, crossword/durability.rs).
 * A vote with vote_bal > 0 and vote_mask == 0 is Some((bal, no shards)) -- a Crossword replica whose assignment row is
 * empty still records its ballot when it accepts -- and, at a ballot above the others, discards the shards gathered
 * at lower ballots.  merged[i] = shard set inst.reqs_cw ends with (shards voted at the highest ballot; max_bal[i] that
 * ballot; order-independent because absorb_other only adds).  action[i]: bit0 USE (>= data_shards shards), bit1 NULL
 * request batch (fewer, but acks_cnt[i] >= population - fault_tolerance), 0 = not yet; bit2 reconstruct_data
 * needed; bit3 compute_parity needed (avail shards < POPULATION, as the reference compares).  The regeneration
 * itself is ss_rs_reconstruct_batch_dev(present = merged, data_only = 0). */
#define SS_PM_USE 1u
#define SS_PM_NULL 2u
#define SS_PM_RECONSTRUCT 4u
#define SS_PM_PARITY 8u
int ss_prepare_merge_dev(ss_ctx *ctx, const uint64_t *vote_bal, const uint32_t *vote_mask, uint32_t n_replicas,
                         uint64_t n_instances, const uint8_t *acks_cnt, uint32_t data_shards, uint32_t population,
                         uint32_t fault_tolerance, uint64_t *max_bal, uint32_t *merged, uint8_t *action);

/* ---- fused accept step (BASELINE config 3: RSPaxos encode + quorum) -------------------------
 * ONE kernel launch that, for n_groups groups: RS-encodes each group's new request batch
 * (as ss_rs_encode_uniform_dev) and tallies the group's 64-slot ack window
 * (as ss_tally_planes_dev). */
int ss_accept_step_fused_dev(ss_rs_coder *coder, const uint8_t *data, uint64_t data_stride,
                             uint32_t data_len, uint64_t n_groups, uint8_t *parity,
                             uint64_t plane_stride, uint64_t shard_stride, uint32_t flags,
                             const uint64_t *planes, uint32_t n_replicas, uint32_t threshold,
                             uint64_t *committed, uint32_t *commit_bar);

/* ---- step flags: cross-GPU ordering without host synchronisation ---------------------------------------------
 * A flag is a u64 step counter in device memory (ss_dev_alloc + ss_dev_memset 0; exported to peers with
 * ss_ipc_export).  Calls that take an ss_step_sync
 *   - first wait (on the device, inside the kernel) until every wait_flags[i] >= wait_value -- wait_flags is a device
 *     array in LOCAL memory that peers write into;
 *   - after all of the call's stores are visible system-wide, store signal_value to every *signal_flags[i]
 *     (st.release.sys) -- signal_flags is a HOST array of device pointers into local or peer memory.
 * This replaces the per-step stream barrier + ack copies a host would otherwise need: a follower's kernel starts when
 * the leader's shards have landed, the leader's next tally starts when the followers' acks have landed
 * (rspaxos/request.rs:127-142 -> rspaxos/durability.rs:101-118 -> rspaxos/messages.rs:395-465, with NVLink stores in
 * place of TransportHub messages).  Waits are bounded (2 s): on time-out bit 0 of ss_ctx_device_status is set and the
 * kernel proceeds.  n_wait, n_signal <= 32; either part may be empty; a NULL ss_step_sync means no ordering. */
typedef struct ss_step_sync {
    const uint64_t *wait_flags;
    uint32_t n_wait;
    uint64_t wait_value;
    uint64_t *const *signal_flags;
    uint32_t n_signal;
    uint64_t signal_value;
} ss_step_sync;
/* the two halves of an ss_step_sync as stand-alone stream operations (one-warp kernels on the context's stream) */
int ss_flags_wait_dev(ss_ctx *ctx, const ss_step_sync *sync);
int ss_flags_signal_dev(ss_ctx *ctx, const ss_step_sync *sync);
/* Stream-ordering between TWO contexts of one process (e.g. a compute context and a copy context whose
 * ss_copy_d2d pushes run on the copy engines while the next step computes): an event recorded on one context's stream
 * can be waited for by another's (cudaEventRecord / cudaStreamWaitEvent). */
int ss_event_create(ss_ctx *ctx, void **event);
int ss_event_destroy(ss_ctx *ctx, void *event);
int ss_event_record(ss_ctx *ctx, void *event);
int ss_event_wait(ss_ctx *ctx, void *event);
/* reads (and clears) the context's device status word; synchronises the context's stream */
#define SS_DEV_STATUS_FLAG_TIMEOUT 1u
#define SS_DEV_STATUS_FRAME_OVERFLOW 4u   /* ss_frame_accept_pack_dev / _ragged_dev: a frame did not fit its room */
int ss_ctx_device_status(ss_ctx *ctx, uint32_t *status);

/* Fused encode + tally + REPLICATE (the multi-GPU accept step): as ss_accept_step_fused_dev, but shard j of the
 * local groups (data shards included) is written to shard_planes[j] + g*shard_stride, where each shard_planes[j]
 * is a device pointer into LOCAL memory or into a PEER GPU's memory (ss_ipc_open): the encode kernel itself
 * delivers every replica's shard over NVLink -- no pack pass, no separate collective.  shard_planes is a HOST
 * array of d+p pointers; every target slot is 16-byte aligned with capacity round_up(L,16).  Any code with d <= 8
 * data shards (every Summerset cluster code; others are specialised at run time), 16-byte-aligned uniform payloads of
 * any length (SS_ERR_UNSUPPORTED otherwise).  sync (may be NULL): the tally waits for
 * sync->wait_flags (the followers' ack flags) and the followers are signalled when every shard has landed. */
int ss_accept_step_replicate_dev(ss_rs_coder *coder, const uint8_t *data, uint64_t data_stride, uint32_t data_len,
                                 uint64_t n_groups, uint8_t *const *shard_planes, uint64_t shard_stride,
                                 const uint64_t *planes, uint32_t n_replicas, uint32_t threshold,
                                 uint64_t *committed, uint32_t *commit_bar, const ss_step_sync *sync);

/* Host-buffer form of the fused accept step (the call a host without device-resident state makes): payloads, ack
 * planes, parity planes, commit words and commit_bar are HOST arrays with the layouts of ss_accept_step_fused_dev;
 * chunks of groups are uploaded, run through the ONE fused kernel and downloaded with copy and compute overlapped
 * (three staging buffers on separate copy streams).  Returns when every result is in host memory.  Pinned host
 * buffers (ss_host_alloc) are needed for the overlap. */
int ss_accept_step_fused(ss_rs_coder *coder, const uint8_t *data, uint64_t data_stride, uint32_t data_len,
                         uint64_t n_groups, uint8_t *parity, uint64_t plane_stride, uint64_t shard_stride,
                         const uint64_t *planes, uint32_t n_replicas, uint32_t threshold, uint64_t *committed,
                         uint32_t *commit_bar);

/* The simulated followers' side of the step (rspaxos/durability.rs:101-118: log the Accept, reply): once the leaders'
 * shards have landed (sync->wait_flags), ack plane r -- ack_src[r*n_groups .. +n_groups), this GPU's followers' ack
 * bits for the groups they follow -- is stored to ack_dst[r] (n_groups words in the leader GPU's memory, local or
 * peer; a NULL entry is skipped), then the leaders are signalled.  ack_dst is a HOST array of n_replicas pointers. */
int ss_follower_ack_dev(ss_ctx *ctx, const uint64_t *ack_src, uint64_t *const *ack_dst, uint32_t n_replicas,
                        uint64_t n_groups, const ss_step_sync *sync);

/* Crossword encode + distribute (BASELINE config 4; crossword/request.rs:82-87,137-185): RS-encodes a ragged batch with
 * the coder's (d, T-d) code and writes, for every codeword g, the spr[g] shards the balanced round-robin assignment gives
 * replica r -- shards {(r*dj + k) mod T : k < spr[g]}, dj = T / n_replicas (crossword/mod.rs:866-888) -- into
 * replica_logs[r] at rep_off[g] + k*SS_CW_SLOT_PITCH(L_g), k = 0..spr-1 (bytes past L_g zero; the pitch is L_g rounded up
 * to 32 bytes so that every slot of a log built from 32-byte aligned offsets starts on a DRAM sector, which a 16-byte
 * pitch does not give).  replica_logs is a HOST array
 * of n_replicas device pointers, local or peer (ss_ipc_open): the kernel's stores are the shard transfer.  Per codeword
 * (n-1)*spr*L_g bytes cross to other replicas, as in the reference.  Any code with d <= 8 and T a multiple of
 * n_replicas <= 16 (crossword/mod.rs:805-830); n = 5 with RS(3,2) runs the hand-specialised kernel. */
#define SS_CW_SLOT_PITCH(L) ((((uint64_t)(L)) + 31u) & ~(uint64_t)31u)
int ss_crossword_distribute_dev(ss_rs_coder *coder, const uint8_t *data, const uint64_t *data_off,
                                const uint32_t *data_len, const uint8_t *spr, const uint64_t *rep_off,
                                uint64_t n, uint8_t *const *replica_logs, uint32_t n_replicas);

/* Accept-frame packer (the step after the path, SURVEY 8f-2): for n uniform codewords, builds the byte frames an
 * unmodified Summerset peer reads off its TCP connection -- 8-byte big-endian body length (utils/safetcp.rs:30-88)
 * + bincode(PeerMessage::Msg { msg: PeerMsg::Accept { slot, ballot, reqs_cw } }) (server/transport.rs:37-40,
 * rspaxos/mod.rs:283-288) where reqs_cw = the codeword holding only shard `shard_idx` (what subset_copy builds for
 * that peer, rspaxos/request.rs:127-142), encoded per utils/rscoding.rs:54-71 with data_copy = None.
 * shard_plane: shard `shard_idx` of codeword g at shard_plane + g*shard_stride.  Frame g is written inside
 * out[g*frame_stride .. (g+1)*frame_stride) at frame_off[g] (so that the shard bytes are 16-byte aligned) and is
 * frame_len[g] bytes long.  frame_stride: multiple of 16, >= shard_len + 96 + d + p.  msg_variant = the index of
 * the Accept variant in the protocol's PeerMsg enum (2 for RSPaxos).  This is the single-shard fast path (the shard
 * is copied with aligned 128-bit accesses on both sides); ss_frame_accept_pack_dev is the general packer.  bincode
 * layout from knowledge of the crate: unpinned against the reference (it cannot run here); tested byte for byte against
 * the oracle's independent C encoder (oracle/ss_wire.c). */
int ss_frame_accept_batch_dev(ss_ctx *ctx, const uint8_t *shard_plane, uint64_t shard_stride, uint32_t shard_idx,
                              uint32_t data_shards, uint32_t parity_shards, uint32_t data_len, uint32_t msg_variant,
                              const uint64_t *slot, const uint64_t *ballot, uint64_t n, uint8_t *out,
                              uint64_t frame_stride, uint64_t *frame_off, uint32_t *frame_len);

/* ---- wire / WAL formats on the device (SURVEY 8f-2) -------------------------------------------------------------
 * General Accept packer: for n codewords and ONE destination, builds either the frames an unmodified Summerset peer
 * reads off its TCP connection -- 8-byte big-endian body length (utils/safetcp.rs:30-88) + bincode(PeerMessage::Msg {
 * msg: PeerMsg::Accept { slot, ballot, reqs_cw [, assignment] } }) (server/transport.rs:37-40, rspaxos/mod.rs:283-288,
 * crossword/mod.rs:356-362) -- or the records StorageHub appends -- 8-byte big-endian length (server/storage.rs:333-337)
 * + bincode(WalEntry::AcceptData { slot, ballot, reqs_cw }) (rspaxos/mod.rs:219-228).  reqs_cw carries exactly the shards
 * policies[policy_idx[g]][peer] names (what subset_copy(.., false) builds for that peer: one shard in RSPaxos,
 * rspaxos/request.rs:127-142; spr shards in Crossword, crossword/request.rs:164-185), data_copy None, encoded per
 * utils/rscoding.rs:43-72; with_assignment appends assignment: Vec<Bitmap> = that policy row (utils/bitmap.rs:20-30).
 * policies: DEVICE array [n_policies][population] of shard bitmasks; policy_idx: device [n] or NULL (policy 0); an
 * index >= n_policies also selects policy 0 (here and in ss_frame_accept_pack_ragged_dev).
 * Frame g is written inside out[g*frame_stride ..) at frame_off[g] (placed so that its first shard's bytes are 16-byte
 * aligned) and is frame_len[g] bytes long; frame_stride >= ss_frame_accept_max_len(spec, max shards per frame) -- a
 * frame that would not fit its slot is not written: frame_len[g] = 0 and bit 2 of ss_ctx_device_status is set.
 * bincode layout from knowledge of the crate: unpinned against the reference; tested byte for byte against the oracle's
 * independent C encoder (oracle/ss_wire.c), and decode(encode(x)) == x. */
#define SS_FRAME_PEER_ACCEPT 0u
#define SS_FRAME_WAL_ACCEPT_DATA 1u
typedef struct ss_frame_spec {
    uint32_t kind;             /* SS_FRAME_PEER_ACCEPT / SS_FRAME_WAL_ACCEPT_DATA */
    uint32_t msg_variant;      /* index of Accept in the protocol's PeerMsg enum (2), or of AcceptData in WalEntry (1) */
    uint32_t data_shards, parity_shards, data_len;
    uint32_t population;       /* replicas (columns of the policy table) */
    uint32_t with_assignment;  /* Crossword Accept: append assignment: Vec<Bitmap> */
    uint32_t assign_size;      /* bit length of each assignment Bitmap (= rs_total_shards) */
} ss_frame_spec;
uint64_t ss_frame_accept_max_len(const ss_frame_spec *spec, uint32_t max_shards_per_frame);
int ss_frame_accept_pack_dev(ss_ctx *ctx, const ss_frame_spec *spec, const uint8_t *shard_planes, uint64_t plane_stride,
                             uint64_t shard_stride, const uint32_t *policies, uint32_t n_policies,
                             const uint8_t *policy_idx, uint32_t peer, const uint64_t *slot, const uint64_t *ballot,
                             uint64_t n, uint8_t *out, uint64_t frame_stride, uint64_t *frame_off, uint32_t *frame_len);
/* The same frames / records for RAGGED codewords (spec->data_len is ignored): frame g is what the packer above writes
 * for a codeword of data_len[g] bytes whose shard j sits at shard_planes + j*plane_stride + shard_off[g] -- the store
 * ss_engine_propose_ragged fills -- and its RSCodeword header carries that data_len and shard_len = ceil(data_len/d)
 * (rscoding.rs:43-72,177-199).  No frame is written for data_len[g] == 0 or slot[g] == UINT64_MAX (frame_len 0), so
 * that call's slot_out / shard_off feed this one directly.  Packed output: frame g's region is round_up(pad + len, 16)
 * bytes (pad: the 16-byte alignment of its first carried shard, as above); the regions follow each other in group
 * order from out (16-byte aligned), frame_off[g] = the frame's start, *total (device u64, may be NULL) = the bytes the
 * whole batch needs.  A frame whose region ends past out_capacity is not written: frame_len 0 and
 * SS_DEV_STATUS_FRAME_OVERFLOW. */
int ss_frame_accept_pack_ragged_dev(ss_ctx *ctx, const ss_frame_spec *spec, const uint8_t *shard_planes, uint64_t plane_stride,
                                    const uint64_t *shard_off, const uint32_t *data_len, const uint32_t *policies,
                                    uint32_t n_policies, const uint8_t *policy_idx, uint32_t peer, const uint64_t *slot,
                                    const uint64_t *ballot, uint64_t n, uint8_t *out, uint64_t out_capacity,
                                    uint64_t *frame_off, uint32_t *frame_len, uint64_t *total);

/* AcceptReply frames -> ack records.  buf holds frames as read off the peers' connections (8-byte big-endian length +
 * body each); frame i starts at frame_off[i], came from replica frame_peer[i] of group frame_group[i].  A well-formed
 * PeerMessage::Msg{PeerMsg::AcceptReply{slot, ballot}} (rspaxos/mod.rs:290-291; with_size: crossword's
 * {slot, ballot, size, reply_ts}, crossword/mod.rs:365-373) yields rec_kind[i] = reply_variant and the record
 * (group, slot - window_base[group], peer, ballot) in the layout ss_ack_ingest_dev / ss_engine_ingest take; slots below
 * the group's window base (`slot < start_slot`, messages.rs:377) or beyond the 64-slot window get rec_slot = 0xff, which
 * the ingest kernel drops.  Other messages: rec_kind = their PeerMsg variant index (0x80000000 | k for the
 * PeerMessage variants LeaseMsg / Leave / LeaveReply) -- the host handles them; malformed: SS_FRAME_KIND_MALFORMED. */
#define SS_FRAME_KIND_MALFORMED 0xffffffffu
int ss_accept_reply_parse_dev(ss_ctx *ctx, const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off,
                              const uint32_t *frame_group, const uint8_t *frame_peer, const uint64_t *window_base,
                              uint64_t n_frames, uint64_t n_groups, uint32_t reply_variant, int with_size,
                              uint32_t *rec_group, uint8_t *rec_slot, uint8_t *rec_peer, uint64_t *rec_ballot,
                              uint32_t *rec_kind);

/* WalEntry::CommitSlot { slot } records (rspaxos/mod.rs:231; commit_variant = 2) for every instance that committed in a
 * tick: newly[g] bit s (ss_engine_tick's output) -> one 24-byte cell in `entries` holding the 8-byte big-endian length
 * + bincode record of absolute slot window_base[g] + s, with entry_group / entry_len beside it.  *n_entries (device u64)
 * = number of records; cells beyond `capacity` are counted but not written.  Cell order is unspecified (every group
 * has its own WAL; the host routes by entry_group). */
int ss_wal_commit_pack_dev(ss_ctx *ctx, const uint64_t *newly, const uint64_t *window_base, uint64_t n_groups,
                           uint32_t commit_variant, uint8_t *entries, uint32_t *entry_group, uint32_t *entry_len,
                           uint64_t capacity, uint64_t *n_entries);

/* Reconstruct serving (SURVEY 8f-4; crossword/messages.rs:577-632, rspaxos/messages.rs:468-517) for n_requests
 * (slot, exclude) pairs of a Reconstruct message: request i concerns the instance of group req_group[i] whose shards sit
 * in shard_planes (shard j at shard_planes + j*plane_stride + req_group[i]*shard_stride), of which this replica holds
 * req_held[i]; req_status[i] is the instance's Status (>= 2 = Accepting).  reply_mask[i] = held & flip(exclude) -- 0 when
 * the status is below Accepting or nothing is left, in which case the slot gets no entry in the reply -- and the
 * selected shards are copied in index order, each in a round_up(shard_len,16)-byte slot, to out + reply_off[i]
 * (16-byte aligned offsets). */
int ss_reconstruct_serve_dev(ss_ctx *ctx, const uint8_t *shard_planes, uint64_t plane_stride, uint64_t shard_stride,
                             uint32_t total_shards, uint32_t shard_len, const uint32_t *req_group,
                             const uint32_t *req_held, const uint32_t *req_excl, const uint8_t *req_status,
                             const uint64_t *reply_off, uint64_t n_requests, uint32_t *reply_mask, uint8_t *out);

/* Crossword follower gossip planning (SURVEY 8f-4; crossword/gossiping.rs:35-84 gossip_targets_excl) for
 * n_instances committed-but-incomplete instances of replica `me`: walking peers me+1, me+2, ... (mod population) and
 * skipping the instance's source peer (src_peer[i]) and peers absent from `peer_alive`, a peer is selected when its
 * assigned shards (policies[policy_idx[i]][peer]; an index >= n_policies selects policy 0) include one not yet held/asked for;
 * excl[peer*N + i] = the availability map at that moment (what the Reconstruct message tells the peer to leave out,
 * crossword/messages.rs:577-632); the walk stops once data_shards shards are covered.  targets[i] = selected peers.
 * excl entries of unselected peers are left untouched. */
int ss_gossip_plan_dev(ss_ctx *ctx, uint32_t me, uint32_t population, uint32_t data_shards, const uint8_t *src_peer,
                       const uint32_t *avail, const uint8_t *policy_idx, const uint32_t *policies_host,
                       uint32_t n_policies, uint32_t peer_alive, uint64_t n_instances, uint32_t *targets, uint32_t *excl);

/* ---- batched multi-group consensus engine ----------------------------------------------------------------------
 * The leader-side state of n_groups independent replica groups lives in HBM as a struct of arrays; the host drives all
 * groups together, once per event-loop turn.  Paxos-family group g holds the 64 absolute slots [window_base[g],
 * window_base[g] + 64) (window_base = the reference's start_slot, 0 at creation); every per-slot array is a RING:
 * absolute slot s lives at position s & 63.
 *   ss_engine_propose   one new instance per group at window position `slot` (absolute slot window_base + slot), or
 *   ss_engine_propose_next  at each group's first Null slot: RS-encode the request batches into the shard planes
 *                       (per-peer packed send buffers) and enter Status::Accepting under the group's
 *                       prepared ballot with an empty ack set   (multipaxos/request.rs:112-221,
 *                       rspaxos/request.rs:72-142, crossword/request.rs:82-185)
 *   ss_engine_ingest    a batch of AcceptReply records through handle_msg_accept_reply's filters
 *                       (multipaxos/messages.rs:377-409, rspaxos/messages.rs:402-437, crossword/messages.rs:489-530)
 *   ss_engine_tick      ONE kernel: commit decision of every Accepting instance (MultiPaxos quorum_cnt,
 *                       multipaxos/messages.rs:412-413; RSPaxos majority + fault_tolerance, rspaxos/messages.rs:438-440;
 *                       Crossword #acks >= majority && coverage_under_faults >= d, crossword/messages.rs:535-542),
 *                       committed |= newly, accepting &= ~newly, commit_bar = committed prefix
 *                       (multipaxos/durability.rs:161-170)
 *   ss_engine_advance   retire committed prefixes: window_base moves forward (multipaxos/snapshot.rs:121-171)
 * Raft / CRaft engines keep match_slot / next_slot / log terms instead: ss_engine_raft_append (the leader appends
 * entries in its term), ss_engine_raft_ingest (successful AppendEntriesReply, raft/messages.rs:243-252) and
 * ss_engine_tick (commit scan raft/messages.rs:254-275,295 with quorum_cnt -- CRaft: majority + fault_tolerance,
 * craft/messages.rs:300-308 -- and last_snap, raft/messages.rs:298-309).  Conflict replies, elections, heartbeats,
 * durability and execution stay in the host's event loop (out of scope, SURVEY.md 2b).
 * All array arguments are DEVICE pointers; calls are asynchronous on the context's stream. */
typedef struct ss_engine ss_engine;
#define SS_PROTO_MULTIPAXOS 0u
#define SS_PROTO_RSPAXOS 1u
#define SS_PROTO_CROSSWORD 2u
#define SS_PROTO_RAFT 3u
#define SS_PROTO_CRAFT 4u
typedef struct ss_engine_config {
    uint32_t protocol;          /* SS_PROTO_* */
    uint32_t population;        /* n <= 12 */
    uint32_t fault_tolerance;   /* f <= n - majority (rspaxos/mod.rs:599-605); ignored by MultiPaxos / Raft */
    uint32_t data_len;          /* bytes of every request batch (RS-coded protocols) */
    uint32_t rs_total_shards;   /* Crossword: T (0 = n; must be a multiple of n, crossword/mod.rs:805-830) */
    uint32_t rs_data_shards;    /* Crossword: d (0 = majority) */
    uint32_t keep_slots;        /* depth of the shard store: proposals of slot s live in store s % keep_slots (0 = 1) */
    uint32_t raft_window;       /* Raft: uncommitted-tail capacity per group, power of two (0 = 64) */
} ss_engine_config;
/* device pointers into the engine's state (valid until ss_engine_destroy), for hosts that read results in place or
 * install state (recovery, tests).  Arrays a protocol does not use are NULL. */
typedef struct ss_engine_view {
    uint64_t n_groups;
    uint32_t population, threshold, data_shards, total_shards, shard_len, shard_stride, raft_window, pad0;
    uint64_t plane_stride;      /* bytes between shard planes of one proposal */
    uint64_t slot_stride;       /* bytes between the shard stores of consecutive keep slots */
    /* per-slot words and arrays are ring-indexed: absolute slot s at bit / entry s & 63 (ss_engine_window_get) */
    uint64_t *planes;           /* [n][G]  valid-ack bit-planes */
    uint64_t *bal_prepared;     /* [G] */
    uint64_t *inst_bal;         /* [G*64] */
    uint64_t *accepting;        /* [G]  bit s & 63 = Status::Accepting */
    uint64_t *committed;        /* [G]  bit s & 63 = Status::Committed */
    uint32_t *commit_bar;       /* [G]  window-relative: the absolute commit bar is window_base + commit_bar */
    uint8_t *shards;            /* [keep][T][G][shard_stride] */
    uint8_t *policy_idx;        /* Crossword [G*64]: assignment policy of each instance */
    uint32_t *match, *next_slot;/* Raft [n-1][G] */
    uint32_t *last_commit, *log_end, *curr_term, *last_snap;   /* Raft [G] */
    uint32_t *terms;            /* Raft [G][raft_window]: term of slot s at index s & (raft_window-1) */
} ss_engine_view;
int ss_engine_create(ss_ctx *ctx, const ss_engine_config *cfg, uint64_t n_groups, ss_engine **out);
int ss_engine_destroy(ss_engine *engine);
int ss_engine_view_get(ss_engine *engine, ss_engine_view *view);
/* bal_prepared of every group (become_a_leader ... handle_msg_prepare_reply, outside this path) */
int ss_engine_set_prepared_ballots(ss_engine *engine, const uint64_t *ballots);
/* Crossword: the assignment policies instances may use (policies_host[k*n + r] = shard bitmask of replica r, as
 * ss_tally_crossword_dev) and whether the balanced closed form applies (crossword/mod.rs:849-850) */
int ss_engine_set_policies(ss_engine *engine, const uint32_t *policies_host, uint32_t n_policies, int balanced);
/* payloads: request batch of group g at payloads + g*payload_stride (data_len bytes; NULL for MultiPaxos).  policy:
 * Crossword only, [G] policy index of the new instance (NULL = 0; an index >= n_policies is stored as given, and
 * ss_engine_tick never commits that instance).  *shard_planes (may be NULL) receives the base of
 * this proposal's T shard planes: shard j of group g at base + j*plane_stride + g*shard_stride.  `slot` (< 64) is
 * relative to each group's window base: the instance is absolute slot window_base[g] + slot, its shards go to shard
 * store slot % keep_slots. */
int ss_engine_propose(ss_engine *engine, uint32_t slot, const uint8_t *payloads, uint64_t payload_stride,
                      const uint8_t *policy, uint8_t **shard_planes);
/* group g proposes at its first Null slot of [window_base[g], window_base[g]+64) (rspaxos/mod.rs:434-442);
 * slot_out[g] (device u64, may be NULL) = that absolute slot, or UINT64_MAX when the window is full (then bit 3 of
 * ss_ctx_device_status is set and the group is left unchanged).  Shards of this proposal go to shard store `store`
 * (< keep_slots) -- caller-managed, so the encode stays the uniform row kernel at full speed; a full group's shards are
 * written there too but belong to no instance.  slot_out is exactly the `slot` array ss_frame_accept_pack_dev takes:
 * a host goes straight from the proposal to its Accept frames.  Other arguments as ss_engine_propose. */
#define SS_DEV_STATUS_WINDOW_FULL 8u
int ss_engine_propose_next(ss_engine *engine, uint32_t store, const uint8_t *payloads, uint64_t payload_stride,
                           const uint8_t *policy, uint64_t *slot_out, uint8_t **shard_planes);
/* Ragged proposals (RSPaxos / Crossword engines; others return SS_ERR_INVALID_ARG): group g's request batch is
 * arena[data_off[g] .. +data_len[g]), of any length, as ExternalApi::get_req_batch drains it (server/external.rs:323-345)
 * and handle_req_batch codes it (rspaxos/request.rs:72, crossword/request.rs:82; L_g = ceil(data_len[g]/d),
 * rscoding.rs:177-199).  data_len[g] == 0: the group has nothing to propose -- slot_out[g] = UINT64_MAX, no status bit,
 * the group is untouched.  A group with a batch proposes at its first Null slot as ss_engine_propose_next does (a full
 * window: slot_out UINT64_MAX, SS_DEV_STATUS_WINDOW_FULL, no room taken in the store).
 * Store: CALLER-owned, T planes at shards + j*plane_stride (plane_stride a multiple of 32, shards 16-byte aligned).
 * Every proposing group takes a slot of SS_CW_SLOT_PITCH(L_g) bytes in each plane; shard_off[g] (device [G]) = the
 * exclusive prefix sum of those pitches in group order, computed on the device (UINT64_MAX: the group did not propose);
 * *need (device u64, may be NULL) = the total pitch the batch asked for.  A group whose slot would end past plane_stride
 * is not proposed (slot_out UINT64_MAX, SS_DEV_STATUS_STORE_FULL, group unchanged); the offsets are monotone, so the
 * groups that fit are a prefix of the proposing groups.  After the call plane j holds shard j of every proposing group
 * at shard_off[g], zero-padded to round_up(L_g,16) (bytes from there to the pitch are not written) -- one launch of the
 * ragged encoder (ss_rs_encode_batch_dev, SS_RS_OUT_PADDED16 | SS_RS_EMIT_DATA).  slot_out and shard_off feed
 * ss_frame_accept_pack_ragged_dev directly.  policy: Crossword [G] policy index (NULL = 0).  No host synchronisation;
 * per-group scratch is allocated on the first call.  Uniform and ragged proposals may be mixed on one engine
 * (cfg.data_len sizes only the engine's own uniform store: a host that only proposes ragged batches passes 1). */
#define SS_DEV_STATUS_STORE_FULL 16u
int ss_engine_propose_ragged(ss_engine *engine, const uint8_t *arena, const uint64_t *data_off, const uint32_t *data_len,
                             const uint8_t *policy, uint8_t *shards, uint64_t plane_stride, uint64_t *shard_off,
                             uint64_t *slot_out, uint64_t *need);
/* rec_slot is window-relative, as ss_accept_reply_parse_dev emits it with this engine's window_base: 0xff and values
 * >= 64 are dropped, rel is absolute slot window_base[g] + rel. */
int ss_engine_ingest(ss_engine *engine, const uint32_t *rec_group, const uint8_t *rec_slot, const uint8_t *rec_peer,
                     const uint64_t *rec_ballot, uint64_t n_records);
/* newly (may be NULL): [G] bit i = instance window_base[g] + i committed in THIS tick (what the host logs as
 * WalEntry::CommitSlot: ss_wal_commit_pack_dev with this engine's window_base) */
int ss_engine_tick(ss_engine *engine, uint64_t *newly);
/* retires committed prefixes (multipaxos/snapshot.rs:121-171, start_slot advance): upto (device [G] absolute slots, or
 * NULL = the whole committed prefix) -- k = clamp(upto[g] - window_base[g], 0, committed prefix); the k retired ring
 * positions are cleared (committed, accepting, ack planes), window_base[g] += k and commit_bar[g] -= k. */
int ss_engine_advance(ss_engine *engine, const uint64_t *upto);
/* *window_base = the engine's device array [G] of window bases (valid until ss_engine_destroy); a host may install
 * bases through it, e.g. a snapshot's start_slot on recovery, while the window holds no instance.  Until the first
 * ss_engine_advance or ss_engine_window_get call every base is 0 and the tick does not read them.  Raft / CRaft
 * engines (which keep their own ring) return SS_ERR_INVALID_ARG from propose_next, advance and window_get. */
int ss_engine_window_get(ss_engine *engine, uint64_t **window_base);
/* Raft: n_new[g] entries appended by the leader in curr_term[g]; exceeding raft_window uncommitted entries sets bit 1
 * of ss_ctx_device_status and leaves that group unchanged */
#define SS_DEV_STATUS_RAFT_WINDOW_FULL 2u
int ss_engine_raft_append(ss_engine *engine, const uint32_t *n_new);
int ss_engine_raft_ingest(ss_engine *engine, const uint32_t *rec_group, const uint8_t *rec_peer,
                          const uint32_t *rec_end_slot, uint64_t n_records);

/* ---- batched acceptor (RSPaxos / Crossword follower side of the accept path) -----------------------------------
 * The follower half of SURVEY 3.2 step 4 for n_groups groups this replica follows: Accept frames in (rspaxos/messages.rs
 * handle_msg_accept, crossword/messages.rs:403-470), held shards into a caller-owned store, WalEntry::AcceptData records
 * and AcceptReply frames out (rspaxos/durability.rs:101-118, crossword/durability.rs:96-125).  Per-group state lives in
 * HBM as a struct of arrays; per-slot arrays are rings of 64 indexed like the engine's (absolute slot s at s & 63).
 * One stated difference from the reference: the instance log is the engine's 64-slot window [window_base,
 * window_base + 64), not a vector that grows without bound; a frame beyond it takes no part in the call and the host
 * re-submits it after ss_acceptor_advance. */
typedef struct ss_acceptor ss_acceptor;
typedef struct ss_acceptor_config {
    uint32_t protocol;          /* SS_PROTO_RSPAXOS or SS_PROTO_CROSSWORD */
    uint32_t population;        /* replicas, 1..32 */
    uint32_t me;                /* this replica's id (Crossword reply size: assignment[me]) */
    uint32_t data_shards, total_shards;   /* the code every Accept must carry: 1 <= d <= T <= 32 */
    uint32_t accept_variant;    /* index of Accept in PeerMsg (2) */
    uint32_t wal_variant;       /* index of AcceptData in WalEntry (1) */
    uint32_t reply_variant;     /* index of AcceptReply in PeerMsg (3) */
} ss_acceptor_config;
typedef struct ss_acceptor_view {
    uint64_t n_groups;
    uint32_t protocol, population, me, data_shards, total_shards, pad0;
    uint64_t *window_base;      /* [G] start_slot */
    uint64_t *bal_max_seen;     /* [G] */
    uint64_t *inst_bal;         /* [G*64] */
    uint64_t *accepting;        /* [G] bit s & 63 = Status::Accepting */
    uint64_t *shard_addr;       /* [G*64] device address of the instance's first held shard in the caller's store */
    uint32_t *held;             /* [G*64] shard mask the instance holds */
    uint32_t *data_len;         /* [G*64] */
    uint32_t *assignment;       /* Crossword [G*64]: the instance's assignment row of `me`; NULL for RSPaxos */
    uint8_t *source;            /* [G*64] peer the Accept came from (replica_bk.source) */
} ss_acceptor_view;
/* Configuration checks come first (SS_ERR_INVALID_ARG); a NULL ctx then gives SS_ERR_NO_DEVICE when the machine has no
 * usable device, SS_ERR_INVALID_ARG otherwise.  All state starts at zero. */
int ss_acceptor_create(ss_ctx *ctx, const ss_acceptor_config *cfg, uint64_t n_groups, ss_acceptor **out);
int ss_acceptor_destroy(ss_acceptor *acceptor);
int ss_acceptor_view_get(ss_acceptor *acceptor, ss_acceptor_view *view);
/* *window_base = the acceptor's device array [G] of window bases; a host may install bases (a snapshot's start_slot)
 * while the window holds no instance. */
int ss_acceptor_window_get(ss_acceptor *acceptor, uint64_t **window_base);
/* retires window prefixes: upto (device [G] absolute slots, required -- the host decides what is retired):
 * k = clamp(upto[g] - window_base[g], 0, 64); the k retired ring positions leave Accepting and Committed and
 * window_base[g] += k. */
int ss_acceptor_advance(ss_acceptor *acceptor, const uint64_t *upto);
/* Verdicts of ss_acceptor_accept, beside the PeerMsg variant index k (another message; 0x80000000 | k for the
 * PeerMessage variants) and SS_FRAME_KIND_MALFORMED */
#define SS_ACCEPT_VERDICT_ACCEPTED 0xfffffff0u
#define SS_ACCEPT_VERDICT_STALE_SLOT 0xfffffff1u      /* slot < window_base: ignored (messages.rs `slot < start_slot`) */
#define SS_ACCEPT_VERDICT_STALE_BALLOT 0xfffffff2u    /* ballot < bal_max_seen as it stands when the frame is reached */
#define SS_ACCEPT_VERDICT_BEYOND_WINDOW 0xfffffff3u   /* slot >= window_base + 64: re-submit after ss_acceptor_advance */
#define SS_ACCEPT_VERDICT_STORE_FULL 0xfffffff4u      /* its store region ends past store_capacity */
#define SS_ACCEPT_VERDICT_WAL_FULL 0xfffffff5u        /* its WAL region ends past wal_capacity */
/* One batch of frames (device pointers; asynchronous on the context's stream, no host synchronisation).
 * buf holds frames as read off the leaders' connections at any byte alignment; frame i starts at frame_off[i] and came
 * from replica frame_peer[i] for group frame_group[i] (a group >= n_groups: malformed).  verdict[i] is one of the above.
 * Malformed: truncated or not decodable as a PeerMessage::Msg{Accept{slot, ballot, reqs_cw[, assignment]}}; a codeword
 * whose (d, p) is not the acceptor's code; shard_len != ceil(data_len / d) (rscoding.rs:177-181); a present shard of
 * another length; data_len >= 2^32; a body longer than 2^32 - 65 bytes; Crossword: an assignment that is not
 * `population` bitmaps of total_shards bits.  Non-minimal varints are read as the oracle's decoder reads them (tag 251
 * + u16 for a small value is that value) and stay as they came in the verbatim part of the record.
 * Ballot order (check_leader, rspaxos/leadership.rs:11-17, replayed in frame order): frame i of group g is checked
 * against max(bal_max_seen[g] before the call, the ballots of every earlier well-formed frame of g inside the window);
 * frames of different groups are independent.  Placement follows: the frames that pass take store and WAL regions by
 * exclusive scans in frame order; one whose region ends past store_capacity / wal_capacity is STORE_FULL / WAL_FULL
 * (SS_DEV_STATUS_STORE_FULL / SS_DEV_STATUS_FRAME_OVERFLOW), changes nothing and does not raise bal_max_seen.  At the
 * end bal_max_seen[g] = max(before, accepted ballots).  When several accepted frames name one (group, slot), the last in
 * frame order defines the instance (inst.bal, source, shards, assignment); every accepted frame still gets its record.
 * Outputs of accepted frame i (UINT64_MAX offsets and 0 lengths for the others):
 *   store: its held shards in index order at store + store_off[i] + k*SS_CW_SLOT_PITCH(L), bytes L..round_up(L,16)
 *          zero (the layout ss_engine_propose_ragged writes); store_off = exclusive scan of popcount(held)*pitch
 *   wal:   WalEntry::AcceptData at wal + wal_off[i] (16-byte aligned scan), wal_len[i] bytes: 8-byte big-endian length,
 *          wal_variant, then the frame's bytes from `slot` on, verbatim (rspaxos/mod.rs:219-228; Crossword keeps
 *          assignment, crossword/mod.rs:288-293)
 *   reply: PeerMessage::Msg{AcceptReply{slot, ballot[, size, reply_ts: None]}} in the 48-byte cell replies + 48*i,
 *          reply_len[i] bytes, to be sent to replica reply_dst[i] (0xff for frames not accepted).  ballot and
 *          destination are the instance's inst.bal and source after the whole call; Crossword size =
 *          popcount(assignment[me]) * (data_len / d + 1), the reference's formula (crossword/durability.rs:113-119).
 *          The host sends these cells only once the WAL records of the call are durable.
 * totals (device u64[2], may be NULL): the store and WAL bytes the batch asked for.  store and wal 16-byte aligned.
 * Cost: the ballot order and the placement walk each group's frames on one thread, so a batch costs its largest
 * per-group run of frames in those two steps (a batch that is mostly one group, e.g. a follower catching up, runs that
 * bookkeeping serially); the copy pass is a warp per frame whatever the grouping. */
int ss_acceptor_accept(ss_acceptor *acceptor, const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off,
                       const uint32_t *frame_group, const uint8_t *frame_peer, uint64_t n_frames, uint8_t *store,
                       uint64_t store_capacity, uint64_t *store_off, uint8_t *wal, uint64_t wal_capacity, uint64_t *wal_off,
                       uint32_t *wal_len, uint8_t *replies, uint32_t *reply_len, uint8_t *reply_dst, uint32_t *verdict,
                       uint64_t *totals);
/* Commit and execute on the acceptor: the commit half of heard_heartbeat (rspaxos/leadership.rs:222-311,
 * crossword/leadership.rs:260-359) and handle_logged_commit_slot's execution walk (rspaxos/durability.rs:125-186,
 * crossword/durability.rs:142-206).  Three more per-group arrays, all zero at creation: committed (ring word, bit s & 63
 * = Status::Committed), commit_bar (absolute: the first slot not yet submitted for execution) and exec_bar (absolute:
 * installed by the host as its state machine reports results, handle_cmd_result; the heartbeat filter reads it).
 * ss_acceptor_accept takes an accepted slot back to Accepting from Committed (rspaxos/messages.rs:363) and
 * ss_acceptor_advance clears committed on the retired positions.  Both walks start at max(commit_bar, window_base), so a
 * base installed by the host or moved by advance needs no fix-up.  Peer-side bookkeeping of heard_heartbeat stays on the
 * host: the Heartbeat reply, hear timers, peer_exec_bar and snap_bar.  The `Executed` status (empty batches) is not
 * tracked. */
typedef struct ss_acceptor_commit_view {
    uint64_t n_groups;
    uint64_t *committed;        /* [G] bit s & 63 = Status::Committed */
    uint64_t *commit_bar;       /* [G] */
    uint64_t *exec_bar;         /* [G] */
} ss_acceptor_commit_view;
int ss_acceptor_commit_view_get(ss_acceptor *acceptor, ss_acceptor_commit_view *view);
/* Heartbeat records (device arrays [n]: group, peer, ballot, commit_bar, exec_bar), replayed per group in record order
 * as if they arrived one at a time.  For each record of group g: if peer != me, bal_max_seen rises to its ballot
 * (check_leader); the record is skipped if ballot < bal_max_seen or its exec_bar < exec_bar[g]; otherwise slots from
 * max(commit_bar[g], window_base[g]) up to min(record's commit_bar, window_base[g] + 64) are walked: the walk breaks at
 * inst_bal < ballot or at a slot that is neither Accepting nor Committed, passes a committed slot, and commits the
 * others (committed bit set, accepting bit cleared, a WalEntry::CommitSlot to log).  Slots at or beyond window_base + 64
 * are left for a later heartbeat after ss_acceptor_advance.  Records with group >= n_groups are ignored.
 * newly (device [G], may be NULL): bit i = instance window_base[g] + i committed by THIS call, in window order as
 * ss_engine_tick writes it -- ss_wal_commit_pack_dev(newly, window_base, ...) packs the CommitSlot records. */
int ss_acceptor_heartbeat(ss_acceptor *acceptor, const uint32_t *hb_group, const uint8_t *hb_peer, const uint64_t *hb_ballot,
                          const uint64_t *hb_commit_bar, const uint64_t *hb_exec_bar, uint64_t n_records, uint64_t *newly);
/* Execution, once the CommitSlot records of earlier heartbeat calls are durable: for every group, from
 * max(commit_bar, window_base) while the slot is inside the window and committed, an instance holding fewer than d
 * shards postpones the walk (RSPaxos majority = d, Crossword num_data_shards); otherwise it executes and commit_bar
 * moves past it.  Its payload is get_data's input, the first data_len bytes of the concatenated data shards
 * (rscoding.rs:177-199, 581-683); a data shard not held is regenerated from the first d held shards in index order, as
 * reconstruct_data does (rscoding.rs:490-537).  The shards are read through shard_addr: the caller's acceptor stores
 * must still hold them.
 * Outputs, executed instances ordered by (group, slot): record k = rec_group[k], rec_slot[k] (absolute), rec_off[k],
 * rec_len[k] (= data_len); the payload at out + rec_off[k] in a region of round_up(data_len, 16) bytes, zero past
 * data_len (regions placed by exclusive scans; out 16-byte aligned).  totals (device u64[2], may be NULL): records and
 * bytes the walk asked for.  An instance whose record index reaches rec_capacity or whose region ends past out_capacity
 * does not execute and its group's walk stops there (SS_DEV_STATUS_EXEC_FULL); the offsets are monotone, so the
 * records written are a prefix and a host drains by calling again.  A committed instance with data_len == 0 is a null
 * codeword that get_data and reconstruct_data refuse (rscoding.rs:495-497, 581-583): it does not execute, its group's
 * walk stops there (SS_DEV_STATUS_EXEC_NULL). */
#define SS_DEV_STATUS_EXEC_FULL 32u
#define SS_DEV_STATUS_EXEC_NULL 64u
int ss_acceptor_execute(ss_acceptor *acceptor, uint8_t *out, uint64_t out_capacity, uint32_t *rec_group, uint64_t *rec_slot,
                        uint64_t *rec_off, uint32_t *rec_len, uint64_t rec_capacity, uint64_t *totals);
/* Reconstruct reads on the acceptor: handle_msg_reconstruct (rspaxos/messages.rs:468-516, crossword/messages.rs:577-632)
 * serves Reconstruct frames from the held shards, handle_msg_reconstruct_reply (rspaxos/messages.rs:519-594,
 * crossword/messages.rs:635-722) absorbs ReconstructReply shards into the store; ss_acceptor_execute then runs the
 * instances that now hold d shards.  Neither call writes a WAL record, as in the reference.  Frames are taken as by
 * ss_acceptor_accept: buf at any byte alignment, frame i at frame_off[i], of group frame_group[i] (>= n_groups:
 * malformed), from replica frame_peer[i] (the reply goes back to it).  The variant indices are arguments: Reconstruct is
 * PeerMsg 4 and ReconstructReply 5 in both protocols (rspaxos/mod.rs:249-310, crossword/mod.rs:324-398).  Verdicts:
 * SS_ACCEPT_VERDICT_ACCEPTED (handled), another message's variant index (0x80000000 | k for the PeerMessage variants),
 * SS_FRAME_KIND_MALFORMED (not decodable as the requested message), and the ones below.
 * Stated differences from the reference:
 *   1. absorb ignores entries beyond the 64-slot window (the reference indexes past its vector; its debug_assert says
 *      this does not happen);
 *   2. absorb ignores entries for instances that are neither Accepting nor Committed, and for null instances
 *      (data_len == 0): the reference debug_asserts status >= Committed, and absorb_other would adopt the entry's
 *      lengths while keeping zero-length shards, a codeword it cannot decode;
 *   3. an entry that fails absorb_other's checks (data_len / shard_len) is rejected alone; in the reference the error
 *      aborts the rest of that message, in HashMap iteration order, which is not deterministic;
 *   4. a present shard of the wrong length makes the frame malformed, as in ss_acceptor_accept; the reference would
 *      absorb it;
 *   5. served codewords carry the held shards and data_len, always with data_copy None; a reference replica that has
 *      executed an instance also sends the data shards reconstruct_data regenerated and, in RSPaxos, data_copy.
 *      Receivers ignore data_copy, and gossip only asks a peer for shards of its own assignment row, which it holds. */
#define SS_RECON_VERDICT_NULL_CODEWORD 0xfffffff6u    /* Crossword serve: a listed instance is a null codeword */
#define SS_RECON_VERDICT_SHARD_RANGE 0xfffffff7u      /* Crossword serve: flip(exclusion) selects a shard index >= T */
#define SS_RECON_VERDICT_OUT_FULL 0xfffffff8u         /* serve: the reply's region ends past out_capacity */
/* Serve: frame i is PeerMessage::Msg{Reconstruct{slots: Vec<usize>}} (RSPaxos) or {slots_excl: Vec<(usize, Bitmap)>}
 * (Crossword; a Bitmap is size, block count and u64 blocks as ssor_bitmap_encode writes it, read as Bitmap::decode
 * does: any number of blocks, padded with zeros or cut to the size).  The listed slots are walked in order: a slot
 * below window_base, at or beyond window_base + 64, or of an instance neither Accepting nor Committed is skipped.  The
 * entry is the held set (RSPaxos, skipped when empty) or held & flip(exclusion) (Crossword, skipped when empty), where
 * subset_copy walks the bits [0, size mod 256): its iterator stops at Bitmap::size(), a u8 (bitmap.rs:103-105,
 * 258-270).  Crossword subset_copy fails, and the reference sends nothing for the whole message, when a listed instance
 * is a null codeword (data_len == 0) or flip selects an index >= T (a bit of [T, size mod 256) left clear): the frame
 * gets SS_RECON_VERDICT_NULL_CODEWORD / _SHARD_RANGE and no reply.  A slot listed twice
 * is one entry, with the value of its last occurrence (Crossword: the last with a non-empty subset).
 * The reply is PeerMessage::Msg{ReconstructReply{slots_data}}, framed with the 8-byte big-endian length: the map length,
 * then per entry slot, inst.bal and the RSCodeword (d, p, data_len, shard_len, T shard Options, data_copy None) whose
 * shards are read through shard_addr.  Map order is unspecified in the reference; entries here follow the order of
 * their defining occurrences.  A frame whose map is empty gets reply_len 0 (the reference sends nothing).
 * Outputs: reply i at out + reply_off[i], reply_len[i] bytes; regions of round_up(reply_len, 16) bytes packed in frame
 * order by an exclusive scan (out 16-byte aligned; bytes past reply_len are not written); reply_off UINT64_MAX for
 * frames without a reply.  A reply whose region ends past out_capacity is not written: SS_RECON_VERDICT_OUT_FULL and
 * SS_DEV_STATUS_FRAME_OVERFLOW; the offsets are monotone, so the written replies are a prefix.  *total (device u64, may
 * be NULL) = the bytes the batch asked for.  Acceptor state is not changed.
 * Cost: the walk and the copy take a warp per frame; the copy writes the entries of a frame one after another. */
int ss_acceptor_reconstruct_serve(ss_acceptor *acceptor, const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off,
                                  const uint32_t *frame_group, const uint8_t *frame_peer, uint64_t n_frames,
                                  uint32_t reconstruct_variant, uint32_t reply_variant, uint8_t *out, uint64_t out_capacity,
                                  uint64_t *reply_off, uint64_t *reply_len, uint32_t *verdict, uint64_t *total);
/* Absorb: frame i is PeerMessage::Msg{ReconstructReply{slots_data: HashMap<usize, (Ballot, RSCodeword)>}}.  Every
 * codeword must carry the acceptor's d and p, shard_len = ceil(data_len / d) and exactly T shard Options, each present
 * shard shard_len bytes; data_copy is None or Some followed by exactly data_len bytes (a reference RSPaxos replica
 * that has executed the instance sends its cached batch, rscoding.rs:593-602).  A frame that does not decode so is
 * malformed and absorbs nothing.  A key repeated inside one frame counts once, with its last value (a HashMap decode
 * keeps the last insert).  Entries are taken in frame order, then wire order; an entry (slot, ballot, codeword) of
 * group g is ignored when the slot is outside [window_base, window_base + 64), the instance is neither Accepting nor
 * Committed, slot < exec_bar[g] (Executed), ballot < inst_bal, the instance is null, or data_len differs from the
 * instance's (absorb_other); otherwise it adds the shards the instance does not hold yet, so of two entries carrying
 * one shard index the first wins.  Every instance whose held mask grows gets a new region of
 * popcount(new held) * SS_CW_SLOT_PITCH(L) bytes in `store`, placed by an exclusive scan in (group, slot) order: the old
 * shards (copied from the old shard_addr) and the new ones in index order, in the padded layout ss_acceptor_accept
 * writes; held and shard_addr then name it.  An instance whose region would end past store_capacity is left unchanged
 * and its frames get SS_ACCEPT_VERDICT_STORE_FULL (SS_DEV_STATUS_STORE_FULL); the placed instances are a prefix, and
 * submitting the same frames again absorbs what was left.  absorbed[i] = the entries of frame i that added shards to a
 * placed instance; *total (device u64, may be NULL) = the store bytes the batch asked for.  store 16-byte aligned, not
 * overlapping the shards the instances hold.
 * Cost: a group's frames are walked by one warp (once to plan, twice to copy), so a batch costs its largest per-group
 * run of entries; the copies take the whole warp. */
int ss_acceptor_absorb(ss_acceptor *acceptor, const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off,
                       const uint32_t *frame_group, const uint8_t *frame_peer, uint64_t n_frames, uint32_t reply_variant,
                       uint8_t *store, uint64_t store_capacity, uint32_t *absorbed, uint32_t *verdict, uint64_t *total);
/* Prepare on the acceptor, the follower half of leader fail-over: handle_msg_prepare (rspaxos/messages.rs:13-84,
 * crossword/messages.rs:63-136) and, once its PrepareBal records are durable, the follower branch of
 * handle_logged_prepare_bal (rspaxos/durability.rs:10-79, crossword/durability.rs:9-79).  Five more arrays, all zero at
 * creation: preparing (ring word, bit s & 63 = Status::Preparing), inst.voted = (voted_bal, voted_mask) kept apart from
 * inst_bal and held, and replica_bk's trigger_slot and endprep_slot - trigger_slot (always < 64).  An accepted Accept
 * sets voted = (ballot, the frame's shards), clears preparing and sets trigger and span to 0 (replica_bk = {source, 0,
 * 0}, rspaxos/messages.rs:365-372); ss_acceptor_advance clears preparing on the retired positions; absorb leaves the vote
 * alone, and shard j of the vote sits at rank popcount(held & ((1 << j) - 1)) of the instance's store region, since the
 * vote stays a subset of held.  A Preparing instance is neither Accepting nor Committed: it stops the heartbeat commit
 * walk and the execution walk, and serve and absorb skip it, as the reference's `status < Accepting` checks do. */
typedef struct ss_acceptor_prepare_view {
    uint64_t n_groups;
    uint64_t *preparing;        /* [G] bit s & 63 = Status::Preparing */
    uint64_t *voted_bal;        /* [G*64] ballot of inst.voted; 0 = voted None */
    uint32_t *voted_mask;       /* [G*64] shard set of inst.voted */
    uint64_t *prep_trigger;     /* [G*64] replica_bk.trigger_slot */
    uint8_t *prep_span;         /* [G*64] replica_bk.endprep_slot - trigger_slot */
} ss_acceptor_prepare_view;
int ss_acceptor_prepare_view_get(ss_acceptor *acceptor, ss_acceptor_prepare_view *view);
/* Prepare frames, taken as by ss_acceptor_accept: buf at any byte alignment, frame i at frame_off[i], of group
 * frame_group[i] (>= n_groups: malformed), from replica frame_peer[i].  Frame i is PeerMessage::Msg{Prepare{trigger_slot,
 * ballot}}; prepare_variant (PeerMsg::Prepare, 0) and wal_variant (WalEntry::PrepareBal, 0; below 2^16) are arguments.
 * verdict[i]: SS_ACCEPT_VERDICT_ACCEPTED; SS_ACCEPT_VERDICT_STALE_SLOT (trigger_slot < window_base, ignored);
 * SS_ACCEPT_VERDICT_STALE_BALLOT (ballot < bal_max_seen as it stands when the frame is reached);
 * SS_ACCEPT_VERDICT_BEYOND_WINDOW (trigger_slot >= window_base + 64: re-submit after ss_acceptor_advance);
 * SS_ACCEPT_VERDICT_WAL_FULL (below); another message's variant index (0x80000000 | k for the PeerMessage variants);
 * SS_FRAME_KIND_MALFORMED: truncated, trailing bytes, a variant >= 2^16, or a Prepare whose frame_peer is `me`.
 * Each group's frames are replayed in frame order as if they arrived one at a time.  A frame that passes raises
 * bal_max_seen to its ballot; endprep_slot = max(window_base + the last window position that is Preparing, Accepting or
 * Committed, trigger_slot), with the positions earlier frames of the call made Preparing counted as such; every slot of
 * [trigger_slot, endprep_slot] gets inst_bal = ballot, Status::Preparing (also over Committed), source = frame_peer and
 * the frame's trigger and span; a slot that was null (neither Preparing, Accepting nor Committed) also gets voted None
 * (voted_bal = voted_mask = 0), as a fresh null_instance() has it, so a retired position leaks no earlier vote.  Of
 * several frames covering one slot the last applied defines it.
 * Records: one WalEntry::PrepareBal{slot, ballot} per slot of each applied frame's range, numbered by an exclusive scan
 * of the per-frame counts in frame order; record k is the 32-byte cell wal + 32k (8-byte big-endian length + bincode
 * body, at most 29 bytes, zero to the end of the cell), with rec_group[k], rec_slot[k] (absolute) and rec_frame[k]
 * beside it.  totals (device u64[2], may be NULL): the records and the WAL bytes (32 per record) the batch asked for.
 * Capacity: the first frame in frame order whose records end past rec_capacity or past wal_capacity / 32 cells gets
 * SS_ACCEPT_VERDICT_WAL_FULL and changes nothing, and so does every later frame whose verdict came from the replay
 * (ACCEPTED or STALE_BALLOT); SS_DEV_STATUS_FRAME_OVERFLOW.  The applied frames are then a prefix in frame order, and
 * within each group a prefix of its frames, so the ranges computed for them stay exact; the host re-submits the rest.
 * Unlike ss_acceptor_accept's per-frame cut this cut is a suffix, because a Prepare's range depends on the Prepares before
 * it in its group.  wal 16-byte aligned.
 * Stated differences from the reference: the window (a trigger beyond it is re-submitted; the reference grows its log
 * with null instances instead, and endprep_slot never reaches past the window); the capacity suffix above; a Prepare
 * from `me` is malformed, where check_leader debug-asserts peer != me.  Peer-side bookkeeping of check_leader (leader
 * change, hear timers) stays on the host.
 * Cost: the walk and the apply pass take a thread per group segment, so a batch costs its largest per-group run of
 * frames there; the record cells and per-slot writes take a warp per applied frame. */
int ss_acceptor_prepare(ss_acceptor *acceptor, const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off,
                        const uint32_t *frame_group, const uint8_t *frame_peer, uint64_t n_frames, uint32_t prepare_variant,
                        uint32_t wal_variant, uint8_t *wal, uint64_t wal_capacity, uint32_t *rec_group, uint64_t *rec_slot,
                        uint32_t *rec_frame, uint64_t rec_capacity, uint32_t *verdict, uint64_t *totals);
/* PrepareReply frames for PrepareBal records that became durable (device arrays [n_records], normally rec_group /
 * rec_slot of ss_acceptor_prepare).  The instance's state is read when this call runs, as the reference reads inst.bal,
 * replica_bk and inst.voted when the log result arrives.  Record k produces nothing (reply_len 0, reply_off UINT64_MAX,
 * reply_dst 0xff) when its group is >= n_groups, its slot is outside [window_base, window_base + 64), or the instance is
 * null (no replica_bk).  Otherwise it produces PeerMessage::Msg{PrepareReply{slot, trigger_slot, endprep_slot, ballot:
 * inst_bal, voted}}, framed with the 8-byte big-endian length, for replica reply_dst[k] = source; reply_variant is
 * PeerMsg::PrepareReply (1).  voted = Some((voted_bal, RSCodeword)) when voted_bal > 0, else None; the codeword carries
 * d, p, data_len, shard_len, T shard Options with the voted_mask shards read through shard_addr at their rank in held,
 * and data_copy None.  An instance accepted after the Prepare replies with trigger and endprep 0, as the reference does.
 * Regions of round_up(reply_len, 16) bytes are placed by an exclusive scan in record order at out + reply_off[k] (out
 * 16-byte aligned; bytes past reply_len are not written).  A reply whose region ends past out_capacity is not written:
 * reply_off UINT64_MAX with reply_len kept, reply_dst 0xff, SS_DEV_STATUS_FRAME_OVERFLOW; the offsets are monotone, so
 * the written replies are a prefix and a host drains by calling again with the rest.  *total (device u64, may be NULL)
 * = the bytes the batch asked for.  Acceptor state is not changed.
 * The records of ss_acceptor_step_up go through this call too: their instances have source = me, so their replies have
 * reply_dst = me, the new leader's reply from itself (rspaxos/durability.rs:29-48).  Nothing here refuses that; the host
 * hands those frames to ss_prepare_reply_parse_dev with its peers' replies instead of sending them.
 * Cost: a thread per record sizes, a warp per record writes. */
int ss_acceptor_prepare_reply(ss_acceptor *acceptor, const uint32_t *rec_group, const uint64_t *rec_slot, uint64_t n_records,
                              uint32_t reply_variant, uint8_t *out, uint64_t out_capacity, uint64_t *reply_off,
                              uint64_t *reply_len, uint8_t *reply_dst, uint64_t *total);
/* WAL recovery on the acceptor: recover_apply_entry and recover_from_wal (rspaxos/recovery.rs:10-181,
 * crossword/recovery.rs:10-186) for the records the acceptor writes -- WalEntry::PrepareBal{slot, ballot}
 * (ss_acceptor_prepare), AcceptData{slot, ballot, reqs_cw[, assignment]} (ss_acceptor_accept) and CommitSlot{slot}
 * (ss_wal_commit_pack_dev) -- replayed into the window and the shard store without a record crossing to the host.
 * Record i is at buf + rec_off[i] (any byte alignment) as the device writes it: an 8-byte big-endian length, then the
 * bincode WalEntry, whose variant is prepare_variant (PrepareBal, 0), cfg.wal_variant (AcceptData, 1) or commit_variant
 * (CommitSlot, 2); the three must differ.  Record i belongs to group rec_group[i]; a group's records are replayed in
 * array order, which is WAL order, on top of the state the acceptor holds (normally a fresh acceptor whose window_base
 * the host installed from the snapshot's start_slot); groups are independent.
 *   PrepareBal: inst_bal = ballot, Status::Preparing (also over Accepting or Committed).
 *   AcceptData: inst_bal = ballot, Status::Accepting (also out of Committed), held = the record's shards with its
 *               data_len, voted = (ballot, held); Crossword: assignment[me] and the whole row set into assign_rows.  The
 *               record is decoded by the rules ss_acceptor_accept applies to the Accept body (code, shard_len, shard
 *               lengths, assignment shape, non-minimal varints).
 *   CommitSlot: Status::Committed (also on a null position, as the reference does).
 * A position that was null (neither Preparing, Accepting nor Committed) when a record first touches it starts as a
 * fresh null_instance(): inst_bal 0, no shards, data_len 0, voted None (Crossword: empty assignment), so a retired
 * position leaks nothing into the replay.  Every position a record touches gets source 0xff and trigger / span 0
 * (replica_bk is None after recovery).  bal_max_seen[g] = max(before, the ballot of every applied record).
 * commit_bar, exec_bar and gossip_bar are not changed.
 * Shards: of the applied AcceptData records of one (group, slot) the last defines the instance; only its shards are
 * copied into `store`, popcount(held) * SS_CW_SLOT_PITCH(L) bytes in the padded layout ss_acceptor_accept writes, and
 * shard_addr names that copy.  Regions are placed by an exclusive scan in (group, window position) order; *total
 * (device u64, may be NULL) = the store bytes the batch asked for.  store 16-byte aligned.
 * verdict[i]:
 *   SS_ACCEPT_VERDICT_ACCEPTED         applied;
 *   SS_ACCEPT_VERDICT_STALE_SLOT       slot < window_base: ignored, as in the reference;
 *   SS_ACCEPT_VERDICT_BEYOND_WINDOW    slot >= window_base + 64: this record and every later record of its group are
 *                                      not applied; the host executes, advances and re-submits them;
 *   SS_FRAME_KIND_MALFORMED            the length runs past buf_len, trailing bytes, a variant that is none of the
 *                                      three, a record that fails the accept decode rules, or a group >= n_groups.  For
 *                                      a valid group the group's log ends there, as the reference's read loop ends at
 *                                      the first entry it cannot decode and truncates: every later record of the group
 *                                      gets SS_RECOVER_VERDICT_AFTER_END;
 *   SS_ACCEPT_VERDICT_STORE_FULL       the capacity cut is per group: a group whose store region ends past
 *                                      store_capacity applies nothing, its records that would apply get STORE_FULL and
 *                                      SS_DEV_STATUS_STORE_FULL is set.  The offsets are monotone, so the placed groups
 *                                      are a prefix in group order; re-submitting the STORE_FULL records finishes the job.
 * Stated differences from the reference:
 *   1. the 64-slot window, with the suffix cut and re-submission above (the reference grows its log with null
 *      instances);
 *   2. execution is not replayed: the reference executes each contiguous committed prefix as it reads and then sets
 *      exec_bar = commit_bar; here the host runs ss_acceptor_execute after the call and installs exec_bar as it does
 *      today.  The two differ only for a slot whose CommitSlot is followed in the same WAL by a PrepareBal or AcceptData
 *      of that slot: the reference has already executed it, here it waits for a heartbeat to commit it again;
 *   3. the per-group capacity cut;
 *   4. bal_prep_sent and bal_prepared are leader words, which the acceptor does not have: they are not recovered.
 * Cost: the walk and the replay take a thread per group segment, so a batch costs its largest per-group run of records
 * there; the shard copies take a warp per defining record. */
#define SS_RECOVER_VERDICT_AFTER_END 0xfffffff9u   /* after a malformed record of its group: the group's log ended */
int ss_acceptor_recover(ss_acceptor *acceptor, const uint8_t *buf, uint64_t buf_len, const uint64_t *rec_off,
                        const uint32_t *rec_group, uint64_t n_records, uint32_t prepare_variant, uint32_t commit_variant,
                        uint8_t *store, uint64_t store_capacity, uint32_t *verdict, uint64_t *total);
/* Reconstruct requests from the acceptor, for the committed instances it cannot execute from its own shards: Crossword
 * follower gossip (trigger_gossiping with gossip_targets_excl, crossword/gossiping.rs:35-192; the reference runs it on
 * the gossip timer in the groups this replica does not lead, crossword/mod.rs:1150) and the reconstruct half of a new
 * leader's become_a_leader (recon_slots, rspaxos/leadership.rs:99-172, crossword/leadership.rs:105-190).  The peers
 * serve them with ss_acceptor_reconstruct_serve, this acceptor absorbs the replies with ss_acceptor_absorb and
 * ss_acceptor_execute runs what now holds d shards, all without the window state leaving the device.
 * Two more arrays: assign_rows (Crossword only, [G*64*population] u32, population * 256 bytes per group: row r of the
 * instance at ring position p of group g at (g*64 + p)*population + r, the instance's whole `assignment: Vec<Bitmap>`,
 * written by ss_acceptor_accept from the frame that defines the instance, beside assignment[me]) and gossip_bar ([G],
 * zero at creation; ss_acceptor_advance leaves it alone).  assign_rows is NULL for RSPaxos. */
typedef struct ss_acceptor_gossip_view {
    uint64_t n_groups;
    uint32_t population, pad0;
    uint32_t *assign_rows;      /* Crossword [G*64*population]; NULL for RSPaxos */
    uint64_t *gossip_bar;       /* [G] absolute */
} ss_acceptor_gossip_view;
int ss_acceptor_gossip_view_get(ss_acceptor *acceptor, ss_acceptor_gossip_view *view);
/* Gossip (Crossword only; RSPaxos: SS_ERR_INVALID_ARG).  groups (device u32 [n_listed]) lists the groups to walk, in
 * the order their frames come out (the host leaves out the groups it leads); NULL walks every group in index order.  A
 * listed group >= n_groups is ignored; a group listed twice is planned twice from the state before the call.
 * peer_alive (device [G] u32 peer masks) may be NULL: every peer alive.  batch_size >= 1 (the host resolves
 * gossip_batch_size == 0 to msg_chunk_size); reconstruct_variant is PeerMsg::Reconstruct (4).
 * Per listed group g, trigger_gossiping: log_end = window_base + 1 + the last window position that is Preparing,
 * Accepting or Committed (window_base when none is); until = log_end - tail_ignores (0 below); slot_up_to = gossip_bar;
 * every slot of [max(gossip_bar, window_base), until) in order sets slot_up_to = slot, then: slot < exec_bar is Executed
 * and passed; a slot that is not Committed stops the walk; a Committed instance holding fewer than d shards is planned by
 * gossip_targets_excl (src_peer = source, avail = held, the instance's assign_rows, peer_alive[g]; the walk of
 * ss_gossip_plan_dev), and every selected peer gets the entry (slot, Bitmap{size T, avail at that moment}).  A null
 * instance (data_len 0) is planned like any other.  Then gossip_bar = max(gossip_bar, slot_up_to): the last slot
 * visited is walked again next time, as in the reference.
 * Frames: each peer's entries in slot order, cut into frames of batch_size entries (the last one partial); frame =
 * 8-byte big-endian length + PeerMessage::Msg{Reconstruct{slots_excl: Vec<(usize, Bitmap)>}}, the Bitmap as
 * ssor_bitmap_encode writes it (size, one block, the block) -- what ss_acceptor_reconstruct_serve parses.  Frames are
 * ordered by (listed group, peer, chunk): frame f is frame_group[f], for replica frame_dst[f], at out + frame_off[f]
 * (16-byte aligned regions of round_up(frame_len, 16) bytes placed by exclusive scans of the per-group frames and bytes;
 * out 16-byte aligned; bytes past frame_len are not written).  totals (device u64[2], may be NULL): the frames and bytes
 * the call asked for.
 * Capacity is per group: a listed group whose frames end past frame_capacity or whose region ends past out_capacity
 * writes no frame and keeps its gossip_bar; its frame records below frame_capacity get frame_off UINT64_MAX, frame_len 0
 * and frame_dst 0xff; SS_DEV_STATUS_FRAME_OVERFLOW.  The ends are monotone, so the written groups are a prefix of the
 * list, and calling again with the same arguments plans the rest as this call would have.
 * Stated differences from the reference:
 *   1. log_end is the window, not start_slot + insts.len(): the reference also counts trailing null instances that a
 *      Prepare or a step-up appended to its vector;
 *   2. Executed is slot < exec_bar (the host installs exec_bar), as in ss_acceptor_absorb;
 *   3. the per-group capacity cut above (the reference sends every frame);
 *   4. assign_rows costs population * 256 bytes per group of device memory on a Crossword acceptor.
 * Cost: a warp per listed group, each lane two window positions; gossip_targets_excl runs once per instance and once
 * more per selected peer, so a group costs O(population^2) per position in the worst case. */
int ss_acceptor_gossip(ss_acceptor *acceptor, const uint32_t *groups, uint64_t n_listed, const uint32_t *peer_alive,
                       uint64_t tail_ignores, uint64_t batch_size, uint32_t reconstruct_variant, uint8_t *out,
                       uint64_t out_capacity, uint32_t *frame_group, uint8_t *frame_dst, uint64_t *frame_off,
                       uint32_t *frame_len, uint64_t frame_capacity, uint64_t *totals);
/* Step-up reads (RSPaxos and Crossword): the reconstruct half of become_a_leader.  groups, outputs and capacity as for
 * ss_acceptor_gossip; chunk_size (msg_chunk_size) >= 1.  Per listed group every slot of
 * [max(exec_bar, window_base), window_base + 64) is walked with no stop, and each Committed instance holding fewer than
 * d shards (RSPaxos: majority, the acceptor's d) is listed; the list is cut into frames of chunk_size entries,
 * PeerMessage::Msg{Reconstruct{slots}} (RSPaxos) or {slots_excl} with the exclusion = held as a size-T Bitmap
 * (Crossword), each with frame_dst 0xff: the host broadcasts it.  No state changes; the Prepare, PrepareBal and ballot
 * parts of become_a_leader are ss_acceptor_step_up, which runs first: the instances it leaves Preparing are not listed. */
int ss_acceptor_step_up_reads(ss_acceptor *acceptor, const uint32_t *groups, uint64_t n_listed, uint64_t chunk_size,
                              uint32_t reconstruct_variant, uint8_t *out, uint64_t out_capacity, uint32_t *frame_group,
                              uint8_t *frame_dst, uint64_t *frame_off, uint32_t *frame_len, uint64_t frame_capacity,
                              uint64_t *totals);
/* Step-up (RSPaxos and Crossword): the Prepare half of become_a_leader (rspaxos/leadership.rs:45-185,
 * crossword/leadership.rs:47-190) on this replica's acceptor, whose window is the new leader's instance log.  groups
 * (device u32 [n_listed]) lists the groups to step up in; NULL steps up every group in index order.  A listed group >=
 * n_groups is ignored: verdict SS_FRAME_KIND_MALFORMED, ballot, trigger_slot and endprep_slot 0.  Each group's entries run
 * in list order as if they came one at a time, so a group listed twice steps up twice: the second entry takes
 * make_greater_ballot of the first entry's ballot, finds the same trigger, endprep and instances, and defines them.
 * Per entry of group g, in window terms:
 *   ballot b = make_greater_ballot(bal_max_seen[g]) = ((bal_max_seen[g] >> 8) + 1) << 8 | (me + 1), in u64
 *     (rspaxos/mod.rs:446-454); then bal_max_seen[g] = b;
 *   log_end = window_base + 1 + the last window position that is Preparing, Accepting or Committed (window_base when
 *     none is), as in ss_acceptor_gossip; a slot is done when it is Committed or below exec_bar (Executed);
 *   trigger_slot = the first slot of [window_base, log_end) that is not done, log_end when every slot is done (the
 *     reference pushes a null instance there; here that position is taken into the Prepare); endprep_slot = the last
 *     slot that is not done, trigger_slot when every slot is done;
 *   trigger_slot = window_base + 64: SS_ACCEPT_VERDICT_BEYOND_WINDOW and nothing changes; the host advances and lists
 *     the group again;
 *   every slot of [max(exec_bar, window_base), endprep_slot] that is not Committed gets inst_bal = b, Status::Preparing
 *     (Accepting cleared), source = me, trigger_slot and endprep_slot - trigger_slot (replica_bk, read by
 *     ss_acceptor_prepare_reply).  A slot that was null becomes a fresh null_instance(): voted None, held 0, data_len 0
 *     (Crossword: an empty assignment row); an accepted instance keeps its vote, held shards and store region.
 *     Committed instances are not touched: ss_acceptor_step_up_reads lists them afterwards.
 * Records: one WalEntry::PrepareBal{slot, b} per marked slot, in slot order, numbered by an exclusive scan in list order;
 * record k is the 32-byte cell wal + 32k that ss_acceptor_prepare writes, with rec_group[k] and rec_slot[k] (absolute).
 * Frames: one PeerMessage::Msg{Prepare{trigger_slot, ballot: b}} per applied entry, numbered by an exclusive scan in list
 * order: frame f is the 32-byte cell out + 32f (8-byte big-endian length + body, at most 30 bytes, zero to the end of the
 * cell), frame_off[f] = 32f, frame_len[f], frame_group[f] and frame_dst[f] = 0xff: the host broadcasts it.
 * prepare_variant (PeerMsg::Prepare, 0) and wal_variant (WalEntry::PrepareBal, 0) are below 2^16.
 * Per listed entry i: verdict[i], ballot[i] = b, trigger_slot[i] and endprep_slot[i], the values the entry takes when
 * the whole list applies.  verdict[i]: SS_ACCEPT_VERDICT_ACCEPTED, SS_ACCEPT_VERDICT_BEYOND_WINDOW, or
 * SS_ACCEPT_VERDICT_WAL_FULL: its records end past rec_capacity or past wal_capacity / 32 cells, or its frame past
 * frame_capacity or past out_capacity / 32 cells.  Such an entry changes nothing, and neither does any later entry: the
 * ends are monotone, so the applied entries are a prefix of the list; SS_DEV_STATUS_FRAME_OVERFLOW is set, its frame
 * record below frame_capacity gets frame_off UINT64_MAX, frame_len 0 and frame_dst 0xff, and calling again with the
 * rest of the list finishes the job.  totals (device u64[4], may be NULL): the records, WAL bytes, frames and frame
 * bytes the call asked for.  wal and out 16-byte aligned.
 * The leader's own vote: once the PrepareBal records are durable, the host passes rec_group / rec_slot to
 * ss_acceptor_prepare_reply, which sends a replica's PrepareReply to the instance's source.  Here that is me: the
 * replies with reply_dst = me are the leader's "reply from myself" (rspaxos/durability.rs:29-48), carrying its voted
 * shards, and ss_prepare_reply_parse_dev reads them like any peer's.
 * What stays with the host: disallow_step_up, the timeout_source check, the leader status, the heartbeat broadcast,
 * peer_exec_bar and the engine's bal_prepared (cleared through ss_engine_set_prepared_ballots); bal_prep_sent is
 * ballot[i], which the acceptor does not keep.
 * Stated differences from the reference:
 *   1. the 64-slot window, not start_slot + insts.len(): the reference also counts trailing null instances that a
 *      Prepare or an earlier step-up appended to its vector, and a trigger at window_base + 64 is BEYOND_WINDOW;
 *   2. the capacity cut above (the reference logs and sends everything).
 * Cost: the walk and the apply pass take a thread per group segment; the records, frames and per-slot writes take a warp
 * per applied entry. */
int ss_acceptor_step_up(ss_acceptor *acceptor, const uint32_t *groups, uint64_t n_listed, uint32_t prepare_variant,
                        uint32_t wal_variant, uint8_t *wal, uint64_t wal_capacity, uint32_t *rec_group, uint64_t *rec_slot,
                        uint64_t rec_capacity, uint8_t *out, uint64_t out_capacity, uint32_t *frame_group, uint8_t *frame_dst,
                        uint64_t *frame_off, uint32_t *frame_len, uint64_t frame_capacity, uint32_t *verdict, uint64_t *ballot,
                        uint64_t *trigger_slot, uint64_t *endprep_slot, uint64_t *totals);
/* PrepareReply frames -> one record per frame for the new leader (a thread per frame, no copies; the PrepareReply
 * counterpart of ss_accept_reply_parse_dev).  Frame i at buf + frame_off[i] (any alignment) must be
 * PeerMessage::Msg{PrepareReply{slot, trigger_slot, endprep_slot, ballot, voted}} whose codeword, when voted is Some,
 * carries this d and p, shard_len = ceil(data_len / d) with data_len < 2^32, exactly T shard Options each present one
 * shard_len bytes, and data_copy None or Some followed by exactly data_len bytes -- the rules ss_acceptor_absorb applies.
 * kind = reply_variant for such a frame; another message's variant index (0x80000000 | k for the PeerMessage variants);
 * SS_FRAME_KIND_MALFORMED otherwise (including trailing bytes and variants >= 2^16).  The other fields are zero and
 * shards_at UINT64_MAX unless kind = reply_variant.  Group, peer and instance indexing stay the caller's: it scatters
 * vote_bal / vote_mask into the [r*N + i] arrays ss_prepare_merge_dev takes. */
typedef struct ss_prepare_reply_rec {
    uint64_t slot, trigger_slot, endprep_slot, ballot;
    uint64_t vote_bal;          /* 0 for voted None */
    uint64_t shards_at;         /* offset in buf of the codeword's first shard Option tag; UINT64_MAX for None */
    uint32_t vote_mask;         /* shards present */
    uint32_t data_len;
    uint32_t kind;
    uint32_t pad;
} ss_prepare_reply_rec;
int ss_prepare_reply_parse_dev(ss_ctx *ctx, const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off, uint64_t n_frames,
                               uint32_t data_shards, uint32_t total_shards, uint32_t reply_variant, ss_prepare_reply_rec *rec);
/* PrepareReply absorb on the new leader (RSPaxos and Crossword engines): handle_msg_prepare_reply (rspaxos/messages.rs:
 * 88-326, crossword/messages.rs:140-400) for a batch of PrepareReply frames over many groups, after ss_acceptor_step_up
 * on this replica's acceptor `acceptor`.  The engine and the acceptor must share context, protocol, n_groups, population,
 * d and T (else SS_ERR_INVALID_ARG, as is any other protocol); a code with d + p > 12 gives SS_ERR_UNSUPPORTED, because
 * the batched reconstruct does not take it.
 * Frames are taken as ss_acceptor_prepare takes them: buf at any byte alignment, frame i at frame_off[i], of group
 * frame_group[i] (>= n_groups: malformed), from replica frame_peer[i] (>= population: malformed); reply_variant is
 * PeerMsg::PrepareReply (1), wal_variant WalEntry::PrepareBal (0).  The leader's own replies, the frames of
 * ss_acceptor_prepare_reply with reply_dst = me, go in the same batch as any peer's.  bal_prep_sent (device [G]) is the
 * ballot ss_acceptor_step_up returned for the group, 0 where this replica is not preparing: is_leader and bal_prep_sent
 * stay with the host.  policy (Crossword, device [G], may be NULL = 0) is the assignment policy of the re-accepts.
 * Each group's frames are replayed in frame order as if they arrived one at a time.  Per frame, decoded by the decoder of
 * ss_prepare_reply_parse_dev, in the reference's order:
 *   slot < window_base: SS_ACCEPT_VERDICT_STALE_SLOT;
 *   ballot != bal_prep_sent[g], bal_prep_sent[g] = 0, or a trigger_slot outside the window or whose instance this leader
 *     did not prepare before the call (source != me: leader_bk is None; a position the call filled lies past the
 *     leader's endprep_slot, so it is no trigger of this leader): SS_PREP_VERDICT_IGNORED;
 *   slot >= window_base + 64: SS_ACCEPT_VERDICT_BEYOND_WINDOW, re-submitted after an advance;
 *   external fill (messages.rs:127-170): every position from the log end (one past the last position that is Preparing,
 *     Accepting or Committed, counting the positions earlier frames of the call filled) through the slot becomes a fresh
 *     null instance, Preparing on the acceptor with inst_bal = bal_prep_sent, source = me and the trigger's trigger and
 *     span, and gets one WalEntry::PrepareBal 32-byte cell as ss_acceptor_prepare writes them;
 *   the instance is not Preparing (or was decided at this ballot), or ballot < inst_bal: SS_PREP_VERDICT_IGNORED;
 *   vote merge (ss_prepare_merge_dev's rule): a higher vote ballot replaces prepare_max_bal and the gathered codeword,
 *     which takes a new store slot sized by its data_len (an empty Some clears the shards); an equal one adds the shards
 *     not gathered yet; a same-ballot codeword with another data_len is rejected alone, SS_PREP_VERDICT_DATA_LEN, where
 *     absorb_other errors; SS_ACCEPT_VERDICT_ACCEPTED otherwise;
 *   slot == endprep_slot: the peer joins prepare_acks; whenever the count is then at least the majority, bal_prepared[g]
 *     = ballot and every Preparing position from the trigger on that is not decided is decided by ss_prepare_merge_dev's
 *     rule: USE (at least d shards gathered), NULL (fewer, but acks >= population - f: RSCodeword::from_data(ReqBatch::new(),
 *     d, p), which is data_len 1 -- bincode 2 standard() writes an empty Vec as the single byte 0x00, from knowledge of the
 *     crate, unpinned -- shard_len 1 and every shard zero), or not yet: a later decision point decides it.  The first
 *     quorum of a ballot rebuilds the engine's window of g from the acceptor (window_base, committed, commit_bar = its
 *     committed prefix, accepting and ack planes cleared); each decided instance enters Accepting as a proposal does,
 *     with an empty ack set, inst_bal = ballot and (Crossword) policy_idx = policy[g].
 * The engine keeps the bookkeeping between calls: per group the ballot it belongs to, prepare_acks and the decided
 * positions, per ring position prepare_max_bal and the gathered codeword; it resets when bal_prep_sent[g] differs from
 * that ballot, so a second step-up needs no host reset.
 * Store: CALLER-owned, T planes at shards + j*plane_stride (plane_stride a multiple of 32, shards 16-byte aligned), the
 * layout ss_engine_propose_ragged writes.  Slots of SS_CW_SLOT_PITCH(shard_len) bytes in every plane are bump-allocated
 * in group order from *store_used (device u64, in/out, rounded up to 32); an abandoned slot is not reused.  Shard j of
 * a gathered codeword is at shards + j*plane_stride + its slot, bytes shard_len..round_up(shard_len, 16) zero.
 * Outputs, the decided list ordered by group, then by the frame that decided the instance, then by slot, as separate
 * arrays in the order ss_frame_accept_pack_ragged_dev takes them: dec_slot (absolute), dec_ballot, dec_shard_off,
 * dec_data_len, dec_policy (may be NULL), dec_group.  Every decided codeword holds all T shards: the missing ones of a
 * USE codeword are regenerated in place by one ss_rs_reconstruct_batch_dev launch over the list's capacity; entries
 * past the decided count get dec_data_len 0.  The external fill's cells at wal + 32k with rec_group[k], rec_slot[k].
 * pending[g] (device [G]): the acceptor's Preparing ring positions not yet decided at bal_prep_sent[g] (0 where it is
 * 0).  verdict[i] per frame.  totals (device u64[3], may be NULL): decided records, PrepareBal records and store bytes
 * the call asked for.
 * Capacity is per group, as in ss_acceptor_recover: a group whose store slots end past plane_stride, whose cells end
 * past min(rec_capacity, wal_capacity / 32) or whose decided records end past dec_capacity applies none of its frames;
 * its well-formed frames get SS_ACCEPT_VERDICT_STORE_FULL (SS_DEV_STATUS_STORE_FULL) or SS_ACCEPT_VERDICT_WAL_FULL
 * (SS_DEV_STATUS_FRAME_OVERFLOW).  The ends are monotone in group order, so the applied groups are a prefix and
 * re-submitting the cut frames finishes the job.
 * After the call the host packs each peer's Accept, and its own, with ss_frame_accept_pack_ragged_dev over the decided
 * list (peer = r), and hands its own frame to its own ss_acceptor_accept in the same turn, before any other frame of
 * those groups: that call leaves Preparing with voted = (ballot, my shards), writes the AcceptData record and emits the
 * self AcceptReply, which goes through ss_accept_reply_parse_dev to ss_engine_ingest (handle_logged_accept_data);
 * ss_engine_tick then commits.
 * Stated differences from the reference:
 *   1. the 64-slot window, with BEYOND_WINDOW and re-submission;
 *   2. proposals are fenced by the host: the reference's first_null_slot skips Preparing slots, ss_engine_propose_* do
 *      not know them, so a host does not propose in a group while pending[g] != 0;
 *   3. parity is always regenerated: where the reference skips compute_parity (avail_shards >= population, Crossword
 *      with T > n), its Accepts carry None for the missing parity shards, here the regenerated ones;
 *   4. the per-group capacity cut;
 *   5. a same-ballot codeword with another data_len is rejected alone (SS_PREP_VERDICT_DATA_LEN);
 *   6. `external` and the client replies stay with the host.
 * Cost: decode a thread per frame; the walk a warp per group segment, twice (count, then apply), so a batch costs its
 * largest per-group run of frames there; the shard copy a warp per frame; the reconstruct a warp per decided record of
 * the capacity. */
#define SS_PREP_VERDICT_IGNORED 0xfffffffau       /* not this leader's Prepare, not Preparing, or ballot < inst_bal */
#define SS_PREP_VERDICT_DATA_LEN 0xfffffffbu      /* a same-ballot codeword whose data_len differs: rejected alone */
int ss_engine_prepare_absorb(ss_engine *engine, ss_acceptor *acceptor, const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off,
                             const uint32_t *frame_group, const uint8_t *frame_peer, uint64_t n_frames, uint32_t reply_variant,
                             uint32_t wal_variant, const uint64_t *bal_prep_sent, const uint8_t *policy, uint8_t *shards,
                             uint64_t plane_stride, uint64_t *store_used, uint8_t *wal, uint64_t wal_capacity, uint32_t *rec_group,
                             uint64_t *rec_slot, uint64_t rec_capacity, uint64_t *dec_slot, uint64_t *dec_ballot,
                             uint64_t *dec_shard_off, uint32_t *dec_data_len, uint8_t *dec_policy, uint32_t *dec_group,
                             uint64_t dec_capacity, uint64_t *pending, uint32_t *verdict, uint64_t *totals);
/* Soft fallback on a Crossword leader: fallback_redo_accepts (crossword/leadership.rs:389-550), which the reference runs
 * from bcast_heartbeats when peer_alive loses a member (:247-251), for a list of groups this replica leads.  Other
 * engines, and a Crossword engine before ss_engine_set_policies, give SS_ERR_INVALID_ARG.
 * Codeword locations: a Crossword engine records, per ring position, where the full T-shard codeword of the instance
 * that last entered Accepting there lives (shard 0, plane stride, data_len; 16 bytes per position, 1 KiB per group):
 * ss_engine_propose / _next its own store, ss_engine_propose_ragged shards + shard_off[g], ss_engine_prepare_absorb the
 * decided codeword's slot in that call's store (a NULL decision: the zero codeword of data_len 1).  So a Crossword host
 * that calls the fallback keeps the store of every Accepting instance alive and unmodified until the instance commits or
 * retires; hosts that never call it are unaffected.  The fallback's own output store is not recorded: the host may reuse
 * it once the Accepts are packed.  Plane strides on a Crossword engine are below 2^36 (else SS_ERR_INVALID_ARG).
 * groups (device u32 [n_listed]); peer_alive (device [G] replica masks, NULL = every one of the population alive;
 * bits past the population are ignored); policy (device u8 [G]): the index of pick_assignment_policy's result for the
 * group, which the host computes.
 * Per listed entry, in list order, every window position in slot order that is Accepting and not Committed:
 *   kept when the engine is balanced, its policy_idx < n_policies and popcount(policies[policy_idx][0]) >= min_spr,
 *     min_spr = (majority + f + 1 - alive) * (d / majority) in u8 arithmetic (adaptive.rs:98-106), alive the popcount
 *     of peer_alive[g];
 *   redone otherwise (every such instance of an unbalanced engine): inst_bal = bal_prepared[g], its bit cleared in every
 *     ack plane, policy_idx = policy[g], its full codeword copied from the recorded location into a bump-allocated
 *     SS_CW_SLOT_PITCH(shard_len) slot of every plane of the CALLER-owned store (shards + j*plane_stride, plane_stride a
 *     multiple of 32, shards 16-byte aligned, from *store_used, device u64 in/out rounded up to 32; bytes
 *     shard_len..round_up(shard_len, 16) zero), and one record appended to the decided list.
 * accepting, committed and commit_bar do not change.  A position with no recorded location (state installed through
 * the view) is kept.  A group listed twice is processed once per entry, as two reference calls would be: the second
 * entry redoes its instances again only when policy[g] is not responsive either.
 * Outputs: the decided list in the order and layout of ss_engine_prepare_absorb's (dec_slot absolute, dec_ballot,
 * dec_shard_off, dec_data_len, dec_policy (may be NULL), dec_group), which ss_frame_accept_pack_ragged_dev takes;
 * verdict[i]: SS_ACCEPT_VERDICT_ACCEPTED (applied, possibly with nothing to redo), SS_FRAME_KIND_MALFORMED (group >=
 * n_groups: nothing happens), SS_ACCEPT_VERDICT_STORE_FULL (SS_DEV_STATUS_STORE_FULL) or SS_ACCEPT_VERDICT_WAL_FULL
 * (SS_DEV_STATUS_FRAME_OVERFLOW) for an entry whose store slots end past plane_stride or whose records end past
 * dec_capacity: it changes nothing, and neither does any later entry, since the ends are monotone in list order, so
 * re-submitting the cut entries finishes the job.  totals (device u64[2], may be NULL): the records and store bytes the
 * whole list asked for.
 * After the call the host does what it does after ss_engine_prepare_absorb: ss_frame_accept_pack_ragged_dev over the
 * decided list for every peer (dead ones too, as the reference sends to them) and for itself, its own frame to its own
 * ss_acceptor_accept in the same turn, then ss_accept_reply_parse_dev, ss_engine_ingest and ss_engine_tick.  The Accepts
 * go out under bal_prepared, normally the instance's ballot already, so a late AcceptReply of the old round is still
 * credited, under the new assignment: an AcceptReply carries none.
 * Stated differences from the reference:
 *   1. the 64-slot window;
 *   2. one policy per group, not one per data_len: it differs only under the adaptive or b_to_d_threshold chooser, which
 *      is the host's;
 *   3. where (majority + f + 1 - alive) underflows u8 (more replicas alive than majority + f + 1) the threshold is 0 and
 *      every balanced instance is kept; the reference panics there (u8 overflow, or brr_assignments has no entry);
 *   4. the per-entry capacity cut;
 *   5. pending_accepts, the RTT bookkeeping and the heartbeats injected every msg_chunk_size Accepts stay with the host.
 * Cost: the walk a warp per listed entry, each lane two window positions; the copy a warp per decided record. */
int ss_engine_fallback_redo(ss_engine *engine, const uint32_t *groups, uint64_t n_listed, const uint32_t *peer_alive,
                            const uint8_t *policy, uint8_t *shards, uint64_t plane_stride, uint64_t *store_used, uint64_t *dec_slot,
                            uint64_t *dec_ballot, uint64_t *dec_shard_off, uint32_t *dec_data_len, uint8_t *dec_policy,
                            uint32_t *dec_group, uint64_t dec_capacity, uint32_t *verdict, uint64_t *totals);

/* ---- batched CRaft follower (the Raft-family counterpart of the acceptor) ----------------------------------------
 * For n_groups CRaft groups this replica follows: AppendEntries frames in (handle_msg_append_entries,
 * craft/messages.rs:14-252, with check_term, craft/leadership.rs:16-75), the entries' shards into a caller-owned store,
 * DurEntry::LogEntry and DurEntry::Metadata records and AppendEntriesReply frames out (craft/durability.rs:129-160).
 * The code is derived from the population: d = majority, p = population - majority (craft/mod.rs:527-536).
 * State lives in HBM as a struct of arrays.  Per group: start_slot, log_end, curr_term, leader (0xff = None),
 * last_commit, last_snap.  Per log position, a ring of `window` entries (slot s at s & (window - 1)): term, data_len,
 * held (shard mask) and shard_addr (device address of the first held shard in the caller's store, shards in index order
 * at SS_CW_SLOT_PITCH(shard_len) apart, the layout ss_acceptor_accept writes).  At creation every group holds the slot-0
 * null entry recovery pushes (craft/recovery.rs:99-125): start_slot 0, log_end 1, term 0, no shards.
 * Stated differences from the reference:
 *   1. the log is a ring of `window` entries, not a vector: a frame with an entry at or past start_slot + window takes no
 *      part in the call (SS_FOLLOWER_VERDICT_BEYOND_WINDOW) and is re-submitted after ss_follower_advance;
 *   2. a non-empty frame whose entries are all present with matching terms appends nothing and gets the immediate reply
 *      {curr_term, prev_slot + n, None}; the reference, with first_new left at prev_slot + 1, would push every entry
 *      again at the end of its log (messages.rs:102-182).  The reply's bytes are the same; no record is written;
 *   3. the append does not track role: the host submits frames only for the groups it follows; heard_heartbeat and the
 *      timers stay on the host; the elections keep their role beside this state (CRaft elections, below), where a
 *      same-term frame ends a candidacy as the candidate same-term hack does;
 *   4. the capacity cut is a suffix in frame order (below);
 *   5. absorbed entries (messages.rs:143-154) take a region after every frame's region, placed in the order the group
 *      walks reach them; one that does not fit keeps the shards it held (SS_DEV_STATUS_STORE_FULL). */
typedef struct ss_follower ss_follower;
typedef struct ss_follower_config {
    uint32_t protocol;          /* SS_PROTO_CRAFT (the field leaves room for plain Raft without an ABI change) */
    uint32_t population;        /* replicas, 1..32 */
    uint32_t me;                /* this replica's id: a frame from `me` is malformed */
    uint32_t window;            /* ring entries per group, power of two, 2..4096 (0 = 64) */
    uint32_t append_variant;    /* index of AppendEntries in PeerMsg (0), < 2^16 */
    uint32_t reply_variant;     /* index of AppendEntriesReply in PeerMsg (1), < 251: a reply fills at most 47 bytes of
                                   its 48-byte cell */
    uint32_t meta_variant;      /* index of Metadata in DurEntry (0), < 2^16 */
    uint32_t log_variant;       /* index of LogEntry in DurEntry (1), < 2^16 */
} ss_follower_config;
typedef struct ss_follower_view {
    uint64_t n_groups;
    uint32_t protocol, population, me, data_shards, total_shards, window;
    uint64_t *start_slot, *log_end, *curr_term, *last_commit, *last_snap;   /* [G] */
    uint8_t *leader;            /* [G] 0xff = None */
    uint64_t *term;             /* [G*window] */
    uint64_t *shard_addr;       /* [G*window] */
    uint32_t *held;             /* [G*window] */
    uint32_t *data_len;         /* [G*window] */
} ss_follower_view;
/* Configuration checks first (SS_ERR_INVALID_ARG, including protocol != SS_PROTO_CRAFT); a NULL ctx then gives
 * SS_ERR_NO_DEVICE when the machine has no usable device, SS_ERR_INVALID_ARG otherwise. */
int ss_follower_create(ss_ctx *ctx, const ss_follower_config *cfg, uint64_t n_groups, ss_follower **out);
int ss_follower_destroy(ss_follower *follower);
int ss_follower_view_get(ss_follower *follower, ss_follower_view *view);
/* the snapshot's start_slot move (craft/snapshot.rs:130-198): upto (device [G] absolute slots) -- start_slot moves by
 * k = clamp(upto - start_slot, 0, last_commit - start_slot), so never past last_commit.  A host that executes behind
 * last_commit passes last_exec (ss_follower_exec_view) through upto, so that no entry leaves before it executes. */
int ss_follower_advance(ss_follower *follower, const uint64_t *upto);
typedef struct ss_follower_exec_view {
    uint64_t n_groups;
    uint64_t *last_exec;        /* [G] the last executed slot; 0 at creation (the slot-0 null entry) */
} ss_follower_exec_view;
int ss_follower_exec_view_get(ss_follower *follower, ss_follower_exec_view *view);
/* Execution of the committed entries, the walk of handle_msg_append_entries (craft/messages.rs:198-240): for every
 * group, from max(last_exec + 1, start_slot) while the slot is at most last_commit, an entry holding fewer than d shards
 * stops the walk (the commit walk never passes one, but state installed through the view may hold one); an entry with
 * data_len == 0 is a null codeword get_data refuses (rscoding.rs:581-583): it does not execute and its group's walk
 * stops there (SS_DEV_STATUS_EXEC_NULL); any other executes and last_exec moves to it.  Its payload is get_data's
 * output, the first data_len bytes of data shards 0..d-1 concatenated (rscoding.rs:581-683): a held data shard is read
 * at shard_addr + rank * SS_CW_SLOT_PITCH(shard_len) (rank among the held shards, the store layout of
 * ss_follower_append), a missing one is regenerated from the first d held shards in index order, as reconstruct_data
 * chooses them (rscoding.rs:490-537).  The caller's stores must still hold the shards.
 * Outputs, records, capacities, totals and status bits are those of ss_acceptor_execute: executed entries ordered by
 * (group, slot), record k = rec_group[k], rec_slot[k] (absolute), rec_off[k], rec_len[k] (= data_len); the payload at
 * out + rec_off[k] in a region of round_up(data_len, 16) bytes, zero past data_len, placed by exclusive scans (out
 * 16-byte aligned); totals (device u64[2], may be NULL): records and bytes the walk asked for; an entry whose record
 * index reaches rec_capacity or whose region ends past out_capacity does not execute and its group's walk stops there
 * (SS_DEV_STATUS_EXEC_FULL).  The records written are a prefix; a host drains by calling again. */
int ss_follower_execute(ss_follower *follower, uint8_t *out, uint64_t out_capacity, uint32_t *rec_group, uint64_t *rec_slot,
                        uint64_t *rec_off, uint32_t *rec_len, uint64_t rec_capacity, uint64_t *totals);
/* Verdicts of ss_follower_append, beside the PeerMsg variant index k (another message; 0x80000000 | k for the
 * PeerMessage variants) and SS_FRAME_KIND_MALFORMED */
#define SS_FOLLOWER_VERDICT_ACCEPTED 0xfffffff0u      /* log matched: appended, absorbed or found its entries present */
#define SS_FOLLOWER_VERDICT_REJECTED 0xfffffff1u      /* conflict reply sent, nothing appended */
#define SS_FOLLOWER_VERDICT_BEYOND_WINDOW 0xfffffff3u /* an entry at or past start_slot + window: re-submit after advance */
#define SS_FOLLOWER_VERDICT_STORE_FULL 0xfffffff4u    /* cut by the store capacity (below) */
#define SS_FOLLOWER_VERDICT_WAL_FULL 0xfffffff5u      /* cut by the WAL capacity (below) */
/* One batch of frames, taken as ss_acceptor_accept takes them: buf at any byte alignment, frame i at frame_off[i], of
 * group frame_group[i] (>= n_groups: malformed), from replica frame_peer[i].  Frame i is PeerMessage::Msg{AppendEntries
 * {term, prev_slot, prev_term, entries: Vec<LogEntry{term, reqs_cw, external, log_offset}>, leader_commit, last_snap}}.
 * Malformed: truncated, trailing bytes, a variant >= 2^16, a codeword that is not this code, shard_len !=
 * ceil(data_len / d), data_len >= 2^32, a present shard of another length, data_copy other than None, external not 0/1,
 * a body over 2^32 - 65 bytes, or a frame from `me` or from a peer >= population.
 * Each group's frames are replayed in frame order as if they arrived one at a time:
 *   term check: term > curr_term raises curr_term (voted_for None) and sets leader; that frame gets
 *     DurEntry::Metadata{curr_term, voted_for: 255} in the 32-byte cell meta + 32*i (meta_len[i] bytes: 8-byte
 *     big-endian length, meta_variant, curr_term, 0xff; zero to the end of the cell; 0 = no record), which the host makes
 *     durable before any other action of the frame.  A frame with term >= curr_term sets leader = frame_peer.
 *   rejection: term < curr_term, prev_slot outside [start_slot, log_end) or term[prev_slot] != prev_term (also for an
 *     empty frame): reply {curr_term, prev_slot + n, Some((conflict_term, conflict_slot))} with messages.rs:52-69's walk
 *     back over the ring, to frame_peer, sent at once.
 *   acceptance: entry k at slot prev_slot + 1 + k appends when it is at or past log_end; one whose term differs from
 *     the held one truncates the log at its slot (trunc_slot[i] = that slot, else UINT64_MAX: the host applies
 *     LogAction::Truncate at the slot's file offset before the frame's records) and appends from there; a matching one
 *     absorbs the frame's shards when the held entry has fewer than d data shards, the same data_len and another shard
 *     map.  Appended entries get DurEntry::LogEntry records one after the other from wal + wal_off[i], each at a 16-byte
 *     aligned offset: 8-byte big-endian length, log_variant, the entry's bytes from term through external verbatim,
 *     log_offset as varint 0; wal_len[i] = the bytes from wal_off[i] to the end of the last one's 16-byte slot.  Their
 *     shards go one entry after the other from store + store_off[i].  A frame that appended anything gets the reply
 *     {curr_term, prev_slot + n, None} for reply_dst[i] = leader as the whole call left it, sent once its records are
 *     durable; a frame that appended nothing (wal_len 0, store_off and wal_off UINT64_MAX) gets the same bytes for
 *     frame_peer at once.  Then leader_commit > last_commit walks last_commit + 1 ..= min(leader_commit,
 *     first_new - 1, log_end - 1) and stops at an entry holding fewer than d shards, first_new being the first slot
 *     the frame appended, or prev_slot + 1 when it appended nothing: the reference's cap prev_slot + entries.len()
 *     is taken after its append loop drained entries[first_new - prev_slot - 1 ..] (messages.rs:160-203), so a frame
 *     never commits the entries it appends itself.  last_snap = max(last_snap, the frame's).  A rejected frame also
 *     raises last_snap.
 * Replies: PeerMessage::Msg{AppendEntriesReply} in the 48-byte cell replies + 48*i, reply_len[i] bytes (0 = none),
 * reply_dst[i] (0xff = none).  commit_lo (device [G], may be NULL): each group's last_commit before the call.
 * Capacity: every frame that reaches the replay reserves, before it, a store region of the popcount(held) *
 * SS_CW_SLOT_PITCH(shard_len) of all its entries and a WAL region of all its entries' 16-byte record slots, placed by
 * exclusive scans in frame order.  The first frame in frame order whose region ends past store_capacity or
 * wal_capacity, and every later frame that would reach the replay, is cut: STORE_FULL or WAL_FULL (the first frame's
 * reason), nothing changes, SS_DEV_STATUS_STORE_FULL / SS_DEV_STATUS_FRAME_OVERFLOW.  The handled frames are then a
 * prefix in frame order and, within each group, a prefix of its frames; the host re-submits the rest.
 * totals (device u64[2], may be NULL): the store bytes (regions and absorbs) and WAL bytes the batch asked for.
 * Non-handled frames get UINT64_MAX offsets and zero lengths.  store and wal 16-byte aligned.
 * Cost: the replay walks each group's frames on one thread, so a batch costs its largest per-group run of frames there
 * (a follower catching up on one group replays serially); absorbs are copied by that thread too.  The records and
 * shards take a warp per frame. */
int ss_follower_append(ss_follower *follower, const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off,
                       const uint32_t *frame_group, const uint8_t *frame_peer, uint64_t n_frames, uint8_t *store,
                       uint64_t store_capacity, uint64_t *store_off, uint8_t *wal, uint64_t wal_capacity, uint64_t *wal_off,
                       uint64_t *wal_len, uint8_t *meta, uint32_t *meta_len, uint8_t *replies, uint32_t *reply_len,
                       uint8_t *reply_dst, uint64_t *trunc_slot, uint32_t *verdict, uint64_t *commit_lo, uint64_t *totals);
/* The leader's side: AppendEntriesReply frames (buf, frame_off, frame_group, frame_peer as above; frame_peer is the
 * peer index ss_engine_raft_ingest takes) -> records in its layout: rec_group, rec_peer, rec_end_slot.  curr_term is the
 * CRaft engine's [G] array (ss_engine_view.curr_term).  rec_kind: SS_APPEND_REPLY_INGEST for a success reply whose term
 * is at most curr_term[g] and end_slot < 2^32; SS_APPEND_REPLY_HIGHER_TERM (check_term makes the leader step down and
 * drop the reply, messages.rs:272-274), _CONFLICT (the next_slot back-off stays with the host), _END_RANGE; another
 * message's variant index (0x80000000 | k for PeerMessage variants) or SS_FRAME_KIND_MALFORMED (also a group >=
 * n_groups).  Every record but INGEST gets rec_group UINT32_MAX, which the ingest drops.  rec_term, rec_conflict_term and
 * rec_conflict_slot hold the decoded fields of a frame of one of the four kinds above (the conflict ones 0 for a
 * success reply); every field is 0 for another message or a malformed frame.  reply_variant < 2^16 (SS_ERR_INVALID_ARG
 * otherwise, before any other check), as for ss_engine_craft_backoff. */
#define SS_APPEND_REPLY_INGEST 0xfffffff0u
#define SS_APPEND_REPLY_CONFLICT 0xfffffff1u
#define SS_APPEND_REPLY_HIGHER_TERM 0xfffffff2u
#define SS_APPEND_REPLY_END_RANGE 0xfffffff3u
int ss_append_reply_parse_dev(ss_ctx *ctx, const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off, const uint32_t *frame_group,
                              const uint8_t *frame_peer, const uint32_t *curr_term, uint64_t n_frames, uint64_t n_groups,
                              uint32_t reply_variant, uint32_t *rec_group, uint8_t *rec_peer, uint32_t *rec_end_slot,
                              uint64_t *rec_term, uint64_t *rec_conflict_term, uint64_t *rec_conflict_slot, uint32_t *rec_kind);

/* ---- the CRaft leader's log (SS_PROTO_CRAFT engines; every other protocol gets SS_ERR_INVALID_ARG) ----------------
 * The leader half of the loop the follower above closes: request batches coded into the leader's log
 * (handle_req_batch, craft/request.rs:70-116), AppendEntries frames out (handle_logged_leader_append,
 * craft/durability.rs:12-127, and bcast_heartbeats, craft/leadership.rs:249-279), conflict replies backed off on the device
 * (handle_msg_append_entries_reply's conflict branch, craft/messages.rs:386-406).  The code is (d, p) = (majority,
 * population - majority) (craft/mod.rs:527-536), so population >= 3.
 * Peer indexing: the engine's match / next_slot / try_next rows are the population - 1 peers with `me` excluded
 * (raft/mod.rs:560-562): peer index q <-> replica q < me ? q : q + 1.  The same index is the frame_peer of
 * ss_append_reply_parse_dev and the rec_peer of ss_engine_raft_ingest.
 * State, allocated when the log is first used: log_start [G]; try_next [P][G]; per position of the engine's raft_window
 * ring (slot s at s & (W - 1)): data_len, shard_addr (shard j of the entry at shard_addr + j * plane_stride, 16-byte
 * aligned) and log_offset.  Entry terms are the engine's `terms` ring: while the log is in use every slot of
 * [log_start, log_end) stays in the ring.  Slot 0 is the null entry (data_len 0, term 0).
 * Taking the log into use: ss_engine_craft_log_view_get or any call below.  From then on ss_engine_raft_append returns
 * SS_ERR_INVALID_ARG (an entry without a codeword cannot be sent); once ss_engine_raft_append has run, the calls below
 * return SS_ERR_INVALID_ARG.  An engine that never uses the log behaves as before.
 * Stated differences from the reference:
 *   1. try_next is kept apart from the success-reply ingest: every pack first takes try = max(try_next, next_slot), which
 *      is the reference's try_next_slot = max(try_next_slot, end_slot + 1) of messages.rs:281-283 applied lazily;
 *   2. within one batch of replies, success replies (ss_engine_raft_ingest) are applied before conflicts, and a pair's
 *      several conflicts are walked in frame order but answered by one resend, [next_slot, the last one's end_slot];
 *      when the last one finds next_slot == 1 the pair gets no resend at all (want_end UINT64_MAX), where the reference
 *      would already have resent for the earlier ones -- the next pack from try_next = 1 sends the log from slot 1;
 *   3. the log is a ring of raft_window entries: a proposal that would hold more than raft_window slots of
 *      [log_start, log_end] is refused (SS_DEV_STATUS_RAFT_WINDOW_FULL);
 *   4. a prev_slot below log_start is not an error but pair status SS_APPEND_PAIR_SNAPSHOTTED;
 *   5. switch_assignment_mode (craft/leadership.rs:282-288) is split: the full_copy flag of ss_engine_craft_propose and
 *      ss_frame_append_pack_dev chooses which shards a record or frame carries, ss_engine_craft_set_full_copy the commit
 *      threshold; the detection (population - alive >= fault_tolerance) and the resend of the entries already sent
 *      with one shard (left commented out at leadership.rs:100-135; a host rewinds try_next through the log view) stay
 *      with the host. */
typedef struct ss_engine_craft_log_view {
    uint64_t n_groups;
    uint32_t population, raft_window, data_shards, total_shards;
    uint64_t plane_stride;      /* of every ss_engine_craft_propose so far (0: none yet) */
    uint64_t *log_start;        /* [G] the reference's start_slot */
    uint32_t *try_next;         /* [P][G] try_next_slot */
    uint32_t *data_len;         /* [G][raft_window] */
    uint64_t *shard_addr;       /* [G][raft_window] device address of shard 0's slot */
    uint64_t *log_offset;       /* [G][raft_window] the entry's offset in the leader's log file: the host may rewrite it
                                   once the entry's write has landed (durability.rs:181-186); the packer sends what is there */
} ss_engine_craft_log_view;
int ss_engine_craft_log_view_get(ss_engine *engine, ss_engine_craft_log_view *view);
/* handle_req_batch for every group g with data_len[g] > 0: one entry at log_end[g] in curr_term[g] (terms ring and log_end
 * written as ss_engine_raft_append does).  The batch arena[data_off[g] .. + data_len[g]) is coded with d = majority,
 * p = population - majority by one launch of the ragged encoder (SS_RS_OUT_PADDED16 | SS_RS_EMIT_DATA): shard j goes to
 * the caller-owned plane shards + j * plane_stride at shard_off[g], SS_CW_SLOT_PITCH(ceil(data_len / d)) bytes per group,
 * placed by an exclusive scan in group order; *need (device, may be NULL) = the total pitch.  The entry records
 * shard_addr = shards + shard_off[g] and log_offset[g] (device [G], NULL = 0).  plane_stride: a multiple of 32, the same
 * on every call; shards and wal 16-byte aligned.  The caller may rotate several stores: a store must outlive its entries
 * until ss_engine_craft_advance retires them.
 * The leader's own DurEntry::LogEntry record{term, reqs_cw: shard `me` (shards 0..majority when full_copy), external:
 * true, log_offset: 0} (request.rs:79-104) goes to wal + wal_off[g], its 16-byte-aligned region placed by an exclusive
 * scan in group order: 8-byte big-endian length, DurEntry variant 1, the entry; wal_len[g] = its length.
 * Refusals leave the group unchanged: slot_out, shard_off and wal_off UINT64_MAX, wal_len 0:
 *   log_end + 1 - log_start > raft_window   SS_DEV_STATUS_RAFT_WINDOW_FULL (no room taken)
 *   a slot past plane_stride               SS_DEV_STATUS_STORE_FULL
 *   a record region past wal_capacity      SS_DEV_STATUS_FRAME_OVERFLOW
 * The offsets are monotone, so the groups that propose are a prefix of those that fit the window.  Groups with
 * data_len 0 get the same UINT64_MAX outputs and no status bit.  No host synchronisation. */
int ss_engine_craft_propose(ss_engine *engine, uint32_t me, const uint8_t *arena, const uint64_t *data_off, const uint32_t *data_len,
                            uint8_t *shards, uint64_t plane_stride, uint64_t *shard_off, uint64_t *slot_out, uint64_t *need,
                            const uint64_t *log_offset, uint8_t *wal, uint64_t wal_capacity, uint64_t *wal_off, uint64_t *wal_len,
                            int full_copy);
/* the snapshot's start_slot move (craft/snapshot.rs:142,184): log_start moves by clamp(upto - log_start, 0,
 * min(last_snap, last_commit) - log_start); upto is device [G].  A host that executes behind last_commit passes its
 * last_exec (ss_engine_craft_exec_view) through upto, so that no entry leaves before it executes. */
int ss_engine_craft_advance(ss_engine *engine, const uint64_t *upto);
/* The commit threshold of ss_engine_tick, the commit half of switch_assignment_mode (craft/leadership.rs:282-288):
 * non-zero sets it to majority, as a leader in full-copy mode commits (craft/messages.rs:300-310), zero restores
 * majority + fault_tolerance.  ss_engine_view.threshold reports it; the next tick uses it.  SS_PROTO_CRAFT engines only
 * (SS_ERR_INVALID_ARG otherwise), whether or not the log is in use; it writes no device state. */
int ss_engine_craft_set_full_copy(ss_engine *engine, int full_copy);
typedef struct ss_engine_craft_exec_view {
    uint64_t n_groups;
    uint64_t *last_exec;        /* [G] the last executed slot; 0 when the log is taken into use (the slot-0 null entry) */
} ss_engine_craft_exec_view;
int ss_engine_craft_exec_view_get(ss_engine *engine, ss_engine_craft_exec_view *view);
/* Execution on the leader, the execution half of handle_msg_append_entries_reply's success branch
 * (craft/messages.rs:316-359): for every group, from max(last_exec + 1, log_start) while the slot is at most
 * last_commit, an entry with data_len == 0 is a null codeword get_data refuses (rscoding.rs:581-583): it does not
 * execute and its group's walk stops there (SS_DEV_STATUS_EXEC_NULL); any other executes and last_exec moves to it.
 * An entry holding fewer than d shards (one a step-up took over and no absorb has completed; ss_engine_craft_recon_view)
 * stops the walk with no status bit, as in ss_follower_execute: ss_engine_craft_reconstruct_reads lists it.  The payload
 * is get_data's output, the first data_len bytes of data shards 0..d-1 concatenated (rscoding.rs:581-683), read at
 * shard_addr + j * plane_stride; a missing data shard is regenerated from the first d held shards in index order, as
 * reconstruct_data chooses them (rscoding.rs:490-537).  The planes of ss_engine_craft_propose and ss_engine_craft_step_up
 * must still hold the entries.  Outputs, records, capacities, totals and status bits are those of ss_acceptor_execute (see
 * ss_follower_execute).  Takes the log into use, and is refused once ss_engine_raft_append has run. */
int ss_engine_craft_execute(ss_engine *engine, uint8_t *out, uint64_t out_capacity, uint32_t *rec_group, uint64_t *rec_slot,
                            uint64_t *rec_off, uint32_t *rec_len, uint64_t rec_capacity, uint64_t *totals);
typedef struct ss_append_pack_spec {
    uint32_t me;                /* the leader's replica id, < population */
    uint32_t append_variant;    /* index of AppendEntries in PeerMsg (0), < 2^16 */
    uint32_t msg_chunk_size;    /* entries per frame, >= 1 (the reference's default is 10, mod.rs:101) */
    uint32_t full_copy;         /* non-zero: every entry carries shards 0..majority instead of the peer's own */
    uint32_t heartbeat;         /* non-zero: one empty frame per pair (bcast_heartbeats) */
    uint32_t pad0;
} ss_append_pack_spec;
/* pair_status[q * G + g] */
#define SS_APPEND_PAIR_SENT 0u          /* frames written */
#define SS_APPEND_PAIR_NOTHING 1u       /* nothing to send */
#define SS_APPEND_PAIR_SNAPSHOTTED 2u   /* prev_slot < log_start: the reference errs ("snapshotted slot queried") */
#define SS_APPEND_PAIR_OVERFLOW 3u      /* cut by out_capacity or max_frames: nothing written, try_next unchanged */
#define SS_APPEND_PAIR_NOT_LEADER 4u    /* the engine does not lead the group (ss_engine_craft_role_view): nothing written,
                                           try_next unchanged */
/* AppendEntries frames for every (peer q, group g), after try = max(try_next, next_slot):
 *   entries (heartbeat == 0): end = want_end ? min(want_end[q*G + g], log_end - 1) : log_end - 1 (want_end device
 *     [P][G], may be NULL; UINT64_MAX: NOTHING for that pair).  try < 1 or prev_slot = try - 1 >= log_end: NOTHING;
 *     prev_slot < log_start: SNAPSHOTTED; end >= try: the entries [try, end] go out in frames of msg_chunk_size entries
 *     and try_next = end + 1 (durability.rs:60-125); otherwise NOTHING.
 *   heartbeat: one empty frame with prev_slot = min(try - 1, log_end - 1) (SNAPSHOTTED below log_start); want_end is
 *     not read.
 * Every pair not cut leaves try_next = try or, when entries went out, end + 1.
 * Frame bytes: PeerMessage::Msg{AppendEntries{term: curr_term, prev_slot, prev_term: term of prev_slot, entries,
 * leader_commit: last_commit, last_snap}} behind its 8-byte big-endian length; each entry LogEntry{term, reqs_cw:
 * RSCodeword holding replica(q)'s shard (shards 0..majority when full_copy), data_copy None, external: false,
 * log_offset} -- the bytes ss_follower_append takes.
 * Placement: frame k at out + frame_off[k], frame_len[k] bytes, in its own 16-byte-aligned region (the bytes from
 * frame_len to the region's end are not written), regions back to back in (peer, group, chunk) order, so each peer's
 * frames are contiguous; frame_group[k] = g, frame_peer[k] = q.  A pair whose region ends past out_capacity or whose
 * frames end past max_frames is not written: OVERFLOW, SS_DEV_STATUS_FRAME_OVERFLOW.  The offsets are monotone, so the
 * written pairs are a prefix of those with frames.  *n_frames (device) = the frames written; entries from there on are
 * not written.  *total (device, may be NULL) = the bytes every pair with frames asked for.  out 16-byte aligned.
 * Cost: a warp per pair plans and places (lanes over its frames), a warp per frame writes it. */
int ss_frame_append_pack_dev(ss_engine *engine, const ss_append_pack_spec *spec, const uint64_t *want_end, uint8_t *out,
                             uint64_t out_capacity, uint64_t *frame_off, uint64_t *frame_len, uint32_t *frame_group, uint8_t *frame_peer,
                             uint64_t max_frames, uint64_t *n_frames, uint32_t *pair_status, uint64_t *total);
/* The conflict branch for the reply frames of one ss_append_reply_parse_dev call (the same buf, frame_off, frame_group,
 * frame_peer, its rec_kind and reply_variant): each SS_APPEND_REPLY_CONFLICT frame's end_slot and (conflict_term,
 * conflict_slot) are decoded again, and each pair's conflicts are applied in frame order: next_slot == 1 -> try_next = 1,
 * no resend; otherwise next_slot - 1, then down while next_slot > log_start, term[next_slot] == conflict_term,
 * next_slot >= conflict_slot and next_slot > 1; try_next = next_slot; want_end[q*G + g] = end_slot.  Pairs without a
 * conflict get want_end UINT64_MAX.  The resend is ss_frame_append_pack_dev(..., want_end, ...); a walk that stops at
 * log_start makes that pack report SNAPSHOTTED for the pair.  (population - 1) * n_groups < 2^32 - 1. */
int ss_engine_craft_backoff(ss_engine *engine, const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off,
                            const uint32_t *frame_group, const uint8_t *frame_peer, const uint32_t *rec_kind, uint64_t n_frames,
                            uint32_t reply_variant, uint64_t *want_end);

/* ---- CRaft leader fail-over: step-up and reconstruct reads (SS_PROTO_CRAFT engines) ------------------------------------
 * A new leader's log comes from this replica's follower (ss_engine_craft_step_up, the log half of become_the_leader,
 * craft/leadership.rs:212-246).  In 1-shard mode a follower holds one shard of most entries, so the leader then lists the
 * committed entries it holds fewer than d = majority shards of (ss_engine_craft_reconstruct_reads, craft/messages.rs:316-371),
 * the followers serve them (ss_follower_reconstruct_serve, messages.rs:621-662), the leader absorbs the replies
 * (ss_engine_craft_absorb, messages.rs:664-744 without its execution loop) and ss_engine_craft_execute runs what now holds
 * d shards, regenerating missing data shards.
 * Two more arrays of the leader's log: held ([G][raft_window] shard masks; ss_engine_craft_propose writes every shard's bit,
 * step-up the follower's mask) and last_recon ([G], the reference's last_recon, mod.rs:345-347; zero when the log is taken
 * into use, left alone by step-up: the reference keeps it across roles).  An entry's AppendEntries carries held & wanted
 * (subset_copy, rscoding.rs:255-293): a shard the leader does not hold goes out as None.  A log that is never stepped up
 * holds every shard of every entry and behaves as before.
 * Stated differences from the reference:
 *   1. heartbeats and the `external` flag of unreplied entries (leadership.rs:236-243) stay with the host; step-down
 *      (engine -> follower) is ss_engine_craft_step_down and elections run on the follower (ss_follower_campaign /
 *      _vote / _tally), both below;
 *   2. the packer's leader_commit is the engine's last_commit, the quorum commit point; the reference sends its executed
 *      prefix, which lags behind while reconstruct reads are outstanding;
 *   3. execution after an absorb goes up to the tick's last_commit, which keeps the current-term rule; the reference's loop
 *      runs to shadow_last_commit (the k-th match, no term check; messages.rs:673-686), which ss_raft_kth_match_dev gives a
 *      host that wants it;
 *   4. served codewords carry the held shards only; a reference follower that executed also sends regenerated data
 *      shards and data_copy;
 *   5. absorb ignores slots at or past log_end, where the reference would index past its vector;
 *   6. an entry failing absorb_other's checks is rejected alone; in the reference it aborts the rest of the message, in
 *      HashMap order. */
typedef struct ss_engine_craft_recon_view {
    uint64_t n_groups;
    uint32_t raft_window, total_shards;
    uint32_t *held;             /* [G][raft_window] shard masks */
    uint64_t *last_recon;       /* [G] the last slot a reconstruct read listed */
} ss_engine_craft_recon_view;
/* Takes the log into use.  The held masks are kept from the first call of this view, step-up, reconstruct reads or
 * absorb on (every mask starts full: only ss_engine_craft_propose made entries until then); before that propose does not
 * write them and pack and execute do not read them. */
int ss_engine_craft_recon_view_get(ss_engine *engine, ss_engine_craft_recon_view *view);
/* verdict[i] of ss_engine_craft_step_up; every one but DONE leaves the group unchanged */
#define SS_STEPUP_VERDICT_DONE 0u
#define SS_STEPUP_VERDICT_IGNORED 1u      /* group >= n_groups, or listed earlier in the same call */
#define SS_STEPUP_VERDICT_WINDOW 2u       /* the follower's log_end - start_slot > raft_window */
#define SS_STEPUP_VERDICT_RANGE 3u        /* log_end, last_snap, a ring term or term[i] >= 2^32 (the engine's arrays are u32) */
#define SS_STEPUP_VERDICT_STALE_TERM 4u   /* term[i] < the follower's curr_term */
#define SS_STEPUP_VERDICT_STORE_FULL 5u   /* the group's slots end past plane_stride (SS_DEV_STATUS_STORE_FULL) */
/* Step-up for the listed groups (device u32 [n_listed]; a group >= n_groups, or one listed before in the call, is
 * ignored), each in term[i] (device u64 [n_listed], the term the host's election won), from `follower`, this replica's
 * follower (same context, population, n_groups and protocol; SS_ERR_INVALID_ARG otherwise, and for an engine that ran
 * ss_engine_raft_append).  The verdicts above are checked in that order.  For a stepped-up group g:
 *   - [start_slot, log_end) of the follower's ring goes into the engine's: terms, data_len, held, log_offset 0;
 *   - every non-null entry gets a SS_CW_SLOT_PITCH(ceil(data_len / d)) slot in every plane shards + j * plane_stride,
 *     the slots placed in (listing, slot) order by an exclusive scan (shard_off[i]: listing i's first slot, UINT64_MAX
 *     when not stepped up; *need, device, may be NULL: the bytes asked for).  Held shard j (rank k in the follower's
 *     store) is copied to plane j, round_up(shard_len, 16) bytes; the absent ones stay reserved for an absorb;
 *   - log_start = start_slot, log_end, last_commit, last_snap and last_exec (ss_follower_exec_view) are the follower's,
 *     curr_term = term[i]; for every peer next_slot = try_next = log_end and match = 0 (leadership.rs:225-234);
 *     last_recon is left alone.  The log_offset ring is the host's to rewrite through ss_engine_craft_log_view.
 * The offsets are monotone, so the groups cut by plane_stride are a suffix of those that passed the other checks.
 * plane_stride: a non-zero multiple of 32, the same as every ss_engine_craft_propose's; shards 16-byte aligned and alive
 * while the entries are.  The follower's state is only read.
 * Cost: a thread per listing sizes and writes the state; the copies take a warp per entry, with aligned 128-bit accesses. */
int ss_engine_craft_step_up(ss_engine *engine, const ss_follower *follower, const uint32_t *groups, uint64_t n_listed,
                            const uint64_t *term, uint8_t *shards, uint64_t plane_stride, uint64_t *shard_off, uint64_t *need,
                            uint32_t *verdict);
/* Reconstruct reads: for each listed group (groups device u32 [n_listed], NULL = every group in index order; a group >=
 * n_groups is ignored, one listed twice is planned twice from the state before the call), the slots s from
 * max(last_exec + 1, log_start, last_recon + 1) through last_commit whose entry holds fewer than d shards are listed as
 * (s, term); then last_recon = the last slot listed.  The list is cut into frames of chunk_size (>= 1) entries: 8-byte
 * big-endian length + PeerMessage::Msg{Reconstruct{slots: Vec<(usize, Term)>}} (reconstruct_variant, 4; mod.rs:239-246),
 * each with frame_dst 0xff: the host broadcasts it.  Outputs, placement, totals and the per-group capacity cut are those of
 * ss_acceptor_step_up_reads; a cut group keeps its last_recon.  Cost: a thread per listed group. */
int ss_engine_craft_reconstruct_reads(ss_engine *engine, const uint32_t *groups, uint64_t n_listed, uint64_t chunk_size,
                                      uint32_t reconstruct_variant, uint8_t *out, uint64_t out_capacity, uint32_t *frame_group,
                                      uint8_t *frame_dst, uint64_t *frame_off, uint32_t *frame_len, uint64_t frame_capacity,
                                      uint64_t *totals);
/* Serve on the follower: frame i (taken as by ss_follower_append) is PeerMessage::Msg{Reconstruct{slots: Vec<(usize,
 * Term)>}}.  A listed (slot, term) is skipped when the slot is outside [start_slot, log_end) or the ring's term differs;
 * otherwise the entry is the held shards as an RSCodeword (d, p, data_len, shard_len, T shard Options, data_copy None).
 * A (slot, term) listed again is one entry; entries follow their first occurrence.  The reply is
 * PeerMessage::Msg{ReconstructReply{slots_data: HashMap<usize, RSCodeword>}} (reply_variant, 5) for frame_peer[i]; an
 * empty map gets no reply.  Verdicts, outputs, placement, the out_capacity cut and *total are those of
 * ss_acceptor_reconstruct_serve.  Follower state is not changed.  Cost: a thread per frame sizes, a warp per reply writes;
 * a frame of k entries takes O(k^2) decode steps for the repeat check. */
int ss_follower_reconstruct_serve(ss_follower *follower, const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off,
                                  const uint32_t *frame_group, const uint8_t *frame_peer, uint64_t n_frames,
                                  uint32_t reconstruct_variant, uint32_t reply_variant, uint8_t *out, uint64_t out_capacity,
                                  uint64_t *reply_off, uint64_t *reply_len, uint32_t *verdict, uint64_t *total);
/* Absorb on the leader: frame i is PeerMessage::Msg{ReconstructReply{slots_data: HashMap<usize, RSCodeword>}}, decoded by
 * ss_acceptor_absorb's rules (this d and p, shard_len = ceil(data_len / d), exactly T shard Options each present one
 * shard_len bytes, data_copy None or Some followed by exactly data_len bytes); a frame that does not decode so is
 * malformed (also a group >= n_groups) and absorbs nothing.  A key repeated in a frame keeps its last value.  Entries are
 * taken in frame order, then wire order: one is ignored when its slot is outside [log_start, log_end), the entry is null
 * or its data_len differs; otherwise each shard the entry lacks is written to its reserved plane slot (round_up(shard_len,
 * 16) bytes, the pad zero) and its held bit set, so the first carrier of a shard index wins (absorb_other,
 * rscoding.rs:296-343).  No store capacity is needed: step-up reserved every slot.  absorbed[i] = the entries of frame i
 * that added shards; verdict[i]: SS_ACCEPT_VERDICT_ACCEPTED, another message's variant index or SS_FRAME_KIND_MALFORMED.
 * ss_engine_craft_execute runs afterwards.  Cost: a group's frames are walked by one warp, the copies take the warp. */
int ss_engine_craft_absorb(ss_engine *engine, const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off,
                           const uint32_t *frame_group, const uint8_t *frame_peer, uint64_t n_frames, uint32_t reply_variant,
                           uint32_t *absorbed, uint32_t *verdict);

/* ---- CRaft elections on the follower ---------------------------------------------------------------------------------
 * Choosing a new leader: a replica campaigns for the groups whose leader timed out (become_a_candidate,
 * craft/leadership.rs:143-209), the other replicas answer its RequestVote frames (handle_msg_request_vote,
 * craft/messages.rs:499-591) and the candidate tallies the RequestVoteReply frames (handle_msg_request_vote_reply,
 * messages.rs:593-619) into won_group / won_term, which go straight to ss_engine_craft_step_up (n_listed = n_groups).
 * The PeerMsg variant indices are arguments: RequestVote 2, RequestVoteReply 3 (mod.rs:239-246); each < 2^16.
 * State, per group, allocated on the first call below or of the view: vote_term, voted_for (0xff = None), role_term,
 * role (SS_FOLLOWER_ROLE_*) and votes (a mask by replica id).  They are read through the follower's curr_term and leader:
 *   - voted_for counts only while vote_term == curr_term;
 *   - a group is a candidate or elected only while role_term == curr_term and leader == me.
 * So ss_follower_append changes none of them, yet its check_term (a higher term: voted_for None, votes cleared, role
 * Follower) ends a vote and a candidacy, and so does a same-term AppendEntries, which sets leader to its sender (the
 * candidate same-term hack, messages.rs:33-43).
 * Stated differences from the reference:
 *   1. a campaign sets leader = me, which is how the state above knows a candidacy;
 *   2. the candidate's Metadata record is made durable before its RequestVote goes out; the reference sends first;
 *   3. a reply is counted only when the group is a candidate at curr_term, reply.term == curr_term and granted; the
 *      reference counts any reply past check_term, a refusal or a reply to an older campaign included;
 *   4. election timers, heartbeats and disallow_step_up stay with the host; a leader steps down through
 *      ss_engine_craft_step_down (below), run on each batch before these calls take it. */
#define SS_FOLLOWER_ROLE_FOLLOWER 0u
#define SS_FOLLOWER_ROLE_CANDIDATE 1u
#define SS_FOLLOWER_ROLE_ELECTED 2u
typedef struct ss_follower_vote_view {
    uint64_t n_groups;
    uint64_t *vote_term;        /* [G] the term voted_for belongs to */
    uint8_t *voted_for;         /* [G] 0xff = None */
    uint64_t *role_term;        /* [G] the term role belongs to */
    uint8_t *role;              /* [G] SS_FOLLOWER_ROLE_* */
    uint32_t *votes;            /* [G] votes granted to this replica's candidacy, bit r = replica r */
} ss_follower_vote_view;
int ss_follower_vote_view_get(ss_follower *follower, ss_follower_vote_view *view);
/* verdict[i] of ss_follower_campaign, checked in this order; every one but DONE leaves the group unchanged */
#define SS_CAMPAIGN_VERDICT_DONE 0u
#define SS_CAMPAIGN_VERDICT_IGNORED 1u        /* group >= n_groups, or listed earlier in the same call */
#define SS_CAMPAIGN_VERDICT_NOT_FOLLOWER 2u   /* already a candidate or elected at curr_term */
#define SS_CAMPAIGN_VERDICT_OTHER_LEADER 3u   /* leader is set and is not timeout_source[i] */
#define SS_CAMPAIGN_VERDICT_RANGE 4u          /* curr_term + 1 >= 2^32: the engine's terms are u32 */
/* Campaigns for the listed groups (device u32 [n_listed]); timeout_source (device u8 [n_listed], NULL = no check) is the
 * replica whose silence started listing i.  For a DONE group: curr_term += 1, voted_for = me, votes = {me}, role
 * candidate, leader = me; DurEntry::Metadata{curr_term, voted_for: me} in the 32-byte cell meta + 32*i (meta_len[i]
 * bytes, the cell format of ss_follower_append); PeerMessage::Msg{RequestVote{term: curr_term, last_slot: log_end - 1,
 * last_term: the ring's term at last_slot}} (request_vote_variant) behind its 8-byte big-endian length in the 48-byte
 * cell frames + 48*i (frame_len[i] bytes, frame_dst[i] = 0xff: the same bytes go to every peer).  The host makes the
 * record durable, then broadcasts the frame.  Other listings: meta_len and frame_len 0, frame_dst 0xff, cells not
 * written.  Cells are zero past their length.  Cost: a sort of the listings and a thread per listing. */
int ss_follower_campaign(ss_follower *follower, const uint32_t *groups, uint64_t n_listed, const uint8_t *timeout_source,
                         uint32_t request_vote_variant, uint8_t *meta, uint32_t *meta_len, uint8_t *frames, uint32_t *frame_len,
                         uint8_t *frame_dst, uint32_t *verdict);
/* Verdicts of ss_follower_vote, beside the PeerMsg variant index k (another message; 0x80000000 | k for the
 * PeerMessage variants) and SS_FRAME_KIND_MALFORMED */
#define SS_VOTE_VERDICT_GRANTED 0xfffffff0u       /* reply {curr_term, true} */
#define SS_VOTE_VERDICT_DENIED_STALE 0xfffffff1u  /* term < curr_term: reply {curr_term, false} */
#define SS_VOTE_VERDICT_NO_REPLY 0xfffffff2u      /* voted for another candidate, or its log is behind: no reply */
/* RequestVote frames, taken as ss_follower_append takes frames: frame i is PeerMessage::Msg{RequestVote{term, last_slot,
 * last_term}} (request_vote_variant) from candidate frame_peer[i] for group frame_group[i].  Malformed: truncated,
 * trailing bytes, a variant >= 2^16, a peer that is `me` or >= population, a group >= n_groups.
 * Each group's frames are replayed in frame order:
 *   check_term: term > curr_term raises curr_term, clears the vote and sets leader = the candidate;
 *   term < curr_term: reply {curr_term, false};
 *   otherwise the vote is granted when voted_for is None or the candidate, and last_term >= the term of this log's last
 *     entry || (last_term == curr_term && last_slot + 1 >= log_end) -- the reference's test verbatim, which also grants
 *     an equal last term with a shorter log; a grant sets voted_for; a vote not granted gets no reply.
 * Outputs per frame: DurEntry::Metadata{curr_term, voted_for} as the frame left them in the 32-byte cell meta + 32*i
 * when the frame raised the term or granted (meta_len[i], 0 = none); PeerMessage::Msg{RequestVoteReply{term, granted}}
 * (reply_variant) in the 32-byte cell replies + 32*i (reply_len[i], 0 = none) for reply_dst[i] (0xff = none), sent once
 * the frame's record is durable; the verdict.  Cells are zero past their length and not written when it is 0.
 * Cost: a sort of the frames and a thread per group's run of them. */
int ss_follower_vote(ss_follower *follower, const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off,
                     const uint32_t *frame_group, const uint8_t *frame_peer, uint64_t n_frames, uint32_t request_vote_variant,
                     uint32_t reply_variant, uint8_t *meta, uint32_t *meta_len, uint8_t *replies, uint32_t *reply_len,
                     uint8_t *reply_dst, uint32_t *verdict);
/* Verdicts of ss_follower_tally, checked in this order, beside another message's variant index and
 * SS_FRAME_KIND_MALFORMED */
#define SS_TALLY_VERDICT_HIGHER_TERM 0xfffffff0u      /* term > curr_term: stepped down, Metadata{term, None} */
#define SS_TALLY_VERDICT_ELECTED_ALREADY 0xfffffff1u  /* the group is elected at curr_term: ignored */
#define SS_TALLY_VERDICT_NOT_CANDIDATE 0xfffffff2u    /* the group is not a candidate at curr_term */
#define SS_TALLY_VERDICT_STALE_TERM 0xfffffff3u       /* a reply to an older campaign */
#define SS_TALLY_VERDICT_DENIED 0xfffffff4u           /* granted == false */
#define SS_TALLY_VERDICT_DUPLICATE 0xfffffff5u        /* this peer's vote is counted already */
#define SS_TALLY_VERDICT_COUNTED 0xfffffff6u          /* counted, no majority yet */
#define SS_TALLY_VERDICT_WON 0xfffffff7u              /* counted, and the votes reach majority: role elected */
/* RequestVoteReply frames, taken as ss_follower_vote takes frames: frame i is PeerMessage::Msg{RequestVoteReply{term,
 * granted}} (reply_variant; granted a 0/1 byte, anything else malformed) from frame_peer[i].  Each group's frames are
 * replayed in frame order with the verdicts above; a HIGHER_TERM frame writes DurEntry::Metadata{term, None} into the
 * 32-byte cell meta + 32*i (meta_len[i], 0 = none) and sets leader = frame_peer[i].
 * won_group (device u32 [n_groups]): the groups this call elected and that are still elected at its end, in group
 * order, then UINT32_MAX up to n_groups; won_term (device u64 [n_groups]) their curr_term, 0 past them; *n_won (device
 * u64, may be NULL) their count.  Pass won_group / won_term to ss_engine_craft_step_up with n_listed = n_groups: it
 * ignores the UINT32_MAX entries.  Cost: a sort of the frames, a thread per group's run of them, a scan. */
int ss_follower_tally(ss_follower *follower, const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off,
                      const uint32_t *frame_group, const uint8_t *frame_peer, uint64_t n_frames, uint32_t reply_variant,
                      uint8_t *meta, uint32_t *meta_len, uint32_t *verdict, uint32_t *won_group, uint64_t *won_term,
                      uint64_t *n_won);

/* ---- CRaft WAL recovery on the follower ------------------------------------------------------------------------------
 * recover_from_wal (craft/recovery.rs:11-165) for the records a CRaft replica writes -- DurEntry::Metadata{curr_term,
 * voted_for} (the 32-byte cells of ss_follower_append, _campaign, _vote, _tally and ss_engine_craft_step_down) and
 * DurEntry::LogEntry{entry} (ss_follower_append's records, and the leader's own) -- replayed into the term, the vote,
 * the log ring and the shard store without a record crossing to the host.  A restarted replica is a follower.
 * Record i is at buf + rec_off[i] (any byte alignment) as the device writes it: an 8-byte big-endian length, then the
 * bincode DurEntry, whose variant is cfg.meta_variant (Metadata) or cfg.log_variant (LogEntry); the two must differ
 * (SS_ERR_INVALID_ARG).  Record i belongs to group rec_group[i]; a group's records are replayed in array order, which is
 * WAL order; groups are independent.  The call imposes no file layout: the host hands the Metadata record over first,
 * wherever its file keeps it.
 * Per group with records:
 *   Metadata (the first record): curr_term, leader = 0xff, vote_term = curr_term, voted_for (0xff = None; any other byte
 *     is kept as it is).  The election words are taken into use as by ss_follower_vote_view_get; the group is not a
 *     candidate afterwards, since leader != me.
 *   LogEntry k (the k-th record after it): slot start_slot + k, with the record's term, data_len and held shards, decoded
 *     by the rules ss_follower_append applies to an entry (this code, shard_len = ceil(data_len / d), present shards of
 *     that length, data_copy None, external 0 or 1, non-minimal varints); log_offset is read and ignored.  Its shards go
 *     into `store`, popcount(held) * SS_CW_SLOT_PITCH(shard_len) bytes in the padded layout ss_follower_append writes,
 *     and shard_addr names that copy.
 *   When at least one LogEntry applied: log_end = start_slot + (the LogEntry records applied), and every other ring
 *     position of the group is zeroed, so the result does not depend on what the follower held before.
 *   start_slot, last_commit, last_snap and last_exec are not changed: the host installs them from the snapshot through
 *   the views first, as recover_from_snapshot (craft/snapshot.rs:203-232) does.  A group with no records is not touched.
 * Regions are placed by an exclusive scan in (group, record) order; *total (device u64, may be NULL) = the store bytes
 * the batch asked for.  store 16-byte aligned.
 * verdict[i]:
 *   SS_FOLLOWER_VERDICT_ACCEPTED       applied;
 *   SS_FRAME_KIND_MALFORMED            the length runs past buf_len, trailing bytes, a variant that is neither of the two,
 *                                      an entry that fails the rules above, a Metadata record that is not first or a
 *                                      second one, or a group >= n_groups.  For a valid group the group's log ends
 *                                      there: every later record of the group gets SS_RECOVER_VERDICT_AFTER_END;
 *   SS_FOLLOWER_VERDICT_BEYOND_WINDOW  the group's log holds more than `window` LogEntry records: the whole group is
 *                                      refused, every record of it gets this verdict, nothing of it changes and
 *                                      SS_DEV_STATUS_FRAME_OVERFLOW is set; the host needs a follower with a larger
 *                                      window;
 *   SS_FOLLOWER_VERDICT_STORE_FULL     the capacity cut is per group: a group whose store region ends past
 *                                      store_capacity applies nothing, its records that would apply get STORE_FULL and
 *                                      SS_DEV_STATUS_STORE_FULL is set.  The offsets are monotone, so the placed groups
 *                                      are a prefix in group order; re-submitting the STORE_FULL records finishes the job.
 * The file never holds superseded entries: a conflicting append truncates it first (trunc_slot of ss_follower_append).
 * Absorbed shards and the shards a leader holds only in memory are never written, so they do not come back.
 * Stated differences from the reference:
 *   1. the ring: a log longer than `window` refuses the whole group (above).  A shorter log would be unsafe: a follower
 *      that lost an acknowledged entry can vote for a candidate that lacks it.  A host that discards its WAL prefix
 *      whenever it advances the follower, as take_new_snapshot does, never meets this case;
 *   2. a record that does not decode, or a misplaced Metadata record, ends the group's log; the reference aborts the
 *      replica's recovery;
 *   3. the per-group capacity cut;
 *   4. external and log_offset are not kept: the follower has no such fields, and the host keeps the file offsets;
 *   5. the snapshot state stays with the host.
 * Cost: the walk and the apply take a thread per group segment, so a batch costs its largest per-group run of records
 * there (and the apply writes the group's whole ring); the shard copies take a warp per applied LogEntry. */
int ss_follower_recover(ss_follower *follower, const uint8_t *buf, uint64_t buf_len, const uint64_t *rec_off,
                        const uint32_t *rec_group, uint64_t n_records, uint8_t *store, uint64_t store_capacity,
                        uint32_t *verdict, uint64_t *total);

/* ---- CRaft step-down: check_term for the groups a replica leads (SS_PROTO_CRAFT engines) -------------------------------
 * An engine leads the groups whose `led` byte is set.  The bytes are allocated on the first ss_engine_craft_step_down or
 * ss_engine_craft_role_view_get, every one set (until then the engine leads every group, as before); a host whose
 * replica leads only some groups clears the others through the view; ss_engine_craft_step_up sets it for the groups it
 * steps up.  For a group whose byte is clear:
 *   - ss_engine_craft_propose refuses it as it refuses a full window (shard_off, slot_out, wal_off UINT64_MAX, wal_len 0,
 *     no WAL record) and sets SS_DEV_STATUS_NOT_LEADER;
 *   - ss_frame_append_pack_dev gives its pairs SS_APPEND_PAIR_NOT_LEADER in entry and heartbeat mode: no frame, try_next
 *     unchanged;
 *   - ss_engine_craft_execute skips it (it executes on the follower now);
 *   - ss_engine_craft_reconstruct_reads lists nothing for it and keeps its last_recon.
 * Back-off, absorb, ingest and tick only touch the engine's own words; the raised curr_term keeps the tick's current-term
 * rule from committing the group.  An engine that never allocates `led` runs the same kernels as before. */
#define SS_DEV_STATUS_NOT_LEADER 128u
typedef struct ss_engine_craft_role_view {
    uint64_t n_groups;
    uint8_t *led;               /* [G] 1: this engine leads the group */
} ss_engine_craft_role_view;
int ss_engine_craft_role_view_get(ss_engine *engine, ss_engine_craft_role_view *view);
/* PeerMsg variant indices of the messages that carry a term (mod.rs:207-247), each < 2^16 */
typedef struct ss_step_down_spec {
    uint32_t append_variant;        /* AppendEntries, 0 */
    uint32_t append_reply_variant;  /* AppendEntriesReply, 1 */
    uint32_t request_vote_variant;  /* RequestVote, 2 */
    uint32_t vote_reply_variant;    /* RequestVoteReply, 3 */
} ss_step_down_spec;
/* verdict[i] of ss_engine_craft_step_down, beside SS_FRAME_KIND_MALFORMED and 0x80000000 | k (a PeerMessage variant
 * other than Msg), checked in this order */
#define SS_STEPDOWN_VERDICT_PASS 0xfffffff0u        /* hand the frame to its usual handler */
#define SS_STEPDOWN_VERDICT_RANGE 0xfffffff1u       /* a led group's term >= 2^32 (the engine's terms are u32): unchanged */
#define SS_STEPDOWN_VERDICT_STORE_FULL 0xfffffff2u  /* cut by store_capacity: the group stays led (SS_DEV_STATUS_STORE_FULL) */
#define SS_STEPDOWN_VERDICT_DEPOSED 0xfffffff3u     /* this frame stepped the group down */
/* check_term (craft/leadership.rs:16-75) of the four messages that carry a term, for a batch of incoming frames, run
 * before the batch goes to ss_follower_append, ss_follower_vote, ss_follower_tally or ss_append_reply_parse_dev.  Frames
 * are taken as ss_follower_append takes them.  `engine` and `follower` are this replica's: same context, population,
 * n_groups and protocol, and the follower's window >= the engine's raft_window (SS_ERR_INVALID_ARG otherwise).
 * Each frame is decoded by the rules of the call that takes it (AppendEntries: ss_follower_append's; RequestVote and
 * RequestVoteReply: ss_follower_vote's and _tally's; AppendEntriesReply: ss_append_reply_parse_dev's, and a frame_peer
 * that is a peer, since it becomes the follower's leader); one that does not decode is SS_FRAME_KIND_MALFORMED and deposes
 * nobody.  Every PeerMsg variant other than the four (CRaft's are Reconstruct and ReconstructReply) carries no term and
 * PASSes, whatever its index: its own handler reports an unknown one.  Each group's frames are replayed in frame order: for a led group the first frame with
 * term > the engine's curr_term (and < 2^32) deposes it (DEPOSED); its later frames, and every frame of a group that is
 * not led, PASS, as do frames with a stale or equal term.  The host drops a DEPOSED frame, as the reference does, unless
 * it is a RequestVote, which goes on to ss_follower_vote.
 * A deposed group g, on the follower:
 *   - start_slot = max(start_slot, log_start), log_end = the engine's; each slot of [start_slot, log_end) holds the
 *     engine's term, data_len and held (every shard while the engine's held masks are not in use);
 *   - last_commit, last_snap and last_exec become the max of the follower's and the engine's, so no executed entry runs
 *     again;
 *   - curr_term = max(curr_term, term); when it rises, DurEntry::Metadata{curr_term, None} goes into the 32-byte cell
 *     meta + 32*i (meta_len[i], 0 = none; the cell format of ss_follower_append); leader = frame_peer[i];
 * and on the engine: led = 0, curr_term = term, match = 0 for its peers; nothing else changes.
 * Shards: an entry the follower held already -- the same slot inside its old [start_slot, log_end), the same term,
 * data_len and held -- keeps its shard_addr (Log Matching: the same bytes).  Every other non-null entry is copied from
 * the engine's planes into store, its held shards in rank order SS_CW_SLOT_PITCH(ceil(data_len / d)) apart,
 * round_up(shard_len, 16) bytes each; the regions are placed by an exclusive scan over the DEPOSED frames in frame order
 * (store_off[i]: the frame's first byte, UINT64_MAX for the other frames; *need, device, may be NULL: the bytes asked
 * for).  The offsets are monotone, so the frames cut by store_capacity are a suffix; their groups stay led and unchanged,
 * and every term-carrying frame of a cut group after its deposing frame is STORE_FULL too, so none reaches a handler.
 * The same batch with a larger store finishes them (groups deposed already PASS).  Afterwards the follower references
 * nothing in the engine's planes.  store: 16-byte aligned.
 * Stated differences from the reference:
 *   1. check_term runs over the whole batch before the handlers, not message by message;
 *   2. the RANGE verdict;
 *   3. the capacity cut;
 *   4. the reuse rule above;
 *   5. timers and heartbeats stay with the host, as for the elections.
 * Cost: a thread per frame decodes, a thread per DEPOSED frame walks its group's span, and the copies take a warp per
 * copied entry.  Device scratch, grow-only and kept by the engine: 8 * (n_groups + 3 * n_frames + min(n_frames, n_groups)
 * * raft_window) bytes plus scan tiles (the copy list is sized for every slot of every deposed span: 512 MiB for 2^20
 * groups at raft_window 64). */
int ss_engine_craft_step_down(ss_engine *engine, ss_follower *follower, const ss_step_down_spec *spec, const uint8_t *buf,
                              uint64_t buf_len, const uint64_t *frame_off, const uint32_t *frame_group, const uint8_t *frame_peer,
                              uint64_t n_frames, uint8_t *store, uint64_t store_capacity, uint64_t *store_off, uint8_t *meta,
                              uint32_t *meta_len, uint32_t *verdict, uint64_t *need);

/* ---- tuning / introspection (bench + tests) ------------------------------------------------ */
/* Tuning knob for experiments; 0 = the defaults.
 *   bits 0-3  kernel choice / register budget: 1 = flat one-column-per-thread RS(3,2) kernel instead of the row kernel,
 *             5 = bit-plane generic kernels instead of the Horner ones, 8 = global-table Horner reconstruct instead of the
 *             shared-memory small-code kernel; 3 / 6 / 7 = 32 / 64 / 56-register builds of the row kernel (default 40)
 *   bit 4     row kernel: contiguous chunk of codewords per CTA instead of grid-stride
 *   bits 5-7  row kernel waves of CTAs per resident set: {64 (default), 1, 32, 4, 16, 256, 128, 8}; the RS(3,2) row kernel
 *             of ss_rs_reconstruct_uniform_dev reads the same bits with its own table {16 (default), 1, 32, 4, 64, 256, 128, 8}
 *   bits 8-9  cache operator of the plane stores in replicate mode: .cs (default), write-back, .cg, .wt
 *   bit 10    row kernel: fixed instead of rotating warp -> column-block assignment
 *   bit 18    the accept step (parity to local planes, up to 256 columns) on the bulk-copy kernel instead of the row kernel;
 *             bits 19-20 its resident CTAs per SM {4 (default), 2, 3, 6}, bit 21 interleaved instead of contiguous codewords
 *   ss_crossword_distribute_dev, bits 0-3: 6 / 7 = a warp takes runs of 8 / 4 codewords from a shared counter and pools the
 *             short ones into shared passes (3.3x on batches of sub-KB payloads, 1-2 % behind on mixed sizes), 4 = the
 *             general (any code) kernel also for RS(3,2) / n = 5
 *   d <= 8 codes other than RS(3,2) (horner_encode_row_kernel / horner_encode_packed_kernel):
 *   bits 0-3  1 = flat kernel; 2 / 3 / 4 = 48 / 64 / 80-register builds of the row layout (default by width)
 *   bit 11    run-time coefficient masks even when the matrix is one of the compile-time cluster codes
 *   bit 13    never / bit 14 always use the packed layout (m codewords side by side per CTA, tail columns apart)
 *   bit 15    software-pipelined packed loop also for shards that are not 16-byte aligned
 *   bit 16    small-code reconstruct kernel: two columns per lane and pass (80 registers) instead of one (64)
 *   bit 17    no run-time specialisation: codes without a compile-time table use the run-time-mask kernels */
int ss_rs_set_variant(ss_rs_coder *coder, int variant);
/* Codes without a compile-time table (anything but the cluster codes RS(2,1) RS(3,1) RS(3,2) RS(4,2) RS(4,3) RS(5,4)) with
 * d <= 8 get their row / packed encode kernels specialised at run time by NVRTC for the coder's own parity rows (once
 * per coder, on the first batched encode).  ss_rs_jit_status tells what happened; if libnvrtc is unavailable the coder
 * keeps the run-time-mask kernels.  ss_jit_selftest compiles the kernels for RS(d,p) without a GPU and returns the
 * CUBIN size (> 0) or a negative error code with the compiler log in `log`. */
const char *ss_rs_jit_status(const ss_rs_coder *coder);
long ss_jit_selftest(int data_shards, int parity_shards, char *log, size_t log_cap);
/* name of the kernel the last batch call on this coder launched (static string) */
const char *ss_rs_last_kernel(const ss_rs_coder *coder);

#ifdef __cplusplus
}
#endif
#endif /* SUMMERSET_B200_H */
