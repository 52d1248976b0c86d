// ss_internal.hpp -- shared declarations between the C-ABI layer (capi.cu) and the kernel files.
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <cstdint>
#include <cstdio>
#include <string>
#include <vector>

#include "../../include/summerset_b200.h"
#include "device_common.cuh"

namespace ssb {

// ---- error plumbing -------------------------------------------------------------------------
int set_error(int code, const char *fmt, ...);
int cuda_error(cudaError_t e, const char *what, const char *file, int line);

#define SS_CUDA(call)                                                        \
    do {                                                                     \
        cudaError_t _e = (call);                                             \
        if (_e != cudaSuccess) return ::ssb::cuda_error(_e, #call, __FILE__, __LINE__); \
    } while (0)

#define SS_TRY(call)                \
    do {                            \
        int _rc = (call);           \
        if (_rc != SS_OK) return _rc; \
    } while (0)

// ---- coefficient programs consumed by the generic (bit-plane) coding kernel --------------------
// One "program" says: read d source shards, produce n_out output shards, out_j = sum_i c[j][i]*src_i.
// splat[(j*d + i)*8 + k] = the byte gfmul(c[j][i], 1<<k) replicated into all four bytes of a word.
constexpr int kMaxD = 32;
constexpr int kMaxP = 8;
struct ProgHeader {           // 64 bytes, followed by p*d*8 uint32 splats, then p*d*8 uint32 Horner bit masks
    uint8_t n_out;
    uint8_t n_missing_data;   // how many of dst[] are data shards (they come first)
    uint8_t valid;            // 0: fewer than d shards present (nothing can be computed)
    uint8_t pad0;
    uint8_t src[kMaxD];       // source shard index per input
    uint8_t dst[kMaxP];       // destination shard index per output
    uint8_t top[kMaxP];       // highest set bit over the coefficients of output j (Horner start), 0 if all zero
    // d <= 4 fast path (transposed mask table hmT): its rows may use the XOR chain below instead of a dense row
    uint8_t topT[2];          // Horner start of hmT rows 0 and 1
    uint8_t chain1;           // 1: output 1 = (hmT row 1 applied to the sources) ^ output 0
    uint8_t pad1[9];
};
// Horner masks: hmask[(j*d + i)*8 + k] = 0xffffffff if bit k of c[j][i] is set, else 0.
static_assert(sizeof(ProgHeader) == 64, "ProgHeader must be 64 bytes");

// Compact per-pattern program of the small-code reconstruct kernel (d <= 4): 32-byte header followed by
// p rows of 8 uint4 (row j, bit k: the 0/~0 masks of the up-to-4 sources).  The whole table of 2^(d+p)
// programs is staged in shared memory when it fits.
struct FastProgHeader {
    uint8_t valid, n_out, chain1, pad0;
    uint8_t src[4];
    uint8_t dst[kMaxP];
    uint8_t top[kMaxP];
    uint8_t pad1[8];
};
static_assert(sizeof(FastProgHeader) == 32, "FastProgHeader must be 32 bytes");

}  // namespace ssb

// ---- opaque handles -------------------------------------------------------------------------
struct ss_ctx {
    int device = -1;
    cudaStream_t stream = nullptr;
    bool owns_stream = false;
    int sm_count = 0;
    uint64_t launches = 0;
    // coders / engines created on this context hold a reference; ss_ctx_destroy defers the teardown to the last of them
    std::atomic<int> live_handles{1};   // 1 = the context's own reference (ss_ctx_destroy drops it), + 1 per coder / engine
    std::atomic<bool> closing{false};
    // grow-only device scratch (scan temporaries, LUTs)
    void *scratch = nullptr;
    size_t scratch_bytes = 0;
    // host-buffer pipeline (lazily created): H2D stream, D2H stream, triple-buffered staging
    static constexpr int kStages = 3;
    cudaStream_t h2d_stream = nullptr, d2h_stream = nullptr;
    cudaEvent_t ev_h2d[kStages] = {}, ev_kernel[kStages] = {}, ev_done[kStages] = {};
    bool pipeline_ready = false;
    void *stage_in[kStages] = {};
    void *stage_out[kStages] = {};
    size_t stage_in_bytes = 0, stage_out_bytes = 0;
    // pinned host staging of the single-codeword host-slice calls (grow-only)
    void *pinned = nullptr;
    size_t pinned_bytes = 0;
    // device status word (bit 0: a step-flag wait timed out), allocated with the context
    uint32_t *dev_status = nullptr;
};

struct ss_rs_coder {
    ss_ctx *ctx = nullptr;
    int d = 0, p = 0;
    std::vector<uint8_t> matrix;      // (d+p) x d
    bool is_rs32 = false;             // matrix parity rows == {01 01 01},{0f 08 06}: hand-specialised kernel
    int variant = 0;
    const char *last_kernel = "none";
    // device tables
    void *enc_prog = nullptr;         // ProgHeader + splats for encode
    void *enc_hmT8 = nullptr;         // d <= 8: encode masks transposed, hmT8[(j*8 + k)*8 + i] (row kernel)
    uint8_t enc_top[ssb::kMaxP] = {};
    int static_code = -1;             // index of the compile-time specialised cluster code equal to this matrix, or -1      // Horner start bit of every parity row
    void *dec_progs = nullptr;        // one program per present-pattern (2^(d+p) of them), or null
    void *dec_progs_data = nullptr;   // same, data_only flavour
    void *fast_progs = nullptr;       // d <= 4: compact programs (FastProgHeader + hmT rows), all patterns
    void *fast_progs_data = nullptr;
    size_t fast_stride = 0;
    size_t prog_stride = 0;           // bytes per program
    bool batch_ok = false;            // d,p within the batched kernels' limits
    bool dec_ok = false;              // d+p small enough for the per-pattern decode table
    // run-time specialised encode kernels (jit.cu): 0 = not tried, 1 = ready, -1 = unavailable (run-time-mask kernels stay)
    int jit_state[5] = {};
    std::string jit_message;
    void *jit_library[5] = {};
    cudaKernel_t jit_kernel[5] = {};  // row<128>, row<256>, packed<aligned,pipe>, packed<unaligned,pipe>, packed<unaligned>
    std::vector<uint8_t> verify_buf;  // ss_rs_verify: recomputed parity (grow-only, reused across calls)
    std::vector<uint8_t *> verify_ptrs;
};

namespace ssb {

int ctx_bind(ss_ctx *ctx);                              // cudaSetDevice(ctx->device)
void ctx_retain(ss_ctx *ctx);                           // a handle (coder, engine) starts referring to ctx
void ctx_release(ss_ctx *ctx);                          // ... and stops; tears ctx down if it was destroyed meanwhile
int ctx_scratch(ss_ctx *ctx, size_t bytes, void **out); // grow-only scratch

// closes every kernel launch: reports a launch error, else counts the launch (ss_ctx_launch_count)
inline int launched(ss_ctx *ctx) {
    SS_CUDA(cudaGetLastError());
    ctx->launches++;
    return SS_OK;
}

// enough CTAs of per_cta items, capped at 64 per SM
inline uint32_t launch_grid(ss_ctx *ctx, uint64_t items, uint32_t per_cta) {
    uint64_t ctas = (items + per_cta - 1) / per_cta;
    const uint64_t cap = static_cast<uint64_t>(ctx->sm_count) * 8ull * 8ull;
    if (ctas > cap) ctas = cap;
    if (ctas == 0) ctas = 1;
    return static_cast<uint32_t>(ctas);
}

// zeroed on the context's stream: a cudaMemset would go to the legacy default stream, which a non-blocking context
// stream does not wait for, so it could land after the caller's first writes (window_base) or the first accept
template <typename T>
int dalloc(ss_ctx *ctx, T **p, size_t count, bool zero = true) {
    SS_CUDA(cudaMalloc(reinterpret_cast<void **>(p), count * sizeof(T) ? count * sizeof(T) : 1));
    if (zero) SS_CUDA(cudaMemsetAsync(*p, 0, count * sizeof(T), ctx->stream));
    return SS_OK;
}

// bits of a radix-sort key up to v
inline int key_bits(uint64_t v) {
    int b = 1;
    while (b < 32 && (v >> b) != 0u) ++b;
    return b;
}

// exclusive prefix sum of x[0..n) in place (engine.cu); partials: scan_tiles(n) words of device scratch; total (device,
// may be NULL) = the sum of all n values.  Deterministic: integer sums in a fixed order.
uint64_t scan_tiles(uint64_t n);
int launch_exclusive_scan_u64(ss_ctx *ctx, uint64_t *x, uint64_t n, uint64_t *partials, uint64_t *total);

// ---- kernel launchers (defined in the .cu files) ---------------------------------------------
struct EncGeom {
    // sources: payload arena
    const uint8_t *data;
    const uint64_t *data_off;   // ragged (null => uniform)
    const uint32_t *data_len;   // ragged
    uint64_t data_stride;       // uniform
    uint32_t uni_len;           // uniform
    // outputs: parity planes
    uint8_t *parity;
    uint64_t plane_stride;
    const uint64_t *par_off;    // ragged
    uint64_t shard_stride;      // uniform
    uint64_t n;
    uint32_t flags;
    uint8_t *const *plane_ptrs = nullptr;   // replicate mode: d+p explicit plane bases (local or peer memory)
    dev::FlagWait wait = {nullptr, 0, 0, 0, nullptr};   // replicate mode: flags to wait for before the tally
};

struct TallyArgs {              // optional fused tally
    const uint64_t *planes = nullptr;
    uint32_t R = 0, threshold = 0;
    uint64_t G = 0;
    uint64_t *committed = nullptr;
    uint32_t *commit_bar = nullptr;
};

int launch_rs_encode(ss_rs_coder *coder, const EncGeom &g, const TallyArgs *tally);
// index of the compile-time specialised code whose parity rows equal matrix[(d..d+p) x d], or -1
int match_static_code(int d, int p, const uint8_t *matrix);
int launch_rs_reconstruct(ss_rs_coder *coder, uint8_t *shards, uint64_t plane_stride,
                          const uint64_t *off, const uint32_t *data_len, const uint32_t *present,
                          uint64_t n, int data_only, int32_t *status, uint32_t flags);
int launch_rs_reconstruct_uniform(ss_rs_coder *coder, uint8_t *shards, uint64_t plane_stride, uint64_t shard_stride,
                                  uint32_t data_len, const uint32_t *present, uint64_t n, int data_only, int32_t *status);
int launch_tally_planes(ss_ctx *ctx, const uint64_t *planes, uint32_t R, uint64_t G, uint32_t thr,
                        uint64_t *committed, uint32_t *commit_bar);
int launch_tally_masks(ss_ctx *ctx, const void *masks, uint32_t mask_bytes, uint64_t n, uint32_t thr,
                       uint64_t *commit_bits);
int launch_ack_ingest(ss_ctx *ctx, const uint32_t *rec_group, const uint8_t *rec_slot,
                      const uint8_t *rec_peer, const uint64_t *rec_ballot, uint64_t n_records,
                      const uint64_t *bal_prepared, const uint64_t *inst_bal, const uint64_t *accepting,
                      const uint64_t *window_base /* NULL: rec_slot is the bit position itself */,
                      uint32_t R, uint64_t G, uint64_t *planes);
int launch_tally_crossword(ss_ctx *ctx, const void *masks, uint32_t mask_bytes, const uint8_t *policy_idx,
                           uint64_t n, const uint32_t *policies_host, uint32_t n_policies,
                           uint32_t n_replicas, uint32_t T, uint32_t d, uint32_t majority, uint32_t f,
                           int balanced, uint64_t *commit_bits);
int launch_raft_scan(ss_ctx *ctx, const uint32_t *match, uint32_t n_peers, uint64_t G,
                     const uint32_t *last_commit, const uint32_t *log_end, const uint32_t *curr_term,
                     const uint32_t *terms, uint32_t window, uint32_t threshold, uint32_t *new_commit,
                     uint32_t *window_overflow, uint32_t ring = 0);
// same scan over the engine's ring-indexed term store (terms[g*W + (slot & (W-1))]); new_commit may alias last_commit
int launch_raft_scan_ring(ss_ctx *ctx, const uint32_t *match, uint32_t n_peers, uint64_t G, const uint32_t *last_commit,
                          const uint32_t *log_end, const uint32_t *curr_term, const uint32_t *terms, uint32_t window,
                          uint32_t threshold, uint32_t *new_commit);
// (policy, ack set) -> commit bit table of the Crossword predicate, from DEVICE policies
int launch_crossword_lut(ss_ctx *ctx, const uint32_t *d_policies, uint32_t n_policies, uint32_t n_replicas, uint32_t T, uint32_t d,
                         uint32_t majority, uint32_t f, int balanced, uint32_t *d_lut_bits);

// run-time specialisation of the row / packed encode kernels for a coder's matrix (jit.cu)
int jit_ensure(ss_rs_coder *coder, int which);
void jit_release(ss_rs_coder *coder);

// multi-GPU step flags
int make_flag_wait(ss_ctx *ctx, const ss_step_sync *sync, dev::FlagWait *out);
int launch_flag_signal(ss_ctx *ctx, const ss_step_sync *sync);
int launch_flag_wait(ss_ctx *ctx, const dev::FlagWait &w);
int launch_follower_ack(ss_ctx *ctx, const uint64_t *ack_src, uint64_t *const *ack_dst, uint32_t R, uint64_t G,
                        const dev::FlagWait &wait);

int launch_kth_match(ss_ctx *ctx, const uint32_t *match, uint32_t n_peers, uint64_t G, uint32_t k, uint32_t *out);
int launch_prepare_merge(ss_ctx *ctx, const uint64_t *vote_bal, const uint32_t *vote_mask, uint32_t R, uint64_t N,
                         const uint8_t *acks_cnt, uint32_t d, uint32_t population, uint32_t f, uint64_t *max_bal,
                         uint32_t *merged, uint8_t *action);

int launch_crossword_distribute(ss_rs_coder *coder, const uint8_t *data, const uint64_t *data_off,
                                const uint32_t *data_len, const uint8_t *spr, const uint64_t *rep_off, uint64_t n,
                                uint8_t *const *replica_logs, uint32_t n_replicas);

int launch_frame_accept(ss_ctx *ctx, const uint8_t *plane, uint64_t shard_stride, uint32_t shard_idx, uint32_t d, uint32_t p,
                        uint32_t data_len, uint32_t msg_variant, const uint64_t *slot, const uint64_t *ballot, uint64_t n,
                        uint8_t *out, uint64_t frame_stride, uint64_t *frame_off, uint32_t *frame_len);

int launch_gossip_plan(ss_ctx *ctx, uint32_t me, uint32_t population, uint32_t d, const uint8_t *src_peer,
                       const uint32_t *avail, const uint8_t *policy_idx, const uint32_t *policies_host, uint32_t n_policies,
                       uint32_t peer_alive, uint64_t N, uint32_t *targets, uint32_t *excl);

}  // namespace ssb
