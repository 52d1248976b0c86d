// engine_state.hpp -- the engine handle (ss_engine_*), shared by engine.cu and the CRaft leader's log (craft_leader.cu).
#pragma once
#include "ss_internal.hpp"

// Where an Accepting Crossword instance's full T-shard codeword lives, so ss_engine_fallback_redo can send it again:
// shard j at addr + j * (stride16 << 4), data_len bytes of payload.  16 bytes per ring position, 1 KiB per group (1 GiB
// at 2^20 groups); plane strides are multiples of 16 below 2^36, so stride16 fits 32 bits.  addr 0: no location recorded.
struct alignas(16) ss_cw_loc {
    uint64_t addr;
    uint32_t stride16;
    uint32_t data_len;
};
constexpr uint64_t kCwLocStrideLimit = 1ull << 36;

struct ss_engine {
    ss_ctx *ctx = nullptr;
    ss_rs_coder *coder = nullptr;
    ss_engine_config cfg{};
    uint64_t G = 0;
    uint32_t n = 0, majority = 0, threshold = 0, d = 0, T = 0;
    uint32_t L = 0, ds = 0;
    // Paxos family
    uint64_t *planes = nullptr, *bal_prepared = nullptr, *inst_bal = nullptr, *accepting = nullptr, *committed = nullptr;
    uint64_t *window_base = nullptr;        // [G] absolute slot of window position 0
    bool windowed = false;                  // a base may be non-zero: set by ss_engine_advance / ss_engine_window_get
    uint32_t *commit_bar = nullptr;
    uint8_t *shards = nullptr;
    // ragged proposals: allocated on the first ss_engine_propose_ragged call
    uint32_t *rg_len = nullptr;             // [G] effective length (0 = the group does not propose)
    uint64_t *rg_partials = nullptr;        // [scan_tiles(G)] tile sums of the pitch scan
    uint64_t *rg_need = nullptr;            // [1] total pitch, when the caller does not ask for it
    // Crossword
    uint8_t *policy_idx = nullptr;          // [G*64]
    uint32_t *policies = nullptr, *lut_bits = nullptr;
    uint32_t n_policies = 0, lut_words = 0;
    int balanced = 1;
    ss_cw_loc *cw_loc = nullptr;            // [G*64] written by every path into Accepting (enter_accepting)
    // soft fallback (engine_fallback.cu), allocated on the first ss_engine_fallback_redo: fb_first [G] the first list
    // entry of each group (UINT32_MAX between calls); per listed entry the redone ring positions and the records and
    // store bytes they add, then their scans
    uint32_t *fb_first = nullptr;
    uint64_t *fb_mask = nullptr, *fb_cnt = nullptr, *fb_partials = nullptr, *fb_words = nullptr;
    uint64_t fb_cap = 0;
    // Raft
    uint32_t *match = nullptr, *next_slot = nullptr, *last_commit = nullptr, *log_end = nullptr, *curr_term = nullptr,
             *terms = nullptr, *last_snap = nullptr;
    uint8_t *touched = nullptr;
    uint32_t W = 0, n_peers = 0;
    // CRaft leader's log (craft_leader.cu): host-side flags, state allocated when the log is first used
    bool log_in_use = false;                // ss_engine_craft_log_view_get or ss_engine_craft_propose ran
    bool raft_appended = false;             // ss_engine_raft_append ran: entries without a codeword, no log calls
    uint64_t log_plane_stride = 0;          // of every craft propose (0 = none yet)
    uint64_t *log_start = nullptr;          // [G]
    uint32_t *try_next = nullptr;           // [P][G]
    uint32_t *ent_len = nullptr;            // [G][W] data_len per ring position
    uint64_t *ent_addr = nullptr;           // [G][W] shard_addr (shard j at + j * plane_stride)
    uint64_t *ent_log_offset = nullptr;     // [G][W]
    uint64_t *cl_partials = nullptr;        // [scan_tiles(max(G, P*G))]
    uint64_t *cl_words = nullptr;           // [4] scan totals the caller does not ask for
    uint32_t *cl_eff = nullptr;             // [G] effective propose length
    uint64_t *cl_wal = nullptr;             // [G] propose: WAL record lengths
    uint64_t *pk_frames = nullptr, *pk_bytes = nullptr, *pk_range = nullptr;   // [P*G] pack scratch
    uint64_t *last_exec = nullptr;          // [G] last executed slot (ss_engine_craft_execute)
    uint32_t *held = nullptr;               // [G][W] shards the leader holds (propose: all; step-up: the follower's),
                                            // kept from the first step-up or recon view on (craft_held_in_use)
    uint64_t *last_recon = nullptr;         // [G] last slot a reconstruct read listed (ss_engine_craft_reconstruct_reads)
    uint8_t *matrix = nullptr;              // [T*d] the coder's coding matrix: execute regenerates missing data shards
    bool held_partial = false;              // a held mask may lack shards (step-up ran, or the recon view was handed out);
                                            // until then propose, pack and execute neither write nor read held
    uint8_t *led = nullptr;                 // [G] 1: the engine leads the group (craft_stepdown.cu), allocated on the first
                                            // step-down or role view; until then every group is led and the log calls run
                                            // their kLed = false kernels
    uint64_t *rc_words = nullptr;           // [n] recon scratch (listed groups / frames), grow-only with rc_cap
    uint64_t rc_cap = 0;
    uint64_t *ex_cnt = nullptr, *ex_bytes = nullptr;   // [G] execute scratch: records and payload bytes, then their scans
    uint64_t *ex_words = nullptr;           // [3] records written, and the totals when the caller passes none
    uint64_t bo_cap = 0;                    // backoff scratch, grow-only
    uint32_t *bo_keys = nullptr, *bo_idx = nullptr;
    void *bo_sort_tmp = nullptr;
    size_t bo_sort_bytes = 0;
    // RSPaxos / Crossword Prepare phase (engine_prepare.cu), allocated on the first ss_engine_prepare_absorb: the
    // bookkeeping of ballot pa_ballot[g] (reset when bal_prep_sent differs): prepare_acks, the decided ring positions,
    // and per ring position [G*64] prepare_max_bal and the gathered codeword (shards, data_len, slot offset)
    uint64_t *pa_ballot = nullptr, *pa_done = nullptr, *pa_max_bal = nullptr, *pa_off = nullptr;
    uint32_t *pa_acks = nullptr, *pa_mask = nullptr, *pa_len = nullptr;
    uint64_t *pa_words = nullptr;           // [5] applied store bytes and decided records, the totals the caller does not ask for
    uint64_t pa_cap = 0, pa_dec_cap = 0;    // per-frame and per-decided-record scratch, grow-only
    ss_prepare_reply_rec *pa_rec = nullptr;
    uint64_t *pa_cnt = nullptr, *pa_dst = nullptr, *pa_fill = nullptr, *pa_partials = nullptr;
    uint32_t *pa_take = nullptr, *pa_present = nullptr;
    int32_t *pa_status = nullptr;
};

namespace ssb {
__device__ __forceinline__ void put_cw_loc(ss_cw_loc *__restrict__ cw_loc, uint64_t at, const uint8_t *shard0, uint64_t plane_stride,
                                           uint32_t data_len) {
    ss_cw_loc v;
    v.addr = reinterpret_cast<uint64_t>(shard0);
    v.stride16 = static_cast<uint32_t>(plane_stride >> 4);
    v.data_len = data_len;
    cw_loc[at] = v;
}

// instance s of group g enters Accepting; acc / cm are the group's accepting / committed words as loaded.  cw_loc
// (Crossword engines; nullptr otherwise or when the caller records the location itself) receives where the instance's
// full codeword lives: shard 0 at shard0, plane_stride apart, data_len bytes.
__device__ __forceinline__ void enter_accepting(uint64_t g, uint64_t s, uint64_t acc, uint64_t cm, uint64_t *__restrict__ planes,
                                                uint32_t R, uint64_t G, const uint64_t *__restrict__ bal_prepared,
                                                uint64_t *__restrict__ inst_bal, uint64_t *__restrict__ accepting,
                                                uint64_t *__restrict__ committed, uint8_t *__restrict__ policy_idx,
                                                const uint8_t *__restrict__ new_policy, ss_cw_loc *__restrict__ cw_loc,
                                                const uint8_t *shard0, uint64_t plane_stride, uint32_t data_len) {
    const uint32_t pos = static_cast<uint32_t>(s & 63u);
    const uint64_t bit = 1ull << pos;
    accepting[g] = acc | bit;                              // Status::Accepting (request.rs: inst.status = Accepting)
    committed[g] = cm & ~bit;                              // a re-used window slot starts uncommitted
    inst_bal[g * 64 + pos] = bal_prepared[g];              // inst.bal = bal_prepared
    for (uint32_t r = 0; r < R; ++r) planes[static_cast<uint64_t>(r) * G + g] &= ~bit;   // fresh accept_acks
    if (policy_idx != nullptr) policy_idx[g * 64 + pos] = new_policy != nullptr ? new_policy[g] : 0;
    if (cw_loc != nullptr) put_cw_loc(cw_loc, g * 64 + pos, shard0, plane_stride, data_len);
}

// frees the Prepare-phase state and scratch (engine_prepare.cu)
void prepare_free(ss_engine *e);
// frees the soft fallback's scratch (engine_fallback.cu)
void fallback_free(ss_engine *e);
// frees the CRaft log's state and scratch (craft_leader.cu)
void craft_log_free(ss_engine *e);
// the configuration checks every log call makes, and taking the log into use on the first call (craft_leader.cu)
int craft_check(ss_engine *e);
int craft_log_init(ss_engine *e);
// held is kept from here on: every mask starts full (only propose made entries so far), and propose writes it (craft_leader.cu)
int craft_held_in_use(ss_engine *e);
// the led bytes, allocated on first use with every group led (craft_stepdown.cu)
int craft_led_in_use(ss_engine *e);
// led = 1 for the groups of the listings step-up took (verdict DONE), once the bytes exist (craft_stepdown.cu)
int craft_led_mark(ss_engine *e, const uint32_t *groups, const uint32_t *verdict, uint64_t n);
// the log's grow-only sort scratch (bo_*) for n keys of `bits` bits, shared by the back-off and absorb (craft_leader.cu)
int backoff_scratch(ss_engine *e, uint64_t n, int bits);
// the recon / step-down scratch (rc_words), grow-only: `words` u64 (craft_recon.cu)
int rc_scratch(ss_engine *e, uint64_t words);
}  // namespace ssb
