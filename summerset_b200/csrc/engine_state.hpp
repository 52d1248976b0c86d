// engine_state.hpp -- the engine handle (ss_engine_*), shared by engine.cu and the CRaft leader's log (craft_leader.cu).
#pragma once
#include "ss_internal.hpp"

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
    uint64_t *ex_cnt = nullptr, *ex_bytes = nullptr;   // [G] execute scratch: records and payload bytes, then their scans
    uint64_t *ex_words = nullptr;           // [3] records written, and the totals when the caller passes none
    uint64_t bo_cap = 0;                    // backoff scratch, grow-only
    uint32_t *bo_keys = nullptr, *bo_idx = nullptr;
    void *bo_sort_tmp = nullptr;
    size_t bo_sort_bytes = 0;
};

namespace ssb {
// frees the CRaft log's state and scratch (craft_leader.cu)
void craft_log_free(ss_engine *e);
}  // namespace ssb
