// follower_state.hpp -- the CRaft follower handle (ss_follower_*), shared by follower.cu, the reconstruct serve and
// step-up calls (craft_recon.cu), the elections (craft_election.cu) and the WAL replay (craft_recover.cu).
#pragma once
#include "ss_internal.hpp"

namespace ssb {
struct FolHdr;                      // one decoded AppendEntries frame (follower.cu)
}  // namespace ssb

struct ss_follower;
namespace ssb {
// grows the per-call scratch to n frames: headers, sort keys, scan partials (follower.cu)
int fol_scratch(ss_follower *f, uint64_t n);
// allocates the election arrays on first use (craft_election.cu)
int el_state(ss_follower *f);
}  // namespace ssb

struct ss_follower {
    ss_ctx *ctx = nullptr;
    ss_follower_config cfg{};
    uint32_t d = 0, T = 0, W = 0;
    uint64_t G = 0;
    uint64_t *start_slot = nullptr, *log_end = nullptr, *curr_term = nullptr, *last_commit = nullptr, *last_snap = nullptr;
    uint8_t *leader = nullptr;
    uint64_t *term = nullptr, *shard_addr = nullptr;
    uint32_t *held = nullptr, *data_len = nullptr;
    uint64_t *last_exec = nullptr;  // [G] last executed slot (ss_follower_execute)
    uint8_t *matrix = nullptr;      // [T*d] the coder's coding matrix (gf256.hpp), row-major
    uint64_t *ex_cnt = nullptr, *ex_bytes = nullptr, *ex_partials = nullptr, *ex_words = nullptr;   // execute scratch
    // per-call scratch, grow-only
    uint64_t cap_frames = 0;
    ssb::FolHdr *hdr = nullptr;
    uint32_t *keys = nullptr, *idx = nullptr;   // [2][cap]
    uint64_t *partials = nullptr;
    void *sort_tmp = nullptr;
    size_t sort_tmp_bytes = 0;
    uint64_t *words = nullptr;      // [4]: cut key, absorb cursor, totals when the caller passes none
    // elections (craft_election.cu), allocated on first use: [G] each
    uint64_t *vote_term = nullptr, *role_term = nullptr;
    uint8_t *voted_for = nullptr, *role = nullptr;
    uint32_t *votes = nullptr;
    uint64_t won_cap = 0;
    uint64_t *won_flag = nullptr;   // [won_cap + 1] the tally's per-segment flags and their scan, grow-only
};
