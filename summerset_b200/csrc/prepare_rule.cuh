// prepare_rule.cuh -- the Prepare-phase decision for one recovering instance (rspaxos/messages.rs:229-259,
// crossword/messages.rs:280-312), shared by ss_prepare_merge_dev (tally_kernels.cu) and ss_engine_prepare_absorb
// (engine_prepare.cu).
#pragma once
#include <cstdint>

namespace ssb {

// cw: the shards gathered at the highest voted ballot; acks(): the prepare_acks count, read only when fewer than d shards
// are gathered.  Returns the SS_PM_* bits: USE (at least d shards), else NULL (acks >= population - f), else 0 (not
// yet); RECONSTRUCT when fewer than d data shards are among them; PARITY when the codeword then has fewer than
// `population` shards, as the reference compares.
template <typename Acks>
__device__ __forceinline__ uint32_t prepare_action(uint32_t cw, Acks &&acks, uint32_t d, uint32_t data_mask, uint32_t population,
                                                   uint32_t f) {
    uint32_t avail = __popc(cw), act = 0;
    if (avail >= d) {
        act = 1u;
        if (static_cast<uint32_t>(__popc(cw & data_mask)) < d) act |= 4u;
    } else if (acks() >= population - f) {
        act = 2u;
        avail = d;
    }
    if (act != 0u && avail < population) act |= 8u;
    return act;
}

}  // namespace ssb
