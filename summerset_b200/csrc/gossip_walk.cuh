// gossip_walk.cuh -- Crossword's gossip_targets_excl for one instance (crossword/gossiping.rs:35-84), shared by the
// stand-alone planner (tally_kernels.cu, ss_gossip_plan_dev) and the acceptor's gossip pass (acceptor.cu).
#pragma once
#include "device_common.cuh"

namespace ssb {

// Greedy walk over the peers me+1, me+2, ... (mod population): the source peer and the peers absent from `alive` are
// skipped; a peer whose assigned shards (row(peer)) include one not yet available is selected, on_pick(peer, avail)
// sees the availability map of that moment (the exclusion the peer is sent), and its shards join avail; the walk stops
// once d shards are covered.  Returns the selected peers.
template <typename Row, typename OnPick>
__device__ __forceinline__ uint32_t gossip_walk(uint32_t me, uint32_t population, uint32_t d, uint32_t src, uint32_t avail,
                                                uint32_t alive, Row &&row, OnPick &&on_pick) {
    uint32_t t = 0;
    for (uint32_t pp = me + 1u; pp < me + population; ++pp) {
        const uint32_t peer = pp % population;
        if (peer == src || !((alive >> peer) & 1u)) continue;
        const uint32_t useful = row(peer) & ~avail;
        if (useful != 0u) {
            on_pick(peer, avail);
            t |= 1u << peer;
            avail |= useful;
        }
        if (static_cast<uint32_t>(__popc(avail)) >= d) break;
    }
    return t;
}

}  // namespace ssb
