"""Multi-GPU accept step (SURVEY.md 8e, DESIGN.md section 6): one process per GPU, groups sharded across ranks,
replica r of a group led from rank h simulated on rank (h + r) % world.

The reference's leader sends shard r of every new instance to peer r (rspaxos/request.rs:127-142), the follower logs
it and replies (rspaxos/durability.rs:101-118), and the leader tallies the replies (rspaxos/messages.rs:395-465).
Here, per step k and per rank:

  E_k  ss_accept_step_replicate_dev   waits for the followers' ack flags of step k - lag, tallies those ack planes,
                                      RS-encodes the local groups and stores shard plane r straight into the log of
                                      the GPU that simulates replica r (NVLink stores), then raises shard flag r there
  A_k  ss_follower_ack_dev            waits for the shard flags of step k from the leaders of the replicas hosted
                                      here, stores their ack planes into those leaders' ack buffers, raises ack flags

No host synchronisation and no NCCL call sits between steps: ordering is carried by u64 step counters in device memory
(st.release.sys / ld.acquire.sys).  With lag = 2 the tally of step k reads the acks of step k - 2 (logs and ack buffers
double-buffered), so ranks may drift one step apart instead of meeting at every step.

Two ways to move the shard planes (tools/nvlink_probe.cu measures both per direction, with traffic in both directions):
  mode "p2p"  the encode kernel stores every remote shard straight into the follower GPU's log (fused compute + transfer,
              one kernel; NVLink-bound at the SM store rate)
  mode "ce"   the encode kernel writes the remote planes into a local staging buffer at HBM speed and a second context
              pushes them with the copy engines (ss_copy_d2d on its own stream) WHILE the next step encodes; the shard
              flags are raised behind the copies, the follower kernel runs on that second stream too.  Needs lag = 2.

This module is host-side plumbing only (buffers, CUDA-IPC handles, pointer tables); bench.py and the tests share it.
"""
from __future__ import annotations

from typing import Callable, List, Optional, Sequence

import torch

from .api import Context, ReedSolomon, StepSync, round_up, shard_len
from .sharding import replica_rank

FLAG_SLOTS = 16        # u64 counters per flag array (>= replicas)


class ReplicatedAcceptStep:
    """Per-rank state of the multi-GPU accept step.

    exchange(obj) -> list of every rank's obj, in rank order (torch.distributed.all_gather_object, or the identity
    for world == 1).  `follower_acks` int64 [R, n]: the ack bit-planes this rank's simulated followers reply with.
    """

    def __init__(self, ctx: Context, rs: ReedSolomon, n_groups: int, data_len: int, n_replicas: int, world: int,
                 rank: int, exchange: Callable[[object], List[object]], lag: int = 2, mode: str = "p2p"):
        assert lag in (1, 2) and mode in ("p2p", "ce")
        if mode == "ce":
            assert lag == 2, "the copy-engine mode overlaps step k's transfer with step k+1's encode: it needs lag 2"
        self.mode = mode
        self.ctx, self.rs, self.n, self.data_len, self.R = ctx, rs, n_groups, data_len, n_replicas
        self.world, self.rank, self.lag, self.nbuf = world, rank, lag, lag
        assert n_replicas == rs.d + rs.p and n_replicas <= FLAG_SLOTS
        self.L = shard_len(data_len, rs.d)
        self.ds = round_up(self.L, 16)
        self.plane_bytes = n_groups * self.ds
        self.log_bytes = self.nbuf * n_replicas * self.plane_bytes
        self.acks_bytes = self.nbuf * n_replicas * n_groups * 8
        self.log = ctx.dev_alloc(self.log_bytes)
        self.acks = ctx.dev_alloc(self.acks_bytes)
        self.flags = ctx.dev_alloc(2 * FLAG_SLOTS * 8)          # [0..16): shard flags, [16..32): ack flags
        self.flags.tensor().zero_()
        self.acks.tensor().zero_()
        torch.cuda.synchronize()
        handles = exchange((ctx.ipc_export(self.log), ctx.ipc_export(self.acks), ctx.ipc_export(self.flags))
                           if world > 1 else None)
        self.peer_log, self.peer_acks, self.peer_flags = {}, {}, {}
        for q in range(world):
            if q == rank:
                self.peer_log[q], self.peer_acks[q], self.peer_flags[q] = self.log, self.acks, self.flags
            else:
                self.peer_log[q] = ctx.ipc_open(handles[q][0], self.log_bytes)
                self.peer_acks[q] = ctx.ipc_open(handles[q][1], self.acks_bytes)
                self.peer_flags[q] = ctx.ipc_open(handles[q][2], 2 * FLAG_SLOTS * 8)
        R, n = n_replicas, n_groups
        self.follower_of = [replica_rank(rank, r, world) for r in range(R)]       # where replica r of MY groups lives
        self.leader_of = [(rank - r) % world for r in range(R)]                   # whose replica r lives HERE
        # pointer tables per buffer index
        self.shard_ptrs = [[self.peer_log[self.follower_of[r]].ptr + (b * R + r) * self.plane_bytes for r in range(R)]
                           for b in range(self.nbuf)]
        self.ack_dst = [[self.peer_acks[self.leader_of[r]].ptr + (b * R + r) * n * 8 for r in range(R)]
                        for b in range(self.nbuf)]
        self.acks_view = self.acks.tensor().view(torch.int64).view(self.nbuf, R, n)
        self.log_view = self.log.tensor().view(self.nbuf, R, n, self.ds)
        # E_k: wait on my ack flags, signal shard flag r on the rank hosting replica r of my groups
        self.sync_e = StepSync(self.flags.ptr + FLAG_SLOTS * 8, R, 0,
                               [self.peer_flags[self.follower_of[r]].ptr + r * 8 for r in range(R)], 0)
        # A_k: wait on my shard flags, signal ack flag r on the leader rank of the replica r hosted here
        self.sync_a = StepSync(self.flags.ptr, R, 0,
                               [self.peer_flags[self.leader_of[r]].ptr + (FLAG_SLOTS + r) * 8 for r in range(R)], 0)
        self.k = 0
        if mode == "ce":
            # second context = the copy/follower stream; staging planes for the remote replicas; events between the two
            self.comm = Context(ctx.device, own_stream=True)
            self.staging = ctx.dev_alloc(self.nbuf * R * self.plane_bytes)
            self.remote = [r for r in range(R) if self.follower_of[r] != rank]
            self.local = [r for r in range(R) if self.follower_of[r] == rank]
            self.enc_ptrs = [[(self.staging.ptr if r in self.remote else self.log.ptr) + (b * R + r) * self.plane_bytes for r in range(R)]
                             for b in range(self.nbuf)]
            self.ev_enc = [ctx.event_create() for _ in range(self.nbuf)]
            self.ev_copied = [ctx.event_create() for _ in range(self.nbuf)]
            self.ev_done = ctx.event_create()
            # E_k raises only the flags of the replicas hosted here; the copy stream raises the remote ones behind the copies
            self.sync_e_local = StepSync(0, 0, 0, [self.flags.ptr + r * 8 for r in self.local], 0)
            self.sync_w = StepSync(self.flags.ptr + FLAG_SLOTS * 8, R, 0, [], 0)       # stand-alone wait on my ack flags
            self.sync_aw = StepSync(self.flags.ptr, R, 0, [], 0)                        # stand-alone wait on my shard flags
            self.sync_a_sig = StepSync(0, 0, 0, [self.peer_flags[self.leader_of[r]].ptr + (FLAG_SLOTS + r) * 8 for r in range(R)], 0)
            self.sync_c = StepSync(0, 0, 0, [self.peer_flags[self.follower_of[r]].ptr + r * 8 for r in self.remote], 0)

    def remote_planes(self) -> int:
        return sum(1 for q in self.follower_of if q != self.rank)

    def fill_acks(self, planes: torch.Tensor) -> None:
        """initial content of every ack buffer (what the tally of the first `lag` steps reads)"""
        for b in range(self.nbuf):
            self.acks_view[b].copy_(planes)

    def step(self, data: torch.Tensor, follower_acks: torch.Tensor, threshold: int, committed: torch.Tensor,
             commit_bar: Optional[torch.Tensor]) -> int:
        """One accept step (E_k then A_k on the context's stream).  Returns k."""
        self.k += 1
        k, b = self.k, self.k % self.nbuf
        if self.mode == "ce":
            return self._step_ce(k, b, data, follower_acks, threshold, committed, commit_bar)
        self.sync_e.c.wait_value = max(0, k - self.lag)
        self.sync_e.c.signal_value = k
        self.rs.accept_step_replicate(data, self.data_len, self.shard_ptrs[b], self.ds,
                                      self.acks_view[(k - self.lag) % self.nbuf], threshold, committed, commit_bar,
                                      self.sync_e)
        self.sync_a.c.wait_value = k
        self.sync_a.c.signal_value = k
        self.ctx.follower_ack(follower_acks, self.ack_dst[b], self.sync_a)
        return k

    def _step_ce(self, k, b, data, follower_acks, threshold, committed, commit_bar) -> int:
        ctx, comm, R = self.ctx, self.comm, self.R
        if k > self.nbuf:
            ctx.event_wait(self.ev_copied[b])              # staging[b] was last read by the copies of step k - nbuf
        # The flags E_k waits for are raised by follower kernels, one of which runs on THIS GPU's copy stream: a grid-filling
        # kernel must not spin on them (its CTAs could occupy every SM slot the producer needs).  So the wait is a one-warp
        # kernel ahead of E_k on the compute stream, and E_k itself starts without polling.
        self.sync_w.c.wait_value = max(0, k - self.lag)
        ctx.flags_wait(self.sync_w)
        self.sync_e_local.c.signal_value = k
        # E_k: tally (acks of step k - lag), encode; local replicas' planes into my log, remote ones into staging[b]
        self.rs.accept_step_replicate(data, self.data_len, self.enc_ptrs[b], self.ds, self.acks_view[(k - self.lag) % self.nbuf],
                                      threshold, committed, commit_bar, self.sync_e_local)
        ctx.event_record(self.ev_enc[b])
        # copy stream: push the remote planes with the copy engines while the compute stream goes on to E_{k+1}
        comm.event_wait(self.ev_enc[b])
        for r in self.remote:
            off = (b * R + r) * self.plane_bytes
            comm.copy_d2d(self.peer_log[self.follower_of[r]].ptr + off, self.staging.ptr + off, self.plane_bytes)
        self.sync_c.c.signal_value = k
        comm.flags_signal(self.sync_c)                     # shard flags of the remote followers, behind the copies
        comm.event_record(self.ev_copied[b])
        # A_k on the copy stream (it must not hold up E_{k+1}): one-warp wait for the shards that land HERE, then the ack kernel
        self.sync_aw.c.wait_value = k
        comm.flags_wait(self.sync_aw)
        self.sync_a_sig.c.signal_value = k
        comm.follower_ack(follower_acks, self.ack_dst[b], self.sync_a_sig)
        return k

    def drain(self) -> None:
        """Make the compute stream wait for everything queued on the copy stream (end of a timed region)."""
        if self.mode == "ce":
            self.comm.event_record(self.ev_done)
            self.ctx.event_wait(self.ev_done)

    def encode_only(self, data: torch.Tensor, threshold: int, committed: torch.Tensor, commit_bar: Optional[torch.Tensor]) -> None:
        """The E kernel alone into the current buffers, without flags (kernel-only timing)."""
        b = self.k % self.nbuf
        ptrs = self.enc_ptrs[b] if self.mode == "ce" else self.shard_ptrs[b]
        self.rs.accept_step_replicate(data, self.data_len, ptrs, self.ds, self.acks_view[b], threshold, committed, commit_bar, None)

    def my_shards(self, buf: Optional[int] = None) -> List[torch.Tensor]:
        """Shard plane r of MY groups as stored by the last step, read from wherever it lives (local memory or the
        peer's HBM through the IPC mapping): R tensors uint8 [n, ds]."""
        b = self.k % self.nbuf if buf is None else buf
        out = []
        for r in range(self.R):
            t = self.peer_log[self.follower_of[r]].tensor().view(self.nbuf, self.R, self.n, self.ds)
            out.append(t[b, r])
        return out

    def close(self) -> None:
        if self.mode == "ce":
            self.comm.sync()
            for ev in self.ev_enc + self.ev_copied + [self.ev_done]:
                self.ctx.event_destroy(ev)
            self.staging.free()
            self.comm.close()
        for q in range(self.world):
            if q != self.rank:
                self.peer_log[q].free(); self.peer_acks[q].free(); self.peer_flags[q].free()
        self.log.free(); self.acks.free(); self.flags.free()
