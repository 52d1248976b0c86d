"""Python binding of the batched multi-group consensus engine (ss_engine_* in include/summerset_b200.h).

The engine itself is native: the state of G independent replica groups lives in HBM and every transition --
propose bookkeeping, AcceptReply / AppendEntriesReply ingest, the fused commit tick -- is a CUDA kernel behind the C
ABI (summerset_b200/csrc/engine.cu).  This module only marshals arguments and wraps the engine's device arrays as
torch tensors (zero-copy views) so tests can read results and install state; it runs no torch ops on them.

    LeaderEngine(ctx, protocol, G, population, ...)   protocol in {"multipaxos", "rspaxos", "crossword"}
        propose(slot, payloads[, policy])   multipaxos/request.rs:112-221, rspaxos/request.rs:72-142, crossword/request.rs:82-185
        propose_next(store, payloads[, policy])   the same at each group's first Null slot (rspaxos/mod.rs:434-442)
        propose_ragged(arena, data_off, data_len, store[, policy])   variable-length batches into a caller-owned store
        fallback_redo(groups, policy, store, store_used, dec_capacity[, peer_alive])   Crossword's soft fallback
                                            (crossword/leadership.rs:389-550): unresponsive Accepting instances re-assigned
        on_accept_replies(records)          handle_msg_accept_reply filters (multipaxos/messages.rs:377-409, ...)
        tick()                              commit decision + commit_bar, one kernel
        advance([upto])                     retire committed prefixes: window_base moves on (multipaxos/snapshot.rs:121-171)
    Acceptor(ctx, protocol, G, population, me, d, T)   protocol in {"rspaxos", "crossword"}: the follower side
        accept(buf, frame_off, frame_group, frame_peer, store, wal)   handle_msg_accept over a batch of Accept frames
                                            (rspaxos/messages.rs:329-392, crossword/messages.rs:403-470): store, AcceptData
                                            records and AcceptReply cells
        advance(upto)                       retire window prefixes
        heartbeat(group, peer, ballot, commit_bar, exec_bar)   heard_heartbeat's commit walk (rspaxos/leadership.rs:222-311)
        execute(out, rec_capacity)          handle_logged_commit_slot's execution walk (rspaxos/durability.rs:125-186):
                                            request batches decoded from the held shards
        prepare(buf, ..., wal, rec_capacity)   handle_msg_prepare (rspaxos/messages.rs:13-84): PrepareBal records
        prepare_reply(rec_group, rec_slot, out)   handle_logged_prepare_bal's follower branch: PrepareReply frames
        gossip(out, frame_capacity, batch_size)   Crossword trigger_gossiping (crossword/gossiping.rs:88-192): Reconstruct
                                            frames for the committed instances missing shards, to the peers gossip_targets_excl picks
        step_up_reads(out, frame_capacity, chunk_size)   become_a_leader's recon_slots (rspaxos/leadership.rs:99-172):
                                            Reconstruct frames to broadcast
    prepare_reply_parse(ctx, buf, frame_off, d, T)   the new leader's side: PrepareReply frames -> vote records
    RaftEngine(ctx, G, population[, fault_tolerance, craft])
        append(n_new) / on_append_replies(records) / tick()      raft/messages.rs:243-309, craft/messages.rs:300-308
        CRaft leader's log: propose(me, arena, data_off, data_len, store, wal)   handle_req_batch (craft/request.rs:70-116)
        pack_append(me, out, max_frames[, want_end, heartbeat])   AppendEntries frames (craft/durability.rs:12-127)
        backoff(buf, frame_off, frame_group, frame_peer, rec_kind)   the conflict branch (craft/messages.rs:386-406)
        advance_log(upto) / log_view()      the snapshot's start_slot move; log_start, try_next and the entry rings
        execute(out, rec_capacity) / exec_view()   the committed entries' request batches (craft/messages.rs:316-359)
        step_up(follower, groups, term, store) / reconstruct_reads(out, ...) / absorb(buf, ...) / recon_view()
                                            fail-over: become_the_leader's log half, Reconstruct reads, their replies
        set_full_copy(on)                   the commit threshold of full-copy mode (craft/leadership.rs:282-288)
    Follower(ctx, G, population, me[, window])   the CRaft follower
        append(buf, frame_off, frame_group, frame_peer, store, wal)   handle_msg_append_entries (craft/messages.rs:14-252):
                                            store, LogEntry / Metadata records, AppendEntriesReply cells
        advance(upto)                       the snapshot's start_slot move
        execute(out, rec_capacity)          the committed entries' request batches (craft/messages.rs:198-240)
        reconstruct_serve(buf, ...)         a new leader's Reconstruct reads (craft/messages.rs:621-662)
        campaign(groups) / vote(buf, ...) / tally(buf, ...) / vote_view()   elections: become_a_candidate
                                            (craft/leadership.rs:143-209), handle_msg_request_vote and _reply
                                            (craft/messages.rs:499-619); tally's won_group / won_term feed step_up
    append_reply_parse(ctx, buf, frame_off, frame_group, frame_peer, curr_term, G)   the leader's side: AppendEntriesReply
                                            frames -> RaftEngine.on_append_replies records
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from ._lib import check
from .api import Context

_PROTO = {"multipaxos": _lib.SS_PROTO_MULTIPAXOS, "rspaxos": _lib.SS_PROTO_RSPAXOS, "crossword": _lib.SS_PROTO_CROSSWORD,
          "raft": _lib.SS_PROTO_RAFT, "craft": _lib.SS_PROTO_CRAFT}


class _DevArray:
    """__cuda_array_interface__ carrier for a raw device pointer owned by the engine"""

    def __init__(self, ptr: int, shape: Tuple[int, ...], typestr: str):
        self.__cuda_array_interface__ = {"shape": shape, "typestr": typestr, "data": (ptr, False), "version": 2}


def _execute(fn, h, out: torch.Tensor, rec_capacity: int, out_capacity: Optional[int]) -> dict:
    """one call of an execution walk with ss_acceptor_execute's argument list after the handle"""
    assert out.dtype == torch.uint8 and out.is_contiguous()
    dev = out.device
    res = dict(rec_group=torch.empty(rec_capacity, dtype=torch.int32, device=dev),
               rec_slot=torch.empty(rec_capacity, dtype=torch.int64, device=dev),
               rec_off=torch.empty(rec_capacity, dtype=torch.int64, device=dev),
               rec_len=torch.empty(rec_capacity, dtype=torch.int32, device=dev),
               totals=torch.empty(2, dtype=torch.int64, device=dev))
    p = lambda x: x.data_ptr()
    check(fn(h, p(out), out.numel() if out_capacity is None else out_capacity, p(res["rec_group"]), p(res["rec_slot"]),
             p(res["rec_off"]), p(res["rec_len"]), rec_capacity, p(res["totals"])))
    return res


class _EngineBase:
    def __init__(self, ctx: Context, cfg: _lib.EngineConfig, n_groups: int):
        self.ctx, self.lib, self.G = ctx, ctx.lib, n_groups
        h = C.c_void_p()
        check(self.lib.ss_engine_create(ctx.h, C.byref(cfg), n_groups, C.byref(h)))
        self.h = h
        self.view = _lib.EngineView()
        check(self.lib.ss_engine_view_get(self.h, C.byref(self.view)))
        self.dev = torch.device("cuda", ctx.device)

    def _tensor(self, ptr: Optional[int], shape: Tuple[int, ...], typestr: str, dtype: torch.dtype) -> Optional[torch.Tensor]:
        if not ptr:
            return None
        return torch.as_tensor(_DevArray(ptr, shape, typestr), device=self.dev).view(dtype).view(shape)

    def close(self) -> None:
        if getattr(self, "h", None) is not None and self.h:
            self.lib.ss_engine_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class LeaderEngine(_EngineBase):
    SLOTS = 64

    def __init__(self, ctx: Context, protocol: str, n_groups: int, population: int = 5, fault_tolerance: int = 0,
                 data_len: int = 0, keep_slots: int = 1, rs_total_shards: int = 0, rs_data_shards: int = 0):
        assert protocol in ("multipaxos", "rspaxos", "crossword")
        cfg = _lib.EngineConfig(_PROTO[protocol], population, fault_tolerance, data_len, rs_total_shards, rs_data_shards,
                                keep_slots, 0)
        super().__init__(ctx, cfg, n_groups)
        v, G = self.view, n_groups
        self.protocol, self.n = protocol, population
        self.threshold, self.d, self.T, self.L, self.ds = v.threshold, v.data_shards, v.total_shards, v.shard_len, v.shard_stride
        self.keep = max(1, keep_slots)
        self.planes = self._tensor(v.planes, (population, G), "<i8", torch.int64)
        self.bal_prepared = self._tensor(v.bal_prepared, (G,), "<i8", torch.int64)
        self.inst_bal = self._tensor(v.inst_bal, (G * 64,), "<i8", torch.int64)
        self.accepting = self._tensor(v.accepting, (G,), "<i8", torch.int64)
        self.committed = self._tensor(v.committed, (G,), "<i8", torch.int64)
        self.commit_bar = self._tensor(v.commit_bar, (G,), "<i4", torch.int32)
        self.shards = self._tensor(v.shards, (self.keep, self.T, G, self.ds), "|u1", torch.uint8) if v.shards else None
        self.policy_idx = self._tensor(v.policy_idx, (G * 64,), "|u1", torch.uint8)
        self._window_base = None

    @property
    def window_base(self) -> torch.Tensor:
        """int64 [G]: absolute slot of window position 0 per group; the per-slot words above are rings (slot s at bit
        s & 63).  Fetched on first use: from then on the engine's tick reads the bases (until then they are all 0)."""
        if self._window_base is None:
            wb = C.c_void_p()
            check(self.lib.ss_engine_window_get(self.h, C.byref(wb)))
            self._window_base = self._tensor(wb.value, (self.G,), "<i8", torch.int64)
        return self._window_base

    def set_prepared_ballots(self, ballots: torch.Tensor) -> None:
        assert ballots.is_cuda and ballots.dtype == torch.int64 and ballots.numel() == self.G
        check(self.lib.ss_engine_set_prepared_ballots(self.h, ballots.data_ptr()))

    def set_policies(self, policies: Sequence[Sequence[int]], balanced: bool) -> None:
        pol = np.ascontiguousarray(np.array(policies, dtype=np.uint32))
        assert pol.shape[1] == self.n
        check(self.lib.ss_engine_set_policies(self.h, pol.ctypes.data, pol.shape[0], 1 if balanced else 0))

    def propose(self, slot: int, payloads: Optional[torch.Tensor], policy: Optional[torch.Tensor] = None) -> Optional[torch.Tensor]:
        """payloads uint8 [G, >= data_len] on the device (None for MultiPaxos).  Returns the proposal's shard planes
        [T, G, ds] (plane r = the packed Accept payloads for the peer(s) holding shard r), or None for MultiPaxos."""
        base = C.c_void_p()
        stride = payloads.shape[1] if payloads is not None else 0
        check(self.lib.ss_engine_propose(self.h, slot, payloads.data_ptr() if payloads is not None else None, stride,
                                         policy.data_ptr() if policy is not None else None, C.byref(base)))
        return self.shards[slot % self.keep] if self.shards is not None else None

    def prepare_absorb(self, acceptor: "Acceptor", buf: torch.Tensor, frame_off: torch.Tensor, frame_group: torch.Tensor,
                       frame_peer: torch.Tensor, bal_prep_sent: torch.Tensor, store: torch.Tensor, store_used: torch.Tensor,
                       wal: torch.Tensor, rec_capacity: int, dec_capacity: int, policy: Optional[torch.Tensor] = None,
                       wal_capacity: Optional[int] = None, reply_variant: int = 1, wal_variant: int = 0) -> dict:
        """handle_msg_prepare_reply for a batch of PrepareReply frames (buf uint8 at any alignment, frame_off int64, frame_group
        int32, frame_peer uint8, each [n]; the leader's own replies included) after acceptor.step_up on this replica's
        acceptor.  bal_prep_sent: int64 [G], the step-up's ballot per group, 0 where not preparing; policy: Crossword uint8
        [G].  Gathered codewords go to store (uint8 [T, plane_stride], caller-owned, the ragged proposal layout) from
        store_used (int64 [1], in/out); the external fill's PrepareBal cells to wal (uint8, 16-byte aligned).  Returns device
        tensors rec_group (int32), rec_slot (int64), each [rec_capacity]; the decided list dec_slot, dec_ballot,
        dec_shard_off (int64), dec_data_len (int32), dec_policy (uint8), dec_group (int32), each [dec_capacity], ready for
        ss_frame_accept_pack_ragged_dev; pending (int64 [G]), verdict (int32 [n]) and totals (int64 [3]: decided records,
        PrepareBal records and store bytes asked for)."""
        assert buf.dtype == torch.uint8 and frame_off.dtype == torch.int64 and frame_group.dtype == torch.int32
        assert frame_peer.dtype == torch.uint8 and bal_prep_sent.dtype == torch.int64 and bal_prep_sent.numel() == self.G
        assert store.dtype == torch.uint8 and store.dim() == 2 and store.is_contiguous() and store_used.dtype == torch.int64
        assert wal.dtype == torch.uint8 and (policy is None or (policy.dtype == torch.uint8 and policy.numel() == self.G))
        n, dev = frame_off.numel(), self.dev
        e = lambda k, dt: torch.empty(max(k, 1), dtype=dt, device=dev)
        res = dict(rec_group=e(rec_capacity, torch.int32), rec_slot=e(rec_capacity, torch.int64), dec_slot=e(dec_capacity, torch.int64),
                   dec_ballot=e(dec_capacity, torch.int64), dec_shard_off=e(dec_capacity, torch.int64),
                   dec_data_len=e(dec_capacity, torch.int32), dec_policy=e(dec_capacity, torch.uint8),
                   dec_group=e(dec_capacity, torch.int32), pending=e(self.G, torch.int64), verdict=e(n, torch.int32),
                   totals=e(3, torch.int64))
        p = lambda x: None if x is None else x.data_ptr()
        check(self.lib.ss_engine_prepare_absorb(self.h, acceptor.h, p(buf), buf.numel(), p(frame_off), p(frame_group), p(frame_peer), n,
                                                reply_variant, wal_variant, p(bal_prep_sent), p(policy), p(store), store.shape[1],
                                                p(store_used), p(wal), wal.numel() if wal_capacity is None else wal_capacity,
                                                p(res["rec_group"]), p(res["rec_slot"]), rec_capacity, p(res["dec_slot"]),
                                                p(res["dec_ballot"]), p(res["dec_shard_off"]), p(res["dec_data_len"]),
                                                p(res["dec_policy"]), p(res["dec_group"]), dec_capacity, p(res["pending"]),
                                                p(res["verdict"]), p(res["totals"])))
        return res

    def fallback_redo(self, groups: torch.Tensor, policy: torch.Tensor, store: torch.Tensor, store_used: torch.Tensor,
                      dec_capacity: int, peer_alive: Optional[torch.Tensor] = None) -> dict:
        """Crossword's fallback_redo_accepts for the listed groups (int32 [n]): every Accepting instance whose policy is not
        responsive for peer_alive (int32 [G] replica masks, None = all alive) takes policy (uint8 [G]), loses its acks and
        has its codeword copied from where it was proposed into store (uint8 [T, plane_stride], caller-owned) from
        store_used (int64 [1], in/out).  Returns device tensors dec_slot, dec_ballot, dec_shard_off (int64), dec_data_len
        (int32), dec_policy (uint8), dec_group (int32), each [dec_capacity], ready for ss_frame_accept_pack_ragged_dev;
        verdict (int32 [n]) and totals (int64 [2]: records and store bytes asked for)."""
        assert groups.dtype == torch.int32 and policy.dtype == torch.uint8 and policy.numel() == self.G
        assert store.dtype == torch.uint8 and store.dim() == 2 and store.is_contiguous() and store_used.dtype == torch.int64
        assert peer_alive is None or (peer_alive.dtype == torch.int32 and peer_alive.numel() == self.G)
        n, dev = groups.numel(), self.dev
        e = lambda k, dt: torch.empty(max(k, 1), dtype=dt, device=dev)
        res = dict(dec_slot=e(dec_capacity, torch.int64), dec_ballot=e(dec_capacity, torch.int64), dec_shard_off=e(dec_capacity, torch.int64),
                   dec_data_len=e(dec_capacity, torch.int32), dec_policy=e(dec_capacity, torch.uint8),
                   dec_group=e(dec_capacity, torch.int32), verdict=torch.empty(n, dtype=torch.int32, device=dev),
                   totals=e(2, torch.int64))
        p = lambda x: None if x is None else x.data_ptr() or None
        check(self.lib.ss_engine_fallback_redo(self.h, p(groups), n, p(peer_alive), p(policy), p(store), store.shape[1], p(store_used),
                                               p(res["dec_slot"]), p(res["dec_ballot"]), p(res["dec_shard_off"]),
                                               p(res["dec_data_len"]), p(res["dec_policy"]), p(res["dec_group"]), dec_capacity,
                                               p(res["verdict"]), p(res["totals"])))
        return res

    def propose_next(self, store: int, payloads: Optional[torch.Tensor],
                     policy: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
        """One new instance per group at its first Null slot; shards into shard store `store` (< keep_slots).
        Returns (slot_out int64 [G]: the absolute slot, or -1 (UINT64_MAX) for a group whose window is full,
        the store's shard planes [T, G, ds] or None for MultiPaxos)."""
        base = C.c_void_p()
        stride = payloads.shape[1] if payloads is not None else 0
        slot_out = torch.empty(self.G, dtype=torch.int64, device=self.dev)
        check(self.lib.ss_engine_propose_next(self.h, store, payloads.data_ptr() if payloads is not None else None, stride,
                                              policy.data_ptr() if policy is not None else None, slot_out.data_ptr(),
                                              C.byref(base)))
        return slot_out, (self.shards[store] if self.shards is not None else None)

    def propose_ragged(self, arena: torch.Tensor, data_off: torch.Tensor, data_len: torch.Tensor, store: torch.Tensor,
                       policy: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """Ragged request batches (RSPaxos / Crossword): group g proposes arena[data_off[g] : +data_len[g]] at its first
        Null slot, or nothing when data_len[g] == 0.  store: caller-owned uint8 [T, plane_stride] (plane_stride a
        multiple of 32); shard j of a proposing group lands at store[j, shard_off[g]:], zero-padded to 16 bytes.
        Returns (slot_out int64 [G], shard_off int64 [G], need int64 [1]); -1 (UINT64_MAX) marks a group that did not
        propose, need = the total slot pitch the batch asked for."""
        assert arena.is_cuda and arena.dtype == torch.uint8
        assert data_off.dtype == torch.int64 and data_len.dtype == torch.int32 and data_len.numel() == self.G
        assert store.dtype == torch.uint8 and store.dim() == 2 and store.shape[0] == self.T and store.is_contiguous()
        slot_out = torch.empty(self.G, dtype=torch.int64, device=self.dev)
        shard_off = torch.empty(self.G, dtype=torch.int64, device=self.dev)
        need = torch.empty(1, dtype=torch.int64, device=self.dev)
        check(self.lib.ss_engine_propose_ragged(self.h, arena.data_ptr(), data_off.data_ptr(), data_len.data_ptr(),
                                                policy.data_ptr() if policy is not None else None, store.data_ptr(),
                                                store.shape[1], shard_off.data_ptr(), slot_out.data_ptr(), need.data_ptr()))
        return slot_out, shard_off, need

    def advance(self, upto: Optional[torch.Tensor] = None) -> None:
        """Retires committed prefixes up to the absolute slots upto (int64 [G]), or all of them when upto is None."""
        assert upto is None or (upto.is_cuda and upto.dtype == torch.int64 and upto.numel() == self.G)
        check(self.lib.ss_engine_advance(self.h, upto.data_ptr() if upto is not None else None))

    def on_accept_replies(self, rec_group: torch.Tensor, rec_slot: torch.Tensor, rec_peer: torch.Tensor, rec_ballot: torch.Tensor) -> None:
        assert rec_group.dtype == torch.int32 and rec_slot.dtype == torch.uint8 and rec_peer.dtype == torch.uint8 and rec_ballot.dtype == torch.int64
        check(self.lib.ss_engine_ingest(self.h, rec_group.data_ptr(), rec_slot.data_ptr(), rec_peer.data_ptr(), rec_ballot.data_ptr(),
                                        rec_group.numel()))

    def tick(self, newly: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """One fused kernel.  Returns (committed words, commit_bar): views of the engine state."""
        check(self.lib.ss_engine_tick(self.h, newly.data_ptr() if newly is not None else None))
        return self.committed, self.commit_bar


class RSPaxosLeaderEngine(LeaderEngine):
    """RSPaxos leader (rspaxos/request.rs:72-142, rspaxos/messages.rs:395-465)."""

    def __init__(self, ctx: Context, n_groups: int, population: int = 5, fault_tolerance: int = 1, data_len: int = 4096,
                 device=None, keep_slots: int = 1):
        super().__init__(ctx, "rspaxos", n_groups, population, fault_tolerance, data_len, keep_slots)


class RaftEngine(_EngineBase):
    def __init__(self, ctx: Context, n_groups: int, population: int = 7, fault_tolerance: int = 0, craft: bool = False,
                 window: int = 64):
        cfg = _lib.EngineConfig(_PROTO["craft" if craft else "raft"], population, fault_tolerance, 0, 0, 0, 0, window)
        super().__init__(ctx, cfg, n_groups)
        v, G, P = self.view, n_groups, population - 1
        self.P, self.W, self.threshold = P, v.raft_window, v.threshold
        self.match = self._tensor(v.match, (P, G), "<i4", torch.int32)
        self.next_slot = self._tensor(v.next_slot, (P, G), "<i4", torch.int32)
        self.last_commit = self._tensor(v.last_commit, (G,), "<i4", torch.int32)
        self.log_end = self._tensor(v.log_end, (G,), "<i4", torch.int32)
        self.curr_term = self._tensor(v.curr_term, (G,), "<i4", torch.int32)
        self.last_snap = self._tensor(v.last_snap, (G,), "<i4", torch.int32)
        self.terms = self._tensor(v.terms, (G, self.W), "<i4", torch.int32)

    def append(self, n_new: torch.Tensor) -> None:
        assert n_new.is_cuda and n_new.dtype == torch.int32 and n_new.numel() == self.G
        check(self.lib.ss_engine_raft_append(self.h, n_new.data_ptr()))

    def on_append_replies(self, rec_group: torch.Tensor, rec_peer: torch.Tensor, rec_end_slot: torch.Tensor) -> None:
        assert rec_group.dtype == torch.int32 and rec_peer.dtype == torch.uint8 and rec_end_slot.dtype == torch.int32
        check(self.lib.ss_engine_raft_ingest(self.h, rec_group.data_ptr(), rec_peer.data_ptr(), rec_end_slot.data_ptr(), rec_group.numel()))

    def tick(self) -> Tuple[torch.Tensor, torch.Tensor]:
        check(self.lib.ss_engine_tick(self.h, None))
        return self.last_commit, self.last_snap

    # ---- the CRaft leader's log (ss_engine_craft_*): using it refuses append() from then on, and vice versa ----
    def log_view(self) -> dict:
        """Takes the log into use and returns zero-copy views: log_start int64 [G], try_next int32 [P, G], and per ring
        position data_len int32, shard_addr and log_offset int64 [G, W]."""
        v = _lib.CraftLogView()
        check(self.lib.ss_engine_craft_log_view_get(self.h, C.byref(v)))
        G, W = self.G, self.W
        return dict(log_start=self._tensor(v.log_start, (G,), "<i8", torch.int64),
                    try_next=self._tensor(v.try_next, (self.P, G), "<i4", torch.int32),
                    data_len=self._tensor(v.data_len, (G, W), "<i4", torch.int32),
                    shard_addr=self._tensor(v.shard_addr, (G, W), "<i8", torch.int64),
                    log_offset=self._tensor(v.log_offset, (G, W), "<i8", torch.int64), plane_stride=v.plane_stride)

    def propose(self, me: int, arena: torch.Tensor, data_off: torch.Tensor, data_len: torch.Tensor, store: torch.Tensor,
                wal: torch.Tensor, log_offset: Optional[torch.Tensor] = None, wal_capacity: Optional[int] = None,
                full_copy: bool = False) -> dict:
        """One entry per group with a batch (data_len int32 [G] > 0), coded into store (uint8 [T, plane_stride], caller-owned,
        alive until advance_log retires its entries) and the leader's LogEntry record into wal (uint8, 16-byte aligned).
        Returns device tensors slot_out, shard_off, wal_off (int64 [G], -1 = not proposed), wal_len (int64 [G]) and
        need (int64 [1])."""
        assert arena.dtype == torch.uint8 and data_off.dtype == torch.int64 and data_len.dtype == torch.int32
        assert store.dtype == torch.uint8 and store.dim() == 2 and store.is_contiguous() and wal.dtype == torch.uint8
        assert log_offset is None or (log_offset.dtype == torch.int64 and log_offset.numel() == self.G)
        e = lambda n=self.G: torch.empty(n, dtype=torch.int64, device=self.dev)
        out = dict(slot_out=e(), shard_off=e(), wal_off=e(), wal_len=e(), need=e(1))
        p = lambda x: None if x is None else x.data_ptr()
        check(self.lib.ss_engine_craft_propose(self.h, me, p(arena), p(data_off), p(data_len), p(store), store.shape[1],
                                               p(out["shard_off"]), p(out["slot_out"]), p(out["need"]), p(log_offset), p(wal),
                                               wal.numel() if wal_capacity is None else wal_capacity, p(out["wal_off"]),
                                               p(out["wal_len"]), 1 if full_copy else 0))
        return out

    def pack_append(self, me: int, out: torch.Tensor, max_frames: int, want_end: Optional[torch.Tensor] = None,
                    heartbeat: bool = False, full_copy: bool = False, msg_chunk_size: int = 10, append_variant: int = 0,
                    out_capacity: Optional[int] = None) -> dict:
        """AppendEntries frames for every (peer, group) into out (uint8, 16-byte aligned).  Returns device tensors
        frame_off, frame_len (int64 [max_frames]), frame_group (int32), frame_peer (uint8: the peer index), n_frames and
        total (int64 [1]) and pair_status (int32 [P, G])."""
        assert out.dtype == torch.uint8 and (want_end is None or (want_end.dtype == torch.int64 and want_end.numel() == self.P * self.G))
        dev, cap = out.device, max(max_frames, 1)
        res = dict(frame_off=torch.empty(cap, dtype=torch.int64, device=dev), frame_len=torch.empty(cap, dtype=torch.int64, device=dev),
                   frame_group=torch.empty(cap, dtype=torch.int32, device=dev), frame_peer=torch.empty(cap, dtype=torch.uint8, device=dev),
                   n_frames=torch.empty(1, dtype=torch.int64, device=dev), total=torch.empty(1, dtype=torch.int64, device=dev),
                   pair_status=torch.empty((self.P, self.G), dtype=torch.int32, device=dev))
        spec = _lib.AppendPackSpec(me, append_variant, msg_chunk_size, 1 if full_copy else 0, 1 if heartbeat else 0, 0)
        p = lambda x: None if x is None else x.data_ptr()
        check(self.lib.ss_frame_append_pack_dev(self.h, C.byref(spec), p(want_end), p(out), out.numel() if out_capacity is None else out_capacity,
                                                p(res["frame_off"]), p(res["frame_len"]), p(res["frame_group"]), p(res["frame_peer"]),
                                                max_frames, p(res["n_frames"]), p(res["pair_status"]), p(res["total"])))
        return res

    def backoff(self, buf: torch.Tensor, frame_off: torch.Tensor, frame_group: torch.Tensor, frame_peer: torch.Tensor,
                rec_kind: torch.Tensor, reply_variant: int = 1) -> torch.Tensor:
        """The conflict replies among the frames append_reply_parse took (with its rec_kind): next_slot and try_next walk
        back.  Returns want_end (int64 [P, G], -1 = no resend), which pack_append(want_end=...) takes."""
        assert buf.dtype == torch.uint8 and frame_off.dtype == torch.int64 and frame_group.dtype == torch.int32
        assert frame_peer.dtype == torch.uint8 and rec_kind.dtype == torch.int32
        want_end = torch.empty((self.P, self.G), dtype=torch.int64, device=self.dev)
        check(self.lib.ss_engine_craft_backoff(self.h, buf.data_ptr(), buf.numel(), frame_off.data_ptr(), frame_group.data_ptr(),
                                               frame_peer.data_ptr(), rec_kind.data_ptr(), frame_off.numel(), reply_variant,
                                               want_end.data_ptr()))
        return want_end

    def advance_log(self, upto: torch.Tensor) -> None:
        """log_start moves towards upto (int64 [G]), never past min(last_snap, last_commit)."""
        assert upto.is_cuda and upto.dtype == torch.int64 and upto.numel() == self.G
        check(self.lib.ss_engine_craft_advance(self.h, upto.data_ptr()))

    def set_full_copy(self, on: bool) -> None:
        """The commit threshold of the next tick: majority when on, majority + fault_tolerance when off."""
        check(self.lib.ss_engine_craft_set_full_copy(self.h, 1 if on else 0))
        check(self.lib.ss_engine_view_get(self.h, C.byref(self.view)))
        self.threshold = self.view.threshold

    def exec_view(self) -> dict:
        """Takes the log into use and returns last_exec int64 [G] (zero-copy)."""
        v = _lib.CraftExecView()
        check(self.lib.ss_engine_craft_exec_view_get(self.h, C.byref(v)))
        return dict(last_exec=self._tensor(v.last_exec, (self.G,), "<i8", torch.int64))

    def execute(self, out: torch.Tensor, rec_capacity: int, out_capacity: Optional[int] = None) -> dict:
        """Executes the committed entries from last_exec + 1: payloads into out (uint8, 16-byte aligned, one
        round_up(data_len, 16) region each).  Returns device tensors rec_group (int32), rec_slot, rec_off (int64),
        rec_len (int32), each [rec_capacity], and totals (int64 [2]: records and bytes asked for)."""
        return _execute(self.lib.ss_engine_craft_execute, self.h, out, rec_capacity, out_capacity)

    # ---- fail-over: step-up from this replica's follower, reconstruct reads, absorbing the replies ----
    def recon_view(self) -> dict:
        """Takes the log into use and returns zero-copy views: held int32 [G, W] (shard masks) and last_recon int64 [G]."""
        v = _lib.CraftReconView()
        check(self.lib.ss_engine_craft_recon_view_get(self.h, C.byref(v)))
        return dict(held=self._tensor(v.held, (self.G, self.W), "<i4", torch.int32),
                    last_recon=self._tensor(v.last_recon, (self.G,), "<i8", torch.int64))

    def step_up(self, follower: "Follower", groups: torch.Tensor, term: torch.Tensor, store: torch.Tensor) -> dict:
        """The log half of become_the_leader for the listed groups (int32 [n]) in term (int64 [n]), taken from this
        replica's follower; the entries' shards go into store (uint8 [T, plane_stride], caller-owned, alive while the
        entries are).  Returns device tensors shard_off (int64 [n], -1 = not stepped up), verdict (int32 [n]) and need
        (int64 [1])."""
        assert groups.dtype == torch.int32 and term.dtype == torch.int64 and groups.numel() == term.numel()
        assert store.dtype == torch.uint8 and store.dim() == 2 and store.is_contiguous()
        n, dev = groups.numel(), self.dev
        out = dict(shard_off=torch.empty(n, dtype=torch.int64, device=dev), verdict=torch.empty(n, dtype=torch.int32, device=dev),
                   need=torch.empty(1, dtype=torch.int64, device=dev))
        p = lambda x: x.data_ptr()
        check(self.lib.ss_engine_craft_step_up(self.h, follower.h, p(groups), n, p(term), p(store), store.shape[1], p(out["shard_off"]),
                                               p(out["need"]), p(out["verdict"])))
        return out

    # ---- step-down: check_term for the groups this engine leads ----
    def role_view(self) -> dict:
        """Takes the log into use and returns a zero-copy view: led uint8 [G] (1: this engine leads the group; every byte set
        on first use).  Clearing a byte fences the group from propose, pack, execute and reconstruct_reads."""
        v = _lib.CraftRoleView()
        check(self.lib.ss_engine_craft_role_view_get(self.h, C.byref(v)))
        return dict(led=self._tensor(v.led, (self.G,), "|u1", torch.uint8))

    def step_down(self, follower: "Follower", buf: torch.Tensor, frame_off: torch.Tensor, frame_group: torch.Tensor,
                  frame_peer: torch.Tensor, store: torch.Tensor, store_capacity: Optional[int] = None, append_variant: int = 0,
                  append_reply_variant: int = 1, request_vote_variant: int = 2, vote_reply_variant: int = 3) -> dict:
        """check_term over a batch of incoming frames (taken as Follower.append takes frames) before their handlers run:
        the first higher-term frame of a led group deposes it, and the engine's log goes back to this replica's follower,
        the entries it lacks copied into store (uint8, 16-byte aligned, alive while the entries are).  Returns device
        tensors store_off (int64 [n], -1 = no region), meta (uint8 [n, 32]) and meta_len, verdict (int32 [n]) and need
        (int64 [1])."""
        assert buf.dtype == torch.uint8 and frame_off.dtype == torch.int64 and frame_group.dtype == torch.int32
        assert frame_peer.dtype == torch.uint8 and store.dtype == torch.uint8
        n, dev = frame_off.numel(), buf.device
        out = dict(store_off=torch.empty(n, dtype=torch.int64, device=dev), meta=torch.zeros((n, 32), dtype=torch.uint8, device=dev),
                   meta_len=torch.empty(n, dtype=torch.int32, device=dev), verdict=torch.empty(n, dtype=torch.int32, device=dev),
                   need=torch.empty(1, dtype=torch.int64, device=dev))
        spec = _lib.StepDownSpec(append_variant, append_reply_variant, request_vote_variant, vote_reply_variant)
        p = lambda x: x.data_ptr()
        check(self.lib.ss_engine_craft_step_down(self.h, follower.h, C.byref(spec), p(buf), buf.numel(), p(frame_off), p(frame_group),
                                                 p(frame_peer), n, p(store), store.numel() if store_capacity is None else store_capacity,
                                                 p(out["store_off"]), p(out["meta"]), p(out["meta_len"]), p(out["verdict"]),
                                                 p(out["need"])))
        return out

    def reconstruct_reads(self, out: torch.Tensor, frame_capacity: int, chunk_size: int, groups: Optional[torch.Tensor] = None,
                          out_capacity: Optional[int] = None, reconstruct_variant: int = 4) -> dict:
        """Reconstruct{slots: Vec<(slot, term)>} frames for the committed entries past last_recon holding fewer than d
        shards, each to be broadcast.  Outputs as Acceptor.step_up_reads()."""
        assert out.dtype == torch.uint8 and (groups is None or groups.dtype == torch.int32)
        dev, cap = out.device, max(frame_capacity, 1)
        res = dict(frame_group=torch.empty(cap, dtype=torch.int32, device=dev), frame_dst=torch.empty(cap, dtype=torch.uint8, device=dev),
                   frame_off=torch.empty(cap, dtype=torch.int64, device=dev), frame_len=torch.empty(cap, dtype=torch.int32, device=dev),
                   totals=torch.empty(2, dtype=torch.int64, device=dev))
        p = lambda x: None if x is None else x.data_ptr()
        check(self.lib.ss_engine_craft_reconstruct_reads(self.h, p(groups), 0 if groups is None else groups.numel(), chunk_size,
                                                         reconstruct_variant, p(out), out.numel() if out_capacity is None else out_capacity,
                                                         p(res["frame_group"]), p(res["frame_dst"]), p(res["frame_off"]),
                                                         p(res["frame_len"]), frame_capacity, p(res["totals"])))
        return res

    def absorb(self, buf: torch.Tensor, frame_off: torch.Tensor, frame_group: torch.Tensor, frame_peer: torch.Tensor,
               reply_variant: int = 5) -> dict:
        """Absorbs ReconstructReply frames into the slots step_up reserved.  Returns device tensors absorbed (int32: entries
        of each frame that added shards) and verdict (int32)."""
        assert buf.dtype == torch.uint8 and frame_off.dtype == torch.int64 and frame_group.dtype == torch.int32
        assert frame_peer.dtype == torch.uint8
        n, dev = frame_off.numel(), buf.device
        res = dict(absorbed=torch.empty(n, dtype=torch.int32, device=dev), verdict=torch.empty(n, dtype=torch.int32, device=dev))
        p = lambda x: x.data_ptr()
        check(self.lib.ss_engine_craft_absorb(self.h, p(buf), buf.numel(), p(frame_off), p(frame_group), p(frame_peer), n, reply_variant,
                                              p(res["absorbed"]), p(res["verdict"])))
        return res


class Acceptor:
    """The follower side of the RSPaxos / Crossword accept path for G groups (ss_acceptor_* in include/summerset_b200.h).
    State tensors are zero-copy views of the acceptor's device arrays; per-slot arrays are rings (slot s at s & 63)."""

    REPLY_CELL = 48

    def __init__(self, ctx: Context, protocol: str, n_groups: int, population: int, me: int, data_shards: int, total_shards: int,
                 accept_variant: int = 2, wal_variant: int = 1, reply_variant: int = 3):
        assert protocol in ("rspaxos", "crossword")
        self.ctx, self.lib, self.G = ctx, ctx.lib, n_groups
        self.protocol, self.n, self.me, self.d, self.T = protocol, population, me, data_shards, total_shards
        cfg = _lib.AcceptorConfig(_PROTO[protocol], population, me, data_shards, total_shards, accept_variant, wal_variant,
                                  reply_variant)
        h = C.c_void_p()
        check(self.lib.ss_acceptor_create(ctx.h, C.byref(cfg), n_groups, C.byref(h)))
        self.h = h
        v = self.view = _lib.AcceptorView()
        check(self.lib.ss_acceptor_view_get(self.h, C.byref(v)))
        self.dev = torch.device("cuda", ctx.device)
        G = n_groups
        t = lambda ptr, shape, ts, dt: None if not ptr else torch.as_tensor(_DevArray(ptr, shape, ts), device=self.dev).view(dt).view(shape)
        self.window_base = t(v.window_base, (G,), "<i8", torch.int64)
        self.bal_max_seen = t(v.bal_max_seen, (G,), "<i8", torch.int64)
        self.inst_bal = t(v.inst_bal, (G * 64,), "<i8", torch.int64)
        self.accepting = t(v.accepting, (G,), "<i8", torch.int64)
        self.shard_addr = t(v.shard_addr, (G * 64,), "<i8", torch.int64)
        self.held = t(v.held, (G * 64,), "<i4", torch.int32)
        self.data_len = t(v.data_len, (G * 64,), "<i4", torch.int32)
        self.assignment = t(v.assignment, (G * 64,), "<i4", torch.int32)
        self.source = t(v.source, (G * 64,), "|u1", torch.uint8)
        cv = self.commit_view = _lib.AcceptorCommitView()
        check(self.lib.ss_acceptor_commit_view_get(self.h, C.byref(cv)))
        self.committed = t(cv.committed, (G,), "<i8", torch.int64)
        self.commit_bar = t(cv.commit_bar, (G,), "<i8", torch.int64)
        self.exec_bar = t(cv.exec_bar, (G,), "<i8", torch.int64)
        pv = self.prepare_view = _lib.AcceptorPrepareView()
        check(self.lib.ss_acceptor_prepare_view_get(self.h, C.byref(pv)))
        self.preparing = t(pv.preparing, (G,), "<i8", torch.int64)
        self.voted_bal = t(pv.voted_bal, (G * 64,), "<i8", torch.int64)
        self.voted_mask = t(pv.voted_mask, (G * 64,), "<i4", torch.int32)
        self.prep_trigger = t(pv.prep_trigger, (G * 64,), "<i8", torch.int64)
        self.prep_span = t(pv.prep_span, (G * 64,), "|u1", torch.uint8)
        gv = self.gossip_view = _lib.AcceptorGossipView()
        check(self.lib.ss_acceptor_gossip_view_get(self.h, C.byref(gv)))
        self.assign_rows = t(gv.assign_rows, (G * 64 * population,), "<i4", torch.int32)
        self.gossip_bar = t(gv.gossip_bar, (G,), "<i8", torch.int64)

    def accept(self, buf: torch.Tensor, frame_off: torch.Tensor, frame_group: torch.Tensor, frame_peer: torch.Tensor,
               store: torch.Tensor, wal: torch.Tensor, store_capacity: Optional[int] = None, wal_capacity: Optional[int] = None) -> dict:
        """buf uint8 (frames at any alignment), frame_off int64 [n], frame_group int32 [n], frame_peer uint8 [n]; store / wal:
        caller-owned uint8 buffers (16-byte aligned).  Returns the per-frame outputs as device tensors: store_off, wal_off
        (int64, -1 = not accepted), wal_len, reply_len, verdict (int32), reply_dst (uint8), replies (uint8 [n, 48]) and
        totals (int64 [2]: store and WAL bytes asked for)."""
        assert buf.dtype == torch.uint8 and frame_off.dtype == torch.int64 and frame_group.dtype == torch.int32
        assert frame_peer.dtype == torch.uint8 and store.dtype == torch.uint8 and wal.dtype == torch.uint8
        n, dev = frame_off.numel(), buf.device
        e = lambda dt, *shape: torch.empty(shape if shape else (n,), dtype=dt, device=dev)
        out = dict(store_off=e(torch.int64), wal_off=e(torch.int64), wal_len=e(torch.int32),
                   replies=torch.zeros((n, self.REPLY_CELL), dtype=torch.uint8, device=dev), reply_len=e(torch.int32),
                   reply_dst=e(torch.uint8), verdict=e(torch.int32), totals=e(torch.int64, 2))
        p = lambda x: x.data_ptr()
        check(self.lib.ss_acceptor_accept(self.h, p(buf), buf.numel(), p(frame_off), p(frame_group), p(frame_peer), n, p(store),
                                          store.numel() if store_capacity is None else store_capacity, p(out["store_off"]), p(wal),
                                          wal.numel() if wal_capacity is None else wal_capacity, p(out["wal_off"]), p(out["wal_len"]),
                                          p(out["replies"]), p(out["reply_len"]), p(out["reply_dst"]), p(out["verdict"]),
                                          p(out["totals"])))
        return out

    def advance(self, upto: torch.Tensor) -> None:
        """Retires window prefixes up to the absolute slots upto (int64 [G])."""
        assert upto.is_cuda and upto.dtype == torch.int64 and upto.numel() == self.G
        check(self.lib.ss_acceptor_advance(self.h, upto.data_ptr()))

    def heartbeat(self, group: torch.Tensor, peer: torch.Tensor, ballot: torch.Tensor, commit_bar: torch.Tensor,
                  exec_bar: torch.Tensor) -> torch.Tensor:
        """Heartbeat records group int32 [n], peer uint8 [n], ballot / commit_bar / exec_bar int64 [n] (heard_heartbeat's
        commit half, per group in record order).  Returns newly (int64 [G], window order): the instances this call
        committed, which ss_wal_commit_pack_dev packs as CommitSlot records with window_base."""
        assert group.dtype == torch.int32 and peer.dtype == torch.uint8
        assert ballot.dtype == commit_bar.dtype == exec_bar.dtype == torch.int64
        n = group.numel()
        assert peer.numel() == ballot.numel() == commit_bar.numel() == exec_bar.numel() == n
        newly = torch.empty(self.G, dtype=torch.int64, device=self.dev)
        check(self.lib.ss_acceptor_heartbeat(self.h, group.data_ptr(), peer.data_ptr(), ballot.data_ptr(), commit_bar.data_ptr(),
                                             exec_bar.data_ptr(), n, newly.data_ptr()))
        return newly

    def execute(self, out: torch.Tensor, rec_capacity: int, out_capacity: Optional[int] = None) -> dict:
        """Executes the committed instances handle_logged_commit_slot would: payloads into out (uint8, 16-byte aligned,
        one round_up(data_len, 16) region each).  Returns device tensors rec_group (int32), rec_slot, rec_off (int64),
        rec_len (int32), each [rec_capacity], and totals (int64 [2]: records and bytes asked for)."""
        return _execute(self.lib.ss_acceptor_execute, self.h, out, rec_capacity, out_capacity)

    def reconstruct_serve(self, buf: torch.Tensor, frame_off: torch.Tensor, frame_group: torch.Tensor, frame_peer: torch.Tensor,
                          out: torch.Tensor, out_capacity: Optional[int] = None, reconstruct_variant: int = 4,
                          reply_variant: int = 5) -> dict:
        """Serves Reconstruct frames (handle_msg_reconstruct) from the held shards: ReconstructReply frames into out
        (uint8, 16-byte aligned, one round_up(reply_len, 16) region per frame with a reply, packed in frame order).
        Returns device tensors reply_off (int64, -1 = no reply), reply_len (int64, 0 = nothing to send), verdict (int32)
        and total (int64 [1]: the bytes the batch asked for); reply i goes to frame_peer[i]."""
        assert buf.dtype == torch.uint8 and frame_off.dtype == torch.int64 and frame_group.dtype == torch.int32
        assert frame_peer.dtype == torch.uint8 and out.dtype == torch.uint8
        n, dev = frame_off.numel(), buf.device
        res = dict(reply_off=torch.empty(n, dtype=torch.int64, device=dev), reply_len=torch.empty(n, dtype=torch.int64, device=dev),
                   verdict=torch.empty(n, dtype=torch.int32, device=dev), total=torch.empty(1, dtype=torch.int64, device=dev))
        p = lambda x: x.data_ptr()
        check(self.lib.ss_acceptor_reconstruct_serve(self.h, p(buf), buf.numel(), p(frame_off), p(frame_group), p(frame_peer), n,
                                                     reconstruct_variant, reply_variant, p(out),
                                                     out.numel() if out_capacity is None else out_capacity, p(res["reply_off"]),
                                                     p(res["reply_len"]), p(res["verdict"]), p(res["total"])))
        return res

    def absorb(self, buf: torch.Tensor, frame_off: torch.Tensor, frame_group: torch.Tensor, frame_peer: torch.Tensor,
               store: torch.Tensor, store_capacity: Optional[int] = None, reply_variant: int = 5) -> dict:
        """Absorbs ReconstructReply frames (handle_msg_reconstruct_reply): every instance that gains shards moves to a new
        region of store (uint8, 16-byte aligned, caller-owned; keep it alive while the instances hold it).  Returns
        device tensors absorbed (int32: entries of each frame that added shards), verdict (int32) and total (int64 [1]:
        the store bytes the batch asked for).  ss_acceptor_execute then runs what now holds d shards."""
        assert buf.dtype == torch.uint8 and frame_off.dtype == torch.int64 and frame_group.dtype == torch.int32
        assert frame_peer.dtype == torch.uint8 and store.dtype == torch.uint8
        n, dev = frame_off.numel(), buf.device
        res = dict(absorbed=torch.empty(n, dtype=torch.int32, device=dev), verdict=torch.empty(n, dtype=torch.int32, device=dev),
                   total=torch.empty(1, dtype=torch.int64, device=dev))
        p = lambda x: x.data_ptr()
        check(self.lib.ss_acceptor_absorb(self.h, p(buf), buf.numel(), p(frame_off), p(frame_group), p(frame_peer), n, reply_variant,
                                          p(store), store.numel() if store_capacity is None else store_capacity, p(res["absorbed"]),
                                          p(res["verdict"]), p(res["total"])))
        return res

    def prepare(self, buf: torch.Tensor, frame_off: torch.Tensor, frame_group: torch.Tensor, frame_peer: torch.Tensor,
                wal: torch.Tensor, rec_capacity: int, wal_capacity: Optional[int] = None, prepare_variant: int = 0,
                wal_variant: int = 0) -> dict:
        """Takes Prepare frames (handle_msg_prepare): the covered slots become Preparing at the frame's ballot.  wal: uint8,
        16-byte aligned, one 32-byte PrepareBal cell per record.  Returns device tensors rec_group (int32), rec_slot (int64),
        rec_frame (int32), each [rec_capacity], verdict (int32 [n]) and totals (int64 [2]: records and WAL bytes asked for)."""
        assert buf.dtype == torch.uint8 and frame_off.dtype == torch.int64 and frame_group.dtype == torch.int32
        assert frame_peer.dtype == torch.uint8 and wal.dtype == torch.uint8
        n, dev = frame_off.numel(), buf.device
        cap = max(rec_capacity, 1)
        res = dict(rec_group=torch.empty(cap, dtype=torch.int32, device=dev), rec_slot=torch.empty(cap, dtype=torch.int64, device=dev),
                   rec_frame=torch.empty(cap, dtype=torch.int32, device=dev), verdict=torch.empty(n, dtype=torch.int32, device=dev),
                   totals=torch.empty(2, dtype=torch.int64, device=dev))
        p = lambda x: x.data_ptr()
        check(self.lib.ss_acceptor_prepare(self.h, p(buf), buf.numel(), p(frame_off), p(frame_group), p(frame_peer), n, prepare_variant,
                                           wal_variant, p(wal), wal.numel() if wal_capacity is None else wal_capacity, p(res["rec_group"]),
                                           p(res["rec_slot"]), p(res["rec_frame"]), rec_capacity, p(res["verdict"]), p(res["totals"])))
        return res

    def prepare_reply(self, rec_group: torch.Tensor, rec_slot: torch.Tensor, out: torch.Tensor, out_capacity: Optional[int] = None,
                      reply_variant: int = 1) -> dict:
        """PrepareReply frames for durable PrepareBal records (handle_logged_prepare_bal, follower branch), read from the
        instances' state now: into out (uint8, 16-byte aligned, round_up(reply_len, 16) regions packed in record order).
        Returns device tensors reply_off (int64, -1 = not written), reply_len (int64, 0 = no reply), reply_dst (uint8) and
        total (int64 [1]: the bytes the batch asked for)."""
        assert rec_group.dtype == torch.int32 and rec_slot.dtype == torch.int64 and out.dtype == torch.uint8
        n, dev = rec_group.numel(), out.device
        res = dict(reply_off=torch.empty(n, dtype=torch.int64, device=dev), reply_len=torch.empty(n, dtype=torch.int64, device=dev),
                   reply_dst=torch.empty(n, dtype=torch.uint8, device=dev), total=torch.empty(1, dtype=torch.int64, device=dev))
        p = lambda x: x.data_ptr()
        check(self.lib.ss_acceptor_prepare_reply(self.h, p(rec_group), p(rec_slot), n, reply_variant, p(out),
                                                 out.numel() if out_capacity is None else out_capacity, p(res["reply_off"]),
                                                 p(res["reply_len"]), p(res["reply_dst"]), p(res["total"])))
        return res

    def recover(self, buf: torch.Tensor, rec_off: torch.Tensor, rec_group: torch.Tensor, store: torch.Tensor,
                store_capacity: Optional[int] = None, prepare_variant: int = 0, commit_variant: int = 2) -> dict:
        """Replays WAL records (recover_apply_entry): buf uint8 holds PrepareBal, AcceptData and CommitSlot records as the
        device wrote them (8-byte big-endian length + bincode WalEntry, any alignment), record i at rec_off[i] (int64) of
        group rec_group[i] (int32), each group's records in WAL order.  The defining AcceptData shards go to store (uint8,
        16-byte aligned, caller-owned; keep it alive while the instances hold it).  Returns device tensors verdict (int32
        [n]) and total (int64 [1]: the store bytes the batch asked for)."""
        assert buf.dtype == torch.uint8 and rec_off.dtype == torch.int64 and rec_group.dtype == torch.int32
        assert store.dtype == torch.uint8 and rec_group.numel() == rec_off.numel()
        n, dev = rec_off.numel(), buf.device
        res = dict(verdict=torch.empty(n, dtype=torch.int32, device=dev), total=torch.empty(1, dtype=torch.int64, device=dev))
        p = lambda x: x.data_ptr()
        check(self.lib.ss_acceptor_recover(self.h, p(buf), buf.numel(), p(rec_off), p(rec_group), n, prepare_variant, commit_variant,
                                           p(store), store.numel() if store_capacity is None else store_capacity, p(res["verdict"]),
                                           p(res["total"])))
        return res

    def _requests(self, step_up: bool, out: torch.Tensor, frame_capacity: int, groups: Optional[torch.Tensor], batch: int,
                  out_capacity: Optional[int], reconstruct_variant: int, peer_alive: Optional[torch.Tensor] = None,
                  tail_ignores: int = 0) -> dict:
        assert out.dtype == torch.uint8
        assert groups is None or groups.dtype == torch.int32
        assert peer_alive is None or (peer_alive.dtype == torch.int32 and peer_alive.numel() == self.G)
        dev = out.device
        cap = max(frame_capacity, 1)
        res = dict(frame_group=torch.empty(cap, dtype=torch.int32, device=dev), frame_dst=torch.empty(cap, dtype=torch.uint8, device=dev),
                   frame_off=torch.empty(cap, dtype=torch.int64, device=dev), frame_len=torch.empty(cap, dtype=torch.int32, device=dev),
                   totals=torch.empty(2, dtype=torch.int64, device=dev))
        p = lambda x: None if x is None else x.data_ptr()
        oc = out.numel() if out_capacity is None else out_capacity
        gp, n = p(groups), 0 if groups is None else groups.numel()
        if step_up:
            check(self.lib.ss_acceptor_step_up_reads(self.h, gp, n, batch, reconstruct_variant, p(out), oc, p(res["frame_group"]),
                                                     p(res["frame_dst"]), p(res["frame_off"]), p(res["frame_len"]), frame_capacity,
                                                     p(res["totals"])))
        else:
            check(self.lib.ss_acceptor_gossip(self.h, gp, n, p(peer_alive), tail_ignores, batch, reconstruct_variant, p(out), oc,
                                              p(res["frame_group"]), p(res["frame_dst"]), p(res["frame_off"]), p(res["frame_len"]),
                                              frame_capacity, p(res["totals"])))
        return res

    def gossip(self, out: torch.Tensor, frame_capacity: int, batch_size: int, groups: Optional[torch.Tensor] = None,
               peer_alive: Optional[torch.Tensor] = None, tail_ignores: int = 0, out_capacity: Optional[int] = None,
               reconstruct_variant: int = 4) -> dict:
        """Crossword follower gossip (trigger_gossiping) over the listed groups (int32, None = all): Reconstruct{slots_excl}
        frames into out (uint8, 16-byte aligned), ordered by (listed group, peer, chunk); gossip_bar moves for the groups
        placed.  peer_alive: int32 [G] peer masks (None = all alive).  Returns device tensors frame_group (int32),
        frame_dst (uint8), frame_off (int64, -1 = not written), frame_len (int32), each [frame_capacity], and totals
        (int64 [2]: frames and bytes asked for)."""
        return self._requests(False, out, frame_capacity, groups, batch_size, out_capacity, reconstruct_variant, peer_alive, tail_ignores)

    def step_up_reads(self, out: torch.Tensor, frame_capacity: int, chunk_size: int, groups: Optional[torch.Tensor] = None,
                      out_capacity: Optional[int] = None, reconstruct_variant: int = 4) -> dict:
        """The reconstruct reads of become_a_leader over the listed groups: Reconstruct frames of chunk_size entries for
        every committed instance holding fewer than d shards, each to be broadcast (frame_dst 0xff).  Outputs as gossip();
        no state changes."""
        return self._requests(True, out, frame_capacity, groups, chunk_size, out_capacity, reconstruct_variant)

    def step_up(self, wal: torch.Tensor, rec_capacity: int, out: torch.Tensor, frame_capacity: int,
                groups: Optional[torch.Tensor] = None, wal_capacity: Optional[int] = None, out_capacity: Optional[int] = None,
                prepare_variant: int = 0, wal_variant: int = 0) -> dict:
        """The Prepare half of become_a_leader over the listed groups (int32, None = all): a greater ballot, the
        in-progress instances Preparing with source = me, one 32-byte PrepareBal cell per marked slot into wal and one
        32-byte Prepare frame per group into out (uint8, 16-byte aligned), each to be broadcast.  Returns device tensors
        rec_group (int32), rec_slot (int64), each [rec_capacity]; frame_group (int32), frame_dst (uint8), frame_off (int64,
        -1 = not written), frame_len (int32), each [frame_capacity]; verdict (int32), ballot, trigger_slot, endprep_slot
        (int64), each [n]; totals (int64 [4]: records, WAL bytes, frames, frame bytes asked for).  Once the records are
        durable, prepare_reply(rec_group, rec_slot) gives the leader's own votes (reply_dst = me)."""
        assert wal.dtype == torch.uint8 and out.dtype == torch.uint8
        assert groups is None or groups.dtype == torch.int32
        dev = out.device
        n = self.G if groups is None else groups.numel()
        rc, fc, m = max(rec_capacity, 1), max(frame_capacity, 1), max(n, 1)
        e = lambda k, dt: torch.empty(k, dtype=dt, device=dev)
        res = dict(rec_group=e(rc, torch.int32), rec_slot=e(rc, torch.int64), frame_group=e(fc, torch.int32),
                   frame_dst=e(fc, torch.uint8), frame_off=e(fc, torch.int64), frame_len=e(fc, torch.int32), verdict=e(m, torch.int32),
                   ballot=e(m, torch.int64), trigger_slot=e(m, torch.int64), endprep_slot=e(m, torch.int64), totals=e(4, torch.int64))
        p = lambda x: None if x is None else x.data_ptr()
        check(self.lib.ss_acceptor_step_up(self.h, p(groups), 0 if groups is None else n, prepare_variant, wal_variant, p(wal),
                                           wal.numel() if wal_capacity is None else wal_capacity, p(res["rec_group"]),
                                           p(res["rec_slot"]), rec_capacity, p(out), out.numel() if out_capacity is None else out_capacity,
                                           p(res["frame_group"]), p(res["frame_dst"]), p(res["frame_off"]), p(res["frame_len"]),
                                           frame_capacity, p(res["verdict"]), p(res["ballot"]), p(res["trigger_slot"]),
                                           p(res["endprep_slot"]), p(res["totals"])))
        return res

    def close(self) -> None:
        if getattr(self, "h", None) is not None and self.h:
            self.lib.ss_acceptor_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


PREPARE_REPLY_REC = 64      # sizeof(ss_prepare_reply_rec)


def prepare_reply_parse(ctx: Context, buf: torch.Tensor, frame_off: torch.Tensor, data_shards: int, total_shards: int,
                        reply_variant: int = 1) -> dict:
    """PrepareReply frames (buf uint8 at any alignment, frame_off int64 [n]) -> one ss_prepare_reply_rec per frame, as
    device tensors: slot, trigger_slot, endprep_slot, ballot, vote_bal, shards_at (int64; -1 = voted None), vote_mask,
    data_len, kind (int32).  The new leader scatters vote_bal / vote_mask into ss_prepare_merge_dev's [r*N + i] arrays."""
    assert buf.dtype == torch.uint8 and frame_off.dtype == torch.int64
    n = frame_off.numel()
    rec = torch.empty((n, PREPARE_REPLY_REC), dtype=torch.uint8, device=buf.device)
    check(ctx.lib.ss_prepare_reply_parse_dev(ctx.h, buf.data_ptr(), buf.numel(), frame_off.data_ptr(), n, data_shards, total_shards,
                                             reply_variant, rec.data_ptr()))
    q, w = rec.view(torch.int64), rec.view(torch.int32)
    names = ("slot", "trigger_slot", "endprep_slot", "ballot", "vote_bal", "shards_at")
    out = {k: q[:, j] for j, k in enumerate(names)}
    out.update(vote_mask=w[:, 12], data_len=w[:, 13], kind=w[:, 14])
    return out


class Follower:
    """The CRaft follower for G groups (ss_follower_* in include/summerset_b200.h): AppendEntries frames in, LogEntry and
    Metadata records and AppendEntriesReply cells out.  State tensors are zero-copy views of the follower's device arrays;
    per-position arrays are rings of `window` entries (slot s at s & (window - 1))."""

    REPLY_CELL = 48
    META_CELL = 32
    VOTE_CELL = 48              # RequestVote frames of campaign()
    VOTE_REPLY_CELL = 32        # RequestVoteReply frames of vote()

    def __init__(self, ctx: Context, n_groups: int, population: int, me: int, window: int = 0, append_variant: int = 0,
                 reply_variant: int = 1, meta_variant: int = 0, log_variant: int = 1):
        self.ctx, self.lib, self.G = ctx, ctx.lib, n_groups
        cfg = _lib.FollowerConfig(_PROTO["craft"], population, me, window, append_variant, reply_variant, meta_variant, log_variant)
        h = C.c_void_p()
        check(self.lib.ss_follower_create(ctx.h, C.byref(cfg), n_groups, C.byref(h)))
        self.h = h
        v = self.view = _lib.FollowerView()
        check(self.lib.ss_follower_view_get(self.h, C.byref(v)))
        self.dev = torch.device("cuda", ctx.device)
        self.n, self.me, self.d, self.T, self.W = population, me, v.data_shards, v.total_shards, v.window
        G, W = n_groups, v.window
        t = lambda ptr, shape, ts, dt: torch.as_tensor(_DevArray(ptr, shape, ts), device=self.dev).view(dt).view(shape)
        self.start_slot = t(v.start_slot, (G,), "<i8", torch.int64)
        self.log_end = t(v.log_end, (G,), "<i8", torch.int64)
        self.curr_term = t(v.curr_term, (G,), "<i8", torch.int64)
        self.last_commit = t(v.last_commit, (G,), "<i8", torch.int64)
        self.last_snap = t(v.last_snap, (G,), "<i8", torch.int64)
        self.leader = t(v.leader, (G,), "|u1", torch.uint8)
        self.term = t(v.term, (G, W), "<i8", torch.int64)
        self.shard_addr = t(v.shard_addr, (G, W), "<i8", torch.int64)
        self.held = t(v.held, (G, W), "<i4", torch.int32)
        self.data_len = t(v.data_len, (G, W), "<i4", torch.int32)
        ev = self.exec_view = _lib.FollowerExecView()
        check(self.lib.ss_follower_exec_view_get(self.h, C.byref(ev)))
        self.last_exec = t(ev.last_exec, (G,), "<i8", torch.int64)

    def append(self, buf: torch.Tensor, frame_off: torch.Tensor, frame_group: torch.Tensor, frame_peer: torch.Tensor,
               store: torch.Tensor, wal: torch.Tensor, store_capacity: Optional[int] = None,
               wal_capacity: Optional[int] = None) -> dict:
        """buf uint8 (frames at any alignment), frame_off int64 [n], frame_group int32 [n], frame_peer uint8 [n]; store / wal:
        caller-owned uint8 buffers (16-byte aligned).  Returns the per-frame outputs as device tensors: store_off, wal_off,
        wal_len, trunc_slot (int64, -1 = none), meta (uint8 [n, 32]) and meta_len, replies (uint8 [n, 48]) and reply_len,
        reply_dst (uint8), verdict (int32), commit_lo (int64 [G]) and totals (int64 [2])."""
        assert buf.dtype == torch.uint8 and frame_off.dtype == torch.int64 and frame_group.dtype == torch.int32
        assert frame_peer.dtype == torch.uint8 and store.dtype == torch.uint8 and wal.dtype == torch.uint8
        n, dev = frame_off.numel(), buf.device
        e = lambda dt, *shape: torch.empty(shape if shape else (n,), dtype=dt, device=dev)
        out = dict(store_off=e(torch.int64), wal_off=e(torch.int64), wal_len=e(torch.int64),
                   meta=torch.zeros((n, self.META_CELL), dtype=torch.uint8, device=dev), meta_len=e(torch.int32),
                   replies=torch.zeros((n, self.REPLY_CELL), dtype=torch.uint8, device=dev), reply_len=e(torch.int32),
                   reply_dst=e(torch.uint8), trunc_slot=e(torch.int64), verdict=e(torch.int32), commit_lo=e(torch.int64, self.G),
                   totals=e(torch.int64, 2))
        p = lambda x: x.data_ptr()
        check(self.lib.ss_follower_append(self.h, p(buf), buf.numel(), p(frame_off), p(frame_group), p(frame_peer), n, p(store),
                                          store.numel() if store_capacity is None else store_capacity, p(out["store_off"]), p(wal),
                                          wal.numel() if wal_capacity is None else wal_capacity, p(out["wal_off"]), p(out["wal_len"]),
                                          p(out["meta"]), p(out["meta_len"]), p(out["replies"]), p(out["reply_len"]),
                                          p(out["reply_dst"]), p(out["trunc_slot"]), p(out["verdict"]), p(out["commit_lo"]),
                                          p(out["totals"])))
        return out

    def advance(self, upto: torch.Tensor) -> None:
        """The snapshot's start_slot move, never past last_commit (upto int64 [G], absolute slots)."""
        assert upto.is_cuda and upto.dtype == torch.int64 and upto.numel() == self.G
        check(self.lib.ss_follower_advance(self.h, upto.data_ptr()))

    def execute(self, out: torch.Tensor, rec_capacity: int, out_capacity: Optional[int] = None) -> dict:
        """Executes the committed entries from last_exec + 1, regenerating missing data shards: payloads into out
        (uint8, 16-byte aligned, one round_up(data_len, 16) region each).  Returns what Acceptor.execute returns."""
        return _execute(self.lib.ss_follower_execute, self.h, out, rec_capacity, out_capacity)

    def reconstruct_serve(self, buf: torch.Tensor, frame_off: torch.Tensor, frame_group: torch.Tensor, frame_peer: torch.Tensor,
                          out: torch.Tensor, out_capacity: Optional[int] = None, reconstruct_variant: int = 4,
                          reply_variant: int = 5) -> dict:
        """Serves a new leader's Reconstruct{slots: Vec<(slot, term)>} frames from the held shards.  Outputs as
        Acceptor.reconstruct_serve()."""
        assert buf.dtype == torch.uint8 and frame_off.dtype == torch.int64 and frame_group.dtype == torch.int32
        assert frame_peer.dtype == torch.uint8 and out.dtype == torch.uint8
        n, dev = frame_off.numel(), buf.device
        res = dict(reply_off=torch.empty(n, dtype=torch.int64, device=dev), reply_len=torch.empty(n, dtype=torch.int64, device=dev),
                   verdict=torch.empty(n, dtype=torch.int32, device=dev), total=torch.empty(1, dtype=torch.int64, device=dev))
        p = lambda x: x.data_ptr()
        check(self.lib.ss_follower_reconstruct_serve(self.h, p(buf), buf.numel(), p(frame_off), p(frame_group), p(frame_peer), n,
                                                     reconstruct_variant, reply_variant, p(out),
                                                     out.numel() if out_capacity is None else out_capacity, p(res["reply_off"]),
                                                     p(res["reply_len"]), p(res["verdict"]), p(res["total"])))
        return res

    def recover(self, buf: torch.Tensor, rec_off: torch.Tensor, rec_group: torch.Tensor, store: torch.Tensor,
                store_capacity: Optional[int] = None) -> dict:
        """Replays WAL records (recover_from_wal): buf uint8 holds DurEntry::Metadata and DurEntry::LogEntry records as the
        device wrote them (8-byte big-endian length + bincode DurEntry, any alignment), record i at rec_off[i] (int64) of
        group rec_group[i] (int32), each group's Metadata record first and the rest in WAL order.  The entries' shards go
        to store (uint8, 16-byte aligned, caller-owned; keep it alive while the log holds it).  Returns device tensors
        verdict (int32 [n]) and total (int64 [1]: the store bytes the batch asked for)."""
        assert buf.dtype == torch.uint8 and rec_off.dtype == torch.int64 and rec_group.dtype == torch.int32
        assert store.dtype == torch.uint8 and rec_group.numel() == rec_off.numel()
        n, dev = rec_off.numel(), buf.device
        res = dict(verdict=torch.empty(n, dtype=torch.int32, device=dev), total=torch.empty(1, dtype=torch.int64, device=dev))
        p = lambda x: x.data_ptr()
        check(self.lib.ss_follower_recover(self.h, p(buf), buf.numel(), p(rec_off), p(rec_group), n, p(store),
                                           store.numel() if store_capacity is None else store_capacity, p(res["verdict"]),
                                           p(res["total"])))
        return res

    # ---- elections: campaigns, RequestVote frames answered, votes tallied ----
    def vote_view(self) -> dict:
        """Takes the election state into use and returns zero-copy views: vote_term int64 [G], voted_for uint8 [G] (0xff =
        None), role_term int64 [G], role uint8 [G] (SS_FOLLOWER_ROLE_*) and votes int32 [G] (bit r = replica r).  voted_for
        counts while vote_term == curr_term, role while role_term == curr_term and leader == me."""
        v = _lib.FollowerVoteView()
        check(self.lib.ss_follower_vote_view_get(self.h, C.byref(v)))
        G = self.G
        t = lambda ptr, ts, dt: torch.as_tensor(_DevArray(ptr, (G,), ts), device=self.dev).view(dt).view((G,))
        return dict(vote_term=t(v.vote_term, "<i8", torch.int64), voted_for=t(v.voted_for, "|u1", torch.uint8),
                    role_term=t(v.role_term, "<i8", torch.int64), role=t(v.role, "|u1", torch.uint8),
                    votes=t(v.votes, "<i4", torch.int32))

    def campaign(self, groups: torch.Tensor, timeout_source: Optional[torch.Tensor] = None, request_vote_variant: int = 2) -> dict:
        """become_a_candidate for the listed groups (int32 [n]; timeout_source uint8 [n] or None = no leader check).
        Returns device tensors meta (uint8 [n, 32]) and meta_len, frames (uint8 [n, 48]: the RequestVote to broadcast) and
        frame_len, frame_dst (uint8) and verdict (int32)."""
        assert groups.dtype == torch.int32 and (timeout_source is None or timeout_source.dtype == torch.uint8)
        n, dev = groups.numel(), groups.device
        e = lambda dt: torch.empty(n, dtype=dt, device=dev)
        out = dict(meta=torch.zeros((n, self.META_CELL), dtype=torch.uint8, device=dev), meta_len=e(torch.int32),
                   frames=torch.zeros((n, self.VOTE_CELL), dtype=torch.uint8, device=dev), frame_len=e(torch.int32),
                   frame_dst=e(torch.uint8), verdict=e(torch.int32))
        p = lambda x: None if x is None else x.data_ptr()
        check(self.lib.ss_follower_campaign(self.h, p(groups), n, p(timeout_source), request_vote_variant, p(out["meta"]),
                                            p(out["meta_len"]), p(out["frames"]), p(out["frame_len"]), p(out["frame_dst"]),
                                            p(out["verdict"])))
        return out

    def vote(self, buf: torch.Tensor, frame_off: torch.Tensor, frame_group: torch.Tensor, frame_peer: torch.Tensor,
             request_vote_variant: int = 2, reply_variant: int = 3) -> dict:
        """handle_msg_request_vote over a batch of RequestVote frames (taken as append takes frames).  Returns device
        tensors meta (uint8 [n, 32]) and meta_len, replies (uint8 [n, 32]) and reply_len, reply_dst (uint8) and verdict."""
        assert buf.dtype == torch.uint8 and frame_off.dtype == torch.int64 and frame_group.dtype == torch.int32
        assert frame_peer.dtype == torch.uint8
        n, dev = frame_off.numel(), buf.device
        e = lambda dt: torch.empty(n, dtype=dt, device=dev)
        out = dict(meta=torch.zeros((n, self.META_CELL), dtype=torch.uint8, device=dev), meta_len=e(torch.int32),
                   replies=torch.zeros((n, self.VOTE_REPLY_CELL), dtype=torch.uint8, device=dev), reply_len=e(torch.int32),
                   reply_dst=e(torch.uint8), verdict=e(torch.int32))
        p = lambda x: x.data_ptr()
        check(self.lib.ss_follower_vote(self.h, p(buf), buf.numel(), p(frame_off), p(frame_group), p(frame_peer), n,
                                        request_vote_variant, reply_variant, p(out["meta"]), p(out["meta_len"]), p(out["replies"]),
                                        p(out["reply_len"]), p(out["reply_dst"]), p(out["verdict"])))
        return out

    def tally(self, buf: torch.Tensor, frame_off: torch.Tensor, frame_group: torch.Tensor, frame_peer: torch.Tensor,
              reply_variant: int = 3) -> dict:
        """handle_msg_request_vote_reply over a batch of RequestVoteReply frames.  Returns device tensors meta (uint8
        [n, 32]) and meta_len, verdict, and won_group (int32 [G], -1 past the elected groups), won_term (int64 [G]) and
        n_won (int64 [1]): pass won_group / won_term to RaftEngine.step_up."""
        assert buf.dtype == torch.uint8 and frame_off.dtype == torch.int64 and frame_group.dtype == torch.int32
        assert frame_peer.dtype == torch.uint8
        n, dev = frame_off.numel(), buf.device
        out = dict(meta=torch.zeros((n, self.META_CELL), dtype=torch.uint8, device=dev), meta_len=torch.empty(n, dtype=torch.int32, device=dev),
                   verdict=torch.empty(n, dtype=torch.int32, device=dev), won_group=torch.empty(self.G, dtype=torch.int32, device=dev),
                   won_term=torch.empty(self.G, dtype=torch.int64, device=dev), n_won=torch.empty(1, dtype=torch.int64, device=dev))
        p = lambda x: x.data_ptr()
        check(self.lib.ss_follower_tally(self.h, p(buf), buf.numel(), p(frame_off), p(frame_group), p(frame_peer), n, reply_variant,
                                         p(out["meta"]), p(out["meta_len"]), p(out["verdict"]), p(out["won_group"]),
                                         p(out["won_term"]), p(out["n_won"])))
        return out

    def close(self) -> None:
        if getattr(self, "h", None) is not None and self.h:
            self.lib.ss_follower_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def append_reply_parse(ctx: Context, buf: torch.Tensor, frame_off: torch.Tensor, frame_group: torch.Tensor,
                       frame_peer: torch.Tensor, curr_term: torch.Tensor, n_groups: int, reply_variant: int = 1) -> dict:
    """AppendEntriesReply frames -> the records RaftEngine.on_append_replies takes (rec_group, rec_peer, rec_end_slot) plus
    rec_term, rec_conflict_term, rec_conflict_slot and rec_kind (ss_append_reply_parse_dev).  curr_term: the CRaft
    engine's int32 [G] view."""
    n, dev = frame_off.numel(), buf.device
    e = lambda dt: torch.empty(n, dtype=dt, device=dev)
    out = dict(rec_group=e(torch.int32), rec_peer=e(torch.uint8), rec_end_slot=e(torch.int32), rec_term=e(torch.int64),
               rec_conflict_term=e(torch.int64), rec_conflict_slot=e(torch.int64), rec_kind=e(torch.int32))
    p = lambda x: x.data_ptr()
    check(ctx.lib.ss_append_reply_parse_dev(ctx.h, p(buf), buf.numel(), p(frame_off), p(frame_group), p(frame_peer), p(curr_term), n,
                                            n_groups, reply_variant, p(out["rec_group"]), p(out["rec_peer"]), p(out["rec_end_slot"]),
                                            p(out["rec_term"]), p(out["rec_conflict_term"]), p(out["rec_conflict_slot"]),
                                            p(out["rec_kind"])))
    return out
