"""The CRaft leader's log: ss_engine_craft_propose, ss_frame_append_pack_dev, ss_engine_craft_backoff, ss_engine_craft_advance.

`Leader` restates, per group and per message, handle_req_batch (craft/request.rs:70-116), handle_logged_leader_append
(craft/durability.rs:12-127), bcast_heartbeats (craft/leadership.rs:249-279), the conflict branch of
handle_msg_append_entries_reply (craft/messages.rs:386-406) and the start_slot move (craft/snapshot.rs:142,184), with the
engine's success-reply ingest and commit tick.  The bincode encoders and the follower's restatement come from
tests/test_follower.py.  GPU tests compare every shard, record and frame byte, every frame array and every state word of
the device leader with the restatement, and close the loop through device followers.
"""
from __future__ import annotations

import ctypes as C
import random

import numpy as np
import pytest

from oracle import pyoracle as oracle
from tests import test_follower as tf

U64 = (1 << 64) - 1
SENT, NOTHING, SNAPSHOTTED, OVERFLOW = range(4)
STATUS_RAFT_WINDOW_FULL, STATUS_FRAME_OVERFLOW, STATUS_STORE_FULL = 2, 4, 16
pitch = lambda L: (L + 31) & ~31
r16 = lambda x: (x + 15) & ~15


def encode(batch: bytes, d: int, p: int):
    """RSCodeword::from_data + compute_parity: the d + p shards of a batch"""
    data = oracle.cw_split(batch, d)
    shards = [data[i].copy() for i in range(d)] + [np.zeros(data.shape[1], dtype=np.uint8) for _ in range(p)]
    assert oracle.rs_encode(d, p, shards) == 0
    return [s.tobytes() for s in shards]


def leader_record(term, d, p, data_len, shards: dict) -> bytes:
    """DurEntry::LogEntry{LogEntry{term, reqs_cw, external: true, log_offset: 0}} behind its length"""
    return tf.framed(tf.vi(1) + tf.entry(term, d, p, data_len, shards, True, 0))


class Leader:
    """one group's CRaft leader; log[s] = [term, data_len, shards or None, log_offset] for s in [start, le)"""

    def __init__(self, n: int, me: int, W: int, threshold: int):
        self.n, self.me, self.W, self.threshold = n, me, W, threshold
        self.d, self.P = n // 2 + 1, n - 1
        self.start, self.le, self.ct, self.lc, self.ls = 0, 1, 0, 0, 0
        self.log = {0: [0, 0, None, 0]}
        self.next, self.match, self.try_next = [1] * self.P, [0] * self.P, [0] * self.P

    def replica(self, q):
        return q if q < self.me else q + 1

    def propose(self, batch: bytes, log_offset=0, full_copy=False):
        """handle_req_batch -> (slot, record), or None when the ring would hold more than W slots"""
        if self.le + 1 - self.start > self.W:
            return None
        d, p = self.d, self.n - self.d
        sh = encode(batch, d, p)
        s = self.le
        self.log[s] = [self.ct, len(batch), sh, log_offset]
        self.le += 1
        keep = range(d) if full_copy else [self.me]
        return s, leader_record(self.ct, d, p, len(batch), {j: sh[j] for j in keep})

    def ent(self, s, q, full_copy):
        t, dl, sh, lo = self.log[s]
        keep = range(self.d) if full_copy else [self.replica(q)]
        return tf.Ent(t, self.d, self.n - self.d, dl, {j: sh[j] for j in keep}, False, lo)

    def plan(self, q, chunk, want_end=None, heartbeat=False, full_copy=False, variant=0):
        """-> (status, frames [(prev, prev_term, [Ent])], try_next after a written pack)"""
        t = max(self.try_next[q], self.next[q])
        if heartbeat:
            prev = min(t - 1, self.le - 1)                        # leadership.rs:258-261
            if prev < self.start:
                return SNAPSHOTTED, [], t
            return SENT, [(prev, self.log[prev][0], [])], t
        end = self.le - 1
        if want_end is not None:
            if want_end == U64:
                return NOTHING, [], t
            end = min(want_end, end)
        if t < 1:
            return NOTHING, [], t
        prev = t - 1
        if prev < self.start:                                     # durability.rs:37-39: "snapshotted slot queried"
            return SNAPSHOTTED, [], t
        if prev >= self.le or end < t:
            return NOTHING, [], t
        frames = []
        for first in range(t, end + 1, chunk):                    # durability.rs:87-120: chunks of msg_chunk_size
            last = min(end, first + chunk - 1)
            frames.append((first - 1, self.log[first - 1][0], [self.ent(s, q, full_copy) for s in range(first, last + 1)]))
        return SENT, frames, end + 1

    def frame_bytes(self, fr, variant=0):
        prev, pt, ents = fr
        return tf.append_entries(self.ct, prev, pt, [e.wire() for e in ents], self.lc, self.ls, variant)

    def conflict(self, q, end_slot, c_term, c_slot):
        """messages.rs:386-406 -> want_end (U64: no resend)"""
        if self.next[q] == 1:
            self.try_next[q] = 1
            return U64
        ns = self.next[q] - 1
        while ns > self.start and self.log[ns][0] == c_term and ns >= c_slot and ns > 1:
            ns -= 1
        self.next[q] = ns
        self.try_next[q] = ns
        return end_slot

    def success(self, q, end_slot):
        """ss_engine_raft_ingest: a reply behind next_slot is dropped (messages.rs:243-252)"""
        if self.next[q] > end_slot + 1:
            return False
        self.next[q] = end_slot + 1
        self.match[q] = max(self.match[q], end_slot)
        return True

    def tick(self, touched):
        """the commit scan (messages.rs:254-275: own term only, 1 + matches >= threshold) and last_snap (:298-309)"""
        for s in range(self.lc + 1, self.le):
            if self.log[s][0] == self.ct and 1 + sum(m >= s for m in self.match) >= self.threshold:
                new = s
                self.lc = max(self.lc, new)
        if touched:
            self.ls = max(self.ls, min(self.match))

    def advance(self, upto):
        lim = min(self.ls, self.lc)
        if upto > self.start and lim > self.start:
            new = min(upto, lim)
            for s in range(self.start, new):
                self.log.pop(s, None)
            self.start = new


# ---- CPU: the restatement on hand-worked cases --------------------------------------------------------------------
def _leader(n=5, me=0, W=64, f=0, terms=(2, 2, 2)):
    ld = Leader(n, me, W, n // 2 + 1 + f)
    for t in terms:
        ld.ct = t
        ld.propose(bytes([t]) * 7)
    return ld


def test_model_walk_back_over_a_term_run():
    ld = _leader(terms=(1, 1, 1, 2, 2))
    ld.next[0] = 6                                                # follower holds term 1 at slots 1..3, diverges later
    assert ld.conflict(0, 5, 2, 4) == 5
    assert ld.next[0] == 3 and ld.try_next[0] == 3               # 5 -> 4 (term 2 >= slot 4) -> 3 stops: term 1 at 3
    ld.next[0] = 4
    assert ld.conflict(0, 5, 1, 1) == 5 and ld.next[0] == 1      # 3, 2, 1 all term 1 >= slot 1; stops at ns > 1
    st, frames, nt = ld.plan(0, 10, want_end=5)
    assert st == SENT and [f[0] for f in frames] == [0] and len(frames[0][2]) == 5 and nt == 6


def test_model_next_slot_one_stops():
    ld = _leader()
    assert ld.next[1] == 1
    ld.try_next[1] = 3
    assert ld.conflict(1, 3, 0, 1) == U64 and ld.try_next[1] == 1 and ld.next[1] == 1


def test_model_snapshotted_pair():
    ld = _leader()
    ld.lc = ld.ls = 3
    ld.advance(3)
    assert ld.start == 3
    ld.next[2] = 2                                                # prev_slot 1 < start_slot 3
    assert ld.plan(2, 10)[0] == SNAPSHOTTED
    assert ld.plan(2, 10, heartbeat=True)[0] == SNAPSHOTTED
    ld.advance(9)
    assert ld.start == 3                                          # never past min(last_snap, last_commit)


@pytest.mark.parametrize("chunk,firsts", [(1, [1, 2, 3, 4, 5, 6, 7]), (3, [1, 4, 7]), (10, [1])])
def test_model_chunking(chunk, firsts):
    ld = _leader(terms=(1,) * 7)
    st, frames, nt = ld.plan(0, chunk)
    assert st == SENT and [f[0] + 1 for f in frames] == firsts and nt == 8
    assert sum(len(f[2]) for f in frames) == 7
    ld.try_next[0] = nt
    assert ld.plan(0, chunk)[0] == NOTHING


def test_model_heartbeat_after_the_log_end():
    ld = _leader()
    ld.try_next[3] = 9                                            # past log_end 4
    st, frames, nt = ld.plan(3, 10, heartbeat=True)
    assert st == SENT and frames == [(3, 2, [])] and nt == 9
    ld.ct, ld.lc, ld.ls = 2, 2, 1
    assert ld.frame_bytes(frames[0]) == tf.append_entries(2, 3, 2, [], 2, 1)


# ---- CPU: hand-worked bytes ---------------------------------------------------------------------------------------
def test_append_entries_carrying_shard_2_of_rs32():
    # RS(3,2), population 5: two entries of 4-byte batches (shard_len 2) to replica 2
    s2a, s2b = b"\x11\x22", b"\x33\x44"
    e1 = tf.entry(7, 3, 2, 4, {2: s2a}, False, 0)
    e2 = tf.entry(7, 3, 2, 4, {2: s2b}, False, 300)
    assert e1 == bytes([7, 3, 2, 4, 2, 5, 0, 0, 1, 2, 0x11, 0x22, 0, 0, 0, 0, 0])
    assert e2 == bytes([7, 3, 2, 4, 2, 5, 0, 0, 1, 2, 0x33, 0x44, 0, 0, 0, 0, 0xFB, 0x2C, 0x01])
    f = tf.append_entries(7, 4, 6, [e1, e2], 3, 1)
    body = bytes([0, 0, 7, 4, 6, 2]) + e1 + e2 + bytes([3, 1])
    assert f == bytes([0, 0, 0, 0, 0, 0, 0, len(body)]) + body and len(body) == 44


def test_full_copy_entry_and_heartbeat_bytes():
    e = tf.entry(2, 2, 1, 3, {0: b"\xaa\xbb", 1: b"\xcc\x00"}, False, 5)
    assert e == bytes([2, 2, 1, 3, 2, 3, 1, 2, 0xAA, 0xBB, 1, 2, 0xCC, 0, 0, 0, 0, 5])
    assert tf.append_entries(9, 300, 8, [], 299, 250) == bytes([0] * 7 + [12, 0, 0, 9, 0xFB, 0x2C, 0x01, 8, 0, 0xFB, 0x2B, 0x01, 250])


def test_leader_record_bytes():
    rec = leader_record(3, 2, 1, 3, {1: b"\x05\x06"})
    assert rec == bytes([0] * 7 + [16, 1, 3, 2, 1, 3, 2, 3, 0, 1, 2, 5, 6, 0, 0, 1, 0])


@pytest.mark.parametrize("v", [250, 251, 65535, 65536])
def test_varint_widths_in_entries(v):
    w = len(tf.vi(v))
    assert w == {250: 1, 251: 3, 65535: 3, 65536: 5}[v]
    L = -(-v // 3)
    e = tf.entry(1, 3, 2, v, {0: bytes(L)}, False, v)
    assert len(e) == 1 + 2 + w + len(tf.vi(L)) + 1 + 5 + len(tf.vi(L)) + L + 1 + 1 + w
    f = tf.append_entries(1, v, 1, [], v, v)
    assert len(f) == 8 + 1 + 1 + 1 + w + 1 + 1 + 2 * w


def test_refusals_without_an_engine():
    # the argument checks that come before the engine's own; the checks that need an engine (protocol, population, a
    # changed plane_stride, raft_append against the log) need a device to create one and are in test_refusals_on_engines
    from summerset_b200 import _lib
    lib = _lib.load()

    def refused(rc, why):
        assert rc == _lib.SS_ERR_INVALID_ARG and why in lib.ss_last_error().decode(), (rc, lib.ss_last_error(), why)

    spec = lambda chunk=10, variant=0: C.byref(_lib.AppendPackSpec(0, variant, chunk, 0, 0, 0))
    refused(lib.ss_frame_append_pack_dev(None, spec(chunk=0), *([0] * 11)), "msg_chunk_size")
    refused(lib.ss_frame_append_pack_dev(None, spec(variant=1 << 16), *([0] * 11)), "append_variant")
    refused(lib.ss_frame_append_pack_dev(None, None, *([0] * 11)), "null spec")
    refused(lib.ss_frame_append_pack_dev(None, spec(), None, 8, *([0] * 9)), "16-byte aligned")
    refused(lib.ss_frame_append_pack_dev(None, spec(variant=(1 << 16) - 1), *([0] * 11)), "null engine")
    refused(lib.ss_engine_craft_propose(None, 0, 0, 0, 0, 0, 48, *([0] * 9)), "plane_stride")
    refused(lib.ss_engine_craft_propose(None, 0, 0, 0, 0, 0, 0, *([0] * 9)), "plane_stride")
    refused(lib.ss_engine_craft_propose(None, 0, 0, 0, 0, 8, 64, *([0] * 9)), "16-byte aligned")
    refused(lib.ss_engine_craft_propose(None, 0, 0, 0, 0, 0, 64, *([0] * 9)), "null engine")
    refused(lib.ss_engine_craft_backoff(None, 0, 0, 0, 0, 0, 0, 0, 1 << 16, 0), "reply_variant")
    refused(lib.ss_engine_craft_backoff(None, 0, 0, 0, 0, 0, 0, 0, 1, 0), "null engine")
    refused(lib.ss_engine_craft_advance(None, None), "null engine")
    refused(lib.ss_engine_craft_log_view_get(None, None), "null view")


# ---- GPU ------------------------------------------------------------------------------------------------------------
def _ctx():
    from summerset_b200.api import Context
    return Context(0)


@pytest.mark.gpu
def test_refusals_on_engines():
    import torch
    from summerset_b200 import _lib
    from summerset_b200.engine import LeaderEngine, RaftEngine
    ctx = _ctx()
    lib = ctx.lib
    dev = "cuda:0"
    z = lambda n, dt=torch.int64: torch.zeros(n, dtype=dt, device=dev)
    spec = _lib.AppendPackSpec(0, 0, 10, 0, 0, 0)
    paxos = LeaderEngine(ctx, "rspaxos", 4, 5, 1, 16)
    raft = RaftEngine(ctx, 4, 5, craft=False)
    store0, wal0, out0 = (torch.zeros(n, dtype=torch.uint8, device=dev) for n in (5 * 4096, 4096, 4096))
    for e in (paxos, raft):                                       # every call refuses every protocol but CRaft
        assert lib.ss_engine_craft_log_view_get(e.h, C.byref(_lib.CraftLogView())) == _lib.SS_ERR_INVALID_ARG
        assert lib.ss_engine_craft_advance(e.h, z(4).data_ptr()) == _lib.SS_ERR_INVALID_ARG
        assert lib.ss_engine_craft_propose(e.h, 0, out0.data_ptr(), z(4).data_ptr(), z(4, torch.int32).data_ptr(), store0.data_ptr(),
                                           4096, z(4).data_ptr(), z(4).data_ptr(), None, None, wal0.data_ptr(), 4096, z(4).data_ptr(),
                                           z(4).data_ptr(), 0) == _lib.SS_ERR_INVALID_ARG
        assert lib.ss_frame_append_pack_dev(e.h, C.byref(spec), None, out0.data_ptr(), 4096, z(8).data_ptr(), z(8).data_ptr(),
                                            z(8, torch.int32).data_ptr(), z(8, torch.uint8).data_ptr(), 8, z(1).data_ptr(),
                                            z(16, torch.int32).data_ptr(), None) == _lib.SS_ERR_INVALID_ARG
        assert lib.ss_engine_craft_backoff(e.h, out0.data_ptr(), 16, z(1).data_ptr(), z(1, torch.int32).data_ptr(),
                                           z(1, torch.uint8).data_ptr(), z(1, torch.int32).data_ptr(), 1, 1,
                                           z(16).data_ptr()) == _lib.SS_ERR_INVALID_ARG
        assert "CRaft" in lib.ss_last_error().decode()
    eng = RaftEngine(ctx, 4, 5, craft=True)
    out = torch.zeros(1 << 16, dtype=torch.uint8, device=dev)
    fa = [z(8), z(8), z(8, torch.int32), z(8, torch.uint8)]
    args = lambda sp: (eng.h, C.byref(sp), None, out.data_ptr(), out.numel(), *[a.data_ptr() for a in fa], 8, z(1).data_ptr(),
                       z(16, torch.int32).data_ptr(), None)
    assert lib.ss_frame_append_pack_dev(*args(_lib.AppendPackSpec(5, 0, 10, 0, 0, 0))) == _lib.SS_ERR_INVALID_ARG   # me >= n
    assert lib.ss_frame_append_pack_dev(*args(_lib.AppendPackSpec(0, 0, 0, 0, 0, 0))) == _lib.SS_ERR_INVALID_ARG
    assert lib.ss_frame_append_pack_dev(*args(_lib.AppendPackSpec(0, 1 << 16, 10, 0, 0, 0))) == _lib.SS_ERR_INVALID_ARG
    assert lib.ss_frame_append_pack_dev(*args(spec)) == _lib.SS_OK
    arena = torch.zeros(64, dtype=torch.uint8, device=dev)
    dl = torch.full((4,), 8, dtype=torch.int32, device=dev)
    off = torch.zeros(4, dtype=torch.int64, device=dev)
    store, wal = torch.zeros((5, 4096), dtype=torch.uint8, device=dev), torch.zeros(4096, dtype=torch.uint8, device=dev)
    with pytest.raises(Exception):
        eng.propose(5, arena, off, dl, store, wal)                # me >= population
    with pytest.raises(Exception):
        eng.propose(0, arena, off, dl, torch.zeros((5, 4008), dtype=torch.uint8, device=dev), wal)   # stride % 32
    eng.propose(0, arena, off, dl, store, wal)
    with pytest.raises(Exception):
        eng.propose(0, arena, off, dl, torch.zeros((5, 2048), dtype=torch.uint8, device=dev), wal)   # a changed stride
    with pytest.raises(Exception):
        eng.append(torch.ones(4, dtype=torch.int32, device=dev))  # raft_append once the log is in use
    other = RaftEngine(ctx, 4, 5, craft=True)
    other.append(torch.ones(4, dtype=torch.int32, device=dev))
    with pytest.raises(Exception):
        other.log_view()                                          # the log after raft_append
    small = RaftEngine(ctx, 4, 2, craft=True)
    with pytest.raises(Exception):
        small.log_view()                                          # no parity shard at population 2
    torch.cuda.synchronize()
    for e in (paxos, raft, eng, other, small):
        e.close()


def _dls(d):
    return [1, d - 1 if d > 1 else 2, 2, 100, 250 * d, 251 * d + 1, 3000, 65536 + 3]


@pytest.mark.gpu
@pytest.mark.parametrize("n", [3, 5, 7, 9, 12])
def test_propose_matches_the_restatement(n):
    import torch
    from summerset_b200.engine import RaftEngine
    ctx = _ctx()
    G, W, me = 24, 8, n - 1
    d, p = n // 2 + 1, n - n // 2 - 1
    rng = random.Random(n)
    dev = "cuda:0"
    stride = G * pitch(-(-65539 // d))

    def run(eng, models, view, stride, lens, full_copy, wal_cut, store_cut):
        batches = [rng.randbytes(x) for x in lens]
        arena_np, offs = bytearray(), []
        for b in batches:
            arena_np += bytes(rng.randint(0, 7))                  # odd offsets
            offs.append(len(arena_np))
            arena_np += b
        fits = [g for g in range(G) if lens[g] and models[g].le + 1 - models[g].start <= W]
        keep = range(d) if full_copy else [me]
        recs = {g: len(leader_record(models[g].ct, d, p, lens[g], {j: bytes(-(-lens[g] // d)) for j in keep})) for g in fits}
        k = rng.randint(0, len(fits)) if (wal_cut or store_cut) else len(fits)
        wal_cap = sum(r16(recs[g]) for g in fits[:k]) if wal_cut else 1 << 22
        store = torch.full((n, stride), 0xA5, dtype=torch.uint8, device=dev)
        wal = torch.full((wal_cap + 64,), 0xA5, dtype=torch.uint8, device=dev)
        lo = [rng.choice((0, 250, 251, 65535, 65536)) for _ in range(G)]
        out = eng.propose(me, torch.tensor(np.frombuffer(bytes(arena_np) + b"\0", dtype=np.uint8), device=dev),
                          torch.tensor(offs, dtype=torch.int64, device=dev), torch.tensor(lens, dtype=torch.int32, device=dev), store,
                          wal, torch.tensor(lo, dtype=torch.int64, device=dev), wal_capacity=wal_cap, full_copy=full_copy)
        torch.cuda.synchronize()
        st = ctx.device_status()
        o = {kk: v.cpu().numpy() for kk, v in out.items()}
        sto, wl = store.cpu().numpy(), wal.cpu().numpy()
        so, wo, run_s, run_w, placed = {}, {}, 0, 0, []
        for g in fits:
            so[g], wo[g] = run_s, run_w
            run_s += pitch(-(-lens[g] // d))
            run_w += r16(recs[g])
            if run_s <= stride and run_w <= wal_cap:
                placed.append(g)
        assert int(o["need"][0]) == run_s
        assert bool(st & STATUS_RAFT_WINDOW_FULL) == any(lens[g] and g not in fits for g in range(G))
        assert bool(st & STATUS_STORE_FULL) == (run_s > stride)
        assert bool(st & STATUS_FRAME_OVERFLOW) == (run_w > wal_cap)
        for g in range(G):
            m = models[g]
            if g not in placed:
                assert o["slot_out"][g] == -1 and o["shard_off"][g] == -1 and o["wal_off"][g] == -1 and o["wal_len"][g] == 0, g
                continue
            s, rec = m.propose(batches[g], lo[g], full_copy)
            assert int(o["slot_out"][g]) == s and int(o["shard_off"][g]) == so[g] and int(o["wal_off"][g]) == wo[g], g
            assert int(o["wal_len"][g]) == len(rec) and wl[wo[g]:wo[g] + len(rec)].tobytes() == rec, g
            L = -(-lens[g] // d)
            for j in range(n):
                assert sto[j, so[g]:so[g] + L].tobytes() == m.log[s][2][j], (g, j)
                assert not sto[j, so[g] + L:so[g] + r16(L)].any()
        used_s = sum(pitch(-(-lens[g] // d)) for g in placed)
        used_w = sum(r16(recs[g]) for g in placed)
        assert (sto[:, used_s:] == 0xA5).all() and (wl[used_w:] == 0xA5).all()
        le, tm = eng.log_end.cpu().numpy(), eng.terms.cpu().numpy()
        dl_ring, lo_ring, sa = view["data_len"].cpu().numpy(), view["log_offset"].cpu().numpy(), view["shard_addr"].cpu().numpy()
        for g, m in enumerate(models):
            assert le[g] == m.le
            for s in range(m.start, m.le):
                assert tm[g][s % W] == m.log[s][0] and dl_ring[g][s % W] == m.log[s][1] and lo_ring[g][s % W] == m.log[s][3]
            if g in placed:
                assert sa[g][(m.le - 1) % W] == store.data_ptr() + so[g]
        return store

    eng = RaftEngine(ctx, G, n, craft=True, window=W)
    eng.curr_term.fill_(3)
    view = eng.log_view()
    models = [Leader(n, me, W, eng.threshold) for _ in range(G)]
    for m in models:
        m.ct = 3
    keep = []
    for rnd in range(9):
        lens = [0 if rng.random() < 0.2 else rng.choice(_dls(d)) for _ in range(G)]
        keep.append(run(eng, models, view, stride, lens, rnd % 2 == 1, rnd % 3 == 2, False))
        if rnd % 3 == 1:                                          # retire part of the log so the window frees up
            for m in models:
                m.lc = m.ls = m.le - 1
            eng.last_commit.copy_(torch.tensor([m.lc for m in models], dtype=torch.int32, device=dev))
            eng.last_snap.copy_(eng.last_commit)
            upto = [rng.randint(m.start, m.le) for m in models]
            eng.advance_log(torch.tensor(upto, dtype=torch.int64, device=dev))
            for m, u in zip(models, upto):
                m.advance(u)
            torch.cuda.synchronize()
            assert view["log_start"].cpu().tolist() == [m.start for m in models]
    eng.close()
    # the store cut: a plane_stride that holds the slots of the first proposing groups only
    for k in (0, 5, G):
        eng = RaftEngine(ctx, G, n, craft=True, window=W)
        view = eng.log_view()
        models = [Leader(n, me, W, eng.threshold) for _ in range(G)]
        lens = [rng.choice(_dls(d)[:-1]) for _ in range(G)]
        cap = max(32, sum(pitch(-(-x // d)) for x in lens[:k]))
        run(eng, models, view, cap, lens, False, False, True)
        eng.close()


def _pack_raw(eng, me, out, out_capacity, max_frames, want_end=None, heartbeat=False, full_copy=False, chunk=10, variant=0):
    """pack with canaries around every output array"""
    import torch
    from summerset_b200 import _lib
    dev, PG = out.device, eng.P * eng.G
    fill = lambda n, dt, v: torch.full((n + 8,), v, dtype=dt, device=dev)
    a = dict(frame_off=fill(max_frames, torch.int64, 0x5A5A), frame_len=fill(max_frames, torch.int64, 0x5A5A),
             frame_group=fill(max_frames, torch.int32, 0x5A5A), frame_peer=fill(max_frames, torch.uint8, 0x5A),
             n_frames=fill(1, torch.int64, 0x5A5A), total=fill(1, torch.int64, 0x5A5A), pair_status=fill(PG, torch.int32, 0x5A5A))
    spec = _lib.AppendPackSpec(me, variant, chunk, 1 if full_copy else 0, 1 if heartbeat else 0, 0)
    p = lambda k: a[k][4:].data_ptr()
    _lib.check(eng.lib.ss_frame_append_pack_dev(eng.h, C.byref(spec), None if want_end is None else want_end.data_ptr(), out.data_ptr(),
                                                out_capacity, p("frame_off"), p("frame_len"), p("frame_group"), p("frame_peer"),
                                                max_frames, p("n_frames"), p("pair_status"), p("total")))
    torch.cuda.synchronize()
    r = {k: v.cpu().numpy() for k, v in a.items()}
    for k, v in r.items():
        assert (v[:4] == v[0]).all() and (v[-4:] == v[0]).all() and v[0] == (0x5A if k == "frame_peer" else 0x5A5A), k
    return {k: v[4:-4] for k, v in r.items()}


def _check_pack(eng, models, view, o, out_np, me, out_capacity, max_frames, want_end=None, heartbeat=False, full_copy=False, chunk=10):
    """every frame byte, frame array, pair status and try_next against the restatement; applies the pack to the models"""
    G, P = eng.G, eng.P
    plans, run_b, run_f, cut_seen = [], 0, 0, False
    total = 0
    for q in range(P):
        for g in range(G):
            we = None if want_end is None else int(want_end[q][g]) & U64
            st, frames, nt = models[g].plan(q, chunk, we, heartbeat, full_copy)
            fb = [models[g].frame_bytes(f) for f in frames]
            b = sum(r16(len(x)) for x in fb)
            total += b
            plans.append((q, g, st, fb, nt, b))
    k = 0
    for q, g, st, fb, nt, b in plans:
        m = models[g]
        got = int(o["pair_status"][q * G + g])
        if st == SENT and (run_b + b > out_capacity or run_f + len(fb) > max_frames):
            cut_seen = True
            assert got == OVERFLOW, (q, g, got)
            run_b += b
            run_f += len(fb)
            continue
        assert got == st, (q, g, got, st)
        if st == SENT:
            assert not cut_seen                                   # the written pairs are a prefix
            for x in fb:
                off = int(o["frame_off"][k])
                assert off == run_b and int(o["frame_len"][k]) == len(x) and o["frame_group"][k] == g and o["frame_peer"][k] == q
                assert out_np[off:off + len(x)].tobytes() == x, (q, g, k)
                run_b += r16(len(x))
                k += 1
            run_f += len(fb)
        m.try_next[q] = nt
    assert int(o["n_frames"][0]) == k and int(o["total"][0]) == total
    assert (out_np[min(out_capacity, len(out_np)):] == 0xA5).all()
    tn = view["try_next"].cpu().numpy()
    for g, m in enumerate(models):
        assert [int(tn[q][g]) for q in range(P)] == m.try_next, g
    return k


@pytest.mark.gpu
@pytest.mark.parametrize("n", [5, 7])
def test_pack_matches_the_restatement(n):
    import torch
    from summerset_b200.engine import RaftEngine
    ctx = _ctx()
    G, W, me = 12, 16, 2
    d = n // 2 + 1
    rng = random.Random(100 + n)
    dev = "cuda:0"
    eng = RaftEngine(ctx, G, n, craft=True, window=W)
    view = eng.log_view()
    models = [Leader(n, me, W, eng.threshold) for _ in range(G)]
    stride = G * pitch(-(-65539 // d))
    stores = []
    P = n - 1
    cases = 0
    for rnd in range(14):
        term = 2 + rnd // 4
        eng.curr_term.fill_(term)
        for m in models:
            m.ct = term
        for _ in range(3):                                        # batches into most groups
            lens = [0 if rng.random() < 0.25 else rng.choice((1, d - 1, 100, 251 * d, 3000) if rng.random() > 0.05 else (65539,)) for _ in range(G)]
            lens = [x if models[g].le + 1 - models[g].start <= W else 0 for g, x in enumerate(lens)]
            batches = [rng.randbytes(x) for x in lens]
            arena_np, offs = bytearray(), []
            for b in batches:
                offs.append(len(arena_np))
                arena_np += b
            store = torch.zeros((n, stride), dtype=torch.uint8, device=dev)
            stores.append(store)
            lo = [rng.choice((0, 250, 251, 65535, 65536, 1 << 32)) for _ in range(G)]
            eng.propose(me, torch.tensor(np.frombuffer(bytes(arena_np) + b"\0", dtype=np.uint8), device=dev),
                        torch.tensor(offs, dtype=torch.int64, device=dev), torch.tensor(lens, dtype=torch.int32, device=dev), store,
                        torch.zeros(1 << 22, dtype=torch.uint8, device=dev), torch.tensor(lo, dtype=torch.int64, device=dev))
            for g, m in enumerate(models):
                if lens[g]:
                    m.propose(batches[g], lo[g])
        # lagging and leading peers: next_slot anywhere in [start, le], try_next around it
        ns = np.zeros((P, G), dtype=np.int32)
        tn = np.zeros((P, G), dtype=np.int32)
        for g, m in enumerate(models):
            for q in range(P):
                m.next[q] = rng.randint(max(1, m.start), m.le)
                m.try_next[q] = max(0, m.next[q] + rng.randint(-2, 3))
                ns[q][g], tn[q][g] = m.next[q], m.try_next[q]
            m.lc = max(m.lc, rng.randint(m.start, m.le - 1))
            m.ls = max(m.ls, rng.randint(m.start, m.lc))
        eng.next_slot.copy_(torch.tensor(ns, device=dev))
        view["try_next"].copy_(torch.tensor(tn, device=dev))
        eng.last_commit.copy_(torch.tensor([m.lc for m in models], dtype=torch.int32, device=dev))
        eng.last_snap.copy_(torch.tensor([m.ls for m in models], dtype=torch.int32, device=dev))
        mode = rnd % 7
        heartbeat, full_copy = mode == 3, mode == 4
        chunk = (1, 3, 10)[rnd % 3]
        want = None
        if mode in (1, 5):
            want = np.array([[rng.choice((U64, 0, m.le - 1, m.le + 3, max(0, m.next[q] + rng.randint(-1, 4)))) for m in models]
                             for q in range(P)], dtype=np.uint64)
        # the exact bytes and frames of the pairs before a random cut, or room for everything
        out_cap, max_frames = 1 << 22, 4096
        if mode in (2, 5, 6):
            sizes = []
            for q in range(P):
                for g, m in enumerate(models):
                    st, frames, _ = m.plan(q, chunk, None if want is None else int(want[q][g]), heartbeat, full_copy)
                    sizes.append((sum(r16(len(m.frame_bytes(f))) for f in frames), len(frames)))
            k = rng.randint(0, len(sizes))
            if mode == 6:
                max_frames = sum(s[1] for s in sizes[:k])
            else:
                out_cap = sum(s[0] for s in sizes[:k]) + (rng.randint(0, 15) if mode == 5 else 0)
        out = torch.full((out_cap + 64,), 0xA5, dtype=torch.uint8, device=dev)
        wt = None if want is None else torch.tensor(want.view(np.int64), device=dev)
        o = _pack_raw(eng, me, out, out_cap, max_frames, wt, heartbeat, full_copy, chunk)
        _check_pack(eng, models, view, o, out.cpu().numpy(), me, out_cap, max_frames, want, heartbeat, full_copy, chunk)
        st = ctx.device_status()
        assert bool(st & STATUS_FRAME_OVERFLOW) == bool((o["pair_status"] == OVERFLOW).any())
        cases += int((o["pair_status"] == SNAPSHOTTED).sum() > 0) + int((o["pair_status"] == OVERFLOW).sum() > 0)
        # retire part of the log: the ring wraps over the following rounds
        upto = [rng.randint(m.start, m.le) for m in models]
        eng.advance_log(torch.tensor(upto, dtype=torch.int64, device=dev))
        for m, u in zip(models, upto):
            m.advance(u)
        torch.cuda.synchronize()
        assert view["log_start"].cpu().tolist() == [m.start for m in models]
    assert max(m.le for m in models) > 2 * W and cases >= 3
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [5, 7])
def test_closed_loop_with_device_followers(n):
    closed_loop(n)


def closed_loop(n, append_variant=0, reply_variant=1, meta_variant=0, log_variant=1, leader_reply_variant=None):
    """leader 1 packs, device followers append and reply, the leader parses, ingests and backs off, all against the
    restatements, with the given PeerMsg and DurEntry variant indices.  leader_reply_variant: the followers' replies are
    re-encoded with this AppendEntriesReply index (one a follower cannot emit, >= 251) before the leader takes them."""
    import torch
    from summerset_b200.engine import Follower, RaftEngine, append_reply_parse
    ctx = _ctx()
    G, me, term = 64, 1, 2
    d, p, P = n // 2 + 1, n - n // 2 - 1, n - 1
    rng = random.Random(7 * n)
    dev = "cuda:0"
    t = lambda a, dt: torch.tensor(a, dtype=dt, device=dev)
    eng = RaftEngine(ctx, G, n, craft=True)
    view = eng.log_view()
    eng.curr_term.fill_(term)
    L = [Leader(n, me, eng.W, eng.threshold) for _ in range(G)]
    for m in L:
        m.ct = term
    reps = [r for r in range(n) if r != me]                       # replica of peer q is reps[q]
    fols = [Follower(ctx, G, n, r, 0, append_variant, reply_variant, meta_variant, log_variant) for r in reps]
    fmodels = [[tf.Group(n, fols[0].W, reply_variant, meta_variant) for _ in range(G)] for _ in reps]
    lrv = reply_variant if leader_reply_variant is None else leader_reply_variant
    keep = []                                                     # every store a live entry may point into
    seen = dict(conflict=0, trunc=0)

    def deliver(q, frames):
        """frames [(group, bytes, (prev, pt, ents, commit, snap))] to follower q and its models -> reply frames"""
        if not frames:
            return []
        buf, offs = bytearray(), []
        for g, x, _ in frames:
            buf += bytes(rng.randint(0, 3))
            offs.append(len(buf))
            buf += x
        store = torch.zeros(2 * len(buf) + (1 << 16), dtype=torch.uint8, device=dev)
        wal = torch.zeros(2 * len(buf) + (1 << 16), dtype=torch.uint8, device=dev)
        keep.append(store)
        o = fols[q].append(t(np.frombuffer(bytes(buf), dtype=np.uint8), torch.uint8), t(offs, torch.int64),
                           t([f[0] for f in frames], torch.int32), t([me] * len(frames), torch.uint8), store, wal)
        torch.cuda.synchronize()
        rl, cells, tr = o["reply_len"].cpu().numpy(), o["replies"].cpu().numpy(), o["trunc_slot"].cpu().numpy()
        out = []
        for i, (g, x, (prev, pt, ents, cm, sn)) in enumerate(frames):
            want = fmodels[q][g].handle(me, term, prev, pt, ents, cm, sn)
            assert cells[i][:rl[i]].tobytes() == want["reply"], (q, g, i)
            seen["trunc"] += want["trunc"] is not None
            assert (int(tr[i]) != -1) == (want["trunc"] is not None)
            tm, end, conf = tf._parse_reply_py(want["reply"], reply_variant)[1]
            out.append((g, q, tf.reply(tm, end, conf, lrv)))
        return out

    def round_trip(want_np):
        """pack (want_end or all), compare, deliver, parse, ingest, back off -> the next want_end, or None when quiet"""
        out = torch.full((1 << 24,), 0xA5, dtype=torch.uint8, device=dev)
        wt = None if want_np is None else torch.tensor(want_np.view(np.int64), device=dev)
        o = _pack_raw(eng, me, out, 1 << 24, 1 << 14, wt, chunk=3, variant=append_variant)
        out_np = out.cpu().numpy()
        # the restatement's frames, with their structure for the follower models
        per_q = [[] for _ in range(P)]
        k = 0
        for q in range(P):
            for g, m in enumerate(L):
                st, frames, nt = m.plan(q, 3, None if want_np is None else int(want_np[q][g]))
                assert int(o["pair_status"][q * G + g]) == st
                for f in frames:
                    x = m.frame_bytes(f, append_variant)
                    off = int(o["frame_off"][k])
                    assert out_np[off:off + len(x)].tobytes() == x and o["frame_group"][k] == g and o["frame_peer"][k] == q
                    per_q[q].append((g, x, (f[0], f[1], f[2], m.lc, m.ls)))
                    k += 1
                m.try_next[q] = nt
        assert int(o["n_frames"][0]) == k
        if k == 0:
            return None
        replies = []
        for q in range(P):
            replies += deliver(q, per_q[q])
        buf, offs = bytearray(), []
        for g, q, x in replies:
            offs.append(len(buf))
            buf += x
        tb = t(np.frombuffer(bytes(buf), dtype=np.uint8), torch.uint8)
        fo, fg, fp = t(offs, torch.int64), t([r[0] for r in replies], torch.int32), t([r[1] for r in replies], torch.uint8)
        rec = append_reply_parse(ctx, tb, fo, fg, fp, eng.curr_term, G, lrv)
        eng.on_append_replies(rec["rec_group"], rec["rec_peer"], rec["rec_end_slot"])
        want = eng.backoff(tb, fo, fg, fp, rec["rec_kind"], lrv)
        torch.cuda.synchronize()
        touched = set()
        for g, q, x in replies:                                   # success replies first, then conflicts in frame order
            kind, fdec = tf._parse_reply_py(x, lrv)
            tm, end, conf = fdec
            if conf is None and L[g].success(q, end):
                touched.add(g)
        want_model = np.full((P, G), U64, dtype=np.uint64)
        for g, q, x in replies:
            tm, end, conf = tf._parse_reply_py(x, lrv)[1]
            if conf is not None:
                seen["conflict"] += 1
                want_model[q][g] = L[g].conflict(q, end, conf[0], conf[1])
        assert (want.cpu().numpy().view(np.uint64) == want_model).all()
        check_engine()
        round_trip.touched |= touched
        return want_model if (want_model != U64).any() else None

    round_trip.touched = set()

    def check_engine():
        ns, mt, tn = eng.next_slot.cpu().numpy(), eng.match.cpu().numpy(), view["try_next"].cpu().numpy()
        for g, m in enumerate(L):
            assert [int(ns[q][g]) for q in range(P)] == m.next, (g, m.next)
            assert [int(mt[q][g]) for q in range(P)] == m.match, g
            assert [int(tn[q][g]) for q in range(P)] == m.try_next, g
        assert eng.last_commit.cpu().tolist() == [m.lc for m in L]
        assert eng.last_snap.cpu().tolist() == [m.ls for m in L]
        assert view["log_start"].cpu().tolist() == [m.start for m in L]

    # followers seeded by an older leader of term 1: entries that diverge from this leader's
    for q in range(P):
        seed = []
        for g in range(G):
            if rng.random() < 0.5:
                k = rng.randint(1, 3)
                ents = [tf.Ent(1, d, p, 9, {reps[q]: rng.randbytes(-(-9 // d))}, True, 0) for _ in range(k)]
                seed.append((g, tf.append_entries(1, 0, 0, [e.wire() for e in ents], 0, 0, append_variant), (0, 0, ents, 0, 0)))
        buf, offs = bytearray(), []
        for g, x, _ in seed:
            offs.append(len(buf))
            buf += x
        store = torch.zeros(len(buf) * 2 + 4096, dtype=torch.uint8, device=dev)
        keep.append(store)
        fols[q].append(t(np.frombuffer(bytes(buf), dtype=np.uint8), torch.uint8), t(offs, torch.int64), t([s[0] for s in seed], torch.int32),
                       t([reps[(q + 1) % P]] * len(seed), torch.uint8), store, torch.zeros(len(buf) * 2 + 4096, dtype=torch.uint8, device=dev))
        for g, x, (prev, pt, ents, cm, sn) in seed:
            fmodels[q][g].handle(reps[(q + 1) % P], 1, prev, pt, ents, cm, sn)
    stride = G * pitch(-(-5000 // d))
    for rnd in range(8):
        lens = [0 if rng.random() < 0.3 else rng.choice((1, 7, 300, 4096, 5000)) for _ in range(G)]
        batches = [rng.randbytes(x) for x in lens]
        arena, offs = bytearray(), []
        for b in batches:
            offs.append(len(arena))
            arena += b
        store = torch.zeros((n, stride), dtype=torch.uint8, device=dev)
        keep.append(store)
        eng.propose(me, t(np.frombuffer(bytes(arena) + b"\0", dtype=np.uint8), torch.uint8), t(offs, torch.int64), t(lens, torch.int32),
                    store, torch.zeros(1 << 22, dtype=torch.uint8, device=dev))
        for g, m in enumerate(L):
            if lens[g]:
                m.propose(batches[g])
        if rnd == 0:                                              # a new leader's next_slot: its log end
            eng.next_slot.copy_(torch.tensor([[m.le for m in L]] * P, dtype=torch.int32, device=dev))
            for m in L:
                m.next = [m.le] * P
        want = round_trip(None)
        loops = 0
        while want is not None and loops < 6:
            want = round_trip(want)
            loops += 1
        eng.tick()
        for g, m in enumerate(L):
            m.tick(g in round_trip.touched)
        round_trip.touched = set()
        torch.cuda.synchronize()
        check_engine()
        for q in range(P):
            v = {k: getattr(fols[q], k).cpu().numpy() for k in ("log_end", "curr_term", "last_commit", "last_snap", "term")}
            for g, fm in enumerate(fmodels[q]):
                assert (v["log_end"][g], v["curr_term"][g], v["last_commit"][g], v["last_snap"][g]) == (fm.le, fm.ct, fm.lc, fm.ls), (q, g)
                for s in range(fm.start, fm.le):
                    assert v["term"][g][s % fols[q].W] == fm.log[s][0]
        if rnd % 3 == 2:
            upto = [m.lc for m in L]
            eng.advance_log(torch.tensor(upto, dtype=torch.int64, device=dev))
            for m, u in zip(L, upto):
                m.advance(u)
    assert seen["conflict"] > 0 and seen["trunc"] > 0
    # every follower holds its own shard of every committed entry, byte for byte
    stores = [(s.data_ptr(), s.cpu().numpy()) for s in keep]

    def read(addr, nb):
        for b, arr in stores:
            if b <= addr and addr + nb <= b + arr.size:
                return arr.reshape(-1)[addr - b:addr - b + nb].tobytes()
        raise AssertionError("shard address outside every store")

    checked = 0
    for q in range(P):
        sa, held, tm = fols[q].shard_addr.cpu().numpy(), fols[q].held.cpu().numpy(), fols[q].term.cpu().numpy()
        W = fols[q].W
        for g, m in enumerate(L):
            for s in range(max(1, m.start), m.lc + 1):
                tt, dl, sh, _ = m.log[s]
                assert tm[g][s % W] == tt and held[g][s % W] == 1 << reps[q], (q, g, s)
                assert read(int(sa[g][s % W]), -(-dl // d)) == sh[reps[q]], (q, g, s)
                checked += 1
    assert checked > G
    for f in fols:
        f.close()
    eng.close()
