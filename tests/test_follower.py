"""The CRaft follower (ss_follower_*) and the leader's AppendEntriesReply parser (ss_append_reply_parse_dev).

`Group.handle` restates handle_msg_append_entries (craft/messages.rs:14-252) with check_term (craft/leadership.rs:16-75)
per message, over the follower's state and its window rule; the byte encoders below restate the bincode formats
(craft/mod.rs:124-241) and are pinned by hand-worked vectors and by the oracle's varint and RSCodeword encoders.  GPU
tests compare every store byte, record, cell, verdict and state word of the device follower with the restatement.
"""
from __future__ import annotations

import ctypes as C
import random

import numpy as np
import pytest

from oracle import pyoracle as oracle

ACCEPTED, REJECTED, BEYOND, STORE_FULL, WAL_FULL = 0xFFFFFFF0, 0xFFFFFFF1, 0xFFFFFFF3, 0xFFFFFFF4, 0xFFFFFFF5
MALFORMED = 0xFFFFFFFF
INGEST, CONFLICT, HIGHER, END_RANGE = 0xFFFFFFF0, 0xFFFFFFF1, 0xFFFFFFF2, 0xFFFFFFF3
U64 = (1 << 64) - 1


# ---- bincode restatement ---------------------------------------------------------------------------------------
def vi(v: int) -> bytes:
    if v < 251:
        return bytes([v])
    if v < 1 << 16:
        return b"\xfb" + v.to_bytes(2, "little")
    if v < 1 << 32:
        return b"\xfc" + v.to_bytes(4, "little")
    return b"\xfd" + v.to_bytes(8, "little")


def framed(body: bytes) -> bytes:
    return len(body).to_bytes(8, "big") + body


def codeword(d: int, p: int, data_len: int, shards: dict) -> bytes:
    L = -(-data_len // d)
    out = bytes([d, p]) + vi(data_len) + vi(L) + vi(d + p)
    for j in range(d + p):
        out += b"\x01" + vi(L) + shards[j] if j in shards else b"\x00"
    return out + b"\x00"


def entry(term, d, p, data_len, shards, external=True, log_offset=0) -> bytes:
    return vi(term) + codeword(d, p, data_len, shards) + bytes([1 if external else 0]) + vi(log_offset)


def append_entries(term, prev, prev_term, entries, commit, snap, variant=0) -> bytes:
    return framed(vi(0) + vi(variant) + vi(term) + vi(prev) + vi(prev_term) + vi(len(entries)) + b"".join(entries) + vi(commit) + vi(snap))


def reply(term, end_slot, conflict=None, variant=1) -> bytes:
    body = vi(0) + vi(variant) + vi(term) + vi(end_slot)
    body += b"\x00" if conflict is None else b"\x01" + vi(conflict[0]) + vi(conflict[1])
    return framed(body)


def dur_log_entry(entry_bytes_to_external: bytes, variant=1) -> bytes:
    return framed(vi(variant) + entry_bytes_to_external + vi(0))


def dur_metadata(curr_term, variant=0) -> bytes:
    return framed(vi(variant) + vi(curr_term) + b"\xff")


# ---- the per-message restatement ---------------------------------------------------------------------------------
class Ent:
    def __init__(self, term, d, p, data_len, shards, external=True, log_offset=0):
        self.term, self.d, self.p, self.dl, self.shards = term, d, p, data_len, dict(shards)
        self.external, self.log_offset = external, log_offset

    def wire(self):
        return entry(self.term, self.d, self.p, self.dl, self.shards, self.external, self.log_offset)

    def to_external(self):
        return self.wire()[:-len(vi(self.log_offset))]

    @property
    def held(self):
        return sum(1 << j for j in self.shards)


class Group:
    """one group's follower state; log[s] = (term, data_len, {shard: bytes}) for s in [start, le)"""

    def __init__(self, n: int, W: int, reply_variant=1, meta_variant=0):
        self.d, self.T, self.W = n // 2 + 1, n, W
        self.rv, self.mv = reply_variant, meta_variant             # AppendEntriesReply in PeerMsg, Metadata in DurEntry
        self.absorb_room = True                                   # False: absorbs find no room and change nothing
        self.start, self.le, self.ct, self.ldr, self.lc, self.ls = 0, 1, 0, 0xFF, 0, 0
        self.log = {0: (0, 0, {})}

    def handle(self, peer, term, prev, prev_term, ents, commit, snap):
        """-> dict(verdict, meta, reply, reply_to ('peer' / 'leader'), trunc, appended [Ent])"""
        o = dict(meta=None, reply=None, reply_to=None, trunc=None, appended=[], verdict=ACCEPTED)
        n = len(ents)
        if n and prev + n >= self.start + self.W:
            o["verdict"] = BEYOND
            return o
        if term > self.ct:
            self.ct = term
            o["meta"] = dur_metadata(term, self.mv)
            self.ldr = peer
        if term == self.ct:
            self.ldr = peer
        inside = self.start <= prev < self.le
        if term < self.ct or not inside or self.log[prev][0] != prev_term:
            ctm = self.log[prev][0] if inside else 0
            cs = prev
            while ctm > 0 and cs > self.start and self.log[cs - 1][0] == ctm:
                cs -= 1
            o.update(verdict=REJECTED, reply=reply(self.ct, prev + n, (ctm, cs), self.rv), reply_to="peer")
            self.ls = max(self.ls, snap)
            return o
        appending = False
        first_new = prev + 1
        for k, e in enumerate(ents):
            s = prev + 1 + k
            if not appending:
                if s < self.le and self.log[s][0] != e.term:
                    o["trunc"] = s
                    for q in range(s, self.le):
                        del self.log[q]
                    self.le = s
                appending = s >= self.le
                if appending:
                    first_new = s
            if appending:
                self.log[s] = (e.term, e.dl, dict(e.shards))
                self.le = s + 1
                o["appended"].append(e)
            else:
                t, dl, sh = self.log[s]
                held = sum(1 << j for j in sh)
                if bin(held & ((1 << self.d) - 1)).count("1") < self.d and dl == e.dl and held != e.held and self.absorb_room:
                    self.log[s] = (t, dl, {**e.shards, **sh})
        o["reply"] = reply(self.ct, prev + n, variant=self.rv)
        o["reply_to"] = "leader" if o["appended"] else "peer"
        if commit > self.lc:
            # entries.len() after the append loop's drain is first_new - prev - 1 (messages.rs:160-203)
            nc = min(commit, first_new - 1, self.le - 1)
            for s in range(self.lc + 1, nc + 1):
                if len(self.log[s][2]) < self.d:
                    break
                self.lc = s
        self.ls = max(self.ls, snap)
        return o

    def advance(self, upto):
        if upto > self.start:
            new = min(upto, max(self.lc, self.start))
            for s in range(self.start, new):
                del self.log[s]
            self.start = new


# ---- CPU: encoders against hand-worked bytes and the oracle -----------------------------------------------------
def test_append_entries_two_entries_bytes():
    e1 = entry(3, 2, 1, 3, {0: b"\xaa\xbb", 2: b"\x01\x02"}, True, 0)
    e2 = entry(4, 2, 1, 1, {1: b"\x07"}, False, 300)
    assert e1 == bytes([3, 2, 1, 3, 2, 3, 1, 2, 0xAA, 0xBB, 0, 1, 2, 1, 2, 0, 1, 0])
    assert e2 == bytes([4, 2, 1, 1, 1, 3, 0, 1, 1, 7, 0, 0, 0, 0xFB, 0x2C, 0x01])
    f = append_entries(4, 7, 3, [e1, e2], 6, 2)
    body = bytes([0, 0, 4, 7, 3, 2]) + e1 + e2 + bytes([6, 2])
    assert f == len(body).to_bytes(8, "big") + body
    assert f[:8] == bytes([0, 0, 0, 0, 0, 0, 0, 42])


def test_codeword_matches_oracle_encoder():
    for d, p, dl in ((2, 1, 3), (3, 2, 4096), (5, 4, 250), (3, 2, 70000)):
        L = -(-dl // d)
        rng = np.random.default_rng(dl)
        shards = {j: rng.integers(0, 256, L, dtype=np.uint8).tobytes() for j in range(d + p) if j % 2 == 0}
        wal = oracle.wal_accept_data(0, 0, d, p, dl, [shards.get(j) for j in range(d + p)])
        assert wal[8 + 3:] == codeword(d, p, dl, shards)          # AcceptData variant 1, slot 0, ballot 0, then the codeword
    for v in (0, 250, 251, 65535, 65536, (1 << 32) - 1, 1 << 32, U64):
        assert vi(v) == oracle.varint(v)


def test_dur_entries_and_reply_bytes():
    e = entry(5, 3, 2, 2, {4: b"\x10"}, True, 99)
    rec = dur_log_entry(e[:-1])
    # length 17; LogEntry; term 5; d 3, p 2, data_len 2, shard_len 1, 5 Options (four None, one Some [0x10]); data_copy
    # None; external true; log_offset 0 (99 on the wire)
    assert rec == bytes([0, 0, 0, 0, 0, 0, 0, 17, 1, 5, 3, 2, 2, 1, 5, 0, 0, 0, 0, 1, 1, 0x10, 0, 1, 0])
    assert dur_metadata(300) == bytes([0, 0, 0, 0, 0, 0, 0, 5, 0, 0xFB, 0x2C, 0x01, 0xFF])
    assert reply(7, 12) == bytes([0, 0, 0, 0, 0, 0, 0, 5, 0, 1, 7, 12, 0])
    assert reply(7, 300, (6, 251)) == bytes([0, 0, 0, 0, 0, 0, 0, 11, 0, 1, 7, 0xFB, 0x2C, 0x01, 1, 6, 0xFB, 0xFB, 0])
    longest = reply(U64, U64, (U64, U64))
    assert len(longest) == 47                                     # fits the 48-byte reply cell


def _e(term, n=5, shards=None, dl=10):
    d = n // 2 + 1
    L = -(-dl // d)
    return Ent(term, d, n - d, dl, shards if shards is not None else {0: bytes([term]) * L})


def test_model_conflict_walk_back_and_truncation():
    g = Group(5, 64)
    assert g.handle(1, 1, 0, 0, [_e(1), _e(1), _e(2)], 0, 0)["verdict"] == ACCEPTED
    assert g.le == 4
    o = g.handle(1, 2, 3, 9, [], 0, 0)                            # heartbeat with a stale prev_term
    assert o["verdict"] == REJECTED and o["reply"] == reply(2, 3, (2, 3))
    o = g.handle(1, 2, 2, 5, [_e(3)], 0, 0)
    assert o["reply"] == reply(2, 3, (1, 1))                      # walk back over the term-1 run to slot 1
    o = g.handle(2, 3, 1, 1, [_e(1), _e(3), _e(3)], 0, 0)         # truncation in the middle of the frame
    assert o["verdict"] == ACCEPTED and o["trunc"] == 3 and len(o["appended"]) == 2 and g.le == 5
    assert o["meta"] == dur_metadata(3) and o["reply_to"] == "leader" and g.ldr == 2
    o = g.handle(2, 3, 0, 0, [_e(1), _e(1)], 0, 0)                # all present: nothing appended, immediate reply
    assert o["appended"] == [] and o["reply"] == reply(3, 2) and o["reply_to"] == "peer"
    o = g.handle(1, 1, 4, 3, [], 0, 0)                            # lower term
    assert o["verdict"] == REJECTED and o["reply"] == reply(3, 4, (3, 3)) and g.ldr == 2
    g.lc = 2
    g.advance(2)
    o = g.handle(2, 3, 1, 1, [], 0, 0)                            # prev_slot < start_slot
    assert o["reply"] == reply(3, 1, (0, 1))


def test_model_absorb_and_commit():
    g = Group(5, 64)
    g.handle(1, 1, 0, 0, [_e(1, shards={0: b"ab"}, dl=5)], 1, 0)
    assert g.lc == 0                                              # a frame never commits what it appends itself
    o = g.handle(1, 1, 0, 0, [_e(1, shards={1: b"cd", 2: b"ef"}, dl=5)], 1, 0)
    assert o["appended"] == [] and sorted(g.log[1][2]) == [0, 1, 2] and g.lc == 0   # all present: the cap is prev_slot
    g.handle(1, 1, 1, 1, [], 1, 0)
    assert g.lc == 1
    g.handle(1, 1, 1, 1, [_e(1, shards={0: b"xy"}, dl=5)], 5, 0)
    assert g.lc == 1                                              # one shard: the commit walk stops


def test_follower_refusals_without_gpu():
    from summerset_b200 import _lib
    lib = _lib.load()
    h = C.c_void_p()
    ok = _lib.FollowerConfig(_lib.SS_PROTO_CRAFT, 5, 0, 64, 0, 1, 0, 1)
    for bad in (_lib.FollowerConfig(_lib.SS_PROTO_RAFT, 5, 0, 64, 0, 1, 0, 1),
                _lib.FollowerConfig(_lib.SS_PROTO_RSPAXOS, 5, 0, 64, 0, 1, 0, 1),
                _lib.FollowerConfig(_lib.SS_PROTO_CRAFT, 5, 5, 64, 0, 1, 0, 1),
                _lib.FollowerConfig(_lib.SS_PROTO_CRAFT, 0, 0, 64, 0, 1, 0, 1),
                _lib.FollowerConfig(_lib.SS_PROTO_CRAFT, 5, 0, 48, 0, 1, 0, 1),
                _lib.FollowerConfig(_lib.SS_PROTO_CRAFT, 5, 0, 8192, 0, 1, 0, 1),
                _lib.FollowerConfig(_lib.SS_PROTO_CRAFT, 5, 0, 64, 0, 251, 0, 1),       # a reply would overrun its cell
                _lib.FollowerConfig(_lib.SS_PROTO_CRAFT, 5, 0, 64, 1 << 16, 1, 0, 1),
                _lib.FollowerConfig(_lib.SS_PROTO_CRAFT, 5, 0, 64, 0, 1, 1 << 16, 1),
                _lib.FollowerConfig(_lib.SS_PROTO_CRAFT, 5, 0, 64, 0, 1, 0, 1 << 16)):
        assert lib.ss_follower_create(None, C.byref(bad), 4, C.byref(h)) == _lib.SS_ERR_INVALID_ARG
    assert lib.ss_follower_create(None, None, 4, C.byref(h)) == _lib.SS_ERR_INVALID_ARG
    assert lib.ss_follower_create(None, C.byref(ok), 0, C.byref(h)) == _lib.SS_ERR_INVALID_ARG
    assert lib.ss_follower_create(None, C.byref(ok), 4, None) == _lib.SS_ERR_INVALID_ARG
    assert lib.ss_follower_append(None, *([0] * 22)) == _lib.SS_ERR_INVALID_ARG
    assert lib.ss_follower_advance(None, None) == _lib.SS_ERR_INVALID_ARG
    assert lib.ss_append_reply_parse_dev(None, *([0] * 16)) == _lib.SS_ERR_INVALID_ARG
    import torch
    if not torch.cuda.is_available():
        assert lib.ss_follower_create(None, C.byref(ok), 4, C.byref(h)) == _lib.SS_ERR_NO_DEVICE


# ---- GPU --------------------------------------------------------------------------------------------------------
def _leader_stream(rng: random.Random, n: int, peers, n_frames: int, sharded: bool, me: int, dls):
    """frames of successive leaders for one group: each extends or rewrites the log of the last"""
    d = n // 2 + 1
    log = [0]                                                     # leader's view of terms per slot
    ents = {}
    frames = []
    term = 1
    for _ in range(n_frames):
        r = rng.random()
        if r < 0.15:
            term += 1
            cut = rng.randint(1, len(log))                        # new leader with a different suffix
            del log[cut:]
        if r < 0.55 or len(log) == 1:
            for _ in range(rng.randint(1, 3)):
                s = len(log)
                dl = rng.choice(dls) if rng.random() > 0.04 else rng.choice((70000, 140000))   # 5-byte varints
                L = -(-dl // d)
                payload = {j: rng.randbytes(L) for j in range(n)}
                keep = {me % n: payload[me % n]} if sharded else {j: payload[j] for j in range(d)}
                ents[(s, term)] = (dl, payload, keep)
                log.append(term)
        prev = rng.randint(max(0, len(log) - 5), len(log) - 1)
        k = rng.randint(0, len(log) - 1 - prev)
        es = []
        for s in range(prev + 1, prev + 1 + k):
            dl, payload, keep = ents[(s, log[s])]
            if rng.random() < 0.2:                                # a re-send with another shard map: absorb
                keep = {j: payload[j] for j in range(d)}
            es.append(Ent(log[s], d, n - d, dl, keep, rng.random() < 0.5, rng.choice((0, 7, 300))))
        t = term if rng.random() > 0.1 else max(1, term - 1)
        pt = log[prev] if rng.random() > 0.1 else log[prev] + 1
        frames.append((rng.choice(peers), t, prev, pt, es, rng.randint(0, len(log)), rng.randint(0, 3)))
    return frames


def _raw_cw(d, p, dl, L, opts, tail=b"\x00"):
    """an RSCodeword spelled field by field: opts = per shard None or (length varint value, bytes)"""
    out = bytes([d, p]) + vi(dl) + vi(L) + vi(len(opts))
    for o in opts:
        out += b"\x00" if o is None else b"\x01" + vi(o[0]) + o[1]
    return out + tail


def _bad_frames(rng: random.Random, n: int, me: int, G: int):
    """(group, peer, bytes, verdict) for frames the follower must refuse without touching any state"""
    d, p = n // 2 + 1, n - n // 2 - 1
    peer = (me + 1) % n
    good_cw = codeword(d, p, 5, {0: bytes(-(-5 // d))})
    L = -(-5 // d)
    wrap = lambda cw, ext=b"\x01": vi(3) + cw + ext + vi(0)
    ae = lambda ents, term=9, prev=0: vi(0) + vi(0) + vi(term) + vi(prev) + vi(0) + vi(len(ents)) + b"".join(ents) + vi(0) + vi(0)
    body = ae([wrap(good_cw)])
    g = rng.randrange(G)
    out = [
        (g, peer, framed(body[:-1]), MALFORMED),                                   # truncated
        (g, peer, framed(body + b"\x00"), MALFORMED),                              # trailing bytes
        (g, peer, framed(ae([wrap(codeword(d + 1, p - 1 if p > 1 else p, 5, {}))])), MALFORMED),   # another code
        (g, peer, framed(ae([wrap(_raw_cw(d, p, 5, L + 1, [None] * n))])), MALFORMED),            # shard_len != ceil
        (g, peer, framed(ae([wrap(_raw_cw(d, p, 5, L, [(L + 1, bytes(L + 1))] + [None] * (n - 1)))])), MALFORMED),
        (g, peer, framed(ae([wrap(_raw_cw(d, p, 5, L, [None] * n, b"\x01" + vi(5) + bytes(5)))])), MALFORMED),  # data_copy
        (g, peer, framed(ae([wrap(good_cw, b"\x02")])), MALFORMED),                # external not a bool
        (g, peer, framed(ae([wrap(_raw_cw(d, p, 1 << 32, -(-(1 << 32) // d), [None] * n))])), MALFORMED),
        (g, peer, framed(ae([wrap(_raw_cw(d, p, 5, L, [None] * (n - 1)))])), MALFORMED),          # T - 1 Options
        (g, me, framed(body), MALFORMED),                                          # from me
        (g, n, framed(body), MALFORMED),                                           # from a peer >= population
        (G + 3, peer, framed(body), MALFORMED),                                    # a group >= n_groups
        (g, peer, framed(vi(1) + vi(4)), 0x80000001),                              # LeaseMsg
        (g, peer, framed(vi(0) + vi(3) + vi(9) + vi(0) + vi(0)), 3),               # another PeerMsg
        (g, peer, framed(vi(0) + vi(1 << 16)), MALFORMED),                         # variant >= 2^16
    ]
    return out


class Harness:
    """one device follower and its restatement, fed batch after batch"""

    def __init__(self, n, G, window=64, sharded=False, seed=0, frames_per_group=6, dls=(1, 10, 250, 251, 3000), append_variant=0,
                 reply_variant=1, meta_variant=0, log_variant=1, me=None, ctx=None):
        import torch
        from summerset_b200.api import Context
        from summerset_b200.engine import Follower
        self.torch = torch
        self.rng = random.Random(seed)
        self.n, self.G, self.me, self.d = n, G, n - 1 if me is None else me, n // 2 + 1
        self.ctx = Context(0) if ctx is None else ctx
        self.av, self.lv = append_variant, log_variant
        self.fol = Follower(self.ctx, G, n, self.me, window, append_variant, reply_variant, meta_variant, log_variant)
        self.W = self.fol.W
        self.models = [Group(n, self.W, reply_variant, meta_variant) for _ in range(G)]
        peers = [q for q in range(n) if q != self.me]
        self.streams = [_leader_stream(self.rng, n, peers, frames_per_group, sharded, self.me, dls) for _ in range(G)]
        self.stores = []                                          # every store a live entry may point into
        self.host_stores = []                                     # (address, host copy) of each store after its call
        self.absorb_room = 1 << 25                                # store bytes past the frames' regions for absorbed entries
        self.pending = [[] for _ in range(G)]                     # BEYOND frames to re-submit

    def take(self, k):
        """the next k frames of every group's stream, after its re-submitted ones"""
        out = []
        for g in range(self.G):
            out += [(g, f) for f in self.pending[g]]
            self.pending[g] = []
            out += [(g, f) for f in self.streams[g][:k]]
            self.streams[g] = self.streams[g][k:]
        return out

    def batch(self, frames, bad=(), store_short=None, wal_short=None):
        torch, rng, d = self.torch, self.rng, self.d
        # shuffle groups against each other, keeping each group's frames in order
        keyed = {}
        for g, f in frames:
            keyed.setdefault(g, []).append(f)
        order = [g for g in keyed for _ in keyed[g]]
        rng.shuffle(order)
        seq, nxt = [], {g: 0 for g in keyed}
        for g in order:
            seq.append(("ok", g, keyed[g][nxt[g]]))
            nxt[g] += 1
        for b in bad:
            seq.insert(rng.randrange(len(seq) + 1), ("bad",) + b)
        buf, offs, grp, peer = bytearray(), [], [], []
        for it in seq:
            if it[0] == "ok":
                pe, t, prev, pt, es, cm, sn = it[2]
                w, g = append_entries(t, prev, pt, [e.wire() for e in es], cm, sn, self.av), it[1]
            else:
                _, g, pe, w, _v = it
            buf += bytes(rng.randint(0, 5))                       # odd offsets
            offs.append(len(buf)); grp.append(g); peer.append(pe)
            buf += w
        pitch = lambda L: (L + 31) & ~31
        r16 = lambda x: (x + 15) & ~15
        so = wo = 0
        for it in seq:                                            # the regions frames reaching the replay reserve
            if it[0] != "ok":
                continue
            g, (pe, t, prev, pt, es, cm, sn) = it[1], it[2]
            if es and prev + len(es) >= self.models[g].start + self.W:
                continue
            so += sum(len(e.shards) * pitch(-(-e.dl // d)) for e in es)
            wo += sum(r16(len(dur_log_entry(e.to_external(), self.lv))) for e in es)
        scap = so - store_short if store_short is not None else None
        wcap = wo - wal_short if wal_short is not None else None
        dev = "cuda:0"
        store = torch.full((max(so, 1) + self.absorb_room,), 0xA5, dtype=torch.uint8, device=dev)
        wal = torch.full((max(wo, 1) + 4096,), 0xA5, dtype=torch.uint8, device=dev)
        self.stores.append(store)
        tb = torch.tensor(np.frombuffer(bytes(buf), dtype=np.uint8), device=dev)
        out = self.fol.append(tb, torch.tensor(offs, dtype=torch.int64, device=dev), torch.tensor(grp, dtype=torch.int32, device=dev),
                              torch.tensor(peer, dtype=torch.uint8, device=dev), store, wal, scap, wcap)
        torch.cuda.synchronize()
        o = {k: v.cpu().numpy() for k, v in out.items()}
        o["verdict"] = o["verdict"].view(np.uint32)
        st, wl = store.cpu().numpy(), wal.cpu().numpy()
        assert int(o["totals"][1]) == wo
        lc_before = [m.lc for m in self.models]
        assert o["commit_lo"].tolist() == lc_before
        # the cut: the first frame in frame order whose reserved region ends past a capacity
        cut_i = cut_kind = None
        s_run = w_run = 0
        for i, it in enumerate(seq):
            if it[0] != "ok":
                continue
            g, (pe, t, prev, pt, es, cm, sn) = it[1], it[2]
            if es and prev + len(es) >= self.models[g].start + self.W:
                continue
            s_run += sum(len(e.shards) * pitch(-(-e.dl // d)) for e in es)
            w_run += sum(r16(len(dur_log_entry(e.to_external(), self.lv))) for e in es)
            if cut_i is None and ((scap is not None and s_run > scap) or (wcap is not None and w_run > wcap)):
                cut_i, cut_kind = i, STORE_FULL if scap is not None and s_run > scap else WAL_FULL
        for m in self.models:
            m.absorb_room = scap is None                          # an exact store leaves no room after the regions
        s_written, w_written = np.zeros(st.size, dtype=bool), np.zeros(wl.size, dtype=bool)
        for i, it in enumerate(seq):
            if it[0] == "bad":
                assert o["verdict"][i] == it[4], (i, hex(o["verdict"][i]), hex(it[4]))
                assert o["reply_len"][i] == 0 and o["meta_len"][i] == 0 and o["wal_len"][i] == 0
                assert o["store_off"][i] == -1 and o["wal_off"][i] == -1 and o["trunc_slot"][i] == -1
                continue
            g, (pe, t, prev, pt, es, cm, sn) = it[1], it[2]
            m = self.models[g]
            if cut_i is not None and i >= cut_i and not (es and prev + len(es) >= m.start + m.W):
                assert o["verdict"][i] == cut_kind, (i, hex(o["verdict"][i]))
                assert o["reply_len"][i] == 0 and o["meta_len"][i] == 0 and o["wal_len"][i] == 0
                continue
            want = m.handle(pe, t, prev, pt, es, cm, sn)
            assert int(o["verdict"][i]) == want["verdict"], (i, hex(int(o["verdict"][i])), hex(want["verdict"]))
            if want["verdict"] == BEYOND:
                self.pending[g].append(it[2])
            ml = int(o["meta_len"][i])
            assert (o["meta"][i][:ml].tobytes() if ml else None) == want["meta"]
            if ml:
                assert not o["meta"][i][ml:].any()
            rl = int(o["reply_len"][i])
            assert (o["replies"][i][:rl].tobytes() if rl else None) == want["reply"]
            assert int(o["trunc_slot"][i]) == (-1 if want["trunc"] is None else want["trunc"])
            if want["verdict"] != ACCEPTED or not want["appended"]:
                assert o["wal_len"][i] == 0 and o["store_off"][i] == -1 and o["wal_off"][i] == -1
                assert o["reply_dst"][i] == (pe if rl else 0xFF)
                continue
            at, sat = int(o["wal_off"][i]), int(o["store_off"][i])
            for e in want["appended"]:
                rec = dur_log_entry(e.to_external(), self.lv)
                assert wl[at:at + len(rec)].tobytes() == rec
                w_written[at:at + len(rec)] = True
                at += r16(len(rec))
                L = -(-e.dl // d)
                for j in sorted(e.shards):
                    assert st[sat:sat + L].tobytes() == e.shards[j]
                    assert not st[sat + L:sat + r16(L)].any()
                    s_written[sat:sat + r16(L)] = True
                    sat += pitch(L)
            assert int(o["wal_len"][i]) == at - int(o["wal_off"][i])
        # outside the records and the appended shards only the absorbed entries' regions, placed after every frame's
        # region, may have changed
        s_written[so:int(o["totals"][0])] = True
        assert (st[~s_written] == 0xA5).all(), "store bytes outside the written regions changed"
        assert (wl[~w_written] == 0xA5).all(), "WAL bytes outside the records changed"
        self.check_state(o, seq)
        return o, seq, (so, wo)

    def check_state(self, o=None, seq=()):
        fol, d = self.fol, self.d
        pitch = lambda L: (L + 31) & ~31
        v = {k: getattr(fol, k).cpu().numpy() for k in ("start_slot", "log_end", "curr_term", "last_commit", "last_snap", "leader",
                                                         "term", "held", "data_len", "shard_addr")}
        # a store is written only by the call it was passed to, so each is copied to the host once, after that call
        for s in self.stores[len(self.host_stores):]:
            self.host_stores.append((s.data_ptr(), s.cpu().numpy()))
        stores = self.host_stores
        used = {len(stores) - 1} if stores else set()

        def read(addr, nb):
            for k, (b, arr) in enumerate(stores):
                if b <= addr and addr + nb <= b + arr.size:
                    used.add(k)
                    return arr[addr - b:addr - b + nb].tobytes()
            raise AssertionError("shard address outside every store")

        for g, m in enumerate(self.models):
            assert (v["start_slot"][g], v["log_end"][g], v["curr_term"][g], v["last_commit"][g], v["last_snap"][g], v["leader"][g]) == \
                   (m.start, m.le, m.ct, m.lc, m.ls, m.ldr), g
            for s in range(m.start, m.le):
                t, dl, sh = m.log[s]
                pos = s & (self.W - 1)
                held = int(v["held"][g][pos]) & 0xFFFFFFFF                # shard 31 is the sign bit of the int32 view
                assert v["term"][g][pos] == t and v["data_len"][g][pos] == dl and held == sum(1 << j for j in sh), (g, s)
                if not sh:
                    continue
                L = -(-dl // d)
                a = int(v["shard_addr"][g][pos])
                for r, j in enumerate(sorted(sh)):
                    assert read(a + r * pitch(L), L) == sh[j], (g, s, j)
        # a store no live entry points into is let go: later calls read only the shards of live entries
        keep = sorted(used)
        self.stores, self.host_stores = [self.stores[k] for k in keep], [stores[k] for k in keep]
        if o is not None:
            for i, it in enumerate(seq):
                if it[0] == "ok" and int(o["verdict"][i]) == ACCEPTED and o["wal_len"][i]:
                    assert o["reply_dst"][i] == self.models[it[1]].ldr

    def advance(self):
        upto = [m.lc for m in self.models]
        self.fol.advance(self.torch.tensor(upto, dtype=self.torch.int64, device="cuda:0"))
        for m in self.models:
            m.advance(m.lc)
        self.torch.cuda.synchronize()
        self.check_state()


# (population, me): me = n - 1 keeps the id the population alone; populations 2 (d = 2, p = 0), 16, 31 and 32 (d = 17,
# shard 31 held) and me = 0 and n // 2 move the peers around `me`
POPULATIONS = [pytest.param(n, n - 1, id=str(n)) for n in (2, 3, 5, 7, 9, 16, 31, 32)]
POPULATIONS += [pytest.param(n, me, id=f"{n}-me{me}") for n in (2, 3, 5, 7, 9, 16, 31, 32) for me in sorted({0, n // 2} - {n - 1})]


@pytest.mark.gpu
@pytest.mark.parametrize("n,me", POPULATIONS)
@pytest.mark.parametrize("sharded", [True, False])
def test_follower_matches_restatement(n, me, sharded):
    h = Harness(n, 64, sharded=sharded, seed=n * 10 + sharded + (0 if me == n - 1 else 1000 * (me + 1)), me=me)
    h.batch(h.take(6), bad=_bad_frames(h.rng, n, h.me, h.G) + _bad_frames(h.rng, n, h.me, h.G))


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["store", "wal"])
@pytest.mark.parametrize("short", [0, 1])
def test_follower_capacity_cut(which, short):
    # the regions of the frames that reach the replay, to the byte, then one byte less
    h = Harness(5, 32, sharded=True, seed=7, frames_per_group=4)
    o, seq, _ = h.batch(h.take(4), store_short=short if which == "store" else None, wal_short=short if which == "wal" else None)
    cut = (o["verdict"] == STORE_FULL) | (o["verdict"] == WAL_FULL)
    assert cut.any() == bool(short)


def wrap_after_advance(h, rounds, grow=3, send=5, dls=(1, 10, 251, 3000), until=None):
    """Rounds of frames that run each group's log around its ring: leaders append 1..grow entries a round, back off to
    the follower's log, rewrite uncommitted suffixes in new terms and send up to `send` entries a frame, past the window
    too; BEYOND frames come back after each advance.  Stops after `rounds` or once until(h) holds; returns the number of
    BEYOND verdicts."""
    rng, d, n = h.rng, h.d, h.n
    peers = [q for q in range(n) if q != h.me]
    logs = [[(0, None)] for _ in range(h.G)]                      # the leader's (term, Ent) per slot
    terms = [1] * h.G
    safe = [0] * h.G                                              # the highest commit sent: no leader rewrites below it
    beyond = 0
    for _ in range(rounds):
        frames = []
        for g, m in enumerate(h.models):
            log = logs[g]
            if rng.random() < 0.2:                                # a new leader rewrites the uncommitted suffix
                terms[g] += 1
                del log[rng.randint(safe[g] + 1, len(log)):]
            safe[g] = len(log) - 1                                # the entries of earlier rounds commit from now on
            for _ in range(rng.randint(1, grow)):
                dl = rng.choice(dls)
                L = -(-dl // d)
                log.append((terms[g], Ent(terms[g], d, n - d, dl, {j: rng.randbytes(L) for j in range(d)}, True, 0)))
            prev = min(m.le, len(log)) - 1                        # next_slot after the leader's back-off
            while prev > m.start and m.log.get(prev, (None,))[0] != log[prev][0]:
                prev -= 1
            for _ in range(rng.randint(1, 2)):
                k = rng.randint(0, send)
                es = [e for _, e in log[prev + 1:prev + 1 + k]]
                frames.append((g, (peers[rng.randrange(n - 1)], terms[g], prev, log[prev][0], es, safe[g], 0)))
                prev = min(prev + len(es), len(log) - 1)
        h.pending, pend = [[] for _ in range(h.G)], h.pending
        o, seq, _ = h.batch([(g, f) for g in range(h.G) for f in pend[g]] + frames)
        beyond += int((o["verdict"] == BEYOND).sum())
        h.advance()
        if until is not None and until(h):
            break
    return beyond


@pytest.mark.gpu
def test_follower_window_wrap_after_advance():
    # a ring of 8: each group's log runs several times around it, frames of up to 8 entries run past its end
    h = Harness(5, 16, window=8, seed=3, frames_per_group=0)
    beyond = wrap_after_advance(h, 14, grow=4, send=8)
    assert beyond > 0
    assert max(m.le for m in h.models) > 3 * h.W                  # ring positions were reused
    assert max(m.start for m in h.models) > 2 * h.W


def _parse_reply_py(fr: bytes, variant: int):
    """-> (kind, term, end_slot, conflict) as the leader decodes an AppendEntriesReply frame; kind None = decoded"""
    if len(fr) < 8:
        return MALFORMED, None
    ln = int.from_bytes(fr[:8], "big")
    b = fr[8:8 + ln]
    if len(b) != ln:
        return MALFORMED, None
    pos = 0

    def get():
        nonlocal pos
        if pos >= len(b):
            raise ValueError
        t = b[pos]
        w = 1 if t < 251 else {251: 3, 252: 5, 253: 9}.get(t)
        if w is None or pos + w > len(b):
            raise ValueError
        v = t if t < 251 else int.from_bytes(b[pos + 1:pos + w], "little")
        pos += w
        return v

    try:
        v = get()
        if v != 0:
            return (0x80000000 | v if v < 1 << 16 else MALFORMED), None
        v = get()
        if v != variant:
            return (v if v < 1 << 16 else MALFORMED), None
        term, end = get(), get()
        if pos >= len(b):
            raise ValueError
        tag = b[pos]
        pos += 1
        conflict = None
        if tag == 1:
            conflict = (get(), get())
        elif tag != 0:
            raise ValueError
        if pos != len(b):
            raise ValueError
        return None, (term, end, conflict)
    except ValueError:
        return MALFORMED, None


@pytest.mark.gpu
def test_replies_close_the_loop_through_the_engine():
    import torch
    from summerset_b200.engine import RaftEngine, append_reply_parse
    n, G = 5, 16
    h = Harness(n, G, seed=11, frames_per_group=5)
    o, seq, _ = h.batch(h.take(5))
    ctx = h.ctx
    eng = RaftEngine(ctx, G, n, fault_tolerance=0, craft=True)
    P = n - 1
    le = max(m.le for m in h.models) - 1
    eng.append(torch.full((G,), min(le, 60), dtype=torch.int32, device="cuda:0"))
    term = max(m.ct for m in h.models)
    eng.curr_term.fill_(term)
    eng.terms.fill_(term)
    frames = []                                                   # (group, peer, bytes)
    for i, it in enumerate(seq):
        rl = int(o["reply_len"][i])
        if rl:
            frames.append((it[1], i % P, o["replies"][i][:rl].tobytes()))
    ok = reply(term, 3)
    frames += [(0, 1, reply(term + 1, 3)), (1, 2, reply(1, 1 << 32)), (2, 3, reply(term, 4, (term, 2))),
               (3, 0, framed(ok[8:-1])), (3, 0, framed(ok[8:] + b"\x00")), (4, 1, framed(ok[8:-1] + b"\x02")),
               (5, 2, framed(vi(2) + vi(1))), (6, 3, framed(vi(0) + vi(0) + vi(5))), (G + 1, 0, ok),
               (7, 0, framed(vi(0) + vi(1) + vi(1 << 40) + vi(3) + b"\x00"))]
    buf, offs = bytearray(), []
    for g, pe, fr in frames:
        buf += bytes(random.Random(len(buf)).randint(0, 3))
        offs.append(len(buf))
        buf += fr
    dev = "cuda:0"
    t = lambda a, dt: torch.tensor(a, dtype=dt, device=dev)
    rec = append_reply_parse(ctx, t(np.frombuffer(bytes(buf), dtype=np.uint8), torch.uint8), t(offs, torch.int64),
                             t([f[0] for f in frames], torch.int32), t([f[1] for f in frames], torch.uint8), eng.curr_term, G)
    torch.cuda.synchronize()
    r = {k: v.cpu().numpy() for k, v in rec.items()}
    ct_eng = eng.curr_term.cpu().numpy().view(np.uint32)
    want_g, want_p, want_e = [], [], []
    for k, (g, pe, fr) in enumerate(frames):
        kind, f = _parse_reply_py(fr, 1)
        if kind is None and g >= G:
            kind, f = MALFORMED, None
        if kind is None:
            tm, end, conf = f
            kind = HIGHER if tm > ct_eng[g] else CONFLICT if conf else END_RANGE if end >= 1 << 32 else INGEST
        else:
            tm = end = 0
            conf = None
        assert (int(r["rec_kind"][k]) & 0xFFFFFFFF) == kind, (k, hex(int(r["rec_kind"][k]) & 0xFFFFFFFF), hex(kind))
        assert int(r["rec_term"][k]) & U64 == tm and int(r["rec_conflict_term"][k]) & U64 == (conf[0] if conf else 0)
        assert int(r["rec_conflict_slot"][k]) & U64 == (conf[1] if conf else 0)
        ing = kind == INGEST
        want_g.append(g if ing else 0xFFFFFFFF); want_p.append(pe if ing else 0xFF); want_e.append(end if ing else 0)
        assert int(r["rec_group"][k]) & 0xFFFFFFFF == want_g[-1] and int(r["rec_peer"][k]) == want_p[-1]
        assert int(r["rec_end_slot"][k]) & 0xFFFFFFFF == want_e[-1]
    kinds = (r["rec_kind"].view(np.uint32)).tolist()
    for k in (INGEST, CONFLICT, HIGHER, END_RANGE, MALFORMED, 0x80000002, 0):
        assert k in kinds, hex(k)
    ns, mt, lc, ls = (eng.next_slot.cpu().numpy().view(np.uint32).copy(), eng.match.cpu().numpy().view(np.uint32).copy(),
                      eng.last_commit.cpu().numpy().view(np.uint32).copy(), eng.last_snap.cpu().numpy().view(np.uint32).copy())
    lend, ctm, tms = (eng.log_end.cpu().numpy().view(np.uint32).copy(), eng.curr_term.cpu().numpy().view(np.uint32).copy(),
                      eng.terms.cpu().numpy().view(np.uint32).copy())
    eng.on_append_replies(rec["rec_group"], rec["rec_peer"], rec["rec_end_slot"])
    eng.tick()
    torch.cuda.synchronize()
    # the oracle takes the records decoded here in Python, not the device's
    oracle.raft_reply_stream(np.array(want_g, dtype=np.uint32), np.array(want_p, dtype=np.uint8),
                             np.array(want_e, dtype=np.uint64).astype(np.uint32), P, eng.threshold, ns, mt, lc, ls, lend, ctm, tms)
    assert (eng.next_slot.cpu().numpy().view(np.uint32) == ns).all()
    assert (eng.match.cpu().numpy().view(np.uint32) == mt).all()
    assert (eng.last_commit.cpu().numpy().view(np.uint32) == lc).all()
    assert (eng.last_snap.cpu().numpy().view(np.uint32) == ls).all()
    eng.close()


@pytest.mark.gpu
def test_codeword_parsers_agree_with_the_acceptor():
    # the follower's cw_parse and the acceptor's inline parse of the same codewords: both accept or both refuse
    import torch
    from summerset_b200.engine import Acceptor, Follower
    from summerset_b200.api import Context
    n, d, p = 5, 3, 2
    L = -(-5 // d)
    cws = [codeword(d, p, 5, {0: bytes(L)}), codeword(d, p, 5, {j: bytes([j]) * L for j in range(5)}), codeword(d, p, 0, {}),
           codeword(d, p, 70000, {}), codeword(d + 1, p - 1, 5, {}), codeword(d, p + 1, 5, {}),
           _raw_cw(d, p, 5, L + 1, [None] * 5), _raw_cw(d, p, 5, L - 1, [None] * 5),
           _raw_cw(d, p, 5, L, [(L + 1, bytes(L + 1))] + [None] * 4), _raw_cw(d, p, 5, L, [None] * 4),
           _raw_cw(d, p, 5, L, [None] * 6), _raw_cw(d, p, 5, L, [None] * 5, b"\x01" + vi(5) + bytes(5)),
           _raw_cw(d, p, 5, L, [None] * 5, b"\x02"), _raw_cw(d, p, 1 << 32, -(-(1 << 32) // d), [None] * 5),
           bytes([d, p]) + vi(5) + b"\xfb\x02\x00" + vi(5) + b"\x00" * 6,                   # non-minimal shard_len
           _raw_cw(d, p, 5, L, [None] * 4 + [(L, bytes(L))])[:-3]]                          # truncated
    ctx = Context(0)
    acc = Acceptor(ctx, "rspaxos", len(cws), n, 1, d, n)
    fol = Follower(ctx, len(cws), n, 1)
    dev = "cuda:0"
    t = lambda a, dt: torch.tensor(a, dtype=dt, device=dev)
    verdicts = []
    for kind in ("acc", "fol"):
        buf, offs = bytearray(), []
        for cw in cws:
            buf += b"\x00"
            offs.append(len(buf))
            buf += framed(vi(0) + vi(2) + vi(1) + vi(1) + cw) if kind == "acc" else \
                framed(vi(0) + vi(0) + vi(1) + vi(0) + vi(0) + vi(1) + vi(1) + cw + b"\x01" + vi(0) + vi(0) + vi(0))
        args = (t(np.frombuffer(bytes(buf), dtype=np.uint8), torch.uint8), t(offs, torch.int64),
                t(list(range(len(cws))), torch.int32), t([0] * len(cws), torch.uint8),
                torch.zeros(1 << 20, dtype=torch.uint8, device=dev), torch.zeros(1 << 20, dtype=torch.uint8, device=dev))
        out = acc.accept(*args) if kind == "acc" else fol.append(*args)
        torch.cuda.synchronize()
        verdicts.append(out["verdict"].cpu().numpy().view(np.uint32))
    bad_a, bad_f = verdicts[0] == MALFORMED, verdicts[1] == MALFORMED
    assert bad_a.tolist() == bad_f.tolist()
    assert bad_a.sum() >= 8 and (~bad_a).sum() >= 4
    acc.close()
    fol.close()
