"""CRaft elections on the follower: ss_follower_campaign, ss_follower_vote, ss_follower_tally and the vote view.

`Node` restates, per message, become_a_candidate (craft/leadership.rs:143-209), handle_msg_request_vote
(craft/messages.rs:499-591) and handle_msg_request_vote_reply (:593-619) with check_term, over the follower state of
tests/test_follower.py's `Group` (whose append handler is unchanged) and the election words the device keeps beside it:
vote_term / voted_for, counted while vote_term == curr_term, and role_term / role / votes, counted while
role_term == curr_term and leader == me.  GPU tests compare every cell, verdict, won entry and state word with the
restatement, and run a leader crash end to end: campaigns, votes, tally, step-up, reconstruct reads and execution.
"""
from __future__ import annotations

import ctypes as C
import random

import numpy as np
import pytest

from tests import test_craft_leader as tl
from tests import test_craft_stepup as ts
from tests import test_follower as tf

vi, framed = tf.vi, tf.framed
NONE = 0xFF
U32 = (1 << 32) - 1
U64 = (1 << 64) - 1
MALFORMED = 0xFFFFFFFF
FOLLOWER, CANDIDATE, ELECTED = range(3)
DONE, IGNORED, NOT_FOLLOWER, OTHER_LEADER, RANGE = range(5)
GRANTED, DENIED_STALE, NO_REPLY = range(0xFFFFFFF0, 0xFFFFFFF3)
HIGHER, ELECTED_ALREADY, NOT_CANDIDATE, STALE, DENIED, DUPLICATE, COUNTED, WON = range(0xFFFFFFF0, 0xFFFFFFF8)
RV, RVR = 2, 3                      # PeerMsg::RequestVote, PeerMsg::RequestVoteReply (craft/mod.rs:239-246)
CANARY = 0xA5


# ---- bincode ------------------------------------------------------------------------------------------------------
def request_vote(term, last_slot, last_term, variant=RV) -> bytes:
    """PeerMessage::Msg{RequestVote{term, last_slot, last_term}} behind its length"""
    return framed(vi(0) + vi(variant) + vi(term) + vi(last_slot) + vi(last_term))


def vote_reply(term, granted, variant=RVR) -> bytes:
    """PeerMessage::Msg{RequestVoteReply{term, granted}} behind its length"""
    return framed(vi(0) + vi(variant) + vi(term) + bytes([1 if granted else 0]))


def metadata(term, voted_for, variant=0) -> bytes:
    """DurEntry::Metadata{curr_term, voted_for} (None = ReplicaId::MAX) behind its length"""
    return framed(vi(variant) + vi(term) + bytes([voted_for]))


# ---- the per-message restatement ----------------------------------------------------------------------------------
class Node(tf.Group):
    """one group's follower state at replica `me`, with the election words; returns what each message produces"""

    def __init__(self, n, W, me, request_vote_variant=RV, reply_variant=RVR, meta_variant=0):
        super().__init__(n, W, meta_variant=meta_variant)
        self.me, self.maj, self.n = me, n // 2 + 1, n
        self.rvv, self.rpv = request_vote_variant, reply_variant
        self.vt, self.vf, self.rt, self.role, self.votes = 0, NONE, 0, FOLLOWER, 0

    def voted(self):
        return self.vf if self.vt == self.ct else NONE

    def role_now(self):
        return self.role if self.rt == self.ct and self.ldr == self.me else FOLLOWER

    def campaign(self, timeout_source=None):
        """-> (verdict, meta, frame)"""
        if self.role_now() != FOLLOWER:
            return NOT_FOLLOWER, None, None
        if timeout_source is not None and self.ldr != NONE and self.ldr != timeout_source:
            return OTHER_LEADER, None, None
        if self.ct + 1 >= 1 << 32:
            return RANGE, None, None
        self.ct += 1
        self.ldr = self.me
        self.vt, self.vf, self.rt, self.role, self.votes = self.ct, self.me, self.ct, CANDIDATE, 1 << self.me
        last = self.le - 1
        return DONE, metadata(self.ct, self.me, self.mv), request_vote(self.ct, last, self.log[last][0], self.rvv)

    def vote(self, cand, term, last_slot, last_term):
        """-> (verdict, meta, reply)"""
        vf, meta = self.voted(), False
        if term > self.ct:                                        # check_term
            self.ct, vf, self.ldr, meta = term, NONE, cand, True
        if term < self.ct:
            v, rep = DENIED_STALE, vote_reply(self.ct, False, self.rpv)
        elif (vf in (NONE, cand)) and (last_term >= self.log[self.le - 1][0] or (last_term == self.ct and last_slot + 1 >= self.le)):
            vf, meta = cand, True
            v, rep = GRANTED, vote_reply(self.ct, True, self.rpv)
        else:
            v, rep = NO_REPLY, None
        if meta:
            self.vt, self.vf = self.ct, vf
        return v, metadata(self.ct, vf, self.mv) if meta else None, rep

    def tally(self, peer, term, granted):
        """-> (verdict, meta)"""
        if term > self.ct:                                        # check_term: step down
            self.ct, self.ldr, self.vt, self.vf = term, peer, term, NONE
            return HIGHER, metadata(term, NONE, self.mv)
        r = self.role_now()
        if r == ELECTED:
            return ELECTED_ALREADY, None
        if r != CANDIDATE:
            return NOT_CANDIDATE, None
        if term < self.ct:
            return STALE, None
        if not granted:
            return DENIED, None
        if self.votes >> peer & 1:
            return DUPLICATE, None
        self.votes |= 1 << peer
        if bin(self.votes).count("1") >= self.maj:
            self.role = ELECTED
            return WON, None
        return COUNTED, None


def campaign_batch(nodes, listing, sources):
    seen, out = set(), []
    for i, g in enumerate(listing):
        if g >= len(nodes) or g in seen:
            out.append((IGNORED, None, None))
            continue
        seen.add(g)
        out.append(nodes[g].campaign(None if sources is None else sources[i]))
    return out


def tally_batch(nodes, frames):
    """frames: (g, peer, term, granted) -> (per-frame results, won groups in group order)"""
    res, won = [], set()
    for g, peer, term, granted in frames:
        v, m = nodes[g].tally(peer, term, granted)
        res.append((v, m))
        if v == WON:
            won.add(g)
        elif v == HIGHER:
            won.discard(g)
    return res, sorted(won)


# ---- CPU: bytes -------------------------------------------------------------------------------------------------------
def test_request_vote_bytes_at_every_varint_width():
    assert request_vote(5, 7, 4) == bytes([0, 0, 0, 0, 0, 0, 0, 5, 0, 2, 5, 7, 4])
    assert request_vote(300, 70000, 1 << 40) == (bytes([0] * 7 + [19, 0, 2, 0xFB, 0x2C, 0x01, 0xFC, 0x70, 0x11, 0x01, 0x00, 0xFD])
                                                 + bytes([0, 0, 0, 0, 0, 1, 0, 0]))
    widest = request_vote(U64, U64, U64, variant=65535)            # the widest frame: 39 bytes of its 48-byte cell
    assert widest == bytes([0] * 7 + [31, 0, 0xFB, 0xFF, 0xFF]) + (b"\xfd" + b"\xff" * 8) * 3 and len(widest) == 39


def test_request_vote_reply_and_metadata_bytes():
    assert vote_reply(7, True) == bytes([0] * 7 + [4, 0, 3, 7, 1])
    assert vote_reply(251, False) == bytes([0] * 7 + [6, 0, 3, 0xFB, 0xFB, 0x00, 0])
    assert vote_reply(1 << 16, True) == bytes([0] * 7 + [8, 0, 3, 0xFC, 0, 0, 1, 0, 1])
    assert vote_reply(U64, True, variant=65535) == bytes([0] * 7 + [14, 0, 0xFB, 0xFF, 0xFF, 0xFD] + [0xFF] * 8 + [1])
    assert metadata(3, 1) == bytes([0] * 7 + [3, 0, 3, 1])
    assert metadata(1 << 32, NONE) == bytes([0] * 7 + [11, 0, 0xFD, 0, 0, 0, 0, 1, 0, 0, 0, 0xFF])
    widest = metadata(U64, NONE, variant=65535)                     # 21 bytes of its 32-byte cell
    assert widest == bytes([0] * 7 + [13, 0xFB, 0xFF, 0xFF, 0xFD] + [0xFF] * 9) and len(widest) == 21
    assert metadata(2, NONE) == tf.dur_metadata(2)                  # the append's check_term cell


# ---- CPU: the restatement ---------------------------------------------------------------------------------------------
def _node(n=5, me=0, terms=(0,), ct=0, ldr=NONE):
    nd = Node(n, 64, me)
    nd.log = {s: (t, 0, {}) for s, t in enumerate(terms)}
    nd.le, nd.ct, nd.ldr = len(terms), ct, ldr
    return nd


def test_model_grant_quirk_equal_last_term_shorter_log():
    # my log: slots 0..4, last term 3; the candidate's last entry is slot 2 of term 3 -- textbook Raft refuses (shorter
    # log), the reference's test grants: last_term >= my last term
    nd = _node(terms=(0, 1, 3, 3, 3), ct=3)
    assert nd.vote(2, 4, 2, 3) == (GRANTED, metadata(4, 2), vote_reply(4, True))
    # an older last term is refused unless last_term == curr_term and last_slot + 1 >= log_end
    nd = _node(terms=(0, 1, 3, 3, 3), ct=3)
    assert nd.vote(2, 4, 9, 1) == (NO_REPLY, metadata(4, NONE), None)
    nd = _node(terms=(0, 1, 4, 4, 5), ct=5)
    assert nd.vote(1, 5, 4, 5)[0] == GRANTED                        # last_term 5 >= 5
    nd = _node(terms=(0, 1, 4, 4, 6), ct=6)
    assert nd.vote(1, 6, 4, 5)[0] == NO_REPLY                       # 5 < 6 and 5 != curr_term
    nd = _node(terms=(0, 7), ct=7)
    nd.log[1] = (8, 0, {})                                          # a last term above curr_term (installed state)
    assert nd.vote(1, 7, 1, 7)[0] == GRANTED                        # last_term == curr_term, last_slot + 1 >= log_end
    nd = _node(terms=(0, 7), ct=7)
    nd.log[1] = (8, 0, {})
    assert nd.vote(1, 7, 0, 7)[0] == NO_REPLY                       # a slot short


def test_model_vote_repeats_other_candidates_and_stale_terms():
    nd = _node(terms=(0, 2), ct=2, ldr=0)
    assert nd.vote(1, 2, 1, 2)[0] == GRANTED and nd.voted() == 1
    assert nd.vote(1, 2, 1, 2) == (GRANTED, metadata(2, 1), vote_reply(2, True))   # the same candidate again
    assert nd.vote(3, 2, 1, 2) == (NO_REPLY, None, None)                        # another candidate, same term
    assert nd.vote(3, 1, 1, 2) == (DENIED_STALE, None, vote_reply(2, False))
    assert nd.vote(3, 3, 1, 2) == (GRANTED, metadata(3, 3), vote_reply(3, True)) and nd.ldr == 3
    # a candidate refuses another's RequestVote in its own term
    nd = _node(me=0, terms=(0, 2), ct=2)
    assert nd.campaign()[0] == DONE and nd.ct == 3
    assert nd.vote(4, 3, 1, 2) == (NO_REPLY, None, None) and nd.role_now() == CANDIDATE


def test_model_tally_stale_duplicate_and_higher_term_replies():
    nd = _node(n=5, me=2, terms=(0, 1), ct=1, ldr=0)
    assert nd.campaign(timeout_source=0)[0] == DONE and nd.ct == 2 and nd.ldr == 2
    assert nd.tally(1, 1, True) == (STALE, None)                   # a reply to an older campaign
    assert nd.tally(1, 2, False) == (DENIED, None)
    assert nd.tally(1, 2, True) == (COUNTED, None)
    assert nd.tally(1, 2, True) == (DUPLICATE, None)               # votes are a set
    assert nd.tally(3, 2, True) == (WON, None) and nd.role_now() == ELECTED
    assert nd.tally(4, 2, True) == (ELECTED_ALREADY, None)
    assert nd.tally(4, 3, False) == (HIGHER, metadata(3, NONE)) and nd.role_now() == FOLLOWER and nd.ldr == 4
    assert nd.tally(1, 3, True) == (NOT_CANDIDATE, None)
    # within one batch a later higher term takes the win back
    a = _node(n=3, me=0, terms=(0,), ct=0)
    b = _node(n=3, me=0, terms=(0,), ct=0)
    a.campaign(), b.campaign()
    res, won = tally_batch([a, b], [(0, 1, 1, True), (1, 2, 1, True), (1, 1, 5, False)])
    assert [v for v, _ in res] == [WON, WON, HIGHER] and won == [0]


def test_model_same_term_append_ends_a_candidacy():
    nd = _node(n=5, me=1, terms=(0, 1, 1), ct=1, ldr=0)
    assert nd.campaign(0)[0] == DONE and nd.role_now() == CANDIDATE
    o = nd.handle(3, 2, 2, 1, [], 0, 0)                             # the elected leader's heartbeat, same term
    assert o["verdict"] == tf.ACCEPTED and o["meta"] is None and nd.ldr == 3 and nd.role_now() == FOLLOWER
    assert nd.voted() == 1                                          # the vote stands for the term
    assert nd.tally(2, 2, True) == (NOT_CANDIDATE, None)
    assert nd.campaign(None)[0] == DONE and nd.ct == 3              # a later timeout starts a new campaign
    o = nd.handle(4, 5, 2, 1, [], 0, 0)                             # a term raise ends it too
    assert o["meta"] == tf.dur_metadata(5) and nd.role_now() == FOLLOWER and nd.voted() == NONE


def test_model_campaign_verdict_order():
    nd = _node(me=0, ct=4, ldr=2)
    assert campaign_batch([nd], [0, 0, 7], [1, 2, 2]) == [(OTHER_LEADER, None, None), (IGNORED, None, None), (IGNORED, None, None)]
    assert nd.campaign(2)[0] == DONE
    assert nd.campaign(2)[0] == NOT_FOLLOWER                        # before OTHER_LEADER
    nd = _node(me=0, ct=U32, ldr=3)
    assert nd.campaign(1)[0] == OTHER_LEADER                        # before RANGE
    assert nd.campaign(3)[0] == RANGE and nd.campaign(None)[0] == RANGE
    nd = _node(me=0, ct=U32 - 1, terms=(0, 9))
    assert nd.campaign() == (DONE, metadata(U32, 0), request_vote(U32, 1, 9))


# ---- CPU: refusals --------------------------------------------------------------------------------------------------
def test_refusals_without_a_device():
    from summerset_b200 import _lib
    lib = _lib.load()

    def refused(rc, why):
        assert rc == _lib.SS_ERR_INVALID_ARG and why in lib.ss_last_error().decode(), (rc, lib.ss_last_error(), why)

    refused(lib.ss_follower_vote_view_get(None, C.byref(_lib.FollowerVoteView())), "null argument")
    refused(lib.ss_follower_campaign(None, 16, 1, None, 1 << 16, 16, 16, 16, 16, 16, 16), "2^16")
    refused(lib.ss_follower_campaign(None, 16, 1, None, RV, 16, 16, 16, 16, 16, 16), "null follower")
    refused(lib.ss_follower_vote(None, 16, 0, 16, 16, 16, 1, 1 << 16, RVR, 16, 16, 16, 16, 16, 16), "2^16")
    refused(lib.ss_follower_vote(None, 16, 0, 16, 16, 16, 1, RV, 1 << 16, 16, 16, 16, 16, 16, 16), "2^16")
    refused(lib.ss_follower_vote(None, 16, 0, 16, 16, 16, 1, RV, RVR, 16, 16, 16, 16, 16, 16), "null follower")
    refused(lib.ss_follower_tally(None, 16, 0, 16, 16, 16, 1, 1 << 16, 16, 16, 16, 16, 16, None), "2^16")
    refused(lib.ss_follower_tally(None, 16, 0, 16, 16, 16, 1, RVR, 16, 16, 16, 16, 16, None), "null follower")


def test_no_device_without_a_context():
    from summerset_b200 import _lib
    lib = _lib.load()
    h = C.c_void_p()
    cfg = _lib.FollowerConfig(_lib.SS_PROTO_CRAFT, 5, 1, 0, 0, 1, 0, 1)
    rc = lib.ss_follower_create(None, C.byref(cfg), 4, C.byref(h))
    import torch
    assert rc == (_lib.SS_ERR_INVALID_ARG if torch.cuda.is_available() else _lib.SS_ERR_NO_DEVICE)


# ---- GPU: against the restatement -------------------------------------------------------------------------------------
PAD = 64


def _canary(n, dt):
    """a device buffer of n + PAD elements filled with the canary byte -> (tensor, the first n)"""
    import torch
    t = torch.full(((n + PAD) * torch.tensor([], dtype=dt).element_size(),), CANARY, dtype=torch.uint8, device="cuda:0").view(dt)
    return t


def _padded_ok(t, n):
    b = t.cpu().numpy().view(np.uint8)
    es = t.element_size()
    return (b[n * es:] == CANARY).all()


def _cells_ok(cells, lens, want, width):
    """cell i holds want[i] then zeros to its end, or is untouched (all canary) when want[i] is None"""
    c = cells.cpu().numpy().view(np.uint8)
    assert _padded_ok(cells, len(want) * width)
    ln = lens.cpu().numpy()
    for i, w in enumerate(want):
        cell = c[i * width:(i + 1) * width]
        if w is None:
            assert ln[i] == 0 and (cell == CANARY).all(), i
        else:
            assert ln[i] == len(w) and cell[:len(w)].tobytes() == w and (cell[len(w):] == 0).all(), (i, cell.tobytes(), w)


class _Rig:
    """one device follower (replica `me`) and the restatement of each of its G groups"""

    def __init__(self, n, G, seed, request_vote_variant=RV, reply_variant=RVR, meta_variant=0):
        import torch
        from summerset_b200 import _lib
        from summerset_b200.engine import Follower
        self.rng = random.Random(seed)
        self.n, self.G, self.W = n, G, 64
        self.me = self.rng.randrange(n)
        self.ctx = ts._ctx()
        self.lib = self.ctx.lib
        self.rvv, self.rpv = request_vote_variant, reply_variant
        self.fol = Follower(self.ctx, G, n, self.me, window=self.W, meta_variant=meta_variant)
        self.vv = self.fol.vote_view()
        self.nodes = [Node(n, self.W, self.me, request_vote_variant, reply_variant, meta_variant) for _ in range(G)]
        cts = [0, 1, 2, 5, 250, 251, 300, 70000, (1 << 32) - 2, U32, 1 << 40]
        ct_t, le_t, ld_t = [], [], []
        term = self.fol.term.cpu().numpy()
        for g, nd in enumerate(self.nodes):
            ct = self.rng.choice(cts)
            le = self.rng.randint(1, 6)
            terms = [0] + sorted(self.rng.randint(0, min(ct, 4)) if self.rng.random() < 0.7 else ct for _ in range(le - 1))
            nd.log = {s: (t, 0, {}) for s, t in enumerate(terms)}
            nd.le, nd.ct = le, ct
            nd.ldr = self.rng.choice([NONE, NONE, self.me, self.rng.randrange(n)])
            for s, t in enumerate(terms):
                term[g][s & (self.W - 1)] = t
            ct_t.append(ct), le_t.append(le), ld_t.append(nd.ldr)
        self.fol.term.copy_(torch.from_numpy(term))
        self.fol.curr_term.copy_(ts._t(ct_t, torch.int64))
        self.fol.log_end.copy_(ts._t(le_t, torch.int64))
        self.fol.leader.copy_(ts._t(ld_t, torch.uint8))
        torch.cuda.synchronize()
        self._lib = _lib

    def check_state(self):
        import torch
        torch.cuda.synchronize()
        f, vv = self.fol, self.vv
        assert f.curr_term.cpu().tolist() == [nd.ct for nd in self.nodes]
        assert f.leader.cpu().tolist() == [nd.ldr for nd in self.nodes]
        assert f.log_end.cpu().tolist() == [nd.le for nd in self.nodes]
        assert vv["vote_term"].cpu().tolist() == [nd.vt for nd in self.nodes]
        assert vv["voted_for"].cpu().tolist() == [nd.vf for nd in self.nodes]
        assert vv["role_term"].cpu().tolist() == [nd.rt for nd in self.nodes]
        assert vv["role"].cpu().tolist() == [nd.role for nd in self.nodes]
        assert (vv["votes"].cpu().numpy().view(np.uint32) == np.array([nd.votes for nd in self.nodes], dtype=np.uint32)).all()

    def campaign(self, listing, sources):
        import torch
        n = len(listing)
        want = campaign_batch(self.nodes, listing, sources)
        grp = _canary(n, torch.int32)
        grp[:n] = ts._t(np.array(listing, dtype=np.uint32).view(np.int32), torch.int32)
        src = None
        if sources is not None:
            src = _canary(n, torch.uint8)
            src[:n] = ts._t(sources, torch.uint8)
        meta, ml, fr, fl, fd, vd = (_canary(32 * n, torch.uint8), _canary(n, torch.int32), _canary(48 * n, torch.uint8),
                                    _canary(n, torch.int32), _canary(n, torch.uint8), _canary(n, torch.int32))
        p = lambda x: None if x is None else x.data_ptr()
        self._lib.check(self.lib.ss_follower_campaign(self.fol.h, p(grp), n, p(src), self.rvv, p(meta), p(ml), p(fr), p(fl), p(fd), p(vd)))
        torch.cuda.synchronize()
        assert (vd.cpu().numpy()[:n].view(np.uint32) == [v for v, _, _ in want]).all() and _padded_ok(vd, n)
        _cells_ok(meta, ml, [m for _, m, _ in want], 32)
        _cells_ok(fr, fl, [x for _, _, x in want], 48)
        assert (fd.cpu().numpy()[:n] == NONE).all() and _padded_ok(fd, n)
        self.check_state()
        return want

    def _frames(self, frames):
        """(g, peer, bytes) -> device buf, frame_off, frame_group, frame_peer"""
        import torch
        buf, offs = ts._buf([x for _, _, x in frames], self.rng)
        return (buf, ts._t(offs, torch.int64), ts._t(np.array([g for g, _, _ in frames], dtype=np.uint32).view(np.int32), torch.int32),
                ts._t([p for _, p, _ in frames], torch.uint8))

    def vote(self, frames):
        """frames: (g, peer, bytes, decoded (term, last_slot, last_term) or a fixed verdict)"""
        import torch
        n = len(frames)
        want = []
        for g, peer, _, dec in frames:
            want.append(self.nodes[g].vote(peer, *dec) + (peer,) if isinstance(dec, tuple) else (dec, None, None, None))
        buf, fo, fg, fp = self._frames([(g, p, x) for g, p, x, _ in frames])
        meta, ml, rep, rl, rd, vd = (_canary(32 * n, torch.uint8), _canary(n, torch.int32), _canary(32 * n, torch.uint8),
                                     _canary(n, torch.int32), _canary(n, torch.uint8), _canary(n, torch.int32))
        p = lambda x: x.data_ptr()
        self._lib.check(self.lib.ss_follower_vote(self.fol.h, p(buf), buf.numel(), p(fo), p(fg), p(fp), n, self.rvv, self.rpv, p(meta), p(ml),
                                                  p(rep), p(rl), p(rd), p(vd)))
        torch.cuda.synchronize()
        assert (vd.cpu().numpy()[:n].view(np.uint32) == [w[0] for w in want]).all() and _padded_ok(vd, n)
        _cells_ok(meta, ml, [w[1] for w in want], 32)
        _cells_ok(rep, rl, [w[2] for w in want], 32)
        assert rd.cpu().tolist()[:n] == [NONE if w[2] is None else w[3] for w in want] and _padded_ok(rd, n)
        self.check_state()
        return want

    def tally(self, frames):
        """frames: (g, peer, bytes, decoded (term, granted) or a fixed verdict)"""
        import torch
        n, G = len(frames), self.G
        want, decoded = [], [(g, p, *dec) for g, p, _, dec in frames if isinstance(dec, tuple)]
        res, won = tally_batch(self.nodes, decoded)
        it = iter(res)
        for _, _, _, dec in frames:
            want.append(next(it) if isinstance(dec, tuple) else (dec, None))
        buf, fo, fg, fp = self._frames([(g, p, x) for g, p, x, _ in frames])
        meta, ml, vd = _canary(32 * n, torch.uint8), _canary(n, torch.int32), _canary(n, torch.int32)
        wg, wt, nw = _canary(G, torch.int32), _canary(G, torch.int64), _canary(1, torch.int64)
        p = lambda x: x.data_ptr()
        self._lib.check(self.lib.ss_follower_tally(self.fol.h, p(buf), buf.numel(), p(fo), p(fg), p(fp), n, self.rpv, p(meta), p(ml), p(vd),
                                                   p(wg), p(wt), p(nw)))
        torch.cuda.synchronize()
        assert (vd.cpu().numpy()[:n].view(np.uint32) == [w[0] for w in want]).all() and _padded_ok(vd, n)
        _cells_ok(meta, ml, [w[1] for w in want], 32)
        wgn = wg.cpu().numpy()[:G].view(np.uint32)
        assert wgn.tolist() == won + [U32] * (G - len(won)) and _padded_ok(wg, G)
        assert wt.cpu().tolist()[:G] == [self.nodes[g].ct for g in won] + [0] * (G - len(won)) and _padded_ok(wt, G)
        assert int(nw[0]) == len(won) and _padded_ok(nw, 1)
        self.check_state()
        return want, won


def _bad_votes(rig):
    """malformed and other-message RequestVote frames, and their verdicts"""
    G, n, me = rig.G, rig.n, rig.me
    ok = request_vote(1, 0, 0, rig.rvv)
    other = (me + 1) % n
    foreign = 0 if rig.rvv else 1                                  # another PeerMsg (AppendEntries by default)
    return [(0, other, framed(ok[8:-1]), MALFORMED),                             # truncated body
            (0, other, framed(ok[8:] + b"\x00"), MALFORMED),                      # a trailing byte
            (1, me, ok, MALFORMED),                                               # from me
            (1, n if n < 32 else 200, ok, MALFORMED),                             # a peer past the population
            (G + 3, other, ok, MALFORMED),                                        # a group past n_groups
            (2, other, request_vote(1, 0, 0, variant=foreign), foreign),          # another PeerMsg
            (2, other, framed(vi(1) + vi(0)), 0x80000001),                        # another PeerMessage
            (2, other, framed(vi(0) + vi(70000)), MALFORMED)]                     # a variant >= 2^16


def _bad_replies(rig):
    G, n, me = rig.G, rig.n, rig.me
    other = (me + 1) % n
    ok = vote_reply(1, True, rig.rpv)
    foreign = 1 if rig.rpv != 1 else 0
    return [(0, other, framed(ok[8:-1]), MALFORMED), (0, other, framed(ok[8:] + b"\x01"), MALFORMED),
            (0, other, framed(vi(0) + vi(rig.rpv) + vi(1) + b"\x02"), MALFORMED),    # granted is not a bool
            (1, me, ok, MALFORMED), (G, other, ok, MALFORMED), (1, other, vote_reply(1, True, variant=foreign), foreign)]


def _round(rig, k_vote, k_tally):
    rng, G, n, me = rig.rng, rig.G, rig.n, rig.me
    peers = [r for r in range(n) if r != me]
    # campaigns: every group once or more, some out of range, timeout sources old leaders or others
    listing = [g for g in range(G) if rng.random() < 0.7]
    listing += [rng.randrange(G) for _ in range(G // 4)] + [G, U32]
    rng.shuffle(listing)
    sources = [rig.nodes[g].ldr if g < G and rng.random() < 0.7 else rng.randrange(n) for g in listing]
    rig.campaign(listing, sources if rng.random() < 0.8 else None)
    # RequestVotes from other candidates: several per term, repeats, raises in the middle of a group's run
    frames, prev = [], []
    for _ in range(k_vote):
        if prev and rng.random() < 0.15:
            frames.append(rng.choice(prev))
            continue
        g = rng.randrange(G)
        nd = rig.nodes[g]
        term = max(0, nd.ct + rng.choice([-1, 0, 0, 1, 1, 2] if g % 3 else [-1, 0]))  # a third keep their candidacies
        ls = max(0, nd.le - 1 + rng.choice([-2, -1, 0, 0, 1, 5]))
        lt = max(0, nd.log[nd.le - 1][0] + rng.choice([-1, 0, 0, 1]))
        if rng.random() < 0.2:
            lt = term
        cand = rng.choice(peers)
        f = (g, cand, request_vote(term, ls, lt, rig.rvv), (term, ls, lt))
        frames.append(f)
        prev.append(f)
    bad = _bad_votes(rig)
    for b in bad:
        frames.insert(rng.randrange(len(frames) + 1), b)
    rig.vote(frames)
    # replies: the candidates' groups most often, old-term and duplicate replies, a higher term now and then
    frames, prev = [], []
    cands = [g for g in range(G) if rig.nodes[g].role_now() == CANDIDATE] or [0]
    for _ in range(k_tally):
        if prev and rng.random() < 0.15:
            frames.append(rng.choice(prev))
            continue
        g = rng.choice(cands) if rng.random() < 0.8 else rng.randrange(G)
        nd = rig.nodes[g]
        term = max(0, nd.ct + rng.choice([-1, 0, 0, 0, 0, 0, 1] if rng.random() < 0.9 else [3]))
        granted = rng.random() < 0.8
        f = (g, rng.choice(peers), vote_reply(term, granted, rig.rpv), (term, granted))
        frames.append(f)
        prev.append(f)
    for g in cands[:len(cands) // 3]:                            # enough granted replies, first, to elect some groups
        ct = rig.nodes[g].ct
        for q in peers:
            frames.insert(0, (g, q, vote_reply(ct, True, rig.rpv), (ct, True)))
    for b in _bad_replies(rig):
        frames.insert(rng.randrange(len(frames) + 1), b)
    return rig.tally(frames)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [3, 5, 7, 9, 32])
def test_elections_match_the_restatement(n):
    rig = _Rig(n, 96, seed=7000 + n)
    rig.check_state()                                               # the view starts with no vote and no candidacy
    total_won = 0
    for k in range(3):
        _, won = _round(rig, 3 * rig.G, 4 * rig.G)
        total_won += len(won)
    assert total_won > 0
    rig.fol.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [3, 5])
def test_append_after_a_campaign_ends_the_candidacy(n):
    import torch
    rig = _Rig(n, 32, seed=7100 + n)
    G, me = rig.G, rig.me
    rig.campaign(list(range(G)), None)
    cands = [g for g in range(G) if rig.nodes[g].role_now() == CANDIDATE]
    assert cands
    other = (me + 1) % n
    frames, want = [], []
    for k, g in enumerate(cands):
        nd = rig.nodes[g]
        term = nd.ct + (1 if k % 3 == 2 else 0)                  # a same-term heartbeat ends it, a raise too
        prev = nd.le - 1
        frames.append((g, other, tf.append_entries(term, prev, nd.log[prev][0], [], 0, 0)))
        want.append(nd.handle(other, term, prev, nd.log[prev][0], [], 0, 0))
    buf, fo, fg, fp = rig._frames(frames)
    store = torch.zeros(1 << 12, dtype=torch.uint8, device="cuda:0")
    a = rig.fol.append(buf, fo, fg, fp, store, torch.zeros(1 << 12, dtype=torch.uint8, device="cuda:0"))
    torch.cuda.synchronize()
    assert (a["verdict"].cpu().numpy().view(np.uint32) == [w["verdict"] for w in want]).all()
    ml, mc = a["meta_len"].cpu().tolist(), a["meta"].cpu().numpy()
    for i, w in enumerate(want):
        assert (mc[i][:ml[i]].tobytes() if ml[i] else None) == w["meta"]
    rig.check_state()
    assert all(rig.nodes[g].role_now() == FOLLOWER for g in cands)
    # the replies that would have elected them now find no candidacy
    rig.tally([(g, p, vote_reply(rig.nodes[g].ct, True), (rig.nodes[g].ct, True)) for g in cands for p in range(n) if p != me])
    rig.fol.close()


# ---- GPU: a closed loop ------------------------------------------------------------------------------------------------
def _deliver(fol, frames, rng, call):
    """frames (g, from, bytes) handed to a follower's vote or tally"""
    import torch
    buf, offs = ts._buf([x for _, _, x in frames], rng)
    fo, fg, fp = ts._t(offs, torch.int64), ts._t([g for g, _, _ in frames], torch.int32), ts._t([p for _, p, _ in frames], torch.uint8)
    r = getattr(fol, call)(buf, fo, fg, fp)
    torch.cuda.synchronize()
    return r


def _propose(eng, me, lens, stride, keep, batch, rng):
    """one entry for each group with lens[g] > 0, in 1-shard mode"""
    import torch
    bs = [rng.randbytes(x) for x in lens]
    arena, offs = bytearray(), []
    for b in bs:
        offs.append(len(arena))
        arena += b
    store = torch.zeros((eng.P + 1, stride), dtype=torch.uint8, device="cuda:0")
    keep.append(store)
    o = eng.propose(me, ts._t(np.frombuffer(bytes(arena) + b"\0", dtype=np.uint8), torch.uint8), ts._t(offs, torch.int64),
                    ts._t(lens, torch.int32), store, torch.zeros(1 << 22, dtype=torch.uint8, device="cuda:0"))
    slots = o["slot_out"].cpu().tolist()
    for g, x in enumerate(lens):
        if x:
            assert slots[g] >= 0
            batch[(g, slots[g])] = bs[g]


def _replicate(ctx, eng, me, fols, keep, rng, groups=None, append_variant=0, reply_variant=1):
    """the leader's entries, then a heartbeat, to every live follower (only the frames of `groups`, None = all: an
    engine's heartbeat also goes out for the groups it never stepped up); their replies ingested and ticked.  The
    followers must be configured with the same AppendEntries and AppendEntriesReply variants."""
    import torch
    from summerset_b200.engine import append_reply_parse
    dev = "cuda:0"
    for heartbeat in (False, True):
        out = torch.zeros(1 << 22, dtype=torch.uint8, device=dev)
        o = eng.pack_append(me, out, 1 << 12, heartbeat=heartbeat, msg_chunk_size=4, append_variant=append_variant)
        torch.cuda.synchronize()
        nf = int(o["n_frames"][0])
        fo, fg, fp = o["frame_off"][:nf], o["frame_group"][:nf], o["frame_peer"][:nf]
        replies = []
        for r, f in fols.items():
            q = r if r < me else r - 1
            keep_ = fp == q
            if groups is not None:
                keep_ &= torch.isin(fg, ts._t(groups, torch.int32))
            sel = keep_.nonzero().flatten()
            if sel.numel() == 0:
                continue
            st = torch.zeros(1 << 22, dtype=torch.uint8, device=dev)
            keep.append(st)
            a = f.append(out, fo[sel].contiguous(), fg[sel].contiguous(), torch.full_like(fp[sel], me), st,
                         torch.zeros(1 << 22, dtype=torch.uint8, device=dev))
            torch.cuda.synchronize()
            assert (a["verdict"].cpu().numpy().view(np.uint32) == tf.ACCEPTED).all()
            rl, cells = a["reply_len"].cpu().numpy(), a["replies"].cpu().numpy()
            replies += [(g, q, cells[i][:rl[i]].tobytes()) for i, g in enumerate(fg[sel].cpu().tolist())]
        if not replies:
            continue
        tb, offs = ts._buf([x for _, _, x in replies], rng)
        fo2, fg2 = ts._t(offs, torch.int64), ts._t([x[0] for x in replies], torch.int32)
        rec = append_reply_parse(ctx, tb, fo2, fg2, ts._t([x[1] for x in replies], torch.uint8), eng.curr_term, eng.G, reply_variant)
        eng.on_append_replies(rec["rec_group"], rec["rec_peer"], rec["rec_end_slot"])
        eng.tick()
        torch.cuda.synchronize()


@pytest.mark.gpu
def test_closed_loop_election_after_a_leader_crash():
    """Five replicas: leader 0 replicates two terms of 1-shard entries to 1..4 and crashes.  Replicas 1-4 campaign --
    one per group, or two at once for the split-vote groups, whose voters each grant the first RequestVote they see --
    then vote and tally, and each winner steps up from its follower straight from the tally's outputs, commits an entry
    of its term, reads back the shards it lacks and executes: every proposed batch comes back byte for byte, and no group
    elects two leaders in a term."""
    import torch
    from summerset_b200.engine import Follower, RaftEngine
    ctx = ts._ctx()
    n, G, W = 5, 40, 64
    d, T = n // 2 + 1, n
    dev = "cuda:0"
    rng = random.Random(7200)
    fols = {r: Follower(ctx, G, n, r, window=W) for r in range(1, n)}
    stride = G * tl.pitch(-(-3000 // d)) * 8
    keep, batch = [], {}
    old = RaftEngine(ctx, G, n, craft=True, window=W)
    old.log_view()
    for term in (1, 2):
        old.curr_term.fill_(term)
        for _ in range(2):
            _propose(old, 0, [rng.choice((1, 16, 17, 300, 3000)) for _ in range(G)], stride, keep, batch, rng)
            _replicate(ctx, old, 0, fols, keep, rng)
    le = old.log_end.cpu().tolist()
    assert old.last_commit.cpu().tolist() == [x - 1 for x in le]
    old.close()                                                 # leader 0 crashes
    # campaigns: group g's candidate is 1 + g % 4; every fifth group also has 1 + (g + 1) % 4 in the same term
    split = {g for g in range(G) if g % 5 == 0}
    cands = {g: [1 + g % 4] + ([1 + (g + 1) % 4] if g in split else []) for g in range(G)}
    rv = {}                                                     # (g, candidate) -> its RequestVote
    for r, f in fols.items():
        mine = [g for g in range(G) if r in cands[g]]
        c = f.campaign(ts._t(mine, torch.int32), ts._t([0] * len(mine), torch.uint8))
        torch.cuda.synchronize()
        assert (c["verdict"].cpu().numpy() == DONE).all() and (c["frame_dst"].cpu().numpy() == NONE).all()
        fl, fr = c["frame_len"].cpu().tolist(), c["frames"].cpu().numpy()
        for i, g in enumerate(mine):
            rv[(g, r)] = fr[i][:fl[i]].tobytes()
    # votes: in a split group the two other voters see the two candidates in opposite orders and grant the first
    replies = {r: [] for r in fols}
    for v, f in fols.items():
        frames = []
        for g in range(G):
            cs = [c for c in cands[g] if c != v]
            if len(cs) == 2 and (v + g) % 2:
                cs.reverse()
            frames += [(g, c, rv[(g, c)]) for c in cs]
        r_ = _deliver(f, frames, rng, "vote")
        rl, cells, dst = r_["reply_len"].cpu().tolist(), r_["replies"].cpu().numpy(), r_["reply_dst"].cpu().tolist()
        for i, (g, c, _) in enumerate(frames):
            if rl[i]:
                assert dst[i] == c
                replies[c].append((g, v, cells[i][:rl[i]].tobytes()))
    winners, engines = {}, {}
    for r, f in fols.items():
        rng.shuffle(replies[r])
        t = _deliver(f, replies[r], rng, "tally")
        nw = int(t["n_won"][0])
        wg, wt = t["won_group"].cpu().tolist(), t["won_term"].cpu().tolist()
        assert wg[nw:] == [-1] * (G - nw) and wg[:nw] == sorted(wg[:nw])
        for g, term in zip(wg[:nw], wt[:nw]):
            assert (g, term) not in winners, "two leaders in one term"
            winners[(g, term)] = r
        eng = RaftEngine(ctx, G, n, craft=True, window=W)
        eng.recon_view(), eng.log_view()
        planes = torch.zeros((T, stride), dtype=torch.uint8, device=dev)
        keep.append(planes)
        o = eng.step_up(f, t["won_group"], t["won_term"], planes)        # straight from the tally, no host step between
        torch.cuda.synchronize()
        vd = o["verdict"].cpu().tolist()
        assert vd[:nw] == [ts.DONE] * nw and vd[nw:] == [ts.IGNORED] * (G - nw)
        engines[r] = eng
    assert sorted(g for g, _ in winners) == sorted(set(range(G)) - split)
    for g in split:                                             # split votes: both candidates stay candidates
        for c in cands[g]:
            vv = fols[c].vote_view()
            assert int(vv["role"][g]) == CANDIDATE and int(vv["role_term"][g]) == int(fols[c].curr_term[g])
            assert int(fols[c].leader[g]) == c and bin(int(vv["votes"][g])).count("1") == 2
    # each winner commits an entry of its term, reads back the shards it lacks from the other survivors, executes
    for r, eng in engines.items():
        mine = sorted(g for (g, _), w in winners.items() if w == r)
        _propose(eng, r, [300 if g in mine else 0 for g in range(G)], stride, keep, batch, rng)
        _replicate(ctx, eng, r, {q: f for q, f in fols.items() if q != r}, keep, rng, mine)
        elc = eng.last_commit.cpu().tolist()
        assert all(elc[g] == int(eng.log_end[g]) - 1 for g in mine)
        out = torch.zeros(1 << 22, dtype=torch.uint8, device=dev)
        rr = eng.reconstruct_reads(out, 1 << 12, 4, groups=ts._t(mine, torch.int32))
        torch.cuda.synchronize()
        nf = int(rr["totals"][0])
        assert nf > 0
        fo, fg = rr["frame_off"][:nf], rr["frame_group"][:nf]
        reps = []
        for q, f in fols.items():
            if q == r:
                continue
            rout = torch.zeros(1 << 22, dtype=torch.uint8, device=dev)
            s_ = f.reconstruct_serve(out, fo, fg, torch.full((nf,), r, dtype=torch.uint8, device=dev), rout)
            torch.cuda.synchronize()
            ro = rout.cpu().numpy()
            for i in range(nf):
                ln = int(s_["reply_len"][i])
                if ln:
                    off = int(s_["reply_off"][i])
                    reps.append((int(fg[i]), q if q < r else q - 1, ro[off:off + ln].tobytes()))
        tb, offs = ts._buf([x for _, _, x in reps], rng)
        a = eng.absorb(tb, ts._t(offs, torch.int64), ts._t([x[0] for x in reps], torch.int32), ts._t([x[1] for x in reps], torch.uint8))
        res = torch.zeros(1 << 22, dtype=torch.uint8, device=dev)
        ex = eng.execute(res, 1 << 12)
        torch.cuda.synchronize()
        assert (a["verdict"].cpu().numpy().view(np.uint32) == ts.ACCEPTED).all()
        nrec = int(ex["totals"][0])
        recs = list(zip(*(ex[k][:nrec].cpu().tolist() for k in ("rec_group", "rec_slot", "rec_off", "rec_len"))))
        assert [(g, s) for g, s, _, _ in recs] == sorted(k for k in batch if k[0] in mine)
        rn = res.cpu().numpy()
        for g, s, off, dl in recs:
            assert rn[off:off + dl].tobytes() == batch[(g, s)], (g, s)
    for e in engines.values():
        e.close()
    for f in fols.values():
        f.close()
