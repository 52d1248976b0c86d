"""Prepare on the device acceptor (ss_acceptor_prepare / ss_acceptor_prepare_reply, summerset_b200/csrc/acceptor.cu) and
the new leader's PrepareReply parser (ss_prepare_reply_parse_dev, summerset_b200/csrc/wire_kernels.cu).

`PModel` extends `tests/test_acceptor_commit.Model` with a per-message restatement of handle_msg_prepare
(rspaxos/messages.rs:13-84, crossword/messages.rs:63-136) and of the follower branch of handle_logged_prepare_bal
(rspaxos/durability.rs:10-79, crossword/durability.rs:9-79): Status::Preparing, inst.voted kept apart from inst.bal and
the held shards, and replica_bk = {source, trigger_slot, endprep_slot}; an Accept resets replica_bk to {source, 0, 0}
and sets the vote.  Expected bytes come from the oracle's encoders (varint, ssor_rscodeword_encode).  The GPU tests
compare every WAL cell, reply byte and state word, the prepare view included, with canaries around the outputs, and run
the closed loop leader -> acceptors -> Prepare -> PrepareReply -> parse -> merge -> reconstruct -> new Accepts.
"""
import copy
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import pyoracle
from summerset_b200 import _lib
from tests.test_acceptor import ACC, BEYOND, FRAME_OVERFLOW, MALFORMED, STALE_BAL, STALE_SLOT, WAL_FULL_V, _buffer, _t, _vget
from tests.test_acceptor_commit import Model, Rig, _codeword, _pitch, _r16
from tests.test_acceptor_reconstruct import _frame, _nm, _var, absorb_model, cw_bytes, reply_frame, serve_model, recon_frame

PREP, PREP_REPLY, PREP_WAL = 0, 1, 0
U64 = (1 << 64) - 1


# ---------------------------------------------------------------------------------------------
# wire helpers
# ---------------------------------------------------------------------------------------------
def prep_frame(trigger, ballot, variant=PREP, nm=False, tail=b""):
    """PeerMessage::Msg{Prepare{trigger_slot, ballot}}; nm: every field as a non-minimal varint where one exists"""
    v = (lambda x: _nm(x) if nm and x < 1 << 16 else _var(x))
    return _frame(v(0) + v(variant) + v(trigger) + v(ballot) + tail)


def parse_prepare(frame, variant=PREP):
    """-> (trigger, ballot) or the verdict of a frame that is not a well-formed Prepare"""
    if len(frame) < 8 or int.from_bytes(frame[:8], "big") != len(frame) - 8:
        return MALFORMED
    b, n, vals = frame[8:], 0, []
    for k in range(4):
        r = _vget(b, n)
        if r is None:
            return MALFORMED
        if k == 0 and r[0] != 0:
            return 0x80000000 | r[0] if r[0] < 65536 else MALFORMED
        if k == 1 and r[0] != variant:
            return r[0] if r[0] < 65536 else MALFORMED
        vals.append(r[0])
        n = r[1]
    return (vals[2], vals[3]) if n == len(b) else MALFORMED


def wal_cell(slot, ballot, variant=PREP_WAL):
    body = _var(variant) + _var(slot) + _var(ballot)
    rec = len(body).to_bytes(8, "big") + body
    assert len(rec) <= 29
    return rec + bytes(32 - len(rec))


def prep_reply_bytes(slot, trig, endp, bal, voted, d, T, variant=PREP_REPLY):
    """voted: None or (vote_bal, dlen, shards[T] bytes|None)"""
    body = _var(0) + _var(variant) + _var(slot) + _var(trig) + _var(endp) + _var(bal)
    if voted is None:
        body += b"\x00"
    else:
        vb, dlen, sh = voted
        body += b"\x01" + _var(vb) + cw_bytes(d, T - d, dlen, -(-dlen // d) if dlen else 0, sh)
    return _frame(body)


# ---------------------------------------------------------------------------------------------
# the model
# ---------------------------------------------------------------------------------------------
class PModel(Model):
    """instances: st "P" / "A" / "C"; vb / vm / vsh = inst.voted (ballot, shard mask, shards); src, trig, span = replica_bk"""

    def accept(self, g, slot, bal, held, dlen, shards, src=0):
        if not super().accept(g, slot, bal, held, dlen, shards):
            return False
        self.inst[g][slot].update(vb=bal, vm=held, vsh=list(shards) if shards else None, src=src, trig=0, span=0)
        return True

    def heartbeat(self, recs):
        """Model.heartbeat, with a Preparing instance stopping the walk (status < Accepting)"""
        hidden = self._hide_preparing()
        try:
            return super().heartbeat(recs)
        finally:
            self._restore(hidden)

    def _hide_preparing(self):
        hidden = []
        for g in range(self.G):
            for s in [s for s, i in self.inst[g].items() if i["st"] == "P"]:
                hidden.append((g, s, self.inst[g].pop(s)))
        return hidden

    def _restore(self, hidden):
        for g, s, inst in hidden:
            self.inst[g][s] = inst

    def live_only(self):
        """a copy whose instance dicts hold only Accepting / Committed instances (the same dict objects), for the serve
        and absorb models, which treat any instance they find as status >= Accepting"""
        m = copy.copy(self)
        m.inst = [{s: i for s, i in d.items() if i["st"] != "P"} for d in self.inst]
        return m

    def words(self):
        acc, com = [0] * self.G, [0] * self.G
        for g in range(self.G):
            for s, inst in self.inst[g].items():
                if inst["st"] == "A":
                    acc[g] |= 1 << (s & 63)
                elif inst["st"] == "C":
                    com[g] |= 1 << (s & 63)
        return acc, com

    def prep_words(self):
        return [sum(1 << (s & 63) for s, i in self.inst[g].items() if i["st"] == "P") for g in range(self.G)]

    def prepare_one(self, g, peer, frame):
        """handle_msg_prepare for one frame -> (verdict, [(slot, ballot)] records)"""
        p = parse_prepare(frame) if g < self.G else MALFORMED
        if not isinstance(p, tuple):
            return p, []
        if peer == self.me:
            return MALFORMED, []
        trig, bal = p
        base = self.base[g]
        if trig < base:
            return STALE_SLOT, []
        if trig >= base + 64:
            return BEYOND, []
        if bal < self.bmax[g]:
            return STALE_BAL, []
        self.bmax[g] = bal
        endp = max(max(self.inst[g]) if self.inst[g] else base, trig)     # rposition(status > Null), unwrap_or(0)
        recs = []
        for s in range(trig, endp + 1):
            inst = self.inst[g].get(s)
            if inst is None:                                             # a fresh null_instance(): voted None
                inst = self.inst[g][s] = dict(bal=0, held=0, dlen=0, shards=None, st="P", vb=0, vm=0, vsh=None)
            inst.update(bal=bal, st="P", src=peer, trig=trig, span=endp - trig)
            recs.append((s, bal))
        return ACC, recs

    def prepare(self, frames, groups, peers, cap):
        """one ss_acceptor_prepare call -> (verdicts, records [(g, slot, bal, frame)], totals, status)"""
        trial = copy.deepcopy(self)
        counts, kinds = [], []
        for fr, g, pr in zip(frames, groups, peers):
            v, r = trial.prepare_one(g, pr, fr)
            kinds.append(v)
            counts.append(len(r))
        ends = np.cumsum([0] + counts)
        cut = next((i for i in range(len(frames)) if ends[i + 1] > cap), len(frames))
        verdicts, recs, status = [], [], 0
        for i, (fr, g, pr) in enumerate(zip(frames, groups, peers)):
            if i >= cut and kinds[i] in (ACC, STALE_BAL):
                verdicts.append(WAL_FULL_V)
                status = FRAME_OVERFLOW
                continue
            if i >= cut:
                verdicts.append(kinds[i])
                continue
            v, r = self.prepare_one(g, pr, fr)
            assert v == kinds[i]
            verdicts.append(v)
            recs += [(g, s, b, i) for s, b in r]
        return verdicts, recs, [int(ends[-1]), 32 * int(ends[-1])], status

    def prepare_reply(self, g, slot):
        """the follower branch of handle_logged_prepare_bal -> (frame bytes, destination) or None"""
        if g >= self.G or slot < self.base[g] or slot >= self.base[g] + 64:
            return None
        inst = self.inst[g].get(slot)
        if inst is None:
            return None
        voted = None
        if inst["vb"] > 0:
            voted = (inst["vb"], inst["dlen"], [inst["vsh"][j] if (inst["vm"] >> j) & 1 else None for j in range(self.T)])
        return prep_reply_bytes(slot, inst["trig"], inst["trig"] + inst["span"], inst["bal"], voted, self.d, self.T), inst["src"]


def parse_prep_reply(frame, d, T, variant=PREP_REPLY):
    """-> dict of the record ss_prepare_reply_parse_dev writes, or the kind of a frame that is not one"""
    if len(frame) < 8 or int.from_bytes(frame[:8], "big") != len(frame) - 8:
        return MALFORMED
    b, n, vals = frame[8:], 0, []
    for k in range(6):
        r = _vget(b, n)
        if r is None:
            return MALFORMED
        if k == 0 and r[0] != 0:
            return 0x80000000 | r[0] if r[0] < 65536 else MALFORMED
        if k == 1 and r[0] != variant:
            return r[0] if r[0] < 65536 else MALFORMED
        vals.append(r[0])
        n = r[1]
    rec = dict(slot=vals[2], trigger_slot=vals[3], endprep_slot=vals[4], ballot=vals[5], vote_bal=0, vote_mask=0, data_len=0,
               shards_at=U64)
    if n >= len(b) or b[n] > 1:
        return MALFORMED
    n += 1
    if b[n - 1] == 1:
        r = _vget(b, n)
        if r is None:
            return MALFORMED
        rec["vote_bal"], n = r
        if len(b) - n < 2 or b[n] != d or b[n + 1] != T - d:
            return MALFORMED
        n += 2
        cw = []
        for _ in range(3):
            r = _vget(b, n)
            if r is None:
                return MALFORMED
            cw.append(r[0])
            n = r[1]
        dl, sl, t = cw
        if dl >= 1 << 32 or t != T or sl != -(-dl // d):
            return MALFORMED
        rec["shards_at"], rec["data_len"] = 8 + n, dl
        for j in range(T):
            if n >= len(b) or b[n] > 1:
                return MALFORMED
            n += 1
            if b[n - 1] == 0:
                continue
            r = _vget(b, n)
            if r is None or r[0] != sl or len(b) - r[1] < sl:
                return MALFORMED
            n = r[1] + sl
            rec["vote_mask"] |= 1 << j
        if n >= len(b) or b[n] > 1:
            return MALFORMED
        n += 1
        if b[n - 1] == 1:
            if len(b) - n < dl:
                return MALFORMED
            n += dl
    return rec if n == len(b) else MALFORMED


# ---------------------------------------------------------------------------------------------
# CPU: model rules, symbols, refusals
# ---------------------------------------------------------------------------------------------
def _acc(m, g, s, bal, held=0b111, dlen=10, src=0):
    sh = [bytes([j]) * (-(-dlen // m.d)) if (held >> j) & 1 else None for j in range(m.T)]
    assert m.accept(g, s, bal, held, dlen, sh, src)


def test_model_endprep():
    m = PModel(2, 5, 1, 3, 5)
    m.base = [100, 100]
    assert m.prepare_one(0, 2, prep_frame(105, 3)) == (ACC, [(105, 3)])            # no non-null slot: endprep = trigger
    _acc(m, 1, 100, 1)
    _acc(m, 1, 130, 1)
    v, r = m.prepare_one(1, 2, prep_frame(110, 3))                                 # the last non-null slot
    assert v == ACC and [s for s, _ in r] == list(range(110, 131))
    assert m.inst[1][110]["trig"] == 110 and m.inst[1][110]["span"] == 20 and m.inst[1][100]["st"] == "A"
    assert m.inst[1][120]["vb"] == 0 and m.inst[1][130]["vb"] == 1                 # a null slot's vote is None
    assert m.prepare_one(1, 2, prep_frame(99, 9)) == (STALE_SLOT, [])
    assert m.prepare_one(1, 2, prep_frame(164, 9)) == (BEYOND, [])
    assert m.prepare_one(1, 2, prep_frame(110, 2)) == (STALE_BAL, [])
    assert m.prepare_one(1, 1, prep_frame(110, 9)) == (MALFORMED, [])              # from me
    assert m.prepare_one(1, 2, prep_frame(110, 9, tail=b"\0")) == (MALFORMED, [])
    assert m.prepare_one(1, 2, _frame(b"\x00\x02")) == (2, []) and m.prepare_one(1, 2, _frame(b"\x02")) == (0x80000002, [])
    assert m.prepare_one(1, 2, prep_frame(110, 3))[0] == ACC                        # an equal ballot passes


def test_model_overlapping_prepares():
    m = PModel(1, 5, 1, 3, 5)
    _acc(m, 0, 5, 1)
    v1, r1 = m.prepare_one(0, 2, prep_frame(3, 4))                                  # 3..5
    v2, r2 = m.prepare_one(0, 3, prep_frame(1, 5))                                  # 1..5: the earlier range counts as Preparing
    v3, r3 = m.prepare_one(0, 4, prep_frame(9, 6))                                  # above the previous endprep: 9..9
    assert [s for s, _ in r1] == [3, 4, 5] and [s for s, _ in r2] == [1, 2, 3, 4, 5] and [s for s, _ in r3] == [9]
    assert m.inst[0][4]["src"] == 3 and m.inst[0][4]["trig"] == 1 and m.inst[0][9]["src"] == 4
    v4, r4 = m.prepare_one(0, 2, prep_frame(7, 7))                                  # inside: 7..9
    assert [s for s, _ in r4] == [7, 8, 9]
    # the capacity suffix: a cut at frame 1 leaves frame 0 applied and later frames WAL_FULL
    m = PModel(1, 5, 1, 3, 5)
    fr = [prep_frame(3, 4), prep_frame(1, 5), prep_frame(0, 1), prep_frame(70, 9)]
    v, recs, tot, st = m.prepare(fr, [0] * 4, [2] * 4, 3)
    assert v == [ACC, WAL_FULL_V, WAL_FULL_V, BEYOND] and tot == [4, 128] and st == FRAME_OVERFLOW and len(recs) == 1


def test_model_vote_kept_and_dropped():
    m = PModel(1, 5, 1, 3, 5)
    _acc(m, 0, 0, 4, held=0b00110)
    m.prepare_one(0, 2, prep_frame(0, 6))
    inst = m.inst[0][0]
    assert inst["bal"] == 6 and inst["vb"] == 4 and inst["vm"] == 0b00110 and inst["st"] == "P"   # kept across a Prepare
    inst["held"] = 0b11111                                                                  # an absorb grows held only
    frame, dst = m.prepare_reply(0, 0)
    assert dst == 2 and parse_prep_reply(frame, 3, 5)["vote_mask"] == 0b00110
    m.advance([1])                                                                          # retired; a null position
    m.prepare_one(0, 3, prep_frame(1, 7))
    assert m.inst[0][1]["vb"] == 0 and parse_prep_reply(m.prepare_reply(0, 1)[0], 3, 5)["vote_bal"] == 0
    assert m.prepare_reply(0, 0) is None and m.prepare_reply(0, 2) is None


def test_model_reaccept_resets_bookkeeping():
    m = PModel(1, 5, 1, 3, 5)
    _acc(m, 0, 0, 1)
    m.prepare_one(0, 2, prep_frame(0, 5))
    _acc(m, 0, 0, 5, src=2)                                                                 # re-accepted at the new ballot
    rec = parse_prep_reply(m.prepare_reply(0, 0)[0], 3, 5)
    assert (rec["trigger_slot"], rec["endprep_slot"], rec["ballot"], rec["vote_bal"]) == (0, 0, 5, 5)
    assert m.words()[0] == [1] and m.prep_words() == [0]


def test_model_preparing_blocks_commit():
    m = PModel(1, 5, 1, 3, 5)
    for s in range(3):
        _acc(m, 0, s, 1)
    m.prepare_one(0, 2, prep_frame(1, 1))                                                  # 1..2 Preparing at ballot 1
    assert m.heartbeat([(0, 0, 1, 3, 0)]) == [0b1]                                         # the walk stops at slot 1
    assert sorted(m.live_only().inst[0]) == [0]


def test_acceptor_prepare_symbols_and_refusals():
    lib = _lib.load()
    for name in ("ss_acceptor_prepare_view_get", "ss_acceptor_prepare", "ss_acceptor_prepare_reply", "ss_prepare_reply_parse_dev"):
        assert hasattr(lib, name)
    assert lib.ss_version() == 200
    v = _lib.AcceptorPrepareView()
    assert lib.ss_acceptor_prepare_view_get(None, C.byref(v)) == _lib.SS_ERR_INVALID_ARG
    assert lib.ss_acceptor_prepare(None, None, 0, None, None, None, 0, 0, 0, None, 0, None, None, None, 0, None, None) == _lib.SS_ERR_INVALID_ARG
    assert lib.ss_acceptor_prepare_reply(None, None, None, 0, 1, None, 0, None, None, None, None) == _lib.SS_ERR_INVALID_ARG
    assert lib.ss_prepare_reply_parse_dev(None, None, 0, None, 0, 3, 5, 1, None) == _lib.SS_ERR_INVALID_ARG
    assert C.sizeof(_lib.AcceptorPrepareView) == 48 and C.sizeof(_lib.PrepareReplyRec) == 64
    cfg = _lib.AcceptorConfig(_lib.SS_PROTO_RSPAXOS, 5, 0, 3, 5, 2, 1, 3)
    h = C.c_void_p()
    rc = lib.ss_acceptor_create(None, C.byref(cfg), 4, C.byref(h))
    assert rc in (_lib.SS_ERR_NO_DEVICE, _lib.SS_ERR_INVALID_ARG)
    if not torch.cuda.is_available():
        assert rc == _lib.SS_ERR_NO_DEVICE


# ---------------------------------------------------------------------------------------------
# GPU helpers
# ---------------------------------------------------------------------------------------------
class PRig(Rig):
    """Rig with PModel; prepare / prepare_reply compared byte for byte with the model"""

    def __init__(self, ctx, protocol, G, n, me, d, T):
        super().__init__(ctx, protocol, G, n, me, d, T)
        self.m = PModel(G, n, me, d, T)

    def check_state(self):
        super().check_state()
        a, m = self.acc, self.m
        u = lambda t: [int(x) for x in t.cpu().numpy().view(np.uint64)]
        assert u(a.preparing) == m.prep_words()
        ib, vb, vm = u(a.inst_bal), u(a.voted_bal), a.voted_mask.cpu().numpy().view(np.uint32)
        trig, span, src = u(a.prep_trigger), a.prep_span.cpu().numpy(), a.source.cpu().numpy()
        for g in range(m.G):
            for s, inst in m.inst[g].items():
                at = g * 64 + (s & 63)
                got = (ib[at], vb[at], int(vm[at]) if inst["vb"] else 0, trig[at], int(span[at]), int(src[at]))
                assert got == (inst["bal"], inst["vb"], inst["vm"] if inst["vb"] else 0, inst["trig"], inst["span"], inst["src"]), (g, s)

    def prepare(self, items, rec_cap=None, wal_cap=None):
        """items: (g, peer, frame bytes) in frame order -> (verdicts, records)"""
        frames = [f for _, _, f in items]
        groups = [g for g, _, _ in items]
        peers = [p for _, p, _ in items]
        _, _, tot, _ = copy.deepcopy(self.m).prepare(frames, groups, peers, 1 << 62)
        rc = tot[0] if rec_cap is None else rec_cap
        wc = 32 * tot[0] if wal_cap is None else wal_cap
        cap = min(rc, wc // 32)
        buf, offs = _buffer(self.rng, frames)
        canary = self.rng.integers(0, 256, wc + 64, dtype=np.uint8)
        wal = _t(canary.copy())
        res = self.acc.prepare(_t(buf), _t(offs), _t(np.array(groups, dtype=np.uint32)), _t(np.array(peers, dtype=np.uint8)), wal,
                               rc, wc)
        verdicts, recs, totals, status = self.m.prepare(frames, groups, peers, cap)
        got = {k: v.cpu().numpy() for k, v in res.items()}
        assert [int(x) for x in got["totals"]] == totals
        assert [int(x) for x in got["verdict"].view(np.uint32)] == verdicts
        assert self.ctx.device_status() == status
        n = len(recs)
        assert [int(x) for x in got["rec_group"][:n]] == [r[0] for r in recs]
        assert [int(x) for x in got["rec_slot"][:n].view(np.uint64)] == [r[1] for r in recs]
        assert [int(x) for x in got["rec_frame"][:n]] == [r[3] for r in recs]
        want = canary.copy()
        for k, (g, s, b, _) in enumerate(recs):
            want[32 * k:32 * k + 32] = np.frombuffer(wal_cell(s, b), dtype=np.uint8)
        gw = wal.cpu().numpy()
        if not np.array_equal(gw, want):
            bad = np.nonzero(gw != want)[0]
            pytest.fail(f"wal: {len(bad)} bytes differ, first at {bad[0]}")
        self.check_state()
        return verdicts, recs

    def prepare_reply(self, recs, out_cap=None, parse=True):
        """recs: (g, slot) -> the replies, checked against the model, and parsed back by ss_prepare_reply_parse_dev"""
        from summerset_b200.engine import prepare_reply_parse
        want = [self.m.prepare_reply(g, s) for g, s in recs]
        regions = [_r16(len(w[0])) if w else 0 for w in want]
        total = sum(regions)
        cap = total if out_cap is None else out_cap
        canary = self.rng.integers(0, 256, cap + 64, dtype=np.uint8)
        out = _t(canary.copy())
        res = self.acc.prepare_reply(_t(np.array([g for g, _ in recs], dtype=np.uint32)),
                                     _t(np.array([s for _, s in recs], dtype=np.uint64)), out, cap)
        got = {k: v.cpu().numpy() for k, v in res.items()}
        assert int(got["total"][0]) == total
        exp, at, status, frames = canary.copy(), 0, 0, []
        for k, w in enumerate(want):
            ro, rl, rd = int(got["reply_off"][k].view(np.uint64)), int(got["reply_len"][k]), int(got["reply_dst"][k])
            if w is None:
                assert (ro, rl, rd) == (U64, 0, 0xff), k
                continue
            fr, dst = w
            assert rl == len(fr), k
            if at + regions[k] > cap:
                assert (ro, rd) == (U64, 0xff), k
                status = FRAME_OVERFLOW
            else:
                assert (ro, rd) == (at, dst), k
                exp[at:at + len(fr)] = np.frombuffer(fr, dtype=np.uint8)
                frames.append((k, at, fr))
            at += regions[k]
        assert self.ctx.device_status() == status
        go = out.cpu().numpy()
        if not np.array_equal(go, exp):
            bad = np.nonzero(go != exp)[0]
            pytest.fail(f"replies: {len(bad)} bytes differ, first at {bad[0]}")
        if parse and frames:
            offs = np.array([a for _, a, _ in frames], dtype=np.uint64)
            pr = prepare_reply_parse(self.ctx, out, _t(offs), self.m.d, self.m.T)
            pr = {k: v.cpu().numpy() for k, v in pr.items()}
            for q, (k, a, fr) in enumerate(frames):
                w = parse_prep_reply(fr, self.m.d, self.m.T)
                assert int(pr["kind"][q]) == PREP_REPLY
                for f in ("slot", "trigger_slot", "endprep_slot", "ballot", "vote_bal"):
                    assert int(pr[f][q]) & U64 == w[f], (k, f)
                assert int(pr["vote_mask"][q]) & 0xffffffff == w["vote_mask"] and int(pr["data_len"][q]) == w["data_len"]
                sa = int(np.int64(pr["shards_at"][q]).view(np.uint64))
                assert sa == (U64 if w["shards_at"] == U64 else a + w["shards_at"])
        self.check_state()
        return got, frames


def _fill(rig, G, k, bal=1, held=None, lens=(1, 17, 251, 1366)):
    d, T = rig.m.d, rig.m.T
    items = []
    for g in range(G):
        for s in range(k):
            data, sh = _codeword(rig.rng, int(lens[(g + s) % len(lens)]), d, T)
            h = held if held is not None else int(rig.rng.integers(1, 1 << T))
            items.append((g, rig.m.base[g] + s, bal, h, data, sh))
    rig.accept(items)


def _all_recs(rig):
    return [(g, s) for g in range(rig.m.G) for s in sorted(rig.m.inst[g])]


# ---------------------------------------------------------------------------------------------
# GPU 1: populations and codes
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 2, 3, 5, 7, 9, 12, 32])
@pytest.mark.parametrize("protocol", ["rspaxos", "crossword"])
def test_prepare_populations(ctx, protocol, n):
    cases = [(n // 2 + 1, n)] if protocol == "rspaxos" else sorted({(n // 2 + 1, n), (1, min(2 * n, 32)), (min(2 * n, 32),) * 2})
    for d, T in cases:
        me = n - 1
        rig = PRig(ctx, protocol, 6, n, me, d, T)
        rig.set_base([int(x) for x in rig.rng.integers(0, 1 << 40, 6)])
        held = (1 << me) if protocol == "rspaxos" and T == n else None
        _fill(rig, 6, 5, held=held)
        peer = 0 if n > 1 else 1                                         # n = 1: every Prepare comes from me... except a stranger
        items = [(g, peer, prep_frame(rig.m.base[g] + (g % 3), 2)) for g in range(6)]
        rig.prepare(items)
        rig.prepare_reply(_all_recs(rig))


@pytest.mark.gpu
def test_prepare_crossword_empty_row(ctx, oracle):
    """Crossword with an empty assignment row at me: votes are Some((bal, no shards))"""
    n, T, d = 5, 5, 3
    rig = PRig(ctx, "crossword", 4, n, 2, d, T)
    frames, groups = [], []
    for g in range(4):
        for s in range(3):
            dlen = 1 + 97 * (g + s)
            body = _var(0) + _var(2) + _var(s) + _var(3) + cw_bytes(d, T - d, dlen, -(-dlen // d), [None] * T)
            body += _var(n) + b"".join(oracle.bitmap_encode(T, 0) for _ in range(n))      # assignment: every row empty
            frames.append(_frame(body))
            groups.append(g)
            assert rig.m.accept(g, s, 3, 0, dlen, [None] * T)
    buf, offs = _buffer(rig.rng, frames)
    store = torch.empty(64, dtype=torch.uint8, device="cuda")
    wal = torch.empty(sum(len(f) + 48 for f in frames), dtype=torch.uint8, device="cuda")
    rig.stores.append(store)
    res = rig.acc.accept(_t(buf), _t(offs), _t(np.array(groups, dtype=np.uint32)), _t(np.zeros(12, np.uint8)), store, wal)
    assert (res["verdict"].cpu().numpy().view(np.uint32) == ACC).all() and ctx.device_status() == 0
    rig.prepare([(g, 0, prep_frame(0, 4)) for g in range(4)])
    got, frames = rig.prepare_reply(_all_recs(rig))
    assert frames and all(parse_prep_reply(f, d, T)["vote_bal"] == 3 for _, _, f in frames)


# ---------------------------------------------------------------------------------------------
# GPU 2: wire edges and verdicts
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_prepare_wire_edges(ctx):
    rig = PRig(ctx, "crossword", 8, 5, 1, 3, 5)
    bases = [0, 250, 251, 1 << 16, (1 << 32) - 3, 1 << 33, (1 << 63), 7]
    rig.set_base(bases)
    _fill(rig, 8, 2, bal=1)
    items = []
    for g in range(8):
        b = bases[g]
        items += [(g, 2, prep_frame(b, 250)), (g, 3, prep_frame(b + 1, 251, nm=True)), (g, 4, prep_frame(b, (1 << 16) + g)),
                  (g, 0, prep_frame(b + 3, (1 << 32) + g)), (g, 2, prep_frame(b + 2, (1 << 40) + g, nm=True))]
    # refusals: truncated, trailing, other messages both sides of 2^16, from me, stale, beyond, lower ballot, group >= G
    items += [(0, 2, _frame(prep_frame(0, 1 << 50)[8:-1])), (1, 2, prep_frame(250, 1 << 50, tail=b"\0")), (2, 2, _frame(_var(0) + _var(2))),
              (3, 2, _frame(_var(0) + _var(70000) + _var(1) + _var(1))), (4, 2, _frame(_var(3))), (4, 2, _frame(_var(1 << 20))),
              (5, 1, prep_frame(1 << 33, 1 << 50)), (6, 2, prep_frame((1 << 63) - 1, 1 << 50)), (7, 2, prep_frame(7 + 64, 1 << 50)),
              (7, 2, prep_frame(7, 5)), (8, 2, prep_frame(0, 1 << 50)), (0, 2, _frame(b""))]
    items += [(g, 3, prep_frame(bases[g] + 1, (1 << 40) + g)) for g in range(8)]          # an equal ballot passes
    rig.prepare(items)
    rig.prepare_reply(_all_recs(rig) + [(9, 0), (0, 1 << 40)])


@pytest.mark.gpu
def test_prepare_variants(ctx):
    """Prepare, WAL and reply variants of every varint width"""
    for pv, wv, rv in [(0, 0, 1), (250, 251, 252), (65535, 300, 65535)]:
        rig = PRig(ctx, "rspaxos", 2, 5, 1, 3, 5)
        _fill(rig, 2, 3, held=0b10)
        frames = [(g, 0, prep_frame(0, 9, variant=pv)) for g in range(2)]
        buf, offs = _buffer(rig.rng, [f for _, _, f in frames])
        wal = torch.zeros(32 * 8, dtype=torch.uint8, device="cuda")
        res = rig.acc.prepare(_t(buf), _t(offs), _t(np.array([0, 1], dtype=np.uint32)), _t(np.zeros(2, np.uint8)), wal, 8,
                              prepare_variant=pv, wal_variant=wv)
        assert (res["verdict"].cpu().numpy().view(np.uint32) == ACC).all() and int(res["totals"][0]) == 6
        cells = wal.cpu().numpy().reshape(8, 32)
        slots = res["rec_slot"].cpu().numpy()[:6]
        for k in range(6):
            assert cells[k].tobytes() == wal_cell(int(slots[k]), 9, wv)
        out = torch.zeros(4096, dtype=torch.uint8, device="cuda")
        rr = rig.acc.prepare_reply(res["rec_group"][:6], res["rec_slot"][:6], out, reply_variant=rv)
        from summerset_b200.engine import prepare_reply_parse
        pr = prepare_reply_parse(ctx, out, rr["reply_off"], 3, 5, reply_variant=rv)
        assert (pr["kind"].cpu().numpy() == rv).all() and (pr["vote_bal"].cpu().numpy() == 1).all()
        ctx.device_status()


@pytest.mark.gpu
def test_prepare_several_per_group(ctx):
    """several Prepares per group from different peers, triggers below, inside and above the previous endprep, over
    Accepting, Committed, absorbed, ballot-0 votes and retired positions"""
    n, T, d = 5, 5, 3
    rig = PRig(ctx, "crossword", 6, n, 4, d, T)
    rng = rig.rng
    _fill(rig, 6, 10, bal=0)                                                   # ballot-0 votes: None
    _fill(rig, 6, 6, bal=2)
    rig.commit_all()
    rig.execute(check_data=False)
    # absorb a few shards into group 0 (held grows past the vote)
    m = rig.m
    fr = []
    for s in range(3):
        inst = m.inst[0][s]
        full = [bytes(rng.integers(0, 256, -(-inst["dlen"] // d), dtype=np.uint8)) for _ in range(T)]
        sh = [inst["shards"][j] if (inst["held"] >> j) & 1 else full[j] for j in range(T)]
        fr.append(reply_frame([(s, 2, inst["dlen"], sh)], d, T))
    buf, offs = _buffer(rng, fr)
    store = torch.empty(1 << 16, dtype=torch.uint8, device="cuda")
    rig.stores.append(store)
    rig.acc.absorb(_t(buf), _t(offs), _t(np.zeros(3, np.uint32)), _t(np.ones(3, np.uint8)), store)
    absorb_model(m.live_only(), fr, [0] * 3, 1 << 16)
    assert ctx.device_status() == 0
    upto = [0, 4, 0, 0, 0, 0]
    rig.acc.advance(_t(np.array(upto, dtype=np.uint64)))
    rig.m.advance(upto)
    items = []
    for g in range(6):
        for q in range(4):
            trig = m.base[g] + int(rng.choice([0, 2, 5, 12, 30]))
            items.append((g, int(rng.integers(0, 4)), prep_frame(trig, 3 + q + int(rng.integers(0, 2)))))
    items.append((1, 0, prep_frame(m.base[1] + 63, 20)))                      # the whole window
    rig.prepare(items)
    rig.prepare_reply(_all_recs(rig))
    # a re-accept after the Prepare: trigger and endprep 0
    rig.accept([(2, m.base[2] + 1, 30, 0b111) + _codeword(rng, 40, d, T)])
    rig.prepare_reply(_all_recs(rig))


# ---------------------------------------------------------------------------------------------
# GPU 3: capacities
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_prepare_wal_cut_every_boundary(ctx):
    """a small batch cut at every frame boundary: the applied frames are a prefix; re-submitting completes it"""
    def batch(rig):
        b = rig.m.base
        return [(0, 2, prep_frame(b[0] + 3, 4)), (1, 2, prep_frame(b[1], 4)), (0, 3, prep_frame(b[0] + 1, 5)),
                (0, 2, prep_frame(b[0] + 1, 4)), (1, 3, prep_frame(b[1] + 9, 6)), (0, 0, prep_frame(b[0] + 20, 6))]
    probe = PRig(ctx, "rspaxos", 2, 5, 1, 3, 5)
    _fill(probe, 2, 8, held=0b10)
    _, _, tot, _ = copy.deepcopy(probe.m).prepare([f for _, _, f in batch(probe)], [0, 1, 0, 0, 1, 0], [2, 2, 3, 2, 3, 0], 1 << 62)
    for cap in range(0, tot[0] + 1):
        for which in ("rec", "wal"):
            rig = PRig(ctx, "rspaxos", 2, 5, 1, 3, 5)
            _fill(rig, 2, 8, held=0b10)
            items = batch(rig)
            v, _ = rig.prepare(items, rec_cap=cap if which == "rec" else None, wal_cap=32 * cap + 31 if which == "wal" else None)
            rest = [it for it, x in zip(items, v) if x == WAL_FULL_V]
            if rest:
                rig.prepare(rest)
            full = PRig(ctx, "rspaxos", 2, 5, 1, 3, 5)
            _fill(full, 2, 8, held=0b10)
            full.prepare(batch(full))
            assert full.m.prep_words() == rig.m.prep_words()
            assert {(g, s): (i["bal"], i["trig"], i["span"], i["src"]) for g in range(2) for s, i in full.m.inst[g].items()} == \
                   {(g, s): (i["bal"], i["trig"], i["span"], i["src"]) for g in range(2) for s, i in rig.m.inst[g].items()}


@pytest.mark.gpu
def test_prepare_reply_cut_and_drain(ctx):
    rig = PRig(ctx, "crossword", 4, 5, 1, 3, 5)
    _fill(rig, 4, 6, bal=2, lens=(100, 3000, 17))
    rig.prepare([(g, 0, prep_frame(0, 3)) for g in range(4)])
    recs = _all_recs(rig)
    want = [rig.m.prepare_reply(g, s) for g, s in recs]
    regions = np.cumsum([_r16(len(w[0])) for w in want])
    for edge in (int(regions[5]), int(regions[5]) - 1, int(regions[0]) - 1):
        got, frames = rig.prepare_reply(recs, out_cap=edge)
        left = [r for r, o in zip(recs, got["reply_off"].view(np.uint64)) if int(o) == U64]
        assert len(frames) + len(left) == len(recs) and left == recs[len(frames):]
        rig.prepare_reply(left)


# ---------------------------------------------------------------------------------------------
# GPU 4: Preparing instances and the other handlers
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_preparing_blocks_commit_execute_serve_absorb(ctx):
    n, T, d = 5, 5, 3
    rig = PRig(ctx, "crossword", 3, n, 1, d, T)
    rng = rig.rng
    _fill(rig, 3, 8, bal=2, held=0b00011)
    rig.prepare([(g, 2, prep_frame(3 + g, 2)) for g in range(3)])            # 3.. / 4.. / 5.. Preparing at ballot 2
    rig.heartbeat([(g, 2, 2, 64, 0) for g in range(3)])                      # commits stop at the Preparing slots
    rig.execute(check_data=False)
    m = rig.m
    # serve: Reconstruct over every slot; Preparing instances are skipped
    fr = [recon_frame([(s, 5, [0]) for s in range(8)], True) for _ in range(3)]
    buf, offs = _buffer(rng, fr)
    out = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    res = rig.acc.reconstruct_serve(_t(buf), _t(offs), _t(np.arange(3, dtype=np.uint32)), _t(np.zeros(3, np.uint8)), out)
    lo = m.live_only()
    ro, rl = res["reply_off"].cpu().numpy(), res["reply_len"].cpu().numpy()
    ob = out.cpu().numpy()
    for g in range(3):
        v, want = serve_model(lo, True, g, fr[g])
        assert v == ACC and ob[int(ro[g]):int(ro[g]) + int(rl[g])].tobytes() == want
    # absorb: entries for Preparing instances are ignored
    fr = []
    for g in range(3):
        ents = []
        for s in range(8):
            inst = m.inst[g][s]
            ents.append((s, 2, inst["dlen"], [inst["shards"][j] if (inst["held"] >> j) & 1 else bytes(-(-inst["dlen"] // d))
                                                for j in range(T)]))
        fr.append(reply_frame(ents, d, T))
    buf, offs = _buffer(rng, fr)
    store = torch.empty(1 << 18, dtype=torch.uint8, device="cuda")
    rig.stores.append(store)
    ab = rig.acc.absorb(_t(buf), _t(offs), _t(np.arange(3, dtype=np.uint32)), _t(np.zeros(3, np.uint8)), store)
    verdicts, counts, total, status, _ = absorb_model(lo, fr, [0, 1, 2], 1 << 18)
    assert [int(x) for x in ab["absorbed"].cpu().numpy()] == counts and int(ab["total"][0]) == total
    assert ctx.device_status() == status
    assert [int(x) for x in rig.acc.held.cpu().numpy().view(np.uint32)[:8]] == [m.inst[0][s]["held"] for s in range(8)]
    rig.prepare_reply(_all_recs(rig))


# ---------------------------------------------------------------------------------------------
# GPU 5: scale -- grid caps, one big group, sort-key edges
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_prepare_one_group_20k_frames(ctx):
    rig = PRig(ctx, "rspaxos", 3, 5, 1, 3, 5)
    _fill(rig, 3, 10, held=0b10)
    rng = rig.rng
    items = [(0, int(rng.integers(2, 5)), prep_frame(int(rng.integers(0, 70)), int(q // 50))) for q in range(20000)]
    items += [(1, 2, prep_frame(5, 1)), (2, 3, prep_frame(0, 2))]
    rig.prepare(items)
    rig.prepare_reply(_all_recs(rig))


@pytest.mark.gpu
@pytest.mark.parametrize("G", [1, 2, 255, 256, 257, 65536, 65537])
def test_prepare_sort_key_edges_and_grid_caps(ctx, G):
    rig = PRig(ctx, "crossword", G, 5, 3, 3, 5)
    rng = rig.rng
    gs = sorted({0, G - 1, G // 2} | {int(x) for x in rng.integers(0, G, 40)})
    items = []
    for g in gs:
        data, sh = _codeword(rng, int(rng.integers(1, 200)), 3, 5)
        items.append((g, int(rng.integers(0, 4)), 1, 0b10110, data, sh))
    rig.accept(items)
    nfr = 100000 if G == 65537 else 3000                              # past the warp kernels' grid cap
    gsel = rng.integers(0, G + 1, nfr)
    frames = [(int(g), int(rng.integers(0, 3)), prep_frame(int(rng.integers(0, 66)), int(rng.integers(0, 4)))) for g in gsel]
    rig.prepare(frames)
    rig.prepare_reply([(g, s) for g in gs for s in range(4)] + [(G, 0)])


# ---------------------------------------------------------------------------------------------
# GPU 6: the parser on malformed frames
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_prepare_reply_parse_refusals(ctx):
    from summerset_b200.engine import prepare_reply_parse
    d, T = 3, 5
    sh = [b"abcd", None, b"efgh", b"ijkl", None]
    good = prep_reply_bytes(7, 3, 9, 11, (5, 10, sh), d, T)
    body = good[8:]
    cases = [good, prep_reply_bytes(7, 3, 9, 11, None, d, T), _frame(body[:-1]), _frame(body + b"\0"),
             prep_reply_bytes(7, 3, 9, 11, (5, 10, sh), 2, 5), prep_reply_bytes(7, 3, 9, 11, (5, 10, sh), 3, 6),
             _frame(body[:-1] + b"\x01" + bytes(10)), _frame(body[:-1] + b"\x01" + bytes(9)), _frame(body[:-1] + b"\x02"),
             _frame(_var(0) + _var(3) + _var(1)), _frame(_var(2)), _frame(_var(0) + _var(1 << 17)), _frame(_var(1 << 17)),
             _frame(body.replace(b"\x01\x00\x01", b"\x01\x00\x02", 1)), prep_reply_bytes(1 << 40, 1 << 33, 1 << 34, 1 << 62, (1, 1, [b"x", None, None, None, None]), d, T)]
    # a shard of the wrong length
    bad_len = bytearray(good)
    i = bad_len.index(b"abcd") - 1
    bad_len[i] = 3
    cases.append(bytes(bad_len))
    rng = np.random.default_rng(5)
    buf, offs = _buffer(rng, cases)
    pr = prepare_reply_parse(ctx, _t(buf), _t(offs), d, T)
    pr = {k: v.cpu().numpy() for k, v in pr.items()}
    for q, fr in enumerate(cases):
        w = parse_prep_reply(fr, d, T)
        kind = int(pr["kind"][q]) & 0xffffffff
        if isinstance(w, dict):
            assert kind == PREP_REPLY, q
            for f in ("slot", "trigger_slot", "endprep_slot", "ballot", "vote_bal"):
                assert int(np.int64(pr[f][q]).view(np.uint64)) == w[f], (q, f)
            assert int(pr["vote_mask"][q]) == w["vote_mask"]
        else:
            assert kind == w, q


# ---------------------------------------------------------------------------------------------
# GPU 7: closed loop -- leader proposals, a lost leader, Prepare on the survivors, merge, reconstruct, new Accepts
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("protocol,n,T,d", [("rspaxos", 3, 3, 2), ("rspaxos", 5, 5, 3), ("rspaxos", 7, 7, 4),
                                            ("crossword", 5, 5, 3), ("crossword", 7, 14, 7)])
def test_closed_loop_failover(ctx, oracle, protocol, n, T, d):
    from summerset_b200 import workloads as wl
    from summerset_b200.engine import Acceptor, LeaderEngine, prepare_reply_parse
    from tests.test_failover import _replay
    cw = protocol == "crossword"
    G, rounds = 16, 3
    rng = np.random.default_rng(n * 100 + T)
    eng = LeaderEngine(ctx, protocol, G, n, 1, 1, **(dict(rs_total_shards=T, rs_data_shards=d) if cw else {}))
    bal = rng.integers(1, 1 << 20, G).astype(np.uint64)
    eng.set_prepared_ballots(_t(bal))
    if cw:
        policies = np.array([oracle.cw_brr_assignment(n, T, d)], dtype=np.uint32)
        eng.set_policies([list(map(int, q)) for q in policies], True)
    else:
        policies = np.array([[1 << r for r in range(n)]], dtype=np.uint32)
    survivors = list(range(1, n))                       # replica 0 led; replica 1 becomes the new leader
    accs = {r: Acceptor(ctx, protocol, G, n, r, d, T) for r in survivors}
    keep, sent = [], {}
    for rnd in range(rounds):
        lens = (wl.cfg4_lengths(G, seed_extra=rnd)[0] // 16 + rng.integers(1, 7, G)).astype(np.uint32)
        data_off = (16 + np.cumsum(lens.astype(np.int64) + 5) - lens.astype(np.int64)).astype(np.uint64)
        arena = rng.integers(0, 256, int(data_off[-1]) + int(lens[-1]) + 64, dtype=np.uint8)
        L = (lens.astype(np.int64) + d - 1) // d
        store = torch.zeros((T, int(((L + 31) // 32 * 32).sum()) + 32), dtype=torch.uint8, device="cuda")
        keep.append(store)
        slot_out, shard_off, _ = eng.propose_ragged(_t(arena), _t(data_off), _t(lens), store, _t(np.zeros(G, np.uint8)) if cw else None)
        slots = slot_out.cpu().numpy().view(np.uint64)
        for g in range(G):
            sent[(g, int(slots[g]))] = arena[int(data_off[g]):int(data_off[g]) + int(lens[g])].tobytes()
        for r in survivors:
            out, off, fl, _ = ctx.frame_accept_pack_ragged(store, shard_off, _t(lens), d, T - d, policies, _t(np.zeros(G, np.uint8)), r,
                                                           slot_out, _t(bal), with_assignment=cw)
            oh, flh, bh = off.cpu().numpy(), fl.cpu().numpy(), out.cpu().numpy()
            # frames withheld before the last round: replica r misses group g's Accept when (g + r + rnd) % 4 == 0
            gs = [g for g in range(G) if rnd == rounds - 1 or (g + r + rnd) % 4 != 0]
            frames = [bh[int(oh[g]):int(oh[g]) + int(flh[g])].tobytes() for g in gs]
            buf, offs = _buffer(rng, frames)
            astore = torch.empty(sum(len(f) for f in frames) * 2 + 64, dtype=torch.uint8, device="cuda")
            awal = torch.empty(sum(len(f) + 48 for f in frames) + 64, dtype=torch.uint8, device="cuda")
            keep.append(astore)
            res = accs[r].accept(_t(buf), _t(offs), _t(np.array(gs, dtype=np.uint32)), _t(np.zeros(len(gs), np.uint8)), astore, awal)
            assert (res["verdict"].cpu().numpy().view(np.uint32) == ACC).all()
        if rnd == 0:                                    # the leader's heartbeat commits round 0
            for r in survivors:
                accs[r].heartbeat(_t(np.arange(G, dtype=np.uint32)), _t(np.zeros(G, np.uint8)), _t(bal), _t(slots + np.uint64(1)),
                                  _t(np.zeros(G, np.uint64)))
    assert ctx.device_status() == 0
    # replica 1's Prepare at a higher ballot, trigger = window base, goes to the other survivors and to itself as acceptor
    nb = bal + np.uint64(1 << 21)
    votes = {}
    for r in survivors:
        frames = [prep_frame(0, int(nb[g])) for g in range(G)]
        buf, offs = _buffer(rng, frames)
        wal = torch.empty(G * 64 * 32, dtype=torch.uint8, device="cuda")
        peer = 1 if r != 1 else 2                        # a replica's own Prepare arrives as its PrepareBal; model it from a peer
        res = accs[r].prepare(_t(buf), _t(offs), _t(np.arange(G, dtype=np.uint32)), _t(np.full(G, peer, np.uint8)), wal, G * 64)
        assert (res["verdict"].cpu().numpy().view(np.uint32) == ACC).all()
        nrec = int(res["totals"][0])
        assert nrec == G * rounds
        out = torch.empty(nrec * 4096, dtype=torch.uint8, device="cuda")
        rr = accs[r].prepare_reply(res["rec_group"][:nrec], res["rec_slot"][:nrec], out)
        assert ctx.device_status() == 0
        pr = prepare_reply_parse(ctx, out, rr["reply_off"], d, T)
        pr = {k: v.cpu().numpy() for k, v in pr.items()}
        assert (pr["kind"] == PREP_REPLY).all()
        rg = res["rec_group"][:nrec].cpu().numpy()
        for k in range(nrec):
            assert int(pr["endprep_slot"][k]) == rounds - 1 and int(pr["trigger_slot"][k]) == 0
            votes[(r, int(rg[k]), int(pr["slot"][k]))] = (int(pr["vote_bal"][k]), int(pr["vote_mask"][k]) & 0xffffffff, k, pr, out)
    # the merge over the survivors' replies equals the one-at-a-time replay
    N = G * rounds
    R = len(survivors)
    vb = np.zeros((R, N), np.uint64)
    vm = np.zeros((R, N), np.uint32)
    for ri, r in enumerate(survivors):
        for g in range(G):
            for s in range(rounds):
                vb[ri, g * rounds + s], vm[ri, g * rounds + s] = votes[(r, g, s)][:2]
    acks = np.full(N, R, np.uint8)
    mb, mg, act = ctx.prepare_merge(_t(vb), _t(vm.view(np.int32)), _t(acks), d, n, n - R)
    mb, mg = mb.cpu().numpy().view(np.uint64), mg.cpu().numpy().view(np.uint32)
    for i in range(N):
        assert (int(mb[i]), int(mg[i])) == _replay([(int(vb[r, i]), int(vm[r, i])) for r in range(R)]), i
    # ss_rs_reconstruct_batch_dev regenerates every decided instance from the voted shards the replies carry
    from summerset_b200.api import ReedSolomon
    lens = np.array([len(sent[divmod(i, rounds)]) for i in range(N)], dtype=np.int32)
    Ls = (lens.astype(np.int64) + d - 1) // d
    pitch = (Ls + 31) // 32 * 32
    off = np.concatenate([[0], np.cumsum(pitch)[:-1]]).astype(np.int64)
    ps = int(pitch.sum()) + 32
    sh = np.full((T, ps), 0xEE, dtype=np.uint8)
    host_out = {}
    for i in range(N):
        g, s = divmod(i, rounds)
        for r in survivors:
            b_, m_, k, pr, out = votes[(r, g, s)]
            if b_ != int(mb[i]) or b_ == 0:
                continue
            ob = host_out.setdefault(r, out.cpu().numpy())
            at = int(pr["shards_at"][k])
            for j in range(T):
                at += 1
                if ob[at - 1] == 1:
                    at = _vget(ob, at)[1]
                    sh[j, off[i]:off[i] + Ls[i]] = ob[at:at + Ls[i]]
                    at += int(Ls[i])
    if T <= 12:
        rs = ReedSolomon(ctx, d, T - d)
        sh_d = _t(sh)
        st = rs.reconstruct_batch(sh_d, ps, _t(off), _t(lens), _t(mg.view(np.int32)), False).cpu().numpy()
        got = sh_d.cpu().numpy()
    else:                                               # the batched device reconstruct takes d + p <= 12: the oracle's
        got, st = sh, np.zeros(N, np.int32)             # rs_reconstruct(data_only) regenerates the wider codes
        for i in range(N):
            if bin(int(mg[i])).count("1") < d:
                st[i] = _lib.SS_ERR_TOO_FEW_SHARDS_PRESENT
                continue
            cw_ = [sh[j, off[i]:off[i] + Ls[i]].copy() if (int(mg[i]) >> j) & 1 else None for j in range(T)]
            if any(cw_[j] is None for j in range(d)):
                assert pyoracle.rs_reconstruct(d, T - d, cw_, True) == 0
            for j in range(d):
                sh[j, off[i]:off[i] + Ls[i]] = cw_[j]
    decided = 0
    for i in range(N):
        g, s = divmod(i, rounds)
        if bin(int(mg[i])).count("1") < d:
            assert st[i] == _lib.SS_ERR_TOO_FEW_SHARDS_PRESENT
            continue
        assert st[i] == 0
        data = b"".join(got[j, off[i]:off[i] + Ls[i]].tobytes() for j in range(d))[:lens[i]]
        assert data == sent[(g, s)], (g, s)
        decided += 1
    assert decided > 0
    # new Accepts at the new ballot return the Preparing positions to Accepting
    r = survivors[-1]
    frames, gs = [], []
    for g in range(G):
        for s in range(rounds):
            data, sh = _codeword(rng, len(sent[(g, s)]), d, T)
            frames.append(pyoracle.frame_accept(2, s, int(nb[g]), d, T - d, len(data), [x if j == r % T else None for j, x in enumerate(sh)],
                                                [1 << (r % T)] * n if cw else None, T))
            gs.append(g)
    buf, offs = _buffer(rng, frames)
    astore = torch.empty(sum(len(f) for f in frames) * 2 + 64, dtype=torch.uint8, device="cuda")
    awal = torch.empty(sum(len(f) + 48 for f in frames) + 64, dtype=torch.uint8, device="cuda")
    res = accs[r].accept(_t(buf), _t(offs), _t(np.array(gs, dtype=np.uint32)), _t(np.full(len(gs), 1, np.uint8)), astore, awal)
    assert (res["verdict"].cpu().numpy().view(np.uint32) == ACC).all()
    assert (accs[r].preparing.cpu().numpy() == 0).all()
    assert (accs[r].accepting.cpu().numpy().view(np.uint64) == (1 << rounds) - 1).all()
    eng.close()
    for a in accs.values():
        a.close()
