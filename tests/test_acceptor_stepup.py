"""Step-up on the device acceptor (ss_acceptor_step_up, summerset_b200/csrc/acceptor_stepup.cu): the Prepare half of a new
RSPaxos / Crossword leader's become_a_leader, and its own vote through the unchanged ss_acceptor_prepare_reply.

`SModel` extends `tests/test_acceptor_prepare.PModel` with a restatement of become_a_leader (rspaxos/leadership.rs:45-185,
crossword/leadership.rs:47-190) over the window, written as the reference computes it: trigger_slot = position of the
first instance below Committed, endprep_slot = rposition, a null instance pushed when every instance is done, then
every instance from exec_bar on that is below Committed prepared at make_greater_ballot(bal_max_seen).  The GPU tests
compare every record cell, frame byte, per-entry output and state word with it, with canaries around the outputs, and
run the fail-over loop with the new leader's own step-up in place of a Prepare modelled from a peer.
"""
import copy
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import pyoracle
from summerset_b200 import _lib
from tests.test_acceptor import ACC, BEYOND, FRAME_OVERFLOW, MALFORMED, WAL_FULL_V, _buffer, _t, _vget
from tests.test_acceptor_commit import _codeword
from tests.test_acceptor_prepare import PREP, PREP_REPLY, PREP_WAL, U64, PModel, PRig, _fill, parse_prep_reply, prep_frame, wal_cell
from tests.test_acceptor_reconstruct import _frame, _var, cw_bytes


def greater_ballot(bal, me):
    """make_greater_ballot (rspaxos/mod.rs:446-454) in u64"""
    return ((((bal >> 8) + 1) << 8) | (me + 1)) & U64


def prep_cell(trigger, ballot, variant=PREP):
    """the 32-byte frame cell ss_acceptor_step_up writes: the Prepare frame, zero to the end of the cell"""
    f = prep_frame(trigger, ballot, variant)
    assert len(f) <= 32
    return f + bytes(32 - len(f))


# ---------------------------------------------------------------------------------------------
# the model
# ---------------------------------------------------------------------------------------------
class SModel(PModel):
    def step_up_one(self, g):
        """become_a_leader for group g -> (verdict, ballot, trigger_slot, endprep_slot, [(slot, ballot)] records)"""
        base, eb = self.base[g], self.eb[g]
        # insts: the window up to the last instance that is not null; Executed = below exec_bar
        n = max(self.inst[g]) + 1 - base if self.inst[g] else 0
        status = ["E" if base + k < eb else self.inst[g].get(base + k, {"st": "N"})["st"] for k in range(n)]
        below = [k for k, st in enumerate(status) if st in ("N", "P", "A")]     # status < Committed
        b = greater_ballot(self.bmax[g], self.me)
        trig = base + (below[0] if below else n)
        endp = base + (below[-1] if below else n)
        if trig >= base + 64:                                                    # the null instance would fall outside
            return BEYOND, b, trig, endp, []
        if trig == base + n:
            status.append("N")                                                   # self.insts.push(null_instance())
        self.bmax[g] = b
        recs = []
        for k in range(max(eb - base, 0), len(status)):
            if status[k] not in ("N", "P", "A"):
                continue
            s = base + k
            inst = self.inst[g].get(s)
            if inst is None:                                                     # a fresh null_instance()
                inst = self.inst[g][s] = dict(bal=0, held=0, dlen=0, shards=None, st="P", vb=0, vm=0, vsh=None)
            inst.update(bal=b, st="P", src=self.me, trig=trig, span=endp - trig)
            recs.append((s, b))
        return ACC, b, trig, endp, recs

    def step_up(self, groups, rec_cap, frame_cap):
        """one ss_acceptor_step_up call -> (per entry (verdict, ballot, trigger, endprep), records [(g, slot, ballot)],
        frames [(g, trigger, ballot)], totals, status)"""
        trial = copy.deepcopy(self)
        res = [trial.step_up_one(g) if g < self.G else (MALFORMED, 0, 0, 0, []) for g in groups]
        rends = np.cumsum([0] + [len(r[4]) for r in res])[1:]
        fends = np.cumsum([0] + [int(r[0] == ACC) for r in res])[1:]
        entries, recs, frames, status = [], [], [], 0
        for i, g in enumerate(groups):
            v, b, trig, endp, _ = res[i]
            if v == ACC and (rends[i] > rec_cap or fends[i] > frame_cap):
                v, status = WAL_FULL_V, FRAME_OVERFLOW
            elif v == ACC:
                r = self.step_up_one(g)
                assert r == res[i]
                recs += [(g, s, bb) for s, bb in r[4]]
                frames.append((g, trig, b))
            entries.append((v, b, trig, endp))
        tr, tf = (int(rends[-1]), int(fends[-1])) if groups else (0, 0)
        return entries, recs, frames, [tr, 32 * tr, tf, 32 * tf], status


# ---------------------------------------------------------------------------------------------
# CPU: the restatement, the bytes, symbols and refusals
# ---------------------------------------------------------------------------------------------
def _acc(m, g, s, bal, held=0b111, dlen=10, src=0):
    sh = [bytes([j]) * (-(-dlen // m.d)) if (held >> j) & 1 else None for j in range(m.T)]
    assert m.accept(g, s, bal, held, dlen, sh, src)


def _commit(m, g, s):
    m.inst[g][s]["st"] = "C"


def test_make_greater_ballot():
    assert greater_ballot(0, 0) == 0x101 and greater_ballot(0, 4) == 0x105
    assert greater_ballot(0x1234_05, 1) == 0x1235_02 and greater_ballot(0x1234_ff, 31) == 0x1235_20
    assert greater_ballot(U64 - 300, 2) == ((((U64 - 300) >> 8) + 1) << 8 | 3) and greater_ballot(U64 - 300, 2) > U64 - 300
    assert greater_ballot(U64, 2) == 3 and greater_ballot(U64 - 255, 0) == 1                # (2^56 << 8) wraps in u64


def test_model_trigger_and_endprep_with_holes():
    m = SModel(1, 5, 2, 3, 5)
    m.base = [100]
    m.bmax = [0x0301]
    for s in (100, 101, 103, 106, 110):
        _acc(m, 0, s, 0x0301)
    _commit(m, 0, 100)
    _commit(m, 0, 110)
    v, b, trig, endp, recs = m.step_up_one(0)
    assert (v, b, trig, endp) == (ACC, 0x0403, 101, 109) and m.bmax == [0x0403]    # a hole below a committed slot is open
    assert [s for s, _ in recs] == list(range(101, 110))                         # holes included, 110 committed
    assert m.inst[0][102]["vb"] == 0 and m.inst[0][103]["vb"] == 0x0301           # a hole is fresh; a vote is kept
    assert m.inst[0][104]["src"] == 2 and m.inst[0][104]["trig"] == 101 and m.inst[0][104]["span"] == 8
    assert m.inst[0][110]["st"] == "C" and m.inst[0][100]["bal"] == 0x0301
    # a repeated step-up: the same range at the next ballot
    v, b, trig, endp, recs = m.step_up_one(0)
    assert (v, b, trig, endp) == (ACC, 0x0503, 101, 109) and len(recs) == 9


def test_model_all_committed_takes_the_null_trigger():
    m = SModel(2, 5, 1, 3, 5)
    for s in range(4):
        _acc(m, 0, s, 1)
        _commit(m, 0, s)
    assert m.step_up_one(0)[:4] == (ACC, 0x102, 4, 4) and sorted(m.inst[0]) == [0, 1, 2, 3, 4]
    assert m.inst[0][4]["st"] == "P" and m.inst[0][4]["vb"] == 0
    assert m.step_up_one(1)[:4] == (ACC, 0x102, 0, 0)                           # an empty window: trigger = base


def test_model_exec_bar_in_the_window():
    m = SModel(1, 5, 0, 3, 5)
    for s in range(8):
        _acc(m, 0, s, 1)
    for s in (0, 1, 2, 5):
        _commit(m, 0, s)
    m.eb = [4]                                                                  # 3 is below exec_bar: done, not touched
    v, b, trig, endp, recs = m.step_up_one(0)
    assert (trig, endp) == (4, 7) and [s for s, _ in recs] == [4, 6, 7] and m.inst[0][3]["st"] == "A"
    m = SModel(1, 5, 0, 3, 5)
    _acc(m, 0, 0, 1)
    m.eb = [9]                                                                  # exec_bar past the log: nothing to mark
    assert m.step_up_one(0)[2:] == (1, 1, [])


def test_model_full_window_is_beyond():
    m = SModel(1, 5, 0, 3, 5)
    m.base = [64]
    for s in range(64, 128):
        _acc(m, 0, s, 7)
        _commit(m, 0, s)
    v, b, trig, endp, recs = m.step_up_one(0)
    assert (v, trig, endp, recs) == (BEYOND, 128, 128, []) and m.bmax == [7]
    m.inst[0][127]["st"] = "A"                                                 # the last one open: it is the range
    assert m.step_up_one(0)[:4] == (ACC, 0x101, 127, 127)


def test_model_cut_and_duplicates():
    m = SModel(3, 5, 0, 3, 5)
    for g in range(3):
        for s in range(3):
            _acc(m, g, s, 1)
    entries, recs, frames, tot, st = copy.deepcopy(m).step_up([0, 1, 0, 7, 2], 1 << 40, 1 << 40)
    assert [e[0] for e in entries] == [ACC, ACC, ACC, MALFORMED, ACC] and tot == [12, 384, 4, 128] and st == 0
    assert entries[2][1] == greater_ballot(entries[0][1], 0) and entries[3][1:] == (0, 0, 0)
    entries, recs, frames, tot, st = m.step_up([0, 1, 0, 7, 2], 7, 1 << 40)      # room for two entries' records
    assert [e[0] for e in entries] == [ACC, ACC, WAL_FULL_V, MALFORMED, WAL_FULL_V] and st == FRAME_OVERFLOW
    assert len(recs) == 6 and len(frames) == 2 and m.bmax == [entries[0][1], entries[1][1], 1]


def test_frame_and_record_cells():
    # hand-worked bytes: PeerMessage::Msg = 0, Prepare = 0, trigger 5, ballot 0x102 (tag 251 + u16 LE)
    assert prep_cell(5, 0x102) == bytes([0, 0, 0, 0, 0, 0, 0, 6, 0, 0, 5, 251, 2, 1]) + bytes(18)
    assert wal_cell(5, 0x102) == bytes([0, 0, 0, 0, 0, 0, 0, 5, 0, 5, 251, 2, 1]) + bytes(19)
    # the widest cells fit 32 bytes: variant < 2^16, 9-byte slot and ballot
    big = prep_cell(U64, U64, 65535)
    assert int.from_bytes(big[:8], "big") == 22 and big[8:11] == _var(0) + _var(65535)[:2] and big[30:] == b"\0\0"
    assert len(wal_cell(U64, U64, 65535).rstrip(b"\0")) <= 29
    assert prep_cell(3, 7, 250)[:-(32 - len(prep_frame(3, 7, 250)))] == prep_frame(3, 7, 250)


def test_acceptor_step_up_symbols_and_refusals():
    lib = _lib.load()
    assert hasattr(lib, "ss_acceptor_step_up")
    args = lambda a, pv, wv: (a, None, 0, pv, wv, None, 0, None, None, 0, None, 0, None, None, None, None, 0, None, None, None, None, None)
    assert lib.ss_acceptor_step_up(*args(None, 0, 0)) == _lib.SS_ERR_INVALID_ARG
    assert b"null acceptor" in lib.ss_last_error()
    for pv, wv in ((1 << 16, 0), (0, 1 << 16), (1 << 31, 5)):
        assert lib.ss_acceptor_step_up(*args(None, pv, wv)) == _lib.SS_ERR_INVALID_ARG
        assert b"below 2^16" in lib.ss_last_error()
    h = C.c_void_p()
    for proto in (_lib.SS_PROTO_MULTIPAXOS, _lib.SS_PROTO_RAFT, _lib.SS_PROTO_CRAFT):       # only RSPaxos / Crossword acceptors
        cfg = _lib.AcceptorConfig(proto, 5, 0, 3, 5, 2, 1, 3)
        assert lib.ss_acceptor_create(None, C.byref(cfg), 4, C.byref(h)) == _lib.SS_ERR_INVALID_ARG
    cfg = _lib.AcceptorConfig(_lib.SS_PROTO_CROSSWORD, 5, 0, 3, 5, 2, 1, 3)
    rc = lib.ss_acceptor_create(None, C.byref(cfg), 4, C.byref(h))
    assert rc in (_lib.SS_ERR_NO_DEVICE, _lib.SS_ERR_INVALID_ARG)
    if not torch.cuda.is_available():
        assert rc == _lib.SS_ERR_NO_DEVICE


# ---------------------------------------------------------------------------------------------
# GPU helpers
# ---------------------------------------------------------------------------------------------
class SRig(PRig):
    """PRig with SModel; step_up compared byte for byte with the restatement"""

    def __init__(self, ctx, protocol, G, n, me, d, T):
        super().__init__(ctx, protocol, G, n, me, d, T)
        self.m = SModel(G, n, me, d, T)

    def set_exec_bar(self, eb):
        self.m.eb = list(eb)
        self.acc.exec_bar.copy_(_t(np.array(eb, dtype=np.uint64)))

    def check_state(self):
        super().check_state()
        a, m = self.acc, self.m
        held, dlen = a.held.cpu().numpy().view(np.uint32), a.data_len.cpu().numpy().view(np.uint32)
        asg = a.assignment.cpu().numpy() if a.assignment is not None else None
        rows = a.assign_rows.cpu().numpy().reshape(m.G * 64, m.n) if a.assign_rows is not None else None
        for g in range(m.G):
            for s, inst in m.inst[g].items():
                at = g * 64 + (s & 63)
                assert (int(held[at]), int(dlen[at])) == (inst["held"], inst["dlen"]), (g, s)
                if inst["dlen"] == 0 and asg is not None:                         # a null instance: an empty assignment
                    assert asg[at] == 0 and not rows[at].any(), (g, s)

    def step_up(self, groups, rec_cap=None, wal_cap=None, frame_cap=None, out_cap=None, pv=PREP, wv=PREP_WAL):
        """groups: a list, or None for every group -> (entries, records)"""
        lst = list(range(self.m.G)) if groups is None else list(groups)
        _, _, _, tot, _ = copy.deepcopy(self.m).step_up(lst, 1 << 62, 1 << 62)
        rc = tot[0] if rec_cap is None else rec_cap
        wc = tot[1] if wal_cap is None else wal_cap
        fc = tot[2] if frame_cap is None else frame_cap
        oc = tot[3] if out_cap is None else out_cap
        wcan = self.rng.integers(0, 256, wc + 64, dtype=np.uint8)
        ocan = self.rng.integers(0, 256, oc + 64, dtype=np.uint8)
        wal, out = _t(wcan.copy()), _t(ocan.copy())
        gt = None if groups is None else _t(np.array(lst, dtype=np.uint32))
        res = self.acc.step_up(wal, rc, out, fc, groups=gt, wal_capacity=wc, out_capacity=oc, prepare_variant=pv, wal_variant=wv)
        entries, recs, frames, totals, status = self.m.step_up(lst, min(rc, wc // 32), min(fc, oc // 32))
        got = {k: v.cpu().numpy() for k, v in res.items()}
        assert [int(x) for x in got["totals"]] == totals
        assert self.ctx.device_status() == status
        n = len(lst)
        assert [int(x) for x in got["verdict"][:n].view(np.uint32)] == [e[0] for e in entries]
        for f, j in (("ballot", 1), ("trigger_slot", 2), ("endprep_slot", 3)):
            assert [int(x) for x in got[f][:n].view(np.uint64)] == [e[j] for e in entries], f
        k = len(recs)
        assert [int(x) for x in got["rec_group"][:k]] == [r[0] for r in recs]
        assert [int(x) for x in got["rec_slot"][:k].view(np.uint64)] == [r[1] for r in recs]
        want = wcan.copy()
        for q, (g, s, b) in enumerate(recs):
            want[32 * q:32 * q + 32] = np.frombuffer(wal_cell(s, b, wv), dtype=np.uint8)
        gw = wal.cpu().numpy()
        if not np.array_equal(gw, want):
            pytest.fail(f"wal: {int((gw != want).sum())} bytes differ, first at {np.nonzero(gw != want)[0][0]}")
        nf = len(frames)
        want = ocan.copy()
        for q, (g, trig, b) in enumerate(frames):
            want[32 * q:32 * q + 32] = np.frombuffer(prep_cell(trig, b, pv), dtype=np.uint8)
            assert (int(got["frame_group"][q]), int(got["frame_dst"][q]), int(got["frame_off"][q])) == (g, 0xff, 32 * q)
            assert int(got["frame_len"][q]) == len(prep_frame(trig, b, pv))
        go = out.cpu().numpy()
        if not np.array_equal(go, want):
            pytest.fail(f"frames: {int((go != want).sum())} bytes differ, first at {np.nonzero(go != want)[0][0]}")
        cut = sum(e[0] == WAL_FULL_V for e in entries)                       # the cut entries' frame records
        for q in range(nf, min(nf + cut, fc)):
            assert (int(got["frame_off"][q].view(np.uint64)), int(got["frame_len"][q]), int(got["frame_dst"][q])) == (U64, 0, 0xff), q
        self.check_state()
        return entries, recs


def _step_and_reply(rig, groups=None, **kw):
    """step-up, then the leader's own PrepareReply for every record: reply_dst = me, parsed like a peer's"""
    entries, recs = rig.step_up(groups, **kw)
    if recs:
        got, frames = rig.prepare_reply([(g, s) for g, s, _ in recs])
        assert all(int(x) == rig.m.me for x in got["reply_dst"])
        assert len(frames) == len(recs)
    return entries, recs


# ---------------------------------------------------------------------------------------------
# GPU 1: populations and codes
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 2, 3, 5, 7, 9, 12, 32])
@pytest.mark.parametrize("protocol", ["rspaxos", "crossword"])
def test_step_up_populations(ctx, protocol, n):
    cases = [(n // 2 + 1, n)] if protocol == "rspaxos" else sorted({(n // 2 + 1, n), (1, min(2 * n, 32)), (min(2 * n, 32),) * 2})
    for d, T in cases:
        me = n - 1
        rig = SRig(ctx, protocol, 6, n, me, d, T)
        rig.set_base([int(x) for x in rig.rng.integers(0, 1 << 40, 6)])
        held = (1 << me) if protocol == "rspaxos" and T == n else None
        _fill(rig, 6, 5, held=held)
        b = rig.m.base
        rig.heartbeat([(g, (me + 1) % max(n, 2), 1, b[g] + (g % 4), 0) for g in range(6)])     # 0..3 committed slots
        _step_and_reply(rig)


@pytest.mark.gpu
def test_step_up_crossword_empty_row(ctx, oracle):
    """Crossword instances accepted with an empty row at me: the leader's own votes are Some((bal, no shards))"""
    n, T, d = 5, 5, 3
    rig = SRig(ctx, "crossword", 4, n, 2, d, T)
    frames, groups = [], []
    for g in range(4):
        for s in range(3):
            dlen = 1 + 97 * (g + s)
            body = _var(0) + _var(2) + _var(s) + _var(3) + cw_bytes(d, T - d, dlen, -(-dlen // d), [None] * T)
            body += _var(n) + b"".join(oracle.bitmap_encode(T, 0) for _ in range(n))
            frames.append(_frame(body))
            groups.append(g)
            assert rig.m.accept(g, s, 3, 0, dlen, [None] * T)
    buf, offs = _buffer(rig.rng, frames)
    store = torch.empty(64, dtype=torch.uint8, device="cuda")
    wal = torch.empty(sum(len(f) + 48 for f in frames), dtype=torch.uint8, device="cuda")
    rig.stores.append(store)
    res = rig.acc.accept(_t(buf), _t(offs), _t(np.array(groups, dtype=np.uint32)), _t(np.zeros(12, np.uint8)), store, wal)
    assert (res["verdict"].cpu().numpy().view(np.uint32) == ACC).all() and ctx.device_status() == 0
    entries, recs = rig.step_up(None)
    got, fr = rig.prepare_reply([(g, s) for g, s, _ in recs])
    assert fr and all(parse_prep_reply(f, d, T)["vote_bal"] == 3 and parse_prep_reply(f, d, T)["vote_mask"] == 0 for _, _, f in fr)


# ---------------------------------------------------------------------------------------------
# GPU 2: window edges, ballots, variants
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_step_up_window_edges(ctx):
    n, T, d = 5, 5, 3
    G = 10
    rig = SRig(ctx, "crossword", G, n, 3, d, T)
    rng = rig.rng
    bases = [0, 250, 1 << 16, (1 << 32) - 3, 1 << 33, 1 << 63, 7, 100, 0, 64]
    rig.set_base(bases)
    items = []
    for g, slots in enumerate([range(5), (0, 3, 9), range(64), range(40), (2,), (), range(10), range(20), range(64), range(64)]):
        for s in slots:
            data, sh = _codeword(rng, int(rng.integers(1, 300)), d, T)
            items.append((g, bases[g] + s, 1 + g, int(rng.integers(1, 1 << T)), data, sh))
    rig.accept(items)
    b = rig.m.base
    hb = [(0, 0, 1, b[0] + 3, 0), (2, 0, 3, b[2] + 64, 0), (3, 0, 4, b[3] + 40, 0), (6, 0, 7, b[6] + 4, 0), (7, 0, 8, b[7] + 20, 0),
          (8, 0, 9, b[8] + 64, 0), (9, 0, 10, b[9] + 10, 0)]
    rig.heartbeat(hb)
    rig.execute(check_data=False)
    rig.set_exec_bar([rig.m.cb[g] if g != 6 else b[6] + 8 for g in range(G)])   # group 6: exec_bar past the committed prefix
    # group 1: an earlier Prepare left Preparing instances; group 9: the window wrapped after an advance
    rig.prepare([(1, 0, prep_frame(b[1] + 2, 50))])
    upto = [b[g] + (6 if g == 9 else 0) for g in range(G)]
    rig.acc.advance(_t(np.array(upto, dtype=np.uint64)))
    rig.m.advance(upto)
    # ballots near 2^64 and at 0 on groups 4 and 5
    bms = rig.acc.bal_max_seen.cpu().numpy().view(np.uint64).copy()
    bms[4], bms[5] = U64 - 77, 0
    rig.acc.bal_max_seen.copy_(_t(bms))
    rig.m.bmax = [int(x) for x in bms]
    entries, _ = _step_and_reply(rig)
    v = [e[0] for e in entries]
    assert v[2] == BEYOND and v[8] == BEYOND and v.count(ACC) == G - 2
    # BEYOND groups finish after an advance; the rest step up again at the next ballot
    upto = [b[g] + 1 for g in range(G)]
    rig.acc.advance(_t(np.array(upto, dtype=np.uint64)))
    rig.m.advance(upto)
    entries, _ = _step_and_reply(rig, [2, 8, 0, 4])
    assert [e[0] for e in entries] == [ACC] * 4


@pytest.mark.gpu
def test_step_up_variants(ctx):
    for pv, wv in [(0, 0), (250, 251), (65535, 300), (7, 65535)]:
        rig = SRig(ctx, "rspaxos", 3, 5, 1, 3, 5)
        _fill(rig, 3, 3, held=0b10)
        rig.step_up([2, 0], pv=pv, wv=wv)


# ---------------------------------------------------------------------------------------------
# GPU 3: capacities, duplicates, out-of-range entries
# ---------------------------------------------------------------------------------------------
def _cut_rig(ctx):
    rig = SRig(ctx, "rspaxos", 4, 5, 1, 3, 5)
    for g, k in enumerate((3, 0, 5, 2)):
        for s in range(k):
            data, sh = _codeword(rig.rng, 40 + s, 3, 5)
            rig.accept([(g, s, 1, 0b10, data, sh)])
    return rig


@pytest.mark.gpu
def test_step_up_cut_every_boundary(ctx):
    """the list cut at every record and frame boundary by each of the four capacities, then drained"""
    lst = [2, 0, 1, 3, 2, 9, 0]
    full = _cut_rig(ctx)
    full.step_up(lst)
    tot = copy.deepcopy(_cut_rig(ctx).m).step_up(lst, 1 << 62, 1 << 62)[3]
    for which in ("rec", "wal", "frame", "out"):
        top = tot[0] if which in ("rec", "wal") else tot[2]
        for cap in range(0, top + 1):
            rig = _cut_rig(ctx)
            kw = {"rec": dict(rec_cap=cap), "wal": dict(wal_cap=32 * cap + 31), "frame": dict(frame_cap=cap),
                  "out": dict(out_cap=32 * cap + 17)}[which]
            entries, _ = rig.step_up(lst, **kw)
            rest = [g for g, e in zip(lst, entries) if e[0] == WAL_FULL_V]
            if rest:
                rig.step_up(rest)
            assert rig.m.prep_words() == full.m.prep_words() and rig.m.bmax == full.m.bmax
            assert {(g, s): (i["bal"], i["trig"], i["span"], i["src"]) for g in range(4) for s, i in full.m.inst[g].items()} == \
                   {(g, s): (i["bal"], i["trig"], i["span"], i["src"]) for g in range(4) for s, i in rig.m.inst[g].items()}


@pytest.mark.gpu
def test_step_up_duplicates_and_out_of_range(ctx):
    """a group listed several times steps up once per entry in list order; entries >= n_groups are ignored"""
    G = 300
    rig = SRig(ctx, "crossword", G, 7, 4, 4, 7)
    for g in range(0, G, 37):
        data, sh = _codeword(rig.rng, 100, 4, 7)
        rig.accept([(g, 1, 2, 0b1111, data, sh)])
    rng = rig.rng
    lst = [int(x) for x in rng.integers(0, G + 3, 5000)] + [G, (1 << 32) - 1, 0, 0, 0]
    entries, _ = _step_and_reply(rig, lst)
    # each occurrence of a group took the next greater ballot
    seen = {}
    for g, e in zip(lst, entries):
        if g >= G:
            assert e == (MALFORMED, 0, 0, 0)
            continue
        assert e[1] == greater_ballot(seen.get(g, 0), 4)
        seen[g] = e[1]


@pytest.mark.gpu
@pytest.mark.parametrize("G", [1, 255, 256, 257, 65537])
def test_step_up_sort_key_edges_and_grid_caps(ctx, G):
    rig = SRig(ctx, "rspaxos", G, 5, 2, 3, 5)
    rng = rig.rng
    gs = sorted({0, G - 1, G // 2} | {int(x) for x in rng.integers(0, G, 30)})
    for g in gs:
        data, sh = _codeword(rng, int(rng.integers(1, 200)), 3, 5)
        rig.accept([(g, int(rng.integers(0, 4)), 1, 0b10110, data, sh)])
    rig.step_up(None)
    rig.step_up([int(x) for x in rng.integers(0, G + 1, 100000 if G == 65537 else 3000)])


# ---------------------------------------------------------------------------------------------
# GPU 4: Preparing instances stop the commit walk and execution
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_step_up_blocks_commit_and_execute(ctx):
    n, T, d = 5, 5, 3
    rig = SRig(ctx, "crossword", 3, n, 1, d, T)
    _fill(rig, 3, 8, bal=2, held=0b00111)
    rig.heartbeat([(g, 2, 2, g + 1, 0) for g in range(3)])                     # slots below g + 1 committed
    rig.execute(check_data=False)
    rig.set_exec_bar(rig.m.cb)
    entries, _ = rig.step_up(None)
    assert [e[2] for e in entries] == [1, 2, 3]
    # the leader's own heartbeat at its new ballot and a stale one from the old leader commit nothing past the trigger
    rig.heartbeat([(g, 1, entries[g][1], 64, 0) for g in range(3)] + [(g, 2, 2, 64, 0) for g in range(3)])
    recs, _ = rig.execute(check_data=False)
    assert recs == []
    assert [int(x) for x in rig.acc.commit_bar.cpu().numpy()] == [1, 2, 3]


# ---------------------------------------------------------------------------------------------
# GPU 5: the closed loop -- the new leader's own step-up, the survivors' Prepare, every reply merged
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("protocol,n,T,d", [("rspaxos", 3, 3, 2), ("rspaxos", 5, 5, 3), ("rspaxos", 7, 7, 4),
                                            ("crossword", 5, 5, 3), ("crossword", 7, 14, 7)])
def test_step_up_closed_loop(ctx, oracle, protocol, n, T, d):
    from summerset_b200 import workloads as wl
    from summerset_b200.engine import Acceptor, LeaderEngine, prepare_reply_parse
    cw = protocol == "crossword"
    G, rounds, leader = 16, 3, 1
    rng = np.random.default_rng(n * 100 + T + 1)
    eng = LeaderEngine(ctx, protocol, G, n, 1, 1, **(dict(rs_total_shards=T, rs_data_shards=d) if cw else {}))
    bal = rng.integers(1, 1 << 20, G).astype(np.uint64)
    eng.set_prepared_ballots(_t(bal))
    if cw:
        policies = np.array([oracle.cw_brr_assignment(n, T, d)], dtype=np.uint32)
        eng.set_policies([list(map(int, q)) for q in policies], True)
    else:
        policies = np.array([[1 << r for r in range(n)]], dtype=np.uint32)
    survivors = list(range(1, n))                       # replica 0 led; replica 1 steps up
    accs = {r: Acceptor(ctx, protocol, G, n, r, d, T) for r in survivors}
    m = SModel(G, n, leader, d, T)                      # the new leader's acceptor, restated from the history
    keep = []
    for rnd in range(rounds):
        lens = (wl.cfg4_lengths(G, seed_extra=rnd)[0] // 16 + rng.integers(1, 7, G)).astype(np.uint32)
        data_off = (16 + np.cumsum(lens.astype(np.int64) + 5) - lens.astype(np.int64)).astype(np.uint64)
        arena = rng.integers(0, 256, int(data_off[-1]) + int(lens[-1]) + 64, dtype=np.uint8)
        L = (lens.astype(np.int64) + d - 1) // d
        store = torch.zeros((T, int(((L + 31) // 32 * 32).sum()) + 32), dtype=torch.uint8, device="cuda")
        keep.append(store)
        slot_out, shard_off, _ = eng.propose_ragged(_t(arena), _t(data_off), _t(lens), store, _t(np.zeros(G, np.uint8)) if cw else None)
        slots = slot_out.cpu().numpy().view(np.uint64)
        for r in survivors:
            out, off, fl, _ = ctx.frame_accept_pack_ragged(store, shard_off, _t(lens), d, T - d, policies, _t(np.zeros(G, np.uint8)), r,
                                                           slot_out, _t(bal), with_assignment=cw)
            oh, flh, bh = off.cpu().numpy(), fl.cpu().numpy(), out.cpu().numpy()
            gs = [g for g in range(G) if rnd == rounds - 1 or (g + r + rnd) % 4 != 0]
            frames = [bh[int(oh[g]):int(oh[g]) + int(flh[g])].tobytes() for g in gs]
            buf, offs = _buffer(rng, frames)
            astore = torch.empty(sum(len(f) for f in frames) * 2 + 64, dtype=torch.uint8, device="cuda")
            awal = torch.empty(sum(len(f) + 48 for f in frames) + 64, dtype=torch.uint8, device="cuda")
            keep.append(astore)
            res = accs[r].accept(_t(buf), _t(offs), _t(np.array(gs, dtype=np.uint32)), _t(np.zeros(len(gs), np.uint8)), astore, awal)
            assert (res["verdict"].cpu().numpy().view(np.uint32) == ACC).all()
            if r == leader:
                for g in gs:
                    m.bmax[g] = int(bal[g])
                    m.inst[g][int(slots[g])] = dict(bal=int(bal[g]), held=int(policies[0][leader]), dlen=int(lens[g]), shards=None,
                                                    st="A", vb=int(bal[g]), vm=int(policies[0][leader]), vsh=None, src=0, trig=0, span=0)
        if rnd == 0:                                    # the old leader's heartbeat commits round 0 where it was accepted
            for r in survivors:
                accs[r].heartbeat(_t(np.arange(G, dtype=np.uint32)), _t(np.zeros(G, np.uint8)), _t(bal), _t(slots + np.uint64(1)),
                                  _t(np.zeros(G, np.uint64)))
            for g in range(G):
                if 0 in m.inst[g]:
                    m.inst[g][0]["st"] = "C"
    assert ctx.device_status() == 0
    # the new leader's step-up: records, frames, outputs as the restatement has them
    ldr = accs[leader]
    wal = torch.empty(G * 64 * 32, dtype=torch.uint8, device="cuda")
    pout = torch.empty(G * 32, dtype=torch.uint8, device="cuda")
    st = ldr.step_up(wal, G * 64, pout, G)
    entries, recs, frames, totals, status = m.step_up(list(range(G)), 1 << 40, 1 << 40)
    assert ctx.device_status() == status == 0
    assert [int(x) for x in st["totals"].cpu().numpy()] == totals
    assert [int(x) for x in st["verdict"].cpu().numpy().view(np.uint32)] == [e[0] for e in entries] == [ACC] * G
    assert [int(x) for x in st["ballot"].cpu().numpy().view(np.uint64)] == [greater_ballot(int(b), leader) for b in bal]
    assert [int(x) for x in st["trigger_slot"].cpu().numpy()] == [e[2] for e in entries]
    assert [int(x) for x in st["endprep_slot"].cpu().numpy()] == [e[3] for e in entries]
    nrec = totals[0]
    assert [(int(g), int(s)) for g, s in zip(st["rec_group"][:nrec].cpu().numpy(), st["rec_slot"][:nrec].cpu().numpy())] == \
           [(g, s) for g, s, _ in recs]
    pb = pout.cpu().numpy()
    for q, (g, trig, b) in enumerate(frames):
        assert pb[32 * q:32 * q + 32].tobytes() == prep_cell(trig, b)
    # the Prepare frames to the other survivors, as read off the leader's connection
    fl = st["frame_len"].cpu().numpy()
    pframes = [pb[32 * q:32 * q + int(fl[q])].tobytes() for q in range(G)]
    replies = {}                                        # (r, g, slot) -> (vote_bal, vote_mask, shards, data_len)

    def collect(r, out, off_t, rg, rs):
        pr = prepare_reply_parse(ctx, out, off_t, d, T)
        pr = {k: v.cpu().numpy() for k, v in pr.items()}
        ob = out.cpu().numpy()
        assert (pr["kind"] == PREP_REPLY).all()
        for k in range(len(rg)):
            shards = {}
            at = int(pr["shards_at"][k])
            Ls = -(-int(pr["data_len"][k]) // d) if pr["data_len"][k] else 0
            if int(pr["vote_bal"][k]) != 0:
                for j in range(T):
                    at += 1
                    if ob[at - 1] == 1:
                        at = _vget(ob, at)[1]
                        shards[j] = ob[at:at + Ls].tobytes()
                        at += Ls
            replies[(r, int(rg[k]), int(pr["slot"][k]))] = (int(pr["vote_bal"][k]), int(pr["vote_mask"][k]) & 0xffffffff, shards,
                                                            int(pr["data_len"][k]))
            assert int(pr["slot"][k]) == int(rs[k])
    for r in survivors:
        if r == leader:                                 # the leader's own replies: the unchanged reply path, reply_dst = me
            rg, rs = st["rec_group"][:nrec], st["rec_slot"][:nrec]
        else:
            buf, offs = _buffer(rng, pframes)
            fwal = torch.empty(G * 64 * 32, dtype=torch.uint8, device="cuda")
            res = accs[r].prepare(_t(buf), _t(offs), _t(np.arange(G, dtype=np.uint32)), _t(np.full(G, leader, np.uint8)), fwal, G * 64)
            assert (res["verdict"].cpu().numpy().view(np.uint32) == ACC).all()
            k = int(res["totals"][0])
            rg, rs = res["rec_group"][:k], res["rec_slot"][:k]
        out = torch.empty(len(rg) * 4096 + 16, dtype=torch.uint8, device="cuda")
        rr = accs[r].prepare_reply(rg, rs, out)
        assert ctx.device_status() == 0
        dst = rr["reply_dst"].cpu().numpy()
        assert (dst == leader).all()                     # the followers' source and the leader's own: me
        collect(r, out, rr["reply_off"], rg.cpu().numpy(), rs.cpu().numpy())
    # the merge over every survivor's reply for the leader's prepared instances equals the oracle's stream and decision
    inst = [(g, s) for g, s, _ in recs]
    N, R = len(inst), len(survivors)
    vb = np.zeros((R, N), np.uint64)
    vm = np.zeros((R, N), np.uint32)
    for ri, r in enumerate(survivors):
        for i, (g, s) in enumerate(inst):
            vb[ri, i], vm[ri, i] = replies[(r, g, s)][:2]
    acks = np.full(N, R, np.uint8)
    mb, mg, act = ctx.prepare_merge(_t(vb), _t(vm.view(np.int32)), _t(acks), d, n, n - R)
    mb, mg, act = mb.cpu().numpy().view(np.uint64), mg.cpu().numpy().view(np.uint32), act.cpu().numpy()
    decided = 0
    for i in range(N):
        has = (vb[:, i] > 0).astype(np.uint8)
        want_b, want_m = oracle.prepare_merge_stream(has, vb[:, i], vm[:, i])
        assert (int(mb[i]), int(mg[i])) == (want_b, want_m), i
        assert int(act[i]) == oracle.prepare_decide(want_m, R, d, n, n - R), i
        decided += int(act[i]) & oracle.PM_USE
    assert decided > 0
    # the leader's own vote is in the merge: its voted shards come back byte for byte in its own replies
    for g, s in inst:
        b_, m_, sh, _ = replies[(leader, g, s)]
        li = m.inst[g].get(s)
        assert (b_, m_) == ((li["vb"], li["vm"]) if li["vb"] else (0, 0)), (g, s)
    # the reconstruct reads, called afterwards, list the restatement's recon_slots
    rout = torch.empty(G * 4096, dtype=torch.uint8, device="cuda")
    rd = ldr.step_up_reads(rout, G * 64, 64)
    nf = int(rd["totals"][0])
    ob, fo, fg = rout.cpu().numpy(), rd["frame_off"].cpu().numpy(), rd["frame_group"].cpu().numpy()
    listed = set()
    for f in range(nf):
        b = ob[int(fo[f]):]
        q = 8
        q = _vget(b, q)[1]
        q = _vget(b, q)[1]
        cnt, q = _vget(b, q)
        for _ in range(cnt):
            s, q = _vget(b, q)
            listed.add((int(fg[f]), s))
            if cw:
                for _ in range(3):
                    q = _vget(b, q)[1]
    recon = {(g, s) for g in range(G) for s, i in m.inst[g].items() if i["st"] == "C" and s >= m.eb[g]
             and bin(i["held"]).count("1") < d}
    assert listed == recon
    eng.close()
    for a in accs.values():
        a.close()
