"""WAL recovery on the device acceptor (ss_acceptor_recover, summerset_b200/csrc/acceptor_recover.cu).

`RModel` restates recover_apply_entry (rspaxos/recovery.rs:10-119, crossword/recovery.rs:10-124) per record over the
acceptor's 64-slot window, and recover_from_wal's read loop, which ends a group's log at the first record it cannot
decode.  Records are decoded by hand: an AcceptData body is handed to `tests/test_acceptor._decode` behind an Accept
header, so it is held to the rules ss_acceptor_accept applies to the Accept body.  Record bytes are cross-checked with
the oracle's ssor_wal_accept_data / ssor_wal_commit_slot and the PrepareBal cell ss_acceptor_prepare writes.  The GPU
tests collect the records a live acceptor writes (accept, prepare, heartbeat + ss_wal_commit_pack_dev), replay them into
a fresh acceptor and compare every state word, every shard read through shard_addr and the execution records.
"""
import copy
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import pyoracle
from summerset_b200 import _lib
from tests.test_acceptor import ACC, BEYOND, MALFORMED, STALE_SLOT, STORE_FULL, STORE_FULL_V, Cfg, _acceptor, _buffer, _decode, _t, _vget
from tests.test_acceptor_commit import _codeword, _pitch, _r16
from tests.test_acceptor_prepare import wal_cell
from tests.test_acceptor_reconstruct import _frame, _nm, _var

AFTER_END = _lib.SS_RECOVER_VERDICT_AFTER_END
PREP_V, COMMIT_V = 0, 2
U64 = (1 << 64) - 1


# ---------------------------------------------------------------------------------------------
# records and the restatement
# ---------------------------------------------------------------------------------------------
def prepare_bal(slot, ballot, nm=False):
    """WalEntry::PrepareBal as ss_acceptor_prepare writes it: the first 8 + length bytes of its 32-byte cell"""
    if nm:
        body = _var(PREP_V) + (_nm(slot) if slot < 1 << 16 else _var(slot)) + (_nm(ballot) if ballot < 1 << 16 else _var(ballot))
        return _frame(body)
    cell = wal_cell(slot, ballot, PREP_V)
    return cell[:8 + int.from_bytes(cell[:8], "big")]


def commit_slot(slot, nm=False):
    return _frame(_var(COMMIT_V) + (_nm(slot) if nm and slot < 1 << 16 else _var(slot)))


def accept_data(cfg, slot, ballot, dlen, shards, rows=None, nm=False):
    """WalEntry::AcceptData as ss_acceptor_accept writes it: wal_variant, then the Accept body from `slot` on"""
    fr = pyoracle.frame_accept(cfg.av, slot, ballot, cfg.d, cfg.T - cfg.d, dlen, shards, rows if cfg.cw else None, cfg.T)
    f = _decode(fr, cfg)
    assert isinstance(f, dict)
    tail = fr[f["slot_at"]:f["end"]]
    if nm and slot < 1 << 16:                                     # slot as tag 251 + u16
        tail = _nm(slot) + tail[len(_var(slot)):]
    return _frame(_var(cfg.wv) + tail)


def parse_record(rec, cfg):
    """-> ("P", slot, ballot) / ("C", slot) / ("A", slot, ballot, Accept fields) or MALFORMED"""
    if len(rec) < 8:
        return MALFORMED
    ln = int.from_bytes(rec[:8], "big")
    if ln > len(rec) - 8:
        return MALFORMED
    b = rec[8:8 + ln]
    r = _vget(b, 0)
    if r is None:
        return MALFORMED
    v, n = r
    if v == cfg.wv:
        f = _decode(_frame(_var(0) + _var(cfg.av) + b[n:]), cfg)
        return ("A", f["slot"], f["ballot"], f) if isinstance(f, dict) else MALFORMED
    if v not in (PREP_V, COMMIT_V):
        return MALFORMED
    vals = []
    for _ in range(2 if v == PREP_V else 1):
        r = _vget(b, n)
        if r is None:
            return MALFORMED
        vals.append(r[0])
        n = r[1]
    if n != len(b):
        return MALFORMED
    return ("P", vals[0], vals[1]) if v == PREP_V else ("C", vals[0])


class RModel:
    """inst[g][slot] (non-null instances only): st "P" / "A" / "C", bal, held, dlen, shards, vb, vm, asg, rows, src,
    trig, span, store (the region offset of a recovered instance)"""

    def __init__(self, cfg, G):
        self.cfg, self.G = cfg, G
        self.base, self.bmax = [0] * G, [0] * G
        self.inst = [dict() for _ in range(G)]

    def apply_entry(self, g, p):
        """recover_apply_entry for one record inside the window"""
        slot = p[1]
        inst = self.inst[g].get(slot)
        if inst is None:                                          # a fresh null_instance()
            inst = self.inst[g][slot] = dict(st=None, bal=0, held=0, dlen=0, shards=None, vb=0, vm=0, asg=0,
                                             rows=[0] * self.cfg.n if self.cfg.cw else None, store=None)
        inst.update(src=0xff, trig=0, span=0)
        if p[0] == "C":
            inst["st"] = "C"
            return
        inst["bal"] = p[2]
        self.bmax[g] = max(self.bmax[g], p[2])
        if p[0] == "P":
            inst["st"] = "P"
            return
        f = p[3]
        inst.update(st="A", held=f["held"], dlen=f["dlen"], shards=f["shards"], vb=p[2], vm=f["held"], L=f["L"])
        if self.cfg.cw:
            inst.update(asg=f["asg"][self.cfg.me], rows=list(f["asg"]))

    def recover(self, recs, groups, cap):
        """one ss_acceptor_recover call -> (verdicts, total, status)"""
        parsed = [parse_record(r, self.cfg) for r in recs]
        verdicts = [None] * len(recs)
        applied, by_group = {}, {}
        for i, g in enumerate(groups):
            by_group.setdefault(g, []).append(i)
        for g in range(self.G):
            for inst in self.inst[g].values():
                inst["store"] = None                               # check_state reads the regions this call placed
        for g in sorted(by_group):
            idxs = by_group[g]
            if g >= self.G:
                for i in idxs:
                    verdicts[i] = MALFORMED
                continue
            ended = cut = False
            applied[g] = []
            for i in idxs:
                p = parsed[i]
                if ended:
                    v = AFTER_END
                elif p == MALFORMED:
                    v, ended = MALFORMED, True
                elif cut or p[1] >= self.base[g] + 64:
                    v, cut = BEYOND, True
                elif p[1] < self.base[g]:
                    v = STALE_SLOT
                else:
                    v = ACC
                    applied[g].append(i)
                verdicts[i] = v
        # the defining AcceptData of each slot, and each group's bytes
        define, size = {}, [0] * self.G
        for g, idxs in applied.items():
            last = {}
            for i in idxs:
                if parsed[i][0] == "A":
                    last[parsed[i][1]] = i
            define[g] = last
            size[g] = sum(bin(parsed[i][3]["held"]).count("1") * _pitch(parsed[i][3]["L"]) for i in last.values())
        offs = np.concatenate([[0], np.cumsum(size)]).astype(np.int64)
        status = 0
        for g, idxs in applied.items():
            if int(offs[g + 1]) > cap:
                for i in idxs:
                    verdicts[i] = STORE_FULL_V
                    status = STORE_FULL
                continue
            for i in idxs:
                self.apply_entry(g, parsed[i])
            o = int(offs[g])
            for s in sorted(define[g]):                            # window order
                inst = self.inst[g][s]
                inst["store"] = o
                o += bin(inst["held"]).count("1") * _pitch(inst["L"])
        return verdicts, int(offs[-1]), status

    def words(self):
        w = {k: [0] * self.G for k in "PAC"}
        for g in range(self.G):
            for s, inst in self.inst[g].items():
                w[inst["st"]][g] |= 1 << (s & 63)
        return w

    def advance(self, upto):
        for g, u in enumerate(upto):
            k = min(max(u - self.base[g], 0), 64)
            for s in [s for s in self.inst[g] if s < self.base[g] + k]:
                del self.inst[g][s]
            self.base[g] += k


# ---------------------------------------------------------------------------------------------
# CPU: the restatement on hand-built sequences, record bytes, refusals
# ---------------------------------------------------------------------------------------------
RS = Cfg("rspaxos", 5, 1, 3, 5)


def _shards(cfg, dlen, held, fill=1):
    L = -(-dlen // cfg.d)
    return [bytes([fill + j]) * L if (held >> j) & 1 else None for j in range(cfg.T)]


def _ad(cfg, slot, bal, held=0b00111, dlen=9, fill=1, rows=None):
    return accept_data(cfg, slot, bal, dlen, _shards(cfg, dlen, held, fill), rows=rows)


def test_model_prepare_bal_over_null_accepting_committed():
    m = RModel(RS, 1)
    recs = [_ad(RS, 1, 3), _ad(RS, 2, 3), commit_slot(2), prepare_bal(0, 5), prepare_bal(1, 5), prepare_bal(2, 5)]
    v, total, st = m.recover(recs, [0] * 6, 1 << 20)
    assert v == [ACC] * 6 and st == 0 and total == 2 * 3 * 32
    assert [m.inst[0][s]["st"] for s in range(3)] == ["P"] * 3 and m.bmax == [5]
    assert m.inst[0][0]["vb"] == 0 and m.inst[0][0]["held"] == 0                       # null: voted None, no shards
    assert (m.inst[0][1]["vb"], m.inst[0][1]["vm"], m.inst[0][1]["bal"]) == (3, 0b111, 5)   # the vote stays
    assert m.inst[0][2]["src"] == 0xff and m.inst[0][2]["trig"] == 0


def test_model_accept_data_out_of_committed_and_commit_on_null():
    m = RModel(RS, 1)
    v, _, _ = m.recover([_ad(RS, 4, 1), commit_slot(4), _ad(RS, 4, 2, held=0b11000, fill=7), commit_slot(9)], [0] * 4, 1 << 20)
    assert v == [ACC] * 4
    assert m.inst[0][4]["st"] == "A" and m.inst[0][4]["held"] == 0b11000 and m.inst[0][4]["vb"] == 2 and m.inst[0][4]["bal"] == 2
    assert m.inst[0][9]["st"] == "C" and m.inst[0][9]["held"] == 0 and m.inst[0][9]["bal"] == 0
    assert m.words()["C"] == [1 << 9] and m.bmax == [2]


def test_model_two_accept_data_for_one_slot():
    m = RModel(RS, 1)
    v, total, _ = m.recover([_ad(RS, 0, 1, held=0b11111), _ad(RS, 0, 1, held=0b00001, fill=9)], [0, 0], 1 << 20)
    assert v == [ACC, ACC] and total == 32 and m.inst[0][0]["held"] == 1 and m.inst[0][0]["shards"][0] == bytes([9]) * 3


def test_model_stale_beyond_and_malformed():
    m = RModel(RS, 3)
    m.base = [10, 10, 10]
    recs = [_ad(RS, 9, 1), _ad(RS, 10, 1), prepare_bal(74, 2), commit_slot(10), prepare_bal(12, 1),      # group 0
            _ad(RS, 11, 1), None, commit_slot(11), _ad(RS, 12, 1),                                         # group 1
            commit_slot(10)]                                                                               # group 5
    groups = [0, 0, 0, 0, 0, 1, 1, 1, 1, 5]
    recs[6] = _frame(_var(PREP_V) + _var(11) + _var(2) + b"\0")                                             # trailing byte
    v, total, st = m.recover(recs, groups, 1 << 20)
    assert v == [STALE_SLOT, ACC, BEYOND, BEYOND, BEYOND, ACC, MALFORMED, AFTER_END, AFTER_END, MALFORMED]
    assert sorted(m.inst[0]) == [10] and sorted(m.inst[1]) == [11] and total == 2 * 3 * 32
    assert parse_record(_frame(_var(7) + _var(1)), RS) == MALFORMED                                        # another variant
    assert parse_record(commit_slot(3)[:-1], RS) == MALFORMED


def test_model_store_cut_per_group():
    m = RModel(RS, 3)
    recs = [_ad(RS, 0, 1), _ad(RS, 0, 1), prepare_bal(0, 1), _ad(RS, 0, 1)]
    v, total, st = m.recover(recs, [0, 1, 1, 2], 2 * 96)
    assert total == 3 * 96 and v == [ACC, ACC, ACC, STORE_FULL_V] and st == STORE_FULL
    assert m.inst[1][0]["st"] == "P" and m.inst[1][0]["store"] == 96 and 0 not in m.inst[2]


def test_record_bytes_every_varint_width(oracle):
    for x in (0, 1, 250, 251, 0xffff, 0x10000, 0xffffffff, 1 << 32, U64):
        for y in (0, 250, 251, 0x10000, 1 << 40):
            sh = _shards(RS, 10, 0b10101)
            want = oracle.wal_accept_data(x, y, 3, 2, 10, sh)
            assert accept_data(RS, x, y, 10, sh) == want
            p = parse_record(want, RS)
            assert p[:3] == ("A", x, y) and p[3]["held"] == 0b10101 and p[3]["dlen"] == 10
            assert parse_record(prepare_bal(x, y), RS) == ("P", x, y)
            assert parse_record(prepare_bal(x, y, nm=True), RS) == ("P", x, y)
        assert commit_slot(x) == oracle.wal_commit_slot(x)
        assert parse_record(commit_slot(x, nm=True), RS) == ("C", x)
        cell = wal_cell(x, 7)
        assert prepare_bal(x, 7) == cell[:8 + cell[7]] and not any(cell[8 + cell[7]:])
        if x < 1 << 16:
            nm = accept_data(RS, x, 5, 10, _shards(RS, 10, 1), nm=True)
            assert parse_record(nm, RS)[:3] == ("A", x, 5)


def test_recover_symbols_and_refusals():
    lib = _lib.load()
    assert hasattr(lib, "ss_acceptor_recover")
    assert lib.ss_acceptor_recover(None, None, 0, None, None, 0, 0, 2, None, 0, None, None) == _lib.SS_ERR_INVALID_ARG
    cfg = _lib.AcceptorConfig(_lib.SS_PROTO_RSPAXOS, 5, 0, 3, 5, 2, 1, 3)
    h = C.c_void_p()
    rc = lib.ss_acceptor_create(None, C.byref(cfg), 4, C.byref(h))
    assert rc in (_lib.SS_ERR_NO_DEVICE, _lib.SS_ERR_INVALID_ARG)
    if not torch.cuda.is_available():
        assert rc == _lib.SS_ERR_NO_DEVICE


# ---------------------------------------------------------------------------------------------
# GPU helpers
# ---------------------------------------------------------------------------------------------
class Live:
    """a live acceptor; every WAL record its calls write, with its group, in call order"""

    def __init__(self, ctx, cfg, G, base, rng):
        self.ctx, self.cfg, self.G, self.rng = ctx, cfg, G, rng
        self.acc = _acceptor(ctx, cfg, G)
        self.acc.window_base.copy_(_t(np.array(base, dtype=np.uint64)))
        self.recs, self.stores = [], []

    def accept(self, items):
        """items: (g, slot, ballot, held, dlen); Crossword rows are random"""
        cfg, frames, groups = self.cfg, [], []
        for g, s, bal, held, dlen in items:
            _, sh = _codeword(self.rng, dlen, cfg.d, cfg.T)
            rows = [int(x) for x in self.rng.integers(0, 1 << cfg.T, cfg.n)] if cfg.cw else None
            frames.append(pyoracle.frame_accept(cfg.av, s, bal, cfg.d, cfg.T - cfg.d, dlen,
                                                [sh[j] if (held >> j) & 1 else None for j in range(cfg.T)], rows, cfg.T))
            groups.append(g)
        buf, offs = _buffer(self.rng, frames)
        need = sum(bin(h).count("1") * _pitch(-(-dl // cfg.d)) for _, _, _, h, dl in items)
        store = torch.zeros(need + 64, dtype=torch.uint8, device="cuda")
        wal = torch.zeros(sum(len(f) + 48 for f in frames) + 64, dtype=torch.uint8, device="cuda")
        self.stores.append(store)
        out = self.acc.accept(_t(buf), _t(offs), _t(np.array(groups, dtype=np.uint32)), _t(np.full(len(items), 0, np.uint8)),
                              store, wal)
        v = out["verdict"].cpu().numpy().view(np.uint32)
        wo, wl, w = out["wal_off"].cpu().numpy(), out["wal_len"].cpu().numpy(), wal.cpu().numpy()
        for i, g in enumerate(groups):
            if int(v[i]) == ACC:
                self.recs.append((g, w[wo[i]:wo[i] + wl[i]].tobytes()))
        assert self.ctx.device_status() == 0
        return v

    def prepare(self, items):
        """items: (g, peer, trigger, ballot)"""
        from tests.test_acceptor_prepare import prep_frame
        frames = [prep_frame(t, b) for _, _, t, b in items]
        buf, offs = _buffer(self.rng, frames)
        wal = torch.zeros(32 * 64 * len(items) + 64, dtype=torch.uint8, device="cuda")
        res = self.acc.prepare(_t(buf), _t(offs), _t(np.array([g for g, _, _, _ in items], dtype=np.uint32)),
                               _t(np.array([p for _, p, _, _ in items], dtype=np.uint8)), wal, 64 * len(items))
        n = int(res["totals"][0])
        w, rg = wal.cpu().numpy(), res["rec_group"].cpu().numpy()
        for k in range(n):
            cell = w[32 * k:32 * k + 32].tobytes()
            self.recs.append((int(rg[k]), cell[:8 + cell[7]]))
        assert self.ctx.device_status() == 0

    def heartbeat(self, recs):
        cols = list(zip(*recs))
        newly = self.acc.heartbeat(_t(np.array(cols[0], dtype=np.uint32)), _t(np.array(cols[1], dtype=np.uint8)),
                                   _t(np.array(cols[2], dtype=np.uint64)), _t(np.array(cols[3], dtype=np.uint64)),
                                   _t(np.array(cols[4], dtype=np.uint64)))
        entries, eg, el, cnt = self.ctx.wal_commit_pack(newly, self.acc.window_base, 64 * self.G)
        n = int(cnt[0])
        e, g_, l_ = entries.cpu().numpy(), eg.cpu().numpy(), el.cpu().numpy()
        cells = sorted((int(g_[k]), e[k, :l_[k]].tobytes()) for k in range(n))   # per group in slot order
        self.recs += cells


def _nm_some(recs, cfg, rng):
    """every third PrepareBal / CommitSlot / AcceptData re-spelt with non-minimal varints where the values allow"""
    out = []
    for k, (g, r) in enumerate(recs):
        if k % 3 == 0:
            p = parse_record(r, cfg)
            if p[0] == "P":
                r = prepare_bal(p[1], p[2], nm=True)
            elif p[0] == "C":
                r = commit_slot(p[1], nm=True)
            elif p[1] < 1 << 16:
                b = r[8:]
                n = len(_var(cfg.wv))
                tail = b[n + len(_var(p[1])):]
                r = _frame(b[:n] + _nm(p[1]) + tail)
            assert parse_record(r, cfg)[:2] == p[:2]
        out.append((g, r))
    return out


def _recover(ctx, acc, m, recs, rng, cap=None, pad=64, check=True):
    """one ss_acceptor_recover call checked against the restatement; returns (verdicts, store)"""
    buf, offs = _buffer(rng, [r for _, r in recs])
    groups = [g for g, _ in recs]
    want_v, total, status = copy.deepcopy(m).recover([r for _, r in recs], groups, 1 << 62)
    cap = total if cap is None else cap
    canary = rng.integers(0, 256, pad + cap + pad, dtype=np.uint8)
    full = _t(canary.copy())
    store = full[pad:pad + cap] if cap else full[pad:pad + 16]
    res = acc.recover(_t(buf), _t(offs), _t(np.array(groups, dtype=np.uint32)), store, cap)
    want_v, total, status = m.recover([r for _, r in recs], groups, cap)
    assert [int(x) for x in res["verdict"].cpu().numpy().view(np.uint32)] == want_v
    assert int(res["total"][0]) == total
    assert ctx.device_status() == status
    if check:
        written = check_state(acc, m, full, pad)
        st = full.cpu().numpy()
        bad = np.nonzero((st != canary) & ~written)[0]                 # pads, gaps between regions, round16(L)..pitch
        assert len(bad) == 0, f"{len(bad)} store bytes outside the shards changed, first at {bad[0] - pad} of the store"
    return want_v, full


def check_state(acc, m, full, pad):
    """every state word against the restatement; the shards through shard_addr with bytes L..round16(L) zero.  Returns
    the mask of the store bytes the call was to write (each held shard's first round16(L) bytes): the padded layout
    ss_acceptor_accept writes leaves round16(L)..pitch and everything outside the regions untouched"""
    torch.cuda.synchronize()
    cfg = m.cfg
    u = lambda t: [int(x) for x in t.cpu().numpy().view(np.uint64)]
    w = m.words()
    assert u(acc.window_base) == m.base and u(acc.bal_max_seen) == m.bmax
    assert u(acc.preparing) == w["P"] and u(acc.accepting) == w["A"] and u(acc.committed) == w["C"]
    ib, vb, sa = u(acc.inst_bal), u(acc.voted_bal), u(acc.shard_addr)
    held, dl, vm = (x.cpu().numpy().view(np.uint32) for x in (acc.held, acc.data_len, acc.voted_mask))
    src, span, trig = acc.source.cpu().numpy(), acc.prep_span.cpu().numpy(), u(acc.prep_trigger)
    asg = acc.assignment.cpu().numpy().view(np.uint32) if cfg.cw else None
    rows = acc.assign_rows.cpu().numpy().view(np.uint32) if cfg.cw else None
    st = full.cpu().numpy()
    base_ptr = full.data_ptr()
    written = np.zeros(len(st), dtype=bool)
    for g in range(m.G):
        for s, inst in m.inst[g].items():
            at = g * 64 + (s & 63)
            got = (ib[at], vb[at], int(vm[at]), int(held[at]), int(dl[at]))
            assert got == (inst["bal"], inst["vb"], inst["vm"], inst["held"], inst["dlen"]), (g, s)
            if "src" in inst:
                assert (int(src[at]), int(span[at]), trig[at]) == (inst["src"], inst["span"], inst["trig"]), (g, s)
            if cfg.cw:
                assert int(asg[at]) == inst["asg"], (g, s)
                assert [int(x) for x in rows[at * cfg.n:(at + 1) * cfg.n]] == inst["rows"], (g, s)
            if inst.get("store") is not None:
                o = sa[at] - base_ptr
                assert o == pad + inst["store"], (g, s)
                L, k = inst["L"], 0
                for j in range(cfg.T):
                    if not (inst["held"] >> j) & 1:
                        continue
                    q = o + k * _pitch(L)
                    assert st[q:q + L].tobytes() == inst["shards"][j], (g, s, j)
                    assert not st[q + L:q + _r16(L)].any(), (g, s, j)
                    written[q:q + _r16(L)] = True
                    k += 1
    return written


def _state_equals_live(live, rec):
    """the fields the reference recovers: inst_bal, status words, voted, held, data_len, assignment, assign_rows and the
    shard bytes, equal between the live acceptor and the recovered one"""
    a, b = live.acc, rec
    torch.cuda.synchronize()
    for name in ("preparing", "accepting", "committed", "bal_max_seen", "window_base"):
        assert torch.equal(getattr(a, name), getattr(b, name)), name
    live_words = (a.preparing | a.accepting | a.committed).cpu().numpy().view(np.uint64)
    d = live.cfg.d
    for name in ("inst_bal", "voted_bal", "voted_mask", "held", "data_len") + (("assignment",) if live.cfg.cw else ()):
        x, y = getattr(a, name).cpu().numpy(), getattr(b, name).cpu().numpy()
        for g in range(live.G):
            for p in range(64):
                if (int(live_words[g]) >> p) & 1:
                    assert x[g * 64 + p] == y[g * 64 + p], (name, g, p)
    if live.cfg.cw:
        n = live.cfg.n
        x, y = a.assign_rows.cpu().numpy(), b.assign_rows.cpu().numpy()
        vb = a.voted_bal.cpu().numpy()
        for g in range(live.G):
            for p in range(64):
                at = g * 64 + p
                if (int(live_words[g]) >> p) & 1 and vb[at] != 0:
                    assert (x[at * n:(at + 1) * n] == y[at * n:(at + 1) * n]).all(), (g, p)


def _exec(acc, cap=1 << 22):
    out = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    res = acc.execute(out, 4096, cap)
    n = int(res["totals"][0])
    recs = []
    o = out.cpu().numpy()
    for k in range(n):
        off, ln = int(res["rec_off"][k]), int(res["rec_len"][k])
        recs.append((int(res["rec_group"][k]), int(res["rec_slot"][k]), o[off:off + ln].tobytes()))
    return recs


# ---------------------------------------------------------------------------------------------
# GPU: round trip at every population and code
# ---------------------------------------------------------------------------------------------
def _cases(protocol, n):
    return [(n // 2 + 1, n)] if protocol == "rspaxos" else sorted({(n // 2 + 1, n), (1, min(2 * n, 32)), (min(2 * n, 32),) * 2})


def _drive(live, G, rng):
    """accepts, re-accepts out of Committed, Prepares over committed slots, heartbeats; bases from live"""
    cfg = live.cfg
    base = [int(x) for x in live.acc.window_base.cpu().numpy()]
    lens = (1, 17, 251, 1366)
    full = (1 << cfg.T) - 1
    live.accept([(g, base[g] + s, 1, int(rng.integers(1, 1 << cfg.T)) if g % 2 else full, lens[(g + s) % 4])
                 for g in range(G) for s in range(6)])
    peer = (cfg.me + 1) % cfg.n if cfg.n > 1 else 1
    live.heartbeat([(g, peer, 1, base[g] + 4, 0) for g in range(G)])
    live.accept([(g, base[g] + 1, 2, full, 33) for g in range(0, G, 2)] + [(g, base[g] + 1, 2, 1, 40) for g in range(0, G, 3)])
    live.prepare([(g, peer, base[g] + 2 + g % 2, 3) for g in range(1, G, 2)])
    live.accept([(g, base[g] + 3, 3, full, 9) for g in range(1, G, 4)])
    live.heartbeat([(g, peer, 2, base[g] + 64, 0) for g in range(0, G, 2)])


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 2, 3, 5, 7, 9, 12, 32])
@pytest.mark.parametrize("protocol", ["rspaxos", "crossword"])
def test_recover_round_trip(ctx, protocol, n):
    for d, T in _cases(protocol, n):
        cfg = Cfg(protocol, n, n - 1, d, T)
        G = 6
        rng = np.random.default_rng(n * 131 + d * 7 + T)
        base = [int(rng.integers(0, 1 << 40)) if g % 2 else int(rng.integers(0, 60000)) for g in range(G)]
        live = Live(ctx, cfg, G, base, rng)
        _drive(live, G, rng)
        recs = _nm_some(live.recs, cfg, rng)
        rec = _acceptor(ctx, cfg, G)
        rec.window_base.copy_(_t(np.array(base, dtype=np.uint64)))
        m = RModel(cfg, G)
        m.base = list(base)
        v, store = _recover(ctx, rec, m, recs, rng)
        assert all(x == ACC for x in v)
        _state_equals_live(live, rec)
        assert _exec(live.acc) == _exec(rec)


@pytest.mark.gpu
def test_recover_execution_difference(ctx):
    """stated difference 2: a CommitSlot followed by an AcceptData of the same slot leaves it Accepting and unexecuted
    (the reference executed it at the CommitSlot); a heartbeat commits it again and it executes the later batch"""
    cfg = Cfg("rspaxos", 5, 1, 3, 5)
    rng = np.random.default_rng(5)
    rec = _acceptor(ctx, cfg, 1)
    m = RModel(cfg, 1)
    a1, a2 = _codeword(rng, 30, 3, 5), _codeword(rng, 40, 3, 5)
    recs = [(0, accept_data(cfg, 0, 1, 30, a1[1])), (0, commit_slot(0)), (0, accept_data(cfg, 0, 2, 40, a2[1])),
            (0, accept_data(cfg, 1, 2, 30, a1[1])), (0, commit_slot(1))]
    _recover(ctx, rec, m, recs, rng)
    assert _exec(rec) == []                                        # slot 0 waits; slot 1 is behind it
    rec.heartbeat(_t(np.zeros(1, np.uint32)), _t(np.zeros(1, np.uint8)), _t(np.array([2], np.uint64)), _t(np.array([2], np.uint64)),
                  _t(np.zeros(1, np.uint64)))
    assert _exec(rec) == [(0, 0, a2[0]), (0, 1, a1[0])]


# ---------------------------------------------------------------------------------------------
# GPU: windows, store cut, log ends, grid caps
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("protocol", ["rspaxos", "crossword"])
def test_recover_three_windows(ctx, protocol):
    cfg = Cfg(protocol, 5, 2, 3, 5)
    rng = np.random.default_rng(11)
    G = 3
    recs, unbounded = [], RModel(cfg, G)
    for g in range(G):
        for s in range(0, 180, 1 + g):
            data, sh = _codeword(rng, int(rng.integers(1, 300)), 3, 5)
            held = int(rng.integers(1, 32)) | 0b111
            rows = [int(x) for x in rng.integers(0, 32, 5)]
            recs.append((g, accept_data(cfg, s, 1 + s // 50, len(data), [sh[j] if (held >> j) & 1 else None for j in range(5)], rows)))
            if s % 3 == 0:
                recs.append((g, commit_slot(s)))
            if s % 7 == 0:
                recs.append((g, prepare_bal(s, 2 + s // 50)))
    for g, r in recs:                                              # the restatement without a window
        unbounded.apply_entry(g, parse_record(r, cfg))
    rec = _acceptor(ctx, cfg, G)
    m = RModel(cfg, G)
    pending, stores = recs, []
    for _ in range(4):
        v, store = _recover(ctx, rec, m, pending, rng)
        stores.append(store)
        pending = [x for x, vv in zip(pending, v) if vv == BEYOND]
        if not pending:
            break
        _exec(rec)
        upto = [m.base[g] + 64 if any(gg == g for gg, _ in pending) else m.base[g] for g in range(G)]
        rec.advance(_t(np.array(upto, dtype=np.uint64)))
        m.advance(upto)
    assert not pending and m.base == [128, 128, 128]
    while unbounded.base != m.base:                                # advance retires at most 64 slots a call
        unbounded.advance(m.base)
    for g in range(G):
        assert sorted(m.inst[g]) == sorted(unbounded.inst[g])
        for s, inst in m.inst[g].items():
            want = unbounded.inst[g][s]
            for k in ("st", "bal", "held", "dlen", "vb", "vm", "asg", "rows", "shards"):
                assert inst[k] == want[k], (g, s, k)


@pytest.mark.gpu
def test_recover_store_cut_every_boundary(ctx):
    cfg = Cfg("crossword", 5, 0, 2, 5)
    rng = np.random.default_rng(3)
    G = 5
    recs = []
    for g in range(G):
        for s in range(g + 1):
            data, sh = _codeword(rng, 50 + 40 * g, 2, 5)
            recs.append((g, accept_data(cfg, s, 1, len(data), sh, [31] * 5)))
        recs.append((g, prepare_bal(9, 1)))
    sizes = np.cumsum([0] + [(g + 1) * 5 * _pitch(-(-(50 + 40 * g) // 2)) for g in range(G)])
    for cut in sorted({int(x) for x in sizes} | {int(x) - 1 for x in sizes[1:]}):
        rec = _acceptor(ctx, cfg, G)
        m = RModel(cfg, G)
        v, _ = _recover(ctx, rec, m, recs, rng, cap=cut)
        left = [x for x, vv in zip(recs, v) if vv == STORE_FULL_V]
        placed = {g for (g, _), vv in zip(recs, v) if vv == ACC}
        assert placed == set(range(int(np.searchsorted(sizes, cut, side="right")) - 1))
        if left:                                                   # drain
            v2, _ = _recover(ctx, rec, m, left, rng)
            assert all(x == ACC for x in v2)
        assert m.words()["A"] == [(1 << (g + 1)) - 1 for g in range(G)]


@pytest.mark.gpu
def test_recover_log_ends(ctx):
    cfg = Cfg("rspaxos", 5, 1, 3, 5)
    rng = np.random.default_rng(4)
    G = 3
    data, sh = _codeword(rng, 20, 3, 5)
    good = lambda s: accept_data(cfg, s, 1, 20, sh)
    recs = [(0, good(0)), (1, good(0)), (1, _frame(_var(9) + _var(1))), (1, good(1)), (1, commit_slot(0)), (0, good(1)),
            (7, good(2)), (2, prepare_bal(3, 4)), (2, _frame(_var(COMMIT_V) + _var(3) + b"\0")), (2, commit_slot(3))]
    rec = _acceptor(ctx, cfg, G)
    m = RModel(cfg, G)
    v, _ = _recover(ctx, rec, m, recs, rng)
    assert v == [ACC, ACC, MALFORMED, AFTER_END, AFTER_END, ACC, MALFORMED, ACC, MALFORMED, AFTER_END]
    # a truncated last record: its length runs past the buffer
    last = good(5)
    trunc = (int.from_bytes(last[:8], "big") + 1000).to_bytes(8, "big") + last[8:]
    v, _ = _recover(ctx, rec, m, [(0, good(4)), (0, trunc)], rng)
    assert v == [ACC, MALFORMED]


def _warp_cap(ctx):
    return ctx.sm_count * 64 * 8        # launch_grid: 64 CTAs per SM, 8 warps per CTA: recover_copy_kernel


def _thread_cap(ctx):
    return ctx.sm_count * 64 * 256      # a thread per record or segment: header, walk and apply


@pytest.mark.gpu
def test_recover_one_group_20k_records(ctx):
    cfg = Cfg("rspaxos", 3, 0, 2, 3)
    rng = np.random.default_rng(8)
    data, sh = _codeword(rng, 7, 2, 3)
    recs = []
    for k in range(20000):
        s = k % 64
        recs.append((0, [accept_data(cfg, s, 1 + k // 64, 7, sh), prepare_bal(s, 1 + k // 64), commit_slot(s)][k % 3]))
    rec = _acceptor(ctx, cfg, 1)
    m = RModel(cfg, 1)
    _recover(ctx, rec, m, recs, rng)


@pytest.mark.gpu
def test_recover_past_the_grid_caps(ctx):
    """more groups with a defining AcceptData than the copy kernel has warps, behind more records of a group past
    n_groups than the per-record and per-segment kernels have threads; checked without the per-record restatement"""
    cfg = Cfg("rspaxos", 3, 0, 2, 3)
    rng = np.random.default_rng(9)
    G, X = _warp_cap(ctx) + 1000, _thread_cap(ctx) + 1000
    data, sh = _codeword(rng, 5, 2, 3)
    ad, cs = accept_data(cfg, 1, 3, 5, sh), commit_slot(0)
    assert len(ad) < 48 and len(cs) < 16
    n = G + G // 2 + X
    groups = np.concatenate([np.arange(G), np.arange(0, G, 2), np.full(X, G + 5)]).astype(np.uint32)
    offs = np.concatenate([1 + 48 * np.arange(G), 1 + 48 * G + 16 * np.arange(G // 2 + X)]).astype(np.uint64)
    buf = np.zeros(48 * G + 16 * (G // 2 + X) + 16, dtype=np.uint8)
    buf[offs[:G, None].astype(np.int64) + np.arange(len(ad))] = np.frombuffer(ad, np.uint8)
    buf[offs[G:, None].astype(np.int64) + np.arange(len(cs))] = np.frombuffer(cs, np.uint8)
    rec = _acceptor(ctx, cfg, G)
    total = G * 3 * 32
    full = torch.full((total + 128,), 0xA5, dtype=torch.uint8, device="cuda")
    res = rec.recover(_t(buf), _t(offs), _t(groups), full[64:64 + total])
    v = res["verdict"].cpu().numpy().view(np.uint32)
    assert (v[:G + G // 2] == ACC).all() and (v[G + G // 2:] == MALFORMED).all() and int(res["total"][0]) == total
    assert ctx.device_status() == 0
    u, c = rec.accepting.cpu().numpy().view(np.uint64), rec.committed.cpu().numpy().view(np.uint64)
    assert (u[1::2] == 2).all() and (u[0::2] == 2).all() and (c[0::2] == 1).all() and (c[1::2] == 0).all()
    addr = rec.shard_addr.view(G, 64)[:, 1].cpu().numpy().view(np.uint64) - np.uint64(full.data_ptr() + 64)
    assert (addr == np.arange(G, dtype=np.uint64) * np.uint64(96)).all()
    st = full.cpu().numpy()
    assert (st[:64] == 0xA5).all() and (st[64 + total:] == 0xA5).all()          # the pads around the store
    want = np.full((3, 32), 0xA5, np.uint8)                                     # L = 3: bytes 3..16 zero, 16..32 untouched
    for j in range(3):
        want[j, :16] = 0
        want[j, :3] = np.frombuffer(sh[j], np.uint8)
    assert (st[64:64 + total].reshape(G, 3, 32) == want).all()


@pytest.mark.gpu
def test_recover_resubmitted_window_resets_retired_positions(ctx):
    """a re-submitted window whose first record for a retired position is a CommitSlot or a PrepareBal: the position
    starts as a fresh null_instance(), so the retired instance's ballot, shards, vote and assignment do not leak, and a
    committed null instance does not execute the retired instance's batch"""
    cfg = Cfg("crossword", 5, 2, 3, 5)
    rng = np.random.default_rng(21)
    G = 2
    rec = _acceptor(ctx, cfg, G)
    m = RModel(cfg, G)
    first, stores = [], []
    for g in range(G):
        for s in range(64):
            data, sh = _codeword(rng, 40 + s, 3, 5)
            first.append((g, accept_data(cfg, s, 3, len(data), sh, [31] * 5)))
            first.append((g, commit_slot(s)))
    v, store = _recover(ctx, rec, m, first, rng)
    stores.append(store)
    assert all(x == ACC for x in v) and len(_exec(rec)) == 2 * 64
    rec.advance(_t(np.array([64, 64], dtype=np.uint64)))
    m.advance([64, 64])
    data, sh = _codeword(rng, 30, 3, 5)
    second = [(0, commit_slot(64 + k) if k % 2 == 0 else prepare_bal(64 + k, 5)) for k in range(64)]
    second += [(1, commit_slot(64)), (1, prepare_bal(65, 5)), (1, accept_data(cfg, 65, 5, 30, sh, [7] * 5)), (1, commit_slot(65))]
    v, store = _recover(ctx, rec, m, second, rng)
    stores.append(store)
    assert all(x == ACC for x in v)
    assert m.inst[0][64]["held"] == 0 and m.inst[0][65]["bal"] == 5 and m.inst[1][65]["vb"] == 5
    assert _exec(rec) == []                                        # slot 64 of both groups: committed, no shards


@pytest.mark.gpu
def test_recover_argument_refusals_and_empty_batch(ctx):
    cfg = Cfg("rspaxos", 5, 1, 3, 5)                               # AcceptData is variant 1
    acc = _acceptor(ctx, cfg, 2)
    dev = "cuda"
    rec = commit_slot(0)
    buf = torch.zeros(64, dtype=torch.uint8, device=dev)
    buf[:len(rec)] = torch.tensor(list(rec), dtype=torch.uint8)
    off, grp = torch.zeros(1, dtype=torch.int64, device=dev), torch.zeros(1, dtype=torch.int32, device=dev)
    store = torch.zeros(64, dtype=torch.uint8, device=dev)
    verdict = torch.full((1,), 7, dtype=torch.int32, device=dev)
    total = torch.full((1,), 7, dtype=torch.int64, device=dev)
    p = lambda x: x.data_ptr()

    def call(pv=0, cv=2, n=1, b=p(buf), o=p(off), g=p(grp), s=p(store), v=p(verdict), t=p(total)):
        return acc.lib.ss_acceptor_recover(acc.h, b, 64, o, g, n, pv, cv, s, 64, v, t)

    bad = _lib.SS_ERR_INVALID_ARG
    assert call(pv=1) == bad and call(cv=1) == bad and call(pv=2) == bad            # the three variants must differ
    for k in ("b", "o", "g", "s", "v"):
        assert call(**{k: None}) == bad, k
    assert call(s=p(store) + 8) == bad                                             # store not 16-byte aligned
    assert call(n=1 << 31) == bad
    torch.cuda.synchronize()
    assert int(verdict[0]) == 7 and int(total[0]) == 7 and ctx.device_status() == 0   # nothing ran
    assert call(n=0) == _lib.SS_OK and int(total[0]) == 0                          # an empty batch: *total = 0
    assert acc.lib.ss_acceptor_recover(acc.h, None, 0, None, None, 0, 0, 2, None, 0, None, None) == _lib.SS_OK
    assert call(t=None) == _lib.SS_OK and int(verdict[0]) == ACC - (1 << 32)       # total may be NULL
    assert int(acc.committed[0]) == 1 and ctx.device_status() == 0
