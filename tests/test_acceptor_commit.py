"""Commit and execute on the device acceptor (ss_acceptor_heartbeat / ss_acceptor_execute, summerset_b200/csrc/acceptor.cu).

`Model` restates, per message and over the acceptor's 64-slot window rule:
  * handle_msg_accept's effect on the instance (rspaxos/messages.rs:329-392): a well-formed Accept inside the window at a
    ballot >= bal_max_seen makes the slot Accepting with the frame's shards, also when it was Committed;
  * the commit half of heard_heartbeat (rspaxos/leadership.rs:222-311, crossword/leadership.rs:260-359);
  * handle_logged_commit_slot (rspaxos/durability.rs:125-186, crossword/durability.rs:142-206), called for each newly
    committed slot in ascending order once the CommitSlot records are durable (here: at the execute call); it walks only
    when the slot is the commit_bar.  The device walks every group on every call; a walk stopped by the call's capacity
    or by a null codeword is retried by the next call, which the model keeps as a pending slot.
Payloads are checked against the request batches the shards were cut from and against the oracle's
rs_reconstruct(data_only) on the held shards.
"""
import copy
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import pyoracle
from summerset_b200 import _lib
from tests.test_acceptor import ACC, _buffer, _t

EXEC_FULL, EXEC_NULL = _lib.SS_DEV_STATUS_EXEC_FULL, _lib.SS_DEV_STATUS_EXEC_NULL
U64 = (1 << 64) - 1
LENS_L = [1, 15, 16, 17, 250, 251, 1366, 21846, 65536]


def _r16(x):
    return (x + 15) // 16 * 16


def _pitch(L):
    return (L + 31) // 32 * 32


class Model:
    def __init__(self, G, n, me, d, T):
        self.G, self.n, self.me, self.d, self.T = G, n, me, d, T
        self.base, self.bmax, self.cb, self.eb = [0] * G, [0] * G, [0] * G, [0] * G
        self.inst = [dict() for _ in range(G)]       # slot -> dict(bal, held, dlen, shards, st "A" / "C")
        self.pending = [set() for _ in range(G)]     # committed slots whose CommitSlot record is not yet handled

    def accept(self, g, slot, bal, held, dlen, shards):
        """one well-formed Accept -> accepted?"""
        if g >= self.G or slot < self.base[g] or slot >= self.base[g] + 64 or bal < self.bmax[g]:
            return False
        self.bmax[g] = bal
        self.inst[g][slot] = dict(bal=bal, held=held, dlen=dlen, shards=shards, st="A")
        return True

    def heartbeat(self, recs):
        """recs: (group, peer, ballot, commit_bar, exec_bar) in record order -> newly words (window order)"""
        newly = [0] * self.G
        start = [max(c, b) for c, b in zip(self.cb, self.base)]
        for g, peer, bal, hcb, heb in recs:
            if g >= self.G:
                continue
            if peer != self.me and bal > self.bmax[g]:          # check_leader
                self.bmax[g] = bal
            if bal < self.bmax[g] or heb < self.eb[g]:
                continue
            for s in range(start[g], min(hcb, self.base[g] + 64)):
                inst = self.inst[g].get(s)
                if inst is None or inst["bal"] < bal:
                    break
                if inst["st"] == "C":
                    continue
                inst["st"] = "C"
                newly[g] |= 1 << (s - self.base[g])
                self.pending[g].add(s)
        return newly

    def advance(self, upto):
        for g, u in enumerate(upto):
            k = min(max(u - self.base[g], 0), 64)
            for s in [s for s in self.inst[g] if s < self.base[g] + k]:
                del self.inst[g][s]
            self.base[g] += k

    def execute(self, out_cap, rec_cap):
        """-> (records [(g, slot, off, dlen)], totals, status bits)"""
        walks = []
        for g in range(self.G):
            cbe = max(self.cb[g], self.base[g])
            trig = cbe in self.pending[g]
            self.pending[g] = set()
            run, null = [], False
            s = cbe
            while trig and s < self.base[g] + 64:
                inst = self.inst[g].get(s)
                if inst is None or inst["st"] != "C" or bin(inst["held"]).count("1") < self.d:
                    break                                         # not committed, or postponed
                if inst["dlen"] == 0:
                    null = True
                    break
                run.append(s)
                s += 1
            walks.append((run, null, s))
        totals = [sum(len(w[0]) for w in walks), sum(_r16(self.inst[g][s]["dlen"]) for g, w in enumerate(walks) for s in w[0])]
        recs, status, ro, bo = [], 0, 0, 0
        for g, (run, null, stop) in enumerate(walks):
            full = False
            for s in run:
                sz = _r16(self.inst[g][s]["dlen"])
                if full or ro >= rec_cap or bo + sz > out_cap:
                    if not full:
                        self.pending[g].add(s)
                    full = True
                else:
                    recs.append((g, s, bo, self.inst[g][s]["dlen"]))
                    self.cb[g] = s + 1
                ro += 1
                bo += sz
            if full:
                status |= EXEC_FULL
            elif null:
                status |= EXEC_NULL
                self.pending[g].add(stop)
        return recs, totals, status

    def payload(self, g, s):
        """get_data's bytes, with reconstruct_data by the oracle when a data shard is not held"""
        inst = self.inst[g][s]
        sh = [None if x is None else np.frombuffer(x, dtype=np.uint8).copy() for x in inst["shards"]]
        if any(sh[j] is None for j in range(self.d)):
            assert pyoracle.rs_reconstruct(self.d, self.T - self.d, sh, True) == 0
        return b"".join(sh[j].tobytes() for j in range(self.d))[:inst["dlen"]]

    def words(self):
        acc, com = [0] * self.G, [0] * self.G
        for g in range(self.G):
            for s, inst in self.inst[g].items():
                if inst["st"] == "A":
                    acc[g] |= 1 << (s & 63)
                else:
                    com[g] |= 1 << (s & 63)
        return acc, com


# ---------------------------------------------------------------------------------------------
# CPU: the model on hand-written cases, symbols and refusals
# ---------------------------------------------------------------------------------------------
def _inst(m, g, s, bal, held=0b111, dlen=10):
    assert m.accept(g, s, bal, held, dlen, None)


def test_model_heartbeat_rules():
    m = Model(2, 5, 1, 3, 5)
    for s in range(6):
        _inst(m, 0, s, 5)
    m.inst[0][2]["bal"] = 4                              # a slot accepted at a lower ballot: the walk breaks there
    assert m.heartbeat([(0, 1, 9, 10, 0)]) == [0, 0] and m.bmax[0] == 5         # peer == me raises nothing; 9 >= 5
    assert m.heartbeat([(0, 0, 5, 10, 0)]) == [0b11, 0]                          # 9 not seen: bal 5 commits 0, 1
    assert m.heartbeat([(0, 2, 7, 10, 0), (0, 0, 5, 10, 0)]) == [0, 0] and m.bmax[0] == 7   # the second record is stale
    m.inst[0][2]["bal"] = 7
    for s in range(6):
        m.inst[0][s]["bal"] = 7
    m.eb[0] = 3
    assert m.heartbeat([(0, 2, 7, 10, 2)]) == [0, 0]                            # exec_bar behind ours
    assert m.heartbeat([(0, 2, 7, 4, 3)]) == [0b1100, 0]                        # continue past 0, 1; stop at 4
    assert m.heartbeat([(0, 2, 7, 10, 3)]) == [0b110000, 0]                     # then the Null slot 6 breaks
    assert m.heartbeat([(5, 2, 99, 10, 3)]) == [0, 0]                           # group >= G
    recs, tot, st = m.execute(1 << 20, 100)
    assert [r[1] for r in recs] == list(range(6)) and tot == [6, 96] and st == 0 and m.cb[0] == 6


def test_model_execute_stops():
    m = Model(3, 5, 1, 3, 5)
    _inst(m, 0, 0, 1, held=0b11)                        # two shards: postponed
    _inst(m, 0, 1, 1)
    _inst(m, 1, 0, 1, dlen=0)                           # a null codeword
    _inst(m, 2, 0, 1, dlen=20)
    _inst(m, 2, 1, 1, dlen=20)
    m.heartbeat([(g, 0, 1, 2, 0) for g in range(3)])
    recs, tot, st = m.execute(1 << 20, 100)
    assert recs == [(2, 0, 0, 20), (2, 1, 32, 20)] and tot == [2, 64] and st == EXEC_NULL and m.cb == [0, 0, 2]
    # the null codeword is reported again by the next call, the postponed instance stays
    recs, tot, st = m.execute(1 << 20, 100)
    assert recs == [] and st == EXEC_NULL
    # capacity: exactly one region fits
    m = Model(1, 5, 1, 3, 5)
    _inst(m, 0, 0, 1, dlen=20)
    _inst(m, 0, 1, 1, dlen=20)
    m.heartbeat([(0, 0, 1, 2, 0)])
    assert m.execute(32, 100) == ([(0, 0, 0, 20)], [2, 64], EXEC_FULL)
    assert m.execute(32, 100) == ([(0, 1, 0, 20)], [1, 32], 0)


def test_model_reaccept_and_window():
    m = Model(1, 5, 1, 3, 5)
    for s in range(64):
        _inst(m, 0, s, 1, dlen=1)
    m.heartbeat([(0, 0, 1, 100, 0)])
    assert m.words()[1] == [U64]
    assert m.accept(0, 3, 2, 0b111, 1, None)           # a committed slot re-accepted is Accepting again
    assert m.words()[0] == [1 << 3]
    recs, _, _ = m.execute(1 << 20, 1000)
    assert len(recs) == 3 and m.cb[0] == 3
    m.advance([40])
    _inst(m, 0, 64, 2)
    assert m.base[0] == 40 and m.heartbeat([(0, 0, 2, 70, 0)]) == [0]   # slot 3 was retired; start = base = 40, inst_bal 1 < 2


def test_acceptor_commit_symbols_and_refusals():
    lib = _lib.load()
    for name in ("ss_acceptor_commit_view_get", "ss_acceptor_heartbeat", "ss_acceptor_execute"):
        assert hasattr(lib, name)
    assert lib.ss_version() == 200
    v = _lib.AcceptorCommitView()
    assert lib.ss_acceptor_commit_view_get(None, C.byref(v)) == _lib.SS_ERR_INVALID_ARG
    assert lib.ss_acceptor_heartbeat(None, None, None, None, None, None, 0, None) == _lib.SS_ERR_INVALID_ARG
    assert lib.ss_acceptor_execute(None, None, 0, None, None, None, None, 0, None) == _lib.SS_ERR_INVALID_ARG
    assert C.sizeof(_lib.AcceptorCommitView) == 32


# ---------------------------------------------------------------------------------------------
# GPU helpers
# ---------------------------------------------------------------------------------------------
def _codeword(rng, dlen, d, T):
    """a request batch of dlen random bytes cut into d data shards, plus T - d parity shards"""
    data = rng.integers(0, 256, dlen, dtype=np.uint8).tobytes()
    if dlen == 0:
        return data, [b""] * T
    sh = pyoracle.cw_split(data, d)
    L = sh.shape[1]
    full = [np.ascontiguousarray(sh[j]) for j in range(d)] + [np.zeros(L, np.uint8) for _ in range(T - d)]
    if T > d:
        assert pyoracle.rs_encode(d, T - d, full) == 0
    return data, [x.tobytes() for x in full]


class Rig:
    """one device acceptor and its model; keeps every store alive, since execute reads the shards in place"""

    def __init__(self, ctx, protocol, G, n, me, d, T):
        from summerset_b200.engine import Acceptor
        self.ctx, self.cw = ctx, protocol == "crossword"
        self.acc = Acceptor(ctx, protocol, G, n, me, d, T)
        self.m = Model(G, n, me, d, T)
        self.stores = []
        self.rng = np.random.default_rng(G * 31 + n * 7 + d + T)
        self.data = {}                                        # (g, slot) -> request batch of the accepted instance

    def set_base(self, base):
        self.m.base = list(base)
        self.acc.window_base.copy_(_t(np.array(base, dtype=np.uint64)))

    def accept(self, items):
        """items: (g, slot, ballot, held, data, shards) with shards cut from data"""
        d, T = self.m.d, self.m.T
        frames, groups = [], []
        for g, s, bal, held, data, shards in items:
            sh = [shards[j] if (held >> j) & 1 else None for j in range(T)]
            frames.append(pyoracle.frame_accept(2, s, bal, d, T - d, len(data), sh, [held] * self.m.n if self.cw else None, T))
            groups.append(g)
        buf, offs = _buffer(self.rng, frames)
        L = [-(-len(it[4]) // d) for it in items]
        store = torch.empty(sum(bin(it[3]).count("1") * _pitch(l) for it, l in zip(items, L)) + 64, dtype=torch.uint8, device="cuda")
        wal = torch.empty(sum(len(f) + 48 for f in frames) + 64, dtype=torch.uint8, device="cuda")
        self.stores.append(store)
        out = self.acc.accept(_t(buf), _t(offs), _t(np.array(groups, dtype=np.uint32)), _t(np.zeros(len(items), np.uint8)), store, wal)
        want = []
        for g, s, bal, held, data, shards in items:
            ok = self.m.accept(g, s, bal, held, len(data), [shards[j] if (held >> j) & 1 else None for j in range(T)])
            want.append(ACC if ok else None)
            if ok:
                self.data[(g, s)] = data
        v = out["verdict"].cpu().numpy().view(np.uint32)
        for i, w in enumerate(want):
            assert (int(v[i]) == ACC) == (w == ACC), i
        assert self.ctx.device_status() == 0

    def heartbeat(self, recs):
        cols = list(zip(*recs)) if recs else [[]] * 5
        newly = self.acc.heartbeat(_t(np.array(cols[0], dtype=np.uint32)), _t(np.array(cols[1], dtype=np.uint8)),
                                   _t(np.array(cols[2], dtype=np.uint64)), _t(np.array(cols[3], dtype=np.uint64)),
                                   _t(np.array(cols[4], dtype=np.uint64)))
        want = self.m.heartbeat(recs)
        assert [int(x) for x in newly.cpu().numpy().view(np.uint64)] == want
        self.check_state()
        return newly

    def execute(self, out_cap=None, rec_cap=None, check_data=True):
        m = self.m
        _, tot, _ = copy.deepcopy(m).execute(1 << 62, 1 << 62)     # the walk without capacities sizes the buffers
        oc = tot[1] if out_cap is None else out_cap
        rc = tot[0] if rec_cap is None else rec_cap
        canary = self.rng.integers(0, 256, oc + 64, dtype=np.uint8)
        out = _t(canary.copy())
        res = self.acc.execute(out, max(rc, 1), oc)
        recs, totals, status = m.execute(oc, rc)
        assert self.ctx.device_status() == status
        got = {k: v.cpu().numpy() for k, v in res.items()}
        assert [int(x) for x in got["totals"]] == totals
        n = len(recs)
        assert [int(x) for x in got["rec_group"][:n]] == [r[0] for r in recs]
        assert [int(x) for x in got["rec_slot"][:n].view(np.uint64)] == [r[1] for r in recs]
        assert [int(x) for x in got["rec_off"][:n]] == [r[2] for r in recs]
        assert [int(x) for x in got["rec_len"][:n]] == [r[3] for r in recs]
        want = canary.copy()
        for g, s, off, dl in recs:
            p = m.payload(g, s)
            if check_data:
                assert p == self.data[(g, s)], (g, s)
            want[off:off + _r16(dl)] = 0
            want[off:off + dl] = np.frombuffer(p, dtype=np.uint8)
        gotb = out.cpu().numpy()
        if not np.array_equal(gotb, want):
            bad = np.nonzero(gotb != want)[0]
            pytest.fail(f"payload: {len(bad)} bytes differ, first at {bad[0]}")
        self.check_state()
        return recs, status

    def check_state(self):
        torch.cuda.synchronize()
        a, m = self.acc, self.m
        u = lambda t: [int(x) for x in t.cpu().numpy().view(np.uint64)]
        acc, com = m.words()
        assert u(a.window_base) == m.base
        assert u(a.bal_max_seen) == m.bmax
        assert u(a.accepting) == acc
        assert u(a.committed) == com
        assert u(a.commit_bar) == m.cb
        assert u(a.exec_bar) == m.eb

    def commit_all(self):
        """one heartbeat per group at each group's instance ballot, covering the whole window"""
        recs = []
        for g in range(self.m.G):
            if self.m.inst[g]:
                bal = max(i["bal"] for i in self.m.inst[g].values())
                recs.append((g, (self.m.me + 1) % self.m.n if self.m.n > 1 else 0, bal, self.m.base[g] + 64, 0))
        return self.heartbeat(recs)


def _masks(T, d):
    return [h for h in range(1, 1 << T) if bin(h).count("1") >= d]


# ---------------------------------------------------------------------------------------------
# GPU 1: codes and erasures
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("T", range(1, 9))
def test_execute_every_mask_small_codes(ctx, T):
    """every held mask with >= d shards, every d <= T, shard lengths around 16 and the varint edges"""
    for d in range(1, T + 1):
        masks = _masks(T, d)
        G = len(masks)
        rig = Rig(ctx, "crossword", G, T, 0, d, T)
        rng = rig.rng
        rig.set_base([int(x) for x in rng.integers(0, 1 << 40, G)])
        items = []
        for g, h in enumerate(masks):
            L = LENS_L[(g + d) % 6]
            dlen = max(1, L * d - int(rng.integers(0, d))) if d > 1 else L
            data, sh = _codeword(rng, dlen, d, T)
            items.append((g, rig.m.base[g], 1 + g % 3, h, data, sh))
        rig.accept(items)
        rig.commit_all()
        recs, st = rig.execute()
        assert len(recs) == G and st == 0


@pytest.mark.gpu
@pytest.mark.parametrize("d", [1, 16, 31, 32])
def test_execute_t32(ctx, d):
    T = 32
    rig = Rig(ctx, "crossword", 40, 32, 5, d, T)
    rng = rig.rng
    masks = [(1 << T) - 1] + [int(h) for h in rng.integers(1, 1 << 32, 400, dtype=np.uint64) if bin(int(h)).count("1") >= d][:30]
    while len(masks) < 40:                              # d near T: masks with one or no shard missing
        drop = [int(x) for x in rng.choice(T, T - d, replace=False)] if T > d else []
        masks.append((1 << T) - 1 - sum(1 << j for j in drop))
    items = []
    for g, h in enumerate(masks):
        L = LENS_L[g % len(LENS_L)]
        dlen = max(1, L * d - int(rng.integers(0, d)))
        data, sh = _codeword(rng, dlen, d, T)
        items.append((g, 0, 1, h, data, sh))
    rig.accept(items)
    rig.commit_all()
    recs, st = rig.execute()
    assert len(recs) == 40 and st == 0


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 3, 5])
def test_rspaxos_one_shard(ctx, n):
    """an RSPaxos follower holds its own shard: execution is postponed unless d = 1"""
    d = n // 2 + 1
    me = n - 1
    rig = Rig(ctx, "rspaxos", 6, n, me, d, n)
    rng = rig.rng
    items = []
    for g in range(6):
        data, sh = _codeword(rng, 1 + 97 * g, d, n)
        items.append((g, 0, 3, 1 << me, data, sh))
    rig.accept(items)
    rig.commit_all()
    recs, st = rig.execute()
    assert st == 0 and len(recs) == (6 if d == 1 else 0)
    assert rig.m.words()[1] == [1] * 6


@pytest.mark.gpu
@pytest.mark.parametrize("me,missing", [(0, 0), (1, 1), (3, 2)])
def test_crossword_balanced_and_unbalanced(ctx, me, missing):
    """n = 5, T = 5, d = 3: spr = 3 rows put 0, 1 or 2 data shards outside `me`'s row; unbalanced rows beside them"""
    n, T, d = 5, 5, 3
    row = int(pyoracle.cw_brr_assignment(n, T, 3)[me])
    assert sum(1 for j in range(d) if not (row >> j) & 1) == missing
    unbalanced = [0b11100, 0b10011, 0b01110, 0b11111, 0b01011]
    G = 24
    rig = Rig(ctx, "crossword", G, n, me, d, T)
    rng = rig.rng
    items = []
    for g in range(G):
        dlen = int(rng.choice([1, 2, 250, 251, 752, 4096, 65536, 65537]))
        data, sh = _codeword(rng, dlen, d, T)
        items.append((g, 0, 2, row if g % 2 == 0 else unbalanced[g % 5], data, sh))
    rig.accept(items)
    rig.commit_all()
    recs, st = rig.execute()
    assert len(recs) == G and st == 0


@pytest.mark.gpu
@pytest.mark.parametrize("n", range(1, 33))
def test_execute_populations(ctx, n):
    """populations 1..32 at T = n and T = 2n (up to 32), me at n - 1, rows of spr = d"""
    for T in sorted({n, min(2 * n, 32)}):
        d = n // 2 + 1 if T == n else min(T, n)
        rig = Rig(ctx, "crossword", 8, n, n - 1, d, T)
        rng = rig.rng
        rows = pyoracle.cw_brr_assignment(n, T, d)
        items = []
        for g in range(8):
            h = int(rows[n - 1]) if g < 4 else int(rng.integers(1, 1 << T))
            if bin(h).count("1") < d:
                h = (1 << T) - 1
            dlen = int(rng.choice([1, 17, 251, 1366, 5000]))
            data, sh = _codeword(rng, dlen, d, T)
            items.append((g, 0, 1, h, data, sh))
        rig.accept(items)
        rig.commit_all()
        recs, st = rig.execute()
        assert len(recs) == 8 and st == 0


# ---------------------------------------------------------------------------------------------
# GPU 2: heartbeat edges, windows, re-accepts, many groups
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_heartbeat_edges(ctx):
    n, T, d = 5, 5, 3
    rig = Rig(ctx, "crossword", 4, n, 1, d, T)
    rng = rig.rng
    cw = lambda: _codeword(rng, int(rng.integers(1, 300)), d, T)
    items = []
    for s in range(64):
        data, sh = cw()
        items.append((0, s, 5 if s != 10 else 4, 0b11111, data, sh))
    for s in (0, 1, 3):                                     # group 1: a Null slot at 2
        data, sh = cw()
        items.append((1, s, 5, 0b00111, data, sh))
    rig.accept(items)
    rig.heartbeat([(0, 1, 9, 100, 0), (1, 0, 5, 100, 0)])   # peer == me raises nothing; group 1 stops at the Null slot
    rig.heartbeat([(0, 2, 8, 100, 0), (0, 0, 5, 100, 0)])  # check_leader raises to 8: the second record is stale
    rig.heartbeat([(0, 2, 8, 5, 0), (0, 2, 4, 100, 0), (7, 0, 99, 100, 0)])   # nothing at ballot 8 yet; group >= G
    rig.accept([(0, s, 8, 0b11111) + cw() for s in range(12)])  # re-accepts at 8; slot 10 had ballot 4
    rig.heartbeat([(0, 2, 8, 5, 0)])
    rig.heartbeat([(0, 2, 8, 11, 0)])                       # continue past 0..4, commit 5..10
    rig.execute()
    rig.m.eb[0] = rig.m.cb[0]
    rig.acc.exec_bar.copy_(_t(np.array(rig.m.eb, dtype=np.uint64)))
    rig.heartbeat([(0, 2, 8, 100, rig.m.eb[0] - 1)])        # exec_bar behind ours: skipped
    rig.accept([(0, s, 8, 0b11111) + cw() for s in range(12, 64)])
    rig.heartbeat([(0, 2, 8, 1000, rig.m.eb[0])])           # stops at the window end
    rig.accept([(0, 3, 9, 0b11111) + cw()])                 # a committed, executed slot re-accepted: Accepting again
    rig.execute()
    upto = [40, 2, 0, 0]
    rig.acc.advance(_t(np.array(upto, dtype=np.uint64)))
    rig.m.advance(upto)
    rig.check_state()
    rig.accept([(0, s, 9, 0b01011) + cw() for s in range(64, 104)])
    rig.heartbeat([(0, 2, 9, 1000, rig.m.eb[0])])           # the rest, after advance
    rig.execute()
    # a host-installed window base above commit_bar
    rig.set_base([rig.m.base[0], rig.m.base[1], 500, 0])
    rig.accept([(2, 500 + s, 3, 0b10101) + cw() for s in range(5)])
    rig.heartbeat([(2, 0, 3, 503, 0)])
    recs, _ = rig.execute()
    assert [r[1] for r in recs if r[0] == 2] == [500, 501, 502] and rig.m.cb[2] == 503


@pytest.mark.gpu
def test_heartbeat_many_groups_and_records(ctx):
    """interleaved heartbeats of many groups in one call, scratch regrown across calls, > 65536 records in one group"""
    n, T, d = 5, 10, 6
    G = 37
    rig = Rig(ctx, "crossword", G, n, 2, d, T)
    rng = rig.rng
    rig.set_base([int(x) for x in rng.integers(0, 1 << 33, G)])
    for rnd, nrec in enumerate([10, 300, 3000, 70000]):
        items = []
        for _ in range(150):
            g = int(rng.integers(0, G))
            s = rig.m.base[g] + int(rng.integers(0, 70))
            held = int(rng.integers(1, 1 << T))
            data, sh = _codeword(rng, int(rng.integers(1, 400)), d, T)
            items.append((g, s, int(rng.integers(1, 6)) + rnd, held, data, sh))
        rig.accept(items)
        recs = []
        for _ in range(nrec):
            g = 0 if nrec == 70000 else int(rng.integers(0, G + 1))
            base = rig.m.base[g] if g < G else 0
            recs.append((g, int(rng.integers(0, n)), int(rng.integers(0, 8)) + rnd, base + int(rng.integers(0, 70)), int(rng.integers(0, 3))))
        rig.heartbeat(recs)
        rig.execute()
        upto = [b + int(rng.integers(0, 30)) for b in rig.m.base]
        rig.acc.advance(_t(np.array(upto, dtype=np.uint64)))
        rig.m.advance(upto)
        rig.check_state()


# ---------------------------------------------------------------------------------------------
# GPU 3: capacities
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("which", ["out", "rec"])
def test_execute_capacity(ctx, which):
    G = 30
    for short in (0, 1):
        rig = Rig(ctx, "crossword", G, 5, 3, 3, 5)
        rng = rig.rng
        items = []
        for g in range(G):
            for s in range(3):
                data, sh = _codeword(rng, int(rng.integers(1, 3000)), 3, 5)
                items.append((g, s, 1, 0b11001, data, sh))
        rig.accept(items)
        rig.commit_all()
        k = 40                                               # records 0..k-1 fit exactly
        lens = [len(rig.data[(g, s)]) for g in range(G) for s in range(3)]
        edge = sum(_r16(x) for x in lens[:k])
        if which == "out":
            recs, st = rig.execute(out_cap=edge - short, rec_cap=1000)
        else:
            recs, st = rig.execute(out_cap=1 << 24, rec_cap=k - short)
        assert st == EXEC_FULL and len(recs) == k - short
        calls = 0
        while rig.m.cb != [3] * G:                          # drain
            rig.execute(out_cap=edge, rec_cap=k)
            calls += 1
        assert calls >= 2


# ---------------------------------------------------------------------------------------------
# GPU 4: closed loop -- leader proposal -> Accept frames -> acceptor -> heartbeat -> CommitSlot -> execute
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("protocol,n,T,d,me", [("crossword", 5, 5, 3, 0), ("crossword", 5, 5, 3, 1), ("crossword", 5, 5, 3, 3),
                                               ("crossword", 7, 14, 7, 4), ("rspaxos", 5, 5, 3, 1)])
def test_closed_loop(ctx, oracle, protocol, n, T, d, me):
    from summerset_b200 import workloads as wl
    from summerset_b200.engine import Acceptor, LeaderEngine
    cw = protocol == "crossword"
    G = 64
    rng = np.random.default_rng(n * 10 + me)
    eng = LeaderEngine(ctx, protocol, G, n, 0 if n == 1 else 1, 1, **(dict(rs_total_shards=T, rs_data_shards=d) if cw else {}))
    d, p, T = eng.d, eng.T - eng.d, eng.T
    bal = rng.integers(1, 1 << 30, G).astype(np.uint64)
    eng.set_prepared_ballots(_t(bal))
    if cw:
        policies = np.array([oracle.cw_brr_assignment(n, T, d)], dtype=np.uint32)
        eng.set_policies([list(map(int, q)) for q in policies], True)
    else:
        policies = np.array([[1 << r for r in range(n)]], dtype=np.uint32)
    acc = Acceptor(ctx, protocol, G, n, me, d, T)
    stores, sent_data, total = [], {}, 0
    for rnd in range(3):
        lens = (wl.cfg4_lengths(G, seed_extra=rnd)[0] // 4 + rng.integers(0, 7, G)).astype(np.uint32)
        gaps = rng.integers(0, 32, G)
        ends = np.cumsum(lens.astype(np.int64) + gaps)
        data_off = (16 + ends - lens.astype(np.int64)).astype(np.uint64)
        arena = rng.integers(0, 256, 16 + int(ends[-1]) + 32, dtype=np.uint8)
        L = (lens.astype(np.int64) + d - 1) // d
        store = torch.zeros((T, int(((L + 31) // 32 * 32).sum()) + 32), dtype=torch.uint8, device="cuda")
        pol = np.zeros(G, np.uint8)
        slot_out, shard_off, _ = eng.propose_ragged(_t(arena), _t(data_off), _t(lens), store, _t(pol) if cw else None)
        out, off, fl, _ = ctx.frame_accept_pack_ragged(store, shard_off, _t(lens), d, p, policies, _t(pol), me, slot_out, _t(bal),
                                                       with_assignment=cw)
        slots = slot_out.cpu().numpy().view(np.uint64)
        off_h, fl_h = off.cpu().numpy(), fl.cpu().numpy()
        buf_np = out.cpu().numpy()
        frames = [buf_np[int(off_h[g]):int(off_h[g]) + int(fl_h[g])].tobytes() for g in range(G)]
        buf, offs = _buffer(rng, frames)
        astore = torch.empty(sum(len(f) for f in frames) * 2 + 64, dtype=torch.uint8, device="cuda")
        awal = torch.empty(sum(len(f) + 48 for f in frames) + 64, dtype=torch.uint8, device="cuda")
        stores.append(astore)
        res = acc.accept(_t(buf), _t(offs), _t(np.arange(G, dtype=np.uint32)), _t(np.zeros(G, np.uint8)), astore, awal)
        assert (res["verdict"].cpu().numpy().view(np.uint32) == ACC).all()
        for g in range(G):
            sent_data[(g, int(slots[g]))] = arena[int(data_off[g]):int(data_off[g]) + int(lens[g])].tobytes()
        # the leader's heartbeat: commit_bar = one past this round's slot
        newly = acc.heartbeat(_t(np.arange(G, dtype=np.uint32)), _t(np.zeros(G, np.uint8)), _t(bal), _t(slots + np.uint64(1)),
                              _t(np.zeros(G, np.uint64)))
        entries, eg, el, cnt = ctx.wal_commit_pack(newly, acc.window_base, G)
        assert int(cnt.item()) == G
        ent, egh, elh = entries.cpu().numpy(), eg.cpu().numpy(), el.cpu().numpy()
        for i in range(G):
            assert ent[i, :elh[i]].tobytes() == oracle.wal_commit_slot(int(slots[egh[i]]))
        outb = torch.empty(int(sum(_r16(int(x)) for x in lens)) + 16, dtype=torch.uint8, device="cuda")
        ex = acc.execute(outb, G)
        assert ctx.device_status() == 0
        postponed = bin(int(policies[0][me])).count("1") < d    # an RSPaxos follower holds one shard
        nrec = 0 if postponed else G
        assert int(ex["totals"][0].item()) == nrec
        ob = outb.cpu().numpy()
        for k in range(nrec):
            g, s, o, ln = int(ex["rec_group"][k]), int(ex["rec_slot"][k]), int(ex["rec_off"][k]), int(ex["rec_len"][k])
            assert (g, s) == (k, int(slots[k])) and ob[o:o + ln].tobytes() == sent_data[(g, s)]
            total += 1
        assert (acc.commit_bar.cpu().numpy() == (0 if postponed else slots.astype(np.int64) + 1)).all()
    assert total == (0 if postponed else 3 * G)
    eng.close()
    acc.close()
