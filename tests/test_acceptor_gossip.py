"""Reconstruct requests from the device acceptor (ss_acceptor_gossip / ss_acceptor_step_up_reads, summerset_b200/csrc/acceptor.cu).

`gossip_model` restates trigger_gossiping (crossword/gossiping.rs:88-192) per group with the oracle's
gossip_targets_excl, and `step_up_model` the recon_slots of become_a_leader (rspaxos/leadership.rs:99-172,
crossword/leadership.rs:105-190), over the acceptor's state as `tests/test_acceptor_commit.Model` keeps it, extended
with each instance's source and whole assignment and a per-group gossip_bar; `call_model` adds the per-group capacity
cut of the header comment.  Expected frames come from `frame_reconstruct`, built on the oracle's varint and Bitmap
encoders.  The
GPU tests compare every frame byte, offset, length, destination, the canaries around `out`, gossip_bar and assign_rows
with the model, and run the closed loops leader -> acceptors -> commit -> device-built requests -> serve -> absorb ->
execute.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import pyoracle
from summerset_b200 import _lib
from tests.test_acceptor import ACC, FRAME_OVERFLOW, _buffer, _t
from tests.test_acceptor_commit import _codeword, _r16
from tests.test_acceptor_reconstruct import RRig, _bits, _pc, _var, recon_frame

RECON = 4
U64 = (1 << 64) - 1


def frame_reconstruct(variant, slots, excl=None, T=0):
    """PeerMessage::Msg{Reconstruct{slots}} (excl None, RSPaxos) or {slots_excl} with one size-T Bitmap per slot
    (Crossword), framed with the 8-byte big-endian length"""
    items = list(slots) if excl is None else [(s, T, [e]) for s, e in zip(slots, excl)]
    return recon_frame(items, excl is not None, variant)


# ---------------------------------------------------------------------------------------------
# the models
# ---------------------------------------------------------------------------------------------
def gossip_walk(m, g, bar, tail):
    """trigger_gossiping's walk -> (slots to plan, gossip_bar after it); Executed = slot < exec_bar, log_end = the window"""
    base = m.base[g]
    live = [s for s in m.inst[g] if base <= s < base + 64]
    log_end = max(live) + 1 if live else base
    until = log_end - tail if log_end > tail else 0
    up_to, plan = bar, []
    for s in range(max(bar, base), until):
        up_to = s
        if s < m.eb[g]:
            continue
        inst = m.inst[g].get(s)
        if inst is None or inst["st"] != "C":
            break
        if _pc(inst["held"]) < m.d:
            plan.append(s)
    return plan, max(bar, up_to)


def gossip_model(m, g, bar, tail, alive, batch, variant=RECON):
    """-> ([(peer, frame bytes)] in (peer, chunk) order, gossip_bar after the walk)"""
    plan, nb = gossip_walk(m, g, bar, tail)
    per = [[] for _ in range(m.n)]
    for s in plan:
        inst = m.inst[g][s]
        t, excl = pyoracle.gossip_targets_excl(m.me, m.n, m.d, inst["src"], inst["held"], inst["rows"], alive)
        for q in _bits(t):
            per[q].append((s, int(excl[q])))
    frames = []
    for q in range(m.n):
        for c in range(0, len(per[q]), batch):
            ch = per[q][c:c + batch]
            frames.append((q, frame_reconstruct(variant, [s for s, _ in ch], [e for _, e in ch], m.T)))
    return frames, nb


def step_up_model(m, g, cw, chunk, variant=RECON):
    """-> [(0xff, frame bytes)]: every committed instance of [max(exec_bar, base), base + 64) with fewer than d shards"""
    base = m.base[g]
    lst = [s for s in range(max(m.eb[g], base), base + 64)
           if s in m.inst[g] and m.inst[g][s]["st"] == "C" and _pc(m.inst[g][s]["held"]) < m.d]
    out = []
    for c in range(0, len(lst), chunk):
        ch = lst[c:c + chunk]
        out.append((0xFF, frame_reconstruct(variant, ch, [m.inst[g][s]["held"] for s in ch] if cw else None, m.T)))
    return out


def call_model(m, step_up, cw, groups, alive, tail, batch, out_cap, frame_cap):
    """one call over the listed groups (None: all), every entry planned from the state before the call.  -> dict:
    recs [(group, dst, off, bytes) or (group, None) for a cut record below frame_cap], totals, status; m.gbar moves"""
    lst = list(range(m.G)) if groups is None else list(groups)
    bar0 = list(m.gbar)
    recs, fo, oo, status, newbar = [], 0, 0, 0, {}
    for g in lst:
        if g >= m.G:
            continue
        if step_up:
            frames, nb = step_up_model(m, g, cw, batch), bar0[g]
        else:
            frames, nb = gossip_model(m, g, bar0[g], tail, alive[g] if alive is not None else (1 << 32) - 1, batch)
        size = sum(_r16(len(f)) for _, f in frames)
        if fo + len(frames) <= frame_cap and oo + size <= out_cap:
            o = oo
            for q, f in frames:
                recs.append((g, q, o, f))
                o += _r16(len(f))
            newbar[g] = nb
        else:
            status |= FRAME_OVERFLOW
            recs += [(g, None)] * max(0, min(len(frames), frame_cap - fo))
        fo += len(frames)
        oo += size
    for g, b in newbar.items():
        m.gbar[g] = b
    return dict(recs=recs, totals=[fo, oo], status=status)


# ---------------------------------------------------------------------------------------------
# CPU: the models on hand-written cases, symbols and refusals
# ---------------------------------------------------------------------------------------------
class _M:
    """Model-shaped state for the CPU cases"""

    def __init__(self, G, n, me, d, T):
        self.G, self.n, self.me, self.d, self.T = G, n, me, d, T
        self.base, self.eb, self.gbar = [0] * G, [0] * G, [0] * G
        self.inst = [dict() for _ in range(G)]

    def put(self, g, s, held, st="C", src=0, rows=None, dlen=9):
        self.inst[g][s] = dict(bal=1, held=held, dlen=dlen, st=st, src=src, rows=rows or [(1 << self.T) - 1] * self.n)


def test_model_gossip_walk_rules(oracle):
    m = _M(1, 5, 1, 3, 5)
    m.base[0] = 10
    for s in range(10, 16):
        m.put(0, s, 0b00010)
    m.inst[0][13]["st"] = "A"                                         # Accepting: the walk stops there
    assert gossip_walk(m, 0, 0, 0) == ([10, 11, 12], 13)             # the stop is slot_up_to
    m.gbar[0] = 13
    assert gossip_walk(m, 0, 13, 0) == ([], 13)                      # revisited, and stopped again
    m.inst[0][13]["st"] = "C"
    assert gossip_walk(m, 0, 13, 0) == ([13, 14, 15], 15)            # the last slot visited is slot_up_to: walked again
    assert gossip_walk(m, 0, 15, 0) == ([15], 15)
    m.eb[0] = 12
    m.inst[0][11]["st"] = "A"                                         # below exec_bar: Executed, passed whatever it holds
    assert gossip_walk(m, 0, 0, 0) == ([12, 13, 14, 15], 15)
    m.eb[0] = 0
    m.inst[0][11]["st"] = "C"
    m.inst[0][12]["held"] = 0b00111                                   # d shards held: walked, not planned
    assert gossip_walk(m, 0, 0, 0) == ([10, 11, 13, 14, 15], 15)
    # tail_ignores: log_end = 16 here; below, at and above it
    assert gossip_walk(m, 0, 0, 2) == ([10, 11, 13], 13)
    assert gossip_walk(m, 0, 0, 6) == ([], 0)                        # until = base: nothing walked, the bar stays
    assert gossip_walk(m, 0, 11, 16) == ([], 11) and gossip_walk(m, 0, 0, 17) == ([], 0)
    # log_end counts an Accepting or Preparing instance past a null slot; the null slot stops the walk
    m.put(0, 20, 0b1, st="P")
    assert gossip_walk(m, 0, 0, 0) == ([10, 11, 13, 14, 15], 16)
    assert gossip_walk(m, 0, 0, 4)[1] == 16 and gossip_walk(m, 0, 0, 5) == ([10, 11, 13, 14, 15], 15)
    # an empty window: log_end = base
    assert gossip_walk(_M(1, 5, 1, 3, 5), 0, 7, 0) == ([], 7)


def test_model_gossip_targets_and_frames(oracle):
    m = _M(1, 5, 1, 3, 5)
    rows = [1 << r for r in range(5)]                                 # one shard per replica
    m.put(0, 0, 0b00010, src=0, rows=rows)                            # me = 1 holds shard 1; the leader 0 is skipped
    m.put(0, 1, 0b00010, src=2, rows=rows)                            # source 2 skipped: peers 3, 4
    m.put(0, 2, 0, src=0, rows=rows, dlen=0)                          # a null instance: planned like any other
    m.put(0, 3, 0b00010, src=0, rows=[0, 0b10, 0, 0b11111, 0])        # empty rows ask nothing; peer 3 covers d alone
    fr, bar = gossip_model(m, 0, 0, 0, 0b11111, 10)
    assert bar == 3
    # exclusions: the availability of the moment each peer is picked, before its shards join it
    want = {2: [(0, 0b00010), (2, 0b00000)], 3: [(0, 0b00110), (1, 0b00010), (2, 0b00100), (3, 0b00010)],
            4: [(1, 0b01010), (2, 0b01100)]}
    got = {q: frame_reconstruct(RECON, *zip(*want[q]), 5) for q in want}
    assert fr == [(q, got[q]) for q in sorted(want)]
    # a dead peer is skipped and the walk goes on; the source is never asked, even when d is not covered
    fr, _ = gossip_model(m, 0, 0, 0, 0b11011, 10)                     # peer 2 dead
    assert [q for q, _ in fr] == [3, 4]
    # chunk edges: 4 entries for peer 3 at batch 1, 3, 4 and 5
    for b, cuts in ((1, [1, 1, 1, 1]), (3, [3, 1]), (4, [4]), (5, [4])):
        fr, _ = gossip_model(m, 0, 0, 0, 0b11111, b)
        sizes = [len(_parse_slots(f)) for q, f in fr if q == 3]
        assert sizes == cuts, b
    assert _parse_slots(frame_reconstruct(RECON, [1 << 40], [7], 5)) == [(1 << 40, 5, [7])]


def _parse_slots(frame):
    from tests.test_acceptor_reconstruct import parse_reconstruct
    return parse_reconstruct(frame, True)


def test_model_step_up_rules(oracle):
    m = _M(1, 5, 1, 3, 5)
    m.base[0] = 100
    for s in range(100, 110):
        m.put(0, s, 0b00010)
    m.inst[0][103]["st"] = "A"                                        # not committed: skipped, no stop
    m.inst[0][105]["held"] = 0b10101                                  # enough shards
    m.put(0, 150, 0b1)                                                # past a null gap
    m.eb[0] = 101
    fr = step_up_model(m, 0, False, 3)
    want = [[101, 102, 104], [106, 107, 108], [109, 150]]
    assert fr == [(0xFF, frame_reconstruct(RECON, w)) for w in want]
    fr = step_up_model(m, 0, True, 64)
    assert fr == [(0xFF, frame_reconstruct(RECON, sum(want, []), [m.inst[0][s]["held"] for s in sum(want, [])], 5))]
    # the encoder's bytes, written out: length, Msg, variant, count, then slots (and size, block count, block)
    assert frame_reconstruct(RECON, [7]) == bytes.fromhex("000000000000000400040107")
    assert frame_reconstruct(RECON, [1, 300], [3, 0], 5) == bytes.fromhex("000000000000000d00040201050103fb2c01050100")


def test_model_capacity_cut(oracle):
    m = _M(3, 5, 1, 3, 5)
    for g in range(3):
        for s in range(3):
            m.put(g, s, 0b00010, rows=[1 << r for r in range(5)])
    full = call_model(m, False, True, None, None, 0, 1, 1 << 30, 1 << 30)
    m.gbar = [0] * 3
    per = full["totals"][0] // 3
    cut = call_model(m, False, True, [0, 0, 2, 1], None, 0, 1, 1 << 30, 2 * per + 1)
    assert cut["status"] == FRAME_OVERFLOW and cut["totals"][0] == 4 * per
    assert [r[0] for r in cut["recs"] if r[1] is not None] == [0] * (2 * per)       # the repeat is planned again
    assert [r for r in cut["recs"] if r[1] is None] == [(2, None)]                  # the record below the cap
    assert m.gbar == [2, 0, 0]


def test_gossip_symbols_and_refusals():
    lib = _lib.load()
    for name in ("ss_acceptor_gossip_view_get", "ss_acceptor_gossip", "ss_acceptor_step_up_reads"):
        assert hasattr(lib, name)
    assert lib.ss_version() == 200
    v = _lib.AcceptorGossipView()
    assert C.sizeof(_lib.AcceptorGossipView) == 32
    assert lib.ss_acceptor_gossip_view_get(None, C.byref(v)) == _lib.SS_ERR_INVALID_ARG
    assert lib.ss_acceptor_gossip(None, None, 0, None, 0, 1, 4, None, 0, None, None, None, None, 0, None) == _lib.SS_ERR_INVALID_ARG
    assert lib.ss_acceptor_step_up_reads(None, None, 0, 1, 4, None, 0, None, None, None, None, 0, None) == _lib.SS_ERR_INVALID_ARG


@pytest.mark.skipif(torch.cuda.is_available(), reason="only meaningful on a box without a GPU")
def test_gossip_without_device():
    lib = _lib.load()
    h = C.c_void_p()
    cfg = _lib.AcceptorConfig(_lib.SS_PROTO_CROSSWORD, 5, 1, 3, 5, 2, 1, 3)
    assert lib.ss_acceptor_create(None, C.byref(cfg), 4, C.byref(h)) == _lib.SS_ERR_NO_DEVICE and not h


# ---------------------------------------------------------------------------------------------
# GPU helpers
# ---------------------------------------------------------------------------------------------
def accept_frame(s, bal, d, T, dlen, sh, rows):
    """an Accept frame; the oracle's encoder, or by hand for a codeword without shards"""
    if any(x is not None for x in sh):
        return pyoracle.frame_accept(2, s, bal, d, T - d, dlen, sh, rows, T)
    body = _var(0) + _var(2) + _var(s) + _var(bal) + bytes([d, T - d]) + _var(dlen) + _var(-(-dlen // d)) + _var(T) + b"\0" * (T + 1)
    if rows is not None:
        body += _var(len(rows)) + b"".join(pyoracle.bitmap_encode(T, r) for r in rows)
    return len(body).to_bytes(8, "big") + body


class GRig(RRig):
    def __init__(self, ctx, protocol, G, n, me, d, T):
        super().__init__(ctx, protocol, G, n, me, d, T)
        self.m.gbar = [0] * G

    def accept_items(self, items):
        """items: (g, slot, ballot, held, dlen, rows, src); the last accepted frame of a slot defines the instance"""
        m, d, T = self.m, self.m.d, self.m.T
        frames, groups, peers, want = [], [], [], []
        for g, s, bal, held, dlen, rows, src in items:
            _, shards = _codeword(self.rng, dlen, d, T)
            sh = [shards[j] if (held >> j) & 1 else None for j in range(T)]
            frames.append(accept_frame(s, bal, d, T, dlen, sh, rows if self.cw else None))
            groups.append(g)
            peers.append(src)
            if m.accept(g, s, bal, held, dlen, sh):
                m.inst[g][s].update(src=src, rows=list(rows))
                want.append(ACC)
            else:
                want.append(None)
        buf, offs = _buffer(self.rng, frames)
        store = torch.empty(sum(_pc(it[3]) * ((-(-it[4] // d) + 31) // 32 * 32) for it in items) + 64, dtype=torch.uint8, device="cuda")
        wal = torch.empty(sum(len(f) + 48 for f in frames) + 64, dtype=torch.uint8, device="cuda")
        self.stores.append(store)
        out = self.acc.accept(_t(buf), _t(offs), _t(np.array(groups, dtype=np.uint32)), _t(np.array(peers, dtype=np.uint8)), store, wal)
        v = out["verdict"].cpu().numpy().view(np.uint32)
        for i, w in enumerate(want):
            assert (int(v[i]) == ACC) == (w == ACC), i
        assert self.ctx.device_status() == 0

    def set_bars(self, eb=None, gbar=None):
        if eb is not None:
            self.m.eb = list(eb)
            self.acc.exec_bar.copy_(_t(np.array(eb, dtype=np.uint64)))
        if gbar is not None:
            self.m.gbar = list(gbar)
            self.acc.gossip_bar.copy_(_t(np.array(gbar, dtype=np.uint64)))

    def check_rows(self):
        m = self.m
        assert [int(x) for x in self.acc.gossip_bar.cpu().numpy().view(np.uint64)] == m.gbar
        if not self.cw:
            assert self.acc.assign_rows is None
            return
        rows = self.acc.assign_rows.cpu().numpy().view(np.uint32).reshape(m.G, 64, m.n)
        for g in range(m.G):
            for s, inst in m.inst[g].items():
                assert [int(x) for x in rows[g, s & 63]] == inst["rows"], (g, s)

    def requests(self, step_up, batch, groups=None, alive=None, tail=0, out_delta=None, frame_delta=None, frame_cap=None):
        """one call, every output against call_model; deltas cut the capacities relative to what the call asks for"""
        m = self.m
        snap = list(m.gbar)
        want_all = call_model(m, step_up, self.cw, groups, alive, tail, batch, 1 << 62, 1 << 62)
        m.gbar = snap
        fcap = want_all["totals"][0] + (frame_delta or 0) if frame_cap is None else frame_cap
        ocap = want_all["totals"][1] + (out_delta or 0)
        want = call_model(m, step_up, self.cw, groups, alive, tail, batch, max(ocap, 0), max(fcap, 0))
        canary = self.rng.integers(0, 256, max(ocap, 0) + 64, dtype=np.uint8)
        out = _t(canary.copy())
        gl = None if groups is None else _t(np.array(groups, dtype=np.uint32))
        al = None if alive is None else _t(np.array(alive, dtype=np.uint32))
        if step_up:
            res = self.acc.step_up_reads(out, max(fcap, 0), batch, gl, out_capacity=max(ocap, 0))
        else:
            res = self.acc.gossip(out, max(fcap, 0), batch, gl, al, tail, out_capacity=max(ocap, 0))
        got = {k: v.cpu().numpy() for k, v in res.items()}
        assert [int(x) for x in got["totals"]] == want["totals"]
        assert self.ctx.device_status() == want["status"]
        exp = canary.copy()
        ob = out.cpu().numpy()
        for f, r in enumerate(want["recs"]):
            grp, dst = int(got["frame_group"][f]), int(got["frame_dst"][f])
            off, ln = int(got["frame_off"][f]), int(got["frame_len"][f])
            if r[1] is None:
                assert (grp, dst, off, ln) == (r[0], 0xFF, -1, 0), f
                continue
            assert (grp, dst, off, ln) == (r[0], r[1], r[2], len(r[3])), f
            assert ob[off:off + ln].tobytes() == r[3], f
            exp[off:off + ln] = np.frombuffer(r[3], dtype=np.uint8)
        if not np.array_equal(ob, exp):
            pytest.fail(f"request output: {int((ob != exp).sum())} bytes differ")
        self.check_state()
        self.check_rows()
        return want, got


def _rows(rng, n, T, kind):
    if kind < T and kind >= 1:                                        # balanced, spr = kind
        return [int(x) for x in pyoracle.cw_brr_assignment(n, T, kind)]
    return [0 if rng.integers(0, 5) == 0 else int(rng.integers(0, 1 << T)) for _ in range(n)]   # unbalanced, empty rows


def _fill(rig, rng, bases, dense=12):
    """contiguous runs from each base (some null instances, some short of d shards), a few past a gap, committed by one
    heartbeat, then some slots re-accepted (Accepting again) -- twice in one call with different rows"""
    m = rig.m
    n, d, T = m.n, m.d, m.T
    rig.set_base(bases)
    items = []
    for g in range(m.G):
        k = int(rng.integers(0, dense + 1))
        pos = list(range(k)) + [int(x) for x in rng.integers(k + 1, 64, int(rng.integers(0, 3)))]
        for w in sorted(set(pos)):
            held = int(rng.integers(0, 1 << T))
            if rng.integers(0, 2):
                held &= int(rng.integers(0, 1 << T))                  # often fewer than d shards
            dlen = int(rng.integers(1, 200))
            if rng.integers(0, 9) == 0:
                held, dlen = 0, 0                                     # a null instance
            kind = int(rng.integers(1, T + 3))
            items.append((g, bases[g] + w, 5, held, dlen, _rows(rng, n, T, kind), int(rng.integers(0, n))))
    rig.accept_items(items)
    rig.commit_all()
    again = []
    for g in range(m.G):
        for s in list(m.inst[g])[:2]:
            if rng.integers(0, 3) == 0:
                for _ in range(2):
                    again.append((g, s, 5, int(rng.integers(0, 1 << T)), int(rng.integers(1, 50)), _rows(rng, n, T, 0),
                                  int(rng.integers(0, n))))
    if again:
        rig.accept_items(again)
    rig.check_rows()


BASES = [0, 3, 250, 65535, (1 << 32) - 20, (1 << 32) + 5, U64 - 200, U64 - 65]
GOSSIP_CODES = ([(n, max(1, n // 2), n) for n in range(1, 33)] + [(7, d, 32) for d in (1, 16, 31, 32)])


# ---------------------------------------------------------------------------------------------
# GPU: the matrix
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n,d,T", GOSSIP_CODES)
def test_gossip_matrix(ctx, n, d, T):
    G = len(BASES)
    rig = GRig(ctx, "crossword", G, n, n // 2, d, T)
    rng = rig.rng
    _fill(rig, rng, BASES)
    rig.set_bars(eb=[b + int(rng.integers(0, 6)) if rng.integers(0, 2) else 0 for b in BASES])
    for rnd, batch in enumerate((1, 2, 10, 64, 65)):
        alive = [int(rng.integers(0, 1 << n)) | (1 << rig.m.me) for _ in range(G)] if rnd % 2 else None
        tail = int(rng.choice([0, 1, 3, 70]))
        groups = [None, [int(x) for x in rng.integers(0, G, 5)], [3, 3, 1, G + 2, 7, 0]][rnd % 3]
        rig.requests(False, batch, groups, alive, tail)
        rig.requests(True, batch, groups)
        if rnd == 2:
            rig.set_bars(gbar=[b + int(rng.integers(0, 40)) for b in BASES[:G - 2]] + [0, U64 - 70])
    rig.requests(False, 3)                                              # the bars as the calls left them: re-walks


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 2, 3, 5, 8, 17, 32])
def test_step_up_rspaxos(ctx, n):
    d = n // 2 + 1
    rig = GRig(ctx, "rspaxos", len(BASES), n, n - 1, d, n)
    rng = rig.rng
    _fill(rig, rng, BASES)
    rig.set_bars(eb=[b + int(rng.integers(0, 6)) if rng.integers(0, 2) else 0 for b in BASES])
    for chunk in (1, 2, 10, 64, 65):
        rig.requests(True, chunk, [None, [5, 5, 0, 99]][chunk % 2])


@pytest.mark.gpu
@pytest.mark.parametrize("protocol", ["crossword", "rspaxos"])
def test_capacity_cut_and_drain(ctx, protocol):
    n, d, T = 5, 3, 5
    cw = protocol == "crossword"
    rig = GRig(ctx, protocol, 40, n, 1, d, T)
    rng = rig.rng
    _fill(rig, rng, [int(x) for x in rng.integers(0, 1 << 20, 40)], dense=30)
    step = not cw
    for od, fd in ((0, 0), (-1, None), (None, -1), (-300, None), (None, -7)):
        rig.requests(step, 2, None, None, 0, od, fd)
    if cw:
        # a drain: calls with a third of the frame room walk every group; then only the revisited slots are asked for
        rig.set_bars(gbar=[0] * 40)
        snap = list(rig.m.gbar)
        cap = call_model(rig.m, False, True, None, None, 0, 3, 1 << 62, 1 << 62)["totals"][0] // 3
        rig.m.gbar = snap
        for calls in range(1, 50):
            want, _ = rig.requests(False, 3, frame_cap=cap)
            if not want["status"]:
                break
        assert 3 <= calls < 50                                                                  # everything walked: a call repeats only the revisits
        before = list(rig.m.gbar)
        rig.requests(False, 3)
        assert rig.m.gbar == before


@pytest.mark.gpu
def test_reaccept_defines_assign_rows(ctx):
    """of two accepted frames of one slot in one call the last defines the rows the gossip plans with"""
    n, d, T = 5, 3, 5
    rig = GRig(ctx, "crossword", 2, n, 1, d, T)
    first, last = [0b11111, 0, 0, 0, 0], [0, 0, 0b00100, 0b01000, 0b10000]
    rig.accept_items([(g, s, 3, 0b00010, 30, first if k == 0 else last, 0) for g in range(2) for s in range(3) for k in range(2)])
    rig.commit_all()
    rig.check_rows()
    want, _ = rig.requests(False, 64)
    assert sorted({r[1] for r in want["recs"]}) == [2, 3]              # the last rows: peers 2 and 3 cover d
    rig.accept_items([(0, 1, 3, 0b00010, 30, first, 0)])                    # Accepting again, rows of the later call
    rig.check_rows()
    rig.set_bars(gbar=[0, 0])
    rig.requests(False, 64)


def _warp_cap(ctx):
    return ctx.sm_count * 64 * 8          # launch_grid: 64 CTAs per SM, 8 warps per CTA


@pytest.mark.gpu
def test_requests_past_the_grid_cap(ctx):
    """more listed groups than the size and write passes have warps: later groups take a warp's second sweep"""
    n, d, T, me = 5, 3, 5, 1
    G = _warp_cap(ctx) + 1000
    rig = GRig(ctx, "crossword", G, n, me, d, T)
    rng = rig.rng
    live = [g for g in range(G) if g % 211 == 0 or g >= G - 400]
    rows = [int(x) for x in pyoracle.cw_brr_assignment(n, T, 1)]
    rig.accept_items([(g, s, 2, 1 << me, 40, rows, 0) for g in live for s in range(1 + g % 3)])
    rig.commit_all()
    want, _ = rig.requests(False, 2)
    assert len(want["recs"]) >= len(live) * 2
    rig.set_bars(gbar=[0] * G)
    rig.requests(True, 1)
    rig.requests(False, 1, list(range(G - 1, -1, -1)))


@pytest.mark.gpu
def test_request_refusals(ctx):
    rs = GRig(ctx, "rspaxos", 2, 5, 1, 3, 5)
    cw = GRig(ctx, "crossword", 2, 5, 1, 3, 5)
    x = torch.zeros(256, dtype=torch.uint8, device="cuda")
    p = x.data_ptr()
    lib = rs.acc.lib
    assert lib.ss_acceptor_gossip(rs.acc.h, None, 0, None, 0, 1, 4, p, 64, p, p, p, p, 4, None) == _lib.SS_ERR_INVALID_ARG
    assert lib.ss_acceptor_gossip(cw.acc.h, None, 0, None, 0, 0, 4, p, 64, p, p, p, p, 4, None) == _lib.SS_ERR_INVALID_ARG
    assert lib.ss_acceptor_step_up_reads(cw.acc.h, None, 0, 0, 4, p, 64, p, p, p, p, 4, None) == _lib.SS_ERR_INVALID_ARG
    assert lib.ss_acceptor_gossip(cw.acc.h, None, 0, None, 0, 1, 4, p + 8, 64, p, p, p, p, 4, None) == _lib.SS_ERR_INVALID_ARG
    assert lib.ss_acceptor_step_up_reads(rs.acc.h, None, 0, 1, 4, p, 64, None, p, p, p, 4, None) == _lib.SS_ERR_INVALID_ARG
    tot = torch.full((2,), 7, dtype=torch.int64, device="cuda")
    g = torch.zeros(1, dtype=torch.int32, device="cuda")
    assert lib.ss_acceptor_gossip(cw.acc.h, g.data_ptr(), 0, None, 0, 1, 4, None, 0, None, None, None, None, 0, tot.data_ptr()) == _lib.SS_OK
    assert tot.tolist() == [0, 0]
    assert rs.acc.assign_rows is None and cw.acc.assign_rows.numel() == 2 * 64 * 5


# ---------------------------------------------------------------------------------------------
# GPU: closed loops through the leader path, requests built on the device
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("protocol,n,T,d,spr", [("crossword", 5, 5, 3, 1), ("crossword", 5, 5, 3, 2), ("crossword", 7, 14, 7, 2),
                                                 ("rspaxos", 5, 5, 3, 1)])
def test_closed_loop_device_requests(ctx, oracle, protocol, n, T, d, spr):
    from summerset_b200 import workloads as wl
    from summerset_b200.engine import Acceptor, LeaderEngine
    cw = protocol == "crossword"
    G = 64
    rng = np.random.default_rng(n * 100 + T + spr)
    eng = LeaderEngine(ctx, protocol, G, n, 1, 1, **(dict(rs_total_shards=T, rs_data_shards=d) if cw else {}))
    d, p, T = eng.d, eng.T - eng.d, eng.T
    bal = rng.integers(1, 1 << 30, G).astype(np.uint64)
    eng.set_prepared_ballots(_t(bal))
    if cw:
        policies = np.array([oracle.cw_brr_assignment(n, T, spr)], dtype=np.uint32)
        eng.set_policies([list(map(int, q)) for q in policies], False)
    else:
        policies = np.array([[1 << r for r in range(n)]], dtype=np.uint32)
    accs = [Acceptor(ctx, protocol, G, n, r, d, T) for r in range(n)]
    keep, delivered, me = [], 0, 1
    fol = accs[me]
    held_me = int(policies[0][me])
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
        slots = slot_out.cpu().numpy().view(np.uint64)
        for r, acc in enumerate(accs):
            out, off, fl, _ = ctx.frame_accept_pack_ragged(store, shard_off, _t(lens), d, p, policies, _t(pol), r, slot_out, _t(bal),
                                                           with_assignment=cw)
            off_h, fl_h, ob = off.cpu().numpy(), fl.cpu().numpy(), out.cpu().numpy()
            frames = [ob[int(off_h[g]):int(off_h[g]) + int(fl_h[g])].tobytes() for g in range(G)]
            buf, offs = _buffer(rng, frames)
            astore = torch.empty(sum(len(f) for f in frames) * 2 + 64, dtype=torch.uint8, device="cuda")
            awal = torch.empty(sum(len(f) + 48 for f in frames) + 64, dtype=torch.uint8, device="cuda")
            keep.append(astore)
            res = acc.accept(_t(buf), _t(offs), _t(np.arange(G, dtype=np.uint32)), _t(np.zeros(G, np.uint8)), astore, awal)
            assert (res["verdict"].cpu().numpy().view(np.uint32) == ACC).all()
            acc.heartbeat(_t(np.arange(G, dtype=np.uint32)), _t(np.zeros(G, np.uint8)), _t(bal), _t(slots + np.uint64(1)),
                          _t(np.zeros(G, np.uint64)))
        if cw:
            rows = fol.assign_rows.cpu().numpy().view(np.uint32).reshape(G, 64, n)
            assert all((rows[g, int(slots[g]) & 63] == policies[0]).all() for g in range(G))
        sent = [arena[int(data_off[g]):int(data_off[g]) + int(lens[g])].tobytes() for g in range(G)]
        outb = torch.empty(int(sum(_r16(int(x)) for x in lens)) + 16, dtype=torch.uint8, device="cuda")
        ex = fol.execute(outb, G)
        assert int(ex["totals"][0].item()) == (G if _pc(held_me) >= d else 0)
        if _pc(held_me) >= d:
            continue
        # the requests, built on the device: Crossword gossip at the follower, RSPaxos step-up reads at a new leader
        rbuf = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
        if cw:
            req = fol.gossip(rbuf, 4 * G * n, 1)
        else:
            req = fol.step_up_reads(rbuf, 4 * G, 10)
        assert ctx.device_status() == 0
        nf = int(req["totals"][0].item())
        rb = rbuf.cpu().numpy()
        dev_frames = [(int(req["frame_group"][f]), int(req["frame_dst"][f]),
                       rb[int(req["frame_off"][f]):int(req["frame_off"][f]) + int(req["frame_len"][f])].tobytes()) for f in range(nf)]
        # the hand-built requests of the host-side loop: the same frames
        hand = []
        for g in range(G):
            if cw:
                t, excl = oracle.gossip_targets_excl(me, n, d, 0, held_me, policies[0], (1 << n) - 1)
                hand += [(g, q, recon_frame([(int(slots[g]), T, [int(excl[q])])], True)) for q in _bits(t)]
            else:
                hand.append((g, 0xFF, recon_frame([int(slots[g])], False)))
        assert dev_frames == hand
        reqs = {}
        for g, q, f in dev_frames:
            for dst in ([q] if q != 0xFF else [x for x in range(n) if x != me]):
                reqs.setdefault(dst, []).append((g, f))
        replies, rgroups = [], []
        for q, lst in sorted(reqs.items()):
            buf, offs = _buffer(rng, [f for _, f in lst])
            out = torch.empty(1 << 22, dtype=torch.uint8, device="cuda")
            res = accs[q].reconstruct_serve(_t(buf), _t(offs), _t(np.array([g for g, _ in lst], dtype=np.uint32)),
                                            _t(np.full(len(lst), me, np.uint8)), out)
            assert (res["verdict"].cpu().numpy().view(np.uint32) == ACC).all()
            ro, rl, ob = res["reply_off"].cpu().numpy(), res["reply_len"].cpu().numpy(), out.cpu().numpy()
            for k, (g, _) in enumerate(lst):
                assert rl[k] > 0
                replies.append(ob[int(ro[k]):int(ro[k]) + int(rl[k])].tobytes())
                rgroups.append(g)
        buf, offs = _buffer(rng, replies)
        fstore = torch.empty(1 << 24, dtype=torch.uint8, device="cuda")
        keep.append(fstore)
        res = fol.absorb(_t(buf), _t(offs), _t(np.array(rgroups, dtype=np.uint32)), _t(np.zeros(len(replies), np.uint8)), fstore)
        assert (res["verdict"].cpu().numpy().view(np.uint32) == ACC).all() and ctx.device_status() == 0
        ex = fol.execute(outb, G)
        assert ctx.device_status() == 0 and int(ex["totals"][0].item()) == G
        ob = outb.cpu().numpy()
        for k in range(G):
            g, s, o, ln = int(ex["rec_group"][k]), int(ex["rec_slot"][k]), int(ex["rec_off"][k]), int(ex["rec_len"][k])
            assert (g, s) == (k, int(slots[k])) and ob[o:o + ln].tobytes() == sent[g]
            delivered += 1
        # nothing is left to ask for: a second request call is empty
        again = fol.gossip(rbuf, 4 * G * n, 1) if cw else fol.step_up_reads(rbuf, 4 * G, 10)
        assert int(again["totals"][0].item()) == 0
        upto = _t(slots.astype(np.uint64) + np.uint64(1))
        for acc in accs:
            acc.advance(upto)
        eng.advance(None)
    assert delivered == (3 * G if _pc(int(policies[0][me])) < d else 0)
    eng.close()
    for acc in accs:
        acc.close()
