"""The Paxos-family engine's sliding instance window (ss_engine_propose_next / ss_engine_advance / ss_engine_window_get:
summerset_b200/csrc/engine.cu) over many windows, against the oracle's per-message handlers run at ABSOLUTE slots.

Every group proposes at its first Null slot (rspaxos/mod.rs:434-442), AcceptReply frames at absolute slots go through
ss_accept_reply_parse_dev with the engine's window_base (replies below it are dropped, multipaxos/messages.rs:377), and
committed prefixes are retired by moving window_base forward (multipaxos/snapshot.rs:121-171).  The oracle holds slots
0..255 (rec_slot is u8), so a model slot m stands for absolute slot B + m, B = 0 except in the large-base run.
"""
import ctypes as C
import functools

import numpy as np
import pytest
import torch

from summerset_b200 import _lib
from summerset_b200 import workloads as wl
from summerset_b200._lib import SummersetError

DEV = "cuda:0"
S = 256
REPLY = 3                                   # the AcceptReply variant index the frames carry
U64MAX = np.uint64(0xFFFF_FFFF_FFFF_FFFF)
WINDOW_FULL = 8                             # SS_DEV_STATUS_WINDOW_FULL


def _t(a):
    a = np.ascontiguousarray(a)
    if a.dtype == np.uint64:
        a = a.view(np.int64)
    elif a.dtype == np.uint32:
        a = a.view(np.int32)
    return torch.from_numpy(a).to(DEV)


def _u64(t):
    return t.cpu().numpy().view(np.uint64)


def _ring_to_window(x, base):
    r = base.astype(np.uint64) & np.uint64(63)
    return (x >> r) | (x << ((np.uint64(64) - r) & np.uint64(63)))


class _Model:
    """Oracle state [G, S] at model slots; mb = model window base, top = one past the highest proposed slot."""

    def __init__(self, G, bal):
        self.G, self.bal = G, bal
        self.status = np.zeros(G * S, dtype=np.uint8)
        self.acks = np.zeros(G * S, dtype=np.uint16)
        self.inst_bal = np.zeros(G * S, dtype=np.uint64)
        self.pidx = np.zeros(G * S, dtype=np.uint8)
        self.mb = np.zeros(G, dtype=np.int64)
        self.top = np.zeros(G, dtype=np.int64)

    def window(self, st):
        idx = self.mb[:, None] + np.arange(64)
        assert idx.max() < S
        bits = np.take_along_axis(self.status.reshape(self.G, S) == st, idx, axis=1)
        return np.packbits(bits, axis=1, bitorder="little").view(np.uint64).reshape(-1)

    def first_null(self, oracle):
        idx = self.mb[:, None] + np.arange(64)
        null = np.take_along_axis(self.status.reshape(self.G, S) == oracle.ST_NULL, idx, axis=1)
        return np.where(null.any(axis=1), self.mb + null.argmax(axis=1), -1)

    def propose(self, oracle, slot, pol):
        g = np.nonzero(slot >= 0)[0]
        k = g * S + slot[g]
        self.status[k] = oracle.ST_ACCEPTING
        self.acks[k] = 0
        self.inst_bal[k] = self.bal[g]
        self.pidx[k] = pol[g]
        self.top[g] = np.maximum(self.top[g], slot[g] + 1)


@functools.lru_cache(maxsize=None)
def _frame(oracle, slot, ballot, with_size):
    return oracle.frame_accept_reply(REPLY, slot, ballot, with_size, 7)


def _reply_frames(oracle, rng, model, n, nrec, weight, B, with_size):
    """AcceptReplies at absolute slots: mostly to proposed instances of the window (older ones more often), plus
    retired slots, never-proposed slots (some beyond the window), slots far beyond anything the oracle holds, stale
    ballots, out-of-range peers and duplicates.  Returns the frames' parse inputs and the oracle's record stream."""
    G = model.G
    rg = rng.choice(G, nrec, p=weight / weight.sum()).astype(np.uint32)
    lo, hi = model.mb[rg], model.top[rg]
    span = np.maximum(hi - lo, 1)
    slot = lo + np.min(rng.integers(0, 1 << 30, (3, nrec)), axis=0) % span
    r = rng.random(nrec)
    retired = r < 0.1
    slot[retired] = np.maximum(lo[retired] - 1 - rng.integers(0, 5, int(retired.sum())), 0)
    fresh = (r >= 0.1) & (r < 0.15)
    slot[fresh] = np.minimum(hi[fresh] + rng.integers(0, 80, int(fresh.sum())), S - 1)
    far = (r >= 0.15) & (r < 0.17)                        # parsed to 0xff; not fed to the oracle
    peer = rng.integers(0, n + 1, nrec).astype(np.uint8)  # n = out-of-range peer
    ballot = model.bal[rg].copy()
    stale = rng.random(nrec) < 0.08
    ballot[stale] += rng.integers(1, 3, int(stale.sum())).astype(np.uint64)
    frames = [_frame(oracle, B + (1 << 40) + int(s) if f else B + int(s), int(b), with_size) for s, b, f in zip(slot, ballot, far)]
    offs = np.concatenate([[0], np.cumsum([len(f) for f in frames])[:-1]]).astype(np.uint64)
    buf = np.frombuffer(b"".join(frames), dtype=np.uint8).copy()
    keep = ~far
    return (buf, offs, rg, peer), (rg[keep], slot[keep].astype(np.uint8), peer[keep], ballot[keep])


def _check_wal(ctx, oracle, newly, window_base, B, mb, want_newly):
    total = int(sum(bin(int(w)).count("1") for w in want_newly))
    entries, eg, el, cnt = ctx.wal_commit_pack(newly, window_base, max(total, 1))
    torch.cuda.synchronize()
    assert int(cnt) == total
    entries, eg, el = entries.cpu().numpy(), eg.cpu().numpy(), el.cpu().numpy()
    got = sorted((int(eg[i]), entries[i, :el[i]].tobytes()) for i in range(total))
    want = sorted((g, oracle.wal_commit_slot(B + int(mb[g]) + s)) for g in np.nonzero(want_newly)[0] for s in range(64)
                  if (int(want_newly[g]) >> s) & 1)
    assert got == want


def _run_window(ctx, oracle, eng, model, rounds, rng, n, tally, B=0, with_size=False, policies=None, data_len=0):
    """propose_next (1..4 per round) -> two parsed reply batches, each ingested and ticked -> advance with a per-group
    random upto (every fourth round: NULL).  Checks every step against the model."""
    G = model.G
    weight = np.where(rng.random(G) < 0.2, 0.1, 1.0)     # slow groups: their windows fill
    newly = torch.zeros(G, dtype=torch.int64, device=DEV)
    seen_full = 0
    for rnd in range(rounds):
        for k in range(int(rng.integers(1, 5))):
            want = model.first_null(oracle)
            full = want < 0
            pol = rng.integers(0, len(policies), G).astype(np.uint8) if policies is not None else np.zeros(G, np.uint8)
            payload = _t(wl.payload_uniform(G, data_len, seed_extra=1000 * rnd + k)) if data_len else None
            slot_out, _ = eng.propose_next(0, payload, _t(pol) if policies is not None else None)
            status = ctx.device_status()
            got = _u64(slot_out)
            assert (got[~full] == (B + want[~full]).astype(np.uint64)).all(), (rnd, k)
            assert (got[full] == U64MAX).all()
            assert status == (WINDOW_FULL if full.any() else 0)
            seen_full += int(full.sum())
            model.propose(oracle, want, pol)
        for _ in range(2):
            (buf, offs, fg, fp), recs = _reply_frames(oracle, rng, model, n, 16 * G, weight, B, with_size)
            rg, rs_, rp, rb, rk = ctx.accept_reply_parse(_t(buf), _t(offs), _t(fg), _t(fp), eng.window_base, REPLY, with_size)
            eng.on_accept_replies(rg, rs_, rp, rb)
            before = model.window(oracle.ST_COMMITTED)
            committed, bar = eng.tick(newly)
            torch.cuda.synchronize()
            assert (rk.cpu().numpy() == REPLY).all()
            tally(*recs)
            want_c = model.window(oracle.ST_COMMITTED)
            wb = _u64(eng.window_base)
            assert (wb == (B + model.mb).astype(np.uint64)).all()
            assert (_ring_to_window(_u64(committed), wb) == want_c).all(), rnd
            assert (_ring_to_window(_u64(eng.accepting), wb) == model.window(oracle.ST_ACCEPTING)).all(), rnd
            want_newly = want_c & ~before
            assert (_u64(newly) == want_newly).all(), rnd
            want_bar = np.array([oracle.commit_bar(int(w)) for w in want_c], dtype=np.uint32)
            assert (bar.cpu().numpy().view(np.uint32) == want_bar).all(), rnd
            _check_wal(ctx, oracle, newly, eng.window_base, B, model.mb, want_newly)
        # retire: everything / part / a target below the base / nothing
        bar_m = np.array([oracle.commit_bar(int(w)) for w in model.window(oracle.ST_COMMITTED)], dtype=np.int64)
        if rnd % 4 == 3:
            eng.advance()
            k = bar_m
        else:
            cls = rng.integers(0, 4, G)
            abs_base = B + model.mb
            upto = np.select([cls == 0, cls == 1, cls == 2],
                             [abs_base + 64 + rng.integers(0, 1 << 20, G), abs_base + rng.integers(0, 70, G) % (bar_m + 2),
                              np.maximum(abs_base - rng.integers(1, 5, G), 0)], abs_base)
            eng.advance(_t(upto.astype(np.uint64)))
            k = np.clip(upto - abs_base, 0, bar_m)
        model.mb += k
        torch.cuda.synchronize()
        assert (_u64(eng.window_base) == (B + model.mb).astype(np.uint64)).all(), rnd
        assert (eng.commit_bar.cpu().numpy().view(np.uint32) == (bar_m - k).astype(np.uint32)).all(), rnd
    return seen_full


def _tally_fn(oracle, model, protocol, n, f, thr, T=0, d=0, balanced=True, policies=None):
    majority = n // 2 + 1
    if protocol == "crossword":
        return lambda rg, rs_, rp, rb: oracle.tally_stream_crossword(rg, rs_, rp, rb, S, n, T, d, majority, f, balanced, policies,
                                                                     model.pidx, model.bal, model.inst_bal, model.status, model.acks)
    return lambda rg, rs_, rp, rb: oracle.tally_stream(rg, rs_, rp, rb, S, n, thr, model.bal, model.inst_bal, model.status, model.acks)


@pytest.mark.gpu
@pytest.mark.parametrize("protocol,n,f,data_len,G,cw", [
    ("rspaxos", 5, 1, 4096, 1000, None), ("rspaxos", 7, 1, 1000, 1000, None),
    ("multipaxos", 5, 0, 0, 1000, None), ("multipaxos", 4, 0, 0, 1001, None),      # odd G: the one-group-per-thread tick
    ("crossword", 5, 2, 1500, 1000, (5, 3, True)), ("crossword", 5, 1, 1500, 1000, (5, 3, False))])
def test_engine_window_multi_window_run(ctx, oracle, protocol, n, f, data_len, G, cw):
    from summerset_b200.engine import LeaderEngine
    rng = np.random.default_rng(n * 100 + f * 10 + G + (cw[2] if cw else 7))
    majority = n // 2 + 1
    policies = T = d = None
    balanced = True
    if protocol == "crossword":
        T, d, balanced = cw
        eng = LeaderEngine(ctx, protocol, G, n, f, data_len, rs_total_shards=T, rs_data_shards=d)
        if balanced:
            policies = np.stack([oracle.cw_brr_assignment(n, T, spr) for spr in range(T // n, d + 1, T // n)])
        else:
            policies = np.stack([oracle.cw_brr_assignment(n, T, d)] +
                                [rng.integers(1, 1 << T, size=n).astype(np.uint32) for _ in range(3)])
        eng.set_policies([list(map(int, q)) for q in policies], balanced)
    else:
        eng = LeaderEngine(ctx, protocol, G, n, f, data_len)
    thr = majority + f if protocol == "rspaxos" else majority
    bal = rng.integers(1, 1 << 30, G).astype(np.uint64)
    eng.set_prepared_ballots(_t(bal))
    model = _Model(G, bal)
    assert (_u64(eng.window_base) == 0).all()
    tally = _tally_fn(oracle, model, protocol, n, f, thr, T, d, balanced, policies)
    seen_full = _run_window(ctx, oracle, eng, model, 60, rng, n, tally, 0, protocol == "crossword", policies, data_len)
    # ring positions were reused after retirement, bases diverged, and some windows filled
    assert model.mb.max() >= 64 and model.top.max() >= 100 and len(np.unique(model.mb)) > 20 and seen_full > 0
    assert model.top.max() < S
    eng.close()


@pytest.mark.gpu
def test_engine_window_large_base_crosses_2_32(ctx, oracle):
    """Bases installed at 2^32 - 10 through ss_engine_window_get: slot arithmetic past 32 bits."""
    from summerset_b200.engine import LeaderEngine
    rng = np.random.default_rng(232)
    G, n, f = 600, 5, 1
    B = (1 << 32) - 10
    eng = LeaderEngine(ctx, "rspaxos", G, n, f, 512)
    bal = rng.integers(1, 1 << 30, G).astype(np.uint64)
    eng.set_prepared_ballots(_t(bal))
    eng.window_base.fill_(B)
    model = _Model(G, bal)
    _run_window(ctx, oracle, eng, model, 12, rng, n, _tally_fn(oracle, model, "rspaxos", n, f, 4), B, False, None, 512)
    assert (B + model.mb).max() > (1 << 32) and (B + model.top).max() > (1 << 32) + 10
    eng.close()


@pytest.mark.gpu
def test_engine_window_shard_stores(ctx, oracle):
    """keep_slots = 3, store cycling: each proposal's planes are the oracle encode + contiguous split; the other stores
    are untouched."""
    from summerset_b200.engine import LeaderEngine
    G, n, f, data_len = 512, 5, 1, 3000
    d, p = 3, 2
    eng = LeaderEngine(ctx, "rspaxos", G, n, f, data_len, keep_slots=3)
    eng.set_prepared_ballots(_t(np.arange(1, G + 1, dtype=np.uint64)))
    eng.shards.fill_(0x5A)
    L = oracle.cw_shard_len(data_len, d)
    for i in range(7):
        store = i % 3
        before = eng.shards.clone()
        payload = wl.payload_uniform(G, data_len, seed_extra=500 + i)
        slot_out, sh = eng.propose_next(store, _t(payload))
        torch.cuda.synchronize()
        assert (_u64(slot_out) == i).all()
        assert sh.data_ptr() == eng.shards[store].data_ptr()
        got = sh.cpu().numpy()
        assert (got[d:] == oracle.rs_encode_uniform(d, p, payload, data_len)).all()
        for g in (0, 1, G // 2, G - 1):
            assert (got[:d, g, :L] == oracle.cw_split(payload[g, :data_len].tobytes(), d)).all()
        for other in range(3):
            if other != store:
                assert torch.equal(eng.shards[other], before[other])
    eng.close()


@pytest.mark.gpu
def test_engine_window_advance_edges(ctx, oracle):
    """upto below the base is a no-op, upto past the committed prefix is clamped, NULL retires exactly commit_bar, a
    slot re-proposed at a retired ring position starts with no acks and no committed bit, a full window is refused."""
    from summerset_b200.engine import LeaderEngine
    G, n = 64, 3
    eng = LeaderEngine(ctx, "multipaxos", G, n)
    bal = np.arange(1, G + 1, dtype=np.uint64)
    eng.set_prepared_ballots(_t(bal))

    def ack(rel_slots):          # every peer acks these window-relative slots of every group
        rg = np.repeat(np.arange(G, dtype=np.uint32), len(rel_slots) * n)
        rs_ = np.tile(np.repeat(np.array(rel_slots, dtype=np.uint8), n), G)
        rp = np.tile(np.arange(n, dtype=np.uint8), G * len(rel_slots))
        eng.on_accept_replies(_t(rg), _t(rs_), _t(rp), _t(bal[rg]))
        eng.tick()

    def state():
        torch.cuda.synchronize()
        return _u64(eng.window_base).copy(), eng.commit_bar.cpu().numpy().copy()

    for _ in range(6):
        eng.propose_next(0, None)
    ack([0, 1, 2, 3])
    assert (state()[1] == 4).all()
    eng.advance(_t(np.full(G, 2, dtype=np.uint64)))                   # part of the prefix
    assert (state()[0] == 2).all() and (state()[1] == 2).all()
    eng.advance(_t(np.full(G, 1, dtype=np.uint64)))                   # below the base: no-op
    assert (state()[0] == 2).all() and (state()[1] == 2).all()
    eng.advance(_t(np.full(G, 1000, dtype=np.uint64)))                # past the committed prefix: clamped
    assert (state()[0] == 4).all() and (state()[1] == 0).all()
    assert (_u64(eng.planes) & np.uint64(0xF) == 0).all() and (_u64(eng.committed) & np.uint64(0xF) == 0).all()
    ack([0, 1])                                                       # slots 4 and 5
    assert (state()[1] == 2).all()
    eng.advance()                                                     # NULL: exactly commit_bar
    assert (state()[0] == 6).all() and (state()[1] == 0).all()
    assert ctx.device_status() == 0
    # slots 6..69 fill the window; slot 64 lands on ring position 0, where slot 0 had every peer's ack
    for i in range(64):
        slot_out, _ = eng.propose_next(0, None)
        assert (_u64(slot_out) == 6 + i).all()
    torch.cuda.synchronize()
    assert (_u64(eng.planes) == 0).all()
    assert (_u64(eng.committed) == 0).all() and (_u64(eng.accepting) == U64MAX).all()
    assert (_u64(eng.inst_bal).reshape(G, 64)[:, 0] == bal).all()
    assert ctx.device_status() == 0
    snap = [t.clone() for t in (eng.planes, eng.inst_bal, eng.accepting, eng.committed, eng.commit_bar, eng.window_base)]
    slot_out, _ = eng.propose_next(0, None)                          # full window: refused, reported, unchanged
    assert (_u64(slot_out) == U64MAX).all() and ctx.device_status() == WINDOW_FULL
    for a, b in zip(snap, (eng.planes, eng.inst_bal, eng.accepting, eng.committed, eng.commit_bar, eng.window_base)):
        assert torch.equal(a, b)
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("protocol", ["crossword", "rspaxos"])
def test_engine_window_propose_next_equals_propose_at_base_0(ctx, oracle, protocol):
    """On a fresh engine, propose_next x k leaves the same full state, byte for byte, as propose(0..k-1)."""
    from summerset_b200.engine import LeaderEngine
    G, n, f, data_len, k = 300, 5, 1, 700, 9
    kw = dict(rs_total_shards=5, rs_data_shards=3) if protocol == "crossword" else {}
    engs = [LeaderEngine(ctx, protocol, G, n, f, data_len, **kw) for _ in range(2)]
    bal = np.arange(7, G + 7, dtype=np.uint64)
    rng = np.random.default_rng(5)
    for e in engs:
        e.set_prepared_ballots(_t(bal))
        if protocol == "crossword":
            e.set_policies([list(map(int, oracle.cw_brr_assignment(n, 5, spr))) for spr in (1, 2, 3)], True)
    for i in range(k):
        payload = _t(wl.payload_uniform(G, data_len, seed_extra=40 + i))
        pol = _t(rng.integers(0, 3, G).astype(np.uint8)) if protocol == "crossword" else None
        slot_out, _ = engs[0].propose_next(0, payload, pol)
        engs[1].propose(i, payload, pol)
        torch.cuda.synchronize()
        assert (_u64(slot_out) == i).all()
    names = ["planes", "bal_prepared", "inst_bal", "accepting", "committed", "commit_bar", "shards", "window_base"]
    if protocol == "crossword":
        names.append("policy_idx")
    for name in names:
        assert torch.equal(getattr(engs[0], name), getattr(engs[1], name)), name
    for e in engs:
        e.close()


@pytest.mark.gpu
def test_engine_window_errors(ctx):
    """Raft engines and out-of-range shard stores are rejected with SS_ERR_INVALID_ARG."""
    from summerset_b200.engine import LeaderEngine, RaftEngine
    raft = RaftEngine(ctx, 16, 5)
    lib = raft.lib
    out = C.c_void_p()
    assert lib.ss_engine_propose_next(raft.h, 0, None, 0, None, None, None) == _lib.SS_ERR_INVALID_ARG
    assert lib.ss_engine_advance(raft.h, None) == _lib.SS_ERR_INVALID_ARG
    assert lib.ss_engine_window_get(raft.h, C.byref(out)) == _lib.SS_ERR_INVALID_ARG
    raft.close()
    eng = LeaderEngine(ctx, "rspaxos", 16, 5, 1, 64, keep_slots=3)
    with pytest.raises(SummersetError) as ei:
        eng.propose_next(3, _t(np.zeros((16, 64), dtype=np.uint8)))
    assert ei.value.code == _lib.SS_ERR_INVALID_ARG
    eng.close()


def test_engine_window_calls_reject_null_engine():
    lib = _lib.load()
    out = C.c_void_p()
    assert lib.ss_engine_propose_next(None, 0, None, 0, None, None, None) == _lib.SS_ERR_INVALID_ARG
    assert lib.ss_engine_advance(None, None) == _lib.SS_ERR_INVALID_ARG
    assert lib.ss_engine_window_get(None, C.byref(out)) == _lib.SS_ERR_INVALID_ARG
