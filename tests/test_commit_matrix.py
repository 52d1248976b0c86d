"""The commit side at every population, window and grid size the C ABI accepts: the Paxos-family engine tick
(summerset_b200/csrc/engine.cu) at populations 1-12 with every tick kernel instance, the Raft scan's window_overflow
counter, the grid-stride loops of the engine, ingest and tally kernels past their grid cap, and what an out-of-range
policy_idx does in each call.  Everything is checked against the CPU oracle's per-message handlers (oracle/ss_oracle.c)
or a numpy restatement built on its batch calls.
"""
import re

import numpy as np
import pytest
import torch

from summerset_b200 import workloads as wl
from summerset_b200._lib import SummersetError

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
S = 256                                     # model slots: slot m of the oracle state is absolute slot m
ERR_TOO_FEW_PARITY_SHARDS, ERR_INVALID_ARG = -5, -20
CW_DATA_LEN = 200


def _t(a):
    a = np.ascontiguousarray(a)
    if a.dtype == np.uint64:
        a = a.view(np.int64)
    elif a.dtype == np.uint32:
        a = a.view(np.int32)
    elif a.dtype == np.uint16:
        a = a.view(np.int16)
    return torch.from_numpy(a).to(DEV)


def _u64(t):
    return t.cpu().numpy().view(np.uint64)


def _u32(t):
    return t.cpu().numpy().view(np.uint32)


def _ring_to_window(x, base):
    r = np.asarray(base).astype(np.uint64) & np.uint64(63)
    return (x >> r) | (x << ((np.uint64(64) - r) & np.uint64(63)))


def _prefix(x):
    """commit_bar of window words: the number of trailing one bits"""
    y = ~np.asarray(x, dtype=np.uint64)
    low = y & (~y + np.uint64(1))
    return np.where(y == 0, 64, np.log2(np.maximum(low, np.uint64(1)).astype(np.float64))).astype(np.uint32)


def _grid_cap_threads():
    """threads of the capped grid eng_grid / stream_grid launch: 32 CTAs of 256 threads per SM"""
    return torch.cuda.get_device_properties(0).multi_processor_count * 32 * 256


def _policies(oracle, rng, n, T, d, balanced):
    dj = T // n
    if balanced:
        return np.stack([oracle.cw_brr_assignment(n, T, spr) for spr in range(dj, d + 1, dj)])
    return np.stack([oracle.cw_brr_assignment(n, T, d)] + [rng.integers(1, 1 << T, size=n).astype(np.uint32) for _ in range(3)])


# ---- Paxos-family engine matrix -----------------------------------------------------------------------------------
def _engine_configs():
    cfgs = [("multipaxos", n, 0, None) for n in range(1, 13)]
    cfgs += [("rspaxos", n, (n - n // 2 - 1) // 2, None) for n in range(3, 13)]
    cfgs += [("crossword", n, (n - n // 2 - 1) // 2, (n, n // 2 + 1, n % 2 == 1)) for n in range(3, 13)]
    # T = 24, d = 16: the engine's uniform encoder takes at most 8 parity shards
    cfgs += [("crossword", 6, 1, (12, 7, True)), ("crossword", 12, 1, (24, 16, False))]
    return cfgs


# G parity, whether the host fetched window_base (and advances), and the alignment of the tick's newly buffer: an even
# G with a 16-byte aligned (or absent) buffer takes the two-groups-per-thread tick, the others the scalar one
LAYOUTS = [("odd", False, 16), ("odd", True, 16), ("even", False, 16), ("even", True, 16), ("even", False, 8), ("even", True, 8)]


class _Model:
    """Oracle state [G, S] at absolute slots; mb = window base, top = one past the highest proposed slot."""

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


def _replies(rng, model, n, nrec):
    """AcceptReplies at absolute slots: mostly to proposed instances (duplicates included), some to retired or
    never-proposed slots, stale ballots and out-of-range peers.  Returns the engine's records (window-relative slots;
    0xff outside the window) and the oracle's (absolute slots)."""
    G = model.G
    rg = rng.integers(0, G, nrec).astype(np.uint32)
    lo, hi = model.mb[rg], model.top[rg]
    slot = lo + rng.integers(0, 1 << 30, nrec) % np.maximum(hi - lo, 1)
    r = rng.random(nrec)
    slot[r < 0.05] = np.maximum(lo[r < 0.05] - 1, 0)
    fresh = (r >= 0.05) & (r < 0.1)
    slot[fresh] = np.minimum(hi[fresh] + rng.integers(0, 70, int(fresh.sum())), S - 1)
    peer = rng.integers(0, n + 1, nrec).astype(np.uint8)        # n = out-of-range peer
    ballot = model.bal[rg].copy()
    stale = rng.random(nrec) < 0.08
    ballot[stale] += rng.integers(1, 3, int(stale.sum())).astype(np.uint64)
    rel = slot - lo
    rel_u8 = np.where((rel >= 0) & (rel < 64), rel, 0xFF).astype(np.uint8)
    return (rg, rel_u8, peer, ballot), (rg, slot.astype(np.uint8), peer, ballot)


@pytest.mark.parametrize("layout", LAYOUTS, ids=[f"{p}-{'win' if w else 'nowin'}-al{a}" for p, w, a in LAYOUTS])
@pytest.mark.parametrize("protocol,n,f,cw", _engine_configs(),
                         ids=[f"{p}-n{n}" + (f"-T{c[0]}" if c else "") for p, n, f, c in _engine_configs()])
def test_paxos_engine_matrix(ctx, oracle, protocol, n, f, cw, layout):
    """Proposals at each group's first Null slot, two AcceptReply batches per round, each ingested and ticked:
    committed, accepting, commit_bar and newly equal the per-message handler's state bit for bit.  Windowed runs
    retire committed prefixes between rounds, so the tick reads non-zero bases."""
    from summerset_b200.engine import LeaderEngine
    parity, windowed, align = layout
    rng = np.random.default_rng(n * 1000 + len(protocol) * 10 + (cw[0] if cw else 0) + 7 * windowed + align)
    G = 1000 if parity == "even" else 1001
    majority = n // 2 + 1
    policies, T, d, balanced = None, 0, 0, True
    if protocol == "crossword":
        T, d, balanced = cw
        eng = LeaderEngine(ctx, protocol, G, n, f, CW_DATA_LEN, rs_total_shards=T, rs_data_shards=d)
        policies = _policies(oracle, rng, n, T, d, balanced)
        eng.set_policies([list(map(int, q)) for q in policies], balanced)
    else:
        eng = LeaderEngine(ctx, protocol, G, n, f, CW_DATA_LEN if protocol == "rspaxos" else 0)
    thr = majority + f if protocol == "rspaxos" else majority
    assert eng.threshold == (0 if protocol == "crossword" else thr)
    bal = rng.integers(1, 1 << 30, G).astype(np.uint64)
    eng.set_prepared_ballots(_t(bal))
    if windowed:
        assert (_u64(eng.window_base) == 0).all()              # fetching the bases switches the tick to reading them
    model = _Model(G, bal)
    buf = torch.zeros(G + 2, dtype=torch.int64, device=DEV)
    newly = buf[:G] if align == 16 else buf[1:G + 1]
    assert newly.data_ptr() % 16 == (0 if align == 16 else 8)
    if protocol == "crossword":
        tally = lambda rg, rs_, rp, rb: oracle.tally_stream_crossword(
            rg, rs_, rp, rb, S, n, T, d, majority, f, balanced, policies, model.pidx, model.bal, model.inst_bal, model.status, model.acks)
    else:
        tally = lambda rg, rs_, rp, rb: oracle.tally_stream(rg, rs_, rp, rb, S, n, thr, model.bal, model.inst_bal, model.status, model.acks)
    proposed = 0
    for rnd in range(5):
        for k in range(int(rng.integers(1, 4))):
            want = model.first_null(oracle)
            pol = np.zeros(G, dtype=np.uint8)
            if policies is not None:
                pol = rng.integers(0, len(policies), G).astype(np.uint8)
                bad = rng.random(G) < 0.05
                pol[bad] = rng.integers(len(policies), 256, int(bad.sum()))     # out of range: never commits
            payload = _t(wl.payload_uniform(G, CW_DATA_LEN, seed_extra=10 * rnd + k)) if protocol != "multipaxos" else None
            slot_out, _ = eng.propose_next(0, payload, _t(pol) if policies is not None else None)
            torch.cuda.synchronize()
            assert (want >= 0).all()
            assert (_u64(slot_out) == want.astype(np.uint64)).all(), (rnd, k)
            model.propose(oracle, want, pol)
            proposed += G
        for _ in range(2):
            recs, orecs = _replies(rng, model, n, 3 * G * (n + 1))
            before = model.window(oracle.ST_COMMITTED)
            eng.on_accept_replies(_t(recs[0]), _t(recs[1]), _t(recs[2]), _t(recs[3]))
            committed, bar = eng.tick(newly)
            torch.cuda.synchronize()
            tally(*orecs)
            want_c = model.window(oracle.ST_COMMITTED)
            wb = model.mb.astype(np.uint64)
            assert (_ring_to_window(_u64(committed), wb) == want_c).all(), rnd
            assert (_ring_to_window(_u64(eng.accepting), wb) == model.window(oracle.ST_ACCEPTING)).all(), rnd
            assert (_u64(newly) == (want_c & ~before)).all(), rnd
            assert (_u32(bar) == _prefix(want_c)).all(), rnd
        assert buf[0 if align == 8 else G].item() == 0 and buf[G + 1].item() == 0      # no write outside newly
        if windowed and rnd % 2 == 1:
            bar_m = _prefix(model.window(oracle.ST_COMMITTED)).astype(np.int64)
            eng.advance()
            model.mb += bar_m
            torch.cuda.synchronize()
            assert (_u64(eng.window_base) == model.mb.astype(np.uint64)).all()
    frac = (model.status == oracle.ST_COMMITTED).sum() / proposed
    assert 0.05 < frac <= 1.0, frac
    if windowed:
        assert model.mb.max() > 0
    eng.close()


@pytest.mark.parametrize("protocol,n", [("rspaxos", 1), ("rspaxos", 2), ("crossword", 1), ("crossword", 2)])
def test_rs_engines_refuse_populations_without_parity(ctx, protocol, n):
    """RSPaxos codes (majority, n - majority): at n = 1, 2 there is no parity shard, and ReedSolomon::new fails
    (SS_ERR_TOO_FEW_PARITY_SHARDS).  Crossword's default code (T = n, d = majority) has d >= T there
    (SS_ERR_INVALID_ARG, crossword/mod.rs:805-830)."""
    from summerset_b200.engine import LeaderEngine
    with pytest.raises(SummersetError) as e:
        LeaderEngine(ctx, protocol, 64, n, 0, CW_DATA_LEN)
    assert e.value.code == (ERR_TOO_FEW_PARITY_SHARDS if protocol == "rspaxos" else ERR_INVALID_ARG)


# ---- every tick instance runs ---------------------------------------------------------------------------------------
def test_tick_dispatch_reaches_every_instance(ctx, oracle):
    """One tick per engine tick kernel instance, one stateless scan per raft_scan_kernel instance and one Raft engine
    tick per engine_raft_snap_kernel instance, recorded with torch.profiler."""
    from torch.profiler import ProfilerActivity, profile

    from summerset_b200.engine import LeaderEngine, RaftEngine
    engines = []
    for n, G, win, proto in [(3, 64, False, "multipaxos"), (3, 64, True, "multipaxos"), (5, 64, False, "multipaxos"),
                             (5, 64, True, "multipaxos"), (7, 64, False, "multipaxos"), (7, 64, True, "multipaxos"),
                             (4, 64, False, "multipaxos"), (4, 64, True, "multipaxos"), (4, 63, False, "multipaxos"),
                             (4, 63, True, "multipaxos"), (5, 64, False, "crossword"), (5, 64, True, "crossword")]:
        e = LeaderEngine(ctx, proto, G, n, 0, CW_DATA_LEN if proto == "crossword" else 0)
        if proto == "crossword":
            e.set_policies([list(map(int, oracle.cw_brr_assignment(n, n, 3)))], True)
        if win:
            e.window_base.fill_(5)
        engines.append(e)
    rafts = [RaftEngine(ctx, 64, pop, 0, False, 64) for pop in (4, 8, 12)]
    w = {P: wl.cfg5_raft(64, P + 1, 64, seed_extra=P) for P in (2, 4, 6, 8, 16)}
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for e in engines:
            e.tick()
        for r in rafts:
            r.tick()
        for P, x in w.items():
            ctx.raft_commit_scan(_t(x["match"]), _t(x["last_commit"]), _t(x["log_end"]), _t(x["curr_term"]), _t(x["terms"]), 2)
        torch.cuda.synchronize()
    names = {re.sub(r"\s+", "", ev.name) for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA}
    if not any("kernel" in s for s in names):
        pytest.skip("torch.profiler recorded no CUDA kernels on this machine")
    want = [f"engine_tick_x2_kernel<{r},{w}>" for r in (3, 5, 7, 0) for w in ("false", "true")]
    want += [f"engine_tick_kernel<{w}>" for w in ("false", "true")]
    want += [f"engine_tick_crossword_kernel<{w}>" for w in ("false", "true")]
    want += [f"raft_scan_kernel<{p}>" for p in (2, 4, 6, 8, 16)]
    want += [f"engine_raft_snap_kernel<{p}>" for p in (4, 8, 16)]
    missing = [k for k in want if not any(k in s for s in names)]
    assert not missing, (missing, sorted(names))
    for e in engines + rafts:
        e.close()


# ---- window_overflow ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("W", [16, 7])
def test_raft_scan_window_overflow(ctx, oracle, W):
    """Groups whose candidate range min(kth_match, log_end - 1) - last_commit exceeds W are counted; their new_commit
    is the scan over the W entries the kernel can examine (log_end clamped to last_commit + 1 + W); the other groups
    are unaffected.  W % 4 == 0 takes the vectorised walk, W % 4 != 0 the cooperative one."""
    rng = np.random.default_rng(W)
    G, P, thr = 5000, 6, 4
    last_commit = rng.integers(0, 1 << 20, G).astype(np.uint32)
    over = rng.random(G) < 0.3
    extra = np.where(over, rng.integers(1, 3 * W, G), -rng.integers(0, W, G))
    log_end = (last_commit.astype(np.int64) + 1 + W + extra).astype(np.uint32)
    match = (last_commit[None, :] + rng.integers(0, 4 * W, (P, G))).astype(np.uint32)
    curr_term = rng.integers(3, 100, G).astype(np.uint32)
    terms = np.where(rng.random((G, W)) < 0.6, curr_term[:, None], curr_term[:, None] - 1).astype(np.uint32)
    cnt = torch.zeros(1, dtype=torch.int32, device=DEV)
    out = ctx.raft_commit_scan(_t(match), _t(last_commit), _t(log_end), _t(curr_term), _t(terms), thr, window_overflow=cnt)
    torch.cuda.synchronize()
    kth = -np.sort(-match.astype(np.int64), axis=0)[thr - 2]
    upper = np.minimum(kth, log_end.astype(np.int64) - 1)
    want_cnt = int(((upper - last_commit) > W).sum())
    assert 0 < want_cnt < G
    assert int(cnt.item()) == want_cnt
    clamped = np.minimum(log_end, last_commit + np.uint32(1 + W)).astype(np.uint32)
    want = oracle.raft_scan_batch(match, last_commit, clamped, curr_term, terms, thr)
    got = _u32(out)
    assert (got == want).all()
    inside = log_end.astype(np.int64) - last_commit - 1 <= W
    assert (got[inside] == oracle.raft_scan_batch(match, last_commit, log_end, curr_term, terms, thr)[inside]).all()


# ---- past the grid cap ----------------------------------------------------------------------------------------------
def test_multipaxos_tick_advance_propose_past_grid_cap(ctx, oracle):
    """G = 2 * cap + 1 groups (odd: the scalar tick) with random installed state: one tick, one advance and one
    propose_next, each against a numpy model."""
    from summerset_b200.engine import LeaderEngine
    cap = _grid_cap_threads()
    assert ctx.sm_count * 32 * 256 == cap
    G, n, rng = 2 * cap + 1, 5, np.random.default_rng(11)
    eng = LeaderEngine(ctx, "multipaxos", G, n)
    planes = rng.integers(0, 1 << 63, (n, G), dtype=np.uint64) | rng.integers(0, 1 << 63, (n, G), dtype=np.uint64)
    cm0 = rng.integers(0, 1 << 63, G, dtype=np.uint64) & rng.integers(0, 1 << 63, G, dtype=np.uint64)
    base = rng.integers(0, 1 << 40, G).astype(np.uint64)
    eng.planes.copy_(_t(planes)); eng.committed.copy_(_t(cm0)); eng.accepting.fill_(-1)
    eng.window_base.copy_(_t(base))
    newly = torch.zeros(G, dtype=torch.int64, device=DEV)
    eng.tick(newly)
    torch.cuda.synchronize()
    tw, _ = oracle.tally_planes(planes, n // 2 + 1)
    cm = cm0 | tw
    assert (_u64(eng.committed) == cm).all()
    assert (_u64(eng.accepting) == ~tw).all()
    assert (_u64(newly) == _ring_to_window(tw, base)).all()
    bar = _prefix(_ring_to_window(cm, base))
    assert (_u32(eng.commit_bar) == bar).all()
    del newly
    eng.advance()
    torch.cuda.synchronize()
    # the retired prefix is cleared from every per-slot word; the window moves past it
    base2 = base + bar.astype(np.uint64)
    k = bar.astype(np.uint64)
    keep_w = np.where(k == 64, np.uint64(0), ~np.uint64(0) << np.minimum(k, np.uint64(63)))
    keep = _ring_to_window(keep_w, (np.uint64(64) - (base & np.uint64(63))) & np.uint64(63))     # window -> ring
    acc2, cm2 = ~tw & keep, cm & keep
    assert (_u64(eng.window_base) == base2).all() and (_u32(eng.commit_bar) == 0).all()
    assert (_u64(eng.accepting) == acc2).all() and (_u64(eng.committed) == cm2).all()
    assert (_u64(eng.planes) == planes & keep[None, :]).all()
    slot_out, _ = eng.propose_next(0, None)
    full_status = ctx.device_status()
    rel = _prefix(_ring_to_window(acc2 | cm2, base2)).astype(np.uint64)
    want = np.where(rel == 64, ~np.uint64(0), base2 + rel)
    assert (_u64(slot_out) == want).all()
    assert full_status == (8 if (rel == 64).any() else 0)          # SS_DEV_STATUS_WINDOW_FULL
    eng.close()


def test_crossword_tick_past_grid_cap(ctx, oracle):
    """One Crossword tick over 2 * cap + 1 groups with random planes, accepting words and policy indices (some out of
    range): the commit bits are a vectorised look-up of the oracle's predicate."""
    from summerset_b200.engine import LeaderEngine
    cap = _grid_cap_threads()
    G, n, T, d, f, rng = 2 * cap + 1, 5, 5, 3, 1, np.random.default_rng(12)
    eng = LeaderEngine(ctx, "crossword", G, n, f, 1)
    policies = _policies(oracle, rng, n, T, d, False)
    K = len(policies)
    eng.set_policies([list(map(int, q)) for q in policies], False)
    planes = rng.integers(0, 1 << 63, (n, G), dtype=np.uint64) | rng.integers(0, 1 << 63, (n, G), dtype=np.uint64)
    acc = rng.integers(0, 1 << 63, G, dtype=np.uint64) | rng.integers(0, 1 << 63, G, dtype=np.uint64)
    pidx = rng.integers(0, K + 1, G * 64).astype(np.uint8)
    eng.planes.copy_(_t(planes)); eng.accepting.copy_(_t(acc)); eng.policy_idx.copy_(torch.from_numpy(pidx).to(DEV))
    eng.tick()
    torch.cuda.synchronize()
    # row K: an out-of-range policy never commits
    lut = np.array([[oracle.cw_committed(T, n, d, n // 2 + 1, f, a, policies[k], False) for a in range(1 << n)]
                    for k in range(K)] + [[False] * (1 << n)], dtype=bool)
    bits = lambda w: np.unpackbits(w.view(np.uint8).reshape(G, 8), axis=1, bitorder="little")      # [G, 64], bit s
    ack = np.zeros((G, 64), dtype=np.uint16)
    for r in range(n):
        ack |= bits(planes[r]).astype(np.uint16) << r
    ok = lut[pidx.reshape(G, 64), ack] & (bits(acc) == 1)
    del ack
    tw = np.packbits(ok, axis=1, bitorder="little").view(np.uint64).reshape(-1)
    assert (_u64(eng.committed) == tw).all()
    assert (_u64(eng.accepting) == acc & ~tw).all()
    assert (_u32(eng.commit_bar) == _prefix(tw)).all()
    eng.close()


def test_raft_append_ingest_tick_past_grid_cap(ctx, oracle):
    """One append, one ingest of 3 * (2 * cap + 1) AppendEntriesReplies and one tick over 2 * cap + 1 Raft groups, against
    the per-record handler."""
    from summerset_b200.engine import RaftEngine
    cap = _grid_cap_threads()
    G, pop, W, rng = 2 * cap + 1, 5, 8, np.random.default_rng(13)
    P, thr = pop - 1, pop // 2 + 1
    eng = RaftEngine(ctx, G, pop, 0, False, W)
    curr_term = rng.integers(2, 9, G).astype(np.uint32)
    eng.curr_term.copy_(_t(curr_term))
    n_new = rng.integers(0, W + 1, G).astype(np.uint32)
    eng.append(_t(n_new))
    log_end = (1 + n_new).astype(np.uint32)
    terms = np.zeros((G, W), dtype=np.uint32)
    wrote = ((np.arange(W)[None, :] - 1) & (W - 1)) < n_new[:, None]
    terms[wrote] = np.broadcast_to(curr_term[:, None], terms.shape)[wrote]
    torch.cuda.synchronize()
    assert (_u32(eng.log_end) == log_end).all() and (_u32(eng.terms) == terms).all()
    nrec = 3 * G
    rg = rng.integers(0, G, nrec).astype(np.uint32)
    rp = rng.integers(0, P + 1, nrec).astype(np.uint8)
    rend = (rng.integers(0, 1 << 30, nrec) % log_end[rg]).astype(np.uint32)
    eng.on_append_replies(_t(rg), torch.from_numpy(rp).to(DEV), _t(rend))
    lc, ls = eng.tick()
    torch.cuda.synchronize()
    next_slot = np.ones((P, G), dtype=np.uint32); match = np.zeros((P, G), dtype=np.uint32)
    last_commit = np.zeros(G, dtype=np.uint32); last_snap = np.zeros(G, dtype=np.uint32)
    oracle.raft_reply_stream(rg, rp, rend, P, thr, next_slot, match, last_commit, last_snap, log_end, curr_term, terms)
    assert (_u32(eng.next_slot) == next_slot).all() and (_u32(eng.match) == match).all()
    assert (_u32(lc) == last_commit).all() and (_u32(ls) == last_snap).all()
    assert (last_commit > 0).mean() > 0.1 and (last_snap > 0).any()
    eng.close()


def test_ack_ingest_past_grid_cap(ctx, oracle):
    """ss_ack_ingest_dev over 2 * cap + 1 records: the planes hold exactly the records that pass the handler's filters,
    and their tally equals the per-ack handler's."""
    cap = _grid_cap_threads()
    G, R, thr, rng = 50000, 5, 3, np.random.default_rng(14)
    nrec = 2 * cap + 1
    bal = rng.integers(1, 1 << 30, G).astype(np.uint64)
    # inst.bal: mostly the prepared ballot or below it, sometimes above (the reply is then dropped)
    inst_bal = (bal[:, None] - rng.integers(0, 2, (G, 64)).astype(np.uint64) + (rng.random((G, 64)) < 0.05)).reshape(-1)
    accepting = rng.integers(0, 1 << 63, G, dtype=np.uint64) | rng.integers(0, 1 << 63, G, dtype=np.uint64)
    rg = rng.integers(0, G + 2, nrec).astype(np.uint32)
    rs_ = rng.integers(0, 66, nrec).astype(np.uint8)
    rp = rng.integers(0, R + 1, nrec).astype(np.uint8)
    rb = bal[np.minimum(rg, G - 1)] + (rng.random(nrec) < 0.05).astype(np.uint64)
    planes = torch.zeros((R, G), dtype=torch.int64, device=DEV)
    ctx.ack_ingest(_t(rg), _t(rs_), _t(rp), _t(rb), _t(bal), _t(inst_bal), _t(accepting), R, planes)
    torch.cuda.synchronize()
    g = np.minimum(rg, G - 1).astype(np.int64)
    s = np.minimum(rs_, 63).astype(np.uint64)
    ok = (rg < G) & (rs_ < 64) & (rp < R) & (rb == bal[g]) & (((accepting[g] >> s) & np.uint64(1)) == 1) & \
         (rb >= inst_bal[g * 64 + s.astype(np.int64)])
    want = np.zeros((R, G), dtype=np.uint64)
    np.bitwise_or.at(want, (rp[ok].astype(np.int64), g[ok]), np.uint64(1) << s[ok])
    assert (_u64(planes).reshape(R, G) == want).all()
    status = np.where(np.unpackbits(accepting.view(np.uint8).reshape(G, 8), axis=1, bitorder="little").reshape(-1) == 1,
                      oracle.ST_ACCEPTING, oracle.ST_NULL).astype(np.uint8)
    acks = np.zeros(G * 64, dtype=np.uint16)
    inb = (rg < G) & (rs_ < 64)                                   # the oracle indexes without bounds checks
    oracle.tally_stream(rg[inb], rs_[inb], rp[inb], rb[inb], 64, R, thr, bal, inst_bal, status, acks)
    c, _ = ctx.tally_planes(planes, thr)
    torch.cuda.synchronize()
    assert (_u64(c) == np.packbits(status.reshape(G, 64) == oracle.ST_COMMITTED, axis=1, bitorder="little").view(np.uint64).reshape(-1)).all()


@pytest.mark.parametrize("width", [1, 2])
def test_tally_masks_past_grid_cap(ctx, oracle, width):
    """tally_masks over more instances than the capped grid covers in one pass: 16 (8-bit masks) or 8 (16-bit masks)
    instances per thread."""
    cap = _grid_cap_threads()
    rng = np.random.default_rng(15 + width)
    n = (16 if width == 1 else 8) * cap + 77
    masks = rng.integers(0, 1 << (8 if width == 1 else 13), n).astype(np.uint8 if width == 1 else np.uint16)
    thr = 4
    bits = ctx.tally_masks(_t(masks), thr)
    torch.cuda.synchronize()
    got = np.unpackbits(bits.cpu().numpy().view(np.uint8), bitorder="little")
    assert (got[:n] == oracle.tally_masks(masks.astype(np.uint16), thr)).all()
    assert (got[n:] == 0).all()


# ---- out-of-range policy_idx ----------------------------------------------------------------------------------------
def test_out_of_range_policy_frames_and_gossip_use_policy_0(ctx, oracle):
    """The Accept packer and the gossip planner treat policy_idx >= n_policies as policy 0 (the tally and the engine
    tick never commit such an instance: test_crossword_matches_oracle, test_paxos_engine_matrix)."""
    rng = np.random.default_rng(16)
    n_rep, T, d, p, N, data_len = 5, 10, 6, 4, 257, 700
    policies = [list(map(int, oracle.cw_brr_assignment(n_rep, T, spr))) for spr in (2, 4, 6)]
    pidx = rng.integers(0, 3, N).astype(np.uint8)
    bad = rng.random(N) < 0.3
    pidx[bad] = rng.integers(3, 256, int(bad.sum()))
    as0 = np.where(bad, 0, pidx).astype(np.uint8)
    L = oracle.cw_shard_len(data_len, d)
    planes = torch.from_numpy(rng.integers(0, 256, (T, N, (L + 15) // 16 * 16)).astype(np.uint8)).to(DEV)
    slot = _t(rng.integers(0, 1 << 40, N).astype(np.uint64))
    ballot = _t(rng.integers(1, 1 << 40, N).astype(np.uint64))
    for peer in (0, 3):
        a = ctx.frame_accept_pack(planes, data_len, d, p, policies, _t(pidx), peer, slot, ballot, with_assignment=True)
        b = ctx.frame_accept_pack(planes, data_len, d, p, policies, _t(as0), peer, slot, ballot, with_assignment=True)
        torch.cuda.synchronize()
        for x, y in zip(a, b):
            assert torch.equal(x, y)
    me, alive = 1, 0b11011
    src = rng.integers(0, n_rep, N).astype(np.uint8)
    avail = rng.integers(0, 1 << T, N).astype(np.uint32)
    targets, excl = ctx.gossip_plan(me, n_rep, d, _t(src), _t(avail), _t(pidx), policies, alive)
    torch.cuda.synchronize()
    targets = _u32(targets); excl = _u32(excl)
    for i in np.nonzero(bad)[0]:
        wt, we = oracle.gossip_targets_excl(me, n_rep, d, int(src[i]), int(avail[i]), policies[0], alive)
        assert int(targets[i]) == wt
        for peer in range(n_rep):
            assert int(excl[peer, i]) == (int(we[peer]) if (wt >> peer) & 1 else 0xFFFFFFFF)
