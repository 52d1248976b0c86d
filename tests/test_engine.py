"""The batched consensus engine behind the C ABI (ss_engine_*: summerset_b200/csrc/engine.cu, bound by
summerset_b200/engine.py) over several ticks vs the oracle's incremental per-message handlers on the identical
interleaved stream.

Paxos family: proposals enter Accepting, AcceptReplies (with duplicates, stale ballots, replies for instances not yet
proposed or already committed, out-of-range peers) arrive in batches; commit words, commit_bar, the newly-committed
words and every shard plane must match bit for bit
  MultiPaxos  multipaxos/request.rs:112-221, multipaxos/messages.rs:370-443, multipaxos/durability.rs:148-218
  RSPaxos     rspaxos/request.rs:72-142, rspaxos/messages.rs:395-465
  Crossword   crossword/request.rs:82-185, crossword/messages.rs:15-62,481-574 (balanced and unbalanced assignments)
Raft / CRaft: appends, batches of successful AppendEntriesReplies, commit scan + last_snap
  raft/messages.rs:243-309, craft/messages.rs:300-308
"""
import numpy as np
import pytest
import torch

from summerset_b200 import workloads as wl

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _t(a):
    a = np.ascontiguousarray(a)
    if a.dtype == np.uint64:
        a = a.view(np.int64)
    elif a.dtype == np.uint32:
        a = a.view(np.int32)
    return torch.from_numpy(a).to(DEV)


def _reply_stream(rng, G, population, bal, nrec):
    rg = rng.integers(0, G, nrec).astype(np.uint32)
    cand = np.array([0, 1, 2, 3, 63, 5, 40], dtype=np.uint8)       # 5 and 40 are never proposed
    rs_ = cand[rng.integers(0, len(cand), nrec)]
    rp = rng.integers(0, population + 1, nrec).astype(np.uint8)    # population = out-of-range peer
    rb = bal[rg].copy()
    stale = rng.random(nrec) < 0.08
    rb[stale] += rng.integers(1, 3, int(stale.sum())).astype(np.uint64)
    return rg, rs_, rp, rb


def _words(status, G, S, oracle):
    return np.packbits(status.reshape(G, S) == oracle.ST_COMMITTED, axis=1, bitorder="little").view(np.uint64).reshape(-1)


@pytest.mark.parametrize("protocol,population,f,data_len", [
    ("rspaxos", 5, 1, 4096), ("rspaxos", 5, 0, 300), ("rspaxos", 7, 1, 1000), ("rspaxos", 3, 0, 64),
    ("multipaxos", 5, 0, 0), ("multipaxos", 3, 0, 0), ("multipaxos", 7, 0, 0), ("multipaxos", 4, 0, 0)])
def test_engine_multi_tick_matches_incremental_handlers(ctx, oracle, protocol, population, f, data_len):
    from summerset_b200.engine import LeaderEngine
    rng = np.random.default_rng(population * 10 + f + (7 if protocol == "multipaxos" else 0))
    G, S = 1200 if population != 4 else 1201, 64            # odd G exercises the one-group-per-thread tick kernel
    eng = LeaderEngine(ctx, protocol, G, population, f, data_len)
    majority = population // 2 + 1
    d, p = majority, population - majority
    thr = majority + f if protocol == "rspaxos" else majority           # rspaxos/messages.rs:438-440 / multipaxos/mod.rs:774
    assert eng.threshold == thr
    bal = rng.integers(1, 1 << 30, G).astype(np.uint64)
    eng.set_prepared_ballots(_t(bal))
    status = np.zeros(G * S, dtype=np.uint8)
    acks = np.zeros(G * S, dtype=np.uint16)
    inst_bal = np.zeros(G * S, dtype=np.uint64)
    newly = torch.zeros(G + 2, dtype=torch.int64, device=DEV)[:G] if G % 2 == 0 else torch.zeros(G, dtype=torch.int64, device=DEV)
    n_rounds = 5
    for rnd in range(n_rounds):
        slot = rnd if rnd < 4 else 63                      # also exercise the top bit of the window
        if protocol == "rspaxos":
            payload = wl.payload_uniform(G, data_len, seed_extra=100 + rnd)
            sh = eng.propose(slot, _t(payload))
            torch.cuda.synchronize()
            # --- shard planes: data shards are the contiguous split, parity is the oracle's
            L = oracle.cw_shard_len(data_len, d)
            got = sh.cpu().numpy()
            assert (got[d:] == oracle.rs_encode_uniform(d, p, payload, data_len)).all()
            for g in (0, 1, G // 2, G - 1):
                assert (got[:d, g, :L] == oracle.cw_split(payload[g, :data_len].tobytes(), d)).all()
            assert (got[:d, :, L:] == 0).all()
        else:
            assert eng.propose(slot, None) is None          # MultiPaxos replicates the whole batch: nothing to code
        # --- oracle: the instance enters Accepting
        status.reshape(G, S)[:, slot] = oracle.ST_ACCEPTING
        acks.reshape(G, S)[:, slot] = 0
        inst_bal.reshape(G, S)[:, slot] = bal
        rg, rs_, rp, rb = _reply_stream(rng, G, population, bal, 40000)
        for half in range(2):
            sl = slice(half * 20000, (half + 1) * 20000)
            before = _words(status, G, S, oracle)
            eng.on_accept_replies(_t(rg[sl]), torch.from_numpy(rs_[sl]).to(DEV), torch.from_numpy(rp[sl]).to(DEV), _t(rb[sl]))
            committed, bar = eng.tick(newly)
            torch.cuda.synchronize()
            oracle.tally_stream(rg[sl], rs_[sl], rp[sl], rb[sl], S, population, thr, bal, inst_bal, status, acks)
            want = _words(status, G, S, oracle)
            assert (committed.cpu().numpy().view(np.uint64) == want).all(), (rnd, half)
            assert (newly.cpu().numpy().view(np.uint64) == (want & ~before)).all(), "newly-committed words"
            want_bar = np.array([oracle.commit_bar(int(w)) for w in want], dtype=np.uint32)
            assert (bar.cpu().numpy().view(np.uint32) == want_bar).all()
            # committed instances have left Accepting; the others are still in it
            acc = eng.accepting.cpu().numpy().view(np.uint64)
            want_acc = np.packbits(status.reshape(G, S) == oracle.ST_ACCEPTING, axis=1, bitorder="little").view(np.uint64).reshape(-1)
            assert (acc == want_acc).all()
    frac = (status == oracle.ST_COMMITTED).sum() / (G * n_rounds)
    assert 0.2 < frac <= 1.0
    eng.close()


@pytest.mark.parametrize("population,T,d,f,balanced", [(5, 5, 3, 2, True), (5, 5, 3, 1, True), (5, 10, 6, 1, True),
                                                      (7, 7, 4, 2, True), (5, 5, 3, 1, False), (3, 3, 2, 0, True)])
def test_crossword_engine_matches_incremental_handler(ctx, oracle, population, T, d, f, balanced):
    """crossword/messages.rs:481-574 with per-instance assignment policies (balanced round-robin with every spr, or
    unbalanced bitmask assignments through the subset-enumeration branch)."""
    from summerset_b200.engine import LeaderEngine
    rng = np.random.default_rng(T * 100 + d * 10 + f)
    G, S, data_len = 900, 64, 1500
    majority = population // 2 + 1
    dj = T // population
    if balanced:
        policies = np.stack([oracle.cw_brr_assignment(population, T, spr) for spr in range(dj, d + 1, dj)])
    else:
        policies = np.stack([oracle.cw_brr_assignment(population, T, d)] +
                            [rng.integers(1, 1 << T, size=population).astype(np.uint32) for _ in range(3)])
    K = policies.shape[0]
    eng = LeaderEngine(ctx, "crossword", G, population, f, data_len, rs_total_shards=T, rs_data_shards=d)
    assert (eng.T, eng.d) == (T, d)
    eng.set_policies([list(map(int, q)) for q in policies], balanced)
    bal = rng.integers(1, 1 << 30, G).astype(np.uint64)
    eng.set_prepared_ballots(_t(bal))
    status = np.zeros(G * S, dtype=np.uint8)
    acks = np.zeros(G * S, dtype=np.uint16)
    inst_bal = np.zeros(G * S, dtype=np.uint64)
    pidx = np.zeros(G * S, dtype=np.uint8)
    for rnd in range(4):
        slot = rnd if rnd < 3 else 63
        payload = wl.payload_uniform(G, data_len, seed_extra=300 + rnd)
        pol = rng.integers(0, K, G).astype(np.uint8)
        sh = eng.propose(slot, _t(payload), torch.from_numpy(pol).to(DEV))
        torch.cuda.synchronize()
        got = sh.cpu().numpy()
        assert got.shape[0] == T
        assert (got[d:] == oracle.rs_encode_uniform(d, T - d, payload, data_len)).all()
        L = oracle.cw_shard_len(data_len, d)
        for g in (0, G - 1):
            assert (got[:d, g, :L] == oracle.cw_split(payload[g, :data_len].tobytes(), d)).all()
        status.reshape(G, S)[:, slot] = oracle.ST_ACCEPTING
        acks.reshape(G, S)[:, slot] = 0
        inst_bal.reshape(G, S)[:, slot] = bal
        pidx.reshape(G, S)[:, slot] = pol
        rg, rs_, rp, rb = _reply_stream(rng, G, population, bal, 30000)
        for half in range(2):
            sl = slice(half * 15000, (half + 1) * 15000)
            eng.on_accept_replies(_t(rg[sl]), torch.from_numpy(rs_[sl]).to(DEV), torch.from_numpy(rp[sl]).to(DEV), _t(rb[sl]))
            committed, bar = eng.tick()
            torch.cuda.synchronize()
            oracle.tally_stream_crossword(rg[sl], rs_[sl], rp[sl], rb[sl], S, population, T, d, majority, f, balanced, policies,
                                          pidx, bal, inst_bal, status, acks)
            want = _words(status, G, S, oracle)
            assert (committed.cpu().numpy().view(np.uint64) == want).all(), (rnd, half)
            want_bar = np.array([oracle.commit_bar(int(w)) for w in want], dtype=np.uint32)
            assert (bar.cpu().numpy().view(np.uint32) == want_bar).all()
    frac = (status == oracle.ST_COMMITTED).sum() / (G * 4)
    assert 0.02 < frac <= 1.0
    eng.close()


def _raft_append(rng, W, curr_term, last_commit, log_end, terms):
    """The leader appends half to a full ring per group, never more than the ring can hold: n_new, and the host model's
    log_end and terms (ring position (log_end + i) & (W-1)) updated in place."""
    G = len(log_end)
    room = (W - (log_end - last_commit - 1)).astype(np.int64)
    n_new = np.minimum(rng.integers((W + 1) // 2, W + 1, G), room).astype(np.uint32)
    n_new[rng.random(G) < 0.1] = 0
    wrote = ((np.arange(W)[None, :] - log_end[:, None].astype(np.int64)) & (W - 1)) < n_new[:, None]
    terms[wrote] = np.broadcast_to(curr_term[:, None], terms.shape)[wrote]
    log_end += n_new
    return n_new


def _raft_rewrite_tail(rng, W, curr_term, last_commit, log_end, terms):
    """A new leader inherits a tail with older-term entries: rewrite half the uncommitted entries of 30 % of the groups."""
    G = len(log_end)
    off = (np.arange(W)[None, :] - (last_commit[:, None].astype(np.int64) + 1)) & (W - 1)
    tail = off < (log_end - last_commit - 1)[:, None].astype(np.int64)
    old = tail & (rng.random(G) < 0.3)[:, None] & (rng.random((G, W)) < 0.5)
    terms[old] = np.broadcast_to(curr_term[:, None] - 1, terms.shape)[old]


def _raft_replies(rng, P, log_end):
    """Successful AppendEntriesReplies: a few out-of-range groups and peers, end_slot in [0, log_end) (a follower never
    acknowledges past the leader's log), mostly near the top of the log, some stale."""
    G = len(log_end)
    nrec = 6 * G * (P + 1)
    rg = rng.integers(0, G + 3, nrec).astype(np.uint32)
    rp = rng.integers(0, P + 1, nrec).astype(np.uint8)
    hi = log_end[np.minimum(rg, G - 1)].astype(np.int64)
    rend = np.where(rng.random(nrec) < 0.7, np.maximum(hi - rng.geometric(0.3, nrec), 0),
                    rng.integers(0, 1 << 30, nrec) % hi).astype(np.uint32)
    return rg, rp, rend


@pytest.mark.parametrize("W", [1, 2, 4, 8, 64, 4096])
@pytest.mark.parametrize("population", range(2, 13))
def test_raft_engine_matches_per_reply_handler(ctx, oracle, population, W):
    """Appends + batches of successful AppendEntriesReplies (duplicates, stale end_slots, out-of-range peers) over several
    ticks: match_slot / next_slot / last_commit / last_snap and the term ring equal the per-reply handler's end state,
    with adversarial term rings (older-term entries inside the uncommitted tail).  The logs grow to several times the
    window, so every ring index wraps.  Odd populations from 5 up run CRaft (threshold majority + f)."""
    from summerset_b200.engine import RaftEngine
    craft = population >= 5 and population % 2 == 1
    f = min(2, population - population // 2 - 1) if craft else 0
    rng = np.random.default_rng(population * 7 + W)
    G, P = 1500, population - 1
    eng = RaftEngine(ctx, G, population, f, craft, W)
    majority = population // 2 + 1
    thr = majority + f if craft else majority
    assert eng.threshold == thr and eng.W == W
    curr_term = rng.integers(2, 9, G).astype(np.uint32)
    eng.curr_term.copy_(_t(curr_term))
    # host model of the engine state
    next_slot = np.ones((P, G), dtype=np.uint32); match = np.zeros((P, G), dtype=np.uint32)
    last_commit = np.zeros(G, dtype=np.uint32); last_snap = np.zeros(G, dtype=np.uint32)
    log_end = np.ones(G, dtype=np.uint32); terms = np.zeros((G, W), dtype=np.uint32)
    for rnd in range(10):
        n_new = _raft_append(rng, W, curr_term, last_commit, log_end, terms)
        eng.append(_t(n_new))
        torch.cuda.synchronize()
        assert (eng.log_end.cpu().numpy().view(np.uint32) == log_end).all(), rnd
        assert (eng.terms.cpu().numpy().view(np.uint32) == terms).all(), rnd
        if rnd == 2:
            _raft_rewrite_tail(rng, W, curr_term, last_commit, log_end, terms)
            eng.terms.copy_(_t(terms))
        rg, rp, rend = _raft_replies(rng, P, log_end)
        eng.on_append_replies(_t(rg), torch.from_numpy(rp).to(DEV), _t(rend))
        lc, ls = eng.tick()
        torch.cuda.synchronize()
        oracle.raft_reply_stream(rg, rp, rend, P, thr, next_slot, match, last_commit, last_snap, log_end, curr_term, terms)
        assert (eng.next_slot.cpu().numpy().view(np.uint32) == next_slot).all(), rnd
        assert (eng.match.cpu().numpy().view(np.uint32) == match).all(), rnd
        assert (lc.cpu().numpy().view(np.uint32) == last_commit).all(), rnd
        assert (ls.cpu().numpy().view(np.uint32) == last_snap).all(), rnd
    # the ring wrapped: logs several windows long, commits past the first window
    assert (log_end > 3 * W).mean() > 0.9 and (last_commit > W).mean() > 0.9
    assert ctx.device_status() == 0
    # appending past the ring's capacity is refused and reported
    eng.append(_t(np.full(G, W + 1, dtype=np.uint32)))
    torch.cuda.synchronize()
    assert ctx.device_status() == 2 and (eng.log_end.cpu().numpy().view(np.uint32) == log_end).all()
    eng.close()
