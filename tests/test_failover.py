"""Leader fail-over and follower recovery on the device, at every population and code the ABI accepts.

The calls a fail-over runs: ss_prepare_merge_dev (the new leader merges PrepareReply votes and decides per instance),
ss_gossip_plan_dev (a Crossword follower picks the peers to ask for missing shards), ss_reconstruct_serve_dev (a peer
answers a Reconstruct request), ss_wal_commit_pack_dev (CommitSlot records) and ss_raft_kth_match_dev.  Each is compared
bit for bit with the CPU oracle and with a vectorised numpy restatement of the same rule; the end-to-end tests chain them
the way a fail-over does: acceptor state -> votes -> merge -> reconstruct -> new Accepts.

`_replay` restates handle_msg_prepare_reply per reply (rspaxos/messages.rs:182-259, crossword/messages.rs:233-312) with
the vote rule of rspaxos/durability.rs and crossword/durability.rs: a reply carries `voted = Some(..)` iff its ballot is
non-zero; a higher ballot replaces the shards gathered so far, an equal one is absorbed (union).
"""
import numpy as np
import pytest
import torch

from summerset_b200 import _lib
from tests.test_acceptor import Cfg, _acceptor, _buffer, _pitch

DEV = "cuda:0"
U64MAX = (1 << 64) - 1
EXTREME_BALLOTS = np.array([1, 1 << 63, U64MAX], dtype=np.uint64)
USE, NULL, RECONSTRUCT, PARITY = 1, 2, 4, 8


def _t(a):
    a = np.ascontiguousarray(a)
    if a.dtype == np.uint64:
        a = a.view(np.int64)
    elif a.dtype == np.uint32:
        a = a.view(np.int32)
    return torch.from_numpy(a).to(DEV)


def _u32(x):
    return x.cpu().numpy().view(np.uint32)


def _u64(x):
    return x.cpu().numpy().view(np.uint64)


def _popc(x):
    return np.bitwise_count(np.asarray(x, dtype=np.uint32)).astype(np.int64)


# ---------------------------------------------------------------------------------------------
# models
# ---------------------------------------------------------------------------------------------
def _replay(votes):
    """handle_msg_prepare_reply, one reply at a time: votes = [(ballot, shard mask)] in arrival order, ballot 0 = None"""
    mb, cw = 0, 0
    for b, m in votes:
        if b == 0:                   # voted == None
            continue
        if b > mb:                   # a higher ballot: the codeword gathered so far is dropped
            mb, cw = b, m
        elif b == mb:                # absorb_other
            cw |= m
    return mb, cw


def _merge_np(bal, mask):
    """the same for a whole batch: bal uint64 [R, N], mask uint32 [R, N]"""
    voted = bal > 0
    mb = np.where(voted, bal, np.uint64(0)).max(axis=0)
    at = voted & (bal == mb[None, :])
    return mb, np.bitwise_or.reduce(np.where(at, mask, np.uint32(0)), axis=0).astype(np.uint32)


def _decide_np(merged, acks, d, population, f):
    """ssor_prepare_decide for a batch"""
    pc = _popc(merged)
    pcd = _popc(merged & np.uint32(0xFFFFFFFF if d >= 32 else (1 << d) - 1))
    use = pc >= d
    null = ~use & (acks.astype(np.int64) >= population - f)
    avail = np.where(use, pc, d)
    act = use * USE | (use & (pcd < d)) * RECONSTRUCT | null * NULL | ((use | null) & (avail < population)) * PARITY
    return act.astype(np.uint8)


def _ballots(rng, shape):
    """ballots from {0, 1, 2}, so that ties are common, and now and then 1, 2^63 or 2^64 - 1"""
    b = rng.integers(0, 3, shape).astype(np.uint64)
    ext = rng.random(shape) < 0.05
    b[ext] = EXTREME_BALLOTS[rng.integers(0, 3, int(ext.sum()))]
    return b


def _gossip_np(me, population, d, src, avail, pidx, policies, alive):
    """gossip_targets_excl (crossword/gossiping.rs:35-84) for a batch; excl rows of unselected peers stay 0xFFFFFFFF"""
    pol = np.asarray(policies, dtype=np.uint32).reshape(-1, population)
    k = np.where(pidx < len(pol), pidx, 0)
    av = avail.astype(np.uint32).copy()
    t = np.zeros(len(av), dtype=np.uint32)
    ex = np.full((population, len(av)), 0xFFFFFFFF, dtype=np.uint32)
    active = np.ones(len(av), dtype=bool)
    for pp in range(me + 1, me + population):
        peer = pp % population
        consider = active & (src != peer) & bool((alive >> peer) & 1)
        useful = pol[k, peer] & ~av
        sel = consider & (useful != 0)
        ex[peer, sel] = av[sel]
        t[sel] |= np.uint32(1 << peer)
        av = np.where(sel, av | useful, av)
        active &= ~(consider & (_popc(av) >= d))      # coverage is tested after the peer is considered
    return t, ex


# ---------------------------------------------------------------------------------------------
# CPU: the replay against the oracle
# ---------------------------------------------------------------------------------------------
def test_replay_matches_oracle_stream(oracle):
    rng = np.random.default_rng(40)
    for _ in range(3000):
        R = int(rng.integers(1, 33))
        bal = _ballots(rng, R)
        mask = rng.integers(0, 1 << 32, R, dtype=np.uint64).astype(np.uint32)
        mask[rng.random(R) < 0.3] = 0                           # Some((bal, empty)) at any ballot, and None with a mask
        votes = [(int(b), int(m)) for b, m in zip(bal, mask)]
        want = oracle.prepare_merge_stream(bal > 0, bal, mask)
        assert _replay(votes) == want
        assert _replay(votes[::-1]) == want                     # any arrival order
        mb, mg = _merge_np(bal[:, None], mask[:, None])
        assert (int(mb[0]), int(mg[0])) == want
    # an empty vote at a higher, an equal and a lower ballot than the shard-carrying ones
    for votes, want in [([(1, 0b011), (2, 0)], (2, 0)), ([(2, 0), (1, 0b011)], (2, 0)), ([(1, 0b011), (1, 0)], (1, 0b011)),
                        ([(2, 0b100), (1, 0)], (2, 0b100)), ([(U64MAX, 0), (1 << 63, 0b1)], (U64MAX, 0)),
                        ([(1 << 63, 0b1), (U64MAX, 0b10), (U64MAX, 0)], (U64MAX, 0b10)), ([(0, 0b111)], (0, 0))]:
        b = np.array([v[0] for v in votes], dtype=np.uint64)
        m = np.array([v[1] for v in votes], dtype=np.uint32)
        assert _replay(votes) == want == oracle.prepare_merge_stream(b > 0, b, m)


def test_empty_higher_ballot_vote_clears_the_merged_set(oracle):
    """RSPaxos-shaped n = 5, d = 3, f = 1: three replicas voted their shards at ballot 1, one replica (a Crossword
    replica with an empty assignment row, say) accepted at ballot 2 with no shards.  The reply at ballot 2 discards
    the shards of ballot 1: the instance is NULL once n - f replies are in, or waits; it is never USE."""
    bal = np.array([1, 1, 1, 2, 0], dtype=np.uint64)
    mask = np.array([0b00001, 0b00010, 0b00100, 0, 0], dtype=np.uint32)
    votes = list(zip(bal.tolist(), mask.tolist()))
    assert _replay(votes) == (2, 0) == oracle.prepare_merge_stream(bal > 0, bal, mask)
    assert oracle.prepare_decide(0, 4, 3, 5, 1) == NULL | PARITY
    assert oracle.prepare_decide(0, 3, 3, 5, 1) == 0
    # deciding "no vote" by the mask instead keeps ballot 1's three shards and would decide USE
    assert oracle.prepare_merge_stream(mask != 0, bal, mask) == (1, 0b111)
    assert oracle.prepare_decide(0b111, 4, 3, 5, 1) & USE
    mb, mg = _merge_np(bal[:, None], mask[:, None])
    assert (int(mb[0]), int(mg[0])) == (2, 0)
    assert list(_decide_np(mg, np.array([4]), 3, 5, 1)) == [NULL | PARITY]


def test_numpy_restatements_match_the_oracle(oracle):
    """the batch models the GPU tests compare with whole batches, against the oracle instance by instance"""
    rng = np.random.default_rng(41)
    R, N = 7, 400
    bal = _ballots(rng, (R, N))
    mask = rng.integers(0, 1 << 9, (R, N)).astype(np.uint32)
    mask[rng.random((R, N)) < 0.2] = 0
    acks = rng.integers(0, 9, N).astype(np.uint8)
    mb, mg = _merge_np(bal, mask)
    for d, f in [(3, 1), (9, 0), (4, 7), (32, 3)]:
        act = _decide_np(mg, acks, d, 7, f)
        for i in range(N):
            assert (int(mb[i]), int(mg[i])) == oracle.prepare_merge_stream(bal[:, i] > 0, bal[:, i], mask[:, i])
            assert int(act[i]) == oracle.prepare_decide(int(mg[i]), int(acks[i]), d, 7, f)
    for population in (1, 2, 5, 32):
        pol = rng.integers(0, 1 << 32, (3, population), dtype=np.uint64).astype(np.uint32)
        src = rng.integers(0, population, N).astype(np.uint8)
        avail = rng.integers(0, 1 << 32, N, dtype=np.uint64).astype(np.uint32) & rng.integers(0, 1 << 32, N, dtype=np.uint64).astype(np.uint32)
        pidx = rng.integers(0, 5, N).astype(np.uint8)
        for me in {0, population // 2, population - 1}:
            for d in (1, 12, 32):
                alive = int(rng.integers(0, 1 << population)) | (1 << me)
                t, ex = _gossip_np(me, population, d, src, avail, pidx, pol, alive)
                for i in range(0, N, 7):
                    wt, we = oracle.gossip_targets_excl(me, population, d, int(src[i]), int(avail[i]),
                                                        pol[int(pidx[i]) if pidx[i] < 3 else 0], alive)
                    assert int(t[i]) == wt
                    assert all(int(ex[p, i]) == (int(we[p]) if (wt >> p) & 1 else 0xFFFFFFFF) for p in range(population))


# ---------------------------------------------------------------------------------------------
# GPU: prepare merge
# ---------------------------------------------------------------------------------------------
def _check_merge(ctx, oracle, bal, mask, acks, d, population, f, sample=211):
    """one launch against the batch model, and against the oracle plus the replay on a strided sample (and the tail)"""
    mb, mg, act = ctx.prepare_merge(_t(bal), _t(mask), _t(acks), d, population, f)
    mb, mg, act = _u64(mb), _u32(mg), act.cpu().numpy()
    wb, wm = _merge_np(bal, mask)
    wa = _decide_np(wm, acks, d, population, f)
    assert np.array_equal(mb, wb) and np.array_equal(mg, wm) and np.array_equal(act, wa), (d, population, f)
    N = bal.shape[1]
    for i in sorted(set(range(0, N, max(1, N // sample))) | set(range(max(0, N - 64), N))):
        votes = [(int(b), int(m)) for b, m in zip(bal[:, i], mask[:, i])]
        w = oracle.prepare_merge_stream(bal[:, i] > 0, bal[:, i], mask[:, i])
        assert _replay(votes) == w == (int(mb[i]), int(mg[i])), i
        assert int(act[i]) == oracle.prepare_decide(w[1], int(acks[i]), d, population, f), i
    return mb, mg, act


def _acks(rng, N, population, f):
    """acks_cnt at population - f - 1, exactly population - f, 255, and anything in between"""
    edge = [population - f - 1, population - f, 255]
    a = rng.integers(0, population + 1, N)
    pick = rng.random(N) < 0.6
    a[pick] = np.array(edge)[rng.integers(0, 3, int(pick.sum()))]
    return np.clip(a, 0, 255).astype(np.uint8)


def _fs(population):
    return sorted({0, 1, (population - 1) // 2, population} & set(range(population + 1)))


@pytest.mark.gpu
@pytest.mark.parametrize("population", range(3, 13))
def test_prepare_merge_rspaxos_populations(ctx, oracle, population):
    """RSPaxos: replica r votes shard r (disjoint one-shard votes), d = majority"""
    rng = np.random.default_rng(100 + population)
    N, R, d = 3001, population, population // 2 + 1
    bal = _ballots(rng, (R, N))
    mask = np.broadcast_to((1 << np.arange(R, dtype=np.uint32))[:, None], (R, N)).copy()
    for f in _fs(population):
        act = _check_merge(ctx, oracle, bal, mask, _acks(rng, N, population, f), d, population, f)[2]
        kinds = {int(a) & (USE | NULL) for a in act}
        assert {USE, NULL} <= kinds and (0 in kinds or f == population)      # f = population never waits


CW_CODES = [(5, 5, 3), (7, 7, 4), (3, 6, 4), (5, 10, 6), (4, 8, 5), (6, 12, 7), (12, 24, 13)]


def _cw_tables(oracle, rng, n, T):
    """the balanced round-robin assignment at every spr, plus an unbalanced table with one empty row"""
    tables = [oracle.cw_brr_assignment(n, T, spr) for spr in range(1, T + 1)]
    unb = rng.integers(1, 1 << T, n).astype(np.uint32)
    unb[int(rng.integers(0, n))] = 0
    return np.stack(tables + [unb])


@pytest.mark.gpu
@pytest.mark.parametrize("n,T,d", CW_CODES)
def test_prepare_merge_crossword_codes(ctx, oracle, n, T, d):
    """Crossword: every replica votes its assignment row; rows overlap once spr > T / n, and the empty row of the
    unbalanced table is a vote with a ballot and no shards"""
    rng = np.random.default_rng(200 + n * T)
    N = 4001
    tables = _cw_tables(oracle, rng, n, T)
    tid = rng.integers(0, len(tables), N)
    tid[:200] = len(tables) - 1
    mask = np.ascontiguousarray(tables[tid].T)
    bal = _ballots(rng, (n, N))
    for f in _fs(n):
        _, mg, act = _check_merge(ctx, oracle, bal, mask, _acks(rng, N, n, f), d, n, f)
        assert (act & RECONSTRUCT).any() and (act & USE).any()
    # the empty row at the highest ballot clears what the others voted
    empty = int(np.nonzero(tables[-1] == 0)[0][0])
    b2 = np.ones((n, N), dtype=np.uint64)
    b2[empty] = 2
    _, mg, act = _check_merge(ctx, oracle, b2, np.ascontiguousarray(np.broadcast_to(tables[-1][:, None], (n, N))), np.full(N, n, np.uint8),
                              d, n, 1)
    assert (mg == 0).all() and ((act & (USE | NULL)) == NULL).all()


@pytest.mark.gpu
@pytest.mark.parametrize("R,d,population", [(1, 1, 1), (1, 3, 5), (31, 16, 31), (32, 17, 32), (32, 32, 32), (31, 32, 32)])
def test_prepare_merge_wide_votes(ctx, oracle, R, d, population):
    """R = 1, 31 and 32 vote rows; d = 32 with T = 32 (the data mask of every bit); masks use bit 31"""
    rng = np.random.default_rng(300 + R * 64 + d)
    N = 3001
    bal = _ballots(rng, (R, N))
    mask = rng.integers(0, 1 << 32, (R, N), dtype=np.uint64).astype(np.uint32)
    mask[:, :50] = 0xFFFFFFFF
    mask[rng.random((R, N)) < 0.15] = 0
    mask[:, 50:100] = np.uint32(1 << 31)
    for f in _fs(population):
        _check_merge(ctx, oracle, bal, mask, _acks(rng, N, population, f), d, population, f)


@pytest.mark.gpu
def test_prepare_merge_past_the_grid_cap(ctx, oracle):
    """one launch of more instances than the sm_count x 32 CTAs of 256 threads: the grid-stride loop covers the tail"""
    rng = np.random.default_rng(310)
    N = ctx.sm_count * 32 * 256 + 1001
    R, d, population, f = 5, 3, 5, 1
    bal = _ballots(rng, (R, N))
    mask = rng.integers(0, 1 << 5, (R, N)).astype(np.uint32)
    _check_merge(ctx, oracle, bal, mask, _acks(rng, N, population, f), d, population, f, sample=300)


@pytest.mark.gpu
def test_prepare_merge_refusals(ctx):
    lib = ctx.lib
    N = 64
    bal = torch.ones((33, N), dtype=torch.int64, device=DEV)
    mask = torch.ones((33, N), dtype=torch.int32, device=DEV)
    acks = torch.full((N,), 3, dtype=torch.uint8, device=DEV)
    mb = torch.full((N,), 7, dtype=torch.int64, device=DEV)
    mg = torch.full((N,), 7, dtype=torch.int32, device=DEV)
    act = torch.full((N,), 7, dtype=torch.uint8, device=DEV)
    call = lambda R, n, d, pop, f: lib.ss_prepare_merge_dev(ctx.h, bal.data_ptr(), mask.data_ptr(), R, n, acks.data_ptr(), d, pop, f,
                                                           mb.data_ptr(), mg.data_ptr(), act.data_ptr())
    assert call(0, N, 3, 5, 1) == _lib.SS_ERR_INVALID_ARG
    assert call(33, N, 3, 5, 1) == _lib.SS_ERR_INVALID_ARG
    assert call(5, N, 3, 5, 6) == _lib.SS_ERR_INVALID_ARG
    assert call(5, 0, 3, 5, 1) == _lib.SS_OK
    torch.cuda.synchronize()
    assert (mb == 7).all() and (mg == 7).all() and (act == 7).all()
    assert call(32, N, 3, 5, 5) == _lib.SS_OK                           # f == population is the largest accepted
    torch.cuda.synchronize()
    assert (_u32(mg) == 1).all() and (mb.cpu() == 1).all()


# ---------------------------------------------------------------------------------------------
# GPU: gossip planning
# ---------------------------------------------------------------------------------------------
def _sparse_rows(rng, K, population):
    pol = np.zeros((K, population), dtype=np.uint32)
    for b in range(3):
        pol |= (np.uint32(1) << rng.integers(0, 32, (K, population)).astype(np.uint32))
    pol[:, ::3] |= np.uint32(1 << 31)
    pol[0, :population // 2] |= np.uint32(0x0F0F0F0F)
    return pol


def _check_gossip(ctx, oracle, me, population, d, src, avail, pidx, pol, alive, sample=60, run=None):
    if run is None:
        run = ctx.gossip_plan(me, population, d, _t(src), _t(avail), _t(pidx), pol.tolist(), alive)
    t, ex = _u32(run[0]), _u32(run[1])
    wt, wx = _gossip_np(me, population, d, src, avail, pidx, pol, alive)
    assert np.array_equal(t, wt) and np.array_equal(ex, wx), (me, population, d, alive)
    N = len(avail)
    for i in sorted(set(range(0, N, max(1, N // sample))) | set(range(max(0, N - 16), N))):
        ot, oe = oracle.gossip_targets_excl(me, population, d, int(src[i]), int(avail[i]), pol[int(pidx[i]) if pidx[i] < len(pol) else 0], alive)
        assert int(t[i]) == ot
        for p in range(population):
            assert int(ex[p, i]) == (int(oe[p]) if (ot >> p) & 1 else 0xFFFFFFFF)
    return t


@pytest.mark.gpu
@pytest.mark.parametrize("population", [1, 2, 3, 5, 16, 31, 32])
def test_gossip_plan_populations(ctx, oracle, population):
    """me at 0, the middle and population - 1 (the walk wraps); only me alive, all, random; src_peer == me and any
    other; 16 policies, indices up to 19 (>= 16 selects policy 0); d reached by the first peer (d = 1) or never (32)"""
    rng = np.random.default_rng(400 + population)
    N = 1500
    pol = _sparse_rows(rng, 16, population)
    all_alive = (1 << population) - 1
    seen_first, seen_never = False, False
    for me in sorted({0, population // 2, population - 1}):
        src = rng.integers(0, population, N).astype(np.uint8)
        src[::5] = me
        for alive in (1 << me, all_alive, (int(rng.integers(0, 1 << population)) | (1 << me)) & all_alive):
            for d in (1, int(rng.integers(2, 32)), 32):
                avail = (rng.integers(0, 1 << 32, N, dtype=np.uint64) & rng.integers(0, 1 << 32, N, dtype=np.uint64)).astype(np.uint32)
                avail[::4] = 0
                avail[1::9] |= np.uint32(1 << 31)
                pidx = rng.integers(0, 20, N).astype(np.uint8)
                t = _check_gossip(ctx, oracle, me, population, d, src, avail, pidx, pol, alive)
                if d == 1:
                    seen_first |= bool((_popc(t) == 1).any())
                if d == 32:
                    seen_never |= bool((_popc(t) > 1).any())
    assert population == 1 or seen_first
    assert population < 5 or seen_never


@pytest.mark.gpu
def test_gossip_plan_past_the_grid_cap_and_back_to_back(ctx, oracle):
    rng = np.random.default_rng(450)
    population, me, d = 5, 3, 3
    N = ctx.sm_count * 32 * 256 + 777
    pol = [oracle.cw_brr_assignment(5, 5, spr) for spr in (1, 2, 3)]
    src = rng.integers(0, population, N).astype(np.uint8)
    avail = rng.integers(0, 1 << 5, N).astype(np.uint32)
    pidx = rng.integers(0, 4, N).astype(np.uint8)
    _check_gossip(ctx, oracle, me, population, d, src, avail, pidx, np.stack(pol), 0b11011, sample=400)
    # two calls with different policy tables, no synchronisation between them: the table goes through the context's
    # shared scratch buffer, so the second upload must not overwrite what the first kernel reads
    N = 20000
    src, avail, pidx = src[:N].copy(), avail[:N].copy(), pidx[:N].copy()
    pol_a = np.stack(pol)
    pol_b = _sparse_rows(rng, 16, population) & np.uint32(0x1F)
    a = ctx.gossip_plan(me, population, d, _t(src), _t(avail), _t(pidx), pol_a.tolist(), 0b11111)
    b = ctx.gossip_plan(me, population, d, _t(src), _t(avail), _t(pidx), pol_b.tolist(), 0b11111)
    torch.cuda.synchronize()
    _check_gossip(ctx, oracle, me, population, d, src, avail, pidx, pol_a, 0b11111, run=a)
    _check_gossip(ctx, oracle, me, population, d, src, avail, pidx, pol_b, 0b11111, run=b)


@pytest.mark.gpu
def test_gossip_plan_refusals(ctx):
    lib = ctx.lib
    N = 8
    z8 = torch.zeros(N, dtype=torch.uint8, device=DEV)
    z32 = torch.zeros(N, dtype=torch.int32, device=DEV)
    t = torch.empty(N, dtype=torch.int32, device=DEV)
    ex = torch.empty(33 * N, dtype=torch.int32, device=DEV)
    pol = np.ones(17 * 33, dtype=np.uint32)
    call = lambda me, pop, k, n=N: lib.ss_gossip_plan_dev(ctx.h, me, pop, 3, z8.data_ptr(), z32.data_ptr(), z8.data_ptr(), pol.ctypes.data,
                                                         k, 0xFFFFFFFF, n, t.data_ptr(), ex.data_ptr())
    assert call(0, 5, 0) == _lib.SS_ERR_INVALID_ARG
    assert call(0, 5, 17) == _lib.SS_ERR_INVALID_ARG
    assert call(0, 33, 1) == _lib.SS_ERR_INVALID_ARG
    assert call(5, 5, 1) == _lib.SS_ERR_INVALID_ARG
    assert call(0, 0, 1) == _lib.SS_ERR_INVALID_ARG
    assert call(4, 5, 16) == _lib.SS_OK and call(31, 32, 1) == _lib.SS_OK and call(0, 5, 0, 0) == _lib.SS_OK
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------
# GPU: reconstruct serving
# ---------------------------------------------------------------------------------------------
def _serve(ctx, planes, plane_stride, ss, T, L, group, held, excl, status, reply_off, out_bytes):
    """raw ss_reconstruct_serve_dev; planes: device uint8, shard j of group g at j*plane_stride + g*ss"""
    n = len(group)
    out = torch.full((out_bytes,), 0x77, dtype=torch.uint8, device=DEV)
    mask = torch.full((n,), -1, dtype=torch.int32, device=DEV)
    args = [_t(group), _t(held), _t(excl), _t(status), _t(reply_off)]
    rc = ctx.lib.ss_reconstruct_serve_dev(ctx.h, planes.data_ptr(), plane_stride, ss, T, L, *[a.data_ptr() for a in args], n,
                                          mask.data_ptr(), out.data_ptr())
    assert rc == _lib.SS_OK, ctx.lib.ss_last_error()
    return _u32(mask), out.cpu().numpy()


def _serve_case(ctx, oracle, rng, T, L, n_groups, n_req, extra_pad=True, check_oracle=True):
    Lp = (L + 15) // 16 * 16
    ss = Lp + (16 * int(rng.integers(1, 4)) if extra_pad else 0)          # shard_stride wider than the padded shard
    plane_stride = n_groups * ss + 48                                    # not n x shard_stride
    planes_h = rng.integers(0, 256, T * plane_stride, dtype=np.uint8)
    planes = _t(planes_h)
    group = rng.integers(0, n_groups, n_req).astype(np.uint32)
    held = rng.integers(0, 1 << 32, n_req, dtype=np.uint64).astype(np.uint32)          # bits at and above T too
    excl = (rng.integers(0, 1 << 32, n_req, dtype=np.uint64) & rng.integers(0, 1 << 32, n_req, dtype=np.uint64)).astype(np.uint32)
    excl[::13] = 0xFFFFFFFF
    status = rng.integers(0, 5, n_req).astype(np.uint8)
    status[:5] = [0, 1, 2, 3, 4]
    held[:5], excl[:5] = 0xFFFFFFFF, 0                                   # the status boundary: served from 2 (Accepting) up
    all_ =np.uint32(0xFFFFFFFF if T >= 32 else (1 << T) - 1)
    want = np.where(status >= 2, held & ~excl & all_, np.uint32(0)).astype(np.uint32)
    if check_oracle:
        assert all(int(w) == oracle.reconstruct_serve_mask(int(h), int(x), T, int(s)) for w, h, x, s in zip(want, held, excl, status))
    cnt = _popc(want)
    gaps = 16 * rng.integers(0, 4, n_req)
    sizes = cnt * Lp + gaps
    reply_off = (np.concatenate([[0], np.cumsum(sizes)[:-1]]) + gaps).astype(np.uint64)          # canary gaps between replies
    total = int(reply_off[-1]) + int(cnt[-1]) * Lp + 64
    got_mask, out = _serve(ctx, planes, plane_stride, ss, T, L, group, held, excl, status, reply_off, total)
    assert np.array_equal(got_mask, want)
    exp = np.full(total, 0x77, dtype=np.uint8)
    for i in np.nonzero(want)[0]:
        o = int(reply_off[i])
        for j in range(T):
            if (int(want[i]) >> j) & 1:
                s = j * plane_stride + int(group[i]) * ss
                exp[o:o + Lp] = planes_h[s:s + Lp]                       # subset_copy: the shard, in its padded slot
                o += Lp
    if not np.array_equal(out, exp):
        bad = np.nonzero(out != exp)[0]
        pytest.fail(f"T={T} L={L}: {len(bad)} bytes differ, first at {bad[0]}")
    return want


@pytest.mark.gpu
@pytest.mark.parametrize("T", [1, 2, 5, 12, 31, 32])
def test_reconstruct_serve_shapes(ctx, oracle, T):
    """held / exclude bits at and above T, shard lengths around every 16-byte and 32-lane edge (past 32 x 16 bytes each
    lane loops), a shard_stride wider than the padded shard, a plane_stride that is not n x shard_stride, statuses 0-4,
    and replies at non-contiguous offsets whose gaps must keep their canary"""
    rng = np.random.default_rng(500 + T)
    for L in (1, 15, 16, 17, 511, 512, 513, 65537):
        big = L > 1000
        want = _serve_case(ctx, oracle, rng, T, L, 4 if big else 40, 24 if big else 300)
        assert (want != 0).any()


@pytest.mark.gpu
def test_reconstruct_serve_past_the_grid_cap(ctx, oracle):
    """more requests than sm_count x 64 CTAs of 8 warps (a warp per request)"""
    rng = np.random.default_rng(550)
    n_req = ctx.sm_count * 64 * 8 + 300
    _serve_case(ctx, oracle, rng, 5, 16, 50, n_req, check_oracle=False)


@pytest.mark.gpu
def test_reconstruct_serve_refusals(ctx):
    lib = ctx.lib
    n, L, T = 4, 100, 5
    planes = torch.zeros(T * n * 128 + 64, dtype=torch.uint8, device=DEV)
    z32 = torch.zeros(n, dtype=torch.int32, device=DEV)
    st = torch.full((n,), 2, dtype=torch.uint8, device=DEV)
    off = torch.zeros(n, dtype=torch.int64, device=DEV)
    mask = torch.empty(n, dtype=torch.int32, device=DEV)
    out = torch.zeros(T * 128 + 64, dtype=torch.uint8, device=DEV)
    P, O = planes.data_ptr(), out.data_ptr()

    def call(T=T, L=L, ss=112, ps=n * 112, p=P, o=O, n=n):
        return lib.ss_reconstruct_serve_dev(ctx.h, p, ps, ss, T, L, z32.data_ptr(), z32.data_ptr(), z32.data_ptr(), st.data_ptr(),
                                            off.data_ptr(), n, mask.data_ptr(), o)
    assert call(T=0) == _lib.SS_ERR_INVALID_ARG
    assert call(T=33) == _lib.SS_ERR_INVALID_ARG
    assert call(L=0) == _lib.SS_ERR_INVALID_ARG
    assert call(p=P + 1) == _lib.SS_ERR_INVALID_ARG
    assert call(o=O + 8) == _lib.SS_ERR_INVALID_ARG
    assert call(ss=120) == _lib.SS_ERR_INVALID_ARG
    assert call(ps=n * 112 + 4) == _lib.SS_ERR_INVALID_ARG
    assert call(ss=96) == _lib.SS_ERR_INVALID_ARG                         # shorter than the padded shard (112)
    assert call() == _lib.SS_OK and call(n=0, T=0) == _lib.SS_OK
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------
# GPU: CommitSlot packer
# ---------------------------------------------------------------------------------------------
def _commit_pack(ctx, newly, base, variant, capacity, cnt=None, spare=6):
    """raw ss_wal_commit_pack_dev into canary-filled buffers with `spare` cells past capacity"""
    cells = capacity + spare
    entries = torch.full((cells, 24), 0xA5, dtype=torch.uint8, device=DEV)
    eg = torch.full((cells,), -1, dtype=torch.int32, device=DEV)
    el = torch.full((cells,), -1, dtype=torch.int32, device=DEV)
    cnt = torch.full((1,), 12345, dtype=torch.int64, device=DEV) if cnt is None else cnt
    nt, bt = _t(newly), _t(base)
    rc = ctx.lib.ss_wal_commit_pack_dev(ctx.h, nt.data_ptr(), bt.data_ptr(), len(newly), variant, entries.data_ptr(), eg.data_ptr(),
                                        el.data_ptr(), capacity, cnt.data_ptr())
    assert rc == _lib.SS_OK
    return entries.cpu().numpy(), eg.cpu().numpy(), el.cpu().numpy(), int(cnt.cpu()[0]), cnt


def _commit_records(oracle, newly, base, variant):
    out = []
    for g in np.nonzero(newly)[0]:
        w = int(newly[g])
        for s in range(64):
            if (w >> s) & 1:
                slot = (int(base[g]) + s) & U64MAX
                body = oracle.varint(variant) + oracle.varint(slot)
                rec = len(body).to_bytes(8, "big") + body
                if variant == 2:
                    assert rec == oracle.wal_commit_slot(slot)
                out.append((int(g), rec))
    return sorted(out)


def _check_cells(entries, eg, el, want, written):
    got = sorted((int(eg[e]), entries[e, :int(el[e])].tobytes()) for e in range(written))
    if written == len(want):
        assert got == want
    else:
        pool = list(want)
        for x in got:                                                    # a sub-multiset of the records
            pool.remove(x)
    assert (entries[written:] == 0xA5).all() and (eg[written:] == -1).all() and (el[written:] == -1).all()
    assert (el[:written] > 8).all()


@pytest.mark.gpu
@pytest.mark.parametrize("variant", [0, 2, 250, 251, 65535, (1 << 32) - 1])
def test_wal_commit_pack_varint_widths(ctx, oracle, variant):
    """window bases that put base + s across every varint width inside one window, every bit of one group set, and
    capacity = total - 1, total and 0: cells past capacity stay untouched and the count is still exact"""
    rng = np.random.default_rng(600 + variant % 1000)
    base = np.array([0, 251 - 32, 65536 - 32, (1 << 32) - 32, (1 << 63) - 10, U64MAX - 63, 7, 250], dtype=np.uint64)
    G = 300
    base = np.concatenate([base, rng.integers(0, 1 << 62, G - len(base), dtype=np.uint64)]).astype(np.uint64)
    newly = (rng.integers(0, 1 << 62, G, dtype=np.uint64) & rng.integers(0, 1 << 62, G, dtype=np.uint64)).astype(np.uint64)
    newly[:6] = np.uint64(U64MAX)                                        # every bit of the window
    newly[6] = np.uint64(1 << 63)
    newly[7] = np.uint64(1)
    newly[10::5] = 0
    want = _commit_records(oracle, newly, base, variant)
    total = len(want)
    for capacity in (total + 3, total, total - 1, 0):
        entries, eg, el, cnt, _ = _commit_pack(ctx, newly, base, variant, capacity)
        assert cnt == total, capacity
        _check_cells(entries, eg, el, want, min(capacity, total))


@pytest.mark.gpu
def test_wal_commit_pack_past_the_grid_cap_and_repeated(ctx, oracle):
    """more groups than sm_count x 64 CTAs of 256 threads; a second call on the same buffers resets n_entries"""
    rng = np.random.default_rng(650)
    G = ctx.sm_count * 64 * 256 + 999
    newly = np.zeros(G, dtype=np.uint64)
    pick = np.concatenate([rng.choice(G - 999, 3000, replace=False), np.arange(G - 999, G)])
    newly[pick] = rng.integers(1, 1 << 62, len(pick), dtype=np.uint64) & rng.integers(1, 1 << 62, len(pick), dtype=np.uint64)
    newly[G - 1] = np.uint64(U64MAX)
    base = rng.integers(0, 1 << 40, G, dtype=np.uint64).astype(np.uint64)
    want = _commit_records(oracle, newly, base, 2)
    entries, eg, el, cnt, cnt_t = _commit_pack(ctx, newly, base, 2, len(want))
    assert cnt == len(want)
    _check_cells(entries, eg, el, want, len(want))
    # the same n_entries buffer again (and smaller input): the count starts from 0, it does not accumulate
    newly2 = newly[:5000].copy()
    want2 = _commit_records(oracle, newly2, base[:5000], 2)
    entries, eg, el, cnt, _ = _commit_pack(ctx, newly2, base[:5000], 2, len(want2), cnt=cnt_t)
    assert cnt == len(want2)
    _check_cells(entries, eg, el, want2, len(want2))


# ---------------------------------------------------------------------------------------------
# GPU: k-th largest match at the bucket edges
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n_peers", [1, 3, 5, 7, 9, 15])
def test_kth_match_bucket_edges(ctx, oracle, n_peers):
    rng = np.random.default_rng(700 + n_peers)
    G = 4099
    for hi in (3, 1 << 32):
        m = rng.integers(0, hi, (n_peers, G), dtype=np.uint64).astype(np.uint32)
        m[:, :4] = 0xFFFFFFFF
        desc = -np.sort(-m.astype(np.int64), axis=0)
        for k in range(1, n_peers + 1):
            got = _u32(ctx.raft_kth_match(_t(m), k))
            assert np.array_equal(got, desc[k - 1].astype(np.uint32)), k
            assert all(int(got[g]) == oracle.craft_shadow_last_commit(m[:, g], k + 1) for g in range(0, G, 211)), k


# ---------------------------------------------------------------------------------------------
# GPU end to end: leader fail-over
# ---------------------------------------------------------------------------------------------
def _codeword(oracle, data, d, p):
    """the oracle's encoding of a payload: d data shards then p parity shards, L bytes each"""
    split = oracle.cw_split(data, d)
    L = split.shape[1]
    shards = [np.ascontiguousarray(split[j]) for j in range(d)] + [np.zeros(L, dtype=np.uint8) for _ in range(p)]
    assert oracle.rs_encode(d, p, shards) == 0
    return shards


def _unbalanced_rows(n, T, d):
    """an unbalanced assignment that leaves replica n - 2 out: the other rows are windows of d - 1 shards, so that
    any two of them cover d"""
    rows = [sum(1 << ((r + k) % T) for k in range(d - 1)) for r in range(n)]
    rows[n - 2] = 0
    return np.array([rows], dtype=np.uint32)


FAILOVER_CASES = [("rspaxos", 5, 1, 0, 0, "-"), ("rspaxos", 7, 2, 0, 0, "-"), ("crossword", 5, 1, 5, 3, "balanced"),
                  ("crossword", 5, 1, 10, 6, "balanced"), ("crossword", 5, 1, 5, 3, "empty-row")]


class _Cluster:
    """a LeaderEngine (replica 0) and device acceptors 1 .. n-1 run through the closed loop of test_acceptor_closed_loop"""

    def __init__(self, ctx, oracle, rng, protocol, n, f, T, d, kind, G):
        from summerset_b200.engine import LeaderEngine
        self.ctx, self.oracle, self.rng, self.n, self.f, self.G = ctx, oracle, rng, n, f, G
        self.cw = protocol == "crossword"
        self.eng = LeaderEngine(ctx, protocol, G, n, f, 1, rs_total_shards=T, rs_data_shards=d)
        self.bal = rng.integers(1, 1 << 30, G).astype(np.uint64)
        self.eng.set_prepared_ballots(_t(self.bal))
        self.d, self.T = self.eng.d, self.eng.T
        self.p = self.T - self.d
        if not self.cw:
            self.policies = np.array([[1 << r for r in range(n)]], dtype=np.uint32)
        elif kind == "balanced":
            self.policies = np.stack([oracle.cw_brr_assignment(n, self.T, spr) for spr in range(self.T // n, self.d + 1, self.T // n)])
        else:
            self.policies = _unbalanced_rows(n, self.T, self.d)
        if self.cw:
            self.eng.set_policies([list(map(int, q)) for q in self.policies], kind == "balanced")
        self.protocol = protocol
        self.accs = {r: _acceptor(ctx, Cfg(protocol, n, r, self.d, self.T), G) for r in range(1, n)}
        self.stores = []                 # every acceptor store stays alive: the acceptors' shard_addr point into them
        self.inst = {}                   # (g, slot) -> payload, policy index, shard length

    def round(self, loss):
        from summerset_b200 import workloads as wl
        rng, G, d, p, cw = self.rng, self.G, self.d, self.p, self.cw
        lens = np.where(rng.random(G) < 0.1, 0, wl.cfg4_lengths(G, seed_extra=len(self.inst))[0] // 8 + 1).astype(np.uint32)
        pol = rng.integers(0, len(self.policies), G).astype(np.uint8)
        gaps = rng.integers(0, 32, G)
        ends = np.cumsum(lens.astype(np.int64) + gaps)
        data_off = (16 + ends - lens.astype(np.int64)).astype(np.uint64)
        arena = rng.integers(0, 256, 16 + int(ends[-1]) + 32, dtype=np.uint8)
        L = (lens.astype(np.int64) + d - 1) // d
        store = torch.zeros((self.T, int(((L + 31) // 32 * 32).sum()) + 32), dtype=torch.uint8, device=DEV)
        slot_out, shard_off, _ = self.eng.propose_ragged(_t(arena), _t(data_off), _t(lens), store, _t(pol) if cw else None)
        assert self.ctx.device_status() == 0
        slots = _u64(slot_out)
        recs, rec_group, rec_peer = [], [], []
        for g in range(G):
            if slots[g] != np.uint64(U64MAX):
                s = int(slots[g])
                self.inst[(g, s)] = dict(data=arena[int(data_off[g]):int(data_off[g]) + int(lens[g])].tobytes(), pol=int(pol[g]), L=int(L[g]))
                recs.append(self.oracle.frame_accept_reply(3, s, int(self.bal[g]), cw, 0))     # the leader's self-ack
                rec_group.append(g)
                rec_peer.append(0)
        for r, acc in self.accs.items():
            out, off, fl, _ = self.ctx.frame_accept_pack_ragged(store, shard_off, _t(lens), d, p, self.policies, _t(pol), r, slot_out,
                                                                _t(self.bal), with_assignment=cw)
            fl_h, off_h, buf_np = fl.cpu().numpy(), off.cpu().numpy(), out.cpu().numpy()
            sent = [g for g in range(G) if fl_h[g] > 0 and rng.random() >= loss]          # lost Accepts
            frames = [buf_np[int(off_h[g]):int(off_h[g]) + int(fl_h[g])].tobytes() for g in sent]
            cells, rl = self._accept(acc, r, frames, sent, [int(slots[g]) for g in sent], [int(pol[g]) for g in sent])
            for i, g in enumerate(sent):
                if rng.random() >= loss:                                                    # lost replies
                    recs.append(cells[i, :rl[i]].tobytes())
                    rec_group.append(g)
                    rec_peer.append(r)
        buf, offs = _buffer(rng, recs, odd=False)
        rg, rs_, rp, rb, rk = self.ctx.accept_reply_parse(_t(buf), _t(offs), _t(np.array(rec_group, dtype=np.uint32)),
                                                          _t(np.array(rec_peer, dtype=np.uint8)), self.eng.window_base, 3, cw)
        assert (rk.cpu().numpy() == 3).all()
        self.eng.on_accept_replies(rg, rs_, rp, rb)
        self.eng.tick()
        torch.cuda.synchronize()

    def _accept(self, acc, r, frames, groups, slots, pols, src=0):
        total = sum(bin(int(self.policies[q][r])).count("1") * _pitch(self.inst[(g, s)]["L"]) for g, s, q in zip(groups, slots, pols)) + 32
        astore = torch.empty(total, dtype=torch.uint8, device=DEV)
        awal = torch.empty(sum(len(x) + 32 for x in frames) + 32, dtype=torch.uint8, device=DEV)
        self.stores.append(astore)
        buf, offs = _buffer(self.rng, frames)
        res = acc.accept(_t(buf), _t(offs), _t(np.array(groups, dtype=np.uint32)), _t(np.full(len(frames), src, np.uint8)), astore, awal)
        assert (res["verdict"].cpu().numpy().view(np.uint32) == _lib.SS_ACCEPT_VERDICT_ACCEPTED).all()
        return res["replies"].cpu().numpy(), res["reply_len"].cpu().numpy()

    def views(self):
        """per acceptor: (Accepting bit, inst_bal, held, shard_addr) of every proposed instance"""
        keys = sorted(self.inst)
        k = np.array([g * 64 + (s & 63) for g, s in keys], dtype=np.int64)
        gs = np.array([g for g, _ in keys], dtype=np.int64)
        ss = np.array([s & 63 for _, s in keys], dtype=np.uint64)
        out = {}
        for r, acc in self.accs.items():
            accepting = ((_u64(acc.accepting)[gs] >> ss) & np.uint64(1)).astype(bool)
            out[r] = (accepting, _u64(acc.inst_bal)[k], _u32(acc.held)[k], _u64(acc.shard_addr)[k])
        return keys, out

    def close(self):
        self.eng.close()
        for acc in self.accs.values():
            acc.close()


def _read(stores, addr, n):
    for base, arr in stores:
        if base <= addr and addr + n <= base + len(arr):
            return arr[addr - base:addr - base + n]
    raise AssertionError(f"address {addr:#x} is in no acceptor store")


@pytest.mark.gpu
@pytest.mark.parametrize("protocol,n,f,T,d,kind", FAILOVER_CASES)
def test_failover_recovers_every_committed_instance(ctx, oracle, protocol, n, f, T, d, kind):
    """rounds of the closed loop, Accepts and replies lost in the last one, then the leader dies: a survivor prepares
    at a higher ballot with quorums from below a majority to n - 1.  Votes come from the responders' acceptor views;
    the merge equals the model; no instance the old engine committed is decided NULL; USE instances rebuild, from the
    shards the responders' stores hold, the codeword the oracle encodes; the rebuilt codewords are accepted again by
    the survivors at the new ballot, byte for byte."""
    from summerset_b200.api import ReedSolomon
    rng = np.random.default_rng(800 + n * 10 + T + len(kind))
    G = 48
    cl = _Cluster(ctx, oracle, rng, protocol, n, f, T, d, kind, G)
    d, p, T, cw = cl.d, cl.p, cl.T, cl.cw
    for rnd in range(3):
        cl.round(loss=0.45 if rnd == 2 else 0.1)
    committed_w = _u64(cl.eng.committed)
    assert (_u64(cl.eng.window_base) == 0).all()
    keys, views = cl.views()
    N = len(keys)
    committed = np.array([bool((int(committed_w[g]) >> s) & 1) for g, s in keys])
    assert committed.any() and not committed.all()
    stores = [(t.data_ptr(), t.cpu().numpy()) for t in cl.stores]
    survivors = list(range(1, n))
    new_leader = survivors[int(rng.integers(0, len(survivors)))]
    majority = n // 2 + 1
    rs = ReedSolomon(ctx, d, p)
    for Q in range(max(1, majority - 1), n):
        others = [r for r in survivors if r != new_leader]
        resp = [new_leader] + list(rng.choice(others, Q - 1, replace=False))
        bal_v = np.zeros((n, N), dtype=np.uint64)                        # row r: replica r's vote; the dead leader and
        mask_v = np.zeros((n, N), dtype=np.uint32)                       # the replicas that did not answer have none
        for r in resp:
            accepting, ib, held, _ = views[r]
            bal_v[r] = np.where(accepting, ib, np.uint64(0))
            mask_v[r] = held
        acks = np.full(N, Q, dtype=np.uint8)
        mb, mg, act = ctx.prepare_merge(_t(bal_v), _t(mask_v), _t(acks), d, n, f)
        mb, mg, act = _u64(mb), _u32(mg), act.cpu().numpy()
        wb, wm = _merge_np(bal_v, mask_v)
        assert np.array_equal(mb, wb) and np.array_equal(mg, wm) and np.array_equal(act, _decide_np(wm, acks, d, n, f)), Q
        # safety: a committed instance is recovered (USE) or waits; a NULL would overwrite a chosen value
        assert not (act[committed] & NULL).any(), (Q, [keys[i] for i in np.nonzero(committed & ((act & NULL) != 0))[0]])
        if Q == n - 1 and f >= 1:
            assert (act[committed] & USE).all(), Q                       # every survivor answered
        # rebuild from the merged shards the responders' stores hold
        Ls = np.array([cl.inst[k]["L"] for k in keys], dtype=np.int64)
        pitch = (Ls + 31) // 32 * 32
        off = np.concatenate([[0], np.cumsum(pitch)[:-1]]).astype(np.int64)
        ps = int(pitch.sum()) + 32
        sh = np.full((T, ps), 0xEE, dtype=np.uint8)
        for i, key in enumerate(keys):
            L = int(Ls[i])
            for j in range(T):
                if not (int(mg[i]) >> j) & 1:
                    continue
                r = next(r for r in resp if bal_v[r, i] == mb[i] and (int(mask_v[r, i]) >> j) & 1)
                _, _, held, addr = views[r]
                k = bin(int(held[i]) & ((1 << j) - 1)).count("1")
                sh[j, off[i]:off[i] + L] = _read(stores, int(addr[i]) + k * _pitch(L), L)
        sh_d = _t(sh)
        lens = np.array([len(cl.inst[k]["data"]) for k in keys], dtype=np.int32)
        st = rs.reconstruct_batch(sh_d, ps, _t(off), _t(lens), _t(mg), False).cpu().numpy()
        got = sh_d.cpu().numpy()
        use = (act & USE) != 0
        assert (st[use] == 0).all() and (st[_popc(mg) < d] == _lib.SS_ERR_TOO_FEW_SHARDS_PRESENT).all()
        assert (use | (_popc(mg) < d)).all()
        cws = {}
        for i in np.nonzero(use)[0]:
            cws[i] = _codeword(oracle, cl.inst[keys[i]]["data"], d, p)
            for j in range(T):
                assert np.array_equal(got[j, off[i]:off[i] + Ls[i]], cws[i][j]), (Q, keys[i], j)
    assert use.any()
    # the new leader re-proposes the recovered values at its ballot; every survivor accepts them
    new_bal = cl.bal + np.uint64(1) + rng.integers(0, 1 << 20, G).astype(np.uint64)
    idx = np.nonzero(use)[0]
    slot_a = np.array([keys[i][1] for i in idx], dtype=np.uint64)
    grp = [keys[i][0] for i in idx]
    pol = np.array([cl.inst[keys[i]]["pol"] for i in idx], dtype=np.uint8)
    sub = lambda a: _t(np.ascontiguousarray(a))
    for r in survivors:
        out, fo, fl, _ = ctx.frame_accept_pack_ragged(sh_d, sub(off[idx]), sub(lens[idx]), d, p, cl.policies, sub(pol), r, sub(slot_a),
                                                      sub(new_bal[grp]), with_assignment=cw)
        assert ctx.device_status() == 0
        fl_h, fo_h, buf = fl.cpu().numpy(), fo.cpu().numpy(), out.cpu().numpy()
        assert (fl_h > 0).all()
        frames = [buf[int(fo_h[i]):int(fo_h[i]) + int(fl_h[i])].tobytes() for i in range(len(idx))]
        cl._accept(cl.accs[r], r, frames, grp, list(map(int, slot_a)), list(map(int, pol)), src=new_leader)
    torch.cuda.synchronize()
    stores = [(t.data_ptr(), t.cpu().numpy()) for t in cl.stores[-len(survivors):]]
    _, views = cl.views()
    for r in survivors:
        accepting, ib, held, addr = views[r]
        for q, i in enumerate(idx):
            g, s = keys[i]
            row = int(cl.policies[int(pol[q])][r])
            assert accepting[i] and int(ib[i]) == int(new_bal[g]) and int(held[i]) == row, (r, g, s)
            L = int(Ls[i])
            for k, j in enumerate(j for j in range(T) if (row >> j) & 1):
                assert np.array_equal(_read(stores, int(addr[i]) + k * _pitch(L), L), cws[i][j]), (r, g, s, j)
    rs.close()
    cl.close()


# ---------------------------------------------------------------------------------------------
# GPU end to end: a Crossword follower's gossip round
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n,T,d", [(5, 5, 3), (7, 7, 4), (5, 10, 6)])
def test_gossip_round_fills_a_follower(ctx, oracle, n, T, d):
    """codewords from the oracle, each replica holding its assignment row; a follower plans, every target serves
    held = its row minus the exclusion the plan gave it; replies are pairwise disjoint and disjoint from what the
    follower holds, reach d whenever the live peers cover it, and rebuild the original data shards"""
    from summerset_b200.api import ReedSolomon, round_up
    rng = np.random.default_rng(900 + n * T)
    N, data_len, p = 600, 1500, T - d
    data = rng.integers(0, 256, (N, data_len), dtype=np.uint8)
    L = -(-data_len // d)
    ds = round_up(L, 16)
    planes = np.zeros((T, N, ds), dtype=np.uint8)
    for g in range(N):
        planes[:, g, :L] = np.stack(_codeword(oracle, data[g].tobytes(), d, p))
    planes_d = _t(planes)
    dj = T // n
    policies = np.stack([oracle.cw_brr_assignment(n, T, spr) for spr in range(dj, d + 1, dj)])
    pidx = rng.integers(0, len(policies), N).astype(np.uint8)
    rows = policies[pidx]                                                 # [N, n]
    rs = ReedSolomon(ctx, d, p)
    for me, alive in [(0, (1 << n) - 1), (n - 1, ((1 << n) - 1) & ~0b10), (n // 2, (1 << (n // 2)) | 0b1 | (1 << (n - 1)))]:
        src = rng.integers(0, n, N).astype(np.uint8)
        src[src == me] = (me + 1) % n
        own = rows[:, me].astype(np.uint32)
        t, ex = ctx.gossip_plan(me, n, d, _t(src), _t(own), _t(pidx), policies.tolist(), alive)
        t, ex = _u32(t), _u32(ex)
        wt, wx = _gossip_np(me, n, d, src, own, pidx, policies, alive)
        assert np.array_equal(t, wt) and np.array_equal(ex, wx)
        union = np.zeros(N, dtype=np.uint32)
        got_sh = np.full((T, N, ds), 0xEE, dtype=np.uint8)
        for j in range(T):
            sel = ((own >> j) & 1) == 1
            got_sh[j, sel] = planes[j, sel]
        for peer in range(n):
            req = np.nonzero((t >> peer) & 1)[0]
            if len(req) == 0:
                continue
            held = rows[req, peer].astype(np.uint32)
            cnt = _popc(held & ~ex[peer, req])
            reply_off = (np.concatenate([[0], np.cumsum(cnt)[:-1]]) * ds).astype(np.uint64)
            mask, out = _serve(ctx, planes_d, N * ds, ds, T, L, req.astype(np.uint32), held, ex[peer, req],
                               np.full(len(req), 3, np.uint8), reply_off, int(cnt.sum()) * ds + 64)
            assert (mask == held & ~ex[peer, req]).all()
            assert not (mask & union[req]).any() and not (mask & own[req]).any()              # nothing asked twice
            union[req] |= mask
            for q, g in enumerate(req):
                o = int(reply_off[q])
                for j in range(T):
                    if (int(mask[q]) >> j) & 1:
                        assert np.array_equal(out[o:o + ds], planes[j, g]), (peer, g, j)
                        got_sh[j, g] = out[o:o + ds]
                        o += ds
        live = [q for q in range(n) if q != me and (alive >> q) & 1]
        for g in range(N):
            cover = int(own[g])
            for q in live:
                if q != src[g]:
                    cover |= int(rows[g, q])
            assert (bin(int(own[g] | union[g])).count("1") >= d) == (bin(cover).count("1") >= d), (me, g)
        present = own | union
        sh_d = _t(got_sh.reshape(T, -1))
        st = rs.reconstruct_batch(sh_d, N * ds, _t(np.arange(N, dtype=np.int64) * ds), _t(np.full(N, data_len, np.int32)),
                                  _t(present), True).cpu().numpy()
        got = sh_d.cpu().numpy().reshape(T, N, ds)
        ok = _popc(present) >= d
        assert ok.any() and (st[ok] == 0).all() and (st[~ok] == _lib.SS_ERR_TOO_FEW_SHARDS_PRESENT).all()
        assert np.array_equal(got[:d, ok, :L], planes[:d, ok, :L])
    rs.close()
