"""The CRaft follower's append and advance (ss_follower_append / ss_follower_advance, summerset_b200/csrc/follower.cu)
across what their ABI accepts.

tests/test_follower.py pins the semantics with its restatement (`Group`) and its rig (`Harness`); this file runs them
where the append's kernels change course:
  A  population 1, where every frame is malformed (populations 2 to 32 and `me` at 0 and n // 2: test_follower.py)
  B  windows 2, 4, 64, 4096 and 0 (= 64), each ring run around more than twice, a full ring of one term refused with a
     conflict walk over all of it; window 1 refused at creation
  C  batch sizes across the scan tiles and past the copy kernel's grid cap
  D  past the header, cut and replay kernels' grid cap, and the advance past its own
  E  sort keys at and around powers of two
  F  one hot group of 20k frames, replayed serially
  G  the absorb cursor at the store capacity
  H  one follower whose scratch the append, the vote and the recovery grow and refill
  I  a non-blocking context stream while torch's default stream is busy
Every store and WAL buffer starts at a 0xA5 canary that must survive outside the written regions.
"""
import ctypes as C
import random

import numpy as np
import pytest
import torch

from summerset_b200 import _lib
from tests.test_follower import (ACCEPTED, BEYOND, MALFORMED, REJECTED, U64, Ent, Group, Harness, append_entries,
                                 dur_log_entry, dur_metadata, entry, framed, reply, vi, wrap_after_advance)

DEV = "cuda:0"
CANARY = 0xA5
ST_STORE_FULL = 16                     # SS_DEV_STATUS_STORE_FULL


def pitch(L):
    return (L + 31) & ~31


def r16(x):
    return (x + 15) & ~15


def _t(a, dt):
    return torch.tensor(np.asarray(a), device=DEV).view(dt) if isinstance(a, np.ndarray) else torch.tensor(a, dtype=dt, device=DEV)


def _thread_cap(ctx):
    return ctx.sm_count * 64 * 256        # launch_grid: 64 CTAs per SM; header, cut, replay and advance: a thread per item


def _copy_cap(ctx):
    return ctx.sm_count * 64 * 8          # the copy kernel: a warp (frame) per 32 threads


_STATE = ("start_slot", "log_end", "curr_term", "last_commit", "last_snap", "leader", "term", "held", "data_len", "shard_addr")


def _state(fol):
    torch.cuda.synchronize()
    return {k: getattr(fol, k).cpu().numpy().copy() for k in _STATE}


def _run(fol, items, store_len=1 << 16, store_cap=None, wal_len=1 << 16):
    """one append of (group, peer, frame bytes) items at odd offsets into canaried store and WAL buffers ->
    (numpy outputs, store, wal)"""
    buf, offs = bytearray(), []
    for k, (_, _, fr) in enumerate(items):
        buf += bytes(k % 3)
        offs.append(len(buf))
        buf += fr
    store = torch.full((store_len,), CANARY, dtype=torch.uint8, device=DEV)
    wal = torch.full((wal_len,), CANARY, dtype=torch.uint8, device=DEV)
    out = fol.append(_t(np.frombuffer(bytes(buf), np.uint8).copy(), torch.uint8), _t(offs, torch.int64),
                     _t([g for g, _, _ in items], torch.int32), _t([p for _, p, _ in items], torch.uint8), store, wal, store_cap)
    torch.cuda.synchronize()
    o = {k: v.cpu().numpy() for k, v in out.items()}
    o["verdict"] = o["verdict"].view(np.uint32)
    return o, store, wal


def _following_stream(rng, n, me, W, n_frames, grow=0.5, dls=(1, 10, 250)):
    """one group's frames from leaders that keep up with the follower (a scratch restatement says where its log ends,
    so most frames append at its end, unlike _leader_stream's, which run ahead of it and are mostly refused): entries
    hold shard `me` only, re-sends of held entries carry d other shards (absorbs), new leaders rewrite the uncommitted
    suffix, and some frames carry a stale term or a wrong prev_term (refused) or run past the window"""
    d = n // 2 + 1
    peers = [q for q in range(n) if q != me]
    sim = Group(n, W)
    log, term, frames = [(0, 0, {})], 1, []                         # the leader's (term, data_len, shards) per slot
    for _ in range(n_frames):
        if rng.random() < 0.1:
            term += 1
            del log[rng.randint(min(sim.lc + 1, len(log)), len(log)):]
        if rng.random() < grow or len(log) == 1:
            for _ in range(rng.randint(1, 3)):
                dl = rng.choice(dls)
                log.append((term, dl, {j: rng.randbytes(-(-dl // d)) for j in range(n)}))
        prev = min(sim.le, len(log)) - 1                             # next_slot after the leader's back-off
        while prev > sim.start and sim.log[prev][0] != log[prev][0]:
            prev -= 1
        resend = rng.random() < 0.2
        if resend:
            prev = rng.randint(max(sim.start, prev - 3), prev)
        es = []
        for s in range(prev + 1, prev + 1 + rng.randint(0, min(5, len(log) - 1 - prev))):
            t, dl, sh = log[s]
            keep = range(1, d + 1) if resend else (me,)
            es.append(Ent(t, d, n - d, dl, {j % n: sh[j % n] for j in keep}, rng.random() < 0.5, rng.choice((0, 7, 300))))
        t = term if rng.random() > 0.05 else max(1, term - 1)
        pt = log[prev][0] if rng.random() > 0.05 else log[prev][0] + 1
        f = (rng.choice(peers), t, prev, pt, es, rng.randint(0, len(log) - 1), rng.randint(0, 3))
        sim.handle(*f)
        frames.append(f)
    return frames


def _take_exact(h, n):
    """the next n frames, groups taken in turn, each group's re-submitted frames before its stream's"""
    queues = [h.pending[g] + h.streams[g] for g in range(h.G)]
    out, k = [], [0] * h.G
    while len(out) < n:
        before = len(out)
        for g in range(h.G):
            if k[g] < len(queues[g]) and len(out) < n:
                out.append((g, queues[g][k[g]]))
                k[g] += 1
        assert len(out) > before, "the streams ran dry"
    for g in range(h.G):
        h.pending[g], h.streams[g] = [], queues[g][k[g]:]
    return out


# ---------------------------------------------------------------------------------------------
# A: population 1
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_population_one_refuses_every_frame(ctx):
    """n = 1: the only replica is `me`, so a frame from `me` and one from any peer >= 1 are both malformed; nothing is
    written and no state word changes"""
    from summerset_b200.engine import Follower
    G = 5
    fol = Follower(ctx, G, 1, 0)
    assert (fol.d, fol.T) == (1, 1)
    before = _state(fol)
    rng = random.Random(1)
    items = []
    for g in range(G):
        for peer in (0, 1, 2, 31, 255):
            ents = [entry(1, 1, 0, dl, {0: rng.randbytes(dl)}) for dl in (1, 300)]
            items += [(g, peer, append_entries(1, 0, 0, ents, 0, 0)), (g, peer, append_entries(2, 0, 0, [], 0, 0))]
    rng.shuffle(items)
    ctx.device_status()
    o, store, wal = _run(fol, items)
    assert (o["verdict"] == MALFORMED).all()
    n = len(items)
    assert (o["store_off"] == -1).all() and (o["wal_off"] == -1).all() and (o["trunc_slot"] == -1).all()
    assert not o["wal_len"].any() and not o["meta_len"].any() and not o["reply_len"].any()
    assert (o["reply_dst"] == 0xFF).all() and not o["meta"].any() and not o["replies"].any()
    assert o["totals"].tolist() == [0, 0] and not o["commit_lo"].any() and o["meta"].shape == (n, 32)
    assert (store.cpu().numpy() == CANARY).all() and (wal.cpu().numpy() == CANARY).all()
    after = _state(fol)
    for k in _STATE:
        assert np.array_equal(after[k], before[k]), k
    assert (after["log_end"] == 1).all() and (after["leader"] == 0xFF).all()
    assert ctx.device_status() == 0
    fol.close()


# ---------------------------------------------------------------------------------------------
# B: windows
# ---------------------------------------------------------------------------------------------
def test_window_one_is_refused():
    """a one-entry ring holds only start_slot: every entry would be BEYOND_WINDOW, nothing could commit and start_slot
    could never move, so creation refuses it; 2 and 4096 pass the configuration checks"""
    lib = _lib.load()
    real = torch.cuda.is_available()
    ctx = None
    if real:
        from summerset_b200.api import Context
        ctx = Context(0)
    for W, want in ((1, _lib.SS_ERR_INVALID_ARG), (3, _lib.SS_ERR_INVALID_ARG), (8192, _lib.SS_ERR_INVALID_ARG),
                    (2, _lib.SS_OK if real else _lib.SS_ERR_NO_DEVICE), (4096, _lib.SS_OK if real else _lib.SS_ERR_NO_DEVICE)):
        h = C.c_void_p()
        cfg = _lib.FollowerConfig(_lib.SS_PROTO_CRAFT, 3, 0, W, 0, 1, 0, 1)
        assert lib.ss_follower_create(ctx.h if real else None, C.byref(cfg), 4, C.byref(h)) == want, W
        assert bool(h) == (want == _lib.SS_OK)
        if h:
            lib.ss_follower_destroy(h)
    if real:
        ctx.close()
    # the restatement at W = 1: an appending frame is always beyond the window, so nothing ever commits
    m = Group(3, 1)
    for _ in range(3):
        assert m.handle(0, 1, m.le - 1, 0, [Ent(1, 2, 1, 1, {0: b"x", 1: b"y"})], 5, 0)["verdict"] == BEYOND
        m.advance(m.lc + 5)
    assert (m.start, m.le, m.lc) == (0, 1, 0)


def _advance_to(h, upto):
    """advance with upto[g] for the groups listed (start_slot, which moves nothing, for the others)"""
    u = [upto.get(g, m.start) for g, m in enumerate(h.models)]
    h.fol.advance(torch.tensor(u, dtype=torch.int64, device=DEV))
    for g, m in enumerate(h.models):
        m.advance(u[g])
    torch.cuda.synchronize()
    h.check_state()


def _fill_ring_with_one_term(h):
    """group 0 ends holding a full ring of one term, start_slot included; a frame whose prev_term does not match its
    last entry is refused with a conflict walk back over the whole ring"""
    m, W, d, n = h.models[0], h.W, h.d, h.n
    peer = next(q for q in range(n) if q != h.me)
    t = m.ct + 1
    one = lambda: Ent(t, d, n - d, 1, {j: h.rng.randbytes(1) for j in range(d)}, True, 0)
    h.pending = [[] for _ in range(h.G)]

    def send(f):
        o, _, _ = h.batch([(0, f)])
        assert int(o["verdict"][0]) in (ACCEPTED, REJECTED)
        return o

    send((peer, t, m.le - 1, m.log[m.le - 1][0], [], m.le - 1, 0))   # a new leader's heartbeat commits the whole log
    assert m.lc == m.le - 1
    _advance_to(h, {0: m.lc})
    s0 = m.start + 1
    send((peer, t, m.start, m.log[m.start][0], [one() for _ in range(W - 1)], 0, 0))
    send((peer, t, m.le - 1, t, [], m.le - 1, 0))
    assert m.lc == m.le - 1 == s0 + W - 2
    _advance_to(h, {0: s0})
    send((peer, t, m.le - 1, t, [one()], 0, 0))
    assert (m.start, m.le) == (s0, s0 + W) and all(m.log[s][0] == t for s in range(s0, s0 + W))
    o = send((peer, t, m.le - 1, t + 1, [], 0, 0))
    assert int(o["verdict"][0]) == REJECTED
    assert o["replies"][0][:int(o["reply_len"][0])].tobytes() == reply(t, s0 + W - 1, (t, s0))


@pytest.mark.gpu
@pytest.mark.parametrize("window", [2, 4, 64, 4096, 0])
def test_windows_run_around_the_ring(window):
    """test_follower_window_wrap_after_advance's rounds until every group's log ran past 3 W and its start past 2 W, at
    entries per round and per frame that scale with W; then a full ring of one term"""
    W = window or 64
    G = 2 if W == 4096 else 8
    h = Harness(5, G, window=window, seed=40 + W + (window == 0), frames_per_group=0, me=1)
    assert h.W == W
    h.absorb_room = 1 << 12                                        # the rounds' entries hold d shards: nothing absorbs
    grow, send = (3, min(5, W - 1)) if W <= 8 else (W, W)
    done = lambda h: all(m.le > 3 * W and m.start > 2 * W for m in h.models)
    beyond = wrap_after_advance(h, 400, grow, send, (1, 10, 251) if W < 4096 else (1, 10), until=done)
    assert done(h) and beyond > 0
    _fill_ring_with_one_term(h)


# ---------------------------------------------------------------------------------------------
# C: batch sizes
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n", [2047, 2048, 2049, 4097, "copy_cap+1000"])
def test_batch_sizes(ctx, n):
    """store and WAL offsets scanned across the 2048-frame scan tiles, and the copy kernel past its grid cap"""
    if n == "copy_cap+1000":
        n = _copy_cap(ctx) + 1000
    G = n // 40
    h = Harness(3, G, window=16, seed=n, frames_per_group=0, ctx=ctx)
    h.absorb_room = 1 << 22
    h.streams = [_following_stream(h.rng, 3, h.me, h.W, 41) for _ in range(G)]
    frames = _take_exact(h, n)
    assert len(frames) == n
    o, _, (so, _) = h.batch(frames)
    v = o["verdict"]
    assert (v == ACCEPTED).sum() > n // 4 and (v == REJECTED).any() and (v == BEYOND).any()
    assert int(o["totals"][0]) > so                                # entries absorbed shards


# ---------------------------------------------------------------------------------------------
# D: past the header / replay grid cap, and the advance past its grid cap
# ---------------------------------------------------------------------------------------------
def _one_entry_frames(G, tail):
    """one frame per group g: AppendEntries{term 1, prev 0, prev_term 0, [one entry of term 1 holding shards 0 and 1
    (d = 2, data_len 2: one byte each)], commit 0, snap 0} at population 3; then `tail` such frames naming groups >= G.
    -> (buf, offsets, groups, peers, frame template, payload bytes [N, 2], payload positions in the frame)"""
    tmpl = append_entries(1, 0, 0, [entry(1, 2, 1, 2, {0: b"\x11", 1: b"\x22"})], 0, 0)
    at = (tmpl.index(b"\x11", 8), tmpl.index(b"\x22", 8))
    F, N = len(tmpl), G + tail
    i = np.arange(N, dtype=np.int64)
    pay = np.stack([(i * 7 + 3) & 255, (i * 13 + 5) & 255], axis=1).astype(np.uint8)
    fr = np.tile(np.frombuffer(tmpl, np.uint8), (N, 1))
    fr[:, at[0]], fr[:, at[1]] = pay[:, 0], pay[:, 1]
    buf = np.concatenate([np.full(3, 0xEE, np.uint8), fr.reshape(-1), np.full(16, 0xEE, np.uint8)])
    offs = 3 + F * i
    groups = np.where(i < G, i, np.array([G, G + 1, (1 << 31) - 1])[i % 3]).astype(np.int32)
    peers = (i % 2).astype(np.uint8)                               # me = 2
    return buf, offs, groups, peers, tmpl, pay, at


@pytest.mark.gpu
def test_past_the_header_grid_cap(ctx):
    """header / cut / replay cap + 1000 groups with one frame each and 500 frames of unknown groups behind them: every
    frame of a known group appends slot 1, so offsets, records, cells, store bytes and state follow from i in numpy"""
    from summerset_b200.engine import Follower
    tail = 500
    G = _thread_cap(ctx) + 1000
    fol = Follower(ctx, G, 3, 2, window=2)
    buf, offs, groups, peers, tmpl, pay, at = _one_entry_frames(G, tail)
    N = G + tail
    rec = dur_log_entry(Ent(1, 2, 1, 2, {0: b"\x11", 1: b"\x22"}).to_external())
    R = r16(len(rec))
    store = torch.full((64 * N + 4096,), CANARY, dtype=torch.uint8, device=DEV)
    wal = torch.full((R * N + 4096,), CANARY, dtype=torch.uint8, device=DEV)
    ctx.device_status()
    out = fol.append(_t(buf, torch.uint8), _t(offs, torch.int64), _t(groups, torch.int32), _t(peers, torch.uint8), store, wal)
    torch.cuda.synchronize()
    o = {k: v.cpu().numpy() for k, v in out.items()}
    v = o["verdict"].view(np.uint32)
    assert (v[:G] == ACCEPTED).all() and (v[G:] == MALFORMED).all()
    i = np.arange(G, dtype=np.int64)
    assert np.array_equal(o["store_off"][:G], 64 * i) and np.array_equal(o["wal_off"][:G], R * i)
    assert (o["store_off"][G:] == -1).all() and (o["wal_off"][G:] == -1).all() and (o["trunc_slot"] == -1).all()
    assert (o["wal_len"][:G] == R).all() and not o["wal_len"][G:].any()
    assert o["totals"].tolist() == [64 * G, R * G] and not o["commit_lo"].any()
    # cells: Metadata{1, None} and AppendEntriesReply{1, 1, None} to the sender (the group's leader once it appended)
    meta, rep = dur_metadata(1), reply(1, 1)
    want_meta = np.zeros((N, 32), np.uint8)
    want_meta[:G, :len(meta)] = np.frombuffer(meta, np.uint8)
    want_rep = np.zeros((N, 48), np.uint8)
    want_rep[:G, :len(rep)] = np.frombuffer(rep, np.uint8)
    assert np.array_equal(o["meta"], want_meta) and np.array_equal(o["replies"], want_rep)
    assert (o["meta_len"][:G] == len(meta)).all() and (o["reply_len"][:G] == len(rep)).all()
    assert not o["meta_len"][G:].any() and not o["reply_len"][G:].any()
    assert np.array_equal(o["reply_dst"][:G], peers[:G]) and (o["reply_dst"][G:] == 0xFF).all()
    # the store: shards 0 and 1 in 32-byte slots, zero to 16 bytes, the canary after
    ws = np.full(store.numel(), CANARY, np.uint8)
    slots = ws[:64 * G].reshape(G, 2, 32)
    slots[:, :, :16] = 0
    slots[:, :, 0] = pay[:G]
    assert np.array_equal(store.cpu().numpy(), ws)
    # the WAL: one LogEntry record per frame at R-byte strides, the canary in the padding
    r_at = (rec.index(b"\x11", 8), rec.index(b"\x22", 8))                  # past the length, which is 17
    ww = np.full(wal.numel(), CANARY, np.uint8)
    recs = ww[:R * G].reshape(G, R)
    recs[:, :len(rec)] = np.frombuffer(rec, np.uint8)
    recs[:, r_at[0]], recs[:, r_at[1]] = pay[:G, 0], pay[:G, 1]
    assert np.array_equal(wal.cpu().numpy(), ww)
    st = _state(fol)
    assert (st["start_slot"] == 0).all() and (st["log_end"] == 2).all() and (st["curr_term"] == 1).all()
    assert not st["last_commit"].any() and not st["last_snap"].any() and np.array_equal(st["leader"], peers[:G])
    assert (st["term"][:, 0] == 0).all() and (st["held"][:, 0] == 0).all() and (st["data_len"][:, 0] == 0).all()
    assert (st["term"][:, 1] == 1).all() and (st["held"][:, 1] == 3).all() and (st["data_len"][:, 1] == 2).all()
    assert np.array_equal(st["shard_addr"][:, 1].view(np.uint64), np.uint64(store.data_ptr()) + (64 * i).astype(np.uint64))
    assert ctx.device_status() == 0
    fol.close()


@pytest.mark.gpu
def test_advance_past_its_grid_cap(ctx):
    """advance-kernel cap + 1000 groups at W = 2: slot 1 appended everywhere, committed where the heartbeat says so,
    then two advances with upto at 0, start_slot, last_commit, last_commit + 5 and 2^64 - 1, group by group"""
    from summerset_b200.engine import Follower
    G = _thread_cap(ctx) + 1000
    fol = Follower(ctx, G, 3, 2, window=2)
    buf, offs, groups, peers, _, _, _ = _one_entry_frames(G, 0)
    store = torch.full((64 * G,), CANARY, dtype=torch.uint8, device=DEV)
    wal = torch.full((64 * G,), CANARY, dtype=torch.uint8, device=DEV)
    out = fol.append(_t(buf, torch.uint8), _t(offs, torch.int64), _t(groups, torch.int32), _t(peers, torch.uint8), store, wal)
    torch.cuda.synchronize()
    assert (out["verdict"].cpu().numpy().view(np.uint32) == ACCEPTED).all()
    # heartbeats {term 1, prev 1, prev_term 1, commit c}: c = 1 commits slot 1 (two shards: a majority), c = 0 does not
    g = np.arange(G, dtype=np.int64)
    commit = (g % 3 != 0).astype(np.int64)
    hb = [np.frombuffer(append_entries(1, 1, 1, [], c, 0), np.uint8) for c in (0, 1)]
    F = len(hb[0])
    assert len(hb[1]) == F
    fr = np.where(commit[:, None] == 1, hb[1], hb[0]).astype(np.uint8)
    out = fol.append(_t(fr.reshape(-1).copy(), torch.uint8), _t(F * g, torch.int64), _t(g.astype(np.int32), torch.int32),
                     _t((g % 2).astype(np.uint8), torch.uint8), store, wal)
    torch.cuda.synchronize()
    assert (out["verdict"].cpu().numpy().view(np.uint32) == ACCEPTED).all() and out["totals"].cpu().tolist() == [0, 0]
    lc = fol.last_commit.cpu().numpy().view(np.uint64)
    assert np.array_equal(lc, commit.astype(np.uint64))
    rule = lambda s, u: np.where(u <= s, s, np.minimum(u, np.maximum(lc, s)))
    s = np.zeros(G, np.uint64)
    for kind in ((g % 2) * 4, (g // 2) % 5):
        u = np.select([kind == 0, kind == 1, kind == 2, kind == 3], [np.zeros(G, np.uint64), s, lc, lc + np.uint64(5)],
                      np.uint64(U64)).astype(np.uint64)
        fol.advance(_t(u.view(np.int64), torch.int64))
        torch.cuda.synchronize()
        s = rule(s, u)
        assert np.array_equal(fol.start_slot.cpu().numpy().view(np.uint64), s)
    assert s.any() and not s.all()
    assert (fol.log_end.cpu().numpy() == 2).all() and np.array_equal(fol.last_commit.cpu().numpy().view(np.uint64), lc)
    fol.close()


# ---------------------------------------------------------------------------------------------
# E: sort keys around powers of two
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("G", [1, 2, 3, 4, 5, 255, 256, 257, 65535, 65536, 65537])
def test_sort_keys(ctx, G):
    """frames of the last group, of group 0 and of groups >= G (sorted under key G) shuffled together: a key one bit
    short merges the unknown groups into group 0's segment, or groups into each other, and breaks their frame order"""
    h = Harness(3, G, seed=G, frames_per_group=0, ctx=ctx, me=0)
    h.absorb_room = 1 << 22
    for g in sorted({0, G - 1}):
        h.streams[g] = _following_stream(h.rng, 3, h.me, h.W, 16)
    body = append_entries(9, 0, 0, [entry(9, 2, 1, 2, {0: b"a"})], 0, 0)
    bad = [(g, 1, body, MALFORMED) for g in (G, G + 1, (1 << 31) - 1) for _ in range(3)]
    o, seq, _ = h.batch(h.take(16), bad=bad)
    assert [int(o["verdict"][i]) for i, it in enumerate(seq) if it[0] == "bad"] == [MALFORMED] * len(bad)
    assert (o["verdict"] == ACCEPTED).sum() >= 4


# ---------------------------------------------------------------------------------------------
# F: one hot group
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_one_hot_group(ctx):
    """20k frames of one group at W = 4096 replayed serially on one thread, with 30 frames of each other group around
    them: term changes, truncations, re-sends that absorb entries appended earlier in the same call, heartbeats that
    commit"""
    hot = 5
    h = Harness(5, 12, window=4096, seed=2024, frames_per_group=0, ctx=ctx, me=2)
    h.streams = [_following_stream(h.rng, 5, h.me, h.W, 20000 if g == hot else 30, 0.1 if g == hot else 0.5) for g in range(h.G)]
    frames = h.take(20000)
    lc0 = h.models[hot].lc
    o, seq, (so, _) = h.batch(frames)
    rows = [i for i, it in enumerate(seq) if it[1] == hot]
    assert len(rows) == 20000
    v = o["verdict"][rows]
    assert (v == ACCEPTED).sum() > 5000 and (v == REJECTED).sum() > 1000
    assert (o["trunc_slot"][rows] != -1).sum() > 100 and (o["meta_len"][rows] > 0).sum() > 100
    assert int(o["totals"][0]) > so and h.models[hot].lc > lc0


# ---------------------------------------------------------------------------------------------
# G: the absorb cursor at the store capacity
# ---------------------------------------------------------------------------------------------
def _absorb_rig(ctx, G, dls):
    """a population-5 follower (d = 3) whose group g holds slots 1.. of term 1 with data lengths dls, shard 0 only,
    in a store the rig keeps; -> (follower, models, shards {(g, slot): {j: bytes}}, store)"""
    from summerset_b200.engine import Follower
    rng = random.Random(len(dls) * 10 + G)
    fol = Follower(ctx, G, 5, 4, window=64)
    models = [Group(5, 64) for _ in range(G)]
    full, items = {}, []
    for g in range(G):
        ents = []
        for dl in dls:
            L = -(-dl // 3)
            sh = {j: rng.randbytes(L) for j in range(5)}
            full[(g, len(ents) + 1)] = (dl, sh)
            ents.append(Ent(1, 3, 2, dl, {0: sh[0]}))
        items.append((g, 0, append_entries(1, 0, 0, [e.wire() for e in ents], 0, 0)))
        assert models[g].handle(0, 1, 0, 0, ents, 0, 0)["verdict"] == ACCEPTED
    o, store, _ = _run(fol, items, store_len=1 << 20)
    assert (o["verdict"] == ACCEPTED).all()
    return fol, models, full, store


def _resend(full, g, s, shards=(1, 2)):
    """AppendEntries re-sending slot s of group g with other shards of the same entry: an absorb"""
    dl, sh = full[(g, s)]
    return Ent(1, 3, 2, dl, {j: sh[j] for j in shards})


def _absorb_call(ctx, fol, models, full, sends, cap_of):
    """the re-sends (group, slot), in frame order, into a fresh canaried store whose capacity is cap_of(so, absorbs)
    (so: the frames' reserved regions, absorbs: each absorb's bytes); -> (outputs, store, so, absorbs)"""
    ents = [_resend(full, g, s) for g, s in sends]
    so = sum(2 * pitch(-(-e.dl // 3)) for e in ents)
    absorbs = [3 * pitch(-(-e.dl // 3)) for e in ents]
    items = [(g, 1, append_entries(1, s - 1, 0 if s == 1 else 1, [e.wire()], 0, 0)) for (g, s), e in zip(sends, ents)]
    ctx.device_status()
    o, store, _ = _run(fol, items, store_len=so + sum(absorbs) + 4096, store_cap=cap_of(so, absorbs))
    assert (o["verdict"] == ACCEPTED).all()
    assert int(o["totals"][0]) == so + sum(absorbs)                # refused absorbs are counted too
    for k, ((g, s), e) in enumerate(zip(sends, ents)):
        want = models[g].handle(1, 1, s - 1, 0 if s == 1 else 1, [e], 0, 0)
        assert o["replies"][k][:int(o["reply_len"][k])].tobytes() == want["reply"] and o["reply_dst"][k] == 1
        assert o["wal_len"][k] == 0 and o["store_off"][k] == -1 and o["wal_off"][k] == -1
    return o, store, so, absorbs


def _absorbed(store_np, base, addr, dl, sh):
    """the union of shards 0, 1 and 2 at addr: each at its 32-byte-multiple slot, zero to 16 bytes, canary after"""
    L = -(-dl // 3)
    o = addr - base
    for r in range(3):
        q = o + r * pitch(L)
        assert store_np[q:q + L].tobytes() == sh[r]
        assert not store_np[q + L:q + r16(L)].any() and (store_np[q + r16(L):q + pitch(L)] == CANARY).all()


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["exact", "one_byte_short", "cursor_past_capacity"])
def test_absorb_at_the_store_capacity(ctx, case):
    """one group, so the absorbs take the cursor in frame order: a store that fits them to the byte takes them; one
    byte short, the entry keeps its one shard and STORE_FULL is set while the frame is accepted; a large absorb that
    does not fit leaves the cursor past the capacity, so a smaller one behind it that would have fit is refused too"""
    dls = {"exact": (3000, 30), "one_byte_short": (3000,), "cursor_past_capacity": (3000, 30)}[case]
    fol, models, full, old_store = _absorb_rig(ctx, 1, dls)
    before = _state(fol)
    sends = [(0, s) for s in range(1, len(dls) + 1)]
    cap_of = {"exact": lambda so, ab: so + sum(ab), "one_byte_short": lambda so, ab: so + sum(ab) - 1,
              "cursor_past_capacity": lambda so, ab: so + ab[1]}[case]
    o, store, so, absorbs = _absorb_call(ctx, fol, models, full, sends, cap_of)
    fits = case == "exact"
    assert ctx.device_status() == (0 if fits else ST_STORE_FULL)
    after = _state(fol)
    st, base = store.cpu().numpy(), store.data_ptr()
    written = np.zeros(st.size, bool)
    at = so
    for (g, s), ab in zip(sends, absorbs):
        dl, sh = full[(g, s)]
        if fits:
            assert after["held"][g][s] == 7 and after["shard_addr"][g][s] == base + at
            _absorbed(st, base, base + at, dl, sh)
            written[at:at + ab] = True
            at += ab
        else:
            assert after["held"][g][s] == 1 and after["shard_addr"][g][s] == before["shard_addr"][g][s]
    assert (st[~written] == CANARY).all()
    for k in ("start_slot", "log_end", "curr_term", "last_commit", "last_snap", "term", "data_len"):
        assert np.array_equal(after[k], before[k]), k
    assert (after["leader"] == 1).all()                             # the re-sends came from replica 1 in the same term
    fol.close()


@pytest.mark.gpu
def test_absorbs_of_many_groups_at_the_store_capacity(ctx):
    """eight groups absorb one equal-sized entry each into room for two and a half: exactly two take a region, in
    whichever order the groups reached the cursor, each complete with the right bytes and apart from the other; the
    rest keep their shard"""
    G = 8
    fol, models, full, old_store = _absorb_rig(ctx, G, (700,))
    before = _state(fol)
    sends = [(g, 1) for g in range(G)]
    o, store, so, absorbs = _absorb_call(ctx, fol, models, full, sends, lambda so, ab: so + 2 * ab[0] + ab[0] // 2)
    assert ctx.device_status() == ST_STORE_FULL
    after = _state(fol)
    st, base = store.cpu().numpy(), store.data_ptr()
    written = np.zeros(st.size, bool)
    took = []
    for g in range(G):
        if after["held"][g][1] == 1:
            assert after["shard_addr"][g][1] == before["shard_addr"][g][1]
            continue
        assert after["held"][g][1] == 7
        a = int(after["shard_addr"][g][1]) - base
        assert so <= a and a + absorbs[g] <= so + 2 * absorbs[0] + absorbs[0] // 2 and (a - so) % absorbs[0] == 0
        assert not written[a:a + absorbs[g]].any()
        written[a:a + absorbs[g]] = True
        _absorbed(st, base, base + a, *full[(g, 1)])
        took.append(g)
    assert len(took) == 2 and (st[~written] == CANARY).all()
    fol.close()


# ---------------------------------------------------------------------------------------------
# H: one follower across calls that share its scratch
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_scratch_shared_across_calls(ctx):
    """append 4097 frames, append 3, vote 5000 RequestVote frames, recover 100 records, append 2049, on one follower:
    the vote and the recovery name groups >= G, so they are refused and change no state, yet they regrow and refill the
    header, key, index, partial and sort scratch the appends use"""
    h = Harness(5, 100, window=16, seed=99, frames_per_group=0, ctx=ctx, me=3)
    h.absorb_room = 1 << 22
    h.streams = [_following_stream(h.rng, 5, h.me, h.W, 62) for _ in range(h.G)]
    G = h.G
    h.batch(_take_exact(h, 4097))
    o, _, _ = h.batch(_take_exact(h, 3))
    assert len(o["verdict"]) == 3
    rng = random.Random(5)
    votes = [framed(vi(0) + vi(2) + vi(rng.randint(1, 1 << 40)) + vi(rng.randint(0, 300)) + vi(rng.randint(0, 9))) for _ in range(5000)]
    buf, offs = bytearray(), []
    for fr in votes:
        buf += bytes(rng.randint(0, 3))
        offs.append(len(buf))
        buf += fr
    vg = [G + k % 7 if k % 5 else (1 << 31) - 1 for k in range(5000)]
    res = h.fol.vote(_t(np.frombuffer(bytes(buf), np.uint8).copy(), torch.uint8), _t(offs, torch.int64), _t(vg, torch.int32),
                     _t([k % 3 for k in range(5000)], torch.uint8))
    torch.cuda.synchronize()
    assert (res["verdict"].cpu().numpy().view(np.uint32) == MALFORMED).all() and not res["meta_len"].cpu().numpy().any()
    recs, rg = [], []
    for k in range(10):
        recs.append(dur_metadata(k + 50))
        rg.append(G + k)
        for s in range(9):
            recs.append(dur_log_entry(Ent(k + 50, 3, 2, 10, {j: rng.randbytes(4) for j in range(s % 5 + 1)}).to_external()))
            rg.append(G + k)
    assert len(recs) == 100
    buf, offs = bytearray(), []
    for r in recs:
        buf += bytes(rng.randint(0, 3))
        offs.append(len(buf))
        buf += r
    rstore = torch.full((1 << 16,), CANARY, dtype=torch.uint8, device=DEV)
    res = h.fol.recover(_t(np.frombuffer(bytes(buf), np.uint8).copy(), torch.uint8), _t(offs, torch.int64), _t(rg, torch.int32), rstore)
    torch.cuda.synchronize()
    assert (res["verdict"].cpu().numpy().view(np.uint32) == MALFORMED).all() and int(res["total"][0]) == 0
    assert (rstore.cpu().numpy() == CANARY).all()
    h.check_state()
    o, _, _ = h.batch(_take_exact(h, 2049))
    assert (o["verdict"] == ACCEPTED).sum() > 2049 // 4


# ---------------------------------------------------------------------------------------------
# I: a non-blocking context stream while torch's default stream is busy
# ---------------------------------------------------------------------------------------------
SLEEP_CYCLES = 1_000_000_000          # about 0.5 s at the H100's clocks


@pytest.mark.gpu
def test_follower_on_a_non_blocking_stream():
    """Creation zeroes the follower's arrays and installs the slot-0 null entry on the context's stream: with torch's
    default stream busy, start_slot and curr_term written through the view right after creation, the null entry and the
    first append on a non-blocking context stream all hold"""
    from summerset_b200.api import Context
    ctx = Context(0, own_stream=True)
    lib = ctx.lib
    s = torch.cuda.ExternalStream(lib.ss_ctx_stream(ctx.h), device=DEV)
    torch.cuda.synchronize()
    torch.cuda._sleep(SLEEP_CYCLES)
    h = Harness(5, 37, sharded=True, seed=8, frames_per_group=6, ctx=ctx, me=0)
    G = h.G
    start = np.array([0 if g % 3 else 1 for g in range(G)], dtype=np.uint64)         # a log start past the null entry
    term = np.array([(g * 7) % 4 for g in range(G)], dtype=np.uint64)
    pinned = []
    for arr, dst in ((start, h.fol.view.start_slot), (term, h.fol.view.curr_term)):
        p = C.c_void_p()
        assert lib.ss_host_alloc(ctx.h, arr.nbytes, C.byref(p)) == _lib.SS_OK
        C.memmove(p.value, arr.ctypes.data, arr.nbytes)
        assert lib.ss_copy_h2d(ctx.h, dst, p, arr.nbytes) == _lib.SS_OK
        pinned.append(p)
    for g, m in enumerate(h.models):
        m.start, m.ct = int(start[g]), int(term[g])
    with torch.cuda.stream(s):
        o, _, _ = h.batch(h.take(6))
    ctx.sync()
    assert (o["verdict"] == ACCEPTED).any() and (o["verdict"] == REJECTED).any()
    assert ctx.device_status() == 0
    for p in pinned:
        assert lib.ss_host_free(ctx.h, p) == _lib.SS_OK
    h.fol.close()
    ctx.close()
