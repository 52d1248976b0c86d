"""CRaft execution's shard decode: the bytes executed are the bytes proposed, on every CRaft path that decodes.

Three instances of exec_payload_kernel (csrc/exec_walk.cuh) turn CRaft shards back into request batches through
warp_exec_payload: CraftShards<false> (the leader before any step-up, every shard held), CraftShards<true> (the leader
once the recon view is taken: shard j at shard_addr + j * plane_stride, the sources of a missing data shard the first d
held shards) and FolLog (the follower: held shard of rank k at shard_addr + k * pitch(L)).  Every record is
compared with the request batch it was proposed from and with the C oracle's Reed-Solomon reconstruct fed the first d
held shards; the CPU tier pins the restatement in tests/test_craft_execute.py to the same oracle.

Held masks: every mask of at least d shards up to n = 12; above, a fixed seeded set (see `masks`).  Lengths: 1, 15, 16,
17, d - 1, d, d + 1, 16d - 1, 16d, 16d + 1, 4095 and 65536, so 16-byte output columns straddle up to 16 shards (L = 1 at
d = 16 and 17) and every shard-boundary phase of a column is reached.  Shards a kernel must not read are poisoned:
the leader's planes of non-held shards (0xA5, then 0x00) and the follower's slot pads (0xA5).
"""
from __future__ import annotations

import random

import numpy as np
import pytest

from oracle import pyoracle as oracle
from tests import test_craft_execute as tx
from tests import test_craft_stepup as ts

r16, pitch, popc, coded, payload, walk = tx.r16, tx.pitch, tx.popc, tx.coded, tx.payload, tx.walk
EXEC_FULL, EXEC_NULL = tx.EXEC_FULL, tx.EXEC_NULL


def code(n):
    """CRaft's code at population n: (majority, n - majority) (craft/mod.rs:527-536)"""
    return n // 2 + 1, n - n // 2 - 1


def lengths(d):
    return sorted({1, 15, 16, 17, d - 1, d, d + 1, 16 * d - 1, 16 * d, 16 * d + 1, 4095, 65536})


def masks(n):
    """the held masks a population's decode is tested at: every mask of at least d shards up to n = 12; above, all
    shards, the first d, the last d, every parity shard with the lowest data shards, every rotation of d consecutive
    shards, each single data shard missing, 64 seeded masks of exactly d shards and 32 with more"""
    d, p = code(n)
    full = (1 << n) - 1
    if n <= 12:
        return [m for m in range(1 << n) if popc(m) >= d]
    rng = random.Random(n)
    out = [full, (1 << d) - 1, full ^ ((1 << (n - d)) - 1), (full ^ ((1 << d) - 1)) | ((1 << (d - p)) - 1)]
    out += [sum(1 << ((r + k) % n) for k in range(d)) for r in range(n)]
    out += [full ^ (1 << i) for i in range(d)]
    out += [sum(1 << j for j in rng.sample(range(n), d)) for _ in range(64)]
    out += [sum(1 << j for j in rng.sample(range(n), rng.randint(d + 1, n))) for _ in range(32)]
    return list(dict.fromkeys(out))


def few_mask(n):
    """d - 1 shards: data shard 0 and the parity shards missing"""
    d, _ = code(n)
    return ((1 << (d - 1)) - 1) << 1


def oracle_decode(sh, held, d, p, dl):
    """the data bytes ssor_rs_reconstruct(data_only) regenerates from the first d held shards of sh"""
    first = [j for j in range(d + p) if held >> j & 1][:d]
    rec = [sh[j].copy() if j in first else None for j in range(d + p)]
    assert oracle.rs_reconstruct(d, p, rec, data_only=True) == 0
    return b"".join(rec[i].tobytes() for i in range(d))[:dl]


# ---- CPU: the restatement against the oracle ------------------------------------------------------------------------
def test_mask_sets():
    assert [len(masks(n)) for n in (3, 4, 5, 12)] == [4, 5, 16, 1586]
    for n in range(3, 33):
        d, p = code(n)
        ms = masks(n)
        assert all(popc(m) >= d and m < 1 << n for m in ms) and len(set(ms)) == len(ms)
        assert (1 << n) - 1 in ms and (1 << d) - 1 in ms and popc(few_mask(n)) == d - 1
        # the most data shards any decodable mask can miss: p
        assert max(d - popc(m & ((1 << d) - 1)) for m in ms) == p


@pytest.mark.parametrize("n", range(3, 33))
def test_restatement_matches_the_oracle(n):
    d, p = code(n)
    rng = np.random.default_rng(n)
    for dl in lengths(d):
        batch = rng.integers(0, 256, dl, dtype=np.uint8).tobytes()
        sh = coded(batch, d, p)
        for m in masks(n):
            got = payload([sh[j] for j in range(n) if m >> j & 1], m, d, p, dl)
            assert got[:dl] == oracle_decode(sh, m, d, p, dl) == batch and not any(got[dl:]), (dl, m)


# ---- GPU ------------------------------------------------------------------------------------------------------------
def _oracle_check(out, recs, batch, held_of, d, p):
    """every record's payload bytes against the oracle's decode from the entry's first d held shards"""
    for g, s, off, dl in recs:
        b = batch[(g, s)]
        assert out[off:off + dl].tobytes() == oracle_decode(coded(b, d, p), held_of(g, s), d, p, dl), (g, s)


def _no_status(ctx):
    st = ctx.device_status()
    assert not st & (EXEC_FULL | EXEC_NULL), st


@pytest.mark.gpu
@pytest.mark.parametrize("n", range(3, 13))
def test_leader_decodes_every_held_mask(n):
    """G = every mask + 1 groups, entry k of group g of length lengths[(g + k) % K]: one execute call covers every
    (mask, length) cell.  The fully held log runs through the gather-only payload kernel before the recon view and
    through the regenerating one after it, byte-identically; then each group's mask is written into held, the planes of
    the shards it lacks are poisoned, and the regen kernel must still execute the batches."""
    import torch
    from summerset_b200.engine import RaftEngine
    ctx = tx._ctx()
    d, p = code(n)
    ms, lens = masks(n), lengths(d)
    G, K, W = len(ms) + 1, len(lens), 16
    few_g, few_s = G - 1, K // 2 + 1                              # the group whose walk stops at d - 1 shards
    full = (1 << n) - 1
    rng = random.Random(6000 + n)
    eng = RaftEngine(ctx, G, n, craft=True, window=W)
    ev, lv = eng.exec_view(), eng.log_view()
    eng.curr_term.fill_(1)
    size = lambda dl: pitch(-(-dl // d))
    stride = max(sum(size(lens[(g + k) % K]) for g in range(G)) for k in range(K))
    stores, batch = [], {}
    for k in range(K):                                            # call k proposes slot k + 1 of every group
        store, got = tx._propose(eng, 0, [lens[(g + k) % K] for g in range(G)], rng, n, stride)
        assert sorted(got) == list(range(G)) and {s for s, _ in got.values()} == {k + 1}
        stores.append(store)
        for g, (s, b) in got.items():
            batch[(g, s)] = b
    eng.last_commit.fill_(K)
    held = {(g, s): (ms[g] if g < len(ms) else few_mask(n) if s == few_s else full) for g in range(G) for s in range(1, K + 1)}
    state = lambda hm: [dict(start=0, last_exec=0, lc=K, ent={s: (len(batch[(g, s)]), hm(g, s)) for s in range(1, K + 1)})
                        for g in range(G)]

    def run(want):
        ev["last_exec"].zero_()
        ctx.device_status()
        o, out = tx._execute(eng, G * K, 1 << 40, want["totals"][1])
        tx._check(o, out, want, lambda g, s: batch[(g, s)], 1 << 40)
        assert ev["last_exec"].cpu().tolist() == want["last_exec"]
        _no_status(ctx)
        return o, out

    # the same fully held log through both kernels
    every = walk(state(lambda g, s: full), G * K, 1 << 40)
    assert len(every["records"]) == G * K
    o_a, out_a = run(every)                                       # the gather-only payload kernel
    rv = eng.recon_view()
    assert (rv["held"][:, 1:K + 1] == full).all()
    o_b, out_b = run(every)                                       # the regenerating payload kernel, every mask full
    assert np.array_equal(out_a, out_b) and all(np.array_equal(o_a[k], o_b[k]) for k in o_a)
    # each group's mask, the other shards' plane slots poisoned
    hv = np.zeros((G, W), dtype=np.int64)
    for (g, s), m in held.items():
        hv[g][s % W] = m
    rv["held"].copy_(torch.tensor(hv, dtype=torch.int32, device="cuda:0"))
    addr = lv["shard_addr"].cpu().numpy()
    want = walk(state(lambda g, s: held[(g, s)]), G * K, 1 << 40, need_d=d)
    assert want["last_exec"][few_g] == few_s - 1 and len(want["records"]) == (G - 1) * K + few_s - 1
    planes = [x.cpu().numpy() for x in stores]
    for poison in (0xA5, 0x00):
        for (g, s), m in held.items():
            pl = planes[s - 1]
            off = int(addr[g][s % W]) - stores[s - 1].data_ptr()
            for j in range(n):
                if not m >> j & 1:
                    pl[j, off:off + size(len(batch[(g, s)]))] = poison
        for x, pl in zip(stores, planes):
            x.copy_(torch.from_numpy(pl))
        o, out = run(want)
        if poison:
            _oracle_check(out, want["records"], batch, lambda g, s: held[(g, s)], d, p)
    eng.close()
    del stores


@pytest.mark.gpu
@pytest.mark.parametrize("n", range(3, 33))
def test_follower_decodes_every_held_mask(n):
    """G = every mask + 1 groups installed through the follower's views, entry k of group g of length
    lengths[(g + k) % K]; slot pads poisoned, every entry 16 bytes past a 32-byte boundary"""
    from summerset_b200.engine import Follower
    ctx = tx._ctx()
    d, p = code(n)
    ms, lens = masks(n), lengths(d)
    G, K, W = len(ms) + 1, len(lens), 16
    few_g, few_s = G - 1, K // 2 + 1
    full = (1 << n) - 1
    rng = random.Random(7000 + n)
    fol = Follower(ctx, G, n, 0, window=W)
    groups, batch = [], {}
    for g in range(G):
        ent = {}
        for k in range(K):
            b = rng.randbytes(lens[(g + k) % K])
            ent[k + 1] = (len(b), ms[g] if g < len(ms) else few_mask(n) if k + 1 == few_s else full, b)
            batch[(g, k + 1)] = b
        groups.append(dict(start=0, le=K + 1, lc=K, last_exec=0, ent=ent))
    store = tx._install(fol, G, groups, W, fill=0xA5, skew=16)
    model = [dict(start=0, last_exec=0, lc=K, ent={s: e[:2] for s, e in gr["ent"].items()}) for gr in groups]
    want = walk(model, G * K, 1 << 40, need_d=d)
    assert want["last_exec"][few_g] == few_s - 1 and len(want["records"]) == (G - 1) * K + few_s - 1
    ctx.device_status()
    o, out = tx._execute(fol, G * K, 1 << 40, want["totals"][1])
    tx._check(o, out, want, lambda g, s: batch[(g, s)], 1 << 40)
    assert fol.last_exec.cpu().tolist() == want["last_exec"]
    _no_status(ctx)
    _oracle_check(out, want["records"], batch, lambda g, s: groups[g]["ent"][s][1], d, p)
    del store
    fol.close()


# ---- GPU: past the grid caps ----------------------------------------------------------------------------------------
def _expected(rec_len, src, src_off):
    """-> (rec_off, the output buffer): each record's bytes src[src_off : src_off + rec_len] in a round_up(len, 16)
    region, zero pad, regions back to back"""
    size = (rec_len + 15) & ~15
    rec_off = np.concatenate(([0], np.cumsum(size)[:-1])).astype(np.int64)
    out = np.zeros(int(size.sum()), dtype=np.uint8)
    start = np.concatenate(([0], np.cumsum(rec_len)[:-1]))
    within = np.arange(int(rec_len.sum())) - np.repeat(start, rec_len)
    out[np.repeat(rec_off, rec_len) + within] = src[np.repeat(src_off, rec_len) + within]
    return rec_off, out


def _execute_all(obj, nrec, nbytes):
    """one execute call with room for exactly nrec records and nbytes, canaries after them"""
    return tx._execute(obj, nrec, nbytes, nbytes)


def _compare(o, out, rec_group, rec_slot, rec_len, rec_off, want_out):
    n = len(rec_group)
    assert tuple(int(x) for x in o["totals"]) == (n, len(want_out))
    assert np.array_equal(o["rec_group"][:n], rec_group) and np.array_equal(o["rec_slot"][:n], rec_slot)
    assert np.array_equal(o["rec_len"][:n], rec_len) and np.array_equal(o["rec_off"][:n], rec_off)
    assert np.array_equal(out[:len(want_out)], want_out) and (out[len(want_out):] == 0xA5).all()


def _propose_np(eng, lens, rng, stride):
    """one propose round of random batches (numpy) -> (store, arena, data_off, slot_out)"""
    import torch
    dev = "cuda:0"
    arena = rng.integers(0, 256, int(lens.sum()) + 1, dtype=np.uint8)
    off = np.concatenate(([0], np.cumsum(lens)[:-1])).astype(np.int64)
    store = torch.zeros((eng.P + 1, stride), dtype=torch.uint8, device=dev)
    wal = torch.zeros(len(lens) * 128, dtype=torch.uint8, device=dev)     # a one-shard LogEntry of L <= 16 fits 128 bytes
    o = eng.propose(0, torch.from_numpy(arena).to(dev), torch.from_numpy(off).to(dev),
                    torch.from_numpy(lens.astype(np.int32)).to(dev), store, wal)
    slots = o["slot_out"].cpu().numpy()
    return store, arena, off, slots


@pytest.mark.gpu
def test_leader_regen_past_the_payload_grid_cap():
    """sm_count * 64 * 8 + 4099 records in one call, more than the capped grid of the regenerating payload kernel has warps:
    two entries per group (one in the last group), full and partial masks mixed, the planes of the missing shards
    poisoned"""
    import torch
    from summerset_b200.engine import RaftEngine
    ctx = tx._ctx()
    n = 5
    d, p = code(n)
    nrec = ctx.sm_count * 64 * 8 + 4099
    G, W = (nrec + 1) // 2, 4
    rng = np.random.default_rng(8)
    eng = RaftEngine(ctx, G, n, craft=True, window=W)
    ev, lv = eng.exec_view(), eng.log_view()
    eng.curr_term.fill_(1)
    lens = rng.integers(1, 16 * d + 1, (G, 2))                    # L <= 16: a 32-byte slot per plane and group
    lens[G - 1, 1] = 0                                            # nrec is odd
    stride = G * 32
    rounds = [_propose_np(eng, lens[:, k], rng, stride) for k in range(2)]
    for k, (store, _, _, slots) in enumerate(rounds):
        assert np.array_equal(slots, np.where(lens[:, k] > 0, k + 1, -1))
    rv = eng.recon_view()
    ms = np.array(masks(n))
    held = ms[rng.integers(0, len(ms), (G, 2))]
    assert (held == (1 << n) - 1).any() and (held & ((1 << d) - 1) != (1 << d) - 1).any()
    hv = rv["held"].cpu().numpy()
    hv[:, 1:3] = held
    rv["held"].copy_(torch.from_numpy(hv).to("cuda:0"))
    addr = lv["shard_addr"].cpu().numpy()
    for k, (store, _, _, _) in enumerate(rounds):
        live = lens[:, k] > 0
        assert np.array_equal(addr[live, k + 1] - store.data_ptr(), 32 * np.nonzero(live)[0])
        pl = store.cpu().numpy().reshape(n, G, 32)
        for j in range(n):
            pl[j][live & (held[:, k] >> j & 1 == 0)] = 0xA5
        store.copy_(torch.from_numpy(pl.reshape(n, stride)))
    eng.last_commit.copy_(eng.log_end - 1)
    valid = lens > 0
    assert valid.sum() == nrec
    rec_group, rec_k = np.nonzero(valid)
    rec_len = lens[valid]
    src = np.concatenate([rounds[0][1], rounds[1][1]])
    src_off = np.where(rec_k == 0, rounds[0][2][rec_group], len(rounds[0][1]) + rounds[1][2][rec_group])
    rec_off, want_out = _expected(rec_len, src, src_off)
    ctx.device_status()
    o, out = _execute_all(eng, nrec, len(want_out))
    _compare(o, out, rec_group, rec_k + 1, rec_len, rec_off, want_out)
    assert np.array_equal(ev["last_exec"].cpu().numpy(), valid.sum(1))
    _no_status(ctx)
    eng.close()
    del rounds


def _sample_check(out, rec_off, rec_len, src, src_off, held, d, p, rng):
    """a seeded sample of records against the oracle's decode"""
    for r in rng.choice(len(rec_len), 64, replace=False):
        b = src[src_off[r]:src_off[r] + rec_len[r]].tobytes()
        assert out[rec_off[r]:rec_off[r] + rec_len[r]].tobytes() == oracle_decode(coded(b, d, p), int(held[r]), d, p, len(b)) == b


@pytest.mark.gpu
def test_leader_past_the_group_grid_cap():
    """sm_count * 64 * 256 + 1000 groups, more than the capped grids of the leader's exec_count_kernel and
    exec_place_kernel have threads: one short entry per group, some not proposed and some not committed, so the
    group scan places records unevenly; the gather-only payload kernel strides past its cap too"""
    import torch
    from summerset_b200.engine import RaftEngine
    ctx = tx._ctx()
    n = 3
    d, p = code(n)
    G = ctx.sm_count * 64 * 256 + 1000
    rng = np.random.default_rng(9)
    eng = RaftEngine(ctx, G, n, craft=True, window=2)
    ev = eng.exec_view()
    eng.curr_term.fill_(1)
    lens = np.where(rng.random(G) < 0.05, 0, rng.integers(1, 32 * d + 1, G))   # L <= 32: a 32-byte slot per plane
    store, arena, off, slots = _propose_np(eng, lens, rng, G * 32)
    assert np.array_equal(slots, np.where(lens > 0, 1, -1))
    lc = np.where((lens > 0) & (rng.random(G) >= 0.05), 1, 0)
    eng.last_commit.copy_(torch.from_numpy(lc.astype(np.int32)).to("cuda:0"))
    rec_group = np.nonzero(lc)[0]
    rec_len = lens[rec_group]
    rec_off, want_out = _expected(rec_len, arena, off[rec_group])
    ctx.device_status()
    o, out = _execute_all(eng, len(rec_group), len(want_out))
    _compare(o, out, rec_group, np.ones(len(rec_group)), rec_len, rec_off, want_out)
    assert np.array_equal(ev["last_exec"].cpu().numpy(), lc)
    _no_status(ctx)
    _sample_check(out, rec_off, rec_len, arena, off[rec_group], np.full(len(rec_group), (1 << n) - 1), d, p, rng)
    eng.close()
    del store


@pytest.mark.gpu
def test_follower_past_the_group_grid_cap():
    """sm_count * 64 * 256 + 1000 groups, more than the capped grids of the follower's exec_count_kernel and
    exec_place_kernel have threads, and far more records than its exec_payload_kernel's capped grid has warps: one short entry per group
    installed through the views, held masks of every decodable kind, some of d - 1 shards (the walk stops) and some
    not committed; entries 16 bytes past a 32-byte boundary, slot pads poisoned"""
    import torch
    from summerset_b200.engine import Follower
    ctx = tx._ctx()
    n = 5
    d, p = code(n)
    G, W, Kp = ctx.sm_count * 64 * 256 + 1000, 2, 4096
    rng = np.random.default_rng(10)
    dev = "cuda:0"
    # a pool of batches, coded by the oracle; each entry holds its own copy of one of them
    plen = rng.integers(1, 16 * d + 1, Kp)                         # L <= 16
    pool = rng.integers(0, 256, int(plen.sum()), dtype=np.uint8)
    poff = np.concatenate(([0], np.cumsum(plen)[:-1]))
    psh = np.full((Kp, n, 32), 0xA5, dtype=np.uint8)
    for i in range(Kp):
        for j, x in enumerate(coded(pool[poff[i]:poff[i] + plen[i]].tobytes(), d, p)):
            psh[i, j, :len(x)] = x
    ms = np.array(masks(n) + [few_mask(n)])
    which = rng.integers(0, Kp, G)
    held = ms[rng.integers(0, len(ms), G)]
    lc = np.where(rng.random(G) < 0.05, 0, 1)
    blob = np.full(16 + G * n * 32 + 16, 0xA5, dtype=np.uint8)
    slots = blob[16:16 + G * n * 32].reshape(G, n, 32)
    for m in ms:
        at = np.nonzero(held == m)[0]
        for k, j in enumerate(j for j in range(n) if m >> j & 1):
            slots[at, k] = psh[which[at], j]
    fol = Follower(ctx, G, n, 0, window=W)
    store = torch.from_numpy(blob).to(dev)
    col = lambda v, dt: torch.from_numpy(np.stack([np.zeros(G, dtype=dt), v.astype(dt)], 1)).to(dev)
    fol.shard_addr.copy_(col(store.data_ptr() + 16 + np.arange(G, dtype=np.int64) * n * 32, np.int64))
    fol.held.copy_(col(held, np.int32))
    fol.data_len.copy_(col(plen[which], np.int32))
    fol.term.copy_(col(np.ones(G), np.int64))
    fol.start_slot.zero_()
    fol.log_end.fill_(2)
    fol.last_commit.copy_(torch.from_numpy(lc.astype(np.int64)).to(dev))
    fol.last_exec.zero_()
    run = (lc == 1) & (held != few_mask(n))
    rec_group = np.nonzero(run)[0]
    rec_len = plen[which[rec_group]]
    rec_off, want_out = _expected(rec_len, pool, poff[which[rec_group]])
    assert len(rec_group) > 16 * ctx.sm_count * 64 * 8
    ctx.device_status()
    o, out = _execute_all(fol, len(rec_group), len(want_out))
    _compare(o, out, rec_group, np.ones(len(rec_group)), rec_len, rec_off, want_out)
    assert np.array_equal(fol.last_exec.cpu().numpy(), run.astype(np.int64))
    _no_status(ctx)
    _sample_check(out, rec_off, rec_len, pool, poff[which[rec_group]], held[rec_group], d, p, rng)
    fol.close()
    del store


# ---- GPU: fail-over end to end at the populations the closed loop in tests/test_craft_stepup.py skips -----------
@pytest.mark.gpu
@pytest.mark.parametrize("n", [3, 4, 6, 8, 9, 10, 11, 12])
@pytest.mark.parametrize("full_copy", [False, True])
def test_closed_loop_fail_over(n, full_copy):
    ts._failover(n, full_copy)
