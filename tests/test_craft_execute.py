"""CRaft execution: ss_engine_craft_execute, ss_follower_execute and the full-copy commit threshold
(ss_engine_craft_set_full_copy).

`walk` restates both execution walks -- the leader's (the execution half of handle_msg_append_entries_reply's success
branch, craft/messages.rs:316-359) and the follower's (handle_msg_append_entries, craft/messages.rs:198-240) -- with the
record placement, the capacity cuts and last_exec of ss_acceptor_execute's contract.  `payload` restates the payload
warp (csrc/exec_walk.cuh): 16-byte output columns gathered across shard boundaries, a missing data shard regenerated
with the inverse of M[first d held shards].  The leader's and the follower's per-message restatements and the bincode
encoders come from tests/test_craft_leader.py and tests/test_follower.py.  GPU tests compare every record, offset, zero
pad, last_exec and payload byte with the restatement and with the request batches themselves.
"""
from __future__ import annotations

import ctypes as C
import functools
import random

import numpy as np
import pytest

from oracle import pyoracle as oracle
from tests import test_craft_leader as tl
from tests import test_follower as tf

EXEC_FULL, EXEC_NULL = 32, 64
r16, pitch = tl.r16, tl.pitch
popc = lambda x: bin(x).count("1")


# ---- the restatements ---------------------------------------------------------------------------------------------
def walk(groups, rec_capacity, out_capacity, need_d=0):
    """groups: [dict(start, last_exec, lc, ent={slot: (data_len, held)})]; need_d > 0: the follower's held-shard stop.
    -> dict(records [(group, slot, off, data_len)] in record order, last_exec [G], full, null, totals (records, bytes))"""
    plans = []
    for gr in groups:
        s, run, null = max(gr["last_exec"] + 1, gr["start"]), [], False
        while s <= gr["lc"]:
            dl, held = gr["ent"][s]
            if need_d and popc(held) < need_d:
                break
            if dl == 0:
                null = True
                break
            run.append((s, dl))
            s += 1
        plans.append((run, null))
    ro_at, bo_at, ro, bo = [], [], 0, 0
    for run, _ in plans:                                          # exclusive scans in group order
        ro_at.append(ro)
        bo_at.append(bo)
        ro += len(run)
        bo += sum(r16(dl) for _, dl in run)
    res = dict(records=[], last_exec=[], full=False, null=False, totals=(ro, bo))
    for g, ((run, null), gr) in enumerate(zip(plans, groups)):
        ro, bo, done = ro_at[g], bo_at[g], 0
        for s, dl in run:
            if ro >= rec_capacity or bo > out_capacity or r16(dl) > out_capacity - bo:
                res["full"] = True
                break
            res["records"].append((g, s, bo, dl))
            ro, bo, done = ro + 1, bo + r16(dl), done + 1
        else:
            res["null"] |= null
        res["last_exec"].append(run[done - 1][0] if done else gr["last_exec"])
    return res


# GF(2^8) with the code's polynomial 0x11D
_EXP, _LOG = [0] * 512, [0] * 256
_v = 1
for _i in range(255):
    _EXP[_i] = _EXP[_i + 255] = _v
    _LOG[_v] = _i
    _v = (_v << 1) ^ (0x11D if _v & 0x80 else 0)
gmul = lambda a, b: _EXP[_LOG[a] + _LOG[b]] if a and b else 0
_MUL = np.array([[gmul(a, b) for b in range(256)] for a in range(256)], dtype=np.uint8)   # _MUL[a][x] = a * x


@functools.lru_cache(maxsize=None)
def decode_rows(d, p, held):
    """inverse(M[the first d held shards]) by the warp's Gauss-Jordan: pivots in column order, rows never swapped;
    -> rows[i] = the coefficients of data shard i over sources 0..d-1"""
    m = oracle.rs_matrix(d, p)
    src = [j for j in range(d + p) if held >> j & 1][:d]
    a = [[int(m[r][c]) for c in range(d)] for r in src]
    inv = [[int(c == r) for c in range(d)] for r in range(d)]
    piv, used = [0] * d, 0
    for c in range(d):
        f = [a[r][c] for r in range(d)]
        cand = [r for r in range(d) if f[r] and not used >> r & 1]
        p_ = cand[0]
        used |= 1 << p_
        piv[c] = p_
        sc = _EXP[255 - _LOG[f[p_]]]
        a[p_] = [gmul(x, sc) for x in a[p_]]
        inv[p_] = [gmul(x, sc) for x in inv[p_]]
        for r in range(d):
            if r != p_ and f[r]:
                a[r] = [x ^ gmul(f[r], y) for x, y in zip(a[r], a[p_])]
                inv[r] = [x ^ gmul(f[r], y) for x, y in zip(inv[r], inv[p_])]
    return [inv[piv[i]] for i in range(d)]


def payload(stored, held, d, p, dl):
    """the bytes the warp writes: stored[k] = the held shard of rank k (L bytes); round_up(dl, 16) bytes, zero past dl"""
    L = -(-dl // d)
    rows = decode_rows(d, p, held) if held & ((1 << d) - 1) != (1 << d) - 1 else None
    src = [np.frombuffer(bytes(x), dtype=np.uint8)[:L] for x in stored]

    def shard(i):                                                 # data shard i: held, or regenerated from sources 0..d-1
        if held >> i & 1:
            return src[popc(held & ((1 << i) - 1))]
        acc = np.zeros(L, dtype=np.uint8)
        for q in range(d):
            acc ^= _MUL[rows[i][q]][src[q]]
        return acc

    data = np.stack([shard(i) for i in range(d)])
    pos = np.arange(dl)
    out = np.zeros(r16(dl), dtype=np.uint8)
    out[:dl] = data[pos // L, pos % L]                            # byte pos of a 16-byte column, which may straddle shards
    return out.tobytes()


def coded(batch, d, p):
    """every shard of RSCodeword::from_data(batch) + compute_parity"""
    return [np.frombuffer(s, dtype=np.uint8) for s in tl.encode(batch, d, p)]


# ---- CPU: hand-worked walks ---------------------------------------------------------------------------------------
def _groups():
    # group 0: slots 1..4 committed; group 1: a null entry at 3; group 2: nothing committed past last_exec;
    # group 3: last_exec behind start_slot (advanced past it by a host)
    return [dict(start=0, last_exec=0, lc=4, ent={s: (10 * s, 0) for s in range(1, 6)}),
            dict(start=0, last_exec=0, lc=5, ent={1: (17, 0), 2: (16, 0), 3: (0, 0), 4: (5, 0), 5: (5, 0)}),
            dict(start=2, last_exec=3, lc=3, ent={2: (1, 0), 3: (1, 0)}),
            dict(start=6, last_exec=2, lc=7, ent={6: (33, 0), 7: (1, 0)})]


def test_walk_places_records_by_group_scans():
    r = walk(_groups(), 100, 1 << 20)
    assert [(g, s) for g, s, _, _ in r["records"]] == [(0, 1), (0, 2), (0, 3), (0, 4), (1, 1), (1, 2), (3, 6), (3, 7)]
    assert [off for _, _, off, _ in r["records"]] == [0, 16, 48, 80, 128, 160, 176, 224]
    assert r["last_exec"] == [4, 2, 3, 7] and r["null"] and not r["full"] and r["totals"] == (8, 240)


@pytest.mark.parametrize("rec_cap,out_cap,n,last_exec", [(3, 1 << 20, 3, [3, 0, 3, 2]), (5, 1 << 20, 5, [4, 1, 3, 2]),
                                                         (100, 127, 3, [3, 0, 3, 2]), (100, 128, 4, [4, 0, 3, 2]),
                                                         (100, 160, 5, [4, 1, 3, 2]), (0, 1 << 20, 0, [0, 0, 3, 2])])
def test_walk_capacity_cuts_are_a_prefix(rec_cap, out_cap, n, last_exec):
    r = walk(_groups(), rec_cap, out_cap)
    assert len(r["records"]) == n and r["last_exec"] == last_exec and r["full"]
    assert not r["null"]                                          # the group with the null entry was cut before it
    assert r["totals"] == (8, 240)                                # the totals count what the walk asked for


def test_walk_drains_over_calls():
    groups, seen, calls = _groups(), [], 0
    while True:
        r = walk(groups, 2, 64)
        seen += [(g, s) for g, s, _, _ in r["records"]]
        for gr, le in zip(groups, r["last_exec"]):
            gr["last_exec"] = le
        calls += 1
        if not r["records"]:
            break
    assert seen == [(0, 1), (0, 2), (0, 3), (0, 4), (1, 1), (1, 2), (3, 6), (3, 7)] and calls == 6


def test_walk_starts_after_an_advance_and_stops_at_few_shards():
    g = dict(start=0, last_exec=0, lc=6, ent={s: (9, 0b00111 if s != 5 else 0b00001) for s in range(1, 8)})
    assert walk([g], 10, 1 << 10, need_d=3)["last_exec"] == [4]   # the follower stops at the 1-shard entry
    g["last_exec"], g["start"] = 1, 3                             # a host advanced start_slot past last_exec
    r = walk([g], 10, 1 << 10, need_d=3)
    assert [s for _, s, _, _ in r["records"]] == [3, 4] and not r["null"]
    assert [s for _, s, _, _ in walk([g], 10, 1 << 10)["records"]] == [3, 4, 5, 6]   # the leader has no such stop


@pytest.mark.parametrize("dl", [1, 2, 15, 16, 17, 31, 32, 46, 47, 48, 49, 50, 64, 65])
@pytest.mark.parametrize("held", [0b11111, 0b00111, 0b11110, 0b11101, 0b11011, 0b11100, 0b10110, 0b01011])
def test_payload_bytes_at_rs32(dl, held):
    # RS(3,2): L = ceil(dl / 3) from 1 to 22, so columns straddle shards (always for L < 16) and data_len % 3 varies;
    # held patterns with none, one (shard 0, 1 or 2) and two data shards missing
    d, p = 3, 2
    rng = np.random.default_rng(dl * 64 + held)
    batch = rng.integers(0, 256, dl, dtype=np.uint8).tobytes()
    sh = coded(batch, d, p)
    stored = [sh[j] for j in range(d + p) if held >> j & 1]
    got = payload(stored, held, d, p, dl)
    assert got[:dl] == batch and not any(got[dl:])
    first = [j for j in range(d + p) if held >> j & 1][:d]
    rec = [sh[j].copy() if j in first else None for j in range(d + p)]
    assert oracle.rs_reconstruct(d, p, rec, data_only=True) == 0
    assert got[:dl] == b"".join(rec[i].tobytes() for i in range(d))[:dl]


def test_refusals_without_a_device():
    from summerset_b200 import _lib
    lib = _lib.load()

    def refused(rc, why):
        assert rc == _lib.SS_ERR_INVALID_ARG and why in lib.ss_last_error().decode(), (rc, lib.ss_last_error(), why)

    b = [16] * 4
    refused(lib.ss_engine_craft_execute(None, None, 0, *b, 1, None), "null buffer")
    refused(lib.ss_engine_craft_execute(None, 16, 0, None, 16, 16, 16, 1, None), "null buffer")
    refused(lib.ss_engine_craft_execute(None, 8, 0, *b, 1, None), "16-byte aligned")
    refused(lib.ss_engine_craft_execute(None, 16, 0, *b, 1, None), "null engine")
    refused(lib.ss_engine_craft_exec_view_get(None, None), "null view")
    refused(lib.ss_engine_craft_exec_view_get(None, C.byref(_lib.CraftExecView())), "null engine")
    refused(lib.ss_engine_craft_set_full_copy(None, 1), "null engine")
    refused(lib.ss_follower_execute(None, 16, 0, *b, 1, None), "null follower")
    refused(lib.ss_follower_exec_view_get(None, C.byref(_lib.FollowerExecView())), "null argument")


# ---- GPU ------------------------------------------------------------------------------------------------------------
def _ctx():
    from summerset_b200.api import Context
    return Context(0)


def _execute(obj, rec_cap, out_cap, room):
    """obj.execute into a buffer of room bytes (at least what the call writes) and canaries after it -> (outputs as
    numpy arrays, the buffer)"""
    import torch
    out = torch.full((min(room, out_cap) + 64,), 0xA5, dtype=torch.uint8, device="cuda:0")
    o = obj.execute(out, rec_cap, out_cap)
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in o.items()}, out.cpu().numpy()


def _check(o, out, want, batch_of, out_cap):
    """every record, offset, payload byte and zero pad against the restatement and the batches"""
    n = len(want["records"])
    for k, (g, s, off, dl) in enumerate(want["records"]):
        assert (int(o["rec_group"][k]), int(o["rec_slot"][k]), int(o["rec_off"][k]), int(o["rec_len"][k])) == (g, s, off, dl), k
        assert out[off:off + dl].tobytes() == batch_of(g, s), (g, s)
        assert not out[off + dl:off + r16(dl)].any()
    used = want["records"][-1][2] + r16(want["records"][-1][3]) if n else 0
    assert (out[used:] == 0xA5).all() and used <= out_cap
    assert tuple(int(x) for x in o["totals"]) == want["totals"]


@pytest.mark.gpu
def test_refusals_on_engines():
    import torch
    from summerset_b200 import _lib
    from summerset_b200.engine import Follower, LeaderEngine, RaftEngine
    ctx = _ctx()
    lib = ctx.lib
    out = torch.zeros(4096, dtype=torch.uint8, device="cuda:0")
    paxos = LeaderEngine(ctx, "rspaxos", 4, 5, 1, 16)
    raft = RaftEngine(ctx, 4, 5, craft=False)
    for e in (paxos, raft):
        with pytest.raises(_lib.SummersetError, match="CRaft"):
            RaftEngine.execute(e, out, 8)
        with pytest.raises(_lib.SummersetError, match="CRaft"):
            RaftEngine.exec_view(e)
        assert lib.ss_engine_craft_set_full_copy(e.h, 1) == _lib.SS_ERR_INVALID_ARG
        assert "CRaft" in lib.ss_last_error().decode()
    appended = RaftEngine(ctx, 4, 5, craft=True)
    appended.append(torch.ones(4, dtype=torch.int32, device="cuda:0"))
    with pytest.raises(_lib.SummersetError, match="raft_append"):
        appended.execute(out, 8)
    appended.set_full_copy(True)                                  # the threshold switch works with or without the log
    assert appended.threshold == 3
    fol = Follower(ctx, 4, 5, 0)
    with pytest.raises(_lib.SummersetError, match="16-byte"):
        fol.execute(out[1:], 8)
    torch.cuda.synchronize()
    for e in (paxos, raft, appended, fol):
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [5, 7, 9])
def test_full_copy_threshold_switch(n):
    import torch
    from summerset_b200.engine import RaftEngine
    ctx = _ctx()
    G, W, P = 64, 16, n - 1
    maj = n // 2 + 1
    rng = random.Random(n)
    dev = "cuda:0"
    for f in range(0, n - maj + 1):
        eng = RaftEngine(ctx, G, n, fault_tolerance=f, craft=True, window=W)
        assert eng.threshold == maj + f
        le = [rng.randint(2, W) for _ in range(G)]
        terms = np.zeros((G, W), dtype=np.int32)
        match = np.zeros((P, G), dtype=np.int32)
        for g in range(G):
            terms[g, 1:le[g]] = sorted(rng.choice((2, 3)) for _ in range(le[g] - 1))   # older-term entries first
            acks = rng.randint(maj - 1, maj + f - 2) if f else maj - 1                    # majority <= 1 + acks < majority + f
            for q in rng.sample(range(P), acks):
                match[q][g] = rng.randint(1, le[g] - 1)
        eng.curr_term.fill_(3)
        eng.log_end.copy_(torch.tensor(le, dtype=torch.int32, device=dev))
        eng.terms.copy_(torch.tensor(terms, device=dev))
        eng.match.copy_(torch.tensor(match, device=dev))

        def new_commit(thr):
            # messages.rs:254-275: the highest slot of the current term that 1 + matches >= threshold hold
            out = []
            for g in range(G):
                c = 0
                for s in range(1, le[g]):
                    if terms[g][s] == 3 and 1 + sum(match[q][g] >= s for q in range(P)) >= thr:
                        c = s
                out.append(c)
            return out

        eng.tick()
        assert eng.last_commit.cpu().tolist() == ([0] * G if f else new_commit(maj))
        eng.set_full_copy(True)
        assert eng.threshold == maj
        eng.last_commit.zero_()
        eng.tick()
        want = new_commit(maj)
        assert eng.last_commit.cpu().tolist() == want and (f == 0 or any(want))
        eng.set_full_copy(False)
        assert eng.threshold == maj + f
        eng.last_commit.zero_()
        eng.tick()
        assert eng.last_commit.cpu().tolist() == ([0] * G if f else want)
        eng.close()


def _propose(eng, me, lens, rng, n, stride):
    """one propose round; -> (store, {group: (slot, batch)})"""
    import torch
    dev = "cuda:0"
    batches = [rng.randbytes(x) for x in lens]
    arena, offs = bytearray(), []
    for b in batches:
        arena += bytes(rng.randint(0, 3))
        offs.append(len(arena))
        arena += b
    store = torch.zeros((n, stride), dtype=torch.uint8, device=dev)
    o = eng.propose(me, torch.tensor(np.frombuffer(bytes(arena) + b"\0", dtype=np.uint8), device=dev),
                    torch.tensor(offs, dtype=torch.int64, device=dev), torch.tensor(lens, dtype=torch.int32, device=dev), store,
                    torch.zeros(1 << 22, dtype=torch.uint8, device=dev))
    slots = o["slot_out"].cpu().tolist()
    return store, {g: (slots[g], batches[g]) for g in range(len(lens)) if lens[g] and slots[g] >= 0}


@pytest.mark.gpu
@pytest.mark.parametrize("n", [3, 5, 7, 9, 12])
def test_leader_execute_matches_the_restatement(n):
    import torch
    from summerset_b200.engine import RaftEngine
    ctx = _ctx()
    G, W, me = 24, 8, 0
    d = n // 2 + 1
    rng = random.Random(1000 + n)
    dev = "cuda:0"
    lens_all = [1, 15, 16, 17, 16 * d - 1, 16 * d + 1, 64 * 1024, 3, 100, 4095]
    stride = G * pitch(-(-65536 // d)) * 2
    eng = RaftEngine(ctx, G, n, craft=True, window=W)
    ev = eng.exec_view()
    lv = eng.log_view()
    assert ev["last_exec"].cpu().tolist() == [0] * G
    eng.curr_term.fill_(2)
    keep, batch = [], {}
    state = [dict(start=0, last_exec=0, lc=0, ent={}) for _ in range(G)]
    for rnd in range(12):
        for _ in range(2):                                        # several entries per group per round
            lens = [0 if rng.random() < 0.2 else rng.choice(lens_all) for _ in range(G)]
            store, got = _propose(eng, me, lens, rng, n, stride)
            keep.append(store)
            for g, (s, b) in got.items():
                batch[(g, s)] = b
                state[g]["ent"][s] = (len(b), 0)
        le = eng.log_end.cpu().tolist()
        lc = [le[g] - 1 if rng.random() < 0.6 else rng.randint(st["lc"], le[g] - 1) for g, st in enumerate(state)]
        eng.last_commit.copy_(torch.tensor(lc, dtype=torch.int32, device=dev))
        eng.last_snap.copy_(eng.last_commit)
        for st, c in zip(state, lc):
            st["lc"] = c
        cut = rnd % 4 == 3
        want = walk(state, 1 << 20, 1 << 26)
        if cut:                                                   # every record and byte boundary of this call, drained
            recs = want["records"]
            bounds = [(k, 1 << 26) for k in range(1, len(recs) + 1)] + [(1 << 20, off) for _, _, off, _ in recs] + \
                     [(1 << 20, off + r16(dl) - 1) for _, _, off, dl in recs[:8]]
            for rc, oc in bounds:
                w = walk(state, rc, oc)
                o, out = _execute(eng, rc, oc, want["totals"][1])
                _check(o, out, w, lambda g, s: batch[(g, s)], oc)
                assert bool(ctx.device_status() & EXEC_FULL) == w["full"]
                assert ev["last_exec"].cpu().tolist() == w["last_exec"]
                ev["last_exec"].copy_(torch.tensor([st["last_exec"] for st in state], dtype=torch.int64, device=dev))
            calls = 0
            while True:                                           # drain with room for three records a call
                w = walk(state, 3, 1 << 26)
                o, out = _execute(eng, 3, 1 << 26, want["totals"][1])
                _check(o, out, w, lambda g, s: batch[(g, s)], 1 << 26)
                for st, x in zip(state, w["last_exec"]):
                    st["last_exec"] = x
                calls += 1
                if not w["records"]:
                    break
            assert calls > 1
        else:
            o, out = _execute(eng, 1 << 12, 1 << 26, want["totals"][1])
            _check(o, out, want, lambda g, s: batch[(g, s)], 1 << 26)
            for st, x in zip(state, want["last_exec"]):
                st["last_exec"] = x
        ctx.device_status()
        assert ev["last_exec"].cpu().tolist() == [st["last_exec"] for st in state]
        # retire what executed: the ring wraps over the rounds
        upto = ev["last_exec"].clone()
        eng.advance_log(upto)
        ls = lv["log_start"].cpu().tolist()
        for st, s in zip(state, ls):
            assert s == max(st["start"], st["last_exec"])          # last_snap = last_commit >= last_exec
            st["start"] = s
    assert max(le) > 2 * W
    # a null entry installed through the log view stops the walk with the status bit: everything executes and retires,
    # one more entry per group, group 3's made null
    le = eng.log_end.cpu().tolist()
    eng.last_commit.copy_(torch.tensor([x - 1 for x in le], dtype=torch.int32, device=dev))
    eng.last_snap.copy_(eng.last_commit)
    for st, x in zip(state, le):
        st["lc"] = x - 1
    w = walk(state, 1 << 12, 1 << 26)
    o, out = _execute(eng, 1 << 12, 1 << 26, w["totals"][1])
    _check(o, out, w, lambda g, s: batch[(g, s)], 1 << 26)
    eng.advance_log(ev["last_exec"].clone())
    for st, x in zip(state, w["last_exec"]):
        st["last_exec"] = st["start"] = x
    store, got = _propose(eng, me, [7] * G, rng, n, stride)
    assert len(got) == G
    for g, (s, b) in got.items():
        batch[(g, s)] = b
        state[g]["ent"][s] = (7, 0)
        state[g]["lc"] = s
    s3 = got[3][0]
    lv["data_len"][3][s3 % W] = 0
    state[3]["ent"][s3] = (0, 0)
    eng.last_commit.copy_(torch.tensor([st["lc"] for st in state], dtype=torch.int32, device=dev))
    w = walk(state, 1 << 12, 1 << 26)
    ctx.device_status()
    o, out = _execute(eng, 1 << 12, 1 << 26, w["totals"][1])
    _check(o, out, w, lambda g, s: batch[(g, s)], 1 << 26)
    assert w["null"] and len(w["records"]) == G - 1 and ctx.device_status() & EXEC_NULL
    assert ev["last_exec"].cpu().tolist() == w["last_exec"]
    eng.close()


def _install(fol, G, groups, W, fill=0, skew=0):
    """state through the follower's view: groups[g] = dict(start, lc, le, ent={slot: (data_len, held, batch)}); shards
    from the oracle's encoder in the padded layout (held shard of rank k at shard_addr + k * pitch(L)), each slot's pad
    filled with the byte `fill`, every entry `skew` bytes past a 32-byte boundary of the store -> the store"""
    import torch
    d, p = fol.d, fol.T - fol.d
    dev = "cuda:0"
    blob, addr = bytearray([fill] * skew), {}
    for g, gr in enumerate(groups):
        for s, (dl, held, b) in gr["ent"].items():
            if dl == 0:
                continue
            sh = coded(b, d, p)
            L = -(-dl // d)
            addr[(g, s)] = len(blob)
            for j in range(d + p):
                if held >> j & 1:
                    blob += sh[j].tobytes() + bytes([fill] * (pitch(L) - L))
    store = torch.tensor(np.frombuffer(bytes(blob) + bytes(16), dtype=np.uint8), device=dev)
    base = store.data_ptr()
    sa = np.zeros((G, W), dtype=np.int64)
    held = np.zeros((G, W), dtype=np.uint32)                       # shard 31's bit does not fit an int32
    dlen = np.zeros((G, W), dtype=np.int32)
    term = np.zeros((G, W), dtype=np.int64)
    for g, gr in enumerate(groups):
        for s, (dl, h, _) in gr["ent"].items():
            sa[g][s % W] = base + addr.get((g, s), 0)
            held[g][s % W], dlen[g][s % W], term[g][s % W] = h, dl, 1
    t = lambda a: torch.tensor(a, device=dev)
    fol.shard_addr.copy_(t(sa))
    fol.held.copy_(t(held.view(np.int32)))
    fol.data_len.copy_(t(dlen))
    fol.term.copy_(t(term))
    fol.start_slot.copy_(t(np.array([gr["start"] for gr in groups], dtype=np.int64)))
    fol.log_end.copy_(t(np.array([gr["le"] for gr in groups], dtype=np.int64)))
    fol.last_commit.copy_(t(np.array([gr["lc"] for gr in groups], dtype=np.int64)))
    fol.last_exec.copy_(t(np.array([gr["last_exec"] for gr in groups], dtype=np.int64)))
    return store


@pytest.mark.gpu
@pytest.mark.parametrize("n", [5, 7, 9, 12])
def test_follower_execute_matches_the_restatement(n):
    import torch
    from summerset_b200.engine import Follower
    ctx = _ctx()
    d, T = n // 2 + 1, n
    rng = random.Random(2000 + n)
    W = 16
    # every held pattern with at least d shards at n = 5 (every erasure the code recovers), a seeded sample above
    masks = [m for m in range(1 << T) if popc(m) >= d]
    if n > 5:
        masks = [(1 << T) - 1, (1 << d) - 1] + rng.sample(masks, 40)
    lens = [1, 15, 16, 17, 16 * d - 1, 16 * d + 1, 100, 4095, 64 * 1024]
    G = -(-len(masks) // 6)
    fol = Follower(ctx, G, n, 0, window=W)
    groups, batch, k = [], {}, 0
    for g in range(G):
        start = rng.choice((0, 5, 100, 1000))                    # windows that wrap the ring
        ent = {}
        last = start
        for s in range(max(start, 1), max(start, 1) + 6):
            m = masks[k % len(masks)]
            k += 1
            b = rng.randbytes(rng.choice(lens))
            ent[s] = (len(b), m, b)
            batch[(g, s)] = b
            last = s
        groups.append(dict(start=start, le=last + 1, lc=last - rng.randint(0, 2), last_exec=max(start, 1) - 1, ent=ent))
    # fewer than d shards stops one group's walk; a null entry with d shards stops another's with the status bit
    few, null = groups[0], groups[1]
    s_few, s_null = sorted(few["ent"])[2], sorted(null["ent"])[1]
    few["ent"][s_few] = (few["ent"][s_few][0], (1 << (d - 1)) - 1, few["ent"][s_few][2])
    null["ent"][s_null] = (0, (1 << d) - 1, b"")
    null["lc"] = max(null["lc"], s_null)
    store = _install(fol, G, groups, W)
    model = [dict(start=gr["start"], last_exec=gr["last_exec"], lc=gr["lc"], ent={s: (e[0], e[1]) for s, e in gr["ent"].items()})
             for gr in groups]
    want = walk(model, 1 << 20, 1 << 26, need_d=d)
    assert want["null"] and want["last_exec"][0] == s_few - 1
    ctx.device_status()
    o, out = _execute(fol, 1 << 12, 1 << 26, want["totals"][1])
    _check(o, out, want, lambda g, s: batch[(g, s)], 1 << 26)
    assert fol.last_exec.cpu().tolist() == want["last_exec"]
    st = ctx.device_status()
    assert st & EXEC_NULL and not st & EXEC_FULL
    # a second call executes nothing; advance(upto = last_exec) retires the executed entries
    o, out = _execute(fol, 1 << 12, 1 << 26, 0)
    assert int(o["totals"][0]) == 0
    fol.advance(fol.last_exec.clone())
    torch.cuda.synchronize()
    assert fol.start_slot.cpu().tolist() == [max(gr["start"], min(x, gr["lc"])) for gr, x in zip(groups, want["last_exec"])]
    del store
    fol.close()


def _loop(n, f, resend):
    """A device leader and device followers, population - majority of them silent: 1-shard entries do not commit, the
    leader switches to full copy, and (resend) the host rewinds try_next and packs a full-copy resend that the live
    followers absorb; a heartbeat round follows and both sides execute."""
    import torch
    from summerset_b200.engine import Follower, RaftEngine, append_reply_parse
    ctx = _ctx()
    G, me, term = 32, 0, 1
    maj, P = n // 2 + 1, n - 1
    d = maj
    live = list(range(maj - 1))                                   # peer indices that answer; the rest are silent
    rng = random.Random(3000 + 10 * n + resend)
    dev = "cuda:0"
    t = lambda a, dt: torch.tensor(a, dtype=dt, device=dev)
    eng = RaftEngine(ctx, G, n, fault_tolerance=f, craft=True)
    view = eng.log_view()
    eng.curr_term.fill_(term)
    fols = {q: Follower(ctx, G, n, q + 1) for q in live}
    keep, batch = [], {}
    stride = G * pitch(-(-5000 // d))

    def round_trip(full_copy=False, heartbeat=False):
        out = torch.zeros(1 << 24, dtype=torch.uint8, device=dev)
        o = eng.pack_append(me, out, 1 << 14, heartbeat=heartbeat, full_copy=full_copy, msg_chunk_size=4)
        torch.cuda.synchronize()
        nf = int(o["n_frames"][0])
        fo, fg, fp = o["frame_off"][:nf], o["frame_group"][:nf], o["frame_peer"][:nf]
        replies = []
        for q in live:
            sel = (fp == q).nonzero().flatten()
            if sel.numel() == 0:
                continue
            st, wal = torch.zeros(1 << 24, dtype=torch.uint8, device=dev), torch.zeros(1 << 24, dtype=torch.uint8, device=dev)
            keep.append(st)
            r = fols[q].append(out, fo[sel].contiguous(), fg[sel].contiguous(), torch.zeros_like(fp[sel]), st, wal)
            torch.cuda.synchronize()
            rl, cells = r["reply_len"].cpu().numpy(), r["replies"].cpu().numpy()
            assert (r["verdict"].cpu().numpy().view(np.uint32) == tf.ACCEPTED).all()
            for i, g in enumerate(fg[sel].cpu().tolist()):
                replies.append((g, q, cells[i][:rl[i]].tobytes()))
        buf, offs = bytearray(), []
        for g, q, x in replies:
            offs.append(len(buf))
            buf += x
        tb = t(np.frombuffer(bytes(buf), dtype=np.uint8), torch.uint8)
        rec = append_reply_parse(ctx, tb, t(offs, torch.int64), t([r[0] for r in replies], torch.int32),
                                 t([r[1] for r in replies], torch.uint8), eng.curr_term, G)
        eng.on_append_replies(rec["rec_group"], rec["rec_peer"], rec["rec_end_slot"])
        eng.tick()
        torch.cuda.synchronize()

    for _ in range(3):                                            # 1-shard entries, three rounds
        lens = [rng.choice((1, 15, 16, 17, 300, 5000)) for _ in range(G)]
        store, got = _propose(eng, me, lens, rng, n, stride)
        keep.append(store)
        for g, (s, b) in got.items():
            batch[(g, s)] = b
        round_trip()
    le = eng.log_end.cpu().tolist()
    assert eng.last_commit.cpu().tolist() == [0] * G             # 1 + live acks = majority < majority + f
    eng.set_full_copy(True)
    if resend:                                                    # the resend the reference leaves commented out
        eng.next_slot[live] = 1
        view["try_next"][live] = 1
        round_trip(full_copy=True)
    else:
        eng.tick()
    assert eng.last_commit.cpu().tolist() == [x - 1 for x in le]  # majority acks now commit every entry
    round_trip(heartbeat=True)
    # the leader executes every batch in slot order
    ev = eng.exec_view()
    o, out = _execute(eng, 1 << 12, 1 << 24, 1 << 24)
    nrec = len(batch)
    assert int(o["totals"][0]) == nrec
    recs = sorted(zip(o["rec_group"][:nrec].tolist(), o["rec_slot"][:nrec].tolist(), o["rec_off"][:nrec].tolist(), o["rec_len"][:nrec].tolist()))
    assert [(g, s) for g, s, _, _ in recs] == sorted(batch)
    for g, s, off, dl in recs:
        assert out[off:off + dl].tobytes() == batch[(g, s)]
    assert ev["last_exec"].cpu().tolist() == [x - 1 for x in le]
    for q in live:
        fol = fols[q]
        o, out = _execute(fol, 1 << 12, 1 << 24, 1 << 24)
        if resend:                                                # absorbed data shards: every entry executes, decoded
            assert fol.last_commit.cpu().tolist() == [x - 1 for x in le]
            assert int(o["totals"][0]) == nrec
            for k in range(nrec):
                g, s, off, dl = (int(o[x][k]) for x in ("rec_group", "rec_slot", "rec_off", "rec_len"))
                assert out[off:off + dl].tobytes() == batch[(g, s)]
            assert fol.last_exec.cpu().tolist() == [x - 1 for x in le]
        else:                                                     # the commit walk stops at the first 1-shard entry
            assert fol.last_commit.cpu().tolist() == [0] * G and int(o["totals"][0]) == 0
        fol.advance(fol.last_exec.clone())
    eng.advance_log(ev["last_exec"].clone())
    torch.cuda.synchronize()
    # the leader's log_start stops at last_snap, the silent peers' match (craft/snapshot.rs:142,184)
    assert view["log_start"].cpu().tolist() == [min(x - 1, sn) for x, sn in zip(le, eng.last_snap.cpu().tolist())]
    for q in live:
        assert fols[q].start_slot.cpu().tolist() == ([x - 1 for x in le] if resend else [0] * G)
        fols[q].close()
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n,f", [(5, 1), (7, 2)])
@pytest.mark.parametrize("resend", [True, False])
def test_closed_loop_full_copy_fallback(n, f, resend):
    _loop(n, f, resend)
