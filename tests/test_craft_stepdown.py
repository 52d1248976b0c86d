"""CRaft step-down on the device: ss_engine_craft_step_down, the led bytes and the calls that respect them.

`check_term_batch` restates check_term (craft/leadership.rs:16-75) over a batch of frames for the groups an engine
leads: the first frame of a led group with a higher term deposes it, the rest pass.  GPU tests build a leader's log by
step-up and proposals, depose it with a higher-term RequestVote and compare the follower's ring, words and shards with
the engine's log; they check the capacity cut, the fencing of propose / pack / execute / reconstruct reads, and that the
deposed replica no longer grants its vote to a candidate lacking the entries it committed.
"""
from __future__ import annotations

import ctypes as C
import random

import numpy as np
import pytest

from tests import test_craft_election as te
from tests import test_craft_leader as tl
from tests import test_craft_stepup as ts
from tests import test_follower as tf

vi, framed = tf.vi, tf.framed
NONE = 0xFF
MALFORMED = 0xFFFFFFFF
PASS, RANGE, STORE_FULL, DEPOSED = range(0xFFFFFFF0, 0xFFFFFFF4)
AE, AER, RV, RVR, RC = 0, 1, 2, 3, 4        # PeerMsg variants (craft/mod.rs:207-247)


# ---- the restatement ------------------------------------------------------------------------------------------------
def check_term_batch(frames, led, curr_term):
    """frames: (group, kind, term) with kind 'term' (a decoded term-carrying message), 'pass' (no term) or a verdict
    (malformed / another message).  Returns the verdicts and the term each deposed group took."""
    led, ct = dict(led), dict(curr_term)
    out, deposed = [], {}
    for g, kind, term in frames:
        if kind == "pass":
            out.append(PASS)
        elif kind != "term":
            out.append(kind)
        elif not led[g] or term <= ct[g]:
            out.append(PASS)
        elif term >= 1 << 32:
            out.append(RANGE)
        else:
            led[g], ct[g], deposed[g] = 0, term, term
            out.append(DEPOSED)
    return out, deposed


def test_model_verdict_order_and_first_deposes():
    led, ct = {0: 1, 1: 1, 2: 0}, {0: 5, 1: 5, 2: 5}
    frames = [(0, "term", 5), (0, "term", 4), (0, MALFORMED, 0), (0, "pass", 0), (0, "term", 1 << 32), (0, "term", 7),
              (0, "term", 9), (1, 0x80000001, 0), (2, "term", 9), (1, "term", 6)]
    v, dep = check_term_batch(frames, led, ct)
    assert v == [PASS, PASS, MALFORMED, PASS, RANGE, DEPOSED, PASS, 0x80000001, PASS, DEPOSED]
    assert dep == {0: 7, 1: 6}


def test_model_range_leaves_the_group_led():
    v, dep = check_term_batch([(0, "term", 1 << 40), (0, "term", (1 << 32) - 1)], {0: 1}, {0: 0})
    assert v == [RANGE, DEPOSED] and dep == {0: (1 << 32) - 1}


def test_metadata_cell_at_every_varint_width():
    """DurEntry::Metadata{curr_term, None}: meta_variant 0, the term's varint, voted_for ReplicaId::MAX"""
    want = {7: [7], 300: [251, 0x2C, 0x01], 70000: [252, 0x70, 0x11, 0x01, 0x00], (1 << 32) - 1: [252, 255, 255, 255, 255]}
    for term, tv in want.items():
        body = bytes([0] + tv + [NONE])
        assert te.metadata(term, NONE) == len(body).to_bytes(8, "big") + body


def test_refusals_without_a_device():
    from summerset_b200 import _lib
    lib = _lib.load()
    spec = _lib.StepDownSpec(AE, AER, RV, RVR)

    def refused(rc, why):
        assert rc == _lib.SS_ERR_INVALID_ARG and why in lib.ss_last_error().decode(), (rc, lib.ss_last_error(), why)

    args = lambda s, f=16: (None, f, s, 16, 0, 16, 16, 16, 1, 16, 0, 16, 16, 16, 16, None)
    refused(lib.ss_engine_craft_step_down(*args(C.byref(spec), None)), "null follower")
    refused(lib.ss_engine_craft_step_down(*args(None)), "null spec")
    for bad in (_lib.StepDownSpec(AE, AER, RV, 1 << 16), _lib.StepDownSpec(AE, AE, RV, RVR)):
        refused(lib.ss_engine_craft_step_down(*args(C.byref(bad))), "variants")
    refused(lib.ss_engine_craft_role_view_get(None, None), "null view")
    refused(lib.ss_engine_craft_role_view_get(None, C.byref(_lib.CraftRoleView())), "null engine")


def test_no_device_without_a_context():
    """no follower (nor engine) comes without a device, and step-down refuses what creation left null"""
    import torch
    from summerset_b200 import _lib
    lib = _lib.load()
    h = C.c_void_p()
    cfg = _lib.FollowerConfig(_lib.SS_PROTO_CRAFT, 5, 1, 0, 0, 1, 0, 1)
    rc = lib.ss_follower_create(None, C.byref(cfg), 4, C.byref(h))
    assert rc == (_lib.SS_ERR_INVALID_ARG if torch.cuda.is_available() else _lib.SS_ERR_NO_DEVICE) and not h.value
    spec = _lib.StepDownSpec(AE, AER, RV, RVR)
    assert lib.ss_engine_craft_step_down(None, h, C.byref(spec), 16, 0, 16, 16, 16, 1, 16, 0, 16, 16, 16, 16, None) == _lib.SS_ERR_INVALID_ARG


# ---- GPU ------------------------------------------------------------------------------------------------------------
def _frames(frames, rng):
    import torch
    buf, offs = ts._buf([x for _, _, x in frames], rng)
    return buf, ts._t(offs, torch.int64), ts._t([g for g, _, _ in frames], torch.int32), ts._t([p for _, p, _ in frames], torch.uint8)


class _Rig:
    """n replicas; leader 0 replicates term-1 entries to every follower; replica 1 steps up from its follower in term 2,
    proposes term-2 entries (committed through replicas 3.., so a majority holds them) and absorbs nothing."""

    def __init__(self, n, G=24, W=32, seed=0):
        import torch
        from summerset_b200.engine import Follower, RaftEngine
        self.n, self.G, self.W, self.d, self.me = n, G, W, n // 2 + 1, 1
        self.meta_variant = 0
        self.ctx = ts._ctx()
        self.rng = rng = random.Random(9000 + n + seed)
        self.fols = {r: Follower(self.ctx, G, n, r, window=W) for r in range(1, n)}
        self.stride = G * tl.pitch(-(-3000 // self.d)) * 8
        self.keep, self.batch = [], {}
        old = RaftEngine(self.ctx, G, n, craft=True, window=W)
        old.log_view()
        old.curr_term.fill_(1)
        for _ in range(2):
            te._propose(old, 0, [rng.choice((0, 1, 17, 300, 3000)) for _ in range(G)], self.stride, self.keep, self.batch, rng)
            te._replicate(self.ctx, old, 0, self.fols, self.keep, rng)
        old.close()
        self.eng = eng = RaftEngine(self.ctx, G, n, craft=True, window=W)
        eng.recon_view(), eng.log_view()
        self.planes = torch.zeros((n, self.stride), dtype=torch.uint8, device="cuda:0")
        o = eng.step_up(self.fols[1], ts._t(list(range(G)), torch.int32), ts._t([2] * G, torch.int64), self.planes)
        torch.cuda.synchronize()
        assert (o["verdict"].cpu().numpy() == ts.DONE).all()
        # term-2 entries for the even groups, committed by 1 and the replicas past 2 (replica 2 keeps a term-1 log)
        te._propose(eng, 1, [300 if g % 2 == 0 else 0 for g in range(G)], self.stride, self.keep, self.batch, rng)
        te._replicate(self.ctx, eng, 1, {r: f for r, f in self.fols.items() if r > 2}, self.keep, rng)

    def snapshot(self):
        f, e = self.fols[self.me], self.eng
        return {k: getattr(f, k).clone() for k in ("start_slot", "log_end", "curr_term", "last_commit", "last_snap", "leader",
                                                   "term", "shard_addr", "held", "data_len", "last_exec")} | \
               {"e_" + k: getattr(e, k).clone() for k in ("curr_term", "match", "log_end", "last_commit")}

    def request_vote(self, cand, term):
        """candidate `cand`'s RequestVote for every group, from its own follower's log"""
        f = self.fols[cand]
        le, terms = f.log_end.cpu().tolist(), f.term.cpu().numpy()
        return [(g, cand, te.request_vote(term, le[g] - 1, int(terms[g][(le[g] - 1) % self.W]))) for g in range(self.G)]


def _check_deposed(rig, before, groups, term, peer, store, res, i_of, held_all=False):
    """the follower of replica rig.me against the engine's log for each deposed group (term: one for all, or by group;
    held_all: the engine's held masks are not in use, every entry holds every shard)"""
    import torch
    torch.cuda.synchronize()
    f, e = rig.fols[rig.me], rig.eng
    W, d = rig.W, rig.d
    tt = term if isinstance(term, dict) else {g: term for g in groups}
    held = np.full((rig.G, W), (1 << rig.n) - 1, dtype=np.uint32) if held_all else e.recon_view()["held"].cpu().numpy().view(np.uint32)
    lv = e.log_view()
    ls, eaddr, edl, ps = lv["log_start"].cpu().tolist(), lv["shard_addr"].cpu().numpy(), lv["data_len"].cpu().numpy(), lv["plane_stride"]
    eterms, ele, elc, ect = e.terms.cpu().numpy(), e.log_end.cpu().tolist(), e.last_commit.cpu().tolist(), [x & 0xFFFFFFFF for x in e.curr_term.cpu().tolist()]
    eex, led = e.exec_view()["last_exec"].cpu().tolist(), e.role_view()["led"].cpu().tolist()
    ematch = e.match.cpu().numpy()
    F = {k: getattr(f, k).cpu().numpy() for k in ("start_slot", "log_end", "curr_term", "last_commit", "last_snap", "leader", "term",
                                                  "shard_addr", "held", "data_len", "last_exec")}
    B = {k: v.cpu().numpy() for k, v in before.items()}
    # the engine's planes: the step-up's, and the stores its proposals coded into
    bufs = [(t.data_ptr(), t.numel(), t) for t in [rig.planes] + [k for k in rig.keep if k.dim() == 2]]
    host = {}

    def plane_bytes(addr, n):
        for base, size, t in bufs:
            if base <= addr < base + size:
                if base not in host:
                    host[base] = t.cpu().numpy().reshape(-1)
                return host[base][addr - base:addr - base + n].tobytes()
        raise AssertionError(hex(addr))
    st = store.cpu().numpy()
    sbase = store.data_ptr()
    meta, ml = res["meta"].cpu().numpy(), res["meta_len"].cpu().tolist()
    for g in groups:
        i = i_of[g]
        fs0, le0 = int(B["start_slot"][g]), int(B["log_end"][g])
        ns, le = max(fs0, ls[g]), ele[g]
        assert int(F["start_slot"][g]) == ns and int(F["log_end"][g]) == le
        assert int(F["last_commit"][g]) == max(int(B["last_commit"][g]), elc[g])
        assert int(F["last_exec"][g]) == max(int(B["last_exec"][g]), eex[g])
        assert int(F["curr_term"][g]) == max(int(B["curr_term"][g]), tt[g]) and int(F["leader"][g]) == peer
        raised = tt[g] > int(B["curr_term"][g])
        want_meta = te.metadata(tt[g], NONE, rig.meta_variant)
        assert ml[i] == (len(want_meta) if raised else 0)
        if raised:
            assert meta[i][:ml[i]].tobytes() == want_meta and not meta[i][ml[i]:].any()
        for s in range(ns, le):
            p = s % W
            et, dl, h = int(eterms[g][p]), int(edl[g][p]), int(held[g][p])
            assert int(F["term"][g][p]) == et and int(F["data_len"][g][p]) == dl and int(F["held"][g][p]) & 0xFFFFFFFF == h
            if dl == 0:
                continue
            reused = fs0 <= s < le0 and int(B["term"][g][p]) == et and int(B["data_len"][g][p]) == dl \
                and int(B["held"][g][p]) & 0xFFFFFFFF == h
            addr = int(F["shard_addr"][g][p])
            if reused:
                assert addr == int(B["shard_addr"][g][p])
                continue
            L = -(-dl // d)
            pitch = tl.pitch(L)
            assert sbase <= addr < sbase + st.size
            for r, j in enumerate(j for j in range(rig.n) if (h >> j) & 1):
                dst = addr - sbase + r * pitch
                assert st[dst:dst + L].tobytes() == plane_bytes(int(eaddr[g][p]) + j * ps, L), (g, s, j)
        assert ect[g] == tt[g] and (ematch[:, g] == 0).all() and led[g] == 0


@pytest.mark.gpu
@pytest.mark.parametrize("n", [3, 5, 7, 9, 12])
def test_step_down_matches_the_restatement(n):
    """replica 2's term-3 RequestVote deposes replica 1's engine; frames of other kinds pass or keep their verdicts"""
    import torch
    rig = _Rig(n)
    G = rig.G
    before = rig.snapshot()
    rv = rig.request_vote(2, 3)
    # group order mixed with a Reconstruct frame, a truncated RequestVote with a high term, a stale reply and a
    # second higher-term RequestVote that must pass
    frames, kinds = [], []
    for g in range(G):
        if g % 3 == 0:
            frames.append((g, 2, framed(vi(0) + vi(RC) + vi(0))))
            kinds.append(PASS)
            frames.append((g, 2, framed(vi(0) + vi(RV) + vi(9) + vi(1))))        # last_term missing
            kinds.append(MALFORMED)
        frames.append((g, 2, te.vote_reply(1, True)))
        kinds.append(PASS)
        frames.append(rv[g])
        kinds.append(DEPOSED)
        frames.append((g, 0, te.request_vote(4, 1, 1)))
        kinds.append(PASS)
    buf, fo, fg, fp = _frames(frames, rig.rng)
    store = torch.zeros(1 << 22, dtype=torch.uint8, device="cuda:0")
    res = rig.eng.step_down(rig.fols[1], buf, fo, fg, fp, store)
    torch.cuda.synchronize()
    vd = res["verdict"].cpu().numpy().view(np.uint32).tolist()
    assert vd == kinds
    so = res["store_off"].cpu().tolist()
    i_of = {g: i for i, (g, _, x) in enumerate(frames) if kinds[i] == DEPOSED}
    assert all(so[i] == -1 for i in range(len(frames)) if kinds[i] != DEPOSED)
    offs = [so[i_of[g]] for g in range(G)]
    assert offs == sorted(offs) and int(res["need"][0]) <= store.numel()
    _check_deposed(rig, before, range(G), 3, 2, store, res, i_of)
    f = rig.fols[1]
    # a second call with the same batch: every group is deposed already
    res2 = rig.eng.step_down(rig.fols[1], buf, fo, fg, fp, store)
    torch.cuda.synchronize()
    vd2 = res2["verdict"].cpu().numpy().view(np.uint32).tolist()
    assert vd2 == [PASS if k == DEPOSED else k for k in kinds]
    # vote safety: candidate 2 lacks the committed term-2 entries of the even groups
    v = f.vote(buf, fo[[i_of[g] for g in range(G)]].contiguous(), fg[[i_of[g] for g in range(G)]].contiguous(),
               fp[[i_of[g] for g in range(G)]].contiguous())
    torch.cuda.synchronize()
    vv = v["verdict"].cpu().numpy().view(np.uint32).tolist()
    assert all(vv[g] == te.NO_REPLY for g in range(G) if g % 2 == 0), vv


@pytest.mark.gpu
def test_without_step_down_the_stale_ring_grants():
    """what the vote-safety check covers: replica 1's follower ring predates its leadership and grants the vote"""
    import torch
    rig = _Rig(5)
    buf, fo, fg, fp = _frames(rig.request_vote(2, 3), rig.rng)
    v = rig.fols[1].vote(buf, fo, fg, fp)
    torch.cuda.synchronize()
    vv = v["verdict"].cpu().numpy().view(np.uint32).tolist()
    assert all(vv[g] == te.GRANTED for g in range(rig.G) if g % 2 == 0), vv


@pytest.mark.gpu
def test_capacity_cut_is_a_suffix_and_a_second_call_finishes():
    import torch
    rig = _Rig(5, seed=1)
    G = rig.G
    before = rig.snapshot()
    # each group: the deposing RequestVote, then a higher-term reply from another peer, which must not reach a handler
    # while its group still leads
    frames = []
    for x in rig.request_vote(2, 3):
        frames += [x, (x[0], 3, te.vote_reply(4, False))]
    buf, fo, fg, fp = _frames(frames, rig.rng)
    store = torch.zeros(1 << 22, dtype=torch.uint8, device="cuda:0")
    probe = rig.eng.step_down(rig.fols[1], buf, fo, fg, fp, store, store_capacity=0)
    torch.cuda.synchronize()
    assert probe["verdict"].cpu().numpy().view(np.uint32).tolist() == [STORE_FULL] * (2 * G)  # group 0 copies bytes
    assert (probe["store_off"].cpu().numpy() == -1).all()
    rig.ctx.device_status()
    half = rig.eng.step_down(rig.fols[1], buf, fo, fg, fp, store, store_capacity=int(probe["need"][0]) // 2)
    torch.cuda.synchronize()
    vd = half["verdict"].cpu().numpy().view(np.uint32).tolist()
    cut = vd.index(STORE_FULL) // 2
    assert 0 < cut < G and vd == [DEPOSED, PASS] * cut + [STORE_FULL, STORE_FULL] * (G - cut)
    assert (rig.ctx.device_status() & 16) != 0
    for g in range(cut, G):
        assert int(rig.fols[1].log_end[g]) == int(before["log_end"][g])
        assert int(rig.fols[1].curr_term[g]) == int(before["curr_term"][g])
        assert int(rig.eng.role_view()["led"][g]) == 1 and int(rig.eng.curr_term[g]) == 2
    store2 = torch.zeros(1 << 22, dtype=torch.uint8, device="cuda:0")
    res = rig.eng.step_down(rig.fols[1], buf, fo, fg, fp, store2)
    torch.cuda.synchronize()
    vd2 = res["verdict"].cpu().numpy().view(np.uint32).tolist()
    assert vd2 == [PASS, PASS] * cut + [DEPOSED, PASS] * (G - cut)
    store = store2
    _check_deposed(rig, before, range(cut, G), 3, 2, store, res, {g: 2 * g for g in range(G)})


def _fence_run(rig, fence):
    """execute, propose, pack (entry and heartbeat) and reconstruct reads; with fence, group 0 is first deposed and group
    1 cleared through the role view.  Returns the outputs of every group keyed by group, and the fenced checks' inputs."""
    import torch
    G, e = rig.G, rig.eng
    got = {}
    if fence:
        frames = [x for x in rig.request_vote(2, 3) if x[0] == 0]
        buf, fo, fg, fp = _frames(frames, rig.rng)
        e.step_down(rig.fols[1], buf, fo, fg, fp, torch.zeros(1 << 22, dtype=torch.uint8, device="cuda:0"))
        e.role_view()["led"][1] = 0                                  # cleared by the host
    torch.cuda.synchronize()
    rig.ctx.device_status()
    out = torch.zeros(1 << 22, dtype=torch.uint8, device="cuda:0")
    ex = e.execute(out, 1 << 12)
    torch.cuda.synchronize()
    o_ = out.cpu().numpy()
    for g, s_, off, dl in zip(*(ex[k][:int(ex["totals"][0])].cpu().tolist() for k in ("rec_group", "rec_slot", "rec_off", "rec_len"))):
        got[("exec", g, s_)] = o_[off:off + dl].tobytes()
    arena = ts._t(np.frombuffer(bytes(range(256)) * (300 * G // 256 + 1) + b"\0", dtype=np.uint8), torch.uint8)
    planes = torch.zeros((rig.n, rig.stride), dtype=torch.uint8, device="cuda:0")
    rig.keep.append(planes)
    wal = torch.zeros(1 << 22, dtype=torch.uint8, device="cuda:0")
    o = e.propose(1, arena, ts._t([300 * g for g in range(G)], torch.int64), ts._t([300] * G, torch.int32), planes, wal)
    torch.cuda.synchronize()
    got["status_propose"] = rig.ctx.device_status()
    w_ = wal.cpu().numpy()
    for g, (sl, wo, wl) in enumerate(zip(*(o[k].cpu().tolist() for k in ("slot_out", "wal_off", "wal_len")))):
        got[("propose", g)] = (sl, w_[wo:wo + wl].tobytes() if wo >= 0 else b"", wl)
    for hb in (False, True):
        tn = e.log_view()["try_next"].cpu().numpy().copy()
        pk = e.pack_append(1, out, 1 << 12, heartbeat=hb, msg_chunk_size=4)
        torch.cuda.synchronize()
        o_ = out.cpu().numpy()
        nf = int(pk["n_frames"][0])
        seen = {}
        for f_, ln, g, q in zip(*(pk[k][:nf].cpu().tolist() for k in ("frame_off", "frame_len", "frame_group", "frame_peer"))):
            seen[(q, g)] = seen.get((q, g), 0) + 1
            got[("pack", hb, q, g, seen[(q, g)])] = o_[f_:f_ + ln].tobytes()
        ps, tn2 = pk["pair_status"].cpu().numpy(), e.log_view()["try_next"].cpu().numpy()
        for g in range(G):
            got[("pair", hb, g)] = (ps[:, g].tolist(), tn[:, g].tolist(), tn2[:, g].tolist())
    rr = e.reconstruct_reads(out, 1 << 12, 4)
    torch.cuda.synchronize()
    o_ = out.cpu().numpy()
    nf = int(rr["totals"][0])
    for k, (g, f_, ln) in enumerate(zip(*(rr[x][:nf].cpu().tolist() for x in ("frame_group", "frame_off", "frame_len")))):
        got[("recon", g, k)] = o_[f_:f_ + ln].tobytes()
    got["last_recon"] = e.recon_view()["last_recon"].cpu().tolist()
    return got


@pytest.mark.gpu
def test_fencing_after_step_down_and_through_the_role_view():
    """group 0 deposed, group 1 cleared through the view: propose, pack, execute and reconstruct reads skip both, and
    every other group's outputs are byte-identical to a twin run where nothing was fenced"""
    import torch
    fenced_rig, plain_rig = _Rig(5, seed=2), _Rig(5, seed=2)
    fz, pl = _fence_run(fenced_rig, True), _fence_run(plain_rig, False)
    fenced = {0, 1}
    gof = lambda k: k[2] if k[0] == "exec" else k[1] if k[0] in ("propose", "recon") else k[3] if k[0] == "pack" else k[2]
    keyed = lambda d: {k: v for k, v in d.items() if isinstance(k, tuple) and gof(k) not in fenced}
    # reconstruct frames are numbered across groups: compare them by group
    by_group = lambda d: {k: v for k, v in keyed(d).items() if k[0] != "recon"}
    assert by_group(fz) == by_group(pl)
    assert fz["last_recon"][2:] == pl["last_recon"][2:]
    rec = lambda d: sorted((k[1], v) for k, v in keyed(d).items() if k[0] == "recon")
    assert rec(fz) == rec(pl)
    for g in fenced:
        assert not any(k[0] == "exec" and k[1] == g for k in fz if isinstance(k, tuple))
        assert fz[("propose", g)] == (-1, b"", 0)
        for hb in (False, True):
            st, before, after = fz[("pair", hb, g)]
            assert st == [4] * 4 and before == after
            assert not any(k[0] == "pack" and k[3] == g for k in fz if isinstance(k, tuple))
        assert not any(k[0] == "recon" and k[1] == g for k in fz if isinstance(k, tuple))
    assert fz["status_propose"] & 128 and not pl["status_propose"] & 128
    # a step-up makes the group led again
    e = fenced_rig.eng
    su = e.step_up(fenced_rig.fols[1], ts._t([1], torch.int32), ts._t([5], torch.int64), torch.zeros_like(fenced_rig.planes))
    torch.cuda.synchronize()
    assert int(su["verdict"][0]) == ts.DONE and int(e.role_view()["led"][1]) == 1 and int(e.role_view()["led"][0]) == 0


# ---- every message kind, malformed frames, the held-free path, canaries ----------------------------------------------
class _PlainRig:
    """replica 0 leads every group and was never stepped up (no held masks): two committed rounds of term-1 entries
    replicated to 1.., one more proposed and not sent; replica 0's own follower is empty.  Every follower and the
    replication between them use the given PeerMsg and DurEntry variant indices."""

    def __init__(self, n, G=16, W=32, append_variant=0, reply_variant=1, meta_variant=0, log_variant=1):
        import torch
        from summerset_b200.engine import Follower, RaftEngine
        self.n, self.G, self.W, self.d, self.me = n, G, W, n // 2 + 1, 0
        self.meta_variant = meta_variant
        self.ctx = ts._ctx()
        self.rng = rng = random.Random(7700 + n)
        self.fols = {r: Follower(self.ctx, G, n, r, window=W, append_variant=append_variant, reply_variant=reply_variant,
                                 meta_variant=meta_variant, log_variant=log_variant) for r in range(n)}
        self.stride = G * tl.pitch(-(-3000 // self.d)) * 8
        self.keep, self.batch = [], {}
        self.eng = eng = RaftEngine(self.ctx, G, n, craft=True, window=W)
        eng.log_view()
        eng.curr_term.fill_(1)
        for _ in range(2):
            te._propose(eng, 0, [rng.choice((0, 1, 17, 300, 3000)) for _ in range(G)], self.stride, self.keep, self.batch, rng)
            te._replicate(self.ctx, eng, 0, {r: f for r, f in self.fols.items() if r}, self.keep, rng, None, append_variant,
                          reply_variant)
        te._propose(eng, 0, [rng.choice((1, 300)) for _ in range(G)], self.stride, self.keep, self.batch, rng)
        self.planes = self.keep[0]
        torch.cuda.synchronize()

    def snapshot(self):
        return _Rig.snapshot(self)


def _step_down_raw(eng, fol, buf, fo, fg, fp, store, pad=64, variants=(AE, AER, RV, RVR)):
    """ss_engine_craft_step_down with every output inside canaries (0xA5) that must come back untouched"""
    import torch
    from summerset_b200 import _lib
    n, dev = fo.numel(), "cuda:0"
    mk = lambda cnt, dt: torch.full((cnt + 2 * pad,), 0xA5 if dt == torch.uint8 else -0x5A5A5A5B, dtype=dt, device=dev)
    so, meta, ml, vd, need = mk(n, torch.int64), mk(32 * n, torch.uint8), mk(n, torch.int32), mk(n, torch.int32), mk(1, torch.int64)
    spec = _lib.StepDownSpec(*variants)
    at = lambda t: t.data_ptr() + pad * t.element_size()
    rc = eng.lib.ss_engine_craft_step_down(eng.h, fol.h, C.byref(spec), buf.data_ptr(), buf.numel(), fo.data_ptr(), fg.data_ptr(),
                                           fp.data_ptr(), n, store.data_ptr(), store.numel(), at(so), at(meta), at(ml), at(vd), at(need))
    assert rc == 0
    torch.cuda.synchronize()
    for t in (so, meta, ml, vd, need):
        c = t.cpu().numpy()
        assert (c[:pad] == c[0]).all() and (c[-pad:] == c[0]).all() and c[0] == (0xA5 if t.dtype == torch.uint8 else -0x5A5A5A5B)
    return dict(store_off=so[pad:pad + n], meta=meta[pad:pad + 32 * n].view(n, 32), meta_len=ml[pad:pad + n], verdict=vd[pad:pad + n],
                need=need[pad:pad + 1])


def _malformed(kind, term):
    """a frame of each term-carrying variant that its own call refuses, carrying a high term"""
    return {AE: framed(vi(0) + vi(AE) + vi(term) + vi(0)),                             # prev_term onwards missing
            AER: framed(vi(0) + vi(AER) + vi(term) + vi(1)),                           # conflict tag missing
            RV: framed(vi(0) + vi(RV) + vi(term) + vi(1)),                             # last_term missing
            RVR: framed(vi(0) + vi(RVR) + vi(term) + bytes([2]))}[kind]                # granted not a bool


@pytest.mark.gpu
@pytest.mark.parametrize("n", [3, 5, 9])
def test_every_message_deposes_and_malformed_frames_do_not(n):
    """each group is deposed by one kind of message (AppendEntries, one past the follower's window included,
    AppendEntriesReply, RequestVote, RequestVoteReply) at a term of each varint width, after a malformed frame of each
    variant with a higher term; the engine never had held masks, so every entry is copied with every shard"""
    import torch
    rig = _PlainRig(n)
    G, W, d = rig.G, rig.W, rig.d
    before = rig.snapshot()
    widths = [7, 300, 70000, (1 << 32) - 1]
    big = (1 << 32) - 2
    frames, kinds, tt, i_of = [], [], {}, {}
    for g in range(G):
        kind, t = g % 4, widths[(g // 4) % 4]
        tt[g] = t
        for k in range(4):                                            # malformed frames of the four variants
            frames.append((g, 1 + k % (n - 1), _malformed(k, big)))
            kinds.append(MALFORMED)
        if kind == AE:
            if g % 8 == 0:                                            # past the follower's window: still a term
                L = -(-10 // d)
                ent = tf.entry(t, d, n - d, 10, {0: bytes(L)})
                x = tf.append_entries(t, W + 5, 1, [ent], 0, 0)
            else:
                x = tf.append_entries(t, 0, 0, [], 0, 0)
        elif kind == AER:
            x = tf.reply(t, 1)
        elif kind == RV:
            x = te.request_vote(t, 0, 0)
        else:
            x = te.vote_reply(t, False)
        i_of[g] = len(frames)
        frames.append((g, 1, x))
        kinds.append(DEPOSED)
        frames.append((g, 2, te.vote_reply(big, True)))               # after the deposition: passes
        kinds.append(PASS)
    # a reply from this replica itself is malformed (its sender would become the follower's leader)
    frames.append((0, 0, tf.reply(big, 1)))
    kinds.append(MALFORMED)
    buf, fo, fg, fp = _frames(frames, rig.rng)
    store = torch.zeros(1 << 23, dtype=torch.uint8, device="cuda:0")
    res = _step_down_raw(rig.eng, rig.fols[0], buf, fo, fg, fp, store)
    vd = res["verdict"].cpu().numpy().view(np.uint32).tolist()
    assert vd == kinds
    _check_deposed(rig, before, range(G), tt, 1, store, res, i_of, held_all=True)


# ---- the closed loop: deposed, truncated, elected again ------------------------------------------------------------
def _prop(eng, me, lens, stride, keep, batch, rng, full_copy):
    import torch
    bs = [rng.randbytes(x) for x in lens]
    arena, offs = bytearray(), []
    for b in bs:
        offs.append(len(arena))
        arena += b
    store = torch.zeros((eng.P + 1, stride), dtype=torch.uint8, device="cuda:0")
    keep.append(store)
    o = eng.propose(me, ts._t(np.frombuffer(bytes(arena) + b"\0", dtype=np.uint8), torch.uint8), ts._t(offs, torch.int64),
                    ts._t(lens, torch.int32), store, torch.zeros(1 << 22, dtype=torch.uint8, device="cuda:0"), full_copy=full_copy)
    slots = o["slot_out"].cpu().tolist()
    out = {}
    for g, x in enumerate(lens):
        if x:
            assert slots[g] >= 0
            out[(g, slots[g])] = bs[g]
    batch.update(out)
    return out


def _rep(ctx, eng, me, fols, keep, rng, full_copy, heartbeat_only=False):
    """the leader's entries then a heartbeat to the followers `fols`, replies ingested and ticked; returns each
    follower's trunc_slot per group"""
    import torch
    from summerset_b200.engine import append_reply_parse
    dev = "cuda:0"
    trunc = {}
    for heartbeat in ((True,) if heartbeat_only else (False, True)):
        out = torch.zeros(1 << 22, dtype=torch.uint8, device=dev)
        o = eng.pack_append(me, out, 1 << 12, heartbeat=heartbeat, msg_chunk_size=4, full_copy=full_copy)
        torch.cuda.synchronize()
        nf = int(o["n_frames"][0])
        fo, fg, fp = o["frame_off"][:nf], o["frame_group"][:nf], o["frame_peer"][:nf]
        replies = []
        for r, f in fols.items():
            q = r if r < me else r - 1
            sel = (fp == q).nonzero().flatten()
            if sel.numel() == 0:
                continue
            st = torch.zeros(1 << 22, dtype=torch.uint8, device=dev)
            keep.append(st)
            a = f.append(out, fo[sel].contiguous(), fg[sel].contiguous(), torch.full_like(fp[sel], me), st,
                         torch.zeros(1 << 22, dtype=torch.uint8, device=dev))
            torch.cuda.synchronize()
            assert (a["verdict"].cpu().numpy().view(np.uint32) == tf.ACCEPTED).all()
            for g, ts_ in zip(fg[sel].cpu().tolist(), a["trunc_slot"].cpu().tolist()):
                if ts_ >= 0:
                    trunc.setdefault(r, {})[g] = ts_
            rl, cells = a["reply_len"].cpu().numpy(), a["replies"].cpu().numpy()
            replies += [(g, q, cells[i][:rl[i]].tobytes()) for i, g in enumerate(fg[sel].cpu().tolist())]
        if replies:
            tb, offs = ts._buf([x for _, _, x in replies], rng)
            rec = append_reply_parse(ctx, tb, ts._t(offs, torch.int64), ts._t([x[0] for x in replies], torch.int32),
                                     ts._t([x[1] for x in replies], torch.uint8), eng.curr_term, eng.G)
            eng.on_append_replies(rec["rec_group"], rec["rec_peer"], rec["rec_end_slot"])
            eng.tick()
            torch.cuda.synchronize()
    return trunc


def _exec(x):
    import torch
    out = torch.zeros(1 << 23, dtype=torch.uint8, device="cuda:0")
    ex = x.execute(out, 1 << 14)
    torch.cuda.synchronize()
    o_ = out.cpu().numpy()
    return [((g, s), o_[off:off + dl].tobytes())
            for g, s, off, dl in zip(*(ex[k][:int(ex["totals"][0])].cpu().tolist() for k in ("rec_group", "rec_slot", "rec_off", "rec_len")))]


def _elect(ctx, fols, cand, voters, G, source, rng):
    """cand campaigns for every group, voters answer, cand tallies: returns the tally's outputs"""
    import torch
    c = fols[cand].campaign(ts._t(list(range(G)), torch.int32), ts._t([source] * G, torch.uint8))
    torch.cuda.synchronize()
    assert (c["verdict"].cpu().numpy() == te.DONE).all()
    fl, fr = c["frame_len"].cpu().tolist(), c["frames"].cpu().numpy()
    replies = []
    for v in voters:
        r_ = te._deliver(fols[v], [(g, cand, fr[g][:fl[g]].tobytes()) for g in range(G)], rng, "vote")
        rl, cells = r_["reply_len"].cpu().tolist(), r_["replies"].cpu().numpy()
        assert (r_["verdict"].cpu().numpy().view(np.uint32) == te.GRANTED).all()
        replies += [(g, v, cells[g][:rl[g]].tobytes()) for g in range(G)]
    t = te._deliver(fols[cand], replies, rng, "tally")
    assert int(t["n_won"][0]) == G
    return t


@pytest.mark.gpu
@pytest.mark.parametrize("n", [5, 7])
def test_closed_loop_deposed_leader_rejoins_and_leads_again(n):
    """full copy: replica 0 leads and commits, proposes a suffix that never leaves it; replica 1 is elected, steps up and
    its first heartbeat deposes replica 0, whose next AppendEntries truncates that suffix; every replica executes exactly
    the committed sequence, replica 0 running no batch twice; replica 0 is then elected again, steps up from its
    follower, proposes, and the cluster commits and executes"""
    import torch
    from summerset_b200.engine import Follower, RaftEngine
    ctx = ts._ctx()
    G, W = 12, 64
    d = n // 2 + 1
    rng = random.Random(4400 + n)
    fols = {r: Follower(ctx, G, n, r, window=W) for r in range(n)}
    stride = G * tl.pitch(-(-3000 // d)) * 8
    keep, batch, committed = [], {}, {}
    lens = lambda: [rng.choice((1, 17, 300, 3000)) for _ in range(G)]
    e0 = RaftEngine(ctx, G, n, craft=True, window=W)
    e0.set_full_copy(True)
    e0.log_view()
    e0.curr_term.fill_(1)
    for _ in range(2):
        committed.update(_prop(e0, 0, lens(), stride, keep, batch, rng, True))
        _rep(ctx, e0, 0, {r: f for r, f in fols.items() if r}, keep, rng, True)
    assert e0.last_commit.cpu().tolist() == [x - 1 for x in e0.log_end.cpu().tolist()]
    ran0 = _exec(e0)                                              # replica 0 executes as the leader
    lost = _prop(e0, 0, lens(), stride, keep, batch, rng, True)   # never leaves replica 0: cut off
    # replica 1 is elected in term 2 and steps up from its follower
    t = _elect(ctx, fols, 1, range(2, n), G, 0, rng)
    e1 = RaftEngine(ctx, G, n, craft=True, window=W)
    e1.set_full_copy(True)
    e1.recon_view(), e1.log_view()
    p1 = torch.zeros((n, stride), dtype=torch.uint8, device="cuda:0")
    keep.append(p1)
    su = e1.step_up(fols[1], t["won_group"], t["won_term"], p1)
    torch.cuda.synchronize()
    assert (su["verdict"].cpu().numpy() == ts.DONE).all()
    # its first heartbeat reaches replica 0 and deposes it; the frame is dropped
    out = torch.zeros(1 << 22, dtype=torch.uint8, device="cuda:0")
    hb = e1.pack_append(1, out, 1 << 12, heartbeat=True, full_copy=True)
    torch.cuda.synchronize()
    nf = int(hb["n_frames"][0])
    sel = (hb["frame_peer"][:nf] == 0).nonzero().flatten()
    store0 = torch.zeros(1 << 24, dtype=torch.uint8, device="cuda:0")
    keep.append(store0)
    sd = e0.step_down(fols[0], out, hb["frame_off"][sel].contiguous(), hb["frame_group"][sel].contiguous(),
                      torch.ones(sel.numel(), dtype=torch.uint8, device="cuda:0"), store0)
    torch.cuda.synchronize()
    assert (sd["verdict"].cpu().numpy().view(np.uint32) == DEPOSED).all() and sel.numel() == G
    assert (e0.role_view()["led"].cpu().numpy() == 0).all()
    assert fols[0].log_end.cpu().tolist() == e0.log_end.cpu().tolist() and (fols[0].curr_term.cpu().numpy() == 2).all()
    assert _exec(e0) == []                                        # fenced: replica 0's engine runs nothing now
    # replica 1 proposes in term 2; its next AppendEntries truncates replica 0's suffix
    committed.update(_prop(e1, 1, lens(), stride, keep, batch, rng, True))
    trunc = _rep(ctx, e1, 1, {r: f for r, f in fols.items() if r != 1}, keep, rng, True)
    assert trunc.get(0, {}) == {g: s for (g, s) in lost}, "replica 0's uncommitted suffix is truncated"
    assert e1.last_commit.cpu().tolist() == [x - 1 for x in e1.log_end.cpu().tolist()]
    seq = sorted(committed)
    ran0 += _exec(fols[0])
    assert sorted(k for k, _ in ran0) == seq and len(ran0) == len(seq), "replica 0 runs each committed batch once"
    assert all(v == committed[k] for k, v in ran0)
    ran1 = _exec(e1)
    assert [k for k, _ in ran1] == seq and all(v == committed[k] for k, v in ran1)
    for r in range(2, n):
        ran = _exec(fols[r])
        assert sorted(k for k, _ in ran) == seq and all(v == committed[k] for k, v in ran)
    # replica 0 is elected again in term 3, steps up from its follower, proposes; the cluster commits and executes
    e1.close()
    t = _elect(ctx, fols, 0, range(2, n), G, 1, rng)
    p0 = torch.zeros((n, stride), dtype=torch.uint8, device="cuda:0")
    keep.append(p0)
    su = e0.step_up(fols[0], t["won_group"], t["won_term"], p0)
    torch.cuda.synchronize()
    assert (su["verdict"].cpu().numpy() == ts.DONE).all() and (e0.role_view()["led"].cpu().numpy() == 1).all()
    new = _prop(e0, 0, lens(), stride, keep, batch, rng, True)
    committed.update(new)
    _rep(ctx, e0, 0, {r: f for r, f in fols.items() if r >= 2}, keep, rng, True)
    assert e0.last_commit.cpu().tolist() == [x - 1 for x in e0.log_end.cpu().tolist()]
    ran0 += _exec(e0)
    assert sorted(k for k, _ in ran0) == sorted(committed) and len(ran0) == len(committed)
    assert all(v == committed[k] for k, v in ran0)
    for r in range(2, n):
        assert sorted(k for k, _ in _exec(fols[r])) == sorted(new)
    e0.close()
    for f in fols.values():
        f.close()
