"""ss_engine_prepare_absorb: the new RSPaxos / Crossword leader's PrepareReply absorb (handle_msg_prepare_reply,
rspaxos/messages.rs:88-326, crossword/messages.rs:140-400) on the device.

`AbsorbModel` restates the handler in window terms, with ss_prepare_merge_dev's merge and decision rule: the CPU tests
check it on hand-built cases, the GPU tests check the device against it, and the closed fail-over loop runs the whole
sequence step-up -> prepare -> prepare_reply -> prepare_absorb -> pack -> accept -> ingest -> tick -> heartbeat ->
execute and compares the executed payloads with what the old leader committed."""
import numpy as np
import pytest
import torch

from summerset_b200 import _lib
from tests.test_acceptor import ACC, BEYOND, MALFORMED, _buffer, _t

STALE = 0xFFFFFFF1
STORE_FULL, WAL_FULL = 0xFFFFFFF4, 0xFFFFFFF5
IGNORED, DATA_LEN = _lib.SS_PREP_VERDICT_IGNORED, _lib.SS_PREP_VERDICT_DATA_LEN
REPLY = 1
USE, NULL = 1, 2


def decide(mask, acks, d, n, f):
    """ss_prepare_merge_dev's decision (SS_PM_USE / SS_PM_NULL / 0)"""
    if bin(mask).count("1") >= d:
        return USE
    return NULL if acks >= n - f else 0


class AbsorbModel:
    """handle_msg_prepare_reply for one leader over G groups, in window terms.  acc[g] holds what the handler reads of
    the replica's acceptor: base, preparing / settled (Accepting | Committed) ring words, inst_bal and source per ring
    position.  The engine's bookkeeping lives in bk[g]."""

    def __init__(self, n, f, d, T, me):
        self.n, self.f, self.d, self.T, self.me = n, f, d, T, me
        self.maj = n // 2 + 1
        self.bk = {}

    def absorb(self, frames, acc, bps):
        """frames: [(g, peer, rec)], rec a dict (kind, slot, trigger, endprep, ballot, vote_bal, vote_mask, data_len).
        Returns (verdicts per frame, decided [(g, slot, action, mask, data_len)], cells [(g, slot)]) with the decided
        list and the cells ordered by group, then frame."""
        verdict = [None] * len(frames)
        decided, cells = [], []
        self.ends = {}                                  # g -> [decided records, cells, store bytes] this call
        order = sorted(range(len(frames)), key=lambda i: frames[i][0])
        for i in order:
            g, peer, r = frames[i]
            a = acc[g]
            b = bps[g]
            bk = self.bk.get(g)
            if bk is None or bk["ballot"] != b:
                bk = self.bk[g] = dict(ballot=b, acks=0, done=0, pos={})
            base = a["base"]
            e = self.ends.setdefault(g, [0, 0, 0])
            if r["kind"] != REPLY:
                verdict[i] = r["kind"]
                continue
            if r["slot"] < base:
                verdict[i] = STALE
                continue
            tp = r["trigger"] & 63
            if b == 0 or r["ballot"] != b or not (base <= r["trigger"] < base + 64) or \
                    (not (a["filled"] >> tp) & 1 and a["source"][tp] != self.me):
                verdict[i] = IGNORED
                continue
            if r["slot"] >= base + 64:
                verdict[i] = BEYOND
                continue
            w, p = r["slot"] - base, r["slot"] & 63
            live = [((a["prep"] | a["settled"]) >> ((base + x) & 63)) & 1 for x in range(64)]
            end = max([x + 1 for x in range(64) if live[x]], default=0)
            for x in range(end, w + 1):                  # the external fill
                q = (base + x) & 63
                a["prep"] |= 1 << q
                a["filled"] |= 1 << q
                a["inst_bal"][q] = b
                cells.append((g, base + x))
                e[1] += 1
            ib = b if (a["filled"] >> p) & 1 else a["inst_bal"][p]
            if not ((a["prep"] & ~bk["done"]) >> p) & 1 or r["ballot"] < ib:
                verdict[i] = IGNORED
                continue
            st = bk["pos"].setdefault(p, [0, 0, 0])
            v = ACC
            if r["vote_bal"] != 0:
                if r["vote_bal"] > st[0]:
                    st[:] = [r["vote_bal"], r["vote_mask"], r["data_len"]]
                    e[2] += (-(-r["data_len"] // self.d) + 31) // 32 * 32
                elif r["vote_bal"] == st[0]:
                    if r["data_len"] != st[2]:
                        v = DATA_LEN
                    else:
                        st[1] |= r["vote_mask"]
            verdict[i] = v
            if v != ACC or r["slot"] != r["endprep"]:
                continue
            bk["acks"] |= 1 << peer
            cnt = bin(bk["acks"]).count("1")
            if cnt < self.maj:
                continue
            tw = r["trigger"] - base
            for x in range(tw, 64):
                q = (base + x) & 63
                if not ((a["prep"] & ~bk["done"]) >> q) & 1:
                    continue
                mask = bk["pos"].get(q, [0, 0, 0])[1]
                act = decide(mask, cnt, self.d, self.n, self.f)
                if act:
                    e[0] += 1
                    e[2] += 32 if act == NULL else 0
                    bk["done"] |= 1 << q
                    st = bk["pos"].get(q, [0, 0, 0])
                    decided.append((g, base + x, act, st[1] if act == USE else (1 << self.T) - 1, st[2] if act == USE else 1))
        return verdict, decided, cells


def rec(slot, trigger, endprep, ballot, vote_bal=0, vote_mask=0, data_len=0, kind=REPLY):
    return dict(kind=kind, slot=slot, trigger=trigger, endprep=endprep, ballot=ballot, vote_bal=vote_bal, vote_mask=vote_mask,
                data_len=data_len)


def acc_state(base=0, prep=0, settled=0, me=1, src=None):
    return dict(base=base, prep=prep, settled=settled, filled=0, inst_bal=[0] * 64,
                source=[me if src is None else src] * 64)


# ---------------------------------------------------------------------------------------------
# CPU: the restatement on hand-built cases
# ---------------------------------------------------------------------------------------------
def _m(n=5, f=1, d=3):
    return AbsorbModel(n, f, d, n, 1)


def test_model_higher_replaces_equal_merges_empty_clears():
    m = _m()
    a = {0: acc_state(prep=0b1, me=1)}
    a[0]["inst_bal"][0] = 9
    fr = [(0, 1, rec(0, 0, 1, 9, 5, 0b00011, 10)), (0, 2, rec(0, 0, 1, 9, 5, 0b00100, 10)),
          (0, 3, rec(0, 0, 1, 9, 7, 0b01000, 10)), (0, 4, rec(0, 0, 1, 9, 7, 0b10000, 10))]
    v, dec, cells = m.absorb(fr, a, {0: 9})
    assert v == [ACC] * 4 and dec == [] and cells == []
    assert m.bk[0]["pos"][0] == [7, 0b11000, 10]
    v, _, _ = m.absorb([(0, 0, rec(0, 0, 1, 9, 8, 0, 10))], a, {0: 9})   # Some with no shards at a higher ballot
    assert v == [ACC] and m.bk[0]["pos"][0] == [8, 0, 10]
    v, _, _ = m.absorb([(0, 1, rec(0, 0, 1, 9, 8, 0b1, 11))], a, {0: 9})  # same ballot, other data_len: rejected alone
    assert v == [DATA_LEN] and m.bk[0]["pos"][0] == [8, 0, 10]


def test_model_acks_count_only_at_endprep_and_decide():
    m = _m()                                            # n = 5, f = 1, d = 3: majority 3, NULL from 4 acks
    a = {0: acc_state(prep=0b111)}
    for q in range(3):
        a[0]["inst_bal"][q] = 9
    fr = lambda peer: [(0, peer, rec(0, 0, 2, 9, 4, 1 << peer, 12)),
                       (0, peer, rec(1, 0, 2, 9, 4, 1 << peer, 12) if peer == 1 else rec(1, 0, 2, 9)), (0, peer, rec(2, 0, 2, 9))]
    v, dec, _ = m.absorb(fr(1) + fr(2), a, {0: 9})       # two peers: no quorum yet
    assert v == [ACC] * 6 and dec == [] and m.bk[0]["acks"] == 0b110
    v, dec, _ = m.absorb(fr(3)[:2], a, {0: 9})           # not at endprep: no ack
    assert dec == [] and m.bk[0]["acks"] == 0b110
    v, dec, _ = m.absorb(fr(3)[2:], a, {0: 9})           # the third endprep reply: slot 0 has 3 shards, the rest wait
    assert dec == [(0, 0, USE, 0b1110, 12)]
    v, dec, _ = m.absorb([(0, 4, rec(2, 0, 2, 9))], a, {0: 9})   # a fourth ack reaches n - f: the rest go NULL
    assert dec == [(0, 1, NULL, 0b11111, 1), (0, 2, NULL, 0b11111, 1)]


def test_model_use_null_wait_and_later_decision():
    m = _m(n=5, f=1, d=3)
    a = {0: acc_state(prep=0b11)}
    a[0]["inst_bal"][0] = a[0]["inst_bal"][1] = 9
    fr = [(0, p, rec(0, 0, 1, 9, 3, 1 << p, 8)) for p in (0, 1, 2)] + [(0, p, rec(1, 0, 1, 9)) for p in (0, 1, 2)]
    v, dec, _ = m.absorb(fr, a, {0: 9})
    assert v == [ACC] * 6 and dec == [(0, 0, USE, 0b111, 8)]     # slot 0 has d shards; slot 1 waits (3 acks < 4)
    v, dec, _ = m.absorb([(0, 3, rec(1, 0, 1, 9))], a, {0: 9})
    assert dec == [(0, 1, NULL, 0b11111, 1)]
    v, dec, _ = m.absorb([(0, 4, rec(0, 0, 1, 9, 3, 1 << 4, 8))], a, {0: 9})   # decided: ignored
    assert v == [IGNORED] and dec == []


def test_model_filters_wrong_ballot_non_leader_trigger_duplicates():
    m = _m()
    a = {0: acc_state(base=64, prep=0b1, me=1), 1: acc_state(prep=0b1, src=3)}
    a[0]["inst_bal"][0] = 9
    fr = [(0, 1, rec(70, 64, 64, 8)), (0, 1, rec(10, 64, 64, 9)), (1, 1, rec(0, 0, 0, 9)), (0, 1, rec(64, 64, 64, 9)),
          (0, 1, rec(64, 64, 64, 9)), (0, 1, rec(200, 64, 200, 9)), (0, 2, rec(64, 64, 64, 9, kind=MALFORMED))]
    v, dec, cells = m.absorb(fr, a, {0: 9, 1: 9})
    assert v == [IGNORED, STALE, IGNORED, ACC, ACC, BEYOND, MALFORMED]
    assert m.bk[0]["acks"] == 0b10                      # a duplicate counts once


def test_model_external_fill():
    m = _m()
    a = {0: acc_state(base=128, prep=0b11)}
    a[0]["inst_bal"][0] = a[0]["inst_bal"][1] = 9
    v, dec, cells = m.absorb([(0, 2, rec(133, 128, 133, 9, 4, 0b100, 5))], a, {0: 9})
    assert v == [ACC] and cells == [(0, s) for s in range(130, 134)]
    v, dec, cells = m.absorb([(0, 3, rec(131, 128, 133, 9))], a, {0: 9})
    assert v == [ACC] and cells == []                  # inside the filled range: nothing more to fill


def test_model_second_step_up_resets():
    m = _m()
    a = {0: acc_state(prep=0b1)}
    a[0]["inst_bal"][0] = 9
    m.absorb([(0, 1, rec(0, 0, 0, 9, 4, 0b1, 5)), (0, 2, rec(0, 0, 0, 9))], a, {0: 9})
    assert m.bk[0]["acks"] == 0b110
    a[0]["inst_bal"][0] = 10
    v, _, _ = m.absorb([(0, 3, rec(0, 0, 0, 10))], a, {0: 10})
    assert v == [ACC] and m.bk[0]["acks"] == 0b1000 and m.bk[0]["pos"] == {0: [0, 0, 0]}


def test_prepare_absorb_symbols_and_refusals():
    lib = _lib.load()
    assert hasattr(lib, "ss_engine_prepare_absorb")
    args = [None] * 30
    for k in (3, 7, 8, 9, 13, 16, 19, 26):
        args[k] = 0
    assert lib.ss_engine_prepare_absorb(*args) == _lib.SS_ERR_INVALID_ARG
    assert b"null engine or acceptor" in lib.ss_last_error()


# ---------------------------------------------------------------------------------------------
# GPU: the closed fail-over loop, every reply through the device
# ---------------------------------------------------------------------------------------------
def _acc_snapshot(acc, G):
    base = acc.window_base.cpu().numpy().view(np.uint64)
    prep = acc.preparing.cpu().numpy().view(np.uint64)
    settled = (acc.accepting | acc.committed).cpu().numpy().view(np.uint64)
    ib = acc.inst_bal.cpu().numpy().view(np.uint64).reshape(G, 64)
    src = acc.source.cpu().numpy().reshape(G, 64)
    return {g: dict(base=int(base[g]), prep=int(prep[g]), settled=int(settled[g]), filled=0, inst_bal=[int(x) for x in ib[g]],
                    source=[int(x) for x in src[g]]) for g in range(G)}


def _recs(ctx, buf, offs, d, T):
    from summerset_b200.engine import prepare_reply_parse
    pr = {k: v.cpu().numpy() for k, v in prepare_reply_parse(ctx, _t(buf), _t(offs), d, T).items()}
    return [dict(kind=int(pr["kind"][k]) & 0xffffffff, slot=int(pr["slot"][k]), trigger=int(pr["trigger_slot"][k]),
                 endprep=int(pr["endprep_slot"][k]), ballot=int(pr["ballot"][k]), vote_bal=int(pr["vote_bal"][k]),
                 vote_mask=int(pr["vote_mask"][k]) & 0xffffffff, data_len=int(pr["data_len"][k])) for k in range(len(offs))]


@pytest.mark.gpu
@pytest.mark.parametrize("protocol,n,T,d", [("rspaxos", 3, 3, 2), ("rspaxos", 5, 5, 3), ("rspaxos", 7, 7, 4),
                                            ("crossword", 5, 5, 3), ("crossword", 5, 10, 4)])
@pytest.mark.parametrize("split", [1, 3])
def test_closed_failover_loop(ctx, oracle, protocol, n, T, d, split):
    from summerset_b200 import workloads as wl
    from summerset_b200.engine import Acceptor, LeaderEngine
    cw = protocol == "crossword"
    G, rounds, old, leader, f = 16, 3, 0, 1, 1
    rng = np.random.default_rng(n * 1000 + T * 10 + split)
    code = dict(rs_total_shards=T, rs_data_shards=d) if cw else {}
    eng = LeaderEngine(ctx, protocol, G, n, f, 1, **code)
    bal = rng.integers(1, 1 << 20, G).astype(np.uint64)
    eng.set_prepared_ballots(_t(bal))
    if cw:
        policies = np.array([oracle.cw_brr_assignment(n, T, d)], dtype=np.uint32)
        eng.set_policies([list(map(int, q)) for q in policies], True)
    else:
        policies = np.array([[1 << r for r in range(n)]], dtype=np.uint32)
    pol0 = _t(np.zeros(G, np.uint8))
    survivors = list(range(1, n))
    accs = {r: Acceptor(ctx, protocol, G, n, r, d, T) for r in survivors}
    keep, payload, committed_old, orig, chosen = [], {}, set(), {}, set()
    for rnd in range(rounds):
        lens = (wl.cfg4_lengths(G, seed_extra=rnd)[0] // 16 + rng.integers(1, 7, G)).astype(np.uint32)
        data_off = (16 + np.cumsum(lens.astype(np.int64) + 5) - lens.astype(np.int64)).astype(np.uint64)
        arena = rng.integers(0, 256, int(data_off[-1]) + int(lens[-1]) + 64, dtype=np.uint8)
        L = (lens.astype(np.int64) + d - 1) // d
        store = torch.zeros((T, int(((L + 31) // 32 * 32).sum()) + 32), dtype=torch.uint8, device="cuda")
        keep.append(store)
        slot_out, shard_off, _ = eng.propose_ragged(_t(arena), _t(data_off), _t(lens), store, pol0 if cw else None)
        slots = slot_out.cpu().numpy().view(np.uint64)
        so = shard_off.cpu().numpy()
        for g in range(G):
            payload[(g, int(slots[g]))] = arena[int(data_off[g]):int(data_off[g]) + int(lens[g])].tobytes()
            orig[(g, int(slots[g]))] = (store, int(so[g]), int(L[g]))
            if 0 < rnd < rounds - 1:
                chosen.add((g, int(slots[g])))          # every survivor accepted it: a chosen value
        for r in survivors:
            out, off, fl, _ = ctx.frame_accept_pack_ragged(store, shard_off, _t(lens), d, T - d, policies, pol0, r, slot_out, _t(bal),
                                                           with_assignment=cw)
            oh, flh, bh = off.cpu().numpy(), fl.cpu().numpy(), out.cpu().numpy()
            gs = [g for g in range(G) if rnd < rounds - 1 or (g + r) % 4 != 0]          # the last round is lossy
            frames = [bh[int(oh[g]):int(oh[g]) + int(flh[g])].tobytes() for g in gs]
            buf, offs = _buffer(rng, frames)
            astore = torch.empty(sum(len(x) for x in frames) * 2 + 64, dtype=torch.uint8, device="cuda")
            awal = torch.empty(sum(len(x) + 48 for x in frames) + 64, dtype=torch.uint8, device="cuda")
            keep.append(astore)
            res = accs[r].accept(_t(buf), _t(offs), _t(np.array(gs, dtype=np.uint32)), _t(np.zeros(len(gs), np.uint8)), astore, awal)
            assert (res["verdict"].cpu().numpy().view(np.uint32) == ACC).all()
        if rnd == 0:                                    # the old leader committed round 0 and told the survivors
            for g in range(G):
                committed_old.add((g, int(slots[g])))
            for r in survivors:
                accs[r].heartbeat(_t(np.arange(G, dtype=np.uint32)), _t(np.zeros(G, np.uint8)), _t(bal), _t(slots + np.uint64(1)),
                                  _t(np.zeros(G, np.uint64)))
    # the old leader dies: round 1 is accepted everywhere but not known committed, round 2 reached only some survivors
    assert ctx.device_status() == 0
    ldr = accs[leader]
    st = ldr.step_up(torch.empty(G * 64 * 32, dtype=torch.uint8, device="cuda"), G * 64, torch.empty(G * 32, dtype=torch.uint8,
                     device="cuda"), G)
    assert (st["verdict"].cpu().numpy().view(np.uint32) == ACC).all()
    new_bal = st["ballot"].cpu().numpy().view(np.uint64)
    nrec = int(st["totals"][0])
    # the step-up's Prepare frames to the other survivors, then every reply
    st2_frames = []
    trig = st["trigger_slot"].cpu().numpy()
    from tests.test_acceptor_stepup import prep_cell
    for g in range(G):
        c = prep_cell(int(trig[g]), int(new_bal[g]))
        st2_frames.append(c[:8 + int.from_bytes(c[:8], "big")])
    frames, peers, groups = [], [], []
    for r in survivors:
        if r == leader:
            rg, rs = st["rec_group"][:nrec], st["rec_slot"][:nrec]
        else:
            buf, offs = _buffer(rng, st2_frames)
            res = accs[r].prepare(_t(buf), _t(offs), _t(np.arange(G, dtype=np.uint32)), _t(np.full(G, leader, np.uint8)),
                                  torch.empty(G * 64 * 32, dtype=torch.uint8, device="cuda"), G * 64)
            assert (res["verdict"].cpu().numpy().view(np.uint32) == ACC).all()
            k = int(res["totals"][0])
            rg, rs = res["rec_group"][:k], res["rec_slot"][:k]
        out = torch.empty(len(rg) * 4096 + 16, dtype=torch.uint8, device="cuda")
        rr = accs[r].prepare_reply(rg, rs, out)
        ob, ro, rl = out.cpu().numpy(), rr["reply_off"].cpu().numpy(), rr["reply_len"].cpu().numpy()
        for k, g in enumerate(rg.cpu().numpy()):
            frames.append(ob[int(ro[k]):int(ro[k]) + int(rl[k])].tobytes())
            peers.append(r)
            groups.append(int(g))
    # replicas interleaved at random, each one's replies in order (one connection each), a few duplicates after them,
    # odd alignments, split across calls
    queues = {r: [i for i in range(len(frames)) if peers[i] == r] for r in survivors}
    idx = []
    while any(queues.values()):
        r = int(rng.choice([r for r in queues if queues[r]]))
        idx.append(queues[r].pop(0))
    idx += list(rng.integers(0, len(frames), len(frames) // 5))
    frames, peers, groups = [frames[i] for i in idx], [peers[i] for i in idx], [groups[i] for i in idx]
    model = AbsorbModel(n, f, d, T, leader)
    snap = _acc_snapshot(ldr, G)
    bps = {g: int(new_bal[g]) for g in range(G)}
    pstore = torch.full((T, 1 << 16), 0xA5, dtype=torch.uint8, device="cuda")
    used = torch.zeros(1, dtype=torch.int64, device="cuda")
    eng_new = LeaderEngine(ctx, protocol, G, n, f, 1, **code)
    if cw:
        eng_new.set_policies([list(map(int, q)) for q in policies], True)
    dl = dict(slot=[], ballot=[], off=[], len=[], group=[])
    for part in np.array_split(np.arange(len(frames)), split):
        fr = [frames[i] for i in part]
        buf, offs = _buffer(rng, fr)
        recs = _recs(ctx, buf, offs, d, T)
        want_v, want_dec, want_cells = model.absorb([(groups[i], peers[i], recs[k]) for k, i in enumerate(part)], snap, bps)
        res = eng_new.prepare_absorb(ldr, _t(buf), _t(offs), _t(np.array([groups[i] for i in part], np.uint32)),
                                     _t(np.array([peers[i] for i in part], np.uint8)), _t(new_bal), pstore, used,
                                     torch.empty(G * 64 * 32, dtype=torch.uint8, device="cuda"), G * 64, G * 64,
                                     policy=pol0 if cw else None)
        assert ctx.device_status() == 0
        assert [int(x) for x in res["verdict"].cpu().numpy().view(np.uint32)] == want_v
        tot = [int(x) for x in res["totals"].cpu().numpy()]
        assert tot[:2] == [len(want_dec), len(want_cells)]
        k = tot[0]
        got = list(zip(res["dec_group"][:k].cpu().numpy().tolist(), res["dec_slot"][:k].cpu().numpy().tolist(),
                       res["dec_data_len"][:k].cpu().numpy().tolist()))
        assert got == [(g, s, ln) for g, s, _, _, ln in want_dec]
        assert (res["dec_ballot"][:k].cpu().numpy().view(np.uint64) == [bps[g] for g, *_ in want_dec]).all()
        for key in dl:
            dl[key].append(res["dec_" + ("shard_off" if key == "off" else "data_len" if key == "len" else key)][:k])
    assert int(eng_new.bal_prepared.cpu().numpy().view(np.uint64)[0]) in (0, int(new_bal[0]))
    dec = {k: torch.cat(v) for k, v in dl.items()}
    ndec = dec["slot"].numel()
    assert ndec > 0
    # every decided codeword holds the original payload's shards (USE), none is NULL for an instance the old leader committed
    sb = pstore.cpu().numpy()
    ds, dg, do, dn = (dec["slot"].cpu().numpy(), dec["group"].cpu().numpy(), dec["off"].cpu().numpy(), dec["len"].cpu().numpy())
    for k in range(ndec):
        g, s = int(dg[k]), int(ds[k])
        if (g, s) in chosen:                            # USE, with the old leader's codeword byte for byte, parity included
            ost, oo, oL = orig[(g, s)]
            assert int(dn[k]) == len(payload[(g, s)]), (g, s)
            ob = ost.cpu().numpy()
            for j in range(T):
                assert sb[j, int(do[k]):int(do[k]) + oL].tobytes() == ob[j, oo:oo + oL].tobytes(), (g, s, j)
        if (g, s) in committed_old:
            assert int(dn[k]) == len(payload[(g, s)]), (g, s)
        if int(dn[k]) == len(payload.get((g, s), b"")) and int(dn[k]) > 1:
            Lk = -(-int(dn[k]) // d)
            data = b"".join(sb[j, int(do[k]):int(do[k]) + Lk].tobytes() for j in range(d))[:int(dn[k])]
            assert data == payload[(g, s)], (g, s)
        else:
            assert int(dn[k]) == 1 and all(sb[j, int(do[k])] == 0 for j in range(T))
    # pack -> every survivor's accept (the leader's own included) -> parse -> ingest -> tick
    ballots = dec["ballot"]
    pol_dec = _t(np.zeros(ndec, np.uint8))
    for r in survivors:
        out, off, fl, _ = ctx.frame_accept_pack_ragged(pstore, dec["off"], dec["len"], d, T - d, policies, pol_dec, r, dec["slot"],
                                                       ballots, with_assignment=cw)
        oh, flh, bh = off.cpu().numpy(), fl.cpu().numpy(), out.cpu().numpy()
        fr = [bh[int(oh[k]):int(oh[k]) + int(flh[k])].tobytes() for k in range(ndec)]
        buf, offs = _buffer(rng, fr)
        astore = torch.empty(sum(len(x) for x in fr) * 2 + 64, dtype=torch.uint8, device="cuda")
        awal = torch.empty(sum(len(x) + 48 for x in fr) + 64, dtype=torch.uint8, device="cuda")
        keep.append(astore)
        res = accs[r].accept(_t(buf), _t(offs), dec["group"], _t(np.full(ndec, leader, np.uint8)), astore, awal)
        assert (res["verdict"].cpu().numpy().view(np.uint32) == ACC).all()
        reps = res["replies"].cpu().numpy()
        rl = res["reply_len"].cpu().numpy()
        rbuf, roffs = _buffer(rng, [reps[k, :int(rl[k])].tobytes() for k in range(ndec)])
        rg, rs_, rp, rb, rk = ctx.accept_reply_parse(_t(rbuf), _t(roffs), dec["group"], _t(np.full(ndec, r, np.uint8)),
                                                     eng_new.window_base, with_size=cw)
        eng_new.on_accept_replies(rg, rs_, rp, rb)
    assert chosen <= {(int(dg[k]), int(ds[k])) for k in range(ndec)}
    newly = torch.empty(G, dtype=torch.int64, device="cuda")
    eng_new.tick(newly)
    if cw or eng_new.threshold <= len(survivors):       # every survivor acked: each decided instance commits
        cm = eng_new.committed.cpu().numpy().view(np.uint64)
        for k in range(ndec):
            assert (int(cm[int(dg[k])]) >> (int(ds[k]) & 63)) & 1, (int(dg[k]), int(ds[k]))
    # the new leader's own acceptor voted (new ballot, its row)
    vb = ldr.voted_bal.cpu().numpy().view(np.uint64).reshape(G, 64)
    for k in range(ndec):
        assert int(vb[int(dg[k]), int(ds[k]) & 63]) == bps[int(dg[k])]
    # heartbeat with the new commit_bar, then every survivor executes the old leader's committed payloads byte for byte
    cb = (eng_new.window_base + eng_new.commit_bar.to(torch.int64)).cpu().numpy().view(np.uint64)
    for r in survivors:
        accs[r].heartbeat(_t(np.arange(G, dtype=np.uint32)), _t(np.full(G, leader, np.uint8)), _t(new_bal), _t(cb),
                          _t(np.zeros(G, np.uint64)))
        out = torch.empty(1 << 16, dtype=torch.uint8, device="cuda")
        ex = accs[r].execute(out, G * 64)
        ne = int(ex["totals"][0])
        ob, eg, es, eo, el = (out.cpu().numpy(), ex["rec_group"][:ne].cpu().numpy(), ex["rec_slot"][:ne].cpu().numpy(),
                              ex["rec_off"][:ne].cpu().numpy(), ex["rec_len"][:ne].cpu().numpy())
        got = {(int(eg[k]), int(es[k])): ob[int(eo[k]):int(eo[k]) + int(el[k])].tobytes() for k in range(ne)}
        for key in got:
            assert got[key] == payload[key], key
        if cw and r == leader:                          # RSPaxos replicas hold one shard each: they execute after reads
            assert committed_old <= set(got)
    assert ctx.device_status() == 0
    eng.close()
    eng_new.close()
    for a in accs.values():
        a.close()


# ---------------------------------------------------------------------------------------------
# GPU: hand-built windows -- every output against the restatement, the external fill, the cut at every boundary, drains
# ---------------------------------------------------------------------------------------------
N5, D3, F1, ME1, K = 5, 3, 1, 1, 5
BAL = (7 << 8) | (ME1 + 1)


def _setup(ctx, G):
    """the leader's acceptor as ss_acceptor_step_up leaves it: window positions [0, K) Preparing at BAL, source me,
    trigger = base, span K - 1; every base differs, so ring and window orders differ"""
    from summerset_b200.engine import Acceptor, LeaderEngine
    eng = LeaderEngine(ctx, "rspaxos", G, N5, F1, 1)
    acc = Acceptor(ctx, "rspaxos", G, N5, ME1, D3, N5)
    base = np.array([64 * (g % 3) + 13 * g for g in range(G)], np.uint64)
    acc.window_base.copy_(_t(base))
    prep = np.zeros(G, np.uint64)
    ib = np.zeros((G, 64), np.uint64)
    trig = np.zeros((G, 64), np.uint64)
    for g in range(G):
        for w in range(K):
            q = (int(base[g]) + w) & 63
            prep[g] |= np.uint64(1 << q)
            ib[g, q] = BAL
            trig[g, q] = base[g]
    acc.preparing.copy_(_t(prep))
    acc.inst_bal.copy_(_t(ib.reshape(-1)))
    acc.prep_trigger.copy_(_t(trig.reshape(-1)))
    acc.prep_span.fill_(K - 1)
    acc.source.fill_(ME1)
    acc.bal_max_seen.fill_(BAL)
    return eng, acc, base


def _replies(rng, G, base):
    """per group, in replica order (each replica's replies in slot order, as one connection delivers them): the leader's
    own and three peers'; replica 3 has a longer log (endprep = base + K + 1), so its last replies fill two positions.
    Votes: each replica its own shard, at ballots that make some instances replace and some merge; returns (frames,
    groups, peers, payloads)"""
    from tests.test_acceptor_prepare import prep_reply_bytes
    frames, groups, peers, payloads = [], [], [], {}
    for g in range(G):
        b = int(base[g])
        for w in range(K + 2):
            payloads[(g, b + w)] = rng.integers(0, 256, int(rng.integers(1, 90)), dtype=np.uint8).tobytes()
        for r in (ME1, 0, 2, 3):
            endp = b + K + 1 if r == 3 else b + K - 1
            for w in range(endp - b + 1):
                data = payloads[(g, b + w)]
                vb = 0 if (w + r + g) % 5 == 0 else 3 + ((w + g) % 2) * (r % 2)
                voted = None
                if vb:
                    L = -(-len(data) // D3)
                    sh = [None] * N5
                    padded = data.ljust(L * D3, b"\x00")
                    shards = [np.frombuffer(padded[j * L:(j + 1) * L], np.uint8).copy() for j in range(D3)] + \
                             [np.zeros(L, np.uint8) for _ in range(N5 - D3)]
                    from oracle import pyoracle
                    pyoracle.rs_encode(D3, N5 - D3, shards)
                    sh[r] = shards[r].tobytes()
                    voted = (vb, len(data), sh)
                frames.append(prep_reply_bytes(b + w, b, endp, BAL, voted, D3, N5))
                groups.append(g)
                peers.append(r)
    return frames, groups, peers, payloads


def _interleave(rng, G, frames, groups, peers, extra=()):
    """groups interleaved at random, each group's frames kept in order; `extra` (frame, group, peer) appended"""
    queues = {g: [i for i in range(len(frames)) if groups[i] == g] for g in range(G)}
    order = []
    while any(queues.values()):
        g = int(rng.choice([g for g in queues if queues[g]]))
        order.append(queues[g].pop(0))
    fr = [frames[i] for i in order] + [x[0] for x in extra]
    return fr, [groups[i] for i in order] + [x[1] for x in extra], [peers[i] for i in order] + [x[2] for x in extra]


def _run(ctx, eng, acc, rng, fr, gr, pe, store, used, rec_cap=1 << 12, dec_cap=1 << 12):
    buf, offs = _buffer(rng, fr)
    G = eng.G
    res = eng.prepare_absorb(acc, _t(buf), _t(offs), _t(np.array(gr, np.uint32)), _t(np.array(pe, np.uint8)),
                             _t(np.full(G, BAL, np.uint64)), store, used, torch.zeros(1 << 17, dtype=torch.uint8, device="cuda"),
                             rec_cap, dec_cap)
    return res, buf, offs


def _model_frames(ctx, buf, offs, gr, pe, G):
    recs = _recs(ctx, buf, offs, D3, N5)
    out = []
    for k, r in enumerate(recs):
        if gr[k] >= G or pe[k] >= N5:
            r = dict(r, kind=MALFORMED)
        out.append((gr[k] if gr[k] < G else 0, pe[k], r))
    return out


def _check_outputs(res, want_dec, want_cells, wal_base=0):
    from tests.test_acceptor_prepare import wal_cell
    nd, nc = len(want_dec), len(want_cells)
    got = list(zip(res["dec_group"][:nd].cpu().numpy().tolist(), res["dec_slot"][:nd].cpu().numpy().tolist(),
                   res["dec_data_len"][:nd].cpu().numpy().tolist()))
    assert got == [(g, s, ln) for g, s, _, _, ln in want_dec]
    assert (res["dec_ballot"][:nd].cpu().numpy().view(np.uint64) == BAL).all()
    assert (res["dec_policy"][:nd].cpu().numpy() == 0).all()
    assert list(zip(res["rec_group"][:nc].cpu().numpy().tolist(), res["rec_slot"][:nc].cpu().numpy().tolist())) == want_cells
    return [wal_cell(s, BAL) for _, s in want_cells]


@pytest.mark.gpu
def test_absorb_outputs_fill_and_state(ctx, oracle):
    G = 7
    rng = np.random.default_rng(5)
    eng, acc, base = _setup(ctx, G)
    frames, groups, peers, payloads = _replies(rng, G, base)
    extra = [(frames[0], G + 3, ME1), (frames[1], 1 << 20, 0), (frames[2], 0, N5)]   # out-of-range groups, a bad peer
    fr, gr, pe = _interleave(rng, G, frames, groups, peers, extra)
    model = AbsorbModel(N5, F1, D3, N5, ME1)
    snap = _acc_snapshot(acc, G)
    store = torch.full((N5, 1 << 14), 0xA5, dtype=torch.uint8, device="cuda")
    used = torch.full((1,), 40, dtype=torch.int64, device="cuda")     # rounded up to 64 before the first slot
    res, buf, offs = _run(ctx, eng, acc, rng, fr, gr, pe, store, used)
    want_v, want_dec, want_cells = model.absorb(_model_frames(ctx, buf, offs, gr, pe, G), snap, {g: BAL for g in range(G)})
    assert ctx.device_status() == 0
    v = [int(x) for x in res["verdict"].cpu().numpy().view(np.uint32)]
    assert v[-3:] == [MALFORMED] * 3 and v[:-3] == want_v[:-3]
    tot = [int(x) for x in res["totals"].cpu().numpy()]
    assert tot == [len(want_dec), len(want_cells), sum(e[2] for e in model.ends.values())]
    assert int(used.item()) == 64 + tot[2]
    assert len(want_cells) == 2 * G and {a for _, _, a, _, _ in want_dec} == {USE, NULL}
    # the PrepareBal cells, bytes and records
    cells = _check_outputs(res, want_dec, want_cells)
    wal = None
    # the acceptor: filled positions fresh and Preparing at BAL, source me, the trigger's trigger and span
    prep = acc.preparing.cpu().numpy().view(np.uint64)
    ib = acc.inst_bal.cpu().numpy().view(np.uint64).reshape(G, 64)
    src, tr, sp = (acc.source.cpu().numpy().reshape(G, 64), acc.prep_trigger.cpu().numpy().view(np.uint64).reshape(G, 64),
                   acc.prep_span.cpu().numpy().reshape(G, 64))
    vbl, vm, held = (acc.voted_bal.cpu().numpy().reshape(G, 64), acc.voted_mask.cpu().numpy().reshape(G, 64),
                     acc.held.cpu().numpy().reshape(G, 64))
    for g in range(G):
        assert int(prep[g]) == snap[g]["prep"]
        for w in (K, K + 1):
            q = (int(base[g]) + w) & 63
            assert (int(ib[g, q]), int(src[g, q]), int(tr[g, q]), int(sp[g, q])) == (BAL, ME1, int(base[g]), K - 1)
            assert (int(vbl[g, q]), int(vm[g, q]), int(held[g, q])) == (0, 0, 0)
    # the engine: bal_prepared, the rebuilt window, the decided instances Accepting at BAL with empty ack sets
    assert (eng.bal_prepared.cpu().numpy().view(np.uint64) == BAL).all()
    assert (eng.window_base.cpu().numpy().view(np.uint64) == base).all()
    accw = eng.accepting.cpu().numpy().view(np.uint64)
    eib = eng.inst_bal.cpu().numpy().view(np.uint64).reshape(G, 64)
    want_acc = np.zeros(G, np.uint64)
    for g, s, *_ in want_dec:
        want_acc[g] |= np.uint64(1 << (s & 63))
        assert int(eib[g, s & 63]) == BAL
    assert (accw == want_acc).all() and (eng.committed.cpu().numpy() == 0).all() and (eng.planes.cpu().numpy() == 0).all()
    assert (res["pending"].cpu().numpy() == 0).all()
    # store: USE codewords are the payload's full codeword (parity regenerated), NULL ones all zero; canary elsewhere
    sb = store.cpu().numpy()
    mask = np.zeros_like(sb, dtype=bool)
    do = res["dec_shard_off"].cpu().numpy()
    for k, (g, s, act, _, ln) in enumerate(want_dec):
        o = int(do[k])
        L = -(-ln // D3)
        if act == NULL:
            want = [np.zeros(1, np.uint8)] * N5
        else:
            data = payloads[(g, s)]
            assert ln == len(data)
            padded = data.ljust(L * D3, b"\x00")
            want = [np.frombuffer(padded[j * L:(j + 1) * L], np.uint8).copy() for j in range(D3)] + [np.zeros(L, np.uint8)
                                                                                                  for _ in range(N5 - D3)]
            oracle.rs_encode(D3, N5 - D3, want)
        for j in range(N5):
            assert sb[j, o:o + L].tobytes() == want[j].tobytes(), (g, s, j)
            assert not sb[j, o + L:o + (L + 15) // 16 * 16].any()
            mask[j, o:o + (L + 15) // 16 * 16] = True
    assert (sb[~mask] == 0xA5).all()
    del cells, wal
    eng.close()
    acc.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["dec", "cells", "store"])
def test_absorb_cut_every_boundary_then_drain(ctx, kind):
    G = 5
    rng = np.random.default_rng(11)
    eng, acc, base = _setup(ctx, G)
    frames, groups, peers, _ = _replies(rng, G, base)
    fr, gr, pe = _interleave(rng, G, frames, groups, peers)
    store = torch.full((N5, 1 << 14), 0xA5, dtype=torch.uint8, device="cuda")
    used = torch.zeros(1, dtype=torch.int64, device="cuda")
    snap = _acc_snapshot(acc, G)
    full, buf, offs = _run(ctx, eng, acc, rng, fr, gr, pe, store, used)
    model = AbsorbModel(N5, F1, D3, N5, ME1)
    want_v, want_dec, want_cells = model.absorb(_model_frames(ctx, buf, offs, gr, pe, G), snap, {g: BAL for g in range(G)})
    eng.close()
    acc.close()
    col = {"dec": 0, "cells": 1, "store": 2}[kind]
    ends = np.cumsum([model.ends[g][col] for g in range(G)])
    full_off = full["dec_shard_off"][:len(want_dec)].cpu().numpy()
    for b in range(G):
        cap = int(ends[b]) - (32 if kind == "store" else 1)
        if cap < (32 if kind == "store" else 0):
            continue
        first_cut = next(g for g in range(G) if ends[g] > cap)
        eng, acc, _ = _setup(ctx, G)
        used.zero_()
        st = torch.full((N5, 1 << 14 if kind != "store" else max(cap, 32)), 0xA5, dtype=torch.uint8, device="cuda")
        assert ctx.device_status() == 0
        kw = dict(rec_cap=cap if kind == "cells" else 1 << 12, dec_cap=cap if kind == "dec" else 1 << 12)
        res, _, _ = _run(ctx, eng, acc, rng, fr, gr, pe, st, used, **kw)
        assert ctx.device_status() == (16 if kind == "store" else 4)   # STORE_FULL / FRAME_OVERFLOW
        v = [int(x) for x in res["verdict"].cpu().numpy().view(np.uint32)]
        cutv = STORE_FULL if kind == "store" else WAL_FULL
        for i in range(len(fr)):
            assert v[i] == (want_v[i] if gr[i] < first_cut else cutv), (b, i)
        applied = [x for x in want_dec if x[0] < first_cut]
        assert [int(x) for x in res["dec_slot"][:len(applied)].cpu().numpy()] == [x[1] for x in applied]
        # the drain: the cut frames again, with room; the outputs are the uncut call's suffix, at the same store offsets
        idx = [i for i in range(len(fr)) if v[i] == cutv]
        st2 = store if kind != "store" else torch.full((N5, 1 << 14), 0xA5, dtype=torch.uint8, device="cuda")
        if kind == "store":
            st2[:, :st.shape[1]] = st
        res2, _, _ = _run(ctx, eng, acc, rng, [fr[i] for i in idx], [gr[i] for i in idx], [pe[i] for i in idx], st2, used)
        assert [int(x) for x in res2["verdict"].cpu().numpy().view(np.uint32)] == [want_v[i] for i in idx]
        rest = want_dec[len(applied):]
        assert [int(x) for x in res2["dec_slot"][:len(rest)].cpu().numpy()] == [x[1] for x in rest]
        assert (res2["dec_shard_off"][:len(rest)].cpu().numpy() == full_off[len(applied):]).all()
        assert (eng.bal_prepared.cpu().numpy().view(np.uint64) == BAL).all()
        eng.close()
        acc.close()


@pytest.mark.gpu
def test_absorb_refusals(ctx):
    from summerset_b200.engine import Acceptor, LeaderEngine
    lib = ctx.lib
    store = torch.zeros((5, 64), dtype=torch.uint8, device="cuda")
    z = torch.zeros(64, dtype=torch.int64, device="cuda")

    def call(e, a):
        p = z.data_ptr()
        return lib.ss_engine_prepare_absorb(e.h, a.h, p, 8, p, p, p, 0, 1, 0, p, None, store.data_ptr(), 64, p, p, 64, p, p, 1,
                                            p, p, p, p, None, p, 1, p, p, None)
    acc = Acceptor(ctx, "rspaxos", 4, 5, 1, 3, 5)
    for e, why in ((LeaderEngine(ctx, "multipaxos", 4, 5), b"RSPaxos and Crossword"),
                   (LeaderEngine(ctx, "rspaxos", 8, 5, 1, 1), b"must share"),
                   (LeaderEngine(ctx, "rspaxos", 4, 7, 1, 1), b"must share"),
                   (LeaderEngine(ctx, "crossword", 4, 5, 1, 1), b"must share")):
        assert call(e, acc) == _lib.SS_ERR_INVALID_ARG
        assert why in lib.ss_last_error()
        e.close()
    ok = LeaderEngine(ctx, "rspaxos", 4, 5, 1, 1)
    assert call(ok, acc) == 0
    ok.close()
    acc.close()
