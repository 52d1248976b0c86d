"""Crossword's soft fallback on the leader (ss_engine_fallback_redo): fallback_redo_accepts (crossword/leadership.rs:389-550)
restated in window terms, checked on hand-built windows on the CPU and bit for bit against the device on the GPU -- the
engine's words, the decided list and every plane of every redone codeword against the oracle's encoding -- plus a
closed loop in which a peer dies and the re-sent Accepts commit what the old assignment no longer could."""
import copy

import numpy as np
import pytest
import torch

from summerset_b200 import _lib
from tests.test_acceptor import ACC, MALFORMED, STORE_FULL_V, WAL_FULL_V, _buffer, _t

FRAME_OVERFLOW, STORE_FULL = 4, 16


def popcount(x):
    return bin(int(x)).count("1")


def min_spr_u8(d, majority, f, alive):
    """adaptive.rs:98-106 in u8 arithmetic; where majority + f + 1 - alive would underflow, 0 (the reference panics)"""
    top = (majority + f + 1) & 0xFF
    if alive > top:
        return 0
    return ((top - alive) * (d // majority)) & 0xFF


def pitch(data_len, d):
    L = -(-data_len // d)
    return (L + 31) // 32 * 32


def redo_model(st, entries, peer_alive, policy, policies, balanced, n, d, f, used0, cap, dec_cap):
    """fallback_redo_accepts per listed entry, in list order, on a window state st (numpy arrays: base, acc, cm, bp [G];
    inst_bal, pidx, lens [G, 64] ring-indexed, lens -1 where no codeword location is recorded; planes [n, G]).
    Returns verdicts, the decided list [(g, slot, ballot, off, data_len, policy)], totals, store_used and the state."""
    G = len(st["base"])
    maj = n // 2 + 1
    pop = (1 << n) - 1
    # every entry as if the whole list applied (the counts, ends and totals), then the cut
    shadow = copy.deepcopy(st)
    plans, rec_end, byte_end = [], 0, 0
    for g in entries:
        if g >= G:
            plans.append(None)
            continue
        alive = popcount((0xFFFFFFFF if peer_alive is None else int(peer_alive[g])) & pop)
        spr = min_spr_u8(d, maj, f, alive)
        resp = lambda k: balanced and k < len(policies) and popcount(policies[k][0]) >= spr
        b = int(shadow["base"][g])
        open_ = int(shadow["acc"][g]) & ~int(shadow["cm"][g])
        redo = [w for w in range(64) if (open_ >> ((b + w) & 63)) & 1 and shadow["lens"][g, (b + w) & 63] >= 0
                and not resp(int(shadow["pidx"][g, (b + w) & 63]))]
        nbytes = sum(pitch(int(shadow["lens"][g, (b + w) & 63]), d) for w in redo)
        for w in redo:
            q = (b + w) & 63
            shadow["inst_bal"][g, q] = shadow["bp"][g]
            shadow["planes"][:, g] &= ~np.uint64(1 << q)
            shadow["pidx"][g, q] = policy[g]
        plans.append((g, redo, rec_end, byte_end))
        rec_end += len(redo)
        byte_end += nbytes
    totals = [rec_end, byte_end]
    used = (used0 + 31) // 32 * 32
    out = copy.deepcopy(st)
    verdict, dec, cut, top = [], [], False, 0
    for k, pl in enumerate(plans):
        if pl is None:
            verdict.append(MALFORMED)
            continue
        g, redo, r0, s0 = pl
        b = int(out["base"][g])
        lens = [int(out["lens"][g, (b + w) & 63]) for w in redo]
        r_end, s_end = r0 + len(redo), s0 + sum(pitch(x, d) for x in lens)
        sf = used > cap or s_end > cap - used
        if cut or sf or r_end > dec_cap:
            cut = True
            verdict.append(STORE_FULL_V if sf else WAL_FULL_V)
            continue
        verdict.append(ACC)
        top = max(top, s_end)
        at = used + s0
        for w, ln in zip(redo, lens):
            q = (b + w) & 63
            out["inst_bal"][g, q] = out["bp"][g]
            out["planes"][:, g] &= ~np.uint64(1 << q)
            out["pidx"][g, q] = policy[g]
            dec.append((g, b + w, int(out["bp"][g]), at, ln, int(policy[g])))
            at += pitch(ln, d)
    return dict(verdict=verdict, dec=dec, totals=totals, used=used0 if top == 0 else used + top, state=out)


# ---------------------------------------------------------------------------------------------
# CPU: the restatement on hand-built windows, exact outcomes
# ---------------------------------------------------------------------------------------------
def _brr(n, T, spr):
    """BRR assignment (crossword/mod.rs): replica r holds shards (r * T/n + i) % T, i < spr"""
    dj = T // n
    return [sum(1 << ((r * dj + i) % T) for i in range(spr)) for r in range(n)]


def _state(G, n, open_pos, lens=7, pidx=0, base=0, bp=9, committed=()):
    st = dict(base=np.full(G, base, np.uint64), acc=np.zeros(G, np.uint64), cm=np.zeros(G, np.uint64), bp=np.full(G, bp, np.uint64),
              inst_bal=np.full((G, 64), 3, np.uint64), pidx=np.full((G, 64), pidx, np.uint8), lens=np.full((G, 64), -1, np.int64),
              planes=np.full((n, G), 0xFF, np.uint64))
    for g in range(G):
        for w in open_pos:
            q = (base + w) & 63
            st["acc"][g] |= np.uint64(1 << q)
            st["lens"][g, q] = lens
        for w in committed:
            q = (base + w) & 63
            st["cm"][g] |= np.uint64(1 << q)
            st["acc"][g] &= ~np.uint64(1 << q)
            st["lens"][g, q] = lens
    return st


def _run(st, entries, alive_mask, policy, policies, balanced=True, n=5, d=3, f=2, cap=1 << 20, dec_cap=1 << 10, used0=0):
    G = len(st["base"])
    return redo_model(st, entries, np.full(G, alive_mask, np.uint32), np.full(G, policy, np.uint8), policies, balanced, n, d, f, used0,
                      cap, dec_cap)


def test_model_keep_or_redo_at_each_alive_count():
    # n = 5, RS(3,2), f = 2: min_spr = 6 - alive, so spr 1 is responsive at 5 alive, spr 2 at 4, spr 3 at 3
    pols = [_brr(5, 5, s) for s in (1, 2, 3)]
    for alive, kept in ((5, {0, 1, 2}), (4, {1, 2}), (3, {2})):
        mask = (1 << alive) - 1
        for k in range(3):
            st = _state(1, 5, [0, 2, 5], pidx=k, base=62)
            res = _run(st, [0], mask, 2, pols)
            assert res["verdict"] == [ACC]
            if k in kept:
                assert res["dec"] == [] and res["totals"] == [0, 0] and res["used"] == 0
            else:
                assert [(s, b, ln, p) for _, s, b, _, ln, p in res["dec"]] == [(62, 9, 7, 2), (64, 9, 7, 2), (67, 9, 7, 2)]
                assert [o for *_, o, _, _ in res["dec"]] == [0, 32, 64] and res["used"] == 96
                out = res["state"]
                for w in (0, 2, 5):
                    q = (62 + w) & 63
                    assert out["inst_bal"][0, q] == 9 and out["pidx"][0, q] == 2
                    assert all((int(out["planes"][r, 0]) >> q) & 1 == 0 for r in range(5))
                assert int(out["planes"][0, 0]) == 0xFF & ~(1 << 0) & ~(1 << 3)
                assert (out["acc"] == st["acc"]).all() and (out["cm"] == st["cm"]).all()


def test_model_unbalanced_redoes_every_open_instance():
    pols = [_brr(5, 5, 3)]
    st = _state(1, 5, [1, 3], committed=[2])
    assert len(_run(st, [0], 0b11111, 0, pols, balanced=True)["dec"]) == 0
    res = _run(st, [0], 0b11111, 0, pols, balanced=False)
    assert [s for _, s, *_ in res["dec"]] == [1, 3]                   # the committed slot 2 is not touched


def test_model_underflow_keeps_every_balanced_instance():
    # n = 7, f = 0, majority 4: with six alive, 4 + 0 + 1 - 6 underflows u8; the threshold is 0
    assert min_spr_u8(4, 4, 0, 6) == 0 and min_spr_u8(4, 4, 0, 5) == 0 and min_spr_u8(4, 4, 0, 4) == 1
    pols = [[0] * 7]                                                 # even an empty row is responsive
    st = _state(1, 7, [0, 1])
    assert _run(st, [0], 0b0111111, 0, pols, n=7, d=4, f=0)["dec"] == []
    assert len(_run(st, [0], 0b0111111, 0, pols, balanced=False, n=7, d=4, f=0)["dec"]) == 2


def test_model_out_of_range_policy_is_not_responsive():
    pols = [_brr(5, 5, 3)]
    st = _state(1, 5, [0, 1], pidx=1)
    res = _run(st, [0], 0b11111, 0, pols)
    assert len(res["dec"]) == 2 and res["state"]["pidx"][0, 0] == 0
    # re-assigned to an index past the table: a second entry redoes them again
    res = _run(st, [0, 0], 0b11111, 5, pols)
    assert [s for _, s, *_ in res["dec"]] == [0, 1, 0, 1] and res["verdict"] == [ACC, ACC]


def test_model_duplicates_and_out_of_range_groups():
    pols = [_brr(5, 5, s) for s in (1, 2)]
    st = _state(2, 5, [0, 4], pidx=0)
    res = _run(st, [1, 7, 1, 0], 0b01111, 1, pols)                    # 4 alive: spr 1 redone, spr 2 responsive
    assert res["verdict"] == [ACC, MALFORMED, ACC, ACC]
    assert [(g, s) for g, s, *_ in res["dec"]] == [(1, 0), (1, 4), (0, 0), (0, 4)]
    assert res["totals"] == [4, 128]


def test_model_cut_is_per_entry_and_a_prefix():
    pols = [_brr(5, 5, 1)]
    st = _state(3, 5, [0, 1])
    res = _run(st, [0, 1, 2], 0b1111, 0, pols, cap=128)
    assert res["verdict"] == [ACC, ACC, STORE_FULL_V] and len(res["dec"]) == 4
    assert res["state"]["pidx"][2, 0] == 0 and res["state"]["pidx"][1, 0] == 0
    res = _run(st, [0, 1, 2], 0b1111, 0, pols, dec_cap=3)
    assert res["verdict"] == [ACC, WAL_FULL_V, WAL_FULL_V] and len(res["dec"]) == 2 and res["totals"] == [6, 192]


def test_fallback_symbols_and_refusals():
    lib = _lib.load()
    args = [None] * 17
    for k in (2, 6, 14):
        args[k] = 0
    assert lib.ss_engine_fallback_redo(*args) == _lib.SS_ERR_INVALID_ARG
    assert b"null engine" in lib.ss_last_error()


# ---------------------------------------------------------------------------------------------
# GPU: windows built by every proposal path, checked bit for bit
# ---------------------------------------------------------------------------------------------
def _codeword(oracle, data, d, T):
    """the full T-shard codeword of a request batch: data shards, then parity from the oracle"""
    L = -(-len(data) // d)
    padded = data.ljust(L * d, b"\x00")
    shards = [np.frombuffer(padded[j * L:(j + 1) * L], np.uint8).copy() for j in range(d)] + [np.zeros(L, np.uint8) for _ in range(T - d)]
    if T > d:
        oracle.rs_encode(d, T - d, shards)
    return shards


def _policies(oracle, n, T, d):
    sprs = sorted({1, max(1, T // n), d, min(T, d + 1)})
    return sprs, [[int(x) for x in oracle.cw_brr_assignment(n, T, s)] for s in sprs]


class Window:
    """one Crossword engine whose windows hold instances of every proposal path; payload[(g, ring position)] is the
    request batch the position's current instance carries"""

    def __init__(self, ctx, oracle, n, T, d, f, G, seed, balanced=True, with_absorb=False):
        from summerset_b200.engine import LeaderEngine
        self.ctx, self.oracle, self.n, self.T, self.d, self.f, self.G = ctx, oracle, n, T, d, f, G
        self.rng = rng = np.random.default_rng(seed)
        self.DL = 40 + 7 * n
        self.eng = eng = LeaderEngine(ctx, "crossword", G, n, f, self.DL, keep_slots=4, rs_total_shards=T, rs_data_shards=d)
        self.sprs, self.pols = _policies(oracle, n, T, d)
        self.balanced = balanced
        eng.set_policies(self.pols, balanced)
        self.keep = []
        self.payload = {}
        base = np.array([[0, 60, 64 * 3 + 61, 5, 63, 64 + 32][g % 6] + 64 * (g // 6) for g in range(G)], np.uint64)
        eng.window_base.copy_(_t(base))
        eng.set_prepared_ballots(_t(rng.integers(1, 1 << 40, G).astype(np.uint64)))
        self.base = base
        K = len(self.pols)
        pol = lambda: _t(rng.integers(0, K + 1, G).astype(np.uint8))     # index K: past the table
        self.ragged(pol())                                               # window position 0
        self.uniform(1, 1, pol())                                        # 1
        self.next(2, pol())                                              # 2
        self.ragged(pol())                                               # 3
        self.uniform(0, 0, pol())                                        # 0 again: a ragged position reused
        self.ragged(pol())                                               # 4
        self.next(3, pol())                                              # 5

    def ragged(self, policy):
        G, d, rng = self.G, self.d, self.rng
        lens = rng.integers(1, 300, G).astype(np.uint32)
        data_off = (np.cumsum(lens.astype(np.int64) + 3) - lens.astype(np.int64)).astype(np.uint64)
        arena = rng.integers(0, 256, int(data_off[-1]) + int(lens[-1]) + 16, dtype=np.uint8)
        L = (lens.astype(np.int64) + d - 1) // d
        store = torch.zeros((self.T, int(((L + 31) // 32 * 32).sum()) + 64), dtype=torch.uint8, device="cuda")
        self.keep.append(store)
        slot_out, shard_off, _ = self.eng.propose_ragged(_t(arena), _t(data_off), _t(lens), store, policy)
        for g, s in enumerate(slot_out.cpu().numpy().view(np.uint64)):
            self.payload[(g, int(s) & 63)] = arena[int(data_off[g]):int(data_off[g]) + int(lens[g])].tobytes()

    def uniform(self, slot, store, policy):
        pay = self.rng.integers(0, 256, (self.G, self.DL), dtype=np.uint8)
        self.eng.propose(slot, _t(pay), policy)
        for g in range(self.G):
            self.payload[(g, (int(self.base[g]) + slot) & 63)] = pay[g].tobytes()
        assert slot % 4 == store

    def next(self, store, policy):
        pay = self.rng.integers(0, 256, (self.G, self.DL), dtype=np.uint8)
        slot_out, _ = self.eng.propose_next(store, _t(pay), policy)
        for g, s in enumerate(slot_out.cpu().numpy().view(np.uint64)):
            self.payload[(g, int(s) & 63)] = pay[g].tobytes()

    def settle(self):
        """a random part of each window committed, random acks on the rest, some groups at a newer prepared ballot"""
        eng, rng, G, n = self.eng, self.rng, self.G, self.n
        acc = eng.accepting.cpu().numpy().view(np.uint64)
        full = np.array([int(acc[g]) & int(rng.integers(0, 1 << 62)) for g in range(G)], np.uint64)
        pl = eng.planes.cpu().numpy().view(np.uint64).copy()
        for r in range(n):
            pl[r] |= full
        eng.planes.copy_(_t(pl))
        eng.tick()
        pl = eng.planes.cpu().numpy().view(np.uint64).copy()
        pl |= rng.integers(0, 1 << 62, pl.shape).astype(np.uint64)
        eng.planes.copy_(_t(pl))
        bp = eng.bal_prepared.cpu().numpy().view(np.uint64).copy()
        bp[::3] += np.uint64(256)
        eng.set_prepared_ballots(_t(bp))

    def state(self):
        e, G = self.eng, self.G
        lens = np.full((G, 64), -1, np.int64)
        for (g, q), data in self.payload.items():
            lens[g, q] = len(data)
        return dict(base=e.window_base.cpu().numpy().view(np.uint64).copy(), acc=e.accepting.cpu().numpy().view(np.uint64).copy(),
                    cm=e.committed.cpu().numpy().view(np.uint64).copy(), bp=e.bal_prepared.cpu().numpy().view(np.uint64).copy(),
                    inst_bal=e.inst_bal.cpu().numpy().view(np.uint64).reshape(G, 64).copy(),
                    pidx=e.policy_idx.cpu().numpy().reshape(G, 64).copy(), lens=lens,
                    planes=e.planes.cpu().numpy().view(np.uint64).copy())

    def inputs(self, n_entries):
        rng, G, n = self.rng, self.G, self.n
        maj = n // 2 + 1
        alive = np.array([(int(rng.choice([m for m in range(1 << n) if popcount(m) >= maj])) | (int(rng.integers(0, 4)) << n))
                          for _ in range(G)], np.uint32)
        policy = rng.integers(0, len(self.pols) + 1, G).astype(np.uint8)
        entries = [int(x) for x in rng.permutation(G)][:n_entries] + [int(rng.integers(0, G)), G + 2, int(rng.integers(0, G))]
        return entries, alive, policy

    def redo(self, entries, alive, policy, store, used, dec_cap):
        return self.eng.fallback_redo(_t(np.array(entries, np.uint32)), _t(policy), store, used, dec_cap, _t(alive))

    def check(self, before, want, res, store, canary=0xA5, check_store=True):
        e, G, d, T = self.eng, self.G, self.d, self.T
        assert [int(x) for x in res["verdict"].cpu().numpy().view(np.uint32)] == want["verdict"]
        assert [int(x) for x in res["totals"].cpu().numpy()] == want["totals"]
        k = len(want["dec"])
        got = list(zip(res["dec_group"][:k].cpu().numpy().tolist(), res["dec_slot"][:k].cpu().numpy().view(np.uint64).tolist(),
                       res["dec_ballot"][:k].cpu().numpy().view(np.uint64).tolist(), res["dec_shard_off"][:k].cpu().numpy().tolist(),
                       res["dec_data_len"][:k].cpu().numpy().tolist(), res["dec_policy"][:k].cpu().numpy().tolist()))
        assert got == want["dec"]
        now, w = self.state(), want["state"]
        for key in ("inst_bal", "pidx", "planes"):
            assert (now[key] == w[key]).all(), key
        for key in ("acc", "cm", "base", "bp"):
            assert (now[key] == before[key]).all(), key
        if check_store:
            sb = store.cpu().numpy()
            mask = np.zeros(sb.shape, bool)
            for g, s, _, off, ln, _ in want["dec"]:
                L = -(-ln // d)
                cw = _codeword(self.oracle, self.payload[(g, s & 63)], d, T)
                for j in range(T):
                    assert sb[j, off:off + L].tobytes() == cw[j].tobytes(), (g, s, j)
                    assert not sb[j, off + L:off + (L + 15) // 16 * 16].any()
                    mask[j, off:off + (L + 15) // 16 * 16] = True
            assert (sb[~mask] == canary).all()

    def close(self):
        self.eng.close()


# every Crossword population and code the engine takes with T <= 2n and T <= 12, and two wider codes
CODES = [(1, 2, 1), (2, 4, 2), (3, 3, 2), (3, 6, 2), (3, 6, 4), (4, 4, 3), (4, 8, 3), (4, 8, 6), (5, 5, 3), (5, 10, 3), (5, 10, 6),
         (5, 10, 9), (6, 6, 4), (6, 12, 4), (6, 12, 8), (7, 7, 4), (8, 8, 5), (9, 9, 5), (10, 10, 6), (11, 11, 6), (12, 12, 7),
         (4, 16, 9), (8, 16, 10)]


@pytest.mark.gpu
@pytest.mark.parametrize("n,T,d", CODES)
@pytest.mark.parametrize("balanced", [True, False])
def test_fallback_matches_restatement(ctx, oracle, n, T, d, balanced):
    f = (n - (n // 2 + 1))
    w = Window(ctx, oracle, n, T, d, f, 12, seed=n * 97 + T * 7 + d + balanced, balanced=balanced)
    w.settle()
    entries, alive, policy = w.inputs(9)
    before = w.state()
    store = torch.full((T, 1 << 16), 0xA5, dtype=torch.uint8, device="cuda")
    used = torch.full((1,), 40, dtype=torch.int64, device="cuda")
    want = redo_model(before, entries, alive, policy, w.pols, balanced, n, d, f, 40, 1 << 16, 1 << 12)
    cb = w.eng.commit_bar.clone()
    res = w.redo(entries, alive, policy, store, used, 1 << 12)
    assert ctx.device_status() == 0
    w.check(before, want, res, store)
    assert int(used.item()) == want["used"]
    assert torch.equal(cb, w.eng.commit_bar)
    if balanced:
        assert len(want["dec"]) > 0
    w.close()


@pytest.mark.gpu
def test_fallback_none_alive_mask_and_empty_list(ctx, oracle):
    w = Window(ctx, oracle, 5, 5, 3, 2, 6, seed=3)
    before = w.state()
    store = torch.full((5, 1 << 14), 0xA5, dtype=torch.uint8, device="cuda")
    used = torch.zeros(1, dtype=torch.int64, device="cuda")
    policy = np.zeros(6, np.uint8)
    res = w.eng.fallback_redo(_t(np.zeros(0, np.uint32)), _t(policy), store, used, 16)
    assert [int(x) for x in res["totals"].cpu().numpy()] == [0, 0] and int(used.item()) == 0
    entries = list(range(6))
    want = redo_model(before, entries, None, policy, w.pols, True, 5, 3, 2, 0, 1 << 14, 1 << 10)
    res = w.eng.fallback_redo(_t(np.array(entries, np.uint32)), _t(policy), store, used, 1 << 10)
    w.check(before, want, res, store)
    w.close()


def _absorb_window(ctx, oracle, G, seed):
    """n = 5, RS(3,2), f = 1: the new leader's engine proposes ragged batches, then ss_engine_prepare_absorb rebuilds its
    window from the acceptor (decided instances on positions the proposals used), then every proposal path again"""
    from summerset_b200.engine import Acceptor
    from tests.test_engine_prepare import USE, AbsorbModel, BAL, K, ME1, _acc_snapshot, _interleave, _model_frames, _replies
    w = Window.__new__(Window)
    w.ctx, w.oracle, w.n, w.T, w.d, w.f, w.G = ctx, oracle, 5, 5, 3, 1, G
    w.rng = rng = np.random.default_rng(seed)
    w.DL, w.keep, w.payload, w.balanced = 50, [], {}, True
    from summerset_b200.engine import LeaderEngine
    w.eng = LeaderEngine(ctx, "crossword", G, 5, 1, w.DL, keep_slots=4, rs_total_shards=5, rs_data_shards=3)
    w.sprs, w.pols = _policies(oracle, 5, 5, 3)
    w.eng.set_policies(w.pols, True)
    w.eng.set_prepared_ballots(_t(np.full(G, 5, np.uint64)))
    w.base = np.zeros(G, np.uint64)
    pol0 = _t(np.zeros(G, np.uint8))
    for _ in range(3):
        w.ragged(pol0)                                                   # ring positions 0..2, replaced below
    acc = Acceptor(ctx, "crossword", G, 5, ME1, 3, 5)
    base = np.array([64 * (g % 3) + 13 * g for g in range(G)], np.uint64)
    acc.window_base.copy_(_t(base))
    prep = np.zeros(G, np.uint64)
    ib = np.zeros((G, 64), np.uint64)
    trig = np.zeros((G, 64), np.uint64)
    for g in range(G):
        for x in range(K):
            q = (int(base[g]) + x) & 63
            prep[g] |= np.uint64(1 << q)
            ib[g, q] = BAL
            trig[g, q] = base[g]
    acc.preparing.copy_(_t(prep))
    acc.inst_bal.copy_(_t(ib.reshape(-1)))
    acc.prep_trigger.copy_(_t(trig.reshape(-1)))
    acc.prep_span.fill_(K - 1)
    acc.source.fill_(ME1)
    acc.bal_max_seen.fill_(BAL)
    frames, groups, peers, payloads = _replies(rng, G, base)
    fr, gr, pe = _interleave(rng, G, frames, groups, peers)
    buf, offs = _buffer(rng, fr)
    snap = _acc_snapshot(acc, G)
    pstore = torch.zeros((5, 1 << 15), dtype=torch.uint8, device="cuda")
    w.keep.append(pstore)
    used = torch.zeros(1, dtype=torch.int64, device="cuda")
    policy = _t(rng.integers(0, len(w.pols), G).astype(np.uint8))
    res = w.eng.prepare_absorb(acc, _t(buf), _t(offs), _t(np.array(gr, np.uint32)), _t(np.array(pe, np.uint8)),
                               _t(np.full(G, BAL, np.uint64)), pstore, used, torch.zeros(1 << 17, dtype=torch.uint8, device="cuda"),
                               1 << 12, 1 << 12, policy=policy)
    want_v, want_dec, _ = AbsorbModel(5, 1, 3, 5, ME1).absorb(_model_frames(ctx, buf, offs, gr, pe, G), snap, {g: BAL for g in range(G)})
    assert [int(x) for x in res["verdict"].cpu().numpy().view(np.uint32)] == want_v
    for g, s, act, _, ln in want_dec:                                   # a NULL decision: the zero codeword of data_len 1
        w.payload[(g, s & 63)] = payloads[(g, s)] if act == USE else b"\x00"
        assert act == USE or ln == 1
    w.base = base
    K2 = len(w.pols)
    pol = lambda: _t(rng.integers(0, K2 + 1, G).astype(np.uint8))
    w.uniform(1, 1, pol())                                               # an absorb-decided position reused
    w.ragged(pol())
    w.next(2, pol())
    w.acc = acc
    return w, want_dec


@pytest.mark.gpu
def test_fallback_after_absorb_and_every_proposal_path(ctx, oracle):
    from tests.test_engine_prepare import NULL, USE
    G = 7
    w, want_dec = _absorb_window(ctx, oracle, G, seed=21)
    assert {a for _, _, a, _, _ in want_dec} == {USE, NULL}
    w.settle()
    entries, alive, policy = w.inputs(G)
    before = w.state()
    store = torch.full((5, 1 << 15), 0xA5, dtype=torch.uint8, device="cuda")
    used = torch.full((1,), 7, dtype=torch.int64, device="cuda")
    want = redo_model(before, entries, alive, policy, w.pols, True, 5, 3, 1, 7, 1 << 15, 1 << 12)
    res = w.redo(entries, alive, policy, store, used, 1 << 12)
    assert ctx.device_status() == 0
    w.check(before, want, res, store)
    assert int(used.item()) == want["used"]
    w.acc.close()
    w.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["store", "list"])
def test_fallback_cut_every_boundary_then_drain(ctx, oracle, kind):
    n, T, d, f, G = 5, 5, 3, 2, 6
    probe = Window(ctx, oracle, n, T, d, f, G, seed=77)
    probe.settle()
    entries, alive, policy = probe.inputs(G)
    before = probe.state()
    full = redo_model(before, entries, alive, policy, probe.pols, True, n, d, f, 0, 1 << 16, 1 << 12)
    probe.close()
    # every entry's end, as if the whole list applied
    ends, rec, byt = [], 0, 0
    st = before
    for g in entries:
        one = redo_model(st, [g], alive, policy, probe.pols, True, n, d, f, 0, 1 << 16, 1 << 12)
        st = one["state"]
        rec += one["totals"][0]
        byt += one["totals"][1]
        ends.append(byt if kind == "store" else rec)
    caps = sorted({c for e in ends if e > 0 for c in (e, e - (32 if kind == "store" else 1)) if c > 0})
    assert len(caps) >= 4
    for cap in caps:
        w = Window(ctx, oracle, n, T, d, f, G, seed=77)
        w.settle()
        w.inputs(G)                                                      # the same draws as the probe
        plane = cap if kind == "store" else 1 << 16
        dec_cap = 1 << 12 if kind == "store" else cap
        store = torch.full((T, max(plane, 32)), 0xA5, dtype=torch.uint8, device="cuda")
        used = torch.zeros(1, dtype=torch.int64, device="cuda")
        want = redo_model(before, entries, alive, policy, w.pols, True, n, d, f, 0, plane, dec_cap)
        res = w.redo(entries, alive, policy, store, used, dec_cap)
        w.check(before, want, res, store)
        cut = [k for k, v in enumerate(want["verdict"]) if v in (STORE_FULL_V, WAL_FULL_V)]
        assert not cut or cut == [x for x in range(cut[0], len(entries)) if entries[x] < G]     # a prefix applies
        if cut:
            assert ctx.device_status() & (STORE_FULL if kind == "store" else FRAME_OVERFLOW)
        # the drain: the cut entries again, into a fresh store
        rest = [entries[k] for k in cut]
        mid = w.state()
        store2 = torch.full((T, 1 << 16), 0xA5, dtype=torch.uint8, device="cuda")
        used2 = torch.zeros(1, dtype=torch.int64, device="cuda")
        want2 = redo_model(mid, rest, alive, policy, w.pols, True, n, d, f, 0, 1 << 16, 1 << 12)
        res2 = w.redo(rest, alive, policy, store2, used2, 1 << 12)
        w.check(mid, want2, res2, store2)
        assert all(v in (ACC, MALFORMED) for v in want2["verdict"])
        fin = w.state()
        for key in ("inst_bal", "pidx", "planes"):
            assert (fin[key] == full["state"][key]).all(), key
        assert [x[:3] + x[4:] for x in want["dec"] + want2["dec"]] == [x[:3] + x[4:] for x in full["dec"]]
        w.close()


@pytest.mark.gpu
def test_fallback_refusals(ctx, oracle):
    from summerset_b200.engine import LeaderEngine
    lib = ctx.lib
    G = 4
    store = torch.zeros((5, 4096), dtype=torch.uint8, device="cuda")
    used = torch.zeros(1, dtype=torch.int64, device="cuda")
    groups, policy = _t(np.arange(G, dtype=np.uint32)), _t(np.zeros(G, np.uint8))
    rs = LeaderEngine(ctx, "rspaxos", G, 5, 1, 64)
    with pytest.raises(Exception, match="Crossword engines only"):
        rs.fallback_redo(groups, policy, store, used, 16)
    rs.close()
    cw = LeaderEngine(ctx, "crossword", G, 5, 1, 64, rs_total_shards=5, rs_data_shards=3)
    with pytest.raises(Exception, match="set_policies"):
        cw.fallback_redo(groups, policy, store, used, 16)
    cw.set_policies([list(map(int, oracle.cw_brr_assignment(5, 5, 3)))], True)
    out = [torch.empty(16, dtype=dt, device="cuda") for dt in (torch.int64, torch.int64, torch.int64, torch.int32, torch.uint8, torch.int32)]
    verdict = torch.empty(G, dtype=torch.int32, device="cuda")
    p = lambda x: x.data_ptr()

    def call(groups_p=p(groups), policy_p=p(policy), shards=p(store), stride=4096, used_p=p(used), dec=tuple(p(x) for x in out),
             verdict_p=p(verdict)):
        return lib.ss_engine_fallback_redo(cw.h, groups_p, G, None, policy_p, shards, stride, used_p, *dec, 16, verdict_p, None)

    assert call() == 0
    for kw in (dict(groups_p=None), dict(policy_p=None), dict(shards=None), dict(used_p=None), dict(verdict_p=None),
               dict(dec=(None,) + tuple(p(x) for x in out[1:]))):
        assert call(**kw) == _lib.SS_ERR_INVALID_ARG and b"null buffer" in lib.ss_last_error()
    for stride in (0, 4008, 1 << 36):
        assert call(stride=stride) == _lib.SS_ERR_INVALID_ARG and b"plane_stride" in lib.ss_last_error()
    assert call(shards=p(store) + 8) == _lib.SS_ERR_INVALID_ARG and b"16-byte aligned" in lib.ss_last_error()
    # dec_policy may be NULL
    assert call(dec=tuple(p(x) for x in out[:4]) + (None, p(out[5]))) == 0
    torch.cuda.synchronize()
    assert ctx.device_status() == 0
    cw.close()


# ---------------------------------------------------------------------------------------------
# GPU: the closed loop -- a peer dies, the open instances cannot commit, the fallback re-sends them and they commit
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n,T,d,f,spr_old,spr_new", [(5, 5, 3, 2, 1, 3), (3, 6, 4, 1, 2, 4)])
def test_closed_loop_peer_death(ctx, oracle, n, T, d, f, spr_old, spr_new):
    from summerset_b200.engine import Acceptor, LeaderEngine
    G, leader, dead = 16, 0, n - 1
    rng = np.random.default_rng(n * 31 + T)
    pols = [[int(x) for x in oracle.cw_brr_assignment(n, T, s)] for s in (spr_old, spr_new)]
    policies = np.array(pols, dtype=np.uint32)
    eng = LeaderEngine(ctx, "crossword", G, n, f, 1, rs_total_shards=T, rs_data_shards=d)
    eng.set_policies(pols, True)
    bal = np.full(G, (3 << 8) | (leader + 1), np.uint64)
    eng.set_prepared_ballots(_t(bal))
    accs = {r: Acceptor(ctx, "crossword", G, n, r, d, T) for r in range(n)}
    keep = []
    lens = rng.integers(1, 2000, G).astype(np.uint32)
    data_off = (np.cumsum(lens.astype(np.int64) + 5) - lens.astype(np.int64)).astype(np.uint64)
    arena = rng.integers(0, 256, int(data_off[-1]) + int(lens[-1]) + 64, dtype=np.uint8)
    L = (lens.astype(np.int64) + d - 1) // d
    store = torch.zeros((T, int(((L + 31) // 32 * 32).sum()) + 32), dtype=torch.uint8, device="cuda")
    pol_old = _t(np.zeros(G, np.uint8))
    slot_out, shard_off, _ = eng.propose_ragged(_t(arena), _t(data_off), _t(lens), store, pol_old)
    slots = slot_out.cpu().numpy().view(np.uint64)
    payload = {(g, int(slots[g])): arena[int(data_off[g]):int(data_off[g]) + int(lens[g])].tobytes() for g in range(G)}
    replies = {}

    def deliver(r, st, off, dl, pol, slot, ballots, groups):
        out, o, fl, _ = ctx.frame_accept_pack_ragged(st, off, dl, d, T - d, policies, pol, r, slot, ballots, with_assignment=True)
        oh, flh, bh = o.cpu().numpy(), fl.cpu().numpy(), out.cpu().numpy()
        fr = [bh[int(oh[k]):int(oh[k]) + int(flh[k])].tobytes() for k in range(len(groups))]
        buf, offs = _buffer(rng, fr)
        astore = torch.empty(sum(len(x) for x in fr) * 2 + 64, dtype=torch.uint8, device="cuda")
        awal = torch.empty(sum(len(x) + 48 for x in fr) + 64, dtype=torch.uint8, device="cuda")
        keep.append(astore)
        res = accs[r].accept(_t(buf), _t(offs), _t(np.array(groups, np.uint32)), _t(np.full(len(groups), leader, np.uint8)), astore, awal)
        assert (res["verdict"].cpu().numpy().view(np.uint32) == ACC).all()
        reps, rl = res["replies"].cpu().numpy(), res["reply_len"].cpu().numpy()
        return [reps[k, :int(rl[k])].tobytes() for k in range(len(groups))]

    def ingest(r, reps, groups):
        rbuf, roffs = _buffer(rng, reps)
        rg, rs_, rp, rb, _ = ctx.accept_reply_parse(_t(rbuf), _t(roffs), _t(np.array(groups, np.uint32)), _t(np.full(len(groups), r, np.uint8)),
                                                     eng.window_base, with_size=True)
        eng.on_accept_replies(rg, rs_, rp, rb)

    gs = list(range(G))
    for r in range(n):                                                   # 1. every replica accepts under the old policy
        replies[r] = deliver(r, store, shard_off, _t(lens), pol_old, slot_out, _t(bal), gs)
    landed = [g for g in gs if g % 3 == 0]                               # 2. the dead peer's acks reached the leader for some
    for r in range(n - 2):
        ingest(r, replies[r], gs)
    ingest(dead, [replies[dead][g] for g in landed], landed)
    eng.tick()                                                           # 3. without the dead peer nothing can commit
    assert (eng.committed.cpu().numpy() == 0).all()
    # 4. the dead peer is gone: the spr_old instances are re-assigned the responsive policy and sent again
    alive = _t(np.full(G, ((1 << n) - 1) & ~(1 << dead), np.uint32))
    new_pol = np.ones(G, np.uint8)
    before = {k: v.clone() for k, v in (("acc", eng.accepting), ("cm", eng.committed))}
    out = torch.full((T, 1 << 16), 0xA5, dtype=torch.uint8, device="cuda")
    used = torch.zeros(1, dtype=torch.int64, device="cuda")
    res = eng.fallback_redo(_t(np.array(gs, np.uint32)), _t(new_pol), out, used, 64, peer_alive=alive)
    assert (res["verdict"].cpu().numpy().view(np.uint32) == ACC).all()
    k = int(res["totals"][0])
    assert k == G and (eng.planes.cpu().numpy() == 0).all()
    assert torch.equal(before["acc"], eng.accepting) and torch.equal(before["cm"], eng.committed)
    dec = {x: res["dec_" + x][:k] for x in ("slot", "ballot", "shard_off", "data_len", "policy", "group")}
    dg = [int(x) for x in dec["group"].cpu().numpy()]
    for r in range(n - 1):                                               # survivors and the leader itself
        reps = deliver(r, out, dec["shard_off"], dec["data_len"], dec["policy"], dec["slot"], dec["ballot"], dg)
        ingest(r, reps, dg)
        if r == n - 2:
            ingest(r, replies[r], gs)                                    # late old-round acks: credited as well
    newly = torch.empty(G, dtype=torch.int64, device="cuda")
    eng.tick(newly)
    cm = eng.committed.cpu().numpy().view(np.uint64)
    for g in gs:
        assert (int(cm[g]) >> (int(slots[g]) & 63)) & 1, g
    # the survivors learn the commit and execute the original batches byte for byte
    cb = (eng.window_base + eng.commit_bar.to(torch.int64)).cpu().numpy().view(np.uint64)
    for r in range(n - 1):
        accs[r].heartbeat(_t(np.arange(G, dtype=np.uint32)), _t(np.full(G, leader, np.uint8)), _t(bal), _t(cb), _t(np.zeros(G, np.uint64)))
        ob = torch.empty(1 << 16, dtype=torch.uint8, device="cuda")
        ex = accs[r].execute(ob, G * 64)
        ne = int(ex["totals"][0])
        obh, eg, es, eo, el = (ob.cpu().numpy(), ex["rec_group"][:ne].cpu().numpy(), ex["rec_slot"][:ne].cpu().numpy(),
                               ex["rec_off"][:ne].cpu().numpy(), ex["rec_len"][:ne].cpu().numpy())
        got = {(int(eg[x]), int(es[x])): obh[int(eo[x]):int(eo[x]) + int(el[x])].tobytes() for x in range(ne)}
        assert got == payload, r
    assert ctx.device_status() == 0
    eng.close()
    for a in accs.values():
        a.close()
