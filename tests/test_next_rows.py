"""SURVEY 8f "next" rows built so far: CRaft thresholds / shadow_last_commit (f1) and the prepare-phase shard
merge + decision (f3).  CPU tests pin the oracle restatements against independent models; GPU tests compare
the kernels with the oracle, bit-exact."""
import itertools

import numpy as np
import pytest
import torch

from summerset_b200 import workloads as wl

DEV = "cuda:0"


# ---------------------------------------------------------------------------------------------
# CPU: oracle semantics
# ---------------------------------------------------------------------------------------------
def test_craft_threshold_and_shadow_commit(oracle):
    """craft/messages.rs:300-308, :677-690"""
    assert oracle.craft_threshold(3, 1, False) == 4 and oracle.craft_threshold(3, 1, True) == 3
    rng = np.random.default_rng(0)
    for n, f in [(5, 1), (7, 1), (7, 2), (3, 0), (9, 2)]:
        majority = n // 2 + 1
        for full in (False, True):
            thr = oracle.craft_threshold(majority, f, full)
            for _ in range(200):
                match = rng.integers(0, 50, n - 1)
                want = sorted(match, reverse=True)[thr - 2]
                assert oracle.craft_shadow_last_commit(match, thr) == want
                # consistency with the scan: with every entry in the current term, new_commit == min(shadow, log_end-1)
                lc, le = 0, 60
                terms = np.full(64, 7, dtype=np.uint32)
                got = oracle.raft_scan(match, lc, le, 7, terms, thr)
                assert got == max(lc, min(int(want), le - 1))


def test_raft_last_snap_is_min_match(oracle):
    """raft/messages.rs:298-309: the loop keeps the last slot every server has == min(min peer match, end_slot)."""
    rng = np.random.default_rng(3)
    for _ in range(500):
        match = rng.integers(0, 40, 6)
        last_snap, end_slot = int(rng.integers(0, 20)), int(rng.integers(0, 40))
        want = max(last_snap, min(int(match.min()), end_slot)) if end_slot > last_snap else last_snap
        assert oracle.raft_snap_scan(match, last_snap, end_slot) == want


def test_prepare_merge_is_order_independent_and_decides_like_the_handler(oracle):
    """rspaxos/messages.rs:182-259: the merged shard set does not depend on reply order; decision table."""
    rng = np.random.default_rng(1)
    for _ in range(300):
        R = 5
        has = rng.random(R) < 0.7
        bal = rng.integers(0, 4, R).astype(np.uint64)
        mask = np.array([1 << r for r in range(R)], dtype=np.uint32)       # RSPaxos: replica r voted shard r
        base = oracle.prepare_merge_stream(has, bal, mask)
        for perm in itertools.islice(itertools.permutations(range(R)), 24):
            p = list(perm)
            assert oracle.prepare_merge_stream(has[p], bal[p], mask[p]) == base
        votes = [(int(bal[r]), int(mask[r])) for r in range(R) if has[r]]
        mb = max([b for b, _ in votes], default=0)
        want = 0
        for b, m in votes:
            if b == mb:
                want |= m
        assert base == (mb, want)
    # decision table, n=5 d=3 f=1
    U, N, RC, PA = oracle.PM_USE, oracle.PM_NULL, oracle.PM_RECONSTRUCT, oracle.PM_PARITY
    assert oracle.prepare_decide(0b00111, 3, 3, 5, 1) == U | PA                 # all data, parity to compute
    assert oracle.prepare_decide(0b11111, 3, 3, 5, 1) == U                      # complete codeword
    assert oracle.prepare_decide(0b11001, 3, 3, 5, 1) == U | RC | PA            # enough shards, data missing
    assert oracle.prepare_decide(0b00011, 3, 3, 5, 1) == 0                      # too few, acks < n - f: wait
    assert oracle.prepare_decide(0b00011, 4, 3, 5, 1) == N | PA                 # too few, acks >= n - f: null batch
    assert oracle.prepare_decide(0, 5, 3, 5, 1) == N | PA
    # Crossword quirk (SURVEY 8a.10): T = 10 > population = 5: 6 shards present -> parity NOT recomputed
    assert oracle.prepare_decide(0b0000111111, 3, 6, 5, 2) == U


def test_gossip_targets_excl_semantics(oracle):
    """crossword/gossiping.rs:35-84 on hand cases (n=5, d=3, balanced spr=1: replica r holds shard r)."""
    asg = oracle.cw_brr_assignment(5, 5, 1)
    # I am replica 2 holding shard 2, leader was 0, everyone alive: ask 3 (shard 3) then 4 (shard 4) -> 3 shards, stop
    t, excl = oracle.gossip_targets_excl(2, 5, 3, 0, 0b00100, asg, 0b11111)
    assert t == 0b11000 and excl[3] == 0b00100 and excl[4] == 0b01100
    # peer 3 dead: ask 4, skip source 0, then 1
    t, excl = oracle.gossip_targets_excl(2, 5, 3, 0, 0b00100, asg, 0b10111)
    assert t == 0b10010 and excl[4] == 0b00100 and excl[1] == 0b10100
    # spr=2 assignment: one peer already covers two missing shards
    asg2 = oracle.cw_brr_assignment(5, 5, 2)
    t, excl = oracle.gossip_targets_excl(2, 5, 3, 0, int(asg2[2]), asg2, 0b11111)
    assert t == 0b01000 and excl[3] == int(asg2[2])
    # coverage is checked AFTER a peer is considered (:80-82): even with d shards held the first useful peer is asked
    t, excl = oracle.gossip_targets_excl(2, 5, 3, 0, 0b00111, asg, 0b11111)
    assert t == 0b01000 and excl[3] == 0b00111


def test_wire_format_encoders():
    """summerset_b200/wire.py: bincode-standard varints, RSCodeword Encode (rscoding.rs:54-71), framing (safetcp.rs)."""
    from summerset_b200 import wire
    assert wire.varint(0) == b"\x00" and wire.varint(250) == b"\xfa" and wire.varint(251) == b"\xfb\xfb\x00"
    assert wire.varint(65535) == b"\xfb\xff\xff" and wire.varint(65536) == b"\xfc\x00\x00\x01\x00"
    assert wire.varint((1 << 32) - 1) == b"\xfc\xff\xff\xff\xff" and wire.varint(1 << 32) == b"\xfd" + (1 << 32).to_bytes(8, "little")
    for v in [0, 1, 250, 251, 300, 65535, 65536, 1 << 31, (1 << 32) - 1, 1 << 32, (1 << 64) - 1]:
        assert wire.read_varint(wire.varint(v) + b"zz", 0) == (v, len(wire.varint(v)))
    # TestData("interesting_value") codeword, the shard replica 1 receives (SURVEY 8c KAT)
    f = wire.rspaxos_accept_frame(7, 300, 3, 2, 18, 1, bytes.fromhex("657374696e67"))
    assert f.hex() == "0000000000000018" + "00" + "02" + "07" + "fb2c01" + "03" + "02" + "12" + "06" + "05" + "00" + "0106" + "657374696e67" + "000000" + "00"
    cw, pos = wire.decode_rscodeword(f, 8 + 2 + 1 + 3)
    assert pos == len(f) and cw["shards"] == [None, b"esting", None, None, None] and not cw["has_copy"]
    assert (cw["d"], cw["p"], cw["data_len"], cw["shard_len"]) == (3, 2, 18, 6)
    assert wire.rspaxos_accept_reply_frame(5, 9) == (4).to_bytes(8, "big") + bytes([0, 3, 5, 9])
    assert wire.wal_commit_slot(1000) == bytes([2, 251]) + (1000).to_bytes(2, "little")


# ---------------------------------------------------------------------------------------------
# GPU parity
# ---------------------------------------------------------------------------------------------
def _t(a):
    a = np.ascontiguousarray(a)
    if a.dtype == np.uint64:
        a = a.view(np.int64)
    elif a.dtype == np.uint32:
        a = a.view(np.int32)
    return torch.from_numpy(a).to(DEV)


@pytest.mark.gpu
@pytest.mark.parametrize("n,f", [(5, 1), (7, 2), (3, 0), (9, 2), (11, 2), (13, 3), (17, 4)])
def test_craft_on_gpu(ctx, oracle, n, f):
    majority = n // 2 + 1
    G = 5003
    w = wl.cfg5_raft(G, n, 64, seed_extra=n + f)
    for full in (False, True):
        thr = oracle.craft_threshold(majority, f, full)
        out = ctx.raft_commit_scan(_t(w["match"]), _t(w["last_commit"]), _t(w["log_end"]), _t(w["curr_term"]),
                                   _t(w["terms"]), thr)
        sh = ctx.raft_kth_match(_t(w["match"]), thr - 1) if thr >= 2 else None
        torch.cuda.synchronize()
        want = oracle.raft_scan_batch(w["match"], w["last_commit"], w["log_end"], w["curr_term"], w["terms"], thr)
        assert (out.cpu().numpy().view(np.uint32) == want).all()
        if sh is not None:
            want_sh = np.array([oracle.craft_shadow_last_commit(w["match"][:, g], thr) for g in range(G)], dtype=np.uint32)
            assert (sh.cpu().numpy().view(np.uint32) == want_sh).all()
    # last_snap bound: every server has the entry (raft/messages.rs:298-309)
    allm = ctx.raft_kth_match(_t(w["match"]), n - 1)
    torch.cuda.synchronize()
    assert (allm.cpu().numpy().view(np.uint32) == w["match"].min(axis=0)).all()
    # every k over match values from a small range, so that ties are common: k-th largest = shadow_last_commit with
    # threshold k + 1 (craft/messages.rs:677-690)
    P = n - 1
    m = np.random.default_rng(n).integers(0, 4, (P, G)).astype(np.uint32)
    desc = -np.sort(-m.astype(np.int64), axis=0)
    for k in range(1, P + 1):
        out = ctx.raft_kth_match(_t(m), k)
        torch.cuda.synchronize()
        got = out.cpu().numpy().view(np.uint32)
        assert (got == desc[k - 1]).all(), k
        assert all(int(got[g]) == oracle.craft_shadow_last_commit(m[:, g], k + 1) for g in range(0, G, 97)), k


@pytest.mark.gpu
def test_prepare_merge_by_ballot_on_gpu_and_recovery_roundtrip(ctx, oracle):
    """merge + decision vs oracle, then the full fail-over data path on the GPU: reconstruct_all on the merged
    shard sets regenerates the codewords the USE decision promises (rspaxos/messages.rs:227-259).  A replica that
    did not vote replies ballot 0 (rspaxos/durability.rs: `voted` is None iff its ballot is 0); a non-zero ballot
    with no shards is a vote, which tests/test_failover.py covers."""
    from summerset_b200.api import ReedSolomon, round_up, shard_len
    rng = np.random.default_rng(2)
    R, d, p, population, f = 5, 3, 2, 5, 1
    N = 4099
    has = rng.random((R, N)) < 0.75
    bal = np.where(has, rng.integers(1, 4, (R, N)), 0).astype(np.uint64)          # a replica with no vote replies ballot 0
    mask = np.where(has, (1 << np.arange(R))[:, None], 0).astype(np.uint32)
    acks = rng.integers(3, 6, N).astype(np.uint8)
    mb, mg, act = ctx.prepare_merge(_t(bal), _t(mask), torch.from_numpy(acks).to(DEV), d, population, f)
    torch.cuda.synchronize()
    mb, mg, act = mb.cpu().numpy().view(np.uint64), mg.cpu().numpy().view(np.uint32), act.cpu().numpy()
    for i in range(N):
        wb, wm = oracle.prepare_merge_stream(has[:, i], bal[:, i], mask[:, i])
        assert (int(mb[i]), int(mg[i])) == (wb, wm)
        assert int(act[i]) == oracle.prepare_decide(wm, int(acks[i]), d, population, f)
    # data path: codewords whose action has USE are reconstructed in full from the merged shard set
    data_len = 1000
    rs = ReedSolomon(ctx, d, p)
    data = wl.payload_uniform(N, data_len, seed_extra=5)
    L = shard_len(data_len, d); ds = round_up(L, 16)
    full = np.zeros((d + p, N, ds), dtype=np.uint8)
    for g in range(N):
        full[:d, g, :L] = oracle.cw_split(data[g, :data_len].tobytes(), d)
    full[d:] = oracle.rs_encode_uniform(d, p, data, data_len)
    damaged = full.copy()
    for j in range(d + p):
        damaged[j, ((mg >> j) & 1) == 0] = 0xEE
    sh = torch.from_numpy(damaged).to(DEV)
    off = torch.arange(N, dtype=torch.int64, device=DEV) * ds
    st = rs.reconstruct_batch(sh, N * ds, off, torch.full((N,), data_len, dtype=torch.int32, device=DEV), _t(mg), False)
    torch.cuda.synchronize()
    got = sh.cpu().numpy(); st = st.cpu().numpy()
    use = (act & 1) == 1
    assert (st[use] == 0).all() and (st[~use & (np.array([bin(int(m)).count("1") for m in mg]) < d)] == -10).all()
    assert (got[:, use, :L] == full[:, use, :L]).all()


@pytest.mark.gpu
@pytest.mark.parametrize("variant,kernel", [(0, "rs32_crossword_distribute_kernel<1>"), (6, "rs32_crossword_distribute_kernel<8,dynamic>"),
                                            (7, "rs32_crossword_distribute_kernel<4,dynamic>")])
def test_crossword_distribute_matches_assignment_and_oracle(ctx, oracle, variant, kernel):
    """config 4 distribute (crossword/request.rs:137-185): every replica's log holds exactly the shards the balanced
    round-robin assignment gives it (crossword/mod.rs:866-888), bytes equal to the oracle's encode."""
    from summerset_b200.api import ReedSolomon, cw_slot_pitch
    rng = np.random.default_rng(6)
    d, p, n_rep = 3, 2, 5
    rs = ReedSolomon(ctx, d, p)
    rs.set_variant(variant)
    lens = np.concatenate([rng.integers(1, 3000, 300), wl.CFG4_SIZES, wl.CFG4_SIZES + 1, [0, 1, 2, 16, 48, 4096, 3072, 3073, 9001]]).astype(np.uint32)
    rng.shuffle(lens)
    n = len(lens)
    spr = rng.integers(1, 4, n).astype(np.uint8)
    lay = wl.ragged_layout(lens, d)
    arena = rng.integers(0, 256, lay["data_bytes"] + 64, dtype=np.uint8)
    L = lay["L"].astype(np.int64)
    Lpad = cw_slot_pitch(L)
    slot_bytes = spr.astype(np.int64) * Lpad
    rep_off = np.concatenate([[0], np.cumsum(slot_bytes)[:-1]]).astype(np.int64)
    total = int(slot_bytes.sum())
    logs = torch.full((n_rep, total + 64), 0x33, dtype=torch.uint8, device=DEV)
    rs.crossword_distribute(torch.from_numpy(arena).to(DEV), torch.from_numpy(lay["data_off"].astype(np.int64)).to(DEV),
                            torch.from_numpy(lens.astype(np.int32)).to(DEV), torch.from_numpy(spr).to(DEV),
                            torch.from_numpy(rep_off).to(DEV), [logs[r].data_ptr() for r in range(n_rep)])
    torch.cuda.synchronize()
    assert rs.last_kernel() == kernel
    got = logs.cpu().numpy()
    par = np.zeros((p, lay["plane_bytes"]), dtype=np.uint8)
    oracle.rs_encode_batch(d, p, arena, lay["data_off"], lens, par.reshape(-1), lay["plane_bytes"], lay["par_off"])
    for g in range(n):
        if lens[g] == 0:
            continue
        Lg = int(L[g]); lp = int(Lpad[g])
        shards = list(oracle.cw_split(arena[int(lay["data_off"][g]):int(lay["data_off"][g]) + int(lens[g])].tobytes(), d))
        shards += [par[j, int(lay["par_off"][g]):int(lay["par_off"][g]) + Lg] for j in range(p)]
        asg = oracle.cw_brr_assignment(n_rep, 5, int(spr[g]))
        for r in range(n_rep):
            held = [(r + k) % 5 for k in range(int(spr[g]))]
            assert sum(1 << j for j in held) == int(asg[r])              # the reference's assignment, bit for bit
            for k, j in enumerate(held):
                o = int(rep_off[g]) + k * lp
                assert (got[r, o:o + Lg] == shards[j]).all(), (g, r, k, j)
                assert (got[r, o + Lg:o + lp] == 0).all()
    assert (got[:, total:] == 0x33).all()                               # nothing written past the logs


@pytest.mark.gpu
@pytest.mark.parametrize("n_rep,T,d,variant", [(5, 5, 3, 4), (5, 10, 6, 0), (7, 7, 4, 0), (3, 3, 2, 0), (3, 6, 4, 0), (4, 8, 5, 0), (9, 9, 5, 0),
                                               (7, 7, 4, 1 << 11), (9, 9, 5, 1 << 11), (3, 3, 2, 1 << 11)])
def test_crossword_distribute_general_codes(ctx, oracle, n_rep, T, d, variant):
    """ss_crossword_distribute_dev for any (T, d, n) with T % n == 0 (crossword/mod.rs:805-830): replica r's log holds
    shards {(r*dj + k) mod T : k < spr} (crossword/mod.rs:866-888), bytes equal to the oracle's encode.  variant 4 runs
    the general kernel on the RS(3,2) / n = 5 case too, so the two kernels are checked against the same oracle."""
    from summerset_b200.api import ReedSolomon, cw_slot_pitch
    rng = np.random.default_rng(T * 10 + n_rep)
    p = T - d
    dj = T // n_rep
    rs = ReedSolomon(ctx, d, p)
    rs.set_variant(variant)
    lens = np.concatenate([rng.integers(1, 3000, 150), [0, 1, 2, 16, 48, 4096, 9001, 20000]]).astype(np.uint32)
    rng.shuffle(lens)
    n = len(lens)
    choices = np.arange(dj, d + 1, dj)                                   # the spr values the assignment policy can pick
    spr = choices[rng.integers(0, len(choices), n)].astype(np.uint8)
    lay = wl.ragged_layout(lens, d)
    arena = rng.integers(0, 256, lay["data_bytes"] + 64, dtype=np.uint8)
    L = lay["L"].astype(np.int64)
    Lpad = cw_slot_pitch(L)
    slot_bytes = spr.astype(np.int64) * Lpad
    rep_off = np.concatenate([[0], np.cumsum(slot_bytes)[:-1]]).astype(np.int64)
    total = int(slot_bytes.sum())
    logs = torch.full((n_rep, total + 64), 0x33, dtype=torch.uint8, device=DEV)
    rs.crossword_distribute(torch.from_numpy(arena).to(DEV), torch.from_numpy(lay["data_off"].astype(np.int64)).to(DEV),
                            torch.from_numpy(lens.astype(np.int32)).to(DEV), torch.from_numpy(spr).to(DEV),
                            torch.from_numpy(rep_off).to(DEV), [logs[r].data_ptr() for r in range(n_rep)])
    torch.cuda.synchronize()
    # the cluster codes (RS(2,1), (4,3), (5,4), (4,2)) have compile-time tables; variant bit 11 forces the run-time masks
    static = (d, T - d) in ((2, 1), (4, 3), (5, 4), (4, 2), (3, 1)) and not (variant >> 11) & 1
    assert rs.last_kernel() == ("crossword_distribute_generic_kernel<static>" if static else "crossword_distribute_generic_kernel")
    got = logs.cpu().numpy()
    par = np.zeros((p, lay["plane_bytes"]), dtype=np.uint8)
    oracle.rs_encode_batch(d, p, arena, lay["data_off"], lens, par.reshape(-1), lay["plane_bytes"], lay["par_off"])
    for g in range(n):
        if lens[g] == 0:
            continue
        Lg = int(L[g]); lp = int(Lpad[g])
        shards = list(oracle.cw_split(arena[int(lay["data_off"][g]):int(lay["data_off"][g]) + int(lens[g])].tobytes(), d))
        shards += [par[j, int(lay["par_off"][g]):int(lay["par_off"][g]) + Lg] for j in range(p)]
        asg = oracle.cw_brr_assignment(n_rep, T, int(spr[g]))
        for r in range(n_rep):
            held = [(r * dj + k) % T for k in range(int(spr[g]))]
            assert sum(1 << j for j in held) == int(asg[r])              # the reference's assignment, bit for bit
            for k, j in enumerate(held):
                o = int(rep_off[g]) + k * lp
                assert (got[r, o:o + Lg] == shards[j]).all(), (g, r, k, j)
                assert (got[r, o + Lg:o + lp] == 0).all()
    assert (got[:, total:] == 0x33).all()


SPECIAL = [0, 1, 250, 251, 252, 65535, 65536, (1 << 32) - 1, 1 << 32, (1 << 63) + 5]      # every varint boundary


def _slots_ballots(rng, n):
    slot = np.array([SPECIAL[i % len(SPECIAL)] if i < 40 else int(rng.integers(0, 1 << 40)) for i in range(n)], dtype=np.uint64)
    ballot = np.array([SPECIAL[(i // 3) % len(SPECIAL)] if i < 60 else int(rng.integers(0, 1 << 20)) for i in range(n)], dtype=np.uint64)
    return slot, ballot


def _shard_planes(oracle, d, p, data, data_len):
    from summerset_b200.api import round_up, shard_len
    n = data.shape[0]
    L = shard_len(data_len, d); ds = round_up(L, 16)
    planes = np.zeros((d + p, n, ds), dtype=np.uint8)
    for g in range(n):
        planes[:d, g, :L] = oracle.cw_split(data[g, :data_len].tobytes(), d)
    planes[d:] = oracle.rs_encode_uniform(d, p, data, data_len)
    return planes, L, ds


@pytest.mark.gpu
@pytest.mark.parametrize("d,p,data_len,shard_idx", [(3, 2, 4096, 0), (3, 2, 4096, 4), (3, 2, 18, 1), (3, 2, 1, 2), (4, 3, 1000, 5),
                                                     (3, 2, 80000, 3)])
def test_accept_frames_single_shard_fast_path_matches_oracle(ctx, oracle, d, p, data_len, shard_idx):
    """ss_frame_accept_batch_dev (one shard per frame, aligned copy) == the oracle's C encoder (oracle/ss_wire.c) byte for
    byte, for slots / ballots on every varint boundary; the output buffer is NOT zeroed beforehand."""
    from summerset_b200 import wire
    from summerset_b200.api import ReedSolomon
    rng = np.random.default_rng(8)
    n = 257
    data = wl.payload_uniform(n, data_len, seed_extra=shard_idx)
    planes, L, ds = _shard_planes(oracle, d, p, data, data_len)
    slot, ballot = _slots_ballots(rng, n)
    out, off, ln = ctx.frame_accept_batch(torch.from_numpy(planes[shard_idx]).to(DEV), shard_idx, d, p, data_len, _t(slot), _t(ballot))
    torch.cuda.synchronize()
    out = out.cpu().numpy().reshape(-1); off = off.cpu().numpy(); ln = ln.cpu().numpy()
    for g in range(n):
        shards = [None] * (d + p)
        shards[shard_idx] = planes[shard_idx, g, :L].tobytes()
        want = oracle.frame_accept(2, int(slot[g]), int(ballot[g]), d, p, data_len, shards)
        got = out[int(off[g]):int(off[g]) + int(ln[g])].tobytes()
        assert got == want, (g, int(slot[g]), int(ballot[g]))
        assert got == wire.rspaxos_accept_frame(int(slot[g]), int(ballot[g]), d, p, data_len, shard_idx, shards[shard_idx])  # host encoder too
        assert (int(off[g]) + len(want) - L - (d + p - shard_idx)) % 16 == 0     # shard payload 16-byte aligned
        dec = oracle.decode_accept(got, 0)                                       # decode(encode(x)) == x
        assert dec and (dec["slot"], dec["ballot"], dec["d"], dec["p"], dec["data_len"], dec["shard_len"]) == \
            (int(slot[g]), int(ballot[g]), d, p, data_len, L) and dec["shards"] == shards


@pytest.mark.gpu
def test_accept_frames_many_shards_and_late_shard_index(ctx, oracle):
    """ADVICE r1: more than 32 shards (None runs longer than a warp) and a shard index far beyond the old header array."""
    rng = np.random.default_rng(9)
    d, p, data_len, n = 40, 30, 4000, 33
    L = (data_len + d - 1) // d; ds = (L + 15) // 16 * 16
    for shard_idx in (0, 33, 69):
        plane = rng.integers(0, 256, (n, ds), dtype=np.uint8)
        plane[:, L:] = 0
        slot, ballot = _slots_ballots(rng, n)
        out, off, ln = ctx.frame_accept_batch(torch.from_numpy(plane).to(DEV), shard_idx, d, p, data_len, _t(slot), _t(ballot))
        torch.cuda.synchronize()
        out = out.cpu().numpy().reshape(-1); off = off.cpu().numpy(); ln = ln.cpu().numpy()
        for g in range(n):
            shards = [None] * (d + p)
            shards[shard_idx] = plane[g, :L].tobytes()
            assert out[int(off[g]):int(off[g]) + int(ln[g])].tobytes() == oracle.frame_accept(2, int(slot[g]), int(ballot[g]), d, p, data_len, shards)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["rspaxos_accept", "crossword_accept", "wal_accept_data"])
@pytest.mark.parametrize("data_len", [1, 100, 4096, 9001])
def test_general_frame_packer_matches_oracle(ctx, oracle, kind, data_len):
    """ss_frame_accept_pack_dev: PeerMsg::Accept frames for one peer with the shards of its assignment (one in RSPaxos,
    spr in Crossword, plus assignment: Vec<Bitmap>) and WalEntry::AcceptData records, byte for byte against the oracle's
    encoder (rspaxos/mod.rs:212-232,283-288, crossword/mod.rs:356-362, rscoding.rs:43-72, bitmap.rs:20-30)."""
    rng = np.random.default_rng(len(kind) + data_len)
    d, p, pop, n = 3, 2, 5, 131
    T = d + p
    data = wl.payload_uniform(n, data_len, seed_extra=data_len)
    planes, L, ds = _shard_planes(oracle, d, p, data, data_len)
    slot, ballot = _slots_ballots(rng, n)
    if kind == "crossword_accept":
        policies = [list(map(int, oracle.cw_brr_assignment(pop, T, spr))) for spr in (1, 2, 3)]
        policies.append([int(x) for x in rng.integers(0, 1 << T, pop)])           # an unbalanced assignment, possibly empty masks
        pidx = rng.integers(0, len(policies), n).astype(np.uint8)
    else:
        policies = [[1 << r for r in range(pop)]]                                 # replica r holds shard r (rspaxos/request.rs:135-137)
        pidx = np.zeros(n, dtype=np.uint8)
    for peer in (0, 3, 4):
        out, off, ln = ctx.frame_accept_pack(torch.from_numpy(planes).to(DEV), data_len, d, p, policies, torch.from_numpy(pidx).to(DEV),
                                             peer, _t(slot), _t(ballot), kind=1 if kind == "wal_accept_data" else 0,
                                             msg_variant=1 if kind == "wal_accept_data" else 2, with_assignment=kind == "crossword_accept")
        torch.cuda.synchronize()
        out = out.cpu().numpy().reshape(-1); off = off.cpu().numpy(); ln = ln.cpu().numpy()
        for g in range(n):
            mask = policies[int(pidx[g])][peer]
            shards = [planes[j, g, :L].tobytes() if (mask >> j) & 1 else None for j in range(T)]
            if not any(s is not None for s in shards):
                # a peer the assignment gives nothing: every shard None, the codeword still states its geometry
                got = out[int(off[g]):int(off[g]) + int(ln[g])].tobytes()
                dec = oracle.decode_accept(got, 0, kind == "crossword_accept")
                assert dec and dec["shards"] == [None] * T and dec["shard_len"] == L and dec["slot"] == int(slot[g])
                continue
            if kind == "wal_accept_data":
                want = oracle.wal_accept_data(int(slot[g]), int(ballot[g]), d, p, data_len, shards)
            else:
                want = oracle.frame_accept(2, int(slot[g]), int(ballot[g]), d, p, data_len, shards,
                                           policies[int(pidx[g])] if kind == "crossword_accept" else None, T)
            got = out[int(off[g]):int(off[g]) + int(ln[g])].tobytes()
            assert got == want, (kind, peer, g)
            dec = oracle.decode_accept(got, 1 if kind == "wal_accept_data" else 0, kind == "crossword_accept")
            assert dec and dec["shards"] == shards and dec["ballot"] == int(ballot[g])
            if kind == "crossword_accept":
                assert dec["assignment"] == policies[int(pidx[g])] and dec["assign_size"] == T


@pytest.mark.gpu
def test_frame_packer_refuses_frames_that_do_not_fit(ctx, oracle):
    """a slot too small for its frame: nothing is written for that codeword, frame_len = 0, status bit 2"""
    d, p, pop, n, data_len = 3, 2, 5, 40, 4096
    data = wl.payload_uniform(n, data_len, seed_extra=5)
    planes, L, ds = _shard_planes(oracle, d, p, data, data_len)
    slot = np.arange(n, dtype=np.uint64); ballot = np.full(n, 7, dtype=np.uint64)
    policies = [[0b00111, 0b01110, 0b11100, 0b11001, 0b10011]]                       # three shards per peer
    small = ((L + 128) + 15) // 16 * 16                                              # room for one shard only
    out, off, ln = ctx.frame_accept_pack(torch.from_numpy(planes).to(DEV), data_len, d, p, policies, None, 0, _t(slot), _t(ballot),
                                         frame_stride=small)
    torch.cuda.synchronize()
    assert int(ln.abs().sum()) == 0 and (out.cpu().numpy() == 0xA5).all()
    assert ctx.device_status() == 4
    out, off, ln = ctx.frame_accept_pack(torch.from_numpy(planes).to(DEV), data_len, d, p, policies, None, 0, _t(slot), _t(ballot))
    torch.cuda.synchronize()
    assert (ln.cpu().numpy() > 3 * L).all() and ctx.device_status() == 0


@pytest.mark.gpu
@pytest.mark.parametrize("with_size", [False, True])
def test_accept_reply_parser_feeds_ingest(ctx, oracle, with_size):
    """AcceptReply frames (rspaxos/mod.rs:290-291; crossword/mod.rs:365-373 with size + reply_ts) interleaved with other
    messages, a truncated frame and garbage -> records identical to the oracle's parser, window-relative slots, and the
    records drive ss_ack_ingest_dev to the same planes as the oracle's per-message handler."""
    rng = np.random.default_rng(21 + with_size)
    G, R, n = 300, 5, 5000
    base = rng.integers(0, 1 << 34, G).astype(np.uint64)
    bal = rng.integers(1, 1 << 33, G).astype(np.uint64)
    frames, fgroup, fpeer = [], [], []
    for i in range(n):
        g = int(rng.integers(0, G)); peer = int(rng.integers(0, R))
        r = rng.random()
        slot = int(base[g]) + int(rng.integers(-3, 70))            # below the window, inside, beyond
        slot = max(slot, 0)
        ballot = int(bal[g]) if rng.random() < 0.8 else int(rng.integers(1, 1 << 33))
        if r < 0.8:
            fr = oracle.frame_accept_reply(3, slot, ballot, with_size, int(rng.integers(0, 1 << 20)))
            if with_size and rng.random() < 0.3:                    # reply_ts: Some(SystemTime{secs, nanos})
                body = fr[8:-1] + b"\x01" + oracle.varint(1_700_000_000) + oracle.varint(123456789)
                fr = len(body).to_bytes(8, "big") + body
        elif r < 0.9:
            fr = oracle.frame_accept_reply(6, slot, ballot)         # some other PeerMsg (Heartbeat index): not ours
        elif r < 0.95:
            fr = oracle.frame_accept_reply(3, slot, ballot, with_size, 5)[:-2]      # truncated body, stale length
        else:
            fr = (9).to_bytes(8, "big") + bytes(rng.integers(251, 256, 9).astype(np.uint8))   # garbage varints
        frames.append(fr); fgroup.append(g); fpeer.append(peer)
    offs = np.concatenate([[0], np.cumsum([len(f) for f in frames])]).astype(np.uint64)
    buf = np.frombuffer(b"".join(frames), dtype=np.uint8)
    rg, rs_, rp, rb, rk = ctx.accept_reply_parse(torch.from_numpy(buf.copy()).to(DEV), _t(offs[:-1]), _t(np.array(fgroup, dtype=np.uint32)),
                                                 torch.from_numpy(np.array(fpeer, dtype=np.uint8)).to(DEV), _t(base), 3, with_size)
    torch.cuda.synchronize()
    rg, rs_, rp, rb, rk = (x.cpu().numpy() for x in (rg, rs_, rp, rb, rk))
    n_ok = 0
    for i in range(n):
        # the parser only sees the bytes up to the next frame's offset... the oracle gets the same view: the whole rest of the buffer
        ln, slot, ballot, size, kind = oracle.parse_accept_reply(buf[int(offs[i]):].tobytes()[:4096], 3, with_size)
        if ln > 0:
            n_ok += 1
            assert rk[i] == 3 and int(rb[i]) == ballot
            rel = slot - int(base[fgroup[i]])
            assert rs_[i] == (rel if 0 <= rel < 64 else 0xff)
        elif ln == -2:
            assert np.uint32(rk[i]) == np.uint32(kind) and rs_[i] == 0xff
        else:
            assert np.uint32(rk[i]) == 0xFFFFFFFF and rs_[i] == 0xff
        assert rg[i] == fgroup[i] and rp[i] == fpeer[i]
    assert n_ok > 0.6 * n
    # the records go straight into the ingest kernel
    inst_bal = np.zeros(G * 64, dtype=np.uint64); accepting = np.full(G, np.uint64(0xFFFFFFFFFFFFFFFF)); status = np.full(G * 64, oracle.ST_ACCEPTING, dtype=np.uint8)
    acks = np.zeros(G * 64, dtype=np.uint16)
    planes = torch.zeros((R, G), dtype=torch.int64, device=DEV)
    ctx.ack_ingest(_t(rg.view(np.uint32)), torch.from_numpy(rs_).to(DEV), torch.from_numpy(rp).to(DEV), _t(rb.view(np.uint64)),
                   _t(bal), _t(inst_bal), _t(accepting), R, planes)
    torch.cuda.synchronize()
    keep = rs_ != 0xff
    oracle.tally_stream(rg.view(np.uint32)[keep], rs_[keep], rp[keep], rb.view(np.uint64)[keep], 64, R, 99, bal, inst_bal, status, acks)
    got = planes.cpu().numpy().view(np.uint64)
    for r in range(R):
        want_plane = np.packbits(((acks.reshape(G, 64) >> r) & 1).astype(np.uint8), axis=1, bitorder="little").view(np.uint64).reshape(-1)
        assert (got[r] == want_plane).all()


@pytest.mark.gpu
def test_wal_commit_slot_packer(ctx, oracle):
    """newly committed instances -> WalEntry::CommitSlot{slot} records (rspaxos/mod.rs:231) with the StorageHub length prefix"""
    rng = np.random.default_rng(31)
    G = 4001
    newly = (rng.integers(0, 1 << 62, G).astype(np.uint64) & rng.integers(0, 1 << 62, G).astype(np.uint64) & rng.integers(0, 1 << 62, G).astype(np.uint64))
    newly[::7] = 0
    newly[5] = np.uint64(1 << 63)
    base = rng.integers(0, 1 << 40, G).astype(np.uint64)
    base[:4] = [0, 186, 250, 65530]                                 # varint boundaries
    total = int(sum(bin(int(w)).count("1") for w in newly))
    entries, eg, el, cnt = ctx.wal_commit_pack(_t(newly), _t(base), total + 10)
    torch.cuda.synchronize()
    assert int(cnt) == total
    entries = entries.cpu().numpy(); eg = eg.cpu().numpy(); el = el.cpu().numpy()
    got = sorted((int(eg[e]), entries[e, :int(el[e])].tobytes()) for e in range(total))
    want = sorted((g, oracle.wal_commit_slot(int(base[g]) + s)) for g in range(G) for s in range(64) if (int(newly[g]) >> s) & 1)
    assert got == want
    # capacity smaller than needed: counted, nothing written past the end
    entries2, _, _, cnt2 = ctx.wal_commit_pack(_t(newly), _t(base), 16)
    torch.cuda.synchronize()
    assert int(cnt2) == total and entries2.shape[0] == 16


@pytest.mark.gpu
@pytest.mark.parametrize("T,data_len", [(5, 4096), (5, 18), (7, 1000), (10, 3000)])
def test_reconstruct_serving_matches_oracle(ctx, oracle, T, data_len):
    """crossword/messages.rs:577-632: reply shards = held & flip(exclude) for instances at least Accepting, copied out
    packed; no entry when the status is lower or nothing is left."""
    from summerset_b200.api import round_up
    rng = np.random.default_rng(T + data_len)
    d = T // 2 + 1 if T != 10 else 6
    n = 500
    L = (data_len + d - 1) // d; ds = round_up(L, 16)
    planes = rng.integers(0, 256, (T, n, ds), dtype=np.uint8)
    planes[:, :, L:] = 0
    R = 1300
    req_group = rng.integers(0, n, R).astype(np.uint32)
    held = rng.integers(0, 1 << T, R).astype(np.uint32)
    excl = rng.integers(0, 1 << T, R).astype(np.uint32)
    excl[::11] = (1 << T) - 1                                       # requester already has everything
    status = rng.integers(0, 5, R).astype(np.uint8)
    want_mask = np.array([oracle.reconstruct_serve_mask(int(h), int(x), T, int(st)) for h, x, st in zip(held, excl, status)], dtype=np.uint32)
    cnt = np.array([bin(int(m)).count("1") for m in want_mask], dtype=np.int64)
    reply_off = np.concatenate([[0], np.cumsum(cnt * ds)[:-1]]).astype(np.uint64)
    total = int((cnt * ds).sum())
    mask, out = ctx.reconstruct_serve(torch.from_numpy(planes).to(DEV), L, _t(req_group), _t(held), _t(excl), torch.from_numpy(status).to(DEV),
                                      _t(reply_off), total + 64)
    torch.cuda.synchronize()
    assert (mask.cpu().numpy().view(np.uint32) == want_mask).all()
    out = out.cpu().numpy()
    assert (out[total:] == 0x77).all()
    for i in range(R):
        o = int(reply_off[i])
        for j in range(T):
            if (int(want_mask[i]) >> j) & 1:
                assert (out[o:o + ds] == planes[j, req_group[i]]).all(), (i, j)      # subset_copy: the shard, bit for bit
                o += ds
    assert (want_mask != 0).mean() > 0.3


@pytest.mark.gpu
def test_gossip_plan_on_gpu(ctx, oracle):
    rng = np.random.default_rng(11)
    for n, T, d in [(5, 5, 3), (7, 7, 4), (5, 10, 6)]:
        dj = T // n
        policies = [oracle.cw_brr_assignment(n, T, spr) for spr in range(dj, d + 1, dj)]
        policies.append(rng.integers(0, 1 << T, size=n).astype(np.uint32))          # an unbalanced one
        K = len(policies)
        N = 6007
        me = int(rng.integers(0, n))
        alive = int(rng.integers(0, 1 << n)) | (1 << me)
        src = rng.integers(0, n, N).astype(np.uint8)
        avail = rng.integers(0, 1 << T, N).astype(np.uint32)
        pidx = rng.integers(0, K, N).astype(np.uint8)
        targets, excl = ctx.gossip_plan(me, n, d, torch.from_numpy(src).to(DEV), _t(avail), torch.from_numpy(pidx).to(DEV),
                                        [list(map(int, q)) for q in policies], alive)
        torch.cuda.synchronize()
        targets = targets.cpu().numpy().view(np.uint32); excl = excl.cpu().numpy().view(np.uint32)
        for i in range(N):
            wt, we = oracle.gossip_targets_excl(me, n, d, int(src[i]), int(avail[i]), policies[int(pidx[i])], alive)
            assert int(targets[i]) == wt, (n, i)
            for peer in range(n):
                if (wt >> peer) & 1:
                    assert int(excl[peer, i]) == int(we[peer])
                else:
                    assert int(excl[peer, i]) == 0xFFFFFFFF       # untouched
