"""GPU parity tests for the quorum tallies, ack ingest, Crossword predicate and Raft scan: CUDA kernels
through the C ABI vs the CPU oracle's restatement of the reference handlers, bit-exact."""
from pathlib import Path

import numpy as np
import pytest
import torch

from summerset_b200 import workloads as wl

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _t(a, dtype=None):
    a = np.ascontiguousarray(a)
    if a.dtype == np.uint64:
        a = a.view(np.int64)
    elif a.dtype == np.uint32:
        a = a.view(np.int32)
    elif a.dtype == np.uint16:
        a = a.view(np.int16)
    return torch.from_numpy(a).to(DEV)


@pytest.mark.parametrize("R", [1, 3, 5, 7, 9, 16])
def test_tally_planes_matches_oracle(ctx, oracle, R):
    for G in (1, 2, 63, 1000, 70001):
        planes = wl.cfg2_planes(G, R, 0.7, seed_extra=R)
        for thr in sorted({0, 1, R // 2 + 1, R // 2 + 1 + (R // 2) // 2, R, R + 1, 40}):
            c, bar = ctx.tally_planes(_t(planes), thr)
            torch.cuda.synchronize()
            cw, bw = oracle.tally_planes(planes, thr)
            assert (c.cpu().numpy().view(np.uint64) == cw).all(), (R, G, thr)
            assert (bar.cpu().numpy().view(np.uint32) == bw).all(), (R, G, thr)


def test_tally_planes_host_entry_point(ctx, oracle):
    planes = wl.cfg2_planes(5000, 5, 0.9)
    c, bar = ctx.tally_planes_host(planes, 3)
    cw, bw = oracle.tally_planes(planes, 3)
    assert (c == cw).all() and (bar == bw).all()


def test_tally_golden_fixture(ctx):
    z = np.load(Path(__file__).parent / "golden" / "tally_golden.npz")
    c, bar = ctx.tally_planes(_t(z["planes"]), int(z["threshold"]))
    torch.cuda.synchronize()
    assert (c.cpu().numpy().view(np.uint64) == z["committed"]).all()
    assert (bar.cpu().numpy().view(np.uint32) == z["commit_bar"]).all()
    out = ctx.raft_commit_scan(_t(z["raft_match"]), _t(z["raft_last_commit"]), _t(z["raft_log_end"]),
                               _t(z["raft_curr_term"]), _t(z["raft_terms"]), int(z["raft_threshold"]))
    torch.cuda.synchronize()
    assert (out.cpu().numpy().view(np.uint32) == z["raft_new_commit"]).all()


@pytest.mark.parametrize("width", [1, 2])
def test_tally_masks_matches_oracle(ctx, oracle, width):
    rng = np.random.default_rng(width)
    for n in (1, 15, 16, 17, 63, 64, 65, 1000, 100003):
        nbits = 8 if width == 1 else 13
        masks = rng.integers(0, 1 << nbits, n).astype(np.uint8 if width == 1 else np.uint16)
        for thr in (0, 1, 3, 4, 8, 9, 14):
            bits = ctx.tally_masks(_t(masks), thr)
            torch.cuda.synchronize()
            got = np.unpackbits(bits.cpu().numpy().view(np.uint8), bitorder="little")
            want = oracle.tally_masks(masks.astype(np.uint16), thr)
            assert (got[:n] == want).all(), (n, thr)
            assert (got[n:] == 0).all()


def test_masks_and_planes_agree(ctx):
    """the two layouts of the same votes give the same commit bits"""
    G, R = 2000, 5
    planes = wl.cfg2_planes(G, R, 0.6)
    bits = np.unpackbits(planes.view(np.uint8).reshape(R, G, 8), axis=2, bitorder="little")   # [R, G, 64]
    masks = np.zeros((G, 64), dtype=np.uint8)
    for r in range(R):
        masks |= (bits[r] << r).astype(np.uint8)
    c, _ = ctx.tally_planes(_t(planes), 3)
    m = ctx.tally_masks(_t(masks.reshape(-1)), 3)
    torch.cuda.synchronize()
    assert torch.equal(c, m)


def test_ack_ingest_matches_stream_handler(ctx, oracle):
    """record stream with duplicates / stale ballots / non-accepting instances / bad peers ->
    planes; then the tally equals the end state of the reference's per-ack handler."""
    G, R, thr = 3000, 5, 3
    planes = wl.cfg2_planes(G, R, 0.6, seed_extra=9)
    rec = wl.ack_records(planes, seed_extra=9)
    dplanes = torch.zeros((R, G), dtype=torch.int64, device=DEV)
    ctx.ack_ingest(_t(rec["rec_group"]), _t(rec["rec_slot"]), _t(rec["rec_peer"]), _t(rec["rec_ballot"]),
                   _t(rec["bal_prepared"]), _t(rec["inst_bal"]), _t(rec["accepting"]), R, dplanes)
    c, _ = ctx.tally_planes(dplanes, thr)
    torch.cuda.synchronize()
    status = np.zeros(G * 64, dtype=np.uint8)
    acc_bits = np.unpackbits(rec["accepting"].view(np.uint8).reshape(G, 8), axis=1, bitorder="little").reshape(-1)
    status[acc_bits == 1] = oracle.ST_ACCEPTING
    status[acc_bits == 0] = oracle.ST_NULL
    acks = np.zeros(G * 64, dtype=np.uint16)
    oracle.tally_stream(rec["rec_group"], rec["rec_slot"], rec["rec_peer"], rec["rec_ballot"], 64, R, thr,
                        rec["bal_prepared"], rec["inst_bal"], status, acks)
    want = np.packbits(status.reshape(G, 64) == oracle.ST_COMMITTED, axis=1, bitorder="little").view(np.uint64).reshape(-1)
    assert (c.cpu().numpy().view(np.uint64) == want).all()
    # the ingested planes hold exactly the valid acks (a superset of what the handler recorded
    # before it stopped at the threshold)
    got_planes = dplanes.cpu().numpy().view(np.uint64)
    ok = rec["inst_bal"].reshape(G, 64) <= rec["bal_prepared"][:, None]
    okw = np.packbits(ok, axis=1, bitorder="little").view(np.uint64).reshape(-1)
    assert (got_planes == (planes & rec["accepting"][None, :] & okw[None, :])).all()


@pytest.mark.parametrize("balanced", [True, False])
def test_crossword_matches_oracle(ctx, oracle, balanced):
    """Up to 12 replicas and 16 policies (a 16 x 2^12-bit LUT, 8 KB of shared memory).  A policy_idx >= n_policies
    never commits, as in the engine tick."""
    rng = np.random.default_rng(17)
    for n, T, d, f, K in [(5, 5, 3, 2, 0), (5, 5, 3, 1, 0), (5, 5, 3, 0, 0), (7, 7, 4, 3, 0), (3, 3, 2, 1, 0), (5, 10, 6, 2, 0),
                          (9, 9, 5, 2, 0), (10, 10, 6, 2, 0), (11, 11, 6, 3, 0), (12, 12, 7, 2, 0), (12, 24, 13, 1, 0),
                          (12, 12, 7, 2, 16)]:
        majority = n // 2 + 1
        dj = T // n
        if balanced:
            policies = [oracle.cw_brr_assignment(n, T, spr) for spr in range(dj, d + 1, dj)]
        else:
            policies = [rng.integers(0, 1 << T, size=n).astype(np.uint32) for _ in range(4)]
            policies.append(oracle.cw_brr_assignment(n, T, dj))
        if K:                                                       # cycle / draw up to exactly K policies
            while len(policies) < K:
                policies.append(policies[len(policies) % 4] if balanced else rng.integers(0, 1 << T, size=n).astype(np.uint32))
            policies = policies[:K]
        K = len(policies)
        N = 20011
        width = np.uint8 if n <= 8 else np.uint16
        masks = rng.integers(0, 1 << n, N).astype(width)
        pidx = rng.integers(0, K, N).astype(np.uint8)
        bad = rng.random(N) < 0.05
        pidx[bad] = rng.integers(K, 256, int(bad.sum()))              # out-of-range policy: never commits
        bits = ctx.tally_crossword(_t(masks), _t(pidx), [list(map(int, pol)) for pol in policies], T, d, majority, f, balanced)
        torch.cuda.synchronize()
        got = np.unpackbits(bits.cpu().numpy().view(np.uint8), bitorder="little")[:N]
        lut = np.array([[oracle.cw_committed(T, n, d, majority, f, a, policies[k], balanced) for a in range(1 << n)]
                        for k in range(K)], dtype=np.uint8)
        want = np.where(bad, 0, lut[np.minimum(pidx, K - 1), masks.astype(np.int64)]).astype(np.uint8)
        assert (got == want).all(), (n, T, d, f, K)
        assert want[~bad].any() and not got[bad].any()


@pytest.mark.parametrize("n_rep,thr", [(7, 4), (5, 3), (3, 2), (9, 5), (5, 4), (7, 6), (2, 2), (1, 1), (5, 9),
                                       # 9..16 peers: the NP = 16 instance; thresholds 1, majority and n_rep
                                       (10, 1), (10, 6), (10, 10), (12, 1), (12, 7), (12, 12), (13, 1), (13, 7), (13, 13),
                                       (17, 1), (17, 9), (17, 17)])
def test_raft_scan_matches_oracle(ctx, oracle, n_rep, thr):
    # W % 4 != 0 takes the cooperative warp walk, W % 4 == 0 the vectorised one
    for G, W in [(1, 64), (33, 64), (5000, 64), (777, 17), (300, 200), (777, 1), (777, 2), (777, 3)]:
        w = wl.cfg5_raft(G, n_rep, W, seed_extra=n_rep * 10 + thr)
        match = w["match"] if n_rep > 1 else np.zeros((0, G), dtype=np.uint32)
        if n_rep == 1:
            mt = torch.zeros((0, G), dtype=torch.int32, device=DEV)
        else:
            mt = _t(match)
        out = ctx.raft_commit_scan(mt, _t(w["last_commit"]), _t(w["log_end"]), _t(w["curr_term"]), _t(w["terms"]), thr)
        torch.cuda.synchronize()
        want = oracle.raft_scan_batch(match, w["last_commit"], w["log_end"], w["curr_term"], w["terms"], thr)
        assert (out.cpu().numpy().view(np.uint32) == want).all(), (G, W)


def test_raft_adversarial_terms(ctx, oracle):
    """arbitrary (non-monotone) term windows, short logs, stale matches"""
    rng = np.random.default_rng(4)
    G, W, P = 4096, 64, 6
    last_commit = rng.integers(0, 1000, G).astype(np.uint32)
    log_len = rng.integers(0, W + 1, G).astype(np.uint32)           # entries after last_commit
    log_end = last_commit + 1 + log_len
    log_end[::97] = 0                                               # degenerate: empty log
    match = rng.integers(0, 1100, (P, G)).astype(np.uint32)
    curr = rng.integers(1, 4, G).astype(np.uint32)
    terms = rng.integers(1, 4, (G, W)).astype(np.uint32)
    for thr in (1, 2, 4, 7, 8):
        out = ctx.raft_commit_scan(_t(match), _t(last_commit), _t(log_end), _t(curr), _t(terms), thr)
        torch.cuda.synchronize()
        want = np.array([oracle.raft_scan(match[:, g], int(last_commit[g]), int(log_end[g]), int(curr[g]),
                                          terms[g], thr) if log_end[g] > 0 else last_commit[g] for g in range(G)],
                        dtype=np.uint32)
        assert (out.cpu().numpy().view(np.uint32) == want).all(), thr


def test_full_size_tally_properties(ctx, oracle):
    """BASELINE config 2 at full size: 2^20 groups x 64 slots, n=5, threshold 3."""
    G, R = 1 << 20, 5
    g = torch.Generator(device=DEV); g.manual_seed(wl.SEED_BASE + 2)
    planes = torch.randint(-(1 << 62), 1 << 62, (R, G), dtype=torch.int64, device=DEV, generator=g)
    planes[0] = -1                                                  # leader always acks
    c3, bar = ctx.tally_planes(planes, 3)
    c4, _ = ctx.tally_planes(planes, 4)
    c0, _ = ctx.tally_planes(planes, 0)
    c6, _ = ctx.tally_planes(planes, 6)
    torch.cuda.synchronize()
    assert int((c4 & ~c3).abs().sum()) == 0                         # monotone in the threshold
    assert bool((c0 == -1).all()) and bool((c6 == 0).all())
    # complement symmetry: count >= 3 of 5  <=>  NOT (count of complements >= 3)
    cc, _ = ctx.tally_planes(~planes, 3)
    assert torch.equal(cc, ~c3)
    idx = torch.arange(0, G, 4099, device=DEV)
    cw, bw = oracle.tally_planes(planes[:, idx].cpu().numpy().view(np.uint64), 3)
    assert (c3[idx].cpu().numpy().view(np.uint64) == cw).all() and (bar[idx].cpu().numpy().view(np.uint32) == bw).all()
