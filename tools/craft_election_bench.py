"""CRaft elections at n = 5, 2^20 groups whose leader (replica 0) died: every group elects replica 1.

  campaign  ss_follower_campaign on replica 1: every group, Metadata cells and one RequestVote frame each
  vote      ss_follower_vote on replica 2: replica 1's G RequestVote frames, Metadata and RequestVoteReply cells
            (replicas 3 and 4 answer too, untimed)
  tally     ss_follower_tally on replica 1: the 3 G replies of replicas 2-4, shuffled by frame; won_group / won_term
  step_up   ss_engine_craft_step_up(won_group, won_term, n_listed = G) from replica 1's follower

Each group's log holds slot 1 of term 1, a null entry, so step-up copies no shards: these calls move little data and
are bound by their launches, the sort and the per-group replay.  Timed with CUDA events: median of --steps calls after
--warmup; the state a call changes is restored outside the timed window.  Frames/s = frames taken (campaign: groups
listed) over the median.  b.copy_(a) of the tally's frame bytes in the same run gives the copy bandwidth the card
reaches at that size.  Check: the vote grants every frame and the tally elects every group in term 2.

Usage: python tools/craft_election_bench.py [--groups N] [--steps K] [--warmup W]
Prints the card name and power limit, one line per measurement and one JSON line.  Fails without a GPU.
"""
import argparse
import json
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))
from craft_recon_bench import timed  # noqa: E402
from engine_ragged_bench import card, stats  # noqa: E402
from summerset_b200 import _lib  # noqa: E402
from summerset_b200.api import Context  # noqa: E402
from summerset_b200.engine import Follower, RaftEngine  # noqa: E402

N = 5


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--groups", type=int, default=1 << 20)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("craft_election_bench needs a GPU")
    G = a.groups
    dev = torch.device("cuda", 0)
    ctx = Context(0)
    name, power = card()
    print(f"card: {name}, power limit {power}")
    fols = {}
    for r in range(1, N):
        f = fols[r] = Follower(ctx, G, N, r)
        f.log_end.fill_(2)
        f.term[:, 1] = 1
        f.curr_term.fill_(1)
        f.leader.fill_(0)
    groups = torch.arange(G, dtype=torch.int32, device=dev)
    source = torch.zeros(G, dtype=torch.uint8, device=dev)
    results = {}
    c = {}

    def reset(f):
        f.curr_term.fill_(1)
        f.leader.fill_(0)

    ms = timed(lambda: c.update(fols[1].campaign(groups, source)), lambda: reset(fols[1]), a)
    torch.cuda.synchronize()
    assert (c["verdict"] == _lib.SS_CAMPAIGN_VERDICT_DONE).all() and (fols[1].curr_term == 2).all()
    results["campaign"] = dict(**stats(ms), frames=G)
    # replica 1's RequestVote cells as one frame buffer
    buf = c["frames"].view(-1)
    off = torch.arange(G, dtype=torch.int64, device=dev) * Follower.VOTE_CELL
    peer1 = torch.ones(G, dtype=torch.uint8, device=dev)
    replies = []
    for r in (2, 3, 4):
        v = {}
        if r == 2:
            ms = timed(lambda: v.update(fols[r].vote(buf, off, groups, peer1)), lambda: reset(fols[r]), a)
            results["vote"] = dict(**stats(ms), frames=G)
        else:
            v.update(fols[r].vote(buf, off, groups, peer1))
        torch.cuda.synchronize()
        assert (v["verdict"] == _lib.SS_VOTE_VERDICT_GRANTED - (1 << 32)).all()
        replies.append((v["replies"].view(-1), r))
    rbuf = torch.cat([x for x, _ in replies])
    perm = torch.randperm(3 * G, device=dev)
    roff = (torch.arange(3 * G, dtype=torch.int64, device=dev) * Follower.VOTE_REPLY_CELL)[perm]
    rgrp = torch.cat([groups] * 3)[perm]
    rpeer = torch.cat([torch.full((G,), r, dtype=torch.uint8, device=dev) for _, r in replies])[perm]
    vv = fols[1].vote_view()

    def candidate():
        fols[1].curr_term.fill_(2)
        fols[1].leader.fill_(1)
        vv["role_term"].fill_(2)
        vv["role"].fill_(_lib.SS_FOLLOWER_ROLE_CANDIDATE)
        vv["votes"].fill_(1 << 1)

    t = {}
    ms = timed(lambda: t.update(fols[1].tally(rbuf, roff, rgrp, rpeer)), candidate, a)
    torch.cuda.synchronize()
    assert int(t["n_won"][0]) == G and torch.equal(t["won_group"], groups) and (t["won_term"] == 2).all()
    results["tally"] = dict(**stats(ms), frames=3 * G)
    eng = RaftEngine(ctx, G, N, craft=True)
    eng.recon_view()
    planes = torch.zeros((N, 32), dtype=torch.uint8, device=dev)
    s = {}
    ms = timed(lambda: s.update(eng.step_up(fols[1], t["won_group"], t["won_term"], planes)), lambda: None, a)
    torch.cuda.synchronize()
    assert (s["verdict"] == 0).all() and (eng.curr_term == 2).all()
    results["step_up"] = dict(**stats(ms), frames=G)
    dst = torch.empty_like(rbuf)
    ms = timed(lambda: dst.copy_(rbuf), lambda: None, a)
    results["copy"] = dict(**stats(ms), bytes=2 * rbuf.numel())
    for k, v in results.items():
        if "frames" in v:
            v["mframes_per_s"] = round(v["frames"] / (v["median_ms"] * 1e-3) / 1e6, 1)
            rate = f"{v['mframes_per_s']:.1f} M frames/s"
        else:
            v["tb_per_s"] = round(v["bytes"] / (v["median_ms"] * 1e-3) / 1e12, 3)
            rate = f"{v['tb_per_s']:.3f} TB/s"
        print(f"{k:10s} {v['median_ms']:8.3f} ms  (min {v['min_ms']:.3f}, max {v['max_ms']:.3f})  {rate}")
    print(json.dumps(dict(bench="craft_election", card=name, power_limit=power, groups=G, n=N, **results)))
    for f in fols.values():
        f.close()
    eng.close()


if __name__ == "__main__":
    main()
