"""CRaft leader fail-over at n = 5 (RS(3,2)), 2^14 groups, 32 committed entries of 4 KB per group in 1-shard mode.

  step_up   ss_engine_craft_step_up: replica 1's follower log becomes the new leader's, its one held shard per entry
            copied into the leader's planes
  serve     ss_follower_reconstruct_serve on replica 2: the new leader's Reconstruct frames (10 slots each) answered
            with the shard it holds
  absorb    ss_engine_craft_absorb: the replies of replicas 2 and 3, two shards per entry written into the reserved slots
  execute   ss_engine_craft_execute: every entry now holds shards 1, 2 and 3, so data shard 0 is regenerated

The entries are coded by a first leader (ss_engine_craft_propose, one plane set per round); the followers' state is
installed through their views, each holding shard r of every entry in place in those planes.  Timed with CUDA events:
median of --steps calls after --warmup; the state a call changes is restored outside the timed window.  Bytes moved are
the algorithmic bytes: shard bytes read plus shard, frame or payload bytes written.  b.copy_(a) of the execute's bytes
in the same run gives the copy bandwidth the card reaches (it counts 2x its bytes).  Check: every payload equals its batch.

Usage: python tools/craft_recon_bench.py [--groups N] [--steps K] [--warmup W]
Prints the card name and power limit, one line per measurement and one JSON line.  Fails without a GPU.
"""
import argparse
import json
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))
from engine_ragged_bench import card, stats  # noqa: E402
from summerset_b200.api import Context  # noqa: E402
from summerset_b200.engine import Follower, RaftEngine  # noqa: E402

N, DATA_LEN, ENTRIES, CHUNK = 5, 4096, 32, 10
D = N // 2 + 1
L = -(-DATA_LEN // D)
PITCH = (L + 31) & ~31
R16 = (L + 15) & ~15


def timed(fn, prep, a):
    ms = []
    for step in range(a.warmup + a.steps):
        prep()
        e = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        e[0].record()
        fn()
        e[1].record()
        torch.cuda.synchronize()
        if step >= a.warmup:
            ms.append(e[0].elapsed_time(e[1]))
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--groups", type=int, default=1 << 14)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("craft_recon_bench needs a GPU")
    G, E = a.groups, ENTRIES
    dev = torch.device("cuda", 0)
    ctx = Context(0)
    name, power = card()
    print(f"card: {name}, power limit {power}")
    gen = torch.Generator(device=dev).manual_seed(1)
    arena = torch.randint(0, 256, (G * DATA_LEN + 16 * E,), dtype=torch.uint8, device=dev, generator=gen)
    first = RaftEngine(ctx, G, N, craft=True)
    first.curr_term.fill_(1)
    plane_sets = []
    for k in range(E):                                            # slot k + 1: the batches at arena + 16k
        planes = torch.zeros((N, G * PITCH), dtype=torch.uint8, device=dev)
        o = first.propose(0, arena, torch.arange(G, dtype=torch.int64, device=dev) * DATA_LEN + 16 * k,
                          torch.full((G,), DATA_LEN, dtype=torch.int32, device=dev), planes,
                          torch.zeros(G * 4096, dtype=torch.uint8, device=dev))
        torch.cuda.synchronize()
        assert (o["slot_out"] == k + 1).all()
        plane_sets.append(planes)
    first.close()
    fols = {}
    for r in (1, 2, 3):
        f = fols[r] = Follower(ctx, G, N, r)
        f.log_end.fill_(E + 1)
        f.curr_term.fill_(1)
        f.term[:, 1:E + 1] = 1
        f.data_len[:, 1:E + 1] = DATA_LEN
        f.held[:, 1:E + 1] = 1 << r
        for k in range(E):
            f.shard_addr[:, k + 1] = plane_sets[k][r].data_ptr() + torch.arange(G, dtype=torch.int64, device=dev) * PITCH
    eng = RaftEngine(ctx, G, N, craft=True)
    rv, lv, ev = eng.recon_view(), eng.log_view(), eng.exec_view()
    planes = torch.zeros((N, G * E * PITCH), dtype=torch.uint8, device=dev)
    groups = torch.arange(G, dtype=torch.int32, device=dev)
    term = torch.full((G,), 2, dtype=torch.int64, device=dev)
    results = {}
    res = {}
    ms = timed(lambda: res.update(eng.step_up(fols[1], groups, term, planes)), lambda: None, a)
    assert (res["verdict"] == 0).all() and int(res["need"][0]) == G * E * PITCH
    results["step_up"] = dict(**stats(ms), bytes=2 * G * E * R16)
    # the leader's log now ends at slot E, committed (as the tick commits it once an entry of term 2 is acknowledged)
    eng.last_commit.fill_(E)
    out = torch.zeros(G * 256, dtype=torch.uint8, device=dev)
    r = eng.reconstruct_reads(out, G * 8, CHUNK)
    torch.cuda.synchronize()
    nf = int(r["totals"][0])
    assert nf == G * -(-E // CHUNK)
    fo, fg = r["frame_off"][:nf], r["frame_group"][:nf]
    peer = torch.ones(nf, dtype=torch.uint8, device=dev)
    replies = {}
    for q in (2, 3):
        rout = torch.zeros(nf * (CHUNK * (L + 24) + 64), dtype=torch.uint8, device=dev)
        s = {}
        if q == 2:
            ms = timed(lambda: s.update(fols[q].reconstruct_serve(out, fo, fg, peer, rout)), lambda: None, a)
        else:
            s.update(fols[q].reconstruct_serve(out, fo, fg, peer, rout))
        torch.cuda.synchronize()
        assert (s["reply_len"] > 0).all()
        replies[q] = (rout, s)
        if q == 2:
            results["serve"] = dict(**stats(ms), bytes=G * E * L + int(s["total"][0]) + int(r["totals"][1]))
    # one buffer with both followers' replies, in frame order
    buf = torch.cat([replies[2][0], replies[3][0]])
    off = torch.cat([replies[2][1]["reply_off"], replies[3][1]["reply_off"] + replies[2][0].numel()])
    rg = torch.cat([fg, fg])
    rp = torch.cat([torch.full((nf,), 1, dtype=torch.uint8, device=dev), torch.full((nf,), 2, dtype=torch.uint8, device=dev)])
    abs_res = {}
    one = rv["held"][:, 1:E + 1].clone()

    def reset_held():
        rv["held"][:, 1:E + 1] = one

    ms = timed(lambda: abs_res.update(eng.absorb(buf, off, rg, rp)), reset_held, a)
    torch.cuda.synchronize()
    assert int(abs_res["absorbed"].sum()) == 2 * G * E and (abs_res["verdict"] == -16).all()
    assert (rv["held"][:, 1:E + 1] == 0b1110).all()
    results["absorb"] = dict(**stats(ms), bytes=2 * G * E * (L + R16))
    pay = torch.zeros(G * E * DATA_LEN, dtype=torch.uint8, device=dev)
    ex = {}
    ms = timed(lambda: ex.update(eng.execute(pay, G * E)), lambda: ev["last_exec"].zero_(), a)
    torch.cuda.synchronize()
    assert int(ex["totals"][0]) == G * E
    got = pay.view(G, E, DATA_LEN)
    for k in range(E):
        want = torch.stack([arena[16 * k + g * DATA_LEN:16 * k + (g + 1) * DATA_LEN] for g in range(0, G, max(1, G // 64))])
        assert torch.equal(got[::max(1, G // 64), k], want), "a payload differs from its batch"
    moved = G * E * (D * L + DATA_LEN)
    results["execute"] = dict(**stats(ms), bytes=moved)
    src = torch.empty(G * E * DATA_LEN, dtype=torch.uint8, device=dev)
    ms = timed(lambda: pay.copy_(src), lambda: None, a)
    results["copy"] = dict(**stats(ms), bytes=2 * G * E * DATA_LEN)
    for k, v in results.items():
        v["tb_per_s"] = round(v["bytes"] / (v["median_ms"] * 1e-3) / 1e12, 3)
        print(f"{k:10s} {v['median_ms']:8.3f} ms  (min {v['min_ms']:.3f}, max {v['max_ms']:.3f})  {v['bytes'] / 1e9:.3f} GB  "
              f"{v['tb_per_s']:.3f} TB/s")
    print(json.dumps(dict(bench="craft_recon", card=name, power_limit=power, groups=G, entries=E, data_len=DATA_LEN, n=N, **results)))
    for f in fols.values():
        f.close()
    eng.close()


if __name__ == "__main__":
    main()
