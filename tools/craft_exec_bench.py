"""CRaft execution at n = 5 (RS(3,2)), 2^18 groups, 4 KB request batches, one committed entry per group.

  leader            ss_engine_craft_execute: the batches gathered from the data planes ss_engine_craft_propose wrote
  follower gather   ss_follower_execute, every entry holding data shards 0-2 (what a full-copy follower holds)
  follower decode   ss_follower_execute, every entry holding shards 0, 2 and 3: data shard 1 is regenerated

The follower's store is built from the leader's planes in the padded layout (held shard of rank k at
shard_addr + k * 1376), and its state installed through its views.  Timed with CUDA events: median of --steps launches
after --warmup; last_exec is rewound outside the timed window.  Bytes moved: d * L shard bytes read plus data_len
payload bytes written per entry (the algorithmic bytes), over the call's time; b.copy_(a) of as many bytes in the same
run gives the copy bandwidth the card reaches (it counts 2x its bytes).  Check: every payload equals its batch.

Usage: python tools/craft_exec_bench.py [--groups N] [--steps K] [--warmup W]
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

N, ME, DATA_LEN = 5, 0, 4096
D = N // 2 + 1
L = -(-DATA_LEN // D)
PITCH = (L + 31) & ~31


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
    ap.add_argument("--groups", type=int, default=1 << 18)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("craft_exec_bench needs a GPU")
    G = a.groups
    dev = torch.device("cuda", 0)
    ctx = Context(0)
    name, power = card()
    print(f"card: {name}, power limit {power}")
    gen = torch.Generator(device=dev).manual_seed(1)
    arena = torch.randint(0, 256, (G * DATA_LEN + 16,), dtype=torch.uint8, device=dev, generator=gen)
    batches = arena[:G * DATA_LEN].view(G, DATA_LEN)
    eng = RaftEngine(ctx, G, N, fault_tolerance=1, craft=True)
    eng.curr_term.fill_(1)
    ev = eng.exec_view()
    planes = torch.zeros((N, G * PITCH), dtype=torch.uint8, device=dev)
    o = eng.propose(ME, arena, torch.arange(G, dtype=torch.int64, device=dev) * DATA_LEN,
                    torch.full((G,), DATA_LEN, dtype=torch.int32, device=dev), planes,
                    torch.zeros(G * 4096, dtype=torch.uint8, device=dev))
    torch.cuda.synchronize()
    assert (o["slot_out"] == 1).all() and (o["shard_off"] == torch.arange(G, device=dev) * PITCH).all()
    eng.last_commit.fill_(1)                                      # every entry committed
    out = torch.zeros(G * DATA_LEN, dtype=torch.uint8, device=dev)
    moved = G * (D * L + DATA_LEN)
    results = {}

    def check(res):
        torch.cuda.synchronize()
        assert int(res["totals"][0]) == G and (res["rec_off"] == torch.arange(G, device=dev) * DATA_LEN).all()
        assert torch.equal(out.view(G, DATA_LEN), batches), "a payload differs from its batch"

    res = {}
    ms = timed(lambda: res.update(eng.execute(out, G)), lambda: ev["last_exec"].zero_(), a)
    check(res)
    results["leader"] = dict(**stats(ms), tb_per_s=round(moved / (np.median(ms) * 1e-3) / 1e12, 3))
    eng.close()

    fol = Follower(ctx, G, N, 1)
    W = fol.W
    for case, rows in (("follower_gather", (0, 1, 2)), ("follower_decode", (0, 2, 3))):
        # [G][3][PITCH]: the held shards of each entry in rank order, taken from the leader's planes
        store = planes[list(rows)].view(len(rows), G, PITCH).permute(1, 0, 2).contiguous()
        fol.start_slot.zero_()
        fol.log_end.fill_(2)
        fol.last_commit.fill_(1)
        fol.held[:, 1] = sum(1 << r for r in rows)
        fol.data_len[:, 1] = DATA_LEN
        fol.term[:, 1] = 1
        fol.shard_addr[:, 1] = store.data_ptr() + torch.arange(G, dtype=torch.int64, device=dev) * (len(rows) * PITCH)
        out.zero_()
        res = {}
        ms = timed(lambda: res.update(fol.execute(out, G)), lambda: fol.last_exec.zero_(), a)
        check(res)
        results[case] = dict(**stats(ms), tb_per_s=round(moved / (np.median(ms) * 1e-3) / 1e12, 3))
        del store
    fol.close()
    src = torch.empty(G * DATA_LEN, dtype=torch.uint8, device=dev)
    ms = timed(lambda: out.copy_(src), lambda: None, a)
    results["copy"] = dict(**stats(ms), tb_per_s=round(2 * G * DATA_LEN / (np.median(ms) * 1e-3) / 1e12, 3))
    for k, v in results.items():
        print(f"{k:16s} {v['median_ms']:8.3f} ms  (min {v['min_ms']:.3f}, max {v['max_ms']:.3f})  {v['tb_per_s']:.3f} TB/s")
    print(json.dumps(dict(bench="craft_exec", card=name, power_limit=power, groups=G, data_len=DATA_LEN, n=N, **results)))


if __name__ == "__main__":
    main()
