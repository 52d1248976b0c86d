"""ss_engine_fallback_redo: Crossword's soft fallback in every group of a 2^20-group engine (n = 5, RS(3,2), f = 2) with a
quarter, half or the whole 64-slot window Accepting.

Accepting means: window positions [0, k) of each group, k in {16, 32, 64}, hold instances proposed by ss_engine_propose
under the spr = 1 balanced policy, each a 48-byte batch (shard_len 16, one 32-byte slot per plane).  The engine keeps one
shard store (keep_slots = 1), so every position's recorded location is that store: the bytes repeat, the work does not.
One replica is dead, so min_spr = 2 and every instance is redone under the spr = 2 policy: k decided records per group
and k * T * 32 bytes of copied codeword.  Between launches, outside the timed window, policy_idx goes back to 0 and
store_used to 0.
Timed with CUDA events (median of --steps launches after --warmup), alternated with b.copy_(a) of the copied codeword
bytes alone, the bound the issue's cost asks to compare against.
Check before timing: the verdicts, the totals and a sample of decided records and copied shards.

Usage: python tools/engine_fallback_bench.py [--groups N ...] [--steps K] [--warmup W]
Prints the card name, power limit and max SM clock, one line per measurement and one JSON line.  Fails without a GPU.
"""
import argparse
import json
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))
from acceptor_exec_bench import timed  # noqa: E402
from acceptor_prepare_bench import max_sm_clock  # noqa: E402
from engine_ragged_bench import card, stats  # noqa: E402
from oracle import pyoracle as oracle  # noqa: E402
from summerset_b200.api import Context  # noqa: E402
from summerset_b200.engine import LeaderEngine  # noqa: E402

N, T, D, F = 5, 5, 3, 2
DATA_LEN = 48
PITCH = 32                                          # SS_CW_SLOT_PITCH(ceil(48 / 3))


def run(ctx, G, k, a, dev):
    eng = LeaderEngine(ctx, "crossword", G, N, F, DATA_LEN, keep_slots=1, rs_total_shards=T, rs_data_shards=D)
    eng.set_prepared_ballots(torch.full((G,), (1 << 8) | 1, dtype=torch.int64, device=dev))
    eng.set_policies([[int(x) for x in oracle.cw_brr_assignment(N, T, s)] for s in (1, 2)], True)
    payloads = torch.randint(0, 256, (G, DATA_LEN), dtype=torch.uint8, device=dev)
    pol0 = torch.zeros(G, dtype=torch.uint8, device=dev)
    for s in range(k):
        eng.propose(s, payloads, pol0)
    groups = torch.arange(G, dtype=torch.int32, device=dev)
    policy = torch.ones(G, dtype=torch.uint8, device=dev)
    alive = torch.full((G,), 0b01111, dtype=torch.int32, device=dev)
    n_rec = G * k
    store = torch.empty((T, n_rec * PITCH), dtype=torch.uint8, device=dev)
    used = torch.zeros(1, dtype=torch.int64, device=dev)
    out = {}

    def prep():
        eng.policy_idx.zero_()
        used.zero_()

    def call():
        out["res"] = eng.fallback_redo(groups, policy, store, used, n_rec, peer_alive=alive)

    prep()
    call()
    res = out["res"]
    tot = [int(x) for x in res["totals"].cpu()]
    good = tot == [n_rec, n_rec * PITCH] and bool((res["verdict"] == 0xFFFFFFF0 - (1 << 32)).all())
    idx = torch.randint(0, n_rec, (256,), device=dev)
    sl, gr, of = res["dec_slot"][idx].cpu().numpy(), res["dec_group"][idx].cpu().numpy(), res["dec_shard_off"][idx].cpu().numpy()
    for x in range(len(idx)):
        g, o = int(gr[x]), int(of[x])
        got = store[:, o:o + PITCH].cpu()
        good &= int(sl[x]) < k and bool((got[0, :16] == payloads[g, :16].cpu()).all()) and not bool(got[:, 16:].any())
        good &= bool((got[:, :16] == eng.shards[0][:, g, :16].cpu()).all())
    a_src = torch.empty(n_rec * PITCH * T, dtype=torch.uint8, device=dev)
    b_dst = torch.empty_like(a_src)
    t_call, t_copy = [], []
    for _ in range(a.rounds):
        t_call += timed(call, prep, a)
        t_copy += timed(lambda: b_dst.copy_(a_src), lambda: None, a)
    row = {"groups": G, "accepting": k, "records": n_rec, "copied_bytes": n_rec * PITCH * T, "call": stats(t_call), "copy": stats(t_copy)}
    print(f"G={G} accepting={k}: call {row['call']['median_ms']} ms, copy_ {row['copy']['median_ms']} ms, check {'ok' if good else 'FAILED'}",
          flush=True)
    eng.close()
    return row, good


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--groups", type=int, nargs="+", default=[1 << 20])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=2, help="call and copy_ alternate this many times")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("engine_fallback_bench needs a CUDA GPU: there is no CPU fallback")
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    name, power = card()
    clock = max_sm_clock()
    print(f"card: {name}, power limit {power}, max SM clock {clock}", flush=True)
    ctx = Context(0)
    rows, ok = [], True
    for G in a.groups:
        for k in (16, 32, 64):
            row, good = run(ctx, G, k, a, dev)
            rows.append(row)
            ok &= good
    print(json.dumps({"card": name, "power_limit": power, "max_sm_clock": clock, "steps": a.steps, "checked": ok, "rows": rows}),
          flush=True)
    ctx.close()
    if not ok:
        sys.exit("fallback check failed")


if __name__ == "__main__":
    main()
