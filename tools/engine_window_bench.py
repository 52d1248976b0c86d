"""Steady-state Paxos-family leader loop with a sliding instance window, on one GPU: 2^20 RSPaxos groups, n = 5, f = 1
(RS(3,2) shards), 4096-byte request batches.  Every step is

    propose_next (encode + first-Null bookkeeping) -> ingest of a seeded AcceptReply batch -> tick -> advance (NULL)

The reply batch acks the new instance from four of the five replicas (the commit threshold), so every step commits and
retires one slot per group; the run covers more than 64 slots per group, so every window position is reused.  Each call
is timed with CUDA events and reported with the bytes the algorithm has to move and the rate that implies.  The tick is
also timed alone: on an engine whose window never moved (it skips the window_base load), and at all-zero and at spread
window bases.

Usage: python tools/engine_window_bench.py [--groups N] [--steps K] [--warmup W]
Prints the card name and power limit, one line per call and one JSON line.  Fails without a GPU.
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from summerset_b200 import workloads as wl  # noqa: E402
from summerset_b200.api import Context  # noqa: E402
from summerset_b200.engine import LeaderEngine  # noqa: E402

N, F, DATA_LEN = 5, 1, 4096
ACKS = 4                      # majority + fault_tolerance


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def algorithmic_bytes(G, R, ds, T, n_rec):
    """bytes each call has to read and write, from the shapes (8-byte words unless noted)"""
    return {
        # payload read, T shard planes written; window_base, accepting, committed, bal_prepared read; accepting,
        # committed, inst_bal, slot_out written; every ack plane read and written
        "propose_next": G * DATA_LEN + T * G * ds + G * (4 * 8 + 4 * 8 + R * 16),
        # records (group u32, slot u8, peer u8, ballot u64); per group bal_prepared, window_base, accepting, inst_bal
        # read and every ack plane read and written
        "ingest": n_rec * 14 + G * (4 * 8 + R * 16),
        # ack planes and window_base read; accepting and committed read and written; commit_bar (u32) and newly written
        "tick": G * (R * 8 + 8 + 4 * 8 + 4 + 8),
        # window_base, committed, accepting, every ack plane read and written; commit_bar written
        "advance": G * (3 * 16 + R * 16 + 4),
    }


def time_calls(calls, steps):
    """runs the calls in order `steps` times with an event between each; mean ms per call"""
    ev = [[torch.cuda.Event(enable_timing=True) for _ in range(len(calls) + 1)] for _ in range(steps)]
    for s in range(steps):
        ev[s][0].record()
        for i, (_, fn) in enumerate(calls):
            fn()
            ev[s][i + 1].record()
    torch.cuda.synchronize()
    return {name: sum(ev[s][i].elapsed_time(ev[s][i + 1]) for s in range(steps)) / steps for i, (name, _) in enumerate(calls)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--groups", type=int, default=1 << 20)
    ap.add_argument("--steps", type=int, default=80)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("engine_window_bench needs a CUDA GPU: there is no CPU fallback")
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    name, power = card()
    print(f"card: {name}, power limit {power}", flush=True)
    G = a.groups
    ctx = Context(0)
    eng = LeaderEngine(ctx, "rspaxos", G, N, F, DATA_LEN)
    bal = torch.arange(1, G + 1, dtype=torch.int64, device=dev)
    eng.set_prepared_ballots(bal)
    payload = torch.from_numpy(wl.payload_uniform(G, DATA_LEN, seed_extra=77)).to(dev)
    # seeded reply batch: every group's newest instance (window position 0 after each advance) is acked by ACKS
    # distinct replicas, records in a seeded random order
    rng = np.random.default_rng(2024)
    perm = torch.from_numpy(rng.permutation(G * ACKS)).to(dev)
    peers = torch.from_numpy(np.argsort(rng.random((G, N)), axis=1)[:, :ACKS].reshape(-1).astype(np.uint8)).to(dev)
    rec_group = torch.arange(G, dtype=torch.int32, device=dev).repeat_interleave(ACKS)[perm].contiguous()
    rec_peer = peers[perm].contiguous()
    rec_slot = torch.zeros(G * ACKS, dtype=torch.uint8, device=dev)
    rec_ballot = bal.repeat_interleave(ACKS)[perm].contiguous()
    newly = torch.empty(G, dtype=torch.int64, device=dev)
    calls = [("propose_next", lambda: eng.propose_next(0, payload)),
             ("ingest", lambda: eng.on_accept_replies(rec_group, rec_slot, rec_peer, rec_ballot)),
             ("tick", lambda: eng.tick(newly)),
             ("advance", lambda: eng.advance())]
    time_calls(calls, a.warmup)
    ms = time_calls(calls, a.steps)
    # every step committed and retired exactly one slot per group
    total = a.warmup + a.steps
    assert (eng.window_base == total).all().item() and (eng.commit_bar == 0).all().item() and total > 64
    assert ctx.device_status() == 0
    nbytes = algorithmic_bytes(G, N, eng.ds, eng.T, G * ACKS)
    result = {"card": name, "power_limit": power, "groups": G, "steps": a.steps, "slots_per_group": total, "calls": {}}
    for k, v in ms.items():
        gbs = nbytes[k] / (v * 1e-3) / 1e9
        result["calls"][k] = {"ms": round(v, 4), "bytes": nbytes[k], "GB/s": round(gbs, 1)}
        print(f"{k:14s} {v:9.4f} ms  {nbytes[k] / 1e6:10.1f} MB  {gbs:8.1f} GB/s", flush=True)
    # the tick alone: an engine whose window never moved (all bases 0, the tick skips the base load), and this engine
    # at all-zero and at spread bases (the base-aware tick)
    fresh = LeaderEngine(ctx, "multipaxos", G, N)
    spread = torch.from_numpy(rng.integers(0, 1 << 40, G).astype(np.int64)).to(dev)
    tick_ms = {}
    for label, e, base in (("unmoved", fresh, None), ("zero", eng, torch.zeros(G, dtype=torch.int64, device=dev)),
                           ("spread", eng, spread)):
        if base is not None:
            e.window_base.copy_(base)
        tick = [("tick", lambda: e.tick(newly))]
        time_calls(tick, 10)
        tick_ms[label] = min(time_calls(tick, 100)["tick"] for _ in range(3))
        b = nbytes["tick"] - (G * 8 if base is None else 0)
        print(f"tick, {label:7s} bases {tick_ms[label]:9.4f} ms  {b / (tick_ms[label] * 1e-3) / 1e9:8.1f} GB/s", flush=True)
    fresh.close()
    result["tick_bases_ms"] = {k: round(v, 4) for k, v in tick_ms.items()}
    print(json.dumps(result), flush=True)
    eng.close()
    ctx.close()


if __name__ == "__main__":
    main()
