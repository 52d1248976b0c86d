"""ss_acceptor_recover on the WAL an acceptor writes for the cfg-4 mix (request batches of 256 B .. 64 KB,
workloads.cfg4_lengths) at 2^19 groups: a Crossword batch (n = 5, T = 5, d = 3, the cfg-4 spr assignment) and an RSPaxos
batch (n = 5, RS(3,2)).

For each protocol the leader path builds peer 0's Accept frames (tools/acceptor_bench.leader_frames); a live acceptor
takes them, a heartbeat commits every instance and ss_wal_commit_pack_dev packs the CommitSlot records.  The WAL is the
AcceptData records followed by the CommitSlot cells, each group's records in WAL order.  Then, timed with CUDA events
(median of --steps launches after --warmup):
  * ss_acceptor_recover of the whole WAL into a second acceptor, fresh for every launch: its state arrays are zeroed,
    as ss_acceptor_create leaves them, before each launch and outside the timed window.
  * b.copy_(a) of as many bytes as the replay moves, in the same run: the copy bandwidth the card reaches
Rates are algorithmic bytes: records read + store regions written (recover), 2x the bytes (copy).  Checks: every
verdict is "accepted", the store total is what the live acceptor took, and the recovered status words, ballots, held
masks, data lengths and shards equal the live acceptor's.

Usage: python tools/acceptor_recover_bench.py [--groups N] [--steps K] [--warmup W]
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
from acceptor_bench import N, leader_frames, timed  # noqa: E402

STATE = ("window_base", "bal_max_seen", "inst_bal", "accepting", "shard_addr", "held", "data_len", "assignment", "source",
         "committed", "commit_bar", "exec_bar", "preparing", "voted_bal", "voted_mask", "prep_trigger", "prep_span",
         "assign_rows", "gossip_bar")


def timed_fresh(acc, fn, a):
    """CUDA-event times of fn, each launch on an acceptor whose state is zeroed first (untimed)"""
    state = [t for t in (getattr(acc, k) for k in STATE) if t is not None]
    ms = []
    for step in range(a.warmup + a.steps):
        for t in state:
            t.zero_()
        e = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        e[0].record()
        fn()
        e[1].record()
        torch.cuda.synchronize()
        if step >= a.warmup:
            ms.append(e[0].elapsed_time(e[1]))
    return ms
from engine_ragged_bench import card, stats  # noqa: E402
from summerset_b200 import _lib  # noqa: E402
from summerset_b200 import workloads as wl  # noqa: E402
from summerset_b200.api import Context  # noqa: E402
from summerset_b200.engine import Acceptor  # noqa: E402


def run(ctx, protocol, lens, spr, arena, data_off, a):
    G = len(lens)
    dev = torch.device("cuda", 0)
    frames, off, fl, frame_bytes, d, L, policies, _ = leader_frames(ctx, protocol, lens, spr, arena, data_off)
    cw = protocol == "crossword"
    live = Acceptor(ctx, protocol, G, N, 0, d, 5)
    groups = torch.arange(G, dtype=torch.int32, device=dev)
    mask0 = np.array([bin(int(policies[(spr[g] - 1) if cw else 0][0])).count("1") for g in range(G)], dtype=np.int64)
    store_need = int((mask0 * ((L + 31) // 32 * 32)).sum())
    lstore = torch.zeros(store_need + 64, dtype=torch.uint8, device=dev)
    wal = torch.empty(frame_bytes + 16 * G + 64, dtype=torch.uint8, device=dev)
    res = live.accept(frames, off, groups, torch.full((G,), 1, dtype=torch.uint8, device=dev), lstore, wal)
    assert bool((res["verdict"] == _lib.SS_ACCEPT_VERDICT_ACCEPTED - (1 << 32)).all()) and ctx.device_status() == 0
    bal = live.bal_max_seen.clone()
    newly = live.heartbeat(groups, torch.full((G,), 1, dtype=torch.uint8, device=dev), bal, live.window_base + 64,
                           torch.zeros(G, dtype=torch.int64, device=dev))
    entries, eg, el, cnt = ctx.wal_commit_pack(newly, live.window_base, G)
    assert int(cnt[0]) == G and ctx.device_status() == 0
    # the WAL: AcceptData records where the acceptor wrote them, then the 24-byte CommitSlot cells
    wal_end = int(res["totals"][1])
    buf = torch.cat([wal[:wal_end], entries.view(-1)])
    rec_off = torch.cat([res["wal_off"], wal_end + 24 * torch.arange(G, dtype=torch.int64, device=dev)])
    rec_group = torch.cat([groups, eg])
    rec_bytes = int(res["wal_len"].to(torch.int64).sum()) + int(el.to(torch.int64).sum())
    rec = Acceptor(ctx, protocol, G, N, 0, d, 5)
    rstore = torch.zeros(store_need + 64, dtype=torch.uint8, device=dev)
    args = (buf, rec_off, rec_group, rstore)
    out = rec.recover(*args)
    ctx.device_status()
    t_rec = timed_fresh(rec, lambda: rec.recover(*args), a)
    for t in (getattr(rec, k) for k in STATE):
        if t is not None:
            t.zero_()
    out = rec.recover(*args)
    status = ctx.device_status()
    verdict = out["verdict"].cpu().numpy().view(np.uint32)
    ok = bool((verdict == _lib.SS_ACCEPT_VERDICT_ACCEPTED).all()) and status == 0 and int(out["total"][0]) == store_need
    for name in ("accepting", "committed", "preparing", "bal_max_seen", "inst_bal", "held", "data_len", "voted_bal", "voted_mask"):
        ok &= bool(torch.equal(getattr(live, name), getattr(rec, name)))
    # shards: both stores are packed in group order, so the regions and every byte (zero-filled pads included) match
    la, ra = live.shard_addr.view(G, 64)[:, 0] - lstore.data_ptr(), rec.shard_addr.view(G, 64)[:, 0] - rstore.data_ptr()
    ok &= bool(torch.equal(la, ra)) and bool(torch.equal(lstore[:store_need], rstore[:store_need]))
    moved = rec_bytes + store_need
    src = buf[:moved] if buf.numel() >= moved else torch.cat([buf, rstore])[:moved]
    dst = torch.empty_like(src)
    t_copy = timed(lambda: dst.copy_(src), a)
    gbs = lambda nbytes, ms: round(nbytes / (float(np.median(ms)) * 1e-3) / 1e9, 1)
    result = {"records": G * 2, "record_bytes": rec_bytes, "store_bytes": store_need, "all_recovered": ok,
              "recover": {**stats(t_rec), "bytes": moved, "GB/s": gbs(moved, t_rec)},
              "copy": {**stats(t_copy), "bytes": 2 * moved, "GB/s": gbs(2 * moved, t_copy)}}
    live.close()
    rec.close()
    del frames, lstore, rstore, wal, buf, src, dst
    torch.cuda.empty_cache()
    return result, ok


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--groups", type=int, default=1 << 19)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("acceptor_recover_bench needs a CUDA GPU: there is no CPU fallback")
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    name, power = card()
    print(f"card: {name}, power limit {power}", flush=True)
    G = a.groups
    lens, spr = wl.cfg4_lengths(G)
    lay = wl.ragged_layout(lens, 3)
    gen = torch.Generator(device=dev)
    gen.manual_seed(wl.SEED_BASE + 4)
    arena = torch.randint(0, 256, (lay["data_bytes"] + 64,), dtype=torch.uint8, device=dev, generator=gen)
    ctx = Context(0)
    result = {"card": name, "power_limit": power, "groups": G, "steps": a.steps}
    all_ok = True
    for protocol in ("crossword", "rspaxos"):
        r, ok = run(ctx, protocol, lens, spr, arena, lay["data_off"], a)
        all_ok &= ok
        result[protocol] = r
        for k in ("recover", "copy"):
            v = r[k]
            print(f"{protocol:9s} {k:8s} median {v['median_ms']:8.3f} ms  min {v['min_ms']:8.3f}  max {v['max_ms']:8.3f}  "
                  f"{v['bytes'] / 1e9:7.3f} GB  {v['GB/s']:8.1f} GB/s", flush=True)
    print(json.dumps(result), flush=True)
    ctx.close()
    if not all_ok:
        sys.exit("recover check failed")


if __name__ == "__main__":
    main()
