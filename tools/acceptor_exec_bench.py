"""ss_acceptor_heartbeat and ss_acceptor_execute on the cfg-4 mix (request batches of 256 B .. 64 KB,
workloads.cfg4_lengths) at 2^19 groups: Crossword n = 5, T = 5, d = 3, every instance with the balanced spr = 3 rows
(replica r holds shards r, r+1, r+2 mod 5).

For `me` = 0 (the follower holds data shards 0-2: execution only gathers), 1 (shard 0 is decoded) and 3 (shards 1 and 2
are decoded), the leader path (ss_engine_propose_ragged + ss_frame_accept_pack_ragged_dev) builds `me`'s Accept frames
once and one acceptor takes them.  Then, timed with CUDA events (median of --steps launches after --warmup; the state a
launch consumes is restored between launches, outside the timed window):
  * ss_acceptor_heartbeat: one heartbeat per group committing its instance
  * ss_acceptor_execute: every group's instance, payloads decoded from the held shards
  * b.copy_(a) of as many bytes as the payloads, in the same run: the copy bandwidth the card reaches
The execute rate counts algorithmic bytes: d*L source bytes read plus data_len payload bytes written per instance
(the copy counts 2x its bytes).  Check: every payload equals the leader's request batch, byte for byte.

Usage: python tools/acceptor_exec_bench.py [--groups N] [--steps K] [--warmup W]
Prints the card name and power limit, one line per measurement and one JSON line.  Fails without a GPU.
"""
import argparse
import ctypes as C
import json
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))
from engine_ragged_bench import card, stats  # noqa: E402
from oracle import pyoracle as oracle  # noqa: E402
from summerset_b200 import _lib  # noqa: E402
from summerset_b200 import workloads as wl  # noqa: E402
from summerset_b200._lib import check  # noqa: E402
from summerset_b200.api import Context  # noqa: E402
from summerset_b200.engine import Acceptor, LeaderEngine  # noqa: E402

N, T, D = 5, 5, 3


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


def frames_for(ctx, me, lens, arena, data_off, dev):
    """`me`'s Accept frames of one proposal per group (every group at slot 0, ballot g + 1)"""
    G = len(lens)
    eng = LeaderEngine(ctx, "crossword", G, N, 1, 1, rs_total_shards=T, rs_data_shards=D)
    bal = torch.arange(1, G + 1, dtype=torch.int64, device=dev)
    eng.set_prepared_ballots(bal)
    policies = np.array([oracle.cw_brr_assignment(N, T, 3)], dtype=np.uint32)
    eng.set_policies([list(map(int, q)) for q in policies], True)
    pol = torch.zeros(G, dtype=torch.uint8, device=dev)
    L = (lens.astype(np.int64) + D - 1) // D
    store = torch.zeros((T, int(((L + 31) // 32 * 32).sum())), dtype=torch.uint8, device=dev)
    ln = torch.from_numpy(lens.view(np.int32)).to(dev)
    slot_out, shard_off, _ = eng.propose_ragged(arena, torch.from_numpy(data_off.view(np.int64)).to(dev), ln, store, pol)
    assert ctx.device_status() == 0
    spec = _lib.FrameSpec(0, 2, D, T - D, 0, N, 1, T)
    pol_dev = torch.from_numpy(policies.view(np.int32)).to(dev)
    off = torch.empty(G, dtype=torch.int64, device=dev)
    fl = torch.empty(G, dtype=torch.int32, device=dev)
    total = torch.empty(1, dtype=torch.int64, device=dev)
    frames = torch.empty(16, dtype=torch.uint8, device=dev)

    def pack(capacity):
        check(ctx.lib.ss_frame_accept_pack_ragged_dev(ctx.h, C.byref(spec), store.data_ptr(), store.shape[1], shard_off.data_ptr(),
                                                      ln.data_ptr(), pol_dev.data_ptr(), 1, pol.data_ptr(), me, slot_out.data_ptr(),
                                                      bal.data_ptr(), G, frames.data_ptr(), capacity, off.data_ptr(), fl.data_ptr(),
                                                      total.data_ptr()))

    pack(0)
    ctx.device_status()                                  # clears the overflow bit of the sizing call
    cap = int(total)
    frames = torch.empty(cap, dtype=torch.uint8, device=dev)
    pack(cap)
    assert ctx.device_status() == 0
    eng.close()
    return frames, off, fl, bal, int(policies[0][me]), L


def run(ctx, me, lens, arena, arena_z, lay, a, dev):
    G = len(lens)
    frames, off, fl, bal, row, L = frames_for(ctx, me, lens, arena, lay["data_off"], dev)
    acc = Acceptor(ctx, "crossword", G, N, me, D, T)
    held = bin(row).count("1")
    astore = torch.empty(int(held * ((L + 31) // 32 * 32).sum()) + 64, dtype=torch.uint8, device=dev)
    wal = torch.empty(int(fl.to(torch.int64).sum()) + 16 * G + 64, dtype=torch.uint8, device=dev)
    groups = torch.arange(G, dtype=torch.int32, device=dev)
    res = acc.accept(frames, off, groups, torch.full((G,), 1, dtype=torch.uint8, device=dev), astore, wal)
    checks = {"accepted": bool((res["verdict"].cpu().numpy().view(np.uint32) == _lib.SS_ACCEPT_VERDICT_ACCEPTED).all())}
    del frames, wal, res
    torch.cuda.empty_cache()
    # heartbeat: from the leader (peer 1, or 2 when me = 1), commit_bar 1
    peer = torch.full((G,), 2 if me == 1 else 1, dtype=torch.uint8, device=dev)
    hcb = torch.ones(G, dtype=torch.int64, device=dev)
    heb = torch.zeros(G, dtype=torch.int64, device=dev)
    accepting0 = acc.accepting.clone()

    def hb_prep():
        acc.committed.zero_()
        acc.accepting.copy_(accepting0)

    t_hb = timed(lambda: acc.heartbeat(groups, peer, bal, hcb, heb), hb_prep, a)
    hb_prep()
    newly = acc.heartbeat(groups, peer, bal, hcb, heb)
    checks["committed"] = bool((newly == 1).all().item()) and ctx.device_status() == 0
    # execute
    payload_bytes = int(lay["data_bytes"])
    out = torch.empty(payload_bytes, dtype=torch.uint8, device=dev)
    rec = {}

    def ex():
        rec.update(acc.execute(out, G))

    t_ex = timed(ex, lambda: acc.commit_bar.zero_(), a)
    status = ctx.device_status()
    checks["status"] = status
    checks["totals"] = [int(x) for x in rec["totals"].cpu()] == [G, payload_bytes]
    checks["offsets"] = bool(torch.equal(rec["rec_off"], torch.from_numpy(lay["data_off"].view(np.int64)).to(dev)))
    checks["payloads"] = bool(torch.equal(out, arena_z[:payload_bytes]))
    ok = status == 0 and all(v for k, v in checks.items() if k != "status")
    exec_bytes = int((D * L).sum() + lens.astype(np.int64).sum())
    # copy bandwidth on as many bytes as the payloads, same run
    src = arena_z[:payload_bytes]
    t_copy = timed(lambda: out.copy_(src), lambda: None, a)
    gbs = lambda nbytes, ms: round(nbytes / (float(np.median(ms)) * 1e-3) / 1e9, 1)
    r = {"me": me, "decoded_data_shards": sum(1 for j in range(D) if not (row >> j) & 1), "payload_bytes": payload_bytes,
         "checked": ok, "checks": checks,
         "heartbeat": stats(t_hb),
         "execute": {**stats(t_ex), "bytes": exec_bytes, "GB/s": gbs(exec_bytes, t_ex)},
         "copy": {**stats(t_copy), "bytes": 2 * payload_bytes, "GB/s": gbs(2 * payload_bytes, t_copy)}}
    acc.close()
    del astore, out
    torch.cuda.empty_cache()
    return r, ok


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--groups", type=int, default=1 << 19)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("acceptor_exec_bench needs a CUDA GPU: there is no CPU fallback")
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    name, power = card()
    print(f"card: {name}, power limit {power}", flush=True)
    G = a.groups
    lens, _ = wl.cfg4_lengths(G)
    lens = lens.astype(np.uint32)
    lay = wl.ragged_layout(lens, D)
    gen = torch.Generator(device=dev)
    gen.manual_seed(wl.SEED_BASE + 4)
    arena = torch.randint(0, 256, (lay["data_bytes"] + 64,), dtype=torch.uint8, device=dev, generator=gen)
    # the arena with each batch's padding to 16 bytes zeroed: what execute writes
    arena_z = arena.clone()
    ends = torch.from_numpy((lay["data_off"] + lens.astype(np.uint64)).view(np.int64)).to(dev)
    pad = torch.from_numpy((-lens.astype(np.int64)) % 16).to(dev)
    k = torch.arange(16, device=dev)
    idx = (ends[:, None] + k[None, :])[k[None, :] < pad[:, None]]
    arena_z[idx] = 0
    ctx = Context(0)
    result = {"card": name, "power_limit": power, "groups": G, "steps": a.steps}
    all_ok = True
    for me in (0, 1, 3):
        r, ok = run(ctx, me, lens, arena, arena_z, lay, a, dev)
        all_ok &= ok
        result[f"me{me}"] = r
        for key in ("heartbeat", "execute", "copy"):
            v = r[key]
            extra = f"  {v['bytes'] / 1e9:7.3f} GB  {v['GB/s']:8.1f} GB/s" if "bytes" in v else ""
            print(f"me={me} ({r['decoded_data_shards']} decoded) {key:9s} median {v['median_ms']:8.3f} ms  min {v['min_ms']:8.3f}  "
                  f"max {v['max_ms']:8.3f}{extra}", flush=True)
    print(json.dumps(result), flush=True)
    ctx.close()
    if not all_ok:
        sys.exit("acceptor execute check failed")


if __name__ == "__main__":
    main()
