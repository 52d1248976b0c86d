"""ss_acceptor_accept on the frames for peer 0 of the cfg-4 mix (request batches of 256 B .. 64 KB, workloads.cfg4_lengths)
at 2^19 groups: a Crossword batch (n = 5, T = 5, d = 3, the cfg-4 spr assignment) and an RSPaxos batch (n = 5, RS(3,2)).

For each protocol the leader path (ss_engine_propose_ragged + ss_frame_accept_pack_ragged_dev) builds the frames once;
then, timed with CUDA events (median of --steps launches after --warmup):
  * ss_acceptor_accept of the whole batch into one acceptor (every frame is accepted on every launch: same slots,
    ballots equal to bal_max_seen)
  * ss_frame_accept_pack_ragged_dev on the same batch (the leader-side packer)
  * b.copy_(a) of as many bytes as the frames, in the same run: the copy bandwidth the card reaches
Rates are algorithmic bytes: frames read + store regions + WAL records written + 48-byte reply cells (acceptor), frames
written (packer), 2x the bytes (copy).  Checks: every verdict is "accepted" and the store / WAL totals are what the
frames ask for.

Usage: python tools/acceptor_bench.py [--groups N] [--steps K] [--warmup W]
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

N = 5


def timed(fn, a):
    ms = []
    for step in range(a.warmup + a.steps):
        e = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        e[0].record()
        fn()
        e[1].record()
        torch.cuda.synchronize()
        if step >= a.warmup:
            ms.append(e[0].elapsed_time(e[1]))
    return ms


def leader_frames(ctx, protocol, lens, spr, arena, data_off):
    """the frames for peer 0 that the leader path builds -> (frames, frame_off, frame_len, frame_bytes, d, L, policies,
    repack: a callable that packs them again)"""
    G = len(lens)
    dev = torch.device("cuda", 0)
    cw = protocol == "crossword"
    eng = LeaderEngine(ctx, protocol, G, N, 1, 1, **(dict(rs_total_shards=5, rs_data_shards=3) if cw else {}))
    bal = torch.arange(1, G + 1, dtype=torch.int64, device=dev)
    eng.set_prepared_ballots(bal)
    policies = np.array([[1 << r for r in range(N)]], dtype=np.uint32)
    pol = None
    if cw:
        policies = np.stack([oracle.cw_brr_assignment(N, 5, s) for s in (1, 2, 3)]).astype(np.uint32)
        eng.set_policies([list(map(int, q)) for q in policies], True)
        pol = torch.from_numpy((spr - 1).astype(np.uint8)).to(dev)
    d, p = eng.d, eng.T - eng.d
    L = (lens.astype(np.int64) + d - 1) // d
    store = torch.zeros((eng.T, int(((L + 31) // 32 * 32).sum())), dtype=torch.uint8, device=dev)
    ln = torch.from_numpy(lens.view(np.int32)).to(dev)
    slot_out, shard_off, _ = eng.propose_ragged(arena, torch.from_numpy(data_off.view(np.int64)).to(dev), ln, store, pol)
    assert ctx.device_status() == 0
    spec = _lib.FrameSpec(0, 2, d, p, 0, N, 1 if cw else 0, 5)
    pol_dev = torch.from_numpy(policies.view(np.int32)).to(dev)
    off = torch.empty(G, dtype=torch.int64, device=dev)
    fl = torch.empty(G, dtype=torch.int32, device=dev)
    total = torch.empty(1, dtype=torch.int64, device=dev)
    frames = torch.empty(16, dtype=torch.uint8, device=dev)

    def pack(capacity):
        check(ctx.lib.ss_frame_accept_pack_ragged_dev(ctx.h, C.byref(spec), store.data_ptr(), store.shape[1], shard_off.data_ptr(),
                                                      ln.data_ptr(), pol_dev.data_ptr(), policies.shape[0],
                                                      pol.data_ptr() if pol is not None else None, 0, slot_out.data_ptr(),
                                                      bal.data_ptr(), G, frames.data_ptr(), capacity, off.data_ptr(),
                                                      fl.data_ptr(), total.data_ptr()))

    pack(0)
    ctx.device_status()                                  # clears the overflow bit of the sizing call
    cap = int(total)
    frames = torch.empty(cap, dtype=torch.uint8, device=dev)
    pack(cap)
    assert ctx.device_status() == 0
    frame_bytes = int(fl.to(torch.int64).sum())
    return frames, off, fl, frame_bytes, d, L, policies, lambda: pack(cap)


def run(ctx, protocol, lens, spr, arena, data_off, a):
    G = len(lens)
    dev = torch.device("cuda", 0)
    cw = protocol == "crossword"
    frames, off, fl, frame_bytes, d, L, policies, repack = leader_frames(ctx, protocol, lens, spr, arena, data_off)
    t_pack = timed(repack, a)
    # the acceptor: peer 0's frames where the packer left them (16-byte regions; the shards inside are at any offset)
    acc = Acceptor(ctx, protocol, G, N, 0, d, 5)
    groups = torch.arange(G, dtype=torch.int32, device=dev)
    peers = torch.full((G,), 1, dtype=torch.uint8, device=dev)
    mask0 = np.array([bin(int(policies[(spr[g] - 1) if cw else 0][0])).count("1") for g in range(G)], dtype=np.int64)
    store_need = int((mask0 * ((L + 31) // 32 * 32)).sum())
    astore = torch.empty(store_need + 64, dtype=torch.uint8, device=dev)
    wal = torch.empty(frame_bytes + 16 * G + 64, dtype=torch.uint8, device=dev)
    res = acc.accept(frames, off, groups, peers, astore, wal)
    ctx.device_status()
    args = (frames, off, groups, peers, astore, wal)
    t_acc = timed(lambda: acc.accept(*args), a)
    res = acc.accept(*args)
    status = ctx.device_status()
    verdict = res["verdict"].cpu().numpy().view(np.uint32)
    wal_bytes = int(res["wal_len"].to(torch.int64).sum())
    totals = res["totals"].cpu().numpy()
    ok = bool((verdict == _lib.SS_ACCEPT_VERDICT_ACCEPTED).all()) and status == 0 and int(totals[0]) == store_need
    acc_bytes = frame_bytes + store_need + wal_bytes + 48 * G
    # copy bandwidth on as many bytes as the frames, same run
    src = frames[:frame_bytes]
    dst = torch.empty_like(src)
    t_copy = timed(lambda: dst.copy_(src), a)
    gbs = lambda nbytes, ms: round(nbytes / (float(np.median(ms)) * 1e-3) / 1e9, 1)
    out = {"frames_bytes": frame_bytes, "store_bytes": store_need, "wal_bytes": wal_bytes, "all_accepted": ok,
           "accept": {**stats(t_acc), "bytes": acc_bytes, "GB/s": gbs(acc_bytes, t_acc)},
           "frame_pack": {**stats(t_pack), "bytes": frame_bytes, "GB/s": gbs(frame_bytes, t_pack)},
           "copy": {**stats(t_copy), "bytes": 2 * frame_bytes, "GB/s": gbs(2 * frame_bytes, t_copy)}}
    acc.close()
    del repack, frames, astore, wal, src, dst
    torch.cuda.empty_cache()
    return out, ok


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--groups", type=int, default=1 << 19)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("acceptor_bench needs a CUDA GPU: there is no CPU fallback")
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
        for k in ("accept", "frame_pack", "copy"):
            v = r[k]
            print(f"{protocol:9s} {k:10s} median {v['median_ms']:8.3f} ms  min {v['min_ms']:8.3f}  max {v['max_ms']:8.3f}  "
                  f"{v['bytes'] / 1e9:7.3f} GB  {v['GB/s']:8.1f} GB/s", flush=True)
    print(json.dumps(result), flush=True)
    ctx.close()
    if not all_ok:
        sys.exit("acceptor check failed")


if __name__ == "__main__":
    main()
