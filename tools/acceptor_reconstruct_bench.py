"""ss_acceptor_reconstruct_serve and ss_acceptor_absorb on the cfg-4 mix (request batches of 256 B .. 64 KB,
workloads.cfg4_lengths) at 2^19 groups: RSPaxos n = 5, d = 3, where every follower holds one shard and execution is
postponed until a reconstruct read brings two more.

The leader path (ss_engine_propose_ragged + ss_frame_accept_pack_ragged_dev) builds the Accept frames of replicas 1, 2
and 3 once; three acceptors take them and commit.  Replica 1 then asks replicas 2 and 3 for every group's instance
(one Reconstruct{slots: [0]} frame per group and peer).  Timed with CUDA events (median of --steps launches after
--warmup; the state a launch consumes is restored between launches, outside the timed window):
  * ss_acceptor_reconstruct_serve at replica 2: one frame per group
  * ss_acceptor_absorb at replica 1: both peers' replies, 2 frames per group
  * b.copy_(a) of as many bytes as each call moves, in the same run: the copy bandwidth the card reaches
Algorithmic bytes: serve = shards read + reply bytes written; absorb = reply bytes read + old shards read + new regions
written (the copy counts 2x its bytes).  Check: after the absorb, ss_acceptor_execute delivers every request batch byte
for byte.

Usage: python tools/acceptor_reconstruct_bench.py [--groups N] [--steps K] [--warmup W]
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
from acceptor_exec_bench import timed  # noqa: E402
from engine_ragged_bench import card, stats  # noqa: E402
from summerset_b200 import _lib  # noqa: E402
from summerset_b200 import workloads as wl  # noqa: E402
from summerset_b200._lib import check  # noqa: E402
from summerset_b200.api import Context  # noqa: E402
from summerset_b200.engine import Acceptor, LeaderEngine  # noqa: E402

N, D = 5, 3
ME, PEERS = 1, (2, 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--groups", type=int, default=1 << 19)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("acceptor_reconstruct_bench needs a CUDA GPU: there is no CPU fallback")
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    name, power = card()
    print(f"card: {name}, power limit {power}", flush=True)
    G = a.groups
    lens, _ = wl.cfg4_lengths(G)
    lens = lens.astype(np.uint32)
    lay = wl.ragged_layout(lens, D)
    gen = torch.Generator(device=dev)
    gen.manual_seed(wl.SEED_BASE + 5)
    arena = torch.randint(0, 256, (lay["data_bytes"] + 64,), dtype=torch.uint8, device=dev, generator=gen)
    arena_z = arena.clone()                               # each batch's padding to 16 bytes zeroed: what execute writes
    ends = torch.from_numpy((lay["data_off"] + lens.astype(np.uint64)).view(np.int64)).to(dev)
    pad = torch.from_numpy((-lens.astype(np.int64)) % 16).to(dev)
    k = torch.arange(16, device=dev)
    arena_z[(ends[:, None] + k[None, :])[k[None, :] < pad[:, None]]] = 0
    ctx = Context(0)
    # the leader's proposal and the Accept frames of replicas 1-3
    eng = LeaderEngine(ctx, "rspaxos", G, N, 1, 1)
    bal = torch.arange(1, G + 1, dtype=torch.int64, device=dev)
    eng.set_prepared_ballots(bal)
    L = (lens.astype(np.int64) + D - 1) // D
    pitch = (L + 31) // 32 * 32
    store = torch.zeros((N, int(pitch.sum())), dtype=torch.uint8, device=dev)
    ln = torch.from_numpy(lens.view(np.int32)).to(dev)
    slot_out, shard_off, _ = eng.propose_ragged(arena, torch.from_numpy(lay["data_off"].view(np.int64)).to(dev), ln, store, None)
    assert ctx.device_status() == 0
    spec = _lib.FrameSpec(0, 2, D, N - D, 0, N, 0, 0)
    policies = torch.tensor([[1 << r for r in range(N)]], dtype=torch.int32, device=dev)
    pol = torch.zeros(G, dtype=torch.uint8, device=dev)
    groups = torch.arange(G, dtype=torch.int32, device=dev)
    accs, keep = {}, []
    for r in (ME,) + PEERS:
        off = torch.empty(G, dtype=torch.int64, device=dev)
        fl = torch.empty(G, dtype=torch.int32, device=dev)
        total = torch.empty(1, dtype=torch.int64, device=dev)
        cap = int(G * 64 + (pitch + 64).sum())
        frames = torch.empty(cap, dtype=torch.uint8, device=dev)
        check(ctx.lib.ss_frame_accept_pack_ragged_dev(ctx.h, C.byref(spec), store.data_ptr(), store.shape[1], shard_off.data_ptr(),
                                                      ln.data_ptr(), policies.data_ptr(), 1, pol.data_ptr(), r, slot_out.data_ptr(),
                                                      bal.data_ptr(), G, frames.data_ptr(), cap, off.data_ptr(), fl.data_ptr(),
                                                      total.data_ptr()))
        assert ctx.device_status() == 0
        acc = accs[r] = Acceptor(ctx, "rspaxos", G, N, r, D, N)
        astore = torch.empty(int(pitch.sum()) + 64, dtype=torch.uint8, device=dev)
        wal = torch.empty(int(fl.to(torch.int64).sum()) + 16 * G + 64, dtype=torch.uint8, device=dev)
        res = acc.accept(frames, off, groups, torch.zeros(G, dtype=torch.uint8, device=dev), astore, wal)
        assert (res["verdict"].cpu().numpy().view(np.uint32) == _lib.SS_ACCEPT_VERDICT_ACCEPTED).all()
        acc.heartbeat(groups, torch.zeros(G, dtype=torch.uint8, device=dev), bal, torch.ones(G, dtype=torch.int64, device=dev),
                      torch.zeros(G, dtype=torch.int64, device=dev))
        keep.append(astore)
        del frames, wal, res
    eng.close()
    del store
    torch.cuda.empty_cache()
    # Reconstruct{slots: [0]} per group: 8-byte length 4, Msg, variant 4, one slot, slot 0
    req = torch.tensor([0, 0, 0, 0, 0, 0, 0, 4, 0, 4, 1, 0], dtype=torch.uint8, device=dev).repeat(G)
    req_off = torch.arange(G, dtype=torch.int64, device=dev) * 12
    peer_me = torch.full((G,), ME, dtype=torch.uint8, device=dev)
    reply_cap = int(G * 48 + (L + 16).sum()) // 16 * 16 + 16 * G
    replies = {q: torch.empty(reply_cap, dtype=torch.uint8, device=dev) for q in PEERS}
    served = {}
    for q in PEERS:
        served[q] = accs[q].reconstruct_serve(req, req_off, groups, peer_me, replies[q])
    res_serve = {}
    t_serve = timed(lambda: res_serve.update(accs[PEERS[0]].reconstruct_serve(req, req_off, groups, peer_me, replies[PEERS[0]])),
                    lambda: None, a)
    checks = {"served": all(bool((s["verdict"].cpu().numpy().view(np.uint32) == _lib.SS_ACCEPT_VERDICT_ACCEPTED).all()) for s in served.values())}
    reply_bytes = int(served[PEERS[0]]["reply_len"].sum())
    serve_bytes = int(L.sum()) + reply_bytes
    # both replies into one receive buffer, frames interleaved per group
    used = int(served[PEERS[0]]["total"].item())
    buf = torch.cat([replies[q][:used] for q in PEERS])
    foff = torch.stack([served[q]["reply_off"] + i * used for i, q in enumerate(PEERS)], dim=1).reshape(-1).contiguous()
    fgrp = groups.repeat_interleave(2)
    fpeer = torch.tensor(PEERS, dtype=torch.uint8, device=dev).repeat(G)
    del replies
    fol = accs[ME]
    held0, addr0 = fol.held.clone(), fol.shard_addr.clone()
    fstore = torch.empty(int(3 * pitch.sum()) + 64, dtype=torch.uint8, device=dev)
    res_abs = {}

    def restore():
        fol.held.copy_(held0)
        fol.shard_addr.copy_(addr0)

    t_abs = timed(lambda: res_abs.update(fol.absorb(buf, foff, fgrp, fpeer, fstore)), restore, a)
    checks["absorbed"] = bool((res_abs["absorbed"] == 1).all().item()) and int(res_abs["total"].item()) == int(3 * pitch.sum())
    absorb_bytes = 2 * reply_bytes + int(pitch.sum()) + int(3 * pitch.sum())
    status = ctx.device_status()
    out = torch.empty(lay["data_bytes"], dtype=torch.uint8, device=dev)
    ex = fol.execute(out, G)
    checks["executed"] = int(ex["totals"][0].item()) == G
    checks["payloads"] = bool(torch.equal(out, arena_z[:lay["data_bytes"]]))
    status |= ctx.device_status()
    ok = status == 0 and all(checks.values())
    gbs = lambda nbytes, ms: round(nbytes / (float(np.median(ms)) * 1e-3) / 1e9, 1)
    res = {"card": name, "power_limit": power, "groups": G, "steps": a.steps, "checked": ok, "checks": checks, "status": status}
    for key, t, nbytes in (("serve", t_serve, serve_bytes), ("absorb", t_abs, absorb_bytes)):
        src = torch.empty(nbytes // 2, dtype=torch.uint8, device=dev)
        dst = torch.empty_like(src)
        t_copy = timed(lambda: dst.copy_(src), lambda: None, a)
        res[key] = {**stats(t), "bytes": nbytes, "GB/s": gbs(nbytes, t)}
        res[key + "_copy"] = {**stats(t_copy), "bytes": 2 * (nbytes // 2), "GB/s": gbs(2 * (nbytes // 2), t_copy)}
        for k2 in (key, key + "_copy"):
            v = res[k2]
            print(f"{k2:12s} median {v['median_ms']:8.3f} ms  min {v['min_ms']:8.3f}  max {v['max_ms']:8.3f}  {v['bytes'] / 1e9:7.3f} GB  "
                  f"{v['GB/s']:8.1f} GB/s", flush=True)
        del src, dst
    print(json.dumps(res), flush=True)
    for acc in accs.values():
        acc.close()
    ctx.close()
    if not ok:
        sys.exit("acceptor reconstruct check failed")


if __name__ == "__main__":
    main()
