"""CRaft step-down bench: ss_engine_craft_step_down for n = 5 and 2^16 groups whose leader's log holds 32 committed 4 KB
entries, deposed by one higher-term RequestVote per group, in two cases:

  reused   the engine stepped up from this replica's follower and is deposed at once: every entry is the follower's
           own, nothing is copied
  half     the engine stepped up from 16 entries and proposed 16 more in its term: those 16 are copied into the store

Each step builds a fresh engine (step-up, proposals) untimed and times the step-down alone with CUDA events.  The copied
bytes (*need) are reported as a rate next to a plain torch copy_ of the same byte count.  Prints the card name and power
limit, one line per case and one JSON line.  Fails without a GPU.
"""
import argparse
import json
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))
from engine_ragged_bench import card, stats  # noqa: E402
from summerset_b200.api import Context  # noqa: E402
from summerset_b200.engine import Follower, RaftEngine  # noqa: E402

N, ME, W, DL, ENTRIES = 5, 1, 64, 4096, 32
D = N // 2 + 1
L = -(-DL // D)
PITCH = (L + 31) & ~31


def vi(v):
    if v < 251:
        return bytes([v])
    return bytes([251]) + v.to_bytes(2, "little") if v < 1 << 16 else bytes([252]) + v.to_bytes(4, "little")


def install(fol, G, k, store):
    """k committed term-1 entries (slots 1..k) of DL bytes per group, this replica's shard held, in store"""
    dev = store.device
    fol.start_slot.zero_()
    fol.log_end.fill_(k + 1)
    fol.curr_term.fill_(1)
    fol.last_commit.fill_(k)
    fol.last_snap.zero_()
    fol.last_exec.fill_(k)
    fol.leader.fill_(0)
    fol.term.zero_()
    fol.term[:, 1:k + 1] = 1
    fol.data_len.zero_()
    fol.data_len[:, 1:k + 1] = DL
    fol.held.zero_()
    fol.held[:, 1:k + 1] = 1 << ME
    idx = torch.arange(G * k, dtype=torch.int64, device=dev).view(G, k)
    fol.shard_addr.zero_()
    fol.shard_addr[:, 1:k + 1] = store.data_ptr() + idx * PITCH


def rv_frames(G, dev):
    """RequestVote{term 3, last_slot 0, last_term 0} from replica 2 for every group"""
    body = vi(0) + vi(2) + vi(3) + vi(0) + vi(0)
    fr = len(body).to_bytes(8, "big") + body
    pad = (len(fr) + 15) & ~15
    buf = torch.zeros(G * pad, dtype=torch.uint8, device=dev)
    buf.view(G, pad)[:, :len(fr)] = torch.tensor(list(fr), dtype=torch.uint8, device=dev)
    return (buf, torch.arange(G, dtype=torch.int64, device=dev) * pad, torch.arange(G, dtype=torch.int32, device=dev),
            torch.full((G,), 2, dtype=torch.uint8, device=dev))


def one(ctx, fol, G, case, frames, fstore, planes, stride, region, arena, store):
    """a fresh leader's log, then the timed step-down: (ms, copied bytes)"""
    dev = planes.device
    k = ENTRIES if case == "reused" else ENTRIES // 2
    install(fol, G, k, fstore)
    eng = RaftEngine(ctx, G, N, craft=True, window=W)
    eng.recon_view(), eng.log_view()
    groups = torch.arange(G, dtype=torch.int32, device=dev)
    o = eng.step_up(fol, groups, torch.full((G,), 2, dtype=torch.int64, device=dev), planes[:N * stride].view(N, stride))
    assert int(o["verdict"].max()) == 0
    if case == "half":
        wal = torch.empty(G * 2 * PITCH + (1 << 20), dtype=torch.uint8, device=dev)
        offs = torch.arange(G, dtype=torch.int64, device=dev) * DL
        lens = torch.full((G,), DL, dtype=torch.int32, device=dev)
        base = k * G * PITCH
        for r in range(ENTRIES - k):
            at = base + r * region
            eng.propose(ME, arena, offs, lens, planes[at:at + N * stride].view(N, stride), wal)
        eng.last_commit.copy_(eng.log_end - 1)       # the proposals committed: a majority acknowledged them
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    res = eng.step_down(fol, *frames, store)
    b.record()
    torch.cuda.synchronize()
    v = res["verdict"].to(torch.int64) & 0xFFFFFFFF
    assert bool((v == 0xFFFFFFF3).all()), "every group deposed"
    need = int(res["need"][0])
    eng.close()
    return a.elapsed_time(b), need


def copy_ms(nbytes, dev, steps):
    src = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    dst = torch.empty_like(src)
    dst.copy_(src)
    ts = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        dst.copy_(src)
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return ts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--groups", type=int, default=1 << 16)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("craft_stepdown_bench needs a GPU")
    G = a.groups
    dev = torch.device("cuda", 0)
    ctx = Context(0)
    name, power = card()
    print(f"card: {name}, power limit {power}")
    fol = Follower(ctx, G, N, ME, window=W)
    fstore = torch.zeros(G * ENTRIES * PITCH + 64, dtype=torch.uint8, device=dev)
    fstore.view(-1)[:G * ENTRIES * PITCH].view(-1, PITCH)[:, :L] = torch.randint(0, 256, (1, L), dtype=torch.uint8, device=dev)
    region = G * PITCH                                        # one proposal round's slots in each plane
    stride = ENTRIES * G * PITCH
    planes = torch.zeros(N * stride + ENTRIES * region, dtype=torch.uint8, device=dev)
    arena = torch.randint(0, 256, (G * DL + 1,), dtype=torch.uint8, device=dev)
    store = torch.empty(G * (ENTRIES // 2) * N * PITCH + (1 << 20), dtype=torch.uint8, device=dev)
    frames = rv_frames(G, dev)
    results = {}
    for case in ("reused", "half"):
        ms, need = [], 0
        for s in range(a.warmup + a.steps):
            t, need = one(ctx, fol, G, case, frames, fstore, planes, stride, region, arena, store)
            if s >= a.warmup:
                ms.append(t)
        st = stats(ms)
        r = dict(ms=st, copied_bytes=need, copied_GBps=need / (st["median_ms"] * 1e-3) / 1e9 if need else 0.0)
        if need:
            cs = stats(copy_ms(need, dev, a.steps))
            r.update(copy_ms=cs, copy_GBps=need / (cs["median_ms"] * 1e-3) / 1e9)
        results[case] = r
        line = f"{case}: step-down {st['median_ms']:.3f} ms median, {need} bytes copied"
        if need:
            line += f" ({r['copied_GBps']:.0f} GB/s; copy_ of the same bytes {cs['median_ms']:.3f} ms, {r['copy_GBps']:.0f} GB/s)"
        print(line)
    print(json.dumps(dict(bench="craft_stepdown", card=name, power_limit=power, groups=G, n=N, entries=ENTRIES, data_len=DL,
                          **results)))


if __name__ == "__main__":
    main()
