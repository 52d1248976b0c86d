"""ss_follower_append on a CRaft workload: n = 5 (RS(3,2)), 2^18 groups, one AppendEntries frame of 4 entries per group,
4 KB request batches, one 1366-byte shard per entry (sharded mode: the follower's own shard).  Then a one-group catch-up
batch: 1023 frames of 4 entries, one after the other, for a single group with a 4096-entry window.

Every launch starts from the state at creation (log_end, curr_term and leader are reset before it, outside the timed
region), so every frame appends its 4 entries on every launch.  Timed with CUDA events: median of --steps launches
after --warmup.  Bytes moved: frames read + store regions + LogEntry records + 48-byte reply cells + 32-byte Metadata
cells, over kernel time, against the H100 SXM data-sheet HBM3 bandwidth of 3.35 TB/s.  Checks: every frame is accepted
and the WAL total is the bytes of the records.

Usage: python tools/follower_bench.py [--groups N] [--steps K] [--warmup W]
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
from engine_ragged_bench import card  # noqa: E402
from summerset_b200 import _lib  # noqa: E402
from summerset_b200.api import Context  # noqa: E402
from summerset_b200.engine import Follower  # noqa: E402

N, ME, DATA_LEN, ENTRIES = 5, 4, 4096, 4
D = N // 2 + 1
L = -(-DATA_LEN // D)
PEAK = 3350.0


def vi(v):
    if v < 251:
        return bytes([v])
    if v < 1 << 16:
        return b"\xfb" + v.to_bytes(2, "little")
    if v < 1 << 32:
        return b"\xfc" + v.to_bytes(4, "little")
    return b"\xfd" + v.to_bytes(8, "little")


def frame_template(prev):
    """AppendEntries{term 1, prev, prev_term (0 or 1), 4 entries of term 1 holding shard ME, leader_commit 0, last_snap 0};
    -> (bytes, offsets of the shard bytes)"""
    body = vi(0) + vi(0) + vi(1) + vi(prev) + vi(0 if prev == 0 else 1) + vi(ENTRIES)
    shard_at = []
    for _ in range(ENTRIES):
        body += vi(1) + bytes([D, N - D]) + vi(DATA_LEN) + vi(L) + vi(N)
        for j in range(N):
            if j == ME:
                body += b"\x01" + vi(L)
                shard_at.append(8 + len(body))
                body += bytes(L)
            else:
                body += b"\x00"
        body += b"\x00" + b"\x01" + vi(0)                         # data_copy None, external, log_offset
    body += vi(0) + vi(0)
    return len(body).to_bytes(8, "big") + body, shard_at


def build(frames, dev, gen):
    """frames: [(group, prev)] -> buf, frame_off, frame_group, frame_peer (device); shard bytes random"""
    parts, offs, at = [], [], 0
    for g, prev in frames:
        t = frame_template(prev)[0] if not parts or prev != frames[0][1] else parts[0]
        parts.append(t)
        offs.append(at)
        at += len(t) + 1                                           # frames at odd offsets
    if len({prev for _, prev in frames}) == 1:                    # one template: tile it on the device
        t, shard_at = frame_template(frames[0][1])
        F = len(t) + 1
        row = torch.zeros(F, dtype=torch.uint8)
        row[:len(t)] = torch.tensor(list(t), dtype=torch.uint8)
        buf = row.to(dev).repeat(len(frames))
        view = buf.view(len(frames), F)
        for s in shard_at:
            view[:, s:s + L] = torch.randint(0, 256, (len(frames), L), dtype=torch.uint8, device=dev, generator=gen)
    else:
        host = bytearray()
        for (g, prev), p in zip(frames, parts):
            host += p + b"\x00"
        buf = torch.tensor(np.frombuffer(bytes(host), dtype=np.uint8), device=dev)
    n = len(frames)
    return (buf, torch.tensor(offs, dtype=torch.int64, device=dev), torch.tensor([g for g, _ in frames], dtype=torch.int32, device=dev),
            torch.zeros(n, dtype=torch.uint8, device=dev))


def measure(ctx, name, G, window, frames, a):
    dev = "cuda:0"
    gen = torch.Generator(device=dev)
    gen.manual_seed(1)
    fol = Follower(ctx, G, N, ME, window)
    buf, off, grp, peer = build(frames, dev, gen)
    n = len(frames)
    rec_slot = ((len(vi(1)) + 2 + len(vi(DATA_LEN)) + len(vi(L)) + 1 + N + len(vi(L)) + L + 1 + 1) + 8 + 1 + 1 + 15) & ~15
    store_need = n * ENTRIES * ((L + 31) & ~31)
    wal_need = n * ENTRIES * rec_slot
    store = torch.empty(store_need, dtype=torch.uint8, device=dev)
    wal = torch.empty(wal_need, dtype=torch.uint8, device=dev)
    ms = []
    out = None
    for step in range(a.warmup + a.steps):
        fol.log_end.fill_(1)
        fol.curr_term.fill_(0)
        fol.leader.fill_(0xFF)
        fol.last_commit.fill_(0)
        e = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        e[0].record()
        out = fol.append(buf, off, grp, peer, store, wal)
        e[1].record()
        torch.cuda.synchronize()
        if step >= a.warmup:
            ms.append(e[0].elapsed_time(e[1]))
    v = out["verdict"].cpu().numpy().view(np.uint32)
    assert (v == _lib.SS_FOLLOWER_VERDICT_ACCEPTED).all(), "every frame must append"
    wal_bytes = int(out["wal_len"].sum())
    assert int(out["totals"][1]) == wal_bytes == wal_need, (int(out["totals"][1]), wal_bytes, wal_need)
    moved = buf.numel() + store_need + wal_bytes + 48 * n + 32 * int((out["meta_len"] > 0).sum())
    med = float(np.median(ms))
    r = {"frames": n, "entries": n * ENTRIES, "ms": med, "frames_per_s": n / med * 1e3, "entries_per_s": n * ENTRIES / med * 1e3,
         "bytes_moved": moved, "GBps": moved / med / 1e6, "frac_of_3350": moved / med / 1e6 / PEAK}
    print(f"{name}: {n} frames, {med:.3f} ms, {r['frames_per_s']:.3g} frames/s, {r['entries_per_s']:.3g} entries/s, "
          f"{r['GBps']:.0f} GB/s ({100 * r['frac_of_3350']:.0f} % of 3.35 TB/s)", flush=True)
    fol.close()
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--groups", type=int, default=1 << 18)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("follower_bench needs a GPU")
    torch.cuda.set_device(0)
    name, power = card()
    print(f"card: {name}, power limit {power}", flush=True)
    ctx = Context(0)
    result = {"card": name, "power_limit": power, "steps": a.steps,
              "workload": f"CRaft n={N}, one frame of {ENTRIES} entries per group, {DATA_LEN} B batches, one {L}-byte shard per entry"}
    result["many_groups"] = measure(ctx, "many groups", a.groups, 64, [(g, 0) for g in range(a.groups)], a)
    result["catch_up"] = measure(ctx, "one-group catch-up", 1, 4096, [(0, ENTRIES * f) for f in range(1023)], a)
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
