"""The CRaft leader's log on a CRaft workload: n = 5 (RS(3,2)), 4 KB request batches, msg_chunk_size 10.

  propose + pack   2^18 groups: ss_engine_craft_propose codes one batch per group into the log (five 1366-byte shards and
                   the leader's LogEntry record), then ss_frame_append_pack_dev packs one AppendEntries frame per (peer,
                   group) carrying that peer's shard.  Each launch pair starts from a fresh log position: log_end and
                   try_next are rewound outside the timed region.
  catch-up         256 groups with a 4096-entry window hold 4000 entries each; one peer is 4000 entries behind, so each
                   group sends it 400 frames of 10 entries.  try_next is rewound outside the timed region.

Timed with CUDA events: median of --steps launches after --warmup; the propose + pack case also reports the two
calls' shares.  Bytes moved: batches read + shards written + records
written for the propose, shards read + frames written for the pack, over kernel time.

Usage: python tools/craft_leader_bench.py [--groups N] [--steps K] [--warmup W]
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
from summerset_b200.engine import RaftEngine  # noqa: E402

N, ME, DATA_LEN, CHUNK = 5, 0, 4096, 10
D = N // 2 + 1
L = -(-DATA_LEN // D)
PITCH = (L + 31) & ~31


def timed(fn, a):
    """-> (median ms of the whole run, median ms up to the event run() records in between, run()'s result)"""
    ms, first = [], []
    for step in range(a.warmup + a.steps):
        reset, run = fn()
        reset()
        e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        e[0].record()
        out = run(e[1])
        e[2].record()
        torch.cuda.synchronize()
        if step >= a.warmup:
            ms.append(e[0].elapsed_time(e[2]))
            first.append(e[0].elapsed_time(e[1]))
    return float(np.median(ms)), float(np.median(first)), out


def propose_pack(ctx, G, a):
    dev = "cuda:0"
    eng = RaftEngine(ctx, G, N, craft=True)
    eng.curr_term.fill_(1)
    view = eng.log_view()
    arena = torch.randint(0, 256, (G * DATA_LEN,), dtype=torch.uint8, device=dev)
    off = torch.arange(G, dtype=torch.int64, device=dev) * DATA_LEN
    dl = torch.full((G,), DATA_LEN, dtype=torch.int32, device=dev)
    store = torch.empty((N, G * PITCH), dtype=torch.uint8, device=dev)
    wal = torch.empty(G * 2048, dtype=torch.uint8, device=dev)
    P = N - 1
    out = torch.empty(P * G * 1424, dtype=torch.uint8, device=dev)
    res = {}

    def fn():
        def reset():
            eng.log_end.fill_(1)
            eng.next_slot.fill_(1)
            view["try_next"].fill_(0)

        def run(mid):
            res["p"] = eng.propose(ME, arena, off, dl, store, wal)
            mid.record()
            res["k"] = eng.pack_append(ME, out, P * G, msg_chunk_size=CHUNK)
            return res
        return reset, run

    med, med_p, r = timed(fn, a)
    nf, total = int(r["k"]["n_frames"][0]), int(r["k"]["total"][0])
    assert nf == P * G and (r["k"]["pair_status"] == _lib.SS_APPEND_PAIR_SENT).all()
    assert (r["p"]["slot_out"] == 1).all()
    wal_bytes = int(r["p"]["wal_len"].sum())
    frame_bytes = int(r["k"]["frame_len"][:nf].sum())
    moved = G * DATA_LEN + N * G * PITCH + wal_bytes + P * G * L + frame_bytes
    eng.close()
    return med, moved, {"groups": G, "frames": nf, "frame_bytes": frame_bytes, "region_bytes": total, "propose_ms": round(med_p, 4),
                        "pack_ms": round(med - med_p, 4)}


def catch_up(ctx, G, a):
    dev = "cuda:0"
    ENT, W = 4000, 4096
    eng = RaftEngine(ctx, G, N, craft=True, window=W)
    eng.curr_term.fill_(1)
    view = eng.log_view()
    arena = torch.randint(0, 256, (G * DATA_LEN,), dtype=torch.uint8, device=dev)
    off = torch.arange(G, dtype=torch.int64, device=dev) * DATA_LEN
    dl = torch.full((G,), DATA_LEN, dtype=torch.int32, device=dev)
    store = torch.empty((N, ENT * G * PITCH), dtype=torch.uint8, device=dev)
    wal = torch.empty(G * 2048, dtype=torch.uint8, device=dev)
    # the log: 4000 entries per group, each proposal into its own stretch of one store
    so, slot, wo, wl = (torch.empty(G, dtype=torch.int64, device=dev) for _ in range(4))
    for k in range(ENT):
        _lib.check(eng.lib.ss_engine_craft_propose(eng.h, ME, arena.data_ptr(), off.data_ptr(), dl.data_ptr(),
                                                   store.data_ptr() + k * G * PITCH, ENT * G * PITCH, so.data_ptr(), slot.data_ptr(),
                                                   None, None, wal.data_ptr(), wal.numel(), wo.data_ptr(), wl.data_ptr(), 0))
    torch.cuda.synchronize()
    assert (eng.log_end == ENT + 1).all()
    P = N - 1
    frames = ENT // CHUNK
    out = torch.empty(G * frames * (CHUNK * 1400 + 64) + P * G * 64, dtype=torch.uint8, device=dev)
    ns = torch.full((P, G), ENT + 1, dtype=torch.int32, device=dev)
    ns[0].fill_(1)                                                # peer 0 is 4000 entries behind

    def fn():
        def reset():
            eng.next_slot.copy_(ns)
            view["try_next"].fill_(0)

        def run(mid):
            mid.record()
            return eng.pack_append(ME, out, G * frames + 16, msg_chunk_size=CHUNK)
        return reset, run

    med, _, r = timed(fn, a)
    nf = int(r["n_frames"][0])
    assert nf == G * frames, nf
    frame_bytes = int(r["frame_len"][:nf].sum())
    moved = G * ENT * L + frame_bytes
    eng.close()
    return med, moved, {"groups": G, "entries_behind": ENT, "frames": nf, "frame_bytes": frame_bytes}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--groups", type=int, default=1 << 18)
    ap.add_argument("--catchup-groups", type=int, default=256)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("craft_leader_bench needs a GPU")
    torch.cuda.set_device(0)
    name, power = card()
    print(f"card: {name}, power limit {power}", flush=True)
    ctx = Context(0)
    result = {"card": name, "power_limit": power, "steps": a.steps,
              "workload": f"CRaft n={N}, {DATA_LEN} B batches, msg_chunk_size {CHUNK}, one {L}-byte shard per entry and peer"}
    for key, f, G in (("propose_pack", propose_pack, a.groups), ("catch_up", catch_up, a.catchup_groups)):
        med, moved, info = f(ctx, G, a)
        info.update(ms=round(med, 4), bytes_moved=moved, GBps=round(moved / med / 1e6, 1))
        print(f"{key}: {info}", flush=True)
        result[key] = info
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
