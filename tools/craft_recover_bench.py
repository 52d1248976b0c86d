"""ss_follower_recover on the WAL a CRaft follower writes: n = 5 (RS(3,2)), 4 KB request batches, one 1366-byte shard
per entry (sharded mode: the follower's own shard).  Two shapes:
  * bulk: 2^16 groups x 32 entries (about 3 GB of records and 3 GB of store);
  * bookkeeping-bound: 2^20 groups x 1 entry.

The WAL is built by the real path: replica 0's CRaft engine proposes the entries (ss_engine_craft_propose), packs one
AppendEntries frame per group for replica 1 (ss_frame_append_pack_dev through RaftEngine.pack_append) and a live
follower takes them (ss_follower_append).  Each group's records are the Metadata cell the append wrote, the slot-0 null
entry and the LogEntry records, in WAL order.  Then, timed with CUDA events (median of --steps launches after --warmup):
  * ss_follower_recover of the whole WAL into a second follower whose state is re-zeroed to the state at creation before
    each launch, outside the timed window;
  * b.copy_(a) of as many bytes as the replay moves, in the same run.
Rates are algorithmic bytes: records read + store written (recover), 2x the bytes (copy).  Checks: every verdict is
"accepted", and the recovered log_end, terms, held masks and data lengths equal the live follower's.

Usage: python tools/craft_recover_bench.py [--steps K] [--warmup W] [--bulk-groups N] [--book-groups N]
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
from summerset_b200.engine import Follower, RaftEngine  # noqa: E402

N, DATA_LEN = 5, 4096
D = N // 2 + 1
L = -(-DATA_LEN // D)
PITCH = (L + 31) & ~31


def live_wal(ctx, G, E, dev):
    """the leader proposes E entries per group and packs them for replica 1, whose follower appends them: -> (buf,
    rec_off, rec_group, the live follower)"""
    eng = RaftEngine(ctx, G, N, craft=True, window=64)
    eng.log_view()
    eng.curr_term.fill_(1)
    gen = torch.Generator(device=dev)
    gen.manual_seed(3)
    stores = []
    for _ in range(E):
        arena = torch.randint(0, 256, (G * DATA_LEN + 1,), dtype=torch.uint8, device=dev, generator=gen)
        off = torch.arange(G, dtype=torch.int64, device=dev) * DATA_LEN
        ln = torch.full((G,), DATA_LEN, dtype=torch.int32, device=dev)
        st = torch.zeros((eng.P + 1, G * PITCH), dtype=torch.uint8, device=dev)
        stores.append(st)
        o = eng.propose(0, arena, off, ln, st, torch.empty(G * 1536, dtype=torch.uint8, device=dev))
        assert (o["slot_out"] >= 0).all()
        del arena
    frame_bytes = G * (64 + E * (L + 64))
    out = torch.empty(frame_bytes * (N - 1), dtype=torch.uint8, device=dev)
    p = eng.pack_append(0, out, G * (N - 1), msg_chunk_size=E)
    torch.cuda.synchronize()
    nf = int(p["n_frames"][0])
    sel = (p["frame_peer"][:nf] == 0).nonzero().flatten()
    assert sel.numel() == G
    fol = Follower(ctx, G, N, 1, 64)
    fstore = torch.empty(G * E * PITCH, dtype=torch.uint8, device=dev)
    wal = torch.empty(G * E * 1536, dtype=torch.uint8, device=dev)
    fg = p["frame_group"][sel].contiguous()
    a = fol.append(out, p["frame_off"][sel].contiguous(), fg, torch.zeros(G, dtype=torch.uint8, device=dev), fstore, wal)
    torch.cuda.synchronize()
    assert (a["verdict"].cpu().numpy().view(np.uint32) == _lib.SS_FOLLOWER_VERDICT_ACCEPTED).all()
    del out, stores, eng
    # the records: every group's Metadata cell, one shared slot-0 null entry, then the appended records (one size)
    wal_len = a["wal_len"]
    slot = int(wal_len[0]) // E
    assert (wal_len == slot * E).all()
    body = bytes([1, 0, D, N - D, 0, 0, N] + [0] * N + [0, 0, 0])   # LogEntry{0, the null codeword, false, 0}
    null = len(body).to_bytes(8, "big") + body
    assert (a["meta_len"] > 0).all()
    used = int(a["totals"][1])
    meta_at, null_at = used, used + G * 32
    buf = torch.cat([wal[:used], a["meta"].reshape(-1), torch.tensor(list(null), dtype=torch.uint8, device=dev)])
    rec_off = torch.cat([meta_at + 32 * torch.arange(G, dtype=torch.int64, device=dev), torch.full((G,), null_at, dtype=torch.int64, device=dev),
                         (a["wal_off"][:, None] + slot * torch.arange(E, device=dev)[None, :]).reshape(-1)])
    rec_group = torch.cat([fg, fg, fg.repeat_interleave(E)])
    rec_bytes = int(a["meta_len"].sum()) + G * len(null) + G * E * int.from_bytes(wal[:8].cpu().numpy().tobytes(), "big") + G * E * 8
    del wal
    return buf, rec_off, rec_group, rec_bytes, fol, fstore


def timed(fn, reset, a):
    ms = []
    for step in range(a.warmup + a.steps):
        reset()
        e = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        e[0].record()
        fn()
        e[1].record()
        torch.cuda.synchronize()
        if step >= a.warmup:
            ms.append(e[0].elapsed_time(e[1]))
    return float(np.median(ms))


def measure(ctx, name, G, E, a):
    dev = torch.device("cuda", 0)
    buf, rec_off, rec_group, rec_bytes, live, live_store = live_wal(ctx, G, E, dev)
    fol = Follower(ctx, G, N, 1, 64)
    vv = fol.vote_view()
    store = torch.empty(G * E * PITCH, dtype=torch.uint8, device=dev)
    res = {}

    def reset():
        for t in (fol.start_slot, fol.curr_term, fol.last_commit, fol.last_snap, fol.term, fol.shard_addr, fol.held, fol.data_len,
                  fol.last_exec, vv["vote_term"], vv["role_term"], vv["role"], vv["votes"]):
            t.zero_()
        fol.log_end.fill_(1)
        fol.leader.fill_(0xFF)
        vv["voted_for"].fill_(0xFF)

    def run():
        res.update(fol.recover(buf, rec_off, rec_group, store))

    ms = timed(run, reset, a)
    v = res["verdict"].cpu().numpy().view(np.uint32)
    assert (v == _lib.SS_FOLLOWER_VERDICT_ACCEPTED).all(), "every record must apply"
    total = int(res["total"][0])
    assert total == G * E * PITCH
    for k in ("log_end", "curr_term", "term", "held", "data_len"):
        assert torch.equal(getattr(fol, k), getattr(live, k)), k
    moved = rec_bytes + total
    del live_store, live
    src = torch.empty(moved, dtype=torch.uint8, device=dev)
    dst = torch.empty_like(src)
    copy_ms = timed(lambda: dst.copy_(src), lambda: None, a)
    r = {"groups": G, "entries_per_group": E, "records": int(rec_off.numel()), "ms": ms, "records_per_s": rec_off.numel() / ms * 1e3,
         "bytes_moved": moved, "GBps": moved / ms / 1e6, "copy_ms": copy_ms, "copy_GBps": 2 * moved / copy_ms / 1e6}
    r["frac_of_copy"] = r["GBps"] / r["copy_GBps"]
    print(f"{name}: {G} groups x {E} entries, {r['records']} records, {moved / 1e9:.2f} GB in {ms:.3f} ms = {r['GBps']:.0f} GB/s, "
          f"{r['records_per_s']:.3g} records/s; copy_ {copy_ms:.3f} ms = {r['copy_GBps']:.0f} GB/s "
          f"({100 * r['frac_of_copy']:.0f} % of it)", flush=True)
    fol.close()
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--bulk-groups", type=int, default=1 << 16)
    ap.add_argument("--book-groups", type=int, default=1 << 20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("craft_recover_bench needs a GPU")
    torch.cuda.set_device(0)
    name, power = card()
    print(f"card: {name}, power limit {power}", flush=True)
    ctx = Context(0)
    result = {"card": name, "power_limit": power, "steps": a.steps, "warmup": a.warmup,
              "workload": f"CRaft n={N}, {DATA_LEN} B batches, one {L}-byte shard per entry, WAL from the live append path"}
    result["bulk"] = measure(ctx, "bulk", a.bulk_groups, 32, a)
    torch.cuda.empty_cache()
    result["bookkeeping"] = measure(ctx, "bookkeeping-bound", a.book_groups, 1, a)
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
