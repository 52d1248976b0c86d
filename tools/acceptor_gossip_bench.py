"""ss_acceptor_gossip and ss_acceptor_step_up_reads on full 64-slot windows at 2^19 groups: Crossword n = 5, T = 5,
d = 3, balanced assignments with spr in {1, 2, 3}, batch / chunk size 10.

Replica 1's state is installed through the acceptor's views: every window position committed, held = its own
assignment row (spr shards, so spr < 3 leaves every instance short of d), source = replica 0 (the leader), the same
assignment rows for every instance.  Timed with CUDA events (median of --steps launches after --warmup; gossip_bar is
zeroed between launches, outside the timed window):
  * gossip: every group walked from slot 0, each instance planned by gossip_targets_excl, Reconstruct{slots_excl}
    frames for the selected peers
  * step_up: the same instances listed for a new leader's broadcast
Check: the totals match the frame count the plan implies, and group 0's and the last group's frames match frames
encoded on the CPU with the oracle's varint and Bitmap encoders, byte for byte.

Usage: python tools/acceptor_gossip_bench.py [--groups N] [--steps K] [--warmup W]
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
from acceptor_exec_bench import timed  # noqa: E402
from engine_ragged_bench import card, stats  # noqa: E402
from oracle import pyoracle  # noqa: E402
from summerset_b200.api import Context  # noqa: E402
from summerset_b200.engine import Acceptor  # noqa: E402

N, T, D, ME, BATCH = 5, 5, 3, 1, 10


def frame_reconstruct(slots, excl):
    """PeerMessage::Msg{Reconstruct{slots_excl}} with size-T Bitmaps, from the oracle's varint and Bitmap encoders"""
    body = pyoracle.varint(0) + pyoracle.varint(4) + pyoracle.varint(len(slots))
    body += b"".join(pyoracle.varint(s) + pyoracle.bitmap_encode(T, e) for s, e in zip(slots, excl))
    return len(body).to_bytes(8, "big") + body


def expected(rows, held, step_up):
    """frames of one group: (dst, bytes) in (peer, chunk) order"""
    slots = list(range(64))
    if step_up:
        lists = {0xFF: [(s, held) for s in slots]} if bin(held).count("1") < D else {}
    else:
        lists = {}
        if bin(held).count("1") < D:
            t, excl = pyoracle.gossip_targets_excl(ME, N, D, 0, held, rows, (1 << N) - 1)
            lists = {q: [(s, int(excl[q])) for s in slots] for q in range(N) if (t >> q) & 1}
    out = []
    for q, ents in sorted(lists.items()):
        for c in range(0, len(ents), BATCH):
            ch = ents[c:c + BATCH]
            out.append((q, frame_reconstruct([s for s, _ in ch], [e for _, e in ch])))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--groups", type=int, default=1 << 19)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("acceptor_gossip_bench needs a CUDA GPU: there is no CPU fallback")
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    name, power = card()
    print(f"card: {name}, power limit {power}", flush=True)
    G = a.groups
    ctx = Context(0)
    res = {"card": name, "power_limit": power, "groups": G, "steps": a.steps, "batch": BATCH}
    ok = True
    for spr in (1, 2, 3):
        rows = [int(x) for x in pyoracle.cw_brr_assignment(N, T, spr)]
        held = rows[ME]
        acc = Acceptor(ctx, "crossword", G, N, ME, D, T)
        acc.committed.fill_(-1)
        acc.held.fill_(held)
        acc.data_len.fill_(3000)
        acc.source.fill_(0)
        acc.assign_rows.copy_(torch.tensor(rows, dtype=torch.int32, device=dev).repeat(G * 64))
        for key, step_up in (("gossip", False), ("step_up", True)):
            want = expected(rows, held, step_up)
            nf = len(want) * G
            nbytes = sum((len(f) + 15) // 16 * 16 for _, f in want) * G
            out = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=dev)
            got = {}
            if step_up:
                fn = lambda: got.update(acc.step_up_reads(out, max(nf, 1), BATCH))
            else:
                fn = lambda: got.update(acc.gossip(out, max(nf, 1), BATCH))
            t = timed(fn, lambda: acc.gossip_bar.zero_(), a)
            status = ctx.device_status()
            check = status == 0 and [int(x) for x in got["totals"]] == [nf, nbytes]
            if nf:
                ob = out.cpu().numpy()
                fo, fl = got["frame_off"].cpu().numpy(), got["frame_len"].cpu().numpy()
                fd = got["frame_dst"].cpu().numpy()
                for base in (0, nf - len(want)):
                    for j, (q, f) in enumerate(want):
                        k = base + j
                        check = check and int(fd[k]) == q and ob[int(fo[k]):int(fo[k]) + int(fl[k])].tobytes() == f
            ok = ok and check
            r = res[f"{key}_spr{spr}"] = {**stats(t), "frames": nf, "bytes": nbytes, "checked": check,
                                          "GB/s": round(nbytes / (float(np.median(t)) * 1e-3) / 1e9, 1)}
            print(f"{key:8s} spr {spr}  median {r['median_ms']:8.3f} ms  min {r['min_ms']:8.3f}  max {r['max_ms']:8.3f}  "
                  f"{nf:9d} frames  {nbytes / 1e6:8.1f} MB  {r['GB/s']:7.1f} GB/s written  checked={check}", flush=True)
            del out, got
        acc.close()
        torch.cuda.empty_cache()
    res["checked"] = ok
    print(json.dumps(res), flush=True)
    ctx.close()
    if not ok:
        sys.exit("acceptor gossip check failed")


if __name__ == "__main__":
    main()
