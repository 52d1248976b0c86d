"""ss_acceptor_prepare and ss_acceptor_prepare_reply on the cfg-4 mix (request batches of 256 B .. 64 KB,
workloads.cfg4_lengths): RSPaxos n = 5 (d = 3, a follower holds one shard) and Crossword n = T = 5 (d = 3, spr = 3).

Each group's window is filled with k accepted instances, k in {1, 8, 64}, by the accept pass (the leader path's Accept
frames of replica 1, one proposal per group per slot).  Up to 2^19 groups; a window of k instances holds k shard sets
per group, so the group count is capped so that the follower's store stays within --store-gb (printed per row).
Then one Prepare per group with trigger = window_base at a higher ballot.  Timed with CUDA events (median of --steps
launches after --warmup; the state a launch consumes is restored between launches, outside the timed window), alternated
with b.copy_(a) of the same algorithmic bytes:
  * prepare: frames read + state written (inst_bal, source, trigger, span per slot; four words per group) + records
    written (32-byte cells, group, slot, frame)
  * reply:   voted shards read + reply bytes written
Check before timing: a sample of groups' WAL cells and replies compared byte for byte with the model of
tests/test_acceptor_prepare.py (the varint and RSCodeword encoders of the oracle).

Usage: python tools/acceptor_prepare_bench.py [--groups N] [--steps K] [--warmup W] [--store-gb S]
Prints the card name, power limit and max SM clock, one line per measurement and one JSON line.  Fails without a GPU.
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))
from acceptor_exec_bench import timed  # noqa: E402
from engine_ragged_bench import card, stats  # noqa: E402
from oracle import pyoracle  # noqa: E402
from summerset_b200 import _lib  # noqa: E402
from summerset_b200 import workloads as wl  # noqa: E402
from summerset_b200.api import Context  # noqa: E402
from summerset_b200.engine import Acceptor, LeaderEngine  # noqa: E402

N, D, ME = 5, 3, 1


def max_sm_clock():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def var(v):
    return pyoracle.varint(v)


def run(ctx, protocol, k, G, a, dev):
    cw = protocol == "crossword"
    lens, _ = wl.cfg4_lengths(G)
    lens = lens.astype(np.uint32)
    lay = wl.ragged_layout(lens, D)
    gen = torch.Generator(device=dev)
    gen.manual_seed(wl.SEED_BASE + 7)
    arena = torch.randint(0, 256, (lay["data_bytes"] + 64,), dtype=torch.uint8, device=dev, generator=gen)
    L = (lens.astype(np.int64) + D - 1) // D
    pitch = (L + 31) // 32 * 32
    eng = LeaderEngine(ctx, protocol, G, N, 1, 1, **(dict(rs_total_shards=N, rs_data_shards=D) if cw else {}))
    bal = torch.arange(1, G + 1, dtype=torch.int64, device=dev)
    eng.set_prepared_ballots(bal)
    if cw:
        policies = np.array([pyoracle.cw_brr_assignment(N, N, 3)], dtype=np.uint32)
        eng.set_policies([list(map(int, q)) for q in policies], True)
    else:
        policies = np.array([[1 << r for r in range(N)]], dtype=np.uint32)
    held_per = bin(int(policies[0][ME])).count("1")
    acc = Acceptor(ctx, protocol, G, N, ME, D, N)
    groups = torch.arange(G, dtype=torch.int32, device=dev)
    zeros8 = torch.zeros(G, dtype=torch.uint8, device=dev)
    pol = torch.zeros(G, dtype=torch.uint8, device=dev)
    ln = torch.from_numpy(lens.view(np.int32)).to(dev)
    doff = torch.from_numpy(lay["data_off"].view(np.int64)).to(dev)
    lstore = torch.zeros((N, int(pitch.sum())), dtype=torch.uint8, device=dev)
    astore = torch.empty(k * held_per * int(pitch.sum()) + 64, dtype=torch.uint8, device=dev)
    wal = None
    at = 0
    for s in range(k):
        slot_out, shard_off, _ = eng.propose_ragged(arena, doff, ln, lstore, pol if cw else None)
        out, off, fl, _ = ctx.frame_accept_pack_ragged(lstore, shard_off, ln, D, N - D, policies, pol, ME, slot_out, bal,
                                                       with_assignment=cw)
        if wal is None:
            wal = torch.empty(int(fl.to(torch.int64).sum()) + 64 * G + 64, dtype=torch.uint8, device=dev)
        res = acc.accept(out, off, groups, zeros8, astore[at:], wal)
        assert (res["verdict"].cpu().numpy().view(np.uint32) == _lib.SS_ACCEPT_VERDICT_ACCEPTED).all()
        at += int(res["totals"][0].item())
        at = (at + 15) // 16 * 16
        del out, off, fl, res
    assert ctx.device_status() == 0
    eng.close()
    del lstore, wal
    torch.cuda.empty_cache()
    # one Prepare{trigger 0, ballot G + 1 + g} per group, from replica 0
    nb = np.arange(G + 1, 2 * G + 1, dtype=np.uint64)
    frames = [var(0) + var(0) + var(0) + var(int(b)) for b in nb]
    blobs = b"".join(len(f).to_bytes(8, "big") + f for f in frames)
    foff = np.cumsum([0] + [8 + len(f) for f in frames[:-1]]).astype(np.int64)
    buf = torch.frombuffer(bytearray(blobs), dtype=torch.uint8).to(dev)
    foff_d = torch.from_numpy(foff).to(dev)
    nrec = G * k
    pwal = torch.empty(nrec * 32, dtype=torch.uint8, device=dev)
    saved = {n: getattr(acc, n).clone() for n in ("bal_max_seen", "inst_bal", "accepting", "committed", "preparing", "source",
                                                   "prep_trigger", "prep_span", "voted_bal", "voted_mask")}

    def restore():
        for n, t in saved.items():
            getattr(acc, n).copy_(t)

    res_p = {}
    t_prep = timed(lambda: res_p.update(acc.prepare(buf, foff_d, groups, zeros8, pwal, nrec)), restore, a)
    restore()
    res_p = acc.prepare(buf, foff_d, groups, zeros8, pwal, nrec)
    checks = {"prepared": bool((res_p["verdict"].cpu().numpy().view(np.uint32) == _lib.SS_ACCEPT_VERDICT_ACCEPTED).all())
              and int(res_p["totals"][0].item()) == nrec}
    # the replies
    vshard = int((L * held_per).sum()) * k
    reply_cap = int(nrec * 64 + k * (L * held_per + 16 * held_per + 64).sum())
    rout = torch.empty(reply_cap // 16 * 16 + 16, dtype=torch.uint8, device=dev)
    res_r = {}
    t_rep = timed(lambda: res_r.update(acc.prepare_reply(res_p["rec_group"], res_p["rec_slot"], rout)), lambda: None, a)
    checks["replied"] = bool((res_r["reply_off"] >= 0).all().item())
    reply_bytes = int(res_r["reply_len"].sum().item())
    # byte-for-byte sample against the model's encoders
    rg, rs_ = res_p["rec_group"].cpu().numpy(), res_p["rec_slot"].cpu().numpy()
    ro, rl = res_r["reply_off"].cpu().numpy(), res_r["reply_len"].cpu().numpy()
    cells = pwal.cpu().numpy()
    arena_h = arena.cpu().numpy()
    ok_bytes = True
    rng = np.random.default_rng(k)
    for idx in rng.choice(nrec, min(64, nrec), replace=False):
        g, s = int(rg[idx]), int(rs_[idx])
        body = var(0) + var(s) + var(int(nb[g]))
        cell = len(body).to_bytes(8, "big") + body
        ok_bytes &= cells[32 * idx:32 * idx + len(cell)].tobytes() == cell
        data = arena_h[int(lay["data_off"][g]):int(lay["data_off"][g]) + int(lens[g])].tobytes()
        sh = pyoracle.cw_split(data, D)
        full = [np.ascontiguousarray(sh[j]) for j in range(D)] + [np.zeros(sh.shape[1], np.uint8) for _ in range(N - D)]
        assert pyoracle.rs_encode(D, N - D, full) == 0
        mask = int(policies[0][ME])
        from tests.test_acceptor_reconstruct import cw_bytes
        cwb = cw_bytes(D, N - D, int(lens[g]), int(L[g]), [full[j].tobytes() if (mask >> j) & 1 else None for j in range(N)])
        want_body = var(0) + var(1) + var(s) + var(0) + var(k - 1) + var(int(nb[g])) + b"\x01" + var(g + 1) + cwb
        want = len(want_body).to_bytes(8, "big") + want_body
        got = rout[int(ro[idx]):int(ro[idx]) + int(rl[idx])].cpu().numpy().tobytes()
        ok_bytes &= got == want
    checks["bytes"] = bool(ok_bytes)
    status = ctx.device_status()
    prep_bytes = len(blobs) + nrec * (8 + 8 + 8 + 1) + G * 4 * 8 + nrec * (32 + 4 + 8 + 4)
    rep_bytes = vshard + reply_bytes
    gbs = lambda nbytes, ms: round(nbytes / (float(np.median(ms)) * 1e-3) / 1e9, 1)
    row = {"protocol": protocol, "k": k, "groups": G, "status": status, "checks": checks}
    for key, t, nbytes in (("prepare", t_prep, prep_bytes), ("reply", t_rep, rep_bytes)):
        src = torch.empty(nbytes // 2, dtype=torch.uint8, device=dev)
        dst = torch.empty_like(src)
        t_copy = timed(lambda: dst.copy_(src), lambda: None, a)
        row[key] = {**stats(t), "bytes": nbytes, "GB/s": gbs(nbytes, t)}
        row[key + "_copy"] = {**stats(t_copy), "bytes": 2 * (nbytes // 2), "GB/s": gbs(2 * (nbytes // 2), t_copy)}
        for k2 in (key, key + "_copy"):
            v = row[k2]
            print(f"{protocol:9s} k={k:2d} G={G:7d} {k2:12s} median {v['median_ms']:8.3f} ms  {v['bytes'] / 1e9:7.3f} GB  "
                  f"{v['GB/s']:8.1f} GB/s", flush=True)
        del src, dst
    acc.close()
    return row, status == 0 and all(checks.values())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--groups", type=int, default=1 << 19)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--store-gb", type=float, default=12.0)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("acceptor_prepare_bench needs a CUDA GPU: there is no CPU fallback")
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    name, power = card()
    clock = max_sm_clock()
    print(f"card: {name}, power limit {power}, max SM clock {clock}", flush=True)
    ctx = Context(0)
    lens, _ = wl.cfg4_lengths(a.groups)
    per_group = float(((lens.astype(np.int64) + D - 1) // D + 32).mean())
    rows, ok = [], True
    for protocol, held in (("rspaxos", 1), ("crossword", 3)):
        for k in (1, 8, 64):
            G = int(min(a.groups, a.store_gb * 1e9 / (k * held * per_group)))
            G = max(1 << 10, 1 << (G.bit_length() - 1))
            row, good = run(ctx, protocol, k, G, a, dev)
            rows.append(row)
            ok &= good
            torch.cuda.empty_cache()
    print(json.dumps({"card": name, "power_limit": power, "max_sm_clock": clock, "steps": a.steps, "checked": ok, "rows": rows}),
          flush=True)
    ctx.close()
    if not ok:
        sys.exit("acceptor prepare check failed")


if __name__ == "__main__":
    main()
