"""ss_engine_prepare_absorb: the new leader's PrepareReply absorb in every group of a 2^19- or 2^20-group RSPaxos engine
(n = 5, d = 3, f = 1, me = 1) with a quarter, half or the whole 64-slot window Preparing.

Preparing means: window positions [0, k) of each group, k in {16, 32, 64}, are Preparing on the leader's acceptor at the
step-up's ballot, with source = me, as ss_acceptor_step_up leaves them.  The batch holds a quorum of replies for each of
them: the leader's own and two peers', each voting at one ballot with its own data shard of a 64-byte payload, so the
third endprep reply of each group decides all k instances USE and the reconstruct regenerates both parity shards.  Every
group's replies are the same bytes (window base 0, one ballot), so buf holds 3k frames and frame_off points every
group's frames at them; frames are ordered by group, then replica, then slot.  Between launches, outside the timed
window, a call with bal_prep_sent = 0 resets the engine's bookkeeping and store_used goes back to 0.
Timed with CUDA events (median of --steps launches after --warmup), alternated with b.copy_(a) of the same algorithmic
bytes: per frame its bytes, frame_off, group, peer and verdict; per decided record the T shard slots written and its six
fields; per group bal_prep_sent and pending.
Check before timing: every verdict and total, and a sample of decided codewords whose data shards must be the payload.

Usage: python tools/engine_prepare_bench.py [--groups N ...] [--steps K] [--warmup W]
Prints the card name, power limit and max SM clock, one line per measurement and one JSON line.  Fails without a GPU.
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
from acceptor_prepare_bench import max_sm_clock  # noqa: E402
from engine_ragged_bench import card, stats  # noqa: E402
from summerset_b200 import _lib  # noqa: E402
from summerset_b200._lib import check  # noqa: E402
from summerset_b200.api import Context  # noqa: E402
from summerset_b200.engine import Acceptor, LeaderEngine  # noqa: E402

N, D, F, ME = 5, 3, 1, 1
BALLOT = (1 << 8) | (ME + 1)
DATA_LEN = 64
L = -(-DATA_LEN // D)
PITCH = (L + 31) // 32 * 32


def _v(x):
    """a bincode 2 standard() varint"""
    if x < 251:
        return bytes([x])
    if x < 1 << 16:
        return b"\xfb" + x.to_bytes(2, "little")
    if x < 1 << 32:
        return b"\xfc" + x.to_bytes(4, "little")
    return b"\xfd" + x.to_bytes(8, "little")


def reply_frame(slot, endprep, shard_idx, shard):
    """PeerMessage::Msg{PrepareReply{slot, trigger_slot 0, endprep_slot, BALLOT, voted: Some((1, codeword))}}, the
    codeword carrying one shard"""
    cw = bytes([D, N - D]) + _v(DATA_LEN) + _v(L) + _v(N)
    for j in range(N):
        cw += (b"\x01" + _v(L) + shard) if j == shard_idx else b"\x00"
    cw += b"\x00"
    body = b"\x00" + _v(1) + _v(slot) + _v(0) + _v(endprep) + _v(BALLOT) + b"\x01" + _v(1) + cw
    return len(body).to_bytes(8, "big") + body


def run(ctx, G, k, a, dev):
    payload = np.random.default_rng(k).integers(0, 256, DATA_LEN, dtype=np.uint8).tobytes()
    shards = [payload[j * L:(j + 1) * L].ljust(L, b"\x00") for j in range(D)]
    peers = [0, ME, 2]                                  # the leader and two peers, each voting its own data shard
    frames, offs, at = [], [], 0
    for r in peers:
        for s in range(k):
            f = reply_frame(s, k - 1, r, shards[r])
            frames.append(f)
            offs.append(at)
            at += len(f)
    buf = torch.from_numpy(np.frombuffer(b"".join(frames) + bytes(16), dtype=np.uint8).copy()).to(dev)
    per = 3 * k
    n = G * per
    frame_off = torch.tensor(offs, dtype=torch.int64, device=dev).repeat(G)
    frame_group = torch.arange(G, dtype=torch.int32, device=dev).repeat_interleave(per)
    frame_peer = torch.tensor(peers, dtype=torch.uint8, device=dev).repeat_interleave(k).repeat(G)
    eng = LeaderEngine(ctx, "rspaxos", G, N, F, 1)
    acc = Acceptor(ctx, "rspaxos", G, N, ME, D, N)
    acc.preparing.fill_(-1 if k == 64 else (1 << k) - 1)
    acc.inst_bal.fill_(BALLOT)
    acc.source.fill_(ME)
    acc.bal_max_seen.fill_(BALLOT)
    bps = torch.full((G,), BALLOT, dtype=torch.int64, device=dev)
    zero = torch.zeros(G, dtype=torch.int64, device=dev)
    ndec = G * k
    store = torch.empty((N, ndec * PITCH), dtype=torch.uint8, device=dev)
    used = torch.zeros(1, dtype=torch.int64, device=dev)
    wal = torch.empty(32, dtype=torch.uint8, device=dev)
    e = lambda m, dt: torch.empty(max(m, 1), dtype=dt, device=dev)
    out = dict(rec_group=e(1, torch.int32), rec_slot=e(1, torch.int64), dec_slot=e(ndec, torch.int64), dec_ballot=e(ndec, torch.int64),
               dec_shard_off=e(ndec, torch.int64), dec_data_len=e(ndec, torch.int32), dec_group=e(ndec, torch.int32),
               pending=e(G, torch.int64), verdict=e(n, torch.int32), totals=e(3, torch.int64))
    p = lambda x: None if x is None else x.data_ptr()
    lib = ctx.lib

    def call(b):
        check(lib.ss_engine_prepare_absorb(eng.h, acc.h, p(buf), buf.numel(), p(frame_off), p(frame_group), p(frame_peer), n, 1, 0,
                                           p(b), None, p(store), store.shape[1], p(used), p(wal), 32, p(out["rec_group"]),
                                           p(out["rec_slot"]), 1, p(out["dec_slot"]), p(out["dec_ballot"]), p(out["dec_shard_off"]),
                                           p(out["dec_data_len"]), None, p(out["dec_group"]), ndec, p(out["pending"]),
                                           p(out["verdict"]), p(out["totals"])))

    def restore():
        call(zero)
        used.zero_()

    t_call = timed(lambda: call(bps), restore, a)
    restore()
    call(bps)
    torch.cuda.synchronize()
    tot = [int(x) for x in out["totals"].cpu().numpy()]
    checks = {"verdicts": bool((out["verdict"].cpu().numpy().view(np.uint32) == _lib.SS_ACCEPT_VERDICT_ACCEPTED).all()),
              "totals": tot == [ndec, 0, ndec * PITCH], "pending": bool((out["pending"] == 0).all().item()),
              "status": ctx.device_status() == 0}
    rng = np.random.default_rng(k + 1)
    ok = True
    dg, ds, do = out["dec_group"].cpu().numpy(), out["dec_slot"].cpu().numpy(), out["dec_shard_off"].cpu().numpy()
    for idx in rng.choice(ndec, 64, replace=False):
        ok &= (int(dg[idx]), int(ds[idx])) == (idx // k, idx % k)
        data = b"".join(store[j, int(do[idx]):int(do[idx]) + L].cpu().numpy().tobytes() for j in range(D))
        ok &= data[:DATA_LEN] == payload
    checks["bytes"] = bool(ok)
    nbytes = n * (len(frames[0]) + 8 + 4 + 1 + 4) + ndec * (N * PITCH + 8 + 8 + 8 + 4 + 4) + G * 16
    eng.close()                                         # the copy's buffers take the room the call's scratch held
    acc.close()
    del store, frame_off, frame_group, frame_peer, out
    torch.cuda.empty_cache()
    src = torch.empty(nbytes // 2, dtype=torch.uint8, device=dev)
    dst = torch.empty_like(src)
    t_copy = timed(lambda: dst.copy_(src), lambda: None, a)
    gbs = lambda nb, ms: round(nb / (float(np.median(ms)) * 1e-3) / 1e9, 1)
    row = {"k": k, "groups": G, "frames": n, "checks": checks,
           "prepare_absorb": {**stats(t_call), "bytes": nbytes, "GB/s": gbs(nbytes, t_call)},
           "copy": {**stats(t_copy), "bytes": 2 * (nbytes // 2), "GB/s": gbs(2 * (nbytes // 2), t_copy)}}
    for key in ("prepare_absorb", "copy"):
        v = row[key]
        print(f"k={k:2d} G={G:8d} {key:14s} median {v['median_ms']:8.3f} ms  {v['bytes'] / 1e9:7.3f} GB  {v['GB/s']:8.1f} GB/s",
              flush=True)
    del src, dst
    torch.cuda.empty_cache()
    return row, all(checks.values())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--groups", type=int, nargs="+", default=[1 << 19, 1 << 20])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("engine_prepare_bench needs a CUDA GPU: there is no CPU fallback")
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    name, power = card()
    clock = max_sm_clock()
    print(f"card: {name}, power limit {power}, max SM clock {clock}", flush=True)
    ctx = Context(0)
    rows, ok = [], True
    for G in a.groups:
        for k in (16, 32, 64):
            row, good = run(ctx, G, k, a, dev)
            rows.append(row)
            ok &= good
    print(json.dumps({"card": name, "power_limit": power, "max_sm_clock": clock, "steps": a.steps, "checked": ok, "rows": rows}),
          flush=True)
    ctx.close()
    if not ok:
        sys.exit("prepare absorb check failed")


if __name__ == "__main__":
    main()
