"""Ragged proposals on the cfg-4 mix (BASELINE config 4: request batches of 256 B .. 64 KB, workloads.cfg4_lengths),
2^19 groups, for a Crossword engine (n = 5, T = 5, d = 3) and an RSPaxos engine (n = 5, RS(3,2)).

For each engine:
  * ss_engine_propose_ragged, end to end (prepare, pitch scan, clamp + bookkeeping, one ragged encode), timed with CUDA
    events alternately with a bare ss_rs_encode_batch_dev (SS_RS_OUT_PADDED16 | SS_RS_EMIT_DATA) on the same layout; the
    difference is what the device-side placement and bookkeeping cost.  The engine's window is emptied between launches
    (outside the timed region) so every launch proposes every group.
  * ss_frame_accept_pack_ragged_dev for peer 0 (Crossword: the spr shards of the cfg-4 assignment, with_assignment).
  * rates from the bytes the algorithm moves: propose (d+p)*L_g + d*L_g per group (payload read, parity written, data
    shards emitted), frames the bytes written.
  * checks: the engine's planes equal the bare encoder's byte for byte; a sample of peer 0's frames equals the oracle's.

Usage: python tools/engine_ragged_bench.py [--groups N] [--steps K] [--warmup W] [--sample S]
Prints the card name and power limit, one line per measurement and one JSON line.  Fails without a GPU.
"""
import argparse
import ctypes as C
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from oracle import pyoracle as oracle  # noqa: E402
from summerset_b200 import _lib  # noqa: E402
from summerset_b200 import workloads as wl  # noqa: E402
from summerset_b200._lib import check  # noqa: E402
from summerset_b200.api import Context, ReedSolomon  # noqa: E402
from summerset_b200.engine import LeaderEngine  # noqa: E402

N = 5
FLAGS = 1 | 2                 # SS_RS_OUT_PADDED16 | SS_RS_EMIT_DATA


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def stats(ms):
    return {"median_ms": round(float(np.median(ms)), 4), "min_ms": round(float(np.min(ms)), 4), "max_ms": round(float(np.max(ms)), 4)}


def run_engine(ctx, protocol, lens, spr, arena, data_off, a):
    G = len(lens)
    dev = torch.device("cuda", 0)
    kw = dict(rs_total_shards=5, rs_data_shards=3) if protocol == "crossword" else {}
    eng = LeaderEngine(ctx, protocol, G, N, 1, 1, **kw)
    bal = np.arange(1, G + 1, dtype=np.uint64)
    eng.set_prepared_ballots(torch.from_numpy(bal.view(np.int64)).to(dev))
    policies = np.array([[1 << r for r in range(N)]], dtype=np.uint32)              # RSPaxos: replica r holds shard r
    pol = None
    if protocol == "crossword":
        policies = np.stack([oracle.cw_brr_assignment(N, 5, s) for s in (1, 2, 3)]).astype(np.uint32)
        eng.set_policies([list(map(int, q)) for q in policies], True)
        pol = torch.from_numpy((spr - 1).astype(np.uint8)).to(dev)
    d, p = eng.d, eng.T - eng.d
    L = (lens.astype(np.int64) + d - 1) // d
    plane_stride = int(((L + 31) // 32 * 32).sum())
    store = torch.zeros((eng.T, plane_stride), dtype=torch.uint8, device=dev)
    bare = torch.zeros_like(store)
    ln = torch.from_numpy(lens.view(np.int32)).to(dev)
    do = torch.from_numpy(data_off.view(np.int64)).to(dev)
    coder = ReedSolomon(ctx, d, p)                  # the bare encode: a coder of the engine's code
    out = {}

    def reset():
        eng.accepting.zero_()
        eng.committed.zero_()

    # layout of the bare encode: the engine's own offsets (every group proposes at slot 0 of an empty window)
    reset()
    slot_out, shard_off, need = eng.propose_ragged(arena, do, ln, store, pol)
    torch.cuda.synchronize()
    assert ctx.device_status() == 0 and int(need) == plane_stride and bool((slot_out == 0).all())

    def bare_encode():
        check(ctx.lib.ss_rs_encode_batch_dev(coder.h, arena.data_ptr(), do.data_ptr(), ln.data_ptr(), G,
                                             bare.data_ptr() + d * plane_stride, plane_stride, shard_off.data_ptr(), FLAGS))

    t_eng, t_bare = [], []
    for step in range(a.warmup + a.steps):
        reset()
        e = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        e[0].record()
        eng.propose_ragged(arena, do, ln, store, pol)
        e[1].record()
        e[2].record()
        bare_encode()
        e[3].record()
        torch.cuda.synchronize()
        if step >= a.warmup:
            t_eng.append(e[0].elapsed_time(e[1]))
            t_bare.append(e[2].elapsed_time(e[3]))
    assert ctx.device_status() == 0
    same = bool(torch.equal(store, bare))
    nbytes = int(((d + p) * L + d * L).sum())
    out["propose_ragged"] = {**stats(t_eng), "bytes": nbytes, "GB/s": round(nbytes / (np.median(t_eng) * 1e-3) / 1e9, 1)}
    out["bare_encode"] = {**stats(t_bare), "bytes": nbytes, "GB/s": round(nbytes / (np.median(t_bare) * 1e-3) / 1e9, 1)}
    ovh = float(np.median(t_eng) - np.median(t_bare))
    out["overhead_ms"] = round(ovh, 4)
    out["overhead_pct"] = round(100.0 * ovh / float(np.median(t_bare)), 2)
    out["planes_equal_bare_encode"] = same
    del bare
    torch.cuda.empty_cache()

    # frames for peer 0: a first call with no room gives the exact size
    spec = _lib.FrameSpec(0, 2, d, p, 0, N, 1 if protocol == "crossword" else 0, 5)
    pol_dev = torch.from_numpy(policies.view(np.int32)).to(dev)
    bal_d = torch.from_numpy(bal.view(np.int64)).to(dev)
    off = torch.empty(G, dtype=torch.int64, device=dev)
    fl = torch.empty(G, dtype=torch.int32, device=dev)
    total = torch.empty(1, dtype=torch.int64, device=dev)
    fout = torch.empty(16, dtype=torch.uint8, device=dev)

    def pack(capacity):
        check(ctx.lib.ss_frame_accept_pack_ragged_dev(ctx.h, C.byref(spec), store.data_ptr(), plane_stride, shard_off.data_ptr(),
                                                      ln.data_ptr(), pol_dev.data_ptr(), policies.shape[0],
                                                      pol.data_ptr() if pol is not None else None, 0, slot_out.data_ptr(),
                                                      bal_d.data_ptr(), G, fout.data_ptr(), capacity, off.data_ptr(),
                                                      fl.data_ptr(), total.data_ptr()))

    pack(0)
    ctx.device_status()                                  # clears the overflow bit of the sizing call
    cap = int(total)
    fout = torch.empty(cap, dtype=torch.uint8, device=dev)
    t_fr = []
    for step in range(a.warmup + a.steps):
        e = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        e[0].record()
        pack(cap)
        e[1].record()
        torch.cuda.synchronize()
        if step >= a.warmup:
            t_fr.append(e[0].elapsed_time(e[1]))
    assert ctx.device_status() == 0
    written = int(fl.to(torch.int64).sum())
    out["frame_pack_peer0"] = {**stats(t_fr), "frames_bytes": written, "region_bytes": cap,
                               "GB/s": round(written / (np.median(t_fr) * 1e-3) / 1e9, 1)}
    # a sample of frames against the oracle's encoder
    rng = np.random.default_rng(4)
    sample = np.sort(rng.choice(G, a.sample, replace=False))
    so, offs, fls = shard_off.cpu().numpy(), off.cpu().numpy(), fl.cpu().numpy()
    pidx = (spr - 1) if protocol == "crossword" else np.zeros(G, np.int64)
    ok = 0
    for g in sample:
        mask = int(policies[pidx[g]][0])
        Lg = int(L[g])
        shards = [store[j, int(so[g]):int(so[g]) + Lg].cpu().numpy().tobytes() if (mask >> j) & 1 else None for j in range(5)]
        want = oracle.frame_accept(2, 0, int(bal[g]), d, p, int(lens[g]), shards,
                                   list(map(int, policies[pidx[g]])) if protocol == "crossword" else None, 5)
        got = fout[int(offs[g]):int(offs[g]) + int(fls[g])].cpu().numpy().tobytes()
        ok += got == want
    out["frames_equal_oracle"] = f"{ok}/{len(sample)}"
    eng.close()
    coder.close()
    del store, fout
    torch.cuda.empty_cache()
    return out, same and ok == len(sample)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--groups", type=int, default=1 << 19)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--sample", type=int, default=256)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("engine_ragged_bench needs a CUDA GPU: there is no CPU fallback")
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
    result = {"card": name, "power_limit": power, "groups": G, "steps": a.steps, "payload_bytes": int(lens.astype(np.int64).sum())}
    all_ok = True
    for protocol in ("crossword", "rspaxos"):
        r, ok = run_engine(ctx, protocol, lens, spr, arena, lay["data_off"], a)
        all_ok &= ok
        result[protocol] = r
        for k in ("propose_ragged", "bare_encode", "frame_pack_peer0"):
            v = r[k]
            print(f"{protocol:9s} {k:17s} median {v['median_ms']:8.3f} ms  min {v['min_ms']:8.3f}  max {v['max_ms']:8.3f}  "
                  f"{v['GB/s']:8.1f} GB/s", flush=True)
        print(f"{protocol:9s} overhead of placement + bookkeeping: {r['overhead_ms']:.4f} ms ({r['overhead_pct']:.2f} %); "
              f"planes == bare encode: {r['planes_equal_bare_encode']}; frames == oracle: {r['frames_equal_oracle']}", flush=True)
    print(json.dumps(result), flush=True)
    ctx.close()
    if not all_ok:
        sys.exit("byte comparison failed")


if __name__ == "__main__":
    main()
