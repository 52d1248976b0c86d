#!/usr/bin/env python
"""A/B of the fused RS(3,2) accept-step kernels on the cfg3 shape (2^20 groups x 4096 B, 5 replicas, 4-of-5 tally),
one GPU: the bulk-copy kernel (variant bit 18) against the row kernel (variant 0, the default), alternated ROUNDS times
in one process so that both see the same card, clocks and neighbours.  Per run:
    kernel ms   CUDA events around each launch, averaged over STEPS launches
    step ms     one event pair around STEPS back-to-back launches, divided by STEPS (how bench.py times a step)
Reports median / min / max of both per kernel, the card's name and power limit, and checks that the two kernels' outputs
are identical byte for byte: both parity planes, the commit words and commit_bar of every group, with and without the
tally.  Extra variants to time (tuning) may be given as arguments.  Usage: python tools/accept_ab.py [variant ...]
"""
import statistics
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from summerset_b200.api import SS_RS_OUT_PADDED16, Context, ReedSolomon  # noqa: E402
from summerset_b200._lib import check  # noqa: E402

N, DATA_LEN, R, THRESH, D, P = 1 << 20, 4096, 5, 4, 3, 2
ROUNDS, STEPS, WARMUP = 6, 20, 5
BULK = 1 << 18


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.TimeoutExpired) as e:
        return f"unknown ({e})"


def main() -> int:
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    ctx = Context(0)
    rs = ReedSolomon(ctx, D, P)
    L, ds, ps = rs.parity_layout(DATA_LEN, N)
    gen = torch.Generator(device=dev); gen.manual_seed(20261015)
    data = torch.randint(0, 256, (N, DATA_LEN), dtype=torch.uint8, device=dev, generator=gen)
    u = torch.randint(0, 256, (R, N, 64), dtype=torch.uint8, device=dev, generator=gen) < 230
    w = torch.tensor([1 << i for i in range(63)] + [-(1 << 63)], dtype=torch.int64, device=dev)
    planes = (u.to(torch.int64) * w).sum(dim=2)
    planes[0] = -1
    del u
    out = {}
    for v in (BULK, 0):
        out[v] = (torch.full((P, N, ds), 0xA5, dtype=torch.uint8, device=dev), torch.zeros(N, dtype=torch.int64, device=dev),
                  torch.zeros(N, dtype=torch.int32, device=dev))

    def launch(v, tally=True):
        par, com, bar = out[v if v in out else BULK]
        rs.set_variant(v)
        if tally:
            check(ctx.lib.ss_accept_step_fused_dev(rs.h, data.data_ptr(), DATA_LEN, DATA_LEN, N, par.data_ptr(), ps, ds,
                                                   SS_RS_OUT_PADDED16, planes.data_ptr(), R, THRESH, com.data_ptr(), bar.data_ptr()))
        else:
            check(ctx.lib.ss_rs_encode_uniform_dev(rs.h, data.data_ptr(), DATA_LEN, DATA_LEN, N, par.data_ptr(), ps, ds,
                                                   SS_RS_OUT_PADDED16))

    def run(v):
        for _ in range(WARMUP):
            launch(v)
        torch.cuda.synchronize()
        a = torch.cuda.Event(enable_timing=True); b = torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(STEPS):
            launch(v)
        b.record()
        torch.cuda.synchronize()
        step = a.elapsed_time(b) / STEPS
        evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(STEPS)]
        for e0, e1 in evs:
            e0.record(); launch(v); e1.record()
        torch.cuda.synchronize()
        return sum(e0.elapsed_time(e1) for e0, e1 in evs) / STEPS, step

    print(f"# card, power limit, max SM clock: {card()}", flush=True)
    print(f"# cfg3 shape: {N} groups x {DATA_LEN} B, RS({D},{P}), {R} replicas, tally {THRESH} of {R}; "
          f"{ROUNDS} alternated rounds of {STEPS} launches per kernel", flush=True)
    variants = [BULK, 0] + [int(a, 0) for a in sys.argv[1:]]
    times = {v: [] for v in variants}
    names = {}
    for r in range(ROUNDS):
        for v in (variants if r % 2 == 0 else variants[::-1]):
            k, s = run(v)
            times[v].append((k, s))
            names[v] = rs.last_kernel()
            print(f"round {r}  variant {v:#8x}  {names[v]:34s} kernel {k:7.4f} ms  step {s:7.4f} ms", flush=True)
    alg = N * ((D + P) * L + (R + 1) * 8 + 4)
    print(f"\n{'variant':>10s} {'kernel':34s} {'kernel ms med/min/max':>26s} {'step ms med/min/max':>26s} {'GB/s (med kernel)':>18s}")
    for v in variants:
        ks = [t[0] for t in times[v]]; ss = [t[1] for t in times[v]]
        km = statistics.median(ks)
        print(f"{v:#10x} {names[v]:34s} {km:8.4f} {min(ks):8.4f} {max(ks):8.4f} "
              f"{statistics.median(ss):8.4f} {min(ss):8.4f} {max(ss):8.4f} {alg / (km * 1e-3) / 1e9:18.1f}")
    new_k = [t[0] for t in times[BULK]]; old_k = [t[0] for t in times[0]]
    print(f"\nbulk vs row: median kernel time {statistics.median(new_k) / statistics.median(old_k) - 1:+.2%}; "
          f"worst bulk run {max(new_k):.4f} ms vs best row run {min(old_k):.4f} ms")

    # ---- outputs: every byte of both kernels' results ----
    for t in out.values():
        t[0].fill_(0xA5); t[1].zero_(); t[2].zero_()
    launch(BULK); launch(0)
    torch.cuda.synchronize()
    same = [torch.equal(out[BULK][i], out[0][i]) for i in range(3)]
    print(f"with tally: parity planes identical = {same[0]}, commit words identical = {same[1]}, commit_bar identical = {same[2]}")
    for t in out.values():
        t[0].fill_(0x5A)
    launch(BULK, tally=False); launch(0, tally=False)
    torch.cuda.synchronize()
    same_nt = torch.equal(out[BULK][0], out[0][0])
    print(f"without tally: parity planes identical = {same_nt}")
    rs.set_variant(0)
    return 0 if all(same) and same_nt else 1


if __name__ == "__main__":
    sys.exit(main())
