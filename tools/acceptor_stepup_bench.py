"""ss_acceptor_step_up: a new leader's step-up in every group of a 2^20-group RSPaxos acceptor (n = 5, d = 3, me = 1)
with a quarter, half or the whole 64-slot window in flight.

In flight means Accepting: window positions [0, k) of each group, k in {16, 32, 64}, are Accepting at ballot g + 1 and
the rest is null, so every group prepares k instances and writes k PrepareBal records and one Prepare frame.  The state
is installed through the acceptor's views (step-up reads no shard), and restored between launches outside the timed
window.  Timed with CUDA events (median of --steps launches after --warmup), alternated with b.copy_(a) of the same
algorithmic bytes: per group the state words read and written and the per-entry outputs (12 words), per slot the
per-slot arrays written (inst_bal, prep_trigger, source, prep_span) and the record (32-byte cell, group, slot), per frame
the 32-byte cell and its four records.
Check before timing: every verdict and total, and a sample of records and frames compared byte for byte with the
encoders of tests/test_acceptor_prepare.py.

Usage: python tools/acceptor_stepup_bench.py [--groups N] [--steps K] [--warmup W]
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
from summerset_b200.api import Context  # noqa: E402
from summerset_b200.engine import Acceptor  # noqa: E402
from tests.test_acceptor_prepare import prep_frame, wal_cell  # noqa: E402

N, D, ME = 5, 3, 1


def run(ctx, G, k, a, dev):
    acc = Acceptor(ctx, "rspaxos", G, N, ME, D, N)
    acc.accepting.fill_(-1 if k == 64 else (1 << k) - 1)
    bal = torch.arange(1, G + 1, dtype=torch.int64, device=dev)
    acc.bal_max_seen.copy_(bal)
    acc.inst_bal.copy_(bal.repeat_interleave(64))
    nrec = G * k
    wal = torch.empty(nrec * 32, dtype=torch.uint8, device=dev)
    out = torch.empty(G * 32, dtype=torch.uint8, device=dev)
    saved = {n: getattr(acc, n).clone() for n in ("bal_max_seen", "inst_bal", "accepting", "preparing", "source", "prep_trigger",
                                                   "prep_span")}

    def restore():
        for n, t in saved.items():
            getattr(acc, n).copy_(t)

    res = {}
    t_step = timed(lambda: res.update(acc.step_up(wal, nrec, out, G)), restore, a)
    restore()
    res = acc.step_up(wal, nrec, out, G)
    torch.cuda.synchronize()
    tot = [int(x) for x in res["totals"].cpu().numpy()]
    checks = {"verdicts": bool((res["verdict"].cpu().numpy().view(np.uint32) == _lib.SS_ACCEPT_VERDICT_ACCEPTED).all()),
              "totals": tot == [nrec, 32 * nrec, G, 32 * G], "status": ctx.device_status() == 0}
    rng = np.random.default_rng(k)
    ok = True
    cells, frames = wal.cpu().numpy(), out.cpu().numpy()
    rg, rs_ = res["rec_group"].cpu().numpy(), res["rec_slot"].cpu().numpy()
    for idx in rng.choice(nrec, 64, replace=False):
        g, s = int(rg[idx]), int(rs_[idx])
        b = ((g + 1 >> 8) + 1) << 8 | (ME + 1)
        ok &= (g, s) == (idx // k, idx % k) and cells[32 * idx:32 * idx + 32].tobytes() == wal_cell(s, b)
        f = prep_frame(0, ((idx // k + 1 >> 8) + 1) << 8 | (ME + 1))
        ok &= frames[32 * (idx // k):32 * (idx // k) + len(f)].tobytes() == f
    checks["bytes"] = bool(ok)
    nbytes = G * 12 * 8 + nrec * (8 + 8 + 1 + 1 + 32 + 4 + 8) + G * (32 + 4 + 1 + 8 + 4)
    src = torch.empty(nbytes // 2, dtype=torch.uint8, device=dev)
    dst = torch.empty_like(src)
    t_copy = timed(lambda: dst.copy_(src), lambda: None, a)
    gbs = lambda nb, ms: round(nb / (float(np.median(ms)) * 1e-3) / 1e9, 1)
    row = {"k": k, "groups": G, "checks": checks, "step_up": {**stats(t_step), "bytes": nbytes, "GB/s": gbs(nbytes, t_step)},
           "copy": {**stats(t_copy), "bytes": 2 * (nbytes // 2), "GB/s": gbs(2 * (nbytes // 2), t_copy)}}
    for key in ("step_up", "copy"):
        v = row[key]
        print(f"k={k:2d} G={G:8d} {key:8s} median {v['median_ms']:8.3f} ms  {v['bytes'] / 1e9:7.3f} GB  {v['GB/s']:8.1f} GB/s",
              flush=True)
    acc.close()
    del wal, out, src, dst
    torch.cuda.empty_cache()
    return row, all(checks.values())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--groups", type=int, default=1 << 20)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("acceptor_stepup_bench needs a CUDA GPU: there is no CPU fallback")
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    name, power = card()
    clock = max_sm_clock()
    print(f"card: {name}, power limit {power}, max SM clock {clock}", flush=True)
    ctx = Context(0)
    rows, ok = [], True
    for k in (16, 32, 64):
        row, good = run(ctx, a.groups, k, a, dev)
        rows.append(row)
        ok &= good
    print(json.dumps({"card": name, "power_limit": power, "max_sm_clock": clock, "steps": a.steps, "checked": ok, "rows": rows}),
          flush=True)
    ctx.close()
    if not ok:
        sys.exit("acceptor step-up check failed")


if __name__ == "__main__":
    main()
