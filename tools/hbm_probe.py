#!/usr/bin/env python
"""HBM bandwidth by traffic mix, to read the roofline fractions of kernels that are not 1:1 read:write.
MEASURED_PEAKS.json's hbm_gbs is a COPY figure (one byte read per byte written).  The encode kernels read more than they
write (RS(2,1) 2:1, RS(3,2) 3:2 ...), the Crossword distribute kernel writes five times what it reads.  This probe
times, with CUDA events on one H100:
    write-only   cudaMemsetAsync through ss_dev_memset
    copy  1:1    cudaMemcpyAsync device-to-device through ss_copy_d2d, and torch's copy_ (how MEASURED_PEAKS.json is measured)
    read-mostly  our tally kernel over 16 ack planes (128 B read per 12 B written)
Run on a GPU box:  python tools/hbm_probe.py
"""
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from summerset_b200.api import Context  # noqa: E402
from summerset_b200._lib import check  # noqa: E402

ctx = Context(0)
dev = torch.device("cuda", 0)
N = 1 << 32
a = torch.empty(N, dtype=torch.uint8, device=dev)
b = torch.empty(N, dtype=torch.uint8, device=dev)
a.zero_(); b.zero_()


def timed(fn, nbytes, reps=10):
    fn(); torch.cuda.synchronize()
    best = 1e30
    for _ in range(reps):
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1))
    return nbytes / (best * 1e-3) / 1e9


print("write-only  cudaMemsetAsync 4 GiB            %7.0f GB/s" % timed(lambda: check(ctx.lib.ss_dev_memset(ctx.h, a.data_ptr(), 0, N)), N))
print("write-only  torch fill_ 4 GiB                %7.0f GB/s" % timed(lambda: a.fill_(7), N))
print("copy 1:1    cudaMemcpyAsync d2d 4 GiB        %7.0f GB/s (read + write bytes)" % timed(lambda: check(ctx.lib.ss_copy_d2d(ctx.h, b.data_ptr(), a.data_ptr(), N)), 2 * N))
print("copy 1:1    torch copy_ 4 GiB                %7.0f GB/s (read + write bytes)" % timed(lambda: b.copy_(a), 2 * N))
G, R = 1 << 24, 16
planes = torch.randint(0, 1 << 62, (R, G), dtype=torch.int64, device=dev)
committed = torch.empty(G, dtype=torch.int64, device=dev)
bar = torch.empty(G, dtype=torch.int32, device=dev)
print("read-mostly tally of 16 planes, 2^24 groups  %7.0f GB/s (128 B read : 12 B written per group)"
      % timed(lambda: ctx.tally_planes(planes, 9, True, committed, bar), G * (R * 8 + 12)))
print("read-only   torch sum over 4 GiB             %7.0f GB/s" % timed(lambda: a.view(torch.int32).sum(), N))
