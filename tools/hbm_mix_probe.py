#!/usr/bin/env python
"""The HBM ceiling of the RS(3,2) accept step's traffic mix (read 4096 B, write 2 x 1376 B per group, 2^20 groups),
beside pure-read, pure-write and 1:1 copy at the same shape.  Compiles tools/hbm_mix_probe.cu for sm_90a into a
temporary directory (nothing is written to the tree), prints the card's name, power limit and maximum SM clock
(a read-only nvidia-smi query), then runs the probe on GPU 0.  Usage: python tools/hbm_mix_probe.py
"""
import os
import subprocess
import sys
import tempfile
from pathlib import Path

HERE = Path(__file__).resolve().parent
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.TimeoutExpired) as e:
        return f"unknown ({e})"


def main() -> int:
    with tempfile.TemporaryDirectory() as tmp:
        exe = Path(tmp) / "hbm_mix_probe"
        subprocess.run([NVCC, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-o", str(exe),
                        str(HERE / "hbm_mix_probe.cu")], check=True)
        print(f"# card, power limit, max SM clock: {card()}", flush=True)
        return subprocess.run([str(exe)]).returncode


if __name__ == "__main__":
    sys.exit(main())
