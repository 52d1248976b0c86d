"""Builds libsummerset_b200.so (the C-ABI library) in-tree with nvcc for sm_90a (H100).

Usage: python -m summerset_b200.build [--force] [--verbose]
The .so is git-ignored but travels to the GPU box with the gpurun snapshot.
"""
from __future__ import annotations

import os
import subprocess
import sys
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
OUT = PKG / "libsummerset_b200.so"
SOURCES = ["capi.cu", "rs_kernels.cu", "tally_kernels.cu", "engine.cu", "wire_kernels.cu", "acceptor.cu", "acceptor_recover.cu", "acceptor_stepup.cu", "engine_prepare.cu", "engine_fallback.cu", "follower.cu", "craft_leader.cu", "craft_recon.cu", "craft_election.cu", "craft_stepdown.cu", "craft_recover.cu", "jit.cu"]
HEADERS = ["ss_internal.hpp", "device_common.cuh", "gf256.hpp", "static_codes.hpp", "rs32_decode.cuh", "horner_row_kernels.cuh",
           "wire_common.cuh", "window_ring.cuh", "gossip_walk.cuh", "codeword_wire.cuh", "engine_state.hpp", "prepare_rule.cuh", "acceptor_state.hpp", "follower_state.hpp", "exec_walk.cuh", "craft_frames.cuh",
           "../../include/summerset_b200.h"]
JIT_PARTS = ["device_common.cuh", "static_codes.hpp", "horner_row_kernels.cuh"]     # what NVRTC compiles at run time (jit.cu)
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CCBIN = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
FLAGS = [
    "-O3", "-std=c++17", "-lineinfo",
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-Xcompiler", "-fPIC",
    "-ccbin", CCBIN,
    "--expt-relaxed-constexpr",
]


def needs_build() -> bool:
    if not OUT.exists():
        return True
    t = OUT.stat().st_mtime
    deps = [CSRC / s for s in SOURCES] + [(CSRC / h).resolve() for h in HEADERS] + [Path(__file__)]
    return any(d.stat().st_mtime > t for d in deps)


def gen_jit_source() -> None:
    """csrc/jit_source.inc: the text of the kernels NVRTC specialises per coder, as one C++ raw string literal
    (local #include lines removed: the three headers are concatenated in dependency order)."""
    text = []
    for part in JIT_PARTS:
        for line in (CSRC / part).read_text().splitlines():
            if line.startswith('#include "') or line.startswith("#pragma once"):
                continue
            text.append(line)
    body = 'R"SSJIT(' + "\n".join(text) + '\n)SSJIT"\n'
    out = CSRC / "jit_source.inc"
    if not out.exists() or out.read_text() != body:
        out.write_text(body)


def build(force: bool = False, verbose: bool = False) -> Path:
    if not force and not needs_build():
        return OUT
    gen_jit_source()
    objs = []
    procs = []
    for s in SOURCES:
        o = CSRC / (s + ".o")
        cmd = [NVCC, *FLAGS, "-c", str(CSRC / s), "-o", str(o)]
        if verbose:
            cmd[1:1] = ["-Xptxas", "-v"]
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(str(o))
    failed = False
    for s, pr in procs:
        out, _ = pr.communicate()
        if pr.returncode != 0:
            failed = True
            sys.stderr.write(f"[build] {s} FAILED\n{out}\n")
        elif verbose or out.strip():
            sys.stderr.write(f"[build] {s}\n{out}\n")
    if failed:
        raise RuntimeError("nvcc compilation failed")
    link = [NVCC, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-ccbin", CCBIN,
            "-Xcompiler", "-fPIC", "-o", str(OUT), *objs, "-ldl"]
    r = subprocess.run(link, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("nvcc link failed")
    return OUT


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(p)
