"""Builds and runs tests/cpp/test_rscoding.cpp -- the reference's bitmap.rs / rscoding.rs unit tests restated
against the C++ host mirror (summerset_b200/host/summerset_host.hpp) over the C ABI."""
import os
import subprocess
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent


# The executables are built into a per-module temporary directory, never into the source tree: the tree the suite
# runs from may be read-only, and a binary left there by an earlier run (or another user) must not be reused.
@pytest.fixture(scope="module")
def out_dir(tmp_path_factory):
    from summerset_b200 import build as b
    b.build()
    return tmp_path_factory.mktemp("cpp_host")


@pytest.fixture(scope="module")
def cpp_bin(out_dir):
    exe = out_dir / "test_rscoding"
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.run([gxx, "-std=c++17", "-O1", "-Wall", str(ROOT / "tests" / "cpp" / "test_rscoding.cpp"), "-o", str(exe),
                    f"-L{ROOT / 'summerset_b200'}", "-lsummerset_b200", f"-Wl,-rpath,{ROOT / 'summerset_b200'}"], check=True)
    return exe


@pytest.fixture(scope="module")
def demo_bin(out_dir):
    exe = out_dir / "c_abi_demo"
    gcc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
    subprocess.run([gcc, "-O2", "-Wall", "-std=c11", str(ROOT / "examples" / "c_abi_demo.c"), f"-I{ROOT / 'include'}",
                    f"-L{ROOT / 'summerset_b200'}", "-lsummerset_b200", f"-Wl,-rpath,{ROOT / 'summerset_b200'}",
                    "-o", str(exe)], check=True)
    return exe


def test_cpp_host_mirror_bookkeeping(cpp_bin):
    env = dict(os.environ)
    if not torch.cuda.is_available():
        env["SS_EXPECT_NO_GPU"] = "1"
    r = subprocess.run([str(cpp_bin), "host"], capture_output=True, text=True, env=env, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr


@pytest.mark.gpu
def test_cpp_reference_tests_on_gpu(cpp_bin):
    r = subprocess.run([str(cpp_bin), "gpu"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "gpu: 0 failure(s)" in r.stdout


def test_plain_c_client_compiles_and_refuses_without_gpu(demo_bin):
    """the header is valid C11 and a plain-C client links; without a GPU it gets SS_ERR_NO_DEVICE, never a fallback"""
    if not torch.cuda.is_available():
        r = subprocess.run([str(demo_bin)], capture_output=True, text=True, timeout=60)
        assert r.returncode == 3 and "no CPU fallback" in r.stderr


@pytest.mark.gpu
def test_plain_c_client_on_gpu(demo_bin):
    r = subprocess.run([str(demo_bin)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "bit-exact" in r.stdout and "verify after encode: ok" in r.stdout and "-> -10" in r.stdout


def test_static_code_tables_match_crate_construction(tmp_path):
    """tests/cpp/test_static_codes.cpp: compile-time parity rows of the cluster codes == gf256.hpp's coding matrix
    (host-only, no GPU, no CUDA)."""
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    exe = tmp_path / "test_static_codes"
    subprocess.run([gxx, "-std=c++17", "-O1", "-Wall", str(ROOT / "tests" / "cpp" / "test_static_codes.cpp"), "-o", str(exe)],
                   check=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "0 failure(s)" in r.stdout
