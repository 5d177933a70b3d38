"""CPU: the owners of device memory, pinned memory, streams and events (csrc/psb_mem.cuh).

The header is built with the host compiler against stub runtime functions whose allocator fails on demand,
and the library's sources are scanned so that every allocation goes through it."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "pocketsphinx_b200", "csrc")
CUDA_INC = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")


def test_owners_after_failed_allocations(tmp_path):
    if not shutil.which("g++") or not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")):
        pytest.skip("needs g++ and the CUDA runtime headers")
    exe = str(tmp_path / "mem_driver")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I", CUDA_INC, "-I", CSRC,
                           os.path.join(ROOT, "tests", "emul", "mem_driver.cpp"), "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.strip() == "ok", out.stdout + out.stderr


OWNED_CALLS = re.compile(r"\b(cudaMalloc|cudaMallocHost|cudaFree|cudaFreeHost|cudaStreamCreate\w*|cudaStreamDestroy|"
                         r"cudaEventCreate\w*|cudaEventDestroy)\b")


def test_only_the_owners_allocate():
    hits = []
    for name in sorted(os.listdir(CSRC)):
        if name == "psb_mem.cuh" or not name.endswith((".cu", ".cuh", ".h")):
            continue
        for i, line in enumerate(open(os.path.join(CSRC, name)), 1):
            if OWNED_CALLS.search(line):
                hits.append("%s:%d: %s" % (name, i, line.strip()))
    assert not hits, "\n".join(hits)
