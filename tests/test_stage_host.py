"""The control-plane staging (bng_b200/csrc/stage.hpp), on the host alone against a fake CUDA runtime: region offsets,
chunk boundaries, one copy each way and one synchronisation per chunk, the loop stopped at the first failure with the
earlier chunks' outputs delivered, and the counted dump's min(count, cap) (tests/host/test_stage_host.cpp, built by
build())."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "test_stage_host.cpp")
FAKE = os.path.join(ROOT, "tests", "host", "fake_cuda")
BIN = os.path.join(ROOT, "tests", "host", "test_stage_host")


def build_stage_host_test():
    deps = [SRC, os.path.join(FAKE, "cuda_runtime_api.h"), os.path.join(ROOT, "bng_b200", "csrc", "stage.hpp")]
    if not os.path.exists(BIN) or any(os.path.getmtime(BIN) < os.path.getmtime(d) for d in deps):
        subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-I", FAKE, SRC, "-o", BIN], check=True)


def test_stage():
    build_stage_host_test()
    r = subprocess.run([BIN], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
