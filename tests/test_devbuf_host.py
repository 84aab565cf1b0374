"""The owners of the context's grow-only buffers (bng_b200/csrc/devbuf.hpp), on the host alone against a fake CUDA
runtime: failed growths leave no stale error and no freed pointer in use, sets grow all or none, and every allocation
is freed once (tests/host/test_devbuf_host.cpp, built by build())."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "test_devbuf_host.cpp")
FAKE = os.path.join(ROOT, "tests", "host", "fake_cuda")
BIN = os.path.join(ROOT, "tests", "host", "test_devbuf_host")


def build_devbuf_host_test():
    deps = [SRC, os.path.join(FAKE, "cuda_runtime_api.h"), os.path.join(ROOT, "bng_b200", "csrc", "devbuf.hpp")]
    if not os.path.exists(BIN) or any(os.path.getmtime(BIN) < os.path.getmtime(d) for d in deps):
        subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-I", FAKE, SRC, "-o", BIN], check=True)


def test_devbuf():
    build_devbuf_host_test()
    r = subprocess.run([BIN], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
