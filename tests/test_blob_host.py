"""The section framing shared by bng_snapshot, bng_delta_export and bng_sub_export (bng_b200/csrc/blob.hpp), on the
host alone: exact bytes, round trips and refusals of malformed sections (tests/host/test_blob_host.cpp, built by
build())."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "test_blob_host.cpp")
BIN = os.path.join(ROOT, "tests", "host", "test_blob_host")


def build_blob_host_test():
    deps = [SRC, os.path.join(ROOT, "bng_b200", "csrc", "blob.hpp")]
    if not os.path.exists(BIN) or any(os.path.getmtime(BIN) < os.path.getmtime(d) for d in deps):
        subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", SRC, "-o", BIN], check=True)


def test_blob_framing():
    build_blob_host_test()
    r = subprocess.run([BIN], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
