"""Per-subscriber accounting on the host side: the declarations of include/bng_b200.h against the bng_acct dtype,
and the C++ counter source and shard routing (tests/host/test_acct_host.cpp, built by build())."""
import ctypes
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "test_acct_host.cpp")
BIN = os.path.join(ROOT, "tests", "host", "test_acct_host")
HOST = os.path.join(ROOT, "bng_b200", "host")
HEADER = os.path.join(ROOT, "include", "bng_b200.h")


def build_acct_host_test():
    deps = [SRC, HEADER] + [os.path.join(HOST, h) for h in ("bng_host.hpp", "bng_shard.hpp")]
    if not os.path.exists(BIN) or any(os.path.getmtime(BIN) < os.path.getmtime(d) for d in deps):
        subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", SRC, "-o", BIN, "-L" + os.path.join(ROOT, "bng_b200"),
                        "-lbng_b200", "-Wl,-rpath,$ORIGIN/../../bng_b200"], check=True)


def _header():
    return re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)


def test_header_declares_accounting():
    src = _header()
    assert re.search(r"int\s+bng_acct_enable\s*\(\s*bng_ctx\s*\*\s*\w*\s*,\s*int\s+\w+\s*,\s*int\s+\w+\s*\)", src)
    assert re.search(r"int\s+bng_acct_read\s*\(\s*bng_ctx\s*\*\s*\w*\s*,\s*const\s+uint32_t\s*\*\s*\w+\s*,\s*uint64_t\s+\w+\s*,"
                     r"\s*bng_acct\s*\*\s*\w+\s*,\s*int32_t\s*\*\s*\w+\s*\)", src)
    assert re.search(r"int64_t\s+bng_acct_dump\s*\(\s*bng_ctx\s*\*\s*\w*\s*,\s*uint32_t\s*\*\s*\w+\s*,\s*bng_acct\s*\*\s*\w+\s*,"
                     r"\s*uint64_t\s+\w+\s*\)", src)
    assert re.search(r"#define\s+BNG_ABI_VERSION\s+2\b", src) and re.search(r"#define\s+BNG_NUM_STATS\s+40\b", src)


def test_struct_layout_matches_dtype():
    from bng_b200 import layouts as L
    body = re.search(r"typedef\s+struct\s+bng_acct\s*\{(.*?)\}\s*bng_acct\s*;", _header(), flags=re.S).group(1)
    fields = []
    for decl in body.split(";"):
        decl = decl.strip()
        if decl:
            assert decl.startswith("uint64_t"), decl
            fields += [f.strip() for f in decl[len("uint64_t"):].split(",")]

    class Acct(ctypes.Structure):
        _fields_ = [(f, ctypes.c_uint64) for f in fields]

    assert ctypes.sizeof(Acct) == L.bng_acct.itemsize == 64
    assert list(L.bng_acct.names) == fields
    for f in fields:
        assert getattr(Acct, f).offset == L.bng_acct.fields[f][1], f


def test_counter_source_and_shard_routing():
    build_acct_host_test()
    r = subprocess.run([BIN, "cpu"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr


@pytest.mark.gpu
def test_counter_source_on_gpu():
    build_acct_host_test()
    r = subprocess.run([BIN, "gpu"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
