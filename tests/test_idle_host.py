"""Idle detection on the host side: the declarations of include/bng_b200.h against the bng_idle dtype, and the C++
idle::Monitor and shard fan-out (tests/host/test_idle_host.cpp, built by build())."""
import ctypes
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "test_idle_host.cpp")
BIN = os.path.join(ROOT, "tests", "host", "test_idle_host")
HOST = os.path.join(ROOT, "bng_b200", "host")
HEADER = os.path.join(ROOT, "include", "bng_b200.h")


def build_idle_host_test():
    deps = [SRC, HEADER] + [os.path.join(HOST, h) for h in ("bng_host.hpp", "bng_shard.hpp")]
    if not os.path.exists(BIN) or any(os.path.getmtime(BIN) < os.path.getmtime(d) for d in deps):
        subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", SRC, "-o", BIN, "-L" + os.path.join(ROOT, "bng_b200"),
                        "-lbng_b200", "-Wl,-rpath,$ORIGIN/../../bng_b200"], check=True)


def _header():
    return re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)


def test_header_declares_idle_detection():
    src = _header()
    ctx = r"\s*bng_ctx\s*\*\s*\w*\s*,"
    assert re.search(r"int\s+bng_idle_enable\s*\(" + ctx + r"\s*int\s+\w+\s*,\s*int\s+\w+\s*\)", src)
    assert re.search(r"int\s+bng_idle_timeout_set\s*\(" + ctx + r"\s*const\s+uint32_t\s*\*\s*\w+\s*,\s*const\s+uint32_t\s*\*\s*\w+\s*,"
                     r"\s*uint64_t\s+\w+\s*,\s*int32_t\s*\*\s*\w+\s*\)", src)
    assert re.search(r"int\s+bng_idle_read\s*\(" + ctx + r"\s*const\s+uint32_t\s*\*\s*\w+\s*,\s*uint64_t\s+\w+\s*,"
                     r"\s*bng_idle\s*\*\s*\w+\s*,\s*int32_t\s*\*\s*\w+\s*\)", src)
    assert re.search(r"int64_t\s+bng_idle_scan\s*\(" + ctx + r"\s*uint64_t\s+\w+\s*,\s*uint32_t\s+\w+\s*,\s*uint32_t\s+\w+\s*,"
                     r"\s*uint32_t\s*\*\s*\w+\s*,\s*bng_idle\s*\*\s*\w+\s*,\s*uint64_t\s+\w+\s*\)", src)
    from bng_b200 import layouts as L
    for name, v in (("UP", L.IDLE_UP), ("DOWN", L.IDLE_DOWN), ("STARTED", L.IDLE_STARTED), ("NEVER", L.IDLE_NEVER)):
        m = re.search(r"#define\s+BNG_IDLE_" + name + r"\s+(0x[0-9A-Fa-f]+|\d+)u?\b", src)
        assert m and int(m.group(1), 0) == v, name
    assert re.search(r"#define\s+BNG_ABI_VERSION\s+2\b", src)


def test_struct_layout_matches_dtype():
    from bng_b200 import layouts as L
    body = re.search(r"typedef\s+struct\s+bng_idle\s*\{(.*?)\}\s*bng_idle\s*;", _header(), flags=re.S).group(1)
    fields = []
    for decl in body.split(";"):
        decl = decl.strip()
        if decl:
            typ, names = decl.split(None, 1)
            ct = {"uint64_t": ctypes.c_uint64, "uint32_t": ctypes.c_uint32}[typ]
            fields += [(f.strip(), ct) for f in names.split(",")]

    class Idle(ctypes.Structure):
        _fields_ = fields

    assert ctypes.sizeof(Idle) == L.bng_idle.itemsize == 32
    assert list(L.bng_idle.names) == [f for f, _ in fields]
    for f, ct in fields:
        assert getattr(Idle, f).offset == L.bng_idle.fields[f][1], f
        assert ctypes.sizeof(ct) == L.bng_idle.fields[f][0].itemsize, f


def test_monitor_and_shard_fanout():
    build_idle_host_test()
    r = subprocess.run([BIN, "cpu"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr


@pytest.mark.gpu
def test_monitor_and_router_on_gpu():
    build_idle_host_test()
    r = subprocess.run([BIN, "gpu"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
