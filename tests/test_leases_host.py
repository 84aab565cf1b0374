"""DHCP lease census and sweep on the host side: the declarations of include/bng_b200.h against the layouts dtypes, and
the C++ dhcp::PoolMonitor thresholds, dhcp::Server::CleanupExpiredLeases loop and shard::Router merge
(tests/host/test_lease_host.cpp, built by build())."""
import ctypes
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "test_lease_host.cpp")
BIN = os.path.join(ROOT, "tests", "host", "test_lease_host")
HOST = os.path.join(ROOT, "bng_b200", "host")
HEADER = os.path.join(ROOT, "include", "bng_b200.h")


def build_lease_host_test():
    deps = [SRC, HEADER] + [os.path.join(HOST, h) for h in ("bng_host.hpp", "bng_shard.hpp", "bng_dhcp_slow.hpp")]
    if not os.path.exists(BIN) or any(os.path.getmtime(BIN) < os.path.getmtime(d) for d in deps):
        subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", SRC, "-o", BIN, "-L" + os.path.join(ROOT, "bng_b200"),
                        "-lbng_b200", "-Wl,-rpath,$ORIGIN/../../bng_b200"], check=True)


def _header():
    return re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)


def test_header_declares_the_calls():
    src = _header()
    assert re.search(r"int\s+bng_dhcp_lease_census\s*\(\s*bng_ctx\s*\*\s*\w*\s*,\s*uint64_t\s+\w+\s*,\s*bng_lease_sum\s*\*\s*\w+\s*,"
                     r"\s*uint32_t\s*\*\s*\w+\s*,\s*bng_lease_pool_use\s*\*\s*\w+\s*,\s*uint64_t\s+\w+\s*\)", src)
    assert re.search(r"int64_t\s+bng_dhcp_lease_sweep\s*\(\s*bng_ctx\s*\*\s*\w*\s*,\s*uint64_t\s+\w+\s*,\s*uint32_t\s+\w+\s*,"
                     r"\s*bng_lease_removed\s*\*\s*\w+\s*,\s*uint64_t\s+\w+\s*,\s*uint64_t\s+\w+\s*\[4\]\s*\)", src)
    assert re.search(r"#define\s+BNG_ABI_VERSION\s+2\b", src)


def test_symbols_are_listed():
    from bng_b200.dataplane import EXPORTED_SYMBOLS
    assert {"bng_dhcp_lease_census", "bng_dhcp_lease_sweep", "bng_lease_table_rebuilds",
            "bng_dhcp_lease_addr_order"} <= set(EXPORTED_SYMBOLS)


def _struct(name):
    body = re.search(r"typedef\s+struct\s+" + name + r"\s*\{(.*?)\}\s*" + name + r"\s*;", _header(), flags=re.S).group(1)
    fields = []
    for decl in body.split(";"):
        decl = decl.strip()
        if decl:
            typ, names = decl.split(None, 1)
            ct = {"uint64_t": ctypes.c_uint64, "uint32_t": ctypes.c_uint32, "uint8_t": ctypes.c_uint8}[typ]
            for f in names.split(","):
                m = re.match(r"\s*(\w+)\s*(?:\[(\d+)\])?\s*$", f)
                fields.append((m.group(1), ct * int(m.group(2)) if m.group(2) else ct))

    class S(ctypes.Structure):
        _fields_ = fields

    return S, fields


@pytest.mark.parametrize("name,size", [("bng_lease_pool_use", 64), ("bng_lease_removed", 64), ("bng_lease_sum", 88)])
def test_struct_layout_matches_dtype(name, size):
    from bng_b200 import layouts as L
    dt = getattr(L, name)
    S, fields = _struct(name)
    assert ctypes.sizeof(S) == dt.itemsize == size
    assert list(dt.names) == [f for f, _ in fields]
    for f, ct in fields:
        assert getattr(S, f).offset == dt.fields[f][1], f
        assert ctypes.sizeof(ct) == dt.fields[f][0].itemsize, f


def test_monitor_cleanup_loop_and_router_merge():
    build_lease_host_test()
    r = subprocess.run([BIN, "cpu"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr


@pytest.mark.gpu
def test_server_loader_monitor_and_router_on_gpu():
    build_lease_host_test()
    r = subprocess.run([BIN, "gpu"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
