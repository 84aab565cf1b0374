"""Host side of the DHCPv6 fast path: ebpf::Loader's cache calls, shard::Route::ByValueMAC for dhcpv6_bindings (a
client re-bound under another MAC leaves its old shard) and shard::Router::DHCPv6Enable
(tests/host/test_dhcpv6_host.cpp, built by build())."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "test_dhcpv6_host.cpp")
BIN = os.path.join(ROOT, "tests", "host", "test_dhcpv6_host")
HOST = os.path.join(ROOT, "bng_b200", "host")
HEADER = os.path.join(ROOT, "include", "bng_b200.h")


def build_dhcpv6_host_test():
    deps = [SRC, HEADER] + [os.path.join(HOST, h) for h in ("bng_host.hpp", "bng_shard.hpp")]
    if not os.path.exists(BIN) or any(os.path.getmtime(BIN) < os.path.getmtime(d) for d in deps):
        subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", SRC, "-o", BIN, "-L" + os.path.join(ROOT, "bng_b200"),
                        "-lbng_b200", "-Wl,-rpath,$ORIGIN/../../bng_b200"], check=True)


def test_routing_and_null_context():
    build_dhcpv6_host_test()
    r = subprocess.run([BIN, "cpu"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr


@pytest.mark.gpu
def test_loader_and_router():
    build_dhcpv6_host_test()
    r = subprocess.run([BIN, "gpu"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
