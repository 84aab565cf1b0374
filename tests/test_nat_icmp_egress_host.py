"""Host side of upstream ICMP error translation: nat::Manager applying
ManagerConfig::EnableUpstreamICMPErrorTranslation at Start, shard::Router::NatICMPErrorsEgressEnable reaching every
shard, and two shards steered by SteerUpstream against one context (tests/host/test_nat_icmp_egress_host.cpp, built by
build())."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "test_nat_icmp_egress_host.cpp")
BIN = os.path.join(ROOT, "tests", "host", "test_nat_icmp_egress_host")
HOST = os.path.join(ROOT, "bng_b200", "host")
HEADER = os.path.join(ROOT, "include", "bng_b200.h")


def build_nat_icmp_egress_host_test():
    deps = [SRC, HEADER] + [os.path.join(HOST, h) for h in ("bng_host.hpp", "bng_shard.hpp")]
    if not os.path.exists(BIN) or any(os.path.getmtime(BIN) < os.path.getmtime(d) for d in deps):
        subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", SRC, "-o", BIN, "-L" + os.path.join(ROOT, "bng_b200"),
                        "-lbng_b200", "-Wl,-rpath,$ORIGIN/../../bng_b200"], check=True)


def test_null_context():
    build_nat_icmp_egress_host_test()
    r = subprocess.run([BIN, "cpu"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr


@pytest.mark.gpu
def test_manager_start_and_router():
    build_nat_icmp_egress_host_test()
    r = subprocess.run([BIN, "gpu"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
