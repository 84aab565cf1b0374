"""Host side of antispoof by delegated prefix: antispoof::Manager applying ManagerConfig::ValidateIPv6Prefixes at
Start and shard::Router's AntispoofIPv6PrefixesEnable reaching every shard, with a subscriber's binding and prefixes
routed to one shard (tests/host/test_antispoof_v6_host.cpp, built by build())."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "test_antispoof_v6_host.cpp")
BIN = os.path.join(ROOT, "tests", "host", "test_antispoof_v6_host")
HOST = os.path.join(ROOT, "bng_b200", "host")
HEADER = os.path.join(ROOT, "include", "bng_b200.h")


def build_antispoof_v6_host_test():
    deps = [SRC, HEADER] + [os.path.join(HOST, h) for h in ("bng_host.hpp", "bng_shard.hpp")]
    if not os.path.exists(BIN) or any(os.path.getmtime(BIN) < os.path.getmtime(d) for d in deps):
        subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", SRC, "-o", BIN, "-L" + os.path.join(ROOT, "bng_b200"),
                        "-lbng_b200", "-Wl,-rpath,$ORIGIN/../../bng_b200"], check=True)


def test_null_context():
    build_antispoof_v6_host_test()
    r = subprocess.run([BIN, "cpu"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr


@pytest.mark.gpu
def test_manager_start_and_router():
    build_antispoof_v6_host_test()
    r = subprocess.run([BIN, "gpu"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
