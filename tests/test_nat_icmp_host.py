"""Host side of ICMP error translation: nat::Manager applying ManagerConfig::EnableICMPErrorTranslation at Start,
Directory::SteerDownstream steering an error by the flow it quotes (also under AddressSanitizer), shard::Router's
NatICMPErrorsEnable reaching every shard and its Directory, and two shards steered by SteerDownstream against one
context (tests/host/test_nat_icmp_host.cpp, built by build())."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "test_nat_icmp_host.cpp")
BIN = os.path.join(ROOT, "tests", "host", "test_nat_icmp_host")
HOST = os.path.join(ROOT, "bng_b200", "host")
HEADER = os.path.join(ROOT, "include", "bng_b200.h")


def build_nat_icmp_host_test():
    deps = [SRC, HEADER] + [os.path.join(HOST, h) for h in ("bng_host.hpp", "bng_shard.hpp")]
    if not os.path.exists(BIN) or any(os.path.getmtime(BIN) < os.path.getmtime(d) for d in deps):
        subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", SRC, "-o", BIN, "-L" + os.path.join(ROOT, "bng_b200"),
                        "-lbng_b200", "-Wl,-rpath,$ORIGIN/../../bng_b200"], check=True)


def test_null_context_and_steering():
    build_nat_icmp_host_test()
    r = subprocess.run([BIN, "cpu"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr


def test_steering_reads_nothing_past_the_frame(tmp_path):
    """The CPU checks again, built with AddressSanitizer: steering short ICMP errors held in buffers of exactly their
    length must not read past them."""
    exe = str(tmp_path / "test_nat_icmp_host_asan")
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-fsanitize=address", "-fno-omit-frame-pointer", SRC, "-o", exe,
                    "-L" + os.path.join(ROOT, "bng_b200"), "-lbng_b200", "-Wl,-rpath," + os.path.join(ROOT, "bng_b200")],
                   check=True)
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:protect_shadow_gap=0")
    r = subprocess.run([exe, "cpu"], capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stdout + r.stderr


@pytest.mark.gpu
def test_manager_start_and_router():
    build_nat_icmp_host_test()
    r = subprocess.run([BIN, "gpu"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
