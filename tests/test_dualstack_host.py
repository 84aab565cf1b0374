"""Host side of dual-stack attribution: the header's subscriber_ipv6 key against the Python dtype, and the C++
intercept::ParseCC on IPv6 records, the Directory's longest-prefix steering, subscriber_ipv6 routed by value,
Router::Move carrying prefixes and 2- / 8-shard runs (tests/host/test_dualstack_host.cpp, built by build())."""
import os
import re
import subprocess

import numpy as np
import pytest

from bng_b200 import layouts as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "test_dualstack_host.cpp")
BIN = os.path.join(ROOT, "tests", "host", "test_dualstack_host")
HOST = os.path.join(ROOT, "bng_b200", "host")
HEADER = os.path.join(ROOT, "include", "bng_b200.h")


def build_dualstack_host_test():
    deps = [SRC, HEADER] + [os.path.join(HOST, h) for h in ("bng_host.hpp", "bng_shard.hpp")]
    if not os.path.exists(BIN) or any(os.path.getmtime(BIN) < os.path.getmtime(d) for d in deps):
        subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", SRC, "-o", BIN, "-L" + os.path.join(ROOT, "bng_b200"),
                        "-lbng_b200", "-Wl,-rpath,$ORIGIN/../../bng_b200"], check=True)


def test_parse_cc_directory_and_routes():
    build_dualstack_host_test()
    r = subprocess.run([BIN, "cpu"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr


@pytest.mark.gpu
def test_router_move_and_sharded_runs():
    build_dualstack_host_test()
    r = subprocess.run([BIN, "gpu"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr


def test_prefix_lengths_binding():
    from bng_b200 import dataplane
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    assert re.search(r"int\s+bng_ipv6_prefix_lengths\s*\(\s*bng_ctx\s*\*\s*ctx\s*,\s*uint32_t\s*\*\s*counts\s*\)", src)
    assert "bng_ipv6_prefix_lengths" in dataplane.EXPORTED_SYMBOLS


def test_header_key_matches_dtype():
    src = open(os.path.join(ROOT, "include", "bng_b200.h")).read()
    m = re.search(r"typedef struct bng_ipv6_prefix_key \{(.*?)\} bng_ipv6_prefix_key;", src, re.S)
    assert m, "include/bng_b200.h lacks struct bng_ipv6_prefix_key"
    fields = re.findall(r"(uint\d+)_t\s+(\w+)(?:\[(\d+)\])?;", m.group(1))
    assert fields == [("uint32", "prefixlen", ""), ("uint8", "addr", "16")]
    dt = L.bng_ipv6_prefix_key
    assert dt.itemsize == 20 and dt.fields["prefixlen"][1] == 0 and dt.fields["addr"][1] == 4
    assert L.MAP_DTYPES["subscriber_ipv6"] == (dt, ("u1", 4))


def test_key_bytes_are_the_lpm_trie_layout():
    k = np.zeros(1, L.bng_ipv6_prefix_key)
    k["prefixlen"] = 56
    k["addr"] = np.arange(16, dtype=np.uint8)
    b = L.as_bytes(k).reshape(-1)
    assert b[:4].tolist() == [56, 0, 0, 0] and b[4:].tolist() == list(range(16))
