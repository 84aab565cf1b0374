"""Lawful intercept on the host side: the bng_li_record declaration of include/bng_b200.h against the layouts.py dtype,
and intercept::ParseCC / PumpRecords of bng_host.hpp on synthetic records (tests/host/test_li_host.cpp, built by
build())."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "test_li_host.cpp")
BIN = os.path.join(ROOT, "tests", "host", "test_li_host")
HEADER = os.path.join(ROOT, "include", "bng_b200.h")


def build_li_host_test():
    deps = [SRC, HEADER, os.path.join(ROOT, "bng_b200", "host", "bng_host.hpp")]
    if not os.path.exists(BIN) or any(os.path.getmtime(BIN) < os.path.getmtime(d) for d in deps):
        subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", SRC, "-o", BIN], check=True)


def _header():
    return re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)


def test_header_declares_interception():
    src = _header()
    for pat in (r"int\s+bng_li_configure\s*\(\s*bng_ctx\s*\*\s*\w*\s*,\s*uint32_t\s+\w+\s*,\s*uint32_t\s+\w+\s*\)",
                r"uint32_t\s+bng_li_record_size\s*\(\s*bng_ctx\s*\*\s*\w*\s*\)",
                r"int\s+bng_li_target_set\s*\(\s*bng_ctx\s*\*\s*\w*\s*,\s*uint32_t\s+\w+\s*,\s*uint32_t\s+\w+\s*\)",
                r"int\s+bng_li_target_del\s*\(\s*bng_ctx\s*\*\s*\w*\s*,\s*uint32_t\s+\w+\s*\)",
                r"int\s+bng_li_drain\s*\(\s*bng_ctx\s*\*\s*\w*\s*,\s*void\s*\*\s*\w+\s*,\s*uint64_t\s+\w+\s*,\s*uint64_t\s*\*\s*\w+\s*\)",
                r"uint64_t\s+bng_li_lost\s*\(\s*bng_ctx\s*\*\s*\w*\s*\)"):
        assert re.search(pat, src), pat
    assert re.search(r"#define\s+BNG_LI_UPLINK\s+0\b", src) and re.search(r"#define\s+BNG_LI_DOWNLINK\s+1\b", src)
    assert re.search(r"#define\s+BNG_ABI_VERSION\s+2\b", src)


def test_record_layout_matches_dtype():
    from bng_b200 import layouts as L
    build_li_host_test()
    out = subprocess.run([BIN, "layout"], capture_output=True, text=True, check=True).stdout.split("\n")
    got = dict(line.split() for line in out if line)
    assert int(got.pop("size")) == L.bng_li_record.itemsize == 64
    assert list(got) == list(L.bng_li_record.names)
    for f, off in got.items():
        assert int(off) == L.bng_li_record.fields[f][1], f
    assert (L.bng_li_record.fields["ts_ns"][1], L.bng_li_record.fields["frame"][1], L.bng_li_record.fields["cap_len"][1],
            L.bng_li_record.fields["dir"][1], L.bng_li_record.fields["prog"][1]) == (0, 16, 32, 36, 38)


def test_pump_cc_parse():
    build_li_host_test()
    r = subprocess.run([BIN, "cpu"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
