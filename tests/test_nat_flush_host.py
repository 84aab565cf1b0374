"""NAT flow-state flush on the host side: the declaration of include/bng_b200.h against the Python binding, and the
C++ shard routing and manager call (tests/host/test_nat_flush_host.cpp, built by build())."""
import ctypes
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "test_nat_flush_host.cpp")
BIN = os.path.join(ROOT, "tests", "host", "test_nat_flush_host")
HOST = os.path.join(ROOT, "bng_b200", "host")
HEADER = os.path.join(ROOT, "include", "bng_b200.h")


def build_nat_flush_host_test():
    deps = [SRC, HEADER] + [os.path.join(HOST, h) for h in ("bng_host.hpp", "bng_shard.hpp")]
    if not os.path.exists(BIN) or any(os.path.getmtime(BIN) < os.path.getmtime(d) for d in deps):
        subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", SRC, "-o", BIN, "-L" + os.path.join(ROOT, "bng_b200"),
                        "-lbng_b200", "-Wl,-rpath,$ORIGIN/../../bng_b200"], check=True)


C_TYPES = {"bng_ctx*": ctypes.c_void_p, "constuint32_t*": ctypes.c_void_p, "uint64_t": ctypes.c_uint64,
           "uint64_t[3]": ctypes.POINTER(ctypes.c_uint64), "int": ctypes.c_int}


def test_header_declaration_matches_the_binding():
    from bng_b200 import dataplane
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    m = re.search(r"(\w+)\s+bng_nat_flush\s*\(([^)]*)\)\s*;", src)
    assert m, "bng_nat_flush is not declared"
    args = []
    for p in m.group(2).split(","):
        p = re.sub(r"\s+", " ", p.strip())
        name = re.search(r"(\w+)\s*(\[\d+\])?$", p)
        typ = (p[:name.start()] + (name.group(2) or "")).replace(" ", "")
        args.append(C_TYPES[typ])
    lib = dataplane.load_library() if os.path.exists(dataplane.LIB_PATH) else None
    if lib is None:
        pytest.fail("libbng_b200.so is not built")
    fn = lib.bng_nat_flush
    assert C_TYPES[m.group(1)] is fn.restype
    assert len(fn.argtypes) == len(args)
    for got, want in zip(fn.argtypes, args):
        assert got is want or (issubclass(got, ctypes._Pointer) and issubclass(want, ctypes._Pointer)
                               and got._type_ is want._type_), (got, want)
    assert "bng_nat_flush" in dataplane.EXPORTED_SYMBOLS


def test_shard_grouping():
    build_nat_flush_host_test()
    r = subprocess.run([BIN, "cpu"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr


@pytest.mark.gpu
def test_router_and_manager_on_two_shards():
    build_nat_flush_host_test()
    r = subprocess.run([BIN, "gpu"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
