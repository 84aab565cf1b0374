"""Subscriber hand-over on the host side: the declarations of include/bng_b200.h against the Python binding, and the
C++ pins, routes, Router::Move and Router::Drain (tests/host/test_move_host.cpp, built by build())."""
import ctypes
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "test_move_host.cpp")
BIN = os.path.join(ROOT, "tests", "host", "test_move_host")
HOST = os.path.join(ROOT, "bng_b200", "host")
HEADER = os.path.join(ROOT, "include", "bng_b200.h")


def build_move_host_test():
    deps = [SRC, HEADER] + [os.path.join(HOST, h) for h in ("bng_host.hpp", "bng_shard.hpp")]
    if not os.path.exists(BIN) or any(os.path.getmtime(BIN) < os.path.getmtime(d) for d in deps):
        subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", SRC, "-o", BIN, "-L" + os.path.join(ROOT, "bng_b200"),
                        "-lbng_b200", "-Wl,-rpath,$ORIGIN/../../bng_b200"], check=True)


C_TYPES = {"bng_ctx*": ctypes.c_void_p, "constuint32_t*": ctypes.c_void_p, "constuint64_t*": ctypes.c_void_p,
           "constvoid*": ctypes.c_void_p, "void*": ctypes.c_void_p, "uint64_t": ctypes.c_uint64,
           "uint32_t": ctypes.c_uint32, "uint64_t*": ctypes.POINTER(ctypes.c_uint64), "int": ctypes.c_int}


@pytest.mark.parametrize("fn_name", ["bng_sub_export", "bng_sub_import"])
def test_header_declaration_matches_the_binding(fn_name):
    from bng_b200 import dataplane
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    m = re.search(r"(\w+)\s+" + fn_name + r"\s*\(([^)]*)\)\s*;", src)
    assert m, f"{fn_name} is not declared"
    args = []
    for p in m.group(2).split(","):
        p = re.sub(r"\s+", " ", p.strip())
        name = re.search(r"(\w+)$", p)
        args.append(C_TYPES[p[:name.start()].replace(" ", "")])
    if not os.path.exists(dataplane.LIB_PATH):
        pytest.fail("libbng_b200.so is not built")
    fn = getattr(dataplane.load_library(), fn_name)
    assert C_TYPES[m.group(1)] is fn.restype
    assert len(fn.argtypes) == len(args)
    for got, want in zip(fn.argtypes, args):
        assert got is want or (issubclass(got, ctypes._Pointer) and issubclass(want, ctypes._Pointer)
                               and got._type_ is want._type_), (got, want)
    assert fn_name in dataplane.EXPORTED_SYMBOLS
    assert re.search(r"#define\s+BNG_SUB_DETACH\s+1u", src)
    assert dataplane.SUB_DETACH == 1


def test_pins_routes_and_drain_targets():
    build_move_host_test()
    r = subprocess.run([BIN, "cpu"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr


@pytest.mark.gpu
def test_router_move_and_drain_on_two_shards():
    build_move_host_test()
    r = subprocess.run([BIN, "gpu"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
