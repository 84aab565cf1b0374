"""Incremental replication on the host side: the bng_delta_* declarations, the blob framing as ha::ParseDelta reads it
against bng_b200.layouts.parse_delta, and ha::DataplaneSync's sequence handling (tests/host/test_delta_host.cpp, built
by build())."""
import os
import re
import struct
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "test_delta_host.cpp")
BIN = os.path.join(ROOT, "tests", "host", "test_delta_host")
HEADER = os.path.join(ROOT, "include", "bng_b200.h")


def build_delta_host_test():
    deps = [SRC, HEADER, os.path.join(ROOT, "bng_b200", "host", "bng_host.hpp")]
    if not os.path.exists(BIN) or any(os.path.getmtime(BIN) < os.path.getmtime(d) for d in deps):
        subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", SRC, "-o", BIN], check=True)


def test_header_declares_replication():
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    for pat in (r"int\s+bng_delta_enable\s*\(\s*bng_ctx\s*\*\s*\w*\s*,\s*int\s+\w+\s*\)",
                r"int\s+bng_delta_export\s*\(\s*bng_ctx\s*\*\s*\w*\s*,\s*uint64_t\s+\w+\s*,\s*uint32_t\s+\w+\s*,\s*void\s*\*\s*\w+\s*,"
                r"\s*uint64_t\s+\w+\s*,\s*uint64_t\s*\*\s*\w+\s*\)",
                r"int\s+bng_delta_apply\s*\(\s*bng_ctx\s*\*\s*\w*\s*,\s*const\s+void\s*\*\s*\w+\s*,\s*uint64_t\s+\w+\s*\)",
                r"int\s+bng_delta_info\s*\(\s*bng_ctx\s*\*\s*\w*\s*,\s*uint64_t\s*\*\s*\w+\s*,\s*uint64_t\s*\*\s*\w+\s*\)"):
        assert re.search(pat, src), pat
    assert re.search(r"#define\s+BNG_DELTA_FULL\s+1u\b", src) and re.search(r"#define\s+BNG_DELTA_EXACT\s+2u\b", src)
    assert re.search(r"#define\s+BNG_ABI_VERSION\s+2\b", src)


def _blob(seed=7):
    """A delta with a hash-map section (deletions and upserts), a whole array section and an empty one."""
    r = np.random.default_rng(seed)
    secs = [("nat_sessions", 0, 16, 80, 3, 5), ("nat_pool", 1, 4, 16, 0, 256), ("eim_table", 0, 8, 32, 0, 0),
            ("subscriber_acct", 5, 4, 64, 2, 1)]
    out = bytearray(b"BNGDELT1" + struct.pack("<QQQII", 0xDEADBEEF12345678, 41, 42, 2, len(secs)))
    for name, kind, ks, vs, nd, nu in secs:
        out += name.encode().ljust(40, b"\0") + struct.pack("<IIIIQ", kind, ks, vs, nd, nu)
        out += r.integers(0, 256, nd * ks + nu * (ks + vs), dtype=np.uint8).tobytes()
    return bytes(out), secs


def _summary_py(blob):
    from bng_b200 import layouts as L
    h, secs = L.parse_delta(blob)

    def s(b):
        v = 0
        for x in b.reshape(-1).tolist():
            v = (v * 131 + x) & (2**64 - 1)
        return v

    lines = [f"header {h['stream_id']} {h['seq_from']} {h['seq_to']} {h['flags']} {h['sections']}"]
    for name, (kind, dk, uk, uv) in secs.items():
        ks = dk.shape[1] if dk.size else uk.shape[1]
        lines.append(f"{name} {kind} {ks} {uv.shape[1]} {dk.shape[0]} {uk.shape[0]} {s(dk)} "
                     f"{s(np.concatenate([uk.reshape(-1), uv.reshape(-1)]))}")
    return lines


def test_blob_framing_python_and_cpp_agree(tmp_path):
    build_delta_host_test()
    blob, secs = _blob()
    p = tmp_path / "d.bin"
    p.write_bytes(blob)
    got = subprocess.run([BIN, "parse", str(p)], capture_output=True, text=True, check=True).stdout.split("\n")
    assert [x for x in got if x] == _summary_py(blob)
    assert len(got) - 2 == len(secs)
    p.write_bytes(blob[:-1])  # truncated: both refuse
    assert subprocess.run([BIN, "parse", str(p)], capture_output=True, text=True, check=True).stdout.strip() == "invalid"
    from bng_b200 import layouts as L
    try:
        L.parse_delta(blob + b"\0")
        raise AssertionError("trailing bytes accepted")
    except ValueError:
        pass


def test_dataplane_sync_sequence_handling():
    build_delta_host_test()
    r = subprocess.run([BIN, "cpu"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
