"""TEST INFRASTRUCTURE — ctypes front-end to the CPU oracles.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline /
``--impl reference`` leg may import this module.  The product path
(``bng_b200``) never does.

Two libraries export the same ``ora_*`` API (oracle/oracle_api.h):

* ``oracle/_ref/libbng_ref.so``  — the reference's own eBPF C sources compiled
  natively (kind ``"reference"``); built only where ``/root/reference`` exists,
  but the built file travels with the repository snapshot.
* ``oracle/libbng_port.so``      — the plain-C restatement (kind ``"port"``).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF_LIB = os.path.join(HERE, "_ref", "libbng_ref.so")
PORT_LIB = os.path.join(HERE, "libbng_port.so")


class _Batch(C.Structure):
    _fields_ = [
        ("pkts", C.c_void_p),
        ("off16", C.c_void_p),
        ("len", C.c_void_p),
        ("verdict", C.c_void_p),
        ("priority", C.c_void_p),
        ("n", C.c_uint32),
        ("stride", C.c_uint32),
        ("now_ns", C.c_uint64),
        ("now_v", C.c_void_p),
    ]


class _Info(C.Structure):
    _fields_ = [
        ("type", C.c_uint32),
        ("key_size", C.c_uint32),
        ("value_size", C.c_uint32),
        ("max_entries", C.c_uint32),
        ("count", C.c_uint64),
    ]


def build(which: str = "all") -> None:
    """Compile the oracle libraries (``make -C oracle``)."""
    subprocess.run(["make", "-s", "-C", HERE, which], check=True)


def available(kind: str) -> bool:
    return os.path.exists(REF_LIB if kind == "reference" else PORT_LIB)


class Oracle:
    """One instance of an oracle library.  The map state lives in the library, so every Oracle built from the same
    file shares it; `path` names a copy of the library to get a second, independent state."""

    def __init__(self, kind: str = "reference", path: str | None = None):
        path = path or (REF_LIB if kind == "reference" else PORT_LIB)
        if not os.path.exists(path):
            raise FileNotFoundError(f"oracle library missing: {path} (run `make -C oracle`)")
        self.kind = kind
        self.lib = lib = C.CDLL(path)
        lib.ora_impl.restype = C.c_char_p
        lib.ora_map_name.restype = C.c_char_p
        lib.ora_prog_name.restype = C.c_char_p
        lib.ora_map_id.argtypes = [C.c_char_p]
        lib.ora_prog_id.argtypes = [C.c_char_p]
        lib.ora_map_get_info.argtypes = [C.c_int, C.POINTER(_Info)]
        lib.ora_map_update.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_uint64]
        lib.ora_map_update_batch.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64]
        lib.ora_map_lookup.argtypes = [C.c_int, C.c_void_p, C.c_void_p]
        lib.ora_map_delete.argtypes = [C.c_int, C.c_void_p]
        lib.ora_map_dump.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_uint64]
        lib.ora_map_dump.restype = C.c_uint64
        lib.ora_prog_run.argtypes = [C.c_int, C.POINTER(_Batch)]
        lib.ora_events_drain.argtypes = [C.c_int, C.c_void_p, C.c_uint64]
        lib.ora_events_drain.restype = C.c_uint64
        lib.ora_event_size.argtypes = [C.c_int]
        lib.ora_event_size.restype = C.c_uint32
        lib.ora_arena_alloc.argtypes = [C.c_size_t]
        lib.ora_arena_alloc.restype = C.c_void_p
        lib.ora_arena_free.argtypes = [C.c_void_p, C.c_size_t]
        lib.ora_reset()
        self.impl = lib.ora_impl().decode()
        self._arenas = []

    # ---- maps ----
    def reset(self) -> None:
        self.lib.ora_reset()

    def map_names(self):
        return [self.lib.ora_map_name(i).decode() for i in range(self.lib.ora_map_count_all())]

    def map_id(self, name: str) -> int:
        i = self.lib.ora_map_id(name.encode())
        if i < 0:
            raise KeyError(name)
        return i

    def map_info(self, name: str) -> dict:
        inf = _Info()
        self.lib.ora_map_get_info(self.map_id(name), C.byref(inf))
        return {f: getattr(inf, f) for f, _ in _Info._fields_}

    @staticmethod
    def _buf(b):
        if isinstance(b, np.ndarray):
            b = np.ascontiguousarray(b)
            return b, b.ctypes.data
        bb = (C.c_char * len(b)).from_buffer_copy(bytes(b))
        return bb, C.addressof(bb)

    def update(self, name: str, key, val, flags: int = 0) -> int:
        k, kp = self._buf(key)
        v, vp = self._buf(val)
        return self.lib.ora_map_update(self.map_id(name), kp, vp, flags)

    def update_batch(self, name: str, keys: np.ndarray, vals: np.ndarray, flags: int = 0) -> int:
        keys = np.ascontiguousarray(keys)
        vals = np.ascontiguousarray(vals)
        n = keys.shape[0]
        return self.lib.ora_map_update_batch(self.map_id(name), keys.ctypes.data, vals.ctypes.data, n, flags)

    def lookup(self, name: str, key):
        inf = self.map_info(name)
        k, kp = self._buf(key)
        out = np.zeros(inf["value_size"], dtype=np.uint8)
        r = self.lib.ora_map_lookup(self.map_id(name), kp, out.ctypes.data)
        return None if r else out

    def delete(self, name: str, key) -> int:
        k, kp = self._buf(key)
        return self.lib.ora_map_delete(self.map_id(name), kp)

    def dump(self, name: str):
        """(keys[n,key_size], vals[n,value_size]) as uint8, sorted by key bytes."""
        inf = self.map_info(name)
        cap = max(int(inf["count"]), 1)
        keys = np.zeros((cap, max(inf["key_size"], 1)), dtype=np.uint8)
        vals = np.zeros((cap, max(inf["value_size"], 1)), dtype=np.uint8)
        n = self.lib.ora_map_dump(self.map_id(name), keys.ctypes.data, vals.ctypes.data, cap)
        keys, vals = keys[:n], vals[:n]
        return sort_kv(keys, vals)

    def drain(self, name: str) -> np.ndarray:
        mid = self.map_id(name)
        sz = self.lib.ora_event_size(mid)
        inf = self.map_info(name)
        n = int(inf["count"])
        if not n or not sz:
            return np.zeros((0, sz or 1), dtype=np.uint8)
        out = np.zeros((n, sz), dtype=np.uint8)
        got = self.lib.ora_events_drain(mid, out.ctypes.data, n)
        return out[:got]

    # ---- packets ----
    def arena(self, nbytes: int) -> np.ndarray:
        """uint8 array backed by memory below 4 GiB (in-place runs for the reference build)."""
        nbytes = max(int(nbytes), 16)
        p = self.lib.ora_arena_alloc(nbytes)
        if not p:
            raise MemoryError("MAP_32BIT arena allocation failed")
        arr = np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(p))
        self._arenas.append((p, nbytes))
        return arr

    def free_arenas(self) -> None:
        for p, n in self._arenas:
            self.lib.ora_arena_free(p, n)
        self._arenas = []

    def prog_names(self):
        out = []
        i = 0
        while True:
            nm = self.lib.ora_prog_name(i)
            if nm is None:
                break
            out.append(nm.decode())
            i += 1
        return out

    def run(self, prog: str, pkts: np.ndarray, lens: np.ndarray, now_ns: int, off16=None, stride: int = 0,
            priority=None, now_v=None):
        """Run ``prog`` over the batch IN PLACE (pkts, lens and priority are modified).

        Returns the verdict array (uint8[n]).
        """
        pid = self.lib.ora_prog_id(prog.encode())
        if pid < 0:
            raise KeyError(prog)
        n = int(lens.shape[0])
        assert pkts.dtype == np.uint8 and pkts.flags.c_contiguous
        assert lens.dtype == np.uint32 and lens.flags.c_contiguous
        verdict = np.zeros(n, dtype=np.uint8)
        b = _Batch()
        b.pkts = pkts.ctypes.data
        if off16 is not None:
            assert off16.dtype == np.uint32 and off16.flags.c_contiguous
            b.off16 = off16.ctypes.data
        else:
            b.off16 = None
            assert stride > 0
        b.len = lens.ctypes.data
        b.verdict = verdict.ctypes.data
        if priority is not None:
            assert priority.dtype == np.uint32
            b.priority = priority.ctypes.data
        else:
            b.priority = None
        b.n = n
        b.stride = stride
        b.now_ns = now_ns
        if now_v is not None:
            assert now_v.dtype == np.uint64 and now_v.flags.c_contiguous and now_v.shape[0] == n
            b.now_v = now_v.ctypes.data
        else:
            b.now_v = None
        r = self.lib.ora_prog_run(pid, C.byref(b))
        if r:
            raise RuntimeError(f"ora_prog_run({prog}) = {r}")
        return verdict


def sort_kv(keys: np.ndarray, vals: np.ndarray):
    """Canonical order for comparing table dumps as key->value sets."""
    if keys.shape[0] == 0:
        return keys, vals
    order = np.lexsort(keys.T[::-1])
    return keys[order], vals[order]
