"""ctypes binding of the C ABI in ``include/bng_b200.h`` (libbng_b200.so).

This is plumbing for tests, ``bench.py`` and Python callers; the product is
the shared library.  There is no CPU path: if the library or a CUDA device is
missing, construction raises.
"""
from __future__ import annotations

import ctypes as C
import errno
import os

import numpy as np

from .layouts import as_bytes, bng_acct, bng_idle, bng_li_record, bng_nat_pub_use, bng_nat_sub_use, bng_nat_usage_sum
from .layouts import bng_ipv6_prefix_key, bng_lease_pool_use, bng_lease_removed, bng_lease_sum

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("BNG_B200_LIB") or os.path.join(HERE, "libbng_b200.so")  # override: A/B builds

MEM_DEVICE, MEM_HOST = 0, 1
ANY, NOEXIST, EXIST = 0, 1, 2
DELTA_FULL, DELTA_EXACT = 1, 2
SUB_DETACH = 1

PROGRAMS = (
    "antispoof_ingress", "qos_egress_prog", "qos_ingress_prog", "nat44_egress", "nat44_ingress",
    "nat44_hairpin_xdp", "dhcp_fastpath_prog", "pipeline_up", "pipeline_tc",
)


class OpenOpts(C.Structure):
    _fields_ = [
        ("struct_size", C.c_uint32), ("device", C.c_int32), ("max_batch", C.c_uint32),
        ("max_subscribers", C.c_uint32), ("max_nat_sessions", C.c_uint32), ("max_eim_mappings", C.c_uint32),
        ("event_capacity", C.c_uint32), ("rank", C.c_uint32), ("world", C.c_uint32),
    ]


class MapInfo(C.Structure):
    _fields_ = [
        ("type", C.c_uint32), ("key_size", C.c_uint32), ("value_size", C.c_uint32),
        ("max_entries", C.c_uint32), ("count", C.c_uint64),
    ]


class Batch(C.Structure):
    _fields_ = [
        ("pkts", C.c_void_p), ("off16", C.c_void_p), ("len", C.c_void_p), ("verdict", C.c_void_p),
        ("priority", C.c_void_p), ("n", C.c_uint32), ("stride", C.c_uint32), ("now_ns", C.c_uint64),
        ("mem", C.c_uint32), ("arena_bytes", C.c_uint32), ("now_ns_v", C.c_void_p),
    ]


_lib = None


def load_library() -> C.CDLL:
    """Load libbng_b200.so and declare prototypes.  Raises if it was not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: build it with `make -C bng_b200/csrc` "
            "(or __graft_entry__.build()); bng_b200 has no CPU fallback")
    lib = C.CDLL(LIB_PATH)
    vp, i32, u32, u64 = C.c_void_p, C.c_int, C.c_uint32, C.c_uint64
    protos = {
        "bng_open": ([C.POINTER(OpenOpts)], vp),
        "bng_close": ([vp], i32),
        "bng_last_error": ([vp], C.c_char_p),
        "bng_abi_version": ([], u32),
        "bng_map_id": ([vp, C.c_char_p], i32),
        "bng_map_get_info": ([vp, i32, C.POINTER(MapInfo)], i32),
        "bng_map_update": ([vp, i32, vp, vp, u64], i32),
        "bng_map_update_batch": ([vp, i32, vp, vp, u64, u64], i32),
        "bng_map_lookup": ([vp, i32, vp, vp], i32),
        "bng_map_delete": ([vp, i32, vp], i32),
        "bng_map_update_staged": ([vp, i32, vp, vp], i32),
        "bng_staged_info": ([vp, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64)], i32),
        "bng_comm_unique_id": ([vp, u64], i32),
        "bng_comm_init": ([vp, vp, u32, u32], i32),
        "bng_sync_reduce": ([vp, vp], i32),
        "bng_sweep": ([vp, u64, C.POINTER(u64)], i32),
        "bng_snapshot": ([vp, vp, u64], C.c_int64),
        "bng_restore": ([vp, vp, u64], i32),
        "bng_lru_evictions": ([vp], u64),
        "bng_table_rebuilds": ([vp], u64),
        "bng_map_dump": ([vp, i32, vp, vp, u64], C.c_int64),
        "bng_map_clear": ([vp, i32], i32),
        "bng_prog_id": ([vp, C.c_char_p], i32),
        "bng_prog_run": ([vp, i32, C.POINTER(Batch)], i32),
        "bng_sync": ([vp], i32),
        "bng_stream": ([vp], vp),
        "bng_events_drain": ([vp, i32, vp, u64, C.POINTER(u64)], i32),
        "bng_event_size": ([vp, i32], u32),
        "bng_shard_of_mac": ([u64, u32], u32),
        "bng_stats_device_ptr": ([vp, C.POINTER(vp), C.POINTER(u32)], i32),
        "bng_launch_count": ([vp], u64),
        "bng_ipv6_prefix_lengths": ([vp, vp], i32),
        "bng_qos_ipv6_enable": ([vp, i32], i32),
        "bng_antispoof_ipv6_prefixes_enable": ([vp, i32], i32),
        "bng_nat_icmp_errors_enable": ([vp, i32], i32),
        "bng_nat_icmp_errors_egress_enable": ([vp, i32], i32),
        "bng_dhcpv6_enable": ([vp, i32], i32),
        "bng_nd_enable": ([vp, i32], i32),
        "bng_lru_overflow": ([vp], u64),
        "bng_events_lost": ([vp], u64),
        "bng_prof_enable": ([vp, i32], i32),
        "bng_prof_read": ([vp, C.c_char_p, u64], C.c_int64),
        "bng_host_alloc": ([C.c_size_t], vp),
        "bng_host_free": ([vp], None),
        "bng_acct_enable": ([vp, i32, i32], i32),
        "bng_acct_read": ([vp, vp, u64, vp, vp], i32),
        "bng_acct_dump": ([vp, vp, vp, u64], C.c_int64),
        "bng_nat_flush": ([vp, vp, u64, u64, C.POINTER(u64)], i32),
        "bng_li_configure": ([vp, u32, u32], i32),
        "bng_li_record_size": ([vp], u32),
        "bng_li_target_set": ([vp, u32, u32], i32),
        "bng_li_target_del": ([vp, u32], i32),
        "bng_li_drain": ([vp, vp, u64, C.POINTER(u64)], i32),
        "bng_li_lost": ([vp], u64),
        "bng_delta_enable": ([vp, i32], i32),
        "bng_delta_export": ([vp, u64, u32, vp, u64, C.POINTER(u64)], i32),
        "bng_delta_apply": ([vp, vp, u64], i32),
        "bng_delta_info": ([vp, C.POINTER(u64), C.POINTER(u64)], i32),
        "bng_idle_enable": ([vp, i32, i32], i32),
        "bng_idle_timeout_set": ([vp, vp, vp, u64, vp], i32),
        "bng_idle_read": ([vp, vp, u64, vp, vp], i32),
        "bng_idle_scan": ([vp, u64, u32, u32, vp, vp, u64], C.c_int64),
        "bng_nat_usage": ([vp, u32, vp, vp, vp, u64, vp, vp, u64], i32),
        "bng_dhcp_lease_census": ([vp, u64, vp, vp, vp, u64], i32),
        "bng_dhcp_lease_sweep": ([vp, u64, u32, vp, u64, vp], C.c_int64),
        "bng_lease_table_rebuilds": ([vp], u64),
        "bng_dhcp_lease_addr_order": ([vp, u32], i32),
        "bng_sub_export": ([vp, vp, u64, vp, u64, u32, vp, u64, C.POINTER(u64)], i32),
        "bng_sub_import": ([vp, vp, u64], i32),
    }
    for name, (args, res) in protos.items():
        fn = getattr(lib, name)
        fn.argtypes = args
        fn.restype = res
    _lib = lib
    return lib


EXPORTED_SYMBOLS = (
    "bng_open", "bng_close", "bng_last_error", "bng_abi_version", "bng_map_id", "bng_map_get_info",
    "bng_map_update", "bng_map_update_batch", "bng_map_lookup", "bng_map_delete", "bng_map_clear", "bng_map_dump",
    "bng_prog_id",
    "bng_prog_run", "bng_sync", "bng_stream", "bng_events_drain", "bng_event_size", "bng_shard_of_mac",
    "bng_stats_device_ptr", "bng_launch_count", "bng_lru_overflow", "bng_events_lost", "bng_prof_enable",
    "bng_prof_read", "bng_host_alloc", "bng_host_free", "bng_map_update_staged", "bng_staged_info",
    "bng_comm_unique_id", "bng_comm_init", "bng_sync_reduce", "bng_sweep", "bng_lru_evictions", "bng_snapshot", "bng_restore", "bng_table_rebuilds",
    "bng_acct_enable", "bng_acct_read", "bng_acct_dump", "bng_nat_flush",
    "bng_li_configure", "bng_li_record_size", "bng_li_target_set", "bng_li_target_del", "bng_li_drain", "bng_li_lost",
    "bng_delta_enable", "bng_delta_export", "bng_delta_apply", "bng_delta_info",
    "bng_idle_enable", "bng_idle_timeout_set", "bng_idle_read", "bng_idle_scan", "bng_nat_usage",
    "bng_dhcp_lease_census", "bng_dhcp_lease_sweep", "bng_lease_table_rebuilds", "bng_dhcp_lease_addr_order",
    "bng_sub_export", "bng_sub_import", "bng_ipv6_prefix_lengths", "bng_qos_ipv6_enable",
    "bng_nat_icmp_errors_enable", "bng_antispoof_ipv6_prefixes_enable", "bng_dhcpv6_enable", "bng_nd_enable",
    "bng_nat_icmp_errors_egress_enable",
)


class BngError(OSError):
    pass


def _addr_words(addrs) -> np.ndarray:
    """Subscriber addresses as u32 words holding the 4 key bytes: from u8[n, 4] key bytes or u32[n]."""
    a = np.asarray(addrs)
    return np.ascontiguousarray(a).view("<u4").reshape(-1) if a.dtype == np.uint8 else np.ascontiguousarray(a, "<u4").reshape(-1)


def _ptr(x):
    """Device/host address of a numpy array, torch tensor, int or None."""
    if x is None:
        return None
    if isinstance(x, int):
        return x
    if isinstance(x, np.ndarray):
        return x.ctypes.data
    if hasattr(x, "data_ptr"):
        return x.data_ptr()
    raise TypeError(type(x))


def shard_of_mac(mac_key: int, world: int) -> int:
    return load_library().bng_shard_of_mac(mac_key, world)


class Dataplane:
    """One dataplane context on one GPU (``bng_open`` .. ``bng_close``)."""

    def __init__(self, device: int = -1, max_batch: int = 0, max_subscribers: int = 0, max_nat_sessions: int = 0,
                 max_eim_mappings: int = 0, event_capacity: int = 0, rank: int = 0, world: int = 1):
        self.lib = load_library()
        o = OpenOpts(C.sizeof(OpenOpts), device, max_batch, max_subscribers, max_nat_sessions, max_eim_mappings,
                     event_capacity, rank, world)
        self.h = self.lib.bng_open(C.byref(o))
        if not self.h:
            raise RuntimeError("bng_open failed: " + self.lib.bng_last_error(None).decode())
        self._ids = {}
        self._info = {}

    def close(self):
        if self.h:
            self.lib.bng_close(self.h)
            self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def _chk(self, r, what):
        if r < 0:
            raise BngError(-r, f"{what}: {errno.errorcode.get(-r, r)} ({self.lib.bng_last_error(self.h).decode()})")
        return r

    # ---- maps ----
    def map_id(self, name: str) -> int:
        if name not in self._ids:
            i = self.lib.bng_map_id(self.h, name.encode())
            if i < 0:
                raise KeyError(name)
            self._ids[name] = i
        return self._ids[name]

    def map_info(self, name: str) -> dict:
        inf = MapInfo()
        self._chk(self.lib.bng_map_get_info(self.h, self.map_id(name), C.byref(inf)), "map_get_info")
        return {f: getattr(inf, f) for f, _ in MapInfo._fields_}

    def _sizes(self, name):
        if name not in self._info:
            i = self.map_info(name)
            self._info[name] = (i["key_size"], i["value_size"])
        return self._info[name]

    def update(self, name: str, key, value, flags: int = ANY) -> int:
        """bpf(2) BPF_MAP_UPDATE_ELEM; returns 0 or a negative errno (no exception)."""
        k = np.ascontiguousarray(as_bytes(np.asarray(key))).reshape(-1)
        v = np.ascontiguousarray(as_bytes(np.asarray(value))).reshape(-1)
        ks, vs = self._sizes(name)
        assert k.size == ks and v.size == vs, (name, k.size, ks, v.size, vs)
        return self.lib.bng_map_update(self.h, self.map_id(name), k.ctypes.data, v.ctypes.data, flags)

    def update_batch(self, name: str, keys, values, flags: int = ANY) -> int:
        k = np.ascontiguousarray(as_bytes(keys))
        v = np.ascontiguousarray(as_bytes(values))
        ks, vs = self._sizes(name)
        assert k.shape[1] == ks and v.shape[1] == vs and k.shape[0] == v.shape[0], (name, k.shape, v.shape, ks, vs)
        return self.lib.bng_map_update_batch(self.h, self.map_id(name), k.ctypes.data, v.ctypes.data, k.shape[0], flags)

    def lookup(self, name: str, key):
        k = np.ascontiguousarray(as_bytes(np.asarray(key))).reshape(-1)
        ks, vs = self._sizes(name)
        assert k.size == ks
        out = np.zeros(vs, dtype=np.uint8)
        r = self.lib.bng_map_lookup(self.h, self.map_id(name), k.ctypes.data, out.ctypes.data)
        if r == -errno.ENOENT:
            return None
        self._chk(r, "map_lookup")
        return out

    def update_staged(self, name: str, key, value) -> int:
        """Queue a BPF_ANY upsert; applied at the next batch boundary / sync / read of the same map."""
        k = np.ascontiguousarray(as_bytes(np.asarray(key))).reshape(-1)
        v = np.ascontiguousarray(as_bytes(np.asarray(value))).reshape(-1)
        ks, vs = self._sizes(name)
        assert k.size == ks and v.size == vs, (name, k.size, ks, v.size, vs)
        return self.lib.bng_map_update_staged(self.h, self.map_id(name), k.ctypes.data, v.ctypes.data)

    def staged_info(self) -> dict:
        p, f, e = C.c_uint64(), C.c_uint64(), C.c_uint64()
        self._chk(self.lib.bng_staged_info(self.h, C.byref(p), C.byref(f), C.byref(e)), "staged_info")
        return {"pending": p.value, "flushes": f.value, "errors": e.value}

    def delete(self, name: str, key) -> int:
        k = np.ascontiguousarray(as_bytes(np.asarray(key))).reshape(-1)
        return self.lib.bng_map_delete(self.h, self.map_id(name), k.ctypes.data)

    def clear(self, name: str) -> int:
        return self.lib.bng_map_clear(self.h, self.map_id(name))

    def dump(self, name: str):
        """(keys u8[n,ks], values u8[n,vs]) sorted by key bytes."""
        inf = self.map_info(name)
        cap = max(int(inf["count"]), 1)
        keys = np.zeros((cap, max(inf["key_size"], 1)), dtype=np.uint8)
        vals = np.zeros((cap, max(inf["value_size"], 1)), dtype=np.uint8)
        n = self._chk(self.lib.bng_map_dump(self.h, self.map_id(name), keys.ctypes.data, vals.ctypes.data, cap), "dump")
        keys, vals = keys[:n], vals[:n]
        if n:
            order = np.lexsort(keys.T[::-1])
            keys, vals = keys[order], vals[order]
        return keys, vals

    def ipv6_prefixes_set(self, prefixes, lens, addrs=None, remove: bool = False) -> int:
        """Install subscribers' IPv6 addresses and prefixes (Framed-IPv6-Prefix, Delegated-IPv6-Prefix) in
        subscriber_ipv6, or with remove=True delete them.  prefixes: u8[n, 16] or 16-byte bytes objects; lens: the
        prefix lengths; addrs: the owners' IPv4 addresses (u8[n, 4] key bytes or u32 words; not needed to remove).
        Returns 0 or the first negative errno (a removal that finds a prefix absent reports -ENOENT)."""
        p = np.asarray([np.frombuffer(x, np.uint8) if isinstance(x, (bytes, bytearray)) else x for x in prefixes], np.uint8)
        keys = np.zeros(len(p), bng_ipv6_prefix_key)
        keys["prefixlen"] = np.asarray(lens, np.uint32).reshape(-1)
        keys["addr"] = p.reshape(-1, 16)
        if remove:
            rs = [self.delete("subscriber_ipv6", k) for k in keys]
            return next((r for r in rs if r), 0)
        return self.update_batch("subscriber_ipv6", keys, _addr_words(addrs).reshape(-1, 1).view(np.uint8))

    def qos_ipv6_enable(self, on: bool = True):
        """Shape IPv6 frames with their subscriber_ipv6 owner's token bucket (qos_ingress_prog, qos_egress_prog and the
        two pipelines), from the next run on; off by default.  Context state: snapshots, deltas and hand-over blobs do
        not carry it."""
        self._chk(self.lib.bng_qos_ipv6_enable(self.h, 1 if on else 0), "qos_ipv6_enable")

    def antispoof_ipv6_prefixes_enable(self, on: bool = True):
        """Let antispoof_ingress (standalone and in the two pipelines) allow an IPv6 source that lies in its binding's
        own subscriber_ipv6 prefixes, from the next run on; off by default (include/bng_b200.h).  Context state:
        snapshots, deltas and hand-over blobs do not carry it."""
        self._chk(self.lib.bng_antispoof_ipv6_prefixes_enable(self.h, 1 if on else 0), "antispoof_ipv6_prefixes_enable")

    def dhcpv6_enable(self, on: bool = True):
        """Let dhcp_fastpath_prog answer bound DHCPv6 clients' Solicit, Request, Renew and Rebind from dhcpv6_bindings,
        from the next run on; off by default (include/bng_b200.h).  Context state: snapshots, deltas and hand-over
        blobs do not carry it."""
        self._chk(self.lib.bng_dhcpv6_enable(self.h, 1 if on else 0), "dhcpv6_enable")

    def nd_enable(self, on: bool = True):
        """Let dhcp_fastpath_prog answer IPv6 Router Solicitations with a per-subscriber Router Advertisement (nd_config,
        nd_bindings) and Neighbor Solicitations for the router's link-local address, from the next run on; off by
        default (include/bng_b200.h).  Context state: snapshots, deltas and hand-over blobs do not carry it."""
        self._chk(self.lib.bng_nd_enable(self.h, 1 if on else 0), "nd_enable")

    def nat_icmp_errors_enable(self, on: bool = True):
        """Translate inbound ICMP errors (Destination Unreachable, Time Exceeded, Parameter Problem) in nat44_ingress
        by the flow they quote, from the next run on; off by default (include/bng_b200.h).  Context state: snapshots,
        deltas and hand-over blobs do not carry it."""
        self._chk(self.lib.bng_nat_icmp_errors_enable(self.h, 1 if on else 0), "nat_icmp_errors_enable")

    def nat_icmp_errors_egress_enable(self, on: bool = True):
        """Translate subscribers' ICMP errors (Destination Unreachable, Time Exceeded, Parameter Problem) in
        nat44_egress, pipeline_up and pipeline_tc by the flow they quote, from the next run on; off by default
        (include/bng_b200.h).  Context state: snapshots, deltas and hand-over blobs do not carry it."""
        self._chk(self.lib.bng_nat_icmp_errors_egress_enable(self.h, 1 if on else 0), "nat_icmp_errors_egress_enable")

    def ipv6_prefix_lengths(self) -> np.ndarray:
        """Live subscriber_ipv6 entries per prefix length, u32[129]."""
        out = np.zeros(129, np.uint32)
        self._chk(self.lib.bng_ipv6_prefix_lengths(self.h, out.ctypes.data), "ipv6_prefix_lengths")
        return out

    def stats(self, name: str) -> np.ndarray:
        """A statistics map (antispoof_stats, qos_stats_map, nat_stats_map, stats_map) as u64[]."""
        v = self.lookup(name, np.uint32(0))
        return v.view("<u8").copy()

    def drain(self, name: str) -> np.ndarray:
        mid = self.map_id(name)
        sz = self.lib.bng_event_size(self.h, mid)
        n = int(self.map_info(name)["count"])
        out = np.zeros((max(n, 1), sz), dtype=np.uint8)
        got = C.c_uint64(0)
        self._chk(self.lib.bng_events_drain(self.h, mid, out.ctypes.data, n, C.byref(got)), "events_drain")
        return out[: got.value]

    # ---- programs ----
    def prog_id(self, name: str) -> int:
        i = self.lib.bng_prog_id(self.h, name.encode())
        if i < 0:
            raise KeyError(name)
        return i

    def run(self, prog, pkts, lens, now_ns: int, off16=None, stride: int = 0, priority=None, verdict=None,
            mem: int = MEM_HOST, arena_bytes: int | None = None, now_v=None):
        """Run a program over a batch, in place.  Host arrays (numpy) with ``mem=MEM_HOST`` return
        synchronised; device buffers (torch tensors / raw pointers) with ``mem=MEM_DEVICE`` are queued on
        the context's stream (call :meth:`sync`).  Returns the verdict array/tensor."""
        pid = prog if isinstance(prog, int) else self.prog_id(prog)
        n = int(lens.shape[0])
        if verdict is None:
            if mem == MEM_HOST:
                verdict = np.zeros(n, dtype=np.uint8)
            else:
                import torch
                verdict = torch.zeros(n, dtype=torch.uint8, device=lens.device)
        b = Batch()
        b.pkts = _ptr(pkts)
        b.off16 = _ptr(off16)
        b.len = _ptr(lens)
        b.verdict = _ptr(verdict)
        b.priority = _ptr(priority)
        b.n = n
        b.stride = stride
        b.now_ns = now_ns
        b.mem = mem
        b.now_ns_v = _ptr(now_v)
        if arena_bytes is None:
            arena_bytes = int(pkts.nbytes) if isinstance(pkts, np.ndarray) else int(pkts.numel() * pkts.element_size())
        b.arena_bytes = (arena_bytes + 15) // 16
        self._chk(self.lib.bng_prog_run(self.h, pid, C.byref(b)), f"prog_run({prog})")
        return verdict

    def sync(self):
        self._chk(self.lib.bng_sync(self.h), "sync")

    def snapshot(self) -> bytes:
        n = self._chk(self.lib.bng_snapshot(self.h, None, 0), "snapshot")
        buf = C.create_string_buffer(n)
        self._chk(self.lib.bng_snapshot(self.h, buf, n), "snapshot")
        return buf.raw

    def restore(self, blob: bytes):
        buf = C.create_string_buffer(blob, len(blob))
        self._chk(self.lib.bng_restore(self.h, buf, len(blob)), "restore")

    # ---- per-subscriber traffic accounting ----
    def acct_enable(self, prog, on: bool = True):
        """Count the octets and packets of `prog`'s runs per subscriber address (off by default)."""
        pid = prog if isinstance(prog, int) else self.prog_id(prog)
        self._chk(self.lib.bng_acct_enable(self.h, pid, 1 if on else 0), f"acct_enable({prog})")

    def acct_read(self, addrs):
        """addrs: u8[n, 4] (qos_ingress key bytes) or u32[n] -> (bng_acct records[n], found bool[n])."""
        a = _addr_words(addrs)
        out = np.zeros(len(a), dtype=bng_acct)
        res = np.zeros(len(a), dtype=np.int32)
        self._chk(self.lib.bng_acct_read(self.h, a.ctypes.data, len(a), out.ctypes.data, res.ctypes.data), "acct_read")
        return out, res == 0

    def acct_dump(self):
        """(addresses u32[n], bng_acct records[n]) of every subscriber address, sorted by address bytes."""
        cap = max(int(self.map_info("subscriber_nat")["count"]) + int(self.map_info("qos_ingress")["count"]), 1)
        a = np.zeros(cap, dtype="<u4")
        out = np.zeros(cap, dtype=bng_acct)
        n = self._chk(self.lib.bng_acct_dump(self.h, a.ctypes.data, out.ctypes.data, cap), "acct_dump")
        a, out = a[:n], out[:n]
        order = np.argsort(a.byteswap(), kind="stable")
        return a[order], out[order]

    # ---- per-subscriber idle detection ----
    def idle_enable(self, prog, on: bool = True):
        """Stamp the last-activity clocks of `prog`'s subscribers (off by default; independent of accounting)."""
        pid = prog if isinstance(prog, int) else self.prog_id(prog)
        self._chk(self.lib.bng_idle_enable(self.h, pid, 1 if on else 0), f"idle_enable({prog})")

    def idle_timeout_set(self, addrs, timeouts_s):
        """Idle-Timeout of each address (u8[n, 4] key bytes or u32[n]) in seconds: 0 = the scan's default,
        layouts.IDLE_NEVER = never idle.  Returns found bool[n] (False: the address has no entry)."""
        a = _addr_words(addrs)
        t = np.ascontiguousarray(np.broadcast_to(np.asarray(timeouts_s, "<u4"), a.shape))
        res = np.zeros(len(a), dtype=np.int32)
        self._chk(self.lib.bng_idle_timeout_set(self.h, a.ctypes.data, t.ctypes.data, len(a), res.ctypes.data), "idle_timeout_set")
        return res == 0

    def idle_read(self, addrs):
        """addrs: u8[n, 4] (qos_ingress key bytes) or u32[n] -> (bng_idle records[n], found bool[n])."""
        a = _addr_words(addrs)
        out = np.zeros(len(a), dtype=bng_idle)
        res = np.zeros(len(a), dtype=np.int32)
        self._chk(self.lib.bng_idle_read(self.h, a.ctypes.data, len(a), out.ctypes.data, res.ctypes.data), "idle_read")
        return out, res == 0

    def idle_scan(self, now_ns: int, default_s: int = 0, flags: int = 3, cap: int | None = None):
        """(addresses u32[k], bng_idle records[k], found) of the subscribers idle at now_ns, sorted by address bytes;
        found is the number of idle records, k = min(found, cap) (cap None: room for every subscriber)."""
        if cap is None:
            cap = max(int(self.map_info("subscriber_nat")["count"]) + int(self.map_info("qos_ingress")["count"]), 1)
        a = np.zeros(max(cap, 1), dtype="<u4")
        out = np.zeros(max(cap, 1), dtype=bng_idle)
        n = self._chk(self.lib.bng_idle_scan(self.h, now_ns, default_s, flags, a.ctypes.data, out.ctypes.data, cap), "idle_scan")
        k = min(n, cap)
        a, out = a[:k], out[:k]
        order = np.argsort(a.byteswap(), kind="stable")
        return a[order], out[order], n

    def nat_flush(self, addrs, now_ns: int):
        """Remove the NAT flow state of a set of subscriber addresses (u8[n, 4] subscriber_nat key bytes or u32[n]):
        their sessions, the reverse entries that lead to them and their EIM mappings; their sessions_active becomes 0.
        Returns (sessions, reverse entries, EIM mappings) removed."""
        a = _addr_words(addrs)
        out = (C.c_uint64 * 3)()
        self._chk(self.lib.bng_nat_flush(self.h, a.ctypes.data if len(a) else None, len(a), now_ns, out), "nat_flush")
        return tuple(int(x) for x in out)

    # ---- NAT port-usage census ----
    def nat_usage(self, min_permille: int = 0, cap: int | None = None):
        """Port utilisation per subscriber and per public address (include/bng_b200.h, bng_nat_usage).  Returns
        (summary dict, subscriber addresses u32[k], bng_nat_sub_use[k], public addresses u32[m], bng_nat_pub_use[m]),
        each kind sorted by address bytes: the subscribers whose permille >= min_permille and every public address,
        at most `cap` of each (None: all of them)."""
        sub_cap = cap if cap is not None else max(int(self.map_info("subscriber_nat")["count"]), 1)
        pub_cap = cap if cap is not None else sub_cap + 64
        while True:
            s = np.zeros(1, dtype=bng_nat_usage_sum)
            sa, so = np.zeros(max(sub_cap, 1), "<u4"), np.zeros(max(sub_cap, 1), bng_nat_sub_use)
            pa, po = np.zeros(max(pub_cap, 1), "<u4"), np.zeros(max(pub_cap, 1), bng_nat_pub_use)
            self._chk(self.lib.bng_nat_usage(self.h, min_permille, s.ctypes.data, sa.ctypes.data, so.ctypes.data, sub_cap,
                                             pa.ctypes.data, po.ctypes.data, pub_cap), "nat_usage")
            summary = {k: int(s[0][k]) for k in bng_nat_usage_sum.names}
            if cap is not None or summary["pubs_found"] <= pub_cap:
                break
            pub_cap = summary["pubs_found"]  # more public addresses than the first guess: ask again with room for all
        ks, kp = min(summary["subs_found"], sub_cap), min(summary["pubs_found"], pub_cap)
        sa, so, pa, po = sa[:ks], so[:ks], pa[:kp], po[:kp]
        os_, op = np.argsort(sa.byteswap(), kind="stable"), np.argsort(pa.byteswap(), kind="stable")
        return summary, sa[os_], so[os_], pa[op], po[op]

    # ---- DHCP lease census and expiry sweep ----
    def lease_census(self, now_ns: int, cap: int | None = None):
        """Per-pool utilisation of the DHCP lease maps at now_ns (include/bng_b200.h, bng_dhcp_lease_census).  Returns
        (summary dict, pool ids u32[k], bng_lease_pool_use[k]) sorted by pool id: every pool, or at most `cap` of them."""
        room = cap if cap is not None else 64
        while True:
            s = np.zeros(1, dtype=bng_lease_sum)
            ids, out = np.zeros(max(room, 1), "<u4"), np.zeros(max(room, 1), bng_lease_pool_use)
            self._chk(self.lib.bng_dhcp_lease_census(self.h, now_ns, s.ctypes.data, ids.ctypes.data, out.ctypes.data, room),
                      "lease_census")
            summary = {k: (int(s[0][k]) if s[0][k].ndim == 0 else [int(x) for x in s[0][k]]) for k in bng_lease_sum.names}
            if cap is not None or summary["pools_found"] <= room:
                break
            room = summary["pools_found"]  # more pools than the first guess: ask again with room for all
        k = min(summary["pools_found"], room)
        o = np.argsort(ids[:k], kind="stable")
        return summary, ids[:k][o], out[:k][o]

    def lease_sweep(self, now_ns: int, grace_s: int = 0, cap: int | None = None):
        """Remove the lease entries past lease_expiry + grace_s at now_ns (include/bng_b200.h, bng_dhcp_lease_sweep).
        Returns (found, bng_lease_removed[k] sorted by (map, key bytes), removed per map [4]).  cap None: one call with
        room for every entry the three maps hold; else at most `cap` are removed and found may exceed k."""
        if cap is None:
            cap = max(sum(int(self.map_info(m)["count"]) for m in
                          ("subscriber_pools", "vlan_subscriber_pools", "circuit_id_subscribers")), 1)
        out = np.zeros(max(cap, 1), bng_lease_removed)
        removed = (C.c_uint64 * 4)()
        found = self._chk(self.lib.bng_dhcp_lease_sweep(self.h, now_ns, grace_s, out.ctypes.data if cap else None, cap, removed),
                          "lease_sweep")
        out = out[:min(found, cap)]
        o = np.lexsort([out["key"][:, j] for j in range(31, -1, -1)] + [out["map"]])
        return found, out[o], [int(x) for x in removed]

    def lease_addr_order(self, wire: bool):
        """How this context's control plane stores allocated_ip and ip_pool.network: the numeric value in a native word
        (False, the default: the Go loader and the C++ mirror) or the four bytes in wire order (True: synth.py, the
        test scripts).  The census's prefix test follows it."""
        self._chk(self.lib.bng_dhcp_lease_addr_order(self.h, 1 if wire else 0), "lease_addr_order")

    def lease_table_rebuilds(self) -> int:
        return self.lib.bng_lease_table_rebuilds(self.h)

    # ---- lawful intercept: content of communication ----
    def li_configure(self, snaplen: int = 0, capacity: int = 0):
        """(Re)create the capture ring: `capacity` records of `snaplen` bytes (0: 1518 bytes, 2^15 records).  Records
        not yet drained are discarded and counted in li_lost."""
        self._chk(self.lib.bng_li_configure(self.h, snaplen, capacity), "li_configure")

    @property
    def li_record_size(self) -> int:
        return self.lib.bng_li_record_size(self.h)

    def li_target_set(self, addr: int, target_id: int):
        """Capture the frames of `addr` (u32 holding the qos_ingress key bytes) as `target_id`."""
        self._chk(self.lib.bng_li_target_set(self.h, int(addr), int(target_id)), "li_target_set")

    def li_target_del(self, addr: int) -> int:
        """Stop capturing `addr`; returns 0 or -ENOENT (no exception)."""
        return self.lib.bng_li_target_del(self.h, int(addr))

    def li_drain(self, cap: int | None = None):
        """(bng_li_record headers[n], list of the captured bytes of each record) in (batch, frame) order; at most
        `cap` records (None: all), the rest stay for the next call."""
        rs = self.lib.bng_li_record_size(self.h)
        if rs == 0:
            return np.zeros(0, bng_li_record), []
        out, got = [], 0
        while cap is None or got < cap:
            want = 1 << 14 if cap is None else min(cap - got, 1 << 14)
            buf = np.zeros((want, rs), np.uint8)
            n = C.c_uint64(0)
            self._chk(self.lib.bng_li_drain(self.h, buf.ctypes.data, want, C.byref(n)), "li_drain")
            out.append(buf[: n.value])
            got += n.value
            if n.value < want:
                break
        raw = np.concatenate(out) if out else np.zeros((0, rs), np.uint8)
        hdr = raw[:, :64].copy().view(bng_li_record).reshape(-1)
        return hdr, [raw[i, 64:64 + int(h["cap_len"])].copy() for i, h in enumerate(hdr)]

    @property
    def li_lost(self) -> int:
        return self.lib.bng_li_lost(self.h)

    # ---- incremental replication to a standby ----
    def delta_enable(self, on: bool = True):
        """Start (or stop) tracking changes for delta_export; starting sets the baseline to empty and a new stream id."""
        self._chk(self.lib.bng_delta_enable(self.h, 1 if on else 0), "delta_enable")

    def delta_export(self, refresh_ns: int = 0, full: bool = False, exact: bool = False) -> bytes:
        """The changes since the previous export as one blob for delta_apply on the standby."""
        flags = (DELTA_FULL if full else 0) | (DELTA_EXACT if exact else 0)
        cap = 1 << 20  # most deltas are small; a larger one is sized by -ENOSPC, which leaves the baseline as it was
        while True:
            buf = np.empty(cap, np.uint8)  # not zero-filled: a FULL delta can be hundreds of MB
            n = C.c_uint64(0)
            r = self.lib.bng_delta_export(self.h, refresh_ns, flags, buf.ctypes.data, cap, C.byref(n))
            if r != -errno.ENOSPC:
                break
            cap = n.value
        self._chk(r, "delta_export")
        return buf[: n.value].tobytes()

    def delta_apply(self, blob: bytes) -> int:
        """Apply a delta of the active context; returns 0 or -ESTALE (a gap or another stream: ask for a FULL one)."""
        r = self.lib.bng_delta_apply(self.h, blob, len(blob))
        return r if r == -errno.ESTALE else self._chk(r, "delta_apply")

    def delta_info(self) -> tuple:
        """(stream id, sequence): of the last export with tracking enabled, else of the last delta applied."""
        s, q = C.c_uint64(), C.c_uint64()
        self._chk(self.lib.bng_delta_info(self.h, C.byref(s), C.byref(q)), "delta_info")
        return s.value, q.value

    # ---- subscriber hand-over between contexts ----
    def sub_export(self, addrs, macs=(), detach: bool = False) -> bytes:
        """The state of a set of subscribers (addresses as u8[n, 4] key bytes or u32[n]; MACs as the u64 key words of
        subscriber_bindings / subscriber_pools) as one blob for sub_import on another context; detach removes it here."""
        a = _addr_words(addrs) if len(addrs) else np.zeros(0, "<u4")
        m = np.ascontiguousarray(np.asarray(macs, dtype="<u8").reshape(-1))
        flags = SUB_DETACH if detach else 0
        cap = 1 << 16  # a larger blob is sized by -ENOSPC, which writes and removes nothing
        while True:
            buf = np.empty(cap, np.uint8)
            n = C.c_uint64(0)
            r = self.lib.bng_sub_export(self.h, a.ctypes.data if len(a) else None, len(a), m.ctypes.data if len(m) else None,
                                        len(m), flags, buf.ctypes.data, cap, C.byref(n))
            if r != -errno.ENOSPC:
                break
            cap = n.value
        self._chk(r, "sub_export")
        return buf[: n.value].tobytes()

    def sub_import(self, blob: bytes) -> int:
        """Take the subscribers of a sub_export blob into this context; returns 0 (errors raise BngError)."""
        return self._chk(self.lib.bng_sub_import(self.h, blob, len(blob)), "sub_import")

    def sweep(self, now_ns: int) -> int:
        """Session expiry sweep at now_ns; returns the number of sessions removed."""
        n = C.c_uint64(0)
        self._chk(self.lib.bng_sweep(self.h, now_ns, C.byref(n)), "sweep")
        return n.value

    @property
    def table_rebuilds(self) -> int:
        return self.lib.bng_table_rebuilds(self.h)

    @property
    def lru_evictions(self) -> int:
        return self.lib.bng_lru_evictions(self.h)

    @property
    def stream(self) -> int:
        return self.lib.bng_stream(self.h) or 0

    # ---- multi-GPU plumbing / diagnostics ----
    def stats_device_ptr(self):
        p = C.c_void_p()
        n = C.c_uint32()
        self._chk(self.lib.bng_stats_device_ptr(self.h, C.byref(p), C.byref(n)), "stats_device_ptr")
        return p.value, n.value

    @staticmethod
    def comm_unique_id() -> bytes:
        """128-byte NCCL unique id (rank 0 makes it, the host plumbing distributes it)."""
        try:  # a process that will use torch must have torch's libnccl resident before the library resolves the name
            import torch  # noqa: F401
        except Exception:
            pass
        buf = C.create_string_buffer(128)
        r = load_library().bng_comm_unique_id(buf, 128)
        if r < 0:
            raise BngError(-r, "bng_comm_unique_id")
        return buf.raw

    def comm_init(self, uid: bytes, rank: int, world: int):
        buf = C.create_string_buffer(uid, 128)
        self._chk(self.lib.bng_comm_init(self.h, buf, rank, world), "comm_init")

    def sync_reduce(self) -> np.ndarray:
        """Flush staged upserts and all-reduce the packed counter vector over the communicator; u64[40] totals."""
        out = np.zeros(40, dtype=np.uint64)
        self._chk(self.lib.bng_sync_reduce(self.h, out.ctypes.data), "sync_reduce")
        return out

    def prof_enable(self, on: bool = True):
        self._chk(self.lib.bng_prof_enable(self.h, 1 if on else 0), "prof_enable")

    def prof_read(self) -> dict:
        """{kernel name: (launches, total_ms)} since prof_enable(True)."""
        buf = C.create_string_buffer(8192)
        self._chk(self.lib.bng_prof_read(self.h, buf, 8192), "prof_read")
        out = {}
        for line in buf.value.decode().splitlines():
            name, n, ms = line.rsplit(" ", 2)
            out[name] = (int(n), float(ms))
        return out

    @property
    def launch_count(self) -> int:
        return self.lib.bng_launch_count(self.h)

    @property
    def lru_overflow(self) -> int:
        return self.lib.bng_lru_overflow(self.h)

    @property
    def events_lost(self) -> int:
        return self.lib.bng_events_lost(self.h)
