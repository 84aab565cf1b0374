"""bng_b200 — H100-native subscriber dataplane (antispoof, NAT44, QoS, DHCP fast path).

The product is ``libbng_b200.so`` (C ABI in ``include/bng_b200.h``);
:class:`Dataplane` is its ctypes binding.  Importing this package never
falls back to a CPU implementation.
"""
from .dataplane import (ANY, EXIST, MEM_DEVICE, MEM_HOST, NOEXIST, PROGRAMS, BngError, Dataplane, load_library,
                        shard_of_mac)

__all__ = ["Dataplane", "BngError", "load_library", "shard_of_mac", "PROGRAMS", "MEM_DEVICE", "MEM_HOST", "ANY",
           "NOEXIST", "EXIST"]
