"""Byte layouts of the reference's eBPF map keys/values, events and verdicts,
as numpy dtypes.  These are the ABI between the control plane and the
dataplane; the C side addresses the same bytes by offset.

All multi-byte scalars are little-endian *as the eBPF programs see them*.
Addresses and ports that the programs compare against packet fields are kept
as raw wire-order bytes (``u1`` arrays) so nobody has to reason about the
reference's numeric/native-endian marshalling quirk (SURVEY.md §7.3-3).
"""
import numpy as np

# verdicts
TC_ACT_OK, TC_ACT_SHOT = 0, 2
XDP_DROP, XDP_PASS, XDP_TX = 1, 2, 3

# bpf/antispoof.c:29-33
ANTISPOOF_DISABLED, ANTISPOOF_STRICT, ANTISPOOF_LOOSE, ANTISPOOF_LOG_ONLY = 0, 1, 2, 3

# bpf/nat44.c:56-62
NAT_FLAG_EIM, NAT_FLAG_EIF, NAT_FLAG_HAIRPIN = 0x01, 0x02, 0x04
NAT_FLAG_ALG_FTP, NAT_FLAG_ALG_SIP, NAT_FLAG_PORT_PARITY, NAT_FLAG_PORT_CONTIGUITY = 0x08, 0x10, 0x20, 0x40

# bpf/antispoof.c:36-43 (24 B)
subscriber_binding = np.dtype([
    ("ipv4_addr", "u1", 4), ("ipv6_addr", "u1", 16), ("ipv4_valid", "u1"), ("ipv6_valid", "u1"),
    ("mode", "u1"), ("_pad", "u1")])
# bpf/antispoof.c:79-83 (8 B)
antispoof_config = np.dtype([("default_mode", "u1"), ("log_violations", "u1"), ("_pad", "u1", 6)])
# bpf/antispoof.c:58-65 (48 B)
antispoof_stats = np.dtype([(n, "<u8") for n in (
    "packets_allowed", "packets_dropped", "packets_logged", "ipv4_violations", "ipv6_violations", "unknown_mac")])
# bpf/antispoof.c:46-55 (56 B)
spoof_event = np.dtype([
    ("timestamp", "<u8"), ("src_mac", "u1", 6), ("protocol", "u1"), ("_pad", "u1"),
    ("spoofed_ip", "u1", 4), ("allowed_ip", "u1", 4), ("spoofed_ipv6", "u1", 16), ("allowed_ipv6", "u1", 16)])
# bpf/antispoof.c:108-111 (8 B)
lpm_key_v4 = np.dtype([("prefixlen", "<u4"), ("ip", "u1", 4)])

# bpf/qos_ratelimit.c:24-31 (32 B)
token_bucket = np.dtype([
    ("tokens", "<u8"), ("last_update", "<u8"), ("rate_bps", "<u8"), ("burst_bytes", "<u4"),
    ("priority", "u1"), ("_pad", "u1", 3)])
# bpf/qos_ratelimit.c:53-58 (32 B)
qos_stats = np.dtype([(n, "<u8") for n in ("packets_passed", "packets_dropped", "bytes_passed", "bytes_dropped")])

# bpf/nat44.c:92-99 (16 B)
nat_key = np.dtype([
    ("src_ip", "u1", 4), ("dst_ip", "u1", 4), ("src_port", "u1", 2), ("dst_port", "u1", 2),
    ("protocol", "u1"), ("_pad", "u1", 3)])
# bpf/nat44.c:104-109 (8 B).  internal_port is whatever 16-bit value the program
# put there: the network-order port for real mappings, a host-order candidate
# for the collision probes of allocate_port_from_block (bpf/nat44.c:450-455).
eim_key = np.dtype([("internal_ip", "u1", 4), ("internal_port", "<u2"), ("protocol", "u1"), ("_pad", "u1")])
# bpf/nat44.c:112-120 (32 B); external_port is HOST order
eim_mapping = np.dtype([
    ("external_ip", "u1", 4), ("external_port", "<u2"), ("_pad", "<u2"), ("created", "<u8"),
    ("last_used", "<u8"), ("ref_count", "<u4"), ("flags", "<u4")])
# bpf/nat44.c:123-141 (80 B, 4 B implicit padding before last_seen and at the tail)
nat_session = np.dtype([
    ("nat_ip", "u1", 4), ("nat_port", "u1", 2), ("orig_port", "u1", 2), ("orig_ip", "u1", 4),
    ("dest_ip", "u1", 4), ("dest_port", "u1", 2), ("_pad1", "<u2"), ("_ipad", "u1", 4),
    ("last_seen", "<u8"), ("created", "<u8"), ("packets_out", "<u8"), ("packets_in", "<u8"),
    ("bytes_out", "<u8"), ("bytes_in", "<u8"), ("state", "u1"), ("protocol", "u1"), ("flags", "u1"),
    ("is_hairpin", "u1"), ("_tpad", "u1", 4)])
# bpf/nat44.c:144-155 (32 B)
port_block = np.dtype([
    ("public_ip", "u1", 4), ("port_start", "<u2"), ("port_end", "<u2"), ("next_port", "<u4"),
    ("ports_in_use", "<u4"), ("allocated_at", "<u8"), ("subscriber_id", "<u4"), ("block_size_log2", "u1"),
    ("flags", "u1"), ("_pad", "u1", 2)])
# bpf/nat44.c:158-164 (64 B)
subscriber_nat = np.dtype([
    ("block", port_block), ("sessions_active", "<u8"), ("sessions_total", "<u8"), ("bytes_out", "<u8"),
    ("bytes_in", "<u8")])
# bpf/nat44.c:167-173 (16 B)
nat_pool_entry = np.dtype([
    ("public_ip", "u1", 4), ("subscribers", "<u4"), ("ports_per_sub", "<u2"), ("max_subscribers", "<u2"),
    ("flags", "<u4")])
# bpf/nat44.c:176-190 (104 B)
nat_stats = np.dtype([(n, "<u8") for n in (
    "packets_snat", "packets_dnat", "packets_hairpin", "packets_dropped", "packets_passed", "sessions_created",
    "sessions_expired", "port_exhaustion", "eim_hits", "eim_misses", "alg_triggers", "conntrack_lookups",
    "conntrack_hits")])
# bpf/nat44.c:193-205 (40 B, 4 B tail padding)
nat_log_entry = np.dtype([
    ("timestamp", "<u8"), ("event_type", "<u4"), ("subscriber_id", "<u4"), ("private_ip", "u1", 4),
    ("public_ip", "u1", 4), ("private_port", "u1", 2), ("public_port", "u1", 2), ("dest_ip", "u1", 4),
    ("dest_port", "u1", 2), ("protocol", "u1"), ("flags", "u1"), ("_tpad", "u1", 4)])
# bpf/nat44.c:208-213 (8 B)
alg_config = np.dtype([("port", "<u2"), ("protocol", "u1"), ("alg_type", "u1"), ("flags", "<u4")])
# bpf/nat44.c:271-277 (16 B)
nat_config = np.dtype([
    ("flags", "<u4"), ("port_range_start", "<u2"), ("port_range_end", "<u2"), ("default_ports_per_sub", "<u4"),
    ("_pad", "<u4")])

# bpf/maps.h:89-97 (packed, 25 B)
pool_assignment = np.dtype([
    ("pool_id", "<u4"), ("allocated_ip", "u1", 4), ("vlan_id", "<u4"), ("client_class", "u1"),
    ("lease_expiry", "<u8"), ("flags", "u1"), ("_pad", "u1", 3)])
# bpf/maps.h:110-113 (4 B)
vlan_key = np.dtype([("s_tag", "<u2"), ("c_tag", "<u2")])
# bpf/maps.h:135-144 (packed, 28 B)
ip_pool = np.dtype([
    ("network", "u1", 4), ("prefix_len", "u1"), ("_pad1", "u1", 3), ("gateway", "u1", 4),
    ("dns_primary", "u1", 4), ("dns_secondary", "u1", 4), ("lease_time", "<u4"), ("_pad2", "<u4")])
# bpf/maps.h:154-159 (16 B)
dhcp_server_config = np.dtype([
    ("server_mac", "u1", 6), ("_pad", "u1", 2), ("server_ip", "u1", 4), ("interface_index", "<u4")])
# bpf/maps.h:171-184 (80 B)
dhcp_stats = np.dtype([(n, "<u8") for n in (
    "total_requests", "fastpath_hits", "fastpath_misses", "errors", "cache_expired", "option82_present",
    "option82_absent", "broadcast_replies", "unicast_replies", "vlan_packets")])
# bpf/maps.h:218-220 (32 B)
circuit_id_key = np.dtype([("data", "u1", 32)])

# include/bng_b200.h struct bng_acct (64 B): per-subscriber traffic totals, not a reference map
bng_acct = np.dtype([(n, "<u8") for n in (
    "up_packets", "up_bytes", "up_drop_packets", "up_drop_bytes",
    "down_packets", "down_bytes", "down_drop_packets", "down_drop_bytes")])

# lawful-intercept record header (include/bng_b200.h: struct bng_li_record, 64 B); the captured bytes follow it
LI_UPLINK, LI_DOWNLINK = 0, 1
bng_li_record = np.dtype([
    ("ts_ns", "<u8"), ("batch", "<u8"), ("frame", "<u4"), ("target_id", "<u4"), ("addr", "<u4"), ("wire_len", "<u4"),
    ("cap_len", "<u4"), ("dir", "u1"), ("verdict", "u1"), ("prog", "u1"), ("pad", "u1", 25)])

assert subscriber_binding.itemsize == 24 and token_bucket.itemsize == 32 and bng_acct.itemsize == 64
assert bng_li_record.itemsize == 64
assert nat_key.itemsize == 16 and eim_key.itemsize == 8 and eim_mapping.itemsize == 32
assert nat_session.itemsize == 80 and port_block.itemsize == 32 and subscriber_nat.itemsize == 64
assert nat_stats.itemsize == 104 and nat_log_entry.itemsize == 40 and nat_config.itemsize == 16
assert pool_assignment.itemsize == 25 and ip_pool.itemsize == 28 and dhcp_server_config.itemsize == 16
assert dhcp_stats.itemsize == 80 and spoof_event.itemsize == 56 and antispoof_stats.itemsize == 48

# Bytes of each value that the reference leaves uninitialised or that hold
# compiler padding; comparisons mask them (offset, length).
PADDING = {
    "nat_sessions": [(20, 4), (76, 4)],
    "nat_log_rb": [(36, 4)],
}

# map name -> (key dtype or None, value dtype)
MAP_DTYPES = {
    "subscriber_bindings": ("<u8", subscriber_binding),
    "antispoof_config": ("<u4", antispoof_config),
    "antispoof_stats": ("<u4", antispoof_stats),
    "allowed_ranges_v4": (lpm_key_v4, "u1"),
    "qos_egress": (("u1", 4), token_bucket),
    "qos_ingress": (("u1", 4), token_bucket),
    "qos_stats_map": ("<u4", qos_stats),
    "nat_sessions": (nat_key, nat_session),
    "nat_reverse": (nat_key, nat_key),
    "eim_table": (eim_key, eim_mapping),
    "subscriber_nat": (("u1", 4), subscriber_nat),
    "nat_pool": ("<u4", nat_pool_entry),
    "hairpin_ips": (("u1", 4), "u1"),
    "nat_config_map": ("<u4", nat_config),
    "nat_stats_map": ("<u4", nat_stats),
    "alg_ports": ("<u4", alg_config),
    "subscriber_pools": ("<u8", pool_assignment),
    "vlan_subscriber_pools": (vlan_key, pool_assignment),
    "ip_pools": ("<u4", ip_pool),
    "server_config": ("<u4", dhcp_server_config),
    "stats_map": ("<u4", dhcp_stats),
    "circuit_id_map": ("<u8", "<u8"),
    "circuit_id_subscribers": (circuit_id_key, pool_assignment),
}


def as_bytes(arr) -> np.ndarray:
    """View any (structured) array as uint8[n, itemsize]."""
    a = np.ascontiguousarray(arr)
    if a.ndim == 0:
        a = a.reshape(1)
    return a.view(np.uint8).reshape(a.shape[0], -1) if a.dtype.itemsize > 1 or a.ndim == 1 else a
