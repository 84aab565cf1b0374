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

# include/bng_b200.h struct bng_idle (32 B): per-subscriber last-activity stamps and idle timeout
IDLE_UP, IDLE_DOWN, IDLE_STARTED, IDLE_NEVER = 1, 2, 4, 0xFFFFFFFF
bng_idle = np.dtype([("up_ns", "<u8"), ("down_ns", "<u8"), ("since_ns", "<u8"), ("timeout_s", "<u4"), ("flags", "<u4")])

# include/bng_b200.h struct bng_ipv6_prefix_key (20 B): the key of subscriber_ipv6 (not a reference map), laid out as a
# BPF_MAP_TYPE_LPM_TRIE key for IPv6; the value is the subscriber's IPv4 address (4 key bytes of qos_ingress)
bng_ipv6_prefix_key = np.dtype([("prefixlen", "<u4"), ("addr", "u1", 16)])
assert bng_ipv6_prefix_key.itemsize == 20

# include/bng_b200.h: the DHCPv6 fast path's cache (not reference maps).  dhcpv6_bindings: key (32 B) -> binding (64 B);
# dhcpv6_server_config: one 96-byte entry; dhcpv6_stats: BNG_DHCPV6_NUM_STATS u64 counters
DHCPV6_NA, DHCPV6_PD = 1, 2
bng_dhcpv6_client_key = np.dtype([("duid_len", "u1"), ("duid", "u1", 31)])
bng_dhcpv6_binding = np.dtype([
    ("mac", "u1", 6), ("flags", "u1"), ("pd_len", "u1"), ("iaid_na", "<u4"), ("iaid_pd", "<u4"),
    ("preferred_lft", "<u4"), ("valid_lft", "<u4"), ("expires_s", "<u8"), ("addr", "u1", 16), ("prefix", "u1", 16)])
bng_dhcpv6_server_config = np.dtype([
    ("server_mac", "u1", 6), ("duid_len", "u1"), ("dns_count", "u1"), ("server_ip", "u1", 16), ("duid", "u1", 32),
    ("dns", "u1", (2, 16)), ("_pad", "u1", 8)])
DHCPV6_STATS = ("total", "solicit", "request", "renew", "rebind", "advertise", "reply", "miss", "expired", "unsupported",
                "no_room", "malformed")
dhcpv6_stats = np.dtype([(n, "<u8") for n in DHCPV6_STATS])
assert bng_dhcpv6_client_key.itemsize == 32 and bng_dhcpv6_binding.itemsize == 64
assert bng_dhcpv6_server_config.itemsize == 96 and dhcpv6_stats.itemsize == 96

# include/bng_b200.h: Router and Neighbor Solicitations answered on the GPU (not reference maps).  nd_config: one
# 320-byte entry (the RA template); nd_bindings: the subscriber_bindings MAC word -> binding (48 B); nd_stats:
# BNG_ND_NUM_STATS u64 counters
ND_PIO_L, ND_PIO_A = 0x80, 0x40
bng_nd_config = np.dtype([
    ("router_mac", "u1", 6), ("_pad0", "u1", 2), ("ra_head_len", "<u2"), ("ra_tail_len", "<u2"), ("_pad1", "u1", 4),
    ("router_ll", "u1", 16), ("ra", "u1", 288)])
bng_nd_binding = np.dtype([
    ("prefix", "u1", 16), ("prefix_len", "u1"), ("pio_flags", "u1"), ("_pad0", "u1", 2), ("valid_lft", "<u4"),
    ("preferred_lft", "<u4"), ("_pad1", "u1", 4), ("expires_s", "<u8"), ("_pad2", "u1", 8)])
ND_STATS = ("total", "rs", "ns", "ra", "na", "miss", "expired", "not_target", "malformed", "unsupported", "no_room")
nd_stats = np.dtype([(n, "<u8") for n in ND_STATS])
assert bng_nd_config.itemsize == 320 and bng_nd_binding.itemsize == 48 and nd_stats.itemsize == 88

# lawful-intercept record header (include/bng_b200.h: struct bng_li_record, 64 B); the captured bytes follow it
LI_UPLINK, LI_DOWNLINK = 0, 1
bng_li_record = np.dtype([
    ("ts_ns", "<u8"), ("batch", "<u8"), ("frame", "<u4"), ("target_id", "<u4"), ("addr", "<u4"), ("wire_len", "<u4"),
    ("cap_len", "<u4"), ("dir", "u1"), ("verdict", "u1"), ("prog", "u1"), ("pad", "u1", 25)])

# include/bng_b200.h NAT port-usage census (bng_nat_usage): per-subscriber record, per-public-address record, summary
bng_nat_sub_use = np.dtype([
    ("sessions", "<u8"), ("eim", "<u8"), ("public_ip", "<u4"), ("block_ports", "<u4"), ("in_use", "<u4", 3),
    ("in_use_any", "<u4"), ("outside", "<u4"), ("unreachable", "<u4"), ("permille", "<u4"), ("pad", "<u4", 3)])
bng_nat_pub_use = np.dtype([
    ("sessions", "<u8"), ("eim", "<u8"), ("block_ports", "<u8"), ("blocks", "<u4"), ("in_use", "<u4", 3),
    ("in_use_any", "<u4"), ("unreachable", "<u4"), ("pad", "<u4", 4)])
bng_nat_usage_sum = np.dtype([(n, "<u8") for n in (
    "subscribers", "sessions", "eim", "triples", "unreachable", "stale_reverse", "orphan_sessions", "orphan_eim",
    "subs_found", "pubs_found")])

# include/bng_b200.h DHCP lease census and sweep: per-pool record, summary, removed-entry record
bng_lease_pool_use = np.dtype([
    ("entries", "<u8", 3), ("expired", "<u8"), ("addrs", "<u4"), ("addrs_outside", "<u4"), ("conflicts", "<u4"),
    ("prefix_hosts", "<u4"), ("permille", "<u4"), ("known", "u1"), ("pad", "u1", 11)])
bng_lease_sum = np.dtype([
    ("entries", "<u8", 3), ("expired", "<u8", 3), ("addrs", "<u8"), ("conflicts", "<u8"), ("unknown_pool", "<u8"),
    ("cid_dangling", "<u8"), ("pools_found", "<u8")])
bng_lease_removed = np.dtype([
    ("key", "u1", 32), ("lease_expiry", "<u8"), ("pool_id", "<u4"), ("allocated_ip", "u1", 4), ("vlan_id", "<u4"),
    ("map", "u1"), ("client_class", "u1"), ("flags", "u1"), ("pad", "u1", 9)])
LEASE_MAPS = ("subscriber_pools", "vlan_subscriber_pools", "circuit_id_subscribers")  # bng_lease_removed.map

assert bng_lease_pool_use.itemsize == 64 and bng_lease_removed.itemsize == 64 and bng_lease_sum.itemsize == 88
assert bng_nat_sub_use.itemsize == 64 and bng_nat_pub_use.itemsize == 64 and bng_nat_usage_sum.itemsize == 80
assert subscriber_binding.itemsize == 24 and token_bucket.itemsize == 32 and bng_acct.itemsize == 64
assert bng_li_record.itemsize == 64
assert bng_idle.itemsize == 32
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
    "subscriber_ipv6": (bng_ipv6_prefix_key, ("u1", 4)),
    "dhcpv6_bindings": (bng_dhcpv6_client_key, bng_dhcpv6_binding),
    "dhcpv6_server_config": ("<u4", bng_dhcpv6_server_config),
    "dhcpv6_stats": ("<u4", dhcpv6_stats),
    "nd_bindings": ("<u8", bng_nd_binding),
    "nd_config": ("<u4", bng_nd_config),
    "nd_stats": ("<u4", nd_stats),
}


def as_bytes(arr) -> np.ndarray:
    """View any (structured) array as uint8[n, itemsize]."""
    a = np.ascontiguousarray(arr)
    if a.ndim == 0:
        a = a.reshape(1)
    return a.view(np.uint8).reshape(a.shape[0], -1) if a.dtype.itemsize > 1 or a.ndim == 1 else a


# bng_delta_export blobs (include/bng_b200.h): a 40-byte header, then sections in bng_snapshot's 64-byte framing
delta_header = np.dtype([("magic", "S8"), ("stream_id", "<u8"), ("seq_from", "<u8"), ("seq_to", "<u8"),
                         ("flags", "<u4"), ("sections", "<u4")])
delta_section = np.dtype([("name", "S40"), ("kind", "<u4"), ("key_size", "<u4"), ("value_size", "<u4"),
                          ("n_del", "<u4"), ("n_up", "<u8")])
assert delta_header.itemsize == 40 and delta_section.itemsize == 64


def parse_delta(blob: bytes) -> tuple:
    """(header record, {section name: (kind, deleted keys u8[n_del, ks], upserted keys u8[n_up, ks], values u8[n_up, vs])})."""
    b = np.frombuffer(blob, np.uint8)
    hdr = b[:delta_header.itemsize].view(delta_header)[0]
    if hdr["magic"] != b"BNGDELT1":
        raise ValueError("not a delta blob")
    out, p = {}, delta_header.itemsize
    for _ in range(int(hdr["sections"])):
        s = b[p:p + delta_section.itemsize].view(delta_section)[0]
        p += delta_section.itemsize
        ks, vs, nd, nu = int(s["key_size"]), int(s["value_size"]), int(s["n_del"]), int(s["n_up"])
        dk = b[p:p + nd * ks].reshape(nd, ks)
        p += nd * ks
        uk = b[p:p + nu * ks].reshape(nu, ks)
        p += nu * ks
        uv = b[p:p + nu * vs].reshape(nu, vs)
        p += nu * vs
        out[s["name"].decode()] = (int(s["kind"]), dk, uk, uv)
    if p != len(b):
        raise ValueError(f"delta blob: {len(b) - p} trailing bytes")
    return hdr, out
