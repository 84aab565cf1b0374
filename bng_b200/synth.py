"""Synthetic subscribers, flows, frames and map contents for tests and bench.py
(SURVEY.md §8d).  PRNG: splitmix64, seed 0xB2000000 + config number.
Subscriber i: MAC 02:00:ii:ii:ii:ii (big-endian i), private IP 100.64.0.0 + i.
Frames are Ethernet II without FCS; every frame's storage is padded to 16 B.
"""
from __future__ import annotations

import numpy as np

from . import layouts as L

MASK64 = (1 << 64) - 1


def splitmix64_array(seed: int, n: int) -> np.ndarray:
    """n successive splitmix64 outputs (uint64), vectorised."""
    with np.errstate(over="ignore"):
        i = np.arange(1, n + 1, dtype=np.uint64)
        x = np.uint64(seed & MASK64) + i * np.uint64(0x9E3779B97F4A7C15)
        x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return x ^ (x >> np.uint64(31))


def splitmix64_scalar(x: int) -> int:
    x = (x + 0x9E3779B97F4A7C15) & MASK64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & MASK64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & MASK64
    return x ^ (x >> 31)


def shard_of_mac(mac_key, world: int):
    """Same function as bng_shard_of_mac(): splitmix64(mac_key) % world (vectorised)."""
    if world <= 1:
        return np.zeros(np.shape(mac_key), dtype=np.uint32)
    with np.errstate(over="ignore"):
        x = np.asarray(mac_key, dtype=np.uint64) + np.uint64(0x9E3779B97F4A7C15)
        x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        x = x ^ (x >> np.uint64(31))
    return (x % np.uint64(world)).astype(np.uint32)


# ---------------------------------------------------------------------------
# addressing helpers
# ---------------------------------------------------------------------------
def sub_mac_key(i) -> np.ndarray:
    """u64 key of subscriber MAC 02:00:ii:ii:ii:ii (mac_to_u64: first byte most significant)."""
    return (np.uint64(0x020000000000) | np.asarray(i, dtype=np.uint64)).astype(np.uint64)


def sub_ip(i) -> np.ndarray:
    """numeric (host-order) private address 100.64.0.0 + i"""
    return (np.uint32(0x64400000) + np.asarray(i, dtype=np.uint32)).astype(np.uint32)


def ip_bytes(ip_numeric) -> np.ndarray:
    """numeric address -> wire-order bytes u8[..., 4]"""
    a = np.asarray(ip_numeric, dtype=np.uint32)
    return np.stack([(a >> 24) & 0xFF, (a >> 16) & 0xFF, (a >> 8) & 0xFF, a & 0xFF], axis=-1).astype(np.uint8)


def mac_bytes(mac_key) -> np.ndarray:
    a = np.asarray(mac_key, dtype=np.uint64)
    return np.stack([(a >> np.uint64(8 * (5 - k))) & np.uint64(0xFF) for k in range(6)], axis=-1).astype(np.uint8)


def port_bytes(port_host) -> np.ndarray:
    a = np.asarray(port_host, dtype=np.uint32)
    return np.stack([(a >> 8) & 0xFF, a & 0xFF], axis=-1).astype(np.uint8)


def ip_checksum(hdr20: np.ndarray) -> np.ndarray:
    """Internet checksum over u8[n,20] headers with the check field zeroed; returns u8[n,2] wire bytes."""
    w = hdr20.astype(np.uint32)
    s = (w[:, 0::2] << 8 | w[:, 1::2]).sum(axis=1)
    s = (s & 0xFFFF) + (s >> 16)
    s = (s & 0xFFFF) + (s >> 16)
    c = (~s) & 0xFFFF
    return np.stack([c >> 8, c & 0xFF], axis=-1).astype(np.uint8)


# ---------------------------------------------------------------------------
# frame headers
# ---------------------------------------------------------------------------
def ipv4_headers(src_mac, dst_mac, src_ip, dst_ip, proto, sport, dport, frame_len, l4_check=None, tcp_flags=0x10,
                 ihl: int = 5) -> np.ndarray:
    """First 64 bytes of n Ethernet/IPv4/{TCP,UDP,ICMP} frames as u8[n,64].

    Addresses are numeric, ports host order; `proto` per frame (6/17/1, others
    get an empty L4).  For ICMP, `sport` is the echo id.  `l4_check` is the
    16-bit checksum field value to place (host order; None = pseudo-random
    non-zero).
    """
    n = max(np.size(a) for a in (src_mac, dst_mac, src_ip, dst_ip, proto, sport, dport, frame_len))
    src_ip = np.broadcast_to(np.asarray(src_ip, dtype=np.uint32), (n,))
    dst_ip = np.broadcast_to(np.asarray(dst_ip, dtype=np.uint32), (n,))
    h = np.zeros((n, 64), dtype=np.uint8)
    h[:, 0:6] = mac_bytes(dst_mac)
    h[:, 6:12] = mac_bytes(src_mac)
    h[:, 12] = 0x08
    h[:, 13] = 0x00
    frame_len = np.broadcast_to(np.asarray(frame_len, dtype=np.uint32), (n,))
    proto = np.broadcast_to(np.asarray(proto, dtype=np.uint32), (n,))
    sport = np.broadcast_to(np.asarray(sport, dtype=np.uint32), (n,))
    dport = np.broadcast_to(np.asarray(dport, dtype=np.uint32), (n,))
    h[:, 14] = 0x40 | ihl
    tot = frame_len - 14
    h[:, 16:18] = port_bytes(tot)
    h[:, 18:20] = port_bytes(np.arange(n) & 0xFFFF)  # id
    h[:, 20] = 0x40  # DF
    h[:, 22] = 64
    h[:, 23] = proto
    h[:, 26:30] = ip_bytes(src_ip)
    h[:, 30:34] = ip_bytes(dst_ip)
    h[:, 24:26] = ip_checksum(h[:, 14:34])
    l4 = 14 + 4 * ihl
    if l4_check is None:
        ck = (splitmix64_array(0x5EED, n) & np.uint64(0xFFFF)).astype(np.uint32)
        ck = np.where(ck == 0, 1, ck)
    else:
        ck = np.broadcast_to(np.asarray(l4_check, dtype=np.uint32), (n,))
    tcp = proto == 6
    udp = proto == 17
    icmp = proto == 1
    if l4 + 20 <= 64:
        pb_s, pb_d, ckb = port_bytes(sport), port_bytes(dport), port_bytes(ck)
        for m, off_ck in ((tcp, 16), (udp, 6)):
            if m.any():
                h[m, l4:l4 + 2] = pb_s[m]
                h[m, l4 + 2:l4 + 4] = pb_d[m]
                h[m, l4 + off_ck:l4 + off_ck + 2] = ckb[m]
        if tcp.any():
            h[tcp, l4 + 12] = 0x50
            h[tcp, l4 + 13] = np.broadcast_to(np.asarray(tcp_flags, dtype=np.uint8), (n,))[tcp]
            h[tcp, l4 + 14:l4 + 16] = [0xFF, 0xFF]
        if udp.any():
            h[udp, l4 + 4:l4 + 6] = port_bytes(frame_len - l4)[udp]
        if icmp.any():
            h[icmp, l4] = 8
            h[icmp, l4 + 2:l4 + 4] = ckb[icmp]
            h[icmp, l4 + 4:l4 + 6] = pb_s[icmp]
            h[icmp, l4 + 6:l4 + 8] = port_bytes(np.arange(n) & 0xFFFF)[icmp]
    return h


IMIX_SIZES = np.array([64, 594, 1518], dtype=np.uint32)
IMIX_WEIGHTS = np.array([7, 4, 1], dtype=np.float64)


def imix_lengths(n: int, seed: int) -> np.ndarray:
    """7:4:1 mix of 64/594/1518-byte frames (average 361.8 B)."""
    r = splitmix64_array(seed, n) % np.uint64(12)
    return np.where(r < 7, 64, np.where(r < 11, 594, 1518)).astype(np.uint32)


def pack_arena(headers: np.ndarray, lens: np.ndarray):
    """Lay frames out in one arena with 16-byte aligned slots.

    Returns (arena u8[], off16 u32[n]).  Only the header bytes carry data; the
    payload is zero (no program reads it).
    """
    n = headers.shape[0]
    slot = ((lens.astype(np.uint64) + 15) // 16)
    off16 = np.zeros(n, dtype=np.uint64)
    np.cumsum(slot[:-1], out=off16[1:])
    total = int((off16[-1] + slot[-1]) * 16) if n else 0
    arena = np.zeros(total + 64, dtype=np.uint8)
    hw = headers.shape[1]
    idx = (off16 * 16)[:, None] + np.arange(hw, dtype=np.uint64)[None, :]
    keep = np.arange(hw)[None, :] < np.minimum(lens, hw)[:, None]
    arena[idx[keep]] = headers[keep]
    return arena, off16.astype(np.uint32)


# ---------------------------------------------------------------------------
# map contents
# ---------------------------------------------------------------------------
def bindings(n_subs: int, mode: int = L.ANTISPOOF_STRICT):
    keys = sub_mac_key(np.arange(n_subs))
    v = np.zeros(n_subs, dtype=L.subscriber_binding)
    v["ipv4_addr"] = ip_bytes(sub_ip(np.arange(n_subs)))
    v["ipv4_valid"] = 1
    v["mode"] = mode
    return keys, v


# The reference's DefaultPolicies (pkg/radius/policy.go:70-128):
# (name, download_bps, upload_bps, burst_size, priority)
QOS_TIERS = (
    ("residential-50mbps", 50_000_000, 10_000_000, 1_000_000, 4),
    ("residential-100mbps", 100_000_000, 20_000_000, 2_000_000, 4),
    ("residential-500mbps", 500_000_000, 50_000_000, 5_000_000, 4),
    ("residential-1gbps", 1_000_000_000, 100_000_000, 10_000_000, 4),
    ("business-100mbps", 100_000_000, 100_000_000, 2_000_000, 6),
    ("business-1gbps", 1_000_000_000, 1_000_000_000, 10_000_000, 6),
    ("guest", 10_000_000, 5_000_000, 500_000, 2),
    ("unlimited", 0, 0, 0, 4),
)


def qos_default_burst(bps: int) -> int:
    """clamp(bps/8, 64 KiB, 10 MiB) with the Go manager's u32 truncation (pkg/qos/manager.go:181-209)."""
    b = (bps // 8) & 0xFFFFFFFF
    return int(min(max(b, 65536), 10 * 1024 * 1024))


def qos_buckets(n_subs: int, upload: bool = True):
    """token_bucket values exactly as SetSubscriberPolicy -> SetSubscriberQoS writes them
    (pkg/qos/manager.go:167-245): tokens = burst, last_update = 0; the download bucket uses the
    policy's BurstSize (default rule when 0), the upload bucket always recomputes its burst."""
    keys = ip_bytes(sub_ip(np.arange(n_subs)))
    v = np.zeros(n_subs, dtype=L.token_bucket)
    tier = np.arange(n_subs) % len(QOS_TIERS)
    if upload:
        rates = [t[2] for t in QOS_TIERS]
        bursts = [qos_default_burst(t[2]) for t in QOS_TIERS]
    else:
        rates = [t[1] for t in QOS_TIERS]
        bursts = [t[3] if t[3] else qos_default_burst(t[1]) for t in QOS_TIERS]
    v["rate_bps"] = np.array(rates, dtype=np.uint64)[tier]
    v["burst_bytes"] = np.array(bursts, dtype=np.uint32)[tier]
    v["tokens"] = v["burst_bytes"]
    v["priority"] = np.array([t[4] for t in QOS_TIERS], dtype=np.uint8)[tier]
    return keys, v


def nat_blocks(n_subs: int, first_public_ip: int = 0xCB007100, ports_per_sub: int = 1024, port_lo: int = 1024,
               port_hi: int = 65535):
    """subscriber_nat values as Manager.AllocateNAT produces them (pkg/nat/manager.go:398-494):
    subscriber k of a public IP gets ports [lo + k*pps, lo + (k+1)*pps - 1], 63 subscribers per IP by
    default, sequential subscriber ids from 1.  Returns (keys u8[n,4], values, public_ips numeric)."""
    per_ip = (port_hi - port_lo + 1) // ports_per_sub
    idx = np.arange(n_subs)
    ipn = first_public_ip + idx // per_ip
    k = idx % per_ip
    v = np.zeros(n_subs, dtype=L.subscriber_nat)
    v["block"]["public_ip"] = ip_bytes(ipn)
    v["block"]["port_start"] = port_lo + k * ports_per_sub
    v["block"]["port_end"] = port_lo + (k + 1) * ports_per_sub - 1
    v["block"]["next_port"] = port_lo + k * ports_per_sub
    v["block"]["subscriber_id"] = idx + 1
    v["block"]["block_size_log2"] = int(np.log2(ports_per_sub))
    keys = ip_bytes(sub_ip(idx))
    return keys, v, np.unique(ipn).astype(np.uint32)


def nat_config(flags: int = 0x0F, ports_per_sub: int = 1024):
    v = np.zeros(1, dtype=L.nat_config)
    v["flags"] = flags
    v["port_range_start"] = 1024
    v["port_range_end"] = 65535
    v["default_ports_per_sub"] = ports_per_sub
    return v


def flows(n_subs: int, flows_per_sub: int, seed: int):
    """Distinct 5-tuples: 61 % TCP, 37 % UDP, 2 % ICMP echo.  Returns a dict of arrays of
    length n_subs*flows_per_sub: sub, proto, sport, dport, dst_ip (numeric/host order)."""
    n = n_subs * flows_per_sub
    r = splitmix64_array(seed, n)
    sub = np.repeat(np.arange(n_subs, dtype=np.uint32), flows_per_sub)
    j = np.tile(np.arange(flows_per_sub, dtype=np.uint32), n_subs)
    sel = (r % np.uint64(100)).astype(np.uint32)
    proto = np.where(sel < 61, 6, np.where(sel < 98, 17, 1)).astype(np.uint32)
    sport = (10000 + j * 7 + (sub % 5)).astype(np.uint32)  # unique per subscriber
    dport = np.where(proto == 1, 0, np.array([443, 80, 53, 8080, 123, 5000], dtype=np.uint32)[(r >> np.uint64(8)) % np.uint64(6)])
    dst_ip = (np.uint32(0x08080000) + ((r >> np.uint64(16)) & np.uint64(0xFFFF)).astype(np.uint32)).astype(np.uint32)
    return {"sub": sub, "proto": proto, "sport": sport, "dport": dport.astype(np.uint32), "dst_ip": dst_ip}


def flow_frames(fl: dict, pick: np.ndarray, lens: np.ndarray, gw_mac: int = 0x02FFFFFFFFFE, udp_zero_every: int = 0):
    """Headers for frames of flows fl[pick] (upstream direction, subscriber -> internet)."""
    sub = fl["sub"][pick]
    ck = None
    if udp_zero_every:
        base = (splitmix64_array(0xC0FFEE, len(pick)) & np.uint64(0xFFFF)).astype(np.uint32)
        base = np.where(base == 0, 1, base)
        zero = (fl["proto"][pick] == 17) & ((pick % udp_zero_every) == 0)
        ck = np.where(zero, 0, base)
    return ipv4_headers(sub_mac_key(sub), np.uint64(gw_mac), sub_ip(sub), fl["dst_ip"][pick], fl["proto"][pick],
                        fl["sport"][pick], fl["dport"][pick], lens, l4_check=ck)


# ---------------------------------------------------------------------------
# DHCPv6 (include/bng_b200.h: the DHCPv6 fast path)
# ---------------------------------------------------------------------------
DHCPV6_ALL_SERVERS = bytes.fromhex("ff020000000000000000000000010002")


def dhcpv6_option(code: int, data: bytes = b"") -> bytes:
    return code.to_bytes(2, "big") + len(data).to_bytes(2, "big") + bytes(data)


def dhcpv6_ia(code: int, iaid: int, t1: int = 0, t2: int = 0, sub: bytes = b"") -> bytes:
    """An IA_NA (3) or IA_PD (25) option as a client sends it: IAID, T1, T2, then any sub-options."""
    return dhcpv6_option(code, iaid.to_bytes(4, "big") + t1.to_bytes(4, "big") + t2.to_bytes(4, "big") + sub)


def udp6_checksum(src: bytes, dst: bytes, udp: bytes) -> int:
    """The UDP checksum over the IPv6 pseudo-header (RFC 8200 §8.1) of a UDP datagram whose checksum field is 0."""
    data = src + dst + len(udp).to_bytes(4, "big") + b"\x00\x00\x00\x11" + udp
    if len(data) & 1:
        data += b"\x00"
    s = int(np.frombuffer(data, ">u2").astype(np.uint64).sum())
    while s >> 16:
        s = (s & 0xFFFF) + (s >> 16)
    c = ~s & 0xFFFF
    return c or 0xFFFF


def dhcpv6_frame(src_mac: bytes, msg_type: int, xid: int, options: bytes, dst_mac: bytes = b"\x33\x33\x00\x01\x00\x02",
                 src_ip: bytes | None = None, dst_ip: bytes = DHCPV6_ALL_SERVERS, tags=(), sport: int = 546,
                 dport: int = 547, next_header: int = 17, hop_limit: int = 1) -> bytes:
    """An Ethernet frame carrying one DHCPv6 client message: type, 24-bit transaction id, the options as given.
    tags: (tpid, vid) pairs outermost first.  The source defaults to the link-local EUI-64 address of src_mac."""
    if src_ip is None:
        eui = bytes([src_mac[0] ^ 2]) + src_mac[1:3] + b"\xff\xfe" + src_mac[3:6]
        src_ip = b"\xfe\x80" + bytes(6) + eui
    msg = bytes([msg_type]) + (int(xid) & 0xFFFFFF).to_bytes(3, "big") + options
    udp = sport.to_bytes(2, "big") + dport.to_bytes(2, "big") + (8 + len(msg)).to_bytes(2, "big") + b"\x00\x00" + msg
    ck = udp6_checksum(src_ip, dst_ip, udp)
    udp = udp[:6] + ck.to_bytes(2, "big") + udp[8:]
    ip = (b"\x60\x00\x00\x00" + len(udp).to_bytes(2, "big") + bytes([next_header, hop_limit]) + src_ip + dst_ip)
    l2 = bytes(dst_mac) + bytes(src_mac)
    for tpid, vid in tags:
        l2 += tpid.to_bytes(2, "big") + (vid & 0xFFF).to_bytes(2, "big")
    return l2 + b"\x86\xdd" + ip + udp


def dhcpv6_client_key(duid: bytes) -> np.ndarray:
    k = np.zeros(1, L.bng_dhcpv6_client_key)
    k["duid_len"] = len(duid)
    k["duid"][0, :len(duid)] = np.frombuffer(bytes(duid), np.uint8)
    return k


def dhcpv6_duid(i: int, length: int = 14) -> bytes:
    """A DUID-LLT-shaped client identifier of `length` bytes for client i (distinct per i for length >= 5)."""
    base = b"\x00\x01\x00\x01" + int(0x2A000000 + i).to_bytes(4, "big") + (0x020000000000 + i).to_bytes(6, "big")
    base += bytes(32)
    b = bytearray(base[:length])
    if length < 10:  # keep short DUIDs distinct
        v = (i * 2654435761) & ((1 << (8 * length)) - 1)
        b = bytearray(v.to_bytes(length, "big"))
    return bytes(b)


# ---------------------------------------------------------------------------
# ICMPv6 Router and Neighbor Solicitations (include/bng_b200.h: bng_nd_enable)
# ---------------------------------------------------------------------------
ALL_NODES = bytes.fromhex("ff020000000000000000000000000001")
ALL_ROUTERS = bytes.fromhex("ff020000000000000000000000000002")


def link_local(mac: bytes) -> bytes:
    """The EUI-64 link-local address of a MAC (RFC 4291 appendix A)."""
    return b"\xfe\x80" + bytes(6) + bytes([mac[0] ^ 2]) + mac[1:3] + b"\xff\xfe" + mac[3:6]


def solicited_node(addr: bytes) -> bytes:
    """ff02::1:ffXX:XXXX with the address's low 24 bits (RFC 4291 §2.7.1)."""
    return bytes.fromhex("ff0200000000000000000001ff") + bytes(addr[13:16])


def icmp6_checksum(src: bytes, dst: bytes, msg: bytes) -> int:
    """The ICMPv6 checksum (RFC 4443 §2.3) of a message whose checksum field is 0."""
    data = src + dst + len(msg).to_bytes(4, "big") + b"\x00\x00\x00\x3a" + msg
    if len(data) & 1:
        data += b"\x00"
    s = int(np.frombuffer(data, ">u2").astype(np.uint64).sum())
    while s >> 16:
        s = (s & 0xFFFF) + (s >> 16)
    return ~s & 0xFFFF


def icmp6_frame(src_mac: bytes, msg: bytes, src_ip: bytes, dst_ip: bytes, dst_mac: bytes | None = None, tags=(),
                hop_limit: int = 255, next_header: int = 58, checksum: bool = True) -> bytes:
    """An Ethernet frame carrying one ICMPv6 message (bytes 2-3, the checksum, filled in unless checksum=False).
    dst_mac defaults to the destination's multicast MAC (33:33 + its low 32 bits); tags: (tpid, vid) outermost first."""
    if checksum:
        msg = msg[:2] + b"\x00\x00" + msg[4:]
        msg = msg[:2] + icmp6_checksum(src_ip, dst_ip, msg).to_bytes(2, "big") + msg[4:]
    if dst_mac is None:
        dst_mac = b"\x33\x33" + dst_ip[12:16]
    ip = b"\x60\x00\x00\x00" + len(msg).to_bytes(2, "big") + bytes([next_header, hop_limit]) + src_ip + dst_ip
    l2 = bytes(dst_mac) + bytes(src_mac)
    for tpid, vid in tags:
        l2 += tpid.to_bytes(2, "big") + (vid & 0xFFF).to_bytes(2, "big")
    return l2 + b"\x86\xdd" + ip + msg


def nd_option(kind: int, data: bytes) -> bytes:
    """An ND option (RFC 4861 §4.6): type, length in units of 8 bytes, data padded to the length."""
    n = (2 + len(data) + 7) // 8
    return bytes([kind, n]) + data + bytes(n * 8 - 2 - len(data))


def rs_frame(src_mac: bytes, src_ip: bytes | None = None, dst_ip: bytes = ALL_ROUTERS, slla: bool = True,
             options: bytes = b"", code: int = 0, **kw) -> bytes:
    """A Router Solicitation (RFC 4861 §4.1) from src_mac, from its link-local address unless src_ip is given, with a
    Source Link-Layer Address option when slla."""
    if src_ip is None:
        src_ip = link_local(src_mac)
    msg = bytes([133, code, 0, 0]) + bytes(4) + (nd_option(1, src_mac) if slla else b"") + options
    return icmp6_frame(src_mac, msg, src_ip, dst_ip, **kw)


def ns_frame(src_mac: bytes, target: bytes, src_ip: bytes | None = None, dst_ip: bytes | None = None, slla: bool = True,
             options: bytes = b"", code: int = 0, **kw) -> bytes:
    """A Neighbor Solicitation (RFC 4861 §4.3) for target, to its solicited-node address unless dst_ip is given; src_ip
    defaults to src_mac's link-local address (pass bytes(16) for duplicate address detection)."""
    if src_ip is None:
        src_ip = link_local(src_mac)
    if dst_ip is None:
        dst_ip = solicited_node(target)
    msg = bytes([135, code, 0, 0]) + bytes(4) + bytes(target) + (nd_option(1, src_mac) if slla else b"") + options
    return icmp6_frame(src_mac, msg, src_ip, dst_ip, **kw)
