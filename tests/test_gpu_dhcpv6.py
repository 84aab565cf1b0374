"""The DHCPv6 fast path (bng_dhcpv6_enable, include/bng_b200.h): dhcp_fastpath_prog answers a bound client's Solicit,
Request, Renew and Rebind from dhcpv6_bindings with what pkg/dhcpv6's buildAdvertise / buildReply would send.

Expected results: the oracle's own dhcp_fastpath_prog runs on the whole batch and gives every verdict, byte, length and
stats_map counter.  The rule, restated below, then overrides verdict, bytes and length of the frames it answers and
gives dhcpv6_stats.  The program writes no table and no frame's outcome depends on another, so that combination is the
specification.  The restatement is checked on the CPU by a separate RFC 8415 decoder and by literal byte vectors
worked out from pkg/dhcpv6/protocol.go's serialization."""
import errno

import numpy as np
import pytest

import harness
from bng_b200 import Dataplane
from bng_b200 import layouts as L
from bng_b200 import synth as S

FEEDS = [False, True, "device"]
FEED_IDS = ["pageable", "pinned", "device"]
T0 = 1_000_000 * 1_000_000_000  # 1e6 s
ST = {n: i for i, n in enumerate(L.DHCPV6_STATS)}
SERVER_MAC = bytes.fromhex("02aabbccdd01")
SERVER_IP = bytes.fromhex("fe800000000000000000000000000001")
SERVER_DUID = bytes.fromhex("000300010a0b0c0d0e0f")  # DUID-LL, 10 bytes
DNS = (bytes.fromhex("20010db8000000000000000000000053"), bytes.fromhex("20010db8000000000000000000000054"))


# ---------------------------------------------------------------------------
# the rule, restated
# ---------------------------------------------------------------------------
def config(dns_count=2, duid=SERVER_DUID, server_ip=SERVER_IP):
    return {"mac": SERVER_MAC, "ip": server_ip, "duid": duid, "dns": DNS[:dns_count]}


def cfg_value(cfg):
    v = np.zeros(1, L.bng_dhcpv6_server_config)
    if cfg is None:
        return v
    v["server_mac"][0] = np.frombuffer(cfg["mac"], np.uint8)
    v["duid_len"] = len(cfg["duid"])
    v["dns_count"] = len(cfg["dns"])
    v["server_ip"][0] = np.frombuffer(cfg["ip"], np.uint8)
    v["duid"][0, :len(cfg["duid"])] = np.frombuffer(cfg["duid"], np.uint8)
    for k, d in enumerate(cfg["dns"]):
        v["dns"][0, k] = np.frombuffer(d, np.uint8)
    return v


class Binding:
    def __init__(self, mac, na=True, pd=True, iaid_na=1, iaid_pd=2, pref=3600, valid=7200, expires_s=2_000_000,
                 addr=None, pd_len=56, prefix=None, i=0):
        self.mac, self.iaid_na, self.iaid_pd, self.pref, self.valid = bytes(mac), iaid_na, iaid_pd, pref, valid
        self.flags = (L.DHCPV6_NA if na else 0) | (L.DHCPV6_PD if pd else 0)
        self.expires_s, self.pd_len = expires_s, pd_len
        self.addr = addr or bytes.fromhex("20010db8ffff0000000000000000") + i.to_bytes(2, "big")
        self.prefix = prefix or bytes.fromhex("20010db8") + (i & 0xFFFF).to_bytes(2, "big") + bytes(10)

    def value(self):
        v = np.zeros(1, L.bng_dhcpv6_binding)
        v["mac"][0] = np.frombuffer(self.mac, np.uint8)
        v["flags"], v["pd_len"], v["iaid_na"], v["iaid_pd"] = self.flags, self.pd_len, self.iaid_na, self.iaid_pd
        v["preferred_lft"], v["valid_lft"], v["expires_s"] = self.pref, self.valid, self.expires_s
        v["addr"][0] = np.frombuffer(self.addr, np.uint8)
        v["prefix"][0] = np.frombuffer(self.prefix, np.uint8)
        return v


def opt(code, data=b""):
    return S.dhcpv6_option(code, data)


def build_reply(msg_type, xid, client_id, cfg, b, want_na, want_pd, rapid):
    """What buildAdvertise / buildReply (+ Rapid Commit) serialize, in their order."""
    adv = msg_type == 1 and not rapid
    t1, t2 = (b.pref // 2) & 0xFFFFFFFF, ((b.pref * 4) & 0xFFFFFFFF) // 5
    o = opt(1, client_id) + opt(2, cfg["duid"])
    if adv:
        o += opt(7, b"\xff")
    if want_na:
        o += opt(3, b.iaid_na.to_bytes(4, "big") + t1.to_bytes(4, "big") + t2.to_bytes(4, "big") +
                 opt(5, b.addr + b.pref.to_bytes(4, "big") + b.valid.to_bytes(4, "big")))
    if want_pd:
        o += opt(25, b.iaid_pd.to_bytes(4, "big") + t1.to_bytes(4, "big") + t2.to_bytes(4, "big") +
                 opt(26, b.pref.to_bytes(4, "big") + b.valid.to_bytes(4, "big") + bytes([b.pd_len]) + b.prefix))
    if cfg["dns"]:
        o += opt(23, b"".join(cfg["dns"]))
    if not adv:
        o += opt(13, b"\x00\x00Success")
    if msg_type == 1 and rapid:
        o += opt(14)
    return bytes([2 if adv else 7]) + xid + o


def rule(f, ln, dlen, room, now_ns, cfg, binds):
    """(counters, reply frame or None) for one frame that dhcp_one passed as not IPv4; ([], None): not a candidate.
    f: the frame's bytes (at least dlen of them)."""
    if dlen < 14:
        return [], None
    et, l3 = f[12:14], 14
    if et in (b"\x81\x00", b"\x88\xa8"):
        if dlen < 18:
            return [], None
        et, l3 = f[16:18], 18
        if et == b"\x81\x00":
            if dlen < 22:
                return [], None
            et, l3 = f[20:22], 22
    if et != b"\x86\xdd" or l3 + 48 > dlen:
        return [], None
    if f[l3] >> 4 != 6 or f[l3 + 6] != 17 or f[l3 + 42:l3 + 44] != b"\x02\x23":
        return [], None
    dst = f[l3 + 24:l3 + 40]
    if dst != S.DHCPV6_ALL_SERVERS and dst != (cfg["ip"] if cfg else bytes(16)):
        return [], None
    c = ["total"]
    udp, m = l3 + 40, l3 + 48
    if cfg is None or ln > 448:
        return c + ["unsupported"], None
    ulen = int.from_bytes(f[udp + 4:udp + 6], "big")
    if ulen < 12 or udp + ulen > dlen:
        return c + ["malformed"], None
    t = f[m]
    if t not in (1, 3, 5, 6):
        return c + ["unsupported"], None
    c.append({1: "solicit", 3: "request", 5: "renew", 6: "rebind"}[t])
    end, o, opts = udp + ulen, m + 4, []
    while o < end:
        if o + 4 > end or len(opts) == 32:
            return c + ["malformed"], None
        code, olen = int.from_bytes(f[o:o + 2], "big"), int.from_bytes(f[o + 2:o + 4], "big")
        if o + 4 + olen > end:
            return c + ["malformed"], None
        opts.append((code, bytes(f[o + 4:o + 4 + olen])))
        o += 4 + olen
    get = lambda k: [d for cd, d in opts if cd == k]
    cid, sid, na, pd = get(1), get(2), get(3), get(25)
    bad = (len(cid) != 1 or not 1 <= len(cid[0]) <= 31 or get(4) or len(na) > 1 or len(pd) > 1
           or any(len(x) < 12 for x in na + pd) or not (na or pd))
    if t in (1, 6):
        bad = bad or sid
    else:
        bad = bad or len(sid) != 1 or sid[0] != cfg["duid"]
    if bad:
        return c + ["unsupported"], None
    b = binds.get(cid[0])
    if b is None or b.mac != bytes(f[6:12]):
        return c + ["miss"], None
    if now_ns // 1_000_000_000 > b.expires_s:
        return c + ["expired"], None
    if (na and (not b.flags & 1 or int.from_bytes(na[0][:4], "big") != b.iaid_na)) or \
       (pd and (not b.flags & 2 or int.from_bytes(pd[0][:4], "big") != b.iaid_pd)):
        return c + ["unsupported"], None
    rapid = bool(get(14))
    msg = build_reply(t, bytes(f[m + 1:m + 4]), cid[0], cfg, b, bool(na), bool(pd), rapid)
    total = m + len(msg)
    if total > room:
        return c + ["no_room"], None
    ul = 8 + len(msg)
    udpb = b"\x02\x23\x02\x22" + ul.to_bytes(2, "big") + b"\x00\x00" + msg
    ck = S.udp6_checksum(cfg["ip"], bytes(f[l3 + 8:l3 + 24]), udpb)
    udpb = udpb[:6] + ck.to_bytes(2, "big") + udpb[8:]
    ip = b"\x60\x00\x00\x00" + ul.to_bytes(2, "big") + b"\x11\x40" + cfg["ip"] + bytes(f[l3 + 8:l3 + 24])
    out = bytes(f[6:12]) + cfg["mac"] + bytes(f[12:l3]) + ip + udpb
    return c + ["advertise" if msg[0] == 2 else "reply"], out


# ---------------------------------------------------------------------------
# an independent RFC 8415 decoder (CPU checks of the restatement)
# ---------------------------------------------------------------------------
def decode(frame):
    l3 = 14
    while frame[l3 - 2:l3] in (b"\x81\x00", b"\x88\xa8"):
        l3 += 4
    assert frame[l3 - 2:l3] == b"\x86\xdd"
    ip, udp = frame[l3:l3 + 40], frame[l3 + 40:]
    plen = int.from_bytes(ip[4:6], "big")
    assert ip[0] == 0x60 and ip[6] == 17 and ip[7] == 64 and plen == len(udp)
    assert udp[:4] == b"\x02\x23\x02\x22" and int.from_bytes(udp[4:6], "big") == len(udp)
    assert S.udp6_checksum(ip[8:24], ip[24:40], udp[:6] + b"\0\0" + udp[8:]) == int.from_bytes(udp[6:8], "big")
    msg = udp[8:]
    opts, o = [], 4
    while o < len(msg):
        code, n = int.from_bytes(msg[o:o + 2], "big"), int.from_bytes(msg[o + 2:o + 4], "big")
        opts.append((code, msg[o + 4:o + 4 + n]))
        o += 4 + n
    assert o == len(msg)
    return {"dst_mac": frame[:6], "src_mac": frame[6:12], "src": ip[8:24], "dst": ip[24:40], "type": msg[0],
            "xid": msg[1:4], "opts": opts}


def ia_decode(data, sub_code):
    iaid, t1, t2 = (int.from_bytes(data[k:k + 4], "big") for k in (0, 4, 8))
    sc, sl = int.from_bytes(data[12:14], "big"), int.from_bytes(data[14:16], "big")
    assert sc == sub_code and 16 + sl == len(data)
    return iaid, t1, t2, data[16:]


def client(i=0, duid_len=14, tags=(), **kw):
    mac = bytes.fromhex("02000000") + i.to_bytes(2, "big")
    return mac, S.dhcpv6_duid(i, duid_len)


def request(mac, duid, t=1, xid=0x123456, na=1, pd=2, sid=None, rapid=False, extra=b"", tags=(), dst_ip=None, **kw):
    o = opt(1, duid)
    if sid is not None:
        o += opt(2, sid)
    if rapid:
        o += opt(14)
    if na is not None:
        o += S.dhcpv6_ia(3, na)
    if pd is not None:
        o += S.dhcpv6_ia(25, pd)
    o += opt(6, b"\x00\x17\x00\x18") + extra  # Option Request: DNS servers, domain list
    return S.dhcpv6_frame(mac, t, xid, o, tags=tags, dst_ip=dst_ip or S.DHCPV6_ALL_SERVERS, **kw)


def test_restatement_against_decoder():
    cfg = config(2)
    for t, rapid, want in ((1, False, 2), (1, True, 7), (3, False, 7), (5, False, 7), (6, False, 7)):
        for na, pd in ((1, None), (None, 2), (1, 2)):
            for tags in ((), ((0x8100, 7),), ((0x88A8, 7), (0x8100, 9))):
                mac, duid = client(3, 18)
                b = Binding(mac, iaid_na=1, iaid_pd=2, pref=0xFFFFFFFF, valid=0xFFFFFFFF, i=3)
                f = request(mac, duid, t, 0xABCDEF, na, pd, SERVER_DUID if t in (3, 5) else None, rapid, tags=tags)
                c, out = rule(f, len(f), len(f), 2048, T0, cfg, {duid: b})
                assert c[-1] == ("advertise" if want == 2 else "reply"), c
                d = decode(out)
                assert d["type"] == want and d["xid"] == bytes.fromhex("abcdef")
                assert d["dst_mac"] == mac and d["src_mac"] == SERVER_MAC and d["src"] == SERVER_IP
                assert d["dst"] == f[14 + 4 * len(tags) + 8:14 + 4 * len(tags) + 24]
                codes = [k for k, _ in d["opts"]]
                expect = [1, 2] + ([7] if want == 2 else []) + ([3] if na else []) + ([25] if pd else []) + [23]
                expect += [13] if want == 7 else []
                expect += [14] if t == 1 and rapid else []
                assert codes == expect
                od = dict(d["opts"])
                assert od[1] == duid and od[2] == SERVER_DUID and od[23] == DNS[0] + DNS[1]
                if na:
                    iaid, t1, t2, sub = ia_decode(od[3], 5)
                    assert (iaid, t1, t2) == (1, 2147483647, 858993458)
                    assert sub == b.addr + b.pref.to_bytes(4, "big") + b.valid.to_bytes(4, "big")
                if pd:
                    iaid, t1, t2, sub = ia_decode(od[25], 26)
                    assert (iaid, t1, t2) == (2, 2147483647, 858993458)
                    assert sub[8] == 56 and sub[9:25] == b.prefix
                if want == 7:
                    assert od[13] == b"\x00\x00Success"


def test_literal_vectors():
    """Three messages worked out by hand from protocol.go's Serialize / SerializeOptions (2-byte code, 2-byte length,
    data) and server.go's option order, for client DUID 00030001020000000005, server DUID 000300010a0b0c0d0e0f,
    IA_NA IAID 1 -> 2001:db8:ffff::5, preferred 3600, valid 7200 (T1 1800, T2 2880), one DNS server."""
    cfg = config(1)
    mac = bytes.fromhex("020000000005")
    duid = bytes.fromhex("00030001020000000005")
    b = Binding(mac, pd=False, iaid_na=1, addr=bytes.fromhex("20010db8ffff00000000000000000005"))
    head = "0001000a00030001020000000005" + "0002000a000300010a0b0c0d0e0f"
    ia_na = ("00030028" + "00000001" + "00000708" + "00000b40" + "00050018" + "20010db8ffff00000000000000000005" +
             "00000e10" + "00001c20")
    dns = "00170010" + "20010db8000000000000000000000053"
    status = "000d0009" + "0000" + "53756363657373"
    vectors = {
        (1, False): "02" + "0a0b0c" + head + "000700" + "01ff" + ia_na + dns,
        (3, False): "07" + "0a0b0c" + head + ia_na + dns + status,
        (1, True): "07" + "0a0b0c" + head + ia_na + dns + status + "000e0000",
    }
    for (t, rapid), hexmsg in vectors.items():
        f = request(mac, duid, t, 0x0A0B0C, 1, None, SERVER_DUID if t == 3 else None, rapid)
        _, out = rule(f, len(f), len(f), 2048, T0, cfg, {duid: b})
        assert out[62:].hex() == hexmsg


# ---------------------------------------------------------------------------
# expected results and the run
# ---------------------------------------------------------------------------
def oracle_kind():
    from oracle import pyoracle
    return "reference" if pyoracle.available("reference") else "port"


def expected(arena, lens, off16, stride, now, now_v, cfg, binds):
    """The oracle's dhcp_fastpath_prog on the whole batch, then the restated rule on the frames it passes."""
    ob = harness.OracleBackend(oracle_kind())
    try:
        a, l = arena.copy(), lens.copy()
        v = ob.run("dhcp_fastpath_prog", a, l, now, off16, stride, None, now_v=now_v).copy()
        st = ob.stats("stats_map")
    finally:
        ob.close()
    cnt = np.zeros(12, np.uint64)
    for i in range(len(lens)):
        if v[i] != 2:
            continue
        off = int(off16[i]) * 16 if off16 is not None else i * stride
        ln = int(lens[i])
        dlen = ln if off16 is not None else min(ln, stride)
        room = stride if off16 is None else (ln + 15) & ~15
        c, out = rule(arena[off:off + dlen].tobytes(), ln, dlen, room, int(now_v[i]) if now_v is not None else now,
                      cfg, binds)
        for k in c:
            cnt[ST[k]] += 1
        if out is not None:
            v[i] = 3
            l[i] = len(out)
            a[off:off + len(out)] = np.frombuffer(out, np.uint8)
            a[off + len(out):off + ((len(out) + 15) & ~15)] = 0
    return a, l, v, st, cnt


def gpu_setup(dp, cfg, binds, on=True):
    if cfg is not None:
        assert dp.update("dhcpv6_server_config", np.uint32(0), cfg_value(cfg)) == 0
    if binds:
        ks = np.concatenate([S.dhcpv6_client_key(k) for k in binds])
        vs = np.concatenate([b.value() for b in binds.values()])
        assert dp.update_batch("dhcpv6_bindings", ks, vs) == 0
    dp.dhcpv6_enable(on)


def run_gpu(feed, arena, lens, off16, stride, now, now_v, cfg, binds, dp=None, **opts):
    be = harness.GpuBackend(dp=dp, pinned=feed, **opts)
    if dp is None:
        gpu_setup(be.dp, cfg, binds)
    a, l = arena.copy(), lens.copy()
    v = be.run("dhcp_fastpath_prog", a, l, now, off16, stride, None, now_v=now_v)
    res = a, l, v, be.stats("stats_map"), be.stats("dhcpv6_stats")
    if dp is None:
        be.close()
    return res


def check(got, want, what=""):
    ga, gl, gv, gs, g6 = got
    wa, wl, wv, ws, w6 = want
    bad = np.nonzero((gv != wv) | (gl != wl))[0]
    assert not len(bad), f"{what}: frames {bad[:10]} verdict {gv[bad[:10]]} vs {wv[bad[:10]]} len {gl[bad[:10]]} vs {wl[bad[:10]]}"
    assert np.array_equal(gs, ws), f"{what}: stats_map {gs} vs {ws}"
    assert np.array_equal(g6, w6), f"{what}: dhcpv6_stats {dict(zip(L.DHCPV6_STATS, g6))} vs {dict(zip(L.DHCPV6_STATS, w6))}"
    diff = np.nonzero(ga != wa)[0]
    assert not len(diff), f"{what}: arena bytes differ at {diff[:10]}"


def dhcpv4_discover(mac, xid=1):
    """A DHCPv4 DISCOVER from a MAC with no lease: the oracle counts it a miss."""
    bootp = bytearray(240)
    bootp[0], bootp[1], bootp[2] = 1, 1, 6
    bootp[4:8] = xid.to_bytes(4, "big")
    bootp[28:34] = mac
    bootp[236:240] = bytes.fromhex("63825363")
    dh = bytes(bootp) + bytes([53, 1, 1, 255]) + bytes(60)
    udp = (68).to_bytes(2, "big") + (67).to_bytes(2, "big") + (8 + len(dh)).to_bytes(2, "big") + b"\0\0" + dh
    ip = bytearray(b"\x45\x00" + (20 + len(udp)).to_bytes(2, "big") + bytes(4) + b"\x40\x11\x00\x00" + bytes(4) + b"\xff" * 4)
    return b"\xff" * 6 + mac + b"\x08\x00" + bytes(ip) + udp


def case_corpus(seed=1):
    """(frames, binds, cfg) covering the rule's branches."""
    rng = np.random.default_rng(seed)
    cfg = config(2)
    binds, frames = {}, []
    for i, dl in enumerate((1, 10, 14, 18, 31)):
        mac, duid = client(100 + i, dl)
        binds[duid] = Binding(mac, iaid_na=7, iaid_pd=8, i=100 + i)
        for t in range(1, 14):
            for rapid in (False, True):
                sid = SERVER_DUID if t in (3, 5) else None
                frames.append(request(mac, duid, t, rng.integers(1 << 24), 7, 8, sid, rapid))
    mac, duid = client(1, 14)
    binds[duid] = Binding(mac, iaid_na=7, iaid_pd=8, i=1)
    emac, eduid = client(2, 14)
    binds[eduid] = Binding(emac, iaid_na=7, iaid_pd=8, i=2, expires_s=T0 // 10**9 + 50)
    nmac, nduid = client(3, 14)
    binds[nduid] = Binding(nmac, pd=False, iaid_na=7, i=3)
    for t in (1, 3, 5, 6):
        sid = SERVER_DUID if t in (3, 5) else None
        for na, pd in ((7, None), (None, 8), (7, 8), (9, 8), (7, 9), (None, None)):
            frames.append(request(mac, duid, t, 5, na, pd, sid))
        frames.append(request(nmac, nduid, t, 5, 7, 8, sid))  # an IA the binding lacks
        frames.append(request(mac, duid, t, 5, 7, 8, sid, extra=S.dhcpv6_ia(3, 7)))  # two IA_NAs
        frames.append(request(mac, duid, t, 5, 7, 8, sid, extra=S.dhcpv6_ia(4, 7)))  # IA_TA
        frames.append(request(mac, duid, t, 5, 7, 8, None))  # Server ID missing
        frames.append(request(mac, duid, t, 5, 7, 8, b"\x00\x03\x00\x01" + bytes(6)))  # foreign / present
        frames.append(request(mac, duid, t, 5, 7, 8, SERVER_DUID))
        frames.append(request(mac, S.dhcpv6_duid(999, 14), t, 5, 7, 8, sid))  # unknown DUID
        frames.append(request(emac, eduid, t, 5, 7, 8, sid))  # straddles expiry with per-frame clocks
        frames.append(request(bytes.fromhex("02ffffffffff"), duid, t, 5, 7, 8, sid))  # MAC mismatch
        frames.append(request(mac, duid, t, 5, 7, 8, sid, next_header=0))  # extension header
        frames.append(request(mac, duid, t, 5, 7, 8, sid, dst_ip=bytes.fromhex("ff0200000000000000000000000000fb")))
        frames.append(request(mac, duid, t, 5, 7, 8, sid, dst_ip=SERVER_IP))
        frames.append(request(mac, duid, t, 5, 7, 8, sid, sport=40000))
        frames.append(request(mac, S.dhcpv6_duid(5, 32), t, 5, 7, 8, sid))  # 32-byte DUID
        for tags in (((0x8100, 5),), ((0x88A8, 5), (0x8100, 6)), ((0x8100, 5), (0x8100, 6)), ((0x88A8, 5), (0x88A8, 6))):
            frames.append(request(mac, duid, t, 5, 7, 8, sid, tags=tags))
        frames.append(dhcpv4_discover(mac))
        frames.append(S.dhcpv6_frame(mac, t, 5, opt(1, duid) + S.dhcpv6_ia(3, 7), dport=53))  # ordinary UDP
    # the options truncated at every byte: the UDP length cut short
    f = bytearray(request(mac, duid, 3, 5, 7, 8, SERVER_DUID))
    for ul in range(8, len(f) - 62 + 8 + 1):
        g = bytearray(f)
        g[58:60] = ul.to_bytes(2, "big")
        frames.append(bytes(g))
    g = bytearray(f)
    g[58:60] = (len(f) - 54 + 1).to_bytes(2, "big")  # past the frame
    frames.append(bytes(g))
    many = opt(1, duid) + S.dhcpv6_ia(3, 7) + opt(8, b"\0\0") * 31  # 33 options
    frames.append(S.dhcpv6_frame(mac, 1, 5, many))
    frames.append(S.dhcpv6_frame(mac, 1, 5, many[:-6]))  # 32
    return frames, binds, cfg


def arena_of(frames, lens, stride):
    n = len(frames)
    a = np.zeros(n * stride, np.uint8)
    for i, f in enumerate(frames):
        k = min(len(f), stride)
        a[i * stride:i * stride + k] = np.frombuffer(f[:k], np.uint8)
    return a


def offset_arena(frames, lens):
    hdr = np.zeros((len(frames), 512), np.uint8)
    for i, f in enumerate(frames):
        hdr[i, :min(len(f), 512)] = np.frombuffer(f[:512], np.uint8)
    return S.pack_arena(hdr, lens)


def clocks(n, per_frame):
    if not per_frame:
        return None
    return (T0 + np.arange(n, dtype=np.uint64) * np.uint64(1_000_000_000 // 4)).astype(np.uint64)


# ---------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("per_frame", [False, True], ids=["batch_clock", "frame_clock"])
@pytest.mark.parametrize("feed", FEEDS, ids=FEED_IDS)
@pytest.mark.parametrize("stride", [128, 256, 384, 512, 2048, 0])
def test_cases(feed, per_frame, stride):
    frames, binds, cfg = case_corpus()
    lens = np.array([len(f) for f in frames], np.uint32)
    now_v = clocks(len(frames), per_frame)
    if stride:
        arena, off16 = arena_of(frames, lens, stride), None
    else:
        arena, off16 = offset_arena(frames, lens)
    want = expected(arena, lens, off16, stride, T0, now_v, cfg, binds)
    answered = want[4][ST["advertise"]] + want[4][ST["reply"]]
    if stride == 128:  # no reply fits a 128-byte slot
        assert want[4][ST["no_room"]] > 30 and answered == 0
    elif stride == 0:  # len rounded up to 16: most replies are longer than their request
        assert want[4][ST["no_room"]] > 30
    else:
        assert answered > 30
    got = run_gpu(feed, arena, lens, off16, stride, T0, now_v, cfg, binds)
    check(got, want, f"feed {feed} stride {stride}")


@pytest.mark.gpu
@pytest.mark.parametrize("feed", FEEDS, ids=FEED_IDS)
@pytest.mark.parametrize("dns", [0, 1, 2])
def test_every_length(feed, dns):
    """Every length from 14 to 460 of a Solicit and a Request, in a 512-byte stride, with 0-2 DNS servers."""
    cfg = config(dns)
    mac, duid = client(1, 14)
    binds = {duid: Binding(mac, iaid_na=7, iaid_pd=8, i=1)}
    base = [request(mac, duid, 1, 5, 7, 8, None), request(mac, duid, 3, 5, 7, 8, SERVER_DUID, rapid=True)]
    frames = [f + bytes(512 - len(f)) for f in base for _ in range(14, 461)]
    lens = np.array([ln for _ in base for ln in range(14, 461)], np.uint32)
    arena = arena_of(frames, lens, 512)
    want = expected(arena, lens, None, 512, T0, None, cfg, binds)
    got = run_gpu(feed, arena, lens, None, 512, T0, None, cfg, binds)
    check(got, want, f"lengths, feed {feed}")


@pytest.mark.gpu
def test_zero_copy_chunk_edges():
    """2^18 + 3 frames on the pinned feed (a chunk edge inside the batch) equal the device and pageable feeds."""
    frames, binds, cfg = case_corpus()
    n = (1 << 18) + 3
    idx = np.random.default_rng(5).integers(len(frames), size=n)
    lens = np.array([len(frames[k]) for k in idx], np.uint32)
    stride = 512
    arena = np.zeros((len(frames), stride), np.uint8)
    for k, f in enumerate(frames):
        arena[k, :min(len(f), stride)] = np.frombuffer(f[:stride], np.uint8)
    arena = arena[idx].reshape(-1)
    now_v = clocks(n, True)
    res = [run_gpu(feed, arena, lens, None, stride, T0, now_v, cfg, binds) for feed in FEEDS]
    for r in res[1:]:
        check(r, res[0], "pinned / device vs pageable")
    _, off16 = S.pack_arena(arena.reshape(n, stride), lens)
    oa, _ = S.pack_arena(arena.reshape(n, stride), lens)
    res = [run_gpu(feed, oa, lens, off16, 0, T0, now_v, cfg, binds) for feed in FEEDS]
    for r in res[1:]:
        check(r, res[0], "offset table: pinned / device vs pageable")


@pytest.mark.gpu
def test_randomized_differential_2_20():
    """2^20 frames drawn from the corpus, byte-mutated at random in the message, against the expected results."""
    frames, binds, cfg = case_corpus(7)
    rng = np.random.default_rng(11)
    n, stride = 1 << 20, 384
    idx = rng.integers(len(frames), size=n)
    table = np.zeros((len(frames), stride), np.uint8)
    for k, f in enumerate(frames):
        table[k, :min(len(f), stride)] = np.frombuffer(f[:stride], np.uint8)
    arena = table[idx]
    lens = np.array([len(f) for f in frames], np.uint32)[idx]
    mut = rng.random(n) < 0.3
    pos = rng.integers(62, 200, size=n)
    arena[np.nonzero(mut)[0], pos[mut]] = rng.integers(256, size=int(mut.sum()), dtype=np.uint8)
    arena = arena.reshape(-1)
    # the expected results only for the distinct frames: equal frames get equal outcomes (no order dependence)
    uniq, inv = np.unique(np.concatenate([arena.reshape(n, stride), lens.view(np.uint8).reshape(n, 4)], 1), axis=0,
                          return_inverse=True)
    ua = np.ascontiguousarray(uniq[:, :stride]).reshape(-1)
    ul = np.ascontiguousarray(uniq[:, stride:]).view(np.uint32).reshape(-1)
    wa, wl, wv, _, _ = expected(ua, ul, None, stride, T0, None, cfg, binds)
    got = run_gpu(True, arena, lens, None, stride, T0, None, cfg, binds)
    inv = inv.reshape(-1)
    assert np.array_equal(got[2], wv[inv]) and np.array_equal(got[1], wl[inv])
    assert np.array_equal(got[0].reshape(n, stride), wa.reshape(-1, stride)[inv])
    assert got[4][ST["reply"]] + got[4][ST["advertise"]] > 1000


@pytest.mark.gpu
def test_slow_path_lifecycle():
    """Solicits of unbound clients pass; the restated Go server answers them and binds; the next batch's Renews come
    back from the GPU identical to what that server sends."""
    cfg = config(1)
    clients = [client(i, 14) for i in range(200)]
    frames = [request(m, d, 1, i, i + 1, i + 2, None) for i, (m, d) in enumerate(clients)]
    lens = np.array([len(f) for f in frames], np.uint32)
    with Dataplane(max_subscribers=1 << 12, max_batch=1 << 12) as dp:
        gpu_setup(dp, cfg, {})
        binds = {}
        arena = arena_of(frames, lens, 512)
        got = run_gpu(False, arena, lens, None, 512, T0, None, cfg, binds, dp=dp)
        assert (got[2] == 2).all() and got[4].sum() == 0  # no binding yet: "on" launches what "off" does
        for i, (m, d) in enumerate(clients):  # the slow path binds
            binds[d] = Binding(m, iaid_na=i + 1, iaid_pd=i + 2, i=i)
            assert dp.update_staged("dhcpv6_bindings", S.dhcpv6_client_key(d), binds[d].value()) == 0
        renews = [request(m, d, 5, 0x100 + i, i + 1, i + 2, SERVER_DUID) for i, (m, d) in enumerate(clients)]
        rl = np.array([len(f) for f in renews], np.uint32)
        ra = arena_of(renews, rl, 512)
        got = run_gpu(False, ra, rl, None, 512, T0, None, cfg, binds, dp=dp)
        assert (got[2] == 3).all()
        for i, (m, d) in enumerate(clients):
            f = renews[i]
            model = build_reply(5, f[63:66], d, cfg, binds[d], True, True, False)
            assert got[0][i * 512 + 62:i * 512 + 62 + len(model)].tobytes() == model


def prof_names(dp):
    return sorted(dp.prof_read())


@pytest.mark.gpu
@pytest.mark.parametrize("how", ["never", "on_off", "empty", "unconfigured"])
def test_off_is_today(how):
    frames, binds, cfg = case_corpus()
    lens = np.array([len(f) for f in frames], np.uint32)
    arena = arena_of(frames, lens, 512)
    outs = []
    for variant in ("plain", how):
        with Dataplane(max_subscribers=1 << 12, max_batch=1 << 12) as dp:
            if variant != "plain":
                if how == "on_off":
                    gpu_setup(dp, cfg, binds, on=True)
                    dp.dhcpv6_enable(False)
                elif how == "empty":
                    gpu_setup(dp, cfg, {}, on=True)
                elif how == "unconfigured":
                    gpu_setup(dp, None, binds, on=True)
                elif how == "never":
                    gpu_setup(dp, cfg, binds, on=False)
            dp.prof_enable(True)
            n0 = dp.launch_count
            res = run_gpu(False, arena, lens, None, 512, T0, None, cfg, binds, dp=dp)
            outs.append((res, dp.launch_count - n0, prof_names(dp)))
    (a, n_a, p_a), (b, n_b, p_b) = outs
    check(b, a, how)
    assert b[4].sum() == 0 and n_a == n_b and p_a == p_b


@pytest.mark.gpu
def test_map_lifecycle():
    with Dataplane(max_subscribers=64, max_batch=1 << 10) as dp:
        mac, duid = client(1, 14)
        key, val = S.dhcpv6_client_key(duid), Binding(mac, i=1).value()
        assert dp.map_info("dhcpv6_bindings")["max_entries"] == 64

        def einval(k, v):
            assert dp.update("dhcpv6_bindings", k, v) == -errno.EINVAL
            assert dp.update_staged("dhcpv6_bindings", k, v) == -errno.EINVAL
            # a batch applies none of its entries
            both_k, both_v = np.concatenate([S.dhcpv6_client_key(b"ok"), k]), np.concatenate([val, v])
            assert dp.update_batch("dhcpv6_bindings", both_k, both_v) == -errno.EINVAL
            assert dp.map_info("dhcpv6_bindings")["count"] == 0

        for dl in (0, 32):
            k = key.copy()
            k["duid_len"] = dl
            einval(k, val)
        k = key.copy()
        k["duid"][0, 20] = 1
        einval(k, val)
        for flags, pl in ((0, 56), (4, 56), (3, 0), (2, 129)):
            v = val.copy()
            v["flags"], v["pd_len"] = flags, pl
            einval(key, v)
        v = val.copy()
        v["prefix"][0, 7] = 1  # past /56
        einval(key, v)
        v = val.copy()
        v["flags"], v["pd_len"], v["prefix"][0, 15] = 1, 0, 1  # NA only: pd_len and prefix are not read
        assert dp.update("dhcpv6_bindings", key, v) == 0
        for bad in ({"duid_len": 33}, {"dns_count": 3}):
            c = cfg_value(config())
            for f, x in bad.items():
                c[f] = x
            assert dp.update("dhcpv6_server_config", np.uint32(0), c) == -errno.EINVAL
        # batch, staged, E2BIG, delete, clear
        ks = np.concatenate([S.dhcpv6_client_key(S.dhcpv6_duid(i, 14)) for i in range(64)])
        vs = np.concatenate([Binding(client(i)[0], i=i).value() for i in range(64)])
        dp.clear("dhcpv6_bindings")
        assert dp.update_batch("dhcpv6_bindings", ks[:63], vs[:63]) == 0
        assert dp.update_staged("dhcpv6_bindings", ks[63:], vs[63:]) == 0
        assert dp.map_info("dhcpv6_bindings")["count"] == 64
        assert dp.update("dhcpv6_bindings", S.dhcpv6_client_key(b"extra"), vs[:1]) == -errno.E2BIG
        assert dp.delete("dhcpv6_bindings", ks[:1]) == 0
        assert dp.lookup("dhcpv6_bindings", ks[:1]) is None
        assert dp.lookup("dhcpv6_bindings", ks[1:2]).tobytes() == vs[1:2].tobytes()
        # snapshot / restore, delta export / apply
        assert dp.update("dhcpv6_server_config", np.uint32(0), cfg_value(config())) == 0
        blob = dp.snapshot()
        dk, dv = dp.dump("dhcpv6_bindings")
        with Dataplane(max_subscribers=64, max_batch=1 << 10) as dp2:
            dp2.restore(blob)
            k2, v2 = dp2.dump("dhcpv6_bindings")
            assert sorted(map(bytes, k2)) == sorted(map(bytes, dk)) and len(v2) == 63
            assert dp2.lookup("dhcpv6_server_config", np.uint32(0)).tobytes() == cfg_value(config()).tobytes()
        dp.clear("dhcpv6_bindings")
        assert dp.map_info("dhcpv6_bindings")["count"] == 0
        with Dataplane(max_subscribers=64, max_batch=1 << 10) as dp3:
            dp.delta_enable(True)
            assert dp3.delta_apply(dp.delta_export(full=True)) == 0
            dp.update_batch("dhcpv6_bindings", ks[:10], vs[:10])
            assert dp3.delta_apply(dp.delta_export()) == 0
            assert dp3.map_info("dhcpv6_bindings")["count"] == 10
            dp.delete("dhcpv6_bindings", ks[:1])
            assert dp3.delta_apply(dp.delta_export()) == 0
            assert dp3.map_info("dhcpv6_bindings")["count"] == 9


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 8])
def test_sharded_union(world):
    """Bindings routed by their MAC's shard and frames steered by source MAC: the union equals one context."""
    frames, binds, cfg = case_corpus()
    lens = np.array([len(f) for f in frames], np.uint32)
    stride = 512
    arena = arena_of(frames, lens, stride)
    one = run_gpu(False, arena, lens, None, stride, T0, None, cfg, binds)
    macs = np.array([int.from_bytes(f[6:12], "big") for f in frames], np.uint64)
    shard = S.shard_of_mac(macs, world)
    got_a, got_l, got_v = arena.copy(), lens.copy(), np.zeros(len(frames), np.uint8)
    st6 = np.zeros(12, np.uint64)
    for s in range(world):
        mine = {d: b for d, b in binds.items() if S.shard_of_mac(np.uint64(int.from_bytes(b.mac, "big")), world) == s}
        sel = np.nonzero(shard == s)[0]
        if not len(sel):
            continue
        sub = [frames[i] for i in sel]
        with Dataplane(max_subscribers=1 << 12, max_batch=1 << 12) as dp:
            gpu_setup(dp, cfg, mine)
            r = run_gpu(False, arena_of(sub, lens[sel], stride), lens[sel].copy(), None, stride, T0, None, cfg, mine, dp=dp)
        got_a.reshape(-1, stride)[sel] = r[0].reshape(-1, stride)
        got_l[sel], got_v[sel] = r[1], r[2]
        st6 += r[4]
    assert np.array_equal(got_v, one[2]) and np.array_equal(got_l, one[1]) and np.array_equal(got_a, one[0])
    assert np.array_equal(st6, one[4])
