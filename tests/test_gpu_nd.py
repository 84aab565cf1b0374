"""Router and Neighbor Solicitations answered on the GPU (bng_nd_enable, include/bng_b200.h): dhcp_fastpath_prog answers
a subscriber's RS with a Router Advertisement of its own (the nd_config template plus its nd_bindings prefix) and an NS
for the router's link-local address with a Neighbor Advertisement.

Expected results: the oracle's own dhcp_fastpath_prog runs on the whole batch and gives every verdict, byte, length and
stats_map counter.  The rule, restated below, then overrides verdict, bytes and length of the frames it answers and
gives nd_stats (and, with bng_dhcpv6_enable on too, the DHCPv6 rule of test_gpu_dhcpv6 gives dhcpv6_stats).  The
program writes no table and no frame's outcome depends on another, so that combination is the specification.  The
restatement is checked on the CPU by a separate RFC 4861 decoder, a second checksum implementation and literal byte
vectors."""
import errno

import numpy as np
import pytest

import harness
import test_gpu_dhcpv6 as D6
from bng_b200 import Dataplane
from bng_b200 import layouts as L
from bng_b200 import synth as S

FEEDS = [False, True, "device"]
FEED_IDS = ["pageable", "pinned", "device"]
T0 = 1_000_000 * 1_000_000_000  # 1e6 s
ST = {n: i for i, n in enumerate(L.ND_STATS)}
ROUTER_MAC = bytes.fromhex("02aabbccdd01")
ROUTER_LL = bytes.fromhex("fe800000000000000000000000000001")
SHARED = (bytes.fromhex("20010db8ff0000000000000000000000"), bytes.fromhex("20010db8fe0000000000000000000000"))
DNS = (bytes.fromhex("20010db8000000000000000000000053"), bytes.fromhex("20010db8000000000000000000000054"))


# ---------------------------------------------------------------------------
# the configuration: buildRA's bytes, split where the subscriber's prefix goes
# ---------------------------------------------------------------------------
def ra_template(n_shared=2, dns=2, domains=("isp.example", "example.net"), mtu=1500, managed=False, other=False,
                lifetime=1800):
    """(head, tail) as pkg/slaac's buildRA orders its options (the C++ slaac::BuildRA is checked against literal
    vectors in tests/host/test_nd_host.cpp)."""
    head = bytes([134, 0, 0, 0, 64, (0x80 if managed else 0) | (0x40 if other else 0)]) + lifetime.to_bytes(2, "big")
    head += bytes(8) + bytes([1, 1]) + ROUTER_MAC
    if mtu:
        head += bytes([5, 1, 0, 0]) + mtu.to_bytes(4, "big")
    for p in SHARED[:n_shared]:
        head += bytes([3, 4, 64, 0x80 | (0 if managed else 0x40)]) + (2592000).to_bytes(4, "big")
        head += (604800).to_bytes(4, "big") + bytes(4) + p
    tail = b""
    if dns:
        tail += bytes([25, 1 + 2 * dns, 0, 0]) + (3 * lifetime).to_bytes(4, "big") + b"".join(DNS[:dns])
    if domains:
        names = b"".join(b"".join(bytes([len(x)]) + x.encode() for x in d.split(".") if x) + b"\0" for d in domains)
        names += bytes((8 - (8 + len(names)) % 8) % 8)
        tail += bytes([31, (8 + len(names)) // 8, 0, 0]) + (3 * lifetime).to_bytes(4, "big") + names
    return head, tail


def config(n_shared=2, dns=2, domains=("isp.example", "example.net"), **kw):
    head, tail = ra_template(n_shared, dns, domains, **kw)
    return {"mac": ROUTER_MAC, "ll": ROUTER_LL, "head": head, "tail": tail}


def cfg_value(cfg):
    v = np.zeros(1, L.bng_nd_config)
    if cfg is None:
        return v
    v["router_mac"][0] = np.frombuffer(cfg["mac"], np.uint8)
    v["ra_head_len"], v["ra_tail_len"] = len(cfg["head"]), len(cfg["tail"])
    v["router_ll"][0] = np.frombuffer(cfg["ll"], np.uint8)
    ra = cfg["head"] + cfg["tail"]
    v["ra"][0, :len(ra)] = np.frombuffer(ra, np.uint8)
    return v


class Binding:
    def __init__(self, prefix_len=64, pio_flags=0xC0, valid=7200, preferred=3600, expires_s=2_000_000, i=0, prefix=None):
        self.prefix_len, self.valid, self.preferred, self.expires_s = prefix_len, valid, preferred, expires_s
        self.pio_flags = pio_flags if prefix_len else 0
        full = prefix or bytes.fromhex("20010db8") + (i & 0xFFFF).to_bytes(2, "big") + bytes.fromhex("00ab") + bytes(7) + bytes([i & 0xFF])
        bits = int.from_bytes(full, "big") & (((1 << prefix_len) - 1) << (128 - prefix_len)) if prefix_len else 0
        self.prefix = bits.to_bytes(16, "big")

    def value(self):
        v = np.zeros(1, L.bng_nd_binding)
        v["prefix"][0] = np.frombuffer(self.prefix, np.uint8)
        v["prefix_len"], v["pio_flags"] = self.prefix_len, self.pio_flags
        v["valid_lft"], v["preferred_lft"], v["expires_s"] = self.valid, self.preferred, self.expires_s
        return v

    def pio(self):
        return (bytes([3, 4, self.prefix_len, self.pio_flags]) + self.valid.to_bytes(4, "big") +
                self.preferred.to_bytes(4, "big") + bytes(4) + self.prefix)


def mac_key(mac):
    return np.array([int.from_bytes(mac, "big")], np.uint64)


# ---------------------------------------------------------------------------
# the rule, restated
# ---------------------------------------------------------------------------
def ones_sum(data):
    """The 16-bit one's-complement sum of data (zero-padded to even length), end-around carries folded."""
    if len(data) & 1:
        data += b"\0"
    s = sum(int.from_bytes(data[k:k + 2], "big") for k in range(0, len(data), 2))
    while s >> 16:
        s = (s & 0xFFFF) + (s >> 16)
    return s


def pseudo(src, dst, n):
    return src + dst + n.to_bytes(4, "big") + b"\0\0\0\x3a"


def rule(f, ln, dlen, room, now_ns, cfg, binds):
    """(counters, reply frame or None) for one frame that dhcp_one (and the DHCPv6 rule) passed; ([], None): not a
    candidate.  f: the frame's bytes (at least dlen of them); binds: MAC bytes -> Binding."""
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
    if et != b"\x86\xdd" or l3 + 41 > dlen or f[l3] >> 4 != 6 or f[l3 + 6] != 58:
        return [], None
    ll = cfg["ll"] if cfg else bytes(16)
    t, dst, icmp = f[l3 + 40], bytes(f[l3 + 24:l3 + 40]), l3 + 40
    if not ((t == 133 and dst in (S.ALL_ROUTERS, ll)) or (t == 135 and dst in (ll, S.solicited_node(ll)))):
        return [], None
    rs, c = t == 133, ["total"]
    if cfg is None or ln > 448:
        return c + ["unsupported"], None
    plen = int.from_bytes(f[l3 + 4:l3 + 6], "big")
    if plen < (8 if rs else 24) or icmp + plen > dlen:
        return c + ["malformed"], None
    c.append("rs" if rs else "ns")
    src = bytes(f[l3 + 8:l3 + 24])
    unspec = src == bytes(16)
    bad = f[l3 + 7] != 255 or f[icmp + 1] != 0
    bad = bad or ones_sum(pseudo(src, dst, plen) + bytes(f[icmp:icmp + plen])) != 0xFFFF
    o, end, n, slla = icmp + (8 if rs else 24), icmp + plen, 0, False
    while o < end and not bad:
        if o + 2 > end or f[o + 1] == 0 or o + 8 * f[o + 1] > end or n == 32:
            bad = True
            break
        n, slla, o = n + 1, slla or f[o] == 1, o + 8 * f[o + 1]
    bad = bad or (unspec and slla)
    if not rs:
        bad = bad or f[icmp + 8] == 0xFF or (unspec and dst == ll)
    if bad:
        return c + ["malformed"], None
    if not rs and bytes(f[icmp + 8:icmp + 24]) != ll:
        return c + ["not_target"], None
    if rs:
        b = binds.get(bytes(f[6:12]))
        if b is None:
            return c + ["miss"], None
        if now_ns // 1_000_000_000 > b.expires_s:
            return c + ["expired"], None
        body = cfg["head"] + (b.pio() if b.prefix_len else b"") + cfg["tail"]
    else:
        body = bytes([136, 0, 0, 0, 0xA0 if unspec else 0xE0, 0, 0, 0]) + ll + bytes([2, 1]) + cfg["mac"]
    if icmp + len(body) > room:
        return c + ["no_room"], None
    to = S.ALL_NODES if unspec else src
    ck = (~ones_sum(pseudo(ll, to, len(body)) + body)) & 0xFFFF
    body = body[:2] + ck.to_bytes(2, "big") + body[4:]
    ip = b"\x60\x00\x00\x00" + len(body).to_bytes(2, "big") + b"\x3a\xff" + ll + to
    return c + ["ra" if rs else "na"], bytes(f[6:12]) + cfg["mac"] + bytes(f[12:l3]) + ip + body


# ---------------------------------------------------------------------------
# an independent RFC 4861 decoder (CPU checks of the restatement)
# ---------------------------------------------------------------------------
def decode(frame):
    l3 = 14
    while frame[l3 - 2:l3] in (b"\x81\x00", b"\x88\xa8"):
        l3 += 4
    assert frame[l3 - 2:l3] == b"\x86\xdd"
    ip, msg = frame[l3:l3 + 40], frame[l3 + 40:]
    assert ip[:4] == b"\x60\x00\x00\x00" and ip[6] == 58 and ip[7] == 255
    assert int.from_bytes(ip[4:6], "big") == len(msg)
    assert S.icmp6_checksum(ip[8:24], ip[24:40], msg[:2] + b"\0\0" + msg[4:]) == int.from_bytes(msg[2:4], "big")
    out = {"dst_mac": frame[:6], "src_mac": frame[6:12], "src": ip[8:24], "dst": ip[24:40], "type": msg[0], "code": msg[1]}
    if msg[0] == 134:
        out.update(hop_limit=msg[4], flags=msg[5], lifetime=int.from_bytes(msg[6:8], "big"),
                   reachable=int.from_bytes(msg[8:12], "big"), retrans=int.from_bytes(msg[12:16], "big"))
        o = 16
    else:
        assert msg[0] == 136 and len(msg) == 32
        out.update(flags=msg[4], target=msg[8:24])
        o = 24
    opts = []
    while o < len(msg):
        n = msg[o + 1] * 8
        assert n
        opts.append((msg[o], msg[o:o + n]))
        o += n
    assert o == len(msg)
    out["opts"] = opts
    return out


def pio_decode(opt):
    return {"len": opt[2], "L": bool(opt[3] & 0x80), "A": bool(opt[3] & 0x40), "valid": int.from_bytes(opt[4:8], "big"),
            "preferred": int.from_bytes(opt[8:12], "big"), "prefix": opt[16:32]}


def host_mac(i):
    return bytes.fromhex("0200000a") + int(i).to_bytes(2, "big")


def test_restatement_against_decoder():
    for n_shared in (0, 1, 2):
        for dns in (0, 2):
            cfg = config(n_shared, dns, ("isp.example",) if dns else ())
            for pl, flags in ((0, 0), (48, 0x80), (64, 0xC0), (128, 0x40)):
                for tags in ((), ((0x8100, 7),), ((0x88A8, 7), (0x8100, 9))):
                    for src in (None, bytes(16), bytes.fromhex("20010db8000100000000000000000005")):
                        mac = host_mac(3)
                        b = Binding(pl, flags, i=3)
                        f = S.rs_frame(mac, src_ip=src, slla=src != bytes(16), tags=tags)
                        c, out = rule(f, len(f), len(f), 2048, T0, cfg, {mac: b})
                        assert c == ["total", "rs", "ra"], c
                        d = decode(out)
                        assert d["type"] == 134 and d["code"] == 0 and d["hop_limit"] == 64 and d["lifetime"] == 1800
                        assert d["dst_mac"] == mac and d["src_mac"] == ROUTER_MAC and d["src"] == ROUTER_LL
                        assert d["dst"] == (S.ALL_NODES if src == bytes(16) else (src or S.link_local(mac)))
                        kinds = [k for k, _ in d["opts"]]
                        assert kinds == [1, 5] + [3] * (n_shared + (pl > 0)) + ([25, 31] if dns else [])
                        assert d["opts"][0][1][2:] == ROUTER_MAC
                        pios = [pio_decode(o) for k, o in d["opts"] if k == 3]
                        assert [p["prefix"] for p in pios[:n_shared]] == list(SHARED[:n_shared])
                        assert all(p["L"] and p["A"] and p["valid"] == 2592000 for p in pios[:n_shared])
                        if pl:
                            p = pios[-1]
                            assert (p["len"], p["L"], p["A"]) == (pl, bool(flags & 0x80), bool(flags & 0x40))
                            assert (p["valid"], p["preferred"], p["prefix"]) == (7200, 3600, b.prefix)
                        # and the NS for router_ll
                        f = S.ns_frame(mac, ROUTER_LL, src_ip=src, slla=src != bytes(16), tags=tags)
                        c, out = rule(f, len(f), len(f), 2048, T0, cfg, {})
                        assert c == ["total", "ns", "na"], c
                        d = decode(out)
                        assert d["type"] == 136 and d["target"] == ROUTER_LL
                        assert d["flags"] == (0xA0 if src == bytes(16) else 0xE0)
                        assert d["opts"] == [(2, b"\x02\x01" + ROUTER_MAC)]


def test_literal_vectors():
    """An RS from fe80::a:0:5 (MAC 02:00:00:0a:00:05, no options) and an NS for fe80::1 from the same host, answered with
    a template of one MTU option and no shared prefix; binding 2001:db8:5::/64, L|A, valid 7200, preferred 3600.
    ICMPv6 bodies worked out by hand from RFC 4861 §4.2 / §4.4; the checksums agree with both implementations."""
    cfg = config(0, 0, ())
    mac = bytes.fromhex("02000000000a")
    src = bytes.fromhex("fe80000000000000000000fffe00000a")
    b = Binding(64, 0xC0, prefix=bytes.fromhex("20010db8000500000000000000000000"))
    f = S.rs_frame(mac, src_ip=src, slla=False)
    _, out = rule(f, len(f), len(f), 2048, T0, cfg, {mac: b})
    ra = out[54:]
    assert out[:14].hex() == "02000000000a" + "02aabbccdd01" + "86dd"
    assert out[14:54].hex() == "60000000" "0040" "3aff" + ROUTER_LL.hex() + src.hex()
    assert ra[:2].hex() + ra[4:].hex() == ("8600" + "40000708" "00000000" "00000000" + "010102aabbccdd01" +
                                           "05010000000005dc" + "030440c0" "00001c20" "00000e10" "00000000" +
                                           "20010db8000500000000000000000000")
    assert int.from_bytes(ra[2:4], "big") == S.icmp6_checksum(ROUTER_LL, src, ra[:2] + b"\0\0" + ra[4:])
    f = S.ns_frame(mac, ROUTER_LL, src_ip=src, dst_ip=S.solicited_node(ROUTER_LL))
    _, out = rule(f, len(f), len(f), 2048, T0, cfg, {})
    na = out[54:]
    assert na[:2].hex() + na[4:].hex() == "8800" + "e0000000" + ROUTER_LL.hex() + "020102aabbccdd01"
    assert int.from_bytes(na[2:4], "big") == S.icmp6_checksum(ROUTER_LL, src, na[:2] + b"\0\0" + na[4:])
    assert ones_sum(pseudo(ROUTER_LL, src, 32) + na) == 0xFFFF


def test_synth_checksums():
    """The frame builders' checksums pass the rule's own sum (two implementations of RFC 4443 §2.3)."""
    for src in (None, bytes(16)):
        for f in (S.rs_frame(host_mac(1), src_ip=src, slla=src is None),
                  S.ns_frame(host_mac(1), ROUTER_LL, src_ip=src, slla=src is None)):
            m = f[54:]
            assert ones_sum(pseudo(f[22:38], f[38:54], len(m)) + m) == 0xFFFF


# ---------------------------------------------------------------------------
# expected results and the run
# ---------------------------------------------------------------------------
def oracle_kind():
    from oracle import pyoracle
    return "reference" if pyoracle.available("reference") else "port"


def expected(arena, lens, off16, stride, now, now_v, nd, d6=None):
    """The oracle's dhcp_fastpath_prog on the whole batch, then the DHCPv6 rule (d6 = (cfg, binds) when it runs) and
    the ND rule (nd = (cfg, binds) when it runs) on the frames it passes."""
    ob = harness.OracleBackend(oracle_kind())
    try:
        a, l = arena.copy(), lens.copy()
        v = ob.run("dhcp_fastpath_prog", a, l, now, off16, stride, None, now_v=now_v).copy()
        st = ob.stats("stats_map")
    finally:
        ob.close()
    cnt, cnt6 = np.zeros(len(L.ND_STATS), np.uint64), np.zeros(len(L.DHCPV6_STATS), np.uint64)
    for i in range(len(lens)):
        if v[i] != 2:
            continue
        off = int(off16[i]) * 16 if off16 is not None else i * stride
        ln = int(lens[i])
        dlen = ln if off16 is not None else min(ln, stride)
        room = stride if off16 is None else (ln + 15) & ~15
        fb = arena[off:off + dlen].tobytes()
        t = int(now_v[i]) if now_v is not None else now
        c, out = ([], None)
        if d6 is not None:
            c, out = D6.rule(fb, ln, dlen, room, t, d6[0], d6[1])
            for k in c:
                cnt6[D6.ST[k]] += 1
        if not c and nd is not None:
            c, out = rule(fb, ln, dlen, room, t, nd[0], nd[1])
            for k in c:
                cnt[ST[k]] += 1
        if out is not None:
            v[i] = 3
            l[i] = len(out)
            a[off:off + len(out)] = np.frombuffer(out, np.uint8)
            a[off + len(out):off + ((len(out) + 15) & ~15)] = 0
    return a, l, v, st, cnt, cnt6


def gpu_setup(dp, cfg, binds, on=True):
    if cfg is not None:
        assert dp.update("nd_config", np.uint32(0), cfg_value(cfg)) == 0
    if binds:
        ks = np.concatenate([mac_key(m) for m in binds])
        vs = np.concatenate([b.value() for b in binds.values()])
        assert dp.update_batch("nd_bindings", ks, vs) == 0
    dp.nd_enable(on)


def run_gpu(feed, arena, lens, off16, stride, now, now_v, cfg, binds, dp=None, d6=None, nd_on=True, **opts):
    be = harness.GpuBackend(dp=dp, pinned=feed, **opts)
    if dp is None:
        gpu_setup(be.dp, cfg, binds, nd_on)
        if d6 is not None:
            D6.gpu_setup(be.dp, d6[0], d6[1])
    a, l = arena.copy(), lens.copy()
    v = be.run("dhcp_fastpath_prog", a, l, now, off16, stride, None, now_v=now_v)
    res = a, l, v, be.stats("stats_map"), be.stats("nd_stats"), be.stats("dhcpv6_stats")
    if dp is None:
        be.close()
    return res


def check(got, want, what=""):
    ga, gl, gv, gs, gn, g6 = got
    wa, wl, wv, ws, wn, w6 = want
    bad = np.nonzero((gv != wv) | (gl != wl))[0]
    assert not len(bad), f"{what}: frames {bad[:10]} verdict {gv[bad[:10]]} vs {wv[bad[:10]]} len {gl[bad[:10]]} vs {wl[bad[:10]]}"
    assert np.array_equal(gs, ws), f"{what}: stats_map {gs} vs {ws}"
    assert np.array_equal(gn, wn), f"{what}: nd_stats {dict(zip(L.ND_STATS, gn))} vs {dict(zip(L.ND_STATS, wn))}"
    assert np.array_equal(g6, w6), f"{what}: dhcpv6_stats {g6} vs {w6}"
    diff = np.nonzero(ga != wa)[0]
    assert not len(diff), f"{what}: arena bytes differ at {diff[:10]}"


def with_len(f, plen):
    """f with its IPv6 payload length set to plen (the bytes stay)."""
    g = bytearray(f)
    g[18:20] = plen.to_bytes(2, "big")
    return bytes(g)


def flip(f, pos):
    g = bytearray(f)
    g[pos] ^= 0x5A
    return bytes(g)


def case_corpus(seed=1, cfg=None):
    """(frames, binds, cfg) covering the rule's branches."""
    rng = np.random.default_rng(seed)
    cfg = cfg or config(2)
    binds, frames = {}, []
    glob = bytes.fromhex("20010db8000100000000000000000005")
    k = 0
    for pl in (0, 48, 64, 128):
        for flags in ((0,) if pl == 0 else (0, 0x80, 0x40, 0xC0)):
            mac = host_mac(100 + k)
            binds[mac] = Binding(pl, flags, i=100 + k, valid=int(rng.integers(1 << 32)), preferred=int(rng.integers(1 << 32)))
            for src in (None, bytes(16), glob):
                frames.append(S.rs_frame(mac, src_ip=src, slla=src != bytes(16)))
            frames.append(S.rs_frame(mac, dst_ip=ROUTER_LL))
            k += 1
    mac = host_mac(1)
    binds[mac] = Binding(64, 0xC0, i=1)
    emac = host_mac(2)
    binds[emac] = Binding(64, 0xC0, i=2, expires_s=T0 // 10**9 + 50)
    umac = host_mac(3)  # unbound
    dad_cpe = bytes.fromhex("20010db8000100000000000000") + ROUTER_LL[13:]  # its solicited-node group is router_ll's
    for m in (mac, umac):
        for src in (None, bytes(16), glob):
            sl = src != bytes(16)
            base_rs = S.rs_frame(m, src_ip=src, slla=sl)
            base_ns = S.ns_frame(m, ROUTER_LL, src_ip=src, slla=sl)
            frames += [base_rs, base_ns, S.ns_frame(m, ROUTER_LL, src_ip=src, dst_ip=ROUTER_LL, slla=sl)]
            for hl in (254, 255, 64):
                frames += [S.rs_frame(m, src_ip=src, slla=sl, hop_limit=hl), S.ns_frame(m, ROUTER_LL, src_ip=src, slla=sl, hop_limit=hl)]
            frames += [S.rs_frame(m, src_ip=src, slla=sl, code=1), S.ns_frame(m, ROUTER_LL, src_ip=src, slla=sl, code=3)]
            for pos in (56, 57):  # each checksum byte flipped
                frames += [flip(base_rs, pos), flip(base_ns, pos)]
            for tags in (((0x8100, 5),), ((0x88A8, 5), (0x8100, 6)), ((0x8100, 5), (0x8100, 6)), ((0x88A8, 5), (0x88A8, 6))):
                frames += [S.rs_frame(m, src_ip=src, slla=sl, tags=tags), S.ns_frame(m, ROUTER_LL, src_ip=src, slla=sl, tags=tags)]
            frames += [S.rs_frame(m, src_ip=src, slla=sl, next_header=0), S.ns_frame(m, ROUTER_LL, src_ip=src, slla=sl, next_header=0)]
        frames.append(S.rs_frame(m, src_ip=bytes(16), slla=True))  # SLLA with ::
        frames.append(S.ns_frame(m, ROUTER_LL, src_ip=bytes(16), slla=True))
        frames.append(S.ns_frame(m, ROUTER_LL, src_ip=bytes(16), dst_ip=ROUTER_LL, slla=False))  # DAD sent to the address
        frames.append(S.ns_frame(m, ROUTER_LL, src_ip=bytes(16), slla=False))  # DAD for router_ll: answered to ff02::1
        frames.append(S.ns_frame(m, dad_cpe, src_ip=bytes(16), slla=False))  # a CPE's own DAD: not_target
        frames.append(S.ns_frame(m, glob, src_ip=bytes(16), slla=False))  # another group: not a candidate
        frames.append(S.ns_frame(m, bytes.fromhex("ff020000000000000000000000000001"), dst_ip=ROUTER_LL))  # multicast target
        frames.append(S.ns_frame(m, glob, dst_ip=ROUTER_LL))  # a foreign target
        frames.append(S.rs_frame(m, dst_ip=S.ALL_NODES))  # not to the routers
        frames.append(S.ns_frame(m, ROUTER_LL, dst_ip=S.solicited_node(glob)))
        frames.append(S.icmp6_frame(m, bytes([128, 0, 0, 0]) + bytes(4), S.link_local(m), ROUTER_LL))  # echo request
        frames.append(S.rs_frame(m, options=S.nd_option(14, bytes(6)) * 31))  # SLLA + 31: 32 options
        frames.append(S.rs_frame(m, options=S.nd_option(14, bytes(6)) * 32))  # 33
        frames.append(S.rs_frame(m, options=bytes([14, 0]) + bytes(6)))  # length 0
        frames.append(S.ns_frame(m, ROUTER_LL, options=bytes([14, 2]) + bytes(6)))  # past the end
        frames.append(S.rs_frame(m, options=bytes(16), slla=False))  # a zero option type with length 0
        frames.append(D6.dhcpv4_discover(m))
    # truncated at every byte: the payload length cut short, and one past the frame
    for f in (S.rs_frame(mac, options=S.nd_option(14, bytes(14))), S.ns_frame(mac, ROUTER_LL, options=S.nd_option(14, bytes(6)))):
        for plen in range(0, len(f) - 54 + 2):
            frames.append(with_len(f, plen))
    out = []
    for i, f in enumerate(frames):  # the expiring binding's RS spread through the batch: per-frame clocks straddle it
        out.append(f)
        if i % 8 == 0:
            out.append(S.rs_frame(emac))
    return out, binds, cfg


def arena_of(frames, lens, stride):
    return D6.arena_of(frames, lens, stride)


def offset_arena(frames, lens):
    return D6.offset_arena(frames, lens)


def clocks(n, per_frame):
    return D6.clocks(n, per_frame)


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
    want = expected(arena, lens, off16, stride, T0, now_v, (cfg, binds))
    w = want[4]
    assert w[ST["na"]] > 10 and w[ST["malformed"]] > 50 and w[ST["not_target"]] > 1 and w[ST["miss"]] > 10
    if stride in (128, 256, 0):  # an RA with two shared prefixes, RDNSS and DNSSL is 262 bytes with its headers
        assert w[ST["no_room"]] > 10
    if stride == 128:
        assert w[ST["ra"]] == 0
    if stride >= 384:
        assert w[ST["ra"]] > 30
    if per_frame:
        assert w[ST["expired"]] > 10
    got = run_gpu(feed, arena, lens, off16, stride, T0, now_v, cfg, binds)
    check(got, want, f"feed {feed} stride {stride}")


@pytest.mark.gpu
@pytest.mark.parametrize("feed", FEEDS, ids=FEED_IDS)
@pytest.mark.parametrize("n_shared", [0, 1, 2])
def test_every_length(feed, n_shared):
    """Every length from 14 to 460 of a short and a 446-byte RS and NS, in a 512-byte stride, against 0-2 shared
    prefixes: cut short (malformed), whole, followed by padding, past the 400-byte staging slot, past 448 (unsupported)."""
    cfg = config(n_shared)
    mac = host_mac(1)
    binds = {mac: Binding(64, 0xC0, i=1)}
    base = [S.rs_frame(mac), S.rs_frame(mac, options=S.nd_option(14, bytes(14)) * 23 + S.nd_option(14, bytes(6))),
            S.ns_frame(mac, ROUTER_LL), S.ns_frame(mac, ROUTER_LL, options=S.nd_option(14, bytes(14)) * 22 + S.nd_option(14, bytes(6)))]
    assert len(base[1]) == len(base[3]) == 446
    frames = [f + bytes(512 - len(f)) for f in base for _ in range(14, 461)]
    lens = np.array([ln for _ in base for ln in range(14, 461)], np.uint32)
    arena = arena_of(frames, lens, 512)
    want = expected(arena, lens, None, 512, T0, None, (cfg, binds))
    assert want[4][ST["ra"]] > 100 and want[4][ST["na"]] > 100
    got = run_gpu(feed, arena, lens, None, 512, T0, None, cfg, binds)
    check(got, want, f"lengths, feed {feed}")


@pytest.mark.gpu
@pytest.mark.parametrize("v6_on", [False, True], ids=["v6_off", "v6_on"])
@pytest.mark.parametrize("nd_on", [False, True], ids=["nd_off", "nd_on"])
@pytest.mark.parametrize("feed", FEEDS, ids=FEED_IDS)
def test_with_dhcpv4_and_dhcpv6(feed, nd_on, v6_on):
    """ND frames interleaved with DHCPv4 and DHCPv6 ones, with every combination of the two switches."""
    frames, binds, cfg = case_corpus(3)
    f6, b6, c6 = D6.case_corpus(3)
    mix = [x for pair in zip(frames, f6) for x in pair] + frames[len(f6):] + f6[len(frames):]
    lens = np.array([len(f) for f in mix], np.uint32)
    now_v = clocks(len(mix), True)
    arena = arena_of(mix, lens, 512)
    want = expected(arena, lens, None, 512, T0, now_v, (cfg, binds) if nd_on else None, (c6, b6) if v6_on else None)
    be = harness.GpuBackend(pinned=feed)
    gpu_setup(be.dp, cfg, binds, nd_on)
    D6.gpu_setup(be.dp, c6, b6, v6_on)
    a, l = arena.copy(), lens.copy()
    v = be.run("dhcp_fastpath_prog", a, l, T0, None, 512, None, now_v=now_v)
    got = a, l, v, be.stats("stats_map"), be.stats("nd_stats"), be.stats("dhcpv6_stats")
    be.close()
    check(got, want, f"nd {nd_on} v6 {v6_on}")


@pytest.mark.gpu
def test_zero_copy_chunk_edges():
    """2^18 + 3 frames on the pinned feed (a chunk edge inside the batch) equal the device and pageable feeds, and
    the expected results."""
    frames, binds, cfg = case_corpus()
    n = (1 << 18) + 3
    idx = np.random.default_rng(5).integers(len(frames), size=n)
    lens = np.array([len(frames[k]) for k in idx], np.uint32)
    stride = 512
    table = np.zeros((len(frames), stride), np.uint8)
    for k, f in enumerate(frames):
        table[k, :min(len(f), stride)] = np.frombuffer(f[:stride], np.uint8)
    arena = table[idx].reshape(-1)
    res = [run_gpu(feed, arena, lens, None, stride, T0, None, cfg, binds) for feed in FEEDS]
    for r in res[1:]:
        check(r, res[0], "pinned / device vs pageable")
    wa, wl, wv, _, _, _ = expected(table.reshape(-1), np.array([len(f) for f in frames], np.uint32), None, stride, T0,
                                   None, (cfg, binds))
    assert np.array_equal(res[0][2], wv[idx]) and np.array_equal(res[0][1], wl[idx])
    assert np.array_equal(res[0][0].reshape(n, stride), wa.reshape(-1, stride)[idx])
    oa, off16 = S.pack_arena(arena.reshape(n, stride), lens)
    res = [run_gpu(feed, oa, lens, off16, 0, T0, None, cfg, binds) for feed in FEEDS]
    for r in res[1:]:
        check(r, res[0], "offset table: pinned / device vs pageable")


@pytest.mark.gpu
def test_randomized_differential_2_20():
    """2^20 frames drawn from the corpus, byte-mutated at random in the IPv6 header and the message, against the
    expected results."""
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
    pos = rng.integers(14, 120, size=n)
    arena[np.nonzero(mut)[0], pos[mut]] = rng.integers(256, size=int(mut.sum()), dtype=np.uint8)
    arena = arena.reshape(-1)
    # the expected results only for the distinct frames: equal frames get equal outcomes (no order dependence)
    uniq, inv = np.unique(np.concatenate([arena.reshape(n, stride), lens.view(np.uint8).reshape(n, 4)], 1), axis=0,
                          return_inverse=True)
    ua = np.ascontiguousarray(uniq[:, :stride]).reshape(-1)
    ul = np.ascontiguousarray(uniq[:, stride:]).view(np.uint32).reshape(-1)
    wa, wl, wv, _, _, _ = expected(ua, ul, None, stride, T0, None, (cfg, binds))
    got = run_gpu(True, arena, lens, None, stride, T0, None, cfg, binds)
    inv = inv.reshape(-1)
    assert np.array_equal(got[2], wv[inv]) and np.array_equal(got[1], wl[inv])
    assert np.array_equal(got[0].reshape(n, stride), wa.reshape(-1, stride)[inv])
    assert got[4][ST["ra"]] > 10000 and got[4][ST["na"]] > 10000


@pytest.mark.gpu
def test_slow_path_lifecycle():
    """RS of unbound subscribers pass (miss); once bound they are answered with their own prefix; at the expiry second
    they still are, a second later they pass (expired); unbound again, they miss."""
    cfg = config(1)
    macs = [host_mac(i) for i in range(200)]
    rs = [S.rs_frame(m) for m in macs]
    lens = np.array([len(f) for f in rs], np.uint32)
    arena = arena_of(rs, lens, 512)
    with Dataplane(max_subscribers=1 << 12, max_batch=1 << 12) as dp:
        gpu_setup(dp, cfg, {})
        got = run_gpu(False, arena, lens, None, 512, T0, None, cfg, {}, dp=dp)
        assert (got[2] == 2).all() and got[4][ST["miss"]] == 200
        exp_s = T0 // 10**9 + 10
        binds = {m: Binding(64, 0xC0, i=i, expires_s=exp_s) for i, m in enumerate(macs)}
        for m, b in binds.items():  # the slow path binds (staged: visible from the next batch)
            assert dp.update_staged("nd_bindings", mac_key(m), b.value()) == 0
        for now, answered in ((T0, True), (exp_s * 10**9 + 999_999_999, True), ((exp_s + 1) * 10**9, False)):
            got = run_gpu(False, arena, lens, None, 512, now, None, cfg, binds, dp=dp)
            want = expected(arena, lens, None, 512, now, None, (cfg, binds))
            assert (got[2] == (3 if answered else 2)).all()
            assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
            if answered:
                for i, m in enumerate(macs):
                    opts = decode(got[0][i * 512:i * 512 + got[1][i]].tobytes())["opts"]
                    assert [o for k, o in opts if k == 3][-1] == binds[m].pio()
        for m in macs:
            assert dp.delete("nd_bindings", mac_key(m)) == 0
        n0 = dp.stats("nd_stats")[ST["miss"]]
        got = run_gpu(False, arena, lens, None, 512, T0, None, cfg, {}, dp=dp)
        assert (got[2] == 2).all() and got[4][ST["miss"]] - n0 == 200


def prof_names(dp):
    return sorted(dp.prof_read())


@pytest.mark.gpu
@pytest.mark.parametrize("how", ["never", "on_off", "unconfigured", "bindings_only"])
def test_off_is_today(how):
    frames, binds, cfg = case_corpus()
    lens = np.array([len(f) for f in frames], np.uint32)
    arena = arena_of(frames, lens, 512)
    outs = []
    for variant in ("plain", how):
        with Dataplane(max_subscribers=1 << 12, max_batch=1 << 12) as dp:
            if variant != "plain":
                if how == "never":
                    gpu_setup(dp, cfg, binds, on=False)
                elif how == "on_off":
                    gpu_setup(dp, cfg, binds, on=True)
                    dp.nd_enable(False)
                elif how == "unconfigured":
                    gpu_setup(dp, None, {}, on=True)
                elif how == "bindings_only":
                    gpu_setup(dp, None, binds, on=True)
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
        assert dp.map_info("nd_bindings")["max_entries"] == 64
        key, val = mac_key(host_mac(1)), Binding(64, 0xC0, i=1).value()

        def einval(v):
            assert dp.update("nd_bindings", key, v) == -errno.EINVAL
            assert dp.update_staged("nd_bindings", key, v) == -errno.EINVAL
            # a batch applies none of its entries
            both_k, both_v = np.concatenate([mac_key(host_mac(2)), key]), np.concatenate([val, v])
            assert dp.update_batch("nd_bindings", both_k, both_v) == -errno.EINVAL
            assert dp.map_info("nd_bindings")["count"] == 0

        for field, x in (("prefix_len", 129), ("pio_flags", 0x20), ("pio_flags", 0x01)):
            v = val.copy()
            v[field] = x
            einval(v)
        v = val.copy()
        v["prefix"][0, 8] = 1  # past /64
        einval(v)
        for field in ("_pad0", "_pad1", "_pad2"):
            v = val.copy()
            v[field][0, 1] = 1
            einval(v)
        v = np.zeros(1, L.bng_nd_binding)
        v["prefix"][0, 0] = 0x20  # prefix_len 0 with a prefix
        einval(v)
        v = np.zeros(1, L.bng_nd_binding)
        v["pio_flags"] = 0x80  # ... or with flags
        einval(v)
        v = np.zeros(1, L.bng_nd_binding)
        v["expires_s"] = 5  # prefix_len 0 alone: a default route only
        assert dp.update("nd_bindings", key, v) == 0
        v = Binding(128, 0xC0, i=3).value()
        assert dp.update("nd_bindings", key, v) == 0

        good = cfg_value(config(2))
        assert dp.update("nd_config", np.uint32(0), good) == 0

        def cfg_einval(c):
            assert dp.update("nd_config", np.uint32(0), c) == -errno.EINVAL
            assert dp.lookup("nd_config", np.uint32(0)).tobytes() == good.tobytes()

        for field, x in (("ra_head_len", 8), ("ra_head_len", 28), ("ra_head_len", 88), ("ra_tail_len", 4), ("ra_tail_len", 288)):
            c = good.copy()
            c[field] = x
            cfg_einval(c)
        for k, x in ((0, 133), (1, 1), (2, 1), (3, 1), (17, 0), (97, 0)):  # type, code, checksum, SLLA length, RDNSS length
            c = good.copy()
            c["ra"][0, k] = x
            cfg_einval(c)
        c = good.copy()
        c["ra"][0, 287] = 1  # past head + tail
        cfg_einval(c)
        c = good.copy()
        c["router_ll"][0, 0] = 0x20
        cfg_einval(c)
        c = good.copy()
        c["router_mac"][0, 0] = 0x01  # multicast
        cfg_einval(c)
        c = good.copy()
        c["router_mac"][0] = 0
        cfg_einval(c)
        c = good.copy()
        c["_pad1"][0, 0] = 1
        cfg_einval(c)
        c = np.zeros(1, L.bng_nd_config)
        c["router_ll"][0, 0] = 0xFE  # unconfigured must be all zero past the MAC
        cfg_einval(c)
        assert dp.update("nd_config", np.uint32(0), np.zeros(1, L.bng_nd_config)) == 0
        assert dp.update("nd_config", np.uint32(0), good) == 0
        # batch, staged, E2BIG, delete, clear
        ks = np.concatenate([mac_key(host_mac(i)) for i in range(64)])
        vs = np.concatenate([Binding(64, 0xC0, i=i).value() for i in range(64)])
        dp.clear("nd_bindings")
        assert dp.update_batch("nd_bindings", ks[:63], vs[:63]) == 0
        assert dp.update_staged("nd_bindings", ks[63:], vs[63:]) == 0
        assert dp.map_info("nd_bindings")["count"] == 64
        assert dp.update("nd_bindings", mac_key(host_mac(999)), vs[:1]) == -errno.E2BIG
        assert dp.delete("nd_bindings", ks[:1]) == 0
        assert dp.lookup("nd_bindings", ks[:1]) is None
        assert dp.lookup("nd_bindings", ks[1:2]).tobytes() == vs[1:2].tobytes()
        # snapshot / restore, delta export / apply
        blob = dp.snapshot()
        dk, _ = dp.dump("nd_bindings")
        with Dataplane(max_subscribers=64, max_batch=1 << 10) as dp2:
            dp2.restore(blob)
            k2, v2 = dp2.dump("nd_bindings")
            assert sorted(map(bytes, k2)) == sorted(map(bytes, dk)) and len(v2) == 63
            assert dp2.lookup("nd_config", np.uint32(0)).tobytes() == good.tobytes()
            # the restored configuration is live: an NS is answered once the switch is on
            f = S.ns_frame(host_mac(5), ROUTER_LL)
            dp2.nd_enable(True)
            got = run_gpu(False, arena_of([f], np.array([len(f)], np.uint32), 128), np.array([len(f)], np.uint32), None,
                          128, T0, None, None, None, dp=dp2)
            assert got[2][0] == 3
        dp.clear("nd_bindings")
        assert dp.map_info("nd_bindings")["count"] == 0
        with Dataplane(max_subscribers=64, max_batch=1 << 10) as dp3:
            dp.delta_enable(True)
            assert dp3.delta_apply(dp.delta_export(full=True)) == 0
            assert dp3.lookup("nd_config", np.uint32(0)).tobytes() == good.tobytes()
            dp.update_batch("nd_bindings", ks[:10], vs[:10])
            assert dp3.delta_apply(dp.delta_export()) == 0
            assert dp3.map_info("nd_bindings")["count"] == 10
            dp.delete("nd_bindings", ks[:1])
            assert dp3.delta_apply(dp.delta_export()) == 0
            assert dp3.map_info("nd_bindings")["count"] == 9


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
    st = np.zeros(len(L.ND_STATS), np.uint64)
    for s in range(world):
        mine = {m: b for m, b in binds.items() if S.shard_of_mac(mac_key(m), world)[0] == s}
        sel = np.nonzero(shard == s)[0]
        if not len(sel):
            continue
        sub = [frames[i] for i in sel]
        with Dataplane(max_subscribers=1 << 12, max_batch=1 << 12) as dp:
            gpu_setup(dp, cfg, mine)
            r = run_gpu(False, arena_of(sub, lens[sel], stride), lens[sel].copy(), None, stride, T0, None, cfg, mine, dp=dp)
        got_a.reshape(-1, stride)[sel] = r[0].reshape(-1, stride)
        got_l[sel], got_v[sel] = r[1], r[2]
        st += r[4]
    assert np.array_equal(got_v, one[2]) and np.array_equal(got_l, one[1]) and np.array_equal(got_a, one[0])
    assert np.array_equal(st, one[4])


@pytest.mark.gpu
def test_handover():
    """bng_sub_export carries the nd_bindings of the MACs it is given (and writes no section when there is none);
    detach removes them, import answers with them, a full destination refuses the blob whole and the source takes it
    back."""
    cfg = config(2)
    macs = [host_mac(i) for i in range(40)]
    binds = {m: Binding(64, 0xC0, i=i) for i, m in enumerate(macs)}
    moved = macs[:10] + [host_mac(500)]  # the last has no binding
    mk = np.concatenate([mac_key(m) for m in moved])
    rs = [S.rs_frame(m) for m in macs[:10]]
    lens = np.array([len(f) for f in rs], np.uint32)
    arena = arena_of(rs, lens, 512)
    with Dataplane(max_subscribers=64, max_batch=1 << 10) as a, Dataplane(max_subscribers=64, max_batch=1 << 10) as b:
        gpu_setup(a, cfg, {})
        blob0 = a.sub_export([], mk)  # no binding yet: the blob has no nd_bindings section
        gpu_setup(a, None, binds)
        blob1 = a.sub_export([], mk)
        assert b"nd_bindings" not in blob0 and b"nd_bindings" in blob1
        assert len(blob1) == len(blob0) + 64 + 10 * (8 + 48)
        assert a.map_info("nd_bindings")["count"] == 40  # no detach: nothing removed
        blob = a.sub_export([], mk, detach=True)
        assert blob == blob1 and a.map_info("nd_bindings")["count"] == 30
        got = run_gpu(False, arena, lens, None, 512, T0, None, cfg, binds, dp=a)
        assert (got[2] == 2).all()  # gone here: miss
        # a destination without room refuses the whole blob
        gpu_setup(b, cfg, {host_mac(1000 + i): Binding(64, 0xC0, i=i) for i in range(60)})
        with pytest.raises(Exception):
            b.sub_import(blob)
        assert b.map_info("nd_bindings")["count"] == 60
        # rollback: the source takes its subscribers back
        assert a.sub_import(blob) == 0 and a.map_info("nd_bindings")["count"] == 40
        for m in moved[:10]:
            assert a.lookup("nd_bindings", mac_key(m)).tobytes() == binds[m].value().tobytes()
        # with room, the destination answers them with their own prefixes
        b.clear("nd_bindings")
        assert b.sub_import(blob) == 0 and b.map_info("nd_bindings")["count"] == 10
        got = run_gpu(False, arena, lens, None, 512, T0, None, cfg, binds, dp=b)
        want = expected(arena, lens, None, 512, T0, None, (cfg, binds))
        assert (got[2] == 3).all() and np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
        # blobs without the section import as before
        assert b.sub_import(blob0) == 0 and b.map_info("nd_bindings")["count"] == 10
