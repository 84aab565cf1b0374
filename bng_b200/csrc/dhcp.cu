// bng_b200 — dhcp_fastpath_prog as a batch kernel (bpf/dhcp_fastpath.c:619-813
// with bpf/maps.h).  One thread per frame: parse Eth/(QinQ)/IPv4/UDP/BOOTP,
// identify the subscriber (VLAN pair -> circuit-id -> chaddr), and rewrite the
// request into an OFFER/ACK in place.  No state depends on frame order, so the
// whole program is a single data-parallel pass; counters go through per-block
// shared accumulators.
#include "kernels.h"
#include "progs.cuh"

#define XDP_PASS_ 2
#define XDP_TX_ 3

// pool_assignment (packed, 25 B) at `a`: pool_id@0 allocated_ip@4 vlan_id@8
// client_class@12 lease_expiry@13 flags@21  (bpf/maps.h:89-97)
__device__ __forceinline__ u64 rd_u64_unaligned(const u8 *p) {
    u64 v = 0;
#pragma unroll
    for (int i = 7; i >= 0; i--) v = (v << 8) | p[i];
    return v;
}

__device__ __forceinline__ void zero_range(u8 *q, u32 n) { // q 2-byte aligned, n even
    while (n >= 2 && ((uintptr_t)q & 15)) {
        *(u16 *)q = 0;
        q += 2;
        n -= 2;
    }
    while (n >= 16) {
        *(uint4 *)q = make_uint4(0, 0, 0, 0);
        q += 16;
        n -= 16;
    }
    while (n >= 2) {
        *(u16 *)q = 0;
        q += 2;
        n -= 2;
    }
}

__device__ __forceinline__ void put_opt32(u8 *o, int &off, u8 code, u32 v_le) { // value bytes in memory order
    o[off++] = code;
    o[off++] = 4;
    o[off++] = (u8)v_le;
    o[off++] = (u8)(v_le >> 8);
    o[off++] = (u8)(v_le >> 16);
    o[off++] = (u8)(v_le >> 24);
}

// dlen: bytes of the frame present in its slot (every bounds check); len: the frame length (tail adjustment)
__device__ __forceinline__ int dhcp_one(const DevCtx &c, BlockStats &bs, u8 *p, u32 &len, const u32 dlen, u64 now) {
    // ---- parse_packet_headers(), :352-428 ----
    if (dlen < 14) return XDP_PASS_;
    u32 proto = rd16(p, 12);
    u32 l3 = 14, vlan_off = 0, vlan_id = 0, inner_id = 0;
    bool tagged = false;
    if (proto == 0x0081u || proto == 0xA888u) { // 802.1Q / 802.1ad
        if (dlen < 18) return XDP_PASS_;
        tagged = true;
        vlan_id = bswap16(rd16(p, 14)) & 0x0FFF;
        vlan_off = 4;
        proto = rd16(p, 16);
        l3 = 18;
        bstats_add(bs, ST_DHCP_VLAN, 1);
        if (proto == 0x0081u) {
            if (dlen < 22) return XDP_PASS_;
            inner_id = bswap16(rd16(p, 18)) & 0x0FFF;
            vlan_off = 8;
            proto = rd16(p, 20);
            l3 = 22;
        }
    }
    if (proto != ETH_P_IP_LE) return XDP_PASS_;
    if (l3 + 20 > dlen) return XDP_PASS_;
    if (p[l3 + 9] != 17) return XDP_PASS_;
    u32 udp = l3 + (u32)(p[l3] & 0x0f) * 4;
    if (udp + 8 > dlen) return XDP_PASS_;
    if (rd16(p, udp + 2) != 0x4300u) return XDP_PASS_; // bpf_htons(67)
    u32 dh = udp + 8;
    if (dh + 240 > dlen) return XDP_PASS_;

    // ---- :627-645 ----
    if (p[dh] != 1) return XDP_PASS_;
    if (rd32(p, dh + 236) != 0x63538263u) return XDP_PASS_; // bpf_htonl(0x63825363)
    bstats_add(bs, ST_DHCP_TOTAL, 1);
    u32 opts = dh + 240;
    u32 msg_type = 0;
    if (opts + 12 <= dlen) { // get_dhcp_msg_type(), :216-250
        const u8 *o = p + opts;
        if (o[0] == 53 && o[1] == 1) msg_type = o[2];
        else if (o[1] == 53 && o[2] == 1) msg_type = o[3];
        else if (o[3] == 53 && o[4] == 1) msg_type = o[5];
        else if (o[4] == 53 && o[5] == 1) msg_type = o[6];
        else if (o[5] == 53 && o[6] == 1) msg_type = o[7];
        else if (o[6] == 53 && o[7] == 1) msg_type = o[8];
    }
    if (msg_type != 1 && msg_type != 3) {
        bstats_add(bs, ST_DHCP_MISS, 1);
        return XDP_PASS_;
    }

    // ---- subscriber lookup, :653-687 ----
    const u8 *a = nullptr; // -> pool_assignment
    if (tagged) {
        u64 vk = (u64)(vlan_id | (inner_id << 16));
        const u8 *s = tbl_find_conv<1>(c.vlan_pools, &vk);
        if (s) a = s + c.vlan_pools.voff;
    }
    if (!a && opts + 64 <= dlen) { // extract_circuit_id_fixed(), :267-323
        const u8 *o = p + opts;
        int cid_at = -1;
        u32 cid_len = 0;
        if (o[3] == 82) {
            u32 l82 = o[4];
            if (l82 >= 4 && opts + 5 + l82 <= dlen && o[5] == 1) {
                u32 cl = o[6];
                if (cl > 0 && cl <= 32 && opts + 7 + cl <= dlen) {
                    cid_at = 7;
                    cid_len = cl;
                }
            }
        }
        if (cid_at < 0) {
            for (int pos = 12; pos < 20; pos++) {
                if (o[pos] == 82 && opts + pos + 8 <= dlen) {
                    u32 l82 = o[pos + 1];
                    if (l82 >= 4 && o[pos + 2] == 1) {
                        u32 cl = o[pos + 3];
                        if (cl > 0 && cl <= 32 && opts + pos + 4 + cl <= dlen) {
                            cid_at = pos + 4;
                            cid_len = cl;
                            break;
                        }
                    }
                }
            }
        }
        if (cid_at >= 0) {
            u64 ck[4] = {0, 0, 0, 0};
            for (u32 k = 0; k < cid_len; k++) ck[k >> 3] |= (u64)o[cid_at + k] << ((k & 7) * 8);
            const u8 *s = tbl_find_conv<4>(c.cid_subs, ck);
            if (s) {
                a = s + c.cid_subs.voff;
                bstats_add(bs, ST_DHCP_O82_PRESENT, 1);
            }
        }
    }
    if (!a) {
        u64 mk = 0;
#pragma unroll
        for (int k = 0; k < 6; k++) mk = (mk << 8) | p[dh + 28 + k]; // chaddr
        const u8 *s = tbl_find_conv<1>(c.sub_pools, &mk);
        if (s) a = s + c.sub_pools.voff;
    }
    if (!a) {
        bstats_add(bs, ST_DHCP_MISS, 1);
        return XDP_PASS_;
    }

    // ---- lease / pool / config, :689-713 ----
    u64 now_s = now / 1000000000ull;
    if (now_s > rd_u64_unaligned(a + 13)) {
        bstats_add(bs, ST_DHCP_EXPIRED, 1);
        return XDP_PASS_;
    }
    u64 pk = *(const u32 *)a;
    const u8 *pool = tbl_find_conv<1>(c.ip_pools, &pk);
    if (!pool) {
        bstats_add(bs, ST_DHCP_ERROR, 1);
        return XDP_PASS_;
    }
    pool += c.ip_pools.voff; // ip_pool: network@0 prefix_len@4 gateway@8 dns1@12 dns2@16 lease_time@20
    bstats_add(bs, ST_DHCP_HIT, 1);
    const u8 *cfg = c.server_config; // server_mac@0 server_ip@8
    u32 allocated_ip = *(const u32 *)(a + 4);
    u32 gateway = *(const u32 *)(pool + 8);
    u32 cfg_ip = *(const u32 *)(cfg + 8);
    u32 server_ip = cfg_ip != 0 ? cfg_ip : gateway;
    u8 reply_type = msg_type == 1 ? 2 : 5;
    u32 giaddr = rd32(p, dh + 24);
    u16 smac0 = *(const u16 *)(cfg + 0), smac1 = *(const u16 *)(cfg + 2), smac2 = *(const u16 *)(cfg + 4);

    if (giaddr != 0) { // relayed: unicast back to the relay agent, :726-743
        wr16(p, 0, rd16(p, 6));
        wr16(p, 2, rd16(p, 8));
        wr16(p, 4, rd16(p, 10));
        wr32(p, l3 + 16, giaddr);
        wr16(p, udp + 2, 0x4300u);
        bstats_add(bs, ST_DHCP_UCAST, 1);
    } else { // setup_reply_l2_headers(), :436-482
        u16 flags = bswap16(rd16(p, dh + 10));
        bool bcast = (flags & 0x8000) || rd32(p, dh + 12) == 0;
        if (bcast) {
            wr16(p, 0, 0xFFFF);
            wr16(p, 2, 0xFFFF);
            wr16(p, 4, 0xFFFF);
            bstats_add(bs, ST_DHCP_BCAST, 1);
        } else {
            wr16(p, 0, rd16(p, dh + 28));
            wr16(p, 2, rd16(p, dh + 30));
            wr16(p, 4, rd16(p, dh + 32));
            bstats_add(bs, ST_DHCP_UCAST, 1);
        }
        wr32(p, l3 + 16, 0xFFFFFFFFu);
        wr16(p, udp + 2, 0x4400u); // bpf_htons(68)
    }
    wr16(p, 6, smac0);
    wr16(p, 8, smac1);
    wr16(p, 10, smac2);
    wr32(p, l3 + 12, server_ip);
    p[l3 + 8] = 64;
    wr16(p, l3 + 10, 0);
    wr16(p, udp + 0, 0x4300u);
    wr16(p, udp + 6, 0);

    // ---- BOOTP fixed part, :758-766 ----
    p[dh + 0] = 2;
    p[dh + 3] = 0;
    wr32(p, dh + 16, allocated_ip);
    wr32(p, dh + 20, server_ip);
    zero_range(p + dh + 44, 192);

    // The options bounds check comes AFTER the header rewrite (:769): a frame
    // shorter than options+64 leaves here rewritten but XDP_PASSed.
    if (opts + 64 > dlen) return XDP_PASS_;

    // ---- build_dhcp_options(), :519-602 ----
    u8 *o = p + opts;
    int off = 0;
    u32 lease = *(const u32 *)(pool + 20);
    u32 plen = pool[4];
    u32 mask = plen == 0 ? 0u : (plen >= 32 ? 0xFFFFFFFFu : bswap32(0xFFFFFFFFu << (32 - plen)));
    o[off++] = 53;
    o[off++] = 1;
    o[off++] = reply_type;
    put_opt32(o, off, 54, server_ip);
    put_opt32(o, off, 51, bswap32(lease));
    put_opt32(o, off, 1, mask);
    put_opt32(o, off, 3, gateway);
    u32 dns1 = *(const u32 *)(pool + 12), dns2 = *(const u32 *)(pool + 16);
    if (dns1 != 0) {
        o[off++] = 6;
        o[off++] = dns2 != 0 ? 8 : 4;
        for (int k = 0; k < 4; k++) o[off++] = (u8)(dns1 >> (8 * k));
        if (dns2 != 0)
            for (int k = 0; k < 4; k++) o[off++] = (u8)(dns2 >> (8 * k));
    }
    put_opt32(o, off, 58, bswap32(lease / 2));
    put_opt32(o, off, 59, bswap32((lease * 7u) / 8u));
    o[off++] = 255;

    // ---- lengths, checksum, tail adjust, :779-812 ----
    u16 dhcp_len = (u16)(240 + off);
    u16 udp_len = (u16)(8 + dhcp_len);
    u16 ip_len = (u16)(20 + udp_len);
    u16 total = (u16)(14 + vlan_off + ip_len);
    wr16(p, l3 + 2, bswap16(ip_len));
    wr16(p, udp + 4, bswap16(udp_len));
    u32 sum = 0;
#pragma unroll
    for (int k = 0; k < 10; k++) sum += rd16(p, l3 + 2 * k); // ip_checksum(), :488-503 (check is 0 here)
    sum = (sum & 0xFFFF) + (sum >> 16);
    sum = (sum & 0xFFFF) + (sum >> 16);
    wr16(p, l3 + 10, (u16)~sum);
    int delta = (int)total - (int)(u16)len;
    if (delta != 0) {
        long nl = (long)len + delta;
        if (nl < 14) { // bpf_xdp_adjust_tail() refuses to go below the Ethernet header
            bstats_add(bs, ST_DHCP_ERROR, 1);
            return XDP_PASS_;
        }
        len = (u32)nl;
    }
    return XDP_TX_;
}

// ---- DHCPv6 (include/bng_b200.h, bng_dhcpv6_enable): a bound client's Solicit / Request / Renew / Rebind answered
// from dhcpv6_bindings with what pkg/dhcpv6's buildAdvertise / buildReply would send ----
enum { D6_TOTAL, D6_SOLICIT, D6_REQUEST, D6_RENEW, D6_REBIND, D6_ADVERTISE, D6_REPLY, D6_MISS, D6_EXPIRED, D6_UNSUP, D6_NOROOM, D6_MALFORMED };

__device__ __forceinline__ u32 be16(const u8 *p, u32 o) { return ((u32)p[o] << 8) | p[o + 1]; }
__device__ __forceinline__ void put16(u8 *p, u32 &o, u32 v) {
    p[o] = (u8)(v >> 8);
    p[o + 1] = (u8)v;
    o += 2;
}
__device__ __forceinline__ void put32(u8 *p, u32 &o, u32 v) {
    put16(p, o, v >> 16);
    put16(p, o, v);
}
__device__ __forceinline__ void put_bytes(u8 *p, u32 &o, const u8 *s, u32 n) {
    for (u32 k = 0; k < n; k++) p[o + k] = s[k];
    o += n;
}

// The L3 offset of a DHCPv6 candidate, 0 for any other frame: tags as dhcp_one parses them, ethertype 0x86DD, the IPv6
// and UDP headers present, version 6, next header 17, destination port 547, destination ff02::1:2 or server_ip.
__device__ __forceinline__ u32 dhcpv6_candidate(const u8 *p, u32 dlen, const u8 *cfg) {
    if (dlen < 14) return 0;
    u32 proto = rd16(p, 12), l3 = 14;
    if (proto == 0x0081u || proto == 0xA888u) {
        if (dlen < 18) return 0;
        proto = rd16(p, 16);
        l3 = 18;
        if (proto == 0x0081u) {
            if (dlen < 22) return 0;
            proto = rd16(p, 20);
            l3 = 22;
        }
    }
    if (proto != 0xDD86u || l3 + 48 > dlen) return 0;
    if ((p[l3] >> 4) != 6 || p[l3 + 6] != 17 || rd16(p, l3 + 42) != 0x2302u) return 0; // bpf_htons(547)
    const u32 d0 = rd32(p, l3 + 24), d1 = rd32(p, l3 + 28), d2 = rd32(p, l3 + 32), d3 = rd32(p, l3 + 36);
    const bool all_servers = d0 == 0x000002FFu && d1 == 0 && d2 == 0 && d3 == 0x02000100u; // ff02::1:2
    const u32 *sip = (const u32 *)(cfg + 8);
    const bool ours = d0 == sip[0] && d1 == sip[1] && d2 == sip[2] && d3 == sip[3];
    return all_servers || ours ? l3 : 0;
}

// One candidate at L3 offset l3.  The request is parsed completely (the Client ID into the lookup key's registers,
// the IAs' IAIDs and positions) before the first byte of the reply is written over it.
__device__ __forceinline__ int dhcpv6_one(const Dhcp6Args &a, u32 *st, u8 *p, u32 &len, const u32 dlen, u64 now, u32 l3) {
    const u8 *cfg = a.cfg; // server_mac@0 duid_len@6 dns_count@7 server_ip@8 duid@24 dns@56
    const u32 udp = l3 + 40, m = udp + 8;
    atomicAdd(&st[D6_TOTAL], 1u);
    const u32 sduid = cfg[6];
    if (sduid == 0 || len > 448) {
        atomicAdd(&st[D6_UNSUP], 1u);
        return XDP_PASS_;
    }
    const u32 ulen = be16(p, udp + 4);
    if (ulen < 12 || udp + ulen > dlen) {
        atomicAdd(&st[D6_MALFORMED], 1u);
        return XDP_PASS_;
    }
    const u32 type = p[m];
    if (type != 1 && type != 3 && type != 5 && type != 6) {
        atomicAdd(&st[D6_UNSUP], 1u);
        return XDP_PASS_;
    }
    atomicAdd(&st[type == 1 ? D6_SOLICIT : type == 3 ? D6_REQUEST : type == 5 ? D6_RENEW : D6_REBIND], 1u);

    // ---- the option walk ----
    const u32 end = udp + ulen;
    u32 cid = 0, cid_len = 0, n_cid = 0, sid = 0, sid_len = 0, n_sid = 0, na = 0, na_len = 0, n_na = 0, pd = 0,
        pd_len = 0, n_pd = 0, nopt = 0;
    bool ta = false, rapid = false;
    for (u32 o = m + 4; o < end;) {
        if (o + 4 > end || ++nopt > 32) {
            atomicAdd(&st[D6_MALFORMED], 1u);
            return XDP_PASS_;
        }
        const u32 code = be16(p, o), olen = be16(p, o + 2);
        if (o + 4 + olen > end) {
            atomicAdd(&st[D6_MALFORMED], 1u);
            return XDP_PASS_;
        }
        if (code == 1) cid = o + 4, cid_len = olen, n_cid++;
        else if (code == 2) sid = o + 4, sid_len = olen, n_sid++;
        else if (code == 3) na = o + 4, na_len = olen, n_na++;
        else if (code == 4) ta = true;
        else if (code == 25) pd = o + 4, pd_len = olen, n_pd++;
        else if (code == 14) rapid = true;
        o += 4 + olen;
    }
    bool unsup = n_cid != 1 || cid_len < 1 || cid_len > 31 || ta || n_na > 1 || n_pd > 1 || (n_na && na_len < 12) ||
                 (n_pd && pd_len < 12) || (n_na | n_pd) == 0;
    if (type == 1 || type == 6) unsup = unsup || n_sid != 0;
    else if (!unsup) {
        unsup = n_sid != 1 || sid_len != sduid;
        for (u32 k = 0; k < sid_len && !unsup; k++) unsup = p[sid + k] != cfg[24 + k];
    }
    if (unsup) {
        atomicAdd(&st[D6_UNSUP], 1u);
        return XDP_PASS_;
    }

    // ---- the binding ----
    u64 kw[4] = {cid_len, 0, 0, 0}; // struct bng_dhcpv6_client_key {duid_len; duid[31]}
#pragma unroll
    for (int k = 0; k < 31; k++) {
        const u64 v = (u32)k < cid_len ? p[cid + k] : 0;
        kw[(k + 1) >> 3] |= v << (((k + 1) & 7) * 8);
    }
    const u8 *s = tbl_find_conv<4>(a.bind, kw);
    const u8 *v = s ? s + a.bind.voff : nullptr; // mac@0 flags@6 pd_len@7 iaid_na@8 iaid_pd@12 preferred@16 valid@20
                                                 // expires_s@24 addr@32 prefix@48
    if (!v || *(const u16 *)v != rd16(p, 6) || *(const u16 *)(v + 2) != rd16(p, 8) || *(const u16 *)(v + 4) != rd16(p, 10)) {
        atomicAdd(&st[D6_MISS], 1u);
        return XDP_PASS_;
    }
    if (now / 1000000000ull > *(const u64 *)(v + 24)) {
        atomicAdd(&st[D6_EXPIRED], 1u);
        return XDP_PASS_;
    }
    const u32 flags = v[6];
    const u32 iaid_na = n_na ? (be16(p, na) << 16 | be16(p, na + 2)) : 0, iaid_pd = n_pd ? (be16(p, pd) << 16 | be16(p, pd + 2)) : 0;
    if ((n_na && (!(flags & 1) || iaid_na != *(const u32 *)(v + 8))) || (n_pd && (!(flags & 2) || iaid_pd != *(const u32 *)(v + 12)))) {
        atomicAdd(&st[D6_UNSUP], 1u);
        return XDP_PASS_;
    }
    const bool adv = type == 1 && !rapid, rc_reply = type == 1 && rapid;
    const u32 dns = cfg[7];
    const u32 total = m + 4 + (4 + cid_len) + (4 + sduid) + (adv ? 5u : 13u) + (n_na ? 44u : 0u) + (n_pd ? 45u : 0u) +
                      (dns ? 4u + 16u * dns : 0u) + (rc_reply ? 4u : 0u);
    const u32 room = a.room_stride ? a.room_stride : (len + 15u) & ~15u;
    if (total > room) {
        atomicAdd(&st[D6_NOROOM], 1u);
        return XDP_PASS_;
    }

    // ---- the reply, over the request ----
    p[m] = adv ? 2 : 7; // the transaction id stays
    u32 o = m + 4;
    put16(p, o, 1);
    put16(p, o, cid_len);
#pragma unroll
    for (int k = 0; k < 31; k++)
        if ((u32)k < cid_len) p[o + k] = (u8)(kw[(k + 1) >> 3] >> (((k + 1) & 7) * 8));
    o += cid_len;
    put16(p, o, 2);
    put16(p, o, sduid);
    put_bytes(p, o, cfg + 24, sduid);
    if (adv) {
        put16(p, o, 7);
        put16(p, o, 1);
        p[o++] = 255;
    }
    const u32 pref = *(const u32 *)(v + 16), valid = *(const u32 *)(v + 20);
    const u32 t1 = pref / 2u, t2 = (pref * 4u) / 5u;
    if (n_na) {
        put16(p, o, 3);
        put16(p, o, 40);
        put32(p, o, iaid_na);
        put32(p, o, t1);
        put32(p, o, t2);
        put16(p, o, 5);
        put16(p, o, 24);
        put_bytes(p, o, v + 32, 16);
        put32(p, o, pref);
        put32(p, o, valid);
    }
    if (n_pd) {
        put16(p, o, 25);
        put16(p, o, 41);
        put32(p, o, iaid_pd);
        put32(p, o, t1);
        put32(p, o, t2);
        put16(p, o, 26);
        put16(p, o, 25);
        put32(p, o, pref);
        put32(p, o, valid);
        p[o++] = v[7];
        put_bytes(p, o, v + 48, 16);
    }
    if (dns) {
        put16(p, o, 23);
        put16(p, o, 16 * dns);
        put_bytes(p, o, cfg + 56, 16 * dns);
    }
    if (!adv) {
        put16(p, o, 13);
        put16(p, o, 9);
        put16(p, o, 0);
        put32(p, o, 0x53756363u); // "Success"
        put16(p, o, 0x6573u);
        p[o++] = 's';
    }
    if (rc_reply) {
        put16(p, o, 14);
        put16(p, o, 0);
    }
    for (u32 k = o; k & 15; k++) p[k] = 0; // to the reply's next 16-byte boundary (a frame starts on one): no stale byte
    const u32 ul = o - udp;
    // Ethernet: back to the client, from the server; the tags stay
    wr16(p, 0, rd16(p, 6));
    wr16(p, 2, rd16(p, 8));
    wr16(p, 4, rd16(p, 10));
    wr16(p, 6, *(const u16 *)(cfg + 0));
    wr16(p, 8, *(const u16 *)(cfg + 2));
    wr16(p, 10, *(const u16 *)(cfg + 4));
    // IPv6
    wr32(p, l3, 0x00000060u);
    wr16(p, l3 + 4, bswap16((u16)ul));
    p[l3 + 6] = 17;
    p[l3 + 7] = 64;
    const u32 *sip = (const u32 *)(cfg + 8);
#pragma unroll
    for (int k = 0; k < 4; k++) {
        wr32(p, l3 + 24 + 4 * k, rd32(p, l3 + 8 + 4 * k));
        wr32(p, l3 + 8 + 4 * k, sip[k]);
    }
    // UDP, with the checksum over the pseudo-header (words read in memory order: the sum is byte-order neutral)
    wr16(p, udp + 0, 0x2302u); // bpf_htons(547)
    wr16(p, udp + 2, 0x2202u); // bpf_htons(546)
    wr16(p, udp + 4, bswap16((u16)ul));
    wr16(p, udp + 6, 0);
    u32 sum = bswap16((u16)ul) + 0x1100u; // upper-layer length, next header 17
#pragma unroll
    for (int k = 0; k < 16; k++) sum += rd16(p, l3 + 8 + 2 * k);
    for (u32 k = 0; k + 1 < ul; k += 2) sum += rd16(p, udp + k);
    if (ul & 1) sum += p[udp + ul - 1];
    sum = (sum & 0xFFFF) + (sum >> 16);
    sum = (sum & 0xFFFF) + (sum >> 16);
    u16 ck = (u16)~sum;
    wr16(p, udp + 6, ck ? ck : 0xFFFFu);
    len = o;
    atomicAdd(&st[adv ? D6_ADVERTISE : D6_REPLY], 1u);
    return XDP_TX_;
}

// ---- Router and Neighbor Solicitations (include/bng_b200.h, bng_nd_enable): an RS answered with the nd_config
// template and the subscriber's own Prefix Information option, an NS for router_ll with a Neighbor Advertisement ----
enum { ND_TOTAL, ND_RS, ND_NS, ND_RA, ND_NA, ND_MISS, ND_EXPIRED, ND_NOT_TARGET, ND_MALFORMED, ND_UNSUP, ND_NOROOM };

// The L3 offset of an ND candidate, 0 for any other frame: tags as dhcp_one parses them, ethertype 0x86DD, the IPv6
// header and the first ICMPv6 byte present, version 6, next header 58, and an RS to ff02::2 or router_ll or an NS to
// router_ll or its solicited-node address.
__device__ __forceinline__ u32 nd_candidate(const u8 *p, u32 dlen, const u8 *cfg) {
    if (dlen < 14) return 0;
    u32 proto = rd16(p, 12), l3 = 14;
    if (proto == 0x0081u || proto == 0xA888u) {
        if (dlen < 18) return 0;
        proto = rd16(p, 16);
        l3 = 18;
        if (proto == 0x0081u) {
            if (dlen < 22) return 0;
            proto = rd16(p, 20);
            l3 = 22;
        }
    }
    if (proto != 0xDD86u || l3 + 41 > dlen) return 0;
    if ((p[l3] >> 4) != 6 || p[l3 + 6] != 58) return 0;
    const u32 t = p[l3 + 40];
    if (t != 133 && t != 135) return 0;
    const u32 d0 = rd32(p, l3 + 24), d1 = rd32(p, l3 + 28), d2 = rd32(p, l3 + 32), d3 = rd32(p, l3 + 36);
    const u32 *ll = (const u32 *)(cfg + 16); // router_ll, words in memory order
    if (d0 == ll[0] && d1 == ll[1] && d2 == ll[2] && d3 == ll[3]) return l3;
    if (d0 != 0x000002FFu || d1 != 0) return 0;
    if (t == 133) return d2 == 0 && d3 == 0x02000000u ? l3 : 0;              // ff02::2
    return d2 == 0x01000000u && d3 == ((ll[3] & 0xFFFFFF00u) | 0xFFu) ? l3 : 0; // ff02::1:ff00:0/104 | router_ll's low 24 bits
}

// One candidate at L3 offset l3.  Everything the reply needs from the request (its MAC and IPv6 source) is read before
// the first byte of the reply is written; the reply's ICMPv6 part is written in 2-byte stores.
__device__ __forceinline__ int nd_one(const NdArgs &a, u32 *st, u8 *p, u32 &len, const u32 dlen, u64 now, u32 l3) {
    const u8 *cfg = a.cfg; // router_mac@0 ra_head_len@8 ra_tail_len@10 router_ll@16 ra@32
    const u32 icmp = l3 + 40;
    const bool rs = p[icmp] == 133;
    atomicAdd(&st[ND_TOTAL], 1u);
    const u32 head = *(const u16 *)(cfg + 8), tail = *(const u16 *)(cfg + 10);
    if (head == 0 || len > 448) {
        atomicAdd(&st[ND_UNSUP], 1u);
        return XDP_PASS_;
    }
    const u32 plen = be16(p, l3 + 4);
    if (plen < (rs ? 8u : 24u) || icmp + plen > dlen) {
        atomicAdd(&st[ND_MALFORMED], 1u);
        return XDP_PASS_;
    }
    atomicAdd(&st[rs ? ND_RS : ND_NS], 1u);

    // ---- validity (RFC 4861 §6.1.1, §7.1.1) ----
    const u32 s0 = rd32(p, l3 + 8), s1 = rd32(p, l3 + 12), s2 = rd32(p, l3 + 16), s3 = rd32(p, l3 + 20);
    const bool unspec = (s0 | s1 | s2 | s3) == 0;
    bool bad = p[l3 + 7] != 255 || p[icmp + 1] != 0;
    // the checksum over the pseudo-header (words read in memory order: the sum is byte-order neutral)
    u32 sum = bswap16((u16)plen) + 0x3A00u; // upper-layer length, next header 58
#pragma unroll
    for (int k = 0; k < 16; k++) sum += rd16(p, l3 + 8 + 2 * k);
    for (u32 k = 0; k + 1 < plen; k += 2) sum += rd16(p, icmp + k);
    if (plen & 1) sum += p[icmp + plen - 1];
    sum = (sum & 0xFFFF) + (sum >> 16);
    sum = (sum & 0xFFFF) + (sum >> 16);
    bad = bad || sum != 0xFFFFu;
    const u32 end = icmp + plen;
    u32 nopt = 0;
    bool slla = false;
    for (u32 o = icmp + (rs ? 8u : 24u); o < end && !bad;) {
        if (o + 2 > end || p[o + 1] == 0 || o + 8u * p[o + 1] > end || ++nopt > 32) {
            bad = true;
            break;
        }
        slla = slla || p[o] == 1;
        o += 8u * p[o + 1];
    }
    bad = bad || (unspec && slla);
    if (!rs) bad = bad || p[icmp + 8] == 0xFF || (unspec && p[l3 + 24] != 0xFF); // multicast target; :: to router_ll
    if (bad) {
        atomicAdd(&st[ND_MALFORMED], 1u);
        return XDP_PASS_;
    }
    const u32 *ll = (const u32 *)(cfg + 16);
    if (!rs && (rd32(p, icmp + 8) != ll[0] || rd32(p, icmp + 12) != ll[1] || rd32(p, icmp + 16) != ll[2] ||
                rd32(p, icmp + 20) != ll[3])) {
        atomicAdd(&st[ND_NOT_TARGET], 1u);
        return XDP_PASS_;
    }

    // ---- the binding (RS) ----
    const u8 *v = nullptr; // prefix@0 prefix_len@16 pio_flags@17 valid@20 preferred@24 expires_s@32
    if (rs) {
        u64 mk = 0;
#pragma unroll
        for (int k = 0; k < 6; k++) mk = (mk << 8) | p[6 + k];
        const u8 *s = tbl_find_conv<1>(a.bind, &mk);
        if (!s) {
            atomicAdd(&st[ND_MISS], 1u);
            return XDP_PASS_;
        }
        v = s + a.bind.voff;
        if (now / 1000000000ull > *(const u64 *)(v + 32)) {
            atomicAdd(&st[ND_EXPIRED], 1u);
            return XDP_PASS_;
        }
    }
    const u32 pl = rs ? v[16] : 0;
    const u32 ilen = rs ? head + (pl ? 32u : 0u) + tail : 32u;
    const u32 room = a.room_stride ? a.room_stride : (len + 15u) & ~15u;
    if (icmp + ilen > room) {
        atomicAdd(&st[ND_NOROOM], 1u);
        return XDP_PASS_;
    }

    // ---- the reply, over the request ----
    u32 o = icmp;
    if (rs) {
        const u8 *ra = cfg + 32;
        for (u32 k = 0; k < head; k += 4) wr32(p, o + k, *(const u32 *)(ra + k));
        o += head;
        if (pl) {
            wr16(p, o, 0x0403u);
            wr16(p, o + 2, (u16)(pl | (u32)v[17] << 8));
            wr32(p, o + 4, __byte_perm(*(const u32 *)(v + 20), 0, 0x0123));
            wr32(p, o + 8, __byte_perm(*(const u32 *)(v + 24), 0, 0x0123));
            wr32(p, o + 12, 0);
#pragma unroll
            for (int k = 0; k < 4; k++) wr32(p, o + 16 + 4 * k, *(const u32 *)(v + 4 * k));
            o += 32;
        }
        for (u32 k = 0; k < tail; k += 4) wr32(p, o + k, *(const u32 *)(ra + head + k));
        o += tail;
    } else {
        wr32(p, o, 0x00000088u); // type 136, code 0, checksum 0 for now
        wr32(p, o + 4, unspec ? 0xA0u : 0xE0u);
#pragma unroll
        for (int k = 0; k < 4; k++) wr32(p, o + 8 + 4 * k, ll[k]);
        wr16(p, o + 24, 0x0102u); // Target Link-Layer Address, 1 x 8 bytes
#pragma unroll
        for (int k = 0; k < 3; k++) wr16(p, o + 26 + 2 * k, *(const u16 *)(cfg + 2 * k));
        o += 32;
    }
    for (u32 k = o; k & 15; k += 2) wr16(p, k, 0); // to the reply's next 16-byte boundary (a frame starts on one)
    // Ethernet: back to the requester, from the router; the tags stay
    wr16(p, 0, rd16(p, 6));
    wr16(p, 2, rd16(p, 8));
    wr16(p, 4, rd16(p, 10));
#pragma unroll
    for (int k = 0; k < 3; k++) wr16(p, 6 + 2 * k, *(const u16 *)(cfg + 2 * k));
    // IPv6
    wr32(p, l3, 0x00000060u);
    wr16(p, l3 + 4, bswap16((u16)ilen));
    wr16(p, l3 + 6, 0xFF3Au); // next header 58, hop limit 255
#pragma unroll
    for (int k = 0; k < 4; k++) wr32(p, l3 + 8 + 4 * k, ll[k]);
    wr32(p, l3 + 24, unspec ? 0x000002FFu : s0); // ff02::1 for ::
    wr32(p, l3 + 28, unspec ? 0u : s1);
    wr32(p, l3 + 32, unspec ? 0u : s2);
    wr32(p, l3 + 36, unspec ? 0x01000000u : s3);
    u32 ck = bswap16((u16)ilen) + 0x3A00u;
#pragma unroll
    for (int k = 0; k < 16; k++) ck += rd16(p, l3 + 8 + 2 * k);
    for (u32 k = 0; k < ilen; k += 2) ck += rd16(p, icmp + k);
    ck = (ck & 0xFFFF) + (ck >> 16);
    ck = (ck & 0xFFFF) + (ck >> 16);
    wr16(p, icmp + 2, (u16)~ck);
    len = o;
    atomicAdd(&st[rs ? ND_RA : ND_NA], 1u);
    return XDP_TX_;
}

// Tile kernel (one mbarrier per block rather than per-thread barriers without any block-wide synchronisation): a
// request is up to ~350 bytes that the program reads sparsely and rewrites almost
// entirely (L2 headers, BOOTP fixed part, 192 zeroed bytes, options), so frames are staged through
// shared memory with the TMA: every thread bulk-copies its frame (cp.async.bulk, completion on an
// mbarrier), runs the program on the shared-memory copy, and bulk-stores it back.  HBM sees two
// streaming passes per frame instead of scattered 1-16 byte accesses.
#define DH_TILE 128
// Bytes staged per frame, also the slot stride in shared memory.  400 = 16 x 25: a multiple of 16 (bulk
// copies) whose word stride (100) spreads same-offset accesses of the 32 lanes over 8 banks; 384 or 448
// would put them on 1 or 2.  Frames whose options end beyond it (QinQ + IPv4 options) run in place.
#define DH_SLOT 400

// Tile mode: in a fixed-stride arena (a receive ring: what a NIC fills) the 128 frames of a tile are one
// contiguous run, so the whole tile moves with ONE bulk copy each way instead of one per frame — the per-frame
// version issues 2 x 2^22 TMA operations per batch, a few dozen cycles apart on every SM, and that, not HBM,
// bounds it.  Every other arena (an offset table, or slots that do not fit a staging slot) moves frame by frame.
// V6: DHCPv6 candidates among the frames dhcp_one passed as not IPv4 are answered by dhcpv6_one (bng_dhcpv6_enable)
// ND: so are Router and Neighbor Solicitations among the frames still passed, by nd_one (bng_nd_enable)
template <bool V6, bool ND>
__global__ void __launch_bounds__(DH_TILE) k_dhcp_fastpath(const __grid_constant__ DevCtx c, const __grid_constant__ DevBatch b,
                                                           const __grid_constant__ Dhcp6Args a, const __grid_constant__ NdArgs na) {
    extern __shared__ __align__(128) u8 stage[]; // DH_TILE * DH_SLOT
    __shared__ BlockStats bs;
    __shared__ u64 bar, bar1;
    __shared__ u32 s6[V6 ? ST_DHCP6_N : 1];
    if constexpr (V6) {
        if (threadIdx.x < ST_DHCP6_N) s6[threadIdx.x] = 0;
    }
    __shared__ u32 snd[ND ? ST_ND_N : 1];
    if constexpr (ND) {
        if (threadIdx.x < ST_ND_N) snd[threadIdx.x] = 0;
    }
    bstats_init(bs);
    const u32 bar_a = (u32)__cvta_generic_to_shared(&bar), bar1_a = (u32)__cvta_generic_to_shared(&bar1);
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar_a), "r"(DH_TILE));
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar1_a));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    // tile mode: fixed stride no larger than a staging slot, every frame's bytes inside its slot
    const bool tile_mode = !b.off16 && b.stride <= DH_SLOT && b.cap == b.stride;
    const u32 sstride = tile_mode ? b.stride : DH_SLOT; // slot stride in shared memory
    u8 *mine = stage + (size_t)threadIdx.x * sstride;
    const u32 mine_a = (u32)__cvta_generic_to_shared(mine), stage_a = (u32)__cvta_generic_to_shared(stage);
    u32 phase = 0;
    for (u32 base = blockIdx.x * DH_TILE; base < b.n; base += gridDim.x * DH_TILE) {
        const u32 i = base + threadIdx.x;
        const bool act = i < b.n;
        u32 len = act ? b.len[i] : 0;
        u8 *g = act ? frame_ptr(b, i) : b.pkts;
        const u32 present = frame_dlen(b, len);
        u32 nbytes = ((present < DH_SLOT ? present : DH_SLOT) + 15u) & ~15u;
        if (nbytes > DH_SLOT) nbytes = DH_SLOT;
        const u32 tile_bytes = (b.n - base < (u32)DH_TILE ? b.n - base : (u32)DH_TILE) * b.stride;
        // ---- stage in ----
        if (tile_mode) {
            if (threadIdx.x == 0) {
                asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar1_a), "r"(tile_bytes) : "memory");
                asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(stage_a),
                             "l"(b.pkts + (size_t)base * b.stride), "r"(tile_bytes), "r"(bar1_a)
                             : "memory");
            }
        } else if (nbytes) {
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_a), "r"(nbytes) : "memory");
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(mine_a),
                         "l"(g), "r"(nbytes), "r"(bar_a)
                         : "memory");
        } else {
            asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar_a) : "memory");
        }
        u32 done = 0;
        while (!done) {
            asm volatile(
                "{\n\t.reg .pred p;\n\t"
                "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
                "selp.u32 %0, 1, 0, p;\n\t}"
                : "=r"(done)
                : "r"(tile_mode ? bar1_a : bar_a), "r"(phase)
                : "memory");
        }
        phase ^= 1;
        // ---- the program, on the staged copy ----
        bool direct = false; // the program would reach past the staged bytes: run it on the frame itself
        if (act && present > DH_SLOT) {
            u32 et = rd16(mine, 12), l3 = 14;
            if (et == 0x0081u || et == 0xA888u) {
                l3 = 18;
                if (rd16(mine, 16) == 0x0081u) l3 = 22;
            }
            direct = l3 + (u32)(mine[l3] & 0x0f) * 4 + 8 + 240 + 64 > DH_SLOT;
            if constexpr (V6 || ND) {
                if (rd16(mine, l3 - 2) == 0xDD86u) direct = true; // an IPv6 frame is decided by its ethertype
            }
        }
        u32 grown = 0; // V6, ND: the bytes of an answered frame, rounded up to 16
        if (act) {
            const u32 l0 = len;
            u8 *fp = direct ? g : mine;
            const u32 dl = frame_dlen(b, l0);
            int v = dhcp_one(c, bs, fp, len, dl, frame_now(b, i));
            if constexpr (V6) {
                if (v == XDP_PASS_) {
                    const u32 l3 = dhcpv6_candidate(fp, dl, a.cfg);
                    if (l3 && (v = dhcpv6_one(a, s6, fp, len, dl, frame_now(b, i), l3)) == XDP_TX_) grown = (len + 15u) & ~15u;
                }
            }
            if constexpr (ND) { // disjoint from DHCPv6's candidates: next header 58, not 17
                if (v == XDP_PASS_) {
                    const u32 l3 = nd_candidate(fp, dl, na.cfg);
                    if (l3 && (v = nd_one(na, snd, fp, len, dl, frame_now(b, i), l3)) == XDP_TX_) grown = (len + 15u) & ~15u;
                }
            }
            b.verdict[i] = (u8)v;
            if (len != l0) b.len[i] = len;
        }
        if (direct) nbytes = 0;
        if constexpr (V6 || ND) { // a reply can be longer than its request: store it back whole
            u32 *need = V6 ? a.need : na.need;
            if (!direct && grown > nbytes) nbytes = grown;
            if (grown && need && grown > need[i]) need[i] = grown;
        }
        // ---- stage out (every staged frame: a passed frame may have been rewritten, :769) ----
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        if (tile_mode) {
            __syncthreads(); // every thread's writes to the tile are done (and fenced) before the one store reads it
            if (threadIdx.x == 0) {
                asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(b.pkts + (size_t)base * b.stride), "r"(stage_a),
                             "r"(tile_bytes)
                             : "memory");
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); // the tile buffer is reused
            }
        } else if (nbytes) {
            asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(g), "r"(mine_a), "r"(nbytes) : "memory");
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); // the slot is reused by the next tile
        }
        __syncthreads();
    }
    if (tile_mode && threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
    bstats_flush(bs, c.stats);
    if constexpr (V6) {
        if (threadIdx.x < ST_DHCP6_N && s6[threadIdx.x]) atomicAdd(&a.stats[threadIdx.x], (u64)s6[threadIdx.x]);
    }
    if constexpr (ND) {
        if (threadIdx.x < ST_ND_N && snd[threadIdx.x]) atomicAdd(&na.stats[threadIdx.x], (u64)snd[threadIdx.x]);
    }
}

// (A double-buffered variant — two staging slots per thread, the load of tile i+1 issued before the program runs on
// tile i — was tried and dropped: it was slower.)

static std::string dhcp_name(bool v6, bool nd) {
    const std::string tags = std::string(v6 ? ",v6" : "") + (nd ? ",nd" : "");
    return "k_dhcp_fastpath" + (tags.empty() ? tags : "<" + tags.substr(1) + ">");
}

cudaError_t run_dhcp_fastpath(Launcher &L, const DevCtx &c, const DevBatch &b, const Dhcp6Args *d6, const NdArgs *nd) {
    const int smem = DH_TILE * DH_SLOT;
    long want = ((long)b.n + DH_TILE - 1) / DH_TILE;
    long cap = (long)L.num_sms * 4; // 4 x 50 KB of staging per SM (of the 228 KB an H100 SM has)
    int grid = (int)(want < cap ? (want < 1 ? 1 : want) : cap);
    return with_flags(
        [&](auto v6f, auto ndf) {
            constexpr bool V6 = decltype(v6f)::value, ND = decltype(ndf)::value;
            int &set = L.dhcp_smem_set[V6 * 2 + ND];
            if (!set) { // function attributes are per device: set on the device this context runs on
                cudaError_t e = cudaFuncSetAttribute(k_dhcp_fastpath<V6, ND>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
                if (e != cudaSuccess) return e;
                set = 1;
            }
            prof_begin(L, prof_name<dhcp_name, V6, ND>());
            k_dhcp_fastpath<V6, ND><<<grid, DH_TILE, smem, L.stream>>>(c, b, V6 ? *d6 : Dhcp6Args{}, ND ? *nd : NdArgs{});
            prof_end(L);
            L.launches++;
            return cudaGetLastError();
        },
        d6 != nullptr, nd != nullptr);
}
