// bng_b200 — per-frame logic of the reference's TC programs, written for the
// batch model: a data-parallel CLASSIFY phase that does everything whose
// result does not depend on the order of frames inside the batch, and an
// ordered RESOLVE phase (one sequential worker per subscriber, frames in index
// order) for the rest.  Field offsets are those of the reference's structs;
// each function cites the lines it must agree with bit for bit.
#pragma once
#include "common.cuh"

#define ETH_P_IP_LE 0x0008u   // bpf_htons(0x0800) as the programs compare it
#define ETH_P_IPV6_LE 0xDD86u // bpf_htons(0x86DD)
#define NO_KEY 0xFFFFFFFFu

#define TC_OK 0
#define TC_SHOT 2

// nat_config.flags, bpf/nat44.c:56-62
#define NATF_EIM 0x01u
#define NATF_HAIRPIN 0x04u
#define NATF_ALG_FTP 0x08u
#define NATF_ALG_SIP 0x10u
#define NATF_PARITY 0x20u

// ---------------------------------------------------------------------------
// antispoof_ingress — bpf/antispoof.c:188-293.  Stateless apart from counters
// and the violation log, so it is entirely a classify-phase program.
// ---------------------------------------------------------------------------
// antispoof_stats of one thread, in registers: flushed once per thread at the end of the kernel (a 64-bit shared
// atomic per dropped frame was 17 % of k_antispoof's stall samples: it compiles to a CAS loop with lane election)
struct AsCnt {
    u32 allowed;
    u32 rare; // logged | v4 violations << 10 | v6 violations << 20: a thread sees at most a few hundred frames per launch
};
#define ASC_LOGGED 1u
#define ASC_V4 (1u << 10)
#define ASC_V6 (1u << 20)
__device__ __forceinline__ void ascnt_flush(BlockStats &bs, const AsCnt &n) { // all 32 lanes
    const u32 lg = n.rare & 1023u, v4 = (n.rare >> 10) & 1023u, v6 = n.rare >> 20;
    warp_stat_flush(bs, ST_AS_ALLOWED, n.allowed);
    warp_stat_flush(bs, ST_AS_LOGGED, lg);
    warp_stat_flush(bs, ST_AS_V4_VIOL, v4);
    warp_stat_flush(bs, ST_AS_V6_VIOL, v6);
    warp_stat_flush(bs, ST_AS_DROPPED, v4 + v6);
}
// ... which bounds the batch: 1023 trips of the persistent grid (132 x 4 x 256 threads on an H100 SXM) = 138 M frames
__device__ __forceinline__ void ascnt_spill(BlockStats &bs, AsCnt &n) { // called once per trip; keeps the 10-bit fields from wrapping
    if (__any_sync(0xffffffffu, ((n.rare & 1023u) | ((n.rare >> 10) & 1023u) | (n.rare >> 20)) >= 1000u)) {
        AsCnt t = n;
        t.allowed = 0;
        const u32 lg = t.rare & 1023u, v4 = (t.rare >> 10) & 1023u, v6 = t.rare >> 20;
        warp_stat_flush(bs, ST_AS_LOGGED, lg);
        warp_stat_flush(bs, ST_AS_V4_VIOL, v4);
        warp_stat_flush(bs, ST_AS_V6_VIOL, v6);
        warp_stat_flush(bs, ST_AS_DROPPED, v4 + v6);
        n.rare = 0;
    }
}

// log_violation(), bpf/antispoof.c:150-175.  A violating frame used to reserve its record with an atomicAdd on the
// ring's one counter and wait for the answer before its warp could go on: 40 k same-address atomics per 4 M frames
// at 1 % violations, all serialised on one address.  The lanes now drop
// what the record needs into a queue of their WARP in shared memory, and the warp writes a batch of records at a
// time — one atomic for the batch, one lane per record, 64-byte records side by side (spoof_flush).  The order of the
// records in the ring is immaterial: the drain sorts by (batch, frame).
#ifndef SPOOFQ_CAP
#define SPOOFQ_CAP 64
#endif // // flushed from 32 up, at most 32 more per trip of the frame loop
struct SpoofQ {
    u32 n, pad[3];
    uint4 e[SPOOFQ_CAP][2]; // {now, source MAC, ip version} {spoofed, allowed, frame index}
};
__device__ __forceinline__ void spoofq_init(SpoofQ *q) { // q: this block's queues, one per warp
    if ((threadIdx.x & 31) == 0) q[threadIdx.x >> 5].n = 0;
    __syncwarp();
}
// q == nullptr: the record is reserved and written on the spot (the pipeline's classify kernel, where the queue's
// shared memory and the per-trip check cost more than the 1 % of frames that log gain).
__device__ __forceinline__ void spoof_log(const DevCtx &c, SpoofQ *q, AsCnt &cn, u32 idx, u64 now, const Hdr64 &h, u32 spoofed,
                                          u32 allowed_ip, bool v6) {
    // the record is emitted, then packets_logged is bumped whether or not the output succeeded (:171-174)
    const u32 m01 = (u32)h.b16(6) | ((u32)h.b16(8) << 16);
    const u32 m2 = (u32)h.b16(10) | ((v6 ? 6u : 4u) << 16);
    if (q) {
        const u32 m = __activemask(), lane = threadIdx.x & 31, leader = __ffs(m) - 1;
        u32 at = 0;
        if (lane == leader) at = atomicAdd(&q->n, (u32)__popc(m)); // (divergent groups of one warp may interleave: atomic)
        at = __shfl_sync(m, at, leader) + __popc(m & ((1u << lane) - 1));
        q->e[at][0] = make_uint4((u32)now, (u32)(now >> 32), m01, m2);
        q->e[at][1] = make_uint4(v6 ? 0 : spoofed, v6 ? 0 : allowed_ip, idx, 0);
    } else {
        u8 *r = ev_reserve(c, c.spoof_ev, idx);
        if (r) {
            ((uint4 *)r)[0] = make_uint4((u32)now, (u32)(now >> 32), m01, m2);
            ((uint4 *)r)[1] = make_uint4(v6 ? 0 : spoofed, v6 ? 0 : allowed_ip, 0, 0);
            ((uint4 *)r)[2] = make_uint4(0, 0, 0, 0);
            ((uint2 *)r)[6] = make_uint2(0, 0);
        }
    }
    cn.rare += ASC_LOGGED;
}
// The whole warp, converged: every queued violation becomes a spoof_events record.
__device__ __forceinline__ void spoof_flush(const DevCtx &c, SpoofQ &q) {
    __syncwarp();
    const u32 n = *(volatile u32 *)&q.n;
    if (!n) return;
    const u32 lane = threadIdx.x & 31;
    const EvRing &r = c.spoof_ev;
    u32 pos = 0;
    if (lane == 0) {
        pos = atomicAdd(r.count, n);
        if (pos + n > r.cap) { // staging ring full: the tail has no slot
            const u32 over = pos >= r.cap ? n : pos + n - r.cap;
            atomicSub(r.count, over);
            atomicAdd(&c.stats[r.lost_stat], (u64)over);
        }
    }
    pos = __shfl_sync(0xffffffffu, pos, 0);
    for (u32 e = lane; e < n; e += 32) {
        if (pos + e >= r.cap) break;
        u8 *rec = r.buf + (size_t)(pos + e) * r.rec_bytes; // 56 bytes of payload, then the tag
        const uint4 a = q.e[e][0], x = q.e[e][1];
        ((uint4 *)rec)[0] = a;
        ((uint4 *)rec)[1] = make_uint4(x.x, x.y, 0, 0);
        ((uint4 *)rec)[2] = make_uint4(0, 0, 0, 0);
        ((uint4 *)rec)[3] = make_uint4(0, 0, x.z, c.batch_seq);
    }
    __syncwarp();
    if (lane == 0) q.n = 0;
    __syncwarp();
}

// `bind` is the subscriber_bindings slot of the frame's source MAC (or null),
// `cfg` = default_mode | log_violations << 8; packets_allowed is counted in the
// caller's register counter n_allowed (flushed once per thread).
// A subscriber_bindings slot (32 B: key, then struct subscriber_binding) as one 32-byte load.
struct BindVal {
    bool has;
    U256 s; // w[0..1] key, w[2] ipv4_addr, w[3..6] ipv6_addr, w[7] ipv4_valid | ipv6_valid << 8 | mode << 16
};
__device__ __forceinline__ BindVal bind_load(const u8 *slot) {
    BindVal b;
    b.has = slot != nullptr;
    if (slot) b.s = ldg256(slot);
    return b;
}
__device__ __forceinline__ int antispoof_eval(const DevCtx &c, SpoofQ *sq, const Hdr64 &h, u32 len, u32 idx, u64 now, const BindVal &bv,
                                              u32 cfg, AsCnt &cn) {
    u32 &n_allowed = cn.allowed;
    const bool bind = bv.has;
    if (len < 14) return TC_OK; // :195-196, no stats
    u32 default_mode = cfg & 0xff, log_viol = (cfg >> 8) & 0xff;
    u32 b_ipv4 = 0, b_flags = 0; // flags word: ipv4_valid | ipv6_valid<<8 | mode<<16
    if (bind) {
        b_ipv4 = bv.s.w[2];
        b_flags = bv.s.w[7];
    }
    u32 mode = bind ? ((b_flags >> 16) & 0xff) : default_mode;
    if (mode == 0) { // ANTISPOOF_DISABLED :213-216
        n_allowed++;
        return TC_OK;
    }
    u32 proto = h.b16(12);
    if (proto == ETH_P_IP_LE) {
        if (len < 34) return TC_OK; // :221-222, no stats
        u32 src = h.b32(26);
        bool allowed = false;
        if (bind && (b_flags & 0xff)) {
            if (mode == 1 || mode == 3) allowed = (src == b_ipv4);
        } else if (mode == 2) {
            allowed = lpm_match(c.ranges_v4, src, 32);
        }
        if (!allowed) {
            if (log_viol) spoof_log(c, sq, cn, idx, now, h, src, bind ? b_ipv4 : 0, false);
            if (mode == 3) {
                n_allowed++;
                return TC_OK;
            }
            cn.rare += ASC_V4;
            return TC_SHOT;
        }
        n_allowed++;
        return TC_OK;
    }
    if (proto == ETH_P_IPV6_LE) {
        if (len < 54) return TC_OK; // :258-259
        bool allowed = false;
        if (bind && ((b_flags >> 8) & 0xff)) {
            allowed = true;
#pragma unroll
            for (int k = 0; k < 4; k++) // ip6->saddr at frame bytes 22..37, binding ipv6_addr at value+4
                allowed = allowed && (h.b32(22 + 4 * k) == bv.s.w[3 + k]);
        } else if (mode == 2) {
            allowed = true;
        }
        if (!allowed && mode != 3) {
            if (log_viol) spoof_log(c, sq, cn, idx, now, h, 0, 0, true);
            cn.rare += ASC_V6;
            return TC_SHOT;
        }
        n_allowed++;
        return TC_OK;
    }
    n_allowed++; // :290-292
    return TC_OK;
}

// ---------------------------------------------------------------------------
// QoS — bpf/qos_ratelimit.c.  token_bucket at slot+16:
//   tokens@16 last_update@24 rate_bps@32 burst_bytes@40 priority@44
// ---------------------------------------------------------------------------
struct TokenBucket {
    u64 tokens, last_update, rate_bps;
    u32 burst;
    u32 prio;
};

__device__ __forceinline__ void tb_load(TokenBucket &tb, const u8 *slot) {
    tb.tokens = *(const u64 *)(slot + 16);
    tb.last_update = *(const u64 *)(slot + 24);
    tb.rate_bps = *(const u64 *)(slot + 32);
    tb.burst = *(const u32 *)(slot + 40);
    tb.prio = *(const u8 *)(slot + 44);
}

// token_bucket_check(), bpf/qos_ratelimit.c:70-104, one frame; all arithmetic
// is u64 with natural wrap-around, exactly as the eBPF program computes it.
// The refill half of token_bucket_check() (:80-94).  Idempotent for a given
// `now`: a second call sees elapsed == 0 and tokens already clamped.
__device__ __forceinline__ void tb_refill(TokenBucket &tb, u64 now) {
    if (tb.last_update == now && tb.tokens <= (u64)tb.burst) return;
    u64 elapsed = now - tb.last_update;
    u64 add = (elapsed * (tb.rate_bps / 8)) / 1000000000ull;
    tb.tokens += add;
    if (tb.tokens > (u64)tb.burst) tb.tokens = tb.burst;
    tb.last_update = now;
}

__device__ __forceinline__ bool tb_step(TokenBucket &tb, u64 now, u32 pkt_len) {
    u64 elapsed = now - tb.last_update;
    u64 add = (elapsed * (tb.rate_bps / 8)) / 1000000000ull;
    tb.tokens += add;
    if (tb.tokens > (u64)tb.burst) tb.tokens = tb.burst;
    tb.last_update = now;
    if (tb.tokens >= (u64)pkt_len) {
        tb.tokens -= pkt_len;
        return true;
    }
    return false;
}

// classify for qos_{egress,ingress}_prog (:126-172, :178-222): returns the
// ordering key (bucket slot index) when the frame has to go through the
// ordered token-bucket walk, NO_KEY when its verdict is already final.
__device__ __forceinline__ u32 qos_classify_one(const DevCtx &c, BlockStats &bs, const Tbl &t, const Hdr64 &h,
                                                u32 len, u32 dlen, bool egress, u32 *prio_out, bool *prio_set) {
    *prio_set = false; // dlen: bytes present (bounds checks), len: skb->len (byte counters)
    if (dlen < 14) return NO_KEY;
    if (h.b16(12) != ETH_P_IP_LE) return NO_KEY;
    if (dlen < 34) return NO_KEY;
    u64 k = egress ? h.b32(30) : h.b32(26);
    const u8 *slot = tbl_find<1, false>(t, &k);
    if (!slot) return NO_KEY; // no policy: TC_ACT_OK without statistics
    u64 rate = *(const u64 *)(slot + QOS_RATE_COPY); // mirror of rate_bps in the key's sector
    if (rate == 0) { // unlimited: pass, bucket untouched (:77-78)
        bstats_add(bs, ST_QOS_PASS_PKTS, 1);
        bstats_add(bs, ST_QOS_PASS_BYTES, len);
        if (egress) {
            *prio_out = *(const u8 *)(slot + 44);
            *prio_set = true;
        }
        return NO_KEY;
    }
    return (u32)((slot - t.slots) / t.slot_bytes);
}

// ---------------------------------------------------------------------------
// NAT44 — bpf/nat44.c.  Slot layouts (key, then the reference value verbatim):
//   subscriber_nat: key u32 @0, value @8:  block.public_ip@8 port_start@12 port_end@14
//                   next_port@16 ports_in_use@20 allocated_at@24 subscriber_id@32
//                   sessions_active@40 sessions_total@48 bytes_out@56 bytes_in@64
//   nat_sessions:   key 16 B @0, then the hot/cold layout of common.cuh (SES_* offsets)
//   nat_reverse:    key 16 B @0, value (nat_key) @16
//   eim_table:      key 8 B @0,  value @8: external_ip@8 external_port@12 created@16
//                   last_used@24 ref_count@32 flags@36
// ---------------------------------------------------------------------------
__device__ __forceinline__ bool is_private_ip(u32 ip_le) { // bpf/nat44.c:340-363
    u32 o1 = ip_le & 0xff, o2 = (ip_le >> 8) & 0xff;       // first/second octet on the wire
    if (o1 == 10) return true;
    if (o1 == 172 && o2 >= 16 && o2 <= 31) return true;
    if (o1 == 192 && o2 == 168) return true;
    if (o1 == 100 && o2 >= 64 && o2 <= 127) return true;
    return false;
}

// Per-lane state of the ordered NAT phase: the log record reserved for this frame.
struct NatPend {
    u8 *log_rec; // staged nat_log_rb record reserved for this frame (nullptr: ring full)
    bool logged;
    bool lazy;   // nothing reserved up front: the record is reserved when it is written (a deferred TC frame, which is
                 // most often a session hit and logs nothing)
};

__device__ __forceinline__ void nat_log(const DevCtx &c, u32 idx, u64 now, u32 type, u32 sub_id, u32 priv_ip,
                                        u32 pub_ip, u16 priv_port, u16 pub_port, u32 dst_ip, u16 dst_port, u8 proto,
                                        u8 flags, NatPend *pd = nullptr) { // log_nat_event(), :531-562
    u8 *r;
    if (pd && !pd->lazy) { // the resolve kernel reserved the record up front (one atomic per 32 frames)
        r = pd->log_rec;
        pd->logged = true;
    } else {
        r = ev_reserve(c, c.natlog_ev, idx);
    }
    if (!r) return;
    ((u64 *)r)[0] = now;
    ((u32 *)r)[2] = type;
    ((u32 *)r)[3] = sub_id;
    ((u32 *)r)[4] = priv_ip;
    ((u32 *)r)[5] = pub_ip;
    ((u32 *)r)[6] = (u32)priv_port | ((u32)pub_port << 16);
    ((u32 *)r)[7] = dst_ip;
    ((u32 *)r)[8] = (u32)dst_port | ((u32)proto << 16) | ((u32)flags << 24);
    ((u32 *)r)[9] = 0;
}

// allocate_port_from_block(), :408-466.  `sub` is the subscriber_nat slot;
// only the subscriber's own resolve worker touches next_port.
__device__ __forceinline__ u16 nat_alloc_port(const DevCtx &c, u8 *sub, bool parity, u16 orig_port, u32 internal_ip,
                                              u8 proto) {
    u32 port_start = *(const u16 *)(sub + 12), port_end = *(const u16 *)(sub + 14);
    u32 next = *(volatile u32 *)(sub + 16);
    u16 found = 0;
    for (int i = 0; i < 64; i++) {
        u16 port = (u16)next;
        next += 1;
        if (port > port_end) port = (u16)port_start;
        if (next > port_end) next = port_start;
        if (parity && ((port & 1) != (orig_port & 1))) continue;
        u64 ek = (u64)internal_ip | ((u64)port << 32) | ((u64)proto << 48);
        if (tbl_find<1, true, true>(c.eim, &ek)) continue;
        found = port;
        break;
    }
    *(volatile u32 *)(sub + 16) = next;
    return found;
}

// Applies the SNAT rewrite of :752-798 to the frame in global memory.
__device__ __forceinline__ void nat_snat_rewrite(u8 *p, u32 l4, u32 proto, u32 old_ip, u32 nat_ip, u16 nat_port) {
    wr32(p, 26, nat_ip);
    wr16(p, 24, csum_upd32(rd16(p, 24), old_ip, nat_ip));
    if (proto == 6) {
        u16 old_port = rd16(p, l4);
        wr16(p, l4, nat_port);
        u16 ck = rd16(p, l4 + 16);
        ck = csum_upd32(ck, old_ip, nat_ip);
        ck = csum_upd16(ck, old_port, nat_port);
        wr16(p, l4 + 16, ck);
    } else if (proto == 17) {
        u16 old_port = rd16(p, l4);
        wr16(p, l4, nat_port);
        u16 ck = rd16(p, l4 + 6);
        if (ck != 0) {
            ck = csum_upd32(ck, old_ip, nat_ip);
            ck = csum_upd16(ck, old_port, nat_port);
            if (ck == 0) ck = 0xffff;
            wr16(p, l4 + 6, ck);
        }
    } else if (proto == 1) {
        u16 old_id = rd16(p, l4 + 4);
        wr16(p, l4 + 4, nat_port);
        wr16(p, l4 + 2, csum_upd16(rd16(p, l4 + 2), old_id, nat_port));
    }
}

// A freshly claimed nat_sessions slot becomes struct nat_session new_session (:713-728).
__device__ __forceinline__ void nat_ses_fill(u8 *ns, u32 nat_ip, u16 nat_port, u16 sport, u32 saddr, u32 daddr, u16 dport,
                                             u32 proto, u8 is_hairpin, u32 len, u64 now, u32 epoch) {
    *(u32 *)(ns + SES_NAT_IP) = nat_ip;
    *(u32 *)(ns + SES_NAT_PORT) = (u32)nat_port | (epoch << 16);
    *(u64 *)(ns + SES_OUT_LO) = 1ull | ((u64)len << 32); // packets_out = 1, bytes_out = len
    *(u64 *)(ns + SES_LAST_SEEN) = now;
    *(u32 *)(ns + SES_ORIG_IP) = saddr;
    *(u32 *)(ns + SES_STATE) = (proto << 8) | ((u32)is_hairpin << 24); // state NEW, protocol, flags 0, hairpin
    *(u64 *)(ns + SES_ORIG_PORT) = (u64)sport;                           // orig_port, then 6 unused bytes
    *(u64 *)(ns + SES_IN_LO) = 0;
    *(u64 *)(ns + SES_OUT_HI) = 0;
    *(u64 *)(ns + SES_IN_HI) = 0;
    *(u64 *)(ns + SES_CREATED) = now;
    *(u32 *)(ns + SES_DEST_IP) = daddr;
    *(u32 *)(ns + SES_DEST_PORT) = (u32)dport; // dest_port, _pad1 = 0
    *(u64 *)(ns + SES_PAD_A) = 0;              // the struct's padding bytes
}

// The parse of nat44_egress up to the session lookup (:569-665), shared by the sequential and the
// warp-cooperative paths of the ordered phase.  `sub` is the frame's subscriber_nat slot (never null here).
struct NatFlow {
    u32 saddr, daddr, proto, l4;
    u16 sport, dport;
    u8 is_hairpin;
    bool ok;     // reaches the session lookup
    bool alg;    // stopped at an ALG trigger (:615-642); alg_type then says which
    u8 alg_type;
};
// count: bump the hairpin / ALG statistics and write the ALG log record (false when an earlier phase did it for this frame)
__device__ __forceinline__ NatFlow nat_parse(const DevCtx &c, BlockStats &bs, const u8 *p, u32 dlen, u32 idx, u64 now,
                                             const u8 *sub, u32 cfg_flags, const bool COUNT) {
    NatFlow f;
    f.ok = f.alg = false;
    f.alg_type = 0;
    f.saddr = rd32(p, 26);
    f.daddr = rd32(p, 30);
    f.proto = p[23];
    f.l4 = 14 + (u32)(p[14] & 0x0f) * 4;
    f.sport = f.dport = 0;
    f.is_hairpin = 0;
    if (f.proto == 6 || f.proto == 17) {
        if (f.l4 + (f.proto == 6 ? 20u : 8u) > dlen) return f;
        f.sport = rd16(p, f.l4);
        f.dport = rd16(p, f.l4 + 2);
        u32 alg_mask = f.proto == 6 ? (NATF_ALG_FTP | NATF_ALG_SIP) : NATF_ALG_SIP;
        if (cfg_flags & alg_mask) {
            u64 ak = ((u32)bswap16(f.dport) << 16) | f.proto;
            const u8 *alg = tbl_find<1, false>(c.alg, &ak);
            if (alg) { // ALG traffic goes to userspace untranslated (:615-642)
                f.alg = true;
                f.alg_type = alg[8 + 3];
                if (COUNT) {
                    bstats_add(bs, ST_NAT_ALG, 1);
                    nat_log(c, idx, now, 7, *(const u32 *)(sub + 32), f.saddr, 0, f.sport, 0, f.daddr, f.dport, (u8)f.proto,
                            alg[8 + 3]);
                }
                return f;
            }
        }
    } else if (f.proto == 1) {
        if (f.l4 + 8 > dlen) return f;
        f.sport = rd16(p, f.l4 + 4); // echo id stands in for the source port (:647-649)
    } else {
        return f;
    }
    if (cfg_flags & NATF_HAIRPIN) {
        u64 hk = f.daddr;
        if (tbl_find<1, false>(c.hairpin, &hk)) {
            f.is_hairpin = 1;
            if (COUNT) bstats_add(bs, ST_NAT_HAIRPIN, 1);
        }
    }
    f.ok = true;
    return f;
}

struct NatOut {
    int verdict;
    bool miss; // classify only: the session does not exist yet, the ordered phase has to create it
};

// nat44_egress, :565-802, from the subscriber_nat lookup on (the caller did the Ethernet / IPv4 / private-source
// checks and found `sub`).
//   RESOLVE=false (classify, frames with IPv4 options): everything up to the session lookup, the hit
//     path, and the rewrite for hits.  A session miss is reported back.
//   RESOLVE=true: full sequential semantics for one frame, executed by the
//     subscriber's worker in frame-index order; `count_parse` says whether the
//     parse-stage counters (hairpin, ALG) are still to be bumped (classify did
//     it for frames it looked at; frames deferred past the QoS stage come fresh).
template <bool RESOLVE>
__device__ __forceinline__ NatOut nat_egress_one(const DevCtx &c, BlockStats &bs, u8 *p, u8 *sub, u32 len, u32 dlen, u32 idx,
                                                 u64 now, NatPend *pd = nullptr, const bool count_parse = !RESOLVE,
                                                 const bool stamped = false) {
    NatOut o;
    o.verdict = TC_OK;
    o.miss = false;
    const u32 cfg_flags = *(const u32 *)c.nat_config;
    const NatFlow f = nat_parse(c, bs, p, dlen, idx, now, sub, cfg_flags, count_parse);
    if (!f.ok) return o;
    const u32 saddr = f.saddr, daddr = f.daddr, proto = f.proto;
    const u16 sport = f.sport, dport = f.dport;
    u64 key[2];
    key[0] = (u64)saddr | ((u64)daddr << 32);
    key[1] = (u64)sport | ((u64)dport << 16) | ((u64)proto << 32);
    u8 *ses = tbl_find<2, RESOLVE, RESOLVE>(c.sessions, key);
    u32 nat_ip;
    u16 nat_port;
    if (ses) { // :674-680
        const u32 tr = *(const volatile u32 *)(ses + SES_NAT_PORT);
        nat_ip = *(const u32 *)(ses + SES_NAT_IP);
        nat_port = (u16)tr;
        ses_touch(ses, now, tr >> 16, c.epoch, stamped);
        ses_count(ses, SES_OUT_LO, len);
    } else {
        if (!RESOLVE) {
            o.miss = true;
            return o;
        }
        u32 sub_id = *(const u32 *)(sub + 32);
        u32 pub_ip = *(const u32 *)(sub + 8);
        bool have = false;
        if (cfg_flags & NATF_EIM) { // get_eim_mapping(), :469-528
            u64 ek = (u64)saddr | ((u64)sport << 32) | ((u64)proto << 48);
            u8 *m = tbl_find<1, true, true>(c.eim, &ek);
            if (m) {
                *(u64 *)(m + 24) = now;
                *(u32 *)(m + 32) += 1;
                bstats_add(bs, ST_NAT_EIM_HIT, 1);
            } else {
                u16 ext = nat_alloc_port(c, sub, (cfg_flags & NATF_PARITY) != 0, sport, saddr, (u8)proto);
                if (ext == 0) {
                    bstats_add(bs, ST_NAT_EXHAUST, 1);
                } else {
                    bool created;
                    m = tbl_find_or_claim<1, true>(c.eim, &ek, &created, nullptr, c.stats);
                    if (m && created) {
                        *(u32 *)(m + 8) = pub_ip;
                        *(u32 *)(m + 12) = ext; // external_port (host order) + zero pad
                        *(u64 *)(m + 16) = now;
                        *(u64 *)(m + 24) = now;
                        *(u32 *)(m + 32) = 1;
                        *(u32 *)(m + 36) = 0;
                        tbl_publish<false>(m, ek);
                        bstats_add(bs, ST_NAT_EIM_MISS, 1);
                    } else if (m) { // "someone else created it" branch (:521-527)
                        *(u32 *)(m + 32) += 1;
                        bstats_add(bs, ST_NAT_EIM_HIT, 1);
                    } else {
                        bstats_add(bs, ST_LRU_OVERFLOW, 1);
                    }
                }
            }
            if (m) {
                nat_ip = *(const u32 *)(m + 8);
                nat_port = bswap16(*(const u16 *)(m + 12));
                have = true;
            }
        }
        if (!have) { // :694-708
            u16 ap = nat_alloc_port(c, sub, (cfg_flags & NATF_PARITY) != 0, bswap16(sport), saddr, (u8)proto);
            if (ap == 0) {
                bstats_add(bs, ST_NAT_EXHAUST, 1);
                bstats_add(bs, ST_NAT_DROPPED, 1);
                nat_log(c, idx, now, 5, sub_id, saddr, pub_ip, sport, 0, daddr, dport, (u8)proto, 0, pd);
                o.verdict = TC_SHOT;
                return o;
            }
            nat_ip = pub_ip;
            nat_port = bswap16(ap);
        }
        bool created;
        u8 *ns = tbl_find_or_claim<2, true>(c.sessions, key, &created, nullptr, c.stats); // BPF_ANY (:730)
        if (ns) {
            nat_ses_fill(ns, nat_ip, nat_port, sport, saddr, daddr, dport, proto, f.is_hairpin, len, now, c.epoch);
            if (created) tbl_publish<false>(ns, key[0]);
        } else {
            bstats_add(bs, ST_LRU_OVERFLOW, 1);
        }
        u64 rk[2];
        rk[0] = (u64)daddr | ((u64)nat_ip << 32);
        rk[1] = (u64)dport | ((u64)nat_port << 16) | ((u64)proto << 32);
        u8 *rs = tbl_find_or_claim<2, true>(c.reverse, rk, &created, nullptr, c.stats); // BPF_ANY (:740)
        if (rs) {
            *(u64 *)(rs + 16) = key[0];
            *(u64 *)(rs + 24) = key[1];
            if (created) tbl_publish<false>(rs, rk[0]);
        } else {
            bstats_add(bs, ST_LRU_OVERFLOW, 1);
        }
        atomicAdd((u64 *)(sub + 40), 1ull);
        atomicAdd((u64 *)(sub + 48), 1ull);
        bstats_add(bs, ST_NAT_CREATED, 1);
        nat_log(c, idx, now, 1, sub_id, saddr, nat_ip, sport, nat_port, daddr, dport, (u8)proto, f.is_hairpin, pd);
    }
    nat_snat_rewrite(p, f.l4, proto, saddr, nat_ip, nat_port);
    bstats_add(bs, ST_NAT_SNAT, 1);
    return o;
}

// ---------------------------------------------------------------------------
// The ordered phase, warp-cooperatively: up to 32 new-flow frames of ONE subscriber (consecutive in index
// order) are created together.  The sequential walk above spends ~15 dependent table accesses per flow
// with one lane active; here every lane parses its frame, probes nat_sessions / eim_table and proposes its
// port at once, and the creations are committed in parallel.  That is only equivalent to running the
// frames one after the other when they do not interact, so the warp first finds the longest PREFIX (in
// index order) of the frames still to do that provably does not — nothing is modified until it has —
// commits that prefix and returns its lane mask; the caller runs the first frame after it through the
// sequential code and calls again for the rest.  A frame ends the prefix when
//   - an EARLIER frame of the chunk has the same 5-tuple, the same (address, port, protocol) endpoint
//     without a mapping yet, or the same nat_reverse key (the later frame must see what the earlier one
//     created, :469-487, :674, :740)
//   - its proposed port collides with an existing endpoint or with one an earlier frame of the chunk
//     creates (allocate_port_from_block() would skip it, :450-459)
//   - its proposed port lies past the end of the block (the counter wraps at that frame)
// and nothing is committed (mask 0) when port parity is filtered or a flow table is within 64 entries of
// max_entries: those chunks go frame by frame.
// Exhaustion never happens on the cooperative path: every proposed port is inside the block.
// ---------------------------------------------------------------------------
__device__ __forceinline__ u32 nat_chunk_coop(const DevCtx &c, BlockStats &bs, const DevBatch &b, u8 *sub, bool mine, u32 idx,
                                              u32 len, NatPend &pend, u32 lane, const bool count_parse = false) {
    const u32 cfg_flags = *(const u32 *)c.nat_config;
    if (cfg_flags & NATF_PARITY) return 0;
    const bool eim_on = (cfg_flags & NATF_EIM) != 0;
    u8 *p = mine ? frame_ptr(b, idx) : nullptr;
    const u64 now = mine ? frame_now(b, idx) : 0;
    const bool stamped = b.nowv != nullptr;
    const u32 dlen = frame_dlen(b, len);
    // ---- parse.  The common frame (ihl = 5, classify has already vetted it: not ALG traffic, L4 header in bounds)
    //      comes in with two 32-byte loads and is rewritten in registers, like classify does; anything else takes
    //      the byte-wise parse of the sequential code ----
    NatFlow f;
    f.ok = f.alg = false;
    Hdr64 h;
    bool fast = false, wide = false;
    if (mine && !count_parse) {
        wide = FRAME_WIDE_OK(b, p);
        if (wide) {
            const U256 a0 = ldg256(p), a1 = ldg256(p + 32);
#pragma unroll
            for (int k = 0; k < 8; k++) h.w[k] = a0.w[k], h.w[8 + k] = a1.w[k];
        } else {
            hdr_load(h, p, dlen < 64 ? dlen : 64);
        }
        const u32 proto = h.b8(23);
        fast = dlen >= 34 && h.b16(12) == ETH_P_IP_LE && (h.b8(14) & 0x0f) == 5 &&
               (proto == 6 ? dlen >= 54u : ((proto == 17 || proto == 1) && dlen >= 42u));
        if (fast) {
            f.saddr = h.b32(26), f.daddr = h.b32(30), f.proto = proto, f.l4 = 34;
            f.sport = proto == 1 ? h.b16(38) : h.b16(34);
            f.dport = proto == 1 ? (u16)0 : h.b16(36);
            f.is_hairpin = 0;
            if (cfg_flags & NATF_HAIRPIN) {
                u64 hk = f.daddr;
                if (tbl_find<1, false>(c.hairpin, &hk)) f.is_hairpin = 1;
            }
            f.ok = true;
        }
    }
    // (nothing is counted here: a frame that is not in the committed prefix comes back and is parsed again)
    if (mine && !fast) f = nat_parse(c, bs, p, dlen, idx + b.base, now, sub, cfg_flags, false);
    const bool go = mine && f.ok;
    // ---- probes: where the flow's entries are, or would go ----
    u64 key[2] = {0, 0}, ek = 0;
    u8 *ses = nullptr, *m = nullptr;
    u32 ses_ins = 0xFFFFFFFFu, eim_ins = 0xFFFFFFFFu, rev_ins = 0xFFFFFFFFu;
    if (go) {
        key[0] = (u64)f.saddr | ((u64)f.daddr << 32);
        key[1] = (u64)f.sport | ((u64)f.dport << 16) | ((u64)f.proto << 32);
        ek = (u64)f.saddr | ((u64)f.sport << 32) | ((u64)f.proto << 48);
        ses = tbl_find_ins<2>(c.sessions, key, &ses_ins);
        if (!ses && eim_on) m = tbl_find_ins<1>(c.eim, &ek, &eim_ins);
    }
    const bool create = go && !ses;          // needs a session
    const bool alloc = create && !m;         // ... and a port (EIM: a new mapping)
    const u32 below = (1u << lane) - 1;
    const u32 cmask = __ballot_sync(0xffffffffu, create), amask = __ballot_sync(0xffffffffu, alloc);
    bool clash = false, all_clash = false; // clash: this frame ends the prefix; all_clash: nothing can be committed
    if (cmask) {
        // same 5-tuple as an earlier creating lane?
        const u32 g0 = __match_any_sync(0xffffffffu, create ? key[0] : (u64)lane | (1ull << 63));
        const u32 g1 = __match_any_sync(0xffffffffu, create ? key[1] : (u64)lane | (1ull << 63));
        if (create && (g0 & g1 & cmask & below)) clash = true;
        // same endpoint as an earlier lane that would create its mapping?
        if (eim_on) {
            const u32 ge = __match_any_sync(0xffffffffu, alloc ? ek : (u64)lane | (1ull << 63));
            if (alloc && (ge & amask & below)) clash = true;
        }
    }
    const u32 nalloc = __popc(amask);
    u32 port = 0;
    const u32 port_start = *(const u16 *)(sub + 12), port_end = *(const u16 *)(sub + 14);
    const u32 next = *(volatile u32 *)(sub + 16);
    const u32 pub_ip = *(const u32 *)(sub + 8);
    if (nalloc) {
        if (next > 0xFFFFu) all_clash = true;
        port = next + __popc(amask & below);
        if (alloc && port > port_end) clash = true; // the counter wraps here: that frame goes through the sequential code
    }
    // translation of every creating lane, and its nat_reverse key
    u32 nat_ip = 0;
    u16 nat_port = 0;
    u64 rk[2] = {0, 0};
    u8 *rev = nullptr;
    if (create) {
        nat_ip = m ? *(const u32 *)(m + 8) : pub_ip;
        nat_port = m ? bswap16(*(const u16 *)(m + 12)) : bswap16((u16)port);
        rk[0] = (u64)f.daddr | ((u64)nat_ip << 32);
        rk[1] = (u64)f.dport | ((u64)nat_port << 16) | ((u64)f.proto << 32);
    }
    // second round of probes, in flight together: is the proposed port taken (:450-459)?  does the reverse key exist
    // already (:740 is BPF_ANY: then it is overwritten in place)?
    const u64 ck = (u64)f.saddr | ((u64)port << 32) | ((u64)f.proto << 48);
    if (alloc && !clash && !all_clash && tbl_has<1>(c.eim, &ck)) clash = true;
    if (create && !clash && !all_clash) rev = tbl_find_ins<2>(c.reverse, rk, &rev_ins);
    if (nalloc && eim_on) { // ... or about to be taken: an endpoint an earlier lane creates whose network-order port reads as my candidate
        for (u32 j = 0; j < 32; j++) {
            const u64 o = __shfl_sync(0xffffffffu, ek, j);
            if (alloc && j < lane && ((amask >> j) & 1) && o == ck) clash = true;
        }
    }
    const u32 ncreate = __popc(cmask);
    if (ncreate) {
        // an earlier flow of the chunk must not own the same nat_reverse key (a port handed out twice after the
        // counter wrapped: the later frame has to win)
        const u32 r0 = __match_any_sync(0xffffffffu, create ? rk[0] : (u64)lane | (1ull << 63));
        const u32 r1 = __match_any_sync(0xffffffffu, create ? rk[1] : (u64)lane | (1ull << 63));
        if (create && (r0 & r1 & cmask & below)) clash = true;
    }
    if (__any_sync(0xffffffffu, all_clash)) return 0;
    // the prefix: every frame of this call below the first one that interacts with an earlier frame
    const u32 todo = __ballot_sync(0xffffffffu, mine), cl = __ballot_sync(0xffffffffu, clash);
    const u32 take = cl ? (todo & ((1u << (__ffs(cl) - 1)) - 1)) : todo;
    if (!take) return 0;
    const bool in = (take >> lane) & 1;
    const u32 nalloc_take = __popc(amask & take);
    // room for what the prefix creates, reserved exactly (a table at max_entries sends the chunk to the sequential
    // code, which evicts); surplus — a nat_reverse key that existed, a slot found again — is given back below
    const u32 n_ses = __popc(cmask & take), n_eim = eim_on ? nalloc_take : 0;
    // (lanes 0, 1, 2 reserve in the three tables at once: one round trip instead of three)
    u32 res_ok = 1;
    if (n_ses) {
        if (lane == 0) res_ok = tbl_reserve(c.sessions, n_ses);
        if (lane == 1) res_ok = tbl_reserve(c.reverse, n_ses);
        if (lane == 2 && n_eim) res_ok = tbl_reserve(c.eim, n_eim);
        const u32 okm = __ballot_sync(0xffffffffu, res_ok != 0);
        if (okm != 0xffffffffu) { // one of the tables is at max_entries: give the others back, go sequential
            if (lane == 0 && res_ok) tbl_unreserve(c.sessions, n_ses);
            if (lane == 1 && res_ok) tbl_unreserve(c.reverse, n_ses);
            if (lane == 2 && n_eim && res_ok) tbl_unreserve(c.eim, n_eim);
            return 0;
        }
    }

    // ---- commit: nothing below depends on another lane of the chunk ----
    if (nalloc_take && lane == 0) {
        const u32 nn = next + nalloc_take;
        *(volatile u32 *)(sub + 16) = nn > port_end ? port_start : nn;
    }
    u32 n_hit = 0, n_miss = 0, n_created = 0, n_snat = 0, back_ses = 0, back_rev = 0, back_eim = 0;
    if (mine && in && count_parse) { // parse-stage counters of a frame nobody has counted yet (TC order)
        if (f.alg) {
            bstats_add(bs, ST_NAT_ALG, 1);
            nat_log(c, idx + b.base, now, 7, *(const u32 *)(sub + 32), f.saddr, 0, f.sport, 0, f.daddr, f.dport, (u8)f.proto, f.alg_type);
        } else if (f.ok && f.is_hairpin) {
            bstats_add(bs, ST_NAT_HAIRPIN, 1);
        }
    }
    if (go && in) {
        const u32 sub_id = *(const u32 *)(sub + 32);
        if (ses) { // created earlier in this batch (or by a previous chunk): the hit path, :674-680
            const u32 tr = *(const volatile u32 *)(ses + SES_NAT_PORT);
            nat_ip = *(const u32 *)(ses + SES_NAT_IP);
            nat_port = (u16)tr;
            ses_touch(ses, now, tr >> 16, c.epoch, stamped);
            ses_count(ses, SES_OUT_LO, len);
        } else {
            // the three claims first, so that their atomics are in flight together
            bool created;
            u8 *nm = nullptr, *ns, *rs = rev;
            u64 got[3];
            const u32 e_i = (!m && eim_on) ? eim_ins : 0xFFFFFFFFu, r_i = rs ? 0xFFFFFFFFu : rev_ins;
            tbl_cas3(c.eim, e_i, c.sessions, ses_ins, c.reverse, r_i, got);
            nm = tbl_claim_finish<1>(c.eim, e_i, got[0], &ek);
            ns = tbl_claim_finish<2>(c.sessions, ses_ins, got[1], key);
            bool rs_new = false;
            if (!rs) {
                rs = tbl_claim_finish<2>(c.reverse, r_i, got[2], rk);
                rs_new = rs != nullptr;
            }
            // (a slot another subscriber's worker took in the meantime: walk again)
            bool nm_new = nm != nullptr, ns_new = ns != nullptr;
            if (!m && eim_on && !nm) {
                nm = tbl_find_or_claim<1, true, true>(c.eim, &ek, &created);
                nm_new = nm && created;
            }
            if (!ns) {
                ns = tbl_find_or_claim<2, true, true>(c.sessions, key, &created);
                ns_new = ns && created;
            }
            if (!rs) {
                rs = tbl_find_or_claim<2, true, true>(c.reverse, rk, &created);
                rs_new = rs && created;
            }
            back_ses = !ns_new, back_rev = !rs_new, back_eim = (!m && eim_on && !nm_new);
            if (m) { // existing endpoint mapping (:482-487); two lanes may share it: the later frame's clock stays
                if (stamped)
                    atomicMax((unsigned long long *)(m + 24), (unsigned long long)now);
                else
                    *(u64 *)(m + 24) = now;
                atomicAdd((u32 *)(m + 32), 1u);
                n_hit = 1;
            } else if (eim_on) { // new mapping (:495-517)
                if (nm && nm_new) {
                    *(u32 *)(nm + 8) = pub_ip;
                    *(u32 *)(nm + 12) = port;
                    *(u64 *)(nm + 16) = now;
                    *(u64 *)(nm + 24) = now;
                    *(u32 *)(nm + 32) = 1;
                    *(u32 *)(nm + 36) = 0;
                    tbl_publish<false>(nm, ek);
                } else {
                    bstats_add(bs, ST_LRU_OVERFLOW, 1); // unreachable: room was checked
                }
                n_miss = 1;
            }
            if (ns) {
                nat_ses_fill(ns, nat_ip, nat_port, f.sport, f.saddr, f.daddr, f.dport, f.proto, f.is_hairpin, len, now, c.epoch);
                if (ns_new) tbl_publish<false>(ns, key[0]);
            } else {
                bstats_add(bs, ST_LRU_OVERFLOW, 1);
            }
            if (rs) {
                *(u64 *)(rs + 16) = key[0];
                *(u64 *)(rs + 24) = key[1];
                if (rs_new) tbl_publish<false>(rs, rk[0]);
            } else {
                bstats_add(bs, ST_LRU_OVERFLOW, 1);
            }
            n_created = 1;
            nat_log(c, idx + b.base, now, 1, sub_id, f.saddr, nat_ip, f.sport, nat_port, f.daddr, f.dport, (u8)f.proto, f.is_hairpin,
                    &pend);
        }
        if (fast) { // :752-798 on the header in registers, whole sectors back (as classify does for hits)
            h.s32(26, nat_ip);
            h.s16(24, csum_upd32(h.b16(24), f.saddr, nat_ip));
            if (f.proto == 6) {
                h.s16(34, nat_port);
                u16 ck2 = csum_upd32(h.b16(50), f.saddr, nat_ip);
                h.s16(50, csum_upd16(ck2, f.sport, nat_port));
            } else if (f.proto == 17) {
                h.s16(34, nat_port);
                u16 ck2 = h.b16(40);
                if (ck2 != 0) {
                    ck2 = csum_upd32(ck2, f.saddr, nat_ip);
                    ck2 = csum_upd16(ck2, f.sport, nat_port);
                    if (ck2 == 0) ck2 = 0xffff;
                    h.s16(40, ck2);
                }
            } else {
                h.s16(38, nat_port);
                h.s16(36, csum_upd16(h.b16(36), f.sport, nat_port));
            }
            if (wide) {
                stg256(p, &h.w[0]);
                if (f.proto == 6)
                    stg256(p + 32, &h.w[8]);
                else
                    hdr_store_chunk(h, p, 2);
            } else {
                hdr_store_chunk(h, p, 1);
                hdr_store_chunk(h, p, 2);
                if (f.proto == 6) hdr_store_chunk(h, p, 3);
            }
        } else {
            nat_snat_rewrite(p, f.l4, f.proto, f.saddr, nat_ip, nat_port);
        }
        n_snat = 1;
    }
    const u32 t_created = __reduce_add_sync(0xffffffffu, n_created), t_hit = __reduce_add_sync(0xffffffffu, n_hit),
              t_miss = __reduce_add_sync(0xffffffffu, n_miss), t_snat = __reduce_add_sync(0xffffffffu, n_snat);
    const u32 b_ses = __reduce_add_sync(0xffffffffu, back_ses), b_rev = __reduce_add_sync(0xffffffffu, back_rev),
              b_eim = __reduce_add_sync(0xffffffffu, back_eim);
    if (lane == 0) {
        tbl_unreserve(c.sessions, b_ses);
        tbl_unreserve(c.reverse, b_rev);
        tbl_unreserve(c.eim, b_eim);
        if (t_created) {
            atomicAdd((u64 *)(sub + 40), (u64)t_created);
            atomicAdd((u64 *)(sub + 48), (u64)t_created);
            bstats_add(bs, ST_NAT_CREATED, t_created);
        }
        if (t_hit) bstats_add(bs, ST_NAT_EIM_HIT, t_hit);
        if (t_miss) bstats_add(bs, ST_NAT_EIM_MISS, t_miss);
        if (t_snat) bstats_add(bs, ST_NAT_SNAT, t_snat);
    }
    return take;
}

// nat44_ingress, :805-948.  Every update is commutative (or made so with a
// CAS on the state byte), so this is a classify-only program.
__device__ __forceinline__ int nat_ingress_one(const DevCtx &c, BlockStats &bs, u8 *p, u32 len, u32 dlen, u64 now, bool stamped = false) {
    if (dlen < 14) return TC_OK;
    if (rd16(p, 12) != ETH_P_IP_LE) return TC_OK;
    if (dlen < 34) return TC_OK;
    u32 saddr = rd32(p, 26), daddr = rd32(p, 30);
    u32 proto = p[23];
    u32 l4 = 14 + (u32)(p[14] & 0x0f) * 4;
    u16 sport = 0, dport = 0;
    if (proto == 6) {
        if (l4 + 20 > dlen) return TC_OK;
        sport = rd16(p, l4);
        dport = rd16(p, l4 + 2);
    } else if (proto == 17) {
        if (l4 + 8 > dlen) return TC_OK;
        sport = rd16(p, l4);
        dport = rd16(p, l4 + 2);
    } else if (proto == 1) {
        if (l4 + 8 > dlen) return TC_OK;
        sport = 0;
        dport = rd16(p, l4 + 4);
    } else {
        return TC_OK;
    }
    u64 rk[2];
    rk[0] = (u64)saddr | ((u64)daddr << 32);
    rk[1] = (u64)sport | ((u64)dport << 16) | ((u64)proto << 32);
    u8 *rs = tbl_find<2, true>(c.reverse, rk);
    if (!rs) {
        bstats_add(bs, ST_NAT_PASSED, 1);
        return TC_OK;
    }
    u64 ok[2];
    ok[0] = *(const u64 *)(rs + 16);
    ok[1] = *(const u64 *)(rs + 24);
    u8 *ses = tbl_find<2, false>(c.sessions, ok);
    if (!ses) {
        // Stale reverse entry: the first frame (in index order) deletes it and
        // counts sessions_expired, later ones miss the reverse map (:871-876,
        // :861-867).  Which frame wins the erase is immaterial: all are passed
        // unmodified and the counters sum the same.
        if (tbl_erase<2>(c.reverse, rk))
            bstats_add(bs, ST_NAT_EXPIRED, 1);
        else
            bstats_add(bs, ST_NAT_PASSED, 1);
        return TC_OK;
    }
    ses_touch(ses, now, *(const volatile u16 *)(ses + SES_EPOCH), c.epoch, stamped);
    ses_count(ses, SES_IN_LO, len);
    if (proto == 6) { // :885-895; CLOSING(3) is absorbing, NEW(0)->ESTABLISHED(1) on ack
        u32 tf = p[l4 + 13];
        bool finrst = (tf & 0x05) != 0, ack = (tf & 0x10) != 0;
        if (finrst || ack) {
            u32 *sw = (u32 *)(ses + SES_STATE);
            u32 cur = *(volatile u32 *)sw;
            while (true) {
                u32 st = cur & 0xff, nst = st;
                if (finrst)
                    nst = 3;
                else if (st == 0)
                    nst = 1;
                if (nst == st) break;
                u32 prev = atomicCAS(sw, cur, (cur & ~0xffu) | nst);
                if (prev == cur) break;
                cur = prev;
            }
        }
    }
    u32 new_ip = *(const u32 *)(ses + SES_ORIG_IP);
    u16 new_port = *(const u16 *)(ses + SES_ORIG_PORT);
    wr32(p, 30, new_ip);
    wr16(p, 24, csum_upd32(rd16(p, 24), daddr, new_ip));
    if (proto == 6) {
        u16 old_port = rd16(p, l4 + 2);
        wr16(p, l4 + 2, new_port);
        u16 ck = rd16(p, l4 + 16);
        ck = csum_upd32(ck, daddr, new_ip);
        ck = csum_upd16(ck, old_port, new_port);
        wr16(p, l4 + 16, ck);
    } else if (proto == 17) {
        u16 old_port = rd16(p, l4 + 2);
        wr16(p, l4 + 2, new_port);
        u16 ck = rd16(p, l4 + 6);
        if (ck != 0) {
            ck = csum_upd32(ck, daddr, new_ip);
            ck = csum_upd16(ck, old_port, new_port);
            if (ck == 0) ck = 0xffff;
            wr16(p, l4 + 6, ck);
        }
    } else {
        u16 old_id = rd16(p, l4 + 4);
        wr16(p, l4 + 4, new_port);
        wr16(p, l4 + 2, csum_upd16(rd16(p, l4 + 2), old_id, new_port));
    }
    bstats_add(bs, ST_NAT_DNAT, 1);
    return TC_OK;
}
