// bng_b200 — pipeline_up CLASSIFY kernel: antispoof_ingress -> nat44_egress ->
// qos_ingress_prog keyed on the pre-NAT source address (SURVEY.md §7.3-8).
//
// All three stages key their mutable state on the subscriber's private
// address, so one group-by serves both the NAT new-flow ordering and the
// token-bucket ordering.  The per-address state is reached through the
// subscriber directory (common.cuh): ONE 16-byte probe tells whether the
// address owns a subscriber_nat entry, a qos_ingress bucket, and whether that
// bucket is unlimited; the directory slot is the ordering key.  MISS_FLAG in
// the value marks frames whose NAT session must be created in the ordered phase.
//
// The body is written as a sequence of warp-convergent phases (a predicate per
// frame, __syncwarp() between phases): divergence would serialise the memory
// latency of every phase once per divergent group, which is what bounds a
// gather-heavy kernel like this one.
#pragma once

// Resident blocks per SM each instantiation is compiled for (registers: 65536 / (256 x blocks)).  Fewer warps that do
// not spill beat more warps that do: at 4 blocks the pipeline instantiations get 64 registers and spill 48 bytes, at
// 3 they use 72 and spill nothing; <false,false> spills 56 bytes at 5 blocks (48 registers) and nothing at 4 (62).
// On H100 the smaller counts shorten classify by ~9 % on pipeline_imix and ~13 % on nat_steady_64 (DESIGN.md §9).
// The pipelines run best at 2 blocks (16 warps, 75 registers): classify is bound by a memory resource its warps
// share, not by the latency one warp waits out, and at 3 blocks each trip takes longer than the extra warps make up
// for (about 8 % of classify on pipeline_imix, DESIGN.md §5).
#define CLASSIFY_BLOCKS 2
#define CLASSIFY_BLOCKS_NAT 4
#define CLASSIFY_BPS(AS) ((AS) ? CLASSIFY_BLOCKS : CLASSIFY_BLOCKS_NAT)

// AS: run antispoof_ingress first; QOS: honour the qos_ingress bucket.  <false,false> is the
// standalone nat44_egress classify.
// TC: the order the reference's own TC hooks give (pkg/antispoof/tc_linux.go:32-43, pkg/qos/tc_linux.go:44-55,
// pkg/nat/tc_linux.go:37-66): antispoof -> qos_ingress -> nat44_egress.  A frame the token bucket drops never
// reaches NAT, so whatever NAT would do to a frame with a rate-limited bucket — session counters, rewrite,
// new flows, even the "no allocation" statistic — waits for the bucket's verdict: the frame goes to the ordered
// phase with DEFER_FLAG and nat44_egress runs there, after token_bucket_check().
// ACCT: traffic accounting is on for this run: attr[i] := the directory slot frame i is charged to (its source
// address as it entered), or DIR_NONE when the frame is not attributable or antispoof dropped it (acct.cu).  A
// template parameter, so that the instantiations without it are the code they were.
// V6 (bng_qos_ipv6_enable, while subscriber_ipv6 has live entries; QOS only): an untagged IPv6 frame that antispoof
// passed and whose source (bytes 22-37) has a subscriber_ipv6 owner is shaped by the owner's qos_ingress bucket: it
// skips the IPv4 directory and session probes, and the directory phase finds the owner (v6_owner) and the owner's
// directory slot in their place.  The frame gets the owner's ordering key, so the ordered phase charges it in index
// order with the owner's IPv4 frames; it never carries MISS_FLAG or DEFER_FLAG, so there it meets only the bucket, and
// nothing of NAT ever sees it.  With ACCT its attribution word is the owner's slot.
// AS6 (bng_antispoof_ipv6_prefixes_enable, while subscriber_ipv6 has live entries; AS only): antispoof_eval<true>, an
// IPv6 frame on antispoof's drop path whose source is in its binding's own prefixes is allowed.  The frame's source is
// already in h.  With V6 too, the owner antispoof found (the binding's ipv4_addr) stands in for phase 3's v6_owner.
// ICMPERR (bng_nat_icmp_errors_egress_enable): an ICMP error frame (protocol 1, type 3 / 11 / 12) on the SNAT path
// does not take the session probe: it becomes a miss (MISS_FLAG, an ordering key), so that the ordered phase looks up
// the flow it quotes in index order with the subscriber's other new flows (DESIGN.md §24).  No load past h.
template <bool AS, bool QOS, bool TC = false, bool ACCT = false, bool V6 = false, bool AS6 = false, bool ICMPERR = false>
__global__ void __launch_bounds__(BLOCK, CLASSIFY_BPS(AS))
    k_pipe_classify(const __grid_constant__ DevCtx c, const __grid_constant__ DevBatch b, u32 *skey, u32 *sval, u32 *cnt, u32 *T,
                    u32 *attr, const __grid_constant__ Tbl v6) {
    static_assert(!V6 || QOS, "IPv6 frames only ever meet a token bucket");
    static_assert(!AS6 || AS, "the prefixes widen antispoof's verdicts");
    __shared__ SmallTabs st;
    scratch_reset(cnt, T);
    __shared__ BlockStats bs;
    __shared__ u64 bar;
    __shared__ V6Lens lens;
    smem_stage_begin(&st, c.small, (u32)sizeof(SmallTabs), &bar);
    bstats_init(bs);
    if (V6 || AS6) v6_lens_load(lens, v6.plens);
    smem_stage_wait(&bar);
    const u32 lane = threadIdx.x & 31;
#define as_cfg (st.as_cfg) /* read from shared memory / the constant bank where used: no live registers */
#define nflags (st.nat_flags)
#define epoch (c.epoch)
    AsCnt cn = {0, 0};
    u32 n_snat = 0, n_qpass = 0, n_qbytes = 0; // (bytes in 32 bits: flushed per trip well before they could wrap)
    // warp-uniform trip count: every lane stays in the loop, inactive lanes are predicated off
    for (u32 base = blockIdx.x * BLOCK + (threadIdx.x & ~31u); base < b.n; base += gridDim.x * BLOCK) {
        const u32 i = base + lane;
        const bool act = i < b.n;
        const u32 len = act ? b.len[i] : 0;      // skb->len: byte counters, token bucket
        const u32 dlen = frame_dlen(b, len);     // data_end - data: every bounds check
        u8 *p = act ? frame_ptr(b, i) : b.pkts;
        const bool wide = __all_sync(0xffffffffu, !act || FRAME_WIDE_OK(b, p));
        Hdr64 h;
        hdr_load_wide(h, p, dlen, wide);

        // ---- phase 1: keys, and the first probe of every table this frame may need ----
        const bool ip4 = dlen >= 34 && h.b16(12) == ETH_P_IP_LE;
        const bool ip6 = V6 && dlen >= 38 && h.b16(12) == ETH_P_IPV6_LE; // untagged, the source's 16 bytes present
        const u32 saddr = h.b32(26), daddr = h.b32(30), proto = h.b8(23);
        const bool ihl5 = (h.b8(14) & 0x0f) == 5;
        u64 mk = mac_key(h, 6);
        const u32 bi = tbl_hash<1>(&mk) & c.bindings.home_mask;
        u64 sk = saddr;
        const u32 di = tbl_hash<1>(&sk) & c.subdir.home_mask;
        u16 sport, dport;
        if (proto == 1) {
            sport = h.b16(38); // echo id stands in for the source port (bpf/nat44.c:647-649)
            dport = 0;
        } else {
            sport = h.b16(34);
            dport = h.b16(36);
        }
        u64 key[2];
        key[0] = (u64)saddr | ((u64)daddr << 32);
        key[1] = (u64)sport | ((u64)dport << 16) | ((u64)proto << 32);
        const u32 hi = tbl_hash<2>(key) & c.sessions.mask;
        // whole 32-byte sectors per probe: the binding slot, and the flow slot's key + translation + counters; the
        // directory's home slot is one 16-byte load
        BindVal bv;
        U256 s0;
        bv.s.w[0] = bv.s.w[1] = s0.w[0] = s0.w[1] = 0xFFFFFFFFu; // K_EMPTY
        s0.w[2] = s0.w[3] = 0;
        uint4 d0 = make_uint4(0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu);
        const u8 *bslot0 = tbl_slot(c.bindings, bi);
        u8 *sslot0 = tbl_slot(c.sessions, hi);
        if (AS && dlen >= 14) bv.s = ldg256(bslot0);
        if (ip4) {
            d0 = *(const uint4 *)tbl_slot(c.subdir, di);
            s0 = ldg256(sslot0);
        }
        const u64 kw0 = (u64)s0.w[0] | ((u64)s0.w[1] << 32), kw1 = (u64)s0.w[2] | ((u64)s0.w[3] << 32);

        // ---- phase 2: antispoof_ingress ----
        int v = TC_OK;
        bool own6 = false; // AS6: antispoof allowed the frame by its binding's prefixes
        if (AS) {
            const u8 *bind = nullptr;
            if (dlen >= 14 && mk < K_BUSY) {
                const u64 w0 = (u64)bv.s.w[0] | ((u64)bv.s.w[1] << 32);
                if (w0 == mk) {
                    bind = bslot0;
                } else if (w0 != K_EMPTY) {
                    bind = tbl_finish<1>(c.bindings, &mk, bi, w0, true);
                    if (bind) bv.s = ldg256(bind);
                }
            }
            __syncwarp();
            bv.has = bind != nullptr;
            if (AS6)
                v = antispoof_eval<true>(c, nullptr, h, dlen, i + b.base, act ? frame_now(b, i) : 0, bv, as_cfg, cn, &v6, &lens, &own6);
            else
                v = antispoof_eval(c, nullptr, h, dlen, i + b.base, act ? frame_now(b, i) : 0, bv, as_cfg, cn); // (the clock is read where it is used: no live register)
            __syncwarp();
        }
        const bool alive = act && v != TC_SHOT && ip4;
        const bool alive6 = V6 && act && v != TC_SHOT && ip6;

        // ---- phase 3: the subscriber directory: does this address own a NAT block / a bucket? ----
        u32 nat_slot = DIR_NONE, qos_slot = DIR_NONE, dir_idx = ACCT ? DIR_NONE : 0; // (ACCT: DIR_NONE = no entry)
        if (alive) {
            const u64 k0 = (u64)d0.x | ((u64)d0.y << 32);
            if (k0 == sk) {
                nat_slot = d0.z, qos_slot = d0.w, dir_idx = di;
            } else if (k0 != K_EMPTY) {
                const u8 *de = tbl_finish<1>(c.subdir, &sk, di, k0, true);
                if (de) {
                    const u64 w = *(const u64 *)(de + 8);
                    nat_slot = (u32)w;
                    qos_slot = (u32)(w >> 32);
                    dir_idx = (u32)((de - c.subdir.slots) >> 4);
                }
            }
        }
        if (V6 && alive6) { // the owner's directory entry stands in for the frame's own
            u32 a[4], owner;
#pragma unroll
            for (int j = 0; j < 4; j++) a[j] = h.b32(22 + 4 * j);
            if (AS6 && own6) owner = bv.s.w[2];
            if ((AS6 && own6) || v6_owner(v6, lens, a, &owner)) {
                const u32 s = dir_slot_of(c.subdir, owner);
                if (s != DIR_NONE) {
                    qos_slot = (u32)(*(const u64 *)(c.subdir.slots + (size_t)s * 16 + 8) >> 32);
                    dir_idx = s;
                }
            }
        }
        __syncwarp();
        if (!QOS) qos_slot = DIR_NONE;
        const bool defer = TC && alive && qos_slot != DIR_NONE && !(qos_slot & DIR_QOS_UNLIMITED);
        const bool priv = alive && !defer && is_private_ip(saddr); // only private sources are translated (:583-585)
        const bool has_sub = priv && nat_slot != DIR_NONE;
        if (priv && !has_sub) bstats_add(bs, ST_NAT_PASSED, 1); // no allocation: to userspace (:592-596)
        // L4 header in bounds and a translatable protocol (:608-653); fixed offsets need ihl = 5
        bool go = has_sub && ihl5 && (proto == 6 ? dlen >= 54u : ((proto == 17 || proto == 1) && dlen >= 42u));
        if (go && proto != 1 && (nflags & (proto == 6 ? (NATF_ALG_FTP | NATF_ALG_SIP) : NATF_ALG_SIP)) && st.alg_n) {
            int ax = alg_find(st, ((u32)bswap16(dport) << 16) | proto);
            if (ax >= 0) { // ALG traffic goes to userspace untranslated (:615-642)
                bstats_add(bs, ST_NAT_ALG, 1);
                const u8 *sub = tbl_slot(c.sub_nat, nat_slot);
                nat_log(c, i + b.base, frame_now(b, i), 7, *(const u32 *)(sub + 32), saddr, 0, sport, 0, daddr, dport, (u8)proto, st.alg_type[ax]);
                go = false;
            }
        }
        __syncwarp();
        if (go && (nflags & NATF_HAIRPIN) && hp_contains(st, daddr)) bstats_add(bs, ST_NAT_HAIRPIN, 1);
        __syncwarp();
        const bool err = ICMPERR && go && proto == 1 && icmp_error_type(h.b8(34)); // (go: ihl 5, bytes 0-41 present)
        u8 *ses = go && !err ? tbl_finish<2>(c.sessions, key, hi, kw0, kw1 == key[1]) : nullptr;
        __syncwarp();

        // ---- phase 4: session hit: counters and the SNAT rewrite (:674-680, :752-798) ----
        bool miss = go && !ses;
        if (ses) {
            // the key's own sector also carries nat_ip, nat_port | epoch, and the out-direction counters
            uint2 tr = make_uint2(s0.w[4], s0.w[5]);
            if (ses != sslot0) tr = *(const uint2 *)(ses + SES_NAT_IP); // found on a later probe
            const u32 nat_ip = tr.x;
            const u16 nat_port = (u16)tr.y;
            ses_touch(ses, frame_now(b, i), tr.y >> 16, epoch, b.nowv != nullptr);
            ses_count(ses, SES_OUT_LO, len);
            h.s32(26, nat_ip);
            h.s16(24, csum_upd32(h.b16(24), saddr, nat_ip));
            if (proto == 6) {
                h.s16(34, nat_port);
                u16 ck = csum_upd32(h.b16(50), saddr, nat_ip);
                h.s16(50, csum_upd16(ck, sport, nat_port));
            } else if (proto == 17) {
                h.s16(34, nat_port);
                u16 ck = h.b16(40);
                if (ck != 0) {
                    ck = csum_upd32(ck, saddr, nat_ip);
                    ck = csum_upd16(ck, sport, nat_port);
                    if (ck == 0) ck = 0xffff;
                    h.s16(40, ck);
                }
            } else {
                h.s16(38, nat_port);
                h.s16(36, csum_upd16(h.b16(36), sport, nat_port));
            }
            // Whole sectors: bytes 0-31 (the Ethernet header goes back unchanged), then 32-63 whenever the frame owns
            // them (TCP rewrites its checksum at 50-51; UDP and ICMP write back bytes 48-63 as they were loaded), else
            // 32-47.  A partial sector is a read-modify-write at HBM once its line has left L2: storing the unchanged
            // 16 bytes too made classify ~8 % faster on pipeline_imix (DESIGN.md §9).
            if (wide) {
                stg256(p, &h.w[0]);
                if (proto == 6 || dlen >= 64)
                    stg256(p + 32, &h.w[8]);
                else
                    hdr_store_chunk(h, p, 2);
            } else {
                hdr_store_chunk(h, p, 1);
                hdr_store_chunk(h, p, 2);
                if (proto == 6) hdr_store_chunk(h, p, 3);
            }
            n_snat++;
        }
        __syncwarp();

        // ---- IPv4 options: fields are not at fixed offsets, take the generic path (rare) ----
        if (has_sub && !ihl5) {
            NatOut o = nat_egress_one<false>(c, bs, p, tbl_slot(c.sub_nat, nat_slot), len, dlen, i + b.base, frame_now(b, i), nullptr, true, b.nowv != nullptr);
            v = o.verdict;
            miss = o.miss;
        }
        __syncwarp();

        // ---- phase 5: ordering key = the directory slot ----
        u32 okey = NO_KEY, oval = i;
        if ((alive || alive6) && v != TC_SHOT) {
            if (qos_slot != DIR_NONE && (qos_slot & DIR_QOS_UNLIMITED) && !miss) {
                n_qpass++; // unlimited bucket and nothing left to order (bpf/qos_ratelimit.c:77-78)
                n_qbytes += len;
            } else if (qos_slot != DIR_NONE || miss) {
                okey = key_pack(dir_idx, len, b.kshift);
            }
            if (miss) oval |= MISS_FLAG;
            if (defer) oval |= DEFER_FLAG;
        }
        if (act) {
            b.verdict[i] = (u8)v;
            skey[i] = okey;
            sval[i] = oval;
        }
        if (ACCT) {
            // a frame too short for classify's IPv4 parse (bytes 26-29 present, 30-33 not) is still its source's
            u32 aw = (alive || alive6) ? dir_idx : DIR_NONE;
            if (act && !ip4 && dlen >= 30 && h.b16(12) == ETH_P_IP_LE && (!AS || v != TC_SHOT)) {
                const u8 *de = tbl_find<1, false>(c.subdir, &sk);
                if (de) aw = (u32)((de - c.subdir.slots) >> 4);
            }
            if (act) attr[i] = aw;
        }
        if (AS) ascnt_spill(bs, cn);
        if (QOS && __any_sync(0xffffffffu, n_qbytes >= 0x04000000u)) {
            warp_stat_flush(bs, ST_QOS_PASS_BYTES, n_qbytes);
            n_qbytes = 0;
        }
    }
#undef as_cfg
#undef nflags
#undef epoch
    if (AS) ascnt_flush(bs, cn);
    warp_stat_flush(bs, ST_NAT_SNAT, n_snat);
    if (QOS) {
        warp_stat_flush(bs, ST_QOS_PASS_PKTS, n_qpass);
        warp_stat_flush(bs, ST_QOS_PASS_BYTES, n_qbytes);
    }
    bstats_flush(bs, c.stats);
}
