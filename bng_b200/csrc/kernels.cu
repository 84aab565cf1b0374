// bng_b200 — batch kernels for the TC programs (antispoof, QoS, NAT44) and the
// upstream pipeline.
//
// Execution model (DESIGN.md §3).  Frames of a batch must take effect in index
// order.  Three phases run back to back on the context's stream:
//   CLASSIFY  one thread per frame over a persistent grid (a multiple of the
//             SM count).  The first 64 bytes of the frame are held in
//             registers (2 x 32-byte loads, or 4 x 16-byte for unaligned
//             frames), the first probe slot of every table the frame may need
//             is fetched up front as whole 32-byte sectors so the loads are in
//             flight together, and everything whose effect commutes is
//             finished here: verdicts, session counters (one atomic), the
//             in-place SNAT rewrite (whole-sector stores).  Frames
//             whose effect depends on earlier frames of the same subscriber
//             (new NAT flows, token-bucket decisions) only get an ordering key.
//   GROUP     a stable LSD radix sort (8-bit digits) of (key, frame index)
//             pairs groups those frames by subscriber while keeping index
//             order inside a group.  The first pass also compacts: frames
//             without a key never enter the sort, and every later kernel reads
//             its element count from device memory, so an all-hit batch costs
//             a few empty launches and no host round trip.
//   RESOLVE   one warp per subscriber walks its group: 256 (key + length, frame)
//             pairs per sweep are staged in shared memory with coalesced
//             loads (the frame length rides in the spare bits of the ordering
//             key), new flows are created warp-cooperatively in index order,
//             and the token bucket is applied with warp-uniform fast paths
//             (whole chunk passes / whole chunk drops) before falling back to
//             a lane-by-lane scan.
// The kernels after CLASSIFY are launched with programmatic stream
// serialisation (launch_dep / pdl_wait): their launch overlaps the tail of the
// kernel before them.
#include <string.h>

#include "kernels.h"
#include "progs.cuh"

#define BLOCK 256
#define MISS_FLAG 0x80000000u
#define DEFER_FLAG 0x20000000u // pipeline_tc: nat44_egress runs in the ordered phase, after the token bucket passed the frame

// device-side counters (Scratch::counters)
#define IDX_MASK 0x1FFFFFFFu // frame index bits of a grouped value (flags above)
enum { CNT_M = 0, CNT_NSEG = 1, CNT_DEFERRED = 2, CNT_MAXKEY = 3, CNT_WORK = 4 };

// The group-by's device counters and per-pass digit totals start every batch at zero: the classify kernel that feeds
// it clears them (block 0) instead of two memset launches ahead of it — nothing reads them before the kernel ends.
__device__ __forceinline__ void scratch_reset(u32 *cnt, u32 *T) {
    if (blockIdx.x == 0) {
        for (u32 i = threadIdx.x; i < 16 + 4 * 256; i += blockDim.x) (i < 16 ? cnt[i] : T[i - 16]) = 0;
    }
}

// The grouped (key, value) arrays live in one of two ping-pong buffers depending on how many radix
// passes actually ran: passes whose digit is zero for every key of the batch (largest key < 2^(8p))
// are skipped on the device, so the consumers pick the buffer from the device-side maximum.
struct Grouped {
    const u32 *ka, *va, *kb, *vb; // pass 0 writes a -> b, pass 1 b -> a, ...
    int passes;
    u32 kshift; // the keys carry the frame length above this bit (0: they do not), DevBatch.kshift
};
__device__ __forceinline__ bool rs_pass_needed(const u32 *cnt, int shift) { return shift == 0 || (cnt[CNT_MAXKEY] >> shift) != 0; }
__device__ __forceinline__ void grouped_select(const Grouped &g, const u32 *cnt, const u32 *&k, const u32 *&v) {
    int done = 1;
    while (done < g.passes && rs_pass_needed(cnt, 8 * done)) done++;
    k = (done & 1) ? g.kb : g.ka;
    v = (done & 1) ? g.vb : g.va;
}

// ---------------------------------------------------------------------------
// antispoof_ingress
// V6 (bng_antispoof_ipv6_prefixes_enable, while subscriber_ipv6 has live entries): antispoof_eval<true>, a
// subscriber's own prefixes count as its IPv6 addresses; only frames on the IPv6 drop path probe the table.
// ---------------------------------------------------------------------------
#define AS_MINB 5
template <bool V6>
__global__ void __launch_bounds__(BLOCK, AS_MINB) k_antispoof(const __grid_constant__ DevCtx c, const __grid_constant__ DevBatch b,
                                                              const __grid_constant__ Tbl v6) {
    __shared__ BlockStats bs;
    __shared__ SpoofQ sqs[BLOCK / 32];
    __shared__ V6Lens lens;
    static_assert(64 <= SPOOFQ_CAP, "a trip's 32 frames must fit in what a flush at 32 leaves free");
    bstats_init(bs);
    spoofq_init(sqs);
    if (V6) v6_lens_load(lens, v6.plens);
    SpoofQ &sq = sqs[threadIdx.x >> 5];
    u32 cfg = *(const u16 *)c.as_config;
    AsCnt cn = {0, 0};
    const u32 lane = threadIdx.x & 31;
    // warp-uniform trip count: the warp decides together whether its frames allow 32-byte loads
    for (u32 base = blockIdx.x * BLOCK + (threadIdx.x & ~31u); base < b.n; base += gridDim.x * BLOCK) {
        if (*(volatile u32 *)&sq.n >= 32) spoof_flush(c, sq); // (warp-uniform: the queue is the warp's own)
        const u32 i = base + lane;
        const bool act = i < b.n;
        const u32 len = act ? frame_dlen(b, b.len[i]) : 0; // antispoof only bounds-checks: the bytes present
        // antispoof_ingress reads the Ethernet header and the IPv4 source address (bytes 26-29): the first 32-byte
        // sector of the frame.  Only an IPv6 frame needs more (its source address ends at byte 37).
        const u8 *p = act ? frame_ptr(b, i) : b.pkts;
        Hdr64 h;
        hdr_load_wide(h, p, len < 32 ? len : 32, __all_sync(0xffffffffu, !act || FRAME_WIDE_OK(b, p)));
        if (len > 32 && h.b16(12) == ETH_P_IPV6_LE) hdr_load(h, p, len < 48 ? len : 48);
        // first probe = the home PAIR of 32-byte slots (key + binding each), both in flight at once; a third slot
        // is needed by ~0.1 % of the lookups (the table is sparse)
        BindVal bv;
        U256 s1;
        u64 mk = mac_key(h, 6);
        bv.has = false;
        const u32 hi = tbl_hash<1>(&mk) & c.bindings.home_mask;
        if (len >= 14) {
            bv.s = ldg256(tbl_slot(c.bindings, hi));
            s1 = ldg256(tbl_slot(c.bindings, hi + 1));
            const u64 w0 = (u64)bv.s.w[0] | ((u64)bv.s.w[1] << 32), w1 = (u64)s1.w[0] | ((u64)s1.w[1] << 32);
            if (w0 == mk) {
                bv.has = true;
            } else if (w0 != K_EMPTY && w1 == mk) {
                bv.has = true;
                bv.s = s1;
            } else if (w0 != K_EMPTY && w1 != K_EMPTY) {
                bv = bind_load(tbl_finish<1>(c.bindings, &mk, hi + 1, w1, true));
            }
        }
        if (V6) {
            bool own6 = false;
            if (act) b.verdict[i] = (u8)antispoof_eval<true>(c, &sq, h, len, i + b.base, frame_now(b, i), bv, cfg, cn, &v6, &lens, &own6);
        } else if (act) {
            b.verdict[i] = (u8)antispoof_eval(c, &sq, h, len, i + b.base, frame_now(b, i), bv, cfg, cn);
        }
        ascnt_spill(bs, cn);
    }
    spoof_flush(c, sq);
    ascnt_flush(bs, cn);
    bstats_flush(bs, c.stats);
}

// ---------------------------------------------------------------------------
// qos_egress_prog / qos_ingress_prog: classify
// V6 (bng_qos_ipv6_enable, while subscriber_ipv6 has live entries): an untagged IPv6 frame whose source (22-37,
// ingress) or destination (38-53, egress) has a subscriber_ipv6 owner takes the owner's bucket, as an IPv4 frame from
// or to the owner would: its ordering key is that bucket's slot.
// ---------------------------------------------------------------------------
template <bool V6>
__global__ void __launch_bounds__(BLOCK)
    k_qos_classify(const __grid_constant__ DevCtx c, const __grid_constant__ DevBatch b, int egress, u32 *skey, u32 *sval, u32 *cnt, u32 *T,
                   const __grid_constant__ Tbl v6) {
    __shared__ BlockStats bs;
    __shared__ V6Lens lens;
    scratch_reset(cnt, T);
    bstats_init(bs);
    if (V6) v6_lens_load(lens, v6.plens);
    const Tbl &t = egress ? c.qos_eg : c.qos_in;
    constexpr u32 HB = V6 ? 54 : 34; // header bytes read: through the IPv4 addresses, or through the IPv6 destination
    for (u32 i = blockIdx.x * BLOCK + threadIdx.x; i < b.n; i += gridDim.x * BLOCK) {
        u32 len = b.len[i];
        const u32 dlen = frame_dlen(b, len);
        const u8 *p = frame_ptr(b, i);
        Hdr64 h;
        hdr_load_wide(h, p, dlen < HB ? dlen : HB, __all_sync(__activemask(), FRAME_WIDE_OK(b, p)));
        u32 prio;
        bool prio_set;
        u32 key;
        if (V6 && dlen >= (egress ? 54u : 38u) && h.b16(12) == ETH_P_IPV6_LE) {
            u32 a[4], owner;
#pragma unroll
            for (int j = 0; j < 4; j++) a[j] = egress ? h.b32(38 + 4 * j) : h.b32(22 + 4 * j); // (constant offsets: h stays in registers)
            prio_set = false;
            key = v6_owner(v6, lens, a, &owner) ? qos_bucket_one(bs, t, owner, len, egress != 0, &prio, &prio_set) : NO_KEY;
        } else {
            key = qos_classify_one(c, bs, t, h, len, dlen, egress != 0, &prio, &prio_set);
        }
        if (prio_set && b.priority) b.priority[i] = prio;
        b.verdict[i] = TC_OK;
        skey[i] = key == NO_KEY ? NO_KEY : key_pack(key, len, b.kshift);
        sval[i] = i;
    }
    bstats_flush(bs, c.stats);
}

// ---------------------------------------------------------------------------
// nat44_ingress, nat44_hairpin_xdp
// ---------------------------------------------------------------------------
// Header in registers, whole-sector probes (nat_reverse slot = key + original tuple in one 32-byte load,
// nat_sessions sector 0 = key + translation + last_seen), the TCP state CAS only when the state would
// change, the rewrite stored back as whole sectors.  Frames with IPv4 options take nat_ingress_one().
// ICMPERR (bng_nat_icmp_errors_enable): an ICMP error frame is keyed by the flow it quotes, not by bytes 4-5 of its
// ICMP header; it takes nat_icmp_error_one() on its own lane (errors are rare).
template <bool ICMPERR>
__global__ void __launch_bounds__(BLOCK) k_nat_ingress(const __grid_constant__ DevCtx c, const __grid_constant__ DevBatch b) {
    __shared__ BlockStats bs;
    bstats_init(bs);
    const u32 lane = threadIdx.x & 31;
    u32 n_dnat = 0, n_passed = 0;
    for (u32 base = blockIdx.x * BLOCK + (threadIdx.x & ~31u); base < b.n; base += gridDim.x * BLOCK) {
        const u32 i = base + lane;
        const bool act = i < b.n;
        const u32 len = act ? b.len[i] : 0;
        const u32 dlen = frame_dlen(b, len);
        u8 *p = act ? frame_ptr(b, i) : b.pkts;
        const bool wide = __all_sync(0xffffffffu, !act || FRAME_WIDE_OK(b, p));
        Hdr64 h;
        hdr_load_wide(h, p, dlen, wide);
        if (act) b.verdict[i] = TC_OK; // nat44_ingress never drops
        const bool ip4 = dlen >= 34 && h.b16(12) == ETH_P_IP_LE;
        if (ip4 && (h.b8(14) & 0x0f) != 5) { // options: fields are not at fixed offsets (rare)
            nat_ingress_one<ICMPERR>(c, bs, p, len, dlen, frame_now(b, i), b.nowv != nullptr);
            continue;
        }
        if (ICMPERR && ip4 && h.b8(23) == 1 && dlen >= 42 && icmp_error_type(h.b8(34))) {
            if (nat_icmp_error_one(c, p, h, dlen))
                n_dnat++;
            else
                n_passed++;
            continue;
        }
        const u32 saddr = h.b32(26), daddr = h.b32(30), proto = h.b8(23);
        u16 sport = 0, dport = 0;
        bool go = ip4;
        if (proto == 6) {
            go = go && dlen >= 54;
            sport = h.b16(34), dport = h.b16(36);
        } else if (proto == 17) {
            go = go && dlen >= 42;
            sport = h.b16(34), dport = h.b16(36);
        } else if (proto == 1) {
            go = go && dlen >= 42;
            dport = h.b16(38); // the echo id is the "destination port" of a reply (bpf/nat44.c:845-848)
        } else {
            go = false;
        }
        u64 rk[2];
        rk[0] = (u64)saddr | ((u64)daddr << 32);
        rk[1] = (u64)sport | ((u64)dport << 16) | ((u64)proto << 32);
        // ---- nat_reverse: 32-byte slot = key, then the original tuple ----
        u64 ok[2] = {0, 0};
        bool have = false;
        if (go && rk[0] < K_BUSY) {
            const u8 *s0 = tbl_slot(c.reverse, tbl_hash<2>(rk) & c.reverse.mask);
            U256 r = ldg256(s0);
            const u64 w0 = (u64)r.w[0] | ((u64)r.w[1] << 32), w1 = (u64)r.w[2] | ((u64)r.w[3] << 32);
            if (w0 == rk[0] && w1 == rk[1]) {
                have = true;
            } else if (w0 != K_EMPTY) { // collision: the general probe loop
                const u8 *rs = tbl_find<2, true>(c.reverse, rk);
                if (rs) {
                    r = ldg256(rs);
                    have = true;
                }
            }
            ok[0] = (u64)r.w[4] | ((u64)r.w[5] << 32);
            ok[1] = (u64)r.w[6] | ((u64)r.w[7] << 32);
        }
        if (go && !have) n_passed++; // no mapping: to the stack untouched (:861-867)
        // ---- nat_sessions: sector 0 (key, epoch) and sector 1 (last_seen, orig_ip, state, orig_port, in counters),
        //      requested together: one round trip, not two ----
        u8 *ses = nullptr;
        u32 seen = 0;
        U256 s1; // w[2] orig_ip, w[3] state word, w[4] orig_port
#pragma unroll
        for (int k = 0; k < 8; k++) s1.w[k] = 0;
        if (have && ok[0] < K_BUSY) {
            u8 *s0 = tbl_slot(c.sessions, tbl_hash<2>(ok) & c.sessions.mask);
            const U256 s = ldg256(s0);
            s1 = ldg256(s0 + 32);
            const u64 w0 = (u64)s.w[0] | ((u64)s.w[1] << 32), w1 = (u64)s.w[2] | ((u64)s.w[3] << 32);
            seen = s.w[5] >> 16;
            if (w0 == ok[0] && w1 == ok[1]) {
                ses = s0;
            } else if (w0 != K_EMPTY) {
                ses = tbl_find<2, false>(c.sessions, ok);
                if (ses) {
                    seen = *(const u16 *)(ses + SES_EPOCH);
                    s1 = ldg256(ses + 32);
                }
            }
        }
        if (have && !ses) { // stale reverse entry: one frame deletes it (sessions_expired), the others miss (:871-876)
            if (tbl_erase<2>(c.reverse, rk))
                bstats_add(bs, ST_NAT_EXPIRED, 1);
            else
                n_passed++;
        }
        if (ses) {
            ses_touch(ses, frame_now(b, i), seen, c.epoch, b.nowv != nullptr);
            ses_count(ses, SES_IN_LO, len);
            if (proto == 6) { // :885-895; CLOSING(3) is absorbing, NEW(0) -> ESTABLISHED(1) on ack
                const u32 tf = h.b8(47);
                const bool finrst = (tf & 0x05) != 0, ack = (tf & 0x10) != 0;
                u32 cur = s1.w[3];
                while (finrst || ack) {
                    const u32 st = cur & 0xff, nst = finrst ? 3u : (st == 0 ? 1u : st);
                    if (nst == st) break;
                    const u32 prev = atomicCAS((u32 *)(ses + SES_STATE), cur, (cur & ~0xffu) | nst);
                    if (prev == cur) break;
                    cur = prev;
                }
            }
            const u32 new_ip = s1.w[2];
            const u16 new_port = (u16)s1.w[4]; // orig_port
            h.s32(30, new_ip);
            h.s16(24, csum_upd32(h.b16(24), daddr, new_ip));
            if (proto == 6) {
                h.s16(36, new_port);
                u16 ck = csum_upd32(h.b16(50), daddr, new_ip);
                h.s16(50, csum_upd16(ck, dport, new_port));
            } else if (proto == 17) {
                h.s16(36, new_port);
                u16 ck = h.b16(40);
                if (ck != 0) {
                    ck = csum_upd32(ck, daddr, new_ip);
                    ck = csum_upd16(ck, dport, new_port);
                    if (ck == 0) ck = 0xffff;
                    h.s16(40, ck);
                }
            } else {
                h.s16(38, new_port);
                h.s16(36, csum_upd16(h.b16(36), dport, new_port));
            }
            if (wide) {
                stg256(p, &h.w[0]);
                if (proto == 6)
                    stg256(p + 32, &h.w[8]);
                else
                    hdr_store_chunk(h, p, 2);
            } else {
                hdr_store_chunk(h, p, 1);
                hdr_store_chunk(h, p, 2);
                if (proto == 6) hdr_store_chunk(h, p, 3);
            }
            n_dnat++;
        }
    }
    __syncwarp();
    warp_stat_flush(bs, ST_NAT_DNAT, n_dnat);
    warp_stat_flush(bs, ST_NAT_PASSED, n_passed);
    bstats_flush(bs, c.stats);
}

// bpf/nat44.c:951-991: statistics only, always XDP_PASS (2).
__global__ void __launch_bounds__(BLOCK) k_nat_hairpin_xdp(const __grid_constant__ DevCtx c, const __grid_constant__ DevBatch b) {
    __shared__ BlockStats bs;
    bstats_init(bs);
    u32 flags = *(const u32 *)c.nat_config;
    for (u32 i = blockIdx.x * BLOCK + threadIdx.x; i < b.n; i += gridDim.x * BLOCK) {
        b.verdict[i] = 2;
        if (!(flags & NATF_HAIRPIN)) continue;
        u32 len = frame_dlen(b, b.len[i]);
        const u8 *p = frame_ptr(b, i);
        if (len < 14 || rd16(p, 12) != ETH_P_IP_LE || len < 34) continue;
        if (!is_private_ip(rd32(p, 26))) continue;
        u64 hk = rd32(p, 30);
        if (tbl_find<1, false>(c.hairpin, &hk)) bstats_add(bs, ST_NAT_HAIRPIN, 1);
    }
    bstats_flush(bs, c.stats);
}

#include "pipe_classify.cuh"

// ---------------------------------------------------------------------------
// GROUP: stable LSD radix sort with compaction and device-side counts.
// Pass 0 reads n (host-known) keys and skips NO_KEY entries; later passes
// read *cnt[CNT_M] elements.  Every block owns one contiguous range of the
// input, so (digit, block) order of the scanned histogram is index order.
// ---------------------------------------------------------------------------
#define RS_BLOCKS_PER_SM 3 // what the scatter's 71 registers x 256 threads lets an SM hold: one wave, whole tiles
#define RS_HIST_VEC 4      // 16-byte key loads in flight per thread in k_rs_hist

__device__ __forceinline__ void rs_range(u32 total, u32 &lo, u32 &hi) {
    u32 per = (total + gridDim.x - 1) / gridDim.x;
    per = (per + BLOCK - 1) / BLOCK * BLOCK;
    u64 l = (u64)blockIdx.x * per, r = l + per;
    lo = l < total ? (u32)l : total;
    hi = r < total ? (u32)r : total;
}

__global__ void __launch_bounds__(BLOCK) k_rs_hist(const u32 *keys, u32 n_host, u32 *cnt, int first, int shift, u32 *H, u32 *T,
                                                   u32 *anyv, u32 kmask) {
    __shared__ u32 h[256];
    __shared__ u32 smax;
    pdl_wait();
    if (!rs_pass_needed(cnt, shift)) return; // every key has a zero digit here: the pass would be the identity
    h[threadIdx.x] = 0;
    if (threadIdx.x == 0) smax = 0;
    __syncthreads();
    u32 mymax = 0;
    u32 total = first ? n_host : cnt[CNT_M];
    u32 lo, hi;
    rs_range(total, lo, hi);
    // RS_HIST_VEC 16-byte loads per thread are issued before any of their keys is counted: one 4-byte load at a
    // time leaves the pass latency-bound (lo is a multiple of BLOCK, so every vector is aligned)
    for (u32 i0 = lo + threadIdx.x * 4; i0 < hi; i0 += BLOCK * 4 * RS_HIST_VEC) {
        uint4 v[RS_HIST_VEC];
#pragma unroll
        for (int u = 0; u < RS_HIST_VEC; u++) {
            const u32 i = i0 + u * BLOCK * 4;
            if (i + 3 < hi) {
                v[u] = *(const uint4 *)(keys + i);
            } else {
                v[u].x = i < hi ? keys[i] : NO_KEY;
                v[u].y = i + 1 < hi ? keys[i + 1] : NO_KEY;
                v[u].z = i + 2 < hi ? keys[i + 2] : NO_KEY;
                v[u].w = NO_KEY;
            }
        }
#pragma unroll
        for (int u = 0; u < 4 * RS_HIST_VEC; u++) {
            const uint4 &q = v[u / 4];
            u32 k = (u & 3) == 0 ? q.x : (u & 3) == 1 ? q.y : (u & 3) == 2 ? q.z : q.w;
            if (k != NO_KEY) {
                k &= kmask; // (the bits above the key carry the frame length: DevBatch.kshift)
                atomicAdd(&h[(k >> shift) & 0xff], 1u);
                mymax = k > mymax ? k : mymax;
            }
        }
    }
    __syncthreads();
    if (first) {
        int any = __syncthreads_or(mymax != 0 || h[0] != 0); // a block of NO_KEYs only has nothing to scatter
        if (threadIdx.x == 0) anyv[blockIdx.x] = (u32)any;
        mymax = __reduce_max_sync(0xffffffffu, mymax);
        if ((threadIdx.x & 31) == 0 && mymax) atomicMax(&smax, mymax);
        __syncthreads();
        if (threadIdx.x == 0 && smax) atomicMax(&cnt[CNT_MAXKEY], smax);
    }
    u32 v = h[threadIdx.x];
    H[threadIdx.x * gridDim.x + blockIdx.x] = v;
    if (v) atomicAdd(&T[threadIdx.x], v); // per-digit totals over all blocks
}

// Exclusive scan of the 256 x nblocks histogram in (digit, block) order.  One block per digit:
// base = total of the smaller digits (from T), then a block-wide scan of the digit's row.
__global__ void __launch_bounds__(1024) k_rs_scan(u32 *H, const u32 *T, u32 nblocks, u32 *cnt, int first, int shift) {
    __shared__ u32 wsum[32];
    __shared__ u32 s_base;
    pdl_wait();
    if (!rs_pass_needed(cnt, shift)) return;
    const u32 d = blockIdx.x, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    u32 t = (threadIdx.x < 256 && threadIdx.x < d) ? T[threadIdx.x] : 0; // digits below d
    t = __reduce_add_sync(0xffffffffu, t);
    if (lane == 0) wsum[w] = t;
    __syncthreads();
    if (threadIdx.x == 0) {
        u32 b = 0;
        for (int i = 0; i < 8; i++) b += wsum[i];
        s_base = b;
    }
    __syncthreads();
    u32 v = threadIdx.x < nblocks ? H[d * nblocks + threadIdx.x] : 0;
    u32 inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        u32 n = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= (u32)o) inc += n;
    }
    __syncthreads();
    if (lane == 31) wsum[w] = inc;
    __syncthreads();
    if (w == 0) {
        u32 x = wsum[lane], xi = x;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            u32 n = __shfl_up_sync(0xffffffffu, xi, o);
            if (lane >= (u32)o) xi += n;
        }
        wsum[lane] = xi - x; // exclusive warp offsets
    }
    __syncthreads();
    if (threadIdx.x < nblocks) H[d * nblocks + threadIdx.x] = s_base + wsum[w] + inc - v;
    if (first && d == 255 && threadIdx.x == 1023) cnt[CNT_M] = s_base + wsum[31] + inc; // = number of valid keys
}

// Stable scatter of one radix pass.  A tile is 8 warps x RS_ROWS x 32 elements; warp w owns the
// contiguous elements [w * RS_ROWS * 32, (w + 1) * RS_ROWS * 32) of the tile and walks them row by row,
// so index order is (warp, row, lane).  Ranks inside a row come from one ballot per digit bit, ranks across
// the rows of a warp from a warp-private running histogram in shared memory; thread d then turns the
// 8 per-warp totals of digit d into tile-local offsets.  The tile is reordered by digit in shared
// memory and written out from there, so that a warp's store covers runs of consecutive addresses
// (one run per digit) instead of 32 scattered words.
#define RS_ROWS 8
#define RS_TILE (RS_ROWS * BLOCK)
#define RS_WARPS (BLOCK / 32)
__global__ void __launch_bounds__(BLOCK) k_rs_scatter(const u32 *keys, const u32 *vals, u32 *okeys, u32 *ovals, u32 n_host,
                                                      const u32 *cnt, int first, int shift, const u32 *H, const u32 *anyv, u32 kmask) {
    __shared__ u16 wh[RS_WARPS][256]; // per-warp digit counts, then the warp's offset inside the digit's run
    __shared__ u32 stage_k[RS_TILE], stage_v[RS_TILE];
    __shared__ u32 tstart[256]; // tile-local start of digit d
    __shared__ u32 gdelta[256]; // global position of a staged element = gdelta[digit] + its tile-local position
    __shared__ u32 wsum[RS_WARPS];
    __shared__ u32 tile_n;
    pdl_wait();
    if (!rs_pass_needed(cnt, shift)) return;
    if (first && !anyv[blockIdx.x]) return; // nothing but NO_KEY in this block's range
    u32 goff = H[threadIdx.x * gridDim.x + blockIdx.x]; // thread d owns the running global offset of digit d
    u32 total = first ? n_host : cnt[CNT_M];
    u32 lo, hi;
    rs_range(total, lo, hi);
    const u32 lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const u32 toff = w * (RS_ROWS * 32) + lane; // + r * 32
    u32 nk[RS_ROWS], nv[RS_ROWS]; // next tile, fetched while the current one goes through shared memory
#pragma unroll
    for (int r = 0; r < RS_ROWS; r++) {
        u32 i = lo + toff + r * 32;
        nk[r] = NO_KEY;
        nv[r] = 0;
        if (i < hi) {
            nk[r] = keys[i];
            nv[r] = vals[i];
        }
    }
    for (u32 base = lo; base < hi; base += RS_TILE) {
        u32 k[RS_ROWS], v[RS_ROWS], rank[RS_ROWS];
#pragma unroll
        for (int r = 0; r < RS_ROWS; r++) {
            k[r] = nk[r];
            v[r] = nv[r];
            u32 i = base + RS_TILE + toff + r * 32;
            nk[r] = NO_KEY;
            nv[r] = 0;
            if (i < hi) {
                nk[r] = keys[i];
                nv[r] = vals[i];
            }
        }
#pragma unroll
        for (int j = 0; j < 256 / 32; j++) wh[w][j * 32 + lane] = 0;
        __syncwarp();
#pragma unroll
        for (int r = 0; r < RS_ROWS; r++) {
            const bool ok = k[r] != NO_KEY;
            const u32 d = ok ? (((k[r] & kmask) >> shift) & 0xff) : 0;
            // the valid lanes with the same digit: one ballot per digit bit (cheaper than match.any)
            u32 peers = __ballot_sync(0xffffffffu, ok);
#pragma unroll
            for (int bit = 0; bit < 8; bit++) {
                const bool one = (d >> bit) & 1;
                const u32 ones = __ballot_sync(0xffffffffu, one);
                peers &= one ? ones : ~ones;
            }
            u32 before = ok ? wh[w][d] : 0; // elements of digit d in the earlier rows of this warp
            u32 rk = __popc(peers & ((1u << lane) - 1));
            __syncwarp();
            if (ok && rk == 0) wh[w][d] = (u16)(before + __popc(peers));
            __syncwarp();
            rank[r] = before + rk;
        }
        __syncthreads();
        { // thread d: exclusive offsets of digit d over the warps; then the block-wide exclusive scan of
          // the per-digit totals gives each digit's start inside the tile
            u32 run = 0;
#pragma unroll
            for (int j = 0; j < RS_WARPS; j++) {
                u32 t = wh[j][threadIdx.x];
                wh[j][threadIdx.x] = (u16)run;
                run += t;
            }
            u32 inc = run;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                u32 x = __shfl_up_sync(0xffffffffu, inc, o);
                if (lane >= (u32)o) inc += x;
            }
            if (lane == 31) wsum[w] = inc;
            __syncthreads();
            u32 pre = 0;
#pragma unroll
            for (int j = 0; j < RS_WARPS; j++) pre += j < (int)w ? wsum[j] : 0;
            u32 ts = pre + inc - run;
            tstart[threadIdx.x] = ts;
            gdelta[threadIdx.x] = goff - ts;
            goff += run;
            if (threadIdx.x == BLOCK - 1) tile_n = ts + run;
        }
        __syncthreads();
#pragma unroll
        for (int r = 0; r < RS_ROWS; r++) {
            if (k[r] != NO_KEY) {
                u32 d = ((k[r] & kmask) >> shift) & 0xff;
                u32 lp = tstart[d] + wh[w][d] + rank[r];
                stage_k[lp] = k[r];
                stage_v[lp] = v[r];
            }
        }
        __syncthreads();
        const u32 tn = tile_n;
        for (u32 j = threadIdx.x; j < tn; j += BLOCK) {
            u32 kk = stage_k[j];
            u32 g = gdelta[((kk & kmask) >> shift) & 0xff] + j;
            okeys[g] = kk;
            ovals[g] = stage_v[j];
        }
        __syncthreads();
    }
}

// group heads: positions where the sorted key changes (any order; groups are independent).
// 16 keys per thread and trip (four 128-bit loads in flight), one atomic per warp for the heads its lanes found.
__global__ void __launch_bounds__(BLOCK) k_heads(const __grid_constant__ Grouped g, u32 *seg, u32 *cnt) {
    const u32 *skey, *sval_unused;
    pdl_wait();
    grouped_select(g, cnt, skey, sval_unused);
    const u32 m = cnt[CNT_M];
    const u32 kmask = key_mask_of(g.kshift);
    const u32 lane = threadIdx.x & 31;
    for (u32 wbase = 16 * (blockIdx.x * BLOCK + (threadIdx.x & ~31u)); wbase < m; wbase += 16 * gridDim.x * BLOCK) { // warp-uniform
        const u32 j = wbase + 16 * lane;
        u32 k[16];
        u32 prev = 0;
        if (j < m) prev = j ? skey[j - 1] & kmask : ~(skey[0] & kmask);
        if (j + 15 < m) {
#pragma unroll
            for (int q = 0; q < 4; q++) {
                const uint4 v = *(const uint4 *)(skey + j + 4 * q);
                k[4 * q] = v.x, k[4 * q + 1] = v.y, k[4 * q + 2] = v.z, k[4 * q + 3] = v.w;
            }
        } else {
#pragma unroll
            for (int t = 0; t < 16; t++) k[t] = j + t < m ? skey[j + t] : 0;
        }
        u32 hm = 0;
#pragma unroll
        for (int t = 0; t < 16; t++) {
            const u32 kk = k[t] & kmask;
            if (j + t < m && kk != prev) hm |= 1u << t;
            prev = kk;
        }
        const u32 mine = __popc(hm);
        u32 inc = mine;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const u32 x = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= (u32)o) inc += x;
        }
        const u32 total = __shfl_sync(0xffffffffu, inc, 31);
        if (!total) continue;
        u32 basepos = 0;
        if (lane == 31) basepos = atomicAdd(&cnt[CNT_NSEG], total);
        basepos = __shfl_sync(0xffffffffu, basepos, 31) + inc - mine;
        while (hm) {
            const u32 t = __ffs(hm) - 1;
            hm &= hm - 1;
            seg[basepos++] = j + t;
        }
    }
}

// ---------------------------------------------------------------------------
// RESOLVE: one block of RS_TEAM threads per group, frames in index order.  The block is a single warp:
// concurrency across groups hides more latency than parallelism inside one.
//   stage   all threads copy the group's (value, length) pairs into shared memory, RS_STAGE frames per
//           sweep, with coalesced loads: the length comes out of the key word (DevBatch.kshift), so nothing
//           depends on the frame index just loaded (a fat group — 3 000 frames per subscriber when 10 k
//           subscribers are sharded over 8 GPUs — used to be ~50 serial round trips of one warp).
//   NAT     warp 0 creates the new flows (MISS_FLAG) chunk by chunk, warp-cooperatively when the chunk's
//           flows provably do not interact (nat_chunk_coop), else one lane at a time in index order.
//   QOS     warp 0 applies token_bucket_check() to the staged lengths with warp-uniform fast paths
//           (whole chunk fits / nothing fits / lane-by-lane), out of shared memory.
//   write   all threads publish verdicts / priorities and count.
// The group key is the subscriber-directory slot (programs with a NAT stage) or the bucket's own slot.
// ---------------------------------------------------------------------------
#define DROP_FLAG 0x40000000u // staged value: nat44_egress dropped the frame (port exhaustion): no QoS stage
#define RS_TEAM 32
#define RS_PER_THREAD 8

// The NAT stage of one 32-frame chunk that holds new flows (mm: their lanes), kept out of line: the steady state
// never calls it, and its registers (the frame header, three table probes, the translation) must not cost the
// staging loop and the token-bucket walk theirs.  Returns true for a frame nat44_egress dropped (port exhaustion).
// The sequential nat44_egress of one frame, out of line (rare; keeps its registers and code out of the walk).
// ICMPERR: an ICMP error frame (outer ihl 5) first meets the rule of bng_nat_icmp_errors_egress_enable, which
// translates it by the flow it quotes; where that does not apply, nat44_egress as always.  `fresh` (a frame the token
// bucket deferred): the parse's hairpin statistic is still to be counted.
template <bool ICMPERR>
static __device__ __noinline__ int nat_egress_seq(const DevCtx &c, BlockStats &bs, const DevBatch &b, u8 *sub, u32 idx, u32 len, NatPend *pend,
                                                 bool fresh) {
    if (ICMPERR) {
        u8 *p = frame_ptr(b, idx);
        const u32 dlen = frame_dlen(b, len);
        if (icmp_error_frame(p, dlen) && nat_icmp_error_egress_one(c, p, dlen)) {
            if (fresh && (*(const u32 *)c.nat_config & NATF_HAIRPIN)) {
                u64 hk = rd32(p, 30);
                if (tbl_find<1, false>(c.hairpin, &hk)) bstats_add(bs, ST_NAT_HAIRPIN, 1);
            }
            bstats_add(bs, ST_NAT_SNAT, 1);
            return TC_OK;
        }
    }
    NatOut o = nat_egress_one<true>(c, bs, frame_ptr(b, idx), sub, len, frame_dlen(b, len), idx + b.base, frame_now(b, idx), pend, fresh,
                                    b.nowv != nullptr);
    return o.verdict;
}

// ICMPERR: an ICMP error frame ends nat_chunk_coop's prefix and goes through nat_egress_seq<true>() in its turn.
template <bool ICMPERR>
__device__ __forceinline__ bool resolve_nat_chunk(const DevCtx &c, const DevBatch &b, BlockStats &bs, u8 *sub, u32 idx, u32 len,
                                                      bool is_miss, bool fresh, u32 mm, u32 lane) {
    NatPend pend;
    // one nat_log_rb reservation for all new flows of this chunk that classify found (every one of them logs at most
    // one record; a slot left unused is tagged invalid for the drain).  A deferred TC frame has not been looked up
    // yet and is most often a session hit: it reserves its record when it writes one, so hits cost no staging space.
    const EvRing &r = c.natlog_ev;
    const u32 pre = __ballot_sync(0xffffffffu, is_miss && !fresh);
    u32 nrec = __popc(pre), basepos = 0;
    if (nrec) {
        if (lane == 0) basepos = atomicAdd(r.count, nrec);
        basepos = __shfl_sync(0xffffffffu, basepos, 0);
        if (lane == 0 && basepos + nrec > r.cap) { // staging ring full: the tail of the chunk has no slot
            u32 over = basepos >= r.cap ? nrec : basepos + nrec - r.cap;
            atomicSub(r.count, over);
            atomicAdd(&c.stats[r.lost_stat], (u64)over);
        }
    }
    const u32 rpos = basepos + __popc(pre & ((1u << lane) - 1));
    pend.log_rec = (is_miss && !fresh && rpos < r.cap) ? r.buf + (size_t)rpos * r.rec_bytes : nullptr;
    pend.logged = false;
    pend.lazy = fresh;
    if (pend.log_rec) *(uint2 *)(pend.log_rec + r.rec_bytes - 8) = make_uint2(idx + b.base, c.batch_seq);
    bool dropped = false;
    u32 todo = mm;
    while (todo) {
        // the longest prefix of the remaining new flows that does not interact: all at once
        const u32 took = nat_chunk_coop<ICMPERR>(c, bs, b, sub, is_miss && ((todo >> lane) & 1), idx, len, pend, lane, fresh);
        todo &= ~took;
        if (lane == 0 && took) bstats_add(bs, ST_NAT_COOP, __popc(took));
        if (!todo) break;
        const u32 l = __ffs(todo) - 1; // ... then the frame that does, through the sequential code
        todo &= todo - 1;
        if (lane == l) {
            if (nat_egress_seq<ICMPERR>(c, bs, b, sub, idx, len, &pend, fresh) == TC_SHOT) {
                b.verdict[idx] = TC_SHOT;
                dropped = true;
            }
            bstats_add(bs, ST_NAT_SEQ, 1);
        }
        __syncwarp();
    }
    if (is_miss && !pend.logged && pend.log_rec) // e.g. the session was created earlier in this batch
        *(uint2 *)(pend.log_rec + r.rec_bytes - 8) = make_uint2(0xFFFFFFFFu, c.batch_seq);
    return dropped;
}

// TC (pipeline_tc): the token bucket runs BEFORE the NAT stage: QoS walk first, then nat44_egress — hits and
// new flows alike — for the frames it passed (DEFER_FLAG), with the parse-stage counters still to be counted.
// ICMPERR (bng_nat_icmp_errors_egress_enable): an ICMP error frame in the NAT stage is looked up by the flow it quotes
// first (resolve_nat_chunk).
template <bool NAT, bool QOS, bool EGRESS, bool TC = false, bool ICMPERR = false>
__global__ void __launch_bounds__(RS_TEAM, 16) k_resolve(const __grid_constant__ DevCtx c, const __grid_constant__ DevBatch b,
                                                      const __grid_constant__ Grouped g, const u32 *seg, u32 *cnt) {
    constexpr int STAGE = RS_TEAM * RS_PER_THREAD;
    __shared__ BlockStats bs;
    __shared__ u32 s_sv[STAGE], s_len[STAGE];
    __shared__ u32 s_cnt, s_next;
    bstats_init(bs);
    pdl_wait();
    const u32 *skey, *sval;
    grouped_select(g, cnt, skey, sval);
    const Tbl &qt = EGRESS ? c.qos_eg : c.qos_in;
    const u32 tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const u32 m = cnt[CNT_M], nseg = cnt[CNT_NSEG];
    const u32 kmask = key_mask_of(g.kshift);
    u32 pp = 0, dp = 0; // per-thread partial QoS counters
    u64 pb = 0, db = 0;
    // groups are handed out dynamically (fat and thin groups mix: a static stride leaves blocks idle at the end)
    for (;;) {
        if (tid == 0) s_next = atomicAdd(&cnt[CNT_WORK], 1u);
        __syncthreads();
        const u32 s = s_next;
        if (s >= nseg) break;
        const u32 start = seg[s];
        const u32 key = skey[start] & kmask;
        u8 *sub = nullptr, *slot = nullptr;
        if (NAT) {
            const u64 w = *(const u64 *)(c.subdir.slots + (size_t)key * 16 + 8);
            const u32 ns = (u32)w, qs = (u32)(w >> 32);
            if (ns != DIR_NONE) sub = tbl_slot(c.sub_nat, ns);
            if (QOS && qs != DIR_NONE) slot = tbl_slot(qt, qs & DIR_SLOT_MASK);
        } else {
            slot = tbl_slot(qt, key);
        }
        TokenBucket tb;
        if (QOS && slot) tb_load(tb, slot);
        for (u32 pos = start;; pos += STAGE) {
            // ---- stage ----
            if (tid == 0) s_cnt = STAGE;
            __syncthreads();
            {
                u32 kk[RS_PER_THREAD], sv[RS_PER_THREAD];
                bool ok[RS_PER_THREAD];
#pragma unroll
                for (int t = 0; t < RS_PER_THREAD; t++) {
                    const u32 q = pos + t * RS_TEAM + tid;
                    kk[t] = q < m ? skey[q] : 0;
                    sv[t] = q < m ? sval[q] : 0;
                    ok[t] = q < m && (kk[t] & kmask) == key;
                }
                u32 first_bad = STAGE;
#pragma unroll
                for (int t = 0; t < RS_PER_THREAD; t++) {
                    const u32 j = t * RS_TEAM + tid;
                    if (ok[t]) {
                        // the length came with the key (DevBatch.kshift); a jumbo frame's, or any when the key space
                        // leaves no room, is looked up
                        u32 l = g.kshift ? kk[t] >> g.kshift : KEY_LEN_SAT;
                        if (l == KEY_LEN_SAT) l = b.len[sv[t] & IDX_MASK];
                        s_sv[j] = sv[t];
                        s_len[j] = l;
                    } else if (j < first_bad) {
                        first_bad = j;
                    }
                }
                if (first_bad < STAGE) atomicMin(&s_cnt, first_bad); // keys are sorted: the valid positions are a prefix
            }
            __syncthreads();
            const u32 n_here = s_cnt;
            const u32 nchunk = (n_here + 31) / 32;
            // a fat group: the next sweep's two cache-line runs are requested now (into L1, no registers held) and
            // arrive while this sweep is walked
            if (n_here == (u32)STAGE && tid < 2 * (STAGE * 4 / 128)) {
                const u32 *base = tid < STAGE / 32 ? skey : sval;
                const u32 q = pos + STAGE + (tid % (STAGE / 32)) * 32;
                if (q < m) asm volatile("prefetch.global.L1 [%0];" ::"l"(base + q));
            }
            // ---- NAT stage of this subscriber's frames, strictly in index order: new flows (MISS_FLAG) and, in TC
            //      order, every frame that waited for the token bucket (DEFER_FLAG) and was not dropped by it ----
            auto nat_phase = [&]() {
              if (warp == 0) {
                for (u32 cb = 0; cb < nchunk; cb++) {
                    const u32 j = cb * 32 + lane;
                    const bool valid = j < n_here;
                    const u32 sv = valid ? s_sv[j] : 0;
                    bool is_miss = valid && (sv & MISS_FLAG);
                    bool fresh = false; // a deferred frame: the whole of nat44_egress is still to run
                    if (TC && valid && (sv & DEFER_FLAG) && !(sv & DROP_FLAG)) {
                        // :583-596 for a frame nobody has looked at yet: private source? allocation?
                        const u8 *fp = frame_ptr(b, sv & IDX_MASK);
                        if (is_private_ip(rd32(fp, 26))) {
                            if (sub)
                                is_miss = fresh = true;
                            else
                                bstats_add(bs, ST_NAT_PASSED, 1);
                        }
                    }
                    const u32 mm = __ballot_sync(0xffffffffu, is_miss);
                    if (!mm) continue; // (the steady state: nothing to create, the call below never happens)
                    if (resolve_nat_chunk<ICMPERR>(c, b, bs, sub, sv & IDX_MASK, valid ? s_len[j] : 0, is_miss, fresh, mm, lane)) s_sv[j] = sv | DROP_FLAG;
                }
              }
            };
            if (NAT && !TC && sub) nat_phase();
            if (NAT && QOS) __syncthreads();
            // ---- token bucket over the staged lengths; verdicts, priorities and statistics as the walk goes ----
            if (QOS && slot && warp == 0) {
                for (u32 cb = 0; cb < nchunk; cb++) {
                    const u32 j = cb * 32 + lane;
                    const u32 sv = j < n_here ? s_sv[j] : DROP_FLAG;
                    const bool elig = !(sv & DROP_FLAG);
                    const u32 len = elig ? s_len[j] : 0;
                    u32 em = __ballot_sync(0xffffffffu, elig);
                    if (!em) continue;
                    bool pass = true;
                    if (tb.rate_bps != 0 && b.nowv) {
                        // a clock value per frame: token_bucket_check() frame by frame, refill included (:80-94)
                        const u64 mynow = elig ? b.nowv[sv & IDX_MASK] : 0;
                        pass = false;
                        while (em) {
                            const u32 l = __ffs(em) - 1;
                            em &= em - 1;
                            const u32 ll = __shfl_sync(0xffffffffu, len, l);
                            const u64 tn = __shfl_sync(0xffffffffu, mynow, l);
                            const bool ok = tb_step(tb, tn, ll);
                            if (lane == l) pass = ok;
                        }
                    } else if (tb.rate_bps != 0) { // rate 0: unlimited, bucket untouched (bpf/qos_ratelimit.c:77-78)
                        tb_refill(tb, b.now);
                        const u32 tot = __reduce_add_sync(0xffffffffu, len);
                        const u32 mn = __reduce_min_sync(0xffffffffu, elig ? len : 0xffffffffu);
                        if (tb.tokens >= (u64)tot) { // the whole chunk fits
                            tb.tokens -= tot;
                        } else if (tb.tokens < (u64)mn) { // nothing in the chunk fits
                            pass = false;
                        } else { // mixed: frame by frame, uniform across the warp
                            pass = false;
                            while (em) {
                                const u32 l = __ffs(em) - 1;
                                em &= em - 1;
                                const u32 ll = __shfl_sync(0xffffffffu, len, l);
                                const bool ok = tb.tokens >= (u64)ll;
                                if (ok) tb.tokens -= ll;
                                if (lane == l) pass = ok;
                            }
                        }
                    }
                    if (elig) {
                        const u32 idx = sv & IDX_MASK;
                        if (pass) {
                            pp++;
                            pb += len;
                            if (EGRESS && b.priority) b.priority[idx] = tb.prio;
                        } else {
                            dp++;
                            db += len;
                            b.verdict[idx] = TC_SHOT;
                            if (TC) s_sv[j] = sv | DROP_FLAG; // never reaches the NAT stage
                        }
                    }
                }
            }
            if (NAT && TC) { // the frames the bucket dropped are marked; everything else goes through nat44_egress now
                __syncthreads();
                nat_phase();
            }
            if (n_here < (u32)STAGE) break; // the group ended inside this sweep
            __syncthreads();                // ... else the staging buffers are reused
        }
        if (QOS && slot && tid == 0) {
            *(u64 *)(slot + 16) = tb.tokens;
            *(u64 *)(slot + 24) = tb.last_update;
        }
        __syncthreads();
    }
    if (QOS) {
        warp_stat_flush(bs, ST_QOS_PASS_PKTS, pp);
        warp_stat_flush64(bs, ST_QOS_PASS_BYTES, pb);
        warp_stat_flush(bs, ST_QOS_DROP_PKTS, dp);
        warp_stat_flush64(bs, ST_QOS_DROP_BYTES, db);
    }
    bstats_flush(bs, c.stats);
}

// ---------------------------------------------------------------------------
// host-side launchers
// ---------------------------------------------------------------------------
static inline int grid_for(const Launcher &L, u32 n, int blocks_per_sm) {
    long want = ((long)n + BLOCK - 1) / BLOCK;
    long cap = (long)L.num_sms * blocks_per_sm;
    if (want < 1) want = 1;
    return (int)(want < cap ? want : cap);
}

static int bits_for(u64 max_key_exclusive) {
    int b = 1;
    while ((1ull << b) < max_key_exclusive) b++;
    return b;
}

static inline u32 *sort_T(Launcher &L) { return (u32 *)L.s.cub_tmp + 256 * 1024; } // per-pass digit totals (group_by_key)

size_t sort_temp_bytes(u32 n) { // histogram matrix: 256 digits x blocks
    (void)n;
    return (size_t)(256 * 1024 + 4 * 256 + 1024) * sizeof(u32); // H, per-pass digit totals, per-block "any key" flags
}

void prof_begin(Launcher &L, const char *name) {
    if (!L.prof || L.npend >= 32) return;
    int acc = -1;
    for (int i = 0; i < L.nacc; i++)
        if (L.acc_name[i] == name || !strcmp(L.acc_name[i], name)) acc = i;
    if (acc < 0) {
        if (L.nacc >= 32) return;
        acc = L.nacc++;
        L.acc_name[acc] = name;
        L.acc_ms[acc] = 0;
        L.acc_n[acc] = 0;
    }
    ProfPending &p = L.pend[L.npend];
    p.acc = acc;
    if (cudaEventCreate(&p.a) != cudaSuccess || cudaEventCreate(&p.b) != cudaSuccess) return;
    cudaEventRecord(p.a, L.stream);
    L.npend++;
    L.prof = 2; // a begin is open
}
void prof_end(Launcher &L) {
    if (L.prof != 2) return;
    cudaEventRecord(L.pend[L.npend - 1].b, L.stream);
    L.prof = 1;
}
void prof_collect(Launcher &L) {
    for (int i = 0; i < L.npend; i++) {
        float ms = 0;
        if (cudaEventElapsedTime(&ms, L.pend[i].a, L.pend[i].b) == cudaSuccess) {
            L.acc_ms[L.pend[i].acc] += ms;
            L.acc_n[L.pend[i].acc]++;
        }
        cudaEventDestroy(L.pend[i].a);
        cudaEventDestroy(L.pend[i].b);
    }
    L.npend = 0;
}

// Programmatic dependent launch for the kernels that FOLLOW the classify kernel of a batch (radix passes, group
// heads, resolve): the launch may be processed while its predecessor in the stream is still running — its blocks are
// set up early and wait in pdl_wait() (griddepcontrol.wait: returns once the preceding grid has completed and its
// memory operations are visible), which takes the launch latency out of the chain of eight dependent kernels that
// a small batch consists of.  Every kernel launched this way calls pdl_wait() before its first global access.
template <typename... KArgs, typename... Args>
static inline void launch_dep(void (*kern)(KArgs...), dim3 grid, dim3 block, cudaStream_t st, Args &&...args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = 0;
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    cudaLaunchKernelEx(&cfg, kern, KArgs(args)...);
}

// name: what the launch is timed as (bng_prof_enable)
#define LAUNCH_AS(name, kern, n, bps, ...)                              \
    do {                                                                \
        prof_begin(L, name);                                            \
        kern<<<grid_for(L, n, bps), BLOCK, 0, L.stream>>>(__VA_ARGS__); \
        prof_end(L);                                                    \
        L.launches++;                                                   \
    } while (0)
#define LAUNCH(kern, n, bps, ...) LAUNCH_AS(#kern, kern, n, bps, __VA_ARGS__)

// Groups the (key, value) pairs in (key_a, val_a)[0..n) by key, stably, skipping NO_KEY.
// On return *sk / *sv name the buffers holding the grouped pairs; counters[CNT_M] holds their
// number and seg[0..counters[CNT_NSEG]) the group heads.
static cudaError_t group_by_key(Launcher &L, u32 n, u64 key_space, u32 kshift, Grouped *out) {
    Scratch &s = L.s;
    int passes = (bits_for(key_space) + 7) / 8;
    int rsb = L.num_sms * RS_BLOCKS_PER_SM;
    if (rsb > 1024) rsb = 1024;
    u32 *H = (u32 *)s.cub_tmp, *T = H + 256 * 1024, *ANYV = T + 4 * 256;
    cudaError_t e = cudaSuccess; // (counters and T were cleared by the classify kernel: scratch_reset)
    u32 *ik = s.key_a, *iv = s.val_a, *ok = s.key_b, *ov = s.val_b;
    prof_begin(L, "group_by_key");
    for (int p = 0; p < passes; p++) {
        int first = p == 0;
        launch_dep(k_rs_hist, rsb, BLOCK, L.stream, ik, n, s.counters, first, 8 * p, H, T + 256 * p, ANYV, key_mask_of(kshift));
        launch_dep(k_rs_scan, 256, 1024, L.stream, H, T + 256 * p, (u32)rsb, s.counters, first, 8 * p);
        launch_dep(k_rs_scatter, rsb, BLOCK, L.stream, ik, iv, ok, ov, n, s.counters, first, 8 * p, H, ANYV, key_mask_of(kshift));
        L.launches += 3;
        u32 *t = ik;
        ik = ok;
        ok = t;
        t = iv;
        iv = ov;
        ov = t;
    }
    Grouped g;
    g.ka = s.key_a;
    g.va = s.val_a;
    g.kb = s.key_b;
    g.vb = s.val_b;
    g.passes = passes;
    g.kshift = kshift;
    *out = g;
    launch_dep(k_heads, grid_for(L, (n + 15) / 16, 4), BLOCK, L.stream, g, s.qslot, s.counters);
    L.launches++;
    prof_end(L);
    return cudaGetLastError();
}

// Room for the frame length above the ordering key?  (KEY_BITS covers the reference's capacities.)
static inline u32 kshift_for(u64 key_space) { return bits_for(key_space) <= KEY_BITS ? KEY_BITS : 0; }

static const char *tf(bool b) { return b ? "true" : "false"; }
static std::string resolve_name(bool nat, bool qos, bool egress, bool tc, bool icmperr) {
    return std::string("(k_resolve<") + tf(nat) + ", " + tf(qos) + ", " + tf(egress) + (tc ? ", tc" : "") + (icmperr ? ", icmperr" : "") + ">)";
}
// TC is printed when TC or ACCT is set, ACCT only when set, then a tag per optional stage
static std::string classify_name(bool as, bool qos, bool tc, bool acct, bool v6, bool as6, bool icmperr) {
    return std::string("(k_pipe_classify<") + tf(as) + ", " + tf(qos) + (tc || acct ? std::string(", ") + tf(tc) : "") +
           (acct ? ", true" : "") + (v6 ? ", v6" : "") + (as6 ? ", as6" : "") + (icmperr ? ", icmperr" : "") + ">)";
}
static std::string antispoof_name(bool v6) { return std::string("k_antispoof") + (v6 ? "<v6>" : ""); }
static std::string qos_name(bool v6) { return std::string("k_qos_classify") + (v6 ? "<v6>" : ""); }
static std::string nat_ingress_name(bool icmperr) { return std::string("k_nat_ingress") + (icmperr ? "<icmperr>" : ""); }

// k_resolve walks one group per block and a batch of n frames can hold n groups: the grid is sized for n blocks,
// capped at what the GPU holds at once (the blocks loop over the groups).
template <bool NAT, bool QOS, bool EGRESS, bool TC = false, bool ICMPERR = false>
static void launch_resolve(Launcher &L, const DevCtx &c, const DevBatch &b, const Grouped &g) {
    int &per_sm = L.resolve_bps[ICMPERR * 16 + NAT * 8 + QOS * 4 + EGRESS * 2 + TC]; // resident blocks per SM of this instantiation
    if (!per_sm) {
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_resolve<NAT, QOS, EGRESS, TC, ICMPERR>, RS_TEAM, 0) != cudaSuccess ||
            per_sm < 1)
            per_sm = 8;
    }
    long cap = (long)L.num_sms * per_sm, want = b.n ? b.n : 1;
    int grid = (int)(want < cap ? want : cap);
    prof_begin(L, prof_name<resolve_name, NAT, QOS, EGRESS, TC, ICMPERR>());
    launch_dep(k_resolve<NAT, QOS, EGRESS, TC, ICMPERR>, grid, RS_TEAM, L.stream, c, b, g, L.s.qslot, L.s.counters);
    prof_end(L);
    L.launches++;
}

cudaError_t run_antispoof(Launcher &L, const DevCtx &c, const DevBatch &b, const Tbl *as6) {
    with_flags(
        [&](auto v6) {
            constexpr bool V6 = decltype(v6)::value;
            LAUNCH_AS((prof_name<antispoof_name, V6>()), k_antispoof<V6>, b.n, 8, c, b, V6 ? *as6 : Tbl{});
        },
        as6 != nullptr);
    return cudaGetLastError();
}

cudaError_t run_qos(Launcher &L, const DevCtx &c, const DevBatch &b0, bool egress, const Tbl *v6) {
    const Tbl &t = egress ? c.qos_eg : c.qos_in;
    DevBatch b = b0;
    b.kshift = kshift_for((u64)t.mask + 1);
    with_flags(
        [&](auto shape6) {
            constexpr bool V6 = decltype(shape6)::value;
            LAUNCH_AS((prof_name<qos_name, V6>()), k_qos_classify<V6>, b.n, 8, c, b, egress ? 1 : 0, L.s.key_a, L.s.val_a, L.s.counters,
                      sort_T(L), V6 ? *v6 : Tbl{});
        },
        v6 != nullptr);
    Grouped g;
    cudaError_t e = group_by_key(L, b.n, (u64)t.mask + 1, b.kshift, &g);
    if (e != cudaSuccess) return e;
    with_flags([&](auto eg) { launch_resolve<false, true, decltype(eg)::value>(L, c, b, g); }, egress);
    return cudaGetLastError();
}

// The programs keyed on the subscriber directory (nat44_egress, pipeline_up, pipeline_tc): classify, group by
// directory slot, resolve.  With accounting on (L.acct_attr), classify is the ACCT instantiation.  v6 (the pipelines
// only): IPv6 frames are shaped, classify is the V6 instantiation.  as6 (the pipelines only): antispoof allows IPv6
// sources in their subscriber's prefixes, classify is the AS6 instantiation.  icmperr
// (bng_nat_icmp_errors_egress_enable): the ICMPERR instantiations of classify and resolve.
template <bool AS, bool QOS, bool TC>
static cudaError_t run_dir_prog(Launcher &L, const DevCtx &c, const DevBatch &b0, const Tbl *v6, const Tbl *as6, bool icmperr) {
    DevBatch b = b0;
    b.kshift = kshift_for((u64)c.subdir.mask + 1);
    // (nat44_egress has neither a bucket nor antispoof and is never given the tables)
    with_flags(
        [&](auto acct, auto shape6, auto spoof6, auto icmp) {
            constexpr bool ACCT = decltype(acct)::value, V6 = decltype(shape6)::value, AS6 = decltype(spoof6)::value,
                           ICMPERR = decltype(icmp)::value;
            LAUNCH_AS((prof_name<classify_name, AS, QOS, TC, ACCT, V6, AS6, ICMPERR>()), (k_pipe_classify<AS, QOS, TC, ACCT, V6, AS6, ICMPERR>),
                      b.n, CLASSIFY_BPS(AS), c, b, L.s.key_a, L.s.val_a, L.s.counters, sort_T(L), L.acct_attr,
                      AS6 ? *as6 : (V6 ? *v6 : Tbl{}));
        },
        L.acct_attr != nullptr, only<QOS>(v6 != nullptr), only<AS>(as6 != nullptr), icmperr);
    Grouped g;
    cudaError_t e = group_by_key(L, b.n, (u64)c.subdir.mask + 1, b.kshift, &g);
    if (e != cudaSuccess) return e;
    with_flags([&](auto icmp) { launch_resolve<true, QOS, false, TC, decltype(icmp)::value>(L, c, b, g); }, icmperr);
    return cudaGetLastError();
}

cudaError_t run_nat_egress(Launcher &L, const DevCtx &c, const DevBatch &b, bool icmp_errors_eg) {
    return run_dir_prog<false, false, false>(L, c, b, nullptr, nullptr, icmp_errors_eg);
}

cudaError_t run_nat_ingress(Launcher &L, const DevCtx &c, const DevBatch &b, bool icmp_errors) {
    with_flags(
        [&](auto icmp) {
            constexpr bool ICMPERR = decltype(icmp)::value;
            LAUNCH_AS((prof_name<nat_ingress_name, ICMPERR>()), k_nat_ingress<ICMPERR>, b.n, 6, c, b);
        },
        icmp_errors);
    return cudaGetLastError();
}

cudaError_t run_nat_hairpin_xdp(Launcher &L, const DevCtx &c, const DevBatch &b) {
    LAUNCH(k_nat_hairpin_xdp, b.n, 8, c, b);
    return cudaGetLastError();
}

cudaError_t run_pipeline_up(Launcher &L, const DevCtx &c, const DevBatch &b, const Tbl *v6, const Tbl *as6, bool icmp_errors_eg) {
    return run_dir_prog<true, true, false>(L, c, b, v6, as6, icmp_errors_eg);
}

cudaError_t run_pipeline_tc(Launcher &L, const DevCtx &c, const DevBatch &b, const Tbl *v6, const Tbl *as6, bool icmp_errors_eg) {
    return run_dir_prog<true, true, true>(L, c, b, v6, as6, icmp_errors_eg);
}
