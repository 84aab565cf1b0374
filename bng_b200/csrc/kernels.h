// bng_b200 — internal interface between the C-ABI layer (ctx.cu) and the
// kernel translation units.
#pragma once
#include <string>
#include <type_traits>

#include "common.cuh"

// Picks a kernel instantiation from runtime switches: calls f with each runtime bool lifted to std::true_type or
// std::false_type, which f reads as decltype(x)::value.  An argument that already is a std::bool_constant passes
// through, so a caller pins the combinations that cannot occur (only<>) and they are never instantiated.
template <class F>
decltype(auto) with_flags(F &&f) {
    return f();
}
template <class F, class A, class... R>
decltype(auto) with_flags(F &&f, A a, R... r) {
    auto rest = [&](auto x) { return with_flags([&](auto... y) { return f(x, y...); }, r...); };
    if constexpr (std::is_same_v<A, bool>)
        return a ? rest(std::true_type{}) : rest(std::false_type{});
    else
        return rest(a);
}
// the switch b where the instantiation has the stage it selects (C), else always off
template <bool C>
auto only(bool b) {
    if constexpr (C)
        return b;
    else
        return std::false_type{};
}
// The profile name of an instantiation, built once by name(F...) and kept for the process: prof_begin keeps the pointer.
template <auto name, bool... F>
const char *prof_name() {
    static const std::string s = name(F...);
    return s.c_str();
}

struct Scratch {
    u32 *key_a, *key_b, *val_a, *val_b; // ordering keys / frame indices, unsorted and grouped
    u32 *qslot;                         // group heads (positions in the grouped arrays)
    void *cub_tmp;
    size_t cub_tmp_bytes;
    u32 *counters; // 16 x u32 of per-run device counters
    u32 cap;       // frames the arrays above can hold
    u32 *attr;     // [cap] per-frame accounting attribution (directory slot or DIR_NONE); allocated with the counters
};

// optional per-kernel timing (bng_prof_enable): CUDA events around every launch
struct ProfPending {
    int acc;
    cudaEvent_t a, b;
};

struct Launcher {
    cudaStream_t stream;
    int num_sms;
    Scratch s;
    u32 *acct_attr; // non-null: the upstream classify of this run records each frame's attribution here (acct.cu)
    unsigned long long launches;
    // per-context (= per-device) launch configuration, filled on first use: nothing here may be process-wide,
    // one process can hold contexts on several GPUs
    int dhcp_smem_set[4]; // cudaFuncAttributeMaxDynamicSharedMemorySize applied on this context's device, by <V6, ND> bits
    int resolve_bps[32]; // resident blocks per SM of the k_resolve instantiations, by <NAT, QOS, EGRESS, TC, ICMPERR> bits
    int prof;
    ProfPending pend[32];
    int npend;
    const char *acc_name[32];
    double acc_ms[32];
    unsigned long long acc_n[32];
    int nacc;
};

void prof_begin(Launcher &L, const char *name);
void prof_end(Launcher &L);
void prof_collect(Launcher &L); // call after the stream has been synchronised

size_t sort_temp_bytes(u32 n);

// as6 (antispoof_ingress and the pipelines): subscriber_ipv6 when antispoof allows IPv6 sources in their subscriber's
// prefixes (bng_antispoof_ipv6_prefixes_enable, and the table has live entries), else nullptr
cudaError_t run_antispoof(Launcher &L, const DevCtx &c, const DevBatch &b, const Tbl *as6);
// v6: subscriber_ipv6 when IPv6 frames are shaped by their owner's bucket (bng_qos_ipv6_enable, and the table has live
// entries), else nullptr
cudaError_t run_qos(Launcher &L, const DevCtx &c, const DevBatch &b, bool egress, const Tbl *v6);
// icmp_errors_eg (nat44_egress and the pipelines): subscribers' ICMP errors are translated by the flow they quote
// (bng_nat_icmp_errors_egress_enable)
cudaError_t run_nat_egress(Launcher &L, const DevCtx &c, const DevBatch &b, bool icmp_errors_eg);
// icmp_errors: ICMP errors are translated by the flow they quote (bng_nat_icmp_errors_enable)
cudaError_t run_nat_ingress(Launcher &L, const DevCtx &c, const DevBatch &b, bool icmp_errors);
cudaError_t run_nat_hairpin_xdp(Launcher &L, const DevCtx &c, const DevBatch &b);
cudaError_t run_pipeline_up(Launcher &L, const DevCtx &c, const DevBatch &b, const Tbl *v6, const Tbl *as6, bool icmp_errors_eg);
cudaError_t run_pipeline_tc(Launcher &L, const DevCtx &c, const DevBatch &b, const Tbl *v6, const Tbl *as6, bool icmp_errors_eg);
// The DHCPv6 fast path (include/bng_b200.h, bng_dhcpv6_enable): its tables and where its counters go.  The counters
// follow the ST_COUNT of the packed statistics vector, which then holds ST_ALL; the kernels' per-block accumulators
// (BlockStats) keep ST_COUNT.
#define ST_DHCP6 ST_COUNT
#define ST_DHCP6_N 12
#define DHCP6_CFG_BYTES 96
struct Dhcp6Args {
    Tbl bind;         // dhcpv6_bindings: 32-byte key (4 words), 64-byte value at 32
    const u8 *cfg;    // dhcpv6_server_config[0]
    u64 *stats;       // ST_DHCP6_N counters
    u32 room_stride;  // a frame's storage: room_stride bytes, or 0: its len rounded up to 16 (an offset table)
    u32 *need;        // pinned zero-copy feed: bytes the scatter writes back, raised to cover a grown reply; else nullptr
};
// Router and Neighbor Solicitations (include/bng_b200.h, bng_nd_enable): their counters follow dhcpv6_stats
#define ST_ND (ST_DHCP6 + ST_DHCP6_N)
#define ST_ND_N 11
#define ST_ALL (ST_COUNT + ST_DHCP6_N + ST_ND_N)
#define ND_CFG_BYTES 320
struct NdArgs {
    Tbl bind;         // nd_bindings: the 8-byte MAC word, 48-byte value at 8
    const u8 *cfg;    // nd_config[0]
    u64 *stats;       // ST_ND_N counters
    u32 room_stride;  // as Dhcp6Args
    u32 *need;
};
// d6: the DHCPv6 tables when the fast path answers DHCPv6 (bng_dhcpv6_enable, a configured server and live bindings),
// else nullptr; nd: the ND tables when it answers Router and Neighbor Solicitations (bng_nd_enable and a configured
// nd_config), else nullptr
cudaError_t run_dhcp_fastpath(Launcher &L, const DevCtx &c, const DevBatch &b, const Dhcp6Args *d6, const NdArgs *nd);

// header gather / scatter between a pinned host arena and a compact device copy (hostio.cu); icmp_errors (TC only):
// also bytes 64-79 of an ICMP error frame, for nat44_ingress with bng_nat_icmp_errors_enable and for nat44_egress and
// the pipelines with bng_nat_icmp_errors_egress_enable
cudaError_t run_gather_frames(cudaStream_t st, int blocks, const u8 *arena, const u32 *off16, const u32 *len, u32 stride,
                              u32 n, u32 slot, bool tc, bool icmp_errors, u8 *dst, u32 *need);
cudaError_t run_scatter_frames(cudaStream_t st, int blocks, u8 *arena, const u32 *off16, const u32 *need, u32 stride, u32 n,
                               u32 slot, const u8 *src);

// table maintenance (tableops.cu); keys/values/results are device pointers
enum { TOP_UPDATE = 0, TOP_LOOKUP = 1, TOP_DELETE = 2 };
// dir / dir_role: the subscriber directory and which half of it table t feeds (0 none, 1 subscriber_nat, 2 qos_ingress)
// acct / idle: the per-subscriber counter and idle records (nullptr until first enabled); a directory slot that is
// claimed for an address has both records zeroed
cudaError_t run_table_op(Launcher &L, const Tbl &t, int op, const u8 *keys, u8 *vals, int *results, u64 n, u32 flags,
                         const Tbl &dir, int dir_role, u64 *acct, u64 *idle);
cudaError_t run_dir_clear_half(Launcher &L, const Tbl &dir, int role);
cudaError_t run_epoch_reset(Launcher &L, const Tbl &sessions);
cudaError_t run_table_rebuild(Launcher &L, const Tbl &old_table, const Tbl &empty_table);
// session expiry sweep (sweep.cu); n_expired: device counter, incremented by the number of sessions removed
cudaError_t run_nat_sweep(Launcher &L, const DevCtx &c, u64 now, u32 *n_expired /* [0] expired, [1] tombstones seen */);
// NAT flow-state flush (flush.cu).  The address set: mask + 1 (a power of two >= 2 x the distinct addresses) u64
// words, 0 = empty, ADDRSET_LIVE | address = member; linear probing from aset_home().  Built on the host.
#define ADDRSET_LIVE (1ull << 32)
struct AddrSet {
    const u64 *words;
    u32 mask;
};
__host__ __device__ __forceinline__ u32 aset_home(u32 addr, u32 mask) {
    u32 h = addr; // murmur3 finaliser: the last octet sits in the top byte of the word, so every bit must mix down
    h ^= h >> 16;
    h *= 0x85EBCA6Bu;
    h ^= h >> 13;
    h *= 0xC2B2AE35u;
    h ^= h >> 16;
    return h & mask;
}
#ifdef __CUDACC__
__device__ __forceinline__ bool aset_has(const AddrSet &a, u32 addr) {
    for (u32 i = aset_home(addr, a.mask);; i = (i + 1) & a.mask) {
        const u64 w = a.words[i];
        if (w == 0) return false;
        if ((u32)w == addr) return true;
    }
}
#endif
cudaError_t run_nat_flush(Launcher &L, const DevCtx &c, const AddrSet &a, u64 now, u32 *cnt /* [4], see flush.cu */);
cudaError_t run_table_dump(Launcher &L, const Tbl &t, u8 *keys_out, u8 *vals_out, u32 *count_out, u64 cap);

// per-subscriber traffic accounting (acct.cu).  A record is ACCT_WORDS u64 (struct bng_acct), index-aligned with the
// subscriber directory.  Modes of run_acct: where a frame's subscriber comes from.
#define ACCT_WORDS 8
enum { ACCT_ATTR = 0, ACCT_SRC = 1, ACCT_DST = 2 }; // attribution words of classify / header source / header destination
// the directory slot of an address, or DIR_NONE
__device__ __forceinline__ u32 dir_slot_of(const Tbl &dir, u32 addr) {
    const u64 k = addr;
    const u8 *s = tbl_find<1, false>(dir, &k);
    return s ? (u32)((s - dir.slots) >> 4) : DIR_NONE;
}
#ifdef __CUDACC__
// subscriber_ipv6 (common.cuh): the value of the entry (len, the address's first len bits), if there is one
__device__ __forceinline__ bool lpm6_probe(const Tbl &t, u32 len, const u32 *a, u32 *val) {
    u64 kw[LPM6_KW];
    lpm6_key(kw, len, a);
    const u8 *s = tbl_find<LPM6_KW, false>(t, kw);
    if (s) *val = *(const u32 *)(s + t.voff);
    return s != nullptr;
}
// The prefix lengths that have live entries, longest first, in shared memory: built once per block from the table's
// counts by the whole block (blockDim.x >= 160), so a frame probes only the lengths in use.
struct V6Lens {
    u8 len[LPM6_LENS];
    u32 n, wcnt[5];
};
__device__ __forceinline__ void v6_lens_load(V6Lens &s, const u32 *plens) {
    const u32 t = threadIdx.x, lane = t & 31, w = t >> 5; // thread t stands for length 128 - t
    const bool live = t < LPM6_LENS && plens[LPM6_LENS - 1 - t] != 0;
    const u32 m = __ballot_sync(0xffffffffu, live);
    if (lane == 0 && w < 5) s.wcnt[w] = __popc(m);
    __syncthreads();
    if (live) {
        u32 pos = __popc(m & ((1u << lane) - 1));
        for (u32 j = 0; j < w; j++) pos += s.wcnt[j];
        s.len[pos] = (u8)(LPM6_LENS - 1 - t);
    }
    if (t == 0) s.n = s.wcnt[0] + s.wcnt[1] + s.wcnt[2] + s.wcnt[3] + s.wcnt[4];
    __syncthreads();
}
// The owner of an IPv6 address: the value of the longest prefix in subscriber_ipv6 that covers it (a subscriber IPv4
// address in qos_ingress key order).  One probe per prefix length in use until one hits.
__device__ __forceinline__ bool v6_owner(const Tbl &t, const V6Lens &s, const u32 *a, u32 *owner) {
    for (u32 k = 0; k < s.n; k++)
        if (lpm6_probe(t, s.len[k], a, owner)) return true;
    return false;
}
// the 16 address bytes at frame offset off as four little-endian words (off even)
__device__ __forceinline__ void v6_addr(const u8 *p, u32 off, u32 *a) {
#pragma unroll
    for (int j = 0; j < 4; j++) a[j] = rd32(p, off + 4 * j);
}
#endif
// acct: count the frames into the counter records (nullptr: no counting); idle: stamp the idle records of the frames
// that pass (nullptr: no stamping).  At least one of the two is given.  v6: subscriber_ipv6 while it has live entries
// (IPv6 frames are attributed through it), else nullptr.
cudaError_t run_acct(Launcher &L, const Tbl &dir, const DevBatch &b, int mode, u64 *acct, u64 *idle, const Tbl *v6);
// results[i] = 0 / -ENOENT, out[i] zeroed on a miss; acct may be nullptr (every record reads as zero)
cudaError_t run_acct_read(Launcher &L, const Tbl &dir, const u64 *acct, const u32 *addrs, u64 n, u64 *out, int *results);
// every directory address with its record, compacted at *count (grows past cap: only cap are written)
cudaError_t run_acct_dump(Launcher &L, const Tbl &dir, const u64 *acct, u32 *addrs_out, u64 *out, u32 *count, u64 cap);
// record of every address of the list that has a directory entry := the given one (snapshot restore)
cudaError_t run_acct_load(Launcher &L, const Tbl &dir, u64 *acct, const u32 *addrs, const u64 *recs, u64 n);

// per-subscriber idle detection (idle.cu).  A record is IDLE_WORDS u64, index-aligned with the subscriber directory:
// word 0 the timeout (low half) and a scratch word of run_idle_timeout_set (high half, 0 between calls), then the
// upstream stamp, the downstream stamp and since, each as clock + 1 (0: none).  run_acct stamps words 1 and 2.
#define IDLE_WORDS 4
enum { IDLE_UP = 1, IDLE_DOWN = 2, IDLE_SINCE = 3 };
// every live directory slot: unstarted records start at now; the idle ones are compacted at *count (which grows past
// cap: only cap are written) as (address, struct bng_idle)
cudaError_t run_idle_scan(Launcher &L, const Tbl &dir, u64 *idle, u64 now, u32 default_s, u32 flags, u32 *addrs_out, u64 *out,
                          u32 *count, u64 cap);
// results[i] = 0 / -ENOENT, out[i] (struct bng_idle) zeroed on a miss; idle may be nullptr (every record reads as zero)
cudaError_t run_idle_read(Launcher &L, const Tbl &dir, const u64 *idle, const u32 *addrs, u64 n, u64 *out, int *results);
// timeout of every listed address that has a directory entry := timeouts[i], the last of a repeated address winning
cudaError_t run_idle_timeout_set(Launcher &L, const Tbl &dir, u64 *idle, const u32 *addrs, const u32 *timeouts, u64 n, int *results);
// every record's stamps and since := none (the timeouts stay)
cudaError_t run_idle_restart(Launcher &L, const Tbl &dir, u64 *idle);
// whole record of every listed address that has a directory entry := recs[i] (struct bng_idle, as run_idle_read gives
// it); the addresses are distinct (subscriber hand-over, bng_sub_import)
cudaError_t run_idle_load(Launcher &L, const Tbl &dir, u64 *idle, const u32 *addrs, const u64 *recs, u64 n);

// subscriber hand-over between contexts (move.cu).  The slot lists of the three flow tables live in one array:
// nat_sessions' at [0, ns), nat_reverse's at [ns, ns + nr), eim_table's at [ns + nr, ns + nr + ne) (table slot counts).
// cnt: [0..2] entries listed per table, [3] nat_sessions tombstones seen (zeroed by the caller).
cudaError_t run_move_select(Launcher &L, const DevCtx &c, const AddrSet &a, u32 *lists, u32 *cnt);
// tombstones the listed slots (no log record, no statistic); n[k] entries of table k's list
cudaError_t run_move_detach(Launcher &L, const DevCtx &c, const u32 *lists, const u32 n[3]);
// the slots of subscriber_ipv6 whose value is in the address set, listed at `list` (room for every slot), *cnt of them
cudaError_t run_move_select_v6(Launcher &L, const Tbl &v6, const AddrSet &a, u32 *list, u32 *cnt);

// NAT port-usage census (natuse.cu).  Scratch of its own, zeroed before every census:
//   set        set_mask + 1 u64 words, 0 = empty: the distinct held triples and ports, overall and per subscriber.  A
//              live session or EIM entry puts at most four keys in, so 4 x (max_nat_sessions + max_eim_mappings) keys
//              fit in the power of two >= 4/3 of that (load <= 3/4).  Slot indices and directory slots are < 2^30.
//   sub        NU_SUB_WORDS u32 per subscriber directory slot: sessions, eim, in_use[3], in_use_any, outside, unreachable
//   pub        pub_mask + 1 records of NU_PUB_WORDS u64: ADDRSET_LIVE | address (0 = empty), the sum of block_ports, then
//              u32 sessions, eim, blocks, in_use[3], in_use_any, unreachable
//   sum        NU_SUM_WORDS u64: the struct bng_nat_usage_sum fields in order, then the census's own words
#define NU_SUB_WORDS 8
#define NU_PUB_WORDS 6
#define NU_NONE 0xFFFFFFFFu
enum {
    NU_SUBSCRIBERS, NU_SESSIONS, NU_EIM, NU_TRIPLES, NU_UNREACHABLE, NU_STALE, NU_ORPHAN_SES, NU_ORPHAN_EIM, // summed per thread
    NU_SUBS_FOUND, NU_PUBS_FOUND,
    NU_PUB_RESERVED, // public-address slots reserved so far (reservations past half the table: overflow)
    NU_OVERFLOW,     // the public-address table was too small: grow it and run again
    NU_SET_FULL,     // the set was full (its sizing rules that out)
    NU_SUM_WORDS
};
#define NU_LOCAL (NU_ORPHAN_EIM + 1)
struct NatUse {
    u64 *set;
    u32 set_mask, pub_mask;
    u32 *sub;
    u64 *pub;
    u64 *sum;
    // qualifying records (struct bng_nat_sub_use / bng_nat_pub_use, 16 u32 each) and their addresses, up to the caps
    u32 *sub_addrs, *sub_out, *pub_addrs, *pub_out;
    u64 sub_cap, pub_cap;
};
cudaError_t run_nat_usage_flows(Launcher &L, const DevCtx &c, const NatUse &u);
// qualifying subscriber records (permille >= min_permille) and every public-address record, compacted
cudaError_t run_nat_usage_emit(Launcher &L, const DevCtx &c, const NatUse &u, u32 min_permille);

// DHCP lease census and expiry sweep (leases.cu).  Scratch of the census, zeroed before every census:
//   set        set_mask + 1 u64 words, 0 = empty.  An unexpired lease entry creates at most three keys (leases.cu), so
//              3 x (the three lease maps' max_entries) keys fit in the power of two >= 4/3 of that (load <= 3/4).
//   pools      LS_POOL_WORDS u64 per pool record: n_known records index-aligned with ip_pools' slots, then unk_mask + 1
//              records of a hash keyed by the pool_ids that have no ip_pools entry (LS_P_KEY: ADDRSET_LIVE | pool_id,
//              0 = empty).  Record indices are < 2^26.
//   sum        LS_SUM_WORDS u64: the struct bng_lease_sum fields in order, then the census's own words
#define LS_POOL_WORDS 8
enum { LS_P_ENTRIES = 0, LS_P_EXPIRED = 3, LS_P_ADDRS, LS_P_OUTSIDE, LS_P_CONFLICTS, LS_P_KEY };
#define LS_NONE 0xFFFFFFFFu
enum {
    LS_ENT0, LS_ENT1, LS_ENT2, LS_EXP0, LS_EXP1, LS_EXP2, LS_ADDRS, LS_CONFLICTS, LS_UNKNOWN_POOL, LS_CID_DANGLING, // summed per thread
    LS_POOLS_FOUND,
    LS_UNK_CLAIMED,  // unknown-pool slots claimed so far (half the hash claimed: overflow)
    LS_OVERFLOW,     // the unknown-pool hash was too small: grow it and run again
    LS_SET_FULL,     // the set was full (its sizing rules that out)
    LS_SUM_WORDS
};
#define LS_LOCAL (LS_CID_DANGLING + 1)
struct LeaseUse {
    u64 *set;
    u32 set_mask, unk_mask, n_known;
    u32 wire; // the prefix test's byte order (bng_dhcp_lease_addr_order)
    u64 *pools, *sum;
    u32 *ids_out, *out; // pool ids and records (struct bng_lease_pool_use, 16 u32 each), up to cap
    u64 cap;
};
cudaError_t run_lease_census(Launcher &L, const DevCtx &c, const LeaseUse &u, u64 now_s);
cudaError_t run_lease_pools(Launcher &L, const DevCtx &c, const LeaseUse &u);
// The sweep's words (zeroed by the caller): due entries found, entries removed from the three lease maps and from
// circuit_id_map, tombstones seen in the four tables (its own included), "the MAC set was full" (sized against it) and
// "a due entry was gone before its erase" (nothing runs beside the sweep); either of the two fails the call.
enum { LS_W_FOUND = 0, LS_W_REMOVED = 1, LS_W_TOMBS = 5, LS_W_SET_FULL = 9, LS_W_LOST = 10, LS_W_WORDS = 11 };
struct LeaseSweep {
    u64 now_s, grace_s, cap;
    u32 *out;  // struct bng_lease_removed, 16 u32 each, cap of them
    u64 *cnt;
    u64 *macs; // mac_mask + 1 words, zeroed: the MACs of the subscriber_pools entries removed (>= 2 x cap slots)
    u32 mac_mask;
};
// removes the due entries whose output slot is below cap, then the circuit_id_map entries that name a removed MAC
cudaError_t run_lease_sweep(Launcher &L, const DevCtx &c, const LeaseSweep &w);

// lawful intercept (li.cu).  A record is LI_HDR bytes of header (struct bng_li_record) and the captured bytes, zero
// padded to rec_bytes.  The targets are an AddrSet with target ids index-aligned to its words.
#define LI_HDR 64
#define LI_NOSLOT 0xFFFFFFFFu // match without a ring slot (the ring was full)
#define LI_VOID 0xFFu         // verdict byte of a record the drain skips (a frame antispoof dropped)
struct LiRing {
    u8 *buf;   // cap records of rec_bytes
    u64 *ctl;  // [0] slots handed out (may pass cap), [1] records lost, [2] (u32) uplink matches of the run
    uint2 *match; // uplink: (frame, ring slot or LI_NOSLOT) of every match of the run, in no order
    u32 cap, rec_bytes, snaplen, prog;
    AddrSet tgt;
    const u32 *ids;
    u64 batch;
};
// Where the bytes of a chunk of a pinned host batch live (run_host_zero_copy): the program sees a compact copy of
// the first need[i] bytes (rounded up to 16) of each frame; the rest stays in the mapped host arena, which the TC
// programs never touch.  arena == nullptr: the DevBatch holds whole frames.
struct LiSrc {
    const u8 *arena;   // device view of the chunk's host arena
    const u32 *off16;  // the chunk's offsets, or nullptr (fixed stride)
    const u32 *need;   // bytes of each frame in the compact copy, or nullptr: the compact slot is the whole storage
    u32 stride;        // the caller's stride
};
// UP: before the program (the frame as it entered), reserves the slots and lists the matches; then run_li_verdict
// after the program.  !UP: after the program, complete records.  attr: classify's attribution words in the pipelines
// (a SHOT frame without one was dropped by antispoof), else nullptr.
// v6: as run_acct's.
cudaError_t run_li_capture(Launcher &L, const LiRing &r, const DevBatch &b, const LiSrc &src, bool up, const Tbl *v6);
cudaError_t run_li_verdict(Launcher &L, const LiRing &r, const DevBatch &b, const u32 *attr);

// incremental replication (delta.cu).  A table as the diff sees it: nslots slots whose first kw words are the key (word
// 0 doubles as the slot state) and whose words [kw, sw) hold the compared bytes; the shadow keeps those sw words per
// slot as last sent.  vals != nullptr: words [kw, sw) and the value come from vals + slot * vstride instead of the slot
// (the accounting records beside the subscriber directory).
#define DELTA_MAXW 16
#define DELTA_NO_TIME 0xFFFFFFFFu
struct DeltaTbl {
    const u8 *slots;
    const u8 *vals;
    u64 *shadow;
    u64 nslots;
    u32 slot_bytes, vstride;
    u32 kw, sw;
    u32 tw;                     // word of the time field (DELTA_NO_TIME: none); sent again once it moves > refresh
    u32 key_size, value_size, voff, vlayout;
    u64 refresh;
    u64 mask[DELTA_MAXW];       // per word: the bits compared exactly
};
// del / up: slot lists of the two classes (room for nslots each); cnt[0], cnt[1]: their lengths (zeroed by the caller).
// full: the shadow is taken as empty (every live entry is an upsert, nothing is deleted)
cudaError_t run_delta_diff(Launcher &L, const DeltaTbl &t, u32 *del, u32 *up, u32 *cnt, bool full);
cudaError_t run_delta_emit(Launcher &L, const DeltaTbl &t, const u32 *del, u32 n_del, const u32 *up, u32 n_up, u8 *del_keys,
                           u8 *up_keys, u8 *up_vals);
cudaError_t run_delta_commit(Launcher &L, const DeltaTbl &t, const u32 *del, u32 n_del, const u32 *up, u32 n_up);
