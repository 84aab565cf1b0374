// bng_b200 — device-side building blocks shared by every kernel:
// table descriptors, the open-addressing hash, packet access, statistics and
// event staging.  sm_90a only; no host fallback exists for anything here.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

typedef unsigned long long u64;
typedef uint32_t u32;
typedef uint16_t u16;
typedef uint8_t u8;

// ---------------------------------------------------------------------------
// Packed statistics vector.  One u64 per counter of the reference's four
// stats structs, in declaration order, so a map lookup is a plain copy:
//   antispoof_stats  bpf/antispoof.c:58-65      [ST_AS, +6)
//   qos_stats        bpf/qos_ratelimit.c:53-58  [ST_QOS, +4)
//   nat_stats        bpf/nat44.c:176-190        [ST_NAT, +13)
//   dhcp_stats       bpf/maps.h:171-184         [ST_DHCP, +10)
// followed by dataplane-internal diagnostics.
// ---------------------------------------------------------------------------
enum {
    ST_AS = 0,
    ST_AS_ALLOWED = 0, ST_AS_DROPPED, ST_AS_LOGGED, ST_AS_V4_VIOL, ST_AS_V6_VIOL, ST_AS_UNKNOWN_MAC,
    ST_QOS = 6,
    ST_QOS_PASS_PKTS = 6, ST_QOS_DROP_PKTS, ST_QOS_PASS_BYTES, ST_QOS_DROP_BYTES,
    ST_NAT = 10,
    ST_NAT_SNAT = 10, ST_NAT_DNAT, ST_NAT_HAIRPIN, ST_NAT_DROPPED, ST_NAT_PASSED, ST_NAT_CREATED,
    ST_NAT_EXPIRED, ST_NAT_EXHAUST, ST_NAT_EIM_HIT, ST_NAT_EIM_MISS, ST_NAT_ALG, ST_NAT_CT_LOOKUPS, ST_NAT_CT_HITS,
    ST_DHCP = 23,
    ST_DHCP_TOTAL = 23, ST_DHCP_HIT, ST_DHCP_MISS, ST_DHCP_ERROR, ST_DHCP_EXPIRED, ST_DHCP_O82_PRESENT,
    ST_DHCP_O82_ABSENT, ST_DHCP_BCAST, ST_DHCP_UCAST, ST_DHCP_VLAN,
    ST_LRU_OVERFLOW = 33,
    ST_EV_LOST_SPOOF = 34,
    ST_EV_LOST_NATLOG = 35,
    ST_TABLE_FULL = 36,
    ST_NAT_COOP = 37, // ordered-phase chunks created warp-cooperatively ...
    ST_NAT_SEQ = 38,  // ... and chunks that had to be walked one frame at a time (diagnostics)
    ST_LRU_EVICT = 39, // entries evicted from a full LRU map to make room for an insert
    ST_COUNT = 40,
};

// ---------------------------------------------------------------------------
// Open-addressing hash table.  Every slot starts with a 64-bit key word that
// doubles as the slot's state: K_EMPTY / K_TOMB / K_BUSY are reserved values
// (no frame can produce them and host updates carrying them are refused).
// Keys shorter than 8 bytes are zero-extended; longer keys continue in the
// following words.  The value sits at `voff`, verbatim in the reference's
// layout, so device code addresses the reference's fields by offset.
// ---------------------------------------------------------------------------
#define K_EMPTY 0xFFFFFFFFFFFFFFFFull
#define K_TOMB 0xFFFFFFFFFFFFFFFEull
#define K_BUSY 0xFFFFFFFFFFFFFFFDull

struct Tbl {
    u8 *slots;
    u32 *count;      // live entries
    u32 mask;        // capacity - 1 (capacity is a power of two)
    u32 home_mask;   // hash -> home slot: mask, or mask & ~1 for even home slots (bng_open: bindings, subscriber directory)
    u32 slot_bytes;  // multiple of 32
    u32 voff;        // value offset inside the slot
    u32 max_entries; // the reference map's max_entries
    u32 key_size;
    u32 value_size;
    u32 vlayout; // 0: value stored verbatim at voff; VL_SESSION: nat_sessions hot/cold layout below
    // BPF_MAP_TYPE_LRU_HASH: an insert into a full map evicts instead of failing.  0: plain hash (-E2BIG);
    // LRU_TS | offset << 8: evict the entry with the oldest u64 timestamp at that slot offset among the
    // slots next to the new key's home; LRU_ANY: no timestamp in the value (nat_reverse): the first live one.
    u32 lru;
    // LPM-keyed tables only (subscriber_ipv6, below), else nullptr: LPM6_LENS live-entry counts, one per prefix length,
    // kept by the table-op kernels beside `count`
    u32 *plens;
};
#define LRU_NONE 0u
#define LRU_TS 1u
#define LRU_ANY 2u
#define LRU_WINDOW 16u

// nat_sessions slots are 128 B, laid out by what the per-frame paths touch (DESIGN.md §4):
//   sector 0 [0,32)   key 16 | nat_ip 4 | nat_port 2 | epoch 2 | out_lo 8
//            everything an upstream HIT needs — probe, translation and the out-direction counters — is
//            ONE 32-byte sector: one 32-byte load plus one 64-bit atomic on the same sector.
//   sector 1 [32,64)  last_seen 8 | orig_ip 4 | state word 4 | orig_port 2 | pad 6 | in_lo 8
//            what a downstream hit adds (original tuple, TCP state, in-direction counters), and last_seen.
//   sector 2 [64,96)  out_hi 8 | in_hi 8 | created 8 | dest_ip 4 | dest_port 2 | _pad1 2   (creation / carries / ABI)
//   sector 3 [96,104) the struct's padding bytes (they cross the ABI verbatim); [104,112) SES_SIDE (ses_touch_exact)
// `epoch` is not part of struct nat_session: it is the batch (low 16 bits of the batch sequence, 0 = never)
// in which last_seen was last stored.  Every frame of a batch would store the same last_seen = now, so only
// a frame that finds an older epoch stores it (and the epoch): one extra store per flow and batch instead of
// a second sector written by every frame.  bng_prog_run() clears all epochs whenever the 16-bit batch
// counter wraps (k_epoch_reset), so a stale epoch can never alias the current one.
// The reference layout of struct nat_session (bpf/nat44.c:123-141) is restored by ses_abi_to_slot()
// whenever a value crosses the ABI.
#define VL_SESSION 1u
#define VL_QOS 2u         // value verbatim at voff, plus a copy of rate_bps at QOS_RATE_COPY
#define QOS_RATE_COPY 8u  // qos slot: key u64 @0, rate_bps copy @8, struct token_bucket @16
enum {
    SES_NAT_IP = 16,    // u32
    SES_NAT_PORT = 20,  // u16
    SES_EPOCH = 22,     // u16, dataplane-internal
    // The two counters of a direction advance with ONE 64-bit atomic: the low words of packets and
    // bytes share a u64 (packets in bits 0-31, bytes in bits 32-63), their high words a second u64 that
    // is touched only when a low word wraps (ses_count()).
    SES_OUT_LO = 24,    // u64: packets_out[31:0] | bytes_out[31:0] << 32
    SES_LAST_SEEN = 32, // u64
    SES_ORIG_IP = 40,   // u32
    SES_STATE = 44,     // u8 state, protocol@45, flags@46, is_hairpin@47
    SES_ORIG_PORT = 48, // u16
    SES_IN_LO = 56,
    SES_OUT_HI = 64, // u64: packets_out[63:32] | bytes_out[63:32] << 32
    SES_IN_HI = 72,
    SES_CREATED = 80,
    SES_DEST_IP = 88,   // u32
    SES_DEST_PORT = 92, // u16, _pad1@94
    SES_PAD_A = 96,     // struct bytes 20..23
    SES_PAD_B = 100,    // struct bytes 76..79
    SES_SIDE = 104,     // u64, dataplane-internal: per-frame clock values of a batch that replaces last_seen (ses_touch_exact)
};
// byte offset inside struct nat_session -> byte offset inside the slot
__host__ __device__ __forceinline__ u32 ses_abi_to_slot(u32 a) {
    if (a < 4) return SES_NAT_IP + a;
    if (a < 6) return SES_NAT_PORT + (a - 4);
    if (a < 8) return SES_ORIG_PORT + (a - 6);
    if (a < 12) return SES_ORIG_IP + (a - 8);
    if (a < 16) return SES_DEST_IP + (a - 12);
    if (a < 20) return SES_DEST_PORT + (a - 16);
    if (a < 24) return SES_PAD_A + (a - 20);
    if (a < 32) return SES_LAST_SEEN + (a - 24);
    if (a < 40) return SES_CREATED + (a - 32);
    if (a < 44) return SES_OUT_LO + (a - 40); // packets_out
    if (a < 48) return SES_OUT_HI + (a - 44);
    if (a < 52) return SES_IN_LO + (a - 48); // packets_in
    if (a < 56) return SES_IN_HI + (a - 52);
    if (a < 60) return SES_OUT_LO + 4 + (a - 56); // bytes_out
    if (a < 64) return SES_OUT_HI + 4 + (a - 60);
    if (a < 68) return SES_IN_LO + 4 + (a - 64); // bytes_in
    if (a < 72) return SES_IN_HI + 4 + (a - 68);
    if (a < 76) return SES_STATE + (a - 72);
    return SES_PAD_B + (a - 76);
}
__host__ __device__ __forceinline__ u32 ses_hi_of(u32 lo_off) { return lo_off == SES_OUT_LO ? (u32)SES_OUT_HI : (u32)SES_IN_HI; }
#ifdef __CUDACC__
// Rare half of ses_touch(): a per-frame clock, and a last_seen that no batch of that clock may have stored — epoch 0:
// the control plane wrote it (bng_map_update, a restore, a hand-over import, a delta), possibly on another host's
// clock — or one that this batch's first frame may be replacing right now (epoch == the batch's).  The reference
// overwrites, so the last frame's `now` must end in last_seen, whatever was there.  The first frame claims the
// epoch (a CAS on the word it shares with nat_port, which no frame changes) and replaces the stored value outright.
// Every other frame records its `now` in the dataplane-only word SES_SIDE first and then raises last_seen; the
// claimer folds SES_SIDE in after its exchange, so a frame whose raise landed before the exchange is not lost.
// SES_SIDE starts at 0 wherever a session is written whole (nat_ses_fill, val_to_slot), and only frames raise it
// after that; the clock is monotonic from batch to batch (include/bng_b200.h), so what it holds from earlier batches
// is never above this batch's frames.
static __device__ __noinline__ void ses_touch_exact(u8 *ses, u64 now, u32 seen, u32 epoch) {
    unsigned long long *ls = (unsigned long long *)(ses + SES_LAST_SEEN), *side = (unsigned long long *)(ses + SES_SIDE);
    if (seen == 0) {
        u32 *pe = (u32 *)(ses + SES_NAT_PORT); // nat_port | epoch << 16
        const u32 cur = *(volatile u32 *)pe;
        if ((cur >> 16) == 0 && atomicCAS(pe, cur, (cur & 0xFFFFu) | (epoch << 16)) == cur) {
            atomicExch(ls, (unsigned long long)now);
            __threadfence();
            const u64 s = *(volatile u64 *)side;
            if (s > now) atomicMax(ls, (unsigned long long)s);
            return;
        }
    }
    atomicMax(side, (unsigned long long)now);
    __threadfence();
    atomicMax(ls, (unsigned long long)now);
}
// session->last_seen = now (bpf/nat44.c:677,881), once per flow and batch: `seen` is the epoch the caller
// read with the probe, `epoch` the current batch's.
// With per-frame timestamps (stamped) the frames of a batch carry different values and the LAST frame's must
// stay.  The clock is monotonic, so that is the maximum of the frames' values and of any earlier batch's stamp
// (a non-zero epoch other than this batch's); anything else takes ses_touch_exact().
__device__ __forceinline__ void ses_touch(u8 *ses, u64 now, u32 seen, u32 epoch, bool stamped = false) {
    if (stamped) {
        if (seen != 0 && seen != epoch)
            atomicMax((unsigned long long *)(ses + SES_LAST_SEEN), (unsigned long long)now);
        else
            ses_touch_exact(ses, now, seen, epoch);
    } else if (seen != epoch) {
        *(u64 *)(ses + SES_LAST_SEEN) = now;
        *(u16 *)(ses + SES_EPOCH) = (u16)epoch;
    }
}
// Rare half of ses_count(): a low word wrapped.  c: the packet word carried into the byte word (undo
// it there, count it in the high packet word); w: the byte word wrapped upwards.  The high words of
// packets and bytes are advanced with one 32-bit atomic each, so neither can carry into the other.
static __device__ __noinline__ void ses_count_carry(u8 *ses, u32 lo_off, u32 c, u32 w) {
    u32 *hi = (u32 *)(ses + ses_hi_of(lo_off)); // hi[0]: packets[63:32], hi[1]: bytes[63:32]
    u32 dbytes = w;
    if (c) {
        u64 old = atomicAdd((unsigned long long *)(ses + lo_off), 0xFFFFFFFF00000000ull); // byte word -= 1
        if ((old >> 32) == 0) dbytes -= 1;                                                // ... which wrapped downwards
        atomicAdd(hi, 1u);
    }
    if (dbytes) atomicAdd(hi + 1, dbytes);
}
// packets += 1, bytes += len on the counter pair at lo_off (SES_OUT_LO / SES_IN_LO): exact u64
// arithmetic, every wrap of a low word is seen by exactly one caller through the value the atomic returns.
__device__ __forceinline__ void ses_count(u8 *ses, u32 lo_off, u32 len) {
    const u64 old = atomicAdd((unsigned long long *)(ses + lo_off), 1ull | ((u64)len << 32));
    const u32 c = (u32)old == 0xFFFFFFFFu;
    const u32 w = (u32)(((old >> 32) + len + c) >> 32);
    if (c | w) ses_count_carry(ses, lo_off, c, w);
}
#endif

// ---------------------------------------------------------------------------
// Subscriber directory: one 16-byte slot per private address that owns a subscriber_nat entry and / or a
// qos_ingress bucket: { u64 key (the address, zero-extended; doubles as the slot state), u32 nat slot,
// u32 qos slot | DIR_QOS_UNLIMITED } with DIR_NONE for "no entry".  Derived state, maintained by the
// table-update kernels (tableops.cu) whenever one of the two maps changes.  The upstream classify kernels
// probe it instead of the two maps (one 128-bit load instead of two probes with a collision loop each),
// and its slot index is the ordering key of the group-by: a dense 2^k key space whatever capacity the two
// maps were opened with.
// ---------------------------------------------------------------------------
#define DIR_NONE 0xFFFFFFFFu
#define DIR_QOS_UNLIMITED 0x80000000u // rate_bps == 0: the bucket never drops and is never written (bpf/qos_ratelimit.c:77-78)
#define DIR_SLOT_MASK 0x7FFFFFFFu

struct LpmTbl { // BPF_MAP_TYPE_LPM_TRIE with a 4-byte address: {prefixlen, addr bytes, value}
    u32 *ents;  // 3 x u32 per entry: prefixlen, addr (memory order), value
    u32 *count;
    u32 max_entries;
};

struct EvRing { // staged event records: {payload, u32 frame index, u32 batch seq}
    u8 *buf;
    u32 *count;
    u32 cap;
    u32 rec_bytes; // payload + 8, a multiple of 16
    u32 lost_stat;
    u32 pad;
};

struct DevCtx {
    Tbl bindings;   // subscriber_bindings      u64 mac   -> 24 B
    Tbl qos_eg;     // qos_egress               u32 ip    -> 32 B token_bucket (at slot+16)
    Tbl qos_in;     // qos_ingress
    Tbl sub_nat;    // subscriber_nat           u32 ip    -> 64 B
    Tbl sessions;   // nat_sessions             16 B      -> 80 B
    Tbl reverse;    // nat_reverse              16 B      -> 16 B
    Tbl eim;        // eim_table                8 B       -> 32 B
    Tbl hairpin;    // hairpin_ips              u32       -> u8
    Tbl alg;        // alg_ports                u32       -> 8 B
    Tbl sub_pools;  // subscriber_pools         u64 mac   -> 25 B
    Tbl vlan_pools; // vlan_subscriber_pools    4 B       -> 25 B
    Tbl cid_subs;   // circuit_id_subscribers   32 B      -> 25 B
    Tbl ip_pools;   // ip_pools                 u32       -> 28 B
    Tbl cid_map;    // circuit_id_map           u64       -> u64 (never read by a program)
    Tbl subdir;     // derived: private address -> {subscriber_nat slot, qos_ingress slot}
    LpmTbl ranges_v4;  // allowed_ranges_v4
    LpmTbl priv_ranges; // nat_private_ranges (never read by a program)
    u8 *as_config;     // antispoof_config[1]   8 B
    u8 *nat_config;    // nat_config_map[1]     16 B
    u8 *server_config; // server_config[1]      16 B
    u8 *nat_pool;      // nat_pool[256]         16 B each (never read by a program)
    u64 *stats;        // ST_COUNT counters
    EvRing spoof_ev;   // spoof_events, payload 56 B
    EvRing natlog_ev;  // nat_log_rb,   payload 40 B
    const struct SmallTabs *small; // compact image of the tiny read-mostly maps (TMA-staged into shared memory)
    u32 batch_seq;
    u32 epoch; // (batch_seq % 65535) + 1: what ses_touch() stamps (0 = never)
};

// Compact image of the maps that every frame consults but only the control
// plane writes: antispoof_config, nat_config_map.flags, alg_ports (<= 64
// entries) and hairpin_ips (<= 1000 entries, as a 2048-slot u32 hash).  The
// host rebuilds it on every update of one of those maps; kernels bulk-copy it
// into shared memory (cp.async.bulk + mbarrier) at block start.
#define HP_SLOTS 2048
#define HP_EMPTY 0xFFFFFFFFu
struct __align__(16) SmallTabs {
    u32 as_cfg;    // default_mode | log_violations << 8
    u32 nat_flags; // nat_config.flags
    u32 alg_n;
    u32 hp_n;
    u32 alg_key[64];  // (port << 16) | protocol, as the alg_ports key
    u8 alg_type[64];  // alg_config.alg_type
    u32 hp_hash[HP_SLOTS];
};
static_assert(sizeof(SmallTabs) % 16 == 0, "bulk copies move multiples of 16 bytes");

__host__ __device__ __forceinline__ u32 hp_index(u32 ip) { return (ip * 0x9E3779B1u) >> 21; }

// one batch, device view
struct DevBatch {
    u8 *pkts;
    const u32 *off16;
    u32 *len;
    u8 *verdict;
    u32 *priority;
    u32 n;
    u32 stride;
    u64 now;
    u32 base; // index of frame 0 within the caller's batch (event records carry base + i)
    // Bytes of a frame that are physically present in its slot (0 = the whole frame): the programs'
    // bounds checks run against min(len, cap) — the linear data area, data_end - data in the reference —
    // while byte counters use len (skb->len).  Fixed-stride arenas have cap = stride, so a frame whose
    // length claims more than its slot holds (a header-split receive ring) is parsed as far as the slot
    // goes and can never reach into its neighbour.
    u32 cap;
    u64 arena_len; // bytes addressable from pkts (0 = unknown: no access may run past a frame's 16-byte chunks)
    const u64 *nowv; // per-frame bpf_ktime_get_ns() (monotonic), or nullptr: `now` for every frame
    // Ordering keys carry the frame length above bit `kshift` (0: they do not), so that the ordered phase reads a
    // subscriber's (key, frame, length) with two coalesced loads instead of gathering len[frame] afterwards.
    u32 kshift;
};
// First statement (before any global access) of a kernel launched with programmatic stream serialisation
// (kernels.cu: launch_dep): returns when the preceding grid of the stream has completed and its writes are visible.
// A no-op in a kernel launched the ordinary way.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
// key | min(len, KEY_LEN_SAT) << KEY_BITS: 21 key bits hold the largest directory / bucket table of the reference's
// capacities (2 x 1 M slots); 11 bits hold the length of every frame but a jumbo (KEY_LEN_SAT: "look it up";
// 0x7FF is never written, so a packed key cannot read as NO_KEY).  Tables beyond 2^21 slots: no packing.
#define KEY_BITS 21
#define KEY_LEN_SAT 0x7FEu
__host__ __device__ __forceinline__ u32 key_mask_of(u32 kshift) { return kshift ? (1u << kshift) - 1 : 0xFFFFFFFFu; }
__device__ __forceinline__ u32 key_pack(u32 key, u32 len, u32 kshift) {
    return kshift ? key | ((len < KEY_LEN_SAT ? len : KEY_LEN_SAT) << kshift) : key;
}
// may the 64 bytes at p be read with 32-byte accesses?
#define FRAME_WIDE_OK(b, p) ((((uintptr_t)(p)) & 31) == 0 && (u64)((p) - (b).pkts) + 64 <= (b).arena_len)

// ---------------------------------------------------------------------------
// small helpers
// ---------------------------------------------------------------------------
__host__ __device__ __forceinline__ u64 mix64(u64 x) {
    x ^= x >> 33;
    x *= 0xff51afd7ed558ccdull;
    x ^= x >> 33;
    x *= 0xc4ceb9fe1a85ec53ull;
    x ^= x >> 33;
    return x;
}

__host__ __device__ __forceinline__ u64 splitmix64(u64 x) {
    x += 0x9e3779b97f4a7c15ull;
    x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ull;
    x = (x ^ (x >> 27)) * 0x94d049bb133111ebull;
    return x ^ (x >> 31);
}

__device__ __forceinline__ u16 bswap16(u16 x) { return (u16)((x << 8) | (x >> 8)); }
__device__ __forceinline__ u32 bswap32(u32 x) { return __byte_perm(x, 0, 0x0123); }

// 32-bit multiply/xorshift hash of the key words (cheap on the integer pipes;
// slot placement is an internal matter, not part of the ABI).
__device__ __forceinline__ u32 hash_word(u64 k, u32 seed) {
    u32 h = ((u32)k * 0x9E3779B1u) ^ ((u32)(k >> 32) * 0x85EBCA77u) ^ seed;
    h ^= h >> 16;
    h *= 0x7FEB352Du;
    h ^= h >> 15;
    return h;
}

template <int KW>
__device__ __forceinline__ u32 tbl_hash(const u64 *k) {
    u32 h = 0x2545F491u;
#pragma unroll
    for (int i = 0; i < KW; i++) h = hash_word(k[i], h);
    return h;
}

__device__ __forceinline__ u8 *tbl_slot(const Tbl &t, u32 i) { return t.slots + (size_t)i * t.slot_bytes; }

__device__ __forceinline__ u64 ld_vol64(const u8 *p) { return *(volatile const u64 *)p; }

// Find the slot holding key k (KW 64-bit words), or nullptr.  VOL selects
// L1-bypassing loads of the state word, needed in kernels that insert
// concurrently.
// SKIP_BUSY: a slot another thread is filling right now is stepped over instead of waited for.  Legal
// wherever a key can only be inserted by the thread that looks it up (the ordered phase: every flow
// key belongs to one subscriber, every subscriber to one worker) — and necessary there, because the
// workers of 32 subscribers share a warp and a lane must never wait for another lane of its own warp.
template <int KW, bool VOL, bool SKIP_BUSY = false>
__device__ __forceinline__ u8 *tbl_find(const Tbl &t, const u64 *k) {
    if (k[0] >= K_BUSY) return nullptr;
    u32 i = (u32)tbl_hash<KW>(k) & t.home_mask;
    for (u32 probe = 0; probe <= t.mask; probe++) {
        u8 *s = tbl_slot(t, i);
        u64 w0 = VOL ? ld_vol64(s) : *(const u64 *)s;
        if (VOL && !SKIP_BUSY) {
            while (w0 == K_BUSY) {
                __nanosleep(32);
                w0 = ld_vol64(s);
            }
        }
        if (w0 == K_EMPTY) return nullptr;
        if (w0 == k[0]) {
            bool eq = true;
#pragma unroll
            for (int j = 1; j < KW; j++) eq = eq && (((const u64 *)s)[j] == k[j]);
            if (eq) return s;
        }
        i = (i + 1) & t.mask;
    }
    return nullptr;
}

// Approximate LRU eviction (the kernel's LRU hash is approximate too: per-CPU lists, batched promotion): when
// an LRU map is at max_entries, one of the LRU_WINDOW slots following the new key's home slot gives way —
// the one least recently used by its timestamp.  The victim becomes a tombstone; whatever still refers to it
// (a nat_reverse entry whose session went, an EIM reference) is dealt with the way the reference deals with
// entries the kernel evicted underneath it (stale-reverse path, bpf/nat44.c:871-876).
__device__ __forceinline__ bool tbl_evict_near(const Tbl &t, u32 home, u64 *stats) {
    const u32 mode = t.lru & 0xff, ts_off = t.lru >> 8;
    // Many workers insert at once when a batch brings more new flows than the table holds: a victim may be taken by
    // somebody else between the scan and the CAS, and a window may hold no live entry at all.  Try again, moving on.
    for (u32 attempt = 0; attempt < 16; attempt++) {
        u8 *best = nullptr;
        u64 best_ts = ~0ull, best_w = 0;
        for (u32 j = 0; j < LRU_WINDOW; j++) {
            u8 *s = t.slots + (size_t)((home + (attempt >> 1) * LRU_WINDOW + j) & t.mask) * t.slot_bytes;
            const u64 w0 = *(volatile const u64 *)s;
            if (w0 >= K_BUSY) continue;
            const u64 ts = mode == LRU_TS ? *(volatile const u64 *)(s + ts_off) : j;
            if (ts < best_ts) {
                best_ts = ts;
                best = s;
                best_w = w0;
            }
        }
        if (best && atomicCAS((u64 *)best, best_w, K_TOMB) == best_w) {
            atomicSub(t.count, 1u);
            if (stats) atomicAdd(&stats[ST_LRU_EVICT], 1ull);
            return true;
        }
    }
    return false;
}

// tbl_find that also reports where an insert of k would go: *ins = index of the first tombstone on the probe path,
// else of the EMPTY slot that ended it (0xFFFFFFFF: none seen).  A following tbl_claim_at() then costs one CAS
// instead of a second walk.  SKIP_BUSY semantics (ordered phase: a key has one owner).
// The state words of PROBE_W consecutive slots are requested together: in a table that lives in DRAM every probe
// step is a full memory round trip, and the longest chain among a warp's 32 lanes (3-4 steps at load 0.25) costs
// that many round trips per lookup.  Every speculative slot is a 64-byte DRAM burst, though, and the cold-start
// kernel is bound by the rate of scattered DRAM bursts, so the window stays narrow.
#define PROBE_W 2
template <int KW>
__device__ __forceinline__ u8 *tbl_find_ins(const Tbl &t, const u64 *k, u32 *ins) {
    *ins = 0xFFFFFFFFu;
    if (k[0] >= K_BUSY) return nullptr;
    u32 i = (u32)tbl_hash<KW>(k) & t.home_mask;
    for (u32 probe = 0; probe <= t.mask; probe += PROBE_W) {
        u64 w[PROBE_W];
#pragma unroll
        for (int j = 0; j < PROBE_W; j++) w[j] = ld_vol64(tbl_slot(t, (i + j) & t.mask));
#pragma unroll
        for (int j = 0; j < PROBE_W; j++) {
            const u32 si = (i + j) & t.mask;
            if (w[j] == K_EMPTY) {
                if (*ins == 0xFFFFFFFFu) *ins = si;
                return nullptr;
            }
            if (w[j] == K_TOMB && *ins == 0xFFFFFFFFu) *ins = si;
            if (w[j] == k[0]) {
                u8 *s = tbl_slot(t, si);
                bool eq = true;
#pragma unroll
                for (int q = 1; q < KW; q++) eq = eq && (((volatile const u64 *)s)[q] == k[q]);
                if (eq) return s;
            }
        }
        i = (i + PROBE_W) & t.mask;
    }
    return nullptr;
}
// Existence test with the same windowed probing (allocate_port_from_block()'s collision check, bpf/nat44.c:450-455)
template <int KW>
__device__ __forceinline__ bool tbl_has(const Tbl &t, const u64 *k) {
    u32 ins;
    return tbl_find_ins<KW>(t, k, &ins) != nullptr;
}
// Claims slot `ins` (as reported by tbl_find_ins for a key that was absent) for k: EMPTY/TOMB -> BUSY with one
// CAS, key words 1.. written; nullptr when somebody else took the slot meanwhile (the caller then walks again
// with tbl_find_or_claim).  The caller has already reserved the entry in t.count (tbl_reserve).
template <int KW>
__device__ __forceinline__ u8 *tbl_claim_at(const Tbl &t, u32 ins, const u64 *k) {
    if (ins == 0xFFFFFFFFu) return nullptr;
    u8 *s = tbl_slot(t, ins);
    const u64 got = atomicCAS((u64 *)s, K_EMPTY, K_BUSY); // (the slot was EMPTY a moment ago, more often than a tombstone)
    if (got != K_EMPTY && !(got == K_TOMB && atomicCAS((u64 *)s, K_TOMB, K_BUSY) == K_TOMB)) return nullptr;
#pragma unroll
    for (int j = 1; j < KW; j++) ((u64 *)s)[j] = k[j];
    return s;
}
// The first step of three claims at once (the three atomics are independent: one round trip, not three).  got[] =
// what each CAS returned; a slot index of 0xFFFFFFFF is skipped (got = K_BUSY: "not claimed").
__device__ __forceinline__ void tbl_cas3(const Tbl &a, u32 ia, const Tbl &b, u32 ib, const Tbl &c, u32 ic, u64 got[3]) {
    got[0] = got[1] = got[2] = K_BUSY;
    if (ia != 0xFFFFFFFFu) got[0] = atomicCAS((u64 *)tbl_slot(a, ia), K_EMPTY, K_BUSY);
    if (ib != 0xFFFFFFFFu) got[1] = atomicCAS((u64 *)tbl_slot(b, ib), K_EMPTY, K_BUSY);
    if (ic != 0xFFFFFFFFu) got[2] = atomicCAS((u64 *)tbl_slot(c, ic), K_EMPTY, K_BUSY);
}
// ... and the rest of one of them: the slot is ours when the CAS found it EMPTY, or when it was a tombstone and a
// second CAS takes that; key words 1.. are then written.
template <int KW>
__device__ __forceinline__ u8 *tbl_claim_finish(const Tbl &t, u32 ins, u64 got, const u64 *k) {
    if (ins == 0xFFFFFFFFu) return nullptr;
    u8 *s = tbl_slot(t, ins);
    if (got != K_EMPTY && !(got == K_TOMB && atomicCAS((u64 *)s, K_TOMB, K_BUSY) == K_TOMB)) return nullptr;
#pragma unroll
    for (int j = 1; j < KW; j++) ((u64 *)s)[j] = k[j];
    return s;
}

// Reserves room for n new entries: true when they fit under max_entries (t.count then includes them; give back
// what is not used with tbl_unreserve).  One atomic for a whole chunk of inserts, and exact: the count can never
// overshoot max_entries, however many warps insert at once.
__device__ __forceinline__ bool tbl_reserve(const Tbl &t, u32 n) {
    if (atomicAdd(t.count, n) + n > t.max_entries) {
        atomicSub(t.count, n);
        return false;
    }
    return true;
}
__device__ __forceinline__ void tbl_unreserve(const Tbl &t, u32 n) {
    if (n) atomicSub(t.count, n);
}

// tbl_find for code that goes on for hundreds of instructions after the lookup: the lanes that entered together
// leave together (lanes whose probe ended wait for the longest chain), so what follows runs once for the warp, not
// once per distinct chain length — without it the compiler's tail duplication can make dhcp_fastpath execute its
// body several times per warp with few lanes active.  Read-only tables.
template <int KW>
__device__ __forceinline__ const u8 *tbl_find_conv(const Tbl &t, const u64 *k) {
    const unsigned m = __activemask();
    const u8 *res = nullptr;
    bool done = k[0] >= K_BUSY;
    u32 i = (u32)tbl_hash<KW>(k) & t.home_mask, left = t.mask + 1;
    while (__any_sync(m, !done)) {
        if (!done) {
            const u8 *s = tbl_slot(t, i);
            const u64 w0 = *(const u64 *)s;
            if (w0 == K_EMPTY) {
                done = true;
            } else {
                bool eq = w0 == k[0];
#pragma unroll
                for (int j = 1; j < KW; j++) eq = eq && (((const u64 *)s)[j] == k[j]);
                if (eq) {
                    res = s;
                    done = true;
                } else {
                    i = (i + 1) & t.mask;
                    done = --left == 0;
                }
            }
        }
    }
    return res;
}

// Find-or-claim.  Returns the slot; *created says whether this call claimed
// it.  A claimed slot is left in the K_BUSY state with key words 1.. written:
// the caller fills the value and then calls tbl_publish().  Returns nullptr
// when the table is full (max_entries reached or no free slot).
// `pending` (optional): the caller batches its live-entry accounting — the claim is checked against
// count + *pending and counted in *pending, and the caller adds *pending to t.count once (one global
// atomic per warp instead of one per insert, which on a million-insert batch is the difference
// between a same-address atomic storm and none).  The max_entries check is then approximate by at
// most the inserts in flight, which only matters for the LRU maps at the very edge of capacity.
// RESERVED: the caller holds a reservation for the entry (tbl_reserve): no accounting, no max_entries check here.
template <int KW, bool SKIP_BUSY = false, bool RESERVED = false>
__device__ __forceinline__ u8 *tbl_find_or_claim(const Tbl &t, const u64 *k, bool *created, u32 *pending = nullptr,
                                                 u64 *stats = nullptr) {
    *created = false;
    if (k[0] >= K_BUSY) return nullptr;
    const u32 home = (u32)tbl_hash<KW>(k) & t.home_mask;
    u32 i = home;
    int tomb = -1;
    for (u32 probe = 0; probe <= t.mask + 1;) {
        // one step past the last slot: the table has no EMPTY slot left on this path (churn turned them all into
        // tombstones); the key is not there, and the first tombstone seen takes it
        const bool wrapped = probe == t.mask + 1;
        if (wrapped && tomb < 0) return nullptr;
        u8 *s = tbl_slot(t, i);
        u64 w0 = wrapped ? K_EMPTY : ld_vol64(s);
        while (!SKIP_BUSY && w0 == K_BUSY) {
            __nanosleep(32);
            w0 = ld_vol64(s);
        }
        if (w0 == k[0]) {
            bool eq = true;
#pragma unroll
            for (int j = 1; j < KW; j++) eq = eq && (((volatile const u64 *)s)[j] == k[j]);
            if (eq) return s;
        }
        if (w0 == K_TOMB && tomb < 0) tomb = (int)i;
        if (w0 == K_EMPTY) {
            u32 target = tomb >= 0 ? (u32)tomb : i;
            u64 expect = tomb >= 0 ? K_TOMB : K_EMPTY;
            u8 *ts = tbl_slot(t, target);
            if (RESERVED) {
            } else if (pending) {
                if (*(volatile u32 *)t.count + *pending >= t.max_entries && !(t.lru && tbl_evict_near(t, home, stats))) return nullptr;
            } else if (atomicAdd(t.count, 1u) >= t.max_entries) {
                if (!(t.lru && tbl_evict_near(t, home, stats))) { // (the victim's count goes, ours stays)
                    atomicSub(t.count, 1u);
                    return nullptr;
                }
            }
            u64 old = atomicCAS((u64 *)ts, expect, K_BUSY);
            if (old == expect) {
#pragma unroll
                for (int j = 1; j < KW; j++) ((u64 *)ts)[j] = k[j];
                *created = true;
                if (pending) ++*pending;
                return ts;
            }
            // lost the race for that slot: undo the reservation and look again
            if (!pending && !RESERVED) atomicSub(t.count, 1u);
            if (tomb >= 0 || wrapped) {
                tomb = -1;
                i = home;
                probe = 0;
            }
            continue; // re-examine the same slot (it may now hold our key)
        }
        i = (i + 1) & t.mask;
        probe++;
    }
    return nullptr;
}

// FENCE orders the value stores before the key for readers in other warps.  The ordered phase publishes
// without it: a flow key is only ever looked up by the worker that inserted it (other workers step over
// the slot whatever its state), lanes of one warp are ordered by __syncwarp(), and the kernel boundary
// orders everything for whoever comes next — three device-wide fences per new flow were 40 % of a
// cold-start batch.
template <bool FENCE = true>
__device__ __forceinline__ void tbl_publish(u8 *slot, u64 k0) {
    if (FENCE) __threadfence();
    *(volatile u64 *)slot = k0;
}

template <int KW>
__device__ __forceinline__ bool tbl_erase(const Tbl &t, const u64 *k) {
    u8 *s = tbl_find<KW, true>(t, k);
    if (!s) return false;
    u64 old = atomicCAS((u64 *)s, k[0], K_TOMB);
    if (old != k[0]) return false;
    atomicSub(t.count, 1u);
    return true;
}

// longest-prefix match over 4 address bytes in memory order (byte 0 first),
// as BPF_MAP_TYPE_LPM_TRIE compares them.  `addr` is the little-endian load of
// those bytes.  Returns true when any entry with prefixlen <= maxlen matches.
__device__ __forceinline__ bool lpm_match(const LpmTbl &t, u32 addr, u32 maxlen) {
    u32 n = *t.count;
    u32 a = bswap32(addr); // byte 0 becomes the most significant
    for (u32 i = 0; i < n; i++) {
        u32 pl = t.ents[3 * i];
        if (pl > maxlen) continue;
        u32 e = bswap32(t.ents[3 * i + 1]);
        u32 m = pl == 0 ? 0u : (0xFFFFFFFFu << (32 - pl));
        if (((a ^ e) & m) == 0) return true;
    }
    return false;
}

// ---------------------------------------------------------------------------
// subscriber_ipv6: IPv6 prefix -> subscriber IPv4 address, an exact-match hash of (prefixlen, masked prefix) keys
// probed once per prefix length in use, longest first.  The 20-byte key {u32 prefixlen; u8 addr[16]} (the layout of
// a BPF_MAP_TYPE_LPM_TRIE key) is stored in three key words, the last one's high half zero; the u32 value sits at 24.
// A 32-byte slot: one probe is one sector.  An address is handled as four little-endian words of its bytes in memory
// order (a[0] holds bytes 0-3, as rd32 loads them).
// ---------------------------------------------------------------------------
#define LPM6_KEY 20u
#define LPM6_KW 3
#define LPM6_LENS 129u
// the first `keep` bits (network order) of a little-endian word of address bytes
__host__ __device__ __forceinline__ u32 lpm6_keep(u32 w, int keep) {
    if (keep <= 0) return 0;
    if (keep >= 32) return w;
    const u32 m = 0xFFFFFFFFu << (32 - keep); // in numeric (big-endian) order; byte-swapped to memory order below
    const u32 ml = (m >> 24) | ((m >> 8) & 0xFF00u) | ((m << 8) & 0xFF0000u) | (m << 24);
    return w & ml;
}
// key words of (len, the address's first len bits)
__host__ __device__ __forceinline__ void lpm6_key(u64 *kw, u32 len, const u32 *a) {
    const int l = (int)len;
    kw[0] = (u64)len | (u64)lpm6_keep(a[0], l) << 32;
    kw[1] = (u64)lpm6_keep(a[1], l - 32) | (u64)lpm6_keep(a[2], l - 64) << 32;
    kw[2] = (u64)lpm6_keep(a[3], l - 96);
}

// ---------------------------------------------------------------------------
// per-block statistics: counters accumulate in shared memory and are flushed
// with one global atomic per non-zero counter per block.
// ---------------------------------------------------------------------------
struct BlockStats {
    u64 v[ST_COUNT];
};

__device__ __forceinline__ void bstats_init(BlockStats &s) {
    for (int i = threadIdx.x; i < ST_COUNT; i += blockDim.x) s.v[i] = 0;
    __syncthreads();
}
__device__ __forceinline__ void bstats_add(BlockStats &s, int idx, u64 v) { atomicAdd(&s.v[idx], v); }
__device__ __forceinline__ void bstats_flush(BlockStats &s, u64 *g) {
    __syncthreads();
    for (int i = threadIdx.x; i < ST_COUNT; i += blockDim.x)
        if (s.v[i]) atomicAdd(&g[i], s.v[i]);
}

// Flush a per-thread register counter: warp reduction, one shared atomic per
// warp.  Must be reached by all 32 lanes.
__device__ __forceinline__ void warp_stat_flush(BlockStats &s, int idx, u32 v) {
    u32 t = __reduce_add_sync(0xffffffffu, v);
    if ((threadIdx.x & 31) == 0 && t) atomicAdd(&s.v[idx], (u64)t);
}
__device__ __forceinline__ void warp_stat_flush64(BlockStats &s, int idx, u64 v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0 && v) atomicAdd(&s.v[idx], v);
}

// Warp-aggregated increment of a shared counter: one shared atomic per warp.
__device__ __forceinline__ void bstats_inc_pred(BlockStats &s, int idx, bool pred) {
    unsigned m = __ballot_sync(__activemask(), pred);
    if (pred) {
        int leader = __ffs(m) - 1;
        if ((threadIdx.x & 31) == leader) atomicAdd(&s.v[idx], (u64)__popc(m));
    }
}

// ---------------------------------------------------------------------------
// event staging
// ---------------------------------------------------------------------------
__device__ __forceinline__ u8 *ev_reserve(const DevCtx &c, const EvRing &r, u32 frame_idx) {
    u32 pos = atomicAdd(r.count, 1u);
    if (pos >= r.cap) {
        atomicSub(r.count, 1u);
        atomicAdd(&c.stats[r.lost_stat], 1ull);
        return nullptr;
    }
    u8 *rec = r.buf + (size_t)pos * r.rec_bytes; // 16-byte aligned payload first, tag last
    *(uint2 *)(rec + r.rec_bytes - 8) = make_uint2(frame_idx, c.batch_seq);
    return rec;
}

// ---------------------------------------------------------------------------
// frame access.  Frames start on 16-byte boundaries; all multi-byte fields
// are read the way the eBPF programs read them: little-endian loads of wire
// bytes.  Even offsets are 2-byte aligned, so u16 accesses are always legal.
// ---------------------------------------------------------------------------
__device__ __forceinline__ u64 frame_now(const DevBatch &b, u32 i) { return b.nowv ? b.nowv[i] : b.now; }
__device__ __forceinline__ u32 frame_dlen(const DevBatch &b, u32 len) { return (b.cap && len > b.cap) ? b.cap : len; }
__device__ __forceinline__ u8 *frame_ptr(const DevBatch &b, u32 i) {
    return b.pkts + (b.off16 ? (size_t)b.off16[i] * 16 : (size_t)i * b.stride);
}
__device__ __forceinline__ u16 rd16(const u8 *p, u32 off) { return *(const u16 *)(p + off); }
__device__ __forceinline__ u32 rd32(const u8 *p, u32 off) {
    return (u32)rd16(p, off) | ((u32)rd16(p, off + 2) << 16);
}
__device__ __forceinline__ void wr16(u8 *p, u32 off, u16 v) { *(u16 *)(p + off) = v; }
__device__ __forceinline__ void wr32(u8 *p, u32 off, u32 v) {
    wr16(p, off, (u16)v);
    wr16(p, off + 2, (u16)(v >> 16));
}

// The first 64 bytes of a frame held in registers (16 little-endian words).
struct Hdr64 {
    u32 w[16];
    __device__ __forceinline__ u8 b8(u32 off) const { return (u8)(w[off >> 2] >> ((off & 3) * 8)); }
    __device__ __forceinline__ u16 b16(u32 off) const { // off even
        return (u16)(w[off >> 2] >> ((off & 2) * 8));
    }
    __device__ __forceinline__ u32 b32(u32 off) const { // off even
        return (off & 2) ? (u32)(w[off >> 2] >> 16) | (w[(off >> 2) + 1] << 16) : w[off >> 2];
    }
    __device__ __forceinline__ void s16(u32 off, u16 v) {
        u32 sh = (off & 2) * 8;
        w[off >> 2] = (w[off >> 2] & ~(0xFFFFu << sh)) | ((u32)v << sh);
    }
    __device__ __forceinline__ void s32(u32 off, u32 v) {
        s16(off, (u16)v);
        s16(off + 2, (u16)(v >> 16));
    }
};

// Loads the 16-byte chunks of the frame that contain bytes < min(len, 64).
__device__ __forceinline__ void hdr_load(Hdr64 &h, const u8 *p, u32 len) {
#pragma unroll
    for (int c = 0; c < 4; c++) {
        uint4 v = make_uint4(0, 0, 0, 0);
        if ((u32)c * 16 < len) v = *(const uint4 *)(p + c * 16);
        h.w[4 * c + 0] = v.x;
        h.w[4 * c + 1] = v.y;
        h.w[4 * c + 2] = v.z;
        h.w[4 * c + 3] = v.w;
    }
}
__device__ __forceinline__ void hdr_store_chunk(const Hdr64 &h, u8 *p, int c) {
    *(uint4 *)(p + c * 16) = make_uint4(h.w[4 * c], h.w[4 * c + 1], h.w[4 * c + 2], h.w[4 * c + 3]);
}

// 32-byte global accesses: one whole sector per lane, issued as two back-to-back 128-bit accesses (the
// widest global load/store sm_90 has: LDG/STG.E.128).  Both halves are issued before either result is
// used, so a sector costs one round trip and is never fetched piecemeal across dependent loads.
// p must be 32-byte aligned.
struct __align__(16) U256 {
    u32 w[8];
};
// Each half is one inline-asm ld/st.global.v4.u32 with the default L2 policy (DESIGN.md §5 has the eviction
// hints that were measured and not kept).
#define BNG_LDG128(r, q)                                                                                         \
    asm volatile("ld.global.v4.u32 {%0,%1,%2,%3}, [%4];"                                                         \
                 : "=r"((r)[0]), "=r"((r)[1]), "=r"((r)[2]), "=r"((r)[3])                                        \
                 : "l"(q)                                                                                        \
                 : "memory")
#define BNG_STG128(q, w)                                                                                         \
    asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(q), "r"((w)[0]), "r"((w)[1]), "r"((w)[2]),         \
                 "r"((w)[3])                                                                                     \
                 : "memory")
__device__ __forceinline__ U256 ldg256(const void *p) {
    U256 r;
    const u8 *q = (const u8 *)p;
    BNG_LDG128(&r.w[0], q);
    BNG_LDG128(&r.w[4], q + 16);
    return r;
}
__device__ __forceinline__ void stg256(void *p, const u32 *w) {
    u8 *q = (u8 *)p;
    BNG_STG128(q, &w[0]);
    BNG_STG128(q + 16, &w[4]);
}
#undef BNG_LDG128
#undef BNG_STG128
// Frame header load: two 32-byte loads when the whole warp's frames allow it (32-byte aligned and 64
// bytes inside the arena), 16-byte chunks otherwise.  `wide` must be warp-uniform.
__device__ __forceinline__ void hdr_load_wide(Hdr64 &h, const u8 *p, u32 len, bool wide) {
    if (wide) {
        U256 a, b;
#pragma unroll
        for (int k = 0; k < 8; k++) a.w[k] = b.w[k] = 0;
        if (len > 0) a = ldg256(p);
        if (len > 32) b = ldg256(p + 32);
#pragma unroll
        for (int k = 0; k < 8; k++) {
            h.w[k] = a.w[k];
            h.w[8 + k] = b.w[k];
        }
    } else {
        hdr_load(h, p, len);
    }
}

// MAC bytes [off, off+6) as the reference's big-endian u64 key
// (bpf/antispoof.c:122-129, bpf/dhcp_fastpath.c:175-182).
__device__ __forceinline__ u64 mac_key(const Hdr64 &h, u32 off) {
    if (off == 6) // the source MAC: bytes 6-7 are the high half of word 1, bytes 8-11 word 2; two byte permutes
        return ((u64)__byte_perm(h.w[1], 0, 0x4423) << 32) | __byte_perm(h.w[2], 0, 0x0123);
    u64 k = 0;
#pragma unroll
    for (int i = 0; i < 6; i++) k = (k << 8) | h.b8(off + i);
    return k;
}

// RFC 1624-style incremental checksum helpers, op-for-op as bpf/nat44.c:378-398.
__device__ __forceinline__ u16 csum_fold32(u32 c) {
    c = (c & 0xffff) + (c >> 16);
    c = (c & 0xffff) + (c >> 16);
    return (u16)~c;
}
__device__ __forceinline__ u16 csum_upd32(u16 csum, u32 old_val, u32 new_val) {
    u32 sum = ~((u32)csum) & 0xffff;
    sum += ~old_val & 0xffff;
    sum += ~(old_val >> 16) & 0xffff;
    sum += new_val & 0xffff;
    sum += new_val >> 16;
    return csum_fold32(sum);
}
__device__ __forceinline__ u16 csum_upd16(u16 csum, u16 old_val, u16 new_val) {
    u32 sum = ~((u32)csum) & 0xffff;
    sum += ~(u32)old_val & 0xffff;
    sum += (u32)new_val & 0xffff;
    return csum_fold32(sum);
}

// ---------------------------------------------------------------------------
// TMA bulk copy of a small global image into shared memory (sm_90):
// one thread arms an mbarrier with the byte count and issues cp.async.bulk;
// everyone waits on the barrier's phase 0.
// ---------------------------------------------------------------------------
__device__ __forceinline__ void smem_stage_begin(void *smem_dst, const void *gsrc, u32 bytes, u64 *bar) {
    if (threadIdx.x == 0) {
        u32 bar_a = (u32)__cvta_generic_to_shared(bar);
        u32 dst_a = (u32)__cvta_generic_to_shared(smem_dst);
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar_a));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_a), "r"(bytes) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_a),
                     "l"(gsrc), "r"(bytes), "r"(bar_a)
                     : "memory");
    }
    __syncthreads(); // the barrier is initialised before anyone polls it
}
__device__ __forceinline__ void smem_stage_wait(u64 *bar) {
    u32 bar_a = (u32)__cvta_generic_to_shared(bar);
    u32 done = 0;
    while (!done) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(bar_a)
            : "memory");
    }
}

__device__ __forceinline__ bool hp_contains(const SmallTabs &st, u32 ip) {
    if (ip == HP_EMPTY) return (st.hp_n >> 31) != 0;
    if ((st.hp_n & 0x7fffffffu) == 0) return false;
    u32 i = hp_index(ip);
    for (u32 probe = 0; probe < HP_SLOTS; probe++) {
        u32 v = st.hp_hash[i];
        if (v == ip) return true;
        if (v == HP_EMPTY) return false;
        i = (i + 1) & (HP_SLOTS - 1);
    }
    return false;
}
__device__ __forceinline__ int alg_find(const SmallTabs &st, u32 key) { // index into alg_type[] or -1
    for (u32 i = 0; i < st.alg_n; i++)
        if (st.alg_key[i] == key) return (int)i;
    return -1;
}

// Continue a probe whose first slot (index i0) has already been fetched:
// w0 is that slot's state word, rest_eq whether the remaining key words
// matched.  Read-only tables (no concurrent inserts in this kernel).
template <int KW>
__device__ __forceinline__ u8 *tbl_finish(const Tbl &t, const u64 *k, u32 i0, u64 w0, bool rest_eq) {
    if (k[0] >= K_BUSY) return nullptr;
    if (w0 == k[0] && rest_eq) return tbl_slot(t, i0);
    if (w0 == K_EMPTY) return nullptr;
    u32 i = (i0 + 1) & t.mask;
    for (u32 probe = 1; probe <= t.mask; probe++) {
        u8 *s = tbl_slot(t, i);
        u64 w = *(const u64 *)s;
        if (w == K_EMPTY) return nullptr;
        if (w == k[0]) {
            bool eq = true;
#pragma unroll
            for (int j = 1; j < KW; j++) eq = eq && (((const u64 *)s)[j] == k[j]);
            if (eq) return s;
        }
        i = (i + 1) & t.mask;
    }
    return nullptr;
}
