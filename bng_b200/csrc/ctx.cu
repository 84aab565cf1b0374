// bng_b200 — C-ABI layer (include/bng_b200.h): context, map registry with the
// reference's map names / key / value layouts, control-plane map commands,
// batch program runs, event drain.  Everything that touches table or frame
// contents is a CUDA kernel; this file only moves bytes and launches.
#include <errno.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#include <dlfcn.h>
#include <sys/mman.h>

#include <nccl.h> // types only: the library is resolved at run time (bng_comm_init), never linked

#include <algorithm>
#include <mutex>
#include <string>
#include <string_view>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "../../include/bng_b200.h"
#include "blob.hpp"
#include "devbuf.hpp"
#include "kernels.h"

namespace {

enum Kind { KIND_HASH, KIND_ARRAY, KIND_STATS, KIND_LPM, KIND_EVENT };

// bpf_map_type values the reference declares
enum { T_HASH = 1, T_ARRAY = 2, T_PERF = 4, T_PERCPU_ARRAY = 6, T_LRU = 9, T_LPM = 11, T_RINGBUF = 27 };

struct MapReg {
    const char *name;
    u32 type, key_size, value_size, max_entries;
    Kind kind;
    Tbl *tbl;          // KIND_HASH: descriptor inside dev
    u8 **arr;          // KIND_ARRAY: device base pointer
    int stat_base;     // KIND_STATS
    LpmTbl *lpm;       // KIND_LPM
    EvRing *ring;      // KIND_EVENT
    u32 ev_payload;    // KIND_EVENT
    std::vector<u32> lpm_host; // KIND_LPM: authoritative host copy (3 x u32 per entry)
    std::vector<u8> ev_pending; // KIND_EVENT: ordered, capacity-filtered payloads not yet drained
};

thread_local std::string g_open_err;

} // namespace

// buffers of the zero-copy pipeline: three stages (in, compute, out) in flight need three
#define ZC_BUFS 3

struct bng_ctx {
    std::mutex mu;
    int device = 0;
    DevCtx dev{};
    Launcher L{};
    std::vector<MapReg> maps;
    std::vector<void *> allocs;
    std::string err;
    // the batch arrays that L.s points into (ensure_scratch)
    DevBuf<u32> key_a, key_b, val_a, val_b, qslot, attr;
    DevBuf<u8> cub_tmp;
    // staging for control-plane commands
    DevBuf<u8> io_dev;
    PinnedBuf<u8> io_host;
    // staging for BNG_MEM_HOST batches
    DevBuf<u8> hb_pkts;
    DevBuf<u32> hb_off, hb_len, hb_prio;
    DevBuf<u64> hb_now;
    DevBuf<u8> hb_verdict;
    u64 lost_base[2] = {0, 0};
    // zero-copy pipeline for BNG_MEM_HOST batches in pinned memory: two chunk buffers, three streams
    cudaStream_t s_in = nullptr, s_out = nullptr;
    cudaEvent_t ev_in[ZC_BUFS] = {}, ev_comp[ZC_BUFS] = {}, ev_out[ZC_BUFS] = {};
    DevBuf<u8> zc_hdr[ZC_BUFS], zc_verdict[ZC_BUFS];
    DevBuf<u32> zc_off[ZC_BUFS], zc_len[ZC_BUFS], zc_len0[ZC_BUFS], zc_prio[ZC_BUFS];
    DevBuf<u64> zc_now[ZC_BUFS];
    u32 zc_chunk = 1u << 18; // frames per chunk of the zero-copy pipeline
    // staged upserts (bng_map_update_staged): per map, keys/values in arrival order, applied at the next batch boundary
    struct Staged {
        std::vector<u8> keys, vals;
        u64 n = 0;
    };
    std::vector<Staged> staged;
    u64 staged_total = 0, staged_errors = 0, staged_flushes = 0;
    u64 rebuilds = 0; // flow-table rebuilds (tombstone compaction) so far
    u64 evict_at_rebuild = 0; // ST_LRU_EVICT when the flow tables were last rebuilt
    // BNG_MEM_DEVICE batches do not synchronise: each one queues a copy of ST_LRU_EVICT into evict_word and records
    // evict_ev; a later call looks at the copy once the event has completed (poll_compact_locked)
    PinnedBuf<u64> evict_word;
    cudaEvent_t evict_ev = nullptr;
    bool evict_pending = false;
    bool small_dirty = false; // a map feeding the SmallTabs image changed since the image was built
    // grow-only scratch of map dumps (no allocation per call)
    DevBuf<u8> dump_k, dump_v;
    DevBuf<u32> dump_c;
    // multi-GPU reconciliation (bng_comm_init / bng_sync_reduce)
    ncclComm_t comm = nullptr;
    u32 comm_rank = 0, comm_world = 1;
    DevBuf<u64> stats_global; // all-reduced counter vector
    // per-subscriber traffic accounting (bng_acct_*): records index-aligned with the subscriber directory, allocated
    // by the first bng_acct_enable (or a restore that carries records); acct_progs: bit p = program p is accounted
    DevBuf<u64> acct;
    u32 acct_progs = 0;
    DevBuf<u8> acct_dump_buf; // grow-only scratch of bng_acct_dump: records, then addresses
    // per-subscriber idle detection (bng_idle_*, idle.cu): records index-aligned with the subscriber directory, allocated
    // by the first bng_idle_enable / bng_idle_timeout_set (or a restore / delta that carries timeouts); idle_progs: bit
    // p = program p stamps
    DevBuf<u64> idle;
    u32 idle_progs = 0;
    DevBuf<u8> idle_scan_buf; // grow-only scratch of bng_idle_scan: records, then addresses, then the count
    // NAT port-usage census (bng_nat_usage, natuse.cu): scratch allocated by the first call (nu_sum != null)
    DevBuf<u64> nu_set, nu_pub, nu_sum;
    DevBuf<u32> nu_sub;
    u32 nu_set_mask = 0, nu_pub_mask = 0;
    DevBuf<u8> nu_out; // grow-only: the qualifying records and their addresses
    // DHCP lease census and sweep (leases.cu): scratch allocated by the first call that needs it
    DevBuf<u64> ls_set, ls_pools, ls_sum; // the census's (ls_sum != null), kernels.h: LeaseUse
    u32 ls_set_mask = 0, ls_unk_mask = 0;
    DevBuf<u8> ls_out;   // grow-only: the records of either call, then the census's pool ids
    DevBuf<u64> ls_macs; // grow-only: the sweep's words (LS_W_WORDS), then its MAC set
    u32 ls_wire = 0; // bng_dhcp_lease_addr_order
    u64 lease_rebuilds = 0; // rebuilds of the lease maps and circuit_id_map (not part of `rebuilds`)
    u64 seq = 0; // the batch sequence in 64 bits (dev.batch_seq holds its low 32): bng_li_record.batch
    // lawful intercept (bng_li_*, li.cu): allocated by the first bng_li_configure / bng_li_target_set (li_ctl != null)
    u64 *li_ctl = nullptr;   // device: LiRing::ctl
    u64 *li_words = nullptr; // device: the target set (AddrSet words, LI_TSLOTS), and its ids
    u32 *li_ids = nullptr;
    u32 li_mask = 0;
    bool li_dirty = false;   // the host's targets changed since the device copy was made
    std::unordered_map<u32, u32> li_targets; // authoritative: address -> target id
    DevBuf<u8> li_ring;
    u32 li_cap = 0, li_rec = 0, li_snap = 0;
    DevBuf<uint2> li_match; // [L.s.cap]
    std::vector<u8> li_pending; // records copied out of the ring, ordered, not yet drained
    u64 li_lost_host = 0;       // records discarded by a reconfiguration
    // incremental replication (bng_delta_*, delta.cu).  Exporter: one shadow per hash map (map id), and one of the
    // accounting records (map -1) once they exist; empty while tracking is off.
    struct DeltaShadow {
        int map;
        DevBuf<u64> words;
        u64 nslots;
        u32 sw;
    };
    std::vector<DeltaShadow> dshadow;
    bool delta_full = true;                 // the next export is FULL
    u64 delta_stream = 0, delta_seq = 0;    // exporter: stream id, sequence of the last export
    std::vector<std::pair<u32, u32>> delta_li; // interception targets as last sent, by address
    bool delta_li_sent = false;
    DevBuf<u32> dlist;                      // diff lists of one table: deletions at [0, n), upserts at [n, 2n)
    DevBuf<u32> dsent;                      // the lists of every table of an export, kept for the commit
    DevBuf<u8> demit;                       // records of one table
    u64 dapply_stream = 0, dapply_seq = 0;  // applier: the last delta applied
    // subscriber hand-over (bng_sub_export, move.cu): the flow tables' slot lists, allocated by the first export, and
    // a grow-only staging buffer (address set and keys in, gathered entries and lookups out)
    DevBuf<u32> mv_lists;
    DevBuf<u8> mv_buf;
    // subscriber_ipv6 (not a map of the reference): IPv6 prefix -> subscriber IPv4 address, the attribution of IPv6
    // frames; v6_live is its live-entry count as of the last command that changed it (0: the IPv6 kernels stay off)
    Tbl v6{};
    u32 v6_live = 0;
    // bng_qos_ipv6_enable: IPv6 frames are shaped by their owner's token bucket (context state: no snapshot, delta or
    // hand-over blob carries it)
    bool qos_v6 = false;
    // bng_nat_icmp_errors_enable: nat44_ingress translates ICMP errors by the flow they quote (context state, as
    // qos_v6)
    bool nat_icmp = false;
    // bng_nat_icmp_errors_egress_enable: nat44_egress and the pipelines translate subscribers' ICMP errors by the flow
    // they quote (context state, as qos_v6)
    bool nat_icmp_eg = false;
    // bng_antispoof_ipv6_prefixes_enable: antispoof_ingress allows IPv6 sources in their binding's own subscriber_ipv6
    // prefixes (context state, as qos_v6)
    bool as_v6 = false;
    // The DHCPv6 fast path (not maps of the reference, include/bng_b200.h): dhcpv6_bindings, dhcpv6_server_config, and
    // the host's copies of what selects k_dhcp_fastpath<v6>: the bindings' live-entry count as of the last command
    // that changed it, and the server configuration as last written
    Tbl d6b{};
    u8 *d6cfg = nullptr;
    u32 d6_live = 0;
    u8 d6cfg_host[DHCP6_CFG_BYTES] = {};
    // bng_dhcpv6_enable: dhcp_fastpath_prog answers bound DHCPv6 clients (context state, as qos_v6)
    bool dhcp6 = false;
    // Router and Neighbor Solicitations (not maps of the reference, include/bng_b200.h): nd_bindings, nd_config, the
    // host's copy of the configuration as last written (it selects k_dhcp_fastpath<nd>) and the bindings' live-entry
    // count as of the last command that changed it (bng_sub_export looks them up only while there are some)
    Tbl ndb{};
    u8 *ndcfg = nullptr;
    u32 nd_live = 0;
    u8 ndcfg_host[ND_CFG_BYTES] = {};
    // bng_nd_enable: dhcp_fastpath_prog answers Router and Neighbor Solicitations (context state, as qos_v6)
    bool nd = false;
};

namespace {

int fail(bng_ctx *c, int code, const char *fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    if (c)
        c->err = buf;
    else
        g_open_err = buf;
    return code;
}

#define CU(c, call)                                                                        \
    do {                                                                                   \
        cudaError_t e__ = (call);                                                          \
        if (e__ != cudaSuccess) return fail(c, -EIO, "%s: %s", #call, cudaGetErrorString(e__)); \
    } while (0)

u32 zc_chunk_frames() { // frames per chunk of the zero-copy pipeline; BNG_ZC_CHUNK_LOG2 overrides for tuning (read at bng_open)
    const char *e = getenv("BNG_ZC_CHUNK_LOG2");
    int lg = e ? atoi(e) : 18; // (tools/e2e_chunk_sweep.sh: 2^18 is the best or equal-best for both host layouts)
    if (lg < 10) lg = 10;
    if (lg > 22) lg = 22;
    return 1u << lg;
}

u32 pow2_at_least(u64 v) {
    u64 p = 1;
    while (p < v) p <<= 1;
    return (u32)p;
}

int dev_alloc(bng_ctx *c, void **p, size_t bytes, int fill) {
    CU(c, cudaMalloc(p, bytes ? bytes : 16));
    c->allocs.push_back(*p);
    CU(c, cudaMemset(*p, fill, bytes ? bytes : 16));
    return 0;
}

int make_table(bng_ctx *c, Tbl *t, u32 key_size, u32 value_size, u32 voff, u32 max_entries, u32 vlayout = 0,
               u32 slot_bytes = 0, u32 sparsity = 2) {
    u32 cap = pow2_at_least(std::max<u64>(64, (u64)max_entries * sparsity));
    t->mask = cap - 1;
    t->home_mask = cap - 1;
    t->voff = voff;
    t->key_size = key_size;
    t->value_size = value_size;
    t->max_entries = max_entries;
    t->vlayout = vlayout;
    t->lru = LRU_NONE;
    t->slot_bytes = slot_bytes ? slot_bytes : ((voff + value_size + 31u) & ~31u);
    int r = dev_alloc(c, (void **)&t->slots, (size_t)cap * t->slot_bytes, 0xFF);
    if (r) return r;
    return dev_alloc(c, (void **)&t->count, 16, 0);
}

// A growth of devbuf.hpp that failed, as the caller's error: -ENOMEM when the allocation was refused, else (a replacing
// growth's copy or stream synchronisation) -EIO with the runtime's text.
int grow_failed(bng_ctx *c, const char *what, size_t bytes, const char *of = nullptr, cudaError_t e = cudaErrorMemoryAllocation) {
    if (e != cudaErrorMemoryAllocation) return fail(c, -EIO, "%s: %s", what, cudaGetErrorString(e));
    return fail(c, -ENOMEM, "%s: %zu bytes of device memory%s%s", what, bytes, of ? " for the " : "", of ? of : "");
}

// The batch arrays of L.s for cap frames, all of them or none (L.s then holds null pointers and cap 0).  attr: with the
// attribution words (accounting, idle detection and interception use them), li: with interception's match list.
int scratch_locked(bng_ctx *c, u32 cap, bool attr, bool li) {
    Scratch &s = c->L.s;
    const size_t w = (size_t)cap * 4, m = li ? (size_t)cap * sizeof(uint2) : 0, sort = std::max<size_t>(sort_temp_bytes(cap), 16);
    const bool ok = devbuf::grow_all({{&c->key_a, w}, {&c->key_b, w}, {&c->val_a, w}, {&c->val_b, w}, {&c->qslot, w},
                                      {&c->attr, attr ? w : 0}, {&c->li_match, m}, {&c->cub_tmp, sort}});
    s.key_a = c->key_a, s.key_b = c->key_b, s.val_a = c->val_a, s.val_b = c->val_b, s.qslot = c->qslot, s.attr = c->attr;
    s.cub_tmp = c->cub_tmp, s.cub_tmp_bytes = ok ? sort_temp_bytes(cap) : 0;
    s.cap = ok ? cap : 0;
    return ok ? 0 : grow_failed(c, "batch scratch", (attr ? 6 : 5) * w + m + sort);
}

int ensure_scratch(bng_ctx *c, u32 n) {
    if (n <= c->L.s.cap) return 0;
    return scratch_locked(c, std::max<u32>(n, 1024), c->acct || c->idle || c->li_ctl, c->li_ctl);
}

int ensure_io(bng_ctx *c, size_t bytes) {
    const size_t nb = std::max<size_t>(bytes, 1 << 20);
    if (!devbuf::grow_all({{&c->io_dev, nb}, {&c->io_host, nb}})) return grow_failed(c, "staging", 2 * nb);
    return 0;
}

MapReg *get_map(bng_ctx *c, int id) {
    if (!c || id < 0 || id >= (int)c->maps.size()) return nullptr;
    return &c->maps[id];
}

void add_hash(bng_ctx *c, const char *name, u32 type, u32 ks, u32 vs, u32 max, Tbl *t) {
    MapReg m{};
    m.name = name; m.type = type; m.key_size = ks; m.value_size = vs; m.max_entries = max;
    m.kind = KIND_HASH; m.tbl = t;
    c->maps.push_back(m);
}
void add_array(bng_ctx *c, const char *name, u32 vs, u32 max, u8 **base) {
    MapReg m{};
    m.name = name; m.type = T_ARRAY; m.key_size = 4; m.value_size = vs; m.max_entries = max;
    m.kind = KIND_ARRAY; m.arr = base;
    c->maps.push_back(m);
}
void add_stats(bng_ctx *c, const char *name, u32 type, u32 vs, int base) {
    MapReg m{};
    m.name = name; m.type = type; m.key_size = 4; m.value_size = vs; m.max_entries = 1;
    m.kind = KIND_STATS; m.stat_base = base;
    c->maps.push_back(m);
}
void add_lpm(bng_ctx *c, const char *name, u32 max, LpmTbl *l) {
    MapReg m{};
    m.name = name; m.type = T_LPM; m.key_size = 8; m.value_size = 1; m.max_entries = max;
    m.kind = KIND_LPM; m.lpm = l;
    c->maps.push_back(m);
}
void add_event(bng_ctx *c, const char *name, u32 type, u32 ks, u32 vs, u32 max, EvRing *r, u32 payload) {
    MapReg m{};
    m.name = name; m.type = type; m.key_size = ks; m.value_size = vs; m.max_entries = max;
    m.kind = KIND_EVENT; m.ring = r; m.ev_payload = payload;
    c->maps.push_back(m);
}

int make_ring(bng_ctx *c, EvRing *r, u32 payload, u32 cap, u32 lost_stat) {
    r->rec_bytes = (payload + 8 + 15u) & ~15u;
    r->cap = cap;
    r->lost_stat = lost_stat;
    int e = dev_alloc(c, (void **)&r->buf, (size_t)cap * r->rec_bytes, 0);
    if (e) return e;
    return dev_alloc(c, (void **)&r->count, 16, 0);
}

int make_lpm(bng_ctx *c, LpmTbl *l, u32 max) {
    l->max_entries = max;
    int e = dev_alloc(c, (void **)&l->ents, (size_t)max * 12, 0);
    if (e) return e;
    return dev_alloc(c, (void **)&l->count, 16, 0);
}

// ---- subscriber_ipv6 ----
// the host's copy of the live-entry count, which selects the IPv6 instantiations of the attribution kernels
int v6_refresh_locked(bng_ctx *c) {
    CU(c, cudaMemcpyAsync(&c->v6_live, c->v6.count, 4, cudaMemcpyDeviceToHost, c->L.stream));
    CU(c, cudaStreamSynchronize(c->L.stream));
    return 0;
}
// The key as the table holds it: bits past prefixlen cleared (the device masks too; the host does it where keys are
// compared as bytes, so that two spellings of one prefix count as one key)
void v6_mask_key(u8 *key) {
    u32 w[5];
    memcpy(w, key, 20);
    if (w[0] >= LPM6_LENS) return; // refused by the device
    u64 kw[LPM6_KW];
    lpm6_key(kw, w[0], w + 1);
    w[1] = (u32)(kw[0] >> 32), w[2] = (u32)kw[1], w[3] = (u32)(kw[1] >> 32), w[4] = (u32)kw[2];
    memcpy(key, w, 20);
}

// ---- dhcpv6_bindings ----
int d6_refresh_locked(bng_ctx *c) {
    CU(c, cudaMemcpyAsync(&c->d6_live, c->d6b.count, 4, cudaMemcpyDeviceToHost, c->L.stream));
    CU(c, cudaStreamSynchronize(c->L.stream));
    return 0;
}
// An entry the fast path could not use the way it reads it (include/bng_b200.h: the update's -EINVAL)
bool d6_bad_binding(const u8 *key, const u8 *val) {
    const u32 dl = key[0];
    if (dl == 0 || dl > 31) return true;
    for (u32 k = 1 + dl; k < 32; k++)
        if (key[k]) return true;
    const u32 flags = val[6], pl = val[7];
    if ((flags & ~3u) || !flags) return true;
    if (flags & BNG_DHCPV6_PD) {
        if (pl == 0 || pl > 128) return true;
        for (u32 b = pl; b < 128; b++)
            if ((val[48 + b / 8] >> (7 - b % 8)) & 1) return true;
    }
    return false;
}

// ---- nd_bindings, nd_config ----
int nd_refresh_locked(bng_ctx *c) {
    CU(c, cudaMemcpyAsync(&c->nd_live, c->ndb.count, 4, cudaMemcpyDeviceToHost, c->L.stream));
    CU(c, cudaStreamSynchronize(c->L.stream));
    return 0;
}
// A binding the fast path could not use the way it reads it (include/bng_b200.h: the update's -EINVAL).  val: struct
// bng_nd_binding: prefix@0 prefix_len@16 pio_flags@17 pad@18 valid@20 preferred@24 pad@28 expires_s@32 pad@40
bool nd_bad_binding(const u8 *val) {
    const u32 pl = val[16], fl = val[17];
    if (pl > 128 || (fl & ~(u32)(BNG_ND_PIO_L | BNG_ND_PIO_A))) return true;
    if (pl == 0 && fl) return true;
    for (u32 b = pl; b < 128; b++)
        if ((val[b / 8] >> (7 - b % 8)) & 1) return true;
    for (u32 k : {18u, 19u, 28u, 29u, 30u, 31u, 40u, 41u, 42u, 43u, 44u, 45u, 46u, 47u})
        if (val[k]) return true;
    return false;
}
// The RA template's options from `o` to `end`: each has a length byte >= 1 and the walk ends exactly at `end`
bool nd_options_ok(const u8 *ra, u32 o, u32 end) {
    while (o < end) {
        if (o + 2 > end || ra[o + 1] == 0) return false;
        o += 8u * ra[o + 1];
    }
    return o == end;
}
// A configuration the fast path could not copy as its rule says (include/bng_b200.h: the update's -EINVAL).  v: struct
// bng_nd_config: router_mac@0 pad@6 ra_head_len@8 ra_tail_len@10 pad@12 router_ll@16 ra@32
bool nd_bad_config(const u8 *v) {
    u16 head, tail;
    memcpy(&head, v + 8, 2);
    memcpy(&tail, v + 10, 2);
    if (head == 0) { // unconfigured: all zero past the MAC
        for (u32 k = 6; k < ND_CFG_BYTES; k++)
            if (v[k]) return true;
        return false;
    }
    if (v[6] || v[7] || v[12] || v[13] || v[14] || v[15]) return true;
    if (head < 16 || (head & 7) || (tail & 7) || head + tail > 288) return true;
    const u8 *ra = v + 32;
    if (ra[0] != 134 || ra[1] != 0 || ra[2] || ra[3]) return true;
    if (!nd_options_ok(ra, 16, head) || !nd_options_ok(ra, head, head + tail)) return true;
    if (v[16] != 0xFE || (v[17] & 0xC0) != 0x80) return true; // fe80::/10
    if ((v[0] & 1) || !(v[0] | v[1] | v[2] | v[3] | v[4] | v[5])) return true;
    for (u32 k = head + tail; k < 288; k++)
        if (ra[k]) return true;
    return false;
}

// ---- control-plane commands on hash maps ----
int hash_cmd(bng_ctx *c, MapReg *m, int op, const void *keys, void *vals, u64 n, u32 flags, int *first_err, u64 *n_err = nullptr) {
    const Tbl &t = *m->tbl;
    const u64 chunk_max = 1u << 18;
    *first_err = 0;
    for (u64 done = 0; done < n; done += chunk_max) {
        u64 k = std::min(chunk_max, n - done);
        size_t kb = k * t.key_size, vb = k * t.value_size, rb = k * 4;
        size_t koff = 0, voff = (kb + 255) & ~(size_t)255, roff = (voff + vb + 255) & ~(size_t)255;
        int r = ensure_io(c, roff + rb);
        if (r) return r;
        memcpy(c->io_host + koff, (const u8 *)keys + done * t.key_size, kb);
        if (op == TOP_UPDATE) memcpy(c->io_host + voff, (const u8 *)vals + done * t.value_size, vb);
        size_t up = op == TOP_UPDATE ? voff + vb : kb;
        CU(c, cudaMemcpyAsync(c->io_dev, c->io_host, up, cudaMemcpyHostToDevice, c->L.stream));
        const int role = m->tbl == &c->dev.sub_nat ? 1 : (m->tbl == &c->dev.qos_in ? 2 : 0);
        CU(c, run_table_op(c->L, t, op, c->io_dev + koff, c->io_dev + voff, (int *)(c->io_dev + roff), k, flags, c->dev.subdir,
                           role, c->acct, c->idle));
        size_t dfrom = op == TOP_LOOKUP ? voff : roff;
        CU(c, cudaMemcpyAsync(c->io_host + dfrom, c->io_dev + dfrom, roff + rb - dfrom, cudaMemcpyDeviceToHost, c->L.stream));
        CU(c, cudaStreamSynchronize(c->L.stream));
        const int *res = (const int *)(c->io_host + roff);
        for (u64 i = 0; i < k; i++)
            if (res[i]) {
                if (!*first_err) *first_err = res[i];
                if (n_err) ++*n_err;
            }
        if (op == TOP_LOOKUP) {
            for (u64 i = 0; i < k; i++)
                if (!res[i])
                    memcpy((u8 *)vals + (done + i) * t.value_size, c->io_host + voff + i * t.value_size, t.value_size);
        }
    }
    if (m->tbl == &c->v6 && op != TOP_LOOKUP) return v6_refresh_locked(c);
    if (m->tbl == &c->d6b && op != TOP_LOOKUP) return d6_refresh_locked(c);
    if (m->tbl == &c->ndb && op != TOP_LOOKUP) return nd_refresh_locked(c);
    return 0;
}

int lpm_upload(bng_ctx *c, MapReg *m) {
    u32 n = (u32)(m->lpm_host.size() / 3);
    if (n) CU(c, cudaMemcpyAsync(m->lpm->ents, m->lpm_host.data(), (size_t)n * 12, cudaMemcpyHostToDevice, c->L.stream));
    CU(c, cudaMemcpyAsync(m->lpm->count, &n, 4, cudaMemcpyHostToDevice, c->L.stream));
    CU(c, cudaStreamSynchronize(c->L.stream));
    return 0;
}

bool lpm_same(u32 pl, u32 a, u32 b) { // first pl bits equal, bytes in memory order
    u32 x = __builtin_bswap32(a) ^ __builtin_bswap32(b);
    u32 mask = pl == 0 ? 0u : (pl >= 32 ? 0xFFFFFFFFu : (0xFFFFFFFFu << (32 - pl)));
    return (x & mask) == 0;
}

// an opt-in switch of the context (bng_qos_ipv6_enable and its kind): in effect from the next run on
int set_switch(bng_ctx *c, bool bng_ctx::*sw, int on) {
    if (!c) return -EINVAL;
    std::lock_guard<std::mutex> g(c->mu);
    c->*sw = on != 0;
    return 0;
}

} // namespace

// ---- staged upserts ----
// The reference's Go callers issue one Map.Put per lease / session event (pkg/dhcp/server.go:708,780,798); a
// synchronous bng_map_update costs a host->device copy, a kernel and a device->host copy each.  Staged updates
// (BPF_ANY semantics) are queued on the host and applied together: at the next batch boundary (bng_prog_run),
// at bng_sync, and before anything reads or changes the same map (so a staged Put is always visible to a
// later Lookup / Delete / dump of that map).  Within one flush the LAST staged value of a key wins, as it
// would had the Puts been applied one by one.
int flush_staged_locked(bng_ctx *c, int only_map);
bool feeds_small_tabs_p(const MapReg *m);
int small_refresh_p(bng_ctx *c);

int flush_staged_locked(bng_ctx *c, int only_map) {
    if (!c->staged_total) return 0;
    int rc = 0;
    for (size_t mi = 0; mi < c->staged.size(); mi++) {
        bng_ctx::Staged &q = c->staged[mi];
        if (!q.n || (only_map >= 0 && (int)mi != only_map)) continue;
        MapReg *m = &c->maps[mi];
        const u32 ks = m->key_size, vs = m->value_size;
        // last occurrence of every key, in order of that occurrence
        std::unordered_map<std::string, u64> last;
        last.reserve(q.n * 2);
        for (u64 i = 0; i < q.n; i++) last[std::string((const char *)&q.keys[i * ks], ks)] = i;
        std::vector<u8> k2, v2;
        k2.reserve(last.size() * ks);
        v2.reserve(last.size() * vs);
        u64 uniq = 0;
        for (u64 i = 0; i < q.n; i++) {
            auto it = last.find(std::string((const char *)&q.keys[i * ks], ks));
            if (it->second != i) continue;
            k2.insert(k2.end(), &q.keys[i * ks], &q.keys[i * ks] + ks);
            v2.insert(v2.end(), &q.vals[i * vs], &q.vals[i * vs] + vs);
            uniq++;
        }
        int first = 0;
        u64 nerr = 0;
        int r = hash_cmd(c, m, TOP_UPDATE, k2.data(), v2.data(), uniq, BNG_ANY, &first, &nerr);
        if (!r && feeds_small_tabs_p(m)) c->small_dirty = true;
        c->staged_errors += nerr;
        c->staged_total -= q.n;
        c->staged_flushes++;
        q.keys.clear();
        q.vals.clear();
        q.n = 0;
        if (r && !rc) rc = r;
    }
    return rc;
}

// ---- NCCL, resolved at run time: the host process brings its own libnccl (the Go control plane links it, a
// Python process has torch's loaded already); nothing here links against it ----
struct NcclApi {
    void *handle = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*AllReduce)(const void *, void *, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    const char *(*GetErrorString)(ncclResult_t) = nullptr;
    std::string err;
};
NcclApi *nccl_api() {
    static NcclApi api;
    static std::once_flag once;
    std::call_once(once, [] {
        // the copy the host process already has (a Python process with torch loaded brings its own, newer than the
        // system's; loading another libnccl.so.2 first would shadow it for everything loaded later), else by name
        const char *path = getenv("BNG_NCCL_LIB");
        api.handle = path ? nullptr : dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);
        if (!api.handle) api.handle = dlopen(path ? path : "libnccl.so.2", RTLD_NOW | RTLD_LOCAL);
        if (!api.handle) {
            api.err = std::string("dlopen libnccl.so.2: ") + (dlerror() ? dlerror() : "?");
            return;
        }
        api.GetUniqueId = (decltype(api.GetUniqueId))dlsym(api.handle, "ncclGetUniqueId");
        api.CommInitRank = (decltype(api.CommInitRank))dlsym(api.handle, "ncclCommInitRank");
        api.AllReduce = (decltype(api.AllReduce))dlsym(api.handle, "ncclAllReduce");
        api.CommDestroy = (decltype(api.CommDestroy))dlsym(api.handle, "ncclCommDestroy");
        api.GetErrorString = (decltype(api.GetErrorString))dlsym(api.handle, "ncclGetErrorString");
        if (!api.GetUniqueId || !api.CommInitRank || !api.AllReduce || !api.CommDestroy) api.err = "libnccl.so.2 lacks the expected symbols";
    });
    return api.err.empty() ? &api : nullptr;
}

// ===========================================================================
extern "C" {

static int small_refresh(bng_ctx *c);
static bool feeds_small_tabs(const MapReg *m);

uint32_t bng_abi_version(void) { return BNG_ABI_VERSION; }

const char *bng_last_error(bng_ctx *ctx) { return ctx ? ctx->err.c_str() : g_open_err.c_str(); }

uint32_t bng_shard_of_mac(uint64_t mac_key, uint32_t world) {
    if (world <= 1) return 0;
    return (uint32_t)(splitmix64(mac_key) % world);
}

// Pinned, GPU-mapped host memory for frame arenas (BNG_MEM_HOST batches are then read in place, zero-copy).
// The arena is backed by 2 MB transparent huge pages and registered with cudaHostRegister: behind an IOMMU in
// translated mode the GPU's scattered 64-byte header reads cost one translation per page touched, and a
// receive ring in 4 KB pages thrashes the IOTLB.  Falls back to cudaHostAlloc when huge pages or
// registration are not available.  BNG_HOST_ARENA=pinned forces the fallback.
namespace {
struct HostArena {
    void *map_base;  // mmap() result (nullptr: cudaHostAlloc)
    size_t map_bytes;
    size_t reg_bytes;
};
std::mutex g_arena_mu;
std::vector<std::pair<void *, HostArena>> g_arenas;
} // namespace

void *bng_host_alloc(size_t bytes) {
    if (!bytes) bytes = 16;
    const char *mode = getenv("BNG_HOST_ARENA");
    const size_t huge = (size_t)2 << 20;
    if (!mode || strcmp(mode, "pinned") != 0) {
        size_t size = (bytes + huge - 1) / huge * huge;
        void *base = mmap(nullptr, size + huge, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
        if (base != MAP_FAILED) {
            u8 *p = (u8 *)(((uintptr_t)base + huge - 1) & ~(uintptr_t)(huge - 1));
#ifdef MADV_HUGEPAGE
            madvise(p, size, MADV_HUGEPAGE);
#endif
            for (size_t o = 0; o < size; o += 4096) p[o] = 0; // first touch on the caller's (NUMA-bound) thread
            // Whether the fault path found free 2 MB pages is luck (the same process can get one arena in huge
            // pages and the next in 4 KB pages).  MADV_COLLAPSE (Linux 6.1+) collapses
            // the range synchronously, compacting memory if it has to; best effort, errors ignored.
#ifndef MADV_COLLAPSE
#define MADV_COLLAPSE 25
#endif
            for (size_t o = 0; o < size; o += (size_t)64 << 20)
                madvise(p + o, std::min<size_t>((size_t)64 << 20, size - o), MADV_COLLAPSE);
            if (cudaHostRegister(p, size, cudaHostRegisterPortable | cudaHostRegisterMapped) == cudaSuccess) {
                std::lock_guard<std::mutex> g(g_arena_mu);
                g_arenas.push_back({p, HostArena{base, size + huge, size}});
                return p;
            }
            cudaGetLastError();
            munmap(base, size + huge);
        }
    }
    void *p = nullptr;
    if (cudaMallocHost(&p, bytes) != cudaSuccess) return nullptr;
    std::lock_guard<std::mutex> g(g_arena_mu);
    g_arenas.push_back({p, HostArena{nullptr, 0, 0}});
    return p;
}
void bng_host_free(void *p) {
    if (!p) return;
    HostArena a{nullptr, 0, 0};
    bool found = false;
    {
        std::lock_guard<std::mutex> g(g_arena_mu);
        for (size_t i = 0; i < g_arenas.size(); i++)
            if (g_arenas[i].first == p) {
                a = g_arenas[i].second;
                g_arenas.erase(g_arenas.begin() + i);
                found = true;
                break;
            }
    }
    if (!found) return; // not ours
    if (a.map_base) {
        cudaDeviceSynchronize(); // nothing may still be reading the arena when its mapping goes away
        cudaHostUnregister(p);
        munmap(a.map_base, a.map_bytes);
    } else {
        cudaFreeHost(p);
    }
}

int bng_close(bng_ctx *c) {
    if (!c) return -EINVAL;
    {
        std::lock_guard<std::mutex> g(c->mu);
        cudaSetDevice(c->device);
        if (c->L.stream) cudaStreamSynchronize(c->L.stream);
        if (c->comm) {
            if (NcclApi *a = nccl_api()) a->CommDestroy(c->comm);
            c->comm = nullptr;
        }
        for (void *p : c->allocs) cudaFree(p);
        if (c->evict_ev) cudaEventDestroy(c->evict_ev);
        for (int i = 0; i < ZC_BUFS; i++) {
            if (c->ev_in[i]) cudaEventDestroy(c->ev_in[i]);
            if (c->ev_comp[i]) cudaEventDestroy(c->ev_comp[i]);
            if (c->ev_out[i]) cudaEventDestroy(c->ev_out[i]);
        }
        if (c->s_in) cudaStreamDestroy(c->s_in);
        if (c->s_out) cudaStreamDestroy(c->s_out);
        if (c->L.stream) cudaStreamDestroy(c->L.stream);
    }
    delete c; // and with it the buffers it owns (devbuf.hpp)
    return 0;
}

bng_ctx *bng_open(const bng_open_opts *o) {
    bng_open_opts opts;
    memset(&opts, 0, sizeof(opts));
    opts.device = -1;
    if (o) memcpy(&opts, o, std::min<size_t>(sizeof(opts), o->struct_size ? o->struct_size : sizeof(opts)));
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0) {
        fail(nullptr, 0, "no CUDA device (%s): the bng_b200 dataplane has no CPU path",
             e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
        return nullptr;
    }
    bng_ctx *c = new bng_ctx();
    int dev = opts.device;
    if (dev < 0 && cudaGetDevice(&dev) != cudaSuccess) dev = 0;
    c->device = dev;
#define OPEN_CU(call)                                                          \
    do {                                                                       \
        cudaError_t e__ = (call);                                              \
        if (e__ != cudaSuccess) {                                              \
            fail(nullptr, 0, "%s: %s", #call, cudaGetErrorString(e__));        \
            bng_close(c);                                                      \
            return nullptr;                                                    \
        }                                                                      \
    } while (0)
#define OPEN_R(call)                                 \
    do {                                             \
        if ((call) != 0) {                           \
            g_open_err = c->err;                     \
            bng_close(c);                            \
            return nullptr;                          \
        }                                            \
    } while (0)
    OPEN_CU(cudaSetDevice(dev));
    cudaDeviceProp prop;
    OPEN_CU(cudaGetDeviceProperties(&prop, dev));
    if (prop.major != 9 || prop.minor != 0) { // sm_90a code runs on compute capability 9.0 alone
        fail(nullptr, 0, "device %d is sm_%d%d; this library is built for sm_90a (H100) only", dev, prop.major, prop.minor);
        bng_close(c);
        return nullptr;
    }
    c->L.num_sms = prop.multiProcessorCount;
    c->zc_chunk = zc_chunk_frames();
    OPEN_CU(cudaStreamCreateWithFlags(&c->L.stream, cudaStreamNonBlocking));

    u32 max_subs = opts.max_subscribers ? opts.max_subscribers : 1000000u;
    u32 max_sess = opts.max_nat_sessions ? opts.max_nat_sessions : 4000000u;
    u32 max_eim = opts.max_eim_mappings ? opts.max_eim_mappings : 2000000u;
    u32 ev_cap = opts.event_capacity ? opts.event_capacity : (1u << 21);
    u32 max_vlan = std::min<u32>(100000u, std::max<u32>(max_subs, 64));
    DevCtx &d = c->dev;

    // subscriber_bindings: 32-byte slots, L2-resident; k_antispoof probes the home PAIR of slots at once, so that a
    // second, dependent probe — which stalls its whole warp — is rarely needed
    OPEN_R(make_table(c, &d.bindings, 8, 24, 8, max_subs, 0, 0, 4));
    d.bindings.home_mask = d.bindings.mask & ~1u;
    OPEN_R(make_table(c, &d.qos_eg, 4, 32, 16, max_subs, VL_QOS));
    OPEN_R(make_table(c, &d.qos_in, 4, 32, 16, max_subs, VL_QOS));
    OPEN_R(make_table(c, &d.sub_nat, 4, 64, 8, max_subs));
    OPEN_R(make_table(c, &d.sessions, 16, 80, 16, max_sess, VL_SESSION, 128));
    OPEN_R(make_table(c, &d.reverse, 16, 16, 16, max_sess));
    OPEN_R(make_table(c, &d.eim, 8, 32, 8, max_eim));
    d.sessions.lru = LRU_TS | ((u32)SES_LAST_SEEN << 8); // the three LRU_HASH maps of bpf/nat44.c:218-244
    d.reverse.lru = LRU_ANY;
    d.eim.lru = LRU_TS | (24u << 8); // eim_mapping.last_used
    OPEN_R(make_table(c, &d.hairpin, 4, 1, 8, 1000));
    OPEN_R(make_table(c, &d.alg, 4, 8, 8, 64));
    OPEN_R(make_table(c, &d.sub_pools, 8, 25, 8, max_subs));
    OPEN_R(make_table(c, &d.vlan_pools, 4, 25, 8, max_vlan));
    OPEN_R(make_table(c, &d.cid_subs, 32, 25, 32, max_subs));
    OPEN_R(make_table(c, &d.ip_pools, 4, 28, 8, 10000));
    OPEN_R(make_table(c, &d.cid_map, 8, 8, 8, max_subs));
    // subscriber_ipv6: a WAN /64 or /128 and a delegated prefix per subscriber; 32-byte slots (key words, value at 24)
    OPEN_R(make_table(c, &c->v6, LPM6_KEY, 4, 24, 2 * max_subs));
    OPEN_R(dev_alloc(c, (void **)&c->v6.plens, LPM6_LENS * 4, 0));
    // dhcpv6_bindings: 96-byte slots (32-byte key, the 64-byte binding at 32)
    OPEN_R(make_table(c, &c->d6b, 32, 64, 32, max_subs));
    OPEN_R(dev_alloc(c, (void **)&c->d6cfg, DHCP6_CFG_BYTES, 0));
    // nd_bindings: 64-byte slots (the MAC word, the 48-byte binding at 8)
    OPEN_R(make_table(c, &c->ndb, 8, 48, 8, max_subs));
    OPEN_R(dev_alloc(c, (void **)&c->ndcfg, ND_CFG_BYTES, 0));
    // subscriber directory: 16-byte slots, as many as the per-subscriber maps have, room for both maps' keys
    OPEN_R(make_table(c, &d.subdir, 4, 8, 8, max_subs, 0, 16));
    d.subdir.max_entries = std::min<u64>(2ull * max_subs, d.subdir.mask);
    d.subdir.home_mask = d.subdir.mask & ~1u; // even home slots: part of the directory's slot layout
    OPEN_R(make_lpm(c, &d.ranges_v4, 256));
    OPEN_R(make_lpm(c, &d.priv_ranges, 64));
    OPEN_R(dev_alloc(c, (void **)&d.as_config, 16, 0));
    OPEN_R(dev_alloc(c, (void **)&d.nat_config, 16, 0));
    OPEN_R(dev_alloc(c, (void **)&d.server_config, 16, 0));
    OPEN_R(dev_alloc(c, (void **)&d.nat_pool, 256 * 16, 0));
    OPEN_R(dev_alloc(c, (void **)&d.stats, ST_ALL * 8, 0));
    OPEN_R(make_ring(c, &d.spoof_ev, 56, ev_cap, ST_EV_LOST_SPOOF));
    OPEN_R(make_ring(c, &d.natlog_ev, 40, ev_cap, ST_EV_LOST_NATLOG));
    OPEN_R(dev_alloc(c, (void **)&c->L.s.counters, 64, 0));
    OPEN_R(ensure_scratch(c, opts.max_batch ? opts.max_batch : (1u << 22)));
    OPEN_R(ensure_io(c, 1 << 20));
    OPEN_R(dev_alloc(c, (void **)&d.small, sizeof(SmallTabs), 0xFF));

    // registry: the reference's map names, types, sizes (bpf/antispoof.c:71-119,
    // bpf/qos_ratelimit.c:37-65, bpf/nat44.c:218-320, bpf/maps.h:99-234)
    add_hash(c, "subscriber_bindings", T_HASH, 8, 24, max_subs, &d.bindings);
    add_array(c, "antispoof_config", 8, 1, &d.as_config);
    add_stats(c, "antispoof_stats", T_PERCPU_ARRAY, 48, ST_AS);
    add_event(c, "spoof_events", T_PERF, 4, 4, 0, &d.spoof_ev, 56);
    add_lpm(c, "allowed_ranges_v4", 256, &d.ranges_v4);
    add_hash(c, "qos_egress", T_HASH, 4, 32, max_subs, &d.qos_eg);
    add_hash(c, "qos_ingress", T_HASH, 4, 32, max_subs, &d.qos_in);
    add_stats(c, "qos_stats_map", T_PERCPU_ARRAY, 32, ST_QOS);
    add_hash(c, "nat_sessions", T_LRU, 16, 80, max_sess, &d.sessions);
    add_hash(c, "nat_reverse", T_LRU, 16, 16, max_sess, &d.reverse);
    add_hash(c, "eim_table", T_LRU, 8, 32, max_eim, &d.eim);
    add_hash(c, "subscriber_nat", T_HASH, 4, 64, max_subs, &d.sub_nat);
    add_array(c, "nat_pool", 16, 256, &d.nat_pool);
    add_hash(c, "hairpin_ips", T_HASH, 4, 1, 1000, &d.hairpin);
    add_array(c, "nat_config_map", 16, 1, &d.nat_config);
    add_stats(c, "nat_stats_map", T_PERCPU_ARRAY, 104, ST_NAT);
    add_event(c, "nat_log_rb", T_RINGBUF, 0, 0, 1u << 20, &d.natlog_ev, 40);
    add_hash(c, "alg_ports", T_HASH, 4, 8, 64, &d.alg);
    add_lpm(c, "nat_private_ranges", 64, &d.priv_ranges);
    add_hash(c, "subscriber_pools", T_HASH, 8, 25, max_subs, &d.sub_pools);
    add_hash(c, "vlan_subscriber_pools", T_HASH, 4, 25, max_vlan, &d.vlan_pools);
    add_hash(c, "ip_pools", T_HASH, 4, 28, 10000, &d.ip_pools);
    add_array(c, "server_config", 16, 1, &d.server_config);
    add_stats(c, "stats_map", T_ARRAY, 80, ST_DHCP);
    add_hash(c, "circuit_id_map", T_HASH, 8, 8, max_subs, &d.cid_map);
    add_hash(c, "circuit_id_subscribers", T_HASH, 32, 25, max_subs, &d.cid_subs);
    // not a map of the reference: IPv6 prefix -> subscriber IPv4 address (include/bng_b200.h), reported as an LPM trie
    add_hash(c, "subscriber_ipv6", T_LPM, LPM6_KEY, 4, 2 * max_subs, &c->v6);
    // not maps of the reference: the DHCPv6 fast path's cache (include/bng_b200.h)
    add_hash(c, "dhcpv6_bindings", T_HASH, 32, 64, max_subs, &c->d6b);
    add_array(c, "dhcpv6_server_config", DHCP6_CFG_BYTES, 1, &c->d6cfg);
    add_stats(c, "dhcpv6_stats", T_ARRAY, ST_DHCP6_N * 8, ST_DHCP6);
    // not maps of the reference: Router and Neighbor Solicitations answered on the GPU (include/bng_b200.h)
    add_hash(c, "nd_bindings", T_HASH, 8, 48, max_subs, &c->ndb);
    add_array(c, "nd_config", ND_CFG_BYTES, 1, &c->ndcfg);
    add_stats(c, "nd_stats", T_ARRAY, ST_ND_N * 8, ST_ND);
    c->staged.resize(c->maps.size());
    OPEN_R(small_refresh(c));
    cudaError_t se = cudaStreamSynchronize(c->L.stream);
    if (se != cudaSuccess) {
        fail(nullptr, 0, "init: %s", cudaGetErrorString(se));
        bng_close(c);
        return nullptr;
    }
    return c;
}

// ---------------------------------------------------------------------------
// maps
// ---------------------------------------------------------------------------
int bng_map_id(bng_ctx *c, const char *name) {
    if (!c || !name) return -EINVAL;
    for (size_t i = 0; i < c->maps.size(); i++)
        if (!strcmp(c->maps[i].name, name)) return (int)i;
    return -ENOENT;
}

int bng_map_get_info(bng_ctx *c, int map, bng_map_info *out) {
    MapReg *m = get_map(c, map);
    if (!m || !out) return -EINVAL;
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    out->type = m->type;
    out->key_size = m->key_size;
    out->value_size = m->value_size;
    out->max_entries = m->max_entries;
    out->count = m->max_entries;
    if (int fr = flush_staged_locked(c, map)) return fr;
    if (m->kind == KIND_HASH) {
        u32 cnt = 0;
        CU(c, cudaMemcpyAsync(&cnt, m->tbl->count, 4, cudaMemcpyDeviceToHost, c->L.stream));
        CU(c, cudaStreamSynchronize(c->L.stream));
        out->count = cnt;
    } else if (m->kind == KIND_LPM) {
        out->count = m->lpm_host.size() / 3;
    } else if (m->kind == KIND_EVENT) {
        u32 cnt = 0;
        CU(c, cudaMemcpyAsync(&cnt, m->ring->count, 4, cudaMemcpyDeviceToHost, c->L.stream));
        CU(c, cudaStreamSynchronize(c->L.stream));
        out->count = cnt + m->ev_pending.size() / m->ev_payload;
    }
    return 0;
}

static int small_refresh(bng_ctx *c);
static bool feeds_small_tabs(const MapReg *m);

int bng_map_update_batch(bng_ctx *c, int map, const void *keys, const void *values, uint64_t n, uint64_t flags) {
    MapReg *m = get_map(c, map);
    if (!m || !keys || !values) return -EINVAL;
    if (flags > BNG_EXIST) return -EINVAL;
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    if (int fr = flush_staged_locked(c, map)) return fr; // staged Puts of this map come first
    switch (m->kind) {
    case KIND_HASH: {
        // The reference applies the entries of a batch one after the other; one kernel launch applies them
        // concurrently, which is only the same thing when no key occurs twice.  The batch is therefore cut
        // wherever a key repeats (usually nowhere) and the pieces run in order.
        int first = 0, r = 0;
        const u32 ks = m->key_size;
        if (m->tbl == &c->d6b)
            for (u64 i = 0; i < n; i++)
                if (d6_bad_binding((const u8 *)keys + i * ks, (const u8 *)values + i * m->value_size)) return -EINVAL;
        if (m->tbl == &c->ndb)
            for (u64 i = 0; i < n; i++)
                if (nd_bad_binding((const u8 *)values + i * m->value_size)) return -EINVAL;
        std::vector<u8> masked;
        if (m->tbl == &c->v6) { // two spellings of one prefix are one key
            masked.assign((const u8 *)keys, (const u8 *)keys + n * ks);
            for (u64 i = 0; i < n; i++) v6_mask_key(masked.data() + i * ks);
            keys = masked.data();
        }
        u64 seg = 0;
        if (n > 1) {
            std::unordered_set<std::string_view> seen;
            seen.reserve((size_t)n * 2);
            for (u64 i = 0; i < n && !r; i++) {
                std::string_view kv((const char *)keys + i * ks, ks);
                if (!seen.insert(kv).second) { // key seen in this piece: run the piece, start the next one here
                    int f2 = 0;
                    r = hash_cmd(c, m, TOP_UPDATE, (const u8 *)keys + seg * ks, (u8 *)values + seg * m->value_size, i - seg, (u32)flags, &f2);
                    if (f2 && !first) first = f2;
                    seg = i;
                    seen.clear();
                    seen.insert(kv);
                }
            }
        }
        if (!r) {
            int f2 = 0;
            r = hash_cmd(c, m, TOP_UPDATE, (const u8 *)keys + seg * ks, (u8 *)values + seg * m->value_size, n - seg, (u32)flags, &f2);
            if (f2 && !first) first = f2;
        }
        if (!r && feeds_small_tabs(m)) c->small_dirty = true; // the image is rebuilt once, at the next batch boundary
        return r ? r : first;
    }
    case KIND_ARRAY:
    case KIND_STATS:
        for (u64 i = 0; i < n; i++) {
            u32 idx = ((const u32 *)keys)[i];
            if (idx >= m->max_entries) return -E2BIG;
            if (flags == BNG_NOEXIST) return -EEXIST;
            if (m->arr == &c->d6cfg) { // duid_len, dns_count
                const u8 *v = (const u8 *)values + i * m->value_size;
                if (v[6] > 32 || v[7] > 2) return -EINVAL;
            }
            if (m->arr == &c->ndcfg && nd_bad_config((const u8 *)values + i * m->value_size)) return -EINVAL;
            u8 *dst = m->kind == KIND_ARRAY ? *m->arr + (size_t)idx * m->value_size : (u8 *)(c->dev.stats + m->stat_base);
            CU(c, cudaMemcpyAsync(dst, (const u8 *)values + i * m->value_size, m->value_size, cudaMemcpyHostToDevice,
                                  c->L.stream));
        }
        CU(c, cudaStreamSynchronize(c->L.stream));
        if (feeds_small_tabs(m)) c->small_dirty = true;
        if (m->arr == &c->d6cfg && n) memcpy(c->d6cfg_host, (const u8 *)values + (n - 1) * m->value_size, DHCP6_CFG_BYTES);
        if (m->arr == &c->ndcfg && n) memcpy(c->ndcfg_host, (const u8 *)values + (n - 1) * m->value_size, ND_CFG_BYTES);
        return 0;
    case KIND_LPM:
        for (u64 i = 0; i < n; i++) {
            const u32 *k = (const u32 *)((const u8 *)keys + i * 8);
            u32 pl = k[0], addr = k[1], val = ((const u8 *)values)[i];
            if (pl > 32) return -EINVAL;
            bool found = false;
            for (size_t e = 0; e < m->lpm_host.size(); e += 3)
                if (m->lpm_host[e] == pl && lpm_same(pl, m->lpm_host[e + 1], addr)) {
                    if (flags == BNG_NOEXIST) return -EEXIST;
                    m->lpm_host[e + 2] = val;
                    found = true;
                }
            if (!found) {
                if (flags == BNG_EXIST) return -ENOENT;
                if (m->lpm_host.size() / 3 >= m->max_entries) return -ENOSPC;
                m->lpm_host.insert(m->lpm_host.end(), {pl, addr, val});
            }
        }
        return lpm_upload(c, m);
    default:
        return -EINVAL;
    }
}

int bng_map_update(bng_ctx *c, int map, const void *key, const void *value, uint64_t flags) {
    return bng_map_update_batch(c, map, key, value, 1, flags);
}

int bng_map_lookup(bng_ctx *c, int map, const void *key, void *value_out) {
    MapReg *m = get_map(c, map);
    if (!m || !key || !value_out) return -EINVAL;
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    if (int fr = flush_staged_locked(c, map)) return fr;
    switch (m->kind) {
    case KIND_HASH: {
        int first = 0;
        int r = hash_cmd(c, m, TOP_LOOKUP, key, value_out, 1, 0, &first);
        return r ? r : first;
    }
    case KIND_ARRAY:
    case KIND_STATS: {
        u32 idx = *(const u32 *)key;
        if (idx >= m->max_entries) return -ENOENT;
        const u8 *src = m->kind == KIND_ARRAY ? *m->arr + (size_t)idx * m->value_size : (const u8 *)(c->dev.stats + m->stat_base);
        CU(c, cudaMemcpyAsync(value_out, src, m->value_size, cudaMemcpyDeviceToHost, c->L.stream));
        CU(c, cudaStreamSynchronize(c->L.stream));
        return 0;
    }
    case KIND_LPM: {
        const u32 *k = (const u32 *)key;
        u32 pl = std::min<u32>(k[0], 32), addr = k[1];
        int best = -1;
        for (size_t e = 0; e < m->lpm_host.size(); e += 3) {
            u32 epl = m->lpm_host[e];
            if (epl > pl) continue;
            if (best >= 0 && epl <= m->lpm_host[best]) continue;
            if (lpm_same(epl, m->lpm_host[e + 1], addr)) best = (int)e;
        }
        if (best < 0) return -ENOENT;
        *(u8 *)value_out = (u8)m->lpm_host[best + 2];
        return 0;
    }
    default:
        return -EINVAL;
    }
}

int bng_map_delete(bng_ctx *c, int map, const void *key) {
    MapReg *m = get_map(c, map);
    if (!m || !key) return -EINVAL;
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    if (int fr = flush_staged_locked(c, map)) return fr;
    if (m->kind == KIND_HASH) {
        int first = 0;
        int r = hash_cmd(c, m, TOP_DELETE, key, nullptr, 1, 0, &first);
        if (!r && !first && feeds_small_tabs(m)) c->small_dirty = true;
        return r ? r : first;
    }
    if (m->kind == KIND_LPM) {
        const u32 *k = (const u32 *)key;
        for (size_t e = 0; e < m->lpm_host.size(); e += 3)
            if (m->lpm_host[e] == k[0] && lpm_same(k[0], m->lpm_host[e + 1], k[1])) {
                m->lpm_host.erase(m->lpm_host.begin() + e, m->lpm_host.begin() + e + 3);
                return lpm_upload(c, m);
            }
        return -ENOENT;
    }
    return -EINVAL; // arrays cannot be deleted from (kernel: -EINVAL)
}

static int64_t map_dump_locked(bng_ctx *c, MapReg *m, void *keys_out, void *values_out, uint64_t cap);

// Removes every entry of a hash map (the control plane's equivalent of closing and re-creating the map).
int bng_map_clear(bng_ctx *c, int map) {
    MapReg *m = get_map(c, map);
    if (!m || m->kind != KIND_HASH) return -EINVAL;
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    if (c->staged_total) { // staged Puts of a map that is being emptied are void
        bng_ctx::Staged &q = c->staged[map];
        c->staged_total -= q.n;
        q.keys.clear();
        q.vals.clear();
        q.n = 0;
    }
    const Tbl &t = *m->tbl;
    CU(c, cudaMemsetAsync(t.slots, 0xFF, ((size_t)t.mask + 1) * t.slot_bytes, c->L.stream));
    CU(c, cudaMemsetAsync(t.count, 0, 4, c->L.stream));
    if (t.plens) CU(c, cudaMemsetAsync(t.plens, 0, LPM6_LENS * 4, c->L.stream));
    if (m->tbl == &c->v6) c->v6_live = 0;
    if (m->tbl == &c->d6b) c->d6_live = 0;
    if (m->tbl == &c->ndb) c->nd_live = 0;
    if (m->tbl == &c->dev.sub_nat || m->tbl == &c->dev.qos_in)
        CU(c, run_dir_clear_half(c->L, c->dev.subdir, m->tbl == &c->dev.sub_nat ? 1 : 2));
    CU(c, cudaStreamSynchronize(c->L.stream));
    if (feeds_small_tabs(m)) c->small_dirty = true;
    return 0;
}

int64_t bng_map_dump(bng_ctx *c, int map, void *keys_out, void *values_out, uint64_t cap) {
    MapReg *m = get_map(c, map);
    if (!m || !keys_out || !values_out) return -EINVAL;
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    if (int fr = flush_staged_locked(c, map)) return fr;
    return map_dump_locked(c, m, keys_out, values_out, cap);
}

// Rebuilds the SmallTabs image from the authoritative device state of
// antispoof_config, nat_config_map, alg_ports and hairpin_ips and uploads it.
static int small_refresh(bng_ctx *c) {
    c->small_dirty = false;
    SmallTabs *im = new SmallTabs();
    memset(im, 0, sizeof(*im));
    for (u32 i = 0; i < HP_SLOTS; i++) im->hp_hash[i] = HP_EMPTY;
    u8 cfg[16];
    int rc = 0;
    cudaError_t e = cudaMemcpy(cfg, c->dev.as_config, 8, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) {
        im->as_cfg = (u32)cfg[0] | ((u32)cfg[1] << 8);
        e = cudaMemcpy(cfg, c->dev.nat_config, 16, cudaMemcpyDeviceToHost);
    }
    if (e == cudaSuccess) memcpy(&im->nat_flags, cfg, 4);
    if (e != cudaSuccess) rc = fail(c, -EIO, "small_refresh: %s", cudaGetErrorString(e));
    MapReg *alg = nullptr, *hp = nullptr;
    for (auto &m : c->maps) {
        if (!strcmp(m.name, "alg_ports")) alg = &m;
        if (!strcmp(m.name, "hairpin_ips")) hp = &m;
    }
    if (!rc && alg) {
        u32 keys[64];
        u8 vals[64 * 8];
        int64_t n = map_dump_locked(c, alg, keys, vals, 64);
        if (n < 0) rc = (int)n;
        for (int64_t i = 0; !rc && i < n; i++) {
            im->alg_key[i] = keys[i];
            im->alg_type[i] = vals[i * 8 + 3];
        }
        if (!rc) im->alg_n = (u32)n;
    }
    if (!rc && hp) {
        std::vector<u32> keys(1000);
        std::vector<u8> vals(1000);
        int64_t n = map_dump_locked(c, hp, keys.data(), vals.data(), 1000);
        if (n < 0) rc = (int)n;
        u32 bcast = 0;
        for (int64_t i = 0; !rc && i < n; i++) {
            if (keys[i] == HP_EMPTY) { // 255.255.255.255 cannot live in the u32 hash: flagged in hp_n bit 31
                bcast = 0x80000000u;
                continue;
            }
            u32 s = hp_index(keys[i]);
            while (im->hp_hash[s] != HP_EMPTY) s = (s + 1) & (HP_SLOTS - 1);
            im->hp_hash[s] = keys[i];
        }
        if (!rc) im->hp_n = (u32)n | bcast;
    }
    if (!rc) {
        e = cudaMemcpy((void *)c->dev.small, im, sizeof(SmallTabs), cudaMemcpyHostToDevice);
        if (e != cudaSuccess) rc = fail(c, -EIO, "small_refresh upload: %s", cudaGetErrorString(e));
    }
    delete im;
    return rc;
}

} // extern "C"
bool feeds_small_tabs_p(const MapReg *m) { return feeds_small_tabs(m); }
int small_refresh_p(bng_ctx *c) { return small_refresh(c); }
extern "C" {

static bool feeds_small_tabs(const MapReg *m) {
    return !strcmp(m->name, "antispoof_config") || !strcmp(m->name, "nat_config_map") || !strcmp(m->name, "alg_ports") ||
           !strcmp(m->name, "hairpin_ips");
}

static int64_t map_dump_locked(bng_ctx *c, MapReg *m, void *keys_out, void *values_out, uint64_t cap) {
    if (m->kind == KIND_LPM) {
        u64 n = std::min<u64>(cap, m->lpm_host.size() / 3);
        for (u64 i = 0; i < n; i++) {
            memcpy((u8 *)keys_out + i * 8, &m->lpm_host[3 * i], 8);
            ((u8 *)values_out)[i] = (u8)m->lpm_host[3 * i + 2];
        }
        return (int64_t)n;
    }
    if (m->kind == KIND_ARRAY || m->kind == KIND_STATS) {
        u64 n = std::min<u64>(cap, m->max_entries);
        const u8 *src = m->kind == KIND_ARRAY ? *m->arr : (const u8 *)(c->dev.stats + m->stat_base);
        for (u32 i = 0; i < n; i++) ((u32 *)keys_out)[i] = i;
        CU(c, cudaMemcpyAsync(values_out, src, n * m->value_size, cudaMemcpyDeviceToHost, c->L.stream));
        CU(c, cudaStreamSynchronize(c->L.stream));
        return (int64_t)n;
    }
    if (m->kind != KIND_HASH) return -EINVAL;
    if (cap == 0) return 0;
    const Tbl &t = *m->tbl;
    const size_t kb = std::max<size_t>(cap * t.key_size, 1 << 16), vb = std::max<size_t>(cap * t.value_size, 1 << 16);
    if (kb > c->dump_k.size() || vb > c->dump_v.size()) c->dump_k.reset(), c->dump_v.reset(); // both are sized for this dump
    if (!devbuf::grow_all({{&c->dump_k, kb}, {&c->dump_v, vb}, {&c->dump_c, 16}})) return grow_failed(c, "dump", kb + vb + 16);
    u8 *dk = c->dump_k, *dv = c->dump_v;
    u32 *dc = c->dump_c;
    int rc = 0;
    u32 cnt = 0;
    cudaMemsetAsync(dc, 0, 16, c->L.stream);
    cudaError_t e = run_table_dump(c->L, t, dk, dv, dc, cap);
    if (e == cudaSuccess) e = cudaMemcpyAsync(&cnt, dc, 4, cudaMemcpyDeviceToHost, c->L.stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->L.stream);
    if (e == cudaSuccess && cnt) {
        u64 n = std::min<u64>(cnt, cap);
        e = cudaMemcpy(keys_out, dk, n * t.key_size, cudaMemcpyDeviceToHost);
        if (e == cudaSuccess) e = cudaMemcpy(values_out, dv, n * t.value_size, cudaMemcpyDeviceToHost);
        cnt = (u32)n;
    }
    if (e != cudaSuccess) rc = fail(c, -EIO, "dump: %s", cudaGetErrorString(e));
    return rc ? rc : (int64_t)cnt;
}

// ---------------------------------------------------------------------------
// programs
// ---------------------------------------------------------------------------
static const char *const k_prog_names[] = {
    "antispoof_ingress",  // bpf/antispoof.c:188-189
    "qos_egress_prog",    // bpf/qos_ratelimit.c:126-127
    "qos_ingress_prog",   // bpf/qos_ratelimit.c:178-179
    "nat44_egress",       // bpf/nat44.c:565-566
    "nat44_ingress",      // bpf/nat44.c:805-806
    "nat44_hairpin_xdp",  // bpf/nat44.c:951-952
    "dhcp_fastpath_prog", // bpf/dhcp_fastpath.c:619-620
    "pipeline_up",        // antispoof_ingress -> nat44_egress -> qos_ingress_prog (pre-NAT key)
    "pipeline_tc",        // antispoof_ingress -> qos_ingress_prog -> nat44_egress: the order of the reference's TC hooks
};
enum { P_ANTISPOOF, P_QOS_EG, P_QOS_IN, P_NAT_EG, P_NAT_IN, P_NAT_HAIRPIN, P_DHCP, P_PIPE_UP, P_PIPE_TC, P_COUNT };

int bng_prog_id(bng_ctx *c, const char *name) {
    if (!c || !name) return -EINVAL;
    for (int i = 0; i < P_COUNT; i++)
        if (!strcmp(k_prog_names[i], name)) return i;
    return -ENOENT;
}

// the accounting mode of each program: where its frames' subscriber is found (-1: not accountable)
static const int k_acct_mode[] = {-1, ACCT_DST, ACCT_SRC, ACCT_ATTR, ACCT_DST, -1, -1, ACCT_ATTR, ACCT_ATTR};

// the interception direction of each program: BNG_LI_UPLINK (0), BNG_LI_DOWNLINK (1), -1: never captures
static const int k_li_dir[] = {-1, 1, 0, 0, 1, -1, -1, 0, 0};

// The storage of the caller's frames, for replies longer than their request (k_dhcp_fastpath<v6>, <nd>): room_stride bytes
// each, or 0: len rounded up to 16; need: the pinned zero-copy feed's bytes to scatter back, else nullptr.
struct FrameRoom {
    u32 room_stride;
    u32 *need;
};

// Are ICMP errors translated by the flow they quote in this program?  nat44_ingress: bng_nat_icmp_errors_enable;
// nat44_egress and the pipelines: bng_nat_icmp_errors_egress_enable.
static bool icmp_errors(const bng_ctx *c, int prog) {
    if (prog == P_NAT_IN) return c->nat_icmp;
    return (prog == P_NAT_EG || prog == P_PIPE_UP || prog == P_PIPE_TC) && c->nat_icmp_eg;
}

static int dispatch(bng_ctx *c, int prog, const DevBatch &b, const LiSrc &src = LiSrc{}, const FrameRoom *room = nullptr) {
    cudaError_t e = cudaSuccess;
    const bool acct = c->acct && ((c->acct_progs >> prog) & 1);
    const bool idle = c->idle && ((c->idle_progs >> prog) & 1);
    const int li = c->li_targets.empty() ? -1 : k_li_dir[prog]; // no target: not one kernel more
    const bool pipe = prog == P_PIPE_UP || prog == P_PIPE_TC;
    const Tbl *v6 = c->v6_live ? &c->v6 : nullptr; // an empty table launches exactly what it did before it existed
    const Tbl *qv6 = c->qos_v6 ? v6 : nullptr;     // ... and so does shaping IPv6 with it
    const Tbl *as6 = c->as_v6 ? v6 : nullptr;      // ... and antispoof allowing the prefixes' sources
    // the upstream classify records attributions: for accounting and idle detection, and in the pipelines to tell
    // antispoof's drops
    c->L.acct_attr = (acct || idle || (li == 0 && pipe)) ? c->L.s.attr : nullptr;
    LiRing r{};
    if (li >= 0) {
        r.buf = c->li_ring, r.ctl = c->li_ctl, r.match = c->li_match;
        r.cap = c->li_cap, r.rec_bytes = c->li_rec, r.snaplen = c->li_snap, r.prog = (u32)prog;
        r.tgt = AddrSet{c->li_words, c->li_mask}, r.ids = c->li_ids, r.batch = c->seq;
    }
    if (li == 0) { // the frames as they entered, before the program rewrites them
        e = cudaMemsetAsync(c->li_ctl + 2, 0, 4, c->L.stream);
        if (e == cudaSuccess) e = run_li_capture(c->L, r, b, src, true, v6);
        if (e != cudaSuccess) return fail(c, -EIO, "launch k_li_capture: %s", cudaGetErrorString(e));
    }
    switch (prog) {
    case P_ANTISPOOF: e = run_antispoof(c->L, c->dev, b, as6); break;
    case P_QOS_EG: e = run_qos(c->L, c->dev, b, true, qv6); break;
    case P_QOS_IN: e = run_qos(c->L, c->dev, b, false, qv6); break;
    case P_NAT_EG: e = run_nat_egress(c->L, c->dev, b, icmp_errors(c, prog)); break;
    case P_NAT_IN: e = run_nat_ingress(c->L, c->dev, b, icmp_errors(c, prog)); break;
    case P_NAT_HAIRPIN: e = run_nat_hairpin_xdp(c->L, c->dev, b); break;
    case P_DHCP: {
        // DHCPv6 needs the switch, a configured server and a binding: otherwise "on" launches what "off" does
        Dhcp6Args d6{};
        const bool v6 = c->dhcp6 && c->d6_live && c->d6cfg_host[6];
        if (v6) {
            d6.bind = c->d6b, d6.cfg = c->d6cfg, d6.stats = c->dev.stats + ST_DHCP6;
            d6.room_stride = room ? room->room_stride : (b.off16 ? 0u : b.stride);
            d6.need = room ? room->need : nullptr;
        }
        // ND needs the switch and a configured nd_config (NS answers need no binding)
        NdArgs nd{};
        const bool ndo = c->nd && (c->ndcfg_host[8] | c->ndcfg_host[9]);
        if (ndo) {
            nd.bind = c->ndb, nd.cfg = c->ndcfg, nd.stats = c->dev.stats + ST_ND;
            nd.room_stride = room ? room->room_stride : (b.off16 ? 0u : b.stride);
            nd.need = room ? room->need : nullptr;
        }
        e = run_dhcp_fastpath(c->L, c->dev, b, v6 ? &d6 : nullptr, ndo ? &nd : nullptr);
        break;
    }
    case P_PIPE_UP: e = run_pipeline_up(c->L, c->dev, b, qv6, as6, icmp_errors(c, prog)); break;
    case P_PIPE_TC: e = run_pipeline_tc(c->L, c->dev, b, qv6, as6, icmp_errors(c, prog)); break;
    default: return -EINVAL;
    }
    // after the program, before anything copies the frames out: the downstream modes read the rewritten headers
    if (e == cudaSuccess && (acct || idle)) e = run_acct(c->L, c->dev.subdir, b, k_acct_mode[prog], acct ? c->acct.get() : nullptr, idle ? c->idle.get() : nullptr, v6);
    if (e == cudaSuccess && li == 0) e = run_li_verdict(c->L, r, b, pipe ? c->L.s.attr : nullptr);
    if (e == cudaSuccess && li == 1) e = run_li_capture(c->L, r, b, src, false, v6);
    if (e != cudaSuccess) return fail(c, -EIO, "launch %s: %s", k_prog_names[prog], cudaGetErrorString(e));
    return 0;
}

// BNG_MEM_HOST with a pinned arena: chunked three-stage pipeline
//   s_in   : header gather straight from the mapped host arena (+ offsets / lengths H2D)
//   stream : the program on the compact device copy (chunks strictly in order: index-order semantics)
//   s_out  : header scatter back into the host arena (+ verdict / length D2H)
// so PCIe reads, PCIe writes and compute of successive chunks overlap, and only the bytes a
// program can touch ever cross the bus.
#define ZC_CHUNK (c->zc_chunk)
static int maybe_compact_locked(bng_ctx *c);
static int poll_compact_locked(bng_ctx *c);
static int queue_evict_read_locked(bng_ctx *c);
static int li_upload_locked(bng_ctx *c);
static int run_host_zero_copy(bng_ctx *c, int prog, bng_batch *bb, u8 *arena_dev) {
    // Bytes of a frame a program can touch (hostio.cu): 96 for the TC programs (Ethernet + IPv4 with options + 20
    // bytes of L4), 448 for dhcp_fastpath_prog.  Frames that ARE a fixed slot no larger than that (64-byte
    // frames, a header-split receive ring) move as they are with the copy engines.
    const bool tc = prog != P_DHCP;
    const u32 hb_need = tc ? 96u : 448u;
    const bool contiguous = !bb->off16 && bb->stride <= hb_need;
    const u32 hb = contiguous ? bb->stride : hb_need;         // compact slot stride
    // The TC programs write below byte 16 only in frames with ihl = 0, but the first 16 bytes are written back all
    // the same: ONE 64-byte PCIe write per frame rather than a 16- and a 32-byte one (what the link counts is TLPs,
    // not bytes).
    for (cudaStream_t *st : {&c->s_in, &c->s_out})
        if (!*st) CU(c, cudaStreamCreateWithFlags(st, cudaStreamNonBlocking));
    for (int i = 0; i < ZC_BUFS; i++)
        for (cudaEvent_t *ev : {&c->ev_in[i], &c->ev_comp[i], &c->ev_out[i]})
            if (!*ev) CU(c, cudaEventCreateWithFlags(ev, cudaEventDisableTiming));
    devbuf::Want zc[ZC_BUFS * 7];
    const size_t cw = (size_t)ZC_CHUNK * 4, hdr = (size_t)ZC_CHUNK * hb + 64;
    for (int i = 0; i < ZC_BUFS; i++) {
        devbuf::Want *w = zc + 7 * i;
        w[0] = {&c->zc_off[i], cw}, w[1] = {&c->zc_len[i], cw}, w[2] = {&c->zc_len0[i], cw}, w[3] = {&c->zc_prio[i], cw};
        w[4] = {&c->zc_verdict[i], ZC_CHUNK}, w[5] = {&c->zc_now[i], (size_t)ZC_CHUNK * 8}, w[6] = {&c->zc_hdr[i], hdr};
    }
    if (!devbuf::grow_all(zc)) return grow_failed(c, "zero-copy staging", ZC_BUFS * (6 * cw + hdr));
    cudaStream_t sc = c->L.stream;
    const u32 nchunks = (bb->n + ZC_CHUNK - 1) / ZC_CHUNK;
    // BNG_ZC_TRACE=1: a timeline of the three stages of every chunk on stderr (timing events on the three streams)
    static const bool trace = getenv("BNG_ZC_TRACE") != nullptr;
    std::vector<cudaEvent_t> tev;
    auto mark = [&](cudaStream_t st) {
        if (!trace) return;
        cudaEvent_t e;
        cudaEventCreate(&e);
        cudaEventRecord(e, st);
        tev.push_back(e);
    };
    mark(c->s_in); // t0
    for (u32 k = 0; k < nchunks; k++) {
        const int buf = k % ZC_BUFS;
        const u32 base = k * ZC_CHUNK, cn = std::min<u32>(ZC_CHUNK, bb->n - base);
        // ---- in ----
        if (k >= ZC_BUFS) CU(c, cudaStreamWaitEvent(c->s_in, c->ev_out[buf], 0));
        mark(c->s_in);
        if (bb->off16) CU(c, cudaMemcpyAsync(c->zc_off[buf], bb->off16 + base, (size_t)cn * 4, cudaMemcpyHostToDevice, c->s_in));
        CU(c, cudaMemcpyAsync(c->zc_len[buf], bb->len + base, (size_t)cn * 4, cudaMemcpyHostToDevice, c->s_in));
        if (bb->priority)
            CU(c, cudaMemcpyAsync(c->zc_prio[buf], bb->priority + base, (size_t)cn * 4, cudaMemcpyHostToDevice, c->s_in));
        if (bb->now_ns_v)
            CU(c, cudaMemcpyAsync(c->zc_now[buf], bb->now_ns_v + base, (size_t)cn * 8, cudaMemcpyHostToDevice, c->s_in));
        u8 *chunk_arena = bb->off16 ? arena_dev : arena_dev + (size_t)base * bb->stride;
        if (contiguous) {
            CU(c, cudaMemcpyAsync(c->zc_hdr[buf], (u8 *)bb->pkts + (size_t)base * hb, (size_t)cn * hb, cudaMemcpyHostToDevice,
                                  c->s_in));
        } else {
            CU(c, run_gather_frames(c->s_in, c->L.num_sms, chunk_arena, bb->off16 ? c->zc_off[buf].get() : nullptr, c->zc_len[buf],
                                    bb->stride, cn, hb, tc, icmp_errors(c, prog), c->zc_hdr[buf], c->zc_len0[buf]));
            c->L.launches++;
        }
        CU(c, cudaEventRecord(c->ev_in[buf], c->s_in));
        mark(c->s_in);
        // ---- compute ----
        CU(c, cudaStreamWaitEvent(sc, c->ev_in[buf], 0));
        mark(sc);
        DevBatch b{};
        b.pkts = c->zc_hdr[buf];
        b.off16 = nullptr;
        b.len = c->zc_len[buf];
        b.verdict = c->zc_verdict[buf];
        b.priority = bb->priority ? c->zc_prio[buf].get() : nullptr;
        b.n = cn;
        b.stride = hb;
        b.now = bb->now_ns;
        b.nowv = bb->now_ns_v ? c->zc_now[buf].get() : nullptr;
        b.base = base;
        b.cap = hb; // bounds checks never look past a compact slot (a no-op for whole frames: hostio.cu)
        b.arena_len = (u64)cn * hb;
        // interception copies the bytes past the compact copy straight from the host arena
        const LiSrc src{chunk_arena, bb->off16 ? c->zc_off[buf].get() : nullptr, contiguous ? nullptr : c->zc_len0[buf].get(), bb->stride};
        // a DHCPv6 or ND reply may outgrow its request: bounded by the host frame's storage, written back up to its length
        const FrameRoom room{bb->off16 ? 0u : bb->stride, contiguous ? nullptr : c->zc_len0[buf].get()};
        int r = dispatch(c, prog, b, src, &room);
        if (r) return r;
        CU(c, cudaEventRecord(c->ev_comp[buf], sc));
        mark(sc);
        // ---- out ----
        CU(c, cudaStreamWaitEvent(c->s_out, c->ev_comp[buf], 0));
        mark(c->s_out);
        if (contiguous) {
            CU(c, cudaMemcpyAsync((u8 *)bb->pkts + (size_t)base * hb, c->zc_hdr[buf], (size_t)cn * hb, cudaMemcpyDeviceToHost,
                                  c->s_out));
        } else {
            CU(c, run_scatter_frames(c->s_out, c->L.num_sms, chunk_arena, bb->off16 ? c->zc_off[buf].get() : nullptr, c->zc_len0[buf],
                                     bb->stride, cn, hb, c->zc_hdr[buf]));
            c->L.launches++;
        }
        CU(c, cudaMemcpyAsync(bb->verdict + base, c->zc_verdict[buf], cn, cudaMemcpyDeviceToHost, c->s_out));
        if (prog == P_DHCP)
            CU(c, cudaMemcpyAsync(bb->len + base, c->zc_len[buf], (size_t)cn * 4, cudaMemcpyDeviceToHost, c->s_out));
        if (bb->priority)
            CU(c, cudaMemcpyAsync(bb->priority + base, c->zc_prio[buf], (size_t)cn * 4, cudaMemcpyDeviceToHost, c->s_out));
        CU(c, cudaEventRecord(c->ev_out[buf], c->s_out));
        mark(c->s_out);
    }
    CU(c, cudaStreamSynchronize(c->s_out));
    CU(c, cudaStreamSynchronize(sc));
    if (trace) {
        for (u32 k = 0; k < nchunks; k++) {
            float t[6];
            for (int j = 0; j < 6; j++) cudaEventElapsedTime(&t[j], tev[0], tev[1 + 6 * k + j]);
            fprintf(stderr, "zc chunk %u: in %.3f-%.3f  compute %.3f-%.3f  out %.3f-%.3f ms\n", k, t[0], t[1], t[2], t[3], t[4], t[5]);
        }
        for (cudaEvent_t e : tev) cudaEventDestroy(e);
    }
    prof_collect(c->L);
    return maybe_compact_locked(c);
}

int bng_prog_run(bng_ctx *c, int prog, bng_batch *bb) {
    if (!c || !bb || prog < 0 || prog >= P_COUNT) return -EINVAL;
    if (bb->n == 0) return 0;
    if (!bb->pkts || !bb->len || !bb->verdict) return -EINVAL;
    if (!bb->off16 && (bb->stride == 0 || (bb->stride & 15))) return -EINVAL;
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    int r = ensure_scratch(c, bb->n);
    if (r) return r;
    if ((r = poll_compact_locked(c)) != 0) return r;     // what an earlier device-resident batch left to compact
    if ((r = flush_staged_locked(c, -1)) != 0) return r; // the batch boundary: staged upserts become visible
    if (c->small_dirty && (r = small_refresh_p(c)) != 0) return r; // ... and the shared-memory image of the small maps is rebuilt
    if (c->li_dirty && (r = li_upload_locked(c)) != 0) return r;   // ... and the interception targets in force now
    c->seq++;
    c->dev.batch_seq++;
    c->dev.epoch = c->dev.batch_seq % 65535u + 1; // what a session hit stamps next to last_seen (common.cuh)
    if (c->dev.epoch == 1 && c->dev.batch_seq > 1) CU(c, run_epoch_reset(c->L, c->dev.sessions)); // the 16-bit stamp wraps
    DevBatch b{};
    b.n = bb->n;
    b.stride = bb->stride;
    b.now = bb->now_ns;
    // bytes the kernels may touch from pkts: a fixed-stride arena holds n * stride; with an offset table
    // the caller's arena_bytes (16-byte units, possibly rounded up) says, and 0 means unknown
    b.arena_len = bb->off16 ? (bb->arena_bytes ? (u64)bb->arena_bytes * 16 - 15 : 0) : (u64)bb->n * bb->stride;
    b.cap = bb->off16 ? 0u : bb->stride; // a fixed-stride slot holds at most stride bytes of its frame
    if (bb->mem == BNG_MEM_HOST && bb->now_ns_v) // the per-frame clock is monotonic (bpf_ktime_get_ns)
        for (u32 i = 1; i < bb->n; i++)
            if (bb->now_ns_v[i] < bb->now_ns_v[i - 1]) return fail(c, -EINVAL, "now_ns_v is not non-decreasing at frame %u", i);
    if (bb->mem == BNG_MEM_DEVICE) {
        b.nowv = (const u64 *)bb->now_ns_v;
        b.pkts = (u8 *)bb->pkts;
        b.off16 = bb->off16;
        b.len = bb->len;
        b.verdict = bb->verdict;
        b.priority = bb->priority;
        if ((r = dispatch(c, prog, b)) != 0) return r;
        // only the programs that create flows evict from the flow tables
        return (prog == P_NAT_EG || prog == P_PIPE_UP || prog == P_PIPE_TC) ? queue_evict_read_locked(c) : 0;
    }
    if (bb->mem != BNG_MEM_HOST) return -EINVAL;
    {
        // Pinned (cudaHostAlloc / cudaHostRegister) arenas are read in place.  The pointer's registered type is
        // what decides: on systems with HMM / ATS cudaHostGetDevicePointer() also succeeds for PAGEABLE memory,
        // which the GPU would then reach through page faults.
        cudaPointerAttributes at{};
        void *mapped = nullptr;
        if (cudaPointerGetAttributes(&at, bb->pkts) == cudaSuccess && at.type == cudaMemoryTypeHost &&
            cudaHostGetDevicePointer(&mapped, bb->pkts, 0) == cudaSuccess && mapped)
            return run_host_zero_copy(c, prog, bb, (u8 *)mapped);
        cudaGetLastError(); // pageable memory: whole-arena staging copies
    }
    size_t arena = bb->off16 ? (size_t)bb->arena_bytes * 16 : (size_t)bb->n * bb->stride;
    if (arena == 0) return -EINVAL;
    cudaStream_t st = c->L.stream;
    const size_t fw = (size_t)bb->n * 4;
    if (!devbuf::grow_all({{&c->hb_pkts, arena}, {&c->hb_off, fw}, {&c->hb_len, fw}, {&c->hb_prio, fw}, {&c->hb_verdict, bb->n},
                           {&c->hb_now, (size_t)bb->n * 8}}))
        return grow_failed(c, "host staging", arena + (size_t)bb->n * 21);
    CU(c, cudaMemcpyAsync(c->hb_pkts, bb->pkts, arena, cudaMemcpyHostToDevice, st));
    if (bb->off16) CU(c, cudaMemcpyAsync(c->hb_off, bb->off16, (size_t)bb->n * 4, cudaMemcpyHostToDevice, st));
    CU(c, cudaMemcpyAsync(c->hb_len, bb->len, (size_t)bb->n * 4, cudaMemcpyHostToDevice, st));
    if (bb->priority) CU(c, cudaMemcpyAsync(c->hb_prio, bb->priority, (size_t)bb->n * 4, cudaMemcpyHostToDevice, st));
    if (bb->now_ns_v) CU(c, cudaMemcpyAsync(c->hb_now, bb->now_ns_v, (size_t)bb->n * 8, cudaMemcpyHostToDevice, st));
    b.nowv = bb->now_ns_v ? c->hb_now.get() : nullptr;
    b.pkts = c->hb_pkts;
    b.off16 = bb->off16 ? c->hb_off.get() : nullptr;
    b.len = c->hb_len;
    b.verdict = c->hb_verdict;
    b.priority = bb->priority ? c->hb_prio.get() : nullptr;
    r = dispatch(c, prog, b);
    if (r) return r;
    CU(c, cudaMemcpyAsync(bb->pkts, c->hb_pkts, arena, cudaMemcpyDeviceToHost, st));
    CU(c, cudaMemcpyAsync(bb->len, c->hb_len, (size_t)bb->n * 4, cudaMemcpyDeviceToHost, st));
    CU(c, cudaMemcpyAsync(bb->verdict, c->hb_verdict, (size_t)bb->n, cudaMemcpyDeviceToHost, st));
    if (bb->priority) CU(c, cudaMemcpyAsync(bb->priority, c->hb_prio, (size_t)bb->n * 4, cudaMemcpyDeviceToHost, st));
    CU(c, cudaStreamSynchronize(st));
    prof_collect(c->L);
    return maybe_compact_locked(c);
}

int bng_sync(bng_ctx *c) {
    if (!c) return -EINVAL;
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    int r = flush_staged_locked(c, -1);
    CU(c, cudaStreamSynchronize(c->L.stream));
    prof_collect(c->L);
    if (!r) r = maybe_compact_locked(c);
    return r;
}

int bng_map_update_staged(bng_ctx *c, int map, const void *key, const void *value) {
    MapReg *m = get_map(c, map);
    if (!m || !key || !value) return -EINVAL;
    if (m->kind != KIND_HASH) return bng_map_update(c, map, key, value, BNG_ANY); // arrays / tries: nothing to batch
    if (m->tbl == &c->d6b && d6_bad_binding((const u8 *)key, (const u8 *)value)) return -EINVAL;
    if (m->tbl == &c->ndb && nd_bad_binding((const u8 *)value)) return -EINVAL;
    std::lock_guard<std::mutex> g(c->mu);
    bng_ctx::Staged &q = c->staged[map];
    q.keys.insert(q.keys.end(), (const u8 *)key, (const u8 *)key + m->key_size);
    if (m->tbl == &c->v6) { // the last staged value of a prefix wins, however its key was spelled
        u8 *k = q.keys.data() + q.keys.size() - m->key_size;
        u32 pl;
        memcpy(&pl, k, 4);
        if (pl >= LPM6_LENS) {
            q.keys.resize(q.keys.size() - m->key_size);
            return -EINVAL;
        }
        v6_mask_key(k);
    }
    q.vals.insert(q.vals.end(), (const u8 *)value, (const u8 *)value + m->value_size);
    q.n++;
    c->staged_total++;
    if (q.n >= (1u << 18)) { // bound the host-side queue
        cudaSetDevice(c->device);
        return flush_staged_locked(c, map);
    }
    return 0;
}

int bng_staged_info(bng_ctx *c, uint64_t *pending, uint64_t *flushes, uint64_t *errors) {
    if (!c) return -EINVAL;
    std::lock_guard<std::mutex> g(c->mu);
    if (pending) *pending = c->staged_total;
    if (flushes) *flushes = c->staged_flushes;
    if (errors) *errors = c->staged_errors;
    return 0;
}

// ---- multi-GPU reconciliation ----
int bng_comm_unique_id(void *id_out, uint64_t cap) {
    if (!id_out || cap < sizeof(ncclUniqueId)) return -EINVAL;
    NcclApi *a = nccl_api();
    if (!a) return -ENOSYS;
    ncclUniqueId id;
    if (a->GetUniqueId(&id) != ncclSuccess) return -EIO;
    memcpy(id_out, &id, sizeof(id));
    return 0;
}

int bng_comm_init(bng_ctx *c, const void *id, uint32_t rank, uint32_t world) {
    if (!c || !id || world == 0 || rank >= world) return -EINVAL;
    NcclApi *a = nccl_api();
    if (!a) return fail(c, -ENOSYS, "NCCL is not available in this process (set BNG_NCCL_LIB)");
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    if (c->comm) return fail(c, -EEXIST, "communicator already initialised");
    ncclUniqueId uid;
    memcpy(&uid, id, sizeof(uid));
    ncclResult_t r = a->CommInitRank(&c->comm, (int)world, uid, (int)rank);
    if (r != ncclSuccess) {
        c->comm = nullptr;
        return fail(c, -EIO, "ncclCommInitRank: %s", a->GetErrorString ? a->GetErrorString(r) : "error");
    }
    c->comm_rank = rank;
    c->comm_world = world;
    return 0;
}

int bng_sync_reduce(bng_ctx *c, uint64_t *totals_out) {
    if (!c) return -EINVAL;
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    int fr = flush_staged_locked(c, -1);
    if (!c->stats_global.grow(ST_ALL * 8)) return grow_failed(c, "sync_reduce", ST_ALL * 8);
    if (c->comm) {
        NcclApi *a = nccl_api();
        ncclResult_t r = a->AllReduce(c->dev.stats, c->stats_global, ST_ALL, ncclUint64, ncclSum, c->comm, c->L.stream);
        if (r != ncclSuccess) return fail(c, -EIO, "ncclAllReduce: %s", a->GetErrorString ? a->GetErrorString(r) : "error");
    } else {
        CU(c, cudaMemcpyAsync(c->stats_global, c->dev.stats, ST_ALL * 8, cudaMemcpyDeviceToDevice, c->L.stream));
    }
    if (totals_out) CU(c, cudaMemcpyAsync(totals_out, c->stats_global, ST_COUNT * 8, cudaMemcpyDeviceToHost, c->L.stream));
    CU(c, cudaStreamSynchronize(c->L.stream));
    prof_collect(c->L);
    return fr;
}

void *bng_stream(bng_ctx *c) { return c ? (void *)c->L.stream : nullptr; }

// Rebuilds a hash table in place (same capacity): what deletes, expiry and eviction left as tombstones is gone and
// every probe chain is as short as the load factor allows.  Only for tables nothing else indexes by slot number
// (the NAT flow tables; subscriber_nat / qos_ingress slots are referenced by the subscriber directory).
static int table_rebuild_locked(bng_ctx *c, Tbl *t, bool flow = true) {
    Tbl nw = *t;
    nw.lru = LRU_NONE;
    nw.max_entries = nw.mask; // the copy must never refuse or evict
    size_t bytes = ((size_t)t->mask + 1) * t->slot_bytes;
    DevBuf<u8> slots;
    DevBuf<u32> cnt;
    if (!devbuf::grow_all({{&slots, bytes}, {&cnt, 16}})) return grow_failed(c, "rebuild", bytes + 16);
    nw.slots = slots, nw.count = cnt;
    cudaError_t e = cudaMemsetAsync(nw.slots, 0xFF, bytes, c->L.stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(cnt, 0, 16, c->L.stream);
    if (e == cudaSuccess) e = run_table_rebuild(c->L, *t, nw);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->L.stream);
    if (e != cudaSuccess) return fail(c, -EIO, "rebuild: %s", cudaGetErrorString(e));
    for (auto &p : c->allocs)
        if (p == t->slots) p = nw.slots;
    DevBuf<u8> old(t->slots, bytes); // the table's slots before the rebuild, freed on return
    t->slots = slots.release();
    (flow ? c->rebuilds : c->lease_rebuilds)++;
    return 0;
}

// Tombstone compaction between batches: every eviction from a full LRU table leaves a tombstone, and a table that
// churns at capacity runs out of EMPTY slots (every lookup of an absent key then walks the whole table).  Rebuilds
// the three flow tables once the evictions since the last rebuild exceed a quarter of nat_sessions' slots, given
// the eviction count `ev` read at some point of the stream after the last rebuild.
static int compact_if_due_locked(bng_ctx *c, u64 ev) {
    if (ev - c->evict_at_rebuild <= (c->dev.sessions.mask + 1) / 4) return 0;
    c->evict_at_rebuild = ev;
    int r;
    if ((r = table_rebuild_locked(c, &c->dev.sessions)) != 0) return r;
    if ((r = table_rebuild_locked(c, &c->dev.reverse)) != 0) return r;
    return table_rebuild_locked(c, &c->dev.eim);
}

// Where the stream is synchronised anyway (host-fed batches, bng_sync): the count as of now.
static int maybe_compact_locked(bng_ctx *c) {
    u64 ev = 0;
    CU(c, cudaMemcpyAsync(&ev, c->dev.stats + ST_LRU_EVICT, 8, cudaMemcpyDeviceToHost, c->L.stream));
    CU(c, cudaStreamSynchronize(c->L.stream));
    c->evict_pending = false; // (a queued read is older than this one)
    return compact_if_due_locked(c, ev);
}

// A BNG_MEM_DEVICE batch returns without synchronising: it queues a copy of the eviction count behind itself, and
// the next bng_prog_run / bng_sweep applies the rule to it if the copy has landed by then (else a later call does).
// The steady state costs one 8-byte copy per batch and no host wait; only a rebuild itself synchronises.
static int queue_evict_read_locked(bng_ctx *c) {
    if (!c->evict_word.grow(8)) return grow_failed(c, "evict_word", 8);
    if (!c->evict_ev) CU(c, cudaEventCreateWithFlags(&c->evict_ev, cudaEventDisableTiming));
    CU(c, cudaMemcpyAsync(c->evict_word, c->dev.stats + ST_LRU_EVICT, 8, cudaMemcpyDeviceToHost, c->L.stream));
    CU(c, cudaEventRecord(c->evict_ev, c->L.stream));
    c->evict_pending = true;
    return 0;
}

static int poll_compact_locked(bng_ctx *c) {
    if (!c->evict_pending) return 0;
    const cudaError_t e = cudaEventQuery(c->evict_ev);
    if (e == cudaErrorNotReady) return 0;
    c->evict_pending = false;
    CU(c, e);
    return compact_if_due_locked(c, *(volatile u64 *)c->evict_word);
}

// After a pass that removes flow state (bng_sweep, bng_nat_flush), given the nat_sessions tombstones it counted:
// once a quarter of nat_sessions' slots are tombstones, rebuild the three flow tables (they churn together).
static int rebuild_if_tombstoned_locked(bng_ctx *c, u32 tombs) {
    if (tombs <= (c->dev.sessions.mask + 1) / 4) return 0;
    int r;
    if ((r = table_rebuild_locked(c, &c->dev.sessions)) != 0) return r;
    if ((r = table_rebuild_locked(c, &c->dev.reverse)) != 0) return r;
    return table_rebuild_locked(c, &c->dev.eim);
}

// Start of a pass over the flow tables that is a batch of its own between program runs (bng_sweep, bng_nat_flush):
// staged upserts first, then the batch sequence advances as a program run's does.
static int flow_pass_begin_locked(bng_ctx *c) {
    int r = poll_compact_locked(c);
    if (r) return r;
    if ((r = flush_staged_locked(c, -1)) != 0) return r;
    c->seq++;
    c->dev.batch_seq++;
    c->dev.epoch = c->dev.batch_seq % 65535u + 1;
    if (c->dev.epoch == 1 && c->dev.batch_seq > 1) CU(c, run_epoch_reset(c->L, c->dev.sessions));
    return 0;
}

// Session expiry sweep (sweep.cu): removes every nat_sessions entry idle for longer than the timeout of its
// protocol / TCP state at now_ns, with its nat_reverse entry, its EIM reference, the subscriber's active-session
// count; counts sessions_expired and logs NAT_LOG_SESSION_DELETE.  A batch of its own between program runs.
int bng_sweep(bng_ctx *c, uint64_t now_ns, uint64_t *expired_out) {
    if (!c) return -EINVAL;
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    int r = flow_pass_begin_locked(c);
    if (r) return r;
    u32 *cnt = c->L.s.counters + 8; // scratch words 8.. are free between program runs
    CU(c, cudaMemsetAsync(cnt, 0, 8, c->L.stream));
    CU(c, run_nat_sweep(c->L, c->dev, now_ns, cnt));
    u32 n[2] = {0, 0};
    CU(c, cudaMemcpyAsync(n, cnt, 8, cudaMemcpyDeviceToHost, c->L.stream));
    CU(c, cudaStreamSynchronize(c->L.stream));
    prof_collect(c->L);
    if (expired_out) *expired_out = n[0];
    return rebuild_if_tombstoned_locked(c, n[1]);
}

// NAT flow-state flush of a set of subscriber addresses (flush.cu).  The set is built here in the pinned staging
// buffer and copied behind whatever the stream already holds.
int bng_nat_flush(bng_ctx *c, const uint32_t *addrs, uint64_t n, uint64_t now_ns, uint64_t removed_out[3]) {
    if (!c || (n && !addrs)) return -EINVAL;
    if (removed_out) removed_out[0] = removed_out[1] = removed_out[2] = 0;
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    if (n == 0) return flush_staged_locked(c, -1);
    u64 slots = 64;
    while (slots < 2 * n) slots *= 2;
    if (slots > (1ull << 32)) return fail(c, -EINVAL, "nat_flush: %llu addresses", (unsigned long long)n);
    int r = flow_pass_begin_locked(c);
    if (r) return r;
    if ((r = ensure_io(c, slots * 8)) != 0) return r;
    u64 *set = (u64 *)c->io_host.get();
    memset(set, 0, slots * 8);
    const u32 mask = (u32)(slots - 1);
    for (u64 k = 0; k < n; k++) {
        u32 i = aset_home(addrs[k], mask);
        while (set[i] && (u32)set[i] != addrs[k]) i = (i + 1) & mask;
        set[i] = ADDRSET_LIVE | addrs[k];
    }
    CU(c, cudaMemcpyAsync(c->io_dev, c->io_host, slots * 8, cudaMemcpyHostToDevice, c->L.stream));
    u32 *cnt = c->L.s.counters + 8; // scratch words 8.. are free between program runs
    CU(c, cudaMemsetAsync(cnt, 0, 16, c->L.stream));
    CU(c, run_nat_flush(c->L, c->dev, AddrSet{(const u64 *)c->io_dev.get(), mask}, now_ns, cnt));
    u32 got[4] = {0, 0, 0, 0};
    CU(c, cudaMemcpyAsync(got, cnt, 16, cudaMemcpyDeviceToHost, c->L.stream));
    CU(c, cudaStreamSynchronize(c->L.stream));
    prof_collect(c->L);
    if (removed_out)
        for (int k = 0; k < 3; k++) removed_out[k] = got[k];
    return rebuild_if_tombstoned_locked(c, got[3]);
}

// ---------------------------------------------------------------------------
// events
// ---------------------------------------------------------------------------
uint32_t bng_event_size(bng_ctx *c, int map) {
    MapReg *m = get_map(c, map);
    return (m && m->kind == KIND_EVENT) ? m->ev_payload : 0;
}

int bng_events_drain(bng_ctx *c, int map, void *buf, uint64_t cap_records, uint64_t *n_out) {
    MapReg *m = get_map(c, map);
    if (!m || m->kind != KIND_EVENT || !n_out) return -EINVAL;
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    EvRing &r = *m->ring;
    u32 cnt = 0;
    CU(c, cudaMemcpyAsync(&cnt, r.count, 4, cudaMemcpyDeviceToHost, c->L.stream));
    CU(c, cudaStreamSynchronize(c->L.stream));
    if (cnt > r.cap) cnt = r.cap;
    if (cnt) {
        std::vector<u8> raw((size_t)cnt * r.rec_bytes);
        CU(c, cudaMemcpy(raw.data(), r.buf, raw.size(), cudaMemcpyDeviceToHost));
        CU(c, cudaMemsetAsync(r.count, 0, 4, c->L.stream));
        CU(c, cudaStreamSynchronize(c->L.stream));
        // emission order of the reference: batch order, then frame index
        std::vector<u32> order(cnt);
        for (u32 i = 0; i < cnt; i++) order[i] = i;
        const u8 *base = raw.data();
        u32 rb = r.rec_bytes;
        const u32 payload = m->ev_payload;
        std::sort(order.begin(), order.end(), [&](u32 a, u32 b) {
            const u32 *ta = (const u32 *)(base + (size_t)a * rb + rb - 8);
            const u32 *tb = (const u32 *)(base + (size_t)b * rb + rb - 8);
            if (ta[1] != tb[1]) return ta[1] < tb[1];
            if (ta[0] != tb[0]) return ta[0] < tb[0];
            // records of one sweep (marker 0xFFFFFFFE, no frame index): by content, so the order is defined
            return memcmp(base + (size_t)a * rb + 8, base + (size_t)b * rb + 8, payload - 8) < 0;
        });
        // BPF_MAP_TYPE_RINGBUF capacity: 8-byte header + payload rounded to 8;
        // a reserve fails once producer-consumer distance would exceed size-1
        u64 per = ((u64)m->ev_payload + 8 + 7) & ~7ull;
        u64 used = (m->ev_pending.size() / m->ev_payload) * per;
        for (u32 i = 0; i < cnt; i++) {
            const u32 *tag = (const u32 *)(base + (size_t)order[i] * rb + rb - 8);
            if (tag[0] == 0xFFFFFFFFu) continue; // reserved by the resolve kernel but never written
            if (m->type == T_RINGBUF) {
                if (used + per > (u64)m->max_entries - 1) continue; // bpf_ringbuf_reserve() == NULL
                used += per;
            }
            const u8 *rec = base + (size_t)order[i] * rb;
            m->ev_pending.insert(m->ev_pending.end(), rec, rec + m->ev_payload);
        }
    }
    u64 have = m->ev_pending.size() / m->ev_payload;
    u64 n = std::min<u64>(have, cap_records);
    if (n && buf) memcpy(buf, m->ev_pending.data(), n * m->ev_payload);
    if (n) m->ev_pending.erase(m->ev_pending.begin(), m->ev_pending.begin() + n * m->ev_payload);
    *n_out = n;
    return 0;
}

// ---------------------------------------------------------------------------
// per-subscriber traffic accounting (acct.cu)
// ---------------------------------------------------------------------------
static_assert(sizeof(bng_acct) == ACCT_WORDS * 8, "struct bng_acct is the device record");

// The records (one per directory slot) and the per-frame attribution words, on first use.
static int acct_alloc_locked(bng_ctx *c) {
    if (c->acct) return 0;
    // a failure releases the whole batch scratch (all or none): the next batch grows it again for its own size
    if (int r = scratch_locked(c, c->L.s.cap, true, c->li_ctl)) return r;
    const size_t bytes = ((size_t)c->dev.subdir.mask + 1) * sizeof(bng_acct);
    if (!c->acct.grow(bytes)) return grow_failed(c, "accounting", bytes);
    CU(c, cudaMemsetAsync(c->acct, 0, bytes, c->L.stream));
    return 0;
}

// the directory follows subscriber_nat and qos_ingress: their staged upserts come first
static int acct_flush_locked(bng_ctx *c) {
    for (const char *m : {"subscriber_nat", "qos_ingress"})
        if (int fr = flush_staged_locked(c, bng_map_id(c, m))) return fr;
    return 0;
}

static int64_t acct_dump_locked(bng_ctx *c, uint32_t *addrs_out, bng_acct *out, uint64_t cap) {
    if (cap == 0) return 0;
    const u64 ecap = std::min<u64>(cap, (u64)c->dev.subdir.mask + 1); // no more entries than slots
    const size_t aoff = ecap * sizeof(bng_acct), coff = (aoff + ecap * 4 + 15) & ~(size_t)15, need = coff + 16;
    if (!c->acct_dump_buf.grow(need)) return grow_failed(c, "acct_dump", need);
    u8 *buf = c->acct_dump_buf;
    u32 *cnt = (u32 *)(buf + coff), n = 0;
    CU(c, cudaMemsetAsync(cnt, 0, 4, c->L.stream));
    CU(c, run_acct_dump(c->L, c->dev.subdir, c->acct, (u32 *)(buf + aoff), (u64 *)buf, cnt, ecap));
    CU(c, cudaMemcpyAsync(&n, cnt, 4, cudaMemcpyDeviceToHost, c->L.stream));
    CU(c, cudaStreamSynchronize(c->L.stream));
    const u64 got = std::min<u64>(n, ecap);
    if (got) {
        CU(c, cudaMemcpy(out, buf, got * sizeof(bng_acct), cudaMemcpyDeviceToHost));
        CU(c, cudaMemcpy(addrs_out, buf + aoff, got * 4, cudaMemcpyDeviceToHost));
    }
    return (int64_t)got;
}

int bng_acct_enable(bng_ctx *c, int prog, int on) {
    if (!c || prog < 0 || prog >= P_COUNT) return -EINVAL;
    if (k_acct_mode[prog] < 0) return -EOPNOTSUPP;
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    if (on) {
        if (int r = acct_alloc_locked(c)) return r;
        c->acct_progs |= 1u << prog;
    } else {
        c->acct_progs &= ~(1u << prog);
    }
    return 0;
}

int bng_acct_read(bng_ctx *c, const uint32_t *addrs, uint64_t n, bng_acct *out, int32_t *results) {
    if (!c || (n && (!addrs || !out || !results))) return -EINVAL;
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    if (int fr = acct_flush_locked(c)) return fr;
    const u64 chunk_max = 1u << 16;
    for (u64 done = 0; done < n; done += chunk_max) {
        const u64 k = std::min(chunk_max, n - done);
        const size_t ooff = (k * 4 + 255) & ~(size_t)255, roff = ooff + k * sizeof(bng_acct);
        if (int r = ensure_io(c, roff + k * 4)) return r;
        memcpy(c->io_host, addrs + done, k * 4);
        CU(c, cudaMemcpyAsync(c->io_dev, c->io_host, k * 4, cudaMemcpyHostToDevice, c->L.stream));
        CU(c, run_acct_read(c->L, c->dev.subdir, c->acct, (const u32 *)c->io_dev.get(), k, (u64 *)(c->io_dev + ooff), (int *)(c->io_dev + roff)));
        CU(c, cudaMemcpyAsync(c->io_host + ooff, c->io_dev + ooff, roff + k * 4 - ooff, cudaMemcpyDeviceToHost, c->L.stream));
        CU(c, cudaStreamSynchronize(c->L.stream));
        memcpy(out + done, c->io_host + ooff, k * sizeof(bng_acct));
        memcpy(results + done, c->io_host + roff, k * 4);
    }
    return 0;
}

int64_t bng_acct_dump(bng_ctx *c, uint32_t *addrs_out, bng_acct *out, uint64_t cap) {
    if (!c || (cap && (!addrs_out || !out))) return -EINVAL;
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    if (int fr = acct_flush_locked(c)) return fr;
    return acct_dump_locked(c, addrs_out, out, cap);
}

// ---------------------------------------------------------------------------
// per-subscriber idle detection (idle.cu; stamped by k_acct)
// ---------------------------------------------------------------------------
static_assert(sizeof(bng_idle) == IDLE_WORDS * 8, "struct bng_idle has the size of the device record");

// The records (one per directory slot, every field none) and the per-frame attribution words, on first use.
static int idle_alloc_locked(bng_ctx *c) {
    if (c->idle) return 0;
    // a failure releases the whole batch scratch (all or none): the next batch grows it again for its own size
    if (int r = scratch_locked(c, c->L.s.cap, true, c->li_ctl)) return r;
    const size_t bytes = ((size_t)c->dev.subdir.mask + 1) * sizeof(bng_idle);
    if (!c->idle.grow(bytes)) return grow_failed(c, "idle detection", bytes);
    CU(c, cudaMemsetAsync(c->idle, 0, bytes, c->L.stream));
    return 0;
}

// stamps and since of every record := none (restore, delta apply)
static int idle_restart_locked(bng_ctx *c) {
    if (c->idle) CU(c, run_idle_restart(c->L, c->dev.subdir, c->idle));
    return 0;
}

// timeouts of n addresses from host memory, chunked through the staging buffers; results may be nullptr
static int idle_timeouts_locked(bng_ctx *c, const uint32_t *addrs, const uint32_t *timeouts, uint64_t n, int32_t *results) {
    if (int r = idle_alloc_locked(c)) return r;
    const u64 chunk_max = 1u << 18;
    for (u64 done = 0; done < n; done += chunk_max) {
        const u64 k = std::min(chunk_max, n - done);
        const size_t toff = (k * 4 + 255) & ~(size_t)255, roff = toff * 2;
        if (int r = ensure_io(c, roff + k * 4)) return r;
        memcpy(c->io_host, addrs + done, k * 4);
        memcpy(c->io_host + toff, timeouts + done, k * 4);
        CU(c, cudaMemcpyAsync(c->io_dev, c->io_host, toff + k * 4, cudaMemcpyHostToDevice, c->L.stream));
        CU(c, run_idle_timeout_set(c->L, c->dev.subdir, c->idle, (const u32 *)c->io_dev.get(), (const u32 *)(c->io_dev + toff), k,
                                   (int *)(c->io_dev + roff)));
        if (results) CU(c, cudaMemcpyAsync(c->io_host + roff, c->io_dev + roff, k * 4, cudaMemcpyDeviceToHost, c->L.stream));
        CU(c, cudaStreamSynchronize(c->L.stream));
        if (results) memcpy(results + done, c->io_host + roff, k * 4);
    }
    return 0;
}

// records of n addresses from host memory, chunked through the staging buffers
static int idle_read_locked(bng_ctx *c, const uint32_t *addrs, uint64_t n, bng_idle *out, int32_t *results) {
    const u64 chunk_max = 1u << 16;
    for (u64 done = 0; done < n; done += chunk_max) {
        const u64 k = std::min(chunk_max, n - done);
        const size_t ooff = (k * 4 + 255) & ~(size_t)255, roff = ooff + k * sizeof(bng_idle);
        if (int r = ensure_io(c, roff + k * 4)) return r;
        memcpy(c->io_host, addrs + done, k * 4);
        CU(c, cudaMemcpyAsync(c->io_dev, c->io_host, k * 4, cudaMemcpyHostToDevice, c->L.stream));
        CU(c, run_idle_read(c->L, c->dev.subdir, c->idle, (const u32 *)c->io_dev.get(), k, (u64 *)(c->io_dev + ooff), (int *)(c->io_dev + roff)));
        CU(c, cudaMemcpyAsync(c->io_host + ooff, c->io_dev + ooff, roff + k * 4 - ooff, cudaMemcpyDeviceToHost, c->L.stream));
        CU(c, cudaStreamSynchronize(c->L.stream));
        memcpy(out + done, c->io_host + ooff, k * sizeof(bng_idle));
        memcpy(results + done, c->io_host + roff, k * 4);
    }
    return 0;
}

// (address, timeout) of every record, by address, for the snapshot: the directory's addresses (k_acct_dump lists them
// whether or not accounting records exist), then their records
static int idle_timeouts_dump_locked(bng_ctx *c, std::vector<u32> *addrs, std::vector<u32> *timeouts) {
    u32 n32 = 0;
    CU(c, cudaMemcpy(&n32, c->dev.subdir.count, 4, cudaMemcpyDeviceToHost));
    std::vector<u32> a(std::max<u32>(n32, 1));
    std::vector<bng_acct> unused(a.size());
    const int64_t got = acct_dump_locked(c, a.data(), unused.data(), a.size()); // the directory's addresses
    if (got < 0) return (int)got;
    a.resize((size_t)got);
    std::vector<bng_idle> recs(a.size());
    std::vector<int32_t> res(a.size());
    if (int r = idle_read_locked(c, a.data(), a.size(), recs.data(), res.data())) return r;
    addrs->clear();
    timeouts->clear();
    std::vector<size_t> order(a.size());
    for (size_t i = 0; i < order.size(); i++) order[i] = i;
    std::sort(order.begin(), order.end(), [&](size_t x, size_t y) { return a[x] < a[y]; });
    for (size_t i : order) addrs->push_back(a[i]), timeouts->push_back(recs[i].timeout_s);
    return 0;
}

int bng_idle_enable(bng_ctx *c, int prog, int on) {
    if (!c || prog < 0 || prog >= P_COUNT) return -EINVAL;
    if (k_acct_mode[prog] < 0) return -EOPNOTSUPP;
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    if (on) {
        if (int r = idle_alloc_locked(c)) return r;
        c->idle_progs |= 1u << prog;
    } else {
        c->idle_progs &= ~(1u << prog);
    }
    return 0;
}

int bng_idle_timeout_set(bng_ctx *c, const uint32_t *addrs, const uint32_t *timeouts_s, uint64_t n, int32_t *results) {
    if (!c || (n && (!addrs || !timeouts_s || !results))) return -EINVAL;
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    if (int fr = acct_flush_locked(c)) return fr;
    return idle_timeouts_locked(c, addrs, timeouts_s, n, results);
}

int bng_idle_read(bng_ctx *c, const uint32_t *addrs, uint64_t n, bng_idle *out, int32_t *results) {
    if (!c || (n && (!addrs || !out || !results))) return -EINVAL;
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    if (int fr = acct_flush_locked(c)) return fr;
    return idle_read_locked(c, addrs, n, out, results);
}

int64_t bng_idle_scan(bng_ctx *c, uint64_t now_ns, uint32_t default_s, uint32_t flags, uint32_t *addrs_out, bng_idle *out, uint64_t cap) {
    if (!c || !(flags & (BNG_IDLE_UP | BNG_IDLE_DOWN)) || (flags & ~(BNG_IDLE_UP | BNG_IDLE_DOWN)) || (cap && (!addrs_out || !out)))
        return -EINVAL;
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    if (int fr = acct_flush_locked(c)) return fr;
    if (!c->idle) return 0; // no record exists yet: nobody can be idle
    const u64 ecap = std::min<u64>(cap, (u64)c->dev.subdir.mask + 1); // no more entries than slots
    const size_t aoff = ecap * sizeof(bng_idle), coff = (aoff + ecap * 4 + 15) & ~(size_t)15, need = coff + 16;
    if (!c->idle_scan_buf.grow(need)) return grow_failed(c, "idle_scan", need);
    u8 *buf = c->idle_scan_buf;
    u32 *cnt = (u32 *)(buf + coff), n = 0;
    CU(c, cudaMemsetAsync(cnt, 0, 4, c->L.stream));
    CU(c, run_idle_scan(c->L, c->dev.subdir, c->idle, now_ns, default_s, flags, (u32 *)(buf + aoff), (u64 *)buf, cnt, ecap));
    CU(c, cudaMemcpyAsync(&n, cnt, 4, cudaMemcpyDeviceToHost, c->L.stream));
    CU(c, cudaStreamSynchronize(c->L.stream));
    const u64 got = std::min<u64>(n, ecap);
    if (got) {
        CU(c, cudaMemcpy(out, buf, got * sizeof(bng_idle), cudaMemcpyDeviceToHost));
        CU(c, cudaMemcpy(addrs_out, buf + aoff, got * 4, cudaMemcpyDeviceToHost));
    }
    return (int64_t)n;
}

// ---------------------------------------------------------------------------
// NAT port-usage census (natuse.cu)
// ---------------------------------------------------------------------------
static_assert(sizeof(bng_nat_sub_use) == 64 && sizeof(bng_nat_pub_use) == 64, "the census writes 16 u32 per record");
static_assert(sizeof(bng_nat_usage_sum) == (NU_PUBS_FOUND + 1) * 8, "struct bng_nat_usage_sum is the head of the census's sum words");

static u64 nu_pow2(u64 v) {
    u64 p = 64;
    while (p < v) p <<= 1;
    return p;
}

// the public-address table: pub_mask + 1 slots
static int nu_pub_alloc(bng_ctx *c, u64 slots) {
    if (slots > (1ull << 32)) return fail(c, -ENOMEM, "nat_usage: %llu public-address slots", (unsigned long long)slots);
    const size_t bytes = slots * NU_PUB_WORDS * 8; // the old table stays when the new one does not fit
    if (cudaError_t e = c->nu_pub.grow_keep(bytes, 0, c->L.stream)) return grow_failed(c, "nat_usage", bytes, "public-address table", e);
    c->nu_pub_mask = (u32)(slots - 1);
    return 0;
}

// The census's scratch, on first use (kernels.h: NatUse).  All of it or none.
static int nu_alloc_locked(bng_ctx *c) {
    if (c->nu_sum) return 0;
    const u64 keys = 4ull * ((u64)c->dev.sessions.max_entries + c->dev.eim.max_entries);
    const u64 set_slots = nu_pow2((keys * 4 + 2) / 3);
    const u64 dir_slots = (u64)c->dev.subdir.mask + 1;
    if (set_slots > (1ull << 30) || dir_slots > (1ull << 30))
        return fail(c, -ENOMEM, "nat_usage: %llu set slots / %llu directory slots exceed 2^30", (unsigned long long)set_slots,
                    (unsigned long long)dir_slots);
    if (!devbuf::grow_all({{&c->nu_set, set_slots * 8}, {&c->nu_sub, dir_slots * NU_SUB_WORDS * 4}, {&c->nu_sum, NU_SUM_WORDS * 8}}))
        return grow_failed(c, "nat_usage", set_slots * 8 + dir_slots * NU_SUB_WORDS * 4 + NU_SUM_WORDS * 8, "census");
    if (int r = nu_pub_alloc(c, 1u << 16)) {
        c->nu_set.reset(), c->nu_sub.reset(), c->nu_sum.reset();
        return r;
    }
    c->nu_set_mask = (u32)(set_slots - 1);
    return 0;
}

int bng_nat_usage(bng_ctx *c, uint32_t min_permille, bng_nat_usage_sum *sum, uint32_t *sub_addrs, bng_nat_sub_use *sub_out,
                  uint64_t sub_cap, uint32_t *pub_addrs, bng_nat_pub_use *pub_out, uint64_t pub_cap) {
    if (!c || !sum || min_permille > 1000 || (sub_cap && (!sub_addrs || !sub_out)) || (pub_cap && (!pub_addrs || !pub_out)))
        return -EINVAL;
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    int r = flush_staged_locked(c, -1);
    if (r) return r;
    if ((r = nu_alloc_locked(c)) != 0) return r;
    const u64 scap = std::min<u64>(sub_cap, (u64)c->dev.subdir.mask + 1); // no more records than directory slots
    u64 sum_w[NU_SUM_WORDS];
    for (;;) {
        const u64 pcap = std::min<u64>(pub_cap, (u64)c->nu_pub_mask + 1);
        const u64 rec_b = (scap + pcap) * 64, need = rec_b + (scap + pcap) * 4;
        if (!c->nu_out.grow(need)) return grow_failed(c, "nat_usage", need, "records");
        NatUse u{};
        u.set = c->nu_set, u.set_mask = c->nu_set_mask, u.sub = c->nu_sub, u.pub = c->nu_pub, u.pub_mask = c->nu_pub_mask;
        u.sum = c->nu_sum;
        u.sub_out = (u32 *)c->nu_out.get(), u.pub_out = (u32 *)(c->nu_out + scap * 64);
        u.sub_addrs = (u32 *)(c->nu_out + rec_b), u.pub_addrs = u.sub_addrs + scap;
        u.sub_cap = scap, u.pub_cap = pcap;
        const u64 dir_slots = (u64)c->dev.subdir.mask + 1;
        CU(c, cudaMemsetAsync(c->nu_set, 0, ((u64)c->nu_set_mask + 1) * 8, c->L.stream));
        CU(c, cudaMemsetAsync(c->nu_sub, 0, dir_slots * NU_SUB_WORDS * 4, c->L.stream));
        CU(c, cudaMemsetAsync(c->nu_pub, 0, ((u64)c->nu_pub_mask + 1) * NU_PUB_WORDS * 8, c->L.stream));
        CU(c, cudaMemsetAsync(c->nu_sum, 0, NU_SUM_WORDS * 8, c->L.stream));
        CU(c, run_nat_usage_flows(c->L, c->dev, u));
        CU(c, cudaMemcpyAsync(sum_w, c->nu_sum, sizeof(sum_w), cudaMemcpyDeviceToHost, c->L.stream));
        CU(c, cudaStreamSynchronize(c->L.stream));
        if (sum_w[NU_SET_FULL]) return fail(c, -EIO, "nat_usage: the triple set is full");
        if (sum_w[NU_OVERFLOW]) { // more public addresses than half the table: grow it past the reservations and count again
            prof_collect(c->L);
            if ((r = nu_pub_alloc(c, nu_pow2(2 * sum_w[NU_PUB_RESERVED]))) != 0) return r;
            continue;
        }
        CU(c, run_nat_usage_emit(c->L, c->dev, u, min_permille));
        CU(c, cudaMemcpyAsync(sum_w, c->nu_sum, sizeof(sum_w), cudaMemcpyDeviceToHost, c->L.stream));
        CU(c, cudaStreamSynchronize(c->L.stream));
        prof_collect(c->L);
        const u64 ns = std::min<u64>(sum_w[NU_SUBS_FOUND], scap), np = std::min<u64>(sum_w[NU_PUBS_FOUND], pcap);
        if (ns) {
            CU(c, cudaMemcpy(sub_out, u.sub_out, ns * 64, cudaMemcpyDeviceToHost));
            CU(c, cudaMemcpy(sub_addrs, u.sub_addrs, ns * 4, cudaMemcpyDeviceToHost));
        }
        if (np) {
            CU(c, cudaMemcpy(pub_out, u.pub_out, np * 64, cudaMemcpyDeviceToHost));
            CU(c, cudaMemcpy(pub_addrs, u.pub_addrs, np * 4, cudaMemcpyDeviceToHost));
        }
        break;
    }
    memcpy(sum, sum_w, sizeof(*sum));
    return 0;
}

// ---------------------------------------------------------------------------
// DHCP lease census and expiry sweep (leases.cu)
// ---------------------------------------------------------------------------
static_assert(sizeof(bng_lease_pool_use) == 64 && sizeof(bng_lease_removed) == 64, "the lease kernels write 16 u32 per record");
static_assert(sizeof(bng_lease_sum) == (LS_POOLS_FOUND + 1) * 8, "struct bng_lease_sum is the head of the census's sum words");

// the output records of either call (and the census's pool ids behind them): grow-only
static int ls_out_locked(bng_ctx *c, u64 bytes) {
    return c->ls_out.grow(bytes) ? 0 : grow_failed(c, "dhcp leases", bytes, "records");
}

// leases.cu reads the lease slots by fixed offsets
static int ls_layout_locked(bng_ctx *c) {
    const DevCtx &d = c->dev;
    if (d.sub_pools.slot_bytes != 64 || d.vlan_pools.slot_bytes != 64 || d.cid_subs.slot_bytes != 64 || d.sub_pools.voff != 8 ||
        d.vlan_pools.voff != 8 || d.cid_subs.voff != 32)
        return fail(c, -EINVAL, "dhcp leases: unexpected slot layout of the lease maps");
    return 0;
}

// pool records: one per ip_pools slot, then the hash of unknown pool_ids (unk_slots of them)
static int ls_pools_alloc(bng_ctx *c, u64 unk_slots) {
    const u64 n = (u64)c->dev.ip_pools.mask + 1 + unk_slots;
    if (n > (1ull << 26)) return fail(c, -ENOMEM, "lease_census: %llu pool records", (unsigned long long)n);
    const size_t bytes = n * LS_POOL_WORDS * 8; // the old records stay when the new ones do not fit
    if (cudaError_t e = c->ls_pools.grow_keep(bytes, 0, c->L.stream)) return grow_failed(c, "dhcp leases", bytes, "pool records", e);
    c->ls_unk_mask = (u32)(unk_slots - 1);
    return 0;
}

// The census's scratch, on first use (kernels.h: LeaseUse).  All of it or none.
static int ls_alloc_locked(bng_ctx *c) {
    if (c->ls_sum) return 0;
    const u64 keys = 3ull * ((u64)c->dev.sub_pools.max_entries + c->dev.vlan_pools.max_entries + c->dev.cid_subs.max_entries);
    const u64 set_slots = nu_pow2((keys * 4 + 2) / 3);
    if (set_slots > (1ull << 32)) return fail(c, -ENOMEM, "lease_census: %llu set slots", (unsigned long long)set_slots);
    if (!devbuf::grow_all({{&c->ls_set, set_slots * 8}, {&c->ls_sum, LS_SUM_WORDS * 8}}))
        return grow_failed(c, "dhcp leases", set_slots * 8 + LS_SUM_WORDS * 8, "census");
    if (int r = ls_pools_alloc(c, 1u << 14)) {
        c->ls_set.reset(), c->ls_sum.reset();
        return r;
    }
    c->ls_set_mask = (u32)(set_slots - 1);
    return 0;
}

int bng_dhcp_lease_census(bng_ctx *c, uint64_t now_ns, bng_lease_sum *sum, uint32_t *pool_ids, bng_lease_pool_use *out, uint64_t cap) {
    if (!c || !sum || (cap && (!pool_ids || !out))) return -EINVAL;
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    int r = flush_staged_locked(c, -1);
    if (r) return r;
    if ((r = ls_layout_locked(c)) != 0 || (r = ls_alloc_locked(c)) != 0) return r;
    u64 sum_w[LS_SUM_WORDS];
    for (;;) {
        LeaseUse u{};
        u.set = c->ls_set, u.set_mask = c->ls_set_mask, u.unk_mask = c->ls_unk_mask, u.n_known = c->dev.ip_pools.mask + 1;
        u.pools = c->ls_pools, u.sum = c->ls_sum, u.wire = c->ls_wire;
        const u64 recs = (u64)u.n_known + u.unk_mask + 1;
        u.cap = std::min<u64>(cap, recs); // no more records than record slots
        if ((r = ls_out_locked(c, u.cap * 68)) != 0) return r;
        u.out = (u32 *)c->ls_out.get(), u.ids_out = (u32 *)(c->ls_out + u.cap * 64);
        CU(c, cudaMemsetAsync(c->ls_set, 0, ((u64)c->ls_set_mask + 1) * 8, c->L.stream));
        CU(c, cudaMemsetAsync(c->ls_pools, 0, recs * LS_POOL_WORDS * 8, c->L.stream));
        CU(c, cudaMemsetAsync(c->ls_sum, 0, LS_SUM_WORDS * 8, c->L.stream));
        CU(c, run_lease_census(c->L, c->dev, u, now_ns / 1000000000ull));
        CU(c, cudaMemcpyAsync(sum_w, c->ls_sum, sizeof(sum_w), cudaMemcpyDeviceToHost, c->L.stream));
        CU(c, cudaStreamSynchronize(c->L.stream));
        if (sum_w[LS_SET_FULL]) return fail(c, -EIO, "lease_census: the address set is full");
        if (sum_w[LS_OVERFLOW]) { // more unknown pool_ids than half the hash: grow it past the claims and count again
            prof_collect(c->L);
            if ((r = ls_pools_alloc(c, nu_pow2(4 * sum_w[LS_UNK_CLAIMED]))) != 0) return r;
            continue;
        }
        CU(c, run_lease_pools(c->L, c->dev, u));
        CU(c, cudaMemcpyAsync(sum_w, c->ls_sum, sizeof(sum_w), cudaMemcpyDeviceToHost, c->L.stream));
        CU(c, cudaStreamSynchronize(c->L.stream));
        prof_collect(c->L);
        if (const u64 n = std::min<u64>(sum_w[LS_POOLS_FOUND], u.cap)) {
            CU(c, cudaMemcpy(out, u.out, n * 64, cudaMemcpyDeviceToHost));
            CU(c, cudaMemcpy(pool_ids, u.ids_out, n * 4, cudaMemcpyDeviceToHost));
        }
        break;
    }
    memcpy(sum, sum_w, sizeof(*sum));
    return 0;
}

int64_t bng_dhcp_lease_sweep(bng_ctx *c, uint64_t now_ns, uint32_t grace_s, bng_lease_removed *out, uint64_t cap, uint64_t removed_out[4]) {
    if (!c || (cap && !out)) return -EINVAL;
    if (removed_out) removed_out[0] = removed_out[1] = removed_out[2] = removed_out[3] = 0;
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    int r = flow_pass_begin_locked(c);
    if (r) return r;
    if ((r = ls_layout_locked(c)) != 0) return r;
    DevCtx &d = c->dev;
    // no more entries can be due than the three maps hold
    const u64 ecap = std::min<u64>(cap, (u64)d.sub_pools.max_entries + d.vlan_pools.max_entries + d.cid_subs.max_entries);
    const u64 mac_slots = nu_pow2(2 * std::min<u64>(ecap, d.sub_pools.max_entries));
    if (mac_slots > (1ull << 32)) return fail(c, -ENOMEM, "lease_sweep: %llu MAC set slots", (unsigned long long)mac_slots);
    if ((r = ls_out_locked(c, ecap * 64)) != 0) return r;
    if (!c->ls_macs.grow((LS_W_WORDS + mac_slots) * 8)) return grow_failed(c, "dhcp leases", (LS_W_WORDS + mac_slots) * 8, "MAC set");
    LeaseSweep w{};
    w.now_s = now_ns / 1000000000ull, w.grace_s = grace_s, w.cap = ecap;
    w.out = (u32 *)c->ls_out.get(), w.cnt = c->ls_macs, w.macs = c->ls_macs + LS_W_WORDS, w.mac_mask = (u32)(mac_slots - 1);
    CU(c, cudaMemsetAsync(c->ls_macs, 0, (LS_W_WORDS + mac_slots) * 8, c->L.stream));
    CU(c, run_lease_sweep(c->L, d, w));
    u64 cnt[LS_W_WORDS];
    CU(c, cudaMemcpyAsync(cnt, w.cnt, sizeof(cnt), cudaMemcpyDeviceToHost, c->L.stream));
    CU(c, cudaStreamSynchronize(c->L.stream));
    prof_collect(c->L);
    if (cnt[LS_W_SET_FULL]) return fail(c, -EIO, "lease_sweep: the MAC set is full");
    if (cnt[LS_W_LOST]) return fail(c, -EIO, "lease_sweep: a due entry changed under the sweep");
    if (const u64 n = std::min<u64>(cnt[LS_W_FOUND], ecap)) CU(c, cudaMemcpy(out, w.out, n * 64, cudaMemcpyDeviceToHost));
    if (removed_out) memcpy(removed_out, cnt + LS_W_REMOVED, 4 * 8);
    // A mass expiry tombstones most of a table, and the fast path's probes walk the tombstones.  A dry run changes
    // nothing, so it rebuilds nothing.  The removals stand and are reported even when a rebuild finds no memory: the
    // table it could not rebuild stays as it was and the next sweep tries again (bng_last_error has the text).
    Tbl *tb[4] = {&d.sub_pools, &d.vlan_pools, &d.cid_subs, &d.cid_map};
    for (int k = 0; k < 4 && ecap; k++)
        if (cnt[LS_W_TOMBS + k] > ((u64)tb[k]->mask + 1) / 4 && table_rebuild_locked(c, tb[k], false) != 0) break;
    return (int64_t)cnt[LS_W_FOUND];
}

int bng_dhcp_lease_addr_order(bng_ctx *c, uint32_t order) {
    if (!c || order > BNG_LEASE_ADDR_WIRE) return -EINVAL;
    std::lock_guard<std::mutex> g(c->mu);
    c->ls_wire = order;
    return 0;
}

uint64_t bng_lease_table_rebuilds(bng_ctx *c) { return c ? c->lease_rebuilds : 0; }

// ---------------------------------------------------------------------------
// lawful intercept (li.cu)
// ---------------------------------------------------------------------------
static_assert(sizeof(bng_li_record) == LI_HDR, "struct bng_li_record is the device record's header");
#define LI_TSLOTS (2 * BNG_LI_MAX_TARGETS) // the target set at its fullest: load 1/2

// A ring of cap records of 64 + snaplen (rounded up to 16) bytes.  The previous ring, if any, is discarded only once
// the new one exists; its records (drained or not) are counted as lost.
static int li_collect_locked(bng_ctx *c);
static int li_ring_locked(bng_ctx *c, u32 snaplen, u32 cap) {
    const u32 rec = LI_HDR + ((snaplen + 15u) & ~15u);
    DevBuf<u8> ring;
    if (!ring.grow((size_t)cap * rec)) return grow_failed(c, "li_configure", (size_t)cap * rec);
    if (c->li_ring) {
        if (int r = li_collect_locked(c)) return r;
        c->li_lost_host += c->li_pending.size() / c->li_rec;
        c->li_pending.clear();
    }
    c->li_ring = std::move(ring), c->li_cap = cap, c->li_rec = rec, c->li_snap = snaplen;
    CU(c, cudaMemsetAsync(c->li_ctl, 0, 8, c->L.stream)); // no slot handed out
    return 0;
}

// Everything interception needs, on first use: control words, target set, match list, attribution words; the ring
// with the given size unless one exists.
static int li_alloc_locked(bng_ctx *c, u32 snaplen = 1518, u32 cap = 1u << 15) {
    if (!c->li_ctl) {
        // a failure releases the whole batch scratch (all or none): the next batch grows it again for its own size
        if (int r = scratch_locked(c, c->L.s.cap, true, true)) return r;
        if (int r = dev_alloc(c, (void **)&c->li_words, LI_TSLOTS * 8, 0)) return r;
        if (int r = dev_alloc(c, (void **)&c->li_ids, LI_TSLOTS * 4, 0)) return r;
        u64 *ctl = nullptr;
        if (int r = dev_alloc(c, (void **)&ctl, 32, 0)) return r;
        c->li_ctl = ctl;
    }
    return c->li_ring ? 0 : li_ring_locked(c, snaplen, cap);
}

// The device copy of the targets (bng_prog_run, when they changed): an AddrSet of a power of two >= 2n slots.
static int li_upload_locked(bng_ctx *c) {
    u32 slots = 64;
    while (slots < 2 * c->li_targets.size()) slots *= 2;
    std::vector<u64> words(slots, 0);
    std::vector<u32> ids(slots, 0);
    const u32 mask = slots - 1;
    for (const auto &t : c->li_targets) {
        u32 i = aset_home(t.first, mask);
        while (words[i]) i = (i + 1) & mask;
        words[i] = ADDRSET_LIVE | t.first;
        ids[i] = t.second;
    }
    // pageable sources: the copies are staged before the calls return, so the vectors may go
    CU(c, cudaMemcpyAsync(c->li_words, words.data(), (size_t)slots * 8, cudaMemcpyHostToDevice, c->L.stream));
    CU(c, cudaMemcpyAsync(c->li_ids, ids.data(), (size_t)slots * 4, cudaMemcpyHostToDevice, c->L.stream));
    c->li_mask = mask;
    c->li_dirty = false;
    return 0;
}

// Moves the ring's records to li_pending, ordered by (batch, frame), void ones left out; the ring is empty after.
static int li_collect_locked(bng_ctx *c) {
    u64 cnt = 0;
    CU(c, cudaMemcpyAsync(&cnt, c->li_ctl, 8, cudaMemcpyDeviceToHost, c->L.stream));
    CU(c, cudaStreamSynchronize(c->L.stream));
    cnt = std::min<u64>(cnt, c->li_cap);
    if (!cnt) return 0;
    const size_t rb = c->li_rec;
    std::vector<u8> raw(cnt * rb);
    CU(c, cudaMemcpyAsync(raw.data(), c->li_ring, raw.size(), cudaMemcpyDeviceToHost, c->L.stream));
    CU(c, cudaMemsetAsync(c->li_ctl, 0, 8, c->L.stream));
    CU(c, cudaStreamSynchronize(c->L.stream));
    std::vector<u32> order;
    order.reserve(cnt);
    for (u32 i = 0; i < cnt; i++)
        if (((const bng_li_record *)(raw.data() + i * rb))->verdict != LI_VOID) order.push_back(i);
    auto at = [&](u32 i) { return (const bng_li_record *)(raw.data() + i * rb); };
    std::sort(order.begin(), order.end(), [&](u32 a, u32 b) {
        return at(a)->batch != at(b)->batch ? at(a)->batch < at(b)->batch : at(a)->frame < at(b)->frame;
    });
    const size_t have = c->li_pending.size();
    c->li_pending.resize(have + order.size() * rb);
    for (size_t k = 0; k < order.size(); k++) memcpy(&c->li_pending[have + k * rb], at(order[k]), rb);
    return 0;
}

int bng_li_configure(bng_ctx *c, uint32_t snaplen, uint32_t capacity) {
    if (!c || snaplen > 65535 || capacity > (1u << 30)) return -EINVAL;
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    snaplen = snaplen ? snaplen : 1518;
    capacity = capacity ? capacity : (1u << 15);
    if (!c->li_ring) return li_alloc_locked(c, snaplen, capacity);
    return li_ring_locked(c, snaplen, capacity);
}

uint32_t bng_li_record_size(bng_ctx *c) {
    if (!c) return 0;
    std::lock_guard<std::mutex> g(c->mu);
    return c->li_ring ? c->li_rec : 0;
}

int bng_li_target_set(bng_ctx *c, uint32_t addr, uint32_t target_id) {
    if (!c) return -EINVAL;
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    if (int r = li_alloc_locked(c)) return r;
    if (c->li_targets.size() >= BNG_LI_MAX_TARGETS && !c->li_targets.count(addr)) return -E2BIG;
    c->li_targets[addr] = target_id;
    c->li_dirty = true;
    return 0;
}

int bng_li_target_del(bng_ctx *c, uint32_t addr) {
    if (!c) return -EINVAL;
    std::lock_guard<std::mutex> g(c->mu);
    if (!c->li_targets.erase(addr)) return -ENOENT;
    c->li_dirty = true;
    return 0;
}

int bng_li_drain(bng_ctx *c, void *buf, uint64_t cap_records, uint64_t *n_out) {
    if (!c || !n_out || (cap_records && !buf)) return -EINVAL;
    *n_out = 0;
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    if (!c->li_ring) return 0;
    if (int r = li_collect_locked(c)) return r;
    const u64 n = std::min<u64>(c->li_pending.size() / c->li_rec, cap_records);
    if (n) {
        memcpy(buf, c->li_pending.data(), n * c->li_rec);
        c->li_pending.erase(c->li_pending.begin(), c->li_pending.begin() + n * c->li_rec);
    }
    *n_out = n;
    return 0;
}

uint64_t bng_li_lost(bng_ctx *c) {
    if (!c) return 0;
    std::lock_guard<std::mutex> g(c->mu);
    if (!c->li_ctl) return 0;
    cudaSetDevice(c->device);
    u64 v = 0;
    if (cudaMemcpyAsync(&v, c->li_ctl + 1, 8, cudaMemcpyDeviceToHost, c->L.stream) != cudaSuccess) return 0;
    cudaStreamSynchronize(c->L.stream);
    return v + c->li_lost_host;
}

// ---------------------------------------------------------------------------
// state blobs: snapshot / restore, incremental replication, subscriber hand-over.  All three share the section
// framing of blob.hpp; each entry point keeps its own policy for the sections it reads.
// ---------------------------------------------------------------------------
namespace {
using blob::kAcct, blob::kLi, blob::kIdle;

// what the grow-only staging of an export allocates when it needs `bytes`: half as much again, at least 1 MiB
u64 with_slack(u64 bytes) { return std::max<u64>(bytes + bytes / 2, 1 << 20); }

// a non-event map, whole, as one section
int map_section_locked(bng_ctx *c, MapReg *m, blob::Writer &w) {
    u64 cnt = m->max_entries;
    if (m->kind == KIND_HASH) {
        u32 n32 = 0;
        CU(c, cudaMemcpy(&n32, m->tbl->count, 4, cudaMemcpyDeviceToHost));
        cnt = n32;
    } else if (m->kind == KIND_LPM) {
        cnt = m->lpm_host.size() / 3;
    } else if (m->kind == KIND_STATS) {
        cnt = 1;
    }
    std::vector<u8> keys((size_t)std::max<u64>(cnt, 1) * m->key_size), vals((size_t)std::max<u64>(cnt, 1) * m->value_size);
    const int64_t got = cnt ? map_dump_locked(c, m, keys.data(), vals.data(), cnt) : 0;
    if (got < 0) return (int)got;
    w.section(m->name, (u32)m->kind, m->key_size, m->value_size, (u64)got, keys.data(), vals.data());
    return 0;
}

// the interception targets, by address
std::vector<std::pair<u32, u32>> li_sorted(const bng_ctx *c) {
    std::vector<std::pair<u32, u32>> t(c->li_targets.begin(), c->li_targets.end());
    std::sort(t.begin(), t.end());
    return t;
}

void li_section(blob::Writer &w, const std::vector<std::pair<u32, u32>> &t) {
    std::vector<u32> a, id;
    for (const auto &e : t) a.push_back(e.first), id.push_back(e.second);
    w.pairs(kLi, blob::kLiKind, a, id);
}

// a map emptied ahead of loading a blob's section into it
int map_clear_for_load(bng_ctx *c, int id) {
    MapReg *m = get_map(c, id);
    if (m->kind == KIND_HASH) return bng_map_clear(c, id);
    if (m->kind != KIND_LPM) return 0;
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    m->lpm_host.clear();
    return lpm_upload(c, m);
}

// every accounting record and idle record at zero, no interception target: what a full load starts from
int records_reset_locked(bng_ctx *c) {
    if (c->acct) CU(c, cudaMemsetAsync(c->acct, 0, ((size_t)c->dev.subdir.mask + 1) * sizeof(bng_acct), c->L.stream));
    if (c->idle) CU(c, cudaMemsetAsync(c->idle, 0, ((size_t)c->dev.subdir.mask + 1) * sizeof(bng_idle), c->L.stream));
    CU(c, cudaStreamSynchronize(c->L.stream));
    if (!c->li_targets.empty()) c->li_targets.clear(), c->li_dirty = true;
    return 0;
}

size_t al256(size_t v) { return (v + 255) & ~(size_t)255; }

// n (address, record) pairs into the addresses' directory slots, chunked through the staging buffers: accounting
// records (rs = sizeof(bng_acct)) or whole idle records (rs = sizeof(bng_idle))
int load_records_locked(bng_ctx *c, const u8 *addrs, const u8 *recs, u64 n, size_t rs) {
    const bool acct = rs == sizeof(bng_acct);
    if (int r = acct ? acct_alloc_locked(c) : idle_alloc_locked(c)) return r;
    const u64 chunk_max = 1u << 16;
    for (u64 done = 0; done < n; done += chunk_max) {
        const u64 k = std::min(chunk_max, n - done);
        const size_t roff = al256(k * 4);
        if (int r = ensure_io(c, roff + k * rs)) return r;
        memcpy(c->io_host, addrs + done * 4, k * 4);
        memcpy(c->io_host + roff, recs + done * rs, k * rs);
        CU(c, cudaMemcpyAsync(c->io_dev, c->io_host, roff + k * rs, cudaMemcpyHostToDevice, c->L.stream));
        if (acct)
            CU(c, run_acct_load(c->L, c->dev.subdir, c->acct, (const u32 *)c->io_dev.get(), (const u64 *)(c->io_dev + roff), k));
        else
            CU(c, run_idle_load(c->L, c->dev.subdir, c->idle, (const u32 *)c->io_dev.get(), (const u64 *)(c->io_dev + roff), k));
        CU(c, cudaStreamSynchronize(c->L.stream));
    }
    return 0;
}

// n (address, target id) pairs into the interception targets; replace: they are the only targets afterwards
int li_targets_load_locked(bng_ctx *c, const u8 *addrs, const u8 *ids, u64 n, bool replace) {
    if (int r = li_alloc_locked(c)) return r;
    if (replace) c->li_targets.clear();
    for (u64 k = 0; k < n; k++) {
        u32 a, id;
        memcpy(&a, addrs + k * 4, 4);
        memcpy(&id, ids + k * 4, 4);
        c->li_targets[a] = id;
    }
    c->li_dirty = true;
    return 0;
}
} // namespace

// ---------------------------------------------------------------------------
// snapshot / restore (SURVEY.md §8f-4: device-table state for HA hand-over, reference pkg/ha)
// A snapshot is a self-describing blob: header, then one section per hash / array / LPM / statistics map (event rings
// are not state), then the records.  Restore clears each map it finds in the blob and loads the entries through the
// ordinary update path, so derived state (subscriber directory, the shared-memory image of the small maps) is rebuilt
// on the way and a snapshot taken with one set of table capacities restores into another.
// ---------------------------------------------------------------------------
int64_t bng_snapshot(bng_ctx *c, void *buf, uint64_t cap) {
    if (!c) return -EINVAL;
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    if (int fr = flush_staged_locked(c, -1)) return fr;
    CU(c, cudaStreamSynchronize(c->L.stream));
    blob::Writer w(16);
    for (auto &m : c->maps) {
        if (m.kind == KIND_EVENT) continue;
        if (int r = map_section_locked(c, &m, w)) return r;
    }
    if (c->acct) {
        u32 n32 = 0;
        CU(c, cudaMemcpy(&n32, c->dev.subdir.count, 4, cudaMemcpyDeviceToHost));
        const u64 cnt = std::max<u32>(n32, 1);
        std::vector<u32> addrs(cnt);
        std::vector<bng_acct> recs(cnt);
        int64_t got = acct_dump_locked(c, addrs.data(), recs.data(), cnt);
        if (got < 0) return got;
        w.section(kAcct, blob::kAcctKind, 4, sizeof(bng_acct), (u64)got, addrs.data(), recs.data());
    }
    if (c->li_ctl) li_section(w, li_sorted(c));
    if (c->idle) {
        std::vector<u32> a, t;
        if (int r = idle_timeouts_dump_locked(c, &a, &t)) return r;
        w.pairs(kIdle, blob::kIdleKind, a, t);
    }
    memcpy(w.out.data(), blob::kSnapMagic, 8);
    memcpy(w.out.data() + 8, &w.sections, 8);
    if (buf && cap >= w.out.size()) memcpy(buf, w.out.data(), w.out.size());
    return (int64_t)w.out.size(); // the size needed; nothing was copied when cap is smaller
}

int bng_restore(bng_ctx *c, const void *buf, uint64_t len) {
    if (!c || !buf || len < 16 || memcmp(buf, blob::kSnapMagic, 8)) return -EINVAL;
    u64 n;
    memcpy(&n, (const u8 *)buf + 8, 8);
    std::vector<blob::Section> secs;
    std::string err;
    if (!blob::read_sections((const u8 *)buf + 16, (const u8 *)buf + len, n, false, false, secs, err))
        return fail(c, -EINVAL, "snapshot: %s", err.c_str());
    // the whole blob is checked before anything changes: maps this library does not have are skipped, the records
    // are taken once the maps (and so the directory) are in place
    std::vector<std::pair<int, const blob::Section *>> maps;
    const blob::Section *acct = nullptr, *li = nullptr, *idle = nullptr;
    for (const blob::Section &s : secs) {
        const blob::SectionHdr &h = s.h;
        bool ok = h.key_size == 4;
        if (!strcmp(h.name, kAcct)) {
            ok = ok && h.value_size == sizeof(bng_acct), acct = &s;
        } else if (!strcmp(h.name, kLi)) {
            ok = ok && h.value_size == 4 && h.count <= BNG_LI_MAX_TARGETS, li = &s;
        } else if (!strcmp(h.name, kIdle)) {
            ok = ok && h.value_size == 4, idle = &s;
        } else {
            const int id = bng_map_id(c, h.name);
            if (id < 0) continue;
            const MapReg *m = get_map(c, id);
            ok = m->key_size == h.key_size && m->value_size == h.value_size;
            maps.emplace_back(id, &s);
        }
        if (!ok) return fail(c, -EINVAL, "snapshot: %s has another layout", h.name);
    }
    { // the blob's records replace these; a blob without them leaves every record at zero and every clock restarts
        std::lock_guard<std::mutex> g(c->mu);
        cudaSetDevice(c->device);
        if (int r = records_reset_locked(c)) return r;
    }
    for (const auto &[id, s] : maps) {
        if (int r = map_clear_for_load(c, id)) return r;
        if (s->h.count) {
            if (int r = bng_map_update_batch(c, id, s->keys, s->vals, s->h.count, BNG_ANY))
                return fail(c, r, "snapshot: loading %s failed", s->h.name);
        }
    }
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    if (acct && acct->h.count) {
        if (int r = load_records_locked(c, acct->keys, acct->vals, acct->h.count, sizeof(bng_acct))) return r;
    }
    if (li && li->h.count) {
        if (int r = li_targets_load_locked(c, li->keys, li->vals, li->h.count, true)) return r;
    }
    if (idle) {
        const u64 k = idle->h.count;
        std::vector<u32> a(k), t(k);
        if (k) memcpy(a.data(), idle->keys, k * 4), memcpy(t.data(), idle->vals, k * 4);
        if (int r = idle_timeouts_locked(c, a.data(), t.data(), k, nullptr)) return r;
        if (int r = idle_restart_locked(c)) return r;
    }
    return 0;
}

// ---------------------------------------------------------------------------
// incremental replication (delta.cu; the blob is described in include/bng_b200.h)
// ---------------------------------------------------------------------------
namespace {
// shadow ids beside the hash maps' (map ids): the accounting records, the idle records
const int kShadowAcct = -1, kShadowIdle = -2;

// A hash map's (or the accounting or idle records') view for the diff: which words of a slot are compared, which is the
// time word.  Volatile fields are left out of the mask unless exact.
DeltaTbl delta_view(bng_ctx *c, const bng_ctx::DeltaShadow &s, u64 refresh, bool exact) {
    DeltaTbl t{};
    t.shadow = s.words;
    t.nslots = s.nslots;
    t.sw = s.sw;
    t.tw = DELTA_NO_TIME;
    t.refresh = refresh;
    auto set = [&](u32 pos) { t.mask[pos / 8] |= 0xFFull << (8 * (pos % 8)); };
    if (s.map == kShadowIdle) { // idle records: the directory's address, then the timeout (no time word; clocks are not sent)
        const Tbl &d = c->dev.subdir;
        t.slots = d.slots, t.slot_bytes = d.slot_bytes, t.vals = (const u8 *)c->idle.get(), t.vstride = sizeof(bng_idle);
        t.kw = 1, t.key_size = 4, t.value_size = 4;
        for (u32 b = 0; b < 4; b++) set(8 + b);
        return t;
    }
    if (s.map < 0) { // accounting records: the directory's address, then the record
        const Tbl &d = c->dev.subdir;
        t.slots = d.slots, t.slot_bytes = d.slot_bytes, t.vals = (const u8 *)c->acct.get(), t.vstride = sizeof(bng_acct);
        t.kw = 1, t.key_size = 4, t.value_size = sizeof(bng_acct);
        for (u32 b = 0; b < sizeof(bng_acct); b++) set(8 + b);
        return t;
    }
    const MapReg &m = c->maps[s.map];
    const Tbl &tb = *m.tbl;
    t.slots = tb.slots, t.slot_bytes = tb.slot_bytes;
    t.kw = tb.key_size <= 8 ? 1 : (tb.key_size + 7) / 8;
    t.key_size = tb.key_size, t.value_size = tb.value_size, t.voff = tb.voff, t.vlayout = tb.vlayout;
    const bool ses = tb.vlayout == VL_SESSION, eim = !strcmp(m.name, "eim_table");
    const bool qos = !strcmp(m.name, "qos_ingress") || !strcmp(m.name, "qos_egress");
    for (u32 b = 0; b < tb.value_size; b++) {
        const u32 pos = ses ? ses_abi_to_slot(b) : tb.voff + b;
        if (ses && pos >= SES_PAD_A) continue; // the struct's padding: never compared
        if (!exact) {
            if (ses && b >= 24 && b < 32) continue;              // last_seen: the time rule
            if (ses && b >= 40 && b < 72) continue;              // packets_* / bytes_*
            if (eim && b >= 16 && b < 24) continue;              // last_used: the time rule
            if (qos && b < 16) continue;                         // tokens; last_update: the time rule
        }
        set(pos);
    }
    if (!exact) {
        if (ses) t.tw = SES_LAST_SEEN / 8;
        if (eim || qos) t.tw = (tb.voff + (eim ? 16 : 8)) / 8;
    }
    return t;
}

int delta_words(const Tbl &t, bool ses) { // shadow words of a slot: through the last compared byte
    return ses ? SES_PAD_A / 8 : (int)((t.voff + t.value_size + 7) / 8);
}

int delta_shadow_locked(bng_ctx *c, int map, const Tbl &t, u32 sw) {
    const u64 nslots = (u64)t.mask + 1;
    const size_t bytes = nslots * sw * 8;
    DevBuf<u64> words;
    if (!words.grow(bytes))
        return grow_failed(c, "delta_enable", bytes,
                      (std::string("shadow of ") + (map == kShadowAcct ? kAcct : (map == kShadowIdle ? kIdle : c->maps[map].name))).c_str());
    CU(c, cudaMemsetAsync(words, 0xFF, bytes, c->L.stream)); // every slot empty: nothing sent yet
    c->dshadow.push_back({map, std::move(words), nslots, sw});
    if (!c->dlist.grow(nslots * 8)) return grow_failed(c, "delta_enable", nslots * 8);
    return 0;
}

void delta_free_locked(bng_ctx *c) {
    cudaStreamSynchronize(c->L.stream);
    c->dshadow.clear();
}
} // namespace

int bng_delta_enable(bng_ctx *c, int on) {
    if (!c) return -EINVAL;
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    delta_free_locked(c);
    if (!on) return 0;
    for (size_t mi = 0; mi < c->maps.size(); mi++) {
        const MapReg &m = c->maps[mi];
        if (m.kind != KIND_HASH) continue;
        if (int r = delta_shadow_locked(c, (int)mi, *m.tbl, delta_words(*m.tbl, m.tbl->vlayout == VL_SESSION))) {
            delta_free_locked(c);
            return r;
        }
    }
    if (c->acct) {
        if (int r = delta_shadow_locked(c, kShadowAcct, c->dev.subdir, 1 + ACCT_WORDS)) {
            delta_free_locked(c);
            return r;
        }
    }
    if (c->idle) {
        if (int r = delta_shadow_locked(c, kShadowIdle, c->dev.subdir, 2)) {
            delta_free_locked(c);
            return r;
        }
    }
    CU(c, cudaStreamSynchronize(c->L.stream));
    u64 id = 0;
    FILE *f = fopen("/dev/urandom", "rb");
    if (f) {
        if (fread(&id, 8, 1, f) != 1) id = 0;
        fclose(f);
    }
    id ^= splitmix64((u64)(uintptr_t)c ^ ((u64)clock() << 32) ^ (u64)time(nullptr));
    c->delta_stream = id ? id : 1;
    c->delta_seq = 0;
    c->delta_full = true;
    c->delta_li.clear();
    c->delta_li_sent = false;
    return 0;
}

int bng_delta_export(bng_ctx *c, uint64_t refresh_ns, uint32_t flags, void *buf, uint64_t cap, uint64_t *len_out) {
    if (!c || !len_out || (cap && !buf) || (flags & ~(BNG_DELTA_FULL | BNG_DELTA_EXACT))) return -EINVAL;
    *len_out = 0;
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    if (c->dshadow.empty()) return fail(c, -EINVAL, "delta_export: change tracking is not enabled");
    int r = flow_pass_begin_locked(c);
    if (r) return r;
    // records that began after tracking did start from "empty"
    auto has_shadow = [&](int id) {
        for (const auto &s : c->dshadow)
            if (s.map == id) return true;
        return false;
    };
    if (c->acct && !has_shadow(kShadowAcct)) {
        if ((r = delta_shadow_locked(c, kShadowAcct, c->dev.subdir, 1 + ACCT_WORDS)) != 0) return r;
    }
    if (c->idle && !has_shadow(kShadowIdle)) {
        if ((r = delta_shadow_locked(c, kShadowIdle, c->dev.subdir, 2)) != 0) return r;
    }
    const bool full = (flags & BNG_DELTA_FULL) || c->delta_full, exact = flags & BNG_DELTA_EXACT;
    blob::Writer w(sizeof(blob::DeltaHdr));
    struct Pending {
        DeltaTbl t;
        u64 at;
        u32 n_del, n_up;
    };
    std::vector<Pending> commits;
    u64 sent_used = 0;
    u32 *cnt = c->L.s.counters + 8; // scratch words 8.. are free between program runs
    for (const auto &s : c->dshadow) {
        const DeltaTbl t = delta_view(c, s, refresh_ns, exact);
        u32 *del = c->dlist, *up = c->dlist + s.nslots;
        CU(c, cudaMemsetAsync(cnt, 0, 8, c->L.stream));
        CU(c, run_delta_diff(c->L, t, del, up, cnt, full));
        u32 n[2] = {0, 0};
        CU(c, cudaMemcpyAsync(n, cnt, 8, cudaMemcpyDeviceToHost, c->L.stream));
        CU(c, cudaStreamSynchronize(c->L.stream));
        const u64 kb_del = (u64)n[0] * t.key_size, kb_up = (u64)n[1] * t.key_size, vb = (u64)n[1] * t.value_size;
        const u64 eb = kb_del + kb_up + vb, sb = (sent_used + n[0] + n[1]) * 4;
        if (cudaError_t e = eb > c->demit.size() ? c->demit.grow_keep(with_slack(eb), 0, c->L.stream) : cudaSuccess)
            return grow_failed(c, "delta_export", with_slack(eb), nullptr, e);
        if (cudaError_t e = sb > c->dsent.size() ? c->dsent.grow_keep(with_slack(sb), sent_used * 4, c->L.stream) : cudaSuccess)
            return grow_failed(c, "delta_export", with_slack(sb), nullptr, e);
        CU(c, run_delta_emit(c->L, t, del, n[0], up, n[1], c->demit, c->demit + kb_del, c->demit + kb_del + kb_up));
        if (n[0]) CU(c, cudaMemcpyAsync(c->dsent + sent_used, del, (u64)n[0] * 4, cudaMemcpyDeviceToDevice, c->L.stream));
        if (n[1]) CU(c, cudaMemcpyAsync(c->dsent + sent_used + n[0], up, (u64)n[1] * 4, cudaMemcpyDeviceToDevice, c->L.stream));
        commits.push_back({t, sent_used, n[0], n[1]});
        sent_used += n[0] + n[1];
        if (s.map == kShadowAcct)
            w.header(kAcct, blob::kAcctKind, 4, sizeof(bng_acct), n[1], n[0]);
        else if (s.map == kShadowIdle)
            w.header(kIdle, blob::kIdleKind, 4, 4, n[1], n[0]);
        else
            w.header(c->maps[s.map].name, KIND_HASH, t.key_size, t.value_size, n[1], n[0]);
        const size_t at = w.out.size();
        w.out.resize(at + kb_del + kb_up + vb);
        if (w.out.size() > at) CU(c, cudaMemcpyAsync(w.out.data() + at, c->demit, kb_del + kb_up + vb, cudaMemcpyDeviceToHost, c->L.stream));
        CU(c, cudaStreamSynchronize(c->L.stream));
    }
    for (auto &m : c->maps) { // the small maps, whole
        if (m.kind == KIND_HASH || m.kind == KIND_EVENT) continue;
        if ((r = map_section_locked(c, &m, w)) != 0) return r;
    }
    const std::vector<std::pair<u32, u32>> li = li_sorted(c);
    const bool li_send = c->li_ctl && (full || !c->delta_li_sent || li != c->delta_li);
    if (li_send) li_section(w, li);
    blob::DeltaHdr h{};
    memcpy(h.magic, blob::kDeltaMagic, 8);
    h.stream = c->delta_stream, h.seq_from = c->delta_seq, h.seq_to = c->delta_seq + 1;
    h.flags = (full ? BNG_DELTA_FULL : 0) | (exact ? BNG_DELTA_EXACT : 0), h.sections = (u32)w.sections;
    memcpy(w.out.data(), &h, sizeof(h));
    *len_out = w.out.size();
    prof_collect(c->L);
    if (cap < w.out.size()) return -ENOSPC; // the shadows are as they were: the next call covers the same changes
    memcpy(buf, w.out.data(), w.out.size());
    // the baseline moves to what this delta carries
    if (full)
        for (const auto &s : c->dshadow) CU(c, cudaMemsetAsync(s.words, 0xFF, s.nslots * s.sw * 8, c->L.stream));
    for (const auto &p : commits)
        CU(c, run_delta_commit(c->L, p.t, c->dsent + p.at, p.n_del, c->dsent + p.at + p.n_del, p.n_up));
    CU(c, cudaStreamSynchronize(c->L.stream));
    c->delta_seq++;
    c->delta_full = false;
    if (li_send) c->delta_li = li, c->delta_li_sent = true;
    return 0;
}

int bng_delta_apply(bng_ctx *c, const void *buf, uint64_t len) {
    if (!c || !buf || len < sizeof(blob::DeltaHdr)) return -EINVAL;
    blob::DeltaHdr h;
    memcpy(&h, buf, sizeof(h));
    if (memcmp(h.magic, blob::kDeltaMagic, 8)) return fail(c, -EINVAL, "delta_apply: not a delta");
    const bool full = h.flags & BNG_DELTA_FULL;
    std::vector<blob::Section> all;
    std::string err;
    if (!blob::read_sections((const u8 *)buf + sizeof(h), (const u8 *)buf + len, h.sections, true, false, all, err))
        return fail(c, -EINVAL, "delta_apply: %s", err.c_str());
    // the whole blob is checked before anything changes; maps this library does not have are skipped
    enum { ACCT = -2, LI = -3, IDLE = -4 };
    std::vector<std::pair<int, const blob::Section *>> secs;
    for (const blob::Section &s : all) {
        const blob::SectionHdr &sh = s.h;
        if (sh.count > (1ull << 40) || sh.key_size > 64 || sh.value_size > 4096)
            return fail(c, -EINVAL, "delta_apply: %s has a bad header", sh.name);
        int id;
        bool ok = sh.key_size == 4;
        if (!strcmp(sh.name, kAcct)) {
            id = ACCT, ok = ok && sh.value_size == sizeof(bng_acct);
        } else if (!strcmp(sh.name, kLi)) {
            id = LI, ok = ok && sh.value_size == 4 && sh.count <= BNG_LI_MAX_TARGETS;
        } else if (!strcmp(sh.name, kIdle)) {
            id = IDLE, ok = ok && sh.value_size == 4;
        } else {
            if ((id = bng_map_id(c, sh.name)) < 0) continue;
            const MapReg *m = get_map(c, id);
            ok = m->key_size == sh.key_size && m->value_size == sh.value_size && (u32)m->kind == sh.kind && (m->kind == KIND_HASH || !s.n_del);
        }
        if (!ok) return fail(c, -EINVAL, "delta_apply: %s has another layout", sh.name);
        secs.emplace_back(id, &s);
    }
    {
        std::lock_guard<std::mutex> g(c->mu);
        cudaSetDevice(c->device);
        if (!full && (h.stream != c->dapply_stream || h.seq_from != c->dapply_seq || !c->dapply_stream))
            return fail(c, -ESTALE, "delta_apply: stream %llx seq %llu, expected stream %llx seq %llu", (unsigned long long)h.stream,
                        (unsigned long long)h.seq_from, (unsigned long long)c->dapply_stream, (unsigned long long)c->dapply_seq);
        c->dapply_stream = 0; // until this apply has completed, only a FULL delta is accepted
        if (full) {
            if (int r = records_reset_locked(c)) return r;
        }
    }
    for (const auto &[id, s] : secs) {
        if (id < 0) continue;
        MapReg *m = get_map(c, id);
        if (full || m->kind != KIND_HASH) {
            if (int r = map_clear_for_load(c, id)) return r;
        }
        if (s->n_del) {
            std::lock_guard<std::mutex> g(c->mu);
            cudaSetDevice(c->device);
            if (int r = flush_staged_locked(c, id)) return r;
            int first = 0; // a key the standby no longer has is no error
            if (int r = hash_cmd(c, m, TOP_DELETE, s->dels, nullptr, s->n_del, 0, &first)) return r;
            if (feeds_small_tabs(m)) c->small_dirty = true;
        }
        if (s->h.count) {
            if (int r = bng_map_update_batch(c, id, s->keys, s->vals, s->h.count, BNG_ANY)) return fail(c, r, "delta_apply: loading %s failed", s->h.name);
        }
    }
    // after the maps: the records go to the addresses' directory slots
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    for (const auto &[id, s] : secs) {
        const u64 n = s->h.count;
        if (id == ACCT && n) {
            if (int r = load_records_locked(c, s->keys, s->vals, n, sizeof(bng_acct))) return r;
        } else if (id == LI) {
            if (int r = li_targets_load_locked(c, s->keys, s->vals, n, true)) return r;
        } else if (id == IDLE) {
            std::vector<u32> a(n), t(n);
            if (n) memcpy(a.data(), s->keys, n * 4), memcpy(t.data(), s->vals, n * 4);
            if (int r = idle_timeouts_locked(c, a.data(), t.data(), n, nullptr)) return r;
        }
    }
    // every clock restarts: at a takeover no clock here started before the last delta applied
    if (int r = idle_restart_locked(c)) return r;
    CU(c, cudaStreamSynchronize(c->L.stream));
    c->dapply_stream = h.stream;
    c->dapply_seq = h.seq_to;
    return 0;
}

int bng_delta_info(bng_ctx *c, uint64_t *stream_id, uint64_t *seq) {
    if (!c) return -EINVAL;
    std::lock_guard<std::mutex> g(c->mu);
    const bool exporter = !c->dshadow.empty();
    if (stream_id) *stream_id = exporter ? c->delta_stream : c->dapply_stream;
    if (seq) *seq = exporter ? c->delta_seq : c->dapply_seq;
    return 0;
}

// ---------------------------------------------------------------------------
// subscriber hand-over between contexts (move.cu; the blob is described in include/bng_b200.h)
// ---------------------------------------------------------------------------
namespace {
// what a subscriber owns: maps keyed by its address, by its MAC, and the flow tables (selected by k_move_select)
const char *const kMoveAddrMaps[] = {"subscriber_nat", "qos_ingress", "qos_egress"};
const char *const kMoveMacMaps[] = {"subscriber_bindings", "subscriber_pools"};
const char *const kMoveFlowMaps[] = {"nat_sessions", "nat_reverse", "eim_table"};
} // namespace

int bng_sub_export(bng_ctx *c, const uint32_t *addrs, uint64_t n_addrs, const uint64_t *macs, uint64_t n_macs, uint32_t flags,
                   void *buf, uint64_t cap, uint64_t *len_out) {
    if (!c || !len_out || (n_addrs && !addrs) || (n_macs && !macs) || (cap && !buf) || (flags & ~BNG_SUB_DETACH)) return -EINVAL;
    *len_out = 0;
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    if (int fr = flush_staged_locked(c, -1)) return fr;
    // distinct addresses and MACs, in the order given
    std::vector<u32> A;
    std::vector<u64> M;
    {
        std::unordered_set<u32> seen;
        for (u64 i = 0; i < n_addrs; i++)
            if (seen.insert(addrs[i]).second) A.push_back(addrs[i]);
    }
    {
        std::unordered_set<u64> seen;
        for (u64 i = 0; i < n_macs; i++)
            if (seen.insert(macs[i]).second) M.push_back(macs[i]);
    }
    const u64 na = A.size(), nm = M.size();
    u64 slots = 64;
    while (slots < 2 * na) slots *= 2;
    if (slots > (1ull << 32)) return fail(c, -EINVAL, "sub_export: %llu addresses", (unsigned long long)na);
    const DevCtx &d = c->dev;
    const u64 ns = (u64)d.sessions.mask + 1, nr = (u64)d.reverse.mask + 1, ne = (u64)d.eim.mask + 1, n6s = (u64)c->v6.mask + 1;
    // the slot lists (4 bytes per slot of the three flow tables and subscriber_ipv6), allocated by the first export that
    // has addresses
    if (na && !c->mv_lists.grow((ns + nr + ne + n6s) * 4)) return grow_failed(c, "sub_export", (ns + nr + ne + n6s) * 4);
    u32 *v6_list = c->mv_lists ? c->mv_lists + ns + nr + ne : nullptr;
    // staging: [in] address set, addresses, MACs, counters; [out] lookups by key, then the gathered flow entries
    MapReg *am[3], *mm[2], *fm[3];
    for (int k = 0; k < 3; k++) am[k] = get_map(c, bng_map_id(c, kMoveAddrMaps[k])), fm[k] = get_map(c, bng_map_id(c, kMoveFlowMaps[k]));
    for (int k = 0; k < 2; k++) mm[k] = get_map(c, bng_map_id(c, kMoveMacMaps[k]));
    const size_t aoff = al256(slots * 8), moff = al256(aoff + na * 4), coff = al256(moff + nm * 8), out0 = al256(coff + 32);
    size_t at = out0, am_v[3], am_r[3], mm_v[2], mm_r[2], acct_v = 0, acct_r = 0, idle_v = 0, idle_r = 0;
    for (int k = 0; k < 3; k++) am_v[k] = at, am_r[k] = al256(at + na * am[k]->value_size), at = al256(am_r[k] + na * 4);
    for (int k = 0; k < 2; k++) mm_v[k] = at, mm_r[k] = al256(at + nm * mm[k]->value_size), at = al256(mm_r[k] + nm * 4);
    if (c->acct) acct_v = at, acct_r = al256(at + na * sizeof(bng_acct)), at = al256(acct_r + na * 4);
    if (c->idle) idle_v = at, idle_r = al256(at + na * sizeof(bng_idle)), at = al256(idle_r + na * 4);
    // nd_bindings by MAC, only while it has entries: an export from a context that never used it launches nothing more
    MapReg *ndm = get_map(c, bng_map_id(c, "nd_bindings"));
    const bool nd = nm && c->nd_live;
    size_t nd_v = 0, nd_r = 0;
    if (nd) nd_v = at, nd_r = al256(at + nm * ndm->value_size), at = al256(nd_r + nm * 4);
    const size_t flow0 = at;
    if (cudaError_t e = flow0 > c->mv_buf.size() ? c->mv_buf.grow_keep(with_slack(flow0), 0, c->L.stream) : cudaSuccess)
        return grow_failed(c, "sub_export", with_slack(flow0), nullptr, e);
    // the inputs are built in the pinned staging buffer and copied on the context's stream, ahead of the kernels that
    // read them (as bng_nat_flush does)
    if (int r = ensure_io(c, out0)) return r;
    u8 *in = c->io_host;
    memset(in, 0, out0);
    u64 *set = (u64 *)in;
    const u32 mask = (u32)(slots - 1);
    for (u32 a : A) {
        u32 i = aset_home(a, mask);
        while (set[i]) i = (i + 1) & mask;
        set[i] = ADDRSET_LIVE | a;
    }
    if (na) memcpy(in + aoff, A.data(), na * 4);
    if (nm) memcpy(in + moff, M.data(), nm * 8);
    u8 *dv = c->mv_buf;
    CU(c, cudaMemcpyAsync(dv, in, out0, cudaMemcpyHostToDevice, c->L.stream));
    for (int k = 0; k < 3; k++)
        CU(c, run_table_op(c->L, *am[k]->tbl, TOP_LOOKUP, dv + aoff, dv + am_v[k], (int *)(dv + am_r[k]), na, 0, d.subdir, 0, nullptr, nullptr));
    for (int k = 0; k < 2; k++)
        CU(c, run_table_op(c->L, *mm[k]->tbl, TOP_LOOKUP, dv + moff, dv + mm_v[k], (int *)(dv + mm_r[k]), nm, 0, d.subdir, 0, nullptr, nullptr));
    if (nd) CU(c, run_table_op(c->L, c->ndb, TOP_LOOKUP, dv + moff, dv + nd_v, (int *)(dv + nd_r), nm, 0, d.subdir, 0, nullptr, nullptr));
    if (c->acct) CU(c, run_acct_read(c->L, d.subdir, c->acct, (const u32 *)(dv + aoff), na, (u64 *)(dv + acct_v), (int *)(dv + acct_r)));
    if (c->idle) CU(c, run_idle_read(c->L, d.subdir, c->idle, (const u32 *)(dv + aoff), na, (u64 *)(dv + idle_v), (int *)(dv + idle_r)));
    u32 *cnt = (u32 *)(dv + coff);
    CU(c, cudaMemsetAsync(cnt, 0, 32, c->L.stream));
    if (na) CU(c, run_move_select(c->L, d, AddrSet{(const u64 *)dv, mask}, c->mv_lists, cnt));
    // subscriber_ipv6 by value, only while it has entries: an export from a context that never used it launches nothing more
    if (na && c->v6_live) CU(c, run_move_select_v6(c->L, c->v6, AddrSet{(const u64 *)dv, mask}, v6_list, cnt + 4));
    u32 n4[5] = {0, 0, 0, 0, 0}; // entries listed in nat_sessions, nat_reverse, eim_table; tombstones; subscriber_ipv6
    CU(c, cudaMemcpyAsync(n4, cnt, 20, cudaMemcpyDeviceToHost, c->L.stream));
    CU(c, cudaStreamSynchronize(c->L.stream));
    // the delta exporter's gather turns the slot lists into ABI keys and values
    size_t fk[3], fv[3];
    at = flow0;
    for (int k = 0; k < 3; k++) {
        const Tbl &t = *fm[k]->tbl;
        fk[k] = at, fv[k] = at + (size_t)n4[k] * t.key_size, at = al256(fv[k] + (size_t)n4[k] * t.value_size);
    }
    const u32 n6 = n4[4];
    const size_t v6k = at, v6v = al256(v6k + (size_t)n6 * LPM6_KEY), v6r = al256(v6v + (size_t)n6 * 4); // v6r: the detach's results
    if (n6) at = al256(v6r + (size_t)n6 * 4);
    if (cudaError_t e = at > c->mv_buf.size() ? c->mv_buf.grow_keep(with_slack(at), flow0, c->L.stream) : cudaSuccess)
        return grow_failed(c, "sub_export", with_slack(at), nullptr, e);
    dv = c->mv_buf;
    for (int k = 0; k < 3 && c->mv_lists; k++) {
        const u32 *lists[3] = {c->mv_lists, c->mv_lists + ns, c->mv_lists + ns + nr};
        const Tbl &t = *fm[k]->tbl;
        DeltaTbl v{};
        v.slots = t.slots, v.slot_bytes = t.slot_bytes, v.nslots = (u64)t.mask + 1;
        v.key_size = t.key_size, v.value_size = t.value_size, v.voff = t.voff, v.vlayout = t.vlayout;
        CU(c, run_delta_emit(c->L, v, nullptr, 0, lists[k], n4[k], nullptr, dv + fk[k], dv + fv[k]));
    }
    if (n6) {
        DeltaTbl v{};
        v.slots = c->v6.slots, v.slot_bytes = c->v6.slot_bytes, v.nslots = n6s;
        v.key_size = c->v6.key_size, v.value_size = c->v6.value_size, v.voff = c->v6.voff;
        CU(c, run_delta_emit(c->L, v, nullptr, 0, v6_list, n6, nullptr, dv + v6k, dv + v6v));
    }
    std::vector<u8> got(at - out0);
    CU(c, cudaMemcpyAsync(got.data(), dv + out0, got.size(), cudaMemcpyDeviceToHost, c->L.stream)); // the one copy out
    CU(c, cudaStreamSynchronize(c->L.stream));
    prof_collect(c->L);
    auto host = [&](size_t off) { return got.data() + (off - out0); };
    // the blob: snapshot framing, one section per map, then the records and the interception targets
    blob::Writer w(16);
    auto by_key = [&](MapReg *m, const u8 *keys, u64 n, size_t voff, size_t roff, bool skip_empty = false) {
        const int *res = (const int *)host(roff);
        const u8 *vals = host(voff);
        std::vector<u8> kv, vv;
        for (u64 i = 0; i < n; i++)
            if (res[i] == 0) {
                kv.insert(kv.end(), keys + i * m->key_size, keys + (i + 1) * m->key_size);
                vv.insert(vv.end(), vals + i * m->value_size, vals + (i + 1) * m->value_size);
            }
        const u64 k = kv.size() / m->key_size;
        if (skip_empty && !k) return false;
        w.section(m->name, KIND_HASH, m->key_size, m->value_size, k, kv.data(), vv.data());
        return true;
    };
    for (int k = 0; k < 3; k++) by_key(am[k], (const u8 *)A.data(), na, am_v[k], am_r[k]);
    for (int k = 0; k < 2; k++) by_key(mm[k], (const u8 *)M.data(), nm, mm_v[k], mm_r[k]);
    // only when there is one, so that blobs without ND bindings stay as they were
    const bool nd_sec = nd && by_key(ndm, (const u8 *)M.data(), nm, nd_v, nd_r, true);
    for (int k = 0; k < 3; k++) {
        const MapReg *m = fm[k];
        w.section(m->name, KIND_HASH, m->key_size, m->value_size, n4[k], host(fk[k]), host(fv[k]));
    }
    const MapReg *m6 = get_map(c, bng_map_id(c, "subscriber_ipv6"));
    // only when there is one, so that blobs without IPv6 prefixes stay as they were
    if (n6) w.section(m6->name, KIND_HASH, m6->key_size, m6->value_size, n6, host(v6k), host(v6v));
    auto records = [&](const char *name, u32 kind, size_t rs, size_t voff, size_t roff) {
        const int *res = (const int *)host(roff);
        std::vector<u32> a;
        std::vector<u8> v;
        for (u64 i = 0; i < na; i++)
            if (res[i] == 0) a.push_back(A[i]), v.insert(v.end(), host(voff) + i * rs, host(voff) + (i + 1) * rs);
        w.section(name, kind, 4, (u32)rs, a.size(), a.data(), v.data());
    };
    if (c->acct) records(kAcct, blob::kAcctKind, sizeof(bng_acct), acct_v, acct_r);
    if (c->idle) records(blob::kIdleRec, blob::kIdleRecKind, sizeof(bng_idle), idle_v, idle_r);
    std::vector<u32> li_a;
    if (c->li_ctl) {
        std::vector<u32> ids;
        for (u32 a : A) {
            auto it = c->li_targets.find(a);
            if (it != c->li_targets.end()) li_a.push_back(a), ids.push_back(it->second);
        }
        w.pairs(kLi, blob::kLiKind, li_a, ids);
    }
    memcpy(w.out.data(), blob::kMoveMagic, 8);
    memcpy(w.out.data() + 8, &w.sections, 8);
    *len_out = w.out.size();
    if (cap < w.out.size()) return -ENOSPC; // nothing written, nothing removed
    memcpy(buf, w.out.data(), w.out.size());
    if (!(flags & BNG_SUB_DETACH)) return 0;
    // Detach exactly what was exported: the listed flow slots, then the keyed entries through the table-op path (the
    // subscriber directory follows subscriber_nat and qos_ingress, and with it the records' lifetime).  Every input is
    // already on the device and nothing below allocates, so once the blob is written the removal cannot fail part way
    // for want of memory.  Deleting every given key deletes exactly the entries found: nothing ran in between, and a
    // key without an entry is a miss that changes nothing.
    if (c->mv_lists) CU(c, run_move_detach(c->L, d, c->mv_lists, n4));
    for (int k = 0; k < 5; k++) {
        MapReg *m = k < 3 ? am[k] : mm[k - 3];
        const int role = m->tbl == &d.sub_nat ? 1 : (m->tbl == &d.qos_in ? 2 : 0);
        CU(c, run_table_op(c->L, *m->tbl, TOP_DELETE, dv + (k < 3 ? aoff : moff), nullptr, (int *)(dv + (k < 3 ? am_r[k] : mm_r[k - 3])),
                           k < 3 ? na : nm, 0, d.subdir, role, c->acct, c->idle));
    }
    if (n6) CU(c, run_table_op(c->L, c->v6, TOP_DELETE, dv + v6k, nullptr, (int *)(dv + v6r), n6, 0, d.subdir, 0, nullptr, nullptr));
    if (nd_sec) CU(c, run_table_op(c->L, c->ndb, TOP_DELETE, dv + moff, nullptr, (int *)(dv + nd_r), nm, 0, d.subdir, 0, nullptr, nullptr));
    if (!li_a.empty()) {
        for (u32 a : li_a) c->li_targets.erase(a);
        c->li_dirty = true;
    }
    CU(c, cudaStreamSynchronize(c->L.stream));
    prof_collect(c->L);
    if (n6) {
        if (int r = v6_refresh_locked(c)) return r;
    }
    if (nd_sec) {
        if (int r = nd_refresh_locked(c)) return r;
    }
    // the flush's rebuild rule; a rebuild that finds no memory leaves the tables as they were, and the detach stands
    if (rebuild_if_tombstoned_locked(c, n4[3] + n4[0])) cudaGetLastError();
    return 0;
}

int bng_sub_import(bng_ctx *c, const void *buf, uint64_t len) {
    if (!c) return -EINVAL;
    if (!buf || len < 16 || memcmp(buf, blob::kMoveMagic, 8)) return fail(c, -EINVAL, "sub_import: not a hand-over blob");
    u64 n;
    memcpy(&n, (const u8 *)buf + 8, 8);
    std::vector<blob::Section> all;
    std::string err;
    if (!blob::read_sections((const u8 *)buf + 16, (const u8 *)buf + len, n, false, true, all, err))
        return fail(c, -EINVAL, "sub_import: %s", err.c_str());
    // the whole blob is checked before anything changes: every section must be one this library writes
    enum { ACCT = -1, IDLE = -2, LI = -3 };
    std::vector<std::pair<int, const blob::Section *>> secs;
    for (const blob::Section &s : all) {
        const blob::SectionHdr &sh = s.h;
        int id;
        bool ok = sh.key_size == 4;
        if (!strcmp(sh.name, kAcct)) {
            id = ACCT, ok = ok && sh.kind == blob::kAcctKind && sh.value_size == sizeof(bng_acct);
        } else if (!strcmp(sh.name, blob::kIdleRec)) {
            id = IDLE, ok = ok && sh.kind == blob::kIdleRecKind && sh.value_size == sizeof(bng_idle);
        } else if (!strcmp(sh.name, kLi)) {
            id = LI, ok = ok && sh.kind == blob::kLiKind && sh.value_size == 4 && sh.count <= BNG_LI_MAX_TARGETS;
        } else {
            id = bng_map_id(c, sh.name);
            const MapReg *m = id >= 0 ? get_map(c, id) : nullptr;
            ok = m && m->kind == KIND_HASH && sh.kind == KIND_HASH && m->key_size == sh.key_size && m->value_size == sh.value_size;
        }
        if (!ok) return fail(c, -EINVAL, "sub_import: %s is not a section of this library's layout", sh.name);
        secs.emplace_back(id, &s);
    }
    {   // room: nothing may be refused or evicted part way
        std::lock_guard<std::mutex> g(c->mu);
        cudaSetDevice(c->device);
        if (int fr = flush_staged_locked(c, -1)) return fr;
        std::unordered_map<int, u64> want;
        std::unordered_set<u32> li_new;
        for (const auto &[id, s] : secs) {
            if (id >= 0) want[id] += s->h.count;
            if (id == LI)
                for (u64 k = 0; k < s->h.count; k++) {
                    u32 a;
                    memcpy(&a, s->keys + k * 4, 4);
                    if (!c->li_targets.count(a)) li_new.insert(a);
                }
        }
        for (const auto &w : want) {
            const MapReg *m = get_map(c, w.first);
            u32 live = 0;
            CU(c, cudaMemcpyAsync(&live, m->tbl->count, 4, cudaMemcpyDeviceToHost, c->L.stream));
            CU(c, cudaStreamSynchronize(c->L.stream));
            if ((u64)live + w.second > m->max_entries)
                return fail(c, -E2BIG, "sub_import: %s holds %u of %u entries, the blob brings %llu", m->name, live, m->max_entries,
                            (unsigned long long)w.second);
        }
        if (c->li_targets.size() + li_new.size() > BNG_LI_MAX_TARGETS)
            return fail(c, -E2BIG, "sub_import: more than %d interception targets", BNG_LI_MAX_TARGETS);
    }
    for (const auto &[id, s] : secs) {
        if (id < 0 || !s->h.count) continue;
        if (int r = bng_map_update_batch(c, id, s->keys, s->vals, s->h.count, BNG_ANY)) return fail(c, r, "sub_import: loading %s failed", s->h.name);
    }
    // after the maps: the records go to the addresses' (new) directory slots
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    for (const auto &[id, s] : secs) {
        const u64 n = s->h.count;
        if (!n) continue;
        if (id == ACCT || id == IDLE) {
            if (int r = load_records_locked(c, s->keys, s->vals, n, id == ACCT ? sizeof(bng_acct) : sizeof(bng_idle))) return r;
        } else if (id == LI) {
            if (int r = li_targets_load_locked(c, s->keys, s->vals, n, false)) return r;
        }
    }
    return 0;
}

// ---------------------------------------------------------------------------
// multi-GPU plumbing and diagnostics
// ---------------------------------------------------------------------------
int bng_stats_device_ptr(bng_ctx *c, void **dptr, uint32_t *n_u64) {
    if (!c || !dptr) return -EINVAL;
    *dptr = c->dev.stats;
    if (n_u64) *n_u64 = ST_COUNT; // dhcpv6_stats and nd_stats follow them in the same buffer (include/bng_b200.h)
    return 0;
}

uint64_t bng_launch_count(bng_ctx *c) { return c ? c->L.launches : 0; }

int bng_dhcpv6_enable(bng_ctx *c, int on) { return set_switch(c, &bng_ctx::dhcp6, on); }
int bng_nd_enable(bng_ctx *c, int on) { return set_switch(c, &bng_ctx::nd, on); }
int bng_qos_ipv6_enable(bng_ctx *c, int on) { return set_switch(c, &bng_ctx::qos_v6, on); }
int bng_antispoof_ipv6_prefixes_enable(bng_ctx *c, int on) { return set_switch(c, &bng_ctx::as_v6, on); }
int bng_nat_icmp_errors_enable(bng_ctx *c, int on) { return set_switch(c, &bng_ctx::nat_icmp, on); }
int bng_nat_icmp_errors_egress_enable(bng_ctx *c, int on) { return set_switch(c, &bng_ctx::nat_icmp_eg, on); }

int bng_ipv6_prefix_lengths(bng_ctx *c, uint32_t *counts) {
    if (!c || !counts) return -EINVAL;
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    if (int fr = flush_staged_locked(c, bng_map_id(c, "subscriber_ipv6"))) return fr;
    CU(c, cudaMemcpyAsync(counts, c->v6.plens, LPM6_LENS * 4, cudaMemcpyDeviceToHost, c->L.stream));
    CU(c, cudaStreamSynchronize(c->L.stream));
    return 0;
}

int bng_prof_enable(bng_ctx *c, int on) {
    if (!c) return -EINVAL;
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->L.stream);
    prof_collect(c->L);
    c->L.prof = on ? 1 : 0;
    if (on) c->L.nacc = 0;
    return 0;
}

int64_t bng_prof_read(bng_ctx *c, char *buf, uint64_t cap) {
    if (!c || !buf || !cap) return -EINVAL;
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->L.stream);
    prof_collect(c->L);
    std::string out;
    char line[256];
    for (int i = 0; i < c->L.nacc; i++) {
        snprintf(line, sizeof(line), "%s %llu %.6f\n", c->L.acc_name[i], c->L.acc_n[i], c->L.acc_ms[i]);
        out += line;
    }
    size_t n = std::min<size_t>(out.size(), cap - 1);
    memcpy(buf, out.data(), n);
    buf[n] = 0;
    return (int64_t)n;
}

static uint64_t read_stat(bng_ctx *c, int idx) {
    if (!c) return 0;
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    u64 v = 0;
    if (cudaMemcpyAsync(&v, c->dev.stats + idx, 8, cudaMemcpyDeviceToHost, c->L.stream) != cudaSuccess) return 0;
    cudaStreamSynchronize(c->L.stream);
    return v;
}
uint64_t bng_lru_overflow(bng_ctx *c) { return read_stat(c, ST_LRU_OVERFLOW); }
uint64_t bng_lru_evictions(bng_ctx *c) { return read_stat(c, ST_LRU_EVICT); }
uint64_t bng_table_rebuilds(bng_ctx *c) { return c ? c->rebuilds : 0; }
uint64_t bng_events_lost(bng_ctx *c) { return read_stat(c, ST_EV_LOST_SPOOF) + read_stat(c, ST_EV_LOST_NATLOG); }

} // extern "C"
