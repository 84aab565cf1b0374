/* bng_b200 — C ABI of the H100-native subscriber dataplane.
 *
 * This is the drop-in boundary for the reference's eBPF hot path: everything
 * the Go control plane does to the dataplane goes through cilium/ebpf
 * `*ebpf.Map` Put/Lookup/Delete calls and program attach
 * (reference pkg/ebpf/loader.go:211-315,357-655; pkg/antispoof/manager.go:127-381;
 * pkg/qos/manager.go:89-320; pkg/nat/manager.go:563-821).  The functions below
 * are what a cgo shim binds instead (see INTEGRATION.md): maps are addressed
 * by the reference's map names and use the reference's key/value byte layouts
 * verbatim (bpf/antispoof.c:36-119, bpf/qos_ratelimit.c:24-65,
 * bpf/nat44.c:92-320, bpf/maps.h:89-234); programs are addressed by the
 * reference's program (ELF section function) names and run over BATCHES of
 * frames on the GPU instead of per packet in the kernel.
 *
 * Conventions
 *   - every function returns 0 or a negative errno, as bpf(2) does
 *     (-ENOENT lookup/delete miss, -EEXIST BPF_NOEXIST clash, -E2BIG map full,
 *     -EINVAL bad argument, -ENOMEM, -EIO CUDA failure; bng_last_error() has text)
 *   - key/value buffers are borrowed for the duration of the call only
 *   - all entry points are thread-safe (one mutex per context); program runs
 *     on one context are serialised on that context's CUDA stream.  Nothing in
 *     the library is process-wide: one process may hold contexts on several GPUs
 *   - reserved keys: a hash-map key whose first 8 bytes (zero-extended when the
 *     key is shorter) are 0xFFFFFFFFFFFFFFFD..FF cannot be stored (update:
 *     -EINVAL, lookup/delete: -ENOENT); no frame produces such a key except a
 *     nat_reverse lookup for 255.255.255.253-255 -> 255.255.255.255, which misses
 *   - PERCPU_ARRAY statistics maps read back as aggregated totals
 *   - there is NO CPU fallback: without a CUDA device bng_open() fails
 */
#ifndef BNG_B200_H
#define BNG_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BNG_ABI_VERSION 2

/* bpf(2) BPF_MAP_UPDATE_ELEM flags (include/uapi/linux/bpf.h) */
#define BNG_ANY 0u
#define BNG_NOEXIST 1u
#define BNG_EXIST 2u

/* verdict codes, identical to the kernel's */
#define BNG_TC_ACT_OK 0
#define BNG_TC_ACT_SHOT 2
#define BNG_XDP_DROP 1
#define BNG_XDP_PASS 2
#define BNG_XDP_TX 3

/* where the buffers of a bng_batch live */
#define BNG_MEM_DEVICE 0u /* device pointers; the run is asynchronous on bng_stream() */
#define BNG_MEM_HOST 1u   /* host pointers; the call copies in, runs, copies out, and returns synchronised */

typedef struct bng_ctx bng_ctx;

typedef struct bng_open_opts {
    uint32_t struct_size;      /* sizeof(bng_open_opts) */
    int32_t device;            /* CUDA device ordinal, -1 = current device */
    uint32_t max_batch;        /* largest bng_batch.n this context will see (scratch sizing); 0 = 1<<22 */
    uint32_t max_subscribers;  /* capacity of the per-subscriber hashes; 0 = reference MAX_SUBSCRIBERS (1e6) */
    uint32_t max_nat_sessions; /* nat_sessions / nat_reverse; 0 = reference MAX_NAT_SESSIONS (4e6) */
    uint32_t max_eim_mappings; /* eim_table; 0 = reference MAX_EIM_MAPPINGS (2e6) */
    uint32_t event_capacity;   /* staged event records per ring; 0 = 1<<21 */
    uint32_t rank;             /* this context's shard index (informational; see bng_shard_of_mac) */
    uint32_t world;            /* number of shards */
} bng_open_opts;

typedef struct bng_map_info {
    uint32_t type; /* enum bpf_map_type value the reference declares */
    uint32_t key_size;
    uint32_t value_size;
    uint32_t max_entries;
    uint64_t count; /* live entries (hash maps) */
} bng_map_info;

/* One batch of Ethernet frames (no FCS).  Frame i occupies bytes
 * [off16[i]*16, off16[i]*16 + len[i]) of the arena, or starts at i*stride when
 * off16 is NULL; every frame's storage must be readable and writable up to the
 * next multiple of 16 bytes.  Frames are applied in index order: the result is
 * bit-identical to running the reference program on frame 0, then 1, ...
 * with bpf_ktime_get_ns() returning now_ns throughout the batch — or, when
 * now_ns_v is given, now_ns_v[i] while frame i runs (the reference reads the
 * clock per packet: bpf/nat44.c:669, bpf/qos_ratelimit.c:80).  Per-frame
 * timestamps must be what that clock gives: monotonic, i.e. non-decreasing in
 * index order and from batch to batch (-EINVAL when a host array is not). */
typedef struct bng_batch {
    void *pkts;            /* arena base */
    const uint32_t *off16; /* [n] frame offsets in 16-byte units, or NULL */
    uint32_t *len;         /* [n] in: frame length (skb->len / data_end-data); out: length after the program */
    uint8_t *verdict;      /* [n] out: TC_ACT_* (tc programs, pipelines) or XDP_* (xdp programs) */
    uint32_t *priority;    /* [n] in/out skb->priority (qos_egress_prog writes it); may be NULL */
    uint32_t n;
    uint32_t stride;       /* bytes between frames when off16 == NULL (multiple of 16) */
    uint64_t now_ns;       /* bpf_ktime_get_ns() for this batch */
    uint32_t mem;          /* BNG_MEM_DEVICE or BNG_MEM_HOST */
    uint32_t arena_bytes;  /* size of the arena in 16-byte units (needed for BNG_MEM_HOST copies) */
    const uint64_t *now_ns_v; /* [n] per-frame bpf_ktime_get_ns(), or NULL (same memory space as the other arrays) */
} bng_batch;

/* ---- lifecycle (replaces ebpf.LoadCollectionSpec/NewCollection/Collection.Close,
 *      pkg/ebpf/loader.go:211-222,337-339) ---- */
bng_ctx *bng_open(const bng_open_opts *opts);
int bng_close(bng_ctx *ctx);
const char *bng_last_error(bng_ctx *ctx); /* ctx may be NULL: error of the last failed bng_open on this thread */
uint32_t bng_abi_version(void);

/* ---- maps (replaces coll.Maps[name] + Map.Put/Lookup/Delete) ---- */
int bng_map_id(bng_ctx *ctx, const char *name);
int bng_map_get_info(bng_ctx *ctx, int map, bng_map_info *out);
int bng_map_update(bng_ctx *ctx, int map, const void *key, const void *value, uint64_t flags);
int bng_map_update_batch(bng_ctx *ctx, int map, const void *keys, const void *values, uint64_t n, uint64_t flags);
int bng_map_lookup(bng_ctx *ctx, int map, const void *key, void *value_out);
int bng_map_delete(bng_ctx *ctx, int map, const void *key);
/* Staged upsert (BPF_ANY): queued on the host and applied with all other staged updates at the next batch
 * boundary (bng_prog_run), at bng_sync(), or before the next call that reads or changes the same map —
 * so it is always visible to a later lookup.  The last staged value of a key wins, as with one Put after
 * the other.  This is what the per-lease / per-session Map.Put calls of the Go managers should bind to
 * (pkg/dhcp/server.go:708,780,798; pkg/nat/manager.go:563-640): a synchronous bng_map_update costs two PCIe
 * copies and a kernel launch per call.  Returns 0, or -EINVAL. */
int bng_map_update_staged(bng_ctx *ctx, int map, const void *key, const void *value);
int bng_staged_info(bng_ctx *ctx, uint64_t *pending, uint64_t *flushes, uint64_t *errors);
int bng_map_clear(bng_ctx *ctx, int map); /* drop every entry of a hash map (= close + re-create the eBPF map) */
/* copies up to cap (key,value) pairs out; returns the number written or a negative errno */
int64_t bng_map_dump(bng_ctx *ctx, int map, void *keys_out, void *values_out, uint64_t cap);

/* ---- programs (replaces coll.Programs[name] + link.AttachXDP / netlink FilterAdd;
 *      a batch run is the analogue of BPF_PROG_TEST_RUN over n frames) ---- */
int bng_prog_id(bng_ctx *ctx, const char *name);
int bng_prog_run(bng_ctx *ctx, int prog, bng_batch *batch);
int bng_sync(bng_ctx *ctx);     /* apply staged upserts, wait for everything queued on the context's stream */
void *bng_stream(bng_ctx *ctx); /* the context's cudaStream_t */

/* ---- session expiry (SURVEY.md 8f-3; the reference declares the timeouts, bpf/nat44.c:50-53, and enforces
 *      them nowhere: pkg/nat/manager.go:667-679 is a logger) ----
 * One streaming pass over nat_sessions: a session idle longer than its timeout at now_ns (ICMP 60 s, UDP 120 s,
 * TCP established 7200 s, other TCP states 240 s) is removed with its nat_reverse entry (when that still points
 * at it) and one reference of its EIM mapping (the mapping goes with its last session); the subscriber's
 * sessions_active is decremented, nat_stats.sessions_expired counted, a NAT_LOG_SESSION_DELETE record logged
 * (records of one sweep drain ordered by their bytes).  *expired_out = sessions removed.
 * The three NAT flow maps are BPF_MAP_TYPE_LRU_HASH in the reference: an insert into a full one evicts the least
 * recently used entry among the 16 slots next to the new key's home slot instead of failing. */
int bng_sweep(bng_ctx *ctx, uint64_t now_ns, uint64_t *expired_out);

/* ---- NAT flow-state flush (what a subscriber's release / RADIUS Disconnect needs) ----
 * Removes the NAT flow state of a set of subscriber addresses.  Until it expires, a departed subscriber's flow state
 * keeps translating: return traffic to its public ports is DNATed to the private address (nat44_ingress never
 * consults subscriber_nat), and the address's next holder hits its sessions and EIM mappings upstream.
 * addrs: n host-memory addresses, 4 bytes each, in the byte order of the subscriber_nat / qos_ingress key (as
 * bng_acct_read takes them); duplicates are allowed and every value is an address, 0 and 0xFFFFFFFF included.
 * With A the set of addresses, one call
 *   - deletes every nat_sessions entry whose key src_ip is in A, and writes one NAT_LOG_SESSION_DELETE record per
 *     deleted session to nat_log_rb: the sweep's record (subscriber_id from the address's subscriber_nat entry, 0
 *     without one), with timestamp now_ns, drained ordered by content as the sweep's are; nat_log_rb's capacity and
 *     bng_events_lost apply as usual;
 *   - deletes every nat_reverse entry whose value (the original upstream nat_key) has src_ip in A, stale entries
 *     whose session has already gone included;
 *   - deletes every eim_table entry whose internal_ip is in A, whatever its ref_count;
 *   - sets sessions_active of every subscriber_nat entry keyed by an address in A to 0 (block, next_port and
 *     subscriber_id stay).
 * Nothing else changes: not nat_stats (this is not an expiry), not the accounting records, not qos_* or any other
 * map.  The caller deletes those by key.  Flush before deleting the subscriber_nat entry, so that the records still
 * carry the subscriber_id.
 * Ordering is bng_sweep's: staged upserts are applied first; the call is a batch of its own (it advances the batch
 * sequence) queued on the context's stream behind everything before it, BNG_MEM_DEVICE batches that were not
 * synchronised included; it returns synchronised, and rebuilds the flow tables under bng_sweep's rule.
 * removed_out (may be NULL): sessions, nat_reverse entries and eim_table entries removed.  n == 0 applies the staged
 * upserts and returns 0 with zero counts.  -EINVAL for a NULL ctx, or NULL addrs with n > 0.
 * The pass streams the three flow tables once (about 0.67 GB at the reference's capacities); the set of addresses
 * takes 8 bytes per slot of a power of two >= 2n in the context's staging buffers, which grow to hold it. */
int bng_nat_flush(bng_ctx *ctx, const uint32_t *addrs, uint64_t n, uint64_t now_ns, uint64_t removed_out[3]);

/* ---- events (spoof_events perf buffer, nat_log_rb ring buffer) ----
 * Records come out in the order the reference would have emitted them (batch
 * order, then frame index); nat_log_rb applies the kernel ring's capacity
 * (records that would not have fitted are dropped, as bpf_ringbuf_reserve
 * failing does in bpf/nat44.c:545-547). */
int bng_events_drain(bng_ctx *ctx, int map, void *buf, uint64_t cap_records, uint64_t *n_out);
uint32_t bng_event_size(bng_ctx *ctx, int map);

/* ---- multi-GPU plumbing ----
 * Frames shard by subscriber MAC: shard = bng_shard_of_mac(mac_key, world).
 * The packed statistics vector (all PERCPU/array counters of the four
 * programs, BNG_NUM_STATS u64) can be all-reduced in place by the host's
 * collective library (NCCL) between batches. */
#define BNG_NUM_STATS 40
uint32_t bng_shard_of_mac(uint64_t mac_key, uint32_t world);
int bng_stats_device_ptr(bng_ctx *ctx, void **dptr, uint32_t *n_u64);
/* Counter reconciliation over NCCL (SURVEY.md §8e: "ncclAllReduce(SUM, uint64) on the packed counter vector at
 * bng_sync").  One context per GPU, one communicator over all of them: rank 0 calls bng_comm_unique_id(), the
 * host plumbing hands the 128 bytes to every rank, every rank calls bng_comm_init() (collective).
 * bng_sync_reduce() then flushes staged upserts and all-reduces the BNG_NUM_STATS counters on the context's
 * stream — per-shard counters stay what they are; the totals land in totals_out (host, may be NULL).  Without a
 * communicator it returns this context's own counters.  libnccl.so.2 is resolved at run time from the host
 * process (BNG_NCCL_LIB overrides the name): the library does not link it.  -ENOSYS when it cannot be found. */
int bng_comm_unique_id(void *id_out, uint64_t cap /* >= 128 */);
int bng_comm_init(bng_ctx *ctx, const void *id, uint32_t rank, uint32_t world);
int bng_sync_reduce(bng_ctx *ctx, uint64_t *totals_out /* [BNG_NUM_STATS] */);

/* ---- snapshot / restore (SURVEY.md 8f-4: table state for HA hand-over, reference pkg/ha) ----
 * bng_snapshot() serialises every hash / array / LPM / statistics map into buf and returns the number of bytes
 * the snapshot needs (call with cap 0 to size the buffer; nothing is written when cap is too small).
 * bng_restore() replaces the contents of every map named in the blob; capacities may differ between the two
 * contexts, layouts may not.  Event rings are not part of a snapshot. */
int64_t bng_snapshot(bng_ctx *ctx, void *buf, uint64_t cap);
int bng_restore(bng_ctx *ctx, const void *buf, uint64_t len);

/* ---- per-subscriber traffic accounting (what RADIUS Accounting Interim-Update / Stop report) ----
 * One record per subscriber address: an address that keys a subscriber_nat or a qos_ingress entry (staged upserts
 * included).  Counters are totals since the address got its entry; they never go backwards.
 *   - Bytes are the frame's len as the batch passes it in (skb->len).
 *   - Upstream programs (nat44_egress, qos_ingress_prog, pipeline_up, pipeline_tc) charge a frame to the IPv4 SOURCE
 *     address it entered the program with (before SNAT): untagged Ethernet II, ethertype 0x0800, bytes 26-29 present.
 *   - Downstream programs (nat44_ingress, qos_egress_prog) charge a frame to the IPv4 DESTINATION address it leaves
 *     with (after DNAT), bytes 30-33: a frame nat44_ingress did not translate keeps its public address.
 *   - Verdict TC_ACT_OK counts in the pass pair, TC_ACT_SHOT in the drop pair (NAT port exhaustion, token bucket).
 *     In the two pipelines a frame that antispoof drops is not counted at all: it may have forged its address.
 *   - A frame whose address has no entry when the batch runs is not counted anywhere.
 *   - A record starts at zero when its address gets its entry; it survives updates of either map, the expiry
 *     sweep, LRU eviction and flow-table rebuilds, and ends when the address loses both entries (delete or
 *     bng_map_clear).  Snapshots carry the records (a trailing "subscriber_acct" section), so an HA hand-over keeps
 *     them; bng_restore() of a blob without that section leaves every record at zero.
 * Accounting is enabled per program and off by default.  The first bng_acct_enable() allocates the records:
 * 64 bytes per subscriber-directory slot, i.e. 64 x (the power of two >= max(64, 2 x max_subscribers)) bytes —
 * 128 MiB at the default 1e6 subscribers — plus 4 bytes per frame of max_batch.  A context that never enables
 * accounting allocates neither. */
typedef struct bng_acct {
    uint64_t up_packets, up_bytes;            /* upstream, verdict TC_ACT_OK */
    uint64_t up_drop_packets, up_drop_bytes;  /* upstream, verdict TC_ACT_SHOT */
    uint64_t down_packets, down_bytes;        /* downstream, verdict TC_ACT_OK */
    uint64_t down_drop_packets, down_drop_bytes;
} bng_acct;
/* on != 0 enables accounting of the program's runs from the next bng_prog_run on.  -EOPNOTSUPP for
 * antispoof_ingress, nat44_hairpin_xdp and dhcp_fastpath_prog; -EINVAL for an unknown program id. */
int bng_acct_enable(bng_ctx *ctx, int prog, int on);
/* Records of n addresses (4 bytes each, in the byte order of the qos_ingress key).  results[i] = 0, or -ENOENT
 * when the address has no entry (out[i] is then zeroed).  Staged upserts are applied first and the read sees
 * everything queued on the context's stream, as bng_map_lookup() does.  Returns 0 or a negative errno. */
int bng_acct_read(bng_ctx *ctx, const uint32_t *addrs, uint64_t n, bng_acct *out, int32_t *results);
/* Up to cap (address, record) pairs of the addresses that have an entry, in no particular order (compacted on the
 * GPU, then copied out).  Returns the number written or a negative errno, as bng_map_dump() does. */
int64_t bng_acct_dump(bng_ctx *ctx, uint32_t *addrs_out, bng_acct *out, uint64_t cap);

/* ---- lawful intercept: content of communication (what pkg/intercept's RecordCC takes) ----
 * A frame of a target address is copied, as the subscriber's side of the BNG sees it, into a record on the GPU;
 * bng_li_drain() hands the records out in frame order.
 * Which frames are captured: exactly the frames accounting would charge, attributed by the same rule.
 *   - Upstream programs (nat44_egress, qos_ingress_prog, pipeline_up, pipeline_tc): a frame whose IPv4 SOURCE, as the
 *     frame entered the program, is a target: untagged Ethernet II, ethertype 0x0800, bytes 26-29 present.
 *   - Downstream programs (nat44_ingress, qos_egress_prog): a frame whose IPv4 DESTINATION, as the frame leaves the
 *     program (after DNAT), is a target: bytes 30-33 present.
 *   - The verdict is TC_ACT_OK or TC_ACT_SHOT; both are captured.  In the two pipelines a frame that antispoof drops
 *     is not captured: it may have forged its address.  Other programs never capture.
 *   - A target is any address; it needs no subscriber_nat or qos_ingress entry.  The targets in force are those set
 *     when bng_prog_run is called.
 * What is captured: the first cap_len bytes of the frame as it entered the program (upstream, before SNAT) or as the
 * program left it (downstream, after DNAT).  "Bytes present in the frame's storage" is len with an offset table and
 * min(len, stride) in a fixed-stride arena.  The bytes of a record past cap_len are zero.
 * Drain: records come out ordered by (batch, frame), each bng_li_record_size() bytes.  Records that do not fit in
 * cap_records stay for the next call, as bng_events_drain leaves them; the call sees everything queued on the
 * context's stream.  buf may be NULL when cap_records is 0.
 * Overflow: when the ring is full, the records that do not fit are dropped and counted in bng_li_lost().  Which
 * records of the overflowing batch survive is unspecified; every record that survives is complete and correct.
 * Lifecycle: the first bng_li_configure() or bng_li_target_set() allocates the ring (capacity x record size bytes)
 * and a table of up to BNG_LI_MAX_TARGETS targets; a context that never uses either allocates nothing, and with no
 * target set bng_prog_run launches no kernel for interception.  bng_li_configure() again replaces the ring: records
 * not yet drained are discarded and counted as lost.  bng_snapshot() carries the targets (a trailing "li_targets"
 * section), not the records; bng_restore() of a blob without that section leaves no targets.
 * The batch number is the context's batch sequence: 1 for its first bng_prog_run, advanced by every bng_prog_run,
 * bng_sweep and bng_nat_flush. */
#define BNG_LI_UPLINK 0
#define BNG_LI_DOWNLINK 1
#define BNG_LI_MAX_TARGETS 4096
typedef struct bng_li_record { /* 64 bytes; followed by the captured bytes, up to the record size */
    uint64_t ts_ns;     /* the frame's bpf_ktime_get_ns(): now_ns_v[i], or the batch's now_ns */
    uint64_t batch;     /* the run's batch sequence number: strictly increasing from run to run on a context */
    uint32_t frame;     /* index of the frame in its batch */
    uint32_t target_id; /* as given to bng_li_target_set */
    uint32_t addr;      /* the matched subscriber address, in the byte order of the qos_ingress key */
    uint32_t wire_len;  /* the frame's len (the TC programs never change it) */
    uint32_t cap_len;   /* captured bytes that follow: min(len, bytes present in the frame's storage, snaplen) */
    uint8_t dir;        /* BNG_LI_UPLINK / BNG_LI_DOWNLINK */
    uint8_t verdict;    /* TC_ACT_OK or TC_ACT_SHOT */
    uint8_t prog;       /* bng_prog_id() of the run */
    uint8_t pad[25];    /* zero */
} bng_li_record;
/* snaplen 0 = 1518 bytes, else 1..65535; capacity 0 = 2^15 records, else at most 2^30.  -EINVAL outside those,
 * -ENOMEM when the ring does not fit in device memory (the previous ring is then kept). */
int bng_li_configure(bng_ctx *ctx, uint32_t snaplen, uint32_t capacity);
uint32_t bng_li_record_size(bng_ctx *ctx); /* 64 + snaplen rounded up to 16; 0 before the ring exists */
int bng_li_target_set(bng_ctx *ctx, uint32_t addr, uint32_t target_id); /* insert or replace; -E2BIG when full */
int bng_li_target_del(bng_ctx *ctx, uint32_t addr);                      /* -ENOENT when absent */
/* *n_out = records copied to buf (n_out must not be NULL) */
int bng_li_drain(bng_ctx *ctx, void *buf, uint64_t cap_records, uint64_t *n_out);
uint64_t bng_li_lost(bng_ctx *ctx); /* records dropped because the ring was full, or discarded by a reconfiguration */

/* ---- diagnostics ---- */
uint64_t bng_launch_count(bng_ctx *ctx);  /* kernels launched by this context so far */
uint64_t bng_lru_overflow(bng_ctx *ctx);  /* inserts that found no victim to evict in a full LRU map (should stay 0) */
uint64_t bng_lru_evictions(bng_ctx *ctx); /* entries evicted from full LRU maps by the data path */
/* Flow-table rebuilds so far.  nat_sessions / nat_reverse / eim_table are rebuilt (tombstones dropped) together:
 *  - by bng_sweep and bng_nat_flush, once a quarter of nat_sessions' slots are tombstones after it;
 *  - once LRU evictions since the last rebuild exceed a quarter of nat_sessions' slots.  Host-fed batches and
 *    bng_sync check this with the count as of their end.  A BNG_MEM_DEVICE batch of nat44_egress / pipeline_up /
 *    pipeline_tc does not wait: it queues a copy of the count behind itself, and the next bng_prog_run or bng_sweep
 *    applies the rule to that copy if it has completed by then.  Only a rebuild synchronises the stream. */
uint64_t bng_table_rebuilds(bng_ctx *ctx);
uint64_t bng_events_lost(bng_ctx *ctx);   /* event records dropped because the staging buffer was full */
/* per-kernel device timing (CUDA events around every launch); read returns "name launches total_ms\n" lines */
int bng_prof_enable(bng_ctx *ctx, int on);
int64_t bng_prof_read(bng_ctx *ctx, char *buf, uint64_t cap);
/* Pinned, GPU-mapped host memory for BNG_MEM_HOST frame arenas: 2 MB transparent huge pages registered with
 * CUDA where possible (far fewer IOMMU translations for the GPU's scattered header reads), else cudaHostAlloc. */
void *bng_host_alloc(size_t bytes);
void bng_host_free(void *p);

#ifdef __cplusplus
}
#endif
#endif /* BNG_B200_H */
