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

/* ---- nat44_ingress: inbound ICMP errors to the subscriber whose flow they quote (RFC 5508) ----
 * nat44_ingress keys every ICMPv4 message by bytes 4-5 of its ICMP header, read as an echo id (bpf/nat44.c:846-851).
 * In an ICMP error those bytes are unused, a pointer or the next-hop MTU; the flow is named by the datagram the error
 * quotes.  on != 0: from the next bng_prog_run, nat44_ingress applies the rule below to every ICMP error frame:
 * untagged Ethernet II, ethertype 0x0800, protocol 1, ICMP type 3, 11 or 12, with the 8-byte ICMP header present (as
 * the program checks it today: bytes through 14 + ihl*4 + 7).  Such a frame is never keyed by bytes 4-5.  Offsets
 * below are for an outer header without options: ICMP header 34-41 (checksum 36-37), quoted IPv4 header 42-61
 * (protocol 51, checksum 52-53, source 54-57, destination 58-61), quoted L4 header from 62 (TCP/UDP ports 62-63 and
 * 64-65, UDP checksum 68-69, TCP checksum 78-79; ICMP checksum 64-65, id 66-67).
 *   - Translatable: outer ihl 5; quoted version 4 and ihl 5; quoted protocol 6, 17 or 1; quoted source = outer
 *     destination; and the bytes the lookup needs present ("present": min(len, the slot), as every bounds check):
 *     through 65 for TCP/UDP, 67 for ICMP.
 *   - Lookup: the nat_reverse key nat44_egress wrote for the quoted packet (bpf/nat44.c:733-739): {src_ip = quoted
 *     destination, dst_ip = quoted source, src_port = quoted destination port (0 for ICMP), dst_port = quoted source
 *     port (the quoted ICMP id, of any ICMP type), protocol}; its value is the session key, and the session gives
 *     orig_ip and orig_port.
 *   - Rewrite (csum_upd32 / csum_upd16 steps): outer destination <- orig_ip (outer IPv4 checksum); quoted source <-
 *     orig_ip (quoted IPv4 checksum); quoted source port or ICMP id <- orig_port (quoted L4 checksum: UDP only when
 *     68-69 are present and non-zero, a result of 0 becoming 0xFFFF; TCP only when 78-79 are present; ICMP always,
 *     for the id alone); and every changed word of the ICMP message into the ICMP checksum (36-37), in that order.
 *     ICMPv4 has no pseudo-header, so the outer destination is not part of it.
 *   - Outcome: verdict TC_ACT_OK, as for every nat44_ingress frame.  Translated: packets_dnat.  Not translatable, a
 *     reverse miss, or a stale reverse entry whose session is gone (the entry is NOT erased): passed unchanged,
 *     packets_passed.  The session is not refreshed (last_seen, its epoch stamp, packets_in, bytes_in and the TCP
 *     state stay): anyone on the path can forge an error, and an error must not keep a flow alive.  No other table,
 *     counter or log record changes, so an error frame's result does not depend on its place in the batch.
 *   - Everything else is as before: frames that are not ICMP error frames (types 0, 8, 4, 5 among them), and
 *     nat44_egress, whose upstream ICMP errors bng_nat_icmp_errors_egress_enable covers.  Accounting, idle detection and interception
 *     see a translated error by its new destination, the subscriber's address (captured after DNAT).
 *   - BNG_MEM_HOST with a pinned arena moves bytes 64-79 of an ICMP error frame for nat44_ingress; a fixed-stride
 *     arena of 64-byte slots (a header-split ring) does not hold the quoted ports, so its errors pass unchanged.
 * Off by default: nat44_ingress then runs exactly as before.  The flag is context state: snapshots, deltas and
 * hand-over blobs do not carry it.  Returns 0, or -EINVAL for a NULL ctx. */
int bng_nat_icmp_errors_enable(bng_ctx *ctx, int on);

/* ---- nat44_egress: subscribers' ICMP errors by the flow they quote (RFC 5508, the upstream direction) ----
 * nat44_egress keys every ICMPv4 message by bytes 4-5 of its ICMP header, read as an echo id (bpf/nat44.c:643-649).
 * A subscriber's Destination Unreachable, Time Exceeded or Parameter Problem about a frame it received then creates
 * a bogus ICMP session (a port, a nat_reverse entry, a SESSION_CREATE record), its bytes 4-5 (a pointer, the MTU) are
 * overwritten with the NAT port, and its quote still names the private address and port.  on != 0: from the next
 * bng_prog_run, wherever nat44_egress runs (standalone, pipeline_up, pipeline_tc), the rule below applies at the
 * session lookup, after the private-source check, the subscriber_nat lookup (otherwise packets_passed) and the
 * hairpin statistic, which stay as they are.  It applies to an ICMP error frame: untagged Ethernet II, ethertype
 * 0x0800, protocol 1, ICMP type 3, 11 or 12, the 8-byte ICMP header present.  Offsets as for
 * bng_nat_icmp_errors_enable: quoted IPv4 header 42-61, quoted L4 header from 62.
 *   - Translatable: outer ihl 5; quoted version 4 and ihl 5; quoted protocol 6, 17 or 1; quoted destination (58-61)
 *     = outer source (26-29), so that the quoted flow is the sending subscriber's; and the bytes the lookup needs
 *     present ("present": min(len, the slot)): through 65 for TCP/UDP, 67 for ICMP.
 *   - Lookup: one nat_sessions probe with the key nat44_egress created for the flow the quoted packet belongs to:
 *     {src_ip = quoted destination, dst_ip = quoted source, src_port = quoted destination port (64-65) or the quoted
 *     ICMP id (66-67), dst_port = quoted source port (62-63), 0 for ICMP, protocol = quoted protocol}.
 *   - Rewrite, when the session is live (csum_upd32 / csum_upd16 steps): outer source <- nat_ip (outer IPv4
 *     checksum); quoted destination <- nat_ip (quoted IPv4 checksum); quoted destination port or ICMP id <- nat_port
 *     (quoted L4 checksum: UDP only when 68-69 are present and non-zero, a result of 0 becoming 0xFFFF; TCP only when
 *     78-79 are present; ICMP always, for the id alone); and every changed word of the ICMP message into the ICMP
 *     checksum (36-37), in that order.  ICMPv4 has no pseudo-header, so the outer source is not part of it.
 *   - Outcome of a translated error: verdict TC_ACT_OK, packets_snat.  The session is not refreshed (last_seen, its
 *     epoch stamp, packets_out, bytes_out and the TCP state stay), and nothing is created: no session, nat_reverse or
 *     EIM entry, no port, no log record.
 *   - Everything else is exactly as before, keyed by bytes 4-5 (an echo-keyed session hit or created): errors that
 *     are not translatable, errors whose quoted flow has no live session, frames with outer options, types 0, 8, 4
 *     and 5, and every frame that is not ICMP.  Only the frames the rule translates change.
 *   - The rule reads the tables as the frames before it in the batch (index order) left them: a flow created, or a
 *     session evicted, by an earlier frame of the same subscriber is seen, as in sequential execution.
 *   - Accounting, idle detection and interception see an error by the source address it entered with (captured as
 *     the subscriber sent it).
 *   - BNG_MEM_HOST with a pinned arena moves bytes 64-79 of an ICMP error frame for these programs; a fixed-stride
 *     arena of 64-byte slots (a header-split ring) does not hold the quoted ports, so its errors take today's path.
 * Off by default: the programs then run exactly as before.  The flag is context state: snapshots, deltas and
 * hand-over blobs do not carry it.  Returns 0, or -EINVAL for a NULL ctx. */
int bng_nat_icmp_errors_egress_enable(bng_ctx *ctx, int on);

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
 *   - IPv6 (dual-stack subscribers): an untagged Ethernet II frame with ethertype 0x86DD whose 16 address bytes are
 *     present (source 22-37 upstream, destination 38-53 downstream) is charged to the subscriber_ipv6 owner of that
 *     address (see below), and only when its verdict is TC_ACT_OK; from there the rules here apply unchanged.  With
 *     IPv6 shaping on (bng_qos_ipv6_enable), a frame its owner's token bucket drops counts in the owner's drop pair.
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
 *   - IPv6: an untagged frame with ethertype 0x86DD whose subscriber_ipv6 owner (see below) is a target, by the same
 *     attribution as accounting's; `addr` is the owner's IPv4 address.  The bytes are copied as they are.  With IPv6
 *     shaping on (bng_qos_ipv6_enable), a frame its owner's token bucket drops is captured with TC_ACT_SHOT.
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

/* ---- incremental replication to an HA standby ----
 * The active context exports deltas: what changed in its maps since its previous export; a standby context applies
 * them in order and its maps follow the active's.  bng_snapshot / bng_restore remain the one-off hand-over.
 * bng_delta_enable(on != 0) allocates change tracking (a shadow of every hash map's slots, and of the accounting
 * records once they exist) and sets the baseline to "empty": a new random stream id, sequence 0, and the next export
 * is FULL.  on == 0 frees it.  The shadows take, per slot of each table, its key and its compared bytes as last sent,
 * rounded up to 8-byte words: 1.85 GiB at the default capacities (1e6 subscribers, 4e6 sessions, 2e6 EIM), 2.0 GiB
 * with accounting records, 32 MiB more with idle records.
 * bng_delta_export: a batch of its own, as bng_sweep is (staged upserts are applied first; it sees everything queued
 * on the context's stream).  The blob it writes:
 *   header   char magic[8] = "BNGDELT1"; uint64 stream_id, seq_from, seq_to; uint32 flags, sections  (40 bytes)
 *   sections in bng_snapshot's framing: char name[40]; uint32 kind, key_size, value_size, n_del; uint64 n_up;
 *            then n_del deleted keys, n_up upserted keys, n_up values (ABI layout).
 *   - Hash maps: the change since the previous export.  A key is deleted when the copy last sent had it and the map
 *     no longer has it in that slot; an entry is upserted when its key is new to its slot, when any byte outside the
 *     map's volatile fields differs from the copy last sent, or when its time field is more than refresh_ns past the
 *     copy last sent.  Volatile fields: nat_sessions packets_* / bytes_* (time field last_seen), eim_table (time field
 *     last_used), qos_ingress / qos_egress tokens (time field last_update).  nat_sessions' struct padding is never
 *     compared.  BNG_DELTA_EXACT compares every byte: the standby's maps become byte-identical to the active's.
 *   - Array, LPM and statistics maps: every entry, every time (n_del = 0); they replace the standby's copy.
 *   - "subscriber_acct" (kind 5, once accounting exists): the (address, struct bng_acct) records whose bytes changed.
 *   - "li_targets" (kind 6): the whole interception target set (address, target id), when it changed.
 *   - "subscriber_idle" (kind 7, once idle records exist): the (address, uint32 timeout_s) pairs whose timeout changed
 *     (see bng_idle_* below).
 *   - Event rings are not state and are never sent.
 * seq_to = seq_from + 1.  A FULL delta (BNG_DELTA_FULL, or the first export after enabling) carries every live entry
 * and no deletion.  When cap is smaller than the delta, nothing is written, *len_out is set to the size needed,
 * -ENOSPC is returned and the baseline stays where it was: the next call covers everything since that same baseline.
 * -EINVAL when tracking is not enabled.
 * bng_delta_apply: a FULL delta is always accepted; another one only when its stream id is the one applied last and
 * its seq_from is the seq_to applied last, else -ESTALE and nothing changes.  Per map, the deletions are applied
 * before the upserts; a FULL delta first clears every map it carries, the accounting records and the interception
 * targets, as bng_restore does.  Capacities may differ between the two contexts, layouts may not (-EINVAL).  When an
 * apply fails part way, the standby accepts only a FULL delta next.
 * bng_delta_info: with tracking enabled, the stream id and the sequence of the last export; otherwise those of the
 * last delta applied (0, 0: none). */
#define BNG_DELTA_FULL 1u  /* every live entry, and the applier first clears what the blob covers */
#define BNG_DELTA_EXACT 2u /* compare every byte (no volatile fields, refresh_ns ignored) */
int bng_delta_enable(bng_ctx *ctx, int on);
int bng_delta_export(bng_ctx *ctx, uint64_t refresh_ns, uint32_t flags, void *buf, uint64_t cap, uint64_t *len_out);
int bng_delta_apply(bng_ctx *ctx, const void *buf, uint64_t len);
int bng_delta_info(bng_ctx *ctx, uint64_t *stream_id, uint64_t *seq);

/* ---- subscriber hand-over between contexts (taking a GPU out of service, a CPE swap, rebalancing) ----
 * A subscriber's state lives on one context only (its shard).  bng_sub_export copies a set of subscribers' state out
 * of one context, bng_sub_import takes it into another, bit for bit; bng::shard::Router::Move (bng_shard.hpp) does
 * both and moves the routing with them.  Addresses are the 4 key bytes as subscriber_nat / qos_ingress hold them,
 * MACs the 8-byte key word of subscriber_bindings / subscriber_pools.
 * What the export selects (A: the addresses, M: the MACs):
 *   - subscriber_nat, qos_ingress, qos_egress: the entry keyed by an address in A;
 *   - nat_sessions: key src_ip in A; nat_reverse: value (the upstream nat_key) src_ip in A, stale entries included;
 *     eim_table: internal_ip in A (bng_nat_flush's predicates);
 *   - subscriber_bindings, subscriber_pools: the entry keyed by a MAC in M;
 *   - the accounting record and the whole idle record (timeout, both stamps, since_ns, flags) of every address in A
 *     that has one, and the interception target of every address in A that is one.
 * Replicated maps, statistics and event rings are not part of a subscriber and are never exported.
 * The blob: char magic[8] = "BNGMOVE1"; uint64 sections; then sections in bng_snapshot's framing: char name[40];
 * uint32 kind, key_size, value_size, pad (0); uint64 count; count keys; count values.  One section per map above (kind
 * 0, the map's ABI key / value layout); "subscriber_acct" (kind 5) once accounting records exist and "li_targets"
 * (kind 6) once interception is in use, as the snapshot defines them; "subscriber_idle_rec" (kind 8: address, struct
 * bng_idle) once idle records exist.  Entries within a section are in no particular order.
 * bng_sub_export: staged upserts are applied first and the export sees everything queued on the context's stream, as
 * bng_snapshot does.  It does not advance the batch sequence.  With BNG_SUB_DETACH, exactly the exported entries are
 * removed in the same call: no NAT log record is written and no statistic changes (nothing expired or was deleted);
 * the address maps' entries go through the ordinary delete path, so an address that loses both its subscriber_nat and
 * qos_ingress entries loses its records as a delete does.  The removal follows bng_nat_flush's flow-table rebuild rule.
 * Everything that can fail (memory, copies) happens before the blob is written, so a call that returns an error has
 * removed nothing; once the blob is written the detach completes.  Memory: the first export with addresses allocates
 * the slot lists, 4 bytes per slot of nat_sessions, nat_reverse and eim_table (80 MiB at the reference's capacities),
 * and a staging buffer that grows to the largest blob exported; both are kept until bng_close.
 * When cap is smaller than the blob, nothing is written or removed, *len_out is set to the size needed and -ENOSPC is
 * returned.  Repeated addresses or MACs, and addresses without state, are harmless.  -EINVAL for a NULL ctx or
 * len_out, a NULL array with a count > 0, a NULL buf with cap > 0, or unknown flag bits.
 * bng_sub_import: the whole blob is checked before anything changes: magic, framing and layouts (-EINVAL); room, that
 * is, for each map, its live entries plus the section's entries <= max_entries, and the interception target limit
 * (-E2BIG; deliberately conservative: an import never evicts from an LRU map).  Then every entry is inserted or
 * replaced (BNG_ANY) through bng_map_update_batch's path, after which the records go to the addresses' directory
 * slots and the targets are set (records are allocated if the context had none, as bng_restore does).  Importing a
 * blob into the context it came from restores that context exactly: the rollback of a failed hand-over.  Within one
 * host the clocks agree, so a moved subscriber keeps its idle clock (bng_restore / bng_delta_apply restart clocks).
 * Cost: the export streams the three flow tables once, one sector per slot (about 0.67 GB at the reference's
 * capacities); everything else is by key.  No batch runs anything for this. */
#define BNG_SUB_DETACH 1u /* remove what was exported, in the same call */
int bng_sub_export(bng_ctx *ctx, const uint32_t *addrs, uint64_t n_addrs, const uint64_t *macs, uint64_t n_macs,
                   uint32_t flags, void *buf, uint64_t cap, uint64_t *len_out);
int bng_sub_import(bng_ctx *ctx, const void *buf, uint64_t len);

/* ---- per-subscriber idle detection (what RADIUS Idle-Timeout, attribute 28, needs) ----
 * One record per subscriber address, with the population and lifecycle of the accounting record: an address that keys
 * a subscriber_nat or qos_ingress entry (staged upserts included).  The record starts when the address gets its entry
 * (every field none, timeout 0); it survives updates of either map, the expiry sweep, LRU eviction, flow-table
 * rebuilds and bng_nat_flush, and ends when the address loses both entries.
 *   - Stamps.  Frames are attributed to an address by accounting's rule: upstream programs (nat44_egress,
 *     qos_ingress_prog, pipeline_up, pipeline_tc) by the IPv4 source the frame entered with, downstream programs
 *     (nat44_ingress, qos_egress_prog) by the IPv4 destination it leaves with; in the two pipelines a frame antispoof
 *     drops is attributed to nobody.  Only frames with verdict TC_ACT_OK stamp: a frame the token bucket or port
 *     exhaustion drops was not carried.  The upstream stamp (up_ns) is the largest bpf_ktime_get_ns() of the stamping
 *     frames of upstream programs (now_ns_v[i], or the batch's now_ns), the downstream stamp (down_ns) the same for
 *     downstream programs.  A stamp never goes backwards.  (A clock of UINT64_MAX is stamped as UINT64_MAX - 1.)
 *   - Timeout.  timeout_s 0 means "the scan's default", BNG_IDLE_NEVER "never idle".
 *   - Scan.  bng_idle_scan(now_ns, default_s, flags) visits every record.  flags selects the stamps that count as
 *     activity (BNG_IDLE_UP and / or BNG_IDLE_DOWN).  A record that has not been started (no since_ns) is started:
 *     since_ns := now_ns, and it is not reported; so a subscriber that never sends anything is reported one timeout
 *     after the first scan that saw it, never at once.  A started record's reference time ref is the largest of its
 *     selected stamps and since_ns; it is idle when ref <= now_ns and now_ns - ref > timeout x 10^9 ns (timeout_s, or
 *     default_s when timeout_s is 0; BNG_IDLE_NEVER in either place: never idle).
 * Idle detection is enabled per program and off by default, independently of accounting.  The first
 * bng_idle_enable() or bng_idle_timeout_set() allocates the records: 32 bytes per subscriber-directory slot (64 MiB at
 * the default 1e6 subscribers), plus 4 bytes per frame of max_batch when accounting has not allocated those already.
 * A context that never uses it allocates nothing and launches no kernel more.  Before the records exist a scan finds
 * nothing and a read returns zeroed records.
 * Only the timeouts are configuration.  bng_snapshot() carries them (a trailing "subscriber_idle" section of
 * (address, uint32 timeout_s) pairs, written once records exist); bng_restore() sets them and restarts every clock
 * (stamps and since_ns cleared); a blob without the section leaves every timeout at 0.  bng_delta_export() sends a
 * "subscriber_idle" section (kind 7, once records exist) with the (address, timeout_s) pairs whose timeout changed,
 * all of them in a FULL delta; every bng_delta_apply() restarts every clock of the standby, so that no clock on the
 * standby started earlier than the last delta it applied and a takeover disconnects nobody early. */
#define BNG_IDLE_UP 1u           /* flags: up_ns holds a value; scan: count upstream activity */
#define BNG_IDLE_DOWN 2u         /* flags: down_ns holds a value; scan: count downstream activity */
#define BNG_IDLE_STARTED 4u      /* flags: since_ns holds a value */
#define BNG_IDLE_NEVER 0xFFFFFFFFu /* timeout_s: never idle */
typedef struct bng_idle {       /* 32 bytes */
    uint64_t up_ns, down_ns;    /* the stamps (0 unless the flag is set) */
    uint64_t since_ns;          /* when the first scan saw the record (0 unless BNG_IDLE_STARTED) */
    uint32_t timeout_s, flags;
} bng_idle;
/* on != 0 stamps the program's runs from the next bng_prog_run on.  -EOPNOTSUPP for antispoof_ingress,
 * nat44_hairpin_xdp and dhcp_fastpath_prog; -EINVAL for an unknown program id. */
int bng_idle_enable(bng_ctx *ctx, int prog, int on);
/* timeouts_s[i] becomes the timeout of addrs[i] (4 bytes each, in the byte order of the qos_ingress key).  results[i]
 * = 0, or -ENOENT when the address has no entry.  When an address repeats, the last of its values wins.  Staged
 * upserts are applied first.  Returns 0 or a negative errno. */
int bng_idle_timeout_set(bng_ctx *ctx, const uint32_t *addrs, const uint32_t *timeouts_s, uint64_t n, int32_t *results);
/* Records of n addresses; results[i] = 0, or -ENOENT when the address has no entry (out[i] is then zeroed).  Staged
 * upserts are applied first and the read sees everything queued on the context's stream, as bng_acct_read() does. */
int bng_idle_read(bng_ctx *ctx, const uint32_t *addrs, uint64_t n, bng_idle *out, int32_t *results);
/* The scan above.  Returns the number of idle records found and writes min(found, cap) of them, (address, record) in
 * no particular order; calling it again gives the same answer while nothing stamps.  Staged upserts are applied first
 * and the scan sees everything queued on the context's stream.  -EINVAL when flags selects neither direction or has
 * other bits, or when cap > 0 and an output is NULL. */
int64_t bng_idle_scan(bng_ctx *ctx, uint64_t now_ns, uint32_t default_s, uint32_t flags, uint32_t *addrs_out, bng_idle *out,
                      uint64_t cap);

/* ---- NAT port-usage census (port utilisation per subscriber and per public address; FEATURES.md §5, §9) ----
 * One read-only GPU pass over the NAT tables, read in ABI layout as bng_map_dump returns them.
 *   - Held triple.  Every live nat_sessions entry holds (nat_ip, ntohs(nat_port), protocol): the session's nat_port is
 *     in network order.  Every live eim_table entry holds (external_ip, external_port, key.protocol): external_port is
 *     in host order, the order of port_start / port_end.
 *   - Attributed address: a session's key src_ip, an EIM entry's key internal_ip (bng_nat_flush's attribution).
 *   - Protocol columns: [0] TCP (6), [1] UDP (17), [2] ICMP (1).  Other protocol bytes count in the totals and in
 *     *_any, in no column.
 *   - Unreachable session: a live session whose reverse key (src_ip = key.dst_ip, dst_ip = nat_ip, src_port =
 *     key.dst_port, dst_port = nat_port, protocol = the session's protocol, pad 0), as nat44_egress builds it, has no
 *     nat_reverse entry, or one whose value is not this session's key.  The reference allocator can hand out a
 *     (port, remote endpoint) pair that a live session of another internal endpoint still holds once a block wraps;
 *     the newer session then owns the reverse entry and the older one's return traffic goes to the wrong host.
 *   - Stale reverse entry: a live nat_reverse entry whose value is not the key of a live session.
 * Per-subscriber record: one per subscriber_nat entry; its block B = (public_ip, [port_start, port_end]) and
 * block_ports = port_end >= port_start ? port_end - port_start + 1 : 0.
 * Per-public-address record: one per address that is some subscriber_nat entry's block.public_ip or the public IP of
 * some held triple.  Addresses are 4 bytes in key byte order (as bng_acct_read takes them).
 * A subscriber record qualifies when permille >= min_permille (0 reports every subscriber); every public-address record
 * qualifies.  The call writes min(found, cap) records of each kind, in no particular order; calling it again with
 * nothing run in between gives the same answer.  Staged upserts are applied first and the census sees everything
 * queued on the context's stream; it returns synchronised.  It writes no map byte, counter, event, accounting, idle or
 * interception state, does not advance the batch sequence, and gives a following bng_delta_export nothing to send.
 * -EINVAL for a NULL ctx or sum, min_permille > 1000, or a cap > 0 with NULL outputs.
 * Memory: the first call allocates the census's scratch, kept until bng_close: a set of 8-byte words, the power of two
 * >= 16/3 x (max_nat_sessions + max_eim_mappings) (256 MiB at the default capacities), 32 bytes per subscriber-directory
 * slot (64 MiB at the default 1e6 subscribers), a public-address table of 48 bytes per slot (3 MiB; it grows when more
 * than 32768 public addresses are seen), and room for the records the caps ask for.  A context that never calls
 * bng_nat_usage allocates none of it and launches nothing more.
 * In a sharded deployment each shard counts its own tables: a triple held on two shards (overlapping blocks) counts
 * once per shard. */
typedef struct bng_nat_sub_use {  /* 64 bytes */
    uint64_t sessions;            /* live sessions attributed to the address */
    uint64_t eim;                 /* live EIM entries attributed to the address */
    uint32_t public_ip;           /* block.public_ip */
    uint32_t block_ports;
    uint32_t in_use[3];           /* distinct ports p in the block such that the address holds (public_ip, p, proto) */
    uint32_t in_use_any;          /* distinct ports p in the block held by the address with any protocol */
    uint32_t outside;             /* distinct triples the address holds outside B (other public IP, or port out of range) */
    uint32_t unreachable;         /* its unreachable sessions */
    uint32_t permille;            /* floor(max(in_use[0..2]) * 1000 / block_ports); 0 when block_ports == 0 */
    uint32_t pad[3];              /* zero */
} bng_nat_sub_use;
typedef struct bng_nat_pub_use {  /* 64 bytes */
    uint64_t sessions, eim;       /* live entries holding a triple on it */
    uint64_t block_ports;         /* sum of block_ports of the subscriber_nat entries whose block is on it */
    uint32_t blocks;              /* those entries */
    uint32_t in_use[3], in_use_any; /* distinct ports held on it, per protocol / any protocol */
    uint32_t unreachable;         /* unreachable sessions whose nat_ip is it */
    uint32_t pad[4];              /* zero */
} bng_nat_pub_use;
typedef struct bng_nat_usage_sum {
    uint64_t subscribers;                 /* subscriber_nat entries */
    uint64_t sessions, eim, triples;      /* live entries; distinct held triples */
    uint64_t unreachable, stale_reverse;
    uint64_t orphan_sessions, orphan_eim; /* attributed to an address without a subscriber_nat entry (released, not flushed) */
    uint64_t subs_found, pubs_found;      /* records that qualified (may exceed the caps) */
} bng_nat_usage_sum;
int bng_nat_usage(bng_ctx *ctx, uint32_t min_permille, bng_nat_usage_sum *sum, uint32_t *sub_addrs, bng_nat_sub_use *sub_out,
                  uint64_t sub_cap, uint32_t *pub_addrs, bng_nat_pub_use *pub_out, uint64_t pub_cap);

/* ---- DHCP lease census and expiry sweep ----
 * dhcp_fastpath_prog finds a subscriber's pool_assignment by VLAN pair, then circuit-id, then chaddr, takes the first
 * entry it finds and sends the frame to the slow path when that entry has expired, even if a fresh one exists further
 * down the chain.  The three lease maps (map index 0 subscriber_pools, 1 vlan_subscriber_pools, 2
 * circuit_id_subscribers) live only on the GPU, so finding and removing their expired entries, and counting what the
 * pools hold, are GPU passes.
 *   - Expired at now_ns is exactly the program's test: now_ns / 1000000000 > lease_expiry.  An entry the program would
 *     still serve at now_ns is unexpired.
 *   - Byte order.  Two conventions fill these maps.  The control plane (the reference's Go loader, whose IPToUint32 is
 *     BigEndian.Uint32 stored in a native word, and its C++ mirror in bng_host.hpp / bng_dhcp_slow.hpp) stores the
 *     address's numeric value: BNG_LEASE_ADDR_NUMERIC, the default, and the order in which dhcp::Pool takes an address
 *     back.  The program itself copies allocated_ip into yiaddr and builds the subnet mask with htonl, so tables whose
 *     replies must be right on the wire (the synthetic workloads and the test scripts) hold the four bytes in wire
 *     order: BNG_LEASE_ADDR_WIRE.  bng_dhcp_lease_addr_order tells the context which one its control plane uses; the
 *     census compares the leading prefix_len bits of allocated_ip and ip_pool.network in that order.  Only
 *     addrs_outside and permille depend on it: the two fields always share one convention, and distinct counts and
 *     conflicts compare words.  prefix_len 0 contains every address, 32 only `network`, a prefix_len > 32 none.
 *     Records of removed entries carry allocated_ip as stored.
 *
 * bng_dhcp_lease_census: read-only.  One record for every pool_id that keys an ip_pools entry or is named by any lease
 * entry, expired or not.
 *   - Conflict: an address counts once in `conflicts` of pool P when, within one of the three maps, two or more
 *     unexpired entries naming P hold it (the keys of a map are distinct, so those are two subscribers).  The same
 *     subscriber appearing in different maps is not a conflict, and expired entries never conflict: their address may
 *     have been leased again.
 *   - The call writes min(pools_found, cap) records in no particular order; calling it again with nothing run in
 *     between gives the same answer.  Staged upserts are applied first and the census sees everything queued on the
 *     context's stream; it returns synchronised.  It writes no map byte, counter, event, accounting, idle or
 *     interception state, does not advance the batch sequence, and gives a following bng_delta_export nothing to send.
 *   - -EINVAL for a NULL ctx or sum, or a cap > 0 with NULL outputs.
 *   - Memory: the first call allocates the census's scratch, kept until bng_close: a set of 8-byte words, the power of
 *     two >= 4 x the summed max_entries of the three lease maps (128 MiB at the default capacities), 64 bytes per ip_pools
 *     slot and per slot of the hash of unknown pool_ids (3 MiB; the hash grows, and the census counts again, once
 *     8192 distinct unknown pool_ids have records), and room for the records.  A context that calls neither function allocates none of it.
 *   - In a sharded deployment each shard counts its own tables: an address leased on two shards counts once per shard.
 *
 * bng_dhcp_lease_sweep: removes.  An entry of the three lease maps is due when
 * now_ns / 1000000000 > lease_expiry + grace_s (the sum saturates); with grace_s == 0 that is every entry the program
 * refuses.
 *   - Returns the number of due entries found (or a negative errno).  It removes, and reports in `out`, at most `cap` of
 *     them; which ones when there are more is unspecified, but every removed entry is reported exactly once and every
 *     reported entry is removed.  cap == 0 removes nothing (a dry run; `out` may be NULL).  Repeat the call until the
 *     return value is <= cap.
 *   - circuit_id_map (fnv hash of the circuit-id -> MAC): an entry whose value MAC keys a subscriber_pools entry that
 *     this call removes is removed with it, and no other.
 *   - removed_out (may be NULL): entries removed from map 0, 1, 2 and from circuit_id_map.
 *   - Nothing else changes: not stats_map (cache_expired is the program's counter), not ip_pools, no NAT / QoS map.
 *     bng_map_get_info().count of the four maps drops by what was removed and a later insert finds the room.
 *   - Staged upserts are applied first; the sweep is a batch of its own (it advances the batch sequence) and returns
 *     synchronised.  The removed keys are deletions of the next bng_delta_export.
 *   - Afterwards each of the four tables of which more than a quarter of the slots are tombstones is rebuilt.  These
 *     rebuilds are counted by bng_lease_table_rebuilds, not by bng_table_rebuilds.  A dry run rebuilds nothing.  A
 *     rebuild that finds no memory leaves its table as it was; the call still returns what it removed
 *     (bng_last_error has the text) and the next sweep tries again.
 *   - -EINVAL for a NULL ctx, or cap > 0 with a NULL out. */
typedef struct bng_lease_pool_use { /* 64 bytes; one per pool_id seen */
    uint64_t entries[3];     /* unexpired entries naming the pool, per map */
    uint64_t expired;        /* expired entries naming the pool, the three maps together */
    uint32_t addrs;          /* distinct allocated_ip among its unexpired entries */
    uint32_t addrs_outside;  /* of those, the ones not inside network/prefix_len (all of them when no ip_pools entry) */
    uint32_t conflicts;
    uint32_t prefix_hosts;   /* 2^(32 - prefix_len), saturated at 2^32-1; 0 when prefix_len > 32 or no ip_pools entry */
    uint32_t permille;       /* floor((addrs - addrs_outside) * 1000 / prefix_hosts), 0 when prefix_hosts == 0 */
    uint8_t known;           /* 1 when ip_pools has the pool_id */
    uint8_t pad[11];         /* zero */
} bng_lease_pool_use;
typedef struct bng_lease_sum {
    uint64_t entries[3], expired[3]; /* per map, unexpired / expired */
    uint64_t addrs;                  /* distinct allocated_ip over all unexpired entries */
    uint64_t conflicts;              /* summed over pools */
    uint64_t unknown_pool;           /* unexpired entries whose pool_id has no ip_pools entry (the program counts these as errors) */
    uint64_t cid_dangling;           /* circuit_id_map entries whose value MAC keys no subscriber_pools entry */
    uint64_t pools_found;            /* records that exist (may exceed cap) */
} bng_lease_sum;
int bng_dhcp_lease_census(bng_ctx *ctx, uint64_t now_ns, bng_lease_sum *sum, uint32_t *pool_ids, bng_lease_pool_use *out,
                          uint64_t cap);
typedef struct bng_lease_removed { /* 64 bytes */
    uint8_t key[32];         /* the entry's key, zero-padded: 8-byte MAC word, 4-byte vlan_key, or 32-byte circuit-id */
    uint64_t lease_expiry;
    uint32_t pool_id, allocated_ip, vlan_id;
    uint8_t map;             /* 0 subscriber_pools, 1 vlan_subscriber_pools, 2 circuit_id_subscribers */
    uint8_t client_class, flags;
    uint8_t pad[9];          /* zero */
} bng_lease_removed;
int64_t bng_dhcp_lease_sweep(bng_ctx *ctx, uint64_t now_ns, uint32_t grace_s, bng_lease_removed *out, uint64_t cap,
                             uint64_t removed_out[4]);
#define BNG_LEASE_ADDR_NUMERIC 0u
#define BNG_LEASE_ADDR_WIRE 1u
int bng_dhcp_lease_addr_order(bng_ctx *ctx, uint32_t order); /* -EINVAL for a NULL ctx or another value */
uint64_t bng_lease_table_rebuilds(bng_ctx *ctx); /* rebuilds of the three lease maps and circuit_id_map by the sweep */

/* ---- dual-stack subscribers: the IPv6 prefix table (not one of the reference's maps) ----
 * "subscriber_ipv6" (bng_map_id) maps a subscriber's IPv6 address or prefix (Framed-IPv6-Prefix, Delegated-IPv6-Prefix)
 * to its IPv4 address, the 4 key bytes of qos_ingress.  It is an ordinary map of the registry: bng_map_update, _batch,
 * _staged, _delete, _dump, _clear, snapshots, restore and deltas carry it.  Reported type BPF_MAP_TYPE_LPM_TRIE (11),
 * key struct bng_ipv6_prefix_key (20 bytes), value uint32_t, max_entries 2 x max_subscribers (a WAN /64 or /128 and a
 * delegated prefix per subscriber).
 *   - prefixlen > 128: -EINVAL (update, staged update, delete, lookup).
 *   - Update and delete match exactly on (prefixlen, prefix).  Bits of addr past prefixlen are masked off on the way in,
 *     so two keys that differ only there are one entry, as in the kernel's trie.  Dumps return the masked key, where
 *     the kernel's trie returns what the caller wrote.
 *   - bng_map_lookup is the trie's lookup: the value of the longest prefix of length <= key.prefixlen that covers
 *     key.addr ("whose address is this?"), -ENOENT when none does.
 * The rule every feature that attributes frames uses (accounting, idle detection, lawful intercept, hand-over): an
 * untagged Ethernet II frame with ethertype 0x86DD whose 16 address bytes are present in the frame's storage (source
 * at 22-37 upstream, destination at 38-53 downstream) belongs to the value of the longest prefix in subscriber_ipv6
 * that covers that address; the IPv4 rule then applies to that address unchanged (its directory entry, its record,
 * its target).  No covering prefix (a link-local source, say): nobody.  Tagged IPv6 frames: nobody, as tagged IPv4.
 * Without IPv6 shaping (below), no program here drops an IPv6 frame except antispoof_ingress (NAT and QoS pass
 * non-IPv4 frames), so an IPv6 frame with verdict TC_ACT_SHOT is an antispoof drop, and an IPv6 frame is attributed
 * only when its verdict is TC_ACT_OK.  With shaping on, a frame the owner's token bucket drops is attributed as well
 * (TC_ACT_SHOT, the drop pair); a frame antispoof drops is still nobody's.
 * While the table is empty, every record and every launch is what it is without it: the IPv6 variants of the
 * attribution kernels run only while the table has live entries.  bng_sub_export carries the entries whose value is
 * an exported address, in a "subscriber_ipv6" section written only when there is one; BNG_SUB_DETACH removes them.
 * Memory: 32 bytes per slot of a power of two >= 4 x max_subscribers (128 MiB at the default 1e6), and with change
 * tracking a shadow of the same size. */
typedef struct bng_ipv6_prefix_key {
    uint32_t prefixlen; /* 0..128 */
    uint8_t addr[16];   /* network order */
} bng_ipv6_prefix_key;
/* IPv6 shaping: one token bucket per subscriber, whatever the address family.  on != 0: from the next bng_prog_run,
 * qos_ingress_prog, pipeline_up and pipeline_tc shape an IPv6 frame with the qos_ingress bucket of the subscriber_ipv6
 * owner of its source (bytes 22-37), and qos_egress_prog with the qos_egress bucket of the owner of its destination
 * (38-53).  Which frames: those the rule above attributes (untagged, ethertype 0x86DD, the 16 address bytes present,
 * a covering prefix); in the pipelines only those antispoof_ingress passed.
 *   - The frame is shaped exactly as an IPv4 frame of the same len from the owner (ingress) or to it (egress), at the
 *     same clock and the same position in the batch, would be: token_bucket_check() runs in index order together with
 *     the owner's IPv4 frames, an unlimited bucket passes it, qos_stats_map counts it, and a frame qos_egress_prog
 *     passes gets the bucket's priority.  Its bytes are not changed.
 *   - Nothing else that happens to an IPv6 frame changes: NAT passes it untouched and uncounted (in pipeline_tc too,
 *     where NAT runs after the bucket); nat44_*, antispoof_ingress and dhcp_fastpath_prog are not affected.  Frames
 *     without an owner, tagged frames and frames too short for the address are not shaped.
 *   - Accounting, idle detection and interception see a bucket drop as they see an IPv4 one (above).
 *   - While subscriber_ipv6 is empty, "on" launches exactly what "off" launches.
 * Off by default.  The flag is context state: snapshots, deltas and hand-over blobs do not carry it, so a standby or
 * the destination of a hand-over sets it itself.  Returns 0, or -EINVAL for a NULL ctx. */
int bng_qos_ipv6_enable(bng_ctx *ctx, int on);
/* Antispoof by delegated prefix: a subscriber's own subscriber_ipv6 prefixes count as its IPv6 addresses.  on != 0:
 * from the next bng_prog_run, antispoof_ingress (standalone, and its stage in pipeline_up and pipeline_tc) allows an
 * IPv6 frame that the reference would drop when all of these hold:
 *   - the frame reaches the reference's IPv6 drop: untagged, ethertype 0x86DD at bytes 12-13, at least 54 bytes
 *     present, mode neither disabled nor log-only, not allowed by the exact match with ipv6_addr or by loose mode;
 *   - the source MAC has a subscriber_bindings entry with ipv4_valid set;
 *   - the longest prefix in subscriber_ipv6 that covers the source address (bytes 22-37) has the binding's ipv4_addr
 *     as its value (the same 4 bytes the IPv4 branch compares with saddr).
 * Such a frame gets TC_ACT_OK and adds 1 to packets_allowed, and nothing else: no spoof event, no packets_logged,
 * packets_dropped or ipv6_violations.  From there it is an ordinary passed IPv6 frame: NAT passes it untouched, QoS
 * passes it (or shapes it with its owner's bucket, bng_qos_ipv6_enable), and accounting, idle detection and
 * interception attribute it by the rule above.  Every other frame is unchanged: a source whose longest covering prefix
 * belongs to another subscriber (a longer prefix nested in the binding's own, say), unbound MACs, bindings without
 * ipv4_valid, tagged and short frames, every non-IPv6 frame.
 * While subscriber_ipv6 is empty, "on" launches exactly what "off" launches.  Off by default.  The flag is context
 * state: snapshots, deltas and hand-over blobs do not carry it, so a standby or the destination of a hand-over sets
 * it itself.  Returns 0, or -EINVAL for a NULL ctx. */
int bng_antispoof_ipv6_prefixes_enable(bng_ctx *ctx, int on);

/* ---- DHCPv6 fast path (not one of the reference's maps or programs) ----
 * The DHCPv6 server (pkg/dhcpv6) caches each bound client's answer here, and dhcp_fastpath_prog answers a bound
 * client's Solicit, Request, Renew and Rebind on the GPU with what the server would send.  Three registry maps, carried
 * by every generic path (update, batch, staged, delete, dump, clear, snapshot, restore, deltas); none is carried by
 * bng_sub_export, so a moved client's messages pass to the slow path on the destination until it binds again.
 *   - "dhcpv6_bindings": BPF_MAP_TYPE_HASH, key struct bng_dhcpv6_client_key (32 B), value struct bng_dhcpv6_binding
 *     (64 B), max_entries = max_subscribers.  An update (plain, batch or staged) returns -EINVAL, and a batch applies
 *     none of its entries, when duid_len is 0 or > 31, a key byte past duid_len is non-zero, flags has bits other than
 *     NA | PD or neither, PD is set with pd_len 0 or > 128, or prefix has bits set past pd_len.
 *   - "dhcpv6_server_config": BPF_MAP_TYPE_ARRAY, one struct bng_dhcpv6_server_config (96 B).  duid_len 0 means
 *     unconfigured; duid_len > 32 or dns_count > 2 returns -EINVAL.
 *   - "dhcpv6_stats": BPF_MAP_TYPE_ARRAY, one entry of BNG_DHCPV6_NUM_STATS u64 counters (the BNG_DHCPV6_ST_* order).
 *     They follow the BNG_NUM_STATS counters of the packed statistics vector in the same device buffer
 *     (bng_stats_device_ptr still reports BNG_NUM_STATS), and bng_sync_reduce all-reduces them with the others;
 *     totals_out keeps its BNG_NUM_STATS entries.
 * bng_dhcpv6_enable(ctx, on): on != 0 applies the rule below from the next bng_prog_run of dhcp_fastpath_prog; DHCPv4
 * frames and every other program are unchanged.  Off by default; -EINVAL for a NULL ctx.  The flag is context state:
 * snapshots, deltas and hand-over blobs do not carry it.  While dhcpv6_bindings is empty or the server is
 * unconfigured, "on" launches exactly what "off" launches and counts nothing.
 * The rule.  Bytes are "present" as far as frame_dlen goes: min(len, stride) in a fixed-stride arena, len with an
 * offset table.  A frame that dhcp_one has found not to be IPv4 (stats_map counts it as it always did, vlan_packets
 * included) is a DHCPv6 candidate when it is untagged or carries one or two tags parsed as for DHCPv4 (0x8100 / 0x88A8,
 * then an inner 0x8100), its ethertype is 0x86DD, the 40-byte IPv6 header is present with version 6 and next header 17,
 * the UDP header is present with destination port 547, and the IPv6 destination is ff02::1:2 or server_ip.  For a
 * candidate, total += 1; the first of these that applies passes it (XDP_PASS, frame untouched, one counter):
 *   1. server unconfigured or len > 448: unsupported; UDP length < 12 or past the bytes present: malformed;
 *   2. message type not Solicit (1), Request (3), Renew (5) or Rebind (6): unsupported; otherwise the type's own
 *      counter also counts, whatever follows;
 *   3. the option walk from message byte 4 to the UDP end finds an option running past the end, or more than 32
 *      options: malformed;
 *   4. unsupported: not exactly one Client ID of 1-31 bytes; an IA_TA; more than one IA_NA or IA_PD; an IA_NA or IA_PD
 *      shorter than 12 bytes; neither IA_NA nor IA_PD; a Server ID on a Solicit or Rebind; a Request or Renew without
 *      exactly one Server ID byte-equal to (duid, duid_len);
 *   5. no dhcpv6_bindings entry for the Client ID, or its mac is not the Ethernet source: miss;
 *   6. now_s > expires_s (now_s = the frame's clock / 1e9, as DHCPv4's lease_expiry): expired;
 *   7. an IA_NA while the binding lacks NA or has another iaid_na, or the same for IA_PD: unsupported;
 *   8. the reply does not fit the frame's storage (stride in a fixed-stride arena, len rounded up to 16 with an offset
 *      table): no_room.
 * Otherwise the frame is answered in place: XDP_TX, len = the reply's length, advertise or reply += 1.  Ethernet dst =
 * the request's source, src = server_mac, tags as they were; IPv6 0x60000000, payload length, next header 17, hop
 * limit 64, src = server_ip, dst = the request's source; UDP 547 -> 546, its length and its checksum (0 sent as
 * 0xFFFF); the message: type, the transaction id, then Client ID (copied), Server ID, Preference 255 (Advertise
 * only), IA_NA {IAID, T1, T2, IAADDR {addr, preferred, valid}} if requested, IA_PD {IAID, T1, T2, IAPREFIX {preferred,
 * valid, pd_len, prefix}} if requested, DNS servers (23) when dns_count > 0, Status Code {0, "Success"} (Reply only),
 * Rapid Commit (a Solicit answered with a Reply).  The bytes from the reply's end to the next multiple of 16 (counted
 * from the frame's start) are zeroed; every other byte of the frame's storage is unchanged.  A Solicit with Rapid Commit gets a Reply, any other Solicit an
 * Advertise, the other three types a Reply.  T1 = preferred / 2, T2 = preferred * 4 / 5 in 32-bit unsigned arithmetic.
 * The request's UDP checksum is not verified.  The program writes no table, and no frame's outcome depends on another,
 * so the rule holds frame by frame, wherever the frame sits in the batch. */
#define BNG_DHCPV6_NA 1
#define BNG_DHCPV6_PD 2
#define BNG_DHCPV6_NUM_STATS 12
enum {
    BNG_DHCPV6_ST_TOTAL, BNG_DHCPV6_ST_SOLICIT, BNG_DHCPV6_ST_REQUEST, BNG_DHCPV6_ST_RENEW, BNG_DHCPV6_ST_REBIND,
    BNG_DHCPV6_ST_ADVERTISE, BNG_DHCPV6_ST_REPLY, BNG_DHCPV6_ST_MISS, BNG_DHCPV6_ST_EXPIRED, BNG_DHCPV6_ST_UNSUPPORTED,
    BNG_DHCPV6_ST_NO_ROOM, BNG_DHCPV6_ST_MALFORMED
};
typedef struct bng_dhcpv6_client_key {
    uint8_t duid_len; /* 1..31 */
    uint8_t duid[31]; /* the Client Identifier option's data, zero past duid_len */
} bng_dhcpv6_client_key;
typedef struct bng_dhcpv6_binding {
    uint8_t mac[6];         /* the client's Ethernet address: the request's source must equal it */
    uint8_t flags;          /* BNG_DHCPV6_NA | BNG_DHCPV6_PD */
    uint8_t pd_len;         /* 1..128 with PD */
    uint32_t iaid_na;       /* host order */
    uint32_t iaid_pd;
    uint32_t preferred_lft; /* seconds */
    uint32_t valid_lft;
    uint64_t expires_s;     /* compared with the frame's clock / 1e9 */
    uint8_t addr[16];       /* IA_NA address, network order */
    uint8_t prefix[16];     /* IA_PD prefix, zero past pd_len */
} bng_dhcpv6_binding;
typedef struct bng_dhcpv6_server_config {
    uint8_t server_mac[6];
    uint8_t duid_len;       /* 0 = unconfigured, at most 32 */
    uint8_t dns_count;      /* 0..2 */
    uint8_t server_ip[16];  /* the reply's source, normally link-local */
    uint8_t duid[32];       /* the Server Identifier option's data */
    uint8_t dns[2][16];
    uint8_t _pad[8];
} bng_dhcpv6_server_config;
int bng_dhcpv6_enable(bng_ctx *ctx, int on);

/* ---- Router and Neighbor Solicitations (not one of the reference's maps or programs) ----
 * dhcp_fastpath_prog answers a subscriber's IPv6 Router Solicitation with a Router Advertisement of its own (the
 * shared options pkg/slaac's buildRA would send, plus the subscriber's own Prefix Information option), and a Neighbor
 * Solicitation for the router's link-local address with a Neighbor Advertisement, on the GPU.  Three registry maps,
 * carried by every generic path (update, batch, staged, delete, dump, clear, snapshot, restore, deltas):
 *   - "nd_config": BPF_MAP_TYPE_ARRAY, one struct bng_nd_config (320 B).  ra[0, ra_head_len) is the RA message from its
 *     type byte through the options that precede the per-subscriber prefix (RA header, Source Link-Layer Address, MTU,
 *     the shared Prefix Information options); ra[ra_head_len, ra_head_len + ra_tail_len) the options that follow it
 *     (RDNSS, DNSSL): buildRA's order, split where the subscriber's prefix goes.  ra_head_len 0 means unconfigured, and
 *     then every byte past router_mac must be 0.  Otherwise an update returns -EINVAL unless ra_head_len >= 16 and a
 *     multiple of 8, ra_tail_len a multiple of 8, head + tail <= 288, ra[0] = 134, ra[1] = 0, ra[2] = ra[3] = 0, each
 *     part's option walk (length byte >= 1, in units of 8 bytes) ends exactly at the part's end, router_ll is in
 *     fe80::/10, router_mac is a non-zero unicast address, and ra's bytes past head + tail are 0.  The GPU copies the
 *     template; it does not interpret it.
 *   - "nd_bindings": BPF_MAP_TYPE_HASH, key the 8-byte MAC word of subscriber_bindings, value struct bng_nd_binding
 *     (48 B), max_entries = max_subscribers.  prefix_len 0: no per-subscriber prefix (a DHCPv6-managed subscriber still
 *     gets its default route).  An update (plain, batch or staged) returns -EINVAL, and a batch applies none of its
 *     entries, when prefix_len > 128, prefix has bits set past prefix_len, prefix_len is 0 with a non-zero prefix or
 *     pio_flags, pio_flags has bits other than L (0x80) and A (0x40), or a pad byte is non-zero.
 *   - "nd_stats": BPF_MAP_TYPE_ARRAY, one entry of BNG_ND_NUM_STATS u64 counters (the BNG_ND_ST_* order), stored after
 *     dhcpv6_stats in the same device buffer; bng_sync_reduce all-reduces them.  bng_stats_device_ptr's count and
 *     totals_out are unchanged.
 * bng_sub_export carries the nd_bindings entries keyed by a MAC it is given, in an "nd_bindings" section written only
 * when there is one; BNG_SUB_DETACH removes them and bng_sub_import inserts them.
 * bng_nd_enable(ctx, on): on != 0 applies the rule below from the next bng_prog_run of dhcp_fastpath_prog; every other
 * frame and program is unchanged.  Off by default; -EINVAL for a NULL ctx.  The flag is context state: snapshots,
 * deltas and hand-over blobs do not carry it.  While nd_config is unconfigured, "on" launches exactly what "off"
 * launches and counts nothing.
 * The rule.  Bytes are "present" as far as frame_dlen goes, as for DHCPv6.  A frame that dhcp_one has found not to be
 * IPv4 and that the DHCPv6 rule did not take (it needs next header 17) is a candidate when it is untagged or carries
 * one or two tags parsed as for DHCPv4 and DHCPv6, its ethertype is 0x86DD, the 40-byte IPv6 header is present with
 * version 6 and next header 58 (no extension headers), the first ICMPv6 byte is present, and it is a Router
 * Solicitation (133) to ff02::2 or router_ll, or a Neighbor Solicitation (135) to router_ll or to router_ll's
 * solicited-node address ff02::1:ffXX:XXXX.  Every other frame is untouched and counted nowhere new; stats_map counts
 * every frame as it always did.  For a candidate, total += 1; the first of these that applies passes it (XDP_PASS,
 * frame untouched, one counter):
 *   1. unconfigured or len > 448: unsupported; payload length < 8 (RS) or < 24 (NS), or 40 + payload length past the
 *      bytes present: malformed;
 *   2. (from here on rs or ns also counts, whatever follows)
 *   3. malformed (RFC 4861 §6.1.1, §7.1.1): hop limit != 255; ICMP code != 0; the ICMPv6 checksum over the
 *      pseudo-header and payload length bytes does not sum to 0xFFFF; an option (after the 8-byte RS or 24-byte NS
 *      body) of length 0 or running past the payload's end; more than 32 options; an unspecified (::) source with a
 *      Source Link-Layer Address option; for NS, a multicast target, or an unspecified source sent to router_ll
 *      rather than to its solicited-node address;
 *   4. NS whose target is not router_ll: not_target (a subscriber's own duplicate address detection lands here);
 *   5. RS with no nd_bindings entry for the Ethernet source: miss; RS with now_s > expires_s (now_s = the frame's
 *      clock / 1e9): expired;
 *   6. the reply does not fit the frame's storage (the stride, or len rounded up to 16 with an offset table): no_room.
 * Otherwise the frame is answered in place: XDP_TX, len = the reply's length, ra or na += 1.  Ethernet dst = the
 * request's source, src = router_mac, tags as they were; IPv6 0x60000000, payload length, next header 58, hop limit
 * 255, src = router_ll, dst = the request's source, or ff02::1 when that is ::.  An RA is the template's head, then,
 * when prefix_len > 0, the binding's Prefix Information option {3, 4, prefix_len, pio_flags, valid_lft,
 * preferred_lft, 0, prefix}, then the template's tail, with the ICMPv6 checksum.  An NA is 32 bytes of ICMPv6: type
 * 136, code 0, the checksum, flags R|S|O (0xE0), or R|O (0xA0) when the source is ::, three zero bytes, target =
 * router_ll, and the Target Link-Layer Address option {2, 1, router_mac}.  The bytes from the reply's end to the next
 * multiple of 16 (counted from the frame's start) are zeroed; every other byte of the frame's storage is unchanged.
 * NS answers need no binding: they name only the router's own address.  The program writes no table, and no frame's
 * outcome depends on another, so the rule holds frame by frame, wherever the frame sits in the batch.  The largest
 * reply is 22 + 40 + 288 + 32 = 382 bytes. */
#define BNG_ND_PIO_L 0x80
#define BNG_ND_PIO_A 0x40
#define BNG_ND_NUM_STATS 11
enum {
    BNG_ND_ST_TOTAL, BNG_ND_ST_RS, BNG_ND_ST_NS, BNG_ND_ST_RA, BNG_ND_ST_NA, BNG_ND_ST_MISS, BNG_ND_ST_EXPIRED,
    BNG_ND_ST_NOT_TARGET, BNG_ND_ST_MALFORMED, BNG_ND_ST_UNSUPPORTED, BNG_ND_ST_NO_ROOM
};
typedef struct bng_nd_config {
    uint8_t router_mac[6];   /* the replies' Ethernet source and Target Link-Layer Address */
    uint8_t _pad0[2];
    uint16_t ra_head_len;    /* 0 = unconfigured */
    uint16_t ra_tail_len;
    uint8_t _pad1[4];
    uint8_t router_ll[16];   /* the router's link-local address: the replies' source, the NS target answered */
    uint8_t ra[288];         /* head, then tail; the checksum bytes 0 */
} bng_nd_config;
typedef struct bng_nd_binding {
    uint8_t prefix[16];      /* network order, zero past prefix_len */
    uint8_t prefix_len;      /* 0 = no per-subscriber prefix */
    uint8_t pio_flags;       /* BNG_ND_PIO_L | BNG_ND_PIO_A */
    uint8_t _pad0[2];
    uint32_t valid_lft;      /* seconds, host order */
    uint32_t preferred_lft;
    uint8_t _pad1[4];
    uint64_t expires_s;      /* compared with the frame's clock / 1e9 */
    uint8_t _pad2[8];
} bng_nd_binding;
int bng_nd_enable(bng_ctx *ctx, int on);

/* ---- diagnostics ---- */
uint64_t bng_launch_count(bng_ctx *ctx);  /* kernels launched by this context so far */
/* Live subscriber_ipv6 entries per prefix length, counts[0..128]: the lengths the IPv6 lookup probes are those with a
 * non-zero count.  Staged upserts are applied first. */
int bng_ipv6_prefix_lengths(bng_ctx *ctx, uint32_t *counts /* [129] */);
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
