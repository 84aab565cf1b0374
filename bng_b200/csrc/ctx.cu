// bng_b200 — C-ABI layer (include/bng_b200.h): context, map registry with the
// reference's map names / key / value layouts, control-plane map commands,
// batch program runs, event drain.  Everything that touches table or frame
// contents is a CUDA kernel; this file only moves bytes and launches.
#include <errno.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
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
    // staging for control-plane commands
    u8 *io_dev = nullptr;
    u8 *io_host = nullptr; // pinned
    size_t io_bytes = 0;
    // staging for BNG_MEM_HOST batches
    u8 *hb_pkts = nullptr;
    u32 *hb_off = nullptr, *hb_len = nullptr, *hb_prio = nullptr;
    u64 *hb_now = nullptr;
    u64 *zc_now[ZC_BUFS] = {};
    u8 *hb_verdict = nullptr;
    size_t hb_arena = 0;
    u32 hb_n = 0;
    u64 lost_base[2] = {0, 0};
    // zero-copy pipeline for BNG_MEM_HOST batches in pinned memory: two chunk buffers, three streams
    cudaStream_t s_in = nullptr, s_out = nullptr;
    cudaEvent_t ev_in[ZC_BUFS] = {}, ev_comp[ZC_BUFS] = {}, ev_out[ZC_BUFS] = {};
    u8 *zc_hdr[ZC_BUFS] = {}, *zc_verdict[ZC_BUFS] = {};
    u32 *zc_off[ZC_BUFS] = {}, *zc_len[ZC_BUFS] = {}, *zc_len0[ZC_BUFS] = {}, *zc_prio[ZC_BUFS] = {};
    u32 zc_hb = 0;
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
    u64 *evict_word = nullptr; // pinned
    cudaEvent_t evict_ev = nullptr;
    bool evict_pending = false;
    bool small_dirty = false; // a map feeding the SmallTabs image changed since the image was built
    // grow-only scratch of map dumps (no cudaMalloc / cudaFree per call)
    u8 *dump_k = nullptr, *dump_v = nullptr;
    u32 *dump_c = nullptr;
    size_t dump_kb = 0, dump_vb = 0;
    // multi-GPU reconciliation (bng_comm_init / bng_sync_reduce)
    ncclComm_t comm = nullptr;
    u32 comm_rank = 0, comm_world = 1;
    u64 *stats_global = nullptr; // device: all-reduced counter vector
    // per-subscriber traffic accounting (bng_acct_*): records index-aligned with the subscriber directory, allocated
    // by the first bng_acct_enable (or a restore that carries records); acct_progs: bit p = program p is accounted
    u64 *acct = nullptr;
    u32 acct_progs = 0;
    u8 *acct_dump_buf = nullptr; // grow-only scratch of bng_acct_dump: records, then addresses
    u64 acct_dump_cap = 0;
    u64 seq = 0; // the batch sequence in 64 bits (dev.batch_seq holds its low 32): bng_li_record.batch
    // lawful intercept (bng_li_*, li.cu): allocated by the first bng_li_configure / bng_li_target_set (li_ctl != null)
    u64 *li_ctl = nullptr;   // device: LiRing::ctl
    u64 *li_words = nullptr; // device: the target set (AddrSet words, LI_TSLOTS), and its ids
    u32 *li_ids = nullptr;
    u32 li_mask = 0;
    bool li_dirty = false;   // the host's targets changed since the device copy was made
    std::unordered_map<u32, u32> li_targets; // authoritative: address -> target id
    u8 *li_ring = nullptr;
    u32 li_cap = 0, li_rec = 0, li_snap = 0;
    uint2 *li_match = nullptr; // [L.s.cap]
    std::vector<u8> li_pending; // records copied out of the ring, ordered, not yet drained
    u64 li_lost_host = 0;       // records discarded by a reconfiguration
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

int ensure_scratch(bng_ctx *c, u32 n) {
    Scratch &s = c->L.s;
    if (n <= s.cap) return 0;
    u32 cap = std::max<u32>(n, 1024);
    void **ptrs[] = {(void **)&s.key_a, (void **)&s.key_b, (void **)&s.val_a, (void **)&s.val_b, (void **)&s.qslot, (void **)&s.attr};
    for (void **pp : ptrs) {
        if (pp == (void **)&s.attr && !c->acct && !c->li_ctl) continue; // the attribution words exist once accounting or interception does
        if (*pp) cudaFree(*pp);
        CU(c, cudaMalloc(pp, (size_t)cap * 4));
    }
    if (c->li_ctl) {
        if (c->li_match) cudaFree(c->li_match);
        CU(c, cudaMalloc((void **)&c->li_match, (size_t)cap * sizeof(uint2)));
    }
    if (s.cub_tmp) cudaFree(s.cub_tmp);
    s.cub_tmp_bytes = sort_temp_bytes(cap);
    CU(c, cudaMalloc(&s.cub_tmp, s.cub_tmp_bytes ? s.cub_tmp_bytes : 16));
    s.cap = cap;
    return 0;
}

int ensure_io(bng_ctx *c, size_t bytes) {
    if (bytes <= c->io_bytes) return 0;
    size_t nb = std::max<size_t>(bytes, 1 << 20);
    if (c->io_dev) cudaFree(c->io_dev);
    if (c->io_host) cudaFreeHost(c->io_host);
    c->io_dev = nullptr;
    c->io_host = nullptr;
    c->io_bytes = 0;
    CU(c, cudaMalloc((void **)&c->io_dev, nb));
    CU(c, cudaMallocHost((void **)&c->io_host, nb));
    c->io_bytes = nb;
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
                           role, c->acct));
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
        Scratch &s = c->L.s;
        void *sp[] = {s.key_a, s.key_b, s.val_a, s.val_b, s.qslot, s.attr, s.cub_tmp, s.counters, c->acct_dump_buf, c->li_ring, c->li_match,
                      c->io_dev, c->hb_pkts, c->hb_off, c->hb_len, c->hb_prio, c->hb_verdict, c->hb_now, c->dump_k, c->dump_v, c->dump_c};
        for (void *p : sp)
            if (p) cudaFree(p);
        if (c->io_host) cudaFreeHost(c->io_host);
        if (c->evict_word) cudaFreeHost(c->evict_word);
        if (c->evict_ev) cudaEventDestroy(c->evict_ev);
        for (int i = 0; i < ZC_BUFS; i++) {
            void *zp[] = {c->zc_hdr[i], c->zc_verdict[i], c->zc_off[i], c->zc_len[i], c->zc_len0[i], c->zc_prio[i], c->zc_now[i]};
            for (void *p : zp)
                if (p) cudaFree(p);
            if (c->ev_in[i]) cudaEventDestroy(c->ev_in[i]);
            if (c->ev_comp[i]) cudaEventDestroy(c->ev_comp[i]);
            if (c->ev_out[i]) cudaEventDestroy(c->ev_out[i]);
        }
        if (c->s_in) cudaStreamDestroy(c->s_in);
        if (c->s_out) cudaStreamDestroy(c->s_out);
        if (c->L.stream) cudaStreamDestroy(c->L.stream);
    }
    delete c;
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
    OPEN_R(dev_alloc(c, (void **)&d.stats, ST_COUNT * 8, 0));
    OPEN_R(make_ring(c, &d.spoof_ev, 56, ev_cap, ST_EV_LOST_SPOOF));
    OPEN_R(make_ring(c, &d.natlog_ev, 40, ev_cap, ST_EV_LOST_NATLOG));
    OPEN_CU(cudaMalloc((void **)&c->L.s.counters, 64));
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
            u8 *dst = m->kind == KIND_ARRAY ? *m->arr + (size_t)idx * m->value_size : (u8 *)(c->dev.stats + m->stat_base);
            CU(c, cudaMemcpyAsync(dst, (const u8 *)values + i * m->value_size, m->value_size, cudaMemcpyHostToDevice,
                                  c->L.stream));
        }
        CU(c, cudaStreamSynchronize(c->L.stream));
        if (feeds_small_tabs(m)) c->small_dirty = true;
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
    if (cap * t.key_size > c->dump_kb || cap * t.value_size > c->dump_vb || !c->dump_c) {
        if (c->dump_k) cudaFree(c->dump_k);
        if (c->dump_v) cudaFree(c->dump_v);
        c->dump_k = c->dump_v = nullptr;
        c->dump_kb = c->dump_vb = 0;
        size_t kb = std::max<size_t>(cap * t.key_size, 1 << 16), vb = std::max<size_t>(cap * t.value_size, 1 << 16);
        if (cudaMalloc((void **)&c->dump_k, kb) != cudaSuccess || cudaMalloc((void **)&c->dump_v, vb) != cudaSuccess)
            return fail(c, -ENOMEM, "dump: out of device memory");
        if (!c->dump_c && cudaMalloc((void **)&c->dump_c, 16) != cudaSuccess) return fail(c, -ENOMEM, "dump: out of device memory");
        c->dump_kb = kb, c->dump_vb = vb;
    }
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

static int dispatch(bng_ctx *c, int prog, const DevBatch &b, const LiSrc &src = LiSrc{}) {
    cudaError_t e = cudaSuccess;
    const bool acct = c->acct && ((c->acct_progs >> prog) & 1);
    const int li = c->li_targets.empty() ? -1 : k_li_dir[prog]; // no target: not one kernel more
    const bool pipe = prog == P_PIPE_UP || prog == P_PIPE_TC;
    // the upstream classify records attributions: for accounting, and in the pipelines to tell antispoof's drops
    c->L.acct_attr = (acct || (li == 0 && pipe)) ? c->L.s.attr : nullptr;
    LiRing r{};
    if (li >= 0) {
        r.buf = c->li_ring, r.ctl = c->li_ctl, r.match = c->li_match;
        r.cap = c->li_cap, r.rec_bytes = c->li_rec, r.snaplen = c->li_snap, r.prog = (u32)prog;
        r.tgt = AddrSet{c->li_words, c->li_mask}, r.ids = c->li_ids, r.batch = c->seq;
    }
    if (li == 0) { // the frames as they entered, before the program rewrites them
        e = cudaMemsetAsync(c->li_ctl + 2, 0, 4, c->L.stream);
        if (e == cudaSuccess) e = run_li_capture(c->L, r, b, src, true);
        if (e != cudaSuccess) return fail(c, -EIO, "launch k_li_capture: %s", cudaGetErrorString(e));
    }
    switch (prog) {
    case P_ANTISPOOF: e = run_antispoof(c->L, c->dev, b); break;
    case P_QOS_EG: e = run_qos(c->L, c->dev, b, true); break;
    case P_QOS_IN: e = run_qos(c->L, c->dev, b, false); break;
    case P_NAT_EG: e = run_nat_egress(c->L, c->dev, b); break;
    case P_NAT_IN: e = run_nat_ingress(c->L, c->dev, b); break;
    case P_NAT_HAIRPIN: e = run_nat_hairpin_xdp(c->L, c->dev, b); break;
    case P_DHCP: e = run_dhcp_fastpath(c->L, c->dev, b); break;
    case P_PIPE_UP: e = run_pipeline_up(c->L, c->dev, b); break;
    case P_PIPE_TC: e = run_pipeline_tc(c->L, c->dev, b); break;
    default: return -EINVAL;
    }
    // after the program, before anything copies the frames out: the downstream modes read the rewritten headers
    if (e == cudaSuccess && acct) e = run_acct(c->L, c->dev.subdir, b, k_acct_mode[prog], c->acct);
    if (e == cudaSuccess && li == 0) e = run_li_verdict(c->L, r, b, pipe ? c->L.s.attr : nullptr);
    if (e == cudaSuccess && li == 1) e = run_li_capture(c->L, r, b, src, false);
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
    if (!c->s_in) {
        CU(c, cudaStreamCreateWithFlags(&c->s_in, cudaStreamNonBlocking));
        CU(c, cudaStreamCreateWithFlags(&c->s_out, cudaStreamNonBlocking));
        for (int i = 0; i < ZC_BUFS; i++) {
            CU(c, cudaEventCreateWithFlags(&c->ev_in[i], cudaEventDisableTiming));
            CU(c, cudaEventCreateWithFlags(&c->ev_comp[i], cudaEventDisableTiming));
            CU(c, cudaEventCreateWithFlags(&c->ev_out[i], cudaEventDisableTiming));
            CU(c, cudaMalloc((void **)&c->zc_off[i], ZC_CHUNK * 4));
            CU(c, cudaMalloc((void **)&c->zc_len[i], ZC_CHUNK * 4));
            CU(c, cudaMalloc((void **)&c->zc_len0[i], ZC_CHUNK * 4));
            CU(c, cudaMalloc((void **)&c->zc_prio[i], ZC_CHUNK * 4));
            CU(c, cudaMalloc((void **)&c->zc_verdict[i], ZC_CHUNK));
            CU(c, cudaMalloc((void **)&c->zc_now[i], (size_t)ZC_CHUNK * 8));
        }
    }
    if (c->zc_hb < hb) {
        for (int i = 0; i < ZC_BUFS; i++) {
            if (c->zc_hdr[i]) cudaFree(c->zc_hdr[i]);
            c->zc_hdr[i] = nullptr;
        }
        c->zc_hb = 0;
        for (int i = 0; i < ZC_BUFS; i++) CU(c, cudaMalloc((void **)&c->zc_hdr[i], (size_t)ZC_CHUNK * hb + 64));
        c->zc_hb = hb;
    }
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
            CU(c, run_gather_frames(c->s_in, c->L.num_sms, chunk_arena, bb->off16 ? c->zc_off[buf] : nullptr, c->zc_len[buf],
                                    bb->stride, cn, hb, tc, c->zc_hdr[buf], c->zc_len0[buf]));
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
        b.priority = bb->priority ? c->zc_prio[buf] : nullptr;
        b.n = cn;
        b.stride = hb;
        b.now = bb->now_ns;
        b.nowv = bb->now_ns_v ? c->zc_now[buf] : nullptr;
        b.base = base;
        b.cap = hb; // bounds checks never look past a compact slot (a no-op for whole frames: hostio.cu)
        b.arena_len = (u64)cn * hb;
        // interception copies the bytes past the compact copy straight from the host arena
        const LiSrc src{chunk_arena, bb->off16 ? c->zc_off[buf] : nullptr, contiguous ? nullptr : c->zc_len0[buf], bb->stride};
        int r = dispatch(c, prog, b, src);
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
            CU(c, run_scatter_frames(c->s_out, c->L.num_sms, chunk_arena, bb->off16 ? c->zc_off[buf] : nullptr, c->zc_len0[buf],
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
    if (arena > c->hb_arena) {
        if (c->hb_pkts) cudaFree(c->hb_pkts);
        c->hb_pkts = nullptr;
        c->hb_arena = 0;
        CU(c, cudaMalloc((void **)&c->hb_pkts, arena));
        c->hb_arena = arena;
    }
    if (bb->n > c->hb_n) {
        void **pp[] = {(void **)&c->hb_off, (void **)&c->hb_len, (void **)&c->hb_prio, (void **)&c->hb_verdict, (void **)&c->hb_now};
        for (void **p : pp) {
            if (*p) cudaFree(*p);
            *p = nullptr;
        }
        c->hb_n = 0;
        CU(c, cudaMalloc((void **)&c->hb_off, (size_t)bb->n * 4));
        CU(c, cudaMalloc((void **)&c->hb_len, (size_t)bb->n * 4));
        CU(c, cudaMalloc((void **)&c->hb_prio, (size_t)bb->n * 4));
        CU(c, cudaMalloc((void **)&c->hb_verdict, (size_t)bb->n));
        CU(c, cudaMalloc((void **)&c->hb_now, (size_t)bb->n * 8));
        c->hb_n = bb->n;
    }
    CU(c, cudaMemcpyAsync(c->hb_pkts, bb->pkts, arena, cudaMemcpyHostToDevice, st));
    if (bb->off16) CU(c, cudaMemcpyAsync(c->hb_off, bb->off16, (size_t)bb->n * 4, cudaMemcpyHostToDevice, st));
    CU(c, cudaMemcpyAsync(c->hb_len, bb->len, (size_t)bb->n * 4, cudaMemcpyHostToDevice, st));
    if (bb->priority) CU(c, cudaMemcpyAsync(c->hb_prio, bb->priority, (size_t)bb->n * 4, cudaMemcpyHostToDevice, st));
    if (bb->now_ns_v) CU(c, cudaMemcpyAsync(c->hb_now, bb->now_ns_v, (size_t)bb->n * 8, cudaMemcpyHostToDevice, st));
    b.nowv = bb->now_ns_v ? c->hb_now : nullptr;
    b.pkts = c->hb_pkts;
    b.off16 = bb->off16 ? c->hb_off : nullptr;
    b.len = c->hb_len;
    b.verdict = c->hb_verdict;
    b.priority = bb->priority ? c->hb_prio : nullptr;
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
    std::lock_guard<std::mutex> g(c->mu);
    bng_ctx::Staged &q = c->staged[map];
    q.keys.insert(q.keys.end(), (const u8 *)key, (const u8 *)key + m->key_size);
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
    if (!c->stats_global) {
        CU(c, cudaMalloc((void **)&c->stats_global, ST_COUNT * 8));
        c->allocs.push_back(c->stats_global);
    }
    if (c->comm) {
        NcclApi *a = nccl_api();
        ncclResult_t r = a->AllReduce(c->dev.stats, c->stats_global, ST_COUNT, ncclUint64, ncclSum, c->comm, c->L.stream);
        if (r != ncclSuccess) return fail(c, -EIO, "ncclAllReduce: %s", a->GetErrorString ? a->GetErrorString(r) : "error");
    } else {
        CU(c, cudaMemcpyAsync(c->stats_global, c->dev.stats, ST_COUNT * 8, cudaMemcpyDeviceToDevice, c->L.stream));
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
static int table_rebuild_locked(bng_ctx *c, Tbl *t) {
    Tbl nw = *t;
    nw.lru = LRU_NONE;
    nw.max_entries = nw.mask; // the copy must never refuse or evict
    size_t bytes = ((size_t)t->mask + 1) * t->slot_bytes;
    CU(c, cudaMalloc((void **)&nw.slots, bytes));
    u32 *cnt = nullptr;
    cudaError_t e = cudaMalloc((void **)&cnt, 16);
    if (e != cudaSuccess) {
        cudaFree(nw.slots);
        return fail(c, -ENOMEM, "rebuild: out of device memory");
    }
    nw.count = cnt;
    e = cudaMemsetAsync(nw.slots, 0xFF, bytes, c->L.stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(cnt, 0, 16, c->L.stream);
    if (e == cudaSuccess) e = run_table_rebuild(c->L, *t, nw);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->L.stream);
    cudaFree(cnt);
    if (e != cudaSuccess) {
        cudaFree(nw.slots);
        return fail(c, -EIO, "rebuild: %s", cudaGetErrorString(e));
    }
    for (auto &p : c->allocs)
        if (p == t->slots) p = nw.slots;
    cudaFree(t->slots);
    t->slots = nw.slots;
    c->rebuilds++;
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
    if (!c->evict_word) CU(c, cudaHostAlloc((void **)&c->evict_word, 8, cudaHostAllocDefault));
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
    u64 *set = (u64 *)c->io_host;
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
    CU(c, run_nat_flush(c->L, c->dev, AddrSet{(const u64 *)c->io_dev, mask}, now_ns, cnt));
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
    Scratch &s = c->L.s;
    if (!s.attr) CU(c, cudaMalloc((void **)&s.attr, (size_t)s.cap * 4));
    u64 *a = nullptr;
    const size_t bytes = ((size_t)c->dev.subdir.mask + 1) * sizeof(bng_acct);
    if (cudaMalloc((void **)&a, bytes) != cudaSuccess) return fail(c, -ENOMEM, "accounting: %zu bytes of device memory", bytes);
    c->allocs.push_back(a);
    CU(c, cudaMemsetAsync(a, 0, bytes, c->L.stream));
    c->acct = a;
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
    if (need > c->acct_dump_cap) {
        if (c->acct_dump_buf) cudaFree(c->acct_dump_buf);
        c->acct_dump_buf = nullptr;
        c->acct_dump_cap = 0;
        if (cudaMalloc((void **)&c->acct_dump_buf, need) != cudaSuccess) return fail(c, -ENOMEM, "acct_dump: out of device memory");
        c->acct_dump_cap = need;
    }
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
        CU(c, run_acct_read(c->L, c->dev.subdir, c->acct, (const u32 *)c->io_dev, k, (u64 *)(c->io_dev + ooff), (int *)(c->io_dev + roff)));
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
// lawful intercept (li.cu)
// ---------------------------------------------------------------------------
static_assert(sizeof(bng_li_record) == LI_HDR, "struct bng_li_record is the device record's header");
#define LI_TSLOTS (2 * BNG_LI_MAX_TARGETS) // the target set at its fullest: load 1/2

// A ring of cap records of 64 + snaplen (rounded up to 16) bytes.  The previous ring, if any, is discarded only once
// the new one exists; its records (drained or not) are counted as lost.
static int li_collect_locked(bng_ctx *c);
static int li_ring_locked(bng_ctx *c, u32 snaplen, u32 cap) {
    const u32 rec = LI_HDR + ((snaplen + 15u) & ~15u);
    u8 *ring = nullptr;
    if (cudaMalloc((void **)&ring, (size_t)cap * rec) != cudaSuccess) {
        cudaGetLastError();
        return fail(c, -ENOMEM, "li_configure: %zu bytes of device memory", (size_t)cap * rec);
    }
    if (c->li_ring) {
        if (int r = li_collect_locked(c)) {
            cudaFree(ring);
            return r;
        }
        c->li_lost_host += c->li_pending.size() / c->li_rec;
        c->li_pending.clear();
        cudaFree(c->li_ring);
    }
    c->li_ring = ring, c->li_cap = cap, c->li_rec = rec, c->li_snap = snaplen;
    CU(c, cudaMemsetAsync(c->li_ctl, 0, 8, c->L.stream)); // no slot handed out
    return 0;
}

// Everything interception needs, on first use: control words, target set, match list, attribution words; the ring
// with the given size unless one exists.
static int li_alloc_locked(bng_ctx *c, u32 snaplen = 1518, u32 cap = 1u << 15) {
    if (!c->li_ctl) {
        Scratch &s = c->L.s;
        if (!s.attr) CU(c, cudaMalloc((void **)&s.attr, (size_t)s.cap * 4));
        CU(c, cudaMalloc((void **)&c->li_match, (size_t)s.cap * sizeof(uint2)));
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
// snapshot / restore (SURVEY.md §8f-4: device-table state for HA hand-over, reference pkg/ha)
// A snapshot is a self-describing blob: header, then per map { name, kind, key size, value size, entry count,
// keys, values } for every hash / array / LPM / statistics map (event rings are not state).  Restore clears
// each map it finds in the blob and loads the entries through the ordinary update path, so derived state
// (subscriber directory, the shared-memory image of the small maps) is rebuilt on the way and a snapshot
// taken with one set of table capacities restores into another.
// ---------------------------------------------------------------------------
namespace {
const char kSnapMagic[8] = {'B', 'N', 'G', 'S', 'N', 'A', 'P', '2'};
struct SnapMapHdr {
    char name[40];
    u32 kind, key_size, value_size, pad;
    u64 count;
};
// Trailing section of the accounting records: (address, struct bng_acct) pairs.  No map has this name, so a library
// without accounting steps over it; a context that never allocated records writes no such section.
const char kSnapAcct[] = "subscriber_acct";
const u32 kSnapAcctKind = 5;
// Trailing section of the interception targets: (address, target id) pairs, by address.  Written by a context that
// has used interception; the records are not state and stay out.
const char kSnapLi[] = "li_targets";
const u32 kSnapLiKind = 6;
} // namespace

int64_t bng_snapshot(bng_ctx *c, void *buf, uint64_t cap) {
    if (!c) return -EINVAL;
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    if (int fr = flush_staged_locked(c, -1)) return fr;
    CU(c, cudaStreamSynchronize(c->L.stream));
    std::vector<u8> out(kSnapMagic, kSnapMagic + 8);
    u64 nmaps = 0;
    size_t nmaps_at = out.size();
    out.resize(out.size() + 8);
    for (size_t mi = 0; mi < c->maps.size(); mi++) {
        MapReg *m = &c->maps[mi];
        if (m->kind == KIND_EVENT) continue;
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
        int64_t got = cnt ? map_dump_locked(c, m, keys.data(), vals.data(), cnt) : 0;
        if (got < 0) return got;
        SnapMapHdr h{};
        snprintf(h.name, sizeof(h.name), "%s", m->name);
        h.kind = (u32)m->kind, h.key_size = m->key_size, h.value_size = m->value_size, h.count = (u64)got;
        out.insert(out.end(), (u8 *)&h, (u8 *)&h + sizeof(h));
        out.insert(out.end(), keys.begin(), keys.begin() + (size_t)got * m->key_size);
        out.insert(out.end(), vals.begin(), vals.begin() + (size_t)got * m->value_size);
        nmaps++;
    }
    if (c->acct) {
        u32 n32 = 0;
        CU(c, cudaMemcpy(&n32, c->dev.subdir.count, 4, cudaMemcpyDeviceToHost));
        const u64 cnt = std::max<u32>(n32, 1);
        std::vector<u32> addrs(cnt);
        std::vector<bng_acct> recs(cnt);
        int64_t got = acct_dump_locked(c, addrs.data(), recs.data(), cnt);
        if (got < 0) return got;
        SnapMapHdr h{};
        snprintf(h.name, sizeof(h.name), "%s", kSnapAcct);
        h.kind = kSnapAcctKind, h.key_size = 4, h.value_size = sizeof(bng_acct), h.count = (u64)got;
        out.insert(out.end(), (u8 *)&h, (u8 *)&h + sizeof(h));
        out.insert(out.end(), (u8 *)addrs.data(), (u8 *)(addrs.data() + got));
        out.insert(out.end(), (u8 *)recs.data(), (u8 *)(recs.data() + got));
        nmaps++;
    }
    if (c->li_ctl) {
        std::vector<std::pair<u32, u32>> t(c->li_targets.begin(), c->li_targets.end());
        std::sort(t.begin(), t.end());
        SnapMapHdr h{};
        snprintf(h.name, sizeof(h.name), "%s", kSnapLi);
        h.kind = kSnapLiKind, h.key_size = 4, h.value_size = 4, h.count = t.size();
        out.insert(out.end(), (u8 *)&h, (u8 *)&h + sizeof(h));
        for (auto &e : t) out.insert(out.end(), (u8 *)&e.first, (u8 *)&e.first + 4);
        for (auto &e : t) out.insert(out.end(), (u8 *)&e.second, (u8 *)&e.second + 4);
        nmaps++;
    }
    memcpy(&out[nmaps_at], &nmaps, 8);
    if (buf && cap >= out.size()) memcpy(buf, out.data(), out.size());
    return (int64_t)out.size(); // the size needed; nothing was copied when cap is smaller
}

int bng_restore(bng_ctx *c, const void *buf, uint64_t len) {
    if (!c || !buf || len < 16 || memcmp(buf, kSnapMagic, 8)) return -EINVAL;
    const u8 *p = (const u8 *)buf, *end = p + len;
    u64 nmaps;
    memcpy(&nmaps, p + 8, 8);
    p += 16;
    { // the blob's records replace these; a blob without them leaves every record at zero
        std::lock_guard<std::mutex> g(c->mu);
        cudaSetDevice(c->device);
        if (c->acct) {
            CU(c, cudaMemsetAsync(c->acct, 0, ((size_t)c->dev.subdir.mask + 1) * sizeof(bng_acct), c->L.stream));
            CU(c, cudaStreamSynchronize(c->L.stream));
        }
        if (!c->li_targets.empty()) { // the same for the interception targets
            c->li_targets.clear();
            c->li_dirty = true;
        }
    }
    const u8 *acct_p = nullptr, *li_p = nullptr;
    u64 acct_n = 0, li_n = 0;
    for (u64 k = 0; k < nmaps; k++) {
        if (p + sizeof(SnapMapHdr) > end) return -EINVAL;
        SnapMapHdr h;
        memcpy(&h, p, sizeof(h));
        p += sizeof(h);
        h.name[sizeof(h.name) - 1] = 0;
        const u64 kb = h.count * h.key_size, vb = h.count * h.value_size;
        if (p + kb + vb > end) return -EINVAL;
        if (!strcmp(h.name, kSnapAcct)) { // applied below, once the maps (and so the directory) are in place
            if (h.key_size != 4 || h.value_size != sizeof(bng_acct)) return fail(c, -EINVAL, "snapshot: %s has another layout", h.name);
            acct_p = p;
            acct_n = h.count;
            p += kb + vb;
            continue;
        }
        if (!strcmp(h.name, kSnapLi)) {
            if (h.key_size != 4 || h.value_size != 4 || h.count > BNG_LI_MAX_TARGETS)
                return fail(c, -EINVAL, "snapshot: %s has another layout", h.name);
            li_p = p;
            li_n = h.count;
            p += kb + vb;
            continue;
        }
        int id = bng_map_id(c, h.name);
        if (id >= 0) {
            MapReg *m = get_map(c, id);
            if (m->key_size != h.key_size || m->value_size != h.value_size) return fail(c, -EINVAL, "snapshot: %s has another layout", h.name);
            if (m->kind == KIND_HASH) {
                int r = bng_map_clear(c, id);
                if (r) return r;
            } else if (m->kind == KIND_LPM) {
                std::lock_guard<std::mutex> g(c->mu);
                cudaSetDevice(c->device);
                m->lpm_host.clear();
                int r = lpm_upload(c, m);
                if (r) return r;
            }
            if (h.count) {
                int r = bng_map_update_batch(c, id, p, p + kb, h.count, BNG_ANY);
                if (r) return fail(c, r, "snapshot: loading %s failed", h.name);
            }
        }
        p += kb + vb;
    }
    if (acct_n) {
        std::lock_guard<std::mutex> g(c->mu);
        cudaSetDevice(c->device);
        if (int r = acct_alloc_locked(c)) return r;
        const u64 chunk_max = 1u << 16;
        for (u64 done = 0; done < acct_n; done += chunk_max) {
            const u64 k = std::min(chunk_max, acct_n - done);
            const size_t roff = (k * 4 + 255) & ~(size_t)255;
            if (int r = ensure_io(c, roff + k * sizeof(bng_acct))) return r;
            memcpy(c->io_host, acct_p + done * 4, k * 4);
            memcpy(c->io_host + roff, acct_p + acct_n * 4 + done * sizeof(bng_acct), k * sizeof(bng_acct));
            CU(c, cudaMemcpyAsync(c->io_dev, c->io_host, roff + k * sizeof(bng_acct), cudaMemcpyHostToDevice, c->L.stream));
            CU(c, run_acct_load(c->L, c->dev.subdir, c->acct, (const u32 *)c->io_dev, (const u64 *)(c->io_dev + roff), k));
            CU(c, cudaStreamSynchronize(c->L.stream));
        }
    }
    if (li_n) {
        std::lock_guard<std::mutex> g(c->mu);
        cudaSetDevice(c->device);
        if (int r = li_alloc_locked(c)) return r;
        for (u64 k = 0; k < li_n; k++) {
            u32 a, id;
            memcpy(&a, li_p + k * 4, 4);
            memcpy(&id, li_p + li_n * 4 + k * 4, 4);
            c->li_targets[a] = id;
        }
        c->li_dirty = true;
    }
    return 0;
}

// ---------------------------------------------------------------------------
// multi-GPU plumbing and diagnostics
// ---------------------------------------------------------------------------
int bng_stats_device_ptr(bng_ctx *c, void **dptr, uint32_t *n_u64) {
    if (!c || !dptr) return -EINVAL;
    *dptr = c->dev.stats;
    if (n_u64) *n_u64 = ST_COUNT;
    return 0;
}

uint64_t bng_launch_count(bng_ctx *c) { return c ? c->L.launches : 0; }

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
