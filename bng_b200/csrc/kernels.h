// bng_b200 — internal interface between the C-ABI layer (ctx.cu) and the
// kernel translation units.
#pragma once
#include "common.cuh"

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
    int dhcp_smem_set;  // cudaFuncAttributeMaxDynamicSharedMemorySize applied on this context's device
    int resolve_bps[16]; // resident blocks per SM of the k_resolve instantiations, by <NAT, QOS, EGRESS, TC> bits
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

cudaError_t run_antispoof(Launcher &L, const DevCtx &c, const DevBatch &b);
cudaError_t run_qos(Launcher &L, const DevCtx &c, const DevBatch &b, bool egress);
cudaError_t run_nat_egress(Launcher &L, const DevCtx &c, const DevBatch &b);
cudaError_t run_nat_ingress(Launcher &L, const DevCtx &c, const DevBatch &b);
cudaError_t run_nat_hairpin_xdp(Launcher &L, const DevCtx &c, const DevBatch &b);
cudaError_t run_pipeline_up(Launcher &L, const DevCtx &c, const DevBatch &b);
cudaError_t run_pipeline_tc(Launcher &L, const DevCtx &c, const DevBatch &b);
cudaError_t run_dhcp_fastpath(Launcher &L, const DevCtx &c, const DevBatch &b);

// header gather / scatter between a pinned host arena and a compact device copy (hostio.cu)
cudaError_t run_gather_frames(cudaStream_t st, int blocks, const u8 *arena, const u32 *off16, const u32 *len, u32 stride,
                              u32 n, u32 slot, bool tc, u8 *dst, u32 *need);
cudaError_t run_scatter_frames(cudaStream_t st, int blocks, u8 *arena, const u32 *off16, const u32 *need, u32 stride, u32 n,
                               u32 slot, const u8 *src);

// table maintenance (tableops.cu); keys/values/results are device pointers
enum { TOP_UPDATE = 0, TOP_LOOKUP = 1, TOP_DELETE = 2 };
// dir / dir_role: the subscriber directory and which half of it table t feeds (0 none, 1 subscriber_nat, 2 qos_ingress)
// acct: the per-subscriber counter records (nullptr until accounting is first enabled); a directory slot that is
// claimed for an address has its record zeroed
cudaError_t run_table_op(Launcher &L, const Tbl &t, int op, const u8 *keys, u8 *vals, int *results, u64 n, u32 flags,
                         const Tbl &dir, int dir_role, u64 *acct);
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
cudaError_t run_nat_flush(Launcher &L, const DevCtx &c, const AddrSet &a, u64 now, u32 *cnt /* [4], see flush.cu */);
cudaError_t run_table_dump(Launcher &L, const Tbl &t, u8 *keys_out, u8 *vals_out, u32 *count_out, u64 cap);

// per-subscriber traffic accounting (acct.cu).  A record is ACCT_WORDS u64 (struct bng_acct), index-aligned with the
// subscriber directory.  Modes of run_acct: where a frame's subscriber comes from.
#define ACCT_WORDS 8
enum { ACCT_ATTR = 0, ACCT_SRC = 1, ACCT_DST = 2 }; // attribution words of classify / header source / header destination
cudaError_t run_acct(Launcher &L, const Tbl &dir, const DevBatch &b, int mode, u64 *acct);
// results[i] = 0 / -ENOENT, out[i] zeroed on a miss; acct may be nullptr (every record reads as zero)
cudaError_t run_acct_read(Launcher &L, const Tbl &dir, const u64 *acct, const u32 *addrs, u64 n, u64 *out, int *results);
// every directory address with its record, compacted at *count (grows past cap: only cap are written)
cudaError_t run_acct_dump(Launcher &L, const Tbl &dir, const u64 *acct, u32 *addrs_out, u64 *out, u32 *count, u64 cap);
// record of every address of the list that has a directory entry := the given one (snapshot restore)
cudaError_t run_acct_load(Launcher &L, const Tbl &dir, u64 *acct, const u32 *addrs, const u64 *recs, u64 n);

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
cudaError_t run_li_capture(Launcher &L, const LiRing &r, const DevBatch &b, const LiSrc &src, bool up);
cudaError_t run_li_verdict(Launcher &L, const LiRing &r, const DevBatch &b, const u32 *attr);
