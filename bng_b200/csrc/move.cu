// bng_b200 — subscriber hand-over between contexts (bng_sub_export / bng_sub_import, include/bng_b200.h).
//
// The flow maps are keyed by 5-tuple, not by subscriber, so the export finds a set A of subscriber addresses' flow
// state with one streaming pass over the three tables, with bng_nat_flush's predicates (flush.cu):
//   nat_sessions   key src_ip in A
//   nat_reverse    value (the upstream nat_key) src_ip in A, stale entries included
//   eim_table      key internal_ip in A
// k_move_select only reads: it lists the matching slot indices per table, compacted with one atomic per warp and
// table.  The lists are turned into ABI keys and values by the delta exporter's gather (k_delta_emit, delta.cu), and,
// when the export detaches, k_move_detach tombstones exactly the listed slots.  Unlike the flush, the detach writes
// no log record and touches no counter but the tables' live counts: nothing expired, the state lives on elsewhere.
// The per-address and per-MAC maps are reached by key through the table-op kernels (tableops.cu), so the subscriber
// directory stays derived state.
// subscriber_ipv6 is keyed by prefix and selected by value (the owner's IPv4 address in A): k_move_select_v6 lists its
// matching slots the same way, launched only while the table has live entries.  Its detach deletes the gathered keys
// through the table-op path, which keeps the per-length counts.
#include "kernels.h"

#define MOVE_BLOCK 256

// Appends slot i to a list with one atomic per warp (every lane of the warp calls it, `take` says which ones add).
__device__ __forceinline__ void move_push(u32 *list, u32 *count, bool take, u32 i) {
    const u32 lane = threadIdx.x & 31, m = __ballot_sync(0xffffffffu, take);
    if (!m) return;
    u32 pos = 0;
    if (lane == 0) pos = atomicAdd(count, (u32)__popc(m));
    pos = __shfl_sync(0xffffffffu, pos, 0) + __popc(m & ((1u << lane) - 1));
    if (take) list[pos] = i;
}

// One sector per slot: nat_sessions' and eim_table's key word, nat_reverse's key word and value (the first 32 bytes).
__global__ void __launch_bounds__(MOVE_BLOCK) k_move_select(const __grid_constant__ DevCtx c, const AddrSet a, u32 *lists, u32 *cnt) {
    const u64 ns = (u64)c.sessions.mask + 1, nr = (u64)c.reverse.mask + 1, ne = (u64)c.eim.mask + 1;
    const u64 stride = (u64)gridDim.x * MOVE_BLOCK, first = blockIdx.x * (u64)MOVE_BLOCK + (threadIdx.x & ~31u);
    const u32 lane = threadIdx.x & 31;
    u32 tombs = 0;
    // warp-uniform trip counts: the lists are appended to with warp ballots
    for (u64 base = first; base < ns; base += stride) {
        const u64 i = base + lane;
        bool take = false;
        if (i < ns) {
            const u64 k0 = __ldg((const unsigned long long *)(c.sessions.slots + i * c.sessions.slot_bytes));
            tombs += k0 == K_TOMB;
            take = k0 < K_BUSY && aset_has(a, (u32)k0);
        }
        move_push(lists, cnt, take, (u32)i);
    }
    for (u64 base = first; base < nr; base += stride) {
        const u64 i = base + lane;
        bool take = false;
        if (i < nr) {
            const U256 r = ldg256(c.reverse.slots + i * c.reverse.slot_bytes); // key 16 | value: the upstream nat_key
            const u64 k0 = (u64)r.w[0] | ((u64)r.w[1] << 32);
            take = k0 < K_BUSY && aset_has(a, r.w[4]);
        }
        move_push(lists + ns, cnt + 1, take, (u32)i);
    }
    for (u64 base = first; base < ne; base += stride) {
        const u64 i = base + lane;
        bool take = false;
        if (i < ne) {
            const u64 k0 = __ldg((const unsigned long long *)(c.eim.slots + i * c.eim.slot_bytes)); // internal_ip | ...
            take = k0 < K_BUSY && aset_has(a, (u32)k0);
        }
        move_push(lists + ns + nr, cnt + 2, take, (u32)i);
    }
    const u32 s = __reduce_add_sync(0xffffffffu, tombs);
    if (lane == 0 && s) atomicAdd(cnt + 3, s);
}

__global__ void __launch_bounds__(MOVE_BLOCK) k_move_select_v6(const __grid_constant__ Tbl t, const AddrSet a, u32 *list, u32 *cnt) {
    const u64 n = (u64)t.mask + 1;
    const u32 lane = threadIdx.x & 31;
    for (u64 base = blockIdx.x * (u64)MOVE_BLOCK + (threadIdx.x & ~31u); base < n; base += (u64)gridDim.x * MOVE_BLOCK) {
        const u64 i = base + lane;
        bool take = false;
        if (i < n) {
            const u8 *s = t.slots + i * t.slot_bytes;
            take = __ldg((const unsigned long long *)s) < K_BUSY && aset_has(a, *(const u32 *)(s + t.voff));
        }
        move_push(list, cnt, take, (u32)i);
    }
}

__global__ void k_move_detach(const __grid_constant__ DevCtx c, const u32 *lists, uint3 n) {
    const u64 ns = (u64)c.sessions.mask + 1, nr = (u64)c.reverse.mask + 1;
    const u64 total = (u64)n.x + n.y + n.z;
    for (u64 j = blockIdx.x * (u64)blockDim.x + threadIdx.x; j < total; j += (u64)gridDim.x * blockDim.x) {
        const Tbl &t = j < n.x ? c.sessions : (j < (u64)n.x + n.y ? c.reverse : c.eim);
        const u32 i = j < n.x ? lists[j] : (j < (u64)n.x + n.y ? lists[ns + (j - n.x)] : lists[ns + nr + (j - n.x - n.y)]);
        u64 *s = (u64 *)(t.slots + (u64)i * t.slot_bytes);
        const u64 k0 = *(volatile u64 *)s;
        if (k0 < K_BUSY && atomicCAS((unsigned long long *)s, k0, K_TOMB) == k0) atomicSub(t.count, 1u);
    }
}

static inline int move_grid(const Launcher &L, u64 n) {
    const u64 want = (n + MOVE_BLOCK - 1) / MOVE_BLOCK, cap = (u64)L.num_sms * 8;
    return (int)(want < 1 ? 1 : (want < cap ? want : cap));
}

cudaError_t run_move_select(Launcher &L, const DevCtx &c, const AddrSet &a, u32 *lists, u32 *cnt) {
    prof_begin(L, "k_move_select");
    k_move_select<<<L.num_sms * 8, MOVE_BLOCK, 0, L.stream>>>(c, a, lists, cnt);
    prof_end(L);
    L.launches++;
    return cudaGetLastError();
}

cudaError_t run_move_detach(Launcher &L, const DevCtx &c, const u32 *lists, const u32 n[3]) {
    const u64 total = (u64)n[0] + n[1] + n[2];
    if (total == 0) return cudaSuccess;
    prof_begin(L, "k_move_detach");
    k_move_detach<<<move_grid(L, total), MOVE_BLOCK, 0, L.stream>>>(c, lists, make_uint3(n[0], n[1], n[2]));
    prof_end(L);
    L.launches++;
    return cudaGetLastError();
}

cudaError_t run_move_select_v6(Launcher &L, const Tbl &v6, const AddrSet &a, u32 *list, u32 *cnt) {
    prof_begin(L, "k_move_select_v6");
    k_move_select_v6<<<move_grid(L, (u64)v6.mask + 1), MOVE_BLOCK, 0, L.stream>>>(v6, a, list, cnt);
    prof_end(L);
    L.launches++;
    return cudaGetLastError();
}
