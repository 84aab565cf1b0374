// bng_b200 — DHCP lease census and expiry sweep (bng_dhcp_lease_census / bng_dhcp_lease_sweep, include/bng_b200.h).
// The three lease maps (subscriber_pools, vlan_subscriber_pools, circuit_id_subscribers) have 64-byte slots and are
// streamed in one index space, as k_nat_flush streams the flow tables; circuit_id_map follows them.  Of every lease
// slot only the 32-byte sector that holds the pool_assignment is read (plus the key word of circuit_id_subscribers,
// whose value sits in the slot's second sector).
//
//   k_lease_census  read-only.  Per-pool counters are index-aligned with ip_pools' slots; a pool_id that has no
//                   ip_pools entry gets a record in a scratch hash behind them, reserved before it is claimed: once
//                   half of it is reserved the pass raises the overflow word and the host grows it and counts again.
//                   Distinct addresses and conflicts come from one scratch set of u64 words (p: the pool's record index):
//                     G  (ip)            first insert: a distinct address of the summary
//                     A  (p, ip)         first insert: a distinct address of the pool (and, outside its prefix, one more)
//                     C1 (map, p, ip)    first insert: nothing; a thread that finds it there inserts
//                     C2 (map, p, ip)    first insert: one conflict of the pool
//                   Only the thread whose compare-and-swap put a key in counts it, so every count is exact whatever
//                   the order of the threads.
//   k_lease_pools   compacts one record per pool with one atomic per warp, as k_idle_scan does.
//   k_lease_sweep   lists the due entries of the three lease maps, one atomic per warp reserving their output slots;
//                   an entry whose slot is below the cap is erased (the tables' CAS-guarded tombstone) and reported, and
//                   a subscriber_pools entry's MAC goes into a scratch set.
//   k_lease_cid     queued behind it: erases the circuit_id_map entries whose value MAC is in that set.
#include "kernels.h"

#define LS_BLOCK 256
#define LS_G (1ull << 60)
#define LS_A (2ull << 60)
#define LS_C1 (3ull << 60)
#define LS_C2 (4ull << 60)
#define LS_MAC_TAG (1ull << 48) // a MAC word is 48 bits: the tagged word is never 0, the empty word

struct LeaseEnt {
    u64 k0;
    u32 pool, ip, vlan, tail; // tail: client_class | flags << 8
    u64 expiry;
};

// The entry of slot i of the lease index space (map m), from the sector that holds its pool_assignment (packed:
// pool_id@0 allocated_ip@4 vlan_id@8 client_class@12 lease_expiry@13 flags@21).
__device__ __forceinline__ const u8 *lease_load(const DevCtx &c, u64 i, u64 n0, u64 n1, int *m, LeaseEnt *e) {
    const u8 *s;
    U256 v;
    u32 w3, w4, w5;
    if (i < n0 + n1) {
        *m = i < n0 ? 0 : 1;
        s = i < n0 ? c.sub_pools.slots + i * 64 : c.vlan_pools.slots + (i - n0) * 64;
        v = ldg256(s); // key word | pool_assignment
        e->k0 = (u64)v.w[0] | (u64)v.w[1] << 32;
        e->pool = v.w[2], e->ip = v.w[3], e->vlan = v.w[4];
        w3 = v.w[5], w4 = v.w[6], w5 = v.w[7];
    } else {
        *m = 2;
        s = c.cid_subs.slots + (i - n0 - n1) * 64;
        e->k0 = *(const u64 *)s;
        v = ldg256(s + 32);
        e->pool = v.w[0], e->ip = v.w[1], e->vlan = v.w[2];
        w3 = v.w[3], w4 = v.w[4], w5 = v.w[5];
    }
    e->expiry = (u64)(w3 >> 8) | (u64)w4 << 24 | (u64)(w5 & 0xff) << 56;
    e->tail = (w3 & 0xff) | (w5 & 0xff00);
    return s;
}

// Inserts k into a set of u64 words (0 = empty); *created when this thread put it there.  false: the set is full.
__device__ __forceinline__ bool ls_put(u64 *set, u32 mask, u64 k, bool *created) {
    *created = false;
    u32 i = (u32)mix64(k) & mask;
    for (u32 probe = 0; probe <= mask; probe++, i = (i + 1) & mask) {
        u64 w = set[i];
        if (w == 0) {
            w = atomicCAS((unsigned long long *)(set + i), 0ull, (unsigned long long)k);
            if (w == 0) {
                *created = true;
                return true;
            }
        }
        if (w == k) return true;
    }
    return false;
}

// The record index of a pool_id without an ip_pools entry, inserted on first use; LS_NONE once half the hash is
// claimed (overflow).  Only the thread whose compare-and-swap claims a slot counts it, so threads that race for one
// pool_id count one slot; the probe is bounded because the claims of threads that passed the check together can
// overshoot the half.
__device__ __forceinline__ u32 ls_unknown(const LeaseUse &u, u32 pool) {
    const u64 k = ADDRSET_LIVE | pool;
    u32 i = aset_home(pool, u.unk_mask);
    for (u32 probe = 0; probe <= u.unk_mask; probe++, i = (i + 1) & u.unk_mask) {
        u64 *p = u.pools + ((u64)u.n_known + i) * LS_POOL_WORDS + LS_P_KEY;
        u64 w = *(volatile u64 *)p;
        if (w == 0) {
            if (*(volatile u64 *)(u.sum + LS_UNK_CLAIMED) >= (u.unk_mask + 1ull) / 2) break;
            w = atomicCAS((unsigned long long *)p, 0ull, (unsigned long long)k);
            if (w == 0) {
                atomicAdd((unsigned long long *)(u.sum + LS_UNK_CLAIMED), 1ull);
                return u.n_known + i;
            }
        }
        if (w == k) return u.n_known + i;
    }
    atomicMax((unsigned long long *)(u.sum + LS_OVERFLOW), 1ull);
    return LS_NONE;
}

// Is the address inside network/prefix_len?  wire: both words hold their four bytes in wire order; else each word is the
// address's numeric value (include/bng_b200.h, bng_dhcp_lease_addr_order).
__device__ __forceinline__ bool ls_inside(u32 ip, u32 network, u32 prefix_len, bool wire) {
    if (prefix_len > 32) return false;
    if (prefix_len == 0) return true;
    const u32 d = ip ^ network;
    return ((wire ? bswap32(d) : d) >> (32 - prefix_len)) == 0;
}

__global__ void __launch_bounds__(LS_BLOCK) k_lease_census(const __grid_constant__ DevCtx c, const LeaseUse u, u64 now_s) {
    const u64 n0 = (u64)c.sub_pools.mask + 1, n1 = (u64)c.vlan_pools.mask + 1, n2 = (u64)c.cid_subs.mask + 1;
    const u64 nm = (u64)c.cid_map.mask + 1, total = n0 + n1 + n2 + nm;
    u32 loc[LS_LOCAL] = {};
    for (u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x; i < total; i += (u64)gridDim.x * blockDim.x) {
        if (i >= n0 + n1 + n2) { // circuit_id_map: fnv hash -> MAC
            const u8 *s = c.cid_map.slots + (i - n0 - n1 - n2) * c.cid_map.slot_bytes;
            if (*(const u64 *)s >= K_BUSY) continue;
            const u64 mac = *(const u64 *)(s + c.cid_map.voff);
            loc[LS_CID_DANGLING] += tbl_find<1, false>(c.sub_pools, &mac) == nullptr;
            continue;
        }
        int m;
        LeaseEnt e;
        lease_load(c, i, n0, n1, &m, &e);
        if (e.k0 >= K_BUSY) continue;
        const u64 pk = e.pool;
        const u8 *ps = tbl_find<1, false>(c.ip_pools, &pk);
        const u32 p = ps ? (u32)((ps - c.ip_pools.slots) / c.ip_pools.slot_bytes) : ls_unknown(u, e.pool);
        if (p == LS_NONE) continue; // overflow: the census runs again
        u64 *rec = u.pools + (u64)p * LS_POOL_WORDS;
        if (now_s > e.expiry) {
#pragma unroll
            for (int k = 0; k < 3; k++) loc[LS_EXP0 + k] += m == k;
            atomicAdd((unsigned long long *)(rec + LS_P_EXPIRED), 1ull);
            continue;
        }
#pragma unroll
        for (int k = 0; k < 3; k++) loc[LS_ENT0 + k] += m == k;
        loc[LS_UNKNOWN_POOL] += ps == nullptr;
        atomicAdd((unsigned long long *)(rec + m), 1ull);
        const u64 pip = (u64)p << 32 | e.ip;
        bool made;
        bool ok = ls_put(u.set, u.set_mask, LS_G | e.ip, &made);
        loc[LS_ADDRS] += made;
        if (ok && (ok = ls_put(u.set, u.set_mask, LS_A | pip, &made)) && made) {
            atomicAdd((unsigned long long *)(rec + LS_P_ADDRS), 1ull);
            const u8 *pv = ps + c.ip_pools.voff; // ip_pool: network@0 prefix_len@4
            if (!ps || !ls_inside(e.ip, *(const u32 *)pv, pv[4], u.wire)) atomicAdd((unsigned long long *)(rec + LS_P_OUTSIDE), 1ull);
        }
        if (ok && (ok = ls_put(u.set, u.set_mask, LS_C1 | (u64)m << 58 | pip, &made)) && !made &&
            (ok = ls_put(u.set, u.set_mask, LS_C2 | (u64)m << 58 | pip, &made)) && made) {
            atomicAdd((unsigned long long *)(rec + LS_P_CONFLICTS), 1ull);
            loc[LS_CONFLICTS]++;
        }
        if (!ok) atomicMax((unsigned long long *)(u.sum + LS_SET_FULL), 1ull);
    }
#pragma unroll
    for (int k = 0; k < LS_LOCAL; k++) {
        const u32 s = __reduce_add_sync(0xffffffffu, loc[k]);
        if ((threadIdx.x & 31) == 0 && s) atomicAdd((unsigned long long *)(u.sum + k), (unsigned long long)s);
    }
}

// The output position of a lane that has a record, one atomic per warp (every lane of the warp calls it).
__device__ __forceinline__ u64 ls_reserve(bool hit, u64 *count) {
    const u32 lane = threadIdx.x & 31, m = __ballot_sync(0xffffffffu, hit);
    if (!m) return 0;
    u64 base = 0;
    if (lane == 0) base = atomicAdd((unsigned long long *)count, (unsigned long long)__popc(m));
    return __shfl_sync(0xffffffffu, base, 0) + __popc(m & ((1u << lane) - 1));
}

__device__ __forceinline__ void ls_store(u32 *out, u64 pos, const u32 *rec) {
    uint4 *o = (uint4 *)(out + pos * 16);
#pragma unroll
    for (int j = 0; j < 4; j++) o[j] = make_uint4(rec[4 * j], rec[4 * j + 1], rec[4 * j + 2], rec[4 * j + 3]);
}

__global__ void __launch_bounds__(LS_BLOCK) k_lease_pools(const __grid_constant__ DevCtx c, const LeaseUse u) {
    const u64 total = (u64)u.n_known + u.unk_mask + 1;
    const u32 lane = threadIdx.x & 31;
    // warp-uniform trip count: the output is appended to with warp ballots
    for (u64 base = blockIdx.x * (u64)LS_BLOCK + (threadIdx.x & ~31u); base < total; base += (u64)gridDim.x * LS_BLOCK) {
        const u64 i = base + lane;
        bool hit = false;
        u32 rec[16] = {}, id = 0; // struct bng_lease_pool_use
        if (i < total) {
            const u64 *r = u.pools + i * LS_POOL_WORDS;
            u32 hosts = 0;
            if (i < u.n_known) {
                const u8 *s = c.ip_pools.slots + i * c.ip_pools.slot_bytes;
                const u64 k = *(const u64 *)s;
                if (k < K_BUSY) {
                    const u32 pl = s[c.ip_pools.voff + 4];
                    hit = true, id = (u32)k, rec[13] = 1;
                    hosts = pl == 0 ? 0xFFFFFFFFu : (pl <= 32 ? 1u << (32 - pl) : 0);
                }
            } else if (r[LS_P_KEY]) {
                hit = true, id = (u32)r[LS_P_KEY];
            }
            if (hit) {
#pragma unroll
                for (int k = 0; k < 4; k++) rec[2 * k] = (u32)r[k], rec[2 * k + 1] = (u32)(r[k] >> 32);
                rec[8] = (u32)r[LS_P_ADDRS], rec[9] = (u32)r[LS_P_OUTSIDE], rec[10] = (u32)r[LS_P_CONFLICTS];
                rec[11] = hosts;
                rec[12] = hosts ? (u32)((u64)(rec[8] - rec[9]) * 1000 / hosts) : 0;
            }
        }
        const u64 pos = ls_reserve(hit, u.sum + LS_POOLS_FOUND);
        if (hit && pos < u.cap) {
            u.ids_out[pos] = id;
            ls_store(u.out, pos, rec);
        }
    }
}

__global__ void __launch_bounds__(LS_BLOCK) k_lease_sweep(const __grid_constant__ DevCtx c, const LeaseSweep w) {
    const u64 n0 = (u64)c.sub_pools.mask + 1, n1 = (u64)c.vlan_pools.mask + 1, n2 = (u64)c.cid_subs.mask + 1;
    const u64 total = n0 + n1 + n2;
    const u32 lane = threadIdx.x & 31;
    u32 gone[3] = {}, tombs[3] = {};
    for (u64 base = blockIdx.x * (u64)LS_BLOCK + (threadIdx.x & ~31u); base < total; base += (u64)gridDim.x * LS_BLOCK) {
        const u64 i = base + lane;
        bool due = false;
        int m = 0;
        LeaseEnt e{};
        const u8 *s = nullptr;
        if (i < total) {
            s = lease_load(c, i, n0, n1, &m, &e);
#pragma unroll
            for (int k = 0; k < 3; k++) tombs[k] += m == k && e.k0 == K_TOMB;
            const u64 until = e.expiry + w.grace_s < e.expiry ? ~0ull : e.expiry + w.grace_s;
            due = e.k0 < K_BUSY && w.now_s > until;
        }
        const u64 pos = ls_reserve(due, w.cnt + LS_W_FOUND);
        if (!due || pos >= w.cap) continue;
        const Tbl &t = m == 0 ? c.sub_pools : (m == 1 ? c.vlan_pools : c.cid_subs);
        if (atomicCAS((unsigned long long *)s, (unsigned long long)e.k0, (unsigned long long)K_TOMB) != e.k0) {
            // nothing runs beside the sweep, so the entry is still there; if it is not, the reserved record cannot be
            // filled and the host fails the call instead of reporting a stale one
            atomicMax((unsigned long long *)(w.cnt + LS_W_LOST), 1ull);
            continue;
        }
        atomicSub(t.count, 1u);
#pragma unroll
        for (int k = 0; k < 3; k++) gone[k] += m == k, tombs[k] += m == k;
        u32 rec[16] = {}; // struct bng_lease_removed
        rec[0] = (u32)e.k0, rec[1] = (u32)(e.k0 >> 32);
        if (m == 2) {
            const U256 k = ldg256(s);
#pragma unroll
            for (int j = 2; j < 8; j++) rec[j] = k.w[j];
        }
        rec[8] = (u32)e.expiry, rec[9] = (u32)(e.expiry >> 32), rec[10] = e.pool, rec[11] = e.ip, rec[12] = e.vlan;
        rec[13] = (u32)m | e.tail << 8;
        ls_store(w.out, pos, rec);
        bool made;
        if (m == 0 && !ls_put(w.macs, w.mac_mask, LS_MAC_TAG | e.k0, &made)) atomicMax((unsigned long long *)(w.cnt + LS_W_SET_FULL), 1ull);
    }
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const u32 g = __reduce_add_sync(0xffffffffu, gone[k]), tt = __reduce_add_sync(0xffffffffu, tombs[k]);
        if (lane == 0 && g) atomicAdd((unsigned long long *)(w.cnt + LS_W_REMOVED + k), (unsigned long long)g);
        if (lane == 0 && tt) atomicAdd((unsigned long long *)(w.cnt + LS_W_TOMBS + k), (unsigned long long)tt);
    }
}

__global__ void __launch_bounds__(LS_BLOCK) k_lease_cid(const __grid_constant__ DevCtx c, const LeaseSweep w) {
    const Tbl &t = c.cid_map;
    const u64 slots = (u64)t.mask + 1;
    u32 gone = 0, tombs = 0;
    for (u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x; i < slots; i += (u64)gridDim.x * blockDim.x) {
        u8 *s = t.slots + i * t.slot_bytes;
        const u64 k0 = *(const u64 *)s;
        if (k0 >= K_BUSY) {
            tombs += k0 == K_TOMB;
            continue;
        }
        const u64 k = LS_MAC_TAG | *(const u64 *)(s + t.voff);
        bool in = false;
        u32 j = (u32)mix64(k) & w.mac_mask;
        for (u32 probe = 0; probe <= w.mac_mask && w.macs[j]; probe++, j = (j + 1) & w.mac_mask)
            if (w.macs[j] == k) {
                in = true;
                break;
            }
        if (!in || atomicCAS((unsigned long long *)s, (unsigned long long)k0, (unsigned long long)K_TOMB) != k0) continue;
        atomicSub(t.count, 1u);
        gone++, tombs++;
    }
    const u32 g = __reduce_add_sync(0xffffffffu, gone), tt = __reduce_add_sync(0xffffffffu, tombs);
    if ((threadIdx.x & 31) == 0 && g) atomicAdd((unsigned long long *)(w.cnt + LS_W_REMOVED + 3), (unsigned long long)g);
    if ((threadIdx.x & 31) == 0 && tt) atomicAdd((unsigned long long *)(w.cnt + LS_W_TOMBS + 3), (unsigned long long)tt);
}

static inline int ls_grid(const Launcher &L, u64 n) {
    const u64 want = (n + LS_BLOCK - 1) / LS_BLOCK, cap = (u64)L.num_sms * 8;
    return (int)(want < 1 ? 1 : (want < cap ? want : cap));
}

static inline u64 lease_slots(const DevCtx &c) { return (u64)c.sub_pools.mask + 1 + c.vlan_pools.mask + 1 + c.cid_subs.mask + 1; }

cudaError_t run_lease_census(Launcher &L, const DevCtx &c, const LeaseUse &u, u64 now_s) {
    prof_begin(L, "k_lease_census");
    k_lease_census<<<ls_grid(L, lease_slots(c) + c.cid_map.mask + 1), LS_BLOCK, 0, L.stream>>>(c, u, now_s);
    prof_end(L);
    L.launches++;
    return cudaGetLastError();
}

cudaError_t run_lease_pools(Launcher &L, const DevCtx &c, const LeaseUse &u) {
    prof_begin(L, "k_lease_pools");
    k_lease_pools<<<ls_grid(L, (u64)u.n_known + u.unk_mask + 1), LS_BLOCK, 0, L.stream>>>(c, u);
    prof_end(L);
    L.launches++;
    return cudaGetLastError();
}

cudaError_t run_lease_sweep(Launcher &L, const DevCtx &c, const LeaseSweep &w) {
    prof_begin(L, "k_lease_sweep");
    k_lease_sweep<<<ls_grid(L, lease_slots(c)), LS_BLOCK, 0, L.stream>>>(c, w);
    prof_end(L);
    L.launches++;
    if (w.cap == 0) return cudaGetLastError(); // a dry run removes no lease, so no mapping either
    prof_begin(L, "k_lease_cid");
    k_lease_cid<<<ls_grid(L, (u64)c.cid_map.mask + 1), LS_BLOCK, 0, L.stream>>>(c, w);
    prof_end(L);
    L.launches++;
    return cudaGetLastError();
}
