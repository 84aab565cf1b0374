// bng_b200 — NAT port-usage census (bng_nat_usage, include/bng_b200.h).  A read-only pass over the flow tables: no map
// byte, counter or event is written; everything it counts goes to scratch of its own (NatUse in kernels.h).
//
//   k_natuse_flows  streams nat_sessions, eim_table, nat_reverse and subscriber_nat once (one index space, as
//                   k_nat_flush does).  Every live session or EIM entry holds a triple (public ip, port, protocol) and
//                   is attributed to an address; it puts four keys into one scratch set of u64 words:
//                     T  the triple                      first insert: a distinct triple, counted for its public ip
//                     P  (public ip, port)               first insert: a distinct port of the public ip, any protocol
//                     ST (directory slot, slot of T)     first insert: a distinct triple of the subscriber
//                     SP (directory slot, slot of P)     first insert: a distinct port of the subscriber's block
//                   Only the thread whose compare-and-swap put a key in counts it, so every distinct count is exact
//                   whatever the order of the threads.  Sessions also probe nat_reverse for the unreachable test;
//                   reverse entries probe nat_sessions for the stale test; subscriber_nat entries add their block to
//                   their public address.
//   k_natuse_emit   streams the subscriber directory and the public-address table and compacts the qualifying records
//                   with one atomic per warp, as k_idle_scan does.
//
// Per-subscriber counters are index-aligned with the subscriber directory; per-public-address counters live in a hash
// keyed by the address, whose entries are reserved before they are claimed: once half its slots are reserved, the pass
// raises the overflow word and the host grows the table and runs the census again.
#include "kernels.h"

#define NU_BLOCK 256
// key tags of the scratch set (bits 60-62; a key is never 0, the empty word)
#define NU_T (1ull << 60)
#define NU_P (2ull << 60)
#define NU_ST (3ull << 60)
#define NU_SP (4ull << 60)

// Inserts k; returns its slot and sets *created when this thread put it there.  NU_NONE when the set is full, which
// its sizing rules out (kernels.h); the probe is bounded all the same.
__device__ __forceinline__ u32 nu_put(const NatUse &u, u64 k, bool *created) {
    *created = false;
    u32 i = (u32)mix64(k) & u.set_mask;
    for (u32 probe = 0; probe <= u.set_mask; probe++, i = (i + 1) & u.set_mask) {
        u64 w = u.set[i];
        if (w == 0) {
            w = atomicCAS((unsigned long long *)(u.set + i), 0ull, (unsigned long long)k);
            if (w == 0) {
                *created = true;
                return i;
            }
        }
        if (w == k) return i;
    }
    atomicMax((unsigned long long *)(u.sum + NU_SET_FULL), 1ull);
    return NU_NONE;
}

// The record of a public address (NU_PUB_WORDS in kernels.h), inserted on first use; nullptr once the table is half
// reserved (overflow).
__device__ __forceinline__ u64 *nu_pub(const NatUse &u, u32 ip) {
    const u64 k = ADDRSET_LIVE | ip;
    for (u32 i = aset_home(ip, u.pub_mask);; i = (i + 1) & u.pub_mask) {
        u64 *p = u.pub + (u64)i * NU_PUB_WORDS;
        u64 w = *(volatile u64 *)p;
        if (w == 0) {
            if (atomicAdd((unsigned long long *)(u.sum + NU_PUB_RESERVED), 1ull) >= (u.pub_mask + 1ull) / 2) {
                atomicMax((unsigned long long *)(u.sum + NU_OVERFLOW), 1ull);
                return nullptr;
            }
            w = atomicCAS((unsigned long long *)p, 0ull, (unsigned long long)k);
            if (w == 0) return p;
        }
        if (w == k) return p;
    }
}

__device__ __forceinline__ int nu_col(u32 proto) { return proto == 6 ? 0 : proto == 17 ? 1 : proto == 1 ? 2 : -1; }

// One live entry holding (ip, port, proto), attributed to address a.  ses: a session (else an EIM entry); unr: it is
// an unreachable session.  loc: this thread's summary counts.
__device__ __forceinline__ void nu_held(const DevCtx &c, const NatUse &u, u32 a, u32 ip, u32 port, u32 proto, bool ses, bool unr,
                                        u32 *loc) {
    const u64 tk = (u64)ip | (u64)port << 32 | (u64)proto << 48;
    bool new_t, new_p;
    const u32 it = nu_put(u, NU_T | tk, &new_t);
    const u32 ipp = nu_put(u, NU_P | (tk & 0xFFFFFFFFFFFFull), &new_p);
    if (it == NU_NONE || ipp == NU_NONE) return;
    loc[NU_TRIPLES] += new_t;
    const int col = nu_col(proto);
    if (u64 *r = nu_pub(u, ip)) {
        u32 *p = (u32 *)(r + 2);
        atomicAdd(p + (ses ? 0 : 1), 1u);
        if (new_t && col >= 0) atomicAdd(p + 3 + col, 1u);
        if (new_p) atomicAdd(p + 6, 1u);
        if (unr) atomicAdd(p + 7, 1u);
    }
    const u32 d = dir_slot_of(c.subdir, a);
    const u32 ns = d == DIR_NONE ? DIR_NONE : *(const u32 *)(c.subdir.slots + (u64)d * 16 + 8);
    if (ns == DIR_NONE) { // no subscriber_nat entry for the address
        loc[ses ? NU_ORPHAN_SES : NU_ORPHAN_EIM]++;
        return;
    }
    const u32 *blk = (const u32 *)(c.sub_nat.slots + (u64)ns * c.sub_nat.slot_bytes + c.sub_nat.voff);
    const u32 bip = blk[0], ps = blk[1] & 0xffff, pe = blk[1] >> 16;
    const bool inside = ip == bip && port >= ps && port <= pe;
    u32 *s = u.sub + (u64)d * NU_SUB_WORDS; // [0] sessions [1] eim [2..4] in_use [5] any [6] outside [7] unreachable
    atomicAdd(s + (ses ? 0 : 1), 1u);
    if (unr) atomicAdd(s + 7, 1u);
    bool new_st, new_sp;
    if (nu_put(u, NU_ST | (u64)it << 30 | d, &new_st) == NU_NONE || !new_st) return;
    if (!inside) {
        atomicAdd(s + 6, 1u);
        return;
    }
    if (col >= 0) atomicAdd(s + 2 + col, 1u);
    if (nu_put(u, NU_SP | (u64)ipp << 30 | d, &new_sp) != NU_NONE && new_sp) atomicAdd(s + 5, 1u);
}

__global__ void __launch_bounds__(NU_BLOCK) k_natuse_flows(const __grid_constant__ DevCtx c, const NatUse u) {
    const u64 ns = (u64)c.sessions.mask + 1, ne = (u64)c.eim.mask + 1, nr = (u64)c.reverse.mask + 1;
    const u64 nb = (u64)c.sub_nat.mask + 1, total = ns + ne + nr + nb;
    u32 loc[NU_LOCAL] = {};
    for (u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x; i < total; i += (u64)gridDim.x * blockDim.x) {
        if (i < ns) {
            const u8 *s = c.sessions.slots + i * c.sessions.slot_bytes;
            const U256 s0 = ldg256(s); // key 16 | nat_ip | nat_port (network order) | epoch | out_lo
            const u64 k0 = (u64)s0.w[0] | ((u64)s0.w[1] << 32);
            if (k0 >= K_BUSY) continue;
            const u32 proto = s[SES_STATE + 1], nat_ip = s0.w[4], nat_port = s0.w[5] & 0xffff;
            // the reverse key nat44_egress writes with a new session (bpf/nat44.c:726-733)
            const u64 rk[2] = {(u64)s0.w[1] | (u64)nat_ip << 32, (s0.w[2] >> 16) | nat_port << 16 | (u64)proto << 32};
            const u8 *r = tbl_find<2, false>(c.reverse, rk);
            const u64 k1 = (u64)s0.w[2] | ((u64)s0.w[3] << 32);
            const bool unr = !r || *(const u64 *)(r + 16) != k0 || *(const u64 *)(r + 24) != k1;
            loc[NU_SESSIONS]++;
            loc[NU_UNREACHABLE] += unr;
            nu_held(c, u, s0.w[0], nat_ip, bswap16((u16)nat_port), proto, true, unr, loc);
        } else if (i < ns + ne) {
            const u8 *s = c.eim.slots + (i - ns) * c.eim.slot_bytes;
            const u64 k0 = *(const u64 *)s; // internal_ip | internal_port << 32 | protocol << 48
            if (k0 >= K_BUSY) continue;
            const u64 v = *(const u64 *)(s + c.eim.voff); // external_ip | external_port (host order) << 32
            loc[NU_EIM]++;
            nu_held(c, u, (u32)k0, (u32)v, (u32)(v >> 32) & 0xffff, (u32)(k0 >> 48) & 0xff, false, false, loc);
        } else if (i < ns + ne + nr) {
            const u8 *s = c.reverse.slots + (i - ns - ne) * c.reverse.slot_bytes;
            if (*(const u64 *)s >= K_BUSY) continue;
            const u64 sk[2] = {*(const u64 *)(s + 16), *(const u64 *)(s + 24)}; // the value: a session's key
            loc[NU_STALE] += tbl_find<2, false>(c.sessions, sk) == nullptr;
        } else {
            const u8 *s = c.sub_nat.slots + (i - ns - ne - nr) * c.sub_nat.slot_bytes;
            if (*(const u64 *)s >= K_BUSY) continue;
            const u32 *blk = (const u32 *)(s + c.sub_nat.voff);
            const u32 ps = blk[1] & 0xffff, pe = blk[1] >> 16;
            loc[NU_SUBSCRIBERS]++;
            if (u64 *r = nu_pub(u, blk[0])) {
                atomicAdd((u32 *)(r + 2) + 2, 1u);
                if (pe >= ps) atomicAdd((unsigned long long *)(r + 1), (unsigned long long)(pe - ps + 1));
            }
        }
    }
#pragma unroll
    for (int k = 0; k < NU_LOCAL; k++) {
        const u32 s = __reduce_add_sync(0xffffffffu, loc[k]);
        if ((threadIdx.x & 31) == 0 && s) atomicAdd((unsigned long long *)(u.sum + k), (unsigned long long)s);
    }
}

// Appends the record of a lane that has one at *count, one atomic per warp; false: no room (or nothing to write).
__device__ __forceinline__ bool nu_slot(bool hit, u64 *count, u64 cap, u64 *pos) {
    const u32 lane = threadIdx.x & 31, m = __ballot_sync(0xffffffffu, hit);
    if (!m) return false;
    u64 base = 0;
    if (lane == 0) base = atomicAdd((unsigned long long *)count, (unsigned long long)__popc(m));
    *pos = __shfl_sync(0xffffffffu, base, 0) + __popc(m & ((1u << lane) - 1));
    return hit && *pos < cap;
}

__global__ void __launch_bounds__(NU_BLOCK) k_natuse_emit(const __grid_constant__ DevCtx c, const NatUse u, u32 min_permille) {
    const u64 nd = (u64)c.subdir.mask + 1, total = nd + u.pub_mask + 1;
    const u32 lane = threadIdx.x & 31;
    // warp-uniform trip count: the outputs are appended to with warp ballots
    for (u64 base = blockIdx.x * (u64)NU_BLOCK + (threadIdx.x & ~31u); base < total; base += (u64)gridDim.x * NU_BLOCK) {
        const u64 i = base + lane;
        bool sub_hit = false, pub_hit = false;
        u32 rec[16] = {};
        u32 addr = 0;
        if (i < nd) {
            const u8 *ds = c.subdir.slots + i * 16;
            const u64 k = *(const u64 *)ds;
            const u32 nslot = *(const u32 *)(ds + 8);
            if (k < K_BUSY && nslot != DIR_NONE) {
                const u32 *blk = (const u32 *)(c.sub_nat.slots + (u64)nslot * c.sub_nat.slot_bytes + c.sub_nat.voff);
                const u32 ps = blk[1] & 0xffff, pe = blk[1] >> 16, bp = pe >= ps ? pe - ps + 1 : 0;
                const u32 *s = u.sub + i * NU_SUB_WORDS;
                const u32 mx = max(s[2], max(s[3], s[4]));
                const u32 pm = bp ? (u32)((u64)mx * 1000 / bp) : 0;
                addr = (u32)k;
                // struct bng_nat_sub_use
                rec[0] = s[0], rec[2] = s[1], rec[4] = blk[0], rec[5] = bp;
                rec[6] = s[2], rec[7] = s[3], rec[8] = s[4], rec[9] = s[5], rec[10] = s[6], rec[11] = s[7], rec[12] = pm;
                sub_hit = pm >= min_permille;
            }
        } else if (i < total) {
            const u64 *p = u.pub + (i - nd) * NU_PUB_WORDS;
            if (p[0]) {
                const u32 *q = (const u32 *)(p + 2);
                addr = (u32)p[0];
                // struct bng_nat_pub_use
                rec[0] = q[0], rec[2] = q[1], rec[4] = (u32)p[1], rec[5] = (u32)(p[1] >> 32);
                rec[6] = q[2], rec[7] = q[3], rec[8] = q[4], rec[9] = q[5], rec[10] = q[6], rec[11] = q[7];
                pub_hit = true;
            }
        }
        u64 pos;
        if (nu_slot(sub_hit, u.sum + NU_SUBS_FOUND, u.sub_cap, &pos)) {
            u.sub_addrs[pos] = addr;
            uint4 *o = (uint4 *)(u.sub_out + pos * 16);
#pragma unroll
            for (int j = 0; j < 4; j++) o[j] = make_uint4(rec[4 * j], rec[4 * j + 1], rec[4 * j + 2], rec[4 * j + 3]);
        }
        if (nu_slot(pub_hit, u.sum + NU_PUBS_FOUND, u.pub_cap, &pos)) {
            u.pub_addrs[pos] = addr;
            uint4 *o = (uint4 *)(u.pub_out + pos * 16);
#pragma unroll
            for (int j = 0; j < 4; j++) o[j] = make_uint4(rec[4 * j], rec[4 * j + 1], rec[4 * j + 2], rec[4 * j + 3]);
        }
    }
}

static inline int nu_grid(const Launcher &L, u64 n) {
    const u64 want = (n + NU_BLOCK - 1) / NU_BLOCK, cap = (u64)L.num_sms * 8;
    return (int)(want < 1 ? 1 : (want < cap ? want : cap));
}

cudaError_t run_nat_usage_flows(Launcher &L, const DevCtx &c, const NatUse &u) {
    const u64 total = (u64)c.sessions.mask + 1 + c.eim.mask + 1 + c.reverse.mask + 1 + c.sub_nat.mask + 1;
    prof_begin(L, "k_natuse_flows");
    k_natuse_flows<<<nu_grid(L, total), NU_BLOCK, 0, L.stream>>>(c, u);
    prof_end(L);
    L.launches++;
    return cudaGetLastError();
}

cudaError_t run_nat_usage_emit(Launcher &L, const DevCtx &c, const NatUse &u, u32 min_permille) {
    prof_begin(L, "k_natuse_emit");
    k_natuse_emit<<<nu_grid(L, (u64)c.subdir.mask + 1 + u.pub_mask + 1), NU_BLOCK, 0, L.stream>>>(c, u, min_permille);
    prof_end(L);
    L.launches++;
    return cudaGetLastError();
}
