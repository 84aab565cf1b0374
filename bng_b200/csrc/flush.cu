// bng_b200 — NAT flow-state flush of a set of subscriber addresses (bng_nat_flush).  A subscriber that leaves
// (DHCP release, lease expiry, RADIUS Disconnect) leaves sessions, reverse entries and EIM mappings behind: the
// programs never consult subscriber_nat on the way down (bpf/nat44.c:860-875) nor the block on a session or EIM hit
// (:483-488, :674-680), so until they expire the next holder of the address inherits them.  The flow maps are keyed
// by 5-tuple, not by subscriber, so one streaming pass over the three tables finds them:
//   nat_sessions   key src_ip in A                        deleted, one NAT_LOG_SESSION_DELETE record each
//   nat_reverse    value (the upstream nat_key) src_ip in A   deleted (stale entries included)
//   eim_table      key internal_ip in A                    deleted, whatever its ref_count
//   subscriber_nat key in A                                sessions_active := 0
// Every predicate reads the table's own slot only, so no removal depends on another table's and the threads of the
// pass need no ordering among themselves.  nat_stats is not touched: nothing expired.
// A is an open-addressing set of u64 words built on the host (AddrSet in kernels.h); it is small and read-only, so
// it stays in L2 and the pass is bound by streaming the tables (about 0.67 GB at the reference's capacities).
#include "kernels.h"
#include "progs.cuh"

// cnt: [0] sessions, [1] reverse entries, [2] EIM mappings removed, [3] nat_sessions tombstones after the pass.
// Index space of the grid-stride loop: nat_sessions slots, then nat_reverse slots, eim_table slots, set slots.
__global__ void __launch_bounds__(256) k_nat_flush(const __grid_constant__ DevCtx c, const AddrSet a, u64 now, u32 *cnt) {
    const u64 ns = (u64)c.sessions.mask + 1, nr = (u64)c.reverse.mask + 1, ne = (u64)c.eim.mask + 1;
    const u64 total = ns + nr + ne + a.mask + 1;
    u32 n_ses = 0, n_rev = 0, n_eim = 0, tombs = 0;
    for (u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x; i < total; i += (u64)gridDim.x * blockDim.x) {
        if (i < ns) {
            const Tbl &t = c.sessions;
            u8 *s = t.slots + i * t.slot_bytes;
            const U256 s0 = ldg256(s);
            const u64 k0 = (u64)s0.w[0] | ((u64)s0.w[1] << 32);
            if (k0 >= K_BUSY) {
                tombs += k0 == K_TOMB;
                continue;
            }
            if (!aset_has(a, s0.w[0]) || atomicCAS((u64 *)s, k0, K_TOMB) != k0) continue;
            atomicSub(t.count, 1u);
            n_ses++;
            tombs++;
            // the sweep's record (sweep.cu), with the sweep's marker
            const U256 s1 = ldg256(s + 32);
            const u32 proto = (s1.w[3] >> 8) & 0xff;
            const u32 nat_ip = s0.w[4], nat_port = s0.w[5] & 0xffff;
            const u32 orig_ip = s1.w[2], orig_port = s1.w[4] & 0xffff;
            const u32 dest_ip = *(const u32 *)(s + SES_DEST_IP), dest_port = *(const u16 *)(s + SES_DEST_PORT);
            u64 sk = orig_ip;
            const u8 *sub = tbl_find<1, false>(c.sub_nat, &sk);
            const u32 sub_id = sub ? *(const u32 *)(sub + 32) : 0;
            nat_log(c, 0xFFFFFFFEu, now, 2, sub_id, orig_ip, nat_ip, (u16)orig_port, (u16)nat_port, dest_ip, (u16)dest_port, (u8)proto, 0);
        } else if (i < ns + nr) {
            const Tbl &t = c.reverse;
            u8 *s = t.slots + (i - ns) * t.slot_bytes;
            const U256 r = ldg256(s); // key 16 | value: the upstream nat_key, src_ip first
            const u64 k0 = (u64)r.w[0] | ((u64)r.w[1] << 32);
            if (k0 < K_BUSY && aset_has(a, r.w[4]) && atomicCAS((u64 *)s, k0, K_TOMB) == k0) {
                atomicSub(t.count, 1u);
                n_rev++;
            }
        } else if (i < ns + nr + ne) {
            const Tbl &t = c.eim;
            u8 *s = t.slots + (i - ns - nr) * t.slot_bytes;
            const u64 k0 = *(const u64 *)s; // internal_ip | internal_port << 32 | protocol << 48
            if (k0 < K_BUSY && aset_has(a, (u32)k0) && atomicCAS((u64 *)s, k0, K_TOMB) == k0) {
                atomicSub(t.count, 1u);
                n_eim++;
            }
        } else {
            const u64 w = a.words[i - ns - nr - ne];
            if (!w) continue;
            u64 sk = (u32)w;
            u8 *sub = tbl_find<1, false>(c.sub_nat, &sk);
            if (sub) *(unsigned long long *)(sub + 40) = 0; // sessions_active
        }
    }
    const u32 v[4] = {n_ses, n_rev, n_eim, tombs};
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const u32 s = __reduce_add_sync(0xffffffffu, v[k]);
        if ((threadIdx.x & 31) == 0 && s) atomicAdd(cnt + k, s);
    }
}

cudaError_t run_nat_flush(Launcher &L, const DevCtx &c, const AddrSet &a, u64 now, u32 *cnt) {
    prof_begin(L, "k_nat_flush");
    k_nat_flush<<<L.num_sms * 8, 256, 0, L.stream>>>(c, a, now, cnt);
    prof_end(L);
    L.launches++;
    return cudaGetLastError();
}
