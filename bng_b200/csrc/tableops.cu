// bng_b200 — control-plane side of the device hash tables: the kernels behind
// bng_map_update / lookup / delete / dump (the bpf(2) map commands the Go
// managers issue through cilium/ebpf Map.Put/Lookup/Delete).
#include <errno.h>

#include "kernels.h"

template <int KW>
__device__ __forceinline__ void load_key(const Tbl &t, const u8 *kb, u64 *kw) {
    if (t.key_size == 4) {
        kw[0] = *(const u32 *)kb;
    } else if (KW == LPM6_KW) { // 20 bytes, 4-byte aligned in a packed key array; the last word's high half zero
        const u32 *k = (const u32 *)kb;
        kw[0] = k[0] | (u64)k[1] << 32;
        kw[1] = k[2] | (u64)k[3] << 32;
        kw[2] = k[4];
    } else {
#pragma unroll
        for (int j = 0; j < KW; j++) kw[j] = *(const u64 *)(kb + 8 * j);
    }
}

__device__ __forceinline__ void copy_bytes(u8 *dst, const u8 *src, u32 n) {
    for (u32 i = 0; i < n; i++) dst[i] = src[i];
}

// value in reference (ABI) layout <-> value as stored in the slot
__device__ __forceinline__ void val_to_slot(const Tbl &t, u8 *slot, const u8 *abi) {
    if (t.vlayout == VL_SESSION) {
        for (u32 i = 0; i < t.value_size; i++) slot[ses_abi_to_slot(i)] = abi[i];
        *(u16 *)(slot + SES_EPOCH) = 0; // last_seen came from the control plane: no batch has stamped it
        *(u64 *)(slot + SES_SIDE) = 0;  // ... nor left a clock value in the side word (ses_touch_exact)
    } else {
        copy_bytes(slot + t.voff, abi, t.value_size);
        // token buckets: rate_bps (value offset 16) is mirrored next to the key, so that the per-frame
        // probe learns "unlimited or not" from the key's own 16 bytes.  Device code never changes the rate.
        if (t.vlayout == VL_QOS) *(u64 *)(slot + QOS_RATE_COPY) = *(const u64 *)(slot + t.voff + 16);
    }
}
__device__ __forceinline__ void val_from_slot(const Tbl &t, u8 *abi, const u8 *slot) {
    if (t.vlayout == VL_SESSION) {
        for (u32 i = 0; i < t.value_size; i++) abi[i] = slot[ses_abi_to_slot(i)];
    } else {
        copy_bytes(abi, slot + t.voff, t.value_size);
    }
}

// ---- subscriber directory (common.cuh): derived from subscriber_nat and qos_ingress ----
// role: which half of the directory entry the table being changed owns
enum { DIR_ROLE_NONE = 0, DIR_ROLE_NAT = 1, DIR_ROLE_QOS = 2 };

__device__ __forceinline__ void dir_set(const Tbl &dir, u64 key, int role, u32 val, u64 *acct, u64 *idle) {
    bool created;
    u8 *d = tbl_find_or_claim<1>(dir, &key, &created);
    if (!d) return; // cannot happen: the directory is sized for both maps' max_entries
    if (created) {
        *(u64 *)(d + 8) = ~0ull; // DIR_NONE | DIR_NONE << 32
        if (acct) { // the address's traffic record starts at zero, whoever held the slot before
            u64 *r = acct + (size_t)((d - dir.slots) >> 4) * ACCT_WORDS;
#pragma unroll
            for (int j = 0; j < ACCT_WORDS; j++) r[j] = 0;
        }
        if (idle) { // and its idle record: default timeout, no stamp, not started
            u64 *r = idle + (size_t)((d - dir.slots) >> 4) * IDLE_WORDS;
#pragma unroll
            for (int j = 0; j < IDLE_WORDS; j++) r[j] = 0;
        }
    }
    *(u32 *)(d + (role == DIR_ROLE_NAT ? 8 : 12)) = val;
    if (created) tbl_publish(d, key);
}
__device__ __forceinline__ void dir_unset(const Tbl &dir, u64 key, int role) {
    u8 *d = tbl_find<1, true>(dir, &key);
    if (!d) return;
    *(u32 *)(d + (role == DIR_ROLE_NAT ? 8 : 12)) = DIR_NONE;
    if (*(volatile u64 *)(d + 8) == ~0ull) tbl_erase<1>(dir, &key); // neither map knows the address any more
}
__device__ __forceinline__ u32 dir_value(const Tbl &t, const u8 *slot, int role) {
    u32 idx = (u32)((slot - t.slots) / t.slot_bytes);
    if (role == DIR_ROLE_QOS && *(const u64 *)(slot + QOS_RATE_COPY) == 0) idx |= DIR_QOS_UNLIMITED;
    return idx;
}

template <int KW>
__global__ void k_table_op(const __grid_constant__ Tbl t, int op, const u8 *keys, u8 *vals, int *results, u64 n, u32 flags,
                           const __grid_constant__ Tbl dir, int dir_role, u64 *acct, u64 *idle) {
    for (u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        u64 kw[KW];
        load_key<KW>(t, keys + i * t.key_size, kw);
        int r = 0;
        if (KW == LPM6_KW) { // subscriber_ipv6 (the only table with this key width)
            const u32 pl = (u32)kw[0];
            if (pl >= LPM6_LENS) {
                results[i] = -EINVAL;
                continue;
            }
            const u32 a[4] = {(u32)(kw[0] >> 32), (u32)kw[1], (u32)(kw[1] >> 32), (u32)kw[2]};
            if (op == TOP_LOOKUP) { // the trie's lookup: the longest prefix of length <= prefixlen covering the address
                u32 v = 0;
                r = -ENOENT;
                for (int l = (int)pl; l >= 0 && r; l--)
                    if (t.plens[l] && lpm6_probe(t, (u32)l, a, &v)) r = 0;
                if (!r) *(u32 *)(vals + i * t.value_size) = v;
                results[i] = r;
                continue;
            }
            lpm6_key(kw, pl, a); // update and delete match (prefixlen, prefix) exactly: bits past prefixlen are masked off
        }
        if (kw[0] >= K_BUSY) {
            r = (op == TOP_UPDATE) ? -EINVAL : -ENOENT; // reserved key patterns cannot be stored
        } else if (op == TOP_LOOKUP) {
            const u8 *s = tbl_find<KW, true>(t, kw);
            if (s)
                val_from_slot(t, vals + i * t.value_size, s);
            else
                r = -ENOENT;
        } else if (op == TOP_DELETE) {
            r = tbl_erase<KW>(t, kw) ? 0 : -ENOENT;
            if (!r && dir_role) dir_unset(dir, kw[0], dir_role);
            if (!r && KW == LPM6_KW) atomicSub(t.plens + (u32)kw[0], 1u);
        } else {
            const u8 *v = vals + i * t.value_size;
            u8 *s = nullptr;
            if (flags == 2) { // BPF_EXIST
                s = tbl_find<KW, true>(t, kw);
                if (s)
                    val_to_slot(t, s, v);
                else
                    r = -ENOENT;
            } else {
                bool created;
                s = tbl_find_or_claim<KW>(t, kw, &created);
                if (!s) {
                    r = -E2BIG;
                } else if (!created && flags == 1) { // BPF_NOEXIST
                    r = -EEXIST;
                } else {
                    if (created) // bytes between the key and the value, and the slot tail, stay defined
                        for (u32 z = 8 * KW; z < t.slot_bytes; z += 8) *(u64 *)(s + z) = 0;
                    val_to_slot(t, s, v);
                    if (created) tbl_publish(s, kw[0]);
                    if (created && KW == LPM6_KW) atomicAdd(t.plens + (u32)kw[0], 1u);
                }
            }
            if (!r && dir_role) dir_set(dir, kw[0], dir_role, dir_value(t, s, dir_role), acct, idle);
        }
        results[i] = r;
    }
}

// bng_map_clear() of subscriber_nat / qos_ingress: that half of every directory entry goes
__global__ void k_dir_clear_half(const __grid_constant__ Tbl dir, int role) {
    u64 slots = (u64)dir.mask + 1;
    for (u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x; i < slots; i += (u64)gridDim.x * blockDim.x) {
        u8 *d = dir.slots + i * 16;
        const u64 k = *(volatile u64 *)d;
        if (k >= K_BUSY) continue;
        *(u32 *)(d + (role == DIR_ROLE_NAT ? 8 : 12)) = DIR_NONE;
        if (*(volatile u64 *)(d + 8) == ~0ull && atomicCAS((u64 *)d, k, K_TOMB) == k) atomicSub(dir.count, 1u);
    }
}

// nat_sessions: every slot's epoch back to "never" (the 16-bit batch counter is about to reuse its values)
__global__ void k_epoch_reset(const __grid_constant__ Tbl t) {
    u64 slots = (u64)t.mask + 1;
    for (u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x; i < slots; i += (u64)gridDim.x * blockDim.x) {
        u8 *s = t.slots + i * t.slot_bytes;
        if (*(const u64 *)s < K_BUSY) *(u16 *)(s + SES_EPOCH) = 0;
    }
}

__global__ void k_table_dump(const __grid_constant__ Tbl t, u8 *keys_out, u8 *vals_out, u32 *count_out, u64 cap) {
    u64 slots = (u64)t.mask + 1;
    for (u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x; i < slots; i += (u64)gridDim.x * blockDim.x) {
        const u8 *s = t.slots + i * t.slot_bytes;
        u64 w0 = *(const u64 *)s;
        if (w0 >= K_BUSY) continue;
        u32 pos = atomicAdd(count_out, 1u);
        if (pos >= cap) continue;
        copy_bytes(keys_out + (u64)pos * t.key_size, s, t.key_size);
        val_from_slot(t, vals_out + (u64)pos * t.value_size, s);
    }
}

cudaError_t run_table_op(Launcher &L, const Tbl &t, int op, const u8 *keys, u8 *vals, int *results, u64 n, u32 flags,
                         const Tbl &dir, int dir_role, u64 *acct, u64 *idle) {
    if (n == 0) return cudaSuccess;
    int block = 128;
    u64 want = (n + block - 1) / block;
    int grid = (int)(want < (u64)L.num_sms * 8 ? want : (u64)L.num_sms * 8);
    if (t.key_size <= 8)
        k_table_op<1><<<grid, block, 0, L.stream>>>(t, op, keys, vals, results, n, flags, dir, dir_role, acct, idle);
    else if (t.key_size == 16)
        k_table_op<2><<<grid, block, 0, L.stream>>>(t, op, keys, vals, results, n, flags, dir, 0, nullptr, nullptr);
    else if (t.key_size == LPM6_KEY)
        k_table_op<LPM6_KW><<<grid, block, 0, L.stream>>>(t, op, keys, vals, results, n, flags, dir, 0, nullptr, nullptr);
    else
        k_table_op<4><<<grid, block, 0, L.stream>>>(t, op, keys, vals, results, n, flags, dir, 0, nullptr, nullptr);
    L.launches++;
    return cudaGetLastError();
}

// Re-inserts every live entry of `o` into the empty table `nw` (same geometry): tombstones left behind by
// deletes, expiry and eviction lengthen every probe chain until the table is rebuilt.
template <int KW>
__global__ void k_table_rebuild(const __grid_constant__ Tbl o, const __grid_constant__ Tbl nw) {
    u64 slots = (u64)o.mask + 1;
    for (u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x; i < slots; i += (u64)gridDim.x * blockDim.x) {
        const u8 *s = o.slots + i * o.slot_bytes;
        u64 kw[KW];
        kw[0] = *(const u64 *)s;
        if (kw[0] >= K_BUSY) continue;
#pragma unroll
        for (int j = 1; j < KW; j++) kw[j] = ((const u64 *)s)[j];
        bool created;
        u8 *d = tbl_find_or_claim<KW>(nw, kw, &created);
        if (!d || !created) continue; // cannot happen: same capacity, distinct keys
        for (u32 z = 8 * KW; z < o.slot_bytes; z += 8) *(u64 *)(d + z) = *(const u64 *)(s + z);
        tbl_publish(d, kw[0]);
    }
}

cudaError_t run_table_rebuild(Launcher &L, const Tbl &o, const Tbl &nw) {
    if (o.key_size <= 8)
        k_table_rebuild<1><<<L.num_sms * 8, 256, 0, L.stream>>>(o, nw);
    else if (o.key_size == 16)
        k_table_rebuild<2><<<L.num_sms * 8, 256, 0, L.stream>>>(o, nw);
    else if (o.key_size == LPM6_KEY)
        k_table_rebuild<LPM6_KW><<<L.num_sms * 8, 256, 0, L.stream>>>(o, nw);
    else
        k_table_rebuild<4><<<L.num_sms * 8, 256, 0, L.stream>>>(o, nw);
    L.launches++;
    return cudaGetLastError();
}

cudaError_t run_dir_clear_half(Launcher &L, const Tbl &dir, int role) {
    k_dir_clear_half<<<L.num_sms * 4, 256, 0, L.stream>>>(dir, role);
    L.launches++;
    return cudaGetLastError();
}

cudaError_t run_epoch_reset(Launcher &L, const Tbl &sessions) {
    k_epoch_reset<<<L.num_sms * 8, 256, 0, L.stream>>>(sessions);
    L.launches++;
    return cudaGetLastError();
}

cudaError_t run_table_dump(Launcher &L, const Tbl &t, u8 *keys_out, u8 *vals_out, u32 *count_out, u64 cap) {
    k_table_dump<<<L.num_sms * 4, 256, 0, L.stream>>>(t, keys_out, vals_out, count_out, cap);
    L.launches++;
    return cudaGetLastError();
}
