// bng_b200 — incremental replication of the hash maps to a standby (bng_delta_*, include/bng_b200.h).
//
// Each replicated table has a shadow on the GPU: per slot, the slot's first `sw` 64-bit words (the key words, then
// the words that hold the value's compared bytes) as they were when the slot was last sent.  An export is three passes
// per table on the context's stream, all between program runs:
//   - k_delta_diff streams the slots and the shadow once and classifies every slot: its shadow key is to be deleted
//     (the table no longer holds it there), its entry is to be upserted (new key, a compared byte changed, or the time
//     word moved more than refresh_ns past the copy sent), both, or neither.  It lists the slot indices of the two
//     classes, compacted with one atomic per warp and class.
//   - k_delta_emit turns the lists into records: deleted keys from the shadow, upserted keys and values (ABI layout)
//     from the slots.
//   - k_delta_commit, only once the whole delta fits the caller's buffer, copies the listed slots into the shadow.
// The data path never writes anything for this: a table is compared with its shadow only when a delta is exported.
#include "kernels.h"

#define DELTA_BLOCK 256

__device__ __forceinline__ u64 delta_word(const DeltaTbl &t, u64 i, u32 w) {
    if (t.vals && w >= t.kw) return *(const u64 *)(t.vals + i * t.vstride + (w - t.kw) * 8);
    return *(const u64 *)(t.slots + i * t.slot_bytes + w * 8);
}

// Appends slot i to a list with one atomic per warp (every lane of the warp calls it, `take` says which ones add).
__device__ __forceinline__ void delta_push(u32 *list, u32 *count, bool take, u32 i) {
    const u32 lane = threadIdx.x & 31, m = __ballot_sync(0xffffffffu, take);
    if (!m) return;
    u32 pos = 0;
    if (lane == 0) pos = atomicAdd(count, (u32)__popc(m));
    pos = __shfl_sync(0xffffffffu, pos, 0) + __popc(m & ((1u << lane) - 1));
    if (take) list[pos] = i;
}

__global__ void __launch_bounds__(DELTA_BLOCK) k_delta_diff(const __grid_constant__ DeltaTbl t, u32 *del, u32 *up, u32 *cnt,
                                                            int full) {
    // warp-uniform trip count: the lists are appended to with warp ballots
    for (u64 base = blockIdx.x * (u64)DELTA_BLOCK + (threadIdx.x & ~31u); base < t.nslots; base += (u64)gridDim.x * DELTA_BLOCK) {
        const u64 i = base + (threadIdx.x & 31);
        bool d = false, u = false;
        if (i < t.nslots) {
            const u64 *sh = t.shadow + i * t.sw;
            const u64 c0 = delta_word(t, i, 0);
            const u64 s0 = full ? K_EMPTY : sh[0];
            const bool cl = c0 < K_BUSY, sl = s0 < K_BUSY;
            bool same = cl && sl && c0 == s0;
            for (u32 w = 1; w < t.kw; w++) same = same && delta_word(t, i, w) == sh[w];
            d = sl && !same;
            u = cl && !same;
            if (same) {
                bool diff = false;
#pragma unroll 4
                for (u32 w = t.kw; w < t.sw; w++) {
                    const u64 cw = delta_word(t, i, w), sw = sh[w];
                    diff |= ((cw ^ sw) & t.mask[w]) != 0;
                    if (w == t.tw) diff |= (long long)(cw - sw) > (long long)t.refresh;
                }
                u = diff;
            }
        }
        delta_push(del, cnt, d, (u32)i);
        delta_push(up, cnt + 1, u, (u32)i);
    }
}

// Records of the listed slots: deleted keys from the shadow, upserted (key, value) pairs from the table.
__global__ void k_delta_emit(const __grid_constant__ DeltaTbl t, const u32 *del, u32 n_del, const u32 *up, u32 n_up, u8 *del_keys,
                             u8 *up_keys, u8 *up_vals) {
    const u64 n = (u64)n_del + n_up;
    for (u64 j = blockIdx.x * (u64)blockDim.x + threadIdx.x; j < n; j += (u64)gridDim.x * blockDim.x) {
        if (j < n_del) {
            const u8 *k = (const u8 *)(t.shadow + (u64)del[j] * t.sw);
            for (u32 b = 0; b < t.key_size; b++) del_keys[j * t.key_size + b] = k[b];
            continue;
        }
        const u64 r = j - n_del, i = up[r];
        const u8 *s = t.slots + i * t.slot_bytes;
        for (u32 b = 0; b < t.key_size; b++) up_keys[r * t.key_size + b] = s[b];
        u8 *v = up_vals + r * t.value_size;
        if (t.vals) {
            for (u32 b = 0; b < t.value_size; b++) v[b] = t.vals[i * t.vstride + b];
        } else if (t.vlayout == VL_SESSION) {
            for (u32 b = 0; b < t.value_size; b++) v[b] = s[ses_abi_to_slot(b)];
        } else {
            for (u32 b = 0; b < t.value_size; b++) v[b] = s[t.voff + b];
        }
    }
}

// The shadow of the listed slots := what was sent.  A slot listed for deletion only (nothing live there now) becomes
// empty; a slot listed for an upsert (whether or not it also had a deletion) takes the slot's words.  No slot is
// written by two threads: the two cases exclude each other.
__global__ void k_delta_commit(const __grid_constant__ DeltaTbl t, const u32 *del, u32 n_del, const u32 *up, u32 n_up) {
    const u64 n = (u64)n_del + n_up;
    for (u64 j = blockIdx.x * (u64)blockDim.x + threadIdx.x; j < n; j += (u64)gridDim.x * blockDim.x) {
        const u64 i = j < n_del ? del[j] : up[j - n_del];
        u64 *sh = t.shadow + i * t.sw;
        const u64 c0 = delta_word(t, i, 0);
        if (j < n_del) {
            if (c0 >= K_BUSY) sh[0] = K_EMPTY;
            continue;
        }
        for (u32 w = 0; w < t.sw; w++) sh[w] = delta_word(t, i, w);
    }
}

static inline int delta_grid(const Launcher &L, u64 n) {
    const u64 want = (n + DELTA_BLOCK - 1) / DELTA_BLOCK, cap = (u64)L.num_sms * 8;
    return (int)(want < 1 ? 1 : (want < cap ? want : cap));
}

cudaError_t run_delta_diff(Launcher &L, const DeltaTbl &t, u32 *del, u32 *up, u32 *cnt, bool full) {
    prof_begin(L, "k_delta_diff");
    k_delta_diff<<<delta_grid(L, t.nslots), DELTA_BLOCK, 0, L.stream>>>(t, del, up, cnt, full ? 1 : 0);
    prof_end(L);
    L.launches++;
    return cudaGetLastError();
}

cudaError_t run_delta_emit(Launcher &L, const DeltaTbl &t, const u32 *del, u32 n_del, const u32 *up, u32 n_up, u8 *del_keys,
                           u8 *up_keys, u8 *up_vals) {
    if ((u64)n_del + n_up == 0) return cudaSuccess;
    prof_begin(L, "k_delta_emit");
    k_delta_emit<<<delta_grid(L, (u64)n_del + n_up), DELTA_BLOCK, 0, L.stream>>>(t, del, n_del, up, n_up, del_keys, up_keys, up_vals);
    prof_end(L);
    L.launches++;
    return cudaGetLastError();
}

cudaError_t run_delta_commit(Launcher &L, const DeltaTbl &t, const u32 *del, u32 n_del, const u32 *up, u32 n_up) {
    if ((u64)n_del + n_up == 0) return cudaSuccess;
    prof_begin(L, "k_delta_commit");
    k_delta_commit<<<delta_grid(L, (u64)n_del + n_up), DELTA_BLOCK, 0, L.stream>>>(t, del, n_del, up, n_up);
    prof_end(L);
    L.launches++;
    return cudaGetLastError();
}
