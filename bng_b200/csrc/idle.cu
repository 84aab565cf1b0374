// bng_b200 — per-subscriber idle detection (bng_idle_*, include/bng_b200.h).
//
// One record of IDLE_WORDS u64 per subscriber directory slot (kernels.h).  The data path writes only the two stamps,
// from k_acct (acct.cu).  Everything here is a control-plane call between program runs:
//   - k_idle_scan streams the directory's slots and the records once: it starts the records no scan has seen and
//     compacts the idle ones with one atomic per warp on the output count, as k_acct_dump does;
//   - k_idle_read, k_idle_timeout_set: by address;
//   - k_idle_load: whole records by address (a subscriber handed over from another context, bng_sub_import);
//   - k_idle_restart clears every clock (restore, delta apply): the stamps of another node or of another time are not
//     evidence of activity here.
#include <errno.h>

#include "../../include/bng_b200.h"
#include "kernels.h"

#define IDLE_BLOCK 256

// device record -> struct bng_idle
__device__ __forceinline__ void idle_out(const u64 *r, u64 *o) {
    const u64 up = r[IDLE_UP], dn = r[IDLE_DOWN], si = r[IDLE_SINCE];
    const u32 f = (up ? BNG_IDLE_UP : 0u) | (dn ? BNG_IDLE_DOWN : 0u) | (si ? BNG_IDLE_STARTED : 0u);
    o[0] = up ? up - 1 : 0;
    o[1] = dn ? dn - 1 : 0;
    o[2] = si ? si - 1 : 0;
    o[3] = (r[0] & 0xFFFFFFFFull) | (u64)f << 32;
}

__global__ void __launch_bounds__(IDLE_BLOCK) k_idle_scan(const __grid_constant__ Tbl dir, u64 *idle, u64 now, u32 default_s, u32 flags,
                                                          u32 *addrs_out, u64 *out, u32 *count, u64 cap) {
    const u64 slots = (u64)dir.mask + 1;
    const u32 lane = threadIdx.x & 31;
    // warp-uniform trip count: the output is appended to with warp ballots
    for (u64 base = blockIdx.x * (u64)IDLE_BLOCK + (threadIdx.x & ~31u); base < slots; base += (u64)gridDim.x * IDLE_BLOCK) {
        const u64 i = base + lane;
        const u64 k = i < slots ? *(const u64 *)(dir.slots + i * 16) : K_EMPTY;
        bool hit = false;
        u64 r[IDLE_WORDS];
        if (k < K_BUSY) {
            const ulonglong4 w = *(const ulonglong4 *)(idle + i * IDLE_WORDS);
            r[0] = w.x, r[1] = w.y, r[2] = w.z, r[3] = w.w;
            if (!r[IDLE_SINCE]) {
                idle[i * IDLE_WORDS + IDLE_SINCE] = now + 1 ? now + 1 : ~0ull; // started now, not reported
            } else {
                u64 ref = r[IDLE_SINCE];
                if ((flags & BNG_IDLE_UP) && r[IDLE_UP] > ref) ref = r[IDLE_UP];
                if ((flags & BNG_IDLE_DOWN) && r[IDLE_DOWN] > ref) ref = r[IDLE_DOWN];
                ref -= 1; // stored as clock + 1
                const u32 t0 = (u32)r[0], t = t0 ? t0 : default_s;
                hit = t != BNG_IDLE_NEVER && ref <= now && now - ref > (u64)t * 1000000000ull;
            }
        }
        const u32 m = __ballot_sync(0xffffffffu, hit);
        if (!m) continue;
        u32 pos = 0;
        if (lane == 0) pos = atomicAdd(count, (u32)__popc(m));
        pos = __shfl_sync(0xffffffffu, pos, 0) + __popc(m & ((1u << lane) - 1));
        if (!hit || pos >= cap) continue;
        addrs_out[pos] = (u32)k;
        idle_out(r, out + (u64)pos * IDLE_WORDS);
    }
}

__global__ void k_idle_read(const __grid_constant__ Tbl dir, const u64 *idle, const u32 *addrs, u64 n, u64 *out, int *results) {
    for (u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        const u32 s = dir_slot_of(dir, addrs[i]);
        u64 *o = out + i * IDLE_WORDS;
        if (s != DIR_NONE && idle) {
            idle_out(idle + (size_t)s * IDLE_WORDS, o);
        } else {
#pragma unroll
            for (int j = 0; j < IDLE_WORDS; j++) o[j] = 0;
        }
        results[i] = s != DIR_NONE ? 0 : -ENOENT;
    }
}

// Two passes so that the last value of a repeated address wins: CLAIM raises the record's scratch half-word to the
// largest list index + 1 that names it; !CLAIM writes the value of that index and puts the scratch back to 0.
template <bool CLAIM>
__global__ void k_idle_timeout_set(const __grid_constant__ Tbl dir, u64 *idle, const u32 *addrs, const u32 *timeouts, u64 n, int *results) {
    for (u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        const u32 s = dir_slot_of(dir, addrs[i]);
        if (CLAIM) results[i] = s != DIR_NONE ? 0 : -ENOENT;
        if (s == DIR_NONE) continue;
        u32 *w = (u32 *)(idle + (size_t)s * IDLE_WORDS); // [0] timeout, [1] scratch
        if (CLAIM)
            atomicMax(w + 1, (u32)i + 1);
        else if (atomicCAS(w + 1, (u32)i + 1, 0u) == (u32)i + 1)
            w[0] = timeouts[i];
    }
}

// struct bng_idle -> device record (idle_out's inverse); the scratch half-word is 0, as between calls
__global__ void k_idle_load(const __grid_constant__ Tbl dir, u64 *idle, const u32 *addrs, const u64 *recs, u64 n) {
    for (u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        const u32 s = dir_slot_of(dir, addrs[i]);
        if (s == DIR_NONE) continue;
        const u64 *o = recs + i * IDLE_WORDS;
        const u32 f = (u32)(o[3] >> 32);
        ulonglong4 w;
        w.x = o[3] & 0xFFFFFFFFull;
        w.y = (f & BNG_IDLE_UP) ? o[0] + 1 : 0;
        w.z = (f & BNG_IDLE_DOWN) ? o[1] + 1 : 0;
        w.w = (f & BNG_IDLE_STARTED) ? o[2] + 1 : 0;
        *(ulonglong4 *)(idle + (size_t)s * IDLE_WORDS) = w;
    }
}

__global__ void k_idle_restart(const __grid_constant__ Tbl dir, u64 *idle) {
    const u64 slots = (u64)dir.mask + 1;
    for (u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x; i < slots; i += (u64)gridDim.x * blockDim.x) {
        u64 *r = idle + i * IDLE_WORDS;
        r[IDLE_UP] = r[IDLE_DOWN] = r[IDLE_SINCE] = 0;
    }
}

static inline int idle_grid(const Launcher &L, u64 n) {
    const u64 want = (n + IDLE_BLOCK - 1) / IDLE_BLOCK, cap = (u64)L.num_sms * 8;
    return (int)(want < 1 ? 1 : (want < cap ? want : cap));
}

cudaError_t run_idle_scan(Launcher &L, const Tbl &dir, u64 *idle, u64 now, u32 default_s, u32 flags, u32 *addrs_out, u64 *out,
                          u32 *count, u64 cap) {
    prof_begin(L, "k_idle_scan");
    k_idle_scan<<<idle_grid(L, (u64)dir.mask + 1), IDLE_BLOCK, 0, L.stream>>>(dir, idle, now, default_s, flags, addrs_out, out, count, cap);
    prof_end(L);
    L.launches++;
    return cudaGetLastError();
}

cudaError_t run_idle_read(Launcher &L, const Tbl &dir, const u64 *idle, const u32 *addrs, u64 n, u64 *out, int *results) {
    if (n == 0) return cudaSuccess;
    k_idle_read<<<idle_grid(L, n), IDLE_BLOCK, 0, L.stream>>>(dir, idle, addrs, n, out, results);
    L.launches++;
    return cudaGetLastError();
}

cudaError_t run_idle_timeout_set(Launcher &L, const Tbl &dir, u64 *idle, const u32 *addrs, const u32 *timeouts, u64 n, int *results) {
    if (n == 0) return cudaSuccess;
    k_idle_timeout_set<true><<<idle_grid(L, n), IDLE_BLOCK, 0, L.stream>>>(dir, idle, addrs, timeouts, n, results);
    k_idle_timeout_set<false><<<idle_grid(L, n), IDLE_BLOCK, 0, L.stream>>>(dir, idle, addrs, timeouts, n, results);
    L.launches += 2;
    return cudaGetLastError();
}

cudaError_t run_idle_load(Launcher &L, const Tbl &dir, u64 *idle, const u32 *addrs, const u64 *recs, u64 n) {
    if (n == 0) return cudaSuccess;
    k_idle_load<<<idle_grid(L, n), IDLE_BLOCK, 0, L.stream>>>(dir, idle, addrs, recs, n);
    L.launches++;
    return cudaGetLastError();
}

cudaError_t run_idle_restart(Launcher &L, const Tbl &dir, u64 *idle) {
    k_idle_restart<<<idle_grid(L, (u64)dir.mask + 1), IDLE_BLOCK, 0, L.stream>>>(dir, idle);
    L.launches++;
    return cudaGetLastError();
}
