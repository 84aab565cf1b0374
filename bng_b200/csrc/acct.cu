// bng_b200 — per-subscriber traffic accounting (bng_acct_*, include/bng_b200.h).
//
// One record of ACCT_WORDS u64 per subscriber directory slot (struct bng_acct: upstream pass / drop, downstream
// pass / drop, packets and bytes each).  k_acct runs after a program, on the same stream, one thread per frame: it
// finds the frame's directory slot (the word classify recorded, or the address in the outgoing header), reads the
// verdict and skb->len, and adds the frame to the slot's pass or drop pair.  Frames of one warp that go to the same
// pair are summed first (__match_any_sync): the leader of each group issues the two atomics, so a subscriber that
// owns a whole batch costs one atomic pair per warp, not per frame.
//
// The same pass stamps the idle records (idle.cu) when idle detection is on for the program: the leader of a group of
// passed frames raises the record's stamp of the direction to the group's latest clock with one atomicMax.  With one
// clock for the whole batch the leader reads the stamp first and skips the atomic when it is already there.
//
// V6 (launched only while subscriber_ipv6 has live entries): an untagged IPv6 frame belongs to the owner of its source
// (bytes 22-37, upstream) or destination (38-53, downstream) address, v6_owner, and from there to that IPv4 address's
// directory slot.  In ACCT_ATTR mode only frames classify left unattributed read the frame, and only with verdict
// TC_ACT_OK: a pipeline's TC_ACT_SHOT IPv6 frame without an attribution word is antispoof's (a bucket drop has one,
// k_pipe_classify<V6>).  In the other modes a TC_ACT_SHOT IPv6 frame is a token-bucket drop of a qos program that
// shapes IPv6 (bng_qos_ipv6_enable); without shaping no program in these modes drops an IPv6 frame.
#include <errno.h>

#include "kernels.h"
#include "progs.cuh"

#define ACCT_BLOCK 256

// COUNT: add the frames to the counter records; STAMP: stamp the idle records.  <MODE, true, false> is accounting alone.
template <int MODE, bool COUNT, bool STAMP, bool V6>
__global__ void __launch_bounds__(ACCT_BLOCK) k_acct(const __grid_constant__ Tbl dir, const __grid_constant__ DevBatch b, const u32 *attr,
                                                      u64 *acct, u64 *idle, const __grid_constant__ Tbl v6) {
    const u32 lane = threadIdx.x & 31;
    __shared__ V6Lens lens;
    if (V6) v6_lens_load(lens, v6.plens);
    // warp-uniform trip count: __match_any_sync needs every lane
    for (u32 base = blockIdx.x * ACCT_BLOCK + (threadIdx.x & ~31u); base < b.n; base += gridDim.x * ACCT_BLOCK) {
        const u32 i = base + lane;
        u32 slot = DIR_NONE, len = 0, drop = 0;
        if (i < b.n) {
            const u8 v = b.verdict[i];
            if (v == TC_OK || (COUNT && v == TC_SHOT)) { // stamping alone: dropped frames are nobody's
                len = b.len[i];
                drop = v == TC_SHOT;
                if (MODE == ACCT_ATTR) {
                    slot = attr[i];
                } else {
                    // untagged IPv4 with the address's four bytes present: the source (26-29) as the frame entered,
                    // or the destination (30-33) as it leaves
                    const u32 off = MODE == ACCT_SRC ? 26 : 30;
                    const u8 *p = frame_ptr(b, i);
                    if (frame_dlen(b, len) >= off + 4 && rd16(p, 12) == ETH_P_IP_LE) slot = dir_slot_of(dir, rd32(p, off));
                }
                if (V6 && slot == DIR_NONE && (MODE != ACCT_ATTR || v == TC_OK)) { // untagged IPv6, its sixteen address bytes present
                    const u32 off = MODE == ACCT_DST ? 38 : 22;
                    const u8 *p = frame_ptr(b, i);
                    u32 a[4], owner;
                    if (frame_dlen(b, len) >= off + 16 && rd16(p, 12) == ETH_P_IPV6_LE) {
                        v6_addr(p, off, a);
                        if (v6_owner(v6, lens, a, &owner)) slot = dir_slot_of(dir, owner);
                    }
                }
            }
        }
        const bool has = slot != DIR_NONE;
        const u32 grp = has ? (slot << 1 | drop) : (0xFFFFFFE0u | lane); // (directory slots < 2^31 - 16)
        const u32 peers = __match_any_sync(0xffffffffu, grp);
        u64 bytes = len;
        u64 last = 0; // STAMP: the latest clock of the lane's group of passed frames
        if (STAMP && has && !drop) last = frame_now(b, i);
        if (!__all_sync(0xffffffffu, peers == (1u << lane))) { // some lanes share a record: sum each group
            if (COUNT) bytes = 0;
#pragma unroll
            for (int j = 0; j < 32; j++) {
                if (COUNT) {
                    const u32 lj = __shfl_sync(0xffffffffu, len, j);
                    if ((peers >> j) & 1) bytes += lj;
                }
                if (STAMP && b.nowv) { // (one clock per batch: every lane already holds it)
                    const u64 tj = __shfl_sync(0xffffffffu, last, j);
                    if (((peers >> j) & 1) && tj > last) last = tj;
                }
            }
        }
        if (has && lane == (u32)__ffs(peers) - 1) {
            if (COUNT) {
                u64 *r = acct + (size_t)slot * ACCT_WORDS + (MODE == ACCT_DST ? 4 : 0) + 2 * drop;
                atomicAdd((unsigned long long *)r, (unsigned long long)__popc(peers));
                atomicAdd((unsigned long long *)(r + 1), (unsigned long long)bytes);
            }
            if (STAMP && !drop) {
                u64 *w = idle + (size_t)slot * IDLE_WORDS + (MODE == ACCT_DST ? IDLE_DOWN : IDLE_UP);
                const u64 v = (last < ~0ull ? last : ~0ull - 1) + 1; // clock + 1: 0 is "none"
                // a stale read can only be lower than the stamp (stamps only rise within a launch): no atomic is lost
                if (b.nowv || *w < v) atomicMax((unsigned long long *)w, (unsigned long long)v);
            }
        }
    }
}

__global__ void k_acct_read(const __grid_constant__ Tbl dir, const u64 *acct, const u32 *addrs, u64 n, u64 *out, int *results) {
    for (u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        const u32 s = dir_slot_of(dir, addrs[i]);
        u64 *o = out + i * ACCT_WORDS;
#pragma unroll
        for (int j = 0; j < ACCT_WORDS; j++) o[j] = (s != DIR_NONE && acct) ? acct[(size_t)s * ACCT_WORDS + j] : 0;
        results[i] = s != DIR_NONE ? 0 : -ENOENT;
    }
}

// one atomic per warp on the output count: the interim-update sweep reads 10^5 - 10^6 records at once
__global__ void k_acct_dump(const __grid_constant__ Tbl dir, const u64 *acct, u32 *addrs_out, u64 *out, u32 *count, u64 cap) {
    const u64 slots = (u64)dir.mask + 1;
    const u32 lane = threadIdx.x & 31;
    for (u64 base = blockIdx.x * (u64)blockDim.x + (threadIdx.x & ~31u); base < slots; base += (u64)gridDim.x * blockDim.x) {
        const u64 i = base + lane;
        const u64 k = i < slots ? *(const u64 *)(dir.slots + i * 16) : K_EMPTY;
        const bool live = k < K_BUSY;
        const u32 m = __ballot_sync(0xffffffffu, live);
        if (!m) continue;
        u32 pos = 0;
        if (lane == 0) pos = atomicAdd(count, (u32)__popc(m));
        pos = __shfl_sync(0xffffffffu, pos, 0) + __popc(m & ((1u << lane) - 1));
        if (!live || pos >= cap) continue;
        addrs_out[pos] = (u32)k;
        u64 *o = out + (u64)pos * ACCT_WORDS;
#pragma unroll
        for (int j = 0; j < ACCT_WORDS; j++) o[j] = acct ? acct[i * ACCT_WORDS + j] : 0;
    }
}

__global__ void k_acct_load(const __grid_constant__ Tbl dir, u64 *acct, const u32 *addrs, const u64 *recs, u64 n) {
    for (u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        const u32 s = dir_slot_of(dir, addrs[i]);
        if (s == DIR_NONE) continue;
#pragma unroll
        for (int j = 0; j < ACCT_WORDS; j++) acct[(size_t)s * ACCT_WORDS + j] = recs[i * ACCT_WORDS + j];
    }
}

static inline int acct_grid(const Launcher &L, u64 n, int per_sm) {
    const u64 want = (n + ACCT_BLOCK - 1) / ACCT_BLOCK, cap = (u64)L.num_sms * per_sm;
    return (int)(want < 1 ? 1 : (want < cap ? want : cap));
}

// (COUNT, STAMP) is (1, 1), (1, 0) or (0, 1): at least one of acct and idle is given
template <int MODE, bool V6>
static void launch_acct(Launcher &L, int grid, const Tbl &dir, const DevBatch &b, const u32 *attr, u64 *acct, u64 *idle, const Tbl &v6) {
    auto *k = acct && idle ? k_acct<MODE, true, true, V6> : acct ? k_acct<MODE, true, false, V6> : k_acct<MODE, false, true, V6>;
    k<<<grid, ACCT_BLOCK, 0, L.stream>>>(dir, b, attr, acct, idle, v6);
}

static std::string acct_name(bool v6) { return std::string("k_acct") + (v6 ? "<v6>" : ""); }

cudaError_t run_acct(Launcher &L, const Tbl &dir, const DevBatch &b, int mode, u64 *acct, u64 *idle, const Tbl *v6) {
    const int grid = acct_grid(L, b.n, 8);
    with_flags(
        [&](auto attr6) {
            constexpr bool V6 = decltype(attr6)::value;
            const Tbl t = V6 ? *v6 : Tbl{};
            prof_begin(L, prof_name<acct_name, V6>());
            if (mode == ACCT_ATTR)
                launch_acct<ACCT_ATTR, V6>(L, grid, dir, b, L.acct_attr, acct, idle, t);
            else if (mode == ACCT_SRC)
                launch_acct<ACCT_SRC, V6>(L, grid, dir, b, nullptr, acct, idle, t);
            else
                launch_acct<ACCT_DST, V6>(L, grid, dir, b, nullptr, acct, idle, t);
        },
        v6 != nullptr);
    prof_end(L);
    L.launches++;
    return cudaGetLastError();
}

cudaError_t run_acct_read(Launcher &L, const Tbl &dir, const u64 *acct, const u32 *addrs, u64 n, u64 *out, int *results) {
    if (n == 0) return cudaSuccess;
    k_acct_read<<<acct_grid(L, n, 8), ACCT_BLOCK, 0, L.stream>>>(dir, acct, addrs, n, out, results);
    L.launches++;
    return cudaGetLastError();
}

cudaError_t run_acct_dump(Launcher &L, const Tbl &dir, const u64 *acct, u32 *addrs_out, u64 *out, u32 *count, u64 cap) {
    prof_begin(L, "k_acct_dump");
    k_acct_dump<<<acct_grid(L, (u64)dir.mask + 1, 8), ACCT_BLOCK, 0, L.stream>>>(dir, acct, addrs_out, out, count, cap);
    prof_end(L);
    L.launches++;
    return cudaGetLastError();
}

cudaError_t run_acct_load(Launcher &L, const Tbl &dir, u64 *acct, const u32 *addrs, const u64 *recs, u64 n) {
    if (n == 0) return cudaSuccess;
    k_acct_load<<<acct_grid(L, n, 8), ACCT_BLOCK, 0, L.stream>>>(dir, acct, addrs, recs, n);
    L.launches++;
    return cudaGetLastError();
}
