// bng_b200 — lawful intercept: content-of-communication capture (bng_li_*, include/bng_b200.h).
//
// Separate passes on the context's stream, launched only when a target is set and the program captures (ctx.cu):
//   - upstream, k_li_capture<true> BEFORE the program: the source address as the frame entered is probed in the
//     target set; a warp reserves the ring slots of its matches with one atomic, copies the frames as they are (before
//     SNAT) and lists (frame, slot) in the match list.  The record's verdict byte says LI_VOID until
//   - k_li_verdict, AFTER the program, walks only the match list and writes each record's verdict, or leaves it void
//     when the frame is not captured after all (a pipeline frame antispoof dropped: a SHOT frame without an
//     attribution word from classify);
//   - downstream, k_li_capture<false> AFTER the program: the destination address it leaves with, the frame as the
//     program left it (after DNAT), the verdict: complete records in one pass (the shape of k_acct<ACCT_DST>).
// The target set is a few KB at most (<= BNG_LI_MAX_TARGETS addresses at load <= 1/2): its probes stay in L1 / L2.
// V6 (launched only while subscriber_ipv6 has live entries): an untagged IPv6 frame is captured for the owner of its
// source (bytes 22-37, upstream) or destination (38-53, downstream), v6_owner; that IPv4 address is probed in the target
// set and goes into the record.  Downstream a TC_ACT_OK or TC_ACT_SHOT frame is attributed, as an IPv4 one is (SHOT:
// a token-bucket drop of qos_egress_prog shaping IPv6, bng_qos_ipv6_enable; no other downstream program drops an IPv6
// frame).  Upstream k_li_verdict voids a SHOT one in a pipeline unless classify attributed it (a bucket drop), so an
// antispoof drop stays uncaptured.
#include "kernels.h"
#include "progs.cuh"

#define LI_BLOCK 256

__device__ __forceinline__ int li_find(const AddrSet &t, u32 addr) {
    u32 i = aset_home(addr, t.mask);
    for (;;) {
        const u64 w = __ldg(t.words + i);
        if (!w) return -1;
        if ((u32)w == addr) return (int)i;
        i = (i + 1) & t.mask;
    }
}

// the first n (< 16) bytes of a word group, the rest zero
__device__ __forceinline__ u32 li_keep(u32 w, u32 lo, u32 n) { return n >= lo + 4 ? w : (n <= lo ? 0u : w & ((1u << (8 * (n - lo))) - 1)); }

// bytes [off, off + 16) of a capture of cap_len bytes: from the frame `p` below `split`, from `tail` above; zero past
// cap_len.  A frame's storage is readable up to the next multiple of 16 bytes, so whole units may be loaded.
__device__ __forceinline__ uint4 li_unit(const u8 *p, const u8 *tail, u32 split, u32 cap_len, u32 off, bool aligned) {
    uint4 w = make_uint4(0, 0, 0, 0);
    if (off >= cap_len) return w;
    const u8 *s = (off < split ? p : tail) + off;
    const u32 n = cap_len - off;
    if (aligned) {
        w = *(const uint4 *)s;
        if (n < 16) w = make_uint4(li_keep(w.x, 0, n), li_keep(w.y, 4, n), li_keep(w.z, 8, n), li_keep(w.w, 12, n));
    } else {
#pragma unroll
        for (u32 k = 0; k < 16; k++) {
            const u32 v = k < n ? (u32)s[k] << (8 * (k & 3)) : 0u;
            if (k < 4) w.x |= v;
            else if (k < 8) w.y |= v;
            else if (k < 12) w.z |= v;
            else w.w |= v;
        }
    }
    return w;
}

template <bool UP, bool V6>
__global__ void __launch_bounds__(LI_BLOCK) k_li_capture(const __grid_constant__ LiRing r, const __grid_constant__ DevBatch b,
                                                         const __grid_constant__ LiSrc src, const __grid_constant__ Tbl v6) {
    const u32 lane = threadIdx.x & 31, below = (1u << lane) - 1;
    __shared__ V6Lens lens;
    if (V6) v6_lens_load(lens, v6.plens);
    const u32 units = (r.rec_bytes - LI_HDR) / 16;
    // warp-uniform trip count: the ballots and the cooperative copy need every lane
    for (u32 base = blockIdx.x * LI_BLOCK + (threadIdx.x & ~31u); base < b.n; base += gridDim.x * LI_BLOCK) {
        const u32 i = base + lane;
        int t = -1;
        u32 len = 0, have = 0, addr = 0;
        u8 v = 0;
        const u8 *p = b.pkts;
        if (i < b.n) {
            len = b.len[i];
            // bytes present in the frame's storage: the caller's layout, not the compact copy's
            have = src.arena ? ((src.off16 || len <= src.stride) ? len : src.stride) : frame_dlen(b, len);
            p = frame_ptr(b, i);
            const u32 off = UP ? 26 : 30;
            if (!UP) v = b.verdict[i];
            if ((UP || v == TC_OK || v == TC_SHOT) && have >= off + 4 && rd16(p, 12) == ETH_P_IP_LE) {
                addr = rd32(p, off);
                t = li_find(r.tgt, addr);
            } else if (V6 && (UP || v == TC_OK || v == TC_SHOT) && have >= (UP ? 38u : 54u) && rd16(p, 12) == ETH_P_IPV6_LE) {
                u32 a[4];
                v6_addr(p, UP ? 22 : 38, a);
                if (v6_owner(v6, lens, a, &addr)) t = li_find(r.tgt, addr);
            }
        }
        const u32 m = __ballot_sync(0xffffffffu, t >= 0);
        if (!m) continue;
        const int lead = __ffs(m) - 1;
        unsigned long long first = 0;
        if (lane == (u32)lead) first = atomicAdd((unsigned long long *)r.ctl, (unsigned long long)__popc(m));
        first = __shfl_sync(0xffffffffu, first, lead);
        const u64 pos = first + __popc(m & below);
        const bool hit = t >= 0, kept = hit && pos < r.cap;
        if (UP) { // the verdict pass needs every match, kept or not: whether a lost one counts depends on the verdict
            u32 mi = 0;
            if (lane == (u32)lead) mi = atomicAdd((u32 *)(r.ctl + 2), (u32)__popc(m));
            mi = __shfl_sync(0xffffffffu, mi, lead) + __popc(m & below);
            if (hit) r.match[mi] = make_uint2(i, kept ? (u32)pos : LI_NOSLOT);
        } else {
            const u32 lost = __ballot_sync(0xffffffffu, hit && !kept);
            if (lost && lane == (u32)(__ffs(lost) - 1)) atomicAdd((unsigned long long *)(r.ctl + 1), (unsigned long long)__popc(lost));
        }
        const u32 cap_len = min(min(len, have), r.snaplen);
        u8 *rec = kept ? r.buf + pos * r.rec_bytes : nullptr;
        const u8 *tail = nullptr;
        u32 split = 0xFFFFFFFFu;
        if (kept) {
            if (src.arena) {
                tail = src.arena + (src.off16 ? (size_t)src.off16[i] * 16 : (size_t)i * src.stride);
                if (src.need) split = (src.need[i] + 15u) & ~15u;
            }
            const u64 ts = frame_now(b, i);
            uint4 *h = (uint4 *)rec;
            h[0] = make_uint4((u32)ts, (u32)(ts >> 32), (u32)r.batch, (u32)(r.batch >> 32));
            h[1] = make_uint4(b.base + i, r.ids[t], addr, len);
            h[2] = make_uint4(cap_len, (UP ? 0u : 1u) /* BNG_LI_UPLINK / DOWNLINK */ |(u32)(UP ? LI_VOID : v) << 8 | r.prog << 16, 0, 0);
            h[3] = make_uint4(0, 0, 0, 0);
        }
        // the payloads of the warp's records, one record at a time, 16 bytes per lane
        u32 wm = __ballot_sync(0xffffffffu, kept);
        while (wm) {
            const int j = __ffs(wm) - 1;
            wm &= wm - 1;
            u8 *rj = (u8 *)__shfl_sync(0xffffffffu, (unsigned long long)rec, j);
            const u8 *pj = (const u8 *)__shfl_sync(0xffffffffu, (unsigned long long)p, j);
            const u8 *tj = (const u8 *)__shfl_sync(0xffffffffu, (unsigned long long)tail, j);
            const u32 sj = __shfl_sync(0xffffffffu, split, j), cj = __shfl_sync(0xffffffffu, cap_len, j);
            const bool aligned = (((uintptr_t)pj | (uintptr_t)tj) & 15) == 0;
            for (u32 u = lane; u < units; u += 32) *(uint4 *)(rj + LI_HDR + u * 16) = li_unit(pj, tj, sj, cj, u * 16, aligned);
        }
    }
}

__global__ void __launch_bounds__(LI_BLOCK) k_li_verdict(const __grid_constant__ LiRing r, const __grid_constant__ DevBatch b, const u32 *attr) {
    const u32 n = *(const u32 *)(r.ctl + 2);
    u32 lost = 0;
    for (u32 k = blockIdx.x * LI_BLOCK + threadIdx.x; k < n; k += gridDim.x * LI_BLOCK) {
        const uint2 mt = r.match[k];
        const u8 v = b.verdict[mt.x];
        const bool keep = (v == TC_OK || v == TC_SHOT) && !(attr && v == TC_SHOT && attr[mt.x] == DIR_NONE);
        if (mt.y != LI_NOSLOT) {
            if (keep) r.buf[(size_t)mt.y * r.rec_bytes + 37] = v; // bng_li_record.verdict
        } else {
            lost += keep;
        }
    }
    if (lost) atomicAdd((unsigned long long *)(r.ctl + 1), (unsigned long long)lost);
}

static inline int li_grid(const Launcher &L, u64 n, int per_sm) {
    const u64 want = (n + LI_BLOCK - 1) / LI_BLOCK, cap = (u64)L.num_sms * per_sm;
    return (int)(want < 1 ? 1 : (want < cap ? want : cap));
}

static std::string li_name(bool up, bool v6) { return std::string("k_li_capture<") + (up ? "up" : "down") + (v6 ? ",v6" : "") + ">"; }

cudaError_t run_li_capture(Launcher &L, const LiRing &r, const DevBatch &b, const LiSrc &src, bool up, const Tbl *v6) {
    const int grid = li_grid(L, b.n, 8);
    with_flags(
        [&](auto upf, auto attr6) {
            constexpr bool UP = decltype(upf)::value, V6 = decltype(attr6)::value;
            prof_begin(L, prof_name<li_name, UP, V6>());
            k_li_capture<UP, V6><<<grid, LI_BLOCK, 0, L.stream>>>(r, b, src, V6 ? *v6 : Tbl{});
        },
        up, v6 != nullptr);
    prof_end(L);
    L.launches++;
    return cudaGetLastError();
}

cudaError_t run_li_verdict(Launcher &L, const LiRing &r, const DevBatch &b, const u32 *attr) {
    prof_begin(L, "k_li_verdict");
    k_li_verdict<<<li_grid(L, b.n, 2), LI_BLOCK, 0, L.stream>>>(r, b, attr);
    prof_end(L);
    L.launches++;
    return cudaGetLastError();
}
