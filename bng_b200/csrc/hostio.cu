// bng_b200 — frame I/O for BNG_MEM_HOST batches whose arena is pinned host
// memory: instead of copying whole frames over PCIe, gather kernels read only
// the header bytes the programs can touch straight out of the mapped host
// arena (zero-copy, 16 bytes per lane, a frame's chunks on consecutive lanes so
// each frame is one contiguous PCIe read), the programs run on the compact
// device copy, and scatter kernels write the headers back in place.
//
// How many bytes can a program touch?  The TC programs (antispoof, QoS, NAT44, the pipeline) read at most
// the Ethernet + IPv4 header and 20 bytes of L4 header at 14 + ihl*4: 54 bytes when ihl = 5 — one 64-byte
// slot covers it — and up to 14 + 60 + 20 = 94 bytes when the header carries options (bpf/nat44.c:606-653,
// 752-798).  Compact slots are therefore 96 bytes apart.  The first min(len, 64) bytes of every frame are moved
// both ways, the two further 16-byte chunks only for frames whose ihl says the L4 header reaches them: the scatter
// writes back every chunk the gather moved.  With ICMP error translation on, nat44_ingress also reads the quoted ports
// and L4 checksums of an ICMP error, through byte 79: chunk 4 moves for those frames.  Chunk 0 included, although the TC programs write below byte 16 only
// in nat44_egress on a frame with ihl = 0 (its "TCP source port" is bytes 14-15): a single 64-byte PCIe write per
// frame costs less than the 48 bytes that can change sent as two.  dhcp_fastpath_prog touches up to 14 + 8 (QinQ)
// + 60 + 8 + 240 + 64 = 394 bytes and rewrites the Ethernet header: 448-byte slots, everything scattered back.
#include "kernels.h"

// dst[f][0..need) <- arena[off(f) .. off(f)+need); need[f] = bytes moved
// ICMPERR (TC, nat44_ingress with bng_nat_icmp_errors_enable): an ICMP error frame (ihl 5, protocol 1, type 3 / 11 /
// 12) longer than 64 bytes also moves chunk 4, bytes 64-79, where the quoted ports and L4 checksums end.  The frame's
// four lanes are consecutive lanes of one warp: lane 0 takes the protocol (byte 23) from lane 1 and the type (byte 34)
// from lane 2.
template <bool ICMPERR>
__global__ void __launch_bounds__(256) k_gather_frames(const u8 *__restrict__ arena, const u32 *__restrict__ off16,
                                                       const u32 *__restrict__ len, u32 stride, u32 n, u32 slot, u32 tc,
                                                       u8 *dst, u32 *need) {
    const u32 cpf = tc ? 4u : slot / 16; // lanes per frame (TC: the first 64 bytes; the option tail rides on lane 0)
    const u64 total = (u64)n * cpf;
    for (u64 t = blockIdx.x * (u64)blockDim.x + threadIdx.x; t < total; t += (u64)gridDim.x * blockDim.x) {
        const u32 f = (u32)(t / cpf), ch = (u32)(t % cpf);
        const u32 l = len[f];
        if (!ICMPERR && ch * 16 >= l) {
            if (ch == 0) need[f] = 0;
            continue;
        }
        const u8 *src = arena + (off16 ? (size_t)off16[f] * 16 : (size_t)f * stride);
        u8 *d = dst + (size_t)f * slot;
        uint4 v = make_uint4(0, 0, 0, 0);
        if (!ICMPERR || ch * 16 < l) {
            v = *(const uint4 *)(src + ch * 16);
            *(uint4 *)(d + ch * 16) = v;
        }
        u32 w23 = 0, w34 = 0; // bytes 20-23 and 32-35, for lane 0
        if (ICMPERR) {
            const u32 q = threadIdx.x & 28; // the frame's four lanes (tc: cpf = 4, t % 4 == threadIdx.x % 4)
            w23 = __shfl_sync(0xFu << q, v.y, q + 1);
            w34 = __shfl_sync(0xFu << q, v.x, q + 2);
            if (ch * 16 >= l) {
                if (ch == 0) need[f] = 0;
                continue;
            }
        }
        if (ch) continue;
        u32 nd = l < slot ? l : slot;
        if (tc) {
            nd = l < 64 ? l : 64;
            // bytes 12-13 ethertype, byte 14 version/ihl (all in chunk 0: v.w = bytes 12..15)
            const bool ip4 = l >= 34 && (v.w & 0xFFFFu) == 0x0008u;
            const u32 ihl = (v.w >> 16) & 0x0fu;
            if (ip4 && ihl > 5 && l > 64) { // options push the L4 header past byte 63: move the tail as well
                u32 want = 14 + ihl * 4 + 20;
                want = want < l ? want : l;
                for (u32 c = 4; c * 16 < want; c++) *(uint4 *)(d + c * 16) = *(const uint4 *)(src + c * 16);
                nd = want;
            } else if (ICMPERR && ip4 && ihl == 5 && l > 64 && (w23 >> 24) == 1) {
                const u32 type = (w34 >> 16) & 0xffu;
                if (type == 3 || type == 11 || type == 12) {
                    *(uint4 *)(d + 64) = *(const uint4 *)(src + 64);
                    nd = l < 80 ? l : 80;
                }
            }
        }
        need[f] = nd;
    }
}

// arena[off(f) .. ) <- dst[f][0..need): every chunk the gather moved
__global__ void __launch_bounds__(256) k_scatter_frames(u8 *__restrict__ arena, const u32 *__restrict__ off16,
                                                        const u32 *__restrict__ need, u32 stride, u32 n, u32 slot,
                                                        const u8 *__restrict__ src) {
    const u32 cpf = slot / 16;
    const u64 total = (u64)n * cpf;
    for (u64 t = blockIdx.x * (u64)blockDim.x + threadIdx.x; t < total; t += (u64)gridDim.x * blockDim.x) {
        const u32 f = (u32)(t / cpf), ch = (u32)(t % cpf);
        if (ch * 16 < need[f]) {
            u8 *d = arena + (off16 ? (size_t)off16[f] * 16 : (size_t)f * stride) + ch * 16;
            *(uint4 *)d = *(const uint4 *)(src + (size_t)f * slot + ch * 16);
        }
    }
}

// Both kernels are bound by PCIe, not by the SMs: one 256-thread block per SM keeps hundreds of KB of 16-byte
// accesses in flight, and leaves the SMs to the program kernels of the
// chunk in between.  What limits the pipeline is the link itself (BNG_ZC_TRACE=1 times the stages): the gather's
// read requests and the scatter's small write TLPs share the upstream direction.  Copy-engine traffic (a header-split ring, moved with cudaMemcpyAsync) overlaps cleanly.
cudaError_t run_gather_frames(cudaStream_t st, int blocks, const u8 *arena, const u32 *off16, const u32 *len, u32 stride,
                              u32 n, u32 slot, bool tc, bool icmp_errors, u8 *dst, u32 *need) {
    with_flags(
        [&](auto icmp) {
            k_gather_frames<decltype(icmp)::value><<<blocks, 256, 0, st>>>(arena, off16, len, stride, n, slot, tc ? 1u : 0u, dst, need);
        },
        tc && icmp_errors);
    return cudaGetLastError();
}

cudaError_t run_scatter_frames(cudaStream_t st, int blocks, u8 *arena, const u32 *off16, const u32 *need, u32 stride, u32 n,
                               u32 slot, const u8 *src) {
    k_scatter_frames<<<blocks, 256, 0, st>>>(arena, off16, need, stride, n, slot, src);
    return cudaGetLastError();
}
