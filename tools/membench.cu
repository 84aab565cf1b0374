// Micro-benchmark of the access patterns the dataplane kernels are made of, to
// calibrate what "HBM roofline" means for gather-bound integer work on H100:
//   seq       coalesced 16 B/thread streaming read                      (copy-like)
//   hdr       each thread reads G contiguous bytes at a stride of S bytes (frame headers in an IMIX arena)
//   gather    each thread reads G bytes at R independent pseudo-random slots of a big table
//   chain     gather with a dependent chain of D steps (probe -> value -> ...)
//   red       each thread issues atomicAdd(u64) to a pseudo-random slot
// Prints GB/s of useful bytes and M accesses/s.  Build: nvcc -O3 -gencode arch=compute_90a,code=sm_90a
//
// `membench lanes` instead compares, at classify's shapes (2^22 IMIX frames placed like workloads.slot16, a
// 2^21 x 128-byte table, SMs x 3 blocks of 256), per-lane accesses with the same bytes read by several lanes:
//   hdr       each lane reads its frame's 64-byte header as 4 x 16 B       (32 lines per warp instruction)
//   hdrq      4 lanes per frame, one 16-byte chunk each, 8 frames per instruction, transposed through shared memory
//   hdr+wb    hdr, then the header stored back whole; hdrq+wb the same through the shared rounds
//   probe     each lane reads a random 32-byte slot as 2 x 16 B
//   pair      lanes (2k, 2k+1) read slot 2k, then slot 2k+1, 16 B each, and swap halves with __shfl_xor_sync
//   ... in L2 hdr, hdrq, probe and pair over a footprint that stays in L2, so that DRAM does not bound them
// The forms run alternated, in rounds, and each line reports the range over the rounds.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

typedef unsigned long long u64;
typedef uint32_t u32;

__device__ __forceinline__ u32 hmix(u32 x) {
    x ^= x >> 16;
    x *= 0x7feb352du;
    x ^= x >> 15;
    x *= 0x846ca68bu;
    x ^= x >> 16;
    return x;
}

__global__ void k_seq(const uint4 *__restrict__ p, u64 n16, u32 *sink) {
    u32 acc = 0;
    for (u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x; i < n16; i += (u64)gridDim.x * blockDim.x) {
        uint4 v = p[i];
        acc ^= v.x ^ v.y ^ v.z ^ v.w;
    }
    if (acc == 0x12345) *sink = acc;
}

template <int CH> // CH 16-byte chunks per thread at stride16 16-byte units
__global__ void k_hdr(const uint4 *__restrict__ p, u32 n, u32 stride16, u32 *sink) {
    u32 acc = 0;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint4 *q = p + (u64)i * stride16;
#pragma unroll
        for (int c = 0; c < CH; c++) {
            uint4 v = q[c];
            acc ^= v.x ^ v.w;
        }
    }
    if (acc == 0x12345) *sink = acc;
}

template <int R, int G16> // R independent random slots of G16*16 bytes, slot size = slot16*16 bytes
__global__ void k_gather(const uint4 *__restrict__ t, u32 n, u32 mask, u32 slot16, u32 *sink) {
    u32 acc = 0;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        uint4 v[R][G16];
#pragma unroll
        for (int r = 0; r < R; r++) {
            u32 s = hmix(i * R + r) & mask;
#pragma unroll
            for (int g = 0; g < G16; g++) v[r][g] = t[(u64)s * slot16 + g];
        }
#pragma unroll
        for (int r = 0; r < R; r++)
#pragma unroll
            for (int g = 0; g < G16; g++) acc ^= v[r][g].x ^ v[r][g].w;
    }
    if (acc == 0x12345) *sink = acc;
}

template <int D>
__global__ void k_chain(const uint4 *__restrict__ t, u32 n, u32 mask, u32 slot16, u32 *sink) {
    u32 acc = 0;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        u32 s = hmix(i) & mask;
#pragma unroll
        for (int d = 0; d < D; d++) {
            uint4 v = t[(u64)s * slot16];
            s = hmix(s ^ v.x ^ (u32)d) & mask;
        }
        acc ^= s;
    }
    if (acc == 0x12345) *sink = acc;
}

__global__ void k_red(u64 *t, u32 n, u32 mask, u32 slot8) {
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        u32 s = hmix(i) & mask;
        atomicAdd(&t[(u64)s * slot8], 1ull);
    }
}

// cp.async (LDGSTS) variant of the gather: R x 16 B per thread into shared memory, two tiles in flight
template <int R>
__global__ void k_gather_async(const uint4 *__restrict__ t, u32 n, u32 mask, u32 slot16, u32 *sink) {
    extern __shared__ uint4 sm[]; // [2][R][blockDim]
    u32 acc = 0;
    u32 stride = gridDim.x * blockDim.x;
    u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    int buf = 0;
    auto issue = [&](u32 idx, int b) {
#pragma unroll
        for (int r = 0; r < R; r++) {
            u32 s = hmix(idx * R + r) & mask;
            u32 dst = (u32)__cvta_generic_to_shared(&sm[(b * R + r) * blockDim.x + threadIdx.x]);
            const uint4 *src = t + (u64)s * slot16;
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src));
        }
        asm volatile("cp.async.commit_group;");
    };
    if (i < n) issue(i, 0);
    for (; i < n; i += stride) {
        u32 nx = i + stride;
        if (nx < n) {
            issue(nx, buf ^ 1);
            asm volatile("cp.async.wait_group 1;");
        } else {
            asm volatile("cp.async.wait_group 0;");
        }
#pragma unroll
        for (int r = 0; r < R; r++) {
            uint4 v = sm[(buf * R + r) * blockDim.x + threadIdx.x];
            acc ^= v.x ^ v.w;
        }
        buf ^= 1;
    }
    if (acc == 0x12345) *sink = acc;
}

// ---- `lanes`: classify's header and probe accesses, per lane and shared across lanes ----
#define FULL 0xffffffffu
template <bool WB>
__global__ void k_hdr_lane(uint4 *p, const u32 *__restrict__ off16, u32 n, u32 fmask, u32 *sink) {
    u32 acc = 0;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        uint4 *q = p + off16[i & fmask];
        uint4 v[4];
#pragma unroll
        for (int c = 0; c < 4; c++) v[c] = q[c];
#pragma unroll
        for (int c = 0; c < 4; c++) acc ^= v[c].x ^ v[c].w;
        if (WB) {
            v[0].y ^= acc & 0x100u; // data-dependent, so the store waits for the load as classify's does
#pragma unroll
            for (int c = 0; c < 4; c++) q[c] = v[c];
        }
    }
    if (acc == 0x12345) *sink = acc;
}

// row f of a warp's 32 x 64-byte buffer, chunk c: XOR-swizzled so that neither the round stores (8 lanes = 2 rows x 4
// chunks per phase) nor the row loads (8 lanes = 8 rows x 1 chunk) conflict on banks
__device__ __forceinline__ uint4 &sw(uint4 (*buf)[4], u32 f, u32 c) { return buf[f][c ^ ((f >> 1) & 3)]; }

template <bool WB>
__global__ void k_hdr_quad(uint4 *p, const u32 *__restrict__ off16, u32 n, u32 fmask, u32 *sink) {
    __shared__ uint4 sm[8][32][4];
    uint4(*buf)[4] = sm[threadIdx.x >> 5];
    const u32 lane = threadIdx.x & 31, c = lane & 3;
    u32 acc = 0;
    for (u32 base = blockIdx.x * blockDim.x + (threadIdx.x & ~31u); base < n; base += gridDim.x * blockDim.x) {
        const u32 o = base + lane < n ? off16[(base + lane) & fmask] : 0;
        u32 fo[4];
#pragma unroll
        for (int r = 0; r < 4; r++) {
            const u32 f = 8 * r + (lane >> 2);
            fo[r] = __shfl_sync(FULL, o, f);
            uint4 v = make_uint4(0, 0, 0, 0);
            if (base + f < n) v = p[(u64)fo[r] + c];
            sw(buf, f, c) = v;
        }
        __syncwarp();
        uint4 h[4];
#pragma unroll
        for (int k = 0; k < 4; k++) h[k] = sw(buf, lane, k);
#pragma unroll
        for (int k = 0; k < 4; k++) acc ^= h[k].x ^ h[k].w;
        if (WB) {
            h[0].y ^= acc & 0x100u;
            __syncwarp();
#pragma unroll
            for (int k = 0; k < 4; k++) sw(buf, lane, k) = h[k];
            __syncwarp();
#pragma unroll
            for (int r = 0; r < 4; r++) {
                const u32 f = 8 * r + (lane >> 2);
                if (base + f < n) p[(u64)fo[r] + c] = sw(buf, f, c);
            }
        }
        __syncwarp();
    }
    if (acc == 0x12345) *sink = acc;
}

template <bool PAIR>
__global__ void k_probe32(const uint4 *__restrict__ t, u32 n, u32 mask, u32 slot16, u32 *sink) {
    const u32 lane = threadIdx.x & 31;
    u32 acc = 0;
    for (u32 base = blockIdx.x * blockDim.x + (threadIdx.x & ~31u); base < n; base += gridDim.x * blockDim.x) {
        const u32 s = hmix(base + lane) & mask;
        uint4 h0, h1;
        if (PAIR) {
            const u32 odd = lane & 1;
            const u32 s0 = __shfl_sync(FULL, s, lane & ~1u), s1 = __shfl_sync(FULL, s, lane | 1u);
            const uint4 a = t[(u64)s0 * slot16 + odd], b = t[(u64)s1 * slot16 + odd];
            uint4 x = odd ? a : b;
            x.x = __shfl_xor_sync(FULL, x.x, 1);
            x.y = __shfl_xor_sync(FULL, x.y, 1);
            x.z = __shfl_xor_sync(FULL, x.z, 1);
            x.w = __shfl_xor_sync(FULL, x.w, 1);
            h0 = odd ? x : a;
            h1 = odd ? b : x;
        } else {
            h0 = t[(u64)s * slot16];
            h1 = t[(u64)s * slot16 + 1];
        }
        acc ^= h0.x ^ h1.w ^ (h0.w + h1.x);
    }
    if (acc == 0x12345) *sink = acc;
}

// off16 of n frames with IMIX 7:4:1 lengths (64 / 594 / 1518 B) placed on `align`-byte boundaries
static u32 imix_layout(u32 *off16, u32 n, u32 align) {
    u64 x = 0x2545F4914F6CDD1Dull, cur = 0;
    for (u32 i = 0; i < n; i++) {
        x ^= x << 13, x ^= x >> 7, x ^= x << 17;
        const u32 w = (u32)(x % 12), len = w < 7 ? 64 : w < 11 ? 594 : 1518;
        off16[i] = (u32)cur;
        cur += (len + align - 1) / align * (align / 16);
    }
    return (u32)cur;
}

static int lanes(uint4 *buf, u64 bytes, u32 *sink, int sms) {
    const u32 n = 1u << 22, grid = sms * 3, blk = 256, rounds = 5, reps = 20;
    u32 *h16 = (u32 *)malloc(n * 4ull), *off64, *off16;
    cudaMalloc(&off64, n * 4ull);
    cudaMalloc(&off16, n * 4ull);
    const u32 g64 = imix_layout(h16, n, 64);
    cudaMemcpy(off64, h16, n * 4ull, cudaMemcpyHostToDevice);
    const u32 g16 = imix_layout(h16, n, 16);
    cudaMemcpy(off16, h16, n * 4ull, cudaMemcpyHostToDevice);
    free(h16);
    if ((u64)g64 * 16 + 64 > bytes) return 1;
    const u32 tmask = (1u << 21) - 1; // 2^21 x 128-byte table (256 MB), the first 32-byte sector of a slot
    // the "in L2" lines: the frame index or the slot wraps at 2^15 (the first 32 k frames span 12 MB at align 64;
    // 2^15 slots of 128 B are 4 MB), so after the first pass the same accesses hit in L2 and DRAM drops out
    const u32 l2mask = (1u << 15) - 1;
    printf("--- lanes: %u frames (arena %.2f GB at align 64, %.2f GB at align 16), grid %u x %u, %u rounds of %u launches\n",
           n, g64 * 16e-9, g16 * 16e-9, grid, blk, rounds, reps);
    enum { M = 14 };
    const char *label[M] = {"hdr        align 64", "hdrq       align 64", "hdr        align 16", "hdrq       align 16",
                            "hdr+wb     align 64", "hdrq+wb    align 64", "hdr+wb     align 16", "hdrq+wb    align 16",
                            "probe 32 B per lane", "pair  32 B, 2 lanes", "hdr        in L2", "hdrq       in L2",
                            "probe      in L2", "pair       in L2"};
    float lo[M], hi[M], sum[M];
    for (int m = 0; m < M; m++) lo[m] = 1e30f, hi[m] = 0, sum[m] = 0;
    cudaEvent_t a, b;
    cudaEventCreate(&a);
    cudaEventCreate(&b);
    for (u32 round = 0; round < rounds; round++) {
        for (int m = 0; m < M; m++) {
            const u32 *o = (m & 2) ? off16 : off64;
            auto launch = [&]() {
                switch (m) {
                case 0: case 2: k_hdr_lane<false><<<grid, blk>>>(buf, o, n, FULL, sink); break;
                case 1: case 3: k_hdr_quad<false><<<grid, blk>>>(buf, o, n, FULL, sink); break;
                case 4: case 6: k_hdr_lane<true><<<grid, blk>>>(buf, o, n, FULL, sink); break;
                case 5: case 7: k_hdr_quad<true><<<grid, blk>>>(buf, o, n, FULL, sink); break;
                case 8: k_probe32<false><<<grid, blk>>>(buf, n, tmask, 8, sink); break;
                case 9: k_probe32<true><<<grid, blk>>>(buf, n, tmask, 8, sink); break;
                case 10: k_hdr_lane<false><<<grid, blk>>>(buf, off64, n, l2mask, sink); break;
                case 11: k_hdr_quad<false><<<grid, blk>>>(buf, off64, n, l2mask, sink); break;
                case 12: k_probe32<false><<<grid, blk>>>(buf, n, l2mask, 8, sink); break;
                default: k_probe32<true><<<grid, blk>>>(buf, n, l2mask, 8, sink); break;
                }
            };
            launch();
            cudaEventRecord(a);
            for (u32 k = 0; k < reps; k++) launch();
            cudaEventRecord(b);
            cudaEventSynchronize(b);
            float ms;
            cudaEventElapsedTime(&ms, a, b);
            ms /= reps;
            lo[m] = ms < lo[m] ? ms : lo[m];
            hi[m] = ms > hi[m] ? ms : hi[m];
            sum[m] += ms;
        }
    }
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) {
        printf("CUDA error: %s\n", cudaGetErrorString(e));
        return 1;
    }
    printf("%-22s %10s %10s %10s %12s\n", "form", "min ms", "max ms", "mean ms", "M frames/s");
    for (int m = 0; m < M; m++)
        printf("%-22s %10.4f %10.4f %10.4f %12.0f\n", label[m], lo[m], hi[m], sum[m] / rounds, n / (sum[m] / rounds) / 1e3);
    return 0;
}

static float timeit(void (*launch)(void *), void *arg, int reps) {
    cudaEvent_t a, b;
    cudaEventCreate(&a);
    cudaEventCreate(&b);
    launch(arg);
    cudaDeviceSynchronize();
    cudaEventRecord(a);
    for (int i = 0; i < reps; i++) launch(arg);
    cudaEventRecord(b);
    cudaEventSynchronize(b);
    float ms;
    cudaEventElapsedTime(&ms, a, b);
    return ms / reps;
}

struct Args {
    uint4 *buf;
    u64 bytes;
    u32 *sink;
    u32 n;
    int sms;
    int bps;
};

#define RUN(label, useful_bytes, accesses, ...)                                                    \
    do {                                                                                           \
        cudaEvent_t a, b;                                                                          \
        cudaEventCreate(&a);                                                                       \
        cudaEventCreate(&b);                                                                       \
        __VA_ARGS__;                                                                               \
        cudaDeviceSynchronize();                                                                   \
        cudaEventRecord(a);                                                                        \
        for (int rep = 0; rep < 5; rep++) { __VA_ARGS__; }                                         \
        cudaEventRecord(b);                                                                        \
        cudaEventSynchronize(b);                                                                   \
        float ms;                                                                                  \
        cudaEventElapsedTime(&ms, a, b);                                                           \
        ms /= 5;                                                                                   \
        printf("%-44s %8.3f ms  %8.1f GB/s useful  %8.1f M acc/s\n", label, ms,                    \
               (double)(useful_bytes) / ms / 1e6, (double)(accesses) / ms / 1e3);                  \
        cudaError_t e = cudaGetLastError();                                                        \
        if (e != cudaSuccess) printf("   CUDA error: %s\n", cudaGetErrorString(e));                \
    } while (0)

int main(int argc, char **argv) {
    cudaDeviceProp prop;
    cudaGetDeviceProperties(&prop, 0);
    int sms = prop.multiProcessorCount;
    printf("device %s, %d SMs\n", prop.name, sms);
    const u64 BYTES = 2ull << 30; // 2 GiB table / arena
    uint4 *buf;
    u32 *sink;
    cudaMalloc(&buf, BYTES);
    cudaMalloc(&sink, 64);
    cudaMemset(buf, 1, BYTES);
    if (argc > 1 && !strcmp(argv[1], "lanes")) return lanes(buf, BYTES, sink, sms);
    const u32 n = 1u << 22;
    for (int bps = 4; bps <= 8; bps += 4) {
        int grid = sms * bps, blk = 256;
        printf("--- grid %d x %d (%d blocks/SM)\n", grid, blk, bps);
        RUN("seq 16B/thread over 2 GiB", BYTES, BYTES / 16, (k_seq<<<grid, blk>>>(buf, BYTES / 16, sink)));
        RUN("hdr 64B @ stride 64B (4M frames)", (u64)n * 64, n, (k_hdr<4><<<grid, blk>>>(buf, n, 4, sink)));
        RUN("hdr 64B @ stride 368B (IMIX-like)", (u64)n * 64, n, (k_hdr<4><<<grid, blk>>>(buf, n, 23, sink)));
        RUN("hdr 32B @ stride 368B", (u64)n * 32, n, (k_hdr<2><<<grid, blk>>>(buf, n, 23, sink)));
        u32 mask32 = (u32)(BYTES / 32 - 1), mask64 = (u32)(BYTES / 64 - 1), mask128 = (u32)(BYTES / 128 - 1);
        RUN("gather R=1 x 16B (slot 32B, 2 GiB)", (u64)n * 16, n, (k_gather<1, 1><<<grid, blk>>>(buf, n, mask32, 2, sink)));
        RUN("gather R=1 x 32B", (u64)n * 32, n, (k_gather<1, 2><<<grid, blk>>>(buf, n, mask32, 2, sink)));
        RUN("gather R=4 x 32B", (u64)n * 4 * 32, n * 4ull, (k_gather<4, 2><<<grid, blk>>>(buf, n, mask32, 2, sink)));
        RUN("gather R=8 x 32B", (u64)n * 8 * 32, n * 8ull, (k_gather<8, 2><<<grid, blk>>>(buf, n, mask32, 2, sink)));
        RUN("gather R=4 x 64B (slot 64B)", (u64)n * 4 * 64, n * 4ull, (k_gather<4, 4><<<grid, blk>>>(buf, n, mask64, 4, sink)));
        RUN("gather R=2 x 128B (slot 128B)", (u64)n * 2 * 128, n * 2ull, (k_gather<2, 8><<<grid, blk>>>(buf, n, mask128, 8, sink)));
        RUN("chain D=4 x 16B (dependent)", (u64)n * 4 * 16, n * 4ull, (k_chain<4><<<grid, blk>>>(buf, n, mask32, 2, sink)));
        RUN("red atomicAdd u64 random (2 GiB)", (u64)n * 8, n, (k_red<<<grid, blk>>>((u64 *)buf, n, mask32, 4)));
        RUN("red atomicAdd u64 random (64 MiB)", (u64)n * 8, n,
            (k_red<<<grid, blk>>>((u64 *)buf, n, (u32)((64u << 20) / 32 - 1), 4)));
        RUN("cp.async gather R=4 x 16B, 2 tiles in flight", (u64)n * 4 * 16, n * 4ull,
            (k_gather_async<4><<<grid, blk, 2 * 4 * blk * 16>>>(buf, n, mask32, 2, sink)));
        RUN("cp.async gather R=8 x 16B, 2 tiles in flight", (u64)n * 8 * 16, n * 8ull,
            (k_gather_async<8><<<grid, blk, 2 * 8 * blk * 16>>>(buf, n, mask32, 2, sink)));
    }
    return 0;
}
