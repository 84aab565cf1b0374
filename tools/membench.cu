// Micro-benchmark of the access patterns the dataplane kernels are made of, to
// calibrate what "HBM roofline" means for gather-bound integer work on H100:
//   seq       coalesced 16 B/thread streaming read                      (copy-like)
//   hdr       each thread reads G contiguous bytes at a stride of S bytes (frame headers in an IMIX arena)
//   gather    each thread reads G bytes at R independent pseudo-random slots of a big table
//   chain     gather with a dependent chain of D steps (probe -> value -> ...)
//   red       each thread issues atomicAdd(u64) to a pseudo-random slot
// Prints GB/s of useful bytes and M accesses/s.  Build: nvcc -O3 -gencode arch=compute_90a,code=sm_90a
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

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

int main() {
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
