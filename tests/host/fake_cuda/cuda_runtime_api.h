// A stand-in for the CUDA runtime API, enough for bng_b200/csrc/devbuf.hpp and stage.hpp on a machine without CUDA:
// allocations come from the host heap, the Nth one, the Nth copy or a stream synchronisation can be made to fail, and
// the last error, the live allocations and the copies by direction are tracked (tests/host/test_devbuf_host.cpp,
// tests/host/test_stage_host.cpp).
#pragma once
#include <cstddef>
#include <cstdlib>
#include <cstring>
#include <map>

enum cudaError_t { cudaSuccess = 0, cudaErrorMemoryAllocation = 2, cudaErrorLaunchFailure = 719 };
enum cudaMemcpyKind { cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDefault = 4 };
typedef struct CUstream_st *cudaStream_t;

namespace fake {
enum Kind { DEV, HOST };
struct State {
    long allocs = 0;    // allocation calls so far
    long fail_at = -1;  // the allocation call (0-based) that fails, -1: none
    cudaError_t last = cudaSuccess;
    std::map<void *, Kind> live;
    long bad_frees = 0; // frees of a pointer that is not live, or with the other kind's call
    long syncs = 0;
    bool fail_sync = false; // the next stream synchronisation reports an earlier launch's failure
    long copies = 0;        // copy calls so far
    long fail_copy_at = -1; // the copy call (0-based) that fails, -1: none
    long by_kind[5] = {};   // copies made, by cudaMemcpyKind
};
inline State &st() {
    static State s;
    return s;
}
inline cudaError_t alloc(void **p, size_t bytes, Kind k) {
    if (st().allocs++ == st().fail_at) {
        *p = (void *)0x1; // the runtime leaves no promise about *p on failure
        return st().last = cudaErrorMemoryAllocation;
    }
    *p = malloc(bytes ? bytes : 1);
    st().live[*p] = k;
    return cudaSuccess;
}
inline cudaError_t copy(void *dst, const void *src, size_t n, cudaMemcpyKind k) {
    if (st().copies++ == st().fail_copy_at) return st().last = cudaErrorLaunchFailure;
    st().by_kind[k]++;
    memcpy(dst, src, n);
    return cudaSuccess;
}
inline cudaError_t release(void *p, Kind k) {
    auto it = st().live.find(p);
    if (it == st().live.end() || it->second != k) {
        st().bad_frees++;
        return cudaSuccess;
    }
    st().live.erase(it);
    free(p);
    return cudaSuccess;
}
} // namespace fake

inline cudaError_t cudaMalloc(void **p, size_t bytes) { return fake::alloc(p, bytes, fake::DEV); }
inline cudaError_t cudaMallocHost(void **p, size_t bytes) { return fake::alloc(p, bytes, fake::HOST); }
inline cudaError_t cudaFree(void *p) { return fake::release(p, fake::DEV); }
inline cudaError_t cudaFreeHost(void *p) { return fake::release(p, fake::HOST); }
inline cudaError_t cudaMemcpyAsync(void *dst, const void *src, size_t n, cudaMemcpyKind k, cudaStream_t) { return fake::copy(dst, src, n, k); }
inline cudaError_t cudaMemcpy(void *dst, const void *src, size_t n, cudaMemcpyKind k) { return fake::copy(dst, src, n, k); }
inline cudaError_t cudaMemsetAsync(void *p, int v, size_t n, cudaStream_t) {
    memset(p, v, n);
    return cudaSuccess;
}
inline cudaError_t cudaStreamSynchronize(cudaStream_t) {
    fake::st().syncs++;
    if (fake::st().fail_sync) {
        fake::st().fail_sync = false;
        return fake::st().last = cudaErrorLaunchFailure;
    }
    return cudaSuccess;
}
inline cudaError_t cudaGetLastError() {
    const cudaError_t e = fake::st().last;
    fake::st().last = cudaSuccess;
    return e;
}
