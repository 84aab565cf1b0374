// Owners of the context's grow-only buffers (ctx.cu): one device (cudaMalloc) or pinned host (cudaMallocHost)
// allocation each, freed by the destructor.  It needs nothing but the runtime API, so that a host test can build it
// against a fake runtime (tests/host/test_devbuf_host.cpp).
//
// A growth that fails leaves the runtime's last error cleared: every launcher returns cudaGetLastError(), and an
// allocation the driver refused must not fail the next batch, whose kernels ran.
#pragma once
#include <cuda_runtime_api.h>

namespace devbuf {

enum Mem { DEVICE, PINNED };

// One allocation and its size in bytes; move-only.
class Raw {
  public:
    Raw(const Raw &) = delete;
    Raw &operator=(const Raw &) = delete;
    Raw(Raw &&o) noexcept : p_(o.p_), bytes_(o.bytes_), mem_(o.mem_) { o.p_ = nullptr, o.bytes_ = 0; }
    Raw &operator=(Raw &&o) noexcept {
        if (this != &o) {
            reset();
            p_ = o.p_, bytes_ = o.bytes_, mem_ = o.mem_;
            o.p_ = nullptr, o.bytes_ = 0;
        }
        return *this;
    }
    ~Raw() { reset(); }

    size_t size() const { return bytes_; }

    void reset() {
        if (p_) dealloc(p_);
        p_ = nullptr, bytes_ = 0;
    }

    // Discarding growth to `bytes`, unless it holds as many already.  The old allocation is freed before the new one
    // is made, so the peak is the larger of the two.  false: empty, size 0.
    bool grow(size_t bytes) {
        if (bytes <= bytes_) return true;
        reset();
        if (!alloc(&p_, bytes)) return false;
        bytes_ = bytes;
        return true;
    }

    // Replacing growth to `bytes`, unless it holds as many already: the new allocation is made first, the first `keep`
    // bytes are copied to it on `st`, and the old one is freed once `st` is done with it.  On failure it is unchanged
    // and the result says why: cudaErrorMemoryAllocation (last error cleared) when the allocation was refused, else
    // the error of the copy or of the stream, which may be an earlier launch's and is left for the caller to report.
    cudaError_t grow_keep(size_t bytes, size_t keep, cudaStream_t st) {
        if (bytes <= bytes_) return cudaSuccess;
        void *q = nullptr;
        if (!alloc(&q, bytes)) return cudaErrorMemoryAllocation;
        if (p_) {
            cudaError_t e = keep ? cudaMemcpyAsync(q, p_, keep, cudaMemcpyDefault, st) : cudaSuccess;
            if (e == cudaSuccess) e = cudaStreamSynchronize(st);
            if (e != cudaSuccess) {
                dealloc(q);
                return e;
            }
        }
        reset();
        p_ = q, bytes_ = bytes;
        return cudaSuccess;
    }

  protected:
    explicit Raw(Mem m, void *p = nullptr, size_t bytes = 0) : p_(p), bytes_(bytes), mem_(m) {}
    void *p_;
    size_t bytes_;

  private:
    Mem mem_;

    bool alloc(void **p, size_t bytes) {
        if ((mem_ == PINNED ? cudaMallocHost(p, bytes) : cudaMalloc(p, bytes)) == cudaSuccess) return true;
        *p = nullptr;
        cudaGetLastError();
        return false;
    }
    void dealloc(void *p) { mem_ == PINNED ? cudaFreeHost(p) : cudaFree(p); }
};

// Used where a T * is: converts to the pointer it holds (nullptr while empty).
template <typename T, Mem M = DEVICE>
class Buf : public Raw {
  public:
    Buf() : Raw(M) {}
    Buf(T *p, size_t bytes) : Raw(M, p, bytes) {} // takes over an allocation of this kind
    operator T *() const { return (T *)p_; }
    T *get() const { return (T *)p_; }
    T *release() { // gives the allocation up without freeing it
        T *p = (T *)p_;
        p_ = nullptr, bytes_ = 0;
        return p;
    }
};

// A member of a set of buffers that are sized together, and the bytes it is to hold.
struct Want {
    Raw *buf;
    size_t bytes;
};

// All-or-none discarding growth of a set: every member grows to its bytes or, when one allocation fails, every member
// is freed, so that the set is whole at its new sizes or empty.
template <size_t N>
bool grow_all(const Want (&set)[N]) {
    for (const Want &w : set)
        if (!w.buf->grow(w.bytes)) {
            for (const Want &v : set) v.buf->reset();
            return false;
        }
    return true;
}

} // namespace devbuf

template <typename T>
using DevBuf = devbuf::Buf<T, devbuf::DEVICE>;
template <typename T>
using PinnedBuf = devbuf::Buf<T, devbuf::PINNED>;
